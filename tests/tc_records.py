"""numpy decoding of the per-tile records of the training-mode pass / tensor-core backward (csrc/train_common.cuh),
for the -m gpu parity tests."""
import ctypes as C

import numpy as np


def img_index(Ccols):
    """element (fp16) index of (row r, column col) inside a [128 x Ccols] tile image"""
    r = np.arange(128)[:, None]
    col = np.arange(Ccols)[None, :]
    off = ((r >> 6) * (Ccols >> 6) * 8192 + (col >> 6) * 8192 + ((r & 63) >> 3) * 1024 + (r & 7) * 128
           + ((((col & 63) >> 3) ^ (r & 7)) << 4) + (col & 7) * 2)                  # csrc/train_common.cuh: img_off
    return off // 2


def rec_act_h(l):
    """byte offset of h_l (l < D; l = D: hv) inside an activation record"""
    return 16384 + l * 65536


def rec_grad_step(j):
    """byte offset of dgrad step j's output inside a gradient record"""
    return 32768 + j * 65536


def restate_layout(N, S, D, input_ch_views, sms):
    """csrc/train_common.cuh make_tile_plan and capi.cu make_bwd_layout restated -> the 12 values of
    nerf_b200_march_bwd_tc_layout (Plan's order), nerf_b200_march_bwd_tc_workspace_bytes and nerf_b200_train_record_bytes"""
    want = (N * S + 255) // 256
    grid = max(min(want, sms, N), 1)
    rpc = -(-N // grid)
    grid = -(-N // rpc)
    nst = (rpc * S + 255) // 256
    n_tiles = grid * nst * 2
    rec_act, rec_mask, rec_grad = 16384 + D * 65536 + 32768, D * 4096 + 2048, 32768 + (D + 1) * 65536

    def up(x):
        return (x + 1023) & ~1023
    off_amax = 0
    off_draw = up(off_amax + 256)
    off_encv = up(off_draw + N * S * 16)
    off_dsum = up(off_encv + N * max(input_ch_views, 1) * 4)
    off_gv = up(off_dsum + N * 128 * 4)
    off_partial = up(off_gv + (128 * 256 + 128) * 4)
    off_grad = up(off_partial + sms * 256 * 256 * 4)
    total = up(off_grad + n_tiles * rec_grad)
    layout = (off_draw, off_grad, rec_act, rec_mask, rec_grad, grid, rpc, nst, n_tiles, off_amax, off_dsum, off_partial)
    return layout, total + 1024, (n_tiles * rec_act, n_tiles * rec_mask)


class Plan:
    """tile plan of one pass: nerf_b200_march_bwd_tc_layout"""

    def __init__(self, lib, N, S, net_params, layout=None):
        """the library's layout, or (lib None) the 12 values given, e.g. restate_layout's"""
        if layout is None:
            out = (C.c_int64 * 12)()
            rc = lib.nerf_b200_march_bwd_tc_layout(N, S, C.byref(net_params), out)
            assert rc == 0, lib.nerf_b200_last_error()
            layout = out
        (self.off_draw, self.off_grad, self.rec_act, self.rec_mask, self.rec_grad, self.grid, self.rays_per_cta, self.nst,
         self.n_tiles, self.off_amax, self.off_dsum, self.off_partial) = [int(v) for v in layout]
        self.N, self.S = N, S

    def rows_of_tile(self, t):
        """global row indices of the 128 rows of tile t (-1 for rows outside the CTA's range)"""
        cta, st, X = t // (2 * self.nst), (t // 2) % self.nst, t % 2
        r0 = cta * self.rays_per_cta
        r1 = min(r0 + self.rays_per_cta, self.N)
        nrows = max(r1 - r0, 0) * self.S
        lr = st * 256 + X * 128 + np.arange(128)
        return np.where(lr < nrows, r0 * self.S + lr, -1)

    def cta_nst(self, cta):
        r0 = cta * self.rays_per_cta
        return (max(min(r0 + self.rays_per_cta, self.N) - r0, 0) * self.S + 255) // 256

    def valid_tiles(self):
        return [t for t in range(self.n_tiles) if (t // 2) % self.nst < self.cta_nst(t // (2 * self.nst))]


def gather_image(buf_u8, plan, rec_bytes, off, Ccols):
    """[M, Ccols] float32 matrix (global row order) of the image at byte offset `off` of every tile record"""
    M = plan.N * plan.S
    out = np.full((M, Ccols), np.nan, np.float32)
    half = buf_u8.view(np.float16)
    idx = img_index(Ccols)
    for t in plan.valid_tiles():
        rows = plan.rows_of_tile(t)
        base = (t * rec_bytes + off) // 2
        tile = half[base + idx].astype(np.float32)
        ok = rows >= 0
        out[rows[ok]] = tile[ok]
    return out


def plan_row_keep(plan):
    """bool [len(valid_tiles) * 128]: which rows of the valid tiles, in tile order, are rows of the batch.  The valid tiles of a
    CTA hold its rows in order and the CTAs follow each other, so the kept rows come out in global row order."""
    return np.concatenate([plan.rows_of_tile(t) >= 0 for t in plan.valid_tiles()])


def _valid_records(buf, plan, rec_bytes, off, nbytes):
    """uint8 [n_valid, nbytes]: bytes [off, off + nbytes) of every valid tile's record, from a torch uint8 buffer (any device)"""
    import torch
    recs = buf[:plan.n_tiles * rec_bytes].view(plan.n_tiles, rec_bytes)
    valid = torch.as_tensor(plan.valid_tiles(), device=buf.device)
    return recs[valid, off:off + nbytes]


def gather_image_t(buf, plan, rec_bytes, off, Ccols):
    """gather_image on a torch uint8 buffer, on its device: [M, Ccols] float16 in global row order"""
    import torch
    x = _valid_records(buf, plan, rec_bytes, off, 128 * Ccols * 2).contiguous().view(torch.float16)
    x = x.view(-1, 2, Ccols // 64, 8, 8, 8, 8)                  # [tile][half][K-block][row >> 3][row & 7][16-byte chunk][col & 7]
    r7 = torch.arange(8, device=buf.device)
    x = x[:, :, :, :, r7[:, None], r7[:, None] ^ r7[None, :], :]   # logical chunk c of row r sits at (c ^ (r & 7))
    x = x.permute(0, 1, 3, 4, 2, 5, 6).reshape(-1, Ccols)
    return x[torch.as_tensor(plan_row_keep(plan), device=buf.device)]


def gather_mask_t(buf, plan, layer, D, hv=False):
    """gather_mask on a torch uint8 buffer, on its device: [M, 256 | 128] bool, True where the pre-activation was positive"""
    import torch
    nw = 2 if hv else 4
    w = _valid_records(buf, plan, plan.rec_mask, D * 4096 if hv else layer * 4096, 2 * 128 * nw * 4).contiguous()
    w = w.view(torch.int32).view(-1, 2, 128, nw)               # [tile][column half][row][word]
    sh = 31 - torch.arange(32, device=buf.device, dtype=torch.int32)
    bits = (w[..., None] >> sh) & 1                            # column (32 b + j) of a word at bit (31 - j)
    bits = bits.permute(0, 2, 1, 3, 4).reshape(-1, 2 * nw * 32)
    return bits[torch.as_tensor(plan_row_keep(plan), device=buf.device)] == 0


def gather_mask(buf_u8, plan, layer, D, hv=False):
    """[M, 256 | 128] bool: True where the pre-activation was positive (ReLU gradient 1)"""
    M = plan.N * plan.S
    ncol = 128 if hv else 256
    out = np.zeros((M, ncol), bool)
    words = buf_u8.view(np.uint32)
    for t in plan.valid_tiles():
        rows = plan.rows_of_tile(t)
        base = t * plan.rec_mask + (D * 4096 if hv else layer * 4096)
        tile = np.zeros((128, ncol), bool)
        nw = 2 if hv else 4
        for ch in range(2):
            w = words[(base + ch * (1024 if hv else 2048)) // 4:(base + (ch + 1) * (1024 if hv else 2048)) // 4].reshape(128, nw)
            for b in range(nw):
                bits = (w[:, b][:, None] >> (31 - np.arange(32))[None, :]) & 1
                tile[:, ch * (ncol // 2) + b * 32: ch * (ncol // 2) + b * 32 + 32] = bits == 0
        ok = rows >= 0
        out[rows[ok]] = tile[ok]
    return out
