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

    def __init__(self, lib, N, S, net_params):
        out = (C.c_int64 * 12)()
        rc = lib.nerf_b200_march_bwd_tc_layout(N, S, C.byref(net_params), out)
        assert rc == 0, lib.nerf_b200_last_error()
        (self.off_draw, self.off_grad, self.rec_act, self.rec_mask, self.rec_grad, self.grid, self.rays_per_cta, self.nst,
         self.n_tiles, self.off_amax, self.off_dsum, self.off_partial) = [int(v) for v in out]
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
