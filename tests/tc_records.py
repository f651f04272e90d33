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
