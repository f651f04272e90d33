"""The tensor-core training path at the batch sizes it trains at (4096 rays x 64 + 128 samples and beyond), stage by stage and
teacher-forced: every record, seed, dgrad step and gradient tensor is compared with float64 arithmetic fed the kernels' OWN
inputs for that stage (the recorded activation images, mask bits, previous dgrad step, dL/draw, loss scale and dsum), so each
check measures one stage's arithmetic alone and does not inherit the rounding of the stages before it.

The stage-by-stage tests of tests/test_gpu_train.py and tests/test_gpu_shapes.py stop at 528 tiles; here the plans have 4 000 to
8 500 tiles, 8 to 36 super-tiles per CTA, ragged last CTAs and empty second tiles.  Everything runs on the device in float64,
with the records decoded there (tests/tc_records.py gather_image_t / gather_mask_t) and sums taken over row blocks.  Each
gradient tensor is also checked for SENSITIVITY: its reference with one tile's rows left out (the first tile, one in the middle,
a tile of the last CTA) must fail the gate, so that a skipped, repeated or misplaced tile cannot pass.  Measured
values are written to parity_full_plan.json under $NERF_B200_PARITY_DIR (default: <tmp>/nerf_b200_parity)."""
import json
import math
import os
import tempfile

import numpy as np
import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(ROOT, "tests", "golden")
D, SKIP, L, LV = 8, 4, 10, 4
IC = 3 + 6 * L                    # input_ch of the encoding (63)
BLOCK = 1 << 16                   # rows per float64 block: [65536 x 256] float64 = 128 MB

# rel-L2 gate of each gradient tensor against its teacher-forced float64 sum (fp32 accumulation over up to 10^6 rows), about
# three times the largest deviation measured on an H100 (DESIGN.md section 5): weights 8.5e-5 (pts_linears.0 over 8448 tiles),
# biases 3.3e-5 (alpha_linear.bias, a sum of d_sigma that cancels)
GRAD_GATE = {"weight": 2.5e-4, "bias": 1e-4}
# the rgb + disp + acc + raw loss (a raw seed of noise) cancels more in every sum: measured 6.3e-4 (pts_linears.7.weight)
SEEDS_GATE_FACTOR = {"rgb": 1.0, "all": 8.0}
# fraction of fp16 image elements allowed one ulp from the float64 value rounded once (fp32 accumulation moves a rounding)
ULP1_FRAC = 1e-2


@pytest.fixture(scope="module")
def G():
    import gpu_common
    return gpu_common


def _record(name, value):
    out_dir = os.environ.get("NERF_B200_PARITY_DIR") or os.path.join(tempfile.gettempdir(), "nerf_b200_parity")
    path = os.path.join(out_dir, "parity_full_plan.json")
    os.makedirs(out_dir, exist_ok=True)
    data = {}
    if os.path.isfile(path):
        with open(path) as f:
            data = json.load(f)
    data[name] = value
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)


# ---- cases: each exists for one property of its tile plan -------------------------------------------------------------------

def _full(p):
    return p.N == p.grid * p.rays_per_cta


# id -> (S, N on a 132-SM H100, property of the plan, net, seeds); N is searched downward from there for the card's SM count
CASES = {
    "coarse_4096x64": (64, 4096, lambda p: _full(p) and p.nst == 8, "coarse", "rgb"),
    "fine_4096x192": (192, 4096, lambda p: _full(p) and p.nst == 24, "fine", "rgb"),
    "ragged_last_cta": (192, 4000, lambda p: p.nst == 24 and p.N - (p.grid - 1) * p.rays_per_cta == 1, "fine", "rgb"),
    "empty_second_tile": (128, 924, lambda p: _full(p) and p.rays_per_cta * p.S % 256 == 128, "fine", "rgb"),
    "long_accumulation": (64, 16384, lambda p: p.n_tiles >= 8000 and p.N % p.rays_per_cta != 0, "coarse", "rgb"),
    "noviews_4096x192": (192, 4096, lambda p: _full(p) and p.nst == 24, "noviews", "rgb"),
    "all_seeds_4096x192": (192, 4096, lambda p: _full(p) and p.nst == 24, "fine", "all"),
}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _restated_plan(N, S, sms):
    import tc_records as R
    layout, _, _ = R.restate_layout(N, S, D, 27, sms)
    return R.Plan(None, N, S, None, layout=layout)


def _case_N(S, N0, prop, sms):
    for N in range(N0, 0, -1):
        if prop(_restated_plan(N, S, sms)):
            return N
    raise AssertionError(f"no ray count <= {N0} has the plan property on {sms} SMs")


def _state(kind):
    from oracle import outgrads
    trained = outgrads.trained_states(os.path.join(GOLDEN, "trained_weights.npz"))
    if kind == "noviews":
        return outgrads.noviews_from_trained(trained[1], 1), False
    return trained[0 if kind == "coarse" else 1], True


def _rays(G, N, S, views, seed):
    sb = G.synth.ray_batch("lego", N, seed=seed)
    packed = G.O.pack_rays(int(sb["H"]), int(sb["W"]), sb["K"], sb["rays"][0], sb["rays"][1], bool(sb["ndc"]), float(sb["near"]),
                           float(sb["far"]), views).astype(np.float32)
    t = np.linspace(0., 1., S, dtype=np.float32)
    z = (packed[:, 6:7] * (1 - t) + packed[:, 7:8] * t).astype(np.float32)
    z = np.sort(z + np.random.default_rng(seed).uniform(-0.01, 0.01, z.shape).astype(np.float32), -1)
    return packed, z


# ---- fp16 images against float64 ---------------------------------------------------------------------------------------------

def _gamma(K):
    """relative bound of an fp32 dot product of K exact products on the tensor cores: K/16 k16 chunks added in sequence, each
    chunk a sum of 16, every addition allowed one ulp (2^-23, truncation included)"""
    return (math.ceil(K / 16) + 16) * 2.0 ** -23


def _spacing16(x):
    """spacing of fp16 at |x| (float64): 2^(e - 10), subnormals 2^-24"""
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14))) - 10)


def _ord16(h):
    """fp16 bit patterns as integers in the order of the values (+0 and -0 both 0)"""
    b = h.view(torch.int16).to(torch.int32)
    return torch.where(b < 0, -(b & 0x7FFF), b)


class _Tally:
    """counts of one fp16 image against float64 over row blocks"""

    def __init__(self):
        self.n = self.ulp1 = self.over1 = self.tight_bad = self.loose = self.loose_bad = self.nonfinite = 0
        self.mask_n = self.mask_bad = 0
        self.max_ulp = 0

    def image(self, got, ref, bound):
        """got: fp16 [B, C] from the kernel; ref: float64 value before the fp16 rounding; bound: float64 bound of |ref - the fp32
        value the kernel rounded|.  Where bound < half an fp16 spacing of ref the kernel's value may be at most 1 ulp away;
        elsewhere (values near zero or cancelling) |got - f16(ref)| <= bound + one spacing."""
        self.nonfinite += int((~torch.isfinite(got)).sum())
        ref16 = ref.clamp(-65504.0, 65504.0).to(torch.float16)
        d = (_ord16(got) - _ord16(ref16)).abs()
        sp = _spacing16(ref)
        tight = bound < 0.5 * sp
        g64, r64 = got.double(), ref16.double()
        loose_ok = (g64 - r64).abs() <= bound + torch.maximum(sp, _spacing16(g64))
        self.n += got.numel()
        self.ulp1 += int((d == 1).sum())
        self.over1 += int((d > 1).sum())
        self.max_ulp = max(self.max_ulp, int(d.max()))
        self.tight_bad += int(((d > 1) & tight).sum())
        self.loose += int((~tight).sum())
        self.loose_bad += int((~tight & ~loose_ok).sum())

    def mask(self, bits, pre, bound):
        """bits: the kernel's 'positive' mask; where |pre| > bound the sign of the float64 pre-activation is certain"""
        sure = pre.abs() > bound
        self.mask_n += int(sure.sum())
        self.mask_bad += int(((bits != (pre > 0)) & sure).sum())

    def stats(self):
        s = {"n": self.n, "ulp1_frac": self.ulp1 / max(self.n, 1), "over1": self.over1, "max_ulp": self.max_ulp,
             "loose_frac": self.loose / max(self.n, 1), "tight_bad": self.tight_bad, "loose_bad": self.loose_bad,
             "nonfinite": self.nonfinite}
        if self.mask_n:
            s.update(mask_certain=self.mask_n, mask_bad=self.mask_bad)
        return s

    def check(self, name, fails):
        """-> the counts; appends to `fails` what is outside the rules"""
        s = self.stats()
        if self.nonfinite or self.tight_bad or self.loose_bad or self.mask_bad or s["ulp1_frac"] >= ULP1_FRAC:
            fails.append((name, s))
        return s


def _blocks(M):
    return [slice(r0, min(r0 + BLOCK, M)) for r0 in range(0, M, BLOCK)]


# ---- one case -------------------------------------------------------------------------------------------------------------------

class _Pass:
    """the kernels' own records and workspace values of one training-mode pass + tensor-core backward, decoded on the device"""


def _run(G, case):
    import tc_records as R
    from oracle import outgrads
    from oracle import tc_emul as E
    S, N0, prop, kind, seeds_kind = CASES[case]
    sms = _sms()
    N = _case_N(S, N0, prop, sms)
    state, views = _state(kind)
    net = G.make_net(state, use_viewdirs=views)
    packed, z = _rays(G, N, S, views, seed=N % 97)
    rays, zd = G.dev(packed), G.dev(z)
    stats = {"N": N, "S": S, "sms": sms}
    torch.cuda.reset_peak_memory_stats()
    P = _Pass()
    P.fails, P.mem0 = [], torch.cuda.memory_allocated()
    # training mode computes what inference computes, bit for bit
    o_inf, _, _ = G.march(net, rays, zd, train=False)
    o, act, mask = G.march(net, rays, zd, train=True)
    for k in ("rgb", "disp", "acc", "w", "raw"):
        assert torch.equal(o_inf[k].view(torch.int32), o[k].view(torch.int32)), k
    del o_inf
    plan = R.Plan(G._lib.load(), N, S, net.net_params())
    assert prop(plan), (case, plan.grid, plan.rays_per_cta, plan.nst)
    stats.update(grid=plan.grid, rays_per_cta=plan.rays_per_cta, nst=plan.nst, n_tiles=plan.n_tiles)
    M = N * S
    rng = np.random.default_rng(N)
    if seeds_kind == "rgb":
        seeds = G.dev(((rng.random((N, 3), dtype=np.float32) - 0.5) * (4.0 / (3 * N))).astype(np.float32))
    else:                                   # disp seeded where acc > 0.05: disp = acc / depth is NaN on empty rays, ill-conditioned near them
        on = (o["acc"].cpu().numpy() > 0.05).astype(np.float32)
        sd_ = {"rgb_map": rng.standard_normal((N, 3)) * 1e-3, "disp_map": rng.standard_normal(N) * 1e-2 * on,
               "acc_map": rng.standard_normal(N) * 1e-2, "raw": rng.standard_normal((N, S, 4)) * 1e-4}
        seeds = {k: G.dev(v.astype(np.float32)) for k, v in sd_.items()}
    grads, ws = G.march_bwd_tc(net, rays, zd, o["raw"], act, mask, seeds, on_device=True)

    P.N, P.S, P.M, P.views, P.plan = N, S, M, views, plan
    P.gate_factor = SEEDS_GATE_FACTOR[seeds_kind]
    P.d_raw = ws[plan.off_draw:plan.off_draw + M * 16].view(torch.float32).view(M, 4).double()
    amax = float(ws[plan.off_amax:plan.off_amax + 4].view(torch.float32)[0])
    P.scale = E.loss_scale(amax)
    # dL/draw and the loss scale (the kSeeds adjoint and the atomicMax over every seed's contribution)
    raw64, z64, d64 = o["raw"].double(), zd.double(), rays[:, 3:6].double()
    if seeds_kind == "rgb":
        assert amax == float(seeds.abs().max())
        ref_draw = E.composite_adjoint(raw64, z64, d64, seeds, True)
    else:
        ref_draw = outgrads.adjoint(raw64, z64, d64, True, seeds)
        ref_amax = outgrads.loss_scale_amax(raw64, z64, d64, True, seeds)
        stats["amax_rel"] = abs(amax - ref_amax) / ref_amax
        assert stats["amax_rel"] <= 1e-4 and E.loss_scale(amax) == E.loss_scale(ref_amax), (amax, ref_amax)
    ref_draw = ref_draw.reshape(M, 4)
    assert torch.isfinite(P.d_raw).all()
    stats["d_raw_rel"] = float((P.d_raw - ref_draw).norm() / ref_draw.norm())
    assert stats["d_raw_rel"] < 1e-4, stats
    del ref_draw, raw64
    if views:
        P.dsum = ws[plan.off_dsum:plan.off_dsum + N * 128 * 4].view(torch.float32).view(N, 128).double()
        P.encv = E.T.embed(rays[:, 8:11].double(), LV)                           # per ray
    # decoded images (fp16 on the device) and masks
    P.enc = R.gather_image_t(act, plan, plan.rec_act, 0, 64)
    P.h = [R.gather_image_t(act, plan, plan.rec_act, R.rec_act_h(l), 256) for l in range(D)]
    P.mh = [R.gather_mask_t(mask, plan, l, D) for l in range(D)]
    Gr = ws[plan.off_grad:plan.off_grad + plan.n_tiles * plan.rec_grad]
    P.step = [R.gather_image_t(Gr, plan, plan.rec_grad, R.rec_grad_step(j), 256) if (views or j >= 1) else None for j in range(D + 1)]
    if views:
        P.hv = R.gather_image_t(act, plan, plan.rec_act, R.rec_act_h(D), 128)
        P.mhv = R.gather_mask_t(mask, plan, 0, D, hv=True)
        P.d_hv = R.gather_image_t(Gr, plan, plan.rec_grad, 0, 128)
    del act, mask, ws, Gr
    P.pts = (rays[:, None, 0:3] + rays[:, None, 3:6] * zd[..., None]).reshape(-1, 3)      # the kernel's fp32 samples
    P.sd = {k: torch.from_numpy(v).to(G.DEV).double() for k, v in state.items()}
    P.w16 = {k: E.f16(v) for k, v in P.sd.items() if k.endswith("weight")}
    stats["peak_mem_gb_before_checks"] = (torch.cuda.max_memory_allocated() - P.mem0) / 2 ** 30
    return P, grads, stats


# ---- teacher-forced stages ------------------------------------------------------------------------------------------------------

def _layer_input(P, l, r):
    """the recorded input of pts layer l over rows r (float64) and its weight (fp16 values)"""
    W = P.w16[f"pts_linears.{l}.weight"]
    if l == 0:
        return P.enc[r, :IC].double(), W
    if l == SKIP + 1:
        return torch.cat([P.enc[r, :IC].double(), P.h[l - 1][r].double()], 1), W
    return P.h[l - 1][r].double(), W


def _check_forward(P, stats):
    from oracle import torch_ref as T
    blocks = _blocks(P.M)
    t = _Tally()                                                   # enc: sin / cos of the kernel's own fp32 points
    for r in blocks:
        ref = torch.nn.functional.pad(T.embed(P.pts[r].double(), L), (0, 64 - IC))
        bound = torch.full_like(ref, 4e-6)                          # fp32 sincosf + four angle doublings (csrc/fused_tc.cuh)
        bound[:, :3] = 0.0
        t.image(P.enc[r], ref, bound)
    stats["enc"] = t.check("enc", P.fails)
    for l in range(D):
        t = _Tally()
        b = P.sd[f"pts_linears.{l}.bias"]
        for r in blocks:
            x, W = _layer_input(P, l, r)
            pre = x @ W.t() + b
            bound = _gamma(W.shape[1]) * (x.abs() @ W.abs().t() + b.abs())
            t.image(P.h[l][r], torch.relu(pre), bound)
            t.mask(P.mh[l][r], pre, bound)
        stats[f"h{l}"] = t.check(f"h{l}", P.fails)
    if not P.views:
        return
    # hv through f16(feat) recomputed from the recorded h_{D-1}: feat is not recorded, a one-ulp difference of it is in the bound
    t = _Tally()
    Wf, bf = P.w16["feature_linear.weight"], P.sd["feature_linear.bias"]
    Wv16, Wv, bv = P.w16["views_linears.0.weight"][:, :256], P.sd["views_linears.0.weight"], P.sd["views_linears.0.bias"]
    vb_ray = P.encv @ Wv[:, 256:].t() + bv
    for r in blocks:
        h7 = P.h[D - 1][r].double()
        feat = h7 @ Wf.t() + bf
        feat16 = feat.clamp(-65504.0, 65504.0).to(torch.float16).double()
        dfeat = _spacing16(feat) + _gamma(256) * (h7.abs() @ Wf.abs().t() + bf.abs())
        vb = vb_ray[torch.arange(r.start, r.stop, device=h7.device) // P.S]
        pre = feat16 @ Wv16.t() + vb
        bound = _gamma(256) * (feat16.abs() @ Wv16.abs().t() + vb.abs()) + dfeat @ Wv16.abs().t() + 1e-6 * vb.abs()
        t.image(P.hv[r], torch.relu(pre), bound)
        t.mask(P.mhv[r], pre, bound)
    stats["hv"] = t.check("hv", P.fails)


def _check_backward_images(P, stats):
    blocks = _blocks(P.M)
    sc = P.scale
    # seed: d_hv (rgb_linear) or dA_{D-1} (output_linear), from the kernel's d_raw and loss scale, with the recorded mask
    t = _Tally()
    for r in blocks:
        dr = P.d_raw[r] * sc
        if P.views:
            Wr = P.sd["rgb_linear.weight"]
            ref = (dr[:, :3] @ Wr) * P.mhv[r]
            bound = _gamma(3) * (dr[:, :3].abs() @ Wr.abs())
            t.image(P.d_hv[r], ref, bound)
        else:
            Wo = P.sd["output_linear.weight"][:4]
            ref = (dr @ Wo) * P.mh[D - 1][r]
            bound = _gamma(4) * (dr.abs() @ Wo.abs())
            t.image(P.step[1][r], ref, bound)
    stats["seed"] = t.check("seed", P.fails)
    # dgrad step j from the kernel's own step j - 1 image
    for j in range(0 if P.views else 2, D + 1):
        t = _Tally()
        for r in blocks:
            if j == 0:
                x, W, extra, m = P.d_hv[r].double(), P.w16["views_linears.0.weight"][:, :256], None, None
            elif j == 1:
                x, W, m = P.step[0][r].double(), P.w16["feature_linear.weight"], P.mh[D - 1][r]
                extra = (P.d_raw[r, 3:4] * sc) * P.sd["alpha_linear.weight"]
            else:
                l = D - j
                Wl = P.w16[f"pts_linears.{l + 1}.weight"]
                x, W, extra, m = P.step[j - 1][r].double(), (Wl[:, IC:] if l + 1 == SKIP + 1 else Wl), None, P.mh[l][r]
            pre = x @ W
            mag = x.abs() @ W.abs()
            if extra is not None:
                pre, mag = pre + extra, mag + extra.abs()
            if m is not None:
                pre, mag = pre * m, mag * m
            t.image(P.step[j][r], pre, _gamma(W.shape[0]) * mag)
        stats[f"step{j}"] = t.check(f"step{j}", P.fails)


def _grad_terms(P, r):
    """every gradient tensor's sum over rows r (a slice or an index tensor), float64, from the kernels' images and d_raw"""
    inv = 1.0 / P.scale
    dr = P.d_raw[r]
    out = {}
    for l in range(D):
        dA = P.step[D - l][r].double()
        x, _ = _layer_input(P, l, r)
        out[f"pts_linears.{l}.weight"] = dA.t() @ x * inv
        out[f"pts_linears.{l}.bias"] = dA.sum(0) * inv
    h7 = P.h[D - 1][r].double()
    if P.views:
        d_feat, d_hv = P.step[0][r].double(), P.d_hv[r].double() * inv
        out["feature_linear.weight"] = d_feat.t() @ h7 * inv
        out["feature_linear.bias"] = d_feat.sum(0) * inv
        out["alpha_linear.weight"] = dr[:, 3:4].t() @ h7
        out["alpha_linear.bias"] = dr[:, 3].sum(0, keepdim=True)
        out["rgb_linear.weight"] = dr[:, :3].t() @ P.hv[r].double()
        out["rgb_linear.bias"] = dr[:, :3].sum(0)
        rows = torch.arange(r.start, r.stop, device=dr.device) if isinstance(r, slice) else r
        dbv = d_hv.sum(0)
        wv = torch.empty_like(P.sd["views_linears.0.weight"])
        wv[:, :256] = (d_hv.t() @ h7) @ P.sd["feature_linear.weight"].t() + torch.outer(dbv, P.sd["feature_linear.bias"])
        wv[:, 256:] = d_hv.t() @ P.encv[rows // P.S]
        out["views_linears.0.weight"], out["views_linears.0.bias"] = wv, dbv
    else:
        Wo = P.sd["output_linear.weight"]
        gw, gb = torch.zeros_like(Wo), torch.zeros_like(P.sd["output_linear.bias"])
        gw[:4], gb[:4] = dr.t() @ h7, dr.sum(0)
        out["output_linear.weight"], out["output_linear.bias"] = gw, gb
        out["views_linears.0.weight"] = torch.zeros_like(P.sd["views_linears.0.weight"])
        out["views_linears.0.bias"] = torch.zeros_like(P.sd["views_linears.0.bias"])
    return out


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _check_grads(P, grads, stats):
    ref = None
    for r in _blocks(P.M):
        terms = _grad_terms(P, r)
        ref = terms if ref is None else {k: ref[k] + v for k, v in terms.items()}
    if P.views:                              # the view columns from the kernel's per-ray sums of d_hv
        ref["views_linears.0.weight"][:, 256:] = P.dsum.t() @ P.encv
    assert set(ref) == set(grads)
    # tiles left out: the first and the middle tile that reach the loss (a tile whose rays miss the scene has d_raw = 0 and adds
    # nothing), and the last CTA's tile with the largest sum |d_raw| (its rays may only graze the scene; if they all miss, the
    # last tile that reaches the loss)
    plan = P.plan
    weight = P.d_raw.abs().sum(1).cpu().numpy()
    w_tile = {t: float(weight[plan.rows_of_tile(t)[plan.rows_of_tile(t) >= 0]].sum()) for t in plan.valid_tiles()}
    valid = [t for t, w in w_tile.items() if w > 0]
    last_cta = [t for t in valid if t // (2 * plan.nst) == plan.grid - 1]
    tiles = {"first": valid[0], "middle": valid[len(valid) // 2], "last_cta": max(last_cta, key=w_tile.get) if last_cta else valid[-1]}
    left_out = {}
    for tag, t in tiles.items():
        rows = plan.rows_of_tile(t)
        left_out[tag] = _grad_terms(P, torch.as_tensor(rows[rows >= 0], device=P.d_raw.device))
    dev, margins, blind = {}, {}, []
    for name, r64 in ref.items():
        g = torch.from_numpy(grads[name]).to(r64.device).double()
        assert torch.isfinite(g).all(), name
        if float(r64.abs().max()) == 0.0:                        # views_linears.0 of a net without view directions
            assert not g.any(), name
            continue
        gate = GRAD_GATE[name.rsplit(".", 1)[1]] * P.gate_factor
        dev[name] = _rel(g, r64)
        if dev[name] >= gate:
            P.fails.append((name, dev[name], gate))
        margins[name] = {tag: _rel(r64 - lo[name], r64) / gate for tag, lo in left_out.items()}
        if min(margins[name].values()) <= 1.0:
            blind.append((name, dev[name], margins[name]))
    stats["grad_dev"], stats["tile_margin"] = dev, margins
    stats["tiles_left_out"], stats["last_tile_in_last_cta"] = tiles, bool(last_cta)
    stats["grad_dev_max"] = max(dev.values())
    stats["tile_margin_min"] = min(min(m.values()) for m in margins.values())
    return dev, blind


@pytest.mark.parametrize("case", list(CASES))
def test_full_plan_stages(G, case):
    """training = inference bit for bit; dL/draw and the loss scale; every fp16 record, seed and dgrad step within one ulp of the
    teacher-forced float64 value (the mask bits equal to its sign where the sign is certain); every gradient tensor within
    GRAD_GATE of its teacher-forced float64 sum, and a reference missing any one of three tiles outside it"""
    P, grads, stats = _run(G, case)
    try:
        _check_forward(P, stats)
        _check_backward_images(P, stats)
        dev, blind = _check_grads(P, grads, stats)
    finally:
        stats["peak_mem_gb"] = (torch.cuda.max_memory_allocated() - P.mem0) / 2 ** 30
        _record(case, stats)
    assert not P.fails, ("fp16 images, mask bits or gradient tensors outside the rules", P.fails)
    assert not blind, ("the gate cannot see a missing tile in these tensors (name, deviation, margins)", blind)
