"""The tensor-core path at every network shape and sample count the library accepts, not only the 8 x 256 net with skips = [4],
63 + 27 input channels and 40..192 samples the other files test.

(a) network shapes: depth 2..8, no skip / skip 0 / skip D - 2, multires 0 (i_embed = -1) .. 10, multires_views 0 .. 10, with
    and without view directions.  Per shape: training pass = inference pass bit for bit; every record against the quantisation-
    aware restatement (oracle/tc_emul.py, oracle/noviews.py); every stage of the tensor-core backward against it; the exact
    path against a float64 autograd of the reference's network (oracle/torch_ref.mlp); tensor-core against exact gradients.
(b) sample counts and tile plans: S = 1 .. 1024, rays that straddle warps, tiles and 256-row super-tiles, one ray per CTA, CTAs
    whose rows are a multiple of 256 -- the compositing carry and the record indexing of each.
(c) the backward's limit S <= 1024 (the forward accepts up to 4096).
(d) create_nerf-shaped nets (netdepth 4 with skips = [4], i_embed = -1) through render() + loss.backward() against the
    reference's autograd (tests/golden/shapes.npz) and through FusedTrainStep.
(e) shapes only the exact path serves (netwidth 4 .. 252 other than 256, netdepth 1 and 9 .. 16, multires 11 .. 16): forward,
    run_network and both backward entry points against float64 autograd kernel by kernel, on workspaces whose contents must
    not matter; create_nerf-shaped nets through render() against the reference (tests/golden/exact_shapes.npz); and the
    refusals through render().

conftest.rel_l2 ignores non-finite entries, so every comparison first asserts that the kernel's tensors are finite (disp and its
NaN pattern excepted).  Measured deviations go to parity_shapes.json in $NERF_B200_PARITY_DIR (default: a nerf_b200_parity
directory under the system's temporary directory)."""
import json
import os
import re
import tempfile
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_golden, rel_l2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def G():
    import gpu_common
    return gpu_common


def _record(name, value):
    out_dir = os.environ.get("NERF_B200_PARITY_DIR") or os.path.join(tempfile.gettempdir(), "nerf_b200_parity")
    path = os.path.join(out_dir, "parity_shapes.json")
    os.makedirs(out_dir, exist_ok=True)
    data = {}
    if os.path.isfile(path):
        with open(path) as f:
            data = json.load(f)
    data[name] = value
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)


# id, D, skips, multires, multires_views (None: no view directions), output_ch, parameter seed.  The seeds give batches whose
# rays are neither all empty nor all opaque where the shape allows it: an empty batch has no gradient (rgb_map = 1), and on
# opaque rays the gradients cancel.  Without a skip in the middle, 8 random layers leave no such seed (d8_noskip, d8_s0: opaque).
SHAPES = [("d2_noenc", 2, [], 0, 0, 5, 2), ("d2_s0", 2, [0], 4, 1, 5, 0), ("d3_s0_v63", 3, [0], 5, 10, 5, 0),
          ("d4_s4", 4, [4], 10, 4, 5, 1), ("d6_s4", 6, [4], 10, 4, 5, 0), ("d7_s2", 7, [2], 8, 4, 5, 2),
          ("d8_noskip", 8, [], 10, 4, 5, 9), ("d8_s0", 8, [0], 10, 4, 5, 8), ("d8_s6", 8, [6], 10, 4, 5, 0),
          ("nv_d3", 3, [], 6, None, 4, 0), ("nv_d6_s4", 6, [4], 10, None, 5, 0), ("nv_d2_s0_noenc", 2, [0], 0, None, 5, 0)]


class Shape(types.SimpleNamespace):
    """one network: state dict, the library's NeRF and what the restatements need"""


def _shape(G, sid, D, skips, L, Lv, out_ch, seed=0, sharpen=False, W=256):
    from nerf_pytorch_b200.api import effective_skip
    from oracle import noviews, tc_emul
    ic = tc_emul.input_ch(L)
    views = Lv is not None
    icv = tc_emul.input_ch(Lv) if views else 0
    if views:
        state = G.synth.nerf_state(seed, sharpen, D=D, W=W, input_ch=ic, input_ch_views=icv, skips=skips)
    else:
        state = noviews.nerf_state_noviews(seed, sharpen, output_ch=out_ch, D=D, W=W, input_ch=ic, skips=skips)
    net = G.make_net(state, use_viewdirs=views, output_ch=out_ch, D=D, skips=skips, input_ch=ic, input_ch_views=icv, W=W)
    return Shape(id=sid, W=W, D=D, skip=effective_skip(skips, D), L=L, Lv=Lv if views else 0, views=views, ic=ic, icv=icv,
                 state=state, net=net)


def _rays(G, sh, N, S, seed, scene="lego"):
    sb = G.synth.ray_batch(scene, N, seed=seed)
    packed = G.O.pack_rays(int(sb["H"]), int(sb["W"]), sb["K"], sb["rays"][0], sb["rays"][1], bool(sb["ndc"]), float(sb["near"]),
                           float(sb["far"]), sh.views).astype(np.float32)
    t = np.linspace(0., 1., S, dtype=np.float32)
    z = (packed[:, 6:7] * (1 - t) + packed[:, 7:8] * t).astype(np.float32)
    if S > 1:                                    # uneven spacing like a fine pass
        z = np.sort(z + np.random.default_rng(seed).uniform(-0.01, 0.01, z.shape).astype(np.float32), -1)
    return packed, z


def _pts(packed, z):
    """the samples as the kernels form them: o + d z in fp32, product and sum each rounded"""
    o, d, zz = (torch.from_numpy(a) for a in (packed[:, None, 0:3], packed[:, None, 3:6], z[..., None]))
    return (o + d * zz).reshape(-1, 3)


def _vd_rows(packed, S):
    return torch.from_numpy(np.repeat(packed[:, 8:11], S, 0))


def _finite(name, a):
    a = np.asarray(a)
    assert np.isfinite(a).all(), (name, int((~np.isfinite(a)).sum()))


def _same_nan(name, a, b):
    """disp: the NaN pattern must be the reference's, the rest within tol -> rel-L2 of the finite entries"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.array_equal(np.isnan(a), np.isnan(b)), name
    _finite(name, a[~np.isnan(a)])
    return rel_l2(a, b)


# ---- decoding the records of one training-mode pass ------------------------------------------------------------------------

def _decode(G, sh, act, mask, N, S):
    import tc_records as R
    plan = R.Plan(G._lib.load(), N, S, sh.net.net_params())
    A, Mk = act.cpu().numpy(), mask.cpu().numpy()
    rec = {"enc": R.gather_image(A, plan, plan.rec_act, 0, 64),
           "h": [R.gather_image(A, plan, plan.rec_act, R.rec_act_h(l), 256) for l in range(sh.D)],
           "mh": [R.gather_mask(Mk, plan, l, sh.D) for l in range(sh.D)]}
    if sh.views:
        rec["hv"] = R.gather_image(A, plan, plan.rec_act, R.rec_act_h(sh.D), 128)
        rec["mhv"] = R.gather_mask(Mk, plan, 0, sh.D, hv=True)
    return plan, rec


def _emul_forward(sh, packed, z):
    from oracle import noviews, tc_emul
    sd = {k: torch.from_numpy(v) for k, v in sh.state.items()}
    pts = _pts(packed, z)
    if sh.views:
        return tc_emul.forward(sd, pts, _vd_rows(packed, z.shape[1]), D=sh.D, skip=sh.skip, L=sh.L, Lv=sh.Lv)
    return noviews.forward_noviews(sd, pts, D=sh.D, skip=sh.skip, L=sh.L)


def _check_records(sh, rec, em, stats):
    enc = rec["enc"]
    _finite("enc", enc)
    assert not enc[:, sh.ic:].any(), "encoding columns >= input_ch must be exactly 0"
    stats["enc_close"] = float(np.mean(np.isclose(enc, em["enc64"].numpy(), rtol=2e-3, atol=1e-4)))
    assert stats["enc_close"] > 0.995, stats
    for l in range(sh.D):
        h = rec["h"][l]
        _finite(f"h{l}", h)
        stats[f"h{l}_rel"] = rel_l2(h, em["h16"][l].numpy())
        assert stats[f"h{l}_rel"] < 2e-3, (l, stats)
        stats[f"mask{l}_mismatch"] = float(np.mean(rec["mh"][l] != (h > 0)))
        assert stats[f"mask{l}_mismatch"] < 2e-4, (l, stats)          # fp16 underflow of a positive pre-activation only
    if sh.views:
        _finite("hv", rec["hv"])
        stats["hv_rel"] = rel_l2(rec["hv"], em["hv16"].numpy())
        assert stats["hv_rel"] < 2e-3, stats
        stats["maskv_mismatch"] = float(np.mean(rec["mhv"] != (rec["hv"] > 0)))
        assert stats["maskv_mismatch"] < 2e-4, stats


def _g_rgb(N, seed=11):
    rng = np.random.default_rng(seed)
    return ((rng.random((N, 3), dtype=np.float32) - 0.5) * (4.0 / (3 * N))).astype(np.float32)


def _check_bwd_stages(G, sh, packed, z, o, plan, rec, grads, ws, g_rgb, stats, seeds=None):
    """d_raw, the loss scale, the seed, every dgrad step image and every gradient tensor against the restatement"""
    import tc_records as R
    from oracle import noviews, outgrads, tc_emul as E
    N, S = z.shape
    M = N * S
    raw = o["raw"].cpu()
    d_raw = ws[plan.off_draw:plan.off_draw + M * 16].view(np.float32).reshape(M, 4)
    _finite("d_raw", d_raw)
    amax = float(ws[plan.off_amax:plan.off_amax + 4].view(np.float32)[0])
    zt, dt = torch.from_numpy(z), torch.from_numpy(packed[:, 3:6])
    if seeds is None:
        assert amax == float(np.abs(g_rgb).max())
        ref_draw = E.composite_adjoint(raw, zt, dt, torch.from_numpy(g_rgb), True)
    else:
        sc = {k: v.cpu() for k, v in seeds.items()}
        ref_draw = outgrads.adjoint(raw, zt, dt, True, sc)
        ref_amax = outgrads.loss_scale_amax(raw, zt, dt, True, sc)
        assert abs(amax - ref_amax) <= 1e-4 * ref_amax and E.loss_scale(amax) == E.loss_scale(ref_amax), (amax, ref_amax)
    stats["d_raw_rel"] = rel_l2(d_raw, ref_draw.numpy().reshape(M, 4))
    assert stats["d_raw_rel"] < 1e-4, stats
    scale = E.loss_scale(amax)
    acts = {"enc16": torch.from_numpy(rec["enc"]).double(), "h16": [torch.from_numpy(h).double() for h in rec["h"]]}
    masks = {"h": [torch.from_numpy(m).double() for m in rec["mh"]]}
    sd = {k: torch.from_numpy(v) for k, v in sh.state.items()}
    d64 = torch.from_numpy(d_raw).double()
    if sh.views:
        acts["hv16"] = torch.from_numpy(rec["hv"]).double()
        acts["encv"] = E.T.embed(_vd_rows(packed, S), sh.Lv).double()
        masks["hv"] = torch.from_numpy(rec["mhv"]).double()
        ref_g, st = E.backward(sd, acts, masks, d64, scale, torch.arange(M) // S, N, D=sh.D, skip=sh.skip, L=sh.L)
    else:
        ref_g, st = noviews.backward_noviews(sd, acts, masks, d64, scale, D=sh.D, skip=sh.skip, L=sh.L)
    Gr = ws[plan.off_grad:plan.off_grad + plan.n_tiles * plan.rec_grad]
    if sh.views:
        d_hv = R.gather_image(Gr, plan, plan.rec_grad, 0, 128)
        _finite("d_hv", d_hv)
        stats["d_hv_rel"] = rel_l2(d_hv, st["d_hv16"].numpy())
        assert stats["d_hv_rel"] < 1e-3, stats
    for j in range(0 if sh.views else 1, sh.D + 1):      # step 0: d_feat; step j >= 1: dA of pts layer D - j
        img = R.gather_image(Gr, plan, plan.rec_grad, R.rec_grad_step(j), 256)
        _finite(f"step{j}", img)
        stats[f"step{j}_rel"] = rel_l2(img, st["step"][j].numpy())
        assert stats[f"step{j}_rel"] < 2e-3, (j, stats)
    assert set(ref_g) == set(grads)
    for name, ref in ref_g.items():
        _finite(name, grads[name])
        if float(ref.abs().max()) == 0.0:        # views_linears.0 of a net without view directions: not on the loss's graph
            assert not grads[name].any(), name
            continue
        e = rel_l2(grads[name].reshape(-1), ref.numpy().reshape(-1))
        stats["g_" + name] = e
        assert e < 2e-3, (name, e, stats)


# ---- (a) network shapes ---------------------------------------------------------------------------------------------------

def _exact_reference(sh, packed, z, g_rgb, dtype=torch.float64, seeds=None):
    """autograd of the reference's network (oracle/torch_ref.mlp) and raw2outputs on the kernels' fp32 samples, in float64 (the
    reference) or float32 (how far fp32 arithmetic itself is from it) -> (raw [M,4], maps, grads by state_dict key).  The loss
    is sum(rgb_map * g_rgb), or with `seeds` (rgb_map, disp_map, acc_map, raw -> gradient) the sum of each output times its seed,
    whose float64 dL/draw tests/test_outgrads_cpu.py pins oracle/outgrads.adjoint to.  disp is NaN on empty rays: a zero seed
    keeps it off the loss there."""
    from oracle import torch_ref as T
    N, S = z.shape
    sd = {k: torch.from_numpy(v).to(dtype).requires_grad_(True) for k, v in sh.state.items()}
    x = T.embed(_pts(packed, z).to(dtype), sh.L)
    if sh.views:
        x = torch.cat([x, T.embed(_vd_rows(packed, S).to(dtype), sh.Lv)], -1)
    raw = T.mlp(sd, x, ic=sh.ic, icv=sh.icv, skip=sh.skip, D=sh.D)
    rgb, disp, acc, w = T.composite(raw.reshape(N, S, 4), torch.from_numpy(z).to(dtype), torch.from_numpy(packed[:, 3:6]).to(dtype), True)
    if seeds is None:
        (rgb * torch.from_numpy(g_rgb).to(dtype)).sum().backward()
    else:
        sd_ = {k: v.to(dtype) for k, v in seeds.items()}
        disp_on = torch.where(sd_["disp_map"] != 0, disp, torch.zeros_like(disp))
        ((rgb * sd_["rgb_map"]).sum() + (disp_on * sd_["disp_map"]).sum() + (acc * sd_["acc_map"]).sum() +
         (raw.reshape(N, S, 4) * sd_["raw"]).sum()).backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)).numpy() for k, v in sd.items()}
    maps = {"rgb": rgb.detach().numpy(), "disp": disp.detach().numpy(), "acc": acc.detach().numpy(), "w": w.detach().numpy()}
    return raw.detach().numpy(), maps, grads


@pytest.mark.parametrize("sid,D,skips,L,Lv,out_ch,seed", SHAPES, ids=[s[0] for s in SHAPES])
def test_network_shape(G, sid, D, skips, L, Lv, out_ch, seed):
    N, S = 37, 70
    sh = _shape(G, sid, D, skips, L, Lv, out_ch, seed=seed)
    packed, z = _rays(G, sh, N, S, seed=5)
    rays, zd = G.dev(packed), G.dev(z)
    stats = {}
    # training forward = inference forward, bit for bit (disp is NaN where acc = 0)
    o_inf, _, _ = G.march(sh.net, rays, zd, train=False, L=sh.L, Lv=sh.Lv)
    o, act, mask = G.march(sh.net, rays, zd, train=True, L=sh.L, Lv=sh.Lv)
    for k in ("rgb", "disp", "acc", "w", "raw"):
        assert torch.equal(o_inf[k].view(torch.int32), o[k].view(torch.int32)), k
    for k in ("rgb", "acc", "w", "raw"):
        _finite(k, o[k].cpu().numpy())
    # records
    plan, rec = _decode(G, sh, act, mask, N, S)
    em = _emul_forward(sh, packed, z)
    _check_records(sh, rec, em, stats)
    stats["raw_rel"] = rel_l2(o["raw"].cpu().numpy().reshape(-1, 4), em["raw"].numpy())
    assert stats["raw_rel"] < 2e-3, stats
    # backward stages
    g_rgb = _g_rgb(N)
    grads_tc, ws = G.march_bwd_tc(sh.net, rays, zd, o["raw"], act, mask, G.dev(g_rgb), L=sh.L, Lv=sh.Lv)
    _check_bwd_stages(G, sh, packed, z, o, plan, rec, grads_tc, ws, g_rgb, stats)
    # exact path against the float64 reference
    # each gate is today's fp32 gate plus twice the distance of the same autograd in float32 from float64 (the outgrads rule):
    # large densities and, on opaque rays, cancelling gradient terms make some shapes' fp32 results less certain than others
    o_ex, _, _ = G.march(sh.net, rays, zd, train=False, L=sh.L, Lv=sh.Lv, precision=G._lib.PREC_FP32)
    raw_ref, maps_ref, g_ref = _exact_reference(sh, packed, z, g_rgb)
    raw32, maps32, g32 = _exact_reference(sh, packed, z, g_rgb, torch.float32)
    _finite("exact raw", o_ex["raw"].cpu().numpy())
    stats["exact_raw_rel"] = rel_l2(o_ex["raw"].cpu().numpy().reshape(-1, 4), raw_ref)
    stats["cond_raw"] = rel_l2(raw32, raw_ref)
    assert stats["exact_raw_rel"] <= 2e-5 + 2 * stats["cond_raw"], stats
    for k in ("rgb", "disp", "acc", "w"):
        v = o_ex[k].cpu().numpy()
        stats[f"exact_{k}_rel"] = _same_nan("exact disp", v, maps_ref[k]) if k == "disp" else (_finite(k, v) or rel_l2(v, maps_ref[k]))
        stats[f"cond_{k}"] = rel_l2(maps32[k], maps_ref[k])
        assert stats[f"exact_{k}_rel"] <= 2e-5 + 2 * stats[f"cond_{k}"], (k, stats)
    grads_ex = G.march_bwd_exact(sh.net, rays, zd, G.dev(g_rgb), L=sh.L, Lv=sh.Lv)
    # A tensor whose float32 autograd is already > 1e-4 from float64 (alpha_linear over the opaque rays of d8_noskip / d8_s0)
    # cannot be pinned by one fp32 evaluation against another: it is recorded, not gated, here and in the tensor-core budget.
    devs = {}
    for name, ref in g_ref.items():
        _finite("exact " + name, grads_ex[name])
        if not ref.any():
            assert not grads_ex[name].any() and not grads_tc[name].any(), name
            continue
        stats["exact_g_" + name] = rel_l2(grads_ex[name], ref)
        stats["cond_g_" + name] = rel_l2(g32[name], ref)
        stats["tc_vs_exact_" + name] = rel_l2(grads_tc[name], grads_ex[name])
        if stats["cond_g_" + name] <= 1e-4:
            assert stats["exact_g_" + name] < 1e-4 + 2 * stats["cond_g_" + name], (name, stats)
            devs[name] = stats["tc_vs_exact_" + name]
    assert devs, "the loss has no well-conditioned gradient"
    assert float(np.median([stats["exact_g_" + k] for k in devs])) < 1e-4, stats
    # tensor-core against exact gradients: the end-to-end budget of tests/test_gpu_train.py
    med, worst = float(np.median(list(devs.values()))), max(devs.values())
    stats.update(tc_vs_exact_median=med, tc_vs_exact_worst=worst)
    _record(f"shape_{sid}", stats)
    assert med < 3e-2 and worst < 1.5e-1, (med, worst, devs)


# ---- (b) sample counts and tile plans ---------------------------------------------------------------------------------------

def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# id -> (N, S, the plan property the case is there for)
def _sample_cases():
    sms = _sms()
    return {
        "S1_N1": (1, 1, lambda p: p.grid == 1 and p.nst == 1),
        "S1_N7": (7, 1, lambda p: p.grid == 1 and p.rays_per_cta == 7),
        "S2": (50, 2, lambda p: p.rays_per_cta * 2 <= 256),
        "S33": (40, 33, lambda p: p.rays_per_cta * 33 > 32),
        "S127": (20, 127, lambda p: p.rays_per_cta * 127 > 128),
        "S129": (20, 129, lambda p: p.rays_per_cta * 129 > 128),
        "S256_one_ray_per_cta": (sms, 256, lambda p: p.grid == sms and p.rays_per_cta == 1 and p.nst == 1),
        "S300": (5, 300, lambda p: p.grid == 5 and p.rays_per_cta == 1 and p.nst == 2),      # grid clamped to N
        "S513": (5, 513, lambda p: p.rays_per_cta == 1 and p.nst == 3),
        "S1024": (5, 1024, lambda p: p.rays_per_cta == 1 and p.nst == 4),
        "rows_multiple_of_256": (4 * sms, 128, lambda p: p.grid == sms and p.rays_per_cta * 128 % 256 == 0 and p.nst == 2),
    }


SAMPLE_IDS = ["S1_N1", "S1_N7", "S2", "S33", "S127", "S129", "S256_one_ray_per_cta", "S300", "S513", "S1024", "rows_multiple_of_256"]


@pytest.mark.parametrize("views", [True, False], ids=["views", "noviews"])
@pytest.mark.parametrize("case", SAMPLE_IDS)
def test_sample_count(G, case, views):
    from oracle import torch_ref as T
    N, S, prop = _sample_cases()[case]
    # the no-view head sharpened (SURVEY 8d(ii)): at the default init its rays are nearly transparent (acc ~ 1e-4), where
    # alpha = 1 - exp(-sigma delta) is all cancellation in fp32
    sh = _shape(G, "d8_s4", 8, [4], 10, 4 if views else None, 5, seed=1, sharpen=not views)
    packed, z = _rays(G, sh, N, S, seed=9)
    rays, zd = G.dev(packed), G.dev(z)
    o, act, mask = G.march(sh.net, rays, zd, train=True)
    plan, rec = _decode(G, sh, act, mask, N, S)
    assert prop(plan), (case, plan.grid, plan.rays_per_cta, plan.nst)
    stats = {"grid": plan.grid, "rays_per_cta": plan.rays_per_cta, "nst": plan.nst}
    # the maps and weights are the float64 composite of the kernel's own raw
    raw = o["raw"].cpu().numpy()
    _finite("raw", raw)
    # 1e-5 plus twice the distance of the same composite in float32: on nearly transparent rays alpha = 1 - exp(-sigma delta)
    # cancels in fp32 (the reference's arithmetic), and acc sums S such terms
    ref = dict(zip(("rgb", "disp", "acc", "w"), (t.numpy() for t in T.composite(torch.from_numpy(raw).double(), torch.from_numpy(z).double(),
                                                                               torch.from_numpy(packed[:, 3:6]).double(), True))))
    r32 = dict(zip(("rgb", "disp", "acc", "w"), (t.numpy() for t in T.composite(torch.from_numpy(raw), torch.from_numpy(z),
                                                                               torch.from_numpy(packed[:, 3:6]), True))))
    for k in ("rgb", "disp", "acc", "w"):
        v = o[k].cpu().numpy()
        stats[f"{k}_rel"] = _same_nan(k, v, ref[k]) if k == "disp" else (_finite(k, v) or rel_l2(v, ref[k]))
        stats[f"{k}_cond"] = rel_l2(r32[k], ref[k])
        assert stats[f"{k}_rel"] <= 1e-5 + 2 * stats[f"{k}_cond"], (k, stats)
    # records and every backward stage
    em = _emul_forward(sh, packed, z)
    _check_records(sh, rec, em, stats)
    g_rgb = _g_rgb(N)
    grads, ws = G.march_bwd_tc(sh.net, rays, zd, o["raw"], act, mask, G.dev(g_rgb))
    _check_bwd_stages(G, sh, packed, z, o, plan, rec, grads, ws, g_rgb, stats)
    _record(f"samples_{case}_{'views' if views else 'noviews'}", stats)


def test_all_output_seeds_at_1024_samples(G):
    """One loss on rgb + disp + acc + raw through nerf_b200_march_bwd_tc_outs with one ray over four super-tiles: dL/draw against
    the float64 adjoint (oracle/outgrads.adjoint).  The trained densities leave rays neither empty nor opaque, where an acc or
    disp gradient is more than rounding noise."""
    from oracle import outgrads
    N, S = 32, 1024
    trained = outgrads.trained_states(os.path.join(GOLDEN, "trained_weights.npz"))
    sh = _shape(G, "d8_s4", 8, [4], 10, 4, 5)
    sh.state, sh.net = trained[1], G.make_net(trained[1])
    packed, z = _rays(G, sh, N, S, seed=4)
    rays, zd = G.dev(packed), G.dev(z)
    o, act, mask = G.march(sh.net, rays, zd, train=True)
    plan, rec = _decode(G, sh, act, mask, N, S)
    assert plan.rays_per_cta == 1 and plan.nst == 4
    acc = o["acc"].cpu().numpy()
    assert ((acc > 0.05) & (acc < 0.995)).any(), acc
    rng = np.random.default_rng(4)
    seeds = {"rgb_map": rng.standard_normal((N, 3)) * 1e-3, "disp_map": rng.standard_normal(N) * 1e-2,
             "acc_map": rng.standard_normal(N) * 1e-2, "raw": rng.standard_normal((N, S, 4)) * 1e-4}
    seeds = {k: G.dev(v.astype(np.float32)) for k, v in seeds.items()}
    grads, ws = G.march_bwd_tc(sh.net, rays, zd, o["raw"], act, mask, seeds)
    stats = {}
    _check_bwd_stages(G, sh, packed, z, o, plan, rec, grads, ws, None, stats, seeds=seeds)
    _record("outs_S1024", stats)


# ---- (c) the backward's sample limit -------------------------------------------------------------------------------------

def _render_kw(G, nets, views=True, N_samples=64, N_importance=128):
    return dict(network_fn=nets[0], network_fine=nets[1], network_query_fn=G.query_fn(), N_samples=N_samples,
                N_importance=N_importance, perturb=0., white_bkgd=True, raw_noise_std=0., use_viewdirs=views, ndc=False,
                lindisp=False, near=2., far=6.)


@pytest.mark.parametrize("backward", ["tc", "exact"])
def test_backward_sample_limit(G, backward):
    """64 + 960 = 1024 fine samples train on both backward paths; 64 + 961 renders but loss.backward() raises, naming the limit,
    and leaves every parameter's .grad as it was."""
    sb = G.synth.ray_batch("lego", 16, seed=2)
    target = G.dev(np.random.default_rng(3).random((16, 3), dtype=np.float32))
    nets = [G.make_net(G.synth.nerf_state(0)), G.make_net(G.synth.nerf_state(1))]
    G.nb.set_backward(backward)
    try:
        def step(n_imp):
            rgb, _, _, ex = G.nb.render(400, 400, sb["K"], rays=G.dev(sb["rays"]), retraw=True, **_render_kw(G, nets, N_importance=n_imp))
            assert ex["raw"].shape[1] == 64 + n_imp
            return G.nb.img2mse(rgb, target) + G.nb.img2mse(ex["rgb0"], target)
        step(960).backward()
        before = [p.grad.clone() for n in nets for p in n.parameters()]
        for g in before:
            _finite("grad", g.cpu().numpy())
        assert any(float(g.abs().max()) > 0 for g in before)
        loss = step(961)
        with pytest.raises(RuntimeError, match="1024"):
            loss.backward()
        for p, g in zip([p for n in nets for p in n.parameters()], before):
            assert torch.equal(p.grad, g)
    finally:
        G.nb.set_backward("tc")


# ---- (d) create_nerf-shaped nets through the Python surface ------------------------------------------------------------------

def _fixture_nets(G, fx, case):
    """the nets of case `case` of tests/golden/shapes.npz (parameters regenerated from oracle/synth / oracle/noviews)"""
    from oracle import noviews, tc_emul
    p = f"{case}_"
    views = bool(fx[p + "use_viewdirs"])
    no_enc = int(fx[p + "i_embed"]) == -1
    L, Lv = (0, 0) if no_enc else (int(fx[p + "multires"]), int(fx[p + "multires_views"]))
    ic, icv = tc_emul.input_ch(L), (tc_emul.input_ch(Lv) if views else 0)
    nets = []
    for k, tag in enumerate(("", "_fine")):
        if k == 1 and int(fx[p + "N_importance"]) == 0:
            nets.append(None)
            continue
        D, W = int(fx[p + "netdepth" + tag]), (int(fx[p + "netwidth" + tag]) if p + "netwidth" + tag in fx else 256)
        seed = int(fx[p + "seed_w"]) + k
        if views:
            st = G.synth.nerf_state(seed, False, D=D, W=W, input_ch=ic, input_ch_views=icv, skips=(4,))
        else:
            st = noviews.nerf_state_noviews(seed, output_ch=int(fx[p + "output_ch"]), D=D, W=W, input_ch=ic, skips=(4,))
        nets.append(G.make_net(st, use_viewdirs=views, output_ch=int(fx[p + "output_ch"]), D=D, skips=[4], input_ch=ic,
                               input_ch_views=icv, W=W))
    return nets


def _fixture_query_fn(G, fx, case):
    from nerf_pytorch_b200.api import _QueryFn
    p = f"{case}_"
    i_embed, L, Lv = int(fx[p + "i_embed"]), int(fx[p + "multires"]), int(fx[p + "multires_views"])
    e, _ = G.nb.get_embedder(L, i_embed)
    ed, _ = G.nb.get_embedder(Lv, i_embed)
    return _QueryFn(e, ed, 65536, L, Lv, i_embed)


def _fixture_render(G, fx, case, prec, backward):
    p = f"{case}_"
    nets = _fixture_nets(G, fx, case)
    G.nb.set_precision(prec)
    G.nb.set_backward(backward)
    try:
        rgb, disp, acc, ex = G.nb.render(int(fx[p + "H"]), int(fx[p + "W"]), fx[p + "K"], chunk=32768, rays=G.dev(fx[p + "rays"]),
                                         ndc=bool(fx[p + "ndc"]), near=float(fx[p + "near"]), far=float(fx[p + "far"]),
                                         use_viewdirs=bool(fx[p + "use_viewdirs"]), network_fn=nets[0], network_fine=nets[1],
                                         network_query_fn=_fixture_query_fn(G, fx, case), N_samples=int(fx[p + "N_samples"]),
                                         N_importance=int(fx[p + "N_importance"]), perturb=0., white_bkgd=bool(fx[p + "white_bkgd"]),
                                         raw_noise_std=0., retraw=True)
        target = G.dev(fx[p + "target"])
        loss = G.nb.img2mse(rgb, target)
        if "rgb0" in ex:
            loss = loss + G.nb.img2mse(ex["rgb0"], target)
        loss.backward()
    finally:
        G.nb.set_precision("tc_fp16")
        G.nb.set_backward("tc")
    torch.cuda.synchronize()
    maps = {"rgb_map": rgb, "disp_map": disp, "acc_map": acc}
    return float(loss.item()), {k: v.detach().cpu().numpy() for k, v in maps.items()}, nets


GOLDEN_CASES = ["d4_fine8", "noenc_d2", "nv_d6_S316"]


@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_render_against_reference(G, case):
    """render() + img2mse + loss.backward() on the exact and the tensor-core path against the reference's autograd on the same
    nets (tests/golden/shapes.npz): exact path within 3e-3 plus twice the fp32 conditioning per tensor; tensor-core path
    within the forward and end-to-end budgets of the other files."""
    _check_render_against_reference(G, "shapes", case, (("fp32", "exact"), ("tc_fp16", "tc")))


def _check_render_against_reference(G, fixture, case, arms):
    fx = load_golden(fixture)
    p = f"{case}_"
    stats = {}
    for prec, bwd in arms:
        loss, maps, nets = _fixture_render(G, fx, case, prec, bwd)
        ref_loss = float(fx[p + "loss"])
        stats[f"{bwd}_loss_rel"] = abs(loss - ref_loss) / ref_loss
        assert stats[f"{bwd}_loss_rel"] < (1e-5 if bwd == "exact" else 5e-4), stats
        for k, v in maps.items():
            e = _same_nan(k, v, fx[p + k]) if k == "disp_map" else (_finite(k, v) or rel_l2(v, fx[p + k]))
            stats[f"{bwd}_{k}"] = e
            # disp = 1 / (depth / acc) amplifies rounding where acc is small: 1e-4 for it on the exact path
            assert e < ((1e-4 if k == "disp_map" else 2e-5) if bwd == "exact" else 3e-3), (bwd, k, stats)
        errs = {}
        for tag, net in zip(("c", "f"), nets):
            if net is None:
                continue
            names = [str(s) for s in fx[f"{p}g_{tag}_names"]]
            assert names == [n for n, _ in net.named_parameters()]
            ends = np.cumsum(fx[f"{p}g_{tag}_count"])
            for j, (name, prm) in enumerate(net.named_parameters()):
                g = prm.grad.detach().cpu().numpy().reshape(-1)
                _finite(f"{tag}.{name}", g)
                sl = slice(ends[j - 1] if j else 0, ends[j])
                idx, ref, norm = fx[f"{p}g_{tag}_idx"][sl], fx[f"{p}g_{tag}_val"][sl], float(fx[f"{p}g_{tag}_norm"][j])
                if norm == 0.0:                   # views_linears.0 without view directions: not on the loss's graph
                    assert not g.any(), (tag, name)
                    continue
                err = float(np.linalg.norm(g[idx] - ref) / max(np.linalg.norm(ref), 1e-30))
                errs[f"{tag}.{name}"] = err
                if bwd == "exact":
                    # 3e-3 plus twice the fp32 conditioning (tests/test_gpu_outgrads.py); the fine net three times: its samples
                    # are drawn from the coarse weights (sample_pdf), so an fp32 evaluation moves them as well as its own sums
                    cond = float(fx[f"{p}g_{tag}_cond"][j])
                    assert err < 3e-3 + (2 if tag == "c" else 3) * cond, (tag, name, err, cond)
        med, worst = float(np.median(list(errs.values()))), max(errs.values())
        stats[f"{bwd}_grad_median"], stats[f"{bwd}_grad_worst"] = med, worst
        if bwd == "tc":
            assert med < 3e-2 and worst < 1.5e-1, (med, worst, errs)
    _record(f"golden_{case}", stats)
    return stats


def test_fused_step_netdepth4(G):
    """FusedTrainStep on create_nerf's netdepth 4 coarse net (skips = [4] never reached) with an 8-layer fine net takes the
    steps of render() + autograd + torch.optim.Adam (tests/test_gpu_trainer.py's comparison)."""
    from nerf_pytorch_b200.trainer import FusedTrainStep
    fx = load_golden("shapes")
    N, steps, lrate, decay = 200, 4, 5e-4, 0.002
    sb = G.synth.ray_batch("lego", N, seed=8)
    rays = G.dev(sb["rays"])
    target = G.dev(np.random.default_rng(2).random((N, 3), dtype=np.float32))
    qf = _fixture_query_fn(G, fx, "d4_fine8")

    def kw(nets):
        return dict(_render_kw(G, nets), network_query_fn=qf)
    nets_a = _fixture_nets(G, fx, "d4_fine8")
    assert nets_a[0].D == 4 and nets_a[0].skips == [4]
    opt = torch.optim.Adam([p for n in nets_a for p in n.parameters()], lr=lrate, betas=(0.9, 0.999))
    losses_a, global_step = [], 0
    for _ in range(steps):
        rgb, _, _, ex = G.nb.render(400, 400, sb["K"], chunk=32768, rays=rays, retraw=True, **kw(nets_a))
        opt.zero_grad()
        loss = G.nb.img2mse(rgb, target) + G.nb.img2mse(ex["rgb0"], target)
        loss.backward()
        opt.step()
        for pg in opt.param_groups:
            pg["lr"] = lrate * (0.1 ** (global_step / (decay * 1000)))          # run_nerf.py:779-783
        global_step += 1
        losses_a.append(float(loss))
    nets_b = _fixture_nets(G, fx, "d4_fine8")
    init = [p.detach().clone() for n in nets_b for p in n.parameters()]
    tr = FusedTrainStep(400, 400, sb["K"], N, kw(nets_b), lrate=lrate, lrate_decay=decay, use_graph=True)
    rays_h, tgt_h = rays.cpu().pin_memory(), target.cpu().pin_memory()
    losses_b = [tr(rays_h, tgt_h) for _ in range(steps)]
    _finite("losses", losses_b)
    assert np.allclose(losses_a, losses_b, rtol=2e-4), (losses_a, losses_b)
    worst = 0.0
    for pa, pb, p0 in zip([p for n in nets_a for p in n.parameters()], [p for n in nets_b for p in n.parameters()], init):
        da, db = (pa.detach() - p0).cpu().numpy(), (pb.detach() - p0).cpu().numpy()
        _finite("update", db)
        worst = max(worst, rel_l2(db, da))
    _record("fused_step_netdepth4", {"losses_autograd": losses_a, "losses_fused": losses_b, "update_worst": worst})
    assert worst < 5e-2, worst


# ---- (e) shapes only the exact path serves -------------------------------------------------------------------------------------
# The exact path (mlp_simt_kernel forward, bwd_simt.cuh backward) takes any netwidth <= 256 that is a multiple of 4, netdepth
# 1 .. 16 and any encoding width; the tensor-core path only netwidth 256, netdepth 2 .. 8 and input_ch <= 63.  march_bwd_impl
# recomputes the pass in slabs of up to 512 rays; a slab of M = rays x samples rows with M odd and netwidth / 2 not a multiple of
# 4 is where its buffers after hv would lose their 16-byte alignment (raw is stored and loaded as float4).

# id, W, D, skips, multires, multires_views (None: no view directions), output_ch, N, S, parameter seed (seeds whose rays are not
# all empty: an empty batch has no gradient)
EXACT_SHAPES = [
    ("w100_d3_s0", 100, 3, [0], 10, 4, 5, 37, 65, 0),      # W / 2 = 50, odd M; GEMM tiles with remainders; several wgrad slabs
    ("w252_d9_s7", 252, 9, [7], 10, 4, 5, 37, 65, 0),      # the widest odd-k width, D > 8, skip D - 2
    ("w4_d1", 4, 1, [], 0, 0, 5, 7, 9, 0),                 # smallest net (i_embed = -1): one wgrad slab, one column-sum block
    ("w128_d10", 128, 10, [4], 10, 4, 5, 37, 64, 1),       # --netwidth 128 --netdepth 10
    ("w256_L16", 256, 8, [4], 16, 16, 5, 21, 64, 0),       # octaves up to 2^15, input_ch 99 + 99: the largest shared memory
    ("w64_d16_nv", 64, 16, [14], 11, None, 4, 33, 33, 0),  # D = 16, the no-view head
    ("w200_d12_s0", 200, 12, [0], 13, 5, 5, 600, 33, 1),   # > 512 rays: two ray slabs in march_bwd_impl
    ("w36_d2_nv", 36, 2, [], 6, None, 5, 513, 3, 1),       # odd M in the last ray slab only (1 ray x 3 samples); output_ch 5
]


def _check_exact_grads(sh, grads, g_ref, g32, stats, tag):
    """every gradient tensor against float64 autograd: gated at 1e-4 plus twice the float32 autograd's own distance where that
    is <= 1e-4, recorded elsewhere; tensors off the loss's graph exactly 0 -> names of the gated tensors"""
    gated = []
    for name, ref in g_ref.items():
        _finite(f"{tag} {name}", grads[name])
        if not ref.any():
            assert not grads[name].any(), (tag, name)
            continue
        e, cond = rel_l2(grads[name], ref), rel_l2(g32[name], ref)
        stats[f"{tag}_g_{name}"], stats[f"{tag}_cond_g_{name}"] = e, cond
        if cond <= 1e-4:
            assert e < 1e-4 + 2 * cond, (tag, name, e, cond)
            gated.append(name)
    if "output_linear.weight" in grads:          # rows >= 4 of output_linear never reach raw2outputs
        assert not grads["output_linear.weight"][4:].any() and not grads["output_linear.bias"][4:].any(), tag
    return gated


@pytest.mark.parametrize("sid,W,D,skips,L,Lv,out_ch,N,S,seed", EXACT_SHAPES, ids=[s[0] for s in EXACT_SHAPES])
def test_exact_path_shape(G, sid, W, D, skips, L, Lv, out_ch, N, S, seed):
    sh = _shape(G, sid, D, skips, L, Lv, out_ch, seed=seed, W=W)
    packed, z = _rays(G, sh, N, S, seed=5)
    rays, zd = G.dev(packed), G.dev(z)
    slab_rows = [min(512, N - n0) * S for n0 in range(0, N, 512)]
    stats = {"odd_slab": any(m % 2 for m in slab_rows), "hv_unaligned": (W // 2) % 4 != 0}
    # forward: nerf_b200_march and nerf_b200_run_network in fp32
    g_rgb = _g_rgb(N)
    raw_ref, maps_ref, g_ref = _exact_reference(sh, packed, z, g_rgb)
    raw32, maps32, g32 = _exact_reference(sh, packed, z, g_rgb, torch.float32)
    stats["cond_raw"] = rel_l2(raw32, raw_ref)
    o, _, _ = G.march(sh.net, rays, zd, train=False, L=sh.L, Lv=sh.Lv, precision=G._lib.PREC_FP32)
    vd = G.dev(packed[:, 8:11]) if sh.views else None
    raw_rn = G.run_network_exact(sh.net, _pts(packed, z).to(G.DEV), vd, S, L=sh.L, Lv=sh.Lv)
    for tag, r in (("march", o["raw"]), ("run_network", raw_rn)):
        r = r.cpu().numpy().reshape(-1, 4)
        _finite(f"{tag} raw", r)
        stats[f"{tag}_raw_rel"] = rel_l2(r, raw_ref)
        assert stats[f"{tag}_raw_rel"] <= 2e-5 + 2 * stats["cond_raw"], (tag, stats)
    for k in ("rgb", "disp", "acc", "w"):
        v = o[k].cpu().numpy()
        stats[f"{k}_rel"] = _same_nan("disp", v, maps_ref[k]) if k == "disp" else (_finite(k, v) or rel_l2(v, maps_ref[k]))
        stats[f"cond_{k}"] = rel_l2(maps32[k], maps_ref[k])
        assert stats[f"{k}_rel"] <= 2e-5 + 2 * stats[f"cond_{k}"], (k, stats)
    # backward, rgb seed: the workspace's contents must not matter (0xFF bytes are NaNs)
    g_nan = G.march_bwd_exact(sh.net, rays, zd, G.dev(g_rgb), L=sh.L, Lv=sh.Lv, fill=0xFF)
    g_zero = G.march_bwd_exact(sh.net, rays, zd, G.dev(g_rgb), L=sh.L, Lv=sh.Lv, fill=0)
    for name in g_zero:
        assert np.array_equal(g_nan[name].view(np.uint32), g_zero[name].view(np.uint32)), name
    gated = _check_exact_grads(sh, g_nan, g_ref, g32, stats, "rgb")
    # backward, rgb + disp + acc + raw seeds (nerf_b200_march_bwd_outs).  disp is seeded on rays with acc > 1e-4 only: on emptier
    # rays disp = acc / depth is all rounding.  The raw seed is positive: a zero-mean seed on every sample makes the bias gradients
    # (plain sums of dL/draw over all rows) cancel 40 to 1000-fold, and then the order of the fp32 sums decides their last digits
    rng = np.random.default_rng(4)
    seeds = {"rgb_map": rng.standard_normal((N, 3)) * 1e-3, "disp_map": rng.standard_normal(N) * 1e-2 * (maps_ref["acc"] > 1e-4),
             "acc_map": rng.standard_normal(N) * 1e-2, "raw": rng.random((N, S, 4)) * 1e-4}
    seeds = {k: v.astype(np.float32) for k, v in seeds.items()}
    seeds64 = {k: torch.from_numpy(v).double() for k, v in seeds.items()}
    _, _, go_ref = _exact_reference(sh, packed, z, None, seeds=seeds64)
    _, _, go32 = _exact_reference(sh, packed, z, None, torch.float32, seeds=seeds64)
    go_nan = G.march_bwd_exact(sh.net, rays, zd, {k: G.dev(v) for k, v in seeds.items()}, L=sh.L, Lv=sh.Lv, fill=0xFF)
    go_zero = G.march_bwd_exact(sh.net, rays, zd, {k: G.dev(v) for k, v in seeds.items()}, L=sh.L, Lv=sh.Lv, fill=0)
    for name in go_zero:
        assert np.array_equal(go_nan[name].view(np.uint32), go_zero[name].view(np.uint32)), name
    gated_outs = _check_exact_grads(sh, go_nan, go_ref, go32, stats, "outs")
    stats.update(gated_rgb=len(gated), gated_outs=len(gated_outs))
    _record(f"exact_{sid}", stats)
    assert gated and gated_outs, ("the loss has no well-conditioned gradient", stats)


EXACT_GOLDEN_CASES = ["w128_d10", "L14_Lv8", "w100_nv_odd"]


@pytest.mark.parametrize("case", EXACT_GOLDEN_CASES)
def test_exact_shapes_render_against_reference(G, case):
    """render() + img2mse + loss.backward() in fp32 on create_nerf-shaped nets the tensor-core path refuses, against the
    reference's autograd (tests/golden/exact_shapes.npz), with test_render_against_reference's exact-path gates.  w100_nv_odd:
    netwidth 100 and 33 rays x 33 / 65 samples, odd in both passes."""
    _check_render_against_reference(G, "exact_shapes", case, (("fp32", "exact"),))


# id -> (NeRF arguments, what the message names); skips = [3] with netdepth 4 is a skip after the last layer
RENDER_REFUSED = {"skip_D_minus_1": (dict(D=4, W=64, skips=[3]), "skip layer must be < netdepth - 1"),
                  "W50": (dict(D=2, W=50, skips=[]), "a multiple of 4"),
                  "W260": (dict(D=2, W=260, skips=[]), "netwidth <= 256"),
                  "D17": (dict(D=17, W=16, skips=[]), "netdepth must be in [1, 16]")}


@pytest.mark.parametrize("case", list(RENDER_REFUSED))
def test_exact_path_refusals_through_render(G, case):
    """render() in fp32 refuses the net before it launches anything and leaves every .grad as it was; the coarse net is a
    good one that already holds a gradient."""
    kw_net, msg = RENDER_REFUSED[case]
    sb = G.synth.ray_batch("lego", 16, seed=2)
    good = G.nb.NeRF(D=2, W=64, input_ch=63, input_ch_views=27, output_ch=5, skips=[], use_viewdirs=True).to(G.DEV)
    bad = G.nb.NeRF(input_ch=63, input_ch_views=27, output_ch=5, use_viewdirs=True, **kw_net).to(G.DEV)
    for p in list(good.parameters()) + list(bad.parameters()):
        p.grad = torch.full_like(p, 0.5)
    before = [p.grad.clone() for p in list(good.parameters()) + list(bad.parameters())]
    G.nb.set_precision("fp32")
    try:
        for nets in ((bad, None), (good, bad)):
            n0 = G.nb.launch_count()
            with pytest.raises(RuntimeError, match=re.escape(msg)):
                G.nb.render(400, 400, sb["K"], rays=G.dev(sb["rays"]), **_render_kw(G, nets, N_samples=8, N_importance=8))
            assert G.nb.launch_count() == n0, case
    finally:
        G.nb.set_precision("tc_fp16")
    for p, g in zip(list(good.parameters()) + list(bad.parameters()), before):
        assert torch.equal(p.grad, g)


def test_tensor_core_refusal_of_another_width_points_to_the_exact_path(G):
    sb = G.synth.ray_batch("lego", 16, seed=2)
    net = G.nb.NeRF(D=8, W=128, input_ch=63, input_ch_views=27, output_ch=5, skips=[4], use_viewdirs=True).to(G.DEV)
    with pytest.raises(RuntimeError, match=re.escape("set_precision('fp32')")):
        G.nb.render(400, 400, sb["K"], rays=G.dev(sb["rays"]), **_render_kw(G, (net, net), N_samples=8, N_importance=8))
    G.nb.set_precision("fp32")
    try:
        rgb, _, _, _ = G.nb.render(400, 400, sb["K"], rays=G.dev(sb["rays"]), **_render_kw(G, (net, net), N_samples=8, N_importance=8))
    finally:
        G.nb.set_precision("tc_fp16")
    _finite("rgb", rgb.detach().cpu().numpy())
