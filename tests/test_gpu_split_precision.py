"""Precision tc_split: the fused forward with every tensor-core operand split into hi + lo fp16 halves (three MMAs per K-step
into one fp32 accumulator, march_split_kernel) against the reference's fp32 results -- the gates the exact fp32 path meets.

(a) the trained fixtures (trained_lego_1024 through the C ABI with both passes' weights, fern_ndc_4096 through render()): the
    fp32 branch of test_gpu_parity._check_trained_gates, and rgb_map <= 1e-4 on both;
(b) every tensor-core network shape of test_gpu_shapes.SHAPES: run_network and march against a float64 autograd of the
    reference's network (oracle/torch_ref.mlp), >= 20x closer than tc_fp16;
(c) PSNR on the analytic scene, and gradients through render() + backward() (the exact recompute backward);
(d) plumbing: GraphedRender, run-to-run bits, and the training-mode refusals.
Measured deviations go to parity_split.json in $NERF_B200_PARITY_DIR (default: a nerf_b200_parity directory under the
system's temporary directory)."""
import ctypes as C
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_l2
from test_gpu_parity import _check_trained_gates, _finite_rel, _trained_nets

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def G():
    import gpu_common
    return gpu_common


@pytest.fixture
def split_mode(G):
    G.nb.set_precision("tc_split")
    yield
    G.nb.set_precision("tc_fp16")
    G.nb.set_backward("tc")


def _record(name, value):
    out_dir = os.environ.get("NERF_B200_PARITY_DIR") or os.path.join(tempfile.gettempdir(), "nerf_b200_parity")
    path = os.path.join(out_dir, "parity_split.json")
    os.makedirs(out_dir, exist_ok=True)
    data = {}
    if os.path.isfile(path):
        with open(path) as f:
            data = json.load(f)
    data[name] = value
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)


def _render(G, nets, sb, ndc, near, far, white, **kw):
    return G.nb.render(sb["H"], sb["W"], sb["K"], chunk=32768, rays=G.dev(sb["rays"]), ndc=ndc, near=near, far=far, use_viewdirs=True,
                       network_fn=nets[0], network_fine=nets[1], network_query_fn=G.query_fn(), N_samples=64, N_importance=128,
                       perturb=0., white_bkgd=white, raw_noise_std=0., **kw)


# ---- (a) trained fixtures ------------------------------------------------------------------------------------------------------

def test_trained_lego_1024_meets_the_fp32_gates(G):
    """nerf_b200_render_rays_fwd in TC_SPLIT on the split images, with both passes' weights and z"""
    lib = G._lib.load()
    fx = load_golden("trained_lego_1024")
    sb = G.synth.ray_batch("lego", int(fx["N"]), seed=int(fx["ray_seed"]))
    rays = G.dev(G.O.pack_rays(sb["H"], sb["W"], sb["K"], sb["rays"][0], sb["rays"][1], False, 2.0, 6.0, True).astype(np.float32))
    nets = _trained_nets(G)
    N, Sc, Ni = rays.shape[0], 64, 128
    Sf = Sc + Ni
    cfg = G.cfg(Sc, 11, precision=G._lib.PREC_TC_SPLIT)
    cfg.N_importance = Ni
    z = lambda *s: torch.zeros(s, device=G.DEV)
    o = dict(rgb0=z(N, 3), disp0=z(N), acc0=z(N), w0=z(N, Sc), raw0=z(N, Sc, 4), rgb=z(N, 3), disp=z(N), acc=z(N), w=z(N, Sf), raw=z(N, Sf, 4),
             z_c=z(N, Sc), z_f=z(N, Sf), z_std=z(N))
    out_c = G._lib.NerfPassOut(G.ptr(o["rgb0"]), G.ptr(o["disp0"]), G.ptr(o["acc0"]), C.c_void_p(0), G.ptr(o["w0"]), G.ptr(o["raw0"]))
    out_f = G._lib.NerfPassOut(G.ptr(o["rgb"]), G.ptr(o["disp"]), G.ptr(o["acc"]), C.c_void_p(0), G.ptr(o["w"]), G.ptr(o["raw"]))
    pc, pf = nets[0].net_params(), nets[1].net_params()
    t_vals, u_det = torch.linspace(0., 1., Sc, device=G.DEV), torch.linspace(0., 1., Ni, device=G.DEV)
    ws_bytes = lib.nerf_b200_march_workspace_bytes(N, Sf)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=G.DEV)
    G._lib.check(lib.nerf_b200_render_rays_fwd(G.ptr(rays), N, C.byref(cfg), C.byref(pc), G.ptr(nets[0].packed_split()), C.byref(pf),
                                               G.ptr(nets[1].packed_split()), G.ptr(t_vals), G.ptr(u_det), None, None, None, None,
                                               G.ptr(o["z_c"]), C.byref(out_c), G.ptr(o["z_f"]), G.ptr(o["z_std"]), C.byref(out_f), G.ptr(ws),
                                               ws_bytes, G.stream()), "render_rays_fwd")
    torch.cuda.synchronize()
    o = {k: v.cpu().numpy() for k, v in o.items()}
    st = {}
    for k, ref in (("rgb", "rgb_map"), ("acc", "acc_map"), ("rgb0", "rgb0"), ("acc0", "acc0"), ("w0", "w_coarse"), ("w", "w_fine"),
                   ("z_f", "z_fine"), ("z_std", "z_std")):
        st[ref] = rel_l2(o[k], fx[ref])
    for k, ref in (("raw0", "raw_coarse"), ("raw", "raw_fine")):
        st[ref] = rel_l2(o[k][:256], fx[ref])
    st["disp_map"], _ = _finite_rel(o["disp"], fx["disp_map"])
    st["disp_nan_mask_mismatch"] = float(np.mean(np.isnan(o["disp"]) != np.isnan(fx["disp_map"])))
    _record("trained_lego_1024", st)
    print(st)
    _check_trained_gates(st, "fp32")
    assert st["rgb_map"] <= 1e-4, st


def test_config3_fern_ndc_4096_meets_the_fp32_gates(G, split_mode):
    fx = load_golden("fern_ndc_4096")
    sb = G.synth.ray_batch("fern", 4096, seed=int(fx["ray_seed"]))
    with torch.no_grad():
        rgb, disp, acc, ex = _render(G, _trained_nets(G), sb, True, 0., 1., False)
    st = {"rgb_map": rel_l2(rgb.cpu().numpy(), fx["rgb_map"]), "acc_map": rel_l2(acc.cpu().numpy(), fx["acc_map"]),
          "rgb0": rel_l2(ex["rgb0"].cpu().numpy(), fx["rgb0"]), "acc0": rel_l2(ex["acc0"].cpu().numpy(), fx["acc0"]),
          "z_std": rel_l2(ex["z_std"].cpu().numpy(), fx["z_std"])}
    st["disp_nan_mask_mismatch"] = float(np.mean(np.isnan(disp.cpu().numpy()) != np.isnan(fx["disp_map"])))
    _record("fern_ndc_4096", st)
    print(st)
    _check_trained_gates(st, "fp32")
    assert st["rgb_map"] <= 1e-4, st


# ---- (b) every tensor-core shape -----------------------------------------------------------------------------------------------

def _ref_raw(sh, pts, vd_rows):
    """float64 autograd-free forward of the reference's network (oracle/torch_ref.mlp) on fp32 points"""
    from oracle import torch_ref as T
    sd = {k: torch.from_numpy(v).double() for k, v in sh.state.items()}
    x = T.embed(pts.double().cpu(), sh.L)
    if sh.views:
        x = torch.cat([x, T.embed(vd_rows.double().cpu(), sh.Lv)], -1)
    return T.mlp(sd, x, ic=sh.ic, icv=sh.icv, skip=sh.skip, D=sh.D).numpy()


def _run_network(G, sh, pts, vd, prec):
    from nerf_pytorch_b200.api import _packed_for
    lib = G._lib.load()
    N, S = vd.shape[0], pts.shape[0] // vd.shape[0]
    raw = torch.empty((N * S, 4), device=G.DEV)
    ws_bytes = lib.nerf_b200_march_workspace_bytes(N, S)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=G.DEV)
    n = sh.net.net_params()
    G._lib.check(lib.nerf_b200_run_network(G.ptr(pts), G.ptr(vd if sh.views else None), N, S, C.byref(n), G.ptr(_packed_for(sh.net, prec)),
                                           sh.L, sh.Lv, prec, G.ptr(raw), G.ptr(ws), ws_bytes, G.stream()), "run_network")
    return raw.cpu().numpy()


def _march_raw(G, sh, rays, z, prec):
    from nerf_pytorch_b200.api import _packed_for
    lib = G._lib.load()
    N, S = z.shape
    raw = torch.zeros((N, S, 4), device=G.DEV)
    out = G._lib.NerfPassOut(C.c_void_p(0), C.c_void_p(0), C.c_void_p(0), C.c_void_p(0), C.c_void_p(0), G.ptr(raw))
    ws_bytes = lib.nerf_b200_march_workspace_bytes(N, S)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=G.DEV)
    c = G.cfg(S, rays.shape[1], sh.L, sh.Lv, True, prec)
    n = sh.net.net_params()
    G._lib.check(lib.nerf_b200_march(G.ptr(rays), G.ptr(z), None, N, S, C.byref(n), G.ptr(_packed_for(sh.net, prec)), C.byref(c), C.byref(out),
                                     G.ptr(ws), ws_bytes, G.stream()), "march")
    return raw.reshape(-1, 4).cpu().numpy()


from test_gpu_shapes import SHAPES, _shape  # noqa: E402


@pytest.mark.parametrize("sid,D,skips,L,Lv,out_ch,seed", SHAPES, ids=[s[0] for s in SHAPES])
def test_every_tensor_core_shape_is_fp32_class(G, sid, D, skips, L, Lv, out_ch, seed):
    sh = _shape(G, sid, D, skips, L, Lv, out_ch, seed)
    gen = torch.Generator().manual_seed(7)
    N, S = 48, 40
    o = torch.rand((N, 3), generator=gen) * 2 - 1
    d = torch.nn.functional.normalize(torch.randn((N, 3), generator=gen), dim=-1)
    z = torch.linspace(0.5, 3.0, S).expand(N, S).contiguous()
    pts = (o[:, None] + d[:, None] * z[..., None]).reshape(-1, 3)           # fp32, as the kernel's o + d z
    vd_rows = d[:, None].expand(N, S, 3).reshape(-1, 3)
    rays = torch.cat([o, d, torch.full((N, 1), 0.5), torch.full((N, 1), 3.0)] + ([d] if sh.views else []), -1)
    ref = _ref_raw(sh, pts, vd_rows)
    st = {}
    for prec, name in ((G._lib.PREC_TC_SPLIT, "tc_split"), (G._lib.PREC_TC_FP16, "tc_fp16")):
        rn = _run_network(G, sh, G.dev(pts.numpy()), G.dev(d.numpy()), prec)
        mr = _march_raw(G, sh, G.dev(rays.numpy()), G.dev(z.numpy()), prec)
        assert np.isfinite(rn).all() and np.isfinite(mr).all()
        st[f"run_network_{name}"], st[f"march_{name}"] = rel_l2(rn, ref), rel_l2(mr, ref)
    _record(f"shape_{sid}", st)
    print(sid, st)
    for k in ("run_network", "march"):
        assert st[f"{k}_tc_split"] < 2e-5, st
        assert st[f"{k}_tc_fp16"] >= 20.0 * st[f"{k}_tc_split"], st


# ---- (c) PSNR and gradients ----------------------------------------------------------------------------------------------------

def test_psnr_on_the_analytic_scene_matches_the_reference(G, split_mode):
    from oracle.gen_trained import sphere_targets
    fx = load_golden("trained_lego_1024")
    sb = G.synth.ray_batch("lego", int(fx["N"]), seed=int(fx["ray_seed"]))
    gt = sphere_targets(sb["rays"][0], sb["rays"][1])
    with torch.no_grad():
        rgb = _render(G, _trained_nets(G), sb, False, 2., 6., True)[0]
    st = {"psnr_reference_fp32_cpu": float(-10.0 * np.log10(np.mean((fx["rgb_map"] - gt) ** 2))),
          "psnr_tc_split": float(G.nb.mse2psnr(G.nb.img2mse(rgb, G.dev(gt))).item())}
    _record("psnr_analytic_scene", st)
    print(st)
    assert abs(st["psnr_tc_split"] - st["psnr_reference_fp32_cpu"]) < 1e-3, st


def test_trained_networks_gradients(G, split_mode):
    """render() + img2mse + backward(): the split forward, then the exact recompute backward (whatever set_backward says)"""
    fx = load_golden("trained_lego_grads")
    sb = G.synth.ray_batch("lego", int(fx["N"]), seed=int(fx["ray_seed"]))
    nets = _trained_nets(G)
    n0 = G.nb.launch_count()
    rgb, _, _, ex = _render(G, nets, sb, False, 2., 6., True, retraw=True)
    target = G.dev(fx["target"])
    loss = G.nb.img2mse(rgb, target) + G.nb.img2mse(ex["rgb0"], target)
    loss.backward()
    assert G.nb.launch_count() > n0
    errs = {}
    for tag, net in (("c", nets[0]), ("f", nets[1])):
        for name, p in net.named_parameters():
            g = p.grad.detach().cpu().numpy().reshape(-1)
            idx, ref = fx[f"g_{tag}_{name}_idx"], fx[f"g_{tag}_{name}_val"]
            errs[f"{tag}.{name}"] = float(np.linalg.norm(g[idx] - ref) / max(np.linalg.norm(ref), 1e-12))
    st = {"loss_rel": abs(float(loss) - float(fx["loss"])) / float(fx["loss"]), "median": float(np.median(list(errs.values()))),
          "max": float(max(errs.values()))}
    _record("trained_grads", st)
    print(st)
    assert st["median"] < 1e-3 and st["max"] < 2e-2, st


# ---- (d) plumbing ---------------------------------------------------------------------------------------------------------------

def _bits(t):
    return t.contiguous().view(torch.int32)


def test_graphed_render_and_run_to_run_bits(G, split_mode):
    """GraphedRender at its capacity and at a tail size gives render(chunk=n)'s bits; two renders give the same bits"""
    fx = load_golden("trained_lego_1024")
    sb = G.synth.ray_batch("lego", int(fx["N"]), seed=int(fx["ray_seed"]))
    nets = _trained_nets(G)
    kw = dict(ndc=False, near=2., far=6., use_viewdirs=True, network_fn=nets[0], network_fine=nets[1], network_query_fn=G.query_fn(),
              N_samples=64, N_importance=128, perturb=0., white_bkgd=True, raw_noise_std=0.)
    rays_h = torch.from_numpy(sb["rays"]).pin_memory()
    g = G.nb.GraphedRender(sb["H"], sb["W"], sb["K"], 1024, **kw)
    for n in (1024, 300):
        with torch.no_grad():
            outs = [G.nb.render(sb["H"], sb["W"], sb["K"], chunk=n, rays=rays_h[:, :n].to(G.DEV), **kw) for _ in range(2)]
        want = [torch.cat([rgb, disp[:, None], acc[:, None]], 1).cpu() for rgb, disp, acc, _ in outs]
        assert torch.equal(_bits(want[0]), _bits(want[1])), n
        got = g(rays_h[:, :n]).clone()
        assert torch.equal(_bits(got), _bits(want[0])), n
    # a weight update reaches the split image through refresh()
    with torch.no_grad():
        nets[1].rgb_linear.bias.add_(0.25)
    g.refresh()
    with torch.no_grad():
        rgb = G.nb.render(sb["H"], sb["W"], sb["K"], chunk=1024, rays=rays_h.to(G.DEV), **kw)[0].cpu()
    assert torch.equal(_bits(g(rays_h)[:, :3].clone()), _bits(rgb))


def test_training_mode_is_refused_before_any_launch(G, split_mode):
    from nerf_pytorch_b200.trainer import FusedTrainStep
    sh = _shape(G, "d8_s4", 8, [4], 10, 4, 5, 0)
    N, S = 16, 40
    rays = torch.cat([torch.zeros(N, 3), torch.tensor([[0., 0., 1.]]).expand(N, 3), torch.full((N, 1), 2.), torch.full((N, 1), 6.),
                      torch.tensor([[0., 0., 1.]]).expand(N, 3)], -1)
    z = torch.linspace(2., 6., S).expand(N, S).contiguous()
    n0 = G.nb.launch_count()
    with pytest.raises(RuntimeError, match="exact backward"):
        G.march(sh.net, G.dev(rays.numpy()), G.dev(z.numpy()), True, precision=G._lib.PREC_TC_SPLIT)
    assert G.nb.launch_count() == n0
    H, W, K, _ = G.synth.lego_camera(100)
    kw = dict(network_fn=sh.net, network_fine=None, network_query_fn=G.query_fn(), N_samples=64, N_importance=0, perturb=0.,
              white_bkgd=True, raw_noise_std=0., use_viewdirs=True, ndc=False, near=2., far=6.)
    with pytest.raises(RuntimeError, match="tc_fp16"):
        FusedTrainStep(H, W, K, 256, kw)
    assert G.nb.launch_count() == n0
