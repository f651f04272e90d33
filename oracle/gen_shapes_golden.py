"""Generate tests/golden/shapes.npz and tests/golden/exact_shapes.npz by running the UNMODIFIED reference on CPU  --  build
container only.

    python oracle/gen_shapes_golden.py [shapes | exact_shapes]   # needs the reference checkout (oracle/ref_import.py); writes
                                                                 # tests/golden/ (both files without an argument)

Networks other than the default 8 x 256 with 63 + 27 input channels, built by the reference's create_nerf (skips = [4]):

    d4_fine8   : --netdepth 4 (the skip is never reached) --netdepth_fine 8 --multires 6 --multires_views 2, view directions,
                 32 + 96 samples, 32 lego rays
    noenc_d2   : --i_embed -1 (input_ch 3) --netdepth 2, no view directions, 64 samples, N_importance 0 (output_ch 4), 32 lego rays
    nv_d6_S316 : --netdepth 6 --netdepth_fine 6, no view directions, 16 + 300 samples (one fine ray spans two 256-row
                 super-tiles), 16 fern NDC rays

exact_shapes.npz: create_nerf-shaped nets only the exact path (fp32 CUDA cores) runs -- the tensor-core path takes netwidth 256
and input_ch <= 63 only:

    w128_d10     : --netwidth 128 --netdepth 10 --netwidth_fine 64 --netdepth_fine 4, view directions, 32 + 64 samples, 32 lego rays
    L14_Lv8      : --multires 14 --multires_views 8 (input_ch 87 + 51), view directions, 64 + 64 samples, 16 lego rays
    w100_nv_odd  : --netwidth 100 --netwidth_fine 100, no view directions, 33 + 32 samples, 33 fern NDC rays: N * S is odd in both
                   passes (33 x 33, 33 x 65) and W / 2 = 50 is not a multiple of 4

Stored per case `x` (keys prefixed `x_`): the inputs and settings, the target, rgb_map / disp_map / acc_map, the loss
img2mse(rgb) (+ img2mse(rgb0)), and per net (c, f) 64 sampled entries of every parameter gradient (g_{c,f}_{names,count,idx,val}),
the full gradient norms (g_{c,f}_norm) and, per tensor, the rel-L2 distance of the sampled entries from the same reference run
in float64 (g_{c,f}_cond).  Parameters are regenerated from oracle/synth.nerf_state / oracle/noviews.nerf_state_noviews.
"""
import copy
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import noviews, ref_import, synth  # noqa: E402
from oracle.gen_golden import OUT, load_state, make_args, to_np  # noqa: E402

N_SAMPLED = 64

CASES = {
    "d4_fine8": dict(scene="lego", N=32, netdepth=4, netdepth_fine=8, multires=6, multires_views=2, i_embed=0, use_viewdirs=True,
                     N_samples=32, N_importance=96, seed_w=0),
    "noenc_d2": dict(scene="lego", N=32, netdepth=2, netdepth_fine=2, multires=10, multires_views=4, i_embed=-1, use_viewdirs=False,
                     N_samples=64, N_importance=0, seed_w=2),
    "nv_d6_S316": dict(scene="fern", N=16, netdepth=6, netdepth_fine=6, multires=10, multires_views=4, i_embed=0, use_viewdirs=False,
                       N_samples=16, N_importance=300, seed_w=4),
}

EXACT_CASES = {
    "w128_d10": dict(scene="lego", N=32, netwidth=128, netdepth=10, netwidth_fine=64, netdepth_fine=4, multires=10, multires_views=4,
                     i_embed=0, use_viewdirs=True, N_samples=32, N_importance=64, seed_w=2),
    "L14_Lv8": dict(scene="lego", N=16, netdepth=8, netdepth_fine=8, multires=14, multires_views=8, i_embed=0, use_viewdirs=True,
                    N_samples=64, N_importance=64, seed_w=2),
    "w100_nv_odd": dict(scene="fern", N=33, netwidth=100, netdepth=8, netwidth_fine=100, netdepth_fine=8, multires=10,
                        multires_views=4, i_embed=0, use_viewdirs=False, N_samples=33, N_importance=32, seed_w=0),
}

TABLES = {"shapes": CASES, "exact_shapes": EXACT_CASES}


def input_ch(L, i_embed):
    return 3 if i_embed == -1 else 3 + 6 * L


def states(c, output_ch):
    ic = input_ch(c["multires"], c["i_embed"])
    icv = input_ch(c["multires_views"], c["i_embed"])
    out = []
    for k, (D, W) in enumerate(((c["netdepth"], c.get("netwidth", 256)), (c["netdepth_fine"], c.get("netwidth_fine", 256)))):
        if c["use_viewdirs"]:
            out.append(synth.nerf_state(c["seed_w"] + k, False, D=D, W=W, input_ch=ic, input_ch_views=icv, skips=(4,)))
        else:
            out.append(noviews.nerf_state_noviews(c["seed_w"] + k, output_ch=output_ch, D=D, W=W, input_ch=ic, skips=(4,)))
    return out


def render_loss(rn, kw, sb, target, dtype):
    rays = torch.from_numpy(sb["rays"]).to(dtype)
    rgb, disp, acc, ex = rn.render(sb["H"], sb["W"], sb["K"], chunk=1024 * 32, rays=rays, retraw=True, **kw)
    loss = torch.mean((rgb - target.to(dtype)) ** 2)                  # img2mse (run_nerf_helpers.py:9)
    if "rgb0" in ex:
        loss = loss + torch.mean((ex["rgb0"] - target.to(dtype)) ** 2)
    return loss, rgb, disp, acc


def run_case(rn, fx, tag, c):
    sb = synth.ray_batch(c["scene"], c["N"], seed=7)
    with tempfile.TemporaryDirectory() as tmp:
        args = make_args(tmp, N_importance=c["N_importance"], N_samples=c["N_samples"], use_viewdirs=c["use_viewdirs"],
                         white_bkgd=sb["white_bkgd"], dataset_type="llff" if sb["ndc"] else "blender", perturb=0.0)
        for k in ("netdepth", "netdepth_fine", "multires", "multires_views", "i_embed", "netwidth", "netwidth_fine"):
            if k in c:
                setattr(args, k, c[k])
        kw, _, _, _, _ = rn.create_nerf(args)
    nets = [kw["network_fn"], kw["network_fine"]]
    output_ch = 5 if c["N_importance"] > 0 else 4
    for net, st in zip(nets, states(c, output_ch)):
        if net is not None:
            load_state(net, st)
    kw = dict(kw)
    kw.update(near=sb["near"], far=sb["far"], perturb=0.0, raw_noise_std=0.0)
    target = torch.from_numpy(np.random.default_rng(21).random((c["N"], 3), dtype=np.float32))
    p = tag + "_"
    fx.update({p + k: np.asarray(v) for k, v in c.items() if k != "scene"})
    fx.update({p + k: np.asarray(sb[k]) for k in ("rays", "K", "H", "W", "near", "far", "ndc", "white_bkgd")})
    fx[p + "output_ch"], fx[p + "target"] = np.int32(output_ch), to_np(target)
    with torch.enable_grad():
        loss, rgb, disp, acc = render_loss(rn, kw, sb, target, torch.float32)
        loss.backward()
    fx[p + "loss"] = np.float32(loss.item())
    fx[p + "rgb_map"], fx[p + "disp_map"], fx[p + "acc_map"] = to_np(rgb), to_np(disp), to_np(acc)
    # the same run in float64: how far fp32 arithmetic leaves the reference's own gradient (the loss's conditioning)
    torch.set_default_dtype(torch.float64)
    try:
        nets64 = [copy.deepcopy(n).double() if n is not None else None for n in nets]
        for n in nets64:
            if n is not None:
                n.zero_grad(set_to_none=True)
        with torch.enable_grad():
            render_loss(rn, dict(kw, network_fn=nets64[0], network_fine=nets64[1]), sb, target, torch.float64)[0].backward()
    finally:
        torch.set_default_dtype(torch.float32)
    srng = np.random.default_rng(9)
    for ntag, net, net64 in zip(("c", "f"), nets, nets64):
        if net is None:
            continue
        names, idx, vals, norms, conds = [], [], [], [], []
        for (name, prm), (_, p64) in zip(net.named_parameters(), net64.named_parameters()):
            ii = srng.integers(0, prm.numel(), min(N_SAMPLED, prm.numel())).astype(np.int32)
            g = to_np(prm.grad).reshape(-1) if prm.grad is not None else np.zeros(prm.numel(), np.float32)
            g64 = p64.grad.reshape(-1)[ii] if p64.grad is not None else torch.zeros(len(ii), dtype=torch.float64)
            names.append(name)
            idx.append(ii)
            vals.append(g[ii])
            norms.append(np.linalg.norm(g.astype(np.float64)))
            conds.append(float((torch.from_numpy(g[ii]).double() - g64).norm() / g64.norm().clamp_min(1e-300)))
        fx[p + f"g_{ntag}_names"] = np.array(names)
        fx[p + f"g_{ntag}_count"] = np.array([len(i) for i in idx], np.int32)
        fx[p + f"g_{ntag}_idx"] = np.concatenate(idx)
        fx[p + f"g_{ntag}_val"] = np.concatenate(vals)
        fx[p + f"g_{ntag}_norm"] = np.array(norms, np.float32)
        fx[p + f"g_{ntag}_cond"] = np.array(conds, np.float32)
    print(tag, "loss", float(loss.item()), flush=True)


def main():
    assert ref_import.available(), "reference not found (this script only runs where the reference checkout exists)"
    t0 = time.time()
    torch.manual_seed(0)
    torch.set_num_threads(8)                      # fixed: CPU reductions are then reproducible bit for bit
    rn, _ = ref_import.load()
    os.makedirs(OUT, exist_ok=True)
    for name in sys.argv[1:] or list(TABLES):
        fx = {}
        for tag, c in TABLES[name].items():
            run_case(rn, fx, tag, c)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **fx)
        print("wrote", name, len(fx), "arrays in", round(time.time() - t0, 1), "s")


if __name__ == "__main__":
    main()
