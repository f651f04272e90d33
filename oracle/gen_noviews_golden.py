"""Generate tests/golden/lego_noviews_grads.npz by running the UNMODIFIED reference on CPU  --  build container only.

    python oracle/gen_noviews_golden.py        # needs the reference checkout (oracle/ref_import.py); writes tests/golden/

The network the reference builds without --use_viewdirs (its default, run_nerf.py:467): output_linear head with
output_ch = 5 (N_importance > 0, run_nerf.py:187), separate coarse and fine nets.  Same fixture layout as
lego_grads.npz (oracle/gen_golden.py): the inputs, the reference's outputs, loss = img2mse(rgb) + img2mse(rgb0) and
sampled entries of every parameter gradient (g_{c,f}_{name}_{idx,val,norm,sum}).  views_linears.0 exists in that
network but never reaches the loss: the reference's autograd leaves its .grad None, and the fixture has no entry for it.
Parameters are regenerated from oracle/noviews.nerf_state_noviews(seed) and not stored.
"""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import noviews, ref_import, synth  # noqa: E402
from oracle.gen_golden import OUT, load_state, make_args, to_np  # noqa: E402


def run_noviews_grads(rn, name, N=24, N_importance=128, seed_w=0, ray_seed=0):
    sb = synth.ray_batch("lego", N, seed=ray_seed)
    with tempfile.TemporaryDirectory() as tmp:
        args = make_args(tmp, N_importance=N_importance, use_viewdirs=False, white_bkgd=sb["white_bkgd"], perturb=0.0)
        kw_train, _, _, _, _ = rn.create_nerf(args)
    assert not kw_train["use_viewdirs"] and kw_train["network_fn"].output_linear.out_features == 5
    load_state(kw_train["network_fn"], noviews.nerf_state_noviews(seed_w))
    load_state(kw_train["network_fine"], noviews.nerf_state_noviews(seed_w + 1))
    kw = dict(kw_train)
    kw.update(near=sb["near"], far=sb["far"], perturb=0.0, raw_noise_std=0.0)
    fx = dict(rays=sb["rays"], K=sb["K"], H=sb["H"], W=sb["W"], near=sb["near"], far=sb["far"], ndc=sb["ndc"],
              white_bkgd=sb["white_bkgd"], N_samples=64, N_importance=N_importance, seed_w=seed_w, sharpen=False,
              perturb=0.0, lindisp=False, raw_noise_std=0.0, scene="lego", use_viewdirs=False, output_ch=5)
    with torch.enable_grad():
        rgb, disp, acc, extras = rn.render(sb["H"], sb["W"], sb["K"], chunk=1024 * 32, rays=torch.from_numpy(sb["rays"]),
                                           retraw=True, **kw)
        fx.update(rgb_map=to_np(rgb), disp_map=to_np(disp), acc_map=to_np(acc), raw=to_np(extras["raw"]))
        for k in ("rgb0", "disp0", "acc0", "z_std"):
            fx[k] = to_np(extras[k])
        target = torch.from_numpy(np.random.default_rng(5).random((N, 3), dtype=np.float32))
        fx["target"] = to_np(target)
        loss = torch.mean((rgb - target) ** 2) + torch.mean((extras["rgb0"] - target) ** 2)     # run_nerf.py:765-772
        loss.backward()
        fx["loss"] = np.float32(loss.item())
    rng = np.random.default_rng(9)
    for tag, net in (("c", kw_train["network_fn"]), ("f", kw_train["network_fine"])):
        for pname, prm in net.named_parameters():
            if prm.grad is None:                       # views_linears.0: not on the loss's graph
                continue
            g = to_np(prm.grad).reshape(-1)
            idx = rng.integers(0, g.size, min(256, g.size))
            fx[f"g_{tag}_{pname}_idx"] = idx.astype(np.int64)
            fx[f"g_{tag}_{pname}_val"] = g[idx]
            fx[f"g_{tag}_{pname}_norm"] = np.float32(np.linalg.norm(g.astype(np.float64)))
            fx[f"g_{tag}_{pname}_sum"] = np.float32(g.astype(np.float64).sum())
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **fx)
    print("wrote", name, {k: (v.shape if hasattr(v, "shape") else v) for k, v in fx.items() if not k.startswith("g_")})


def main():
    assert ref_import.available(), "reference not found (this script only runs where the reference checkout exists)"
    torch.manual_seed(0)
    torch.set_num_threads(os.cpu_count())
    rn, _ = ref_import.load()
    os.makedirs(OUT, exist_ok=True)
    run_noviews_grads(rn, "lego_noviews_grads")


if __name__ == "__main__":
    main()
