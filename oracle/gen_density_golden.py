"""Generate tests/golden/density_grid.npz by running the UNMODIFIED reference on CPU  --  build container only.

    python oracle/gen_density_golden.py        # needs the reference checkout (oracle/ref_import.py); writes tests/golden/

The density a mesh is extracted from, the way the original NeRF release's extraction notebook takes it: the reference's own
network_query_fn (run_network) on every point of a grid with zero view directions, sigma = raw[..., 3].  The grid is non-uniform
(sorted random axes over the lego scene, 9 x 7 x 12 points), the nets are

    c, f : the trained coarse and fine nets of trained_weights.npz (view directions)
    nv   : a net without view directions (output_ch 5) with the trained fine net's density (oracle/outgrads.noviews_from_trained)

Stored: the axes xs, ys, zs; per net `<n>_sigma` [9, 7, 12] float32 (the reference in float32) and `<n>_sigma64` (the same
reference network in float64: how far float32 itself is from exact); `weights_sha256` (the digest of trained_weights.npz the
nets were loaded from).  Parameters are not stored.
"""
import hashlib
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import outgrads, ref_import  # noqa: E402
from oracle.gen_golden import OUT, load_state, make_args, to_np  # noqa: E402

SHAPE = (9, 7, 12)


def axes(seed=0):
    rng = np.random.default_rng(seed)
    return [np.sort(rng.uniform(-1.3, 1.3, n)).astype(np.float32) for n in SHAPE]


def sigma_of(kw, net, xs, ys, zs, dtype, views):
    pts = torch.stack(torch.meshgrid(*(torch.from_numpy(a).to(dtype) for a in (xs, ys, zs)), indexing="ij"), -1)
    dirs = torch.zeros(pts.numel() // 3, 3, dtype=dtype) if views else None
    with torch.no_grad():
        raw = kw["network_query_fn"](pts.reshape(-1, 1, 3), dirs, net)
    return to_np(raw[..., 3]).reshape(SHAPE)


def main():
    assert ref_import.available(), "reference not found (this script only runs where the reference checkout exists)"
    torch.manual_seed(0)
    torch.set_num_threads(8)
    rn, _ = ref_import.load()
    path = os.path.join(OUT, "trained_weights.npz")
    trained = outgrads.trained_states(path)
    xs, ys, zs = axes()
    fx = {"xs": xs, "ys": ys, "zs": zs, "weights_sha256": np.frombuffer(hashlib.sha256(open(path, "rb").read()).digest(), np.uint8)}
    for views in (True, False):
        with tempfile.TemporaryDirectory() as tmp:
            kw, _, _, _, _ = rn.create_nerf(make_args(tmp, use_viewdirs=views, perturb=0.0))
        if views:
            nets = (("c", kw["network_fn"], trained[0]), ("f", kw["network_fine"], trained[1]))
        else:
            nets = (("nv", kw["network_fine"], outgrads.noviews_from_trained(trained[1], 1)),)
        for tag, net, state in nets:
            load_state(net, state)
            fx[tag + "_sigma"] = sigma_of(kw, net, xs, ys, zs, torch.float32, views).astype(np.float32)
            fx[tag + "_sigma64"] = sigma_of(kw, net.double(), xs, ys, zs, torch.float64, views)
            net.float()
    np.savez_compressed(os.path.join(OUT, "density_grid.npz"), **fx)
    for k, v in fx.items():
        if k.endswith("_sigma"):
            print(k, "min %.3g max %.3g  >0: %.2f" % (v.min(), v.max(), float(np.mean(v > 0))))


if __name__ == "__main__":
    main()
