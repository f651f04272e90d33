"""Generate tests/golden/outgrads.npz by running the UNMODIFIED reference on CPU  --  build container only.

    python oracle/gen_outgrads_golden.py        # needs the reference checkout (oracle/ref_import.py); writes tests/golden/

Losses that read more of render()'s outputs than rgb_map, each backpropagated on its own through the reference's autograd:

    L_acc  = mse(acc, t_a) + mse(acc0, t_a)
    L_disp = mean(disp) + mean(disp0)
    L_raw  = mean(relu(raw[..., 3])) + mean(raw[..., :3]^2)
    L_all  = img2mse(rgb) + img2mse(rgb0) + L_acc + 0.1 L_disp + 1e-3 L_raw

on three cases:

    a: the trained nets of trained_weights.npz, 256 lego rays, view directions, white background, 64 + 128 samples
    b: a net without view directions (output_ch 5) with the trained density (oracle/outgrads.noviews_from_trained), 64 lego
       rays, 64 + 128
    c: the trained nets on 64 fern NDC rays, perturb and raw_noise_std = 1 through the reference's pytest=True draws, 64 + 64

Stored per case `x` and loss `l` (acc, disp, raw, all), keys prefixed `x_l_`: the loss value, sampled parameter gradients
(g_{c,f}_{val,norm,on}: per net, over its named_parameters()) with, per tensor, the rel-L2 distance of those
sampled entries from the same reference run in float64 (g_{c,f}_cond: the loss's conditioning at fp32), and for each raw2outputs call i (0 coarse,
1 fine) of N_KEEP rays the reference's dL/draw (`r2o{i}_draw`) with the gradients autograd handed to that call's outputs
(`r2o{i}_g_{rgb_map,...}`).  Per case, keys prefixed `x_`: the inputs (rays, K, H, W, near, far, ...), the targets, the
sampled entries g_{c,f}_{names,count,idx} (int32, N_SAMPLED per tensor, concatenated in named_parameters() order, shared
by the losses), the kept rays `r2o_rays` (the first
N_KEEP that are neither empty nor opaque in both passes) and each call's raw / z_vals / rays_d / noise of those rays.
Parameters are regenerated, not stored.
"""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import outgrads, ref_import, synth  # noqa: E402
from oracle.gen_golden import OUT, load_state, make_args, to_np  # noqa: E402
from oracle.outgrads import LOSSES, loss_of  # noqa: E402

N_KEEP = 2                   # rays whose dL/draw is stored (per call, case and loss)
N_SAMPLED = 64               # sampled entries per parameter gradient
OUT_NAMES = ("rgb_map", "disp_map", "acc_map", "weights", "depth_map")       # raw2outputs' return order (run_nerf.py:305)


def spy_grads(rn, raw_noise_std, pytest):
    """Wrap the reference's raw2outputs: keep each call's inputs and retain the gradients of its raw and outputs.
    -> (record list, restore function)."""
    rec = []
    orig = rn.raw2outputs

    def spy(raw, z_vals, rays_d, *a, **k):
        raw.retain_grad()
        # identity copies: their .grad is what the caller's loss hands to each output (acc and disp are computed from the
        # weights and depth the reference returns, so the originals' retained gradients would include those terms)
        out = tuple(o.clone() for o in orig(raw, z_vals, rays_d, *a, **k))
        for o in out:
            if o.requires_grad:
                o.retain_grad()
        noise = np.zeros(z_vals.shape, np.float32)
        if raw_noise_std > 0 and pytest:                 # the draw the reference's pytest hook makes (run_nerf.py:287-291)
            np.random.seed(0)
            noise = (np.random.rand(*list(z_vals.shape)) * raw_noise_std).astype(np.float32)
        rec.append(dict(raw=raw, out=out, inputs=dict(raw=to_np(raw[..., :4]), z=to_np(z_vals), d=to_np(rays_d), noise=noise)))
        return out
    rn.raw2outputs = spy
    return rec, lambda: setattr(rn, "raw2outputs", orig)


def keep_rays(acc, acc0):
    """the first N_KEEP rays that are neither empty nor opaque in both passes: there an acc or disp seed has a gradient that
    is not ~0 (an opaque ray's acc is exactly 1 and its acc gradient rounding noise)"""
    a, a0 = acc.detach().numpy(), acc0.detach().numpy()
    ok = np.flatnonzero((a > 0.05) & (a < 0.995) & (a0 > 0.05) & (a0 < 0.995))
    assert ok.size >= N_KEEP, ok
    return ok[:N_KEEP].astype(np.int64)


def grads_f64(rn, nets, sb, kw, pytest, lname, target, t_acc):
    """the same render + loss + backward with the reference running in float64 (default dtype, parameters and rays): how far
    the reference's own fp32 gradient is from the exact one measures the loss's conditioning (e.g. mean(disp) over nearly
    empty rays, where the gradient grows like 1 / acc)"""
    import copy
    torch.set_default_dtype(torch.float64)
    try:
        nets64 = [copy.deepcopy(n).double() for n in nets]
        for n in nets64:
            n.zero_grad(set_to_none=True)
        kw64 = dict(kw, network_fn=nets64[0], network_fine=nets64[1])
        with torch.enable_grad():
            rgb, disp, acc, ex = rn.render(sb["H"], sb["W"], sb["K"], chunk=1024 * 32, rays=torch.from_numpy(sb["rays"]).double(),
                                           retraw=True, pytest=pytest, **kw64)
            loss_of(lname, rgb, disp, acc, ex, target.double(), t_acc.double()).backward()
    finally:
        torch.set_default_dtype(torch.float32)
    return nets64


def run_case(rn, fx, tag, nets, sb, kw, pytest, raw_noise_std):
    N = sb["rays"].shape[1]
    fx.update({f"{tag}_{k}": v for k, v in dict(rays=sb["rays"], K=sb["K"], H=sb["H"], W=sb["W"], near=sb["near"], far=sb["far"],
                                                    ndc=sb["ndc"], white_bkgd=sb["white_bkgd"]).items()})
    rng = np.random.default_rng(21)
    target = torch.from_numpy(rng.random((N, 3), dtype=np.float32))
    t_acc = torch.from_numpy(rng.random((N,), dtype=np.float32))
    fx[f"{tag}_target"], fx[f"{tag}_t_acc"] = to_np(target), to_np(t_acc)
    # sampled parameter entries: one draw per case, shared by its losses; per net one array over its named_parameters()
    srng = np.random.default_rng(9)
    idx = {}
    for ntag, net in zip(("c", "f"), nets):
        names = [n for n, _ in net.named_parameters()]
        idx[ntag] = [srng.integers(0, prm.numel(), min(N_SAMPLED, prm.numel())).astype(np.int32) for _, prm in net.named_parameters()]
        fx[f"{tag}_g_{ntag}_names"] = np.array(names)
        fx[f"{tag}_g_{ntag}_count"] = np.array([len(i) for i in idx[ntag]], np.int32)
        fx[f"{tag}_g_{ntag}_idx"] = np.concatenate(idx[ntag])
    keep = None
    for lname in LOSSES:
        for net in nets:
            for p in net.parameters():
                p.grad = None
        rec, restore = spy_grads(rn, raw_noise_std, pytest)
        try:
            with torch.enable_grad():
                rgb, disp, acc, ex = rn.render(sb["H"], sb["W"], sb["K"], chunk=1024 * 32, rays=torch.from_numpy(sb["rays"]),
                                               retraw=True, pytest=pytest, **kw)
                loss = loss_of(lname, rgb, disp, acc, ex, target, t_acc)
                loss.backward()
        finally:
            restore()
        p = f"{tag}_{lname}_"
        fx[p + "loss"] = np.float32(loss.item())
        assert len(rec) == 2, len(rec)
        if keep is None:
            keep = keep_rays(acc, ex["acc0"])
            fx[f"{tag}_r2o_rays"] = keep
            for i, r in enumerate(rec):
                for k, v in r["inputs"].items():
                    fx[f"{tag}_r2o{i}_{k}"] = v[keep]
        for i, r in enumerate(rec):
            g = r["raw"].grad
            fx[p + f"r2o{i}_draw"] = to_np(g[keep][..., :4]) if g is not None else np.zeros_like(fx[f"{tag}_r2o{i}_raw"])
            for nm, o in zip(OUT_NAMES, r["out"]):
                if o.grad is not None:
                    fx[p + f"r2o{i}_g_{nm}"] = to_np(o.grad[keep])
        nets64 = grads_f64(rn, nets, sb, kw, pytest, lname, target, t_acc)
        for ntag, net, net64 in zip(("c", "f"), nets, nets64):
            vals, norms, on, cond = [], [], [], []
            for (pname, prm), (_, p64), ii in zip(net.named_parameters(), net64.named_parameters(), idx[ntag]):
                if prm.grad is not None:               # rel-L2 of fp32 vs float64 on the sampled entries
                    g32, g64 = prm.grad.double().reshape(-1)[ii], p64.grad.reshape(-1)[ii]
                    cond.append(float((g32 - g64).norm() / g64.norm().clamp_min(1e-300)))
                else:
                    cond.append(0.0)
                # .grad None: not on this loss's graph (views_linears.0 without view directions; the coarse net under L_raw,
                # which reads the fine pass's raw) -- stored as zeros with on = False
                gg = to_np(prm.grad).reshape(-1) if prm.grad is not None else np.zeros(prm.numel(), np.float32)
                vals.append(gg[ii])
                norms.append(np.linalg.norm(gg.astype(np.float64)))
                on.append(prm.grad is not None)
            fx[p + f"g_{ntag}_val"] = np.concatenate(vals)
            fx[p + f"g_{ntag}_norm"] = np.array(norms, np.float32)
            fx[p + f"g_{ntag}_on"] = np.array(on)
            fx[p + f"g_{ntag}_cond"] = np.array(cond, np.float32)
        print(tag, lname, "loss", float(loss.item()), flush=True)


def main():
    assert ref_import.available(), "reference not found (this script only runs where the reference checkout exists)"
    torch.manual_seed(0)
    torch.set_num_threads(8)                      # fixed: CPU reductions are then reproducible bit for bit
    rn, _ = ref_import.load()
    fx = {}
    # a: trained nets, 256 lego rays, view directions
    sb = synth.ray_batch("lego", 256, seed=12)
    with tempfile.TemporaryDirectory() as tmp:
        kw, _, _, _, _ = rn.create_nerf(make_args(tmp, perturb=0.0))
    stored = np.load(os.path.join(OUT, "trained_weights.npz"))
    for t, key in (("c", "network_fn"), ("f", "network_fine")):
        load_state(kw[key], {k[2:]: stored[k] for k in stored.files if k.startswith(t + ".")})
    kw = dict(kw); kw.update(near=sb["near"], far=sb["far"], perturb=0.0, raw_noise_std=0.0)
    run_case(rn, fx, "a", (kw["network_fn"], kw["network_fine"]), sb, kw, False, 0.0)
    # b: no view directions, output_ch 5, with the trained density (outgrads.noviews_from_trained)
    trained = outgrads.trained_states(os.path.join(OUT, "trained_weights.npz"))
    sb = synth.ray_batch("lego", 64, seed=3)
    with tempfile.TemporaryDirectory() as tmp:
        kw, _, _, _, _ = rn.create_nerf(make_args(tmp, use_viewdirs=False, white_bkgd=sb["white_bkgd"], perturb=0.0))
    assert kw["network_fn"].output_linear.out_features == 5
    load_state(kw["network_fn"], outgrads.noviews_from_trained(trained[0], 0))
    load_state(kw["network_fine"], outgrads.noviews_from_trained(trained[1], 1))
    kw = dict(kw); kw.update(near=sb["near"], far=sb["far"], perturb=0.0, raw_noise_std=0.0)
    run_case(rn, fx, "b", (kw["network_fn"], kw["network_fine"]), sb, kw, False, 0.0)
    # c: the trained nets on fern NDC rays, perturb + raw_noise_std = 1 through the pytest draws
    sb = synth.ray_batch("fern", 64, seed=5)
    with tempfile.TemporaryDirectory() as tmp:
        kw, _, _, _, _ = rn.create_nerf(make_args(tmp, N_importance=64, white_bkgd=sb["white_bkgd"], dataset_type="llff",
                                                  raw_noise_std=1.0, perturb=1.0))
    load_state(kw["network_fn"], trained[0])
    load_state(kw["network_fine"], trained[1])
    kw = dict(kw); kw.update(near=sb["near"], far=sb["far"], perturb=1.0, raw_noise_std=1.0)
    run_case(rn, fx, "c", (kw["network_fn"], kw["network_fine"]), sb, kw, True, 1.0)
    os.makedirs(OUT, exist_ok=True)
    np.savez_compressed(os.path.join(OUT, "outgrads.npz"), **fx)
    print("wrote outgrads", len(fx), "arrays")


if __name__ == "__main__":
    main()
