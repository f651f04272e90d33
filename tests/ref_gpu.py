"""The UNMODIFIED reference (oracle/_ref, oracle/fetch_reference.py) on cuda:0, for the -m gpu tests: its own create_nerf /
render with given weights, fp32 or TF32 matmuls (TF32 is the default of the reference's pinned torch 1.11)."""
import argparse
import importlib.util
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")


def available():
    return os.path.isfile(os.path.join(REF, "run_nerf.py")) and torch.cuda.is_available()


def load(alias="run_nerf_ref_gpu"):
    for name in ("imageio", "matplotlib", "matplotlib.pyplot", "configargparse"):
        sys.modules.setdefault(name, types.ModuleType(name))
    if REF not in sys.path:
        sys.path.insert(0, REF)
    spec = importlib.util.spec_from_file_location(alias, os.path.join(REF, "run_nerf.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def render(mod, state_c, state_f, H, W, K, rays, tf32, ndc=False, near=2., far=6., white_bkgd=True):
    """-> dict of numpy outputs of the reference's render() under no_grad on cuda:0"""
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = tf32
    torch.backends.cudnn.allow_tf32 = tf32
    torch.set_default_tensor_type("torch.cuda.FloatTensor")
    try:
        tmp = tempfile.mkdtemp()
        os.makedirs(os.path.join(tmp, "e"), exist_ok=True)
        args = argparse.Namespace(multires=10, multires_views=4, i_embed=0, use_viewdirs=True, N_importance=128, N_samples=64, netdepth=8, netwidth=256,
                                  netdepth_fine=8, netwidth_fine=256, netchunk=65536, lrate=5e-4, basedir=tmp, expname="e", ft_path=None, no_reload=True,
                                  perturb=0.0, white_bkgd=white_bkgd, raw_noise_std=0.0, dataset_type="llff" if ndc else "blender", no_ndc=False, lindisp=False)
        tr, te, _, _, _ = mod.create_nerf(args)
        te["network_fn"].load_state_dict({k: torch.from_numpy(np.asarray(v)).cuda() for k, v in state_c.items()})
        te["network_fine"].load_state_dict({k: torch.from_numpy(np.asarray(v)).cuda() for k, v in state_f.items()})
        te.update(near=near, far=far)
        with torch.no_grad():
            rgb, disp, acc, ex = mod.render(H, W, K, chunk=32768, rays=torch.from_numpy(rays).cuda(), **te)
        return {"rgb_map": rgb.cpu().numpy(), "disp_map": disp.cpu().numpy(), "acc_map": acc.cpu().numpy(), "rgb0": ex["rgb0"].cpu().numpy(),
                "acc0": ex["acc0"].cpu().numpy(), "z_std": ex["z_std"].cpu().numpy()}
    finally:
        torch.set_default_tensor_type("torch.FloatTensor")
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
