"""Drop the H100 path into the UNMODIFIED reference script.

`run_nerf.train()` resolves `create_nerf`, `render`, `render_path` (-> `render`) and, through them,
`batchify_rays`, `render_rays`, `raw2outputs`, `sample_pdf`, `NeRF`, `get_embedder` as module
globals at call time (SURVEY.md 8b), so rebinding those attributes on the imported module swaps
the implementation with run_nerf.py byte-for-byte unchanged:

    import run_nerf                      # the reference, on sys.path
    import nerf_pytorch_b200.dropin as dropin
    dropin.patch(run_nerf)               # rebinding only; no reference source is modified
    run_nerf.train()
"""
import torch

from . import api

# get_rays / ndc_rays / get_rays_np stay the reference's own (per-image glue of train(), run_nerf.py:677-757; inside render()
# the same arithmetic is nerf_b200_pack_rays).
PATCHED = ["render", "render_rays", "batchify_rays", "batchify", "run_network", "raw2outputs", "create_nerf",
           "sample_pdf", "get_embedder", "Embedder", "NeRF"]


def patch(module, set_default_device=True):
    """Rebind the hot-path names of `module` (the imported reference `run_nerf`) to nerf_b200's.

    The reference relies on a CUDA default tensor type set under `__main__` (run_nerf.py:876) for its
    device-less constructors; a programmatic launcher must do the same, hence set_default_device."""
    if not torch.cuda.is_available():
        raise RuntimeError("nerf_b200.dropin: a CUDA device is required (no CPU fallback exists)")
    for name in PATCHED:
        setattr(module, name, getattr(api, name))
    module.device = torch.device("cuda")
    if set_default_device:
        torch.set_default_device("cuda")
    return module


def unpatch_names():
    return list(PATCHED)
