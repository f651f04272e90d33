"""Static checks of the split training path (set_backward('tc_split')) in the cross-compiled sm_90a library, no GPU needed:
its kernels exist, the MMA kernels issue warpgroup MMAs on bulk-copied operands with saturating fp16 epilogues, and stay in their
register budget without local memory (as the fp16 kernels they are built from)."""
import os
import re
import shutil
import subprocess

import pytest


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    ge.build()
    from nerf_pytorch_b200 import _lib
    return _lib.LIB_PATH


def _cuobjdump(path, flag):
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    return subprocess.run([exe, flag, path], capture_output=True, text=True, timeout=600).stdout


def _bodies(sass):
    bodies, cur = {}, None
    for ln in sass.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1); bodies[cur] = []
        elif cur is not None:
            bodies[cur].append(ln)
    return bodies


def _one(bodies, name):
    names = [k for k in bodies if re.search(r"\b_ZN2nb\d+" + name + r"E", k)]
    assert len(names) == 1, (name, names)
    return "\n".join(bodies[names[0]])


def test_split_training_kernels_in_sass(built):
    bodies = _bodies(_cuobjdump(built, "-sass"))
    fwd, dgrad = _one(bodies, "march_split_train_kernel"), _one(bodies, "dgrad_split_kernel")
    for b in (fwd, dgrad):
        for mnem in ("HGMMA.64x256x16.F32", "UBLKCP.S.G", "UBLKCP.G.S", "SYNCS.PHASECHK.TRANS64.TRYWAIT", "USETMAXREG"):
            assert mnem in b, mnem
        assert "HMMA.16816" not in b
    assert "HGMMA.64x128x16.F32" in fwd                                 # the view layer
    assert "F2FP.SATFINITE" in dgrad                                    # hi and lo of the activation gradients saturate
    for name in ("dhv_seed_heads_split_kernel", "dA_seed_output_split_kernel"):
        assert "F2FP.SATFINITE" in _one(bodies, name), name
    assert not re.search(r"\b(STL|LDL)\b", dgrad)
    # the existing kernels keep one entry each (the split variants have their own names)
    for name in ("march_wg_kernel", "dgrad_wg_kernel", "wgrad_wg_kernel", "dA_seed_output_kernel"):
        assert len([k for k in bodies if name in k]) == (2 if name == "march_wg_kernel" else 1), name


def test_split_mma_kernels_fit_their_resource_budget(built):
    """dgrad_split_kernel: 168 registers at launch (384 threads, one CTA per SM), no stack; march_split_train_kernel: the stack of
    the inference split kernel it shares its code with (the sincosf-free encoding's sinf / cosf slow-path buffer), no more."""
    usage = _cuobjdump(built, "-res-usage").splitlines()

    def res(name):
        found = [usage[i + 1] for i, ln in enumerate(usage[:-1]) if re.search(r"Function _ZN2nb\d+" + name + r"E\S*:", ln)]
        assert len(found) == 1, (name, found)
        m = re.search(r"REG:(\d+) STACK:(\d+)", found[0])
        return int(m.group(1)), int(m.group(2))
    reg, stack = res("dgrad_split_kernel")
    assert reg <= 168 and stack == 0
    reg, stack = res("march_split_train_kernel")
    assert reg <= 168 and stack <= res("march_split_kernel")[1]
