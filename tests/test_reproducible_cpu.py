"""Static evidence (no GPU needed) that training is reproducible: no kernel of libnerf_b200.so adds floats with atomics, whose
order would depend on scheduling.  Every such sum is written as fp32 partials and reduced in a fixed order instead.  The only
memory reductions left are the max over non-negative float bit patterns of the loss-scale search, which does not depend on
order."""
import os
import re
import shutil
import subprocess

import pytest

MAX_ALLOWED = ("absmax_kernel", "raw2outputs_bwd_kernel")
_MEM_ATOMIC = re.compile(r"\b((?:RED|REDG|ATOM|ATOMG|ATOMS)\.[\w.]+)")


@pytest.fixture(scope="module")
def sass():
    import __graft_entry__ as ge
    ge.build()
    from nerf_pytorch_b200 import _lib
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    return subprocess.run([exe, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=600, check=True).stdout


def atomics_by_function(text):
    """{mangled function name: [memory atomic / reduction mnemonics]} of cuobjdump -sass output"""
    out, cur = {}, None
    for ln in text.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            continue
        if cur is None:
            continue
        code = ln.split("*/", 1)[1] if "*/" in ln else ln
        for op in _MEM_ATOMIC.findall(code):
            out.setdefault(cur, []).append(op)
    return out


def float_add(op):
    """a floating-point atomic / reduction add, or a compare-and-swap (how a float add is emulated where no native one exists)"""
    parts = op.split(".")
    return "CAS" in parts or ("ADD" in parts and any(p in ("F16", "F16x2", "BF16", "BF16x2", "F32", "F64") for p in parts))


def test_classifier_on_known_instructions():
    text = """
        Function : _ZN2nb15mse_seed_kernelEPKfS1_xffPfS2_
        /*0310*/                   REDG.E.ADD.F32.FTZ.RN.STRONG.GPU desc[UR4][R2.64], R5 ;
        Function : _ZN2nb13absmax_kernelEPKfxPj
        /*0200*/              @!P0 REDG.E.MAX.STRONG.GPU desc[UR4][R2.64], R7 ;
        /*0210*/                   REDUX.MAX UR5, R4 ;
        Function : k3
        /*0100*/                   ATOMG.E.CAS.STRONG.GPU PT, R9, [R2], R4, R5 ;
        /*0110*/                   ATOMS.ADD.F16x2.RN R0, [R3], R4 ;
        /*0120*/                   ATOM.E.ADD.F64.RN.STRONG.GPU PT, R4, [R2], R6 ;
        /*0130*/                   RED.E.ADD.STRONG.GPU [R2], R5 ;
    """
    got = atomics_by_function(text)
    assert got["_ZN2nb15mse_seed_kernelEPKfS1_xffPfS2_"] == ["REDG.E.ADD.F32.FTZ.RN.STRONG.GPU"]
    assert got["_ZN2nb13absmax_kernelEPKfxPj"] == ["REDG.E.MAX.STRONG.GPU"]           # REDUX is a warp reduction, not memory
    assert [float_add(o) for o in got["k3"]] == [True, True, True, False]             # integer add is not a float add


def test_no_float_atomics_in_the_library(sass):
    found = atomics_by_function(sass)
    assert any("absmax_kernel" in f for f in found)                                   # the parser sees the library's atomics
    bad = {f: ops for f, ops in found.items() if any(float_add(o) for o in ops)}
    assert not bad, f"float atomic adds (order-dependent sums): {bad}"
    stray = {f: ops for f, ops in found.items()
             if any(o.startswith(("RED", "ATOM")) and "MAX" in o.split(".") for o in ops) and not any(k in f for k in MAX_ALLOWED)}
    assert not stray, f"atomic max outside the loss-scale search: {stray}"
