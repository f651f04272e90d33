"""Copy the UNMODIFIED reference scripts (pure Python, no build step: there is no setup.py to pip-install) from the
reference checkout (oracle/ref_import.REF) into git-ignored oracle/_ref/.  tests/test_gpu_dropin.py, tests/ref_gpu.py and
bench.py's comparison arms import them from there; nothing in the product imports or copies reference code.
Run by __graft_entry__.build() where the reference checkout exists."""
import os
import shutil
import sys

from oracle.ref_import import REF as SRC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(ROOT, "oracle", "_ref")


def fetch(verbose=True):
    if not os.path.isdir(SRC):
        return False
    os.makedirs(DST, exist_ok=True)
    for f in sorted(os.listdir(SRC)):
        if f.endswith(".py"):
            shutil.copy2(os.path.join(SRC, f), os.path.join(DST, f))
    os.makedirs(os.path.join(DST, "configs"), exist_ok=True)
    for f in sorted(os.listdir(os.path.join(SRC, "configs"))):
        shutil.copy2(os.path.join(SRC, "configs", f), os.path.join(DST, "configs", f))
    if verbose:
        print("[fetch_reference] copied", sorted(os.listdir(DST)))
    return True


if __name__ == "__main__":
    sys.exit(0 if fetch() else 1)
