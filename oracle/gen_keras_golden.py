"""tests/golden/keras_import.npz: what the UNMODIFIED reference's NeRF.load_weights_from_keras (run_nerf_helpers.py:121-148)
makes of a seeded synthetic Keras-style weight list -- the state_dict keys in order, their shapes, and a fixed seeded sample of
64 values per tensor (the whole dict is 4.8 MB).  Needs the reference checkout (oracle/ref_import.py); run from the repo root:
    python -m oracle.gen_keras_golden
"""
import os

import numpy as np

from oracle import ref_import

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(63, 256)] + [(256, 256)] * 4 + [(319, 256)] + [(256, 256)] * 2 + [(256, 256), (283, 128), (128, 3), (256, 1)]
N_SAMPLE = 64


def keras_weights():
    rng = np.random.default_rng(0)
    weights = []
    for (i, o) in SHAPES:
        weights += [rng.standard_normal((i, o)).astype(np.float32), rng.standard_normal((o,)).astype(np.float32)]
    return weights


def sample_index(numel, k):
    return np.random.default_rng(k).choice(numel, size=min(N_SAMPLE, numel), replace=False).astype(np.int64)


def main():
    assert ref_import.available(), "the reference checkout is needed"
    _, rh = ref_import.load()
    r = rh.NeRF(D=8, W=256, input_ch=63, input_ch_views=27, output_ch=5, skips=[4], use_viewdirs=True)
    r.load_weights_from_keras(keras_weights())
    out = {"keys": np.array(list(r.state_dict().keys()))}
    for k, (name, t) in enumerate(r.state_dict().items()):
        a = t.detach().numpy().reshape(-1)
        idx = sample_index(a.size, k)
        out[f"shape_{k}"] = np.array(t.shape, np.int64)
        out[f"idx_{k}"] = idx
        out[f"val_{k}"] = a[idx]
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "keras_import.npz"), **out)


if __name__ == "__main__":
    main()
