import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def golden_names():
    return sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz"))


def load_golden(name):
    """Returns (fixture dict, Params, X) with inputs regenerated from the stored seeds."""
    import zlib
    from oracle import dsmil_oracle as orc
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    D, C, N = int(g["D"]), int(g["C"]), int(g["N"])
    if "w_Wi" in g:  # shipped checkpoints: weights stored
        p = orc.Params(g["w_Wi"], g["w_bi"], g["w_Wf"], g["w_bf"], g["w_W1"], g["w_b1"], g["w_W2"], g["w_b2"])
        xseed = {"shipped_tcga": 0, "shipped_c16": 1}[name]
        kind = "uniform"
    else:
        p = orc.random_params(D, C, int(g["wseed"]), nonlinear=bool(g["nonlinear"]), passing_v=bool(g["passing_v"]),
                              scale=float(g["wscale"]))
        assert np.uint32(zlib.crc32(p.W1.tobytes())) == g["w_crc"], "numpy RNG stream drifted (weights)"
        xseed, kind = int(g["xseed"]), str(g["kind"])
    X = orc.synthetic_bag(N, D, xseed, kind)
    assert np.uint32(zlib.crc32(X.tobytes())) == g["x_crc"], "numpy RNG stream drifted (features)"
    return g, p, X


def rel_to_max(a, b):
    """max |a-b| relative to max |b| (per-tensor; grads differ by orders of magnitude across tensors)."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    den = max(float(np.max(np.abs(b))) if b.size else 0.0, 1e-30)
    return float(np.max(np.abs(a - b))) / den if b.size else 0.0
