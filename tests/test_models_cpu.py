"""The ensemble forward (dsmil_forward_bags_models, ensemble.forward_bags_models) without a GPU: the exported symbols,
argument validation that returns before any CUDA work, the workspace sizes, which ensembles run fused, and the
Python-side refusals."""
import ctypes as C
import os
import re

import pytest
import torch

from dsmil_wsi_b200 import _lib

ERR_ARG, ERR_WORKSPACE = -1, -2
FAKE = 0x10000          # a non-NULL, 16-byte aligned "device pointer": never dereferenced on these paths
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("dsmil_models_supported", "dsmil_forward_bags_models_workspace_bytes", "dsmil_forward_bags_models")


def params(D=512, C_=2, nonlinear=1, passing_v=0, **over):
    p = _lib.DsmilParams(D, C_, nonlinear, passing_v)
    for name in ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf"):
        setattr(p, name, FAKE)
    for k, v in over.items():
        setattr(p, k, v)
    return p


def arr(ps):
    return (_lib.DsmilParams * len(ps))(*ps)


def i64(xs):
    return (C.c_int64 * len(xs))(*xs)


def ptrs(n, addr=FAKE):
    return (C.c_void_p * n)(*([addr] * n))


def last_error(lib):
    return (lib.dsmil_last_error() or b"").decode()


def call(lib, ps, M, Ns, Xs=None, outs=(FAKE,) * 5, ws=None, ws_bytes=0):
    nb = len(Ns)
    Xs = ptrs(nb) if Xs is None else Xs
    return lib.dsmil_forward_bags_models(ps, M, Xs, i64(Ns), nb, *outs, ws, ws_bytes, None)


def ws_bytes(lib, ps, M, Ns):
    return lib.dsmil_forward_bags_models_workspace_bytes(ps, M, i64(Ns), len(Ns))


def test_symbols_exported_declared_and_bound():
    lib = _lib.load()
    header = open(os.path.join(ROOT, "include", "dsmil_b200.h")).read()
    for name in NAMES:
        assert re.search(rf"\b{name}\s*\(", header), name
        assert hasattr(lib, name), name
        assert name in _lib.SIGNATURES, name


@pytest.mark.parametrize("M", [0, 9, -1])
def test_model_count_out_of_range(M):
    lib = _lib.load()
    ps = arr([params() for _ in range(8)])
    assert call(lib, ps, M, [100]) == ERR_ARG
    assert "M=" in last_error(lib)
    assert not lib.dsmil_models_supported(ps, M)
    assert ws_bytes(lib, ps, M, [100]) == 0


def test_null_params_and_outputs():
    lib = _lib.load()
    assert call(lib, None, 2, [100]) == ERR_ARG and "params is NULL" in last_error(lib)
    assert not lib.dsmil_models_supported(None, 2)
    assert ws_bytes(lib, None, 2, [100]) == 0
    ps = arr([params(), params()])
    for i in range(4):                     # classes, pred, A, B; crit_idx may be NULL
        outs = [FAKE] * 5
        outs[i] = None
        assert call(lib, ps, 2, [100], outs=tuple(outs)) == ERR_ARG and "NULL" in last_error(lib)
    nb = 1
    assert lib.dsmil_forward_bags_models(ps, 2, None, i64([100]), nb, *([FAKE] * 5), None, 0, None) == ERR_ARG
    assert lib.dsmil_forward_bags_models(ps, 2, ptrs(1), None, nb, *([FAKE] * 5), None, 0, None) == ERR_ARG
    assert call(lib, ps, 2, [100], Xs=ptrs(1, 0)) == ERR_ARG        # a NULL bag
    # a member that fails the one-model checks
    assert call(lib, arr([params(), params(Wi=None)]), 2, [100]) == ERR_ARG
    assert "instance-classifier" in last_error(lib)


@pytest.mark.parametrize("field,other", [
    ("D", dict(D=1024)), ("C", dict(C_=1)), ("nonlinear", dict(nonlinear=0, W2=None, b2=None)),
    ("passing_v", dict(passing_v=1)),
])
def test_members_must_share_shape(field, other):
    lib = _lib.load()
    ps = arr([params(), params(), params(**other)])
    assert call(lib, ps, 3, [100, 7]) == ERR_ARG
    msg = last_error(lib)
    assert "model 2" in msg and field in msg
    assert not lib.dsmil_models_supported(ps, 3)


def test_short_workspace():
    lib = _lib.load()
    for ps, M in ((arr([params()] * 5), 5), (arr([params(D=166, C_=1)] * 3), 3)):   # fused and looped shapes
        need = ws_bytes(lib, ps, M, [10_000, 129])
        assert need > 0
        assert call(lib, ps, M, [10_000, 129], ws=None, ws_bytes=0) == ERR_WORKSPACE
        assert call(lib, ps, M, [10_000, 129], ws=FAKE, ws_bytes=need - 1) == ERR_WORKSPACE
        assert "workspace too small" in last_error(lib)


@pytest.mark.parametrize("D,C_", [(512, 1), (512, 2), (1024, 2), (1024, 4), (2048, 2), (166, 1)])
def test_workspace_monotone_and_covers_one_model(D, C_):
    lib = _lib.load()
    base = [10_000, 1, 127, 128, 129]
    for M in range(1, 9):
        ps = arr([params(D, C_)] * M)
        one = lib.dsmil_forward_bags_workspace_bytes(C.byref(ps[0]), i64(base), len(base))
        assert ws_bytes(lib, ps, M, base) >= one > 0
        if M > 1:
            assert ws_bytes(lib, ps, M, base) >= ws_bytes(lib, arr([params(D, C_)] * (M - 1)), M - 1, base)
        assert ws_bytes(lib, ps, M, base + [64]) >= ws_bytes(lib, ps, M, base)          # nb
        assert ws_bytes(lib, ps, M, base[:-1] + [1000]) >= ws_bytes(lib, ps, M, base)   # N
    # the fused layout holds M sets of Q tile blocks: about M x the one-model size
    ps5 = arr([params()] * 5)
    one = lib.dsmil_forward_bags_workspace_bytes(C.byref(ps5[0]), i64([10_000] * 16), 16)
    assert ws_bytes(lib, ps5, 5, [10_000] * 16) >= 5 * 16 * 79 * 128 * 128 * 4 > 4 * one


@pytest.mark.parametrize("D,C_", [(512, 1), (512, 2), (1024, 1), (1024, 2), (1024, 4), (2048, 1), (2048, 2)])
def test_reference_configurations_run_fused_at_five_models(D, C_):
    lib = _lib.load()
    for M in (1, 2, 5):
        assert lib.dsmil_models_supported(arr([params(D, C_)] * M), M) == 1, (D, C_, M)


def test_eight_models_fused_at_512():
    lib = _lib.load()
    assert lib.dsmil_models_supported(arr([params(512, 2)] * 8), 8) == 1


@pytest.mark.parametrize("kw", [dict(passing_v=1), dict(nonlinear=0, W2=None, b2=None), dict(D=166, C_=1),
                                dict(D=512, C_=8), dict(D=4096, C_=1)])
def test_off_the_batched_path_is_not_fused(kw):
    lib = _lib.load()
    assert lib.dsmil_models_supported(arr([params(**kw)] * 2), 2) == 0
    # still a valid call: the loop over dsmil_forward_bags serves it, in a workspace it sizes
    assert ws_bytes(lib, arr([params(**kw)] * 2), 2, [100, 3]) > 0


def test_weights_that_do_not_fit_shared_memory_are_not_fused():
    lib = _lib.load()
    assert lib.dsmil_models_supported(arr([params(2048, 2)] * 8), 8) == 0


# ---- Python refusals (raised before any library call) ------------------------------------------------------------
def _net(D=32, C_=2, nonlinear=True, passing_v=False, ic=None):
    import dsmil as mil
    return mil.MILNet(ic if ic is not None else mil.FCLayer(D, C_),
                      mil.BClassifier(D, C_, nonlinear=nonlinear, passing_v=passing_v))


@pytest.mark.parametrize("other,needle", [
    (dict(D=64), "D=64"), (dict(C_=1), "C=1"), (dict(nonlinear=False), "nonlinear=False"),
])
def test_ensemble_refuses_mismatched_members(other, needle):
    from dsmil_wsi_b200.ensemble import forward_bags_models
    with pytest.raises(ValueError, match=f"member 1: {needle}"):
        forward_bags_models([_net(), _net(**other)], [torch.zeros(4, 32)])


def test_ensemble_refuses_members_on_different_devices():
    from dsmil_wsi_b200.ensemble import forward_bags_models
    a, b = _net(), _net().to("meta")
    with pytest.raises(ValueError, match="member 1 is on meta"):
        forward_bags_models([a, b], [torch.zeros(4, 32)])


def test_ensemble_refuses_passing_v_and_foreign_members():
    import torch.nn as nn
    from dsmil_wsi_b200.ensemble import forward_bags_models
    with pytest.raises(ValueError, match="member 1: .*identity v"):
        forward_bags_models([_net(), _net(passing_v=True)], [torch.zeros(4, 32)])
    with pytest.raises(TypeError, match="member 0"):
        forward_bags_models([nn.Linear(3, 3)], [torch.zeros(4, 32)])
    with pytest.raises(ValueError, match="1 to 8"):
        forward_bags_models([_net()] * 9, [torch.zeros(4, 32)])
    with pytest.raises(ValueError, match="1 to 8"):
        forward_bags_models([], [torch.zeros(4, 32)])
