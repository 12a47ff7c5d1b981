"""The fold step (dsmil_forward_bags_models_train, dsmil_backward_bags_models, ensemble.forward_bags_per_model,
feed.train_epoch_models) without a GPU: the exported symbols, argument validation that returns before any CUDA work,
the workspace sizes, the Python-side refusals and the step schedule over folds of unequal length."""
import ctypes as C
import os
import re

import pytest
import torch

from dsmil_wsi_b200 import _lib, feed

ERR_ARG, ERR_WORKSPACE = -1, -2
FAKE = 0x10000          # a non-NULL, 16-byte aligned "device pointer": never dereferenced on these paths
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("dsmil_forward_bags_models_train_workspace_bytes", "dsmil_forward_bags_models_train",
         "dsmil_backward_bags_models_workspace_bytes", "dsmil_backward_bags_models")


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


def i32(xs):
    return (C.c_int32 * len(xs))(*xs)


def ptrs(n, addr=FAKE):
    return (C.c_void_p * n)(*([addr] * n))


def last_error(lib):
    return (lib.dsmil_last_error() or b"").decode()


def fwd(lib, ps, M, Ns, nbs, Xs=None, outs=(FAKE,) * 7, ws=None, ws_bytes=0):
    Xs = ptrs(len(Ns)) if Xs is None else Xs
    return lib.dsmil_forward_bags_models_train(ps, M, Xs, i64(Ns), i32(nbs), *outs, ws, ws_bytes, None)


def grads(M, **over):
    g = (_lib.DsmilGrads * M)()
    for m in range(M):
        for name, _ in _lib.DsmilGrads._fields_:
            setattr(g[m], name, over.get(name, FAKE if name != "gX" else None))
    return g


def bwd(lib, ps, M, Ns, nbs, Xs=None, ins=(FAKE,) * 5, g=None, ws=None, ws_bytes=0):
    Xs = ptrs(len(Ns)) if Xs is None else Xs
    g = grads(M) if g is None else g
    return lib.dsmil_backward_bags_models(ps, M, Xs, i64(Ns), i32(nbs), *ins, FAKE, FAKE, None, None, g, ws, ws_bytes,
                                          None)


def fwd_ws(lib, ps, M, Ns, nbs):
    return lib.dsmil_forward_bags_models_train_workspace_bytes(ps, M, i64(Ns), i32(nbs))


def bwd_ws(lib, ps, M, Ns, nbs, gX=0):
    return lib.dsmil_backward_bags_models_workspace_bytes(ps, M, i64(Ns), i32(nbs), gX)


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
    ps = arr([params() for _ in range(9)])
    Ns, nbs = [100] * 9, [1] * 9
    assert fwd(lib, ps, M, Ns, nbs) == ERR_ARG and "M=" in last_error(lib)
    assert bwd(lib, ps, M, Ns, nbs, g=grads(9)) == ERR_ARG and "M=" in last_error(lib)
    assert fwd_ws(lib, ps, M, Ns, nbs) == 0
    assert bwd_ws(lib, ps, M, Ns, nbs) == 0


def test_null_arguments():
    lib = _lib.load()
    assert fwd(lib, None, 2, [100, 5], [1, 1]) == ERR_ARG and "params is NULL" in last_error(lib)
    assert bwd(lib, None, 2, [100, 5], [1, 1]) == ERR_ARG and "params is NULL" in last_error(lib)
    ps = arr([params(), params()])
    Ns, nbs = [100, 5], [1, 1]
    for i in range(7):                     # classes, pred, A, B, crit_idx, save_Q, save_H1 (nonlinear q)
        outs = [FAKE] * 7
        outs[i] = None
        assert fwd(lib, ps, 2, Ns, nbs, outs=tuple(outs)) == ERR_ARG and "NULL" in last_error(lib)
    for i in range(5):                     # Q, H1 (nonlinear q), A, B, crit_idx
        ins = [FAKE] * 5
        ins[i] = None
        assert bwd(lib, ps, 2, Ns, nbs, ins=tuple(ins)) == ERR_ARG
    assert lib.dsmil_backward_bags_models(ps, 2, ptrs(2), i64(Ns), i32(nbs), *([FAKE] * 9), None, None, 0,
                                          None) == ERR_ARG   # grads NULL
    for f in (lambda Xs, N, nb: lib.dsmil_forward_bags_models_train(ps, 2, Xs, N, nb, *([FAKE] * 7), None, 0, None),
              lambda Xs, N, nb: lib.dsmil_backward_bags_models(ps, 2, Xs, N, nb, *([FAKE] * 9), grads(2), None, 0,
                                                               None)):
        assert f(None, i64(Ns), i32(nbs)) == ERR_ARG
        assert f(ptrs(2), None, i32(nbs)) == ERR_ARG
        assert f(ptrs(2), i64(Ns), None) == ERR_ARG
    assert fwd(lib, ps, 2, Ns, nbs, Xs=ptrs(2, 0)) == ERR_ARG          # a NULL bag
    assert fwd(lib, ps, 2, [100, 0], nbs) != 0                           # an empty bag
    assert fwd_ws(lib, None, 2, Ns, nbs) == 0 and bwd_ws(lib, None, 2, Ns, nbs) == 0


@pytest.mark.parametrize("nbs", [[0, 1], [1, 0], [2, -1]])
def test_every_model_needs_a_bag(nbs):
    lib = _lib.load()
    ps = arr([params(), params()])
    Ns = [100] * max(1, sum(n for n in nbs if n > 0))
    assert fwd(lib, ps, 2, Ns, nbs) == ERR_ARG and "nb=" in last_error(lib)
    assert bwd(lib, ps, 2, Ns, nbs) == ERR_ARG and "nb=" in last_error(lib)
    assert fwd_ws(lib, ps, 2, Ns, nbs) == 0 and bwd_ws(lib, ps, 2, Ns, nbs) == 0


@pytest.mark.parametrize("field,other", [
    ("D", dict(D=1024)), ("C", dict(C_=1)), ("nonlinear", dict(nonlinear=0, W2=None, b2=None)),
    ("passing_v", dict(passing_v=1)),
])
def test_members_must_share_shape(field, other):
    lib = _lib.load()
    ps = arr([params(), params(), params(**other)])
    Ns, nbs = [100, 7, 3, 9], [2, 1, 1]
    for rc in (fwd(lib, ps, 3, Ns, nbs), bwd(lib, ps, 3, Ns, nbs)):
        assert rc == ERR_ARG
        msg = last_error(lib)
        assert "model 2" in msg and field in msg


def test_passing_v_is_refused_as_the_one_model_calls_refuse_it():
    lib = _lib.load()
    ps = arr([params(passing_v=1)] * 2)
    assert fwd(lib, ps, 2, [10, 10], [1, 1]) == ERR_ARG and "identity v" in last_error(lib)
    assert bwd(lib, ps, 2, [10, 10], [1, 1]) == ERR_ARG and "identity v" in last_error(lib)
    assert fwd_ws(lib, ps, 2, [10, 10], [1, 1]) == 0 and bwd_ws(lib, ps, 2, [10, 10], [1, 1]) == 0


def test_short_workspace():
    lib = _lib.load()
    Ns, nbs = [10_000, 129, 1, 5000, 7], [2, 1, 2]
    for ps in (arr([params()] * 3), arr([params(D=166, C_=1)] * 3)):       # fused and looped shapes
        need = fwd_ws(lib, ps, 3, Ns, nbs)
        assert need > 0
        assert fwd(lib, ps, 3, Ns, nbs) == ERR_WORKSPACE
        assert fwd(lib, ps, 3, Ns, nbs, ws=FAKE, ws_bytes=need - 1) == ERR_WORKSPACE
        assert "workspace too small" in last_error(lib)
        need = bwd_ws(lib, ps, 3, Ns, nbs)
        assert need > 0
        assert bwd(lib, ps, 3, Ns, nbs) == ERR_WORKSPACE
        assert bwd(lib, ps, 3, Ns, nbs, ws=FAKE, ws_bytes=need - 1) == ERR_WORKSPACE
        assert "workspace too small" in last_error(lib)


def _lists(M, base):
    """M models' bag lists: model m has the first len(base) - m % 3 bags of base (at least one)."""
    per = [base[:max(1, len(base) - m % 3)] for m in range(M)]
    return [n for p in per for n in p], [len(p) for p in per]


@pytest.mark.parametrize("D,C_", [(512, 1), (512, 2), (1024, 2), (1024, 4), (2048, 2), (166, 1)])
def test_workspace_monotone_and_covers_the_one_model_calls(D, C_):
    lib = _lib.load()
    base = [10_000, 1, 127, 128, 129]
    for M in range(1, 9):
        ps = arr([params(D, C_)] * M)
        Ns, nbs = _lists(M, base)
        f, b = fwd_ws(lib, ps, M, Ns, nbs), bwd_ws(lib, ps, M, Ns, nbs)
        one_f = one_b = 0
        lo = 0
        for m in range(M):
            sub = Ns[lo:lo + nbs[m]]
            one_f += lib.dsmil_forward_bags_train_workspace_bytes(C.byref(ps[m]), i64(sub), len(sub))
            one_b += lib.dsmil_backward_bags_workspace_bytes(C.byref(ps[m]), i64(sub), len(sub), 0)
            lo += nbs[m]
        assert f >= one_f > 0 and b >= one_b > 0
        if M > 1:
            Np, nbp = _lists(M - 1, base)
            pp = arr([params(D, C_)] * (M - 1))
            assert f >= fwd_ws(lib, pp, M - 1, Np, nbp) and b >= bwd_ws(lib, pp, M - 1, Np, nbp)
        # one more bag for the last model, and a longer last bag
        more = (Ns + [64], nbs[:-1] + [nbs[-1] + 1])
        assert fwd_ws(lib, ps, M, *more) >= f and bwd_ws(lib, ps, M, *more) >= b
        # (the backward's size is the sum of the one-model sizes, which follow how each model's rows are cut into
        #  gradient chunks: covered above, not monotone in the rows)
        rows = (Ns[:-1] + [Ns[-1] + 1000], nbs)
        assert fwd_ws(lib, ps, M, *rows) >= f


# ---- Python refusals (raised before any library call) ------------------------------------------------------------
def _net(D=32, C_=2, nonlinear=True, passing_v=False):
    import dsmil as mil
    return mil.MILNet(mil.FCLayer(D, C_), mil.BClassifier(D, C_, nonlinear=nonlinear, passing_v=passing_v))


@pytest.mark.parametrize("other,needle", [
    (dict(D=64), "D=64"), (dict(C_=1), "C=1"), (dict(nonlinear=False), "nonlinear=False"),
])
def test_per_model_forward_refuses_mismatched_members(other, needle):
    from dsmil_wsi_b200.ensemble import forward_bags_per_model
    with pytest.raises(ValueError, match=f"member 1: {needle}"):
        forward_bags_per_model([_net(), _net(**other)], [[torch.zeros(4, 32)], [torch.zeros(4, 32)]])


def test_per_model_forward_refuses_bad_lists_and_members():
    import torch.nn as nn
    from dsmil_wsi_b200.ensemble import forward_bags_per_model
    x = [torch.zeros(4, 32)]
    with pytest.raises(ValueError, match="member 1 is on meta"):
        forward_bags_per_model([_net(), _net().to("meta")], [x, x])
    with pytest.raises(ValueError, match="member 1: .*identity v"):
        forward_bags_per_model([_net(), _net(passing_v=True)], [x, x])
    with pytest.raises(TypeError, match="member 0"):
        forward_bags_per_model([nn.Linear(3, 3)], [x])
    with pytest.raises(ValueError, match="1 to 8"):
        forward_bags_per_model([_net()] * 9, [x] * 9)
    with pytest.raises(ValueError, match="2 bag lists for 3 members"):
        forward_bags_per_model([_net()] * 3, [x, x])
    with pytest.raises(ValueError, match="member 1 has no bags"):
        forward_bags_per_model([_net()] * 2, [x, []])


def test_train_epoch_models_refuses_bad_folds():
    store = feed.DeviceBagStore(32, device="cpu")
    for n in (5, 6, 7):
        store.add_bag(torch.zeros(n, 32), torch.zeros(2))
    nets = [_net(), _net()]
    opts = [torch.optim.SGD(n.parameters(), lr=0.1) for n in nets]
    crit = torch.nn.BCEWithLogitsLoss()
    with pytest.raises(ValueError, match="1 optimizers for 2 folds"):
        feed.train_epoch_models(nets, store, [[0], [1]], crit, opts[:1])
    with pytest.raises(ValueError, match="3 milnets for 2 folds"):
        feed.train_epoch_models(nets + [_net()], store, [[0], [1]], crit, opts)
    with pytest.raises(ValueError, match="fold 1 has no training bags"):
        feed.train_epoch_models(nets, store, [[0], []], crit, opts)
    with pytest.raises(IndexError, match="fold 0: store index 3"):
        feed.train_epoch_models(nets, store, [[3], [1]], crit, opts)
    with pytest.raises(ValueError, match=r"orders\[1\] is not a permutation"):
        feed.train_epoch_models(nets, store, [[0], [1, 2]], crit, opts, orders=[[0], [1, 1]])
    with pytest.raises(ValueError, match="1 to 8 folds"):
        feed.train_epoch_models([_net()] * 9, store, [[0]] * 9, crit, [opts[0]] * 9)


# ---- the step schedule over folds of unequal length --------------------------------------------------------------
def _mirror(sizes, k):
    """Each fold alone, as train_epoch groups it: consecutive groups of k, the last one short."""
    per = [[(s, min(s + k, n)) for s in range(0, n, k)] for n in sizes]
    steps = []
    for t in range(max(len(p) for p in per)):
        steps.append([(m, *p[t]) for m, p in enumerate(per) if t < len(p)])
    return steps


@pytest.mark.parametrize("sizes", [[5], [3, 3, 3], [7, 1, 4, 9, 2], [1, 16, 15, 17, 8, 4, 2, 1]])
@pytest.mark.parametrize("k", [1, 2, 4, 16])
def test_fold_steps_follow_each_fold_alone(sizes, k):
    steps = feed.fold_steps(sizes, k)
    assert steps == _mirror(sizes, k)
    # every bag of every fold exactly once, in order; a fold leaves the steps once its bags run out
    for m, n in enumerate(sizes):
        got = [i for st in steps for (mm, lo, hi) in st if mm == m for i in range(lo, hi)]
        assert got == list(range(n))
        present = [any(mm == m for mm, _, _ in st) for st in steps]
        assert present == sorted(present, reverse=True)
    assert len(steps) == -(-max(sizes) // k)
