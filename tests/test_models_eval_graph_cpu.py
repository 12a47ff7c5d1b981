"""The capture-safe inference of the fold models without a GPU: argument validation, routes, batch limits and
workspace sizes of dsmil_forward_bags_models_dev / dsmil_generic_forward_bags_models_dev (calls that return before any
CUDA work), and the refusals of feed.eval_epoch_folds, infer_graph.ForwardBagsModelsGraph and per-fold criteria in
feed.train_epoch_models that come before any device work."""
import ctypes as C
import os
import re

import pytest
import torch

import dsmil as mil
from dsmil_wsi_b200 import _lib, feed
from dsmil_wsi_b200.infer_graph import EvalBagsModelsGraph, ForwardBagsModelsGraph
from dsmil_wsi_b200.train_graph import FoldTrainStepGraph

ERR_ARG, ERR_WORKSPACE = -1, -2
FAKE = 0x10000          # a non-NULL, 16-byte aligned "device pointer": never dereferenced on these paths
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("dsmil_forward_bags_models_dev_workspace_bytes", "dsmil_forward_bags_models_dev",
         "dsmil_generic_forward_bags_models_dev_workspace_bytes", "dsmil_generic_forward_bags_models_dev")
TENSOR_CORE = [dict(D=512, C_=2), dict(D=1024, C_=4), dict(D=2048, C_=2)]
GENERIC = [dict(D=166, C_=1), dict(D=230, C_=1), dict(D=230, C_=2, nonlinear=0), dict(D=512, C_=5),
           dict(D=2049, C_=2), dict(D=512, C_=1, nonlinear=0)]


def params(D=512, C_=2, nonlinear=1, passing_v=0, **over):
    p = _lib.DsmilParams(D, C_, nonlinear, passing_v)
    for name in ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf"):
        setattr(p, name, FAKE)
    if not nonlinear:
        p.W2 = p.b2 = None
    for k, v in over.items():
        setattr(p, k, v)
    return p


def arr(ps):
    return (_lib.DsmilParams * len(ps))(*ps)


def i32(xs):
    return (C.c_int32 * len(xs))(*xs)


def last_error(lib):
    return (lib.dsmil_last_error() or b"").decode()


def call_of(gen):
    def call(lib, ps, M, nbs, max_rows=1000, ws=FAKE, wsb=1 << 40, null=None):
        # Xs, Ns, then classes, pred, A, B, crit, status
        b = [None if i == null else FAKE for i in range(8)]
        fn = lib.dsmil_generic_forward_bags_models_dev if gen else lib.dsmil_forward_bags_models_dev
        return fn(ps, M, b[0], b[1], None if nbs is None else i32(nbs), max_rows, *b[2:8], ws, wsb, None)
    return call


def ws_of(gen):
    def ws(lib, ps, M, nbs, max_rows=1000):
        fn = (lib.dsmil_generic_forward_bags_models_dev_workspace_bytes if gen
              else lib.dsmil_forward_bags_models_dev_workspace_bytes)
        return fn(ps, M, None if nbs is None else i32(nbs), max_rows)
    return ws


def test_symbols_exported_declared_and_bound():
    lib = _lib.load()
    header = open(os.path.join(ROOT, "include", "dsmil_b200.h")).read()
    for name in NAMES:
        assert re.search(rf"\b{name}\s*\(", header), name
        assert hasattr(lib, name), name
        assert name in _lib.SIGNATURES, name


@pytest.mark.parametrize("gen", [False, True])
def test_fold_inference_entry_point_validation(gen):
    lib = _lib.load()
    call, ws = call_of(gen), ws_of(gen)
    kw = dict(D=166, C_=1) if gen else dict(D=512, C_=2)
    two = arr([params(**kw), params(**kw)])
    assert call(lib, None, 2, [1, 1]) == ERR_ARG and "params is NULL" in last_error(lib)
    assert ws(lib, None, 2, [1, 1]) == 0
    nine = arr([params(**kw) for _ in range(9)])
    for M in (0, 9, -1):
        assert call(lib, nine, M, [1] * 9) == ERR_ARG and "M=" in last_error(lib)
        assert ws(lib, nine, M, [1] * 9) == 0
    # members of different D / C / q form are named
    for other in (dict(D=kw["D"] + 64), dict(C_=kw["C_"] + 1), dict(nonlinear=0)):
        ps = arr([params(**kw), params(**{**kw, **other})])
        assert call(lib, ps, 2, [1, 1]) == ERR_ARG and "model 1" in last_error(lib), other
        assert ws(lib, ps, 2, [1, 1]) == 0
    # group sizes, each and in all
    for nbs in ([0, 1], [1, 0], [2, -1], [40000, 25536], [65536, 1]):
        assert call(lib, two, 2, nbs) == ERR_ARG, nbs
        assert ws(lib, two, 2, nbs) == 0
    assert call(lib, two, 2, None) == ERR_ARG
    assert ws(lib, two, 2, None) == 0
    for mr in (0, -5, 1 << 32):
        assert call(lib, two, 2, [2, 3], max_rows=mr) == ERR_ARG and "max_rows" in last_error(lib)
        assert ws(lib, two, 2, [2, 3], mr) == 0
    # capacity tiles past an int (twice over on the generic route)
    assert call(lib, two, 2, [30000, 30000], max_rows=1 << 30) == ERR_ARG
    assert ws(lib, two, 2, [30000, 30000], 1 << 30) == 0
    # the bag list, the status words and classes / pred / A / B are required; crit_idx (index 6) may be NULL
    for null in (0, 1, 2, 3, 4, 5, 7):
        assert call(lib, two, 2, [2, 3], null=null) == ERR_ARG, null
    need = ws(lib, two, 2, [2, 3])
    assert need > 0
    assert call(lib, two, 2, [2, 3], null=6, wsb=need - 1) == ERR_WORKSPACE   # passes every check
    assert call(lib, two, 2, [2, 3], wsb=need - 1) == ERR_WORKSPACE and "workspace too small" in last_error(lib)
    assert call(lib, two, 2, [2, 3], ws=None) == ERR_WORKSPACE


def test_routes():
    """Each call takes the shapes of its training twin and refuses the other's (and passing_v)."""
    lib = _lib.load()
    tc, gen = call_of(False), call_of(True)
    for kw in TENSOR_CORE + GENERIC + [dict(passing_v=1), dict(D=166, C_=1, passing_v=1)]:
        for M in (1, 2, 5, 8):
            ps = arr([params(**kw)] * M)
            fused = bool(lib.dsmil_models_supported(ps, M))
            generic = bool(lib.dsmil_generic_models_supported(ps, M))
            assert not (fused and generic)
            for call, ws, ok in ((tc, ws_of(False), fused), (gen, ws_of(True), generic)):
                got = call(lib, ps, M, [1] * M, wsb=1)
                assert got == (ERR_WORKSPACE if ok else ERR_ARG), (kw, M, got)
                assert (ws(lib, ps, M, [1] * M) > 0) == ok, (kw, M)
            if kw in TENSOR_CORE[:2] and M <= 2:
                assert fused
            if kw in GENERIC:
                assert generic
    wide = arr([params(D=2048, C_=2)] * 6)           # a tensor-core shape off the fused fold step: neither
    assert tc(lib, wide, 6, [1] * 6) == ERR_ARG and gen(lib, wide, 6, [1] * 6) == ERR_ARG
    pv = arr([params(D=166, C_=1, passing_v=1)] * 2)
    assert gen(lib, pv, 2, [1, 1]) == ERR_ARG and "identity v" in last_error(lib)


@pytest.mark.parametrize("gen", [False, True])
def test_chunk_capacity_bounds(gen):
    """The same bounds as the training twins: where a training fold call refuses the group sizes, so does this one."""
    lib = _lib.load()
    kw = dict(D=166, C_=1) if gen else dict(D=512, C_=2)
    for M in (1, 5):
        ps = arr([params(**kw)] * M)
        train_ws = (lib.dsmil_generic_forward_bags_models_train_dev_workspace_bytes if gen
                    else lib.dsmil_forward_bags_models_train_dev_workspace_bytes)
        lo, hi = 1, 65535
        while lo < hi:                               # the most bags in all that the training call takes
            mid = (lo + hi + 1) // 2
            nbs = [mid // M + (m < mid % M) for m in range(M)]
            lo, hi = (mid, hi) if train_ws(ps, M, i32(nbs), 2) > 0 else (lo, mid - 1)
        for ne, ok in ((lo, True), (lo + 1, False)):
            nbs = [ne // M + (m < ne % M) for m in range(M)]
            need = ws_of(gen)(lib, ps, M, nbs, 2)
            assert (need > 0) == ok, (M, ne)
            if ok:
                assert call_of(gen)(lib, ps, M, nbs, 2, wsb=need - 1) == ERR_WORKSPACE
            else:
                assert call_of(gen)(lib, ps, M, nbs, 2) == ERR_ARG


@pytest.mark.parametrize("kw", TENSOR_CORE[:2] + GENERIC)
def test_workspace_sizes(kw):
    """Never below the eager fold call's size at capacity, nor the one-model dev calls' sizes together; growing with
    M, the group sizes and max_rows."""
    lib = _lib.load()
    gen = kw in GENERIC
    ws = ws_of(gen)
    one = lib.dsmil_generic_forward_bags_dev_workspace_bytes if gen else lib.dsmil_forward_bags_dev_workspace_bytes
    prev = 0
    for M in (1, 2, 5, 8):
        ps = arr([params(**kw)] * M)
        if not (lib.dsmil_generic_models_supported(ps, M) if gen else lib.dsmil_models_supported(ps, M)):
            continue
        nbs = [4 + m % 3 for m in range(M)]
        got = ws(lib, ps, M, nbs, 500)
        assert got > prev
        prev = got
        assert ws(lib, ps, M, [n + 4 for n in nbs], 500) > got
        assert ws(lib, ps, M, nbs, 900) > got
        for mr in (1, 127, 129, 500, 10000):
            got = ws(lib, ps, M, nbs, mr)
            assert got >= sum(one(C.byref(ps[m]), nbs[m], mr) for m in range(M)), (M, mr)
            Ns = (C.c_int64 * sum(nbs))(*[mr] * sum(nbs))
            assert got >= lib.dsmil_forward_bags_models_train_workspace_bytes(ps, M, Ns, i32(nbs)), (M, mr)


# ---- Python refusals (raised before any device work) ---------------------------------------------------------------
def _net(D=512, C_=2, nonlinear=True):
    return mil.MILNet(mil.FCLayer(D, C_), mil.BClassifier(D, C_, nonlinear=nonlinear))


def _store(D, Ns, C_=2):
    store = feed.DeviceBagStore(D, device="cpu")
    for n in Ns:
        store.add_bag(torch.rand(n, D), torch.zeros(C_))
    return store


def test_eval_epoch_folds_refusals():
    nets = [_net(), _net()]
    store = _store(512, [10, 40, 5, 7])
    crit = torch.nn.BCEWithLogitsLoss()
    for graph in (False, True):
        with pytest.raises(IndexError, match="fold 1: store index 4"):
            feed.eval_epoch_folds(nets, store, [[0], [1, 4]], crit, graph=graph)
        with pytest.raises(IndexError, match="fold 0: store index -1"):
            feed.eval_epoch_folds(nets, store, [[-1], [1]], crit, graph=graph)
        with pytest.raises(ValueError, match="fold 1 has no held-out bags"):
            feed.eval_epoch_folds(nets, store, [[0], []], crit, graph=graph)
        with pytest.raises(ValueError, match="3 criteria for 2 folds"):
            feed.eval_epoch_folds(nets, store, [[0], [1]], [crit] * 3, graph=graph)
        with pytest.raises(ValueError, match="1 milnets for 2 folds"):
            feed.eval_epoch_folds(nets[:1], store, [[0], [1]], crit, graph=graph)
        with pytest.raises(ValueError, match="1 to 8 folds"):
            feed.eval_epoch_folds([nets[0]] * 9, store, [[0]] * 9, crit, graph=graph)
    with pytest.raises(ValueError, match="fold 1, bag 1: 40 rows exceed .*max_rows=30"):
        feed.eval_epoch_folds(nets, store, [[0, 2], [3, 1]], crit, graph=True, max_rows=30)
    with pytest.raises(ValueError, match="bag 1: 40 rows exceed .*max_rows=30"):
        feed.eval_epoch_models(nets, store, crit, graph=True, max_rows=30)
    gnets = [_net(166, 1), _net(166, 1)]
    gstore = _store(166, [3, 4], C_=1)
    with pytest.raises(ValueError, match="D=166, C=1"):       # without generic=True the shape is refused
        feed.eval_epoch_folds(gnets, gstore, [[0], [1]], crit, graph=True)


def test_forward_bags_models_graph_refusals():
    nets = [_net(), _net()]
    crit = torch.nn.BCEWithLogitsLoss()
    with pytest.raises(ValueError, match="2 models and 3 group sizes"):
        ForwardBagsModelsGraph(nets, [1, 1, 1], 40)
    with pytest.raises(ValueError, match="group sizes"):
        ForwardBagsModelsGraph(nets, [1, 0], 40)
    with pytest.raises(ValueError, match="max_rows=0"):
        ForwardBagsModelsGraph(nets, [1, 1], 0)
    with pytest.raises(ValueError, match="1 to 8 folds"):
        ForwardBagsModelsGraph([nets[0]] * 9, [1] * 9, 40)
    with pytest.raises(ValueError, match="fold 1"):
        ForwardBagsModelsGraph([nets[0], _net(1024)], [1, 1], 40)
    with pytest.raises(ValueError, match="D=166"):
        ForwardBagsModelsGraph([_net(166, 1)] * 2, [1, 1], 40)
    with pytest.raises(ValueError, match="3 criteria for 2 models"):
        EvalBagsModelsGraph(nets, [crit] * 3, [1, 1], 40)


def _sgd(net):
    return torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9)


def test_per_fold_criteria_are_counted_before_any_step():
    nets = [_net(166, 1), _net(166, 1)]
    opts = [_sgd(n) for n in nets]
    store = _store(166, [10, 40, 5], C_=1)
    crit = torch.nn.BCEWithLogitsLoss()
    for graph in (False, True):
        with pytest.raises(ValueError, match="3 criteria for 2 folds"):
            feed.train_epoch_models(nets, store, [[0, 2], [1]], [crit] * 3, opts, graph=graph, generic=True)
    with pytest.raises(ValueError, match="1 criteria for 2 folds"):
        FoldTrainStepGraph(nets, [crit], opts, [1, 1], 40, generic=True)
    assert feed.fold_criteria(crit, 3) == [crit] * 3
    two = [torch.nn.BCEWithLogitsLoss(), torch.nn.BCEWithLogitsLoss()]
    assert feed.fold_criteria(two, 2) == two and feed.fold_criteria(tuple(two), 2) == two
