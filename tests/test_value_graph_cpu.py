"""The capture-safe value calls (dsmil_value_forward_bags_dev / dsmil_value_backward_bags_dev) before any device work:
the exported symbols, argument validation, workspace sizes and the Python refusals of value=True."""
import ctypes as C
import os
import re

import pytest
import torch

from dsmil_wsi_b200 import _lib, feed
from dsmil_wsi_b200 import train_graph as TG
from dsmil_wsi_b200.modules import BClassifier, FCLayer, MILNet
from test_value_bags_cpu import FAKE, last_error, ns, params

ERR_ARG, ERR_WORKSPACE = -1, -2
NAMES = ("dsmil_value_forward_bags_dev_workspace_bytes", "dsmil_value_forward_bags_dev",
         "dsmil_value_backward_bags_dev_workspace_bytes", "dsmil_value_backward_bags_dev")
# (D, C, nonlinear q)
SHAPES = [(512, 2, 1), (2048, 2, 1), (166, 1, 1), (230, 3, 0), (96, 5, 1)]


def test_symbols_are_declared_exported_and_bound():
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "dsmil_b200.h")).read()
    lib = _lib.load()
    for name in NAMES:
        assert re.search(rf"\b{name}\(", header), name
        assert name in _lib.SIGNATURES
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]
    # the header states how the gWv partials grow
    assert "(rag_splits + nb) * D^2 floats" in header


def _fwd(lib, p, nb=3, max_rows=100, Xs=FAKE, XVs=None, Ns=FAKE, status=FAKE, out_null=None, saves=(None, None, None),
         ws=FAKE, wsb=1, crit=FAKE):
    outs = [None if i == out_null else FAKE for i in range(4)]
    return lib.dsmil_value_forward_bags_dev(None if p is None else C.byref(p), Xs, XVs, Ns, nb, max_rows, *outs, crit,
                                            *saves, status, ws, wsb, None)


def _bwd(lib, p, nb=3, max_rows=100, Xs=FAKE, Ns=FAKE, status=FAKE, saves=(FAKE, FAKE, FAKE), dA=None, dB=None,
         gX=None, grads=True, ws=FAKE, wsb=1):
    Q, H1, V = saves
    G = _lib.DsmilGrads(*[FAKE] * 10, gX)
    return lib.dsmil_value_backward_bags_dev(None if p is None else C.byref(p), Xs, None, Ns, nb, max_rows, Q, H1, V,
                                             FAKE, FAKE, FAKE, FAKE, FAKE, dA, dB, C.byref(G) if grads else None,
                                             status, ws, wsb, None)


def test_forward_validates_its_arguments():
    lib = _lib.load()
    p = params()
    # a short workspace is the first thing a well-formed call meets
    assert _fwd(lib, p) == ERR_WORKSPACE
    assert _fwd(lib, p, XVs=FAKE) == ERR_WORKSPACE
    assert _fwd(lib, p, saves=(FAKE, FAKE, FAKE)) == ERR_WORKSPACE
    assert _fwd(lib, params(230, 3, 0), saves=(FAKE, None, FAKE)) == ERR_WORKSPACE   # a linear q has no H1
    assert _fwd(lib, p, crit=None) == ERR_WORKSPACE                                  # inference: crit may be NULL
    assert _fwd(lib, None) == ERR_ARG
    assert _fwd(lib, params(passing_v=0)) == ERR_ARG and "passing_v" in last_error(lib)
    assert _fwd(lib, params(Wv=None)) == ERR_ARG and "Wv" in last_error(lib)
    assert _fwd(lib, params(bv=None)) == ERR_ARG
    for nb in (0, -1, 65536):
        assert _fwd(lib, p, nb=nb) == ERR_ARG and "nb" in last_error(lib)
    for mr in (0, -5):
        assert _fwd(lib, p, max_rows=mr) == ERR_ARG and "max_rows" in last_error(lib)
    assert _fwd(lib, p, nb=65535, max_rows=1 << 31) == ERR_ARG and "max_rows" in last_error(lib)
    for kw in ({"Xs": None}, {"Ns": None}, {"status": None}):
        assert _fwd(lib, p, **kw) == ERR_ARG
    for i in range(4):
        assert _fwd(lib, p, out_null=i) == ERR_ARG
    for saves in ((FAKE, None, None), (None, None, FAKE), (FAKE, None, FAKE), (None, FAKE, None)):
        assert _fwd(lib, p, saves=saves) == ERR_ARG and "save" in last_error(lib)
    assert _fwd(lib, p, saves=(FAKE, FAKE, FAKE), crit=None) == ERR_ARG


def test_backward_validates_its_arguments():
    lib = _lib.load()
    p = params()
    assert _bwd(lib, p) == ERR_WORKSPACE
    assert _bwd(lib, params(230, 3, 0), saves=(FAKE, None, FAKE)) == ERR_WORKSPACE
    assert _bwd(lib, None) == ERR_ARG
    assert _bwd(lib, params(passing_v=0)) == ERR_ARG and "passing_v" in last_error(lib)
    assert _bwd(lib, params(Wv=None)) == ERR_ARG
    for nb in (0, -1, 65536):
        assert _bwd(lib, p, nb=nb) == ERR_ARG
    for mr in (0, -5):
        assert _bwd(lib, p, max_rows=mr) == ERR_ARG
    assert _bwd(lib, p, nb=65535, max_rows=1 << 31) == ERR_ARG
    for kw in ({"Xs": None}, {"Ns": None}, {"status": None}, {"grads": False}):
        assert _bwd(lib, p, **kw) == ERR_ARG
    for saves in ((None, FAKE, FAKE), (FAKE, None, FAKE), (FAKE, FAKE, None)):
        assert _bwd(lib, p, saves=saves) == ERR_ARG
    for kw in ({"dA": FAKE}, {"dB": FAKE}, {"gX": FAKE}):
        assert _bwd(lib, p, **kw) == ERR_ARG and "gX" in last_error(lib)


# The largest nb whose ragged GEMMs' chunk capacities stay within 65535 (bag_plan.cuh: rag_splits + nb chunks).  The
# streaming gWi form's rag_splits, 296, is the largest, and the dev calls' bound always counts it; gWv's
# max(1, 296 / ceil(D/128)^2) is never larger.
CAP = 65535 - 296


@pytest.mark.parametrize("D,C_,nl", SHAPES)
def test_chunk_capacity_is_refused(D, C_, nl):
    lib = _lib.load()
    p = params(D, C_, nl)
    nb = CAP
    assert lib.dsmil_value_backward_bags_dev_workspace_bytes(C.byref(p), nb, 1) > 0
    assert lib.dsmil_value_backward_bags_dev_workspace_bytes(C.byref(p), nb + 1, 1) == 0
    assert _bwd(lib, p, nb=nb + 1, max_rows=1) == ERR_ARG and "chunk" in last_error(lib)
    assert _bwd(lib, p, nb=nb, max_rows=1) == ERR_WORKSPACE
    # the gWv chunks alone: rag_splits(D, D) + nb bounds the gWv partials of the workspace
    gwv = (max(1, 296 // (-(-D // 128)) ** 2) + nb) * D * D * 4
    assert lib.dsmil_value_backward_bags_dev_workspace_bytes(C.byref(p), nb, 1) >= gwv


@pytest.mark.parametrize("D,C_,nl", SHAPES)
def test_workspace_sizes(D, C_, nl):
    lib = _lib.load()
    p = C.byref(params(D, C_, nl))
    fwd = lambda nb, mr: lib.dsmil_value_forward_bags_dev_workspace_bytes(p, nb, mr)
    bwd = lambda nb, mr: lib.dsmil_value_backward_bags_dev_workspace_bytes(p, nb, mr)
    for f in (fwd, bwd):
        assert f(1, 1) > 0 and f(16, 10000) > 0
        assert f(2, 100) < f(3, 100) and f(2, 100) < f(2, 5000)     # monotone in nb and max_rows
        assert f(1, 128) <= f(1, 129) and f(7, 40) <= f(8, 40)
        for nb, mr in ((0, 10), (-1, 10), (65536, 10), (3, 0), (3, -5), (65535, 1 << 31)):
            assert f(nb, mr) == 0
    for q in (params(D, C_, nl, passing_v=0), params(D, C_, nl, Wv=None)):
        assert lib.dsmil_value_forward_bags_dev_workspace_bytes(C.byref(q), 4, 100) == 0
        assert lib.dsmil_value_backward_bags_dev_workspace_bytes(C.byref(q), 4, 100) == 0
    # never below the eager value calls' sizes for nb bags of max_rows rows
    for nb, mr in ((1, 1), (3, 127), (16, 129), (40, 1000)):
        eager_f = lib.dsmil_value_forward_bags_workspace_bytes(p, ns(*[mr] * nb), nb)
        eager_b = lib.dsmil_value_backward_bags_workspace_bytes(p, ns(*[mr] * nb), nb, 0)
        assert fwd(nb, mr) >= eager_f > 0 and bwd(nb, mr) >= eager_b > 0


def _net(D=166, C_=1, passing_v=True, dropout_v=0.2, nonlinear=True):
    return MILNet(FCLayer(D, C_), BClassifier(D, C_, dropout_v=dropout_v, nonlinear=nonlinear, passing_v=passing_v))


def test_step_shape_value():
    for D, C_, nl in SHAPES:
        assert TG.step_shape(_net(D, C_, nonlinear=bool(nl)), value=True) == (D, C_)
    with pytest.raises(ValueError, match="passing_v=False"):
        TG.step_shape(_net(passing_v=False), value=True)
    # without value=True the refusals stay as they were
    with pytest.raises(ValueError, match="identity v only"):
        TG.step_shape(_net(), generic=True)
    with pytest.raises(ValueError, match="tensor-core path only"):
        TG.step_shape(_net())


def _store(ns_, D=166):
    store = feed.DeviceBagStore(D, device="cpu")
    for i, n in enumerate(ns_):
        store.add_bag(torch.zeros(n, D), torch.tensor([float(i % 2)]))
    return store


def test_python_refusals_before_any_launch():
    crit = torch.nn.BCEWithLogitsLoss()
    ident = _net(passing_v=False)
    store = _store([4, 9, 3])
    opt = torch.optim.SGD(ident.parameters(), lr=0.1)
    for graph in (False, True):
        with pytest.raises(ValueError, match="passing_v"):
            feed.train_epoch(ident, store, crit, opt, graph=graph, value=True)
        with pytest.raises(ValueError, match="passing_v"):
            feed.eval_epoch(ident, store, crit, graph=graph, value=True)
        with pytest.raises(ValueError, match="passing_v"):
            feed.mil_epoch_train(ident, store, crit, opt, graph=graph, value=True)
        with pytest.raises(ValueError, match="passing_v"):
            feed.mil_epoch_test(ident, store, crit, graph=graph, value=True)
    net = _net()
    opt = torch.optim.SGD(net.parameters(), lr=0.1)
    with pytest.raises(ValueError, match="max_rows=8"):
        feed.train_epoch(net, store, crit, opt, graph=True, value=True, max_rows=8, order=[0, 1, 2])
    with pytest.raises(ValueError, match="max_rows=8"):
        feed.eval_epoch(net, store, crit, graph=True, value=True, max_rows=8)
