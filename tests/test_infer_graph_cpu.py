"""The capture-safe inference entry point and the inference graph, without a GPU: the symbols, argument validation and
workspace sizes of dsmil_forward_bags_dev (calls that return before any CUDA work), and the refusals of
ForwardBagsGraph and feed.eval_epoch(graph=True) that come before any device work."""
import ctypes as C
import os
import re

import pytest
import torch

import dsmil as mil
from dsmil_wsi_b200 import _lib, feed
from dsmil_wsi_b200.infer_graph import EvalBagsGraph, ForwardBagsGraph

ERR_ARG, ERR_WORKSPACE = -1, -2
FAKE = 0x10000          # a non-NULL, 16-byte aligned "device pointer": never dereferenced on these paths
HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "dsmil_b200.h")


def params(D=512, C_=2, nonlinear=1, passing_v=0):
    p = _lib.DsmilParams(D, C_, nonlinear, passing_v)
    for name in ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf"):
        setattr(p, name, FAKE)
    return p


def last_error(lib):
    return (lib.dsmil_last_error() or b"").decode()


def fwd(lib, p, nb=4, max_rows=1000, ws=FAKE, wsb=1 << 40, null=None):
    # Xs, Ns, then classes, pred, A, B, crit, status
    b = [None if i == null else FAKE for i in range(8)]
    return lib.dsmil_forward_bags_dev(None if p is None else C.byref(p), b[0], b[1], nb, max_rows, *b[2:], ws, wsb,
                                      None)


def test_symbols_exported_and_declared():
    lib = _lib.load()
    header = open(HEADER).read()
    for name in ("dsmil_forward_bags_dev_workspace_bytes", "dsmil_forward_bags_dev"):
        assert getattr(lib, name) is not None
        assert name in _lib.SIGNATURES
        assert re.search(rf"\b{name}\(", header), name


def test_dev_inference_validation():
    lib = _lib.load()
    assert fwd(lib, None) == ERR_ARG
    assert fwd(lib, params(nonlinear=0)) == ERR_ARG                     # linear q
    assert fwd(lib, params(passing_v=1)) == ERR_ARG
    assert fwd(lib, params(C_=8)) == ERR_ARG and "C=8" in last_error(lib)
    assert fwd(lib, params(D=230, C_=1)) == ERR_ARG and "D=230" in last_error(lib)
    for nb in (0, -1, 65536):
        assert fwd(lib, params(), nb=nb) == ERR_ARG and "nb" in last_error(lib)
    for mr in (0, -5):
        assert fwd(lib, params(), max_rows=mr) == ERR_ARG and "max_rows" in last_error(lib)
    assert fwd(lib, params(), nb=65535, max_rows=1 << 31) == ERR_ARG      # tiles past an int
    # the bag list, the four outputs and the status word; crit_idx may be NULL, as in dsmil_forward_bags
    for null in (0, 1, 2, 3, 4, 5, 7):
        assert fwd(lib, params(), null=null) == ERR_ARG, null
    need = lib.dsmil_forward_bags_dev_workspace_bytes(C.byref(params()), 4, 1000)
    assert need > 0
    assert fwd(lib, params(), wsb=need - 1) == ERR_WORKSPACE
    assert fwd(lib, params(), ws=None) == ERR_WORKSPACE
    assert fwd(lib, params(), wsb=need - 1, null=6) == ERR_WORKSPACE      # NULL crit_idx passes validation


@pytest.mark.parametrize("D,C_", [(512, 1), (512, 2), (1024, 4), (2048, 2)])
def test_dev_inference_workspace_sizes(D, C_):
    lib = _lib.load()
    p = C.byref(params(D, C_))
    f = lambda nb, mr: lib.dsmil_forward_bags_dev_workspace_bytes(p, nb, mr)
    assert f(1, 1) > 0
    assert f(0, 10) == 0 and f(4, 0) == 0 and f(65536, 10) == 0
    for nb in (1, 2, 4, 16, 17, 100):
        assert f(nb, 1000) <= f(nb + 1, 1000)
        assert f(nb, 1000) <= f(nb, 1001) <= f(nb, 5000)
    for mr in (1, 127, 128, 129, 10000):
        assert f(4, mr) <= f(4, mr + 1)
    # never below the eager call's size for nb bags of max_rows rows
    for nb, mr in [(1, 1), (1, 15000), (4, 129), (16, 10000), (3, 12000)]:
        Ns = (C.c_int64 * nb)(*[mr] * nb)
        assert f(nb, mr) >= lib.dsmil_forward_bags_workspace_bytes(p, Ns, nb)


@pytest.mark.parametrize("D,C_,nonlinear", [(230, 1, True), (512, 2, False), (512, 8, True)])
def test_dev_inference_workspace_zero_off_the_batched_path(D, C_, nonlinear):
    lib = _lib.load()
    assert lib.dsmil_forward_bags_dev_workspace_bytes(C.byref(params(D, C_, int(nonlinear))), 4, 100) == 0
    assert lib.dsmil_forward_bags_dev_workspace_bytes(C.byref(params(passing_v=1)), 4, 100) == 0


def _net(D=512, C_=2, nonlinear=True, passing_v=False):
    return mil.MILNet(mil.FCLayer(D, C_), mil.BClassifier(D, C_, nonlinear=nonlinear, passing_v=passing_v))


def _store(D, Ns, C_=2):
    store = feed.DeviceBagStore(D, device="cpu")
    for n in Ns:
        store.add_bag(torch.rand(n, D), torch.zeros(C_))
    return store


@pytest.mark.parametrize("D,C_,nonlinear,passing_v", [(230, 1, True, False), (512, 2, False, False),
                                                      (512, 8, True, False), (512, 2, True, True)])
def test_graphs_refuse_shapes_off_the_batched_path(D, C_, nonlinear, passing_v):
    net = _net(D, C_, nonlinear, passing_v)
    with pytest.raises(ValueError, match=f"D={D}, C={C_}"):
        ForwardBagsGraph(net, 4, 100)
    with pytest.raises(ValueError, match=f"D={D}, C={C_}"):
        EvalBagsGraph(net, torch.nn.BCEWithLogitsLoss(), 4, 100)
    with pytest.raises(ValueError, match=f"D={D}, C={C_}"):
        feed.eval_epoch(net, _store(D, [10, 20], C_), torch.nn.BCEWithLogitsLoss(), bags_per_launch=2, graph=True)


def test_graph_refuses_bad_sizes():
    for nb, mr in [(0, 10), (65536, 10), (4, 0)]:
        with pytest.raises(ValueError, match="nb=|max_rows="):
            ForwardBagsGraph(_net(), nb, mr)


def test_graph_eval_refuses_a_bag_over_capacity_before_any_launch():
    net = _net()
    store = _store(512, [100, 300, 50])
    with pytest.raises(ValueError, match="max_rows=200"):
        feed.eval_epoch(net, store, torch.nn.BCEWithLogitsLoss(), bags_per_launch=2, graph=True, max_rows=200)
    # with patch dropout the kept rows count: 300 * 0.6 = 180 fits 200, not 150
    with pytest.raises(ValueError, match="max_rows=150"):
        feed.eval_epoch(net, store, torch.nn.BCEWithLogitsLoss(), bags_per_launch=2, dropout_patch=0.4, graph=True,
                        max_rows=150)
