"""The capture-safe batched training entry points and the training graph, without a GPU: argument validation and
workspace sizes of dsmil_forward_bags_train_dev / dsmil_backward_bags_dev (calls that return before any CUDA work),
and the refusals of TrainStepGraph and feed.train_epoch(graph=True) that come before any device work."""
import ctypes as C

import pytest
import torch

import dsmil as mil
from dsmil_wsi_b200 import _lib, feed
from dsmil_wsi_b200.train_graph import TrainStepGraph, check_optimizer

ERR_ARG, ERR_WORKSPACE = -1, -2
FAKE = 0x10000          # a non-NULL, 16-byte aligned "device pointer": never dereferenced on these paths


def params(D=512, C_=2, nonlinear=1, passing_v=0):
    p = _lib.DsmilParams(D, C_, nonlinear, passing_v)
    for name in ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf"):
        setattr(p, name, FAKE)
    return p


def last_error(lib):
    return (lib.dsmil_last_error() or b"").decode()


def fwd(lib, p, nb=4, max_rows=1000, ws=FAKE, wsb=1 << 40, null=None):
    # Xs, Ns, then classes, pred, A, B, crit, save_Q, save_H1, status
    b = [None if i == null else FAKE for i in range(10)]
    return lib.dsmil_forward_bags_train_dev(None if p is None else C.byref(p), b[0], b[1], nb, max_rows, *b[2:], ws,
                                            wsb, None)


def bwd(lib, p, nb=4, max_rows=1000, ws=FAKE, wsb=1 << 40, null=None, dA=None, dB=None, gX=None):
    # Xs, Ns, Q, H1, A, B, crit, d_classes, d_pred, status
    b = [None if i == null else FAKE for i in range(10)]
    g = _lib.DsmilGrads(*([FAKE] * 10), gX)
    return lib.dsmil_backward_bags_dev(None if p is None else C.byref(p), b[0], b[1], nb, max_rows, *b[2:9], dA, dB,
                                       C.byref(g), b[9], ws, wsb, None)


@pytest.mark.parametrize("call", [fwd, bwd])
def test_dev_entry_point_validation(call):
    lib = _lib.load()
    assert call(lib, None) == ERR_ARG
    assert call(lib, params(D=166, C_=1)) == ERR_ARG and "D=166" in last_error(lib)
    assert call(lib, params(passing_v=1)) == ERR_ARG
    assert call(lib, params(nonlinear=0)) == ERR_ARG
    for nb in (0, -1, 65536):
        assert call(lib, params(), nb=nb) == ERR_ARG and "nb" in last_error(lib)
    for mr in (0, -5):
        assert call(lib, params(), max_rows=mr) == ERR_ARG and "max_rows" in last_error(lib)
    assert call(lib, params(), nb=65535, max_rows=1 << 31) == ERR_ARG      # tiles past an int
    # the bag list and the status word (last) are always required
    for null in (0, 1, 9):
        assert call(lib, params(), null=null) == ERR_ARG, null
    # every other buffer of the forward and the saved activations of the backward
    for null in range(2, 9 if call is fwd else 7):
        assert call(lib, params(), null=null) == ERR_ARG, null
    need = (lib.dsmil_forward_bags_train_dev_workspace_bytes if call is fwd else
            lib.dsmil_backward_bags_dev_workspace_bytes)(C.byref(params()), 4, 1000)
    assert need > 0
    assert call(lib, params(), wsb=need - 1) == ERR_WORKSPACE
    assert call(lib, params(), ws=None) == ERR_WORKSPACE


def test_dev_backward_refuses_upstream_A_B_and_features():
    lib = _lib.load()
    assert bwd(lib, params(), dA=FAKE) == ERR_ARG and "d_A" in last_error(lib)
    assert bwd(lib, params(), dB=FAKE) == ERR_ARG
    assert bwd(lib, params(), gX=FAKE) == ERR_ARG


@pytest.mark.parametrize("D,C_", [(512, 2), (1024, 4), (1536, 1)])
def test_dev_workspace_sizes(D, C_):
    lib = _lib.load()
    p = C.byref(params(D, C_))
    f = lambda nb, mr: lib.dsmil_forward_bags_train_dev_workspace_bytes(p, nb, mr)
    b = lambda nb, mr: lib.dsmil_backward_bags_dev_workspace_bytes(p, nb, mr)
    for ws in (f, b):
        assert ws(1, 1) > 0
        assert ws(4, 1000) < ws(8, 1000) and ws(4, 1000) < ws(4, 5000)
        assert ws(0, 10) == 0 and ws(4, 0) == 0
    assert lib.dsmil_forward_bags_train_dev_workspace_bytes(C.byref(params(166, 1)), 4, 100) == 0
    # never below the eager calls' sizes for nb bags of max_rows rows
    for nb, mr in [(1, 1), (1, 15000), (4, 129), (16, 10000), (3, 12000)]:
        Ns = (C.c_int64 * nb)(*[mr] * nb)
        assert f(nb, mr) >= lib.dsmil_forward_bags_train_workspace_bytes(p, Ns, nb)
        assert b(nb, mr) >= lib.dsmil_backward_bags_workspace_bytes(p, Ns, nb, 0)


def _net(D=512, C_=2, nonlinear=True):
    return mil.MILNet(mil.FCLayer(D, C_), mil.BClassifier(D, C_, nonlinear=nonlinear))


def test_train_step_graph_refuses_optimizers_it_cannot_replay():
    net = _net()
    for opt in (torch.optim.RMSprop(net.parameters()), torch.optim.Adam(net.parameters()),
                torch.optim.AdamW(net.parameters(), capturable=False),
                torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9, dampening=0.5)):
        with pytest.raises(ValueError):
            TrainStepGraph(net, torch.nn.BCEWithLogitsLoss(), opt, 4, 100)
    for opt in (torch.optim.SGD(net.parameters(), lr=0.1), torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9),
                torch.optim.Adam(net.parameters(), capturable=True), torch.optim.AdamW(net.parameters(), capturable=True)):
        check_optimizer(opt)


def _store(D, Ns, C_=2):
    store = feed.DeviceBagStore(D, device="cpu")
    for n in Ns:
        store.add_bag(torch.rand(n, D), torch.zeros(C_))
    return store


def test_graph_epoch_refuses_a_bag_over_capacity_before_any_step():
    net = _net()
    store = _store(512, [100, 300, 50])
    opt = torch.optim.SGD(net.parameters(), lr=0.1)
    with pytest.raises(ValueError, match="max_rows=200"):
        feed.train_epoch(net, store, torch.nn.BCEWithLogitsLoss(), opt, order=[0, 1, 2], bags_per_step=2, graph=True,
                         max_rows=200)
    # with patch dropout the kept rows count: 300 * 0.6 = 180 fits
    with pytest.raises(ValueError, match="max_rows=150"):
        feed.train_epoch(net, store, torch.nn.BCEWithLogitsLoss(), opt, dropout_patch=0.4, order=[0, 1, 2],
                         bags_per_step=2, graph=True, max_rows=150)


@pytest.mark.parametrize("D,C_,nonlinear", [(166, 1, True), (512, 2, False), (512, 8, True)])
def test_graph_epoch_refuses_shapes_off_the_batched_path(D, C_, nonlinear):
    net = _net(D, C_, nonlinear)
    store = _store(D, [10, 20], C_)
    with pytest.raises(ValueError, match=f"D={D}, C={C_}"):
        feed.train_epoch(net, store, torch.nn.BCEWithLogitsLoss(), torch.optim.SGD(net.parameters(), lr=0.1),
                         order=[0, 1], bags_per_step=2, graph=True)
