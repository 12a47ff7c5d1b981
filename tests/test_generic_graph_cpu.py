"""The generic batched route's dev calls and graphs before any device work: the widened shape predicate, ABI
validation, workspace sizes against the eager calls', and the Python shape checks (step_shape: the generic shapes are
accepted with generic=True, passing_v and the default keep their refusals)."""
import ctypes as C

import pytest
import torch

import dsmil as mil
from dsmil_wsi_b200 import _lib, feed
from dsmil_wsi_b200.train_graph import step_shape

FAKE = 256
ERR_ARG, ERR_WORKSPACE = -1, -2


def params(D=166, C_=1, nonlinear=1, passing_v=0):
    p = _lib.DsmilParams(D, C_, nonlinear, passing_v)
    for name in ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf"):
        setattr(p, name, FAKE)
    return p


GENERIC = [(166, 1, 1), (230, 1, 1), (512, 3, 0), (96, 2, 1), (1024, 6, 1), (4096, 2, 1), (7, 1, 0), (4096, 8, 0)]


def test_codes_match_the_header():
    lib = _lib.load()
    assert lib.dsmil_generic_bags_supported(None) == 0
    assert ERR_ARG == -1 and ERR_WORKSPACE == -2


@pytest.mark.parametrize("D,C_,nl", GENERIC)
def test_dev_supported_and_workspace_sizes(D, C_, nl):
    lib = _lib.load()
    p = C.byref(params(D, C_, nl))
    assert lib.dsmil_generic_bags_supported(p) == 1
    assert lib.dsmil_shard_bags_supported(p) == 0
    sizes = (lib.dsmil_generic_forward_bags_train_dev_workspace_bytes,
             lib.dsmil_generic_forward_bags_dev_workspace_bytes, lib.dsmil_generic_backward_bags_dev_workspace_bytes)
    for ws in (lib.dsmil_forward_bags_train_dev_workspace_bytes, lib.dsmil_forward_bags_dev_workspace_bytes,
               lib.dsmil_backward_bags_dev_workspace_bytes):
        assert ws(p, 4, 100) == 0                                       # the tensor-core calls keep their shapes
    for ws in sizes:
        f = lambda nb, mr: ws(p, nb, mr)
        assert f(1, 1) > 0
        assert f(4, 1000) < f(8, 1000) and f(4, 1000) < f(4, 5000)
        assert f(0, 10) == 0 and f(4, 0) == 0 and f(65536, 10) == 0
    for nb, mr in [(1, 1), (1, 9473), (5, 33), (16, 2000), (90, 40)]:
        Ns = (C.c_int64 * nb)(*[mr] * nb)
        assert sizes[0](p, nb, mr) >= lib.dsmil_forward_bags_train_workspace_bytes(p, Ns, nb)
        assert sizes[1](p, nb, mr) >= lib.dsmil_forward_bags_workspace_bytes(p, Ns, nb)
        assert sizes[2](p, nb, mr) >= lib.dsmil_backward_bags_workspace_bytes(p, Ns, nb, 0)


def test_passing_v_stays_off_the_dev_calls():
    lib = _lib.load()
    for D, C_ in [(166, 1), (512, 2)]:
        p = C.byref(params(D, C_, 1, 1))
        assert lib.dsmil_generic_bags_supported(p) == 0
        assert lib.dsmil_generic_forward_bags_dev_workspace_bytes(p, 4, 100) == 0
        assert lib.dsmil_generic_forward_bags_train_dev_workspace_bytes(p, 4, 100) == 0
        assert lib.dsmil_generic_backward_bags_dev_workspace_bytes(p, 4, 100) == 0


def _fwd(lib, p, nb=4, max_rows=100, ws=FAKE, wsb=1 << 40, null=None):
    b = [None if i == null else FAKE for i in range(10)]
    return lib.dsmil_generic_forward_bags_train_dev(C.byref(p), b[0], b[1], nb, max_rows, *b[2:], ws, wsb, None)


def _bwd(lib, p, nb=4, max_rows=100, ws=FAKE, wsb=1 << 40, null=None):
    b = [None if i == null else FAKE for i in range(10)]
    g = _lib.DsmilGrads(*([FAKE] * 10), None)
    return lib.dsmil_generic_backward_bags_dev(C.byref(p), b[0], b[1], nb, max_rows, *b[2:9], None, None, C.byref(g), b[9],
                                       ws, wsb, None)


def _inf(lib, p, nb=4, max_rows=100, ws=FAKE, wsb=1 << 40, null=None):
    b = [None if i == null else FAKE for i in range(8)]
    return lib.dsmil_generic_forward_bags_dev(C.byref(p), b[0], b[1], nb, max_rows, *b[2:], ws, wsb, None)


@pytest.mark.parametrize("call", [_fwd, _bwd, _inf])
def test_widened_dev_calls_validate_their_arguments(call):
    lib = _lib.load()
    for D, C_, nl in [(166, 1, 1), (512, 3, 0), (7, 1, 0)]:
        p = params(D, C_, nl)
        # a short or missing workspace is the first thing a well-formed call meets: the shape is accepted
        assert call(lib, p, ws=None) == ERR_WORKSPACE, (D, C_, nl)
        assert call(lib, p, wsb=1) == ERR_WORKSPACE
        assert call(lib, params(D, C_, nl, 1)) == ERR_ARG and "passing_v" in (lib.dsmil_last_error() or b"").decode()
        for nb in (0, 65536):
            assert call(lib, p, nb=nb) == ERR_ARG
        assert call(lib, p, max_rows=0) == ERR_ARG
        assert call(lib, p, nb=65535, max_rows=1 << 30) == ERR_ARG      # twice the capacity tiles past an int
        for null in (0, 1):
            assert call(lib, p, null=null) == ERR_ARG
    assert call(lib, params(512, 2, 1)) == ERR_ARG and "generic" in (lib.dsmil_last_error() or b"").decode()
    # a linear q needs no saved H1 (forward: argument 8; backward: argument 3)
    assert _fwd(lib, params(512, 3, 0), null=8, ws=None) == ERR_WORKSPACE
    assert _fwd(lib, params(166, 1, 1), null=8) == ERR_ARG
    assert _bwd(lib, params(512, 3, 0), null=3, ws=None) == ERR_WORKSPACE
    assert _bwd(lib, params(166, 1, 1), null=3) == ERR_ARG


def _net(D, C_, nonlinear=True, passing_v=False):
    return mil.MILNet(mil.FCLayer(D, C_), mil.BClassifier(D, C_, nonlinear=nonlinear, passing_v=passing_v))


@pytest.mark.parametrize("D,C_,nl", GENERIC)
def test_step_shape_takes_the_generic_shapes(D, C_, nl):
    net = _net(D, C_, bool(nl))
    assert step_shape(net, generic=True) == (D, C_)
    with pytest.raises(ValueError, match=f"tensor-core path only; D={D}, C={C_}"):
        step_shape(net)                          # the default (and the row-sharded and fold steps) keeps its shapes
    assert step_shape(_net(512, 2), generic=True) == (512, 2)


def test_passing_v_is_refused_by_every_graph():
    from dsmil_wsi_b200.infer_graph import ForwardBagsGraph
    net = _net(166, 1, passing_v=True)
    store = feed.DeviceBagStore(166, device="cpu")
    for n in (10, 20):
        store.add_bag(torch.rand(n, 166), torch.zeros(1))
    with pytest.raises(ValueError, match="D=166, C=1.*passing_v=True"):
        step_shape(net, generic=True)
    with pytest.raises(ValueError, match="D=166, C=1"):
        ForwardBagsGraph(net, 4, 100, generic=True)
    with pytest.raises(ValueError, match="D=166, C=1"):
        feed.mil_epoch_train(net, store, torch.nn.BCEWithLogitsLoss(), torch.optim.SGD(net.parameters(), lr=0.1),
                             order=[0, 1], graph=True)
    with pytest.raises(ValueError, match="D=166, C=1"):
        feed.mil_epoch_test(net, store, torch.nn.BCEWithLogitsLoss(), graph=True)
