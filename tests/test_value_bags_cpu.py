"""The batched forward of a model with a value network (passing_v: dsmil_value_forward_bags) before any device work: the
shape predicate, argument validation, workspace sizes and the exported symbols."""
import ctypes as C
import re

import pytest

from dsmil_wsi_b200 import _lib

FAKE = 256
ERR_ARG, ERR_WORKSPACE, ERR_EMPTY = -1, -2, -4
NAMES = ("dsmil_value_bags_supported", "dsmil_value_forward_bags_workspace_bytes", "dsmil_value_forward_bags")


def params(D=512, C_=2, nonlinear=1, passing_v=1, **over):
    p = _lib.DsmilParams(D, C_, nonlinear, passing_v)
    for name in ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf"):
        setattr(p, name, FAKE)
    for k, v in over.items():
        setattr(p, k, v)
    return p


def last_error(lib):
    return (lib.dsmil_last_error() or b"").decode()


def ptrs(n, v=FAKE):
    return (C.c_void_p * n)(*[v] * n)


def ns(*n):
    return (C.c_int64 * len(n))(*n)


VALUE = [(512, 2, 1), (166, 1, 1), (512, 3, 0), (1024, 6, 1), (96, 2, 1), (4096, 8, 0), (7, 1, 1)]


@pytest.mark.parametrize("D,C_,nl", VALUE)
def test_supported_shapes(D, C_, nl):
    lib = _lib.load()
    assert lib.dsmil_value_bags_supported(C.byref(params(D, C_, nl))) == 1
    # identity v keeps its routes; the existing batched predicates keep refusing passing_v
    assert lib.dsmil_value_bags_supported(C.byref(params(D, C_, nl, passing_v=0))) == 0
    assert lib.dsmil_generic_bags_supported(C.byref(params(D, C_, nl))) == 0
    assert lib.dsmil_shard_bags_supported(C.byref(params(D, C_, nl))) == 0


def test_supported_refuses_what_dsmil_forward_refuses():
    lib = _lib.load()
    assert lib.dsmil_value_bags_supported(None) == 0
    for p in (params(Wv=None), params(bv=None), params(D=4097), params(D=0), params(C_=9), params(C_=0)):
        assert lib.dsmil_value_bags_supported(C.byref(p)) == 0


def _call(lib, p, nb=3, Xs=True, XVs=False, Ns=None, out_null=None, saves=(None, None, None), ws=FAKE, wsb=1,
          crit=FAKE):
    Ns = Ns if Ns is not None else ns(*[100] * nb)
    outs = [None if i == out_null else FAKE for i in range(4)]
    return lib.dsmil_value_forward_bags(C.byref(p), ptrs(max(nb, 1)) if Xs else None,
                                        ptrs(max(nb, 1)) if XVs else None, Ns, nb, *outs, crit, *saves, ws, wsb,
                                        None)


def test_forward_validates_its_arguments():
    lib = _lib.load()
    p = params()
    # a short or missing workspace is the first thing a well-formed call meets: the shape and the bags are accepted
    assert _call(lib, p) == ERR_WORKSPACE
    assert _call(lib, p, ws=None, wsb=1 << 40) == ERR_WORKSPACE
    assert _call(lib, p, XVs=True) == ERR_WORKSPACE
    assert _call(lib, p, crit=None) == ERR_WORKSPACE
    assert _call(lib, p, saves=(FAKE, FAKE, FAKE)) == ERR_WORKSPACE
    assert _call(lib, params(512, 3, 0), saves=(FAKE, None, FAKE)) == ERR_WORKSPACE   # a linear q has no H1
    assert _call(lib, params(passing_v=0)) == ERR_ARG and "passing_v" in last_error(lib)
    assert _call(lib, params(Wv=None)) == ERR_ARG and "Wv" in last_error(lib)
    assert _call(lib, params(D=4097)) == ERR_ARG
    for nb in (0, 65536):
        assert _call(lib, p, nb=nb, Ns=ns(*[10] * max(nb, 1))) == ERR_ARG and "nb" in last_error(lib)
    assert _call(lib, p, Xs=False) == ERR_ARG
    for i in range(4):
        assert _call(lib, p, out_null=i) == ERR_ARG
    for saves in ((FAKE, None, None), (None, None, FAKE), (FAKE, None, FAKE), (None, FAKE, None)):
        assert _call(lib, p, saves=saves) == ERR_ARG and "saves" in last_error(lib)
    assert _call(lib, p, Ns=ns(100, 0, 100)) == ERR_EMPTY
    assert _call(lib, p, Ns=ns(100, -1, 100)) == ERR_ARG
    assert lib.dsmil_value_forward_bags(C.byref(p), ptrs(2), (C.c_void_p * 2)(FAKE, None), ns(4, 4), 2, FAKE, FAKE,
                                        FAKE, FAKE, None, None, None, None, FAKE, 1, None) == ERR_ARG
    assert "value input" in last_error(lib)
    assert lib.dsmil_value_forward_bags(None, ptrs(1), None, ns(4), 1, FAKE, FAKE, FAKE, FAKE, None, None, None,
                                        None, FAKE, 1, None) == ERR_ARG


@pytest.mark.parametrize("D,C_,nl", VALUE)
def test_workspace_sizes(D, C_, nl):
    lib = _lib.load()
    p = C.byref(params(D, C_, nl))
    f = lambda *n: lib.dsmil_value_forward_bags_workspace_bytes(p, ns(*n), len(n))
    assert f(1) > 0
    assert f(100, 100) < f(100, 100, 100) and f(100, 100) < f(100, 5000)
    # V and the saves of the batch are packed: the size grows with the rows of every bag, not only the largest
    assert f(5000, 5000) > f(5000, 1)
    for n in [(1,), (10000,), (127, 128, 129), (2049, 1, 10000)]:
        # where phase 1 is k_qmlp_sm90 an unaligned batch loops the single-bag forward: never below its size
        if lib.dsmil_forward_path(p, max(n)) == 2:
            assert f(*n) >= lib.dsmil_forward_workspace_bytes(p, max(n))
    assert lib.dsmil_value_forward_bags_workspace_bytes(p, None, 1) == 0
    assert lib.dsmil_value_forward_bags_workspace_bytes(p, ns(1), 0) == 0
    assert lib.dsmil_value_forward_bags_workspace_bytes(p, ns(*[1] * 65536), 65536) == 0
    assert f(10, 0) == 0 and f(-1) == 0
    assert lib.dsmil_value_forward_bags_workspace_bytes(C.byref(params(D, C_, nl, passing_v=0)), ns(10), 1) == 0


@pytest.mark.parametrize("D,C_,nl,pv", [(166, 1, 1, 0), (512, 3, 0, 0), (512, 2, 1, 1), (166, 1, 1, 1), (512, 2, 1, 0),
                                        (128, 1, 1, 0)])
def test_forward_bags_workspace_covers_its_routes(D, C_, nl, pv):
    """dsmil_forward_bags past 65 535 bags loops the single-bag forward on every shape, and on passing_v up to 65 535
    bags it takes the value batch; the size covers either.  On the tensor-core shapes the loop is all the batch takes
    past 65 535 bags: the size is then the single-bag forward's for the largest bag, which itself covers that bag's
    tensor-core batch of one."""
    lib = _lib.load()
    p = C.byref(params(D, C_, nl, pv))
    Ns = [1 + i % 300 for i in range(65536)]
    Ns[7] = 10000
    assert lib.dsmil_forward_bags_workspace_bytes(p, ns(*Ns), 65536) >= lib.dsmil_forward_workspace_bytes(p, 10000)
    if lib.dsmil_shard_bags_supported(p):
        assert lib.dsmil_forward_bags_workspace_bytes(p, ns(*Ns), 65536) == lib.dsmil_forward_workspace_bytes(p, 10000)
        assert lib.dsmil_forward_bags_workspace_bytes(p, ns(*Ns[:65535]), 65535) > lib.dsmil_forward_workspace_bytes(p, 10000)
        assert (lib.dsmil_forward_workspace_bytes(p, 10000) >=
                lib.dsmil_forward_bags_workspace_bytes(p, ns(10000), 1) > lib.dsmil_forward_workspace_bytes(p, 9000))
    if pv:
        assert (lib.dsmil_forward_bags_workspace_bytes(p, ns(*Ns[:16]), 16) >=
                lib.dsmil_value_forward_bags_workspace_bytes(p, ns(*Ns[:16]), 16) > 0)


def test_symbols_are_declared_and_exported():
    import os
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "dsmil_b200.h")).read()
    lib = _lib.load()
    for name in NAMES:
        assert re.search(rf"\b{name}\(", header), name
        assert name in _lib.SIGNATURES
        assert getattr(lib, name) is not None
