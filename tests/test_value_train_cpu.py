"""The batched backward of a model with a value network (passing_v: dsmil_value_backward_bags) before any device work:
the exported symbols, argument validation, workspace sizes and the Python refusals."""
import ctypes as C
import os
import re

import pytest
import torch

from dsmil_wsi_b200 import _lib
from dsmil_wsi_b200 import functional as Fn
from test_value_bags_cpu import FAKE, VALUE, last_error, ns, params, ptrs

ERR_ARG, ERR_WORKSPACE, ERR_EMPTY = -1, -2, -4
NAMES = ("dsmil_value_backward_bags_workspace_bytes", "dsmil_value_backward_bags")


def test_symbols_are_declared_exported_and_bound():
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "dsmil_b200.h")).read()
    lib = _lib.load()
    for name in NAMES:
        assert re.search(rf"\b{name}\(", header), name
        assert name in _lib.SIGNATURES
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]


def _grads(gX=None):
    return _lib.DsmilGrads(*[FAKE] * 10, gX)


def _call(lib, p, nb=3, Xs=True, XVs=False, Ns=None, saves=None, masks=False, dc=None, gX=None, ws=FAKE, wsb=1,
          grads=True):
    Ns = Ns if Ns is not None else ns(*[100] * max(nb, 1))
    Q, H1, V = saves if saves is not None else (FAKE, FAKE, FAKE)
    return lib.dsmil_value_backward_bags(C.byref(p), ptrs(max(nb, 1)) if Xs else None,
                                         ptrs(max(nb, 1)) if XVs else None, Ns, nb, Q, H1, V, FAKE, FAKE, FAKE, dc,
                                         FAKE, None, None, FAKE if masks else None,
                                         C.byref(_grads(gX)) if grads else None, ws, wsb, None)


def test_backward_validates_its_arguments():
    lib = _lib.load()
    p = params()
    # a short or missing workspace is the first thing a well-formed call meets
    assert _call(lib, p) == ERR_WORKSPACE
    assert _call(lib, p, ws=None, wsb=1 << 40) == ERR_WORKSPACE
    assert _call(lib, p, XVs=True, masks=True, gX=FAKE, dc=FAKE) == ERR_WORKSPACE
    assert _call(lib, params(512, 3, 0), saves=(FAKE, None, FAKE)) == ERR_WORKSPACE   # a linear q has no H1
    assert _call(lib, params(passing_v=0)) == ERR_ARG and "passing_v" in last_error(lib)
    assert _call(lib, params(Wv=None)) == ERR_ARG and "Wv" in last_error(lib)
    assert _call(lib, params(D=4097)) == ERR_ARG
    for nb in (0, 65536):
        assert _call(lib, p, nb=nb, Ns=ns(*[10] * max(nb, 1))) == ERR_ARG and "nb" in last_error(lib)
    assert _call(lib, p, Xs=False) == ERR_ARG
    assert _call(lib, p, grads=False) == ERR_ARG
    for saves in ((None, FAKE, FAKE), (FAKE, FAKE, None)):
        assert _call(lib, p, saves=saves) == ERR_ARG
    assert _call(lib, p, saves=(FAKE, None, FAKE)) == ERR_ARG and "H1" in last_error(lib)
    assert _call(lib, params(Wi=None), gX=FAKE, dc=FAKE) == ERR_ARG and "Wi" in last_error(lib)
    assert _call(lib, p, Ns=ns(100, 0, 100)) == ERR_EMPTY
    assert _call(lib, p, Ns=ns(100, -1, 100)) == ERR_ARG
    G = _grads()
    assert lib.dsmil_value_backward_bags(C.byref(p), ptrs(2), (C.c_void_p * 2)(FAKE, None), ns(4, 4), 2, FAKE, FAKE,
                                         FAKE, FAKE, FAKE, FAKE, None, None, None, None, None, C.byref(G), FAKE, 1,
                                         None) == ERR_ARG
    assert "value input" in last_error(lib)
    assert lib.dsmil_value_backward_bags(None, ptrs(1), None, ns(4), 1, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, None,
                                         None, None, None, None, C.byref(G), FAKE, 1, None) == ERR_ARG


@pytest.mark.parametrize("D,C_,nl", VALUE)
def test_workspace_sizes(D, C_, nl):
    lib = _lib.load()
    p = C.byref(params(D, C_, nl))
    f = lambda *n, gX=0: lib.dsmil_value_backward_bags_workspace_bytes(p, ns(*n), len(n), gX)
    assert f(1) > 0
    assert f(100, 100) < f(100, 100, 100) and f(100, 100) < f(100, 5000)
    assert f(5000, 5000) > f(5000, 1)
    # gX adds the [sum N, D] buffer of dzv Wv
    assert f(1000, 7, gX=1) >= f(1000, 7) + 4 * 1007 * D
    # never below the identity-v backward of the same bags, whose phases it runs
    q = C.byref(params(D, C_, nl, passing_v=0))
    assert f(127, 128, 129) > lib.dsmil_backward_bags_workspace_bytes(q, ns(127, 128, 129), 3, 0)
    assert lib.dsmil_value_backward_bags_workspace_bytes(p, None, 1, 0) == 0
    assert lib.dsmil_value_backward_bags_workspace_bytes(p, ns(1), 0, 0) == 0
    assert lib.dsmil_value_backward_bags_workspace_bytes(p, ns(*[1] * 65536), 65536, 0) == 0
    assert f(10, 0) == 0 and f(-1) == 0
    # the gWv partials: one D x D block per chunk of the value inputs, and every bag is at least one chunk
    assert f(*[100] * 64) >= 64 * 4 * D * D
    assert lib.dsmil_value_backward_bags_workspace_bytes(q, ns(10), 1, 0) == 0


def test_a_batch_past_the_chunk_grids_is_refused_and_sized_zero():
    """65 534 one-row bags and one of 10^6 rows: every ragged GEMM chunk count is past the 65 535 a grid can number;
    the workspace size is 0 and the call refuses the batch before any device work."""
    lib = _lib.load()
    p = params()
    Ns = ns(*([1] * 65534 + [10 ** 6]))
    assert lib.dsmil_value_backward_bags_workspace_bytes(C.byref(p), Ns, 65535, 0) == 0
    assert _call(lib, p, nb=65535, Ns=Ns, wsb=1 << 40) == ERR_ARG and "chunks" in last_error(lib)
    # the same large bag among a hundred small ones fits
    assert lib.dsmil_value_backward_bags_workspace_bytes(C.byref(p), ns(*([1] * 100 + [10 ** 6])), 101, 0) > 0


def test_the_identity_v_backward_keeps_refusing_passing_v():
    lib = _lib.load()
    p = params()
    assert lib.dsmil_backward_bags_workspace_bytes(C.byref(p), ns(10, 10), 2, 0) == 0
    G = _grads()
    assert lib.dsmil_backward_bags(C.byref(p), ptrs(2), ns(10, 10), 2, FAKE, FAKE, FAKE, FAKE, FAKE, None, None, None,
                                   None, C.byref(G), FAKE, 1 << 30, None) == ERR_ARG


def _cpu_params(D=16, C_=2, passing_v=True):
    mk = lambda *s: torch.zeros(*s, requires_grad=True)
    return (mk(C_, D), mk(C_), mk(128, D), mk(128), mk(128, 128), mk(128),
            mk(D, D) if passing_v else None, mk(D) if passing_v else None, mk(C_, C_, D), mk(C_))


def test_python_refusals_before_any_device_work():
    bags = [torch.zeros(3, 16)]
    with pytest.raises(RuntimeError, match="CUDA"):          # CPU tensors: there is no CPU path
        Fn.mil_forward_value_bags(bags, _cpu_params(), grad=True)
    with pytest.raises(ValueError, match="65535"):
        Fn.mil_forward_value_bags(bags * 65536, _cpu_params(), grad=True)
    with torch.no_grad():                                    # grad=True outside grad mode is inference
        with pytest.raises(RuntimeError, match="CUDA"):
            Fn.mil_forward_value_bags(bags * 65536, _cpu_params(), grad=True)
