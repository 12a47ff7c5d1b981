"""C-ABI argument validation and size arithmetic (include/dsmil_b200.h) -- only calls that return before any
CUDA work, so they run without a GPU.  Error behaviour mirrors the reference where it has one: an empty bag is
an error (dsmil.py:53 raises IndexError), everything else is the status / dsmil_last_error() contract."""
import ctypes as C

import pytest

from dsmil_wsi_b200 import _lib

ERR_ARG, ERR_WORKSPACE, ERR_CUDA, ERR_EMPTY = -1, -2, -3, -4
FAKE = 0x10000          # a non-NULL, 16-byte aligned "device pointer": never dereferenced on these paths


def params(D=512, C_=2, nonlinear=1, passing_v=0, **over):
    p = _lib.DsmilParams(D, C_, nonlinear, passing_v)
    for name in ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf"):
        setattr(p, name, FAKE)
    for k, v in over.items():
        setattr(p, k, v)
    return p


def last_error(lib):
    return (lib.dsmil_last_error() or b"").decode()


def forward(lib, p, N, X=FAKE, classes=FAKE, ws=None, ws_bytes=0):
    return lib.dsmil_forward(C.byref(p) if p is not None else None, X, None, N, classes, FAKE, FAKE, FAKE, None,
                             None, None, None, ws, ws_bytes, None)


def test_version_and_header_constants():
    lib = _lib.load()
    assert lib.dsmil_abi_version() == 1
    hdr = open(_lib.LIB_PATH.replace("dsmil_wsi_b200/lib/libdsmil_b200.so", "include/dsmil_b200.h")).read()
    assert "#define DSMIL_ABI_VERSION 1" in hdr and "#define DSMIL_MAX_C 8" in hdr and "#define DSMIL_MAX_D 4096" in hdr
    for name, code in (("DSMIL_ERR_ARG", ERR_ARG), ("DSMIL_ERR_WORKSPACE", ERR_WORKSPACE), ("DSMIL_ERR_CUDA", ERR_CUDA),
                       ("DSMIL_ERR_EMPTY", ERR_EMPTY)):
        assert f"{name} = {code}" in hdr


@pytest.mark.parametrize("make,needle", [
    (lambda: None, "params is NULL"),
    (lambda: params(D=0), "feature size"),
    (lambda: params(D=4097), "feature size"),
    (lambda: params(C_=0), "output classes"),
    (lambda: params(C_=9), "output classes"),
    (lambda: params(W2=None), "W2"),
    (lambda: params(passing_v=1, Wv=None), "Wv"),
    (lambda: params(Wi=None), "instance-classifier"),
    (lambda: params(Wf=None), "NULL weight"),
])
def test_bad_params_are_rejected_with_a_message(make, needle):
    lib = _lib.load()
    assert forward(lib, make(), 100) == ERR_ARG
    assert needle in last_error(lib)


def test_empty_bag_is_an_error_like_the_reference():
    lib = _lib.load()
    assert forward(lib, params(), 0) == ERR_EMPTY
    assert "IndexError" in last_error(lib) and "dsmil.py:53" in last_error(lib)
    assert forward(lib, params(), -3) == ERR_ARG
    assert forward(lib, params(), 1 << 32) == ERR_ARG


def test_null_tensors_and_workspace_are_rejected():
    lib = _lib.load()
    assert forward(lib, params(), 10, X=None) == ERR_ARG and "NULL tensor" in last_error(lib)
    assert forward(lib, params(), 10, classes=None) == ERR_ARG and "classes is NULL" in last_error(lib)
    for p in (params(), params(D=166, C_=1), params(nonlinear=0, W2=None, b2=None)):   # fused and generic routes
        need = lib.dsmil_forward_workspace_bytes(C.byref(p), 10)
        assert forward(lib, p, 10, ws=None, ws_bytes=0) == ERR_WORKSPACE
        assert forward(lib, p, 10, ws=FAKE, ws_bytes=need // 2) == ERR_WORKSPACE
        assert "workspace too small" in last_error(lib)
    # the bag form needs the caller's scores
    p = params()
    rc = lib.dsmil_bag_forward(C.byref(p), FAKE, None, None, 10, FAKE, FAKE, FAKE, None, None, None, None, None, 0, None)
    assert rc == ERR_ARG and "classes_in is NULL" in last_error(lib)


def test_batched_entry_point_validation():
    lib = _lib.load()
    p = params()
    Xs = (C.c_void_p * 2)(FAKE, FAKE)
    Ns = (C.c_int64 * 2)(100, 200)
    call = lambda xs, ns, nb, ws=None, wsb=0: lib.dsmil_forward_bags(C.byref(p), xs, ns, nb, FAKE, FAKE, FAKE, FAKE,
                                                                     None, ws, wsb, None)
    assert call(Xs, Ns, 0) == ERR_ARG
    assert call(None, Ns, 2) == ERR_ARG
    assert call(Xs, Ns, 2) == ERR_WORKSPACE
    need = lib.dsmil_forward_bags_workspace_bytes(C.byref(p), Ns, 2)
    assert need > 0 and call(Xs, Ns, 2, FAKE, need - 1) == ERR_WORKSPACE
    Ns0 = (C.c_int64 * 2)(0, 100)                      # an empty bag inside a batch is the same error as alone
    assert call(Xs, Ns0, 2, FAKE, 1 << 30) == ERR_EMPTY and "IndexError" in last_error(lib)


def test_size_arithmetic():
    lib = _lib.load()
    for Cc in range(1, 9):
        assert lib.dsmil_cand_floats(Cc) % 4 == 0 and lib.dsmil_cand_floats(Cc) >= 131 * Cc
        for D in (1, 166, 230, 512, 1024, 2048):
            r = lib.dsmil_rec_floats(Cc, D)
            assert r % 4 == 0 and Cc * (2 + D) <= r < Cc * (2 + D) + 4
    for p in (params(), params(D=166, C_=1), params(D=1024, C_=4), params(passing_v=1)):
        sizes = [lib.dsmil_forward_workspace_bytes(C.byref(p), n) for n in (1, 128, 129, 10000, 100000)]
        assert sizes[0] > 0 and sizes == sorted(sizes)
        assert lib.dsmil_shard_workspace_bytes(C.byref(p), 10000) == sizes[3]
        b = [lib.dsmil_backward_workspace_bytes(C.byref(p), n, 0) for n in (1, 1000, 100000)]
        assert b[0] > 0 and b == sorted(b)
        assert lib.dsmil_backward_workspace_bytes(C.byref(p), 1000, 1) >= b[1]
    # Q and H1 dominate: at least 2 * N * 128 floats for the generic nonlinear route
    p = params(D=166, C_=1)
    assert lib.dsmil_forward_workspace_bytes(C.byref(p), 10000) >= 2 * 10000 * 128 * 4


def test_path_selector_is_pure_and_consistent():
    """dsmil_forward_path: which kernel family a shape takes (1 generic fp32 FFMA, 2 sm_90a wgmma)."""
    lib = _lib.load()
    assert lib.dsmil_forward_path(C.byref(params()), 10000) == 2
    assert lib.dsmil_forward_path(C.byref(params(D=1024, C_=1)), 10000) == 2
    assert lib.dsmil_forward_path(C.byref(params(D=166, C_=1)), 10000) == 1          # D % 128 != 0
    assert lib.dsmil_forward_path(C.byref(params(nonlinear=0)), 10000) == 1            # linear q
    assert lib.dsmil_forward_path(None, 10000) == 1
    assert lib.dsmil_shard_bags_supported(C.byref(params())) == 1
    assert lib.dsmil_shard_bags_supported(C.byref(params(D=230, C_=1))) == 0
