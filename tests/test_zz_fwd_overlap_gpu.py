"""forward_bags with its attend pass overlapped with phase 1 (k_attend_b launched as a programmatic dependent of
k_qmlp_sm90, each attend CTA waiting for its own bag's phase-1 tiles) against the plain launch one after the other.
Kernel timing (dsmil_profile_enable) records an event between the two launches, so with it on the library takes the
plain launch: both routes must give the same bits.

Covered: tile totals at the overlapped phase-1 grid - 1, the grid and the grid + 1; a one-row bag; 101 small bags
(the bag table stays in global memory); one N = 100 000 bag (782 tiles, so an attend record spans several tiles);
C = 1, 2, 4 at D = 512, 1024, 2048; the bench workload; the training form; and ten back-to-back calls on one
workspace, where a per-bag tile count left over from the previous call would let attend start early."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

from helpers import build_net
from oracle import dsmil_oracle as orc
from test_phase1_schedule_gpu import _sizes_for_tiles
from dsmil_wsi_b200 import _lib

pytestmark = pytest.mark.gpu

TILE = 128


def _phase1_grid():
    return int(_lib.load().dsmil_forward_bags_phase1_ctas(1 << 30))


@contextlib.contextmanager
def _plain_launch():
    lib = _lib.load()
    torch.cuda.synchronize()
    lib.dsmil_profile_enable(1)
    try:
        yield
    finally:
        torch.cuda.synchronize()
        ms, n = (ctypes.c_double * 8)(), (ctypes.c_uint64 * 8)()
        lib.dsmil_profile_read(ms, n)
        lib.dsmil_profile_enable(0)


def _sizes(case):
    g = _phase1_grid()
    if case == "one_row":
        return [1]
    if case == "grid_minus_1":
        return _sizes_for_tiles(g - 1, 5, 11)
    if case == "grid":
        return _sizes_for_tiles(g, 7, 12)
    if case == "grid_plus_1":
        return _sizes_for_tiles(g + 1, 3, 13)
    if case == "many_bags":
        rng = np.random.default_rng(14)
        return [int(n) for n in rng.integers(1, 3 * TILE, 101)]
    if case == "n100k":
        return [100_000]
    if case == "bench":
        return [10_000] * 16
    raise ValueError(case)


def _bags(sizes, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.rand(n, D, generator=g, device="cuda") for n in sizes]


def _assert_same(outs, ref, what):
    assert len(outs) == len(ref), what
    for i, (o, r) in enumerate(zip(outs, ref)):
        for u, v in zip(o, r):
            u, v = u.detach(), v.detach()
            assert u.shape == v.shape and torch.equal(u, v), (what, i)


def _net(D, C, seed):
    return build_net(orc.random_params(D, C, seed, scale=2.0)).eval()


def _plain_and_overlapped(net, xs, grad=False):
    with _plain_launch():
        ref = [tuple(t.clone() for t in o) for o in net.forward_bags(xs, grad=grad)]
    return ref, net.forward_bags(xs, grad=grad)


def test_phase1_grid_query():
    lib = _lib.load()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    g = _phase1_grid()
    assert 1 <= g < sms
    assert lib.dsmil_forward_bags_phase1_ctas(0) == 0
    assert lib.dsmil_forward_bags_phase1_ctas(1) == 1
    assert lib.dsmil_forward_bags_phase1_ctas(g - 1) == g - 1
    assert lib.dsmil_forward_bags_phase1_ctas(g + 1) == g


@pytest.mark.parametrize("case", ["one_row", "grid_minus_1", "grid", "grid_plus_1", "many_bags", "n100k", "bench"])
def test_overlap_equals_plain_launch(case):
    sizes = _sizes(case)
    if case in ("grid_minus_1", "grid", "grid_plus_1"):
        assert sum(-(-n // TILE) for n in sizes) - _phase1_grid() == {"grid_minus_1": -1, "grid": 0, "grid_plus_1": 1}[case]
    net = _net(512, 2, 4100)
    xs = _bags(sizes, 512, 4200)
    with torch.no_grad():
        ref, outs = _plain_and_overlapped(net, xs)
    _assert_same(outs, ref, case)


@pytest.mark.parametrize("D", [512, 1024, 2048])
@pytest.mark.parametrize("C", [1, 2, 4])
def test_overlap_equals_plain_launch_shapes(C, D):
    net = _net(D, C, 4300 + 8 * D + C)
    xs = _bags(_sizes_for_tiles(_phase1_grid() + 1, 4, 15), D, 4400)
    with torch.no_grad():
        ref, outs = _plain_and_overlapped(net, xs)
    _assert_same(outs, ref, (C, D))


def test_overlap_equals_plain_launch_train():
    """dsmil_forward_bags_train: the outputs and, through the Q and H1 it saves, the batched backward's gradients."""
    net = _net(512, 2, 4500).train()
    xs = _bags(_sizes_for_tiles(_phase1_grid() + 1, 6, 16), 512, 4600)

    def step():
        net.zero_grad(set_to_none=True)
        outs = net.forward_bags(xs, grad=True)
        sum(o[1].sum() + o[0].square().sum() for o in outs).backward()
        grads = {k: v.grad.clone() for k, v in net.named_parameters() if v.grad is not None}
        return [tuple(t.detach().clone() for t in o) for o in outs], grads

    with _plain_launch():
        ref, ref_g = step()
    outs, g = step()
    _assert_same(outs, ref, "forward_bags(grad=True)")
    assert ref_g.keys() == g.keys() and len(g) > 0
    for k in g:
        assert torch.equal(g[k], ref_g[k]), k


def test_overlap_back_to_back_calls():
    """Ten calls queued on one workspace without a host sync: each call's memset must reset the per-bag tile counts
    before its attend pass reads them."""
    from dsmil_wsi_b200.functional import ParamPack, _ptr, _stream
    from dsmil_wsi_b200.sharded import milnet_params
    lib = _lib.load()
    net = _net(512, 2, 4700)
    P = ParamPack(*milnet_params(net))
    xs = _bags(_sizes_for_tiles(3 * _phase1_grid() + 5, 12, 17), 512, 4800)
    nb, Ns = len(xs), [x.shape[0] for x in xs]
    c_N = (ctypes.c_int64 * nb)(*Ns)
    c_X = (ctypes.c_void_p * nb)(*[x.data_ptr() for x in xs])
    ws = torch.empty(lib.dsmil_forward_bags_workspace_bytes(P.ref, c_N, nb), dtype=torch.uint8, device="cuda")

    def call():
        out = (torch.empty(sum(Ns), 2, device="cuda"), torch.empty(nb, 2, device="cuda"),
               torch.empty(sum(Ns), 2, device="cuda"), torch.empty(nb, 2, 512, device="cuda"),
               torch.empty(nb, 2, dtype=torch.int64, device="cuda"))
        rc = lib.dsmil_forward_bags(P.ref, c_X, c_N, nb, *[_ptr(t) for t in out], _ptr(ws), ws.numel(), _stream())
        assert rc == 0, lib.dsmil_last_error()
        return out

    with _plain_launch():
        ref = call()
    runs = [call() for _ in range(10)]
    torch.cuda.synchronize()
    for k, out in enumerate(runs):
        for u, v in zip(out, ref):
            assert torch.equal(u, v), f"call {k}"
