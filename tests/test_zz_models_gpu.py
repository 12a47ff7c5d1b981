"""The ensemble forward (dsmil_forward_bags_models) against each member's own forward_bags: every model's classes,
pred, A and B must be torch.equal to milnet_m.forward_bags(bags), and its critical rows to those
functional.mil_forward_bags returns for that model.

Covered: the configurations of the reference's drivers on the batched path (D = 512 with C = 1, 2; D = 1024 with
C = 1, 2, 4; D = 2048 with C = 1, 2) at M = 1, 2, 5, and M = 8 at D = 512; ragged bags of 1, 127, 128, 129 and
10 000 rows; one bag; a batch whose nb * M entries exceed the shared-memory bag table; an unaligned bag view (the
per-model loop); the plain launch that kernel timing forces; IClassifier members; and eval_epoch_models against
eval_epoch."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import build_net
from oracle import dsmil_oracle as orc
from dsmil_wsi_b200 import _lib
from dsmil_wsi_b200 import functional as Fn
from dsmil_wsi_b200.ensemble import forward_bags_models

pytestmark = pytest.mark.gpu

PROF_ATTEND, PROF_FINAL, PROF_FUSED = 2, 3, 4


def _nets(D, C, M, seed=0):
    return [build_net(orc.random_params(D, C, seed + 101 * m, scale=2.0)).eval() for m in range(M)]


def _bags(sizes, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.rand(n, D, generator=g, device="cuda") for n in sizes]


def _params(net):
    ic, bc = net.i_classifier, net.b_classifier
    lin = ic._linear()
    W1, b1, W2, b2 = bc._q_params()
    return (lin.weight, lin.bias, W1, b1, W2, b2, None, None, bc.fcc.weight, bc.fcc.bias)


def _check(nets, bags, outs):
    assert len(outs) == len(nets)
    for m, (net, out) in enumerate(zip(nets, outs)):
        with torch.no_grad():
            ref = net.forward_bags(bags)
            _, ref_crit = Fn.mil_forward_bags(bags, _params(net))
        assert len(out) == len(ref) == len(bags)
        for b, (o, r) in enumerate(zip(out, ref)):
            for what, u, v in zip(("classes", "pred", "A", "B"), o, r):
                assert u.shape == v.shape and torch.equal(u, v), (m, b, what)
        assert torch.equal(out.crit, ref_crit), m


def _run(nets, bags):
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    outs = forward_bags_models(nets, bags)
    torch.cuda.synchronize()
    return outs, _lib.launch_count() - n0


CONFIGS = [(512, 1), (512, 2), (1024, 1), (1024, 2), (1024, 4), (2048, 1), (2048, 2)]


@pytest.mark.parametrize("M", [1, 2, 5])
@pytest.mark.parametrize("D,C", CONFIGS)
def test_reference_configurations(D, C, M):
    nets = _nets(D, C, M, seed=D + C)
    bags = _bags([129, 1000, 37, 256], D, seed=M)
    outs, launches = _run(nets, bags)
    assert launches == 4          # one weight-image prep, phase 1, attend, finalize for the whole ensemble
    _check(nets, bags, outs)


def test_eight_models_at_512():
    nets = _nets(512, 2, 8, seed=8)
    bags = _bags([300, 5, 128, 2000], 512, seed=8)
    outs, launches = _run(nets, bags)
    assert launches == 4
    _check(nets, bags, outs)


@pytest.mark.parametrize("D,C,M", [(512, 2, 5), (1024, 4, 2), (2048, 1, 5)])
def test_ragged_bags(D, C, M):
    nets = _nets(D, C, M, seed=3)
    bags = _bags([1, 127, 128, 129, 10_000], D, seed=4)
    outs, launches = _run(nets, bags)
    assert launches == 4
    _check(nets, bags, outs)


@pytest.mark.parametrize("n", [1, 10_000])
def test_one_bag(n):
    nets = _nets(512, 2, 5, seed=5)
    bags = _bags([n], 512, seed=n)
    outs, _ = _run(nets, bags)
    _check(nets, bags, outs)


def test_table_larger_than_shared_memory():
    nets = _nets(512, 2, 5, seed=6)
    rng = np.random.default_rng(6)
    bags = _bags([int(n) for n in rng.integers(1, 400, 25)], 512, seed=6)    # 125 entries > 96
    outs, launches = _run(nets, bags)
    assert launches == 4
    _check(nets, bags, outs)


def test_unaligned_bag_takes_the_per_model_loop():
    nets = _nets(512, 2, 3, seed=7)
    bags = _bags([300, 129], 512, seed=7)
    flat = torch.empty(200 * 512 + 1, device="cuda")
    flat[1:].copy_(torch.rand(200 * 512, device="cuda"))
    bags.append(flat[1:].view(200, 512))                  # 4 bytes off a 16-byte boundary
    assert bags[-1].data_ptr() % 16 != 0
    outs, launches = _run(nets, bags)
    assert launches > 4
    _check(nets, bags, outs)


def test_plain_launch_under_kernel_timing():
    lib = _lib.load()
    nets = _nets(1024, 2, 5, seed=9)
    bags = _bags([10_000, 129, 1], 1024, seed=9)
    torch.cuda.synchronize()
    ms, n = (ctypes.c_double * 8)(), (ctypes.c_uint64 * 8)()
    lib.dsmil_profile_read(ms, n)                          # drop earlier records
    lib.dsmil_profile_enable(1)
    try:
        outs = forward_bags_models(nets, bags)
        torch.cuda.synchronize()
        lib.dsmil_profile_read(ms, n)
    finally:
        lib.dsmil_profile_enable(0)
    assert (n[PROF_FUSED], n[PROF_ATTEND], n[PROF_FINAL]) == (1, 1, 1)
    _check(nets, bags, outs)
    # and the overlapped launch gives the same bits
    again = forward_bags_models(nets, bags)
    for o, a in zip(outs, again):
        assert all(torch.equal(u, v) for u, v in zip(o.packed, a.packed)) and torch.equal(o.crit, a.crit)


def test_iclassifier_members():
    import dsmil as mil
    D, C = 512, 2
    nets = []
    for m in range(3):
        p = orc.random_params(D, C, 40 + m, scale=2.0)
        ic = mil.IClassifier(torch.nn.Identity(), D, C) if m != 1 else mil.FCLayer(D, C)
        net = mil.MILNet(ic, mil.BClassifier(D, C)).cuda().eval()
        with torch.no_grad():
            lin = ic._linear()
            lin.weight.copy_(torch.from_numpy(np.asarray(p.Wi, np.float32)))
            lin.bias.copy_(torch.from_numpy(np.asarray(p.bi, np.float32)))
        nets.append(net)
    bags = _bags([129, 700], D, seed=41)
    outs = forward_bags_models(nets, bags)
    for net, out in zip(nets, outs):
        with torch.no_grad():
            ref = net.forward_bags(bags)
        for o, r in zip(out, ref):
            assert all(torch.equal(u, v) for u, v in zip(o, r))


@pytest.mark.parametrize("average", [False, True])
@pytest.mark.parametrize("k", [4, 1])
def test_eval_epoch_models_equals_eval_epoch(average, k):
    from dsmil_wsi_b200.feed import DeviceBagStore, eval_epoch, eval_epoch_models
    D, C = 512, 2
    nets = _nets(D, C, 5, seed=11)
    store = DeviceBagStore(D)
    for i in range(9):
        label = torch.zeros(C)
        label[i % C] = float(i % 2)
        store.add_bag(torch.rand(40 + 61 * i, D), label)
    crit = torch.nn.BCEWithLogitsLoss()
    got = eval_epoch_models(nets, store, crit, average=average, bags_per_launch=k)
    assert len(got) == len(nets)
    for net, (loss, labels, preds) in zip(nets, got):
        loss_r, labels_r, preds_r = eval_epoch(net, store, crit, average=average, bags_per_launch=k)
        assert loss == loss_r
        assert labels.dtype == labels_r.dtype and np.array_equal(labels, labels_r)
        assert preds.dtype == preds_r.dtype and np.array_equal(preds, preds_r)
