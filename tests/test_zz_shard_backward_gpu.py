"""Row-sharded reverse pass on the device (SURVEY 8e "Backward"): `dsmil_shard_backward_phase1/2/3` with G logical
shards on one GPU (reductions as local sums) must give the gradients of the single-device backward and of the
fp64 oracle; with >= 2 GPUs the autograd path over NCCL is run as well.  Written after this round's GPU budget
was spent; runs after the parity suites on purpose."""
import os
import socket

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_to_max
from helpers import build_net, caller_loss, grad_name
from oracle import dsmil_oracle as orc

pytestmark = pytest.mark.gpu

ORDER = ["Wi", "bi", "W1", "b1", "W2", "b2", "Wf", "bf"]


def _loss_grads(y):
    def fn(classes, pred, crit):
        with torch.enable_grad():
            c, p = classes.detach().clone().requires_grad_(True), pred.detach().clone().requires_grad_(True)
            caller_loss(c, p, y).backward()
        return c.grad, p.grad
    return fn


@pytest.mark.parametrize("name,G", [("shipped_tcga", 1), ("shipped_tcga", 3), ("shipped_c16", 2), ("musk_d166_n7", 8),
                                    ("lin_d512_c3", 4), ("tree_d1024_c2", 7), ("musk_d166_n1", 2)])
def test_virtual_shards_of_one_bag_give_single_device_gradients(name, G):
    from dsmil_wsi_b200.sharded import CudaShardOps, PerBagShardOps, milnet_params, virtual_sharded_train_step_bags
    g, p, X = load_golden(name)
    net = build_net(p).train()
    x = torch.from_numpy(X).cuda()
    y = torch.from_numpy(np.asarray(g["y"], np.float32).reshape(-1)).cuda()
    # single-device product path (autograd through dsmil_backward; checked against the reference in test_gpu_parity)
    c1, p1, _, _ = net(x)
    caller_loss(c1, p1, y).backward()
    single = {k: v.grad.detach().cpu().numpy() for k, v in net.named_parameters()}
    ops = CudaShardOps(milnet_params(net))
    (classes, pred, A, B, crit), grads = virtual_sharded_train_step_bags(lambda: PerBagShardOps(ops), [x], G,
                                                                         _loss_grads(y))
    assert torch.equal(classes, c1.detach()) and np.array_equal(crit[0].cpu().numpy(), g["idx"])
    one = orc.forward(X, p)
    _, d_cls, d_pred = orc.caller_loss_grads(one, np.asarray(g["y"], np.float64).reshape(-1))
    ref = orc.backward(X, p, one, d_cls, d_pred)
    for short, got in zip(ORDER, grads):
        if got is None:
            assert short in ("W2", "b2") and not p.nonlinear
            continue
        got = got.cpu().numpy()
        want1, want64 = single[grad_name(short, p.nonlinear)], ref[short]
        assert got.shape == want1.shape
        scale = max(np.abs(want64).max(), 1e-30)
        if np.abs(want64).max() < 1e-12:                       # N == 1: the q branch gets exactly no gradient
            assert np.abs(got).max() < 1e-7, short
            continue
        # same kernels and the same fp32 forward as the single-device pass: shard sums only reorder additions
        assert np.abs(got - want1).max() <= 2e-4 * scale, (short, np.abs(got - want1).max() / scale)
        # and the oracle, at the single-device backward's documented tolerance (DESIGN.md §3)
        assert np.abs(got - want64).max() <= 2e-3 * scale, (short, np.abs(got - want64).max() / scale)


def _nccl_train_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from dsmil_wsi_b200.sharded import shard_bounds, sharded_caller_loss, sharded_milnet_forward
        g, p, X = load_golden("shipped_tcga")
        net = build_net(p, device=f"cuda:{rank}").train()
        lo, hi = shard_bounds(X.shape[0], world)[rank]
        y = torch.from_numpy(np.asarray(g["y"], np.float32).reshape(-1)).cuda()
        classes, pred, A, B, crit = sharded_milnet_forward(net, torch.from_numpy(X[lo:hi]).cuda(), lo)
        loss = sharded_caller_loss(classes, pred, crit, lo, y, torch.nn.BCEWithLogitsLoss())
        loss.backward()
        torch.cuda.synchronize()
        ret[rank] = dict(loss=float(loss.detach()), grads={k: v.grad.cpu().numpy() for k, v in net.named_parameters()})
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs (gpurun --gpus 2)")
def test_nccl_two_rank_training_step():
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ret = mp.Manager().dict()
    mp.spawn(_nccl_train_worker, args=(2, port, ret), nprocs=2, join=True)
    g, p, X = load_golden("shipped_tcga")
    one = orc.forward(X, p)
    loss, d_cls, d_pred = orc.caller_loss_grads(one, np.asarray(g["y"], np.float64).reshape(-1))
    ref = orc.backward(X, p, one, d_cls, d_pred)
    for r in range(2):
        assert abs(ret[r]["loss"] - loss) < 1e-5
        for short, want in ref.items():
            got = ret[r]["grads"][grad_name(short, p.nonlinear)]
            assert np.abs(got - want).max() <= 2e-3 * np.abs(want).max(), (r, short)
        for k in ret[r]["grads"]:
            assert np.array_equal(ret[r]["grads"][k], ret[0]["grads"][k]), k
