"""Training on a minibatch of row-sharded bags, without a GPU: argument validation and workspace sizes of the new entry
points (calls that return before any CUDA work), and the host logic of the step -- sharded_forward_bags_train,
sharded_caller_loss_bags, sharded_backward_bags through ShardedMILBagsFn -- over gloo with 2 and 3 ranks and with the
fp64 oracle's one-bag ops run per bag through PerBagShardOps, plus the single-process virtual-rank helper."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import rel_to_max
from oracle import dsmil_oracle as orc
from test_sharded_gloo import OracleTrainOps, _free_port
from dsmil_wsi_b200 import _lib

ERR_ARG, ERR_WORKSPACE, ERR_EMPTY = -1, -2, -4
FAKE = 0x10000          # a non-NULL, 16-byte aligned "device pointer": never dereferenced on these paths
ORDER = ["Wi", "bi", "W1", "b1", "W2", "b2", "Wf", "bf"]


def params(D=512, C_=2, passing_v=0):
    p = _lib.DsmilParams(D, C_, 1, passing_v)
    for name in ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf"):
        setattr(p, name, FAKE)
    return p


def last_error(lib):
    return (lib.dsmil_last_error() or b"").decode()


def arrays(Ns):
    nb = len(Ns)
    return (C.c_void_p * nb)(*[FAKE] * nb), (C.c_int64 * nb)(*Ns), (C.c_int64 * nb)(*[0] * nb)


def _ref(p):
    return None if p is None else C.byref(p)


# every new entry point as f(lib, p, Xs, Ns, offs, nb, ws, wsb, null=<index of one buffer argument to pass as NULL>)
def _call(fn, p, head, bufs, ws, wsb, null):
    bufs = [None if i == null else b for i, b in enumerate(bufs)]
    return fn(_ref(p), *head, *bufs, ws, wsb, None)


def p1_train(lib, p, Xs, Ns, offs, nb, ws=None, wsb=0, null=None):
    return _call(lib.dsmil_shard_bags_phase1_train, p, (Xs, Ns, nb, offs), [FAKE] * 4, ws, wsb, null)


def p2_train(lib, p, Xs, Ns, offs, nb, ws=None, wsb=0, null=None):
    b = [None if i == null else FAKE for i in range(6)]       # Q, cands_all, A, crit_idx, q_max, recs_out
    return lib.dsmil_shard_bags_phase2_train(_ref(p), Xs, Ns, nb, b[0], b[1], 2, *b[2:], ws, wsb, None)


def b1(lib, p, Xs, Ns, offs, nb, ws=None, wsb=0, null=None):
    # A, B, d_classes, d_pred, dA, t, gWi, gbi, gWf, gbf: d_classes, d_pred and the gradients may be NULL
    return _call(lib.dsmil_shard_backward_bags_phase1, p, (Xs, Ns, nb), [FAKE] * 10, ws, wsb, null)


def b2(lib, p, Xs, Ns, offs, nb, ws=None, wsb=0, null=None):
    return _call(lib.dsmil_shard_backward_bags_phase2, p, (Ns, nb), [FAKE] * 5, ws, wsb, null)


def b3(lib, p, Xs, Ns, offs, nb, ws=None, wsb=0, null=None):
    return _call(lib.dsmil_shard_backward_bags_phase3, p, (Xs, Ns, nb, offs), [FAKE] * 10, ws, wsb, null)


def _need(lib, fn, p, Ns):
    _, n, _ = arrays(Ns)
    if fn in (p1_train, p2_train):
        return lib.dsmil_shard_bags_workspace_bytes(C.byref(p), n, len(Ns))
    return lib.dsmil_shard_backward_bags_workspace_bytes(C.byref(p), n, len(Ns))


@pytest.mark.parametrize("fn", [p1_train, p2_train, b1, b2, b3])
def test_entry_point_validation(fn):
    lib = _lib.load()
    p = params()
    Ns = [100, 200, 1]
    Xs, n, offs = arrays(Ns)
    big = 1 << 40
    assert fn(lib, p, Xs, n, offs, 0, FAKE, big) == ERR_ARG and "nb outside" in last_error(lib)
    assert fn(lib, p, Xs, n, offs, 65536, FAKE, big) == ERR_ARG
    assert fn(lib, params(passing_v=1), Xs, n, offs, 3, FAKE, big) == ERR_ARG and "identity v" in last_error(lib)
    assert fn(lib, params(D=500), Xs, n, offs, 3, FAKE, big) == ERR_ARG and "not supported" in last_error(lib)
    assert fn(lib, None, Xs, n, offs, 3, FAKE, big) == ERR_ARG
    assert fn(lib, p, Xs, None, offs, 3, FAKE, big) == ERR_ARG
    if fn is not b2:                           # phase 2 of the backward reads no features
        assert fn(lib, p, None, n, offs, 3, FAKE, big) == ERR_ARG
    required = {p1_train: range(4), p2_train: range(6), b1: [0, 1, 4, 5], b2: range(5), b3: range(6)}[fn]
    for i in required:                          # each required buffer as NULL
        assert fn(lib, p, Xs, n, offs, 3, FAKE, big, null=i) == ERR_ARG, i
    if fn in (p1_train, b3):                   # the host array of row offsets
        assert fn(lib, p, Xs, n, None, 3, FAKE, big) == ERR_ARG
    # a bag with no local row on this rank
    X0, n0, o0 = arrays([100, 0, 1])
    assert fn(lib, p, X0, n0, o0, 3, FAKE, big) == ERR_EMPTY
    need = _need(lib, fn, p, Ns)
    assert need > 0
    assert fn(lib, p, Xs, n, offs, 3, None, 0) == ERR_WORKSPACE
    assert fn(lib, p, Xs, n, offs, 3, FAKE, need - 1) == ERR_WORKSPACE and "workspace too small" in last_error(lib)


def test_inference_phases_refuse_more_than_65535_bags():
    """dsmil_shard_bags_phase1/2/3 number the bags in grid y, as the training phases do: outside [1, 65535] each is
    DSMIL_ERR_ARG before any launch, and the workspace size is 0."""
    lib = _lib.load()
    p = params()
    Xs, n, offs = arrays([3] * 65536)
    calls = {
        "phase1": lambda nb: lib.dsmil_shard_bags_phase1(C.byref(p), Xs, n, nb, offs, FAKE, FAKE, FAKE, 1 << 40, None),
        "phase2": lambda nb: lib.dsmil_shard_bags_phase2(C.byref(p), Xs, n, nb, FAKE, 2, FAKE, FAKE, FAKE, FAKE,
                                                         1 << 40, None),
        "phase3": lambda nb: lib.dsmil_shard_bags_phase3(C.byref(p), Xs, n, nb, FAKE, 2, FAKE, FAKE, FAKE, FAKE,
                                                         1 << 40, None),
    }
    for name, call in calls.items():
        for nb in (0, 65536, 70000):
            assert call(nb) == ERR_ARG and f"nb={nb} outside [1, 65535]" in last_error(lib), (name, nb)
    assert lib.dsmil_shard_bags_workspace_bytes(C.byref(p), n, 65536) == 0
    assert lib.dsmil_shard_bags_workspace_bytes(C.byref(p), n, 65535) > 0


def test_backward_phase1_optional_buffers_pass_validation():
    """d_classes, d_pred and every gradient buffer may be NULL: those arguments fail nothing before the workspace."""
    lib = _lib.load()
    p = params()
    Xs, n, offs = arrays([100, 3])
    for i in (2, 3, 6, 7, 8, 9):
        assert b1(lib, p, Xs, n, offs, 2, None, 0, null=i) == ERR_WORKSPACE, i


@pytest.mark.parametrize("D,C_", [(512, 2), (512, 1), (1024, 4), (2048, 2)])
def test_workspace_sizes_grow_with_rows(D, C_):
    lib = _lib.load()
    p = params(D, C_)
    batches = [[1], [1, 2], [128, 129], [2049, 127, 1], [10000] * 4, [15000] * 16, [15000] * 16 + [1]]
    sizes = []
    for Ns in batches:
        _, n, _ = arrays(Ns)
        sizes.append(lib.dsmil_shard_backward_bags_workspace_bytes(C.byref(p), n, len(Ns)))
        # the single-device batched backward needs no more: the sharded carve only appends the row offsets
        assert sizes[-1] >= lib.dsmil_backward_bags_workspace_bytes(C.byref(p), n, len(Ns), 0)
    assert sizes[0] > 0 and sizes == sorted(sizes)
    _, n, _ = arrays([100])
    assert lib.dsmil_shard_backward_bags_workspace_bytes(C.byref(params(passing_v=1)), n, 1) == 0
    assert lib.dsmil_shard_backward_bags_workspace_bytes(C.byref(params(D=500)), n, 1) == 0
    assert lib.dsmil_shard_backward_bags_workspace_bytes(C.byref(p), n, 0) == 0


# ---- the host logic over gloo, with the one-bag fp64 oracle run per bag through PerBagShardOps ----------------
def _problem(sizes, D=48, C_=2):
    p = orc.random_params(D, C_, seed=31, scale=1.5)
    Xs = [orc.synthetic_bag(n, D, 500 + i, "normal") for i, n in enumerate(sizes)]
    y = (np.random.default_rng(len(sizes)).random((len(sizes), C_)) > 0.5).astype(np.float32)
    return p, Xs, y


def _oracle_batch(p, Xs, y):
    """Mean loss over the bags and the sum of the per-bag oracle gradients of loss_b / nb."""
    nb, loss, want = len(Xs), 0.0, {}
    for X, yb in zip(Xs, y):
        o = orc.forward(X, p)
        l, dc, dp = orc.caller_loss_grads(o, yb.astype(np.float64))
        loss += l / nb
        for k, v in orc.backward(X, p, o, dc / nb, dp / nb).items():
            want[k] = want.get(k, 0) + v
    return loss, want


def _bags_train_worker(rank, world, port, sizes, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from helpers import build_net
        from dsmil_wsi_b200.sharded import (PerBagShardOps, shard_bounds, sharded_caller_loss_bags,
                                            sharded_milnet_forward_bags)
        p, Xs, y = _problem(sizes)
        net = build_net(p, device="cpu")
        xs, offs = [], []
        for X in Xs:
            lo, hi = shard_bounds(X.shape[0], world)[rank]
            xs.append(torch.from_numpy(X[lo:hi]))
            offs.append(lo)
        counts = {"all_gather": 0, "sum": 0, "max": 0}
        real_gather, real_reduce = dist.all_gather_into_tensor, dist.all_reduce

        def gather(*a, **k):
            counts["all_gather"] += 1
            return real_gather(*a, **k)

        def reduce(t, op=dist.ReduceOp.SUM, **k):
            counts["max" if op == dist.ReduceOp.MAX else "sum"] += 1
            return real_reduce(t, op=op, **k)
        dist.all_gather_into_tensor, dist.all_reduce = gather, reduce
        classes, pred, A, B, crit = sharded_milnet_forward_bags(net, xs, offs, ops=PerBagShardOps(OracleTrainOps(p)))
        loss = sharded_caller_loss_bags(classes, pred, crit, offs, torch.from_numpy(y), torch.nn.BCEWithLogitsLoss(),
                                        Ns=[x.shape[0] for x in xs])
        loss.backward()
        ret[rank] = dict(loss=float(loss.detach()), counts=counts, crit=crit.numpy(),
                         grads={k: v.grad.numpy().copy() for k, v in net.named_parameters()})
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,sizes", [(2, [37, 5, 120, 1]), (3, [2, 64, 9, 1, 3]), (2, [11])])
def test_sharded_bags_training_step_over_gloo(world, sizes):
    """Six collectives per step whatever nb (2 all-gathers, 3 all-reduce(sum), 1 all-reduce(max)); every rank ends with
    the same loss and bit-identical gradients, the sum over the bags of the oracle's."""
    from helpers import grad_name
    port = _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_bags_train_worker, args=(world, port, sizes, ret), nprocs=world, join=True)
    p, Xs, y = _problem(sizes)
    loss, want = _oracle_batch(p, Xs, y)
    crit = np.stack([orc.forward(X, p).idx for X in Xs])
    for r in range(world):
        o = ret[r]
        assert o["counts"] == {"all_gather": 2, "sum": 3, "max": 1}, o["counts"]
        assert np.array_equal(o["crit"], crit)
        assert abs(o["loss"] - loss) < 2e-6
        assert o["loss"] == ret[0]["loss"]
        for short, w in want.items():
            assert rel_to_max(o["grads"][grad_name(short, True)], w) < 5e-5, (r, short)
        for k in o["grads"]:
            assert np.array_equal(o["grads"][k], ret[0]["grads"][k]), k


def _loss_grads(y):
    """d(loss)/d(classes, pred) of the minibatch loss over packed, bag-ordered outputs (autograd in torch)."""
    def fn(classes, pred, crit):
        Ns = fn.Ns
        first = torch.tensor([0] + list(np.cumsum(Ns)[:-1]), dtype=torch.int64)
        with torch.enable_grad():
            c, pr = classes.detach().clone().requires_grad_(True), pred.detach().clone().requires_grad_(True)
            crit_fn = torch.nn.BCEWithLogitsLoss()
            yy = torch.from_numpy(y).to(pr.dtype)
            mx = c.gather(0, crit + first[:, None])
            (0.5 * crit_fn(pr, yy) + 0.5 * crit_fn(mx, yy)).backward()
        return c.grad, pr.grad
    return fn


@pytest.mark.parametrize("G,sizes", [(1, [37, 5]), (2, [37, 5, 120, 1]), (3, [2, 64, 9, 3]), (8, [40, 17, 8])])
def test_virtual_sharded_train_step_bags_host_logic(G, sizes):
    from dsmil_wsi_b200.sharded import PerBagShardOps, virtual_sharded_train_step_bags
    p, Xs, y = _problem(sizes)
    loss, want = _oracle_batch(p, Xs, y)
    lg = _loss_grads(y)
    lg.Ns = sizes
    outs, grads = virtual_sharded_train_step_bags(lambda: PerBagShardOps(OracleTrainOps(p)),
                                                  [torch.from_numpy(X) for X in Xs], G, lg)
    classes, pred, A, B, crit = outs
    ones = [orc.forward(X, p) for X in Xs]
    assert np.array_equal(crit.numpy(), np.stack([o.idx for o in ones]))
    assert rel_to_max(classes.numpy(), np.concatenate([o.classes for o in ones])) < 1e-12
    assert rel_to_max(A.numpy(), np.concatenate([o.A for o in ones])) < 2e-6
    assert rel_to_max(pred.numpy(), np.concatenate([o.prediction_bag for o in ones])) < 2e-6
    for short, got in zip(ORDER, grads):
        assert rel_to_max(got.numpy(), want[short]) < 5e-5, short
