"""Training on a minibatch of row-sharded bags, on the device: the three batched sharded backward phases at one rank
against dsmil_backward_bags bit for bit; G virtual ranks on one GPU against forward_bags(grad=True) and the fp64
oracle; determinism; a loss that never waits for the stream; an SGD step through ShardedMILBagsFn + sharded_caller_loss_bags over two processes against
feed.train_epoch(bags_per_step=k); and the same step over NCCL on two GPUs when the box has them."""
import copy
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch

from conftest import rel_to_max
from helpers import build_net, grad_name
from oracle import dsmil_oracle as orc
from dsmil_wsi_b200 import _lib, feed
from dsmil_wsi_b200 import functional as Fn

pytestmark = pytest.mark.gpu

ORDER = ["Wi", "bi", "W1", "b1", "W2", "b2", "Wf", "bf"]
# DESIGN.md §3: gradients 5e-4 rel-to-max; 2e-3 for the q.* gradients of batches with a bag of >= 10 000 rows
TOL, TOL_Q = 5e-4, 2e-3


def _np(t):
    return t.detach().cpu().numpy() if torch.is_tensor(t) else t


def _bags(Ns, D, seed):
    raw = [orc.synthetic_bag(n, D, seed + i) for i, n in enumerate(Ns)]
    return [torch.from_numpy(x).cuda() for x in raw], raw


def _labels(C_, nb, seed):
    return torch.from_numpy((np.random.default_rng(seed).random((nb, C_)) > 0.5).astype(np.float32)).cuda()


def _backward_bags(P, xs, Q, H1, A, B, crit, dc, dp):
    """dsmil_backward_bags on the given saved tensors; gradients in ORDER."""
    lib = _lib.load()
    nb = len(xs)
    c_X, c_N = (C.c_void_p * nb)(*[x.data_ptr() for x in xs]), (C.c_int64 * nb)(*[x.shape[0] for x in xs])
    shapes = [(P.C, P.D), (P.C,), (128, P.D), (128,), (128, 128), (128,), (P.C, P.C, P.D), (P.C,)]
    g = [torch.empty(s, device="cuda") for s in shapes]
    G = _lib.DsmilGrads(*[t.data_ptr() for t in g[:6]], None, None, g[6].data_ptr(), g[7].data_ptr(), None)
    ws = Fn._workspace(lib.dsmil_backward_bags_workspace_bytes(P.ref, c_N, nb, 0), P.device)
    _lib.check(lib.dsmil_backward_bags(P.ref, c_X, c_N, nb, Q.data_ptr(), H1.data_ptr(), A.data_ptr(), B.data_ptr(),
                                       crit.data_ptr(), dc.data_ptr(), dp.data_ptr(), None, None, C.byref(G),
                                       ws.data_ptr(), ws.numel(), Fn._stream()), "dsmil_backward_bags")
    return g


@pytest.mark.parametrize("D,C_,Ns", [(512, 2, [1, 127, 128, 129, 10000]), (1024, 4, [129, 1, 10000, 128, 127])])
def test_one_rank_is_the_single_device_backward_bit_for_bit(D, C_, Ns):
    from dsmil_wsi_b200.sharded import CudaShardBagOps, milnet_params
    p = orc.random_params(D, C_, seed=D + C_)
    net = build_net(p)
    params = milnet_params(net)
    xs, _ = _bags(Ns, D, seed=7 * D)
    bops = CudaShardBagOps(params)
    nb, offs = len(xs), [0] * len(xs)
    # the saved tensors: the training forward of the sharded batch at one rank (its gathers are the identity)
    xs = bops.begin(xs, offs)
    classes, Q, H1, cand = bops.phase1_train()
    A, crit, qmax, recs = bops.phase2_train(Q, cand.reshape(-1), 1)
    A, B, pred = bops.phase3_train(recs.reshape(-1), 1, A)
    first = torch.tensor([0] + list(np.cumsum(Ns)[:-1]), device="cuda")
    assert torch.equal(qmax, Q[crit + first[:, None]])                   # the candidate carries Q's row unchanged
    g = torch.Generator(device="cuda").manual_seed(3)
    dc = torch.randn(sum(Ns), C_, device="cuda", generator=g)
    dp = torch.randn(nb, C_, device="cuda", generator=g)
    want = _backward_bags(bops.P, xs, Q, H1, A, B, crit, dc, dp)
    dA, t, gWi, gbi, gWf, gbf = bops.bwd1(xs, A, B, dc, dp)
    dL, dqm = bops.bwd2(xs, A, dA, t, Q)                                  # all-reduces of one rank: identity
    gW1, gb1, gW2, gb2 = bops.bwd3(xs, offs, Q, H1, dL, dqm, qmax, crit)
    for name, got, w in zip(ORDER, (gWi, gbi, gW1, gb1, gW2, gb2, gWf, gbf), want):
        assert torch.equal(got, w), (name, float((got - w).abs().max()))


def _loss_grads(y):
    """d(loss)/d(classes, pred) of feed.train_epoch's minibatch loss over packed, bag-ordered outputs."""
    def fn(classes, pred, crit):
        Ns = fn.Ns
        first = torch.tensor([0] + list(np.cumsum(Ns)[:-1]), dtype=torch.int64, device=classes.device)
        with torch.enable_grad():
            c, pr = classes.detach().clone().requires_grad_(True), pred.detach().clone().requires_grad_(True)
            bce = torch.nn.BCEWithLogitsLoss()
            (0.5 * bce(pr, y) + 0.5 * bce(c.gather(0, crit + first[:, None]), y)).backward()
        return c.grad, pr.grad
    return fn


def _oracle_sum(p, raw, y):
    want = {}
    for b, X in enumerate(raw):
        o = orc.forward(X, p)
        _, dc, dp = orc.caller_loss_grads(o, y[b].cpu().numpy().astype(np.float64))
        for k, v in orc.backward(X, p, o, dc / len(raw), dp / len(raw)).items():
            want[k] = want.get(k, 0) + v
    return want


def _tol(short, Ns):
    return TOL_Q if (short in ("W1", "b1", "W2", "b2") and max(Ns) >= 10000) else TOL


def _single_device_grads(net, xs, y):
    """Gradients of train_epoch's minibatch loss through forward_bags(grad=True) (on a copy of net), and its outputs."""
    net = copy.deepcopy(net).train()
    outs = net.forward_bags(xs, grad=True)
    pred, mx = feed._group_predictions(outs)
    bce = torch.nn.BCEWithLogitsLoss()
    (0.5 * bce(pred, y) + 0.5 * bce(mx, y)).backward()
    return {k: _np(v.grad) for k, v in net.named_parameters()}, outs, pred


def _check_grads(grads, single, want, Ns, what):
    """Against forward_bags(grad=True) at the gradient tolerance, and against the fp64 oracle at that tolerance or, when
    the single-device path itself is further (the forward's rounding amplified by the softmax over a 10 000-row bag),
    its distance plus 10 %, as tests/test_zz_bags_train_gpu.py allows."""
    for short, got in zip(ORDER, grads):
        tol, one = _tol(short, Ns), single[grad_name(short, True)]
        assert rel_to_max(_np(got), one) <= tol, (what, short, "forward_bags", rel_to_max(_np(got), one))
        tol = max(tol, 1.1 * rel_to_max(one, want[short]))
        assert rel_to_max(_np(got), want[short]) <= tol, (what, short, "oracle", rel_to_max(_np(got), want[short]))


VIRTUAL_NS = [10000, 129, 2049, 17]


@pytest.mark.parametrize("G", [2, 3, 8])
def test_virtual_ranks_match_forward_bags_and_oracle(G):
    from dsmil_wsi_b200.sharded import CudaShardBagOps, milnet_params, virtual_sharded_train_step_bags
    D, C_ = 512, 2
    p = orc.random_params(D, C_, seed=40 + G)
    net = build_net(p).train()
    xs, raw = _bags(VIRTUAL_NS, D, seed=100)
    y = _labels(C_, len(xs), seed=G)
    single, outs, pr1 = _single_device_grads(net, xs, y)
    lg = _loss_grads(y)
    lg.Ns = VIRTUAL_NS
    params = milnet_params(net)
    (classes, pred, A, B, crit), grads = virtual_sharded_train_step_bags(lambda: CudaShardBagOps(params), xs, G, lg)
    ones = [orc.forward(X, p) for X in raw]
    assert torch.equal(crit, outs.crit) and np.array_equal(_np(crit), np.stack([o.idx for o in ones]))
    c1, _, A1, B1 = outs.packed
    assert rel_to_max(_np(classes), _np(c1)) < 2e-6
    assert rel_to_max(_np(A), _np(A1)) < 2e-6 and rel_to_max(_np(B), _np(B1)) < 2e-6
    assert rel_to_max(_np(pred), _np(pr1)) < 1e-5
    assert rel_to_max(_np(A), np.concatenate([o.A for o in ones])) < 2e-5
    assert rel_to_max(_np(B), np.concatenate([o.B for o in ones])) < 1e-5
    _check_grads(grads, single, _oracle_sum(p, raw, y), VIRTUAL_NS, f"G={G}")


def test_virtual_step_is_deterministic():
    from dsmil_wsi_b200.sharded import CudaShardBagOps, milnet_params, virtual_sharded_train_step_bags
    p = orc.random_params(512, 2, seed=5)
    net = build_net(p)
    xs, _ = _bags(VIRTUAL_NS, 512, seed=9)
    lg = _loss_grads(_labels(2, len(xs), seed=1))
    lg.Ns = VIRTUAL_NS
    params = milnet_params(net)
    runs = [virtual_sharded_train_step_bags(lambda: CudaShardBagOps(params), xs, 3, lg) for _ in range(2)]
    for a, b in zip(runs[0][0] + runs[0][1], runs[1][0] + runs[1][1]):
        assert torch.equal(a, b)


def test_caller_loss_does_not_sync_the_host(monkeypatch):
    """The sharded loss of one bag and of three, forward and backward, only enqueues device work: no call waits for
    the stream.  The all-reduce(max) is stubbed as the identity of one rank, so this rank owns every critical row."""
    import torch.distributed as dist
    from dsmil_wsi_b200.sharded import sharded_caller_loss, sharded_caller_loss_bags
    monkeypatch.setattr(dist, "all_reduce", lambda tensor, op=None, group=None, async_op=False: None)
    Ns, offs, C_ = [37, 1, 200], [0, 5, 1000], 2
    g = torch.Generator(device="cuda").manual_seed(11)
    classes = torch.randn(sum(Ns), C_, device="cuda", generator=g)
    pred = torch.randn(len(Ns), C_, device="cuda", generator=g)
    y = (torch.rand(len(Ns), C_, device="cuda", generator=g) > 0.5).float()
    first = [0] + list(np.cumsum(Ns)[:-1])
    local = torch.stack([classes[f:f + n].argmax(0) for f, n in zip(first, Ns)])          # [nb, C] local rows
    crit = local + torch.tensor(offs, device="cuda")[:, None]
    bce = torch.nn.BCEWithLogitsLoss()

    def leaves(nb):
        n = sum(Ns[:nb])
        return classes[:n].clone().requires_grad_(True), pred[:nb].clone().requires_grad_(True)

    def check(loss, c, p, nb):
        """Against the single-device loss of the same bags (its max instance: each bag's critical row)."""
        cr, pr = leaves(nb)
        rows = local[:nb] + torch.tensor(first[:nb], device="cuda")[:, None]
        ref = 0.5 * bce(pr, y[:nb]) + 0.5 * bce(cr.gather(0, rows), y[:nb])
        ref.backward()
        assert torch.equal(loss, ref) and torch.equal(c.grad, cr.grad) and torch.equal(p.grad, pr.grad), nb

    (c1, p1), (c3, p3) = leaves(1), leaves(3)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        one = sharded_caller_loss(c1, p1, crit[0], offs[0], y[0], bce)
        one.backward()
        many = sharded_caller_loss_bags(c3, p3, crit, offs, y, bce, Ns=Ns)
        many.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    check(one, c1, p1, 1)
    check(many, c3, p3, 3)


# ---- an SGD step through the autograd node, two ranks (two processes) ----------------------------------------------
STEP_NS, STEP_D, STEP_C, LR = [10000, 300, 2, 2049], 512, 2, 0.05      # every bag holds a row on each rank


def _step_problem():
    p = orc.random_params(STEP_D, STEP_C, seed=77)
    raw = [orc.synthetic_bag(n, STEP_D, 60 + i) for i, n in enumerate(STEP_NS)]
    y = (np.random.default_rng(8).random((len(raw), STEP_C)) > 0.5).astype(np.float32)
    return p, raw, y


def _step_worker(rank, world, port, backend, ret):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = rank if backend == "nccl" else 0
    torch.cuda.set_device(dev)
    kw = {"device_id": torch.device("cuda", dev)} if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    try:
        from dsmil_wsi_b200.sharded import shard_bounds, sharded_caller_loss_bags, sharded_milnet_forward_bags
        p, raw, y = _step_problem()
        net = build_net(p, device=f"cuda:{dev}").train()
        xs, offs = [], []
        for X in raw:
            lo, hi = shard_bounds(X.shape[0], world)[rank]
            xs.append(torch.from_numpy(X[lo:hi]).cuda())
            offs.append(lo)
        opt = torch.optim.SGD(net.parameters(), lr=LR)
        opt.zero_grad()
        classes, pred, A, B, crit = sharded_milnet_forward_bags(net, xs, offs)
        loss = sharded_caller_loss_bags(classes, pred, crit, offs, torch.from_numpy(y).cuda(),
                                        torch.nn.BCEWithLogitsLoss(), Ns=[x.shape[0] for x in xs])
        loss.backward()
        grads = {k: v.grad.cpu().numpy().copy() for k, v in net.named_parameters()}
        opt.step()
        torch.cuda.synchronize()
        ret[rank] = dict(loss=float(loss.detach()), crit=crit.cpu().numpy(), grads=grads,
                         params={k: v.detach().cpu().numpy().copy() for k, v in net.named_parameters()})
    finally:
        dist.destroy_process_group()


def _run_step(world, backend):
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ret = mp.Manager().dict()
    mp.spawn(_step_worker, args=(world, port, backend, ret), nprocs=world, join=True)
    # the same step on one device through feed.train_epoch(bags_per_step=k)
    p, raw, y = _step_problem()
    net = build_net(p)
    ref = copy.deepcopy(net)
    single, _, _ = _single_device_grads(net, [torch.from_numpy(X).cuda() for X in raw], torch.from_numpy(y).cuda())
    store = feed.DeviceBagStore(STEP_D)
    for X, yb in zip(raw, y):
        store.add_bag(torch.from_numpy(X), torch.from_numpy(yb))
    loss = feed.train_epoch(net, store, torch.nn.BCEWithLogitsLoss(), torch.optim.SGD(net.parameters(), lr=LR),
                            order=list(range(len(raw))), generator=torch.Generator(device="cuda").manual_seed(0),
                            bags_per_step=len(raw))
    want = _oracle_sum(p, raw, torch.from_numpy(y))
    eps = torch.finfo(torch.float32).eps
    crit = np.stack([orc.forward(X, p).idx for X in raw])
    for r in range(world):
        o = ret[r]
        assert np.array_equal(o["crit"], crit)
        assert abs(o["loss"] - loss) <= 1e-5 * max(1.0, abs(loss)) and o["loss"] == ret[0]["loss"]
        _check_grads([o["grads"][grad_name(k, True)] for k in ORDER], single, want, STEP_NS, f"rank {r}")
        for (name, a), b in zip(net.named_parameters(), ref.parameters()):
            short = [k for k in ORDER if grad_name(k, True) == name][0]
            gmax = float(np.abs(want[short]).max())
            tol = 2 * _tol(short, STEP_NS) * LR * gmax + 3 * eps * float(b.detach().abs().max())
            d = float(np.abs(o["params"][name] - _np(a)).max())
            assert d <= tol, (r, name, d, tol)
        for k in o["grads"]:
            assert np.array_equal(o["grads"][k], ret[0]["grads"][k]), k
            assert np.array_equal(o["params"][k], ret[0]["params"][k]), k


def test_sgd_step_two_ranks_on_one_device_matches_train_epoch():
    _run_step(2, "gloo")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_nccl_two_rank_training_step():
    _run_step(2, "nccl")
