"""The row-sharded training step as one CUDA graph, on the device: every capture-safe dsmil_shard_*_dev call against its
eager dsmil_shard_* counterpart, bit for bit, with G virtual ranks on one GPU (one workspace per logical rank,
concatenation and sums as the collectives); one capture of that virtual step replayed over four ragged batches against
virtual_sharded_train_step_bags; and ShardedTrainStepGraph over NCCL (a spawned worker, so this process keeps no
process group) against the eager sharded step, TrainStepGraph and a refused batch."""
import copy
import os
import socket

import pytest
import torch

from conftest import rel_to_max
from helpers import build_net
from oracle import dsmil_oracle as orc
from dsmil_wsi_b200 import _lib
from dsmil_wsi_b200.sharded import (CudaShardBagDevOps, CudaShardBagOps, milnet_params, shard_bounds,
                                    virtual_sharded_train_step_bags)

pytestmark = pytest.mark.gpu

TOL = 5e-4          # DESIGN.md §3: gradients, rel-to-max, bags below 10 000 rows


class Ranks:
    """Static buffers of G logical ranks for nb bags: rank r's slots [nb, cap, D], Ns, row offsets and status."""

    def __init__(self, G, nb, max_N, D):
        self.G, self.nb = G, nb
        self.cap = -(-max_N // G)
        self.slots = [torch.zeros(nb, self.cap, D, device="cuda") for _ in range(G)]
        self.Ns = [torch.ones(nb, dtype=torch.int64, device="cuda") for _ in range(G)]
        self.offs = [torch.zeros(nb, dtype=torch.int64, device="cuda") for _ in range(G)]
        self.status = [torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(G)]

    def load(self, Xs, extra_offset=0):
        """Rank r gets shard_bounds' rows of every bag; returns each rank's (local bags, offsets) for the eager ops."""
        eager = []
        for r in range(self.G):
            xs, offs = [], []
            for b, X in enumerate(Xs):
                lo, hi = shard_bounds(int(X.shape[0]), self.G)[r]
                self.slots[r][b, :hi - lo].copy_(X[lo:hi])
                self.Ns[r][b].fill_(hi - lo)
                self.offs[r][b].fill_(lo + extra_offset)
                xs.append(self.slots[r][b, :hi - lo])
                offs.append(lo + extra_offset)
            eager.append((xs, offs))
        return eager


def _upstream(classes, pred):
    """Upstream gradients that do not depend on the packing: elementwise in the outputs."""
    return torch.tanh(classes), torch.tanh(pred)


def _virtual_step(ops, begins, G, record=None):
    """The sharded training step over G logical ranks: ops[r].begin(*begins[r]), the all-gathers as concatenation,
    the all-reduces as sums.  `record(name, r, tensor)` sees every call's outputs as they leave the call."""
    rec = record or (lambda *a: None)
    xs = [o.begin(*b) for o, b in zip(ops, begins)]
    p1 = [o.phase1_train() for o in ops]
    for r, out in enumerate(p1):
        for n, t in zip(("classes", "Q", "H1", "cand"), out):
            rec(n, r, t)
    cands = torch.cat([p[3].reshape(-1) for p in p1])
    p2 = [o.phase2_train(p[1], cands, G) for o, p in zip(ops, p1)]
    for r, out in enumerate(p2):
        for n, t in zip(("logits", "crit", "qmax", "recs"), out):
            rec(n, r, t)
    recs = torch.cat([p[3].reshape(-1) for p in p2])
    p3 = [o.phase3_train(recs, G, p[0]) for o, p in zip(ops, p2)]
    for r, out in enumerate(p3):
        for n, t in zip(("A", "B", "pred"), out):
            rec(n, r, t)
    up = [_upstream(p[0], q[2]) for p, q in zip(p1, p3)]
    b1 = [o.bwd1(x, q[0], q[1], *u) for o, x, q, u in zip(ops, xs, p3, up)]
    for r, out in enumerate(b1):
        for n, t in zip(("dA", "t", "gWi", "gbi", "gWf", "gbf"), out):
            rec(n, r, t)
    t = torch.stack([b[1] for b in b1]).sum(0)
    b2 = [o.bwd2(x, q[0], b[0], t, p[1]) for o, x, q, b, p in zip(ops, xs, p3, b1, p1)]
    for r, out in enumerate(b2):
        for n, t_ in zip(("dL", "dqm"), out):
            rec(n, r, t_)
    dqm = torch.stack([b[1] for b in b2]).sum(0)
    b3 = [o.bwd3(x, b[1], p[1], p[2], c[0], dqm, q[2], q[1])
          for o, x, b, p, c, q in zip(ops, xs, begins, p1, b2, p2)]
    for r, out in enumerate(b3):
        for n, t_ in zip(("gW1", "gb1", "gW2", "gb2"), out):
            rec(n, r, t_)
    tot = lambda ts: torch.stack(list(ts)).sum(0)
    grads = (tot(b[2] for b in b1), tot(b[3] for b in b1), *(tot(b[i] for b in b3) for i in range(4)), b1[0][4],
             b1[0][5])
    return p3[0][2], p3[0][1], p2[0][1], grads


PER_ROW = {"classes", "Q", "H1", "logits", "A", "dA", "dL"}


def _recorder(store, rows, C_, D):
    """Copies of every output: the live rows of a per-row output (rows[r] on rank r), and the records without the
    padding that rounds them to 4 floats (never written)."""
    used = {"cand": C_ * (3 + 128), "recs": C_ * (2 + D)}

    def rec(name, r, t):
        t = t[:rows[r]] if name in PER_ROW else t
        store[(name, r)] = (t[:, :used[name]] if name in used else t).clone()
    return rec


@pytest.mark.parametrize("D,C_", [(512, 2), (1024, 4)])
@pytest.mark.parametrize("G,Ns,extra", [(1, [1, 127, 128, 129, 3000], 1000), (1, [3, 1, 2, 1, 5], 7),
                                        (2, [3, 127, 128, 129, 3000], 0), (3, [3, 4, 5, 3, 7], 0),
                                        (3, [3000, 129, 3, 128, 127], 0)])
def test_each_dev_call_matches_its_eager_call_bit_for_bit(D, C_, G, Ns, extra):
    net = build_net(orc.random_params(D, C_, seed=D + C_ + G))
    params = milnet_params(net)
    R = Ranks(G, len(Ns), 3000, D)
    g = torch.Generator(device="cuda").manual_seed(G + len(Ns))
    Xs = [torch.rand(n, D, device="cuda", generator=g) for n in Ns]
    eager_in = R.load(Xs, extra)
    rows = [sum(int(x.shape[0]) for x in xs) for xs, _ in eager_in]
    want, got = {}, {}
    ew = _virtual_step([CudaShardBagOps(params) for _ in range(G)], eager_in, G, _recorder(want, rows, C_, D))
    dev = [CudaShardBagDevOps(params, R.Ns[r], R.status[r]) for r in range(G)]
    gw = _virtual_step(dev, [([R.slots[r]], R.offs[r]) for r in range(G)], G, _recorder(got, rows, C_, D))
    assert want.keys() == got.keys()
    for k, v in want.items():
        assert torch.equal(got[k], v), (k, float((got[k].float() - v.float()).abs().max()))
    for a, b in zip(gw[:3] + gw[3], ew[:3] + ew[3]):
        assert torch.equal(a, b)
    assert all(int(s) == 0 for s in R.status)


GRAPH_BATCHES = [[3000, 129, 3, 128, 127], [3, 4, 5, 3, 7], [1500, 2999, 3000, 64, 300], [7, 3000, 3, 1000, 17]]


@pytest.mark.parametrize("G", [2, 3])
def test_one_capture_of_the_virtual_step_replays_every_batch(G):
    D, C_, nb = 512, 2, 5
    net = build_net(orc.random_params(D, C_, seed=11 + G))
    params = milnet_params(net)
    R = Ranks(G, nb, 3000, D)
    g = torch.Generator(device="cuda").manual_seed(G)
    batches = [[torch.rand(n, D, device="cuda", generator=g) for n in Ns] for Ns in GRAPH_BATCHES]
    R.load(batches[0])
    dev = [CudaShardBagDevOps(params, R.Ns[r], R.status[r]) for r in range(G)]
    begins = [([R.slots[r]], R.offs[r]) for r in range(G)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _virtual_step(dev, begins, G)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = _virtual_step(dev, begins, G)
    for Xs in batches:
        R.load(Xs)
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        graph.replay()
        torch.cuda.synchronize()
        assert _lib.launch_count() == n0
        Ns = [int(x.shape[0]) for x in Xs]

        def loss_grads(classes, pred, crit):
            return _upstream(classes, pred)
        (_, pred, _, B, crit), grads = virtual_sharded_train_step_bags(lambda: CudaShardBagOps(params), Xs, G,
                                                                       loss_grads)
        assert torch.equal(outs[0], pred) and torch.equal(outs[1], B) and torch.equal(outs[2], crit), Ns
        for a, b in zip(outs[3], grads):
            assert torch.equal(a, b), Ns
    assert all(int(s) == 0 for s in R.status)


# ---- ShardedTrainStepGraph over NCCL, in spawned workers --------------------------------------------------------------
STEP_D, STEP_C, STEP_NB, STEP_MAXR = 512, 2, 4, 3000
STEP_BATCHES = [[3000, 1, 129, 700], [5, 2999, 128, 3], [64, 65, 3000, 1000]]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _spawn(fn, world, *args):
    import torch.multiprocessing as mp
    mp.spawn(fn, args=(world, _free_port(), *args), nprocs=world, join=True)


def _init(rank, world, port):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))


def _optimizer(kind, net):
    if kind == "sgd":
        return torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9)
    return torch.optim.Adam(net.parameters(), lr=1e-3, betas=(0.5, 0.9), weight_decay=1e-3, capturable=True)


def _problem(seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    bags = [[torch.rand(n, STEP_D, device="cuda", generator=g) for n in Ns] for Ns in STEP_BATCHES]
    labels = [(torch.rand(STEP_NB, STEP_C, device="cuda", generator=g) > 0.5).float() for _ in STEP_BATCHES]
    return bags, labels


def _fill(graph, bags, labels, rank, world):
    """This rank's rows of every bag into the graph's static buffers; returns them for the eager step."""
    xs, offs = [], []
    for b, X in enumerate(bags):
        lo, hi = shard_bounds(int(X.shape[0]), world)[rank]
        graph.slots[b, :hi - lo].copy_(X[lo:hi])
        graph.Ns[b].fill_(hi - lo)
        graph.row_offsets[b].fill_(lo)
        xs.append(X[lo:hi])
        offs.append(lo)
    graph.labels.copy_(labels)
    return xs, offs


def _state(net, opt):
    ps = [p.detach().clone() for p in net.parameters()]
    st = [v.clone() for p in net.parameters() for v in opt.state.get(p, {}).values() if torch.is_tensor(v)]
    return ps + st


def _graph_worker(rank, world, port, kind):
    import torch.distributed as dist
    _init(rank, world, port)
    try:
        from dsmil_wsi_b200.sharded import sharded_caller_loss_bags, sharded_milnet_forward_bags
        from dsmil_wsi_b200.train_graph import ShardedTrainStepGraph, TrainStepGraph
        torch.manual_seed(0)
        base = build_net(orc.random_params(STEP_D, STEP_C, seed=21), device=f"cuda:{rank}").train()
        net_g, net_e, net_1 = copy.deepcopy(base), copy.deepcopy(base), copy.deepcopy(base)
        opt_g, opt_e, opt_1 = _optimizer(kind, net_g), _optimizer(kind, net_e), _optimizer(kind, net_1)
        bce = torch.nn.BCEWithLogitsLoss()
        graph = ShardedTrainStepGraph(net_g, bce, opt_g, STEP_NB, STEP_MAXR)
        single = TrainStepGraph(net_1, bce, opt_1, STEP_NB, STEP_MAXR) if world == 1 else None
        bags, labels = _problem(5)
        for i, (Xs, y) in enumerate(zip(bags, labels)):
            xs, offs = _fill(graph, Xs, y, rank, world)
            loss_g = graph.step()
            opt_e.zero_grad()
            classes, pred, _, _, crit = sharded_milnet_forward_bags(net_e, xs, offs)
            loss_e = sharded_caller_loss_bags(classes, pred, crit, offs, y, bce, Ns=[int(x.shape[0]) for x in xs])
            loss_e.backward()
            opt_e.step()
            torch.cuda.synchronize()
            assert torch.equal(loss_g, loss_e.detach()), (i, float(loss_g), float(loss_e))
            for (name, a), b in zip(net_g.named_parameters(), net_e.parameters()):
                assert torch.equal(a.grad, b.grad), (i, name, float((a.grad - b.grad).abs().max()))
                assert torch.equal(a, b), (i, name)
            if single is not None:
                for b, X in enumerate(Xs):
                    single.slots[b, :X.shape[0]].copy_(X)
                    single.Ns[b].fill_(int(X.shape[0]))
                single.labels.copy_(y)
                single.step()
                torch.cuda.synchronize()
                for (name, a), b in zip(net_g.named_parameters(), net_1.parameters()):
                    d = rel_to_max(a.grad.cpu().numpy(), b.grad.cpu().numpy())
                    assert d <= TOL, (i, name, d)
                with torch.no_grad():                          # keep the single-device replica on the sharded path
                    for a, b in zip(net_g.parameters(), net_1.parameters()):
                        b.copy_(a)
                    for a, b in zip(net_g.parameters(), net_1.parameters()):
                        for k, v in opt_g.state.get(a, {}).items():
                            if torch.is_tensor(v):
                                opt_1.state[b][k].copy_(v)
        assert int(graph.status) == 0
        # refused batches: a local N of 0 on rank 0, then one above max_rows on the last rank
        for bad_rank, bad_n in ((0, 0), (world - 1, STEP_MAXR + 1)):
            before = _state(net_g, opt_g)
            _fill(graph, bags[0], labels[0], rank, world)
            if rank == bad_rank:
                graph.Ns[2].fill_(bad_n)
            loss = graph.step()
            torch.cuda.synchronize()
            assert torch.isnan(loss), (bad_rank, bad_n)
            assert (int(graph.status) == 3) == (rank == bad_rank), int(graph.status)
            for a, b in zip(_state(net_g, opt_g), before):
                assert torch.equal(a, b), (bad_rank, bad_n)
            graph.status.zero_()
        # the next accepted batch steps exactly as if the refused ones had not been fed
        xs, offs = _fill(graph, bags[1], labels[1], rank, world)
        loss_g = graph.step()
        opt_e.zero_grad()
        classes, pred, _, _, crit = sharded_milnet_forward_bags(net_e, xs, offs)
        loss_e = sharded_caller_loss_bags(classes, pred, crit, offs, labels[1], bce, Ns=[int(x.shape[0]) for x in xs])
        loss_e.backward()
        opt_e.step()
        torch.cuda.synchronize()
        assert torch.equal(loss_g, loss_e.detach())
        for a, b in zip(net_g.parameters(), net_e.parameters()):
            assert torch.equal(a, b)
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_sharded_graph_is_the_eager_sharded_step_one_rank(kind):
    _spawn(_graph_worker, 1, kind)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_sharded_graph_is_the_eager_sharded_step_two_ranks_nccl():
    _spawn(_graph_worker, 2, "adam")
