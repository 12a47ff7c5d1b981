"""N>1 host logic on CPU: world_size-2 (and 3) gloo groups run dsmil_wsi_b200.sharded.sharded_forward
with an oracle-backed `ops` object standing in for the CUDA phases (test infrastructure), so the
exchange / merge / record layouts of the multi-GPU path are covered without GPUs."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import load_golden, rel_to_max
from oracle import dsmil_oracle as orc


class OracleShardOps:
    """numpy restatement of the five local steps with the library's record layouts
    (cand: idx[C] int64 | score[C] | qrow[C,128];  rec: m[C] | s[C] | Bp[C,Dv])."""

    def __init__(self, p: orc.Params):
        self.p = p.astype(np.float64)
        self.C, self.D = p.C, p.D
        self.cf = (p.C * 131 + 3) // 4 * 4          # records are padded to 4 floats (include/dsmil_b200.h)
        self.rf = (p.C * (2 + p.D) + 3) // 4 * 4

    def phase1(self, X, row_offset):
        p, C = self.p, self.C
        x = X.numpy().astype(np.float64)
        N = x.shape[0]
        cand = np.zeros(self.cf, np.float32)
        idx = cand[:2 * C].view(np.int64)
        if N == 0:
            idx[:] = np.iinfo(np.int64).max
            cand[2 * C:3 * C] = -np.inf
            return (torch.zeros(0, C, dtype=torch.float64), torch.zeros(0, 128, dtype=torch.float64), X.double(),
                    torch.from_numpy(cand))
        c = x @ p.Wi.T + p.bi
        Q, _ = orc.q_mlp(x, p)
        li = orc.critical_instances(c)
        idx[:] = li + row_offset
        cand[2 * C:3 * C] = c[li, np.arange(C)]
        cand[3 * C:3 * C + C * 128] = Q[li].reshape(-1)
        return torch.from_numpy(c), torch.from_numpy(Q), torch.from_numpy(x), torch.from_numpy(cand)

    def merge_candidates(self, cands, G):
        C = self.C
        recs = cands.numpy().reshape(G, self.cf)
        qmax = np.zeros((C, 128), np.float32)
        crit = np.zeros(C, np.int64)
        for k in range(C):
            best = None
            for g in range(G):
                gi = recs[g, :2 * C].view(np.int64)[k]
                if gi == np.iinfo(np.int64).max:
                    continue
                key = (-recs[g, 2 * C + k], gi, g)
                if best is None or key < best:
                    best = key
            crit[k] = best[1]
            qmax[k] = recs[best[2], 3 * C + k * 128: 3 * C + (k + 1) * 128]
        return torch.from_numpy(qmax), torch.from_numpy(crit)

    def phase2(self, Vv, Q, qmax):
        C, D = self.C, self.D
        rec = np.zeros(self.rf, np.float32)
        if Q.shape[0] == 0:
            rec[:C] = -np.inf
            return torch.zeros(0, C, dtype=torch.float64), torch.from_numpy(rec)
        L = (Q.numpy() @ qmax.numpy().astype(np.float64).T) / orc.SCALE_F32
        m = L.max(0)
        e = np.exp(L - m)
        rec[:C], rec[C:2 * C] = m, e.sum(0)
        rec[2 * C:2 * C + C * D] = (e.T @ Vv.numpy()).reshape(-1)
        return torch.from_numpy(L), torch.from_numpy(rec)

    def merge_partials(self, recs, G):
        C, D = self.C, self.D
        r = recs.numpy().reshape(G, self.rf).astype(np.float64)
        m, s, Bp = r[:, :C], r[:, C:2 * C], r[:, 2 * C:2 * C + C * D].reshape(G, C, D)
        M = m.max(0)
        w = np.where(np.isinf(m), 0.0, np.exp(m - M))
        out = np.zeros(self.rf, np.float32)
        out[:2 * C + C * D] = np.concatenate([M, (s * w).sum(0), (Bp * w[:, :, None]).sum(0).reshape(-1)])
        return torch.from_numpy(out)

    def phase3(self, rec, A):
        C, D, p = self.C, self.D, self.p
        r = rec.numpy().astype(np.float64)
        M, S, Bm = r[:C], r[C:2 * C], r[2 * C:2 * C + C * D].reshape(C, D) / r[C:2 * C, None]
        pred = p.Wf.reshape(C, -1) @ Bm.reshape(-1) + p.bf
        An = np.exp(A.numpy() - M) / S if A.shape[0] else A.numpy()
        return torch.from_numpy(An), torch.from_numpy(Bm.reshape(1, C, D)), torch.from_numpy(pred.reshape(1, C))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, name, N_override, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dsmil_wsi_b200.sharded import shard_bounds, sharded_forward
        g, p, X = load_golden(name)
        if N_override is not None:
            X = X[:N_override]
        lo, hi = shard_bounds(X.shape[0], world)[rank]
        ops = OracleShardOps(p)
        classes, pred, A, B, crit = sharded_forward(ops, torch.from_numpy(X[lo:hi]), lo, group=None)
        ret[rank] = dict(lo=lo, hi=hi, classes=classes.numpy(), pred=pred.numpy(), A=A.numpy(), B=B.numpy(),
                         crit=crit.numpy())
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,name,N_override", [(2, "shipped_tcga", None), (2, "musk_d166_n7", None),
                                                   (3, "lin_d512_c3", None), (2, "musk_d166_n7", 1)])
def test_sharded_forward_over_gloo(world, name, N_override):
    port = _free_port()
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, port, name, N_override, ret), nprocs=world, join=True)
    g, p, X = load_golden(name)
    if N_override is not None:
        X = X[:N_override]
    one = orc.forward(X, p)
    for r in range(world):
        o = ret[r]
        assert np.array_equal(o["crit"], one.idx)                        # replicated, identical on all ranks
        assert rel_to_max(o["pred"], one.prediction_bag) < 2e-6
        assert rel_to_max(o["B"], one.B) < 2e-6
        if o["hi"] > o["lo"]:
            assert rel_to_max(o["classes"], one.classes[o["lo"]:o["hi"]]) < 1e-12
            assert rel_to_max(o["A"], one.A[o["lo"]:o["hi"]]) < 2e-6      # records travel as fp32
    assert sum(ret[r]["hi"] - ret[r]["lo"] for r in range(world)) == X.shape[0]


def test_shard_bounds_cover_and_balance():
    from dsmil_wsi_b200.sharded import shard_bounds
    for N, G in [(10, 3), (7, 8), (100000, 8), (0, 2)]:
        b = shard_bounds(N, G)
        assert b[0][0] == 0 and b[-1][1] == N and all(b[i][1] == b[i + 1][0] for i in range(G - 1))
        sizes = [hi - lo for lo, hi in b]
        assert max(sizes) - min(sizes) <= 1
    assert shard_bounds(10, 3) == list(orc.shard_bounds(10, 3))


# ---- sharded training step: forward + the three-reduction backward through autograd, over gloo -----------------


class OracleTrainOps(OracleShardOps):
    """+ the training phase 1 and the three backward phases, numpy fp64 with fp32 parameter gradients."""

    def phase1_train(self, X, row_offset):
        classes, Q, x, cand = self.phase1(X, row_offset)
        H1 = None
        if self.p.nonlinear:
            H1 = torch.from_numpy(orc.q_mlp(x.numpy(), self.p)[1]) if x.shape[0] else torch.zeros(0, 128, dtype=torch.float64)
        return classes, Q, H1, x, cand

    def bwd1(self, X, A, B, d_classes, d_pred):
        p, C, D = self.p, self.C, self.D
        x, a = X.numpy().astype(np.float64), A.numpy().astype(np.float64)
        dp = np.zeros(C) if d_pred is None else d_pred.numpy().astype(np.float64).reshape(C)
        dc = np.zeros((x.shape[0], C)) if d_classes is None else d_classes.numpy().astype(np.float64)
        Bm = B.numpy().astype(np.float64).reshape(C, D)
        dB = (p.Wf.reshape(C, -1).T @ dp).reshape(C, D)
        dA = x @ dB.T
        f32 = lambda v: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32))
        return (torch.from_numpy(dA), torch.from_numpy((a * dA).sum(0)), f32(dc.T @ x), f32(dc.sum(0)),
                f32(np.outer(dp, Bm.reshape(-1)).reshape(C, C, D)), f32(dp))

    def bwd2(self, A, dA, t, Q):
        dL = A.numpy() * (dA.numpy() - t.numpy()) / np.float64(orc.SCALE_F32)
        return torch.from_numpy(dL), torch.from_numpy(dL.T @ Q.numpy())

    def bwd3(self, X, row_offset, Q, H1, dL, dqm, qmax, crit):
        p, C = self.p, self.C
        x, q = X.numpy().astype(np.float64), Q.numpy()
        dQ = dL.numpy() @ qmax.numpy().astype(np.float64)
        for k in range(C):
            loc = int(crit[k]) - row_offset
            if 0 <= loc < x.shape[0]:
                dQ[loc] += dqm.numpy()[k]
        f32 = lambda v: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32))
        if p.nonlinear:
            h1 = H1.numpy()
            dz2 = dQ * (1 - q * q)
            dz1 = (dz2 @ p.W2) * (h1 > 0)
            return f32(dz1.T @ x), f32(dz1.sum(0)), f32(dz2.T @ h1), f32(dz2.sum(0))
        return f32(dQ.T @ x), f32(dQ.sum(0)), None, None


def _train_worker(rank, world, port, name, N_override, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from helpers import build_net
        from dsmil_wsi_b200.sharded import shard_bounds, sharded_caller_loss, sharded_milnet_forward
        g, p, X = load_golden(name)
        if N_override is not None:
            X = X[:N_override]
        lo, hi = shard_bounds(X.shape[0], world)[rank]
        net = build_net(p, device="cpu")
        y = torch.from_numpy(np.asarray(g["y"], np.float32).reshape(-1))
        counts = {"all_gather": 0, "sum": 0, "max": 0}
        real_gather, real_reduce = dist.all_gather_into_tensor, dist.all_reduce

        def gather(*a, **k):
            counts["all_gather"] += 1
            return real_gather(*a, **k)

        def reduce(t, op=dist.ReduceOp.SUM, **k):
            counts["max" if op == dist.ReduceOp.MAX else "sum"] += 1
            return real_reduce(t, op=op, **k)
        dist.all_gather_into_tensor, dist.all_reduce = gather, reduce
        classes, pred, A, B, crit = sharded_milnet_forward(net, torch.from_numpy(X[lo:hi]), lo, ops=OracleTrainOps(p))
        loss = sharded_caller_loss(classes, pred, crit, lo, y, torch.nn.BCEWithLogitsLoss())
        loss.backward()
        ret[rank] = dict(loss=float(loss.detach()), counts=counts,
                         grads={k: v.grad.numpy().copy() for k, v in net.named_parameters() if v.grad is not None})
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,name,N_override", [(2, "shipped_tcga", None), (3, "lin_d512_c3", None),
                                                   (2, "musk_d166_n7", None), (2, "musk_d166_n7", 1)])
def test_sharded_training_step_over_gloo(world, name, N_override):
    """Every rank ends with the single-device gradients of the callers' loss (train_tcga.py:67-72), and the same
    loss value: two all-gathers in the forward, three all-reduces in the reverse pass, one all-reduce(max) in the
    loss."""
    from helpers import grad_name
    port = _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_train_worker, args=(world, port, name, N_override, ret), nprocs=world, join=True)
    g, p, X = load_golden(name)
    if N_override is not None:
        X = X[:N_override]
    one = orc.forward(X, p)
    y = np.asarray(g["y"], np.float64).reshape(-1)
    loss, d_cls, d_pred = orc.caller_loss_grads(one, y)
    ref = orc.backward(X, p, one, d_cls, d_pred)
    for r in range(world):
        assert ret[r]["counts"] == {"all_gather": 2, "sum": 3, "max": 1}, ret[r]["counts"]
        assert abs(ret[r]["loss"] - loss) < 2e-6
        grads = ret[r]["grads"]
        for short, want in ref.items():
            got = grads[grad_name(short, p.nonlinear)]
            # the forward's records travel as fp32 (A to ~2e-6); the softmax backward amplifies that a few times
            assert got.shape == want.shape
            if np.abs(want).max() < 1e-12:      # N == 1: A == 1, dL == 0 exactly, the q-branch gets no gradient
                assert np.abs(got).max() < 1e-7, (r, short)
            else:
                assert rel_to_max(got, want) < 5e-5, (r, short)
        for k in grads:                                              # replicated bit for bit
            assert np.array_equal(grads[k], ret[0]["grads"][k]), k


@pytest.mark.parametrize("name,G", [("shipped_tcga", 3), ("lin_d512_c3", 4), ("musk_d166_n7", 8), ("musk_d166_n1", 2)])
def test_virtual_sharded_train_step_bags_one_bag_host_logic(name, G):
    """The single-device validation helper (reductions as local sums) with the oracle-backed ops: same indexing
    and record plumbing the GPU test (tests/test_zz_shard_backward_gpu.py) relies on."""
    from dsmil_wsi_b200.sharded import PerBagShardOps, virtual_sharded_train_step_bags
    g, p, X = load_golden(name)
    one = orc.forward(X, p)
    y = np.asarray(g["y"], np.float64).reshape(-1)
    _, d_cls, d_pred = orc.caller_loss_grads(one, y)
    ref = orc.backward(X, p, one, d_cls, d_pred)
    grads_of = lambda classes, pred, crit: (torch.from_numpy(d_cls), torch.from_numpy(d_pred))
    outs, grads = virtual_sharded_train_step_bags(lambda: PerBagShardOps(OracleTrainOps(p)), [torch.from_numpy(X)], G,
                                                  grads_of)
    assert np.array_equal(outs[4][0].numpy(), one.idx) and rel_to_max(outs[2].numpy(), one.A) < 2e-6
    for short, got in zip(["Wi", "bi", "W1", "b1", "W2", "b2", "Wf", "bf"], grads):
        if got is None:
            assert not p.nonlinear and short in ("W2", "b2")
        elif np.abs(ref[short]).max() < 1e-12:
            assert np.abs(got.numpy()).max() < 1e-7
        else:
            assert rel_to_max(got.numpy(), ref[short]) < 5e-5, short


# ---- a batch of row-sharded bags: two collectives per STEP (records packed per bag) ------------------------------


def _bags_worker(rank, world, port, sizes, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dsmil_wsi_b200.sharded import shard_bounds, sharded_forward_bags
        p = orc.random_params(64, 3, 21, scale=1.5)
        ops = OracleShardOps(p)
        xs, offs = [], []
        for i, n in enumerate(sizes):
            X = orc.synthetic_bag(n, 64, 300 + i, "normal")
            lo, hi = shard_bounds(n, world)[rank]
            xs.append(torch.from_numpy(X[lo:hi]))
            offs.append(lo)
        n_coll = {"n": 0}
        real = dist.all_gather_into_tensor

        def counting(*a, **k):
            n_coll["n"] += 1
            return real(*a, **k)
        dist.all_gather_into_tensor = counting
        outs = sharded_forward_bags(ops, xs, offs)
        ret[rank] = dict(collectives=n_coll["n"], offs=offs,
                         outs=[tuple(t.numpy() for t in o) for o in outs])
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,sizes", [(2, [37, 5, 120]), (3, [2, 64, 9, 1])])
def test_sharded_bags_two_collectives_per_step(world, sizes):
    port = _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_bags_worker, args=(world, port, sizes, ret), nprocs=world, join=True)
    p = orc.random_params(64, 3, 21, scale=1.5)
    for r in range(world):
        assert ret[r]["collectives"] == 2                      # not two per bag
        for i, n in enumerate(sizes):
            one = orc.forward(orc.synthetic_bag(n, 64, 300 + i, "normal"), p)
            classes, pred, A, B, crit = ret[r]["outs"][i]
            lo = ret[r]["offs"][i]
            assert np.array_equal(crit, one.idx)
            assert rel_to_max(pred, one.prediction_bag) < 2e-6 and rel_to_max(B, one.B) < 2e-6
            if classes.shape[0]:
                assert rel_to_max(classes, one.classes[lo:lo + classes.shape[0]]) < 1e-12
                assert rel_to_max(A, one.A[lo:lo + A.shape[0]]) < 2e-6
