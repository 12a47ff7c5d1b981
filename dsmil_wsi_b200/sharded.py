"""Row-sharded forward of ONE giant bag over the ranks of a torch.distributed group
(SURVEY §8e / Appendix A.3; north_star: "patches of one giant bag shard across the 8 GPUs ...
NCCL only for the per-class critical-instance max and the attention-weighted partial sums").

One process per GPU.  Rank r owns the contiguous rows [offset_r, offset_r + N_r).  Per forward
there are exactly two data-path collectives, both all-gathers of a few KB:
    exchange 1: candidate record  (global idx, score, q row) per class     C*131 floats / rank
    exchange 2: partial record    (m, s, unnormalised partial B) per class C*(2+D) floats / rank
Everything else is local: phase1/2/3 of the C ABI (include/dsmil_b200.h).  classes and A stay
sharded; prediction_bag, B and the critical indices are replicated.

The host logic is written once, for a batch of bags, over an ops object with the interface of CudaShardBagOps.
CudaShardBagOps runs the batched ABI (dsmil_shard_bags_*): three library calls and two all-gathers per forward step,
and, for training (sharded_milnet_forward_bags + sharded_caller_loss_bags), three more calls and four more collectives
(one all-reduce(max) in the loss, three all-reduce(sum) in the backward), whatever the number of bags.
PerBagShardOps gives that interface to a one-bag ops object (CudaShardOps: the one-bag ABI, dsmil_shard_phase1/2/3,
which also serves the shapes the batched ABI refuses) by running it one bag at a time.  CudaShardBagDevOps gives the
training interface to the capture-safe calls (dsmil_shard_*_dev), so train_graph.ShardedTrainStepGraph records the same
host logic, collectives included, as one CUDA graph.  The one-bag entry points
(sharded_forward, sharded_milnet_forward, sharded_caller_loss) are the batch step with nb = 1 over the one-bag ABI.
The ops object is what the CPU tests replace: they run the same exchange/merge logic over gloo with an oracle-backed
stand-in (the product default, CudaShardOps, has no fallback).
"""
from __future__ import annotations

import ctypes as C
from itertools import accumulate
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib
from . import functional as Fn
from .modules import milnet_params


def shard_bounds(N: int, G: int) -> List[Tuple[int, int]]:
    """Contiguous row blocks; the first N % G ranks get one extra row."""
    base, rem = divmod(N, G)
    out, lo = [], 0
    for r in range(G):
        hi = lo + base + (1 if r < rem else 0)
        out.append((lo, hi))
        lo = hi
    return out


def _bwd1_shares(ops):
    """This rank's gWi, gbi, gWf and gbf: the parameter gradients of a backward phase 1."""
    P = ops.P
    return ops.new(P.C, P.D), ops.new(P.C), ops.new(P.C, P.C, P.D), ops.new(P.C)


def _bwd3_shares(ops):
    """This rank's gW1, gb1, gW2 and gb2 (None for a linear q): the parameter gradients of a backward phase 3."""
    P, Q = ops.P, Fn.Q_DIM
    return (ops.new(Q, P.D), ops.new(Q), ops.new(Q, Q) if P.nonlinear else None,
            ops.new(Q) if P.nonlinear else None)


def _upstream(d_classes, d_pred):
    """The upstream gradients as a backward phase 1 reads them: contiguous float32, or None."""
    return tuple(None if d is None else d.to(torch.float32).contiguous() for d in (d_classes, d_pred))


class CudaShardOps:
    """The five local steps on the current CUDA device through libdsmil_b200.so."""

    def __init__(self, params: Sequence[Optional[torch.Tensor]]):
        self.lib = _lib.load()
        self.P = Fn.ParamPack(*params)
        self.device = self.P.device

    # sizes of the exchanged records (floats)
    def cand_floats(self) -> int:
        return int(self.lib.dsmil_cand_floats(self.P.C))

    def rec_floats(self) -> int:
        return int(self.lib.dsmil_rec_floats(self.P.C, self.P.D))

    def new(self, *shape, dtype=torch.float32):
        return torch.empty(*shape, dtype=dtype, device=self.device)

    def _ws(self, N):
        return Fn._workspace(self.lib.dsmil_shard_workspace_bytes(self.P.ref, N), self.device)

    def _phase1(self, X: torch.Tensor, row_offset: int, train: bool):
        """dsmil_shard_phase1: (classes, Q, H1, V or X, cand).  `train` keeps H1 for the reverse pass (identity v
        only); otherwise a passing_v model gets its V."""
        P, N = self.P, int(X.shape[0])
        if train and P.passing_v:
            raise NotImplementedError("sharded training: identity v only")
        X = Fn._check_feats(X, P.D) if N > 0 else X
        with torch.cuda.device(self.device):
            classes, Q = self.new(N, P.C), self.new(N, Fn.Q_DIM)
            H1 = self.new(N, Fn.Q_DIM) if train and P.nonlinear else None
            V = self.new(N, P.D) if P.passing_v else None
            cand = self.new(self.cand_floats())
            ws = self._ws(N)
            rc = self.lib.dsmil_shard_phase1(P.ref, Fn._ptr(X), None, None, N, int(row_offset), Fn._ptr(classes),
                                             Fn._ptr(Q), Fn._ptr(H1), Fn._ptr(V), Fn._ptr(cand), Fn._ptr(ws),
                                             ws.numel(), Fn._stream())
            _lib.check(rc, "dsmil_shard_phase1")
        return classes, Q, H1, (X if V is None else V), cand

    def phase1(self, X: torch.Tensor, row_offset: int):
        classes, Q, _, Vv, cand = self._phase1(X, row_offset, train=False)
        return classes, Q, Vv, cand

    def merge_candidates(self, cands: torch.Tensor, G: int):
        with torch.cuda.device(self.device):
            qmax = self.new(self.P.C, Fn.Q_DIM)
            crit = self.new(self.P.C, dtype=torch.int64)
            rc = self.lib.dsmil_shard_merge_candidates(self.P.C, Fn._ptr(cands), G, Fn._ptr(qmax), Fn._ptr(crit),
                                                       Fn._stream())
            _lib.check(rc, "dsmil_shard_merge_candidates")
        return qmax, crit

    def phase2(self, Vv: torch.Tensor, Q: torch.Tensor, qmax: torch.Tensor):
        P, N = self.P, int(Q.shape[0])
        with torch.cuda.device(self.device):
            A = self.new(N, P.C)
            rec = self.new(self.rec_floats())
            ws = self._ws(N)
            rc = self.lib.dsmil_shard_phase2(P.ref, Fn._ptr(Vv), Fn._ptr(Q), N, Fn._ptr(qmax), Fn._ptr(A),
                                             Fn._ptr(rec), Fn._ptr(ws), ws.numel(), Fn._stream())
            _lib.check(rc, "dsmil_shard_phase2")
        return A, rec

    def merge_partials(self, recs: torch.Tensor, G: int):
        with torch.cuda.device(self.device):
            out = self.new(self.rec_floats())
            rc = self.lib.dsmil_shard_merge_partials(self.P.C, self.P.D, Fn._ptr(recs), G, Fn._ptr(out), Fn._stream())
            _lib.check(rc, "dsmil_shard_merge_partials")
        return out

    def phase3(self, rec: torch.Tensor, A: torch.Tensor):
        P, N = self.P, int(A.shape[0])
        with torch.cuda.device(self.device):
            B, pred = self.new(1, P.C, P.D), self.new(1, P.C)
            rc = self.lib.dsmil_shard_phase3(P.ref, N, Fn._ptr(rec), Fn._ptr(A), Fn._ptr(B), Fn._ptr(pred),
                                             Fn._stream())
            _lib.check(rc, "dsmil_shard_phase3")
        return A, B, pred


    # ---- training: phase 1 that keeps H1, and the three backward phases (dsmil_shard_backward_*) ----
    def phase1_train(self, X: torch.Tensor, row_offset: int):
        """phase1 with Q and H1 kept row-major for the reverse pass (identity v only): (classes, Q, H1, X, cand)."""
        return self._phase1(X, row_offset, train=True)

    def _bws(self, N):
        return Fn._workspace(self.lib.dsmil_backward_workspace_bytes(self.P.ref, N, 0), self.device)

    def bwd1(self, X, A, B, d_classes, d_pred):
        P, N = self.P, int(X.shape[0])
        with torch.cuda.device(self.device):
            dA, t = self.new(N, P.C), self.new(P.C)
            gWi, gbi, gWf, gbf = _bwd1_shares(self)
            dc, dp = _upstream(d_classes, d_pred)
            ws = self._bws(N)
            rc = self.lib.dsmil_shard_backward_phase1(P.ref, Fn._ptr(X), N, Fn._ptr(A), Fn._ptr(B.contiguous()),
                                                      Fn._ptr(dc), Fn._ptr(dp), Fn._ptr(dA), Fn._ptr(t), Fn._ptr(gWi),
                                                      Fn._ptr(gbi), Fn._ptr(gWf), Fn._ptr(gbf), Fn._ptr(ws), ws.numel(),
                                                      Fn._stream())
            _lib.check(rc, "dsmil_shard_backward_phase1")
        return dA, t, gWi, gbi, gWf, gbf

    def bwd2(self, A, dA, t, Q):
        P, N = self.P, int(A.shape[0])
        with torch.cuda.device(self.device):
            dqm = self.new(P.C, Fn.Q_DIM)
            ws = self._bws(N)
            rc = self.lib.dsmil_shard_backward_phase2(P.ref, N, Fn._ptr(A), Fn._ptr(dA), Fn._ptr(t.contiguous()),
                                                      Fn._ptr(Q), Fn._ptr(dqm), Fn._ptr(ws), ws.numel(), Fn._stream())
            _lib.check(rc, "dsmil_shard_backward_phase2")
        return dA, dqm                                    # dA now holds dL

    def bwd3(self, X, row_offset, Q, H1, dL, dqm, qmax, crit):
        P, N = self.P, int(X.shape[0])
        with torch.cuda.device(self.device):
            gW1, gb1, gW2, gb2 = _bwd3_shares(self)
            ws = self._bws(N)
            rc = self.lib.dsmil_shard_backward_phase3(P.ref, Fn._ptr(X), N, int(row_offset), Fn._ptr(Q), Fn._ptr(H1),
                                                      Fn._ptr(dL), Fn._ptr(dqm.contiguous()), Fn._ptr(qmax.contiguous()),
                                                      Fn._ptr(crit.contiguous()), Fn._ptr(gW1), Fn._ptr(gb1),
                                                      Fn._ptr(gW2), Fn._ptr(gb2), Fn._ptr(ws), ws.numel(), Fn._stream())
            _lib.check(rc, "dsmil_shard_backward_phase3")
        return gW1, gb1, gW2, gb2


class CudaShardBagOps:
    """Batched form of the three local phases (dsmil_shard_bags_*): one library call per phase for ALL bags of
    a step, tensor-core path.  The workspace lives across the phases of one step."""

    def __init__(self, params: Sequence[Optional[torch.Tensor]]):
        self.lib = _lib.load()
        self.P = Fn.ParamPack(*params)
        self.device = self.P.device
        if not self.lib.dsmil_shard_bags_supported(self.P.ref):
            raise RuntimeError("dsmil_b200: this (D, C, q/v variant) has no batched sharded path; use CudaShardOps")

    @staticmethod
    def supported(params) -> bool:
        P = Fn.ParamPack(*params)
        return bool(_lib.load().dsmil_shard_bags_supported(P.ref))

    def begin(self, X_locals: Sequence[torch.Tensor], row_offsets: Sequence[int]):
        P = self.P
        self.xs = [Fn._check_feats(x, P.D) for x in X_locals]
        self.nb = len(self.xs)
        self.Ns = [int(x.shape[0]) for x in self.xs]
        if min(self.Ns) < 1:
            raise ValueError("sharded batches need at least one local row per bag on every rank")
        self.c_N = (C.c_int64 * self.nb)(*self.Ns)
        self.c_X = (C.c_void_p * self.nb)(*[x.data_ptr() for x in self.xs])
        self.c_off = (C.c_int64 * self.nb)(*[int(o) for o in row_offsets])
        self.total = sum(self.Ns)
        key = (tuple(self.Ns), tuple(x.data_ptr() for x in self.xs), tuple(int(o) for o in row_offsets))
        if getattr(self, "_ws_key", None) != key:       # same step again (serving loop / graph capture): keep the workspace
            with torch.cuda.device(self.device):
                self.ws = Fn._workspace(self.lib.dsmil_shard_bags_workspace_bytes(P.ref, self.c_N, self.nb), self.device)
            self._ws_key = key
        self.cand_f = int(self.lib.dsmil_cand_floats(P.C))
        self.rec_f = int(self.lib.dsmil_rec_floats(P.C, P.D))
        return self.xs

    def new(self, *shape, dtype=torch.float32):
        return torch.empty(*shape, dtype=dtype, device=self.device)

    def phase1(self):
        P = self.P
        with torch.cuda.device(self.device):
            self.classes = self.new(self.total, P.C)
            cand = self.new(self.nb, self.cand_f)
            rc = self.lib.dsmil_shard_bags_phase1(P.ref, self.c_X, self.c_N, self.nb, self.c_off, Fn._ptr(self.classes),
                                                  Fn._ptr(cand), Fn._ptr(self.ws), self.ws.numel(), Fn._stream())
            _lib.check(rc, "dsmil_shard_bags_phase1")
        return cand

    def phase2(self, cands_all: torch.Tensor, G: int):
        P = self.P
        with torch.cuda.device(self.device):
            self.A = self.new(self.total, P.C)
            self.crit = self.new(self.nb, P.C, dtype=torch.int64)
            recs = self.new(self.nb, self.rec_f)
            rc = self.lib.dsmil_shard_bags_phase2(P.ref, self.c_X, self.c_N, self.nb, Fn._ptr(cands_all), G, Fn._ptr(self.A),
                                                  Fn._ptr(self.crit), Fn._ptr(recs), Fn._ptr(self.ws), self.ws.numel(),
                                                  Fn._stream())
            _lib.check(rc, "dsmil_shard_bags_phase2")
        return recs

    def phase3(self, recs_all: torch.Tensor, G: int):
        P = self.P
        with torch.cuda.device(self.device):
            B, pred = self.new(self.nb, P.C, P.D), self.new(self.nb, P.C)
            rc = self.lib.dsmil_shard_bags_phase3(P.ref, self.c_X, self.c_N, self.nb, Fn._ptr(recs_all), G, Fn._ptr(self.A),
                                                  Fn._ptr(B), Fn._ptr(pred), Fn._ptr(self.ws), self.ws.numel(), Fn._stream())
            _lib.check(rc, "dsmil_shard_bags_phase3")
        outs, row = [], 0
        for b, n in enumerate(self.Ns):
            outs.append((self.classes[row:row + n], pred[b:b + 1], self.A[row:row + n], B[b:b + 1], self.crit[b]))
            row += n
        return outs

    # ---- training: phases 1 and 2 that keep Q/H1 row-major and q_max, and the three backward phases ----------------
    # (dsmil_shard_bags_phase1/2_train, dsmil_shard_backward_bags_phase1/2/3).  Outputs stay packed [sum N_local, *].
    def phase1_train(self):
        """After begin(): (classes, Q, H1, cand [nb, cand])."""
        P = self.P
        with torch.cuda.device(self.device):
            classes = self.new(self.total, P.C)
            Q, H1 = self.new(self.total, Fn.Q_DIM), self.new(self.total, Fn.Q_DIM)
            cand = self.new(self.nb, self.cand_f)
            rc = self.lib.dsmil_shard_bags_phase1_train(P.ref, self.c_X, self.c_N, self.nb, self.c_off, Fn._ptr(classes),
                                                        Fn._ptr(Q), Fn._ptr(H1), Fn._ptr(cand), Fn._ptr(self.ws),
                                                        self.ws.numel(), Fn._stream())
            _lib.check(rc, "dsmil_shard_bags_phase1_train")
        return classes, Q, H1, cand

    def phase2_train(self, Q: torch.Tensor, cands_all: torch.Tensor, G: int):
        """(A logits, crit [nb, C] global rows, q_max [nb, C, 128], recs [nb, rec])."""
        P = self.P
        with torch.cuda.device(self.device):
            A = self.new(self.total, P.C)
            crit = self.new(self.nb, P.C, dtype=torch.int64)
            qmax = self.new(self.nb, P.C, Fn.Q_DIM)
            recs = self.new(self.nb, self.rec_f)
            rc = self.lib.dsmil_shard_bags_phase2_train(P.ref, self.c_X, self.c_N, self.nb, Fn._ptr(Q), Fn._ptr(cands_all),
                                                        G, Fn._ptr(A), Fn._ptr(crit), Fn._ptr(qmax), Fn._ptr(recs),
                                                        Fn._ptr(self.ws), self.ws.numel(), Fn._stream())
            _lib.check(rc, "dsmil_shard_bags_phase2_train")
        return A, crit, qmax, recs

    def phase3_train(self, recs_all: torch.Tensor, G: int, A: torch.Tensor):
        """dsmil_shard_bags_phase3 on phase2_train's logits: (A normalised in place, B [nb, C, D], pred [nb, C])."""
        P = self.P
        with torch.cuda.device(self.device):
            B, pred = self.new(self.nb, P.C, P.D), self.new(self.nb, P.C)
            rc = self.lib.dsmil_shard_bags_phase3(P.ref, self.c_X, self.c_N, self.nb, Fn._ptr(recs_all), G, Fn._ptr(A),
                                                  Fn._ptr(B), Fn._ptr(pred), Fn._ptr(self.ws), self.ws.numel(), Fn._stream())
            _lib.check(rc, "dsmil_shard_bags_phase3")
        return A, B, pred

    @staticmethod
    def _table(xs):
        nb = len(xs)
        return (C.c_void_p * nb)(*[x.data_ptr() for x in xs]), (C.c_int64 * nb)(*[int(x.shape[0]) for x in xs]), nb

    def bwd1(self, xs, A, B, d_classes, d_pred):
        """(dA, t [nb, C], gWi, gbi, gWf, gbf).  Allocates the backward workspace that bwd2 and bwd3 of the same step
        read the bag tables from."""
        P = self.P
        c_X, c_N, nb = self._table(xs)
        total = sum(int(x.shape[0]) for x in xs)
        with torch.cuda.device(self.device):
            self.bws = Fn._workspace(self.lib.dsmil_shard_backward_bags_workspace_bytes(P.ref, c_N, nb), self.device)
            dA, t = self.new(total, P.C), self.new(nb, P.C)
            gWi, gbi, gWf, gbf = _bwd1_shares(self)
            dc, dp = _upstream(d_classes, d_pred)
            rc = self.lib.dsmil_shard_backward_bags_phase1(P.ref, c_X, c_N, nb, Fn._ptr(A), Fn._ptr(B.contiguous()),
                                                           Fn._ptr(dc), Fn._ptr(dp), Fn._ptr(dA), Fn._ptr(t),
                                                           Fn._ptr(gWi), Fn._ptr(gbi), Fn._ptr(gWf), Fn._ptr(gbf),
                                                           Fn._ptr(self.bws), self.bws.numel(), Fn._stream())
            _lib.check(rc, "dsmil_shard_backward_bags_phase1")
        return dA, t, gWi, gbi, gWf, gbf

    def bwd2(self, xs, A, dA, t, Q):
        """(dL, dqm [nb, C, 128]); dL replaces dA in place."""
        P = self.P
        _, c_N, nb = self._table(xs)
        with torch.cuda.device(self.device):
            dqm = self.new(nb, P.C, Fn.Q_DIM)
            rc = self.lib.dsmil_shard_backward_bags_phase2(P.ref, c_N, nb, Fn._ptr(A), Fn._ptr(dA), Fn._ptr(t.contiguous()),
                                                           Fn._ptr(Q), Fn._ptr(dqm), Fn._ptr(self.bws), self.bws.numel(),
                                                           Fn._stream())
            _lib.check(rc, "dsmil_shard_backward_bags_phase2")
        return dA, dqm

    def bwd3(self, xs, row_offsets, Q, H1, dL, dqm, qmax, crit):
        """(gW1, gb1, gW2, gb2), this rank's shares."""
        P = self.P
        c_X, c_N, nb = self._table(xs)
        c_off = (C.c_int64 * nb)(*[int(o) for o in row_offsets])
        with torch.cuda.device(self.device):
            gW1, gb1, gW2, gb2 = _bwd3_shares(self)
            rc = self.lib.dsmil_shard_backward_bags_phase3(P.ref, c_X, c_N, nb, c_off, Fn._ptr(Q), Fn._ptr(H1), Fn._ptr(dL),
                                                           Fn._ptr(dqm.contiguous()), Fn._ptr(qmax.contiguous()),
                                                           Fn._ptr(crit.contiguous()), Fn._ptr(gW1), Fn._ptr(gb1),
                                                           Fn._ptr(gW2), Fn._ptr(gb2), Fn._ptr(self.bws), self.bws.numel(),
                                                           Fn._stream())
            _lib.check(rc, "dsmil_shard_backward_bags_phase3")
        return gW1, gb1, gW2, gb2


# One bag's own tensor passes through these unchanged, so a batch of one does the device work of the one-bag phases.
def _cat(ts):
    """Per-bag tensors packed in bag order along dim 0 (None for a tensor the model lacks: H1 of a linear q)."""
    return ts[0] if len(ts) == 1 or ts[0] is None else torch.cat(ts)


def _stack(ts):
    """Per-bag records as [nb, *]."""
    return ts[0][None] if len(ts) == 1 else torch.stack(ts)


def _sum(ts):
    """Sum over the bags of per-bag gradient shares (None for gW2 / gb2 of a linear q)."""
    return ts[0] if len(ts) == 1 or ts[0] is None else torch.stack(ts).sum(0)


def _gathered(recs_all, G, nb):
    """The all-gathered records [G][nb][*] of the batch as one contiguous [G][*] block per bag."""
    return [recs_all] if nb == 1 else [r.contiguous() for r in recs_all.view(G, nb, -1).unbind(1)]


def _bags(t, nb):
    """Per-bag [1, *] slices (views) of a tensor with a bag axis."""
    return [t] * nb if t is None or nb == 1 else list(t.split(1))


def _rows(t, xs):
    """Per-bag row blocks (views) of a tensor packed [sum N_local, *] in the order of the bags xs."""
    if t is None or len(xs) == 1:
        return [t] * len(xs)
    return list(t.split([int(x.shape[0]) for x in xs]))


class PerBagShardOps:
    """The interface of CudaShardBagOps over a one-bag ops object (CudaShardOps, or a stand-in with its methods), run
    one bag at a time: per-bag library calls, but the batch's collectives.  This is the sharded path of the shapes the
    batched ABI refuses (linear q, passing_v, D not a multiple of 128, more than 4 classes, D above 2048), and a bag may
    hold no local rows.  For one bag, it returns the one-bag ops' own tensors (viewed as [1, *] where the batch
    interface has a bag axis)."""

    def __init__(self, one):
        self.one = one

    def begin(self, X_locals: Sequence[torch.Tensor], row_offsets: Sequence[int]):
        """Returns the list of bags that phase1_train then fills with each bag's features as the one-bag phase 1
        returned them; phase2_train and the reverse pass (which is handed that list back) read those."""
        self.xs, self.offs = list(X_locals), [int(o) for o in row_offsets]
        return self.xs

    def phase1(self):
        self.p1 = list(map(self.one.phase1, self.xs, self.offs))                   # classes, Q, V (or X), cand
        return _stack([r[3] for r in self.p1])

    def phase2(self, cands_all: torch.Tensor, G: int):
        self.p2 = []
        for (_, Q, Vv, _), cands in zip(self.p1, _gathered(cands_all, G, len(self.xs))):
            qmax, crit = self.one.merge_candidates(cands, G)
            self.p2.append((*self.one.phase2(Vv, Q, qmax), crit))                   # A, rec, crit
        return _stack([r[1] for r in self.p2])

    def phase3(self, recs_all: torch.Tensor, G: int):
        outs = []
        for (classes, *_), (A, _, crit), recs in zip(self.p1, self.p2, _gathered(recs_all, G, len(self.xs))):
            A, B, pred = self.one.phase3(self.one.merge_partials(recs, G), A)
            outs.append((classes, pred, A, B, crit))
        return outs

    def phase1_train(self):
        classes, Q, H1, feats, cand = zip(*map(self.one.phase1_train, self.xs, self.offs))
        self.xs[:] = feats
        return _cat(classes), _cat(Q), _cat(H1), _stack(cand)

    def phase2_train(self, Q: torch.Tensor, cands_all: torch.Tensor, G: int):
        out = []
        for x, q, cands in zip(self.xs, _rows(Q, self.xs), _gathered(cands_all, G, len(self.xs))):
            qmax, crit = self.one.merge_candidates(cands, G)
            out.append((*self.one.phase2(x, q, qmax), crit, qmax))
        A, recs, crit, qmax = zip(*out)
        return _cat(A), _stack(crit), _stack(qmax), _stack(recs)

    def phase3_train(self, recs_all: torch.Tensor, G: int, A: torch.Tensor):
        A, B, pred = zip(*[self.one.phase3(self.one.merge_partials(recs, G), a)
                           for a, recs in zip(_rows(A, self.xs), _gathered(recs_all, G, len(self.xs)))])
        return _cat(A), _cat(B), _cat(pred)

    def bwd1(self, xs, A, B, d_classes, d_pred):
        dA, t, *grads = zip(*map(self.one.bwd1, xs, _rows(A, xs), _bags(B, len(xs)), _rows(d_classes, xs),
                                 _bags(d_pred, len(xs))))
        return (_cat(dA), _stack(t), *map(_sum, grads))                             # grads: gWi, gbi, gWf, gbf

    def bwd2(self, xs, A, dA, t, Q):
        dL, dqm = zip(*map(self.one.bwd2, _rows(A, xs), _rows(dA, xs), t.unbind(), _rows(Q, xs)))
        return _cat(dL), _stack(dqm)

    def bwd3(self, xs, row_offsets, Q, H1, dL, dqm, qmax, crit):
        return tuple(map(_sum, zip(*map(self.one.bwd3, xs, row_offsets, _rows(Q, xs), _rows(H1, xs), _rows(dL, xs),
                                        dqm.unbind(), qmax.unbind(), crit.unbind()))))


class CudaShardBagDevOps:
    """The training interface of CudaShardBagOps (begin, phase1-3_train, bwd1-3) over the capture-safe calls
    (dsmil_shard_bags_*_dev, dsmil_shard_backward_bags_*_dev): every call only enqueues device work, so the sharded step
    and its collectives can be recorded once in a CUDA graph and replayed over batches of new local sizes.

    The batch is static: begin() takes [slots] (slots [nb, max_rows, D]: bag b's local rows are slots[b, :Ns[b]]) and
    the row offsets [nb] int64 on the device; Ns [nb] int64 and status [1] int32 are device tensors given here.  The
    packed per-row outputs have nb * max_rows rows, the live ones at the prefix sums of Ns.  A bag the planner refuses
    sets status, and the step runs on the library's stand-in batch (see include/dsmil_b200.h)."""

    def __init__(self, params: Sequence[Optional[torch.Tensor]], Ns: torch.Tensor, status: torch.Tensor):
        self.lib = _lib.load()
        self.P = Fn.ParamPack(*params)
        self.device = self.P.device
        if not self.lib.dsmil_shard_bags_supported(self.P.ref):
            raise ValueError(f"the capture-safe sharded step runs on the batched tensor-core path only; D={self.P.D}, "
                             f"C={self.P.C}, nonlinear={self.P.nonlinear}, passing_v={self.P.passing_v} is not on it")
        self.Ns, self.status = Ns, status

    def new(self, *shape, dtype=torch.float32):
        return torch.empty(*shape, dtype=dtype, device=self.device)

    def begin(self, X_locals: Sequence[torch.Tensor], row_offsets: torch.Tensor):
        (slots,) = X_locals
        P = self.P
        self.xs = Fn._slot_addrs(slots, P, "slots")
        self.nb, self.max_rows = int(slots.shape[0]), int(slots.shape[1])
        self.rows, self.offs = self.nb * self.max_rows, row_offsets
        with torch.cuda.device(self.device):
            self.ws = Fn._workspace(self.lib.dsmil_shard_bags_train_dev_workspace_bytes(P.ref, self.nb, self.max_rows),
                                    self.device)
        self.cand_f = int(self.lib.dsmil_cand_floats(P.C))
        self.rec_f = int(self.lib.dsmil_rec_floats(P.C, P.D))
        return [slots]

    def phase1_train(self):
        """(classes, Q, H1 [nb * max_rows, *], cand [nb, cand])."""
        P = self.P
        with torch.cuda.device(self.device):
            classes, Q, H1 = self.new(self.rows, P.C), self.new(self.rows, Fn.Q_DIM), self.new(self.rows, Fn.Q_DIM)
            cand = self.new(self.nb, self.cand_f)
            rc = self.lib.dsmil_shard_bags_phase1_train_dev(P.ref, Fn._ptr(self.xs), Fn._ptr(self.Ns), Fn._ptr(self.offs),
                                                            self.nb, self.max_rows, Fn._ptr(classes), Fn._ptr(Q),
                                                            Fn._ptr(H1), Fn._ptr(cand), Fn._ptr(self.status),
                                                            Fn._ptr(self.ws), self.ws.numel(), Fn._stream())
            _lib.check(rc, "dsmil_shard_bags_phase1_train_dev")
        return classes, Q, H1, cand

    def phase2_train(self, Q: torch.Tensor, cands_all: torch.Tensor, G: int):
        P = self.P
        with torch.cuda.device(self.device):
            A = self.new(self.rows, P.C)
            crit = self.new(self.nb, P.C, dtype=torch.int64)
            qmax = self.new(self.nb, P.C, Fn.Q_DIM)
            recs = self.new(self.nb, self.rec_f)
            rc = self.lib.dsmil_shard_bags_phase2_train_dev(P.ref, self.nb, self.max_rows, Fn._ptr(Q), Fn._ptr(cands_all),
                                                            G, Fn._ptr(A), Fn._ptr(crit), Fn._ptr(qmax), Fn._ptr(recs),
                                                            Fn._ptr(self.ws), self.ws.numel(), Fn._stream())
            _lib.check(rc, "dsmil_shard_bags_phase2_train_dev")
        return A, crit, qmax, recs

    def phase3_train(self, recs_all: torch.Tensor, G: int, A: torch.Tensor):
        P = self.P
        with torch.cuda.device(self.device):
            B, pred = self.new(self.nb, P.C, P.D), self.new(self.nb, P.C)
            rc = self.lib.dsmil_shard_bags_phase3_dev(P.ref, self.nb, self.max_rows, Fn._ptr(recs_all), G, Fn._ptr(A),
                                                      Fn._ptr(B), Fn._ptr(pred), Fn._ptr(self.ws), self.ws.numel(),
                                                      Fn._stream())
            _lib.check(rc, "dsmil_shard_bags_phase3_dev")
        return A, B, pred

    def bwd1(self, xs, A, B, d_classes, d_pred):
        P = self.P
        with torch.cuda.device(self.device):
            self.bws = Fn._workspace(self.lib.dsmil_shard_backward_bags_dev_workspace_bytes(P.ref, self.nb, self.max_rows),
                                     self.device)
            dA, t = self.new(self.rows, P.C), self.new(self.nb, P.C)
            gWi, gbi, gWf, gbf = _bwd1_shares(self)
            dc, dp = _upstream(d_classes, d_pred)
            rc = self.lib.dsmil_shard_backward_bags_phase1_dev(P.ref, Fn._ptr(self.xs), Fn._ptr(self.Ns), self.nb,
                                                               self.max_rows, Fn._ptr(A), Fn._ptr(B.contiguous()),
                                                               Fn._ptr(dc), Fn._ptr(dp), Fn._ptr(dA), Fn._ptr(t),
                                                               Fn._ptr(gWi), Fn._ptr(gbi), Fn._ptr(gWf), Fn._ptr(gbf),
                                                               Fn._ptr(self.status), Fn._ptr(self.bws), self.bws.numel(),
                                                               Fn._stream())
            _lib.check(rc, "dsmil_shard_backward_bags_phase1_dev")
        return dA, t, gWi, gbi, gWf, gbf

    def bwd2(self, xs, A, dA, t, Q):
        P = self.P
        with torch.cuda.device(self.device):
            dqm = self.new(self.nb, P.C, Fn.Q_DIM)
            rc = self.lib.dsmil_shard_backward_bags_phase2_dev(P.ref, self.nb, self.max_rows, Fn._ptr(A), Fn._ptr(dA),
                                                               Fn._ptr(t.contiguous()), Fn._ptr(Q), Fn._ptr(dqm),
                                                               Fn._ptr(self.bws), self.bws.numel(), Fn._stream())
            _lib.check(rc, "dsmil_shard_backward_bags_phase2_dev")
        return dA, dqm

    def bwd3(self, xs, row_offsets, Q, H1, dL, dqm, qmax, crit):
        P = self.P
        with torch.cuda.device(self.device):
            gW1, gb1, gW2, gb2 = _bwd3_shares(self)
            rc = self.lib.dsmil_shard_backward_bags_phase3_dev(P.ref, self.nb, self.max_rows, Fn._ptr(row_offsets),
                                                               Fn._ptr(Q), Fn._ptr(H1), Fn._ptr(dL),
                                                               Fn._ptr(dqm.contiguous()), Fn._ptr(qmax.contiguous()),
                                                               Fn._ptr(crit.contiguous()), Fn._ptr(gW1), Fn._ptr(gb1),
                                                               Fn._ptr(gW2), Fn._ptr(gb2), Fn._ptr(self.bws),
                                                               self.bws.numel(), Fn._stream())
            _lib.check(rc, "dsmil_shard_backward_bags_phase3_dev")
        return gW1, gb1, gW2, gb2


@torch.no_grad()
def sharded_forward_bags_batched(bops, X_locals, row_offsets, group=None):
    """The forward of a batch of row-sharded bags: 2 all-gathers per step, whatever the batch.  `bops` is a
    CudaShardBagOps (3 library calls per step) or a PerBagShardOps.  Returns one (classes_local [N_r, C],
    prediction_bag [1, C], A_local [N_r, C], B [1, C, D], crit_idx [C]) per bag."""
    bops.begin(X_locals, row_offsets)
    cand = bops.phase1()
    cands_all, G = _all_gather(cand.view(-1), group)        # exchange 1: [G][nb][cand]
    recs = bops.phase2(cands_all, G)
    recs_all, G = _all_gather(recs.view(-1), group)         # exchange 2: [G][nb][rec]
    return bops.phase3(recs_all, G)


class ShardedBagsGraph:
    """Fixed-shape serving loop: the whole row-sharded step -- three library calls and the two NCCL all-gathers -- is
    captured ONCE in a CUDA graph and replayed, so a step costs one graph launch instead of ~12 host-driven launches
    (the sharded step is latency-, not bandwidth-bound: a few KB cross NVLink).  The bags' storage and shapes must
    stay the same between replays (write new features INTO the same tensors), and so must the weights (the captured
    step reuses the bag table and the bf16 weight images of the warm-up run: build a new graph after a weight update);
    every rank must build and replay the graph collectively."""

    def __init__(self, bops: "CudaShardBagOps", X_locals, row_offsets, group=None, warmup: int = 3):
        self.bops, self.xs, self.offs, self.group = bops, list(X_locals), list(row_offsets), group
        # eager warm-up: uploads the bag table, sets NCCL up for these sizes
        Fn._warm_up(bops.device, warmup, lambda: sharded_forward_bags_batched(bops, self.xs, self.offs, group))
        torch.cuda.synchronize(bops.device)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.outs = sharded_forward_bags_batched(bops, self.xs, self.offs, group)

    @torch.no_grad()
    def replay(self):
        """Runs the captured step on the current stream; returns the (static) output tensors of the step."""
        self.graph.replay()
        return self.outs


def _all_gather(rec: torch.Tensor, group) -> Tuple[torch.Tensor, int]:
    import torch.distributed as dist
    G = dist.get_world_size(group)
    out = torch.empty(G * rec.numel(), dtype=rec.dtype, device=rec.device)
    dist.all_gather_into_tensor(out, rec.contiguous(), group=group)
    return out, G


def sharded_forward(ops, X_local: torch.Tensor, row_offset: int, group=None):
    """Forward of one bag whose rows are spread over the ranks of `group`: `sharded_forward_bags` of a batch of one.
    Returns (classes_local[N_r,C], prediction_bag[1,C], A_local[N_r,C], B[1,C,D], crit_idx[C])."""
    return sharded_forward_bags(ops, [X_local], [row_offset], group)[0]


@torch.no_grad()
def virtual_sharded_forward(ops, X: torch.Tensor, G: int):
    """Same algebra with G logical shards on ONE device and the collectives replaced by local
    concatenation -- lets the sharding logic be validated without G GPUs (SURVEY §4-v)."""
    bounds = shard_bounds(int(X.shape[0]), G)
    loc = [ops.phase1(X[lo:hi], lo) for lo, hi in bounds]
    cands = torch.cat([l[3] for l in loc])
    qmax, crit = ops.merge_candidates(cands, G)
    part = [ops.phase2(l[2], l[1], qmax) for l in loc]
    rec_g = ops.merge_partials(torch.cat([p[1] for p in part]), G)
    outs = [ops.phase3(rec_g, p[0]) for p in part]
    return (torch.cat([l[0] for l in loc]), outs[0][2], torch.cat([o[0] for o in outs]), outs[0][1], crit)


def sharded_forward_bags(ops, X_locals: Sequence[torch.Tensor], row_offsets: Sequence[int], group=None):
    """A batch of giant bags, each row-sharded over the group, through the one-bag ops `ops` (CudaShardOps) a bag at a
    time: the per-bag records are packed so the whole batch costs TWO collectives (not two per bag) -- at a few KB per
    record the exchange is latency-bound, so batching is what keeps NVLink out of the critical path."""
    return sharded_forward_bags_batched(PerBagShardOps(ops), X_locals, row_offsets, group)


# ---- row-sharded training step of a minibatch of bags (SURVEY §8e "Backward"; oracle: backward_sharded) ----------
# Six collectives per step whatever the batch size: the forward's two all-gathers, one all-reduce(max) of nb*C floats
# in the loss and three all-reduce(sum) in the reverse pass (t [nb,C], dq_max [nb,C,128], one flat buffer of parameter
# gradients).  `bops` is a CudaShardBagOps (3 + 3 library calls per step), a PerBagShardOps (the one-bag calls per bag;
# one bag is the one-bag training step), or any object with their begin / phase*_train / bwd1-3 methods (the host
# logic below calls nothing else, so it runs over gloo with a CPU stand-in).


def _all_reduce_sum(t: torch.Tensor, group) -> torch.Tensor:
    import torch.distributed as dist
    dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
    return t


def _reduce_flat(grads, group, reduce):
    """One reduce over the non-None tensors of `grads`, packed into a flat buffer; returns views in the same order."""
    parts = [g for g in grads if g is not None]
    flat = reduce(torch.cat([g.reshape(-1) for g in parts]), group)
    out, off = [], 0
    for g in grads:
        if g is None:
            out.append(None)
            continue
        out.append(flat[off:off + g.numel()].view_as(g))
        off += g.numel()
    return out


class ShardBagsSaved:
    """What one rank keeps between the forward of a row-sharded batch and its reverse pass (per-row tensors packed in
    bag order over the local rows)."""
    __slots__ = ("xs", "row_offsets", "Q", "H1", "A", "B", "qmax", "crit")

    def __init__(self, xs, row_offsets, Q, H1, A, B, qmax, crit):
        # a device tensor of offsets (CudaShardBagDevOps) stays on the device
        offs = row_offsets if torch.is_tensor(row_offsets) else [int(o) for o in row_offsets]
        self.xs, self.row_offsets, self.Q, self.H1 = list(xs), offs, Q, H1
        self.A, self.B, self.qmax, self.crit = A, B, qmax, crit


@torch.no_grad()
def sharded_forward_bags_train(bops, X_locals, row_offsets, group=None, gather=_all_gather):
    """Forward of a batch of row-sharded bags that keeps what `sharded_backward_bags` needs.  Returns
    ((classes_local [sum N_local, C], pred [nb, C], A_local [sum N_local, C], B [nb, C, D], crit [nb, C]), saved);
    pred, B and crit (global rows: the row within the whole bag) are replicated."""
    xs = bops.begin(X_locals, row_offsets)
    classes, Q, H1, cand = bops.phase1_train()
    cands_all, G = gather(cand.reshape(-1), group)                          # exchange 1: [G][nb][cand]
    A, crit, qmax, recs = bops.phase2_train(Q, cands_all, G)
    recs_all, G = gather(recs.reshape(-1), group)                           # exchange 2: [G][nb][rec]
    A, B, pred = bops.phase3_train(recs_all, G, A)
    return (classes, pred, A, B, crit), ShardBagsSaved(xs, row_offsets, Q, H1, A, B, qmax, crit)


@torch.no_grad()
def sharded_backward_bags(bops, saved: ShardBagsSaved, d_classes_local: Optional[torch.Tensor],
                          d_pred: Optional[torch.Tensor], group=None, reduce=_all_reduce_sum):
    """Reverse pass of `sharded_forward_bags_train`: exactly three all-reduce(sum) -- t [nb, C], dq_max [nb, C, 128] and
    one flat buffer of the parameter gradients.  Returns (gWi, gbi, gW1, gb1, gW2, gb2, gWf, gbf), sums over the bags,
    identical on every rank."""
    dA, t, gWi, gbi, gWf, gbf = bops.bwd1(saved.xs, saved.A, saved.B, d_classes_local, d_pred)
    t = reduce(t, group)                                                    # reduce 1
    dL, dqm = bops.bwd2(saved.xs, saved.A, dA, t, saved.Q)
    dqm = reduce(dqm, group)                                                # reduce 2
    gW1, gb1, gW2, gb2 = bops.bwd3(saved.xs, saved.row_offsets, saved.Q, saved.H1, dL, dqm, saved.qmax, saved.crit)
    gWi, gbi, gW1, gb1, gW2, gb2 = _reduce_flat((gWi, gbi, gW1, gb1, gW2, gb2), group, reduce)   # reduce 3
    return gWi, gbi, gW1, gb1, gW2, gb2, gWf, gbf                           # Wf/bf grads are replicated already


class ShardedMILBagsFn(torch.autograd.Function):
    """autograd node of a batch of row-sharded bags: forward = sharded_forward_bags_train, backward =
    sharded_backward_bags.  Every rank of the group must call it (and `.backward()`) in the same order.  args: bops,
    row_offsets, group, nb, the nb local bags, then the ten parameter tensors in ABI order (Wv, bv must be None)."""

    @staticmethod
    def forward(ctx, bops, row_offsets, group, nb, *args):
        ctx.set_materialize_grads(False)          # unused outputs (A, B) arrive as None, not as zero tensors
        outs, saved = sharded_forward_bags_train(bops, args[:nb], row_offsets, group)
        ctx.bops, ctx.saved, ctx.group, ctx.nb = bops, saved, group, nb
        classes, pred, A, B, crit = outs
        ctx.mark_non_differentiable(crit)
        return classes, pred, A, B, crit

    @staticmethod
    def backward(ctx, d_classes, d_pred, d_A, d_B, _d_crit):
        if d_A is not None or d_B is not None:
            raise NotImplementedError("sharded backward: gradients through A / B are not supported "
                                      "(the callers use classes and prediction_bag only, train_tcga.py:67-72)")
        gWi, gbi, gW1, gb1, gW2, gb2, gWf, gbf = sharded_backward_bags(ctx.bops, ctx.saved, d_classes, d_pred, ctx.group)
        return (None, None, None, None, *([None] * ctx.nb), gWi, gbi, gW1, gb1, gW2, gb2, None, None, gWf, gbf)


def sharded_milnet_forward_bags(milnet, X_locals: Sequence[torch.Tensor], row_offsets: Sequence[int], group=None,
                                ops=None):
    """Packed `(classes_local, prediction_bag, A_local, B, crit_idx)` of a batch of bags whose rows live on several
    ranks (bag b: this rank's rows [row_offsets[b], row_offsets[b] + len(X_locals[b])); CudaShardBagOps needs at
    least one per bag), with
    autograd: `loss.backward()` on every rank (loss from `sharded_caller_loss_bags`) leaves identical, fully reduced
    `.grad`s on the parameters.  classes_local / A_local are [sum N_local, C] in bag order; prediction_bag [nb, C],
    B [nb, C, D] and crit_idx [nb, C] (global rows) are replicated."""
    params = milnet_params(milnet)
    ops = ops or CudaShardBagOps(params)
    return ShardedMILBagsFn.apply(ops, [int(o) for o in row_offsets], group, len(X_locals), *X_locals, *params)


def sharded_max_prediction_bags(classes_local: torch.Tensor, crit: torch.Tensor, row_offsets: Sequence[int],
                                Ns: Sequence[int], group=None):
    """Per-bag `torch.max(ins_prediction, 0)[0]`, [nb, C], of bags whose rows are spread over ranks: one all-reduce(max)
    of nb*C floats for the whole batch.  The value is the same on every rank; the gradient flows only into the row
    that holds the maximum, on the rank that owns it.  classes_local is packed [sum Ns, C]; crit [nb, C] holds global
    rows."""
    import torch.distributed as dist
    dev = classes_local.device
    Cc = int(classes_local.shape[1])
    Ns = [int(v) for v in Ns]
    # per bag: row offset, local rows, first packed row.  One bag passes them as kernel arguments; a batch copies them
    # from pinned memory, which does not block the host (a pageable copy would synchronise with the stream).
    if len(Ns) == 1:
        off, n, first = int(row_offsets[0]), Ns[0], 0
    else:
        host = torch.tensor([[int(o) for o in row_offsets], Ns, list(accumulate([0] + Ns[:-1]))], dtype=torch.int64,
                            pin_memory=dev.type == "cuda")
        off, n, first = host.to(dev, non_blocking=True)[:, :, None]
    loc = crit.to(dev) - off
    owned = (loc >= 0) & (loc < n)
    total = int(classes_local.shape[0])
    if total > 0:
        # owned entries index their row; the others any valid row (their value is replaced, their gradient is zero)
        mine = classes_local.gather(0, (first + loc.clamp(min=0)).clamp(max=total - 1))
    else:
        mine = classes_local.new_zeros(len(Ns), Cc)
    glob = torch.where(owned, mine.detach(), torch.full_like(mine, float("-inf")))
    dist.all_reduce(glob, op=dist.ReduceOp.MAX, group=group)
    return torch.where(owned, mine, glob)


def sharded_max_prediction_bags_dev(classes_local: torch.Tensor, crit: torch.Tensor, row_offsets: torch.Tensor,
                                    Ns: torch.Tensor, refused: torch.Tensor, group=None):
    """sharded_max_prediction_bags with the local sizes Ns [nb] and the row offsets [nb] in device tensors (each bag's
    first packed row is the prefix sum of Ns), for a step recorded in a CUDA graph.  `refused` (a device bool scalar:
    this rank refused the batch) rides in the same all-reduce(max) as one extra float, so a step still makes one
    collective here.  Returns (max_prediction [nb, C], refused on any rank: a device bool scalar); the values and
    gradients are those of sharded_max_prediction_bags."""
    import torch.distributed as dist
    Ns = Ns.to(crit.device)
    first = torch.cumsum(Ns, 0) - Ns
    loc = crit - row_offsets[:, None]
    owned = (loc >= 0) & (loc < Ns[:, None])
    total = int(classes_local.shape[0])
    mine = classes_local.gather(0, (first[:, None] + loc.clamp(min=0)).clamp(max=total - 1))
    glob = torch.where(owned, mine.detach(), torch.full_like(mine, float("-inf")))
    buf = torch.cat([glob.reshape(-1), refused.reshape(1).to(glob.dtype)])
    dist.all_reduce(buf, op=dist.ReduceOp.MAX, group=group)
    return torch.where(owned, mine, buf[:-1].view_as(mine)), buf[-1] > 0


def sharded_caller_loss_bags(classes_local, prediction_bag, crit, row_offsets, labels, criterion, group=None, *, Ns):
    """The minibatch loss of feed.train_epoch(bags_per_step=k), 0.5 * criterion(pred [k, C]) + 0.5 * criterion(max
    instance [k, C]), for row-sharded bags: same value on every rank; `loss.backward()` on every rank gives the
    single-device gradients.  Ns: this rank's row count of each bag (the packing of classes_local)."""
    max_prediction = sharded_max_prediction_bags(classes_local, crit, row_offsets, Ns, group)
    tgt = labels.reshape(prediction_bag.shape).to(prediction_bag.dtype)
    return 0.5 * criterion(prediction_bag, tgt) + 0.5 * criterion(max_prediction, tgt)


def sharded_milnet_forward(milnet, X_local: torch.Tensor, row_offset: int, group=None, ops=None):
    """`classes_local, prediction_bag, A_local, B (, crit_idx) = milnet(X)` for a bag whose rows live on several
    ranks, with autograd: `loss.backward()` on every rank (loss from `sharded_caller_loss`) leaves identical, fully
    reduced `.grad`s on the parameters.  A batch of one through `sharded_milnet_forward_bags` over the one-bag ops
    `ops` (default: CudaShardOps, the one-bag ABI, which takes every shape and a rank with no rows of the bag)."""
    ops = PerBagShardOps(ops or CudaShardOps(milnet_params(milnet)))
    classes, pred, A, B, crit = sharded_milnet_forward_bags(milnet, [X_local], [row_offset], group, ops)
    return classes, pred, A, B, crit[0]


def sharded_caller_loss(classes_local, prediction_bag, crit, row_offset, label, criterion, group=None):
    """0.5 * criterion(bag) + 0.5 * criterion(max instance) (train_tcga.py:67-71) for a row-sharded bag: same
    value on every rank; `loss.backward()` on every rank gives the single-device gradients."""
    return sharded_caller_loss_bags(classes_local, prediction_bag.view(1, -1), crit.view(1, -1), [row_offset], label,
                                    criterion, group, Ns=[len(classes_local)])


@torch.no_grad()
def virtual_sharded_train_step_bags(make_ops, Xs: Sequence[torch.Tensor], G: int, loss_grads):
    """A training step of a batch of bags with G logical shards each on ONE device: the all-gathers replaced by
    concatenation and the all-reduces by local sums (same kernels, same record layouts).  `make_ops()` returns a fresh
    ops object per logical rank (each holds its rank's workspaces).  `loss_grads(classes [sum N, C], pred [nb, C],
    crit [nb, C]) -> (d_classes [sum N, C] | None, d_pred [nb, C] | None)`, with classes packed in bag order.  Returns
    ((classes, pred, A, B, crit), grads) with classes / A packed in bag order and grads in the order of
    `sharded_backward_bags`."""
    bounds = [shard_bounds(int(x.shape[0]), G) for x in Xs]              # [bag][rank]
    ranks = []
    for r in range(G):
        ops = make_ops()
        xs = ops.begin([x[b[r][0]:b[r][1]] for x, b in zip(Xs, bounds)], [b[r][0] for b in bounds])
        ranks.append(dict(ops=ops, xs=xs, offs=[b[r][0] for b in bounds], p1=ops.phase1_train()))
    cands = torch.cat([R["p1"][3].reshape(-1) for R in ranks])
    for R in ranks:
        R["p2"] = R["ops"].phase2_train(R["p1"][1], cands, G)             # A, crit, qmax, recs
    recs = torch.cat([R["p2"][3].reshape(-1) for R in ranks])
    for R in ranks:
        R["p3"] = R["ops"].phase3_train(recs, G, R["p2"][0])              # A, B, pred
    B, pred, crit = ranks[0]["p3"][1], ranks[0]["p3"][2], ranks[0]["p2"][1]

    def rank_rows(r):                                                    # this rank's packed rows, per bag
        out, lo = [], 0
        for b in bounds:
            n = b[r][1] - b[r][0]
            out.append((lo, lo + n))
            lo += n
        return out
    rows = [rank_rows(r) for r in range(G)]

    def to_bag_order(per_rank):                                          # [rank][sum N_r, *] -> [sum N, *]
        return torch.cat([per_rank[r][slice(*rows[r][b])] for b in range(len(Xs)) for r in range(G)])

    classes = to_bag_order([R["p1"][0] for R in ranks])
    A = to_bag_order([R["p3"][0] for R in ranks])
    d_classes, d_pred = loss_grads(classes, pred, crit)
    if d_classes is not None:                                            # bag order -> each rank's packing
        start = [0]
        for x in Xs:
            start.append(start[-1] + int(x.shape[0]))
        d_loc = [torch.cat([d_classes[start[b] + bounds[b][r][0]:start[b] + bounds[b][r][1]] for b in range(len(Xs))])
                 for r in range(G)]
    b1 = [R["ops"].bwd1(R["xs"], R["p3"][0], B, None if d_classes is None else d_loc[r], d_pred)
          for r, R in enumerate(ranks)]                                  # dA, t, gWi, gbi, gWf, gbf
    t = torch.stack([b[1] for b in b1]).sum(0)                           # reduce 1
    b2 = [R["ops"].bwd2(R["xs"], R["p3"][0], b[0], t, R["p1"][1]) for R, b in zip(ranks, b1)]
    dqm = torch.stack([b[1] for b in b2]).sum(0)                         # reduce 2
    b3 = [R["ops"].bwd3(R["xs"], R["offs"], R["p1"][1], R["p1"][2], b[0], dqm, R["p2"][2], R["p2"][1])
          for R, b in zip(ranks, b2)]
    tot = lambda ts: None if ts[0] is None else torch.stack(list(ts)).sum(0)   # reduce 3
    gWi, gbi = tot([b[2] for b in b1]), tot([b[3] for b in b1])
    gW1, gb1, gW2, gb2 = (tot([b[i] for b in b3]) for i in range(4))
    return (classes, pred, A, B, crit), (gWi, gbi, gW1, gb1, gW2, gb2, b1[0][4], b1[0][5])
