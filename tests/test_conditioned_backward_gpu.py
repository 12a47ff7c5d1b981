"""Q-MLP and value-network gradients of every backward route against an fp64 backward run on the kernels' OWN saved
activations (the conditioned check).

Every other gradient test compares the device with `orc.backward` run on the oracle's own fp64 forward, so it also
measures the forward's rounding; on the tensor-core forward that rounding (3xBF16 Q, amplified by the softmax over the
instances) dominates, and the q.* bars there are 1e-3 to 2e-3.  Here each case runs the route's own training forward
through the C ABI with saves, copies A, B, Q, H1, V and crit_idx to the host, and runs `orc.backward` in fp64 on
exactly what the backward kernels receive (per bag, summed over the bags of a batch; `orc.backward_sharded` for virtual
ranks).  What is left is the backward's own fp32 arithmetic, so the bars are tight:

    q.* (W1, b1, W2, b2)           1e-4 rel-to-max
    Wi, bi, Wf, bf, Wv, bv         2e-5 rel-to-max
    gX, row by row                 1e-4 of the row's own maximum (floor: 1e-3 of the tensor's maximum)

Measured on one NVIDIA H100 80GB HBM3 (700 W limit), largest over the cases of a route, probes on or off:

    route (cases)             W1      b1      W2      b2      Wv      bv      Wi, bi, Wf, bf    gX
    dsmil_backward            1.4e-6  3.1e-6  1.9e-6  1.8e-6  2.3e-7  1.2e-7  <= 2.4e-7          3.0e-7
    dsmil_backward_bags       1.2e-6  2.5e-6  1.8e-6  1.8e-6                  <= 2.3e-7          3.2e-7
    *_backward_bags_dev       4.6e-6  1.3e-5  9.0e-6  9.5e-6                  <= 2.1e-7
    *_backward_bags_models    3.2e-6  7.4e-6  7.0e-6  6.0e-6                  <= 1.5e-7          1.9e-7
    row-sharded, batched      1.5e-6  3.7e-6  1.7e-6  2.3e-6                  <= 1.5e-7
    row-sharded, per bag      1.5e-6  4.9e-6  2.7e-6  2.7e-6                  <= 2.1e-7

Every bar is more than 7x above them, and none is above the fp32 restatement's error on the same inputs.

Probes.  With A ~ 1/N an ordinary row's share of a q.* reduction is tiny, so a lost row can hide under any bar.  Each
case therefore runs twice: on the saved activations as they are, and with the saved A replaced on the device and in the
host copy by A' = (A + a 1[probe]) / (1 + a n_probe) per bag and column (a n_probe = PROBE_MASS: the probe rows then
hold 4/5 of each column; A' stays positive and sums to 1).  Probe rows are each bag's first and last rows, rows
127-129, and the first and last row of every split or chunk of the q.* reductions: gW1 = dz1^T X (launch_gemm_tn's
tile splits; k_gemm_tn_rag's chunks of rag_rows_per_chunk(128, D, .) rows), gW2 = dz2^T H1 (gemm_tn_split(128, 128,
.)), the column sums of gb1 / gb2 / gbv (colsum_split), t = sum_n A dA (k_bwd_t_partial's 256-row blocks; the
bwd_bags_ctas CTAs of k_bwd_rowdot_b, 8 rows at a time), dq_max = dL^T Q (launch_gemm_tn on one bag) and gWv = dzv^T Xv.
Routes that take d_A weight it on the probe rows too.  The CPU part proves, with the oracle alone, that dropping or
doubling any probe row from any of those reductions moves a checked gradient by more than 20x its bar.

Upstream.  d_classes = 1 + N(0, 1) and d_pred ~ N(0, 1); where a route takes them, d_A ~ N(0, 1) (4x, at least 1 in
magnitude, on probe rows) and d_B = 1e-2 N(0, 1): dA = V dB^T + d_A is then carried by d_A, and dL = A (dA - t) does not
cancel (with N(0, 1) weights on B, dA = X dB^T cancels at D = 2048).  The CPU part asserts the conditioning of every
checked sum, and that the fp32 restatement of the same algebra stays under each bar on the same inputs.
"""
from __future__ import annotations

import ctypes as C
import functools
from dataclasses import dataclass
from typing import Dict, List, Tuple

import numpy as np
import pytest
import torch

from conftest import rel_to_max
from oracle import dsmil_oracle as orc
from test_dense_upstream_grads_gpu import (K_SPLITS, TBK, TBM, _DevRank, ceil_div, colsum_ranges, rag_rows_per_chunk,
                                          rowwise_err, tn_splits, tn_use_gemv)

KQ = 128                   # DSMIL_Q
K_SMS = 132                # kSms (common.cuh): sizes bwd_bags_ctas
PROBE_MASS = 4.0           # a * n_probe
PROBE_DA = 4.0
TOL_Q, TOL_P = 1e-4, 2e-5
Q_NAMES = ("W1", "b1", "W2", "b2")
SENSITIVITY = 20.0
KAPPA_UPSTREAM = 10.0       # gbi and dA - t: set by the upstream choice
KAPPA_SOFTMAX = 200.0      # gb1, gb2, gbv: sum_n dL[n, k] = 0 (A sums to 1), so dz1 / dz2 cancel over the rows


# ---------------------------------------------------------------------------------------------- split mirror
def tn_ranges(M1, M2, N, aligned=True):
    """launch_gemm_tn(P, M1, R, M2, N): [lo, hi) rows of each split (gemm_generic.cuh)."""
    S = tn_splits(M1, M2, N)
    if tn_use_gemv(M1, M2) and aligned:
        rps = ceil_div(N, S)
    else:
        if tn_use_gemv(M1, M2):
            S = max(1, min(S, K_SPLITS // (ceil_div(M1, TBM) * ceil_div(M2, TBM))))
        rps = ceil_div(ceil_div(N, S), TBK) * TBK
    return [(z * rps, min(N, (z + 1) * rps)) for z in range(S)]


def t_blocks(N):
    """k_bwd_t_partial: min(ceil(N / 256), 296) CTAs, grid-stride over 256-row blocks (contiguous while N <= 296 * 256)."""
    assert N <= K_SPLITS * 256
    return [(x * 256, min(N, x * 256 + 256)) for x in range(min(ceil_div(N, 256), K_SPLITS))]


def bwd_bags_ctas(nb, max_N):
    """bag_plan.cuh: CTAs per bag of k_bwd_rowdot_b / k_bwd_dL_b / k_bwd_dq_b, from the batch shape alone."""
    return max(1, min(ceil_div(K_SMS * 8, nb), ceil_div(max_N, 64)))


def rowdot_cta_rows(N, G):
    """First and last row of each of the G CTAs of k_bwd_rowdot_b over one bag: CTA x takes 8-row groups x, x + G, ..."""
    rows, last_grp = set(), (N - 1) // 8
    for x in range(min(G, last_grp + 1)):
        g = last_grp - ((last_grp - x) % G)
        rows |= {8 * x, min(N - 1, 8 * g + 7)}
    return rows


@dataclass
class Layout:
    """The row ranges the q.* reductions of one backward call walk, over its packed rows, and rows of per-bag CTAs."""
    ranges: Dict[str, List[Tuple[int, int]]]
    extra: set
    info: dict


def single_layout(C_, D, N, nonlinear, passing_v):
    """dsmil_backward (and each one-bag sharded phase) over N rows."""
    r = {"W1": tn_ranges(KQ, D, N), "cs": colsum_ranges(N), "t": t_blocks(N), "dqm": tn_ranges(C_, KQ, N)}
    if nonlinear:
        r["W2"] = tn_ranges(KQ, KQ, N)
    if passing_v:
        r["Wv"] = tn_ranges(D, D, N)
    info = {k: (len(v), v[0][1] - v[0][0]) for k, v in r.items()}
    return Layout(r, set(), info)


def batch_layout(C_, D, Ns):
    """dsmil_backward_bags (and the dev, fold and row-sharded batch calls, per model / rank) over bags Ns."""
    total = sum(Ns)
    rps1 = rag_rows_per_chunk(KQ, D, total, False)
    chunks, row = [], 0
    for n in Ns:
        chunks += [(row + r0, row + min(n, r0 + rps1)) for r0 in range(0, n, rps1)]
        row += n
    S2 = tn_splits(KQ, KQ, total)
    rps2 = ceil_div(ceil_div(total, S2), TBK) * TBK
    G = bwd_bags_ctas(len(Ns), max(Ns))
    extra, start = set(), 0
    for n in Ns:
        extra |= {start + r for r in rowdot_cta_rows(n, G)}
        start += n
    r = {"W1": chunks, "W2": [(z * rps2, min(total, (z + 1) * rps2)) for z in range(S2)], "cs": colsum_ranges(total)}
    return Layout(r, extra, {"rps1": rps1, "chunks": len(chunks), "S2": S2, "rps2": rps2, "G": G})


def packed_probes(Ns, lay: Layout):
    rows, start = set(lay.extra), 0
    for n in Ns:
        rows |= {start, start + n - 1} | {start + r for r in (127, 128, 129) if r < n}
        start += n
    for rs in lay.ranges.values():
        rows |= {x for lo, hi in rs if hi > lo for x in (lo, hi - 1)}
    return rows


# --------------------------------------------------------------------------------------------------------- cases
@dataclass(frozen=True)
class Case:
    name: str
    route: str                             # single, bags, dev, models, shard_bags, shard_per_bag
    D: int
    C: int
    Ns: Tuple                              # bag sizes (models: one tuple per fold)
    nonlinear: bool = True
    passing_v: bool = False
    masked: bool = False                   # v's dropout mask (passing_v)
    misaligned: Tuple[int, ...] = ()       # bags 4 bytes past a 16-byte boundary
    tol_q: float = TOL_Q

    @property
    def seed(self):
        return sum(map(ord, self.name)) % 997

    @property
    def folds(self):
        return self.Ns if self.route == "models" else (self.Ns,)

    def params(self, m=0):
        return orc.random_params(self.D, self.C, 300 + self.seed + 17 * m, nonlinear=self.nonlinear,
                                 passing_v=self.passing_v, scale=1.5)

    def bags(self):
        flat = [n for f in self.folds for n in f]
        return [orc.synthetic_bag(n, self.D, 1000 * self.seed + b) for b, n in enumerate(flat)]

    def v_masks(self):
        if not self.masked:
            return [None] * len(self.Ns)
        rng = np.random.default_rng(77 + self.seed)
        return [((rng.random((n, self.D)) >= 0.25) / np.float32(0.75)).astype(np.float32) for n in self.Ns]

    def names(self, instance=True):
        return ((["Wi", "bi"] if instance else []) + ["W1", "b1"] + (["W2", "b2"] if self.nonlinear else []) +
                (["Wv", "bv"] if self.passing_v else []) + ["Wf", "bf"])

    def bar(self, name):
        return self.tol_q if name in Q_NAMES or name == "X" else TOL_P


SINGLE = [
    Case("tc_d512_c2_n10000", "single", 512, 2, (10000,)),
    Case("tc_d512_c6_n2049", "single", 512, 6, (2049,)),
    Case("tc_d2048_c2_n2305", "single", 2048, 2, (2305,)),
    Case("gen_d166_c1_n2049", "single", 166, 1, (2049,)),
    Case("gen_d230_linear_n2305", "single", 230, 2, (2305,), nonlinear=False),
    Case("pv_tc_d512_c2", "single", 512, 2, (2049,), passing_v=True),
    Case("pv_tc_d512_c2_mask", "single", 512, 2, (2049,), passing_v=True, masked=True),
    Case("pv_gen_d96_c2", "single", 96, 2, (4097,), passing_v=True),
    Case("pv_gen_d96_c2_mask", "single", 96, 2, (4097,), passing_v=True, masked=True),
    Case("pv_gen_d166_c1", "single", 166, 1, (2049,), passing_v=True),
    Case("pv_gen_d166_c1_mask", "single", 166, 1, (2049,), passing_v=True, masked=True),
    # gWi through k_gemv_tn<3> and <4> (tn_use_gemv: C <= 4, D % 4 == 0, D <= 1024) and the tile kernel one step past it
    Case("tc_d1024_c1_n2049", "single", 1024, 1, (2049,)),
    Case("tc_d1024_c3_n2049", "single", 1024, 3, (2049,)),
    Case("tc_d1024_c4_n2049", "single", 1024, 4, (2049,)),
    Case("gen_d1028_c4_n2049", "single", 1028, 4, (2049,)),
    Case("tc_d512_c8_n2049", "single", 512, 8, (2049,)),
    Case("tc_d4096_c1_n1025", "single", 4096, 1, (1025,)),
]
BAGS = [
    Case("bags_d512_rps128", "bags", 512, 2, (64, 63, 65, 1, 128, 129, 127, 2049)),
    Case("bags_d2048", "bags", 2048, 2, (256, 255, 257, 1, 3831)),
    Case("bags_d512_misaligned", "bags", 512, 2, (128, 127, 129, 1, 5319), misaligned=(4,)),
    Case("bags_gen_d166", "bags", 166, 1, (128, 127, 129, 1, 3000)),
    # gWi through k_gemv_tn_rag<3> and <4>, and k_gemm_tn_rag one step past D = 1024
    Case("bags_d1024_c1", "bags", 1024, 1, (128, 127, 129, 1, 2049)),
    Case("bags_d1024_c3", "bags", 1024, 3, (128, 127, 129, 1, 2049)),
    Case("bags_d1024_c4", "bags", 1024, 4, (128, 127, 129, 1, 2049)),
    Case("bags_gen_d1028_c4", "bags", 1028, 4, (128, 127, 129, 1, 2049)),
    Case("bags_d512_c8", "bags", 512, 8, (128, 127, 129, 1, 2049)),
]
DEV = [
    Case("dev_d512_rps128", "dev", 512, 2, (64, 63, 65, 1, 128, 129, 127, 2049)),
    Case("dev_gen_d166", "dev", 166, 1, (128, 127, 129, 1, 3000)),
    Case("dev_gen_d230_linear", "dev", 230, 2, (128, 127, 129, 1, 2305), nonlinear=False),
    Case("dev_d1024_c3", "dev", 1024, 3, (128, 127, 129, 1, 2049)),
    Case("dev_d1024_c4", "dev", 1024, 4, (128, 127, 129, 1, 2049)),
]
MODELS = [
    Case("models_m2", "models", 512, 2, ((64, 129, 2049), (128, 1, 700))),
    Case("models_m3", "models", 512, 2, ((127, 3000), (1, 128, 129), (65, 63, 513, 2))),
    Case("models_d1024_c3", "models", 1024, 3, ((129, 1500), (1, 128, 700))),
    Case("models_d1024_c4", "models", 1024, 4, ((129, 1500), (1, 128, 700))),
]
SHARD = [
    Case("shard_bags_d512", "shard_bags", 512, 2, (70, 69, 71, 3, 4097)),
    Case("shard_per_bag_d166", "shard_per_bag", 166, 2, (2049, 1)),
]
ALL = SINGLE + BAGS + DEV + MODELS + SHARD


def layouts(case: Case, G: int = 1):
    """[(global bag-order row of local row 0 of each bag, local bag sizes, Layout)] of every backward call the route
    makes: one per bag (single, per-bag shard), per batch, per fold, or per rank."""
    starts = np.cumsum([0] + [n for f in case.folds for n in f])
    out = []
    if case.route in ("single", "bags", "dev"):
        Ns = list(case.Ns)
        lay = (single_layout(case.C, case.D, Ns[0], case.nonlinear, case.passing_v) if case.route == "single"
               else batch_layout(case.C, case.D, Ns))
        out.append((list(starts[:len(Ns)]), Ns, lay))
    elif case.route == "models":
        b = 0
        for f in case.folds:
            out.append((list(starts[b:b + len(f)]), list(f), batch_layout(case.C, case.D, list(f))))
            b += len(f)
    else:
        for r in range(G):
            bounds = [orc.shard_bounds(n, G)[r] for n in case.Ns]
            Ns = [hi - lo for lo, hi in bounds]
            first = [int(starts[b]) + lo for b, (lo, hi) in enumerate(bounds)]
            if case.route == "shard_bags":
                out.append((first, Ns, batch_layout(case.C, case.D, Ns)))
            else:
                out += [([first[b]], [Ns[b]], single_layout(case.C, case.D, Ns[b], case.nonlinear, False))
                        for b in range(len(Ns)) if Ns[b] > 0]
    return out


def probe_mask(case: Case, G: int = 1):
    """bool [total rows] in bag order: the probe rows of every call of the route."""
    total = sum(n for f in case.folds for n in f)
    mask = np.zeros(total, bool)
    for firsts, Ns, lay in layouts(case, G):
        loc_start = np.cumsum([0] + Ns)
        for pr in packed_probes(Ns, lay):
            b = int(np.searchsorted(loc_start, pr, side="right") - 1)
            mask[firsts[b] + pr - loc_start[b]] = True
    return mask


def inject(A, mask):
    """A' = (A + a 1[probe]) / (1 + a n_probe) of one bag, a n_probe = PROBE_MASS; float32 as the device holds it."""
    n_probe = int(mask.sum())
    if n_probe == 0:
        return A
    a = PROBE_MASS / n_probe
    return ((A.astype(np.float64) + a * mask[:, None]) / (1.0 + PROBE_MASS)).astype(np.float32)


def upstream(case: Case, probes, with_ab: bool):
    """Per bag (d_classes [n, C], d_pred [C], d_A [n, C] | None, d_B [C, D] | None), float32."""
    rng = np.random.default_rng(5000 + case.seed)
    out, start = [], 0
    for n in (n for f in case.folds for n in f):
        dc = 1.0 + rng.standard_normal((n, case.C))
        dp = rng.standard_normal(case.C)
        dA = rng.standard_normal((n, case.C))
        dB = 1e-2 * rng.standard_normal((case.C, case.D))
        pm = probes[start:start + n]
        dA[pm] = PROBE_DA * np.sign(dA[pm]) * np.maximum(np.abs(dA[pm]), 1.0)
        f = lambda a: a.astype(np.float32)
        out.append((f(dc), f(dp), f(dA) if with_ab else None, f(dB) if with_ab else None))
        start += n
    return out


def takes_ab(case: Case):
    return case.route in ("single", "bags", "models")


# ----------------------------------------------------------------------------------- the maskable restatement
REDUCTIONS = ("t", "dqm", "W1", "b1", "W2", "b2", "Wv", "bv")


def restate(X, p: orc.Params, out: orc.FwdOut, d_classes, d_pred, d_A=None, d_B=None, v_mask=None, dtype=np.float64,
            w=None, t_shift=None, need_dX=False, inter=None):
    """orc.backward's algebra in plain numpy at `dtype`, every cross-row reduction weighted per row: w[name] [N] (default
    ones) for t = sum_n A dA, dq_max = dL^T Q and the sums of gW1, gb1, gW2, gb2, gWv, gbv (0 drops row n from that sum,
    2 counts it twice).  t_shift is added to t; `inter`, a dict, receives dA, t, dL, dz2, dz1, dzv and Xv."""
    f = dtype
    N = X.shape[0]
    w = w or {}
    rw = lambda k: np.asarray(w[k], f)[:, None] if k in w else 1
    X = np.asarray(X, f)
    P = p.astype(f)
    Cc = P.C
    A, Q = np.asarray(out.A, f), np.asarray(out.Q, f)
    H1 = None if out.H1 is None else np.asarray(out.H1, f)
    Bm = np.asarray(out.B, f).reshape(Cc, -1)
    idx = out.idx
    g = {}
    dc = np.zeros((N, Cc), f) if d_classes is None else np.asarray(d_classes, f)
    g["Wi"] = dc.T @ X
    g["bi"] = dc.sum(0)
    dp = np.zeros(Cc, f) if d_pred is None else np.asarray(d_pred, f).reshape(Cc)
    g["Wf"] = np.outer(dp, Bm.reshape(-1)).reshape(Cc, Cc, -1)
    g["bf"] = dp.copy()
    dB = (P.Wf.reshape(Cc, -1).T @ dp).reshape(Cc, -1)
    if d_B is not None:
        dB = dB + np.asarray(d_B, f).reshape(Cc, -1)
    V = np.asarray(out.V, f) if P.passing_v else X
    dA = V @ dB.T
    if d_A is not None:
        dA = dA + np.asarray(d_A, f)
    t = (rw("t") * A * dA).sum(0)
    if t_shift is not None:
        t = t + np.asarray(t_shift, f)
    dL = A * (dA - t) / f(orc.SCALE_F32)
    dQ = dL @ Q[idx]
    dqm = (rw("dqm") * dL).T @ Q
    np.add.at(dQ, idx, dqm)
    dz2 = None
    if P.nonlinear:
        dz2 = dQ * (1 - Q * Q)
        g["W2"] = (rw("W2") * dz2).T @ H1
        g["b2"] = (rw("b2") * dz2).sum(0)
        dz1 = (dz2 @ P.W2) * (H1 > 0)
    else:
        dz1 = dQ
    g["W1"] = (rw("W1") * dz1).T @ X
    g["b1"] = (rw("b1") * dz1).sum(0)
    dX = dc @ P.Wi if need_dX else None
    if need_dX:
        dX = dX + dz1 @ P.W1
    dzv = Xv = None
    if P.passing_v:
        Xv = X if v_mask is None else X * np.asarray(v_mask, f)
        dzv = (A @ dB) * (V > 0)
        g["Wv"] = (rw("Wv") * dzv).T @ Xv
        g["bv"] = (rw("bv") * dzv).sum(0)
        if need_dX:
            tv = dzv @ P.Wv
            dX = dX + (tv if v_mask is None else tv * np.asarray(v_mask, f))
    elif need_dX:
        dX = dX + A @ dB
    if need_dX:
        g["X"] = dX
    if inter is not None:
        inter.update(dA=dA, t=t, dL=dL, dz2=dz2, dz1=dz1, dzv=dzv, Xv=Xv, dQ=dQ)
    return g


# ------------------------------------------------------------------------------- CPU stand-in for the device saves
@functools.lru_cache(maxsize=4)
def cpu_inputs(case: Case, probes_on: bool, G: int = 1):
    """The fp32 oracle forward of every bag standing in for the device saves, A' injected when probes_on; per bag
    (params, X, FwdOut, upstream, v_mask)."""
    Xs, masks = case.bags(), case.v_masks()
    probes = probe_mask(case, G)
    ups = upstream(case, probes, takes_ab(case))
    out, b, start = [], 0, 0
    for m, f in enumerate(case.folds):
        p = case.params(m)
        for _ in f:
            X, vm = Xs[b], masks[b] if case.route == "single" else None
            o = orc.forward(X, p, dtype=np.float32, v_mask=vm)
            n = X.shape[0]
            A = inject(o.A, probes[start:start + n]) if probes_on else o.A
            fo = orc.FwdOut(None, None, A, o.B, o.idx, Q=o.Q, H1=o.H1, V=o.V)
            out.append((p, X, fo, ups[b], vm))
            b, start = b + 1, start + n
    return out, probes


def fold_of_bag(case: Case):
    return [m for m, f in enumerate(case.folds) for _ in f]


def sum_by_fold(case, per_bag, names):
    fb = fold_of_bag(case)
    return [{k: sum(g[k] for g, m in zip(per_bag, fb) if m == mm) for k in names} for mm in range(len(case.folds))]


# ===================================================================================== CPU part: no device needed
EXPECT = {
    # gW1 tile splits of 144 rows (74 of them), gW2's 79 of 128, colsum's 157 of 64, t's 40 blocks of 256
    "tc_d512_c2_n10000": lambda i: i["W1"] == (74, 144) and i["W2"] == (79, 128) and i["cs"] == (157, 64)
    and i["t"] == (40, 256) and i["dqm"] == (157, 64),
    # N = 2049: 17 gW1 / gW2 splits of 128 rows (the last holds one row), 33 column-sum splits of 63
    "tc_d512_c6_n2049": lambda i: i["W1"] == (17, 128) and i["dqm"] == (17, 128) and i["cs"] == (33, 63),
    "tc_d2048_c2_n2305": lambda i: i["W1"] == (18, 144) and i["W2"] == (19, 128) and i["dqm"] == (37, 63),
    "gen_d166_c1_n2049": lambda i: i["W1"] == (17, 128) and i["cs"] == (33, 63) and i["t"] == (9, 256),
    "gen_d230_linear_n2305": lambda i: i["W1"] == (19, 128) and "W2" not in i,
    "pv_tc_d512_c2": lambda i: i["Wv"] == (17, 128),
    "pv_tc_d512_c2_mask": lambda i: i["Wv"] == (17, 128),
    "pv_gen_d96_c2": lambda i: i["Wv"] == (33, 128) and i["cs"] == (65, 64),
    "pv_gen_d96_c2_mask": lambda i: i["Wv"] == (33, 128),
    "pv_gen_d166_c1": lambda i: i["Wv"] == (17, 128),
    "pv_gen_d166_c1_mask": lambda i: i["Wv"] == (17, 128),
    # gW1 chunks of 128 rows over bags of 127, 128 and 129; k_bwd_rowdot_b with 33 CTAs per bag
    "bags_d512_rps128": lambda i: i["rps1"] == 128 and i["G"] == 33,
    "bags_d2048": lambda i: i["rps1"] == 256 and i["G"] == 60,
    "bags_d512_misaligned": lambda i: i["rps1"] == 128 and i["G"] == 84,
    "bags_gen_d166": lambda i: i["rps1"] == 128 and i["G"] == 47,
    "dev_d512_rps128": lambda i: i["rps1"] == 128 and i["G"] == 33,
    "dev_gen_d166": lambda i: i["rps1"] == 128 and i["G"] == 47,
    "dev_gen_d230_linear": lambda i: i["rps1"] == 128 and i["G"] == 37,
}


@pytest.mark.parametrize("case", [c for c in ALL if c.name in EXPECT], ids=lambda c: c.name)
def test_case_sits_on_its_split_boundary(case):
    (_, Ns, lay), = layouts(case)
    assert EXPECT[case.name](lay.info), (case.name, lay.info)
    if case.route in ("bags", "dev"):
        rps = lay.info["rps1"]
        assert {rps - 1, rps, rps + 1, 1} <= set(Ns), (case.name, rps, Ns)


def test_cases_reach_every_gwi_form():
    """gWi = d_classes^T X streams through k_gemv_tn<C> (one bag) or k_gemv_tn_rag<C> (a batch) for C = 1..4 while
    tn_use_gemv holds, and through the tile kernels one multiple of 4 past D = 1024 at the same C."""
    for route in ("single", "bags"):
        cases = [c for c in ALL if c.route == route]
        assert {c.C for c in cases if tn_use_gemv(c.C, c.D)} >= {1, 2, 3, 4}, route
        assert any(c.C == 4 and c.D == 1024 for c in cases) and any(c.C == 4 and c.D == 1028 for c in cases), route
    assert tn_use_gemv(4, 1024) and not tn_use_gemv(4, 1028)
    assert {c.C for c in ALL} >= {3, 4, 8} and any(c.D == 4096 and c.route == "single" for c in ALL)


def test_fold_and_rank_layouts_cover_every_row_once():
    """Every packed-row split mirrored here tiles its rows exactly once; each fold has its own chunking; a rank of the
    per-bag sharded case holds no row of the one-row bag."""
    for case in ALL:
        for G in ((1, 2, 3) if case.route.startswith("shard") else (1,)):
            for _, Ns, lay in layouts(case, G):
                total = sum(Ns) if case.route != "single" and case.route != "shard_per_bag" else Ns[0]
                for k, rs in lay.ranges.items():
                    cover = np.zeros(total, np.int64)
                    for lo, hi in rs:
                        cover[lo:max(lo, hi)] += 1
                    assert np.all(cover == 1), (case.name, G, k)
    assert len({lay.info["G"] for _, _, lay in layouts(MODELS[1])}) == len(MODELS[1].folds)
    assert any(hi == lo for lo, hi in orc.shard_bounds(SHARD[1].Ns[1], 2))
    assert all(hi - lo >= 1 for n in SHARD[0].Ns for lo, hi in orc.shard_bounds(n, 3))


def test_restatement_in_fp64_is_the_oracle_backward():
    for case in (SINGLE[0], SINGLE[4], SINGLE[6], BAGS[3]):
        for p, X, fo, (dc, dp, dA, dB), vm in cpu_inputs(case, True)[0][:2]:
            want = orc.backward(X, p, fo, dc, dp, d_A=dA, d_B=dB, need_dX=True, v_mask=vm)
            got = restate(X, p, fo, dc, dp, dA, dB, vm, need_dX=True)
            assert got.keys() == want.keys()
            for k in want:
                assert rel_to_max(got[k], want[k]) <= 1e-12, (case.name, k)


def _cases_with_G():
    """The routes that take d_A.  Without it (dev, row-sharded) dA = X dB^T varies little over the rows, some probe rows
    have dA ~ t and so dL ~ 0, and no weight on A makes them count: there the A injection still runs, unproven."""
    return [(c, 1) for c in ALL if takes_ab(c)]


def _qmove_through_critical_rows(p, X, fo, inter, delta):
    """Moves of W1, b1, W2, b2 when dq_max changes by delta [C, 128]: it enters dQ at the critical rows only."""
    mv = {k: 0.0 for k in ("W1", "b1", "W2", "b2")}
    for k, r in enumerate(fo.idx):
        d = delta[k].astype(np.float64)
        if p.nonlinear:
            Qr, H1r = fo.Q[r].astype(np.float64), fo.H1[r].astype(np.float64)
            dz2 = d * (1 - Qr * Qr)
            mv["W2"] = mv["W2"] + np.outer(dz2, H1r)
            mv["b2"] = mv["b2"] + dz2
            d = (dz2 @ p.W2.astype(np.float64)) * (H1r > 0)
        mv["W1"] = mv["W1"] + np.outer(d, X[r].astype(np.float64))
        mv["b1"] = mv["b1"] + d
    return mv


@pytest.mark.parametrize("case,G", _cases_with_G(), ids=lambda v: v.name if isinstance(v, Case) else f"G{v}")
def test_one_lost_or_repeated_probe_row_moves_a_checked_gradient_past_20x_its_bar(case, G):
    """For every probe row and every reduction it enters (t, dq_max, gW1, gb1, gW2, gb2, gWv, gbv), dropping the row
    from that reduction moves some checked gradient by more than 20x its bar (doubling moves it by the same amount
    the other way: every gradient is affine in each reduction's row weights).  The moves come from the row's own terms
    (and, for t, the response to a unit shift of t); the row-maskable restatement confirms them on a few rows."""
    data, probes = cpu_inputs(case, True, G)
    names = case.names(instance=False)
    bases = [restate(X, p, fo, *u, v_mask=vm) for p, X, fo, u, vm in data]
    fold_base = sum_by_fold(case, bases, names)
    fb = fold_of_bag(case)
    weakest = {}
    start = 0
    for b, ((p, X, fo, u, vm), base) in enumerate(zip(data, bases)):
        n = X.shape[0]
        tot = fold_base[fb[b]]
        inter = {}
        restate(X, p, fo, *u, v_mask=vm, inter=inter)
        resp = []                                    # gradient response to t_k += 1
        for k in range(case.C):
            e = np.zeros(case.C)
            e[k] = 1.0
            g = restate(X, p, fo, *u, v_mask=vm, t_shift=e)
            resp.append({nm: g[nm] - base[nm] for nm in names})
        rel = lambda mv, nm: float(np.max(np.abs(mv))) / float(np.max(np.abs(tot[nm]))) / case.bar(nm)
        X64 = X.astype(np.float64)
        # a one-row bag has A = 1, so dL = A (dA - t) = 0: it adds nothing to any q.* sum, and a lost row of it nothing
        for r in np.nonzero(probes[start:start + n])[0] if n > 1 else ():
            share_t = fo.A[r].astype(np.float64) * inter["dA"][r]
            moves = {"t": max(rel(sum(share_t[k] * resp[k][nm] for k in range(case.C)), nm) for nm in names),
                     "W1": rel(np.outer(inter["dz1"][r], X64[r]), "W1"), "b1": rel(inter["dz1"][r], "b1")}
            dq = _qmove_through_critical_rows(p, X, fo, inter, np.outer(inter["dL"][r], fo.Q[r].astype(np.float64)))
            moves["dqm"] = max(rel(dq[nm], nm) for nm in dq if nm in names)
            if case.nonlinear:
                moves["W2"] = rel(np.outer(inter["dz2"][r], fo.H1[r].astype(np.float64)), "W2")
                moves["b2"] = rel(inter["dz2"][r], "b2")
            if case.passing_v:
                moves["Wv"] = rel(np.outer(inter["dzv"][r], inter["Xv"][r]), "Wv")
                moves["bv"] = rel(inter["dzv"][r], "bv")
            for red, mv in moves.items():
                if mv < weakest.get(red, (np.inf,))[0]:
                    weakest[red] = (mv, b, int(r))
        start += n
    bad = {k: v for k, v in weakest.items() if not v[0] > SENSITIVITY}
    assert not bad, (case.name, G, bad)
    # the shortcut above against the maskable restatement: drop the weakest row from each reduction
    for red, (_, b, r) in weakest.items():
        p, X, fo, u, vm = data[b]
        w = np.ones(X.shape[0])
        w[r] = 0.0
        got = restate(X, p, fo, *u, v_mask=vm, w={red: w})
        moved = max(float(np.max(np.abs(got[nm] - bases[b][nm]))) / float(np.max(np.abs(fold_base[fb[b]][nm]))) /
                    case.bar(nm) for nm in names)
        assert moved > SENSITIVITY, (case.name, red, moved, weakest[red])


def kappa(terms):
    """max_j sum_n |term[n, j]| / max_j |sum_n term[n, j]|: the amplification of a summation's rounding."""
    terms = np.asarray(terms, np.float64).reshape(terms.shape[0], -1)
    return float(np.abs(terms).sum(0).max() / max(np.abs(terms.sum(0)).max(), 1e-300))


@pytest.mark.parametrize("case", ALL, ids=lambda c: c.name)
@pytest.mark.parametrize("probes_on", [False, True], ids=["plain", "probes"])
def test_upstream_conditions_every_checked_sum_and_the_fp32_restatement_fits_the_bars(case, probes_on):
    """kappa of the column sums (gbi, gb1, gb2, gbv) and of the softmax backward's dA - t stays below KAPPA_MAX; the
    fp32 restatement on the same inputs stays under each bar (the device then has headroom only if its error is near
    that of an fp32 evaluation of the same algebra)."""
    data, _ = cpu_inputs(case, probes_on)
    names = case.names()
    g64, g32, worst = [], [], {}
    for p, X, fo, u, vm in data:
        inter = {}
        g64.append(restate(X, p, fo, *u, v_mask=vm, need_dX=True, inter=inter))
        g32.append(restate(X, p, fo, *u, v_mask=vm, dtype=np.float32, need_dX=True))
        if X.shape[0] < 64:
            continue
        k = {"bi": kappa(u[0]), "b1": kappa(inter["dz1"]), "dA-t": float(np.abs(inter["dA"]).max() /
                                                                          np.abs(inter["dA"] - inter["t"]).max())}
        if case.nonlinear:
            k["b2"] = kappa(inter["dz2"])
        if case.passing_v:
            k["bv"] = kappa(inter["dzv"])
        for nm, v in k.items():
            worst[nm] = max(worst.get(nm, 0.0), v)
    assert all(v <= (KAPPA_UPSTREAM if k in ("bi", "dA-t") else KAPPA_SOFTMAX) for k, v in worst.items()), \
        (case.name, worst)
    for want, got in zip(sum_by_fold(case, g64, names), sum_by_fold(case, g32, names)):
        errs = {k: rel_to_max(got[k], want[k]) for k in names}
        assert all(errs[k] < case.bar(k) for k in names), (case.name, errs)
    for a, b in zip(g32, g64):
        assert rowwise_err(a["X"], b["X"]) < case.bar("X"), case.name


# ========================================================================================== GPU part (one H100)
def _np(t):
    return t.detach().cpu().numpy()


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _pack(p):
    from dsmil_wsi_b200 import functional as Fn
    return Fn.ParamPack(*[_t(a) for a in (p.Wi, p.bi, p.W1, p.b1, p.W2, p.b2, p.Wv, p.bv, p.Wf, p.bf)])


def _ws(nbytes):
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device="cuda")


def _nan(*s):
    return torch.full(s, float("nan"), device="cuda")


class _Grads:
    """Device gradient buffers of one parameter set (NaN-filled: an unwritten gradient fails the check)."""

    def __init__(self, case: Case, rows=0):
        D, Cc = case.D, case.C
        shapes = {"Wi": (Cc, D), "bi": (Cc,), "W1": (KQ, D), "b1": (KQ,), "Wf": (Cc, Cc, D), "bf": (Cc,)}
        if case.nonlinear:
            shapes.update(W2=(KQ, KQ), b2=(KQ,))
        if case.passing_v:
            shapes.update(Wv=(D, D), bv=(D,))
        self.t = {k: _nan(*s) for k, s in shapes.items()}
        self.gX = _nan(rows, D) if rows else None

    def struct(self, gX=None):
        from dsmil_wsi_b200 import _lib
        g = lambda k: _ptr(self.t.get(k))
        return _lib.DsmilGrads(*[g(k) for k in ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf")],
                               _ptr(gX if gX is not None else self.gX))

    def host(self):
        return {k: _np(v) for k, v in self.t.items()}


def _bag_tensor(X, misaligned):
    if not misaligned:
        return torch.from_numpy(X).cuda()
    buf = torch.zeros(X.size + 1, device="cuda")
    buf[1:].copy_(torch.from_numpy(X).reshape(-1).cuda())
    x = buf[1:].view(X.shape)
    assert x.data_ptr() % 16 == 4
    return x


def _oracle_crit(X, p):
    c = X.astype(np.float64) @ p.Wi.astype(np.float64).T + p.bi
    s = np.sort(c, axis=0)
    if c.shape[0] > 1:                     # tie-free: the device's fp32 scores pick the same row
        assert np.all(s[-1] - s[-2] > 1e-5 * np.abs(c).max())
    return orc.critical_instances(c)


def _check(case, what, got: Dict[str, np.ndarray], want: Dict[str, np.ndarray], gX=None, gX_want=None):
    errs = {k: rel_to_max(got[k], want[k]) for k in want}
    if gX is not None:
        errs["X"] = max(rowwise_err(a, b) for a, b in zip(gX, gX_want))
    print(f"conditioned {case.route} {case.name} {what}: " + " ".join(f"{k}={e:.2e}" for k, e in errs.items()))
    bad = {k: (e, case.bar(k)) for k, e in errs.items() if not e <= case.bar(k)}
    assert not bad, (what, case.name, bad)


def _saves_and_reference(case, p, Xs, host, probes, ups, crit, vms, need_dX, first_bag=0):
    """Per-bag host saves -> A' injection and the fp64 backward on exactly those inputs.  host: per bag dict of A, B,
    Q, H1, V.  Returns (per-bag A' arrays, summed gradients, per-bag gX)."""
    names = case.names()
    A_new, per = [], []
    starts = np.cumsum([0] + [n for f in case.folds for n in f])
    for j, (X, h) in enumerate(zip(Xs, host)):
        b = first_bag + j
        n = X.shape[0]
        A = inject(h["A"], probes[starts[b]:starts[b] + n]) if probes is not None else h["A"]
        A_new.append(A)
        V = h["V"] if case.passing_v else X          # identity v: V is the bag itself
        fo = orc.FwdOut(None, None, A, h["B"], crit[j], Q=h["Q"], H1=h.get("H1"), V=V)
        dc, dp, dA, dB = ups[b]
        per.append(orc.backward(X, p, fo, dc, dp, d_A=dA, d_B=dB, need_dX=need_dX, v_mask=vms[j]))
    want = {k: sum(g[k] for g in per) for k in names}
    return A_new, want, [g["X"] for g in per] if need_dX else None


def _probe_arg(case, probes_on, G=1):
    return probe_mask(case, G) if probes_on else None


def run_single(case: Case, probes_on: bool):
    from dsmil_wsi_b200 import _lib
    lib = _lib.load()
    p = case.params()
    P = _pack(p)
    X = case.bags()[0]
    vm = case.v_masks()[0]
    N, Cc, D = X.shape[0], case.C, case.D
    x = torch.from_numpy(X).cuda()
    m = _t(vm)
    xv = None if m is None else x * m
    out = dict(classes=_nan(N, Cc), pred=_nan(1, Cc), A=_nan(N, Cc), B=_nan(1, Cc, D), Q=_nan(N, KQ),
               H1=_nan(N, KQ) if case.nonlinear else None, V=_nan(N, D) if case.passing_v else None)
    crit = torch.full((Cc,), -7, dtype=torch.int64, device="cuda")
    ws = _ws(lib.dsmil_forward_workspace_bytes(P.ref, N))
    rc = lib.dsmil_forward(P.ref, x.data_ptr(), _ptr(xv), N, *[_ptr(out[k]) for k in ("classes", "pred", "A", "B")],
                           crit.data_ptr(), _ptr(out["Q"]), _ptr(out["H1"]), _ptr(out["V"]), ws.data_ptr(), ws.numel(),
                           _stream())
    assert rc == 0, lib.dsmil_last_error()
    crit_h = _np(crit)
    assert np.array_equal(crit_h, _oracle_crit(X, p)), case.name
    host = [{k: _np(v) for k, v in out.items() if v is not None}]
    probes = _probe_arg(case, probes_on)
    ups = upstream(case, probe_mask(case), True)
    (A_new,), want, gX_want = _saves_and_reference(case, p, [X], host, probes, ups, [crit_h], [vm], True)
    out["A"].copy_(torch.from_numpy(A_new))
    dc, dp, dA, dB = (_t(a) for a in ups[0])
    g = _Grads(case, N)
    ws = _ws(lib.dsmil_backward_workspace_bytes(P.ref, N, 1))
    G = g.struct()
    rc = lib.dsmil_backward(P.ref, x.data_ptr(), _ptr(xv), N, _ptr(out["Q"]), _ptr(out["H1"]), _ptr(out["V"]),
                            _ptr(out["A"]), _ptr(out["B"]), crit.data_ptr(), _ptr(dc), _ptr(dp), _ptr(dA), _ptr(dB),
                            C.byref(G), _ptr(m), ws.data_ptr(), ws.numel(), _stream())
    assert rc == 0, lib.dsmil_last_error()
    torch.cuda.synchronize()
    _check(case, "probes" if probes_on else "plain", g.host(), want, [_np(g.gX)], gX_want)


def _unpack(t, Ns, row0=0):
    out, lo = [], row0
    for n in Ns:
        out.append(t[lo:lo + n])
        lo += n
    return out


def run_bags(case: Case, probes_on: bool):
    """dsmil_forward_bags_train + dsmil_backward_bags (with gX, d_A and d_B)."""
    from dsmil_wsi_b200 import _lib
    lib = _lib.load()
    p = case.params()
    P = _pack(p)
    Xs = case.bags()
    Ns = list(case.Ns)
    nb, total, Cc, D = len(Ns), sum(Ns), case.C, case.D
    xs = [_bag_tensor(X, b in case.misaligned) for b, X in enumerate(Xs)]
    c_X, c_N = (C.c_void_p * nb)(*[x.data_ptr() for x in xs]), (C.c_int64 * nb)(*Ns)
    o = dict(classes=_nan(total, Cc), pred=_nan(nb, Cc), A=_nan(total, Cc), B=_nan(nb, Cc, D), Q=_nan(total, KQ),
             H1=_nan(total, KQ) if case.nonlinear else None)
    crit = torch.full((nb, Cc), -7, dtype=torch.int64, device="cuda")
    ws = _ws(lib.dsmil_forward_bags_train_workspace_bytes(P.ref, c_N, nb))
    rc = lib.dsmil_forward_bags_train(P.ref, c_X, c_N, nb, *[_ptr(o[k]) for k in ("classes", "pred", "A", "B")],
                                      crit.data_ptr(), _ptr(o["Q"]), _ptr(o["H1"]), ws.data_ptr(), ws.numel(), _stream())
    assert rc == 0, lib.dsmil_last_error()
    crit_h = _np(crit)
    host = _host_bags(o, Ns, 0, 0)
    for b, X in enumerate(Xs):
        assert np.array_equal(crit_h[b], _oracle_crit(X, p)), (case.name, b)
    ups = upstream(case, probe_mask(case), True)
    A_new, want, gX_want = _saves_and_reference(case, p, Xs, host, _probe_arg(case, probes_on), ups, list(crit_h),
                                                [None] * nb, True)
    o["A"].copy_(torch.from_numpy(np.concatenate(A_new)))
    dc, dA = (_t(np.concatenate([u[i] for u in ups])) for i in (0, 2))
    dp, dB = (_t(np.stack([u[i] for u in ups])) for i in (1, 3))
    g = _Grads(case, total)
    G = g.struct()
    ws = _ws(lib.dsmil_backward_bags_workspace_bytes(P.ref, c_N, nb, 1))
    rc = lib.dsmil_backward_bags(P.ref, c_X, c_N, nb, _ptr(o["Q"]), _ptr(o["H1"]), _ptr(o["A"]), _ptr(o["B"]),
                                 crit.data_ptr(), _ptr(dc), _ptr(dp), _ptr(dA), _ptr(dB), C.byref(G), ws.data_ptr(),
                                 ws.numel(), _stream())
    assert rc == 0, lib.dsmil_last_error()
    torch.cuda.synchronize()
    _check(case, "probes" if probes_on else "plain", g.host(), want, [_np(t) for t in _unpack(g.gX, Ns)], gX_want)


def _host_bags(o, Ns, row0, b0):
    """Per-bag host copies of packed saves: rows from row0, bags from b0."""
    h = {k: _np(v) for k, v in o.items() if v is not None}
    out, lo = [], row0
    for j, n in enumerate(Ns):
        d = {k: h[k][lo:lo + n] for k in ("A", "Q", "H1") if k in h}
        d["B"] = h["B"][b0 + j]
        out.append(d)
        lo += n
    return out


def _slots(Xs, D):
    max_rows = max(X.shape[0] for X in Xs)
    slots = torch.zeros(len(Xs), max_rows, D, device="cuda")
    for b, X in enumerate(Xs):
        slots[b, :X.shape[0]].copy_(torch.from_numpy(X))
    return slots, max_rows


def run_dev(case: Case, probes_on: bool):
    """The capture-safe pair (dsmil_forward_bags_train_dev / dsmil_backward_bags_dev or the dsmil_generic_* forms) over
    [nb, max_rows, D] slots: d_classes has nb * max_rows rows, a large dead tail after the live ones; no d_A, d_B, gX."""
    from dsmil_wsi_b200 import _lib
    lib = _lib.load()
    p = case.params()
    P = _pack(p)
    pre = "dsmil_" if lib.dsmil_shard_bags_supported(P.ref) else "dsmil_generic_"
    assert (pre == "dsmil_") == (case.D % 128 == 0)
    Xs = case.bags()
    Ns = list(case.Ns)
    nb, total, Cc, D = len(Ns), sum(Ns), case.C, case.D
    slots, max_rows = _slots(Xs, D)
    rows = nb * max_rows
    xs = slots.data_ptr() + 4 * max_rows * D * torch.arange(nb, dtype=torch.int64, device="cuda")
    Nd = torch.tensor(Ns, dtype=torch.int64, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    o = dict(classes=_nan(rows, Cc), pred=_nan(nb, Cc), A=_nan(rows, Cc), B=_nan(nb, Cc, D), Q=_nan(rows, KQ),
             H1=_nan(rows, KQ))
    crit = torch.full((nb, Cc), -7, dtype=torch.int64, device="cuda")
    ws = _ws(getattr(lib, pre + "forward_bags_train_dev_workspace_bytes")(P.ref, nb, max_rows))
    rc = getattr(lib, pre + "forward_bags_train_dev")(P.ref, xs.data_ptr(), Nd.data_ptr(), nb, max_rows,
                                                      *[_ptr(o[k]) for k in ("classes", "pred", "A", "B")],
                                                      crit.data_ptr(), _ptr(o["Q"]), _ptr(o["H1"]), status.data_ptr(),
                                                      ws.data_ptr(), ws.numel(), _stream())
    assert rc == 0, lib.dsmil_last_error()
    crit_h = _np(crit)
    for b, X in enumerate(Xs):
        assert np.array_equal(crit_h[b], _oracle_crit(X, p)), (case.name, b)
    if not case.nonlinear:
        o["H1"] = None
    host = _host_bags(o, Ns, 0, 0)
    ups = upstream(case, probe_mask(case), False)
    A_new, want, _ = _saves_and_reference(case, p, Xs, host, _probe_arg(case, probes_on), ups, list(crit_h),
                                          [None] * nb, False)
    o["A"][:total].copy_(torch.from_numpy(np.concatenate(A_new)))
    dc = torch.full((rows, Cc), 1.0e4, device="cuda")
    dc[:total] = _t(np.concatenate([u[0] for u in ups]))
    dp = _t(np.stack([u[1] for u in ups]))
    g = _Grads(case)
    G = g.struct()
    ws = _ws(getattr(lib, pre + "backward_bags_dev_workspace_bytes")(P.ref, nb, max_rows))
    rc = getattr(lib, pre + "backward_bags_dev")(P.ref, xs.data_ptr(), Nd.data_ptr(), nb, max_rows, _ptr(o["Q"]),
                                                 _ptr(o["H1"]), _ptr(o["A"]), _ptr(o["B"]), crit.data_ptr(), dc.data_ptr(),
                                                 dp.data_ptr(), None, None, C.byref(G), status.data_ptr(), ws.data_ptr(),
                                                 ws.numel(), _stream())
    assert rc == 0, lib.dsmil_last_error()
    torch.cuda.synchronize()
    assert int(status) == 0
    _check(case, "probes" if probes_on else "plain", g.host(), want)


def run_models(case: Case, probes_on: bool, dev: bool):
    """The fold step (dsmil_forward_bags_models_train / dsmil_backward_bags_models, or their _dev forms over slots):
    each model's gradients against the fp64 backward over its own bags."""
    from dsmil_wsi_b200 import _lib
    lib = _lib.load()
    M = len(case.folds)
    ps = [case.params(m) for m in range(M)]
    packs = [_pack(p) for p in ps]
    c_ps = (_lib.DsmilParams * M)(*[P.struct for P in packs])
    assert lib.dsmil_models_supported(c_ps, M)
    nbs = [len(f) for f in case.folds]
    Ns = [n for f in case.folds for n in f]
    ne, Cc, D = len(Ns), case.C, case.D
    Xs = case.bags()
    c_nb = (C.c_int32 * M)(*nbs)
    if dev:
        slots, max_rows = _slots(Xs, D)
        rows = ne * max_rows
        xs = slots.data_ptr() + 4 * max_rows * D * torch.arange(ne, dtype=torch.int64, device="cuda")
        Nd = torch.tensor(Ns, dtype=torch.int64, device="cuda")
        status = torch.zeros(M, dtype=torch.int32, device="cuda")
        row0 = [max_rows * sum(nbs[:m]) for m in range(M)]      # each model's capacity block
    else:
        xts = [torch.from_numpy(X).cuda() for X in Xs]
        c_X, c_N = (C.c_void_p * ne)(*[x.data_ptr() for x in xts]), (C.c_int64 * ne)(*Ns)
        rows = sum(Ns)
        row0 = list(np.cumsum([0] + [sum(f) for f in case.folds])[:M])
    o = dict(classes=_nan(rows, Cc), pred=_nan(ne, Cc), A=_nan(rows, Cc), B=_nan(ne, Cc, D), Q=_nan(rows, KQ),
             H1=_nan(rows, KQ))
    crit = torch.full((ne, Cc), -7, dtype=torch.int64, device="cuda")
    outs = [_ptr(o[k]) for k in ("classes", "pred", "A", "B")] + [crit.data_ptr(), _ptr(o["Q"]), _ptr(o["H1"])]
    if dev:
        ws = _ws(lib.dsmil_forward_bags_models_train_dev_workspace_bytes(c_ps, M, c_nb, max_rows))
        rc = lib.dsmil_forward_bags_models_train_dev(c_ps, M, xs.data_ptr(), Nd.data_ptr(), c_nb, max_rows, *outs,
                                                     status.data_ptr(), ws.data_ptr(), ws.numel(), _stream())
    else:
        ws = _ws(lib.dsmil_forward_bags_models_train_workspace_bytes(c_ps, M, c_N, c_nb))
        rc = lib.dsmil_forward_bags_models_train(c_ps, M, c_X, c_N, c_nb, *outs, ws.data_ptr(), ws.numel(), _stream())
    assert rc == 0, lib.dsmil_last_error()
    crit_h = _np(crit)
    ups = upstream(case, probe_mask(case), not dev)
    probes = _probe_arg(case, probes_on)
    wants, gX_wants, b0 = [], [], 0
    for m, f in enumerate(case.folds):
        host = _host_bags(o, list(f), row0[m], b0)
        for j in range(len(f)):
            assert np.array_equal(crit_h[b0 + j], _oracle_crit(Xs[b0 + j], ps[m])), (case.name, m, j)
        A_new, want, gXw = _saves_and_reference(case, ps[m], Xs[b0:b0 + len(f)], host, probes, ups,
                                                list(crit_h[b0:b0 + len(f)]), [None] * len(f), not dev, first_bag=b0)
        o["A"][row0[m]:row0[m] + sum(f)].copy_(torch.from_numpy(np.concatenate(A_new)))
        wants.append(want)
        gX_wants.append(gXw)
        b0 += len(f)
    dp = _t(np.stack([u[1] for u in ups]))
    if dev:
        dc = torch.full((rows, Cc), 1.0e4, device="cuda")
        b0 = 0
        for m, f in enumerate(case.folds):
            dc[row0[m]:row0[m] + sum(f)] = _t(np.concatenate([u[0] for u in ups[b0:b0 + len(f)]]))
            b0 += len(f)
        dA = dB = None
    else:
        dc, dA = (_t(np.concatenate([u[i] for u in ups])) for i in (0, 2))
        dB = _t(np.stack([u[3] for u in ups]))
    gs = [_Grads(case) for _ in range(M)]
    gX = None if dev else _nan(rows, D)
    grads = (_lib.DsmilGrads * M)(*[g.struct(None if dev else gX[row0[m]:row0[m] + sum(case.folds[m])])
                                    for m, g in enumerate(gs)])
    ins = [_ptr(o["Q"]), _ptr(o["H1"]), _ptr(o["A"]), _ptr(o["B"]), crit.data_ptr(), _ptr(dc), _ptr(dp), _ptr(dA),
           _ptr(dB), grads]
    if dev:
        ws = _ws(lib.dsmil_backward_bags_models_dev_workspace_bytes(c_ps, M, c_nb, max_rows))
        rc = lib.dsmil_backward_bags_models_dev(c_ps, M, xs.data_ptr(), Nd.data_ptr(), c_nb, max_rows, *ins,
                                                status.data_ptr(), ws.data_ptr(), ws.numel(), _stream())
    else:
        ws = _ws(lib.dsmil_backward_bags_models_workspace_bytes(c_ps, M, c_N, c_nb, 1))
        rc = lib.dsmil_backward_bags_models(c_ps, M, c_X, c_N, c_nb, *ins, ws.data_ptr(), ws.numel(), _stream())
    assert rc == 0, lib.dsmil_last_error()
    torch.cuda.synchronize()
    if dev:
        assert _np(status).tolist() == [0] * M
    for m, f in enumerate(case.folds):
        what = f"{'dev' if dev else 'eager'} model {m} {'probes' if probes_on else 'plain'}"
        gx = None if dev else [_np(t) for t in _unpack(gX, list(f), row0[m])]
        _check(case, what, gs[m].host(), wants[m], gx, gX_wants[m])


class _SwapRank:
    """A logical rank of virtual_sharded_train_step_bags that keeps its saves (Q, H1, q_max) and, before the backward's
    first phase, replaces its rows of A in place (bwd2 then reads the same A) by `swap(rank, A)`."""

    def __init__(self, inner, swap):
        self.inner, self.swap = inner, swap

    def begin(self, X_locals, row_offsets):
        self.Ns, self.offs = [int(x.shape[0]) for x in X_locals], [int(o) for o in row_offsets]
        return self.inner.begin(X_locals, row_offsets)

    def phase1_train(self):
        r = self.inner.phase1_train()
        self.Q, self.H1 = r[1], r[2]
        return r

    def phase2_train(self, Q, cands_all, G):
        r = self.inner.phase2_train(Q, cands_all, G)
        self.qmax = r[2]
        return r

    def phase3_train(self, recs_all, G, A):
        return self.inner.phase3_train(recs_all, G, A)

    def bwd1(self, xs, A, B, d_classes, d_pred):
        self.swap(self, A)
        return self.inner.bwd1(xs, A, B, d_classes, d_pred)

    def bwd2(self, xs, A, dA, t, Q):
        return self.inner.bwd2(xs, A, dA, t, Q)

    def bwd3(self, xs, row_offsets, Q, H1, dL, dqm, qmax, crit):
        return self.inner.bwd3(xs, row_offsets, Q, H1, dL, dqm, qmax, crit)


def run_shard(case: Case, ops: str, G: int, probes_on: bool):
    """virtual_sharded_train_step_bags over G logical ranks on one device; the reference is orc.backward_sharded on the
    ranks' saved Q, H1 and A' assembled in bag order."""
    from dsmil_wsi_b200.sharded import CudaShardBagOps, CudaShardOps, PerBagShardOps, virtual_sharded_train_step_bags
    p = case.params()
    P = _pack(p)
    params = P.tensors
    Xs = case.bags()
    starts = np.cumsum([0] + list(case.Ns))
    probes = probe_mask(case, G)
    ups = upstream(case, probes, False)
    total = int(starts[-1])
    A_bag, Q_bag = np.full((total, case.C), np.nan, np.float32), np.full((total, KQ), np.nan, np.float32)
    H1_bag = np.full((total, KQ), np.nan, np.float32)

    def swap(rank, A):
        live = sum(rank.Ns)
        A_h, Q_h, H_h = _np(A[:live]), _np(rank.Q[:live]), _np(rank.H1[:live])
        lo = 0
        for b, (n, off) in enumerate(zip(rank.Ns, rank.offs)):
            g = slice(int(starts[b]) + off, int(starts[b]) + off + n)
            a = A_h[lo:lo + n]
            if probes_on:          # the bag's probe count over all ranks sets a; A' needs no other rank's A
                n_probe = int(probes[starts[b]:starts[b + 1]].sum())
                a = ((a.astype(np.float64) + PROBE_MASS / n_probe * probes[g][:, None]) /
                     (1.0 + PROBE_MASS)).astype(np.float32)
                A_h[lo:lo + n] = a
            A_bag[g], Q_bag[g], H1_bag[g] = a, Q_h[lo:lo + n], H_h[lo:lo + n]
            lo += n
        A[:live].copy_(torch.from_numpy(A_h))

    make = {"bag_ops": lambda: CudaShardBagOps(params), "bag_dev_ops": lambda: _DevRank(params),
            "per_bag_ops": lambda: PerBagShardOps(CudaShardOps(params))}[ops]
    ranks = []

    def make_rank():
        ranks.append(_SwapRank(make(), swap))
        return ranks[-1]

    dc = _t(np.concatenate([u[0] for u in ups]))
    dp = _t(np.stack([u[1] for u in ups]))
    xs = [torch.from_numpy(X).cuda() for X in Xs]
    (_, _, _, B, crit), grads = virtual_sharded_train_step_bags(make_rank, xs, G, lambda c, pr, cr: (dc, dp))
    torch.cuda.synchronize()
    if ops == "bag_dev_ops":
        assert all(int(r.inner.status) == 0 for r in ranks)
    crit_h = _np(crit).reshape(len(Xs), -1)
    B_h = _np(B).reshape(len(Xs), case.C, case.D)
    names = ["Wi", "bi", "W1", "b1", "W2", "b2", "Wf", "bf"]
    want = {k: 0.0 for k in names}
    for b, X in enumerate(Xs):
        assert np.array_equal(crit_h[b], _oracle_crit(X, p)), (case.name, b)
        sl = slice(int(starts[b]), int(starts[b + 1]))
        # every rank's merged q_max is the saved Q row of the critical instance
        for r in ranks:
            qm = _np(r.qmax).reshape(len(Xs), case.C, KQ)[b]
            assert np.array_equal(qm, Q_bag[sl][crit_h[b]]), (case.name, b)
        fo = orc.FwdOut(None, None, A_bag[sl], B_h[b], crit_h[b], Q=Q_bag[sl], H1=H1_bag[sl])
        g = orc.backward_sharded(X, p, fo, ups[b][0], ups[b][1], G)
        for k in names:
            want[k] = want[k] + g[k]
    got = {k: _np(v) for k, v in zip(names, grads)}
    _check(case, f"{ops} G={G} {'probes' if probes_on else 'plain'}", got, want)


PROBES = pytest.mark.parametrize("probes_on", [False, True], ids=["plain", "probes"])


@pytest.mark.gpu
@PROBES
@pytest.mark.parametrize("case", SINGLE, ids=lambda c: c.name)
def test_single_bag_backward_on_its_own_saves(case, probes_on):
    """dsmil_backward: every parameter gradient and gX (through Wv and v's mask for passing_v)."""
    run_single(case, probes_on)


@pytest.mark.gpu
@PROBES
@pytest.mark.parametrize("case", BAGS, ids=lambda c: c.name)
def test_batched_backward_on_its_own_saves(case, probes_on):
    run_bags(case, probes_on)


@pytest.mark.gpu
@PROBES
@pytest.mark.parametrize("case", DEV, ids=lambda c: c.name)
def test_capture_safe_batched_backward_on_its_own_saves(case, probes_on):
    run_dev(case, probes_on)


@pytest.mark.gpu
@PROBES
@pytest.mark.parametrize("dev", [False, True], ids=["eager", "dev"])
@pytest.mark.parametrize("case", MODELS, ids=lambda c: c.name)
def test_fold_backward_on_its_own_saves(case, dev, probes_on):
    run_models(case, probes_on, dev)


@pytest.mark.gpu
@PROBES
@pytest.mark.parametrize("G", [1, 2, 3])
@pytest.mark.parametrize("ops,case", [("bag_ops", SHARD[0]), ("bag_dev_ops", SHARD[0]), ("per_bag_ops", SHARD[1])],
                         ids=lambda v: v.name if isinstance(v, Case) else v)
def test_row_sharded_backward_on_its_own_saves(ops, case, G, probes_on):
    run_shard(case, ops, G, probes_on)
