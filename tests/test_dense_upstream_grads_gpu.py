"""Instance-classifier and feature gradients against the fp64 oracle under DENSE upstream gradients, on every backward
route, at the row-split and chunk boundaries of the reductions that consume d_classes.

The callers' loss (train_tcga.py:67-71) puts a gradient on `classes` only at each class's arg-max row, so under it
gWi = d_classes^T X (k_gemv_tn / k_gemm_tn, k_gemv_tn_rag / k_gemm_tn_rag), gbi (k_colsum + k_sum_partials) and the
d_classes . Wi term of gX (k_bwd_dx_extra, k_bwd_dx_extra_b) see one non-zero row per class.  Here the loss is

    L = sum wc*classes + sum wA*A + sum wB*B + sum wp*pred        (wc, wA, wB, wp seeded N(0, 1))

(classes and pred only where a route takes no gradient to A and B), and wc is 64x larger on "probe" rows: the first
and last row of every bag, of every row split / chunk the launch uses, and rows 127-129.  A dropped or doubled probe
row moves gWi or gbi far past the tolerance; the CPU part below proves that for every case, with the oracle alone.

The split rules are mirrored here (tn_splits, colsum_splits, rag_rows_per_chunk, rag_splits of gemm_generic.cuh /
bag_plan.cuh) to choose the sizes and the probe rows, and every case asserts the boundary it was chosen for, so a
change of the split rule fails here instead of quietly testing something else.

Tolerances (tests/test_gpu_parity.py, DESIGN.md §3): 5e-5 rel-to-max for Wi, bi, Wf, bf, Wv, bv; the q.* gradients,
behind the softmax over the instances, 5e-5 on the generic forward, 1e-3 on the tensor-core forward and 2e-3 there
for bags of >= 10 000 rows or more than four classes; gX row by row, relative to the row's own maximum with a floor of 1e-3 of the tensor's
maximum, at the q.* tolerance of the route (gX holds the Q-MLP's share) or 5e-5 where it is d_classes . Wi alone.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass
from typing import Dict, List, Tuple

import numpy as np
import pytest
import torch

from conftest import rel_to_max
from oracle import dsmil_oracle as orc

# ---------------------------------------------------------------------------------------- split mirror (host only)
K_SPLITS, TBM, TBK = 296, 128, 16        # kSplits (common.cuh), the TN tile and its k-step (gemm_generic.cuh)
PROBE_SCALE = 64.0


def ceil_div(a, b):
    return -(-a // b)


def tn_use_gemv(M1, M2):
    return M1 <= 4 and M2 % 4 == 0 and M2 // 4 <= 256


def tn_splits(M1, M2, N):
    if tn_use_gemv(M1, M2):
        s, maxs = K_SPLITS, ceil_div(N, 64)
    else:
        s, maxs = K_SPLITS // (ceil_div(M1, TBM) * ceil_div(M2, TBM)), ceil_div(N, 128)
    return max(1, min(s, maxs))


def colsum_splits(N):
    return max(1, min(ceil_div(N, 64), K_SPLITS))


def rag_splits(M1, M2, gemv):
    return K_SPLITS if gemv else max(1, K_SPLITS // (ceil_div(M1, TBM) * ceil_div(M2, TBM)))


def rag_rows_per_chunk(M1, M2, total, gemv):
    if gemv:
        return max(ceil_div(total, K_SPLITS), 64)
    return max(ceil_div(ceil_div(total, rag_splits(M1, M2, False)), TBK) * TBK, 128)


@dataclass
class Plan:
    """The row ranges one reduction over packed rows walks: gWi's splits or chunks and gbi's column-sum splits."""
    kind: str                              # "gemv" (streaming kernel) or "tile" (128 x 128 tile kernel)
    S: int                                 # splits / chunks launched (empty trailing splits included)
    rps: int                               # rows per split / chunk
    gwi: List[Tuple[int, int]]             # [lo, hi) packed rows of each gWi split / chunk (may be empty)
    cs: List[Tuple[int, int]]              # [lo, hi) packed rows of each column-sum split


def colsum_ranges(total):
    S = colsum_splits(total)
    rps = ceil_div(total, S)
    return [(z * rps, min(total, (z + 1) * rps)) for z in range(S)]


def single_plan(C, D, N, aligned=True):
    """launch_gemm_tn(d_classes, C, X, D, N) and launch_colsum(d_classes, C, N): one bag."""
    S = tn_splits(C, D, N)
    if tn_use_gemv(C, D) and aligned:
        kind, rps = "gemv", ceil_div(N, S)
    else:                                  # the tile kernel; an unaligned bag keeps the tile form's split budget
        kind = "tile"
        if tn_use_gemv(C, D):
            S = max(1, min(S, K_SPLITS // (ceil_div(C, TBM) * ceil_div(D, TBM))))
        rps = ceil_div(ceil_div(N, S), TBK) * TBK
    return Plan(kind, S, rps, [(z * rps, min(N, (z + 1) * rps)) for z in range(S)], colsum_ranges(N))


def batched_plan(C, D, Ns, aligned=True):
    """launch_gemm_tn_rag over rag_chunks and launch_colsum over the packed rows: a batch of bags."""
    gemv = tn_use_gemv(C, D) and aligned
    total = sum(Ns)
    rps = rag_rows_per_chunk(C, D, total, gemv)
    chunks, row = [], 0
    for n in Ns:
        chunks += [(row + r0, row + min(n, r0 + rps)) for r0 in range(0, n, rps)]
        row += n
    return Plan("gemv" if gemv else "tile", len(chunks), rps, chunks, colsum_ranges(total))


def probe_rows(Ns, plan: Plan):
    """Packed rows that carry the 64x weight: each bag's first, last and 127-129th rows, and the first and last row of
    every non-empty split or chunk of both reductions."""
    rows, start = set(), 0
    for n in Ns:
        rows |= {start, start + n - 1} | {start + r for r in (127, 128, 129) if r < n}
        start += n
    for lo, hi in plan.gwi + plan.cs:
        if hi > lo:
            rows |= {lo, hi - 1}
    return sorted(rows)


# --------------------------------------------------------------------------------------------------------- cases
@dataclass(frozen=True)
class Case:
    name: str
    D: int
    C: int
    Ns: Tuple[int, ...]
    nonlinear: bool = True
    passing_v: bool = False
    misaligned: Tuple[int, ...] = ()       # bags whose features sit 4 bytes past a 16-byte boundary
    seed: int = 0

    def params(self):
        return orc.random_params(self.D, self.C, 900 + self.seed, nonlinear=self.nonlinear,
                                 passing_v=self.passing_v, scale=1.5)

    def bags(self):
        return [orc.synthetic_bag(n, self.D, 1000 * self.seed + b) for b, n in enumerate(self.Ns)]

    @property
    def generic(self):
        """The Q-MLP runs on the generic (fp32 FFMA) route, not the tensor-core one (sm90::qmlp_supported)."""
        return self.D % 128 != 0 or not self.nonlinear

    def tol_q(self):
        """q.* (and gX) on the tensor-core forward: its 3xBF16 Q rounding, amplified by the softmax backward, grows with
        the bag and with the classes summed into dz (measured 1.09e-3 on b1 at C = 6, N = 2049, where an fp32 forward
        gives 2.6e-5)."""
        if self.generic:
            return 5e-5
        return 2e-3 if (max(self.Ns) >= 10000 or self.C > 4) else 1e-3


def _c(name, D, C, Ns, reseed=0, **kw):
    return Case(name, D, C, tuple(Ns), seed=len(name) * 31 + D + C + sum(Ns) % 977 + reseed, **kw)


# One bag: launch_gemm_tn / launch_colsum.  Each case names the boundary it sits on.
S_N1 = _c("gemv_n1", 512, 1, [1])
S_N64 = _c("gemv_n64_one_split", 512, 2, [64])
S_N65 = _c("gemv_n65_two_splits", 512, 4, [65])
S_N18944 = _c("gemv_n18944_296x64", 512, 1, [18944])
S_N18945 = _c("gemv_n18945_296x65", 512, 2, [18945])
S_N100K = _c("gemv_n100000", 512, 1, [100000], reseed=1)    # the first draw cancels gbi to 5e-5 of sum |wc|
S_D1024 = _c("gemv_d1024_limit", 1024, 4, [18945])
T_D2048 = _c("tile_d2048_one_row_split", 2048, 2, [2305])
T_C5 = _c("tile_c5", 512, 5, [3001])
T_C6 = _c("tile_c6", 512, 6, [2049])
T_C7 = _c("tile_c7", 512, 7, [129])
T_C8 = _c("tile_c8", 512, 8, [3001])
T_D166 = _c("tile_d166", 166, 1, [2049])
T_D230 = _c("tile_d230_linear", 230, 2, [2305], nonlinear=False)
T_MIS = _c("tile_unaligned_fallback", 512, 2, [18945], misaligned=(0,))
G_PV = _c("gemv_d96_passing_v", 96, 2, [18945], passing_v=True)

SINGLE_EXPECT = {
    S_N1: lambda pl: pl.kind == "gemv" and pl.S == 1 and pl.rps == 1,
    S_N64: lambda pl: pl.kind == "gemv" and pl.S == 1 and pl.rps == 64,
    S_N65: lambda pl: pl.kind == "gemv" and pl.S == 2 and pl.gwi == [(0, 33), (33, 65)],
    S_N18944: lambda pl: pl.kind == "gemv" and pl.S == 296 and pl.rps == 64,
    S_N18945: lambda pl: pl.kind == "gemv" and pl.S == 296 and pl.rps == 65 and pl.gwi[-1][0] >= 18945,
    S_N100K: lambda pl: pl.kind == "gemv" and pl.S == 296 and pl.rps == 338,
    S_D1024: lambda pl: pl.kind == "gemv" and 1024 // 4 == 256 and pl.rps == 65,
    # rows per split rounded up to 16: a one-row split, then an empty one
    T_D2048: lambda pl: pl.kind == "tile" and pl.S == 18 and pl.rps == 144 and pl.gwi[-2:] == [(2304, 2305), (2448, 2305)],
    T_C5: lambda pl: pl.kind == "tile" and pl.S == 24 and pl.rps == 128 and pl.gwi[-1] == (2944, 3001),
    T_C6: lambda pl: pl.kind == "tile" and pl.S == 17 and pl.rps == 128 and pl.gwi[-1] == (2048, 2049),
    T_C7: lambda pl: pl.kind == "tile" and pl.S == 2 and pl.gwi == [(0, 80), (80, 129)],
    T_C8: lambda pl: pl.kind == "tile" and pl.S == 24 and pl.gwi[-1] == (2944, 3001),
    T_D166: lambda pl: pl.kind == "tile" and pl.S == 17 and pl.gwi[-1] == (2048, 2049),
    T_D230: lambda pl: pl.kind == "tile" and pl.S == 19 and pl.rps == 128 and pl.gwi[-1] == (2304, 2305),
    # gemv shape, unaligned bag: the tile kernel within 296 / 4 splits
    T_MIS: lambda pl: pl.kind == "tile" and pl.S == 74 and pl.rps == 272,
    G_PV: lambda pl: pl.kind == "gemv" and pl.S == 296 and pl.rps == 65,
}

# Batches: launch_gemm_tn_rag over rag_chunks.  rps = rows per chunk of the batch.
B_SMALL = _c("rag_gemv_rps64", 512, 2, [64, 63, 65, 1, 128, 129, 127, 2049])          # total 2626 < 18 944
B_LARGE = _c("rag_gemv_rps70", 512, 1, [70, 69, 71, 1, 20504])                         # total 20 715 > 18 944
B_D2048 = _c("rag_tile_d2048", 2048, 2, [256, 255, 257, 1, 3831])                      # batched tile chunks
B_MIS = _c("rag_tile_unaligned", 512, 2, [160, 159, 161, 1, 11319], misaligned=(4,))   # gemv_i == false

BATCH_EXPECT = {
    B_SMALL: lambda pl: pl.kind == "gemv" and sum(B_SMALL.Ns) < 18944 and pl.rps == 64,
    B_LARGE: lambda pl: pl.kind == "gemv" and sum(B_LARGE.Ns) > 18944 and pl.rps == 70,
    B_D2048: lambda pl: pl.kind == "tile" and pl.rps == 256,
    B_MIS: lambda pl: pl.kind == "tile" and pl.rps == 160,
}

# Row-sharded batches.  Every rank holds >= 1 row of every bag on the batched ABI; the one-bag ABI case has a bag
# of one row, so that at G >= 2 a rank holds none of it.
SH_BAGS = _c("shard_rag", 512, 2, [70, 69, 71, 3, 20504])
SH_PERBAG = _c("shard_per_bag_d166", 166, 2, [2049, 1])


def plan_for(case: Case, batched: bool) -> Plan:
    if batched:
        return batched_plan(case.C, case.D, list(case.Ns), aligned=not case.misaligned)
    assert len(case.Ns) == 1
    return single_plan(case.C, case.D, case.Ns[0], aligned=not case.misaligned)


def sharded_probe_rows(case: Case, G: int, batched: bool):
    """Packed (bag-order) rows that are probes on some rank: each rank walks its own local rows."""
    rows, start = set(), np.cumsum([0] + list(case.Ns))
    for r in range(G):
        local = [orc.shard_bounds(n, G)[r] for n in case.Ns]
        Ns_r = [hi - lo for lo, hi in local]
        live = [b for b, n in enumerate(Ns_r) if n > 0]
        if batched:
            groups = [(live, batched_plan(case.C, case.D, [Ns_r[b] for b in live]))]
        else:
            groups = [([b], single_plan(case.C, case.D, Ns_r[b])) for b in live]
        for bags, pl in groups:
            lrow = 0
            lstarts = {}
            for b in bags:
                lstarts[b] = lrow
                lrow += Ns_r[b]
            for pr in probe_rows([Ns_r[b] for b in bags], pl):
                b = max(bb for bb in bags if lstarts[bb] <= pr)
                rows.add(int(start[b] + local[b][0] + pr - lstarts[b]))
    return sorted(rows)


def upstream(case: Case, probes, dense_ab=True):
    """Per bag: (wc [N, C] with the probe rows scaled, wA [N, C], wB [C, D], wp [C]) in float32; wA, wB None when the
    route takes no gradient to A and B.  A probe's weight is 64 x a N(0, 1) draw of magnitude >= 1."""
    rng = np.random.default_rng(5000 + case.seed)
    out, start = [], 0
    for n in case.Ns:
        wc = rng.standard_normal((n, case.C))
        wA = rng.standard_normal((n, case.C))
        wB = rng.standard_normal((case.C, case.D))
        wp = rng.standard_normal(case.C)
        local = [r - start for r in probes if start <= r < start + n]
        wc[local] = PROBE_SCALE * np.sign(wc[local]) * np.maximum(np.abs(wc[local]), 1.0)
        f = lambda a: a.astype(np.float32)
        out.append((f(wc), f(wA) if dense_ab else None, f(wB) if dense_ab else None, f(wp)))
        start += n
    return out


# ----------------------------------------------------------------------------------------------- the fp64 oracle
@functools.lru_cache(maxsize=1)
def _bag_data(case: Case):
    p = case.params()
    Xs = case.bags()
    return p, Xs, [orc.forward(X, p) for X in Xs]


@functools.lru_cache(maxsize=2)
def oracle_grads(case: Case, route: str, G: int = 1):
    """Per-bag fp64 gradients of the route's loss: (weights, [grads of bag b]).  route: "scores" (d_classes only, the
    instance stream alone), "dense" (all four terms), "bags" / "dev" / "shard" (the batched routes' probe rows;
    "dev" and "shard" without A and B terms)."""
    p, Xs, outs = _bag_data(case)
    if route in ("scores", "dense"):
        probes = probe_rows(case.Ns, plan_for(case, False))
    elif route == "shard":
        probes = sharded_probe_rows(case, G, batched=case is not SH_PERBAG)
    else:
        probes = probe_rows(case.Ns, plan_for(case, True))
    w = upstream(case, probes, dense_ab=route in ("dense", "bags"))
    per_bag = []
    for X, o, (wc, wA, wB, wp) in zip(Xs, outs, w):
        if route == "scores":
            g = orc.backward(X, p, o, wc, None, need_dX=True)
        elif route == "shard":
            g = orc.backward_sharded(X, p, o, wc, wp, G)
        else:
            g = orc.backward(X, p, o, wc, wp, d_A=wA, d_B=wB, need_dX=route != "dev")
        per_bag.append(g)
    return probes, w, per_bag


def summed(per_bag, names):
    return {k: sum(g[k] for g in per_bag) for k in names}


def rowwise_err(got, want):
    """max over rows of |got - want| / max(row max |want|, 1e-3 * tensor max |want|)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    den = np.maximum(np.abs(want).max(1), 1e-3 * np.abs(want).max())
    return float((np.abs(got - want).max(1) / np.maximum(den, 1e-30)).max())


TOL = 5e-5
Q_NAMES = ("W1", "b1", "W2", "b2")


def tol_of(case: Case, name):
    return case.tol_q() if name in Q_NAMES else TOL


# ------------------------------------------------------------------------------------------------ route catalogue
# route -> cases.  Each route checks gWi, gbi, every other parameter gradient it gives, and gX where it gives it.
R_SCORES = [S_N1, S_N64, S_N65, S_N18944, S_N18945, S_N100K, S_D1024, T_D2048, T_C5, T_C8, T_D166, T_D230, T_MIS]
R_FUSED = [T_D166, T_D230, G_PV, S_N65, S_N18945, S_N100K, S_D1024, T_D2048, T_C5, T_C6, T_C7, T_C8]
R_SPLIT = [S_N18945, T_D166]
R_BAGS = [B_SMALL, B_LARGE, B_D2048, B_MIS]
R_DEV = [B_SMALL, B_LARGE]
R_SHARD = [("bag_ops", SH_BAGS), ("bag_dev_ops", SH_BAGS), ("per_bag_ops", SH_PERBAG)]

ALL_SINGLE = sorted(set(R_SCORES) | set(R_FUSED) | set(R_SPLIT), key=lambda c: c.name)
ALL_BATCH = sorted(set(R_BAGS) | set(R_DEV), key=lambda c: c.name)


# ================================================================================ CPU part: no device needed
@pytest.mark.parametrize("case", ALL_SINGLE, ids=lambda c: c.name)
def test_single_bag_case_sits_on_its_split_boundary(case):
    assert SINGLE_EXPECT[case](plan_for(case, False)), (case.name, plan_for(case, False))


@pytest.mark.parametrize("case", ALL_BATCH, ids=lambda c: c.name)
def test_batch_case_sits_on_its_chunk_boundary(case):
    pl = plan_for(case, True)
    assert BATCH_EXPECT[case](pl), (case.name, pl.kind, pl.rps)
    # bags of exactly rps rows, rps - 1, rps + 1 and one row
    assert {pl.rps, pl.rps - 1, pl.rps + 1, 1} <= set(case.Ns), (case.name, pl.rps, case.Ns)


def test_split_mirror_matches_the_chunk_bound_and_covers_every_row():
    """rag_chunks_cap: at most rag_splits + nb chunks; splits and chunks tile the rows exactly once."""
    for case in ALL_BATCH + [SH_BAGS]:
        pl = plan_for(case, True)
        assert pl.S <= rag_splits(case.C, case.D, pl.kind == "gemv") + len(case.Ns)
        for ranges in (pl.gwi, pl.cs):
            cover = np.zeros(sum(case.Ns), np.int64)
            for lo, hi in ranges:
                cover[lo:hi] += 1
            assert np.all(cover == 1), case.name
    for case in ALL_SINGLE:
        pl = plan_for(case, False)
        for ranges in (pl.gwi, pl.cs):
            cover = np.zeros(case.Ns[0], np.int64)
            for lo, hi in ranges:
                cover[lo:max(lo, hi)] += 1
            assert np.all(cover == 1), case.name


def test_sharded_cases_put_a_rank_without_rows_where_intended():
    for G in (1, 2, 3):
        assert all(hi - lo >= 1 for n in SH_BAGS.Ns for lo, hi in orc.shard_bounds(n, G))
    assert any(hi == lo for lo, hi in orc.shard_bounds(SH_PERBAG.Ns[1], 2))
    assert not batched_shape(SH_PERBAG) and batched_shape(SH_BAGS)


def batched_shape(case):
    """sm90::batched_supported: the batched tensor-core ABI takes D % 128 == 0, D <= 2048, C <= 4, non-linear q."""
    return case.D % 128 == 0 and case.D <= 2048 and case.C <= 4 and case.nonlinear and not case.passing_v


SENSITIVITY = ([(c, "scores", 1) for c in R_SCORES] + [(c, "dense", 1) for c in R_FUSED] +
               [(c, "bags", 1) for c in R_BAGS] + [(c, "dev", 1) for c in R_DEV] +
               [(c, "shard", G) for _, c in R_SHARD[::2] for G in (1, 2, 3)])


@pytest.mark.parametrize("case,route,G", SENSITIVITY, ids=lambda v: v.name if isinstance(v, Case) else str(v))
def test_one_lost_or_repeated_probe_row_moves_the_gradients_past_20x_tolerance(case, route, G):
    """The oracle's gradients are linear in d_classes: removing probe row n moves gWi, gbi and gX by minus that row's
    own share, doubling it by plus the share, and the share is the oracle's backward of d_classes row n alone (a
    one-row bag, no bag-classifier gradient).  Each must move a checked tensor by > 20x the GPU test's tolerance."""
    p, Xs, outs = _bag_data(case)
    probes, w, per_bag = oracle_grads(case, route, G)
    base = summed(per_bag, ("Wi", "bi"))
    # tie-free arg-max: the device's fp32 scores select the same critical rows as the fp64 oracle
    for o in outs:
        if o.classes.shape[0] > 1:
            s = np.sort(o.classes, axis=0)
            assert np.all(s[-1] - s[-2] > 1e-5 * np.abs(o.classes).max()), case.name
    # a well-conditioned gbi: no class's column sum of wc cancels below a tenth of its random-walk size, where any fp32
    # summation order loses digits that no tolerance relative to the result can hold
    wc_all = np.concatenate([wb[0] for wb in w]).astype(np.float64)
    assert np.abs(base["bi"]).max() >= 0.1 * np.sqrt((wc_all ** 2).sum(0)).max(), (case.name, route, base["bi"])
    with_gx = route in ("scores", "dense", "bags")
    tol_x = TOL if route == "scores" else case.tol_q()
    starts = np.cumsum([0] + list(case.Ns))
    gx_max = [np.abs(g["X"]).max() if with_gx else None for g in per_bag]
    assert probes and len(probes) == len(set(probes))
    for r in probes:
        b = int(np.searchsorted(starts, r, side="right") - 1)
        n = r - starts[b]
        X1 = Xs[b][n:n + 1]
        share = orc.backward(X1, p, orc.forward(X1, p), w[b][0][n:n + 1], None, need_dX=True)
        for sign in (-1.0, 1.0):            # removed, doubled
            moved = [rel_to_max(base["Wi"] + sign * share["Wi"], base["Wi"]) / TOL,
                     rel_to_max(base["bi"] + sign * share["bi"], base["bi"]) / TOL]
            if with_gx:
                den = max(np.abs(per_bag[b]["X"][n]).max(), 1e-3 * gx_max[b])
                moved.append(np.abs(share["X"][0]).max() / den / tol_x)
            assert max(moved) > 20.0, (case.name, route, G, r, moved)


# ========================================================================================= GPU part (one H100)
def _np(t):
    return t.detach().cpu().numpy()


def _dev_bag(X, misaligned):
    """X on the device as a leaf that requires grad; misaligned: a view 4 bytes past a 16-byte boundary (the gradient
    is then taken with respect to the view)."""
    if not misaligned:
        return torch.from_numpy(X).cuda().requires_grad_(True)
    buf = torch.zeros(X.size + 1, device="cuda")
    buf[1:].copy_(torch.from_numpy(X).reshape(-1).cuda())
    buf.requires_grad_(True)
    x = buf[1:].view(X.shape)
    assert x.data_ptr() % 16 == 4
    return x


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _check_params(case, got: Dict[str, np.ndarray], want: Dict[str, np.ndarray], what):
    assert got.keys() == want.keys(), (what, sorted(got), sorted(want))
    errs = {k: rel_to_max(got[k], want[k]) for k in want}
    bad = {k: (e, tol_of(case, k)) for k, e in errs.items() if not e <= tol_of(case, k)}
    assert not bad, (what, case.name, bad, errs)


def _net(case):
    from helpers import build_net
    return build_net(case.params()).train()


def _param_names(case, with_instance=True):
    names = (["Wi", "bi"] if with_instance else []) + ["W1", "b1"] + (["W2", "b2"] if case.nonlinear else [])
    names += ["Wv", "bv"] if case.passing_v else []
    return names + ["Wf", "bf"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", R_SCORES, ids=lambda c: c.name)
def test_instance_scores_backward_vs_oracle(case):
    """dsmil_instance_scores_backward through FCLayer(x) with gradients on: gWi, gbi and gX = d_classes . Wi."""
    import dsmil as mil
    p, Xs, _ = _bag_data(case)
    _, w, per_bag = oracle_grads(case, "scores")
    fc = mil.FCLayer(case.D, case.C).cuda()
    with torch.no_grad():
        fc.fc[0].weight.copy_(_t(p.Wi))
        fc.fc[0].bias.copy_(_t(p.bi))
    x = _dev_bag(Xs[0], 0 in case.misaligned)
    feats, c = fc(x)
    assert feats is x
    gWi, gbi, gX = torch.autograd.grad((c * _t(w[0][0])).sum(), [fc.fc[0].weight, fc.fc[0].bias, x])
    want = per_bag[0]
    _check_params(case, {"Wi": _np(gWi), "bi": _np(gbi)}, {"Wi": want["Wi"], "bi": want["bi"]}, "FCLayer")
    assert rowwise_err(_np(gX), want["X"]) <= TOL, (case.name, rowwise_err(_np(gX), want["X"]))


def _dense_loss(outs, wts):
    classes, pred, A, B = outs
    wc, wA, wB, wp = (_t(a) for a in wts)
    return (classes * wc).sum() + (A * wA).sum() + (B[0] * wB).sum() + (pred[0] * wp).sum()


@pytest.mark.gpu
@pytest.mark.parametrize("case", R_FUSED, ids=lambda c: c.name)
def test_fused_single_bag_backward_vs_oracle(case):
    """MILNet(x), one library call each way (dsmil_backward): every parameter gradient and gX."""
    from helpers import grad_name
    p, Xs, _ = _bag_data(case)
    _, w, per_bag = oracle_grads(case, "dense")
    net = _net(case)
    x = _dev_bag(Xs[0], False)
    names = _param_names(case)
    params = dict(net.named_parameters())
    leaves = [params[grad_name(k, case.nonlinear)] for k in names]
    grads = torch.autograd.grad(_dense_loss(net(x), w[0]), leaves + [x])
    _check_params(case, {k: _np(g) for k, g in zip(names, grads)}, {k: per_bag[0][k] for k in names}, "MILNet")
    err = rowwise_err(_np(grads[-1]), per_bag[0]["X"])
    assert err <= case.tol_q(), (case.name, "gX", err)


@pytest.mark.gpu
@pytest.mark.parametrize("case", R_SPLIT, ids=lambda c: c.name)
def test_split_form_backward_vs_oracle(case):
    """feats, c = i_classifier(x); pred, A, B = b_classifier(feats, c): the instance stream's backward
    (dsmil_instance_scores_backward) takes d_classes, the bag node's (dsmil_backward, classes_in path) the rest and no
    Wi / bi gradient; x's gradient is the sum of both nodes' contributions."""
    from helpers import grad_name
    p, Xs, _ = _bag_data(case)
    _, w, per_bag = oracle_grads(case, "dense")
    net = _net(case)
    x = _dev_bag(Xs[0], False)
    feats, c = net.i_classifier(x)
    pred, A, B = net.b_classifier(feats, c)
    names = _param_names(case)
    params = dict(net.named_parameters())
    leaves = [params[grad_name(k, case.nonlinear)] for k in names]
    grads = torch.autograd.grad(_dense_loss((c, pred, A, B), w[0]), leaves + [x])
    _check_params(case, {k: _np(g) for k, g in zip(names, grads)}, {k: per_bag[0][k] for k in names}, "split form")
    err = rowwise_err(_np(grads[-1]), per_bag[0]["X"])
    assert err <= case.tol_q(), (case.name, "gX", err)


@pytest.mark.gpu
def test_foreign_instance_stream_takes_the_split_path_vs_oracle():
    """A MILNet whose i_classifier is a plain torch module: MILNet.forward runs it, then the bag node on its scores."""
    import dsmil as mil
    from helpers import grad_name
    case = S_N18945
    p, Xs, _ = _bag_data(case)
    _, w, per_bag = oracle_grads(case, "dense")

    class Plain(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.lin = torch.nn.Linear(case.D, case.C)

        def forward(self, x):
            return x, self.lin(x)

    ic = Plain().cuda()
    with torch.no_grad():
        ic.lin.weight.copy_(_t(p.Wi))
        ic.lin.bias.copy_(_t(p.bi))
    net = mil.MILNet(ic, _net(case).b_classifier).train()
    x = _dev_bag(Xs[0], False)
    names = _param_names(case, with_instance=False)
    params = dict(net.named_parameters())
    leaves = [params[grad_name(k, case.nonlinear)] for k in names] + [ic.lin.weight, ic.lin.bias]
    grads = torch.autograd.grad(_dense_loss(net(x), w[0]), leaves + [x])
    got = {k: _np(g) for k, g in zip(names + ["Wi", "bi"], grads)}
    # the instance scores come from torch's Linear here (TF32 off by default for fp32 matmul): held to the same bar
    _check_params(case, got, {k: per_bag[0][k] for k in got}, "foreign instance stream")
    err = rowwise_err(_np(grads[-1]), per_bag[0]["X"])
    assert err <= case.tol_q(), (case.name, "gX", err)


@pytest.mark.gpu
@pytest.mark.parametrize("case", R_BAGS, ids=lambda c: c.name)
def test_forward_bags_grad_backward_vs_oracle(case):
    """forward_bags(grad=True) and one dsmil_backward_bags: parameter gradients against the sum over the bags of the
    per-bag oracle gradients, gX bag by bag."""
    from helpers import grad_name
    p, Xs, outs1 = _bag_data(case)
    _, w, per_bag = oracle_grads(case, "bags")
    net = _net(case)
    xs = [_dev_bag(X, b in case.misaligned) for b, X in enumerate(Xs)]
    outs = net.forward_bags(xs, grad=True)
    loss = sum(_dense_loss(outs[b], w[b]) for b in range(len(xs)))
    assert np.array_equal(_np(outs.crit), np.stack([o.idx for o in outs1]))
    names = _param_names(case)
    params = dict(net.named_parameters())
    leaves = [params[grad_name(k, case.nonlinear)] for k in names]
    grads = torch.autograd.grad(loss, leaves + xs)
    _check_params(case, {k: _np(g) for k, g in zip(names, grads)}, summed(per_bag, names), "forward_bags")
    for b, (g, want) in enumerate(zip(grads[len(names):], per_bag)):
        err = rowwise_err(_np(g), want["X"])
        assert err <= case.tol_q(), (case.name, "gX", b, err)


@pytest.mark.gpu
@pytest.mark.parametrize("case", R_DEV, ids=lambda c: c.name)
def test_dev_backward_ignores_dead_rows_and_matches_eager_and_oracle(case):
    """MILBagsDevFn (dsmil_backward_bags_dev): d_classes has nb * max_rows rows and only the live prefix may count.
    The dead tail [total, nb * max_rows) is filled with large values; the gradients must equal the eager call's bits
    (as with a zero tail) and match the oracle."""
    from helpers import grad_name
    from dsmil_wsi_b200 import functional as Fn
    from dsmil_wsi_b200.sharded import milnet_params
    p, Xs, _ = _bag_data(case)
    _, w, per_bag = oracle_grads(case, "dev")
    net = _net(case)
    params = milnet_params(net)
    names = _param_names(case)
    leaves = [dict(net.named_parameters())[grad_name(k, case.nonlinear)] for k in names]
    nb, max_rows, total = len(Xs), max(case.Ns), sum(case.Ns)
    slots = torch.zeros(nb, max_rows, case.D, device="cuda")
    for b, X in enumerate(Xs):
        slots[b, :X.shape[0]].copy_(torch.from_numpy(X))
    Ns = torch.tensor(case.Ns, dtype=torch.int64, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    wc_live = torch.cat([_t(wb[0]) for wb in w])
    wp = torch.stack([_t(wb[3]) for wb in w])

    def dev_grads(tail):
        wc = torch.full((nb * max_rows, case.C), tail, device="cuda")
        wc[:total] = wc_live
        classes, pred, _, _, _ = Fn.MILBagsDevFn.apply(slots, Ns, status, *params)
        return torch.autograd.grad((classes * wc).sum() + (pred * wp).sum(), leaves)

    big = dev_grads(1.0e4)
    zero = dev_grads(0.0)
    outs, _ = Fn.mil_forward_bags([slots[b, :n] for b, n in enumerate(case.Ns)], params, grad=True)
    classes, pred = outs.packed[0], outs.packed[1]
    eager = torch.autograd.grad((classes * wc_live).sum() + (pred * wp).sum(), leaves)
    assert int(status) == 0
    for k, a, z, e in zip(names, big, zero, eager):
        assert torch.equal(a, e) and torch.equal(z, e), (case.name, k, float((a - e).abs().max()))
    _check_params(case, {k: _np(g) for k, g in zip(names, big)}, summed(per_bag, names), "dev")


class _DevRank:
    """One logical rank of virtual_sharded_train_step_bags over CudaShardBagDevOps: begin() packs the rank's local bags
    into slots [nb, max_rows, D] (max_rows: its largest local bag) and hands the offsets over as a device tensor; bwd1
    gets d_classes with nb * max_rows rows, a large dead tail after the live ones."""

    TAIL = 1.0e4

    def __init__(self, params):
        self.params = params

    def begin(self, X_locals, row_offsets):
        from dsmil_wsi_b200.sharded import CudaShardBagDevOps
        nb, D = len(X_locals), int(X_locals[0].shape[1])
        self.Ns_host = [int(x.shape[0]) for x in X_locals]
        self.max_rows = max(self.Ns_host)
        self.slots = torch.zeros(nb, self.max_rows, D, device="cuda")
        for b, x in enumerate(X_locals):
            self.slots[b, :x.shape[0]].copy_(x)
        self.status = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.offs = torch.tensor([int(o) for o in row_offsets], dtype=torch.int64, device="cuda")
        self.ops = CudaShardBagDevOps(self.params, torch.tensor(self.Ns_host, dtype=torch.int64, device="cuda"),
                                      self.status)
        return self.ops.begin([self.slots], self.offs)

    def phase1_train(self):
        return self.ops.phase1_train()

    def phase2_train(self, Q, cands_all, G):
        return self.ops.phase2_train(Q, cands_all, G)

    def phase3_train(self, recs_all, G, A):
        return self.ops.phase3_train(recs_all, G, A)

    def bwd1(self, xs, A, B, d_classes, d_pred):
        dc = torch.full((len(self.Ns_host) * self.max_rows, d_classes.shape[1]), self.TAIL, device="cuda")
        dc[:d_classes.shape[0]] = d_classes
        return self.ops.bwd1(xs, A, B, dc, d_pred)

    def bwd2(self, xs, A, dA, t, Q):
        return self.ops.bwd2(xs, A, dA, t, Q)

    def bwd3(self, xs, row_offsets, Q, H1, dL, dqm, qmax, crit):
        return self.ops.bwd3(xs, self.offs, Q, H1, dL, dqm, qmax, crit)


@pytest.mark.gpu
@pytest.mark.parametrize("G", [1, 2, 3])
@pytest.mark.parametrize("ops,case", R_SHARD, ids=lambda v: v.name if isinstance(v, Case) else v)
def test_virtual_sharded_step_with_dense_loss_grads_vs_oracle(ops, case, G):
    """virtual_sharded_train_step_bags with a dense d_classes: every gradient against the fp64 oracle's row-sharded
    backward (backward_sharded), summed over the bags."""
    from dsmil_wsi_b200.sharded import (CudaShardBagOps, CudaShardOps, PerBagShardOps, milnet_params,
                                        virtual_sharded_train_step_bags)
    p, Xs, outs1 = _bag_data(case)
    _, w, per_bag = oracle_grads(case, "shard", G)
    net = _net(case)
    params = milnet_params(net)
    make = {"bag_ops": lambda: CudaShardBagOps(params), "bag_dev_ops": lambda: _DevRank(params),
            "per_bag_ops": lambda: PerBagShardOps(CudaShardOps(params))}[ops]
    dc = torch.cat([_t(wb[0]) for wb in w])
    dp = torch.stack([_t(wb[3]) for wb in w])
    xs = [torch.from_numpy(X).cuda() for X in Xs]
    ranks = []

    def make_rank():
        ranks.append(make())
        return ranks[-1]

    (_, _, _, _, crit), grads = virtual_sharded_train_step_bags(make_rank, xs, G, lambda c, pr, cr: (dc, dp))
    assert np.array_equal(_np(crit).reshape(len(Xs), -1), np.stack([o.idx for o in outs1]))
    if ops == "bag_dev_ops":
        assert all(int(r.status) == 0 for r in ranks)
    names = ["Wi", "bi", "W1", "b1", "W2", "b2", "Wf", "bf"]
    _check_params(case, {k: _np(g) for k, g in zip(names, grads)}, summed(per_bag, names), f"{ops} G={G}")
