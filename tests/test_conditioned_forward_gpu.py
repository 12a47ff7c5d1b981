"""The forward of every covered route against an fp64 forward run on the kernels' OWN Q (the conditioned check), row by
row, on bags whose attention is peaked.

`test_gpu_parity.py` compares the device with the oracle's own fp64 forward, so its bars (A within 2e-5 of the column
maximum, Q within 1e-4) also carry the 3xBF16 rounding of Q, and its inputs (small random weights, U[0,1) features)
give nearly uniform attention: every online-softmax rescale factor is close to 1, no record's combine weight
underflows, and a bar relative to the column maximum lets a row at 1e-4 of it be 20 % wrong.  Here each case runs the
route's training form with saves (classes, crit, Q, H1, and V on the value route), and the fp64 restatement takes the
kernel's own classes and Q (B over the kernel's own V):

    q_max = Q[crit], L = Q q_max^T / 11.313708305358887, A = softmax over the rows, B = A^T X, pred = Wf B + bf

Every stage is checked element by element against a bound of its own inputs (u = 2^-24):

    classes   |c - c64|      <= C_CLS u (sum_d |x_d Wi_kd| + |bi_k|)
    crit      classes[crit_k, k] is the column maximum of the kernel's own classes, bit for bit (ties not pinned)
    H1 (TC)   |H1 - relu(3xbf16(X, W1) + b1)|       <= C_MM u (sum |x w| + |b|)
    Q (TC)    |Q - tanh(3xbf16(H1, W2) + b2)|       <= (1 - Q64^2) C_MM u (sum |h w| + |b|) + TANH_ABS
    Q (FFMA)  the same against the fp64 products; linear q without the tanh terms
    A         |A - A64| <= tau_n A64,  tau_n = r_n + sum_m A64_m r_m + C_A u,  r_n = eL_n + 2u |L_n - M|,
              eL_n = C_L u sum_j |Q_nj q_max_j| / s + u |L_n| (an error in the maximum M cancels in A);
              where A64 < 2 FLT_MIN: |A| <= 4 FLT_MIN
    B         |B_kd - B64_kd| <= sum_n A64_nk (tau_nk + depth u) |X_nd|   (per column: small columns count), plus
              sum_n A64_nk |X_nd| over the rows with A64 < 2 FLT_MIN (they underflow in fp32) and FLT_MIN sum_n |X_nd|
    pred      |pred - pred64| <= sum_kd |Wf_jkd| bar(B_kd) + C_P u sum_kd |Wf_jkd| sum_n A64_nk |X_nd|

    V         |V - relu(Xv Wv^T + bv)|              <= C_MM u (sum |xv w| + |b|), on the masked input

Routes: dsmil_forward (training, eval overlapped and plain) and dsmil_bag_forward; dsmil_forward_bags[_train] and the
capture-safe pair (dsmil_forward_bags[_train]_dev or dsmil_generic_*); the fold forms (dsmil_forward_bags_models,
_models_train, _models_train_dev); dsmil_value_forward_bags with and without v's mask; and the row-sharded phases at
G = 1, 2, 3 per bag (CudaShardOps, with an empty rank, a probe-free rank whose combine weight underflows, and a crafted Q
given to phase 2) and batched (CudaShardBagOps).  The cases reach every instance of k_qmlp_sm90, k_attend,
k_attend_gb and k_attend_b (test_kernel_instances_gpu.py checks it), with the last column group of each J or NJ full
and partly empty, and k_qmlp_sm90 at D = 128 and at the largest D of each CT (a mirror of qmlp_smem_bytes).  Forms
without saves keep Q in tile blocks and apply the same tanh_ex2 on read, so they are checked against the restatement on the training call's Q, after asserting that they give its
classes and crit bits.

Peaked bags.  Column d0 of W1 is zero and Wi[0, d0] = 1: the class-0 critical row has x[d0] = 8.  Probe rows copy it
except at d0 and at d1 (also a zero column of W1 and Wi), where each holds its own value, so in every kernel their Q is
bit-identical to q_max (asserted), their class-0 logit is the bag maximum and B sees each probe in column d1.  Nonlinear
q: hidden unit J0 reads only column d2 (x[d2] = 16 on the critical and probe rows, 0 elsewhere) and W2[:, J0] = 64 s,
b2 = -bias s for a sign vector s: q_max saturates to s exactly, every other row's tanh is driven towards -s, and class 0's
A spans more than five decades.  Classes k >= 1 take ordinary rows (flag column e_k) as critical rows: there the probes
are the rows of least attention.  Linear q (generic routes): W1[:, d2] = (beta + 1) s and b1 -= beta s, so q_max points
along s and every other row against it: the logits spread over more than 100, and most rows -- whole records of them --
underflow to 0 in fp32 (the last record holds no probe, so it underflows whole).  The rescale cases put the class-0 maximum in the second
tile of an attend record whose first tile holds no probe, so that tile's partial sums are rescaled by e^-10 or less.

Probe rows sit at rows 0, 127-129, the bag's last row, the first and last rows of the first and last tile of every attend
record (recs_for_bag on the tensor-core batch, attend_ctas on the generic one, mirrored here and checked against the
sources' constants), the edges of k_finalize_b's 32 A-slices and, on the sharded cases, each rank's first and last
row.  The CPU part proves with the restatement alone that
dropping or doubling any probe row's term in the normaliser S (tile sums, record combine, A's normalisation see the row
through that one term) or in B (its partial Bp and the record combine of B) moves a checked output by more than 20x its
bar, and that an fp32 restatement of the same algebra on the same inputs stays 4x under every bar.

Measured maxima (error over bar, largest over the cases of a route) and the GPU they were measured on are in DESIGN §3.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import re
from dataclasses import dataclass
from typing import Tuple

import numpy as np
import pytest
import torch

from oracle import dsmil_oracle as orc

KQ = 128
U = 2.0 ** -24
FLT_MIN = float(np.finfo(np.float32).tiny)
SCALE = orc.SCALE_F32
# mirrored from the sources (checked below): fwd_batched.cuh, fwd_kernels.cuh, common.cuh
K_ATT_ROWS, K_MAX_REC_PER_BAG, K_FIN_SLICES = 128, 128, 32
K_ATTEND_ROWS, K_SPLITS = 32, 296
# fwd_sm90.cuh: k_qmlp_sm90's shared memory (W ring of K_WSTAGES chunks, Wi at C rounded up to 1/2/4/8 rows, M members'
# rows and biases in the fold form) against the 227 KB a block may have on sm_90; include/dsmil_b200.h: DSMIL_MAX_D
K_WSTAGES, K_CHUNK_K, K_SMEM_BAGS, BAGDEV_BYTES, K_MAX_C, SMEM_CAP, MAX_D = 4, 64, 96, 40, 8, 232448, 4096
# bar constants (multiples of u); the CPU part shows each is >= 4x the fp32 restatement's error on the same inputs
C_CLS = 64.0
C_MM = 64.0
C_L = 28.0
C_A = 56.0
C_P = 64.0
TANH_ABS = 3e-7              # DESIGN §4.1: tanh_ex2's stated absolute bound
SENSITIVITY = 20.0
RESCALE_MAX = float(np.exp(-10.0))
D0, D1, D2 = 0, 1, 2         # class-0 flag, probe id, saturation driver; e_k = 2 + k flags class k's critical row
J0 = 5                       # the hidden unit that reads only column d2


def ceil_div(a, b):
    return -(-a // b)


def recs_for_bag(N):
    """bag_plan.cuh: k_attend_b records (CTAs) of a bag of N rows."""
    return min(max(ceil_div(N, K_ATT_ROWS), 1), K_MAX_REC_PER_BAG)


def attend_ctas(N):
    """bag_plan.cuh: generic k_attend records of a bag of N rows."""
    return min(max(ceil_div(N, K_ATTEND_ROWS), 1), K_SPLITS)


def ct_of(C_):
    return 1 if C_ <= 1 else 2 if C_ <= 2 else 4 if C_ <= 4 else 8


def qmlp_smem_bytes(C_, D, M=0):
    """fwd_sm90.cuh: qmlp_smem_bytes (M = 0) or qmlp_models_smem_bytes (M members), plus kQmlpStaticSmem."""
    fixed = K_WSTAGES * 2 * (KQ * K_CHUNK_K * 2)
    wi = ct_of(C_) * D if M == 0 else M * (ct_of(C_) * D + 2 * KQ + K_MAX_C)
    return fixed + 4 * wi + 1024 + 2 * KQ * 4 + K_SMEM_BAGS * BAGDEV_BYTES + 256


def qmlp_supported(C_, D, nonlinear=True):
    return nonlinear and D % (2 * K_CHUNK_K) == 0 and qmlp_smem_bytes(C_, D) <= SMEM_CAP


def batched_supported(C_, D, nonlinear=True):
    """fwd_batched.cuh (passing_v aside)."""
    return qmlp_supported(C_, D, nonlinear) and D % 4 == 0 and D <= 2048 and (C_ <= 2 or (C_ <= 4 and D <= 1024))


def models_supported(C_, D, M):
    """dsmil_models_supported: every member on the batched route and the fold kernel's shared memory fits."""
    return batched_supported(C_, D) and qmlp_smem_bytes(C_, D, M) <= SMEM_CAP


def route_edges():
    """{CT: (largest D k_qmlp_sm90 takes, the next multiple of 128 or None at DSMIL_MAX_D)} and the same for the fold
    form of two models."""
    out = {}
    for M in (0, 2):
        for ct in (1, 2, 4, 8):
            ok = (lambda D: qmlp_supported(ct, D)) if M == 0 else (lambda D: models_supported(ct, D, M))
            if ct == 8 and M:
                continue                              # the fold form stops at C = 4
            top = max(D for D in range(128, MAX_D + 1, 128) if ok(D))
            out[(ct, M)] = (top, top + 128 if top + 128 <= MAX_D else None)
    return out


def records(N, kind):
    """[(record, [(lo, hi) of each tile it walks, in order])]: record r takes tiles r, r + P, r + 2P, ..."""
    R, P = (K_ATT_ROWS, recs_for_bag(N)) if kind == "b" else (K_ATTEND_ROWS, attend_ctas(N))
    T = ceil_div(N, R)
    return [[(t * R, min(N, (t + 1) * R)) for t in range(r, T, P)] for r in range(P)]


def fin_slice_rows(N, C_):
    """Rows at the edges of k_finalize_b's kFinSlices A-slices (element e = row * C + k)."""
    per = ceil_div(N * C_, K_FIN_SLICES)
    rows = set()
    for s in range(K_FIN_SLICES):
        lo, hi = per * s, min(N * C_, per * (s + 1))
        if hi > lo:
            rows |= {lo // C_, (hi - 1) // C_}
    return rows


# --------------------------------------------------------------------------------------------------------- cases
@dataclass(frozen=True)
class Case:
    name: str
    route: str                 # single, bags, models, value or shard (see the runners below)
    D: int
    C: int
    Ns: Tuple[int, ...]
    nonlinear: bool = True
    rescale: bool = False      # class-0 maximum in the second tile of a record whose first tile has no probe
    bias: float = 1.5          # nonlinear: b2 = -bias s
    w2_gain: float = 3.0
    beta: float = 10.0         # linear: b1 = -beta s, W1[:, d2] = (beta + 1) s
    passing_v: bool = False
    masked: bool = False       # value route: v's dropout mask
    empty_rank: bool = False   # shard: a rank of G = 3 with no row of the bag holds no probe either (its weight underflows)

    @property
    def seed(self):
        return sum(map(ord, self.name)) % 997

    @property
    def tc_phase1(self):
        return qmlp_supported(self.C, self.D, self.nonlinear)

    @property
    def attend(self):
        """'b': k_attend_b / k_finalize_b (batched_supported); 'g': the generic attend, combine and finalize (also the
        value route's, and the per-bag sharded phase 2's; the batched sharded form, held to the same mirror, walks
        fewer rows per record)."""
        ok = batched_supported(self.C, self.D, self.nonlinear)
        return "b" if ok and not self.passing_v and self.route != "shard" else "g"


SINGLE = [
    Case("tc_d512_c1_n20000_rescale", "single", 512, 1, (20000,), rescale=True, bias=2.5),
    Case("tc_d512_c2_n3000", "single", 512, 2, (3000,)),
    Case("tc_d1024_c4_n2000", "single", 1024, 4, (2000,)),
    Case("tcgen_d512_c6_n1500", "single", 512, 6, (1500,)),
    Case("gen_d166_c2_n2500", "single", 166, 2, (2500,)),
    Case("genlin_d230_c3_n12000_rescale", "single", 230, 3, (12000,), nonlinear=False, rescale=True),
    Case("genlin_d166_c1_n3000", "single", 166, 1, (3000,), nonlinear=False),
    # the generic k_attend<CT, J> (J = ceil(D / 256) rounded up to a power of two; its last 256-column group full or
    # partly empty) and k_qmlp_sm90 at the largest D of each CT, DSMIL_MAX_D = 4096 for CT <= 4
    Case("tc_d4096_c1_n1500", "single", 4096, 1, (1500,)),
    Case("tc_d4096_c2_n1200", "single", 4096, 2, (1200,)),
    Case("tc_d4096_c4_n1000", "single", 4096, 4, (1000,)),
    Case("tc_d2944_c8_n1000", "single", 2944, 8, (1000,)),          # CT = 8: the largest D k_qmlp_sm90 takes
    Case("gen_d3072_c8_n1000", "single", 3072, 8, (1000,)),         # ... and the next multiple of 128: FFMA phase 1
    Case("gen_d4095_c7_n1000", "single", 4095, 7, (1000,)),
    Case("gen_d2049_c2_n1500", "single", 2049, 2, (1500,)),
    Case("genlin_d2048_c2_n2000", "single", 2048, 2, (2000,), nonlinear=False),
    Case("genlin_d1920_c1_n2000", "single", 1920, 1, (2000,), nonlinear=False),
    Case("genlin_d1024_c1_n2000", "single", 1024, 1, (2000,), nonlinear=False),
    Case("genlin_d512_c1_n2000", "single", 512, 1, (2000,), nonlinear=False),
    Case("gen_d300_c2_n2000", "single", 300, 2, (2000,)),
    Case("gen_d1000_c2_n2000", "single", 1000, 2, (2000,)),
    Case("genlin_d512_c3_n2000", "single", 512, 3, (2000,), nonlinear=False),
    Case("gen_d1020_c4_n1500", "single", 1020, 4, (1500,)),
    Case("tc_d1152_c3_n1500", "single", 1152, 3, (1500,)),
    Case("tc_d256_c8_n2000", "single", 256, 8, (2000,)),
    Case("tc_d768_c5_n1500", "single", 768, 5, (1500,)),
    Case("tc_d2048_c8_n1000", "single", 2048, 8, (1000,)),
    Case("tc_d128_c2_n3000", "single", 128, 2, (3000,)),              # k_qmlp_sm90's shortest K loop
]
BAGS = [
    Case("bags_tc_d512_c2", "bags", 512, 2, (1, 127, 128, 129, 3000, 17000), rescale=True, bias=2.5),
    Case("bags_gen_d166_c5", "bags", 166, 5, (1, 31, 32, 33, 2000, 10000)),
    Case("bags_genlin_d230_c2", "bags", 230, 2, (33, 10000), nonlinear=False, rescale=True),
    Case("bags_tc_d512_c1", "bags", 512, 1, (129, 4000)),
    Case("bags_tc_d512_c3", "bags", 512, 3, (2, 128, 2500)),
    Case("bags_gen_d7_c2", "bags", 7, 2, (1, 33, 3000)),
    # k_attend_b<CT, NJ> with its last 512-column group full (D = 512 NJ) or partly empty, and k_qmlp_sm90 at DT = 0
    # in both forms; D = 2048 against 2176 for batched_supported
    Case("bags_tc_d1024_c1", "bags", 1024, 1, (1, 129, 2000)),
    Case("bags_tc_d1024_c2", "bags", 1024, 2, (2, 128, 1500)),
    Case("bags_tc_d2048_c1", "bags", 2048, 1, (129, 1200)),
    Case("bags_tc_d2048_c2", "bags", 2048, 2, (1, 127, 1000)),
    Case("bags_tc_d640_c1", "bags", 640, 1, (33, 1500)),
    Case("bags_tc_d1920_c2", "bags", 1920, 2, (129, 1000)),
    Case("bags_tc_d128_c2", "bags", 128, 2, (1, 129, 3000)),
    Case("bags_tc_d1024_c4", "bags", 1024, 4, (128, 1500)),
    # k_attend_gb<CT, J> over the generic batch, its dev form on the same shapes
    Case("bags_genlin_d256_c1", "bags", 256, 1, (33, 2000), nonlinear=False),
    Case("bags_genlin_d512_c1", "bags", 512, 1, (1, 33, 2000), nonlinear=False),
    Case("bags_genlin_d1024_c1", "bags", 1024, 1, (33, 1500), nonlinear=False),
    Case("bags_genlin_d1920_c1", "bags", 1920, 1, (33, 1200), nonlinear=False),
    Case("bags_tc_d4096_c1", "bags", 4096, 1, (129, 800)),
    Case("bags_gen_d1000_c2", "bags", 1000, 2, (33, 1500)),
    Case("bags_tc_d2176_c2", "bags", 2176, 2, (129, 1200)),
    Case("bags_genlin_d384_c4", "bags", 384, 4, (33, 1500), nonlinear=False),
    Case("bags_gen_d1020_c3", "bags", 1020, 3, (33, 1500)),
    Case("bags_tc_d2048_c3", "bags", 2048, 3, (129, 1000)),
    Case("bags_tc_d4096_c4", "bags", 4096, 4, (33, 700)),
    Case("bags_tc_d512_c6", "bags", 512, 6, (1, 129, 1500)),
    Case("bags_tc_d1280_c8", "bags", 1280, 8, (33, 1000)),
    Case("bags_gen_d777_c5", "bags", 777, 5, (33, 1200)),
    Case("bags_gen_d4095_c8", "bags", 4095, 8, (33, 600)),
]
# the ensemble forms: two models (their own weights) over the same bags
MODELS = [
    Case("models_tc_d512_c2", "models", 512, 2, (129, 3000)),
    Case("models_tc_d512_c1", "models", 512, 1, (129, 1000)),
    Case("models_tc_d512_c3", "models", 512, 3, (129, 1000)),
    Case("models_tc_d1024_c1", "models", 1024, 1, (129, 1000)),
    Case("models_tc_d1024_c2", "models", 1024, 2, (129, 1000)),
    Case("models_tc_d1024_c4", "models", 1024, 4, (129, 800)),      # CT = 4: the largest D of the fold form
    Case("models_tc_d2048_c1", "models", 2048, 1, (129, 800)),      # CT = 1 and 2: the largest (batched_supported)
    Case("models_tc_d2048_c2", "models", 2048, 2, (129, 800)),
]
# dsmil_value_forward_bags (passing_v): V is checked too, and B = A^T V on the kernel's own V
VALUE = [
    Case("value_tc_d512_c2", "value", 512, 2, (129, 2000), passing_v=True),
    Case("value_tc_d512_c2_mask", "value", 512, 2, (129, 2000), passing_v=True, masked=True),
    Case("value_gen_d166_c3_mask", "value", 166, 3, (33, 1500), passing_v=True, masked=True),
    Case("value_tc_d2048_c2", "value", 2048, 2, (129, 800), passing_v=True),
]
# the row-sharded phases at G = 1, 2, 3 virtual ranks: per bag (CudaShardOps) and batched (CudaShardBagOps)
SHARD = [
    Case("shard_tc_d512_c2", "shard", 512, 2, (5, 3001)),
    Case("shard_genlin_d166_c2", "shard", 166, 2, (2, 3001), nonlinear=False, empty_rank=True),
]
ALL = SINGLE + BAGS + MODELS + VALUE + SHARD


def make_params(case: Case, m: int = 0) -> orc.Params:
    p = orc.random_params(case.D, case.C, 700 + case.seed + 31 * m, nonlinear=case.nonlinear, passing_v=case.passing_v)
    rng = np.random.default_rng(900 + case.seed)
    flags = [D0, D1, D2] + [2 + k for k in range(1, case.C)]
    p.Wi[:, flags] = 0.0
    p.Wi[0, D0] = 1.0
    for k in range(1, case.C):
        p.Wi[k, 2 + k] = 1.0
    p.W1[:, flags] = 0.0
    s = np.where(rng.random(KQ) < 0.5, -1.0, 1.0).astype(np.float32)
    if case.nonlinear:
        p.W1[J0, :] = 0.0
        p.W1[J0, D2] = 1.0
        p.b1[J0] = 0.0
        p.W2 *= np.float32(case.w2_gain)
        p.W2[:, J0] = 64.0 * s
        p.b2 = (-case.bias * s).astype(np.float32)
    else:
        p.W1[:, D2] = (case.beta + 1.0) * s
        p.b1 = (p.b1 - case.beta * s).astype(np.float32)
    return p


@dataclass
class Bag:
    X: np.ndarray
    crit0: int                 # the class-0 critical row
    probes: np.ndarray         # sorted probe rows
    rescale_rec: int = -1


def crit_row(case: Case, N):
    if N < 4:
        return 0
    if case.rescale:
        R, P = (K_ATT_ROWS, recs_for_bag(N)) if case.attend == "b" else (K_ATTEND_ROWS, attend_ctas(N))
        if ceil_div(N, R) > P + 1:
            return (P + 1) * R + R // 2          # record 1's second tile
    return N // 2 + 3 if N > 8 else N // 2


def other_crit(N, crit0, k):
    """The critical row of class k >= 1: an ordinary row with x[e_k] = 8."""
    return (crit0 + 7 * k) % N


def probe_rows(case: Case, N, crit0):
    rows = {r for r in (0, 127, 128, 129, N - 1) if r < N}
    recs = records(N, case.attend)
    skip = -1
    for r, tiles in enumerate(recs):
        if any(lo <= crit0 < hi for lo, hi in tiles[1:]):
            skip = r                              # its first tile must stay below the maximum: no probe there
    for r, tiles in enumerate(recs):
        for j in {0, len(tiles) - 1}:
            lo, hi = tiles[j]
            if not (r == skip and j == 0):
                rows |= {lo, hi - 1}
    if case.attend == "b":
        rows |= fin_slice_rows(N, case.C)
    if skip >= 0:
        lo, hi = recs[skip][0]
        rows = {x for x in rows if not lo <= x < hi}
    if not case.nonlinear and case.route != "shard" and len(recs) > 2:
        # the last record holds no probe: with linear q its rows, and so its combine weight, underflow in fp32
        rows = {x for x in rows if not any(lo <= x < hi for lo, hi in recs[-1])}
    if case.route == "shard":
        for G in (2, 3):
            rows |= {x for lo, hi in orc.shard_bounds(N, G) if hi > lo for x in (lo, hi - 1)}
        if case.empty_rank:
            lo, hi = orc.shard_bounds(N, 3)[2]
            rows = {x for x in rows if not lo <= x < hi}
    others = {other_crit(N, crit0, k) for k in range(1, case.C)}
    return np.array(sorted(rows - {crit0} - others), np.int64), skip


@functools.lru_cache(maxsize=None)
def bags(case: Case):
    out = []
    for b, N in enumerate(case.Ns):
        X = orc.synthetic_bag(N, case.D, 1000 * case.seed + b, "uniform" if case.D % 128 == 0 else "normal")
        X[:, [D0, D1, D2] + [2 + k for k in range(1, case.C)]] = 0.0
        if N < 4:
            out.append(Bag(X, 0, np.zeros(0, np.int64)))
            continue
        c0 = crit_row(case, N)
        if case.empty_rank:
            c0 = N // 4                          # the last of three ranks holds no critical row and no probe
        probes, skip = probe_rows(case, N, c0)
        if not case.nonlinear:
            X[c0, 2 + case.C:] = 0.0            # q_max = b1 + s: the largest logit stays near 11.3
        X[c0, D0] = 8.0
        X[c0, D1] = 0.25
        X[c0, D2] = 16.0 if case.nonlinear else 1.0
        for k in range(1, case.C):
            X[other_crit(N, c0, k), 2 + k] = 8.0
        for i, r in enumerate(probes):
            X[r] = X[c0]
            X[r, D0] = 0.0
            X[r, D1] = 1.0 + 0.5 * (i + 1) / len(probes)
        out.append(Bag(X, c0, probes, skip))
    return out


# ---------------------------------------------------------------------------------------------- the restatement
def restate(Q, crit, X, p: orc.Params, dtype=np.float64, wS=None, wB=None):
    """q_max = Q[crit] ... pred in plain numpy at `dtype`; X is the value matrix B is taken over (the bag, or V).  wS /
    wB [N] weight each row's term in the normaliser S and in B (0 drops the row from that sum, 2 counts it twice).
    Returns dict(L, M, A, B, pred)."""
    f = dtype
    Q, X = np.asarray(Q, f), np.asarray(X, f)
    L = (Q @ Q[np.asarray(crit)].T) / f(SCALE)
    M = L.max(0)
    E = np.exp(L - M)
    S = ((E if wS is None else E * np.asarray(wS, f)[:, None])).sum(0)
    A = E / S
    B = (A if wB is None else A * np.asarray(wB, f)[:, None]).T @ X
    Cc = p.C
    pred = np.asarray(p.Wf, f).reshape(Cc, -1) @ B.reshape(-1) + np.asarray(p.bf, f)
    return dict(L=L, M=M, A=A, B=B, pred=pred)


def b_depth(N, kind):
    """Longest chain of fp32 additions into one element of B: a thread's rows of every tile of its record (k_attend_b:
    one row parity of 128-row tiles; k_attend: 32-row tiles), then the record combine (k_finalize_b: P / 8 per thread
    and 8 partials; k_combine_rec: all P in turn)."""
    tiles = records(N, kind)
    tpr, P = max(len(t) for t in tiles), len(tiles)
    return 64 * tpr + ceil_div(P, 8) + 8 if kind == "b" else 32 * tpr + P + 8


def a_bars(Q, crit, X, p, r64, kind):
    """Per element bars of A [N, C] (relative), B [C, D] and pred [C] (absolute) of one bag, from the fp64 restatement
    r64 on the same Q."""
    Q = np.asarray(Q, np.float64)
    qm = Q[np.asarray(crit)]
    L, M, A = r64["L"], r64["M"], r64["A"]
    eL = C_L * U * (np.abs(Q) @ np.abs(qm).T) / SCALE + U * np.abs(L)
    row = eL + 2 * U * np.abs(L - M)            # an error in M cancels between exp(L - M) and S
    tau = row + (A * row).sum(0) + C_A * U
    depth = b_depth(X.shape[0], kind)
    aX = np.abs(np.asarray(X, np.float64))
    # rows of fp64 A below FLT_MIN contribute nothing in fp32 (their exp, or their record's weight, underflows)
    tiny = A < 2 * FLT_MIN
    B_bar = (A * (tau + depth * U)).T @ aX + (A * tiny).T @ aX + FLT_MIN * aX.sum(0)
    mag = A.T @ aX
    Wf = np.abs(np.asarray(p.Wf, np.float64)).reshape(p.C, -1)
    P_bar = Wf @ B_bar.reshape(-1) + C_P * U * (Wf @ mag.reshape(-1))
    return tau, B_bar, P_bar


def over(err, bar):
    """Largest err / bar; an element with a zero bar must be exact (a NaN error fails)."""
    err, bar = np.asarray(err, np.float64), np.asarray(bar, np.float64)
    if np.isnan(err).any():
        return np.inf
    zero = bar == 0
    if np.any(err[zero] != 0):
        return np.inf
    return float(np.max(err[~zero] / bar[~zero])) if (~zero).any() else 0.0


def a_err(A, r64, tau):
    """Largest |A - A64| / (tau A64) over the normal-range entries, and whether the rest are 0 or subnormal."""
    A64 = r64["A"]
    norm = A64 >= 2 * FLT_MIN
    e = np.abs(np.asarray(A, np.float64) - A64)
    worst = over(e[norm], tau[norm] * A64[norm])
    tiny_ok = bool(np.all(np.abs(np.asarray(A, np.float64)[~norm]) <= 4 * FLT_MIN))
    return worst, tiny_ok


def stage_bars(X, p, H1, tc, v_mask=None):
    """Reference and bar of H1 (nonlinear), of Q from the kernel's own H1 (or X, linear q) and of V (passing_v, from
    the masked input)."""
    f = np.float64
    X64 = np.asarray(X, f)
    out = {}
    if p.passing_v:
        Xv = X64 if v_mask is None else X64 * np.asarray(v_mask, f)
        zv = Xv @ p.Wv.astype(f).T + p.bv
        out["V"] = (np.maximum(zv, 0), C_MM * U * (np.abs(Xv) @ np.abs(p.Wv.astype(f)).T + np.abs(p.bv)))
    mm = (lambda a, w: orc.matmul_3xbf16(a, w)) if tc else (lambda a, w: np.asarray(a, f) @ np.asarray(w, f).T)
    if p.nonlinear:
        z1 = mm(X, p.W1) + p.b1
        out["H1"] = (np.maximum(z1, 0), C_MM * U * (np.abs(X64) @ np.abs(p.W1.astype(f)).T + np.abs(p.b1)))
        H = np.asarray(H1, f)
        z2 = mm(H1, p.W2) + p.b2
        q = np.tanh(z2)
        out["Q"] = (q, (1 - q * q) * C_MM * U * (np.abs(H) @ np.abs(p.W2.astype(f)).T + np.abs(p.b2)) + TANH_ABS)
    else:
        z = X64 @ p.W1.astype(f).T + p.b1
        out["Q"] = (z, C_MM * U * (np.abs(X64) @ np.abs(p.W1.astype(f)).T + np.abs(p.b1)))
    return out


def mm3_fp32_stage(X, p, H1):
    """H1 and Q of the tensor-core path restated in fp32: the exact bf16 split products accumulated in float32."""
    def mm(a, w):
        ah, al = orc.split_bf16(a)
        wh, wl = orc.split_bf16(w)
        return (ah @ wh.T + al @ wh.T + ah @ wl.T).astype(np.float32)
    h = np.maximum(mm(np.asarray(X, np.float32), p.W1) + p.b1, np.float32(0))
    return {"H1": h, "Q": np.tanh(mm(np.asarray(H1, np.float32), p.W2) + p.b2)}


def classes_bar(X, p):
    f = np.float64
    c = np.asarray(X, f) @ p.Wi.astype(f).T + p.bi
    return c, C_CLS * U * (np.abs(np.asarray(X, f)) @ np.abs(p.Wi.astype(f)).T + np.abs(p.bi))


# ===================================================================================== CPU part: no device needed
def _src(name):
    return open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dsmil_wsi_b200", "csrc",
                             name)).read()


def test_mirror_constants_are_the_sources():
    def const(src, nm):
        return int(re.search(rf"constexpr int {nm} = (\d+);", src).group(1))
    fb, fk, cm = _src("fwd_batched.cuh"), _src("fwd_kernels.cuh"), _src("common.cuh")
    assert (const(fb, "kAttRows"), const(fb, "kMaxRecPerBag"), const(fb, "kFinSlices")) == \
        (K_ATT_ROWS, K_MAX_REC_PER_BAG, K_FIN_SLICES)
    assert (const(fk, "kAttendRows"), const(cm, "kSplits")) == (K_ATTEND_ROWS, K_SPLITS)
    plan = _src("bag_plan.cuh")
    assert "t < sm90::kMaxRecPerBag ? (t < 1 ? 1 : t) : sm90::kMaxRecPerBag" in plan
    assert "tiles < kSplits ? (tiles < 1 ? 1 : tiles) : kSplits" in plan
    sm, hd = _src("fwd_sm90.cuh"), _src(os.path.join("..", "..", "include", "dsmil_b200.h"))
    assert (const(sm, "kWStages"), const(sm, "kChunkK"), const(sm, "kSmemBags"), const(sm, "kTileM")) == \
        (K_WSTAGES, K_CHUNK_K, K_SMEM_BAGS, KQ)
    for line in ("constexpr int kTileBytes = kQ * kChunkK * 2;", "constexpr int kChunkBytes = 2 * kTileBytes;",
                 "constexpr int kOffWi = kOffWRing + kWStages * kChunkBytes;", "constexpr int kSmemFixed = kOffWi;",
                 "return kSmemFixed + sizeof(float) * ct * D + 1024;",
                 "return kSmemFixed + sizeof(float) * M * (static_cast<size_t>(ct_of(C)) * D + kModelBiasFloats) + 1024;",
                 "constexpr int kModelBiasFloats = 2 * kQ + kMaxC;",
                 "constexpr size_t kQmlpStaticSmem = 2 * kQ * sizeof(float) + kSmemBags * sizeof(BagDev) + 256;",
                 f"p->D % (2 * kChunkK) == 0 && qmlp_smem_bytes(p->C, p->D) + kQmlpStaticSmem <= {SMEM_CAP};",
                 f"return qmlp_models_smem_bytes(C, D, M) + kQmlpStaticSmem <= {SMEM_CAP};",
                 "inline int ct_of(int C) { return C <= 1 ? 1 : (C <= 2 ? 2 : (C <= 4 ? 4 : 8)); }"):
        assert line in sm, line
    # sizeof(BagDev) = 40: a pointer, three 8-byte integers' worth of fields, four ints
    bag = re.search(r"struct BagDev \{(.*?)\};", sm, re.S).group(1)
    assert re.findall(r"^\s*(const float\*|long long|int) ", bag, re.M) == \
        ["const float*", "long long", "long long", "int", "int", "int", "int"]
    assert "return qmlp_supported(p) && !p->passing_v && p->D % 4 == 0 && p->D <= 2048 && p->C <= 4 &&\n" \
           "         ((p->C <= 2) || p->D <= 1024);" in fb
    assert (int(re.search(r"#define DSMIL_MAX_D (\d+)", hd).group(1)),
            int(re.search(r"#define DSMIL_MAX_C (\d+)", hd).group(1))) == (MAX_D, K_MAX_C)
    from dsmil_wsi_b200.sharded import shard_bounds
    for N in (1, 2, 7, 128, 20000):
        for G in (1, 2, 3):
            assert list(shard_bounds(N, G)) == list(orc.shard_bounds(N, G))


def attend_instance(case: Case):
    """(kernel, CT, J or NJ) of the attend pass the case's forward launches."""
    if case.attend == "b":
        return ("k_attend_b", ct_of(case.C), 1 if case.D <= 512 else 2 if case.D <= 1024 else 4)
    J = 1
    while 256 * J < case.D:
        J *= 2
    return ("k_attend" if case.route in ("single", "shard") else "k_attend_gb", ct_of(case.C), J)


def test_cases_reach_every_column_edge_and_route_edge():
    """Each J of the generic attend passes and each NJ of k_attend_b has a case whose last column group is full and
    one where it is partly empty; k_qmlp_sm90 runs at D = 128, at the largest D of each CT (one- and two-model forms)
    and one multiple of 128 beyond it falls to the generic phase 1; D = 2048 and 2176 straddle batched_supported."""
    seen = {}
    for case in ALL:
        kern, ct, j = attend_instance(case)
        width = 512 if kern == "k_attend_b" else 256
        seen.setdefault((kern, j), set()).add(case.D == width * j)
        seen.setdefault((kern, ct, j), set()).add(True)
    for kern, js in (("k_attend", (1, 2, 4, 8, 16)), ("k_attend_gb", (1, 2, 4, 8, 16)), ("k_attend_b", (1, 2, 4))):
        for j in js:
            assert seen.get((kern, j)) == {True, False}, (kern, j, seen.get((kern, j)))
    for ct in (1, 2, 4, 8):
        for kern in ("k_attend", "k_attend_gb"):
            assert all((kern, ct, j) in seen for j in (1, 2, 4, 8, 16)), (kern, ct)
    edges = route_edges()
    assert edges[(8, 0)] == (2944, 3072) and edges[(4, 0)] == (4096, None) and edges[(4, 2)] == (1024, 1152)
    for (ct, M), (top, nxt) in edges.items():
        pool = SINGLE + BAGS if M == 0 else MODELS
        assert any(ct_of(c.C) == ct and c.D == top and c.tc_phase1 for c in pool), (ct, M, top)
        if nxt is not None and M == 0:
            assert any(ct_of(c.C) == ct and c.D == nxt and c.nonlinear and not c.tc_phase1 for c in pool), (ct, nxt)
        if nxt is not None and M:
            assert not models_supported(ct, nxt, M) and qmlp_supported(ct, nxt)
    assert any(c.D == 128 and c.tc_phase1 for c in ALL)
    on_b = {c.D for c in BAGS if c.attend == "b" and c.C <= 2}
    off_b = {c.D for c in BAGS if c.attend == "g" and c.tc_phase1 and c.C <= 2}
    assert 2048 in on_b and 2176 in off_b


def test_records_tile_every_row_once_and_cases_sit_on_their_boundaries():
    for case in ALL:
        for N, bag in zip(case.Ns, bags(case)):
            cover = np.zeros(N, np.int64)
            for tiles in records(N, case.attend):
                for lo, hi in tiles:
                    cover[lo:hi] += 1
            assert np.all(cover == 1), (case.name, N)
            if case.rescale and N == max(case.Ns):
                R = K_ATT_ROWS if case.attend == "b" else K_ATTEND_ROWS
                P = recs_for_bag(N) if case.attend == "b" else attend_ctas(N)
                assert N > P * R and bag.rescale_rec == 1, (case.name, N)     # records own two tiles
    assert {SINGLE[0].attend, SINGLE[3].attend, SINGLE[4].attend} == {"b", "g"} and SINGLE[3].tc_phase1
    assert max(SINGLE[0].Ns) > K_ATT_ROWS * K_MAX_REC_PER_BAG and max(SINGLE[5].Ns) > K_ATTEND_ROWS * K_SPLITS


def v_masks(case: Case):
    """v's dropout mask per bag (scaled by 1 / 0.75), or None."""
    if not case.masked:
        return [None] * len(case.Ns)
    rng = np.random.default_rng(77 + case.seed)
    return [((rng.random((n, case.D)) >= 0.25) / np.float32(0.75)).astype(np.float32) for n in case.Ns]


@functools.lru_cache(maxsize=None)
def cpu_forward(case: Case):
    """The fp32 oracle forward of every bag, standing in for the device's classes, crit, Q and V."""
    p = make_params(case)
    return p, [orc.forward(b.X, p, dtype=np.float32, v_mask=m) for b, m in zip(bags(case), v_masks(case))]


def test_restatement_in_fp64_is_the_oracle_forward():
    for case in (SINGLE[1], SINGLE[5], BAGS[1]):
        p = make_params(case)
        for b in bags(case):
            t = orc.forward(b.X, p)
            r = restate(t.Q, t.idx, b.X, p)
            for k, want in (("A", t.A), ("B", t.B.reshape(p.C, -1)), ("pred", t.prediction_bag.reshape(-1))):
                assert np.max(np.abs(r[k] - want)) <= 1e-12 * max(np.max(np.abs(want)), 1e-300), (case.name, k)


@pytest.mark.parametrize("case", ALL, ids=lambda c: c.name)
def test_bags_are_peaked_and_probe_rows_share_the_maximum(case):
    """Class 0: the probe rows hold the maximum logit; A spans at least five decades (nonlinear) or logits spread over
    more than 100 with rows underflowing in fp32 (linear q); the rescale cases need e^-10 or less on a first tile."""
    p, fos = cpu_forward(case)
    for b, fo in zip(bags(case), fos):
        N = b.X.shape[0]
        if N < 4:
            continue
        assert fo.idx[0] == b.crit0 and all(fo.idx[k] == other_crit(N, b.crit0, k) for k in range(1, case.C)), case.name
        assert np.array_equal(fo.Q[b.probes], np.broadcast_to(fo.Q[b.crit0], (len(b.probes), KQ)))
        r = restate(fo.Q, fo.idx, fo.V, p)
        L = r["L"][:, 0]
        assert np.all(L[b.probes] == L.max())
        if N < 1000:
            continue
        if case.nonlinear:
            A = r["A"][:, 0]
            assert A.max() / A.min() > 1e5, (case.name, A.max() / A.min())
        else:
            zero = r["A"][:, 0].astype(np.float32) == 0
            assert L.max() - L.min() > 100 and np.mean(zero) > 0.5, case.name
            assert any(all(zero[lo:hi].all() for lo, hi in t) for t in records(N, case.attend)), case.name
        if case.empty_rank:               # the probe-free rank: its combine weight exp(m_r - M) underflows in fp32
            lo, hi = orc.shard_bounds(N, 3)[2]
            assert np.float32(np.exp(L[lo:hi].max() - L.max())) == 0, case.name
        if b.rescale_rec >= 0:
            first = records(N, case.attend)[b.rescale_rec][0]
            assert np.exp(L[first[0]:first[1]].max() - L.max()) <= RESCALE_MAX, case.name


def _err_over_bar(case, p, X, fo32, Q):
    """Errors over bars of every stage of the fp32 stand-in fo32 against the fp64 restatement on Q (and fo32's V)."""
    crit = fo32.idx
    r64 = restate(Q, crit, fo32.V, p)
    tau, Bb, Pb = a_bars(Q, crit, fo32.V, p, r64, case.attend)
    ea, tiny_ok = a_err(fo32.A, r64, tau)
    out = {"A": ea, "B": over(np.abs(fo32.B.reshape(p.C, -1) - r64["B"]), Bb),
           "pred": over(np.abs(fo32.prediction_bag.reshape(-1) - r64["pred"]), Pb)}
    c, cb = classes_bar(X, p)
    out["classes"] = over(np.abs(fo32.classes - c), cb)
    return out, tiny_ok


@pytest.mark.parametrize("case", ALL, ids=lambda c: c.name)
def test_fp32_restatement_stays_4x_under_every_bar(case):
    p, fos = cpu_forward(case)
    worst = {}
    for b, fo, vm in zip(bags(case), fos, v_masks(case)):
        errs, tiny_ok = _err_over_bar(case, p, b.X, fo, fo.Q)
        assert tiny_ok, case.name
        st = stage_bars(b.X, p, fo.H1, False, v_mask=vm)
        for k, (ref, bar) in st.items():
            errs[k] = over(np.abs(np.asarray(getattr(fo, k), np.float64) - ref), bar)
        if case.tc_phase1:                 # the 3xBF16 products accumulated in fp32, against the same in fp64
            for k, (ref, bar) in stage_bars(b.X, p, fo.H1, True).items():
                if k != "V":
                    errs[k + "_3xbf16"] = over(np.abs(mm3_fp32_stage(b.X, p, fo.H1)[k] - ref), bar)
        for k, v in errs.items():
            worst[k] = max(worst.get(k, 0.0), v)
    assert all(v <= 0.25 for v in worst.values()), (case.name, worst)


def moves(Q, crit, X, p, r64, bars, rows):
    """For each row: the least over (S, B) x (drop, double) of the largest move of a checked output over its bar."""
    tau, Bb, Pb = bars
    N = X.shape[0]
    norm = r64["A"] >= 2 * FLT_MIN
    out = {}
    for r in rows:
        least = np.inf
        for which in ("S", "B"):
            for wgt in (0.0, 2.0):
                w = np.ones(N)
                w[r] = wgt
                g = restate(Q, crit, X, p, wS=w if which == "S" else None, wB=w if which == "B" else None)
                mv = max(over(np.abs(g["A"] - r64["A"])[norm], (tau * r64["A"])[norm]),
                         over(np.abs(g["B"] - r64["B"]), Bb), over(np.abs(g["pred"] - r64["pred"]), Pb))
                least = min(least, mv)
        out[int(r)] = least
    return out


@pytest.mark.parametrize("case", ALL, ids=lambda c: c.name)
def test_one_lost_or_repeated_probe_row_moves_a_checked_output_past_20x_its_bar(case):
    p, fos = cpu_forward(case)
    for b, fo in zip(bags(case), fos):
        if len(b.probes) == 0:
            continue
        r64 = restate(fo.Q, fo.idx, fo.V, p)
        mv = moves(fo.Q, fo.idx, fo.V, p, r64, a_bars(fo.Q, fo.idx, fo.V, p, r64, case.attend), b.probes)
        weakest = min(mv.items(), key=lambda kv: kv[1])
        assert weakest[1] > SENSITIVITY, (case.name, b.X.shape[0], weakest)


# ========================================================================================== GPU part (one H100)
def _np(t):
    return t.detach().cpu().numpy()


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _pack(p):
    from dsmil_wsi_b200 import functional as Fn
    return Fn.ParamPack(*[None if a is None else _t(a) for a in (p.Wi, p.bi, p.W1, p.b1, p.W2, p.b2, p.Wv, p.bv,
                                                                   p.Wf, p.bf)])


def _ws(nbytes):
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device="cuda")


def _nan(*s):
    return torch.full(s, float("nan"), device="cuda")


def _forward_plain(lib, fn):
    """fn() with the attend pass launched after phase 1 instead of overlapped with it (profiling on); the recorded
    event pairs are drained before profiling is turned off again."""
    torch.cuda.synchronize()
    lib.dsmil_profile_enable(1)
    try:
        return fn()
    finally:
        torch.cuda.synchronize()
        lib.dsmil_profile_read((C.c_double * 8)(), (C.c_uint64 * 8)())
        lib.dsmil_profile_enable(0)


def _outs(o, crit, Ns, row0=0, b0=0, saves=()):
    """Per-bag host copies of packed outputs (rows from row0, bags from b0); saves: the names of kept activations."""
    h = {k: _np(v) for k, v in o.items() if v is not None}
    crit_h = _np(crit).reshape(-1, o["pred"].shape[-1])
    per, lo = [], row0
    for j, n in enumerate(Ns):
        b = b0 + j
        d = {"A": h["A"][lo:lo + n], "pred": h["pred"][b:b + 1], "B": h["B"][b:b + 1], "crit": crit_h[b]}
        for k in ("classes",) + tuple(saves):
            if k in h:
                d[k] = h[k][lo:lo + n]
        per.append(d)
        lo += n
    return per


def _new_outs(rows, nb, case, saves=False):
    Cc, D = case.C, case.D
    o = dict(classes=_nan(rows, Cc), pred=_nan(nb, Cc), A=_nan(rows, Cc), B=_nan(nb, Cc, D))
    if saves:
        o.update(Q=_nan(rows, KQ), H1=_nan(rows, KQ) if case.nonlinear else None,
                 V=_nan(rows, D) if case.passing_v else None)
    return o, torch.full((nb, Cc), -7, dtype=torch.int64, device="cuda")


def run_single(case: Case, lib, P, X):
    """dsmil_forward: training (saves), eval overlapped, eval plain; dsmil_bag_forward on the training call's classes."""
    N = X.shape[0]
    x = _t(X)
    ws = _ws(lib.dsmil_forward_workspace_bytes(P.ref, N))
    outs = {}
    for form in ("train", "eval", "eval_plain", "bag_forward"):
        o, crit = _new_outs(N, 1, case, saves=form == "train")
        heads = [_ptr(o[k]) for k in ("pred", "A", "B")] + [crit.data_ptr(), _ptr(o.get("Q")), _ptr(o.get("H1")), None,
                                                             ws.data_ptr(), ws.numel(), _stream()]
        if form == "bag_forward":
            o.pop("classes")
            cin = _t(outs["train"][0]["classes"])
            call = lambda: lib.dsmil_bag_forward(P.ref, x.data_ptr(), None, cin.data_ptr(), N, *heads)
        else:
            call = lambda: lib.dsmil_forward(P.ref, x.data_ptr(), None, N, o["classes"].data_ptr(), *heads)
        rc = _forward_plain(lib, call) if form == "eval_plain" else call()
        torch.cuda.synchronize()
        assert rc == 0, lib.dsmil_last_error()
        outs[form] = _outs(o, crit, [N], saves=("Q", "H1"))
    return outs


def _slots(Xs, D):
    max_rows = max(X.shape[0] for X in Xs)
    slots = torch.zeros(len(Xs), max_rows, D, device="cuda")
    for b, X in enumerate(Xs):
        slots[b, :X.shape[0]].copy_(torch.from_numpy(X))
    xs = slots.data_ptr() + 4 * max_rows * D * torch.arange(len(Xs), dtype=torch.int64, device="cuda")
    return slots, xs, max_rows


def run_bags(case: Case, lib, P, Xs):
    """dsmil_forward_bags_train (saves), dsmil_forward_bags, and the capture-safe pair over [nb, max_rows, D] slots
    (dsmil_forward_bags_train_dev / _dev, or their dsmil_generic_* forms on the generic shapes)."""
    Ns = list(case.Ns)
    nb, total = len(Ns), sum(Ns)
    xs = [_t(X) for X in Xs]
    c_X, c_N = (C.c_void_p * nb)(*[x.data_ptr() for x in xs]), (C.c_int64 * nb)(*Ns)
    outs = {}
    for form in ("train", "eval"):
        o, crit = _new_outs(total, nb, case, saves=form == "train")
        args = [_ptr(o[k]) for k in ("classes", "pred", "A", "B")] + [crit.data_ptr()]
        if form == "train":
            ws = _ws(lib.dsmil_forward_bags_train_workspace_bytes(P.ref, c_N, nb))
            rc = lib.dsmil_forward_bags_train(P.ref, c_X, c_N, nb, *args, _ptr(o["Q"]), _ptr(o["H1"]), ws.data_ptr(),
                                              ws.numel(), _stream())
        else:
            ws = _ws(lib.dsmil_forward_bags_workspace_bytes(P.ref, c_N, nb))
            rc = lib.dsmil_forward_bags(P.ref, c_X, c_N, nb, *args, ws.data_ptr(), ws.numel(), _stream())
        torch.cuda.synchronize()
        assert rc == 0, lib.dsmil_last_error()
        outs[form] = _outs(o, crit, Ns, saves=("Q", "H1"))
    pre = "dsmil_" if lib.dsmil_shard_bags_supported(P.ref) else "dsmil_generic_"
    assert (pre == "dsmil_") == (case.attend == "b"), case.name
    slots, xd, max_rows = _slots(Xs, case.D)
    Nd = torch.tensor(Ns, dtype=torch.int64, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    for form in ("train_dev", "eval_dev"):
        train = form == "train_dev"
        o, crit = _new_outs(nb * max_rows, nb, case, saves=train)
        name = pre + ("forward_bags_train_dev" if train else "forward_bags_dev")
        ws = _ws(getattr(lib, name + "_workspace_bytes")(P.ref, nb, max_rows))
        saves = [_ptr(o["Q"]), _ptr(o["H1"])] if train else []
        rc = getattr(lib, name)(P.ref, xd.data_ptr(), Nd.data_ptr(), nb, max_rows,
                                *[_ptr(o[k]) for k in ("classes", "pred", "A", "B")], crit.data_ptr(), *saves,
                                status.data_ptr(), ws.data_ptr(), ws.numel(), _stream())
        torch.cuda.synchronize()
        assert rc == 0 and int(status) == 0, (lib.dsmil_last_error(), int(status))
        outs[form] = _outs(o, crit, Ns, saves=("Q", "H1"))
    return outs


def run_models(case: Case, lib, Ps, Xs):
    """The fold forms for M models over the same bags: dsmil_forward_bags_models (eval, model-major outputs),
    dsmil_forward_bags_models_train (each model given the bags) and its _dev form over slots.  Per model: outs."""
    from dsmil_wsi_b200 import _lib
    M, Ns = len(Ps), list(case.Ns)
    nb, total = len(Ns), sum(Ns)
    c_ps = (_lib.DsmilParams * M)(*[P.struct for P in Ps])
    assert lib.dsmil_models_supported(c_ps, M)
    xs = [_t(X) for X in Xs]
    outs = [dict() for _ in range(M)]
    # eval: M x the same nb bags
    c_X, c_N = (C.c_void_p * nb)(*[x.data_ptr() for x in xs]), (C.c_int64 * nb)(*Ns)
    o, crit = _new_outs(M * total, M * nb, case)
    ws = _ws(lib.dsmil_forward_bags_models_workspace_bytes(c_ps, M, c_N, nb))
    rc = lib.dsmil_forward_bags_models(c_ps, M, c_X, c_N, nb, *[_ptr(o[k]) for k in ("classes", "pred", "A", "B")],
                                       crit.data_ptr(), ws.data_ptr(), ws.numel(), _stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.dsmil_last_error()
    for m in range(M):
        outs[m]["models_eval"] = _outs(o, crit, Ns, m * total, m * nb)
    # training: model m's own bags are the same list (entries model-major)
    c_Xt, c_Nt = (C.c_void_p * (M * nb))(*[x.data_ptr() for x in xs] * M), (C.c_int64 * (M * nb))(*Ns * M)
    c_nb = (C.c_int32 * M)(*[nb] * M)
    o, crit = _new_outs(M * total, M * nb, case, saves=True)
    ws = _ws(lib.dsmil_forward_bags_models_train_workspace_bytes(c_ps, M, c_Nt, c_nb))
    rc = lib.dsmil_forward_bags_models_train(c_ps, M, c_Xt, c_Nt, c_nb, *[_ptr(o[k]) for k in ("classes", "pred", "A",
                                                                                               "B")],
                                             crit.data_ptr(), _ptr(o["Q"]), _ptr(o["H1"]), ws.data_ptr(), ws.numel(),
                                             _stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.dsmil_last_error()
    for m in range(M):
        outs[m]["train"] = _outs(o, crit, Ns, m * total, m * nb, saves=("Q", "H1"))
    slots, xd, max_rows = _slots(Xs * M, case.D)
    Nd = torch.tensor(Ns * M, dtype=torch.int64, device="cuda")
    status = torch.zeros(M, dtype=torch.int32, device="cuda")
    o, crit = _new_outs(M * nb * max_rows, M * nb, case, saves=True)
    ws = _ws(lib.dsmil_forward_bags_models_train_dev_workspace_bytes(c_ps, M, c_nb, max_rows))
    rc = lib.dsmil_forward_bags_models_train_dev(c_ps, M, xd.data_ptr(), Nd.data_ptr(), c_nb, max_rows,
                                                 *[_ptr(o[k]) for k in ("classes", "pred", "A", "B")], crit.data_ptr(),
                                                 _ptr(o["Q"]), _ptr(o["H1"]), status.data_ptr(), ws.data_ptr(),
                                                 ws.numel(), _stream())
    torch.cuda.synchronize()
    assert rc == 0 and _np(status).tolist() == [0] * M, lib.dsmil_last_error()
    for m in range(M):
        outs[m]["train_dev"] = _outs(o, crit, Ns, m * nb * max_rows, m * nb, saves=("Q", "H1"))
    return outs


def run_value(case: Case, lib, P, Xs, vms):
    """dsmil_value_forward_bags with saves (Q, H1, V) and without, on v's masked inputs when the case has a mask."""
    Ns = list(case.Ns)
    nb, total = len(Ns), sum(Ns)
    xs = [_t(X) for X in Xs]
    xvs = None if vms[0] is None else [x * _t(m) for x, m in zip(xs, vms)]
    c_X, c_N = (C.c_void_p * nb)(*[x.data_ptr() for x in xs]), (C.c_int64 * nb)(*Ns)
    c_XV = None if xvs is None else (C.c_void_p * nb)(*[x.data_ptr() for x in xvs])
    assert lib.dsmil_value_bags_supported(P.ref)
    ws = _ws(lib.dsmil_value_forward_bags_workspace_bytes(P.ref, c_N, nb))
    outs = {}
    for form in ("train", "eval"):
        o, crit = _new_outs(total, nb, case, saves=form == "train")
        rc = lib.dsmil_value_forward_bags(P.ref, c_X, c_XV, c_N, nb, *[_ptr(o[k]) for k in ("classes", "pred", "A",
                                                                                         "B")],
                                          crit.data_ptr(), _ptr(o.get("Q")), _ptr(o.get("H1")), _ptr(o.get("V")),
                                          ws.data_ptr(), ws.numel(), _stream())
        torch.cuda.synchronize()
        assert rc == 0, lib.dsmil_last_error()
        outs[form] = _outs(o, crit, Ns, saves=("Q", "H1", "V"))
    return outs


def run_shard_per_bag(case: Case, P, X, G, crafted=False):
    """CudaShardOps over G virtual ranks of one bag: phase 1 (training form), the candidate merge, phase 2, the merge
    of the partial records and phase 3.  crafted: phase 2 gets Q x 3 (and its q_max rows) instead of the saved Q."""
    from dsmil_wsi_b200.sharded import CudaShardOps
    ops = CudaShardOps(P.tensors)
    x = _t(X)
    bounds = orc.shard_bounds(X.shape[0], G)
    p1 = [ops.phase1_train(x[lo:hi], lo) for lo, hi in bounds]
    qmax, crit = ops.merge_candidates(torch.stack([r[4] for r in p1]), G)
    Q = torch.cat([r[1] for r in p1])
    assert torch.equal(qmax, Q[crit]), "q_max is not the critical rows' saved Q"
    if crafted:
        Q = Q * 3.0
        qmax = Q[crit].contiguous()
    Ql = [Q[lo:hi] for lo, hi in bounds]
    p2 = [ops.phase2(x[lo:hi], q, qmax) for (lo, hi), q in zip(bounds, Ql)]
    rec = ops.merge_partials(torch.stack([r[1] for r in p2]), G)
    p3 = [ops.phase3(rec, A) for A, _ in p2]
    for _, B, pred in p3[1:]:                      # every rank derives the same B and bag logits
        assert torch.equal(B, p3[0][1]) and torch.equal(pred, p3[0][2])
    o = dict(classes=torch.cat([r[0] for r in p1]), A=torch.cat([r[0] for r in p3]), B=p3[0][1], pred=p3[0][2],
             Q=Q, H1=torch.cat([r[2] for r in p1]) if case.nonlinear else None)
    return _outs(o, crit, [X.shape[0]], saves=("Q", "H1"))[0]


def run_shard_bags(case: Case, P, Xs, G):
    """CudaShardBagOps over G virtual ranks of the whole batch (every rank holds rows of every bag)."""
    from dsmil_wsi_b200.sharded import CudaShardBagOps
    ranks = [CudaShardBagOps(P.tensors) for _ in range(G)]
    bounds = [orc.shard_bounds(X.shape[0], G) for X in Xs]
    xs = [_t(X) for X in Xs]
    for r, ops in enumerate(ranks):
        ops.begin([x[bd[r][0]:bd[r][1]] for x, bd in zip(xs, bounds)], [bd[r][0] for bd in bounds])
    p1 = [ops.phase1_train() for ops in ranks]
    cands = torch.stack([r[3] for r in p1])
    p2 = [ops.phase2_train(r[1], cands, G) for ops, r in zip(ranks, p1)]
    recs = torch.stack([r[3] for r in p2])
    p3 = [ops.phase3_train(recs, G, r[0]) for ops, r in zip(ranks, p2)]
    per = []
    for b, bd in enumerate(bounds):
        rows = lambda t, r: t[sum(bounds[c][r][1] - bounds[c][r][0] for c in range(b)):][:bd[r][1] - bd[r][0]]
        cat = lambda i, k: torch.cat([rows(res[i], r) for r, res in enumerate(k)])
        crit = p2[0][1][b]
        for r in range(1, G):
            assert torch.equal(p2[r][1][b], crit) and torch.equal(p3[r][1][b], p3[0][1][b])
        o = dict(classes=cat(0, p1), A=cat(0, p3), B=p3[0][1][b:b + 1], pred=p3[0][2][b:b + 1], Q=cat(1, p1),
                 H1=cat(2, p1))
        assert torch.equal(p2[0][2][b], o["Q"][crit]), "q_max is not the critical rows' saved Q"
        per.append(_outs(o, crit, [bd[-1][1]], saves=("Q", "H1"))[0])
    return per


def check_forms(name, case: Case, p, outs, ref="train", vms=None):
    """Stage checks of every form that carries its own Q, and A, B, pred of every form against the fp64 restatement on
    its own Q (or, without one, on the `ref` form's Q, after asserting the same classes and crit bits)."""
    bl = bags(case)
    vms = vms or [None] * len(bl)
    worst = {}

    def note(k, v):
        worst[k] = max(worst.get(k, 0.0), v)

    for j, b in enumerate(bl):
        X = b.X
        for form, per in outs.items():
            o = per[j]
            own = "Q" in o
            src = o if own else outs[ref][j]
            crit, Q = src["crit"], src["Q"]
            if not own:
                assert np.array_equal(o["crit"], crit), (name, form, j)
                if "classes" in o:
                    assert np.array_equal(o["classes"], src["classes"]), (name, form, j)
            else:
                c64, cb = classes_bar(X, p)
                note("classes", over(np.abs(o["classes"] - c64), cb))
                cols = np.arange(case.C)
                assert np.array_equal(o["classes"][crit, cols], o["classes"].max(0)), (name, form, j)
                if not o.get("crafted"):
                    for k, (rf, bar) in stage_bars(X, p, o.get("H1"), case.tc_phase1, vms[j]).items():
                        note(k, over(np.abs(o[k] - rf), bar))
                if len(b.probes):
                    assert np.array_equal(Q[b.probes], np.broadcast_to(Q[b.crit0], (len(b.probes), KQ))), (name, j)
            V = src["V"] if case.passing_v else X
            r64 = restate(Q, crit, V, p)
            tau, Bb, Pb = a_bars(Q, crit, V, p, r64, case.attend)
            ea, tiny_ok = a_err(o["A"], r64, tau)
            assert tiny_ok, (name, form, j)
            note(f"A.{form}", ea)
            note(f"B.{form}", over(np.abs(o["B"].reshape(case.C, -1) - r64["B"]), Bb))
            note(f"pred.{form}", over(np.abs(o["pred"].reshape(-1) - r64["pred"]), Pb))
    print(f"conditioned forward {name}: " + " ".join(f"{k}={v:.3g}" for k, v in sorted(worst.items())))
    bad = {k: v for k, v in worst.items() if not v <= 1.0}
    assert not bad, (name, bad)


def _lib_load():
    from dsmil_wsi_b200 import _lib
    return _lib.load()


@pytest.mark.gpu
@pytest.mark.parametrize("case", SINGLE, ids=lambda c: c.name)
def test_single_bag_forward_on_its_own_q(case):
    """dsmil_forward (training, eval overlapped, eval plain) and dsmil_bag_forward on the training call's classes."""
    p = make_params(case)
    check_forms(case.name, case, p, run_single(case, _lib_load(), _pack(p), bags(case)[0].X))


@pytest.mark.gpu
@pytest.mark.parametrize("case", BAGS, ids=lambda c: c.name)
def test_batched_forward_on_its_own_q(case):
    """dsmil_forward_bags[_train] and the capture-safe dev pair (tensor-core or generic)."""
    p = make_params(case)
    check_forms(case.name, case, p, run_bags(case, _lib_load(), _pack(p), [b.X for b in bags(case)]))


@pytest.mark.gpu
@pytest.mark.parametrize("case", MODELS, ids=lambda c: c.name)
def test_fold_forward_on_its_own_q(case):
    ps = [make_params(case, m) for m in range(2)]
    outs = run_models(case, _lib_load(), [_pack(p) for p in ps], [b.X for b in bags(case)])
    for m, (p, o) in enumerate(zip(ps, outs)):
        check_forms(f"{case.name} model {m}", case, p, o)


@pytest.mark.gpu
@pytest.mark.parametrize("case", VALUE, ids=lambda c: c.name)
def test_value_forward_on_its_own_q_and_v(case):
    p = make_params(case)
    vms = v_masks(case)
    check_forms(case.name, case, p, run_value(case, _lib_load(), _pack(p), [b.X for b in bags(case)], vms), vms=vms)


@pytest.mark.gpu
@pytest.mark.parametrize("G", [1, 2, 3])
@pytest.mark.parametrize("case", SHARD, ids=lambda c: c.name)
def test_row_sharded_forward_on_its_own_q(case, G):
    """Per bag (CudaShardOps: at G = 3 the 2-row bag leaves a rank empty, and the linear case's probe-free rank has a
    combine weight that underflows) and, on the tensor-core shape, batched (CudaShardBagOps).  At G = 1 and 3 phase 2
    also takes a crafted Q (3x the saved one, logits 9x) straight into the per-bag attend kernel."""
    p = make_params(case)
    P = _pack(p)
    Xs = [b.X for b in bags(case)]
    outs = {"per_bag": [run_shard_per_bag(case, P, X, G) for X in Xs]}
    if G != 2:
        outs["crafted"] = [dict(run_shard_per_bag(case, P, X, G, crafted=True), crafted=True) for X in Xs]
    if case.tc_phase1 and min(case.Ns) >= G:
        outs["batched"] = run_shard_bags(case, P, Xs, G)
    check_forms(f"{case.name} G={G}", case, p, outs)


def tanh_sweep_values():
    """3072 pre-activations in [-20, 20]: a uniform grid, signed zeros, |z| < 1e-6 and both saturation knees."""
    tiny = np.array([0.0, -0.0, 1e-30, -1e-30, 1e-12, -1e-12, 1e-9, -1e-9, 1e-7, -1e-7, 5e-7, -5e-7, 9.9e-7, -9.9e-7])
    knees = np.concatenate([np.linspace(7.5, 10.5, 400), -np.linspace(7.5, 10.5, 400)])
    grid = np.linspace(-20.0, 20.0, 3072 - len(tiny) - len(knees))
    return np.concatenate([tiny, knees, grid]).astype(np.float32)


@pytest.mark.gpu
def test_tanh_ex2_bound_through_the_phase1_kernel():
    """W2 = 0: the pre-activation is b2 exactly and the saved Q is tanh_ex2(b2); |Q - tanh(b2)| <= TANH_ABS."""
    from dsmil_wsi_b200 import _lib
    lib = _lib.load()
    z = tanh_sweep_values()
    D, N = 128, 3
    X = orc.synthetic_bag(N, D, 11)
    x = _t(X)
    got = []
    for i in range(0, len(z), KQ):
        p = orc.random_params(D, 1, 12)
        p.W2[:] = 0.0
        p.b2 = z[i:i + KQ].copy()
        P = _pack(p)
        o = [_nan(N, 1), _nan(1, 1), _nan(N, 1), _nan(1, 1, D)]
        crit = torch.zeros(1, dtype=torch.int64, device="cuda")
        Q, H1 = _nan(N, KQ), _nan(N, KQ)
        ws = _ws(lib.dsmil_forward_workspace_bytes(P.ref, N))
        rc = lib.dsmil_forward(P.ref, x.data_ptr(), None, N, *[t.data_ptr() for t in o], crit.data_ptr(), Q.data_ptr(),
                               H1.data_ptr(), None, ws.data_ptr(), ws.numel(), _stream())
        assert rc == 0, lib.dsmil_last_error()
        q = _np(Q)
        assert np.all(q == q[0]), "rows with the same b2 must give the same Q"
        got.append(q[0])
    err = np.abs(np.concatenate(got).astype(np.float64) - np.tanh(z.astype(np.float64)))
    print(f"tanh_ex2: max |err| = {err.max():.3g} at z = {z[np.argmax(err)]!r}")
    assert err.max() <= TANH_ABS, (err.max(), z[np.argmax(err)])
