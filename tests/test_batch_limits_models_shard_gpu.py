"""The fold, row-sharded and value-network bag calls at the ends of the batch range they accept, held to the checks of
`test_batch_limits_gpu.py` (LB), and through it to the conditioned forward (FW) and backward (BW) files.

LB covers the one-model calls.  This file covers the calls people train folds, shards and value networks with, by LB's
method: bag b is pattern b mod P and points at that pattern's one device buffer; every occurrence of a pattern must give
the bits of its first occurrence; the first occurrences pass the conditioned forward and backward checks; upstream
gradients change sign every P bags, and a cross-bag sum is compared with sum_p w_p g_p in fp64 under LB's bag-order
and chunk bars.  A call that has a reference call on the same bags (the eager form of a capture-safe call, the one-model
call of a fold slice) must give its bits instead.

Cases (D = 512, C = 2 unless named):
  - the fused fold at nb * M = 65 535 entries: dsmil_forward_bags_models (M = 3 x 21 845), and _models_train with
    dsmil_backward_bags_models (M = 2, nbs = 32 768 and 32 767, so the models' sign windows differ), with d_A, d_B and
    gX.  Each makes as many launches as on one period of bags, fewer than the per-model calls there, so it took the
    fused route at the limit.  Each model's gradients pass the bars
    against fp64 over that model's own bags: the fold's gWf and gbf sum each model's bags in bag order, one chain per
    model.
  - the fold fallback at 65 536 and 70 000 entries: the training forms give each model's one-model bits on its slice.
  - the fold capture-safe pair at the largest total it takes, row capacity filled and 20 rows past it: the eager fold
    calls' bits.
  - the row-sharded eager batch at nb = 65 535: with G = 1 the inference and training phases and the three backward
    phases give dsmil_forward_bags[_train] / dsmil_backward_bags's bits; with G = 2 virtual ranks (every bag split
    between them, at a cut that moves with the pattern) the first occurrences pass the conditioned sharded checks and
    the gradients orc.backward_sharded at BW's bars.
  - the row-sharded capture-safe step (G = 1): forward at nb = 65 535, backward at the largest nb it takes, the eager
    sharded calls' bits; at nb = 65 535 the backward refuses the batch before any launch.
  - candidate records past 2^32 elements of Q (D = 128): k_gather_cand_b's idx, score and q row in every bag, on
    row-major and tile-blocked Q and in the capture-safe form.
  - the capture-safe value calls (D = 128, passing_v, with and without v's mask) at nb = 65 535 (forward) and at the
    largest nb the backward takes: the eager value calls' bits.

The CPU part states the new bounds: the sharded capture-safe backward refuses a chunk capacity past 65 535, as the
one-model pair does; the eager sharded backward's size is 0 past 65 535 bags; and the fold dev pair's largest total.
It also shows LB's 4x / 20x demonstration for the per-model bag-order chains of the fold.

Each large case sizes its memory from the library's workspace functions and skips, naming the bytes, when the card
lacks them.  Largest errors over bars, peak memory and run times are in DESIGN §3.
"""
from __future__ import annotations

import ctypes as C
import time

import numpy as np
import pytest
import torch

import test_conditioned_backward_gpu as BW
import test_conditioned_forward_gpu as FW
from oracle import dsmil_oracle as orc
from test_batch_limits_gpu import (LIMIT, PATTERN, PATTERN_Q, SENSITIVITY, Layout, _bag_ptrs, _check_backward,
                                   _check_period, _first_outs, _forward_batch, _need, _report, chain_bar, cycle,
                                   dev_backward_limit, fp32_chain, same_bits, signed_counts, signs, upstream)
from test_batch_limits_gpu import _release_device_memory  # noqa: F401  (autouse fixture)

KQ = FW.KQ
ERR_ARG = -1
FAKE = 0x10000                 # a non-NULL, 16-byte aligned "device pointer": never dereferenced on refused calls
MAX_ROWS = 300                 # the row capacity of the capture-safe cases' size checks: max(PATTERN)
FOLD_NBS = (32768, 32767)      # the fused fold's training batch: nb * M = 65 535, sign windows that differ per model
EVAL_M = 3                     # the fold eval call takes one bag list for all models: 3 x 21 845 = 65 535 entries
PATTERN_G2 = (2,) + PATTERN[1:]                                   # every bag split between two ranks
PATTERN_QD = tuple(513 + j for j in range(len(PATTERN_Q)))        # capture-safe records: Q past 2^32 at 523 rows a bag
FOLD_CASE = FW.Case("limit_models_d512_c2", "models", 512, 2, PATTERN)
SHARD_CASE = FW.Case("limit_shard_d512_c2", "shard", 512, 2, PATTERN)
SHARD2_CASE = FW.Case("limit_shard_g2_d512_c2", "shard", 512, 2, PATTERN_G2)
CAND_CASE = FW.Case("limit_cand_d128_c2", "bags", 128, 2, PATTERN_Q)
CAND_DEV_CASE = FW.Case("limit_cand_dev_d128_c2", "bags", 128, 2, PATTERN_QD)
VALUE_DEV_CASES = [FW.Case("limit_value_dev_d128_c2", "value", 128, 2, PATTERN, passing_v=True),
                   FW.Case("limit_value_dev_d128_c2_mask", "value", 128, 2, PATTERN, passing_v=True, masked=True)]


def _params_struct(D, C_, passing_v=0):
    from test_shard_bags_train_cpu import params
    p = params(D, C_, passing_v)
    return p, type("P", (), {"ref": C.byref(p)})


# ---- the fold capture-safe pair's capacities, restated from models_dev_caps --------------------------------------
K_SPLITS, TBM = 296, 128


def rag_chunks_cap(M1, M2, gemv, nb):
    s = K_SPLITS if gemv else max(1, K_SPLITS // (-(-M1 // TBM) * -(-M2 // TBM)))
    return s + nb


def models_dev_caps(C_, D, nbs):
    """(entries, chunk capacity of gWi, of gW1) over all models, as models_dev_caps sums them."""
    gemv = C_ <= 4 and D % 4 == 0 and D // 4 <= 256
    return (sum(nbs), sum(rag_chunks_cap(C_, D, gemv, n) for n in nbs), sum(rag_chunks_cap(KQ, D, False, n) for n in nbs))


def split(total, M):
    return [total // M + (1 if m < total % M else 0) for m in range(M)]


def fold_dev_limit(lib, ps, M, max_rows):
    """The largest total of bags, split evenly over M models, that the fold dev backward takes."""
    f = lambda t: lib.dsmil_backward_bags_models_dev_workspace_bytes(ps, M, (C.c_int32 * M)(*split(t, M)), max_rows)
    lo, hi = M, LIMIT
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if f(mid) > 0 else (lo, mid - 1)
    return lo


# ===================================================================================== CPU part: no device needed
@pytest.mark.parametrize("D,C_", [(512, 2), (1024, 4)])
def test_sharded_capture_safe_backward_refuses_a_chunk_grid_past_65535(D, C_):
    """dsmil_shard_backward_bags_phase1/2/3_dev run backward_bags_dev's ragged GEMMs on the same capacities: they take
    the batches dsmil_backward_bags_dev takes, and refuse nb = 65 535 (DSMIL_ERR_ARG, "chunk capacity")."""
    from dsmil_wsi_b200 import _lib
    lib = _lib.load()
    p, P = _params_struct(D, C_)
    nb = dev_backward_limit(lib, P, "dsmil_shard_", MAX_ROWS)
    assert nb == dev_backward_limit(lib, P, "dsmil_", MAX_ROWS) == 65239, nb
    f = lib.dsmil_shard_backward_bags_dev_workspace_bytes
    assert f(P.ref, nb, MAX_ROWS) > 0 and f(P.ref, nb + 1, MAX_ROWS) == 0 and f(P.ref, LIMIT, MAX_ROWS) == 0
    phases = {
        "phase1": lambda: lib.dsmil_shard_backward_bags_phase1_dev(P.ref, FAKE, FAKE, LIMIT, MAX_ROWS, *[FAKE] * 10,
                                                                   FAKE, None, 0, None),
        "phase2": lambda: lib.dsmil_shard_backward_bags_phase2_dev(P.ref, LIMIT, MAX_ROWS, *[FAKE] * 5, None, 0, None),
        "phase3": lambda: lib.dsmil_shard_backward_bags_phase3_dev(P.ref, LIMIT, MAX_ROWS, *[FAKE] * 11, None, 0, None),
    }
    # the workspace given is the size the library returned (0): the refusal names the chunk capacity, not the
    # workspace, and comes before anything is launched
    for name, call in phases.items():
        assert call() == ERR_ARG and b"chunk capacity" in lib.dsmil_last_error(), (name, lib.dsmil_last_error())


def test_eager_sharded_backward_size_is_0_past_65535_bags():
    from dsmil_wsi_b200 import _lib
    lib = _lib.load()
    p, P = _params_struct(512, 2)
    for nb, want in ((LIMIT, True), (LIMIT + 1, False), (70000, False)):
        Ns = (C.c_int64 * nb)(*[10] * nb)
        assert (lib.dsmil_shard_backward_bags_workspace_bytes(P.ref, Ns, nb) > 0) == want, nb


@pytest.mark.parametrize("M", [2, 3])
def test_fold_capture_safe_pair_takes_up_to_its_chunk_capacity(M):
    """The largest total the fold dev pair takes: there the entries and chunk sums of models_dev_caps are within
    65 535, one bag past it both sizes are 0."""
    from dsmil_wsi_b200 import _lib
    from test_models_train_graph_cpu import arr, params
    lib = _lib.load()
    ps = arr([params(512, 2)] * M)
    T = fold_dev_limit(lib, ps, M, MAX_ROWS)
    ne, nci, nc1 = models_dev_caps(2, 512, split(T, M))
    assert ne == T and max(ne, nci, nc1) == 65535, (T, nci, nc1)
    assert T == 65535 - M * K_SPLITS
    for t, ok in ((T, True), (T + 1, False)):
        c_nb = (C.c_int32 * M)(*split(t, M))
        for f in (lib.dsmil_forward_bags_models_train_dev_workspace_bytes,
                  lib.dsmil_backward_bags_models_dev_workspace_bytes):
            assert (f(ps, M, c_nb, MAX_ROWS) > 0) == ok, (M, t, f)


def test_per_model_bag_order_sums_stay_4x_under_their_bars_and_the_last_bag_moves_them_past_20x():
    """The fold's gWf and gbf add each model's own bags in bag order, so each model's chain has its own sign windows
    and length (FOLD_NBS): LB's demonstration holds for each."""
    from test_batch_limits_gpu import cpu_bag_sums
    dp, B = cpu_bag_sums(FOLD_CASE)
    for nb in FOLD_NBS:
        w = signed_counts(nb)
        sums = {"bf": (dp, None, w @ dp, chain_bar(dp, nb)),
                "Wf": (dp[:, :, None], B[:, None, :], np.einsum("p,pk,pi->ki", w, dp, B),
                       chain_bar(dp[:, :, None] * B[:, None, :], nb))}
        for name, (terms, fw, want, bar) in sums.items():
            err = FW.over(np.abs(fp32_chain(terms, nb, fma_with=fw) - want), bar)
            assert err <= 0.25, (nb, name, err)
            for wl in (0.0, 2.0):
                moved = FW.over(np.abs(fp32_chain(terms, nb, fma_with=fw, weight_last=wl) - want), bar)
                assert moved > SENSITIVITY, (nb, name, wl, moved)
            print(f"model of {nb} bags g{name}: fp32 chain {err:.3g} of its bar")


def test_fold_and_sharded_batches_sit_where_they_should():
    assert sum(FOLD_NBS) == LIMIT and LIMIT % EVAL_M == 0
    assert signed_counts(FOLD_NBS[0]).tolist() != signed_counts(FOLD_NBS[1]).tolist()
    assert min(PATTERN_G2) == 2 and len(PATTERN_G2) == len(PATTERN)
    assert sum(cycle(PATTERN_QD, LIMIT)) * KQ > 1 << 32
    assert len(set(np.asarray(signs(LIMIT)).tolist())) == 2


# ========================================================================================== GPU part (one H100)
def _lib_load():
    return FW._lib_load()


def _signed(ups, lay, i):
    """Upstream i of every row (i = 0, 2) or bag (i = 1, 3) of a cycled batch, with the window signs."""
    if i in (0, 2):
        return torch.from_numpy(np.concatenate([u[i] for u in ups])).cuda()[lay.row_src] * lay.row_sign[:, None]
    t = torch.from_numpy(np.stack([u[i] for u in ups])).cuda()[lay.bag_src]
    return t * lay.bag_sign.reshape((-1,) + (1,) * (t.dim() - 1))


def _same(name, a, b):
    assert a.shape == b.shape and torch.equal(a.reshape(-1).view(torch.int32) if a.dtype == torch.float32 else a,
                                              b.reshape(-1).view(torch.int32) if b.dtype == torch.float32 else b), name


def _same_outs(name, o, crit, ref, ref_crit):
    for k, t in ref.items():
        if t is not None and o.get(k) is not None:
            _same(f"{name} {k}", o[k][:t.shape[0]], t)
    _same(f"{name} crit", crit, ref_crit)


def _fold_ptrs(xs, lays):
    """Host bag list of the fold's entries, model-major: each model's bags restart the cycle."""
    Ns = [n for lay in lays for n in lay.Ns]
    ptrs = [xs[b % len(xs)].data_ptr() for lay in lays for b in range(lay.nb)]
    return (C.c_void_p * len(Ns))(*ptrs), (C.c_int64 * len(Ns))(*Ns)


def _models(lib, ps):
    from dsmil_wsi_b200 import _lib
    return (_lib.DsmilParams * len(ps))(*[P.struct for P in ps])


class _HostGrads:
    def __init__(self, t):
        self.t, self.gX = t, None

    def host(self):
        return {k: FW._np(v) for k, v in self.t.items()}


def _launches(fn):
    """The library's launch count of fn() (DSMIL_LAUNCH_OK counts every kernel launch)."""
    from dsmil_wsi_b200 import _lib
    torch.cuda.synchronize()
    before = _lib.launch_count()
    fn()
    torch.cuda.synchronize()
    return _lib.launch_count() - before


def _small_route_counts(lib, packs, xs, case):
    """Launches of the three fold calls on one period of bags per model (the fused route, one launch per stage), and
    of the per-model calls the fallback would make on the same bags: {form: (fused, per model)}."""
    from dsmil_wsi_b200 import _lib
    P_, M = len(xs), len(FOLD_NBS)
    Ns = list(case.Ns)
    total = sum(Ns)
    c_X, c_N = _bag_ptrs(xs, Ns)
    c_Xf, c_Nf = _bag_ptrs(xs * M, Ns * M)
    c_nb = (C.c_int32 * M)(*[P_] * M)
    rc = []
    call = lambda f, *a: rc.append(f(*a))
    counts = {}
    # eval: EVAL_M models over the same bags, against EVAL_M x dsmil_forward_bags
    o, crit = FW._new_outs(EVAL_M * total, EVAL_M * P_, case)
    out = lambda o, crit: [FW._ptr(o[k]) for k in ("classes", "pred", "A", "B")] + [crit.data_ptr()]
    ws = FW._ws(lib.dsmil_forward_bags_models_workspace_bytes(_models(lib, packs), EVAL_M, c_N, P_))
    fused = _launches(lambda: call(lib.dsmil_forward_bags_models, _models(lib, packs), EVAL_M, c_X, c_N, P_,
                                   *out(o, crit), ws.data_ptr(), ws.numel(), FW._stream()))
    o1, crit1 = FW._new_outs(total, P_, case)
    ws1 = FW._ws(lib.dsmil_forward_bags_workspace_bytes(packs[0].ref, c_N, P_))
    per = _launches(lambda: [call(lib.dsmil_forward_bags, P.ref, c_X, c_N, P_, *out(o1, crit1), ws1.data_ptr(),
                                  ws1.numel(), FW._stream()) for P in packs])
    counts["eval"] = (fused, per)
    # training forward and backward: M models over their own bags
    c_ps = _models(lib, packs[:M])
    o, crit = FW._new_outs(M * total, M * P_, case, saves=True)
    saves = lambda o: [FW._ptr(o["Q"]), FW._ptr(o["H1"])]
    ws = FW._ws(lib.dsmil_forward_bags_models_train_workspace_bytes(c_ps, M, c_Nf, c_nb))
    fused = _launches(lambda: call(lib.dsmil_forward_bags_models_train, c_ps, M, c_Xf, c_Nf, c_nb, *out(o, crit),
                                   *saves(o), ws.data_ptr(), ws.numel(), FW._stream()))
    o1, crit1 = FW._new_outs(total, P_, case, saves=True)
    ws1 = FW._ws(lib.dsmil_forward_bags_train_workspace_bytes(packs[0].ref, c_N, P_))
    per = _launches(lambda: [call(lib.dsmil_forward_bags_train, P.ref, c_X, c_N, P_, *out(o1, crit1), *saves(o1),
                                  ws1.data_ptr(), ws1.numel(), FW._stream()) for P in packs[:M]])
    counts["train"] = (fused, per)
    ups = upstream(case)
    up = lambda i, reps: torch.from_numpy(np.concatenate([u[i] for u in ups] * reps) if i in (0, 2) else
                                          np.stack([u[i] for u in ups] * reps)).cuda()
    bcase = BW.Case(case.name, "models", case.D, case.C, (tuple(case.Ns),) * M)
    gs = [BW._Grads(bcase, total) for _ in range(M)]
    grads = (_lib.DsmilGrads * M)(*[g.struct() for g in gs])
    dc, dp, dA, dB = (up(i, M) for i in range(4))
    ins = lambda o, crit, dc, dp, dA, dB: ([FW._ptr(o[k]) for k in ("Q", "H1", "A", "B")] +
                                           [crit.data_ptr(), dc.data_ptr(), dp.data_ptr(), dA.data_ptr(), dB.data_ptr()])
    ws = FW._ws(lib.dsmil_backward_bags_models_workspace_bytes(c_ps, M, c_Nf, c_nb, 1))
    fused = _launches(lambda: call(lib.dsmil_backward_bags_models, c_ps, M, c_Xf, c_Nf, c_nb,
                                   *ins(o, crit, dc, dp, dA, dB), grads, ws.data_ptr(), ws.numel(), FW._stream()))
    G1 = gs[0].struct()
    dc1, dp1, dA1, dB1 = (up(i, 1) for i in range(4))
    ws1 = FW._ws(lib.dsmil_backward_bags_workspace_bytes(packs[0].ref, c_N, P_, 1))
    per = _launches(lambda: [call(lib.dsmil_backward_bags, P.ref, c_X, c_N, P_, *ins(o1, crit1, dc1, dp1, dA1, dB1),
                                  C.byref(G1), ws1.data_ptr(), ws1.numel(), FW._stream()) for P in packs[:M]])
    counts["backward"] = (fused, per)
    assert rc == [0] * len(rc), lib.dsmil_last_error()
    return counts


@pytest.mark.gpu
def test_fused_fold_at_65535_entries():
    """dsmil_forward_bags_models over 3 x 21 845 entries, then dsmil_forward_bags_models_train and
    dsmil_backward_bags_models (d_A, d_B, gX) over nbs = (32 768, 32 767): each takes the fused route (as many launches
    as on one period of bags, fewer than the per-model calls), every occurrence gives its first occurrence's bits, and
    the first occurrences and each model's sums pass the conditioned bars over that model's own bags."""
    case = FOLD_CASE
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    lib = _lib_load()
    ps_h = [FW.make_params(case, m) for m in range(EVAL_M)]
    packs = [FW._pack(p) for p in ps_h]
    pats = FW.bags(case)
    xs = [FW._t(b.X) for b in pats]
    M, nbs = len(FOLD_NBS), list(FOLD_NBS)
    lays = [Layout(case.Ns, n) for n in nbs]
    Ns = [n for lay in lays for n in lay.Ns]
    rows = sum(Ns)
    c_ps = _models(lib, packs[:M])
    c_X, c_N = _fold_ptrs(xs, lays)
    c_nb = (C.c_int32 * M)(*nbs)
    fws = lib.dsmil_forward_bags_models_train_workspace_bytes(c_ps, M, c_N, c_nb)
    bws = lib.dsmil_backward_bags_models_workspace_bytes(c_ps, M, c_N, c_nb, 1)
    assert fws > 0 and bws > 0
    _need(rows * 4 * (2 * KQ + 10 * case.C + 2 * case.D) + max(fws, bws) + rows * 96, case.name)
    small = _small_route_counts(lib, packs, xs, case)
    assert all(fused < per for fused, per in small.values()), small
    counts = {}

    # eval: 3 models over the same 21 845 bags
    ne = LIMIT // EVAL_M
    lay_e = Layout(case.Ns, ne)
    c_Xe, c_Ne = _bag_ptrs(xs, lay_e.Ns)
    oe, crite = FW._new_outs(EVAL_M * lay_e.total, LIMIT, case)
    ws = FW._ws(lib.dsmil_forward_bags_models_workspace_bytes(_models(lib, packs), EVAL_M, c_Ne, ne))
    rc = []
    counts["eval"] = _launches(lambda: rc.append(lib.dsmil_forward_bags_models(
        _models(lib, packs), EVAL_M, c_Xe, c_Ne, ne, *[FW._ptr(oe[k]) for k in ("classes", "pred", "A", "B")],
        crite.data_ptr(), ws.data_ptr(), ws.numel(), FW._stream())))
    assert rc == [0], lib.dsmil_last_error()
    del ws
    eval_first = []
    for m in range(EVAL_M):
        r0, b0 = m * lay_e.total, m * ne
        om = {k: oe[k][r0:r0 + lay_e.total] if k in ("classes", "A") else oe[k][b0:b0 + ne] for k in oe}
        _check_period(f"{case.name} eval model {m}", om, crite[b0:b0 + ne], lay_e)
        eval_first.append(_first_outs(om, crite[b0:b0 + ne], lay_e, case.Ns))
    del oe, crite

    # training forward and backward over each model's own bags
    o, crit = FW._new_outs(rows, LIMIT, case, saves=True)
    ws = FW._ws(fws)
    counts["train"] = _launches(lambda: rc.append(lib.dsmil_forward_bags_models_train(
        c_ps, M, c_X, c_N, c_nb, *[FW._ptr(o[k]) for k in ("classes", "pred", "A", "B")], crit.data_ptr(),
        FW._ptr(o["Q"]), FW._ptr(o["H1"]), ws.data_ptr(), ws.numel(), FW._stream())))
    assert rc == [0, 0], lib.dsmil_last_error()
    del ws
    r0 = [0, lays[0].total]
    sl = lambda m: ({k: v[r0[m]:r0[m] + lays[m].total] if k in ("classes", "A", "Q", "H1") else
                     v[m * nbs[0]:m * nbs[0] + nbs[m]] for k, v in o.items() if v is not None},
                    crit[m * nbs[0]:m * nbs[0] + nbs[m]])
    for m in range(M):
        om, cm = sl(m)
        _check_period(f"{case.name} train model {m}", om, cm, lays[m])
        FW.check_forms(f"{case.name} model {m}", case, ps_h[m], {"train": _first_outs(om, cm, lays[m], case.Ns),
                                                                  "eval": eval_first[m]})
    ups = upstream(case)
    dc = torch.cat([_signed(ups, lay, 0) for lay in lays])
    dA = torch.cat([_signed(ups, lay, 2) for lay in lays])
    dp = torch.cat([_signed(ups, lay, 1) for lay in lays])
    dB = torch.cat([_signed(ups, lay, 3) for lay in lays])
    bcase = BW.Case(case.name, "models", case.D, case.C, (tuple(case.Ns),) * M)
    gs = [BW._Grads(bcase, lays[m].total) for m in range(M)]
    from dsmil_wsi_b200 import _lib
    grads = (_lib.DsmilGrads * M)(*[g.struct() for g in gs])
    ws = FW._ws(bws)
    counts["backward"] = _launches(lambda: rc.append(lib.dsmil_backward_bags_models(
        c_ps, M, c_X, c_N, c_nb, FW._ptr(o["Q"]), FW._ptr(o["H1"]), FW._ptr(o["A"]), FW._ptr(o["B"]), crit.data_ptr(),
        dc.data_ptr(), dp.data_ptr(), dA.data_ptr(), dB.data_ptr(), grads, ws.data_ptr(), ws.numel(), FW._stream())))
    assert rc == [0, 0, 0], lib.dsmil_last_error()
    del ws, dc, dA, dp, dB
    print(f"{case.name} launches at the limit: {counts}; on one period (fused, per model): {small}")
    assert counts == {form: fused for form, (fused, _) in small.items()}, (counts, small)
    for m in range(M):
        om, cm = sl(m)
        same_bits(f"{case.name} model {m} gX", gs[m].gX, lays[m].row_src, sign=lays[m].row_sign)
        _check_backward(case, bcase, ps_h[m], pats, _first_outs(om, cm, lays[m], case.Ns), ups, gs[m], lays[m], t0,
                        nb=nbs[m])


@pytest.mark.gpu
@pytest.mark.parametrize("ne", [LIMIT + 1, 70000])
def test_fold_fallback_past_65535_entries_gives_each_models_bits(ne):
    """dsmil_forward_bags_models_train and dsmil_backward_bags_models (d_A, d_B) over two models of ne / 2 bags: each
    model's outputs and gradients are the bits of dsmil_forward_bags_train / dsmil_backward_bags on its slice."""
    case = FOLD_CASE
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    lib = _lib_load()
    M = 2
    nbs = split(ne, M)
    ps_h = [FW.make_params(case, m) for m in range(M)]
    packs = [FW._pack(p) for p in ps_h]
    xs = [FW._t(b.X) for b in FW.bags(case)]
    lays = [Layout(case.Ns, n) for n in nbs]
    Ns = [n for lay in lays for n in lay.Ns]
    rows = sum(Ns)
    c_ps = _models(lib, packs)
    c_X, c_N = _fold_ptrs(xs, lays)
    c_nb = (C.c_int32 * M)(*nbs)
    fws = lib.dsmil_forward_bags_models_train_workspace_bytes(c_ps, M, c_N, c_nb)
    bws = lib.dsmil_backward_bags_models_workspace_bytes(c_ps, M, c_N, c_nb, 0)
    assert fws > 0 and bws > 0
    _need(rows * 4 * (3 * KQ + 10 * case.C) + max(fws, bws) + rows * 64, f"fold fallback ne={ne}")
    o, crit = FW._new_outs(rows, ne, case, saves=True)
    ws = FW._ws(fws)
    rc = lib.dsmil_forward_bags_models_train(c_ps, M, c_X, c_N, c_nb, *[FW._ptr(o[k]) for k in ("classes", "pred", "A",
                                                                                                "B")],
                                             crit.data_ptr(), FW._ptr(o["Q"]), FW._ptr(o["H1"]), ws.data_ptr(),
                                             ws.numel(), FW._stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.dsmil_last_error()
    del ws
    ups = upstream(case)
    dc = torch.cat([_signed(ups, lay, 0) for lay in lays])
    dA = torch.cat([_signed(ups, lay, 2) for lay in lays])
    dp = torch.cat([_signed(ups, lay, 1) for lay in lays])
    dB = torch.cat([_signed(ups, lay, 3) for lay in lays])
    bcase = BW.Case(case.name, "models", case.D, case.C, (tuple(case.Ns),) * M)
    gs = [BW._Grads(bcase) for _ in range(M)]
    from dsmil_wsi_b200 import _lib
    grads = (_lib.DsmilGrads * M)(*[g.struct() for g in gs])
    ws = FW._ws(bws)
    rc = lib.dsmil_backward_bags_models(c_ps, M, c_X, c_N, c_nb, FW._ptr(o["Q"]), FW._ptr(o["H1"]), FW._ptr(o["A"]),
                                        FW._ptr(o["B"]), crit.data_ptr(), dc.data_ptr(), dp.data_ptr(), dA.data_ptr(),
                                        dB.data_ptr(), grads, ws.data_ptr(), ws.numel(), FW._stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.dsmil_last_error()
    del ws
    r0, b0 = 0, 0
    for m, lay in enumerate(lays):
        name = f"fold fallback ne={ne} model {m}"
        P = packs[m]
        ref, ref_crit = _forward_batch(lib, P, xs, lay, case, True)
        rs, bs = slice(r0, r0 + lay.total), slice(b0, b0 + lay.nb)
        _same_outs(name, {k: (v[rs] if k in ("classes", "A", "Q", "H1") else v[bs]) for k, v in o.items()
                          if v is not None}, crit[bs], ref, ref_crit)
        del ref, ref_crit
        g = BW._Grads(bcase)
        G = g.struct()
        c_Xm, c_Nm = _bag_ptrs(xs, lay.Ns)
        ws = FW._ws(lib.dsmil_backward_bags_workspace_bytes(P.ref, c_Nm, lay.nb, 0))
        rc = lib.dsmil_backward_bags(P.ref, c_Xm, c_Nm, lay.nb, FW._ptr(o["Q"][rs]), FW._ptr(o["H1"][rs]),
                                     FW._ptr(o["A"][rs]), FW._ptr(o["B"][bs]), crit[bs].data_ptr(), dc[rs].data_ptr(),
                                     dp[bs].data_ptr(), dA[rs].data_ptr(), dB[bs].data_ptr(), C.byref(G), ws.data_ptr(),
                                     ws.numel(), FW._stream())
        torch.cuda.synchronize()
        assert rc == 0, lib.dsmil_last_error()
        del ws
        for k, t in g.t.items():
            assert not torch.isnan(t).any(), (name, k)
            _same(f"{name} g{k}", gs[m].t[k], t)
        r0, b0 = r0 + lay.total, b0 + lay.nb
    _report(f"fold fallback ne={ne}", t0)


@pytest.mark.gpu
@pytest.mark.parametrize("extra", [0, 20], ids=["full", "short"])
def test_fold_capture_safe_pair_at_its_largest_total_gives_the_eager_bits(extra):
    """dsmil_forward_bags_models_train_dev and dsmil_backward_bags_models_dev at the largest total they take (two
    models), row capacity max(PATTERN) + extra: every output and gradient is the eager fold calls' bits."""
    case = FOLD_CASE
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    lib = _lib_load()
    M = 2
    packs = [FW._pack(FW.make_params(case, m)) for m in range(M)]
    c_ps = _models(lib, packs)
    max_rows = max(case.Ns) + extra
    T = fold_dev_limit(lib, c_ps, M, max_rows)
    assert T == LIMIT - M * K_SPLITS
    nbs = split(T, M)
    c_nb = (C.c_int32 * M)(*nbs)
    xs = [FW._t(b.X) for b in FW.bags(case)]
    lays = [Layout(case.Ns, n) for n in nbs]
    Ns = [n for lay in lays for n in lay.Ns]
    rows, cap = sum(Ns), T * max_rows
    c_X, c_N = _fold_ptrs(xs, lays)
    sizes = [lib.dsmil_forward_bags_models_train_workspace_bytes(c_ps, M, c_N, c_nb),
             lib.dsmil_backward_bags_models_workspace_bytes(c_ps, M, c_N, c_nb, 0),
             lib.dsmil_forward_bags_models_train_dev_workspace_bytes(c_ps, M, c_nb, max_rows),
             lib.dsmil_backward_bags_models_dev_workspace_bytes(c_ps, M, c_nb, max_rows)]
    assert min(sizes) > 0
    _need((rows + cap) * 4 * (2 * KQ + 4 * case.C) + max(sizes) + rows * 64, f"fold dev max_rows={max_rows}")
    # eager
    o, crit = FW._new_outs(rows, T, case, saves=True)
    outs = [FW._ptr(o[k]) for k in ("classes", "pred", "A", "B")] + [crit.data_ptr(), FW._ptr(o["Q"]), FW._ptr(o["H1"])]
    ws = FW._ws(sizes[0])
    rc = lib.dsmil_forward_bags_models_train(c_ps, M, c_X, c_N, c_nb, *outs, ws.data_ptr(), ws.numel(), FW._stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.dsmil_last_error()
    del ws
    # capture-safe: each model's capacity block of nbs[m] * max_rows rows, its live rows packed from the block's start
    xd = torch.tensor([xs[b % len(xs)].data_ptr() for lay in lays for b in range(lay.nb)], dtype=torch.int64,
                      device="cuda")
    Nd = torch.tensor(Ns, dtype=torch.int64, device="cuda")
    status = torch.zeros(M, dtype=torch.int32, device="cuda")
    od, critd = FW._new_outs(cap, T, case, saves=True)
    ws = FW._ws(sizes[2])
    rc = lib.dsmil_forward_bags_models_train_dev(c_ps, M, xd.data_ptr(), Nd.data_ptr(), c_nb, max_rows,
                                                 *[FW._ptr(od[k]) for k in ("classes", "pred", "A", "B")],
                                                 critd.data_ptr(), FW._ptr(od["Q"]), FW._ptr(od["H1"]),
                                                 status.data_ptr(), ws.data_ptr(), ws.numel(), FW._stream())
    torch.cuda.synchronize()
    assert rc == 0 and FW._np(status).tolist() == [0] * M, lib.dsmil_last_error()
    del ws
    blk = [0, nbs[0] * max_rows]
    er = [0, lays[0].total]
    for m, lay in enumerate(lays):
        for k in ("classes", "A", "Q", "H1"):
            _same(f"fold dev model {m} {k}", od[k][blk[m]:blk[m] + lay.total], o[k][er[m]:er[m] + lay.total])
    for k in ("pred", "B"):
        _same(f"fold dev {k}", od[k], o[k])
    _same("fold dev crit", critd, crit)
    # backward through classes and pred
    ups = upstream(case)
    dc = torch.cat([_signed(ups, lay, 0) for lay in lays])
    dp = torch.cat([_signed(ups, lay, 1) for lay in lays])
    bcase = BW.Case(case.name, "models", case.D, case.C, (tuple(case.Ns),) * M)
    from dsmil_wsi_b200 import _lib
    g_e, g_d = [BW._Grads(bcase) for _ in range(M)], [BW._Grads(bcase) for _ in range(M)]
    grads = (_lib.DsmilGrads * M)(*[g.struct() for g in g_e])
    ws = FW._ws(sizes[1])
    rc = lib.dsmil_backward_bags_models(c_ps, M, c_X, c_N, c_nb, *[FW._ptr(o[k]) for k in ("Q", "H1", "A", "B")],
                                        crit.data_ptr(), dc.data_ptr(), dp.data_ptr(), None, None, grads, ws.data_ptr(),
                                        ws.numel(), FW._stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.dsmil_last_error()
    del ws, o, crit
    dcd = torch.full((cap, case.C), 1.0e4, device="cuda")
    for m, lay in enumerate(lays):
        dcd[blk[m]:blk[m] + lay.total] = dc[er[m]:er[m] + lay.total]
    del dc
    gradsd = (_lib.DsmilGrads * M)(*[g.struct() for g in g_d])
    ws = FW._ws(sizes[3])
    rc = lib.dsmil_backward_bags_models_dev(c_ps, M, xd.data_ptr(), Nd.data_ptr(), c_nb, max_rows,
                                            *[FW._ptr(od[k]) for k in ("Q", "H1", "A", "B")], critd.data_ptr(),
                                            dcd.data_ptr(), dp.data_ptr(), None, None, gradsd, status.data_ptr(),
                                            ws.data_ptr(), ws.numel(), FW._stream())
    torch.cuda.synchronize()
    assert rc == 0 and FW._np(status).tolist() == [0] * M, lib.dsmil_last_error()
    for m in range(M):
        for k, t in g_e[m].t.items():
            assert not torch.isnan(t).any(), (m, k)
            _same(f"fold dev model {m} g{k}", g_d[m].t[k], t)
    _report(f"fold dev T={T} max_rows={max_rows}", t0)


# ---- row-sharded ------------------------------------------------------------------------------------------------
class _Keep:
    """A logical rank that keeps its saves (Q, H1, q_max) and its local row counts."""

    def __init__(self, inner):
        self.inner = inner

    def begin(self, X_locals, row_offsets):
        self.Ns = [int(x.shape[0]) for x in X_locals]
        return self.inner.begin(X_locals, row_offsets)

    def phase1_train(self):
        r = self.inner.phase1_train()
        self.Q, self.H1 = r[1], r[2]
        return r

    def phase2_train(self, Q, cands_all, G):
        r = self.inner.phase2_train(Q, cands_all, G)
        self.qmax = r[2]
        return r

    def __getattr__(self, k):
        return getattr(self.inner, k)


def _step(P, xs, nb, G, ups, lay, make=None):
    """virtual_sharded_train_step_bags over the cycled batch with the signed upstream."""
    from dsmil_wsi_b200.sharded import CudaShardBagOps, virtual_sharded_train_step_bags
    ranks = []

    def make_rank():
        ranks.append(_Keep(CudaShardBagOps(P.tensors) if make is None else make()))
        return ranks[-1]

    Xs = [xs[b % len(xs)] for b in range(nb)]
    loss = lambda c, pr, cr: (_signed(ups, lay, 0), _signed(ups, lay, 1))
    out, grads = virtual_sharded_train_step_bags(make_rank, Xs, G, loss)
    torch.cuda.synchronize()
    return out, grads, ranks


SHARD_NAMES = ("Wi", "bi", "W1", "b1", "W2", "b2", "Wf", "bf")


@pytest.mark.gpu
def test_row_sharded_batch_of_65535_bags_on_one_rank_gives_the_batched_bits():
    """G = 1: dsmil_shard_bags_phase1/2/3 give dsmil_forward_bags's bits; _phase1_train, _phase2_train, phase3 and the
    three backward phases give dsmil_forward_bags_train's outputs and saves and dsmil_backward_bags's gradients."""
    case = SHARD_CASE
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    lib = _lib_load()
    p = FW.make_params(case)
    P = FW._pack(p)
    xs = [FW._t(b.X) for b in FW.bags(case)]
    lay = Layout(case.Ns, LIMIT)
    c_X, c_N = _bag_ptrs(xs, lay.Ns)
    sizes = [lib.dsmil_shard_bags_workspace_bytes(P.ref, c_N, LIMIT),
             lib.dsmil_shard_backward_bags_workspace_bytes(P.ref, c_N, LIMIT),
             lib.dsmil_forward_bags_train_workspace_bytes(P.ref, c_N, LIMIT),
             lib.dsmil_backward_bags_workspace_bytes(P.ref, c_N, LIMIT, 0)]
    assert min(sizes) > 0
    _need(2 * lay.total * 4 * (2 * KQ + 6 * case.C) + 2 * max(sizes) + lay.total * 64, case.name)
    # inference phases against dsmil_forward_bags
    ref, ref_crit = _forward_batch(lib, P, xs, lay, case, False)
    c_off = (C.c_int64 * LIMIT)(*[0] * LIMIT)
    cand_f, rec_f = int(lib.dsmil_cand_floats(case.C)), int(lib.dsmil_rec_floats(case.C, case.D))
    o, crit = FW._new_outs(lay.total, LIMIT, case)
    cand, recs = FW._nan(LIMIT, cand_f), FW._nan(LIMIT, rec_f)
    ws = FW._ws(sizes[0])
    st = FW._stream()
    rcs = [lib.dsmil_shard_bags_phase1(P.ref, c_X, c_N, LIMIT, c_off, o["classes"].data_ptr(), cand.data_ptr(),
                                       ws.data_ptr(), ws.numel(), st),
           lib.dsmil_shard_bags_phase2(P.ref, c_X, c_N, LIMIT, cand.data_ptr(), 1, o["A"].data_ptr(), crit.data_ptr(),
                                       recs.data_ptr(), ws.data_ptr(), ws.numel(), st),
           lib.dsmil_shard_bags_phase3(P.ref, c_X, c_N, LIMIT, recs.data_ptr(), 1, o["A"].data_ptr(), o["B"].data_ptr(),
                                       o["pred"].data_ptr(), ws.data_ptr(), ws.numel(), st)]
    torch.cuda.synchronize()
    assert rcs == [0, 0, 0], lib.dsmil_last_error()
    _same_outs(f"{case.name} eval", o, crit, ref, ref_crit)
    del ws, o, crit, ref, ref_crit, cand, recs
    # the training step against dsmil_forward_bags_train and dsmil_backward_bags (d_classes and d_pred only)
    ups = upstream(case)
    (classes, pred, A, B, crit), grads, (rank,) = _step(P, xs, LIMIT, 1, ups, lay)
    ref, ref_crit = _forward_batch(lib, P, xs, lay, case, True)
    _same_outs(f"{case.name} train", dict(classes=classes, pred=pred, A=A, B=B, Q=rank.Q, H1=rank.H1), crit, ref,
               ref_crit)
    n = torch.tensor(lay.Ns, device="cuda")
    _same(f"{case.name} q_max", rank.qmax, ref["Q"][(torch.cumsum(n, 0) - n)[:, None] + ref_crit])
    bcase = BW.Case(case.name, "bags", case.D, case.C, tuple(case.Ns))
    g = BW._Grads(bcase)
    G = g.struct()
    dc, dp = _signed(ups, lay, 0), _signed(ups, lay, 1)
    ws = FW._ws(sizes[3])
    rc = lib.dsmil_backward_bags(P.ref, c_X, c_N, LIMIT, *[FW._ptr(ref[k]) for k in ("Q", "H1", "A", "B")],
                                 ref_crit.data_ptr(), dc.data_ptr(), dp.data_ptr(), None, None, C.byref(G),
                                 ws.data_ptr(), ws.numel(), FW._stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.dsmil_last_error()
    for k, t in zip(SHARD_NAMES, grads):
        assert not torch.isnan(g.t[k]).any(), k
        _same(f"{case.name} g{k}", t, g.t[k])
    _report(case.name, t0)


@pytest.mark.gpu
def test_row_sharded_batch_of_65535_bags_over_two_ranks():
    """G = 2 virtual ranks, every bag split between them: the first occurrences pass the conditioned sharded forward
    checks (crit, q_max = the critical rows' saved Q, A, B, pred), every occurrence gives its first occurrence's bits,
    and the gradients pass orc.backward_sharded at BW's bars under the bag-order and chunk bars."""
    case = SHARD2_CASE
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    lib = _lib_load()
    p = FW.make_params(case)
    P = FW._pack(p)
    pats = FW.bags(case)
    xs = [FW._t(b.X) for b in pats]
    lay = Layout(case.Ns, LIMIT)
    c_X, c_N = _bag_ptrs(xs, lay.Ns)
    ws = lib.dsmil_shard_bags_workspace_bytes(P.ref, c_N, LIMIT) + lib.dsmil_shard_backward_bags_workspace_bytes(
        P.ref, c_N, LIMIT)
    _need(lay.total * 4 * (2 * KQ + 8 * case.C) + ws + lay.total * 64, case.name)
    ups = upstream(case)
    (classes, pred, A, B, crit), grads, ranks = _step(P, xs, LIMIT, 2, ups, lay)
    o = dict(classes=classes, A=A, pred=pred, B=B)
    _check_period(case.name, o, crit, lay)
    for r, rank in enumerate(ranks):
        same_bits(f"{case.name} rank {r} q_max", rank.qmax, lay.bag_src)
    # the first occurrences in bag order: each rank's rows of bag b follow its rows of the bags before
    Q_h, H1_h = [], []
    lo = [0, 0]
    for b, n in enumerate(case.Ns):
        parts = []
        for r, rank in enumerate(ranks):
            parts.append((rank.Q[lo[r]:lo[r] + rank.Ns[b]], rank.H1[lo[r]:lo[r] + rank.Ns[b]]))
            lo[r] += rank.Ns[b]
        Q_h.append(torch.cat([q for q, _ in parts]))
        H1_h.append(torch.cat([h for _, h in parts]))
        assert Q_h[-1].shape[0] == n and min(rank.Ns[b] for rank in ranks) >= 1
    head = dict(o, Q=torch.cat(Q_h), H1=torch.cat(H1_h))
    first = _first_outs(head, crit, lay, case.Ns)
    for b, f in enumerate(first):
        for r, rank in enumerate(ranks):
            qm = FW._np(rank.qmax[b])
            assert np.array_equal(qm, f["Q"][f["crit"]]), (case.name, r, b)
    FW.check_forms(case.name, case, p, {"train": first})
    bcase = BW.Case(case.name, "shard_bags", case.D, case.C, tuple(case.Ns))
    g = _HostGrads(dict(zip(SHARD_NAMES, grads)))
    _check_backward(case, bcase, p, pats, first, ups, g, lay, t0,
                    backward=lambda X, fo, u: orc.backward_sharded(X, p, fo, u[0], u[1], 2))


def _dev_ops(P, xd, Nd, offd, nb, max_rows, status, forward=True):
    """CudaShardBagDevOps over a bag list of pointers (the cycled batch has no [nb, max_rows, D] slots); the forward
    workspace only for ops that run the forward."""
    from dsmil_wsi_b200 import functional as Fn
    from dsmil_wsi_b200.sharded import CudaShardBagDevOps
    ops = CudaShardBagDevOps(P.tensors, Nd[:nb], status)
    ops.nb, ops.max_rows, ops.rows, ops.offs, ops.xs = nb, max_rows, nb * max_rows, offd[:nb], xd[:nb]
    if forward:
        ops.ws = Fn._workspace(ops.lib.dsmil_shard_bags_train_dev_workspace_bytes(P.ref, nb, max_rows), ops.device)
    ops.cand_f = int(ops.lib.dsmil_cand_floats(P.C))
    ops.rec_f = int(ops.lib.dsmil_rec_floats(P.C, P.D))
    return ops


@pytest.mark.gpu
@pytest.mark.parametrize("extra", [0, 20], ids=["full", "short"])
def test_row_sharded_capture_safe_step_gives_the_eager_sharded_bits(extra):
    """CudaShardBagDevOps (G = 1): the forward at nb = 65 535 and the backward at the largest nb it takes give the
    eager sharded calls' bits, with the row capacity max(PATTERN) + extra; at nb = 65 535 bwd1 refuses the batch."""
    from dsmil_wsi_b200.sharded import CudaShardBagOps
    case = SHARD_CASE
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    lib = _lib_load()
    p = FW.make_params(case)
    P = FW._pack(p)
    xs = [FW._t(b.X) for b in FW.bags(case)]
    lay = Layout(case.Ns, LIMIT)
    max_rows = max(case.Ns) + extra
    cap = LIMIT * max_rows
    nb_b = dev_backward_limit(lib, P, "dsmil_shard_", max_rows)
    assert nb_b == 65239, nb_b
    sizes = [lib.dsmil_shard_bags_train_dev_workspace_bytes(P.ref, LIMIT, max_rows),
             lib.dsmil_shard_backward_bags_dev_workspace_bytes(P.ref, nb_b, max_rows)]
    _need(cap * 4 * (2 * KQ + 4 * case.C) + max(sizes) + lay.total * 4 * (2 * KQ + 4 * case.C) + lay.total * 64,
          f"{case.name} dev max_rows={max_rows}")
    xd = torch.tensor([xs[b % len(xs)].data_ptr() for b in range(LIMIT)], dtype=torch.int64, device="cuda")
    Nd = torch.tensor(lay.Ns, dtype=torch.int64, device="cuda")
    offd = torch.zeros(LIMIT, dtype=torch.int64, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    ups = upstream(case)
    dc, dp = _signed(ups, lay, 0), _signed(ups, lay, 1)
    Xs = [xs[b % len(xs)] for b in range(LIMIT)]
    # eager sharded: forward over all bags, backward over the first nb_b
    e = CudaShardBagOps(P.tensors)
    e.begin(Xs, [0] * LIMIT)
    classes, Q, H1, cand = e.phase1_train()
    A, crit, qmax, recs = e.phase2_train(Q, cand, 1)
    A, B, pred = e.phase3_train(recs, 1, A)
    # capture-safe
    d = _dev_ops(P, xd, Nd, offd, LIMIT, max_rows, status)
    classes_d, Q_d, H1_d, cand_d = d.phase1_train()
    A_d, crit_d, qmax_d, recs_d = d.phase2_train(Q_d, cand_d, 1)
    A_d, B_d, pred_d = d.phase3_train(recs_d, 1, A_d)
    torch.cuda.synchronize()
    assert int(status) == 0
    del d
    r = lay.total
    for name, a, b in (("classes", classes_d[:r], classes), ("Q", Q_d[:r], Q), ("H1", H1_d[:r], H1), ("A", A_d[:r], A),
                       ("B", B_d, B), ("pred", pred_d, pred), ("crit", crit_d, crit), ("q_max", qmax_d, qmax),
                       ("cand", cand_d, cand), ("recs", recs_d, recs)):
        _same(f"{case.name} dev {name}", a, b)
    del classes, classes_d, cand, cand_d, recs, recs_d
    # at nb = 65 535 the backward refuses the batch before it launches anything
    d = _dev_ops(P, xd, Nd, offd, LIMIT, max_rows, status, forward=False)
    dcd = torch.full((cap, case.C), 1.0e4, device="cuda")
    dcd[:r] = dc
    with pytest.raises(RuntimeError, match="chunk capacity"):
        d.bwd1([None], A_d, B_d, dcd, dp)
    del d
    rb = sum(lay.Ns[:nb_b])
    e1 = e.bwd1(Xs[:nb_b], A[:rb], B[:nb_b], dc[:rb], dp[:nb_b])
    e2 = e.bwd2(Xs[:nb_b], A[:rb], e1[0], e1[1], Q[:rb])
    e3 = e.bwd3(Xs[:nb_b], [0] * nb_b, Q[:rb], H1[:rb], e2[0], e2[1], qmax[:nb_b], crit[:nb_b])
    torch.cuda.synchronize()
    del e, Q, H1, A
    d = _dev_ops(P, xd, Nd, offd, nb_b, max_rows, status, forward=False)
    d1 = d.bwd1([None], A_d, B_d[:nb_b], dcd, dp[:nb_b])
    d2 = d.bwd2([None], A_d, d1[0], d1[1], Q_d)
    d3 = d.bwd3([None], offd[:nb_b], Q_d, H1_d, d2[0], d2[1], qmax_d[:nb_b], crit_d[:nb_b])
    torch.cuda.synchronize()
    assert int(status) == 0
    _same(f"{case.name} dev t", d1[1], e1[1])
    _same(f"{case.name} dev dL", d2[0][:rb], e2[0])
    _same(f"{case.name} dev dq_max", d2[1], e2[1])
    for k, a, b in zip(("Wi", "bi", "Wf", "bf", "W1", "b1", "W2", "b2"), list(d1[2:]) + list(d3),
                       list(e1[2:]) + list(e3)):
        assert not torch.isnan(b).any(), k
        _same(f"{case.name} dev g{k}", a, b)
    _report(f"{case.name} dev max_rows={max_rows} nb_b={nb_b}", t0)


# ---- candidate records past 2^32 elements of Q ---------------------------------------------------------------------
def _check_cands(name, cand, classes, Q, Ns, offs, C_):
    """Every bag's record: idx = crit + row offset with crit a row of the bag, score = the bag's largest classes[:, k]
    at that row, qrow = Q's row there, bit for bit."""
    nb = len(Ns)
    rec = cand.reshape(nb, -1)
    idx = rec[:, :2 * C_].contiguous().view(torch.int64)
    score = rec[:, 2 * C_:3 * C_]
    qrow = rec[:, 3 * C_:3 * C_ + C_ * KQ].reshape(nb, C_, KQ)
    n = torch.tensor(Ns, dtype=torch.int64, device="cuda")
    start = torch.cumsum(n, 0) - n
    crit = idx - offs[:, None]
    assert bool(((crit >= 0) & (crit < n[:, None])).all()), f"{name}: a record names a row outside its bag"
    row = start[:, None] + crit
    cols = torch.arange(C_, device="cuda")
    _same(f"{name} score", score.contiguous(), classes[row, cols[None, :]].contiguous())
    bag = torch.repeat_interleave(torch.arange(nb, device="cuda"), n)
    top = torch.full((nb, C_), float("-inf"), device="cuda").scatter_reduce_(0, bag[:, None].expand(-1, C_),
                                                                              classes[:bag.numel()], "amax")
    del bag
    _same(f"{name} score is the bag's maximum", score.contiguous(), top)
    for lo in range(0, nb, 8192):
        _same(f"{name} qrow", qrow[lo:lo + 8192].contiguous(), Q[row[lo:lo + 8192]].contiguous())


@pytest.mark.gpu
def test_candidate_records_read_q_past_2_32_elements():
    """D = 128, 65 535 bags of PATTERN_Q (33.8 M rows): dsmil_shard_bags_phase1_train's records against its row-major
    Q, dsmil_shard_bags_phase1's (tile-blocked Q, tanh_ex2 on the block entry) the same records."""
    case = CAND_CASE
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    lib = _lib_load()
    P = FW._pack(FW.make_params(case))
    xs = [FW._t(b.X) for b in FW.bags(case)]
    Ns = cycle(case.Ns, LIMIT)
    rows = sum(Ns)
    assert rows * KQ > 1 << 32
    c_X, c_N = _bag_ptrs(xs, Ns)
    ws_b = lib.dsmil_shard_bags_workspace_bytes(P.ref, c_N, LIMIT)
    assert ws_b > 0
    _need(rows * 4 * (2 * KQ + 2 * case.C) + ws_b + rows * 16 + (1 << 30), case.name)
    offs_h = [b * 65537 + 3 for b in range(LIMIT)]            # offsets past 2^32 in the last bags
    c_off = (C.c_int64 * LIMIT)(*offs_h)
    offs = torch.tensor(offs_h, dtype=torch.int64, device="cuda")
    cand_f = int(lib.dsmil_cand_floats(case.C))
    classes, Q, H1 = FW._nan(rows, case.C), FW._nan(rows, KQ), FW._nan(rows, KQ)
    cand = FW._nan(LIMIT, cand_f)
    ws = FW._ws(ws_b)
    rc = lib.dsmil_shard_bags_phase1_train(P.ref, c_X, c_N, LIMIT, c_off, classes.data_ptr(), Q.data_ptr(),
                                           H1.data_ptr(), cand.data_ptr(), ws.data_ptr(), ws.numel(), FW._stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.dsmil_last_error()
    del H1
    _check_cands(f"{case.name} row-major", cand, classes, Q, Ns, offs, case.C)
    classes_e, cand_e = FW._nan(rows, case.C), FW._nan(LIMIT, cand_f)
    rc = lib.dsmil_shard_bags_phase1(P.ref, c_X, c_N, LIMIT, c_off, classes_e.data_ptr(), cand_e.data_ptr(),
                                     ws.data_ptr(), ws.numel(), FW._stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.dsmil_last_error()
    _same(f"{case.name} eval classes", classes_e, classes)
    _same(f"{case.name} tile-blocked records", cand_e, cand)
    _report(case.name, t0)


@pytest.mark.gpu
def test_capture_safe_candidate_records_read_q_past_2_32_elements():
    """dsmil_shard_bags_phase1_train_dev over 65 535 bags of 513..523 rows (its capacity buffers for PATTERN_Q's
    1537-row bags would not fit the card): the live Q passes 2^32 elements, and every record holds its row."""
    case = CAND_DEV_CASE
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    lib = _lib_load()
    P = FW._pack(FW.make_params(case))
    xs = [FW._t(b.X) for b in FW.bags(case)]
    Ns = cycle(case.Ns, LIMIT)
    max_rows = max(case.Ns)
    rows, cap = sum(Ns), LIMIT * max_rows
    assert rows * KQ > 1 << 32
    ws_b = lib.dsmil_shard_bags_train_dev_workspace_bytes(P.ref, LIMIT, max_rows)
    assert ws_b > 0
    _need(cap * 4 * (2 * KQ + case.C) + ws_b + rows * 16 + (1 << 30), case.name)
    offs = torch.arange(LIMIT, dtype=torch.int64, device="cuda") * 65537 + 3
    xd = torch.tensor([xs[b % len(xs)].data_ptr() for b in range(LIMIT)], dtype=torch.int64, device="cuda")
    Nd = torch.tensor(Ns, dtype=torch.int64, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    classes, Q, H1 = FW._nan(cap, case.C), FW._nan(cap, KQ), FW._nan(cap, KQ)
    cand = FW._nan(LIMIT, int(lib.dsmil_cand_floats(case.C)))
    ws = FW._ws(ws_b)
    rc = lib.dsmil_shard_bags_phase1_train_dev(P.ref, xd.data_ptr(), Nd.data_ptr(), offs.data_ptr(), LIMIT, max_rows,
                                               classes.data_ptr(), Q.data_ptr(), H1.data_ptr(), cand.data_ptr(),
                                               status.data_ptr(), ws.data_ptr(), ws.numel(), FW._stream())
    torch.cuda.synchronize()
    assert rc == 0 and int(status) == 0, lib.dsmil_last_error()
    del H1, ws
    _check_cands(case.name, cand, classes, Q, Ns, offs, case.C)
    _report(case.name, t0)


# ---- capture-safe value calls ------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", VALUE_DEV_CASES, ids=lambda c: c.name)
def test_capture_safe_value_calls_at_the_limit_give_the_eager_bits(case):
    """dsmil_value_forward_bags_dev (with saves and without) at nb = 65 535 gives dsmil_value_forward_bags's bits, and
    dsmil_value_backward_bags_dev at the largest nb it takes gives dsmil_value_backward_bags's, row capacity
    max(PATTERN); on v's masked inputs for the masked case."""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    lib = _lib_load()
    p = FW.make_params(case)
    P = FW._pack(p)
    xs = [FW._t(b.X) for b in FW.bags(case)]
    vms = FW.v_masks(case)
    xvs = None if vms[0] is None else [x * FW._t(m) for x, m in zip(xs, vms)]
    lay = Layout(case.Ns, LIMIT)
    max_rows = max(case.Ns)
    cap, r = LIMIT * max_rows, lay.total
    nb_b = dev_backward_limit(lib, P, "dsmil_value_", max_rows)
    assert nb_b == 65239, nb_b
    c_X, c_N = _bag_ptrs(xs, lay.Ns)
    c_XV = None if xvs is None else _bag_ptrs(xvs, lay.Ns)[0]
    sizes = [lib.dsmil_value_forward_bags_workspace_bytes(P.ref, c_N, LIMIT),
             lib.dsmil_value_forward_bags_dev_workspace_bytes(P.ref, LIMIT, max_rows),
             lib.dsmil_value_backward_bags_workspace_bytes(P.ref, c_N, nb_b, 0),
             lib.dsmil_value_backward_bags_dev_workspace_bytes(P.ref, nb_b, max_rows)]
    assert min(sizes) > 0
    _need(cap * 4 * (2 * KQ + case.D + 4 * case.C) + max(sizes) + r * 4 * (2 * KQ + case.D) + r * 64, case.name)
    xd = torch.tensor([xs[b % len(xs)].data_ptr() for b in range(LIMIT)], dtype=torch.int64, device="cuda")
    xvd = None if xvs is None else torch.tensor([xvs[b % len(xs)].data_ptr() for b in range(LIMIT)],
                                                dtype=torch.int64, device="cuda")
    Nd = torch.tensor(lay.Ns, dtype=torch.int64, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    keep = None
    for train in (False, True):
        form = "train" if train else "eval"
        ref, ref_crit = FW._new_outs(r, LIMIT, case, saves=train)
        ws = FW._ws(sizes[0])
        rc = lib.dsmil_value_forward_bags(P.ref, c_X, c_XV, c_N, LIMIT,
                                          *[FW._ptr(ref[k]) for k in ("classes", "pred", "A", "B")],
                                          ref_crit.data_ptr(), *[FW._ptr(ref.get(k)) for k in ("Q", "H1", "V")],
                                          ws.data_ptr(), ws.numel(), FW._stream())
        torch.cuda.synchronize()
        assert rc == 0, lib.dsmil_last_error()
        del ws
        o, crit = FW._new_outs(cap, LIMIT, case, saves=train)
        ws = FW._ws(sizes[1])
        rc = lib.dsmil_value_forward_bags_dev(P.ref, xd.data_ptr(), FW._ptr(xvd), Nd.data_ptr(), LIMIT, max_rows,
                                              *[FW._ptr(o[k]) for k in ("classes", "pred", "A", "B")], crit.data_ptr(),
                                              *[FW._ptr(o.get(k)) for k in ("Q", "H1", "V")], status.data_ptr(),
                                              ws.data_ptr(), ws.numel(), FW._stream())
        torch.cuda.synchronize()
        assert rc == 0 and int(status) == 0, lib.dsmil_last_error()
        del ws
        _same_outs(f"{case.name} {form}", o, crit, ref, ref_crit)
        del ref, ref_crit
        if train:
            keep = (o, crit)
        del o, crit
    # the backward through classes and pred over the first nb_b bags of the same saves (the dev saves hold the eager
    # bits in their live rows, so both calls read the same buffers)
    o, crit = keep
    rb = sum(lay.Ns[:nb_b])
    ups = upstream(case)
    dc, dp = _signed(ups, lay, 0)[:rb], _signed(ups, lay, 1)[:nb_b]
    bcase = BW.Case(case.name, "dev", case.D, case.C, tuple(case.Ns), passing_v=True)
    g_e, g_d = BW._Grads(bcase), BW._Grads(bcase)
    G = g_e.struct()
    c_X, c_N = _bag_ptrs(xs, lay.Ns[:nb_b])
    c_XV = None if xvs is None else _bag_ptrs(xvs, lay.Ns[:nb_b])[0]
    saves = [FW._ptr(o[k]) for k in ("Q", "H1", "V", "A", "B")] + [crit.data_ptr()]
    ws = FW._ws(sizes[2])
    rc = lib.dsmil_value_backward_bags(P.ref, c_X, c_XV, c_N, nb_b, *saves, dc.data_ptr(), dp.data_ptr(), None, None,
                                       None, C.byref(G), ws.data_ptr(), ws.numel(), FW._stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.dsmil_last_error()
    del ws
    dcd = torch.full((nb_b * max_rows, case.C), 1.0e4, device="cuda")
    dcd[:rb] = dc
    Gd = g_d.struct()
    ws = FW._ws(sizes[3])
    rc = lib.dsmil_value_backward_bags_dev(P.ref, xd.data_ptr(), FW._ptr(xvd), Nd.data_ptr(), nb_b, max_rows, *saves,
                                           dcd.data_ptr(), dp.data_ptr(), None, None, C.byref(Gd), status.data_ptr(),
                                           ws.data_ptr(), ws.numel(), FW._stream())
    torch.cuda.synchronize()
    assert rc == 0 and int(status) == 0, (lib.dsmil_last_error(), int(status))
    for k, t in g_e.t.items():
        assert not torch.isnan(t).any(), (case.name, k)
        _same(f"{case.name} g{k}", g_d.t[k], t)
    _report(f"{case.name} nb_b={nb_b}", t0)
