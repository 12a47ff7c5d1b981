"""The bag calls at the ends of the batch range they accept, held to the conditioned checks of
`test_conditioned_forward_gpu.py` (FW) and `test_conditioned_backward_gpu.py` (BW).

Every other GPU test launches a few dozen bags at most, so no kernel had run with blockIdx.y near 65 535, no packed
output had passed 2^31 elements, and no bag-order sum had a chain longer than a few dozen bags.  Here each batch is built
from P = 11 distinct bags (FW's peaked bags, row counts including 1, 2, 127, 128 and 129), laid out in a cycle: bag b is
pattern b mod P, its features a pointer into that pattern's one device buffer, so X costs almost nothing whatever the
batch.  Each case checks two things:

  1. periodicity: every occurrence of a pattern gives the bits of its first occurrence (classes, crit, Q, H1, A, B,
     pred; gX rows in the backward), compared on the device through a row map.  A kernel that reads or writes a
     neighbour's slot, or an offset that wraps, breaks it.
  2. the first occurrence of each pattern passes the conditioned checks: FW.check_forms on its own Q, and the fp64
     backward on its own saves (BW's bars, gX row by row).

Upstream gradients repeat with period 2P and change sign every P bags.  The backward is linear in them, so a negated bag
gives exactly the negated terms, every window of 2P bags sums to zero, and the partial sums of every bag-order chain stay
bounded however long the batch.  A cross-bag sum is then sum_p w_p g_p in fp64, w_p the signed count of pattern p; at
nb = 65 535 = 2978 * 22 + 19 three patterns are left over, so no single bag's term is the answer.  gWf and gbf
(k_bwd_bag_b) add nb terms in bag order; their bar is C_SUM u sum_b |S_b| over the fp64 partial sums S_b of that chain.
The other sums (gWi, gbi and the q.* gradients) go through chunk and split partials of at least one per bag: their bar
is (BW's bar + C_SUM u nb) max_b |S_b|, the stage bar and a chain of nb partials, each at most the largest partial sum.
The CPU part shows that an fp32 restatement of each chain, in the kernel's order, stays 4x under its bar, and that
dropping or doubling the last bag's term moves the sum by more than 20x it.

Cases:
  - nb = 65 535: dsmil_forward_bags_train and dsmil_forward_bags, then dsmil_backward_bags with gX, on the tensor-core
    route (D = 512, C = 2) and the generic one (D = 166, C = 5).  The tensor-core bags average more than 128 rows, so gX
    [sum N, 512] passes 2^32 elements (18 GB).
  - nb = 65 535: dsmil_value_forward_bags and dsmil_value_backward_bags; the capture-safe forward pair (tensor-core
    and dsmil_generic_*) with its row capacity filled and not, equal to the eager calls' bits, and the capture-safe
    backward at the largest nb it takes (it refuses a chunk grid past 65 535).
  - nb = 65 536 and 70 000 on the calls that take any nb: dsmil_forward_bags and _train on tensor-core, generic and
    passing_v shapes, and dsmil_forward_bags_models.  Every bag must equal dsmil_forward on that bag alone, bit for bit.
  - Q past 2^32 elements: D = 128, 65 535 bags of 33.8 M rows in all, training and eval forms.
  - One bag of 2^24 + 129 rows at D = 128: its critical rows sit past 2^24, where a row index cannot be held in a
    float, and every row there must give the A bits of the same row one period earlier.

Not covered at the limit: the fused fold calls at nb * M = 65 535, the row-sharded batch, and the capture-safe
backwards of the fold and row-sharded forms.

The large cases first ask torch.cuda.mem_get_info() for the memory they need and skip, naming it, when the card lacks
it.  Largest errors over bars, peak memory and run times are in DESIGN §3.
"""
from __future__ import annotations

import ctypes as C
import functools
import time

import numpy as np
import pytest
import torch

import test_conditioned_backward_gpu as BW
import test_conditioned_forward_gpu as FW
from oracle import dsmil_oracle as orc
from test_dense_upstream_grads_gpu import rowwise_err

U = FW.U
KQ = FW.KQ
LIMIT = 65535                  # the most bags a batched call numbers in one grid dimension
C_SUM = 2.0                    # bag-order sums: first-order bound u sum |S_b|, doubled for the fma and higher orders
SENSITIVITY = 20.0
# row counts of the P = 11 patterns; the tensor-core backward's average more than 128 rows (gX past 2^32 elements at
# D = 512), the D = 128 batch's more than 512 (Q past 2^32 elements)
PATTERN = (1, 2, 127, 128, 129, 33, 300, 64, 257, 3, 31)
PATTERN_GX = (1, 2, 127, 128, 129, 300, 257, 64, 33, 200, 300)
PATTERN_Q = (1, 2, 127, 128, 129, 1000, 1537, 700, 257, 1024, 771)
P_BAGS = len(PATTERN)
BIG_N = (1 << 24) + 129


def cycle(pattern, nb):
    return [pattern[b % len(pattern)] for b in range(nb)]


def signs(nb, P=P_BAGS):
    """+1 on bags [0, P) of every window of 2P bags, -1 on the rest."""
    return np.where((np.arange(nb) // P) % 2 == 0, 1.0, -1.0)


def signed_counts(nb, P=P_BAGS):
    """w_p = sum of the signs of the bags of pattern p."""
    w = np.zeros(P)
    np.add.at(w, np.arange(nb) % P, signs(nb, P))
    return w


def chain_bar(terms_p, nb, P=P_BAGS):
    """Bar of an fp32 sum of nb terms in bag order, term b = sign_b terms_p[b mod P] (terms_p [P, ...] in fp64):
    C_SUM u sum_b |S_b|.  The partial sums repeat with period 2P (each window sums to zero), so sum_b |S_b| is the
    count of each window position times |S| there."""
    s = signs(2 * P, P)
    window = np.cumsum(s.reshape((-1,) + (1,) * (terms_p.ndim - 1)) * np.concatenate([terms_p, terms_p]), axis=0)
    counts = np.bincount(np.arange(nb) % (2 * P), minlength=2 * P).astype(np.float64)
    return C_SUM * U * np.tensordot(counts, np.abs(window), axes=1)


def chain_max(terms_p, P=P_BAGS):
    """The largest |S_b| of that chain over every element."""
    s = signs(2 * P, P)
    return float(np.abs(np.cumsum(s.reshape((-1,) + (1,) * (terms_p.ndim - 1)) *
                                  np.concatenate([terms_p, terms_p]), axis=0)).max())


def fp32_chain(terms_p, nb, P=P_BAGS, fma_with=None, weight_last=1.0):
    """The kernel's chain restated in fp32: s += term_b (gbf) or s = fma(dp_b, B_b, s) (gWf: terms_p are the dp and
    fma_with the B of each pattern), in bag order; weight_last scales the last bag's term (0 drops it, 2 doubles it)."""
    sg = signs(nb, P).astype(np.float32)
    s = np.zeros(terms_p.shape[1:] if fma_with is None else np.broadcast(terms_p[0], fma_with[0]).shape, np.float32)
    for b in range(nb):
        a = terms_p[b % P].astype(np.float32) * sg[b] * np.float32(weight_last if b == nb - 1 else 1.0)
        if fma_with is None:
            s = (s + a).astype(np.float32)
        else:
            s = (np.float64(1.0) * a * fma_with[b % P].astype(np.float64) + s).astype(np.float32)
    return s


# ---------------------------------------------------------------------------------------------------------- cases
LIMIT_CASES = [FW.Case("limit_tc_d512_c2", "bags", 512, 2, PATTERN_GX),
               FW.Case("limit_gen_d166_c5", "bags", 166, 5, PATTERN)]
BEYOND_CASES = [FW.Case("beyond_tc_d512_c2", "bags", 512, 2, PATTERN),
                FW.Case("beyond_gen_d166_c5", "bags", 166, 5, PATTERN),
                FW.Case("beyond_pv_d512_c2", "value", 512, 2, PATTERN, passing_v=True),
                FW.Case("beyond_models_d512_c2", "models", 512, 2, PATTERN)]
Q_CASE = FW.Case("limit_q_tc_d128_c2", "bags", 128, 2, PATTERN_Q)


def upstream(case, P=P_BAGS):
    """Per pattern (d_classes [n, C], d_pred [C], d_A [n, C], d_B [C, D]), float32, as BW.upstream draws them."""
    rng = np.random.default_rng(5000 + case.seed)
    out = []
    for n in case.Ns:
        f = lambda a: a.astype(np.float32)
        out.append((f(1.0 + rng.standard_normal((n, case.C))), f(rng.standard_normal(case.C)),
                    f(rng.standard_normal((n, case.C))), f(1e-2 * rng.standard_normal((case.C, case.D)))))
    return out


@functools.lru_cache(maxsize=None)
def cpu_bag_sums(case):
    """The stand-in terms of gbf and gWf: each pattern's d_pred and the fp32 oracle's B."""
    p, fos = FW.cpu_forward(case)
    dp = np.stack([u[1] for u in upstream(case)]).astype(np.float64)               # [P, C]
    B = np.stack([fo.B.reshape(-1) for fo in fos]).astype(np.float64)               # [P, C * D]
    return dp, B


# ===================================================================================== CPU part: no device needed
def test_window_signs_cancel_and_leave_three_patterns_at_the_limit():
    w = signed_counts(LIMIT)
    assert np.array_equal(w, [0] * 8 + [1] * 3), w              # 65 535 = 2978 * 22 + 19
    assert signs(2 * P_BAGS).sum() == 0
    for pat in (PATTERN, PATTERN_GX, PATTERN_Q):
        assert {1, 2, 127, 128, 129} <= set(pat) and len(pat) == P_BAGS
    assert sum(cycle(PATTERN_GX, LIMIT)) * 512 > 1 << 32
    assert sum(cycle(PATTERN_Q, LIMIT)) * KQ > 1 << 32
    assert BIG_N - 1 > 1 << 24 and float(np.float32(BIG_N - 64)) != BIG_N - 64


@pytest.mark.parametrize("case", LIMIT_CASES, ids=lambda c: c.name)
def test_fp32_bag_order_sums_stay_4x_under_their_bars_and_the_last_bag_moves_them_past_20x(case):
    """gbf = sum_b dp_b and gWf[k] = sum_b dp_b[k] B_b, nb = 65 535 terms in bag order (k_bwd_bag_b)."""
    dp, B = cpu_bag_sums(case)
    w = signed_counts(LIMIT)
    Cc = case.C
    sums = {"bf": (dp, None, w @ dp, chain_bar(dp, LIMIT)),
            "Wf": (dp[:, :, None], B[:, None, :], np.einsum("p,pk,pi->ki", w, dp, B),
                   chain_bar(dp[:, :, None] * B[:, None, :], LIMIT))}
    for name, (terms, fw, want, bar) in sums.items():
        assert want.shape == bar.shape == ((Cc,) if name == "bf" else (Cc, Cc * case.D))
        err = FW.over(np.abs(fp32_chain(terms, LIMIT, fma_with=fw) - want), bar)
        assert err <= 0.25, (case.name, name, err)
        for wl in (0.0, 2.0):
            moved = FW.over(np.abs(fp32_chain(terms, LIMIT, fma_with=fw, weight_last=wl) - want), bar)
            assert moved > SENSITIVITY, (case.name, name, wl, moved)
        print(f"{case.name} g{name}: fp32 chain {err:.3g} of its bar")


# ========================================================================================== GPU part (one H100)


def _need(nbytes, what):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"{what} needs {nbytes / 2 ** 30:.1f} GiB free on the device, {free / 2 ** 30:.1f} GiB is")


class Layout:
    """Row and bag maps of a cycled batch on the device: row_src / bag_src name the same row / bag of the pattern's
    first occurrence; row_sign / bag_sign the upstream's sign."""

    def __init__(self, pattern, nb):
        P = len(pattern)
        self.Ns = cycle(pattern, nb)
        self.nb, self.total, self.first_rows = nb, sum(self.Ns), sum(pattern)
        n = torch.tensor(self.Ns, dtype=torch.int64, device="cuda")
        start = torch.cumsum(n, 0) - n
        bag = torch.repeat_interleave(torch.arange(nb, device="cuda"), n)
        self.bag_src = torch.arange(nb, device="cuda") % P
        self.row_src = start[bag % P] + torch.arange(self.total, device="cuda") - start[bag]
        self.bag_sign = torch.from_numpy(signs(nb, P)).float().cuda()
        self.row_sign = self.bag_sign[bag]
        del bag


def same_bits(name, t, src, ref=None, sign=None):
    """Every row of t has the bits of row src of ref (default t), or equals sign x that row (sign: the upstream's)."""
    ref = t if ref is None else ref
    rows = t.shape[0]
    t2, r2 = t.reshape(rows, -1), ref.reshape(ref.shape[0], -1)
    step = max(1, (1 << 28) // max(t2.shape[1], 1))
    for lo in range(0, rows, step):
        a, b = t2[lo:lo + step], r2[src[lo:lo + step]]
        if sign is not None:
            ok = torch.equal(a, b * sign[lo:lo + step, None]) and not torch.isnan(a).any()
        elif a.dtype == torch.float32:
            ok = torch.equal(a.view(torch.int32), b.view(torch.int32))
        else:
            ok = torch.equal(a, b)
        if not ok:
            bad = (a != b if sign is None else a != b * sign[lo:lo + step, None]).reshape(a.shape[0], -1).any(1)
            first = lo + int(torch.nonzero(bad)[0]) if bad.any() else lo
            raise AssertionError(f"{name}: row {first} differs from row {int(src[first])} of its pattern")


@pytest.fixture(autouse=True)
def _release_device_memory():
    """Each case sizes its skip on the memory free when it starts."""
    yield
    import gc
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def _lib_load():
    return FW._lib_load()


def _bag_ptrs(xs, Ns):
    """Host bag list of the cycled batch (xs [None]: the row counts alone)."""
    nb = len(Ns)
    P = len(xs)
    ptrs = [0 if xs[b % P] is None else xs[b % P].data_ptr() for b in range(nb)]
    return (C.c_void_p * nb)(*ptrs), (C.c_int64 * nb)(*Ns)


def _first_outs(o, crit, lay, pattern, saves=("Q", "H1")):
    """Host per-bag dicts (FW._outs) of the first P bags of packed device outputs."""
    r, P = lay.first_rows, len(pattern)
    head = {k: (None if v is None else (v[:r] if k in ("classes", "A", "Q", "H1", "V") else v[:P])) for k, v in o.items()}
    return FW._outs(head, crit[:P], list(pattern), saves=saves)


def _forward_batch(lib, P, xs, lay, case, train):
    """dsmil_forward_bags_train (saves) or dsmil_forward_bags over the cycled batch; packed device outputs."""
    c_X, c_N = _bag_ptrs(xs, lay.Ns)
    o, crit = FW._new_outs(lay.total, lay.nb, case, saves=train)
    args = [FW._ptr(o[k]) for k in ("classes", "pred", "A", "B")] + [crit.data_ptr()]
    if train:
        ws = FW._ws(lib.dsmil_forward_bags_train_workspace_bytes(P.ref, c_N, lay.nb))
        rc = lib.dsmil_forward_bags_train(P.ref, c_X, c_N, lay.nb, *args, FW._ptr(o["Q"]), FW._ptr(o["H1"]),
                                          ws.data_ptr(), ws.numel(), FW._stream())
    else:
        ws = FW._ws(lib.dsmil_forward_bags_workspace_bytes(P.ref, c_N, lay.nb))
        rc = lib.dsmil_forward_bags(P.ref, c_X, c_N, lay.nb, *args, ws.data_ptr(), ws.numel(), FW._stream())
    torch.cuda.synchronize()
    del ws
    assert rc == 0, (case.name, lay.nb, lib.dsmil_last_error())
    return o, crit


def _check_period(name, o, crit, lay):
    for k in ("classes", "A", "Q", "H1", "V"):
        if o.get(k) is not None:
            same_bits(f"{name} {k}", o[k], lay.row_src)
    for k in ("pred", "B"):
        same_bits(f"{name} {k}", o[k], lay.bag_src)
    same_bits(f"{name} crit", crit, lay.bag_src)


def _report(name, t0):
    torch.cuda.synchronize()
    print(f"{name}: {time.time() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")


@pytest.mark.gpu
@pytest.mark.parametrize("case", LIMIT_CASES, ids=lambda c: c.name)
def test_forward_and_backward_of_65535_bags(case):
    """dsmil_forward_bags_train and dsmil_forward_bags, then dsmil_backward_bags with d_A, d_B and gX, at nb = 65 535."""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    lib = _lib_load()
    p = FW.make_params(case)
    P = FW._pack(p)
    Ns = cycle(case.Ns, LIMIT)
    rows, (_, c_N) = sum(Ns), _bag_ptrs([None], Ns)
    ws = max(lib.dsmil_forward_bags_train_workspace_bytes(P.ref, c_N, LIMIT),
             lib.dsmil_forward_bags_workspace_bytes(P.ref, c_N, LIMIT))
    # the saves and the per-row outputs, the larger forward workspace (the other form's outputs live beside it), gX and
    # the upstream, the backward's workspace, and the row maps
    _need(rows * 4 * (2 * KQ + 8 * case.C + case.D) + ws + lib.dsmil_backward_bags_workspace_bytes(P.ref, c_N, LIMIT, 1)
          + rows * 48, case.name)
    pats = FW.bags(case)
    xs = [FW._t(b.X) for b in pats]
    lay = Layout(case.Ns, LIMIT)
    o, crit = _forward_batch(lib, P, xs, lay, case, True)
    _check_period(f"{case.name} train", o, crit, lay)
    oe, crite = _forward_batch(lib, P, xs, lay, case, False)
    _check_period(f"{case.name} eval", oe, crite, lay)
    FW.check_forms(case.name, case, p, {"train": _first_outs(o, crit, lay, case.Ns),
                                         "eval": _first_outs(oe, crite, lay, case.Ns)})
    del oe, crite

    # the backward over the same saves, upstream of period 2P with alternating sign
    ups = upstream(case)
    pat = lambda i: torch.from_numpy(np.concatenate([u[i] for u in ups])).cuda()
    dc = pat(0)[lay.row_src] * lay.row_sign[:, None]
    dA = pat(2)[lay.row_src] * lay.row_sign[:, None]
    dp = torch.from_numpy(np.stack([u[1] for u in ups])).cuda()[lay.bag_src] * lay.bag_sign[:, None]
    dB = torch.from_numpy(np.stack([u[3] for u in ups])).cuda()[lay.bag_src] * lay.bag_sign[:, None, None]
    bcase = BW.Case(case.name, "bags", case.D, case.C, tuple(case.Ns), nonlinear=case.nonlinear)
    g = BW._Grads(bcase, lay.total)
    G = g.struct()
    c_X, c_N = _bag_ptrs(xs, lay.Ns)
    ws = FW._ws(lib.dsmil_backward_bags_workspace_bytes(P.ref, c_N, LIMIT, 1))
    rc = lib.dsmil_backward_bags(P.ref, c_X, c_N, LIMIT, FW._ptr(o["Q"]), FW._ptr(o["H1"]), FW._ptr(o["A"]),
                                 FW._ptr(o["B"]), crit.data_ptr(), dc.data_ptr(), dp.data_ptr(), dA.data_ptr(),
                                 dB.data_ptr(), C.byref(G), ws.data_ptr(), ws.numel(), FW._stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.dsmil_last_error()
    del ws, dc, dA
    same_bits(f"{case.name} gX", g.gX, lay.row_src, sign=lay.row_sign)

    _check_backward(case, bcase, p, pats, _first_outs(o, crit, lay, case.Ns), ups, g, lay, t0)


def _check_backward(case, bcase, p, pats, host, ups, g, lay, t0, nb=LIMIT, backward=None):
    """First occurrences: the fp64 backward on their own saves (gX row by row, when g has one); the sums over the nb
    bags: sum_p w_p g_p.  backward(X, fo, u) gives a pattern's fp64 gradients (default: orc.backward with gX)."""
    per = []
    for X, h, u in zip([b.X for b in pats], host, ups):
        fo = orc.FwdOut(None, None, h["A"], h["B"], h["crit"], Q=h["Q"], H1=h.get("H1"), V=h.get("V", X))
        per.append(orc.backward(X, p, fo, u[0], u[1], d_A=u[2], d_B=u[3], need_dX=True) if backward is None else
                   backward(X, fo, u))
    P = len(per)
    w = signed_counts(nb, P)
    got = g.host()
    errs = {}
    for k in bcase.names():
        want = sum(wp * gp[k] for wp, gp in zip(w, per))
        if k in ("Wf", "bf"):
            terms = np.stack([gp[k] for gp in per])          # each bag's term: dp_b[k] B_b, or dp_b
            errs[k] = FW.over(np.abs(got[k] - want), chain_bar(terms, nb, P))
        else:                                                 # the chunk and split sums of the other kernels
            terms = np.stack([gp[k] for gp in per])
            errs[k] = float(np.max(np.abs(got[k] - want))) / ((bcase.bar(k) + C_SUM * U * nb) * chain_max(terms, P))
    if g.gX is not None:
        starts = np.cumsum([0] + list(case.Ns))
        gX = FW._np(g.gX[:lay.first_rows])
        errs["X"] = max(rowwise_err(gX[starts[j]:starts[j + 1]], gp["X"]) for j, gp in enumerate(per)) / bcase.bar("X")
    print(f"{case.name} backward, error over bar: " + " ".join(f"{k}={v:.3g}" for k, v in errs.items()))
    _report(case.name, t0)
    bad = {k: v for k, v in errs.items() if not v <= 1.0}
    assert not bad, (case.name, bad)


def _single_refs(lib, P, xs, case, train):
    """dsmil_forward of each pattern alone, packed as the first P bags of a batch (saves on the training form)."""
    Ns = list(case.Ns)
    o, crit = FW._new_outs(sum(Ns), len(Ns), case, saves=train)
    row = 0
    for b, (x, n) in enumerate(zip(xs, Ns)):
        ws = FW._ws(lib.dsmil_forward_workspace_bytes(P.ref, n))
        sl = lambda k, w=1: None if o.get(k) is None else o[k][row:row + n].data_ptr()
        rc = lib.dsmil_forward(P.ref, x.data_ptr(), None, n, sl("classes"), o["pred"][b].data_ptr(),
                               sl("A"), o["B"][b].data_ptr(), crit[b].data_ptr(), sl("Q"), sl("H1"), sl("V"),
                               ws.data_ptr(), ws.numel(), FW._stream())
        assert rc == 0, lib.dsmil_last_error()
        row += n
    torch.cuda.synchronize()
    return o, crit


def _against_singles(name, o, crit, ref, ref_crit, lay):
    for k in ("classes", "A", "Q", "H1", "V"):
        if o.get(k) is not None:
            same_bits(f"{name} {k}", o[k], lay.row_src, ref=ref[k])
    for k in ("pred", "B"):
        same_bits(f"{name} {k}", o[k], lay.bag_src, ref=ref[k])
    same_bits(f"{name} crit", crit, lay.bag_src, ref=ref_crit)


@pytest.mark.gpu
@pytest.mark.parametrize("nb", [LIMIT + 1, 70000])
@pytest.mark.parametrize("case", BEYOND_CASES, ids=lambda c: c.name)
def test_more_than_65535_bags_give_each_bag_its_own_forward(case, nb):
    """dsmil_forward_bags and _train (not on passing_v), or dsmil_forward_bags_models over two models, past 65 535 bags:
    every bag gives the bits dsmil_forward gives it alone."""
    t0 = time.time()
    lib = _lib_load()
    lay = Layout(case.Ns, nb)
    pats = FW.bags(case)
    xs = [FW._t(b.X) for b in pats]
    if case.route == "models":
        from dsmil_wsi_b200 import _lib
        ps = [FW._pack(FW.make_params(case, m)) for m in range(2)]
        c_ps = (_lib.DsmilParams * 2)(*[q.struct for q in ps])
        c_X, c_N = _bag_ptrs(xs, lay.Ns)
        o, crit = FW._new_outs(2 * lay.total, 2 * nb, case)
        ws = FW._ws(lib.dsmil_forward_bags_models_workspace_bytes(c_ps, 2, c_N, nb))
        rc = lib.dsmil_forward_bags_models(c_ps, 2, c_X, c_N, nb, *[FW._ptr(o[k]) for k in ("classes", "pred", "A",
                                                                                            "B")],
                                           crit.data_ptr(), ws.data_ptr(), ws.numel(), FW._stream())
        torch.cuda.synchronize()
        assert rc == 0, (case.name, nb, lib.dsmil_last_error())
        del ws
        for m, P in enumerate(ps):
            ref, ref_crit = _single_refs(lib, P, xs, case, False)
            r0, b0 = m * lay.total, m * nb
            om = {k: o[k][r0:r0 + lay.total] if k in ("classes", "A") else o[k][b0:b0 + nb] for k in o}
            _against_singles(f"{case.name} nb={nb} model {m}", om, crit[b0:b0 + nb], ref, ref_crit, lay)
        _report(f"{case.name} nb={nb}", t0)
        return
    p = FW.make_params(case)
    P = FW._pack(p)
    for train in ((False,) if case.passing_v else (False, True)):
        ref, ref_crit = _single_refs(lib, P, xs, case, train)
        if case.passing_v:
            c_X, c_N = _bag_ptrs(xs, lay.Ns)
            o, crit = FW._new_outs(lay.total, nb, case)
            ws = FW._ws(lib.dsmil_forward_bags_workspace_bytes(P.ref, c_N, nb))
            rc = lib.dsmil_forward_bags(P.ref, c_X, c_N, nb, *[FW._ptr(o[k]) for k in ("classes", "pred", "A", "B")],
                                        crit.data_ptr(), ws.data_ptr(), ws.numel(), FW._stream())
            torch.cuda.synchronize()
            assert rc == 0, (case.name, nb, lib.dsmil_last_error())
        else:
            o, crit = _forward_batch(lib, P, xs, lay, case, train)
        _against_singles(f"{case.name} nb={nb} {'train' if train else 'eval'}", o, crit, ref, ref_crit, lay)
        if train:                       # the first occurrences on their own Q as well
            FW.check_forms(f"{case.name} nb={nb}", case, p, {"train": _first_outs(o, crit, lay, case.Ns)})
    _report(f"{case.name} nb={nb}", t0)


@pytest.mark.gpu
def test_q_past_2_32_elements_over_65535_bags():
    """D = 128: 65 535 bags of 33.8 M rows, so the training form's row-major Q and H1 and the eval form's tile-blocked
    Q pass 2^32 elements; the attend pass reads q_max rows there."""
    case = Q_CASE
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    lib = _lib_load()
    p = FW.make_params(case)
    P = FW._pack(p)
    Ns = cycle(case.Ns, LIMIT)
    rows, (_, c_N) = sum(Ns), _bag_ptrs([None], Ns)
    ws = max(lib.dsmil_forward_bags_train_workspace_bytes(P.ref, c_N, LIMIT),
             lib.dsmil_forward_bags_workspace_bytes(P.ref, c_N, LIMIT))
    _need(rows * (4 * (2 * KQ + 2 * case.C) + 48) + ws + (1 << 30), case.name)
    xs = [FW._t(b.X) for b in FW.bags(case)]
    lay = Layout(case.Ns, LIMIT)
    assert lay.total * KQ > 1 << 32
    outs = {}
    for train in (True, False):
        o, crit = _forward_batch(lib, P, xs, lay, case, train)
        form = "train" if train else "eval"
        _check_period(f"{case.name} {form}", o, crit, lay)
        outs[form] = _first_outs(o, crit, lay, case.Ns)
        del o, crit
    FW.check_forms(case.name, case, p, outs)
    _report(case.name, t0)


@pytest.mark.gpu
def test_one_bag_of_2_24_plus_129_rows():
    """One contiguous bag of 2^24 + 129 rows at D = 128, C = 2: a block of R rows repeated, with each class's critical
    row planted past 2^24 (odd rows: a float would round them).  crit must name those rows exactly, and every row
    gives the classes, Q and A bits of the same row one block earlier."""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    D, Cc, R = 128, 2, 4099
    _need(BIG_N * 4 * (D + 2 * KQ + KQ + 4 * Cc) + (1 << 30), "the 2^24 + 129 row bag")
    lib = _lib_load()
    case = FW.Case("big_bag_tc_d128_c2", "single", D, Cc, (R,))
    p = FW.make_params(case)
    P = FW._pack(p)
    block = orc.synthetic_bag(R, D, 4242, "uniform")
    block[:, [FW.D0, FW.D1, FW.D2, 3]] = 0.0
    x = FW._t(block).repeat(-(-BIG_N // R), 1)[:BIG_N].contiguous()
    crit_rows = [(1 << 24) + 65, (1 << 24) + 127]
    for k, r in enumerate(crit_rows):
        x[r, FW.D0 if k == 0 else 3] = 8.0
    # the rows from two blocks before 2^24 to the end, but the planted rows and the rows one block after them
    tail = torch.arange((1 << 24) - 2 * R, BIG_N, device="cuda")
    tail = tail[~torch.isin(tail, torch.tensor(crit_rows + [r + R for r in crit_rows], device="cuda"))]
    ws = FW._ws(lib.dsmil_forward_workspace_bytes(P.ref, BIG_N))
    for train in (True, False):
        o, crit = FW._new_outs(BIG_N, 1, case, saves=train)
        rc = lib.dsmil_forward(P.ref, x.data_ptr(), None, BIG_N, *[FW._ptr(o[k]) for k in ("classes", "pred", "A", "B")],
                               crit.data_ptr(), FW._ptr(o.get("Q")), FW._ptr(o.get("H1")), None, ws.data_ptr(),
                               ws.numel(), FW._stream())
        torch.cuda.synchronize()
        assert rc == 0, lib.dsmil_last_error()
        assert FW._np(crit).reshape(-1).tolist() == crit_rows, FW._np(crit)
        for k in ("classes", "A", "Q", "H1"):
            if o.get(k) is not None:
                same_bits(f"big bag {k}", o[k][tail], tail - R, ref=o[k])
        assert not torch.isnan(o["A"]).any() and not torch.isnan(o["B"]).any() and not torch.isnan(o["pred"]).any()
        del o
    _report("big bag", t0)


VALUE_CASE = FW.Case("limit_value_d128_c2", "value", 128, 2, PATTERN, passing_v=True)


@pytest.mark.gpu
def test_value_forward_and_backward_of_65535_bags():
    """dsmil_value_forward_bags with saves and without, then dsmil_value_backward_bags with d_A, d_B and gX, at
    nb = 65 535 (passing_v, k_qmlp_sm90 phase 1)."""
    case = VALUE_CASE
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    lib = _lib_load()
    p = FW.make_params(case)
    P = FW._pack(p)
    Ns = cycle(case.Ns, LIMIT)
    rows, (_, c_N) = sum(Ns), _bag_ptrs([None], Ns)
    fws = lib.dsmil_value_forward_bags_workspace_bytes(P.ref, c_N, LIMIT)
    bws = lib.dsmil_value_backward_bags_workspace_bytes(P.ref, c_N, LIMIT, 1)
    assert fws > 0 and bws > 0
    _need(rows * 4 * (2 * KQ + 2 * case.D + 8 * case.C) + max(fws, bws) + rows * 48, case.name)
    pats = FW.bags(case)
    xs = [FW._t(b.X) for b in pats]
    lay = Layout(case.Ns, LIMIT)
    c_X, c_N = _bag_ptrs(xs, lay.Ns)
    ws = FW._ws(fws)
    outs, keep = {}, None
    for form in ("train", "eval"):
        o, crit = FW._new_outs(lay.total, LIMIT, case, saves=form == "train")
        rc = lib.dsmil_value_forward_bags(P.ref, c_X, None, c_N, LIMIT, *[FW._ptr(o[k]) for k in ("classes", "pred", "A",
                                                                                               "B")],
                                          crit.data_ptr(), FW._ptr(o.get("Q")), FW._ptr(o.get("H1")), FW._ptr(o.get("V")),
                                          ws.data_ptr(), ws.numel(), FW._stream())
        torch.cuda.synchronize()
        assert rc == 0, lib.dsmil_last_error()
        _check_period(f"{case.name} {form}", o, crit, lay)
        outs[form] = _first_outs(o, crit, lay, case.Ns, saves=("Q", "H1", "V"))
        if form == "train":
            keep = (o, crit)
    del ws
    FW.check_forms(case.name, case, p, outs)
    o, crit = keep
    ups = upstream(case)
    pat = lambda i: torch.from_numpy(np.concatenate([u[i] for u in ups])).cuda()
    dc = pat(0)[lay.row_src] * lay.row_sign[:, None]
    dA = pat(2)[lay.row_src] * lay.row_sign[:, None]
    dp = torch.from_numpy(np.stack([u[1] for u in ups])).cuda()[lay.bag_src] * lay.bag_sign[:, None]
    dB = torch.from_numpy(np.stack([u[3] for u in ups])).cuda()[lay.bag_src] * lay.bag_sign[:, None, None]
    bcase = BW.Case(case.name, "bags", case.D, case.C, tuple(case.Ns), passing_v=True)
    g = BW._Grads(bcase, lay.total)
    G = g.struct()
    ws = FW._ws(bws)
    rc = lib.dsmil_value_backward_bags(P.ref, c_X, None, c_N, LIMIT, FW._ptr(o["Q"]), FW._ptr(o["H1"]), FW._ptr(o["V"]),
                                       FW._ptr(o["A"]), FW._ptr(o["B"]), crit.data_ptr(), dc.data_ptr(), dp.data_ptr(),
                                       dA.data_ptr(), dB.data_ptr(), None, C.byref(G), ws.data_ptr(), ws.numel(),
                                       FW._stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.dsmil_last_error()
    del ws, dc, dA
    same_bits(f"{case.name} gX", g.gX, lay.row_src, sign=lay.row_sign)
    _check_backward(case, bcase, p, pats, _first_outs(o, crit, lay, case.Ns, saves=("Q", "H1", "V")), ups, g, lay, t0)


def dev_backward_limit(lib, P, pre, max_rows):
    """The largest nb the capture-safe backward takes (its workspace size is 0 past it)."""
    f = getattr(lib, pre + "backward_bags_dev_workspace_bytes")
    lo, hi = 1, LIMIT
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if f(P.ref, mid, max_rows) > 0 else (lo, mid - 1)
    return lo


@pytest.mark.parametrize("D,C_", [(512, 2), (166, 5), (1024, 4)])
def test_capture_safe_backward_refuses_a_chunk_grid_past_65535(D, C_):
    """The dev backward's ragged GEMMs launch one CTA per chunk of the capacity in one grid dimension: near
    nb = 65 535 that passes 65 535, and the call refuses the batch (workspace 0, DSMIL_ERR_ARG) before any launch."""
    from dsmil_wsi_b200 import _lib
    from test_shard_bags_train_cpu import FAKE, params
    lib = _lib.load()
    p = params(D, C_)
    P = type("P", (), {"ref": C.byref(p)})
    pre = "dsmil_" if lib.dsmil_shard_bags_supported(C.byref(p)) else "dsmil_generic_"
    nb = dev_backward_limit(lib, P, pre, 300)
    assert 65000 < nb < LIMIT
    f = getattr(lib, pre + "backward_bags_dev_workspace_bytes")
    assert f(C.byref(p), nb + 1, 300) == 0 and f(C.byref(p), LIMIT, 300) == 0
    grads = _lib.DsmilGrads(*[FAKE] * 10, None)
    rc = getattr(lib, pre + "backward_bags_dev")(C.byref(p), FAKE, FAKE, LIMIT, 300, FAKE, FAKE, FAKE, FAKE, FAKE,
                                                 FAKE, FAKE, None, None, C.byref(grads), FAKE, FAKE, 1 << 40, None)
    assert rc == -1 and b"chunk capacity" in lib.dsmil_last_error()


DEV_CASES = [FW.Case("dev_tc_d512_c2", "bags", 512, 2, PATTERN), FW.Case("dev_gen_d166_c5", "bags", 166, 5, PATTERN)]


@pytest.mark.gpu
@pytest.mark.parametrize("max_rows", [max(PATTERN), 320], ids=["full", "short"])
@pytest.mark.parametrize("case", DEV_CASES, ids=lambda c: c.name)
def test_capture_safe_pair_at_65535_bags_gives_the_eager_bits(case, max_rows):
    """The capture-safe forward (training and eval) and backward at their largest batch, nb = 65 535, with the row
    capacity filled by the largest bag or 84 rows past it: dsmil_forward_bags[_train]_dev / dsmil_backward_bags_dev on
    the tensor-core shape, their dsmil_generic_* twins on the generic one.  Every output and gradient must be the bits
    of the eager calls on the same bags, which the test above holds to the conditioned checks."""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    lib = _lib_load()
    p = FW.make_params(case)
    P = FW._pack(p)
    pre = "dsmil_" if lib.dsmil_shard_bags_supported(P.ref) else "dsmil_generic_"
    assert (pre == "dsmil_") == (case.attend == "b"), case.name
    nb = LIMIT
    Ns = cycle(case.Ns, nb)
    rows, (_, c_N) = sum(Ns), _bag_ptrs([None], Ns)
    sizes = [lib.dsmil_forward_bags_train_workspace_bytes(P.ref, c_N, nb),
             lib.dsmil_forward_bags_workspace_bytes(P.ref, c_N, nb),
             lib.dsmil_backward_bags_workspace_bytes(P.ref, c_N, nb, 0)]
    dev_sizes = [getattr(lib, pre + n + "_workspace_bytes")(P.ref, nb, max_rows)
                 for n in ("forward_bags_train_dev", "forward_bags_dev")] + [
        getattr(lib, pre + "backward_bags_dev_workspace_bytes")(P.ref, nb - 1000, max_rows)]
    assert min(dev_sizes) > 0
    _need(rows * 4 * (2 * KQ + 4 * case.C) + nb * max_rows * 4 * (2 * KQ + 4 * case.C) + max(sizes + dev_sizes)
          + rows * 48, f"{case.name} max_rows={max_rows}")
    xs = [FW._t(b.X) for b in FW.bags(case)]
    lay = Layout(case.Ns, nb)
    xd = torch.tensor([xs[b % P_BAGS].data_ptr() for b in range(nb)], dtype=torch.int64, device="cuda")
    Nd = torch.tensor(lay.Ns, dtype=torch.int64, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    r = lay.total
    saved = {}
    for train in (False, True):
        ref, ref_crit = _forward_batch(lib, P, xs, lay, case, train)
        o, crit = FW._new_outs(nb * max_rows, nb, case, saves=train)
        name = pre + ("forward_bags_train_dev" if train else "forward_bags_dev")
        ws = FW._ws(getattr(lib, name + "_workspace_bytes")(P.ref, nb, max_rows))
        saves = [FW._ptr(o["Q"]), FW._ptr(o["H1"])] if train else []
        rc = getattr(lib, name)(P.ref, xd.data_ptr(), Nd.data_ptr(), nb, max_rows,
                                *[FW._ptr(o[k]) for k in ("classes", "pred", "A", "B")], crit.data_ptr(), *saves,
                                status.data_ptr(), ws.data_ptr(), ws.numel(), FW._stream())
        torch.cuda.synchronize()
        del ws
        assert rc == 0 and int(status) == 0, (lib.dsmil_last_error(), int(status))
        for k in ("classes", "A", "Q", "H1"):
            if o.get(k) is not None:
                assert torch.equal(o[k][:r].view(torch.int32), ref[k].view(torch.int32)), (case.name, name, k)
        for k in ("pred", "B"):
            assert torch.equal(o[k].view(torch.int32), ref[k].view(torch.int32)), (case.name, name, k)
        assert torch.equal(crit, ref_crit), (case.name, name)
        if train:
            saved = dict(eager=(ref, ref_crit), dev=(o, crit))
        del ref, ref_crit
    # the backward through classes and pred (the dev form takes no d_A, d_B or gX), eager against capture-safe
    # the dev backward refuses nb = 65 535 (its chunk grid would pass 65 535) and runs at the largest nb it takes, on
    # the first nb_b bags of the same saves
    assert getattr(lib, pre + "backward_bags_dev_workspace_bytes")(P.ref, nb, max_rows) == 0
    nb = nb_b = dev_backward_limit(lib, P, pre, max_rows)
    assert 65000 < nb_b < LIMIT
    r = sum(lay.Ns[:nb_b])
    ups = upstream(case)
    dc = (torch.from_numpy(np.concatenate([u[0] for u in ups])).cuda()[lay.row_src] * lay.row_sign[:, None])[:r]
    dp = (torch.from_numpy(np.stack([u[1] for u in ups])).cuda()[lay.bag_src] * lay.bag_sign[:, None])[:nb_b]
    bcase = BW.Case(case.name, "dev", case.D, case.C, tuple(case.Ns))
    (o, crit), (od, critd) = saved["eager"], saved["dev"]
    g_e, g_d = BW._Grads(bcase), BW._Grads(bcase)
    G = g_e.struct()
    c_X, c_N = _bag_ptrs(xs, lay.Ns[:nb_b])
    ws = FW._ws(sizes[2])
    rc = lib.dsmil_backward_bags(P.ref, c_X, c_N, nb, FW._ptr(o["Q"]), FW._ptr(o["H1"]), FW._ptr(o["A"]),
                                 FW._ptr(o["B"]), crit.data_ptr(), dc.data_ptr(), dp.data_ptr(), None, None,
                                 C.byref(G), ws.data_ptr(), ws.numel(), FW._stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.dsmil_last_error()
    del ws
    dcd = torch.full((nb * max_rows, case.C), 1.0e4, device="cuda")
    dcd[:r] = dc
    Gd = g_d.struct()
    ws = FW._ws(getattr(lib, pre + "backward_bags_dev_workspace_bytes")(P.ref, nb_b, max_rows))
    rc = getattr(lib, pre + "backward_bags_dev")(P.ref, xd.data_ptr(), Nd.data_ptr(), nb, max_rows, FW._ptr(od["Q"]),
                                                 FW._ptr(od["H1"]), FW._ptr(od["A"]), FW._ptr(od["B"]), critd.data_ptr(),
                                                 dcd.data_ptr(), dp.data_ptr(), None, None, C.byref(Gd),
                                                 status.data_ptr(), ws.data_ptr(), ws.numel(), FW._stream())
    torch.cuda.synchronize()
    assert rc == 0 and int(status) == 0, (lib.dsmil_last_error(), int(status))
    for k, t in g_e.t.items():
        assert not torch.isnan(t).any(), (case.name, k)
        assert torch.equal(t.view(torch.int32), g_d.t[k].view(torch.int32)), (case.name, "backward", k)
    _report(f"{case.name} max_rows={max_rows}", t0)
