"""The batched backward of a model with a value network (passing_v: dsmil_value_backward_bags, and
functional.mil_forward_value_bags(grad=True) over it).

The conditioned check of tests/test_conditioned_backward_gpu.py, on this route: each case runs
dsmil_value_forward_bags with saves, copies A, B, Q, H1, V and crit_idx to the host, and runs `orc.backward` in fp64
per bag on exactly what the backward kernels receive, summed over the bags; with the same bars (q.* and gX row by row
1e-4, Wi, bi, Wf, bf, Wv, bv 2e-5) and the same probes (each run again with the saved A moved onto the rows at the
edges of every split and chunk, the gWv chunks of the value inputs included).  The autograd function against the
per-bag autograd of mil_forward; the same bits on a second run; one launch per stage whatever the batch size; and every
kernel the route launches is one of the library's table (tests/test_kernel_instances_gpu.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import rel_to_max
from oracle import dsmil_oracle as orc
from test_conditioned_backward_gpu import (KQ, Case, _bag_tensor, _check, _Grads, _host_bags, _nan, _np,
                                           _oracle_crit, _pack, _ptr, _saves_and_reference, _stream, _t, _unpack,
                                           _ws, probe_mask, upstream)
from test_dense_upstream_grads_gpu import rag_rows_per_chunk, rowwise_err

pytestmark = pytest.mark.gpu

CASES = [
    Case("value_tc_d512_c2", "bags", 512, 2, (64, 63, 65, 1, 128, 129, 127, 2049), passing_v=True),
    Case("value_gen_d166_c1_mask", "bags", 166, 1, (128, 127, 129, 1, 3000), passing_v=True, masked=True),
    Case("value_linear_d230_c3", "bags", 230, 3, (128, 127, 129, 1, 2305), nonlinear=False, passing_v=True),
    Case("value_d96_c5_mask", "bags", 96, 5, (64, 129, 1, 4097), passing_v=True, masked=True),
    Case("value_tc_d512_misaligned", "bags", 512, 2, (128, 127, 129, 1, 5319), passing_v=True, misaligned=(4,)),
    Case("value_tc_d512_n1_to_10000", "bags", 512, 2, (1, 10000, 777, 2), passing_v=True, masked=True),
]


def value_probes(case: Case):
    """probe_mask's rows of the identity-v batch, plus the first and last row of every gWv chunk of the value inputs
    (rag_rows_per_chunk(D, D, .) rows, never straddling a bag)."""
    mask = probe_mask(case)
    Ns = list(case.Ns)
    rps = rag_rows_per_chunk(case.D, case.D, sum(Ns), False)
    row = 0
    for n in Ns:
        for r0 in range(0, n, rps):
            mask[row + r0] = mask[row + min(n, r0 + rps) - 1] = True
        row += n
    return mask


def _arrays(ts):
    return None if ts is None else (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def run_value_bags(case: Case, probes_on: bool):
    from dsmil_wsi_b200 import _lib
    lib = _lib.load()
    p = case.params()
    P = _pack(p)
    Xs = case.bags()
    Ns = list(case.Ns)
    nb, total, Cc, D = len(Ns), sum(Ns), case.C, case.D
    xs = [_bag_tensor(X, b in case.misaligned) for b, X in enumerate(Xs)]
    vms = case.v_masks()
    ms = [_t(m) for m in vms] if case.masked else None
    vs = [x * m for x, m in zip(xs, ms)] if ms else None
    mask = torch.cat(ms) if ms else None                # packed [sum N, D], as gX
    c_X, c_V, c_N = _arrays(xs), _arrays(vs), (C.c_int64 * nb)(*Ns)
    o = dict(classes=_nan(total, Cc), pred=_nan(nb, Cc), A=_nan(total, Cc), B=_nan(nb, Cc, D), Q=_nan(total, KQ),
             H1=_nan(total, KQ) if case.nonlinear else None, V=_nan(total, D))
    crit = torch.full((nb, Cc), -7, dtype=torch.int64, device="cuda")
    ws = _ws(lib.dsmil_value_forward_bags_workspace_bytes(P.ref, c_N, nb))
    rc = lib.dsmil_value_forward_bags(P.ref, c_X, c_V, c_N, nb, *[_ptr(o[k]) for k in ("classes", "pred", "A", "B")],
                                      crit.data_ptr(), _ptr(o["Q"]), _ptr(o["H1"]), _ptr(o["V"]), ws.data_ptr(),
                                      ws.numel(), _stream())
    assert rc == 0, lib.dsmil_last_error()
    crit_h = _np(crit)
    for b, X in enumerate(Xs):
        assert np.array_equal(crit_h[b], _oracle_crit(X, p)), (case.name, b)
    host = _host_bags(o, Ns, 0, 0)
    for h, V in zip(host, _unpack(_np(o["V"]), Ns)):
        h["V"] = V
    probes = value_probes(case)
    ups = upstream(case, probes, True)
    A_new, want, gX_want = _saves_and_reference(case, p, Xs, host, probes if probes_on else None, ups, list(crit_h),
                                                vms, True)
    o["A"].copy_(torch.from_numpy(np.concatenate(A_new)))
    dc, dA = (_t(np.concatenate([u[i] for u in ups])) for i in (0, 2))
    dp, dB = (_t(np.stack([u[i] for u in ups])) for i in (1, 3))
    g = _Grads(case, total)
    G = g.struct()
    ws = _ws(lib.dsmil_value_backward_bags_workspace_bytes(P.ref, c_N, nb, 1))
    rc = lib.dsmil_value_backward_bags(P.ref, c_X, c_V, c_N, nb, _ptr(o["Q"]), _ptr(o["H1"]), _ptr(o["V"]),
                                       _ptr(o["A"]), _ptr(o["B"]), crit.data_ptr(), _ptr(dc), _ptr(dp), _ptr(dA),
                                       _ptr(dB), _ptr(mask), C.byref(G), ws.data_ptr(), ws.numel(), _stream())
    assert rc == 0, lib.dsmil_last_error()
    torch.cuda.synchronize()
    _check(case, "probes" if probes_on else "plain", g.host(), want, [_np(t) for t in _unpack(g.gX, Ns)], gX_want)


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
@pytest.mark.parametrize("probes_on", [False, True], ids=["plain", "probes"])
def test_value_backward_bags_against_the_fp64_backward_on_its_own_saves(case, probes_on):
    run_value_bags(case, probes_on)


# ------------------------------------------------------------------------------------------- the autograd function
NAMES = ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf")


def _torch_params(D, C_, nonlinear, seed):
    p = orc.random_params(D, C_, seed, nonlinear=nonlinear, passing_v=True, scale=1.5)
    return [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda().requires_grad_()
            for a in (p.Wi, p.bi, p.W1, p.b1, p.W2, p.b2, p.Wv, p.bv, p.Wf, p.bf)]


def _loss_terms(Ns, C_, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
    total, nb = sum(Ns), len(Ns)
    return 1.0 + rn(total, C_), rn(nb, C_), rn(total, C_), 1e-2 * rn(nb, C_, D)


def _loss(classes, pred, A, B, w):
    wc, wp, wa, wb = w
    return (classes * wc).sum() + (pred * wp).sum() + (A * wa).sum() + (B * wb).sum()


def _batched_step(xs, params, vs, ms, w):
    from dsmil_wsi_b200 import functional as Fn
    bags = [x.detach().requires_grad_() for x in xs]
    outs, _ = Fn.mil_forward_value_bags(bags, params, vs, grad=True, v_masks=ms)
    classes, pred, A, B = outs.packed
    for t in params:
        if t is not None:
            t.grad = None
    _loss(classes, pred, A, B, w).backward()
    return (classes, pred, A, B), {n: t.grad.clone() for n, t in zip(NAMES, params) if t is not None}, \
        torch.cat([b.grad for b in bags])


def _per_bag_step(xs, params, vs, ms, w):
    from dsmil_wsi_b200 import functional as Fn
    bags = [x.detach().requires_grad_() for x in xs]
    for t in params:
        if t is not None:
            t.grad = None
    outs = []
    for b, x in enumerate(bags):
        classes, pred, A, B, _ = Fn.mil_forward(x, params, v_input=None if vs is None else vs[b],
                                                v_mask=None if ms is None else ms[b])
        outs.append((classes, pred, A, B))
    packed = tuple(torch.cat([o[i] for o in outs]) for i in range(4))
    _loss(*packed, w).backward()
    return packed, {n: t.grad.clone() for n, t in zip(NAMES, params) if t is not None}, \
        torch.cat([b.grad for b in bags])


STEPS = [(512, 2, True, 0.0), (512, 2, True, 0.2), (166, 1, True, 0.2), (230, 3, False, 0.0)]


@pytest.mark.parametrize("D,C_,nonlinear,p_drop", STEPS)
def test_autograd_step_matches_the_per_bag_autograd(D, C_, nonlinear, p_drop):
    """The same forward bits as mil_forward bag by bag (on the same value inputs), gradients within the conditioned
    bars of the per-bag backward's, and the same gradient bits on a second run."""
    Ns = [1, 127, 128, 129, 2049, 3]
    xs = [torch.from_numpy(orc.synthetic_bag(n, D, 40 + i)).cuda() for i, n in enumerate(Ns)]
    params = _torch_params(D, C_, nonlinear, 11 + D)
    ms = vs = None
    if p_drop > 0:
        torch.manual_seed(3)
        ms = [torch.nn.functional.dropout(torch.ones_like(x), p_drop, True) for x in xs]
        vs = [x * m for x, m in zip(xs, ms)]
    w = _loss_terms(Ns, C_, D, 9)
    out_b, g_b, gx_b = _batched_step(xs, params, vs, ms, w)
    out_p, g_p, gx_p = _per_bag_step(xs, params, vs, ms, w)
    for a, b in zip(out_b, out_p):
        assert torch.equal(a, b)
    for n in g_b:
        bar = 1e-4 if n in ("W1", "b1", "W2", "b2") else 2e-5
        assert rel_to_max(_np(g_b[n]), _np(g_p[n])) <= bar, n
    assert rowwise_err(_np(gx_b), _np(gx_p)) <= 1e-4
    _, g_again, gx_again = _batched_step(xs, params, vs, ms, w)
    assert all(torch.equal(g_b[n], g_again[n]) for n in g_b) and torch.equal(gx_b, gx_again)


def test_one_launch_per_stage_and_only_kernels_of_the_table():
    from dsmil_wsi_b200 import _lib
    from test_kernel_instances_gpu import KERNELS, launched
    D, C_ = 512, 2
    params = _torch_params(D, C_, True, 5)

    def step(nb, masked):
        Ns = [100 + 37 * i for i in range(nb)]
        xs = [torch.from_numpy(orc.synthetic_bag(n, D, 70 + i)).cuda() for i, n in enumerate(Ns)]
        ms = [torch.nn.functional.dropout(torch.ones_like(x), 0.2, True) for x in xs] if masked else None
        vs = [x * m for x, m in zip(xs, ms)] if masked else None
        w = _loss_terms(Ns, C_, D, 1)
        return lambda: _batched_step(xs, params, vs, ms, w)

    for masked in (False, True):
        counts = []
        for nb in (2, 16):
            fn = step(nb, masked)
            fn()
            torch.cuda.synchronize()
            before = _lib.launch_count()
            fn()
            torch.cuda.synchronize()
            counts.append(_lib.launch_count() - before)
        assert counts[0] == counts[1], (masked, counts)
    for masked in (False, True):
        got = launched(step(4, masked))
        assert got and got <= set(KERNELS), sorted(got - set(KERNELS))
        assert {"k_linear_models<3,1>", "k_gemm_tn_rag", "k_bwd_rowdot_b"} <= got


def test_value_inputs_without_masks_are_refused_when_the_bags_need_a_gradient():
    """gX's value path multiplies by each bag's mask: without the masks it would take them as ones."""
    from dsmil_wsi_b200 import functional as Fn
    D, C_ = 96, 2
    params = _torch_params(D, C_, True, 3)
    xs = [torch.rand(n, D, device="cuda") for n in (5, 9)]
    ms = [torch.nn.functional.dropout(torch.ones_like(x), 0.2, True) for x in xs]
    vs = [x * m for x, m in zip(xs, ms)]
    bags = [x.clone().requires_grad_() for x in xs]
    with pytest.raises(ValueError, match="v_masks"):
        Fn.mil_forward_value_bags(bags, params, vs, grad=True)
    with pytest.raises(ValueError, match="v_inputs"):
        Fn.mil_forward_value_bags(xs, params, None, grad=True, v_masks=ms)
    outs, _ = Fn.mil_forward_value_bags(xs, params, vs, grad=True)       # parameter gradients only: no mask needed
    outs.packed[1].sum().backward()
    assert params[6].grad is not None and torch.isfinite(params[6].grad).all()


def test_a_value_input_written_in_place_before_the_backward_is_caught():
    from dsmil_wsi_b200 import functional as Fn
    D, C_ = 96, 2
    params = _torch_params(D, C_, True, 4)
    xs = [torch.rand(n, D, device="cuda") for n in (5, 9)]
    ms = [torch.nn.functional.dropout(torch.ones_like(x), 0.2, True) for x in xs]
    vs = [x * m for x, m in zip(xs, ms)]
    outs, _ = Fn.mil_forward_value_bags(xs, params, vs, grad=True, v_masks=ms)
    vs[1].mul_(2.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        outs.packed[1].sum().backward()
