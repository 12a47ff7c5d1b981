"""The batched forward of models with a value network (passing_v: dsmil_value_forward_bags, MILNet.forward_bags).

Every bag's outputs and saved activations must be bit for bit what dsmil_forward / milnet(x) gives that bag alone, on
ragged batches whose bags straddle the 128-row tiles, in eval mode and with v's dropout mask, on shapes whose phase 1 is
k_qmlp_sm90 (nonlinear q, D % 128 == 0) and on the FFMA ones; and within the fp64 oracle's tolerances.  A batch costs
the same launches whatever its size."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import build_net
from oracle import dsmil_oracle as orc
from test_gpu_parity import _check_forward, _np

pytestmark = pytest.mark.gpu

# (D, C, nonlinear): k_qmlp_sm90 phase 1; FFMA at D = 166; a linear q; C = 6; a small D
SHAPES = [(512, 2, True), (166, 1, True), (512, 3, False), (1024, 6, True), (96, 2, True)]
NS = [1, 127, 128, 129, 2049, 10000]
DROPOUT_V = 0.25


@pytest.fixture(scope="module")
def lib():
    from dsmil_wsi_b200 import _lib
    return _lib.load()


def _params(D, C_, nonlinear, seed=7):
    p = orc.random_params(D, C_, seed + D + C_, nonlinear=nonlinear, passing_v=True)
    # every pre-activation of v's ReLU about 3 away from 0 (as tests/test_forward_routes_gpu.py): a gate within fp32
    # rounding of 0 could open in the kernels and stay shut in the fp64 oracle
    p.bv = np.where(np.arange(D) % 2 == 0, 3.0, -3.0).astype(np.float32)
    return p


def _bags(D, Ns, seed, offset):
    """Bags on the device; offset > 0 places each at `offset` floats into its own buffer (4-byte-aligned views)."""
    out = []
    for i, n in enumerate(Ns):
        X = torch.from_numpy(orc.synthetic_bag(n, D, seed + i, "uniform")).cuda()
        if offset:
            buf = torch.empty(n * D + offset, device="cuda")
            buf[offset:].copy_(X.reshape(-1))
            X = buf[offset:].view(n, D)
        out.append(X)
    return out


def _masks(xs, seed):
    torch.manual_seed(seed)
    return [torch.nn.functional.dropout(torch.ones_like(x), DROPOUT_V, True) for x in xs]


def _pack(net):
    from dsmil_wsi_b200 import functional as Fn
    from dsmil_wsi_b200.sharded import milnet_params
    return Fn.ParamPack(*milnet_params(net))


def _value_call(lib, P, xs, vs, saves, forward_bags=False):
    """dsmil_value_forward_bags, or with forward_bags dsmil_forward_bags (value inputs = the features, no saves)."""
    nb, Ns = len(xs), [int(x.shape[0]) for x in xs]
    total, Cc, D = sum(Ns), P.C, P.D
    new = lambda *s: torch.full(s, float("nan"), device="cuda")
    out = dict(classes=new(total, Cc), pred=new(nb, Cc), A=new(total, Cc), B=new(nb, Cc, D),
               crit=torch.full((nb, Cc), -7, dtype=torch.int64, device="cuda"))
    if saves:
        out.update(Q=new(total, 128), H1=new(total, 128) if P.nonlinear else None, V=new(total, D))
    c_N = (C.c_int64 * nb)(*Ns)
    c_X = (C.c_void_p * nb)(*[x.data_ptr() for x in xs])
    c_V = None if vs is None else (C.c_void_p * nb)(*[v.data_ptr() for v in vs])
    size = lib.dsmil_forward_bags_workspace_bytes if forward_bags else lib.dsmil_value_forward_bags_workspace_bytes
    ws = torch.empty(max(size(P.ref, c_N, nb), 256), dtype=torch.uint8, device="cuda")
    g = lambda k: None if out.get(k) is None else out[k].data_ptr()
    if forward_bags:
        rc = lib.dsmil_forward_bags(P.ref, c_X, c_N, nb, g("classes"), g("pred"), g("A"), g("B"), g("crit"),
                                    ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
        assert rc == 0, lib.dsmil_last_error()
        return out
    rc = lib.dsmil_value_forward_bags(P.ref, c_X, c_V, c_N, nb, g("classes"), g("pred"), g("A"), g("B"), g("crit"),
                                      g("Q"), g("H1"), g("V"), ws.data_ptr(), ws.numel(),
                                      torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.dsmil_last_error()
    return out


def _single_call(lib, P, x, v):
    N, Cc, D = int(x.shape[0]), P.C, P.D
    new = lambda *s: torch.full(s, float("nan"), device="cuda")
    out = dict(classes=new(N, Cc), pred=new(1, Cc), A=new(N, Cc), B=new(1, Cc, D),
               crit=torch.full((Cc,), -7, dtype=torch.int64, device="cuda"), Q=new(N, 128),
               H1=new(N, 128) if P.nonlinear else None, V=new(N, D))
    ws = torch.empty(max(lib.dsmil_forward_workspace_bytes(P.ref, N), 256), dtype=torch.uint8, device="cuda")
    g = lambda k: None if out.get(k) is None else out[k].data_ptr()
    rc = lib.dsmil_forward(P.ref, x.data_ptr(), None if v is None else v.data_ptr(), N, g("classes"), g("pred"), g("A"),
                           g("B"), g("crit"), g("Q"), g("H1"), g("V"), ws.data_ptr(), ws.numel(),
                           torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.dsmil_last_error()
    return out


# bags 1 float off a 16-byte boundary: at (512, 2) the batch loops dsmil_forward (k_qmlp_sm90 needs aligned bags); at
# (512, 3, linear) and (96, 2) k_vproj_b reads them through its scalar path although D % 4 == 0; at 166 every row is
# off.  Mode "bags": eval through dsmil_forward_bags, which takes passing_v on the same route.
OFFSETS = {(512, 2): (0, 1), (166, 1): (1,), (512, 3): (0, 1), (1024, 6): (0,), (96, 2): (0, 1)}


def _cases():
    for D, C_, nl in SHAPES:
        for off in OFFSETS[(D, C_)]:
            for mode in ("eval", "train") + (("bags",) if (D, C_) == (512, 2) else ()):
                yield pytest.param(D, C_, nl, off, mode, id=f"D{D}C{C_}{'nl' if nl else 'lin'}-off{off}-{mode}")


@pytest.mark.parametrize("D,C_,nl,offset,mode", list(_cases()))
def test_every_bag_gets_its_single_bag_bits(lib, D, C_, nl, offset, mode):
    p = _params(D, C_, nl)
    net = build_net(p)
    P = _pack(net)
    xs = _bags(D, NS, 100 + D, offset)
    masks = _masks(xs, 5) if mode == "train" else None
    vs = [x * m for x, m in zip(xs, masks)] if masks else None
    with torch.no_grad():
        batch = _value_call(lib, P, xs, vs, saves=True)
        again = _value_call(lib, P, xs, vs, saves=True)
        infer = _value_call(lib, P, xs, vs, saves=False)
        if mode == "bags":
            fb = _value_call(lib, P, xs, None, saves=False, forward_bags=True)
    torch.cuda.synchronize()
    if mode == "bags":
        for k, t in fb.items():
            assert torch.equal(t, infer[k]), ("dsmil_forward_bags", k)
    for k, t in batch.items():
        if t is not None:
            assert torch.equal(t, again[k]), ("run to run", k)
            if k in infer:
                assert torch.equal(t, infer[k]), ("saves change nothing", k)
    row = 0
    for b, x in enumerate(xs):
        n = int(x.shape[0])
        one = _single_call(lib, P, x, vs[b] if vs else None)
        for k in ("classes", "A", "Q", "H1", "V"):
            if one[k] is not None:
                assert torch.equal(batch[k][row:row + n], one[k]), (b, n, k)
        for k in ("pred", "B", "crit"):
            assert torch.equal(batch[k][b], one[k].reshape(batch[k][b].shape)), (b, n, k)
        t = orc.forward(_np(x), p, v_mask=None if masks is None else _np(masks[b]))
        _check_forward((batch["classes"][row:row + n], batch["pred"][b:b + 1], batch["A"][row:row + n],
                        batch["B"][b:b + 1]), t.classes, t.prediction_bag, t.A, t.B, t.idx, p, None, f"bag {b} N={n}")
        row += n


@pytest.mark.parametrize("D,C_,nl", [SHAPES[0], SHAPES[1], SHAPES[2]])
@pytest.mark.parametrize("mode", ["eval", "train"])
def test_forward_bags_equals_the_per_bag_forward(D, C_, nl, mode):
    p = _params(D, C_, nl)
    net = build_net(p, dropout_v=DROPOUT_V)
    net.train(mode == "train")
    xs = _bags(D, [129, 1, 2049, 128], 300 + D, 0)
    with torch.no_grad():
        torch.manual_seed(11)
        outs = net.forward_bags(xs)
        after_batch = torch.rand(4, device="cuda")
        torch.manual_seed(11)
        singles = [net(x) for x in xs]
        after_loop = torch.rand(4, device="cuda")
    assert len(outs) == len(xs)
    assert torch.equal(after_batch, after_loop)          # the same RNG draws as the per-bag loop
    for b, (o, s) in enumerate(zip(outs, singles)):
        for u, v in zip(o, s):
            assert u.shape == v.shape and torch.equal(u, v), (b, mode)


def test_launches_do_not_grow_with_the_batch(lib):
    p = _params(512, 2, True)
    net = build_net(p).eval()
    bags = _bags(512, [1000 + 37 * i for i in range(16)], 900, 0)

    def launches(xs):
        with torch.no_grad():
            torch.cuda.synchronize()
            n0 = lib.dsmil_launch_count()
            net.forward_bags(xs)
            torch.cuda.synchronize()
            return lib.dsmil_launch_count() - n0

    launches(bags)                                       # warm
    n2, n16 = launches(bags[:2]), launches(bags)
    with torch.no_grad():
        n0 = lib.dsmil_launch_count()
        for x in bags:
            net(x)
        loop = lib.dsmil_launch_count() - n0
    assert n2 == n16, (n2, n16)
    assert n16 < loop / 8, (n16, loop)


@pytest.mark.parametrize("mode", ["eval", "train"])
def test_forward_bags_grad_keeps_the_per_bag_autograd(mode):
    """grad=True gives the outputs and parameter gradients of the per-bag loop bit for bit (v's masks drawn alike)."""
    p = _params(166, 1, True)
    net = build_net(p, dropout_v=DROPOUT_V)
    net.train(mode == "train")
    xs = _bags(166, [50, 300, 129], 1200, 0)
    y = torch.ones(1, 1, device="cuda")

    def step(fn):
        net.zero_grad(set_to_none=True)
        torch.manual_seed(21)
        outs = fn()
        loss = sum(torch.nn.functional.binary_cross_entropy_with_logits(o[1], y) + o[0].max() for o in outs)
        loss.backward()
        return [t.detach().clone() for o in outs for t in o], \
            {k: v.grad.clone() for k, v in net.named_parameters() if v.grad is not None}

    outs_b, grads_b = step(lambda: net.forward_bags(xs, grad=True))
    outs_l, grads_l = step(lambda: [net(x) for x in xs])
    assert all(torch.equal(u, v) for u, v in zip(outs_b, outs_l))
    assert grads_b.keys() == grads_l.keys() and "b_classifier.v.1.weight" in grads_b
    for k in grads_b:
        assert torch.equal(grads_b[k], grads_l[k]), k


def test_more_bags_than_one_call_takes():
    """65 537 bags: two library calls into one packed result, each bag still its single-bag bits."""
    from dsmil_wsi_b200 import functional as Fn
    p = _params(96, 2, True)
    net = build_net(p).eval()
    nb = Fn.MAX_VALUE_BAGS + 2
    Ns = [1 + (i % 3) for i in range(nb)]
    big = torch.rand(sum(Ns), 96, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    xs = list(big.split(Ns))
    with torch.no_grad():
        outs = net.forward_bags(xs)
        assert len(outs) == nb
        for b in (0, 1, Fn.MAX_VALUE_BAGS - 1, Fn.MAX_VALUE_BAGS, nb - 1):
            for u, v in zip(outs[b], net(xs[b])):
                assert u.shape == v.shape and torch.equal(u, v), b
