"""dsmil_forward on shapes whose phase 1 runs on the tensor-core kernel (k_qmlp_sm90) while attend and finalize take the
generic per-bag kernels: nonlinear q with D % 128 == 0 and any of passing_v, C >= 5, C in {3, 4} with D > 1024, D > 2048.
The batched forward does not take these shapes, so this route is the only way into k_qmlp_sm90 at C >= 5 (at D != 512
that is k_qmlp_sm90<8, 0>, the instantiation without the L2 prefetch) and at D > 2048.

Each case checks the route (dsmil_forward_path, dsmil_shard_bags_supported and the profile counters: the attend and
finalize tags are shared by the generic and batch kernels, so the phase-1 tags are what tell the routes apart), the eval
outputs and a training step's outputs and gradients against the fp64 oracle at the tolerances of
tests/test_gpu_parity.py, and that forward_bags, which runs such bags one at a time, equals the per-bag forward bit for
bit."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import rel_to_max
from helpers import build_net, caller_loss, grad_name
from oracle import dsmil_oracle as orc
from test_gpu_parity import _check_forward, _np

pytestmark = pytest.mark.gpu

# (D, C, N, passing_v)
CASES = [(512, 6, 1000, False), (1024, 5, 777, False), (512, 2, 640, True), (2048, 3, 384, False),
         (2560, 1, 1500, False)]
DROPOUT_V = 0.25
Q_PARAMS = ("W1", "b1", "W2", "b2")


@pytest.fixture(params=CASES, ids=lambda c: f"D{c[0]}C{c[1]}N{c[2]}" + ("pv" if c[3] else ""))
def case(request):
    D, C, N, passing_v = request.param
    p = orc.random_params(D, C, 4000 + D + C, passing_v=passing_v)
    if passing_v:
        # v's biases keep every pre-activation of its ReLU about 3 away from 0, half the features on and half off.  A
        # gate within fp32 rounding of 0 could open in the kernels and stay shut in the fp64 oracle, which moves one
        # row's whole share of the Wv gradient (up to ~4e-3 of its largest entry at this size).
        p.bv = np.where(np.arange(D) % 2 == 0, 3.0, -3.0).astype(np.float32)
    X = orc.synthetic_bag(N, D, 4100 + N, "uniform")
    return p, X


@pytest.fixture
def lib():
    from dsmil_wsi_b200 import _lib
    return _lib.load()


def _phase1_launches(lib, fn):
    """fn()'s result and the launches it made of k_scores, the generic Q-MLP and k_qmlp_sm90 (profile tags 0, 1, 4)."""
    ms, n = (ctypes.c_double * 8)(), (ctypes.c_uint64 * 8)()
    torch.cuda.synchronize()
    lib.dsmil_profile_read(ms, n)                # drops the event pairs of earlier calls
    lib.dsmil_profile_enable(1)
    try:
        out = fn()
        torch.cuda.synchronize()
        lib.dsmil_profile_read(ms, n)
    finally:
        lib.dsmil_profile_enable(0)
    return out, (n[0], n[1], n[4])


def _assert_route(lib, net, N):
    from dsmil_wsi_b200 import functional as Fn
    from dsmil_wsi_b200.sharded import milnet_params
    P = Fn.ParamPack(*milnet_params(net))
    assert lib.dsmil_forward_path(P.ref, N) == 2, "phase 1 is not on the tensor-core kernel"
    assert lib.dsmil_shard_bags_supported(P.ref) == 0, "the shape would take the batched forward"


def test_eval_forward_phase1_tensor_core_generic_attend(case, lib):
    p, X = case
    N = X.shape[0]
    net = build_net(p).eval()
    _assert_route(lib, net, N)
    x = torch.from_numpy(X).cuda()
    with torch.no_grad():
        out, launches = _phase1_launches(lib, lambda: net(x))
        idx = net.critical_instances(x)
        k = N // 2 + 1
        bags = net.forward_bags([x, x[:k]])
        singles = [out, net(x[:k])]
    assert launches == (0, 0, 1), launches      # one k_qmlp_sm90, no k_scores and no generic Q-MLP
    t = orc.forward(X, p)
    _check_forward(out, t.classes, t.prediction_bag, t.A, t.B, t.idx, p, idx, f"D{p.D}C{p.C}N{N}")
    for b, (o, s) in enumerate(zip(bags, singles)):
        for u, v in zip(o, s):
            assert u.shape == v.shape and torch.equal(u, v), b


def test_training_step_phase1_tensor_core_generic_attend(case, lib):
    p, X = case
    N, D, C = X.shape[0], p.D, p.C
    net = build_net(p, dropout_v=DROPOUT_V if p.passing_v else 0.0).train()
    _assert_route(lib, net, N)
    torch.manual_seed(1234)
    (classes, pred, A, B), launches = _phase1_launches(lib, lambda: net(torch.from_numpy(X).cuda()))
    assert launches == (0, 0, 1), launches
    mask = None
    if p.passing_v:                              # the dropout mask inside v, drawn as the module draws it
        torch.manual_seed(1234)
        mask = _np(torch.nn.functional.dropout(torch.ones(N, D, device="cuda"), DROPOUT_V, True))
        assert 0.15 < (mask == 0).mean() < 0.35
    t = orc.forward(X, p, v_mask=mask)
    _check_forward((classes, pred, A, B), t.classes, t.prediction_bag, t.A, t.B, t.idx, p, None, "train")
    y = (np.arange(C) % 2).astype(np.float32)
    loss = caller_loss(classes, pred, torch.from_numpy(y).cuda())
    loss.backward()
    tl, d_cls, d_pred = orc.caller_loss_grads(t, y)
    assert abs(loss.item() - tl) < 3e-6
    tg = orc.backward(X, p, t, d_cls, d_pred, v_mask=mask)
    named = dict(net.named_parameters())
    for k, v in tg.items():
        # the q.* gradients pass through the softmax backward, which amplifies the 3xBF16 rounding of Q
        r = rel_to_max(_np(named[grad_name(k, True)].grad), v)
        assert r < (1e-3 if k in Q_PARAMS else 5e-5), (k, r)
