"""The fold step: M fold models, each over its own bags, in one dsmil_forward_bags_models_train call and one
dsmil_backward_bags_models call.  Every model's outputs and gradients (gX included) must be torch.equal to what its
own forward_bags(grad=True) and backward give on its own bags, under the callers' loss and under dense upstream
gradients; the fused route must make the same number of launches for every M; one fold is also held to the fp64
oracle; train_epoch_models must give each fold's standalone epoch bit for bit."""
import numpy as np
import pytest
import torch

from helpers import build_net, grad_name
from oracle import dsmil_oracle as orc
from dsmil_wsi_b200 import _lib, feed
from dsmil_wsi_b200.ensemble import forward_bags_per_model
from test_dense_upstream_grads_gpu import B_SMALL, _bag_data, _check_params, _np, _param_names, oracle_grads, \
    rowwise_err, summed

pytestmark = pytest.mark.gpu

# model m's bags: ragged lists of unequal length, with bags of 1, 127, 128, 129 and 10 000 rows
LISTS = [[129, 10_000, 1], [127], [128, 5, 3000, 1, 129], [10_000, 64], [1, 1], [300], [2000, 128, 127], [77, 4096]]


def _nets(D, C, M, seed=0, **kw):
    return [build_net(orc.random_params(D, C, seed + 101 * m, scale=2.0, **kw)).train() for m in range(M)]


def _bags(lists, D, seed, grad=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [[torch.rand(n, D, generator=g, device="cuda").requires_grad_(grad) for n in ns] for ns in lists]


def _dense(outs, seed):
    """A loss with dense upstream gradients to classes, pred, A and B of every bag (standard normal weights)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    loss = 0
    for o in outs:
        for t in o:
            loss = loss + (t * torch.randn(t.shape, generator=g, device="cuda")).sum()
    return loss


def _callers(outs, labels):
    """The minibatch training loss of every model, summed."""
    loss = 0
    for out, lab in zip(outs, labels):
        bag, mx = feed._group_predictions(out)
        loss = loss + feed.minibatch_loss(torch.nn.BCEWithLogitsLoss(), bag, mx, lab)
    return loss


def _grads(net, xs, loss):
    leaves = list(net.parameters())
    return torch.autograd.grad(loss, leaves + [x for x in xs if x.requires_grad], allow_unused=True)


def _compare(nets, lists, D, seed, loss_kind):
    bags = _bags(lists, D, seed, grad=True)
    labels = [(torch.rand(len(ns), nets[0].b_classifier.fcc.weight.shape[0], device="cuda") > 0.5).float()
              for ns in lists]
    outs, fwd = _launches(lambda: forward_bags_per_model(nets, bags, grad=True))
    # forward: each model's packed outputs against its own forward_bags(grad=True)
    for m, (net, xs, out) in enumerate(zip(nets, bags, outs)):
        ref = net.forward_bags(xs, grad=True)
        for what, u, v in zip(("classes", "pred", "A", "B"), out.packed, ref.packed):
            assert torch.equal(u, v), (m, what)
        assert torch.equal(out.crit, ref.crit), m
    # backward: one loss over all models against each model's own loss alone
    if loss_kind == "dense":
        total = sum(_dense([o for o in out], seed + 7 * m) for m, out in enumerate(outs))
    else:
        total = _callers(outs, labels)
    leaves = [p for net in nets for p in net.parameters()] + [x for xs in bags for x in xs]
    got, bwd = _launches(lambda: torch.autograd.grad(total, leaves, allow_unused=True))
    k = 0
    got_p, got_x = [], []
    for net in nets:
        n = len(list(net.parameters()))
        got_p.append(got[k:k + n])
        k += n
    for xs in bags:
        got_x.append(got[k:k + len(xs)])
        k += len(xs)
    for m, (net, xs) in enumerate(zip(nets, bags)):
        ref = net.forward_bags(xs, grad=True)
        loss = _dense(list(ref), seed + 7 * m) if loss_kind == "dense" else _callers([ref], [labels[m]])
        want = torch.autograd.grad(loss, list(net.parameters()) + list(xs), allow_unused=True)
        for (name, _), u, v in zip(net.named_parameters(), got_p[m], want):
            assert (u is None) == (v is None) and (u is None or torch.equal(u, v)), (m, name)
        for b, (u, v) in enumerate(zip(got_x[m], want[len(got_p[m]):])):
            assert torch.equal(u, v), (m, "gX", b)
    return fwd, bwd


def _launches(fn):
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    r = fn()
    torch.cuda.synchronize()
    return r, _lib.launch_count() - n0


# the fused route's launches: forward 4 (weight-image prep, phase 1, attend, finalize); backward 20 with gX (bag
# classifier; gWi, gbi; dA; dL; dq_max; dz2; gW2, gb2; dz1; gW1, gb1 -- each chunked reduction and its per-model sums;
# then gX and its extra terms), whatever M
FUSED_FWD, FUSED_BWD = 4, 20


def _supported(nets):
    return bool(_lib.load().dsmil_models_supported((_lib.DsmilParams * len(nets))(*[_pack(n).struct for n in nets]),
                                                   len(nets)))


@pytest.mark.parametrize("M", [1, 2, 5, 8])
@pytest.mark.parametrize("D,C", [(512, 2), (1024, 4), (2048, 1)])
def test_each_model_matches_its_own_step(D, C, M):
    nets = _nets(D, C, M, seed=D + C)
    # every shape here is fused, except eight members at C.D = 4096 (1024 / 4), whose Wi rows do not fit shared memory
    fused = not (D == 1024 and M == 8)
    assert _supported(nets) == fused, (D, C, M)
    fwd, bwd = _compare(nets, LISTS[:M], D, seed=M, loss_kind="callers")
    if fused:
        assert (fwd, bwd) == (FUSED_FWD, FUSED_BWD), (D, C, M, fwd, bwd)
    else:
        assert fwd > FUSED_FWD and bwd > FUSED_BWD, (D, C, M, fwd, bwd)


@pytest.mark.parametrize("M", [2, 5])
def test_dense_upstream_gradients(M):
    nets = _nets(512, 2, M, seed=40 + M)
    assert _compare(nets, LISTS[:M], 512, seed=60 + M, loss_kind="dense") == (FUSED_FWD, FUSED_BWD)


@pytest.mark.parametrize("kw", [dict(D=166, C=1), dict(D=512, C=2, nonlinear=False)])
def test_loop_route_matches_the_one_model_calls(kw):
    D, C = kw.pop("D"), kw.pop("C")
    nets = _nets(D, C, 3, seed=7, **kw)
    assert not _supported(nets)
    _compare(nets, LISTS[:3], D, seed=3, loss_kind="dense")


def _pack(net):
    from dsmil_wsi_b200.functional import ParamPack
    ic, bc = net.i_classifier, net.b_classifier
    lin = ic._linear()
    W1, b1, W2, b2 = bc._q_params()
    return ParamPack(lin.weight, lin.bias, W1, b1, W2, b2, None, None, bc.fcc.weight, bc.fcc.bias)


def test_unaligned_bag_takes_the_loop_route():
    nets = _nets(512, 2, 3, seed=11)
    lists = [[129, 40], [300], [7, 1000]]
    bags = _bags(lists, 512, seed=12)
    buf = torch.rand(1000 * 512 + 1, device="cuda")
    bags[2][1] = buf[1:].view(1000, 512)
    assert bags[2][1].data_ptr() % 16 == 4
    outs = forward_bags_per_model(nets, bags, grad=True)
    for m, (net, xs, out) in enumerate(zip(nets, bags, outs)):
        ref = net.forward_bags(xs, grad=True)
        for u, v in zip(out.packed, ref.packed):
            assert torch.equal(u, v), m


def test_launches_do_not_grow_with_the_models():
    nets = _nets(512, 2, 5, seed=21)
    bags = _bags(LISTS[:5], 512, seed=22, grad=True)
    counts = {}
    for M in (1, 5):
        outs, fwd = _launches(lambda: forward_bags_per_model(nets[:M], bags[:M], grad=True))
        loss = sum(_dense(list(out), m) for m, out in enumerate(outs))
        _, bwd = _launches(lambda: loss.backward())
        counts[M] = (fwd, bwd)
    assert counts[5] == counts[1] == (FUSED_FWD, FUSED_BWD), counts


def test_one_fold_against_the_fp64_oracle():
    """Fold 0 holds the bags and parameters of the batched oracle case; the other folds train alongside it."""
    case = B_SMALL
    p, Xs, outs1 = _bag_data(case)
    _, w, per_bag = oracle_grads(case, "bags")
    net0 = build_net(case.params()).train()
    others = _nets(case.D, case.C, 2, seed=5)
    xs0 = [torch.from_numpy(X).cuda().requires_grad_(True) for X in Xs]
    rest = _bags([[300, 1], [129]], case.D, seed=5)
    outs = forward_bags_per_model([net0] + others, [xs0] + rest, grad=True)
    assert np.array_equal(_np(outs[0].crit), np.stack([o.idx for o in outs1]))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    loss = sum((c * t(wc)).sum() + (A * t(wA)).sum() + (B[0] * t(wB)).sum() + (pr[0] * t(wp)).sum()
               for (c, pr, A, B), (wc, wA, wB, wp) in zip(outs[0], w))
    loss = loss + _dense([o for o in outs[1]], 1) + _dense([o for o in outs[2]], 2)
    names = _param_names(case)
    params = dict(net0.named_parameters())
    leaves = [params[grad_name(k, case.nonlinear)] for k in names]
    grads = torch.autograd.grad(loss, leaves + xs0)
    _check_params(case, {k: _np(g) for k, g in zip(names, grads)}, summed(per_bag, names), "fold step")
    for b, (g, want) in enumerate(zip(grads[len(names):], per_bag)):
        err = rowwise_err(_np(g), want["X"])
        assert err <= case.tol_q(), (case.name, "gX", b, err)


# ---- a full epoch of five folds -----------------------------------------------------------------------------------
STORE_NS = [2, 10_000, 1, 129, 5000, 128, 7, 900, 127, 300, 2500, 64, 3, 800, 1500, 256, 40, 12]


def _store(D, C, Ns, seed=4):
    store = feed.DeviceBagStore(D)
    rng = np.random.default_rng(seed)
    for i, n in enumerate(Ns):
        store.add_bag(torch.from_numpy(orc.synthetic_bag(int(n), D, 70 + i)),
                      torch.from_numpy((rng.random(C) > 0.5).astype(np.float32)))
    return store


def _opt(kind, net):
    if kind == "sgd":
        return torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
    return torch.optim.Adam(net.parameters(), lr=1e-3, betas=(0.5, 0.9), weight_decay=1e-3, capturable=True)


@pytest.mark.parametrize("opt", ["sgd", "adam"])
@pytest.mark.parametrize("k", [1, 4])
def test_epochs_match_each_fold_trained_alone(opt, k):
    D, C = 512, 2
    for drop in (0.0, 0.3):
        store = _store(D, C, [n if n > 1 or drop == 0 else 2 for n in STORE_NS])
        rng = np.random.default_rng(k)
        # five folds of unequal size over the store (bags may sit in several folds, as training splits overlap)
        folds = [rng.permutation(len(store))[:n].tolist() for n in (9, 4, 13, 1, 7)]
        ps = [orc.random_params(D, C, seed=31 + m) for m in range(5)]
        fused, alone = [build_net(p) for p in ps], [build_net(p) for p in ps]
        o_f, o_a = [_opt(opt, n) for n in fused], [_opt(opt, n) for n in alone]
        crit = torch.nn.BCEWithLogitsLoss()
        g_f = [torch.Generator(device="cuda").manual_seed(5 + m) for m in range(5)]
        g_a = [torch.Generator(device="cuda").manual_seed(5 + m) for m in range(5)]
        for epoch in range(2):
            orders = [np.random.default_rng(10 * epoch + m).permutation(f).tolist() for m, f in enumerate(folds)]
            got = feed.train_epoch_models(fused, store, folds, crit, o_f, dropout_patch=drop, orders=orders,
                                          generators=g_f, bags_per_step=k)
            for m in range(5):
                want = feed.train_epoch(alone[m], store, crit, o_a[m], dropout_patch=drop, order=orders[m],
                                        generator=g_a[m], bags_per_step=k, graph=(k == 1))
                assert got[m] == want, (opt, k, drop, epoch, m, got[m], want)
        for m in range(5):
            for (name, a), b in zip(fused[m].named_parameters(), alone[m].parameters()):
                assert torch.equal(a, b), (opt, k, drop, m, name, float((a - b).abs().max()))
