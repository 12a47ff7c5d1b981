"""The capture-safe fold step on the generic shapes, on the GPU: dsmil_generic_forward_bags_models_train_dev /
dsmil_generic_backward_bags_models_dev against the one-model generic dev calls on each fold's bags (torch.equal on
every output and gradient), per-fold refusal, one capture replayed over new sizes, the library launches of a replay,
FoldTrainStepGraph(generic=True) against each fold's own TrainStepGraph(generic=True), and
feed.train_epoch_models(graph=True, generic=True) against each fold's own train_epoch(graph=True, generic=True)."""
import numpy as np
import pytest
import torch

from helpers import build_net
from oracle import dsmil_oracle as orc
from dsmil_wsi_b200 import feed
from dsmil_wsi_b200 import functional as Fn
from dsmil_wsi_b200.sharded import milnet_params
from dsmil_wsi_b200.train_graph import FoldTrainStepGraph, TrainStepGraph
from test_zz_models_train_graph_gpu import _capture, _graph_kernels, _leaves, _live, _same, _same_grads, _slots, \
    _upstream

pytestmark = pytest.mark.gpu

# (D, C, nonlinear): Musk, Elephant, a linear q, a k_qmlp_sm90 phase 1 (C > 4, D % 128 == 0), an odd D past 2048
SHAPES = [(166, 1, True), (230, 1, True), (230, 2, False), (512, 6, True), (2049, 2, True)]
IDS = [f"D{d}C{c}{'' if nl else 'lin'}" for d, c, nl in SHAPES]
MAX_ROWS = 9473
# fold m's bags: unequal lists, with bags of 1, 127, 128, 129, 9472 and 9473 rows
LISTS = [[129, 9473, 1], [127], [128, 5, 40, 1, 129], [9472, 64], [1, 2], [300], [40, 128, 127], [13, 9473]]


def _nets(D, C, nonlinear, M, seed):
    return [build_net(orc.random_params(D, C, seed + 101 * m, nonlinear=nonlinear, scale=2.0)).train()
            for m in range(M)]


def _fold_dev(nets, lists, slots, Ns, gc, gp, status=None):
    nbs = tuple(len(ns) for ns in lists)
    status = torch.zeros(len(nets), dtype=torch.int32, device="cuda") if status is None else status
    params = [t for net in nets for t in milnet_params(net)]
    packed = Fn.MILBagsModelsGenericDevFn.apply(nbs, slots, Ns, status, *params)
    grads = torch.autograd.grad([packed[0], packed[1]], _leaves(nets), [gc, gp], allow_unused=True)
    return packed, grads, status


def _one_dev(net, slots, Ns, gc, gp):
    """The one-model generic dev calls on one fold's slots."""
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    packed = Fn.MILBagsDevFn.apply(slots, Ns, status, *milnet_params(net))
    grads = torch.autograd.grad([packed[0], packed[1]], list(net.parameters()), [gc, gp], allow_unused=True)
    return packed, grads, status


def _per_fold(nets, lists, slots, Ns, gc, gp, max_rows):
    """Each fold's one-model dev calls on its own block: live slices and gradients, in fold order."""
    outs, grads, e = [], [], 0
    for net, ns in zip(nets, lists):
        nb = len(ns)
        packed, g, status = _one_dev(net, slots[e:e + nb], Ns[e:e + nb], gc[e * max_rows:(e + nb) * max_rows],
                                     gp[e:e + nb])
        assert int(status) == 0
        outs += _live(packed, [ns], max_rows)
        grads += list(g)
        e += nb
    return outs, grads


@pytest.mark.parametrize("M", [1, 2, 5, 8])
@pytest.mark.parametrize("D,C,nonlinear", SHAPES, ids=IDS)
def test_fold_dev_calls_equal_each_folds_one_model_dev_calls(D, C, nonlinear, M):
    if M in (1, 8) and D not in (166, 230):
        pytest.skip("M = 1 and 8 on the classic-MIL shapes; the others at M = 2 and 5")
    nets = _nets(D, C, nonlinear, M, seed=D + M)
    lists = LISTS[:M]
    slots, Ns = _slots(lists, D, MAX_ROWS, 1)
    gc, gp = _upstream(lists, C, MAX_ROWS, 2)
    packed, grads, status = _fold_dev(nets, lists, slots, Ns, gc, gp)
    assert status.tolist() == [0] * M
    want, want_grads = _per_fold(nets, lists, slots, Ns, gc, gp, MAX_ROWS)
    _same(_live(packed, lists, MAX_ROWS), want, (D, C, M))
    _same_grads(grads, want_grads, (D, C, M))


def test_refusal_is_per_fold():
    D, C, max_rows = 166, 1, 40
    nets = _nets(D, C, True, 3, seed=8)
    lists = [[13, 40], [5, 30, 2], [27, 1]]
    slots, Ns = _slots(lists, D, max_rows, 5)
    gc, gp = _upstream(lists, C, max_rows, 6)
    clean, clean_grads, status = _fold_dev(nets, lists, slots, Ns, gc, gp)
    assert status.tolist() == [0, 0, 0]
    clean = [[t.clone() for t in m] for m in _live(clean, lists, max_rows)]
    k = len(list(nets[0].parameters()))
    for what, b in (("zero rows", 1), ("over capacity", 2), ("zero rows", 0)):
        bad = Ns.clone()
        bad[2 + b] = 0 if what == "zero rows" else max_rows + 1
        packed, grads, status = _fold_dev(nets, lists, slots, bad, gc, gp)
        assert status.tolist() == [0, 1 + b, 0], what
        live = _live(packed, lists, max_rows)
        _same([live[0], live[2]], [clean[0], clean[2]], what)
        _same_grads(grads[:k] + grads[2 * k:], clean_grads[:k] + clean_grads[2 * k:], what)
        assert all(bool(torch.isfinite(t).all()) for t in (packed[1][2:5], packed[3][2:5]))
        assert all(bool(torch.isfinite(g).all()) for g in grads[k:2 * k])
        assert packed[4][2:5].eq(0).all()


def _last_call_kernels(fn):
    """Library kernels (namespace dsmil) that torch.profiler records for one run of fn, an eager fold forward and
    backward, in launch order.  In a process that has run the profiler before, the first kernel records of a profiled
    window can be missing, so the window runs fn twice and the count is the second run's: the records from its
    forward planner on (each run launches k_plan_bags_models twice, for the forward and for the backward).  Kernels
    launched by a graph replay are not counted this way: in such a process torch.profiler may record only some of them,
    or none; the replay's own launches are the graph's kernel nodes (_graph_kernels), the same sequence."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        fn()
        torch.cuda.synchronize()
    recs = sorted((e.time_range.start, e.name) for e in prof.events()
                  if e.device_type == torch.autograd.DeviceType.CUDA and "dsmil::" in e.name)
    names = [n for _, n in recs]
    plans = [i for i, n in enumerate(names) if "k_plan_bags_models" in n]
    assert len(plans) >= 2, names
    return names[plans[-2]:]


def launches_per_replay(D, C, nonlinear, M):
    """DESIGN §4.2j: library launches of one replay of the generic fold forward and backward (d_classes given).
    Forward: the planner, then scores, layer 1, crit/q_max, attend, combine and finalize once for all folds, layer 2
    once per fold; on the k_qmlp_sm90 shapes the weight-image prep and phase 1 once per fold instead of scores and the
    two layers.  Backward: 19 launches for all folds (14 for a linear q)."""
    qmlp = nonlinear and D % 128 == 0
    fwd = 5 + 2 * M if qmlp else 7 + (M if nonlinear else 0)
    return fwd + (19 if nonlinear else 14)


@pytest.mark.parametrize("D,C,nonlinear", [(166, 1, True), (230, 2, False), (512, 6, True)],
                         ids=["D166C1", "D230C2lin", "D512C6"])
def test_one_capture_replays_new_sizes_with_the_eager_dev_calls_bits(D, C, nonlinear):
    max_rows = 3000
    shape = [[1, 1, 1], [1], [1, 1], [1, 1], [1]]
    M = len(shape)
    nets = _nets(D, C, nonlinear, M, seed=3)
    slots, Ns = _slots(shape, D, max_rows, 1)
    gc, gp = _upstream(shape, C, max_rows, 2)
    graph, (packed, grads, status) = _capture(lambda: _fold_dev(nets, shape, slots, Ns, gc, gp))
    names = [k for k in _graph_kernels(graph) if "dsmil" in k]
    want_n = launches_per_replay(D, C, nonlinear, M)
    assert len(names) == want_n, names                         # the launches of every replay
    ran = _last_call_kernels(lambda: _fold_dev(nets, shape, slots, Ns, gc, gp))
    assert len(ran) == want_n, ran                             # torch.profiler's count of the same calls
    rng = np.random.default_rng(D)
    for batch in range(3):
        lists = [[int(rng.choice([1, 2, 127, 128, 129, 2999, 3000, 40])) for _ in ns] for ns in shape]
        fresh, sizes = _slots(lists, D, max_rows, 10 + batch)
        slots.copy_(fresh)
        Ns.copy_(sizes)
        graph.replay()
        assert status.tolist() == [0] * M
        want, want_grads, _ = _fold_dev(nets, lists, slots, Ns, gc, gp)
        _same(_live(packed, lists, max_rows), _live(want, lists, max_rows), f"replay {batch}")
        _same_grads(grads, want_grads, f"replay {batch}")
        per, per_grads = _per_fold(nets, lists, slots, Ns, gc, gp, max_rows)
        _same(_live(packed, lists, max_rows), per, f"replay {batch}, one-model")
        _same_grads(grads, per_grads, f"replay {batch}, one-model")


def _opt(kind, net):
    if kind == "sgd":
        return torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
    return torch.optim.Adam(net.parameters(), lr=2e-4, betas=(0.5, 0.9), weight_decay=5e-3, capturable=True)


def _state(opt):
    return [v for p in opt.param_groups[0]["params"] for v in opt.state.get(p, {}).values() if torch.is_tensor(v)]


def _fill(slots_of, Ns_at, labels_at, lists, D, C, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    for m, ns in enumerate(lists):
        for b, n in enumerate(ns):
            n = min(max(n, 0), slots_of(m).shape[1])
            slots_of(m)[b, :n] = torch.rand(n, D, generator=gen, device="cuda")
        Ns_at(m).copy_(torch.tensor(ns, dtype=torch.int64, device="cuda"))
        labels_at(m).copy_((torch.rand(len(ns), C, generator=gen, device="cuda") > 0.5).float())


@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_fold_graph_matches_each_folds_own_graph_and_guards_per_fold(opt):
    D, C, max_rows, nbs = 230, 1, 13, [2, 1, 3]
    ps = [orc.random_params(D, C, seed=61 + m) for m in range(3)]
    fold, alone = [build_net(p).train() for p in ps], [build_net(p).train() for p in ps]
    o_f, o_a = [_opt(opt, n) for n in fold], [_opt(opt, n) for n in alone]
    crit = torch.nn.BCEWithLogitsLoss()
    fg = FoldTrainStepGraph(fold, crit, o_f, nbs, max_rows, generic=True)
    assert fg.generic
    gs = [TrainStepGraph(alone[m], crit, o_a[m], nbs[m], max_rows, generic=True) for m in range(3)]
    bag0 = [0, 2, 3]
    steps = [[[2, 13], [1], [7, 12, 13]], [[5, 6], [14], [3, 1, 1]], [[13, 13], [4], [0, 5, 6]], [[7, 13], [12], [9, 3, 2]]]
    for t, lists in enumerate(steps):
        refused = [m for m, ns in enumerate(lists) if min(ns) < 1 or max(ns) > max_rows]
        _fill(lambda m: fg.slots[m], lambda m: fg.Ns[bag0[m]:bag0[m] + nbs[m]],
              lambda m: fg.labels[bag0[m]:bag0[m] + nbs[m]], lists, D, C, 20 + t)
        _fill(lambda m: gs[m].slots, lambda m: gs[m].Ns, lambda m: gs[m].labels, lists, D, C, 20 + t)
        kept = [[v.clone() for v in fg._kept[m]] for m in range(3)]
        losses = fg.step().clone()
        for m in range(3):
            if m in refused:                           # the refused fold is not fed to its own graph: it must not move
                assert torch.isnan(losses[m])
                for u, v in zip(fg._kept[m], kept[m]):
                    assert torch.equal(u, v), (t, m)
                continue
            want = gs[m].step()
            assert torch.equal(losses[m], want), (t, m, float(losses[m]), float(want))
            for (name, a), b in zip(fold[m].named_parameters(), alone[m].parameters()):
                assert torch.equal(a.grad, b.grad), (t, m, name)
                assert torch.equal(a, b), (t, m, name)
            for u, v in zip(_state(o_f[m]), _state(o_a[m])):
                assert torch.equal(u, v), (t, m)
    assert fg.status.tolist() == [0, 1, 1]
    assert all(g.status.item() == 0 for g in gs)


def _store(D, C, Ns, seed=4):
    store = feed.DeviceBagStore(D)
    rng = np.random.default_rng(seed)
    for i, n in enumerate(Ns):
        store.add_bag(torch.from_numpy(orc.synthetic_bag(int(n), D, 70 + i)),
                      torch.from_numpy((rng.random(C) > 0.5).astype(np.float32)))
    return store


@pytest.mark.parametrize("opt", ["sgd", "adam"])
@pytest.mark.parametrize("k", [1, 4])
@pytest.mark.parametrize("D,C,nonlinear", [(166, 1, True), (230, 2, False)], ids=["musk", "D230C2lin"])
def test_graph_epochs_match_each_fold_trained_alone(D, C, nonlinear, k, opt):
    rng = np.random.default_rng(k)
    Ns = rng.integers(2, 41, size=24).tolist()
    for drop in (0.0, 0.3):
        store = _store(D, C, Ns)
        folds = [rng.permutation(len(store))[:n].tolist() for n in (9, 4, 13, 1, 7)]
        ps = [orc.random_params(D, C, seed=31 + m, nonlinear=nonlinear) for m in range(5)]
        nets = {w: [build_net(p) for p in ps] for w in ("graph", "alone")}
        opts = {w: [_opt(opt, n) for n in ns] for w, ns in nets.items()}
        gens = {w: [torch.Generator(device="cuda").manual_seed(5 + m) for m in range(5)] for w in nets}
        crit = torch.nn.BCEWithLogitsLoss()
        for epoch in range(2):
            orders = [np.random.default_rng(10 * epoch + m).permutation(f).tolist() for m, f in enumerate(folds)]
            got = feed.train_epoch_models(nets["graph"], store, folds, crit, opts["graph"], dropout_patch=drop,
                                          orders=orders, generators=gens["graph"], bags_per_step=k, graph=True,
                                          generic=True)
            for m in range(5):
                want = feed.train_epoch(nets["alone"][m], store, crit, opts["alone"][m], dropout_patch=drop,
                                        order=orders[m], generator=gens["alone"][m], bags_per_step=k, graph=True,
                                        generic=True)
                assert got[m] == want, (k, drop, epoch, m, got[m], want)
        for m in range(5):
            for (name, a), b in zip(nets["graph"][m].named_parameters(), nets["alone"][m].parameters()):
                assert torch.equal(a, b), (k, drop, m, name)
            for u, v in zip(_state(opts["graph"][m]), _state(opts["alone"][m])):
                assert torch.equal(u, v), (k, drop, m)
