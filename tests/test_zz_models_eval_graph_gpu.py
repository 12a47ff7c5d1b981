"""The capture-safe inference of the fold models on the GPU, bit for bit: dsmil_forward_bags_models_dev and its generic
twin against each model's dsmil_forward_bags and its one-model dev call, and near its slices of the training fold call;
one capture replayed over ragged batches (ForwardBagsModelsGraph); the programmatic edge of the recorded call; per-model
refusal; feed.eval_epoch_folds against each fold's own eval_epoch (eager and graph, per-fold criteria, graph reuse
across calls); eval_epoch_models(graph=True) against the eager call; and per-fold criteria in train_epoch_models."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import build_net
from oracle import dsmil_oracle as orc
from dsmil_wsi_b200 import _lib, feed
from dsmil_wsi_b200 import functional as Fn
from dsmil_wsi_b200.infer_graph import ForwardBagsModelsGraph
from dsmil_wsi_b200.sharded import milnet_params
from test_zz_infer_graph_gpu import _edges, _kernel_name

pytestmark = pytest.mark.gpu

MAX_ROWS = 600
# model m's bags: unequal lists with bags of 1, 127, 128, 129 and max_rows rows
LISTS = [[129, MAX_ROWS, 1], [127], [128, 5, 40, 1, 129], [MAX_ROWS, 64], [1, 2, 300]]


def _nets(D, C, M, seed, nonlinear=True):
    return [build_net(orc.random_params(D, C, seed + 101 * m, nonlinear=nonlinear, scale=2.0)).eval()
            for m in range(M)]


def _slots(lists, D, max_rows, seed):
    ne = sum(len(ns) for ns in lists)
    g = torch.Generator(device="cuda").manual_seed(seed)
    slots = torch.zeros(ne, max_rows, D, device="cuda")
    flat = [n for ns in lists for n in ns]
    for e, n in enumerate(flat):
        slots[e, :n] = torch.rand(n, D, generator=g, device="cuda")
    return slots, torch.tensor(flat, dtype=torch.int64, device="cuda")


def _bag_lists(lists, slots):
    out, e = [], 0
    for ns in lists:
        out.append([slots[e + b, :n] for b, n in enumerate(ns)])
        e += len(ns)
    return out


def _live(packed, lists, max_rows):
    """Model m's live slices of the capacity-packed outputs."""
    classes, pred, A, B, crit = packed
    out, e = [], 0
    for ns in lists:
        r0, rows, nb = e * max_rows, sum(ns), len(ns)
        out.append((classes[r0:r0 + rows], pred[e:e + nb], A[r0:r0 + rows], B[e:e + nb], crit[e:e + nb]))
        e += nb
    return out


def _same(got, want, what):
    for name, u, v in zip(("classes", "pred", "A", "B", "crit"), got, want):
        assert u.shape == v.shape and torch.equal(u, v), (what, name)


def _eager(net, bags):
    outs, crit = Fn._mil_forward_bags_infer(bags, milnet_params(net))
    return [t.clone() for t in outs.packed] + [crit.clone()]


def _one_dev(net, slots, Ns, max_rows, ns):
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    xs = Fn._slot_addrs(slots, Fn.ParamPack(*milnet_params(net)), "slots")
    out = Fn.mil_forward_bags_dev(xs, Ns, status, max_rows, milnet_params(net))
    torch.cuda.synchronize()
    assert int(status) == 0
    return _live(out, [ns], max_rows)[0]


def _models_dev(nets, lists, slots, Ns, max_rows, generic=False, status=None):
    nbs = tuple(len(ns) for ns in lists)
    status = torch.zeros(len(nets), dtype=torch.int32, device="cuda") if status is None else status
    xs = Fn._slot_addrs(slots, Fn.ParamPack(*milnet_params(nets[0])), "slots")
    out = Fn.mil_forward_bags_models_dev(nbs, xs, Ns, status, max_rows, [milnet_params(n) for n in nets],
                                         generic=generic)
    return out, status


def _check_against_references(nets, lists, slots, Ns, max_rows, generic):
    out, status = _models_dev(nets, lists, slots, Ns, max_rows, generic)
    torch.cuda.synchronize()
    assert status.tolist() == [0] * len(nets)
    got = _live(out, lists, max_rows)
    nbs = tuple(len(ns) for ns in lists)
    params = [t for net in nets for t in milnet_params(net)]
    fn = Fn.MILBagsModelsGenericDevFn if generic else Fn.MILBagsModelsDevFn
    with torch.no_grad():
        train = _live(fn.apply(nbs, slots, Ns, torch.zeros(len(nets), dtype=torch.int32, device="cuda"), *params),
                      lists, max_rows)
    e = 0
    for m, (net, ns, bags) in enumerate(zip(nets, lists, _bag_lists(lists, slots))):
        nb = len(ns)
        _same(got[m], _eager(net, bags), ("dsmil_forward_bags", m))
        _same(got[m], _one_dev(net, slots[e:e + nb], Ns[e:e + nb], max_rows, ns), ("one-model dev", m))
        # the training form's instance scores and critical rows are the same bits; its attend pass reads Q row-major
        # after the tanh, and its bag predictions can differ from the inference forward's in the last bits
        for name, u, v in zip(("classes", "pred", "A", "B", "crit"), got[m], train[m]):
            ok = torch.equal(u, v) if name in ("classes", "crit") else torch.allclose(u, v, rtol=1e-5, atol=1e-6)
            assert ok, ("training fold call", m, name)
        e += nb


@pytest.mark.parametrize("D,C,M", [(512, 2, 5), (1024, 4, 3), (2048, 2, 5)])
def test_dev_call_equals_each_models_references(D, C, M):
    nets = _nets(D, C, M, seed=7000 + D + C)
    lists = LISTS[:M]
    slots, Ns = _slots(lists, D, MAX_ROWS, 1)
    _check_against_references(nets, lists, slots, Ns, MAX_ROWS, False)


@pytest.mark.parametrize("D,C,nonlinear", [(166, 1, True), (230, 1, True), (230, 2, False), (512, 5, True)],
                         ids=["musk", "elephant", "D230C2lin", "D512C5"])
def test_generic_dev_call_equals_each_models_references(D, C, nonlinear):
    M = 4
    nets = _nets(D, C, M, seed=7100 + D + C, nonlinear=nonlinear)
    lists = [[13, 40, 1], [2], [40, 40, 7, 1], [5, 39]]
    slots, Ns = _slots(lists, D, 40, 2)
    _check_against_references(nets, lists, slots, Ns, 40, True)


@pytest.mark.parametrize("generic", [False, True])
def test_one_capture_replays_ragged_batches(generic):
    D, C, mr = (512, 2, MAX_ROWS) if not generic else (166, 1, 40)
    nets = _nets(D, C, 3, seed=7200 + D)
    nbs = [3, 1, 2]
    g = ForwardBagsModelsGraph(nets, nbs, mr, generic=generic)
    batches = [[[1, mr, 129 % mr], [127 % mr + 1], [mr, 1]], [[5, 6, 7], [mr], [1, 1]],
               [[mr, mr, mr], [3], [100 % mr + 1, mr]]]
    for k, lists in enumerate(batches):
        gen = torch.Generator(device="cuda").manual_seed(7300 + k)
        bag_lists = [[torch.rand(n, D, generator=gen, device="cuda") for n in ns] for ns in lists]
        outs = g.run(bag_lists)
        for m, (net, bags, o) in enumerate(zip(nets, bag_lists, outs)):
            assert o.Ns == lists[m]
            _same([t.clone() for t in o.packed] + [o.crit.clone()], _eager(net, bags), (k, m))
    torch.cuda.synchronize()
    assert g.status.tolist() == [0, 0, 0]
    nets[1].b_classifier.fcc.weight = torch.nn.Parameter(nets[1].b_classifier.fcc.weight.detach().clone())
    with pytest.raises(RuntimeError, match="replaced"):
        g.run(bag_lists)


def _capture_edges(nets, lists, slots, Ns, max_rows):
    xs = Fn._slot_addrs(slots, Fn.ParamPack(*milnet_params(nets[0])), "slots")
    status = torch.zeros(len(nets), dtype=torch.int32, device="cuda")
    nbs, plist = tuple(len(ns) for ns in lists), [milnet_params(n) for n in nets]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        Fn.mil_forward_bags_models_dev(nbs, xs, Ns, status, max_rows, plist)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(graph):
        out = Fn.mil_forward_bags_models_dev(nbs, xs, Ns, status, max_rows, plist)
    edges = [(_kernel_name(f), _kernel_name(t), d) for f, t, d in _edges(graph.raw_cuda_graph())]
    return graph, out, status, [(f, d.type, d.from_port) for f, t, d in edges if t is not None and "k_attend_b" in t]


def test_programmatic_edge_survives_capture():
    """The recorded fold call holds a programmatic edge from the phase-1 node to the attend node; replays give the
    eager bits.  Under kernel timing the edge is a plain one."""
    nets = _nets(512, 2, 5, seed=7400)
    lists = [[10_000] * 4, [3000, 10_000], [1, 9999, 128], [10_000], [5000] * 3]
    slots, Ns = _slots(lists, 512, 10_000, 3)
    graph, out, status, into_attend = _capture_edges(nets, lists, slots, Ns, 10_000)
    assert len(into_attend) == 1, into_attend
    src, typ, port = into_attend[0]
    assert src is not None and "k_qmlp_sm90" in src, into_attend
    assert typ == 1 and port in (1, 2), into_attend               # cudaGraphDependencyTypeProgrammatic
    graph.instantiate()
    graph.replay()
    torch.cuda.synchronize()
    assert status.tolist() == [0] * 5
    for m, (got, net, bags) in enumerate(zip(_live(out, lists, 10_000), nets, _bag_lists(lists, slots))):
        _same(got, _eager(net, bags), ("replay", m))
    lib = _lib.load()
    ms, n = (ctypes.c_double * 8)(), (ctypes.c_uint64 * 8)()
    lib.dsmil_profile_enable(1)
    try:
        for _ in range(2):          # timing events for the warm-up and the capture, made before the capture
            _models_dev(nets, lists, slots, Ns, 10_000)
        torch.cuda.synchronize()
        lib.dsmil_profile_read(ms, n)
        _, _, _, plain = _capture_edges(nets, lists, slots, Ns, 10_000)
        torch.cuda.synchronize()
    finally:
        lib.dsmil_profile_read(ms, n)
        lib.dsmil_profile_enable(0)
    assert all(typ != 1 for _, typ, _ in plain), plain


@pytest.mark.parametrize("generic", [False, True])
def test_refusal_is_per_model(generic):
    D, C, mr = (512, 2, MAX_ROWS) if not generic else (166, 1, 40)
    nets = _nets(D, C, 3, seed=7500 + D)
    lists = [[100 % mr + 1, 7], [20, 30 % mr + 1, 9], [mr]]
    slots, Ns = _slots(lists, D, mr, 4)
    ref, _ = _models_dev(nets, lists, slots, Ns, mr, generic)
    ref = [[t.clone() for t in x] for x in _live(ref, lists, mr)]
    # a bag over max_rows in model 1 (its second bag)
    bad_Ns = Ns.clone()
    bad_Ns[3] = mr + 1
    out, status = _models_dev(nets, lists, slots, bad_Ns, mr, generic)
    torch.cuda.synchronize()
    assert status.tolist() == [0, 2, 0]
    got = _live(out, lists, mr)
    for m in (0, 2):
        _same(got[m], ref[m], ("over max_rows", m))
    _, _, _, _, crit = got[1]
    assert all(torch.isfinite(t).all() for t in got[1][:4])
    assert (crit == 0).all()
    # features not aligned for the route in model 1 (its first bag): refused by the planner, never read
    xs = Fn._slot_addrs(slots, Fn.ParamPack(*milnet_params(nets[0])), "slots").clone()
    xs[2] += 2
    status = torch.zeros(3, dtype=torch.int32, device="cuda")
    out = Fn.mil_forward_bags_models_dev([2, 3, 1], xs, Ns, status, mr, [milnet_params(n) for n in nets],
                                         generic=generic)
    torch.cuda.synchronize()
    assert status.tolist() == [0, 1, 0]
    got = _live(out, lists, mr)
    for m in (0, 2):
        _same(got[m], ref[m], ("misaligned", m))
    assert all(torch.isfinite(t).all() for t in got[1][:4]) and (got[1][4] == 0).all()


def _store(D, C, Ns, seed):
    rng = np.random.default_rng(seed)
    store = feed.DeviceBagStore(D)
    for i, n in enumerate(Ns):
        store.add_bag(torch.from_numpy(orc.synthetic_bag(int(n), D, seed + i)),
                      torch.from_numpy((rng.random(C) > 0.5).astype(np.float32)))
    return store


def _sub_store(store, fold):
    sub = feed.DeviceBagStore(store.D, device=store.device)
    sub.bags = [store.bags[i] for i in fold]
    return sub


def _criteria(C, M, seed):
    rng = np.random.default_rng(seed)
    return [torch.nn.BCEWithLogitsLoss(pos_weight=torch.full((C,), float(rng.uniform(0.3, 3.0)), device="cuda"))
            for _ in range(M)]


def _assert_fold_results(got, nets, store, folds, criteria, average, k, graph, generic=False):
    assert len(got) == len(folds)
    for m, fold in enumerate(folds):
        want = feed.eval_epoch(nets[m], _sub_store(store, fold), criteria[m], average=average, bags_per_launch=k,
                               graph=graph, generic=generic)
        assert got[m][0] == want[0], (m, got[m][0], want[0])
        assert np.array_equal(got[m][1], want[1]) and got[m][1].dtype == want[1].dtype, m
        assert np.array_equal(got[m][2], want[2]) and got[m][2].dtype == want[2].dtype, m


@pytest.mark.parametrize("k", [1, 16])
@pytest.mark.parametrize("average", [False, True])
@pytest.mark.parametrize("graph", [False, True])
def test_eval_epoch_folds_equals_each_folds_eval_epoch(graph, average, k):
    D, C, M = 512, 2, 4
    rng = np.random.default_rng(7600 + k)
    store = _store(D, C, rng.integers(1, 2500, 60).tolist(), 7700)
    folds = [rng.permutation(len(store))[:n].tolist() for n in (17, 9, 33, 1)]
    nets = _nets(D, C, M, seed=7800)
    criteria = _criteria(C, M, 7900)
    got = feed.eval_epoch_folds(nets, store, folds, criteria, average=average, bags_per_launch=k, graph=graph)
    _assert_fold_results(got, nets, store, folds, criteria, average, k, graph)
    if graph:   # one criterion for all folds
        crit = torch.nn.BCEWithLogitsLoss()
        got = feed.eval_epoch_folds(nets, store, folds, crit, average=average, bags_per_launch=k, graph=True)
        _assert_fold_results(got, nets, store, folds, [crit] * M, average, k, True)


@pytest.mark.parametrize("graph", [False, True])
def test_eval_epoch_folds_generic_musk(graph):
    D, C, M = 166, 1, 5
    rng = np.random.default_rng(8000)
    store = _store(D, C, rng.integers(2, 41, 92).tolist(), 8100)
    order = rng.permutation(len(store)).tolist()
    folds = [feed.cross_validation_set(order, 10, i)[1] for i in range(M)]
    nets = _nets(D, C, M, seed=8200)
    criteria = _criteria(C, M, 8300)
    got = feed.eval_epoch_folds(nets, store, folds, criteria, bags_per_launch=16, graph=graph, generic=True)
    _assert_fold_results(got, nets, store, folds, criteria, False, 16, graph, generic=True)


def test_eval_epoch_folds_reuses_its_graphs_across_calls():
    D, C, M = 512, 2, 3
    store = _store(D, C, [300, 1200, 64, 900, 5, 77, 1024], 8400)
    folds = [[0, 1, 2], [3, 4], [5, 6, 0]]
    nets = _nets(D, C, M, seed=8500)
    criteria = _criteria(C, M, 8600)
    feed.eval_epoch_folds(nets, store, folds, criteria, bags_per_launch=2, graph=True)
    first = dict(feed._FOLD_EVAL_GRAPHS[nets[0]])
    assert len(first) == 2                                         # steps (2, 2, 2) and (1, 0, 1): folds 0 and 2
    with torch.no_grad():
        for net in nets:
            for p in net.parameters():
                p.mul_(0.5)
    got = feed.eval_epoch_folds(nets, store, folds, criteria, bags_per_launch=2, graph=True)
    assert dict(feed._FOLD_EVAL_GRAPHS[nets[0]]) == first and \
        all(feed._FOLD_EVAL_GRAPHS[nets[0]][key] is g for key, g in first.items())
    _assert_fold_results(got, nets, store, folds, criteria, False, 2, True)
    nets[2].b_classifier.fcc.weight = torch.nn.Parameter(nets[2].b_classifier.fcc.weight.detach().clone())
    got = feed.eval_epoch_folds(nets, store, folds, criteria, bags_per_launch=2, graph=True)
    now = feed._FOLD_EVAL_GRAPHS[nets[0]]
    assert all(now[key] is not g for key, g in first.items())      # every graph held fold 2: both re-recorded
    _assert_fold_results(got, nets, store, folds, criteria, False, 2, True)


@pytest.mark.parametrize("average", [False, True])
def test_eval_epoch_models_graph_equals_eager(average):
    D, C, M = 512, 2, 3
    rng = np.random.default_rng(8700)
    store = _store(D, C, rng.integers(1, 2000, 37).tolist(), 8800)
    nets = _nets(D, C, M, seed=8900)
    crit = torch.nn.BCEWithLogitsLoss()
    ref = feed.eval_epoch_models(nets, store, crit, average=average, bags_per_launch=16)
    got = feed.eval_epoch_models(nets, store, crit, average=average, bags_per_launch=16, graph=True)
    for (gl, glab, gp), (rl, rlab, rp) in zip(got, ref):
        assert gl == rl and np.array_equal(glab, rlab) and np.array_equal(gp, rp)


def _opt(net):
    return torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)


@pytest.mark.parametrize("mode", ["eager", "graph", "generic_graph"])
def test_train_epoch_models_with_per_fold_criteria(mode):
    graph, generic = mode != "eager", mode == "generic_graph"
    D, C = (166, 1) if generic else (512, 2)
    rng = np.random.default_rng(9000)
    store = _store(D, C, rng.integers(2, 41 if generic else 900, 24).tolist(), 9100)
    folds = [rng.permutation(len(store))[:n].tolist() for n in (9, 4, 13)]
    ps = [orc.random_params(D, C, seed=9200 + m) for m in range(3)]
    nets = {w: [build_net(p) for p in ps] for w in ("folds", "alone")}
    opts = {w: [_opt(n) for n in ns] for w, ns in nets.items()}
    criteria = _criteria(C, 3, 9300)
    gens = {w: [torch.Generator(device="cuda").manual_seed(9400 + m) for m in range(3)] for w in nets}
    k = 4
    for epoch in range(2):
        orders = [np.random.default_rng(10 * epoch + m).permutation(f).tolist() for m, f in enumerate(folds)]
        got = feed.train_epoch_models(nets["folds"], store, folds, criteria, opts["folds"], orders=orders,
                                      generators=gens["folds"], bags_per_step=k, graph=graph, generic=generic)
        for m in range(3):
            want = feed.train_epoch(nets["alone"][m], store, criteria[m], opts["alone"][m], order=orders[m],
                                    generator=gens["alone"][m], bags_per_step=k, graph=graph, generic=generic)
            assert got[m] == want, (mode, epoch, m, got[m], want)
    for m in range(3):
        for (name, a), b in zip(nets["folds"][m].named_parameters(), nets["alone"][m].parameters()):
            assert torch.equal(a, b), (mode, m, name)
