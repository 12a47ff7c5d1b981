"""The capture-safe fold step on the GPU: dsmil_forward_bags_models_train_dev / dsmil_backward_bags_models_dev against
the eager fold calls and the one-model dev calls (torch.equal on every output and gradient), one capture replayed over
batches of different sizes, per-model refusal, FoldTrainStepGraph against each fold's own TrainStepGraph, and
feed.train_epoch_models(graph=True) against each fold trained alone and against the eager fold epoch."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import build_net
from oracle import dsmil_oracle as orc
from dsmil_wsi_b200 import _lib, feed
from dsmil_wsi_b200 import functional as Fn
from dsmil_wsi_b200.sharded import milnet_params
from dsmil_wsi_b200.train_graph import FoldTrainStepGraph, TrainStepGraph
from test_dense_upstream_grads_gpu import K_SPLITS, rag_rows_per_chunk, tn_use_gemv
from test_zz_infer_graph_gpu import _kernel_name
from test_zz_models_train_gpu import STORE_NS, _nets, _opt, _store

pytestmark = pytest.mark.gpu

MAX_ROWS = 10_000
# model m's bags: unequal lists with bags of 1, 127, 128, 129 rows and one at max_rows
LISTS = [[129, MAX_ROWS, 1], [127], [128, 5, 3000, 1, 129], [MAX_ROWS, 64], [1, 1], [300], [2000, 128, 127], [77, 4096]]


def _boundary_list(C, D):
    """Two bags whose row total sits one past a rag_rows_per_chunk step of gWi's chunking."""
    gemv = tn_use_gemv(C, D)
    total = 64 * K_SPLITS + 1 if gemv else 128 * max(1, K_SPLITS // (-(-D // 128))) + 1
    assert rag_rows_per_chunk(C, D, total, gemv) > rag_rows_per_chunk(C, D, total - 1, gemv)
    return [total // 2, total - total // 2]


def _slots(lists, D, max_rows, seed):
    """Member-major slots [sum nb, max_rows, D] filled with random bags, their sizes on the device, and the bags."""
    ne = sum(len(ns) for ns in lists)
    g = torch.Generator(device="cuda").manual_seed(seed)
    slots = torch.zeros(ne, max_rows, D, device="cuda")
    flat = [n for ns in lists for n in ns]
    for e, n in enumerate(flat):
        slots[e, :n] = torch.rand(n, D, generator=g, device="cuda")
    return slots, torch.tensor(flat, dtype=torch.int64, device="cuda")


def _leaves(nets):
    return [p for net in nets for p in net.parameters()]


def _upstream(lists, C, max_rows, seed):
    """Dense upstream gradients for classes (capacity rows) and pred."""
    ne = sum(len(ns) for ns in lists)
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(ne * max_rows, C, generator=g, device="cuda"), torch.randn(ne, C, generator=g, device="cuda"))


def _dev(nets, lists, slots, Ns, gc, gp, max_rows):
    """The fold dev calls: per-model live slices of (classes, pred, A, B, crit), the gradients, the status words."""
    nbs = tuple(len(ns) for ns in lists)
    status = torch.zeros(len(nets), dtype=torch.int32, device="cuda")
    params = [t for net in nets for t in milnet_params(net)]
    classes, pred, A, B, crit = Fn.MILBagsModelsDevFn.apply(nbs, slots, Ns, status, *params)
    grads = torch.autograd.grad([classes, pred], _leaves(nets), [gc, gp], allow_unused=True)
    return (classes, pred, A, B, crit), grads, status


def _live(packed, lists, max_rows):
    """Model m's live slices of the capacity-packed outputs."""
    classes, pred, A, B, crit = packed
    out, e = [], 0
    for ns in lists:
        r0, rows, nb = e * max_rows, sum(ns), len(ns)
        out.append((classes[r0:r0 + rows], pred[e:e + nb], A[r0:r0 + rows], B[e:e + nb], crit[e:e + nb]))
        e += nb
    return out


def _eager(nets, lists, slots, gc, gp, max_rows):
    """The eager fold calls on the same bags and the same upstream gradients (those of the live rows)."""
    nbs = tuple(len(ns) for ns in lists)
    flat = [n for ns in lists for n in ns]
    bags = [slots[e, :n] for e, n in enumerate(flat)]
    params = [t for net in nets for t in milnet_params(net)]
    classes, pred, A, B, crit = Fn.MILBagsModelsFn.apply(nbs, *bags, *params)
    live, e = [], 0
    for ns in lists:
        live.append(gc[e * max_rows:e * max_rows + sum(ns)])
        e += len(ns)
    grads = torch.autograd.grad([classes, pred], _leaves(nets), [torch.cat(live), gp], allow_unused=True)
    outs, row, e = [], 0, 0
    for ns in lists:
        rows, nb = sum(ns), len(ns)
        outs.append((classes[row:row + rows], pred[e:e + nb], A[row:row + rows], B[e:e + nb], crit[e:e + nb]))
        row, e = row + rows, e + nb
    return outs, grads


def _same(got, want, what):
    for m, (g, w) in enumerate(zip(got, want)):
        for name, u, v in zip(("classes", "pred", "A", "B", "crit"), g, w):
            assert torch.equal(u, v), (what, m, name)


def _same_grads(got, want, what):
    for i, (u, v) in enumerate(zip(got, want)):
        assert (u is None) == (v is None), (what, i)
        if u is not None:
            assert torch.equal(u, v), (what, i, float((u - v).abs().max()))


@pytest.mark.parametrize("M", [1, 2, 5, 8])
@pytest.mark.parametrize("D,C", [(512, 2), (1024, 4), (2048, 1)])
def test_dev_calls_match_the_eager_fold_calls_and_the_one_model_dev_calls(D, C, M):
    nets = _nets(D, C, M)
    ps = (_lib.DsmilParams * M)(*[Fn.ParamPack(*milnet_params(n)).struct for n in nets])
    if not _lib.load().dsmil_models_supported(ps, M):
        pytest.skip("M members of this shape do not fit the fused kernel's shared memory")
    lists = [list(ns) for ns in LISTS[:M]]
    lists[-1] = _boundary_list(C, D)
    max_rows = max(MAX_ROWS, max(n for ns in lists for n in ns))
    slots, Ns = _slots(lists, D, max_rows, 40 + M)
    gc, gp = _upstream(lists, C, max_rows, 50 + M)
    packed, grads, status = _dev(nets, lists, slots, Ns, gc, gp, max_rows)
    assert status.tolist() == [0] * M
    want, want_grads = _eager(nets, lists, slots, gc, gp, max_rows)
    _same(_live(packed, lists, max_rows), want, "eager fold")
    _same_grads(grads, want_grads, "eager fold")
    # model m alone through the one-model dev calls on its block of the slots
    e = 0
    for m, (net, ns) in enumerate(zip(nets, lists)):
        nb = len(ns)
        st = torch.zeros(1, dtype=torch.int32, device="cuda")
        out = Fn.MILBagsDevFn.apply(slots[e:e + nb], Ns[e:e + nb], st, *milnet_params(net))
        g1 = torch.autograd.grad([out[0], out[1]], list(net.parameters()),
                                 [gc[e * max_rows:(e + nb) * max_rows], gp[e:e + nb]], allow_unused=True)
        rows = sum(ns)
        one = (out[0][:rows], out[1], out[2][:rows], out[3], out[4])
        _same([_live(packed, lists, max_rows)[m]], [one], f"one-model dev {m}")
        k = len(list(net.parameters()))
        _same_grads(grads[m * k:(m + 1) * k], g1, f"one-model dev {m}")
        assert st.item() == 0
        e += nb


def _capture(fn):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(graph):
        out = fn()
    return graph, out


def _graph_kernels(graph):
    rt = ctypes.CDLL("libcudart.so.12")
    n = ctypes.c_size_t(0)
    raw = ctypes.c_void_p(graph.raw_cuda_graph())
    assert rt.cudaGraphGetNodes(raw, None, ctypes.byref(n)) == 0
    nodes = (ctypes.c_void_p * n.value)()
    assert rt.cudaGraphGetNodes(raw, nodes, ctypes.byref(n)) == 0
    return [k for k in (_kernel_name(nodes[i]) for i in range(n.value)) if k is not None]


def test_one_capture_replays_every_batch_and_does_not_grow_with_the_models():
    D, C = 512, 2
    counts = {}
    for M in (2, 5):
        nets = _nets(D, C, M, seed=3)
        shape = [[1, 1, 1], [1], [1, 1]] + [[1, 1]] * (M - 3) if M > 3 else [[1, 1, 1], [1]]
        slots, Ns = _slots(shape, D, 3000, 1)
        gc, gp = _upstream(shape, C, 3000, 2)
        launches = _lib.launch_count()
        graph, (packed, grads, status) = _capture(lambda: _dev(nets, shape, slots, Ns, gc, gp, 3000))
        names = _graph_kernels(graph)
        assert sum("k_qmlp_sm90" in k for k in names) == 1
        assert sum("k_plan_bags_models" in k for k in names) == 2            # one per call
        counts[M] = sum("dsmil" in k for k in names)
        rng = np.random.default_rng(M)
        for batch in range(3):
            lists = [[int(rng.choice([1, 127, 128, 129, 2999, 3000, 700])) for _ in ns] for ns in shape]
            fresh, sizes = _slots(lists, D, 3000, 10 + batch)
            slots.copy_(fresh)
            Ns.copy_(sizes)
            before = _lib.launch_count()
            graph.replay()
            assert _lib.launch_count() == before                              # no library call on the host
            assert status.tolist() == [0] * M
            want, want_grads = _eager(nets, lists, slots, gc, gp, 3000)
            _same(_live(packed, lists, 3000), want, f"replay {batch}")
            _same_grads(grads, want_grads, f"replay {batch}")
        assert launches < _lib.launch_count()
    assert counts[2] == counts[5], counts


@pytest.mark.parametrize("M", [2, 5])
def test_dense_upstream_gradients_against_the_fp64_oracle(M):
    """Fold 0 holds the bags, parameters and probe-row upstream gradients of the batched oracle case; the other folds
    train alongside it under dense random upstream gradients."""
    from helpers import grad_name
    from test_dense_upstream_grads_gpu import B_SMALL as case, _bag_data, _check_params, _np, _param_names, \
        oracle_grads, summed
    p, Xs, outs1 = _bag_data(case)
    _, w, per_bag = oracle_grads(case, "dev")
    nets = [build_net(case.params()).train()] + _nets(case.D, case.C, M - 1, seed=5)
    lists = [[int(n) for n in case.Ns]] + [[300, 1], [129], [64, 700, 5], [1]][:M - 1]
    max_rows = max(n for ns in lists for n in ns)
    slots, Ns = _slots(lists, case.D, max_rows, 9)
    gc, gp = _upstream(lists, case.C, max_rows, 10)
    row = 0
    for b, (X, (wc, _, _, wp)) in enumerate(zip(Xs, w)):
        slots[b, :X.shape[0]] = torch.from_numpy(X).cuda()
        gc[row:row + X.shape[0]] = torch.from_numpy(np.ascontiguousarray(wc)).cuda()
        gp[b] = torch.from_numpy(np.ascontiguousarray(wp)).cuda().view(-1)
        row += X.shape[0]
    packed, grads, status = _dev(nets, lists, slots, Ns, gc, gp, max_rows)
    assert status.tolist() == [0] * M
    assert np.array_equal(_np(packed[4][:len(Xs)]), np.stack([o.idx for o in outs1]))
    names = _param_names(case)
    mine = dict(zip([n for n, _ in nets[0].named_parameters()], grads))
    _check_params(case, {k: _np(mine[grad_name(k, case.nonlinear)]) for k in names}, summed(per_bag, names),
                  f"fold dev step, M={M}")


def test_refusal_is_per_model():
    D, C, max_rows = 512, 2, 1000
    nets = _nets(D, C, 3, seed=8)
    lists = [[129, 1000], [5, 300, 64], [127, 1]]
    slots, Ns = _slots(lists, D, max_rows, 5)
    gc, gp = _upstream(lists, C, max_rows, 6)
    clean, clean_grads, status = _dev(nets, lists, slots, Ns, gc, gp, max_rows)
    assert status.tolist() == [0, 0, 0]
    clean = [[t.clone() for t in m] for m in _live(clean, lists, max_rows)]
    k = len(list(nets[0].parameters()))
    for what, b in (("zero rows", 1), ("over capacity", 2), ("zero rows", 0)):
        bad = Ns.clone()
        bad[2 + b] = 0 if what == "zero rows" else max_rows + 1
        packed, grads, status = _dev(nets, lists, slots, bad, gc, gp, max_rows)
        assert status.tolist() == [0, 1 + b, 0], what
        live = _live(packed, lists, max_rows)
        _same([live[0], live[2]], [clean[0], clean[2]], what)
        _same_grads(grads[:k] + grads[2 * k:], clean_grads[:k] + clean_grads[2 * k:], what)
        e, nb = 2, 3
        assert all(bool(torch.isfinite(t).all()) for t in (packed[1][e:e + nb], packed[3][e:e + nb]))
        assert all(bool(torch.isfinite(g).all()) for g in grads[k:2 * k])
        assert packed[4][e:e + nb].eq(0).all()
    # a misaligned feature pointer in model 1: the bag list passed directly
    lib = _lib.load()
    packs = [Fn.ParamPack(*milnet_params(n)) for n in nets]
    ps = (_lib.DsmilParams * 3)(*[P.struct for P in packs])
    nbs = (ctypes.c_int32 * 3)(2, 3, 2)
    xs = slots.data_ptr() + 4 * max_rows * D * torch.arange(7, dtype=torch.int64, device="cuda")
    xs[3] += 4
    ne = 7
    new = lambda *s: torch.empty(*s, device="cuda")
    classes, A, sQ, sH = new(ne * max_rows, C), new(ne * max_rows, C), new(ne * max_rows, 128), new(ne * max_rows, 128)
    pred, B = new(ne, C), new(ne, C, D)
    crit = torch.empty(ne, C, dtype=torch.int64, device="cuda")
    status = torch.zeros(3, dtype=torch.int32, device="cuda")
    ws = torch.empty(lib.dsmil_forward_bags_models_train_dev_workspace_bytes(ps, 3, nbs, max_rows), dtype=torch.uint8,
                     device="cuda")
    rc = lib.dsmil_forward_bags_models_train_dev(ps, 3, xs.data_ptr(), Ns.data_ptr(), nbs, max_rows,
                                                 classes.data_ptr(), pred.data_ptr(), A.data_ptr(), B.data_ptr(),
                                                 crit.data_ptr(), sQ.data_ptr(), sH.data_ptr(), status.data_ptr(),
                                                 ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    assert status.tolist() == [0, 2, 0]
    _same([t[:4] + (t[4],) for t in [_live((classes, pred, A, B, crit), lists, max_rows)[i] for i in (0, 2)]],
          [clean[0], clean[2]], "misaligned")
    assert bool(torch.isfinite(pred).all()) and crit[2:5].eq(0).all()


def _fill(g, slots_of, Ns_at, labels_at, lists, D, C, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    for m, ns in enumerate(lists):
        for b, n in enumerate(ns):
            slots_of(m)[b, :max(n, 0)] = torch.rand(max(n, 0), D, generator=gen, device="cuda")
        Ns_at(m).copy_(torch.tensor(ns, dtype=torch.int64, device="cuda"))
        labels_at(m).copy_((torch.rand(len(ns), C, generator=gen, device="cuda") > 0.5).float())


@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_fold_graph_matches_each_folds_own_graph_and_guards_per_fold(opt):
    D, C, max_rows, nbs = 512, 2, 2000, [2, 1, 3]
    ps = [orc.random_params(D, C, seed=61 + m) for m in range(3)]
    fold, alone = [build_net(p).train() for p in ps], [build_net(p).train() for p in ps]
    o_f, o_a = [_opt(opt, n) for n in fold], [_opt(opt, n) for n in alone]
    crit = torch.nn.BCEWithLogitsLoss()
    fg = FoldTrainStepGraph(fold, crit, o_f, nbs, max_rows)
    gs = [TrainStepGraph(alone[m], crit, o_a[m], nbs[m], max_rows) for m in range(3)]
    bag0 = [0, 2, 3]
    steps = [[[129, 2000], [1], [127, 128, 700]], [[5, 64], [1999], [300, 1, 1]], [[2000, 2000], [640], [0, 50, 60]],
             [[77, 1300], [128], [900, 33, 257]]]
    for t, lists in enumerate(steps):
        refused = [m for m, ns in enumerate(lists) if min(ns) < 1]
        _fill(fg, lambda m: fg.slots[m], lambda m: fg.Ns[bag0[m]:bag0[m] + nbs[m]],
              lambda m: fg.labels[bag0[m]:bag0[m] + nbs[m]], lists, D, C, 20 + t)
        _fill(None, lambda m: gs[m].slots, lambda m: gs[m].Ns, lambda m: gs[m].labels, lists, D, C, 20 + t)
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
    assert fg.status.tolist() == [0, 0, 1]
    assert all(g.status.item() == 0 for g in gs)


@pytest.mark.parametrize("k", [1, 4])
def test_graph_epochs_match_each_fold_trained_alone_and_the_eager_fold_epoch(k):
    D, C = 512, 2
    for drop in (0.0, 0.3):
        store = _store(D, C, [n if n > 1 or drop == 0 else 2 for n in STORE_NS])
        rng = np.random.default_rng(k)
        folds = [rng.permutation(len(store))[:n].tolist() for n in (9, 4, 13, 1, 7)]
        ps = [orc.random_params(D, C, seed=31 + m) for m in range(5)]
        nets = {w: [build_net(p) for p in ps] for w in ("graph", "eager", "alone")}
        opts = {w: [_opt("sgd", n) for n in ns] for w, ns in nets.items()}
        gens = {w: [torch.Generator(device="cuda").manual_seed(5 + m) for m in range(5)] for w in nets}
        crit = torch.nn.BCEWithLogitsLoss()
        for epoch in range(2):
            orders = [np.random.default_rng(10 * epoch + m).permutation(f).tolist() for m, f in enumerate(folds)]
            got = feed.train_epoch_models(nets["graph"], store, folds, crit, opts["graph"], dropout_patch=drop,
                                          orders=orders, generators=gens["graph"], bags_per_step=k, graph=True)
            eager = feed.train_epoch_models(nets["eager"], store, folds, crit, opts["eager"], dropout_patch=drop,
                                            orders=orders, generators=gens["eager"], bags_per_step=k)
            assert got == eager, (k, drop, epoch)
            for m in range(5):
                want = feed.train_epoch(nets["alone"][m], store, crit, opts["alone"][m], dropout_patch=drop,
                                        order=orders[m], generator=gens["alone"][m], bags_per_step=k, graph=True)
                assert got[m] == want, (k, drop, epoch, m, got[m], want)
        for m in range(5):
            for (name, a), b, c in zip(nets["graph"][m].named_parameters(), nets["alone"][m].parameters(),
                                       nets["eager"][m].parameters()):
                assert torch.equal(a, b) and torch.equal(a, c), (k, drop, m, name)
