"""The generic batched forward (identity v off the tensor-core batch) and the graphs it opens to those shapes: the eager
dsmil_forward_bags against per-bag dsmil_forward, the dev calls against the eager calls (directly and replayed from one
capture), train_epoch / eval_epoch / the classic-MIL drivers with graph=True against their eager epochs, refusal, and
the goldens at the oracle tolerances."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_to_max
from helpers import build_net
from oracle import dsmil_oracle as orc
from dsmil_wsi_b200 import _lib, feed
from dsmil_wsi_b200 import functional as Fn
from dsmil_wsi_b200.sharded import milnet_params

pytestmark = pytest.mark.gpu

# (D, C, nonlinear): the classic-MIL sizes, linear q, C above 4, D above 2048 (these two with the tensor-core phase 1)
# and D = 7 (scalar loads everywhere)
SHAPES = [(166, 1, True), (230, 1, True), (512, 3, False), (96, 2, True), (1024, 6, True), (4096, 2, True),
          (7, 1, False)]
ids = [f"D{d}C{c}{'' if nl else 'lin'}" for d, c, nl in SHAPES]
# ragged: N = 1, the kAttendRows (32) edges, and the record cap kSplits * kAttendRows = 9472 rows and one more
SIZES = [[1, 31, 32, 33, 200], [9472, 1, 65, 9473, 7], [3, 1, 2, 1, 5]]
MAXR = 9473


def _net(D, C_, nonlinear, seed):
    return build_net(orc.random_params(D, C_, seed=seed, nonlinear=nonlinear))


def _bags(Ns, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.rand(n, D, device="cuda", generator=g) for n in Ns]


def _same(got, want, what):
    assert got.shape == want.shape and torch.equal(got, want), (what, float((got.float() - want.float()).abs().max()))


@pytest.mark.parametrize("D,C_,nonlinear", SHAPES, ids=ids)
def test_forward_bags_equals_per_bag_forward(D, C_, nonlinear):
    lib = _lib.load()
    net = _net(D, C_, nonlinear, D + C_).eval()
    assert lib.dsmil_shard_bags_supported(Fn.ParamPack(*milnet_params(net)).ref) == 0
    xs = _bags(SIZES[1][:3] + [200], D, 1)
    # a bag 4 bytes past a 16-byte boundary: float4 loads stop (k_scores MODE 0), the bits do not change
    raw = torch.rand(40 * D + 1, device="cuda")
    xs.append(raw[1:].view(40, D))
    with torch.no_grad():
        outs = net.forward_bags(xs)
        for b, x in enumerate(xs):
            for u, v in zip(outs[b], net(x)):
                _same(u, v, (b, x.shape[0]))


class Dev:
    """dsmil_forward_bags_train_dev + dsmil_backward_bags_dev over static slots [nb, max_rows, D]."""

    def __init__(self, lib, P, nb, max_rows):
        self.lib, self.P, self.nb, self.max_rows = lib, P, nb, max_rows
        rows = nb * max_rows
        self.slots = torch.zeros(nb, max_rows, P.D, device="cuda")
        self.xs = torch.tensor([self.slots[b].data_ptr() for b in range(nb)], dtype=torch.int64, device="cuda")
        self.Ns = torch.ones(nb, dtype=torch.int64, device="cuda")
        self.status = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.dc, self.dp = torch.zeros(rows, P.C, device="cuda"), torch.zeros(nb, P.C, device="cuda")
        new = lambda *s: torch.full(s, float("nan"), device="cuda")
        self.out = {"classes": new(rows, P.C), "A": new(rows, P.C), "Q": new(rows, 128),
                    "H1": new(rows, 128) if P.nonlinear else None, "pred": new(nb, P.C), "B": new(nb, P.C, P.D),
                    "crit": torch.full((nb, P.C), -1, dtype=torch.int64, device="cuda")}
        self.g = {n: torch.full_like(t, float("nan")) for n, t in zip(Fn.PARAM_NAMES, P.tensors) if t is not None}
        self.wf = torch.empty(lib.dsmil_generic_forward_bags_train_dev_workspace_bytes(P.ref, nb, max_rows),
                              dtype=torch.uint8, device="cuda")
        self.wb = torch.empty(lib.dsmil_generic_backward_bags_dev_workspace_bytes(P.ref, nb, max_rows), dtype=torch.uint8,
                              device="cuda")

    def run(self):
        lib, P, o = self.lib, self.P, self.out
        ptr = lambda t: None if t is None else t.data_ptr()
        st = torch.cuda.current_stream().cuda_stream
        G = _lib.DsmilGrads(*[ptr(self.g.get(n)) for n in Fn.PARAM_NAMES], None)
        _lib.check(lib.dsmil_generic_forward_bags_train_dev(P.ref, ptr(self.xs), ptr(self.Ns), self.nb, self.max_rows,
                                                    ptr(o["classes"]), ptr(o["pred"]), ptr(o["A"]), ptr(o["B"]),
                                                    ptr(o["crit"]), ptr(o["Q"]), ptr(o["H1"]), ptr(self.status),
                                                    ptr(self.wf), self.wf.numel(), st), "forward dev")
        _lib.check(lib.dsmil_generic_backward_bags_dev(P.ref, ptr(self.xs), ptr(self.Ns), self.nb, self.max_rows, ptr(o["Q"]),
                                               ptr(o["H1"]), ptr(o["A"]), ptr(o["B"]), ptr(o["crit"]), ptr(self.dc),
                                               ptr(self.dp), None, None, C.byref(G), ptr(self.status), ptr(self.wb),
                                               self.wb.numel(), st), "backward dev")
        self._G = G


def _eager(lib, P, xs, dc, dp):
    """The eager dsmil_forward_bags_train + dsmil_backward_bags on the same bags and upstream gradients."""
    nb, Ns = len(xs), [int(x.shape[0]) for x in xs]
    rows = sum(Ns)
    new = lambda *s: torch.full(s, float("nan"), device="cuda")
    o = {"classes": new(rows, P.C), "A": new(rows, P.C), "Q": new(rows, 128), "H1": new(rows, 128) if P.nonlinear else None,
         "pred": new(nb, P.C), "B": new(nb, P.C, P.D), "crit": torch.full((nb, P.C), -1, dtype=torch.int64, device="cuda")}
    g = {n: torch.full_like(t, float("nan")) for n, t in zip(Fn.PARAM_NAMES, P.tensors) if t is not None}
    ptr = lambda t: None if t is None else t.data_ptr()
    G = _lib.DsmilGrads(*[ptr(g.get(n)) for n in Fn.PARAM_NAMES], None)
    c_X, c_N = (C.c_void_p * nb)(*[x.data_ptr() for x in xs]), (C.c_int64 * nb)(*Ns)
    ws = torch.empty(max(lib.dsmil_forward_bags_train_workspace_bytes(P.ref, c_N, nb),
                         lib.dsmil_backward_bags_workspace_bytes(P.ref, c_N, nb, 0)), dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.dsmil_forward_bags_train(P.ref, c_X, c_N, nb, ptr(o["classes"]), ptr(o["pred"]), ptr(o["A"]),
                                            ptr(o["B"]), ptr(o["crit"]), ptr(o["Q"]), ptr(o["H1"]), ptr(ws), ws.numel(),
                                            st), "forward")
    _lib.check(lib.dsmil_backward_bags(P.ref, c_X, c_N, nb, ptr(o["Q"]), ptr(o["H1"]), ptr(o["A"]), ptr(o["B"]),
                                       ptr(o["crit"]), ptr(dc), ptr(dp), None, None, C.byref(G), ptr(ws), ws.numel(),
                                       st), "backward")
    return o, g


def _check_dev(dev, Ns, seed):
    lib, P = dev.lib, dev.P
    g = torch.Generator(device="cuda").manual_seed(seed)
    for b, n in enumerate(Ns):
        dev.slots[b, :n].uniform_(0, 1, generator=g)
        dev.Ns[b].fill_(n)
    total = sum(Ns)
    dc = torch.randn(total, P.C, device="cuda", generator=g)
    dp = torch.randn(len(Ns), P.C, device="cuda", generator=g)
    dev.dc[:total].copy_(dc)
    dev.dp.copy_(dp)
    return dc, dp


@pytest.mark.parametrize("D,C_,nonlinear", SHAPES, ids=ids)
def test_dev_calls_replayed_from_one_capture_equal_eager_calls(D, C_, nonlinear):
    lib = _lib.load()
    P = Fn.ParamPack(*milnet_params(_net(D, C_, nonlinear, 7 + D)))
    dev = Dev(lib, P, len(SIZES[0]), MAXR)
    _check_dev(dev, SIZES[0], 0)
    dev.run()                                  # warm-up outside the capture
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        dev.run()
    for i, Ns in enumerate(SIZES):
        dc, dp = _check_dev(dev, Ns, 10 + i)
        graph.replay()
        want, gw = _eager(lib, P, [dev.slots[b, :n] for b, n in enumerate(Ns)], dc, dp)
        total = sum(Ns)
        for k, v in want.items():
            if v is not None:
                _same(dev.out[k][:total] if k in ("classes", "A", "Q", "H1") else dev.out[k], v, (Ns, k))
        for k, v in gw.items():
            _same(dev.g[k], v, (Ns, "g" + k))
    assert int(dev.status) == 0


@pytest.mark.parametrize("D,C_,nonlinear", SHAPES, ids=ids)
def test_forward_bags_dev_equals_eager(D, C_, nonlinear):
    net = _net(D, C_, nonlinear, 3 + D).eval()
    params = milnet_params(net)
    for i, Ns in enumerate(SIZES):
        xs = _bags(Ns, D, 30 + i)
        ptrs = torch.tensor([x.data_ptr() for x in xs], dtype=torch.int64, device="cuda")
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        classes, pred, A, B, crit = Fn.mil_forward_bags_dev(ptrs, torch.tensor(Ns, device="cuda"), status, MAXR,
                                                            params)
        with torch.no_grad():
            ref = net.forward_bags(xs)
        total = sum(Ns)
        for got, want in zip((classes[:total], pred, A[:total], B), ref.packed):
            _same(got, want, (Ns,))
        for b, x in enumerate(xs):                   # the critical rows: the arg-max of each bag's own scores
            _same(crit[b], ref[b][0].argmax(0), (Ns, "crit", b))
        assert int(status) == 0


def _store(D, C_, Ns, seed=4):
    store = feed.DeviceBagStore(D)
    rng = np.random.default_rng(seed)
    for i, n in enumerate(Ns):
        store.add_bag(torch.from_numpy(orc.synthetic_bag(int(n), D, 70 + i)),
                      torch.from_numpy((rng.random(C_) > 0.5).astype(np.float32)))
    return store


def _opt(kind, net):
    if kind == "sgd":
        return torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
    return torch.optim.Adam(net.parameters(), lr=1e-3, betas=(0.5, 0.9), weight_decay=1e-3, capturable=True)


def _eager_minibatch_epoch(net, store, crit, opt, order, k, drop, gen):
    """train_epoch's minibatch step (forward_bags(grad=True), one backward, one step), at any k including 1."""
    total = 0.0
    for s in range(0, len(order), k):
        group = order[s:s + k]
        opt.zero_grad()
        xs = [feed.dropout_patches(store.bags[i][0], 1 - drop, gen) for i in group]
        labels = torch.cat([store.bags[i][1].view(1, -1) for i in group])
        bag_prediction, max_prediction = feed._group_predictions(net.forward_bags(xs, grad=True))
        loss = feed.minibatch_loss(crit, bag_prediction, max_prediction, labels)
        loss.backward()
        opt.step()
        total += float(loss) * len(group)
    return total / len(order)


MUSK_NS = [2 + (7 * i) % 39 for i in range(90)]          # about 90 bags of 2 to 40 rows


@pytest.mark.parametrize("opt", ["sgd", "adam"])
@pytest.mark.parametrize("D,C_,nonlinear", [(166, 1, True), (512, 3, False)], ids=["D166C1", "D512C3lin"])
def test_graph_epochs_match_eager_minibatch_epochs(D, C_, nonlinear, opt):
    p = orc.random_params(D, C_, seed=31, nonlinear=nonlinear)
    store = _store(D, C_, [3, 40, 2, 33, 700, 31, 9, 64, 5, 2, 120, 17, 32, 4])
    crit = torch.nn.BCEWithLogitsLoss()
    for k in (1, 4):
        for drop in (0.0, 0.3):
            nets = [build_net(p), build_net(p)]
            opts = [_opt(opt, n) for n in nets]
            gens = [torch.Generator(device="cuda").manual_seed(5) for _ in nets]
            order = np.random.default_rng(k).permutation(len(store)).tolist()
            le = _eager_minibatch_epoch(nets[0], store, crit, opts[0], order, k, drop, gens[0])
            lg = feed.train_epoch(nets[1], store, crit, opts[1], dropout_patch=drop, order=order, generator=gens[1],
                                  bags_per_step=k, graph=True, generic=True)
            assert abs(le - lg) <= 1e-6 * max(1.0, abs(le)), (k, drop, le, lg)   # the host sums differ in order
            for (name, a), b in zip(nets[0].named_parameters(), nets[1].parameters()):
                assert torch.equal(a, b), (opt, k, drop, name, float((a - b).abs().max()))


def test_mil_epochs_with_graphs_match_eager():
    D = 166
    p = orc.random_params(D, 1, seed=12)
    store = _store(D, 1, MUSK_NS, seed=8)
    crit = torch.nn.BCEWithLogitsLoss()
    nets = [build_net(p), build_net(p)]
    opts = [torch.optim.SGD(n.parameters(), lr=0.01, momentum=0.9) for n in nets]
    order = np.random.default_rng(3).permutation(len(store)).tolist()
    torch.manual_seed(0)                          # the row permutations of dropout_patches draw from it
    le = _eager_minibatch_epoch(nets[0], store, crit, opts[0], order, 1, 0.0, None)
    torch.manual_seed(0)
    lg = feed.mil_epoch_train(nets[1], store, crit, opts[1], order=order, graph=True)
    assert abs(le - lg) <= 1e-6 * max(1.0, abs(le))
    for a, b in zip(nets[0].parameters(), nets[1].parameters()):
        assert torch.equal(a, b)
    te = feed.mil_epoch_test(nets[0], store, crit)
    tg = feed.mil_epoch_test(nets[1], store, crit, graph=True)
    assert te[0] == tg[0] and te[1] == tg[1]
    for a, b in zip(te[2], tg[2]):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("D,C_,nonlinear", [(230, 1, True), (1024, 6, True), (7, 1, False)],
                         ids=["D230C1", "D1024C6", "D7C1lin"])
def test_eval_epoch_graph_equals_eager(D, C_, nonlinear):
    net = _net(D, C_, nonlinear, 2)
    store = _store(D, C_, [40, 1, 2, 300, 33, 9472, 17, 5, 64], seed=6)
    crit = torch.nn.BCEWithLogitsLoss()
    for average in (False, True):
        e = feed.eval_epoch(net, store, crit, average=average, bags_per_launch=4)
        g = feed.eval_epoch(net, store, crit, average=average, bags_per_launch=4, graph=True, generic=True)
        assert e[0] == g[0] and np.array_equal(e[1], g[1]) and np.array_equal(e[2], g[2])


def test_refused_batches_then_a_correct_one():
    """N = 0, N > max_rows and a misaligned bag (4 bytes off at D % 4 == 0): status 1 + b, NaN loss, parameters and
    optimizer state kept, finite stand-in outputs, and the next batch steps as if the refused one had not been fed."""
    from dsmil_wsi_b200.train_graph import TrainStepGraph
    D, C_, nb, cap = 96, 2, 4, 100
    p = orc.random_params(D, C_, seed=17)
    store = _store(D, C_, [30, 1, 100, 64])
    crit = torch.nn.BCEWithLogitsLoss()
    runs = []
    for refuse in (True, False):
        net = build_net(p)
        g = TrainStepGraph(net, crit, _opt("adam", net), nb, cap, generic=True)
        for b, (f, _) in enumerate(store.bags):
            g.slots[b, :f.shape[0]].copy_(f)
        g.labels.copy_(torch.cat([lab.view(1, -1) for _, lab in store.bags]))
        if refuse:
            for bad, n in ((2, 0), (1, cap + 1)):
                for b, (f, _) in enumerate(store.bags):
                    g.Ns[b].fill_(n if b == bad else f.shape[0])
                before = [t.detach().clone() for t in g._kept]
                g.status.zero_()
                loss = float(g.step())
                assert int(g.status) == bad + 1 and np.isnan(loss)
                for a, b in zip(g._kept, before):
                    assert torch.equal(a, b)
            g.status.zero_()
        for b, (f, _) in enumerate(store.bags):
            g.Ns[b].fill_(f.shape[0])
        runs.append((float(g.step()), [t.detach().clone() for t in net.parameters()]))
        assert int(g.status) == 0
    assert runs[0][0] == runs[1][0]
    for a, b in zip(runs[0][1], runs[1][1]):
        assert torch.equal(a, b)
    # the inference dev call on a misaligned bag: refused, finite stand-in outputs
    net = build_net(p).eval()
    raw = torch.rand(10 * D + 1, device="cuda")
    xs = [torch.rand(5, D, device="cuda"), raw[1:].view(10, D)]
    ptrs = torch.tensor([x.data_ptr() for x in xs], dtype=torch.int64, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = Fn.mil_forward_bags_dev(ptrs, torch.tensor([5, 10], device="cuda"), status, 16, milnet_params(net))
    assert int(status) == 2
    for t in out[:4]:
        assert torch.isfinite(t).all()
    assert int(out[4].min()) == 0 and int(out[4].max()) == 0


@pytest.mark.parametrize("name", ["musk_d166_n7", "eleph_d230_n33", "lin_d512_c3"])
def test_graph_outputs_on_the_goldens(name):
    from dsmil_wsi_b200.infer_graph import ForwardBagsGraph
    g, p, X = load_golden(name)
    net = build_net(p).eval()
    x = torch.from_numpy(X).cuda()
    graph = ForwardBagsGraph(net, 1, X.shape[0] + 3, generic=True)
    out = graph.run([x])
    t = orc.forward(X, p)
    classes, pred, A, B = out[0]
    assert rel_to_max(classes.cpu().numpy(), t.classes) < 2e-6
    assert rel_to_max(A.cpu().numpy(), t.A) < 2e-5
    assert rel_to_max(B.cpu().numpy(), t.B) < 1e-5
    assert np.array_equal(out.crit[0].cpu().numpy(), t.idx)
    with torch.no_grad():
        for u, v in zip(out[0], net(x)):
            _same(u, v, name)
