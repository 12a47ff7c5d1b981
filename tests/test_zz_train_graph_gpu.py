"""The minibatch training step as one CUDA graph over ragged bags: the capture-safe entry points against the eager
dsmil_forward_bags_train / dsmil_backward_bags (bit for bit, called directly and replayed from one capture), and
feed.train_epoch(graph=True) against the eager minibatch epoch and the per-bag loop."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import build_net, caller_loss
from oracle import dsmil_oracle as orc
from dsmil_wsi_b200 import _lib, feed
from dsmil_wsi_b200.functional import ParamPack

pytestmark = pytest.mark.gpu

NAMES = ("Wi", "bi", "W1", "b1", "W2", "b2", "Wf", "bf")


def _pack(p):
    net = build_net(p)
    ic, bc = net.i_classifier, net.b_classifier
    lin = ic._linear()
    W1, b1, W2, b2 = bc._q_params()
    return ParamPack(lin.weight, lin.bias, W1, b1, W2, b2, None, None, bc.fcc.weight, bc.fcc.bias)


class Buffers:
    """Outputs, saved activations and gradients of one batched training call pair, sized for `rows` packed rows."""

    def __init__(self, P, nb, rows):
        new = lambda *s: torch.full(s, float("nan"), device="cuda")
        self.classes, self.A, self.Q, self.H1 = new(rows, P.C), new(rows, P.C), new(rows, 128), new(rows, 128)
        self.pred, self.B = new(nb, P.C), new(nb, P.C, P.D)
        self.crit = torch.full((nb, P.C), -1, dtype=torch.int64, device="cuda")
        self.g = {n: torch.full_like(t, float("nan")) for n, t in zip(("Wi", "bi", "W1", "b1", "W2", "b2"),
                                                                      P.tensors[:6])}
        self.g["Wf"], self.g["bf"] = torch.full_like(P.tensors[8], float("nan")), torch.full_like(P.tensors[9], float("nan"))
        self.G = _lib.DsmilGrads(*[self.g[n].data_ptr() for n in ("Wi", "bi", "W1", "b1", "W2", "b2")], None, None,
                                 self.g["Wf"].data_ptr(), self.g["bf"].data_ptr(), None)

    def live(self, total):
        return {"classes": self.classes[:total], "A": self.A[:total], "Q": self.Q[:total], "H1": self.H1[:total],
                "pred": self.pred, "B": self.B, "crit": self.crit, **{"g" + k: v for k, v in self.g.items()}}


def _eager(lib, P, xs, dc, dp):
    nb, Ns = len(xs), [int(x.shape[0]) for x in xs]
    b = Buffers(P, nb, sum(Ns))
    c_X, c_N = (C.c_void_p * nb)(*[x.data_ptr() for x in xs]), (C.c_int64 * nb)(*Ns)
    ws = torch.empty(max(lib.dsmil_forward_bags_train_workspace_bytes(P.ref, c_N, nb),
                         lib.dsmil_backward_bags_workspace_bytes(P.ref, c_N, nb, 0)), dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.dsmil_forward_bags_train(P.ref, c_X, c_N, nb, b.classes.data_ptr(), b.pred.data_ptr(),
                                            b.A.data_ptr(), b.B.data_ptr(), b.crit.data_ptr(), b.Q.data_ptr(),
                                            b.H1.data_ptr(), ws.data_ptr(), ws.numel(), st), "forward")
    _lib.check(lib.dsmil_backward_bags(P.ref, c_X, c_N, nb, b.Q.data_ptr(), b.H1.data_ptr(), b.A.data_ptr(),
                                       b.B.data_ptr(), b.crit.data_ptr(), dc.data_ptr(), dp.data_ptr(), None, None,
                                       C.byref(b.G), ws.data_ptr(), ws.numel(), st), "backward")
    return b.live(sum(Ns))


class Dev:
    """The two dev calls over static buffers: slots [nb, max_rows, D], Ns, status, d_classes [nb*max_rows, C], d_pred."""

    def __init__(self, lib, P, nb, max_rows):
        self.lib, self.P, self.nb, self.max_rows = lib, P, nb, max_rows
        self.slots = torch.zeros(nb, max_rows, P.D, device="cuda")
        self.xs = torch.tensor([self.slots[b].data_ptr() for b in range(nb)], dtype=torch.int64, device="cuda")
        self.Ns = torch.ones(nb, dtype=torch.int64, device="cuda")
        self.status = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.dc = torch.zeros(nb * max_rows, P.C, device="cuda")
        self.dp = torch.zeros(nb, P.C, device="cuda")
        self.b = Buffers(P, nb, nb * max_rows)
        self.wf = torch.empty(lib.dsmil_forward_bags_train_dev_workspace_bytes(P.ref, nb, max_rows), dtype=torch.uint8,
                              device="cuda")
        self.wb = torch.empty(lib.dsmil_backward_bags_dev_workspace_bytes(P.ref, nb, max_rows), dtype=torch.uint8,
                              device="cuda")

    def load(self, Ns, dc, dp):
        for b, n in enumerate(Ns):
            self.Ns[b].fill_(n)
        self.dc[:dc.shape[0]].copy_(dc)
        self.dp.copy_(dp)

    def run(self):
        lib, P, b = self.lib, self.P, self.b
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(lib.dsmil_forward_bags_train_dev(P.ref, self.xs.data_ptr(), self.Ns.data_ptr(), self.nb,
                                                    self.max_rows, b.classes.data_ptr(), b.pred.data_ptr(),
                                                    b.A.data_ptr(), b.B.data_ptr(), b.crit.data_ptr(), b.Q.data_ptr(),
                                                    b.H1.data_ptr(), self.status.data_ptr(), self.wf.data_ptr(),
                                                    self.wf.numel(), st), "forward dev")
        _lib.check(lib.dsmil_backward_bags_dev(P.ref, self.xs.data_ptr(), self.Ns.data_ptr(), self.nb, self.max_rows,
                                               b.Q.data_ptr(), b.H1.data_ptr(), b.A.data_ptr(), b.B.data_ptr(),
                                               b.crit.data_ptr(), self.dc.data_ptr(), self.dp.data_ptr(), None, None,
                                               C.byref(b.G), self.status.data_ptr(), self.wb.data_ptr(),
                                               self.wb.numel(), st), "backward dev")


def _fill(dev, Ns, seed):
    """Random features into the slots, and random upstream gradients for classes and pred."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    for b, n in enumerate(Ns):
        dev.slots[b, :n].uniform_(0, 1, generator=g)
    dc = torch.randn(sum(Ns), dev.P.C, device="cuda", generator=g)
    dp = torch.randn(len(Ns), dev.P.C, device="cuda", generator=g)
    return dc, dp


def _same(got, want, what):
    for k, v in want.items():
        assert torch.equal(got[k], v), (what, k, float((got[k].float() - v.float()).abs().max()))


MAXR = 3000
BATCHES = [[1, 127, 128, 129, MAXR], [MAXR, 129, 1, 128, 127], [3, 1, 2, 1, 5]]   # the last: sum N << capacity


@pytest.mark.parametrize("D,C_", [(512, 1), (512, 2), (512, 4), (1024, 4), (1536, 1)])
def test_dev_calls_match_eager_calls_bit_for_bit(D, C_):
    lib = _lib.load()
    P = _pack(orc.random_params(D, C_, seed=D + C_))
    dev = Dev(lib, P, len(BATCHES[0]), MAXR)
    for i, Ns in enumerate(BATCHES):
        dc, dp = _fill(dev, Ns, seed=i)
        dev.load(Ns, dc, dp)
        dev.run()
        want = _eager(lib, P, [dev.slots[b, :n] for b, n in enumerate(Ns)], dc, dp)
        _same(dev.b.live(sum(Ns)), want, (D, C_, Ns))
    assert int(dev.status) == 0


def test_one_capture_replays_every_batch_like_the_eager_calls():
    lib = _lib.load()
    P = _pack(orc.random_params(512, 2, seed=3))
    nb = 5
    dev = Dev(lib, P, nb, MAXR)
    dev.load(BATCHES[0], *_fill(dev, BATCHES[0], seed=9))
    dev.run()                                  # warm-up outside the capture
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        dev.run()
    torch.cuda.synchronize()
    for i, Ns in enumerate([[1] * nb, [MAXR, 64, 4096 % MAXR, 1, 300], [129, 128, 127, 2, 1], BATCHES[0]]):
        dc, dp = _fill(dev, Ns, seed=20 + i)
        dev.load(Ns, dc, dp)
        before = _lib.launch_count()
        graph.replay()
        torch.cuda.synchronize()
        assert _lib.launch_count() == before
        want = _eager(lib, P, [dev.slots[b, :n] for b, n in enumerate(Ns)], dc, dp)
        _same(dev.b.live(sum(Ns)), want, Ns)
    assert int(dev.status) == 0


def _store(D, C_, Ns, seed=4):
    store = feed.DeviceBagStore(D)
    rng = np.random.default_rng(seed)
    for i, n in enumerate(Ns):
        store.add_bag(torch.from_numpy(orc.synthetic_bag(int(n), D, 70 + i)),
                      torch.from_numpy((rng.random(C_) > 0.5).astype(np.float32)))
    return store


# about 21 bags from 2 to 12 000 rows (2: a bag that keeps one row under 30 % patch dropout)
STORE_NS = [2, 12000, 1, 129, 5000, 128, 7, 9000, 127, 300, 2500, 64, 11000, 3, 800, 6000, 1500, 256, 40, 3300, 12]


def _opt(kind, net):
    if kind == "sgd":
        return torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
    return torch.optim.Adam(net.parameters(), lr=1e-3, betas=(0.5, 0.9), weight_decay=1e-3, capturable=True)


@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_graph_epochs_match_eager_minibatch_epochs(opt):
    D, C_ = 512, 2
    p = orc.random_params(D, C_, seed=31)
    for k in (4, 16):
        for drop in (0.0, 0.3):
            # with 30 % patch dropout a 1-row bag would be empty (the eager step raises too)
            store = _store(D, C_, [n if n > 1 or drop == 0 else 2 for n in STORE_NS])
            nets = [build_net(p), build_net(p)]
            opts = [_opt(opt, n) for n in nets]
            crit = torch.nn.BCEWithLogitsLoss()
            gens = [torch.Generator(device="cuda").manual_seed(5) for _ in nets]
            for epoch in range(2):
                order = np.random.default_rng(epoch).permutation(len(store)).tolist()
                le = feed.train_epoch(nets[0], store, crit, opts[0], dropout_patch=drop, order=order,
                                      generator=gens[0], bags_per_step=k)
                lg = feed.train_epoch(nets[1], store, crit, opts[1], dropout_patch=drop, order=order,
                                      generator=gens[1], bags_per_step=k, graph=True)
                assert le == lg, (opt, k, drop, epoch, le, lg)
            for (name, a), b in zip(nets[0].named_parameters(), nets[1].parameters()):
                assert torch.equal(a, b), (opt, k, drop, name, float((a - b).abs().max()))


def test_graph_k1_is_within_the_per_bag_loop_tolerances():
    D, C_, lr = 512, 2, 0.05
    p = orc.random_params(D, C_, seed=12)
    store = _store(D, C_, [50, 3000, 129, 700, 1, 2000])
    order = list(range(len(store)))
    net, ref = build_net(p), build_net(p)
    crit = torch.nn.BCEWithLogitsLoss()
    loss = feed.train_epoch(net, store, crit, torch.optim.SGD(net.parameters(), lr=lr), order=order,
                            generator=torch.Generator(device="cuda").manual_seed(1), bags_per_step=1, graph=True)
    # the per-bag loop, with its gradients' sizes for the tolerance
    ref.train()
    opt = torch.optim.SGD(ref.parameters(), lr=lr)
    gen = torch.Generator(device="cuda").manual_seed(1)
    total, gsum = 0.0, {}
    for i in order:
        opt.zero_grad()
        feats, label = store.bags[i]
        c, pr, _, _ = ref(feed.dropout_patches(feats, 1.0, gen))
        l = caller_loss(c, pr, label)
        l.backward()
        total += float(l.detach())
        for name, v in ref.named_parameters():
            gsum[name] = gsum.get(name, 0.0) + float(v.grad.abs().max())
        opt.step()
    want = total / len(order)
    assert abs(loss - want) <= 1e-5 * max(1.0, abs(want))
    eps = torch.finfo(torch.float32).eps
    for (name, a), b in zip(net.named_parameters(), ref.parameters()):
        # test_zz_bags_train_gpu's gradient tolerances x lr, plus one rounding of the parameter per step
        tol = (2e-3 if ".q." in name else 5e-4) * lr * gsum[name] + 3 * len(order) * eps * float(b.detach().abs().max())
        d = float((a - b).detach().abs().max())
        assert d <= tol, (name, d, tol)


def test_graph_epochs_are_deterministic():
    D, C_ = 512, 2
    p = orc.random_params(D, C_, seed=8)
    store = _store(D, C_, STORE_NS[:9])
    runs = []
    for _ in range(2):
        net = build_net(p)
        opt = _opt("adam", net)
        loss = feed.train_epoch(net, store, torch.nn.BCEWithLogitsLoss(), opt, order=list(range(9)),
                                generator=torch.Generator(device="cuda").manual_seed(3), bags_per_step=4, graph=True)
        runs.append((loss, [t.detach().clone() for t in net.parameters()]))
    assert runs[0][0] == runs[1][0]
    for a, b in zip(runs[0][1], runs[1][1]):
        assert torch.equal(a, b)


def test_a_refused_batch_reports_its_status_and_leaves_the_model_alone():
    """An empty bag (N = 0, e.g. all rows dropped by the caller) in a batch fed straight to a TrainStepGraph: the
    status names the bag, the loss is NaN, parameters and optimizer state keep their bits, and the next accepted batch
    steps exactly as if the refused one had never been fed."""
    from dsmil_wsi_b200.train_graph import TrainStepGraph
    D, C_, nb, cap = 512, 2, 4, 600
    p = orc.random_params(D, C_, seed=17)
    store = _store(D, C_, [300, 1, 600, 129])
    crit = torch.nn.BCEWithLogitsLoss()
    runs = []
    for refuse in (True, False):
        net = build_net(p)
        opt = _opt("adam", net)
        g = TrainStepGraph(net, crit, opt, nb, cap)
        labels = torch.cat([lab.view(1, -1) for _, lab in store.bags])
        for b, (f, _) in enumerate(store.bags):
            g.slots[b, :f.shape[0]].copy_(f)
        g.labels.copy_(labels)
        if refuse:
            for b, (f, _) in enumerate(store.bags):
                g.Ns[b].fill_(0 if b == 2 else f.shape[0])
            before = [t.detach().clone() for t in g._kept]
            loss = float(g.step())
            assert int(g.status) == 3 and np.isnan(loss)
            for a, b in zip(g._kept, before):
                assert torch.equal(a, b)
        for b, (f, _) in enumerate(store.bags):
            g.Ns[b].fill_(f.shape[0])
        runs.append((float(g.step()), [t.detach().clone() for t in net.parameters()]))
        assert int(g.status) == (3 if refuse else 0)
    assert runs[0][0] == runs[1][0]
    for a, b in zip(runs[0][1], runs[1][1]):
        assert torch.equal(a, b)
