"""Models with a value network (passing_v) as CUDA graphs: the capture-safe value calls against the eager value calls,
bit for bit, their refusals, TrainStepGraph(value=True), the value=True epochs of feed and the inference graphs."""

import numpy as np
import pytest
import torch

from conftest import rel_to_max
from oracle import dsmil_oracle as orc
from test_zz_value_train_gpu import _torch_params

pytestmark = pytest.mark.gpu

# (D, C, nonlinear q)
SHAPES = [(512, 2, True), (2048, 2, True), (166, 1, True), (230, 3, False), (96, 5, True)]
MAX_ROWS = 300
BATCHES = [[1, 127, 128, 129, MAX_ROWS, 40], [MAX_ROWS] * 6, [5, 1, 2, 3, 257, 7]]


def _bag(n, D, seed):
    return torch.from_numpy(orc.synthetic_bag(n, D, seed)).cuda()


def _live(params):
    return [t for t in params if t is not None]


class _DevPair:
    """One capture of the dev forward + backward (MILValueBagsDevFn and its autograd backward) over static slots."""

    def __init__(self, params, nb, D, C_, distinct):
        from dsmil_wsi_b200 import functional as Fn
        from dsmil_wsi_b200.train_graph import _warm_up
        self.params, self.nb = params, nb
        self.slots = torch.zeros(nb, MAX_ROWS, D, device="cuda")
        self.vslots = torch.zeros_like(self.slots) if distinct else None
        self.Ns = torch.ones(nb, dtype=torch.int64, device="cuda")
        self.status = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.wc = torch.zeros(nb * MAX_ROWS, C_, device="cuda")
        self.wp = torch.zeros(nb, C_, device="cuda")

        def run():
            classes, pred, A, B, crit = Fn.MILValueBagsDevFn.apply(self.slots, self.vslots, self.Ns, self.status,
                                                                   *params)
            saves = classes.grad_fn.saved_tensors[4:7]
            loss = (classes * self.wc).sum() + (pred * self.wp).sum()
            grads = torch.autograd.grad(loss, _live(params))
            return (classes, pred, A, B, crit) + tuple(saves), grads
        _warm_up(torch.device("cuda"), 1, run)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.out = run()

    def replay(self, xs, vs, wc, wp):
        Ns = [int(x.shape[0]) for x in xs]
        self.slots.zero_()
        for b, x in enumerate(xs):
            self.slots[b, :Ns[b]] = x
            if self.vslots is not None:
                self.vslots[b, :Ns[b]] = vs[b]
        self.Ns.copy_(torch.tensor(Ns))
        self.wc.zero_()
        self.wc[:sum(Ns)] = wc
        self.wp.copy_(wp)
        self.graph.replay()
        torch.cuda.synchronize()
        return self.out


def _eager_pair(params, xs, vs, wc, wp):
    from dsmil_wsi_b200 import functional as Fn
    outs, crit = Fn.mil_forward_value_bags(xs, params, vs, grad=True)
    classes, pred, A, B = outs.packed
    nb, nv = len(xs), 0 if vs is None else len(xs)
    saved = classes.grad_fn.saved_tensors
    sQ, sH, sV = saved[nb + nv + 1:nb + nv + 4]
    loss = (classes * wc).sum() + (pred * wp).sum()
    grads = torch.autograd.grad(loss, _live(params))
    return (classes, pred, A, B, crit, sQ, sH, sV), grads


def _assert_pair_equal(dev, eager, total):
    (d_out, d_g), (e_out, e_g) = dev, eager
    for i, (a, b) in enumerate(zip(d_out, e_out)):
        if b is None:
            continue
        a = a[:total] if i in (0, 2, 5, 6, 7) else a
        assert torch.equal(a, b), i
    assert len(d_g) == len(e_g) and all(torch.equal(a, b) for a, b in zip(d_g, e_g))


@pytest.mark.parametrize("distinct", [True, False])
@pytest.mark.parametrize("D,C_,nl", SHAPES)
def test_dev_pair_equals_the_eager_pair(D, C_, nl, distinct):
    params = _torch_params(D, C_, nl, 7 + D)
    pair = _DevPair(params, 6, D, C_, distinct)
    for k, Ns in enumerate(BATCHES):
        xs = [_bag(n, D, 100 * k + i) for i, n in enumerate(Ns)]
        vs = None
        if distinct:
            torch.manual_seed(k)
            vs = [x * torch.nn.functional.dropout(torch.ones_like(x), 0.2, True) for x in xs]
        g = torch.Generator(device="cuda").manual_seed(k)
        wc = 1.0 + torch.randn(sum(Ns), C_, device="cuda", generator=g)
        wp = torch.randn(len(Ns), C_, device="cuda", generator=g)
        dev = pair.replay(xs, vs, wc, wp)
        assert int(pair.status.item()) == 0
        _assert_pair_equal(dev, _eager_pair(params, xs, vs, wc, wp), sum(Ns))


def _addrs(ts, shift=0):
    return torch.tensor([0 if t is None else t.data_ptr() + shift for t in ts], dtype=torch.int64, device="cuda")


@pytest.mark.parametrize("D", [512, 166])
def test_refused_batches_set_status_and_leave_the_next_batch_correct(D):
    from dsmil_wsi_b200 import functional as Fn
    C_ = 2
    params = [t.detach() for t in _torch_params(D, C_, True, 3)]
    nb, mr = 4, 200
    xs = [_bag(n, D, 50 + i) for i, n in enumerate([30, 200, 1, 77])]
    vs = [x * 0.5 for x in xs]
    Ns = torch.tensor([30, 200, 1, 77], dtype=torch.int64, device="cuda")
    shift = 4 if D % 4 == 0 else 2          # breaks 16-byte (D % 4 == 0) or 4-byte alignment
    cases = [
        (_addrs(xs), _addrs(vs), torch.tensor([30, 0, 1, 77], device="cuda"), 2),
        (_addrs(xs), _addrs(vs), torch.tensor([30, 200, 201, 77], device="cuda"), 3),
        (torch.cat([_addrs(xs[:3]), _addrs(xs[3:], shift)]), _addrs(vs), Ns, 4),
        (_addrs(xs), _addrs([vs[0], None, vs[2], vs[3]]), Ns, 2),
        (_addrs(xs), torch.cat([_addrs(vs[:2]), _addrs(vs[2:3], shift), _addrs(vs[3:])]), Ns, 3),
    ]
    ref, _ = Fn.mil_forward_value_bags(xs, params, vs)
    for xa, va, n, want in cases:
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        out = Fn.mil_forward_value_bags_dev(xa, va, n.to(torch.int64), status, mr, params)
        assert int(status.item()) == want
        classes, pred, A, B, crit = out                  # the stand-in batch: one row per bag
        assert all(torch.isfinite(t).all() for t in (classes[:nb], pred, A[:nb], B))
        assert torch.equal(crit, torch.zeros_like(crit))
        status.zero_()
        classes, pred, A, B, crit = Fn.mil_forward_value_bags_dev(_addrs(xs), _addrs(vs), Ns, status, mr, params)
        total = int(Ns.sum())
        assert int(status.item()) == 0
        assert torch.equal(classes[:total], ref.packed[0]) and torch.equal(pred, ref.packed[1])
        assert torch.equal(A[:total], ref.packed[2]) and torch.equal(B, ref.packed[3])


def _net(D, C_, nl, dropout_v, seed):
    from dsmil_wsi_b200.modules import BClassifier, FCLayer, MILNet
    torch.manual_seed(seed)
    return MILNet(FCLayer(D, C_), BClassifier(D, C_, dropout_v=dropout_v, nonlinear=nl, passing_v=True)).cuda()


def _opt(net, kind):
    if kind == "sgd":
        return torch.optim.SGD(net.parameters(), lr=0.05, momentum=0.9)
    return torch.optim.Adam(net.parameters(), lr=1e-3, capturable=True)


def _state(net, opt):
    vals = [p.detach().clone() for p in net.parameters()]
    st = [v.clone() for p in net.parameters() for v in opt.state.get(p, {}).values() if torch.is_tensor(v)]
    return vals + st


@pytest.mark.parametrize("kind", ["sgd", "adam"])
@pytest.mark.parametrize("p_drop", [0.0, 0.2])
def test_train_step_graph_equals_the_eager_value_step(kind, p_drop):
    from dsmil_wsi_b200 import feed
    from dsmil_wsi_b200 import functional as Fn
    from dsmil_wsi_b200.train_graph import TrainStepGraph
    from dsmil_wsi_b200.sharded import milnet_params
    D, C_, nb = 512, 2, 4
    crit = torch.nn.BCEWithLogitsLoss()
    net_g, net_e = _net(D, C_, True, p_drop, 1), _net(D, C_, True, p_drop, 1)
    opt_g, opt_e = _opt(net_g, kind), _opt(net_e, kind)
    g = TrainStepGraph(net_g, crit, opt_g, nb, MAX_ROWS, value=True)
    assert (g.v_inputs is not None) == (p_drop > 0)
    net_g.train(), net_e.train()
    for step in range(3):
        Ns = [[9, MAX_ROWS, 1, 130], [3, 4, 5, 6], [MAX_ROWS] * 4][step]
        xs = [_bag(n, D, 10 * step + i) for i, n in enumerate(Ns)]
        labels = torch.tensor([[float((i + step) % 2), float(i % 2)] for i in range(nb)], device="cuda")
        torch.manual_seed(100 + step)
        vs = [net_e.b_classifier._v_input(x) for x in xs]
        opt_e.zero_grad()
        outs, _ = Fn.mil_forward_value_bags(xs, milnet_params(net_e), None if vs[0] is None else vs, grad=True)
        loss_e = feed.minibatch_loss(crit, *feed._group_predictions(outs), labels)
        loss_e.backward()
        opt_e.step()
        torch.manual_seed(100 + step)
        for b, x in enumerate(xs):
            g.slots[b, :Ns[b]] = x
            g.Ns[b] = Ns[b]
            if g.v_inputs is not None:
                net_g.b_classifier._v_input(g.slots[b, :Ns[b]], out=g.v_inputs[b, :Ns[b]])
        g.labels.copy_(labels)
        loss_g = g.step()
        assert torch.equal(loss_g, loss_e.detach())
        assert all(torch.equal(a, b) for a, b in zip(_state(net_g, opt_g), _state(net_e, opt_e)))
    # a refused batch: NaN loss, parameters and optimizer state kept bit for bit
    before = _state(net_g, opt_g)
    g.Ns[1] = 0
    assert torch.isnan(g.step()).item()
    assert int(g.status.item()) == 2
    assert all(torch.equal(a, b) for a, b in zip(_state(net_g, opt_g), before))


def _store(Ns, D, C_, seed):
    from dsmil_wsi_b200 import feed
    store = feed.DeviceBagStore(D)
    for i, n in enumerate(Ns):
        store.add_bag(_bag(n, D, seed + i), torch.tensor([float((i * 7 + j) % 3 == 0) for j in range(C_)]))
    return store


def _rng_states():
    return torch.cuda.get_rng_state(), torch.get_rng_state()


@pytest.mark.parametrize("k", [1, 5])
def test_train_epoch_graph_equals_the_eager_value_epoch(k):
    from dsmil_wsi_b200 import feed
    D, C_ = 512, 2
    store = _store([40, 200, 7, 129, 128, 1000, 33, 64, 90, 300, 12, 250], D, C_, 300)   # 12 bags: a short last group
    order = list(range(len(store)))[::-1]
    crit = torch.nn.BCEWithLogitsLoss()
    res = []
    for graph in (False, True):
        net = _net(D, C_, True, 0.2, 4)
        opt = _opt(net, "adam")
        torch.manual_seed(21)
        gen = torch.Generator(device="cuda").manual_seed(5)
        loss = feed.train_epoch(net, store, crit, opt, dropout_patch=0.3, order=order, generator=gen,
                                bags_per_step=k, graph=graph, value=True)
        res.append((loss, _state(net, opt), _rng_states(), gen.get_state()))
    (l0, s0, r0, g0), (l1, s1, r1, g1) = res
    assert l0 == l1
    assert all(torch.equal(a, b) for a, b in zip(s0, s1))
    assert all(torch.equal(a, b) for a, b in zip(r0, r1)) and torch.equal(g0, g1)


def _musk(n_bags, D, seed):
    rs = np.random.RandomState(seed)
    return [(int(rs.randint(0, 2)), rs.randn(int(rs.randint(2, 41)), D).astype(np.float32)) for _ in range(n_bags)]


def test_mil_epochs_graph_equal_their_eager_value_forms():
    from dsmil_wsi_b200 import feed
    D, C_ = 166, 1
    store = feed.mil_store(_musk(23, D, 1))
    crit = torch.nn.BCEWithLogitsLoss()
    res = []
    for graph in (False, True):
        net = _net(D, C_, True, 0.2, 6)
        opt = _opt(net, "sgd")
        torch.manual_seed(2)
        losses = [feed.mil_epoch_train(net, store, crit, opt, order=list(range(23)), bags_per_step=4, graph=graph,
                                       value=True) for _ in range(2)]
        test = feed.mil_epoch_test(net, store, crit, bags_per_launch=8, graph=graph, value=True)
        res.append((losses, _state(net, opt), test))
    assert res[0][0] == res[1][0]
    assert all(torch.equal(a, b) for a, b in zip(res[0][1], res[1][1]))
    assert res[0][2][0] == res[1][2][0] and res[0][2][1] == res[1][2][1]
    assert all(np.array_equal(a, b) for a, b in zip(res[0][2][2], res[1][2][2]))


def test_eval_epoch_graph_equals_the_eager_eval_epoch():
    from dsmil_wsi_b200 import feed
    D, C_ = 512, 2
    store = _store([40, 200, 7, 129, 128, 1000, 33, 64, 90, 300, 12], D, C_, 400)
    net = _net(D, C_, True, 0.2, 8)
    crit = torch.nn.BCEWithLogitsLoss()
    for average in (False, True):
        e = feed.eval_epoch(net, store, crit, average=average, bags_per_launch=4)
        g = feed.eval_epoch(net, store, crit, average=average, bags_per_launch=4, graph=True, value=True)
        assert e[0] == g[0] and np.array_equal(e[1], g[1]) and np.array_equal(e[2], g[2])


def test_eager_value_epoch_is_close_to_the_per_bag_default():
    """The batched value step sums its gradients in another order than the per-bag autograd: within the bars the
    batched-vs-per-bag comparison of the value backward uses, after one step on the same draws."""
    from dsmil_wsi_b200 import feed
    D, C_ = 512, 2
    store = _store([40, 200, 7, 129], D, C_, 500)
    crit = torch.nn.BCEWithLogitsLoss()
    grads = []
    for value in (False, True):
        net = _net(D, C_, True, 0.0, 9)
        opt = torch.optim.SGD(net.parameters(), lr=0.0)
        feed.train_epoch(net, store, crit, opt, order=[0, 1, 2, 3], bags_per_step=4, value=value)
        grads.append({n: p.grad.detach().clone() for n, p in net.named_parameters()})
    for n in grads[0]:
        bar = 1e-4 if ".q." in n else 2e-5
        assert rel_to_max(grads[1][n].cpu().numpy(), grads[0][n].cpu().numpy()) <= bar, n


@pytest.mark.parametrize("nb", [1, 16])
def test_forward_bags_graph_equals_forward_bags(nb):
    from dsmil_wsi_b200.infer_graph import ForwardBagsGraph
    D, C_ = 512, 2
    net = _net(D, C_, True, 0.2, 10).eval()
    g = ForwardBagsGraph(net, nb, 2000, value=True)
    for k in range(2):
        xs = [_bag(1 + (37 * i + 500 * k) % 2000, D, 600 + i + 50 * k) for i in range(nb)]
        got = g.run(xs)
        ref = net.forward_bags(xs)
        for a, b in zip(got.packed, ref.packed):
            assert torch.equal(a, b)
        with torch.no_grad():                       # an in-place update is seen by the next replay
            net.b_classifier.v[1].weight.mul_(1.01)
    net.b_classifier.v[1].weight = torch.nn.Parameter(net.b_classifier.v[1].weight.detach().clone())
    with pytest.raises(RuntimeError, match="replaced"):
        g.run(xs)
    net2 = _net(D, C_, True, 0.2, 11).eval()
    g2 = ForwardBagsGraph(net2, nb, 2000, value=True)
    net2.train()
    with pytest.raises(RuntimeError, match="dropout_v"):
        g2.run(xs)


def _kernels_per_replay(g):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.step()
        torch.cuda.synchronize()
    return [e.name for e in prof.events()
            if e.device_type == torch.autograd.DeviceType.CUDA and "dsmil" in e.name]


def test_replay_launches_the_same_kernels_at_any_nb():
    from test_kernel_instances_gpu import KERNELS, launched
    from dsmil_wsi_b200.train_graph import TrainStepGraph
    D, C_ = 512, 2
    counts, keys = [], set()
    for nb in (2, 16):
        net = _net(D, C_, True, 0.2, 12)
        g = TrainStepGraph(net, torch.nn.BCEWithLogitsLoss(), _opt(net, "adam"), nb, 500, value=True)
        g.Ns.fill_(300)
        counts.append(len(_kernels_per_replay(g)))
        keys |= launched(g.step)
    assert counts[0] == counts[1] > 0, counts
    assert keys and keys <= set(KERNELS), sorted(keys - set(KERNELS))
    assert {"k_plan_bags_gen", "k_vproj_b", "k_linear_models<3,1>", "k_gemm_tn_rag"} <= keys
