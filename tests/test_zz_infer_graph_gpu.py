"""dsmil_forward_bags_dev and the inference graphs against the eager dsmil_forward_bags, bit for bit.

Covered: D/C 512/1, 512/2, 1024/4 and 2048/2; ragged batches ([1], [max_rows], [127, 128, 129], mixed); bags that are
separate allocations or views into one store; the direct call and one capture replayed over several batches of
different bag tensors; a refused batch and the batch after it; in-place weight updates between replays; the nb = 1
graph against milnet(x); eval_epoch(graph=True) against eval_epoch(); and, read from the recorded graph itself, the
programmatic edge from phase 1 to the attend pass."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import build_net
from oracle import dsmil_oracle as orc
from dsmil_wsi_b200 import feed
from dsmil_wsi_b200 import functional as Fn
from dsmil_wsi_b200.infer_graph import ForwardBagsGraph
from dsmil_wsi_b200.sharded import milnet_params

pytestmark = pytest.mark.gpu

MAX_ROWS = 600
SHAPES = [(512, 1), (512, 2), (1024, 4), (2048, 2)]


def _net(D, C, seed):
    return build_net(orc.random_params(D, C, seed, scale=2.0)).eval()


def _sizes(case):
    return {"one_row": [1], "full": [MAX_ROWS], "tile_edges": [127, 128, 129],
            "mixed": [300, 1, MAX_ROWS, 45, 256, 513]}[case]


def _bags(sizes, D, seed, views=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if not views:
        return [torch.rand(n, D, generator=g, device="cuda") for n in sizes]
    store = torch.rand(sum(sizes) + 7, D, generator=g, device="cuda")
    offs = np.cumsum([3] + sizes[:-1]).tolist()
    return [store[o:o + n] for o, n in zip(offs, sizes)]


def _eager(net, xs):
    outs, crit = Fn._mil_forward_bags_infer(xs, milnet_params(net))
    return [t.clone() for t in outs.packed] + [crit.clone()]


def _live(packed, total):
    classes, pred, A, B, crit = packed
    return [classes[:total], pred, A[:total], B, crit]


def _assert_equal(got, ref, what):
    names = ("classes", "pred", "A", "B", "crit")
    for n, u, v in zip(names, got, ref):
        assert u.shape == v.shape and torch.equal(u, v), (what, n)


def _direct(net, xs, max_rows=MAX_ROWS, Ns=None):
    dev = xs[0].device
    ptrs = torch.tensor([x.data_ptr() for x in xs], dtype=torch.int64, device=dev)
    Ns = torch.tensor(Ns if Ns is not None else [x.shape[0] for x in xs], dtype=torch.int64, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    out = Fn.mil_forward_bags_dev(ptrs, Ns, status, max_rows, milnet_params(net))
    return out, status


@pytest.mark.parametrize("case", ["one_row", "full", "tile_edges", "mixed"])
@pytest.mark.parametrize("D,C", SHAPES)
def test_direct_call_equals_eager(D, C, case):
    net = _net(D, C, 5000 + D + C)
    sizes = _sizes(case)
    for views in (False, True):
        xs = _bags(sizes, D, 5100 + len(sizes), views)
        out, status = _direct(net, xs)
        ref = _eager(net, xs)
        torch.cuda.synchronize()
        assert int(status.item()) == 0
        _assert_equal(_live(out, sum(sizes)), ref, (case, views))


@pytest.mark.parametrize("D,C", SHAPES)
def test_replay_over_batches_equals_eager(D, C):
    net = _net(D, C, 5200 + D + C)
    g = ForwardBagsGraph(net, 3, MAX_ROWS)
    batches = [[1, MAX_ROWS, 129], [127, 128, 129], [MAX_ROWS, MAX_ROWS, MAX_ROWS], [5, 300, 1], [256, 1, 2]]
    for k, sizes in enumerate(batches):
        xs = _bags(sizes, D, 5300 + k, views=k % 2 == 1)
        outs = g.run(xs)
        got = [t.clone() for t in outs.packed] + [outs.crit.clone()]
        assert outs.Ns == sizes and len(outs) == 3
        ref = _eager(net, xs)
        _assert_equal(got, ref, k)
        for b in range(3):                                        # the per-bag views over the live rows
            for u, v in zip(outs[b], Fn.BagOutputs(*ref[:4], sizes)[b]):
                assert torch.equal(u, v), (k, b)
    torch.cuda.synchronize()
    assert int(g.status.item()) == 0


def test_refused_batch_then_a_correct_one():
    net = _net(512, 2, 5400)
    # on the device: a row count outside [1, max_rows] in the direct call
    xs = _bags([100, 200], 512, 5500)
    for Ns, want in [([100, MAX_ROWS + 1], 2), ([0, 200], 1)]:
        out, status = _direct(net, xs, Ns=Ns)
        torch.cuda.synchronize()
        assert int(status.item()) == want
        classes, pred, A, B, crit = _live(out, 2)                  # the stand-in: one row of zeros per bag
        for t in (classes, pred, A, B):
            assert torch.isfinite(t).all()
        assert torch.equal(crit, torch.zeros_like(crit))
        assert torch.equal(pred, net.b_classifier.fcc.bias.detach().expand(2, 2))
    # through the graph: features that are not 16-byte aligned
    g = ForwardBagsGraph(net, 2, MAX_ROWS)
    base = torch.rand(300 * 512 + 4, device="cuda")
    bad = base[1:1 + 300 * 512].view(300, 512)
    outs = g.run([xs[0], bad])
    torch.cuda.synchronize()
    assert int(g.status.item()) == 2
    for t in outs.packed:
        assert torch.isfinite(t[:2]).all()
    good = _bags([333, 77], 512, 5600)
    outs = g.run(good)
    got = [t.clone() for t in outs.packed] + [outs.crit.clone()]
    _assert_equal(got, _eager(net, good), "after the refusal")
    assert int(g.status.item()) == 2                               # the library never clears it


def test_weight_updates_between_replays():
    net = _net(1024, 4, 5700)
    g = ForwardBagsGraph(net, 2, MAX_ROWS)
    xs = _bags([400, 129], 1024, 5800)
    first = [t.clone() for t in g.run(xs).packed]
    with torch.no_grad():
        for p in net.parameters():
            p.mul_(0.75).add_(0.01)
    outs = g.run(xs)
    got = [t.clone() for t in outs.packed] + [outs.crit.clone()]
    _assert_equal(got, _eager(net, xs), "in-place update")
    assert not torch.equal(got[1], first[1])
    other = _net(1024, 4, 5701)
    net.load_state_dict(other.state_dict())
    outs = g.run(xs)
    got = [t.clone() for t in outs.packed] + [outs.crit.clone()]
    _assert_equal(got, _eager(other, xs), "load_state_dict")
    net.b_classifier.fcc.weight = torch.nn.Parameter(net.b_classifier.fcc.weight.detach().clone())
    with pytest.raises(RuntimeError, match="replaced"):
        g.run(xs)


def test_run_refuses_before_any_launch():
    net = _net(512, 2, 5900)
    g = ForwardBagsGraph(net, 2, 100)
    with pytest.raises(ValueError, match="max_rows=100"):
        g.run(_bags([50, 101], 512, 6000))
    with pytest.raises(ValueError, match="nb=2"):
        g.run(_bags([50], 512, 6000))
    with pytest.raises(IndexError):
        g.run([torch.rand(10, 512, device="cuda"), torch.rand(0, 512, device="cuda")])


@pytest.mark.parametrize("D,C", [(512, 2), (1024, 4)])
def test_one_slide_graph_equals_milnet(D, C):
    net = _net(D, C, 6100 + D)
    g = ForwardBagsGraph(net, 1, 2000)
    for k, n in enumerate([1, 2000, 777, 128, 1500]):
        x = _bags([n], D, 6200 + k)[0]
        with torch.no_grad():
            ref = net(x)
        got = g.run([x])[0]
        for u, v in zip(got, ref):
            assert u.shape == v.shape and torch.equal(u, v), (n, u.shape)


def _store(sizes, D, C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    store = feed.DeviceBagStore(D)
    for n in sizes:
        store.add_bag(torch.rand(n, D, generator=g, device="cuda"),
                      (torch.rand(C, generator=g, device="cuda") > 0.5).float())
    return store


@pytest.mark.parametrize("dropout_patch", [0.0, 0.3])
@pytest.mark.parametrize("average", [False, True])
def test_eval_epoch_graph_equals_eager(average, dropout_patch):
    D, C = 512, 2
    net = _net(D, C, 6300)
    rng = np.random.default_rng(6400)
    store = _store([int(n) for n in rng.integers(1, 1500, 37)], D, C, 6500)   # 16 + 16 + a short group of 5
    crit = torch.nn.BCEWithLogitsLoss()

    def run(graph):
        gen = torch.Generator(device="cuda").manual_seed(6600)
        return feed.eval_epoch(net, store, crit, average=average, bags_per_launch=16, dropout_patch=dropout_patch,
                               generator=gen, graph=graph)

    ref, got = run(False), run(True)
    assert got[0] == ref[0]
    assert np.array_equal(got[1], ref[1]) and got[1].dtype == ref[1].dtype
    assert np.array_equal(got[2], ref[2]) and got[2].dtype == ref[2].dtype


def _edges(raw_graph):
    """(from, to, edge data) of every edge of a cudaGraph_t: cudaGraphGetEdges_v2 of the CUDA runtime."""
    class EdgeData(ctypes.Structure):
        _fields_ = [("from_port", ctypes.c_ubyte), ("to_port", ctypes.c_ubyte), ("type", ctypes.c_ubyte),
                    ("reserved", ctypes.c_ubyte * 5)]

    rt = ctypes.CDLL("libcudart.so.12")
    n = ctypes.c_size_t(0)
    assert rt.cudaGraphGetEdges_v2(ctypes.c_void_p(raw_graph), None, None, None, ctypes.byref(n)) == 0
    frm, to = (ctypes.c_void_p * n.value)(), (ctypes.c_void_p * n.value)()
    data = (EdgeData * n.value)()
    assert rt.cudaGraphGetEdges_v2(ctypes.c_void_p(raw_graph), frm, to, data, ctypes.byref(n)) == 0
    return [(frm[i], to[i], data[i]) for i in range(n.value)]


def _kernel_name(node):
    """The mangled kernel name of a kernel node (driver API), or None for another node type."""
    class KernelParams(ctypes.Structure):
        _fields_ = [("func", ctypes.c_void_p), ("grid", ctypes.c_uint * 3), ("block", ctypes.c_uint * 3),
                    ("smem", ctypes.c_uint), ("params", ctypes.c_void_p), ("extra", ctypes.c_void_p),
                    ("kern", ctypes.c_void_p), ("ctx", ctypes.c_void_p)]

    cu = ctypes.CDLL("libcuda.so.1")
    t = ctypes.c_int(-1)
    assert cu.cuGraphNodeGetType(ctypes.c_void_p(node), ctypes.byref(t)) == 0
    if t.value != 0:                                              # CU_GRAPH_NODE_TYPE_KERNEL
        return None
    kp = KernelParams()
    assert cu.cuGraphKernelNodeGetParams_v2(ctypes.c_void_p(node), ctypes.byref(kp)) == 0
    name = ctypes.c_char_p()
    if kp.func:
        assert cu.cuFuncGetName(ctypes.byref(name), ctypes.c_void_p(kp.func)) == 0
    else:
        assert cu.cuKernelGetName(ctypes.byref(name), ctypes.c_void_p(kp.kern)) == 0
    return name.value.decode()


def test_overlap_survives_capture():
    """The recorded call holds a programmatic edge from the phase-1 kernel node to the attend node (the launch
    attribute became a graph edge, so the replay overlaps them), and replays give the eager bits."""
    net = _net(512, 2, 6700)
    xs = _bags([10_000] * 16, 512, 6800)
    ptrs = torch.tensor([x.data_ptr() for x in xs], dtype=torch.int64, device="cuda")
    Ns = torch.tensor([x.shape[0] for x in xs], dtype=torch.int64, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    params = milnet_params(net)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        Fn.mil_forward_bags_dev(ptrs, Ns, status, 10_000, params)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(graph):
        out = Fn.mil_forward_bags_dev(ptrs, Ns, status, 10_000, params)
    edges = [(_kernel_name(f), _kernel_name(t), d) for f, t, d in _edges(graph.raw_cuda_graph())]
    into_attend = [(f, d.type, d.from_port) for f, t, d in edges if t is not None and "k_attend_b" in t]
    assert len(into_attend) == 1, into_attend
    src, typ, port = into_attend[0]
    assert src is not None and "k_qmlp_sm90" in src, into_attend
    assert typ == 1, into_attend                                  # cudaGraphDependencyTypeProgrammatic
    assert port in (1, 2), into_attend                            # programmatic / launch-completion port
    graph.instantiate()
    graph.replay()
    ref = _eager(net, xs)
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    _assert_equal(_live(out, 160_000), ref, "replay")


def test_eval_epoch_graph_reuses_its_graphs_across_epochs():
    """A second epoch replays the cached graphs, and sees an in-place update of the weights made between epochs."""
    from dsmil_wsi_b200.feed import _EVAL_GRAPHS
    D, C = 512, 2
    net = _net(D, C, 6900)
    store = _store([300, 1200, 64, 900, 5], D, C, 7000)
    crit = torch.nn.BCEWithLogitsLoss()
    feed.eval_epoch(net, store, crit, bags_per_launch=2, graph=True)
    first = dict(_EVAL_GRAPHS[net])
    assert sorted(k[0] for k in first) == [1, 2]
    with torch.no_grad():
        for p in net.parameters():
            p.mul_(0.5)
    got, ref = (feed.eval_epoch(net, store, crit, bags_per_launch=2, graph=gr) for gr in (True, False))
    assert all(_EVAL_GRAPHS[net][k] is g for k, g in first.items())
    assert got[0] == ref[0] and np.array_equal(got[1], ref[1]) and np.array_equal(got[2], ref[2])
