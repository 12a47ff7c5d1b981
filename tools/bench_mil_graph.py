"""The generic batched route: classic-MIL epochs with and without CUDA graphs, and one large generic batch through
forward_bags against the per-bag forward it replaces.

Workloads (synthetic, seeded):
  musk   D = 166, C = 1, 92 bags of 2 to 40 rows (the shape of train_mil.py's Musk sets)
  eleph  D = 230, C = 1, 200 bags of 2 to 13 rows (Elephant / Fox / Tiger)
  For each: the training epoch at k = 1 (the reference's loop: feed.train_epoch per bag, eager) against
  feed.train_epoch(graph=True, generic=True) (which records its graph on every call, so that cost is in the number),
  and the evaluation epoch eager (bags_per_launch = 16) against eval_epoch(graph=True, generic=True) (graphs cached
  after the first call).
  big    16 bags x 10 000 x 512, C = 6 and, separately, linear q with C = 2: one forward_bags call (the generic batched
  route) against the per-bag dsmil_forward loop the call ran before it existed.

Arms alternate within each of `--repeats` repeats; times are host clocks around work that ends in a device
synchronise (epochs) or CUDA events (the big batch).  In the same run, outputs are compared with torch.equal: the
graph epoch's parameters against the eager minibatch epoch's at k = 1 from the same start, the eval results, and
every forward_bags output against the per-bag forward.  The card name and power limit are read in the same run.

    python tools/bench_mil_graph.py --out profiles/h100_mil_graph_1gpu.json
"""
import argparse
import copy
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import dsmil as mil  # noqa: E402
from dsmil_wsi_b200 import feed  # noqa: E402
from bench_models_train import card, events_ms  # noqa: E402


def _store(D, sizes, seed):
    g = torch.Generator().manual_seed(seed)
    store = feed.DeviceBagStore(D)
    for i, n in enumerate(sizes):
        store.add_bag(torch.rand(n, D, generator=g), torch.tensor([float(i % 2)]))
    return store


def _timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def _minibatch_epoch(net, store, crit, opt, order):
    """train_epoch's k-bag step at k = 1: what train_epoch(graph=True) replays, bit for bit."""
    for i in order:
        opt.zero_grad()
        x = feed.dropout_patches(store.bags[i][0], 1.0)
        bp, mp = feed._group_predictions(net.forward_bags([x], grad=True))
        loss = feed.minibatch_loss(crit, bp, mp, store.bags[i][1].view(1, -1))
        loss.backward()
        opt.step()


def mil_workload(name, D, sizes, repeats):
    store = _store(D, sizes, 1)
    crit = torch.nn.BCEWithLogitsLoss()
    torch.manual_seed(0)
    base = mil.MILNet(mil.FCLayer(D, 1), mil.BClassifier(D, 1)).cuda()
    nets = {a: copy.deepcopy(base) for a in ("eager", "graph", "check")}
    opts = {a: torch.optim.SGD(n.parameters(), lr=1e-3, momentum=0.9) for a, n in nets.items()}
    order = np.random.default_rng(2).permutation(len(store)).tolist()
    # bits: one graph epoch against the eager minibatch epoch from the same start (same row permutations)
    torch.manual_seed(5)
    _minibatch_epoch(nets["check"], store, crit, opts["check"], order)
    torch.manual_seed(5)
    feed.train_epoch(nets["graph"], store, crit, opts["graph"], order=order, graph=True, generic=True)
    same_train = all(torch.equal(a, b) for a, b in zip(nets["check"].parameters(), nets["graph"].parameters()))
    feed.train_epoch(nets["eager"], store, crit, opts["eager"], order=order)            # warm-up
    e = feed.eval_epoch(nets["graph"], store, crit)
    g = feed.eval_epoch(nets["graph"], store, crit, graph=True, generic=True)
    same_eval = e[0] == g[0] and np.array_equal(e[2], g[2])
    t = {"train_eager": [], "train_graph": [], "eval_eager": [], "eval_graph": []}
    for _ in range(repeats):
        t["train_eager"].append(_timed(lambda: feed.train_epoch(nets["eager"], store, crit, opts["eager"],
                                                                order=order))[0])
        t["train_graph"].append(_timed(lambda: feed.train_epoch(nets["graph"], store, crit, opts["graph"],
                                                                order=order, graph=True, generic=True))[0])
        t["eval_eager"].append(_timed(lambda: feed.eval_epoch(nets["graph"], store, crit))[0])
        t["eval_graph"].append(_timed(lambda: feed.eval_epoch(nets["graph"], store, crit, graph=True,
                                                              generic=True))[0])
    return {"workload": name, "D": D, "bags": len(sizes), "rows": int(sum(sizes)),
            "ms_per_epoch": {k: [round(v, 3) for v in vs] for k, vs in t.items()},
            "torch_equal": {"train_graph_vs_eager_minibatch_k1": same_train, "eval_graph_vs_eager": same_eval}}


def big_workload(C, nonlinear, repeats, steps):
    torch.manual_seed(3)
    D, nb, N = 512, 16, 10_000
    net = mil.MILNet(mil.FCLayer(D, C), mil.BClassifier(D, C, nonlinear=nonlinear)).cuda().eval()
    xs = [torch.rand(N, D, device="cuda") for _ in range(nb)]
    with torch.no_grad():
        outs = net.forward_bags(xs)
        per = [net(x) for x in xs]
        same = all(torch.equal(u, v) for b in range(nb) for u, v in zip(outs[b], per[b]))
        t = {"forward_bags": [], "per_bag_loop": []}
        for _ in range(repeats):
            t["forward_bags"].append(events_ms(lambda: net.forward_bags(xs), steps, 2))
            t["per_bag_loop"].append(events_ms(lambda: [net(x) for x in xs], steps, 2))
    return {"workload": f"{nb}x{N}x{D} C={C} {'nonlinear' if nonlinear else 'linear'} q", "ms_per_call":
            {k: [round(v, 4) for v in vs] for k, vs in t.items()}, "torch_equal_every_output": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out")
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    res = {"card": card(), "results": [
        mil_workload("musk", 166, rng.integers(2, 41, 92).tolist(), a.repeats),
        mil_workload("eleph", 230, rng.integers(2, 14, 200).tolist(), a.repeats),
        big_workload(6, True, a.repeats, a.steps),
        big_workload(2, False, a.repeats, a.steps)]}
    s = json.dumps(res)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
