"""The fold step of a classic-MIL cross-validation on the generic shapes: five training folds of a 10-fold split
trained one epoch at a time as one replayed fold graph (feed.train_epoch_models(graph=True, generic=True)), as five
one-fold graph epochs (train_epoch(graph=True, generic=True)) and as the eager fold epoch (train_epoch_models).

Workloads (train_mil.py's sets, synthetic features): Musk1-shaped, 92 bags of 2-40 rows at D = 166; Elephant-shaped,
200 bags of 2-13 rows at D = 230; C = 1, nonlinear q; k = 1 and 4 bags per step; capturable Adam with train_mil.py's
betas (0.5, 0.9), lr 2e-4 and weight decay 5e-3.

Epoch arms: host clock around each epoch (each ends in a host sync); the arms alternate within each of `--repeats`
repeats, every arm on its own copies of the models and optimizers from the same start, and after every repeat each
fold's losses and parameters are compared with torch.equal across the arms.  Replay arms: CUDA events over `--steps`
replays of one recorded FoldTrainStepGraph against the five TrainStepGraph replays of the same full step, so the
per-call recording cost of the epochs is separated out.  The card name, power limit and max SM clock are read in the
same run.  Needs a GPU; prints one JSON object (--out: also writes it).

    python tools/bench_models_mil_graph.py --out profiles/h100_models_mil_graph_1gpu.json

--profile (a separate invocation: tracing slows the host) runs torch.profiler over `--steps` replays of the fold graph
and of the five one-fold graphs, and splits each step's kernels and kernel time into the library's, the optimizer
and refusal guard's (foreach / multi-tensor kernels and the copies of the guard) and the rest (the loss).
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
from dsmil_wsi_b200.train_graph import FoldTrainStepGraph, TrainStepGraph  # noqa: E402
from bench_models_train import card, events_ms  # noqa: E402

WORKLOADS = {"musk1": (92, 2, 40, 166), "elephant": (200, 2, 13, 230)}
ARMS = ("fold_graph", "one_fold_graphs", "eager")
FOLDS = 5


def _workload(name, seed=0):
    nb, lo, hi, D = WORKLOADS[name]
    rng = np.random.default_rng(seed)
    store = feed.DeviceBagStore(D)
    for i in range(nb):
        n = int(rng.integers(lo, hi + 1))
        store.add_bag(torch.from_numpy(rng.random((n, D), dtype=np.float32)),
                      torch.tensor([float(i % 2)]))
    perm = rng.permutation(nb)
    tenth = [perm[j::10].tolist() for j in range(10)]
    folds = [[i for j in range(10) if j != f for i in tenth[j]] for f in range(FOLDS)]   # the first five of ten
    return store, folds, D


def _opt(net):
    return torch.optim.Adam(net.parameters(), lr=2e-4, betas=(0.5, 0.9), weight_decay=5e-3, capturable=True)


class Epochs:
    def __init__(self, store, folds, D, k):
        torch.manual_seed(1)
        nets = [mil.MILNet(mil.FCLayer(D, 1), mil.BClassifier(D, 1)).cuda() for _ in range(FOLDS)]
        self.store, self.folds, self.k = store, folds, k
        self.crit = torch.nn.BCEWithLogitsLoss()
        self.nets = {a: [copy.deepcopy(n) for n in nets] for a in ARMS}
        self.opts = {a: [_opt(n) for n in ns] for a, ns in self.nets.items()}
        # per-fold generators, the same seeds in every arm: dropout_patches draws each bag's row permutation from them
        self.gens = {a: [torch.Generator(device="cuda").manual_seed(7 + m) for m in range(FOLDS)] for a in ARMS}
        self.epoch = 0

    def _orders(self):
        return [np.random.default_rng(100 * self.epoch + m).permutation(f).tolist() for m, f in enumerate(self.folds)]

    def run(self, arm):
        orders = self._orders()
        nets, opts, gens = self.nets[arm], self.opts[arm], self.gens[arm]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if arm == "fold_graph":
            losses = feed.train_epoch_models(nets, self.store, self.folds, self.crit, opts, orders=orders,
                                             generators=gens, bags_per_step=self.k, graph=True, generic=True)
        elif arm == "eager":
            losses = feed.train_epoch_models(nets, self.store, self.folds, self.crit, opts, orders=orders,
                                             generators=gens, bags_per_step=self.k)
        else:
            losses = [feed.train_epoch(n, self.store, self.crit, o, order=orders[m], generator=gens[m],
                                       bags_per_step=self.k, graph=True, generic=True)
                      for m, (n, o) in enumerate(zip(nets, opts))]
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, losses

    def same(self, a, b):
        return all(torch.equal(u, v) for na, nb in zip(self.nets[a], self.nets[b])
                   for u, v in zip(na.parameters(), nb.parameters()))


def _replays(store, folds, D, k):
    """A recorded full step of the five folds (k bags each) and the five one-fold graphs of the same step."""
    torch.manual_seed(2)
    nets = [mil.MILNet(mil.FCLayer(D, 1), mil.BClassifier(D, 1)).cuda() for _ in range(FOLDS)]
    twins = [copy.deepcopy(n) for n in nets]
    crit = torch.nn.BCEWithLogitsLoss()
    cap = max(int(f.shape[0]) for f, _ in store.bags)
    fg = FoldTrainStepGraph(nets, crit, [_opt(n) for n in nets], [k] * FOLDS, cap, generic=True)
    gs = [TrainStepGraph(n, crit, _opt(n), k, cap, generic=True) for n in twins]
    for m in range(FOLDS):
        for b, i in enumerate(folds[m][:k]):
            x, y = store.bags[i]
            for slots, Ns, labels, at in ((fg.slots[m], fg.Ns, fg.labels, m * k + b), (gs[m].slots, gs[m].Ns,
                                                                                          gs[m].labels, b)):
                slots[b, :x.shape[0]].copy_(x)
                Ns[at].fill_(int(x.shape[0]))
                labels[at].copy_(y.view(-1))
    return fg, gs


def _profile(fn, steps):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        torch.cuda._sleep(100_000_000)   # lead-in: the kernel trace starts asynchronously
        torch.cuda.synchronize()
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    split = {"library": [0, 0.0], "optimizer_and_guard": [0, 0.0], "loss_and_other": [0, 0.0]}
    for e in p.events():
        if e.device_type != torch.autograd.DeviceType.CUDA or any(s in e.name for s in ("emset", "emcpy", "spin_kernel",
                                                                                          "sleep")):
            continue
        n = e.name
        part = ("library" if "dsmil::" in n else
                "optimizer_and_guard" if any(s in n for s in ("multi_tensor", "foreach", "Foreach", "CatArray",
                                                              "copy_kernel")) else "loss_and_other")
        split[part][0] += 1
        split[part][1] += e.time_range.elapsed_us()
    return {part: {"kernels": c / steps, "kernel_us": round(us / steps, 1)} for part, (c, us) in split.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"card": card(), "folds": FOLDS, "optimizer": "Adam(capturable, betas=(0.5, 0.9), wd=5e-3)"}
    for name in WORKLOADS:
        store, folds, D = _workload(name)
        for k in (1, 4):
            case = f"{name}_k{k}"
            fg, gs = _replays(store, folds, D, k)
            if a.profile:
                res.setdefault("profile_per_step", {})[case] = {
                    "fold_graph": _profile(fg.step, a.steps),
                    "one_fold_graphs": _profile(lambda: [g.step() for g in gs], a.steps)}
                continue
            rep = {"fold_graph": [], "one_fold_graphs": []}
            for _ in range(a.repeats):
                rep["fold_graph"].append(events_ms(fg.step, a.steps, 3))
                rep["one_fold_graphs"].append(events_ms(lambda: [g.step() for g in gs], a.steps, 3))
            res.setdefault("replay_ms_per_step", {})[case] = {arm: [round(v, 4) for v in vs] for arm, vs in rep.items()}
            ep = Epochs(store, folds, D, k)
            times, equal = {arm: [] for arm in ARMS}, []
            for r in range(a.repeats):
                losses = {}
                for arm in ARMS:
                    ms, losses[arm] = ep.run(arm)
                    times[arm].append(round(ms, 2))
                ep.epoch += 1
                equal.append({"one_fold_graphs": losses["fold_graph"] == losses["one_fold_graphs"]
                              and ep.same("fold_graph", "one_fold_graphs"),
                              "eager": losses["fold_graph"] == losses["eager"] and ep.same("fold_graph", "eager")})
            res.setdefault("epoch_ms", {})[case] = times
            res.setdefault("bits_equal_to_fold_graph", {})[case] = equal
            del fg, gs
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
