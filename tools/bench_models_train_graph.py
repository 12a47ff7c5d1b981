"""The fold step replayed as one CUDA graph (train_graph.FoldTrainStepGraph) against the same M fold steps as M
TrainStepGraph replays and as the eager fold step (feed.train_epoch_models' step).  Workload: M folds, each stepping
on its own k bags of 10 000 x 512, C = 2, SGD with momentum, no patch dropout: (M, k) = (5, 1), (5, 4) and (2, 1).

CUDA events over `--steps` steps per arm; the arms alternate within each repeat, so the spread over repeats is the
run-to-run noise.  Before timing, one step of every arm from the same parameters is compared with torch.equal
(losses and updated parameters), and the card name, power limit and max SM clock are read in the same run.  Reports
ms per fold-bag (a step's time / (folds x k)) as ranges over the repeats.  Needs a GPU; prints one JSON object
(--out: also writes it).

    python tools/bench_models_train_graph.py --out profiles/h100_models_train_graph_1gpu.json

--profile (a separate invocation: tracing slows the host) runs torch.profiler over `--steps` steps of the fold graph
and of the M replays and reports, per step: the kernel count, the summed kernel time, the gaps (the span from the
first kernel's start to the last one's end, less the kernel time), and the time of the planner kernel, of the
library's other kernels and of everything else (the loss and the M optimizer steps).
"""
import argparse
import copy
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import dsmil as mil  # noqa: E402
from dsmil_wsi_b200 import feed  # noqa: E402
from dsmil_wsi_b200.ensemble import forward_bags_per_model  # noqa: E402
from dsmil_wsi_b200.train_graph import FoldTrainStepGraph, TrainStepGraph  # noqa: E402
from bench_models_train import card, events_ms  # noqa: E402

ARMS = ("fold_graph", "graphs", "fused")


class Arms:
    """Three copies of the M fold models and optimizers, one per arm, over the same bags and labels."""

    def __init__(self, nets, bags, labels, N):
        self.bags, self.labels = bags, labels
        self.crit = torch.nn.BCEWithLogitsLoss()
        self.nets = {a: [copy.deepcopy(n) for n in nets] for a in ARMS}
        self.opts = {a: [torch.optim.SGD(n.parameters(), lr=1e-3, momentum=0.9) for n in ns]
                     for a, ns in self.nets.items()}
        self.singles = []
        for net, opt, xs, lab in zip(self.nets["graphs"], self.opts["graphs"], bags, labels):
            g = TrainStepGraph(net, self.crit, opt, len(xs), N)
            for b, x in enumerate(xs):
                g.slots[b].copy_(x)
                g.Ns[b].fill_(int(x.shape[0]))
            g.labels.copy_(lab)
            self.singles.append(g)
        self.fold = FoldTrainStepGraph(self.nets["fold_graph"], self.crit, self.opts["fold_graph"],
                                       [len(xs) for xs in bags], N)
        e = 0
        for m, (xs, lab) in enumerate(zip(bags, labels)):
            for b, x in enumerate(xs):
                self.fold.slots[m][b].copy_(x)
                self.fold.Ns[e + b].fill_(int(x.shape[0]))
            self.fold.labels[e:e + len(xs)].copy_(lab)
            e += len(xs)

    def fold_graph(self):
        return list(self.fold.step().clone())

    def graphs(self):
        return [g.step().clone() for g in self.singles]

    def fused(self):
        nets, opts = self.nets["fused"], self.opts["fused"]
        for o in opts:
            o.zero_grad()
        outs = forward_bags_per_model(nets, self.bags, grad=True)
        losses = [feed.minibatch_loss(self.crit, *feed._group_predictions(out), lab)
                  for out, lab in zip(outs, self.labels)]
        sum(losses[1:], losses[0]).backward()
        for o in opts:
            o.step()
        return [l.detach() for l in losses]

    def same_bits(self):
        """One step of every arm from the parameters the copies share now: equal losses and parameters."""
        got = {a: getattr(self, a)() for a in ARMS}
        ok = int(self.fold.status.abs().sum()) == 0
        for a in ARMS[1:]:
            ok = ok and all(torch.equal(u, v) for u, v in zip(got["fold_graph"], got[a]))
            for nf, na in zip(self.nets["fold_graph"], self.nets[a]):
                ok = ok and all(torch.equal(u, v) for u, v in zip(nf.parameters(), na.parameters()))
        return ok


def profile(fn, steps):
    """Per step of fn, from the device-side kernel records of torch.profiler."""
    from torch.profiler import ProfilerActivity, profile as prof
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    with prof(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as p:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    ks = sorted(((e.time_range.start, e.time_range.end, e.name) for e in p.events()
                 if e.device_type == torch.autograd.DeviceType.CUDA and "mem" not in e.name.lower()),
                key=lambda t: t[0])
    busy = sum(e - s for s, e, _ in ks)
    span = ks[-1][1] - ks[0][0]
    plan = sum(e - s for s, e, n in ks if "k_plan_bags" in n)
    lib = sum(e - s for s, e, n in ks if "dsmil" in n) - plan
    per = lambda us: round(us / steps, 2)
    return {"kernels": round(len(ks) / steps, 1), "kernel_us": per(busy), "gap_us": per(span - busy),
            "planner_us": per(plan), "library_us": per(lib), "loss_and_optimizer_us": per(busy - lib - plan)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed steps per arm and repeat")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--cases", default="5x1,5x4,2x1", help="folds x bags per fold per step")
    ap.add_argument("--profile", action="store_true", help="the torch.profiler breakdown instead of the timing")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_models_train_graph needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    N, D, Cc = 10000, 512, 2
    g = torch.Generator(device=dev).manual_seed(0)
    torch.manual_seed(0)
    res = {"card": card(), "steps": a.steps, "repeats": a.repeats, "bag": [N, D], "C": Cc,
           "optimizer": "SGD(momentum=0.9)", "torch_equal": {}}
    res["profile_per_step" if a.profile else "ms_per_fold_bag"] = {}
    for case in a.cases.split(","):
        M, k = (int(v) for v in case.split("x"))
        nets = [mil.MILNet(mil.FCLayer(D, Cc), mil.BClassifier(D, Cc)).to(dev).train() for _ in range(M)]
        bags = [[torch.rand(N, D, generator=g, device=dev) for _ in range(k)] for _ in range(M)]
        labels = [(torch.rand(k, Cc, generator=g, device=dev) > 0.5).float() for _ in range(M)]
        arms = Arms(nets, bags, labels, N)
        res["torch_equal"][case] = arms.same_bits()
        if a.profile:
            res["profile_per_step"][case] = {arm: profile(getattr(arms, arm), a.steps) for arm in ARMS[:2]}
        else:
            ms = {arm: [] for arm in ARMS}
            for _ in range(a.repeats):
                for arm in ARMS:
                    ms[arm].append(round(events_ms(getattr(arms, arm), a.steps, a.warmup) / (M * k), 4))
            res["ms_per_fold_bag"][case] = ms
        del arms
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
