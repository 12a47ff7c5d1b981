"""The fold step (feed.train_epoch_models' step: one ensemble.forward_bags_per_model call, one backward, M optimizer
steps) against the same M fold steps taken one after another, eagerly (milnet.forward_bags(grad=True), backward,
step) and as M TrainStepGraph replays.  Workload: 5 folds, each stepping on its own k bags of 10 000 x 512, C = 2,
at k = 1 and k = 4, SGD with momentum, no patch dropout.

CUDA events over `--steps` steps per arm; the arms alternate within each repeat, so the spread over repeats is the
run-to-run noise.  Before timing, one step of every arm from the same parameters is compared with torch.equal
(losses and updated parameters), and the card name and power limit are read in the same run.  Reports ms per
fold-bag (a step's time / (folds x k)).  Needs a GPU; prints one JSON object (--out: also writes it).

    python tools/bench_models_train.py --steps 20 --repeats 3 --out profiles/h100_models_train_1gpu.json
"""
import argparse
import copy
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import dsmil as mil  # noqa: E402
from dsmil_wsi_b200 import feed  # noqa: E402
from dsmil_wsi_b200.ensemble import forward_bags_per_model  # noqa: E402
from dsmil_wsi_b200.train_graph import TrainStepGraph  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[torch.cuda.current_device()] if out else "unknown"


def events_ms(fn, calls, warm):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


class Arms:
    """Three copies of the M fold models and optimizers, one per arm, over the same bags and labels."""

    def __init__(self, nets, bags, labels, N):
        self.bags, self.labels = bags, labels
        self.crit = torch.nn.BCEWithLogitsLoss()
        self.nets = {a: [copy.deepcopy(n) for n in nets] for a in ("fused", "eager", "graph")}
        self.opts = {a: [torch.optim.SGD(n.parameters(), lr=1e-3, momentum=0.9) for n in ns]
                     for a, ns in self.nets.items()}
        self.graphs = []
        for net, opt, xs, lab in zip(self.nets["graph"], self.opts["graph"], bags, labels):
            g = TrainStepGraph(net, self.crit, opt, len(xs), N)
            for b, x in enumerate(xs):
                g.slots[b].copy_(x)
                g.Ns[b].fill_(int(x.shape[0]))
            g.labels.copy_(lab)
            self.graphs.append(g)

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

    def eager(self):
        losses = []
        for net, opt, xs, lab in zip(self.nets["eager"], self.opts["eager"], self.bags, self.labels):
            opt.zero_grad()
            loss = feed.minibatch_loss(self.crit, *feed._group_predictions(net.forward_bags(xs, grad=True)), lab)
            loss.backward()
            opt.step()
            losses.append(loss.detach())
        return losses

    def graph(self):
        return [g.step().clone() for g in self.graphs]

    def same_bits(self):
        """One step of every arm from the parameters the copies share now: equal losses and parameters."""
        got = {a: getattr(self, a)() for a in ("fused", "eager", "graph")}
        ok = True
        for a in ("eager", "graph"):
            ok = ok and all(torch.equal(u, v) for u, v in zip(got["fused"], got[a]))
            for nf, na in zip(self.nets["fused"], self.nets[a]):
                ok = ok and all(torch.equal(u, v) for u, v in zip(nf.parameters(), na.parameters()))
        return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="timed steps per arm and repeat")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--folds", type=int, default=5)
    ap.add_argument("--k", default="1,4", help="bags per fold per step")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_models_train needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    N, D, Cc, M = 10000, 512, 2, a.folds
    ks = [int(k) for k in a.k.split(",")]
    g = torch.Generator(device=dev).manual_seed(0)
    torch.manual_seed(0)
    nets = [mil.MILNet(mil.FCLayer(D, Cc), mil.BClassifier(D, Cc)).to(dev).train() for _ in range(M)]
    res = {"card": card(), "steps": a.steps, "repeats": a.repeats, "folds": M, "bag": [N, D], "C": Cc,
           "optimizer": "SGD(momentum=0.9)", "ms_per_fold_bag": {}, "graph_over_fused_best": {},
           "eager_over_fused_best": {}, "torch_equal": {}}
    for k in ks:
        bags = [[torch.rand(N, D, generator=g, device=dev) for _ in range(k)] for _ in range(M)]
        labels = [(torch.rand(k, Cc, generator=g, device=dev) > 0.5).float() for _ in range(M)]
        arms = Arms(nets, bags, labels, N)
        res["torch_equal"][str(k)] = arms.same_bits()
        ms = {"fused": [], "eager": [], "graph": []}
        for _ in range(a.repeats):
            for arm in ms:
                ms[arm].append(events_ms(getattr(arms, arm), a.steps, a.warmup) / (M * k))
        res["ms_per_fold_bag"][str(k)] = ms
        res["graph_over_fused_best"][str(k)] = min(ms["graph"]) / min(ms["fused"])
        res["eager_over_fused_best"][str(k)] = min(ms["eager"]) / min(ms["fused"])
        del arms
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
