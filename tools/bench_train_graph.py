"""Training step per bag at k in {1, 4, 16} bags per step: the eager feed step against the same step replayed as one
CUDA graph (train_graph.TrainStepGraph), on bench_train_bags.py's two workloads: 16 x 10 000 x 512 at C = 2 and
16 x 15 000 x 512 at C = 1.  The eager arms are feed.train_epoch's step (k = 1: the per-bag loop, the reference's one
optimizer step per bag; k > 1: the minibatch step), once with the default Adam a user trains with (`eager_k*`) and once
with the capturable Adam the graph needs (`eager_capturable_k*`), whose step count lives on the device.  The graph arm copies each group's bags into the graph's slots (what
train_epoch(graph=True) does with the patch-dropout gather) and replays.  The arms alternate within each repeat, so the
spread over repeats is the run-to-run noise.  A separate torch.profiler run splits the graph step into kernel time and
the gaps between kernels.  Needs a GPU; prints one JSON object (--out: also writes it).

    python tools/bench_train_graph.py --steps 10 --repeats 3 --out /tmp/train_graph.json
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import dsmil as mil  # noqa: E402
from dsmil_wsi_b200 import feed  # noqa: E402
from dsmil_wsi_b200.train_graph import TrainStepGraph  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[torch.cuda.current_device()] if out else "unknown"


def events_ms(fn, reps, warm):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def eager_pass(net, opt, bags, labels, k):
    """One pass over the bags with feed.train_epoch's step at k bags per step (no patch dropout)."""
    crit = torch.nn.BCEWithLogitsLoss()

    def one_bag_steps():
        for x, y in zip(bags, labels):
            opt.zero_grad()
            ins, bag, _, _ = net(x)
            mx, _ = torch.max(ins, 0)
            loss = 0.5 * crit(bag.view(1, -1), y.view(1, -1)) + 0.5 * crit(mx.view(1, -1), y.view(1, -1))
            loss.backward()
            opt.step()

    def group_steps():
        for s in range(0, len(bags), k):
            opt.zero_grad()
            y = torch.stack(labels[s:s + k])
            pred, mx = feed._group_predictions(net.forward_bags(bags[s:s + k], grad=True))
            loss = feed.minibatch_loss(crit, pred, mx, y)
            loss.backward()
            opt.step()

    return one_bag_steps if k == 1 else group_steps


def graph_pass(graph, bags, labels, k):
    def run():
        for s in range(0, len(bags), k):
            for b, x in enumerate(bags[s:s + k]):
                graph.slots[b, :x.shape[0]].copy_(x)
                graph.Ns[b].fill_(x.shape[0])
            torch.stack(labels[s:s + k], out=graph.labels)
            graph.step()
    return run


def kernel_split(run, steps):
    """torch.profiler over `steps` graph passes over the 16 bags: kernel time, and the span from the first kernel's
    start to the last kernel's end; the gaps are span - kernel time.  The "_per_step" figures are per such pass."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            run()
        torch.cuda.synchronize()
    busy, lo, hi, n = 0.0, None, None, 0
    for e in prof.events():
        if getattr(e, "device_type", None) != torch.autograd.DeviceType.CUDA:
            continue
        busy += e.time_range.elapsed_us()
        lo = e.time_range.start if lo is None else min(lo, e.time_range.start)
        hi = e.time_range.end if hi is None else max(hi, e.time_range.end)
        n += 1
    span = (hi - lo) if n else 0.0
    return {"kernels_per_step": n / steps, "kernel_ms_per_step": busy / 1e3 / steps,
            "span_ms_per_step": span / 1e3 / steps, "gap_ms_per_step": (span - busy) / 1e3 / steps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed passes over the 16 bags per arm and repeat")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_train_graph needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = {"card": card(), "steps": a.steps, "repeats": a.repeats, "workloads": []}
    for nb, N, D, Cc in ((16, 10000, 512, 2), (16, 15000, 512, 1)):
        g = torch.Generator(device=dev).manual_seed(0)
        bags = [torch.rand(N, D, generator=g, device=dev) for _ in range(nb)]
        labels = [(torch.rand(Cc, generator=g, device=dev) > 0.5).float() for _ in range(nb)]
        torch.manual_seed(0)
        net = mil.MILNet(mil.FCLayer(D, Cc), mil.BClassifier(D, Cc)).to(dev).train()
        adam = dict(lr=1e-4, betas=(0.5, 0.9), weight_decay=1e-3)
        opt = torch.optim.Adam(net.parameters(), **adam)
        opt_cap = torch.optim.Adam(net.parameters(), **adam, capturable=True)
        crit = torch.nn.BCEWithLogitsLoss()
        arms = {}
        for k in (1, 4, 16):
            arms[f"eager_k{k}"] = eager_pass(net, opt, bags, labels, k)
            arms[f"eager_capturable_k{k}"] = eager_pass(net, opt_cap, bags, labels, k)
            arms[f"graph_k{k}"] = graph_pass(TrainStepGraph(net, crit, opt_cap, k, N), bags, labels, k)
        ms = {name: [] for name in arms}
        for _ in range(a.repeats):
            for name, fn in arms.items():
                ms[name].append(events_ms(fn, a.steps, a.warmup) / nb)
        split = {name: kernel_split(fn, a.steps) for name, fn in arms.items() if name.startswith("graph")}
        res["workloads"].append({"nb": nb, "N": N, "D": D, "C": Cc,
                                 "optimizer": {"eager_k*": f"Adam({adam})",
                                               "eager_capturable_k*, graph_k*": f"Adam({adam}, capturable=True)"},
                                 "train_ms_per_bag": ms,
                                 "graph_pass_profile": split})
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
