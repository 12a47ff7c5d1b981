"""Inference replayed as one CUDA graph (infer_graph.ForwardBagsGraph) against the eager calls, on three workloads:

  single_slide  one 10 000 x 512, C = 2 slide per call: `milnet(x)` against the nb = 1 graph's `run([x])`; a host clock
                around `--calls` calls and a final synchronise (a serving loop is bound by host launch time).
  bench_step    bench.py's workload, 16 x 10 000 x 512, C = 2: `milnet.forward_bags(xs)` against the 16-bag graph's
                `run(xs)`; CUDA events over `--calls` calls, and the host clock.
  eval_epoch    feed.eval_epoch over 64 such bags at bags_per_launch = 16: eager against graph=True (which records its
                graphs, one per group size, on every call); a host clock around each epoch, which ends in its one sync.

The arms alternate within each repeat, so the spread over repeats is the run-to-run noise.  Outputs are compared with
torch.equal in the same run.  Reads the card name and power limit in the same run.  Needs a GPU; prints one JSON object
(--out: also writes it).

    python tools/bench_infer_graph.py --calls 200 --repeats 3 --out /tmp/infer_graph.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import dsmil as mil  # noqa: E402
from dsmil_wsi_b200 import feed  # noqa: E402
from dsmil_wsi_b200.infer_graph import ForwardBagsGraph  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[torch.cuda.current_device()] if out else "unknown"


def host_ms(fn, calls, warm):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(calls):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / calls


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


def same(a, b):
    return all(torch.equal(u, v) for u, v in zip(a, b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200, help="timed calls per arm and repeat (single slide, bench step)")
    ap.add_argument("--epochs", type=int, default=5, help="timed eval epochs per arm and repeat")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_infer_graph needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    nb, N, D, Cc = 16, 10000, 512, 2
    g = torch.Generator(device=dev).manual_seed(0)
    torch.manual_seed(0)
    net = mil.MILNet(mil.FCLayer(D, Cc), mil.BClassifier(D, Cc)).to(dev).eval()
    xs = [torch.rand(N, D, generator=g, device=dev) for _ in range(nb)]
    store = feed.DeviceBagStore(D)
    for _ in range(64):
        store.add_bag(torch.rand(N, D, generator=g, device=dev), (torch.rand(Cc, generator=g, device=dev) > 0.5).float())
    crit = torch.nn.BCEWithLogitsLoss()
    g1, g16 = ForwardBagsGraph(net, 1, N), ForwardBagsGraph(net, nb, N)

    # the same bits, in this run
    with torch.no_grad():
        ref1 = [t.clone() for t in net(xs[0])]
        ref16 = [t.clone() for t in net.forward_bags(xs).packed]
    checks = {"single_slide": same(g1.run(xs[:1])[0], ref1), "bench_step": same(g16.run(xs).packed, ref16)}
    e_eval, g_eval = (feed.eval_epoch(net, store, crit, bags_per_launch=16, graph=gr) for gr in (False, True))
    checks["eval_epoch"] = (e_eval[0] == g_eval[0] and np.array_equal(e_eval[1], g_eval[1])
                            and np.array_equal(e_eval[2], g_eval[2]))

    def eager_one():
        with torch.no_grad():
            net(xs[0])

    def eager_bags():
        with torch.no_grad():
            net.forward_bags(xs)

    workloads = {
        "single_slide": {"eager_milnet": (host_ms, eager_one), "graph_nb1": (host_ms, lambda: g1.run(xs[:1]))},
        "bench_step": {"eager_forward_bags": (events_ms, eager_bags), "graph_nb16": (events_ms, lambda: g16.run(xs)),
                       "eager_forward_bags_host": (host_ms, eager_bags),
                       "graph_nb16_host": (host_ms, lambda: g16.run(xs))},
        "eval_epoch": {"eager": (host_ms, lambda: feed.eval_epoch(net, store, crit, bags_per_launch=16)),
                       "graph": (host_ms, lambda: feed.eval_epoch(net, store, crit, bags_per_launch=16, graph=True))},
    }
    ms = {w: {arm: [] for arm in arms} for w, arms in workloads.items()}
    for _ in range(a.repeats):
        for w, arms in workloads.items():
            calls, warm = (a.epochs, 1) if w == "eval_epoch" else (a.calls, a.warmup)
            for arm, (clock, fn) in arms.items():
                ms[w][arm].append(clock(fn, calls, warm))
    res = {"card": card(), "calls": a.calls, "epochs": a.epochs, "repeats": a.repeats,
           "shapes": {"single_slide": [1, N, D, Cc], "bench_step": [nb, N, D, Cc], "eval_epoch": [64, N, D, Cc, 16]},
           "ms": ms, "torch_equal": checks}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
