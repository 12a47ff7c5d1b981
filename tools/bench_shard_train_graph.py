"""Training step per bag of the row-sharded minibatch step, eager against one CUDA graph, at k in {1, 4, 16} bags per
step on 16 x 10 000 x 512, C = 2 (bench_shard_train_bags.py's workload).  Three arms per k, alternating within each
repeat, so the spread over repeats is the run-to-run noise:
  sharded_eager_k*  -- sharded_milnet_forward_bags + sharded_caller_loss_bags + backward + Adam (6 library calls and 6
                       collectives per step)
  sharded_graph_k*  -- the same step recorded once as train_graph.ShardedTrainStepGraph and replayed
  single_graph_k*   -- the single-device step replayed as train_graph.TrainStepGraph
The graph arms copy each group's bags into the graph's slots and replay.  All arms use the capturable Adam the graphs
need.  The process group has one rank (NCCL), so the collectives cost their launch and synchronisation only: multi-GPU
scaling is not measured here.  Per arm it reports the library launches per step (per replay: 0 for the graph arms) and
the collectives per step (the graph arm's: those recorded, counted while the step is captured).  Needs a GPU; prints
one JSON object (--out: also writes it).

    python tools/bench_shard_train_graph.py --steps 5 --repeats 3 --out /tmp/shard_train_graph.json
"""
import argparse
import json
import os
import socket
import subprocess
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import dsmil as mil  # noqa: E402
from dsmil_wsi_b200 import _lib, feed, sharded  # noqa: E402
from dsmil_wsi_b200.train_graph import ShardedTrainStepGraph, TrainStepGraph  # noqa: E402


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


class Counter:
    """Collectives issued while active (all-gathers, all-reduce(sum), all-reduce(max))."""

    def __enter__(self):
        self.counts = {"all_gather": 0, "all_reduce_sum": 0, "all_reduce_max": 0}
        self.real = dist.all_gather_into_tensor, dist.all_reduce

        def g(*a, **k):
            self.counts["all_gather"] += 1
            return self.real[0](*a, **k)

        def r(t, op=dist.ReduceOp.SUM, **k):
            self.counts["all_reduce_max" if op == dist.ReduceOp.MAX else "all_reduce_sum"] += 1
            return self.real[1](t, op=op, **k)
        dist.all_gather_into_tensor, dist.all_reduce = g, r
        return self

    def __exit__(self, *exc):
        dist.all_gather_into_tensor, dist.all_reduce = self.real


def eager_pass(net, opt, bags, labels, k):
    bce = torch.nn.BCEWithLogitsLoss()

    def run():
        for s in range(0, len(bags), k):
            xs, y = bags[s:s + k], labels[s:s + k]
            zeros = [0] * len(xs)
            opt.zero_grad()
            classes, pred, _, _, crit = sharded.sharded_milnet_forward_bags(net, xs, zeros)
            sharded.sharded_caller_loss_bags(classes, pred, crit, zeros, y, bce,
                                             Ns=[int(x.shape[0]) for x in xs]).backward()
            opt.step()
    return run


def graph_pass(graph, bags, labels, k):
    def run():
        for s in range(0, len(bags), k):
            for b, x in enumerate(bags[s:s + k]):
                graph.slots[b, :x.shape[0]].copy_(x)
                graph.Ns[b].fill_(x.shape[0])
            graph.labels.copy_(labels[s:s + k])
            graph.step()
    return run


def calls_per_step(run, steps):
    """Library launches and collectives per step of one pass (`steps` steps)."""
    torch.cuda.synchronize()
    with Counter() as c:
        n0 = _lib.launch_count()
        run()
        torch.cuda.synchronize()
        n = _lib.launch_count() - n0
    return {"library_kernel_launches": n / steps, **{k: v / steps for k, v in c.counts.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="timed passes over the 16 bags per arm and repeat")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_shard_train_graph needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1, device_id=dev)
    try:
        nb, N, D, Cc = 16, 10000, 512, 2
        g = torch.Generator(device=dev).manual_seed(0)
        bags = [torch.rand(N, D, generator=g, device=dev) for _ in range(nb)]
        labels = (torch.rand(nb, Cc, generator=g, device=dev) > 0.5).float()
        torch.manual_seed(0)
        net = mil.MILNet(mil.FCLayer(D, Cc), mil.BClassifier(D, Cc)).to(dev).train()
        adam = dict(lr=1e-4, betas=(0.5, 0.9), weight_decay=1e-3, capturable=True)
        opt = torch.optim.Adam(net.parameters(), **adam)
        bce = torch.nn.BCEWithLogitsLoss()
        arms, calls = {}, {}
        for k in (1, 4, 16):
            arms[f"sharded_eager_k{k}"] = eager_pass(net, opt, bags, labels, k)
            with Counter() as c:                                # one warm-up step and the captured step
                sg = ShardedTrainStepGraph(net, bce, opt, k, N, warmup=1)
            arms[f"sharded_graph_k{k}"] = graph_pass(sg, bags, labels, k)
            arms[f"single_graph_k{k}"] = graph_pass(TrainStepGraph(net, bce, opt, k, N), bags, labels, k)
            for name in (f"sharded_eager_k{k}", f"sharded_graph_k{k}", f"single_graph_k{k}"):
                calls[name] = calls_per_step(arms[name], nb // k)
            calls[f"sharded_graph_k{k}"]["collectives_recorded"] = {n: v / 2 for n, v in c.counts.items()}
        ms = {name: [] for name in arms}
        for _ in range(a.repeats):
            for name, fn in arms.items():
                ms[name].append(round(events_ms(fn, a.steps, a.warmup) / nb, 4))
        res = {"card": card(), "gpus_visible": torch.cuda.device_count(), "ranks": 1,
               "multi_gpu_scaling": "not measured (one rank)", "nb": nb, "N": N, "D": D, "C": Cc,
               "optimizer": f"Adam({adam})", "steps": a.steps, "repeats": a.repeats, "train_ms_per_bag": ms,
               "per_step_calls": calls}
    finally:
        dist.destroy_process_group()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
