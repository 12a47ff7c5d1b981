"""Training step of a 16-bag minibatch (16 x 10 000 x 512, C = 2) through the row-sharded code at G = 1, three ways:
  sharded_batched  -- sharded_milnet_forward_bags + sharded_caller_loss_bags + backward + Adam (3 + 3 library calls and
                      6 collectives per step, whatever the batch)
  sharded_per_bag  -- the same 16 bags through the per-bag sharded_milnet_forward / sharded_caller_loss loop, gradients
                      accumulated, one Adam step (6 collectives and 8 library calls per bag)
  single_device    -- MILNet.forward_bags(grad=True) and train_epoch's minibatch loss, backward, Adam
The process group has one rank (NCCL), so the collectives cost their launch and synchronisation only: multi-GPU scaling
is not measured here.  The arms alternate within each repeat, so the spread over repeats is the run-to-run noise of the
machine.  Needs a GPU; prints one JSON object (--out: also writes it).

    python tools/bench_shard_train_bags.py --steps 10 --repeats 3 --out /tmp/shard_train_bags.json
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


def arms(net, opt, bags, labels):
    bce = torch.nn.BCEWithLogitsLoss()
    nb = len(bags)
    Ns = [int(x.shape[0]) for x in bags]
    zeros = [0] * nb

    def sharded_batched():
        opt.zero_grad()
        classes, pred, _, _, crit = sharded.sharded_milnet_forward_bags(net, bags, zeros)
        sharded.sharded_caller_loss_bags(classes, pred, crit, zeros, labels, bce, Ns=Ns).backward()
        opt.step()

    def sharded_per_bag():
        opt.zero_grad()
        for x, y in zip(bags, labels):
            classes, pred, _, _, crit = sharded.sharded_milnet_forward(net, x, 0)
            (sharded.sharded_caller_loss(classes, pred, crit, 0, y, bce) / nb).backward()
        opt.step()

    def single_device():
        opt.zero_grad()
        pred, mx = feed._group_predictions(net.forward_bags(bags, grad=True))
        (0.5 * bce(pred, labels) + 0.5 * bce(mx, labels)).backward()
        opt.step()

    return {"sharded_batched": sharded_batched, "sharded_per_bag": sharded_per_bag, "single_device": single_device}


def count_calls(fn):
    """Collectives and library kernel launches of one step."""
    counts = {"all_gather": 0, "all_reduce_sum": 0, "all_reduce_max": 0}
    real_g, real_r = dist.all_gather_into_tensor, dist.all_reduce

    def g(*a, **k):
        counts["all_gather"] += 1
        return real_g(*a, **k)

    def r(t, op=dist.ReduceOp.SUM, **k):
        counts["all_reduce_max" if op == dist.ReduceOp.MAX else "all_reduce_sum"] += 1
        return real_r(t, op=op, **k)
    dist.all_gather_into_tensor, dist.all_reduce = g, r
    try:
        n0 = _lib.launch_count()
        fn()
        torch.cuda.synchronize()
        counts["library_kernel_launches"] = _lib.launch_count() - n0
    finally:
        dist.all_gather_into_tensor, dist.all_reduce = real_g, real_r
    return counts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed steps per arm and repeat")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_shard_train_bags needs a CUDA device")
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
        opt = torch.optim.Adam(net.parameters(), lr=1e-4, betas=(0.5, 0.9), weight_decay=1e-3)
        fns = arms(net, opt, bags, labels)
        calls = {k: count_calls(fn) for k, fn in fns.items()}
        ms = {k: [] for k in fns}
        for _ in range(a.repeats):
            for k, fn in fns.items():
                ms[k].append(events_ms(fn, a.steps, a.warmup))
        res = {"card": card(), "gpus_visible": torch.cuda.device_count(), "ranks": 1,
               "multi_gpu_scaling": "not measured (one rank)", "nb": nb, "N": N, "D": D, "C": Cc,
               "steps": a.steps, "repeats": a.repeats, "step_ms": ms,
               "ms_per_bag": {k: [round(v / nb, 4) for v in vs] for k, vs in ms.items()}, "per_step_calls": calls}
    finally:
        dist.destroy_process_group()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
