"""The ensemble forward (ensemble.forward_bags_models, one dsmil_forward_bags_models call) against M sequential
`milnet_m.forward_bags(xs)` calls, on bench.py's workload: 16 bags x 10 000 x 512, C = 2, for M = 1, 2, 5.

CUDA events over `--calls` calls per arm; the arms alternate within each repeat, so the spread over repeats is the
run-to-run noise.  Outputs are compared with torch.equal in the same run, and the card name and power limit are read
in the same run.  Needs a GPU; prints one JSON object (--out: also writes it).

    python tools/bench_models.py --calls 50 --repeats 3 --out profiles/h100_models_1gpu.json
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
from dsmil_wsi_b200.ensemble import forward_bags_models  # noqa: E402


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50, help="timed calls per arm and repeat")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--models", default="1,2,5")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_models needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    nb, N, D, Cc = 16, 10000, 512, 2
    Ms = [int(m) for m in a.models.split(",")]
    g = torch.Generator(device=dev).manual_seed(0)
    torch.manual_seed(0)
    nets = [mil.MILNet(mil.FCLayer(D, Cc), mil.BClassifier(D, Cc)).to(dev).eval() for _ in range(max(Ms))]
    xs = [torch.rand(N, D, generator=g, device=dev) for _ in range(nb)]

    def looped(M):
        def run():
            with torch.no_grad():
                return [net.forward_bags(xs) for net in nets[:M]]
        return run

    def fused(M):
        return lambda: forward_bags_models(nets[:M], xs)

    # the same bits, in this run
    checks = {}
    for M in Ms:
        got, ref = fused(M)(), looped(M)()
        checks[str(M)] = all(all(torch.equal(u, v) for u, v in zip(o.packed, r.packed)) for o, r in zip(got, ref))
    ms = {str(M): {"fused": [], "loop": []} for M in Ms}
    for _ in range(a.repeats):
        for M in Ms:
            ms[str(M)]["fused"].append(events_ms(fused(M), a.calls, a.warmup))
            ms[str(M)]["loop"].append(events_ms(looped(M), a.calls, a.warmup))
    speedup = {M: min(v["loop"]) / min(v["fused"]) for M, v in ms.items()}
    res = {"card": card(), "calls": a.calls, "repeats": a.repeats, "shape": [nb, N, D, Cc],
           "ms_per_call": ms, "loop_over_fused_best": speedup, "torch_equal": checks}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
