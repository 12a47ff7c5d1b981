"""The batched value-network forward (passing_v) on 16 bags x 10 000 x 512, C = 2, nonlinear q.

    python tools/bench_value_bags.py [--repeats 3] [--steps 50] [--warmup 10] [--out F]

Arms, alternating within each repeat so that a drift of the clock or the power state spreads over all of them:
  loop         the per-bag `milnet(x)` loop (what MILNet.forward_bags ran for passing_v before the value route)
  batched      MILNet.forward_bags: one dsmil_value_forward_bags call, V by k_vproj_b (128 x 128 tile, 8 x 8 / thread)
  linear_b     the same call from a library built with DSMIL_VPROJ_LINEAR_B=1: V by k_linear_b (64 x 128, 4 x 8)
Each arm runs in its own process (the variant through DSMIL_B200_LIBPATH).  A step is CUDA-event time over `steps`
calls; the V kernel's time comes from a torch.profiler run of its own after the timed window, and its rate from the
2 N D^2 FLOPs of the projection (83.9 GFLOP per step).  Both batched arms must give the same output bits.  The card's
name, power limit and SM clock are read in the same run."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NB, N, D, C = 16, 10000, 512, 2
V_FLOP = 2.0 * NB * N * D * D


def child(arm, steps, warmup):
    import torch
    import dsmil as mil
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    net = mil.MILNet(mil.FCLayer(D, C), mil.BClassifier(D, C, nonlinear=True, passing_v=True)).to(dev).eval()
    g = torch.Generator(device=dev).manual_seed(100)
    bags = [torch.rand(N, D, generator=g, device=dev) for _ in range(NB)]
    run = (lambda: [net(x) for x in bags]) if arm == "loop" else (lambda: net.forward_bags(bags))
    with torch.no_grad():
        for _ in range(warmup):
            out = run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            out = run()
        e1.record()
        torch.cuda.synchronize()
        res = {"ms_per_step": e0.elapsed_time(e1) / steps}
        if arm != "loop":
            h = hashlib.sha256()
            for t in out.packed:
                h.update(t.cpu().numpy().tobytes())
            res["outputs_sha256"] = h.hexdigest()
            from torch.profiler import profile, ProfilerActivity
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(10):
                    run()
                torch.cuda.synchronize()
            name = "k_vproj_b" if arm == "batched" else "k_linear_b"
            us = [e.device_time_total / e.count for e in prof.key_averages()
                  if name in e.key and e.count and e.device_time_total > 0]
            # the V projection is the only k_linear_b launch on this shape (its Q-MLP runs in k_qmlp_sm90)
            if us:
                res["v_kernel"] = name
                res["v_kernel_ms"] = max(us) / 1e3
                res["v_kernel_tflops"] = V_FLOP / (max(us) * 1e-6) / 1e12
    print(json.dumps(res))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() or r.stderr.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", choices=["loop", "batched", "linear_b"], default=None)
    args = ap.parse_args()
    if args.child:
        return child(args.child, args.steps, args.warmup)
    from dsmil_wsi_b200 import build
    tmp = tempfile.TemporaryDirectory()
    variant = build.build_variant(os.path.join(tmp.name, "libdsmil_b200_linear_b.so"), ["DSMIL_VPROJ_LINEAR_B=1"])
    arms = [("loop", None), ("batched", None), ("linear_b", variant)]
    res = {"workload": f"{NB} bags x {N} x {D}, C = {C}, nonlinear q, passing_v, eval (no_grad)",
           "v_gflop_per_step": V_FLOP / 1e9, "steps": args.steps, "card_before": card(),
           "runs": {a: [] for a, _ in arms}}
    for rep in range(args.repeats):
        order = arms if rep % 2 == 0 else arms[::-1]
        for name, lib in order:
            env = dict(os.environ)
            if lib:
                env["DSMIL_B200_LIBPATH"] = lib
            else:
                env.pop("DSMIL_B200_LIBPATH", None)
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", name, "--steps", str(args.steps),
                                "--warmup", str(args.warmup)], capture_output=True, text=True, env=env, cwd=ROOT)
            if r.returncode != 0:
                raise RuntimeError(f"{name}: {r.stderr[-2000:]}")
            out = json.loads(r.stdout.strip().splitlines()[-1])
            res["runs"][name].append(out)
            print(rep, name, out, flush=True)
    res["card_after"] = card()
    shas = {o["outputs_sha256"] for a in ("batched", "linear_b") for o in res["runs"][a]}
    res["batched_arms_same_bits"] = len(shas) == 1
    summ = {}
    for a, runs in res["runs"].items():
        s = {"ms_per_step_min": min(o["ms_per_step"] for o in runs), "ms_per_step_max": max(o["ms_per_step"] for o in runs)}
        ks = [o["v_kernel_ms"] for o in runs if "v_kernel_ms" in o]
        if ks:
            s.update(v_kernel=runs[0]["v_kernel"], v_kernel_ms_min=min(ks), v_kernel_ms_max=max(ks),
                     v_kernel_tflops_best=V_FLOP / (min(ks) * 1e-3) / 1e12)
        summ[a] = s
    res["summary"] = summ
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")
    tmp.cleanup()
    if not res["batched_arms_same_bits"]:
        raise SystemExit("the two V kernels gave different bits")


if __name__ == "__main__":
    main()
