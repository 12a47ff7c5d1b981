"""Sweep of the SMs the overlapped forward leaves to the attend pass (DSMIL_PHASE1_RESERVE in abi.cu) on the bench
workload: 16 bags x 10 000 x 512, C = 2, MILNet.forward_bags, CUDA-event time per step.

    python tools/bench_fwd_overlap.py [--reserves 0,8,16,24,32,40,48] [--repeats 3] [--steps 200] [--libs DIR] [--out F]

One library per value is built into a temporary directory (or taken from DIR/r<value>/libdsmil_b200.so), and each arm
runs in its own process through DSMIL_B200_LIBPATH.  The arms alternate within each repeat, so a drift of the clock
or the power state spreads over all of them.  The arm "plain" is the in-tree library with kernel timing on, which
launches the attend pass after phase 1 (the schedule before the overlap).  The card's name, power limit and SM clock
are recorded in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def child(steps, warmup, plain):
    import torch
    from bench import make_params, make_net, NBAG, D
    from dsmil_wsi_b200 import _lib
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    net = make_net(make_params(), dev)
    g = torch.Generator(device=dev).manual_seed(100)
    bags = [torch.rand(NBAG, D, generator=g, device=dev) for _ in range(16)]
    if plain:
        lib.dsmil_profile_enable(1)
    with torch.no_grad():
        for _ in range(warmup):
            net.forward_bags(bags)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            net.forward_bags(bags)
        e1.record()
        torch.cuda.synchronize()
    # the plain launch runs phase 1 on every SM; the overlapped one on what the query reports
    ctas = torch.cuda.get_device_properties(0).multi_processor_count if plain else \
        int(lib.dsmil_forward_bags_phase1_ctas(16 * -(-NBAG // 128)))
    print(json.dumps({"ms_per_step": e0.elapsed_time(e1) / steps, "phase1_ctas": ctas}))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active"
    r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() or r.stderr.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reserves", default="0,8,16,24,32,40,48")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--libs", default=None, help="prebuilt DIR/r<value>/libdsmil_b200.so")
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", choices=["overlap", "plain"], default=None)
    args = ap.parse_args()
    if args.child:
        return child(args.steps, args.warmup, args.child == "plain")
    reserves = [int(r) for r in args.reserves.split(",")]
    tmp = None
    libs = {}
    if args.libs is None:
        from dsmil_wsi_b200 import build
        tmp = tempfile.TemporaryDirectory()
        for r in reserves:
            libs[r] = build.build_variant(os.path.join(tmp.name, f"libdsmil_b200_r{r}.so"), [f"DSMIL_PHASE1_RESERVE={r}"])
    else:
        libs = {r: os.path.join(args.libs, f"r{r}", "libdsmil_b200.so") for r in reserves}
    arms = [("plain", None)] + [(f"reserve_{r}", libs[r]) for r in reserves]
    res = {"workload": "16 bags x 10000 x 512, C = 2, MILNet.forward_bags (no_grad)", "steps": args.steps,
           "card_before": card(), "runs": {a: [] for a, _ in arms}}
    for rep in range(args.repeats):
        order = arms if rep % 2 == 0 else arms[::-1]
        for name, lib in order:
            env = dict(os.environ)
            if lib:
                env["DSMIL_B200_LIBPATH"] = lib
            else:
                env.pop("DSMIL_B200_LIBPATH", None)
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "plain" if lib is None else "overlap",
                                "--steps", str(args.steps), "--warmup", str(args.warmup)],
                               capture_output=True, text=True, env=env, cwd=ROOT)
            if r.returncode != 0:
                raise RuntimeError(f"{name}: {r.stderr[-2000:]}")
            out = json.loads(r.stdout.strip().splitlines()[-1])
            res["runs"][name].append(out["ms_per_step"])
            res.setdefault("phase1_ctas", {})[name] = out["phase1_ctas"]
            print(rep, name, out, flush=True)
    res["card_after"] = card()
    res["summary_ms_per_step"] = {a: {"min": min(v), "max": max(v)} for a, v in res["runs"].items()}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")
    if tmp is not None:
        tmp.cleanup()


if __name__ == "__main__":
    main()
