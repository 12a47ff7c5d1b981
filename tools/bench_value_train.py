"""Training steps of a model with a value network (passing_v): the per-bag autograd against the batched backward.

    python tools/bench_value_train.py [--repeats 3] [--steps 20] [--warmup 5] [--out F]

Workloads:
  wsi    16 bags x 10 000 x 512, C = 2, nonlinear q, Adam, dropout_v 0 and 0.2: one minibatch step
  musk   a Musk-shaped epoch: 92 bags of 2 to 40 rows, D = 166, C = 1, nonlinear q, dropout_v 0.2, minibatches of 16
         bags, then one evaluation over all 92 through MILNet.forward_bags (the same in both arms)
Arms, alternating within each repeat so that a drift of the clock or the power state spreads over both:
  per_bag  MILNet.forward_bags(grad=True): milnet(x) per bag, one dsmil_forward and dsmil_backward per bag
  batched  functional.mil_forward_value_bags(grad=True): one dsmil_value_forward_bags and one
           dsmil_value_backward_bags per minibatch, v's masks drawn per bag beforehand
A step is CUDA-event time over `steps` calls.  The gWv kernel's time comes from a torch.profiler run of its own after
the timed window: gWv = dzv^T Xv is the largest k_gemm_tn_rag launch of a batched wsi step (gW1's has 4x fewer
tiles), against its floor of 2 N D^2 = 83.9 GFLOP at the data sheet's 67 TFLOP/s FP32 (1.25 ms).  The card's name,
power limit and SM clock are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WSI = dict(nb=16, N=10000, D=512, C=2)
GWV_FLOP = 2.0 * WSI["nb"] * WSI["N"] * WSI["D"] ** 2
FP32_PEAK = 67e12


def _net(D, C, p_drop, dev):
    import torch
    import dsmil as mil
    torch.manual_seed(0)
    return mil.MILNet(mil.FCLayer(D, C), mil.BClassifier(D, C, dropout_v=p_drop, nonlinear=True,
                                                          passing_v=True)).to(dev).train()


def _params(net):
    from dsmil_wsi_b200.sharded import milnet_params
    return milnet_params(net)


def _step_fn(arm, net, opt, bags, ys):
    import torch
    from dsmil_wsi_b200 import functional as Fn
    bc = net.b_classifier

    def step():
        opt.zero_grad(set_to_none=True)
        if arm == "per_bag":
            outs = net.forward_bags(bags, grad=True)
            pred = torch.cat([o[1] for o in outs])
        else:
            ms = vs = None
            if bc.v[0].p > 0:
                ms = [bc.v[0](torch.ones_like(x)) for x in bags]
                vs = [x * m for x, m in zip(bags, ms)]
            outs, _ = Fn.mil_forward_value_bags(bags, _params(net), vs, grad=True, v_masks=ms)
            pred = outs.packed[1]
        torch.nn.functional.binary_cross_entropy_with_logits(pred, ys).backward()
        opt.step()
    return step


def _timed(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def wsi_arm(arm, p_drop, steps, warmup, dev):
    import torch
    W = WSI
    net = _net(W["D"], W["C"], p_drop, dev)
    opt = torch.optim.Adam(net.parameters(), lr=1e-4)
    g = torch.Generator(device=dev).manual_seed(100)
    bags = [torch.rand(W["N"], W["D"], generator=g, device=dev) for _ in range(W["nb"])]
    ys = (torch.rand(W["nb"], W["C"], generator=g, device=dev) > 0.5).float()
    fn = _step_fn(arm, net, opt, bags, ys)
    res = {"ms_per_step": _timed(fn, steps, warmup)}
    if arm == "batched":
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
        rag = [e.device_time_total for e in prof.events() if "k_gemm_tn_rag" in e.name and e.device_time_total > 0]
        rag.sort(reverse=True)
        if len(rag) >= 5:
            ms = sum(rag[:5]) / 5 / 1e3   # the five gWv launches are the five largest
            res.update(gwv_kernel_ms=ms, gwv_tflops=GWV_FLOP / (ms * 1e-3) / 1e12,
                       gwv_share_of_fp32_floor=(GWV_FLOP / FP32_PEAK) / (ms * 1e-3))
    return res


def musk_arm(arm, steps, warmup, dev):
    import torch
    D, C, nb, mb = 166, 1, 92, 16
    net = _net(D, C, 0.2, dev)
    opt = torch.optim.Adam(net.parameters(), lr=1e-4)
    g = torch.Generator(device=dev).manual_seed(7)
    Ns = (2 + torch.randint(0, 39, (nb,), generator=g, device=dev)).tolist()
    bags = [torch.rand(n, D, generator=g, device=dev) for n in Ns]
    ys = (torch.rand(nb, C, generator=g, device=dev) > 0.5).float()
    steps_fns = [_step_fn(arm, net, opt, bags[i:i + mb], ys[i:i + mb]) for i in range(0, nb, mb)]

    def epoch():
        net.train()
        for f in steps_fns:
            f()
        net.eval()
        net.forward_bags(bags)   # evaluation: the batched inference of both arms, so the arms differ in training only
    return {"ms_per_epoch": _timed(epoch, steps, warmup)}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() or r.stderr.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_value_train.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda", 0)
    res = {"card_before": card(), "steps": args.steps, "gwv_gflop_per_step": GWV_FLOP / 1e9,
           "gwv_floor_ms_at_67_tflops": GWV_FLOP / FP32_PEAK * 1e3, "runs": {}}
    arms = ["per_bag", "batched"]
    for rep in range(args.repeats):
        for arm in (arms if rep % 2 == 0 else arms[::-1]):
            for p_drop in (0.0, 0.2):
                key = f"wsi_p{p_drop}_{arm}"
                out = wsi_arm(arm, p_drop, args.steps, args.warmup, dev)
                res["runs"].setdefault(key, []).append(out)
                print(rep, key, out, flush=True)
            key = f"musk_{arm}"
            out = musk_arm(arm, args.steps, args.warmup, dev)
            res["runs"].setdefault(key, []).append(out)
            print(rep, key, out, flush=True)
    res["card_after"] = card()
    summ = {}
    for key, runs in res["runs"].items():
        unit = "ms_per_step" if "ms_per_step" in runs[0] else "ms_per_epoch"
        s = {f"{unit}_min": min(o[unit] for o in runs), f"{unit}_max": max(o[unit] for o in runs)}
        ks = [o["gwv_kernel_ms"] for o in runs if "gwv_kernel_ms" in o]
        if ks:
            s.update(gwv_kernel_ms_min=min(ks), gwv_kernel_ms_max=max(ks),
                     gwv_tflops_best=GWV_FLOP / (min(ks) * 1e-3) / 1e12)
        summ[key] = s
    res["summary"] = summ
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
