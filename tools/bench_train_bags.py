"""Training step per bag at bags_per_step in {1, 4, 16} (forward + backward + Adam), and the batched backward's own
time against its byte and FFMA floors, on two 16-bag workloads: 16 x 10 000 x 512 at C = 2 (bench.py's forward
workload) and 16 x 15 000 x 512 at C = 1 (Camelyon16-shaped).  The arms alternate within each repeat, so the spread
over repeats is the run-to-run noise of the machine.  Needs a GPU; prints one JSON object (--out: also writes it).

    python tools/bench_train_bags.py --steps 10 --repeats 3 --out /tmp/train_bags.json
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import dsmil as mil  # noqa: E402
from dsmil_wsi_b200 import _lib, feed  # noqa: E402
from dsmil_wsi_b200 import functional as Fn  # noqa: E402

HBM_BPS = 3.35e12          # H100 SXM data sheet, HBM3
FP32_FLOPS = 67e12         # H100 SXM data sheet, dense FP32


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


def step_fn(net, opt, bags, labels, k):
    crit = torch.nn.BCEWithLogitsLoss()

    def one_bag_steps():            # feed.train_epoch's bags_per_step = 1 loop, without the row permutation
        for x, y in zip(bags, labels):
            opt.zero_grad()
            ins, bag, _, _ = net(x)
            mx, _ = torch.max(ins, 0)
            loss = 0.5 * crit(bag.view(1, -1), y.view(1, -1)) + 0.5 * crit(mx.view(1, -1), y.view(1, -1))
            loss.backward()
            opt.step()

    def group_steps():              # feed.train_epoch's bags_per_step = k > 1 step
        for s in range(0, len(bags), k):
            opt.zero_grad()
            y = torch.stack(labels[s:s + k])
            pred, mx = feed._group_predictions(net.forward_bags(bags[s:s + k], grad=True))
            loss = 0.5 * crit(pred, y) + 0.5 * crit(mx, y)
            loss.backward()
            opt.step()

    return one_bag_steps if k == 1 else group_steps


def backward_call(net, bags):
    """dsmil_backward_bags alone over the whole batch, on the saved activations of one training forward, with the
    upstream gradients of the caller's loss (d_classes at the critical rows, d_pred)."""
    lib = _lib.load()
    ic, bc = net.i_classifier, net.b_classifier
    W1, b1, W2, b2 = bc._q_params()
    P = Fn.ParamPack(ic._linear().weight, ic._linear().bias, W1, b1, W2, b2, None, None, bc.fcc.weight, bc.fcc.bias)
    nb, Ns = len(bags), [int(x.shape[0]) for x in bags]
    total, Cc, D, dev = sum(Ns), P.C, P.D, P.device
    c_X, c_N = (C.c_void_p * nb)(*[x.data_ptr() for x in bags]), (C.c_int64 * nb)(*Ns)
    new = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
    classes, A, pred, B = new(total, Cc), new(total, Cc), new(nb, Cc), new(nb, Cc, D)
    crit = torch.empty(nb, Cc, dtype=torch.int64, device=dev)
    sQ, sH = new(total, 128), new(total, 128)
    ws = Fn._workspace(lib.dsmil_forward_bags_train_workspace_bytes(P.ref, c_N, nb), dev)
    _lib.check(lib.dsmil_forward_bags_train(P.ref, c_X, c_N, nb, classes.data_ptr(), pred.data_ptr(), A.data_ptr(),
                                            B.data_ptr(), crit.data_ptr(), sQ.data_ptr(), sH.data_ptr(),
                                            ws.data_ptr(), ws.numel(), Fn._stream()), "dsmil_forward_bags_train")
    first = torch.tensor([0] + Ns[:-1], device=dev).cumsum(0)
    dc = torch.zeros(total, Cc, device=dev)
    dc.scatter_(0, crit + first[:, None], 0.25 / (nb * Cc))
    dp = torch.full((nb, Cc), 0.25 / (nb * Cc), device=dev)
    grads = {n: torch.empty_like(t) for n, t in zip(("Wi", "bi", "W1", "b1", "W2", "b2", "Wf", "bf"),
                                                      (P.tensors[0], P.tensors[1], W1, b1, W2, b2, bc.fcc.weight,
                                                       bc.fcc.bias))}
    G = _lib.DsmilGrads(*[grads[n].data_ptr() for n in ("Wi", "bi", "W1", "b1", "W2", "b2")], None, None,
                        grads["Wf"].data_ptr(), grads["bf"].data_ptr(), None)
    wsb = Fn._workspace(lib.dsmil_backward_bags_workspace_bytes(P.ref, c_N, nb, 0), dev)

    def call():
        _lib.check(lib.dsmil_backward_bags(P.ref, c_X, c_N, nb, sQ.data_ptr(), sH.data_ptr(), A.data_ptr(),
                                           B.data_ptr(), crit.data_ptr(), dc.data_ptr(), dp.data_ptr(), None, None,
                                           C.byref(G), wsb.data_ptr(), wsb.numel(), Fn._stream()),
                   "dsmil_backward_bags")
    return call


def floors(nb, N, D):
    rows = nb * N
    x_bytes = rows * D * 4
    return {"x_bytes_two_passes": 2 * x_bytes, "byte_floor_ms": 2 * x_bytes / HBM_BPS * 1e3,
            "gW1_flop": 2 * rows * 128 * D, "ffma_floor_ms": 2 * rows * 128 * D / FP32_FLOPS * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed passes over the 16 bags per arm and repeat")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_train_bags needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = {"card": card(), "steps": a.steps, "repeats": a.repeats, "workloads": []}
    for nb, N, D, Cc in ((16, 10000, 512, 2), (16, 15000, 512, 1)):
        g = torch.Generator(device=dev).manual_seed(0)
        bags = [torch.rand(N, D, generator=g, device=dev) for _ in range(nb)]
        labels = [(torch.rand(Cc, generator=g, device=dev) > 0.5).float() for _ in range(nb)]
        torch.manual_seed(0)
        net = mil.MILNet(mil.FCLayer(D, Cc), mil.BClassifier(D, Cc)).to(dev).train()
        opt = torch.optim.Adam(net.parameters(), lr=1e-4, betas=(0.5, 0.9), weight_decay=1e-3)
        arms = {k: step_fn(net, opt, bags, labels, k) for k in (1, 4, 16)}
        bwd = backward_call(net, bags)
        ms = {k: [] for k in arms}
        ms_bwd = []
        for _ in range(a.repeats):
            for k, fn in arms.items():
                ms[k].append(events_ms(fn, a.steps, a.warmup) / nb)
            ms_bwd.append(events_ms(bwd, a.steps, a.warmup))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                bwd()
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", 0)
            if t > 0 and ("dsmil::" in e.key or "Memcpy" in e.key or "Memset" in e.key):
                kernels[e.key.split("(")[0].replace("void ", "")[:60]] = round(t / 1e3 / a.steps, 4)
        res["workloads"].append({
            "nb": nb, "N": N, "D": D, "C": Cc,
            "train_ms_per_bag": {str(k): v for k, v in ms.items()},
            "backward_bags_call_ms": ms_bwd,
            "backward_kernels_ms_per_call": kernels,
            **floors(nb, N, D)})
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
