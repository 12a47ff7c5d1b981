"""Models with a value network (passing_v) as CUDA graphs against their eager forms.

    python tools/bench_value_graph.py [--repeats 3] [--steps 20] [--warmup 5] [--out F]

Workloads and arms (alternating within each repeat, so a drift of the clock or the power state spreads over all):
  musk_k{1,16}  a Musk-shaped training epoch: 92 bags of 2 to 40 rows, D = 166, C = 1, nonlinear q, dropout_v 0.2,
                SGD, k bags per step.  per_bag: feed.train_epoch (per-bag autograd); value: train_epoch(value=True);
                value_graph: train_epoch(graph=True, value=True), which records its graphs on every call, as a user
                pays it.
  wsi           one step of 16 bags x 10 000 x 512, C = 2, nonlinear q, dropout_v 0.2, Adam.  per_bag:
                MILNet.forward_bags(grad=True); value: functional.mil_forward_value_bags(grad=True); value_graph: a
                TrainStepGraph(value=True) replay (v's masks drawn into v_inputs before each replay).
  slide         inference of one 10 000 x 512 slide per call, eval mode: milnet(x), forward_bags([x]) and a
                ForwardBagsGraph(value=True) replay.
  eval64        an evaluation epoch of 64 bags of 2 000 to 10 000 rows, D = 512, 16 bags per launch: eval_epoch and
                eval_epoch(graph=True, value=True).
Every graph arm is compared with its eager value arm by torch.equal in the same run ("equal").  Times are CUDA-event
(or synchronised host clock) times; the card's name, power limit and SM clock are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable: {e}"
    return out


def _net(D, C, p_drop, seed=0):
    import torch
    from dsmil_wsi_b200.modules import BClassifier, FCLayer, MILNet
    torch.manual_seed(seed)
    return MILNet(FCLayer(D, C), BClassifier(D, C, dropout_v=p_drop, nonlinear=True, passing_v=True)).cuda().train()


def _timed(fn, reps):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def _flat(net):
    import torch
    return torch.cat([p.detach().reshape(-1) for p in net.parameters()])


def musk(k, arms, steps, warmup):
    import numpy as np
    import torch
    from dsmil_wsi_b200 import feed
    rs = np.random.RandomState(0)
    bags = [(int(rs.randint(0, 2)), rs.randn(int(rs.randint(2, 41)), 166).astype(np.float32)) for _ in range(92)]
    store = feed.mil_store(bags)
    crit = torch.nn.BCEWithLogitsLoss()
    order = list(range(92))
    out, finals = {}, {}
    for arm in arms:
        net = _net(166, 1, 0.2)
        opt = torch.optim.SGD(net.parameters(), lr=1e-3, momentum=0.9)
        kw = dict(order=order, bags_per_step=k, value=arm != "per_bag", graph=arm == "value_graph")
        torch.manual_seed(1)
        feed.mil_epoch_train(net, store, crit, opt, **kw)          # the epochs compared below
        finals[arm] = _flat(net)
        for _ in range(warmup):
            feed.mil_epoch_train(net, store, crit, opt, **kw)
        out[arm] = _timed(lambda: feed.mil_epoch_train(net, store, crit, opt, **kw), max(1, steps // 4))
    return {"ms_per_epoch": out, "equal": bool(torch.equal(finals["value"], finals["value_graph"]))}


def wsi(arms, steps, warmup):
    import torch
    from dsmil_wsi_b200 import feed
    from dsmil_wsi_b200 import functional as Fn
    from dsmil_wsi_b200.sharded import milnet_params
    from dsmil_wsi_b200.train_graph import TrainStepGraph
    nb, N, D, C = 16, 10000, 512, 2
    g = torch.Generator(device="cuda").manual_seed(0)
    bags = [torch.randn(N, D, device="cuda", generator=g) for _ in range(nb)]
    ys = (torch.rand(nb, C, device="cuda", generator=g) > 0.5).float()
    crit = torch.nn.BCEWithLogitsLoss()
    out, finals = {}, {}
    for arm in arms:
        net = _net(D, C, 0.2)
        opt = torch.optim.Adam(net.parameters(), lr=1e-4, capturable=True)
        bc = net.b_classifier
        if arm == "value_graph":
            sg = TrainStepGraph(net, crit, opt, nb, N, value=True)
            for b, x in enumerate(bags):
                sg.slots[b].copy_(x)
            sg.Ns.fill_(N)
            sg.labels.copy_(ys)

            def step():
                for b in range(nb):
                    bc._v_input(sg.slots[b], out=sg.v_inputs[b])
                sg.step()
        else:
            def step():
                opt.zero_grad(set_to_none=True)
                if arm == "per_bag":
                    outs = net.forward_bags(bags, grad=True)
                else:
                    vs = [bc._v_input(x) for x in bags]
                    outs, _ = Fn.mil_forward_value_bags(bags, milnet_params(net), vs, grad=True)
                loss = feed.minibatch_loss(crit, *feed._group_predictions(outs), ys)
                loss.backward()
                opt.step()
        torch.manual_seed(2)
        step()
        finals[arm] = _flat(net)
        for _ in range(warmup):
            step()
        out[arm] = _timed(step, steps)
    return {"ms_per_step": out, "equal": bool(torch.equal(finals["value"], finals["value_graph"]))}


def slide(steps, warmup):
    import torch
    from dsmil_wsi_b200.infer_graph import ForwardBagsGraph
    net = _net(512, 2, 0.2).eval()
    x = torch.randn(10000, 512, device="cuda")
    fg = ForwardBagsGraph(net, 1, 10000, value=True)
    fns = {"milnet": lambda: net(x), "forward_bags": lambda: net.forward_bags([x]), "graph": lambda: fg.run([x])}
    out = {}
    for name, fn in fns.items():
        for _ in range(warmup):
            fn()
        out[name] = _timed(fn, steps * 5)
    with torch.no_grad():
        ref = net.forward_bags([x]).packed
    equal = all(torch.equal(a, b) for a, b in zip(fg.run([x]).packed, ref))
    return {"ms_per_call": out, "equal": bool(equal)}


def eval64(steps, warmup):
    import numpy as np
    import torch
    from dsmil_wsi_b200 import feed
    store = feed.DeviceBagStore(512)
    g = torch.Generator(device="cuda").manual_seed(3)
    for i in range(64):
        n = 2000 + (i * 1297) % 8001
        store.add_bag(torch.randn(n, 512, device="cuda", generator=g), torch.tensor([float(i % 2), float(i % 3 == 0)]))
    net = _net(512, 2, 0.2)
    crit = torch.nn.BCEWithLogitsLoss()
    fns = {"eager": lambda: feed.eval_epoch(net, store, crit, bags_per_launch=16),
           "graph": lambda: feed.eval_epoch(net, store, crit, bags_per_launch=16, graph=True, value=True)}
    out = {}
    for name, fn in fns.items():
        for _ in range(warmup):
            fn()
        out[name] = _timed(fn, max(1, steps // 2))
    e, gr = fns["eager"](), fns["graph"]()
    equal = e[0] == gr[0] and np.array_equal(e[1], gr[1]) and np.array_equal(e[2], gr[2])
    return {"ms_per_epoch": out, "equal": bool(equal)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_value_graph.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    res = {"card_before": card(), "steps": args.steps, "runs": {}}
    arms = ["per_bag", "value", "value_graph"]
    for rep in range(args.repeats):
        a = arms if rep % 2 == 0 else arms[::-1]
        for key, fn in (("musk_k1", lambda: musk(1, a, args.steps, args.warmup)),
                        ("musk_k16", lambda: musk(16, a, args.steps, args.warmup)),
                        ("wsi", lambda: wsi(a, args.steps, args.warmup)),
                        ("slide", lambda: slide(args.steps, args.warmup)),
                        ("eval64", lambda: eval64(args.steps, args.warmup))):
            out = fn()
            res["runs"].setdefault(key, []).append(out)
            print(rep, key, out, flush=True)
    res["card_after"] = card()
    summ = {}
    for key, runs in res["runs"].items():
        unit = next(k for k in runs[0] if k.startswith("ms_"))
        summ[key] = {arm: [min(r[unit][arm] for r in runs), max(r[unit][arm] for r in runs)] for arm in runs[0][unit]}
        summ[key]["unit"] = unit
        summ[key]["equal_in_every_run"] = all(r["equal"] for r in runs)
    res["summary"] = summ
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
