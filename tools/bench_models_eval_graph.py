"""The validation half of a fold epoch: every fold model over its own held-out bags, as one call of
feed.eval_epoch_folds (replayed fold graphs, graph=True, or eager) against one eval_epoch per fold (graph=True or
eager), and the ensemble evaluation feed.eval_epoch_models eager against graph=True.

Workloads (synthetic features, seeded):
  tcga      5 folds, each validating 16 held-out bags of 2 000-10 000 rows, D = 512, C = 2, k = 16.
  musk1     92 bags of 2-40 rows, D = 166, C = 1, generic=True; the held-out tenths of folds 0-4 of a 10-fold split,
            each fold's BCEWithLogitsLoss with the pos_weight of its own training split (train_mil.py:172-173).
  ensemble  eval_epoch_models, M = 5 over 64 bags of 10 000 x 512, C = 2, k = 16.

Each call is timed with a host clock and ends in its own host sync.  Every arm runs once untimed first (the graph
arms record their graphs then, and later calls replay them), then the arms alternate within each of `--repeats`
repeats, `--calls` calls per arm each.  Every arm's results (loss, labels, predictions) are compared in the same run
with == and np.array_equal against those of the first arm.  The card name, power limit and max SM clock are read in
the same run.  Needs a GPU; prints one JSON object (--out: also writes it).

    python tools/bench_models_eval_graph.py --out profiles/h100_models_eval_graph_1gpu.json

--profile (a separate invocation: tracing slows the host) runs torch.profiler over `--calls` calls of each arm and
reports per call the kernels, their summed time and the span from the first kernel's start to the last one's end
less that time (the gaps).  In a process that has replayed a graph before, the profiler can miss some of a replay's
kernels, so the graph arms' counts are a floor.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import dsmil as mil  # noqa: E402
from dsmil_wsi_b200 import feed  # noqa: E402
from bench_models_train import card  # noqa: E402

FOLDS = 5


def _nets(D, C, M, seed):
    torch.manual_seed(seed)
    return [mil.MILNet(mil.FCLayer(D, C), mil.BClassifier(D, C)).cuda().eval() for _ in range(M)]


def _sub_store(store, fold):
    sub = feed.DeviceBagStore(store.D, device=store.device)
    sub.bags = [store.bags[i] for i in fold]
    return sub


def tcga():
    rng = np.random.default_rng(0)
    D, C = 512, 2
    store = feed.DeviceBagStore(D)
    for i in range(16 * FOLDS):
        n = int(rng.integers(2000, 10001))
        store.add_bag(torch.from_numpy(rng.random((n, D), dtype=np.float32)),
                      torch.from_numpy((rng.random(C) > 0.5).astype(np.float32)))
    folds = [list(range(16 * m, 16 * (m + 1))) for m in range(FOLDS)]
    crit = [torch.nn.BCEWithLogitsLoss()] * FOLDS
    return store, folds, _nets(D, C, FOLDS, 1), crit, dict(bags_per_launch=16)


def musk1():
    rng = np.random.default_rng(1)
    D, nb = 166, 92
    store = feed.DeviceBagStore(D)
    labels = [i % 2 for i in range(nb)]
    for i in range(nb):
        n = int(rng.integers(2, 41))
        store.add_bag(torch.from_numpy(rng.random((n, D), dtype=np.float32)), torch.tensor([float(labels[i])]))
    order = rng.permutation(nb).tolist()
    folds, crit = [], []
    for f in range(FOLDS):
        train, test = feed.cross_validation_set(order, 10, f)
        folds.append(test)
        pw = feed.compute_pos_weight([(labels[i], None) for i in train])
        crit.append(torch.nn.BCEWithLogitsLoss(pos_weight=torch.tensor([pw], device="cuda")))
    return store, folds, _nets(D, 1, FOLDS, 2), crit, dict(bags_per_launch=16, generic=True)


def fold_arms(store, folds, nets, crit, kw):
    generic = kw.get("generic", False)
    k = kw["bags_per_launch"]
    subs = [_sub_store(store, f) for f in folds]
    return {
        "eval_epoch_folds_graph": lambda: feed.eval_epoch_folds(nets, store, folds, crit, graph=True, **kw),
        "eval_epoch_graph_x5": lambda: [feed.eval_epoch(n, s, c, bags_per_launch=k, graph=True, generic=generic)
                                        for n, s, c in zip(nets, subs, crit)],
        "eval_epoch_folds_eager": lambda: feed.eval_epoch_folds(nets, store, folds, crit, **kw),
        "eval_epoch_eager_x5": lambda: [feed.eval_epoch(n, s, c, bags_per_launch=k) for n, s, c in zip(nets, subs, crit)],
    }


def ensemble():
    rng = np.random.default_rng(3)
    D, C = 512, 2
    store = feed.DeviceBagStore(D)
    for _ in range(64):
        store.add_bag(torch.from_numpy(rng.random((10_000, D), dtype=np.float32)),
                      torch.from_numpy((rng.random(C) > 0.5).astype(np.float32)))
    nets, crit = _nets(D, C, FOLDS, 4), torch.nn.BCEWithLogitsLoss()
    return {"eval_epoch_models_eager": lambda: feed.eval_epoch_models(nets, store, crit, bags_per_launch=16),
            "eval_epoch_models_graph": lambda: feed.eval_epoch_models(nets, store, crit, bags_per_launch=16,
                                                                      graph=True)}


def _same(a, b):
    return all(x[0] == y[0] and np.array_equal(x[1], y[1]) and np.array_equal(x[2], y[2]) for x, y in zip(a, b))


def _time(arms, repeats, calls):
    first = {arm: fn() for arm, fn in arms.items()}          # untimed: the graph arms record here
    ref = next(iter(first.values()))
    times, equal = {arm: [] for arm in arms}, []
    for _ in range(repeats):
        out = {}
        for arm, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(calls):
                out[arm] = fn()                                 # each call ends in its host sync
            times[arm].append(round((time.perf_counter() - t0) * 1e3 / calls, 3))
        equal.append({arm: _same(ref, r) for arm, r in out.items()})
    return {"ms_per_call": times, "results_equal_to_first_arm": equal}


def _profile(fn, calls):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        torch.cuda._sleep(100_000_000)   # lead-in: the kernel trace starts asynchronously
        torch.cuda.synchronize()
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    ev = sorted((e for e in p.events() if e.device_type == torch.autograd.DeviceType.CUDA
                 and not any(s in e.name for s in ("emset", "emcpy", "sleep"))), key=lambda e: e.time_range.start)
    busy = sum(e.time_range.elapsed_us() for e in ev)
    lib = [e for e in ev if "dsmil::" in e.name]
    span = (ev[-1].time_range.end - ev[0].time_range.start) if ev else 0
    return {"kernels": len(ev) / calls, "library_kernels": len(lib) / calls,
            "kernel_us": round(busy / calls, 1), "library_kernel_us": round(sum(e.time_range.elapsed_us()
                                                                               for e in lib) / calls, 1),
            "gaps_us": round((span - busy) / calls, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"card": card(), "folds": FOLDS}
    work = {"tcga": lambda: fold_arms(*tcga()), "musk1": lambda: fold_arms(*musk1()), "ensemble": ensemble}
    for name, make in work.items():
        arms = make()
        if a.profile:
            res.setdefault("profile_per_call", {})[name] = {arm: _profile(fn, a.calls) for arm, fn in arms.items()}
        else:
            res[name] = _time(arms, a.repeats, a.calls)
        del arms
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
