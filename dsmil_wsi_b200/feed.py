"""Caller-side bag feed for training (SURVEY §8f-1; reference train_tcga.py:55-83).

The reference's training loop pays, per bag and per epoch: `torch.load(item, map_location='cuda:0')` (disk ->
GPU), a CPU `torch.randperm` + advanced-indexing gather for `dropout_patches`, and a `loss.item()` sync.  Once
the operator takes tens of microseconds those dominate.  Here the bags of the `.pt` cache format
(`[N, D + C]` = features || label repeated per row, train_tcga.py:36-51) live on the device, the patch-dropout
permutation is drawn on the device and applied by `dsmil_gather_rows` (our kernel), and the running loss stays
on the device until the epoch ends.
"""
from __future__ import annotations

import weakref
from typing import Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from . import functional as Fn
from .modules import milnet_params


def gather_rows(feats: torch.Tensor, idx: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[m] = feats[idx[m]] on the device (== `feats[idx]` of train_tcga.py:82).  `out`: a contiguous float32
    [len(idx), D] tensor on the same device to write into (e.g. a slot of a recorded training step)."""
    Fn.require_cuda(feats, "feats")
    feats = Fn._f32c(feats)
    idx = idx.to(device=feats.device, dtype=torch.int64).contiguous()
    M, D = int(idx.numel()), int(feats.shape[1])
    if out is not None and (tuple(out.shape) != (M, D) or out.dtype != torch.float32 or not out.is_contiguous()
                            or out.device != feats.device):
        raise ValueError(f"out must be a contiguous float32 [{M}, {D}] tensor on {feats.device}, got "
                         f"{out.dtype} {tuple(out.shape)} on {out.device}")
    with torch.cuda.device(feats.device):
        if out is None:
            out = torch.empty(M, D, dtype=torch.float32, device=feats.device)
        _lib.check(_lib.load().dsmil_gather_rows(feats.data_ptr(), int(feats.shape[0]), D, idx.data_ptr(), M,
                                                 out.data_ptr(), Fn._stream()), "dsmil_gather_rows")
    return out


def dropout_patches(feats: torch.Tensor, p: float, generator: Optional[torch.Generator] = None,
                    out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """train_tcga.py:78-83 with the arguments of the call site (`dropout_patches(bag_feats, 1 - dropout_patch)`):
    keep int(N * p) rows in random order (p = 1 -> a full random permutation), everything on the device.  `out`: a
    buffer of at least that many rows; the kept rows go to its first rows, which are returned."""
    n = int(feats.shape[0])
    keep = int(n * p)
    perm = torch.randperm(n, device=feats.device, generator=generator)[:keep]
    return gather_rows(feats, perm, None if out is None else out[:keep])


class DeviceBagStore:
    """Bags resident in HBM (80 GB holds thousands of 15 000 x 512 bags), in the `.pt` cache layout."""

    def __init__(self, feats_size: int, device="cuda"):
        self.D = feats_size
        self.device = torch.device(device)
        self.bags: List[Tuple[torch.Tensor, torch.Tensor]] = []

    def add_stacked(self, stacked: torch.Tensor) -> None:
        """stacked: [N, D + C] (train_tcga.py:47-51)."""
        st = stacked.to(self.device, dtype=torch.float32)
        self.bags.append((st[:, : self.D].contiguous(), st[0, self.D:].clone().unsqueeze(0)))

    def add_files(self, paths: Iterable[str]) -> None:
        for p in paths:
            self.add_stacked(torch.load(p, map_location="cpu"))

    def add_bag(self, feats: torch.Tensor, label: torch.Tensor) -> None:
        """feats [N, D] and label [C] given separately (no stacked copy)."""
        if feats.dim() != 2 or feats.shape[1] != self.D:
            raise ValueError(f"feats must be [N, {self.D}], got {tuple(feats.shape)}")
        self.bags.append((feats.to(self.device, dtype=torch.float32, non_blocking=True).contiguous(),
                          label.to(self.device, dtype=torch.float32).reshape(1, -1)))

    def add_bins(self, paths: Iterable[str]) -> None:
        """Binary bag containers (formats.write_bag_bin): payload read straight into pinned memory, then one
        asynchronous H2D copy per bag -- no text parse, no [N, D + C] intermediate."""
        from . import formats
        pin = self.device.type == "cuda"
        for p in paths:
            feats, label = formats.read_bag_bin(p, pin_memory=pin)
            self.add_bag(feats, label)
        if pin:
            torch.cuda.current_stream(self.device).synchronize()   # pinned sources may be freed after this

    def add_index(self, index_csv: str, num_classes: int, tcga_default: bool = False, workers: int = 4) -> None:
        """The reference's route (train_tcga.py:245-250 + :36-51) without the temp_train/*.pt detour.  Bag CSVs
        are parsed by the native reader on `workers` threads (the C call releases the GIL), in index order."""
        from concurrent.futures import ThreadPoolExecutor
        from . import formats
        rows = formats.read_dataset_index(index_csv)
        paths = [formats.tcga_default_feats_path(e) if tcga_default else e for e, _ in rows]
        with ThreadPoolExecutor(max_workers=max(1, workers)) as pool:
            for feats, (_, label) in zip(pool.map(formats.read_bag_csv, paths), rows):
                self.add_bag(torch.from_numpy(feats), torch.from_numpy(formats.bag_label(label, num_classes)))

    def __len__(self):
        return len(self.bags)


def train_epoch(milnet, store: DeviceBagStore, criterion, optimizer, dropout_patch: float = 0.0,
                order: Optional[Sequence[int]] = None, generator: Optional[torch.Generator] = None,
                bags_per_step: int = 1, graph: bool = False, max_rows: Optional[int] = None,
                generic: bool = False, value: bool = False) -> float:
    """One epoch of train_tcga.train() (train_tcga.py:55-76) over device-resident bags; one host sync per epoch.

    bags_per_step = 1: the reference's loop, one forward, backward and optimizer step per bag.  k > 1: minibatches of
    k consecutive bags of `order`; each is one `milnet.forward_bags(xs, grad=True)` call, one backward and one
    optimizer step on the mean over the group of the per-bag 0.5 * criterion(bag) + 0.5 * criterion(max instance)
    (criterion evaluated once on the group's [k, C] rows, which is that mean for an element-averaging criterion such
    as the reference's BCEWithLogitsLoss).  Returns the mean loss per bag either way.

    graph=True: the minibatch step (for any k >= 1, k = 1 included) is recorded once as a CUDA graph
    (train_graph.TrainStepGraph) and replayed for every group; the bags go through the same dropout_patches, straight
    into the graph's slots, and the results are the k-bag step's bits.  max_rows is the per-bag row capacity of the
    graph (default: the largest bag of the store); a bag over it raises ValueError before any step.  Each call records
    its graphs afresh (one warm-up step, one capture, new [k, max_rows, D] slots and a graph memory pool per group size,
    freed when the call returns), so a graph holds the optimizer's hyperparameters of its call, e.g. a learning rate
    that a scheduler changes between epochs.  Needs the batched tensor-core shapes and a capture-safe optimizer
    (SGD, or Adam / AdamW with capturable=True); generic=True also takes the other identity-v shapes (e.g. the
    classic-MIL D = 166 / 230, linear q), over the generic batched route, with the bits of the k-bag step.

    value=True: a model with a value network (passing_v; ValueError otherwise) trains on the batched value step
    instead of its per-bag autograd: each group of k >= 1 bags (k = 1 included) is one
    functional.mil_forward_value_bags(grad=True) call, one backward and one optimizer step on minibatch_loss.  The
    group's dropout_patches are drawn first, then each bag's dropout mask of v in bag order (BClassifier._v_input), as
    forward_bags draws them.  Its gradient sums run in another order than the per-bag step's, so its bits differ from
    the default's, which is why it is an option.  With graph=True the step is a replayed TrainStepGraph(value=True)
    with the same draws in the same order, written into the graph's slots and v_inputs, and the epoch gives the eager
    value=True epoch's bits: losses, parameters, optimizer state and the RNG states after it."""
    if value:
        from .train_graph import step_shape
        step_shape(milnet, value=True)                         # identity v raises here
    milnet.train()
    total = torch.zeros((), device=store.device)
    order = list(order) if order is not None else torch.randperm(len(store)).tolist()
    if graph:
        return _train_epoch_graph(milnet, store, criterion, optimizer, dropout_patch, order, generator,
                                  max(1, bags_per_step), max_rows, generic, value)
    if value or bags_per_step > 1:
        k = max(1, bags_per_step)
        if value:
            bc, params = milnet.b_classifier, milnet_params(milnet)
        for s in range(0, len(order), k):
            group = order[s:s + k]
            optimizer.zero_grad()
            xs = [dropout_patches(store.bags[i][0], 1 - dropout_patch, generator) for i in group]
            labels = torch.cat([store.bags[i][1].view(1, -1) for i in group])
            if value:   # each bag's v mask after the group's patch draws, as forward_bags draws them
                vs = [bc._v_input(x) for x in xs]
                outs, _ = Fn.mil_forward_value_bags(xs, params, None if vs[0] is None else vs, grad=True)
            else:
                outs = milnet.forward_bags(xs, grad=True)
            bag_prediction, max_prediction = _group_predictions(outs)
            loss = minibatch_loss(criterion, bag_prediction, max_prediction, labels)
            loss.backward()
            optimizer.step()
            total += loss.detach() * len(group)
        return float(total.item()) / max(1, len(order))
    for i in order:
        feats, label = store.bags[i]
        optimizer.zero_grad()
        x = dropout_patches(feats, 1 - dropout_patch, generator)
        ins_prediction, bag_prediction, _, _ = milnet(x)
        max_prediction, _ = torch.max(ins_prediction, 0)
        loss = 0.5 * criterion(bag_prediction.view(1, -1), label.view(1, -1)) + \
            0.5 * criterion(max_prediction.view(1, -1), label.view(1, -1))
        loss.backward()
        optimizer.step()
        total += loss.detach()
    return float(total.item()) / max(1, len(order))


def fold_steps(sizes: Sequence[int], k: int) -> List[List[Tuple[int, int, int]]]:
    """The steps of train_epoch_models over folds of `sizes` bags, k bags per step: step s holds (fold, start, stop)
    for every fold that still has bags, its group being bags [start, stop) of its order.  A fold whose bags have run
    out is not in the step."""
    k = max(1, int(k))
    steps = []
    for s in range(0, max(sizes, default=0), k):
        steps.append([(m, s, min(s + k, n)) for m, n in enumerate(sizes) if s < n])
    return steps


def train_epoch_models(milnets, store: DeviceBagStore, folds: Sequence[Sequence[int]], criterion,
                       optimizers, dropout_patch: float = 0.0, orders: Optional[Sequence[Sequence[int]]] = None,
                       generators: Optional[Sequence[Optional[torch.Generator]]] = None,
                       bags_per_step: int = 1, graph: bool = False, max_rows: Optional[int] = None,
                       generic: bool = False) -> List[float]:
    """One epoch of every fold model of a cross-validation (train_tcga.py:252-288, train_mil.py:164-187), the folds
    taking their steps together; returns each fold's mean loss per bag.  folds[m] lists the store indices of fold m's
    training split; orders[m], when given, is the order fold m visits them in (a permutation of folds[m]), else a
    random one (torch.randperm).

    Each step, every fold that still has bags takes its next group of k = bags_per_step (fold_steps): it draws its
    dropout_patches with generators[m], all groups go through one ensemble.forward_bags_per_model call, the step's loss
    is the sum of the folds' minibatch_loss (so each fold's own loss gets a gradient of exactly 1), one backward fills
    every fold's gradients, and each fold's optimizers[m].step() follows.  A fold with no group left is not in the
    call and its optimizer is not stepped.  The epoch makes one host sync.

    With per-fold generators (or no patch dropout) and the same orders, fold m's losses and parameters are bit for bit
    those of train_epoch(milnets[m], store, criterion, optimizers[m], dropout_patch, orders[m], generators[m], k, graph=True)
    (and of the eager minibatch epoch for k >= 2).  Without generators, or with one generator shared by the folds,
    the folds' permutation draws interleave in step order (fold 0's group, then fold 1's, ...), so each fold sees
    different draws than it would alone.

    graph=True: every step is a replay of a train_graph.FoldTrainStepGraph, recorded once per (folds in the step, their
    group sizes) -- for folds whose sizes differ by at most one bag, at most three graphs an epoch -- with the same
    bits.  The bags go through dropout_patches straight into the graph's slots; max_rows is the per-bag row capacity
    (default: the largest bag of the store), and a bag over it raises ValueError before any step.  Needs the fused fold
    shapes (dsmil_models_supported) and capture-safe optimizers, and records its graphs afresh on every call, as
    train_epoch(graph=True) does.  generic=True (with graph=True; the eager step ignores it) also takes folds on the
    generic batched route (train_graph.fold_step_shape: e.g. the classic-MIL D = 166 / 230, a linear q), each fold's
    results then the bits of train_epoch(..., graph=True, generic=True).

    criterion: one criterion for every fold, or one per fold (e.g. each fold's BCEWithLogitsLoss with the pos_weight
    of its own training split, train_mil.py:172-173); fold m's minibatch_loss then uses criterion[m], and its results
    are those of its own train_epoch with that criterion."""
    from .ensemble import forward_bags_per_model
    milnets, M = list(milnets), len(folds)
    if not 1 <= M <= Fn.MAX_MODELS:
        raise ValueError(f"a fold step takes 1 to {Fn.MAX_MODELS} folds, got {M}")
    criteria = fold_criteria(criterion, M)
    for what, seq in (("milnets", milnets), ("optimizers", optimizers), ("orders", orders),
                      ("generators", generators)):
        if seq is not None and len(seq) != M:
            raise ValueError(f"{len(seq)} {what} for {M} folds")
    for m, fold in enumerate(folds):
        if len(fold) == 0:
            raise ValueError(f"fold {m} has no training bags")
        bad = [i for i in fold if not 0 <= i < len(store)]
        if bad:
            raise IndexError(f"fold {m}: store index {bad[0]} outside [0, {len(store)})")
    if orders is None:
        orders = [[fold[i] for i in torch.randperm(len(fold)).tolist()] for fold in folds]
    else:
        orders = [list(o) for o in orders]
        for m, (o, fold) in enumerate(zip(orders, folds)):
            if sorted(o) != sorted(fold):
                raise ValueError(f"orders[{m}] is not a permutation of folds[{m}]")
    gens = list(generators) if generators is not None else [None] * M
    for net in milnets:
        net.train()
    if graph:
        return _train_epoch_models_graph(milnets, store, criterion, optimizers, dropout_patch, orders, gens,
                                         bags_per_step, max_rows, generic, criteria)
    totals = [torch.zeros((), device=store.device) for _ in range(M)]
    for step in fold_steps([len(o) for o in orders], bags_per_step):
        groups = [(m, orders[m][lo:hi]) for m, lo, hi in step]
        for m, _ in groups:
            optimizers[m].zero_grad()
        xs = [[dropout_patches(store.bags[i][0], 1 - dropout_patch, gens[m]) for i in group] for m, group in groups]
        outs = forward_bags_per_model([milnets[m] for m, _ in groups], xs, grad=True)
        loss = None
        for (m, group), out in zip(groups, outs):
            labels = torch.cat([store.bags[i][1].view(1, -1) for i in group])
            bag_prediction, max_prediction = _group_predictions(out)
            lm = minibatch_loss(criteria[m], bag_prediction, max_prediction, labels)
            totals[m] += lm.detach() * len(group)
            loss = lm if loss is None else loss + lm
        loss.backward()
        for m, _ in groups:
            optimizers[m].step()
    host = torch.stack(totals).double().tolist()    # the epoch's one host sync
    return [t / len(o) for t, o in zip(host, orders)]


def fold_criteria(criterion, M: int) -> list:
    """The M folds' criteria: `criterion` itself for every fold, or, given a list or tuple, one per fold (ValueError
    for another count)."""
    if isinstance(criterion, (list, tuple)):
        if len(criterion) != M:
            raise ValueError(f"{len(criterion)} criteria for {M} folds: give one criterion, or one per fold")
        return list(criterion)
    return [criterion] * M


def minibatch_loss(criterion, bag_prediction, max_prediction, labels):
    """The minibatch step's loss over a group's [k, C] predictions and labels."""
    return 0.5 * criterion(bag_prediction, labels) + 0.5 * criterion(max_prediction, labels)


def _graph_rows(store, p, max_rows, bags, what, fold=""):
    """The row counts of the store's bags `bags` after dropout_patches keeps a fraction p of each, and the row capacity
    of the `what` graphs: max_rows, by default the store's largest bag.  A bag over the capacity raises ValueError, and
    one that patch dropout empties IndexError, before any graph is recorded (fold: the prefix naming a bag's fold)."""
    cap = int(max_rows) if max_rows is not None else max([int(f.shape[0]) for f, _ in store.bags], default=1)
    keep = [int(int(store.bags[i][0].shape[0]) * p) for i in bags]
    for i, n in zip(bags, keep):
        if n > cap:
            raise ValueError(f"{fold}bag {i}: {n} rows exceed the {what} graph's max_rows={cap}")
        if n < 1:
            raise IndexError(f"dsmil_b200: {fold}bag {i} is empty after patch dropout (N == 0)")
    return keep, cap


def _train_epoch_graph(milnet, store, criterion, optimizer, dropout_patch, order, generator, k, max_rows, generic,
                       value=False):
    from .train_graph import TrainStepGraph, step_shape
    step_shape(milnet, generic, value)                         # a shape off the batched routes raises here
    p = 1 - dropout_patch
    keep, cap = _graph_rows(store, p, max_rows, order, "training")
    graphs = {}
    total = torch.zeros((), device=store.device)
    for s in range(0, len(order), k):
        group = order[s:s + k]
        g = graphs.get(len(group))
        if g is None:                                          # the first full group, and a short last one
            g = graphs[len(group)] = TrainStepGraph(milnet, criterion, optimizer, len(group), cap, generic=generic,
                                                    value=value)
        for b, i in enumerate(group):
            dropout_patches(store.bags[i][0], p, generator, out=g.slots[b])
            g.Ns[b].fill_(keep[s + b])
        if value and g.v_inputs is not None:                   # then v's masks, in bag order, as the eager step
            for b in range(len(group)):
                milnet.b_classifier._v_input(g.slots[b, :keep[s + b]], out=g.v_inputs[b, :keep[s + b]])
        torch.cat([store.bags[i][1].view(1, -1) for i in group], out=g.labels)
        total += g.step() * len(group)
    # the epoch's one host sync, which also reads the planners' status words
    status = sum((g.status for g in graphs.values()), torch.zeros(1, dtype=torch.int32, device=store.device))
    loss, bad = torch.stack([total.double(), status[0].double()]).tolist()
    if bad:
        raise RuntimeError(f"training graph: a batch held a bag outside [1, {cap}] rows (planner status {int(bad)})")
    return loss / max(1, len(order))


def _train_epoch_models_graph(milnets, store, criterion, optimizers, dropout_patch, orders, gens, k, max_rows,
                              generic, criteria):
    from .train_graph import FoldTrainStepGraph, fold_step_shape
    fold_step_shape(milnets, generic)                          # shapes off the fold routes raise here
    p = 1 - dropout_patch
    keep = {}
    for m, o in enumerate(orders):
        rows, cap = _graph_rows(store, p, max_rows, o, "training", f"fold {m}, ")
        keep.update(zip(o, rows))
    graphs = {}
    totals = [torch.zeros((), device=store.device) for _ in orders]
    bad = torch.zeros(len(orders), dtype=torch.int32, device=store.device)
    for step in fold_steps([len(o) for o in orders], k):
        key = tuple((m, hi - lo) for m, lo, hi in step)
        g = graphs.get(key)
        if g is None:                                          # the full step, short last groups, fewer folds
            # one criterion for all folds stays one object; per-fold criteria go with their folds
            crit = [criteria[m] for m, _ in key] if isinstance(criterion, (list, tuple)) else criterion
            g = graphs[key] = FoldTrainStepGraph([milnets[m] for m, _ in key], crit,
                                                 [optimizers[m] for m, _ in key], [n for _, n in key], cap,
                                                 generic=generic)
        e = 0
        for j, (m, lo, hi) in enumerate(step):
            group = orders[m][lo:hi]
            for b, i in enumerate(group):
                dropout_patches(store.bags[i][0], p, gens[m], out=g.slots[j][b])
                g.Ns[e + b].fill_(keep[i])
            torch.cat([store.bags[i][1].view(1, -1) for i in group], out=g.labels[e:e + len(group)])
            e += len(group)
        losses = g.step()
        for j, (m, lo, hi) in enumerate(step):
            totals[m] += losses[j] * (hi - lo)
    for key, g in graphs.items():
        for j, (m, _) in enumerate(key):
            bad[m] = torch.where(bad[m] != 0, bad[m], g.status[j])
    # the epoch's one host sync, which also reads the planners' status words
    host = torch.cat([torch.stack(totals).double(), bad.double()]).tolist()
    for m, st in enumerate(host[len(orders):]):
        if st:
            raise RuntimeError(f"training graph: fold {m} held a bag outside [1, {cap}] rows (planner status "
                               f"{int(st)})")
    return [t / len(o) for t, o in zip(host, orders)]


def _group_predictions(outs):
    """(bag predictions [k, C], max-instance predictions [k, C]) of a group's forward_bags outputs.  The packed
    outputs of the bag-table call carry each bag's critical rows, the per-class arg-max of its scores: gathering the
    scores there is the per-bag max in one op (the gradient goes to that row, as torch.max's does when the max is
    unique).  The per-bag fallback of forward_bags returns a plain list."""
    if isinstance(outs, Fn.BagOutputs) and outs.crit is not None:
        classes, pred = outs.packed[0], outs.packed[1]
        first = torch.tensor([0] + outs.Ns[:-1], device=classes.device).cumsum(0)
        return pred, classes.gather(0, outs.crit + first[:, None])
    return (torch.cat([bag.view(1, -1) for _, bag, _, _ in outs]),
            torch.stack([torch.max(ins, 0)[0] for ins, _, _, _ in outs]))


def _eval_bag(criterion, ins_prediction, bag_prediction, label, average):
    """One bag's evaluation loss, 0.5 * criterion(bag) + 0.5 * criterion(max instance), and its sigmoid prediction
    (average: sigmoid(max) + sigmoid(bag))."""
    max_prediction, _ = torch.max(ins_prediction, 0)
    loss = (0.5 * criterion(bag_prediction.view(1, -1), label.view(1, -1)) +
            0.5 * criterion(max_prediction.view(1, -1), label.view(1, -1)))
    p = torch.sigmoid(bag_prediction).view(-1)
    return loss, (torch.sigmoid(max_prediction).view(-1) + p if average else p)


def eval_epoch(milnet, store: DeviceBagStore, criterion, average: bool = False, bags_per_launch: int = 16,
               dropout_patch: float = 0.0, generator: Optional[torch.Generator] = None, graph: bool = False,
               max_rows: Optional[int] = None, generic: bool = False, value: bool = False):
    """The measuring half of train_tcga.test() (train_tcga.py:85-107): mean loss, labels [n_bags, C] and
    sigmoid predictions [n_bags, C] (`average=True`: sigmoid(max) + sigmoid(bag), as `args.average`).  The ROC /
    threshold logic that follows in the reference (:108-132) is the caller's and works on these arrays.

    Bags go through `milnet.forward_bags` `bags_per_launch` at a time when the module has it (one batched launch
    sequence for the whole group, the slides/sec path), else one `milnet(x)` per bag; the loss terms stay on the
    device and there is one host sync per epoch instead of two `.item()` per bag.  The reference also routes test
    bags through `dropout_patches` (a row permutation when dropout_patch == 0); a permutation does not change
    any output of the operator except the order of the per-instance rows, so it is skipped unless rows are
    actually dropped.

    graph=True: each group of bags_per_launch bags (and a short last group) replays a recorded graph
    (infer_graph.EvalBagsGraph) of the forward, the per-bag losses and the predictions; the bags are read in place and
    the results are the eager epoch's bits.  max_rows is the per-bag row capacity of the graphs (default: the largest
    bag of the store); a bag over it raises ValueError before any launch.  The graphs stay cached with the model (held
    weakly) and later calls with the same group sizes, capacity, `average` and criterion object replay them: the first
    call pays the recording, and a model whose parameter tensors were replaced gets new graphs.  Needs the batched
    tensor-core shapes; generic=True also takes the other identity-v shapes, over the generic batched route.

    value=True: a model with a value network (passing_v; ValueError otherwise).  The eager epoch is the default one,
    which already runs such a model's batched value forward; with graph=True the graphs record
    dsmil_value_forward_bags_dev (EvalBagsGraph(value=True)) and give the eager epoch's bits."""
    if value:
        from .train_graph import step_shape
        step_shape(milnet, value=True)                         # identity v raises here
    milnet.eval()
    n = len(store)
    if n == 0:
        raise ValueError("eval_epoch over an empty store")
    if graph:
        return _eval_epoch_graph(milnet, store, criterion, average, max(1, bags_per_launch), dropout_patch, generator,
                                 max_rows, generic, value)
    losses, labels, preds = [], [], []
    batched = hasattr(milnet, "forward_bags") and bags_per_launch > 1
    with torch.no_grad():
        for s in range(0, n, max(1, bags_per_launch)):
            group = store.bags[s:s + max(1, bags_per_launch)]
            xs = [dropout_patches(f, 1 - dropout_patch, generator) if dropout_patch > 0 else f for f, _ in group]
            outs = milnet.forward_bags(xs) if batched else [milnet(x) for x in xs]
            for (ins_prediction, bag_prediction, _, _), (_, label) in zip(outs, group):
                loss, pred = _eval_bag(criterion, ins_prediction, bag_prediction, label, average)
                losses.append(loss)
                labels.append(label.view(-1))
                preds.append(pred)
    loss = float(torch.stack([l.reshape(()) for l in losses]).mean().item())
    return loss, torch.stack(labels).cpu().numpy().astype(int), torch.stack(preds).cpu().numpy()


def eval_epoch_models(milnets, store: DeviceBagStore, criterion, average: bool = False, bags_per_launch: int = 16,
                      graph: bool = False, max_rows: Optional[int] = None):
    """eval_epoch for an ensemble (the fold models of train_tcga.py:395-404) over the same bags: one (loss, labels,
    preds) per model, each bit for bit `eval_epoch(milnets[m], store, criterion, average, bags_per_launch)` without
    patch dropout.  Each group of bags_per_launch > 1 bags is one ensemble.forward_bags_models call, and the whole
    call makes one host sync.  The thresholds and the vote over the models (train_tcga.py:113-124, 401-404) are the
    caller's, on these arrays.

    graph=True: each group of bags_per_launch bags (and a short last group) replays an infer_graph.EvalBagsModelsGraph
    in which every model is given the group's bags, cached as eval_epoch_folds caches its graphs; max_rows as
    eval_epoch's.  The results are the eager call's bits.  The members and shapes are those of
    train_graph.fold_step_shape.  Each model reads the group's bags in a pass of its own, so the members' passes over
    a bag do not follow each other in L2 as the eager fused ensemble's do."""
    from .ensemble import forward_bags_models
    milnets = list(milnets)
    for m in milnets:
        m.eval()
    n, k = len(store), max(1, bags_per_launch)
    if n == 0:
        raise ValueError("eval_epoch_models over an empty store")
    if graph:
        M = len(milnets)
        return _eval_folds_graph(milnets, store, [list(range(n))] * M, [criterion] * M, average, k, max_rows, False,
                                 "eval_epoch_models")
    losses = [[] for _ in milnets]
    preds = [[] for _ in milnets]
    with torch.no_grad():
        for s in range(0, n, k):
            group = store.bags[s:s + k]
            xs = [f for f, _ in group]
            # one bag per launch: each model's milnet(x), as eval_epoch takes it
            outs = forward_bags_models(milnets, xs) if k > 1 else [[net(x) for x in xs] for net in milnets]
            for m, out in enumerate(outs):
                for (ins_prediction, bag_prediction, _, _), (_, label) in zip(out, group):
                    loss, pred = _eval_bag(criterion, ins_prediction, bag_prediction, label, average)
                    losses[m].append(loss)
                    preds[m].append(pred)
        M = len(milnets)
        loss = torch.stack([torch.stack([l.reshape(()) for l in ls]).mean() for ls in losses])
        labels = torch.stack([label.view(-1) for _, label in store.bags])
        pred = torch.stack([torch.stack(ps) for ps in preds])
        # the one host sync (float32 and the integer labels are exact in float64)
        host = torch.cat([loss.double(), labels.double().view(-1), pred.double().view(-1)]).cpu().numpy()
    C = int(labels.shape[1])
    lab = host[M:M + n * C].reshape(n, C).astype(int)
    pr = host[M + n * C:].reshape(M, n, C).astype(np.float32)
    return [(float(host[m]), lab.copy(), pr[m]) for m in range(M)]


def eval_epoch_folds(milnets, store: DeviceBagStore, folds: Sequence[Sequence[int]], criterion, average: bool = False,
                     bags_per_launch: int = 16, graph: bool = False, max_rows: Optional[int] = None,
                     generic: bool = False):
    """The validation half of a fold epoch (train_tcga.py:272-287, train_mil.py:177-184): every fold model over its
    own held-out bags, the folds taking their steps together.  folds[m] lists fold m's held-out store indices in the
    order they are evaluated; criterion is one criterion, or one per fold (fold_criteria).  Returns one (loss,
    labels, preds) per fold, fold m's bit for bit `eval_epoch(milnets[m], <a store of folds[m]'s bags in that order>,
    criteria[m], average, bags_per_launch, graph=graph)`.  No patch dropout, as eval_epoch_models.

    The steps follow fold_steps: each step, every fold that still has bags takes its next group of k =
    bags_per_launch.  Eager, each fold model runs its group as eval_epoch does: one forward_bags call (k = 1: one
    milnet(x)).  It does not use ensemble.forward_bags_per_model: that is the training form, whose bag predictions can
    differ from the inference forward's in the last bits.  graph=True: a step replays an infer_graph.EvalBagsModelsGraph, one per (folds
    in the step, their group sizes), with the capacity max_rows (default: the largest bag of the store; a bag over it
    raises ValueError before any launch).  The graphs stay cached with the first model of their step (held weakly), and
    later calls replay them: a call over 50 epochs records on its first only.  A graph is recorded again when one of
    its models' parameter tensors, or its criteria, changed.  Needs the members and shapes of
    train_graph.fold_step_shape (generic=True: also the generic fold shapes).

    One host sync per call; a fold with a bag the library refused raises RuntimeError naming the fold."""
    milnets, M = list(milnets), len(folds)
    if not 1 <= M <= Fn.MAX_MODELS:
        raise ValueError(f"eval_epoch_folds takes 1 to {Fn.MAX_MODELS} folds, got {M}")
    if len(milnets) != M:
        raise ValueError(f"{len(milnets)} milnets for {M} folds")
    criteria = fold_criteria(criterion, M)
    folds = [list(f) for f in folds]
    for m, fold in enumerate(folds):
        if len(fold) == 0:
            raise ValueError(f"fold {m} has no held-out bags")
        bad = [i for i in fold if not 0 <= i < len(store)]
        if bad:
            raise IndexError(f"fold {m}: store index {bad[0]} outside [0, {len(store)})")
    for net in milnets:
        net.eval()
    k = max(1, bags_per_launch)
    if graph:
        return _eval_folds_graph(milnets, store, folds, criteria, average, k, max_rows, generic, "eval_epoch_folds")
    losses = [[] for _ in range(M)]
    preds = [[] for _ in range(M)]
    with torch.no_grad():
        for step in fold_steps([len(f) for f in folds], k):
            groups = [(m, folds[m][lo:hi]) for m, lo, hi in step]
            for m, group in groups:
                net, xs = milnets[m], [store.bags[i][0] for i in group]
                out = net.forward_bags(xs) if k > 1 and hasattr(net, "forward_bags") else [net(x) for x in xs]
                for (ins_prediction, bag_prediction, _, _), i in zip(out, group):
                    loss, pred = _eval_bag(criteria[m], ins_prediction, bag_prediction, store.bags[i][1], average)
                    losses[m].append(loss)
                    preds[m].append(pred)
        loss = torch.stack([torch.stack([l.reshape(()) for l in ls]).mean() for ls in losses])
        return _fold_results(store, folds, loss, [torch.stack(ps) for ps in preds], None)


def _fold_results(store, folds, loss, preds, status):
    """Each fold's (loss, labels, preds) from the device: loss [M], preds[m] [n_m, C] and (graphs) each fold's planner
    status [M], in one host sync (float32 and the integer labels are exact in float64).  RuntimeError naming the first
    fold with a refused bag."""
    M = len(folds)
    labels = torch.stack([store.bags[i][1].view(-1) for f in folds for i in f])
    parts = [loss.double().view(-1)] + ([status.double().view(-1)] if status is not None else [])
    host = torch.cat(parts + [labels.double().view(-1)] + [p.double().view(-1) for p in preds]).cpu().numpy()
    at = M
    if status is not None:
        for m, st in enumerate(host[M:2 * M]):
            if st:
                raise RuntimeError(f"inference graph: fold {m} held a bag the library refused (planner status "
                                   f"{int(st)})")
        at = 2 * M
    C = int(labels.shape[1])
    out = []
    lab = host[at:at + labels.numel()].reshape(-1, C).astype(int)
    at += labels.numel()
    row = 0
    for m, f in enumerate(folds):
        n = len(f)
        out.append((float(host[m]), lab[row:row + n].copy(), host[at:at + n * C].reshape(n, C).astype(np.float32)))
        row, at = row + n, at + n * C
    return out


# first model of a step -> {(the step's models, their group sizes, max_rows, average, generic): EvalBagsModelsGraph},
# as _EVAL_GRAPHS keeps EvalBagsGraph: weakly, off the models themselves
_FOLD_EVAL_GRAPHS = weakref.WeakKeyDictionary()


def _fold_eval_graph(nets, crits, nbs, cap, average, generic):
    """The cached EvalBagsModelsGraph of these models, criteria and group sizes, recorded if there is none or if a
    model's parameter tensors or a criterion changed since."""
    from .infer_graph import EvalBagsModelsGraph
    cached = _FOLD_EVAL_GRAPHS.setdefault(nets[0], {})
    key = (tuple(id(net) for net in nets), tuple(nbs), cap, bool(average), bool(generic))
    g = cached.get(key)
    if (g is None or not g.current() or any(a is not b for a, b in zip(g.members(), nets))
            or any(a is not b for a, b in zip(g.criteria, crits))):
        g = cached[key] = EvalBagsModelsGraph(nets, list(crits), nbs, cap, average, generic=generic)
    return g


def _eval_folds_graph(milnets, store, folds, criteria, average, k, max_rows, generic, what):
    from .train_graph import fold_step_shape
    fold_step_shape(milnets, generic)                          # shapes off the fold routes raise here
    cap = None
    for m, f in enumerate(folds):
        _, cap = _graph_rows(store, 1.0, max_rows, f, "inference", f"fold {m}, ")
    M = len(folds)
    losses = [torch.empty(len(f), device=store.device) for f in folds]
    preds = [torch.empty(len(f), int(store.bags[0][1].numel()), device=store.device) for f in folds]
    status = torch.zeros(M, dtype=torch.int32, device=store.device)
    used = []
    for step in fold_steps([len(f) for f in folds], k):
        nets = [milnets[m] for m, _, _ in step]
        g = _fold_eval_graph(nets, [criteria[m] for m, _, _ in step], [hi - lo for _, lo, hi in step], cap, average,
                             generic)
        groups = [folds[m][lo:hi] for m, lo, hi in step]
        torch.cat([store.bags[i][1].view(1, -1) for group in groups for i in group], out=g.labels)
        g.run([[store.bags[i][0] for i in group] for group in groups])
        e = 0
        for j, (m, lo, hi) in enumerate(step):
            losses[m][lo:hi] = g.loss[e:e + hi - lo]
            preds[m][lo:hi] = g.pred[e:e + hi - lo]
            status[m] = torch.where(status[m] != 0, status[m], g.status[j])
            e += hi - lo
        used.append(g)
    out = _fold_results(store, folds, torch.stack([l.mean() for l in losses]), preds, status)
    for g in used:
        g.status.zero_()
        g.release()
    return out


# model -> {(bags per graph, max_rows, average): EvalBagsGraph}: later epochs replay the graphs of earlier ones (the
# graphs read the parameters in place, so training between epochs is seen); kept off the model itself, as
# embed._GRAPHS, so that deepcopy / pickling of the caller's model never meets a CUDA graph
_EVAL_GRAPHS = weakref.WeakKeyDictionary()


def _eval_epoch_graph(milnet, store, criterion, average, k, dropout_patch, generator, max_rows, generic, value=False):
    from .infer_graph import EvalBagsGraph
    from .train_graph import step_shape
    step_shape(milnet, generic, value)                         # a shape off the batched routes raises here
    p = 1 - dropout_patch
    _, cap = _graph_rows(store, p, max_rows, range(len(store)), "inference")
    n, C = len(store), int(store.bags[0][1].numel())
    cached = _EVAL_GRAPHS.setdefault(milnet, {})
    graphs = {}
    losses = torch.empty(n, device=store.device)
    preds = torch.empty(n, C, device=store.device)
    labels = torch.stack([label.view(-1) for _, label in store.bags])
    for s in range(0, n, k):
        group = store.bags[s:s + k]
        g = graphs.get(len(group))
        if g is None:                                          # the first full group, and a short last one
            key = (len(group), cap, bool(average))
            g = cached.get(key)
            if g is None or g.criterion is not criterion or not g.current():
                g = cached[key] = EvalBagsGraph(milnet, criterion, len(group), cap, average, generic=generic,
                                                value=value)
            graphs[len(group)] = g
        xs = [dropout_patches(f, p, generator) if dropout_patch > 0 else f for f, _ in group]
        g.labels.copy_(labels[s:s + len(group)])
        g.run(xs)
        losses[s:s + len(group)] = g.loss
        preds[s:s + len(group)] = g.pred
    # the epoch's one host sync: the mean loss, the planners' status words, the labels and the predictions (float32
    # and the integer labels are exact in float64)
    status = sum((g.status for g in graphs.values()), torch.zeros(1, dtype=torch.int32, device=store.device))
    host = torch.cat([losses.mean().double().view(1), status.double(), labels.double().view(-1),
                      preds.double().view(-1)]).cpu().numpy()
    for g in graphs.values():
        g.status.zero_()
        g.release()
    if host[1]:
        raise RuntimeError(f"inference graph: a batch held a bag the library refused (planner status {int(host[1])})")
    return (float(host[0]), host[2:2 + n * C].reshape(n, C).astype(int),
            host[2 + n * C:].reshape(n, C).astype(np.float32))


# ---- classic-MIL drivers (train_mil.py) ---------------------------------------------------------------------


def mil_store(bags: Sequence[Tuple[int, "np.ndarray"]], device="cuda") -> DeviceBagStore:
    """`formats.mil_bags(...)` output -> device-resident store (label as a [1, 1] target, train_mil.py:49)."""
    if not bags:
        raise ValueError("no bags")
    store = DeviceBagStore(int(bags[0][1].shape[1]), device=device)
    for label, x in bags:
        store.add_bag(torch.as_tensor(x, dtype=torch.float32), torch.tensor([float(label)]))
    return store


def cross_validation_set(in_list: Sequence, fold: int, index: int):
    """train_mil.py:99-104: chunks of int(len/fold) items; chunk `index` is the test set, the rest (including
    the short tail chunk the integer division leaves) the training set."""
    items = list(in_list)
    n = int(len(items) / fold)
    if n < 1:
        raise ValueError(f"{len(items)} bags cannot be split into {fold} folds")
    chunks = [items[i:i + n] for i in range(0, len(items), n)]
    test = chunks.pop(index)
    return [x for c in chunks for x in c], test


def compute_pos_weight(bags: Sequence[Tuple[int, object]]) -> float:
    """train_mil.py:106-110: negatives / positives over the bag labels (clipped to {0, 1})."""
    pos = sum(int(min(max(b[0], 0), 1)) for b in bags)
    if pos == 0:
        raise ZeroDivisionError("no positive bag in the training split (the reference divides by zero here too)")
    return (len(bags) - pos) / pos


def mil_epoch_train(milnet, store: DeviceBagStore, criterion, optimizer, order: Optional[Sequence[int]] = None,
                    bags_per_step: int = 1, graph: bool = False, max_rows: Optional[int] = None,
                    value: bool = False) -> float:
    """train_mil.epoch_train (train_mil.py:42-59): per bag, shuffle the instances, forward, 0.5/0.5 loss, step
    (bags_per_step > 1: one step per group of bags, as train_epoch).  graph, max_rows: as train_epoch's, on the generic
    batched route too (the classic-MIL shapes are off the tensor-core batch): bags of a few dozen rows cost little on
    the device, so the replayed step saves most of an epoch's host work.  value: as train_epoch's."""
    return train_epoch(milnet, store, criterion, optimizer, dropout_patch=0.0, order=order, bags_per_step=bags_per_step,
                       graph=graph, max_rows=max_rows, generic=True, value=value)


def mil_epoch_test(milnet, store: DeviceBagStore, criterion, bags_per_launch: int = 16, graph: bool = False,
                   max_rows: Optional[int] = None, value: bool = False):
    """train_mil.epoch_test (train_mil.py:61-80): (mean loss, bag labels, sigmoid bag predictions).  graph, max_rows:
    as eval_epoch's, on the generic batched route too; value: as eval_epoch's."""
    loss, labels, preds = eval_epoch(milnet, store, criterion, average=False, bags_per_launch=bags_per_launch,
                                     graph=graph, max_rows=max_rows, generic=True, value=value)
    return loss, [int(l[0]) for l in labels], [p.squeeze() for p in preds]
