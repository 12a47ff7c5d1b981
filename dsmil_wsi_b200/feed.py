"""Caller-side bag feed for training (SURVEY §8f-1; reference train_tcga.py:55-83).

The reference's training loop pays, per bag and per epoch: `torch.load(item, map_location='cuda:0')` (disk ->
GPU), a CPU `torch.randperm` + advanced-indexing gather for `dropout_patches`, and a `loss.item()` sync.  Once
the operator takes tens of microseconds those dominate.  Here the bags of the `.pt` cache format
(`[N, D + C]` = features || label repeated per row, train_tcga.py:36-51) live on the device, the patch-dropout
permutation is drawn on the device and applied by `dsmil_gather_rows` (our kernel), and the running loss stays
on the device until the epoch ends.
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Sequence, Tuple

import torch

from . import _lib
from . import functional as Fn


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
                bags_per_step: int = 1, graph: bool = False, max_rows: Optional[int] = None) -> float:
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
    (SGD, or Adam / AdamW with capturable=True)."""
    milnet.train()
    total = torch.zeros((), device=store.device)
    order = list(order) if order is not None else torch.randperm(len(store)).tolist()
    if graph:
        return _train_epoch_graph(milnet, store, criterion, optimizer, dropout_patch, order, generator,
                                  max(1, bags_per_step), max_rows)
    if bags_per_step > 1:
        for s in range(0, len(order), bags_per_step):
            group = order[s:s + bags_per_step]
            optimizer.zero_grad()
            xs = [dropout_patches(store.bags[i][0], 1 - dropout_patch, generator) for i in group]
            labels = torch.cat([store.bags[i][1].view(1, -1) for i in group])
            bag_prediction, max_prediction = _group_predictions(milnet.forward_bags(xs, grad=True))
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


def minibatch_loss(criterion, bag_prediction, max_prediction, labels):
    """The minibatch step's loss over a group's [k, C] predictions and labels."""
    return 0.5 * criterion(bag_prediction, labels) + 0.5 * criterion(max_prediction, labels)


def _train_epoch_graph(milnet, store, criterion, optimizer, dropout_patch, order, generator, k, max_rows):
    from .train_graph import TrainStepGraph, step_shape
    step_shape(milnet)                                         # a shape off the batched path raises here
    p = 1 - dropout_patch
    keep = [int(int(store.bags[i][0].shape[0]) * p) for i in order]   # dropout_patches' row counts
    cap = int(max_rows) if max_rows is not None else max([int(f.shape[0]) for f, _ in store.bags], default=1)
    for i, n in zip(order, keep):
        if n > cap:
            raise ValueError(f"bag {i}: {n} rows exceed the training graph's max_rows={cap}")
        if n < 1:
            raise IndexError(f"dsmil_b200: bag {i} is empty after patch dropout (N == 0)")
    graphs = {}
    total = torch.zeros((), device=store.device)
    for s in range(0, len(order), k):
        group = order[s:s + k]
        g = graphs.get(len(group))
        if g is None:                                          # the first full group, and a short last one
            g = graphs[len(group)] = TrainStepGraph(milnet, criterion, optimizer, len(group), cap)
        for b, i in enumerate(group):
            dropout_patches(store.bags[i][0], p, generator, out=g.slots[b])
            g.Ns[b].fill_(keep[s + b])
        torch.cat([store.bags[i][1].view(1, -1) for i in group], out=g.labels)
        total += g.step() * len(group)
    # the epoch's one host sync, which also reads the planners' status words
    status = sum((g.status for g in graphs.values()), torch.zeros(1, dtype=torch.int32, device=store.device))
    loss, bad = torch.stack([total.double(), status[0].double()]).tolist()
    if bad:
        raise RuntimeError(f"training graph: a batch held a bag outside [1, {cap}] rows (planner status {int(bad)})")
    return loss / max(1, len(order))


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


def eval_epoch(milnet, store: DeviceBagStore, criterion, average: bool = False, bags_per_launch: int = 16,
               dropout_patch: float = 0.0, generator: Optional[torch.Generator] = None):
    """The measuring half of train_tcga.test() (train_tcga.py:85-107): mean loss, labels [n_bags, C] and
    sigmoid predictions [n_bags, C] (`average=True`: sigmoid(max) + sigmoid(bag), as `args.average`).  The ROC /
    threshold logic that follows in the reference (:108-132) is the caller's and works on these arrays.

    Bags go through `milnet.forward_bags` `bags_per_launch` at a time when the module has it (one batched launch
    sequence for the whole group, the slides/sec path), else one `milnet(x)` per bag; the loss terms stay on the
    device and there is one host sync per epoch instead of two `.item()` per bag.  The reference also routes test
    bags through `dropout_patches` (a row permutation when dropout_patch == 0); a permutation does not change
    any output of the operator except the order of the per-instance rows, so it is skipped unless rows are
    actually dropped."""
    milnet.eval()
    n = len(store)
    if n == 0:
        raise ValueError("eval_epoch over an empty store")
    losses, labels, preds = [], [], []
    batched = hasattr(milnet, "forward_bags") and bags_per_launch > 1
    with torch.no_grad():
        for s in range(0, n, max(1, bags_per_launch)):
            group = store.bags[s:s + max(1, bags_per_launch)]
            xs = [dropout_patches(f, 1 - dropout_patch, generator) if dropout_patch > 0 else f for f, _ in group]
            outs = milnet.forward_bags(xs) if batched else [milnet(x) for x in xs]
            for (ins_prediction, bag_prediction, _, _), (_, label) in zip(outs, group):
                max_prediction, _ = torch.max(ins_prediction, 0)
                losses.append(0.5 * criterion(bag_prediction.view(1, -1), label.view(1, -1)) +
                              0.5 * criterion(max_prediction.view(1, -1), label.view(1, -1)))
                labels.append(label.view(-1))
                p = torch.sigmoid(bag_prediction).view(-1)
                preds.append(torch.sigmoid(max_prediction).view(-1) + p if average else p)
    loss = float(torch.stack([l.reshape(()) for l in losses]).mean().item())
    return loss, torch.stack(labels).cpu().numpy().astype(int), torch.stack(preds).cpu().numpy()


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
                    bags_per_step: int = 1) -> float:
    """train_mil.epoch_train (train_mil.py:42-59): per bag, shuffle the instances, forward, 0.5/0.5 loss, step
    (bags_per_step > 1: one step per group of bags, as train_epoch)."""
    return train_epoch(milnet, store, criterion, optimizer, dropout_patch=0.0, order=order, bags_per_step=bags_per_step)


def mil_epoch_test(milnet, store: DeviceBagStore, criterion, bags_per_launch: int = 16):
    """train_mil.epoch_test (train_mil.py:61-80): (mean loss, bag labels, sigmoid bag predictions)."""
    loss, labels, preds = eval_epoch(milnet, store, criterion, average=False, bags_per_launch=bags_per_launch)
    return loss, [int(l[0]) for l in labels], [p.squeeze() for p in preds]
