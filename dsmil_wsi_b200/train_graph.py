"""The minibatch training step recorded once as a CUDA graph and replayed over batches of ragged bags, on one device
(TrainStepGraph) or row-sharded over the ranks of a process group (ShardedTrainStepGraph).

A k-bag step of feed.train_epoch(bags_per_step=k) costs a few milliseconds of host work: Python autograd, ctypes,
workspace allocation, host-built bag tables and their uploads, the loss ops and the optimizer's launches.  Here the
step -- MILBagsDevFn forward (dsmil_forward_bags_train_dev), the minibatch loss, its backward
(dsmil_backward_bags_dev) and optimizer.step() -- is captured once into a torch.cuda.CUDAGraph over static buffers:
nb slots of max_rows rows, the bag sizes and the labels on the device.  The library's dev entry points read the bag
sizes on the device, so one graph serves every batch of nb bags of 1..max_rows rows, with the bits of the eager step.
"""
from __future__ import annotations

import ctypes

import torch

from . import _lib
from . import feed
from . import functional as Fn
from .modules import BClassifier, FCLayer


def check_optimizer(optimizer) -> None:
    """A replayed step must not read host state the graph froze: SGD (without dampening, whose first step a graph
    cannot tell from the others), or Adam / AdamW with capturable=True."""
    if isinstance(optimizer, torch.optim.SGD):
        for g in optimizer.param_groups:
            if g.get("momentum", 0) and g.get("dampening", 0):
                raise ValueError("TrainStepGraph: SGD with momentum and dampening != 0 is not supported (its first "
                                 "step differs from the others, and a graph replays one step)")
        return
    if isinstance(optimizer, (torch.optim.Adam, torch.optim.AdamW)):
        if all(g.get("capturable", False) for g in optimizer.param_groups):
            return
        raise ValueError(f"TrainStepGraph: {type(optimizer).__name__} must be built with capturable=True to be "
                         "replayed in a CUDA graph")
    raise ValueError(f"TrainStepGraph: optimizer {type(optimizer).__name__} is not known to be capture-safe; use SGD, "
                     "or Adam / AdamW with capturable=True")


def step_shape(milnet):
    """(D, C) of a MILNet whose training step the graph can record: FCLayer + BClassifier with identity v, on the
    batched tensor-core shapes (dsmil_shard_bags_supported).  Anything else raises ValueError naming the shape."""
    ic, bc = getattr(milnet, "i_classifier", None), getattr(milnet, "b_classifier", None)
    if not (isinstance(ic, FCLayer) and isinstance(bc, BClassifier)):
        raise ValueError("graph-captured training needs MILNet(FCLayer, BClassifier); got "
                         f"{type(ic).__name__} + {type(bc).__name__}")
    W1, b1, W2, b2 = bc._q_params()
    Wv, _, _ = bc._v_params()
    C, D = int(bc.fcc.weight.shape[0]), int(bc.fcc.weight.shape[2])
    p = _lib.DsmilParams(D, C, int(W2 is not None), int(Wv is not None))
    if not _lib.load().dsmil_shard_bags_supported(ctypes.byref(p)):
        raise ValueError(f"graph-captured training runs on the batched tensor-core path only; D={D}, C={C}, "
                         f"nonlinear={W2 is not None}, passing_v={Wv is not None} is not on it")
    return D, C


class TrainStepGraph:
    """One recorded minibatch step of nb bags of up to max_rows rows.

    Fill `slots[b, :n_b]` with bag b's features, `Ns[b]` with n_b and `labels` [nb, C], then `step()` replays the
    graph and returns the step's loss (a device scalar, overwritten by the next replay).  A batch with a bag outside
    1..max_rows is refused on the device: the library's planner records it in `status` (the first refusal's 1 + bag
    index; never cleared here, read it when you synchronise), the step's loss is NaN, and the step leaves the
    parameters and the optimizer state as they were (the update is computed and then discarded on the device).

    Warm-up and capture leave the parameters and the optimizer state as they found them, restored in place so the
    graph's addresses stay valid; optimizer state the warm-up creates is reset to its fresh value (zeros).  The graph
    freezes the optimizer's hyperparameters (e.g. its learning rate) at construction.  The parameters' .grad become
    the graph's gradient buffers."""

    def __init__(self, milnet, criterion, optimizer, nb: int, max_rows: int, warmup: int = 1):
        check_optimizer(optimizer)
        D, C = step_shape(milnet)
        nb, max_rows = int(nb), int(max_rows)
        if not 1 <= nb <= 65535 or max_rows < 1:
            raise ValueError(f"TrainStepGraph: nb={nb} outside [1, 65535] or max_rows={max_rows} < 1")
        self.milnet, self.criterion, self.optimizer = milnet, criterion, optimizer
        self.nb, self.max_rows = nb, max_rows
        self.params = [p for g in optimizer.param_groups for p in g["params"]]
        dev = milnet.b_classifier.fcc.weight.device
        Fn.require_cuda(milnet.b_classifier.fcc.weight, "the model")
        self.slots = torch.zeros(nb, max_rows, D, device=dev)
        self.Ns = torch.ones(nb, dtype=torch.int64, device=dev)
        self.labels = torch.zeros(nb, C, device=dev)
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)
        self._step_status = torch.zeros(1, dtype=torch.int32, device=dev)   # this replay's planners
        self._buffers(dev)
        snap = self._snapshot()
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(max(1, warmup)):
                optimizer.zero_grad(set_to_none=True)
                self._step()
        torch.cuda.current_stream(dev).wait_stream(side)
        self._restore(snap)
        optimizer.zero_grad(set_to_none=True)
        # what a refused step puts back: the parameters and every tensor of the optimizer state (it exists now)
        self._kept = self.params + [v for p in self.params for v in optimizer.state.get(p, {}).values()
                                    if torch.is_tensor(v)]
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.loss = self._step(guard=True)
        self.status.zero_()

    def _buffers(self, dev):
        """Static buffers of a subclass's step beyond the slots, sizes, labels and status."""

    def _params(self):
        ic, bc = self.milnet.i_classifier, self.milnet.b_classifier
        lin = ic._linear()
        W1, b1, W2, b2 = bc._q_params()
        return (lin.weight, lin.bias, W1, b1, W2, b2, None, None, bc.fcc.weight, bc.fcc.bias)

    def _loss(self):
        """The recorded forward and minibatch loss: (loss, ok), ok a device bool that is false for a refused batch."""
        classes, pred, _, _, crit = Fn.MILBagsDevFn.apply(self.slots, self.Ns, self._step_status, *self._params())
        ok = self._step_status[0] == 0
        n = self.Ns.clamp(0, self.max_rows)               # the live sizes (a refused batch's stay in range)
        first = torch.cumsum(n, 0) - n                    # each bag's first packed row
        mx = classes.gather(0, crit + first[:, None])     # the per-bag max instance, as feed._group_predictions
        return feed.minibatch_loss(self.criterion, pred, mx, self.labels), ok

    def _step(self, guard=False):
        self._step_status.zero_()
        loss, ok = self._loss()
        # a refused batch: NaN loss and no gradient (where's backward sends none to the unselected side)
        loss = torch.where(ok, loss, torch.full_like(loss, float("nan")))
        loss.backward()
        if guard:
            before = self._flat(self._kept)
        self.optimizer.step()
        if guard:
            # the update stands only for an accepted batch (bit for bit: a copy of the stepped values)
            kept = torch.where(ok, self._flat(self._kept), before)
            with torch.no_grad():
                torch._foreach_copy_(self._kept, [v.view_as(t) for v, t in
                                                  zip(kept.split([t.numel() for t in self._kept]), self._kept)])
        self.status.copy_(torch.where(self.status != 0, self.status, self._step_status))
        return loss.detach()

    @staticmethod
    def _flat(tensors):
        with torch.no_grad():
            return torch.cat([t.detach().reshape(-1).float() for t in tensors])

    def step(self) -> torch.Tensor:
        self.graph.replay()
        return self.loss

    def _snapshot(self):
        with torch.no_grad():
            params = [p.detach().clone() for p in self.params]
            state = {p: {k: (v.clone() if torch.is_tensor(v) else v) for k, v in self.optimizer.state[p].items()}
                     for p in self.params if self.optimizer.state.get(p)}
        return params, state

    def _restore(self, snap):
        params, state = snap
        with torch.no_grad():
            for p, v in zip(self.params, params):
                p.copy_(v)
            for p in self.params:
                cur, old = self.optimizer.state.get(p), state.get(p, {})
                for k, v in (cur or {}).items():
                    if torch.is_tensor(v):
                        v.copy_(old[k]) if k in old else v.zero_()
                    elif k in old:
                        cur[k] = old[k]


class ShardedTrainStepGraph(TrainStepGraph):
    """TrainStepGraph for a minibatch of row-sharded bags: one recorded step per rank of `group` (default: the world),
    replayed over batches of new local sizes.  The step is CudaShardBagDevOps under ShardedMILBagsFn (two all-gathers),
    the minibatch loss with its all-reduce(max) (sharded_max_prediction_bags_dev), the backward (three all-reduce(sum))
    and optimizer.step(): 6 collectives, as the eager sharded step.  Every rank builds the graph and replays it
    collectively, in the same order.

    Fill `slots[b, :n_b]` with this rank's rows of bag b, `Ns[b]` with n_b, `row_offsets[b]` with the global index of
    its first row and `labels` [nb, C], then `step()`.  A local n_b outside 1..max_rows (or a negative offset) refuses
    the batch on EVERY rank: this rank's flag rides in the loss's all-reduce(max), every rank's loss is NaN, and every
    rank keeps its parameters and optimizer state, so the replicas stay equal.  `status` holds this rank's own first
    refusal (1 + bag index), as in TrainStepGraph."""

    def __init__(self, milnet, criterion, optimizer, nb: int, max_rows: int, group=None, warmup: int = 1):
        self.group = group
        super().__init__(milnet, criterion, optimizer, nb, max_rows, warmup)

    def _buffers(self, dev):
        self.row_offsets = torch.zeros(self.nb, dtype=torch.int64, device=dev)

    def _loss(self):
        from . import sharded
        params = self._params()
        ops = sharded.CudaShardBagDevOps(params, self.Ns, self._step_status)
        classes, pred, _, _, crit = sharded.ShardedMILBagsFn.apply(ops, self.row_offsets, self.group, 1, self.slots,
                                                                   *params)
        mx, refused = sharded.sharded_max_prediction_bags_dev(classes, crit, self.row_offsets,
                                                              self.Ns.clamp(0, self.max_rows),
                                                              self._step_status[0] != 0, self.group)
        return feed.minibatch_loss(self.criterion, pred, mx, self.labels), ~refused
