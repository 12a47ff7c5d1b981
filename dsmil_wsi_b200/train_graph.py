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
from .functional import _warm_up
from .modules import BClassifier, FCLayer, milnet_params


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


def _shape_params(D, C, nonlinear, passing_v):
    """A DsmilParams of this shape for the library's shape tests, which read no weights: every weight the form has
    gets a stand-in address (any non-NULL one will do)."""
    p = _lib.DsmilParams(D, C, int(nonlinear), int(passing_v))
    p.Wi = p.bi = p.W1 = p.b1 = p.Wf = p.bf = 16
    if nonlinear:
        p.W2 = p.b2 = 16
    if passing_v:
        p.Wv = p.bv = 16
    return p


def step_shape(milnet, generic: bool = False, value: bool = False):
    """(D, C) of a MILNet whose training step the graph can record: FCLayer + BClassifier with identity v, on the
    batched tensor-core shapes (dsmil_shard_bags_supported), or with generic=True also on the generic batched route
    of the other identity-v shapes (dsmil_generic_bags_supported: e.g. D = 166 / 230, linear q, C > 4, D > 2048).
    value=True: a model with a value network (passing_v) instead, on the value calls' shapes
    (dsmil_value_bags_supported).  Anything else raises ValueError naming the shape."""
    ic, bc = getattr(milnet, "i_classifier", None), getattr(milnet, "b_classifier", None)
    if not (isinstance(ic, FCLayer) and isinstance(bc, BClassifier)):
        raise ValueError("graph-captured training needs MILNet(FCLayer, BClassifier); got "
                         f"{type(ic).__name__} + {type(bc).__name__}")
    W1, b1, W2, b2 = bc._q_params()
    Wv, _, _ = bc._v_params()
    C, D = int(bc.fcc.weight.shape[0]), int(bc.fcc.weight.shape[2])
    p = _shape_params(D, C, W2 is not None, Wv is not None)
    lib = _lib.load()
    if value:
        if Wv is not None and lib.dsmil_value_bags_supported(ctypes.byref(p)):
            return D, C
        raise ValueError(f"value=True records models with a value network only; D={D}, C={C}, "
                         f"nonlinear={W2 is not None}, passing_v={Wv is not None} is not one (identity v: "
                         "value=False)")
    if lib.dsmil_shard_bags_supported(ctypes.byref(p)):
        return D, C
    if generic and lib.dsmil_generic_bags_supported(ctypes.byref(p)):
        return D, C
    if generic:
        raise ValueError(f"graph-captured training takes identity v only; D={D}, C={C}, "
                         f"nonlinear={W2 is not None}, passing_v={Wv is not None} is on no batched route")
    raise ValueError(f"graph-captured training runs on the batched tensor-core path only; D={D}, C={C}, "
                     f"nonlinear={W2 is not None}, passing_v={Wv is not None} is not on it "
                     "(generic=True records the generic batched route of the other identity-v shapes)")


def fold_step_shape(milnets, generic: bool = False):
    """(D, C) of MILNets whose fold step the graph can record: each on step_shape's route, all of one D, C and q form,
    1 to 8 of them, together on the fused fold shapes (dsmil_models_supported).  generic=True also takes folds on the
    generic batched route (dsmil_generic_models_supported: e.g. the classic-MIL D = 166 / 230, a linear q, C > 4,
    D > 2048); tensor-core shapes whose folds do not fit the fused fold step stay refused.  Else ValueError."""
    return _fold_route(milnets, generic)[:2]


def _fold_route(milnets, generic):
    """(D, C, whether the folds take the generic fold calls) of fold_step_shape."""
    milnets = list(milnets)
    if not 1 <= len(milnets) <= Fn.MAX_MODELS:
        raise ValueError(f"a fold step takes 1 to {Fn.MAX_MODELS} folds, got {len(milnets)}")
    shapes = [step_shape(net, generic) for net in milnets]
    for m, sh in enumerate(shapes):
        if sh != shapes[0]:
            raise ValueError(f"fold {m}: (D, C)={sh} differs from fold 0's {shapes[0]}")
    D, C = shapes[0]
    forms = [milnet_q_nonlinear(net) for net in milnets]
    for m, nl in enumerate(forms):
        if nl != forms[0]:
            raise ValueError(f"fold {m}: nonlinear={nl} differs from fold 0's {forms[0]}")
    M, lib = len(milnets), _lib.load()
    ps = (_lib.DsmilParams * M)(*[_shape_params(D, C, forms[0], False)] * M)
    if lib.dsmil_shard_bags_supported(ctypes.byref(ps[0])):
        if lib.dsmil_models_supported(ps, M):
            return D, C, False
        raise ValueError(f"the graph-captured fold step runs on the fused fold shapes only; M={M}, D={D}, "
                         f"C={C} is not on them: train these folds one at a time (train_epoch(graph=True))")
    # off the tensor-core batch: only generic=True gets here (step_shape refuses the shape otherwise)
    if not lib.dsmil_generic_models_supported(ps, M):
        raise ValueError(f"the generic graph-captured fold step does not take M={M}, D={D}, C={C}, "
                         f"nonlinear={forms[0]}")
    return D, C, True


def milnet_q_nonlinear(milnet) -> bool:
    """Whether a MILNet's q is the nonlinear Linear-ReLU-Linear-Tanh (dsmil.py:31) rather than one Linear (:33)."""
    return milnet.b_classifier._q_params()[2] is not None


def _flat(tensors):
    with torch.no_grad():
        return torch.cat([t.detach().reshape(-1).float() for t in tensors])


def _snapshot(optimizer, params):
    with torch.no_grad():
        values = [p.detach().clone() for p in params]
        state = {p: {k: (v.clone() if torch.is_tensor(v) else v) for k, v in optimizer.state[p].items()}
                 for p in params if optimizer.state.get(p)}
    return values, state


def _restore(optimizer, params, snap):
    """Puts parameters and optimizer state back in place; state created since the snapshot is reset to zeros."""
    values, state = snap
    with torch.no_grad():
        for p, v in zip(params, values):
            p.copy_(v)
        for p in params:
            cur, old = optimizer.state.get(p), state.get(p, {})
            for k, v in (cur or {}).items():
                if torch.is_tensor(v):
                    v.copy_(old[k]) if k in old else v.zero_()
                elif k in old:
                    cur[k] = old[k]


def _kept_tensors(optimizer, params):
    """What a refused step puts back: the parameters and every tensor of the optimizer state."""
    return params + [v for p in params for v in optimizer.state.get(p, {}).values() if torch.is_tensor(v)]


def _keep_if(ok, kept, before):
    """The stepped values of `kept` stand only where ok (bit for bit: a copy of them); else `before` returns."""
    new = torch.where(ok, _flat(kept), before)
    with torch.no_grad():
        torch._foreach_copy_(kept, [v.view_as(t) for v, t in zip(new.split([t.numel() for t in kept]), kept)])


def _capture_step(dev, optimizers, params, warmup, step):
    """Records a training step as a CUDA graph.  `step(None)` runs `warmup` times on a side stream; then every
    optimizer's parameters and state go back in place (so the graph's addresses stay valid; state the warm-up created
    is reset to zeros) and `step(kept)` is captured, kept holding each optimizer's tensors that a refused step puts
    back.  Returns (graph, the captured step's result, kept)."""
    snaps = [_snapshot(o, p) for o, p in zip(optimizers, params)]

    def warm():
        for o in optimizers:
            o.zero_grad(set_to_none=True)
        step(None)
    _warm_up(dev, warmup, warm)
    for o, p, snap in zip(optimizers, params, snaps):
        _restore(o, p, snap)
        o.zero_grad(set_to_none=True)
    kept = [_kept_tensors(o, p) for o, p in zip(optimizers, params)]   # the optimizer state exists now
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step(kept)
    return graph, out, kept


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
    the graph's gradient buffers.  generic=True: also the shapes off the tensor-core batch (step_shape), whose step
    records the generic batched route with the bits of its eager step; their bags follow the alignment rule of
    dsmil_generic_forward_bags_train_dev, which the slots meet.

    value=True: a model with a value network (passing_v), whose step records MILValueBagsDevFn with the bits of the
    eager functional.mil_forward_value_bags(grad=True) step.  When the model's dropout_v is > 0 at construction (the
    p is frozen then, as the other hyperparameters), the value inputs are a static `v_inputs` [nb, max_rows, D]
    buffer, which the caller fills as it fills `slots` (bag b's features times its dropout mask; see
    BClassifier._v_input); otherwise `v_inputs` is None and the value inputs are the slots."""

    def __init__(self, milnet, criterion, optimizer, nb: int, max_rows: int, warmup: int = 1, generic: bool = False,
                 value: bool = False):
        check_optimizer(optimizer)
        D, C = step_shape(milnet, generic, value)
        self.value = bool(value)
        nb, max_rows = int(nb), int(max_rows)
        if not 1 <= nb <= 65535 or max_rows < 1:
            raise ValueError(f"TrainStepGraph: nb={nb} outside [1, 65535] or max_rows={max_rows} < 1")
        self.milnet, self.criterion, self.optimizer = milnet, criterion, optimizer
        self.nb, self.max_rows = nb, max_rows
        self.params = [p for g in optimizer.param_groups for p in g["params"]]
        dev = milnet.b_classifier.fcc.weight.device
        Fn.require_cuda(milnet.b_classifier.fcc.weight, "the model")
        self.slots = torch.zeros(nb, max_rows, D, device=dev)
        self.v_inputs = (torch.zeros(nb, max_rows, D, device=dev)
                         if self.value and milnet.b_classifier._v_params()[2] > 0.0 else None)
        self.Ns = torch.ones(nb, dtype=torch.int64, device=dev)
        self.labels = torch.zeros(nb, C, device=dev)
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)
        self._step_status = torch.zeros(1, dtype=torch.int32, device=dev)   # this replay's planners
        self._buffers(dev)
        self.graph, self.loss, (self._kept,) = _capture_step(
            dev, [optimizer], [self.params], warmup, lambda kept: self._step(None if kept is None else kept[0]))
        self.status.zero_()

    def _buffers(self, dev):
        """Static buffers of a subclass's step beyond the slots, sizes, labels and status."""

    def _params(self):
        return milnet_params(self.milnet)

    def _loss(self):
        """The recorded forward and minibatch loss: (loss, ok), ok a device bool that is false for a refused batch."""
        if self.value:
            classes, pred, _, _, crit = Fn.MILValueBagsDevFn.apply(self.slots, self.v_inputs, self.Ns,
                                                                   self._step_status, *self._params())
        else:
            classes, pred, _, _, crit = Fn.MILBagsDevFn.apply(self.slots, self.Ns, self._step_status, *self._params())
        ok = self._step_status[0] == 0
        n = self.Ns.clamp(0, self.max_rows)               # the live sizes (a refused batch's stay in range)
        first = torch.cumsum(n, 0) - n                    # each bag's first packed row
        mx = classes.gather(0, crit + first[:, None])     # the per-bag max instance, as feed._group_predictions
        return feed.minibatch_loss(self.criterion, pred, mx, self.labels), ok

    def _step(self, kept=None):
        """One step; with `kept` (the recorded step) the update stands only for an accepted batch."""
        self._step_status.zero_()
        loss, ok = self._loss()
        # a refused batch: NaN loss and no gradient (where's backward sends none to the unselected side)
        loss = torch.where(ok, loss, torch.full_like(loss, float("nan")))
        loss.backward()
        if kept is not None:
            before = _flat(kept)
        self.optimizer.step()
        if kept is not None:
            _keep_if(ok, kept, before)
        self.status.copy_(torch.where(self.status != 0, self.status, self._step_status))
        return loss.detach()

    def step(self) -> torch.Tensor:
        self.graph.replay()
        return self.loss


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


class FoldTrainStepGraph:
    """One recorded step of the fold models of a cross-validation: fold m takes nbs[m] bags of up to max_rows rows.

    The step is feed.train_epoch_models' step over the capture-safe fold calls (MILBagsModelsDevFn): one forward for
    all folds, each fold's feed.minibatch_loss on its own slices, the sum of the folds' losses, one backward, every
    fold's optimizer.step().  Fill `slots[m][b, :n]` with bag b of fold m, `Ns` [sum nbs] (fold-major) with the row
    counts and `labels` [sum nbs, C], then `step()` replays the graph and returns the M losses (a device tensor,
    overwritten by the next replay).  With the same batches, fold m's losses, gradients and parameters are bit for
    bit those of its own TrainStepGraph.  generic=True: also folds on the generic batched route (fold_step_shape),
    whose step records MILBagsModelsGenericDevFn with the bits of each fold's TrainStepGraph(generic=True); fused
    tensor-core fold shapes keep the fused fold step.

    Refusal is per fold: a fold with a bag outside 1..max_rows has `status[m]` set (the first refusal's 1 + bag index
    within the fold; never cleared here), a NaN loss, and its parameters and optimizer state left as they were; the
    other folds step normally.  Warm-up, capture and hyperparameters behave as in TrainStepGraph.

    criterion: one for every fold, or a list or tuple of one per fold (feed.fold_criteria), fold m's minibatch_loss
    then using criterion[m]."""

    def __init__(self, milnets, criterion, optimizers, nbs, max_rows: int, warmup: int = 1, generic: bool = False):
        milnets, optimizers, nbs = list(milnets), list(optimizers), [int(n) for n in nbs]
        M = len(milnets)
        if len(optimizers) != M or len(nbs) != M:
            raise ValueError(f"FoldTrainStepGraph: {M} milnets, {len(optimizers)} optimizers and {len(nbs)} group "
                             "sizes")
        for opt in optimizers:
            check_optimizer(opt)
        D, C, self.generic = _fold_route(milnets, generic)
        ne, max_rows = sum(nbs), int(max_rows)
        if min(nbs) < 1 or ne > 65535 or max_rows < 1:
            raise ValueError(f"FoldTrainStepGraph: group sizes {nbs} outside [1, 65535] or max_rows={max_rows} < 1")
        self.milnets, self.criterion, self.optimizers = milnets, criterion, optimizers
        self.criteria = feed.fold_criteria(criterion, M)
        self.nbs, self.max_rows = tuple(nbs), max_rows
        self.params = [[p for g in opt.param_groups for p in g["params"]] for opt in optimizers]
        dev = milnets[0].b_classifier.fcc.weight.device
        for net in milnets:
            Fn.require_cuda(net.b_classifier.fcc.weight, "the model")
        self._bag0 = [sum(nbs[:m]) for m in range(M)]                      # each fold's first entry
        self._slots = torch.zeros(ne, max_rows, D, device=dev)
        self.slots = [self._slots[e:e + n] for e, n in zip(self._bag0, nbs)]
        self.Ns = torch.ones(ne, dtype=torch.int64, device=dev)
        self.labels = torch.zeros(ne, C, device=dev)
        self.status = torch.zeros(M, dtype=torch.int32, device=dev)
        self._step_status = torch.zeros(M, dtype=torch.int32, device=dev)   # this replay's planners
        self.graph, self.loss, self._kept = _capture_step(dev, optimizers, self.params, warmup, self._step)
        self.status.zero_()

    def _step(self, kept=None):
        """One step; with `kept` (the recorded step, one list per fold) each fold's update stands only if it was
        accepted."""
        self._step_status.zero_()
        params = [t for net in self.milnets for t in milnet_params(net)]
        fn = Fn.MILBagsModelsGenericDevFn if self.generic else Fn.MILBagsModelsDevFn
        classes, pred, _, _, crit = fn.apply(self.nbs, self._slots, self.Ns, self._step_status, *params)
        n = self.Ns.clamp(0, self.max_rows)                # the live sizes (a refused fold's stay in range)
        losses, oks = [], []
        for m, (e, nb) in enumerate(zip(self._bag0, self.nbs)):
            nm = n[e:e + nb]
            first = torch.cumsum(nm, 0) - nm + e * self.max_rows          # each bag's first packed row
            mx = classes.gather(0, crit[e:e + nb] + first[:, None])
            lm = feed.minibatch_loss(self.criteria[m], pred[e:e + nb], mx, self.labels[e:e + nb])
            ok = self._step_status[m] == 0
            # a refused fold: NaN loss and no gradient (where's backward sends none to the unselected side)
            losses.append(torch.where(ok, lm, torch.full_like(lm, float("nan"))))
            oks.append(ok)
        total = losses[0]
        for lm in losses[1:]:
            total = total + lm
        total.backward()
        if kept is not None:
            before = [_flat(k) for k in kept]
        for opt in self.optimizers:
            opt.step()
        if kept is not None:
            for ok, k, b in zip(oks, kept, before):
                _keep_if(ok, k, b)
        self.status.copy_(torch.where(self.status != 0, self.status, self._step_status))
        return torch.stack([lm.detach() for lm in losses])

    def step(self) -> torch.Tensor:
        self.graph.replay()
        return self.loss

