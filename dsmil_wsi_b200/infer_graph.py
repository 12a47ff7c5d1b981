"""Inference over batches of ragged bags recorded once as a CUDA graph and replayed (ForwardBagsGraph), for serving
loops and the evaluation epoch; and the fold models of a cross-validation, each over its own bags, in one recorded
call (ForwardBagsModelsGraph), for the validation half of a fold epoch.

An eager `milnet(x)` or `milnet.forward_bags(xs)` pays its host cost on every call: ParamPack, workspace allocation,
the host-built bag table and its upload, ctypes.  For one slide per call that host work is most of the call.  Here one
dsmil_forward_bags_dev call is captured over static buffers -- the bags' feature addresses, their row counts and a
status word on the device -- and every batch of nb bags of 1..max_rows rows replays it.  The bags are read where they
are: `run` writes their addresses, not their rows.  The attend pass stays a programmatic dependent of phase 1 inside
the graph, so a replay keeps the eager call's overlap, and its outputs are the eager call's bits.  The fold form
captures one dsmil_forward_bags_models_dev call instead, with the same overlap over the table of every model's bags.
"""
from __future__ import annotations

import weakref
from typing import Sequence

import torch

from . import functional as Fn
from .modules import milnet_params
from .train_graph import _fold_route, step_shape


class ForwardBagsGraph:
    """One recorded inference call over nb bags of up to max_rows rows (nb = 1: one slide per call).

    `run(bags)` takes nb contiguous float32 [N_b, D] CUDA tensors with 1 <= N_b <= max_rows, replays the graph on the
    current stream and returns Fn.BagOutputs over the graph's packed outputs: per-bag (classes, prediction_bag, A, B)
    views, `.packed` and `.crit`.  They are overwritten by the next `run`; clone what must outlive it.  The object keeps
    the last call's bags alive until the next call, since the replay reads them in place.

    The graph reads the parameters in place: in-place updates (an optimizer step, `load_state_dict`) are seen by the
    next replay.  A parameter replaced by another tensor is not, and `run` raises RuntimeError; build a new graph.  A
    bag the library refuses (features not 16-byte aligned) sets `status` to 1 + its index (never cleared here) and the
    batch's outputs are a finite stand-in; read `status` when you synchronise.

    generic=True: also the identity-v shapes off the tensor-core batch (train_graph.step_shape), recorded over the
    generic batched route (dsmil_generic_forward_bags_dev, whose alignment rule refuses a bag of D % 4 == 0 that is not
    16-byte aligned, and otherwise one that is not 4-byte aligned).

    value=True: a model with a value network (passing_v), recorded over dsmil_value_forward_bags_dev with the features
    as value inputs (the generic route's alignment rule), with the bits of forward_bags in eval mode.  A recorded
    inference draws no dropout mask, so `run` refuses the model in train mode with a dropout_v > 0."""

    def __init__(self, milnet, nb: int, max_rows: int, warmup: int = 1, generic: bool = False, value: bool = False):
        self.D, self.C = step_shape(milnet, generic, value)
        self.value = bool(value)
        nb, max_rows = int(nb), int(max_rows)
        if not 1 <= nb <= 65535 or max_rows < 1:
            raise ValueError(f"ForwardBagsGraph: nb={nb} outside [1, 65535] or max_rows={max_rows} < 1")
        self._milnet = weakref.ref(milnet)      # a graph cached on the model must not keep it alive
        self.nb, self.max_rows = nb, max_rows
        self.params = milnet_params(milnet)
        Fn.require_cuda(self.params[-2], "the model")
        dev = self.device = self.params[-2].device
        self._addrs = _param_addrs(milnet)
        _staging(self, nb)
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)
        self._buffers(dev)
        # warm-up and capture on a batch of one-row bags of zeros
        self._scratch = torch.zeros(nb, self.D, device=dev)
        self.bag_list[0] = self._scratch.data_ptr() + 4 * self.D * torch.arange(nb, device=dev)
        self.bag_list[1] = 1
        Fn._warm_up(dev, warmup, self._record)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._record()
        self.status.zero_()

    def _buffers(self, dev):
        """Static buffers of a subclass's recorded work beyond the bag list and status."""

    def _record(self):
        if self.value:
            self.out = Fn.mil_forward_value_bags_dev(self.bag_list[0], None, self.bag_list[1], self.status,
                                                     self.max_rows, self.params)
        else:
            self.out = Fn.mil_forward_bags_dev(self.bag_list[0], self.bag_list[1], self.status, self.max_rows,
                                               self.params)
        self._after(*self.out)

    def _after(self, classes, pred, A, B, crit):
        """Work a subclass records after the forward, in the same graph."""

    def current(self) -> bool:
        """Whether the model is alive and holds the parameter tensors the graph was recorded on."""
        milnet = self._milnet()
        return milnet is not None and _param_addrs(milnet) == self._addrs

    def _load(self, bags):
        """Checks the bags and queues the upload of their addresses and row counts into the bag list."""
        if not self.current():
            raise RuntimeError("ForwardBagsGraph: the model is gone, or a parameter tensor of it was replaced since "
                               "the capture (the graph reads the old one); update parameters in place, or build a new "
                               "graph")
        if self.value:
            bc = self._milnet().b_classifier
            if bc.training and bc._v_params()[2] > 0.0:
                raise RuntimeError("ForwardBagsGraph: the model is in train mode with dropout_v > 0, and a recorded "
                                   "inference draws no dropout mask; call milnet.eval(), or train through "
                                   "TrainStepGraph(value=True)")
        if len(bags) != self.nb:
            raise ValueError(f"ForwardBagsGraph: {len(bags)} bags for a graph of nb={self.nb}")
        Ns = [_bag_rows(b, x, self.D, self.device, self.max_rows) for b, x in enumerate(bags)]
        _stage(self, bags, Ns)
        return Ns

    def release(self):
        """Drops the references to the last call's bags (call it once the stream has run the replay)."""
        self._bags = ()

    def run(self, bags: Sequence[torch.Tensor]) -> Fn.BagOutputs:
        Ns = self._load(bags)
        self.graph.replay()
        classes, pred, A, B, crit = self.out
        total = sum(Ns)
        return Fn.BagOutputs(classes[:total], pred, A[:total], B, Ns, crit)


def _param_addrs(milnet):
    return tuple(None if t is None else t.data_ptr() for t in milnet_params(milnet))


def _bag_rows(b, x, D, device, max_rows, fold=""):
    """The rows of bag b for a recorded inference of row capacity max_rows; ValueError / IndexError for a bag it cannot
    take (fold: the prefix naming the bag's model)."""
    if (not x.is_cuda or x.device != device or x.dtype != torch.float32 or x.dim() != 2
            or x.shape[1] != D or not x.is_contiguous()):
        raise ValueError(f"{fold}bag {b}: need a contiguous float32 [N, {D}] tensor on {device}, got "
                         f"{x.dtype} {tuple(x.shape)} on {x.device}")
    n = int(x.shape[0])
    if n < 1:
        raise IndexError(f"dsmil_b200: {fold}bag {b} is empty (N == 0)")
    if n > max_rows:
        raise ValueError(f"{fold}bag {b}: {n} rows exceed the inference graph's max_rows={max_rows}")
    return n


def _stage(g, bags, Ns):
    """Queues the upload of the bags' addresses and row counts into g.bag_list through g's pinned double-buffered
    staging, and keeps the bags alive until the next call (the replay reads them in place)."""
    i = g._turn
    g._turn ^= 1
    g._copied[i].synchronize()                   # the copy that last read this staging buffer has run
    g._stage_np[i][0] = [x.data_ptr() for x in bags]
    g._stage_np[i][1] = Ns
    g.bag_list.copy_(g._stage[i], non_blocking=True)
    g._copied[i].record()
    g._bags = list(bags)


def _staging(g, n):
    """g's bag list [2, n] on g.device (feature addresses; row counts) and its pinned staging: two buffers, the host
    fills one while the copy from the other may be queued."""
    g.bag_list = torch.zeros(2, n, dtype=torch.int64, device=g.device)
    g._stage = [torch.zeros(2, n, dtype=torch.int64, pin_memory=True) for _ in range(2)]
    g._stage_np = [s.numpy() for s in g._stage]
    g._copied = [torch.cuda.Event() for _ in range(2)]
    g._turn = 0
    g._bags = ()


class EvalBagsGraph(ForwardBagsGraph):
    """ForwardBagsGraph with the evaluation epoch's per-bag work recorded after the forward: each bag's max-instance
    prediction (the scores at its critical rows), its loss 0.5 * criterion(bag) + 0.5 * criterion(max instance) on
    [1, C] rows as feed.eval_epoch computes it, and the sigmoid predictions (average: sigmoid(max) + sigmoid(bag)).
    Fill `labels` [nb, C], then `run(bags)`; `loss` [nb] and `pred` [nb, C] hold the batch's results."""

    def __init__(self, milnet, criterion, nb: int, max_rows: int, average: bool = False, generic: bool = False,
                 value: bool = False):
        self.criterion, self.average = criterion, bool(average)
        super().__init__(milnet, nb, max_rows, generic=generic, value=value)

    def _buffers(self, dev):
        self.labels = torch.zeros(self.nb, self.C, device=dev)

    def _after(self, classes, pred, A, B, crit):
        n = self.bag_list[1].clamp(0, self.max_rows)          # the live sizes (a refused batch's stay in range)
        first = torch.cumsum(n, 0) - n                         # each bag's first packed row
        mx = classes.gather(0, crit + first[:, None])
        y = self.labels
        self.loss = torch.stack([(0.5 * self.criterion(pred[b:b + 1], y[b:b + 1]) +
                                  0.5 * self.criterion(mx[b:b + 1], y[b:b + 1])).reshape(()) for b in range(self.nb)])
        p = torch.sigmoid(pred)
        self.pred = torch.sigmoid(mx) + p if self.average else p


class ForwardBagsModelsGraph:
    """One recorded inference of the fold models of a cross-validation, model m over its own nbs[m] bags of up to
    max_rows rows (dsmil_forward_bags_models_dev): each fold model over its held-out bags in one replay.

    `run(bag_lists)` takes M lists, list m of nbs[m] contiguous float32 [N, D] CUDA tensors with 1 <= N <= max_rows,
    writes every bag's address and size through the pinned double-buffered staging (the bags are read in place),
    replays the graph and returns one Fn.BagOutputs per model, over model m's slices of the graph's packed outputs,
    with `.crit`.  Model m's outputs are bit for bit those of ForwardBagsGraph(milnets[m], nbs[m], max_rows) on its
    bags.  They are overwritten by the next `run`.

    The members and shapes are those of train_graph.fold_step_shape (generic=True: also folds on the generic batched
    route, recorded over dsmil_generic_forward_bags_models_dev).  The graph reads the parameters in place; a member
    whose parameter tensor was replaced makes `run` raise RuntimeError.  Refusal is per model: a bag the library
    refuses in model m (e.g. features not 16-byte aligned) sets `status[m]` to 1 + its index within the model (never
    cleared here), and only model m's outputs are a finite stand-in."""

    def __init__(self, milnets, nbs, max_rows: int, warmup: int = 1, generic: bool = False):
        milnets, nbs = list(milnets), tuple(int(n) for n in nbs)
        if len(nbs) != len(milnets):
            raise ValueError(f"ForwardBagsModelsGraph: {len(milnets)} models and {len(nbs)} group sizes")
        self.D, self.C, self.generic = _fold_route(milnets, generic)
        max_rows, M, ne = int(max_rows), len(nbs), sum(nbs)
        if min(nbs) < 1 or ne > 65535 or max_rows < 1:
            raise ValueError(f"ForwardBagsModelsGraph: group sizes {list(nbs)} outside [1, 65535] or "
                             f"max_rows={max_rows} < 1")
        self._milnets = [weakref.ref(net) for net in milnets]    # a cached graph must not keep the models alive
        self.M, self.nbs, self.max_rows = M, nbs, max_rows
        self._bag0 = [sum(nbs[:m]) for m in range(M)]             # each model's first entry
        params = [milnet_params(net) for net in milnets]
        for p in params:
            Fn.require_cuda(p[-2], "the model")
        self.params = [t for p in params for t in p]
        dev = self.device = params[0][-2].device
        self._addrs = [_param_addrs(net) for net in milnets]
        _staging(self, ne)
        self.status = torch.zeros(M, dtype=torch.int32, device=dev)
        self._buffers(dev)
        # warm-up and capture on one-row bags of zeros
        self._scratch = torch.zeros(ne, self.D, device=dev)
        self.bag_list[0] = self._scratch.data_ptr() + 4 * self.D * torch.arange(ne, device=dev)
        self.bag_list[1] = 1
        Fn._warm_up(dev, warmup, self._record)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._record()
        self.status.zero_()

    def _buffers(self, dev):
        """Static buffers of a subclass's recorded work beyond the bag list and status."""

    def _record(self):
        plist = [self.params[10 * m:10 * (m + 1)] for m in range(self.M)]
        self.out = Fn.mil_forward_bags_models_dev(self.nbs, self.bag_list[0], self.bag_list[1], self.status,
                                                  self.max_rows, plist, generic=self.generic)
        self._after(*self.out)

    def _after(self, classes, pred, A, B, crit):
        """Work a subclass records after the forward, in the same graph."""

    def current(self) -> bool:
        """Whether every model is alive and holds the parameter tensors the graph was recorded on."""
        nets = [r() for r in self._milnets]
        return all(net is not None and _param_addrs(net) == a for net, a in zip(nets, self._addrs))

    def members(self) -> list:
        """The models the graph was recorded on (None for one that is gone)."""
        return [r() for r in self._milnets]

    def _load(self, bag_lists):
        if not self.current():
            raise RuntimeError("ForwardBagsModelsGraph: a model is gone, or a parameter tensor of one was replaced "
                               "since the capture (the graph reads the old one); update parameters in place, or "
                               "build a new graph")
        if len(bag_lists) != self.M:
            raise ValueError(f"ForwardBagsModelsGraph: {len(bag_lists)} bag lists for a graph of {self.M} models")
        Ns = []
        for m, (bags, nb) in enumerate(zip(bag_lists, self.nbs)):
            if len(bags) != nb:
                raise ValueError(f"ForwardBagsModelsGraph: model {m} has {len(bags)} bags for a graph of nb={nb}")
            Ns.append([_bag_rows(b, x, self.D, self.device, self.max_rows, f"model {m}, ")
                       for b, x in enumerate(bags)])
        _stage(self, [x for bags in bag_lists for x in bags], [n for ns in Ns for n in ns])
        return Ns

    def release(self):
        """Drops the references to the last call's bags (call it once the stream has run the replay)."""
        self._bags = ()

    def run(self, bag_lists) -> list:
        Ns = self._load(bag_lists)
        self.graph.replay()
        classes, pred, A, B, crit = self.out
        outs = []
        for e, nb, ns in zip(self._bag0, self.nbs, Ns):
            r = e * self.max_rows
            outs.append(Fn.BagOutputs(classes[r:r + sum(ns)], pred[e:e + nb], A[r:r + sum(ns)], B[e:e + nb], ns,
                                      crit[e:e + nb]))
        return outs


class EvalBagsModelsGraph(ForwardBagsModelsGraph):
    """ForwardBagsModelsGraph with the evaluation epoch's per-bag work recorded after the forward, on each model's
    slices exactly as EvalBagsGraph records it: each bag's max-instance prediction, its loss 0.5 * criterion(bag) +
    0.5 * criterion(max instance) with that model's criterion (`criteria`: one per model, or one for all), and the
    sigmoid predictions (average: sigmoid(max) + sigmoid(bag)).  Fill `labels` [sum nbs, C] (model-major), then
    `run(bag_lists)`; `loss` [sum nbs] and `pred` [sum nbs, C] hold the batch's results, model-major."""

    def __init__(self, milnets, criteria, nbs, max_rows: int, average: bool = False, generic: bool = False):
        milnets = list(milnets)
        if isinstance(criteria, (list, tuple)):
            if len(criteria) != len(milnets):
                raise ValueError(f"EvalBagsModelsGraph: {len(criteria)} criteria for {len(milnets)} models")
            criteria = list(criteria)
        else:
            criteria = [criteria] * len(milnets)
        self.criteria, self.average = criteria, bool(average)
        super().__init__(milnets, nbs, max_rows, generic=generic)

    def _buffers(self, dev):
        self.labels = torch.zeros(sum(self.nbs), self.C, device=dev)

    def _after(self, classes, pred, A, B, crit):
        n = self.bag_list[1].clamp(0, self.max_rows)          # the live sizes (a refused model's stay in range)
        losses, preds = [], []
        for e, nb, criterion in zip(self._bag0, self.nbs, self.criteria):
            nm = n[e:e + nb]
            first = torch.cumsum(nm, 0) - nm + e * self.max_rows   # each bag's first packed row
            mx = classes.gather(0, crit[e:e + nb] + first[:, None])
            pm, y = pred[e:e + nb], self.labels[e:e + nb]
            losses += [(0.5 * criterion(pm[b:b + 1], y[b:b + 1]) +
                        0.5 * criterion(mx[b:b + 1], y[b:b + 1])).reshape(()) for b in range(nb)]
            p = torch.sigmoid(pm)
            preds.append(torch.sigmoid(mx) + p if self.average else p)
        self.loss = torch.stack(losses)
        self.pred = torch.cat(preds)
