"""torch.autograd bridges from PyTorch tensors to the C ABI (include/dsmil_b200.h).

PyTorch is plumbing here (device memory, streams, autograd graph); every FLOP of the DSMIL
aggregator runs in libdsmil_b200.so.  CPU tensors are rejected: there is no CPU path.
"""
from __future__ import annotations

import collections.abc
import ctypes as C
from typing import Optional, Sequence, Tuple

import torch

from . import _lib

Q_DIM = 128


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _f32c(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    if t is None:
        return None
    if t.dtype != torch.float32:
        raise TypeError(f"dsmil_b200 computes in fp32 (as the reference does); got {t.dtype}")
    return t.contiguous()


def require_cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(
            f"dsmil_b200: {what} is on '{t.device}'. The H100-native DSMIL path runs on CUDA only "
            "(no CPU fallback); move the module and the bag to a CUDA device.")


class ParamPack:
    """Raw-pointer view of the parameter tensors, rebuilt on every call (no cached pointers:
    callers deepcopy / .cpu() / .cuda() / reassign sub-modules, SURVEY §7.2-6)."""

    def __init__(self, Wi, bi, W1, b1, W2, b2, Wv, bv, Wf, bf):
        self.tensors = [_f32c(t) for t in (Wi, bi, W1, b1, W2, b2, Wv, bv, Wf, bf)]
        Wi, bi, W1, b1, W2, b2, Wv, bv, Wf, bf = self.tensors
        self.C, self.D = int(Wf.shape[0]), int(Wf.shape[2])
        if Wi is not None and tuple(Wi.shape) != (self.C, self.D):
            raise ValueError(f"instance classifier weight {tuple(Wi.shape)} does not match C={self.C}, D={self.D}")
        self.nonlinear = W2 is not None
        self.passing_v = Wv is not None
        if W1.shape != (Q_DIM, self.D) or Wf.shape != (self.C, self.C, self.D):
            raise ValueError(f"parameter shapes do not form a DSMIL aggregator: W1 {tuple(W1.shape)}, "
                             f"Wf {tuple(Wf.shape)} for D={self.D}, C={self.C}")
        dev = Wf.device
        for t in self.tensors:
            if t is not None:
                require_cuda(t, "a parameter")
                if t.device != dev:
                    raise RuntimeError("dsmil_b200: parameters live on different devices")
        self.device = dev
        self.struct = _lib.DsmilParams(self.D, self.C, int(self.nonlinear), int(self.passing_v),
                                       _ptr(Wi), _ptr(bi), _ptr(W1), _ptr(b1), _ptr(W2), _ptr(b2),
                                       _ptr(Wv), _ptr(bv), _ptr(Wf), _ptr(bf))

    @property
    def ref(self):
        return C.byref(self.struct)


def _workspace(nbytes: int, device) -> torch.Tensor:
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)


def _check_feats(feats: torch.Tensor, D: int) -> torch.Tensor:
    require_cuda(feats, "the bag (feats)")
    if feats.dim() != 2 or feats.shape[1] != D:
        raise ValueError(f"feats must be [N, {D}], got {tuple(feats.shape)}")
    return _f32c(feats)


# --------------------------------------------------------------------------- fused MILNet forward
class MILForwardFn(torch.autograd.Function):
    """(classes, prediction_bag, A, B) = MILNet.forward(feats)   -- dsmil.py:70-74.

    args: feats, v_input (feats after the dropout of dsmil.py:36, or None), v_mask (or None),
          classes_in (None for the fused form; the given scores for b_classifier(feats, c)),
          then the ten parameter tensors (None where the variant has none).
    """

    @staticmethod
    def forward(ctx, want_grad, feats, v_input, v_mask, classes_in, Wi, bi, W1, b1, W2, b2, Wv, bv, Wf, bf):
        lib = _lib.load()
        ctx.set_materialize_grads(False)
        P = ParamPack(Wi, bi, W1, b1, W2, b2, Wv, bv, Wf, bf)
        X = _check_feats(feats, P.D)
        if X.device != P.device:
            raise RuntimeError(f"dsmil_b200: bag on {X.device} but parameters on {P.device}")
        N, Cc, D = int(X.shape[0]), P.C, P.D
        if N == 0:
            raise IndexError("dsmil_b200: empty bag (N == 0); the reference fails at dsmil.py:53 too")
        xv = _f32c(v_input) if (v_input is not None and P.passing_v) else None
        cin = None
        if classes_in is not None:
            require_cuda(classes_in, "classes")
            cin = _f32c(classes_in.reshape(N, Cc))
        # grad mode is already off inside Function.forward, so the caller tells us (mil_forward checks
        # torch.is_grad_enabled()); without it the activations are not saved and Q stays in the blocked workspace
        need_grad = bool(want_grad) and any(ctx.needs_input_grad)
        with torch.cuda.device(X.device):
            new = lambda *s: torch.empty(*s, dtype=torch.float32, device=X.device)
            classes = new(N, Cc) if cin is None else new(0, Cc)  # bag form: scores are an input, not an output
            pred, A, B = new(1, Cc), new(N, Cc), new(1, Cc, D)
            crit = torch.empty(Cc, dtype=torch.int64, device=X.device)
            sQ = new(N, Q_DIM) if need_grad else None
            sH = new(N, Q_DIM) if (need_grad and P.nonlinear) else None
            sV = new(N, D) if (need_grad and P.passing_v) else None
            ws = _workspace(lib.dsmil_forward_workspace_bytes(P.ref, N), X.device)
            if cin is None:
                if Wi is None or bi is None:
                    raise ValueError("fused MILNet forward needs the instance classifier's weight and bias")
                rc = lib.dsmil_forward(P.ref, _ptr(X), _ptr(xv), N, _ptr(classes), _ptr(pred), _ptr(A), _ptr(B),
                                       _ptr(crit), _ptr(sQ), _ptr(sH), _ptr(sV), _ptr(ws), ws.numel(), _stream())
                _lib.check(rc, "dsmil_forward")
            else:
                rc = lib.dsmil_bag_forward(P.ref, _ptr(X), _ptr(xv), _ptr(cin), N, _ptr(pred), _ptr(A), _ptr(B),
                                           _ptr(crit), _ptr(sQ), _ptr(sH), _ptr(sV), _ptr(ws), ws.numel(),
                                           _stream())
                _lib.check(rc, "dsmil_bag_forward")
        ctx.fused_scores = cin is None
        ctx.need = need_grad
        if need_grad:
            ctx.save_for_backward(X, xv, v_mask, sQ, sH, sV, A, B, crit, *[t for t in P.tensors])
        ctx.mark_non_differentiable(crit)
        if cin is not None:
            ctx.mark_non_differentiable(classes)  # given scores only feed the (non-differentiable) arg-max
        return classes, pred, A, B, crit

    @staticmethod
    def backward(ctx, g_classes, g_pred, g_A, g_B, _g_crit):
        lib = _lib.load()
        X, xv, v_mask, sQ, sH, sV, A, B, crit, *params = ctx.saved_tensors
        P = ParamPack(*params)
        N, Cc, D = int(X.shape[0]), P.C, P.D
        needs = ctx.needs_input_grad[1:]  # (want_grad,) feats, v_input, v_mask, classes_in, 10 params
        names = ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf")
        with torch.cuda.device(X.device):
            out = {}
            for i, (nm, t) in enumerate(zip(names, P.tensors)):
                # Wi/bi only get gradient through `classes` in the fused form
                want = t is not None and needs[4 + i] and not (nm in ("Wi", "bi") and not ctx.fused_scores)
                out[nm] = torch.empty_like(t) if want else None
            gX = torch.empty_like(X) if needs[0] else None
            G = _lib.DsmilGrads(*[_ptr(out[n]) for n in ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf")],
                                _ptr(gX))
            dc = _f32c(g_classes) if (g_classes is not None and ctx.fused_scores) else None
            dp = _f32c(g_pred.reshape(-1)) if g_pred is not None else None
            dA = _f32c(g_A) if g_A is not None else None
            dB = _f32c(g_B.reshape(Cc, D)) if g_B is not None else None
            ws = _workspace(lib.dsmil_backward_workspace_bytes(P.ref, N, int(gX is not None)), X.device)
            rc = lib.dsmil_backward(P.ref, _ptr(X), _ptr(xv), N, _ptr(sQ), _ptr(sH), _ptr(sV), _ptr(A), _ptr(B),
                                    _ptr(crit), _ptr(dc), _ptr(dp), _ptr(dA), _ptr(dB), C.byref(G),
                                    _ptr(v_mask), _ptr(ws), ws.numel(), _stream())
            _lib.check(rc, "dsmil_backward")
        return (None, gX, None, None, None, *[out[n] for n in names])


# --------------------------------------------------------------------------- instance scores alone
class InstanceScoresFn(torch.autograd.Function):
    """classes = feats @ Wi.T + bi   -- FCLayer.fc / IClassifier.fc (dsmil.py:11, :24)."""

    @staticmethod
    def forward(ctx, feats, Wi, bi):
        lib = _lib.load()
        require_cuda(Wi, "i_classifier.fc.weight")
        Wi_c, bi_c = _f32c(Wi), _f32c(bi)
        Cc, D = int(Wi_c.shape[0]), int(Wi_c.shape[1])
        X = _check_feats(feats, D)
        N = int(X.shape[0])
        P = _lib.DsmilParams(D, Cc, 0, 0, _ptr(Wi_c), _ptr(bi_c), None, None, None, None, None, None, None, None)
        with torch.cuda.device(X.device):
            classes = torch.empty(N, Cc, dtype=torch.float32, device=X.device)
            _lib.check(lib.dsmil_instance_scores(C.byref(P), _ptr(X), N, _ptr(classes), _stream()),
                       "dsmil_instance_scores")
        ctx.save_for_backward(X, Wi_c, bi_c)
        return classes

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        X, Wi_c, bi_c = ctx.saved_tensors
        Cc, D, N = int(Wi_c.shape[0]), int(Wi_c.shape[1]), int(X.shape[0])
        if N == 0:
            return (torch.zeros_like(X) if ctx.needs_input_grad[0] else None, torch.zeros_like(Wi_c),
                    torch.zeros_like(bi_c))
        P = _lib.DsmilParams(D, Cc, 0, 0, _ptr(Wi_c), _ptr(bi_c), None, None, None, None, None, None, None, None)
        with torch.cuda.device(X.device):
            g = _f32c(g)
            gW = torch.empty_like(Wi_c) if ctx.needs_input_grad[1] else None
            gb = torch.empty_like(bi_c) if ctx.needs_input_grad[2] else None
            gX = torch.empty_like(X) if ctx.needs_input_grad[0] else None
            ws = _workspace(lib.dsmil_backward_workspace_bytes(C.byref(P), N, 0), X.device)
            _lib.check(lib.dsmil_instance_scores_backward(C.byref(P), _ptr(X), N, _ptr(g), _ptr(gW), _ptr(gb),
                                                          _ptr(gX), _ptr(ws), ws.numel(), _stream()),
                       "dsmil_instance_scores_backward")
        return gX, gW, gb


def instance_scores(feats: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    return InstanceScoresFn.apply(feats, weight, bias)


def mil_forward(feats, params: Sequence[Optional[torch.Tensor]], v_input=None, v_mask=None, classes_in=None
                ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """Returns (classes, prediction_bag, A, B, crit_idx)."""
    want_grad = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (feats, *params))
    return MILForwardFn.apply(want_grad, feats, v_input, v_mask, classes_in, *params)


class BagOutputs(collections.abc.Sequence):
    """Per-bag (classes, prediction_bag, A, B) views over the packed outputs of dsmil_forward_bags, created on
    access: materialising 4 views per bag eagerly costs ~1.5 us each on the host -- as long as the GPU work of a
    16-bag step -- so the sequence hands them out lazily.  `.packed` exposes the packed tensors themselves."""

    def __init__(self, classes, pred, A, B, Ns, crit=None):
        self.packed = (classes, pred, A, B)
        self.Ns = list(Ns)
        self.crit = crit          # [nb, C] critical rows within each bag, when the caller kept them
        self._offsets = None

    def __len__(self):
        return len(self.Ns)

    def __getitem__(self, b):
        if isinstance(b, slice):
            return [self[i] for i in range(*b.indices(len(self)))]
        if b < 0:
            b += len(self)
        if not 0 <= b < len(self):
            raise IndexError(b)
        if self._offsets is None:
            self._offsets = [0]
            for n in self.Ns:
                self._offsets.append(self._offsets[-1] + n)
        lo, hi = self._offsets[b], self._offsets[b + 1]
        classes, pred, A, B = self.packed
        return classes[lo:hi], pred[b:b + 1], A[lo:hi], B[b:b + 1]


def _bag_table(bags, P: ParamPack):
    """Checked, contiguous bags and their host arrays (features pointers, row counts) for the bag-table calls."""
    xs = [_check_feats(b, P.D) for b in bags]
    Ns = [int(x.shape[0]) for x in xs]
    if min(Ns) == 0:
        raise IndexError("dsmil_b200: empty bag (N == 0) in the batch")
    for x in xs:
        if x.device != P.device:
            raise RuntimeError(f"dsmil_b200: bag on {x.device} but parameters on {P.device}")
    nb = len(xs)
    return xs, Ns, (C.c_void_p * nb)(*[x.data_ptr() for x in xs]), (C.c_int64 * nb)(*Ns)


class MILBagsFn(torch.autograd.Function):
    """Packed (classes, pred, A, B, crit) of a batch of bags, differentiable: dsmil_forward_bags_train forward,
    dsmil_backward_bags backward (one call each for the whole batch).  args: nb, the nb bags, then the ten parameter
    tensors.  Parameter gradients are sums over the bags, as autograd gives for a loss over the packed outputs."""

    @staticmethod
    def forward(ctx, nb, *args):
        lib = _lib.load()
        ctx.set_materialize_grads(False)
        P = ParamPack(*args[nb:])
        if P.passing_v:
            raise NotImplementedError("forward_bags(grad=True): passing_v models go through MILNet.forward per bag")
        xs, Ns, c_X, c_N = _bag_table(args[:nb], P)
        total, Cc, D, dev = sum(Ns), P.C, P.D, P.device
        with torch.cuda.device(dev):
            new = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
            classes, A = new(total, Cc), new(total, Cc)
            pred, B = new(nb, Cc), new(nb, Cc, D)
            crit = torch.empty(nb, Cc, dtype=torch.int64, device=dev)
            sQ = new(total, Q_DIM)
            sH = new(total, Q_DIM) if P.nonlinear else None
            ws = _workspace(lib.dsmil_forward_bags_train_workspace_bytes(P.ref, c_N, nb), dev)
            rc = lib.dsmil_forward_bags_train(P.ref, c_X, c_N, nb, _ptr(classes), _ptr(pred), _ptr(A), _ptr(B),
                                              _ptr(crit), _ptr(sQ), _ptr(sH), _ptr(ws), ws.numel(), _stream())
            _lib.check(rc, "dsmil_forward_bags_train")
        ctx.nb, ctx.Ns = nb, Ns
        ctx.save_for_backward(*xs, sQ, sH, A, B, crit, *P.tensors)
        ctx.mark_non_differentiable(crit)
        return classes, pred, A, B, crit

    @staticmethod
    def backward(ctx, g_classes, g_pred, g_A, g_B, _g_crit):
        lib = _lib.load()
        nb, Ns = ctx.nb, ctx.Ns
        saved = ctx.saved_tensors
        xs, (sQ, sH, A, B, crit), params = saved[:nb], saved[nb:nb + 5], saved[nb + 5:]
        P = ParamPack(*params)
        need_bags, need_params = ctx.needs_input_grad[1:1 + nb], ctx.needs_input_grad[1 + nb:]
        names = ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf")
        dev = P.device
        c_X = (C.c_void_p * nb)(*[x.data_ptr() for x in xs])
        c_N = (C.c_int64 * nb)(*Ns)
        with torch.cuda.device(dev):
            out = {nm: (torch.empty_like(t) if t is not None and need else None)
                   for nm, t, need in zip(names, P.tensors, need_params)}
            gX = torch.empty(sum(Ns), P.D, dtype=torch.float32, device=dev) if any(need_bags) else None
            G = _lib.DsmilGrads(*[_ptr(out[n]) for n in names], _ptr(gX))
            dc, dp, dA, dB = (_f32c(t) for t in (g_classes, g_pred, g_A, g_B))
            ws = _workspace(lib.dsmil_backward_bags_workspace_bytes(P.ref, c_N, nb, int(gX is not None)), dev)
            rc = lib.dsmil_backward_bags(P.ref, c_X, c_N, nb, _ptr(sQ), _ptr(sH), _ptr(A), _ptr(B), _ptr(crit),
                                         _ptr(dc), _ptr(dp), _ptr(dA), _ptr(dB), C.byref(G), _ptr(ws), ws.numel(),
                                         _stream())
            _lib.check(rc, "dsmil_backward_bags")
        gxs, lo = [], 0
        for n, need in zip(Ns, need_bags):
            gxs.append(gX[lo:lo + n] if need else None)
            lo += n
        return (None, *gxs, *[out[n] for n in names])


class MILBagsDevFn(torch.autograd.Function):
    """MILBagsFn over the capture-safe entry points (dsmil_forward_bags_train_dev / dsmil_backward_bags_dev): the bag
    list lives on the device, so one recorded call serves every batch of nb bags of 1..max_rows rows.

    args: slots [nb, max_rows, D] (bag b is slots[b, :Ns[b]]), Ns [nb] int64 and status [1] int32 on the device, then
    the ten parameter tensors.  The packed per-row outputs (classes, A) have nb * max_rows rows; the live ones are
    packed at the prefix sums of Ns, as MILBagsFn packs them.  Parameter gradients only (no gradient to the slots)."""

    @staticmethod
    def forward(ctx, slots, Ns, status, *params):
        lib = _lib.load()
        ctx.set_materialize_grads(False)
        P = ParamPack(*params)
        if not lib.dsmil_shard_bags_supported(P.ref):
            raise ValueError(f"graph-captured training runs on the batched tensor-core path only; D={P.D}, C={P.C}, "
                             f"nonlinear={P.nonlinear}, passing_v={P.passing_v} is not on it")
        if slots.dim() != 3 or slots.shape[2] != P.D or slots.dtype != torch.float32 or not slots.is_contiguous():
            raise ValueError(f"slots must be contiguous float32 [nb, max_rows, {P.D}], got {tuple(slots.shape)}")
        nb, max_rows = int(slots.shape[0]), int(slots.shape[1])
        dev = P.device
        with torch.cuda.device(dev):
            new = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
            rows = nb * max_rows
            classes, A = new(rows, P.C), new(rows, P.C)
            pred, B = new(nb, P.C), new(nb, P.C, P.D)
            crit = torch.empty(nb, P.C, dtype=torch.int64, device=dev)
            sQ, sH = new(rows, Q_DIM), new(rows, Q_DIM)
            xs = slots.data_ptr() + 4 * max_rows * P.D * torch.arange(nb, dtype=torch.int64, device=dev)
            ws = _workspace(lib.dsmil_forward_bags_train_dev_workspace_bytes(P.ref, nb, max_rows), dev)
            rc = lib.dsmil_forward_bags_train_dev(P.ref, _ptr(xs), _ptr(Ns), nb, max_rows, _ptr(classes), _ptr(pred),
                                                  _ptr(A), _ptr(B), _ptr(crit), _ptr(sQ), _ptr(sH), _ptr(status),
                                                  _ptr(ws), ws.numel(), _stream())
            _lib.check(rc, "dsmil_forward_bags_train_dev")
        ctx.save_for_backward(xs, Ns, status, sQ, sH, A, B, crit, *P.tensors)
        ctx.shape = (nb, max_rows)
        ctx.mark_non_differentiable(crit)
        return classes, pred, A, B, crit

    @staticmethod
    def backward(ctx, g_classes, g_pred, g_A, g_B, _g_crit):
        if ctx.needs_input_grad[0] or g_A is not None or g_B is not None:
            raise NotImplementedError("the graph-captured training step takes gradients through the instance scores "
                                      "and the bag prediction only (no gradient to A, B or the features)")
        lib = _lib.load()
        xs, Ns, status, sQ, sH, A, B, crit, *params = ctx.saved_tensors
        P = ParamPack(*params)
        nb, max_rows = ctx.shape
        names = ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf")
        dev = P.device
        with torch.cuda.device(dev):
            out = {nm: (torch.empty_like(t) if t is not None and need else None)
                   for nm, t, need in zip(names, P.tensors, ctx.needs_input_grad[3:])}
            G = _lib.DsmilGrads(*[_ptr(out[n]) for n in names], None)
            dc, dp = _f32c(g_classes), _f32c(g_pred)
            ws = _workspace(lib.dsmil_backward_bags_dev_workspace_bytes(P.ref, nb, max_rows), dev)
            rc = lib.dsmil_backward_bags_dev(P.ref, _ptr(xs), _ptr(Ns), nb, max_rows, _ptr(sQ), _ptr(sH), _ptr(A),
                                             _ptr(B), _ptr(crit), _ptr(dc), _ptr(dp), None, None, C.byref(G),
                                             _ptr(status), _ptr(ws), ws.numel(), _stream())
            _lib.check(rc, "dsmil_backward_bags_dev")
        return (None, None, None, *[out[n] for n in names])


def mil_forward_bags(bags: Sequence[torch.Tensor], params: Sequence[Optional[torch.Tensor]], *, grad: bool = False):
    """Forward of a STREAM of bags in one library call: returns a lazy sequence of (classes, prediction_bag, A, B)
    per bag -- views into packed device buffers -- plus crit_idx [nb, C] (rows within each bag).

    grad=False (default): inference, dsmil_forward_bags under no_grad.  grad=True with grad mode on: the packed
    outputs carry autograd history (MILBagsFn), so a loss over them trains the whole batch with one backward call;
    identity v only."""
    if not (grad and torch.is_grad_enabled()):
        return _mil_forward_bags_infer(bags, params)
    if len(bags) == 0:
        return [], None
    classes, pred, A, B, crit = MILBagsFn.apply(len(bags), *bags, *params)
    return BagOutputs(classes, pred, A, B, [int(b.shape[0]) for b in bags], crit), crit


@torch.no_grad()
def _mil_forward_bags_infer(bags: Sequence[torch.Tensor], params: Sequence[Optional[torch.Tensor]]):
    lib = _lib.load()
    P = ParamPack(*params)
    if P.passing_v:
        raise NotImplementedError("forward_bags: passing_v models go through MILNet.forward per bag")
    xs = [_check_feats(b, P.D) for b in bags]
    nb = len(xs)
    if nb == 0:
        return [], None
    Ns = [int(x.shape[0]) for x in xs]
    if min(Ns) == 0:
        raise IndexError("dsmil_b200: empty bag (N == 0) in the batch")
    dev = P.device
    for x in xs:
        if x.device != dev:
            raise RuntimeError(f"dsmil_b200: bag on {x.device} but parameters on {dev}")
    total, Cc, D = sum(Ns), P.C, P.D
    c_N = (C.c_int64 * nb)(*Ns)
    c_X = (C.c_void_p * nb)(*[x.data_ptr() for x in xs])
    with torch.cuda.device(dev):
        new = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
        classes, A = new(total, Cc), new(total, Cc)
        pred, B = new(nb, Cc), new(nb, Cc, D)
        crit = torch.empty(nb, Cc, dtype=torch.int64, device=dev)
        ws = _workspace(lib.dsmil_forward_bags_workspace_bytes(P.ref, c_N, nb), dev)
        rc = lib.dsmil_forward_bags(P.ref, c_X, c_N, nb, _ptr(classes), _ptr(pred), _ptr(A), _ptr(B), _ptr(crit),
                                    _ptr(ws), ws.numel(), _stream())
        _lib.check(rc, "dsmil_forward_bags")
    return BagOutputs(classes, pred, A, B, Ns), crit
