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


def _warm_up(dev, steps, run):
    """`run` `steps` times on a side stream, as torch.cuda.graph asks before a capture."""
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(max(1, steps)):
            run()
    torch.cuda.current_stream(dev).wait_stream(side)


def _workspace(nbytes: int, device) -> torch.Tensor:
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)


def _check_feats(feats: torch.Tensor, D: int) -> torch.Tensor:
    require_cuda(feats, "the bag (feats)")
    if feats.dim() != 2 or feats.shape[1] != D:
        raise ValueError(f"feats must be [N, {D}], got {tuple(feats.shape)}")
    return _f32c(feats)


PARAM_NAMES = ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf")


def _bag_outputs(P: ParamPack, rows: int, nb: int, lead=()):
    """Empty packed outputs of a bag call on P's device: classes and A [*lead, rows, C], pred [*lead, nb, C],
    B [*lead, nb, C, D] and crit [*lead, nb, C] int64."""
    new = lambda *s: torch.empty(*lead, *s, dtype=torch.float32, device=P.device)
    return (new(rows, P.C), new(nb, P.C), new(rows, P.C), new(nb, P.C, P.D),
            torch.empty(*lead, nb, P.C, dtype=torch.int64, device=P.device))


def _saves(P: ParamPack, rows: int):
    """Empty activations that a forward saves for its backward: Q [rows, 128], H1 [rows, 128] for a nonlinear q and
    V [rows, D] for passing_v (None where the model has none)."""
    new = lambda *s: torch.empty(*s, dtype=torch.float32, device=P.device)
    return new(rows, Q_DIM), new(rows, Q_DIM) if P.nonlinear else None, new(rows, P.D) if P.passing_v else None


def _param_grads(P: ParamPack, needs, gX: Optional[torch.Tensor] = None):
    """Empty gradients of P's parameters where `needs` (one flag per PARAM_NAMES entry) asks for them, None elsewhere,
    and the DsmilGrads over them and gX."""
    out = [torch.empty_like(t) if t is not None and need else None for t, need in zip(P.tensors, needs)]
    return out, _lib.DsmilGrads(*[_ptr(g) for g in out], _ptr(gX))


def _split_rows(gX: Optional[torch.Tensor], Ns, needs):
    """Each bag's rows of a packed feature gradient where `needs` asks for them, None elsewhere."""
    out, lo = [], 0
    for n, need in zip(Ns, needs):
        out.append(gX[lo:lo + n] if need else None)
        lo += n
    return out


def _slot_addrs(slots, P: ParamPack, what: str):
    """The device addresses of the [max_rows, D] slots of a contiguous float32 [nb, max_rows, D] buffer."""
    if slots.dim() != 3 or slots.shape[2] != P.D or slots.dtype != torch.float32 or not slots.is_contiguous():
        raise ValueError(f"{what} must be contiguous float32 [nb, max_rows, {P.D}], got {tuple(slots.shape)}")
    nb, max_rows = int(slots.shape[0]), int(slots.shape[1])
    return slots.data_ptr() + 4 * max_rows * P.D * torch.arange(nb, dtype=torch.int64, device=slots.device)


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
            sQ, sH, sV = _saves(P, N) if need_grad else (None, None, None)
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
        # Wi/bi only get gradient through `classes` in the fused form
        want = [need and (ctx.fused_scores or nm not in ("Wi", "bi")) for nm, need in zip(PARAM_NAMES, needs[4:])]
        with torch.cuda.device(X.device):
            gX = torch.empty_like(X) if needs[0] else None
            out, G = _param_grads(P, want, gX)
            dc = _f32c(g_classes) if (g_classes is not None and ctx.fused_scores) else None
            dp = _f32c(g_pred.reshape(-1)) if g_pred is not None else None
            dA = _f32c(g_A) if g_A is not None else None
            dB = _f32c(g_B.reshape(Cc, D)) if g_B is not None else None
            ws = _workspace(lib.dsmil_backward_workspace_bytes(P.ref, N, int(gX is not None)), X.device)
            rc = lib.dsmil_backward(P.ref, _ptr(X), _ptr(xv), N, _ptr(sQ), _ptr(sH), _ptr(sV), _ptr(A), _ptr(B),
                                    _ptr(crit), _ptr(dc), _ptr(dp), _ptr(dA), _ptr(dB), C.byref(G),
                                    _ptr(v_mask), _ptr(ws), ws.numel(), _stream())
            _lib.check(rc, "dsmil_backward")
        return (None, gX, None, None, None, *out)


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
        total, dev = sum(Ns), P.device
        with torch.cuda.device(dev):
            classes, pred, A, B, crit = _bag_outputs(P, total, nb)
            sQ, sH, _ = _saves(P, total)
            ws = _workspace(lib.dsmil_forward_bags_train_workspace_bytes(P.ref, c_N, nb), dev)
            rc = lib.dsmil_forward_bags_train(P.ref, c_X, c_N, nb, _ptr(classes), _ptr(pred), _ptr(A), _ptr(B),
                                              _ptr(crit), _ptr(sQ), _ptr(sH), _ptr(ws), ws.numel(), _stream())
            _lib.check(rc, "dsmil_forward_bags_train")
        ctx.nb, ctx.Ns, ctx.c_X, ctx.c_N = nb, Ns, c_X, c_N
        ctx.save_for_backward(*xs, sQ, sH, A, B, crit, *P.tensors)
        ctx.mark_non_differentiable(crit)
        return classes, pred, A, B, crit

    @staticmethod
    def backward(ctx, g_classes, g_pred, g_A, g_B, _g_crit):
        lib = _lib.load()
        nb, Ns, c_X, c_N = ctx.nb, ctx.Ns, ctx.c_X, ctx.c_N
        saved = ctx.saved_tensors
        (sQ, sH, A, B, crit), params = saved[nb:nb + 5], saved[nb + 5:]   # saved[:nb]: the bags c_X points at
        P = ParamPack(*params)
        need_bags, need_params = ctx.needs_input_grad[1:1 + nb], ctx.needs_input_grad[1 + nb:]
        dev = P.device
        with torch.cuda.device(dev):
            gX = torch.empty(sum(Ns), P.D, dtype=torch.float32, device=dev) if any(need_bags) else None
            out, G = _param_grads(P, need_params, gX)
            dc, dp, dA, dB = (_f32c(t) for t in (g_classes, g_pred, g_A, g_B))
            ws = _workspace(lib.dsmil_backward_bags_workspace_bytes(P.ref, c_N, nb, int(gX is not None)), dev)
            rc = lib.dsmil_backward_bags(P.ref, c_X, c_N, nb, _ptr(sQ), _ptr(sH), _ptr(A), _ptr(B), _ptr(crit),
                                         _ptr(dc), _ptr(dp), _ptr(dA), _ptr(dB), C.byref(G), _ptr(ws), ws.numel(),
                                         _stream())
            _lib.check(rc, "dsmil_backward_bags")
        return (None, *_split_rows(gX, Ns, need_bags), *out)


def _dev_prefix(lib, P, what):
    """The name prefix of the capture-safe calls that take P's shape: the tensor-core ones, or their generic forms."""
    if lib.dsmil_shard_bags_supported(P.ref):
        return "dsmil_"
    if lib.dsmil_generic_bags_supported(P.ref):
        return "dsmil_generic_"
    raise ValueError(f"{what} takes identity v only; D={P.D}, C={P.C}, nonlinear={P.nonlinear}, "
                     f"passing_v={P.passing_v} is on no batched route")


class MILBagsDevFn(torch.autograd.Function):
    """MILBagsFn over the capture-safe entry points (dsmil_forward_bags_train_dev / dsmil_backward_bags_dev): the bag
    list lives on the device, so one recorded call serves every batch of nb bags of 1..max_rows rows.

    args: slots [nb, max_rows, D] (bag b is slots[b, :Ns[b]]), Ns [nb] int64 and status [1] int32 on the device, then
    the ten parameter tensors.  The packed per-row outputs (classes, A) have nb * max_rows rows; the live ones are
    packed at the prefix sums of Ns, as MILBagsFn packs them.  Parameter gradients only (no gradient to the slots).
    The tensor-core shapes call the dev entry points; the other identity-v shapes their dsmil_generic_* forms."""

    @staticmethod
    def forward(ctx, slots, Ns, status, *params):
        lib = _lib.load()
        ctx.set_materialize_grads(False)
        P = ParamPack(*params)
        pre = _dev_prefix(lib, P, "graph-captured training")
        xs = _slot_addrs(slots, P, "slots")
        nb, max_rows = int(slots.shape[0]), int(slots.shape[1])
        dev = P.device
        with torch.cuda.device(dev):
            rows = nb * max_rows
            classes, pred, A, B, crit = _bag_outputs(P, rows, nb)
            sQ, sH, _ = _saves(P, rows)
            ws = _workspace(getattr(lib, pre + "forward_bags_train_dev_workspace_bytes")(P.ref, nb, max_rows), dev)
            call = getattr(lib, pre + "forward_bags_train_dev")
            rc = call(P.ref, _ptr(xs), _ptr(Ns), nb, max_rows, _ptr(classes), _ptr(pred), _ptr(A), _ptr(B), _ptr(crit),
                      _ptr(sQ), _ptr(sH), _ptr(status), _ptr(ws), ws.numel(), _stream())
            _lib.check(rc, pre + "forward_bags_train_dev")
        ctx.save_for_backward(xs, Ns, status, sQ, sH, A, B, crit, *P.tensors)
        ctx.shape, ctx.pre = (nb, max_rows), pre
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
        dev = P.device
        with torch.cuda.device(dev):
            out, G = _param_grads(P, ctx.needs_input_grad[3:])
            dc, dp = _f32c(g_classes), _f32c(g_pred)
            ws = _workspace(getattr(lib, ctx.pre + "backward_bags_dev_workspace_bytes")(P.ref, nb, max_rows), dev)
            call = getattr(lib, ctx.pre + "backward_bags_dev")
            rc = call(P.ref, _ptr(xs), _ptr(Ns), nb, max_rows, _ptr(sQ), _ptr(sH), _ptr(A), _ptr(B), _ptr(crit),
                      _ptr(dc), _ptr(dp), None, None, C.byref(G), _ptr(status), _ptr(ws), ws.numel(), _stream())
            _lib.check(rc, ctx.pre + "backward_bags_dev")
        return (None, None, None, *out)


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
def mil_forward_bags_dev(xs: torch.Tensor, Ns: torch.Tensor, status: torch.Tensor, max_rows: int,
                         params: Sequence[Optional[torch.Tensor]]):
    """Inference over a bag list held on the device (dsmil_forward_bags_dev), with no host work that depends on the
    bags: one call can be recorded into a CUDA graph and replayed over every batch of nb bags of 1..max_rows rows.

    xs [nb] int64 (the bags' feature addresses: contiguous float32 [N_b, D]), Ns [nb] int64 and status [1] int32 on
    the device.  Returns the packed (classes, pred, A, B, crit): classes and A have nb * max_rows rows, the live ones
    packed at the prefix sums of Ns, as dsmil_forward_bags packs them.  A refused batch sets status (see the header).
    The shapes off the tensor-core batch call dsmil_generic_forward_bags_dev."""
    lib = _lib.load()
    P = ParamPack(*params)
    pre = _dev_prefix(lib, P, "the device bag list")
    return _infer_bags_dev(P, pre + "forward_bags_dev", xs, None, Ns, status, max_rows)


def _infer_bags_dev(P: ParamPack, call: str, xs, vs, Ns, status, max_rows: int):
    """The body of mil_forward_bags_dev and mil_forward_value_bags_dev: one capture-safe forward `call` without saves.
    A passing_v model's call also takes the value inputs' addresses vs (None: the features) and the NULL saves."""
    lib = _lib.load()
    nb, dev = int(xs.numel()), P.device
    value, saves = ((_ptr(vs),), (None, None, None)) if P.passing_v else ((), ())
    with torch.cuda.device(dev):
        classes, pred, A, B, crit = _bag_outputs(P, nb * max_rows, nb)
        ws = _workspace(getattr(lib, call + "_workspace_bytes")(P.ref, nb, max_rows), dev)
        rc = getattr(lib, call)(P.ref, _ptr(xs), *value, _ptr(Ns), nb, max_rows, _ptr(classes), _ptr(pred), _ptr(A),
                                _ptr(B), _ptr(crit), *saves, _ptr(status), _ptr(ws), ws.numel(), _stream())
        _lib.check(rc, call)
    return classes, pred, A, B, crit


MAX_MODELS = 8   # members of one dsmil_forward_bags_models call


def _model_packs(params_list) -> list:
    """ParamPacks of an ensemble's members: 1 to MAX_MODELS of them, with the same D, C and q form, identity v, on one
    device; ValueError naming the first mismatch."""
    packs = [ParamPack(*p) for p in params_list]
    M = len(packs)
    if not 1 <= M <= MAX_MODELS:
        raise ValueError(f"an ensemble forward takes 1 to {MAX_MODELS} models, got {M}")
    P0 = packs[0]
    for m, P in enumerate(packs[1:], 1):
        for what in ("D", "C", "nonlinear", "passing_v"):
            if getattr(P, what) != getattr(P0, what):
                raise ValueError(f"model {m}: {what}={getattr(P, what)} differs from model 0's {getattr(P0, what)}")
        if P.device != P0.device:
            raise ValueError(f"model {m} is on {P.device}, model 0 on {P0.device}")
    if P0.passing_v:
        raise NotImplementedError("forward_bags: passing_v models go through MILNet.forward per bag")
    return packs


class MILBagsModelsFn(torch.autograd.Function):
    """MILBagsFn for M members, each over its own bags: dsmil_forward_bags_models_train forward and
    dsmil_backward_bags_models backward, one call each for all members.  args: nbs (each member's bag count), the
    sum(nbs) bags (member 0's, then member 1's, ...), then the M members' ten parameter tensors each.  The packed
    outputs are model-major; member m's parameter gradients are sums over its own bags."""

    @staticmethod
    def forward(ctx, nbs, *args):
        lib = _lib.load()
        ctx.set_materialize_grads(False)
        M, ne = len(nbs), sum(nbs)
        packs = _model_packs([args[ne + 10 * m:ne + 10 * (m + 1)] for m in range(M)])
        P0 = packs[0]
        xs, Ns, c_X, c_N = _bag_table(args[:ne], P0)
        total, dev = sum(Ns), P0.device
        ps = (_lib.DsmilParams * M)(*[P.struct for P in packs])
        c_nb = (C.c_int32 * M)(*nbs)
        with torch.cuda.device(dev):
            classes, pred, A, B, crit = _bag_outputs(P0, total, ne)
            sQ, sH, _ = _saves(P0, total)
            ws = _workspace(lib.dsmil_forward_bags_models_train_workspace_bytes(ps, M, c_N, c_nb), dev)
            rc = lib.dsmil_forward_bags_models_train(ps, M, c_X, c_N, c_nb, _ptr(classes), _ptr(pred), _ptr(A),
                                                     _ptr(B), _ptr(crit), _ptr(sQ), _ptr(sH), _ptr(ws), ws.numel(),
                                                     _stream())
            _lib.check(rc, "dsmil_forward_bags_models_train")
        ctx.nbs, ctx.Ns = tuple(nbs), Ns
        ctx.save_for_backward(*xs, sQ, sH, A, B, crit, *[t for P in packs for t in P.tensors])
        ctx.mark_non_differentiable(crit)
        return classes, pred, A, B, crit

    @staticmethod
    def backward(ctx, g_classes, g_pred, g_A, g_B, _g_crit):
        lib = _lib.load()
        nbs, Ns = ctx.nbs, ctx.Ns
        M, ne = len(nbs), sum(nbs)
        saved = ctx.saved_tensors
        xs, (sQ, sH, A, B, crit) = saved[:ne], saved[ne:ne + 5]
        packs = [ParamPack(*saved[ne + 5 + 10 * m:ne + 5 + 10 * (m + 1)]) for m in range(M)]
        need_bags, need_params = ctx.needs_input_grad[1:1 + ne], ctx.needs_input_grad[1 + ne:]
        P0, dev = packs[0], packs[0].device
        c_X = (C.c_void_p * ne)(*[x.data_ptr() for x in xs])
        c_N = (C.c_int64 * ne)(*Ns)
        c_nb = (C.c_int32 * M)(*nbs)
        ps = (_lib.DsmilParams * M)(*[P.struct for P in packs])
        with torch.cuda.device(dev):
            gX = torch.empty(sum(Ns), P0.D, dtype=torch.float32, device=dev) if any(need_bags) else None
            outs, grads, lo, b = [], (_lib.DsmilGrads * M)(), 0, 0
            for m, P in enumerate(packs):
                rows = sum(Ns[b:b + nbs[m]])
                out, grads[m] = _param_grads(P, need_params[10 * m:10 * (m + 1)],
                                             None if gX is None else gX[lo:lo + rows])
                outs += out
                lo, b = lo + rows, b + nbs[m]
            dc, dp, dA, dB = (_f32c(t) for t in (g_classes, g_pred, g_A, g_B))
            ws = _workspace(lib.dsmil_backward_bags_models_workspace_bytes(ps, M, c_N, c_nb, int(gX is not None)),
                            dev)
            rc = lib.dsmil_backward_bags_models(ps, M, c_X, c_N, c_nb, _ptr(sQ), _ptr(sH), _ptr(A), _ptr(B),
                                                _ptr(crit), _ptr(dc), _ptr(dp), _ptr(dA), _ptr(dB), grads, _ptr(ws),
                                                ws.numel(), _stream())
            _lib.check(rc, "dsmil_backward_bags_models")
        return (None, *_split_rows(gX, Ns, need_bags), *outs)


def _fold_packs(pre, nbs, params, what="the graph-captured fold step"):
    """The M members' ParamPacks and their DsmilParams array for the fold dev calls of prefix pre ("dsmil_": the fused
    tensor-core fold shapes, "dsmil_generic_": the generic ones); ValueError off them."""
    lib = _lib.load()
    M = len(nbs)
    packs = _model_packs([params[10 * m:10 * (m + 1)] for m in range(M)])
    P0 = packs[0]
    ps = (_lib.DsmilParams * M)(*[P.struct for P in packs])
    if pre == "dsmil_":
        if min(nbs) < 1 or not lib.dsmil_models_supported(ps, M):
            raise ValueError(f"{what} runs on the fused fold shapes only; M={M}, D={P0.D}, "
                             f"C={P0.C}, nonlinear={P0.nonlinear}, group sizes {tuple(nbs)} are not on them")
    elif min(nbs) < 1 or not lib.dsmil_generic_models_supported(ps, M):
        raise ValueError(f"the generic {what.removeprefix('the ')} runs on the generic batched shapes only; M={M}, "
                         f"D={P0.D}, C={P0.C}, nonlinear={P0.nonlinear}, group sizes {tuple(nbs)} are not on them")
    return packs, ps


def _models_dev_forward(ctx, pre, nbs, slots, Ns, status, params):
    """The body of MILBagsModelsDevFn.forward over the fold dev calls named pre + "forward_bags_models_train_dev"."""
    lib = _lib.load()
    ctx.set_materialize_grads(False)
    M, ne = len(nbs), sum(nbs)
    packs, ps = _fold_packs(pre, nbs, params)
    P0 = packs[0]
    if slots.dim() != 3 or slots.shape[0] != ne or slots.shape[2] != P0.D or slots.dtype != torch.float32 \
            or not slots.is_contiguous():
        raise ValueError(f"slots must be contiguous float32 [{ne}, max_rows, {P0.D}], got {tuple(slots.shape)}")
    xs = _slot_addrs(slots, P0, "slots")
    max_rows, dev = int(slots.shape[1]), P0.device
    c_nb = (C.c_int32 * M)(*nbs)
    call = pre + "forward_bags_models_train_dev"
    with torch.cuda.device(dev):
        rows = ne * max_rows
        classes, pred, A, B, crit = _bag_outputs(P0, rows, ne)
        sQ, sH, _ = _saves(P0, rows)
        ws = _workspace(getattr(lib, call + "_workspace_bytes")(ps, M, c_nb, max_rows), dev)
        rc = getattr(lib, call)(ps, M, _ptr(xs), _ptr(Ns), c_nb, max_rows, _ptr(classes), _ptr(pred), _ptr(A),
                                _ptr(B), _ptr(crit), _ptr(sQ), _ptr(sH), _ptr(status), _ptr(ws), ws.numel(),
                                _stream())
        _lib.check(rc, call)
    ctx.save_for_backward(xs, Ns, status, sQ, sH, A, B, crit, *[t for P in packs for t in P.tensors])
    ctx.nbs, ctx.max_rows, ctx.pre = tuple(nbs), max_rows, pre
    ctx.mark_non_differentiable(crit)
    return classes, pred, A, B, crit


def _models_dev_backward(ctx, g_classes, g_pred, g_A, g_B):
    """The body of MILBagsModelsDevFn.backward over the fold dev calls of the forward's prefix."""
    if ctx.needs_input_grad[1] or g_A is not None or g_B is not None:
        raise NotImplementedError("the graph-captured fold step takes gradients through the instance scores "
                                  "and the bag prediction only (no gradient to A, B or the features)")
    lib = _lib.load()
    xs, Ns, status, sQ, sH, A, B, crit, *params = ctx.saved_tensors
    nbs, max_rows = ctx.nbs, ctx.max_rows
    M = len(nbs)
    packs = [ParamPack(*params[10 * m:10 * (m + 1)]) for m in range(M)]
    dev = packs[0].device
    ps = (_lib.DsmilParams * M)(*[P.struct for P in packs])
    c_nb = (C.c_int32 * M)(*nbs)
    need = ctx.needs_input_grad[4:]
    call = ctx.pre + "backward_bags_models_dev"
    with torch.cuda.device(dev):
        outs, grads = zip(*[_param_grads(P, need[10 * m:10 * (m + 1)]) for m, P in enumerate(packs)])
        grads = (_lib.DsmilGrads * M)(*grads)
        dc, dp = _f32c(g_classes), _f32c(g_pred)
        ws = _workspace(getattr(lib, call + "_workspace_bytes")(ps, M, c_nb, max_rows), dev)
        rc = getattr(lib, call)(ps, M, _ptr(xs), _ptr(Ns), c_nb, max_rows, _ptr(sQ), _ptr(sH), _ptr(A), _ptr(B),
                                _ptr(crit), _ptr(dc), _ptr(dp), None, None, grads, _ptr(status), _ptr(ws),
                                ws.numel(), _stream())
        _lib.check(rc, call)
    return (None, None, None, None, *[g for out in outs for g in out])


class MILBagsModelsDevFn(torch.autograd.Function):
    """MILBagsModelsFn over the capture-safe entry points (dsmil_forward_bags_models_train_dev /
    dsmil_backward_bags_models_dev): every member's bag list lives on the device, so one recorded call serves every
    step of the same group sizes.

    args: nbs (each member's bag count), slots [sum(nbs), max_rows, D] (member-major; bag e is slots[e, :Ns[e]]),
    Ns [sum(nbs)] int64 and status [M] int32 on the device, then the M members' ten parameter tensors each.  The
    packed per-row outputs (classes, A) have sum(nbs) * max_rows rows: member m's block starts at row
    max_rows * sum(nbs[:m]) and packs its live rows at the prefix sums of its own Ns.  Parameter gradients only."""

    @staticmethod
    def forward(ctx, nbs, slots, Ns, status, *params):
        return _models_dev_forward(ctx, "dsmil_", nbs, slots, Ns, status, params)

    @staticmethod
    def backward(ctx, g_classes, g_pred, g_A, g_B, _g_crit):
        return _models_dev_backward(ctx, g_classes, g_pred, g_A, g_B)


class MILBagsModelsGenericDevFn(torch.autograd.Function):
    """MILBagsModelsDevFn on the generic shapes (dsmil_generic_models_supported: e.g. the classic-MIL D = 166 / 230, a
    linear q, C > 4, D > 2048): the same arguments and outputs over dsmil_generic_forward_bags_models_train_dev /
    dsmil_generic_backward_bags_models_dev, member m's slices bit for bit those of MILBagsDevFn on its bags alone."""

    @staticmethod
    def forward(ctx, nbs, slots, Ns, status, *params):
        return _models_dev_forward(ctx, "dsmil_generic_", nbs, slots, Ns, status, params)

    @staticmethod
    def backward(ctx, g_classes, g_pred, g_A, g_B, _g_crit):
        return _models_dev_backward(ctx, g_classes, g_pred, g_A, g_B)


@torch.no_grad()
def mil_forward_bags_models_dev(nbs: Sequence[int], xs: torch.Tensor, Ns: torch.Tensor, status: torch.Tensor,
                                max_rows: int, params_list: Sequence[Sequence[Optional[torch.Tensor]]],
                                generic: bool = False):
    """Inference of M members, each over its OWN bag list held on the device (dsmil_forward_bags_models_dev): the fold
    models' validation, with no host work that depends on the bags, so one call can be recorded into a CUDA graph and
    replayed over every batch of the same group sizes.

    nbs: each member's bag count (host); xs [sum nbs] int64 (the bags' feature addresses, member-major), Ns [sum nbs]
    int64 and status [M] int32 on the device.  Returns the packed (classes, pred, A, B, crit): classes and A have
    sum(nbs) * max_rows rows, member m's block starting at row max_rows * sum(nbs[:m]) with its live rows packed at the
    prefix sums of its own Ns; pred, B and crit are [sum nbs, ...].  Member m's slices are bit for bit those of
    mil_forward_bags_dev on its bags alone.  A member with a refused bag sets status[m] (see the header) and only its
    slices are a stand-in.  generic=True: the generic fold shapes (dsmil_generic_forward_bags_models_dev)."""
    nbs = tuple(int(n) for n in nbs)
    pre = "dsmil_generic_" if generic else "dsmil_"
    packs, ps = _fold_packs(pre, nbs, [t for p in params_list for t in p], "the fold models' inference")
    M, ne, P0 = len(nbs), sum(nbs), packs[0]
    if xs.numel() != ne or Ns.numel() != ne or status.numel() != M:
        raise ValueError(f"xs and Ns need {ne} entries and status {M}; got {xs.numel()}, {Ns.numel()} and "
                         f"{status.numel()}")
    lib = _lib.load()
    c_nb = (C.c_int32 * M)(*nbs)
    call = pre + "forward_bags_models_dev"
    with torch.cuda.device(P0.device):
        classes, pred, A, B, crit = _bag_outputs(P0, ne * max_rows, ne)
        ws = _workspace(getattr(lib, call + "_workspace_bytes")(ps, M, c_nb, max_rows), P0.device)
        rc = getattr(lib, call)(ps, M, _ptr(xs), _ptr(Ns), c_nb, max_rows, _ptr(classes), _ptr(pred), _ptr(A),
                                _ptr(B), _ptr(crit), _ptr(status), _ptr(ws), ws.numel(), _stream())
        _lib.check(rc, call)
    return classes, pred, A, B, crit


def mil_forward_bags_per_model(bag_lists: Sequence[Sequence[torch.Tensor]],
                               params_list: Sequence[Sequence[Optional[torch.Tensor]]], *, grad: bool = False):
    """M parameter sets (1 <= M <= 8, the same D, C and q form, identity v), each over its OWN non-empty list of bags,
    in one dsmil_forward_bags_models_train call.  Returns M BagOutputs over model-major packed tensors, each with
    `.crit`; model m's are bit for bit what mil_forward_bags(bag_lists[m], params_list[m], grad=True) gives.

    grad=True with grad mode on: the packed outputs carry autograd history (MILBagsModelsFn), and one backward over a
    loss of every member's outputs fills every member's gradients with one dsmil_backward_bags_models call."""
    M = len(bag_lists)
    if not 1 <= M <= MAX_MODELS:
        raise ValueError(f"an ensemble forward takes 1 to {MAX_MODELS} models, got {M}")
    if M != len(params_list):
        raise ValueError(f"{M} bag lists for {len(params_list)} parameter sets")
    for m, bags in enumerate(bag_lists):
        if len(bags) == 0:
            raise ValueError(f"model {m} has no bags: every member of a fold step needs at least one")
    nbs = tuple(len(bags) for bags in bag_lists)
    flat = [b for bags in bag_lists for b in bags]
    params = [t for p in params_list for t in p]
    with torch.set_grad_enabled(grad and torch.is_grad_enabled()):
        classes, pred, A, B, crit = MILBagsModelsFn.apply(nbs, *flat, *params)
    outs, row, b = [], 0, 0
    for bags in bag_lists:
        Ns = [int(x.shape[0]) for x in bags]
        rows, nb = sum(Ns), len(bags)
        outs.append(BagOutputs(classes[row:row + rows], pred[b:b + nb], A[row:row + rows], B[b:b + nb], Ns,
                               crit[b:b + nb]))
        row, b = row + rows, b + nb
    return outs


@torch.no_grad()
def mil_forward_bags_models(bags: Sequence[torch.Tensor], params_list: Sequence[Sequence[Optional[torch.Tensor]]]):
    """An ensemble forward: M parameter sets (1 <= M <= 8, the same D, C and q form, identity v) over the same bags in
    one dsmil_forward_bags_models call.  Returns M BagOutputs, one per model, over model-major packed tensors, each
    with `.crit` [nb, C]; model m's are bit for bit what mil_forward_bags(bags, params_list[m]) gives.  On the batched
    tensor-core shapes the whole ensemble costs one launch of each kernel and the passes over a bag follow each
    other while it is in L2."""
    lib = _lib.load()
    packs = _model_packs(params_list)
    M, P0 = len(packs), packs[0]
    nb = len(bags)
    if nb == 0:
        return [BagOutputs(None, None, None, None, [], None) for _ in range(M)]
    xs, Ns, c_X, c_N = _bag_table(bags, P0)
    dev = P0.device
    ps = (_lib.DsmilParams * M)(*[P.struct for P in packs])
    with torch.cuda.device(dev):
        classes, pred, A, B, crit = _bag_outputs(P0, sum(Ns), nb, lead=(M,))
        ws = _workspace(lib.dsmil_forward_bags_models_workspace_bytes(ps, M, c_N, nb), dev)
        rc = lib.dsmil_forward_bags_models(ps, M, c_X, c_N, nb, _ptr(classes), _ptr(pred), _ptr(A), _ptr(B),
                                           _ptr(crit), _ptr(ws), ws.numel(), _stream())
        _lib.check(rc, "dsmil_forward_bags_models")
    return [BagOutputs(classes[m], pred[m], A[m], B[m], Ns, crit[m]) for m in range(M)]


MAX_VALUE_BAGS = 65535   # bags of one dsmil_value_forward_bags / dsmil_value_backward_bags call


def _value_pack(params) -> ParamPack:
    P = ParamPack(*params)
    if not P.passing_v:
        raise ValueError("mil_forward_value_bags takes models with a value network (passing_v); identity v goes "
                         "through mil_forward_bags")
    return P


def _per_bag(vals, xs, P: ParamPack, what: str):
    """Checked, contiguous per-bag tensors shaped like their bags (value inputs or v masks), or None."""
    if vals is None:
        return None
    if len(vals) != len(xs):
        raise ValueError(f"{len(vals)} {what}s for {len(xs)} bags")
    vs = [_check_feats(v, P.D) for v in vals]
    for v, x in zip(vs, xs):
        if v.shape != x.shape or v.device != x.device:
            raise ValueError(f"a {what} {tuple(v.shape)} on {v.device} does not match its bag "
                             f"{tuple(x.shape)} on {x.device}")
    return vs


def _ptr_array(ts):
    return None if ts is None else (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


class MILValueBagsFn(torch.autograd.Function):
    """Packed (classes, pred, A, B, crit) of a batch of bags of a passing_v model, differentiable:
    dsmil_value_forward_bags with saves forward, dsmil_value_backward_bags backward (one call each for the whole
    batch).  args: nb, v_inputs (nb value inputs, or None), v_masks (their nb dropout masks, or None), the nb bags,
    then the ten parameter tensors.  Parameter gradients are sums over the bags, gWv and gbv included; a bag's
    gradient includes the value path, through its mask, so value inputs that are not the bags need their masks when a
    bag gradient is wanted.  The value inputs and masks get no gradient; both are saved for the backward (an in-place
    write to a value input before it fails there, as for any saved tensor)."""

    @staticmethod
    def forward(ctx, nb, v_inputs, v_masks, *args):
        lib = _lib.load()
        ctx.set_materialize_grads(False)
        P = _value_pack(args[nb:])
        xs, Ns, c_X, c_N = _bag_table(args[:nb], P)
        vs, ms = _per_bag(v_inputs, xs, P, "value input"), _per_bag(v_masks, xs, P, "v mask")
        if ms is not None and vs is None:
            raise ValueError("v_masks without v_inputs: the masks are the factors of the value inputs")
        if vs is not None and ms is None and any(ctx.needs_input_grad[3:3 + nb]):
            raise ValueError("the bags' gradients through v_inputs need their v_masks (v_inputs == bags * v_masks)")
        total, dev = sum(Ns), P.device
        with torch.cuda.device(dev):
            classes, pred, A, B, crit = _bag_outputs(P, total, nb)
            sQ, sH, sV = _saves(P, total)
            mask = torch.cat(ms) if ms is not None else None   # packed [sum N, D], as the backward reads it
            ws = _workspace(lib.dsmil_value_forward_bags_workspace_bytes(P.ref, c_N, nb), dev)
            rc = lib.dsmil_value_forward_bags(P.ref, c_X, _ptr_array(vs), c_N, nb, _ptr(classes), _ptr(pred), _ptr(A),
                                              _ptr(B), _ptr(crit), _ptr(sQ), _ptr(sH), _ptr(sV), _ptr(ws),
                                              ws.numel(), _stream())
            _lib.check(rc, "dsmil_value_forward_bags")
        ctx.nb, ctx.Ns, ctx.c_N, ctx.nv = nb, Ns, c_N, 0 if vs is None else nb
        ctx.save_for_backward(*xs, *(vs or ()), mask, sQ, sH, sV, A, B, crit, *P.tensors)
        ctx.mark_non_differentiable(crit)
        return classes, pred, A, B, crit

    @staticmethod
    def backward(ctx, g_classes, g_pred, g_A, g_B, _g_crit):
        lib = _lib.load()
        nb, nv, Ns, c_N = ctx.nb, ctx.nv, ctx.Ns, ctx.c_N
        saved = ctx.saved_tensors
        xs, vs = saved[:nb], saved[nb:nb + nv]
        (mask, sQ, sH, sV, A, B, crit), params = saved[nb + nv:nb + nv + 7], saved[nb + nv + 7:]
        P = ParamPack(*params)
        need_bags, need_params = ctx.needs_input_grad[3:3 + nb], ctx.needs_input_grad[3 + nb:]
        dev = P.device
        with torch.cuda.device(dev):
            gX = torch.empty(sum(Ns), P.D, dtype=torch.float32, device=dev) if any(need_bags) else None
            out, G = _param_grads(P, need_params, gX)
            dc, dp, dA, dB = (_f32c(t) for t in (g_classes, g_pred, g_A, g_B))
            ws = _workspace(lib.dsmil_value_backward_bags_workspace_bytes(P.ref, c_N, nb, int(gX is not None)), dev)
            rc = lib.dsmil_value_backward_bags(P.ref, _ptr_array(xs), _ptr_array(vs or None), c_N, nb, _ptr(sQ),
                                               _ptr(sH), _ptr(sV), _ptr(A), _ptr(B), _ptr(crit), _ptr(dc), _ptr(dp),
                                               _ptr(dA), _ptr(dB), _ptr(mask), C.byref(G), _ptr(ws), ws.numel(),
                                               _stream())
            _lib.check(rc, "dsmil_value_backward_bags")
        return (None, None, None, *_split_rows(gX, Ns, need_bags), *out)


def mil_forward_value_bags(bags: Sequence[torch.Tensor], params: Sequence[Optional[torch.Tensor]],
                           v_inputs: Optional[Sequence[torch.Tensor]] = None, *, grad: bool = False,
                           v_masks: Optional[Sequence[torch.Tensor]] = None):
    """Forward of a stream of bags for a model with a value network (passing_v), in one dsmil_value_forward_bags
    call: returns a lazy sequence of (classes, prediction_bag, A, B) per bag plus crit_idx [nb, C], as
    mil_forward_bags does.  v_inputs: each bag's value input (the features after the dropout mask of dsmil.py:36), or
    None for the features themselves (eval mode, or p = 0).  Every bag's outputs are bit for bit what mil_forward
    gives it alone with the same value input.

    grad=False (default): inference under no_grad.  A batch of more than MAX_VALUE_BAGS bags is split into
    consecutive calls that write into the same packed outputs.
    grad=True with grad mode on: the packed outputs carry autograd history (MILValueBagsFn), and one backward over a
    loss of them runs one dsmil_value_backward_bags call for the whole batch, at most MAX_VALUE_BAGS bags.  v_masks:
    each bag's dropout mask (v_inputs[b] == bags[b] * v_masks[b]), for the value path's share of the bags' gradients,
    required with v_inputs when a bag needs a gradient; None when there is no dropout."""
    if grad and torch.is_grad_enabled():
        nb = len(bags)
        if nb > MAX_VALUE_BAGS:
            raise ValueError(f"a differentiable value batch takes at most {MAX_VALUE_BAGS} bags, got {nb}")
        _value_pack(params)   # identity v is refused before any work
        if nb == 0:
            return [], None
        classes, pred, A, B, crit = MILValueBagsFn.apply(nb, v_inputs, v_masks, *bags, *params)
        return BagOutputs(classes, pred, A, B, [int(b.shape[0]) for b in bags], crit), crit
    return _mil_forward_value_bags_infer(bags, params, v_inputs)


class MILValueBagsDevFn(torch.autograd.Function):
    """MILValueBagsFn over the capture-safe value calls (dsmil_value_forward_bags_dev / dsmil_value_backward_bags_dev),
    as MILBagsDevFn is MILBagsFn's: the bag list lives on the device, so one recorded call serves every batch of nb
    bags of 1..max_rows rows, with the eager calls' bits.

    args: slots [nb, max_rows, D] (bag b is slots[b, :Ns[b]]), v_slots (the value inputs in the same layout, value
    input b is v_slots[b, :Ns[b]]; None: the value inputs are the bags), Ns [nb] int64 and status [1] int32 on the
    device, then the ten parameter tensors of a passing_v model.  The packed per-row outputs (classes, A) have
    nb * max_rows rows, the live ones packed at the prefix sums of Ns.  Parameter gradients only (no gradient to the
    slots), so no v mask is needed."""

    @staticmethod
    def forward(ctx, slots, v_slots, Ns, status, *params):
        lib = _lib.load()
        ctx.set_materialize_grads(False)
        P = _value_pack(params)
        xs = _slot_addrs(slots, P, "slots")
        nb, max_rows = int(slots.shape[0]), int(slots.shape[1])
        xvs = None
        if v_slots is not None:
            if v_slots.shape != slots.shape:
                raise ValueError(f"v_slots {tuple(v_slots.shape)} do not match the slots {tuple(slots.shape)}")
            xvs = _slot_addrs(v_slots, P, "v_slots")
        dev = P.device
        with torch.cuda.device(dev):
            rows = nb * max_rows
            classes, pred, A, B, crit = _bag_outputs(P, rows, nb)
            sQ, sH, sV = _saves(P, rows)
            ws = _workspace(lib.dsmil_value_forward_bags_dev_workspace_bytes(P.ref, nb, max_rows), dev)
            rc = lib.dsmil_value_forward_bags_dev(P.ref, _ptr(xs), _ptr(xvs), _ptr(Ns), nb, max_rows, _ptr(classes),
                                                  _ptr(pred), _ptr(A), _ptr(B), _ptr(crit), _ptr(sQ), _ptr(sH),
                                                  _ptr(sV), _ptr(status), _ptr(ws), ws.numel(), _stream())
            _lib.check(rc, "dsmil_value_forward_bags_dev")
        ctx.save_for_backward(xs, xvs, Ns, status, sQ, sH, sV, A, B, crit, *P.tensors)
        ctx.shape = (nb, max_rows)
        ctx.mark_non_differentiable(crit)
        return classes, pred, A, B, crit

    @staticmethod
    def backward(ctx, g_classes, g_pred, g_A, g_B, _g_crit):
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1] or g_A is not None or g_B is not None:
            raise NotImplementedError("the graph-captured value step takes gradients through the instance scores and "
                                      "the bag prediction only (no gradient to A, B, the features or value inputs)")
        lib = _lib.load()
        xs, xvs, Ns, status, sQ, sH, sV, A, B, crit, *params = ctx.saved_tensors
        P = ParamPack(*params)
        nb, max_rows = ctx.shape
        dev = P.device
        with torch.cuda.device(dev):
            out, G = _param_grads(P, ctx.needs_input_grad[4:])
            dc, dp = _f32c(g_classes), _f32c(g_pred)
            ws = _workspace(lib.dsmil_value_backward_bags_dev_workspace_bytes(P.ref, nb, max_rows), dev)
            rc = lib.dsmil_value_backward_bags_dev(P.ref, _ptr(xs), _ptr(xvs), _ptr(Ns), nb, max_rows, _ptr(sQ),
                                                   _ptr(sH), _ptr(sV), _ptr(A), _ptr(B), _ptr(crit), _ptr(dc),
                                                   _ptr(dp), None, None, C.byref(G), _ptr(status), _ptr(ws),
                                                   ws.numel(), _stream())
            _lib.check(rc, "dsmil_value_backward_bags_dev")
        return (None, None, None, None, *out)


@torch.no_grad()
def mil_forward_value_bags_dev(xs: torch.Tensor, vs: Optional[torch.Tensor], Ns: torch.Tensor, status: torch.Tensor,
                               max_rows: int, params: Sequence[Optional[torch.Tensor]]):
    """Inference of a passing_v model over a bag list held on the device (dsmil_value_forward_bags_dev), as
    mil_forward_bags_dev is for identity v: one call can be recorded into a CUDA graph and replayed over every batch
    of nb bags of 1..max_rows rows.  xs [nb] int64 (the bags' feature addresses), vs [nb] int64 (their value inputs'
    addresses, or None: the value inputs are the features), Ns [nb] int64 and status [1] int32 on the device.  Returns
    the packed (classes, pred, A, B, crit) with nb * max_rows rows of classes and A."""
    return _infer_bags_dev(_value_pack(params), "dsmil_value_forward_bags_dev", xs, vs, Ns, status, max_rows)


@torch.no_grad()
def _mil_forward_value_bags_infer(bags, params, v_inputs):
    lib = _lib.load()
    P = _value_pack(params)
    nb = len(bags)
    if nb == 0:
        return [], None
    xs, Ns, _, _ = _bag_table(bags, P)
    vs = _per_bag(v_inputs, xs, P, "value input")
    dev = P.device
    with torch.cuda.device(dev):
        classes, pred, A, B, crit = _bag_outputs(P, sum(Ns), nb)
        row = 0
        for s in range(0, nb, MAX_VALUE_BAGS):
            e = min(s + MAX_VALUE_BAGS, nb)
            n, rows = e - s, sum(Ns[s:e])
            c_X = (C.c_void_p * n)(*[x.data_ptr() for x in xs[s:e]])
            c_V = None if vs is None else (C.c_void_p * n)(*[v.data_ptr() for v in vs[s:e]])
            c_N = (C.c_int64 * n)(*Ns[s:e])
            ws = _workspace(lib.dsmil_value_forward_bags_workspace_bytes(P.ref, c_N, n), dev)
            rc = lib.dsmil_value_forward_bags(P.ref, c_X, c_V, c_N, n, _ptr(classes[row:]), _ptr(pred[s:]),
                                              _ptr(A[row:]), _ptr(B[s:]), _ptr(crit[s:]), None, None, None, _ptr(ws),
                                              ws.numel(), _stream())
            _lib.check(rc, "dsmil_value_forward_bags")
            row += rows
    return BagOutputs(classes, pred, A, B, Ns, crit), crit


@torch.no_grad()
def _mil_forward_bags_infer(bags: Sequence[torch.Tensor], params: Sequence[Optional[torch.Tensor]]):
    lib = _lib.load()
    P = ParamPack(*params)
    if P.passing_v:
        raise NotImplementedError("forward_bags: passing_v models go through MILNet.forward per bag")
    nb = len(bags)
    if nb == 0:
        return [], None
    xs, Ns, c_X, c_N = _bag_table(bags, P)
    dev = P.device
    with torch.cuda.device(dev):
        classes, pred, A, B, crit = _bag_outputs(P, sum(Ns), nb)
        ws = _workspace(lib.dsmil_forward_bags_workspace_bytes(P.ref, c_N, nb), dev)
        rc = lib.dsmil_forward_bags(P.ref, c_X, c_N, nb, _ptr(classes), _ptr(pred), _ptr(A), _ptr(B), _ptr(crit),
                                    _ptr(ws), ws.numel(), _stream())
        _lib.check(rc, "dsmil_forward_bags")
    return BagOutputs(classes, pred, A, B, Ns), crit
