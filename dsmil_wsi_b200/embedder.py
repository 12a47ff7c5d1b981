"""Embedder side of the hot path (SURVEY 8f-2): the backbone the reference feeds to `IClassifier` is a torchvision
ResNet built with `norm_layer=nn.InstanceNorm2d` (compute_feats.py:146-170).  The convolutions stay cuDNN library
GEMMs; everything between them -- instance norm, the residual add and the ReLU, which the framework runs as two or three
memory-bound passes per convolution -- goes through ONE kernel of libdsmil_b200.so (`dsmil_instnorm_act`,
csrc/embed_kernels.cuh), in NCHW or in channels-last memory (`dsmil_instnorm_act_nhwc`): `embed.embed_bag`
switches the backbone and its input to channels-last (tools/exp_channels_last.py times both layouts).

    fuse_instance_norm(resnet)   rewires the blocks of a torchvision ResNet in place (parameters, buffers and
                                 state_dict keys untouched, so the reference's embedder checkpoints still load);
                                 inference only -- under autograd the original forward runs.

No CPU path: the fused forward raises on CPU tensors like every other entry point of the package.
"""
from __future__ import annotations

import types

import torch
import torch.nn as nn

from . import _lib
from . import functional as Fn


def _is_channels_last(t: torch.Tensor) -> bool:
    """True NHWC memory (a tensor with C == 1 or H*W == 1 satisfies both layouts and counts as NCHW)."""
    return (not t.is_contiguous()) and t.is_contiguous(memory_format=torch.channels_last)


def instnorm_act(x: torch.Tensor, residual: torch.Tensor | None = None, relu: bool = True, eps: float = 1e-5,
                 out: torch.Tensor | None = None) -> torch.Tensor:
    """y = [relu](instance_norm(x) [+ residual]) for a 4-D fp32 tensor, one kernel.  NCHW-contiguous and
    torch.channels_last inputs each have their own kernel (no layout conversion); the result keeps x's layout.
    `out` may be `x` (in place)."""
    Fn.require_cuda(x, "the activation tensor")
    if x.dtype != torch.float32 or x.dim() != 4:
        raise TypeError(f"instnorm_act wants a 4-D fp32 tensor, got {tuple(x.shape)} {x.dtype}")
    N, Cc, H, W = x.shape
    nhwc = _is_channels_last(x) and Cc % 32 == 0
    fmt = torch.channels_last if nhwc else torch.contiguous_format
    if not nhwc:
        x = x.contiguous()
    if residual is not None:
        if residual.shape != x.shape or residual.dtype != torch.float32:
            raise ValueError("residual must match x")
        residual = residual.contiguous(memory_format=fmt)
    y = torch.empty_like(x, memory_format=fmt) if out is None else out
    if y.shape != x.shape or not y.is_contiguous(memory_format=fmt):
        raise ValueError("out must be a tensor of x's shape and memory layout")
    with torch.cuda.device(x.device):
        lib = _lib.load()
        if nhwc:
            rc = lib.dsmil_instnorm_act_nhwc(x.data_ptr(), Fn._ptr(residual), y.data_ptr(), N, H * W, Cc, float(eps),
                                             int(bool(relu)), Fn._stream())
            _lib.check(rc, "dsmil_instnorm_act_nhwc")
        else:
            rc = lib.dsmil_instnorm_act(x.data_ptr(), Fn._ptr(residual), y.data_ptr(), N * Cc, H * W, float(eps),
                                        int(bool(relu)), Fn._stream())
            _lib.check(rc, "dsmil_instnorm_act")
    return y


def _plain_instance_norm(m) -> bool:
    return (isinstance(m, nn.InstanceNorm2d) and not m.affine and not m.track_running_stats)


def _fusable(*norms) -> bool:
    return all(_plain_instance_norm(n) for n in norms)


def _basic_block_forward(self, x):
    # torchvision.models.resnet.BasicBlock.forward with norm / add / relu fused (dsmil.py:21-25 -> backbone)
    if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
        return self._dsmil_orig_forward(x)
    out = self.conv1(x)
    out = instnorm_act(out, None, True, self.bn1.eps, out=out)
    out = self.conv2(out)
    identity = x
    if self.downsample is not None:
        identity = self._dsmil_downsample(x)
    return instnorm_act(out, identity, True, self.bn2.eps, out=out)


def _bottleneck_forward(self, x):
    if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
        return self._dsmil_orig_forward(x)
    out = self.conv1(x)
    out = instnorm_act(out, None, True, self.bn1.eps, out=out)
    out = self.conv2(out)
    out = instnorm_act(out, None, True, self.bn2.eps, out=out)
    out = self.conv3(out)
    identity = x
    if self.downsample is not None:
        identity = self._dsmil_downsample(x)
    return instnorm_act(out, identity, True, self.bn3.eps, out=out)


def _make_downsample(ds):
    """downsample = Sequential(conv1x1, norm): fuse the norm (no ReLU) when it is a plain InstanceNorm2d."""
    if (isinstance(ds, nn.Sequential) and len(ds) == 2 and isinstance(ds[0], nn.Conv2d) and _plain_instance_norm(ds[1])):
        conv, eps = ds[0], ds[1].eps

        def run(x):
            o = conv(x)
            return instnorm_act(o, None, False, eps, out=o)
        return run
    return ds


def _stem_forward(self, x):
    # torchvision ResNet._forward_impl with the stem's norm + relu fused; the rest is the (re-wired) blocks
    if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
        return self._dsmil_orig_forward(x)
    x = self.conv1(x)
    x = instnorm_act(x, None, True, self.bn1.eps, out=x)
    x = self.maxpool(x)
    x = self.layer1(x)
    x = self.layer2(x)
    x = self.layer3(x)
    x = self.layer4(x)
    x = self.avgpool(x)
    x = torch.flatten(x, 1)
    return self.fc(x)


def fuse_instance_norm(backbone: nn.Module) -> int:
    """Re-wires every torchvision BasicBlock / Bottleneck (and the ResNet stem) whose norm layers are plain
    nn.InstanceNorm2d.  Returns the number of norm layers now running in the fused kernel.  Idempotent."""
    from torchvision.models.resnet import BasicBlock, Bottleneck, ResNet
    fused = 0
    for m in backbone.modules():
        if getattr(m, "_dsmil_fused", False):
            continue
        if isinstance(m, BasicBlock) and _fusable(m.bn1, m.bn2):
            fwd, n = _basic_block_forward, 2
        elif isinstance(m, Bottleneck) and _fusable(m.bn1, m.bn2, m.bn3):
            fwd, n = _bottleneck_forward, 3
        else:
            continue
        m._dsmil_orig_forward = m.forward
        m._dsmil_downsample = _make_downsample(m.downsample) if m.downsample is not None else None
        if m.downsample is not None and m._dsmil_downsample is not m.downsample:
            n += 1
        m.forward = types.MethodType(fwd, m)
        m._dsmil_fused = True
        fused += n
    if isinstance(backbone, ResNet) and not getattr(backbone, "_dsmil_fused", False) and _plain_instance_norm(backbone.bn1):
        backbone._dsmil_orig_forward = backbone.forward
        backbone.forward = types.MethodType(_stem_forward, backbone)
        backbone._dsmil_fused = True
        fused += 1
    return fused
