"""Several trained MILNets over the same bags: the fold models of a cross-validation evaluated as one ensemble.

The reference's `5-fold-cv-standalone-test` scheme (train_tcga.py:395-404) runs every fold's best model over the
reserved test bags and takes the mode of their thresholded predictions.  `forward_bags_models` gives each model's
`forward_bags` outputs from one library call (dsmil_forward_bags_models): on the batched tensor-core shapes the M
passes over a bag follow each other while the bag is still in L2.  Thresholds and the vote stay with the caller.
"""
from __future__ import annotations

from typing import List, Sequence

import torch

from . import functional as Fn
from .modules import BClassifier, FCLayer, IClassifier, milnet_params


def _member_params(i, milnet):
    ic, bc = getattr(milnet, "i_classifier", None), getattr(milnet, "b_classifier", None)
    if not (isinstance(bc, BClassifier) and isinstance(ic, (FCLayer, IClassifier))):
        raise TypeError(f"member {i}: an ensemble forward takes MILNets with an FCLayer or IClassifier and a "
                        "BClassifier")
    params = milnet_params(milnet)
    if params[6] is not None:
        raise ValueError(f"member {i}: an ensemble forward takes identity v only (passing_v=False)")
    return params


def _shape(params):
    Wi, W2, Wf = params[0], params[4], params[8]
    return {"D": int(Wf.shape[2]), "C": int(Wf.shape[0]), "nonlinear": W2 is not None}, Wi.device


def _checked_params(milnets):
    """Each member's ten aggregator tensors; ValueError / TypeError naming the first member that does not fit."""
    if not 1 <= len(milnets) <= Fn.MAX_MODELS:
        raise ValueError(f"an ensemble forward takes 1 to {Fn.MAX_MODELS} models, got {len(milnets)}")
    params = [_member_params(i, m) for i, m in enumerate(milnets)]
    shape0, dev0 = _shape(params[0])
    for i, p in enumerate(params[1:], 1):
        shape, dev = _shape(p)
        for what, v in shape.items():
            if v != shape0[what]:
                raise ValueError(f"member {i}: {what}={v} differs from member 0's {what}={shape0[what]}")
        if dev != dev0:
            raise ValueError(f"member {i} is on {dev}, member 0 on {dev0}")
    return params


def forward_bags_per_model(milnets: Sequence[torch.nn.Module], bag_lists: Sequence[Sequence[torch.Tensor]], *,
                           grad: bool = False) -> List[Fn.BagOutputs]:
    """The training form of `forward_bags_models`: member m runs over its OWN bags, bag_lists[m] (at least one), and
    the M members share one library call (dsmil_forward_bags_models_train).  Returns M lazy sequences of per-bag
    (classes, prediction_bag, A, B), each with `.crit`; member m's are bit for bit
    `milnets[m].forward_bags(bag_lists[m], grad=grad)`.  Member checks and errors are those of forward_bags_models.
    grad=True with grad mode on: one backward over a loss of every member's outputs fills every member's gradients
    with one dsmil_backward_bags_models call (the fold models of a cross-validation taking one step together).
    An IClassifier member embeds its own bags first, under autograd when asked."""
    milnets = list(milnets)
    params = _checked_params(milnets)
    if len(bag_lists) != len(milnets):
        raise ValueError(f"{len(bag_lists)} bag lists for {len(milnets)} members")
    for i, bags in enumerate(bag_lists):
        if len(bags) == 0:
            raise ValueError(f"member {i} has no bags: every member of a fold step needs at least one")
    grad = grad and torch.is_grad_enabled()
    with torch.set_grad_enabled(grad):
        feats = [[m.i_classifier.embed(b) for b in bags] if isinstance(m.i_classifier, IClassifier) else list(bags)
                 for m, bags in zip(milnets, bag_lists)]
        return Fn.mil_forward_bags_per_model(feats, params, grad=grad)


@torch.no_grad()
def forward_bags_models(milnets: Sequence[torch.nn.Module], bags: Sequence[torch.Tensor]) -> List[Fn.BagOutputs]:
    """Model m's `milnets[m].forward_bags(bags)` for every member, as M lazy sequences of per-bag
    (classes, prediction_bag, A, B) over model-major packed tensors, each with `.crit` [nb, C].  The members share D,
    C and the q form (nonlinear or not) and live on one device; a mismatch raises ValueError naming it.  Members with
    an FCLayer share one call over the bags; an IClassifier member embeds each bag with its own backbone, and its
    aggregator then runs on those features."""
    milnets = list(milnets)
    params = _checked_params(milnets)
    if not any(isinstance(m.i_classifier, IClassifier) for m in milnets):
        return Fn.mil_forward_bags_models(bags, params)
    outs = []
    for m, p in zip(milnets, params):
        ic = m.i_classifier
        feats = [ic.embed(b) for b in bags] if isinstance(ic, IClassifier) else list(bags)
        outs.append(Fn.mil_forward_bags_models(feats, [p])[0])
    return outs
