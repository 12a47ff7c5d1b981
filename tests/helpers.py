"""Test helpers (test infrastructure; may use oracle/)."""
import ctypes

import numpy as np
import torch

from oracle import dsmil_oracle as orc


def state_dict_from_params(p: orc.Params, iclassifier=False):
    t = lambda a: torch.from_numpy(np.array(a, dtype=np.float32))
    ik = "i_classifier.fc." if iclassifier else "i_classifier.fc.0."
    sd = {ik + "weight": t(p.Wi), ik + "bias": t(p.bi),
          "b_classifier.fcc.weight": t(p.Wf), "b_classifier.fcc.bias": t(p.bf)}
    if p.nonlinear:
        sd.update({"b_classifier.q.0.weight": t(p.W1), "b_classifier.q.0.bias": t(p.b1),
                   "b_classifier.q.2.weight": t(p.W2), "b_classifier.q.2.bias": t(p.b2)})
    else:
        sd.update({"b_classifier.q.weight": t(p.W1), "b_classifier.q.bias": t(p.b1)})
    if p.passing_v:
        sd.update({"b_classifier.v.1.weight": t(p.Wv), "b_classifier.v.1.bias": t(p.bv)})
    return sd


def build_net(p: orc.Params, device="cuda", dropout_v=0.0):
    import dsmil as mil
    net = mil.MILNet(mil.FCLayer(p.D, p.C),
                     mil.BClassifier(p.D, p.C, dropout_v=dropout_v, nonlinear=p.nonlinear, passing_v=p.passing_v))
    net.load_state_dict(state_dict_from_params(p), strict=True)
    return net.to(device)


def caller_loss(classes, pred, y):
    """train_tcga.py:67-71"""
    crit = torch.nn.BCEWithLogitsLoss()
    mx, _ = torch.max(classes, 0)
    return 0.5 * crit(pred.view(1, -1), y.view(1, -1)) + 0.5 * crit(mx.view(1, -1), y.view(1, -1))


GRAD_MAP = {"Wi": "i_classifier.fc.0.weight", "bi": "i_classifier.fc.0.bias",
            "Wf": "b_classifier.fcc.weight", "bf": "b_classifier.fcc.bias",
            "Wv": "b_classifier.v.1.weight", "bv": "b_classifier.v.1.bias"}


def grad_name(short, nonlinear):
    if short in GRAD_MAP:
        return GRAD_MAP[short]
    if nonlinear:
        return {"W1": "b_classifier.q.0.weight", "b1": "b_classifier.q.0.bias",
                "W2": "b_classifier.q.2.weight", "b2": "b_classifier.q.2.bias"}[short]
    return {"W1": "b_classifier.q.weight", "b1": "b_classifier.q.bias"}[short]


def pred_tolerance_ok(pred, ref_pred, p: orc.Params, B_ref, tol):
    """|d| <= tol * max(|logit|, scale of the GEMV terms): the fcc GEMV cancels (SURVEY §7.2-2)."""
    terms = np.abs(p.Wf.reshape(p.C, -1)).astype(np.float64) @ np.abs(np.asarray(B_ref, np.float64).reshape(-1))
    err = np.abs(np.asarray(pred, np.float64).reshape(-1) - np.asarray(ref_pred, np.float64).reshape(-1))
    return bool(np.all(err <= tol * np.maximum(np.abs(np.asarray(ref_pred, np.float64).reshape(-1)), terms))), err


def scores_close(a, b, tol=2e-6):
    """Instance scores from two DIFFERENT kernels (k_qmlp_sm90 / k_scores: each sums the D products of a
    row in its own fixed order): equal to the tolerance every path is held to against the reference (2e-6 of the
    largest score); the arg-max they select is asserted bit-exact separately."""
    a = a.detach().float().cpu().numpy().astype(np.float64)
    b = b.detach().float().cpu().numpy().astype(np.float64)
    return a.shape == b.shape and float(np.max(np.abs(a - b))) <= tol * max(float(np.max(np.abs(b))), 1e-30)
