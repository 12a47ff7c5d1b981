"""Host-side mirror of the reference operator interface (dsmil.py:6-74).

Same class names, constructor signatures, parameter names (state_dict compatible with the
shipped example_aggregator_weights/*.pth), return tuples and train/eval behaviour as the
reference, so `import dsmil as mil` in train_tcga.py / train_mil.py / compute_feats.py /
attention_map.py keeps working unchanged -- but forward/backward run in libdsmil_b200.so.
The parameter containers are real nn.Linear / nn.Conv1d / nn.Sequential children because the
callers rely on it: `.apply(orthogonal_)` with isinstance checks (train_tcga.py:229-239),
deepcopy/.cpu()/.cuda() (:389-390), sub-module reassignment (testing_tcga.py:144).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import functional as Fn


class FCLayer(nn.Module):
    """dsmil.py:6-12 -- instance classifier on pre-computed features; returns (feats, scores)."""

    def __init__(self, in_size, out_size=1):
        super().__init__()
        self.fc = nn.Sequential(nn.Linear(in_size, out_size))

    def _linear(self) -> nn.Linear:
        lin = self.fc[0] if isinstance(self.fc, nn.Sequential) else self.fc
        if not isinstance(lin, nn.Linear):
            raise TypeError("FCLayer.fc must hold an nn.Linear")
        return lin

    def forward(self, feats):
        lin = self._linear()
        x = Fn.instance_scores(feats, lin.weight, lin.bias)
        return feats, x  # the SAME feats object, as the reference (dsmil.py:12)


class IClassifier(nn.Module):
    """dsmil.py:14-25 -- CNN backbone + Linear; returns (feats.view(N,-1), scores).
    The backbone is whatever module the caller passes (compute_feats.py:146-170 builds a
    torchvision ResNet); the Linear and everything after it is ours."""

    def __init__(self, feature_extractor, feature_size, output_class):
        super().__init__()
        self.feature_extractor = feature_extractor
        self.fc = nn.Linear(feature_size, output_class)

    def _linear(self) -> nn.Linear:
        return self.fc

    def embed(self, x):
        feats = self.feature_extractor(x)
        return feats.view(feats.shape[0], -1)

    def forward(self, x):
        feats = self.embed(x)
        c = Fn.instance_scores(feats, self.fc.weight, self.fc.bias)
        return feats, c


class BClassifier(nn.Module):
    """dsmil.py:27-62 -- bag classifier: critical instance, Q(/V) projection, attention over the
    instances, bag embedding, Conv1d bag logits.  forward(feats, c) -> (C, A, B)."""

    def __init__(self, input_size, output_class, dropout_v=0.0, nonlinear=True, passing_v=False):
        super().__init__()
        if nonlinear:
            self.q = nn.Sequential(nn.Linear(input_size, 128), nn.ReLU(), nn.Linear(128, 128), nn.Tanh())
        else:
            self.q = nn.Linear(input_size, 128)
        if passing_v:
            self.v = nn.Sequential(nn.Dropout(dropout_v), nn.Linear(input_size, input_size), nn.ReLU())
        else:
            self.v = nn.Identity()
        self.fcc = nn.Conv1d(output_class, output_class, kernel_size=input_size)

    # -- parameter view -------------------------------------------------------------------------
    def _q_params(self):
        q = self.q
        if isinstance(q, nn.Linear):
            return q.weight, q.bias, None, None
        if (isinstance(q, nn.Sequential) and len(q) == 4 and isinstance(q[0], nn.Linear)
                and isinstance(q[1], nn.ReLU) and isinstance(q[2], nn.Linear) and isinstance(q[3], nn.Tanh)):
            return q[0].weight, q[0].bias, q[2].weight, q[2].bias
        raise TypeError("BClassifier.q must be Linear(D,128) or Sequential(Linear, ReLU, Linear, Tanh) "
                        "(dsmil.py:31,33); other structures have no H100 kernel")

    def _v_params(self):
        v = self.v
        if isinstance(v, nn.Identity):
            return None, None, 0.0
        if (isinstance(v, nn.Sequential) and len(v) == 3 and isinstance(v[0], nn.Dropout)
                and isinstance(v[1], nn.Linear) and isinstance(v[2], nn.ReLU)):
            return v[1].weight, v[1].bias, float(v[0].p)
        raise TypeError("BClassifier.v must be Identity or Sequential(Dropout, Linear, ReLU) (dsmil.py:35-41)")

    def _v_input(self, feats, out=None):
        """A bag's value input in a batched step: feats times v's dropout mask, drawn as nn.Dropout draws it in
        self.forward (dsmil.py:36), into `out` when given; None where no mask is drawn (eval mode, p = 0)."""
        _, _, p_drop = self._v_params()
        if not (self.training and p_drop > 0.0):
            return None
        return torch.mul(feats, self.v[0](torch.ones_like(feats)), out=out)

    def _run(self, feats, i_weight, i_bias, classes_in):
        W1, b1, W2, b2 = self._q_params()
        Wv, bv, p_drop = self._v_params()
        v_input = v_mask = None
        if Wv is not None and self.training and p_drop > 0.0:
            # same RNG consumption as nn.Dropout(feats) in the reference (dsmil.py:36)
            v_mask = self.v[0](torch.ones_like(feats))
            v_input = feats.detach() * v_mask  # derived buffer; its gradient is folded in by dsmil_backward
        params = (i_weight, i_bias, W1, b1, W2, b2, Wv, bv, self.fcc.weight, self.fcc.bias)
        return Fn.mil_forward(feats, params, v_input=v_input, v_mask=v_mask, classes_in=classes_in)

    def forward(self, feats, c):
        _, pred, A, B, _ = self._run(feats, None, None, c)
        return pred, A, B


def milnet_params(milnet):
    """The ten parameter tensors of a MILNet(FCLayer|IClassifier, BClassifier) in ABI order (functional.PARAM_NAMES),
    None where the model has none."""
    lin = milnet.i_classifier._linear()
    bc = milnet.b_classifier
    W1, b1, W2, b2 = bc._q_params()
    Wv, bv, _ = bc._v_params()
    return (lin.weight, lin.bias, W1, b1, W2, b2, Wv, bv, bc.fcc.weight, bc.fcc.bias)


class MILNet(nn.Module):
    """dsmil.py:64-74 -- forward(x) -> (classes, prediction_bag, A, B)."""

    def __init__(self, i_classifier, b_classifier):
        super().__init__()
        self.i_classifier = i_classifier
        self.b_classifier = b_classifier

    def forward(self, x):
        ic, bc = self.i_classifier, self.b_classifier
        if isinstance(bc, BClassifier) and isinstance(ic, (FCLayer, IClassifier)):
            # fused form: scores, arg-max, Q-MLP, attention, bag logits in one library call
            feats = ic.embed(x) if isinstance(ic, IClassifier) else x
            lin = ic._linear()
            classes, pred, A, B, _ = bc._run(feats, lin.weight, lin.bias, None)
            return classes, pred, A, B
        feats, classes = ic(x)                       # foreign instance stream: split form
        prediction_bag, A, B = bc(feats, classes)
        return classes, prediction_bag, A, B

    def forward_bags(self, bags, *, grad=False):
        """Throughput form: a list of bags [N_i, D] -> sequence of (classes, prediction_bag, A, B), computed by ONE
        library call (bag table; see DESIGN.md).  The result is a lazy sequence of views over packed outputs
        (`.packed`).  grad=False (default): inference, no autograd.  grad=True with grad mode on: the packed outputs
        carry autograd history and one backward call covers the whole batch (a minibatch training step).  Models
        with passing_v run one dsmil_value_forward_bags call for inference (in train mode each bag's dropout mask of
        v is drawn in bag order, as `self.forward` draws it) and `self.forward` per bag with grad=True; a foreign
        instance classifier always runs `self.forward` per bag."""
        if not (grad and torch.is_grad_enabled()):
            with torch.no_grad():
                return self._forward_bags(bags, False)
        return self._forward_bags(bags, True)

    def _forward_bags(self, bags, grad):
        ic, bc = self.i_classifier, self.b_classifier
        if not (isinstance(bc, BClassifier) and isinstance(ic, (FCLayer, IClassifier))):
            return [self.forward(b) for b in bags]
        params = milnet_params(self)
        if params[6] is not None:   # Wv: a value network
            if grad:   # autograd through the per-bag forward: the gradients users get from it, bag by bag
                return [self.forward(b) for b in bags]
            return self._forward_value_bags(bags, params)
        feats = [ic.embed(b) if isinstance(ic, IClassifier) else b for b in bags]
        outs, _ = Fn.mil_forward_bags(feats, params, grad=grad)
        return outs

    def _forward_value_bags(self, bags, params):
        """Inference of a passing_v model over the bags in one library call, with the bits and RNG draws of the
        per-bag loop."""
        ic, bc = self.i_classifier, self.b_classifier
        feats, v_inputs = [], []
        for b in bags:   # embedding, then v's dropout mask, bag by bag: the per-bag loop's draws in its order
            f = ic.embed(b) if isinstance(ic, IClassifier) else b
            feats.append(f)
            v_inputs.append(bc._v_input(f))
        if v_inputs and v_inputs[0] is None:
            v_inputs = None
        outs, _ = Fn.mil_forward_value_bags(feats, params, v_inputs)
        return outs

    @torch.no_grad()
    def critical_instances(self, x):
        """Indices dsmil.py:52-53 selects (row 0 of the descending sort), lowest index on ties."""
        ic, bc = self.i_classifier, self.b_classifier
        feats = ic.embed(x) if isinstance(ic, IClassifier) else x
        lin = ic._linear()
        return bc._run(feats, lin.weight, lin.bias, None)[4]
