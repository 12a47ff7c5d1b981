"""Batched training without a GPU: argument validation and size arithmetic of dsmil_forward_bags_train /
dsmil_backward_bags (calls that return before any CUDA work), the minibatch grouping of feed.train_epoch with a
plain-torch stand-in for the operator, and the batched backward's algebra restated in numpy against the per-bag fp64
oracle."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn as nn

from dsmil_wsi_b200 import _lib, feed
from dsmil_wsi_b200 import functional as Fn
from oracle import dsmil_oracle as orc

ERR_ARG, ERR_WORKSPACE, ERR_EMPTY = -1, -2, -4
FAKE = 0x10000          # a non-NULL, 16-byte aligned "device pointer": never dereferenced on these paths


def params(D=512, C_=2, nonlinear=1, passing_v=0):
    p = _lib.DsmilParams(D, C_, nonlinear, passing_v)
    for name in ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf"):
        setattr(p, name, FAKE)
    if not nonlinear:
        p.W2 = p.b2 = None
    return p


def last_error(lib):
    return (lib.dsmil_last_error() or b"").decode()


def arrays(Ns):
    return (C.c_void_p * len(Ns))(*[FAKE] * len(Ns)), (C.c_int64 * len(Ns))(*Ns)


def fwd_train(lib, p, Xs, Ns, nb, ws=None, wsb=0, sQ=FAKE, sH=FAKE):
    return lib.dsmil_forward_bags_train(C.byref(p), Xs, Ns, nb, FAKE, FAKE, FAKE, FAKE, FAKE, sQ, sH, ws, wsb, None)


def bwd(lib, p, Xs, Ns, nb, ws=None, wsb=0, Q=FAKE, H1=FAKE, gX=None):
    g = _lib.DsmilGrads(*([FAKE] * 10), gX)
    return lib.dsmil_backward_bags(C.byref(p), Xs, Ns, nb, Q, H1, FAKE, FAKE, FAKE, None, FAKE, None, None,
                                   C.byref(g), ws, wsb, None)


def test_forward_bags_train_validation():
    lib = _lib.load()
    p = params()
    Xs, Ns = arrays([100, 200])
    assert fwd_train(lib, p, Xs, Ns, 0) == ERR_ARG
    assert fwd_train(lib, p, None, Ns, 2) == ERR_ARG
    assert fwd_train(lib, p, Xs, Ns, 2, sQ=None) == ERR_ARG and "NULL pointer" in last_error(lib)
    assert fwd_train(lib, p, Xs, Ns, 2, sH=None) == ERR_ARG
    assert fwd_train(lib, params(passing_v=1), Xs, Ns, 2) == ERR_ARG and "identity v" in last_error(lib)
    assert fwd_train(lib, p, Xs, Ns, 2) == ERR_WORKSPACE
    need = lib.dsmil_forward_bags_train_workspace_bytes(C.byref(p), Ns, 2)
    assert need > 0 and fwd_train(lib, p, Xs, Ns, 2, FAKE, need - 1) == ERR_WORKSPACE
    assert "workspace too small" in last_error(lib)
    Xs0, Ns0 = arrays([100, 0])
    assert fwd_train(lib, p, Xs0, Ns0, 2, FAKE, 1 << 30) == ERR_EMPTY and "IndexError" in last_error(lib)
    Xs[1] = None
    assert fwd_train(lib, p, Xs, Ns, 2, FAKE, 1 << 30) == ERR_ARG and "NULL features" in last_error(lib)


def test_backward_bags_validation():
    lib = _lib.load()
    p = params()
    Xs, Ns = arrays([100, 200, 3])
    assert bwd(lib, p, Xs, Ns, 0) == ERR_ARG
    assert bwd(lib, p, None, Ns, 3) == ERR_ARG
    assert bwd(lib, p, Xs, Ns, 3, Q=None) == ERR_ARG and "NULL pointer" in last_error(lib)
    assert bwd(lib, p, Xs, Ns, 3, H1=None) == ERR_ARG and "H1" in last_error(lib)
    assert bwd(lib, params(passing_v=1), Xs, Ns, 3) == ERR_ARG and "identity v" in last_error(lib)
    assert bwd(lib, p, Xs, Ns, 3) == ERR_WORKSPACE
    for gX in (None, FAKE):
        need = lib.dsmil_backward_bags_workspace_bytes(C.byref(p), Ns, 3, int(gX is not None))
        assert need > 0 and bwd(lib, p, Xs, Ns, 3, FAKE, need - 1, gX=gX) == ERR_WORKSPACE
    Xs0, Ns0 = arrays([100, 0, 3])
    assert bwd(lib, p, Xs0, Ns0, 3, FAKE, 1 << 40) == ERR_EMPTY and "IndexError" in last_error(lib)
    Xs[2] = None
    assert bwd(lib, p, Xs, Ns, 3, FAKE, 1 << 40) == ERR_ARG and "NULL features" in last_error(lib)


@pytest.mark.parametrize("D,C_,nonlinear", [(512, 2, 1), (512, 1, 1), (1024, 4, 1), (166, 1, 1), (230, 1, 0),
                                            (4096, 8, 1)])
def test_workspace_sizes_grow_with_rows(D, C_, nonlinear):
    lib = _lib.load()
    p = params(D, C_, nonlinear)
    batches = [[1], [1, 2], [128, 129], [2049, 127, 1], [10000] * 4, [15000] * 16, [15000] * 16 + [1]]
    fw, bw = [], []
    for Ns in batches:
        _, n = arrays(Ns)
        fw.append(lib.dsmil_forward_bags_train_workspace_bytes(C.byref(p), n, len(Ns)))
        bw.append(lib.dsmil_backward_bags_workspace_bytes(C.byref(p), n, len(Ns), 0))
        assert lib.dsmil_backward_bags_workspace_bytes(C.byref(p), n, len(Ns), 1) >= bw[-1]
        # the per-bag route of the training forward runs in the same workspace
        assert fw[-1] >= lib.dsmil_forward_workspace_bytes(C.byref(p), max(Ns))
    assert fw[0] > 0 and fw == sorted(fw)
    assert bw[0] > 0 and bw == sorted(bw)
    _, n = arrays([100])
    assert lib.dsmil_forward_bags_train_workspace_bytes(C.byref(params(passing_v=1)), n, 1) == 0
    assert lib.dsmil_backward_bags_workspace_bytes(C.byref(params(passing_v=1)), n, 1, 0) == 0


# ---- minibatch grouping of feed.train_epoch ------------------------------------------------------------------------
class TorchMIL(nn.Module):
    """dsmil.py:46-62 in plain torch; forward_bags packs its outputs like the bag-table call."""

    def __init__(self, D, C):
        super().__init__()
        self.fc = nn.Linear(D, C)
        self.q = nn.Sequential(nn.Linear(D, 128), nn.ReLU(), nn.Linear(128, 128), nn.Tanh())
        self.fcc = nn.Conv1d(C, C, kernel_size=D)
        self.calls = []

    def forward(self, x):
        c = self.fc(x)
        Q = self.q(x)
        idx = torch.argmax(c, 0)
        A = torch.softmax(Q @ Q[idx].t() / torch.sqrt(torch.tensor(128.0)), 0)
        B = (A.t() @ x).unsqueeze(0)
        return c, self.fcc(B).view(1, -1), A, B

    def forward_bags(self, xs, grad=False):
        self.calls.append((len(xs), grad))
        outs = [self(x) for x in xs]
        cat = lambda i: torch.cat([o[i] for o in outs])
        crit = torch.stack([torch.argmax(o[0], 0) for o in outs])
        return Fn.BagOutputs(cat(0), cat(1), cat(2), cat(3), [int(x.shape[0]) for x in xs], crit)


def _store(C, n, D=12, seed=0):
    g = torch.Generator().manual_seed(seed)
    store = feed.DeviceBagStore(D, device="cpu")
    for i in range(n):
        store.add_bag(torch.randn(3 + 2 * i, D, generator=g), (torch.rand(C, generator=g) > 0.5).float())
    return store


class CountingSGD(torch.optim.SGD):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.steps = 0

    def step(self, closure=None):
        self.steps += 1
        return super().step(closure)


@pytest.mark.parametrize("C,k,n", [(1, 4, 10), (2, 3, 9), (3, 16, 5)])
def test_train_epoch_groups_bags_into_one_step(monkeypatch, C, k, n):
    monkeypatch.setattr(feed, "dropout_patches", lambda feats, p, generator=None: feats)   # row gather needs a GPU
    torch.manual_seed(C)
    net = TorchMIL(12, C)
    ref = copy.deepcopy(net)
    store = _store(C, n)
    order = list(range(n))[::-1]
    crit = nn.BCEWithLogitsLoss()
    opt = CountingSGD(net.parameters(), lr=0.1)
    loss = feed.train_epoch(net, store, crit, opt, order=order, bags_per_step=k)
    groups = [order[s:s + k] for s in range(0, n, k)]
    assert net.calls == [(len(g), True) for g in groups] and opt.steps == len(groups)
    # the same epoch as gradient accumulation of (per-bag loss / group size), one SGD step per group
    ropt = torch.optim.SGD(ref.parameters(), lr=0.1)
    total = 0.0
    for g in groups:
        ropt.zero_grad()
        for i in g:
            feats, label = store.bags[i]
            ins, bag, _, _ = ref(feats)
            mx, _ = torch.max(ins, 0)
            l = 0.5 * crit(bag.view(1, -1), label.view(1, -1)) + 0.5 * crit(mx.view(1, -1), label.view(1, -1))
            (l / len(g)).backward()
            total += float(l.detach())
        ropt.step()
    assert abs(loss - total / n) < 1e-6
    for (name, a), b in zip(net.named_parameters(), ref.parameters()):
        assert torch.allclose(a, b, rtol=0, atol=1e-6), name


def test_train_epoch_default_is_one_bag_per_step(monkeypatch):
    monkeypatch.setattr(feed, "dropout_patches", lambda feats, p, generator=None: feats)
    net = TorchMIL(12, 2)
    opt = CountingSGD(net.parameters(), lr=0.1)
    feed.train_epoch(net, _store(2, 5), nn.BCEWithLogitsLoss(), opt, order=list(range(5)))
    assert net.calls == [] and opt.steps == 5


# ---- the batched algebra against the per-bag oracle -----------------------------------------------------------------
def batched_backward(Xs, p, outs, d_cls, d_pred):
    """The reverse pass of dsmil_backward_bags over packed rows, in fp64: every per-bag sum is a segment sum."""
    f = np.float64
    P = p.astype(f)
    Cc = P.C
    Ns = [x.shape[0] for x in Xs]
    nb = len(Ns)
    seg = np.repeat(np.arange(nb), Ns)
    off = np.concatenate([[0], np.cumsum(Ns)[:-1]])
    X = np.concatenate(Xs).astype(f)
    A, Q = np.concatenate([o.A for o in outs]), np.concatenate([o.Q for o in outs])
    B = np.stack([o.B.reshape(Cc, -1) for o in outs])
    crit = np.stack([o.idx for o in outs])
    dc, dp = np.concatenate(d_cls), np.concatenate(d_pred)              # [sum N, C], [nb, C]
    g = {"Wi": dc.T @ X, "bi": dc.sum(0), "Wf": np.einsum("bk,bjd->kjd", dp, B), "bf": dp.sum(0)}
    dB = np.einsum("kjd,bk->bjd", P.Wf, dp)
    dA = np.einsum("nd,njd->nj", X, dB[seg])
    t = np.zeros((nb, Cc))
    np.add.at(t, seg, A * dA)
    dL = A * (dA - t[seg]) / f(orc.SCALE_F32)
    qmax = Q[off[:, None] + crit]                                          # [nb, C, 128]
    dQ = np.einsum("nk,nkj->nj", dL, qmax[seg])
    dqm = np.zeros((nb, Cc, Q.shape[1]))
    np.add.at(dqm, seg, dL[:, :, None] * Q[:, None, :])
    for b in range(nb):
        for k in range(Cc):
            dQ[off[b] + crit[b, k]] += dqm[b, k]
    if P.nonlinear:
        H1 = np.concatenate([o.H1 for o in outs])
        dz2 = dQ * (1 - Q * Q)
        g["W2"], g["b2"] = dz2.T @ H1, dz2.sum(0)
        dz1 = (dz2 @ P.W2) * (H1 > 0)
    else:
        dz1 = dQ
    g["W1"], g["b1"] = dz1.T @ X, dz1.sum(0)
    g["X"] = dz1 @ P.W1 + dc @ P.Wi + np.einsum("nk,nkd->nd", A, dB[seg])
    return g


@pytest.mark.parametrize("D,C_,nonlinear", [(24, 1, True), (20, 3, True), (17, 2, False)])
def test_sum_of_per_bag_oracle_gradients_is_the_batched_algebra(D, C_, nonlinear):
    p = orc.random_params(D, C_, seed=D, nonlinear=nonlinear)
    Ns = [1, 2, 9, 30]
    Xs = [orc.synthetic_bag(n, D, seed=100 + i, kind="normal") for i, n in enumerate(Ns)]
    rng = np.random.default_rng(C_)
    outs, d_cls, d_pred, want = [], [], [], {}
    for X in Xs:
        o = orc.forward(X, p)
        _, dc, dp = orc.caller_loss_grads(o, (rng.random(C_) > 0.5).astype(np.float64))
        dc, dp = dc / len(Ns), dp / len(Ns)                     # the caller's loss is the mean over the bags
        g = orc.backward(X, p, o, dc, dp, need_dX=True)
        for k, v in g.items():
            want[k] = v if k not in want else (np.concatenate([want[k], v]) if k == "X" else want[k] + v)
        outs.append(o), d_cls.append(dc), d_pred.append(dp)
    got = batched_backward(Xs, p, outs, d_cls, d_pred)
    assert sorted(got) == sorted(want)
    for k in want:
        assert np.allclose(got[k], want[k], rtol=1e-12, atol=1e-13 * max(1.0, np.abs(want[k]).max())), k
