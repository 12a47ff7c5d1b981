"""The capture-safe row-sharded training step, without a GPU: the exported symbols, argument validation and workspace
sizes of the six dsmil_shard_*_dev calls (calls that return before any CUDA work), the refusals of
ShardedTrainStepGraph that come before any device work, and the device-offset max-prediction loss with its refusal
flag over gloo with two CPU processes."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import dsmil as mil
from dsmil_wsi_b200 import _lib, feed
from dsmil_wsi_b200.train_graph import ShardedTrainStepGraph

ERR_ARG, ERR_WORKSPACE = -1, -2
FAKE = 0x10000          # a non-NULL, 16-byte aligned "device pointer": never dereferenced on these paths

NEW = ["dsmil_shard_bags_train_dev_workspace_bytes", "dsmil_shard_bags_phase1_train_dev",
       "dsmil_shard_bags_phase2_train_dev", "dsmil_shard_bags_phase3_dev",
       "dsmil_shard_backward_bags_dev_workspace_bytes", "dsmil_shard_backward_bags_phase1_dev",
       "dsmil_shard_backward_bags_phase2_dev", "dsmil_shard_backward_bags_phase3_dev"]


def params(D=512, C_=2, nonlinear=1, passing_v=0):
    p = _lib.DsmilParams(D, C_, nonlinear, passing_v)
    for name in ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf"):
        setattr(p, name, FAKE)
    return p


def last_error(lib):
    return (lib.dsmil_last_error() or b"").decode()


def _ptrs(n, null):
    return [None if i == null else FAKE for i in range(n)]


# Each call with every pointer FAKE except index `null`; the indices below name the pointers each call requires.
def fph1(lib, p, nb=4, max_rows=1000, ws=FAKE, wsb=1 << 40, null=None):
    # Xs, Ns, row_offsets, then classes, save_Q, save_H1, cand_recs, status
    b = _ptrs(8, null)
    return lib.dsmil_shard_bags_phase1_train_dev(p, *b[:3], nb, max_rows, *b[3:], ws, wsb, None)


def fph2(lib, p, nb=4, max_rows=1000, ws=FAKE, wsb=1 << 40, null=None):
    # Q, cands_all, then A, crit_idx, q_max, recs_out
    b = _ptrs(6, null)
    return lib.dsmil_shard_bags_phase2_train_dev(p, nb, max_rows, *b[:2], 2, *b[2:], ws, wsb, None)


def fph3(lib, p, nb=4, max_rows=1000, ws=FAKE, wsb=1 << 40, null=None):
    # recs_all, then A, B, pred
    b = _ptrs(4, null)
    return lib.dsmil_shard_bags_phase3_dev(p, nb, max_rows, b[0], 2, *b[1:], ws, wsb, None)


def bph1(lib, p, nb=4, max_rows=1000, ws=FAKE, wsb=1 << 40, null=None):
    # Xs, Ns, then A, B, d_classes, d_pred, dA, t, gWi, gbi, gWf, gbf, status
    b = _ptrs(13, null)
    return lib.dsmil_shard_backward_bags_phase1_dev(p, *b[:2], nb, max_rows, *b[2:], ws, wsb, None)


def bph2(lib, p, nb=4, max_rows=1000, ws=FAKE, wsb=1 << 40, null=None):
    # A, dA_to_dL, t_global, Q, dqm_local
    b = _ptrs(5, null)
    return lib.dsmil_shard_backward_bags_phase2_dev(p, nb, max_rows, *b, ws, wsb, None)


def bph3(lib, p, nb=4, max_rows=1000, ws=FAKE, wsb=1 << 40, null=None):
    # row_offsets, Q, H1, dL, dqm, q_max, crit, then gW1, gb1, gW2, gb2
    b = _ptrs(11, null)
    return lib.dsmil_shard_backward_bags_phase3_dev(p, nb, max_rows, *b, ws, wsb, None)


FWD_WS, BWD_WS = "dsmil_shard_bags_train_dev_workspace_bytes", "dsmil_shard_backward_bags_dev_workspace_bytes"
# call -> (its workspace query, the bag list / status pointers, the other required pointers)
CALLS = {fph1: (FWD_WS, (0, 1, 7), (2, 3, 4, 5, 6)),
         fph2: (FWD_WS, (), (0, 1, 2, 3, 4, 5)),
         fph3: (FWD_WS, (), (0, 1, 2, 3)),
         bph1: (BWD_WS, (0, 1, 12), (2, 3, 6, 7)),
         bph2: (BWD_WS, (), (0, 1, 2, 3, 4)),
         bph3: (BWD_WS, (), (0, 1, 2, 3, 4, 5, 6))}


def test_every_new_symbol_is_exported():
    lib = _lib.load()
    for name in NEW:
        assert name in _lib.SIGNATURES, name
        assert getattr(lib, name) is not None


@pytest.mark.parametrize("call", list(CALLS), ids=lambda f: f.__name__)
def test_dev_entry_point_validation(call):
    lib = _lib.load()
    ws_name, listed, required = CALLS[call]
    P = lambda **kw: C.byref(params(**kw))
    assert call(lib, None) == ERR_ARG
    assert call(lib, P(D=166, C_=1)) == ERR_ARG and "D=166" in last_error(lib)
    assert call(lib, P(passing_v=1)) == ERR_ARG
    assert call(lib, P(nonlinear=0)) == ERR_ARG
    for nb in (0, -1, 65536):
        assert call(lib, P(), nb=nb) == ERR_ARG and "nb" in last_error(lib)
    for mr in (0, -5):
        assert call(lib, P(), max_rows=mr) == ERR_ARG and "max_rows" in last_error(lib)
    assert call(lib, P(), nb=65535, max_rows=1 << 31) == ERR_ARG      # tiles past an int
    for null in listed:
        assert call(lib, P(), null=null) == ERR_ARG and "bag list or status" in last_error(lib), null
    for null in required:
        assert call(lib, P(), null=null) == ERR_ARG, null
    need = getattr(lib, ws_name)(P(), 4, 1000)
    assert need > 0
    assert call(lib, P(), wsb=need - 1) == ERR_WORKSPACE
    assert call(lib, P(), ws=None) == ERR_WORKSPACE


@pytest.mark.parametrize("D,C_", [(512, 2), (1024, 4), (1536, 1)])
def test_dev_workspace_sizes(D, C_):
    lib = _lib.load()
    p = C.byref(params(D, C_))
    f = lambda nb, mr: lib.dsmil_shard_bags_train_dev_workspace_bytes(p, nb, mr)
    b = lambda nb, mr: lib.dsmil_shard_backward_bags_dev_workspace_bytes(p, nb, mr)
    for ws in (f, b):
        assert ws(1, 1) > 0
        assert ws(4, 1000) < ws(8, 1000) and ws(4, 1000) < ws(4, 5000)
        assert ws(0, 10) == 0 and ws(65536, 10) == 0 and ws(4, 0) == 0
    for q in (lib.dsmil_shard_bags_train_dev_workspace_bytes, lib.dsmil_shard_backward_bags_dev_workspace_bytes):
        assert q(C.byref(params(166, 1)), 4, 100) == 0
        assert q(C.byref(params(nonlinear=0)), 4, 100) == 0
    # never below the eager calls' sizes for nb bags of max_rows rows
    for nb, mr in [(1, 1), (1, 15000), (4, 129), (16, 10000), (3, 12000)]:
        Ns = (C.c_int64 * nb)(*[mr] * nb)
        assert f(nb, mr) >= lib.dsmil_shard_bags_workspace_bytes(p, Ns, nb)
        assert b(nb, mr) >= lib.dsmil_shard_backward_bags_workspace_bytes(p, Ns, nb)


def _net(D=512, C_=2, nonlinear=True):
    return mil.MILNet(mil.FCLayer(D, C_), mil.BClassifier(D, C_, nonlinear=nonlinear))


def test_sharded_graph_refuses_optimizers_it_cannot_replay():
    net = _net()
    for opt in (torch.optim.RMSprop(net.parameters()), torch.optim.Adam(net.parameters()),
                torch.optim.AdamW(net.parameters(), capturable=False),
                torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9, dampening=0.5)):
        with pytest.raises(ValueError):
            ShardedTrainStepGraph(net, torch.nn.BCEWithLogitsLoss(), opt, 4, 100)


@pytest.mark.parametrize("D,C_,nonlinear", [(166, 1, True), (512, 2, False), (512, 8, True)])
def test_sharded_graph_refuses_shapes_off_the_batched_path(D, C_, nonlinear):
    net = _net(D, C_, nonlinear)
    with pytest.raises(ValueError, match=f"D={D}, C={C_}"):
        ShardedTrainStepGraph(net, torch.nn.BCEWithLogitsLoss(), torch.optim.SGD(net.parameters(), lr=0.1), 2, 100)


# ---- the device-offset max prediction over gloo ------------------------------------------------------------------
LOSS_NS, LOSS_C, PAD = [7, 2, 9], 2, 5        # global bag sizes; PAD rows past the live ones, as a graph's capacity


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _loss_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dsmil_wsi_b200.sharded import shard_bounds, sharded_max_prediction_bags, sharded_max_prediction_bags_dev
        g = torch.Generator().manual_seed(3)
        full = [torch.randn(n, LOSS_C, generator=g) for n in LOSS_NS]            # every rank sees the same bags
        labels = (torch.rand(len(LOSS_NS), LOSS_C, generator=g) > 0.5).float()
        crit = torch.stack([x.argmax(0) for x in full])                         # [nb, C] global rows
        bounds = [shard_bounds(n, world)[rank] for n in LOSS_NS]
        offs = [lo for lo, _ in bounds]
        Ns = [hi - lo for lo, hi in bounds]
        local = torch.cat([x[lo:hi] for x, (lo, hi) in zip(full, bounds)])
        bce = torch.nn.BCEWithLogitsLoss()
        pred = torch.randn(len(LOSS_NS), LOSS_C, generator=g)

        a = local.clone().requires_grad_(True)
        want = sharded_max_prediction_bags(a, crit, offs, Ns)
        feed.minibatch_loss(bce, pred, want, labels).backward()

        b = torch.cat([local, torch.randn(PAD, LOSS_C, generator=g)]).requires_grad_(True)
        t_offs, t_Ns = torch.tensor(offs), torch.tensor(Ns)
        got, refused = sharded_max_prediction_bags_dev(b, crit, t_offs, t_Ns, torch.tensor(False))
        feed.minibatch_loss(bce, pred, got, labels).backward()

        out = {}
        for who in range(world):                                                # one rank refuses, then the other
            mx, ref = sharded_max_prediction_bags_dev(b.detach(), crit, t_offs, t_Ns, torch.tensor(rank == who))
            loss = feed.minibatch_loss(bce, pred, mx, labels)
            out[who] = (bool(ref), float(torch.where(~ref, loss, torch.full_like(loss, float("nan")))))
        ret[rank] = dict(want=want.detach().numpy(), got=got.detach().numpy(), refused=bool(refused),
                         ga=a.grad.numpy(), gb=b.grad.numpy(), live=int(local.shape[0]), out=out)
    finally:
        dist.destroy_process_group()


def test_device_offset_max_prediction_matches_and_refuses_on_every_rank():
    world = 2
    ret = mp.Manager().dict()
    mp.spawn(_loss_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    for r in range(world):
        o = ret[r]
        assert np.array_equal(o["got"], o["want"]) and np.array_equal(o["got"], ret[0]["got"]), r
        assert not o["refused"]
        n = o["live"]
        assert np.array_equal(o["gb"][:n], o["ga"]) and not o["gb"][n:].any(), r
        for who in range(world):
            refused, loss = o["out"][who]
            assert refused and np.isnan(loss), (r, who)
