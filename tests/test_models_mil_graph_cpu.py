"""The capture-safe fold step on the generic shapes without a GPU: argument validation, routes, batch limits and
workspace sizes of dsmil_generic_forward_bags_models_train_dev / dsmil_generic_backward_bags_models_dev (calls that
return before any CUDA work), the generic fold planner's table numbering against a Python restatement, and the
refusals of FoldTrainStepGraph(generic=True) and feed.train_epoch_models(graph=True, generic=True) that come before any
device work."""
import ctypes as C
import os
import random
import re
import subprocess

import pytest
import torch

import dsmil as mil
from dsmil_wsi_b200 import _lib, build, feed
from dsmil_wsi_b200.train_graph import FoldTrainStepGraph, fold_step_shape

ERR_ARG, ERR_WORKSPACE = -1, -2
FAKE = 0x10000          # a non-NULL, 16-byte aligned "device pointer": never dereferenced on these paths
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("dsmil_generic_models_supported", "dsmil_generic_forward_bags_models_train_dev_workspace_bytes",
         "dsmil_generic_forward_bags_models_train_dev", "dsmil_generic_backward_bags_models_dev_workspace_bytes",
         "dsmil_generic_backward_bags_models_dev")
K_SPLITS, TBM, KQ = 296, 128, 128


def params(D=166, C_=1, nonlinear=1, passing_v=0, **over):
    p = _lib.DsmilParams(D, C_, nonlinear, passing_v)
    for name in ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf"):
        setattr(p, name, FAKE)
    if not nonlinear:
        p.W2 = p.b2 = None
    for k, v in over.items():
        setattr(p, k, v)
    return p


def arr(ps):
    return (_lib.DsmilParams * len(ps))(*ps)


def i32(xs):
    return (C.c_int32 * len(xs))(*xs)


def last_error(lib):
    return (lib.dsmil_last_error() or b"").decode()


def grads(M, gX=None):
    g = (_lib.DsmilGrads * M)()
    for m in range(M):
        for name, _ in _lib.DsmilGrads._fields_:
            setattr(g[m], name, gX if name == "gX" else FAKE)
    return g


def fwd(lib, ps, M, nbs, max_rows=1000, ws=FAKE, wsb=1 << 40, null=None, **_):
    # Xs, Ns, then classes, pred, A, B, crit, save_Q, save_H1, status
    b = [None if i == null else FAKE for i in range(10)]
    return lib.dsmil_generic_forward_bags_models_train_dev(ps, M, b[0], b[1], None if nbs is None else i32(nbs),
                                                           max_rows, *b[2:], ws, wsb, None)


def bwd(lib, ps, M, nbs, max_rows=1000, ws=FAKE, wsb=1 << 40, null=None, dA=None, dB=None, gX=None, g="default"):
    # Xs, Ns, Q, H1, A, B, crit, d_classes, d_pred, status
    b = [None if i == null else FAKE for i in range(10)]
    g = grads(max(M, 1), gX) if g == "default" else g
    return lib.dsmil_generic_backward_bags_models_dev(ps, M, b[0], b[1], None if nbs is None else i32(nbs), max_rows,
                                                      *b[2:9], dA, dB, g, b[9], ws, wsb, None)


def fwd_ws(lib, ps, M, nbs, max_rows=1000):
    return lib.dsmil_generic_forward_bags_models_train_dev_workspace_bytes(ps, M, i32(nbs), max_rows)


def bwd_ws(lib, ps, M, nbs, max_rows=1000):
    return lib.dsmil_generic_backward_bags_models_dev_workspace_bytes(ps, M, i32(nbs), max_rows)


def test_symbols_exported_declared_and_bound():
    lib = _lib.load()
    header = open(os.path.join(ROOT, "include", "dsmil_b200.h")).read()
    for name in NAMES:
        assert re.search(rf"\b{name}\s*\(", header), name
        assert hasattr(lib, name), name
        assert name in _lib.SIGNATURES, name


@pytest.mark.parametrize("call,ws", [(fwd, fwd_ws), (bwd, bwd_ws)])
def test_generic_fold_dev_entry_point_validation(call, ws):
    lib = _lib.load()
    two = arr([params(), params()])
    assert call(lib, None, 2, [1, 1]) == ERR_ARG and "params is NULL" in last_error(lib)
    nine = arr([params() for _ in range(9)])
    for M in (0, 9, -1):
        assert call(lib, nine, M, [1] * 9) == ERR_ARG and "M=" in last_error(lib)
        assert ws(lib, nine, M, [1] * 9) == 0
    # members of different D / C / q form are named
    for other in (dict(D=230), dict(C_=2), dict(nonlinear=0)):
        ps = arr([params(), params(**other)])
        assert call(lib, ps, 2, [1, 1]) == ERR_ARG and "model 1" in last_error(lib), other
        assert ws(lib, ps, 2, [1, 1]) == 0
    # a value network
    pv = arr([params(passing_v=1)] * 2)
    assert call(lib, pv, 2, [1, 1]) == ERR_ARG and "identity v" in last_error(lib)
    assert ws(lib, pv, 2, [1, 1]) == 0
    # group sizes, each and in all
    for nbs in ([0, 1], [1, 0], [2, -1], [40000, 25536], [65536, 1]):
        assert call(lib, two, 2, nbs) == ERR_ARG, nbs
        assert ws(lib, two, 2, nbs) == 0
    assert call(lib, two, 2, None) == ERR_ARG
    for mr in (0, -5, 1 << 32):
        assert call(lib, two, 2, [2, 3], max_rows=mr) == ERR_ARG and "max_rows" in last_error(lib)
        assert ws(lib, two, 2, [2, 3], mr) == 0
    assert call(lib, two, 2, [30000, 30000], max_rows=1 << 30) == ERR_ARG      # twice the tiles past an int
    # the bag list and the status words (last) are always required; so is every other buffer but H1
    for null in (0, 1, 9) + tuple(range(2, 9 if call is fwd else 7)):
        if (call is fwd and null == 8) or (call is bwd and null == 3):
            continue
        assert call(lib, two, 2, [2, 3], null=null) == ERR_ARG, null
    need = ws(lib, two, 2, [2, 3])
    assert need > 0
    assert call(lib, two, 2, [2, 3], wsb=need - 1) == ERR_WORKSPACE and "workspace too small" in last_error(lib)
    assert call(lib, two, 2, [2, 3], ws=None) == ERR_WORKSPACE


def test_nonlinear_needs_H1_and_a_linear_q_does_not():
    lib = _lib.load()
    nl, lin = arr([params()] * 2), arr([params(D=230, C_=2, nonlinear=0)] * 2)
    assert fwd(lib, nl, 2, [2, 3], null=8) == ERR_ARG and "NULL" in last_error(lib)
    assert bwd(lib, nl, 2, [2, 3], null=3) == ERR_ARG and "NULL" in last_error(lib)
    for call, null in ((fwd, 8), (bwd, 3)):   # passes every check: only the workspace is short
        assert call(lib, lin, 2, [2, 3], null=null, wsb=1) == ERR_WORKSPACE


def test_generic_fold_backward_refuses_upstream_A_B_features_and_null_grads():
    lib = _lib.load()
    two = arr([params(), params()])
    assert bwd(lib, two, 2, [1, 2], dA=FAKE) == ERR_ARG and "d_A" in last_error(lib)
    assert bwd(lib, two, 2, [1, 2], dB=FAKE) == ERR_ARG
    assert bwd(lib, two, 2, [1, 2], gX=FAKE) == ERR_ARG
    g = grads(2)
    g[1].gX = FAKE
    assert bwd(lib, two, 2, [1, 2], g=g) == ERR_ARG
    assert bwd(lib, two, 2, [1, 2], g=None) == ERR_ARG


GENERIC = [dict(D=166, C_=1), dict(D=230, C_=1), dict(D=230, C_=2, nonlinear=0), dict(D=512, C_=6),
           dict(D=2049, C_=2), dict(D=4096, C_=1), dict(D=512, C_=1, nonlinear=0)]
TENSOR_CORE = [dict(D=512, C_=2), dict(D=1024, C_=4), dict(D=2048, C_=2)]


def test_routes():
    """The generic fold calls take exactly the members that dsmil_generic_bags_supported takes, and refuse every
    tensor-core shape, fused fold or not; the tensor-core fold calls keep refusing the generic shapes."""
    lib = _lib.load()
    for kw in GENERIC + TENSOR_CORE + [dict(passing_v=1), dict(D=512, C_=2, passing_v=1)]:
        for M in (1, 2, 5, 6, 8):
            ps = arr([params(**kw)] * M)
            one = bool(lib.dsmil_generic_bags_supported(C.byref(ps[0])))
            assert bool(lib.dsmil_generic_models_supported(ps, M)) == one, (kw, M)
            assert one == (kw in GENERIC), kw
            if not one:
                for call, ws in ((fwd, fwd_ws), (bwd, bwd_ws)):
                    assert call(lib, ps, M, [1] * M) == ERR_ARG, (kw, M)
                    assert ws(lib, ps, M, [1] * M) == 0
            else:
                assert not lib.dsmil_models_supported(ps, M)
                assert lib.dsmil_forward_bags_models_train_dev(ps, M, FAKE, FAKE, i32([1] * M), 10, *[FAKE] * 8,
                                                               FAKE, 1 << 40, None) == ERR_ARG
    # a tensor-core shape that does not fit the fused fold step stays refused here too
    wide = arr([params(D=2048, C_=2)] * 6)
    assert not lib.dsmil_models_supported(wide, 6) and not lib.dsmil_generic_models_supported(wide, 6)
    assert fwd(lib, wide, 6, [1] * 6) == ERR_ARG and "tensor-core" in last_error(lib)


def ceil_div(a, b):
    return -(-a // b)


def rag_splits(M1, D, gemv):
    return K_SPLITS if gemv else max(1, K_SPLITS // (ceil_div(M1, TBM) * ceil_div(D, TBM)))


def largest_ne(C_, D, M):
    """The most bags in all that a fold call of M members takes: entries, and each GEMM's chunk capacity (rag_splits
    per member plus one chunk per bag), within 65535."""
    gemv = C_ <= 4 and D % 4 == 0 and D // 4 <= 256
    allowance = max(rag_splits(C_, D, gemv), rag_splits(KQ, D, False))
    return 65535 - M * allowance


@pytest.mark.parametrize("kw", [dict(D=166, C_=1), dict(D=230, C_=2, nonlinear=0), dict(D=512, C_=6)])
@pytest.mark.parametrize("M", [1, 5])
def test_batch_limits(kw, M):
    lib = _lib.load()
    ps = arr([params(**kw)] * M)
    top = largest_ne(kw["C_"], kw["D"], M)
    if kw["D"] == 166:
        assert top == 65535 - 148 * M
    for ne, ok in ((top, True), (top + 1, False)):
        nbs = [ne // M + (m < ne % M) for m in range(M)]
        assert sum(nbs) == ne
        for call, ws in ((fwd, fwd_ws), (bwd, bwd_ws)):
            need = ws(lib, ps, M, nbs, 2)
            if ok:
                assert need > 0
                assert call(lib, ps, M, nbs, 2, wsb=need - 1) == ERR_WORKSPACE
            else:
                assert need == 0
                assert call(lib, ps, M, nbs, 2) == ERR_ARG and "chunk capacity" in last_error(lib)


@pytest.mark.parametrize("kw", GENERIC)
def test_workspace_sizes(kw):
    lib = _lib.load()
    for f, one in ((fwd_ws, lib.dsmil_generic_forward_bags_train_dev_workspace_bytes),
                   (bwd_ws, lib.dsmil_generic_backward_bags_dev_workspace_bytes)):
        prev = 0
        for M in (1, 2, 5, 8):
            ps = arr([params(**kw)] * M)
            nbs = [4 + m % 3 for m in range(M)]
            got = f(lib, ps, M, nbs, 500)
            assert got > prev
            prev = got
            assert f(lib, ps, M, [n + 4 for n in nbs], 500) > got
            assert f(lib, ps, M, nbs, 900) > got
            for mr in (1, 129, 500):
                got = f(lib, ps, M, nbs, mr)
                assert got >= sum(one(C.byref(ps[m]), nbs[m], mr) for m in range(M))


# ---- the generic fold planner's forward table: one definition on the host and the device -------------------------
PROBE = r"""
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "bag_plan.cuh"
namespace dsmil { void set_error(const char*, ...) {} int cuda_fail(cudaError_t, const char*) { return -3; }
                  void count_launch(int) {} void prof_begin_impl(int, cudaStream_t) {}
                  void prof_end_impl(int, cudaStream_t) {} }
using namespace dsmil;
// D mode max_rows then per model: nb N...  ("-" separates models); prints each entry as k_plan_bags_models numbers
// it for the generic forward, with each model's tiles numbered across the models (mode 1) or from 0 (mode 2)
int main(int argc, char** argv) {
  const int D = atoi(argv[1]), mode = atoi(argv[2]);
  const long long max_rows = atoll(argv[3]);
  std::vector<std::vector<int64_t>> models(1);
  for (int i = 4; i < argc; ++i) {
    if (argv[i][0] == '-') models.emplace_back();
    else models.back().push_back(atoll(argv[i]));
  }
  int tile_all = 0, rec_all = 0, e0 = 0;
  const float* X = reinterpret_cast<const float*>(uintptr_t(0x10000));
  for (size_t m = 0; m < models.size(); ++m) {
    long long row = max_rows * e0;
    int tile = mode == FOLD_GEN_QMLP ? 0 : tile_all, rec = rec_all;
    const int t0 = tile;
    for (int64_t N : models[m]) {
      sm90::BagDev e = gen_bag_entry(X, N, D, row, tile, rec);
      e.pad_ = fold_pad(e.pad_, (int)m);
      printf("%lld %d %d %d %d %d\n", e.row_off, e.tile_off, e.rec_off, e.nrec, fold_pad_mode(e.pad_),
             fold_pad_model(e.pad_));
    }
    tile_all += tile - t0;
    rec_all = rec;
    e0 += (int)models[m].size();
  }
  return 0;
}
"""


def restated_table(D, mode, max_rows, models):
    """The generic fold forward's table: model m's bags at its capacity block (max_rows * its first entry), its own
    live prefix sums inside; 128-row tiles and attend records (one per 32-row tile up to kSplits) numbered across the
    models, tiles from 0 per model in the k_qmlp_sm90 form; the k_scores MODE of 16-byte aligned rows, the model."""
    out, e0, tile_all, rec_all = [], 0, 0, 0
    smode = 2 if D % 64 == 0 else (1 if D % 4 == 0 else 0)
    for m, Ns in enumerate(models):
        row, tile, rec = max_rows * e0, (0 if mode == 2 else tile_all), rec_all
        for N in Ns:
            nrec = min(max(ceil_div(N, 32), 1), K_SPLITS)
            out.append((row, tile, rec, nrec, smode, m))
            row, tile, rec = row + N, tile + ceil_div(N, 128), rec + nrec
        tile_all += sum(ceil_div(N, 128) for N in Ns)
        rec_all = rec
        e0 += len(Ns)
    return out


def test_generic_fold_table_matches_a_restatement(tmp_path):
    src, exe = tmp_path / "probe.cu", tmp_path / "probe"
    src.write_text(PROBE)
    r = subprocess.run([build._nvcc(), "-std=c++17", "-O1", *build.ARCH, "-I", build.CSRC,
                        "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    rng = random.Random(11)
    cases = [(166, 1, 40, [[2, 40, 7], [1]]), (230, 1, 13, [[13], [2, 3], [12, 12, 1]]),
             (512, 2, 9473, [[1, 127, 128, 129], [9472, 9473]]), (2049, 1, 9473, [[9473], [1, 9472]])]
    for _ in range(10):
        M = rng.choice([1, 2, 5, 8])
        mr = rng.choice([40, 200, 9473])
        cases.append((rng.choice([166, 230, 512, 2049]), rng.choice([1, 2]), mr,
                      [[rng.randint(1, mr) for _ in range(rng.randint(1, 6))] for _ in range(M)]))
    for D, mode, mr, models in cases:
        args = [str(D), str(mode), str(mr)]
        for m, Ns in enumerate(models):
            args += (["-"] if m else []) + [str(n) for n in Ns]
        r = subprocess.run([str(exe), *args], capture_output=True, text=True)
        assert r.returncode == 0, (D, models)
        got = [tuple(int(v) for v in line.split()) for line in r.stdout.split("\n") if line.strip()]
        assert got == restated_table(D, mode, mr, models), (D, mode, mr, models)


# ---- Python refusals (raised before any device work) ---------------------------------------------------------------
def _net(D=166, C_=1, nonlinear=True):
    return mil.MILNet(mil.FCLayer(D, C_), mil.BClassifier(D, C_, nonlinear=nonlinear))


def _sgd(net):
    return torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9)


def test_fold_step_shape_routes():
    assert fold_step_shape([_net(), _net()], generic=True) == (166, 1)
    assert fold_step_shape([_net(230, 2, False)] * 3, generic=True) == (230, 2)
    assert fold_step_shape([_net(512, 2)] * 2, generic=True) == (512, 2)       # the fused fold step
    with pytest.raises(ValueError, match="D=166"):
        fold_step_shape([_net(), _net()])
    with pytest.raises(ValueError, match="M=6, D=2048"):
        fold_step_shape([_net(2048, 2)] * 6, generic=True)


def test_generic_fold_graph_refuses_what_it_cannot_record():
    crit = torch.nn.BCEWithLogitsLoss()
    nets = [_net(), _net()]
    opts = [_sgd(n) for n in nets]
    with pytest.raises(ValueError, match="capturable"):
        FoldTrainStepGraph(nets, crit, [opts[0], torch.optim.Adam(nets[1].parameters())], [1, 1], 40, generic=True)
    with pytest.raises(ValueError, match="group sizes"):
        FoldTrainStepGraph(nets, crit, opts, [1, 0], 40, generic=True)
    with pytest.raises(ValueError, match="max_rows=0"):
        FoldTrainStepGraph(nets, crit, opts, [1, 1], 0, generic=True)
    with pytest.raises(ValueError, match="1 to 8 folds"):
        FoldTrainStepGraph([nets[0]] * 9, crit, [opts[0]] * 9, [1] * 9, 40, generic=True)
    for other in (_net(230), _net(166, 2)):
        with pytest.raises(ValueError, match="fold 1"):
            FoldTrainStepGraph([nets[0], other], crit, [opts[0], _sgd(other)], [1, 1], 40, generic=True)
    lin = _net(nonlinear=False)
    with pytest.raises(ValueError, match="fold 1: nonlinear=False"):
        FoldTrainStepGraph([nets[0], lin], crit, [opts[0], _sgd(lin)], [1, 1], 40, generic=True)
    pv = [mil.MILNet(mil.FCLayer(166, 1), mil.BClassifier(166, 1, passing_v=True)) for _ in range(2)]
    with pytest.raises(ValueError, match="identity v"):
        FoldTrainStepGraph(pv, crit, [_sgd(n) for n in pv], [1, 1], 40, generic=True)
    wide = [_net(2048, 2) for _ in range(6)]
    with pytest.raises(ValueError, match="M=6, D=2048"):
        FoldTrainStepGraph(wide, crit, [_sgd(n) for n in wide], [1] * 6, 100, generic=True)


def _store(D, Ns, C_=1):
    store = feed.DeviceBagStore(D, device="cpu")
    for n in Ns:
        store.add_bag(torch.rand(n, D), torch.zeros(C_))
    return store


def test_generic_fold_graph_epoch_refuses_a_bag_over_capacity_before_any_step():
    nets = [_net(), _net()]
    opts = [_sgd(n) for n in nets]
    store = _store(166, [10, 40, 5])
    crit = torch.nn.BCEWithLogitsLoss()
    with pytest.raises(ValueError, match="fold 1, bag 1: 40 rows exceed .*max_rows=30"):
        feed.train_epoch_models(nets, store, [[0, 2], [1, 2]], crit, opts, graph=True, max_rows=30, generic=True)
    with pytest.raises(ValueError, match="max_rows=20"):
        feed.train_epoch_models(nets, store, [[0, 2], [1, 2]], crit, opts, dropout_patch=0.4, graph=True,
                                max_rows=20, generic=True)
    with pytest.raises(ValueError, match="D=166, C=1"):       # without generic=True the shape is refused
        feed.train_epoch_models(nets, store, [[0], [1]], crit, opts, graph=True)
