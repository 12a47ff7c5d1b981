"""The capture-safe fold step without a GPU: argument validation and workspace sizes of
dsmil_forward_bags_models_train_dev / dsmil_backward_bags_models_dev (calls that return before any CUDA work), the
per-model plan formulas shared by the host and the device planner against a Python restatement, and the refusals of
FoldTrainStepGraph and feed.train_epoch_models(graph=True) that come before any device work."""
import ctypes as C
import os
import random
import re
import subprocess

import pytest
import torch

import dsmil as mil
from dsmil_wsi_b200 import _lib, build, feed
from dsmil_wsi_b200.train_graph import FoldTrainStepGraph

ERR_ARG, ERR_WORKSPACE = -1, -2
FAKE = 0x10000          # a non-NULL, 16-byte aligned "device pointer": never dereferenced on these paths
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("dsmil_forward_bags_models_train_dev_workspace_bytes", "dsmil_forward_bags_models_train_dev",
         "dsmil_backward_bags_models_dev_workspace_bytes", "dsmil_backward_bags_models_dev")


def params(D=512, C_=2, nonlinear=1, passing_v=0, **over):
    p = _lib.DsmilParams(D, C_, nonlinear, passing_v)
    for name in ("Wi", "bi", "W1", "b1", "W2", "b2", "Wv", "bv", "Wf", "bf"):
        setattr(p, name, FAKE)
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
    return lib.dsmil_forward_bags_models_train_dev(ps, M, b[0], b[1], None if nbs is None else i32(nbs), max_rows,
                                                   *b[2:], ws, wsb, None)


def bwd(lib, ps, M, nbs, max_rows=1000, ws=FAKE, wsb=1 << 40, null=None, dA=None, dB=None, gX=None, g="default"):
    # Xs, Ns, Q, H1, A, B, crit, d_classes, d_pred, status
    b = [None if i == null else FAKE for i in range(10)]
    g = grads(max(M, 1), gX) if g == "default" else g
    return lib.dsmil_backward_bags_models_dev(ps, M, b[0], b[1], None if nbs is None else i32(nbs), max_rows, *b[2:9],
                                              dA, dB, g, b[9], ws, wsb, None)


def fwd_ws(lib, ps, M, nbs, max_rows=1000):
    return lib.dsmil_forward_bags_models_train_dev_workspace_bytes(ps, M, i32(nbs), max_rows)


def bwd_ws(lib, ps, M, nbs, max_rows=1000):
    return lib.dsmil_backward_bags_models_dev_workspace_bytes(ps, M, i32(nbs), max_rows)


def test_symbols_exported_declared_and_bound():
    lib = _lib.load()
    header = open(os.path.join(ROOT, "include", "dsmil_b200.h")).read()
    for name in NAMES:
        assert re.search(rf"\b{name}\s*\(", header), name
        assert hasattr(lib, name), name
        assert name in _lib.SIGNATURES, name
    assert lib.dsmil_abi_version() == 1


@pytest.mark.parametrize("call,ws", [(fwd, fwd_ws), (bwd, bwd_ws)])
def test_fold_dev_entry_point_validation(call, ws):
    lib = _lib.load()
    two = arr([params(), params()])
    assert call(lib, None, 2, [1, 1]) == ERR_ARG and "params is NULL" in last_error(lib)
    nine = arr([params() for _ in range(9)])
    for M in (0, 9, -1):
        assert call(lib, nine, M, [1] * 9) == ERR_ARG and "M=" in last_error(lib)
        assert ws(lib, nine, M, [1] * 9) == 0
    # members of different D / C / q form
    for other in (dict(D=1024), dict(C_=1), dict(nonlinear=0, W2=None, b2=None)):
        ps = arr([params(), params(**other)])
        assert call(lib, ps, 2, [1, 1]) == ERR_ARG and "model 1" in last_error(lib)
        assert ws(lib, ps, 2, [1, 1]) == 0
    # shapes off dsmil_models_supported
    for M, kw in ((2, dict(C_=5)), (2, dict(nonlinear=0)), (2, dict(D=166, C_=1)), (6, dict(D=2048, C_=2)),
                  (2, dict(passing_v=1))):
        ps = arr([params(**kw) for _ in range(M)])
        assert not lib.dsmil_models_supported(ps, M)
        assert call(lib, ps, M, [1] * M) == ERR_ARG and "not supported" in last_error(lib), kw
        assert ws(lib, ps, M, [1] * M) == 0
    assert lib.dsmil_models_supported(arr([params(D=2048, C_=2)] * 5), 5)
    # group sizes, in all and each
    for nbs in ([0, 1], [1, 0], [2, -1], [40000, 25536], [65536, 1]):
        assert call(lib, two, 2, nbs) == ERR_ARG, nbs
        assert ws(lib, two, 2, nbs) == 0
    assert call(lib, two, 2, None) == ERR_ARG
    for mr in (0, -5, 1 << 32):
        assert call(lib, two, 2, [2, 3], max_rows=mr) == ERR_ARG and "max_rows" in last_error(lib)
        assert ws(lib, two, 2, [2, 3], mr) == 0
    assert call(lib, two, 2, [30000, 30000], max_rows=1 << 31) == ERR_ARG      # tiles past an int
    # the bag list and the status words (last) are always required; so is every other buffer of the forward and
    # the saved activations of the backward
    for null in (0, 1, 9) + tuple(range(2, 9 if call is fwd else 7)):
        assert call(lib, two, 2, [2, 3], null=null) == ERR_ARG, null
    need = ws(lib, two, 2, [2, 3])
    assert need > 0
    assert call(lib, two, 2, [2, 3], wsb=need - 1) == ERR_WORKSPACE and "workspace too small" in last_error(lib)
    assert call(lib, two, 2, [2, 3], ws=None) == ERR_WORKSPACE


def test_fold_dev_backward_refuses_upstream_A_B_features_and_null_grads():
    lib = _lib.load()
    two = arr([params(), params()])
    assert bwd(lib, two, 2, [1, 2], dA=FAKE) == ERR_ARG and "d_A" in last_error(lib)
    assert bwd(lib, two, 2, [1, 2], dB=FAKE) == ERR_ARG
    assert bwd(lib, two, 2, [1, 2], gX=FAKE) == ERR_ARG
    g = grads(2)
    g[1].gX = FAKE                                            # any one member's gX
    assert bwd(lib, two, 2, [1, 2], g=g) == ERR_ARG
    assert bwd(lib, two, 2, [1, 2], g=None) == ERR_ARG


@pytest.mark.parametrize("D,C_", [(512, 2), (1024, 4), (2048, 1)])
def test_fold_dev_workspace_sizes(D, C_):
    lib = _lib.load()
    for f, eager, one in ((fwd_ws, lib.dsmil_forward_bags_models_train_workspace_bytes,
                           lib.dsmil_forward_bags_train_dev_workspace_bytes),
                          (bwd_ws, lib.dsmil_backward_bags_models_workspace_bytes,
                           lib.dsmil_backward_bags_dev_workspace_bytes)):
        prev = 0
        for M in (1, 2, 5, 8):
            ps = arr([params(D, C_)] * M)
            if not lib.dsmil_models_supported(ps, M):
                assert f(lib, ps, M, [2] * M) == 0
                continue
            nbs = [4 + m % 3 for m in range(M)]
            got = f(lib, ps, M, nbs, 5000)
            assert got > prev                                                   # grows with M
            prev = got
            assert f(lib, ps, M, [n + 4 for n in nbs], 5000) > got               # with the bags
            assert f(lib, ps, M, nbs, 9000) > got                                # and with the row capacity
            for mr in (1, 129, 5000, 12000):
                got = f(lib, ps, M, nbs, mr)
                Ns = (C.c_int64 * sum(nbs))(*[mr] * sum(nbs))
                extra = () if f is fwd_ws else (0,)
                assert got >= eager(ps, M, Ns, i32(nbs), *extra)
                assert got >= sum(one(C.byref(ps[m]), nbs[m], mr) for m in range(M))


# ---- the per-model plan: one definition for the host plan and the device planner -----------------------------------
K_SPLITS, TBM, TBK, K_SMS, KQ = 296, 128, 16, 132, 128


def ceil_div(a, b):
    return -(-a // b)


def model_plan(C_, D, Ns, r0):
    """What plan_bwd_models chose for one model of bags Ns whose packed rows start at r0."""
    nb, total = len(Ns), sum(Ns)
    gemv = C_ <= 4 and D % 4 == 0 and D // 4 <= 256

    def rps(M1, gemv):
        if gemv:
            return max(ceil_div(total, K_SPLITS), 64)
        s = max(1, K_SPLITS // (ceil_div(M1, TBM) * ceil_div(D, TBM)))
        return max(ceil_div(ceil_div(total, s), TBK) * TBK, 128)

    def rag(r):
        out, row = [], r0
        for N in Ns:
            out += [(row + lo, min(r, N - lo)) for lo in range(0, N, r)]
            row += N
        return out

    def split(S, r):
        return [(r0 + z * r, min(total, z * r + r) - z * r) for z in range(S)]

    S2 = max(1, min(K_SPLITS, ceil_div(total, 128)))
    Sc = max(1, min(ceil_div(total, 64), K_SPLITS))
    return dict(G=max(1, min(ceil_div(K_SMS * 8, nb), ceil_div(max(Ns), 64))), chi=rag(rps(C_, gemv)),
                ch1=rag(rps(KQ, False)), ch2=split(S2, ceil_div(ceil_div(total, S2), TBK) * TBK),
                chc=split(Sc, ceil_div(total, Sc)))


PROBE = r"""
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "bag_plan.cuh"
namespace dsmil { void set_error(const char*, ...) {} int cuda_fail(cudaError_t, const char*) { return -3; }
                  void count_launch(int) {} void prof_begin_impl(int, cudaStream_t) {}
                  void prof_end_impl(int, cudaStream_t) {} }
using namespace dsmil;
int main(int argc, char** argv) {   // C D r0 N...
  const int C = atoi(argv[1]), D = atoi(argv[2]);
  const long long r0 = atoll(argv[3]);
  std::vector<int64_t> Ns;
  for (int i = 4; i < argc; ++i) Ns.push_back(atoll(argv[i]));
  const int nb = (int)Ns.size();
  int64_t total = 0, mx = 1;
  for (int64_t n : Ns) { total += n; mx = n > mx ? n : mx; }
  const ModelSplits sp = model_splits(C, D, nb, total, mx);
  std::vector<const float*> Xs(nb, nullptr);
  const BagList L{Xs.data(), Ns.data(), nullptr};
  printf("G %d\n", sp.G);
  const int64_t rps[2] = {sp.rps_i, sp.rps_1};
  for (int t = 0; t < 2; ++t) {
    std::vector<TnChunk> ch(rag_chunks_list(L, nb, D, rps[t], r0, nullptr));
    rag_chunks_list(L, nb, D, rps[t], r0, ch.data());
    if ((int)ch.size() > rag_chunks_cap(t ? 128 : C, D, t ? false : tn_use_gemv(C, D), nb)) return 3;
    for (const TnChunk& c : ch) printf("%s %lld %lld\n", t ? "ch1" : "chi", c.prow, c.rows);
  }
  if (sp.t2.S > kModelSplitsCap || sp.cs.S > kModelSplitsCap) return 3;
  for (int z = 0; z < sp.t2.S; ++z) { const TnChunk c = split_chunk(sp.t2, z, r0, nullptr, 0); printf("ch2 %lld %lld\n", c.prow, c.rows); }
  for (int z = 0; z < sp.cs.S; ++z) { const TnChunk c = split_chunk(sp.cs, z, r0, nullptr, 0); printf("chc %lld %lld\n", c.prow, c.rows); }
  return 0;
}
"""


def test_per_model_plan_formulas_match_the_host_plan_they_replaced(tmp_path):
    """bag_plan.cuh's model_splits / rag_chunks_list / split_chunk, which plan_bwd_models and k_plan_bags_models both
    call, built for the host and run on seeded ragged lists, against the arithmetic plan_bwd_models had inline."""
    src, exe = tmp_path / "probe.cu", tmp_path / "probe"
    src.write_text(PROBE)
    r = subprocess.run([build._nvcc(), "-std=c++17", "-O1", *build.ARCH, "-I", build.CSRC,
                        "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    rng = random.Random(7)
    cases = [(2, 512, 0, [1]), (2, 512, 40000, [10000]), (4, 1024, 7, [1, 127, 128, 129]), (1, 2048, 0, [18943, 1]),
             (2, 512, 3 * 12000, [64 * K_SPLITS, 1]), (2, 512, 0, [64 * K_SPLITS + 1]), (4, 1536, 5, [128 * 74 + 1, 9])]
    for _ in range(12):
        nb = rng.choice([1, 2, 5, 16])
        cases.append((rng.choice([1, 2, 3, 4]), rng.choice([512, 1024, 2048]), rng.randrange(0, 10 ** 6),
                      [rng.choice([1, 63, 64, 65, 500, 4097, 12000]) for _ in range(nb)]))
    for C_, D, r0, Ns in cases:
        r = subprocess.run([str(exe), str(C_), str(D), str(r0), *map(str, Ns)], capture_output=True, text=True)
        assert r.returncode == 0, (C_, D, Ns)
        got = dict(chi=[], ch1=[], ch2=[], chc=[])
        for line in r.stdout.split("\n"):
            f = line.split()
            if f and f[0] == "G":
                got["G"] = int(f[1])
            elif f:
                got[f[0]].append((int(f[1]), int(f[2])))
        assert got == model_plan(C_, D, Ns, r0), (C_, D, r0, Ns)


# ---- Python refusals (raised before any device work) ---------------------------------------------------------------
def _net(D=512, C_=2, nonlinear=True):
    return mil.MILNet(mil.FCLayer(D, C_), mil.BClassifier(D, C_, nonlinear=nonlinear))


def _sgd(net):
    return torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9)


def test_fold_graph_refuses_what_it_cannot_record():
    crit = torch.nn.BCEWithLogitsLoss()
    nets = [_net(), _net()]
    for bad in (torch.optim.RMSprop(nets[1].parameters()), torch.optim.Adam(nets[1].parameters()),
                torch.optim.SGD(nets[1].parameters(), lr=0.1, momentum=0.9, dampening=0.5)):
        with pytest.raises(ValueError, match="capturable|capture-safe|dampening"):
            FoldTrainStepGraph(nets, crit, [_sgd(nets[0]), bad], [1, 1], 100)
    opts = [_sgd(n) for n in nets]
    with pytest.raises(ValueError, match="2 milnets, 1 optimizers"):
        FoldTrainStepGraph(nets, crit, opts[:1], [1, 1], 100)
    with pytest.raises(ValueError, match="3 group sizes"):
        FoldTrainStepGraph(nets, crit, opts, [1, 1, 1], 100)
    with pytest.raises(ValueError, match="group sizes"):
        FoldTrainStepGraph(nets, crit, opts, [1, 0], 100)
    with pytest.raises(ValueError, match="max_rows=0"):
        FoldTrainStepGraph(nets, crit, opts, [1, 1], 0)
    with pytest.raises(ValueError, match="1 to 8 folds"):
        FoldTrainStepGraph([nets[0]] * 9, crit, [opts[0]] * 9, [1] * 9, 100)
    other = _net(1024)
    with pytest.raises(ValueError, match="fold 1"):
        FoldTrainStepGraph([nets[0], other], crit, [opts[0], _sgd(other)], [1, 1], 100)
    for kw in (dict(D=166, C_=1), dict(nonlinear=False), dict(C_=8)):
        off = [_net(**kw), _net(**kw)]
        with pytest.raises(ValueError, match="D="):
            FoldTrainStepGraph(off, crit, [_sgd(n) for n in off], [1, 1], 100)
    wide = [_net(2048) for _ in range(6)]                      # each on the batched path, six not in shared memory
    with pytest.raises(ValueError, match="M=6, D=2048"):
        FoldTrainStepGraph(wide, crit, [_sgd(n) for n in wide], [1] * 6, 100)


def _store(D, Ns, C_=2):
    store = feed.DeviceBagStore(D, device="cpu")
    for n in Ns:
        store.add_bag(torch.rand(n, D), torch.zeros(C_))
    return store


def test_fold_graph_epoch_refuses_a_bag_over_capacity_before_any_step():
    nets = [_net(), _net()]
    opts = [_sgd(n) for n in nets]
    store = _store(512, [100, 300, 50])
    crit = torch.nn.BCEWithLogitsLoss()
    with pytest.raises(ValueError, match="fold 1, bag 1: 300 rows exceed .*max_rows=200"):
        feed.train_epoch_models(nets, store, [[0, 2], [1, 2]], crit, opts, graph=True, max_rows=200)
    # with patch dropout the kept rows count: 300 * 0.6 = 180 fits 200, not 150
    with pytest.raises(ValueError, match="max_rows=150"):
        feed.train_epoch_models(nets, store, [[0, 2], [1, 2]], crit, opts, dropout_patch=0.4, graph=True,
                                max_rows=150)
    off = [_net(166, 1), _net(166, 1)]
    with pytest.raises(ValueError, match="D=166, C=1"):
        feed.train_epoch_models(off, _store(166, [10, 20], 1), [[0], [1]], crit, [_sgd(n) for n in off], graph=True)
