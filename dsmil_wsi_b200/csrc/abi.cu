// extern "C" entry points of libdsmil_b200.so (see include/dsmil_b200.h for the contract and the
// reference spans each call replaces).  Host orchestration only; kernels live in *_kernels.cuh
// and fwd_sm90.cuh.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <vector>
#include <algorithm>
#include <climits>

#include "common.cuh"
#include "gemm_generic.cuh"
#include "fwd_kernels.cuh"
#include "bwd_kernels.cuh"
#include "bwd_bags.cuh"
#include "fwd_sm90.cuh"
#include "fwd_batched.cuh"
#include "bag_plan.cuh"
#include "fwd_generic_b.cuh"
#include "embed_kernels.cuh"
#include "jpeg_kernels.cuh"

namespace dsmil {

static thread_local char g_err[512] = "";
__device__ unsigned long long scratch_keys[kMaxC];  // sink for k_scores' arg-max by-product
static std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) at %s", static_cast<int>(e), cudaGetErrorString(e), what);
  return DSMIL_ERR_CUDA;
}
void count_launch(int n) { g_launches.fetch_add(static_cast<uint64_t>(n), std::memory_order_relaxed); }

// train_tcga.py:78-83 dropout_patches: `feats[random_indices]` -- a row gather.  One warp per output row.
__global__ void __launch_bounds__(256)
k_gather_rows(const float* __restrict__ X, int D, const long long* __restrict__ idx, long long M,
              float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long stride = static_cast<long long>(gridDim.x) * 8;
  const bool vec = (D % 4 == 0) && ((reinterpret_cast<uintptr_t>(X) & 15) == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
  for (long long m = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5); m < M; m += stride) {
    const float* src = X + idx[m] * D;
    float* dst = out + m * D;
    if (vec) {
      for (int j = lane; j < (D >> 2); j += 32)
        reinterpret_cast<float4*>(dst)[j] = __ldg(reinterpret_cast<const float4*>(src) + j);
    } else {
      for (int j = lane; j < D; j += 32) dst[j] = __ldg(src + j);
    }
  }
}



// compute_feats.py:19-46 (PIL -> VF.to_tensor): uint8 HWC -> float32 CHW, value / 255 (an IEEE division, as
// torchvision's `img.div(255)`), done on the device so that patches cross PCIe as bytes (4x less H2D traffic).
__global__ void __launch_bounds__(256)
k_u8hwc_to_f32chw(const uint8_t* __restrict__ in, long long B, int H, int W, int Cc, float* __restrict__ out) {
  const long long plane = static_cast<long long>(H) * W;
  const long long total = B * plane;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const long long b = i / plane, px = i % plane;
    const uint8_t* src = in + i * Cc;
    float* dst = out + b * Cc * plane + px;
    for (int c = 0; c < Cc; ++c) dst[c * plane] = __fdiv_rn(static_cast<float>(src[c]), 255.f);
  }
}

// ---- live kernel timing ------------------------------------------------------------------
bool g_prof_on = false;
struct ProfRec { int tag; cudaEvent_t a, b; };
static std::vector<ProfRec> g_prof;       // recorded pairs since the last read
static std::vector<ProfRec> g_prof_pool;  // recycled events
static int g_prof_open[PROF_NTAGS];
void prof_begin_impl(int tag, cudaStream_t st) {
  if (g_prof.size() >= 16384) { g_prof_open[tag] = -1; return; }
  ProfRec r;
  if (!g_prof_pool.empty()) { r = g_prof_pool.back(); g_prof_pool.pop_back(); }
  else { if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) { g_prof_open[tag] = -1; return; } }
  r.tag = tag;
  cudaEventRecord(r.a, st);
  g_prof_open[tag] = static_cast<int>(g_prof.size());
  g_prof.push_back(r);
}
void prof_end_impl(int tag, cudaStream_t st) {
  const int i = g_prof_open[tag];
  if (i >= 0 && i < static_cast<int>(g_prof.size())) cudaEventRecord(g_prof[i].b, st);
}

static int check_params(const dsmil_params_t* p, bool need_scores = false) {
  DSMIL_REQUIRE(p != nullptr, "params is NULL");
  DSMIL_REQUIRE(!need_scores || (p->Wi && p->bi), "NULL instance-classifier weights");
  DSMIL_REQUIRE(p->D >= 1 && p->D <= DSMIL_MAX_D, "feature size D=%d outside [1,%d]", p->D, DSMIL_MAX_D);
  DSMIL_REQUIRE(p->C >= 1 && p->C <= DSMIL_MAX_C, "output classes C=%d outside [1,%d]", p->C, DSMIL_MAX_C);
  DSMIL_REQUIRE(p->W1 && p->b1 && p->Wf && p->bf, "NULL weight pointer");
  DSMIL_REQUIRE(!p->nonlinear || (p->W2 && p->b2), "nonlinear q needs W2/b2");
  DSMIL_REQUIRE(!p->passing_v || (p->Wv && p->bv), "passing_v needs Wv/bv");
  return 0;
}

// 0 when the caller passed a workspace and the carve fits in it; else DSMIL_ERR_WORKSPACE with the size it needs
static int check_workspace(size_t need, bool ok, const void* ws, size_t cap) {
  if (ws && ok) return 0;
  set_error("workspace too small: need %zu bytes, got %zu", need, cap);
  return DSMIL_ERR_WORKSPACE;
}
// check_workspace against the size a *_workspace_bytes call reports
static int need_workspace(size_t need, const void* ws, size_t ws_bytes) {
  return check_workspace(need, ws_bytes >= need, ws, ws ? ws_bytes : 0);
}

// Bags of the batch and their rows; DSMIL_ERR_EMPTY for an empty bag, as dsmil_forward_bags.  Xs == NULL checks the
// row counts only (a phase that reads no features).
static int check_bags(const float* const* Xs, const int64_t* Ns, int nb, int64_t* total, bool* aligned) {
  *total = 0;
  *aligned = true;
  for (int b = 0; b < nb; ++b) {
    DSMIL_REQUIRE(Ns[b] >= 0 && Ns[b] < 0xffffffffll, "bag %d: N=%lld out of range", b, (long long)Ns[b]);
    if (Ns[b] == 0) {
      set_error("bag %d: empty bag (N == 0): the reference raises IndexError at dsmil.py:53", b);
      return DSMIL_ERR_EMPTY;
    }
    if (!Xs) {
      *total += Ns[b];
      continue;
    }
    DSMIL_REQUIRE(Xs[b], "bag %d: NULL features", b);
    *aligned = *aligned && (reinterpret_cast<uintptr_t>(Xs[b]) & 15) == 0;
    *total += Ns[b];
  }
  return 0;
}

static int num_sms() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return kSms;
  if (!cached[dev]) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = kSms;
    cached[dev] = n;
  }
  return cached[dev];
}

// ---- tensor-core phase 1 (k_qmlp_sm90) of nb bags: the single-bag, batched and sharded forwards share it ----------
struct Phase1Ws {
  sm90::BagDev* table;       // [nb]
  unsigned long long* keys;  // [nb][kMaxC] arg-max keys, then the nb finalize arrival counters and the nb phase-1
  unsigned int* counters;    // tile counts (one 8-byte slot per bag holds both): one memset per call zeroes all three
  unsigned int* done;
  uint8_t* wimg;             // bf16 weight images, 1024-byte aligned; NULL on shapes k_qmlp_sm90 does not take
};
static void carve_phase1(Carver& c, const dsmil_params_t* p, int nb, Phase1Ws& w) {
  w.table = c.take<sm90::BagDev>(nb);
  w.keys = c.take<unsigned long long>(static_cast<size_t>(nb) * (kMaxC + 1));
  w.counters = reinterpret_cast<unsigned int*>(w.keys ? w.keys + static_cast<size_t>(nb) * kMaxC : nullptr);
  w.done = w.counters ? w.counters + nb : nullptr;
  w.wimg = nullptr;
  if (sm90::qmlp_supported(p)) {
    const uintptr_t img = reinterpret_cast<uintptr_t>(c.take<uint8_t>(sm90::wimg_bytes(p->D) + 1024));
    w.wimg = reinterpret_cast<uint8_t*>((img + 1023) & ~uintptr_t(1023));
  }
}

// Host copy of the bag table: each bag's first row, 128-row tile and partial record, numbered across the batch
// (bag_entry, as the dev calls' planner numbers it).
static int build_table(const float* const* Xs, const int64_t* Ns, int nb, std::vector<sm90::BagDev>& tbl, int* tiles,
                       int* recs) {
  long long row = 0;
  int tile = 0, rec = 0;
  tbl.resize(nb);
  for (int b = 0; b < nb; ++b) {
    DSMIL_REQUIRE(Ns[b] >= 1 && Ns[b] < 0xffffffffll && Xs[b], "bag %d: empty or NULL", b);
    DSMIL_REQUIRE((reinterpret_cast<uintptr_t>(Xs[b]) & 15) == 0, "bag %d: features must be 16-byte aligned", b);
    tbl[b] = bag_entry(Xs[b], Ns[b], row, tile, rec);
  }
  *tiles = tile;
  *recs = rec;
  return 0;
}

// SMs the overlapped phase 1 leaves to the attend pass (forward_bags_impl).  H100 80GB HBM3 at a 700 W limit, 16 bags
// x 10 000 x 512, C = 2, best of three ms per step: 0 -> 0.335, 8 -> 0.329, 16 -> 0.326, 24 -> 0.322, 32 -> 0.310,
// 40 -> 0.301, 48 -> 0.315; the plain launch 0.365 (DESIGN §4.2, profiles/h100_fwd_overlap_1gpu.json).  A macro so
// that tools/bench_fwd_overlap.py can build the sweep's variants; the library is built with the default.
#ifndef DSMIL_PHASE1_RESERVE
#define DSMIL_PHASE1_RESERVE 40
#endif
constexpr int kPhase1Reserve = DSMIL_PHASE1_RESERVE;
static int overlap_phase1_ctas(int64_t tiles) {
  const int ctas = std::max(num_sms() - kPhase1Reserve, 1);
  return static_cast<int>(std::min<int64_t>(tiles, ctas));
}

// Scores (or, single bag only, the arg-max of the given scores classes_in), arg-max keys and Q (+ H1 when non-NULL)
// of the nb bags; *tiles and *recs return the batch's 128-row tiles and partial records.  upload == false leaves the
// table and the weight images as an earlier call with the same arguments wrote them into the same workspace.
// overlap: phase 1 runs on overlap_phase1_ctas CTAs and counts each bag's finished tiles into w.done, for a
// k_attend_b launched right after it with the same counters.
static int bags_phase1_impl(const dsmil_params_t* p, const Phase1Ws& w, const float* const* Xs, const int64_t* Ns,
                            int nb, const float* classes_in, float* classes, float* Q, float* H1, bool q_blocked,
                            bool upload, int* tiles, int* recs, cudaStream_t st, bool overlap = false) {
  std::vector<sm90::BagDev> tbl;
  int rc;
  if ((rc = build_table(Xs, Ns, nb, tbl, tiles, recs))) return rc;
  if (upload)
    DSMIL_CUDA_OK(cudaMemcpyAsync(w.table, tbl.data(), sizeof(sm90::BagDev) * nb, cudaMemcpyHostToDevice, st));
  DSMIL_CUDA_OK(cudaMemsetAsync(w.keys, 0, sizeof(unsigned long long) * (kMaxC + 1) * nb, st));
  if (upload && (rc = sm90::launch_prep_wimg(p, w.wimg, st))) return rc;
  if (classes_in) {
    const int grid = static_cast<int>(std::min<int64_t>(ceil_div(Ns[0], 256), kSplits));
    k_argmax<<<grid, 256, 0, st>>>(classes_in, Ns[0], p->C, w.keys);
    DSMIL_LAUNCH_OK("k_argmax");
  }
  return sm90::launch_qmlp(p, w.table, nb, *tiles, classes_in ? nullptr : classes, w.keys, Q, H1, w.wimg,
                           overlap ? overlap_phase1_ctas(*tiles) : num_sms(), st, q_blocked, nullptr,
                           overlap ? w.done : nullptr);
}

struct FwdWs : Phase1Ws {
  float *Q, *H1, *V, *cand, *qmax, *recs, *rec;
  int64_t* crit;
  size_t bytes;
};
static FwdWs carve_fwd(const dsmil_params_t* p, int64_t N, void* ws, size_t cap, bool* ok) {
  Carver c(ws, cap);
  FwdWs w;
  const int64_t n = N > 0 ? N : 1;
  carve_phase1(c, p, 1, w);
  w.Q = c.take<float>(n * kQ);
  w.H1 = p->nonlinear ? c.take<float>(n * kQ) : nullptr;
  w.V = p->passing_v ? c.take<float>(n * p->D) : nullptr;
  w.cand = c.take<float>(cand_floats(p->C));
  w.qmax = c.take<float>(static_cast<size_t>(p->C) * kQ);
  w.crit = c.take<int64_t>(kMaxC);
  w.recs = c.take<float>(static_cast<size_t>(attend_ctas(N)) * rec_floats(p->C, p->D));
  w.rec = c.take<float>(rec_floats(p->C, p->D));
  w.bytes = c.off;
  *ok = c.ok();
  return w;
}

// ---- phase 1: scores + arg-max key + Q-MLP (+V) + candidate record --------------------------

static int launch_scores(const dsmil_params_t* p, const float* X, int64_t N, float* classes,
                         unsigned long long* keys, cudaStream_t st) {
  const int C = p->C, D = p->D;
  const size_t smem = sizeof(float) * C * D;
  const int mode = scores_mode(X, D);
  const int grid = static_cast<int>(std::min<int64_t>(ceil_div(N, mode == 2 ? 64 : 8), kSms * 8));
  prof_begin(PROF_SCORES, st);
  if (mode == 2) {
    if (smem > 48 * 1024) DSMIL_CUDA_OK(cudaFuncSetAttribute(k_scores<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_scores<2><<<grid, 256, smem, st>>>(X, N, D, p->Wi, p->bi, C, classes, keys);
  } else if (mode == 1) {
    if (smem > 48 * 1024) DSMIL_CUDA_OK(cudaFuncSetAttribute(k_scores<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_scores<1><<<grid, 256, smem, st>>>(X, N, D, p->Wi, p->bi, C, classes, keys);
  } else {
    if (smem > 48 * 1024) DSMIL_CUDA_OK(cudaFuncSetAttribute(k_scores<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_scores<0><<<grid, 256, smem, st>>>(X, N, D, p->Wi, p->bi, C, classes, keys);
  }
  prof_end(PROF_SCORES, st);
  DSMIL_LAUNCH_OK("k_scores");
  return 0;
}

// Under stream capture (CUDA-graph serving loops) the pageable host->device copies of the bag table cannot be
// recorded; the captured call then reuses the table that the preceding EAGER call with the same arguments wrote into
// the same workspace (dsmil_wsi_b200.sharded.ShardedBagsGraph does exactly that: warm-up run, then capture).
static bool stream_is_capturing(cudaStream_t st) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  return cudaStreamIsCapturing(st, &cs) == cudaSuccess && cs != cudaStreamCaptureStatusNone;
}

// Whether a single-bag phase 1 runs on k_qmlp_sm90, which keeps H1 in registers; the generic path writes it out.
static bool phase1_on_qmlp(const dsmil_params_t* p, const uint8_t* wimg, const float* X) {
  return sm90::qmlp_supported(p) && wimg && (reinterpret_cast<uintptr_t>(X) & 15) == 0;
}

static int phase1_impl(const dsmil_params_t* p, const float* X, const float* xv, const float* classes_in,
                       int64_t N, int64_t row_offset, float* classes, float* Q, float* H1, float* V,
                       float* cand, const Phase1Ws& w, cudaStream_t st) {
  const int C = p->C, D = p->D;
  int rc;
  if (N > 0 && classes_in && classes && classes != classes_in)
    DSMIL_CUDA_OK(cudaMemcpyAsync(classes, classes_in, sizeof(float) * N * C, cudaMemcpyDeviceToDevice, st));
  if (N > 0 && phase1_on_qmlp(p, w.wimg, X)) {
    // tensor-core path: scores + arg-max + Q-MLP in one persistent kernel
    int tiles, recs;
    if ((rc = bags_phase1_impl(p, w, &X, &N, 1, classes_in, classes, Q, H1, false, true, &tiles, &recs, st))) return rc;
  } else {
    DSMIL_CUDA_OK(cudaMemsetAsync(w.keys, 0, sizeof(unsigned long long) * kMaxC, st));
    if (N > 0) {
      if (classes_in) {   // bag form: arg-max of the given scores
        const int grid = static_cast<int>(std::min<int64_t>(ceil_div(N, 256), kSplits));
        k_argmax<<<grid, 256, 0, st>>>(classes_in, N, C, w.keys);
        DSMIL_LAUNCH_OK("k_argmax");
      } else if ((rc = launch_scores(p, X, N, classes, w.keys, st))) {
        return rc;
      }
      prof_begin(PROF_QMLP, st);
      if (p->nonlinear) {
        if ((rc = launch_linear<ACT_RELU, false>(X, N, D, p->W1, p->b1, kQ, H1, nullptr, 0, st))) return rc;
        if ((rc = launch_linear<ACT_TANH, false>(H1, N, kQ, p->W2, p->b2, kQ, Q, nullptr, 0, st))) return rc;
      } else {
        if ((rc = launch_linear<ACT_NONE, false>(X, N, D, p->W1, p->b1, kQ, Q, nullptr, 0, st))) return rc;
      }
      prof_end(PROF_QMLP, st);
    }
  }
  if (N > 0 && p->passing_v &&
      (rc = launch_linear<ACT_RELU, false>(xv ? xv : X, N, D, p->Wv, p->bv, D, V, nullptr, 0, st)))
    return rc;
  const float* cls = classes_in ? classes_in : classes;
  k_gather_cand<<<C, kQ, 0, st>>>(w.keys, cls, Q, N, C, row_offset, cand);
  DSMIL_LAUNCH_OK("k_gather_cand");
  return 0;
}

__global__ void k_empty_rec(float* rec, int C, int Dv) {
  const size_t n = rec_floats(C, Dv);
  for (size_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x)
    rec[i] = (i < static_cast<size_t>(C)) ? -INFINITY : 0.f;
}

template <int CT>
static int launch_attend_j(int J, int grid, cudaStream_t st, const float* V, int Dv, const float* Q, int64_t N,
                           const float* qmax, int C, float* A, float* recs) {
  switch (J) {
    case 1: k_attend<CT, 1><<<grid, 256, 0, st>>>(V, Dv, Q, N, qmax, C, A, recs); break;
    case 2: k_attend<CT, 2><<<grid, 256, 0, st>>>(V, Dv, Q, N, qmax, C, A, recs); break;
    case 4: k_attend<CT, 4><<<grid, 256, 0, st>>>(V, Dv, Q, N, qmax, C, A, recs); break;
    case 8: k_attend<CT, 8><<<grid, 256, 0, st>>>(V, Dv, Q, N, qmax, C, A, recs); break;
    default: k_attend<CT, 16><<<grid, 256, 0, st>>>(V, Dv, Q, N, qmax, C, A, recs); break;
  }
  DSMIL_LAUNCH_OK("k_attend");
  return 0;
}

// ---- phase 2: logits -> A (unnormalised), device-level (m, s, Bp) record ------------------------
static int phase2_impl(const dsmil_params_t* p, const float* V, const float* Q, int64_t N, const float* qmax,
                       float* A, float* rec, float* recs, cudaStream_t st) {
  const int C = p->C, Dv = p->D;
  if (N <= 0) {
    k_empty_rec<<<4, 256, 0, st>>>(rec, C, Dv);
    DSMIL_LAUNCH_OK("k_empty_rec");
    return 0;
  }
  const int grid = attend_ctas(N);
  int j = ceil_div(Dv, 256), J = 1;
  while (J < j) J <<= 1;
  int rc;
  prof_begin(PROF_ATTEND, st);
  if (C == 1) rc = launch_attend_j<1>(J, grid, st, V, Dv, Q, N, qmax, C, A, recs);
  else if (C == 2) rc = launch_attend_j<2>(J, grid, st, V, Dv, Q, N, qmax, C, A, recs);
  else if (C <= 4) rc = launch_attend_j<4>(J, grid, st, V, Dv, Q, N, qmax, C, A, recs);
  else rc = launch_attend_j<8>(J, grid, st, V, Dv, Q, N, qmax, C, A, recs);
  prof_end(PROF_ATTEND, st);
  if (rc) return rc;
  dim3 g2(C, ceil_div(Dv, 256));
  k_combine_rec<<<g2, 256, 0, st>>>(recs, grid, C, Dv, rec);
  DSMIL_LAUNCH_OK("k_combine_rec");
  return 0;
}

static int phase3_impl(const dsmil_params_t* p, int64_t N, const float* rec, float* A, float* B, float* pred,
                       cudaStream_t st) {
  const int grid = static_cast<int>(std::min<int64_t>(std::max<int64_t>(ceil_div(N * p->C, 256), 1), kSplits));
  prof_begin(PROF_FINAL, st);
  k_finalize<<<grid, 256, 0, st>>>(rec, N, p->C, p->D, p->Wf, p->bf, A, B, pred);
  prof_end(PROF_FINAL, st);
  DSMIL_LAUNCH_OK("k_finalize");
  return 0;
}

// ---- batched forward: a stream of bags in a handful of launches (tensor-core path only) -----------
struct BagsWs : Phase1Ws {
  float* Q;
  float* recs;
  float* pred_part;
  long long* row_offsets;   // row-sharded batch only: [nb] device copy
  float* qmax;              // row-sharded batch only: [nb][C][128]
  size_t bytes;
};
static BagsWs carve_bags(const dsmil_params_t* p, const int64_t* Ns, int nb, bool need_Q, bool sharded, void* ws,
                         size_t cap, bool* ok) {
  Carver c(ws, cap);
  BagsWs w;
  int64_t tiles = 0, nrec = 0;
  for (int b = 0; b < nb; ++b) {
    tiles += tiles_for_bag(Ns[b]);
    nrec += recs_for_bag(Ns[b]);
  }
  carve_phase1(c, p, nb, w);
  w.pred_part = c.take<float>(static_cast<size_t>(nb) * sm90::kFinSlices * kMaxC);
  // tile-blocked Q: one 128x128 block per 128-row tile
  w.Q = need_Q ? c.take<float>(static_cast<size_t>(tiles) * sm90::kTileM * kQ) : nullptr;
  w.recs = c.take<float>(static_cast<size_t>(nrec) * rec_floats(p->C, p->D));
  w.row_offsets = sharded ? c.take<long long>(nb) : nullptr;
  w.qmax = sharded ? c.take<float>(static_cast<size_t>(nb) * p->C * kQ) : nullptr;
  w.bytes = c.off;
  *ok = c.ok();
  return w;
}

// Phases 2 and 3 of the batched forward: attend (one CTA per partial record: `recs` of them, or, with recs_dev, the
// first *recs_dev of a capacity grid of `recs`), then each bag's A, B, logits and critical rows.  overlap: the
// attend pass is a programmatic dependent of the phase 1 that bags_phase1_impl(overlap) has just launched.
static int bags_attend_finalize(const dsmil_params_t* p, const BagsWs& w, int nb, const float* Q, bool q_blocked,
                                float* pred, float* A, float* B, int64_t* crit, int recs, const int* recs_dev,
                                cudaStream_t st, bool overlap = false) {
  const int C = p->C, D = p->D;
  int rc;
  sm90::AttendArgs aa{w.table, nb, D, C, Q, q_blocked, w.keys, A, w.recs, nullptr, recs_dev,
                      overlap ? w.done : nullptr};
  if ((rc = sm90::launch_attend_b(aa, recs, st))) return rc;
  sm90::FinalizeArgs fa{w.table, D, C, w.recs, w.keys, p->Wf, p->bf, A, B, pred, reinterpret_cast<long long*>(crit),
                         w.pred_part, w.counters, nullptr, 0, 0};
  return sm90::launch_finalize_b(fa, nb, st);
}

static int forward_bags_impl(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int nb,
                             const float* classes_in, float* classes, float* pred, float* A, float* B,
                             int64_t* crit, float* save_Q, float* save_H1, void* ws, size_t ws_bytes,
                             cudaStream_t st) {
  bool ok;
  BagsWs w = carve_bags(p, Ns, nb, save_Q == nullptr, false, ws, ws_bytes, &ok);
  int rc = check_workspace(w.bytes, ok, ws, ws_bytes);
  if (rc) return rc;
  float* Q = save_Q ? save_Q : w.Q;
  const bool q_blocked = save_Q == nullptr;   // training keeps Q (after tanh) row-major for the backward kernels
  // The attend pass starts on each bag as soon as phase 1 has finished it, while the bag is still in L2 (DESIGN §4.2).
  // Same bits either way.  Not under stream capture, and not while kernels are being timed: the event between the two
  // launches would break the programmatic edge.
  const bool overlap = !g_prof_on && !stream_is_capturing(st);
  int tiles, recs;
  if ((rc = bags_phase1_impl(p, w, Xs, Ns, nb, classes_in, classes, Q, save_H1, q_blocked, true, &tiles, &recs, st,
                             overlap)))
    return rc;
  return bags_attend_finalize(p, w, nb, Q, q_blocked, pred, A, B, crit, recs, nullptr, st, overlap);
}

// ---- batched forward off the tensor-core batch: the generic shapes and the value network, one launch per stage ----
// Every bag's outputs and saves are the bits dsmil_forward gives it alone (fwd_generic_b.cuh, DESIGN §4.2h, §4.2i).
// Phase 1 is the one the single-bag forward takes on the shape: k_qmlp_sm90 where it runs (D % 128 == 0, nonlinear q,
// 16-byte aligned bags), else k_scores at each bag's MODE and the FFMA Q-MLP.  passing_v adds one k_vproj_b for the V
// of every bag, and the attend pass weighs V.
static bool gen_shape(const dsmil_params_t* p) { return !p->passing_v && !sm90::batched_supported(p); }

struct GenWs : Phase1Ws {
  float *Q, *H1;            // row-major [rows][128] where the caller keeps none
  float* qmax;              // [nb][C][128]
  int64_t* crit;            // [nb][C] where the caller wants none
  float *recs, *rec;        // the partial records; each bag's combined one [nb]
  BagsPlan* plan;           // dev calls: the planner's live counts and the stand-in row of a refused batch
  float* zero_row;
  sm90::BagDev* vtab;       // passing_v: [2 nb], the value inputs' table, then the packed V's (gen_forward_run)
  float* V;                 // passing_v: [rows][D] where the caller keeps none
  size_t bytes;
};
// rows, recs: the packed rows and partial records (dev calls: their capacities).  saves: the caller keeps Q, H1 and
// V (the training forms).
static GenWs carve_gen(const dsmil_params_t* p, int nb, int64_t rows, int64_t recs, bool saves, bool dev, void* ws,
                       size_t cap, bool* ok) {
  Carver c(ws, cap);
  GenWs w;
  carve_phase1(c, p, nb, w);
  w.Q = saves ? nullptr : c.take<float>(rows * kQ);
  w.H1 = p->nonlinear && !saves ? c.take<float>(rows * kQ) : nullptr;
  w.qmax = c.take<float>(static_cast<size_t>(nb) * p->C * kQ);
  w.crit = c.take<int64_t>(static_cast<size_t>(nb) * p->C);
  w.recs = c.take<float>(recs * rec_floats(p->C, p->D));
  w.rec = c.take<float>(static_cast<size_t>(nb) * rec_floats(p->C, p->D));
  w.plan = dev ? c.take<BagsPlan>(1) : nullptr;
  w.zero_row = dev ? c.take<float>(p->D) : nullptr;
  w.vtab = p->passing_v ? c.take<sm90::BagDev>(2 * static_cast<size_t>(nb)) : nullptr;
  w.V = p->passing_v && !saves ? c.take<float>(rows * p->D) : nullptr;
  w.bytes = c.off;
  *ok = c.ok();
  return w;
}
static GenWs carve_gen_eager(const dsmil_params_t* p, const int64_t* Ns, int nb, bool saves, void* ws, size_t cap,
                             bool* ok) {
  int64_t rows = 0, recs = 0;
  for (int b = 0; b < nb; ++b) {
    rows += Ns[b];
    recs += attend_ctas(Ns[b]);
  }
  return carve_gen(p, nb, rows, recs, saves, false, ws, cap, ok);
}
static GenWs carve_gen_dev(const dsmil_params_t* p, int nb, int64_t max_rows, bool saves, void* ws, size_t cap,
                           bool* ok) {
  return carve_gen(p, nb, nb * max_rows, static_cast<int64_t>(nb) * attend_ctas(max_rows), saves, true, ws, cap, ok);
}

template <int CT>
static int launch_attend_gb_j(int J, int grid, cudaStream_t st, const sm90::BagDev* bags, int nb, const int* recs_dev,
                              int D, int C, const float* Q, const float* qmax, float* A, float* recs) {
  switch (J) {
    case 1: k_attend_gb<CT, 1><<<grid, 256, 0, st>>>(bags, nb, recs_dev, D, C, Q, qmax, A, recs); break;
    case 2: k_attend_gb<CT, 2><<<grid, 256, 0, st>>>(bags, nb, recs_dev, D, C, Q, qmax, A, recs); break;
    case 4: k_attend_gb<CT, 4><<<grid, 256, 0, st>>>(bags, nb, recs_dev, D, C, Q, qmax, A, recs); break;
    case 8: k_attend_gb<CT, 8><<<grid, 256, 0, st>>>(bags, nb, recs_dev, D, C, Q, qmax, A, recs); break;
    default: k_attend_gb<CT, 16><<<grid, 256, 0, st>>>(bags, nb, recs_dev, D, C, Q, qmax, A, recs); break;
  }
  DSMIL_LAUNCH_OK("k_attend_gb");
  return 0;
}

// The value projection V = relu(Xv Wv^T + bv) over a table whose X are the value inputs, into packed V.  k_vproj_b;
// DSMIL_VPROJ_LINEAR_B=1 builds the variant that runs k_linear_b (k_linear's 64 x 128 tile) instead, with the same
// bits, for tools/bench_value_bags.py.  The library is built with the default.
#ifndef DSMIL_VPROJ_LINEAR_B
#define DSMIL_VPROJ_LINEAR_B 0
#endif
static int launch_vproj_b(const dsmil_params_t* p, const sm90::BagDev* vtab, int nb, int tiles, const int* tiles_dev,
                          float* V, cudaStream_t st) {
  const int D = p->D;
#if DSMIL_VPROJ_LINEAR_B
  k_linear_b<ACT_RELU><<<dim3(2 * tiles, ceil_div(D, LBN)), 256, 0, st>>>(vtab, nb, tiles_dev, D, p->Wv, p->bv, D, V,
                                                                    nullptr);
  DSMIL_LAUNCH_OK("k_linear_b");
#else
  k_vproj_b<<<dim3(tiles, ceil_div(D, VBN)), 256, 0, st>>>(vtab, nb, tiles_dev, D, p->Wv, p->bv, D, V);
  DSMIL_LAUNCH_OK("k_vproj_b");
#endif
  return 0;
}

// The fold form of the generic forward (dsmil_generic_forward_bags_models_train_dev): w.table lists every model's bags,
// model-major, as k_plan_bags_models writes it (bag_plan.cuh: FOLD_GEN / FOLD_GEN_QMLP).  The stages that read weights
// take each entry's model's from `models`; layer 2 of the Q-MLP and a k_qmlp_sm90 phase 1 run one launch per model over
// that model's block (ps[m]'s weights, its live counts in live[m]), on the grids its one-model dev call sizes.
struct GenFolds {
  const dsmil_params_t* ps;       // [M] host
  const int32_t* nbs;             // [M] host: each model's bags
  int M;
  int64_t max_rows;
  const sm90::ModelDev* models;   // [M] device
  const ModelsPlan* plan;         // device: the live tiles and records over all models
  const FoldLive* live;           // device [M]
};

// The generic forward over w.table: `tiles` and `recs` are the table's 128-row tiles and records and `rows` its packed
// rows (dev calls: capacities, the live counts in w.plan, or in f's for a fold call); max_N bounds the bags' rows.  Q
// (and H1 for nonlinear q) receive the Q-MLP's outputs row-major.  w.vtab (passing_v, eager only): nb entries of
// w.table's numbering whose X is each bag's value input, then nb whose X is the bag's packed rows of V; V receives the
// value projection and the attend pass reads it through the second half.  f: the fold form, p then being model 0's.
static int gen_forward_run(const dsmil_params_t* p, const GenWs& w, int nb, int64_t rows, int tiles, int recs,
                           int64_t max_N, float* classes, float* pred, float* A, float* B, int64_t* crit, float* Q,
                           float* H1, float* V, cudaStream_t st, const GenFolds* f = nullptr) {
  const int C = p->C, D = p->D;
  const BagsPlan* pl = w.plan;
  const sm90::BagDev* vtab = w.vtab;
  const int* tiles_dev = f ? &f->plan->tiles : pl ? &pl->tiles : nullptr;
  const int* recs_dev = f ? &f->plan->recs : pl ? &pl->recs : nullptr;
  const sm90::ModelDev* models = f ? f->models : nullptr;
  int rc;
  DSMIL_CUDA_OK(cudaMemsetAsync(w.keys, 0, sizeof(unsigned long long) * kMaxC * nb, st));
  if (sm90::qmlp_supported(p)) {
    if (!f) {
      if ((rc = sm90::launch_prep_wimg(p, w.wimg, st))) return rc;
      if ((rc = sm90::launch_qmlp(p, w.table, nb, tiles, classes, w.keys, Q, H1, w.wimg, num_sms(), st, false,
                                  tiles_dev, nullptr)))
        return rc;
    }
    for (int m = 0, e0 = 0; f && m < f->M; e0 += f->nbs[m], ++m) {   // model m's tiles are numbered from 0
      const int nbm = f->nbs[m];
      if ((rc = sm90::launch_prep_wimg(&f->ps[m], w.wimg, st))) return rc;
      if ((rc = sm90::launch_qmlp(&f->ps[m], w.table + e0, nbm, nbm * tiles_for_bag(f->max_rows), classes,
                                  w.keys + static_cast<size_t>(e0) * kMaxC, Q, H1, w.wimg, num_sms(), st, false,
                                  &f->live[m].tiles, nullptr)))
        return rc;
    }
  } else {
    const size_t smem = sizeof(float) * C * D;
    if (smem > 48 * 1024)
      DSMIL_CUDA_OK(cudaFuncSetAttribute(k_scores_b, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    prof_begin(PROF_SCORES, st);
    k_scores_b<<<tiles, 256, smem, st>>>(w.table, nb, tiles_dev, D, p->Wi, p->bi, C, classes, w.keys, models);
    prof_end(PROF_SCORES, st);
    DSMIL_LAUNCH_OK("k_scores_b");
    prof_begin(PROF_QMLP, st);
    const dim3 g1(2 * tiles, ceil_div(kQ, LBN));
    if (p->nonlinear) k_linear_b<ACT_RELU><<<g1, 256, 0, st>>>(w.table, nb, tiles_dev, D, p->W1, p->b1, kQ, H1, models);
    else k_linear_b<ACT_NONE><<<g1, 256, 0, st>>>(w.table, nb, tiles_dev, D, p->W1, p->b1, kQ, Q, models);
    DSMIL_LAUNCH_OK("k_linear_b");
    if (p->nonlinear && !f &&
        (rc = launch_linear<ACT_TANH, false>(H1, rows, kQ, p->W2, p->b2, kQ, Q, nullptr, 0, st, pl ? &pl->total : nullptr)))
      return rc;
    for (int m = 0, e0 = 0; p->nonlinear && f && m < f->M; e0 += f->nbs[m], ++m) {   // over model m's block
      const int64_t r0 = e0 * f->max_rows;
      if ((rc = launch_linear<ACT_TANH, false>(H1 + r0 * kQ, f->nbs[m] * f->max_rows, kQ, f->ps[m].W2, f->ps[m].b2,
                                               kQ, Q + r0 * kQ, nullptr, 0, st, &f->live[m].total)))
        return rc;
    }
    prof_end(PROF_QMLP, st);
  }
  if (vtab && (rc = launch_vproj_b(p, vtab, nb, tiles, tiles_dev, V, st))) return rc;
  k_crit_qmax_b<<<dim3(C, nb), kQ, 0, st>>>(w.table, w.keys, Q, C, w.qmax, crit);
  DSMIL_LAUNCH_OK("k_crit_qmax_b");
  int j = ceil_div(D, 256), J = 1;
  while (J < j) J <<= 1;
  const sm90::BagDev* atab = vtab ? vtab + nb : w.table;   // the rows the attend pass weighs: V, or the features
  prof_begin(PROF_ATTEND, st);
  if (C == 1) rc = launch_attend_gb_j<1>(J, recs, st, atab, nb, recs_dev, D, C, Q, w.qmax, A, w.recs);
  else if (C == 2) rc = launch_attend_gb_j<2>(J, recs, st, atab, nb, recs_dev, D, C, Q, w.qmax, A, w.recs);
  else if (C <= 4) rc = launch_attend_gb_j<4>(J, recs, st, atab, nb, recs_dev, D, C, Q, w.qmax, A, w.recs);
  else rc = launch_attend_gb_j<8>(J, recs, st, atab, nb, recs_dev, D, C, Q, w.qmax, A, w.recs);
  prof_end(PROF_ATTEND, st);
  if (rc) return rc;
  k_combine_rec_b<<<dim3(C, ceil_div(D, 256), nb), 256, 0, st>>>(w.table, C, D, w.recs, w.rec);
  DSMIL_LAUNCH_OK("k_combine_rec_b");
  const int fgrid = static_cast<int>(std::min<int64_t>(std::max<int64_t>(ceil_div(max_N * C, 256), 1), kSplits));
  prof_begin(PROF_FINAL, st);
  k_finalize_gb<<<dim3(fgrid, nb), 256, 0, st>>>(w.table, w.rec, C, D, p->Wf, p->bf, A, B, pred, models);
  prof_end(PROF_FINAL, st);
  DSMIL_LAUNCH_OK("k_finalize_gb");
  return 0;
}

// The eager generic forward: the table built on the host (each bag's MODE from its own alignment) and uploaded, and for
// passing_v the value table, whose X are the value inputs XVs (NULL: the features) and then each bag's packed rows of
// V.  save_Q / save_H1 / save_V: the training forms' row-major saves, all given or all NULL (inference, into the
// workspace).
static int forward_bags_gen(const dsmil_params_t* p, const float* const* Xs, const float* const* XVs,
                            const int64_t* Ns, int nb, float* classes, float* pred, float* A, float* B, int64_t* crit,
                            float* save_Q, float* save_H1, float* save_V, void* ws, size_t ws_bytes, cudaStream_t st) {
  bool ok;
  GenWs w = carve_gen_eager(p, Ns, nb, save_Q != nullptr, ws, ws_bytes, &ok);
  int rc = check_workspace(w.bytes, ok, ws, ws_bytes);
  if (rc) return rc;
  float* V = save_V ? save_V : w.V;
  std::vector<sm90::BagDev> tbl(nb), vt(p->passing_v ? 2 * static_cast<size_t>(nb) : 0);
  long long row = 0;
  int tile = 0, rec = 0;
  int64_t mx = 1;
  for (int b = 0; b < nb; ++b) {
    tbl[b] = gen_bag_entry(Xs[b], Ns[b], p->D, row, tile, rec);
    mx = std::max<int64_t>(mx, Ns[b]);
    if (p->passing_v) {
      vt[b] = vt[nb + b] = tbl[b];
      vt[b].X = XVs ? XVs[b] : Xs[b];
      vt[nb + b].X = V + tbl[b].row_off * p->D;
    }
  }
  DSMIL_CUDA_OK(cudaMemcpyAsync(w.table, tbl.data(), sizeof(sm90::BagDev) * nb, cudaMemcpyHostToDevice, st));
  if (p->passing_v)
    DSMIL_CUDA_OK(cudaMemcpyAsync(w.vtab, vt.data(), sizeof(sm90::BagDev) * vt.size(), cudaMemcpyHostToDevice, st));
  return gen_forward_run(p, w, nb, row, tile, rec, mx, classes, pred, A, B, crit ? crit : w.crit,
                         save_Q ? save_Q : w.Q, p->nonlinear ? (save_H1 ? save_H1 : w.H1) : nullptr, V, st);
}

static bool value_shape(const dsmil_params_t* p) {
  return p && p->passing_v && p->C >= 1 && p->C <= DSMIL_MAX_C && p->D >= 1 && p->D <= DSMIL_MAX_D;
}

// ---- the route of an eager forward -----------------------------------------------------------------------------------
// One rule for every eager forward of nb bags: the tensor-core batch where the shape takes it and every bag is 16-byte
// aligned; off that batch (the generic shapes and passing_v) the generic batch, unless its phase 1 is k_qmlp_sm90 and
// a bag is not aligned; otherwise one bag at a time.  Either batch numbers its bags in grid y (k_finalize_b, the
// generic per-bag kernels), so past 65535 bags every shape takes the loop.  ROUTE_VAL names the capture-safe calls'
// value route (the generic batch of a passing_v model); no eager forward takes it.
enum Route : unsigned { ROUTE_TC = 1, ROUTE_GEN = 2, ROUTE_LOOP = 4, ROUTE_VAL = 8 };
static Route bags_route(const dsmil_params_t* p, int nb, bool aligned) {
  if (nb > 65535) return ROUTE_LOOP;
  if (sm90::batched_supported(p)) return aligned ? ROUTE_TC : ROUTE_LOOP;
  return aligned || !sm90::qmlp_supported(p) ? ROUTE_GEN : ROUTE_LOOP;
}
// The routes bags_route gives nb bags of this shape at either alignment.
static unsigned bags_routes(const dsmil_params_t* p, int nb) {
  return bags_route(p, nb, true) | bags_route(p, nb, false);
}
// The workspace of an eager forward of these bags that may take any of `routes` (Route bits): the largest of their
// carves as inference takes them.  The loop's is the single-bag forward's for the largest bag: the single-bag kernels'
// carve and, where forward_impl takes an aligned bag to the tensor-core batch of one, that batch's.
static size_t routes_ws_bytes(const dsmil_params_t* p, const int64_t* Ns, int nb, unsigned routes) {
  bool ok;
  size_t bytes = 0;
  if (routes & ROUTE_TC) bytes = carve_bags(p, Ns, nb, true, false, nullptr, 0, &ok).bytes;
  if (routes & ROUTE_GEN) bytes = std::max(bytes, carve_gen_eager(p, Ns, nb, false, nullptr, 0, &ok).bytes);
  if (routes & ROUTE_LOOP) {
    int64_t mx = 0;
    for (int b = 0; b < nb; ++b) mx = std::max<int64_t>(mx, Ns[b]);
    bytes = std::max(bytes, carve_fwd(p, mx, nullptr, 0, &ok).bytes);
    if (mx > 0 && bags_route(p, 1, true) == ROUTE_TC)
      bytes = std::max(bytes, carve_bags(p, &mx, 1, true, false, nullptr, 0, &ok).bytes);
  }
  return bytes;
}

// One bag: the tensor-core batch of one where bags_route takes it, else the single-bag kernels.
static int forward_impl(const dsmil_params_t* p, const float* X, const float* xv, const float* classes_in,
                        int64_t N, float* classes, float* pred, float* A, float* B, int64_t* crit_idx,
                        float* save_Q, float* save_H1, float* save_V, void* ws, size_t ws_bytes, cudaStream_t st) {
  int rc = check_params(p, classes_in == nullptr);
  if (rc) return rc;
  DSMIL_REQUIRE(N >= 0 && N < 0xffffffffll, "N=%lld out of range", (long long)N);
  if (N == 0) {
    set_error("empty bag (N == 0): the reference raises IndexError at dsmil.py:53");
    return DSMIL_ERR_EMPTY;
  }
  DSMIL_REQUIRE(X && pred && A && B && (classes || classes_in), "NULL tensor pointer");
  if (bags_route(p, 1, (reinterpret_cast<uintptr_t>(X) & 15) == 0) == ROUTE_TC)
    return forward_bags_impl(p, &X, &N, 1, classes_in, classes, pred, A, B, crit_idx, save_Q, save_H1, ws, ws_bytes, st);
  bool ok;
  FwdWs w = carve_fwd(p, N, ws, ws_bytes, &ok);
  if ((rc = check_workspace(w.bytes, ok, ws, ws_bytes))) return rc;
  float* Q = save_Q ? save_Q : w.Q;
  float* H1 = p->nonlinear ? (save_H1 ? save_H1 : w.H1) : nullptr;
  float* V = p->passing_v ? (save_V ? save_V : w.V) : nullptr;
  if ((rc = phase1_impl(p, X, xv, classes_in, N, 0, classes, Q, H1, V, w.cand, w, st))) return rc;
  int64_t* crit = crit_idx ? crit_idx : w.crit;
  k_merge_cand<<<p->C, kQ, 0, st>>>(w.cand, 1, 1, p->C, w.qmax, crit);
  DSMIL_LAUNCH_OK("k_merge_cand");
  const float* Vv = p->passing_v ? V : X;
  if ((rc = phase2_impl(p, Vv, Q, N, w.qmax, A, w.rec, w.recs, st))) return rc;
  return phase3_impl(p, N, w.rec, A, B, pred, st);
}

// The eager forward of nb checked bags on their route: the tensor-core batch, the generic (passing_v: value) batch, or
// forward_impl per bag into the same packed outputs.  XVs: passing_v's value inputs (NULL: the features).  save_Q /
// save_H1 / save_V: the training forms' row-major saves, or NULL.
static int forward_bags_route(const dsmil_params_t* p, const float* const* Xs, const float* const* XVs,
                              const int64_t* Ns, int nb, bool aligned, float* classes, float* pred, float* A,
                              float* B, int64_t* crit, float* save_Q, float* save_H1, float* save_V, void* ws,
                              size_t ws_bytes, cudaStream_t st) {
  const Route r = bags_route(p, nb, aligned);
  if (r == ROUTE_TC)
    return forward_bags_impl(p, Xs, Ns, nb, nullptr, classes, pred, A, B, crit, save_Q, save_H1, ws, ws_bytes, st);
  if (r == ROUTE_GEN)
    return forward_bags_gen(p, Xs, XVs, Ns, nb, classes, pred, A, B, crit, save_Q, save_H1, save_V, ws, ws_bytes, st);
  const int C = p->C, D = p->D;
  int64_t row = 0;
  for (int b = 0; b < nb; ++b) {
    const int rc = forward_impl(p, Xs[b], XVs ? XVs[b] : nullptr, nullptr, Ns[b], classes + row * C,
                                pred + static_cast<size_t>(b) * C, A + row * C, B + static_cast<size_t>(b) * C * D,
                                crit ? crit + static_cast<size_t>(b) * C : nullptr,
                                save_Q ? save_Q + row * kQ : nullptr, save_H1 ? save_H1 + row * kQ : nullptr,
                                save_V ? save_V + row * D : nullptr, ws, ws_bytes, st);
    if (rc) return rc;
    row += Ns[b];
  }
  return 0;
}

}  // namespace dsmil

using namespace dsmil;

extern "C" {

int dsmil_abi_version(void) { return DSMIL_ABI_VERSION; }
const char* dsmil_last_error(void) { return g_err; }
uint64_t dsmil_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
int dsmil_forward_path(const dsmil_params_t* p, int64_t N) {
  (void)N;
  return (p && p->C >= 1 && p->C <= DSMIL_MAX_C && p->D >= 1 && p->D <= DSMIL_MAX_D && sm90::qmlp_supported(p)) ? 2 : 1;
}


int dsmil_gather_rows(const float* X, int64_t N, int32_t D, const int64_t* idx, int64_t M, float* out, void* stream) {
  DSMIL_REQUIRE(N >= 0 && M >= 0 && D >= 1 && (M == 0 || (X && idx && out)), "bad arguments");
  if (M == 0) return 0;
  const int grid = static_cast<int>(std::min<int64_t>((M + 7) / 8, kSms * 8));
  k_gather_rows<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(X, D, reinterpret_cast<const long long*>(idx), M, out);
  DSMIL_LAUNCH_OK("k_gather_rows");
  return 0;
}

int dsmil_patches_u8_to_f32(const uint8_t* in, int64_t B, int32_t H, int32_t W, int32_t Cc, float* out, void* stream) {
  DSMIL_REQUIRE(B >= 0 && H >= 1 && W >= 1 && Cc >= 1 && Cc <= 4 && (B == 0 || (in && out)), "bad arguments");
  if (B == 0) return 0;
  const long long total = static_cast<long long>(B) * H * W;
  const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, kSms * 16));
  k_u8hwc_to_f32chw<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(in, B, H, W, Cc, out);
  DSMIL_LAUNCH_OK("k_u8hwc_to_f32chw");
  return 0;
}

int dsmil_instnorm_act(const float* x, const float* residual, float* y, int64_t planes, int32_t HW, float eps,
                       int32_t relu, void* stream) {
  DSMIL_REQUIRE(planes >= 0 && HW >= 1 && HW <= kInPlaneMax && eps >= 0.f && (planes == 0 || (x && y)),
                "bad arguments (HW must be in [1, %d])", kInPlaneMax);
  DSMIL_REQUIRE(planes < (1ll << 31), "too many planes");
  if (planes == 0) return 0;
  return launch_instnorm(x, residual, y, planes, HW, eps, relu, static_cast<cudaStream_t>(stream));
}

int dsmil_instnorm_act_nhwc(const float* x, const float* residual, float* y, int64_t N, int32_t HW, int32_t C, float eps,
                            int32_t relu, void* stream) {
  DSMIL_REQUIRE(N >= 0 && HW >= 1 && C >= 32 && C % 32 == 0 && eps >= 0.f && (N == 0 || (x && y)),
                "bad arguments (C must be a multiple of 32)");
  DSMIL_REQUIRE(N * (C / 32) < (1ll << 31), "too many (sample, channel group) slabs");
  if (N == 0) return 0;
  return launch_instnorm_nhwc(x, residual, y, N, HW, C, eps, relu, static_cast<cudaStream_t>(stream));
}

static JpegBatch carve_jpeg(void* ws, size_t cap, int n, int H, int W, int64_t blob_bytes, size_t* need) {
  Carver cv(ws, cap);
  JpegBatch a{};
  a.n = n; a.H = H; a.W = W;
  a.plane_elems = jpeg_plane_elems(H, W);
  a.unstuffed = cv.take<uint8_t>(static_cast<size_t>(blob_bytes) + 64);
  a.coef = cv.take<int16_t>(static_cast<size_t>(3) * a.plane_elems * n);
  a.planes = cv.take<uint8_t>(static_cast<size_t>(3) * a.plane_elems * n);
  *need = cv.off;
  return a;
}

int32_t dsmil_jpeg_header_bytes_dev(void) { return static_cast<int32_t>(sizeof(dsmil_jpeg_header)); }

int64_t dsmil_jpeg_workspace_bytes(int32_t n, int32_t H, int32_t W, int64_t blob_bytes) {
  if (n < 0 || H < 1 || W < 1 || H > 65535 || W > 65535 || blob_bytes < 0) return -1;
  size_t need = 0;
  carve_jpeg(nullptr, 0, n, H, W, blob_bytes, &need);
  return static_cast<int64_t>(need);
}

int dsmil_jpeg_decode_batch(const uint8_t* blob, int64_t blob_bytes, const void* headers, int32_t n, int32_t H, int32_t W,
                            uint8_t* out_u8, float* out_f32, int32_t f32_channels_last, int32_t* status, void* workspace,
                            int64_t workspace_bytes, void* stream) {
  DSMIL_REQUIRE(n >= 0 && H >= 1 && W >= 1 && H <= 65535 && W <= 65535 && blob_bytes >= 0 &&
                (f32_channels_last == 0 || f32_channels_last == 1), "bad arguments");
  if (n == 0) return 0;
  DSMIL_REQUIRE(blob && headers && status && workspace && (out_u8 || out_f32), "null pointer");
  DSMIL_REQUIRE((reinterpret_cast<uintptr_t>(headers) & 15) == 0 && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0 &&
                (out_f32 == nullptr || (reinterpret_cast<uintptr_t>(out_f32) & 15) == 0) &&
                (out_u8 == nullptr || (reinterpret_cast<uintptr_t>(out_u8) & 3) == 0),
                "headers must be 16-byte, workspace 256-byte, out_f32 16-byte, out_u8 4-byte aligned");
  size_t need = 0;
  JpegBatch a = carve_jpeg(workspace, static_cast<size_t>(workspace_bytes), n, H, W, blob_bytes, &need);
  const int rc = check_workspace(need, static_cast<int64_t>(need) <= workspace_bytes, workspace,
                                 static_cast<size_t>(std::max<int64_t>(workspace_bytes, 0)));
  if (rc) return rc;
  a.blob = blob;
  a.hdr = static_cast<const dsmil_jpeg_header*>(headers);
  a.out_u8 = out_u8;
  a.out_f32 = out_f32;
  a.f32_hwc = f32_channels_last;
  a.status = status;
  return launch_jpeg_decode(a, static_cast<cudaStream_t>(stream));
}

int dsmil_profile_enable(int on) {
  g_prof_on = on != 0;
  return 0;
}
int dsmil_profile_read(double* ms_per_tag, uint64_t* launches_per_tag) {
  DSMIL_REQUIRE(ms_per_tag && launches_per_tag, "NULL output");
  for (int t = 0; t < PROF_NTAGS; ++t) { ms_per_tag[t] = 0.0; launches_per_tag[t] = 0; }
  for (auto& r : g_prof) {
    float ms = 0.f;
    if (cudaEventSynchronize(r.b) == cudaSuccess && cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) {
      ms_per_tag[r.tag] += ms;
      launches_per_tag[r.tag] += 1;
    }
    g_prof_pool.push_back(r);
  }
  g_prof.clear();
  cudaGetLastError();
  return 0;
}

size_t dsmil_cand_floats(int32_t C) { return cand_floats(C); }
size_t dsmil_rec_floats(int32_t C, int32_t Dv) { return rec_floats(C, Dv); }

size_t dsmil_forward_workspace_bytes(const dsmil_params_t* p, int64_t N) {
  if (!p || p->C < 1 || p->C > DSMIL_MAX_C || p->D < 1 || p->D > DSMIL_MAX_D || N < 0) return 0;
  return routes_ws_bytes(p, &N, 1, ROUTE_LOOP);   // the loop's carve is forward_impl's
}

size_t dsmil_forward_bags_workspace_bytes(const dsmil_params_t* p, const int64_t* Ns, int32_t nb) {
  if (!p || !Ns || nb < 1 || p->C < 1 || p->C > DSMIL_MAX_C || p->D < 1 || p->D > DSMIL_MAX_D) return 0;
  // The rule's routes, and on every shape the loop's carve, on identity-v shapes the generic batch's at any nb: one
  // size for the batch whatever its alignment and nb.
  return routes_ws_bytes(p, Ns, nb, bags_routes(p, nb) | ROUTE_LOOP | (gen_shape(p) ? ROUTE_GEN : 0));
}

int dsmil_forward_bags(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                       float* classes, float* pred, float* A, float* B, int64_t* crit_idx, void* workspace,
                       size_t workspace_bytes, void* stream) {
  int rc = check_params(p, true);
  if (rc) return rc;
  DSMIL_REQUIRE(Xs && Ns && nb >= 1 && classes && pred && A && B, "NULL pointer or nb < 1");
  int64_t total;
  bool aligned;
  if ((rc = check_bags(Xs, Ns, nb, &total, &aligned))) return rc;
  // one contract for every route: the size dsmil_forward_bags_workspace_bytes reports
  if ((rc = need_workspace(dsmil_forward_bags_workspace_bytes(p, Ns, nb), workspace, workspace_bytes))) return rc;
  return forward_bags_route(p, Xs, nullptr, Ns, nb, aligned, classes, pred, A, B, crit_idx, nullptr, nullptr, nullptr,
                            workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}
int32_t dsmil_forward_bags_phase1_ctas(int64_t tiles) { return tiles < 1 ? 0 : overlap_phase1_ctas(tiles); }

// ---- ensemble forward: M models over one batch of bags ---------------------------------------------------------------
// The fused form's table has one entry per (bag, model), model-major inside each bag (entry b * M + m), so the M passes
// over a bag follow each other on the persistent grid and the later ones find its features in L2 (DESIGN §4.2e).
// Entry (b, m)'s rows sit at m * sum N + (first row of b) in the packed outputs, which makes classes and A model-major;
// keys, counters, Q tile blocks and records keep the per-entry numbering of the one-model batch.
static int check_models(const dsmil_params_t* ps, int M) {
  DSMIL_REQUIRE(ps != nullptr, "params is NULL");
  DSMIL_REQUIRE(M >= 1 && M <= sm90::kMaxModels, "models: M=%d outside [1,%d]", M, sm90::kMaxModels);
  for (int m = 0; m < M; ++m) {
    const int rc = check_params(&ps[m], true);
    if (rc) return rc;
    DSMIL_REQUIRE(ps[m].D == ps[0].D && ps[m].C == ps[0].C && ps[m].nonlinear == ps[0].nonlinear &&
                      ps[m].passing_v == ps[0].passing_v,
                  "model %d: (D=%d, C=%d, nonlinear=%d, passing_v=%d) differs from model 0's (%d, %d, %d, %d)", m,
                  ps[m].D, ps[m].C, ps[m].nonlinear, ps[m].passing_v, ps[0].D, ps[0].C, ps[0].nonlinear,
                  ps[0].passing_v);
  }
  return 0;
}
static bool models_batched(const dsmil_params_t* ps, int M) {
  for (int m = 0; m < M; ++m)
    if (!dsmil_shard_bags_supported(&ps[m])) return false;
  return true;
}

struct ModelsWs : BagsWs {
  sm90::ModelDev* models;   // [M]
};
// The fused layout of M members over a table of nb * reps entries: the nb bags Ns, each `reps` times (the ensemble
// forward: reps = M, every model over the same bags; the training form: reps = 1, every model's own bags listed
// model-major).  need_Q: room for tile-blocked Q (the training form writes the caller's row-major save_Q instead).
static ModelsWs carve_models(const dsmil_params_t* p, int M, const int64_t* Ns, int nb, int reps, bool need_Q,
                             void* ws, size_t cap, bool* ok) {
  Carver c(ws, cap);
  ModelsWs w;
  int64_t tiles = 0, nrec = 0;
  for (int b = 0; b < nb; ++b) {
    tiles += tiles_for_bag(Ns[b]);
    nrec += recs_for_bag(Ns[b]);
  }
  const size_t ne = static_cast<size_t>(nb) * reps;
  w.table = c.take<sm90::BagDev>(ne);
  w.keys = c.take<unsigned long long>(ne * (kMaxC + 1));   // keys, then the two per-entry counters (carve_phase1)
  w.counters = reinterpret_cast<unsigned int*>(w.keys ? w.keys + ne * kMaxC : nullptr);
  w.done = w.counters ? w.counters + ne : nullptr;
  w.models = c.take<sm90::ModelDev>(M);
  const uintptr_t img = reinterpret_cast<uintptr_t>(c.take<uint8_t>(M * sm90::wimg_bytes(p->D) + 1024));
  w.wimg = reinterpret_cast<uint8_t*>((img + 1023) & ~uintptr_t(1023));
  w.pred_part = c.take<float>(ne * sm90::kFinSlices * kMaxC);
  w.Q = need_Q ? c.take<float>(static_cast<size_t>(reps) * tiles * sm90::kTileM * kQ) : nullptr;
  w.recs = c.take<float>(static_cast<size_t>(reps) * nrec * rec_floats(p->C, p->D));
  w.row_offsets = nullptr;
  w.qmax = nullptr;
  w.bytes = c.off;
  *ok = c.ok();
  return w;
}

// The fused launches over a host table `tbl` (tiles / recs: its 128-row tiles and partial records): one weight-image
// prep, one phase 1, one attend and one finalize for all M members.  Q (+ H1) as launch_qmlp_models takes them.
// nb_out > 0: the ensemble's table, whose entry b * M + m writes pred / B / crit to slot m * nb_out + b; nb_out == 0:
// a table of each model's own bags, model-major, whose entry e writes slot e.
static int models_launch(const dsmil_params_t* ps, int M, const ModelsWs& w, const std::vector<sm90::BagDev>& tbl,
                         int tile, int rec, float* classes, float* Q, float* H1, bool q_blocked, float* pred, float* A,
                         float* B, int64_t* crit, int nb_out, cudaStream_t st) {
  const int C = ps[0].C, D = ps[0].D, ne = static_cast<int>(tbl.size());
  int rc;
  std::vector<sm90::ModelDev> mh(M);
  for (int m = 0; m < M; ++m) {
    const dsmil_params_t& p = ps[m];
    mh[m] = sm90::ModelDev{p.Wi, p.bi, p.W1, p.b1, p.W2, p.b2, p.Wf, p.bf};
  }
  DSMIL_CUDA_OK(cudaMemcpyAsync(w.table, tbl.data(), sizeof(sm90::BagDev) * ne, cudaMemcpyHostToDevice, st));
  DSMIL_CUDA_OK(cudaMemcpyAsync(w.models, mh.data(), sizeof(sm90::ModelDev) * M, cudaMemcpyHostToDevice, st));
  DSMIL_CUDA_OK(cudaMemsetAsync(w.keys, 0, sizeof(unsigned long long) * (kMaxC + 1) * ne, st));
  if ((rc = sm90::launch_prep_wimg_models(w.models, M, D, w.wimg, st))) return rc;
  // overlapped as in forward_bags_impl: not under capture, not while kernels are timed
  const bool overlap = !g_prof_on && !stream_is_capturing(st);
  if ((rc = sm90::launch_qmlp_models(w.models, M, D, C, w.table, ne, tile, classes, w.keys, Q, H1, q_blocked, w.wimg,
                                     overlap ? overlap_phase1_ctas(tile) : num_sms(), st,
                                     overlap ? w.done : nullptr)))
    return rc;
  sm90::AttendArgs aa{w.table, ne, D, C, Q, q_blocked, w.keys, A, w.recs, nullptr, nullptr, overlap ? w.done : nullptr};
  if ((rc = sm90::launch_attend_b(aa, rec, st))) return rc;
  // slot = pad_ * nb_out + entry / nmodels: nmodels = 1 and nb_out = 0 make it the entry itself
  sm90::FinalizeArgs fa{w.table, D, C, w.recs, w.keys, nullptr, nullptr, A, B, pred,
                        reinterpret_cast<long long*>(crit), w.pred_part, w.counters, nullptr, 0, 0,
                        w.models, nb_out > 0 ? M : 1, nb_out};
  return sm90::launch_finalize_b(fa, ne, st);
}

static int forward_bags_models_impl(const dsmil_params_t* ps, int M, const float* const* Xs, const int64_t* Ns,
                                    int nb, int64_t total, float* classes, float* pred, float* A, float* B,
                                    int64_t* crit, void* ws, size_t ws_bytes, cudaStream_t st) {
  const int ne = nb * M;
  bool ok;
  ModelsWs w = carve_models(&ps[0], M, Ns, nb, M, true, ws, ws_bytes, &ok);
  int rc = check_workspace(w.bytes, ok, ws, ws_bytes);
  if (rc) return rc;
  std::vector<sm90::BagDev> tbl(ne);
  long long row = 0;
  int tile = 0, rec = 0;
  for (int b = 0; b < nb; ++b) {
    for (int m = 0; m < M; ++m) {
      long long r = row;
      sm90::BagDev& e = tbl[static_cast<size_t>(b) * M + m];
      e = bag_entry(Xs[b], Ns[b], r, tile, rec);
      e.row_off = m * total + row;
      e.pad_ = m;
    }
    row += Ns[b];
  }
  return models_launch(ps, M, w, tbl, tile, rec, classes, w.Q, nullptr, true, pred, A, B, crit, nb, st);
}

int dsmil_models_supported(const dsmil_params_t* ps, int32_t M) {
  if (!ps || M < 1 || M > sm90::kMaxModels || check_models(ps, M) != 0 || !models_batched(ps, M)) return 0;
  return sm90::qmlp_models_fit(ps[0].C, ps[0].D, M) ? 1 : 0;
}

size_t dsmil_forward_bags_models_workspace_bytes(const dsmil_params_t* ps, int32_t M, const int64_t* Ns, int32_t nb) {
  if (!ps || M < 1 || M > sm90::kMaxModels || !Ns || nb < 1) return 0;
  size_t bytes = 0;
  for (int m = 0; m < M; ++m) {   // the per-model loop
    const size_t b = dsmil_forward_bags_workspace_bytes(&ps[m], Ns, nb);
    if (b == 0) return 0;
    bytes = std::max(bytes, b);
  }
  // the fused layout on every batched shape, whether or not M members fit in shared memory: the size then grows with
  // M, nb and N alike
  bool ok;
  if (models_batched(ps, M)) bytes = std::max(bytes, carve_models(&ps[0], M, Ns, nb, M, true, nullptr, 0, &ok).bytes);
  return bytes;
}

int dsmil_forward_bags_models(const dsmil_params_t* ps, int32_t M, const float* const* Xs, const int64_t* Ns,
                              int32_t nb, float* classes, float* pred, float* A, float* B, int64_t* crit_idx,
                              void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_models(ps, M);
  if (rc) return rc;
  DSMIL_REQUIRE(Xs && Ns && nb >= 1 && classes && pred && A && B, "NULL pointer or nb < 1");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int64_t total;
  bool aligned;
  if ((rc = check_bags(Xs, Ns, nb, &total, &aligned))) return rc;
  const size_t need = dsmil_forward_bags_models_workspace_bytes(ps, M, Ns, nb);
  if ((rc = need_workspace(need, workspace, workspace_bytes))) return rc;
  if (aligned && dsmil_models_supported(ps, M) && static_cast<int64_t>(nb) * M <= 65535)
    return forward_bags_models_impl(ps, M, Xs, Ns, nb, total, classes, pred, A, B, crit_idx, workspace,
                                    workspace_bytes, st);
  // off the fused route: each model's dsmil_forward_bags into its slice
  const int C = ps[0].C, D = ps[0].D;
  for (int m = 0; m < M; ++m) {
    rc = dsmil_forward_bags(&ps[m], Xs, Ns, nb, classes + m * total * C, pred + static_cast<size_t>(m) * nb * C,
                            A + m * total * C, B + static_cast<size_t>(m) * nb * C * D,
                            crit_idx ? crit_idx + static_cast<size_t>(m) * nb * C : nullptr, workspace,
                            workspace_bytes, stream);
    if (rc) return rc;
  }
  return 0;
}

size_t dsmil_shard_workspace_bytes(const dsmil_params_t* p, int64_t N_local) {
  return dsmil_forward_workspace_bytes(p, N_local);
}

int dsmil_forward(const dsmil_params_t* p, const float* X, const float* x_for_v, int64_t N, float* classes,
                  float* pred, float* A, float* B, int64_t* crit_idx, float* save_Q, float* save_H1,
                  float* save_V, void* workspace, size_t workspace_bytes, void* stream) {
  DSMIL_REQUIRE(classes != nullptr, "classes is NULL");
  return forward_impl(p, X, x_for_v, nullptr, N, classes, pred, A, B, crit_idx, save_Q, save_H1, save_V,
                      workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

int dsmil_bag_forward(const dsmil_params_t* p, const float* X, const float* x_for_v, const float* classes_in,
                      int64_t N, float* pred, float* A, float* B, int64_t* crit_idx, float* save_Q,
                      float* save_H1, float* save_V, void* workspace, size_t workspace_bytes, void* stream) {
  DSMIL_REQUIRE(classes_in != nullptr, "classes_in is NULL");
  return forward_impl(p, X, x_for_v, classes_in, N, nullptr, pred, A, B, crit_idx, save_Q, save_H1, save_V,
                      workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

int dsmil_instance_scores(const dsmil_params_t* p, const float* X, int64_t N, float* classes, void* stream) {
  DSMIL_REQUIRE(p && p->Wi && p->bi && p->C >= 1 && p->C <= DSMIL_MAX_C && p->D >= 1 && p->D <= DSMIL_MAX_D,
                "bad params");
  DSMIL_REQUIRE(N >= 0 && (N == 0 || (X && classes)), "NULL tensor pointer");
  if (N == 0) return 0;
  // The arg-max by-product goes to a scratch key slot that is simply ignored here.
  unsigned long long* keys;
  DSMIL_CUDA_OK(cudaGetSymbolAddress(reinterpret_cast<void**>(&keys), scratch_keys));
  return launch_scores(p, X, N, classes, keys, static_cast<cudaStream_t>(stream));
}

// ---- sharded phases -----------------------------------------------------------------------
int dsmil_shard_phase1(const dsmil_params_t* p, const float* X, const float* x_for_v, const float* classes_in,
                       int64_t N_local, int64_t row_offset, float* classes, float* Q, float* H1, float* V,
                       float* cand_rec, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_params(p, classes_in == nullptr);
  if (rc) return rc;
  DSMIL_REQUIRE(N_local >= 0 && N_local < 0xffffffffll, "N_local out of range");
  DSMIL_REQUIRE(cand_rec && (N_local == 0 || (X && Q && (classes || classes_in))), "NULL tensor pointer");
  DSMIL_REQUIRE(N_local == 0 || !p->passing_v || V, "passing_v needs a V buffer");
  bool ok;
  FwdWs w = carve_fwd(p, N_local, workspace, workspace_bytes, &ok);
  if ((rc = check_workspace(w.bytes, ok, workspace, workspace_bytes))) return rc;
  float* h1 = p->nonlinear ? (H1 ? H1 : (phase1_on_qmlp(p, w.wimg, X) ? nullptr : w.H1)) : nullptr;
  return phase1_impl(p, X, x_for_v, classes_in, N_local, row_offset, classes, Q, h1, V, cand_rec, w,
                     static_cast<cudaStream_t>(stream));
}

int dsmil_shard_merge_candidates(int32_t C, const float* cand_recs, int32_t G, float* q_max, int64_t* crit_idx,
                                 void* stream) {
  DSMIL_REQUIRE(C >= 1 && C <= DSMIL_MAX_C && G >= 1 && cand_recs && q_max && crit_idx, "bad arguments");
  k_merge_cand<<<C, kQ, 0, static_cast<cudaStream_t>(stream)>>>(cand_recs, G, 1, C, q_max, crit_idx);
  DSMIL_LAUNCH_OK("k_merge_cand");
  return 0;
}

int dsmil_shard_phase2(const dsmil_params_t* p, const float* Xv, const float* Q, int64_t N_local,
                       const float* q_max, float* A_logits, float* rec, void* workspace, size_t workspace_bytes,
                       void* stream) {
  int rc = check_params(p);
  if (rc) return rc;
  DSMIL_REQUIRE(rec && q_max && (N_local == 0 || (Xv && Q && A_logits)), "NULL tensor pointer");
  bool ok;
  FwdWs w = carve_fwd(p, N_local, workspace, workspace_bytes, &ok);
  if ((rc = check_workspace(w.bytes, ok, workspace, workspace_bytes))) return rc;
  return phase2_impl(p, Xv, Q, N_local, q_max, A_logits, rec, w.recs, static_cast<cudaStream_t>(stream));
}

int dsmil_shard_merge_partials(int32_t C, int32_t Dv, const float* recs, int32_t G, float* rec_out, void* stream) {
  DSMIL_REQUIRE(C >= 1 && C <= DSMIL_MAX_C && Dv >= 1 && G >= 1 && G <= kMaxRecs && recs && rec_out, "bad arguments");
  dim3 g2(C, ceil_div(Dv, 256));
  k_combine_rec<<<g2, 256, 0, static_cast<cudaStream_t>(stream)>>>(recs, G, C, Dv, rec_out);
  DSMIL_LAUNCH_OK("k_combine_rec");
  return 0;
}

int dsmil_shard_phase3(const dsmil_params_t* p, int64_t N_local, const float* rec_global, float* A, float* B,
                       float* pred, void* stream) {
  int rc = check_params(p);
  if (rc) return rc;
  DSMIL_REQUIRE(rec_global && B && pred && (N_local == 0 || A), "NULL tensor pointer");
  return phase3_impl(p, N_local, rec_global, A, B, pred, static_cast<cudaStream_t>(stream));
}

// ---- backward -----------------------------------------------------------------------------
struct BwdWs {
  float *dB, *dA, *tpart, *dqm, *dz2, *dz1, *tnpart, *cspart, *dzv, *tmp;
  size_t bytes;
};
static BwdWs carve_bwd(const dsmil_params_t* p, int64_t N, int need_gX, void* ws, size_t cap, bool* ok) {
  Carver c(ws, cap);
  BwdWs w;
  const int C = p->C, D = p->D;
  const int64_t n = N > 0 ? N : 1;
  w.dB = c.take<float>(static_cast<size_t>(C) * D);
  w.dA = c.take<float>(n * C);
  w.tpart = c.take<float>(kSplits * kMaxC);
  w.dqm = c.take<float>(static_cast<size_t>(C) * kQ);
  w.dz2 = c.take<float>(n * kQ);
  w.dz1 = p->nonlinear ? c.take<float>(n * kQ) : nullptr;
  size_t tn = tn_partial_floats(kQ, D, N);
  tn = std::max(tn, tn_partial_floats(kQ, kQ, N));
  tn = std::max(tn, tn_partial_floats(C, kQ, N));
  tn = std::max(tn, tn_partial_floats(C, D, N));
  if (p->passing_v) tn = std::max(tn, tn_partial_floats(D, D, N));
  w.tnpart = c.take<float>(tn);
  w.cspart = c.take<float>(static_cast<size_t>(kSplits) * std::max(D, kQ));
  w.dzv = p->passing_v ? c.take<float>(n * D) : nullptr;
  w.tmp = (p->passing_v && need_gX) ? c.take<float>(n * D) : nullptr;
  w.bytes = c.off;
  *ok = c.ok();
  return w;
}

size_t dsmil_backward_workspace_bytes(const dsmil_params_t* p, int64_t N, int need_gX) {
  if (!p || p->C < 1 || p->C > DSMIL_MAX_C || p->D < 1 || p->D > DSMIL_MAX_D || N < 0) return 0;
  bool ok;
  return carve_bwd(p, N, need_gX, nullptr, 0, &ok).bytes;
}

// The backward in three phases, cut at its two cross-row sums (t and dq_max).  dsmil_backward runs them in a row;
// the row-sharded backward runs one per call, with the caller's all-reduces in between.  A rank may hold no rows
// (N == 0): the per-row launches are skipped and its weight-gradient shares come out zero.

// Phase 1: dB, gWf/gbf, gWi/gbi, dA = Vv dB^T (+ d_A), and t's per-block partials sum_n A*dA in w.tpart (*gs of them).
static int bwd_phase1_impl(const dsmil_params_t* p, const float* X, const float* Vv, int64_t N, const float* A,
                           const float* B, const float* d_classes, const float* d_pred, const float* d_A,
                           const float* d_B, const dsmil_grads_t* g, float* dA, const BwdWs& w, int* gs,
                           cudaStream_t st) {
  const int C = p->C, D = p->D;
  int rc;
  // bag classifier (dsmil.py:59-61) and B
  k_bwd_bag<<<ceil_div(static_cast<int64_t>(C) * D, 256), 256, 0, st>>>(p->Wf, B, d_pred, d_B, C, D, w.dB, g->gWf,
                                                                        g->gbf);
  DSMIL_LAUNCH_OK("k_bwd_bag");
  // instance classifier (dsmil.py:11): only rows with non-zero upstream grad contribute
  if (g->gWi) {
    if (d_classes && N > 0) { if ((rc = launch_gemm_tn(d_classes, C, X, D, N, w.tnpart, g->gWi, st))) return rc; }
    else DSMIL_CUDA_OK(cudaMemsetAsync(g->gWi, 0, sizeof(float) * C * D, st));
  }
  if (g->gbi) {
    if (d_classes && N > 0) { if ((rc = launch_colsum(d_classes, C, N, w.cspart, g->gbi, st))) return rc; }
    else DSMIL_CUDA_OK(cudaMemsetAsync(g->gbi, 0, sizeof(float) * C, st));
  }
  *gs = static_cast<int>(std::min<int64_t>(ceil_div(N, 256), kSplits));
  if (N == 0) return 0;
  // dA = V dB^T (+ upstream), softmax-over-instances backward (dsmil.py:56-57)
  const size_t smem = sizeof(float) * C * D;
  if (smem > 48 * 1024)
    DSMIL_CUDA_OK(cudaFuncSetAttribute(k_rowdot, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = static_cast<int>(std::min<int64_t>(ceil_div(N, 8), kSms * 8));
  k_rowdot<<<grid, 256, smem, st>>>(Vv, N, D, w.dB, C, d_A, dA);
  DSMIL_LAUNCH_OK("k_rowdot");
  k_bwd_t_partial<<<*gs, 256, 0, st>>>(A, dA, N, C, w.tpart);
  DSMIL_LAUNCH_OK("k_bwd_t_partial");
  return 0;
}

// Phase 2: dL = A (dA - t) / sqrt(128) in place over dA, t the sum of the P partials in `part`; then
// dq_max = dL^T Q (dsmil.py:55), zeros when N == 0.
static int bwd_phase2_impl(const dsmil_params_t* p, int64_t N, const float* A, float* dA, const float* part, int P,
                           const float* Q, float* dqm, const BwdWs& w, cudaStream_t st) {
  if (N > 0) {
    const int gs = static_cast<int>(std::min<int64_t>(ceil_div(N, 256), kSplits));
    k_bwd_dL<<<gs, 256, 0, st>>>(A, dA, N, p->C, part, P);
    DSMIL_LAUNCH_OK("k_bwd_dL");
  }
  return launch_gemm_tn(dA, p->C, Q, kQ, N, w.tnpart, dqm, st);
}

// Phase 3: dQ rows (+ the critical rows' share, dsmil.py:53-54; k_bwd_dq reads qmax == NULL as "critical rows are
// local"), back through the Q-MLP into gW2/gb2 and gW1/gb1.  *dz1 is the layer-1 gradient it leaves in w.
static int bwd_phase3_impl(const dsmil_params_t* p, const float* X, int64_t N, int64_t row_offset, const float* Q,
                           const float* H1, const float* dL, const float* dqm, const float* qmax, const int64_t* crit,
                           const dsmil_grads_t* g, const BwdWs& w, const float** dz1, cudaStream_t st) {
  int rc;
  if (N > 0) {
    const int grid = static_cast<int>(std::min<int64_t>(ceil_div(N * kQ, 256), kSms * 8));
    k_bwd_dq<<<grid, 256, 0, st>>>(dL, Q, qmax, dqm, crit, N, row_offset, p->C, p->nonlinear, w.dz2);
    DSMIL_LAUNCH_OK("k_bwd_dq");
  }
  *dz1 = w.dz2;
  if (p->nonlinear) {
    if (g->gW2 && (rc = launch_gemm_tn(w.dz2, kQ, H1, kQ, N, w.tnpart, g->gW2, st))) return rc;
    if (g->gb2 && (rc = launch_colsum(w.dz2, kQ, N, w.cspart, g->gb2, st))) return rc;
    if (N > 0 && (rc = launch_linear<ACT_MASK_POS, true>(w.dz2, N, kQ, p->W2, nullptr, kQ, w.dz1, H1, 0, st))) return rc;
    *dz1 = w.dz1;
  }
  if (g->gW1 && (rc = launch_gemm_tn(*dz1, kQ, X, p->D, N, w.tnpart, g->gW1, st))) return rc;
  if (g->gb1 && (rc = launch_colsum(*dz1, kQ, N, w.cspart, g->gb1, st))) return rc;
  return 0;
}

int dsmil_backward(const dsmil_params_t* p, const float* X, const float* x_for_v, int64_t N, const float* Q,
                   const float* H1, const float* V, const float* A, const float* B, const int64_t* crit_idx,
                   const float* d_classes, const float* d_pred, const float* d_A, const float* d_B,
                   const dsmil_grads_t* g, const float* v_mask, void* workspace, size_t workspace_bytes,
                   void* stream) {
  int rc = check_params(p);
  if (rc) return rc;
  DSMIL_REQUIRE(N >= 1 && X && Q && A && B && crit_idx && g, "NULL tensor pointer or N < 1");
  DSMIL_REQUIRE(!p->nonlinear || H1, "nonlinear q backward needs saved H1");
  DSMIL_REQUIRE(!p->passing_v || V, "passing_v backward needs saved V");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int C = p->C, D = p->D;
  bool ok;
  BwdWs w = carve_bwd(p, N, g->gX != nullptr, workspace, workspace_bytes, &ok);
  if ((rc = check_workspace(w.bytes, ok, workspace, workspace_bytes))) return rc;
  const float* Xv = x_for_v ? x_for_v : X;
  // one rank: k_bwd_dL sums phase 1's partials of t itself (its summation order; no k_sum_partials launch)
  int gs;
  const float* dz1;
  if ((rc = bwd_phase1_impl(p, X, p->passing_v ? V : X, N, A, B, d_classes, d_pred, d_A, d_B, g, w.dA, w, &gs, st)) ||
      (rc = bwd_phase2_impl(p, N, A, w.dA, w.tpart, gs, Q, w.dqm, w, st)) ||
      (rc = bwd_phase3_impl(p, X, N, 0, Q, H1, w.dA, w.dqm, nullptr, crit_idx, g, w, &dz1, st)))
    return rc;

  const int ge = static_cast<int>(std::min<int64_t>(ceil_div(N * D, 256), kSms * 8));
  if (p->passing_v) {
    k_bwd_dzv<<<ge, 256, 0, st>>>(A, w.dB, V, N, C, D, w.dzv);
    DSMIL_LAUNCH_OK("k_bwd_dzv");
    if (g->gWv && (rc = launch_gemm_tn(w.dzv, D, Xv, D, N, w.tnpart, g->gWv, st))) return rc;
    if (g->gbv && (rc = launch_colsum(w.dzv, D, N, w.cspart, g->gbv, st))) return rc;
  }
  if (g->gX) {
    if ((rc = launch_linear<ACT_NONE, true>(dz1, N, kQ, p->W1, nullptr, D, g->gX, nullptr, 0, st))) return rc;
    k_bwd_dx_extra<<<ge, 256, 0, st>>>(d_classes, p->Wi, p->passing_v ? nullptr : A, w.dB, N, C, D, 1, g->gX);
    DSMIL_LAUNCH_OK("k_bwd_dx_extra");
    if (p->passing_v) {
      if ((rc = launch_linear<ACT_NONE, true>(w.dzv, N, D, p->Wv, nullptr, D, w.tmp, nullptr, 0, st))) return rc;
      k_axpy_mask<<<ge, 256, 0, st>>>(w.tmp, v_mask, N * D, g->gX);
      DSMIL_LAUNCH_OK("k_axpy_mask");
    }
  }
  return 0;
}

// ---- row-sharded backward: dsmil_backward's three phases, one per call (+ the caller's grad all-reduce) ----
int dsmil_shard_backward_phase1(const dsmil_params_t* p, const float* X, int64_t N, const float* A, const float* B,
                                const float* d_classes, const float* d_pred, float* dA, float* t_local, float* gWi,
                                float* gbi, float* gWf, float* gbf, void* workspace, size_t workspace_bytes,
                                void* stream) {
  int rc = check_params(p);
  if (rc) return rc;
  DSMIL_REQUIRE(!p->passing_v, "sharded backward supports the identity v only");
  DSMIL_REQUIRE(N >= 0 && B && t_local && (N == 0 || (X && A && dA)), "NULL tensor pointer or N < 0");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  bool ok;
  BwdWs w = carve_bwd(p, N, 0, workspace, workspace_bytes, &ok);
  if ((rc = check_workspace(w.bytes, ok, workspace, workspace_bytes))) return rc;
  dsmil_grads_t g{};
  g.gWi = gWi; g.gbi = gbi; g.gWf = gWf; g.gbf = gbf;
  int gs;
  if ((rc = bwd_phase1_impl(p, X, X, N, A, B, d_classes, d_pred, nullptr, nullptr, &g, dA, w, &gs, st))) return rc;
  if (N == 0) {
    DSMIL_CUDA_OK(cudaMemsetAsync(t_local, 0, sizeof(float) * p->C, st));
    return 0;
  }
  return launch_sum_partials(w.tpart, gs, p->C, t_local, st);
}

int dsmil_shard_backward_phase2(const dsmil_params_t* p, int64_t N, const float* A, float* dA, const float* t_global,
                                const float* Q, float* dqm_local, void* workspace, size_t workspace_bytes,
                                void* stream) {
  int rc = check_params(p);
  if (rc) return rc;
  DSMIL_REQUIRE(N >= 0 && t_global && dqm_local && (N == 0 || (A && dA && Q)), "NULL tensor pointer or N < 0");
  bool ok;
  BwdWs w = carve_bwd(p, N, 0, workspace, workspace_bytes, &ok);
  if ((rc = check_workspace(w.bytes, ok, workspace, workspace_bytes))) return rc;
  return bwd_phase2_impl(p, N, A, dA, t_global, 1, Q, dqm_local, w, static_cast<cudaStream_t>(stream));
}

int dsmil_shard_backward_phase3(const dsmil_params_t* p, const float* X, int64_t N, int64_t row_offset, const float* Q,
                                const float* H1, const float* dL, const float* dqm_global, const float* q_max,
                                const int64_t* crit_idx, float* gW1, float* gb1, float* gW2, float* gb2,
                                void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_params(p);
  if (rc) return rc;
  DSMIL_REQUIRE(N >= 0 && dqm_global && q_max && crit_idx && (N == 0 || (X && Q && dL)), "NULL tensor pointer or N < 0");
  DSMIL_REQUIRE(!p->nonlinear || N == 0 || H1, "nonlinear q backward needs saved H1");
  bool ok;
  BwdWs w = carve_bwd(p, N, 0, workspace, workspace_bytes, &ok);
  if ((rc = check_workspace(w.bytes, ok, workspace, workspace_bytes))) return rc;
  dsmil_grads_t g{};
  g.gW1 = gW1; g.gb1 = gb1; g.gW2 = gW2; g.gb2 = gb2;
  const float* dz1;
  return bwd_phase3_impl(p, X, N, row_offset, Q, H1, dL, dqm_global, q_max, crit_idx, &g, w, &dz1,
                         static_cast<cudaStream_t>(stream));
}

int dsmil_instance_scores_backward(const dsmil_params_t* p, const float* X, int64_t N, const float* d_classes,
                                   float* gWi, float* gbi, float* gX, void* workspace, size_t workspace_bytes,
                                   void* stream) {
  DSMIL_REQUIRE(p && p->Wi && p->C >= 1 && p->C <= DSMIL_MAX_C && p->D >= 1 && p->D <= DSMIL_MAX_D, "bad params");
  DSMIL_REQUIRE(N >= 1 && X && d_classes, "NULL tensor pointer or N < 1");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int C = p->C, D = p->D;
  Carver c(workspace, workspace_bytes);
  float* tnpart = c.take<float>(tn_partial_floats(C, D, N));
  float* cspart = c.take<float>(static_cast<size_t>(kSplits) * kMaxC);
  int rc = check_workspace(c.off, c.ok(), workspace, workspace_bytes);
  if (rc) return rc;
  if (gWi && (rc = launch_gemm_tn(d_classes, C, X, D, N, tnpart, gWi, st))) return rc;
  if (gbi && (rc = launch_colsum(d_classes, C, N, cspart, gbi, st))) return rc;
  if (gX) {
    const int ge = static_cast<int>(std::min<int64_t>(ceil_div(N * D, 256), kSms * 8));
    k_bwd_dx_extra<<<ge, 256, 0, st>>>(d_classes, p->Wi, nullptr, nullptr, N, C, D, 0, gX);
    DSMIL_LAUNCH_OK("k_bwd_dx_extra");
  }
  return 0;
}

// ---- batched training: forward that keeps Q/H1, and its backward over the bag table ------------------------------
struct BwdBagsWs {
  BagsPlan* plan;            // dev calls: the planner's live counts (G, nci, nc1 are then capacities); NULL: eager
  float* zero_row;           // dev calls: the stand-in bag row of a refused batch
  sm90::BagDev* table;
  TnChunk *chi, *ch1;        // chunk tables of gWi = d_classes^T X and gW1 = dz1^T X
  float *dB, *dA, *dL, *tpart, *dpart, *dqm, *dz2, *dz1, *tnpart, *cspart;
  long long* row_offsets;    // row-sharded batch only: [nb] device copy of each bag's first global row
  int G;                     // CTAs per bag of the per-row kernels (fixes their partial sums)
  bool gemv_i;               // gWi on the streaming kernel
  int nci, nc1;
  int64_t rps_i, rps_1;
  size_t bytes;
};
// `aligned`: every bag 16-byte aligned (the streaming gWi kernel needs it).  The carve reserves room for either gWi
// form, so the reported size does not depend on alignment.  `sharded` appends the row offsets of the row-sharded batch.
// The carve of w for nb bags, n packed rows and room for nchi gWi chunks, w.G / w.nc1 already set.
static void layout_bwd_bags(Carver& c, const dsmil_params_t* p, int nb, int64_t n, int nchi, bool sharded,
                            BwdBagsWs& w) {
  const int C = p->C, D = p->D;
  w.table = c.take<sm90::BagDev>(nb);
  w.chi = c.take<TnChunk>(nchi);
  w.ch1 = c.take<TnChunk>(w.nc1);
  w.dB = c.take<float>(static_cast<size_t>(nb) * C * D);
  w.dA = c.take<float>(n * C);
  w.dL = c.take<float>(n * C);
  w.tpart = c.take<float>(static_cast<size_t>(nb) * w.G * C);
  w.dpart = c.take<float>(static_cast<size_t>(nb) * w.G * C * kQ);
  w.dqm = c.take<float>(static_cast<size_t>(nb) * C * kQ);
  w.dz2 = c.take<float>(n * kQ);
  w.dz1 = p->nonlinear ? c.take<float>(n * kQ) : nullptr;
  size_t tn = static_cast<size_t>(nchi) * C * D;
  tn = std::max(tn, static_cast<size_t>(w.nc1) * kQ * D);
  tn = std::max(tn, tn_partial_floats(kQ, kQ, n));
  w.tnpart = c.take<float>(tn);
  w.cspart = c.take<float>(static_cast<size_t>(kSplits) * kQ);
  w.row_offsets = sharded ? c.take<long long>(nb) : nullptr;
}
static BwdBagsWs carve_bwd_bags(const dsmil_params_t* p, const int64_t* Ns, int nb, bool aligned, bool sharded,
                                void* ws, size_t cap, bool* ok) {
  Carver c(ws, cap);
  BwdBagsWs w;
  const int C = p->C, D = p->D;
  int64_t total = 0, mx = 1;
  for (int b = 0; b < nb; ++b) {
    total += Ns[b];
    mx = std::max<int64_t>(mx, Ns[b]);
  }
  w.plan = nullptr;
  w.zero_row = nullptr;
  w.G = bwd_bags_ctas(nb, mx);
  const bool gemv_ok = tn_use_gemv(C, D);
  w.gemv_i = gemv_ok && aligned;
  const int64_t rps_gemv = rag_rows_per_chunk(C, D, total, true), rps_tile = rag_rows_per_chunk(C, D, total, false);
  const int nci_gemv = gemv_ok ? rag_chunks(nullptr, Ns, nb, D, rps_gemv, nullptr) : 0;
  const int nci_tile = rag_chunks(nullptr, Ns, nb, D, rps_tile, nullptr);
  w.rps_i = w.gemv_i ? rps_gemv : rps_tile;
  w.nci = w.gemv_i ? nci_gemv : nci_tile;
  w.rps_1 = rag_rows_per_chunk(kQ, D, total, false);
  w.nc1 = rag_chunks(nullptr, Ns, nb, D, w.rps_1, nullptr);
  layout_bwd_bags(c, p, nb, std::max<int64_t>(total, 1), std::max(nci_gemv, nci_tile), sharded, w);
  w.bytes = c.off;
  *ok = c.ok();
  return w;
}
// A dev call's carve: every count at its capacity for nb bags of up to max_rows rows (bag_plan.cuh bounds the
// chunks), the bags 16-byte aligned, and the planner's BagsPlan at the end.
static BwdBagsWs carve_bwd_bags_dev(const dsmil_params_t* p, int nb, int64_t max_rows, void* ws, size_t cap,
                                    bool* ok) {
  Carver c(ws, cap);
  BwdBagsWs w;
  const int C = p->C, D = p->D;
  w.G = bwd_bags_ctas(nb, max_rows);
  w.gemv_i = tn_use_gemv(C, D);
  w.nci = rag_chunks_cap(C, D, w.gemv_i, nb);
  w.nc1 = rag_chunks_cap(kQ, D, false, nb);
  w.rps_i = w.rps_1 = 0;
  layout_bwd_bags(c, p, nb, static_cast<int64_t>(nb) * max_rows, w.nci, false, w);
  w.plan = c.take<BagsPlan>(1);
  w.zero_row = c.take<float>(D);
  w.bytes = c.off;
  *ok = c.ok();
  return w;
}

// The batched backward in three phases, cut at its two per-bag cross-row sums (t_b and dq_max_b), as bwd_phase1/2/3_impl
// are for one bag.  dsmil_backward_bags runs them in a row; the row-sharded batch runs one per call, with the caller's
// all-reduces in between.  Phase 1 uploads the bag and chunk tables into w; phases 2 and 3 read them from there.  In a
// dev call (w.plan != NULL) the planner has written the tables, `total` is the row capacity, and every launch that
// depends on the live rows reads its count from w.plan.

// Phase 1: dB, gWf/gbf, gWi/gbi, dA = X dB_b^T (+ d_A) into dA, and t_b's per-CTA partials in w.tpart (w.G per bag).
// V (eager passing_v): the packed V rows [total, D]; the table's X is then each bag's rows of V, so dA = V dB_b^T,
// while gWi and gW1 still reduce against the features Xs.
static int bwd_bags_phase1_impl(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int nb,
                                int64_t total, const float* A, const float* B, const float* d_classes,
                                const float* d_pred, const float* d_A, const float* d_B, const dsmil_grads_t* g,
                                float* dA, const BwdBagsWs& w, cudaStream_t st, const float* V = nullptr) {
  const int C = p->C, D = p->D;
  const BagsPlan* pl = w.plan;
  int rc;
  if (!pl) {
    // the kernels read X, N and row_off of the table (not the forward's tile and record numbering), at any alignment
    std::vector<sm90::BagDev> tbl(nb);
    long long row = 0;
    for (int b = 0; b < nb; ++b) {
      tbl[b] = sm90::BagDev{V ? V + row * D : Xs[b], Ns[b], row, 0, 0, 0, 0};
      row += Ns[b];
    }
    std::vector<TnChunk> chi(w.nci), ch1(w.nc1);
    rag_chunks(Xs, Ns, nb, D, w.rps_i, chi.data());
    rag_chunks(Xs, Ns, nb, D, w.rps_1, ch1.data());
    DSMIL_CUDA_OK(cudaMemcpyAsync(w.table, tbl.data(), sizeof(sm90::BagDev) * nb, cudaMemcpyHostToDevice, st));
    DSMIL_CUDA_OK(cudaMemcpyAsync(w.chi, chi.data(), sizeof(TnChunk) * w.nci, cudaMemcpyHostToDevice, st));
    DSMIL_CUDA_OK(cudaMemcpyAsync(w.ch1, ch1.data(), sizeof(TnChunk) * w.nc1, cudaMemcpyHostToDevice, st));
  }

  // bag classifier (dsmil.py:59-61) and B, summed over the bags
  k_bwd_bag_b<<<ceil_div(static_cast<int64_t>(C) * D, 256), 256, 0, st>>>(p->Wf, B, d_pred, d_B, nb, C, D, w.dB,
                                                                          g->gWf, g->gbf);
  DSMIL_LAUNCH_OK("k_bwd_bag_b");
  // instance classifier (dsmil.py:11)
  if (g->gWi) {
    if (d_classes) {
      if ((rc = launch_gemm_tn_rag(d_classes, C, D, w.chi, w.nci, w.gemv_i, w.tnpart, g->gWi, st, pl ? &pl->nci : nullptr)))
        return rc;
    }
    else DSMIL_CUDA_OK(cudaMemsetAsync(g->gWi, 0, sizeof(float) * C * D, st));
  }
  if (g->gbi) {
    if (d_classes) { if ((rc = launch_colsum(d_classes, C, total, w.cspart, g->gbi, st, pl ? &pl->cs : nullptr))) return rc; }
    else DSMIL_CUDA_OK(cudaMemsetAsync(g->gbi, 0, sizeof(float) * C, st));
  }
  // dA = X dB_b^T (+ d_A) and t_b's partials
  const size_t smem = sizeof(float) * C * D;
  if (smem > 48 * 1024)
    DSMIL_CUDA_OK(cudaFuncSetAttribute(k_bwd_rowdot_b, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_bwd_rowdot_b<<<dim3(w.G, nb), 256, smem, st>>>(w.table, D, w.dB, C, A, d_A, dA, w.tpart, pl ? &pl->G : nullptr);
  DSMIL_LAUNCH_OK("k_bwd_rowdot_b");
  return 0;
}

// Phase 2: dL = A (dA - t_b) / sqrt(128), t_b the sum of the P partials per bag in `tpart` (P == 0 in a dev call:
// phase 1's live G of them); dqm[b] = dL_b^T Q_b, summed over the CTAs' shares in a fixed order.
static int bwd_bags_phase2_impl(const dsmil_params_t* p, int nb, const float* A, const float* dA, const float* tpart,
                                int P, const float* Q, float* dL, float* dqm, const BwdBagsWs& w, cudaStream_t st) {
  const int C = p->C;
  const int* G_dev = w.plan ? &w.plan->G : nullptr;
  k_bwd_dL_b<<<dim3(w.G, nb), 256, 0, st>>>(w.table, C, A, dA, tpart, P, Q, dL, w.dpart, G_dev);
  DSMIL_LAUNCH_OK("k_bwd_dL_b");
  k_sum_segments<<<dim3(ceil_div(C * kQ, 256), nb), 256, 0, st>>>(w.dpart, w.G, C * kQ, dqm, G_dev);
  DSMIL_LAUNCH_OK("k_sum_segments");
  return 0;
}

// Phase 3: dQ -> dz2 (qmax / row_offsets as k_bwd_dq_b reads them: NULL when the critical rows are local), back through
// the Q-MLP into gW2/gb2 and gW1/gb1.  *dz1 is the layer-1 gradient it leaves in w.
static int bwd_bags_phase3_impl(const dsmil_params_t* p, int nb, int64_t total, const float* Q, const float* H1,
                                const float* dL, const float* dqm, const float* qmax, const int64_t* crit,
                                const long long* row_offsets, const dsmil_grads_t* g, const BwdBagsWs& w,
                                const float** dz1, cudaStream_t st) {
  const int D = p->D;
  const BagsPlan* pl = w.plan;
  int rc;
  k_bwd_dq_b<<<dim3(w.G, nb), 256, 0, st>>>(w.table, p->C, dL, Q, qmax, dqm, crit, row_offsets, p->nonlinear, w.dz2);
  DSMIL_LAUNCH_OK("k_bwd_dq_b");
  // back through the Q-MLP: layer 2 over the packed rows, layer 1 against the bags' X
  *dz1 = w.dz2;
  if (p->nonlinear) {
    if (g->gW2 && (rc = launch_gemm_tn(w.dz2, kQ, H1, kQ, total, w.tnpart, g->gW2, st, pl ? &pl->tn2 : nullptr)))
      return rc;
    if (g->gb2 && (rc = launch_colsum(w.dz2, kQ, total, w.cspart, g->gb2, st, pl ? &pl->cs : nullptr))) return rc;
    if ((rc = launch_linear<ACT_MASK_POS, true>(w.dz2, total, kQ, p->W2, nullptr, kQ, w.dz1, H1, 0, st,
                                                pl ? &pl->total : nullptr)))
      return rc;
    *dz1 = w.dz1;
  }
  if (g->gW1 &&
      (rc = launch_gemm_tn_rag(*dz1, kQ, D, w.ch1, w.nc1, false, w.tnpart, g->gW1, st, pl ? &pl->nc1 : nullptr)))
    return rc;
  if (g->gb1 && (rc = launch_colsum(*dz1, kQ, total, w.cspart, g->gb1, st, pl ? &pl->cs : nullptr))) return rc;
  return 0;
}

// The single-device batched backward over a carved w: the three phases in a row (+ gX).  One device: k_bwd_dL_b sums
// phase 1's partials of t itself, and the critical rows are local.
static int backward_bags_run(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int nb, int64_t total,
                             const float* Q, const float* H1, const float* A, const float* B, const int64_t* crit,
                             const float* d_classes, const float* d_pred, const float* d_A, const float* d_B,
                             const dsmil_grads_t* g, const BwdBagsWs& w, cudaStream_t st) {
  const int C = p->C, D = p->D;
  int rc;
  const float* dz1;
  if ((rc = bwd_bags_phase1_impl(p, Xs, Ns, nb, total, A, B, d_classes, d_pred, d_A, d_B, g, w.dA, w, st)) ||
      (rc = bwd_bags_phase2_impl(p, nb, A, w.dA, w.tpart, w.plan ? 0 : w.G, Q, w.dL, w.dqm, w, st)) ||
      (rc = bwd_bags_phase3_impl(p, nb, total, Q, H1, w.dL, w.dqm, nullptr, crit, nullptr, g, w, &dz1, st)))
    return rc;
  if (g->gX) {
    if ((rc = launch_linear<ACT_NONE, true>(dz1, total, kQ, p->W1, nullptr, D, g->gX, nullptr, 0, st))) return rc;
    k_bwd_dx_extra_b<<<dim3(w.G, nb), 256, 0, st>>>(w.table, d_classes, p->Wi, A, w.dB, C, D, g->gX);
    DSMIL_LAUNCH_OK("k_bwd_dx_extra_b");
  }
  return 0;
}

static int backward_bags_impl(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int nb,
                              int64_t total, bool aligned, const float* Q, const float* H1, const float* A,
                              const float* B, const int64_t* crit, const float* d_classes, const float* d_pred,
                              const float* d_A, const float* d_B, const dsmil_grads_t* g, void* ws, size_t ws_bytes,
                              cudaStream_t st) {
  bool ok;
  BwdBagsWs w = carve_bwd_bags(p, Ns, nb, aligned, false, ws, ws_bytes, &ok);
  int rc = check_workspace(w.bytes, ok, ws, ws_bytes);
  if (rc) return rc;
  return backward_bags_run(p, Xs, Ns, nb, total, Q, H1, A, B, crit, d_classes, d_pred, d_A, d_B, g, w, st);
}

// ---- batched value backward (passing_v): dsmil_backward_bags's phases over V, then the value network -------------
// The three phases run with the packed V in the table (dA = V dB_b^T).  Then dzv_b = (A_b dB_b) * [V_b > 0] for every
// bag in one k_linear_models launch (one LinSeg per bag: X = A rows, W = dB_b, K = C, aux = V rows), gWv = dzv^T Xv
// over chunks of the value inputs (k_gemm_tn_rag), gbv the column sums of dzv.  gX (eager only) adds dz1 W1,
// d_classes Wi (no A dB term: with a value network B weighs V, not X) and (dzv Wv) * the packed v mask.
struct ValueBwdWs {
  BwdBagsWs b;               // the identity-v backward's carve
  LinSeg* segs;              // [nb] dzv segments
  TnChunk* chv;              // gWv chunks over the value inputs
  float *dzv, *tmp;          // [total, D]; tmp (gX only) holds dzv Wv
  float *tnpart, *cspart;    // gWv's chunk partials, gbv's split partials
  sm90::BagDev* vtab;        // dev calls: the planner's value table [2 nb]
  int ncv;                   // gWv chunks (dev calls: the capacity, the live count in w.b.plan->pad_)
  int64_t rps_v;
  size_t bytes;
};
// The value tail's regions after w.b, for nb bags, n packed rows and w.ncv gWv chunks.
static void layout_value_bwd(Carver& c, const dsmil_params_t* p, int nb, int64_t n, bool need_gX, ValueBwdWs& w) {
  const int D = p->D;
  w.segs = c.take<LinSeg>(nb);
  w.chv = c.take<TnChunk>(w.ncv);
  w.dzv = c.take<float>(n * D);
  w.tmp = need_gX ? c.take<float>(n * D) : nullptr;
  w.tnpart = c.take<float>(static_cast<size_t>(w.ncv) * D * D);
  w.cspart = c.take<float>(static_cast<size_t>(kSplits) * D);
}
static ValueBwdWs carve_value_bwd(const dsmil_params_t* p, const int64_t* Ns, int nb, bool aligned, bool need_gX,
                                  void* ws, size_t cap, bool* ok) {
  ValueBwdWs w;
  const int D = p->D;
  w.b = carve_bwd_bags(p, Ns, nb, aligned, false, ws, cap, ok);
  int64_t total = 0;
  for (int b = 0; b < nb; ++b) total += Ns[b];
  w.rps_v = rag_rows_per_chunk(D, D, total, false);
  w.ncv = rag_chunks(nullptr, Ns, nb, D, w.rps_v, nullptr);
  w.vtab = nullptr;
  Carver c(ws, cap);
  c.off = w.b.bytes;
  layout_value_bwd(c, p, nb, std::max<int64_t>(total, 1), need_gX, w);
  w.bytes = c.off;
  *ok = c.ok() && *ok;
  return w;
}
// A dev call's carve: carve_bwd_bags_dev's, the value tail at its capacities (the gWv partials for
// rag_chunks_cap(D, D, false, nb) chunks) and the planner's value table.  The phases run on its second half (X = the
// packed V rows), w.b.table holds the planner's table of the features.
static ValueBwdWs carve_value_bwd_dev(const dsmil_params_t* p, int nb, int64_t max_rows, void* ws, size_t cap,
                                      bool* ok) {
  ValueBwdWs w;
  w.b = carve_bwd_bags_dev(p, nb, max_rows, ws, cap, ok);
  w.rps_v = 0;
  w.ncv = rag_chunks_cap(p->D, p->D, false, nb);
  Carver c(ws, cap);
  c.off = w.b.bytes;
  layout_value_bwd(c, p, nb, static_cast<int64_t>(nb) * max_rows, false, w);
  w.vtab = c.take<sm90::BagDev>(2 * static_cast<size_t>(nb));
  w.bytes = c.off;
  *ok = c.ok() && *ok;
  return w;
}

// The tile-form ragged GEMMs number their chunks in grid z.  gWi's tile form (unaligned bags) chunks the rows as gW1
// does (rag_splits is the same for C and 128 left columns), so nc1 bounds it at either alignment.
static bool value_bwd_grids_ok(const ValueBwdWs& w) { return w.ncv <= 65535 && w.b.nc1 <= 65535; }

// The value backward over tables already in w: the three phases with the packed V in w.b.table (dA = V dB_b^T), then
// dzv over w.segs, gWv over w.chv and gbv, and the eager call's gX.  mx: the largest bag (dev calls: max_rows).  In a
// dev call (w.b.plan != NULL) `total` is the row capacity and the GEMMs read their live counts from the plan.
static int value_backward_run(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int nb,
                              int64_t total, int64_t mx, const float* Q, const float* H1, const float* V,
                              const float* A, const float* B, const int64_t* crit, const float* d_classes,
                              const float* d_pred, const float* d_A, const float* d_B, const float* v_mask,
                              const dsmil_grads_t* g, const ValueBwdWs& w, cudaStream_t st) {
  const int C = p->C, D = p->D;
  const BwdBagsWs& wb = w.b;
  const BagsPlan* pl = wb.plan;
  int rc;
  const float* dz1;
  if ((rc = bwd_bags_phase1_impl(p, Xs, Ns, nb, total, A, B, d_classes, d_pred, d_A, d_B, g, wb.dA, wb, st, V)) ||
      (rc = bwd_bags_phase2_impl(p, nb, A, wb.dA, wb.tpart, pl ? 0 : wb.G, Q, wb.dL, wb.dqm, wb, st)) ||
      (rc = bwd_bags_phase3_impl(p, nb, total, Q, H1, wb.dL, wb.dqm, nullptr, crit, nullptr, g, wb, &dz1, st)))
    return rc;
  k_linear_models<ACT_MASK_POS, true><<<dim3(ceil_div(mx, LBM), ceil_div(D, LBN), nb), 256, 0, st>>>(w.segs, C, D);
  DSMIL_LAUNCH_OK("k_linear_models");
  if (g->gWv &&
      (rc = launch_gemm_tn_rag(w.dzv, D, D, w.chv, w.ncv, false, w.tnpart, g->gWv, st, pl ? &pl->pad_ : nullptr)))
    return rc;
  if (g->gbv && (rc = launch_colsum(w.dzv, D, total, w.cspart, g->gbv, st, pl ? &pl->cs : nullptr))) return rc;
  if (!g->gX) return 0;
  const int ge = static_cast<int>(std::min<int64_t>(ceil_div(total * D, 256), kSms * 8));
  if ((rc = launch_linear<ACT_NONE, true>(dz1, total, kQ, p->W1, nullptr, D, g->gX, nullptr, 0, st))) return rc;
  if (d_classes) {
    k_bwd_dx_extra<<<ge, 256, 0, st>>>(d_classes, p->Wi, nullptr, nullptr, total, C, D, 1, g->gX);
    DSMIL_LAUNCH_OK("k_bwd_dx_extra");
  }
  if ((rc = launch_linear<ACT_NONE, true>(w.dzv, total, D, p->Wv, nullptr, D, w.tmp, nullptr, 0, st))) return rc;
  k_axpy_mask<<<ge, 256, 0, st>>>(w.tmp, v_mask, total * D, g->gX);
  DSMIL_LAUNCH_OK("k_axpy_mask");
  return 0;
}

// The eager value backward: the dzv segments and the gWv chunks built on the host and uploaded, then the shared run
// (phase 1 uploads the V table and the chunks of gWi and gW1).
static int value_backward_bags_impl(const dsmil_params_t* p, const float* const* Xs, const float* const* XVs,
                                    const int64_t* Ns, int nb, int64_t total, const float* Q, const float* H1,
                                    const float* V, const float* A, const float* B, const int64_t* crit,
                                    const float* d_classes, const float* d_pred, const float* d_A, const float* d_B,
                                    const float* v_mask, const dsmil_grads_t* g, const ValueBwdWs& w,
                                    cudaStream_t st) {
  const int C = p->C, D = p->D;
  std::vector<LinSeg> segs(nb);
  std::vector<TnChunk> chv(w.ncv);
  int64_t row = 0, mx = 1;
  for (int b = 0; b < nb; ++b) {
    segs[b] = LinSeg{A + row * C, w.b.dB + static_cast<size_t>(b) * C * D, V + row * D, w.dzv + row * D, Ns[b]};
    mx = std::max<int64_t>(mx, Ns[b]);
    row += Ns[b];
  }
  rag_chunks(XVs ? XVs : Xs, Ns, nb, D, w.rps_v, chv.data());
  DSMIL_CUDA_OK(cudaMemcpyAsync(w.segs, segs.data(), sizeof(LinSeg) * nb, cudaMemcpyHostToDevice, st));
  DSMIL_CUDA_OK(cudaMemcpyAsync(w.chv, chv.data(), sizeof(TnChunk) * w.ncv, cudaMemcpyHostToDevice, st));
  return value_backward_run(p, Xs, Ns, nb, total, mx, Q, H1, V, A, B, crit, d_classes, d_pred, d_A, d_B, v_mask, g, w,
                            st);
}

// ---- sharded batch ABI ---------------------------------------------------------------------------
int dsmil_shard_bags_supported(const dsmil_params_t* p) {
  return (p && p->C >= 1 && p->C <= DSMIL_MAX_C && p->D >= 1 && p->D <= DSMIL_MAX_D && sm90::batched_supported(p)) ? 1 : 0;
}
// The batch numbers its bags in grid y (k_gather_cand_b, k_merge_cand, k_finalize_b): 1 <= nb <= 65535.
size_t dsmil_shard_bags_workspace_bytes(const dsmil_params_t* p, const int64_t* Ns, int32_t nb) {
  if (!dsmil_shard_bags_supported(p) || !Ns || nb < 1 || nb > 65535) return 0;
  bool ok;
  return carve_bags(p, Ns, nb, true, true, nullptr, 0, &ok).bytes;
}
// Phase 1 of the row-sharded batch: scores, arg-max keys and Q (+ H1 when non-NULL; Q tile-blocked when q_blocked),
// then each bag's candidate record.  A captured call reuses the table, row offsets and weight images of the preceding
// eager call: re-capture after a weight update.
static int shard_bags_phase1_impl(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int nb,
                                  const int64_t* row_offsets, float* classes, float* Q, float* H1, bool q_blocked,
                                  float* cand_recs, const BagsWs& w, cudaStream_t st) {
  const bool upload = !stream_is_capturing(st);
  int tiles, recs, rc;
  if ((rc = bags_phase1_impl(p, w, Xs, Ns, nb, nullptr, classes, Q, H1, q_blocked, upload, &tiles, &recs, st)))
    return rc;
  if (upload)
    DSMIL_CUDA_OK(cudaMemcpyAsync(w.row_offsets, row_offsets, sizeof(long long) * nb, cudaMemcpyHostToDevice, st));
  sm90::k_gather_cand_b<<<dim3(p->C, nb), kQ, 0, st>>>(w.table, w.keys, classes, Q, q_blocked, w.row_offsets, p->C,
                                                        cand_recs);
  DSMIL_LAUNCH_OK("k_gather_cand_b");
  return 0;
}
// Phase 2: merge the G ranks' candidates into q_max [nb,C,128] and crit_idx, attend on the local rows, and each bag's
// partial record.  Attend runs one CTA per partial record: `recs` of them, or, with recs_dev, the first *recs_dev of a
// capacity grid of `recs`.
static int shard_bags_phase2_impl(const dsmil_params_t* p, int nb, const float* Q, bool q_blocked,
                                  const float* cands_all, int G, float* A, int64_t* crit_idx, float* qmax,
                                  float* recs_out, const BagsWs& w, int recs, const int* recs_dev, cudaStream_t st) {
  int rc;
  k_merge_cand<<<dim3(p->C, nb), kQ, 0, st>>>(cands_all, G, nb, p->C, qmax, crit_idx);
  DSMIL_LAUNCH_OK("k_merge_cand");
  sm90::AttendArgs aa{w.table, nb, p->D, p->C, Q, q_blocked, w.keys, A, w.recs, qmax, recs_dev};
  if ((rc = sm90::launch_attend_b(aa, recs, st))) return rc;
  sm90::FinalizeArgs fa{w.table, p->D, p->C, w.recs, w.keys, p->Wf, p->bf, A, nullptr, nullptr, nullptr,
                         w.pred_part, w.counters, recs_out, 0, 0};
  return sm90::launch_finalize_b(fa, nb, st);
}

int dsmil_shard_bags_phase1(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                            const int64_t* row_offsets, float* classes, float* cand_recs, void* workspace,
                            size_t workspace_bytes, void* stream) {
  int rc = check_params(p, true);
  if (rc) return rc;
  DSMIL_REQUIRE(dsmil_shard_bags_supported(p), "shape not supported by the batched tensor-core path");
  DSMIL_REQUIRE(Xs && Ns && row_offsets && classes && cand_recs, "NULL pointer");
  DSMIL_REQUIRE(nb >= 1 && nb <= 65535, "nb=%d outside [1, 65535]", nb);
  bool ok;
  BagsWs w = carve_bags(p, Ns, nb, true, true, workspace, workspace_bytes, &ok);
  if ((rc = check_workspace(w.bytes, ok, workspace, workspace_bytes))) return rc;
  return shard_bags_phase1_impl(p, Xs, Ns, nb, row_offsets, classes, w.Q, nullptr, true, cand_recs, w,
                                static_cast<cudaStream_t>(stream));
}
int dsmil_shard_bags_phase2(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                            const float* cands_all, int32_t G, float* A, int64_t* crit_idx, float* recs_out,
                            void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_params(p, true);
  if (rc) return rc;
  DSMIL_REQUIRE(dsmil_shard_bags_supported(p) && Xs && Ns && cands_all && G >= 1 && A && crit_idx && recs_out,
                "bad arguments");
  DSMIL_REQUIRE(nb >= 1 && nb <= 65535, "nb=%d outside [1, 65535]", nb);
  bool ok;
  BagsWs w = carve_bags(p, Ns, nb, true, true, workspace, workspace_bytes, &ok);
  if ((rc = check_workspace(w.bytes, ok, workspace, workspace_bytes))) return rc;
  std::vector<sm90::BagDev> tbl;
  int tiles, recs;
  if ((rc = build_table(Xs, Ns, nb, tbl, &tiles, &recs))) return rc;   // the device table was written by phase 1
  return shard_bags_phase2_impl(p, nb, w.Q, true, cands_all, G, A, crit_idx, w.qmax, recs_out, w, recs, nullptr,
                                static_cast<cudaStream_t>(stream));
}
int dsmil_shard_bags_phase3(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                            const float* recs_all, int32_t G, float* A, float* B, float* pred, void* workspace,
                            size_t workspace_bytes, void* stream) {
  int rc = check_params(p, true);
  if (rc) return rc;
  DSMIL_REQUIRE(dsmil_shard_bags_supported(p) && Xs && Ns && recs_all && G >= 1 && G <= sm90::kMaxRecPerBag && A && B && pred,
                "bad arguments");
  DSMIL_REQUIRE(nb >= 1 && nb <= 65535, "nb=%d outside [1, 65535]", nb);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  bool ok;
  BagsWs w = carve_bags(p, Ns, nb, true, true, workspace, workspace_bytes, &ok);
  if ((rc = check_workspace(w.bytes, ok, workspace, workspace_bytes))) return rc;
  sm90::FinalizeArgs fa{w.table, p->D, p->C, recs_all, w.keys, p->Wf, p->bf, A, B, pred, nullptr,
                         w.pred_part, w.counters, nullptr, G, nb};
  return sm90::launch_finalize_b(fa, nb, st);
}


// ---- batched training ------------------------------------------------------------------------------
size_t dsmil_forward_bags_train_workspace_bytes(const dsmil_params_t* p, const int64_t* Ns, int32_t nb) {
  if (!p || p->passing_v) return 0;
  return dsmil_forward_bags_workspace_bytes(p, Ns, nb);
}

int dsmil_forward_bags_train(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                             float* classes, float* pred, float* A, float* B, int64_t* crit_idx, float* save_Q,
                             float* save_H1, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_params(p, true);
  if (rc) return rc;
  DSMIL_REQUIRE(!p->passing_v, "batched training supports the identity v only (passing_v: one bag per call)");
  DSMIL_REQUIRE(Xs && Ns && nb >= 1 && classes && pred && A && B && crit_idx && save_Q && (!p->nonlinear || save_H1),
                "NULL pointer or nb < 1");
  int64_t total;
  bool aligned;
  if ((rc = check_bags(Xs, Ns, nb, &total, &aligned))) return rc;
  if ((rc = need_workspace(dsmil_forward_bags_train_workspace_bytes(p, Ns, nb), workspace, workspace_bytes))) return rc;
  return forward_bags_route(p, Xs, nullptr, Ns, nb, aligned, classes, pred, A, B, crit_idx, save_Q, save_H1, nullptr,
                            workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

size_t dsmil_backward_bags_workspace_bytes(const dsmil_params_t* p, const int64_t* Ns, int32_t nb, int need_gX) {
  (void)need_gX;   // gX is the caller's buffer: the identity-v backward needs no scratch for it
  if (!p || !Ns || nb < 1 || p->passing_v || p->C < 1 || p->C > DSMIL_MAX_C || p->D < 1 || p->D > DSMIL_MAX_D) return 0;
  for (int b = 0; b < nb; ++b)
    if (Ns[b] < 0) return 0;
  bool ok;
  return carve_bwd_bags(p, Ns, nb, true, false, nullptr, 0, &ok).bytes;
}

int dsmil_backward_bags(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                        const float* Q, const float* H1, const float* A, const float* B, const int64_t* crit_idx,
                        const float* d_classes, const float* d_pred, const float* d_A, const float* d_B,
                        const dsmil_grads_t* grads, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_params(p);
  if (rc) return rc;
  DSMIL_REQUIRE(!p->passing_v, "batched backward supports the identity v only (passing_v: dsmil_backward per bag)");
  DSMIL_REQUIRE(Xs && Ns && nb >= 1 && nb <= 65535 && Q && A && B && crit_idx && grads,
                "NULL pointer or nb outside [1, 65535]");
  DSMIL_REQUIRE(!p->nonlinear || H1, "nonlinear q backward needs saved H1");
  DSMIL_REQUIRE(!(grads->gX && d_classes) || p->Wi, "gX through d_classes needs Wi");
  int64_t total;
  bool aligned;
  if ((rc = check_bags(Xs, Ns, nb, &total, &aligned))) return rc;
  const size_t need = dsmil_backward_bags_workspace_bytes(p, Ns, nb, grads->gX != nullptr);
  if ((rc = need_workspace(need, workspace, workspace_bytes))) return rc;
  return backward_bags_impl(p, Xs, Ns, nb, total, aligned, Q, H1, A, B, crit_idx, d_classes, d_pred, d_A, d_B, grads,
                            workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

// ---- the fold models of a cross-validation in one training step: each model over its own bags ---------------------
// Model m's bags are entries [bag[m], bag[m + 1]) of Xs / Ns; its rows start at packed row row[m].  Per-row buffers are
// packed model-major, and so are the per-bag ones.
struct ModelsBags {
  std::vector<int> bag;
  std::vector<int64_t> row;
  int ne;          // entries: the bags of all models
  bool aligned;    // every bag 16-byte aligned
};
static int check_models_bags(const dsmil_params_t* ps, int M, const float* const* Xs, const int64_t* Ns,
                             const int32_t* nbs, ModelsBags* mb) {
  int rc = check_models(ps, M);
  if (rc) return rc;
  DSMIL_REQUIRE(!ps[0].passing_v, "batched training supports the identity v only (passing_v: one bag per call)");
  DSMIL_REQUIRE(Xs && Ns && nbs, "NULL bag list");
  mb->bag.assign(M + 1, 0);
  mb->row.assign(M + 1, 0);
  for (int m = 0; m < M; ++m) {
    DSMIL_REQUIRE(nbs[m] >= 1 && nbs[m] <= 65535, "model %d: nb=%d outside [1, 65535]", m, nbs[m]);
    mb->bag[m + 1] = mb->bag[m] + nbs[m];
  }
  mb->ne = mb->bag[M];
  for (int m = 0; m < M; ++m) {
    int64_t rows;
    bool al;
    if ((rc = check_bags(Xs + mb->bag[m], Ns + mb->bag[m], nbs[m], &rows, &al))) return rc;
    mb->row[m + 1] = mb->row[m] + rows;
    mb->aligned = (m == 0 || mb->aligned) && al;
  }
  return 0;
}
// The loop route gives each model its own slice of the workspace, 256-byte aligned.
static size_t ws_slice(size_t bytes) { return (bytes + 255) & ~size_t(255); }

size_t dsmil_forward_bags_models_train_workspace_bytes(const dsmil_params_t* ps, int32_t M, const int64_t* Ns,
                                                       const int32_t* nbs) {
  if (!ps || M < 1 || M > sm90::kMaxModels || !Ns || !nbs) return 0;
  size_t loop = 0;
  int ne = 0;
  for (int m = 0; m < M; ++m) {
    if (nbs[m] < 1) return 0;
    const size_t b = dsmil_forward_bags_train_workspace_bytes(&ps[m], Ns + ne, nbs[m]);
    if (b == 0) return 0;
    loop += ws_slice(b);
    ne += nbs[m];
  }
  bool ok;
  if (!models_batched(ps, M)) return loop;
  return std::max(loop, carve_models(&ps[0], M, Ns, ne, 1, false, nullptr, 0, &ok).bytes);
}

int dsmil_forward_bags_models_train(const dsmil_params_t* ps, int32_t M, const float* const* Xs, const int64_t* Ns,
                                    const int32_t* nbs, float* classes, float* pred, float* A, float* B,
                                    int64_t* crit_idx, float* save_Q, float* save_H1, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  ModelsBags mb;
  int rc = check_models_bags(ps, M, Xs, Ns, nbs, &mb);
  if (rc) return rc;
  DSMIL_REQUIRE(classes && pred && A && B && crit_idx && save_Q && (!ps[0].nonlinear || save_H1),
                "NULL output pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t need = dsmil_forward_bags_models_train_workspace_bytes(ps, M, Ns, nbs);
  if ((rc = need_workspace(need, workspace, workspace_bytes))) return rc;
  const int C = ps[0].C, D = ps[0].D;
  if (mb.aligned && dsmil_models_supported(ps, M) && mb.ne <= 65535) {
    bool ok;
    ModelsWs w = carve_models(&ps[0], M, Ns, mb.ne, 1, false, workspace, workspace_bytes, &ok);
    if ((rc = check_workspace(w.bytes, ok, workspace, workspace_bytes))) return rc;
    // entry e is bag e of the list, its model in pad_; rows and tiles numbered across all models
    std::vector<sm90::BagDev> tbl(mb.ne);
    long long row = 0;
    int tile = 0, rec = 0;
    for (int m = 0; m < M; ++m)
      for (int e = mb.bag[m]; e < mb.bag[m + 1]; ++e) {
        tbl[e] = bag_entry(Xs[e], Ns[e], row, tile, rec);
        tbl[e].pad_ = m;
      }
    return models_launch(ps, M, w, tbl, tile, rec, classes, save_Q, save_H1, false, pred, A, B, crit_idx, 0, st);
  }
  // off the fused route: each model's dsmil_forward_bags_train into its slices
  size_t off = 0;
  for (int m = 0; m < M; ++m) {
    const int b0 = mb.bag[m];
    const int64_t r0 = mb.row[m];
    const size_t wb = dsmil_forward_bags_train_workspace_bytes(&ps[m], Ns + b0, nbs[m]);
    rc = dsmil_forward_bags_train(&ps[m], Xs + b0, Ns + b0, nbs[m], classes + r0 * C, pred + static_cast<size_t>(b0) * C,
                                  A + r0 * C, B + static_cast<size_t>(b0) * C * D, crit_idx + static_cast<size_t>(b0) * C,
                                  save_Q + r0 * kQ, save_H1 ? save_H1 + r0 * kQ : nullptr,
                                  static_cast<char*>(workspace) + off, wb, stream);
    if (rc) return rc;
    off += ws_slice(wb);
  }
  return 0;
}

// The fused backward's host plan: every split the one-model backward would choose for each model's own batch, on
// the model-major packing.  Xs == NULL: counts only (the workspace size); H1 may then be NULL too.
struct BwdModelsPlan {
  std::vector<sm90::BagDev> table;                 // per entry: X, N, row_off; tile_off = G_m, rec_off, pad_ = m
  std::vector<TnChunk> chi, ch1, ch2, chc;         // gWi, gW1, gW2 and the column sums' chunks
  std::vector<int> nci, nc1, nc2, ncs;             // per model
  int Gmax = 1, slots = 0;                         // largest G, per-CTA partial slots of all entries
  int64_t max_rows = 1;                            // rows of the largest model
};
static void plan_bwd_models(const dsmil_params_t* ps, int M, const float* const* Xs, const int64_t* Ns,
                            const int32_t* nbs, const float* H1, BwdModelsPlan& pl) {
  const int C = ps[0].C, D = ps[0].D;
  pl.nci.assign(M, 0); pl.nc1.assign(M, 0); pl.nc2.assign(M, 0); pl.ncs.assign(M, 0);
  int e = 0;
  long long row = 0;
  for (int m = 0; m < M; ++m) {
    const int nb = nbs[m];
    const int64_t* N = Ns + e;
    int64_t total = 0, mx = 1;
    for (int b = 0; b < nb; ++b) {
      total += N[b];
      mx = std::max<int64_t>(mx, N[b]);
    }
    const long long r0 = row;
    const ModelSplits sp = model_splits(C, D, nb, total, mx);
    const int G = sp.G;
    pl.Gmax = std::max(pl.Gmax, G);
    pl.max_rows = std::max(pl.max_rows, total);
    for (int b = 0; b < nb; ++b, ++e) {
      pl.table.push_back(sm90::BagDev{Xs ? Xs[e] : nullptr, N[b], row, G, pl.slots, 0, m});
      row += N[b];
      pl.slots += G;
    }
    // gWi and gW1: chunks of each bag's rows, as carve_bwd_bags cuts them
    const BagList L{Xs ? Xs + (e - nb) : nullptr, N, nullptr};
    auto rag = [&](std::vector<TnChunk>& out, int64_t rps) {
      const int n = rag_chunks_list(L, nb, D, rps, r0, nullptr);
      const size_t at = out.size();
      out.resize(at + n);
      if (Xs) rag_chunks_list(L, nb, D, rps, r0, out.data() + at);
      return n;
    };
    pl.nci[m] = rag(pl.chi, sp.rps_i);
    pl.nc1[m] = rag(pl.ch1, sp.rps_1);
    // gW2 = dz2^T H1 and the column sums: launch_gemm_tn's tile form and launch_colsum split the model's rows
    for (int z = 0; z < sp.t2.S; ++z) pl.ch2.push_back(split_chunk(sp.t2, z, r0, H1, kQ));
    for (int z = 0; z < sp.cs.S; ++z) pl.chc.push_back(split_chunk(sp.cs, z, r0, nullptr, 0));
    pl.nc2[m] = sp.t2.S;
    pl.ncs[m] = sp.cs.S;
  }
}

struct BwdModelsWs {
  sm90::BagDev* table;
  BwdModelDev* models;
  TnChunk *chi, *ch1, *ch2, *chc;
  SumSeg* segs;              // [6][M]: gWi, gbi, gW2, gb2, gW1, gb1
  LinSeg* lin;               // [2][M]: dz1, gX
  float *dB, *dA, *dL, *tpart, *dpart, *dqm, *dz2, *dz1, *part;
  size_t bytes;
};
static BwdModelsWs carve_bwd_models(const dsmil_params_t* ps, int M, const BwdModelsPlan& pl, int64_t total,
                                    void* ws, size_t cap, bool* ok) {
  const int C = ps[0].C, D = ps[0].D;
  const size_t ne = pl.table.size(), T = std::max<int64_t>(total, 1);
  Carver c(ws, cap);
  BwdModelsWs w;
  w.table = c.take<sm90::BagDev>(ne);
  w.models = c.take<BwdModelDev>(M);
  w.chi = c.take<TnChunk>(pl.chi.size());
  w.ch1 = c.take<TnChunk>(pl.ch1.size());
  w.ch2 = c.take<TnChunk>(pl.ch2.size());
  w.chc = c.take<TnChunk>(pl.chc.size());
  w.segs = c.take<SumSeg>(6 * M);
  w.lin = c.take<LinSeg>(2 * M);
  w.dB = c.take<float>(ne * C * D);
  w.dA = c.take<float>(T * C);
  w.dL = c.take<float>(T * C);
  w.tpart = c.take<float>(static_cast<size_t>(pl.slots) * C);
  w.dpart = c.take<float>(static_cast<size_t>(pl.slots) * C * kQ);
  w.dqm = c.take<float>(ne * C * kQ);
  w.dz2 = c.take<float>(T * kQ);
  w.dz1 = c.take<float>(T * kQ);
  size_t part = pl.chi.size() * C * D;
  part = std::max(part, pl.ch1.size() * kQ * D);
  part = std::max(part, pl.ch2.size() * kQ * kQ);
  part = std::max(part, pl.chc.size() * kQ);
  w.part = c.take<float>(part);
  w.bytes = c.off;
  *ok = c.ok();
  return w;
}

// The fused backward's launches over the tables in w: one per stage for all M models.  The grids are those of gr; in a
// dev call they are capacities, the tables are the planner's and the live chunk counts are read from gr.live.
struct BwdModelsGrid {
  int Gmax, nci, nc1, nc2, ncs;   // per-row CTAs per entry, and the chunks of gWi, gW1, gW2 and the column sums
  int64_t max_rows;               // rows of the largest model
  bool any_gX;
  const ModelsPlan* live;         // dev call: the planner's counts (device memory); NULL: eager
  bool linear_q;                  // generic fold calls of a linear q: no layer 2, dz1 is dz2
};
static int bwd_models_launch(int C, int D, int M, int ne, const BwdModelsWs& w, const BwdModelsGrid& gr,
                             const float* Q, const float* H1, const float* A, const float* B, const int64_t* crit,
                             const float* d_classes, const float* d_pred, const float* d_A, const float* d_B,
                             cudaStream_t st) {
  const ModelsPlan* live = gr.live;
  int rc;
  // each model's partials into its gradients: reduction r of the six
  auto sums = [&](int r, int64_t L) -> int {
    k_sum_partials_models<<<dim3(static_cast<unsigned>(ceil_div(L, 32)), M), 256, 0, st>>>(w.part, w.segs + r * M, L);
    DSMIL_LAUNCH_OK("k_sum_partials_models");
    return 0;
  };
  auto colsums = [&](const float* P, int L, int r) -> int {
    k_colsum_rag<<<static_cast<unsigned>(gr.ncs), 256, 0, st>>>(P, L, w.chc, w.part);
    DSMIL_LAUNCH_OK("k_colsum_rag");
    return sums(r, L);
  };
  const dim3 per_entry(gr.Gmax, ne);
  // phase 1: bag classifier, instance classifier, dA and t's partials
  k_bwd_bag_models<<<dim3(ceil_div(static_cast<int64_t>(C) * D, 256), M), 256, 0, st>>>(w.models, B, d_pred, d_B, C,
                                                                                       D, w.dB);
  DSMIL_LAUNCH_OK("k_bwd_bag_models");
  if (d_classes) {
    const int nz = gr.nci;
    const int* nzd = live ? &live->nci : nullptr;
    if (tn_use_gemv(C, D)) {
      switch (C) {
        case 1: k_gemv_tn_rag<1><<<nz, 256, 0, st>>>(d_classes, D, w.chi, w.part, nzd); break;
        case 2: k_gemv_tn_rag<2><<<nz, 256, 0, st>>>(d_classes, D, w.chi, w.part, nzd); break;
        case 3: k_gemv_tn_rag<3><<<nz, 256, 0, st>>>(d_classes, D, w.chi, w.part, nzd); break;
        default: k_gemv_tn_rag<4><<<nz, 256, 0, st>>>(d_classes, D, w.chi, w.part, nzd); break;
      }
      DSMIL_LAUNCH_OK("k_gemv_tn_rag");
    } else {
      k_gemm_tn_rag<<<dim3(ceil_div(D, TBM), ceil_div(C, TBM), nz), 256, 0, st>>>(d_classes, C, D, w.chi, w.part,
                                                                                 nzd);
      DSMIL_LAUNCH_OK("k_gemm_tn_rag");
    }
    if ((rc = sums(0, static_cast<int64_t>(C) * D)) || (rc = colsums(d_classes, C, 1))) return rc;
  }
  const size_t smem = sizeof(float) * C * D;
  if (smem > 48 * 1024)
    DSMIL_CUDA_OK(cudaFuncSetAttribute(k_bwd_rowdot_models, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_bwd_rowdot_models<<<per_entry, 256, smem, st>>>(w.table, D, w.dB, C, A, d_A, w.dA, w.tpart);
  DSMIL_LAUNCH_OK("k_bwd_rowdot_models");
  // phase 2: dL and dq_max
  k_bwd_dL_models<<<per_entry, 256, 0, st>>>(w.table, C, A, w.dA, w.tpart, Q, w.dL, w.dpart);
  DSMIL_LAUNCH_OK("k_bwd_dL_models");
  k_sum_segments_models<<<dim3(ceil_div(C * kQ, 256), ne), 256, 0, st>>>(w.table, w.dpart, C * kQ, w.dqm);
  DSMIL_LAUNCH_OK("k_sum_segments_models");
  // phase 3: dz2, back through the Q-MLP (through the tanh and layer 2 for a nonlinear q)
  k_bwd_dq_b<<<per_entry, 256, 0, st>>>(w.table, C, w.dL, Q, nullptr, w.dqm, crit, nullptr, gr.linear_q ? 0 : 1, w.dz2);
  DSMIL_LAUNCH_OK("k_bwd_dq_b");
  const unsigned row_tiles = static_cast<unsigned>(ceil_div(gr.max_rows, LBM));
  const float* dz1 = w.dz2;
  if (!gr.linear_q) {
    k_gemm_tn_rag<<<dim3(1, 1, static_cast<unsigned>(gr.nc2)), 256, 0, st>>>(w.dz2, kQ, kQ, w.ch2, w.part,
                                                                             live ? &live->nc2 : nullptr);
    DSMIL_LAUNCH_OK("k_gemm_tn_rag");
    if ((rc = sums(2, static_cast<int64_t>(kQ) * kQ)) || (rc = colsums(w.dz2, kQ, 3))) return rc;
    k_linear_models<ACT_MASK_POS, true><<<dim3(row_tiles, 1, M), 256, 0, st>>>(w.lin, kQ, kQ);
    DSMIL_LAUNCH_OK("k_linear_models");
    dz1 = w.dz1;
  }
  k_gemm_tn_rag<<<dim3(ceil_div(D, TBM), 1, static_cast<unsigned>(gr.nc1)), 256, 0, st>>>(
      dz1, kQ, D, w.ch1, w.part, live ? &live->nc1 : nullptr);
  DSMIL_LAUNCH_OK("k_gemm_tn_rag");
  if ((rc = sums(4, static_cast<int64_t>(kQ) * D)) || (rc = colsums(dz1, kQ, 5))) return rc;
  if (gr.any_gX) {
    k_linear_models<ACT_NONE, true><<<dim3(row_tiles, ceil_div(D, LBN), M), 256, 0, st>>>(w.lin + M, kQ, D);
    DSMIL_LAUNCH_OK("k_linear_models");
    k_bwd_dx_extra_models<<<per_entry, 256, 0, st>>>(w.table, w.models, d_classes, A, w.dB, C, D);
    DSMIL_LAUNCH_OK("k_bwd_dx_extra_models");
  }
  return 0;
}

// One launch per stage for all M models (nonlinear q, C <= 4: the dsmil_models_supported shapes; aligned bags).
static int backward_bags_models_impl(const dsmil_params_t* ps, int M, const float* const* Xs, const int64_t* Ns,
                                     const int32_t* nbs, const ModelsBags& mb, const float* Q, const float* H1,
                                     const float* A, const float* B, const int64_t* crit, const float* d_classes,
                                     const float* d_pred, const float* d_A, const float* d_B,
                                     const dsmil_grads_t* g, void* ws, size_t ws_bytes, cudaStream_t st) {
  const int C = ps[0].C, D = ps[0].D, ne = mb.ne;
  BwdModelsPlan pl;
  plan_bwd_models(ps, M, Xs, Ns, nbs, H1, pl);
  bool ok;
  BwdModelsWs w = carve_bwd_models(ps, M, pl, mb.row[M], ws, ws_bytes, &ok);
  int rc = check_workspace(w.bytes, ok, ws, ws_bytes);
  if (rc) return rc;
  std::vector<BwdModelDev> md(M);
  std::vector<SumSeg> segs(6 * M);
  std::vector<LinSeg> lin(2 * M);
  bool any_gX = false;
  int zi = 0, z1 = 0, z2 = 0;
  for (int m = 0; m < M; ++m) {
    const long long r0 = mb.row[m], rows = mb.row[m + 1] - r0;
    md[m] = BwdModelDev{ps[m].Wf, ps[m].Wi, g[m].gWf, g[m].gbf, g[m].gX, mb.bag[m], nbs[m], r0};
    const bool dc = d_classes != nullptr;
    segs[0 * M + m] = SumSeg{dc ? g[m].gWi : nullptr, zi, pl.nci[m]};
    segs[1 * M + m] = SumSeg{dc ? g[m].gbi : nullptr, 0, 0};   // z0 filled below: the column-sum chunks
    segs[2 * M + m] = SumSeg{g[m].gW2, z2, pl.nc2[m]};
    segs[3 * M + m] = SumSeg{g[m].gb2, 0, 0};
    segs[4 * M + m] = SumSeg{g[m].gW1, z1, pl.nc1[m]};
    segs[5 * M + m] = SumSeg{g[m].gb1, 0, 0};
    zi += pl.nci[m];
    z1 += pl.nc1[m];
    z2 += pl.nc2[m];
    lin[m] = LinSeg{w.dz2 + r0 * kQ, ps[m].W2, H1 + r0 * kQ, w.dz1 + r0 * kQ, rows};
    lin[M + m] = LinSeg{w.dz1 + r0 * kQ, ps[m].W1, nullptr, g[m].gX, rows};
    any_gX = any_gX || g[m].gX != nullptr;
    if (!dc) {   // no gradient through the scores: zero instance-classifier gradients, as the one-model call
      if (g[m].gWi) DSMIL_CUDA_OK(cudaMemsetAsync(g[m].gWi, 0, sizeof(float) * C * D, st));
      if (g[m].gbi) DSMIL_CUDA_OK(cudaMemsetAsync(g[m].gbi, 0, sizeof(float) * C, st));
    }
  }
  for (int m = 0, zc = 0; m < M; zc += pl.ncs[m], ++m)
    for (int r : {1, 3, 5}) {
      segs[r * M + m].z0 = zc;
      segs[r * M + m].S = pl.ncs[m];
    }
  DSMIL_CUDA_OK(cudaMemcpyAsync(w.table, pl.table.data(), sizeof(sm90::BagDev) * ne, cudaMemcpyHostToDevice, st));
  DSMIL_CUDA_OK(cudaMemcpyAsync(w.models, md.data(), sizeof(BwdModelDev) * M, cudaMemcpyHostToDevice, st));
  DSMIL_CUDA_OK(cudaMemcpyAsync(w.chi, pl.chi.data(), sizeof(TnChunk) * pl.chi.size(), cudaMemcpyHostToDevice, st));
  DSMIL_CUDA_OK(cudaMemcpyAsync(w.ch1, pl.ch1.data(), sizeof(TnChunk) * pl.ch1.size(), cudaMemcpyHostToDevice, st));
  DSMIL_CUDA_OK(cudaMemcpyAsync(w.ch2, pl.ch2.data(), sizeof(TnChunk) * pl.ch2.size(), cudaMemcpyHostToDevice, st));
  DSMIL_CUDA_OK(cudaMemcpyAsync(w.chc, pl.chc.data(), sizeof(TnChunk) * pl.chc.size(), cudaMemcpyHostToDevice, st));
  DSMIL_CUDA_OK(cudaMemcpyAsync(w.segs, segs.data(), sizeof(SumSeg) * 6 * M, cudaMemcpyHostToDevice, st));
  DSMIL_CUDA_OK(cudaMemcpyAsync(w.lin, lin.data(), sizeof(LinSeg) * 2 * M, cudaMemcpyHostToDevice, st));

  BwdModelsGrid gr{pl.Gmax, static_cast<int>(pl.chi.size()), static_cast<int>(pl.ch1.size()),
                   static_cast<int>(pl.ch2.size()), static_cast<int>(pl.chc.size()), pl.max_rows, any_gX, nullptr};
  return bwd_models_launch(C, D, M, ne, w, gr, Q, H1, A, B, crit, d_classes, d_pred, d_A, d_B, st);
}
// Whether the fused backward takes these members and bags: the forward's fused shapes, aligned bags, and every grid
// within its limits.
static bool bwd_models_fused(const dsmil_params_t* ps, int M, const int64_t* Ns, const int32_t* nbs, int ne,
                             bool aligned) {
  if (!aligned || ne > 65535 || !dsmil_models_supported(ps, M)) return false;
  BwdModelsPlan pl;
  plan_bwd_models(ps, M, nullptr, Ns, nbs, nullptr, pl);
  return pl.chi.size() <= 65535 && pl.ch1.size() <= 65535 && pl.ch2.size() <= 65535;
}

size_t dsmil_backward_bags_models_workspace_bytes(const dsmil_params_t* ps, int32_t M, const int64_t* Ns,
                                                  const int32_t* nbs, int need_gX) {
  if (!ps || M < 1 || M > sm90::kMaxModels || !Ns || !nbs) return 0;
  size_t bytes = 0;
  int ne = 0;
  for (int m = 0; m < M; ++m) {
    if (nbs[m] < 1) return 0;
    const size_t b = dsmil_backward_bags_workspace_bytes(&ps[m], Ns + ne, nbs[m], need_gX);
    if (b == 0) return 0;
    bytes += ws_slice(b);
    ne += nbs[m];
  }
  if (!models_batched(ps, M)) return bytes;
  // the fused layout on every batched shape, so the size grows with M, the bags and the rows alike
  BwdModelsPlan pl;
  plan_bwd_models(ps, M, nullptr, Ns, nbs, nullptr, pl);
  int64_t total = 0;
  for (int e = 0; e < ne; ++e) total += Ns[e];
  bool ok;
  return std::max(bytes, carve_bwd_models(ps, M, pl, total, nullptr, 0, &ok).bytes);
}

int dsmil_backward_bags_models(const dsmil_params_t* ps, int32_t M, const float* const* Xs, const int64_t* Ns,
                               const int32_t* nbs, const float* Q, const float* H1, const float* A, const float* B,
                               const int64_t* crit_idx, const float* d_classes, const float* d_pred, const float* d_A,
                               const float* d_B, const dsmil_grads_t* grads, void* workspace, size_t workspace_bytes,
                               void* stream) {
  ModelsBags mb;
  int rc = check_models_bags(ps, M, Xs, Ns, nbs, &mb);
  if (rc) return rc;
  DSMIL_REQUIRE(Q && A && B && crit_idx && grads, "NULL pointer");
  DSMIL_REQUIRE(!ps[0].nonlinear || H1, "nonlinear q backward needs saved H1");
  bool gX = false;
  for (int m = 0; m < M; ++m) gX = gX || grads[m].gX != nullptr;
  const size_t need = dsmil_backward_bags_models_workspace_bytes(ps, M, Ns, nbs, gX);
  if ((rc = need_workspace(need, workspace, workspace_bytes))) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (bwd_models_fused(ps, M, Ns, nbs, mb.ne, mb.aligned))
    return backward_bags_models_impl(ps, M, Xs, Ns, nbs, mb, Q, H1, A, B, crit_idx, d_classes, d_pred, d_A, d_B, grads,
                                     workspace, workspace_bytes, st);
  // off the fused route: each model's dsmil_backward_bags on its slices
  const int C = ps[0].C, D = ps[0].D;
  size_t off = 0;
  for (int m = 0; m < M; ++m) {
    const int b0 = mb.bag[m];
    const int64_t r0 = mb.row[m];
    const size_t bo = static_cast<size_t>(b0);
    const size_t wb = dsmil_backward_bags_workspace_bytes(&ps[m], Ns + b0, nbs[m], gX);
    rc = dsmil_backward_bags(&ps[m], Xs + b0, Ns + b0, nbs[m], Q + r0 * kQ, H1 ? H1 + r0 * kQ : nullptr, A + r0 * C,
                             B + bo * C * D, crit_idx + bo * C, d_classes ? d_classes + r0 * C : nullptr,
                             d_pred ? d_pred + bo * C : nullptr, d_A ? d_A + r0 * C : nullptr,
                             d_B ? d_B + bo * C * D : nullptr, &grads[m], static_cast<char*>(workspace) + off, wb,
                             stream);
    if (rc) return rc;
    off += ws_slice(wb);
  }
  return 0;
}


// ---- row-sharded batch training: phases 1 and 2 that keep Q and H1 row-major, and the backward in three calls -------
// What every call of it checks: the batched sharded shapes, identity v, 1 <= nb <= 65535, and at least one local row
// in every bag (need_X == false: a phase that reads no features checks the row counts only).
static int check_shard_bags_train(const dsmil_params_t* p, bool need_scores, const float* const* Xs, bool need_X,
                                  const int64_t* Ns, int nb, int64_t* total, bool* aligned) {
  int rc = check_params(p, need_scores);
  if (rc) return rc;
  DSMIL_REQUIRE(!p->passing_v, "row-sharded batched training supports the identity v only");
  DSMIL_REQUIRE(dsmil_shard_bags_supported(p), "shape not supported by the batched tensor-core path");
  DSMIL_REQUIRE(Ns && (Xs || !need_X) && nb >= 1 && nb <= 65535, "NULL pointer or nb outside [1, 65535]");
  return check_bags(need_X ? Xs : nullptr, Ns, nb, total, aligned);
}

int dsmil_shard_bags_phase1_train(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                                  const int64_t* row_offsets, float* classes, float* save_Q, float* save_H1,
                                  float* cand_recs, void* workspace, size_t workspace_bytes, void* stream) {
  int64_t total;
  bool aligned;
  int rc = check_shard_bags_train(p, true, Xs, true, Ns, nb, &total, &aligned);
  if (rc) return rc;
  DSMIL_REQUIRE(row_offsets && classes && save_Q && save_H1 && cand_recs, "NULL pointer");
  bool ok;
  BagsWs w = carve_bags(p, Ns, nb, true, true, workspace, workspace_bytes, &ok);
  if ((rc = check_workspace(w.bytes, ok, workspace, workspace_bytes))) return rc;
  return shard_bags_phase1_impl(p, Xs, Ns, nb, row_offsets, classes, save_Q, save_H1, false, cand_recs, w,
                                static_cast<cudaStream_t>(stream));
}

int dsmil_shard_bags_phase2_train(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                                  const float* Q, const float* cands_all, int32_t G, float* A, int64_t* crit_idx,
                                  float* q_max, float* recs_out, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  int64_t total;
  bool aligned;
  int rc = check_shard_bags_train(p, true, Xs, true, Ns, nb, &total, &aligned);
  if (rc) return rc;
  DSMIL_REQUIRE(Q && cands_all && G >= 1 && A && crit_idx && q_max && recs_out, "NULL pointer or G < 1");
  bool ok;
  BagsWs w = carve_bags(p, Ns, nb, true, true, workspace, workspace_bytes, &ok);
  if ((rc = check_workspace(w.bytes, ok, workspace, workspace_bytes))) return rc;
  std::vector<sm90::BagDev> tbl;
  int tiles, recs;
  if ((rc = build_table(Xs, Ns, nb, tbl, &tiles, &recs))) return rc;   // the device table was written by phase 1
  return shard_bags_phase2_impl(p, nb, Q, false, cands_all, G, A, crit_idx, q_max, recs_out, w, recs, nullptr,
                                static_cast<cudaStream_t>(stream));
}

size_t dsmil_shard_backward_bags_workspace_bytes(const dsmil_params_t* p, const int64_t* Ns, int32_t nb) {
  if (!dsmil_shard_bags_supported(p) || !Ns || nb < 1 || nb > 65535) return 0;
  for (int b = 0; b < nb; ++b)
    if (Ns[b] < 0) return 0;
  bool ok;
  return carve_bwd_bags(p, Ns, nb, true, true, nullptr, 0, &ok).bytes;
}

int dsmil_shard_backward_bags_phase1(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                                     const float* A, const float* B, const float* d_classes_local,
                                     const float* d_pred, float* dA_local, float* t_local, float* gWi, float* gbi,
                                     float* gWf, float* gbf, void* workspace, size_t workspace_bytes, void* stream) {
  int64_t total;
  bool aligned;
  int rc = check_shard_bags_train(p, false, Xs, true, Ns, nb, &total, &aligned);
  if (rc) return rc;
  DSMIL_REQUIRE(A && B && dA_local && t_local, "NULL tensor pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  bool ok;
  BwdBagsWs w = carve_bwd_bags(p, Ns, nb, aligned, true, workspace, workspace_bytes, &ok);
  if ((rc = check_workspace(w.bytes, ok, workspace, workspace_bytes))) return rc;
  dsmil_grads_t g{};
  g.gWi = gWi; g.gbi = gbi; g.gWf = gWf; g.gbf = gbf;
  if ((rc = bwd_bags_phase1_impl(p, Xs, Ns, nb, total, A, B, d_classes_local, d_pred, nullptr, nullptr, &g, dA_local,
                                 w, st)))
    return rc;
  // t_local[b] = the per-CTA partials summed in a fixed order: with one rank, phase 2 then sees the t_b that
  // dsmil_backward_bags's k_bwd_dL_b forms itself
  k_sum_segments<<<dim3(ceil_div(p->C, 256), nb), 256, 0, st>>>(w.tpart, w.G, p->C, t_local, nullptr);
  DSMIL_LAUNCH_OK("k_sum_segments");
  return 0;
}

int dsmil_shard_backward_bags_phase2(const dsmil_params_t* p, const int64_t* Ns, int32_t nb, const float* A,
                                     float* dA_to_dL, const float* t_global, const float* Q, float* dqm_local,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  int64_t total;
  bool aligned;
  int rc = check_shard_bags_train(p, false, nullptr, false, Ns, nb, &total, &aligned);
  if (rc) return rc;
  DSMIL_REQUIRE(A && dA_to_dL && t_global && Q && dqm_local, "NULL tensor pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  bool ok;
  BwdBagsWs w = carve_bwd_bags(p, Ns, nb, true, true, workspace, workspace_bytes, &ok);
  if ((rc = check_workspace(w.bytes, ok, workspace, workspace_bytes))) return rc;
  // k_bwd_dL_b reads dA and writes dL from different threads: it reads a copy so that dL can replace dA
  DSMIL_CUDA_OK(cudaMemcpyAsync(w.dA, dA_to_dL, sizeof(float) * total * p->C, cudaMemcpyDeviceToDevice, st));
  return bwd_bags_phase2_impl(p, nb, A, w.dA, t_global, 1, Q, dA_to_dL, dqm_local, w, st);
}

int dsmil_shard_backward_bags_phase3(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                                     const int64_t* row_offsets, const float* Q, const float* H1, const float* dL_local,
                                     const float* dqm_global, const float* q_max, const int64_t* crit_idx,
                                     float* gW1, float* gb1, float* gW2, float* gb2, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  int64_t total;
  bool aligned;
  int rc = check_shard_bags_train(p, false, Xs, true, Ns, nb, &total, &aligned);
  if (rc) return rc;
  DSMIL_REQUIRE(row_offsets && Q && H1 && dL_local && dqm_global && q_max && crit_idx, "NULL tensor pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  bool ok;
  BwdBagsWs w = carve_bwd_bags(p, Ns, nb, aligned, true, workspace, workspace_bytes, &ok);
  if ((rc = check_workspace(w.bytes, ok, workspace, workspace_bytes))) return rc;
  DSMIL_CUDA_OK(cudaMemcpyAsync(w.row_offsets, row_offsets, sizeof(long long) * nb, cudaMemcpyHostToDevice, st));
  dsmil_grads_t g{};
  g.gW1 = gW1; g.gb1 = gb1; g.gW2 = gW2; g.gb2 = gb2;
  const float* dz1;
  return bwd_bags_phase3_impl(p, nb, total, Q, H1, dL_local, dqm_global, q_max, crit_idx, w.row_offsets, &g, w, &dz1,
                              st);
}


// ---- capture-safe batched training: the bag list in device memory, every launch sized for a capacity -------------
// Three routes (Route): the tensor-core batch (dsmil_*_dev, planned by k_plan_bags), the generic shapes
// (dsmil_generic_*_dev, planned by k_plan_bags_gen) and the value network (dsmil_value_*_dev: the generic batch of a
// passing_v model, planned by k_plan_bags_gen with its value tables).  Each pair of calls shares one body.
static bool dev_shape(Route r, const dsmil_params_t* p) {
  if (r == ROUTE_TC) return dsmil_shard_bags_supported(p) != 0;
  return (r == ROUTE_VAL ? dsmil_value_bags_supported(p) : dsmil_generic_bags_supported(p)) != 0;
}
// The batch every dev call sizes: 1 <= nb <= 65535 bags of at most max_rows < 2^32 rows.
static bool dev_sizes(int nb, int64_t max_rows) {
  return nb >= 1 && nb <= 65535 && max_rows >= 1 && max_rows < 0xffffffffll;
}
// The 128-row tiles of nb bags of max_rows rows, which the kernels number in an int (twice over off the tensor-core
// route, for k_linear_b's grid).
static bool dev_tiles_ok(Route r, int nb, int64_t max_rows) {
  return (r == ROUTE_TC ? 1 : 2) * static_cast<int64_t>(nb) * ((max_rows + sm90::kTileM - 1) / sm90::kTileM) <= INT_MAX;
}
// A dev call's workspace is never below the eager call's for the same capacity: one buffer serves both forms.
static size_t not_below_eager(size_t dev, size_t (*eager)(const dsmil_params_t*, const int64_t*, int32_t),
                              const dsmil_params_t* p, int nb, int64_t max_rows) {
  const std::vector<int64_t> Ns(nb, max_rows);
  return std::max(dev, eager(p, Ns.data(), nb));
}

// What every dev call checks: the route's shapes, the bag list and status (need_list: the calls that run the planner),
// 1 <= nb <= 65535 and a row capacity whose 128-row tiles the kernels can number in an int (twice over on the generic
// route, for k_linear_b's grid).
static int check_bags_dev(Route r, const dsmil_params_t* p, bool need_scores, bool need_list, const float* const* Xs,
                          const int64_t* Ns, int nb, int64_t max_rows, const int32_t* status) {
  int rc = check_params(p, need_scores);
  if (rc) return rc;
  if (r == ROUTE_TC)
    DSMIL_REQUIRE(dsmil_shard_bags_supported(p),
                  "shape not supported by the batched tensor-core path (D=%d, C=%d, nonlinear=%d, passing_v=%d)", p->D,
                  p->C, p->nonlinear, p->passing_v);
  else if (r == ROUTE_VAL)
    DSMIL_REQUIRE(dsmil_value_bags_supported(p),
                  "the value calls take passing_v models with Wv and bv (D=%d, C=%d, nonlinear=%d, passing_v=%d)",
                  p->D, p->C, p->nonlinear, p->passing_v);
  else
    DSMIL_REQUIRE(dsmil_generic_bags_supported(p),
                  "shape not on the generic batched route, i.e. identity v off dsmil_shard_bags_supported (D=%d, C=%d, "
                  "nonlinear=%d, passing_v=%d)", p->D, p->C, p->nonlinear, p->passing_v);
  DSMIL_REQUIRE(!need_list || (Xs && Ns && status), "NULL bag list or status");
  DSMIL_REQUIRE(nb >= 1 && nb <= 65535, "nb=%d outside [1, 65535]", nb);
  DSMIL_REQUIRE(max_rows >= 1 && max_rows < 0xffffffffll && dev_tiles_ok(r, nb, max_rows),
                "max_rows=%lld out of range for nb=%d", (long long)max_rows, nb);
  return 0;
}

// The route's planner over the device bag list: the table, the live counts and, when chi / ch1 are non-NULL, the
// backward's chunk tables; on the value route also the value tables of v.
static int launch_plan_dev(Route r, const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int nb,
                           int64_t max_rows, float* zero_row, sm90::BagDev* table, TnChunk* chi, TnChunk* ch1,
                           BagsPlan* plan, int32_t* status, cudaStream_t st, const PlanValue& v = PlanValue{}) {
  if (r == ROUTE_TC) {
    k_plan_bags<<<1, 32, 0, st>>>(Xs, Ns, nb, max_rows, p->C, p->D, zero_row, table, chi, ch1, plan, status, nullptr,
                                  nullptr);
    DSMIL_LAUNCH_OK("k_plan_bags");
  } else {
    // the alignment rule (gen_bag_aligned) keeps each form the eager call would choose: gWi streams (tn_use_gemv) only
    // where D % 4 == 0, and there the bags are 16-byte aligned
    k_plan_bags_gen<<<1, 32, 0, st>>>(Xs, Ns, nb, max_rows, p->C, p->D, zero_row, table, chi, ch1, plan, status, v);
    DSMIL_LAUNCH_OK("k_plan_bags_gen");
  }
  return 0;
}

// The forward's carve for nb bags of max_rows rows (need_Q: the tile blocks of Q for the capacity tiles, as inference
// keeps them; otherwise Q and H1 are the caller's; `sharded` adds the row offsets and q_max of the row-sharded batch),
// then the planner's BagsPlan and the zero row of a refused batch.
static BagsWs carve_bags_dev(const dsmil_params_t* p, int nb, int64_t max_rows, bool need_Q, bool sharded, void* ws,
                             size_t cap, bool* ok, BagsPlan** plan, float** zero_row) {
  const std::vector<int64_t> Ns(nb, max_rows);
  BagsWs w = carve_bags(p, Ns.data(), nb, need_Q, sharded, ws, cap, ok);
  Carver c(ws, cap);
  c.off = w.bytes;
  *plan = c.take<BagsPlan>(1);
  *zero_row = c.take<float>(p->D);
  w.bytes = c.off;
  *ok = c.ok();
  return w;
}

// bags_phase1_impl's launches in a dev call, on the planner's table (k_qmlp_sm90 on the capacity grid of 128-row
// tiles), with the weight images rebuilt on every call: a replayed graph sees the weights of the last optimizer step.
// q_blocked: Q in tile blocks (inference).  overlap: as bags_phase1_impl's, on the grid it gives the capacity tiles.
static int bags_phase1_dev(const dsmil_params_t* p, const BagsWs& w, const BagsPlan* plan, int nb, int64_t max_rows,
                           float* classes, float* Q, float* H1, cudaStream_t st, bool q_blocked = false,
                           bool overlap = false) {
  int rc;
  DSMIL_CUDA_OK(cudaMemsetAsync(w.keys, 0, sizeof(unsigned long long) * (kMaxC + 1) * nb, st));
  if ((rc = sm90::launch_prep_wimg(p, w.wimg, st))) return rc;
  const int tiles = nb * tiles_for_bag(max_rows);
  return sm90::launch_qmlp(p, w.table, nb, tiles, classes, w.keys, Q, H1, w.wimg,
                           overlap ? overlap_phase1_ctas(tiles) : num_sms(), st, q_blocked, &plan->tiles,
                           overlap ? w.done : nullptr);
}

// The forward pair's size: train keeps Q (+ H1) in the caller's saves, inference in the workspace.
static size_t forward_bags_dev_ws(Route r, bool train, const dsmil_params_t* p, int nb, int64_t max_rows) {
  if (!dev_shape(r, p) || !dev_sizes(nb, max_rows)) return 0;
  if (r == ROUTE_VAL && !dev_tiles_ok(r, nb, max_rows)) return 0;   // the value calls size no batch they refuse
  bool ok;
  size_t dev;
  if (r == ROUTE_TC) {
    BagsPlan* plan;
    float* zero_row;
    dev = carve_bags_dev(p, nb, max_rows, !train, false, nullptr, 0, &ok, &plan, &zero_row).bytes;
  } else {
    dev = carve_gen_dev(p, nb, max_rows, train, nullptr, 0, &ok).bytes;
  }
  if (r == ROUTE_VAL) return not_below_eager(dev, dsmil_value_forward_bags_workspace_bytes, p, nb, max_rows);
  return not_below_eager(dev, train ? dsmil_forward_bags_train_workspace_bytes : dsmil_forward_bags_workspace_bytes, p,
                         nb, max_rows);
}

// The forward pair's body: the planner writes the table and the live counts, then the route's forward runs on the
// capacity grids.  train: Q (+ H1) into save_Q (save_H1).  Inference keeps Q in the workspace (tile blocks on the
// tensor-core route), and there the attend pass is a programmatic dependent of phase 1 as in dsmil_forward_bags --
// under stream capture too, where the launch attribute becomes a programmatic edge of the graph (DESIGN §4.3).  Only
// kernel timing keeps the plain launch.  The value route (XVs_dev: the value inputs, NULL: the features) also keeps
// V in save_V when training, and runs the value projection of the planner's value table.
static int forward_bags_dev(Route r, bool train, const dsmil_params_t* p, const float* const* Xs_dev,
                            const int64_t* Ns_dev, int nb, int64_t max_rows, float* classes, float* pred, float* A,
                            float* B, int64_t* crit_idx, float* save_Q, float* save_H1, int32_t* status,
                            void* workspace, size_t workspace_bytes, cudaStream_t st,
                            const float* const* XVs_dev = nullptr, float* save_V = nullptr) {
  int rc = check_bags_dev(r, p, true, true, Xs_dev, Ns_dev, nb, max_rows, status);
  if (rc) return rc;
  DSMIL_REQUIRE(classes && pred && A && B &&
                    (!train || (crit_idx && save_Q && (!p->nonlinear || save_H1) && (r != ROUTE_VAL || save_V))),
                "NULL output pointer");
  if ((rc = need_workspace(forward_bags_dev_ws(r, train, p, nb, max_rows), workspace, workspace_bytes))) return rc;
  bool ok;
  if (r != ROUTE_TC) {
    GenWs w = carve_gen_dev(p, nb, max_rows, train, workspace, workspace_bytes, &ok);
    float* V = r == ROUTE_VAL ? (train ? save_V : w.V) : nullptr;
    if ((rc = launch_plan_dev(r, p, Xs_dev, Ns_dev, nb, max_rows, w.zero_row, w.table, nullptr, nullptr, w.plan, status,
                              st, PlanValue{XVs_dev, V, nullptr, nullptr, nullptr, w.vtab, nullptr, nullptr})))
      return rc;
    return gen_forward_run(p, w, nb, nb * max_rows, nb * tiles_for_bag(max_rows), nb * attend_ctas(max_rows), max_rows,
                           classes, pred, A, B, crit_idx ? crit_idx : w.crit, train ? save_Q : w.Q,
                           p->nonlinear ? (train ? save_H1 : w.H1) : nullptr, V, st);
  }
  BagsPlan* plan;
  float* zero_row;
  BagsWs w = carve_bags_dev(p, nb, max_rows, !train, false, workspace, workspace_bytes, &ok, &plan, &zero_row);
  if ((rc = launch_plan_dev(r, p, Xs_dev, Ns_dev, nb, max_rows, zero_row, w.table, nullptr, nullptr, plan, status, st)))
    return rc;
  const bool overlap = !train && !g_prof_on;
  float* Q = train ? save_Q : w.Q;
  if ((rc = bags_phase1_dev(p, w, plan, nb, max_rows, classes, Q, train ? save_H1 : nullptr, st, !train, overlap)))
    return rc;
  return bags_attend_finalize(p, w, nb, Q, !train, pred, A, B, crit_idx, nb * recs_for_bag(max_rows), &plan->recs, st,
                              overlap);
}

// The backward pair's ragged GEMMs launch one CTA per chunk of the capacity in grid z (k_gemm_tn_rag) or x
// (k_gemv_tn_rag), which holds at most 65535 of them: rag_splits plus one short chunk per bag (and on the value
// route the chunks of gWv).
static bool dev_chunks_ok(Route r, const dsmil_params_t* p, int nb) {
  return rag_chunks_cap(p->C, p->D, true, nb) <= 65535 && rag_chunks_cap(p->C, p->D, false, nb) <= 65535 &&
         rag_chunks_cap(kQ, p->D, false, nb) <= 65535 &&
         (r != ROUTE_VAL || rag_chunks_cap(p->D, p->D, false, nb) <= 65535);
}
// The backward pair's size.  The generic and value routes also cover the eager backward's carve (without gX).
static size_t backward_bags_dev_ws(Route r, const dsmil_params_t* p, int nb, int64_t max_rows) {
  if (!dev_shape(r, p) || !dev_sizes(nb, max_rows) || !dev_chunks_ok(r, p, nb)) return 0;
  bool ok;
  if (r == ROUTE_VAL && !dev_tiles_ok(r, nb, max_rows)) return 0;
  if (r == ROUTE_VAL)
    return not_below_eager(carve_value_bwd_dev(p, nb, max_rows, nullptr, 0, &ok).bytes,
                           [](const dsmil_params_t* q, const int64_t* Ns, int32_t n) {
                             return dsmil_value_backward_bags_workspace_bytes(q, Ns, n, 0);
                           }, p, nb, max_rows);
  const size_t dev = carve_bwd_bags_dev(p, nb, max_rows, nullptr, 0, &ok).bytes;
  if (r == ROUTE_TC) return dev;
  return not_below_eager(dev, [](const dsmil_params_t* q, const int64_t* Ns, int32_t n) {
    return dsmil_backward_bags_workspace_bytes(q, Ns, n, 0);
  }, p, nb, max_rows);
}

// The backward pair's body: the planner writes the bag and chunk tables, then the three phases run on the capacity
// grids.  The value route (XVs_dev, V: the forward's value inputs and saved V) has the planner write the value tables
// too, and runs the value backward's phases over the V half of its value table, then its dzv, gWv and gbv.
static int backward_bags_dev(Route r, const dsmil_params_t* p, const float* const* Xs_dev, const int64_t* Ns_dev,
                             int nb, int64_t max_rows, const float* Q, const float* H1, const float* A, const float* B,
                             const int64_t* crit_idx, const float* d_classes, const float* d_pred, const float* d_A,
                             const float* d_B, const dsmil_grads_t* grads, int32_t* status, void* workspace,
                             size_t workspace_bytes, cudaStream_t st, const float* const* XVs_dev = nullptr,
                             const float* V = nullptr) {
  int rc = check_bags_dev(r, p, false, true, Xs_dev, Ns_dev, nb, max_rows, status);
  if (rc) return rc;
  DSMIL_REQUIRE(Q && (!p->nonlinear || H1) && A && B && crit_idx && grads && (r != ROUTE_VAL || V), "NULL pointer");
  DSMIL_REQUIRE(!d_A && !d_B && !grads->gX,
                "the dev backward takes gradients through classes and pred only (no d_A, d_B or gX)");
  DSMIL_REQUIRE(dev_chunks_ok(r, p, nb), "nb=%d: the chunk capacity of the ragged GEMMs passes 65535", nb);
  if ((rc = need_workspace(backward_bags_dev_ws(r, p, nb, max_rows), workspace, workspace_bytes))) return rc;
  bool ok;
  if (r == ROUTE_VAL) {
    ValueBwdWs w = carve_value_bwd_dev(p, nb, max_rows, workspace, workspace_bytes, &ok);
    if ((rc = launch_plan_dev(r, p, Xs_dev, Ns_dev, nb, max_rows, w.b.zero_row, w.b.table, w.b.chi, w.b.ch1, w.b.plan,
                              status, st, PlanValue{XVs_dev, V, A, w.b.dB, w.dzv, w.vtab, w.segs, w.chv})))
      return rc;
    w.b.table = w.vtab + nb;   // the phases weigh V: dA = V dB_b^T
    return value_backward_run(p, nullptr, nullptr, nb, static_cast<int64_t>(nb) * max_rows, max_rows, Q, H1, V, A, B,
                              crit_idx, d_classes, d_pred, nullptr, nullptr, nullptr, grads, w, st);
  }
  BwdBagsWs w = carve_bwd_bags_dev(p, nb, max_rows, workspace, workspace_bytes, &ok);
  if ((rc = launch_plan_dev(r, p, Xs_dev, Ns_dev, nb, max_rows, w.zero_row, w.table, w.chi, w.ch1, w.plan, status,
                            st)))
    return rc;
  return backward_bags_run(p, nullptr, nullptr, nb, static_cast<int64_t>(nb) * max_rows, Q, H1, A, B, crit_idx,
                           d_classes, d_pred, nullptr, nullptr, grads, w, st);
}

size_t dsmil_forward_bags_train_dev_workspace_bytes(const dsmil_params_t* p, int32_t nb, int64_t max_rows) {
  return forward_bags_dev_ws(ROUTE_TC, true, p, nb, max_rows);
}
int dsmil_forward_bags_train_dev(const dsmil_params_t* p, const float* const* Xs_dev, const int64_t* Ns_dev,
                                 int32_t nb, int64_t max_rows, float* classes, float* pred, float* A, float* B,
                                 int64_t* crit_idx, float* save_Q, float* save_H1, int32_t* status, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  return forward_bags_dev(ROUTE_TC, true, p, Xs_dev, Ns_dev, nb, max_rows, classes, pred, A, B, crit_idx, save_Q,
                          save_H1, status, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

size_t dsmil_forward_bags_dev_workspace_bytes(const dsmil_params_t* p, int32_t nb, int64_t max_rows) {
  return forward_bags_dev_ws(ROUTE_TC, false, p, nb, max_rows);
}
int dsmil_forward_bags_dev(const dsmil_params_t* p, const float* const* Xs_dev, const int64_t* Ns_dev, int32_t nb,
                           int64_t max_rows, float* classes, float* pred, float* A, float* B, int64_t* crit_idx,
                           int32_t* status, void* workspace, size_t workspace_bytes, void* stream) {
  return forward_bags_dev(ROUTE_TC, false, p, Xs_dev, Ns_dev, nb, max_rows, classes, pred, A, B, crit_idx, nullptr,
                          nullptr, status, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

size_t dsmil_backward_bags_dev_workspace_bytes(const dsmil_params_t* p, int32_t nb, int64_t max_rows) {
  return backward_bags_dev_ws(ROUTE_TC, p, nb, max_rows);
}
int dsmil_backward_bags_dev(const dsmil_params_t* p, const float* const* Xs_dev, const int64_t* Ns_dev, int32_t nb,
                            int64_t max_rows, const float* Q, const float* H1, const float* A, const float* B,
                            const int64_t* crit_idx, const float* d_classes, const float* d_pred, const float* d_A,
                            const float* d_B, const dsmil_grads_t* grads, int32_t* status, void* workspace,
                            size_t workspace_bytes, void* stream) {
  return backward_bags_dev(ROUTE_TC, p, Xs_dev, Ns_dev, nb, max_rows, Q, H1, A, B, crit_idx, d_classes, d_pred, d_A,
                           d_B, grads, status, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

int dsmil_generic_bags_supported(const dsmil_params_t* p) {
  return (p && p->C >= 1 && p->C <= DSMIL_MAX_C && p->D >= 1 && p->D <= DSMIL_MAX_D && gen_shape(p)) ? 1 : 0;
}

size_t dsmil_generic_forward_bags_train_dev_workspace_bytes(const dsmil_params_t* p, int32_t nb, int64_t max_rows) {
  return forward_bags_dev_ws(ROUTE_GEN, true, p, nb, max_rows);
}
int dsmil_generic_forward_bags_train_dev(const dsmil_params_t* p, const float* const* Xs_dev, const int64_t* Ns_dev,
                                         int32_t nb, int64_t max_rows, float* classes, float* pred, float* A, float* B,
                                         int64_t* crit_idx, float* save_Q, float* save_H1, int32_t* status,
                                         void* workspace, size_t workspace_bytes, void* stream) {
  return forward_bags_dev(ROUTE_GEN, true, p, Xs_dev, Ns_dev, nb, max_rows, classes, pred, A, B, crit_idx, save_Q,
                          save_H1, status, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

size_t dsmil_generic_forward_bags_dev_workspace_bytes(const dsmil_params_t* p, int32_t nb, int64_t max_rows) {
  return forward_bags_dev_ws(ROUTE_GEN, false, p, nb, max_rows);
}
int dsmil_generic_forward_bags_dev(const dsmil_params_t* p, const float* const* Xs_dev, const int64_t* Ns_dev,
                                   int32_t nb, int64_t max_rows, float* classes, float* pred, float* A, float* B,
                                   int64_t* crit_idx, int32_t* status, void* workspace, size_t workspace_bytes,
                                   void* stream) {
  return forward_bags_dev(ROUTE_GEN, false, p, Xs_dev, Ns_dev, nb, max_rows, classes, pred, A, B, crit_idx, nullptr,
                          nullptr, status, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

size_t dsmil_generic_backward_bags_dev_workspace_bytes(const dsmil_params_t* p, int32_t nb, int64_t max_rows) {
  return backward_bags_dev_ws(ROUTE_GEN, p, nb, max_rows);
}
int dsmil_generic_backward_bags_dev(const dsmil_params_t* p, const float* const* Xs_dev, const int64_t* Ns_dev,
                                    int32_t nb, int64_t max_rows, const float* Q, const float* H1, const float* A,
                                    const float* B, const int64_t* crit_idx, const float* d_classes,
                                    const float* d_pred, const float* d_A, const float* d_B, const dsmil_grads_t* grads,
                                    int32_t* status, void* workspace, size_t workspace_bytes, void* stream) {
  return backward_bags_dev(ROUTE_GEN, p, Xs_dev, Ns_dev, nb, max_rows, Q, H1, A, B, crit_idx, d_classes, d_pred, d_A,
                           d_B, grads, status, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

// ---- capture-safe fold step: M models, each over its own device bag list ------------------------------------------
// The grids and workspace regions a fold dev call sizes on the host, from (M, nbs, max_rows) alone.
struct ModelsDevCaps {
  int ne;                     // entries: the bags of all models
  int Gcap;                   // per-row CTAs per entry at most
  int nci, nc1, nc2, ncs;     // chunk capacities over all models
  int64_t max_model_rows;     // row capacity of the largest model
};
// gen: the generic fold calls (dsmil_generic_*_models_*), whose k_linear_b grid numbers twice the capacity tiles; why,
// when given, receives what was out of range.
static bool models_dev_caps(const dsmil_params_t* ps, int M, const int32_t* nbs, int64_t max_rows, ModelsDevCaps* c,
                            bool gen = false, const char** why = nullptr) {
  const char* dummy;
  if (!why) why = &dummy;
  *why = "shape";
  if (!ps || !nbs || !(gen ? dsmil_generic_models_supported(ps, M) : dsmil_models_supported(ps, M))) return false;
  const int C = ps[0].C, D = ps[0].D;
  int64_t ne = 0, nci = 0, nc1 = 0;
  *c = ModelsDevCaps{0, 1, 0, 0, M * kModelSplitsCap, M * kModelSplitsCap, 1};
  for (int m = 0; m < M; ++m) {
    *why = "a model's nb outside [1, 65535] or max_rows out of range";
    if (!dev_sizes(nbs[m], max_rows)) return false;
    ne += nbs[m];
    nci += rag_chunks_cap(C, D, tn_use_gemv(C, D), nbs[m]);
    nc1 += rag_chunks_cap(kQ, D, false, nbs[m]);
    c->Gcap = std::max(c->Gcap, bwd_bags_ctas(nbs[m], max_rows));
    c->max_model_rows = std::max<int64_t>(c->max_model_rows, nbs[m] * max_rows);
  }
  // every grid within its limits: entries and chunk capacities in 16 bits, the capacity tiles in an int
  *why = "chunk capacity: the bags of all models plus the ragged GEMMs' chunk allowance pass 65535";
  if (ne > 65535 || nci > 65535 || nc1 > 65535) return false;
  *why = "max_rows out of range: the capacity tiles pass INT_MAX";
  if ((gen ? 2 : 1) * ne * ((max_rows + sm90::kTileM - 1) / sm90::kTileM) > INT_MAX) return false;
  c->ne = static_cast<int>(ne);
  c->nci = static_cast<int>(nci);
  c->nc1 = static_cast<int>(nc1);
  return true;
}
static int check_models_dev(const dsmil_params_t* ps, int M, const float* const* Xs, const int64_t* Ns,
                            const int32_t* nbs, int64_t max_rows, const int32_t* status, ModelsDevCaps* caps) {
  int rc = check_models(ps, M);
  if (rc) return rc;
  DSMIL_REQUIRE(dsmil_models_supported(ps, M), "shape not supported by the fused fold step (D=%d, C=%d, nonlinear=%d, "
                "passing_v=%d, M=%d)", ps[0].D, ps[0].C, ps[0].nonlinear, ps[0].passing_v, M);
  DSMIL_REQUIRE(Xs && Ns && nbs && status, "NULL bag list or status");
  DSMIL_REQUIRE(models_dev_caps(ps, M, nbs, max_rows, caps),
                "a model's nb outside [1, 65535], too many bags in all, or max_rows=%lld out of range",
                (long long)max_rows);
  return 0;
}
// What the planner is told of the models (weights; with g, where their gradients go).
static PlanModelsArgs plan_models_args(const dsmil_params_t* ps, int M, const float* const* Xs, const int64_t* Ns,
                                       const int32_t* nbs, int64_t max_rows, int32_t* status,
                                       const dsmil_grads_t* g) {
  PlanModelsArgs a{};
  a.Xs = Xs; a.Ns = Ns; a.M = M; a.C = ps[0].C; a.D = ps[0].D; a.max_rows = max_rows; a.status = status;
  for (int m = 0, e0 = 0; m < M; e0 += nbs[m], ++m) {
    const dsmil_params_t& p = ps[m];
    a.m[m].w = sm90::ModelDev{p.Wi, p.bi, p.W1, p.b1, p.W2, p.b2, p.Wf, p.bf};
    if (g) {
      a.m[m].gWi = g[m].gWi; a.m[m].gbi = g[m].gbi; a.m[m].gW1 = g[m].gW1; a.m[m].gb1 = g[m].gb1;
      a.m[m].gW2 = g[m].gW2; a.m[m].gb2 = g[m].gb2; a.m[m].gWf = g[m].gWf; a.m[m].gbf = g[m].gbf;
    }
    a.m[m].e0 = e0;
    a.m[m].nb = nbs[m];
  }
  return a;
}

// The forward's carve for the capacity batch (every bag max_rows rows), then the planner's counts and the zero row.
// need_Q: the tile blocks of Q for the capacity tiles (inference); otherwise Q and H1 are the caller's saves.
static ModelsWs carve_models_dev(const dsmil_params_t* ps, int M, int ne, int64_t max_rows, bool need_Q, void* ws,
                                 size_t cap, bool* ok, ModelsPlan** plan, float** zero_row) {
  const std::vector<int64_t> Ns(ne, max_rows);
  ModelsWs w = carve_models(&ps[0], M, Ns.data(), ne, 1, need_Q, ws, cap, ok);
  Carver c(ws, cap);
  c.off = w.bytes;
  *plan = c.take<ModelsPlan>(1);
  *zero_row = c.take<float>(ps[0].D);
  w.bytes = c.off;
  *ok = c.ok();
  return w;
}

// The fold forward pair's size (train: dsmil_forward_bags_models_train_dev; inference: dsmil_forward_bags_models_dev,
// whose Q stays in the workspace as tile blocks): never below the eager fold call's size for the same capacity, nor
// the one-model dev calls' sizes together.
static size_t forward_bags_models_dev_ws(bool train, const dsmil_params_t* ps, int M, const int32_t* nbs,
                                         int64_t max_rows) {
  ModelsDevCaps caps;
  if (!models_dev_caps(ps, M, nbs, max_rows, &caps)) return 0;
  bool ok;
  ModelsPlan* plan;
  float* zero_row;
  size_t bytes = carve_models_dev(ps, M, caps.ne, max_rows, !train, nullptr, 0, &ok, &plan, &zero_row).bytes;
  const std::vector<int64_t> Ns(caps.ne, max_rows);
  bytes = std::max(bytes, dsmil_forward_bags_models_train_workspace_bytes(ps, M, Ns.data(), nbs));
  size_t each = 0;
  for (int m = 0; m < M; ++m)
    each += ws_slice(train ? dsmil_forward_bags_train_dev_workspace_bytes(&ps[m], nbs[m], max_rows)
                           : dsmil_forward_bags_dev_workspace_bytes(&ps[m], nbs[m], max_rows));
  return std::max(bytes, each);
}

// The fold forward pair's body.  train: as dsmil_forward_bags_train_dev, phase 1 writes the caller's row-major save_Q
// and save_H1 and the attend pass is a plain launch.  Inference: as dsmil_forward_bags_dev, Q stays in the workspace
// as tile blocks, and the attend pass is a programmatic dependent of phase 1 (also under stream capture), each entry
// gated on its tiles' releases in w.done (DESIGN §4.2k); only kernel timing keeps the plain launch.  Either way the
// weight images are rebuilt on every call and the grids are the capacity's, their live counts the planner's.
static int forward_bags_models_dev(bool train, const dsmil_params_t* ps, int M, const float* const* Xs_dev,
                                   const int64_t* Ns_dev, const int32_t* nbs, int64_t max_rows, float* classes,
                                   float* pred, float* A, float* B, int64_t* crit_idx, float* save_Q, float* save_H1,
                                   int32_t* status, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  ModelsDevCaps caps;
  int rc = check_models_dev(ps, M, Xs_dev, Ns_dev, nbs, max_rows, status, &caps);
  if (rc) return rc;
  DSMIL_REQUIRE(classes && pred && A && B && (!train || (crit_idx && save_Q && save_H1)), "NULL output pointer");
  const size_t need = forward_bags_models_dev_ws(train, ps, M, nbs, max_rows);
  if ((rc = need_workspace(need, workspace, workspace_bytes))) return rc;
  const int C = ps[0].C, D = ps[0].D, ne = caps.ne;
  bool ok;
  ModelsPlan* plan;
  float* zero_row;
  ModelsWs w = carve_models_dev(ps, M, ne, max_rows, !train, workspace, workspace_bytes, &ok, &plan, &zero_row);
  PlanModelsArgs pa = plan_models_args(ps, M, Xs_dev, Ns_dev, nbs, max_rows, status, nullptr);
  pa.zero_row = zero_row;
  pa.plan = plan;
  pa.ftable = w.table;
  pa.fmodels = w.models;
  k_plan_bags_models<<<1, 32 * M, 0, st>>>(pa);
  DSMIL_LAUNCH_OK("k_plan_bags_models");
  const bool overlap = !train && !g_prof_on;
  float* Q = train ? save_Q : w.Q;
  const int tiles = ne * tiles_for_bag(max_rows);
  DSMIL_CUDA_OK(cudaMemsetAsync(w.keys, 0, sizeof(unsigned long long) * (kMaxC + 1) * ne, st));
  if ((rc = sm90::launch_prep_wimg_models(w.models, M, D, w.wimg, st))) return rc;
  if ((rc = sm90::launch_qmlp_models(w.models, M, D, C, w.table, ne, tiles, classes, w.keys, Q,
                                     train ? save_H1 : nullptr, !train, w.wimg,
                                     overlap ? overlap_phase1_ctas(tiles) : num_sms(), st,
                                     overlap ? w.done : nullptr, &plan->tiles)))
    return rc;
  sm90::AttendArgs aa{w.table, ne, D, C, Q, !train, w.keys, A, w.recs, nullptr, &plan->recs,
                      overlap ? w.done : nullptr};
  if ((rc = sm90::launch_attend_b(aa, ne * recs_for_bag(max_rows), st))) return rc;
  sm90::FinalizeArgs fa{w.table, D, C, w.recs, w.keys, nullptr, nullptr, A, B, pred,
                        reinterpret_cast<long long*>(crit_idx), w.pred_part, w.counters, nullptr, 0, 0, w.models, 1, 0};
  return sm90::launch_finalize_b(fa, ne, st);
}

size_t dsmil_forward_bags_models_train_dev_workspace_bytes(const dsmil_params_t* ps, int32_t M, const int32_t* nbs,
                                                           int64_t max_rows) {
  return forward_bags_models_dev_ws(true, ps, M, nbs, max_rows);
}

int dsmil_forward_bags_models_train_dev(const dsmil_params_t* ps, int32_t M, const float* const* Xs_dev,
                                        const int64_t* Ns_dev, const int32_t* nbs, int64_t max_rows, float* classes,
                                        float* pred, float* A, float* B, int64_t* crit_idx, float* save_Q,
                                        float* save_H1, int32_t* status, void* workspace, size_t workspace_bytes,
                                        void* stream) {
  return forward_bags_models_dev(true, ps, M, Xs_dev, Ns_dev, nbs, max_rows, classes, pred, A, B, crit_idx, save_Q,
                                 save_H1, status, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

size_t dsmil_forward_bags_models_dev_workspace_bytes(const dsmil_params_t* ps, int32_t M, const int32_t* nbs,
                                                     int64_t max_rows) {
  return forward_bags_models_dev_ws(false, ps, M, nbs, max_rows);
}

int dsmil_forward_bags_models_dev(const dsmil_params_t* ps, int32_t M, const float* const* Xs_dev,
                                  const int64_t* Ns_dev, const int32_t* nbs, int64_t max_rows, float* classes,
                                  float* pred, float* A, float* B, int64_t* crit_idx, int32_t* status, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  return forward_bags_models_dev(false, ps, M, Xs_dev, Ns_dev, nbs, max_rows, classes, pred, A, B, crit_idx, nullptr,
                                 nullptr, status, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

// The backward's carve at the capacities, then the planner's counts and the zero row.
static BwdModelsWs carve_bwd_models_dev(const dsmil_params_t* ps, int M, const ModelsDevCaps& caps, int64_t max_rows,
                                        void* ws, size_t cap, bool* ok, ModelsPlan** plan, float** zero_row) {
  BwdModelsPlan pl;
  pl.table.resize(caps.ne);
  pl.chi.resize(caps.nci);
  pl.ch1.resize(caps.nc1);
  pl.ch2.resize(caps.nc2);
  pl.chc.resize(caps.ncs);
  pl.slots = caps.ne * caps.Gcap;
  BwdModelsWs w = carve_bwd_models(ps, M, pl, caps.ne * max_rows, ws, cap, ok);
  Carver c(ws, cap);
  c.off = w.bytes;
  *plan = c.take<ModelsPlan>(1);
  *zero_row = c.take<float>(ps[0].D);
  w.bytes = c.off;
  *ok = c.ok();
  return w;
}

static int check_generic_models_dev(const dsmil_params_t* ps, int M, const float* const* Xs, const int64_t* Ns,
                                    const int32_t* nbs, int64_t max_rows, const int32_t* status, ModelsDevCaps* caps);

// The backward pair's size and body, for the fused tensor-core fold shapes or (gen) the generic ones.
static size_t backward_bags_models_dev_ws(bool gen, const dsmil_params_t* ps, int M, const int32_t* nbs,
                                          int64_t max_rows) {
  ModelsDevCaps caps;
  if (!models_dev_caps(ps, M, nbs, max_rows, &caps, gen)) return 0;
  bool ok;
  ModelsPlan* plan;
  float* zero_row;
  size_t bytes = carve_bwd_models_dev(ps, M, caps, max_rows, nullptr, 0, &ok, &plan, &zero_row).bytes;
  const std::vector<int64_t> Ns(caps.ne, max_rows);
  bytes = std::max(bytes, dsmil_backward_bags_models_workspace_bytes(ps, M, Ns.data(), nbs, 0));
  size_t each = 0;
  for (int m = 0; m < M; ++m)
    each += ws_slice(gen ? dsmil_generic_backward_bags_dev_workspace_bytes(&ps[m], nbs[m], max_rows)
                         : dsmil_backward_bags_dev_workspace_bytes(&ps[m], nbs[m], max_rows));
  return std::max(bytes, each);
}

static int backward_bags_models_dev(bool gen, const dsmil_params_t* ps, int M, const float* const* Xs_dev,
                                    const int64_t* Ns_dev, const int32_t* nbs, int64_t max_rows, const float* Q,
                                    const float* H1, const float* A, const float* B, const int64_t* crit_idx,
                                    const float* d_classes, const float* d_pred, const float* d_A, const float* d_B,
                                    const dsmil_grads_t* grads, int32_t* status, void* workspace,
                                    size_t workspace_bytes, cudaStream_t st) {
  ModelsDevCaps caps;
  int rc = gen ? check_generic_models_dev(ps, M, Xs_dev, Ns_dev, nbs, max_rows, status, &caps)
               : check_models_dev(ps, M, Xs_dev, Ns_dev, nbs, max_rows, status, &caps);
  if (rc) return rc;
  DSMIL_REQUIRE(Q && (H1 || !ps[0].nonlinear) && A && B && crit_idx && grads, "NULL pointer");
  bool gX = false;
  for (int m = 0; m < M; ++m) gX = gX || grads[m].gX != nullptr;
  DSMIL_REQUIRE(!d_A && !d_B && !gX,
                "the dev backward takes gradients through classes and pred only (no d_A, d_B or gX)");
  const size_t need = backward_bags_models_dev_ws(gen, ps, M, nbs, max_rows);
  if ((rc = need_workspace(need, workspace, workspace_bytes))) return rc;
  const int C = ps[0].C, D = ps[0].D;
  bool ok;
  ModelsPlan* plan;
  float* zero_row;
  BwdModelsWs w = carve_bwd_models_dev(ps, M, caps, max_rows, workspace, workspace_bytes, &ok, &plan, &zero_row);
  PlanModelsArgs pa = plan_models_args(ps, M, Xs_dev, Ns_dev, nbs, max_rows, status, grads);
  pa.Gcap = caps.Gcap;
  pa.zero_row = zero_row;
  pa.plan = plan;
  pa.btable = w.table;
  pa.bmodels = w.models;
  pa.chi = w.chi; pa.ch1 = w.ch1; pa.ch2 = w.ch2; pa.chc = w.chc;
  pa.ncs_cap = caps.ncs;
  pa.segs = w.segs;
  pa.lin = w.lin;
  pa.H1 = H1;
  pa.dz2 = w.dz2;
  pa.dz1 = w.dz1;
  pa.dc = d_classes != nullptr;
  pa.gen = gen ? FOLD_GEN : FOLD_TC;
  k_plan_bags_models<<<1, 32 * M, 0, st>>>(pa);
  DSMIL_LAUNCH_OK("k_plan_bags_models");
  if (!d_classes)   // no gradient through the scores: zero instance-classifier gradients, as the eager call
    for (int m = 0; m < M; ++m) {
      if (grads[m].gWi) DSMIL_CUDA_OK(cudaMemsetAsync(grads[m].gWi, 0, sizeof(float) * C * D, st));
      if (grads[m].gbi) DSMIL_CUDA_OK(cudaMemsetAsync(grads[m].gbi, 0, sizeof(float) * C, st));
    }
  BwdModelsGrid gr{caps.Gcap, caps.nci, caps.nc1, caps.nc2, caps.ncs, caps.max_model_rows, false, plan,
                   !ps[0].nonlinear};
  return bwd_models_launch(C, D, M, caps.ne, w, gr, Q, H1, A, B, crit_idx, d_classes, d_pred, nullptr, nullptr, st);
}

size_t dsmil_backward_bags_models_dev_workspace_bytes(const dsmil_params_t* ps, int32_t M, const int32_t* nbs,
                                                      int64_t max_rows) {
  return backward_bags_models_dev_ws(false, ps, M, nbs, max_rows);
}

int dsmil_backward_bags_models_dev(const dsmil_params_t* ps, int32_t M, const float* const* Xs_dev,
                                   const int64_t* Ns_dev, const int32_t* nbs, int64_t max_rows, const float* Q,
                                   const float* H1, const float* A, const float* B, const int64_t* crit_idx,
                                   const float* d_classes, const float* d_pred, const float* d_A, const float* d_B,
                                   const dsmil_grads_t* grads, int32_t* status, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  return backward_bags_models_dev(false, ps, M, Xs_dev, Ns_dev, nbs, max_rows, Q, H1, A, B, crit_idx, d_classes,
                                  d_pred, d_A, d_B, grads, status, workspace, workspace_bytes,
                                  static_cast<cudaStream_t>(stream));
}

// ---- capture-safe fold step on the generic shapes ------------------------------------------------------------------
// The fold twins of dsmil_generic_forward_bags_train_dev / dsmil_generic_backward_bags_dev: one planner launch
// (k_plan_bags_models with the generic numbering) for all models, then the generic forward over the table of every
// model's bags (gen_forward_run's fold form) or the fused fold backward (bwd_models_launch, linear q included).
int dsmil_generic_models_supported(const dsmil_params_t* ps, int32_t M) {
  if (!ps || M < 1 || M > sm90::kMaxModels || check_models(ps, M) != 0) return 0;
  for (int m = 0; m < M; ++m)
    if (!dsmil_generic_bags_supported(&ps[m])) return 0;
  return 1;
}

static int check_generic_models_dev(const dsmil_params_t* ps, int M, const float* const* Xs, const int64_t* Ns,
                                    const int32_t* nbs, int64_t max_rows, const int32_t* status,
                                    ModelsDevCaps* caps) {
  int rc = check_models(ps, M);
  if (rc) return rc;
  DSMIL_REQUIRE(!ps[0].passing_v, "the generic fold calls take identity v only (passing_v=1)");
  DSMIL_REQUIRE(dsmil_generic_models_supported(ps, M),
                "shape not on the generic batched route, i.e. on the tensor-core fold calls' (D=%d, C=%d, "
                "nonlinear=%d, M=%d)", ps[0].D, ps[0].C, ps[0].nonlinear, M);
  DSMIL_REQUIRE(Xs && Ns && nbs && status, "NULL bag list or status");
  const char* why;
  DSMIL_REQUIRE(models_dev_caps(ps, M, nbs, max_rows, caps, true, &why), "%s (max_rows=%lld)", why,
                (long long)max_rows);
  return 0;
}

// The forward's carve: the generic forward's for the capacity batch of every model's bags (every bag max_rows rows),
// then the members, the planner's counts over all models and each model's own.  saves: the caller keeps Q and H1
// (the training form); inference keeps them, and the critical rows if the caller wants none, in the workspace.
struct GenModelsWs {
  GenWs g;
  sm90::ModelDev* models;
  ModelsPlan* plan;
  FoldLive* live;
  size_t bytes;
};
static GenModelsWs carve_gen_models_dev(const dsmil_params_t* ps, int M, int ne, int64_t max_rows, bool saves,
                                        void* ws, size_t cap, bool* ok) {
  GenModelsWs w;
  w.g = carve_gen_dev(&ps[0], ne, max_rows, saves, ws, cap, ok);
  Carver c(ws, cap);
  c.off = w.g.bytes;
  w.models = c.take<sm90::ModelDev>(M);
  w.plan = c.take<ModelsPlan>(1);
  w.live = c.take<FoldLive>(M);
  w.bytes = c.off;
  *ok = *ok && c.ok();
  return w;
}

// The generic fold forward pair's size (train: the _train_dev call; inference: Q, H1 and the critical rows in the
// workspace), never below the eager fold call's size for the same capacity, nor the one-model generic dev calls'
// sizes together.
static size_t generic_forward_bags_models_dev_ws(bool train, const dsmil_params_t* ps, int M, const int32_t* nbs,
                                                 int64_t max_rows) {
  ModelsDevCaps caps;
  if (!models_dev_caps(ps, M, nbs, max_rows, &caps, true)) return 0;
  bool ok;
  size_t bytes = carve_gen_models_dev(ps, M, caps.ne, max_rows, train, nullptr, 0, &ok).bytes;
  const std::vector<int64_t> Ns(caps.ne, max_rows);
  bytes = std::max(bytes, dsmil_forward_bags_models_train_workspace_bytes(ps, M, Ns.data(), nbs));
  size_t each = 0;
  for (int m = 0; m < M; ++m)
    each += ws_slice(train ? dsmil_generic_forward_bags_train_dev_workspace_bytes(&ps[m], nbs[m], max_rows)
                           : dsmil_generic_forward_bags_dev_workspace_bytes(&ps[m], nbs[m], max_rows));
  return std::max(bytes, each);
}

// The generic fold forward pair's body: one planner launch, then gen_forward_run's fold form.  Inference differs
// from training only in where Q, H1 and the critical rows go (the generic forward has no phase-1 overlap).
static int generic_forward_bags_models_dev(bool train, const dsmil_params_t* ps, int M, const float* const* Xs_dev,
                                           const int64_t* Ns_dev, const int32_t* nbs, int64_t max_rows,
                                           float* classes, float* pred, float* A, float* B, int64_t* crit_idx,
                                           float* save_Q, float* save_H1, int32_t* status, void* workspace,
                                           size_t workspace_bytes, cudaStream_t st) {
  ModelsDevCaps caps;
  int rc = check_generic_models_dev(ps, M, Xs_dev, Ns_dev, nbs, max_rows, status, &caps);
  if (rc) return rc;
  DSMIL_REQUIRE(classes && pred && A && B && (!train || (crit_idx && save_Q && (save_H1 || !ps[0].nonlinear))),
                "NULL output pointer");
  const size_t need = generic_forward_bags_models_dev_ws(train, ps, M, nbs, max_rows);
  if ((rc = need_workspace(need, workspace, workspace_bytes))) return rc;
  const int ne = caps.ne;
  bool ok;
  GenModelsWs w = carve_gen_models_dev(ps, M, ne, max_rows, train, workspace, workspace_bytes, &ok);
  PlanModelsArgs pa = plan_models_args(ps, M, Xs_dev, Ns_dev, nbs, max_rows, status, nullptr);
  pa.zero_row = w.g.zero_row;
  pa.plan = w.plan;
  pa.ftable = w.g.table;
  pa.fmodels = w.models;
  pa.gen = sm90::qmlp_supported(&ps[0]) ? FOLD_GEN_QMLP : FOLD_GEN;
  pa.live = w.live;
  k_plan_bags_models<<<1, 32 * M, 0, st>>>(pa);
  DSMIL_LAUNCH_OK("k_plan_bags_models");
  const GenFolds f{ps, nbs, M, max_rows, w.models, w.plan, w.live};
  float* H1 = ps[0].nonlinear ? (train ? save_H1 : w.g.H1) : nullptr;
  return gen_forward_run(&ps[0], w.g, ne, ne * max_rows, ne * tiles_for_bag(max_rows), ne * attend_ctas(max_rows),
                         max_rows, classes, pred, A, B, crit_idx ? crit_idx : w.g.crit, train ? save_Q : w.g.Q, H1,
                         nullptr, st, &f);
}

size_t dsmil_generic_forward_bags_models_train_dev_workspace_bytes(const dsmil_params_t* ps, int32_t M,
                                                                   const int32_t* nbs, int64_t max_rows) {
  return generic_forward_bags_models_dev_ws(true, ps, M, nbs, max_rows);
}

int dsmil_generic_forward_bags_models_train_dev(const dsmil_params_t* ps, int32_t M, const float* const* Xs_dev,
                                                const int64_t* Ns_dev, const int32_t* nbs, int64_t max_rows,
                                                float* classes, float* pred, float* A, float* B, int64_t* crit_idx,
                                                float* save_Q, float* save_H1, int32_t* status, void* workspace,
                                                size_t workspace_bytes, void* stream) {
  return generic_forward_bags_models_dev(true, ps, M, Xs_dev, Ns_dev, nbs, max_rows, classes, pred, A, B, crit_idx,
                                         save_Q, save_H1, status, workspace, workspace_bytes,
                                         static_cast<cudaStream_t>(stream));
}

size_t dsmil_generic_forward_bags_models_dev_workspace_bytes(const dsmil_params_t* ps, int32_t M, const int32_t* nbs,
                                                             int64_t max_rows) {
  return generic_forward_bags_models_dev_ws(false, ps, M, nbs, max_rows);
}

int dsmil_generic_forward_bags_models_dev(const dsmil_params_t* ps, int32_t M, const float* const* Xs_dev,
                                          const int64_t* Ns_dev, const int32_t* nbs, int64_t max_rows, float* classes,
                                          float* pred, float* A, float* B, int64_t* crit_idx, int32_t* status,
                                          void* workspace, size_t workspace_bytes, void* stream) {
  return generic_forward_bags_models_dev(false, ps, M, Xs_dev, Ns_dev, nbs, max_rows, classes, pred, A, B, crit_idx,
                                         nullptr, nullptr, status, workspace, workspace_bytes,
                                         static_cast<cudaStream_t>(stream));
}

size_t dsmil_generic_backward_bags_models_dev_workspace_bytes(const dsmil_params_t* ps, int32_t M, const int32_t* nbs,
                                                              int64_t max_rows) {
  return backward_bags_models_dev_ws(true, ps, M, nbs, max_rows);
}

int dsmil_generic_backward_bags_models_dev(const dsmil_params_t* ps, int32_t M, const float* const* Xs_dev,
                                           const int64_t* Ns_dev, const int32_t* nbs, int64_t max_rows,
                                           const float* Q, const float* H1, const float* A, const float* B,
                                           const int64_t* crit_idx, const float* d_classes, const float* d_pred,
                                           const float* d_A, const float* d_B, const dsmil_grads_t* grads,
                                           int32_t* status, void* workspace, size_t workspace_bytes, void* stream) {
  return backward_bags_models_dev(true, ps, M, Xs_dev, Ns_dev, nbs, max_rows, Q, H1, A, B, crit_idx, d_classes,
                                  d_pred, d_A, d_B, grads, status, workspace, workspace_bytes,
                                  static_cast<cudaStream_t>(stream));
}

// ---- capture-safe row-sharded batch training: the six calls of the sharded step in dev form -----------------------
// As the dev pair above: the bag list (and the row offsets) in device memory, launches on capacity grids whose live
// counts the planner writes, no host<->device traffic.  Forward phases 2 and 3 read phase 1's table and counts from the
// forward workspace, backward phases 2 and 3 read backward phase 1's from the backward workspace.
size_t dsmil_shard_bags_train_dev_workspace_bytes(const dsmil_params_t* p, int32_t nb, int64_t max_rows) {
  if (!dev_shape(ROUTE_TC, p) || !dev_sizes(nb, max_rows)) return 0;
  bool ok;
  BagsPlan* plan;
  float* zero_row;
  const size_t dev = carve_bags_dev(p, nb, max_rows, false, true, nullptr, 0, &ok, &plan, &zero_row).bytes;
  return not_below_eager(dev, dsmil_shard_bags_workspace_bytes, p, nb, max_rows);
}

// The forward workspace of a sharded dev call, after its checks.
static int shard_bags_dev_ws(const dsmil_params_t* p, int nb, int64_t max_rows, void* workspace,
                             size_t workspace_bytes, BagsWs* w, BagsPlan** plan, float** zero_row) {
  const size_t need = dsmil_shard_bags_train_dev_workspace_bytes(p, nb, max_rows);
  int rc = need_workspace(need, workspace, workspace_bytes);
  if (rc) return rc;
  bool ok;
  *w = carve_bags_dev(p, nb, max_rows, false, true, workspace, workspace_bytes, &ok, plan, zero_row);
  return 0;
}

int dsmil_shard_bags_phase1_train_dev(const dsmil_params_t* p, const float* const* Xs_dev, const int64_t* Ns_dev,
                                      const int64_t* row_offsets_dev, int32_t nb, int64_t max_rows, float* classes,
                                      float* save_Q, float* save_H1, float* cand_recs, int32_t* status,
                                      void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_bags_dev(ROUTE_TC, p, true, true, Xs_dev, Ns_dev, nb, max_rows, status);
  if (rc) return rc;
  DSMIL_REQUIRE(row_offsets_dev && classes && save_Q && save_H1 && cand_recs, "NULL pointer");
  BagsWs w;
  BagsPlan* plan;
  float* zero_row;
  if ((rc = shard_bags_dev_ws(p, nb, max_rows, workspace, workspace_bytes, &w, &plan, &zero_row))) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  k_plan_bags<<<1, 32, 0, st>>>(Xs_dev, Ns_dev, nb, max_rows, p->C, p->D, zero_row, w.table, nullptr, nullptr, plan,
                                status, row_offsets_dev, w.row_offsets);
  DSMIL_LAUNCH_OK("k_plan_bags");
  if ((rc = bags_phase1_dev(p, w, plan, nb, max_rows, classes, save_Q, save_H1, st))) return rc;
  sm90::k_gather_cand_b<<<dim3(p->C, nb), kQ, 0, st>>>(w.table, w.keys, classes, save_Q, false, w.row_offsets, p->C,
                                                        cand_recs);
  DSMIL_LAUNCH_OK("k_gather_cand_b");
  return 0;
}

int dsmil_shard_bags_phase2_train_dev(const dsmil_params_t* p, int32_t nb, int64_t max_rows, const float* Q,
                                      const float* cands_all, int32_t G, float* A, int64_t* crit_idx, float* q_max,
                                      float* recs_out, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_bags_dev(ROUTE_TC, p, true, false, nullptr, nullptr, nb, max_rows, nullptr);
  if (rc) return rc;
  DSMIL_REQUIRE(Q && cands_all && G >= 1 && A && crit_idx && q_max && recs_out, "NULL pointer or G < 1");
  BagsWs w;
  BagsPlan* plan;
  float* zero_row;
  if ((rc = shard_bags_dev_ws(p, nb, max_rows, workspace, workspace_bytes, &w, &plan, &zero_row))) return rc;
  return shard_bags_phase2_impl(p, nb, Q, false, cands_all, G, A, crit_idx, q_max, recs_out, w,
                                nb * recs_for_bag(max_rows), &plan->recs, static_cast<cudaStream_t>(stream));
}

int dsmil_shard_bags_phase3_dev(const dsmil_params_t* p, int32_t nb, int64_t max_rows, const float* recs_all,
                                int32_t G, float* A, float* B, float* pred, void* workspace, size_t workspace_bytes,
                                void* stream) {
  int rc = check_bags_dev(ROUTE_TC, p, true, false, nullptr, nullptr, nb, max_rows, nullptr);
  if (rc) return rc;
  DSMIL_REQUIRE(recs_all && G >= 1 && G <= sm90::kMaxRecPerBag && A && B && pred, "NULL pointer or G out of range");
  BagsWs w;
  BagsPlan* plan;
  float* zero_row;
  if ((rc = shard_bags_dev_ws(p, nb, max_rows, workspace, workspace_bytes, &w, &plan, &zero_row))) return rc;
  sm90::FinalizeArgs fa{w.table, p->D, p->C, recs_all, w.keys, p->Wf, p->bf, A, B, pred, nullptr,
                         w.pred_part, w.counters, nullptr, G, nb};
  return sm90::launch_finalize_b(fa, nb, static_cast<cudaStream_t>(stream));
}

size_t dsmil_shard_backward_bags_dev_workspace_bytes(const dsmil_params_t* p, int32_t nb, int64_t max_rows) {
  if (!dev_shape(ROUTE_TC, p) || !dev_sizes(nb, max_rows) || !dev_chunks_ok(ROUTE_TC, p, nb)) return 0;
  bool ok;
  const size_t dev = carve_bwd_bags_dev(p, nb, max_rows, nullptr, 0, &ok).bytes;
  return not_below_eager(dev, dsmil_shard_backward_bags_workspace_bytes, p, nb, max_rows);
}

// The backward workspace of a sharded dev call, after its checks.  Phases 1 and 3 run backward_bags_dev's ragged
// GEMMs on the same capacities, and phase 2 reads the same workspace, so all three refuse its chunk capacity first.
static int shard_bwd_bags_dev_ws(const dsmil_params_t* p, int nb, int64_t max_rows, void* workspace,
                                 size_t workspace_bytes, BwdBagsWs* w) {
  DSMIL_REQUIRE(dev_chunks_ok(ROUTE_TC, p, nb), "nb=%d: the chunk capacity of the ragged GEMMs passes 65535", nb);
  const size_t need = dsmil_shard_backward_bags_dev_workspace_bytes(p, nb, max_rows);
  int rc = need_workspace(need, workspace, workspace_bytes);
  if (rc) return rc;
  bool ok;
  *w = carve_bwd_bags_dev(p, nb, max_rows, workspace, workspace_bytes, &ok);
  return 0;
}

int dsmil_shard_backward_bags_phase1_dev(const dsmil_params_t* p, const float* const* Xs_dev, const int64_t* Ns_dev,
                                         int32_t nb, int64_t max_rows, const float* A, const float* B,
                                         const float* d_classes_local, const float* d_pred, float* dA_local,
                                         float* t_local, float* gWi, float* gbi, float* gWf, float* gbf,
                                         int32_t* status, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_bags_dev(ROUTE_TC, p, false, true, Xs_dev, Ns_dev, nb, max_rows, status);
  if (rc) return rc;
  DSMIL_REQUIRE(A && B && dA_local && t_local, "NULL tensor pointer");
  BwdBagsWs w;
  if ((rc = shard_bwd_bags_dev_ws(p, nb, max_rows, workspace, workspace_bytes, &w))) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  k_plan_bags<<<1, 32, 0, st>>>(Xs_dev, Ns_dev, nb, max_rows, p->C, p->D, w.zero_row, w.table, w.chi, w.ch1, w.plan,
                                status, nullptr, nullptr);
  DSMIL_LAUNCH_OK("k_plan_bags");
  dsmil_grads_t g{};
  g.gWi = gWi; g.gbi = gbi; g.gWf = gWf; g.gbf = gbf;
  if ((rc = bwd_bags_phase1_impl(p, nullptr, nullptr, nb, static_cast<int64_t>(nb) * max_rows, A, B, d_classes_local,
                                 d_pred, nullptr, nullptr, &g, dA_local, w, st)))
    return rc;
  // t_local[b]: the live partials summed in the eager call's order
  k_sum_segments<<<dim3(ceil_div(p->C, 256), nb), 256, 0, st>>>(w.tpart, w.G, p->C, t_local, &w.plan->G);
  DSMIL_LAUNCH_OK("k_sum_segments");
  return 0;
}

int dsmil_shard_backward_bags_phase2_dev(const dsmil_params_t* p, int32_t nb, int64_t max_rows, const float* A,
                                         float* dA_to_dL, const float* t_global, const float* Q, float* dqm_local,
                                         void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_bags_dev(ROUTE_TC, p, false, false, nullptr, nullptr, nb, max_rows, nullptr);
  if (rc) return rc;
  DSMIL_REQUIRE(A && dA_to_dL && t_global && Q && dqm_local, "NULL tensor pointer");
  BwdBagsWs w;
  if ((rc = shard_bwd_bags_dev_ws(p, nb, max_rows, workspace, workspace_bytes, &w))) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // the copy that lets dL replace dA (as the eager call), over the capacity rows: the live total is on the device
  DSMIL_CUDA_OK(cudaMemcpyAsync(w.dA, dA_to_dL, sizeof(float) * nb * max_rows * p->C, cudaMemcpyDeviceToDevice, st));
  return bwd_bags_phase2_impl(p, nb, A, w.dA, t_global, 1, Q, dA_to_dL, dqm_local, w, st);
}

int dsmil_shard_backward_bags_phase3_dev(const dsmil_params_t* p, int32_t nb, int64_t max_rows,
                                         const int64_t* row_offsets_dev, const float* Q, const float* H1,
                                         const float* dL_local, const float* dqm_global, const float* q_max,
                                         const int64_t* crit_idx, float* gW1, float* gb1, float* gW2, float* gb2,
                                         void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_bags_dev(ROUTE_TC, p, false, false, nullptr, nullptr, nb, max_rows, nullptr);
  if (rc) return rc;
  DSMIL_REQUIRE(row_offsets_dev && Q && H1 && dL_local && dqm_global && q_max && crit_idx, "NULL tensor pointer");
  BwdBagsWs w;
  if ((rc = shard_bwd_bags_dev_ws(p, nb, max_rows, workspace, workspace_bytes, &w))) return rc;
  dsmil_grads_t g{};
  g.gW1 = gW1; g.gb1 = gb1; g.gW2 = gW2; g.gb2 = gb2;
  const float* dz1;
  return bwd_bags_phase3_impl(p, nb, static_cast<int64_t>(nb) * max_rows, Q, H1, dL_local, dqm_global, q_max, crit_idx,
                              reinterpret_cast<const long long*>(row_offsets_dev), &g, w, &dz1,
                              static_cast<cudaStream_t>(stream));
}

int dsmil_value_bags_supported(const dsmil_params_t* p) {
  return value_shape(p) && p->Wv && p->bv ? 1 : 0;
}

size_t dsmil_value_forward_bags_workspace_bytes(const dsmil_params_t* p, const int64_t* Ns, int32_t nb) {
  if (!dsmil_value_bags_supported(p) || !Ns || nb < 1 || nb > 65535) return 0;
  for (int b = 0; b < nb; ++b)
    if (Ns[b] < 1 || Ns[b] >= 0xffffffffll) return 0;
  return routes_ws_bytes(p, Ns, nb, bags_routes(p, nb));
}

int dsmil_value_forward_bags(const dsmil_params_t* p, const float* const* Xs, const float* const* XVs,
                             const int64_t* Ns, int32_t nb, float* classes, float* pred, float* A, float* B,
                             int64_t* crit_idx, float* save_Q, float* save_H1, float* save_V, void* workspace,
                             size_t workspace_bytes, void* stream) {
  int rc = check_params(p, true);
  if (rc) return rc;
  DSMIL_REQUIRE(p->passing_v, "the value route takes passing_v models (identity v: dsmil_forward_bags)");
  DSMIL_REQUIRE(Xs && Ns && nb >= 1 && nb <= 65535 && classes && pred && A && B,
                "NULL pointer or nb outside [1, 65535]");
  const bool saves = save_Q || save_H1 || save_V;
  DSMIL_REQUIRE(!saves || (save_Q && save_V && (!p->nonlinear || save_H1)),
                "saves: save_Q, save_V (and save_H1 for a nonlinear q) together, or none");
  int64_t total;
  bool aligned;
  if ((rc = check_bags(Xs, Ns, nb, &total, &aligned))) return rc;
  for (int b = 0; XVs && b < nb; ++b) DSMIL_REQUIRE(XVs[b], "bag %d: NULL value input", b);
  if ((rc = need_workspace(dsmil_value_forward_bags_workspace_bytes(p, Ns, nb), workspace, workspace_bytes))) return rc;
  return forward_bags_route(p, Xs, XVs, Ns, nb, aligned, classes, pred, A, B, crit_idx, save_Q, save_H1, save_V,
                            workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

size_t dsmil_value_backward_bags_workspace_bytes(const dsmil_params_t* p, const int64_t* Ns, int32_t nb, int need_gX) {
  if (!dsmil_value_bags_supported(p) || !Ns || nb < 1 || nb > 65535) return 0;
  for (int b = 0; b < nb; ++b)
    if (Ns[b] < 1 || Ns[b] >= 0xffffffffll) return 0;
  bool ok;
  const ValueBwdWs w = carve_value_bwd(p, Ns, nb, true, need_gX != 0, nullptr, 0, &ok);
  return value_bwd_grids_ok(w) ? w.bytes : 0;
}

int dsmil_value_backward_bags(const dsmil_params_t* p, const float* const* Xs, const float* const* XVs,
                              const int64_t* Ns, int32_t nb, const float* Q, const float* H1, const float* V,
                              const float* A, const float* B, const int64_t* crit_idx, const float* d_classes,
                              const float* d_pred, const float* d_A, const float* d_B, const float* v_mask,
                              const dsmil_grads_t* grads, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_params(p);
  if (rc) return rc;
  DSMIL_REQUIRE(p->passing_v, "the value backward takes passing_v models (identity v: dsmil_backward_bags)");
  DSMIL_REQUIRE(Xs && Ns && nb >= 1 && nb <= 65535 && Q && V && A && B && crit_idx && grads,
                "NULL pointer or nb outside [1, 65535]");
  DSMIL_REQUIRE(!p->nonlinear || H1, "nonlinear q backward needs saved H1");
  DSMIL_REQUIRE(!(grads->gX && d_classes) || p->Wi, "gX through d_classes needs Wi");
  int64_t total;
  bool aligned;
  if ((rc = check_bags(Xs, Ns, nb, &total, &aligned))) return rc;
  for (int b = 0; XVs && b < nb; ++b) DSMIL_REQUIRE(XVs[b], "bag %d: NULL value input", b);
  bool ok;
  const ValueBwdWs w = carve_value_bwd(p, Ns, nb, aligned, grads->gX != nullptr, workspace, workspace_bytes, &ok);
  DSMIL_REQUIRE(value_bwd_grids_ok(w), "too many bags for the ragged GEMM grids (%d gW1 chunks, %d gWv chunks)",
                w.b.nc1, w.ncv);
  const size_t need = dsmil_value_backward_bags_workspace_bytes(p, Ns, nb, grads->gX != nullptr);
  if ((rc = need_workspace(need, workspace, workspace_bytes))) return rc;
  return value_backward_bags_impl(p, Xs, XVs, Ns, nb, total, Q, H1, V, A, B, crit_idx, d_classes, d_pred, d_A, d_B,
                                  v_mask, grads, w, static_cast<cudaStream_t>(stream));
}

size_t dsmil_value_forward_bags_dev_workspace_bytes(const dsmil_params_t* p, int32_t nb, int64_t max_rows) {
  return forward_bags_dev_ws(ROUTE_VAL, false, p, nb, max_rows);
}
int dsmil_value_forward_bags_dev(const dsmil_params_t* p, const float* const* Xs_dev, const float* const* XVs_dev,
                                 const int64_t* Ns_dev, int32_t nb, int64_t max_rows, float* classes, float* pred,
                                 float* A, float* B, int64_t* crit_idx, float* save_Q, float* save_H1, float* save_V,
                                 int32_t* status, void* workspace, size_t workspace_bytes, void* stream) {
  const bool saves = save_Q || save_H1 || save_V;
  DSMIL_REQUIRE(!saves || (save_Q && save_V && (!p || !p->nonlinear || save_H1)),
                "saves: save_Q, save_V (and save_H1 for a nonlinear q) together, or none");
  return forward_bags_dev(ROUTE_VAL, saves, p, Xs_dev, Ns_dev, nb, max_rows, classes, pred, A, B, crit_idx, save_Q,
                          save_H1, status, workspace, workspace_bytes, static_cast<cudaStream_t>(stream), XVs_dev,
                          save_V);
}

size_t dsmil_value_backward_bags_dev_workspace_bytes(const dsmil_params_t* p, int32_t nb, int64_t max_rows) {
  return backward_bags_dev_ws(ROUTE_VAL, p, nb, max_rows);
}
int dsmil_value_backward_bags_dev(const dsmil_params_t* p, const float* const* Xs_dev, const float* const* XVs_dev,
                                  const int64_t* Ns_dev, int32_t nb, int64_t max_rows, const float* Q,
                                  const float* H1, const float* V, const float* A, const float* B,
                                  const int64_t* crit_idx, const float* d_classes, const float* d_pred,
                                  const float* d_A, const float* d_B, const dsmil_grads_t* grads, int32_t* status,
                                  void* workspace, size_t workspace_bytes, void* stream) {
  return backward_bags_dev(ROUTE_VAL, p, Xs_dev, Ns_dev, nb, max_rows, Q, H1, A, B, crit_idx, d_classes, d_pred, d_A,
                           d_B, grads, status, workspace, workspace_bytes, static_cast<cudaStream_t>(stream), XVs_dev,
                           V);
}

}  // extern "C"
