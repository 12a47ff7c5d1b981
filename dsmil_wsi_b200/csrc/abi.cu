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

static inline int attend_ctas(int64_t N) {
  const int64_t tiles = (N + kAttendRows - 1) / kAttendRows;
  return static_cast<int>(tiles < kSplits ? (tiles < 1 ? 1 : tiles) : kSplits);
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
  unsigned long long* keys;  // [nb][kMaxC] arg-max keys, then nb finalize arrival counters: one memset zeroes both
  unsigned int* counters;
  uint8_t* wimg;             // bf16 weight images, 1024-byte aligned; NULL on shapes k_qmlp_sm90 does not take
};
static void carve_phase1(Carver& c, const dsmil_params_t* p, int nb, Phase1Ws& w) {
  w.table = c.take<sm90::BagDev>(nb);
  w.keys = c.take<unsigned long long>(static_cast<size_t>(nb) * (kMaxC + 1));
  w.counters = reinterpret_cast<unsigned int*>(w.keys ? w.keys + static_cast<size_t>(nb) * kMaxC : nullptr);
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

// Scores (or, single bag only, the arg-max of the given scores classes_in), arg-max keys and Q (+ H1 when non-NULL)
// of the nb bags; *tiles and *recs return the batch's 128-row tiles and partial records.  upload == false leaves the
// table and the weight images as an earlier call with the same arguments wrote them into the same workspace.
static int bags_phase1_impl(const dsmil_params_t* p, const Phase1Ws& w, const float* const* Xs, const int64_t* Ns,
                            int nb, const float* classes_in, float* classes, float* Q, float* H1, bool q_blocked,
                            bool upload, int* tiles, int* recs, cudaStream_t st) {
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
  return sm90::launch_qmlp(p, w.table, nb, *tiles, classes_in ? nullptr : classes, w.keys, Q, H1, w.wimg, num_sms(),
                           st, q_blocked);
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
  const bool vec = (D % 4 == 0) && ((reinterpret_cast<uintptr_t>(X) & 15) == 0);
  const int mode = !vec ? 0 : (D % 64 == 0 ? 2 : 1);
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

static int forward_bags_impl(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int nb,
                             const float* classes_in, float* classes, float* pred, float* A, float* B,
                             int64_t* crit, float* save_Q, float* save_H1, void* ws, size_t ws_bytes,
                             cudaStream_t st);

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
  if (sm90::batched_supported(p) && (reinterpret_cast<uintptr_t>(X) & 15) == 0)
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
// first *recs_dev of a capacity grid of `recs`), then each bag's A, B, logits and critical rows.
static int bags_attend_finalize(const dsmil_params_t* p, const BagsWs& w, int nb, const float* Q, bool q_blocked,
                                float* pred, float* A, float* B, int64_t* crit, int recs, const int* recs_dev,
                                cudaStream_t st) {
  const int C = p->C, D = p->D;
  int rc;
  sm90::AttendArgs aa{w.table, nb, D, C, Q, q_blocked, w.keys, A, w.recs, nullptr, recs_dev};
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
  int tiles, recs;
  if ((rc = bags_phase1_impl(p, w, Xs, Ns, nb, classes_in, classes, Q, save_H1, q_blocked, true, &tiles, &recs, st)))
    return rc;
  return bags_attend_finalize(p, w, nb, Q, q_blocked, pred, A, B, crit, recs, nullptr, st);
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
  bool ok;
  size_t a = carve_fwd(p, N, nullptr, 0, &ok).bytes;
  if (sm90::batched_supported(p) && N > 0) a = std::max(a, carve_bags(p, &N, 1, true, false, nullptr, 0, &ok).bytes);
  return a;
}

size_t dsmil_forward_bags_workspace_bytes(const dsmil_params_t* p, const int64_t* Ns, int32_t nb) {
  if (!p || !Ns || nb < 1 || p->C < 1 || p->C > DSMIL_MAX_C || p->D < 1 || p->D > DSMIL_MAX_D) return 0;
  bool ok;
  // Even on a shape of the tensor-core batch, a bag that is not 16-byte aligned sends dsmil_forward_bags down the
  // per-bag loop: the workspace must cover both layouts.
  int64_t mx = 0;
  for (int b = 0; b < nb; ++b) mx = std::max<int64_t>(mx, Ns[b]);
  size_t bytes = carve_fwd(p, mx, nullptr, 0, &ok).bytes;
  if (sm90::batched_supported(p)) bytes = std::max(bytes, carve_bags(p, Ns, nb, true, false, nullptr, 0, &ok).bytes);
  return bytes;
}

int dsmil_forward_bags(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                       float* classes, float* pred, float* A, float* B, int64_t* crit_idx, void* workspace,
                       size_t workspace_bytes, void* stream) {
  int rc = check_params(p, true);
  if (rc) return rc;
  DSMIL_REQUIRE(Xs && Ns && nb >= 1 && classes && pred && A && B, "NULL pointer or nb < 1");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int64_t total;
  bool aligned;
  if ((rc = check_bags(Xs, Ns, nb, &total, &aligned))) return rc;
  // one contract for both routes below: the size dsmil_forward_bags_workspace_bytes reports
  const size_t need = dsmil_forward_bags_workspace_bytes(p, Ns, nb);
  if ((rc = check_workspace(need, workspace_bytes >= need, workspace, workspace ? workspace_bytes : 0))) return rc;
  if (sm90::batched_supported(p) && aligned)
    return forward_bags_impl(p, Xs, Ns, nb, nullptr, classes, pred, A, B, crit_idx, nullptr, nullptr, workspace,
                             workspace_bytes, st);
  // shapes the tensor-core kernels do not take: same packed outputs, one bag at a time
  int64_t row = 0;
  for (int b = 0; b < nb; ++b) {
    rc = forward_impl(p, Xs[b], nullptr, nullptr, Ns[b], classes + row * p->C, pred + static_cast<size_t>(b) * p->C,
                      A + row * p->C, B + static_cast<size_t>(b) * p->C * p->D,
                      crit_idx ? crit_idx + static_cast<size_t>(b) * p->C : nullptr, nullptr, nullptr, nullptr,
                      workspace, workspace_bytes, st);
    if (rc) return rc;
    row += Ns[b];
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
static int bwd_bags_phase1_impl(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int nb,
                                int64_t total, const float* A, const float* B, const float* d_classes,
                                const float* d_pred, const float* d_A, const float* d_B, const dsmil_grads_t* g,
                                float* dA, const BwdBagsWs& w, cudaStream_t st) {
  const int C = p->C, D = p->D;
  const BagsPlan* pl = w.plan;
  int rc;
  if (!pl) {
    // the kernels read X, N and row_off of the table (not the forward's tile and record numbering), at any alignment
    std::vector<sm90::BagDev> tbl(nb);
    long long row = 0;
    for (int b = 0; b < nb; ++b) {
      tbl[b] = sm90::BagDev{Xs[b], Ns[b], row, 0, 0, 0, 0};
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

// Phase 2: dL = A (dA - t_b) / sqrt(128), t_b the sum of the P partials per bag in `tpart` (a dev call: phase 1's
// live G of them); dqm[b] = dL_b^T Q_b, summed over the CTAs' shares in a fixed order.
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
      (rc = bwd_bags_phase2_impl(p, nb, A, w.dA, w.tpart, w.G, Q, w.dL, w.dqm, w, st)) ||
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

// ---- sharded batch ABI ---------------------------------------------------------------------------
int dsmil_shard_bags_supported(const dsmil_params_t* p) {
  return (p && p->C >= 1 && p->C <= DSMIL_MAX_C && p->D >= 1 && p->D <= DSMIL_MAX_D && sm90::batched_supported(p)) ? 1 : 0;
}
size_t dsmil_shard_bags_workspace_bytes(const dsmil_params_t* p, const int64_t* Ns, int32_t nb) {
  if (!dsmil_shard_bags_supported(p) || !Ns || nb < 1) return 0;
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
// partial record.
static int shard_bags_phase2_impl(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int nb,
                                  const float* Q, bool q_blocked, const float* cands_all, int G, float* A,
                                  int64_t* crit_idx, float* qmax, float* recs_out, const BagsWs& w, cudaStream_t st) {
  std::vector<sm90::BagDev> tbl;
  int tiles = 0, recs = 0, rc;
  if ((rc = build_table(Xs, Ns, nb, tbl, &tiles, &recs))) return rc;   // the device table was written by phase 1
  k_merge_cand<<<dim3(p->C, nb), kQ, 0, st>>>(cands_all, G, nb, p->C, qmax, crit_idx);
  DSMIL_LAUNCH_OK("k_merge_cand");
  sm90::AttendArgs aa{w.table, nb, p->D, p->C, Q, q_blocked, w.keys, A, w.recs, qmax, nullptr};
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
  DSMIL_REQUIRE(Xs && Ns && nb >= 1 && row_offsets && classes && cand_recs, "NULL pointer or nb < 1");
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
  DSMIL_REQUIRE(dsmil_shard_bags_supported(p) && Xs && Ns && nb >= 1 && cands_all && G >= 1 && A && crit_idx && recs_out,
                "bad arguments");
  bool ok;
  BagsWs w = carve_bags(p, Ns, nb, true, true, workspace, workspace_bytes, &ok);
  if ((rc = check_workspace(w.bytes, ok, workspace, workspace_bytes))) return rc;
  return shard_bags_phase2_impl(p, Xs, Ns, nb, w.Q, true, cands_all, G, A, crit_idx, w.qmax, recs_out, w,
                                static_cast<cudaStream_t>(stream));
}
int dsmil_shard_bags_phase3(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                            const float* recs_all, int32_t G, float* A, float* B, float* pred, void* workspace,
                            size_t workspace_bytes, void* stream) {
  int rc = check_params(p, true);
  if (rc) return rc;
  DSMIL_REQUIRE(dsmil_shard_bags_supported(p) && Xs && Ns && nb >= 1 && recs_all && G >= 1 && G <= sm90::kMaxRecPerBag && A && B && pred,
                "bad arguments");
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
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int64_t total;
  bool aligned;
  if ((rc = check_bags(Xs, Ns, nb, &total, &aligned))) return rc;
  const size_t need = dsmil_forward_bags_train_workspace_bytes(p, Ns, nb);
  if ((rc = check_workspace(need, workspace_bytes >= need, workspace, workspace ? workspace_bytes : 0))) return rc;
  if (sm90::batched_supported(p) && aligned)
    return forward_bags_impl(p, Xs, Ns, nb, nullptr, classes, pred, A, B, crit_idx, save_Q, save_H1, workspace,
                             workspace_bytes, st);
  // shapes or bags off the tensor-core batch: one bag at a time into the same packed buffers
  int64_t row = 0;
  for (int b = 0; b < nb; ++b) {
    rc = forward_impl(p, Xs[b], nullptr, nullptr, Ns[b], classes + row * p->C, pred + static_cast<size_t>(b) * p->C,
                      A + row * p->C, B + static_cast<size_t>(b) * p->C * p->D, crit_idx + static_cast<size_t>(b) * p->C,
                      save_Q + row * kQ, save_H1 ? save_H1 + row * kQ : nullptr, nullptr, workspace, workspace_bytes,
                      st);
    if (rc) return rc;
    row += Ns[b];
  }
  return 0;
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
  if ((rc = check_workspace(need, workspace_bytes >= need, workspace, workspace ? workspace_bytes : 0))) return rc;
  return backward_bags_impl(p, Xs, Ns, nb, total, aligned, Q, H1, A, B, crit_idx, d_classes, d_pred, d_A, d_B, grads,
                            workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
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
  return shard_bags_phase2_impl(p, Xs, Ns, nb, Q, false, cands_all, G, A, crit_idx, q_max, recs_out, w,
                                static_cast<cudaStream_t>(stream));
}

size_t dsmil_shard_backward_bags_workspace_bytes(const dsmil_params_t* p, const int64_t* Ns, int32_t nb) {
  if (!dsmil_shard_bags_supported(p) || !Ns || nb < 1) return 0;
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
// What both dev calls check: the batched tensor-core shapes, the bag list, 1 <= nb <= 65535 and a row capacity whose
// 128-row tiles the kernels can number (an int).
static int check_bags_dev(const dsmil_params_t* p, bool need_scores, const float* const* Xs, const int64_t* Ns, int nb,
                          int64_t max_rows, const int32_t* status) {
  int rc = check_params(p, need_scores);
  if (rc) return rc;
  DSMIL_REQUIRE(dsmil_shard_bags_supported(p),
                "shape not supported by the batched tensor-core path (D=%d, C=%d, nonlinear=%d, passing_v=%d)", p->D,
                p->C, p->nonlinear, p->passing_v);
  DSMIL_REQUIRE(Xs && Ns && status, "NULL bag list or status");
  DSMIL_REQUIRE(nb >= 1 && nb <= 65535, "nb=%d outside [1, 65535]", nb);
  DSMIL_REQUIRE(max_rows >= 1 && max_rows < 0xffffffffll &&
                static_cast<int64_t>(nb) * ((max_rows + sm90::kTileM - 1) / sm90::kTileM) <= INT_MAX,
                "max_rows=%lld out of range for nb=%d", (long long)max_rows, nb);
  return 0;
}

// The forward's carve for nb bags of max_rows rows (Q and H1 are the caller's), then the planner's BagsPlan and the
// zero row of a refused batch.
static BagsWs carve_bags_dev(const dsmil_params_t* p, int nb, int64_t max_rows, void* ws, size_t cap, bool* ok,
                             BagsPlan** plan, float** zero_row) {
  const std::vector<int64_t> Ns(nb, max_rows);
  BagsWs w = carve_bags(p, Ns.data(), nb, false, false, ws, cap, ok);
  Carver c(ws, cap);
  c.off = w.bytes;
  *plan = c.take<BagsPlan>(1);
  *zero_row = c.take<float>(p->D);
  w.bytes = c.off;
  *ok = c.ok();
  return w;
}

size_t dsmil_forward_bags_train_dev_workspace_bytes(const dsmil_params_t* p, int32_t nb, int64_t max_rows) {
  if (!dsmil_shard_bags_supported(p) || nb < 1 || nb > 65535 || max_rows < 1 || max_rows >= 0xffffffffll) return 0;
  bool ok;
  BagsPlan* plan;
  float* zero_row;
  const size_t dev = carve_bags_dev(p, nb, max_rows, nullptr, 0, &ok, &plan, &zero_row).bytes;
  // never below the eager call's size for the same capacity: one buffer serves both forms
  const std::vector<int64_t> Ns(nb, max_rows);
  return std::max(dev, dsmil_forward_bags_train_workspace_bytes(p, Ns.data(), nb));
}

int dsmil_forward_bags_train_dev(const dsmil_params_t* p, const float* const* Xs_dev, const int64_t* Ns_dev,
                                 int32_t nb, int64_t max_rows, float* classes, float* pred, float* A, float* B,
                                 int64_t* crit_idx, float* save_Q, float* save_H1, int32_t* status, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  int rc = check_bags_dev(p, true, Xs_dev, Ns_dev, nb, max_rows, status);
  if (rc) return rc;
  DSMIL_REQUIRE(classes && pred && A && B && crit_idx && save_Q && save_H1, "NULL output pointer");
  const size_t need = dsmil_forward_bags_train_dev_workspace_bytes(p, nb, max_rows);
  if ((rc = check_workspace(need, workspace_bytes >= need, workspace, workspace ? workspace_bytes : 0))) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  bool ok;
  BagsPlan* plan;
  float* zero_row;
  BagsWs w = carve_bags_dev(p, nb, max_rows, workspace, workspace_bytes, &ok, &plan, &zero_row);
  k_plan_bags<<<1, 32, 0, st>>>(Xs_dev, Ns_dev, nb, max_rows, p->C, p->D, zero_row, w.table, nullptr, nullptr, plan,
                                status);
  DSMIL_LAUNCH_OK("k_plan_bags");
  // bags_phase1_impl's launches, on the planner's table and with the weight images rebuilt on every call (a replayed
  // graph sees the weights of the last optimizer step)
  DSMIL_CUDA_OK(cudaMemsetAsync(w.keys, 0, sizeof(unsigned long long) * (kMaxC + 1) * nb, st));
  if ((rc = sm90::launch_prep_wimg(p, w.wimg, st))) return rc;
  if ((rc = sm90::launch_qmlp(p, w.table, nb, nb * tiles_for_bag(max_rows), classes, w.keys, save_Q, save_H1, w.wimg,
                              num_sms(), st, false, &plan->tiles)))
    return rc;
  return bags_attend_finalize(p, w, nb, save_Q, false, pred, A, B, crit_idx, nb * recs_for_bag(max_rows), &plan->recs,
                              st);
}

size_t dsmil_backward_bags_dev_workspace_bytes(const dsmil_params_t* p, int32_t nb, int64_t max_rows) {
  if (!dsmil_shard_bags_supported(p) || nb < 1 || nb > 65535 || max_rows < 1 || max_rows >= 0xffffffffll) return 0;
  bool ok;
  return carve_bwd_bags_dev(p, nb, max_rows, nullptr, 0, &ok).bytes;
}

int dsmil_backward_bags_dev(const dsmil_params_t* p, const float* const* Xs_dev, const int64_t* Ns_dev, int32_t nb,
                            int64_t max_rows, const float* Q, const float* H1, const float* A, const float* B,
                            const int64_t* crit_idx, const float* d_classes, const float* d_pred, const float* d_A,
                            const float* d_B, const dsmil_grads_t* grads, int32_t* status, void* workspace,
                            size_t workspace_bytes, void* stream) {
  int rc = check_bags_dev(p, false, Xs_dev, Ns_dev, nb, max_rows, status);
  if (rc) return rc;
  DSMIL_REQUIRE(Q && H1 && A && B && crit_idx && grads, "NULL pointer");
  DSMIL_REQUIRE(!d_A && !d_B && !grads->gX,
                "the dev backward takes gradients through classes and pred only (no d_A, d_B or gX)");
  const size_t need = dsmil_backward_bags_dev_workspace_bytes(p, nb, max_rows);
  if ((rc = check_workspace(need, workspace_bytes >= need, workspace, workspace ? workspace_bytes : 0))) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  bool ok;
  BwdBagsWs w = carve_bwd_bags_dev(p, nb, max_rows, workspace, workspace_bytes, &ok);
  k_plan_bags<<<1, 32, 0, st>>>(Xs_dev, Ns_dev, nb, max_rows, p->C, p->D, w.zero_row, w.table, w.chi, w.ch1, w.plan,
                                status);
  DSMIL_LAUNCH_OK("k_plan_bags");
  return backward_bags_run(p, nullptr, nullptr, nb, static_cast<int64_t>(nb) * max_rows, Q, H1, A, B, crit_idx,
                           d_classes, d_pred, nullptr, nullptr, grads, w, st);
}

}  // extern "C"
