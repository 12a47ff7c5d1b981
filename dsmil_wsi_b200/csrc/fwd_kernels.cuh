// Forward kernels of the DSMIL aggregator that are shape-generic (any D, C <= 8).
//   k_scores        dsmil.py:11 / :24   instance scores + per-class arg-max key (dsmil.py:52 row 0)
//   k_argmax        dsmil.py:52         arg-max key from GIVEN scores (call form b_classifier(feats, c))
//   k_gather_cand   dsmil.py:53-54      critical row -> candidate record (score, global idx, q row)
//   k_merge_cand    SURVEY A.3 exchange 1
//   k_attend        dsmil.py:55-57      logits, online softmax over instances, partial bag vector
//   k_combine_rec   SURVEY A.3 exchange 2 (also combines per-CTA partials on one device)
//   k_finalize      dsmil.py:56 (normalise A), :57 (B), :59-61 (Conv1d == GEMV)
#pragma once
#include "common.cuh"

namespace dsmil {

// ------------------------------------------------------------------------------------------
// scores: one warp per row (grid-stride), Wi staged in shared memory, float4 loads when legal.
// MODE 0: scalar loads (any D).  MODE 1: float4, one warp per row.  MODE 2 (D % 64 == 0): float4, FOUR lanes
// per row with exactly the summation order of the tensor-core kernel's fused scores
// (fwd_sm90.cuh: lane `seg` takes float4 #seg, #seg+4, ... of the row, then xor-shuffles 2,1), so
// FCLayer/IClassifier scores are bit-identical whichever kernel produced them.
template <int MODE>
__global__ void __launch_bounds__(256)
k_scores(const float* __restrict__ X, int64_t N, int D, const float* __restrict__ Wi,
         const float* __restrict__ bi, int C, float* __restrict__ classes,
         unsigned long long* __restrict__ keys) {
  extern __shared__ __align__(16) float sWi[];  // [C*D]
  __shared__ unsigned long long sbest[8][kMaxC];
  for (int i = threadIdx.x; i < C * D; i += blockDim.x) sWi[i] = __ldg(Wi + i);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long best[kMaxC];
#pragma unroll
  for (int k = 0; k < kMaxC; ++k) best[k] = 0ull;
  constexpr int RPW = (MODE == 2) ? 8 : 1;  // rows per warp per iteration
  const int sub = (MODE == 2) ? (lane >> 2) : 0;
  const int seg = (MODE == 2) ? (lane & 3) : lane;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * 8 * RPW;
  for (int64_t n0 = (static_cast<int64_t>(blockIdx.x) * 8 + warp) * RPW; n0 < N; n0 += stride) {
    const int64_t n = n0 + sub;
    const bool live = n < N;
    float acc[kMaxC];
#pragma unroll
    for (int k = 0; k < kMaxC; ++k) acc[k] = 0.f;
    const float* row = X + (live ? n : n0) * D;
    if (MODE >= 1) {
      const float4* r4 = reinterpret_cast<const float4*>(row);
      const int D4 = D >> 2;
      const int step = (MODE == 2) ? 4 : 32;
      for (int j = seg; j < D4; j += step) {
        const float4 x = __ldg(r4 + j);
#pragma unroll
        for (int k = 0; k < kMaxC; ++k)
          if (k < C) {
            const float4 w = *reinterpret_cast<const float4*>(sWi + k * D + j * 4);
            acc[k] = fmaf(x.x, w.x, acc[k]);
            acc[k] = fmaf(x.y, w.y, acc[k]);
            acc[k] = fmaf(x.z, w.z, acc[k]);
            acc[k] = fmaf(x.w, w.w, acc[k]);
          }
      }
    } else {
      for (int j = lane; j < D; j += 32) {
        const float x = __ldg(row + j);
#pragma unroll
        for (int k = 0; k < kMaxC; ++k)
          if (k < C) acc[k] = fmaf(x, sWi[k * D + j], acc[k]);
      }
    }
#pragma unroll
    for (int k = 0; k < kMaxC; ++k)
      if (k < C) {
        float v = acc[k];
        if (MODE == 2) {
          v += __shfl_xor_sync(0xffffffffu, v, 2);
          v += __shfl_xor_sync(0xffffffffu, v, 1);
        } else {
          v = warp_sum(v);
        }
        v += __ldg(bi + k);
        if (seg == 0 && live) {
          classes[n * C + k] = v;
          const unsigned long long key = pack_key(v, static_cast<uint32_t>(n));
          best[k] = key > best[k] ? key : best[k];
        }
      }
  }
#pragma unroll
  for (int k = 0; k < kMaxC; ++k) {
    best[k] = warp_max_u64(best[k]);   // MODE 2 keeps eight partial bests per warp (lanes 0, 4, ..., 28)
    if (lane == 0) sbest[warp][k] = best[k];
  }
  __syncthreads();
  if (threadIdx.x < C) {
    unsigned long long b = 0ull;
    for (int w = 0; w < 8; ++w) b = sbest[w][threadIdx.x] > b ? sbest[w][threadIdx.x] : b;
    if (b) atomicMax(keys + threadIdx.x, b);
  }
}

__global__ void __launch_bounds__(256)
k_argmax(const float* __restrict__ classes, int64_t N, int C, unsigned long long* __restrict__ keys) {
  __shared__ unsigned long long sbest[8][kMaxC];
  unsigned long long best[kMaxC];
#pragma unroll
  for (int k = 0; k < kMaxC; ++k) best[k] = 0ull;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t n = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; n < N; n += stride) {
#pragma unroll
    for (int k = 0; k < kMaxC; ++k)
      if (k < C) {
        const unsigned long long key = pack_key(__ldg(classes + n * C + k), static_cast<uint32_t>(n));
        best[k] = key > best[k] ? key : best[k];
      }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < kMaxC; ++k) {
    best[k] = warp_max_u64(best[k]);
    if (lane == 0) sbest[warp][k] = best[k];
  }
  __syncthreads();
  if (threadIdx.x < C) {
    unsigned long long b = 0ull;
    for (int w = 0; w < 8; ++w) b = sbest[w][threadIdx.x] > b ? sbest[w][threadIdx.x] : b;
    if (b) atomicMax(keys + threadIdx.x, b);
  }
}

// Candidate record layout (floats): idx[C] as int64 (2 floats each) | score[C] | qrow[C*128],
// padded to a multiple of 4 floats so that records packed back to back keep the int64 aligned.
__host__ __device__ inline size_t cand_floats(int C) { return (static_cast<size_t>(C) * (2 + 1 + kQ) + 3) & ~size_t(3); }

__global__ void __launch_bounds__(128)
k_gather_cand(const unsigned long long* __restrict__ keys, const float* __restrict__ classes,
              const float* __restrict__ Q, int64_t N, int C, int64_t row_offset, float* __restrict__ cand) {
  const int k = blockIdx.x;
  int64_t* idx = reinterpret_cast<int64_t*>(cand);
  float* score = cand + 2 * C;
  float* qrow = cand + 3 * C + static_cast<size_t>(k) * kQ;
  const unsigned long long key = keys[k];
  if (N <= 0 || key == 0ull) {  // empty shard: can never win the merge
    if (threadIdx.x == 0) {
      idx[k] = INT64_MAX;
      score[k] = -INFINITY;
    }
    qrow[threadIdx.x] = 0.f;
    return;
  }
  const int64_t row = key_row(key);
  if (threadIdx.x == 0) {
    idx[k] = row + row_offset;
    score[k] = classes[row * C + k];
  }
  qrow[threadIdx.x] = Q[row * kQ + threadIdx.x];
}

// Winner per (bag, class) over the G candidate records cands[g][bag] of each of nb bags: max score (NaN first),
// lowest global index on ties.  grid = (C, nb), 128 threads; q_max [nb][C][128], crit_idx [nb][C].
__global__ void __launch_bounds__(128)
k_merge_cand(const float* __restrict__ cands, int G, int nb, int C, float* __restrict__ q_max,
             int64_t* __restrict__ crit_idx) {
  const int k = blockIdx.x, bag = blockIdx.y;
  const size_t stride = cand_floats(C);
  int best_g = -1;
  uint32_t best_key = 0;
  int64_t best_idx = INT64_MAX;
  for (int g = 0; g < G; ++g) {
    const float* rec = cands + (static_cast<size_t>(g) * nb + bag) * stride;
    const int64_t gi = reinterpret_cast<const int64_t*>(rec)[k];
    if (gi == INT64_MAX) continue;
    const uint32_t key = ordered_key(rec[2 * C + k]);
    if (best_g < 0 || key > best_key || (key == best_key && gi < best_idx)) {
      best_g = g; best_key = key; best_idx = gi;
    }
  }
  float* out = q_max + (static_cast<size_t>(bag) * C + k) * kQ;
  int64_t* crit = crit_idx + static_cast<size_t>(bag) * C;
  if (best_g < 0) {  // every shard empty
    if (threadIdx.x == 0) crit[k] = -1;
    out[threadIdx.x] = 0.f;
    return;
  }
  if (threadIdx.x == 0) crit[k] = best_idx;
  out[threadIdx.x] = cands[(static_cast<size_t>(best_g) * nb + bag) * stride + 3 * C + static_cast<size_t>(k) * kQ + threadIdx.x];
}

// ------------------------------------------------------------------------------------------
// Partial record layout (floats): m[C] | s[C] | Bp[C*Dv], padded to a multiple of 4 floats
__host__ __device__ inline size_t rec_floats(int C, int Dv) { return (static_cast<size_t>(C) * (2 + Dv) + 3) & ~size_t(3); }

constexpr int kAttendRows = 32;

// One CTA walks row tiles t = blockIdx.x, += gridDim.x.  CT = classes rounded up (1,2,4,8),
// J = ceil(Dv/256) rounded up (1,2,4,8,16): thread t owns feature columns t + 256*j.
template <int CT, int J>
__global__ void __launch_bounds__(256)
k_attend(const float* __restrict__ V, int Dv, const float* __restrict__ Q, int64_t N,
         const float* __restrict__ q_max, int C, float* __restrict__ A, float* __restrict__ recs) {
  __shared__ __align__(16) float sq[CT][kQ];
  __shared__ float sL[kAttendRows][CT];
  __shared__ float sE[kAttendRows][CT];
  __shared__ float s_m[CT], s_s[CT], s_scale[CT];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < CT * kQ; i += 256) sq[i / kQ][i % kQ] = (i / kQ) < C ? __ldg(q_max + i) : 0.f;
  if (tid < CT) { s_m[tid] = -INFINITY; s_s[tid] = 0.f; }
  float acc[CT][J];
#pragma unroll
  for (int k = 0; k < CT; ++k)
#pragma unroll
    for (int j = 0; j < J; ++j) acc[k][j] = 0.f;
  __syncthreads();

  const int64_t tiles = (N + kAttendRows - 1) / kAttendRows;
  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int64_t r0 = t * kAttendRows;
    // (a) logits of this tile: warp w takes rows w, w+8, w+16, w+24
#pragma unroll
    for (int rr = 0; rr < kAttendRows / 8; ++rr) {
      const int r = warp + rr * 8;
      const int64_t n = r0 + r;
      if (n < N) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(Q + n * kQ) + lane);
#pragma unroll
        for (int k = 0; k < CT; ++k) {
          const float4 w = *reinterpret_cast<const float4*>(&sq[k][lane * 4]);
          float d = q.x * w.x;
          d = fmaf(q.y, w.y, d);
          d = fmaf(q.z, w.z, d);
          d = fmaf(q.w, w.w, d);
          d = warp_sum(d);
          if (lane == 0) {
            const float L = __fdiv_rn(d, kScale);  // dsmil.py:56: a division by sqrt(128f)
            sL[r][k] = L;
            if (k < C) A[n * C + k] = L;
          }
        }
      } else if (lane < CT) {
        sL[r][lane] = -INFINITY;
      }
    }
    __syncthreads();
    // (b) running max / rescale factor per class
    if (tid < CT) {
      float mx = s_m[tid];
#pragma unroll
      for (int r = 0; r < kAttendRows; ++r) mx = fmaxf(mx, sL[r][tid]);
      // NaN logits (NaN features) poison the column exactly like softmax does in the reference
      const float old = s_m[tid];
      s_scale[tid] = (old == -INFINITY) ? 0.f : expf(old - mx);
      s_m[tid] = mx;
    }
    __syncthreads();
    if (tid < kAttendRows * CT) {
      const int r = tid / CT, k = tid % CT;
      const float L = sL[r][k];
      sE[r][k] = (L == -INFINITY) ? 0.f : expf(L - s_m[k]);
    }
    __syncthreads();
    // (c) accumulate: sum and weighted feature sum
    if (tid < CT) {
      float s = s_s[tid] * s_scale[tid];
#pragma unroll
      for (int r = 0; r < kAttendRows; ++r) s += sE[r][tid];
      s_s[tid] = s;
    }
#pragma unroll
    for (int k = 0; k < CT; ++k) {
      const float sc = s_scale[k];
#pragma unroll
      for (int j = 0; j < J; ++j) acc[k][j] *= sc;
    }
    const int rows = (N - r0) < kAttendRows ? static_cast<int>(N - r0) : kAttendRows;
#pragma unroll 4
    for (int r = 0; r < rows; ++r) {
      const float* vrow = V + (r0 + r) * Dv;
      float x[J];
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const int col = tid + 256 * j;
        x[j] = col < Dv ? __ldg(vrow + col) : 0.f;
      }
#pragma unroll
      for (int k = 0; k < CT; ++k) {
        const float e = sE[r][k];
#pragma unroll
        for (int j = 0; j < J; ++j) acc[k][j] = fmaf(e, x[j], acc[k][j]);
      }
    }
    __syncthreads();
  }
  float* rec = recs + static_cast<size_t>(blockIdx.x) * rec_floats(C, Dv);
  if (tid < C) { rec[tid] = s_m[tid]; rec[C + tid] = s_s[tid]; }
#pragma unroll
  for (int k = 0; k < CT; ++k)
    if (k < C) {
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const int col = tid + 256 * j;
        if (col < Dv) rec[2 * C + static_cast<size_t>(k) * Dv + col] = acc[k][j];
      }
    }
}

// Combine P records (per-CTA partials, or per-rank records) into one, fixed order.
// grid = (C, ceil(Dv/256)); P <= kMaxRecs.
constexpr int kMaxRecs = 1024;
__global__ void __launch_bounds__(256)
k_combine_rec(const float* __restrict__ recs, int P, int C, int Dv, float* __restrict__ out) {
  __shared__ float w[kMaxRecs];
  __shared__ float sM;
  const int k = blockIdx.x;
  const size_t stride = rec_floats(C, Dv);
  if (threadIdx.x == 0) {
    float M = -INFINITY;
    for (int p = 0; p < P; ++p) M = fmaxf(M, recs[p * stride + k]);
    // fmaxf drops NaN; re-inject so NaN partials poison the result like the reference softmax
    for (int p = 0; p < P; ++p) { const float m = recs[p * stride + k]; if (m != m) M = m; }
    sM = M;
  }
  __syncthreads();
  const float M = sM;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const float m = recs[p * stride + k];
    w[p] = (m == -INFINITY) ? 0.f : expf(m - M);
  }
  __syncthreads();
  if (blockIdx.y == 0 && threadIdx.x == 0) {
    float S = 0.f;
    for (int p = 0; p < P; ++p) S = fmaf(recs[p * stride + C + k], w[p], S);
    out[k] = M;
    out[C + k] = S;
  }
  const int d = blockIdx.y * blockDim.x + threadIdx.x;
  if (d < Dv) {
    float b = 0.f;
    for (int p = 0; p < P; ++p) b = fmaf(recs[p * stride + 2 * C + static_cast<size_t>(k) * Dv + d], w[p], b);
    out[2 * C + static_cast<size_t>(k) * Dv + d] = b;
  }
}

// A[n,k] = exp(L - M_k) / S_k in place; block 0 also emits B = Bp / S and the bag logits.
__global__ void __launch_bounds__(256)
k_finalize(const float* __restrict__ rec, int64_t N, int C, int Dv, const float* __restrict__ Wf,
           const float* __restrict__ bf, float* __restrict__ A, float* __restrict__ B,
           float* __restrict__ pred) {
  __shared__ float sM[kMaxC], sS[kMaxC];
  __shared__ float red[8];
  if (threadIdx.x < C) { sM[threadIdx.x] = rec[threadIdx.x]; sS[threadIdx.x] = rec[C + threadIdx.x]; }
  __syncthreads();
  const int64_t total = N * C;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int k = static_cast<int>(i % C);
    A[i] = __fdiv_rn(expf(A[i] - sM[k]), sS[k]);
  }
  if (blockIdx.x != 0) return;
  for (int i = threadIdx.x; i < C * Dv; i += blockDim.x) B[i] = __fdiv_rn(rec[2 * C + i], sS[i / Dv]);
  __syncthreads();  // B written by this block is visible to it after the barrier
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k = 0; k < C; ++k) {
    float p = 0.f;
    const float* wrow = Wf + static_cast<size_t>(k) * C * Dv;
    for (int i = threadIdx.x; i < C * Dv; i += blockDim.x) p = fmaf(__ldg(wrow + i), B[i], p);
    p = warp_sum(p);
    if (lane == 0) red[warp] = p;
    __syncthreads();
    if (threadIdx.x == 0) {
      float s = 0.f;
      for (int w = 0; w < 8; ++w) s += red[w];
      pred[k] = s + __ldg(bf + k);
    }
    __syncthreads();
  }
}

}  // namespace dsmil
