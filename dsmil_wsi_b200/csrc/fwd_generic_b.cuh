// The generic forward over a bag table: the kernels of the per-bag generic forward (fwd_kernels.cuh, k_linear), one
// launch per stage for the whole batch, on the shapes the tensor-core batch does not take (identity v; any D <= 4096,
// C <= 8, either q form).  Each runs the per-bag kernel's body on its bag's rows, so every bag's outputs are the bits
// the per-bag forward gives it (DESIGN §4.2h).  The table (bag_plan.cuh: gen_bag_entry) numbers each bag's 128-row
// tiles (tile_off), its attend_ctas(N) partial records (rec_off, nrec) and carries its k_scores MODE in pad_.
// The fold form (dsmil_generic_forward_bags_models_train_dev) runs the same launches over every model's bags at once:
// its table carries each entry's model beside the MODE (bag_plan.cuh: fold_pad), and the stages that read weights
// (k_scores_b, k_linear_b, k_finalize_gb) take them from `models` [M] by the entry's model.  A one-model table's pad_
// is its MODE (model 0) and `models` is NULL there, so those stages read the weights they are passed.
//   k_scores_b       k_scores per 128-row tile of a bag (the bag's MODE), arg-max keys per bag
//   k_linear_b       layer 1 of the Q-MLP, 64 rows of one bag per CTA (k_linear's tile)
//   k_crit_qmax_b    q_max and the critical rows per (class, bag), as k_gather_cand + k_merge_cand of one bag
//   k_attend_gb      k_attend per (bag, record), attend_ctas(N_b) records per bag
//   k_combine_rec_b  k_combine_rec per bag (grid.z)
//   k_finalize_gb    k_finalize per bag (grid.y)
//   k_vproj_b        the value network's V = relu(Xv W^T + b) per 128-row tile of a bag (passing_v; abi.cu's value
//                    route gives k_attend_gb a table whose X is each bag's packed V)
#pragma once
#include "common.cuh"
#include "gemm_generic.cuh"
#include "fwd_kernels.cuh"
#include "fwd_sm90.cuh"

namespace dsmil {

static_assert(sm90::kTileM == 2 * LBM, "k_linear_b takes two k_linear tiles per 128-row tile");

// pad_ of a generic table entry: the bag's k_scores MODE in bits 0-1, its model (fold tables; 0 otherwise) above them.
__host__ __device__ inline int fold_pad(int mode, int m) { return mode | (m << 2); }
__host__ __device__ inline int fold_pad_mode(int pad) { return pad & 3; }
__host__ __device__ inline int fold_pad_model(int pad) { return pad >> 2; }

// The per-bag kernels' bodies.  They are copies, not shared with k_scores, k_attend and k_finalize: calling a shared
// body from those kernels changes their SASS (DESIGN §4.2h), which the per-bag forward keeps as it was.
// k_scores' body over the rows of one bag: warp w of the CTA takes rows (wbase + w) * RPW, stepping by wstep * RPW,
// below N (one 128-row tile per CTA here).
template <int MODE>
__device__ __forceinline__ void scores_rows(const float* __restrict__ X, int64_t N, int64_t wbase, int64_t wstep, int D,
                                            const float* __restrict__ Wi, const float* __restrict__ bi, int C,
                                            float* __restrict__ classes, unsigned long long* __restrict__ keys) {
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
  const int64_t stride = wstep * RPW;
  for (int64_t n0 = (wbase + warp) * RPW; n0 < N; n0 += stride) {
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
// k_attend's body for CTA `cta` of the `ctas` of one bag: row tiles t = cta, += ctas, its partial record to rec.
template <int CT, int J>
__device__ __forceinline__ void attend_rows(const float* __restrict__ V, int Dv, const float* __restrict__ Q, int64_t N,
                                            const float* __restrict__ q_max, int C, float* __restrict__ A,
                                            float* __restrict__ rec, int cta, int ctas) {
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

  const int tiles = static_cast<int>((N + kAttendRows - 1) / kAttendRows);
  for (int t = cta; t < tiles; t += ctas) {
    const int64_t r0 = static_cast<int64_t>(t) * kAttendRows;
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
// k_finalize's body for block blk of nblk over one bag: A[n,k] = exp(L - M_k) / S_k in place, every nblk-th span of
// 256; block 0 also emits B = Bp / S and the bag logits.
__device__ __forceinline__ void finalize_bag(const float* __restrict__ rec, int64_t N, int C, int Dv,
                                             const float* __restrict__ Wf, const float* __restrict__ bf,
                                             float* __restrict__ A, float* __restrict__ B, float* __restrict__ pred,
                                             int64_t blk, int64_t nblk) {
  __shared__ float sM[kMaxC], sS[kMaxC];
  __shared__ float red[8];
  if (threadIdx.x < C) { sM[threadIdx.x] = rec[threadIdx.x]; sS[threadIdx.x] = rec[C + threadIdx.x]; }
  __syncthreads();
  const int64_t total = N * C;
  const int64_t stride = nblk * blockDim.x;
  for (int64_t i = blk * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int k = static_cast<int>(i % C);
    A[i] = __fdiv_rn(expf(A[i] - sM[k]), sS[k]);
  }
  if (blk != 0) return;
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
// The entry of a table whose ranges [off(b), off(b + 1)) (tile_off, or rec_off with by_rec) hold i: ranges ascending,
// none empty.
__device__ __forceinline__ int bag_of(const sm90::BagDev* __restrict__ bags, int nb, int i, bool by_rec) {
  int lo = 0, hi = nb - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    const int o = by_rec ? bags[mid].rec_off : bags[mid].tile_off;
    if (o <= i) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// grid = tiles (tiles_dev: the live count of a capacity grid); dynamic shared memory C * D floats.  models != NULL:
// Wi / bi of the entry's model instead of the ones passed.
__global__ void __launch_bounds__(256)
k_scores_b(const sm90::BagDev* __restrict__ bags, int nb, const int* __restrict__ tiles_dev, int D,
           const float* __restrict__ Wi, const float* __restrict__ bi, int C, float* __restrict__ classes,
           unsigned long long* __restrict__ keys, const sm90::ModelDev* __restrict__ models) {
  const int t = blockIdx.x;
  if (tiles_dev && t >= *tiles_dev) return;
  const int bag = bag_of(bags, nb, t, false);
  const sm90::BagDev bg = bags[bag];
  if (models) {
    const sm90::ModelDev& md = models[fold_pad_model(bg.pad_)];
    Wi = md.Wi;
    bi = md.bi;
  }
  const int mode = fold_pad_mode(bg.pad_);
  const int64_t tl = t - bg.tile_off;
  const int64_t end = min(static_cast<int64_t>(bg.N), (tl + 1) * sm90::kTileM);
  float* cls = classes + bg.row_off * C;
  unsigned long long* kb = keys + static_cast<size_t>(bag) * kMaxC;
  if (mode == 2) scores_rows<2>(bg.X, end, tl * (sm90::kTileM / 8), 8, D, Wi, bi, C, cls, kb);
  else if (mode == 1) scores_rows<1>(bg.X, end, tl * sm90::kTileM, 8, D, Wi, bi, C, cls, kb);
  else scores_rows<0>(bg.X, end, tl * sm90::kTileM, 8, D, Wi, bi, C, cls, kb);
}

// Y[packed rows, M] = act(X_b W^T + b) over each bag's own rows.  grid = (2 * tiles, ceil(M / LBN)).  models != NULL:
// layer 1 of the entry's model (W1 / b1) instead of W / b.
template <int ACT>
__global__ void __launch_bounds__(256)
k_linear_b(const sm90::BagDev* __restrict__ bags, int nb, const int* __restrict__ tiles_dev, int K,
           const float* __restrict__ W, const float* __restrict__ b, int M, float* __restrict__ Y,
           const sm90::ModelDev* __restrict__ models) {
  const int t = blockIdx.x >> 1;
  if (tiles_dev && t >= *tiles_dev) return;
  const sm90::BagDev bg = bags[bag_of(bags, nb, t, false)];
  const int64_t n0 = static_cast<int64_t>(t - bg.tile_off) * sm90::kTileM + (blockIdx.x & 1) * LBM;
  if (n0 >= bg.N) return;
  if (models) {
    const sm90::ModelDev& md = models[fold_pad_model(bg.pad_)];
    W = md.W1;
    b = md.b1;
  }
  linear_tile<ACT, false>(bg.X, bg.N, n0, K, W, b, M, Y + bg.row_off * M, nullptr, 0);
}

// grid = (C, nb), kQ threads: q_max [nb][C][128] and crit [nb][C] of each bag from its arg-max key.
__global__ void __launch_bounds__(128)
k_crit_qmax_b(const sm90::BagDev* __restrict__ bags, const unsigned long long* __restrict__ keys,
              const float* __restrict__ Q, int C, float* __restrict__ q_max, int64_t* __restrict__ crit) {
  const int k = blockIdx.x, bag = blockIdx.y;
  const unsigned long long key = keys[static_cast<size_t>(bag) * kMaxC + k];
  float* out = q_max + (static_cast<size_t>(bag) * C + k) * kQ;
  int64_t* ci = crit + static_cast<size_t>(bag) * C + k;
  if (key == 0ull) {   // no row scored: what k_merge_cand gives for an empty candidate
    if (threadIdx.x == 0) *ci = -1;
    out[threadIdx.x] = 0.f;
    return;
  }
  const int64_t row = key_row(key);
  if (threadIdx.x == 0) *ci = row;
  out[threadIdx.x] = Q[(bags[bag].row_off + row) * kQ + threadIdx.x];
}

// grid = recs (recs_dev: the live count of a capacity grid): record r of bag b is CTA r - rec_off of b's attend_ctas.
// (256, 1): left to its default target ptxas spills a few registers of some instantiations to hit a higher occupancy.
template <int CT, int J>
__global__ void __launch_bounds__(256, 1)
k_attend_gb(const sm90::BagDev* __restrict__ bags, int nb, const int* __restrict__ recs_dev, int D, int C,
            const float* __restrict__ Q, const float* __restrict__ q_max, float* __restrict__ A,
            float* __restrict__ recs) {
  const int r = blockIdx.x;
  if (recs_dev && r >= *recs_dev) return;
  const int bag = bag_of(bags, nb, r, true);
  const sm90::BagDev bg = bags[bag];
  attend_rows<CT, J>(bg.X, D, Q + bg.row_off * kQ, bg.N, q_max + static_cast<size_t>(bag) * C * kQ, C,
                     A + bg.row_off * C, recs + static_cast<size_t>(r) * rec_floats(C, D), r - bg.rec_off, bg.nrec);
}

// grid = (C, ceil(D / 256), nb): bag z's records into its combined record out[z].
__global__ void __launch_bounds__(256, 1)   // (256, 1): as k_attend_gb, no spill
k_combine_rec_b(const sm90::BagDev* __restrict__ bags, int C, int D, const float* __restrict__ recs,
                float* __restrict__ out) {
  const size_t stride = rec_floats(C, D);
  combine_recs(recs + bags[blockIdx.z].rec_off * stride, bags[blockIdx.z].nrec, C, D, out + blockIdx.z * stride);
}

// grid = (any, nb): bag y's A, B [nb, C, D] and pred [nb, C].  models != NULL: Wf / bf of the entry's model.
// (256, 1): left to its default target ptxas spills the model's two weight pointers to stay within 32 registers.
__global__ void __launch_bounds__(256, 1)
k_finalize_gb(const sm90::BagDev* __restrict__ bags, const float* __restrict__ rec, int C, int D,
              const float* __restrict__ Wf, const float* __restrict__ bf, float* __restrict__ A, float* __restrict__ B,
              float* __restrict__ pred, const sm90::ModelDev* __restrict__ models) {
  const int bag = blockIdx.y;
  const sm90::BagDev bg = bags[bag];
  if (models) {
    const sm90::ModelDev& md = models[fold_pad_model(bg.pad_)];
    Wf = md.Wf;
    bf = md.bf;
  }
  finalize_bag(rec + bag * rec_floats(C, D), bg.N, C, D, Wf, bf, A + bg.row_off * C,
               B + static_cast<size_t>(bag) * C * D, pred + static_cast<size_t>(bag) * C, blockIdx.x, gridDim.x);
}

// ---- the value network's projection over the bag table (passing_v, dsmil.py:35-39) ----------------------------------
// V[packed rows, M] = relu(Xv_b W^T + b) over each bag's own rows, bit for bit what k_linear<ACT_RELU, false> gives the
// bag alone: every output is one fmaf chain over k = 0 .. K-1 in ascending order from 0 (zero padding past K adds
// exact zeros, as in linear_tile), then + b[m], then the ReLU.  Within that order the tile is the k_gemm_tn one: a
// 128 x 128 output block per CTA and 8 x 8 per thread (four 16-byte shared-memory loads per 64 FMAs, where
// linear_tile's 4 x 8 block needs three per 32), k-tiles of Xv and W double-buffered in shared memory, the next one
// fetched into registers while the current one is multiplied.
constexpr int VBM = 128, VBN = 128, VBK = 16;
static_assert(VBM == sm90::kTileM, "k_vproj_b takes one table tile per CTA");

// 8 consecutive k of one row from k on (zeros past K or for a dead row).
__device__ __forceinline__ void vproj_fetch(const float* __restrict__ row, bool live, bool vec, int k, int K,
                                            float (&r)[8]) {
  if (live && vec && k + 8 <= K) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(row + k));
    const float4 c = __ldg(reinterpret_cast<const float4*>(row + k + 4));
    r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w;
    r[4] = c.x; r[5] = c.y; r[6] = c.z; r[7] = c.w;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) r[i] = (live && k + i < K) ? __ldg(row + k + i) : 0.f;
  }
}

// grid = (tiles (tiles_dev: the live count of a capacity grid), ceil(M / VBN)); X of each entry is its value input.
__global__ void __launch_bounds__(256, 2)
k_vproj_b(const sm90::BagDev* __restrict__ bags, int nb, const int* __restrict__ tiles_dev, int K,
          const float* __restrict__ W, const float* __restrict__ b, int M, float* __restrict__ Y) {
  __shared__ __align__(16) float Xs[2][VBK][VBM + 4];
  __shared__ __align__(16) float Ws[2][VBK][VBN + 4];
  const int t = blockIdx.x;
  if (tiles_dev && t >= *tiles_dev) return;
  const sm90::BagDev bg = bags[bag_of(bags, nb, t, false)];
  const int64_t n0 = static_cast<int64_t>(t - bg.tile_off) * VBM;
  const int m0 = blockIdx.y * VBN;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  // loader: row lr of the X tile and of the W tile, k from lk (a warp stores 32 consecutive rows: no bank conflict)
  const int lr = tid & 127, lk = (tid >> 7) * 8;
  const bool xlive = n0 + lr < bg.N, wlive = m0 + lr < M;
  const float* xrow = bg.X + (xlive ? n0 + lr : 0) * K;
  const float* wrow = W + static_cast<int64_t>(wlive ? m0 + lr : 0) * K;
  const bool vec = (K % 4 == 0) && ((reinterpret_cast<uintptr_t>(bg.X) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(W) & 15) == 0);
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  float xr[8], wr[8];
  vproj_fetch(xrow, xlive, vec, lk, K, xr);
  vproj_fetch(wrow, wlive, vec, lk, K, wr);
#pragma unroll
  for (int i = 0; i < 8; ++i) { Xs[0][lk + i][lr] = xr[i]; Ws[0][lk + i][lr] = wr[i]; }
  __syncthreads();
  int buf = 0;
  for (int k0 = 0; k0 < K; k0 += VBK) {
    const bool more = k0 + VBK < K;
    if (more) {
      vproj_fetch(xrow, xlive, vec, k0 + VBK + lk, K, xr);
      vproj_fetch(wrow, wlive, vec, k0 + VBK + lk, K, wr);
    }
#pragma unroll
    for (int kk = 0; kk < VBK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&Xs[buf][kk][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&Xs[buf][kk][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Ws[buf][kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Ws[buf][kk][64 + tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (more) {
#pragma unroll
      for (int i = 0; i < 8; ++i) { Xs[buf ^ 1][lk + i][lr] = xr[i]; Ws[buf ^ 1][lk + i][lr] = wr[i]; }
    }
    __syncthreads();   // the next buffer is written; this one is read by everyone before it is refilled
    buf ^= 1;
  }
  float* Yb = Y + bg.row_off * M;
  const bool vst = (M % 4 == 0) && ((reinterpret_cast<uintptr_t>(Y) & 15) == 0);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t n = n0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (n >= bg.N) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int mb = m0 + h * 64 + tx * 4;
      float y[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) y[j] = mb + j < M ? fmaxf(acc[i][h * 4 + j] + __ldg(b + mb + j), 0.f) : 0.f;
      float* dst = Yb + n * M + mb;
      if (vst && mb + 3 < M) {
        *reinterpret_cast<float4*>(dst) = make_float4(y[0], y[1], y[2], y[3]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (mb + j < M) dst[j] = y[j];
      }
    }
  }
}

}  // namespace dsmil
