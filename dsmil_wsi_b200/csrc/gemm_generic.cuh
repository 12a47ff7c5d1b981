// Generic fp32 FFMA GEMM building blocks (any N, K, M; no alignment assumptions).
// Used by the generic forward for shapes the wgmma kernel does not take (D % 128 != 0, e.g. the
// classic-MIL 166/230 features of train_mil.py:127-141), by the V projection (dsmil.py:35-39) and
// by the backward GEMMs.  Deterministic: split reductions go through partial buffers summed in a
// fixed order, never float atomics.
#pragma once
#include "common.cuh"

namespace dsmil {

enum Act : int { ACT_NONE = 0, ACT_RELU = 1, ACT_TANH = 2, ACT_MASK_POS = 3 };

constexpr int LBM = 64, LBN = 128, LBK = 16;

// Y[N,M] (+)= act(X[N,K] * op(W) + b);  op(W)[k,m] = WT ? W[k*M+m] : W[m*K+k].
// ACT_MASK_POS: y = aux[n,m] > 0 ? y : 0  (ReLU backward through a saved activation).
// The body of CTA (blockIdx.x, blockIdx.y), whose rows start at n0.
template <int ACT, bool WT>
__device__ __forceinline__ void linear_tile(const float* __restrict__ X, int64_t N, int64_t n0, int K,
                                            const float* __restrict__ W, const float* __restrict__ b, int M,
                                            float* __restrict__ Y, const float* __restrict__ aux, int accumulate) {
  __shared__ __align__(16) float As[LBK][LBM + 4];
  __shared__ __align__(16) float Bs[LBK][LBN + 4];
  const int tid = threadIdx.x;
  const int ty = tid >> 4, tx = tid & 15;
  const int m0 = blockIdx.y * LBN;
  float acc[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  const int ar = tid >> 2, akq = (tid & 3) * 4;  // A loader: row, k-quad
  const bool a_vec = (K % 4 == 0) && ((reinterpret_cast<uintptr_t>(X) & 15) == 0);
  for (int k0 = 0; k0 < K; k0 += LBK) {
    {  // ---- A tile
      const int64_t n = n0 + ar;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (n < N) {
        const float* src = X + n * K + k0 + akq;
        if (a_vec && k0 + akq + 3 < K) {
          float4 t = __ldg(reinterpret_cast<const float4*>(src));
          v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
        } else {
#pragma unroll
          for (int i = 0; i < 4; ++i)
            if (k0 + akq + i < K) v[i] = __ldg(src + i);
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) As[akq + i][ar] = v[i];
    }
    if (!WT) {  // ---- B tile from W[m,k]
      const int m = tid >> 1, kq = (tid & 1) * 8;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float v = 0.f;
        if (m0 + m < M && k0 + kq + i < K) v = __ldg(W + static_cast<int64_t>(m0 + m) * K + k0 + kq + i);
        Bs[kq + i][m] = v;
      }
    } else {  // ---- B tile from W[k,m]
      const int kk = tid >> 4, mq = (tid & 15) * 8;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float v = 0.f;
        if (k0 + kk < K && m0 + mq + i < M) v = __ldg(W + static_cast<int64_t>(k0 + kk) * M + m0 + mq + i);
        Bs[kk][mq + i] = v;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < LBK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[kk][64 + tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t n = n0 + ty * 4 + i;
    if (n >= N) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int m = m0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
      if (m >= M) continue;
      float y = acc[i][j] + (b ? __ldg(b + m) : 0.f);
      if (ACT == ACT_RELU) y = fmaxf(y, 0.f);
      if (ACT == ACT_TANH) y = tanhf(y);
      if (ACT == ACT_MASK_POS) y = (__ldg(aux + n * M + m) > 0.f) ? y : 0.f;
      float* dst = Y + n * M + m;
      *dst = accumulate ? (*dst + y) : y;
    }
  }
}
template <int ACT, bool WT>
__global__ void __launch_bounds__(256)
k_linear(const float* __restrict__ X, int64_t N, int K, const float* __restrict__ W,
         const float* __restrict__ b, int M, float* __restrict__ Y, const float* __restrict__ aux,
         int accumulate, const long long* __restrict__ N_dev) {
  const int64_t n0 = static_cast<int64_t>(blockIdx.x) * LBM;
  if (N_dev) {               // the live row count of a capacity grid
    N = *N_dev;
    if (n0 >= N) return;
  }
  linear_tile<ACT, WT>(X, N, n0, K, W, b, M, Y, aux, accumulate);
}

// N_dev != NULL: N is the row capacity (the grid), *N_dev the live row count, read on the device.
template <int ACT, bool WT>
inline int launch_linear(const float* X, int64_t N, int K, const float* W, const float* b, int M, float* Y,
                         const float* aux, int accumulate, cudaStream_t st, const long long* N_dev = nullptr) {
  if (N <= 0) return 0;
  dim3 grid(ceil_div(N, LBM), ceil_div(M, LBN));
  k_linear<ACT, WT><<<grid, 256, 0, st>>>(X, N, K, W, b, M, Y, aux, accumulate, N_dev);
  DSMIL_LAUNCH_OK("k_linear");
  return 0;
}

// ---- out[M1,M2] = sum_n P[n,M1] * R[n,M2]  (reduction over rows; split over grid.z into partials)
// The weight-gradient GEMMs of the backward (gW1 = dz1^T X is 2 GFLOP at N = 15 000).  128 x 128 output tile per CTA,
// 8 x 8 per thread: 64 FMAs per four 16-byte shared-memory loads, so the FMA pipe, not the LSU, is the limiter (the
// former 64 x 64 / 4 x 4 tile was shared-memory-bound at half the FMA rate); the next k-tile is fetched into registers
// while the current one is multiplied.
// gemm_tn_tile: the CTA's tile (blockIdx.y, blockIdx.x) of out[M1,M2] = sum over rows [0, ne) of P[n,M1] * R[n,M2].
constexpr int TBM = 128, TBK = 16;
__device__ __forceinline__ void gemm_tn_tile(const float* __restrict__ P, int M1, const float* __restrict__ R, int M2,
                                             int64_t ne, float* __restrict__ out) {
  __shared__ __align__(16) float Ps[TBK][TBM + 4];
  __shared__ __align__(16) float Rs[TBK][TBM + 4];
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int a0 = blockIdx.y * TBM, b0 = blockIdx.x * TBM;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  // loader role: k-row (tid >> 4) of the tile, columns (tid & 15) * 4 .. + 3 and + 64
  const int ln = tid >> 4, lq = (tid & 15) * 4;
  // float4 rows only when every row is 16-byte aligned (a bag may be a view at any float offset)
  const bool pvec = (M1 & 3) == 0 && (reinterpret_cast<uintptr_t>(P) & 15) == 0;
  const bool rvec = (M2 & 3) == 0 && (reinterpret_cast<uintptr_t>(R) & 15) == 0;
  float4 pf[2], rf[2];
  auto fetch = [&](int64_t n0) {
    const int64_t n = n0 + ln;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int ca = a0 + lq + 64 * h, cb = b0 + lq + 64 * h;
      float4 pv = make_float4(0.f, 0.f, 0.f, 0.f), rv = pv;
      if (n < ne) {
        const float* pp = P + n * M1 + ca;
        const float* rp = R + n * M2 + cb;
        if (pvec && ca + 3 < M1) pv = __ldg(reinterpret_cast<const float4*>(pp));
        else {
          if (ca < M1) pv.x = __ldg(pp);
          if (ca + 1 < M1) pv.y = __ldg(pp + 1);
          if (ca + 2 < M1) pv.z = __ldg(pp + 2);
          if (ca + 3 < M1) pv.w = __ldg(pp + 3);
        }
        if (rvec && cb + 3 < M2) rv = __ldg(reinterpret_cast<const float4*>(rp));
        else {
          if (cb < M2) rv.x = __ldg(rp);
          if (cb + 1 < M2) rv.y = __ldg(rp + 1);
          if (cb + 2 < M2) rv.z = __ldg(rp + 2);
          if (cb + 3 < M2) rv.w = __ldg(rp + 3);
        }
      }
      pf[h] = pv;
      rf[h] = rv;
    }
  };
  if (ne > 0) fetch(0);
  for (int64_t n0 = 0; n0 < ne; n0 += TBK) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      *reinterpret_cast<float4*>(&Ps[ln][lq + 64 * h]) = pf[h];
      *reinterpret_cast<float4*>(&Rs[ln][lq + 64 * h]) = rf[h];
    }
    __syncthreads();
    if (n0 + TBK < ne) fetch(n0 + TBK);
#pragma unroll
    for (int kk = 0; kk < TBK; ++kk) {
      const float4 a_lo = *reinterpret_cast<const float4*>(&Ps[kk][ty * 4]);
      const float4 a_hi = *reinterpret_cast<const float4*>(&Ps[kk][ty * 4 + 64]);
      const float4 b_lo = *reinterpret_cast<const float4*>(&Rs[kk][tx * 4]);
      const float4 b_hi = *reinterpret_cast<const float4*>(&Rs[kk][tx * 4 + 64]);
      const float av[8] = {a_lo.x, a_lo.y, a_lo.z, a_lo.w, a_hi.x, a_hi.y, a_hi.z, a_hi.w};
      const float bv[8] = {b_lo.x, b_lo.y, b_lo.z, b_lo.w, b_hi.x, b_hi.y, b_hi.z, b_hi.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int a = a0 + ty * 4 + (i & 3) + 64 * (i >> 2);
    if (a >= M1) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int b = b0 + tx * 4 + (j & 3) + 64 * (j >> 2);
      if (b < M2) out[static_cast<int64_t>(a) * M2 + b] = acc[i][j];
    }
  }
}
// A row split decided on the device (capacity grids, bag_plan.cuh): the live rows N, rows per split and splits S.
struct RowSplit {
  long long N;
  long long rps;
  int S;
  int pad_;
};

__global__ void __launch_bounds__(256, 2)
k_gemm_tn(const float* __restrict__ P, int M1, const float* __restrict__ R, int M2, int64_t N,
          int64_t rows_per_split, float* __restrict__ part, const RowSplit* __restrict__ dyn) {
  if (dyn) {
    if (static_cast<int>(blockIdx.z) >= dyn->S) return;
    N = dyn->N;
    rows_per_split = dyn->rps;
  }
  const int64_t nb = static_cast<int64_t>(blockIdx.z) * rows_per_split;
  gemm_tn_tile(P + nb * M1, M1, R + nb * M2, M2, min(N, nb + rows_per_split) - nb,
               part + static_cast<int64_t>(blockIdx.z) * M1 * M2);
}

// The same product for a handful of left columns (M1 <= 4: the per-class gradients gWi = d_classes^T X and
// dq_max = dL^T Q): 2 * M1 FLOP per element of R, i.e. a pure stream over R.  Thread = one float4 column group of R,
// 256 / (M2 / 4) rows in flight per CTA; partial per CTA, combined in a fixed order.
constexpr int kGemvMaxM1 = 4;
// gemv_tn_rows: out[M1,M2] = sum over rows [0, ne) of P[n,M1] * R[n,M2], by one CTA.
template <int M1>
__device__ __forceinline__ void gemv_tn_rows(const float* __restrict__ P, const float* __restrict__ R, int M2,
                                             int64_t ne, float* __restrict__ out) {
  __shared__ float s_acc[256][4 * M1 + 1];
  const int G = M2 >> 2;                    // float4 groups per row (<= 256)
  const int rpi = 256 / G;                  // rows per iteration
  const int g = threadIdx.x % G, ro = threadIdx.x / G;
  float acc[M1][4];
#pragma unroll
  for (int c = 0; c < M1; ++c) acc[c][0] = acc[c][1] = acc[c][2] = acc[c][3] = 0.f;
  if (ro < rpi) {
#pragma unroll 4
    for (int64_t n = ro; n < ne; n += rpi) {
      const float4 r = __ldg(reinterpret_cast<const float4*>(R + n * M2) + g);
#pragma unroll
      for (int c = 0; c < M1; ++c) {
        const float pv = __ldg(P + n * M1 + c);
        acc[c][0] = fmaf(pv, r.x, acc[c][0]); acc[c][1] = fmaf(pv, r.y, acc[c][1]);
        acc[c][2] = fmaf(pv, r.z, acc[c][2]); acc[c][3] = fmaf(pv, r.w, acc[c][3]);
      }
    }
  }
#pragma unroll
  for (int c = 0; c < M1; ++c)
#pragma unroll
    for (int q = 0; q < 4; ++q) s_acc[threadIdx.x][4 * c + q] = acc[c][q];
  __syncthreads();
  // thread (g, ro == 0) adds the other row groups in order, then writes its 4 * M1 values
  if (ro == 0) {
    for (int r2 = 1; r2 < rpi; ++r2)
#pragma unroll
      for (int c = 0; c < M1; ++c)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[c][q] += s_acc[r2 * G + g][4 * c + q];
#pragma unroll
    for (int c = 0; c < M1; ++c)
      *reinterpret_cast<float4*>(out + static_cast<int64_t>(c) * M2 + 4 * g) = make_float4(acc[c][0], acc[c][1], acc[c][2], acc[c][3]);
  }
}
template <int M1>
__global__ void __launch_bounds__(256)
k_gemv_tn(const float* __restrict__ P, const float* __restrict__ R, int M2, int64_t N, int64_t rows_per_split,
          float* __restrict__ part) {
  const int64_t nb = static_cast<int64_t>(blockIdx.x) * rows_per_split;
  gemv_tn_rows<M1>(P + nb * M1, R + nb * M2, M2, min(N, nb + rows_per_split) - nb,
                   part + static_cast<int64_t>(blockIdx.x) * M1 * M2);
}

// part[z][M] = sum over the z-th row chunk of P[n, m]
__global__ void __launch_bounds__(256)
k_colsum(const float* __restrict__ P, int M, int64_t N, int64_t rows_per_split, float* __restrict__ part,
         const RowSplit* __restrict__ dyn) {
  if (dyn) {
    if (static_cast<int>(blockIdx.x) >= dyn->S) return;
    N = dyn->N;
    rows_per_split = dyn->rps;
  }
  const int64_t nb = static_cast<int64_t>(blockIdx.x) * rows_per_split;
  const int64_t ne = min(N, nb + rows_per_split);
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    float s = 0.f;
    for (int64_t n = nb; n < ne; ++n) s += __ldg(P + n * M + m);
    part[static_cast<int64_t>(blockIdx.x) * M + m] = s;
  }
}

// out[i] = sum_z part[z][i]  (fixed order: warp w of the CTA adds z = w, w + 8, ... with four independent running sums,
// the eight warp sums are then added in warp order).  32 outputs per CTA, so a short vector (a bias gradient: 128
// values from 235 partials) is no longer one CTA walking 235 dependent steps.
__device__ __forceinline__ void sum_partials(const float* __restrict__ part, int S, int64_t L, float* __restrict__ out) {
  __shared__ float s_w[8][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * 32 + lane;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  if (i < L) {
    int z = w;
    for (; z + 24 < S; z += 32) {
      s0 += part[static_cast<int64_t>(z) * L + i];
      s1 += part[static_cast<int64_t>(z + 8) * L + i];
      s2 += part[static_cast<int64_t>(z + 16) * L + i];
      s3 += part[static_cast<int64_t>(z + 24) * L + i];
    }
    for (; z < S; z += 8) s0 += part[static_cast<int64_t>(z) * L + i];
  }
  s_w[w][lane] = (s0 + s1) + (s2 + s3);
  __syncthreads();
  if (w == 0 && i < L)
    out[i] = ((s_w[0][lane] + s_w[1][lane]) + (s_w[2][lane] + s_w[3][lane])) +
             ((s_w[4][lane] + s_w[5][lane]) + (s_w[6][lane] + s_w[7][lane]));
}
__global__ void __launch_bounds__(256)
k_sum_partials(const float* __restrict__ part, int S, int64_t L, float* __restrict__ out, const int* __restrict__ S_dev) {
  if (S_dev) S = *S_dev;
  sum_partials(part, S, L, out);
}
inline int launch_sum_partials(const float* part, int S, int64_t L, float* out, cudaStream_t st,
                               const int* S_dev = nullptr) {
  k_sum_partials<<<static_cast<unsigned>(ceil_div(L, 32)), 256, 0, st>>>(part, S, L, out, S_dev);
  DSMIL_LAUNCH_OK("k_sum_partials");
  return 0;
}

__host__ __device__ inline bool tn_use_gemv(int M1, int M2) { return M1 <= kGemvMaxM1 && (M2 & 3) == 0 && (M2 >> 2) <= 256; }
__host__ __device__ inline int tn_splits(int M1, int M2, int64_t N) {
  int s, maxs;
  if (tn_use_gemv(M1, M2)) {
    s = kSplits;
    maxs = ceil_div(N, 64);
  } else {
    const int tiles = ceil_div(M1, TBM) * ceil_div(M2, TBM);
    s = kSplits / (tiles > 0 ? tiles : 1);
    maxs = ceil_div(N, 128);
  }
  if (s > maxs) s = maxs;
  if (s < 1) s = 1;
  return s;
}
inline size_t tn_partial_floats(int M1, int M2, int64_t N) {
  return static_cast<size_t>(tn_splits(M1, M2, N)) * M1 * M2;
}
// out[M1,M2] = P^T R, via partials in `part` (>= tn_partial_floats floats).  dyn != NULL: N is the row capacity and
// the split is the device's (the tile form only: M1 > kGemvMaxM1).
inline int launch_gemm_tn(const float* P, int M1, const float* R, int M2, int64_t N, float* part, float* out,
                          cudaStream_t st, const RowSplit* dyn = nullptr) {
  if (dyn) {
    if (tn_use_gemv(M1, M2)) {
      set_error("launch_gemm_tn: a device-side split needs the tile form");
      return DSMIL_ERR_ARG;
    }
    const int S = tn_splits(M1, M2, N);
    k_gemm_tn<<<dim3(ceil_div(M2, TBM), ceil_div(M1, TBM), S), 256, 0, st>>>(P, M1, R, M2, N, 0, part, dyn);
    DSMIL_LAUNCH_OK("k_gemm_tn");
    return launch_sum_partials(part, S, static_cast<int64_t>(M1) * M2, out, st, &dyn->S);
  }
  if (N <= 0) {
    DSMIL_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(float) * M1 * M2, st));
    return 0;
  }
  const int S = tn_splits(M1, M2, N);
  const int64_t L = static_cast<int64_t>(M1) * M2;
  if (tn_use_gemv(M1, M2) && (reinterpret_cast<uintptr_t>(R) & 15) == 0 && (reinterpret_cast<uintptr_t>(part) & 15) == 0) {
    const int64_t rps = (N + S - 1) / S;
    switch (M1) {
      case 1: k_gemv_tn<1><<<S, 256, 0, st>>>(P, R, M2, N, rps, part); break;
      case 2: k_gemv_tn<2><<<S, 256, 0, st>>>(P, R, M2, N, rps, part); break;
      case 3: k_gemv_tn<3><<<S, 256, 0, st>>>(P, R, M2, N, rps, part); break;
      default: k_gemv_tn<4><<<S, 256, 0, st>>>(P, R, M2, N, rps, part); break;
    }
    DSMIL_LAUNCH_OK("k_gemv_tn");
    return launch_sum_partials(part, S, L, out, st);
  }
  int Sg = S;
  if (tn_use_gemv(M1, M2)) {                                 // unaligned operand: the tile kernel, within the same budget
    const int tiles = ceil_div(M1, TBM) * ceil_div(M2, TBM);
    Sg = std::max(1, std::min(S, kSplits / tiles));
  }
  int64_t rps = (N + Sg - 1) / Sg;
  rps = (rps + TBK - 1) / TBK * TBK;
  dim3 grid(ceil_div(M2, TBM), ceil_div(M1, TBM), Sg);
  k_gemm_tn<<<grid, 256, 0, st>>>(P, M1, R, M2, N, rps, part, nullptr);
  DSMIL_LAUNCH_OK("k_gemm_tn");
  return launch_sum_partials(part, Sg, L, out, st);
}
__host__ __device__ inline int colsum_splits(int64_t N) {
  int s = ceil_div(N, 64);
  return s > kSplits ? kSplits : (s < 1 ? 1 : s);
}
// dyn != NULL: N is the row capacity and the split is the device's.
inline int launch_colsum(const float* P, int M, int64_t N, float* part, float* out, cudaStream_t st,
                         const RowSplit* dyn = nullptr) {
  if (dyn) {
    const int S = colsum_splits(N);
    k_colsum<<<S, 256, 0, st>>>(P, M, N, 0, part, dyn);
    DSMIL_LAUNCH_OK("k_colsum");
    return launch_sum_partials(part, S, M, out, st, &dyn->S);
  }
  if (N <= 0) {
    DSMIL_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(float) * M, st));
    return 0;
  }
  const int S = colsum_splits(N);
  const int64_t rps = (N + S - 1) / S;
  k_colsum<<<S, 256, 0, st>>>(P, M, N, rps, part, nullptr);
  DSMIL_LAUNCH_OK("k_colsum");
  return launch_sum_partials(part, S, M, out, st);
}

}  // namespace dsmil
