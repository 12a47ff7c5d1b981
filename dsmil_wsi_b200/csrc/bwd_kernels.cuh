// Backward kernels (reverse of dsmil.py:46-62 as autograd performs it; algebra in SURVEY A.2).
#pragma once
#include "common.cuh"

namespace dsmil {

// dB[k',d] = sum_k Wf[k,k',d] * dp[k] (+ dB_up);  gWf[k,k',d] = dp[k] * B[k',d];  gbf = dp.
__global__ void __launch_bounds__(256)
k_bwd_bag(const float* __restrict__ Wf, const float* __restrict__ B, const float* __restrict__ dp,
          const float* __restrict__ dB_up, int C, int Dv, float* __restrict__ dB, float* __restrict__ gWf,
          float* __restrict__ gbf) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // over C*Dv  (k', d)
  if (i < C && gbf) gbf[i] = dp ? dp[i] : 0.f;
  if (i >= C * Dv) return;
  float acc = dB_up ? dB_up[i] : 0.f;
  const float b = B[i];
  for (int k = 0; k < C; ++k) {
    const float g = dp ? dp[k] : 0.f;
    acc = fmaf(__ldg(Wf + static_cast<size_t>(k) * C * Dv + i), g, acc);
    if (gWf) gWf[static_cast<size_t>(k) * C * Dv + i] = g * b;
  }
  dB[i] = acc;
}

// out[n,k] = sum_d V[n,d] * Wt[k,d] (+ add[n,k]);  one warp per row.
__global__ void __launch_bounds__(256)
k_rowdot(const float* __restrict__ V, int64_t N, int Dv, const float* __restrict__ Wt, int C,
         const float* __restrict__ add, float* __restrict__ out) {
  extern __shared__ __align__(16) float sW[];  // [C*Dv]
  for (int i = threadIdx.x; i < C * Dv; i += blockDim.x) sW[i] = Wt[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * 8;
  for (int64_t n = static_cast<int64_t>(blockIdx.x) * 8 + warp; n < N; n += stride) {
    float acc[kMaxC];
#pragma unroll
    for (int k = 0; k < kMaxC; ++k) acc[k] = 0.f;
    const float* row = V + n * Dv;
    for (int j = lane; j < Dv; j += 32) {
      const float x = __ldg(row + j);
#pragma unroll
      for (int k = 0; k < kMaxC; ++k)
        if (k < C) acc[k] = fmaf(x, sW[k * Dv + j], acc[k]);
    }
#pragma unroll
    for (int k = 0; k < kMaxC; ++k)
      if (k < C) {
        const float v = warp_sum(acc[k]);
        if (lane == 0) out[n * C + k] = v + (add ? add[n * C + k] : 0.f);
      }
  }
}

// part[b][k] = sum over this block's rows of A[n,k] * dA[n,k]
__global__ void __launch_bounds__(256)
k_bwd_t_partial(const float* __restrict__ A, const float* __restrict__ dA, int64_t N, int C,
                float* __restrict__ part) {
  __shared__ float red[8][kMaxC];
  float acc[kMaxC];
#pragma unroll
  for (int k = 0; k < kMaxC; ++k) acc[k] = 0.f;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t n = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; n < N; n += stride) {
#pragma unroll
    for (int k = 0; k < kMaxC; ++k)
      if (k < C) acc[k] = fmaf(A[n * C + k], dA[n * C + k], acc[k]);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < kMaxC; ++k) {
    const float v = warp_sum(acc[k]);
    if (lane == 0) red[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < C) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
    part[blockIdx.x * C + threadIdx.x] = s;
  }
}

// dL[n,k] = A[n,k] * (dA[n,k] - t[k]) / sqrt(128f), in place over dA;  t = sum_b part[b]
__global__ void __launch_bounds__(256)
k_bwd_dL(const float* __restrict__ A, float* __restrict__ dA, int64_t N, int C,
         const float* __restrict__ part, int P) {
  __shared__ float t[kMaxC];
  if (threadIdx.x < C) {
    float s = 0.f;
    for (int b = 0; b < P; ++b) s += part[b * C + threadIdx.x];
    t[threadIdx.x] = s;
  }
  __syncthreads();
  const int64_t total = N * C;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int k = static_cast<int>(i % C);
    dA[i] = __fdiv_rn(A[i] * (dA[i] - t[k]), kScale);
  }
}

// dz[n,j] = (sum_k dL[n,k]*qmax[k,j] + sum_k [n==idx_k] dqm[k,j]) * (tanh ? 1 - Q[n,j]^2 : 1), idx_k = crit[k] -
// row_offset: the dqm share goes to the row whose GLOBAL number n + row_offset is crit[k].  qmax is the forward's
// exchanged q_max when the critical row may live on another rank; NULL reads it from the local rows, Q[idx_k].
__global__ void __launch_bounds__(256)
k_bwd_dq(const float* __restrict__ dL, const float* __restrict__ Q, const float* __restrict__ qmax,
         const float* __restrict__ dqm, const int64_t* __restrict__ crit, int64_t N, int64_t row_offset, int C,
         int through_tanh, float* __restrict__ dz) {
  __shared__ float sq[kMaxC][kQ];
  __shared__ float sd[kMaxC][kQ];
  __shared__ int64_t sidx[kMaxC];
  for (int i = threadIdx.x; i < C * kQ; i += blockDim.x) {
    const int k = i / kQ, j = i % kQ;
    sq[k][j] = qmax ? qmax[i] : Q[(crit[k] - row_offset) * kQ + j];
    sd[k][j] = dqm[i];
  }
  if (threadIdx.x < C) sidx[threadIdx.x] = crit[threadIdx.x] - row_offset;
  __syncthreads();
  const int64_t total = N * kQ;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t n = i / kQ;
    const int j = static_cast<int>(i % kQ);
    float g = 0.f;
    for (int k = 0; k < C; ++k) {
      g = fmaf(dL[n * C + k], sq[k][j], g);
      if (n == sidx[k]) g += sd[k][j];
    }
    if (through_tanh) {
      const float q = Q[i];
      g *= (1.f - q * q);
    }
    dz[i] = g;
  }
}

// gX[n,d] (+)= sum_k dcls[n,k]*Wi[k,d] + sum_k A[n,k]*dB[k,d]   (either term optional)
__global__ void __launch_bounds__(256)
k_bwd_dx_extra(const float* __restrict__ dcls, const float* __restrict__ Wi, const float* __restrict__ A,
               const float* __restrict__ dB, int64_t N, int C, int D, int accumulate, float* __restrict__ gX) {
  const int64_t total = N * D;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t n = i / D;
    const int d = static_cast<int>(i % D);
    float g = accumulate ? gX[i] : 0.f;
    for (int k = 0; k < C; ++k) {
      if (dcls) g = fmaf(dcls[n * C + k], __ldg(Wi + k * D + d), g);
      if (A) g = fmaf(A[n * C + k], __ldg(dB + k * D + d), g);
    }
    gX[i] = g;
  }
}

// dzv[n,d] = (sum_k A[n,k]*dB[k,d]) * [V[n,d] > 0]
__global__ void __launch_bounds__(256)
k_bwd_dzv(const float* __restrict__ A, const float* __restrict__ dB, const float* __restrict__ V, int64_t N,
          int C, int D, float* __restrict__ dzv) {
  const int64_t total = N * D;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t n = i / D;
    const int d = static_cast<int>(i % D);
    float g = 0.f;
    for (int k = 0; k < C; ++k) g = fmaf(A[n * C + k], __ldg(dB + k * D + d), g);
    dzv[i] = V[i] > 0.f ? g : 0.f;
  }
}

// y[i] += t[i] * (mask ? mask[i] : 1)
__global__ void __launch_bounds__(256)
k_axpy_mask(const float* __restrict__ t, const float* __restrict__ mask, int64_t total, float* __restrict__ y) {
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride)
    y[i] += mask ? t[i] * mask[i] : t[i];
}

}  // namespace dsmil
