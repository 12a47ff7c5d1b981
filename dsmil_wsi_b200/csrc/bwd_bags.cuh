// Backward of the batched forward (dsmil_backward_bags): the reverse of dsmil.py:46-62 for nb bags at once, identity
// v only.  Every kernel walks the forward's bag table (sm90::BagDev: X pointer, N, row_off); per-row buffers (classes,
// A, Q, H1 and their gradients) are packed in bag order, [sum N, *].  Parameter gradients are sums over the bags.
// Split sums go through partial buffers whose count depends on the shapes only (never on the SM count) and are added
// in a fixed order: no float atomics, so two runs give the same bits on any H100.  The row-sharded batch
// (dsmil_shard_backward_bags_phase1/2/3) runs the same kernels on each rank's rows, with the all-reduced t and
// dq_max and the merged q_max passed in.
#pragma once
#include "common.cuh"
#include "gemm_generic.cuh"
#include "fwd_sm90.cuh"
#include "bag_plan.cuh"

namespace dsmil {

// The dev calls launch the per-bag kernels on a capacity grid: G_dev points at the live CTAs per bag (the planner's),
// and the CTAs past it return at once.  With G_dev == NULL, G is gridDim.x.

// Bag classifier for all bags (dsmil.py:59-61):  dB[b] = Wf^T dp[b] (+ dB_up[b]);  gWf[k] = sum_b dp[b,k] B[b];
// gbf = sum_b dp[b].  The sums over b run in bag order.
__global__ void __launch_bounds__(256)
k_bwd_bag_b(const float* __restrict__ Wf, const float* __restrict__ B, const float* __restrict__ dp,
            const float* __restrict__ dB_up, int nb, int C, int Dv, float* __restrict__ dB, float* __restrict__ gWf,
            float* __restrict__ gbf) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // over C*Dv  (k', d)
  const size_t CD = static_cast<size_t>(C) * Dv;
  if (i < C && gbf) {
    float s = 0.f;
    if (dp)
      for (int b = 0; b < nb; ++b) s += dp[b * C + i];
    gbf[i] = s;
  }
  if (i >= static_cast<int>(CD)) return;
  for (int b = 0; b < nb; ++b) {
    float acc = dB_up ? dB_up[b * CD + i] : 0.f;
    if (dp)
      for (int k = 0; k < C; ++k) acc = fmaf(__ldg(Wf + k * CD + i), dp[b * C + k], acc);
    dB[b * CD + i] = acc;
  }
  if (gWf)
    for (int k = 0; k < C; ++k) {
      float s = 0.f;
      if (dp)
        for (int b = 0; b < nb; ++b) s = fmaf(dp[b * C + k], B[b * CD + i], s);
      gWf[k * CD + i] = s;
    }
}

// First pass over X.  CTA (x, b) walks the rows n = x*8 + warp, step gridDim.x*8, of bag b:
// dA[n,k] = X[n] . dB[b,k] (+ add[n,k]), one warp per row (scalar loads: any D, any alignment); and the CTA's share of
// t_b[k] = sum_n A[n,k] dA[n,k] goes to tpart[b][x][k].
__global__ void __launch_bounds__(256)
k_bwd_rowdot_b(const sm90::BagDev* __restrict__ bags, int D, const float* __restrict__ dB, int C,
               const float* __restrict__ A, const float* __restrict__ add, float* __restrict__ dA,
               float* __restrict__ tpart, const int* __restrict__ G_dev) {
  extern __shared__ __align__(16) float sW[];  // [C*D]: dB of this CTA's bag
  __shared__ float red[8][kMaxC];
  const int G = G_dev ? *G_dev : static_cast<int>(gridDim.x);
  if (static_cast<int>(blockIdx.x) >= G) return;
  const int b = blockIdx.y;
  const sm90::BagDev bg = bags[b];
  const float* W = dB + static_cast<size_t>(b) * C * D;
  for (int i = threadIdx.x; i < C * D; i += blockDim.x) sW[i] = W[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float tacc[kMaxC];
#pragma unroll
  for (int k = 0; k < kMaxC; ++k) tacc[k] = 0.f;
  const int64_t stride = static_cast<int64_t>(G) * 8;
  for (int64_t n = static_cast<int64_t>(blockIdx.x) * 8 + warp; n < bg.N; n += stride) {
    float acc[kMaxC];
#pragma unroll
    for (int k = 0; k < kMaxC; ++k) acc[k] = 0.f;
    const float* row = bg.X + n * D;
    for (int j = lane; j < D; j += 32) {
      const float x = __ldg(row + j);
#pragma unroll
      for (int k = 0; k < kMaxC; ++k)
        if (k < C) acc[k] = fmaf(x, sW[k * D + j], acc[k]);
    }
    const int64_t r = bg.row_off + n;
#pragma unroll
    for (int k = 0; k < kMaxC; ++k)
      if (k < C) {
        const float v = warp_sum(acc[k]) + (add ? add[r * C + k] : 0.f);   // every lane holds the row's value
        if (lane == 0) dA[r * C + k] = v;
        tacc[k] = fmaf(A[r * C + k], v, tacc[k]);
      }
  }
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < kMaxC; ++k) red[warp][k] = tacc[k];
  __syncthreads();
  if (threadIdx.x < C) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
    tpart[(static_cast<size_t>(b) * G + blockIdx.x) * C + threadIdx.x] = s;
  }
}

// Softmax-over-instances backward (dsmil.py:55-57), segmented per bag.  CTA (x, b), t_b = sum_{x' < P} tpart[b][x']
// (P partials per bag: the first pass's per-CTA shares, or P = 1 for a t that is already summed, e.g. all-reduced
// over the ranks of a row-sharded batch):
// dL[n,k] = A[n,k] (dA[n,k] - t_b[k]) / sqrt(128) for rows n = 2x + h, step 2*gridDim.x, of bag b, and the CTA's share
// of dq_max_b = dL_b^T Q_b, [C,128], in dpart[b][x].  G_dev != NULL (one device, first-pass partials): G and P are
// both *G_dev.
__global__ void __launch_bounds__(256)
k_bwd_dL_b(const sm90::BagDev* __restrict__ bags, int C, const float* __restrict__ A, const float* __restrict__ dA,
           const float* __restrict__ tpart, int P, const float* __restrict__ Q, float* __restrict__ dL,
           float* __restrict__ dpart, const int* __restrict__ G_dev) {
  __shared__ float t[kMaxC];
  __shared__ float red[kMaxC][kQ];
  const int b = blockIdx.y, G = G_dev ? *G_dev : static_cast<int>(gridDim.x);
  if (static_cast<int>(blockIdx.x) >= G) return;
  if (G_dev) P = G;
  if (threadIdx.x < C) {
    float s = 0.f;
    for (int x = 0; x < P; ++x) s += tpart[(static_cast<size_t>(b) * P + x) * C + threadIdx.x];
    t[threadIdx.x] = s;
  }
  __syncthreads();
  const sm90::BagDev bg = bags[b];
  const int j = threadIdx.x & (kQ - 1), h = threadIdx.x >> 7;
  float acc[kMaxC];
#pragma unroll
  for (int k = 0; k < kMaxC; ++k) acc[k] = 0.f;
  for (int64_t n = static_cast<int64_t>(blockIdx.x) * 2 + h; n < bg.N; n += 2 * static_cast<int64_t>(G)) {
    const int64_t r = bg.row_off + n;
    const float q = __ldg(Q + r * kQ + j);
#pragma unroll
    for (int k = 0; k < kMaxC; ++k)
      if (k < C) {
        const float l = __fdiv_rn(A[r * C + k] * (dA[r * C + k] - t[k]), kScale);
        acc[k] = fmaf(l, q, acc[k]);
        if (j == 0) dL[r * C + k] = l;
      }
  }
  if (h == 1)
#pragma unroll
    for (int k = 0; k < kMaxC; ++k)
      if (k < C) red[k][j] = acc[k];
  __syncthreads();
  if (h == 0)
#pragma unroll
    for (int k = 0; k < kMaxC; ++k)
      if (k < C) dpart[((static_cast<size_t>(b) * G + blockIdx.x) * C + k) * kQ + j] = acc[k] + red[k][j];
}

// dqm[b][i] = sum_{x < P} dpart[b][x][i], i < L (in x order); P = *P_dev when P_dev != NULL
__global__ void __launch_bounds__(256)
k_sum_segments(const float* __restrict__ part, int P, int L, float* __restrict__ out, const int* __restrict__ P_dev) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L) return;
  if (P_dev) P = *P_dev;
  float s = 0.f;
  for (int x = 0; x < P; ++x) s += part[(static_cast<size_t>(b) * P + x) * L + i];
  out[static_cast<size_t>(b) * L + i] = s;
}

// dQ rows of bag b (dsmil.py:53-55), then tanh' when q is nonlinear:
// dz[n,j] = (sum_k dL[n,k] q_max_b[k,j] + sum_k [n == idx_bk] dqm[b,k,j]) * (1 - Q[n,j]^2).
// qmax == NULL, row_offsets == NULL: the critical rows are local, idx_bk = crit[b,k] (the row within the bag) and
// q_max_b[k] = Q[row_off + idx_bk].  A row-sharded batch passes the merged qmax [nb,C,128] and each bag's first global
// row row_offsets[b]: crit holds global rows, idx_bk = crit[b,k] - row_offsets[b] (no local row matches when the
// critical row lives on another rank), and q_max_b comes from qmax.
__global__ void __launch_bounds__(256)
k_bwd_dq_b(const sm90::BagDev* __restrict__ bags, int C, const float* __restrict__ dL, const float* __restrict__ Q,
           const float* __restrict__ qmax, const float* __restrict__ dqm, const int64_t* __restrict__ crit,
           const long long* __restrict__ row_offsets, int through_tanh, float* __restrict__ dz) {
  __shared__ float sq[kMaxC][kQ];
  __shared__ float sd[kMaxC][kQ];
  __shared__ int64_t sidx[kMaxC];
  const int b = blockIdx.y;
  const sm90::BagDev bg = bags[b];
  const int64_t off = row_offsets ? row_offsets[b] : 0;
  for (int i = threadIdx.x; i < C * kQ; i += blockDim.x) {
    const int k = i / kQ, j = i % kQ;
    sq[k][j] = qmax ? qmax[static_cast<size_t>(b) * C * kQ + i] : Q[(bg.row_off + crit[b * C + k]) * kQ + j];
    sd[k][j] = dqm[static_cast<size_t>(b) * C * kQ + i];
  }
  if (threadIdx.x < C) sidx[threadIdx.x] = crit[b * C + threadIdx.x] - off;
  __syncthreads();
  const int64_t total = bg.N * kQ;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t n = i / kQ;
    const int j = static_cast<int>(i % kQ);
    const int64_t r = bg.row_off + n;
    float g = 0.f;
    for (int k = 0; k < C; ++k) {
      g = fmaf(dL[r * C + k], sq[k][j], g);
      if (n == sidx[k]) g += sd[k][j];
    }
    if (through_tanh) {
      const float q = Q[r * kQ + j];
      g *= (1.f - q * q);
    }
    dz[r * kQ + j] = g;
  }
}

// gX[n,d] += sum_k dcls[n,k] Wi[k,d] + sum_k A[n,k] dB[b,k,d] over the rows of bag b (dcls may be NULL)
__global__ void __launch_bounds__(256)
k_bwd_dx_extra_b(const sm90::BagDev* __restrict__ bags, const float* __restrict__ dcls, const float* __restrict__ Wi,
                 const float* __restrict__ A, const float* __restrict__ dB, int C, int D, float* __restrict__ gX) {
  const int b = blockIdx.y;
  const sm90::BagDev bg = bags[b];
  const float* dBb = dB + static_cast<size_t>(b) * C * D;
  const int64_t total = bg.N * D;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t r = bg.row_off + i / D;
    const int d = static_cast<int>(i % D);
    float g = gX[r * D + d];
    for (int k = 0; k < C; ++k) {
      if (dcls) g = fmaf(dcls[r * C + k], __ldg(Wi + k * D + d), g);
      g = fmaf(A[r * C + k], __ldg(dBb + k * D + d), g);
    }
    gX[r * D + d] = g;
  }
}

// Ragged out = P^T X: chunk z of the table is one row range of one bag; its partial goes to part[z].  nz_dev != NULL:
// the live chunk count of a capacity grid.
__global__ void __launch_bounds__(256, 2)
k_gemm_tn_rag(const float* __restrict__ P, int M1, int M2, const TnChunk* __restrict__ chunks,
              float* __restrict__ part, const int* __restrict__ nz_dev) {
  if (nz_dev && static_cast<int>(blockIdx.z) >= *nz_dev) return;
  const TnChunk c = chunks[blockIdx.z];
  gemm_tn_tile(P + c.prow * M1, M1, c.R, M2, c.rows, part + static_cast<int64_t>(blockIdx.z) * M1 * M2);
}
template <int M1>
__global__ void __launch_bounds__(256)
k_gemv_tn_rag(const float* __restrict__ P, int M2, const TnChunk* __restrict__ chunks, float* __restrict__ part,
              const int* __restrict__ nz_dev) {
  if (nz_dev && static_cast<int>(blockIdx.x) >= *nz_dev) return;
  const TnChunk c = chunks[blockIdx.x];
  gemv_tn_rows<M1>(P + c.prow * M1, c.R, M2, c.rows, part + static_cast<int64_t>(blockIdx.x) * M1 * M2);
}

// out[M1,M2] = P^T X over nz chunks (device table `chunks`); `part` holds nz * M1 * M2 floats.  nz_dev != NULL: nz is
// the chunk capacity and *nz_dev the live count.
inline int launch_gemm_tn_rag(const float* P, int M1, int M2, const TnChunk* chunks, int nz, bool gemv, float* part,
                              float* out, cudaStream_t st, const int* nz_dev = nullptr) {
  if (gemv) {
    switch (M1) {
      case 1: k_gemv_tn_rag<1><<<nz, 256, 0, st>>>(P, M2, chunks, part, nz_dev); break;
      case 2: k_gemv_tn_rag<2><<<nz, 256, 0, st>>>(P, M2, chunks, part, nz_dev); break;
      case 3: k_gemv_tn_rag<3><<<nz, 256, 0, st>>>(P, M2, chunks, part, nz_dev); break;
      default: k_gemv_tn_rag<4><<<nz, 256, 0, st>>>(P, M2, chunks, part, nz_dev); break;
    }
    DSMIL_LAUNCH_OK("k_gemv_tn_rag");
  } else {
    dim3 grid(ceil_div(M2, TBM), ceil_div(M1, TBM), nz);
    k_gemm_tn_rag<<<grid, 256, 0, st>>>(P, M1, M2, chunks, part, nz_dev);
    DSMIL_LAUNCH_OK("k_gemm_tn_rag");
  }
  return launch_sum_partials(part, nz, static_cast<int64_t>(M1) * M2, out, st, nz_dev);
}

}  // namespace dsmil
