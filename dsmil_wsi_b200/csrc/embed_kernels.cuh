// Embedder kernels of the patch-embedding loop (SURVEY 8f-2): the reference builds its backbone as a torchvision
// ResNet with norm_layer = nn.InstanceNorm2d (compute_feats.py:146-170; affine = False, track_running_stats = False,
// eps = 1e-5), i.e. after every convolution the framework runs  instance_norm -> (+ identity) -> relu  as two or three
// memory-bound passes over the activation tensor.  One kernel does all of it in ONE read and ONE write:
//
//   k_instnorm_plane   one CTA per (n, c) plane of H*W > 1024 elements: the plane is staged in shared memory (<= 16 K
//                      floats: 112x112 = 12 544 is the largest plane of a 224x224 ResNet), mean and biased variance by
//                      two passes over the staged copy (the two-pass form, not E[x^2] - mean^2), then
//                      y = (x - mean) * rsqrt(var + eps) (+ residual) (relu) written out with 16-byte stores
//   k_instnorm_warp    one WARP per plane of <= 1024 elements (56x56 is handled by the CTA kernel; 28x28, 14x14, 7x7
//                      here): the plane lives in registers, 8 planes per CTA
//
//   k_instnorm_nhwc    the channels-last form (the embedding loop runs the ResNet-18 convolutions in cuDNN's NHWC
//                      kernels, tools/exp_channels_last.py compares the two layouts).  Memory is [n][HW][C]; one CTA per (sample, 32-channel group),
//                      lane = channel, warps stride over the pixels, so every warp load is one 128-byte row segment.
//                      Statistics in ONE pass as shifted sums (x - x0, x0 = the channel's first pixel: no
//                      catastrophic cancellation for activations whose mean is far from 0), second pass normalises;
//                      the slab a CTA reads twice is <= 1.6 MB and was just written by the convolution, i.e. the
//                      second read is an L2 hit for every layer but the 112x112 stem.
//
// HBM-bound: algorithmic bytes = 8 B per element (+ 4 with a residual).  fp32 contiguous; in place allowed.
#pragma once
#include "common.cuh"

namespace dsmil {

constexpr int kInPlaneMax = 16384;      // floats staged per plane (64 KB of shared memory)

__device__ __forceinline__ float block_sum_256(float v, float* s_red) {   // fixed-order: warp shuffles, then 8 partials
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  return ((s_red[0] + s_red[1]) + (s_red[2] + s_red[3])) + ((s_red[4] + s_red[5]) + (s_red[6] + s_red[7]));
}

template <bool VEC>
__global__ void __launch_bounds__(256)
k_instnorm_plane(const float* __restrict__ x, const float* __restrict__ res, float* __restrict__ y, int HW, float eps,
                 int relu) {
  extern __shared__ __align__(16) float s_plane[];
  __shared__ float s_red[8];
  const size_t base = static_cast<size_t>(blockIdx.x) * HW;
  const float* xp = x + base;
  float acc = 0.f;
  if (VEC) {
    const float4* x4 = reinterpret_cast<const float4*>(xp);
    float4* s4 = reinterpret_cast<float4*>(s_plane);
    for (int i = threadIdx.x; i < (HW >> 2); i += 256) {
      const float4 v = __ldg(x4 + i);
      s4[i] = v;
      acc += (v.x + v.y) + (v.z + v.w);
    }
  } else {
    for (int i = threadIdx.x; i < HW; i += 256) {
      const float v = __ldg(xp + i);
      s_plane[i] = v;
      acc += v;
    }
  }
  const float mean = block_sum_256(acc, s_red) / static_cast<float>(HW);
  float sq = 0.f;
  for (int i = threadIdx.x; i < HW; i += 256) {
    const float d = s_plane[i] - mean;
    sq = fmaf(d, d, sq);
  }
  const float var = block_sum_256(sq, s_red) / static_cast<float>(HW);       // biased, as F.instance_norm
  const float rstd = rsqrtf(var + eps);
  if (VEC) {
    const float4* s4 = reinterpret_cast<const float4*>(s_plane);
    const float4* r4 = res ? reinterpret_cast<const float4*>(res + base) : nullptr;
    float4* y4 = reinterpret_cast<float4*>(y + base);
    for (int i = threadIdx.x; i < (HW >> 2); i += 256) {
      float4 v = s4[i];
      v.x = (v.x - mean) * rstd; v.y = (v.y - mean) * rstd; v.z = (v.z - mean) * rstd; v.w = (v.w - mean) * rstd;
      if (r4) { const float4 r = __ldg(r4 + i); v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w; }
      if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
      y4[i] = v;
    }
  } else {
    for (int i = threadIdx.x; i < HW; i += 256) {
      float v = (s_plane[i] - mean) * rstd;
      if (res) v += __ldg(res + base + i);
      if (relu) v = fmaxf(v, 0.f);
      y[base + i] = v;
    }
  }
}

// one warp per plane, HW <= 1024: element lane + 32 j lives in register j
__global__ void __launch_bounds__(256)
k_instnorm_warp(const float* __restrict__ x, const float* __restrict__ res, float* __restrict__ y, long long planes, int HW,
                float eps, int relu) {
  const int lane = threadIdx.x & 31;
  const long long plane = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (plane >= planes) return;
  const size_t base = static_cast<size_t>(plane) * HW;
  float v[32];
  float acc = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int i = lane + 32 * j;
    v[j] = i < HW ? __ldg(x + base + i) : 0.f;
    acc += v[j];
  }
  const float mean = warp_sum(acc) / static_cast<float>(HW);
  float sq = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float d = (lane + 32 * j < HW) ? v[j] - mean : 0.f;
    sq = fmaf(d, d, sq);
  }
  const float rstd = rsqrtf(warp_sum(sq) / static_cast<float>(HW) + eps);
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int i = lane + 32 * j;
    if (i < HW) {
      float o = (v[j] - mean) * rstd;
      if (res) o += __ldg(res + base + i);
      if (relu) o = fmaxf(o, 0.f);
      y[base + i] = o;
    }
  }
}

constexpr int kNhwcWarps = 16;

__global__ void __launch_bounds__(32 * kNhwcWarps)
k_instnorm_nhwc(const float* __restrict__ x, const float* __restrict__ res, float* __restrict__ y, int HW, int C, float eps,
                int relu) {
  __shared__ float s_a[kNhwcWarps][32], s_b[kNhwcWarps][32];
  const int groups = C >> 5;
  const int n = blockIdx.x / groups, g = blockIdx.x - n * groups;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t base = (static_cast<size_t>(n) * HW) * C + (g << 5) + lane;
  const float* xp = x + base;
  const float x0 = __ldg(xp);
  float s1 = 0.f, s2 = 0.f;
#pragma unroll 4
  for (int p = warp; p < HW; p += kNhwcWarps) {
    const float d = __ldg(xp + static_cast<size_t>(p) * C) - x0;
    s1 += d;
    s2 = fmaf(d, d, s2);
  }
  s_a[warp][lane] = s1;
  s_b[warp][lane] = s2;
  __syncthreads();
  s1 = 0.f; s2 = 0.f;
#pragma unroll
  for (int w = 0; w < kNhwcWarps; ++w) { s1 += s_a[w][lane]; s2 += s_b[w][lane]; }   // fixed order
  const float inv = 1.f / static_cast<float>(HW);
  const float dm = s1 * inv;                                    // mean - x0
  const float mean = x0 + dm;
  const float var = fmaxf(fmaf(-dm, s1, s2) * inv, 0.f);        // (S2 - S1^2 / HW) / HW, biased as F.instance_norm
  const float rstd = rsqrtf(var + eps);
  float* yp = y + base;
  const float* rp = res ? res + base : nullptr;
#pragma unroll 4
  for (int p = warp; p < HW; p += kNhwcWarps) {
    const size_t o = static_cast<size_t>(p) * C;
    float v = (xp[o] - mean) * rstd;
    if (rp) v += __ldg(rp + o);
    if (relu) v = fmaxf(v, 0.f);
    yp[o] = v;
  }
}

inline int launch_instnorm_nhwc(const float* x, const float* res, float* y, long long N, int HW, int C, float eps, int relu,
                                cudaStream_t st) {
  k_instnorm_nhwc<<<static_cast<unsigned>(N * (C >> 5)), 32 * kNhwcWarps, 0, st>>>(x, res, y, HW, C, eps, relu);
  DSMIL_LAUNCH_OK("k_instnorm_nhwc");
  return 0;
}

inline int launch_instnorm(const float* x, const float* res, float* y, long long planes, int HW, float eps, int relu,
                           cudaStream_t st) {
  if (HW <= 1024) {
    const long long grid = (planes + 7) / 8;
    k_instnorm_warp<<<static_cast<unsigned>(grid), 256, 0, st>>>(x, res, y, planes, HW, eps, relu);
    DSMIL_LAUNCH_OK("k_instnorm_warp");
    return 0;
  }
  const size_t smem = sizeof(float) * static_cast<size_t>(HW);
  const bool vec = (HW % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0) && ((reinterpret_cast<uintptr_t>(y) & 15) == 0) &&
                   (res == nullptr || (reinterpret_cast<uintptr_t>(res) & 15) == 0);
  if (vec) {
    if (smem > 48 * 1024)
      DSMIL_CUDA_OK(cudaFuncSetAttribute(k_instnorm_plane<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    k_instnorm_plane<true><<<static_cast<unsigned>(planes), 256, smem, st>>>(x, res, y, HW, eps, relu);
  } else {
    if (smem > 48 * 1024)
      DSMIL_CUDA_OK(cudaFuncSetAttribute(k_instnorm_plane<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    k_instnorm_plane<false><<<static_cast<unsigned>(planes), 256, smem, st>>>(x, res, y, HW, eps, relu);
  }
  DSMIL_LAUNCH_OK("k_instnorm_plane");
  return 0;
}

}  // namespace dsmil
