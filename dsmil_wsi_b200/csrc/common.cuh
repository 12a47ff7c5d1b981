// Shared device/host helpers for libdsmil_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include "../../include/dsmil_b200.h"

namespace dsmil {

constexpr int kQ = DSMIL_Q;
constexpr int kMaxC = DSMIL_MAX_C;
// dsmil.py:56 divides by sqrt(float32(128)); this is that fp32 value.
constexpr float kScale = 11.313708305358887f;
// SMs of an H100 SXM: sizes the grids of the grid-stride kernels (kSms * 8 CTAs)
constexpr int kSms = 132;
// Largest number of partial sums of a split reduction (attention records, column sums, TN GEMM splits): it fixes the
// fp32 summation order, so it does not follow the SM count -- results are the same on every GPU.  The workspace
// sizes depend on it.
constexpr int kSplits = 296;

// ---- host-side error plumbing -------------------------------------------------------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);
void count_launch(int n = 1);

// ---- optional live kernel timing (bench.py roofline): CUDA events around tagged launches on the
// launching stream; off by default (zero overhead), enabled through dsmil_profile_enable().
enum ProfTag : int { PROF_SCORES = 0, PROF_QMLP = 1, PROF_ATTEND = 2, PROF_FINAL = 3, PROF_FUSED = 4, PROF_NTAGS = 8 };
extern bool g_prof_on;
void prof_begin_impl(int tag, cudaStream_t st);
void prof_end_impl(int tag, cudaStream_t st);
inline void prof_begin(int tag, cudaStream_t st) { if (g_prof_on) prof_begin_impl(tag, st); }
inline void prof_end(int tag, cudaStream_t st) { if (g_prof_on) prof_end_impl(tag, st); }

#define DSMIL_CUDA_OK(expr)                                      \
  do {                                                           \
    cudaError_t _e = (expr);                                     \
    if (_e != cudaSuccess) return ::dsmil::cuda_fail(_e, #expr); \
  } while (0)

#define DSMIL_LAUNCH_OK(name)                                     \
  do {                                                            \
    ::dsmil::count_launch();                                      \
    cudaError_t _e = cudaGetLastError();                          \
    if (_e != cudaSuccess) return ::dsmil::cuda_fail(_e, name);   \
  } while (0)

#define DSMIL_REQUIRE(cond, ...)          \
  do {                                    \
    if (!(cond)) {                        \
      ::dsmil::set_error(__VA_ARGS__);    \
      return DSMIL_ERR_ARG;               \
    }                                     \
  } while (0)

// ---- workspace carving (256-byte aligned bump allocator over caller memory) ------------------
struct Carver {
  char* base;
  size_t off;
  size_t cap;
  bool dry;  // dry run: only measure
  Carver(void* b, size_t c) : base(static_cast<char*>(b)), off(0), cap(c), dry(b == nullptr) {}
  template <typename T>
  T* take(size_t n) {
    size_t bytes = (n * sizeof(T) + 255) & ~size_t(255);
    T* p = dry ? nullptr : reinterpret_cast<T*>(base + off);
    off += bytes;
    return p;
  }
  bool ok() const { return dry || off <= cap; }
};

// ---- device helpers ---------------------------------------------------------------------
// Total order on floats as unsigned ints: larger float -> larger key; NaN (canonicalised to
// +NaN) ranks above +inf, matching torch.sort(descending=True) which puts NaN first.
__device__ __forceinline__ uint32_t ordered_key(float v) {
  uint32_t u = __float_as_uint(v);
  if (v != v) u = 0x7fc00000u;  // canonical +NaN
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
// (score, local row) -> 64-bit key whose max is "largest score, then LOWEST row".
__device__ __forceinline__ unsigned long long pack_key(float v, uint32_t row) {
  return (static_cast<unsigned long long>(ordered_key(v)) << 32) | (0xffffffffu - row);
}
__device__ __forceinline__ uint32_t key_row(unsigned long long k) { return 0xffffffffu - static_cast<uint32_t>(k); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    unsigned long long t = __shfl_xor_sync(0xffffffffu, v, o);
    v = t > v ? t : v;
  }
  return v;
}

__host__ __device__ inline int ceil_div(int64_t a, int64_t b) { return static_cast<int>((a + b - 1) / b); }

}  // namespace dsmil
