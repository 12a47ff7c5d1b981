// sm_90a tensor-core path of phase 1 (dsmil.py:11 scores + :49 Q-MLP), D % 128 == 0.
//
//   k_prep_wimg2    packs W1 / W2 into bf16 hi/lo "images" that are byte-for-byte the shared-memory B-operand tiles
//                   wgmma reads (K-major, SWIZZLE_128B), so they are brought in with plain 1-D bulk copies
//                   (cp.async.bulk), no tensor map.  Inside every 16-wide k step W1's k order is permuted to the
//                   order in which the consumer threads hold X in their A fragments (see kLogicalK below).
//   k_qmlp_sm90     persistent, one CTA per SM, 128-row tiles walked through a bag table (ragged batch of bags):
//        consumer warpgroups x2 : 64 rows of the tile each.  A thread streams its two rows of X with 16-byte loads
//                          straight into registers (one 64-float chunk ahead, across tile boundaries; the chunk
//                          kPrefetchChunks further on in the tile is requested into L2 with them), adds them into
//                          the fp32 instance scores (+ packed arg-max key per bag), splits x = hi + lo (two bf16) and
//                          hands both halves to wgmma as the register A operand -- X never goes through shared memory.
//                          3 products per k step: hi*Whi + lo*Whi + hi*Wlo ("3xBF16", error at the fp32 noise floor --
//                          SURVEY A.4, tests/test_oracle.py), fp32 accumulators in registers (m64n128k16).
//                          Layer 2: H1 = relu(acc + b1), split the same way, is its A operand straight from the
//                          accumulator registers; Q -> global: row-major tanh(acc2 + b2) when training keeps it,
//                          otherwise tile blocks (column-major) of the pre-activation, whose readers apply the tanh
//        producer warpgroup  : gives most of its registers to the consumers (setmaxnreg); one thread streams the W1
//                          chunks and, per tile, the two W2 chunks into a kWStages-deep smem ring (mbarrier full /
//                          empty pairs; a stage is freed when both consumer warpgroups' MMAs on it have retired)
//   smem: W ring kWStages x 32 KB | Wi rows (C rounded up to 1/2/4/8)
#pragma once
#include <cuda_bf16.h>
#include <cstdlib>

#include "common.cuh"

namespace dsmil {
namespace sm90 {

constexpr int kTileM = 128;            // rows per tile (two warpgroups x wgmma M = 64)
constexpr int kChunkK = 64;            // k per smem operand chunk: 64 bf16 = 128 B = one swizzle row
constexpr int kTileBytes = kQ * kChunkK * 2;           // 16 KiB: one [128 features x 64 k] bf16 operand tile
constexpr int kChunkBytes = 2 * kTileBytes;            // hi tile + lo tile
constexpr int kWStages = 4;
// X chunks a consumer thread requests into L2 ahead of its loads.  H100 80GB HBM3 at a 400 W limit, 16 bags x 10 000
// x 512, C = 2, three interleaved runs each (DESIGN §4.1): none 0.210-0.211 ms, 2 0.204, 3 0.207-0.208, 4 0.214
constexpr int kPrefetchChunks = 2;
constexpr int kConsumerWGs = 2;
constexpr int kWarpProd = 4 * kConsumerWGs;      // first warp of the producer warpgroup
constexpr int kThreads = 128 * (kConsumerWGs + 1);
// The pool is what the CTA got at launch: 168 regs x 384 threads = 64512; the producer warpgroup hands most of its
// share to the consumers (an .inc blocks until the .dec has freed enough): 2 x 128 x 232 + 128 x 40 = 64512
constexpr int kRegsConsumer = 232, kRegsProducer = 40;
template <int R> __device__ __forceinline__ void reg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void reg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ float4 ldg_stream(const float4* p) {   // read-once data: keep it out of L1
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// ---- PTX wrappers -------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// A failed probe backs off with nanosleep (sleep_ns > 0) so that a waiting role does not steal issue slots.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, uint32_t sleep_ns = 0) {
  uint32_t done = 0, spins = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (done) break;
    if (sleep_ns) __nanosleep(sleep_ns);
    if (++spins > (1u << 26)) __trap();  // a protocol bug must not hang the GPU
  }
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// wgmma shared-memory matrix descriptor, K-major with 128-byte swizzle: start>>4 [0,14) | LBO>>4 [16,30) (1, unused
// for swizzled K-major) | SBO>>4 [32,46) = 1024 B between 8-row groups | layout [62,64) = 1 (SWIZZLE_128B).
// +32 B along k (one 16-wide bf16 step) is +2 on the descriptor; the tiles are 1024-byte aligned.
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr) {
  return static_cast<uint64_t>(((saddr & 0x3ffffu) >> 4) | (1u << 16)) |
         (static_cast<uint64_t>((1024u >> 4) | (1u << 30)) << 32);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator reads above the wait that completes them
__device__ __forceinline__ void fence_acc(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// d[64 x 128] (+)= A[64 x 16] (bf16 pairs in registers, wgmma A-fragment layout) * B (bf16, smem, K-major)
__device__ __forceinline__ void mma_rs(float (&d)[64], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t b,
                                       uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %68, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
      "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %69, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(acc), "l"(b));
}

// byte offset of element (row, k) inside one [rows x 64] bf16 SWIZZLE_128B tile
__host__ __device__ inline uint32_t swz_off(int row, int k) {
  return static_cast<uint32_t>(row * 128 + ((((k >> 3) ^ (row & 7)) & 7) << 4) + ((k & 7) << 1));
}
// A-fragment order of X: in every 16-wide k step, thread q = lane % 4 of a row loads the float4 at k = 4q .. 4q+3 and
// passes it as the fragment's k = {2q, 2q+1} (first pair) and {2q+8, 2q+9} (second pair).  W1's image stores
// physical k p of a step at this logical k, so the products pair up as in X * W1^T.
__host__ __device__ inline int kLogicalK(int p) {
  const int q = (p & 15) >> 2, t = p & 3;
  return (p & ~15) + (t < 2 ? 2 * q + t : 8 + 2 * q + t - 2);
}

// One bag of a batch, as the kernels see it (device memory, built by the host per call).
struct BagDev {
  const float* X;       // [N, D]
  long long N;
  long long row_off;    // first row of this bag in the packed outputs (classes, A, Q, H1)
  int tile_off;         // first 128-row tile of this bag in the batch-wide tile numbering
  int rec_off;          // first partial record of this bag
  int nrec;             // partial records (== attend CTAs) of this bag
  int pad_;
};

constexpr int kSmemBags = 96;

struct QmlpArgs {
  const BagDev* bags;
  int nb, ntiles;         // bags of the table and their 128-row tiles
  int D, C;
  const float* Wi;
  const float* bi;
  const float* b1;
  const float* b2;
  const uint8_t* w1img;   // D/64 chunks
  const uint8_t* w2img;   // 2 chunks
  float* classes;         // packed [sumN, C] or NULL (scores given by the caller)
  unsigned long long* keys;  // [nbags][kMaxC]
  float* Q;               // packed row-major [sumN,128], or (q_blocked) per-tile column-major blocks [tile][128 col][128 row]
  float* H1;              // packed [sumN,128] or NULL
  bool q_blocked;         // Q in tile blocks of the PRE-activation z2 = acc + b2 (inference path): the tanh moves to
                          // the readers of Q (k_attend_b, k_gather_cand_b).  false: row-major tanh(z2)
  const int* ntiles_dev;  // dev calls: the live tile count (ntiles is then the capacity); NULL: ntiles
};

// Walks the bag table as a role's tile index increases monotonically.
struct TileCursor {
  const BagDev* bags;
  int bag, last;
  __device__ TileCursor(const BagDev* b, int nb) : bags(b), bag(0), last(nb - 1) {}
  __device__ __forceinline__ void seek(int tile) {
    while (bag < last && tile >= bags[bag + 1].tile_off) ++bag;
  }
};

struct f2 { float x, y; };
// tanh(x) = 1 - 2/(exp2(x * 2log2e) + 1) with ex2.approx + rcp.approx: |err| < ~3e-7 absolute, saturates correctly
__device__ __forceinline__ float tanh_ex2(float x) {
  const float t = __fmul_rn(x, 2.8853900817779268f);
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(t));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(__fadd_rn(e, 1.f)));
  return __fmaf_rn(r, -2.f, 1.f);
}
__device__ __forceinline__ f2 fast_tanh2(f2 x) { return f2{tanh_ex2(x.x), tanh_ex2(x.y)}; }

// dynamic smem carve (bytes, from a 1024-aligned base)
constexpr int kOffWRing = 0;                                // kWStages x 32 KiB: W1 chunks AND the two W2 chunks stream here
constexpr int kOffWi = kOffWRing + kWStages * kChunkBytes;  // CT*D floats
constexpr int kSmemFixed = kOffWi;

// CT: classes rounded up to 1/2/4/8.  DT: compile-time feature size (512 = every shipped configuration:
// the chunk loops unroll and the load offsets become immediates) or 0 = run-time D.  DEV: the dev calls' form, whose
// live tile count is read on the device (a.ntiles_dev); the eager form's code does not carry that test.
template <int CT, int DT, bool DEV = false>
__global__ void __launch_bounds__(kThreads, 1)
k_qmlp_sm90(const QmlpArgs a) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment (SWIZZLE_128B atoms)
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t bars[2 * kWStages];
  __shared__ __align__(16) float s_b1[kQ], s_b2[kQ];
  __shared__ BagDev s_bags[kSmemBags];           // the bag table (tile-boundary lookups)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int D = DT ? DT : a.D, C = a.C;
  const int nchunks = D / kChunkK;
  // a tile is live when below the launch's count and, in a dev call, the planner's; the device count is read at each
  // test, not held: the C = 4 run-time-D instantiation has no register to spare for it
  auto live = [&](int t) { return t < a.ntiles && (!DEV || t < *a.ntiles_dev); };
  enum { W_FULL = 0, W_EMPTY = kWStages };
  auto bar = [&](int i) { return smem_u32(&bars[i]); };

  float* sWi = reinterpret_cast<float*>(smem + kOffWi);
  const bool do_scores = a.classes != nullptr;   // bag form (scores given): Wi/bi may be NULL
  if (do_scores)
    for (int i = tid; i < CT * D; i += kThreads) sWi[i] = (i < C * D) ? a.Wi[i] : 0.f;
  if (tid < kQ) { s_b1[tid] = a.b1[tid]; s_b2[tid] = a.b2[tid]; }
  const bool tbl_in_smem = a.nb <= kSmemBags;
  if (tbl_in_smem)
    for (int i = tid; i < a.nb; i += kThreads) s_bags[i] = a.bags[i];
  const BagDev* tbl = tbl_in_smem ? s_bags : a.bags;
  if (tid == 0) {
    for (int s = 0; s < kWStages; ++s) { mbar_init(bar(W_FULL + s), 1); mbar_init(bar(W_EMPTY + s), kConsumerWGs); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= kWarpProd) {
    // =============================== W image producer (bulk copies) ==========================
    // chunk order == the consumers' order: per tile the W1 chunks 0..n-1, then the two W2 chunks of layer 2
    reg_dec<kRegsProducer>();
    if (warp == kWarpProd && lane == 0) {
      uint32_t stage = 0, phase = 0;
      auto push = [&](const uint8_t* src) {
        mbar_wait(bar(W_EMPTY + stage), phase ^ 1, 256);
        mbar_expect_tx(bar(W_FULL + stage), kChunkBytes);
        bulk_g2s(smem_u32(smem + kOffWRing + stage * kChunkBytes), src, kChunkBytes, bar(W_FULL + stage));
        if (++stage == kWStages) { stage = 0; phase ^= 1; }
      };
      for (int tile = blockIdx.x; live(tile); tile += gridDim.x) {
        for (int kc = 0; kc < nchunks; ++kc) push(a.w1img + static_cast<size_t>(kc) * kChunkBytes);
        push(a.w2img);
        push(a.w2img + kChunkBytes);
      }
    }
    return;
  }

  // =============================== consumer warpgroups =========================================
  reg_inc<kRegsConsumer>();
  // wgmma fragment rows: warp w of the warpgroup owns rows 16w .. 16w+15; lane holds rows lane/4 and lane/4 + 8 and,
  // in the accumulator, columns 8j + 2q, 8j + 2q + 1 (q = lane % 4, j = 0..15)
  const int q = lane & 3;
  const int rloc = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);   // first of this thread's rows in the tile
  const uint32_t swi_u32 = smem_u32(sWi) + 16u * q;
  const uint32_t wring = smem_u32(smem + kOffWRing);
  const bool signaller = (warp & 3) == 0 && lane == 0;
  uint32_t ws = 0, wph = 0;
  auto w_next = [&]() -> uint32_t {       // waits for the next ring stage, returns its index
    const uint32_t s = ws;
    mbar_wait(bar(W_FULL + s), wph);
    if (++ws == kWStages) { ws = 0; wph ^= 1; }
    return s;
  };
  auto w_release = [&](uint32_t s) {      // after wg_wait0: this warpgroup's MMAs on stage s have retired
    if (signaller) mbar_arrive(bar(W_EMPTY + s));
  };

  TileCursor cur_bag(tbl, a.nb);
  // state of the tile whose chunks are being LOADED (may already be the next tile): 32-bit row numbers
  uint32_t ld_N = 0, ld_row = 0;               // rows in the bag, this thread's first row in the bag
  bool ld_full = false;                        // whole 128-row tile inside the bag: unpredicated loads
  long long ld_rowoff = 0;
  const float* xrow = nullptr;
  auto open_tile = [&](int t) {
    cur_bag.seek(t);
    const BagDev* bp = tbl + cur_bag.bag;
    ld_N = static_cast<uint32_t>(bp->N);
    ld_rowoff = bp->row_off;
    ld_row = static_cast<uint32_t>(t - bp->tile_off) * kTileM + rloc;
    ld_full = ld_row - rloc + kTileM <= ld_N;
    xrow = bp->X + static_cast<long long>(ld_row) * D + 4 * q;
  };
  // x[2s + i]: row rloc + 8i, floats 64 kc + 16 s + 4q .. +3.  With the loads of chunk kc, chunk kc + kPrefetchChunks
  // of the same tile is requested into L2: a row's chunk is two 128-byte lines, and the four threads of a row pair
  // (q = 0..3) take row rloc + 8 (q >> 1), line q & 1 -- one prefetch per thread, no registers held.  Not with 8
  // class rows and a run-time D: that instantiation has no register to spare for the address and would spill.
  auto load_chunk = [&](int kc, float4 (&x)[8]) {
    if ((CT <= 4 || DT != 0) && kc + kPrefetchChunks < nchunks && (ld_full || ld_row + 8 * (q >> 1) < ld_N))
      prefetch_l2(xrow - 4 * q + static_cast<long long>(q >> 1) * (8ll * D) + (kc + kPrefetchChunks) * kChunkK + (q & 1) * 32);
#pragma unroll
    for (int s = 0; s < 4; ++s)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float4* src = reinterpret_cast<const float4*>(xrow + static_cast<long long>(i) * (8ll * D) + kc * kChunkK + 16 * s);
        x[2 * s + i] = (ld_full || ld_row + 8 * i < ld_N) ? ldg_stream(src) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
  };
  float sc[2][CT];
  // scores of chunk kc + the bf16 hi/lo A fragments of its four k steps (register 4s + 2 pair + row half)
  // sWi rows >= C are zero-filled (CT rows are staged), so the class loop needs no bound check
  auto convert = [&](const float4 (&x)[8], int kc, uint32_t (&hi)[16], uint32_t (&lo)[16]) {
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      if (do_scores) {
#pragma unroll
        for (int k = 0; k < CT; ++k) {
          const float4 w = lds128(swi_u32 + static_cast<uint32_t>(k * D + kc * kChunkK + 16 * s) * 4u);
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const float4 v = x[2 * s + i];
            float t = sc[i][k];
            t = fmaf(v.x, w.x, t); t = fmaf(v.y, w.y, t); t = fmaf(v.z, w.z, t); t = fmaf(v.w, w.w, t);
            sc[i][k] = t;
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        // x = hi + lo, both bf16: hi = RN(x); lo = RN(x - hi); unpacking a bf16 pair is one shift + one mask
        const float4 v = x[2 * s + i];
        const __nv_bfloat162 h01 = __floats2bfloat162_rn(v.x, v.y), h23 = __floats2bfloat162_rn(v.z, v.w);
        const uint32_t u01 = *reinterpret_cast<const uint32_t*>(&h01), u23 = *reinterpret_cast<const uint32_t*>(&h23);
        const __nv_bfloat162 l01 = __floats2bfloat162_rn(v.x - __uint_as_float(u01 << 16), v.y - __uint_as_float(u01 & 0xffff0000u));
        const __nv_bfloat162 l23 = __floats2bfloat162_rn(v.z - __uint_as_float(u23 << 16), v.w - __uint_as_float(u23 & 0xffff0000u));
        hi[4 * s + i] = u01;
        hi[4 * s + 2 + i] = u23;
        lo[4 * s + i] = *reinterpret_cast<const uint32_t*>(&l01);
        lo[4 * s + 2 + i] = *reinterpret_cast<const uint32_t*>(&l23);
      }
    }
  };
  float acc[64];
  auto mma_chunk = [&](const uint32_t (&hi)[16], const uint32_t (&lo)[16], int kc) -> uint32_t {
    const uint32_t st = w_next();
    const uint64_t bh = smem_desc(wring + st * kChunkBytes), bl = bh + (kTileBytes >> 4);
    wg_fence();
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      mma_rs(acc, hi[4 * s], hi[4 * s + 1], hi[4 * s + 2], hi[4 * s + 3], bh + 2 * s, (kc | s) != 0);
      mma_rs(acc, lo[4 * s], lo[4 * s + 1], lo[4 * s + 2], lo[4 * s + 3], bh + 2 * s, 1);
      mma_rs(acc, hi[4 * s], hi[4 * s + 1], hi[4 * s + 2], hi[4 * s + 3], bl + 2 * s, 1);
    }
    wg_commit();
    return st;
  };

  int tile = blockIdx.x;
  float4 x[8];
  if (live(tile)) { open_tile(tile); load_chunk(0, x); }
  uint32_t ha[16], la[16], hb[16], lb[16];
  while (live(tile)) {
    const int my_bag = cur_bag.bag;   // this tile's bag (the load state moves on below)
    const uint32_t t_N = ld_N, t_row = ld_row;
    const long long t_rowoff = ld_rowoff;
    const int next_tile = tile + gridDim.x;
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int k = 0; k < CT; ++k) sc[i][k] = 0.f;
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    convert(x, 0, ha, la);
    load_chunk(1, x);
    // two chunks per iteration: the fragment buffers swap roles (nchunks is even: D % 128 == 0).  The next chunk is
    // converted while the tensor core works on this one; its loads were issued one chunk earlier.
#pragma unroll 1
    for (int kc = 0; kc < nchunks; kc += 2) {
      const uint32_t s0 = mma_chunk(ha, la, kc);
      convert(x, kc + 1, hb, lb);
      if (kc + 2 < nchunks) load_chunk(kc + 2, x);
      else if (live(next_tile)) { open_tile(next_tile); load_chunk(0, x); }
      wg_wait0();
      fence_acc(acc);
      w_release(s0);
      const uint32_t s1 = mma_chunk(hb, lb, kc + 1);
      if (kc + 2 < nchunks) { convert(x, kc + 2, ha, la); load_chunk(kc + 3, x); }
      wg_wait0();
      fence_acc(acc);
      w_release(s1);
    }
    // instance scores of this tile: reduce over the 4 threads (q) that share a row; the per-class arg-max key of the
    // tile goes straight to the bag's key slot (one atomicMax per warp and class)
    if (do_scores) {
      unsigned long long best[CT];
#pragma unroll
      for (int k = 0; k < CT; ++k) best[k] = 0ull;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const uint32_t n = t_row + 8 * i;
#pragma unroll
        for (int k = 0; k < CT; ++k) {
          float v = sc[i][k];
          v += __shfl_xor_sync(0xffffffffu, v, 2);
          v += __shfl_xor_sync(0xffffffffu, v, 1);
          if (q == 0 && k < C && n < t_N) {
            v += a.bi[k];
            a.classes[(t_rowoff + n) * C + k] = v;
            const unsigned long long key = pack_key(v, n);
            best[k] = key > best[k] ? key : best[k];
          }
        }
      }
#pragma unroll
      for (int k = 0; k < CT; ++k) {
        const unsigned long long b = warp_max_u64(best[k]);
        if (lane == 0 && k < C && b) atomicMax(a.keys + static_cast<size_t>(my_bag) * kMaxC + k, b);
      }
    }
    // ---- H1 = relu(acc + b1) (-> global when training keeps it) -> bf16 hi/lo A fragments of layer 2 ----
    // accumulator column block j holds k = 8j + 2q (+1) of layer 2, i.e. k step j/2, fragment register 2 (j%2) + i
    uint32_t h2[32], l2[32];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float2 bb = *reinterpret_cast<const float2*>(&s_b1[8 * j + 2 * q]);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float h0 = fmaxf(acc[4 * j + 2 * i] + bb.x, 0.f), h1 = fmaxf(acc[4 * j + 2 * i + 1] + bb.y, 0.f);
        if (a.H1 != nullptr && t_row + 8 * i < t_N)
          *reinterpret_cast<float2*>(a.H1 + (t_rowoff + t_row + 8 * i) * kQ + 8 * j + 2 * q) = make_float2(h0, h1);
        const __nv_bfloat162 hh = __floats2bfloat162_rn(h0, h1);
        const uint32_t hu = *reinterpret_cast<const uint32_t*>(&hh);
        const __nv_bfloat162 ll = __floats2bfloat162_rn(h0 - __uint_as_float(hu << 16), h1 - __uint_as_float(hu & 0xffff0000u));
        h2[4 * (j >> 1) + 2 * (j & 1) + i] = hu;
        l2[4 * (j >> 1) + 2 * (j & 1) + i] = *reinterpret_cast<const uint32_t*>(&ll);
      }
    }
    // ---- layer 2: Qacc = A2 * W2^T, the two W2 chunks from the ring ----
    float qa[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) qa[i] = 0.f;
    const uint32_t w0 = w_next(), w1 = w_next();
    {
      const uint64_t b0 = smem_desc(wring + w0 * kChunkBytes), b1 = smem_desc(wring + w1 * kChunkBytes);
      wg_fence();
#pragma unroll
      for (int s = 0; s < 8; ++s) {
        const uint64_t bh = (s < 4 ? b0 : b1) + 2 * (s & 3), bl = bh + (kTileBytes >> 4);
        mma_rs(qa, h2[4 * s], h2[4 * s + 1], h2[4 * s + 2], h2[4 * s + 3], bh, s > 0);
        mma_rs(qa, l2[4 * s], l2[4 * s + 1], l2[4 * s + 2], l2[4 * s + 3], bh, 1);
        mma_rs(qa, h2[4 * s], h2[4 * s + 1], h2[4 * s + 2], h2[4 * s + 3], bl, 1);
      }
      wg_commit();
      wg_wait0();
      fence_acc(qa);
      w_release(w0);
      w_release(w1);
    }
    // ---- the pre-activation qa + b2 (tile blocks) or Q = tanh(qa + b2) (row-major) ----
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int c = 8 * j + 2 * q;
      const float2 bb = *reinterpret_cast<const float2*>(&s_b2[c]);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float z0 = qa[4 * j + 2 * i] + bb.x, z1 = qa[4 * j + 2 * i + 1] + bb.y;
        if (a.q_blocked) {
          // tile-blocked, column-major: the 8 rows of a lane quad's column are one 32-byte sector
          float* dst = a.Q + static_cast<size_t>(tile) * (kTileM * kQ) + static_cast<size_t>(c) * kTileM + rloc + 8 * i;
          dst[0] = z0;
          dst[kTileM] = z1;
        } else if (t_row + 8 * i < t_N) {
          // the same tanh_ex2 the readers of the tile blocks apply: train and eval give the same Q bits
          *reinterpret_cast<float2*>(a.Q + (t_rowoff + t_row + 8 * i) * kQ + c) = make_float2(tanh_ex2(z0), tanh_ex2(z1));
        }
      }
    }
    tile = next_tile;
  }
}

// one kernel for both images
__global__ void __launch_bounds__(256)
k_prep_wimg2(const float* __restrict__ W1, int D, const float* __restrict__ W2, uint8_t* __restrict__ img1,
             uint8_t* __restrict__ img2) {
  const int t1 = 128 * D, total = t1 + 128 * kQ;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const bool first = i < t1;
    const int K = first ? D : kQ;
    const int j = first ? i : i - t1;
    const int n = j / K, k = j % K;
    const float w = first ? W1[j] : W2[j];
    const __nv_bfloat16 hi = __float2bfloat16_rn(w);
    const __nv_bfloat16 lo = __float2bfloat16_rn(w - __bfloat162float(hi));
    uint8_t* chunk = (first ? img1 : img2) + static_cast<size_t>(k / kChunkK) * kChunkBytes;
    const uint32_t off = swz_off(n, first ? kLogicalK(k % kChunkK) : k % kChunkK);
    *reinterpret_cast<__nv_bfloat16*>(chunk + off) = hi;
    *reinterpret_cast<__nv_bfloat16*>(chunk + kTileBytes + off) = lo;
  }
}

inline size_t qmlp_smem_bytes(int C, int D) {   // Wi is staged with C rounded up to 1, 2, 4, 8 rows
  const int ct = C <= 1 ? 1 : (C <= 2 ? 2 : (C <= 4 ? 4 : 8));
  return kSmemFixed + sizeof(float) * ct * D + 1024;
}
inline size_t wimg_bytes(int D) { return static_cast<size_t>(D / kChunkK) * kChunkBytes + 2 * kChunkBytes; }
// 227 KB of shared memory per block on sm_90, less the kernel's static arrays (barriers, biases, bag table)
inline bool qmlp_supported(const dsmil_params_t* p) {
  return p->nonlinear && p->D % (2 * kChunkK) == 0 &&
         qmlp_smem_bytes(p->C, p->D) + 2 * kQ * sizeof(float) + kSmemBags * sizeof(BagDev) + 256 <= 232448;
}

inline int launch_prep_wimg(const dsmil_params_t* p, uint8_t* wimg, cudaStream_t st) {
  uint8_t* w2img = wimg + static_cast<size_t>(p->D / kChunkK) * kChunkBytes;
  k_prep_wimg2<<<80, 256, 0, st>>>(p->W1, p->D, p->W2, wimg, w2img);
  DSMIL_LAUNCH_OK("k_prep_wimg2");
  return 0;
}

// scores + arg-max keys + Q (+H1) for the ntiles 128-row tiles of the nb bags of the table.
// wimg must already hold the images (launch_prep_wimg).  ntiles_dev != NULL: ntiles is the capacity, *ntiles_dev the
// live count.
inline int launch_qmlp(const dsmil_params_t* p, const BagDev* bags_dev, int nb, int ntiles, float* classes,
                       unsigned long long* keys, float* Q, float* H1, const uint8_t* wimg, int num_sms, cudaStream_t st,
                       bool q_blocked, const int* ntiles_dev = nullptr) {
  const int D = p->D, C = p->C;
  if (ntiles_dev != nullptr && C > 4) {
    set_error("launch_qmlp: a device tile count needs C <= 4");
    return DSMIL_ERR_ARG;
  }
  const uint8_t* w2img = wimg + static_cast<size_t>(D / kChunkK) * kChunkBytes;
  QmlpArgs a{bags_dev, nb, ntiles, D, C, p->Wi, p->bi, p->b1, p->b2, wimg, w2img, classes, keys, Q, H1, q_blocked,
             ntiles_dev};
  const size_t smem = qmlp_smem_bytes(C, D);
  const int grid = ntiles < num_sms ? ntiles : num_sms;
  auto go = [&](auto kern) -> int {
    // (set on every launch: the instantiations share one function-pointer TYPE, so a cached flag here would be
    //  shared between them -- found by the D=1024 / C=1 shape tests; the call costs ~1 us of host time)
    DSMIL_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    prof_begin(PROF_FUSED, st);
    kern<<<grid, kThreads, smem, st>>>(a);
    prof_end(PROF_FUSED, st);
    DSMIL_LAUNCH_OK("k_qmlp_sm90");
    return 0;
  };
  if (ntiles_dev != nullptr) {   // the dev calls' shapes: C <= 4
    if (D == 512) {
      if (C == 1) return go(k_qmlp_sm90<1, 512, true>);
      if (C == 2) return go(k_qmlp_sm90<2, 512, true>);
      return go(k_qmlp_sm90<4, 512, true>);
    }
    if (C == 1) return go(k_qmlp_sm90<1, 0, true>);
    if (C == 2) return go(k_qmlp_sm90<2, 0, true>);
    return go(k_qmlp_sm90<4, 0, true>);
  }
  if (D == 512) {
    if (C == 1) return go(k_qmlp_sm90<1, 512>);
    if (C == 2) return go(k_qmlp_sm90<2, 512>);
    if (C <= 4) return go(k_qmlp_sm90<4, 512>);
    return go(k_qmlp_sm90<8, 512>);
  }
  if (C == 1) return go(k_qmlp_sm90<1, 0>);
  if (C == 2) return go(k_qmlp_sm90<2, 0>);
  if (C <= 4) return go(k_qmlp_sm90<4, 0>);
  return go(k_qmlp_sm90<8, 0>);
}

}  // namespace sm90
}  // namespace dsmil
