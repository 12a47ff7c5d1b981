// Batched (bag-table) phase 2/3 kernels used with the tensor-core phase 1 (fwd_sm90.cuh).
//   k_attend_b     dsmil.py:53-57  per (bag, CTA): q_max = Q[critical rows], logits -> A (unnormalised),
//                                  online softmax over the instance axis, partial bag vector
//   k_finalize_b   dsmil.py:56-61  per bag: combine partial records, normalise A, B, Conv1d bag logits,
//                                  critical indices
// Requirements: D % 4 == 0, D <= 2048, feature rows 16-byte aligned, identity V.
#pragma once
#include "common.cuh"
#include "fwd_kernels.cuh"
#include "fwd_sm90.cuh"

namespace dsmil {
namespace sm90 {

constexpr int kAttRows = 128;          // rows per attend tile (same tiling as phase 1)
constexpr int kMaxRecPerBag = 128;

struct AttendArgs {
  const BagDev* bags;
  int nb;
  int D, C;
  const float* Q;           // packed [sumN,128] row-major, or tile-blocked column-major (q_blocked)
  bool q_blocked;           // false: row-major Q; true: tile blocks of the pre-activation (tanh applied on read)
  const unsigned long long* keys;  // [nbags][kMaxC]
  float* A;                 // packed [sumN,C]: receives the raw logits here
  float* recs;              // [total records][rec_floats(C,D)]
  const float* qmax_ext;    // sharded: [nbags][C][128] merged critical queries (NULL: gather from Q via keys)
  const int* nrec_dev;      // dev calls: the live record count of a capacity grid (NULL: one CTA per record)
};

// CT = classes rounded up to 1,2,4; NJ = float4 column groups per thread (D <= 512*NJ)
// Occupancy: the D <= 512, C <= 2 instantiations fit 48 registers without spills, i.e. 5 CTAs per SM instead of 4.
// One CTA per 128-row tile makes the 16 x 10 000-row step 1264 CTAs: on 132 SMs 2.39 waves of 528 slots (three
// rounds) become 1.92 waves of 660 (two rounds).  Wider variants keep the default bound (they would spill).
template <int CT, int NJ>
__global__ void __launch_bounds__(256, (NJ == 1 && CT <= 2) ? 5 : 0)
k_attend_b(const AttendArgs a) {
  extern __shared__ __align__(16) float s_dyn[];           // [C][D] cross-half reduction buffer
  __shared__ __align__(16) float sq[CT][kQ];
  __shared__ float sL[kAttRows][CT];
  __shared__ float sE[kAttRows][CT];
  __shared__ float s_red[8][CT];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int C = a.C, D = a.D;
  if (a.nrec_dev != nullptr && static_cast<int>(blockIdx.x) >= *a.nrec_dev) return;
  // which bag does this CTA belong to?
  const int rec = blockIdx.x;
  int bag = 0;
  while (bag < a.nb - 1 && rec >= a.bags[bag + 1].rec_off) ++bag;
  const BagDev bg = a.bags[bag];
  const int cta_in_bag = rec - bg.rec_off;
  const int ntiles = static_cast<int>((bg.N + kAttRows - 1) / kAttRows);

  // q_max rows (dsmil.py:53-54: the critical instances' queries; here gathered from Q, same bits)
  for (int i = tid; i < CT * kQ; i += 256) {
    const int k = i / kQ, j = i % kQ;
    float v = 0.f;
    if (k < C && a.qmax_ext != nullptr) {
      v = a.qmax_ext[(static_cast<size_t>(bag) * C + k) * kQ + j];
    } else if (k < C) {
      const long long row = key_row(a.keys[static_cast<size_t>(bag) * kMaxC + k]);
      v = a.q_blocked ? tanh_ex2(a.Q[static_cast<size_t>(bg.tile_off + row / kAttRows) * (kAttRows * kQ) + j * kAttRows + (row % kAttRows)])
                      : a.Q[(bg.row_off + row) * kQ + j];
    }
    sq[k][j] = v;
  }
  float run_m[CT], run_s[CT];                   // running (max, sum), replicated in every thread
#pragma unroll
  for (int k = 0; k < CT; ++k) { run_m[k] = -INFINITY; run_s[k] = 0.f; }
  float acc[CT][NJ][4];
#pragma unroll
  for (int k = 0; k < CT; ++k)
#pragma unroll
    for (int j = 0; j < NJ; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[k][j][e] = 0.f;
  __syncthreads();

  const int half = tid >> 7, c4 = tid & 127;     // row parity handled / float4 column within a 512-float span
  const int D4 = D >> 2;
  for (int t = cta_in_bag; t < ntiles; t += bg.nrec) {
    const long long r0 = static_cast<long long>(t) * kAttRows;
    const int rows = static_cast<int>((bg.N - r0) < kAttRows ? (bg.N - r0) : kAttRows);
    // (a) logits -> registers of threads 0..127 (row = tid), -inf for rows beyond the bag
    float Lr[CT];
#pragma unroll
    for (int k = 0; k < CT; ++k) Lr[k] = -INFINITY;
    if (a.q_blocked) {
      // thread (row = tid & 127, column half = tid >> 7): 64 coalesced column loads, no shuffles
      const int r = tid & 127, hf = tid >> 7;
      const float* qb = a.Q + static_cast<size_t>(bg.tile_off + t) * (kAttRows * kQ) + static_cast<size_t>(hf * 64) * kAttRows + r;
      float d[CT];
#pragma unroll
      for (int k = 0; k < CT; ++k) d[k] = 0.f;
#pragma unroll 4
      for (int c = 0; c < 64; c += 4) {
        // one base pointer per step: the four loads issue together with immediate offsets
        const float* qc = qb + c * kAttRows;
        // the tanh of dsmil.py:31, deferred from the phase-1 epilogue
        const f2 ta = fast_tanh2(f2{__ldg(qc), __ldg(qc + kAttRows)});
        const f2 tb = fast_tanh2(f2{__ldg(qc + 2 * kAttRows), __ldg(qc + 3 * kAttRows)});
#pragma unroll
        for (int k = 0; k < CT; ++k) {
          const float4 w = *reinterpret_cast<const float4*>(&sq[k][hf * 64 + c]);
          d[k] = fmaf(ta.x, w.x, d[k]); d[k] = fmaf(ta.y, w.y, d[k]); d[k] = fmaf(tb.x, w.z, d[k]); d[k] = fmaf(tb.y, w.w, d[k]);
        }
      }
      if (hf == 1) {
#pragma unroll
        for (int k = 0; k < CT; ++k) sE[r][k] = d[k];          // park the upper-half partial
      }
      __syncthreads();
      if (hf == 0 && r < rows) {
#pragma unroll
        for (int k = 0; k < CT; ++k) {
          Lr[k] = __fdiv_rn(d[k] + sE[r][k], kScale);          // dsmil.py:56: a division by sqrt(128f)
          if (k < C) a.A[(bg.row_off + r0 + r) * C + k] = Lr[k];
        }
      }
    } else {
      // row-major Q (training keeps it for the backward): warp w owns rows w*16 .. w*16+15
#pragma unroll 4
      for (int rr = 0; rr < 16; ++rr) {
        const int r = warp * 16 + rr;
        if (r < rows) {
          const float4 q = __ldg(reinterpret_cast<const float4*>(a.Q + (bg.row_off + r0 + r) * kQ) + lane);
#pragma unroll
          for (int k = 0; k < CT; ++k) {
            const float4 w = *reinterpret_cast<const float4*>(&sq[k][lane * 4]);
            float d = q.x * w.x;
            d = fmaf(q.y, w.y, d);
            d = fmaf(q.z, w.z, d);
            d = fmaf(q.w, w.w, d);
            d = warp_sum(d);
            if (lane == 0) {
              const float L = __fdiv_rn(d, kScale);
              sL[r][k] = L;
              if (k < C) a.A[(bg.row_off + r0 + r) * C + k] = L;
            }
          }
        }
      }
      __syncthreads();
      if (tid < rows) {
#pragma unroll
        for (int k = 0; k < CT; ++k) Lr[k] = sL[tid][k];
      }
    }
    // (b) tile max (warp shuffles + 4 partials), running max / rescale, exp weights, running sum --
    //     every thread derives the same (m, s) from shared partials: no single-thread phases
#pragma unroll
    for (int k = 0; k < CT; ++k) {
      const float v = warp_max(Lr[k]);
      if (lane == 0) s_red[warp][k] = v;       // warps 4..7 hold no rows: -inf
    }
    __syncthreads();
    float mnew[CT], scl[CT], ev[CT];
#pragma unroll
    for (int k = 0; k < CT; ++k) {
      float mx = fmaxf(fmaxf(s_red[0][k], s_red[1][k]), fmaxf(s_red[2][k], s_red[3][k]));
      mnew[k] = fmaxf(run_m[k], mx);
      scl[k] = (run_m[k] == -INFINITY) ? 0.f : expf(run_m[k] - mnew[k]);
      ev[k] = (Lr[k] == -INFINITY) ? 0.f : expf(Lr[k] - mnew[k]);
      if (tid < kAttRows) sE[tid][k] = ev[k];
    }
    __syncthreads();                           // s_red reads done, sE visible
#pragma unroll
    for (int k = 0; k < CT; ++k) {
      const float v = warp_sum(ev[k]);
      if (lane == 0) s_red[warp][k] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < CT; ++k) {
      run_s[k] = run_s[k] * scl[k] + ((s_red[0][k] + s_red[1][k]) + (s_red[2][k] + s_red[3][k]));
      run_m[k] = mnew[k];
    }
    // (c) weighted feature sum: this thread takes rows of its parity, float4 columns c4 + 128*j
#pragma unroll
    for (int k = 0; k < CT; ++k) {
#pragma unroll
      for (int j = 0; j < NJ; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[k][j][e] *= scl[k];
    }
    const float* xb = bg.X + r0 * D;
#pragma unroll 8
    for (int r = half; r < rows; r += 2) {
      float4 x[NJ];
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int col = c4 + 128 * j;
        x[j] = col < D4 ? ldg_stream(reinterpret_cast<const float4*>(xb + static_cast<long long>(r) * D) + col)
                        : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int k = 0; k < CT; ++k) {
        const float e = sE[r][k];
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          acc[k][j][0] = fmaf(e, x[j].x, acc[k][j][0]);
          acc[k][j][1] = fmaf(e, x[j].y, acc[k][j][1]);
          acc[k][j][2] = fmaf(e, x[j].z, acc[k][j][2]);
          acc[k][j][3] = fmaf(e, x[j].w, acc[k][j][3]);
        }
      }
    }
    __syncthreads();
  }
  // fold the two row parities (fixed order: even rows + odd rows) and emit the record
  float* recp = a.recs + static_cast<size_t>(rec) * rec_floats(C, D);
  if (half == 1) {
#pragma unroll
    for (int k = 0; k < CT; ++k)
      if (k < C)
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          const int col = c4 + 128 * j;
          if (col < D4)
            *reinterpret_cast<float4*>(s_dyn + k * D + col * 4) =
                make_float4(acc[k][j][0], acc[k][j][1], acc[k][j][2], acc[k][j][3]);
        }
  }
  __syncthreads();
  if (half == 0) {
#pragma unroll
    for (int k = 0; k < CT; ++k)
      if (k < C)
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          const int col = c4 + 128 * j;
          if (col < D4) {
            const float4 o = *reinterpret_cast<const float4*>(s_dyn + k * D + col * 4);
            float* dst = recp + 2 * C + static_cast<size_t>(k) * D + col * 4;
            dst[0] = acc[k][j][0] + o.x;
            dst[1] = acc[k][j][1] + o.y;
            dst[2] = acc[k][j][2] + o.z;
            dst[3] = acc[k][j][3] + o.w;
          }
        }
  }
  if (tid == 0) {
#pragma unroll
    for (int k = 0; k < CT; ++k)
      if (k < C) { recp[k] = run_m[k]; recp[C + k] = run_s[k]; }
  }
}

struct FinalizeArgs {
  const BagDev* bags;
  int D, C;
  const float* recs;
  const unsigned long long* keys;
  const float* Wf;
  const float* bf;
  float* A;       // packed, logits in / softmax out
  float* B;       // [nbags, C, D]
  float* pred;    // [nbags, C]
  long long* crit;  // [nbags, C] or NULL
  float* pred_part;        // [nbags][kFinSlices][kMaxC] partial bag logits
  unsigned int* counters;  // [nbags] arrival counters (zeroed by the host before the batch)
  // sharded use: (1) emit != NULL: combine this rank's records of each bag into ONE unnormalised record
  // emit[bag] = (M, S, sum Bp*w) and stop (no A / B / logits);  (2) ext_P > 0: the records of bag b are the
  // ext_P per-rank records at recs[(p * ext_nb + b) * stride] (an all-gather result), not the bag table's.
  float* emit;
  int ext_P, ext_nb;
};

constexpr int kFinSlices = 32;

// grid = (kFinSlices, nb).  Every CTA derives (M, S) of its bag from the partial records, normalises its share of the
// rows of A, combines its share of the B columns -- eight threads per column, each summing every eighth record with
// all its loads in flight, partials added in a fixed order (deterministic) -- and contributes a partial Conv1d dot
// product; the last CTA of the bag to finish adds the kFinSlices partials in slice order (dsmil.py:59-61) and writes
// the critical indices.  4 CTAs per SM (64 registers): left free, ptxas squeezes the kernel under 48 registers for a
// fifth CTA and spills.
__global__ void __launch_bounds__(256, 4)
k_finalize_b(const FinalizeArgs a) {
  __shared__ float sw[kMaxRecPerBag][kMaxC];
  __shared__ float sM[kMaxC], sS[kMaxC];
  __shared__ float s_part[8][32];
  __shared__ float red[kMaxC];
  __shared__ unsigned int s_last;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int C = a.C, D = a.D;
  const int bag = blockIdx.y;
  const BagDev bg = a.bags[bag];
  const size_t rstride = rec_floats(C, D);
  const bool ext = a.ext_P > 0;
  const float* recs = ext ? a.recs + static_cast<size_t>(bag) * rstride : a.recs + static_cast<size_t>(bg.rec_off) * rstride;
  const size_t pstride = ext ? rstride * a.ext_nb : rstride;     // distance between consecutive records of the bag
  const int P = ext ? a.ext_P : bg.nrec;
  // (M, S): warp k scans the records of class k; fixed-order combine
  for (int k = warp; k < C; k += 8) {
    float m = -INFINITY;
    for (int p = lane; p < P; p += 32) m = fmaxf(m, recs[p * pstride + k]);
    m = warp_max(m);
    float sacc = 0.f;
    for (int p = lane; p < P; p += 32) {
      const float mp = recs[p * pstride + k];
      const float w = (mp == -INFINITY) ? 0.f : expf(mp - m);
      sw[p][k] = w;
      sacc = fmaf(recs[p * pstride + C + k], w, sacc);
    }
    sacc = warp_sum(sacc);
    if (lane == 0) { sM[k] = m; sS[k] = sacc; }
  }
  __syncthreads();
  if (a.emit == nullptr) {  // normalise this slice's rows of A
    const long long total = bg.N * C;
    const long long per = (total + gridDim.x - 1) / gridDim.x;
    const long long lo = per * blockIdx.x, hi = (lo + per) < total ? (lo + per) : total;
    float* Ab = a.A + bg.row_off * C;
    for (long long i = lo + tid; i < hi; i += 256) {
      const int k = static_cast<int>(i % C);
      Ab[i] = __fdiv_rn(expf(Ab[i] - sM[k]), sS[k]);
    }
  }
  // B columns of this slice: element e = k*D + d; thread (column = tid & 31, record phase rp = tid >> 5)
  const int CD = C * D;
  const int eps = (CD + kFinSlices - 1) / kFinSlices;
  const int e_lo = eps * blockIdx.x, e_hi = (e_lo + eps) < CD ? (e_lo + eps) : CD;
  const int rp = tid >> 5;
  float ppart[kMaxC];
#pragma unroll
  for (int k = 0; k < kMaxC; ++k) ppart[k] = 0.f;
  for (int base = e_lo; base < e_hi; base += 32) {
    const int e = base + lane;
    float acc = 0.f;
    if (e < e_hi) {
      const int k = e / D;
      const float* col = recs + 2 * C + e;
#pragma unroll 1
      for (int p0 = rp; p0 < P; p0 += 64) {   // up to 8 loads in flight per thread: records p0, p0+8, ..., p0+56
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = (p0 + 8 * u < P) ? col[static_cast<size_t>(p0 + 8 * u) * pstride] : 0.f;
#pragma unroll
        for (int u = 0; u < 8; ++u)
          if (p0 + 8 * u < P) acc = fmaf(v[u], sw[p0 + 8 * u][k], acc);
      }
    }
    s_part[rp][lane] = acc;
    __syncthreads();
    if (rp == 0 && e < e_hi) {
      float tot = s_part[0][lane];
#pragma unroll
      for (int r = 1; r < 8; ++r) tot += s_part[r][lane];
      if (a.emit != nullptr) {
        a.emit[static_cast<size_t>(bag) * rstride + 2 * C + e] = tot;
      } else {
        const int k = e / D;
        const float bval = __fdiv_rn(tot, sS[k]);
        a.B[static_cast<size_t>(bag) * CD + e] = bval;
        for (int kk = 0; kk < C; ++kk) ppart[kk] = fmaf(__ldg(a.Wf + static_cast<size_t>(kk) * CD + e), bval, ppart[kk]);
      }
    }
    __syncthreads();
  }
  if (a.emit != nullptr) {
    if (blockIdx.x == 0 && tid < C) {
      a.emit[static_cast<size_t>(bag) * rstride + tid] = sM[tid];
      a.emit[static_cast<size_t>(bag) * rstride + C + tid] = sS[tid];
    }
    return;
  }
  // partial Conv1d logits of this slice: the contributions live in warp 0 (fixed shuffle order)
  if (warp == 0) {
    for (int kk = 0; kk < C; ++kk) {
      const float v = warp_sum(ppart[kk]);
      if (lane == 0) red[kk] = v;
    }
  }
  __syncthreads();
  float* part = a.pred_part + (static_cast<size_t>(bag) * kFinSlices + blockIdx.x) * kMaxC;
  if (tid < C) part[tid] = red[tid];
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(a.counters + bag, 1u);
  __syncthreads();
  if (s_last != kFinSlices - 1) return;
  __threadfence();
  if (tid < C) {
    const volatile float* pp = a.pred_part + static_cast<size_t>(bag) * kFinSlices * kMaxC;
    float sacc = 0.f;
    for (int sl = 0; sl < kFinSlices; ++sl) sacc += pp[sl * kMaxC + tid];
    a.pred[static_cast<size_t>(bag) * C + tid] = sacc + __ldg(a.bf + tid);
    if (a.crit) a.crit[static_cast<size_t>(bag) * C + tid] = key_row(a.keys[static_cast<size_t>(bag) * kMaxC + tid]);
  }
}

// Candidate record of every bag of this rank (layout of fwd_kernels.cuh: idx[C] int64 | score[C] | qrow[C,128]).
// grid = (C, nb), 128 threads.  row_offsets[b] = global index of the bag's first local row.
__global__ void __launch_bounds__(128)
k_gather_cand_b(const BagDev* __restrict__ bags, const unsigned long long* __restrict__ keys,
                const float* __restrict__ classes, const float* __restrict__ Q, bool q_blocked,
                const long long* __restrict__ row_offsets, int C, float* __restrict__ cands) {
  const int k = blockIdx.x, bag = blockIdx.y;
  const BagDev bg = bags[bag];
  float* cand = cands + static_cast<size_t>(bag) * cand_floats(C);
  long long* idx = reinterpret_cast<long long*>(cand);
  float* score = cand + 2 * C;
  float* qrow = cand + 3 * C + static_cast<size_t>(k) * kQ;
  const unsigned long long key = keys[static_cast<size_t>(bag) * kMaxC + k];
  if (bg.N <= 0 || key == 0ull) {
    if (threadIdx.x == 0) { idx[k] = INT64_MAX; score[k] = -INFINITY; }
    qrow[threadIdx.x] = 0.f;
    return;
  }
  const long long row = key_row(key);
  if (threadIdx.x == 0) {
    idx[k] = row + row_offsets[bag];
    score[k] = classes[(bg.row_off + row) * C + k];
  }
  qrow[threadIdx.x] = q_blocked
      ? tanh_ex2(Q[static_cast<size_t>(bg.tile_off + row / kAttRows) * (kAttRows * kQ) + threadIdx.x * kAttRows + (row % kAttRows)])
      : Q[(bg.row_off + row) * kQ + threadIdx.x];
}

inline bool batched_supported(const dsmil_params_t* p) {
  return qmlp_supported(p) && !p->passing_v && p->D % 4 == 0 && p->D <= 2048 && p->C <= 4 &&
         ((p->C <= 2) || p->D <= 1024);
}

inline int launch_attend_b(const AttendArgs& a, int nrecs, cudaStream_t st) {
  const int C = a.C, D = a.D;
  const size_t smem = sizeof(float) * C * D;
  const int NJ = D <= 512 ? 1 : (D <= 1024 ? 2 : 4);
  auto go = [&](auto kern) -> int {
    if (smem > 48 * 1024)
      DSMIL_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    prof_begin(PROF_ATTEND, st);
    kern<<<nrecs, 256, smem, st>>>(a);
    prof_end(PROF_ATTEND, st);
    DSMIL_LAUNCH_OK("k_attend_b");
    return 0;
  };
  if (C == 1) { if (NJ == 1) return go(k_attend_b<1, 1>); if (NJ == 2) return go(k_attend_b<1, 2>); return go(k_attend_b<1, 4>); }
  if (C == 2) { if (NJ == 1) return go(k_attend_b<2, 1>); if (NJ == 2) return go(k_attend_b<2, 2>); return go(k_attend_b<2, 4>); }
  if (NJ == 1) return go(k_attend_b<4, 1>);
  return go(k_attend_b<4, 2>);
}

inline int launch_finalize_b(const FinalizeArgs& a, int nb, cudaStream_t st) {
  prof_begin(PROF_FINAL, st);
  k_finalize_b<<<dim3(kFinSlices, nb), 256, 0, st>>>(a);
  prof_end(PROF_FINAL, st);
  DSMIL_LAUNCH_OK("k_finalize_b");
  return 0;
}

}  // namespace sm90
}  // namespace dsmil
