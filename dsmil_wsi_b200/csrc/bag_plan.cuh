// The integer plan of a batch of bags: the bag table's numbering, the batched backward's CTAs per bag and the chunking
// of its ragged GEMMs.  The eager calls evaluate these formulas on the host from host arrays; the capture-safe calls
// (dsmil_forward_bags_train_dev / dsmil_backward_bags_dev) evaluate the same functions on the device, in k_plan_bags,
// from the bag list in device memory.  One definition for both, so the two cannot drift: a dev call gives the eager
// call's bits.
#pragma once
#include "common.cuh"
#include "gemm_generic.cuh"
#include "fwd_sm90.cuh"
#include "fwd_batched.cuh"

namespace dsmil {

// One row range of the ragged TN GEMMs: rows [prow, prow + rows) of the packed left operand against the bag rows
// starting at R.  A chunk never straddles two bags.
struct TnChunk {
  const float* R;
  long long prow;
  long long rows;
};

// Partial attention records (== k_attend_b CTAs) of a bag of N rows.
__host__ __device__ inline int recs_for_bag(int64_t N) {
  const int64_t t = (N + sm90::kAttRows - 1) / sm90::kAttRows;
  return static_cast<int>(t < sm90::kMaxRecPerBag ? (t < 1 ? 1 : t) : sm90::kMaxRecPerBag);
}
__host__ __device__ inline int tiles_for_bag(int64_t N) { return static_cast<int>((N + sm90::kTileM - 1) / sm90::kTileM); }

// The next bag of the table: its first row, 128-row tile and partial record, numbered across the batch; advances the
// running counters past it.
__host__ __device__ inline sm90::BagDev bag_entry(const float* X, int64_t N, long long& row, int& tile, int& rec) {
  const int nrec = recs_for_bag(N);
  const sm90::BagDev e{X, N, row, tile, rec, nrec, 0};
  row += N;
  tile += tiles_for_bag(N);
  rec += nrec;
  return e;
}

// CTAs per bag of the batched backward's per-row kernels, from the batch size and its largest bag.  It fixes how the
// per-bag sums t_b and dq_max_b are split, so it follows the shapes only.
__host__ __device__ inline int bwd_bags_ctas(int nb, int64_t max_N) {
  const int64_t a = ceil_div(kSms * 8, nb), b = ceil_div(max_N, 64);
  const int64_t g = a < b ? a : b;
  return static_cast<int>(g > 1 ? g : 1);
}

// Rows per chunk of a ragged TN GEMM over the bags, from the shapes alone.  The streaming form (M1 <= 4, float4 rows)
// takes chunks of >= 64 rows, at most about kSplits of them; the 128 x 128 tile form keeps the tiles x chunks CTAs near
// kSplits, as launch_gemm_tn does.
__host__ __device__ inline int rag_splits(int M1, int M2, bool gemv) {
  if (gemv) return kSplits;
  const int tiles = ceil_div(M1, TBM) * ceil_div(M2, TBM);
  return kSplits / tiles > 1 ? kSplits / tiles : 1;
}
__host__ __device__ inline int64_t rag_rows_per_chunk(int M1, int M2, int64_t total, bool gemv) {
  if (gemv) {
    const int64_t r = (total + kSplits - 1) / kSplits;
    return r > 64 ? r : 64;
  }
  const int64_t s = rag_splits(M1, M2, false);
  const int64_t r = ((total + s - 1) / s + TBK - 1) / TBK * TBK;
  return r > 128 ? r : 128;
}
// Chunks of `rps` rows over the bags (the last chunk of a bag may be shorter); returns how many.  Xs == NULL: count
// only.
__host__ __device__ inline int rag_chunks(const float* const* Xs, const int64_t* Ns, int nb, int M2, int64_t rps,
                                          TnChunk* out) {
  int z = 0;
  long long row = 0;
  for (int b = 0; b < nb; ++b) {
    for (int64_t r0 = 0; r0 < Ns[b]; r0 += rps, ++z)
      if (Xs) out[z] = TnChunk{Xs[b] + r0 * M2, row + r0, Ns[b] - r0 < rps ? Ns[b] - r0 : rps};
    row += Ns[b];
  }
  return z;
}
// Most chunks rag_chunks can give for nb bags at any total: rps >= total / rag_splits, so the whole chunks number at
// most rag_splits, and each bag adds at most one short chunk.
__host__ __device__ inline int rag_chunks_cap(int M1, int M2, bool gemv, int nb) { return rag_splits(M1, M2, gemv) + nb; }

// Row splits of the packed-row reductions over `total` rows, as launch_colsum and launch_gemm_tn's tile form choose.
__host__ __device__ inline RowSplit colsum_split(int64_t total) {
  const int S = colsum_splits(total);
  return RowSplit{total, (total + S - 1) / S, S, 0};
}
__host__ __device__ inline RowSplit gemm_tn_split(int M1, int M2, int64_t total) {
  const int S = tn_splits(M1, M2, total);
  return RowSplit{total, ((total + S - 1) / S + TBK - 1) / TBK * TBK, S, 0};
}

// What the host knows of a batch before a call: the live counts.  A dev call's kernels read them from here.
struct BagsPlan {
  long long total;       // live rows
  int tiles, recs;       // forward: 128-row tiles and partial records
  int G;                 // backward: CTAs per bag of the per-row kernels
  int nci, nc1;          // backward: chunks of gWi and gW1
  int pad_;
  RowSplit cs;           // column sums over the packed rows
  RowSplit tn2;          // gW2 = dz2^T H1 over the packed rows
};

// The planner of a dev call: one thread reads the bag list (Xs, Ns: device memory) and writes the bag table, the live
// counts and, when chi / ch1 are non-NULL, the backward's chunk tables.  A bag with N outside [1, max_rows] or
// features that are NULL or not 16-byte aligned sets *status to 1 + its index (the first such bag; a set status is
// never cleared here), and the call then runs on a stand-in batch instead: every bag becomes one row of zeros
// (zero_row, D floats of the workspace).  Every output of a refused call is then finite and every index in range
// (crit_idx 0, pred = bf, B = 0), and nothing reads the caller's bag list.
__global__ void __launch_bounds__(32)
k_plan_bags(const float* const* __restrict__ Xs, const int64_t* __restrict__ Ns, int nb, long long max_rows, int C,
            int D, float* __restrict__ zero_row, sm90::BagDev* __restrict__ table, TnChunk* __restrict__ chi,
            TnChunk* __restrict__ ch1, BagsPlan* __restrict__ plan, int* __restrict__ status) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int bad = 0;
  long long mx = 0;
  for (int b = 0; b < nb && !bad; ++b) {
    const int64_t N = Ns[b];
    if (N < 1 || N > max_rows || Xs[b] == nullptr || (reinterpret_cast<uintptr_t>(Xs[b]) & 15) != 0) bad = b + 1;
    mx = N > mx ? N : mx;
  }
  if (bad) {
    *status = bad;
    for (int i = 0; i < D; ++i) zero_row[i] = 0.f;
    mx = 1;
  }
  BagsPlan pl{};
  long long row = 0;
  int tile = 0, rec = 0;
  for (int b = 0; b < nb; ++b) table[b] = bad ? bag_entry(zero_row, 1, row, tile, rec) : bag_entry(Xs[b], Ns[b], row, tile, rec);
  pl.total = row;
  pl.tiles = tile;
  pl.recs = rec;
  pl.G = bwd_bags_ctas(nb, mx);
  if (bad) {                     // one one-row chunk per bag, as rag_chunks gives for one-row bags
    for (int b = 0; b < nb && (chi || ch1); ++b) {
      if (chi) chi[b] = TnChunk{zero_row, b, 1};
      if (ch1) ch1[b] = TnChunk{zero_row, b, 1};
    }
    pl.nci = chi ? nb : 0;
    pl.nc1 = ch1 ? nb : 0;
  } else {
    if (chi) {
      const bool gemv = tn_use_gemv(C, D);   // the bags are 16-byte aligned
      pl.nci = rag_chunks(Xs, Ns, nb, D, rag_rows_per_chunk(C, D, row, gemv), chi);
    }
    if (ch1) pl.nc1 = rag_chunks(Xs, Ns, nb, D, rag_rows_per_chunk(kQ, D, row, false), ch1);
  }
  pl.cs = colsum_split(row);
  pl.tn2 = gemm_tn_split(kQ, kQ, row);
  *plan = pl;
}

}  // namespace dsmil
