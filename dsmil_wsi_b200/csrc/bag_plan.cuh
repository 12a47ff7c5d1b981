// The integer plan of a batch of bags: the bag table's numbering, the batched backward's CTAs per bag and the chunking
// of its ragged GEMMs.  The eager calls evaluate these formulas on the host from host arrays; the capture-safe calls
// (dsmil_forward_bags_train_dev / dsmil_backward_bags_dev and the dsmil_shard_*_dev calls) evaluate the same functions
// on the device, in k_plan_bags, from the bag list in device memory.  One definition for both, so the two cannot drift:
// a dev call gives the eager call's bits.
#pragma once
#include "common.cuh"
#include "gemm_generic.cuh"
#include "fwd_sm90.cuh"
#include "fwd_batched.cuh"
#include "fwd_generic_b.cuh"

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

// The generic forward (fwd_generic_b.cuh, and the per-bag forward it matches): attend CTAs (== partial records) of a
// bag of N rows, one per kAttendRows-row tile up to kSplits.
__host__ __device__ inline int attend_ctas(int64_t N) {
  const int64_t tiles = (N + kAttendRows - 1) / kAttendRows;
  return static_cast<int>(tiles < kSplits ? (tiles < 1 ? 1 : tiles) : kSplits);
}
// The next bag of a generic-forward table: bag_entry's row and 128-row tile numbering, attend_ctas(N) records, and
// the bag's k_scores MODE in pad_.
__host__ __device__ inline sm90::BagDev gen_bag_entry(const float* X, int64_t N, int D, long long& row, int& tile,
                                                      int& rec) {
  const int nrec = attend_ctas(N);
  const sm90::BagDev e{X, N, row, tile, rec, nrec, scores_mode(X, D)};
  row += N;
  tile += tiles_for_bag(N);
  rec += nrec;
  return e;
}
// The alignment a dev call asks of a bag's features on the generic shapes: 16 bytes when D % 4 == 0 (so that the
// MODE of k_scores and the form of the gWi reduction follow from D alone, as the eager calls choose them for aligned
// bags), 4 bytes otherwise (rows of an odd D are never 16-byte aligned; every form there reads scalars).
__host__ __device__ inline bool gen_bag_aligned(const float* X, int D) {
  return (reinterpret_cast<uintptr_t>(X) & (D % 4 == 0 ? 15 : 3)) == 0;
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
// A bag list as a planner walks it: the caller's (host or device memory), or, with zero_row set, the stand-in batch of
// a refused list, every bag one row of zeros.
struct BagList {
  const float* const* Xs;
  const int64_t* Ns;
  const float* zero_row;
  __host__ __device__ const float* X(int b) const { return zero_row ? zero_row : Xs[b]; }
  __host__ __device__ int64_t N(int b) const { return zero_row ? 1 : Ns[b]; }
};
// rag_chunks over a BagList whose packed rows start at row0.  out == NULL: count only (the features are not read).
__host__ __device__ inline int rag_chunks_list(const BagList& L, int nb, int M2, int64_t rps, long long row0,
                                               TnChunk* out) {
  int z = 0;
  long long row = row0;
  for (int b = 0; b < nb; ++b) {
    const int64_t N = L.N(b);
    for (int64_t r0 = 0; r0 < N; r0 += rps, ++z)
      if (out) out[z] = TnChunk{L.X(b) + r0 * M2, row + r0, N - r0 < rps ? N - r0 : rps};
    row += N;
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
  int pad_;              // generic dev calls of passing_v: the live gWv chunks (k_plan_bags_gen)
  RowSplit cs;           // column sums over the packed rows
  RowSplit tn2;          // gW2 = dz2^T H1 over the packed rows
};

// The planner of a dev call: one thread reads the bag list (Xs, Ns: device memory) and writes the bag table, the live
// counts and, when chi / ch1 are non-NULL, the backward's chunk tables.  A bag with N outside [1, max_rows] or
// features that are NULL or not 16-byte aligned (k_plan_bags_gen: not gen_bag_aligned) sets *status to 1 + its index
// (the first such bag; a set status is never cleared here), and the call then runs on a stand-in batch instead: every
// bag becomes one row of zeros (zero_row, D floats of the workspace).  Every output of a refused call is then finite
// and every index in range (crit_idx 0, pred = bf, B = 0), and nothing reads the caller's bag list.  A row-sharded batch also passes each bag's
// first global row (offs_in, device memory): the planner copies it to offs_out, a negative offset is refused like a
// bad bag, and a refused batch's offsets are 0.
// The walk is one thread's; the warp first stages the list of the first kPlanStaged bags into shared memory with its
// loads in flight together, so the walk does not wait on one global load per bag.
constexpr int kPlanStaged = 256;
__global__ void __launch_bounds__(32)
k_plan_bags(const float* const* __restrict__ Xs, const int64_t* __restrict__ Ns, int nb, long long max_rows, int C,
            int D, float* __restrict__ zero_row, sm90::BagDev* __restrict__ table, TnChunk* __restrict__ chi,
            TnChunk* __restrict__ ch1, BagsPlan* __restrict__ plan, int* __restrict__ status,
            const int64_t* __restrict__ offs_in, long long* __restrict__ offs_out) {
  __shared__ const float* sX[kPlanStaged];
  __shared__ int64_t sN[kPlanStaged];
  if (blockIdx.x != 0) return;
  for (int b = threadIdx.x; b < nb && b < kPlanStaged; b += 32) { sX[b] = Xs[b]; sN[b] = Ns[b]; }
  __syncwarp();
  if (threadIdx.x != 0) return;
  auto X_of = [&](int b) { return b < kPlanStaged ? sX[b] : Xs[b]; };
  auto N_of = [&](int b) { return b < kPlanStaged ? sN[b] : Ns[b]; };
  int bad = 0;
  long long mx = 0;
  for (int b = 0; b < nb && !bad; ++b) {
    const int64_t N = N_of(b);
    const float* X = X_of(b);
    if (N < 1 || N > max_rows || X == nullptr || (reinterpret_cast<uintptr_t>(X) & 15) != 0 ||
        (offs_in && offs_in[b] < 0))
      bad = b + 1;
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
  for (int b = 0; b < nb; ++b) table[b] = bad ? bag_entry(zero_row, 1, row, tile, rec) : bag_entry(X_of(b), N_of(b), row, tile, rec);
  if (offs_out)
    for (int b = 0; b < nb; ++b) offs_out[b] = bad ? 0 : offs_in[b];
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

// One model's rows of a row-wise linear layer (k_linear_models): Y = X op(W) (+ the ReLU mask of aux); Y NULL: skip.
struct LinSeg {
  const float *X, *W, *aux;
  float* Y;
  long long N;
};

// The value network's share of a generic dev call's plan (passing_v; every member NULL elsewhere).  XVs: the bags'
// value inputs (device memory; NULL: the features).  vtab [2 nb]: nb entries of the bag table's numbering whose X is
// each bag's value input, then nb whose X is its packed rows of V ([rows, D] from V).  segs [nb] (backward): bag b's
// dzv_b = (A_b dB_b) * [V_b > 0] as a LinSeg over A [rows, C], dB [nb, C, D], V and dzv [rows, D].  chv (backward):
// the gWv chunks over the value inputs, rag_chunks' for the live total; their live count goes to BagsPlan::pad_.
struct PlanValue {
  const float* const* XVs;
  const float* V;
  const float* A;
  const float* dB;
  float* dzv;
  sm90::BagDev* vtab;
  LinSeg* segs;
  TnChunk* chv;
};

// The planner of the generic shapes' dev calls: k_plan_bags with the alignment rule of gen_bag_aligned and a table of
// gen_bag_entry, no row offsets, and for passing_v the value tables of `v` (as the eager value calls build them on
// the host).  A value input must meet its bag's rule: one that is NULL or not gen_bag_aligned refuses the batch like
// a bad bag, and a refused batch's value tables take the stand-in's zero rows, one row per bag.  A kernel of its
// own, as the k_plan_bags SASS stays what it was.
__global__ void __launch_bounds__(32)
k_plan_bags_gen(const float* const* __restrict__ Xs, const int64_t* __restrict__ Ns, int nb, long long max_rows,
                int C, int D, float* __restrict__ zero_row, sm90::BagDev* __restrict__ table,
                TnChunk* __restrict__ chi, TnChunk* __restrict__ ch1, BagsPlan* __restrict__ plan,
                int* __restrict__ status, const PlanValue v) {
  __shared__ const float* sX[kPlanStaged];
  __shared__ const float* sXV[kPlanStaged];
  __shared__ int64_t sN[kPlanStaged];
  if (blockIdx.x != 0) return;
  for (int b = threadIdx.x; b < nb && b < kPlanStaged; b += 32) {
    sX[b] = Xs[b];
    sN[b] = Ns[b];
    if (v.XVs) sXV[b] = v.XVs[b];
  }
  __syncwarp();
  if (threadIdx.x != 0) return;
  auto X_of = [&](int b) { return b < kPlanStaged ? sX[b] : Xs[b]; };
  auto N_of = [&](int b) { return b < kPlanStaged ? sN[b] : Ns[b]; };
  auto XV_of = [&](int b) { return v.XVs ? (b < kPlanStaged ? sXV[b] : v.XVs[b]) : X_of(b); };
  int bad = 0;
  long long mx = 0;
  for (int b = 0; b < nb && !bad; ++b) {
    const int64_t N = N_of(b);
    const float* X = X_of(b);
    if (N < 1 || N > max_rows || X == nullptr || !gen_bag_aligned(X, D)) bad = b + 1;
    if (v.XVs && (XV_of(b) == nullptr || !gen_bag_aligned(XV_of(b), D))) bad = b + 1;
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
  for (int b = 0; b < nb; ++b) {
    const long long r0 = row;
    const int64_t N = bad ? 1 : N_of(b);
    table[b] = bad ? gen_bag_entry(zero_row, 1, D, row, tile, rec) : gen_bag_entry(X_of(b), N, D, row, tile, rec);
    if (v.vtab) {
      v.vtab[b] = v.vtab[nb + b] = table[b];
      v.vtab[b].X = bad ? zero_row : XV_of(b);
      v.vtab[nb + b].X = v.V + r0 * D;
    }
    if (v.segs)
      v.segs[b] = LinSeg{v.A + r0 * C, v.dB + static_cast<size_t>(b) * C * D, v.V + r0 * D, v.dzv + r0 * D, N};
  }
  pl.total = row;
  pl.tiles = tile;
  pl.recs = rec;
  pl.G = bwd_bags_ctas(nb, mx);
  if (bad) {                     // one one-row chunk per bag, as rag_chunks gives for one-row bags
    for (int b = 0; b < nb && (chi || ch1 || v.chv); ++b) {
      if (chi) chi[b] = TnChunk{zero_row, b, 1};
      if (ch1) ch1[b] = TnChunk{zero_row, b, 1};
      if (v.chv) v.chv[b] = TnChunk{zero_row, b, 1};
    }
    pl.nci = chi ? nb : 0;
    pl.nc1 = ch1 ? nb : 0;
    pl.pad_ = v.chv ? nb : 0;
  } else {
    if (chi) {
      const bool gemv = tn_use_gemv(C, D);   // true only where D % 4 == 0, and such bags are 16-byte aligned
      pl.nci = rag_chunks(Xs, Ns, nb, D, rag_rows_per_chunk(C, D, row, gemv), chi);
    }
    if (ch1) pl.nc1 = rag_chunks(Xs, Ns, nb, D, rag_rows_per_chunk(kQ, D, row, false), ch1);
    if (v.chv) pl.pad_ = rag_chunks(v.XVs ? v.XVs : Xs, Ns, nb, D, rag_rows_per_chunk(D, D, row, false), v.chv);
  }
  pl.cs = colsum_split(row);
  pl.tn2 = gemm_tn_split(kQ, kQ, row);
  *plan = pl;
}

// ---- the fold step: M models, each over its own bags (dsmil_*_bags_models*) --------------------------------------
// What the fused backward's kernels read per model (bwd_bags.cuh).  The eager call fills these on the host; the dev
// call's planner, k_plan_bags_models, on the device.
struct BwdModelDev {
  const float *Wf, *Wi;
  float *gWf, *gbf, *gX;
  int e0, nb;            // the model's first entry, its bags
  long long r0;          // its first packed row
};
// One model's share of a chunked reduction: partials [z0, z0 + S) summed into out (NULL: the gradient is not wanted).
struct SumSeg {
  float* out;
  int z0, S;
};

// Every split the one-model backward would choose for one model's own batch of nb bags, `total` rows, the largest of
// mx: the per-row kernels' CTAs per bag, the rows per chunk of gWi and gW1, and the row splits of gW2 and of the
// column sums.  They follow from that model's live sizes alone, which is what keeps its gradients' bits.
struct ModelSplits {
  int G;
  int64_t rps_i, rps_1;
  RowSplit t2, cs;
};
__host__ __device__ inline ModelSplits model_splits(int C, int D, int nb, int64_t total, int64_t mx) {
  ModelSplits s;
  s.G = bwd_bags_ctas(nb, mx);
  s.rps_i = rag_rows_per_chunk(C, D, total, tn_use_gemv(C, D));   // the fused route's bags are 16-byte aligned
  s.rps_1 = rag_rows_per_chunk(kQ, D, total, false);
  s.t2 = gemm_tn_split(kQ, kQ, total);
  s.cs = colsum_split(total);
  return s;
}
// Split z of `s` as a chunk of a model whose packed rows start at r0; R: the packed right operand ([*, ldr]) or NULL.
__host__ __device__ inline TnChunk split_chunk(const RowSplit& s, int z, long long r0, const float* R, int ldr) {
  const long long lo = z * s.rps, hi = lo + s.rps < s.N ? lo + s.rps : s.N;
  return TnChunk{R ? R + (r0 + lo) * ldr : nullptr, r0 + lo, hi - lo};
}
// Most splits gemm_tn_split(kQ, kQ, .) and colsum_split give at any row count.
constexpr int kModelSplitsCap = kSplits;

// The live counts of a fold dev call, over all models: the forward's tiles and records, the backward's chunks.
struct ModelsPlan {
  int tiles, recs;
  int nci, nc1, nc2, ncs;
};
// One model's live counts in a generic fold forward, for the stages that run one launch per model over its block:
// its packed rows (layer 2 of the Q-MLP) and its 128-row tiles (k_qmlp_sm90).
struct FoldLive {
  long long total;
  int tiles;
};
// The numbering of a fold dev call's forward table (PlanModelsArgs::gen).
enum FoldTable : int {
  FOLD_TC = 0,         // the fused tensor-core fold: bag_entry's records, pad_ = the model
  FOLD_GEN = 1,        // generic: gen_bag_entry's records, pad_ = MODE | model << 2, tiles numbered across the models
  FOLD_GEN_QMLP = 2    // as FOLD_GEN, but each model's tiles numbered from 0 (its own k_qmlp_sm90 launch)
};

// What the host knows of model m in a dev call, passed to the planner by value (a dev call uploads nothing).
struct PlanModel {
  sm90::ModelDev w;
  float *gWi, *gbi, *gW1, *gb1, *gW2, *gb2, *gWf, *gbf;   // backward: the model's gradients (NULL: not wanted)
  int e0, nb;                                              // its first entry of the list, its bags
};
struct PlanModelsArgs {
  const float* const* Xs;     // [sum nb] device memory, model-major
  const int64_t* Ns;
  int M, C, D;
  int Gcap;                   // backward: per-CTA partial slots per entry
  long long max_rows;
  float* zero_row;            // [D]
  int* status;                // [M]
  ModelsPlan* plan;
  sm90::BagDev* ftable;       // forward call: the table in the forward numbering, and the members
  sm90::ModelDev* fmodels;
  sm90::BagDev* btable;       // backward call: the table in the backward numbering (bwd_bags.cuh) ...
  BwdModelDev* bmodels;
  TnChunk *chi, *ch1, *ch2, *chc;   // ... the compacted chunk tables (chc padded to ncs_cap with empty chunks) ...
  int ncs_cap;
  SumSeg* segs;               // ... [6][M] and [2][M], as backward_bags_models_impl lays them out
  LinSeg* lin;
  const float* H1;
  float *dz2, *dz1;
  int dc;                     // gradients flow through the scores (d_classes != NULL)
  int gen;                    // FoldTable: the generic shapes take gen_bag_aligned bags and the generic numbering
  FoldLive* live;             // generic forward: [M] each model's live counts
  PlanModel m[sm90::kMaxModels];
};

// The planner of a fold dev call: warp m plans model m from its own bags, as k_plan_bags plans one model, so model
// m's tables are what its one-model dev call would build, shifted to its capacity block (rows from max_rows * e0).
// The models meet only at prefix sums of their counts: tiles and records of the forward numbering, and the chunk
// tables, which are compacted (model m's chunks follow model m - 1's live ones), so that the GEMM grids' live
// counts are single numbers and the partial buffer is indexed as in the eager call.  A model with a bad bag (N
// outside [1, max_rows], features NULL or not 16-byte aligned) sets status[m] = 1 + the bag's index within the model
// and is planned on its stand-in batch (every bag one row of zeros); the other models' plans do not change.
// The generic shapes (a.gen != FOLD_TC) take the alignment rule of gen_bag_aligned and the generic forward's table:
// model m's entries are what k_plan_bags_gen writes for its bags alone, shifted to its capacity block and to the
// model's first tile and record, with its model beside its MODE in pad_ (fold_pad); FOLD_GEN_QMLP numbers each
// model's tiles from 0, for phase 1 launched per model.  a.live[m] then receives the model's live rows and tiles.
__global__ void __launch_bounds__(32 * sm90::kMaxModels)
k_plan_bags_models(const PlanModelsArgs a) {
  enum { TILES, RECS, NCI, NC1, NC2, NCS, NCNT };
  __shared__ int s_cnt[NCNT][sm90::kMaxModels];
  const int m = threadIdx.x >> 5, lane = threadIdx.x & 31, M = a.M;
  const int e0 = a.m[m].e0, nb = a.m[m].nb;
  const long long cap0 = a.max_rows * e0;
  const bool bwd = a.btable != nullptr, gen = a.gen != FOLD_TC;
  // the first bad bag and the largest bag, the lanes sharing the list
  int bad = nb + 1;
  long long mx = 0;
  for (int b = lane; b < nb; b += 32) {
    const int64_t N = a.Ns[e0 + b];
    const float* X = a.Xs[e0 + b];
    const bool misaligned = gen ? !gen_bag_aligned(X, a.D) : (reinterpret_cast<uintptr_t>(X) & 15) != 0;
    if ((N < 1 || N > a.max_rows || X == nullptr || misaligned) && b + 1 < bad)
      bad = b + 1;
    mx = N > mx ? N : mx;
  }
  for (int o = 16; o > 0; o >>= 1) {
    const int ob = __shfl_xor_sync(0xffffffffu, bad, o);
    const long long om = __shfl_xor_sync(0xffffffffu, mx, o);
    bad = ob < bad ? ob : bad;
    mx = om > mx ? om : mx;
  }
  if (bad > nb) bad = 0;
  if (bad) {
    if (lane == 0) a.status[m] = bad;
    for (int i = lane; i < a.D; i += 32) a.zero_row[i] = 0.f;
    mx = 1;
  }
  const BagList L{a.Xs + e0, a.Ns + e0, bad ? a.zero_row : nullptr};
  long long total = 0;
  if (lane == 0) {
    int tiles = 0, recs = 0;
    for (int b = 0; b < nb; ++b) {
      const int64_t N = L.N(b);
      total += N;
      tiles += tiles_for_bag(N);
      recs += gen ? attend_ctas(N) : recs_for_bag(N);
    }
    s_cnt[TILES][m] = tiles;
    s_cnt[RECS][m] = recs;
    if (a.live) a.live[m] = FoldLive{total, tiles};
  }
  total = __shfl_sync(0xffffffffu, total, 0);
  const ModelSplits sp = model_splits(a.C, a.D, nb, total, mx);
  if (lane == 0) {
    s_cnt[NCI][m] = bwd ? rag_chunks_list(L, nb, a.D, sp.rps_i, 0, nullptr) : 0;
    s_cnt[NC1][m] = bwd ? rag_chunks_list(L, nb, a.D, sp.rps_1, 0, nullptr) : 0;
    s_cnt[NC2][m] = bwd ? sp.t2.S : 0;
    s_cnt[NCS][m] = bwd ? sp.cs.S : 0;
  }
  __syncthreads();
  int at[NCNT], all[NCNT];   // this model's first index of each numbering, and the totals
  for (int i = 0; i < NCNT; ++i) {
    at[i] = all[i] = 0;
    for (int j = 0; j < M; ++j) {
      if (j < m) at[i] += s_cnt[i][j];
      all[i] += s_cnt[i][j];
    }
  }
  if (threadIdx.x == 0) *a.plan = ModelsPlan{all[TILES], all[RECS], all[NCI], all[NC1], all[NC2], all[NCS]};
  if (a.ftable && lane == 0) {
    long long row = cap0;
    int tile = a.gen == FOLD_GEN_QMLP ? 0 : at[TILES], rec = at[RECS];
    for (int b = 0; b < nb; ++b) {
      sm90::BagDev e;
      if (gen) {
        e = gen_bag_entry(L.X(b), L.N(b), a.D, row, tile, rec);
        e.pad_ = fold_pad(e.pad_, m);
      } else {
        e = bag_entry(L.X(b), L.N(b), row, tile, rec);
        e.pad_ = m;
      }
      a.ftable[e0 + b] = e;
    }
    a.fmodels[m] = a.m[m].w;
  }
  if (!bwd) return;
  if (lane == 0) {
    const PlanModel& pm = a.m[m];
    long long row = cap0;
    for (int b = 0; b < nb; ++b) {
      a.btable[e0 + b] = sm90::BagDev{L.X(b), L.N(b), row, sp.G, (e0 + b) * a.Gcap, 0, m};
      row += L.N(b);
    }
    rag_chunks_list(L, nb, a.D, sp.rps_i, cap0, a.chi + at[NCI]);
    rag_chunks_list(L, nb, a.D, sp.rps_1, cap0, a.ch1 + at[NC1]);
    a.bmodels[m] = BwdModelDev{pm.w.Wf, pm.w.Wi, pm.gWf, pm.gbf, nullptr, e0, nb, cap0};
    a.segs[0 * M + m] = SumSeg{a.dc ? pm.gWi : nullptr, at[NCI], s_cnt[NCI][m]};
    a.segs[1 * M + m] = SumSeg{a.dc ? pm.gbi : nullptr, at[NCS], sp.cs.S};
    a.segs[2 * M + m] = SumSeg{pm.gW2, at[NC2], sp.t2.S};
    a.segs[3 * M + m] = SumSeg{pm.gb2, at[NCS], sp.cs.S};
    a.segs[4 * M + m] = SumSeg{pm.gW1, at[NC1], s_cnt[NC1][m]};
    a.segs[5 * M + m] = SumSeg{pm.gb1, at[NCS], sp.cs.S};
    a.lin[m] = LinSeg{a.dz2 + cap0 * kQ, pm.w.W2, a.H1 ? a.H1 + cap0 * kQ : nullptr, a.dz1 + cap0 * kQ, total};
    a.lin[M + m] = LinSeg{a.dz1 + cap0 * kQ, pm.w.W1, nullptr, nullptr, total};
  }
  for (int z = lane; z < sp.t2.S; z += 32) a.ch2[at[NC2] + z] = split_chunk(sp.t2, z, cap0, a.H1, kQ);
  for (int z = lane; z < sp.cs.S; z += 32) a.chc[at[NCS] + z] = split_chunk(sp.cs, z, cap0, nullptr, 0);
  // k_colsum_rag runs on the capacity grid: the chunks past the live ones are empty (their partial is not read)
  for (int z = all[NCS] + threadIdx.x; z < a.ncs_cap; z += blockDim.x) a.chc[z] = TnChunk{nullptr, 0, 0};
}

}  // namespace dsmil
