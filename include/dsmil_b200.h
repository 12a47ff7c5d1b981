/*
 * dsmil_b200.h -- C ABI of libdsmil_b200.so: the DSMIL per-slide aggregator hot path on H100 (sm_90a).
 *
 * The reference (binli123/dsmil-wsi) is pure Python/PyTorch and has no FFI of its own; the
 * "interface" each entry point replaces is therefore a span of reference Python, cited per
 * function as file:line into the reference repo.  INTEGRATION.md shows the ctypes binding a
 * maintainer adds (it is the one dsmil_wsi_b200/_lib.py ships).
 *
 * Conventions
 *  - Every pointer named *_dev / documented "device" is a CUDA device pointer on the CURRENT
 *    device; the library never allocates per call: the caller (PyTorch's caching allocator in
 *    our host mirror) owns every buffer including the workspace.
 *  - All tensors are fp32, row-major, contiguous.  Indices are int64.
 *  - Calls are asynchronous on `stream` (a cudaStream_t passed as void*); no host sync inside.
 *  - Return value: 0 on success, a negative dsmil_status_t otherwise; dsmil_last_error() gives
 *    a thread-local message (CUDA error string included).
 *  - No CPU fallback exists: without a CUDA device every compute entry point returns
 *    DSMIL_ERR_CUDA.
 */
#ifndef DSMIL_B200_H_
#define DSMIL_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DSMIL_ABI_VERSION 1
#define DSMIL_Q 128      /* query width, hard-coded in the reference: dsmil.py:31,33 */
#define DSMIL_MAX_C 8    /* output classes supported by the fused kernels (reference uses 1, 2) */
#define DSMIL_MAX_D 4096 /* feature size bound (reference: 166/230/512/1024/2048) */

typedef enum dsmil_status {
  DSMIL_OK = 0,
  DSMIL_ERR_ARG = -1,       /* bad shape / null pointer / unsupported size */
  DSMIL_ERR_WORKSPACE = -2, /* workspace too small */
  DSMIL_ERR_CUDA = -3,      /* CUDA runtime error (see dsmil_last_error) */
  DSMIL_ERR_EMPTY = -4      /* N == 0 on a single-device forward (reference raises IndexError) */
} dsmil_status_t;

/* Parameter block == the state_dict of MILNet(FCLayer|IClassifier, BClassifier)
 * (dsmil.py:6-12,14-25,27-44; key names in SURVEY.md §8 a3).  Device pointers. */
typedef struct dsmil_params {
  int32_t D;         /* input_size / feature_size */
  int32_t C;         /* output_class */
  int32_t nonlinear; /* 1: q = Linear(D,128)-ReLU-Linear(128,128)-Tanh (dsmil.py:31); 0: Linear(D,128) (:33) */
  int32_t passing_v; /* 1: v = Dropout-Linear(D,D)-ReLU (dsmil.py:35-39); 0: Identity (:41) */
  const float* Wi;   /* [C,D]    i_classifier.fc(.0).weight */
  const float* bi;   /* [C]      i_classifier.fc(.0).bias   */
  const float* W1;   /* [128,D]  b_classifier.q.0.weight  (or q.weight when !nonlinear) */
  const float* b1;   /* [128] */
  const float* W2;   /* [128,128] b_classifier.q.2.weight (NULL when !nonlinear) */
  const float* b2;   /* [128] */
  const float* Wv;   /* [D,D]    b_classifier.v.1.weight  (NULL when !passing_v) */
  const float* bv;   /* [D] */
  const float* Wf;   /* [C,C,D]  b_classifier.fcc.weight (Conv1d(C,C,kernel_size=D), dsmil.py:44) */
  const float* bf;   /* [C] */
} dsmil_params_t;

/* Gradient block: same shapes as dsmil_params_t's tensors; device pointers, OVERWRITTEN
 * (not accumulated).  Any pointer may be NULL to skip that gradient. */
typedef struct dsmil_grads {
  float* gWi; float* gbi;
  float* gW1; float* gb1;
  float* gW2; float* gb2;
  float* gWv; float* gbv;
  float* gWf; float* gbf;
  float* gX;  /* [N,D] gradient w.r.t. the features, NULL unless the caller needs it */
} dsmil_grads_t;

int dsmil_abi_version(void);
const char* dsmil_last_error(void);
/* Number of kernels this library has launched in this process (bench.py's gpu_launches). */
uint64_t dsmil_launch_count(void);
/* Caller-side bag feed (SURVEY 8f-1): `feats[random_indices]` of dropout_patches (train_tcga.py:78-83) as a
 * device row gather: out[m,:] = X[idx[m],:], idx int64 on the device, rows in [0,N). */
int dsmil_gather_rows(const float* X, int64_t N, int32_t D, const int64_t* idx, int64_t M, float* out, void* stream);

/* Patch pre-processing of the embedding loop (compute_feats.py:19-46,72: PIL image -> VF.to_tensor ->
 * .float().cuda()): uint8 HWC patches [B,H,W,Cc] (device) -> float32 CHW [B,Cc,H,W] = value / 255. */
int dsmil_patches_u8_to_f32(const uint8_t* in, int64_t B, int32_t H, int32_t W, int32_t Cc, float* out, void* stream);

/* Backbone of the embedding loop (compute_feats.py:146-170 builds a torchvision ResNet with norm_layer =
 * nn.InstanceNorm2d, dsmil.py:21-25 runs it): after every convolution the reference executes instance_norm ->
 * (+ identity) -> relu as separate passes.  One pass here:  y = [relu]( instance_norm(x) [+ residual] )  over
 * `planes` = N*C planes of HW contiguous fp32 elements (NCHW), biased variance, eps as given, no affine parameters and
 * no running statistics (the nn.InstanceNorm2d defaults the reference uses).  residual may be NULL; y == x is allowed.
 * HW <= 16384. */
int dsmil_instnorm_act(const float* x, const float* residual, float* y, int64_t planes, int32_t HW, float eps,
                       int32_t relu, void* stream);
/* The same operator on channels-last memory, [N][HW][C] fp32 (torch.channels_last: the layout the embedding loop
 * runs this backbone's cuDNN convolutions in).  C a multiple of 32; statistics per (sample, channel) over HW. */
int dsmil_instnorm_act_nhwc(const float* x, const float* residual, float* y, int64_t N, int32_t HW, int32_t C, float eps,
                            int32_t relu, void* stream);

/* Patch loader of the embedding loop on the device (compute_feats.py:26-29 `Image.open(path)` + `VF.to_tensor`,
 * executed by 4 DataLoader workers, compute_feats.py:55): a batch of n JPEG FILES, stored back to back in `blob`
 * (device, blob_bytes long), is decoded to uint8 HWC [n,H,W,3] (== np.asarray(Image.open(f).convert("RGB"))) and / or
 * float32 CHW [n,3,H,W] (== VF.to_tensor of it; with f32_channels_last = 1 the same values in torch.channels_last
 * memory order [n,H,W,3], the layout the backbone's convolutions run fastest in), bit for bit what PIL's libjpeg produces with its defaults (ISLOW
 * IDCT, fancy upsampling).  `headers` = the n fixed-size records written by dsmil_jpeg_parse_batch of
 * libdsmil_host.so (include/dsmil_host.h), copied to the device; dsmil_jpeg_header_bytes_dev() is their size.
 * Decodable: baseline / extended-sequential Huffman, 8 bit, grey or YCbCr 4:4:4 / 4:2:2 / 4:2:0, one interleaved
 * scan, restart intervals allowed, every file H x W.  status[i] (device int32) = 0, -1 corrupt data, -2 a file the
 * parser marked unsupported or of another size (its output rows are left untouched).  Either output may be NULL.
 * Asynchronous on `stream`; workspace (256-byte aligned) of dsmil_jpeg_workspace_bytes(n, H, W, blob_bytes). */
int32_t dsmil_jpeg_header_bytes_dev(void);
int64_t dsmil_jpeg_workspace_bytes(int32_t n, int32_t H, int32_t W, int64_t blob_bytes);
int dsmil_jpeg_decode_batch(const uint8_t* blob, int64_t blob_bytes, const void* headers, int32_t n, int32_t H, int32_t W,
                            uint8_t* out_u8, float* out_f32, int32_t f32_channels_last, int32_t* status, void* workspace,
                            int64_t workspace_bytes, void* stream);

/* Live per-kernel timing for the roofline report (bench.py): when enabled, tagged launches are
 * bracketed by CUDA events on the launching stream.  dsmil_profile_read synchronises those events,
 * returns summed milliseconds and launch counts per tag (arrays of 8: 0 scores, 1 q-mlp, 2 attend,
 * 3 finalize, 4 fused wgmma kernel) and resets the log.  Not thread-safe; bench use only. */
int dsmil_profile_enable(int on);
int dsmil_profile_read(double* ms_per_tag, uint64_t* launches_per_tag);
/* Which kernel family the forward would use for (D,C): 1 = generic fp32 FFMA, 2 = sm_90a wgmma. */
int dsmil_forward_path(const dsmil_params_t* p, int64_t N);

/* ---- single-device forward ------------------------------------------------------------
 * Replaces MILNet.forward with an FCLayer/IClassifier.fc instance stream:
 *   dsmil.py:70-74 (composition), :10-12 / :24 (scores), :46-62 (aggregator).
 * in : X[N,D] device.  out: classes[N,C], pred[1,C], A[N,C], B[1,C,D], crit_idx[C] (the row
 * dsmil.py:52-53 selects; lowest index on ties).  save_Q[N,128] / save_H1[N,128] /
 * save_V[N,D] are optional (NULL) buffers that keep the activations backward needs.
 * x_for_v: when passing_v, the features AFTER the caller applied the dropout mask of
 * dsmil.py:36 (NULL = same as X, i.e. eval mode or p=0). */
size_t dsmil_forward_workspace_bytes(const dsmil_params_t* p, int64_t N);
int dsmil_forward(const dsmil_params_t* p, const float* X, const float* x_for_v, int64_t N,
                  float* classes, float* pred, float* A, float* B, int64_t* crit_idx,
                  float* save_Q, float* save_H1, float* save_V,
                  void* workspace, size_t workspace_bytes, void* stream);

/* A stream of bags in ONE call (throughput form of the same forward; slides/sec in BASELINE.json):
 * Xs[b] -> device features [Ns[b], D] (host arrays of nb entries).  Outputs are packed in bag order:
 * classes / A [sum N, C], pred [nb, C], B [nb, C, D], crit_idx [nb, C].  On the tensor-core path the
 * whole batch costs a handful of launches (one bag table); other shapes, and bags that are not
 * 16-byte aligned, loop. */
size_t dsmil_forward_bags_workspace_bytes(const dsmil_params_t* p, const int64_t* Ns, int32_t nb);
int dsmil_forward_bags(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                       float* classes, float* pred, float* A, float* B, int64_t* crit_idx,
                       void* workspace, size_t workspace_bytes, void* stream);

/* Training form of dsmil_forward_bags: the same packed outputs, plus save_Q [sum N,128] (after the tanh) and, for a
 * nonlinear q, save_H1 [sum N,128], packed in bag order -- what dsmil_backward_bags needs.  crit_idx [nb,C] is
 * required; its entries are rows within each bag.  Identity v only (passing_v: DSMIL_ERR_ARG).  Shapes or bags off
 * the tensor-core batch loop per bag (as dsmil_forward_bags does) into the same packed buffers. */
size_t dsmil_forward_bags_train_workspace_bytes(const dsmil_params_t* p, const int64_t* Ns, int32_t nb);
int dsmil_forward_bags_train(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                             float* classes, float* pred, float* A, float* B, int64_t* crit_idx,
                             float* save_Q, float* save_H1, void* workspace, size_t workspace_bytes, void* stream);
/* Reverse of dsmil_forward_bags_train for all nb bags in one call.  Upstream gradients are packed like the outputs:
 * d_classes / d_A [sum N,C], d_pred [nb,C], d_B [nb,C,D]; each may be NULL == zero.  grads->g* are SUMS over the
 * bags (overwritten; a loss that averages over bags carries its 1/nb itself); grads->gX, when non-NULL, is packed
 * [sum N,D].  Any D and C of dsmil_backward and any alignment of the bags; identity v only.  Deterministic: no
 * float atomics, fixed-order split sums. */
size_t dsmil_backward_bags_workspace_bytes(const dsmil_params_t* p, const int64_t* Ns, int32_t nb, int need_gX);
int dsmil_backward_bags(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                        const float* Q, const float* H1, const float* A, const float* B, const int64_t* crit_idx,
                        const float* d_classes, const float* d_pred, const float* d_A, const float* d_B,
                        const dsmil_grads_t* grads, void* workspace, size_t workspace_bytes, void* stream);

/* Capture-safe forms of dsmil_forward_bags_train / dsmil_backward_bags, for a training step recorded once as a CUDA
 * graph and replayed over batches of different bag sizes.  The bag list is in DEVICE memory: Xs_dev [nb] feature
 * pointers, Ns_dev [nb] row counts.  max_rows is the per-bag row capacity: classes, A, save_Q and save_H1 (and
 * d_classes) are sized for nb * max_rows rows, and hold the live rows packed in bag order at the live prefix sums, as
 * the eager calls pack them.  Each call only enqueues work on `stream` (no host<->device copy, allocation or
 * synchronisation, nothing read from Ns on the host): one recorded call serves every batch of nb bags with
 * 1 <= Ns[b] <= max_rows.  A small planner kernel at the start of each call reads the bag list and writes the bag
 * table and the live counts into the workspace.  A bag with N outside [1, max_rows], or features that are NULL or not
 * 16-byte aligned, sets *status (device int32) to 1 + the first such bag's index, and the call then computes a stand-in
 * batch in which every bag is one row of zeros: every output is finite and every index in range (crit_idx 0, pred =
 * bf, B 0, row b of the packed outputs is bag b's), but none is the batch's, and a caller must discard what it derives
 * from them.  A status is never cleared by the library: the caller zeroes it and reads it when it synchronises.  The forward builds
 * the W1/W2 weight images on every call, so a replay after an optimizer step uses the current weights.
 * Shapes: those of dsmil_shard_bags_supported (identity v).  Gradients through classes and pred only: d_A, d_B and
 * grads->gX must be NULL (DSMIL_ERR_ARG).  On the same bags the results are the eager calls' bits.
 * 1 <= nb <= 65535, max_rows >= 1; a short workspace is DSMIL_ERR_WORKSPACE.  The workspace sizes depend on
 * (nb, max_rows) only and are never below the eager calls' for nb bags of max_rows rows. */
size_t dsmil_forward_bags_train_dev_workspace_bytes(const dsmil_params_t* p, int32_t nb, int64_t max_rows);
int dsmil_forward_bags_train_dev(const dsmil_params_t* p, const float* const* Xs_dev, const int64_t* Ns_dev,
                                 int32_t nb, int64_t max_rows, float* classes, float* pred, float* A, float* B,
                                 int64_t* crit_idx, float* save_Q, float* save_H1, int32_t* status, void* workspace,
                                 size_t workspace_bytes, void* stream);
size_t dsmil_backward_bags_dev_workspace_bytes(const dsmil_params_t* p, int32_t nb, int64_t max_rows);
int dsmil_backward_bags_dev(const dsmil_params_t* p, const float* const* Xs_dev, const int64_t* Ns_dev, int32_t nb,
                            int64_t max_rows, const float* Q, const float* H1, const float* A, const float* B,
                            const int64_t* crit_idx, const float* d_classes, const float* d_pred, const float* d_A,
                            const float* d_B, const dsmil_grads_t* grads, int32_t* status, void* workspace,
                            size_t workspace_bytes, void* stream);

/* Call form (2)+(3) of the boundary (SURVEY §8b): the callers in attention_map.py:74,85 /
 * testing_tcga.py:72,83 run the instance classifier and the bag classifier separately.
 * dsmil_instance_scores == IClassifier.fc / FCLayer.fc (dsmil.py:11,24).
 * dsmil_bag_forward     == BClassifier.forward(feats, c) (dsmil.py:46-62) on GIVEN scores c. */
int dsmil_instance_scores(const dsmil_params_t* p, const float* X, int64_t N, float* classes, void* stream);
/* Reverse of dsmil_instance_scores: gWi[C,D] = d_classes^T X, gbi[C] = column sums, and
 * (optional) gX[N,D] = d_classes Wi.  Workspace: dsmil_backward_workspace_bytes(p, N, 0). */
int dsmil_instance_scores_backward(const dsmil_params_t* p, const float* X, int64_t N, const float* d_classes,
                                   float* gWi, float* gbi, float* gX,
                                   void* workspace, size_t workspace_bytes, void* stream);
int dsmil_bag_forward(const dsmil_params_t* p, const float* X, const float* x_for_v, const float* classes_in,
                      int64_t N, float* pred, float* A, float* B, int64_t* crit_idx,
                      float* save_Q, float* save_H1, float* save_V,
                      void* workspace, size_t workspace_bytes, void* stream);

/* ---- single-device backward ------------------------------------------------------------
 * Reverse of dsmil_forward for upstream gradients d_classes[N,C], d_pred[C], d_A[N,C],
 * d_B[C,Dv] (each may be NULL == zero).  This is what autograd does through dsmil.py:46-62
 * for the callers' loss (train_tcga.py:67-72, train_mil.py:50-56); arg-max indices are
 * non-differentiable, q_max shares the rows of Q.  Needs the forward's saved Q, H1, V, A, B,
 * crit_idx. */
size_t dsmil_backward_workspace_bytes(const dsmil_params_t* p, int64_t N, int need_gX);
int dsmil_backward(const dsmil_params_t* p, const float* X, const float* x_for_v, int64_t N,
                   const float* Q, const float* H1, const float* V, const float* A, const float* B,
                   const int64_t* crit_idx,
                   const float* d_classes, const float* d_pred, const float* d_A, const float* d_B,
                   const dsmil_grads_t* grads, const float* v_mask,
                   void* workspace, size_t workspace_bytes, void* stream);

/* ---- row-sharded forward (one giant bag over G ranks; SURVEY §8e, Appendix A.3) -----------
 * Each rank owns rows [row_offset, row_offset+N_local).  Two exchange steps (all-gather of a
 * few KB, done by the caller with NCCL between the phases):
 *   phase1 -> cand record   [dsmil_cand_floats(C)]  = idx[C] (int64 bits) | score[C] | qrow[C,128] | pad to 4
 *   merge_candidates(G records) -> q_max[C,128], crit_idx[C]
 *   phase2 -> partial record [dsmil_rec_floats(C,Dv)] = m[C] | s[C] | Bpartial[C,Dv] | pad to 4
 *   merge_partials(G records)  -> global record
 *   phase3 -> A (normalised, local rows), B[1,C,Dv], pred[1,C] (replicated)
 * N_local may be 0 on a rank.  dsmil_forward == these five calls with G == 1. */
size_t dsmil_cand_floats(int32_t C);
size_t dsmil_rec_floats(int32_t C, int32_t Dv);
size_t dsmil_shard_workspace_bytes(const dsmil_params_t* p, int64_t N_local);
int dsmil_shard_phase1(const dsmil_params_t* p, const float* X, const float* x_for_v, const float* classes_in,
                       int64_t N_local, int64_t row_offset,
                       float* classes, float* Q, float* H1, float* V, float* cand_rec,
                       void* workspace, size_t workspace_bytes, void* stream);
int dsmil_shard_merge_candidates(int32_t C, const float* cand_recs, int32_t G, float* q_max, int64_t* crit_idx,
                                 void* stream);
int dsmil_shard_phase2(const dsmil_params_t* p, const float* Xv, const float* Q, int64_t N_local,
                       const float* q_max, float* A_logits, float* rec,
                       void* workspace, size_t workspace_bytes, void* stream);
int dsmil_shard_merge_partials(int32_t C, int32_t Dv, const float* recs, int32_t G, float* rec_out, void* stream);
int dsmil_shard_phase3(const dsmil_params_t* p, int64_t N_local, const float* rec_global,
                       float* A, float* B, float* pred, void* stream);

/* ---- row-sharded backward (SURVEY §8e "Backward", Appendix A.2 "Sharded"; identity v only) -----------
 * Reverse pass of the sharded forward for the callers' loss (train_tcga.py:67-72): each rank keeps its rows of
 * X, Q, H1 (saved by dsmil_shard_phase1), the normalised A of phase3 and the replicated B, q_max, crit_idx.
 * Three reductions, done by the caller with NCCL all-reduce(sum) between the phases:
 *   phase1: replicated gWf/gbf (not reduced), local partial gWi/gbi, dA_local[N,C], t_local[C] = sum_n A.dA
 *           -> all-reduce t (C floats)
 *   phase2: dA_local becomes dL_local in place (softmax-over-instances backward with the global t),
 *           dqm_local[C,128] = dL^T Q  -> all-reduce dqm (C*128 floats)
 *   phase3: MLP backward over the local rows; the critical rows' share dqm is added on the rank that owns
 *           row crit_idx[k] (global index - row_offset); local partial gW1/gb1(/gW2/gb2)
 *           -> all-reduce of the parameter gradients
 * d_classes_local may be NULL (no gradient through the instance scores).  N_local may be 0 (all outputs
 * zero).  Workspace: dsmil_backward_workspace_bytes(p, N_local, 0).  dsmil_backward == these three calls with
 * one rank. */
int dsmil_shard_backward_phase1(const dsmil_params_t* p, const float* X, int64_t N_local, const float* A,
                                const float* B, const float* d_classes_local, const float* d_pred,
                                float* dA_local, float* t_local, float* gWi, float* gbi, float* gWf, float* gbf,
                                void* workspace, size_t workspace_bytes, void* stream);
int dsmil_shard_backward_phase2(const dsmil_params_t* p, int64_t N_local, const float* A, float* dA_to_dL,
                                const float* t_global, const float* Q, float* dqm_local,
                                void* workspace, size_t workspace_bytes, void* stream);
int dsmil_shard_backward_phase3(const dsmil_params_t* p, const float* X, int64_t N_local, int64_t row_offset,
                                const float* Q, const float* H1, const float* dL_local, const float* dqm_global,
                                const float* q_max, const int64_t* crit_idx,
                                float* gW1, float* gb1, float* gW2, float* gb2,
                                void* workspace, size_t workspace_bytes, void* stream);

/* The same three phases for a BATCH of row-sharded bags (tensor-core path; dsmil_shard_bags_supported):
 * every rank passes its local rows of all nb bags; records are packed per bag so that a whole step costs
 * two all-gathers.  Xs/Ns/row_offsets are host arrays; the workspace must be the same buffer in all three
 * calls (it carries Q, the bag table and the per-tile partial records between the phases).
 *   phase1 -> classes (packed), cand_recs [nb][dsmil_cand_floats(C)]
 *   phase2 (cands_all [G][nb][cand]) -> A (logits, packed), crit_idx [nb][C], recs_out [nb][dsmil_rec_floats(C,D)]
 *   phase3 (recs_all  [G][nb][rec])  -> A normalised, B [nb][C][D], pred [nb][C] */
int dsmil_shard_bags_supported(const dsmil_params_t* p);
size_t dsmil_shard_bags_workspace_bytes(const dsmil_params_t* p, const int64_t* Ns, int32_t nb);
int dsmil_shard_bags_phase1(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                            const int64_t* row_offsets, float* classes, float* cand_recs,
                            void* workspace, size_t workspace_bytes, void* stream);
int dsmil_shard_bags_phase2(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                            const float* cands_all, int32_t G, float* A, int64_t* crit_idx, float* recs_out,
                            void* workspace, size_t workspace_bytes, void* stream);
int dsmil_shard_bags_phase3(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                            const float* recs_all, int32_t G, float* A, float* B, float* pred,
                            void* workspace, size_t workspace_bytes, void* stream);

/* ---- row-sharded batch training (identity v; dsmil_shard_bags_supported shapes) -------------------------------------
 * A minibatch of row-sharded bags in 3 + 3 library calls and 6 collectives per step, whatever nb: 2 all-gathers in the
 * forward, all-reduce(max) of nb*C floats in the callers' loss, 3 all-reduce(sum) in the backward.
 *
 * Forward: dsmil_shard_bags_phase1_train, then dsmil_shard_bags_phase2_train, then the inference dsmil_shard_bags_phase3
 * unchanged.  The training phases carve the workspace (dsmil_shard_bags_workspace_bytes) exactly as the inference
 * phases do, so phase 3 finishes the step from it.  The differences:
 *   phase1_train keeps Q (after the tanh) and H1 row-major in the caller's save_Q / save_H1, packed [sum N_local, 128]
 *   phase2_train attends on that Q and also returns the merged q_max [nb][C][128]; crit_idx [nb][C] holds GLOBAL rows
 *   (row within the whole bag), as dsmil_shard_bags_phase2.
 * Every bag must hold at least one local row on every rank (else DSMIL_ERR_EMPTY); 1 <= nb <= 65535.
 *
 * Backward: three phases with the caller's all-reduce(sum) between them.  One workspace of
 * dsmil_shard_backward_bags_workspace_bytes for all three calls of a step (phase 1 leaves the bag and chunk tables in
 * it for phases 2 and 3).  Per-row buffers are packed [sum N_local, *] in bag order, as dsmil_backward_bags; parameter
 * gradients are sums over the bags, overwritten.
 *   phase1: dA_local [sum N,C]; t_local [nb][C] (per-bag sum_n A.dA over the local rows, in a fixed order); gWf/gbf
 *           replicated (no reduction); local partial gWi/gbi (d_classes_local may be NULL; any gradient buffer may be
 *           NULL == not wanted)                                       -> all-reduce t (nb*C floats)
 *   phase2: dA becomes dL in place with the global t; dqm_local [nb][C][128] -> all-reduce dqm
 *   phase3: Q-MLP backward over the local rows; the dq_max share goes to the rank that holds row crit_idx[b][k]
 *           (global) - row_offsets[b]; q_max is phase2_train's; local partial gW1/gb1/gW2/gb2
 *                                                                     -> all-reduce the parameter gradients
 * With one rank (identity reductions) the three phases give dsmil_backward_bags's bits.  No gX and no upstream d_A/d_B. */
int dsmil_shard_bags_phase1_train(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                                  const int64_t* row_offsets, float* classes, float* save_Q, float* save_H1,
                                  float* cand_recs, void* workspace, size_t workspace_bytes, void* stream);
int dsmil_shard_bags_phase2_train(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                                  const float* Q, const float* cands_all, int32_t G, float* A, int64_t* crit_idx,
                                  float* q_max, float* recs_out, void* workspace, size_t workspace_bytes,
                                  void* stream);
size_t dsmil_shard_backward_bags_workspace_bytes(const dsmil_params_t* p, const int64_t* Ns, int32_t nb);
int dsmil_shard_backward_bags_phase1(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                                     const float* A, const float* B, const float* d_classes_local,
                                     const float* d_pred, float* dA_local, float* t_local, float* gWi, float* gbi,
                                     float* gWf, float* gbf, void* workspace, size_t workspace_bytes, void* stream);
int dsmil_shard_backward_bags_phase2(const dsmil_params_t* p, const int64_t* Ns, int32_t nb, const float* A,
                                     float* dA_to_dL, const float* t_global, const float* Q, float* dqm_local,
                                     void* workspace, size_t workspace_bytes, void* stream);
int dsmil_shard_backward_bags_phase3(const dsmil_params_t* p, const float* const* Xs, const int64_t* Ns, int32_t nb,
                                     const int64_t* row_offsets, const float* Q, const float* H1, const float* dL_local,
                                     const float* dqm_global, const float* q_max, const int64_t* crit_idx,
                                     float* gW1, float* gb1, float* gW2, float* gb2, void* workspace,
                                     size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DSMIL_B200_H_ */
