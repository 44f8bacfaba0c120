/* libesac_b200.so -- C ABI of the CUDA (H100, sm_90a) ESAC differentiable-RANSAC hot path.
 *
 * Drop-in boundary for the reference's `esac` Python extension
 * (code/esac/esac.cpp:513-516: m.def("forward", &esac_forward), m.def("backward",
 * &esac_backward)).  esacb200_forward / esacb200_backward take exactly the arguments of
 * esac_forward (esac.cpp:64-77) / esac_backward (esac.cpp:213-230) with the at::Tensor arguments
 * flattened to pointer + sizes; everything else in this header is additive (context handling,
 * seeding, a scoring-only entry for measurement, read-back of intermediates for tests).
 *
 * Conventions
 *  - plain C types only, no exceptions across the boundary; every entry returns 0 on success or a
 *    negative esacb200_status, and esacb200_last_error(ctx) holds a message;
 *  - `coords`, `grads`, `assign`, `out_pose`, `gt_pose` may be HOST or DEVICE pointers (detected with
 *    cudaPointerGetAttributes); host buffers are copied on the context's stream (pinned memory gets
 *    full PCIe speed), device buffers are used in place;
 *  - calls are synchronous like the reference's (they return an int / a double), the work is enqueued
 *    on the stream set with esacb200_set_stream (default: a stream owned by the context);
 *  - there is NO CPU fallback: without a CUDA device esacb200_create fails.
 */
#ifndef ESAC_B200_H
#define ESAC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct esacb200_ctx esacb200_ctx;

typedef enum {
    ESACB200_OK = 0,
    ESACB200_ERR_CUDA = -1,       /* a CUDA runtime call failed */
    ESACB200_ERR_ARG = -2,        /* bad size / null pointer / expert index out of range */
    ESACB200_ERR_NO_DEVICE = -3   /* no usable CUDA device */
} esacb200_status;

/* ---- context -------------------------------------------------------------------------------- */
/* Replaces the reference's only persistent state, the static per-thread RNG
 * (thread_rand.cpp:4-5,13-30; default seeds 1305 + thread id). */
int esacb200_create(int device, esacb200_ctx** out);
void esacb200_destroy(esacb200_ctx* ctx);
const char* esacb200_last_error(const esacb200_ctx* ctx);
/* cudaStream_t to enqueue on (0 / NULL = the context's own stream). */
int esacb200_set_stream(esacb200_ctx* ctx, void* cuda_stream);
/* Seed of the minimal-set stream; also resets the call counter (each forward/backward call advances
 * it so successive calls draw fresh samples, as the reference's persistent generators do). */
int esacb200_set_seed(esacb200_ctx* ctx, uint64_t seed);
/* Options: "max_tries" (esac.cpp:44 MAX_SAMPLING_TRIES, default 1000000), "max_ref_steps"
 * (esac.cpp:45 MAX_REF_STEPS, default 100), "fixed_seed" (1: do not advance the call counter),
 * "refine_group" (CTAs per refinement job, 0 = automatic), "refine_jobs_per_group" (jobs a group
 * works through when many hypotheses are refined), "refine_profile", "sample_prefilter" (default 1; 0 sends every sampling
 * try through the exact fp64 path -- the results must not change, only the time), "sample_hint" (default 0.95, 0 = off,
 * below 2: a try whose 4th point the float prefilter puts within this fraction of tau stops the prefiltering of the later
 * tries of its window -- the results must not change, only the time), "hyp_offset" (global index of
 * local hypothesis 0 for the minimal-set stream; sharded runs), "score_ppt" / "score_hc" (scoring launch shape). */
int esacb200_set_option(esacb200_ctx* ctx, const char* key, double value);
/* Inject minimal sets instead of drawing them: cells int32 [M][T][4][2] (x, y), host pointer,
 * copied; T candidate sets per hypothesis tried in order.  NULL clears.  Applies to the next call. */
int esacb200_inject_cells(esacb200_ctx* ctx, const int32_t* cells, int M, int T);

/* ---- the reference's two entry points ------------------------------------------------------- */
/* esac_forward (esac.cpp:64-190).  coords float32 [E,3,H,W] contiguous; assign int64 [M] with element
 * stride `assign_stride` (0 for the reference's expert.expand() tensors, test_esac.py:173); out_pose
 * float32 [4,4] camera->world, written in place; *out_expert = winning expert index (the reference's
 * return value). */
int esacb200_forward(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                     int64_t assign_stride, int M, float* out_pose, int shiftX, int shiftY, float focalLength,
                     float ppointX, float ppointY, float inlierThreshold, float inlierAlpha, float inlierBeta,
                     float maxReproj, int subSampling, int* out_expert);

/* esac_backward (esac.cpp:213-511).  grads float32 [E,3,H,W] is ACCUMULATED in place (+=, esac.cpp:501-506);
 * gt_pose float32 [4,4] camera->world; *out_loss = expected pose loss (the reference's return value). */
int esacb200_backward(esacb200_ctx* ctx, const float* coords, float* grads, int E, int H, int W,
                      const int64_t* assign, int64_t assign_stride, int M, const float* gt_pose, float wLossRot,
                      float wLossTrans, float lossCut, int shiftX, int shiftY, float focalLength, float ppointX,
                      float ppointY, float inlierThreshold, float inlierAlpha, float inlierBeta, float maxReproj,
                      int subSampling, double* out_loss);

/* The hypotheses of esac_backward as a differentiable function, for a pose loss of the caller's choice.
 *
 * esacb200_hypotheses_forward draws, scores and refines exactly what an esacb200_backward call at the same point of the
 * context's call sequence would (same seed use), and writes
 *   out_scores  double [M]    the soft-inlier scores the softmax sees,
 *   out_poses6  double [M,6]  scene pose (rvec, tvec) per hypothesis: refined where p >= PROB_THRESH, initial elsewhere,
 *   out_contrib uint8  [M]    1 where p >= PROB_THRESH (the hypotheses the backward differentiates);
 * p being the hypothesis's softmax probability.  The _floor variants take that threshold as `min_prob` in [0, 1] (NaN or a
 * value outside fails with ESACB200_ERR_ARG before anything is enqueued): exactly the hypotheses with !(p < min_prob) are
 * refined, flagged and differentiated, so min_prob = 0 takes all M, also those whose p underflows to 0.  The entries
 * without the suffix are the _floor ones with min_prob = ESACB200_PROB_THRESH, the reference's own truncation, which is
 * right for its loss softmax(scores) . loss and loses the gradient of any hypothesis below it under other losses
 * (best-of-M, a sharper softmax, a per-hypothesis term).
 * host or device pointers.  Everything its backward needs goes to `tape`: 16-byte aligned device memory of at least
 * esacb200_hypotheses_tape_bytes(E, H, W, M) bytes, owned by the caller and untouched by any other call, so other library
 * calls may run between a forward and its backward.  Returns 0 for non-positive or oversized arguments.
 *
 * esacb200_hypotheses_backward ACCUMULATES (+=) into grads float32 [E,3,H,W] the vector-Jacobian product
 *   sum_h d_scores[h] * d score_h / d coords + d_poses6[h] . d pose_h / d coords
 * over the contributing hypotheses (the reference's truncation; pose_h linearised through the refinement, both > 10 clamps
 * kept).  d_scores double [M] and d_poses6 double [M,6] are host or device pointers; NULL counts as zero.  coords must hold
 * the values the forward saw (host maps are staged again).  A tape may be used by any number of backwards. */
size_t esacb200_hypotheses_tape_bytes(int E, int H, int W, int M);
int esacb200_hypotheses_forward(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                                int64_t assign_stride, int M, int shiftX, int shiftY, float focalLength, float ppointX,
                                float ppointY, float inlierThreshold, float inlierAlpha, float inlierBeta, float maxReproj,
                                int subSampling, void* tape, size_t tape_bytes, double* out_scores, double* out_poses6,
                                uint8_t* out_contrib);
int esacb200_hypotheses_backward(esacb200_ctx* ctx, const void* tape, const float* coords, float* grads, int E, int H, int W,
                                 const double* d_scores, const double* d_poses6);
/* The reference's probability threshold (esac_derivative.h PROB_THRESH): the default floor of the hypotheses node. */
#define ESACB200_PROB_THRESH 0.001
int esacb200_hypotheses_forward_floor(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                                      int64_t assign_stride, int M, int shiftX, int shiftY, float focalLength, float ppointX,
                                      float ppointY, float inlierThreshold, float inlierAlpha, float inlierBeta,
                                      float maxReproj, int subSampling, double min_prob, void* tape, size_t tape_bytes,
                                      double* out_scores, double* out_poses6, uint8_t* out_contrib);

/* The reference's pose loss (esac_loss.h loss) and its dLoss, quirks included, of M scene poses (rvec, tvec) double [M,6]
 * against a float32 [4,4] camera->world ground truth: out_losses double [M], out_dloss6 double [M,6].  Host or device
 * pointers; the arithmetic is esacb200_backward's. */
int esacb200_pose_loss(esacb200_ctx* ctx, int M, const double* poses6, const float* gt16, float wLossRot, float wLossTrans,
                       float lossCut, double* out_losses, double* out_dloss6);
/* esacb200_pose_loss over a batch, in one launch: poses6 double [B,M,6], image b against gt16[b] of float32 [B,4,4];
 * out_losses double [B,M], out_dloss6 double [B,M,6].  Row b is bitwise what esacb200_pose_loss on it gives, which is this
 * entry with B = 1.  No host synchronisation before the launch. */
int esacb200_pose_loss_batch(esacb200_ctx* ctx, int B, int M, const double* poses6, const float* gt16, float wLossRot,
                             float wLossTrans, float lossCut, double* out_losses, double* out_dloss6);

/* The hypotheses node over a ragged batch: every image-sized argument is a host array of B pointers (all device or all
 * host), H / W host int [B], shiftX / shiftY host int [B] or NULL (= 0), f / ppx / ppy host float [B].
 * esacb200_hypotheses_forward_ragged: image b draws, scores and refines what the b-th of B consecutive
 * esacb200_hypotheses_forward calls (or esacb200_backward calls) on the context would, with its own shift and camera, and
 * writes row b of out_scores double [B,M], out_poses6 double [B,M,6], out_contrib uint8 [B,M] (host or device).  tapes[b]
 * is 16-byte aligned device memory of tape_bytes[b] >= esacb200_hypotheses_tape_bytes(E, H[b], W[b], M) bytes.
 * esacb200_hypotheses_backward_ragged ACCUMULATES into grads[b] float32 [E,3,H[b],W[b]] what esacb200_hypotheses_backward
 * on tapes[b] with rows b of d_scores double [B,M] / d_poses6 double [B,M,6] (NULL = zero; M of the tapes) would add.
 * Images are spread over option "batch_workers" internal streams, as for esacb200_backward_batch; errors name the image. */
int esacb200_hypotheses_forward_ragged(esacb200_ctx* ctx, int B, const float* const* coords, const int* H, const int* W, int E,
                                       const int64_t* assign, int64_t assign_stride, int M, const int* shiftX, const int* shiftY,
                                       const float* f, const float* ppx, const float* ppy, float inlierThreshold,
                                       float inlierAlpha, float inlierBeta, float maxReproj, int subSampling,
                                       void* const* tapes, const size_t* tape_bytes, double* out_scores, double* out_poses6,
                                       uint8_t* out_contrib);
int esacb200_hypotheses_forward_ragged_floor(esacb200_ctx* ctx, int B, const float* const* coords, const int* H, const int* W,
                                             int E, const int64_t* assign, int64_t assign_stride, int M, const int* shiftX,
                                             const int* shiftY, const float* f, const float* ppx, const float* ppy,
                                             float inlierThreshold, float inlierAlpha, float inlierBeta, float maxReproj,
                                             int subSampling, double min_prob, void* const* tapes, const size_t* tape_bytes,
                                             double* out_scores, double* out_poses6, uint8_t* out_contrib);
int esacb200_hypotheses_backward_ragged(esacb200_ctx* ctx, int B, const void* const* tapes, const float* const* coords,
                                        float* const* grads, const int* H, const int* W, int E, const double* d_scores,
                                        const double* d_poses6);

/* ---- additive entry points ------------------------------------------------------------------ */
/* esac_backward over hypotheses sharded across processes (one per GPU; experts expert-major, so gradient slices are
 * disjoint).  The path has two exchange steps (SURVEY.md 8e); the library calls `exchange` on the host at each:
 *   phase 1: values = {local max score, local sum exp(score - local max)}  -> replace by the GLOBAL {max, sum exp(score - max)}
 *   phase 2: values = {local sum_h p_h loss_h}                               -> replace by the sum over all ranks
 * (return 0 on success).  The caller implements them with its collective of choice (esac_b200/sharded.py: NCCL
 * all-gather / all-reduce through torch.distributed).  *out_loss = the global expected loss.  Set option "hyp_offset" to
 * the global index of this shard's first hypothesis so that the shards draw the minimal sets of the unsharded problem. */
typedef int (*esacb200_exchange_fn)(void* user, int phase, double* values, int n);
int esacb200_backward_sharded(esacb200_ctx* ctx, const float* coords, float* grads, int E, int H, int W,
                              const int64_t* assign, int64_t assign_stride, int M, const float* gt_pose, float wLossRot,
                              float wLossTrans, float lossCut, int shiftX, int shiftY, float focalLength, float ppointX,
                              float ppointY, float inlierThreshold, float inlierAlpha, float inlierBeta, float maxReproj,
                              int subSampling, esacb200_exchange_fn exchange, void* user, double* out_loss);

/* The local half of a sharded esac_forward, enqueued WITHOUT a host synchronisation: runs sample -> score -> select ->
 * refine on this shard's experts / hypotheses and writes the record the shards exchange,
 *   pack_out[0..M_pad)      soft-inlier scores (esac.cpp:147-150); entries >= M are -inf (shards may hold different numbers
 *                           of hypotheses, the records of a collective must have one size: M_pad = the largest M),
 *   pack_out[M_pad..+16)    camera pose of the local winner,
 *   pack_out[M_pad+16]      expert_offset + its expert (or -1 if hypAssignment held an index outside [0,E)),
 *   pack_out[M_pad+17]      its local hypothesis index,        pack_out[M_pad+18]  M,
 *   pack_out[M_pad+19/20]   options "hyp_offset" / "hyp_stride": local hypothesis k is hypothesis offset + k * stride of the
 *                           unsharded problem (its minimal-set stream and its place in draw()'s first-maximum order),
 * as doubles into DEVICE memory, stream-ordered on the context's stream.  coords / assign must be device pointers (a host
 * buffer would force the synchronisation this entry exists to avoid).  M may be 0 (coords / assign are then ignored).
 * The record has M_pad + 21 doubles. */
int esacb200_forward_pack(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                          int64_t assign_stride, int M, int M_pad, int shiftX, int shiftY, float focalLength, float ppointX,
                          float ppointY, float inlierThreshold, float inlierAlpha, float inlierBeta, float maxReproj,
                          int subSampling, int expert_offset, double* pack_out);

/* ---- sharded entry points over NCCL (one process per GPU) ------------------------------------------------------------
 * The path has ONE exchange in forward (scores -> softMax / draw, esac.cpp:153-155) and TWO in backward (softmax
 * normalisation; the expectation sum_h p_h loss_h, esac.cpp:357-362, esac_derivative.h:372-374); SURVEY.md 8e.  The library
 * issues them itself as NCCL collectives on the context's stream.  NCCL is resolved at run time (dlopen of libnccl.so.2, the
 * copy the process already holds if any), so the library still loads where NCCL is absent.
 * esacb200_nccl_unique_id: 128-byte ncclUniqueId (rank 0 creates it, the caller distributes it by any means).
 * esacb200_comm_init:     ncclCommInitRank on the context's device; collective over all ranks. */
int esacb200_nccl_unique_id(void* out128);
int esacb200_comm_init(esacb200_ctx* ctx, int world, int rank, const void* id128);
int esacb200_comm_destroy(esacb200_ctx* ctx);
/* esac_forward over all shards: local pipeline -> record -> one ncclAllGather -> softMax / draw over the records on the device
 * (first strict maximum in rank-major order) -> one 80-byte read-back.  Every rank receives the global winner's camera pose
 * and (global) expert index.  coords / assign host or device pointers; M may be 0, but not on every rank (esac.forward refuses
 * M = 0 too: every rank then fails with ESACB200_ERR_ARG); M_pad = max M over the ranks. */
int esacb200_forward_sharded(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                             int64_t assign_stride, int M, int M_pad, float* out_pose, int shiftX, int shiftY, float focalLength,
                             float ppointX, float ppointY, float inlierThreshold, float inlierAlpha, float inlierBeta,
                             float maxReproj, int subSampling, int expert_offset, int* out_expert);
/* esac_backward over all shards (gradient slices are disjoint when experts are dealt expert-major: no gradient collective):
 * all-gather of (max score, sum exp) -> global probabilities; all-reduce of the partial expectations -> *out_loss = the
 * global expected loss on every rank.  Option "hyp_offset" as for esacb200_backward_sharded.  M may be 0.
 * reduce_grads != 0: HYPOTHESIS-major sharding -- every rank holds all E planes and a slice of the hypotheses (the refinement
 * of the contributing hypotheses then shards too, which expert-major dealing cannot do when the gating concentrates them on
 * one expert); gradient slices overlap, so the local gradients are summed over the ranks with one ncclAllReduce of E*3*H*W
 * floats and the sum is added to `grads` on every rank (grads stays "+=", esac.cpp:501-506). */
int esacb200_backward_sharded_nccl(esacb200_ctx* ctx, const float* coords, float* grads, int E, int H, int W,
                                   const int64_t* assign, int64_t assign_stride, int M, const float* gt_pose, float wLossRot,
                                   float wLossTrans, float lossCut, int shiftX, int shiftY, float focalLength, float ppointX,
                                   float ppointY, float inlierThreshold, float inlierAlpha, float inlierBeta, float maxReproj,
                                   int subSampling, int reduce_grads, double* out_loss);

/* esac_forward over B images of one shape (the reference's callers loop with batch_size=1, test_esac.py:137):
 * coords float32 [B,E,3,H,W], assign int64 [B,M] (rows contiguous, element stride assign_stride; 0 = one expert for all),
 * out_poses float32 [B,4,4], out_experts int [B] (host).  One host synchronisation for the whole batch; host maps are
 * double-buffered and copied on a second stream, overlapping the previous image's kernels. */
int esacb200_forward_batch(esacb200_ctx* ctx, int B, const float* coords, int E, int H, int W, const int64_t* assign,
                           int64_t assign_stride, int M, float* out_poses, int shiftX, int shiftY, float focalLength,
                           float ppointX, float ppointY, float inlierThreshold, float inlierAlpha, float inlierBeta,
                           float maxReproj, int subSampling, int* out_experts);

/* esacb200_forward_batch with a camera per image (the reference's callers read focallength from every image,
 * test_esac.py:145-147): image b runs with shiftX[b] / shiftY[b], focal length f[b] and principal point (ppx[b], ppy[b]),
 * host arrays of B values.  shiftX / shiftY may be NULL (= 0); f, ppx and ppy may not.  Everything else is as for
 * esacb200_forward_batch, which is this entry with every array holding its scalar. */
int esacb200_forward_batch_cameras(esacb200_ctx* ctx, int B, const float* coords, int E, int H, int W, const int64_t* assign,
                                   int64_t assign_stride, int M, float* out_poses, const int* shiftX, const int* shiftY,
                                   const float* f, const float* ppx, const float* ppy, float inlierThreshold, float inlierAlpha,
                                   float inlierBeta, float maxReproj, int subSampling, int* out_experts);

/* Stream-ordered esac_forward that a CUDA graph can capture.  DEVICE pointers only (a host pointer is an error, reported
 * before anything is enqueued): coords float32 [B,E,3,H,W], assign int64 [B,M] (rows contiguous, element stride
 * assign_stride), shifts int32 [B,2] (shiftX, shiftY), cameras float32 [B,3] (f, ppx, ppy); results out_poses float32
 * [B,4,4] camera->world, out_experts int64 [B], out_status int32 [B].  Status 0 = OK; 1 = the image's assignment held an
 * expert index outside [0,E): its pose is NaN and its expert -1, the other images are unaffected.  B = 1 is one image.
 *
 * The call enqueues on the context's stream and returns: no host synchronisation, no read-back, no event query, and while
 * the stream is being captured (cudaStreamBeginCapture, any capture mode) no allocation.  The seed, shift and camera of
 * every image are read from device memory when the kernels run, so a graph that captured the call replays with the values
 * the arrays hold at replay time.
 *
 * Seeding: the base seed and a call counter live in device memory; an execution reads them and advances the counter by B.
 * esacb200_set_seed resets both, enqueued on the context's stream (a set_seed after a capture applies from the next
 * replay).  Image b of the j-th execution after set_seed(s) draws what the (j*B + b)-th esacb200_forward after set_seed(s)
 * draws, option "fixed_seed" included (its value at enqueue / capture time).  Eager and stream-ordered calls count apart.
 *
 * Workspace: the stream-ordered forward has a workspace of its own, apart from the one the eager calls grow, so eager
 * calls of any shape leave a captured graph's buffers alone.  An uncaptured call grows it as needed; a captured call cannot
 * (that would allocate), so call esacb200_reserve_forward_async with the largest shape before the first capture.  Once a
 * capture has used the workspace nothing in it is freed or reallocated again: a later call or reserve that needs more
 * fails, before enqueuing anything, with a message that names the reserve call.
 *
 * The stage timers of esacb200_get_stats are neither recorded nor updated by these calls. */
int esacb200_forward_async(esacb200_ctx* ctx, int B, const float* coords, int E, int H, int W, const int64_t* assign,
                           int64_t assign_stride, int M, const int32_t* shifts, const float* cameras, float inlierThreshold,
                           float inlierAlpha, float inlierBeta, float maxReproj, int subSampling, float* out_poses,
                           int64_t* out_experts, int32_t* out_status);
/* Sizes the stream-ordered forward's workspace for calls of this shape (and creates its state); allocates, so it may not
 * run while the context's stream is being captured.  B does not change the workspace: the images run one after another. */
int esacb200_reserve_forward_async(esacb200_ctx* ctx, int B, int E, int H, int W, int M, int subSampling);

/* esac_backward enqueued with esacb200_forward_async's contract, so that a training step can be captured in a CUDA graph:
 * device pointers only, checked before anything is enqueued.  coords / grads float32 [B,E,3,H,W] (grads ACCUMULATED, +=,
 * as esacb200_backward), assign int64 [B,M], gt_poses float32 [B,4,4] camera->world, shifts int32 [B,2], cameras float32
 * [B,3]; results out_losses double [B] (the value esacb200_backward returns) and out_status int32 [B].  Status 1 = the
 * image's assignment held an expert index outside [0,E): its loss is NaN and its gradient slice is left untouched; the
 * other images are unaffected.  No host synchronisation, read-back or event query, and no allocation while capturing.
 *
 * esacb200_backward reads the number of contributing hypotheses back to size the refinement's CTA groups; here the
 * refinement kernel picks the same group from the same count on the device, on a grid as large as any count needs, so the
 * results are bitwise those of esacb200_backward.  The ground truth, shift and camera are read when the kernels run.
 *
 * Seeding: the same device-side seed and call counter as esacb200_forward_async (one counter for both): image b of the
 * j-th stream-ordered execution after set_seed(s) draws what the (j*B + b)-th esacb200_forward / esacb200_backward after
 * set_seed(s) draws, "fixed_seed" honoured.  Workspace: esacb200_forward_async's, with its rule; it also holds the
 * backward's buffers once esacb200_reserve_backward_async (or an uncaptured call) has sized them, and a call that needs
 * more after a capture fails, naming the reserve call. */
int esacb200_backward_async(esacb200_ctx* ctx, int B, const float* coords, float* grads, int E, int H, int W,
                            const int64_t* assign, int64_t assign_stride, int M, const float* gt_poses, float wLossRot,
                            float wLossTrans, float lossCut, const int32_t* shifts, const float* cameras, float inlierThreshold,
                            float inlierAlpha, float inlierBeta, float maxReproj, int subSampling, double* out_losses,
                            int32_t* out_status);
/* Sizes the stream-ordered workspace for esacb200_backward_async (and esacb200_forward_async) calls of this shape; allocates,
 * so it may not run while the context's stream is being captured. */
int esacb200_reserve_backward_async(esacb200_ctx* ctx, int B, int E, int H, int W, int M, int subSampling);

/* The hypotheses node (esacb200_hypotheses_forward / _backward) with esacb200_forward_async's contract, so that a training
 * step with the caller's own pose loss can be captured in a CUDA graph: device pointers only, checked before anything is
 * enqueued; no host synchronisation, read-back or event query, and no allocation while capturing.
 *
 * esacb200_hypotheses_forward_async: coords float32 [B,E,3,H,W], assign int64 [B,M] (rows contiguous, element stride
 * assign_stride), shifts int32 [B,2], cameras float32 [B,3] (f, ppx, ppy), read on the device when the kernels run.  Row b
 * of out_scores double [B,M], out_poses6 double [B,M,6] and out_contrib uint8 [B,M] is what esacb200_hypotheses_forward
 * gives; image b's tape is at tapes + b * stride, stride = esacb200_hypotheses_tape_bytes(E,H,W,M) rounded up to 256 bytes,
 * and tapes_bytes must be at least B * stride (16-byte aligned).  The header of a tape holds the shift and camera the
 * forward used.  Seeding: esacb200_forward_async's device-side seed and call counter: image b of the j-th stream-ordered
 * execution after set_seed(s) draws what the (j*B + b)-th esacb200_backward / esacb200_hypotheses_forward after set_seed(s)
 * draws, "fixed_seed" honoured.
 *
 * esacb200_hypotheses_backward_async ACCUMULATES (+=) into grads float32 [B,E,3,H,W] what esacb200_hypotheses_backward on
 * image b's tape with rows b of d_scores double [B,M] / d_poses6 double [B,M,6] (NULL = zero) adds.  It draws nothing and
 * does not advance the call counter.  The forward's shift, camera, sub and thresholds come from the tape header.
 *
 * out_status int32 [B]: 0 = OK; 1 = the image's assignment held an expert index outside [0,E) (forward: its scores and
 * poses are NaN and its contrib 0; backward of such a tape: its gradient slice is left untouched); 2 (backward only) = the
 * tape holds no forward of this E, H, W, M: the gradient slice is left untouched.  The other images are unaffected.
 *
 * Workspace: esacb200_backward_async's, with its rule: call esacb200_reserve_backward_async with the largest shape before
 * the first capture; after a capture a call that needs more fails before enqueuing anything, naming that call. */
int esacb200_hypotheses_forward_async(esacb200_ctx* ctx, int B, const float* coords, int E, int H, int W, const int64_t* assign,
                                      int64_t assign_stride, int M, const int32_t* shifts, const float* cameras,
                                      float inlierThreshold, float inlierAlpha, float inlierBeta, float maxReproj, int subSampling,
                                      void* tapes, size_t tapes_bytes, double* out_scores, double* out_poses6,
                                      uint8_t* out_contrib, int32_t* out_status);
/* The floor is a kernel parameter: a captured graph replays with the min_prob it was captured with. */
int esacb200_hypotheses_forward_async_floor(esacb200_ctx* ctx, int B, const float* coords, int E, int H, int W,
                                            const int64_t* assign, int64_t assign_stride, int M, const int32_t* shifts,
                                            const float* cameras, float inlierThreshold, float inlierAlpha, float inlierBeta,
                                            float maxReproj, int subSampling, double min_prob, void* tapes, size_t tapes_bytes,
                                            double* out_scores, double* out_poses6, uint8_t* out_contrib, int32_t* out_status);
int esacb200_hypotheses_backward_async(esacb200_ctx* ctx, int B, const void* tapes, size_t tapes_bytes, const float* coords,
                                       float* grads, int E, int H, int W, int M, const double* d_scores, const double* d_poses6,
                                       int32_t* out_status);
/* esacb200_pose_loss_batch launched on the caller's device arrays: no staging copy and no synchronisation (poses6 double
 * [B,M,6], gt16 float32 [B,4,4], out_losses double [B,M], out_dloss6 double [B,M,6]); bitwise the same rows. */
int esacb200_pose_loss_async(esacb200_ctx* ctx, int B, int M, const double* poses6, const float* gt16, float wLossRot,
                             float wLossTrans, float lossCut, double* out_losses, double* out_dloss6);

/* esac_backward over B images of one shape (the reference trains with batch_size=1, train_esac.py:96-100, one
 * esac.backward per image): coords / grads float32 [B,E,3,H,W] (grads accumulated in place, as esac.cpp:490-508),
 * assign int64 [B,M] (as in esacb200_forward_batch), gt_poses float32 [B,4,4] (camera->world), shiftX / shiftY int [B]
 * on the host or NULL (= 0: the per-image random shift of train_esac.py:125), out_losses host double [B].
 * Image b draws the minimal sets that the b-th of B consecutive esacb200_backward calls on this context would draw, so
 * the batch returns exactly what that loop returns; images are spread over option "batch_workers" (default 8) internal
 * streams, each with its own workspace and host thread, so their kernels and the per-image host synchronisations overlap. */
int esacb200_backward_batch(esacb200_ctx* ctx, int B, const float* coords, float* grads, int E, int H, int W,
                            const int64_t* assign, int64_t assign_stride, int M, const float* gt_poses, float wLossRot,
                            float wLossTrans, float lossCut, const int* shiftX, const int* shiftY, float focalLength,
                            float ppointX, float ppointY, float inlierThreshold, float inlierAlpha, float inlierBeta,
                            float maxReproj, int subSampling, double* out_losses);

/* esacb200_backward_batch with a camera per image: image b runs with focal length f[b] and principal point
 * (ppx[b], ppy[b]), host arrays of B values that may not be NULL; shiftX / shiftY as for esacb200_backward_batch (NULL = 0).
 * Same worker contexts and the same minimal sets per image as esacb200_backward_batch, which is this entry with every
 * camera array holding its scalar. */
int esacb200_backward_batch_cameras(esacb200_ctx* ctx, int B, const float* coords, float* grads, int E, int H, int W,
                                    const int64_t* assign, int64_t assign_stride, int M, const float* gt_poses, float wLossRot,
                                    float wLossTrans, float lossCut, const int* shiftX, const int* shiftY, const float* f,
                                    const float* ppx, const float* ppy, float inlierThreshold, float inlierAlpha,
                                    float inlierBeta, float maxReproj, int subSampling, double* out_losses);

/* Hypothesis assignment on the device, the three host steps the reference's callers run before esac.forward/backward:
 * util.clamp_probs (util.py:38-48; keep_top < 0 = off), torch.multinomial(probs, M, replacement=True)
 * (train_esac.py:133-137, test_esac.py:169-174; single_expert != 0 = one draw expanded to M, the "expertselection" mode)
 * and torch.histc over the experts (train_esac.py:140).  weights float32 [B,E] >= 0 (host or device, not necessarily
 * normalised), out_assign int64 [B,M], out_hist float32 [B,E] or NULL (both host or device).  The draws are a pure
 * function of (seed, image, hypothesis).  Negative / non-finite weights or an all-zero row are an error, as in torch. */
int esacb200_assign_hypotheses(esacb200_ctx* ctx, int B, int E, int M, const float* weights, int keep_top,
                               int single_expert, uint64_t seed, int64_t* out_assign, float* out_hist);

/* esacb200_assign_hypotheses enqueued on the context's stream with no host synchronisation, so a CUDA graph can capture it.
 * Every pointer is a device pointer: weights float32 [B,E], seed int64 [1] (read when the kernel runs, so a graph can
 * advance it or the caller can rewrite it between replays), out_assign int64 [B,M], out_hist float32 [B,E] or NULL, and
 * out_status int32 [B]: 0, or 1 for a row with a negative / non-finite weight, 2 for a row that sums to 0 (the errors of
 * the eager call; the row's draws are then meaningless).  Given the same seed value it draws exactly what
 * esacb200_assign_hypotheses draws. */
int esacb200_assign_hypotheses_async(esacb200_ctx* ctx, int B, int E, int M, const float* weights, int keep_top,
                                     int single_expert, const int64_t* seed, int64_t* out_assign, float* out_hist,
                                     int* out_status);

/* ---- expert gates: run a region of a captured CUDA graph only where a count on the device is positive ---------------
 * A gate has n <= ESACB200_GATE_MAX switches and serves one graph.  While a stream is being captured:
 *   esacb200_gate_arm   enqueues a kernel that, at every replay of the finalized graph, sets switch i to (counts[i] > 0);
 *                       counts: device float32 [n], typically a hypothesis histogram.  Once per gate.
 *   esacb200_gate_mark  enqueues an empty marker kernel that opens (begin != 0) or closes region `index` of the gate.
 * After the capture ends and before the graph is instantiated, esacb200_gate_finalize rewrites the graph: every region
 * (begin marker, end marker and the nodes downstream of the begin and upstream of the end) moves into the body of an IF
 * conditional node on the gate's conditional handle `index`, which takes its place.  The handles are created on the graph
 * there, with the default value 0 applied at every launch.  Several regions may share an index.  A region must be closed:
 * work forked from it must join before its end, work it waits on must precede its begin, regions may not nest or overlap,
 * the gate must be armed upstream of every region, and a region may hold only kernel, memset, device memcpy, empty,
 * child graph and conditional nodes.  On a violation finalize returns ESACB200_ERR_ARG, names the region and the reason in
 * esacb200_last_error, and leaves the graph untouched: it then runs every region, and its arm kernel does nothing.
 * Conditional nodes need a CUDA 12.3 driver: gate_create fails with ESACB200_ERR_CUDA on an older one.  The gate must
 * outlive the graph's replays (the arm kernel reads the handles from the gate's memory).  A gate's errors are reported on
 * its context. */
#define ESACB200_GATE_MAX 1024
typedef struct esacb200_gate esacb200_gate;
int esacb200_gate_create(esacb200_ctx* ctx, int n, esacb200_gate** out);
void esacb200_gate_destroy(esacb200_gate* gate);
int esacb200_gate_arm(esacb200_gate* gate, const float* counts, void* stream);
int esacb200_gate_mark(esacb200_gate* gate, int index, int begin, void* stream);
int esacb200_gate_finalize(esacb200_gate* gate, void* graph);

/* Robust reprojection loss of the expert refinement stage and its gradient, one fused pass (ref_expert.py:103-146, where
 * it is six elementwise torch ops + autograd): coords float32 [B,3,H,W] (one expert's prediction per image; the reference
 * has B = 1), grads float32 [B,3,H,W] or NULL = d loss_b / d coords (overwritten, not accumulated), gt_poses float32
 * [B,4,4] camera->world (inverted here, ref_expert.py:127), shiftX / shiftY host int [B] or NULL (padX / padY, :110-111),
 * target pixel of cell (x,y) = (x*sub + sub/2 - padX, y*sub + sub/2 - padY) with real-valued sub/2 (:84-89),
 * depth clamped from below at minDepth (0.1, :136), error clamped to [0, maxReproj] (100, :142), square-root loss above
 * cutLoss (:144-146), mean over the H*W cells (:148).  out_losses host double [B].  fp32 arithmetic like the original. */
int esacb200_reproj_loss(esacb200_ctx* ctx, int B, const float* coords, float* grads, int H, int W, const float* gt_poses,
                         const int* shiftX, const int* shiftY, float focalLength, float ppointX, float ppointY,
                         int subSampling, float cutLoss, float maxReproj, float minDepth, double* out_losses);

/* esacb200_reproj_loss with a camera per image: image b is projected with focal length f[b] and principal point
 * (ppx[b], ppy[b]), host arrays of B values that may not be NULL; shiftX / shiftY as for esacb200_reproj_loss (NULL = 0).
 * Still one launch for the batch; esacb200_reproj_loss is this entry with every camera array holding its scalar, and the
 * per-cell arithmetic is the same, so equal cameras give bitwise the same losses and gradients. */
int esacb200_reproj_loss_cameras(esacb200_ctx* ctx, int B, const float* coords, float* grads, int H, int W, const float* gt_poses,
                                 const int* shiftX, const int* shiftY, const float* f, const float* ppx, const float* ppy,
                                 int subSampling, float cutLoss, float maxReproj, float minDepth, double* out_losses);

/* Robust scene-coordinate loss of the expert initialisation stage and its gradient (init_expert.py:106-135, where it is
 * ten elementwise torch ops, four boolean-mask indexings + autograd): pred float32 [B,3,Hp,Wp] (one expert's prediction
 * per image; the reference has B = 1), gt float32 [B,3,Hg,Wg] ground-truth scene coordinates.  The two may differ by at most
 * 1 in H and in W; both are cropped to the top-left min(Hp,Hg) x min(Wp,Wg) window (util.assert_size, util.py:18-36).  A
 * cell is valid iff one of its ground-truth components is nonzero (NaN included); n = ||pred - gt||, per-cell loss n for
 * n <= cutLoss, sqrt(cutLoss * n) above; the image's loss is the sum over valid cells divided by their number (NaN when
 * there is none).  grads float32 [B,3,Hp,Wp] or NULL (loss only) = d loss_b / d pred (overwritten, not accumulated; 0 outside
 * the window, on invalid cells and at n = 0, NaN on NaN cells).  out_losses host double [B]; out_counts host int64 [B] valid
 * cells per image, or NULL.  pred / gt / grads host or device pointers; one host synchronisation, at the end. */
int esacb200_coord_loss(esacb200_ctx* ctx, int B, const float* pred, int Hp, int Wp, const float* gt, int Hg, int Wg,
                        float* grads, float cutLoss, double* out_losses, int64_t* out_counts);

/* Ragged batches: B images of different sizes (19Scenes, Aachen and Dubrovnik keep each image's aspect ratio).  Each
 * image-sized argument is a host array of B pointers to contiguous per-image buffers, with host arrays of B heights and
 * widths.  All pointers of one argument are device pointers or all are host pointers; a mix is an error.  Image b computes
 * exactly what a single-image call on it computes: the same minimal sets (forward / backward), bitwise the same losses and
 * gradients (the two losses).  Size errors name the image.  The one-shape entry points above are these with every image
 * a slice of one tensor, and give bitwise what they gave before.
 *
 * esacb200_forward_batch_cameras on maps coords[b] float32 [E,3,H[b],W[b]]; assign, out_poses, the shifts and cameras as
 * there.  The workspace is sized for the largest image before the first image is enqueued. */
int esacb200_forward_ragged(esacb200_ctx* ctx, int B, const float* const* coords, const int* H, const int* W, int E,
                            const int64_t* assign, int64_t assign_stride, int M, float* out_poses, const int* shiftX,
                            const int* shiftY, const float* f, const float* ppx, const float* ppy, float inlierThreshold,
                            float inlierAlpha, float inlierBeta, float maxReproj, int subSampling, int* out_experts);

/* esacb200_backward_batch_cameras on maps coords[b] / grads[b] float32 [E,3,H[b],W[b]] (grads accumulated in place).  Each
 * worker runs its images largest first. */
int esacb200_backward_ragged(esacb200_ctx* ctx, int B, const float* const* coords, float* const* grads, const int* H, const int* W,
                             int E, const int64_t* assign, int64_t assign_stride, int M, const float* gt_poses, float wLossRot,
                             float wLossTrans, float lossCut, const int* shiftX, const int* shiftY, const float* f,
                             const float* ppx, const float* ppy, float inlierThreshold, float inlierAlpha, float inlierBeta,
                             float maxReproj, int subSampling, double* out_losses);

/* esacb200_reproj_loss_cameras on predictions coords[b] float32 [3,H[b],W[b]]; grads NULL (loss only) or B pointers
 * [3,H[b],W[b]] (overwritten). */
int esacb200_reproj_loss_ragged(esacb200_ctx* ctx, int B, const float* const* coords, float* const* grads, const int* H,
                                const int* W, const float* gt_poses, const int* shiftX, const int* shiftY, const float* f,
                                const float* ppx, const float* ppy, int subSampling, float cutLoss, float maxReproj,
                                float minDepth, double* out_losses);

/* esacb200_coord_loss on pred[b] float32 [3,Hp[b],Wp[b]] and gt[b] float32 [3,Hg[b],Wg[b]], each pair at most 1 apart in H
 * and in W; grads NULL (loss only) or B pointers [3,Hp[b],Wp[b]] (overwritten). */
int esacb200_coord_loss_ragged(esacb200_ctx* ctx, int B, const float* const* pred, const int* Hp, const int* Wp,
                               const float* const* gt, const int* Hg, const int* Wg, float* const* grads, float cutLoss,
                               double* out_losses, int64_t* out_counts);

/* The two losses with esacb200_forward_async's contract, so that a step of init_expert.py / ref_expert.py (the expert's
 * forward, the loss, its backward and the optimiser) can be captured in one CUDA graph.  Ragged form only: host arrays of B
 * image pointers and sizes, as in the ragged calls above; the pointers and sizes are fixed for a capture, and every image
 * pointer, like every other pointer argument, must be DEVICE memory (a host pointer is an error, reported before anything
 * is enqueued).  The call enqueues on the context's stream and returns: no host synchronisation, no read-back, no event
 * query, and while the stream is being captured no allocation.  What changes from step to step is read from device memory
 * when the kernels run: the maps, the ground truths, the pads and the cameras.  B <= 65535.
 *
 * esacb200_reproj_loss_async: esacb200_reproj_loss_ragged on coords[b] float32 [3,H[b],W[b]], grads NULL (loss only) or B
 * pointers [3,H[b],W[b]] (overwritten), gt_poses float32 [B,4,4] camera->world, shifts int32 [B,2] (padX, padY), cameras
 * float32 [B,3] (f, cx, cy).  The ground truth is inverted on the device with the eager call's host arithmetic, so the
 * losses and gradients are bitwise the eager call's.  out_losses double [B]; out_status int32 [B]: 0 = OK, 1 = the image's
 * ground-truth rotation block is singular or NaN (where the eager call fails): its loss is NaN, its gradient slice zero, and
 * the other images are unaffected.
 *
 * esacb200_coord_loss_async: esacb200_coord_loss_ragged on device maps, out_losses double [B], out_counts int64 [B] or NULL;
 * bitwise the eager call's results.  An image without valid cells has a NaN loss, as there; nothing fails on the device.
 *
 * Workspace: the two share one buffer of the stream-ordered context, apart from the forward's and the backward's.  An
 * uncaptured call grows it as needed; a captured call cannot, so call esacb200_reserve_loss_async before the first capture
 * (B images of at most H x W cells: for the coordinate loss, cells of the prediction).  Once a capture has used it, nothing
 * in it is freed or reallocated: a later call or reserve that needs more fails, before enqueuing anything, naming the
 * reserve call.  The first call on a context, of either loss or of esacb200_reserve_loss_async, may not be captured. */
int esacb200_reproj_loss_async(esacb200_ctx* ctx, int B, const float* const* coords, float* const* grads, const int* H,
                               const int* W, const float* gt_poses, const int32_t* shifts, const float* cameras, int subSampling,
                               float cutLoss, float maxReproj, float minDepth, double* out_losses, int32_t* out_status);
int esacb200_coord_loss_async(esacb200_ctx* ctx, int B, const float* const* pred, const int* Hp, const int* Wp,
                              const float* const* gt, const int* Hg, const int* Wg, float* const* grads, float cutLoss,
                              double* out_losses, int64_t* out_counts);
int esacb200_reserve_loss_async(esacb200_ctx* ctx, int B, int H, int W);

/* The four loss calls above on predictions of a chosen element type, for experts trained under autocast.  dtype is one
 * code for the whole call: the predictions and gradients (coords / pred, grads) are B pointers to elements of that type;
 * the ground truth, poses and cameras stay float32.  Each prediction is widened to fp32 and computed exactly as the float32
 * call computes it on the widened map, so the losses are bitwise the float32 call's on the same load path (the vector path
 * needs N % 4 == 0, W >= 4 and planes aligned to 4 elements; the float32 and the 16-bit calls choose it alike for maps
 * aligned alike).  Each gradient is the float32 call's gradient g, times *grad_scale as one fp32 multiply when grad_scale
 * is not NULL, rounded to nearest into dtype: bitwise what autograd gives a 16-bit prediction that was cast to float32
 * before a float32 loss whose upstream gradient is *grad_scale.  grad_scale: a device float, read when the kernels run
 * (so a capture replays with the current scale), or NULL for 1.  ESACB200_FLOAT16 and ESACB200_BFLOAT16 take device
 * pointers only.  An unknown code, a host pointer with a 16-bit code, or a grad_scale with ESACB200_FLOAT32 fails with
 * ESACB200_ERR_ARG before anything is enqueued.  The workspace is the float32 calls' (esacb200_reserve_loss_async covers
 * both); the untyped calls are these with ESACB200_FLOAT32 and grad_scale NULL. */
#define ESACB200_FLOAT32 0
#define ESACB200_FLOAT16 1
#define ESACB200_BFLOAT16 2
int esacb200_reproj_loss_ragged_typed(esacb200_ctx* ctx, int B, int dtype, const void* const* coords, void* const* grads,
                                      const int* H, const int* W, const float* gt_poses, const int* shiftX, const int* shiftY,
                                      const float* f, const float* ppx, const float* ppy, int subSampling, float cutLoss,
                                      float maxReproj, float minDepth, const float* grad_scale, double* out_losses);
int esacb200_coord_loss_ragged_typed(esacb200_ctx* ctx, int B, int dtype, const void* const* pred, const int* Hp, const int* Wp,
                                     const float* const* gt, const int* Hg, const int* Wg, void* const* grads, float cutLoss,
                                     const float* grad_scale, double* out_losses, int64_t* out_counts);
int esacb200_reproj_loss_async_typed(esacb200_ctx* ctx, int B, int dtype, const void* const* coords, void* const* grads,
                                     const int* H, const int* W, const float* gt_poses, const int32_t* shifts,
                                     const float* cameras, int subSampling, float cutLoss, float maxReproj, float minDepth,
                                     const float* grad_scale, double* out_losses, int32_t* out_status);
int esacb200_coord_loss_async_typed(esacb200_ctx* ctx, int B, int dtype, const void* const* pred, const int* Hp, const int* Wp,
                                    const float* const* gt, const int* Hg, const int* Wg, void* const* grads, float cutLoss,
                                    const float* grad_scale, double* out_losses, int64_t* out_counts);

/* Test-time evaluation of estimated poses (test_esac.py:209-247), so that a captured test step evaluates its image on the
 * device.  Image b of B: its camera->world estimate out_poses[b] and ground truth gt_poses[b] (float32 [B,4,4]), its
 * winning expert experts[b] and ground-truth scene scenes[b] (int64 [B]), optionally its hypothesis histogram hist[b]
 * (float32 [B,E], as esacb200_assign_hypotheses_async writes it) and its forward status status[b] (int32 [B]); hist and
 * status may be NULL.  Every pointer is a device pointer.  Its record, 14 doubles, goes to row state[0] + b of records
 * (double [capacity][14]):
 *   0 rotation error in degrees: acos(c) of the nearest rotation (Newton polar factor) to P_R G_R^T, c and s as OpenCV's
 *     Rodrigues forms them, and exactly 0 where s < 1e-5 and c > 0 (errors below ~5.7e-4 deg read 0, as in the reference)
 *   1 translation error |G[:3,3] - P[:3,3]| in centimetres
 *   2 correct (experts[b] == scenes[b]: 1, else 0)   3 scene   4 expert   5 status (0 without a status array)
 *   6 experts active: hist[b] entries > 0 (NaN without a histogram)
 *   7-10 qw qx qy qz and 11-13 tx ty tz of the pose-file line: the general 4x4 inverse of P, the axis-angle vector r of
 *     its rotation's nearest rotation, q = (cos(|r|/2), sin(|r|/2) r/|r|); q_xyz is NaN where |r| = 0, as the reference
 *     writes it.
 * All in fp64 from the float32 inputs.  state: int64 [4], zeroed by the caller before the first call: [0] rows handed out so
 * far (advanced by B by the launch, after every image has read it), [1] set to 1 when a row fell at or past capacity (that
 * row is not written), [2] a ticket the launch leaves zero, [3] unused.
 * esacb200_eval_poses_async enqueues on the context's stream: no host synchronisation, read-back or allocation, so it may be
 * captured.  esacb200_eval_poses is the same followed by a synchronisation of that stream.  Argument errors
 * (ESACB200_ERR_ARG: a NULL or host pointer, B outside [1, 2^24], capacity <= 0, E outside [1, ESACB200_GATE_MAX] with a
 * histogram) are reported before anything is enqueued. */
int esacb200_eval_poses_async(esacb200_ctx* ctx, int B, const float* out_poses, const float* gt_poses, const int64_t* experts,
                              const int64_t* scenes, const float* hist, int E, const int32_t* status, double* records,
                              int64_t capacity, int64_t* state);
int esacb200_eval_poses(esacb200_ctx* ctx, int B, const float* out_poses, const float* gt_poses, const int64_t* experts,
                        const int64_t* scenes, const float* hist, int E, const int32_t* status, double* records,
                        int64_t capacity, int64_t* state);

/* Clustering a large environment into experts (cluster_dataset.py:19-140, 219-240).  Each call checks every argument
 * before it enqueues anything (ESACB200_ERR_ARG) and returns after its work is done.
 *
 * esacb200_cluster_stats_ragged: the statistics of B >= 1 ground-truth maps, map b float32 [3, H[b], W[b]] at maps[b]
 * (all device or all host pointers; 1 <= H*W <= 2^30).  A cell is valid when the float32 sum (x + y) + z is not 0.  Per map:
 * out_median[b*3 + c] torch's lower median of coordinate c over the valid cells (sorted[(n-1)/2], the first NaN when there
 * is one; -0 sorts before +0), out_mean[b*3 + c] the fp64 mean of the valid cells rounded to
 * float32, out_count[b] the valid cells and out_status[b]: 0 ok, 1 no valid cell (median and mean NaN), 2 a non-finite
 * median or mean.  Outputs may be host or device memory.
 *
 * esacb200_kmeans2: cv2.kmeans(points, 2, None, (EPS + MAX_ITER, max_iter, eps), attempts, KMEANS_PP_CENTERS) on n >= 2
 * points (device float32 [n,3]), with its own random stream: draw d of attempt a is mix64-keyed by (seed, split, a, d).  Per
 * attempt (one CTA each, all in one launch): k-means++ seeding with 3 trials, then Lloyd iterations (nearer centre, centre
 * 0 on a tie; a cluster left empty takes the point farthest from the other centre, lowest index on a tie) until max_iter
 * >= 1 iterations or the largest squared centre shift <= eps^2 (eps >= 0).  The attempt with the lowest compactness (fp64
 * sum of squared distances; lowest attempt on a tie) writes out_labels (device int32 [n], 0 / 1), out_centres (device
 * float32 [2,3]) and out_compactness (device double [1]).  1 <= attempts <= 4096, split >= 0.  Every sum has a fixed
 * order: two calls with the same arguments agree bitwise.
 *
 * esacb200_cluster_targets: for N >= 1 images with means (device float32 [N,3]) and labels (device int64 [N], each in
 * [0, K), every cluster non-empty; 1 <= K <= 1024): out_centres (device float32 [K,3]) the fp64 mean of each cluster's
 * image means, out_sizes (device float32 [K]) the fp64 mean squared distance of those means to the float32 centre, and
 * out_probs (device float32 [N,K]) the soft gating targets in the reference's float32 op order:
 * exp(-|m_i - c_k|^2 / size_k / 2 * softness) / sqrt(2 pi size_k), normalised by their sum + 1e-7 (softness > 0). */
int esacb200_cluster_stats_ragged(esacb200_ctx* ctx, int B, const float* const* maps, const int* H, const int* W,
                                  float* out_median, float* out_mean, int32_t* out_count, int32_t* out_status);
int esacb200_kmeans2(esacb200_ctx* ctx, int n, const float* points, uint64_t seed, int split, int attempts, int max_iter,
                     double eps, int32_t* out_labels, float* out_centres, double* out_compactness);
int esacb200_cluster_targets(esacb200_ctx* ctx, int N, const float* means, const int64_t* labels, int K, float softness,
                             float* out_centres, float* out_sizes, float* out_probs);

/* Rendering ground-truth scene-coordinate maps from an SfM reconstruction (setup_aachen.py:184-202,
 * setup_dubrovnik.py:171-190).  The call checks every argument before it enqueues anything (ESACB200_ERR_ARG) and returns
 * after its work is done.
 *
 * esacb200_render_init_maps: C >= 1 cameras; camera c owns the observations offsets[c] .. offsets[c+1] - 1 (host int64
 * [C+1], offsets[0] = 0, non-decreasing, V = offsets[C] <= ESACB200_RENDER_MAX_OBS), in reconstruction file order;
 * observation v sees point indices[v] (int32 [V]) of points (float32 [P,3], 0 <= P <= ESACB200_RENDER_MAX_OBS); both host or
 * device memory; indices may be null when V = 0, points when P = 0.  Per camera (host arrays): poses[c*12 ..] rows 0-2 of the float32 world -> camera
 * pose, focal[c], out_scale[c] (out width / image width) and the out map's H[c] x W[c], each side in
 * [1, ESACB200_RENDER_MAX_SIDE], ESACB200_RENDER_MAX_CELLS cells in all.  Each observation projects in float32 with
 * round-to-nearest and no contraction: cam = ((r0 x + r1 y) + r2 z) + r3 per row, u = ((cam.x f) / cam.z) s + W/2,
 * v = ((cam.y f) / cam.z) s + H/2, cell (int(clamp(v, 0, H-1)), int(clamp(u, 0, W-1))), so off-image points and points behind
 * the camera land on the border.  A cell keeps what the serial test `zbuf == 0 or zbuf > cam.z` over its observations in
 * file order keeps: the nearest depth (the earliest on equal depths) after the cell's last written depth-+-0 point, else that
 * point, else nothing; a depth-0 point is written unless a negative depth came before it in the cell.  Out: camera c's map float32 [3,H[c],W[c]] at out_maps + 3 * (cells of cameras 0..c-1), all-zero where
 * nothing was written (device memory); optionally its z-buffer float32 [H[c],W[c]] at out_zbuf + (cells of cameras 0..c-1)
 * (device memory or null); out_count[c] the cells written and out_status[c] (host or device memory): bit 1 an observation
 * with a point index outside [0, P), bit 2 a NaN projection (cam.z = 0 with cam.x or cam.y = 0); such observations take no
 * part.  The result does not depend on the order of the device's atomics: two calls agree bitwise.  The call allocates
 * its workspace (16 bytes per cell, 8 per observation, plus a device copy of host points and indices) and frees it
 * before it returns, so the context keeps none of it. */
#define ESACB200_RENDER_MAX_SIDE 8192
#define ESACB200_RENDER_MAX_CELLS (1 << 30)
#define ESACB200_RENDER_MAX_OBS 2147483392 /* 2^31 - 256 */
int esacb200_render_init_maps(esacb200_ctx* ctx, int C, const float* points, int64_t P, const int64_t* offsets,
                              const int32_t* indices, const float* poses, const float* focal, const float* out_scale,
                              const int32_t* H, const int32_t* W, float* out_maps, float* out_zbuf, int32_t* out_count,
                              int32_t* out_status);

/* A device-resident image set feeding a captured step (esac_b200/data.py: DeviceImageSet): each step's image, colour
 * jitter, normalisation, shift and ground truth are made on the device from the set's decoded, resized uint8 images, by
 * the rows of a plan the host drew with the reference loop's random calls (room_dataset.py:134-207,
 * cluster_dataset.py:245-275, util.py:4-11).
 *
 * esacb200_data_row: one image of one step.  image indexes the set's records; (padX, padY) is the shift
 * nn.ZeroPad2d((padX, -padX, padY, -padY)) applies; ops[0 .. n_ops-1] are the jitter's ops in the order ColorJitter runs
 * them (ESACB200_DATA_BRIGHTNESS / _CONTRAST / _SATURATION, each at most once, n_ops in [0, 3]) with factors[k] the
 * factor of ops[k].  40 bytes. */
#define ESACB200_DATA_BRIGHTNESS 0
#define ESACB200_DATA_CONTRAST 1
#define ESACB200_DATA_SATURATION 2
#define ESACB200_DATA_MAX_ATTACH 8
#define ESACB200_DATA_MAX_SIDE 8192
#define ESACB200_DATA_MAX_BATCH 4096
typedef struct {
    int32_t image;
    int32_t padX, padY;
    int32_t n_ops;
    int32_t ops[3];
    float factors[3];
} esacb200_data_row;

/* esacb200_data_image: one image of the set.  pixels: byte offset of its RGB uint8 [H,W,3] pixels in the set's pixel
 * storage; gt: float offset of its float32 [3,gt_h,gt_w] ground-truth map in the set's ground-truth storage (-1: none);
 * focal: its focal length, already scaled to the stored image (the camera holds its float32 rounding); scene: the
 * ground-truth scene (-1 for a clustered set); pose: float32 [4,4] camera->world, already offset; group: its shape group,
 * whose image is H x W and whose ground truth is gt_h x gt_w.  120 bytes. */
typedef struct {
    int64_t pixels;
    int64_t gt;
    double focal;
    int64_t scene;
    float pose[16];
    int32_t group;
    int32_t H, W, gt_h, gt_w;
    int32_t unused;
} esacb200_data_image;

/* esacb200_data_state: device memory.  position: the next plan row; rows: the rows the plan holds (from the last upload). */
typedef struct {
    int64_t position;
    int64_t rows;
} esacb200_data_state;

/* esacb200_data_step_async: one step of B images of shape group `group` (images H x W, ground truth gt_h x gt_w), enqueued
 * on the context's stream with no host synchronisation, read-back or allocation, so it may be captured.  It reads plan
 * rows state->position .. + B - 1 (plan: device esacb200_data_row [capacity]) when the kernels run, and writes out_status
 * (device int32 [1]): 0 ok; 1 the plan is exhausted (position + B > rows); 2 a row's image is outside [0, n_images) or not
 * of this group and shape.  On 1 and 2 no other output is written and the position stays; on 0 the position advances by
 * B.  Per image b: out_indices[b] (int64) the row's image, out_scenes[b] (int64) its scene, out_shifts[b] (int32 [2])
 * padX, padY, out_cameras[b] (float32 [3]) (float)focal, W/2, H/2, out_poses[b] (float32 [4,4]) its pose, out_image[b]
 * (float32 [3,H,W]) its pixels through the row's jitter, then (u/255 - mean[c]) / std[c] in float32, shifted by
 * (padX, padY) with zeros outside; out_coords[b] (float32 [3,gt_h,gt_w]) its ground truth (gt and out_coords both null,
 * or both given; every image of the group must then have one), and for k < n_attach out_attach[k][b] the
 * attach_numel[k] floats of attachment k at attach[k] + image * attach_numel[k].
 * Jitter, bitwise PIL's ImageEnhance: blend(a, b, f) = a + f (b - a) in float32 with no contraction, truncated to uint8
 * for 0 <= f <= 1, else clipped to [0, 255] and truncated; brightness blends from 0, saturation from L = (19595 R +
 * 38470 G + 7471 B + 0x8000) >> 16, contrast from int(sum(L) / N + 0.5) (fp64) over the image as the ops before it left it.
 * pixels, gt and attach may be device memory or mapped pinned host memory; images, plan, state, work (int64 [B]) and the
 * outputs are device memory; mean / std are host float[3].  Argument errors (ESACB200_ERR_ARG) are reported before
 * anything is enqueued. */
int esacb200_data_step_async(esacb200_ctx* ctx, const uint8_t* pixels, const float* gt, const esacb200_data_image* images,
                             int64_t n_images, int group, int H, int W, int gt_h, int gt_w, const float* mean,
                             const float* std, int n_attach, const float* const* attach, const int64_t* attach_numel,
                             const esacb200_data_row* plan, int64_t capacity, esacb200_data_state* state, int B,
                             int64_t* work, float* out_image, int32_t* out_shifts, float* out_cameras, float* out_poses,
                             float* out_coords, int64_t* out_scenes, int64_t* out_indices, float* const* out_attach,
                             int32_t* out_status);

/* Soft-inlier scores of given poses (getReproErrs + getHypScores, esac_util.h:235-363) without
 * sampling/selection/refinement: poses6 = host double [M][6] (rvec, tvec); out_scores host double [M]. */
int esacb200_score_poses(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                         int64_t assign_stride, int M, const double* poses6, int shiftX, int shiftY,
                         float focalLength, float ppointX, float ppointY, float inlierThreshold, float inlierAlpha,
                         float inlierBeta, float maxReproj, int subSampling, double* out_scores);

/* Refine given poses (refineHyp, esac_util.h:378-454): poses6 in/out host double [M][6]; out_rounds
 * host int [M] accepted rounds; out_inliers host int [M] size of the final inlier set (may be NULL). */
int esacb200_refine_poses(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                          int64_t assign_stride, int M, double* poses6, int shiftX, int shiftY, float focalLength,
                          float ppointX, float ppointY, float inlierThreshold, float maxReproj, int subSampling,
                          int* out_rounds, int* out_inliers);

typedef struct {
    int M;
    int winner;            /* hypothesis index selected by draw() */
    int n_contrib;         /* hypotheses with p >= PROB_THRESH */
    int refine_rounds;     /* accepted refinement rounds of the winner (forward) */
    double entropy;        /* esac_util.h:489-497 */
    double expected_loss;  /* backward only */
    /* device time of the last call's stages in milliseconds (CUDA events on the launching stream) */
    float ms_h2d, ms_prep, ms_sample, ms_score, ms_select, ms_refine, ms_backward, ms_total;
    int score_launches;    /* launches of the scoring kernel in the last call */
    int kernel_launches;   /* all kernel launches of the last call */
    int score_ppt, score_grid, refine_group;
} esacb200_stats;
int esacb200_get_stats(esacb200_ctx* ctx, esacb200_stats* out);

/* Diagnostics: with option "refine_profile" = 1 block 0 of the refinement kernel accumulates clock64() cycles per phase of
 * an LM evaluation of the root block: [0] produce + receive the command (Rodrigues of the new parameters), [1] pass over
 * the cells, [2] block reduction + slot write, [7] dR/dr + change of variables (root, before its gather), [3] wait for the
 * group's results, [4] slot summation, [5] map the sums to (rvec, tvec), [6] accept / reject + LM step; [8] = number of
 * evaluations.
 * out16: host long long [16]. */
int esacb200_get_refine_profile(esacb200_ctx* ctx, long long* out16);

/* Diagnostics of the last call's sampling stage (summed over its lanes): [0] tries that went through the float prefilter,
 * [1] survivors the fp64 path judged, [2] waves that had work (max over lanes), [3] hypotheses left to the tail kernel,
 * [4] accepted tries staged, [5] lanes, [6] tries of the windows the prefilter skipped because an earlier try was hinted
 * (option "sample_hint"; [0] still counts the whole windows), [7] hinted tries the exact verdict rejected.
 * out8: host long long [8].  Valid after a call that drew hypotheses (those listed
 * at esacb200_get_hypotheses); after any other call it fails with ESACB200_ERR_ARG. */
int esacb200_get_sample_profile(esacb200_ctx* ctx, long long* out8);
/* With option "sample_trace" = 1 the prefilter / exact kernels of the sampling waves stamp %globaltimer: out512 (host uint64
 * [4 lanes][32 waves][2 kernels: prefilter, exact][2: first CTA start, last CTA end], ns; start = ~0 where nothing ran).
 * Only waves 0-31 of each lane are stamped: with option "sample_waves" above 32 the later waves run but are not traced. */
int esacb200_get_sample_trace(esacb200_ctx* ctx, unsigned long long* out512);

/* Read back intermediates of the last call (any pointer may be NULL), M = esacb200_get_stats' M:
 * poses6 double [M][6] initial hypotheses, cells int32 [M][4][2], tries int32 [M], scores / probs double [M],
 * refined6 double [M][6] (backward, hypotheses_forward: refined poses; forward: only the winner's row is meaningful),
 * losses double [M] (backward).
 * Valid after a call that drew hypotheses on this context: forward, backward (and backward_sharded[_nccl] with M > 0),
 * hypotheses_forward, forward_pack / forward_sharded with M > 0, and forward_ragged / forward_batch[_cameras] (the last
 * image's).  `losses` is valid only after backward and its sharded forms.  After any other call (score_poses, refine_poses,
 * the loss entry points, hypotheses_backward, the batches that run on worker contexts) it fails with
 * ESACB200_ERR_ARG and writes nothing. */
int esacb200_get_hypotheses(esacb200_ctx* ctx, double* poses6, int32_t* cells, int32_t* tries, double* scores,
                            double* probs, double* refined6, double* losses);

/* Copies the last call's scores (double [M]) to `dst` (host or device pointer), stream-ordered on the
 * context's stream; used by the multi-GPU path to feed its all-gather without a host round trip.  Valid after the calls
 * listed at esacb200_get_hypotheses and after score_poses; fails with ESACB200_ERR_ARG after any other call, or when M is
 * not the last call's. */
int esacb200_copy_last_scores(esacb200_ctx* ctx, double* dst, int M);

/* ---- expert stack: inference of the reference's Expert FCN (code/expert.py) for E experts ---------------------------
 * TF32 tensor-core operands with fp32 accumulation and fp32 activations (the regime of torch's default
 * cudnn.allow_tf32 = True).  Only (image, expert) pairs with a positive histogram count run; every layer of all of them is
 * one launch.  Expert e's output for image b does not depend on the other pairs of the call.
 *
 * esacb200_experts_pack: params is a host array of E * ESACB200_EXPERT_TENSORS pointers (host or device memory, float32,
 * contiguous), expert by expert, each in the order conv1.weight, conv1.bias, conv2.weight, ..., res2_skip.weight,
 * res2_skip.bias, res3_conv1.weight, ..., fc3.weight, fc3.bias, mean -- the layers of Expert.__init__ with torch's shapes.
 * packed: device, esacb200_experts_packed_floats(E) floats (16-byte aligned).  Synchronous.
 *
 * esacb200_experts_forward_async: image float32 [image_batch,3,H,W] (image_batch 1: one image for the whole batch, or B);
 * hist float32 [B,E] (pair (b, e) runs when hist[b][e] > 0) or NULL (every pair runs); out float32 [B,E,3,ceil(H/8),
 * ceil(W/8)], zero planes for the pairs that do not run.  Enqueued on the context's stream with no host synchronisation
 * (capturable).  workspace: device, 256-byte aligned, at least esacb200_experts_workspace_bytes(B, E, H, W) bytes; it is
 * the caller's, so reserve it before a capture: a call with less fails (ESACB200_ERR_ARG) before enqueuing anything. */
#define ESACB200_EXPERT_TENSORS 35
#define ESACB200_EXPERTS_MAX 1024
#define ESACB200_EXPERTS_MAX_SIDE 8192
#define ESACB200_EXPERTS_MAX_PAIRS 65535
/* Floats of the packed weights of E experts (-1: E outside [1, ESACB200_EXPERTS_MAX]). */
int64_t esacb200_experts_packed_floats(int E);
/* Workspace bytes of one forward (-1: sizes the forward rejects). */
int64_t esacb200_experts_workspace_bytes(int B, int E, int H, int W);
int esacb200_experts_pack(esacb200_ctx* ctx, int E, const float* const* params, float* packed);
int esacb200_experts_forward_async(esacb200_ctx* ctx, int B, int E, int H, int W, const float* image, int image_batch,
                                   const float* hist, const float* packed, void* workspace, int64_t workspace_bytes,
                                   float* out);

/* ---- gating network: inference of the reference's Gating (code/gating.py) of capacity 1 or 2 over E experts ----------
 * conv1 .. conv3 in fp32; conv4 and res1_conv1..3 on the tensor cores (TF32 operands, fp32 accumulation: the experts'
 * kernel); tanh (capacity 1), the mean over the /8 map, fc1 .. fc3 and log_softmax in fp32.  No split-K and no atomics:
 * image b's output is bitwise independent of the batch, of its place in it and of the run.
 *
 * esacb200_gating_pack: params is a host array of ESACB200_GATING_TENSORS pointers (host or device memory, float32,
 * contiguous) in the order conv1.weight, conv1.bias, ..., conv4.bias, res1_conv1.weight, ..., res1_conv3.bias, fc1.weight,
 * ..., fc3.bias -- the layers of Gating.__init__ with torch's shapes (64 * capacity channels at /8, 64 * capacity^2 in fc1
 * and fc2, E out of fc3).  packed: device, esacb200_gating_packed_floats(E, capacity) floats (16-byte aligned).
 * Synchronous.
 *
 * esacb200_gating_forward_async: image float32 [B,3,H,W]; out_log_probs float32 [B,E] (Gating.forward's output);
 * out_probs float32 [B,E] = exp(out_log_probs), what esacb200_assign_hypotheses_async takes, or NULL.  Enqueued on the
 * context's stream with no host synchronisation (capturable); every argument is checked before anything is enqueued.
 * workspace: device, 256-byte aligned, at least esacb200_gating_workspace_bytes(B, E, capacity, H, W) bytes, the caller's. */
#define ESACB200_GATING_TENSORS 20
/* Floats of the packed weights (-1: E outside [1, ESACB200_EXPERTS_MAX] or capacity not 1 or 2). */
int64_t esacb200_gating_packed_floats(int E, int capacity);
/* Workspace bytes of one forward (-1: sizes the forward rejects: B above ESACB200_EXPERTS_MAX_PAIRS, sides above
 * ESACB200_EXPERTS_MAX_SIDE). */
int64_t esacb200_gating_workspace_bytes(int B, int E, int capacity, int H, int W);
int esacb200_gating_pack(esacb200_ctx* ctx, int E, int capacity, const float* const* params, float* packed);
int esacb200_gating_forward_async(esacb200_ctx* ctx, int B, int E, int capacity, int H, int W, const float* image,
                                  const float* packed, void* workspace, int64_t workspace_bytes, float* out_log_probs,
                                  float* out_probs);

/* Device properties the bench needs without importing a CUDA binding: SM count and name. */
int esacb200_device_info(esacb200_ctx* ctx, int* sm_count, char* name, int name_len);

#ifdef __cplusplus
}
#endif
#endif /* ESAC_B200_H */
