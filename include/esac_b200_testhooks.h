/* Test hooks of libesac_b200.so.
 *
 * The esacb200_host_* hooks run single geometry primitives of esac_b200/csrc/esac_geom.cuh / esac_rng.cuh -- the very
 * functions the CUDA kernels call -- on the CPU, so the `-m "not gpu"` tests can check them against OpenCV without a
 * GPU.  They are NOT a CPU fallback: no forward/backward pipeline exists on the host.  esacb200_test_experts_conv runs
 * one layer of the expert stack's device kernels on caller-owned device buffers, so a test can hold that layer alone
 * to a reference; esacb200_test_gathered does the same for the two kernels that merge the shards of a sharded call.
 */
#ifndef ESAC_B200_TESTHOOKS_H
#define ESAC_B200_TESTHOOKS_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* cv::Rodrigues vector -> matrix (+ 3x9 Jacobian, may be NULL) and matrix -> vector. */
void esacb200_host_rodrigues(const double r[3], double R[9], double J[27]);
void esacb200_host_rodrigues_inv(const double R[9], double r[3]);
/* All P3P solutions of 3 unit bearings y[3][3] and 3 scene points x[3][3]; returns the count. */
int esacb200_host_p3p_all(const double* y9, const double* x9, double* Rs36, double* ts12);
/* solvePnP(4 points, SOLVEPNP_P3P) replacement: obj float[4][3], img float[4][2]; pose6 = rvec,tvec.
 * Returns 1 when a pose was found.  *gate = result of the 4-point reprojection gate (esac_util.h:202-223). */
int esacb200_host_p3p_pose(const float* obj12, const float* img8, float f, float ppx, float ppy, float tau,
                           double* pose6, int* gate);
/* One sampling try on given correspondences: *may_pass = float prefilter verdict (0 = certainly rejected),
 * *accept = exact verdict (P3P solved and the 4-point gate passed).  Invariant: accept implies may_pass. */
void esacb200_host_try(const float* obj12, const float* img8, float f, float ppx, float ppy, float tau, float margin,
                       int* may_pass, int* accept);
/* n sampling tries (obj float[n][4][3], img float[n][4][2]) as prefilter_kernel sees them: may_pass[i] = float prefilter
 * verdict at its shipping band, hint[i] = its "near-certain" hint at hint_frac * tau (option sample_hint), accept[i] = exact
 * verdict (as esacb200_host_try's).  Invariants: hint implies may_pass, accept implies may_pass. */
void esacb200_host_tries_hint(int n, const float* obj12n, const float* img8n, float f, float ppx, float ppy, float tau,
                              float hint_frac, int* may_pass, int* hint, int* accept);
/* The sampling kernels' verdict path: the same exact decision, but a try none of whose P3P candidates brings the 4th point
 * within 1.25 tau + 1 px is rejected before polish / alignment (p3p_solve's early exit).  Only the candidate that is far ahead
 * on the 4th point is polished (p3p_solve's favourite).  Invariants: *accept equals esacb200_host_try's, and for an accepted
 * try pose6 (may be NULL) equals esacb200_host_p3p_pose's. */
void esacb200_host_try_verdict(const float* obj12, const float* img8, float f, float ppx, float ppy, float tau, int* accept,
                               double* pose6);
/* cv::projectPoints for one point: float-rounded pixel + fp64 pixel + 2x6 Jacobian (rvec | tvec columns). */
void esacb200_host_project(const double pose6[6], float f, float ppx, float ppy, const float X[3], float uv_f[2],
                           double uv[2], double J12[12]);
/* loss() (esac_loss.h:66-83) on two camera->world 4x4 row-major doubles; dLoss() (94-210) on poses. */
double esacb200_host_loss(const double* T1, const double* T2, double wRot, double wTrans, double cut);
void esacb200_host_dloss(const double est6[6], const double gt6[6], double wRot, double wTrans, double cut,
                         double out6[6]);
void esacb200_host_pose2trans(const double pose6[6], double T16[16]);
void esacb200_host_trans2pose(const double T16[16], double pose6[6]);
/* dProjectdObj (esac_derivative.h:47-102). */
void esacb200_host_dprojectdobj(const float pt[2], const float obj[3], const double pose6[6], float f, float ppx,
                                float ppy, float maxReproj, double out3[3]);
/* Pseudo-inverse of a symmetric 6x6 (cv::Mat::inv(DECOMP_SVD) semantics). */
void esacb200_host_pinv6(const double A[36], double out[36]);
/* CTAs per refinement job for `jobs` jobs on an N-cell map with `coresident` co-resident refinement CTAs and the options
 * refine_group / refine_jobs_per_group: the one rule the host and the stream-ordered backward's refinement kernel both use. */
int esacb200_host_pick_group(int N, int coresident, int group_opt, int jobs_per_group, int jobs);
/* Minimal set of try (seed, h, t): cells int[4][2] (x, y). */
void esacb200_host_draw_cells(uint64_t seed, uint32_t h, uint32_t t, int W, int H, int32_t* cells8);
/* The node types (cudaGraphNodeType values) of a CUDA graph's top level, through the runtime the library uses: writes up
 * to `cap` of them to `types` and returns the node count, or -1 if the runtime refuses the graph. */
int esacb200_graph_node_types(void* graph, int* types, int cap);

struct esacb200_ctx;
/* On the device, on the context's stream, without a host synchronisation: the expert stack's active list of B * E pairs
 * from hist [B,E] (NULL: every pair) into hdr, then one implicit-GEMM convolution of every active pair p = b * E + e
 * (experts_conv_kernel, as ExpertStack and GatingNet run it).  Pair p's block is pairs + p * pair_floats: its NHWC input
 * [hin][win][cin] at in_off, its output [hout][wout][cout] at out_off, and the residual added after the ReLU at res_off
 * (-1: none; res_off == out_off: in place).  Expert e's weights [cout][k][k][cin] are packed + w_off + e * cout * k * k
 * * cin, its biases packed + b_off + e * cout.  hout, wout = ceil(hin / stride), ceil(win / stride).  hdr holds
 * 16 + 2 * B * E ints: the active count, the ascending active list, then B * E flags.  The kernel's contract: k 1 or 3,
 * stride 1 or 2 (not k 1 with stride 2), cin a multiple of 32, cout even, every offset and pair_floats a multiple of 4,
 * the regions inside a block, packed and pairs 16-byte aligned.  Anything else is refused with ESACB200_ERR_ARG. */
int esacb200_test_experts_conv(struct esacb200_ctx* ctx, int B, int E, const float* hist, const float* packed, int64_t w_off,
                               int64_t b_off, int k, int stride, int cin, int cout, int hin, int win, int relu, float* pairs,
                               int64_t pair_floats, int64_t in_off, int64_t out_off, int64_t res_off, int* hdr);
/* The two kernels that merge the shards of a sharded call, on caller-owned device buffers, on the context's stream; the hook
 * synchronises that stream before it returns.  At least one of gathered and pairs is non-NULL.
 * gathered != NULL: select_gathered_kernel (esacb200_forward_sharded's selection) over `world` records of M_pad + 21 doubles
 * laid out as esacb200_forward_pack writes them; out_record receives 20 floats: the winner's pose [16], its expert, the
 * bad-assignment flag, the global index of the winner and its rank (winner and rank -1 when no record holds a hypothesis).
 * pairs != NULL: rescale_probs_gathered_kernel (the NCCL backward's probabilities) over `world` (max, sum exp) pairs [world][2]
 * and one shard's M scores: norm_out[2] = (global max, global sum exp), probs[M], and contrib[M] the ascending local indices
 * whose probability is not below ESACB200_PROB_THRESH, *n_contrib of them.  scores, probs and contrib may be NULL when M = 0.
 * The kernels' contract: world >= 1; M_pad >= 1 with world * M_pad < 2^31; M >= 0; doubles 8-byte and ints 4-byte aligned;
 * in every record 0 <= M <= M_pad and hyp_stride >= 1.  Arguments outside it are refused with ESACB200_ERR_ARG (the records'
 * contents are the caller's to keep). */
int esacb200_test_gathered(struct esacb200_ctx* ctx, int world, int M_pad, const double* gathered, float* out_record,
                           const double* pairs, const double* scores, int M, double* norm_out, double* probs, int* contrib,
                           int* n_contrib);

#ifdef __cplusplus
}
#endif
#endif
