/* Host-side test hooks of libesac_b200.so.
 *
 * These run single geometry primitives of esac_b200/csrc/esac_geom.cuh / esac_rng.cuh -- the very
 * functions the CUDA kernels call -- on the CPU, so the `-m "not gpu"` tests can check them against
 * OpenCV without a GPU.  They are NOT a CPU fallback: no forward/backward pipeline exists on the host.
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

#ifdef __cplusplus
}
#endif
#endif
