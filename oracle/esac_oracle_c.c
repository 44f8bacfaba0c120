/* CPU ORACLE (C/OpenMP restatement) of the ESAC scoring stage -- TEST / BASELINE INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load
 * this file's library; the product path (esac_b200/) never does.
 *
 * Restates, without OpenCV, the reference's hot loop #1:
 *   getReproErrs (no-Jacobian path)   code/esac/esac_util.h:274-318,355-362
 *   getHypScores                       code/esac/esac_util.h:235-260
 *   the `#pragma omp parallel for` over hypotheses that drives them   esac.cpp:131-140
 * cv::projectPoints (OpenCV, not in the reference tree) is restated from its observable arithmetic
 * (SURVEY.md Appendix A, re-verified against cv2 4.13 by tests/test_oracle_c.py): R = Rodrigues(rvec),
 * Xc = R*X + t in double, z = Zc ? 1/Zc : 1, u = Xc*z*f + cx, result rounded to float.
 *
 * PARITY UNPINNED against the compiled reference (it cannot be built here: no OpenCV C++ headers);
 * pinned against the cv2-based Python oracle (oracle/esac_oracle.py), which executes real OpenCV.
 *
 * Build: gcc -O3 -fopenmp -ffp-contract=off -shared -fPIC -o oracle/_build/libesac_oracle.so oracle/esac_oracle_c.c -lm
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* cv::Rodrigues (vector -> matrix) */
static void rodrigues(const double r[3], double R[9]) {
    double rx = r[0], ry = r[1], rz = r[2];
    double theta = sqrt(rx * rx + ry * ry + rz * rz);
    if (theta < DBL_EPSILON) {
        R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1;
        return;
    }
    double c = cos(theta), s = sin(theta), c1 = 1. - c, it = 1. / theta;
    rx *= it; ry *= it; rz *= it;
    R[0] = c + c1 * rx * rx;      R[1] = c1 * rx * ry - s * rz; R[2] = c1 * rx * rz + s * ry;
    R[3] = c1 * rx * ry + s * rz; R[4] = c + c1 * ry * ry;      R[5] = c1 * ry * rz - s * rx;
    R[6] = c1 * rx * rz - s * ry; R[7] = c1 * ry * rz + s * rx; R[8] = c + c1 * rz * rz;
}

/* Soft-inlier score of one hypothesis over one expert plane (x-outer / y-inner like the reference). */
static double score_one(const float* plane, int H, int W, const double pose6[6], int shiftX, int shiftY, float f,
                        float ppx, float ppy, float tau, float alpha, float beta, float maxReproj, int sub) {
    double R[9];
    rodrigues(pose6, R);
    const double* t = pose6 + 3;
    const double fx = (double)f, cx = (double)ppx, cy = (double)ppy;
    const size_t N = (size_t)H * W;
    double score = 0;
    for (int x = 0; x < W; ++x)
        for (int y = 0; y < H; ++y) {
            const size_t p = (size_t)y * W + x;
            const double X = plane[p], Y = plane[N + p], Z = plane[2 * N + p];
            double xc = R[0] * X + R[1] * Y + R[2] * Z + t[0];
            double yc = R[3] * X + R[4] * Y + R[5] * Z + t[1];
            double zc = R[6] * X + R[7] * Y + R[8] * Z + t[2];
            zc = zc != 0. ? 1. / zc : 1.;
            xc *= zc;
            yc *= zc;
            const float u = (float)(xc * fx + cx), v = (float)(yc * fx + cy);
            const float px = (float)(x * sub + sub / 2 - shiftX), py = (float)(y * sub + sub / 2 - shiftY);
            const float dx = px - u, dy = py - v;
            float l = (float)sqrt((double)dx * dx + (double)dy * dy);
            l = (maxReproj < l) ? maxReproj : l; /* std::min(l, maxReproj) */
            double st = beta * (l - tau);        /* float expression, esac_util.h:248 */
            st = 1 / (1 + exp(-st));
            score += 1 - st;
        }
    return score * (double)(alpha / W / H); /* float factor, esac_util.h:256 */
}

/* scores[h] for all hypotheses; OpenMP over h like esac.cpp:131.  Returns the thread count used. */
int esac_oracle_score(const float* coords, int E, int H, int W, const int64_t* assign, int M, const double* poses6,
                      int shiftX, int shiftY, float f, float ppx, float ppy, float tau, float alpha, float beta,
                      float maxReproj, int sub, double* scores, int nthreads) {
    (void)E;
    int used = 1;
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
    used = omp_get_max_threads();
#endif
    const size_t plane = (size_t)3 * H * W;
#pragma omp parallel for schedule(dynamic, 1)
    for (int h = 0; h < M; ++h)
        scores[h] = score_one(coords + (size_t)assign[h] * plane, H, W, poses6 + 6 * (size_t)h, shiftX, shiftY, f, ppx, ppy,
                              tau, alpha, beta, maxReproj, sub);
    return used;
}

int esac_oracle_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
