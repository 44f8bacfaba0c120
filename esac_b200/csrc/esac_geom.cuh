// fp64 geometry primitives of the ESAC hot path, written from the published math (no OpenCV):
//   * Rodrigues vector<->matrix with the analytic 3x9 Jacobian   (replaces cv::Rodrigues; used at
//     esac_util.h:540,560, esac_loss.h:102-103, esac_derivative.h:290, esac.cpp:440)
//   * pinhole projection in the reference's precision mix + its 2x6 pose Jacobian
//                                                              (replaces cv::projectPoints; esac_util.h:202,312,323, esac.cpp:410)
//   * P3P from three 2D-3D correspondences, 4th point disambiguates
//                                                              (replaces cv::solvePnP(SOLVEPNP_P3P); esac_util.h:189-197, esac_derivative.h:153,164)
//   * small dense helpers: 6x6 Cholesky solve, symmetric Jacobi eigen-decomposition (SVD pseudo-inverse,
//     esac.cpp:434)
// Everything is __host__ __device__ so the CPU test-hooks in capi_testhooks.cu can check the very same
// code against cv2 without a GPU.
#pragma once
#include <math.h>
#include <float.h>
#include <stdint.h>

#ifndef ESAC_HD
#ifdef __CUDACC__
#define ESAC_HD __host__ __device__ __forceinline__
#else
#define ESAC_HD inline
#endif
#endif
#ifdef __CUDACC__
#define ESAC_HDN inline __host__ __device__ __noinline__
#else
#define ESAC_HDN inline
#endif

namespace esacb200 {

constexpr double kEps = 0.00000001;       // esac_util.h:39
constexpr double kPiRef = 3.1415926;      // esac_util.h:40 (used by loss())
constexpr double kPi = 3.14159265358979323846;  // CV_PI (used by dLoss())
constexpr double kProbThresh = 0.001;     // esac_derivative.h:33
constexpr double kMaxLoss = 10000000.0;   // esac_loss.h:33

struct Pose {
    double r[3];  // axis-angle (OpenCV rvec), world -> camera
    double t[3];  // translation (OpenCV tvec)
};

// ---------------------------------------------------------------------------------------------
// Rodrigues
// ---------------------------------------------------------------------------------------------
// R row-major 3x3.  J (optional, 27 doubles): J[i*9 + k] = d R[k] / d r[i]  (OpenCV's 3x9 layout).
ESAC_HD void rodrigues_v2m(const double r[3], double R[9], double* J) {
    double rx = r[0], ry = r[1], rz = r[2];
    double theta = sqrt(rx * rx + ry * ry + rz * rz);
    if (theta < DBL_EPSILON) {
        R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1;
        if (J) {
            for (int i = 0; i < 27; ++i) J[i] = 0;
            J[5] = J[15] = J[19] = -1;
            J[7] = J[11] = J[21] = 1;
        }
        return;
    }
    double c = cos(theta), s = sin(theta), c1 = 1. - c, itheta = 1. / theta;
    rx *= itheta; ry *= itheta; rz *= itheta;
    double rrt[9] = {rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz};
    double rxm[9] = {0, -rz, ry, rz, 0, -rx, -ry, rx, 0};
    const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    for (int k = 0; k < 9; ++k) R[k] = c * I[k] + c1 * rrt[k] + s * rxm[k];
    if (J) {
        double drrt[27] = {rx + rx, ry, rz, ry, 0, 0, rz, 0, 0,
                           0, rx, 0, rx, ry + ry, rz, 0, rz, 0,
                           0, 0, rx, 0, 0, ry, rx, ry, rz + rz};
        const double drx[27] = {0, 0, 0, 0, 0, -1, 0, 1, 0,
                                0, 0, 1, 0, 0, 0, -1, 0, 0,
                                0, -1, 0, 1, 0, 0, 0, 0, 0};
        for (int i = 0; i < 3; ++i) {
            double ri = i == 0 ? rx : (i == 1 ? ry : rz);
            double a0 = -s * ri, a1 = (s - 2 * c1 * itheta) * ri, a2 = c1 * itheta;
            double a3 = (c - s * itheta) * ri, a4 = s * itheta;
            for (int k = 0; k < 9; ++k)
                J[i * 9 + k] = a0 * I[k] + a1 * rrt[k] + a2 * drrt[i * 9 + k] + a3 * rxm[k] + a4 * drx[i * 9 + k];
        }
    }
}

// Rotation matrix (assumed orthonormal) -> axis-angle, OpenCV's branch structure.
ESAC_HD void rodrigues_m2v(const double R[9], double r[3]) {
    double rx = R[7] - R[5], ry = R[2] - R[6], rz = R[3] - R[1];
    double s = sqrt((rx * rx + ry * ry + rz * rz) * 0.25);
    double c = (R[0] + R[4] + R[8] - 1) * 0.5;
    c = c > 1. ? 1. : (c < -1. ? -1. : c);
    double theta = acos(c);
    if (s < 1e-5) {
        if (c > 0) {
            r[0] = r[1] = r[2] = 0;
        } else {
            double t;
            t = (R[0] + 1) * 0.5; rx = sqrt(t > 0. ? t : 0.);
            t = (R[4] + 1) * 0.5; ry = sqrt(t > 0. ? t : 0.) * (R[1] < 0 ? -1. : 1.);
            t = (R[8] + 1) * 0.5; rz = sqrt(t > 0. ? t : 0.) * (R[2] < 0 ? -1. : 1.);
            if (fabs(rx) < fabs(ry) && fabs(rx) < fabs(rz) && ((R[5] > 0) != (ry * rz > 0))) rz = -rz;
            theta /= sqrt(rx * rx + ry * ry + rz * rz);
            r[0] = rx * theta; r[1] = ry * theta; r[2] = rz * theta;
        }
    } else {
        double vth = 1 / (2 * s);
        vth *= theta;
        r[0] = rx * vth; r[1] = ry * vth; r[2] = rz * vth;
    }
}

// ---------------------------------------------------------------------------------------------
// projection (cv::projectPoints semantics without distortion): fp64 transform, z ? 1/z : 1,
// u = x*z*f + cx.  No FMA contraction so the value rounds to float like the CPU library's.
// ---------------------------------------------------------------------------------------------
#ifdef __CUDA_ARCH__
#define ESAC_MUL(a, b) __dmul_rn((a), (b))
#define ESAC_ADD(a, b) __dadd_rn((a), (b))
#else
#define ESAC_MUL(a, b) ((a) * (b))
#define ESAC_ADD(a, b) ((a) + (b))
#endif

// Two fp32 values side by side (float2), one IEEE round-to-nearest operation per lane.  The _rn intrinsics keep the
// compiler from contracting a product into a following sum, so every lane rounds exactly where the code says.
#ifdef __CUDACC__
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
#endif

ESAC_HD void transform_point(const double R[9], const double t[3], double X, double Y, double Z,
                             double& x, double& y, double& z) {
    x = ESAC_ADD(ESAC_ADD(ESAC_ADD(ESAC_MUL(R[0], X), ESAC_MUL(R[1], Y)), ESAC_MUL(R[2], Z)), t[0]);
    y = ESAC_ADD(ESAC_ADD(ESAC_ADD(ESAC_MUL(R[3], X), ESAC_MUL(R[4], Y)), ESAC_MUL(R[5], Z)), t[1]);
    z = ESAC_ADD(ESAC_ADD(ESAC_ADD(ESAC_MUL(R[6], X), ESAC_MUL(R[7], Y)), ESAC_MUL(R[8], Z)), t[2]);
}

// Projects one point; returns the float-rounded pixel position like cv::projectPoints into Point2f.
ESAC_HD void project_point_f(const double R[9], const double t[3], double f, double cx, double cy,
                             float Xf, float Yf, float Zf, float& u, float& v) {
    double x, y, z;
    transform_point(R, t, (double)Xf, (double)Yf, (double)Zf, x, y, z);
    z = z != 0. ? 1. / z : 1.;
    x = ESAC_MUL(x, z);
    y = ESAC_MUL(y, z);
    u = (float)ESAC_ADD(ESAC_MUL(x, f), cx);
    v = (float)ESAC_ADD(ESAC_MUL(y, f), cy);
}

// Reprojection error exactly as getReproErrs stores it (esac_util.h:355-360) *before* the clamp:
// float difference of float points, norm in double, cast to float.
ESAC_HD float repro_err_f(const double R[9], const double t[3], double f, double cx, double cy,
                          float Xf, float Yf, float Zf, float px, float py) {
    float u, v;
    project_point_f(R, t, f, cx, cy, Xf, Yf, Zf, u, v);
    float dx = px - u, dy = py - v;
    return (float)sqrt((double)dx * (double)dx + (double)dy * (double)dy);
}

// Projection + 2x6 Jacobian w.r.t. (rvec, tvec) in fp64 (cv::projectPoints' dpdr | dpdt).
// dRdr: Rodrigues Jacobian (27).  Ju/Jv: 6 each.  u/v are the unrounded fp64 pixel positions.
ESAC_HD void project_point_jac(const double R[9], const double t[3], const double dRdr[27], double f,
                               double cx, double cy, double X, double Y, double Z, double& u, double& v,
                               double Ju[6], double Jv[6]) {
    double x = R[0] * X + R[1] * Y + R[2] * Z + t[0];
    double y = R[3] * X + R[4] * Y + R[5] * Z + t[1];
    double z = R[6] * X + R[7] * Y + R[8] * Z + t[2];
    z = z != 0. ? 1. / z : 1.;
    x *= z;
    y *= z;
    u = x * f + cx;
    v = y * f + cy;
    // d(x*z, y*z)/d(Xc) rows
    double dxdX[3] = {z, 0, -x * z};
    double dydX[3] = {0, z, -y * z};
    for (int i = 0; i < 3; ++i) {
        const double* d = dRdr + i * 9;
        double dX = d[0] * X + d[1] * Y + d[2] * Z;
        double dY = d[3] * X + d[4] * Y + d[5] * Z;
        double dZ = d[6] * X + d[7] * Y + d[8] * Z;
        Ju[i] = f * (dxdX[0] * dX + dxdX[2] * dZ);
        Jv[i] = f * (dydX[1] * dY + dydX[2] * dZ);
        Ju[3 + i] = f * dxdX[i];
        Jv[3 + i] = f * dydX[i];
    }
}

// dProjectdObj (esac_derivative.h:47-102): 1x3 derivative of the reprojection error norm w.r.t. the
// scene point.  pt = pixel position (float in the reference), obj = float scene point.
ESAC_HD void d_project_d_obj(float ptx_f, float pty_f, float Xf, float Yf, float Zf, const double R[9],
                             const double t[3], double f, double ppx, double ppy, double max_reproj,
                             double out[3]) {
    double X = (double)Xf, Y = (double)Yf, Z = (double)Zf;
    double ox = R[0] * X + R[1] * Y + R[2] * Z + t[0];
    double oy = R[3] * X + R[4] * Y + R[5] * Z + t[1];
    double oz = R[6] * X + R[7] * Y + R[8] * Z + t[2];
    out[0] = out[1] = out[2] = 0;
    if (fabs(oz) < kEps) return;
    double px = f * ox / oz + ppx;
    double py = f * oy / oz + ppy;
    double ptx = (double)ptx_f, pty = (double)pty_f;
    double err = sqrt((ptx - px) * (ptx - px) + (pty - py) * (pty - py));
    if (!(err <= max_reproj)) return;  // also drops NaN like `err > maxReproErr` never does; see DESIGN.md
    err += kEps;
    for (int c = 0; c < 3; ++c) {
        double pxd = f * R[c] / oz - f * ox / oz / oz * R[6 + c];
        double pyd = f * R[3 + c] / oz - f * oy / oz / oz * R[6 + c];
        out[c] = 0.5 / err * (2 * (ptx - px) * -pxd + 2 * (pty - py) * -pyd);
    }
}

// ---------------------------------------------------------------------------------------------
// small dense algebra (templated: the P3P core also runs in float as a rejection prefilter)
// ---------------------------------------------------------------------------------------------
template <typename T> struct Num;
template <> struct Num<double> {
    static ESAC_HD double sqrt_(double v) { return sqrt(v); }
    static ESAC_HD double acos_(double v) { return acos(v); }
    static ESAC_HD double cos_(double v) { return cos(v); }
    static ESAC_HD double cbrt_(double v) { return cbrt(v); }
    static ESAC_HD double abs_(double v) { return fabs(v); }
    static ESAC_HD double div_(double a, double b) { return a / b; }
    static constexpr double kRelTiny = 1e-14;   // "this coefficient is zero" threshold
    static constexpr double kDiscTol = 1e-13;   // slightly negative discriminants are clamped to 0
    static constexpr double kUncertain = 0.0;   // no uncertainty band in double
};
template <> struct Num<float> {
#ifdef __CUDA_ARCH__
    // the float path only feeds a conservative prefilter: MUFU-based approximations are enough
    static ESAC_HD float sqrt_(float v) { float r; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v)); return r; }
    static ESAC_HD float cos_(float v) { return __cosf(v); }
    static ESAC_HD float div_(float a, float b) { return __fdividef(a, b); }
#else
    static ESAC_HD float sqrt_(float v) { return sqrtf(v); }
    static ESAC_HD float cos_(float v) { return cosf(v); }
    static ESAC_HD float div_(float a, float b) { return a / b; }
#endif
    static ESAC_HD float acos_(float v) { return acosf(v); }
    static ESAC_HD float cbrt_(float v) { return cbrtf(v); }
    static ESAC_HD float abs_(float v) { return fabsf(v); }
    static constexpr float kRelTiny = 1e-6f;
    static constexpr float kDiscTol = 1e-5f;
    static constexpr float kUncertain = 2e-3f;  // sign decisions closer to zero than this (relative) are "uncertain"
};

template <typename T>
ESAC_HD T det3(const T A[9]) {
    return A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
}

// adjugate (transpose of the cofactor matrix) of a 3x3
template <typename T>
ESAC_HD void adj3(const T A[9], T B[9]) {
    B[0] = A[4] * A[8] - A[5] * A[7];
    B[1] = A[2] * A[7] - A[1] * A[8];
    B[2] = A[1] * A[5] - A[2] * A[4];
    B[3] = A[5] * A[6] - A[3] * A[8];
    B[4] = A[0] * A[8] - A[2] * A[6];
    B[5] = A[2] * A[3] - A[0] * A[5];
    B[6] = A[3] * A[7] - A[4] * A[6];
    B[7] = A[1] * A[6] - A[0] * A[7];
    B[8] = A[0] * A[4] - A[1] * A[3];
}

template <typename T>
ESAC_HD T trace_prod3(const T A[9], const T B[9]) {  // tr(A*B)
    return A[0] * B[0] + A[1] * B[3] + A[2] * B[6] + A[3] * B[1] + A[4] * B[4] + A[5] * B[7] + A[6] * B[2] +
           A[7] * B[5] + A[8] * B[8];
}

// The nearest rotation of X (its orthogonal polar factor, what OpenCV takes as U*V^T of an SVD before Rodrigues), in place:
// Newton's iteration X <- (X + X^-T) / 2, eight steps, stopping early on a singular X.
ESAC_HD void polar_newton(double X[9]) {
    for (int it = 0; it < 8; ++it) {
        double C[9];
        adj3(X, C);
        double dd = X[0] * C[0] + X[1] * C[3] + X[2] * C[6];
        if (!(fabs(dd) > 0)) break;
        double Y[9];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) Y[r * 3 + c] = 0.5 * (X[r * 3 + c] + C[c * 3 + r] / dd);  // X^-T[r][c] = adj[c][r]/det
        for (int i = 0; i < 9; ++i) X[i] = Y[i];
    }
}

// The inverse of the affine 4x4 T (row major, last row 0 0 0 1) as cv::Mat::inv and torch's .inverse() compute it, not
// the rigid shortcut: rotation block Ri = adj(R) / det(R), translation t = -Ri * T[:3,3].
ESAC_HD void affine_inverse(const double T[16], double Ri[9], double t[3]) {
    double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
    double B[9];
    adj3(R, B);
    double d = R[0] * B[0] + R[1] * B[3] + R[2] * B[6];
    for (int i = 0; i < 9; ++i) Ri[i] = B[i] / d;
    for (int r = 0; r < 3; ++r) t[r] = -(Ri[r * 3] * T[3] + Ri[r * 3 + 1] * T[7] + Ri[r * 3 + 2] * T[11]);
}

ESAC_HD bool solve3(const double A[9], const double b[3], double x[3]) {
    double B[9];
    adj3(A, B);
    double d = A[0] * B[0] + A[1] * B[3] + A[2] * B[6];
    if (!(fabs(d) > 0)) return false;
    double id = 1. / d;
    x[0] = (B[0] * b[0] + B[1] * b[1] + B[2] * b[2]) * id;
    x[1] = (B[3] * b[0] + B[4] * b[1] + B[5] * b[2]) * id;
    x[2] = (B[6] * b[0] + B[7] * b[1] + B[8] * b[2]) * id;
    return true;
}

// Solve the SPD system A x = b (n = 6) by Cholesky.  A is full symmetric row-major.
ESAC_HD bool chol_solve6(const double A[36], const double b[6], double x[6]) {
    double L[36];
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j <= i; ++j) {
            double s = A[i * 6 + j];
            for (int k = 0; k < j; ++k) s -= L[i * 6 + k] * L[j * 6 + k];
            if (i == j) {
                if (!(s > 0)) return false;
                L[i * 6 + i] = sqrt(s);
            } else {
                L[i * 6 + j] = s / L[j * 6 + j];
            }
        }
    double y[6];
    for (int i = 0; i < 6; ++i) {
        double s = b[i];
        for (int k = 0; k < i; ++k) s -= L[i * 6 + k] * y[k];
        y[i] = s / L[i * 6 + i];
    }
    for (int i = 5; i >= 0; --i) {
        double s = y[i];
        for (int k = i + 1; k < 6; ++k) s -= L[k * 6 + i] * x[k];
        x[i] = s / L[i * 6 + i];
    }
    return true;
}

// Pseudo-inverse of a symmetric PSD 6x6 the way cv::Mat::inv(DECOMP_SVD) does it (esac.cpp:434):
// singular values below 2*DBL_EPSILON*sum(w) are dropped.  Cyclic Jacobi eigen-decomposition.
ESAC_HDN void pinv_sym6(const double Ain[36], double out[36]) {
    double A[36], V[36];
    for (int i = 0; i < 36; ++i) { A[i] = Ain[i]; V[i] = 0; }
    for (int i = 0; i < 6; ++i) V[i * 6 + i] = 1;
    for (int sweep = 0; sweep < 60; ++sweep) {
        double off = 0, dg = 0;
        for (int i = 0; i < 6; ++i) {
            dg += A[i * 6 + i] * A[i * 6 + i];
            for (int j = i + 1; j < 6; ++j) off += A[i * 6 + j] * A[i * 6 + j];
        }
        if (!(off > 1e-60 * dg) || off == 0) break;
        for (int p = 0; p < 5; ++p)
            for (int q = p + 1; q < 6; ++q) {
                double apq = A[p * 6 + q];
                if (apq == 0) continue;
                double app = A[p * 6 + p], aqq = A[q * 6 + q];
                double tau = (aqq - app) / (2 * apq);
                double t = (tau >= 0 ? 1. : -1.) / (fabs(tau) + sqrt(1 + tau * tau));
                double c = 1 / sqrt(1 + t * t), s = t * c;
                for (int k = 0; k < 6; ++k) {
                    double akp = A[k * 6 + p], akq = A[k * 6 + q];
                    A[k * 6 + p] = c * akp - s * akq;
                    A[k * 6 + q] = s * akp + c * akq;
                }
                for (int k = 0; k < 6; ++k) {
                    double apk = A[p * 6 + k], aqk = A[q * 6 + k];
                    A[p * 6 + k] = c * apk - s * aqk;
                    A[q * 6 + k] = s * apk + c * aqk;
                }
                for (int k = 0; k < 6; ++k) {
                    double vkp = V[k * 6 + p], vkq = V[k * 6 + q];
                    V[k * 6 + p] = c * vkp - s * vkq;
                    V[k * 6 + q] = s * vkp + c * vkq;
                }
            }
    }
    double sum = 0;
    for (int i = 0; i < 6; ++i) sum += fabs(A[i * 6 + i]);
    double thr = sum * (DBL_EPSILON * 2);
    double w[6];
    for (int i = 0; i < 6; ++i) {
        double e = A[i * 6 + i];
        w[i] = (fabs(e) > thr) ? 1. / e : 0.;
    }
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) {
            double s = 0;
            for (int k = 0; k < 6; ++k) s += V[i * 6 + k] * w[k] * V[j * 6 + k];
            out[i * 6 + j] = s;
        }
}

// ---------------------------------------------------------------------------------------------
// P3P.  Three unit bearing vectors y[i] (camera frame), three scene points x[i].  Unknown depths
// lam[i] > 0 with |lam_i y_i - lam_j y_j|^2 = |x_i - x_j|^2.  The two homogeneous conics
//     D1 = a23*Q12 - a12*Q23,   D2 = a23*Q13 - a13*Q23
// share the solutions; a degenerate member D1 + g*D2 of their pencil (cubic in g) splits into two
// lines, each line meets a conic in <= 2 points -> <= 4 depth triples (p3p_lambdas, float or double),
// polished by Gauss-Newton on the three distance equations, then turned into (R, t) by aligning the two
// congruent triangles (p3p_solve, double).
// ---------------------------------------------------------------------------------------------
template <typename T>
ESAC_HD T quad3(const T D[9], const T a[3], const T b[3]) {  // a^T D b
    return a[0] * (D[0] * b[0] + D[1] * b[1] + D[2] * b[2]) + a[1] * (D[3] * b[0] + D[4] * b[1] + D[5] * b[2]) +
           a[2] * (D[6] * b[0] + D[7] * b[1] + D[8] * b[2]);
}

// Real roots of c3 g^3 + c2 g^2 + c1 g + c0, produced ON DEMAND: the P3P below almost always needs only the first one, and a
// root costs a cosine plus a Newton polish with four divisions -- a third of the solver's dependency chain when all three are
// computed up front.  cubic_setup returns the number of real roots, cubic_root(i) the i-th of them.
template <typename T>
struct Cubic {
    T a, b, c;       // monic coefficients
    T sq, th;        // three real roots: -2 sqrt(Q), acos(R / sqrt(Q^3))
    T r0, r1;        // closed-form roots of the degenerate (quadratic / linear) and the one-real-root case
    int kind;        // 0: r0 / r1 as they are, 1: trigonometric
};
template <typename T>
ESAC_HD int cubic_setup(T c3, T c2, T c1, T c0, Cubic<T>& q) {
    using N = Num<T>;
    q.kind = 0; q.r0 = q.r1 = 0; q.a = q.b = q.c = 0; q.sq = q.th = 0;
    T scale = N::abs_(c3) + N::abs_(c2) + N::abs_(c1) + N::abs_(c0);
    if (!(scale > 0)) return 0;
    if (N::abs_(c3) < N::kRelTiny * scale) {  // quadratic (the root at infinity is handled by the caller)
        if (N::abs_(c2) < N::kRelTiny * scale) {
            if (N::abs_(c1) > 0) { q.r0 = N::div_(-c0, c1); return 1; }
            return 0;
        }
        T disc = c1 * c1 - 4 * c2 * c0;
        if (disc < 0) return 0;
        T sq = N::sqrt_(disc);
        T w = T(-0.5) * (c1 + (c1 >= 0 ? sq : -sq));
        q.r0 = N::div_(w, c2);
        if (w != 0) { q.r1 = N::div_(c0, w); return 2; }
        return 1;
    }
    const T ic3 = N::div_(T(1), c3);
    q.a = c2 * ic3; q.b = c1 * ic3; q.c = c0 * ic3;
    const T a = q.a, b = q.b, c = q.c;
    T Q = (a * a - 3 * b) * T(1.0 / 9.0), Rr = (2 * a * a * a - 9 * a * b + 27 * c) * T(1.0 / 54.0);
    T Q3 = Q * Q * Q;
    if (Rr * Rr < Q3) {
        q.th = N::acos_(N::div_(Rr, N::sqrt_(Q3)));
        q.sq = -2 * N::sqrt_(Q);
        q.kind = 1;
        return 3;
    }
    T A = -(Rr >= 0 ? T(1) : T(-1)) * N::cbrt_(N::abs_(Rr) + N::sqrt_(Rr * Rr - Q3));
    T B = A != 0 ? N::div_(Q, A) : 0;
    q.r0 = A + B - a * T(1.0 / 3.0);
    q.kind = 2;
    return 1;
}
template <typename T>
ESAC_HD T cubic_root(const Cubic<T>& q, int i) {
    using N = Num<T>;
    if (q.kind == 0) return i == 0 ? q.r0 : q.r1;
    T g;
    if (q.kind == 1) {
        const T twopi = T(2 * 3.14159265358979323846), third = T(1.0 / 3.0);
        const T ang = i == 0 ? q.th : (i == 1 ? q.th + twopi : q.th - twopi);
        g = q.sq * N::cos_(ang * third) - q.a * third;
    } else {
        g = q.r0;
    }
    for (int it = 0; it < 4; ++it) {  // Newton polish on the monic cubic
        T fv = ((g + q.a) * g + q.b) * g + q.c;
        T dv = (3 * g + 2 * q.a) * g + q.b;
        if (!(N::abs_(dv) > 0)) break;
        g -= N::div_(fv, dv);
    }
    return g;
}
// Intersect the line {lam : l.lam = 0} with the conic lam^T D lam = 0; appends direction vectors.
// (kept out of line: three call sites, and the sampling prefilter is instruction-cache bound)
template <typename T>
ESAC_HDN int line_conic(const T l[3], const T D[9], T sol[][3], int n, bool& uncertain) {
    using N = Num<T>;
    int k = 0;
    if (N::abs_(l[1]) > N::abs_(l[k])) k = 1;
    if (N::abs_(l[2]) > N::abs_(l[k])) k = 2;
    if (!(N::abs_(l[k]) > 0)) return n;
    int i = (k + 1) % 3, j = (k + 2) % 3;
    T u[3] = {0, 0, 0}, v[3] = {0, 0, 0};
    const T ilk = N::div_(T(1), l[k]);
    u[i] = 1; u[k] = -l[i] * ilk;
    v[j] = 1; v[k] = -l[j] * ilk;
    T A = quad3(D, u, u), B = quad3(D, u, v), C = quad3(D, v, v);
    T disc = B * B - A * C;
    T mag = B * B + N::abs_(A * C);
    if (N::abs_(disc) < N::kUncertain * mag) uncertain = true;
    if (disc < -N::kDiscTol * mag) return n;
    if (disc < 0) disc = 0;
    T sq = N::sqrt_(disc);
    T q = -(B + (B >= 0 ? sq : -sq));
    if (N::abs_(A) >= N::abs_(C)) {
        if (!(N::abs_(A) > 0)) return n;
        T a1 = N::div_(q, A), a2 = (q != 0) ? N::div_(C, q) : a1;  // alpha = (-B +- sq)/A, beta = 1 (stable form)
        for (int s = 0; s < 2; ++s) {
            T al = s == 0 ? a1 : a2;
            for (int c = 0; c < 3; ++c) sol[n][c] = al * u[c] + v[c];
            ++n;
        }
    } else {
        T b1 = N::div_(q, C), b2 = (q != 0) ? N::div_(A, q) : b1;
        for (int s = 0; s < 2; ++s) {
            T be = s == 0 ? b1 : b2;
            for (int c = 0; c < 3; ++c) sol[n][c] = u[c] + be * v[c];
            ++n;
        }
    }
    return n;
}

template <typename T>
ESAC_HD void cross3(const T a[3], const T b[3], T c[3]) {
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}

// Orthonormal frame of a triangle: e1 along p0-p1, e3 along (p0-p1) x (p1-p2), e2 = e3 x e1 (columns of F).
template <typename T>
ESAC_HD bool tri_frame(const T p0[3], const T p1[3], const T p2[3], T F[9]) {
    using N = Num<T>;
    T d1[3] = {p0[0] - p1[0], p0[1] - p1[1], p0[2] - p1[2]};
    T d2[3] = {p1[0] - p2[0], p1[1] - p2[1], p1[2] - p2[2]};
    T n1 = N::sqrt_(d1[0] * d1[0] + d1[1] * d1[1] + d1[2] * d1[2]);
    if (!(n1 > 0)) return false;
    const T in1 = N::div_(T(1), n1);
    T e1[3] = {d1[0] * in1, d1[1] * in1, d1[2] * in1};
    T e3[3];
    cross3(d1, d2, e3);
    T n3 = N::sqrt_(e3[0] * e3[0] + e3[1] * e3[1] + e3[2] * e3[2]);
    if (!(n3 > 0)) return false;
    const T in3 = N::div_(T(1), n3);
    e3[0] *= in3; e3[1] *= in3; e3[2] *= in3;
    T e2[3];
    cross3(e3, e1, e2);
    for (int r = 0; r < 3; ++r) {
        F[r * 3 + 0] = e1[r];
        F[r * 3 + 1] = e2[r];
        F[r * 3 + 2] = e3[r];
    }
    return true;
}

// Rigid transform mapping triangle x (scene; its frame Fw = tri_frame(x) is the same for every candidate, so the caller
// computes it once) onto triangle P (camera): R row-major, t.
template <typename T>
ESAC_HD bool align_triangles(const T P[3][3], const T x[3][3], const T Fw[9], T R[9], T t[3]) {
    T Fc[9];
    if (!tri_frame(P[0], P[1], P[2], Fc)) return false;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c)
            R[r * 3 + c] = Fc[r * 3 + 0] * Fw[c * 3 + 0] + Fc[r * 3 + 1] * Fw[c * 3 + 1] + Fc[r * 3 + 2] * Fw[c * 3 + 2];
    T mc[3], mw[3];
    for (int c = 0; c < 3; ++c) {
        mc[c] = (P[0][c] + P[1][c] + P[2][c]) * T(1.0 / 3.0);
        mw[c] = (x[0][c] + x[1][c] + x[2][c]) * T(1.0 / 3.0);
    }
    for (int r = 0; r < 3; ++r) t[r] = mc[r] - (R[r * 3] * mw[0] + R[r * 3 + 1] * mw[1] + R[r * 3 + 2] * mw[2]);
    return true;
}

// Depth triples (unpolished), in units where the largest squared side of the scene triangle is 1.
// cs = {c12, c13, c23} cosines between bearings, ss = {s12, s13, s23} normalised squared sides.
// `uncertain` is raised (float only) when a sign decision was taken too close to zero to be trusted.
template <typename T>
ESAC_HD int p3p_lambdas(const T y[3][3], const T x[3][3], T lam[4][3], T& amax, T cs[3], T ss[3], bool& uncertain) {
    using N = Num<T>;
    uncertain = false;
    T d12[3], d13[3], d23[3];
    for (int c = 0; c < 3; ++c) {
        d12[c] = x[0][c] - x[1][c];
        d13[c] = x[0][c] - x[2][c];
        d23[c] = x[1][c] - x[2][c];
    }
    T a12 = d12[0] * d12[0] + d12[1] * d12[1] + d12[2] * d12[2];
    T a13 = d13[0] * d13[0] + d13[1] * d13[1] + d13[2] * d13[2];
    T a23 = d23[0] * d23[0] + d23[1] * d23[1] + d23[2] * d23[2];
    amax = a12 > a13 ? (a12 > a23 ? a12 : a23) : (a13 > a23 ? a13 : a23);
    T amin = a12 < a13 ? (a12 < a23 ? a12 : a23) : (a13 < a23 ? a13 : a23);
    if (!(amax > 0) || !(amin > T(1e-24) * amax) || !(amax < T(1e30))) return 0;
    T c12 = y[0][0] * y[1][0] + y[0][1] * y[1][1] + y[0][2] * y[1][2];
    T c13 = y[0][0] * y[2][0] + y[0][1] * y[2][1] + y[0][2] * y[2][2];
    T c23 = y[1][0] * y[2][0] + y[1][1] * y[2][1] + y[1][2] * y[2][2];
    const T iamax = N::div_(T(1), amax);
    T s12 = a12 * iamax, s13 = a13 * iamax, s23 = a23 * iamax;
    if (N::kUncertain > 0) {  // float prefilter: needle triangles / nearly parallel bearings are left to the exact path
        const T cm = N::abs_(c12) > N::abs_(c13) ? (N::abs_(c12) > N::abs_(c23) ? N::abs_(c12) : N::abs_(c23))
                                                 : (N::abs_(c13) > N::abs_(c23) ? N::abs_(c13) : N::abs_(c23));
        if (amin < T(0.02) * amax || cm > T(0.9999)) uncertain = true;
    }
    cs[0] = c12; cs[1] = c13; cs[2] = c23;
    ss[0] = s12; ss[1] = s13; ss[2] = s23;
    T D1[9] = {s23, -s23 * c12, 0, -s23 * c12, s23 - s12, s12 * c23, 0, s12 * c23, -s12};
    T D2[9] = {s23, 0, -s23 * c13, 0, -s13, s13 * c23, -s23 * c13, s13 * c23, s23 - s13};
    T B1[9], B2[9];
    adj3(D1, B1);
    adj3(D2, B2);
    T k0 = det3(D1), k1 = trace_prod3(B1, D2), k2 = trace_prod3(D1, B2), k3 = det3(D2);
    Cubic<T> cub;
    const int nr = cubic_setup(k3, k2, k1, k0, cub);
    T kscale = N::abs_(k3) + N::abs_(k2) + N::abs_(k1) + N::abs_(k0);
    bool inf_root = N::abs_(k3) < N::kRelTiny * kscale;
    T dirs[8][3];
    int nd = 0;
#pragma unroll 1
    for (int ri = 0; ri < nr + (inf_root ? 1 : 0) && nd == 0; ++ri) {
        T D0[9];
        const T* Dother;
        if (ri >= nr) {  // D2 itself is the degenerate member
            for (int i = 0; i < 9; ++i) D0[i] = D2[i];
            Dother = D1;
        } else {
            T g = cubic_root(cub, ri);
            if (N::abs_(g) <= 1) {
                for (int i = 0; i < 9; ++i) D0[i] = D1[i] + g * D2[i];
                Dother = D2;
            } else {
                T ig = N::div_(T(1), g);
                for (int i = 0; i < 9; ++i) D0[i] = ig * D1[i] + D2[i];
                Dother = D1;
            }
        }
        T B[9];
        adj3(D0, B);  // = -p p^T with p = l x m for a real line pair
        int i = 0;
        if (N::abs_(B[4]) > N::abs_(B[i * 4])) i = 1;
        if (N::abs_(B[8]) > N::abs_(B[i * 4])) i = 2;
        T bii = B[i * 4];
        T nb = 0, nD = 0;
        for (int q = 0; q < 9; ++q) { nb += N::abs_(B[q]); nD += N::abs_(D0[q]); }
        if (N::abs_(bii) < N::kUncertain * nD * nD) uncertain = true;
        if (!(bii < 0)) {
            // rank <= 1 (double line) or complex line pair.  A double line shows up as B == 0.
            if (nb <= N::kRelTiny * nD * nD) {
                int rr = 0;
                for (int q = 1; q < 3; ++q) if (N::abs_(D0[q * 4]) > N::abs_(D0[rr * 4])) rr = q;
                T l[3] = {D0[rr * 3], D0[rr * 3 + 1], D0[rr * 3 + 2]};
                nd = line_conic(l, Dother, dirs, nd, uncertain);
            }
            continue;
        }
        T sq = N::sqrt_(-bii);
        const T isq = N::div_(T(1), sq);
        T p[3] = {B[i] * isq, B[3 + i] * isq, B[6 + i] * isq};
        T C[9] = {D0[0], D0[1] - p[2], D0[2] + p[1], D0[3] + p[2], D0[4], D0[5] - p[0],
                  D0[6] - p[1], D0[7] + p[0], D0[8]};
        int rm = 0, cm = 0;
        T best = -1;
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c)
                if (N::abs_(C[r * 3 + c]) > best) { best = N::abs_(C[r * 3 + c]); rm = r; cm = c; }
        if (!(best > 0)) continue;
        T l[3] = {C[rm * 3], C[rm * 3 + 1], C[rm * 3 + 2]};
        T m[3] = {C[cm], C[3 + cm], C[6 + cm]};
        nd = line_conic(l, Dother, dirs, nd, uncertain);
        nd = line_conic(m, Dother, dirs, nd, uncertain);
    }
    int ns = 0;
#pragma unroll 1
    for (int d = 0; d < nd && ns < 4; ++d) {
        T l0 = dirs[d][0], l1 = dirs[d][1], l2 = dirs[d][2];
        T q12 = l0 * l0 + l1 * l1 - 2 * c12 * l0 * l1;
        T q13 = l0 * l0 + l2 * l2 - 2 * c13 * l0 * l2;
        T q23 = l1 * l1 + l2 * l2 - 2 * c23 * l1 * l2;
        T sc;  // fix the scale with the largest quadratic form
        if (q12 >= q13 && q12 >= q23) sc = N::div_(s12, q12);
        else if (q13 >= q23) sc = N::div_(s13, q13);
        else sc = N::div_(s23, q23);
        if (!(sc > 0) || !(sc < T(1e30))) continue;
        sc = N::sqrt_(sc);
        T mx = N::abs_(l0) > N::abs_(l1) ? N::abs_(l0) : N::abs_(l1);
        mx = mx > N::abs_(l2) ? mx : N::abs_(l2);
        if (N::abs_(l0) < N::kUncertain * mx || N::abs_(l1) < N::kUncertain * mx || N::abs_(l2) < N::kUncertain * mx) uncertain = true;
        int pos = (l0 > 0) + (l1 > 0) + (l2 > 0);
        int neg = (l0 < 0) + (l1 < 0) + (l2 < 0);
        if (neg == 3) sc = -sc;
        else if (pos != 3) continue;
        lam[ns][0] = l0 * sc; lam[ns][1] = l1 * sc; lam[ns][2] = l2 * sc;
        if (N::kUncertain > 0) {  // float prefilter: an inaccurate candidate (distance equations not met) is not trusted
            const T a0 = lam[ns][0], a1 = lam[ns][1], a2 = lam[ns][2];
            T r = N::abs_(a0 * a0 + a1 * a1 - 2 * c12 * a0 * a1 - s12) + N::abs_(a0 * a0 + a2 * a2 - 2 * c13 * a0 * a2 - s13) +
                  N::abs_(a1 * a1 + a2 * a2 - 2 * c23 * a1 * a2 - s23);
            if (!(r < T(1e-4) * (a0 * a0 + a1 * a1 + a2 * a2 + 1))) uncertain = true;
        }
        ++ns;
    }
    return ns;
}

// A 4th correspondence for the early exit of p3p_solve: scene point, pixel, camera, squared pixel distance beyond which a
// candidate is hopeless.
struct FourthPoint {
    double X[3], u, v, f, ppx, ppy, reject2;
};

// All P3P solutions (R row-major, t), polished to machine precision.  Returns the count (0..4).
// With `fourth` (the sampling stage's verdicts): when EVERY candidate depth triple, still unpolished, puts the 4th point
// further than sqrt(reject2) pixels from where it was seen, no solution can pass the 4-point gate and the polish / alignment
// of up to four candidates (most of this function) is skipped: returns -1.  The 4th point is carried over in the frame of
// the scene triangle (x4 - x0 = al u1 + be u2 + ga u1 x u2, coefficients preserved by a rigid motion), so no rotation is
// needed; a candidate whose distance equations are not met to 1e-6 is not trusted and disables the exit.
ESAC_HDN int p3p_solve(const double y[3][3], const double x[3][3], double Rs[4][9], double ts[4][3], const FourthPoint* fourth = nullptr) {
    double lams[4][3], amax, cs[3], ss[3];
    bool unc;
    int nl = p3p_lambdas<double>(y, x, lams, amax, cs, ss, unc);
    const double c12 = cs[0], c13 = cs[1], c23 = cs[2], s12 = ss[0], s13 = ss[1], s23 = ss[2];
    int only = -1;  // >= 0: the one candidate worth polishing (verdict path)
    if (fourth && nl > 0) {
        double u1[3], u2[3], d4[3], nw[3];
        for (int c = 0; c < 3; ++c) { u1[c] = x[1][c] - x[0][c]; u2[c] = x[2][c] - x[0][c]; d4[c] = fourth->X[c] - x[0][c]; }
        cross3(u1, u2, nw);
        const double g11 = u1[0] * u1[0] + u1[1] * u1[1] + u1[2] * u1[2], g22 = u2[0] * u2[0] + u2[1] * u2[1] + u2[2] * u2[2];
        const double g12 = u1[0] * u2[0] + u1[1] * u2[1] + u1[2] * u2[2];
        const double nn = nw[0] * nw[0] + nw[1] * nw[1] + nw[2] * nw[2], det = g11 * g22 - g12 * g12;
        if (det > 1e-12 * g11 * g22 && nn > 0) {
            const double v1 = d4[0] * u1[0] + d4[1] * u1[1] + d4[2] * u1[2], v2 = d4[0] * u2[0] + d4[1] * u2[1] + d4[2] * u2[2];
            const double idet = 1. / det;
            const double al = (v1 * g22 - v2 * g12) * idet, be = (v2 * g11 - v1 * g12) * idet;
            const double ga = (d4[0] * nw[0] + d4[1] * nw[1] + d4[2] * nw[2]) / nn;
            const double sa = sqrt(amax);
            bool hopeless = true, trusted = true;
            double e_best = 1e300, e_second = 1e300;
            int d_best = -1;
            for (int d = 0; d < nl; ++d) {
                const double l0 = lams[d][0], l1 = lams[d][1], l2 = lams[d][2];
                const double res = fabs(l0 * l0 + l1 * l1 - 2 * c12 * l0 * l1 - s12) + fabs(l0 * l0 + l2 * l2 - 2 * c13 * l0 * l2 - s13) +
                                   fabs(l1 * l1 + l2 * l2 - 2 * c23 * l1 * l2 - s23);
                if (!(res < 1e-6)) { trusted = false; break; }
                double P0[3], a1[3], a2[3], m[3];
                for (int c = 0; c < 3; ++c) { P0[c] = l0 * sa * y[0][c]; a1[c] = l1 * sa * y[1][c] - P0[c]; a2[c] = l2 * sa * y[2][c] - P0[c]; }
                cross3(a1, a2, m);
                const double xc = P0[0] + al * a1[0] + be * a2[0] + ga * m[0];
                const double yc = P0[1] + al * a1[1] + be * a2[1] + ga * m[1];
                const double zc = P0[2] + al * a1[2] + be * a2[2] + ga * m[2];
                const double iz = 1. / zc;
                const double du = fourth->ppx + fourth->f * xc * iz - fourth->u, dv = fourth->ppy + fourth->f * yc * iz - fourth->v;
                const double e = du * du + dv * dv;
                if (!(e == e)) { trusted = false; break; }     // NaN: the full path decides
                if (!(e > fourth->reject2)) hopeless = false;  // close enough
                if (e < e_best) { e_second = e_best; e_best = e; d_best = d; }
                else if (e < e_second) e_second = e;
            }
            if (trusted && hopeless) return -1;
            // One candidate far ahead of the others (twice as close to the seen pixel, and by more than a pixel): it is the one
            // solvePnP's "smallest 4th-point error" rule will pick, so only it is polished and aligned.  Ties, untrusted
            // candidates, or a favourite that then fails its own validity checks fall back to the full loop below.
            if (trusted && d_best >= 0 && e_second > 4. * e_best + 1.) only = d_best;
        }
    }
    double Fw[9];
    if (nl > 0 && !tri_frame<double>(x[0], x[1], x[2], Fw)) return 0;
    int ns = 0;
    const double sa = sqrt(amax);
    // candidate d -> polished depths -> pose in slot ns; false when it is not a valid new solution
    auto add = [&](int d) -> bool {
        double lam[3] = {lams[d][0], lams[d][1], lams[d][2]};
        // Gauss-Newton polish on the three (normalised) distance equations
        double res = 0;
        for (int it = 0; it < 6; ++it) {
            double r[3] = {lam[0] * lam[0] + lam[1] * lam[1] - 2 * c12 * lam[0] * lam[1] - s12,
                           lam[0] * lam[0] + lam[2] * lam[2] - 2 * c13 * lam[0] * lam[2] - s13,
                           lam[1] * lam[1] + lam[2] * lam[2] - 2 * c23 * lam[1] * lam[2] - s23};
            res = fabs(r[0]) + fabs(r[1]) + fabs(r[2]);
            if (it == 5 || res < 1e-15) break;  // quadratic convergence: usually two iterations
            double Jm[9] = {2 * lam[0] - 2 * c12 * lam[1], 2 * lam[1] - 2 * c12 * lam[0], 0,
                            2 * lam[0] - 2 * c13 * lam[2], 0, 2 * lam[2] - 2 * c13 * lam[0],
                            0, 2 * lam[1] - 2 * c23 * lam[2], 2 * lam[2] - 2 * c23 * lam[1]};
            double dl[3];
            if (!solve3(Jm, r, dl)) break;  // singular: keep the current estimate
            lam[0] -= dl[0]; lam[1] -= dl[1]; lam[2] -= dl[2];
        }
        if (!(res < 1e-9) || !(lam[0] > 0 && lam[1] > 0 && lam[2] > 0)) return false;
        double P[3][3];
        for (int i = 0; i < 3; ++i)
            for (int c = 0; c < 3; ++c) P[i][c] = lam[i] * sa * y[i][c];
        if (!align_triangles<double>(P, x, Fw, Rs[ns], ts[ns])) return false;
        for (int q = 0; q < ns; ++q) {  // reject duplicates (double roots)
            double dd = 0;
            for (int c = 0; c < 3; ++c) dd += fabs(ts[q][c] - ts[ns][c]);
            for (int c = 0; c < 9; ++c) dd += fabs(Rs[q][c] - Rs[ns][c]);
            if (dd < 1e-9) return false;
        }
        ++ns;
        return true;
    };
    if (only >= 0 && add(only)) return 1;  // (a favourite that fails its own checks: every candidate, as usual)
    ns = 0;
    for (int d = 0; d < nl && ns < 4; ++d) add(d);
    return ns;
}

// Bearing of an image point the way cv::solvePnP hands it to P3P: undistortPoints on float points gives
// (u - cx) * (1/fx) rounded to float (a ~1e-5 px perturbation that shows up in the 4.13 oracle's poses).
ESAC_HD void bearing(float u, float v, double f, double ppx, double ppy, double y[3]) {
    const double ifx = 1. / f;
    double bx = (double)(float)(((double)u - ppx) * ifx), by = (double)(float)(((double)v - ppy) * ifx);
    double n = 1. / sqrt(bx * bx + by * by + 1.);
    y[0] = bx * n; y[1] = by * n; y[2] = n;
}

// solvePnP(4 points, SOLVEPNP_P3P) semantics: solve with the first three correspondences, pick the
// solution with the smallest squared reprojection error of the 4th (Appendix A of SURVEY.md: the
// 4th point only disambiguates).  img = integer pixel positions as float, obj = float scene points.
// Returns false when no solution exists (the reference retries, esac_util.h:189-200).
// reject_px > 0 (sampling verdicts only): give up -- return false -- as soon as no candidate brings the 4th point within
// reject_px pixels (p3p_solve's early exit); the caller must then not use `pose`.
ESAC_HD bool p3p_pose(const float obj[4][3], const float img[4][2], double f, double ppx, double ppy, Pose& pose, double reject_px = 0.) {
    double y[3][3], x[3][3];
    for (int i = 0; i < 3; ++i) {
        bearing(img[i][0], img[i][1], f, ppx, ppy, y[i]);
        for (int c = 0; c < 3; ++c) x[i][c] = (double)obj[i][c];
    }
    double Rs[4][9], ts[4][3];
    FourthPoint fp;
    if (reject_px > 0.) {
        fp.X[0] = obj[3][0]; fp.X[1] = obj[3][1]; fp.X[2] = obj[3][2];
        fp.u = img[3][0]; fp.v = img[3][1]; fp.f = f; fp.ppx = ppx; fp.ppy = ppy; fp.reject2 = reject_px * reject_px;
    }
    int n = p3p_solve(y, x, Rs, ts, reject_px > 0. ? &fp : nullptr);
    if (n <= 0) return false;
    int best = 0;
    double beste = 0;
    for (int s = 0; s < n; ++s) {
        double X = obj[3][0], Y = obj[3][1], Z = obj[3][2];
        double xc = Rs[s][0] * X + Rs[s][1] * Y + Rs[s][2] * Z + ts[s][0];
        double yc = Rs[s][3] * X + Rs[s][4] * Y + Rs[s][5] * Z + ts[s][1];
        double zc = Rs[s][6] * X + Rs[s][7] * Y + Rs[s][8] * Z + ts[s][2];
        const double izc = 1. / zc;
        double u = ppx + f * xc * izc, v = ppy + f * yc * izc;
        double e = (u - img[3][0]) * (u - img[3][0]) + (v - img[3][1]) * (v - img[3][1]);
        if (!(e == e)) e = 1e300;  // NaN sorts last
        if (s == 0 || e < beste) { beste = e; best = s; }
    }
    rodrigues_m2v(Rs[best], pose.r);
    pose.t[0] = ts[best][0]; pose.t[1] = ts[best][1]; pose.t[2] = ts[best][2];
    return true;
}

// The reference's 4-point gate (esac_util.h:202-223): every minimal-set point must reproject within
// the inlier threshold, measured on float-rounded projections.
ESAC_HD bool minimal_set_gate(const float obj[4][3], const float img[4][2], const Pose& pose, double f,
                              double ppx, double ppy, float tau) {
    double R[9];
    rodrigues_v2m(pose.r, R, nullptr);
    for (int j = 0; j < 4; ++j) {
        float u, v;
        project_point_f(R, pose.t, f, ppx, ppy, obj[j][0], obj[j][1], obj[j][2], u, v);
        float dx = img[j][0] - u, dy = img[j][1] - v;
        double n = sqrt((double)dx * (double)dx + (double)dy * (double)dy);
        if (!(n < (double)tau)) return false;
    }
    return true;
}

// ---------------------------------------------------------------------------------------------
// loss / dLoss / pose <-> transform
// ---------------------------------------------------------------------------------------------
// camera->world 4x4 (row-major) of a scene pose: [R^T | -R^T t] (pose2trans, esac_util.h:537-548).
ESAC_HD void pose2trans(const Pose& p, double T[16]) {
    double R[9];
    rodrigues_v2m(p.r, R, nullptr);
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) T[r * 4 + c] = R[c * 3 + r];
        T[r * 4 + 3] = -(R[0 * 3 + r] * p.t[0] + R[1 * 3 + r] * p.t[1] + R[2 * 3 + r] * p.t[2]);
    }
    T[12] = T[13] = T[14] = 0;
    T[15] = 1;
}

// trans2pose (esac_util.h:555-568) for a rigid camera->world transform.
ESAC_HD void trans2pose(const double T[16], Pose& p) {
    double R[9];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) R[r * 3 + c] = T[c * 4 + r];
    rodrigues_m2v(R, p.r);
    for (int r = 0; r < 3; ++r) p.t[r] = -(R[r * 3] * T[3] + R[r * 3 + 1] * T[7] + R[r * 3 + 2] * T[11]);
}

// loss() of esac_loss.h:66-83 on two camera->world transforms.
ESAC_HD double pose_loss(const double T1[16], const double T2[16], double wRot, double wTrans, double cut) {
    double tr = 0;  // trace(R2 * R1^T)
    for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 3; ++k) tr += T2[i * 4 + k] * T1[i * 4 + k];
    tr = fmin(3.0, fmax(-1.0, tr));
    double rotErr = 180 * acos((tr - 1.0) / 2.0) / kPiRef;
    double dx = T1[3] - T2[3], dy = T1[7] - T2[7], dz = T1[11] - T2[11];
    double tErr = sqrt(dx * dx + dy * dy + dz * dz);
    double l = wRot * rotErr + wTrans * tErr;
    if (l > cut) l = sqrt(cut * l);
    return fmin(l, kMaxLoss);
}

// dLoss() of esac_loss.h:94-210, quirks kept: the cut branch scales by 0.5/sqrt(loss) (not
// sqrt(cut*loss)) and the angle uses CV_PI.  out: 1x6 (d/d rvec, d/d tvec).
ESAC_HDN void pose_dloss(const Pose& est, const Pose& gt, double wRot, double wTrans, double cut, double out[6]) {
    double R1[9], R2[9], dRod[27];
    rodrigues_v2m(est.r, R1, dRod);
    rodrigues_v2m(gt.r, R2, nullptr);
    for (int i = 0; i < 6; ++i) out[i] = 0;
    // trace(R1 * R2^T)
    double tr = 0;
    for (int i = 0; i < 9; ++i) tr += R1[i] * R2[i];
    tr = fmin(3.0, fmax(-1.0, tr));
    double rotErr = 180 * acos((tr - 1.0) / 2.0) / kPi;
    double it1[3], it2[3];
    for (int r = 0; r < 3; ++r) {
        it1[r] = R1[r] * est.t[0] + R1[3 + r] * est.t[1] + R1[6 + r] * est.t[2];
        it2[r] = R2[r] * gt.t[0] + R2[3 + r] * gt.t[1] + R2[6 + r] * gt.t[2];
    }
    double dd[3] = {it1[0] - it2[0], it1[1] - it2[1], it1[2] - it2[2]};
    double tErr = sqrt(dd[0] * dd[0] + dd[1] * dd[1] + dd[2] * dd[2]);
    double l = wRot * rotErr + wTrans * tErr;
    bool cutLoss = false;
    if (l > cut) { l = sqrt(l); cutLoss = true; }
    if (l > kMaxLoss) return;
    if ((tErr + rotErr) < kEps) return;
    double g[3] = {dd[0] / tErr, dd[1] / tErr, dd[2] / tErr};  // dDist_dInvT1
    // translation part: g * R1^T  -> columns 3..5
    for (int c = 0; c < 3; ++c) out[3 + c] += (g[0] * R1[c * 3 + 0] + g[1] * R1[c * 3 + 1] + g[2] * R1[c * 3 + 2]) * wTrans;
    // g * dInvT1_dInvRot1 (3x9): entry (r, r + 3c) = est.t[c]
    double gv[9];
    for (int k = 0; k < 9; ++k) gv[k] = 0;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) gv[r + 3 * c] += g[r] * est.t[c];
    // dRod^T is 9x3: (dRod^T)[k][i] = dRod[i*9 + k]
    for (int i = 0; i < 3; ++i) {
        double s = 0;
        for (int k = 0; k < 9; ++k) s += gv[k] * dRod[i * 9 + k];
        out[i] += s * wTrans;
    }
    // rotation part: dTrace(1x9) * dRotDiff^T(9x9, block-diag of R2^T, transposed) * dRod^T
    // dRotDiff (before .t()) has R2^T on the 3 diagonal blocks; after transpose the blocks are R2.
    // row vector w = dTrace * dRotDiff^T: w[3b + c] = sum_r dTrace[3b + r] * R2^T^T[r][c]... expand:
    double w[9];
    {
        // M = blockdiag(inv2, inv2, inv2) with inv2 = R2^T ; dRotDiff = M^T = blockdiag(R2, R2, R2)
        // w = dTrace * dRotDiff ; dTrace has ones at 0, 4, 8
        const int ones[3] = {0, 4, 8};
        for (int k = 0; k < 9; ++k) w[k] = 0;
        for (int q = 0; q < 3; ++q) {
            int row = ones[q];
            int b = row / 3, rr = row % 3;
            for (int c = 0; c < 3; ++c) w[3 * b + c] += R2[rr * 3 + c];
        }
    }
    double denom = 3 - tr * tr + 2 * tr;
    // At a clamped trace (3 or -1) denom is 0 and the reference's coefficient -1/sqrt(0) is -inf.  Its matrix expression
    // coef * dTrace * dRotDiff * dRod carries that -inf into the 1x9 row before the product with dRod, where infinities
    // of both signs (or an inf times a zero) make NaN; the NaN check then returns zeros.  coef * s, with the finished
    // product s, would give +-inf instead (DESIGN.md section 2).
    if (!(denom > 0)) {
        for (int i = 0; i < 6; ++i) out[i] = 0;
        return;
    }
    double coef = (180 / kPi * -1 / sqrt(denom));
    for (int i = 0; i < 3; ++i) {
        double s = 0;
        for (int k = 0; k < 9; ++k) s += w[k] * dRod[i * 9 + k];
        out[i] += coef * s * wRot;
    }
    if (cutLoss)
        for (int i = 0; i < 6; ++i) out[i] *= 0.5 / l;
    bool nan = false;
    for (int i = 0; i < 6; ++i) nan = nan || !(out[i] == out[i]);
    if (nan)
        for (int i = 0; i < 6; ++i) out[i] = 0;
}

}  // namespace esacb200
