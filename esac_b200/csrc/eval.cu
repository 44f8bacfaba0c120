// Test-time evaluation of estimated poses on the device (test_esac.py:209-247): rotation and translation error, whether the
// winning expert is the ground-truth scene, the experts that drew hypotheses, and the pose-file entry, one record per image
// in a caller-owned store whose slot counter lives in device memory, so that a captured test step evaluates its image
// without a host round trip.  One thread per image: the work is a few hundred fp64 operations.
#include "esac_internal.h"

namespace esacb200 {

constexpr int kEvalThreads = 128;

// s and c of rodrigues_m2v (OpenCV's Rodrigues): the sine from the skew part, the cosine from the trace, clamped.  Written
// out here because calling a shared helper from rodrigues_m2v changes the code of the sampling and backward kernels.
__device__ __forceinline__ void rodrigues_sin_cos(const double R[9], double& s, double& c) {
    const double rx = R[7] - R[5], ry = R[2] - R[6], rz = R[3] - R[1];
    s = sqrt((rx * rx + ry * ry + rz * rz) * 0.25);
    c = (R[0] + R[4] + R[8] - 1) * 0.5;
    c = c > 1. ? 1. : (c < -1. ? -1. : c);
}

__device__ void eval_image(const EvalArgs& a, int b, EvalRecord& o) {
    double P[16], G[16];
    for (int i = 0; i < 16; ++i) {
        P[i] = (double)a.out_poses[(size_t)b * 16 + i];
        G[i] = (double)a.gt_poses[(size_t)b * 16 + i];
    }
    // translation error: |G[:3,3] - P[:3,3]| in centimetres
    double d2 = 0.;
    for (int r = 0; r < 3; ++r) {
        const double d = G[r * 4 + 3] - P[r * 4 + 3];
        d2 += d * d;
    }
    o.trans_cm = sqrt(d2) * 100.;
    // rotation error: |Rodrigues(P_R G_R^T)| of the nearest rotation, with OpenCV's exact zero for s < 1e-5, c > 0
    double X[9];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) X[r * 3 + c] = P[r * 4] * G[c * 4] + P[r * 4 + 1] * G[c * 4 + 1] + P[r * 4 + 2] * G[c * 4 + 2];
    polar_newton(X);
    double s, c;
    rodrigues_sin_cos(X, s, c);
    o.rot_deg = (s < 1e-5 && c > 0) ? 0. : acos(c) * 180. / kPi;
    // pose file: the general inverse of the estimate, its rotation as a quaternion through the axis-angle vector
    double Ri[9], r[3];
    affine_inverse(P, Ri, o.t);
    polar_newton(Ri);
    rodrigues_m2v(Ri, r);
    const double angle = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
    const double sh = sin(angle * 0.5);
    o.q[0] = cos(angle * 0.5);
    for (int i = 0; i < 3; ++i) o.q[1 + i] = sh * (r[i] / angle);  // NaN at angle 0, as the reference's axis = rot / angle
    const long long e = a.experts[b], g = a.scenes[b];
    o.correct = e == g ? 1. : 0.;
    o.scene = (double)g;
    o.expert = (double)e;
    o.status = a.status ? (double)a.status[b] : 0.;
    if (a.hist) {
        int n = 0;
        for (int k = 0; k < a.E; ++k) n += a.hist[(size_t)b * a.E + k] > 0.f;
        o.active = (double)n;
    } else {
        o.active = __longlong_as_double(0x7ff8000000000000ll);
    }
}

__global__ void __launch_bounds__(kEvalThreads) eval_poses_kernel(const __grid_constant__ EvalArgs a) {
    __shared__ unsigned long long base;
    if (threadIdx.x == 0) {
        base = *(volatile unsigned long long*)&a.state->count;
        // Every CTA reads the counter before it takes a ticket, so the last CTA to take one advances it after all have read.
        __threadfence();
        if (atomicAdd(&a.state->ticket, 1ull) == gridDim.x - 1) {
            a.state->count = base + (unsigned long long)a.B;
            a.state->ticket = 0;
        }
    }
    __syncthreads();
    const int b = blockIdx.x * kEvalThreads + threadIdx.x;
    if (b >= a.B) return;
    const unsigned long long slot = base + (unsigned long long)b;
    if (slot >= (unsigned long long)a.capacity) {
        a.state->overflow = 1;
        return;
    }
    EvalRecord o;
    eval_image(a, b, o);
    a.records[slot] = o;
}

void launch_eval_poses(const EvalArgs& a, cudaStream_t st) {
    eval_poses_kernel<<<(a.B + kEvalThreads - 1) / kEvalThreads, kEvalThreads, 0, st>>>(a);
}

}  // namespace esacb200
