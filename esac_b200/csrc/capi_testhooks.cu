// The host test hooks of include/esac_b200_testhooks.h: single geometry primitives of the kernels, run on the CPU.
#include "../../include/esac_b200_testhooks.h"
#include "esac_internal.h"
#include "esac_p3p_fast.cuh"
#include "esac_rng.cuh"

#include <vector>

using namespace esacb200;

extern "C" {

// ------------------------------------------------------------------------------------------------
// host test hooks (esac_b200_testhooks.h)
// ------------------------------------------------------------------------------------------------
void esacb200_host_rodrigues(const double r[3], double R[9], double J[27]) { rodrigues_v2m(r, R, J); }
void esacb200_host_rodrigues_inv(const double R[9], double r[3]) { rodrigues_m2v(R, r); }

int esacb200_host_p3p_all(const double* y9, const double* x9, double* Rs36, double* ts12) {
    double y[3][3], x[3][3], Rs[4][9], ts[4][3];
    for (int i = 0; i < 3; ++i)
        for (int c = 0; c < 3; ++c) { y[i][c] = y9[i * 3 + c]; x[i][c] = x9[i * 3 + c]; }
    int n = p3p_solve(y, x, Rs, ts);
    for (int s = 0; s < n; ++s) {
        for (int c = 0; c < 9; ++c) Rs36[s * 9 + c] = Rs[s][c];
        for (int c = 0; c < 3; ++c) ts12[s * 3 + c] = ts[s][c];
    }
    return n;
}

int esacb200_host_p3p_pose(const float* obj12, const float* img8, float f, float ppx, float ppy, float tau, double* pose6,
                           int* gate) {
    float obj[4][3], img[4][2];
    for (int i = 0; i < 4; ++i) {
        for (int c = 0; c < 3; ++c) obj[i][c] = obj12[i * 3 + c];
        for (int c = 0; c < 2; ++c) img[i][c] = img8[i * 2 + c];
    }
    Pose p;
    bool ok = p3p_pose(obj, img, (double)f, (double)ppx, (double)ppy, p);
    if (gate) *gate = 0;
    if (!ok) { for (int i = 0; i < 6; ++i) pose6[i] = 0; return 0; }
    for (int i = 0; i < 3; ++i) { pose6[i] = p.r[i]; pose6[3 + i] = p.t[i]; }
    if (gate) *gate = minimal_set_gate(obj, img, p, (double)f, (double)ppx, (double)ppy, tau) ? 1 : 0;
    return 1;
}

void esacb200_host_try(const float* obj12, const float* img8, float f, float ppx, float ppy, float tau, float margin,
                       int* may_pass, int* accept) {
    float obj[4][3], img[4][2];
    for (int i = 0; i < 4; ++i) {
        for (int c = 0; c < 3; ++c) obj[i][c] = obj12[i * 3 + c];
        for (int c = 0; c < 2; ++c) img[i][c] = img8[i * 2 + c];
    }
    *may_pass = p3p_may_pass_fast(obj, img, f, ppx, ppy, tau, margin) ? 1 : 0;
    Pose p;
    bool ok = p3p_pose(obj, img, (double)f, (double)ppx, (double)ppy, p);
    *accept = (ok && minimal_set_gate(obj, img, p, (double)f, (double)ppx, (double)ppy, tau)) ? 1 : 0;
}

void esacb200_host_tries_hint(int n, const float* obj12n, const float* img8n, float f, float ppx, float ppy, float tau,
                              float hint_frac, int* may_pass, int* hint, int* accept) {
    for (int k = 0; k < n; ++k) {
        float obj[4][3], img[4][2];
        for (int i = 0; i < 4; ++i) {
            for (int c = 0; c < 3; ++c) obj[i][c] = obj12n[k * 12 + i * 3 + c];
            for (int c = 0; c < 2; ++c) img[i][c] = img8n[k * 8 + i * 2 + c];
        }
        bool h;
        may_pass[k] = p3p_may_pass_hint(obj, img, f, ppx, ppy, tau, hint_frac, h) ? 1 : 0;
        hint[k] = h ? 1 : 0;
        Pose p;
        const bool ok = p3p_pose(obj, img, (double)f, (double)ppx, (double)ppy, p);
        accept[k] = (ok && minimal_set_gate(obj, img, p, (double)f, (double)ppx, (double)ppy, tau)) ? 1 : 0;
    }
}

void esacb200_host_try_verdict(const float* obj12, const float* img8, float f, float ppx, float ppy, float tau, int* accept,
                               double* pose6) {
    float obj[4][3], img[4][2];
    for (int i = 0; i < 4; ++i) {
        for (int c = 0; c < 3; ++c) obj[i][c] = obj12[i * 3 + c];
        for (int c = 0; c < 2; ++c) img[i][c] = img8[i * 2 + c];
    }
    Pose p;
    const bool ok = p3p_pose(obj, img, (double)f, (double)ppx, (double)ppy, p, 1.25 * (double)tau + 1.);  // as hyp.cu exact_try(verdict_only)
    *accept = (ok && minimal_set_gate(obj, img, p, (double)f, (double)ppx, (double)ppy, tau)) ? 1 : 0;
    if (pose6 && ok)
        for (int i = 0; i < 3; ++i) { pose6[i] = p.r[i]; pose6[3 + i] = p.t[i]; }
}

void esacb200_host_project(const double pose6[6], float f, float ppx, float ppy, const float X[3], float uv_f[2],
                           double uv[2], double J12[12]) {
    double R[9], dRdr[27];
    rodrigues_v2m(pose6, R, dRdr);
    project_point_f(R, pose6 + 3, (double)f, (double)ppx, (double)ppy, X[0], X[1], X[2], uv_f[0], uv_f[1]);
    double Ju[6], Jv[6];
    project_point_jac(R, pose6 + 3, dRdr, (double)f, (double)ppx, (double)ppy, (double)X[0], (double)X[1], (double)X[2], uv[0],
                      uv[1], Ju, Jv);
    for (int i = 0; i < 6; ++i) { J12[i] = Ju[i]; J12[6 + i] = Jv[i]; }
}

double esacb200_host_loss(const double* T1, const double* T2, double wRot, double wTrans, double cut) {
    return pose_loss(T1, T2, wRot, wTrans, cut);
}

void esacb200_host_dloss(const double est6[6], const double gt6[6], double wRot, double wTrans, double cut, double out6[6]) {
    Pose a, b;
    for (int i = 0; i < 3; ++i) { a.r[i] = est6[i]; a.t[i] = est6[3 + i]; b.r[i] = gt6[i]; b.t[i] = gt6[3 + i]; }
    pose_dloss(a, b, wRot, wTrans, cut, out6);
}

void esacb200_host_pose2trans(const double pose6[6], double T16[16]) {
    Pose a;
    for (int i = 0; i < 3; ++i) { a.r[i] = pose6[i]; a.t[i] = pose6[3 + i]; }
    pose2trans(a, T16);
}

void esacb200_host_trans2pose(const double T16[16], double pose6[6]) {
    Pose a;
    trans2pose(T16, a);
    for (int i = 0; i < 3; ++i) { pose6[i] = a.r[i]; pose6[3 + i] = a.t[i]; }
}

void esacb200_host_dprojectdobj(const float pt[2], const float obj[3], const double pose6[6], float f, float ppx, float ppy,
                                float maxReproj, double out3[3]) {
    double R[9];
    rodrigues_v2m(pose6, R, nullptr);
    d_project_d_obj(pt[0], pt[1], obj[0], obj[1], obj[2], R, pose6 + 3, (double)f, (double)ppx, (double)ppy, (double)maxReproj, out3);
}

void esacb200_host_pinv6(const double A[36], double out[36]) { pinv_sym6(A, out); }
int esacb200_host_pick_group(int N, int coresident, int group_opt, int jobs_per_group, int jobs) {
    return refine_group_rule(N, coresident, group_opt, jobs_per_group, jobs);
}

void esacb200_host_draw_cells(uint64_t seed, uint32_t h, uint32_t t, int W, int H, int32_t* cells8) {
    int cx[4], cy[4];
    draw_minimal_set(seed, h, t, W, H, cx, cy);
    for (int j = 0; j < 4; ++j) { cells8[2 * j] = cx[j]; cells8[2 * j + 1] = cy[j]; }
}

int esacb200_graph_node_types(void* graph, int* types, int cap) {
    typedef int (*GetType)(cudaGraphNode_t, int*);
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuGraphNodeGetType", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
        cudaGetLastError();
        return -1;
    }
    size_t n = 0;
    if (cudaGraphGetNodes((cudaGraph_t)graph, nullptr, &n) != cudaSuccess) { cudaGetLastError(); return -1; }
    std::vector<cudaGraphNode_t> nodes(n);
    if (n && cudaGraphGetNodes((cudaGraph_t)graph, nodes.data(), &n) != cudaSuccess) { cudaGetLastError(); return -1; }
    for (size_t i = 0; i < n && (int)i < cap; ++i) {
        int t = -1;
        if (((GetType)f)(nodes[i], &t) != 0) return -1;
        types[i] = t;
    }
    return (int)n;
}

}  // extern "C"
