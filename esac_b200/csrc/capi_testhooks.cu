// The test hooks of include/esac_b200_testhooks.h: single geometry primitives of the kernels, run on the CPU, one
// layer of the expert stack's convolution on the device, and the two kernels that merge the shards of a sharded call.
#include "../../include/esac_b200_testhooks.h"
#include "capi_internal.h"
#include "esac_p3p_fast.cuh"
#include "esac_rng.cuh"

#include <vector>

using namespace esacb200;
using namespace esacb200::capi;

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

int esacb200_test_experts_conv(esacb200_ctx* ctx, int B, int E, const float* hist, const float* packed, int64_t w_off,
                               int64_t b_off, int k, int stride, int cin, int cout, int hin, int win, int relu, float* pairs,
                               int64_t pair_floats, int64_t in_off, int64_t out_off, int64_t res_off, int* hdr) {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "test_experts_conv";
    if (B < 1 || E < 1 || E > ESACB200_EXPERTS_MAX || (long long)B * E > ESACB200_EXPERTS_MAX_PAIRS)
        return fail(ctx, ESACB200_ERR_ARG, "%s: B=%d E=%d: need E <= %d and B * E <= %d", what, B, E, ESACB200_EXPERTS_MAX,
                    ESACB200_EXPERTS_MAX_PAIRS);
    if ((k != 1 && k != 3) || (stride != 1 && stride != 2) || (k == 1 && stride == 2))
        return fail(ctx, ESACB200_ERR_ARG, "%s: k=%d stride=%d: need k 1 or 3, stride 1 or 2, and stride 1 for k 1", what, k,
                    stride);
    if (cin < 32 || cin % 32 || cout < 2 || cout % 2 || hin < 1 || win < 1 || hin > ESACB200_EXPERTS_MAX_SIDE ||
        win > ESACB200_EXPERTS_MAX_SIDE)
        return fail(ctx, ESACB200_ERR_ARG, "%s: cin=%d cout=%d at %dx%d: need cin a multiple of 32, cout even, sides in [1, %d]",
                    what, cin, cout, hin, win, ESACB200_EXPERTS_MAX_SIDE);
    const int hout = (hin + stride - 1) / stride, wout = (win + stride - 1) / stride;
    const long long in_n = (long long)hin * win * cin, out_n = (long long)hout * wout * cout;
    if (w_off < 0 || b_off < 0 || in_off < 0 || out_off < 0 || res_off < -1 || pair_floats < 1 || w_off % 4 || b_off % 4 ||
        in_off % 4 || out_off % 4 || (res_off >= 0 && res_off % 4) || pair_floats % 4)
        return fail(ctx, ESACB200_ERR_ARG, "%s: offsets and pair_floats must be non-negative multiples of 4 (res_off may be -1)",
                    what);
    if (in_off + in_n > pair_floats || out_off + out_n > pair_floats || (res_off >= 0 && res_off + out_n > pair_floats))
        return fail(ctx, ESACB200_ERR_ARG, "%s: a region runs past the pair's block of %lld floats", what, (long long)pair_floats);
    const void* ptrs[] = {packed, pairs, hdr, hist};
    const char* names[] = {"packed", "pairs", "hdr", "hist"};
    const int rc = device_args(ctx, what, 4, ptrs, names, 1u << 3);
    if (rc) return rc;
    if ((uintptr_t)packed % 16 || (uintptr_t)pairs % 16 || (uintptr_t)hdr % 4 || (uintptr_t)hist % 4)
        return fail(ctx, ESACB200_ERR_ARG, "%s: packed and pairs must be 16-byte, hdr and hist 4-byte aligned", what);
    ExpertsArgs a{};
    a.B = B;
    a.E = E;
    a.H = hin;
    a.W = win;
    a.hist = hist;
    a.packed = packed;
    a.ws_hdr = hdr;
    a.ws_pairs = pairs;
    a.pair_floats = pair_floats;
    ExpertsConvLayer L{};
    L.cin = cin;
    L.cout = cout;
    L.hin = hin;
    L.win = win;
    L.hout = hout;
    L.wout = wout;
    L.in_off = in_off;
    L.out_off = out_off;
    L.res_off = res_off;
    L.w_off = w_off;
    L.b_off = b_off;
    L.relu = relu != 0;
    launch_experts_active(a, ctx->stream);
    CK(cudaGetLastError());
    launch_experts_conv(a, L, k, stride, ctx->stream);
    CK(cudaGetLastError());
    return ESACB200_OK;
}

int esacb200_test_gathered(esacb200_ctx* ctx, int world, int M_pad, const double* gathered, float* out_record,
                           const double* pairs, const double* scores, int M, double* norm_out, double* probs, int* contrib,
                           int* n_contrib) {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "test_gathered";
    if (!gathered && !pairs) return fail(ctx, ESACB200_ERR_ARG, "%s: neither gathered nor pairs: nothing to run", what);
    if (world < 1) return fail(ctx, ESACB200_ERR_ARG, "%s: world=%d: need at least one rank", what, world);
    if (gathered) {
        if (M_pad < 1 || (long long)world * M_pad > 0x7fffffffll)
            return fail(ctx, ESACB200_ERR_ARG, "%s: M_pad=%d world=%d: need M_pad >= 1 and world * M_pad < 2^31", what, M_pad, world);
        const void* ptrs[] = {gathered, out_record};
        const char* names[] = {"gathered", "out_record"};
        const int rc = device_args(ctx, what, 2, ptrs, names);
        if (rc) return rc;
        if ((uintptr_t)gathered % 8 || (uintptr_t)out_record % 4)
            return fail(ctx, ESACB200_ERR_ARG, "%s: gathered must be 8-byte and out_record 4-byte aligned", what);
    }
    if (pairs) {
        if (M < 0) return fail(ctx, ESACB200_ERR_ARG, "%s: M=%d: need M >= 0", what, M);
        const void* ptrs[] = {pairs, norm_out, n_contrib, scores, probs, contrib};
        const char* names[] = {"pairs", "norm_out", "n_contrib", "scores", "probs", "contrib"};
        const int rc = device_args(ctx, what, M > 0 ? 6 : 3, ptrs, names);
        if (rc) return rc;
        if ((uintptr_t)pairs % 8 || (uintptr_t)norm_out % 8 || (uintptr_t)n_contrib % 4 || (uintptr_t)scores % 8 ||
            (uintptr_t)probs % 8 || (uintptr_t)contrib % 4)
            return fail(ctx, ESACB200_ERR_ARG, "%s: the double arrays must be 8-byte and the int arrays 4-byte aligned", what);
    }
    if (gathered) {
        launch_select_gathered(gathered, world, M_pad, (ForwardRecord*)out_record, ctx->stream);
        CK(cudaGetLastError());
    }
    if (pairs) {
        Problem P{};
        P.M = M;
        launch_rescale_probs_gathered(scores, P, pairs, world, norm_out, probs, contrib, n_contrib, kProbThresh, ctx->stream);
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(ctx->stream));
    return ESACB200_OK;
}

}  // extern "C"
