// Backward pass: expected pose loss and its gradient w.r.t. the scene coordinates, matrix-free.
//
// Replaces esac_backward's tail (esac.cpp:353-510) and esac_derivative.h / esac_loss.h:
//   losses + expectation              esac.cpp:354-362, esac_loss.h:66-83
//   path I  (refinement, implicit)    esac.cpp:373-463   J_R = -(J^T J)^-1 J^T, clamp > 10, dLoss * dHyp_dObjs
//   path II (score)                   esac_derivative.h:205-324 (dScore), 347-420 (dSMScore), 128-185 (dPNP)
//   assembly                          esac.cpp:491-508   out[e][c][y][x] += p_h * gradI + gradII   (float += double)
// The reference materialises a 6 x 3N matrix and an N x 6 Jacobian per hypothesis (11 GB at 480x640 x 256);
// here per hypothesis only 27 reduced numbers exist between the passes:
//   A = J^T J at the refined pose over the final inlier set (21), s = sum_cells w * jacobeanHyp row (6);
//   v = -dLoss * pinv(A);   gradI(cell)  = (v . J_cell) * dProjectdObj_refined(cell)
//   gradII(cell) = w(cell) * dProjectdObj_initial(cell) [+ (s * dPNP) for the 3 minimal-set cells]
#include "esac_internal.h"

namespace esacb200 {

constexpr int kBwdThreads = 256;
constexpr int kBwdPix = 4;                       // cells per thread in the reduction passes
constexpr int kBwdTile = kBwdThreads * kBwdPix;  // 1024
constexpr int kRed = 27;

struct HypGrad {
    int h, expert, flagI, pad;
    double p, g;
    double Ri[9], ti[3], dRi[27];
    double Rr[9], tr[3], dRr[27];
    double dl[6], v[6], inv[36], support[12];
    unsigned long long maxjr_bits;
    int cells[8];
};

size_t bwd_hypgrad_bytes() { return sizeof(HypGrad); }
int bwd_red_vals() { return kRed; }
int bwd_tiles(int N) { return (N + kBwdTile - 1) / kBwdTile; }

// trans2pose for the (float) ground truth: general affine inverse like cv::Mat::inv, then Rodrigues.
__device__ void gt_trans2pose(const float* gt, Pose& p, double T[16]) {
    for (int i = 0; i < 16; ++i) T[i] = (double)gt[i];
    double Ri[9];
    affine_inverse(T, Ri, p.t);
    double X[9];  // a copy of Ri: without it nvcc allocates pose_loss_kernel's registers differently (same arithmetic)
    for (int i = 0; i < 9; ++i) X[i] = Ri[i];
    polar_newton(X);
    rodrigues_m2v(X, p.r);
}

struct BwdAux {
    HypGrad* hg;
    double* red;        // [job][tiles][kRed]
    int* expert_njobs;  // [E]
    int tiles;
};

// The fields of job j's record that do not depend on the loss: hypothesis h, its expert, whether it was refined and which
// refinement mask buffer holds its final inliers, initial and refined rotation with their Rodrigues Jacobians, minimal set.
__device__ __forceinline__ void job_record(const BwdArgs& a, int j, int h, HypGrad& g) {
    g.h = h;
    g.expert = a.assign32[h];
    g.flagI = a.rounds[2 * j] > 0 ? 1 : 0;
    g.pad = a.rounds[2 * j + 1];
    rodrigues_v2m(a.init[h].r, g.Ri, g.dRi);
    rodrigues_v2m(a.ref[h].r, g.Rr, g.dRr);
    for (int i = 0; i < 3; ++i) { g.ti[i] = a.init[h].t[i]; g.tr[i] = a.ref[h].t[i]; }
    for (int i = 0; i < 8; ++i) g.cells[i] = a.cells[h * 8 + i];
}

// ---------------------------------------------------------------------------------------------
// B1: losses, expectation, score gradients, per-job records
// ---------------------------------------------------------------------------------------------
// DEV: the ground truth from dv.gt (stream-ordered backward)
template <bool DEV>
__global__ void __launch_bounds__(1024) bwd_loss_kernel(const __grid_constant__ BwdArgs a, BwdAux x,
                                                        const __grid_constant__ BwdDev dv) {
    const Problem& P = a.P;
    __shared__ Pose gtp;
    __shared__ double gtT[16];
    __shared__ double expected;
    const int tid = threadIdx.x;
    if (tid == 0) gt_trans2pose(DEV ? dv.gt : a.gt, gtp, gtT);
    for (int e = tid; e < P.E; e += blockDim.x) x.expert_njobs[e] = 0;
    __syncthreads();
    for (int h = tid; h < P.M; h += blockDim.x) {
        double T[16];
        pose2trans(a.ref[h], T);
        a.losses[h] = pose_loss(T, gtT, (double)a.wRot, (double)a.wTrans, (double)a.cut);
    }
    __syncthreads();
    if (tid == 0) {
        double s = 0;
        for (int h = 0; h < P.M; ++h) s += a.probs[h] * a.losses[h];  // esac.cpp:357-362 order
        *a.out_loss = s;                                              // local (this rank's) part of the expectation
        expected = a.expected_override ? *a.expected_override : s;    // multi-GPU: sum over all ranks
    }
    __syncthreads();
    const int nc = *a.n_contrib;
    for (int j = tid; j < nc; j += blockDim.x) {
        const int h = a.contrib[j];
        HypGrad& g = x.hg[j];
        job_record(a, j, h, g);
        g.p = a.probs[h];
        g.g = a.probs[h] * a.losses[h] - a.probs[h] * expected;  // esac_derivative.h:372-374
        pose_dloss(a.ref[h], gtp, (double)a.wRot, (double)a.wTrans, (double)a.cut, g.dl);
        g.maxjr_bits = 0ull;
        atomicAdd(&x.expert_njobs[g.expert], 1);
    }
}

// jacobeanR / jacobeanHyp row of one cell (esac_util.h:339-351, esac.cpp:419-431): zero row when err > maxReproj.
__device__ __forceinline__ bool jac_row(const double* R, const double* t, const double* dRdr, double f, double cx, double cy,
                                        float X, float Y, float Z, float px, float py, double max_reproj, double row[6]) {
    float uf, vf;
    project_point_f(R, t, f, cx, cy, X, Y, Z, uf, vf);
    const float dxf = uf - px, dyf = vf - py;
    double err = sqrt((double)dxf * (double)dxf + (double)dyf * (double)dyf);
    err = fmax(err, kEps);
    if (!(err <= max_reproj)) return false;  // `err > maxReproj` -> skipped; NaN rows are dropped here (see DESIGN.md)
    double u, v, Ju[6], Jv[6];
    project_point_jac(R, t, dRdr, f, cx, cy, (double)X, (double)Y, (double)Z, u, v, Ju, Jv);
    const double a_ = 1. / err * (double)dxf, b_ = 1. / err * (double)dyf;
#pragma unroll
    for (int i = 0; i < 6; ++i) row[i] = a_ * Ju[i] + b_ * Jv[i];
    return true;
}

// d score / d reprojection error of one cell (esac_derivative.h:261-266)
__device__ __forceinline__ double score_weight(float err_clamped, const Problem& P, double g, double fac) {
    const float stf = P.beta * (err_clamped - P.tau);
    double st = (double)stf;
    st = 1 / (1 + exp(-st));
    return (-st * (1 - st) * (double)P.beta * g) * fac;
}

// The problem B2-B5 work on: BwdArgs::P, or (DEV) a copy in `local` whose sub, tau, alpha, beta and maxReproj come from
// dv.prob when it is set (the stream-ordered hypotheses backward: the forward's values in the tape header).
template <bool DEV>
__device__ __forceinline__ const Problem& bwd_problem(const BwdArgs& a, const BwdDev& dv, Problem& local) {
    if constexpr (DEV) {
        local = a.P;
        if (dv.prob) {
            local.sub = __ldg(&dv.prob->sub);
            local.tau = __ldg(&dv.prob->tau);
            local.alpha = __ldg(&dv.prob->alpha);
            local.beta = __ldg(&dv.prob->beta);
            local.max_reproj = __ldg(&dv.prob->max_reproj);
        }
        return local;
    } else {
        return a.P;
    }
}

template <bool DEV>
__device__ __forceinline__ void block_reduce_store(double (&v)[kRed], double* dst) {
    __shared__ double sred[kBwdThreads / 32][kRed];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    {
        const double s = warp_reduce_scatter<kRed>(v);
        if (lane < kRed) sred[warp][lane] = s;
    }
    __syncthreads();
    if (threadIdx.x < kRed) {
        double s = 0;
#pragma unroll
        for (int w = 0; w < kBwdThreads / 32; ++w) s += sred[w][threadIdx.x];
        dst[threadIdx.x] = s;
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// B2: per (job, tile) partial sums of J^T J (refined pose, final inliers) and sum w * jacobeanHyp (initial pose)
// ---------------------------------------------------------------------------------------------
template <bool DEV>
__global__ void __launch_bounds__(kBwdThreads) bwd_reduce_kernel(const __grid_constant__ BwdArgs a, BwdAux x,
                                                                 const __grid_constant__ BwdDev dv) {
    Problem Pl;
    const Problem& P = bwd_problem<DEV>(a, dv, Pl);
    const int nc = *a.n_contrib;
    const int n_items = nc * x.tiles;
    const double f = (double)dev_f<DEV>(P, dv), cx = (double)dev_ppx<DEV>(P, dv), cy = (double)dev_ppy<DEV>(P, dv),
                 mr = (double)P.max_reproj;
    const float facf = P.alpha / (float)P.W / (float)P.H;
    __shared__ HypGrad sg;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int j = item / x.tiles, tile = item - j * x.tiles;
        __syncthreads();
        for (int i = threadIdx.x; i < (int)(sizeof(HypGrad) / 8); i += blockDim.x) ((double*)&sg)[i] = ((const double*)&x.hg[j])[i];
        __syncthreads();
        const float* pl = a.coords + (size_t)sg.expert * 3 * P.N;
        const uint32_t* mask = a.masks + ((size_t)j * 2 + sg.pad) * a.mask_words;
        double acc[kRed];
#pragma unroll
        for (int i = 0; i < kRed; ++i) acc[i] = 0;
        for (int k = 0; k < kBwdPix; ++k) {
            const int p = tile * kBwdTile + k * kBwdThreads + threadIdx.x;
            if (p >= P.N) continue;
            const int yy = p / P.W, xx = p - yy * P.W;
            const float px = (float)(xx * P.sub + P.sub / 2 - dev_shift_x<DEV>(P, dv));
            const float py = (float)(yy * P.sub + P.sub / 2 - dev_shift_y<DEV>(P, dv));
            const float X = pl[p], Y = pl[P.N + p], Z = pl[2 * (size_t)P.N + p];
            double row[6];
            if (sg.flagI && ((mask[p >> 5] >> (p & 31)) & 1u)) {
                if (jac_row(sg.Rr, sg.tr, sg.dRr, f, cx, cy, X, Y, Z, px, py, mr, row)) {
                    int q = 0;
#pragma unroll
                    for (int i = 0; i < 6; ++i)
#pragma unroll
                        for (int l = i; l < 6; ++l) acc[q++] += row[i] * row[l];
                }
            }
            // path II weight at the initial pose
            float err = repro_err_f(sg.Ri, sg.ti, f, cx, cy, X, Y, Z, px, py);
            err = (P.max_reproj < err) ? P.max_reproj : err;
            const double w = score_weight(err, P, sg.g, (double)facf);
            if (jac_row(sg.Ri, sg.ti, sg.dRi, f, cx, cy, X, Y, Z, px, py, mr, row)) {
#pragma unroll
                for (int i = 0; i < 6; ++i) acc[21 + i] += w * row[i];
            }
        }
        block_reduce_store<DEV>(acc, x.red + ((size_t)j * x.tiles + tile) * kRed);
    }
}

// ---------------------------------------------------------------------------------------------
// B3: per job small algebra: pinv(J^T J), v, dPNP by central differences (18 P3P solves on 18 lanes), support
// ---------------------------------------------------------------------------------------------
template <bool DEV>
__global__ void __launch_bounds__(32) bwd_solve_kernel(const __grid_constant__ BwdArgs a, BwdAux x,
                                                       const __grid_constant__ BwdDev dv) {
    Problem Pl;
    const Problem& P = bwd_problem<DEV>(a, dv, Pl);
    const int nc = *a.n_contrib;
    const int lane = threadIdx.x;
    __shared__ double tot[kRed];
    __shared__ double fb[18][6];
    __shared__ int okf[18];
    __shared__ double dH[6][12];
    for (int j = blockIdx.x; j < nc; j += gridDim.x) {
        HypGrad& g = x.hg[j];
        __syncwarp();
        if (lane < kRed) {
            double s = 0;
            for (int t = 0; t < x.tiles; ++t) s += x.red[((size_t)j * x.tiles + t) * kRed + lane];
            tot[lane] = s;
        }
        __syncwarp();
        // dPNP (esac_derivative.h:128-185): lane = (i*3 + jj)*2 + dir
        const int h = g.h;
        const float* pl = a.coords + (size_t)g.expert * 3 * P.N;
        if (lane < 18) {
            float obj[4][3], img[4][2];
            for (int q = 0; q < 4; ++q) {
                const int cxq = g.cells[2 * q], cyq = g.cells[2 * q + 1];
                const int p = cyq * P.W + cxq;
                obj[q][0] = pl[p]; obj[q][1] = pl[P.N + p]; obj[q][2] = pl[2 * (size_t)P.N + p];
                img[q][0] = (float)(cxq * P.sub + P.sub / 2 - dev_shift_x<DEV>(P, dv));
                img[q][1] = (float)(cyq * P.sub + P.sub / 2 - dev_shift_y<DEV>(P, dv));
            }
            const int col = lane >> 1, dir = lane & 1, pi = col / 3, pj = col % 3;
            const float eps = 0.001f;
            // float arithmetic of the reference (esac_derivative.h:147-171): x += eps (forward solve);
            // x -= 2*eps (backward solve); x += eps (restore -- not always bit-exact, and the restored value
            // is what the later columns see)
            for (int c = 0; c < col; ++c) {
                float r = obj[c / 3][c % 3] + eps;
                r = r - 2 * eps;
                obj[c / 3][c % 3] = r + eps;
            }
            float vfw = obj[pi][pj] + eps;
            float vbw = vfw - 2 * eps;
            obj[pi][pj] = dir == 0 ? vfw : vbw;
            Pose ps;
            const bool ok =
                p3p_pose(obj, img, (double)dev_f<DEV>(P, dv), (double)dev_ppx<DEV>(P, dv), (double)dev_ppy<DEV>(P, dv), ps);
            okf[lane] = ok ? 1 : 0;
            for (int q = 0; q < 3; ++q) { fb[lane][q] = ps.r[q]; fb[lane][3 + q] = ps.t[q]; }
        }
        __syncwarp();
        if (lane == 0) {
            bool good = true;
            for (int q = 0; q < 18; ++q) good = good && okf[q];
            const double two_eps = (double)(2 * 0.001f);
            double mx = -1;
            for (int r = 0; r < 6; ++r)
                for (int c = 0; c < 12; ++c) dH[r][c] = 0;
            if (good) {
                for (int col = 0; col < 9 && good; ++col)
                    for (int r = 0; r < 6; ++r) {
                        const double val = (fb[2 * col][r] - fb[2 * col + 1][r]) / two_eps;
                        if (!(val == val)) good = false;
                        dH[r][col] = val;
                    }
            }
            if (!good)
                for (int r = 0; r < 6; ++r)
                    for (int c = 0; c < 12; ++c) dH[r][c] = 0;
            for (int r = 0; r < 6; ++r)
                for (int c = 0; c < 12; ++c) { const double v_ = fabs(dH[r][c]); if (mx < 0 || v_ > mx) mx = v_; }
            if (mx > 10)
                for (int r = 0; r < 6; ++r)
                    for (int c = 0; c < 12; ++c) dH[r][c] = 0;
            for (int c = 0; c < 12; ++c) {
                double s = 0;
                for (int r = 0; r < 6; ++r) s += tot[21 + r] * dH[r][c];
                g.support[c] = s;
            }
            // path I algebra
            double A[36];
            int q = 0;
            for (int i = 0; i < 6; ++i)
                for (int l = i; l < 6; ++l) { A[i * 6 + l] = tot[q]; A[l * 6 + i] = tot[q]; ++q; }
            pinv_sym6(A, g.inv);
            for (int i = 0; i < 6; ++i) {
                double s = 0;
                for (int l = 0; l < 6; ++l) s += g.dl[l] * g.inv[l * 6 + i];
                g.v[i] = -s;
            }
        }
        (void)h;
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------
// B4: max |J_R| = max_cells,k |(pinv(A) J_cell^T)_k|  (esac.cpp:434-437 clamp)
// ---------------------------------------------------------------------------------------------
template <bool DEV>
__global__ void __launch_bounds__(kBwdThreads) bwd_maxjr_kernel(const __grid_constant__ BwdArgs a, BwdAux x,
                                                                const __grid_constant__ BwdDev dv) {
    Problem Pl;
    const Problem& P = bwd_problem<DEV>(a, dv, Pl);
    const int nc = *a.n_contrib;
    const int n_items = nc * x.tiles;
    const double f = (double)dev_f<DEV>(P, dv), cx = (double)dev_ppx<DEV>(P, dv), cy = (double)dev_ppy<DEV>(P, dv),
                 mr = (double)P.max_reproj;
    __shared__ HypGrad sg;
    __shared__ double smax[kBwdThreads / 32];
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int j = item / x.tiles, tile = item - j * x.tiles;
        __syncthreads();
        for (int i = threadIdx.x; i < (int)(sizeof(HypGrad) / 8); i += blockDim.x) ((double*)&sg)[i] = ((const double*)&x.hg[j])[i];
        __syncthreads();
        if (!sg.flagI) continue;
        const float* pl = a.coords + (size_t)sg.expert * 3 * P.N;
        const uint32_t* mask = a.masks + ((size_t)j * 2 + sg.pad) * a.mask_words;
        double mx = 0;
        for (int k = 0; k < kBwdPix; ++k) {
            const int p = tile * kBwdTile + k * kBwdThreads + threadIdx.x;
            if (p >= P.N) continue;
            if (!((mask[p >> 5] >> (p & 31)) & 1u)) continue;
            const int yy = p / P.W, xx = p - yy * P.W;
            const float px = (float)(xx * P.sub + P.sub / 2 - dev_shift_x<DEV>(P, dv));
            const float py = (float)(yy * P.sub + P.sub / 2 - dev_shift_y<DEV>(P, dv));
            double row[6];
            if (!jac_row(sg.Rr, sg.tr, sg.dRr, f, cx, cy, pl[p], pl[P.N + p], pl[2 * (size_t)P.N + p], px, py, mr, row)) continue;
#pragma unroll
            for (int i = 0; i < 6; ++i) {
                double s = 0;
#pragma unroll
                for (int l = 0; l < 6; ++l) s += sg.inv[i * 6 + l] * row[l];
                mx = fmax(mx, fabs(s));
            }
        }
        for (int o = 16; o; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if ((threadIdx.x & 31) == 0) smax[threadIdx.x >> 5] = mx;
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 1; w < kBwdThreads / 32; ++w) mx = fmax(mx, smax[w]);
            atomicMax(&x.hg[j].maxjr_bits, (unsigned long long)__double_as_longlong(mx));  // order-independent
        }
    }
}

// ---------------------------------------------------------------------------------------------
// B5: assembly, one thread per cell, hypotheses of the cell's expert in ascending order
// ---------------------------------------------------------------------------------------------
template <bool DEV>
__global__ void __launch_bounds__(kBwdThreads) bwd_assemble_kernel(const __grid_constant__ BwdArgs a, BwdAux x,
                                                                   const __grid_constant__ BwdDev dv) {
    const Problem& P = a.P;
#include "bwd_assemble_body.inc"
}

// The stream-ordered instantiation: the image's shift and camera from device memory, and an image whose assignment holds a
// bad expert index (the prep flag) keeps its gradient untouched.  The body is the eager kernel's, text for text: reading the
// camera any other way in the eager kernel itself would change its code.
template <>
__global__ void __launch_bounds__(kBwdThreads) bwd_assemble_kernel<true>(const __grid_constant__ BwdArgs a, BwdAux x,
                                                                         const __grid_constant__ BwdDev dv) {
    if (__ldg(dv.flags)) return;
    Problem Pd = a.P;
    Pd.shiftX = dev_shift_x<true>(a.P, dv); Pd.shiftY = dev_shift_y<true>(a.P, dv);
    Pd.f = dev_f<true>(a.P, dv); Pd.ppx = dev_ppx<true>(a.P, dv); Pd.ppy = dev_ppy<true>(a.P, dv);
    if (dv.prob) {
        Pd.sub = __ldg(&dv.prob->sub); Pd.tau = __ldg(&dv.prob->tau); Pd.alpha = __ldg(&dv.prob->alpha);
        Pd.beta = __ldg(&dv.prob->beta); Pd.max_reproj = __ldg(&dv.prob->max_reproj);
    }
    const Problem& P = Pd;
#include "bwd_assemble_body.inc"
}

// ---------------------------------------------------------------------------------------------
// Hypotheses node (esacb200_hypotheses_forward / _backward): the forward keeps the per-job records and the final inlier
// masks in the caller's tape; the backward rebuilds the records with the caller's upstream gradients and runs B2-B5.
// ---------------------------------------------------------------------------------------------
size_t tape_records_offset() { return kTapeHeadBytes; }
size_t tape_masks_offset(int M) { return kTapeHeadBytes + (size_t)M * sizeof(HypGrad); }
size_t tape_bytes(int M, int N) { return tape_masks_offset(M) + (size_t)M * 2 * ((N + 31) / 32) * 4; }

// Per-job records of the contributing hypotheses, the header (with n_contrib) and a contributing flag per hypothesis.
// DEV (stream-ordered forward): the header's shift and camera are those td.dev held when the forward ran, contrib_flags is
// the caller's row, the kernel also writes the row's scores, poses and status, and the last image of an execution advances
// the call counter.  An image whose assignment held a bad expert index records no job, gets NaN scores and poses, zero
// flags and TapeTail::bad = 1.
template <bool DEV>
__global__ void __launch_bounds__(1024) tape_record_kernel(const __grid_constant__ BwdArgs a, TapeHead head, TapeHead* out_head,
                                                           HypGrad* recs, unsigned char* contrib_flags,
                                                           const __grid_constant__ TapeDev td) {
    const int tid = threadIdx.x;
    bool bad = false;
    if constexpr (DEV) bad = __ldg(td.flags) != 0;
    const int nc = bad ? 0 : *a.n_contrib;
    for (int h = tid; h < a.P.M; h += blockDim.x) contrib_flags[h] = 0;
    __syncthreads();
    for (int j = tid; j < nc; j += blockDim.x) {
        const int h = a.contrib[j];
        HypGrad& g = recs[j];
        job_record(a, j, h, g);
        g.p = 0;
        g.g = 0;
        for (int i = 0; i < 6; ++i) g.dl[i] = 0;
        g.maxjr_bits = 0ull;
        contrib_flags[h] = 1;
    }
    if (tid == 0) {
        head.n_contrib = nc;
        if constexpr (DEV) {
            head.P.shiftX = __ldg(td.dev.shift); head.P.shiftY = __ldg(td.dev.shift + 1);
            head.P.f = __ldg(td.dev.cam); head.P.ppx = __ldg(td.dev.cam + 1); head.P.ppy = __ldg(td.dev.cam + 2);
        }
        *out_head = head;
        if constexpr (DEV) {
            ((TapeTail*)((char*)out_head + kTapeTailOffset))->bad = bad ? 1 : 0;
            *td.status = bad ? 1 : 0;
            if (td.advance) td.seed[1] += (unsigned long long)td.advance;
        }
    }
    if constexpr (DEV) {
        const double nan = __longlong_as_double(0x7ff8000000000000ll);
        for (int h = tid; h < a.P.M; h += blockDim.x) {
            td.out_scores[h] = bad ? nan : td.scores[h];
            const Pose& q = td.poses[h];
            for (int i = 0; i < 3; ++i) {
                td.out_poses6[(size_t)h * 6 + i] = bad ? nan : q.r[i];
                td.out_poses6[(size_t)h * 6 + 3 + i] = bad ? nan : q.t[i];
            }
        }
    }
}

void launch_tape_records(const BwdArgs& a, const TapeHead& head, void* tape, unsigned char* contrib_flags, cudaStream_t st) {
    tape_record_kernel<false><<<1, 1024, 0, st>>>(a, head, (TapeHead*)tape, (HypGrad*)((char*)tape + tape_records_offset()),
                                                  contrib_flags, TapeDev());
}

void launch_tape_records_async(const BwdArgs& a, const TapeHead& head, void* tape, unsigned char* contrib_flags, const TapeDev& td,
                               cudaStream_t st) {
    tape_record_kernel<true><<<1, 1024, 0, st>>>(a, head, (TapeHead*)tape, (HypGrad*)((char*)tape + tape_records_offset()),
                                                 contrib_flags, td);
}

// What the DEV form of bwd_upstream_kernel reads and publishes (launch_backward_upstream_async).
struct UpstreamDev {
    const TapeHead* head = nullptr;
    int M = 0;
    int* count = nullptr;   // the job count B2-B4 read (BwdArgs::n_contrib)
    int* skip = nullptr;    // B5's flag (BwdDev::flags)
    int* status = nullptr;
};

// B1 of the hypotheses node: the tape's records with the caller's upstream gradients.  Path I takes dl = dL/d pose_h with
// multiplier p = 1, path II takes g = dL/d s_h; B2-B5 are then the vector-Jacobian product of (scores, poses).
// DEV (stream-ordered backward): the job count comes from the header, checked here against a.P and ud.M; a tape of another
// problem (status 2) or of a forward with a bad assignment (status 1) runs no job and sets the skip flag.  A null upstream
// counts as zero.
template <bool DEV>
__global__ void __launch_bounds__(1024) bwd_upstream_kernel(const __grid_constant__ BwdArgs a, BwdAux x, const HypGrad* recs,
                                                            const double* d_scores, const double* d_poses6,
                                                            const __grid_constant__ UpstreamDev ud) {
    const int tid = threadIdx.x;
    for (int e = tid; e < a.P.E; e += blockDim.x) x.expert_njobs[e] = 0;
    int nc;
    if constexpr (DEV) {
        const TapeHead* hd = ud.head;
        const bool foreign = hd->magic != kTapeMagic || hd->M != ud.M || hd->P.E != a.P.E || hd->P.H != a.P.H ||
                             hd->P.W != a.P.W || hd->n_contrib < 0 || hd->n_contrib > ud.M;
        const int status = foreign ? 2 : (((const TapeTail*)((const char*)hd + kTapeTailOffset))->bad ? 1 : 0);
        nc = status ? 0 : hd->n_contrib;
        if (tid == 0) {
            *ud.count = nc;
            *ud.skip = status != 0;
            *ud.status = status;
        }
    } else {
        nc = *a.n_contrib;
    }
    const size_t n8 = (size_t)nc * (sizeof(HypGrad) / 8);
    for (size_t i = tid; i < n8; i += blockDim.x) ((double*)x.hg)[i] = ((const double*)recs)[i];
    __syncthreads();
    for (int j = tid; j < nc; j += blockDim.x) {
        HypGrad& g = x.hg[j];
        const int h = g.h;
        g.p = 1.0;
        if constexpr (DEV) {
            g.g = d_scores ? d_scores[h] : 0.0;
            for (int i = 0; i < 6; ++i) g.dl[i] = d_poses6 ? d_poses6[(size_t)h * 6 + i] : 0.0;
        } else {
            g.g = d_scores[h];
            for (int i = 0; i < 6; ++i) g.dl[i] = d_poses6[(size_t)h * 6 + i];
        }
        g.maxjr_bits = 0ull;
        atomicAdd(&x.expert_njobs[g.expert], 1);
    }
}

// The reference's loss and dLoss of B x M scene poses, image b against its own ground truth (esacb200_pose_loss_batch): the
// device functions of B1.  CTA (x, b) handles poses [256x, 256x + 256) of image b and reads that image's ground truth from
// device memory, so no host round trip precedes the launch.  256 threads: at 1024 pose_dloss spills.
__global__ void __launch_bounds__(256) pose_loss_kernel(const Pose* poses, int M, const float* gt16, float wRot, float wTrans,
                                                         float cut, double* losses, double* dloss6) {
    __shared__ Pose gtp;
    __shared__ double gtT[16];
    const int b = blockIdx.y;
    if (threadIdx.x == 0) gt_trans2pose(gt16 + (size_t)b * 16, gtp, gtT);
    __syncthreads();
    const int h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= M) return;
    const size_t i = (size_t)b * M + h;
    double T[16];
    pose2trans(poses[i], T);
    losses[i] = pose_loss(T, gtT, (double)wRot, (double)wTrans, (double)cut);
    pose_dloss(poses[i], gtp, (double)wRot, (double)wTrans, (double)cut, dloss6 + i * 6);
}

void launch_pose_loss(const Pose* poses, int B, int M, const float* gt16, float wRot, float wTrans, float cut, double* losses,
                      double* dloss6, cudaStream_t st) {
    pose_loss_kernel<<<dim3((M + 255) / 256, B), 256, 0, st>>>(poses, M, gt16, wRot, wTrans, cut, losses, dloss6);
}

static BwdAux bwd_aux(const BwdArgs& a) {
    BwdAux x;
    x.hg = (HypGrad*)a.hyp_grad;
    x.red = a.red;
    x.expert_njobs = (int*)a.job_of;  // [E] ints, buffer provided by the caller
    x.tiles = bwd_tiles(a.P.N);
    return x;
}

template <bool DEV>
static void launch_backward_tail(const BwdArgs& a, const BwdAux& x, const BwdDev& dv, int max_jobs, int sm_count, cudaStream_t st);

void launch_backward_losses(const BwdArgs& a, cudaStream_t st) {
    bwd_loss_kernel<false><<<1, 1024, 0, st>>>(a, bwd_aux(a), BwdDev());
}

void launch_backward(const BwdArgs& a, int max_jobs, int sm_count, cudaStream_t st, const BwdDev* dev) {
    const BwdAux x = bwd_aux(a);
    if (dev) {
        bwd_loss_kernel<true><<<1, 1024, 0, st>>>(a, x, *dev);
        launch_backward_tail<true>(a, x, *dev, max_jobs, sm_count, st);
    } else {
        bwd_loss_kernel<false><<<1, 1024, 0, st>>>(a, x, BwdDev());
        launch_backward_tail<false>(a, x, BwdDev(), max_jobs, sm_count, st);
    }
}

void launch_backward_upstream(const BwdArgs& a, const void* tape, const double* d_scores, const double* d_poses6, int max_jobs,
                              int sm_count, cudaStream_t st) {
    const BwdAux x = bwd_aux(a);
    bwd_upstream_kernel<false><<<1, 1024, 0, st>>>(a, x, (const HypGrad*)((const char*)tape + tape_records_offset()), d_scores,
                                                   d_poses6, UpstreamDev());
    launch_backward_tail<false>(a, x, BwdDev(), max_jobs, sm_count, st);
}

void launch_backward_upstream_async(const BwdArgs& a, const void* tape, const double* d_scores, const double* d_poses6, int* count,
                                    int* skip, int* status, const BwdDev& dv, int max_jobs, int sm_count, cudaStream_t st) {
    const BwdAux x = bwd_aux(a);
    UpstreamDev ud;
    ud.head = (const TapeHead*)tape;
    ud.M = a.P.M;
    ud.count = count;
    ud.skip = skip;
    ud.status = status;
    bwd_upstream_kernel<true><<<1, 1024, 0, st>>>(a, x, (const HypGrad*)((const char*)tape + tape_records_offset()), d_scores,
                                                  d_poses6, ud);
    launch_backward_tail<true>(a, x, dv, max_jobs, sm_count, st);
}

// B2-B5: everything after the per-job records, shared by the loss-driven backward and the hypotheses node.
template <bool DEV>
static void launch_backward_tail(const BwdArgs& a, const BwdAux& x, const BwdDev& dv, int max_jobs, int sm_count, cudaStream_t st) {
    long long items = (long long)max_jobs * x.tiles;
    int grid = (int)(items < sm_count * 8ll ? items : sm_count * 8ll);
    if (grid < 1) grid = 1;
    bwd_reduce_kernel<DEV><<<grid, kBwdThreads, 0, st>>>(a, x, dv);
    bwd_solve_kernel<DEV><<<max_jobs < sm_count * 4 ? max_jobs : sm_count * 4, 32, 0, st>>>(a, x, dv);
    bwd_maxjr_kernel<DEV><<<grid, kBwdThreads, 0, st>>>(a, x, dv);
    dim3 ga((a.P.N + kBwdThreads - 1) / kBwdThreads, a.P.E);
    bwd_assemble_kernel<DEV><<<ga, kBwdThreads, 0, st>>>(a, x, dv);
}

// esac.backward's return value for a stream-ordered image: the expected loss (NaN on a bad assignment) and the status; the
// last image of an execution advances the async call counter.
__global__ void finish_backward_async_kernel(const CallStats* stats, const int* flags, double* loss, int* status,
                                             unsigned long long* seed, int advance) {
    if (threadIdx.x == 0) {
        const int bad = flags[0];
        *loss = bad ? __longlong_as_double(0x7ff8000000000000ll) : stats->local_loss;
        *status = bad;
        if (advance) seed[1] += (unsigned long long)advance;
    }
}

void launch_finish_backward_async(const CallStats* stats, const int* flags, double* loss, int* status, unsigned long long* seed,
                                  int advance, cudaStream_t st) {
    finish_backward_async_kernel<<<1, 32, 0, st>>>(stats, flags, loss, status, seed, advance);
}

// dst += src (the rank-summed gradient of a hypothesis-major sharded backward joins the caller's tensor: esac.cpp:501-506 is +=)
__global__ void add_inplace_kernel(float* __restrict__ dst, const float* __restrict__ src, size_t n) {
    const size_t n4 = n / 4;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        float4 a = reinterpret_cast<float4*>(dst)[i];
        const float4 b = reinterpret_cast<const float4*>(src)[i];
        a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        reinterpret_cast<float4*>(dst)[i] = a;
    }
    for (size_t i = n4 * 4 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] += src[i];
}

__global__ void add_inplace_scalar_kernel(float* __restrict__ dst, const float* __restrict__ src, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] += src[i];
}

// flags[e] = 1 when expert e has a contributing hypothesis (p >= PROB_THRESH) on this rank: only those planes receive gradient
__global__ void expert_flags_kernel(const int* contrib, const int* n_contrib, const int* assign32, int E, int* flags) {
    for (int e = threadIdx.x; e < E; e += blockDim.x) flags[e] = 0;
    __syncthreads();
    const int n = *n_contrib;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int e = assign32[contrib[i]];
        if (e >= 0 && e < E) flags[e] = 1;
    }
}
void launch_expert_flags(const int* contrib, const int* n_contrib, const int* assign32, int E, int* flags, cudaStream_t st) {
    expert_flags_kernel<<<1, 256, 0, st>>>(contrib, n_contrib, assign32, E, flags);
}

void launch_add_inplace(float* dst, const float* src, size_t n, cudaStream_t st) {
    if ((((uintptr_t)dst) | ((uintptr_t)src)) & 15) add_inplace_scalar_kernel<<<1184, 256, 0, st>>>(dst, src, n);  // unaligned views
    else add_inplace_kernel<<<1184, 256, 0, st>>>(dst, src, n);
}

}  // namespace esacb200
