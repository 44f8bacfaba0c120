// Pose refinement: iterated inlier re-selection + least-squares PnP.
//
// Replaces refineHyp (esac_util.h:378-454; forward: winner only, esac.cpp:167; backward: every
// hypothesis with p >= PROB_THRESH, esac.cpp:328-347) including the cv::solvePnP(SOLVEPNP_ITERATIVE,
// useExtrinsicGuess=true) it calls (esac_util.h:426-436), which minimises the plain squared
// reprojection error of the current inlier set (SURVEY.md Appendix A).
//
// * The inlier test reproduces getReproErrs' arithmetic exactly (fp64 transform, float-rounded
//   projection, float difference, double norm -> float, clamp, `< tau`), because which cells pass is
//   what makes two implementations agree or not.
// * The least-squares solve reproduces OpenCV's own iteration (cvFindExtrinsicCameraParams2 + CvLevMarq as
//   observed on cv2 4.13: parameters (rvec, tvec), J^T J with its diagonal scaled by 1 + 10^k, k from -3,
//   step accepted when the error norm does not grow, at most 20 iterations, stop when the relative parameter
//   change drops below FLT_EPSILON).  This matters: on world-scale maps (|t| ~ 1e3) that criterion stops long
//   before the minimiser, so only the same iteration gives the same pose and the same next inlier set.
//   Per cell the Jacobian is taken in a cheap, well-conditioned local frame (rotation increment about the
//   plane centre); the reduced 6x6 sums are then mapped to the (rvec, tvec) frame by one 6x6 change of
//   variables per evaluation.
// * A job (one hypothesis) is worked on by a group of `group` CTAs.  The group's first CTA is the ROOT: it alone holds the
//   Levenberg-Marquardt state and takes every decision.  One evaluation = the root broadcasts a command (parameters, R, t)
//   -> every CTA sums its share of the cells (warp shuffle -> shared memory) and publishes 29 block totals in its slot,
//   raising its own epoch flag with a release store -> the root waits for the flags, sums the slots in a fixed order, maps
//   the sums to (rvec, tvec), accepts / rejects, solves for the next step.  Gather + broadcast instead of all-to-all: with
//   every CTA polling every other CTA's flag and re-reading every slot, L2 same-line contention grows with the group size
//   and dominates an evaluation.  Jobs are drawn from a counter by the roots.
#include <cooperative_groups.h>

#include "esac_internal.h"

namespace esacb200 {

constexpr int kRefThreads = 512;
constexpr int kRefWarps = kRefThreads / 32;
constexpr int kRedN = 28;   // 21 (J^T J upper) + 6 (J^T r) + 1 (cost)
constexpr int kSlot = 32;   // doubles per CTA slot / per command record
// A CTA whose share of the map is at most this many 32-cell words keeps its cells in shared memory for the whole job (the
// coordinates never change between evaluations): 96 words = 3072 cells = 36 KB.  Forward at 480x640 on 132 CTAs: 73 words.
constexpr int kCacheWords = 96;
constexpr int kCacheCells = kCacheWords * 32;
// Inlier compaction: after the pass that selects a round's inliers every CTA lists the inlier cells of its share (16-bit
// offsets from its first cell), and the round's LM evaluations walk that list with every lane busy instead of walking all
// cells with the outliers' lanes predicated off -- an fp64 instruction costs the same issue slot however many lanes are on.
// Up to this many 32-cell words per CTA (offsets must fit 16 bits; the popcounts live in shared memory):
constexpr int kMaxCompactWords = 2048;
// Back-off of the exchange's polls (the root's gather and every block's mailbox) between two loads of an element that is not
// there yet.  0, 32 and 64 ns measure the same on the H100 (DESIGN §8).
constexpr unsigned kPollNs = 32;

size_t refine_cache_bytes();
enum { CMD_EVAL = 1, CMD_FIRST = 2, CMD_EXIT = 3 };
// command record (doubles): [0..5] parameters (rvec, tvec), [6..14] R, [15..17] t = R c + tvec, [18] command, [19] job,
// [20] mask buffer the round's tentative inlier set lives in
enum { C_PAR = 0, C_R = 6, C_T = 15, C_CMD = 18, C_JOB = 19, C_SEL = 20, C_COUNT = 21 };

struct RefShared {
    double red[kRefWarps][32];   // per-warp partial sums of the block reduction
    double gat[kRefWarps][32];   // ... of the root's gather (its own buffer: the root's warps may enter the gather while warp 0
                                 // still sums `red` for the block's own totals -- found by compute-sanitizer racecheck)
    double tot[32];
    double cmd[kSlot];
    // ---- root only ----
    double cur[kRedN];   // (rvec, tvec)-frame sums at the last accepted parameters
    double cand[kRedN];  // same at the candidate
    double par[6], prev[6], pose[6], cen[3];
    double Rc[3], dR[27], T[9], G[36], H1[36];
    double A[36], dlt[6];  // root_lm_step's damped matrix and step: in shared memory, not the root thread's local memory
    double prev_cost, best;
    int lamlg, iters, mode, rounds, sel, step, job, h, finished;
    int n_list;                    // inlier cells of this CTA's share in the current round (compaction)
    int wsum[kRefWarps];
    int cnt[kMaxCompactWords];     // per word: popcount, then exclusive prefix
    long long prof_last;  // diagnostics (a.prof != null): clock of the previous phase boundary, thread 0 of block 0
};

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(unsigned* p, unsigned v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// LL exchange element (the protocol NCCL uses for small messages): a double travels as two 8-byte words, each carrying half of
// the value and the exchange's sequence number.  A reader that finds the expected number in BOTH words has the whole value, so
// data and "it is there" arrive in ONE L2 round trip and the writer needs no release fence; buffers are zeroed before a launch
// and sequence numbers start at 1, so a stale element never matches.
__device__ __forceinline__ void st_ll(uint4* p, double v, unsigned seq) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
    asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"((unsigned)b), "r"(seq), "r"((unsigned)(b >> 32)), "r"(seq) : "memory");
}
__device__ __forceinline__ bool ld_ll(const uint4* p, unsigned seq, double& v) {
    uint4 w;
    asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(w.x), "=r"(w.y), "=r"(w.z), "=r"(w.w) : "l"(p) : "memory");
    v = __longlong_as_double((long long)(((unsigned long long)w.z << 32) | w.x));
    return w.y == seq && w.w == seq;
}
// Exchange buffers of a group (uint4 elements): results [block][parity][kSlot], then mailboxes [block][parity][kSlot] -- the
// root writes every block its OWN copy of a command, so a block polls lines nobody else polls.
__device__ __forceinline__ uint4* ll_results(const RefineArgs& a, int grp) {
    return reinterpret_cast<uint4*>(a.scratch) + (size_t)grp * a.group * 4 * kSlot;
}
__device__ __forceinline__ uint4* ll_mailboxes(const RefineArgs& a, int grp) { return ll_results(a, grp) + (size_t)a.group * 2 * kSlot; }

// Phase clock of block 0 / thread 0: adds the cycles since the previous boundary to prof[i] (tools/refine_profile.py).
__device__ __forceinline__ void tick(const RefineArgs& a, RefShared& sh, int i) {
    if (a.prof && blockIdx.x == 0 && threadIdx.x == 0) {
        const long long now = clock64();
        a.prof[i] += now - sh.prof_last;
        sh.prof_last = now;
    }
}

// 10^k for k in [-16, 17]: CvLevMarq's damping factor exp(lambdaLg10 * log(10)) without the two transcendental calls
__device__ __constant__ double kPow10[34] = {1e-16, 1e-15, 1e-14, 1e-13, 1e-12, 1e-11, 1e-10, 1e-9, 1e-8, 1e-7, 1e-6, 1e-5,
                                             1e-4, 1e-3, 1e-2, 1e-1, 1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7,
                                             1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17};
// upper-triangle index of (i, j), i <= j, row-major: 0..20
__device__ __constant__ unsigned char kTriI[21] = {0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 4, 4, 5};
__device__ __constant__ unsigned char kTriJ[21] = {0, 1, 2, 3, 4, 5, 1, 2, 3, 4, 5, 2, 3, 4, 5, 3, 4, 5, 4, 5, 5};
__device__ __constant__ unsigned char kSymIdx[36] = {0, 1, 2, 3, 4, 5, 1, 6, 7, 8, 9, 10, 2, 7, 11, 12, 13, 14,
                                                     3, 8, 12, 15, 16, 17, 4, 9, 13, 16, 18, 19, 5, 10, 14, 17, 19, 20};

// Block reduction of NV doubles held per thread in v[]: totals in sh.tot[0..NV) of THIS block (group == 1) or published in
// this block's slot of the group (group > 1), followed by the release of this block's epoch flag.
template <int NV>
__device__ __forceinline__ void block_reduce_publish(double (&v)[NV], RefShared& sh, const RefineArgs& a, int grp, int cta,
                                                     unsigned seq) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double x = warp_reduce_scatter<NV>(v);
    if (lane < NV) sh.red[warp][lane] = x;
    __syncthreads();
    double s = 0;
    if (tid < NV) {
#pragma unroll
        for (int w = 0; w < kRefWarps; ++w) s += sh.red[w][tid];
    }
    if (a.group == 1) {
        if (tid < NV) sh.tot[tid] = s;
        __syncthreads();
        return;
    }
    if (tid < NV) st_ll(ll_results(a, grp) + ((size_t)cta * 2 + (seq & 1)) * kSlot + tid, s, seq);
}

// Root: wait until every block of the group has published sequence number `seq`, then sum the slots in a fixed order.
template <int NV>
__device__ __forceinline__ void root_gather(RefShared& sh, const RefineArgs& a, int grp, unsigned seq) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint4* res = ll_results(a, grp);
    // thread = (value v = lane, chunk of blocks = warp): up to 10 independent L2 loads in flight per thread, coalesced over v;
    // an element that is not there yet is simply loaded again; partial sums per chunk, then the 16 chunks in a fixed order
    {
        double s = 0;
        if (lane < NV) {
            for (int base = 0; base < a.group; base += 10 * kRefWarps) {
                double x[10];
                unsigned missing = 0;
#pragma unroll
                for (int k = 0; k < 10; ++k) {
                    const int c = base + warp + k * kRefWarps;
                    x[k] = 0.;
                    if (c < a.group && !ld_ll(res + ((size_t)c * 2 + (seq & 1)) * kSlot + lane, seq, x[k])) missing |= 1u << k;
                }
                while (missing) {
                    __nanosleep(kPollNs);  // do not hammer lines their writers are about to store to
#pragma unroll
                    for (int k = 0; k < 10; ++k)
                        if (missing >> k & 1u) {
                            const int c = base + warp + k * kRefWarps;
                            if (ld_ll(res + ((size_t)c * 2 + (seq & 1)) * kSlot + lane, seq, x[k])) missing &= ~(1u << k);
                        }
                }
#pragma unroll
                for (int k = 0; k < 10; ++k) s += x[k];
            }
        }
        sh.gat[warp][lane] = s;
    }
    tick(a, sh, 3);
    __syncthreads();
    if (tid < NV) {
        double s = 0;
#pragma unroll
        for (int w = 0; w < kRefWarps; ++w) s += sh.gat[w][tid];
        sh.tot[tid] = s;
    }
    __syncthreads();
    tick(a, sh, 4);
}

// (row, column) of cell p without an integer division: magic = ceil(2^32 / W) gives floor(p / W) or one more
__device__ __forceinline__ void cell_xy(int p, int W, unsigned magic, int& yy, int& xx) {
    int q = (int)__umulhi((unsigned)p, magic);
    int r = p - q * W;
    if (r < 0) { --q; r += W; }
    yy = q; xx = r;
}

// Per-cell contribution to J^T J (21, upper triangle, row-major) and J^T r (6) for the two residual rows
//   Ju = (c qy, a qz - c qx, -a qy, a, 0, c),  Jv = (-a qz + d qy, -d qx, a qx, 0, a, d)
// written out so the structural zeros cost nothing (x * 0 cannot be dropped by the compiler under IEEE rules).
__device__ __forceinline__ void accumulate_normal(double a_, double c_, double d_, double qx, double qy, double qz, double ru,
                                                  double rv, double* acc) {
    const double u0 = c_ * qy, u1 = a_ * qz - c_ * qx, u2 = -a_ * qy;
    const double v0 = -a_ * qz + d_ * qy, v1 = -d_ * qx, v2 = a_ * qx;
    acc[0] += u0 * u0 + v0 * v0;   // (0,0)
    acc[1] += u0 * u1 + v0 * v1;   // (0,1)
    acc[2] += u0 * u2 + v0 * v2;   // (0,2)
    acc[3] += u0 * a_;             // (0,3)
    acc[4] += v0 * a_;             // (0,4)
    acc[5] += u0 * c_ + v0 * d_;   // (0,5)
    acc[6] += u1 * u1 + v1 * v1;   // (1,1)
    acc[7] += u1 * u2 + v1 * v2;   // (1,2)
    acc[8] += u1 * a_;             // (1,3)
    acc[9] += v1 * a_;             // (1,4)
    acc[10] += u1 * c_ + v1 * d_;  // (1,5)
    acc[11] += u2 * u2 + v2 * v2;  // (2,2)
    acc[12] += u2 * a_;            // (2,3)
    acc[13] += v2 * a_;            // (2,4)
    acc[14] += u2 * c_ + v2 * d_;  // (2,5)
    const double aa = a_ * a_;
    acc[15] += aa;                 // (3,3)
                                   // (3,4) = 0: acc[16] stays 0
    acc[17] += a_ * c_;            // (3,5)
    acc[18] += aa;                 // (4,4)
    acc[19] += a_ * d_;            // (4,5)
    acc[20] += c_ * c_ + d_ * d_;  // (5,5)
    acc[21] += u0 * ru + v0 * rv;
    acc[22] += u1 * ru + v1 * rv;
    acc[23] += u2 * ru + v2 * rv;
    acc[24] += a_ * ru;
    acc[25] += a_ * rv;
    acc[26] += c_ * ru + d_ * rv;
}

// J^T J, J^T r and cost of the reprojection residuals over the masked cells, pose (R, t) in shared memory.
// Coordinates are taken relative to the plane centre c (t here is R*c + t of the true pose): the same least-squares
// problem, but rotation updates pivot inside the scene, which keeps J^T J well conditioned for world-scale maps.
// BUILD_MASK: the pass also decides, for every cell, whether it is an inlier of the true pose (R, t0) -- exactly
// getReproErrs' arithmetic --, writes the bit mask and counts (acc[28]); otherwise the mask is read.
template <bool BUILD_MASK, bool CACHED>
__device__ __forceinline__ void lm_accumulate(const float* __restrict__ pl, const float* __restrict__ cache, const Problem& P,
                                              const double* R, const double* t, const double* c, uint32_t* mask, int w0, int w1,
                                              const double* t0, double (&acc)[kRedN + 1], int* cnt) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < kRedN + 1; ++i) acc[i] = 0;
    const double f = (double)P.f, cx = (double)P.ppx, cy = (double)P.ppy;
    for (int w = w0 + warp; w < w1; w += kRefWarps) {
        const int p = w * 32 + lane;
        const int yy = p / P.W, xx = p - yy * P.W;
        const int ipx = xx * P.sub + P.sub / 2 - P.shiftX, ipy = yy * P.sub + P.sub / 2 - P.shiftY;
        const int lc = (w - w0) * 32 + lane;
        float Xf = 0.f, Yf = 0.f, Zf = 0.f;
        bool inl;
        if (BUILD_MASK) {
            inl = false;
            if (p < P.N) {
                if (CACHED) { Xf = cache[lc]; Yf = cache[kCacheCells + lc]; Zf = cache[2 * kCacheCells + lc]; }
                else { Xf = pl[p]; Yf = pl[P.N + p]; Zf = pl[2 * (size_t)P.N + p]; }
                float err = repro_err_f(R, t0, f, cx, cy, Xf, Yf, Zf, (float)ipx, (float)ipy);
                err = (P.max_reproj < err) ? P.max_reproj : err;  // std::min(err, maxReproj): NaN stays NaN
                inl = err < P.tau;                                  // esac_util.h:406
            }
            const uint32_t bits = __ballot_sync(0xffffffffu, inl);
            if (lane == 0) {
                mask[w] = bits;
                acc[kRedN] += (double)__popc(bits);
                if (cnt) cnt[w - w0] = __popc(bits);
            }
        } else {
            inl = (mask[w] >> lane) & 1u;
            if (inl) {
                if (CACHED) { Xf = cache[lc]; Yf = cache[kCacheCells + lc]; Zf = cache[2 * kCacheCells + lc]; }
                else { Xf = pl[p]; Yf = pl[P.N + p]; Zf = pl[2 * (size_t)P.N + p]; }
            }
        }
        if (inl) {
            const double px = (double)ipx, py = (double)ipy;
            const double X = (double)Xf - c[0], Y = (double)Yf - c[1], Z = (double)Zf - c[2];
            const double qx = R[0] * X + R[1] * Y + R[2] * Z;
            const double qy = R[3] * X + R[4] * Y + R[5] * Z;
            const double qz = R[6] * X + R[7] * Y + R[8] * Z;
            const double zc = qz + t[2];
            const double iz = zc != 0. ? 1. / zc : 1.;
            const double xn = (qx + t[0]) * iz, yn = (qy + t[1]) * iz;
            const double ru = xn * f + cx - px, rv = yn * f + cy - py;
            const double a_ = f * iz, c_ = -f * xn * iz, d_ = -f * yn * iz;
            acc[27] += ru * ru + rv * rv;
            accumulate_normal(a_, c_, d_, qx, qy, qz, ru, rv, acc);
        }
    }
}

// Selection pass of a round: the inlier bit of every cell of the share at the round's pose.  What decides is getReproErrs'
// arithmetic (repro_err_f: fp64 transform, float-rounded projection, float difference, `< tau`), but it only has to be
// carried out where the answer is in doubt: a float evaluation of the same error (coordinates relative to the plane centre,
// like the scoring kernel) comes with a running bound on its own rounding error, and a cell whose error is further from tau
// than that bound plus 4e-3 px is classified by it -- ~35 fp32 instructions instead of ~60 fp64 ones (each of which occupies
// the fp64 pipe 2.7 times as long) for all but a fraction of a percent of the cells.  NaNs fail both comparisons and take the
// exact path.  tc = R c + t0 (the command's t), t0 the true translation.
template <bool CACHED>
__device__ __forceinline__ void lm_select(const float* __restrict__ pl, const float* __restrict__ cache, const Problem& P,
                                          const double* R, const double* t0, const double* tc, const double* c, uint32_t* mask,
                                          int w0, int w1, int* cnt, bool use_pretest) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const double f = (double)P.f, cx = (double)P.ppx, cy = (double)P.ppy;
    const float A0 = (float)R[0], A1 = (float)R[1], A2 = (float)R[2], A3 = (float)R[3], A4 = (float)R[4], A5 = (float)R[5];
    const float A6 = (float)R[6], A7 = (float)R[7], A8 = (float)R[8];
    const float b0 = (float)tc[0], b1 = (float)tc[1], b2 = (float)tc[2];
    const float c0 = (float)c[0], c1 = (float)c[1], c2 = (float)c[2];  // plane centres are floats to begin with: exact
    const float ab0 = fabsf(b0) + fabsf(b1), ab2 = fabsf(b2);
    const bool pretest = use_pretest && P.tau <= P.max_reproj;  // (tau above the clamp makes every cell an inlier: exact path)
    const unsigned wmagic = (unsigned)((0x100000000ull + (unsigned)P.W - 1u) / (unsigned)P.W);
    for (int w = w0 + warp; w < w1; w += kRefWarps) {
        const int p = w * 32 + lane;
        int yy, xx;
        cell_xy(p, P.W, wmagic, yy, xx);
        const float px = (float)(xx * P.sub + P.sub / 2 - P.shiftX), py = (float)(yy * P.sub + P.sub / 2 - P.shiftY);
        const int lc = (w - w0) * 32 + lane;
        bool inl = false;
        if (p < P.N) {
            float Xf, Yf, Zf;
            if (CACHED) { Xf = cache[lc]; Yf = cache[kCacheCells + lc]; Zf = cache[2 * kCacheCells + lc]; }
            else { Xf = pl[p]; Yf = pl[P.N + p]; Zf = pl[2 * (size_t)P.N + p]; }
            const float d0 = Xf - c0, d1 = Yf - c1, d2 = Zf - c2;
            const float xq = fmaf(A0, d0, fmaf(A1, d1, fmaf(A2, d2, b0)));
            const float yq = fmaf(A3, d0, fmaf(A4, d1, fmaf(A5, d2, b1)));
            const float zq = fmaf(A6, d0, fmaf(A7, d1, fmaf(A8, d2, b2)));
            const float iz = __frcp_rn(zq);
            const float xn = xq * iz, yn = yq * iz;
            const float un = P.f * xn, vn = P.f * yn;
            const float du = un + (P.ppx - px), dv = vn + (P.ppy - py);
            const float e2 = du * du + dv * dv;
            const float ad = fabsf(d0) + fabsf(d1) + fabsf(d2);
            // |error of du| + |error of dv| <= eps (f |1/z| (2 |d| + |b0| + |b1| + (|xn| + |yn|)(|d| + |b2|)) + |un| + |vn| + |pp - p|)
            const float bound = 5e-7f * (P.f * fabsf(iz) * (2.f * ad + ab0 + (fabsf(xn) + fabsf(yn)) * (ad + ab2)) + fabsf(un) + fabsf(vn) +
                                         fabsf(P.ppx - px) + fabsf(P.ppy - py));
            const float m = 4e-3f + 2.f * bound;
            const float lo = P.tau - m, hi = P.tau + m;
            if (pretest && lo > 0.f && e2 < lo * lo) {
                inl = true;
            } else if (pretest && e2 > hi * hi) {
                inl = false;
            } else {
                float err = repro_err_f(R, t0, f, cx, cy, Xf, Yf, Zf, px, py);
                err = (P.max_reproj < err) ? P.max_reproj : err;  // std::min(err, maxReproj): NaN stays NaN
                inl = err < P.tau;                                  // esac_util.h:406
            }
        }
        const uint32_t bits = __ballot_sync(0xffffffffu, inl);
        if (lane == 0) { mask[w] = bits; cnt[w - w0] = __popc(bits); }
    }
}

// The same sums over the listed inlier cells only (list[i] = cell offset from the share's first cell).
template <bool CACHED>
__device__ __forceinline__ void lm_accumulate_list(const float* __restrict__ pl, const float* __restrict__ cache, const Problem& P,
                                                   const double* R, const double* t, const double* c, const unsigned short* list,
                                                   int n, int w0, double (&acc)[kRedN + 1]) {
#pragma unroll
    for (int i = 0; i < kRedN + 1; ++i) acc[i] = 0;
    const double f = (double)P.f, cx = (double)P.ppx, cy = (double)P.ppy;
    const unsigned wmagic = (unsigned)((0x100000000ull + (unsigned)P.W - 1u) / (unsigned)P.W);
    // software pipeline: the list entry and the three coordinates of the NEXT cell are requested before the ~95 fp64
    // instructions of the current one (uncached shares read both from L2: two dependent round trips per cell otherwise,
    // which 4 warps per scheduler do not cover)
    int i = threadIdx.x;
    int lc_n = 0;
    float Xn = 0.f, Yn = 0.f, Zn = 0.f;
    if (i < n) {
        lc_n = list[i];
        if (CACHED) { Xn = cache[lc_n]; Yn = cache[kCacheCells + lc_n]; Zn = cache[2 * kCacheCells + lc_n]; }
        else { const int p = w0 * 32 + lc_n; Xn = pl[p]; Yn = pl[P.N + p]; Zn = pl[2 * (size_t)P.N + p]; }
    }
    for (; i < n; i += kRefThreads) {
        const int lc = lc_n;
        const float Xf = Xn, Yf = Yn, Zf = Zn;
        const int i2 = i + kRefThreads;
        if (i2 < n) {
            lc_n = list[i2];
            if (CACHED) { Xn = cache[lc_n]; Yn = cache[kCacheCells + lc_n]; Zn = cache[2 * kCacheCells + lc_n]; }
            else { const int p2 = w0 * 32 + lc_n; Xn = pl[p2]; Yn = pl[P.N + p2]; Zn = pl[2 * (size_t)P.N + p2]; }
        }
        const int p = w0 * 32 + lc;
        int yy, xx;
        cell_xy(p, P.W, wmagic, yy, xx);
        const double px = (double)(xx * P.sub + P.sub / 2 - P.shiftX), py = (double)(yy * P.sub + P.sub / 2 - P.shiftY);
        const double X = (double)Xf - c[0], Y = (double)Yf - c[1], Z = (double)Zf - c[2];
        const double qx = R[0] * X + R[1] * Y + R[2] * Z;
        const double qy = R[3] * X + R[4] * Y + R[5] * Z;
        const double qz = R[6] * X + R[7] * Y + R[8] * Z;
        const double zc = qz + t[2];
        const double iz = zc != 0. ? 1. / zc : 1.;
        const double xn = (qx + t[0]) * iz, yn = (qy + t[1]) * iz;
        const double ru = xn * f + cx - px, rv = yn * f + cy - py;
        const double a_ = f * iz, c_ = -f * xn * iz, d_ = -f * yn * iz;
        acc[27] += ru * ru + rv * rv;
        accumulate_normal(a_, c_, d_, qx, qy, qz, ru, rv, acc);
    }
}

// Builds the CTA's inlier list from the mask words the selection pass just wrote (sh.cnt holds their popcounts): exclusive
// prefix over the words, then every set bit writes its offset.  Fixed order, so the sums stay reproducible run to run.
__device__ __forceinline__ void build_inlier_list(RefShared& sh, const uint32_t* mask, int w0, int w1, unsigned short* list) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nw = w1 - w0;
    __syncthreads();  // popcounts of every warp are in
    int v[4], s = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) { const int i = tid * 4 + k; v[k] = i < nw ? sh.cnt[i] : 0; s += v[k]; }
    int inc = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int x = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += x; }
    if (lane == 31) sh.wsum[warp] = inc;
    __syncthreads();
    int base = 0;
#pragma unroll
    for (int w = 0; w < kRefWarps; ++w) base += w < warp ? sh.wsum[w] : 0;
    int run = base + inc - s;
#pragma unroll
    for (int k = 0; k < 4; ++k) { const int i = tid * 4 + k; if (i < nw) sh.cnt[i] = run; run += v[k]; }
    if (tid == kRefThreads - 1) sh.n_list = run;
    __syncthreads();
    for (int w = w0 + warp; w < w1; w += kRefWarps) {
        const uint32_t bits = mask[w];
        if ((bits >> lane) & 1u) list[sh.cnt[w - w0] + __popc(bits & ((1u << lane) - 1u))] = (unsigned short)((w - w0) * 32 + lane);
    }
    __syncthreads();
}

// 6x6 SPD solve on one thread by 3x3 block elimination with closed-form (adjugate) 3x3 inverses: two reciprocals and a
// handful of short 3x3 products in the dependency chain instead of Cholesky's six dependent square roots / divisions.
// Returns false when a pivot block is not positive definite (the caller then takes the pseudo-inverse route).
__device__ __forceinline__ bool inv3_spd(const double* M, double* Mi) {  // M symmetric 3x3 (row-major 9), Mi its inverse
    const double c00 = M[4] * M[8] - M[5] * M[5], c01 = M[2] * M[5] - M[1] * M[8], c02 = M[1] * M[5] - M[2] * M[4];
    const double det = M[0] * c00 + M[1] * c01 + M[2] * c02;
    const double m2 = M[0] * M[4] - M[1] * M[1];
    if (!(M[0] > 0) || !(m2 > 0) || !(det > 0)) return false;
    const double id = 1. / det;
    Mi[0] = c00 * id; Mi[1] = c01 * id; Mi[2] = c02 * id;
    Mi[3] = Mi[1]; Mi[4] = (M[0] * M[8] - M[2] * M[2]) * id; Mi[5] = (M[1] * M[2] - M[0] * M[5]) * id;
    Mi[6] = Mi[2]; Mi[7] = Mi[5]; Mi[8] = m2 * id;
    return true;
}
__device__ __forceinline__ bool solve6_block(const double* A, const double* b, double* x) {
    double P[9], Q[9], S[9], Pi[9], W[9], Sc[9], Si[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) { P[i * 3 + j] = A[i * 6 + j]; Q[i * 3 + j] = A[i * 6 + 3 + j]; S[i * 3 + j] = A[(i + 3) * 6 + 3 + j]; }
    if (!inv3_spd(P, Pi)) return false;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) W[i * 3 + j] = Pi[i * 3] * Q[j] + Pi[i * 3 + 1] * Q[3 + j] + Pi[i * 3 + 2] * Q[6 + j];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) Sc[i * 3 + j] = S[i * 3 + j] - (Q[i] * W[j] + Q[3 + i] * W[3 + j] + Q[6 + i] * W[6 + j]);
    // symmetrise (Q^T P^-1 Q is symmetric up to rounding)
    Sc[3] = Sc[1] = 0.5 * (Sc[1] + Sc[3]); Sc[6] = Sc[2] = 0.5 * (Sc[2] + Sc[6]); Sc[7] = Sc[5] = 0.5 * (Sc[5] + Sc[7]);
    if (!inv3_spd(Sc, Si)) return false;
    double y1[3], r2[3], x2[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) y1[i] = Pi[i * 3] * b[0] + Pi[i * 3 + 1] * b[1] + Pi[i * 3 + 2] * b[2];
#pragma unroll
    for (int i = 0; i < 3; ++i) r2[i] = b[3 + i] - (Q[i] * y1[0] + Q[3 + i] * y1[1] + Q[6 + i] * y1[2]);
#pragma unroll
    for (int i = 0; i < 3; ++i) x2[i] = Si[i * 3] * r2[0] + Si[i * 3 + 1] * r2[1] + Si[i * 3 + 2] * r2[2];
#pragma unroll
    for (int i = 0; i < 3; ++i) { x[i] = y1[i] - (W[i * 3] * x2[0] + W[i * 3 + 1] * x2[1] + W[i * 3 + 2] * x2[2]); x[3 + i] = x2[i]; }
    return true;
}

// ---- root-only pieces (warp 0 of the root block) -------------------------------------------------------------------
// 1/(2k+1)! and 1/(2k+2)!, k = 0..17: sin(th)/th and (1 - cos(th))/th^2 as power series in x = th^2
__device__ __constant__ double kInvFactOdd[18] = {
    1.0, 0.16666666666666666, 0.008333333333333333, 0.0001984126984126984, 2.7557319223985893e-06, 2.505210838544172e-08, 1.6059043836821613e-10, 7.647163731819816e-13, 2.8114572543455206e-15, 8.22063524662433e-18, 1.9572941063391263e-20, 3.8681701706306835e-23, 6.446950284384474e-26, 9.183689863795546e-29, 1.1309962886447718e-31, 1.2161250415535181e-34, 1.151633562077195e-37, 9.67759295863189e-41};
__device__ __constant__ double kInvFactEven[18] = {
    0.5, 0.041666666666666664, 0.001388888888888889, 2.48015873015873e-05, 2.755731922398589e-07, 2.08767569878681e-09, 1.1470745597729725e-11, 4.779477332387385e-14, 1.5619206968586225e-16, 4.110317623312165e-19, 8.896791392450574e-22, 1.6117375710961184e-24, 2.4795962632247972e-27, 3.279889237069838e-30, 3.7699876288159054e-33, 3.800390754854744e-36, 3.387157535521162e-39, 2.688220266286636e-42};

// R(par) into cmd[C_R..], t = R c + tvec into cmd[C_T..], par into cmd[C_PAR..].  On the critical path of every evaluation,
// so no square root, division or sine / cosine call: with x = |r|^2,  R = (1 - B x) I + B r r^T + A [r]x,
// A = sin(th)/th and B = (1 - cos(th))/th^2 are entire functions of x (18 terms reach 1e-17 for th <= pi; beyond that --
// rotation vectors longer than pi do not occur in practice -- the library functions take over).
__device__ __forceinline__ void root_rotation_fast(RefShared& sh, const double* cen, int lane) {
    const double rx = sh.par[0], ry = sh.par[1], rz = sh.par[2];
    const double x = rx * rx + ry * ry + rz * rz;
    double A, B;
    if (x <= 10.0) {
        A = kInvFactOdd[17];
        B = kInvFactEven[17];
#pragma unroll
        for (int k = 16; k >= 0; --k) {
            A = kInvFactOdd[k] - x * A;
            B = kInvFactEven[k] - x * B;
        }
    } else {
        const double th = sqrt(x);
        double sn, c;
        sincos(th, &sn, &c);
        A = sn / th;
        B = (1. - c) / x;
    }
    if (lane < 9) {
        const int ra = lane / 3, cb = lane - 3 * ra;
        // r[i] by selects: an array indexed by the lane would live in local memory
        auto r3 = [&](int i) { return i == 0 ? rx : (i == 1 ? ry : rz); };
        // [r]x entry (ra, cb): (0,1) = -rz, (0,2) = ry, (1,0) = rz, (1,2) = -rx, (2,0) = -ry, (2,1) = rx
        const int d = cb - ra;
        double rxm = 0.;
        if (d != 0) {
            const int k = 3 - ra - cb;
            const double sgn = (d == 1 || d == -2) ? -1. : 1.;
            rxm = sgn * r3(k);
        }
        sh.cmd[C_R + lane] = (ra == cb ? 1. - B * x : 0.) + B * r3(ra) * r3(cb) + A * rxm;
    }
    __syncwarp();
    if (lane < 3) {
        const double* R = sh.cmd + C_R;
        sh.Rc[lane] = R[lane * 3] * cen[0] + R[lane * 3 + 1] * cen[1] + R[lane * 3 + 2] * cen[2];
        sh.cmd[C_T + lane] = sh.Rc[lane] + sh.par[3 + lane];
    }
    if (lane < 6) sh.cmd[C_PAR + lane] = sh.par[lane];
    __syncwarp();
}

// dR/dr at sh.par (cv::Rodrigues' Jacobian) and Rc = R c from the command's R; off the critical path (the root runs it
// while the other blocks finish their passes).  Change of variables:
//   local (w', t') = Q (w, t), Q = [[I, 0], [-[Rc]x, I]];  (w, t) = P (r, t), P = blkdiag(T, I),
//   T[:, i] = vee((dR/dr_i) R^T);  G = Q P;  JtJ = G^T H G, JtErr = G^T g.
__device__ __forceinline__ void root_rotation_jacobian(RefShared& sh, const double* cen, int lane) {
    const double rx0 = sh.par[0], ry0 = sh.par[1], rz0 = sh.par[2];
    const double theta = sqrt(rx0 * rx0 + ry0 * ry0 + rz0 * rz0);
    auto eps3 = [](int p_, int q_, int r_) { return (double)((p_ - q_) * (q_ - r_) * (r_ - p_)) * 0.5; };
    const bool tiny = theta < DBL_EPSILON;
    double c = 1., sn = 0., it = 0.;
    if (!tiny) { sincos(theta, &sn, &c); it = 1. / theta; }
    const double c1 = 1. - c;
    const double rr0 = rx0 * it, rr1 = ry0 * it, rr2 = rz0 * it;
    auto rr = [&](int i) { return i == 0 ? rr0 : (i == 1 ? rr1 : rr2); };  // selects, not a lane-indexed local array
    if (lane < 27) {  // dR[i*9 + e] = d R[e] / d r_i
        const int i = lane / 9, e_ = lane - 9 * i, ra = e_ / 3, cb = e_ - 3 * ra;
        double v;
        if (tiny) {
            v = -eps3(ra, cb, i);
        } else {
            const double ri = rr(i);
            const double a0 = -sn * ri, a1 = (sn - 2 * c1 * it) * ri, a2 = c1 * it, a3 = (c - sn * it) * ri, a4 = sn * it;
            const double I_e = ra == cb ? 1. : 0.;
            const double rrt = rr(ra) * rr(cb);
            const double drrt = (ra == i ? rr(cb) : 0.) + (cb == i ? rr(ra) : 0.);
            double rxm = 0;  // [r]x entry (ra, cb) = -eps(ra, cb, k) r_k
#pragma unroll
            for (int k = 0; k < 3; ++k) rxm -= eps3(ra, cb, k) * rr(k);
            const double drx = -eps3(ra, cb, i);
            v = a0 * I_e + a1 * rrt + a2 * drrt + a3 * rxm + a4 * drx;
        }
        sh.dR[lane] = v;
    }
    if (lane < 3) {
        const double* R = sh.cmd + C_R;
        sh.Rc[lane] = R[lane * 3] * cen[0] + R[lane * 3 + 1] * cen[1] + R[lane * 3 + 2] * cen[2];
    }
    __syncwarp();
}
__device__ __forceinline__ void root_change_of_variables(RefShared& sh, int lane) {
    const double* R = sh.cmd + C_R;
    if (lane < 9) {  // T[row][i]: rows (2,1), (0,2), (1,0) of (dR_i R^T)
        const int row = lane / 3, i = lane - 3 * row;
        const int p_ = row == 0 ? 2 : (row == 1 ? 0 : 1), q_ = row == 0 ? 1 : (row == 1 ? 2 : 0);
        const double* d = sh.dR + i * 9 + p_ * 3;
        sh.T[lane] = d[0] * R[q_ * 3] + d[1] * R[q_ * 3 + 1] + d[2] * R[q_ * 3 + 2];
    }
    __syncwarp();
    for (int idx = lane; idx < 36; idx += 32) {
        const int row = idx / 6, col = idx - 6 * row;
        double v = 0;
        if (row < 3) {
            v = col < 3 ? sh.T[row * 3 + col] : 0.;
        } else if (col < 3) {
            const int r = row - 3;  // -[Rc]x row r
            const double K0 = r == 0 ? 0. : (r == 1 ? -sh.Rc[2] : sh.Rc[1]);
            const double K1 = r == 0 ? sh.Rc[2] : (r == 1 ? 0. : -sh.Rc[0]);
            const double K2 = r == 0 ? -sh.Rc[1] : (r == 1 ? sh.Rc[0] : 0.);
            v = K0 * sh.T[col] + K1 * sh.T[3 + col] + K2 * sh.T[6 + col];
        } else {
            v = (col - 3 == row - 3) ? 1. : 0.;
        }
        sh.G[idx] = v;
    }
    __syncwarp();
}
// sh.tot (local-frame sums) -> sh.cand ((rvec, tvec)-frame sums)
__device__ __forceinline__ void root_map_sums(RefShared& sh, int lane) {
    for (int idx = lane; idx < 36; idx += 32) {
        const int i = idx / 6, j = idx - 6 * i;
        double v = 0;
#pragma unroll
        for (int q = 0; q < 6; ++q) v += sh.tot[kSymIdx[i * 6 + q]] * sh.G[q * 6 + j];   // tot[16] = (3,4) = 0
        sh.H1[idx] = v;
    }
    __syncwarp();
    if (lane < 21) {
        const int i = kTriI[lane], j = kTriJ[lane];
        double v = 0;
#pragma unroll
        for (int q = 0; q < 6; ++q) v += sh.G[q * 6 + i] * sh.H1[q * 6 + j];
        sh.cand[lane] = v;
    } else if (lane < 27) {
        const int i = lane - 21;
        double v = 0;
#pragma unroll
        for (int q = 0; q < 6; ++q) v += sh.G[q * 6 + i] * sh.tot[21 + q];
        sh.cand[lane] = v;
    } else if (lane == 27) {
        sh.cand[27] = sh.tot[27];
    }
    __syncwarp();
}
// step(): param = prevParam - solve(JtJ with diag * (1 + 10^lamlg), JtErr)   (CvLevMarq::step), thread 0 of the root
__device__ __forceinline__ void root_lm_step(RefShared& sh) {
    double* A = sh.A;  // the fall-backs index A and dlt at run time, which would put register arrays in local memory
    double* dlt = sh.dlt;
    int k = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = i; j < 6; ++j) { A[i * 6 + j] = sh.cur[k]; A[j * 6 + i] = sh.cur[k]; ++k; }
    const double lambda = kPow10[sh.lamlg + 16];
#pragma unroll
    for (int i = 0; i < 6; ++i) A[i * 6 + i] *= 1. + lambda;
    // solve(JtJN, JtErr, DECOMP_SVD): direct solve when the damped matrix is positive definite (the solution is the same
    // up to rounding, which the iteration is insensitive to), SVD-style pseudo-inverse otherwise
    if (!solve6_block(A, &sh.cur[21], dlt) && !chol_solve6(A, &sh.cur[21], dlt)) {
        double Ai[36];
        pinv_sym6(A, Ai);
        for (int i = 0; i < 6; ++i) {
            double d = 0;
            for (int j = 0; j < 6; ++j) d += Ai[i * 6 + j] * sh.cur[21 + j];
            dlt[i] = d;
        }
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) sh.par[i] = sh.prev[i] - dlt[i];
}

// One refinement launch: n_groups groups of a.group CTAs, jobs handed to the groups (refine_body.inc).
template <bool DEV>
__global__ void __launch_bounds__(kRefThreads, 1) refine_kernel(const __grid_constant__ RefineArgs a) {
    __shared__ RefShared sh;
    extern __shared__ float cell_cache[];  // [3][kCacheCells] + the inlier list when the block's share fits (a.cache != 0)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n_groups = gridDim.x / a.group;
#include "refine_body.inc"
}

// refine_kernel<true> with the group picked on the device (a_in.group == 0, stream-ordered backward): the group follows from
// the job count *n_jobs by refine_group_rule, and n_groups, cache and clist from the group as refine_sizes derives them on
// the host.  The grid is the largest any group needs; the CTAs past the chosen group's launch leave at once.  The body is
// refine_kernel's, text for text: an argument copy in refine_kernel itself would change its code.
__global__ void __launch_bounds__(kRefThreads, 1) refine_group_kernel(const __grid_constant__ RefineArgs a_in) {
    constexpr bool DEV = true;
    __shared__ RefShared sh;
    extern __shared__ float cell_cache[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nj = a_in.n_jobs ? *a_in.n_jobs : a_in.n_jobs_host;
    const int g = refine_group_rule(a_in.P.N, a_in.coresident, a_in.group_opt, a_in.jobs_per_group, nj > 1 ? nj : 1);
    const int n_groups = refine_n_groups(a_in.coresident, g, a_in.max_jobs);
    if ((int)blockIdx.x >= n_groups * g) return;
    const int wpc_g = ((a_in.P.N + 31) / 32 + g - 1) / g;
    RefineArgs ad = a_in;
    ad.group = g;
    ad.cache = wpc_g <= kCacheWords ? 1 : 0;
    if (!a_in.compact || ad.cache || wpc_g > kMaxCompactWords) ad.clist = nullptr;
    const RefineArgs& a = ad;
#include "refine_body.inc"
}

// a.group == 0 (group picked on the device): n_groups is the CTA count of the largest launch any group needs.
void launch_refine(const RefineArgs& a, int n_groups, cudaStream_t st) {
    dim3 grid(a.group ? n_groups * a.group : n_groups), block(kRefThreads);
    const size_t smem = a.cache ? refine_cache_bytes() : 0;
    void* params[] = {(void*)&a};
    const void* fn = a.group == 0 ? (const void*)refine_group_kernel
                     : a.dev.shift ? (const void*)refine_kernel<true> : (const void*)refine_kernel<false>;
    // above the 48 KB a kernel gets without asking; the attribute is per device, so it is set on every launch (it is cheap)
    cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)refine_cache_bytes());
    if (a.group != 1) cudaLaunchCooperativeKernel(fn, grid, block, params, smem, st);
    else cudaLaunchKernel(fn, grid, block, params, smem, st);
}

int refine_cache_words() { return kCacheWords; }
size_t refine_cache_bytes() { return (size_t)3 * kCacheCells * sizeof(float) + (size_t)kCacheCells * sizeof(unsigned short); }
int refine_max_compact_words() { return kMaxCompactWords; }
// scratch doubles (zeroed before every launch: LL elements) / flag words a launch of n_groups x group blocks needs
size_t refine_scratch_doubles(int n_groups, int group) { return (size_t)n_groups * group * 4 * kSlot * 2; }
size_t refine_flag_words(int n_groups, int group) { return (size_t)n_groups * (group + 1); }

int refine_max_coresident_blocks(int sm_count) {
    int nb = 0;
    cudaFuncSetAttribute((const void*)refine_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)refine_cache_bytes());
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, refine_kernel<false>, kRefThreads, refine_cache_bytes()) != cudaSuccess) {
        cudaGetLastError();
        nb = 1;
    }
    if (nb < 1) nb = 1;
    return nb * sm_count;
}

__global__ void finish_forward_kernel(const Pose* poses, const int* winner, const int* assign32, const int* flags, ForwardRecord* out) {
    if (threadIdx.x == 0) {
        const int w = *winner;
        double T[16];
        pose2trans(poses[w], T);
        for (int i = 0; i < 16; ++i) out->pose[i] = (float)T[i];
        out->expert = (float)assign32[w];
        out->bad = (float)flags[0];
        out->winner = (float)w;
    }
}

// finish_forward_kernel's pose and expert, written to the caller's arrays of a stream-ordered forward; a bad assignment
// gives a NaN pose, expert -1 and status 1.  The last image of an execution advances the async call counter.
__global__ void finish_forward_async_kernel(const Pose* poses, const int* winner, const int* assign32, const int* flags,
                                            float* pose16, long long* expert, int* status, unsigned long long* seed, int advance) {
    if (threadIdx.x == 0) {
        const int w = *winner;
        const int bad = flags[0];
        double T[16];
        pose2trans(poses[w], T);
        for (int i = 0; i < 16; ++i) pose16[i] = bad ? __int_as_float(0x7fffffff) : (float)T[i];
        *expert = bad ? -1 : (long long)assign32[w];
        *status = bad;
        if (advance) seed[1] += (unsigned long long)advance;
    }
}

__global__ void seed_reset_kernel(unsigned long long* seed, unsigned long long base) {
    seed[0] = base;
    seed[1] = 0;
}

// Index of ShardTail member m among the doubles of the tail.
#define TAIL_AT(m) ((int)(offsetof(ShardTail, m) / sizeof(double)))

// Record one shard contributes to the all-gather of the sharded forward (SURVEY 8e), as doubles: its scores (M_pad; entries
// >= M are -inf: shards may hold different numbers of hypotheses), then a ShardTail from the forward record `fwd`.  M == 0
// gives an all -inf record.  One double per thread.
__global__ void pack_forward_kernel(const double* scores, const ForwardRecord* fwd, int M, int M_pad, int expert_offset,
                                    int hyp_offset, int hyp_stride, double* pack) {
    const double ninf = __longlong_as_double(0xfff0000000000000ull);  // -inf
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < M_pad + kPackTail; i += gridDim.x * blockDim.x) {
        double v;
        if (i < M_pad) v = i < M ? scores[i] : ninf;
        else if (i == M_pad + TAIL_AT(M)) v = (double)M;
        else if (i == M_pad + TAIL_AT(hyp_offset)) v = (double)hyp_offset;
        else if (i == M_pad + TAIL_AT(hyp_stride)) v = (double)hyp_stride;
        else if (M == 0) v = -1.;
        else if (i < M_pad + TAIL_AT(expert)) v = (double)fwd->pose[i - M_pad];
        else if (i == M_pad + TAIL_AT(expert)) v = fwd->bad != 0.f ? -1. : (double)fwd->expert + (double)expert_offset;
        else v = (double)fwd->winner;
        pack[i] = v;
    }
}

void launch_pack_forward(const double* scores, const ForwardRecord* fwd, int M, int M_pad, int expert_offset, int hyp_offset,
                         int hyp_stride, double* pack, cudaStream_t st) {
    pack_forward_kernel<<<(M_pad + kPackTail + 255) / 256, 256, 0, st>>>(scores, fwd, M, M_pad, expert_offset, hyp_offset, hyp_stride, pack);
}

// softMax + draw(training = false) over the gathered records of all shards (esac_util.h:461-530): the first strict maximum in
// the hypothesis order of the UNSHARDED problem (global index = the record's hyp_offset + k * hyp_stride).  One block.
// out: the camera pose of the global winner, its expert, 1 if any shard flagged a bad assignment, its global hypothesis index
// and its owning rank.
__global__ void __launch_bounds__(256) select_gathered_kernel(const double* __restrict__ g, int world, int M_pad, ForwardRecord* out) {
    __shared__ double sbest[8];
    __shared__ long long sidx[8];
    __shared__ int srank[8];
    __shared__ int sbad;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rec = M_pad + kPackTail;
    if (tid == 0) sbad = 0;
    __syncthreads();
    double best = __longlong_as_double(0xfff0000000000000ull);  // -inf
    long long bi = 0x7fffffffffffffffll;
    int br = 0;
    for (int i = tid; i < world * M_pad; i += blockDim.x) {
        const int r = i / M_pad, k = i - r * M_pad;
        const double* rr = g + (size_t)r * rec;
        // (indexed rather than through a ShardTail view, which compiles this loop differently)
        if (k >= (int)rr[M_pad + TAIL_AT(M)]) continue;
        const double v = rr[k];
        const long long gi = (long long)rr[M_pad + TAIL_AT(hyp_offset)] + (long long)k * (long long)rr[M_pad + TAIL_AT(hyp_stride)];
        if (v > best || (v == best && gi < bi)) { best = v; bi = gi; br = r; }
    }
    for (int r = tid; r < world; r += blockDim.x) {
        const ShardTail& t = *(const ShardTail*)(g + (size_t)r * rec + M_pad);
        if (t.M > 0. && t.expert < 0.) atomicExch(&sbad, 1);
    }
    for (int o = 16; o; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o);
        const long long oi = __shfl_xor_sync(0xffffffffu, bi, o);
        const int orr = __shfl_xor_sync(0xffffffffu, br, o);
        if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; br = orr; }
    }
    if (lane == 0) { sbest[warp] = best; sidx[warp] = bi; srank[warp] = br; }
    __syncthreads();
    if (tid == 0) {
        double b = sbest[0];
        long long i = sidx[0];
        int r = srank[0];
        for (int w = 1; w < 8; ++w)
            if (sbest[w] > b || (sbest[w] == b && sidx[w] < i)) { b = sbest[w]; i = sidx[w]; r = srank[w]; }
        if (i == 0x7fffffffffffffffll) { i = 0; r = 0; }
        const ShardTail& t = *(const ShardTail*)(g + (size_t)r * rec + M_pad);
        for (int k = 0; k < 16; ++k) out->pose[k] = (float)t.pose[k];
        out->expert = (float)t.expert;
        out->bad = (float)sbad;
        out->winner = (float)i;
        out->rank = (float)r;
    }
}

#undef TAIL_AT

void launch_select_gathered(const double* gathered, int world, int M_pad, ForwardRecord* rec, cudaStream_t st) {
    select_gathered_kernel<<<1, 256, 0, st>>>(gathered, world, M_pad, rec);
}

void launch_finish_forward_async(const Pose* poses, const int* winner, const int* assign32, const int* flags, float* pose16,
                                 long long* expert, int* status, unsigned long long* seed, int advance, cudaStream_t st) {
    finish_forward_async_kernel<<<1, 32, 0, st>>>(poses, winner, assign32, flags, pose16, expert, status, seed, advance);
}

void launch_seed_reset(unsigned long long* seed, unsigned long long base, cudaStream_t st) {
    seed_reset_kernel<<<1, 1, 0, st>>>(seed, base);
}

void launch_finish_forward(const Pose* poses, const int* winner, const int* assign32, const int* flags, ForwardRecord* rec,
                           cudaStream_t st) {
    finish_forward_kernel<<<1, 32, 0, st>>>(poses, winner, assign32, flags, rec);
}

}  // namespace esacb200
