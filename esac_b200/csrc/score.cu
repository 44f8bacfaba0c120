// Reprojection + soft-inlier scoring (the roofline kernel) and its bookkeeping kernels.
//
// Replaces, for all M hypotheses at once, the reference's per-hypothesis CPU loop
//   getReproErrs (no-Jacobian path)  esac_util.h:274-318,355-362   called from esac.cpp:131-140 / 295-305
//   getHypScores                      esac_util.h:235-260           called from esac.cpp:143 / 308
//   softMax / entropy / draw          esac_util.h:461-530           called from esac.cpp:153-155 / 318-319
//
// Layout: hypotheses are grouped by expert (stable by index), cut into chunks of <= kMaxChunk; a work
// item is (chunk, pixel tile).  A CTA keeps its tile's pixels in registers (re-centred coordinates plus
// the principal-point offset of each cell, two pixels per float2 pair) and streams the chunk's
// folded poses from shared memory, so each coordinate plane is read from HBM/L2 once per chunk instead
// of once per hypothesis.  Per pixel-hypothesis: 9 FFMA for R*X+t, then
//   err = |p| / |z|,  p = (xc + (cx-px) z, yc + (cy-py) z)   ->  err = num * rsqrt(num * z^2)
//   w   = 1 / (1 + 2^(k1*min(err,maxReproj) + k0))           ==  1 - sigmoid(beta*(err - tau))
// i.e. 3 MUFU (rsq, ex2, rcp) and ~20 fp32 ops per cell-hypothesis.  With k1 > 0 ("fold", every practical beta) k1 is
// folded into the rows that carry f and into the pixel offsets, so num * rsqrt(num z^2) is already k1*err, and the two
// cells of a float2 pair share one reciprocal (score_item): 2.5 MUFU and one FMUL less per cell-hypothesis.
//   t = min(num rs + k0 - s, k1 maxReproj + k0 - s),  d = 2^-s + 2^t,  w_a + w_b = 2^-s (d_a + d_b) / (d_a d_b)
// s = kScorePairShift keeps d_a d_b inside fp32 (unscaled, (1 + 2^65)^2 overflows at tau = 10, beta = 0.5, maxReproj = 100).
#include <atomic>

#include "esac_internal.h"

namespace esacb200 {

constexpr int kScoreThreads = 256;
constexpr int kScorePairShift = 32;

// ---------------------------------------------------------------------------------------------
// prep
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) prep_kernel(const float* __restrict__ coords, const long long* __restrict__ assign,
                                                    long long stride, Problem P, int hc, int* assign32, int* counts,
                                                    int* offsets, int* perm, int* slot_of, ChunkDesc* chunks,
                                                    int* n_chunks, int* work_counter, float* centres, int* flags,
                                                    int with_assign) {
    // block 0 (when with_assign): the assignment bookkeeping; every other block: the centre of one expert's plane.  The two
    // roles can be launched separately (with_assign = 1 and no centre blocks / with_assign = 0) when the planes are still
    // on their way from the host.
    const int tid = threadIdx.x;
    if (with_assign && blockIdx.x == 0) {
        if (tid == 0) { *work_counter = 0; flags[0] = 0; }
        for (int e = tid; e < P.E; e += blockDim.x) counts[e] = 0;
        __syncthreads();
        for (int h = tid; h < P.M; h += blockDim.x) {
            long long e = assign[(long long)h * stride];
            if (e < 0 || e >= P.E) { flags[0] = 1; e = 0; }
            assign32[h] = (int)e;
            atomicAdd(&counts[(int)e], 1);
        }
        __syncthreads();
        if (tid == 0) {
            int acc = 0, nc = 0;
            for (int e = 0; e < P.E; ++e) {
                offsets[e] = acc;
                for (int s = 0; s < counts[e]; s += hc) {
                    ChunkDesc c;
                    c.expert = e; c.slot0 = acc + s; c.count = min(hc, counts[e] - s); c.pad = 0;
                    chunks[nc++] = c;
                }
                acc += counts[e];
            }
            offsets[P.E] = acc;
            *n_chunks = nc;
        }
        __syncthreads();
        // stable permutation: warp w ranks the hypotheses of expert e = w, w + nwarps, ... with ballots
        {
            const int lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
            for (int e = warp; e < P.E; e += nwarps) {
                if (counts[e] == 0) continue;
                int pos = offsets[e];
                for (int b = 0; b < P.M; b += 32) {
                    const int h = b + lane;
                    const bool mine = h < P.M && assign32[h] == e;
                    const unsigned m = __ballot_sync(0xffffffffu, mine);
                    if (mine) {
                        const int q = pos + __popc(m & ((1u << lane) - 1u));
                        perm[q] = h;
                        slot_of[h] = q;
                    }
                    pos += __popc(m);
                }
            }
        }
    } else {
        // plane centre: mean of a strided sample (only conditions the fp32 arithmetic, see DESIGN.md)
        const int e = blockIdx.x - with_assign;
        const float* pl = coords + (size_t)e * 3 * P.N;
        const int ns = min(P.N, 4096);
        const int step = max(1, P.N / ns);
        float sx = 0, sy = 0, sz = 0, cnt = 0;
        for (int i = tid; i < ns; i += blockDim.x) {
            int p = min(i * step, P.N - 1);
            float x = pl[p], y = pl[P.N + p], z = pl[2 * P.N + p];
            if (isfinite(x) && isfinite(y) && isfinite(z) && fabsf(x) < 1e18f && fabsf(y) < 1e18f && fabsf(z) < 1e18f) {
                sx += x; sy += y; sz += z; cnt += 1;
            }
        }
        __shared__ float red[4][32];
        for (int o = 16; o; o >>= 1) {
            sx += __shfl_xor_sync(0xffffffffu, sx, o);
            sy += __shfl_xor_sync(0xffffffffu, sy, o);
            sz += __shfl_xor_sync(0xffffffffu, sz, o);
            cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        }
        if ((tid & 31) == 0) { red[0][tid >> 5] = sx; red[1][tid >> 5] = sy; red[2][tid >> 5] = sz; red[3][tid >> 5] = cnt; }
        __syncthreads();
        if (tid == 0) {
            float a = 0, b = 0, c = 0, n = 0;
            for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { a += red[0][w]; b += red[1][w]; c += red[2][w]; n += red[3][w]; }
            float inv = n > 0 ? 1.f / n : 0.f;
            centres[e * 3 + 0] = a * inv; centres[e * 3 + 1] = b * inv; centres[e * 3 + 2] = c * inv;
        }
    }
}

// roles: bit 0 = assignment bookkeeping, bit 1 = plane centres
void launch_prep(const float* coords, const long long* assign, long long assign_stride, const Problem& P, int hc,
                 int* assign32, int* counts, int* offsets, int* perm, int* slot_of, ChunkDesc* chunks, int* n_chunks,
                 int* work_counter, float* centres, int* flags, int roles, cudaStream_t st) {
    const int with_assign = roles & 1, n_centres = (roles & 2) ? P.E : 0;
    if (with_assign + n_centres == 0) return;
    prep_kernel<<<with_assign + n_centres, 1024, 0, st>>>(coords, assign, assign_stride, P, hc, assign32, counts, offsets, perm,
                                                          slot_of, chunks, n_chunks, work_counter, centres, flags, with_assign);
}

// ---------------------------------------------------------------------------------------------
// fold: (rvec, tvec) fp64 -> fp32 rows of diag(f,f,1) R and diag(f,f,1)(R c + t), slot order
// ---------------------------------------------------------------------------------------------
template <bool DEV>
__global__ void fold_kernel(const Pose* __restrict__ poses, const int* __restrict__ perm, const int* __restrict__ assign32,
                            const float* __restrict__ centres, Problem P, float kf, PosePk* __restrict__ out, DevParams dev) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= P.M) return;
    int h = perm[s];
    int e = assign32[h];
    Pose p = poses[h];
    double R[9];
    rodrigues_v2m(p.r, R, nullptr);
    double c[3] = {(double)centres[e * 3], (double)centres[e * 3 + 1], (double)centres[e * 3 + 2]};
    float focal = P.f;
    if constexpr (DEV) focal = __ldg(dev.cam);
    const double f = (double)focal * (double)kf;  // kf = k1 when the scoring kernel folds it, else 1
    float A[12];
    for (int r = 0; r < 3; ++r) {
        double sc = r < 2 ? f : 1.0;
        double b = R[r * 3] * c[0] + R[r * 3 + 1] * c[1] + R[r * 3 + 2] * c[2] + p.t[r];
        A[r * 4 + 0] = (float)(sc * R[r * 3 + 0]);
        A[r * 4 + 1] = (float)(sc * R[r * 3 + 1]);
        A[r * 4 + 2] = (float)(sc * R[r * 3 + 2]);
        A[r * 4 + 3] = (float)(sc * b);
    }
    PosePk pk;
    for (int r = 0; r < 3; ++r) pk.v[r] = make_float4(A[r * 4 + 0], A[r * 4 + 1], A[r * 4 + 2], A[r * 4 + 3]);
    out[s] = pk;
}

void launch_fold(const Pose* poses, const int* perm, const int* assign32, const float* centres, const Problem& P,
                 float kf, PosePk* out, cudaStream_t st, const DevParams* dev) {
    if (dev) fold_kernel<true><<<(P.M + 127) / 128, 128, 0, st>>>(poses, perm, assign32, centres, P, kf, out, *dev);
    else fold_kernel<false><<<(P.M + 127) / 128, 128, 0, st>>>(poses, perm, assign32, centres, P, kf, out, DevParams{});
}

void score_constants(const Problem& P, ScoreArgs& a) {
    const float log2e = 1.4426950408889634f;
    a.k1 = P.beta * log2e;
    a.k0 = -P.beta * P.tau * log2e;
    const float k0s = a.k0 - (float)kScorePairShift;
    a.tmax = fmaf(P.max_reproj, a.k1, k0s);
    // Fold only where the clamp keeps every d <= 2^-s + 2^63 (so d_a d_b stays finite) and 1e-30 k1^2 stays a normal float;
    // everywhere else (beta <= 0, huge beta * maxReproj, non-finite parameters) the per-cell arithmetic is unchanged.
    a.fold = a.k1 >= 1e-3f && std::isfinite(a.k1) && std::isfinite(k0s) && a.tmax <= 63.f;
    if (a.fold) {
        a.k0 = k0s;
        a.tiny = 1e-30f * a.k1 * a.k1;
    } else {
        a.tiny = 1e-30f;
    }
}

// ---------------------------------------------------------------------------------------------
// scoring
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float mufu_rsq(float x) {
    float y;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float mufu_ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float mufu_rcp(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// tileX/Y/Z: when non-null, the tile's three coordinate rows already sit in shared memory (staged by TMA bulk copies);
// otherwise the cells are read from global memory.
template <int PPT, bool TAIL, bool FOLD, bool DEV>
__device__ __forceinline__ void score_item(const ScoreArgs& a, const ChunkDesc cd, const int tile, const float4* sPose,
                                           float (*sWarp)[kMaxChunk], const float* tileX = nullptr,
                                           const float* tileY = nullptr, const float* tileZ = nullptr) {
    constexpr int NP = PPT / 2;                 // pixel pairs per thread
    constexpr int GV = PPT >= 4 ? 4 : 2;        // pixels per load group
    constexpr int NG = PPT / GV;
    constexpr int TP = kScoreThreads * PPT;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const Problem& P = a.P;
    const float* pl = a.coords + (size_t)cd.expert * 3 * P.N;
    const float cX = a.centres[cd.expert * 3], cY = a.centres[cd.expert * 3 + 1], cZ = a.centres[cd.expert * 3 + 2];

    float2 X[NP], Y[NP], Z[NP], A[NP], B[NP], V[NP];
#pragma unroll
    for (int g = 0; g < NG; ++g) {
        const int p0 = tile * TP + g * (kScoreThreads * GV) + tid * GV;
        float x[GV], y[GV], z[GV];
        if (tileX) {
            const int o = g * (kScoreThreads * GV) + tid * GV;  // offset inside the tile
            if (!TAIL) {
                if constexpr (GV == 4) {
                    const float4 vx = *(const float4*)(tileX + o), vy = *(const float4*)(tileY + o), vz = *(const float4*)(tileZ + o);
                    x[0] = vx.x; x[1] = vx.y; x[GV - 2] = vx.z; x[GV - 1] = vx.w;
                    y[0] = vy.x; y[1] = vy.y; y[GV - 2] = vy.z; y[GV - 1] = vy.w;
                    z[0] = vz.x; z[1] = vz.y; z[GV - 2] = vz.z; z[GV - 1] = vz.w;
                } else {
                    const float2 vx = *(const float2*)(tileX + o), vy = *(const float2*)(tileY + o), vz = *(const float2*)(tileZ + o);
                    x[0] = vx.x; x[1] = vx.y; y[0] = vy.x; y[1] = vy.y; z[0] = vz.x; z[1] = vz.y;
                }
            } else {
                const int last = P.N - 1 - tile * TP;  // only the first (N - tile*TP) cells of a ragged tile were copied
#pragma unroll
                for (int i = 0; i < GV; ++i) {
                    const int q = min(o + i, last);
                    x[i] = tileX[q]; y[i] = tileY[q]; z[i] = tileZ[q];
                }
            }
        } else if (a.vec_ok && p0 + GV <= P.N) {
            if constexpr (GV == 4) {
                float4 vx = __ldg((const float4*)(pl + p0));
                float4 vy = __ldg((const float4*)(pl + P.N + p0));
                float4 vz = __ldg((const float4*)(pl + 2 * (size_t)P.N + p0));
                x[0] = vx.x; x[1] = vx.y; x[GV - 2] = vx.z; x[GV - 1] = vx.w;
                y[0] = vy.x; y[1] = vy.y; y[GV - 2] = vy.z; y[GV - 1] = vy.w;
                z[0] = vz.x; z[1] = vz.y; z[GV - 2] = vz.z; z[GV - 1] = vz.w;
            } else {
                float2 vx = __ldg((const float2*)(pl + p0));
                float2 vy = __ldg((const float2*)(pl + P.N + p0));
                float2 vz = __ldg((const float2*)(pl + 2 * (size_t)P.N + p0));
                x[0] = vx.x; x[1] = vx.y; y[0] = vy.x; y[1] = vy.y; z[0] = vz.x; z[1] = vz.y;
            }
        } else {
#pragma unroll
            for (int i = 0; i < GV; ++i) {
                int p = min(p0 + i, P.N - 1);
                x[i] = __ldg(pl + p); y[i] = __ldg(pl + P.N + p); z[i] = __ldg(pl + 2 * (size_t)P.N + p);
            }
        }
        float aa[GV], bb[GV], vv[GV];
#pragma unroll
        for (int i = 0; i < GV; ++i) {
            int p = p0 + i;
            int py = p / P.W, px = p - py * P.W;
            // createSampling (esac_util.h:64-66): integer pixel centre, then ppoint - pixel in float
            aa[i] = dev_ppx<DEV>(P, a) - (float)(px * P.sub + P.sub / 2 - dev_shift_x<DEV>(P, a));
            bb[i] = dev_ppy<DEV>(P, a) - (float)(py * P.sub + P.sub / 2 - dev_shift_y<DEV>(P, a));
            if (FOLD) { aa[i] = __fmul_rn(aa[i], a.k1); bb[i] = __fmul_rn(bb[i], a.k1); }
            vv[i] = (p < P.N) ? 1.f : 0.f;
            x[i] -= cX; y[i] -= cY; z[i] -= cZ;
        }
#pragma unroll
        for (int i = 0; i < GV / 2; ++i) {
            const int j = g * (GV / 2) + i;
            X[j] = make_float2(x[2 * i], x[2 * i + 1]);
            Y[j] = make_float2(y[2 * i], y[2 * i + 1]);
            Z[j] = make_float2(z[2 * i], z[2 * i + 1]);
            A[j] = make_float2(aa[2 * i], aa[2 * i + 1]);
            B[j] = make_float2(bb[2 * i], bb[2 * i + 1]);
            V[j] = make_float2(vv[2 * i], vv[2 * i + 1]);
        }
    }
    const float2 k1 = make_float2(a.k1, a.k1), k0 = make_float2(a.k0, a.k0);
    const float2 one = make_float2(1.f, 1.f), tiny = make_float2(a.tiny, a.tiny);
    const float mr = FOLD ? a.tmax : P.max_reproj;
    const float d0 = 1.f / (float)(1ull << kScorePairShift);

    // soft-inlier sum of this thread's PPT cells for hypothesis hl (pose = 3 x LDS.128, scalars broadcast to float2)
    auto one_hyp = [&](int hl) -> float {
        const float4* q = sPose + hl * 3;
        const float4 r0 = q[0], r1 = q[1], r2 = q[2];
        const float2 a00 = make_float2(r0.x, r0.x), a01 = make_float2(r0.y, r0.y), a02 = make_float2(r0.z, r0.z), b0 = make_float2(r0.w, r0.w);
        const float2 a10 = make_float2(r1.x, r1.x), a11 = make_float2(r1.y, r1.y), a12 = make_float2(r1.z, r1.z), b1 = make_float2(r1.w, r1.w);
        const float2 a20 = make_float2(r2.x, r2.x), a21 = make_float2(r2.y, r2.y), a22 = make_float2(r2.z, r2.z), b2 = make_float2(r2.w, r2.w);
        float2 acc = make_float2(0.f, 0.f);  // FOLD: pair sums in units of 2^-s in acc.x
#pragma unroll
        for (int j = 0; j < NP; ++j) {
            float2 xc = ffma2(a00, X[j], ffma2(a01, Y[j], ffma2(a02, Z[j], b0)));
            float2 yc = ffma2(a10, X[j], ffma2(a11, Y[j], ffma2(a12, Z[j], b1)));
            float2 zc = ffma2(a20, X[j], ffma2(a21, Y[j], ffma2(a22, Z[j], b2)));
            float2 pu = ffma2(A[j], zc, xc);
            float2 pv = ffma2(B[j], zc, yc);
            // num >= 1e-30 (the 1e-30 vanishes in the rounding of any |p|^2 above 1e-22): a cell on the pixel's ray still gets
            // err ~ 0, while zc == 0 gives m = 0 -> rsq = +inf -> err = +inf -> maxReproj, also for a cell AT the camera centre
            // (p = 0), which a 1e-30 added to m instead would score as a perfect inlier.  No extra instruction.
            float2 num = ffma2(pu, pu, ffma2(pv, pv, tiny));
            float2 m = fmul2(fmul2(zc, zc), num);
            float2 rs = make_float2(mufu_rsq(m.x), mufu_rsq(m.y));
            if (FOLD) {
                // NaN (and zc == 0 -> rs = +inf) clamps to tmax exactly as err does below
                const float ta = fminf(__fmaf_rn(num.x, rs.x, k0.x), mr), tb = fminf(__fmaf_rn(num.y, rs.y, k0.x), mr);
                const float da = __fadd_rn(mufu_ex2(ta), d0);
                float db = __fadd_rn(mufu_ex2(tb), d0), ds;
                if (TAIL) {  // valid cells are a prefix of the tile: b masked -> 1/d_a, both masked -> 0
                    const bool vb = V[j].y != 0.f;
                    ds = __fmul_rn(vb ? __fadd_rn(da, db) : da, V[j].x);
                    db = vb ? db : da;
                } else {
                    ds = __fadd_rn(da, db);
                }
                acc.x = __fmaf_rn(ds, mufu_rcp(__fmul_rn(da, db)), acc.x);
                continue;
            }
            float2 err = fmul2(num, rs);
            err.x = fminf(err.x, mr);
            err.y = fminf(err.y, mr);
            float2 t = ffma2(err, k1, k0);
            float2 ex = make_float2(mufu_ex2(t.x), mufu_ex2(t.y));
            float2 den = fadd2(ex, one);
            float2 w = make_float2(mufu_rcp(den.x), mufu_rcp(den.y));
            if (TAIL) acc = ffma2(w, V[j], acc);
            else acc = fadd2(acc, w);
        }
        return FOLD ? acc.x : acc.x + acc.y;
    };

    int hl = 0;
    // four hypotheses per iteration: a transposing butterfly leaves the warp totals of hypotheses hl..hl+3 on
    // lanes 0 / 8 / 16 / 24 with 6 shuffles instead of 20
    for (; hl + 4 <= cd.count; hl += 4) {
        const float v0 = one_hyp(hl), v1 = one_hyp(hl + 1), v2 = one_hyp(hl + 2), v3 = one_hyp(hl + 3);
        const bool hi16 = lane & 16, hi8 = lane & 8;
        float k0_ = hi16 ? v2 : v0, k1_ = hi16 ? v3 : v1;   // kept
        float s0_ = hi16 ? v0 : v2, s1_ = hi16 ? v1 : v3;   // sent
        k0_ += __shfl_xor_sync(0xffffffffu, s0_, 16);
        k1_ += __shfl_xor_sync(0xffffffffu, s1_, 16);
        float c = hi8 ? k1_ : k0_;
        const float d = hi8 ? k0_ : k1_;
        c += __shfl_xor_sync(0xffffffffu, d, 8);
        c += __shfl_xor_sync(0xffffffffu, c, 4);
        c += __shfl_xor_sync(0xffffffffu, c, 2);
        c += __shfl_xor_sync(0xffffffffu, c, 1);
        if ((lane & 7) == 0) sWarp[warp][hl + (lane >> 3)] = c;
    }
    for (; hl < cd.count; ++hl) {
        float s = one_hyp(hl);
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) sWarp[warp][hl] = s;
    }
    __syncthreads();
    if (tid < cd.count) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < kScoreThreads / 32; ++w) s += sWarp[w][tid];
        if (FOLD) s *= 1.f / (float)(1ull << kScorePairShift);  // exact
        a.part[(size_t)(cd.slot0 + tid) * a.T + tile] = s;
    }
}

template <int PPT, bool FOLD, bool DEV>
__global__ void __launch_bounds__(kScoreThreads, 2) score_kernel(const __grid_constant__ ScoreArgs a) {
    __shared__ float4 sPose[kMaxChunk * 3];
    __shared__ float sWarp[kScoreThreads / 32][kMaxChunk];
    __shared__ int sItem;
    constexpr int TP = kScoreThreads * PPT;
    const int tid = threadIdx.x;
    const int n_items = *a.n_chunks * a.T;
    const bool ragged = (a.P.N % TP) != 0;
    for (;;) {
        if (tid == 0) sItem = atomicAdd(a.work_counter, 1);
        __syncthreads();
        const int item = sItem;
        if (item >= n_items) break;
        // tiles vary fastest so concurrently running CTAs share a chunk's poses and stream one plane
        const int chunk = item / a.T, tile = item - chunk * a.T;
        const ChunkDesc cd = a.chunks[chunk];
        const float4* src = (const float4*)(a.poses + cd.slot0);
        for (int i = tid; i < cd.count * 3; i += kScoreThreads) sPose[i] = src[i];
        __syncthreads();
        if (ragged && tile == a.T - 1) score_item<PPT, true, FOLD, DEV>(a, cd, tile, sPose, sWarp);
        else score_item<PPT, false, FOLD, DEV>(a, cd, tile, sPose, sWarp);
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------
// TMA-staged variant: the three rows of a pixel tile are brought into shared memory by cp.async.bulk (UBLKCP) copies that
// complete on an mbarrier; while a CTA scores one (chunk, tile) item the copies for its next item are already in
// flight in the other stage.  Needs 16-byte aligned planes and N % 4 == 0 (else score_kernel above is used).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

template <int PPT, bool FOLD, bool DEV>
__global__ void __launch_bounds__(kScoreThreads, 2) score_kernel_tma(const __grid_constant__ ScoreArgs a) {
    constexpr int TP = kScoreThreads * PPT;
    extern __shared__ __align__(128) float sTile[];  // [2 stages][3 rows][TP]
    __shared__ float4 sPose[kMaxChunk * 3];
    __shared__ float sWarp[kScoreThreads / 32][kMaxChunk];
    __shared__ __align__(8) uint64_t sBar[2];
    __shared__ int sItem[2];
    const int tid = threadIdx.x;
    const int n_items = *a.n_chunks * a.T;
    const bool ragged = (a.P.N % TP) != 0;

    auto issue = [&](int item, int stage) {  // thread 0: start the three row copies of `item` into `stage`
        const int chunk = item / a.T, tile = item - chunk * a.T;
        const int e = a.chunks[chunk].expert;
        const int cells = min(TP, a.P.N - tile * TP);
        const uint32_t bytes = (uint32_t)cells * 4u;
        const float* src = a.coords + (size_t)e * 3 * a.P.N + (size_t)tile * TP;
        float* dst = sTile + (size_t)stage * 3 * TP;
        mbar_expect_tx(&sBar[stage], 3u * bytes);
        tma_bulk_g2s(dst, src, bytes, &sBar[stage]);
        tma_bulk_g2s(dst + TP, src + a.P.N, bytes, &sBar[stage]);
        tma_bulk_g2s(dst + 2 * TP, src + 2 * (size_t)a.P.N, bytes, &sBar[stage]);
    };

    if (tid == 0) {
        mbar_init(&sBar[0], 1);
        mbar_init(&sBar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const int first = atomicAdd(a.work_counter, 1);
        sItem[0] = first;
        if (first < n_items) issue(first, 0);
    }
    __syncthreads();
    uint32_t phase[2] = {0u, 0u};
    for (int it = 0;; ++it) {
        const int stage = it & 1;
        const int item = sItem[stage];
        if (item >= n_items) break;
        if (tid == 0) {  // claim the next item and start its copies into the other stage (free since the last barrier)
            const int nxt = atomicAdd(a.work_counter, 1);
            sItem[stage ^ 1] = nxt;
            if (nxt < n_items) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                issue(nxt, stage ^ 1);
            }
        }
        const int chunk = item / a.T, tile = item - chunk * a.T;
        const ChunkDesc cd = a.chunks[chunk];
        const float4* src = (const float4*)(a.poses + cd.slot0);
        for (int i = tid; i < cd.count * 3; i += kScoreThreads) sPose[i] = src[i];
        mbar_wait(&sBar[stage], phase[stage]);
        phase[stage] ^= 1u;
        __syncthreads();
        const float* tx = sTile + (size_t)stage * 3 * TP;
        if (ragged && tile == a.T - 1) score_item<PPT, true, FOLD, DEV>(a, cd, tile, sPose, sWarp, tx, tx + TP, tx + 2 * TP);
        else score_item<PPT, false, FOLD, DEV>(a, cd, tile, sPose, sWarp, tx, tx + TP, tx + 2 * TP);
        __syncthreads();  // everyone is done with this stage, sPose, sWarp and has read sItem[stage ^ 1]'s predecessor
    }
}

int score_tile_pixels(int ppt) { return kScoreThreads * ppt; }

constexpr int kMaxDevices = 64;

template <bool FOLD, bool DEV>
void launch_score_t(const ScoreArgs& a, int ppt, int grid, cudaStream_t st) {
    if (a.vec_ok && ppt >= 4) {  // TMA path (bulk copies need 16-byte granularity)
        const size_t smem = (size_t)2 * 3 * kScoreThreads * ppt * sizeof(float);
        // The opt-in above 48 KB of dynamic shared memory is a per-DEVICE function attribute (one process may hold contexts
        // on several GPUs, api.context(device)), and launches may come from several host threads (backward_batch workers).
        static std::atomic<unsigned char> attr_set[kMaxDevices][2];  // one table per FOLD / DEV instantiation
        int dev = 0;
        cudaGetDevice(&dev);
        const int which = ppt == 8 ? 0 : 1;
        const bool known = dev >= 0 && dev < kMaxDevices;
        if (!known || !attr_set[dev][which].load(std::memory_order_acquire)) {
            if (ppt == 8) cudaFuncSetAttribute(score_kernel_tma<8, FOLD, DEV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            else cudaFuncSetAttribute(score_kernel_tma<4, FOLD, DEV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (known) attr_set[dev][which].store(1, std::memory_order_release);
        }
        if (ppt == 8) score_kernel_tma<8, FOLD, DEV><<<grid, kScoreThreads, smem, st>>>(a);
        else score_kernel_tma<4, FOLD, DEV><<<grid, kScoreThreads, smem, st>>>(a);
        return;
    }
    if (ppt == 8) score_kernel<8, FOLD, DEV><<<grid, kScoreThreads, 0, st>>>(a);
    else if (ppt == 4) score_kernel<4, FOLD, DEV><<<grid, kScoreThreads, 0, st>>>(a);
    else score_kernel<2, FOLD, DEV><<<grid, kScoreThreads, 0, st>>>(a);
}

void launch_score(const ScoreArgs& a, int ppt, int grid, cudaStream_t st) {
    const bool dev = a.dev.shift != nullptr;
    if (a.fold) dev ? launch_score_t<true, true>(a, ppt, grid, st) : launch_score_t<true, false>(a, ppt, grid, st);
    else dev ? launch_score_t<false, true>(a, ppt, grid, st) : launch_score_t<false, false>(a, ppt, grid, st);
}

// ---------------------------------------------------------------------------------------------
// select: finish scores, softMax, entropy, argmax (draw with training=false), contributing list
// ---------------------------------------------------------------------------------------------
// scores[h] = (alpha/W/H) * sum over tiles of the partial soft-inlier sums: one warp per hypothesis, fixed order
__global__ void __launch_bounds__(256) finish_scores_kernel(const float* __restrict__ part, const int* __restrict__ slot_of,
                                                            Problem P, int T, double* scores) {
    const int lane = threadIdx.x & 31;
    const int h = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (h >= P.M) return;
    // getHypScores' final factor is a float expression: alpha / cols / rows (esac_util.h:256)
    const float facf = P.alpha / (float)P.W / (float)P.H;
    const float* row = part + (size_t)slot_of[h] * T;
    double s = 0;
    for (int t = lane; t < T; t += 32) s += (double)row[t];
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) scores[h] = s * (double)facf;
}

__global__ void __launch_bounds__(1024) select_kernel(const float* __restrict__ part, const int* __restrict__ slot_of,
                                                      Problem P, int T, double* scores, double* probs, double* stats,
                                                      int* winner, int* contrib, int* n_contrib) {
    __shared__ double sred[32];
    __shared__ int sidx[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    (void)part; (void)slot_of; (void)T;
    // max
    double mx = -1e300;
    for (int h = tid; h < P.M; h += blockDim.x) mx = fmax(mx, scores[h]);
    for (int o = 16; o; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) sred[warp] = mx;
    __syncthreads();
    mx = sred[0];
    for (int w = 1; w < nw; ++w) mx = fmax(mx, sred[w]);
    __syncthreads();
    double sum = 0;
    for (int h = tid; h < P.M; h += blockDim.x) {
        double e = exp(scores[h] - mx);
        probs[h] = e;
        sum += e;
    }
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) sred[warp] = sum;
    __syncthreads();
    sum = 0;
    for (int w = 0; w < nw; ++w) sum += sred[w];
    __syncthreads();
    double ent = 0, best = -1;
    int bi = 0x7fffffff;
    for (int h = tid; h < P.M; h += blockDim.x) {
        double p = probs[h] / sum;
        probs[h] = p;
        if (p > 0) ent -= p * log2(p);
        if (!(p < kEps) && (p > best)) { best = p; bi = h; }  // first strict maximum: ascending h per thread
    }
    for (int o = 16; o; o >>= 1) {
        ent += __shfl_xor_sync(0xffffffffu, ent, o);
        double ob = __shfl_xor_sync(0xffffffffu, best, o);
        int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (lane == 0) { sred[warp] = best; sidx[warp] = bi; }
    __syncthreads();
    __shared__ double sent[32];
    if (lane == 0) sent[warp] = ent;
    __syncthreads();
    __shared__ int swc[32];
    __shared__ int srun;
    if (tid == 0) {
        double b = -1; int i = 0x7fffffff; double en = 0;
        for (int w = 0; w < nw; ++w) {
            en += sent[w];
            if (sred[w] > b || (sred[w] == b && sidx[w] < i)) { b = sred[w]; i = sidx[w]; }
        }
        if (i == 0x7fffffff) i = 0;
        *winner = i;
        stats[0] = en; stats[1] = (double)i;
        stats[5] = mx; stats[6] = sum;  // local softmax normalisation, for the multi-GPU exchange
        srun = 0;
    }
    __syncthreads();
    // ordered compaction of the hypotheses with p >= PROB_THRESH (esac.cpp:334, esac_derivative.h:231)
    for (int b = 0; b < P.M; b += blockDim.x) {
        const int h = b + tid;
        const bool flag = h < P.M && !(probs[h] < kProbThresh);
        const unsigned m = __ballot_sync(0xffffffffu, flag);
        if (lane == 0) swc[warp] = __popc(m);
        __syncthreads();
        int off = srun;
        for (int w = 0; w < warp; ++w) off += swc[w];
        if (flag) contrib[off + __popc(m & ((1u << lane) - 1u))] = h;
        __syncthreads();
        if (tid == 0) { int t = 0; for (int w = 0; w < nw; ++w) t += swc[w]; srun += t; }
        __syncthreads();
    }
    if (tid == 0) { *n_contrib = srun; stats[2] = (double)srun; }
}

void launch_select(const float* part, const int* slot_of, const Problem& P, int T, double* scores, double* probs,
                   double* stats, int* winner, int* contrib, int* n_contrib, cudaStream_t st) {
    finish_scores_kernel<<<(P.M * 32 + 255) / 256, 256, 0, st>>>(part, slot_of, P, T, scores);
    select_kernel<<<1, 1024, 0, st>>>(part, slot_of, P, T, scores, probs, stats, winner, contrib, n_contrib);
}


// Multi-GPU backward: hypothesis probabilities w.r.t. the GLOBAL softmax normalisation (max and sum of exp over all
// ranks, exchanged by the host), and the ordered list of contributing hypotheses rebuilt from them.
__global__ void __launch_bounds__(1024) rescale_probs_kernel(const double* __restrict__ scores, Problem P, double gmax, double gsum,
                                                             double* probs, int* contrib, int* n_contrib) {
    __shared__ int swc[32];
    __shared__ int srun;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    if (tid == 0) srun = 0;
    __syncthreads();
    for (int b = 0; b < P.M; b += blockDim.x) {
        const int h = b + tid;
        bool flag = false;
        if (h < P.M) {
            const double p = exp(scores[h] - gmax) / gsum;
            probs[h] = p;
            flag = !(p < kProbThresh);
        }
        const unsigned m = __ballot_sync(0xffffffffu, flag);
        if (lane == 0) swc[warp] = __popc(m);
        __syncthreads();
        int off = srun;
        for (int w = 0; w < warp; ++w) off += swc[w];
        if (flag) contrib[off + __popc(m & ((1u << lane) - 1u))] = h;
        __syncthreads();
        if (tid == 0) { int t = 0; for (int w = 0; w < nw; ++w) t += swc[w]; srun += t; }
        __syncthreads();
    }
    if (tid == 0) *n_contrib = srun;
}

void launch_rescale_probs(const double* scores, const Problem& P, double gmax, double gsum, double* probs, int* contrib,
                          int* n_contrib, cudaStream_t st) {
    rescale_probs_kernel<<<1, 1024, 0, st>>>(scores, P, gmax, gsum, probs, contrib, n_contrib);
}

// The same with the normalisation merged on the device from the all-gathered (max, sum exp(score - max)) pairs of all ranks
// (no host round trip): gmax = max_r m_r, gsum = sum_r s_r exp(m_r - gmax), in rank order.  norm_out[0..1] = (gmax, gsum).
__global__ void __launch_bounds__(1024) rescale_probs_gathered_kernel(const double* __restrict__ scores, Problem P,
                                                                      const double* __restrict__ pairs, int world, double* norm_out,
                                                                      double* probs, int* contrib, int* n_contrib) {
    __shared__ int swc[32];
    __shared__ int srun;
    __shared__ double snorm[2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    if (tid == 0) {
        srun = 0;
        double gmax = -1e300;
        for (int r = 0; r < world; ++r) gmax = fmax(gmax, pairs[2 * r]);
        double gsum = 0;
        for (int r = 0; r < world; ++r) gsum += pairs[2 * r + 1] * exp(pairs[2 * r] - gmax);
        snorm[0] = gmax; snorm[1] = gsum;
        if (norm_out) { norm_out[0] = gmax; norm_out[1] = gsum; }
    }
    __syncthreads();
    const double gmax = snorm[0], gsum = snorm[1];
    for (int b = 0; b < P.M; b += blockDim.x) {
        const int h = b + tid;
        bool flag = false;
        if (h < P.M) {
            const double p = exp(scores[h] - gmax) / gsum;
            probs[h] = p;
            flag = !(p < kProbThresh);
        }
        const unsigned m = __ballot_sync(0xffffffffu, flag);
        if (lane == 0) swc[warp] = __popc(m);
        __syncthreads();
        int off = srun;
        for (int w = 0; w < warp; ++w) off += swc[w];
        if (flag) contrib[off + __popc(m & ((1u << lane) - 1u))] = h;
        __syncthreads();
        if (tid == 0) { int t = 0; for (int w = 0; w < nw; ++w) t += swc[w]; srun += t; }
        __syncthreads();
    }
    if (tid == 0) *n_contrib = srun;
}

void launch_rescale_probs_gathered(const double* scores, const Problem& P, const double* pairs, int world, double* norm_out,
                                   double* probs, int* contrib, int* n_contrib, cudaStream_t st) {
    rescale_probs_gathered_kernel<<<1, 1024, 0, st>>>(scores, P, pairs, world, norm_out, probs, contrib, n_contrib);
}

}  // namespace esacb200
