// Clustering a large environment into experts on the device (cluster_dataset.py:19-140, 219-240): the per-image
// statistics of the ground-truth maps, one 2-means split with k-means++ seeding and several attempts, and the cluster
// centres, sizes and soft gating targets of a finished clustering.  Every sum runs in a fixed order, so every result is
// bitwise repeatable; oracle/cluster_oracle.py restates the k-means reduction tree exactly.
#include <float.h>
#include <limits.h>

#include "esac_internal.h"
#include "esac_rng.cuh"

namespace esacb200 {

namespace {

// ---- per-image statistics ------------------------------------------------------------------------------------------

// A cell has ground truth when its float32 sum (x + y) + z, summed left to right as torch's sum(0), is not 0.
__device__ __forceinline__ bool valid_cell(float x, float y, float z) { return __fadd_rn(__fadd_rn(x, y), z) != 0.f; }

// The order-preserving integer image of a float: unsigned order of keys = numeric order of non-NaN floats (-0 < +0).
__device__ __forceinline__ unsigned float_key(float f) {
    const unsigned u = __float_as_uint(f);
    return u ^ ((unsigned)((int)u >> 31) | 0x80000000u);
}
__device__ __forceinline__ float key_float(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k ^ 0x80000000u) : ~k);
}

// One digit pass of the radix select: the 256-bin histogram is complete; warp 0 finds the bin that holds rank `rank`,
// appends it to the prefix and leaves the rank within that bin.
__device__ __forceinline__ void radix_pick(const unsigned* hist, int shift, unsigned& s_prefix, unsigned& s_rank) {
    const int lane = threadIdx.x;
    unsigned h[8], sum = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        h[q] = hist[lane * 8 + q];
        sum += h[q];
    }
    unsigned incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    const unsigned rank = s_rank;
    const unsigned hit = __ballot_sync(0xffffffffu, incl > rank);
    if (lane == __ffs(hit) - 1) {
        unsigned r = rank - (incl - sum);
        int bin = 0;
        bool found = false;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            if (!found) {
                if (h[q] > r) {
                    bin = q;
                    found = true;
                } else {
                    r -= h[q];
                }
            }
        }
        s_prefix |= (unsigned)(lane * 8 + bin) << shift;
        s_rank = r;
    }
}

// One CTA per map.  Pass 1 counts the valid cells, sums them in fp64 (each thread over a fixed stride, then a fixed tree),
// notes each coordinate's first NaN and copies the valid cells' keys to shared memory while they fit.  Each coordinate's
// lower median (torch.median: sorted[(n-1)/2], the first NaN when there is one) is then a 4-digit radix select over the
// keys in shared memory, or, for a map whose valid cells do not fit, over the map in global memory.
__global__ void __launch_bounds__(kStatsThreads) cluster_stats_kernel(const ClusterMap* __restrict__ maps, int cap,
                                                                     ClusterStats* __restrict__ out) {
    extern __shared__ unsigned keys[];
    __shared__ unsigned hist[256];
    __shared__ double red[3][kStatsThreads];
    __shared__ int cnt_red[kStatsThreads];
    __shared__ int s_pos, s_nan[3];
    __shared__ unsigned s_prefix, s_rank;
    __shared__ float s_med[3];
    const ClusterMap m = maps[blockIdx.x];
    const int n = m.H * m.W;
    const int t = threadIdx.x;
    const float* __restrict__ p = m.p;
    if (t == 0) {
        s_pos = 0;
        s_nan[0] = s_nan[1] = s_nan[2] = INT_MAX;
    }
    __syncthreads();
    double acc[3] = {0., 0., 0.};
    int cnt = 0;
    for (int i = t; i < n; i += kStatsThreads) {
        const float v[3] = {p[i], p[(size_t)n + i], p[2 * (size_t)n + i]};
        if (!valid_cell(v[0], v[1], v[2])) continue;
        ++cnt;
        const int pos = atomicAdd(&s_pos, 1);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            acc[c] += (double)v[c];
            if (v[c] != v[c]) atomicMin(&s_nan[c], i);
            if (pos < cap) keys[c * cap + pos] = float_key(v[c]);
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) red[c][t] = acc[c];
    cnt_red[t] = cnt;
    __syncthreads();
    for (int s = kStatsThreads / 2; s > 0; s >>= 1) {
        if (t < s) {
#pragma unroll
            for (int c = 0; c < 3; ++c) red[c][t] += red[c][t + s];
            cnt_red[t] += cnt_red[t + s];
        }
        __syncthreads();
    }
    const int total = cnt_red[0];
    const float qnan = __uint_as_float(0x7fc00000u);
    for (int c = 0; c < 3; ++c) {
        if (total == 0 || s_nan[c] != INT_MAX) {
            if (t == 0) s_med[c] = total == 0 ? qnan : p[(size_t)c * n + s_nan[c]];
            continue;
        }
        if (t == 0) {
            s_prefix = 0;
            s_rank = (unsigned)(total - 1) / 2;
        }
        unsigned mask = 0;
        for (int shift = 24; shift >= 0; shift -= 8) {
            for (int j = t; j < 256; j += kStatsThreads) hist[j] = 0;
            __syncthreads();
            const unsigned prefix = s_prefix;
            if (total <= cap) {
                const unsigned* kc = keys + c * cap;
                for (int j = t; j < total; j += kStatsThreads) {
                    const unsigned k = kc[j];
                    if ((k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1u);
                }
            } else {
                for (int i = t; i < n; i += kStatsThreads) {
                    const float x = p[i], y = p[(size_t)n + i], z = p[2 * (size_t)n + i];
                    if (!valid_cell(x, y, z)) continue;
                    const unsigned k = float_key(c == 0 ? x : (c == 1 ? y : z));
                    if ((k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1u);
                }
            }
            __syncthreads();
            if (t < 32) radix_pick(hist, shift, s_prefix, s_rank);
            __syncthreads();
            mask |= 255u << shift;
        }
        if (t == 0) s_med[c] = key_float(s_prefix);
        __syncthreads();
    }
    if (t == 0) {
        ClusterStats o;
        o.count = total;
        bool finite = total > 0;
        for (int c = 0; c < 3; ++c) {
            o.median[c] = s_med[c];
            o.mean[c] = total > 0 ? __double2float_rn(red[c][0] / (double)total) : qnan;
            finite = finite && isfinite(o.median[c]) && isfinite(o.mean[c]);
        }
        o.status = total == 0 ? 1 : (finite ? 0 : 2);
        out[blockIdx.x] = o;
    }
}

// ---- 2-means ---------------------------------------------------------------------------------------------------------

constexpr int kKT = kKmeansThreads;

struct Pt {
    double x, y, z;
};

// Points are read through L2 (ld.global.cg): every pass streams them once, and several CTAs read the same points.
__device__ __forceinline__ Pt load_point(const float* __restrict__ p, int i) {
    return {(double)__ldcg(p + 3 * (size_t)i), (double)__ldcg(p + 3 * (size_t)i + 1), (double)__ldcg(p + 3 * (size_t)i + 2)};
}

// Squared distance in fp64, ((dx*dx + dy*dy) + dz*dz) with no contraction, as the oracle computes it.
__device__ __forceinline__ double dist2(const Pt& a, const double* c) {
    const double dx = __dsub_rn(a.x, c[0]), dy = __dsub_rn(a.y, c[1]), dz = __dsub_rn(a.z, c[2]);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// Draw `draw` of attempt `attempt` of split `split`: the repository's counter-based stream (esac_rng.cuh).
__device__ __forceinline__ uint64_t kmeans_draw(uint64_t seed, unsigned split, unsigned attempt, unsigned draw) {
    uint64_t s = mix64(seed + kGold * (uint64_t)(split + 1u));
    s = mix64(s + kGold * (uint64_t)(attempt + 1u));
    return mix64(s + kGold * (uint64_t)(draw + 1u));
}

// The fixed reduction of every k-means sum: thread t adds its contiguous chunk [lo, hi) in index order (its partial, in
// red[q][t]), then red[q][t] += red[q][t + s] for s = T/2 .. 1.  The total lands in red[q][0].
template <int NV>
__device__ __forceinline__ void tree_sum(double (*red)[kKT]) {
    __syncthreads();
    for (int s = kKT / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) {
#pragma unroll
            for (int q = 0; q < NV; ++q) red[q][threadIdx.x] = __dadd_rn(red[q][threadIdx.x], red[q][threadIdx.x + s]);
        }
        __syncthreads();
    }
}

struct KmeansShared {
    double red[8][kKT];
    double pre[kKT + 1];
    double c[2][3];
    double far_d[kKT];
    int far_i[kKT];
    int ci;
};

// Label of a point for centres c: the nearer centre, centre 0 on a tie; the reseeded point takes its new cluster.
__device__ __forceinline__ int nearest(const Pt& P, const double (*c)[3], int i, int reseed, int reseed_label, double& d) {
    const double d0 = dist2(P, c[0]), d1 = dist2(P, c[1]);
    const int lab = i == reseed ? reseed_label : (d1 < d0 ? 1 : 0);
    d = lab ? d1 : d0;
    return lab;
}

// Assigns every point to the current centres and sums, per cluster, its points and their count, and the compactness.
// red[0..5]: the two clusters' coordinate sums, red[6]: compactness, red[7]: points in cluster 1.
__device__ void kmeans_pass(const KmeansArgs& a, KmeansShared& sh, int lo, int hi, int reseed, int reseed_label) {
    double s[2][3] = {{0., 0., 0.}, {0., 0., 0.}}, comp = 0.;
    int n1 = 0;
    for (int i = lo; i < hi; ++i) {
        const Pt P = load_point(a.points, i);
        double d;
        const int lab = nearest(P, sh.c, i, reseed, reseed_label, d);
        comp = __dadd_rn(comp, d);
        if (lab) {
            s[1][0] = __dadd_rn(s[1][0], P.x), s[1][1] = __dadd_rn(s[1][1], P.y), s[1][2] = __dadd_rn(s[1][2], P.z);
            ++n1;
        } else {
            s[0][0] = __dadd_rn(s[0][0], P.x), s[0][1] = __dadd_rn(s[0][1], P.y), s[0][2] = __dadd_rn(s[0][2], P.z);
        }
    }
    const int t = threadIdx.x;
#pragma unroll
    for (int q = 0; q < 6; ++q) sh.red[q][t] = s[q / 3][q % 3];
    sh.red[6][t] = comp;
    sh.red[7][t] = (double)n1;
    tree_sum<8>(sh.red);
}

// The point farthest from centre j, lowest index on ties.
__device__ int farthest(const KmeansArgs& a, KmeansShared& sh, int lo, int hi, int j) {
    double best = -1.;
    int bi = INT_MAX;
    for (int i = lo; i < hi; ++i) {
        const double d = dist2(load_point(a.points, i), sh.c[j]);
        if (d > best) best = d, bi = i;
    }
    const int t = threadIdx.x;
    sh.far_d[t] = best;
    sh.far_i[t] = bi;
    __syncthreads();
    for (int s = kKT / 2; s > 0; s >>= 1) {
        if (t < s) {
            const double d = sh.far_d[t + s];
            const int i = sh.far_i[t + s];
            if (d > sh.far_d[t] || (d == sh.far_d[t] && i < sh.far_i[t])) sh.far_d[t] = d, sh.far_i[t] = i;
        }
        __syncthreads();
    }
    return sh.far_i[0];
}

// An assignment to the current centres; when it leaves a cluster empty, the point farthest from the other centre moves
// there and the sums are taken again.
__device__ void kmeans_assign(const KmeansArgs& a, KmeansShared& sh, int lo, int hi, int& reseed, int& reseed_label) {
    reseed = -1;
    reseed_label = 0;
    kmeans_pass(a, sh, lo, hi, -1, 0);
    const int n1 = (int)sh.red[7][0];
    if (n1 == 0 || n1 == a.n) {
        reseed_label = n1 == 0 ? 1 : 0;
        __syncthreads();
        reseed = farthest(a, sh, lo, hi, 1 - reseed_label);
        kmeans_pass(a, sh, lo, hi, reseed, reseed_label);
    }
}

// One attempt per CTA: k-means++ seeding with 3 trials (OpenCV's generateCentersPP), then Lloyd iterations.
__global__ void __launch_bounds__(kKT, 1) kmeans2_kernel(const __grid_constant__ KmeansArgs a) {
    __shared__ KmeansShared sh;
    const int t = threadIdx.x, n = a.n;
    const unsigned att = blockIdx.x;
    const int chunk = (n + kKT - 1) / kKT;
    const int lo = min(n, t * chunk), hi = min(n, lo + chunk);
    // first centre: the point at floor(u * n)
    const uint64_t r0 = kmeans_draw(a.seed, a.split, att, 0);
    const int i0 = (int)(((r0 >> 32) * (uint64_t)n) >> 32);
    const Pt c0 = load_point(a.points, i0);
    const double cc0[3] = {c0.x, c0.y, c0.z};
    double part = 0.;
    for (int i = lo; i < hi; ++i) part = __dadd_rn(part, dist2(load_point(a.points, i), cc0));
    sh.red[0][t] = part;
    __syncthreads();
    if (t == 0) {
        sh.pre[0] = 0.;
        for (int q = 0; q < kKT; ++q) sh.pre[q + 1] = __dadd_rn(sh.pre[q], sh.red[0][q]);
    }
    tree_sum<1>(sh.red);
    const double sum0 = sh.red[0][0];
    // second centre: of 3 candidates drawn with probability proportional to the squared distance, the one with the lower
    // potential (the first on a tie)
    double best = DBL_MAX;
    int best_i = 0;
    for (unsigned trial = 0; trial < 3; ++trial) {
        const uint64_t r = kmeans_draw(a.seed, a.split, att, 1 + trial);
        const double p = __dmul_rn((double)(r >> 11) * 0x1.0p-53, sum0);
        __syncthreads();
        if (t == 0) sh.ci = n - 1;
        __syncthreads();
        if (lo < hi && sh.pre[t + 1] >= p) {
            double run = 0.;
            for (int i = lo; i < hi; ++i) {
                run = __dadd_rn(run, dist2(load_point(a.points, i), cc0));
                if (__dadd_rn(sh.pre[t], run) >= p) {
                    atomicMin(&sh.ci, i);
                    break;
                }
            }
        }
        __syncthreads();
        const int ci = sh.ci;
        const Pt cand = load_point(a.points, ci);
        const double cc[3] = {cand.x, cand.y, cand.z};
        double pot = 0.;
        for (int i = lo; i < hi; ++i) {
            const Pt P = load_point(a.points, i);
            pot = __dadd_rn(pot, fmin(dist2(P, cc0), dist2(P, cc)));
        }
        sh.red[0][t] = pot;
        tree_sum<1>(sh.red);
        if (sh.red[0][0] < best) best = sh.red[0][0], best_i = ci;
    }
    if (t == 0) {
        const Pt c1 = load_point(a.points, best_i);
        sh.c[0][0] = c0.x, sh.c[0][1] = c0.y, sh.c[0][2] = c0.z;
        sh.c[1][0] = c1.x, sh.c[1][1] = c1.y, sh.c[1][2] = c1.z;
    }
    __syncthreads();
    // Lloyd: assign, move each centre to its points' mean, stop after max_iter or once no centre moved more than eps
    int reseed, reseed_label;
    for (int it = 0; it < a.max_iter; ++it) {
        kmeans_assign(a, sh, lo, hi, reseed, reseed_label);
        const double n1 = sh.red[7][0], cnt[2] = {(double)n - n1, n1};
        double nc[2][3], shift = 0.;
        for (int k = 0; k < 2; ++k) {
            for (int c = 0; c < 3; ++c) nc[k][c] = __ddiv_rn(sh.red[k * 3 + c][0], cnt[k]);
            const Pt q = {nc[k][0], nc[k][1], nc[k][2]};
            shift = fmax(shift, dist2(q, sh.c[k]));
        }
        __syncthreads();
        if (t == 0)
            for (int k = 0; k < 2; ++k)
                for (int c = 0; c < 3; ++c) sh.c[k][c] = nc[k][c];
        __syncthreads();
        if (shift <= a.eps2) break;
    }
    kmeans_assign(a, sh, lo, hi, reseed, reseed_label);
    if (t == 0) {
        KmeansAttempt& o = a.att[att];
        for (int k = 0; k < 2; ++k)
            for (int c = 0; c < 3; ++c) o.centre[k][c] = sh.c[k][c];
        o.compactness = sh.red[6][0];
        o.reseed = reseed;
        o.reseed_label = reseed_label;
    }
}

// The best attempt (lowest compactness, lowest index on a tie): its labels, float32 centres and compactness.
__global__ void __launch_bounds__(kKT) kmeans_pick_kernel(const __grid_constant__ KmeansArgs a) {
    int b = 0;
    for (int q = 1; q < a.attempts; ++q)
        if (a.att[q].compactness < a.att[b].compactness) b = q;
    const KmeansAttempt& A = a.att[b];
    const int i = blockIdx.x * kKT + threadIdx.x;
    if (i < a.n) {
        double d;
        a.labels[i] = nearest(load_point(a.points, i), A.centre, i, A.reseed, A.reseed_label, d);
    }
    if (i == 0) {
        for (int k = 0; k < 2; ++k)
            for (int c = 0; c < 3; ++c) a.centres[k * 3 + c] = __double2float_rn(A.centre[k][c]);
        *a.compactness = A.compactness;
    }
}

// ---- cluster centres, sizes and gating targets ---------------------------------------------------------------------

constexpr int kTargetsThreads = 1024;

// cluster_dataset.py:230-237 in its float32 op order: d = |m - c|, d^2 / size / 2, exp(-(.) * softness) / sqrt(2 pi size).
__device__ __forceinline__ float target_term(const float* m, const float* c, float size, float softness) {
    const float dx = __fsub_rn(m[0], c[0]), dy = __fsub_rn(m[1], c[1]), dz = __fsub_rn(m[2], c[2]);
    const float d = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
    float v = __fdiv_rn(__fdiv_rn(__fmul_rn(d, d), size), 2.f);
    const float e = expf(__fmul_rn(-v, softness));
    return __fdiv_rn(e, sqrtf(__fmul_rn(6.28318548f, size)));  // 2 * math.pi * size: the scalar rounds to float32
}

// One CTA: warp w sums clusters w, w + 32, ... (each lane over a fixed contiguous chunk of images, then a fixed shuffle
// tree): the centre is the fp64 mean of its images' means, the size the fp64 mean squared distance of those means to the
// float32 centre; then every image's K targets, normalised by their float32 sum + 1e-7.
__global__ void __launch_bounds__(kTargetsThreads) cluster_targets_kernel(const __grid_constant__ ClusterTargetsArgs a) {
    __shared__ float sc[kTargetsMaxClusters][3];
    __shared__ float ss[kTargetsMaxClusters];
    const int t = threadIdx.x, w = t >> 5, lane = t & 31, N = a.N;
    const int chunk = (N + 31) / 32;
    const int lo = min(N, lane * chunk), hi = min(N, lo + chunk);
    for (int k = w; k < a.K; k += kTargetsThreads / 32) {
        double s[3] = {0., 0., 0.}, q = 0.;
        int cnt = 0;
        for (int i = lo; i < hi; ++i) {
            if (a.labels[i] != k) continue;
            for (int c = 0; c < 3; ++c) s[c] = __dadd_rn(s[c], (double)a.means[3 * (size_t)i + c]);
            ++cnt;
        }
        for (int o = 16; o > 0; o >>= 1) {
            for (int c = 0; c < 3; ++c) s[c] = __dadd_rn(s[c], __shfl_down_sync(0xffffffffu, s[c], o));
            cnt += __shfl_down_sync(0xffffffffu, cnt, o);
        }
        cnt = __shfl_sync(0xffffffffu, cnt, 0);
        if (lane == 0)
            for (int c = 0; c < 3; ++c) sc[k][c] = __double2float_rn(__ddiv_rn(s[c], (double)cnt));
        __syncwarp();
        const double ck[3] = {(double)sc[k][0], (double)sc[k][1], (double)sc[k][2]};
        for (int i = lo; i < hi; ++i) {
            if (a.labels[i] != k) continue;
            const Pt P = {(double)a.means[3 * (size_t)i], (double)a.means[3 * (size_t)i + 1], (double)a.means[3 * (size_t)i + 2]};
            q = __dadd_rn(q, dist2(P, ck));
        }
        for (int o = 16; o > 0; o >>= 1) q = __dadd_rn(q, __shfl_down_sync(0xffffffffu, q, o));
        if (lane == 0) ss[k] = __double2float_rn(__ddiv_rn(q, (double)cnt));
        __syncwarp();
    }
    __syncthreads();
    for (int k = t; k < a.K; k += kTargetsThreads) {
        for (int c = 0; c < 3; ++c) a.centres[3 * (size_t)k + c] = sc[k][c];
        a.sizes[k] = ss[k];
    }
    for (int i = t; i < N; i += kTargetsThreads) {
        const float m[3] = {a.means[3 * (size_t)i], a.means[3 * (size_t)i + 1], a.means[3 * (size_t)i + 2]};
        float sum = 0.f;
        for (int k = 0; k < a.K; ++k) sum = __fadd_rn(sum, target_term(m, sc[k], ss[k], a.softness));
        const float norm = __fadd_rn(sum, 1e-7f);
        for (int k = 0; k < a.K; ++k) a.probs[(size_t)i * a.K + k] = __fdiv_rn(target_term(m, sc[k], ss[k], a.softness), norm);
    }
}

}  // namespace

void launch_cluster_stats(const ClusterMap* maps, int B, int cap, ClusterStats* out, cudaStream_t st) {
    const size_t smem = (size_t)3 * cap * sizeof(unsigned);
    cudaFuncSetAttribute(cluster_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cluster_stats_kernel<<<B, kStatsThreads, smem, st>>>(maps, cap, out);
}

void launch_kmeans2(const KmeansArgs& a, cudaStream_t st) {
    kmeans2_kernel<<<a.attempts, kKT, 0, st>>>(a);
    kmeans_pick_kernel<<<(a.n + kKT - 1) / kKT, kKT, 0, st>>>(a);
}

void launch_cluster_targets(const ClusterTargetsArgs& a, cudaStream_t st) {
    cluster_targets_kernel<<<1, kTargetsThreads, 0, st>>>(a);
}

}  // namespace esacb200
