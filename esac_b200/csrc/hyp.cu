// Hypothesis sampling: minimal sets -> P3P -> 4-point gate.
//
// Replaces sampleHypotheses (esac_util.h:129-225, called from esac.cpp:112 / 276).  The reference loops tries
// sequentially per hypothesis under `omp parallel for`; the counter-based stream (esac_rng.cuh) makes every try
// addressable, so tries are evaluated in bulk and the LOWEST passing try of each hypothesis is kept -- exactly the
// try the sequential loop would have stopped at.  Wrong experts need ~1/P(4th point lands within tau) ~ 1e3 tries
// per hypothesis, which makes this the most expensive stage of a step; it runs as waves of small kernels:
//
//   wave r (try window [base_h, base_h + span_r) of every unresolved hypothesis; span_0 = 256, then chosen on the
//   device from the acceptance rate seen so far, ~1.25 / p, so that ~70% of the remaining hypotheses resolve per
//   wave and < 2x the necessary tries are evaluated):
//     prefilter_kernel   two tries per thread (float2 pairs), fp32 only, branch-free: discards tries whose
//                        every P3P root misses the 4th point by > 2 tau (>96% on wrong experts); the gathers of a
//                        CTA's next 256-try item are in flight under the math of the current one; survivors are
//                        appended to a global list
//     exact_kernel       one thread per survivor: the fp64 path (p3p_pose + minimal_set_gate) whose verdict is the
//                        only one that counts (it leaves early when no P3P candidate can pass, and polishes only the
//                        candidate far ahead on the 4th point); atomicMin keeps the lowest accepted try per hypothesis
//     (advance)          the last CTA of exact_kernel marks resolved hypotheses, advances the window of the others and
//                        rebuilds the work list
//   tail_kernel          CTA per still-unresolved hypothesis: same two phases inside one CTA up to max_tries
//   emit_kernel          one thread per hypothesis: re-derives the winning (or, when exhausted, the last) try and
//                        writes pose / cells / try count
//
// Keeping the float and double paths in different kernels matters: fused, the kernel stalls on instruction fetch.
#include "esac_internal.h"
#include "esac_p3p_fast.cuh"
#include "esac_rng.cuh"

#include <type_traits>

namespace esacb200 {

constexpr int kTryThreads = 128;
constexpr int kNoTry = 0x7fffffff;
constexpr unsigned long long kNoKey = ~0ull;   // best[h]: (try << 32) | staging slot
constexpr unsigned kNoSlot = 0xffffffffu;

struct SampleArgs {
    const float4* coords4;  // [E][N] interleaved (x, y, z, -) copy of the coordinate planes: one 16-byte sector per gathered cell
    const int* assign32;
    Problem P;
    uint64_t seed;
    int limit;            // tries allowed per hypothesis
    const int* injected;  // [M][inj_T][4][2] or null
    int inj_T;
    int use_prefilter;    // 0: every try goes to the exact path (self-check of the prefilter)
    int hyp_offset;       // global index of local hypothesis h = hyp_offset + h * hyp_stride (multi-GPU shards draw the stream of
    int hyp_stride;       // the unsharded problem; stride > 1: hypotheses dealt round-robin to the ranks)
    int h_first, h_step, Mg;  // this lane's hypotheses: h_first + k * h_step, k < Mg ...
    const int* perm;          // ... or, when set, the hypotheses of experts [e_lo, e_hi): perm[offsets[e_lo] + k]
    const int* offsets;
    int e_lo, e_hi;
    int span0;                // window of the first wave (tries per hypothesis)
    float window;             // later windows: window / (acceptance rate per try seen in the last wave)
    float tail_boost;         // ... times this once <= 64 hypotheses are left (twice this for <= 8)
    SampleState st;
    unsigned long long* trace;  // diagnostics (option sample_trace): [slot][2] first CTA start / last CTA end, globaltimer ns
    int trace_slot;
};
// The DEV kernels' arguments: the seed, shift and camera come from device memory (the eager kernels keep SampleArgs as is).
struct SampleArgsDev : SampleArgs {
    DevParams dev;
};
template <bool DEV>
using SampleArgsT = std::conditional_t<DEV, SampleArgsDev, SampleArgs>;

// The seed of the draws: the argument, or (DEV) what call_seed gives the (seed[1] + index)-th call after set_seed.
template <bool DEV>
__device__ __forceinline__ uint64_t sample_seed(const SampleArgsT<DEV>& a) {
    if constexpr (DEV) {
        const uint64_t base = __ldg(a.dev.seed), calls = __ldg(a.dev.seed + 1) + (uint64_t)a.dev.index;
        if (calls == 0 || a.dev.fixed_seed) return base;
        return mix64(base + kGold * calls);
    } else {
        return a.seed;
    }
}

__device__ __forceinline__ unsigned long long gtime() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
struct TraceScope {  // thread 0 of every CTA stamps its kernel's slot
    unsigned long long* p;
    __device__ TraceScope(const unsigned long long* base, int slot) : p(nullptr) {
        if (base && threadIdx.x == 0) { p = const_cast<unsigned long long*>(base) + 2 * slot; atomicMin(p, gtime()); }
    }
    __device__ ~TraceScope() { if (p) atomicMax(p + 1, gtime()); }
};

// k-th hypothesis of the lane and the lane's size
__device__ __forceinline__ int lane_size(const SampleArgs& a) {
    return a.perm ? a.offsets[a.e_hi] - a.offsets[a.e_lo] : a.Mg;
}
__device__ __forceinline__ int lane_hyp(const SampleArgs& a, int k) {
    return a.perm ? a.perm[a.offsets[a.e_lo] + k] : a.h_first + k * a.h_step;
}

template <bool DEV>
__device__ __forceinline__ void load_try(const SampleArgsT<DEV>& a, int h, int t, int cx[4], int cy[4], float obj[4][3], float img[4][2]) {
    const Problem& P = a.P;
    if (a.injected) {
        const int* c = a.injected + ((size_t)h * a.inj_T + t) * 8;
        for (int j = 0; j < 4; ++j) { cx[j] = c[2 * j]; cy[j] = c[2 * j + 1]; }
    } else {
        draw_minimal_set(sample_seed<DEV>(a), (uint32_t)(h * a.hyp_stride + a.hyp_offset), (uint32_t)t, P.W, P.H, cx, cy);
    }
    const float4* pl = a.coords4 + (size_t)a.assign32[h] * P.N;
    for (int j = 0; j < 4; ++j) {
        const int p = cy[j] * P.W + cx[j];
        const float4 v = __ldg(pl + p);
        obj[j][0] = v.x; obj[j][1] = v.y; obj[j][2] = v.z;
        img[j][0] = (float)(cx[j] * P.sub + P.sub / 2 - dev_shift_x<DEV>(P, a));
        img[j][1] = (float)(cy[j] * P.sub + P.sub / 2 - dev_shift_y<DEV>(P, a));
    }
}

// verdict_only: the caller wants accept / reject and nothing else, so a try none of whose P3P candidates brings the 4th
// point within 1.25 tau + 1 px (measured on the unpolished depths) is rejected before polish / alignment / Rodrigues / gate --
// that is ~60 % of what survives the float prefilter's 2 tau band.  `solved` and `pose` are then meaningless; emit_kernel,
// which needs the failure state of an exhausted hypothesis' last try, calls with verdict_only = false.
template <bool DEV>
__device__ __noinline__ bool exact_try(const SampleArgsT<DEV>& a, int h, int t, Pose& pose, int cx[4], int cy[4], bool& solved,
                                       bool verdict_only = false) {
    float obj[4][3], img[4][2];
    load_try<DEV>(a, h, t, cx, cy, obj, img);
    if constexpr (DEV) {
        const double f = (double)dev_f<DEV>(a.P, a), ppx = (double)dev_ppx<DEV>(a.P, a), ppy = (double)dev_ppy<DEV>(a.P, a);
        solved = p3p_pose(obj, img, f, ppx, ppy, pose, verdict_only ? 1.25 * (double)a.P.tau + 1. : 0.);
        return solved && minimal_set_gate(obj, img, pose, f, ppx, ppy, a.P.tau);
    } else {  // the eager kernels' code as it was: written with the accessors, ptxas schedules its loads differently
        const double f = (double)a.P.f, ppx = (double)a.P.ppx, ppy = (double)a.P.ppy;
        solved = p3p_pose(obj, img, f, ppx, ppy, pose, verdict_only ? 1.25 * (double)a.P.tau + 1. : 0.);
        return solved && minimal_set_gate(obj, img, pose, f, ppx, ppy, a.P.tau);
    }
}

// [E,3,N] planes -> [E,N] float4 cells.  The sampling stage gathers 4 random cells per try, millions of times per
// call; with planar storage every cell costs three 32-byte sectors of L2 traffic, interleaved it costs one.
__global__ void interleave_kernel(const float* __restrict__ coords, float4* __restrict__ out, int E, int N) {
    const size_t total = (size_t)E * N;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t e = i / N, p = i - e * N;
        const float* pl = coords + e * 3 * (size_t)N;
        out[i] = make_float4(pl[p], pl[N + p], pl[2 * (size_t)N + p], 0.f);
    }
}

// state init: every hypothesis unresolved, window at try 0
__global__ void sample_init_kernel(const __grid_constant__ SampleArgs a) {
    const SampleState& st = a.st;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = lane_size(a);
    if (k < n) {
        const int h = lane_hyp(a, k);
        st.best[h] = kNoKey; st.base[h] = 0; st.ovf[h] = kNoTry; st.list[k] = h;
    }
    if (k == 0) {  // unresolved, survivors, staged, span, ticket; diagnostics: tries prefiltered, survivors judged, waves with work
        st.counters[0] = n; st.counters[1] = 0; st.counters[2] = 0; st.counters[3] = a.span0; st.counters[4] = 0;
        st.counters[5] = 0; st.counters[6] = 0; st.counters[7] = 0;
    }
}

// ---- wave phase 1: fp32 prefilter, TWO tries per thread (float2 pairs) ---------------------------------------------
constexpr int kPackTries = 2 * kTryThreads;  // tries per CTA pass: thread i judges tries i and i + 128 of the 256-try chunk
// One work item of the prefilter: 256 consecutive tries of one hypothesis, two per thread.
struct PreItem {
    int h, ta, tb;          // hypothesis, this thread's two tries
    bool valid0, valid1;
    unsigned cell[8];       // (y << 16) | x of the 2 x 4 cells
};
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
}
// Decodes item -> (hypothesis, tries), draws the 2 x 4 cells and starts the 8 gathers of 16 bytes straight into shared
// memory (cp.async: no registers are held while they are in flight).
template <bool DEV>
__device__ __forceinline__ void prefilter_issue(const SampleArgsT<DEV>& a, long long item, int cph, int span, float4 (*dst)[kTryThreads], PreItem& it) {
    const int u = (int)(item / cph), c = (int)(item - (long long)u * cph);
    it.h = a.st.list[u];
    const int t0 = a.st.base[it.h];
    const int off0 = c * kPackTries + threadIdx.x, off1 = off0 + kTryThreads;
    it.valid0 = off0 < span && t0 + off0 < a.limit;
    it.valid1 = off1 < span && t0 + off1 < a.limit;
    // an invalid half re-judges try t0 (in range for every listed hypothesis) and is masked out afterwards
    it.ta = it.valid0 ? t0 + off0 : t0;
    it.tb = it.valid1 ? t0 + off1 : t0;
    if (!(it.valid0 || it.valid1)) return;
    const Problem& P = a.P;
    const float4* pl = a.coords4 + (size_t)a.assign32[it.h] * P.N;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const int t = k == 0 ? it.ta : it.tb;
        int cx[4], cy[4];
        if (a.injected) {
            const int* cc = a.injected + ((size_t)it.h * a.inj_T + t) * 8;
            for (int j = 0; j < 4; ++j) { cx[j] = cc[2 * j]; cy[j] = cc[2 * j + 1]; }
        } else {
            draw_minimal_set(sample_seed<DEV>(a), (uint32_t)(it.h * a.hyp_stride + a.hyp_offset), (uint32_t)t, P.W, P.H, cx, cy);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            it.cell[k * 4 + j] = ((unsigned)cy[j] << 16) | (unsigned)cx[j];
            cp_async16(&dst[k * 4 + j][threadIdx.x], pl + (cy[j] * P.W + cx[j]));
        }
    }
}

// ---- wave phase 1: fp32 prefilter, TWO tries per thread (float2 pairs), gathers one item ahead ----------------------
// The math of an item (~2700 instructions per thread, branch-free) runs while the 8 random 16-byte gathers of the NEXT item
// are in flight: with 16-20 warps per SM (the two-try pack needs ~128 registers) nothing else would cover their L2 latency.
// The stage is bound by register capacity x dependency-chain latency: an SM holds 1024 tries in flight (64 registers per
// try) whatever the packing, and a try's dependent instruction chain is the same.  96 registers
// (5 CTAs per SM) spill.
template <bool DEV>
__global__ void __launch_bounds__(kTryThreads, 4) prefilter_kernel(const __grid_constant__ SampleArgsT<DEV> a) {
    TraceScope trace(a.trace, a.trace_slot);
    __shared__ float4 s_obj[2][8][kTryThreads];  // [buffer][try * 4 + point][thread]
    const int n_unres = a.st.counters[0];
    const int span = a.st.counters[3];
    const int cph = (span + kPackTries - 1) / kPackTries;  // chunks per hypothesis
    const long long n_items = (long long)n_unres * cph;
    const int lane = threadIdx.x & 31, tid = threadIdx.x;
    const Problem& P = a.P;
    PreItem cur, nxt;
    long long item = blockIdx.x;
    if (item < n_items) prefilter_issue<DEV>(a, item, cph, span, s_obj[0], cur);
    asm volatile("cp.async.commit_group;" ::: "memory");
    int buf = 0;
    for (; item < n_items; item += gridDim.x) {
        const long long ni = item + gridDim.x;
        if (ni < n_items) prefilter_issue<DEV>(a, ni, cph, span, s_obj[buf ^ 1], nxt);
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 1;" ::: "memory");  // everything but the group just committed has landed
        bool pass0 = false, pass1 = false;
        if (cur.valid0 || cur.valid1) {
            float obj0[4][3], img0[4][2], obj1[4][3], img1[4][2];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float4 v0 = s_obj[buf][j][tid], v1 = s_obj[buf][4 + j][tid];
                obj0[j][0] = v0.x; obj0[j][1] = v0.y; obj0[j][2] = v0.z;
                obj1[j][0] = v1.x; obj1[j][1] = v1.y; obj1[j][2] = v1.z;
                const unsigned c0 = cur.cell[j], c1 = cur.cell[4 + j];
                img0[j][0] = (float)((int)(c0 & 0xffffu) * P.sub + P.sub / 2 - dev_shift_x<DEV>(P, a));
                img0[j][1] = (float)((int)(c0 >> 16) * P.sub + P.sub / 2 - dev_shift_y<DEV>(P, a));
                img1[j][0] = (float)((int)(c1 & 0xffffu) * P.sub + P.sub / 2 - dev_shift_x<DEV>(P, a));
                img1[j][1] = (float)((int)(c1 >> 16) * P.sub + P.sub / 2 - dev_shift_y<DEV>(P, a));
            }
            if (a.use_prefilter)
                p3p_may_pass_fast2(obj0, img0, obj1, img1, dev_f<DEV>(P, a), dev_ppx<DEV>(P, a), dev_ppy<DEV>(P, a), P.tau,
                                   pass0, pass1);
            else pass0 = pass1 = true;
            pass0 = pass0 && cur.valid0;
            pass1 = pass1 && cur.valid1;
        }
        // warp-aggregated append of the survivors (both halves in one reservation)
        const unsigned m0 = __ballot_sync(0xffffffffu, pass0), m1 = __ballot_sync(0xffffffffu, pass1);
        if (m0 | m1) {
            const int n0 = __popc(m0);
            int basei = 0;
            if (lane == 0) basei = atomicAdd(&a.st.counters[1], n0 + __popc(m1));
            basei = __shfl_sync(0xffffffffu, basei, 0);
            const unsigned lt = (1u << lane) - 1u;
            if (pass0) {
                const int idx = basei + __popc(m0 & lt);
                if (idx < a.st.cap) a.st.surv[idx] = make_int2(cur.h, cur.ta);
                else atomicMin(&a.st.ovf[cur.h], cur.ta);  // list full: this hypothesis resumes from here in the next wave
            }
            if (pass1) {
                const int idx = basei + n0 + __popc(m1 & lt);
                if (idx < a.st.cap) a.st.surv[idx] = make_int2(cur.h, cur.tb);
                else atomicMin(&a.st.ovf[cur.h], cur.tb);
            }
        }
        cur = nxt;
        buf ^= 1;
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}

__device__ void advance_wave(const SampleState& st, int limit, float window, float tail_boost);

// ---- wave phase 2: exact fp64 verdict on the survivors -------------------------------------------------------
template <bool DEV>
__global__ void __launch_bounds__(128) exact_kernel(const __grid_constant__ SampleArgsT<DEV> a) {
    TraceScope trace(a.trace, a.trace_slot);
    const int n = min(a.st.counters[1], a.st.cap);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int2 ht = a.st.surv[i];
        if (ht.y >= a.st.ovf[ht.x]) continue;  // beyond the point where the list overflowed: redone next wave
        Pose pose;
        int cx[4], cy[4];
        bool solved;
        if (exact_try<DEV>(a, ht.x, ht.y, pose, cx, cy, solved, true)) {
            // stage the accepted pose so that emit_kernel does not have to solve it again
            unsigned slot = (unsigned)atomicAdd(&a.st.counters[2], 1);
            if (slot < (unsigned)a.st.cap_acc) {
                Accepted& ac = a.st.stage[slot];
                ac.pose = pose;
                for (int j = 0; j < 4; ++j) { ac.cells[2 * j] = cx[j]; ac.cells[2 * j + 1] = cy[j]; }
            } else {
                slot = kNoSlot;
            }
            atomicMin(&a.st.best[ht.x], ((unsigned long long)(unsigned)ht.y << 32) | slot);
        }
    }
    // the last CTA to get here has every verdict of the wave in front of it: it does the bookkeeping
    __shared__ int s_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(&a.st.counters[4], 1) == (int)gridDim.x - 1;
    __syncthreads();
    if (s_last) {
        __threadfence();
        advance_wave(a.st, a.limit, a.window, a.tail_boost);
    }
}

// ---- wave phase 3: bookkeeping (run by the last CTA of exact_kernel to finish) -------------------------------------
__device__ void advance_wave(const SampleState& st, int limit, float window, float tail_boost) {
    __shared__ int s_fill;
    const int span = st.counters[3];
    if (threadIdx.x == 0) s_fill = 0;
    __syncthreads();
    const int n_unres = st.counters[0];
    // the next list is built in the second half of the buffer, then copied back (single CTA: no races)
    int* next = st.list + st.M;
    for (int u = threadIdx.x; u < n_unres; u += blockDim.x) {
        const int h = st.list[u];
        const int ovf = st.ovf[h];
        const int end = min(st.base[h] + span, ovf);  // tries below `end` have all been judged
        const unsigned long long best = __ldcg(&st.best[h]);
        const bool resolved = (long long)(best >> 32) < (long long)end;
        if (!resolved) {
            if (best != kNoKey) st.best[h] = kNoKey;  // an accept beyond an overflow hole does not count yet
            st.base[h] = end;
            st.ovf[h] = kNoTry;
            if (end < limit) next[atomicAdd(&s_fill, 1)] = h;
        }
    }
    __syncthreads();
    const int nn = s_fill;
    for (int u = threadIdx.x; u < nn; u += blockDim.x) st.list[u] = next[u];
    __syncthreads();
    if (threadIdx.x == 0) {
        // next window: ~1.25 / (acceptance rate per try seen in this wave), a multiple of the CTA size
        const int n_surv = min(st.counters[1], st.cap);
        const double tried = (double)n_unres * (double)span;
        const double hits = n_unres - nn > 0 ? (double)(n_unres - nn) : 0.5;
        // few hypotheses left: their tries cost next to nothing, a further wave costs a full verdict latency -- ask for more
        const double boost = nn <= 8 ? tail_boost * 2. : (nn <= 64 ? tail_boost : 1.);
        double next_span = (double)window * boost * tried / hits;
        next_span = next_span < 256. ? 256. : (next_span > 65536. ? 65536. : next_span);
        st.counters[3] = ((int)next_span + kPackTries - 1) / kPackTries * kPackTries;
        st.counters[0] = nn;
        st.counters[1] = 0;
        st.counters[4] = 0;  // ticket of the next exact_kernel
        if (n_unres > 0) {
            st.counters[5] += n_unres * span;
            st.counters[6] += n_surv;
            st.counters[7] += 1;
        }
    }
}

// ---- tail: CTA per unresolved hypothesis, both phases inside the CTA, up to the try limit --------------------
template <bool DEV>
__global__ void __launch_bounds__(kTryThreads) tail_kernel(const __grid_constant__ SampleArgsT<DEV> a) {
    const int n_unres = a.st.counters[0];
    __shared__ int s_list[kTryThreads * 8];
    __shared__ int s_n, s_best;
    for (int u = blockIdx.x; u < n_unres; u += gridDim.x) {
        const int h = a.st.list[u];
        int base = a.st.base[h];
        __syncthreads();
        if (threadIdx.x == 0) s_best = kNoTry;
        while (base < a.limit) {
            if (threadIdx.x == 0) s_n = 0;
            __syncthreads();
            const int span = min(a.limit - base, kTryThreads * 8);
            for (int t = base + threadIdx.x; t < base + span; t += kTryThreads) {
                int cx[4], cy[4];
                float obj[4][3], img[4][2];
                load_try<DEV>(a, h, t, cx, cy, obj, img);
                if (!a.use_prefilter ||
                    p3p_may_pass_fast(obj, img, dev_f<DEV>(a.P, a), dev_ppx<DEV>(a.P, a), dev_ppy<DEV>(a.P, a), a.P.tau))
                    s_list[atomicAdd(&s_n, 1)] = t;
            }
            __syncthreads();
            const int n = s_n;
            for (int i = threadIdx.x; i < n; i += kTryThreads) {
                Pose pose;
                int cx[4], cy[4];
                bool solved;
                if (exact_try<DEV>(a, h, s_list[i], pose, cx, cy, solved, true)) atomicMin(&s_best, s_list[i]);
            }
            __syncthreads();
            if (s_best != kNoTry) break;
            base += span;
        }
        if (threadIdx.x == 0 && s_best != kNoTry) a.st.best[h] = ((unsigned long long)(unsigned)s_best << 32) | kNoSlot;
    }
}


// ---- emit: pose / cells / try count of every hypothesis ------------------------------------------------------
template <bool DEV>
__global__ void __launch_bounds__(64) emit_kernel(const __grid_constant__ SampleArgsT<DEV> a, Pose* poses, int* cells, int* tries) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= lane_size(a)) return;
    const int h = lane_hyp(a, k);
    const unsigned long long key = a.st.best[h];
    const int t = key != kNoKey ? (int)(key >> 32) : a.limit - 1;  // exhausted: the state of the last try survives (esac_util.h:154-224)
    const unsigned slot = (unsigned)(key & 0xffffffffu);
    Pose pose;
    int cx[4], cy[4];
    if (key != kNoKey && slot != kNoSlot) {
        const Accepted& ac = a.st.stage[slot];
        pose = ac.pose;
        for (int j = 0; j < 4; ++j) { cx[j] = ac.cells[2 * j]; cy[j] = ac.cells[2 * j + 1]; }
    } else {
        bool solved;
        exact_try<DEV>(a, h, t, pose, cx, cy, solved);
        if (!solved) { for (int c = 0; c < 3; ++c) { pose.r[c] = 0; pose.t[c] = 0; } }  // safeSolvePnP failure state
    }
    poses[h] = pose;
    for (int j = 0; j < 4; ++j) { cells[h * 8 + 2 * j] = cx[j]; cells[h * 8 + 2 * j + 1] = cy[j]; }
    tries[h] = t + 1;
}

// The hypotheses are dealt to n_lanes lanes, each with its own work list, survivor list, staging area and stream.
// A wave is a throughput-bound kernel (prefilter) followed by a latency-bound one (exact: a few thousand threads, each a
// ~25 us fp64 dependency chain); with two lanes in flight the exact kernel of one can run under the prefilter of the other
// instead of leaving the GPU idle.  Lanes are dealt by hypothesis parity, or -- when the coordinate maps are still
// arriving from the host in two halves (split_e > 0) -- by expert: lane 0 = experts [0, split_e), released by
// ev_half[0]; lane 1 = the rest, released by ev_half[1], so lane 0 samples while the second half is on the wire.
// What was tried on top of this and measured slower or equal (DESIGN.md section 8): 3-4 lanes, one
// prefilter stream + per-lane verdict streams in forced anti-phase, other window policies, a single persistent kernel with
// work / survivor queues, programmatic dependent launch between the kernels of a lane (the ~4 us gaps close, but the early
// CTAs of one lane starve the other).  option sample_trace shows who runs when.
int launch_sample(const float* coords, float4* coords4, const int* assign32, const Problem& P, uint64_t seed, int max_tries,
                  const int* injected, int inj_T, const SampleState* st, int n_lanes, int sm_count, int use_prefilter,
                  int hyp_offset, int hyp_stride, Pose* poses, int* cells, int* tries, const cudaStream_t* lanes,
                  cudaEvent_t ev_fork, const cudaEvent_t* ev_join, int split_e, const int* perm, const int* offsets,
                  const cudaEvent_t* ev_half, int span0, float window, int n_waves,
                  unsigned long long* trace, float tail_boost, const DevParams* dev) {
    int launches = 0;
    cudaStream_t stream = lanes[0];
    if (!split_e) { interleave_kernel<<<sm_count * 8, 256, 0, stream>>>(coords, coords4, P.E, P.N); ++launches; }
    SampleArgsDev args[4];
    int bound[4];
    for (int g = 0; g < n_lanes; ++g) {
        SampleArgsDev& a = args[g];
        a.coords4 = coords4; a.assign32 = assign32; a.P = P; a.seed = seed;
        a.limit = injected ? (max_tries < inj_T ? max_tries : inj_T) : max_tries;
        a.injected = injected; a.inj_T = inj_T; a.st = st[g]; a.use_prefilter = use_prefilter; a.hyp_offset = hyp_offset; a.hyp_stride = hyp_stride > 0 ? hyp_stride : 1;
        a.h_first = g; a.h_step = n_lanes; a.Mg = (P.M - g + n_lanes - 1) / n_lanes;
        a.perm = nullptr; a.offsets = nullptr; a.e_lo = a.e_hi = 0;
        a.span0 = span0; a.window = window; a.trace = trace; a.trace_slot = 0; a.tail_boost = tail_boost;
        a.dev = dev ? *dev : DevParams{};
        bound[g] = a.Mg;  // host-side bound on the lane size (grid sizing)
        if (split_e) {
            a.perm = perm; a.offsets = offsets;
            a.e_lo = g == 0 ? 0 : split_e;
            a.e_hi = g == 0 ? split_e : P.E;
            bound[g] = P.M;
        }
    }
    if (n_lanes > 1) {
        cudaEventRecord(ev_fork, stream);
        for (int g = 1; g < n_lanes; ++g) cudaStreamWaitEvent(lanes[g], ev_fork, 0);
    }
    for (int g = 0; g < n_lanes; ++g) {
        cudaStream_t sg = lanes[g];
        SampleArgsDev& a = args[g];
        const SampleArgs& ae = a;  // what the eager kernels take
        if (split_e) {
            cudaStreamWaitEvent(sg, ev_half[g], 0);
            const int ne = a.e_hi - a.e_lo;
            interleave_kernel<<<sm_count * 8, 256, 0, sg>>>(coords + (size_t)a.e_lo * 3 * P.N, coords4 + (size_t)a.e_lo * P.N, ne, P.N);
            ++launches;
        }
        if (bound[g] <= 0) continue;
        sample_init_kernel<<<(bound[g] + 255) / 256, 256, 0, sg>>>(ae); ++launches;
        // persistent: every CTA resident (4 x 128 threads x 128 registers fill an SM's register file), ~14 items each in a bulk wave;
        // 3 CTAs per SM + 64-thread verdict CTAs in the room that leaves was measured slower
        const int grid = sm_count * 4;
        for (int r = 0; r < n_waves; ++r) {
            a.trace_slot = (g * 32 + r) * 2;
            if (dev) prefilter_kernel<true><<<grid, kTryThreads, 0, sg>>>(a);
            else prefilter_kernel<false><<<grid, kTryThreads, 0, sg>>>(ae);
            ++launches;
            a.trace_slot = (g * 32 + r) * 2 + 1;
            if (dev) exact_kernel<true><<<sm_count * 4, 128, 0, sg>>>(a);  // its last CTA also advances the windows
            else exact_kernel<false><<<sm_count * 4, 128, 0, sg>>>(ae);
            ++launches;
        }
        const int tail_grid = bound[g] < sm_count * 4 ? bound[g] : sm_count * 4;
        if (dev) {
            tail_kernel<true><<<tail_grid, kTryThreads, 0, sg>>>(a);
            emit_kernel<true><<<(bound[g] + 63) / 64, 64, 0, sg>>>(a, poses, cells, tries);
        } else {
            tail_kernel<false><<<tail_grid, kTryThreads, 0, sg>>>(ae);
            emit_kernel<false><<<(bound[g] + 63) / 64, 64, 0, sg>>>(ae, poses, cells, tries);
        }
        launches += 2;
    }
    for (int g = 1; g < n_lanes; ++g) {
        cudaEventRecord(ev_join[g], lanes[g]);
        cudaStreamWaitEvent(stream, ev_join[g], 0);
    }
    return launches;
}

__global__ void trace_init_kernel(unsigned long long* trace, int slots) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < slots) { trace[2 * i] = ~0ull; trace[2 * i + 1] = 0ull; }
}
void launch_trace_init(unsigned long long* trace, int slots, cudaStream_t st) { trace_init_kernel<<<(slots + 255) / 256, 256, 0, st>>>(trace, slots); }

}  // namespace esacb200
