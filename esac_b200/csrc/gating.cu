// Hypothesis assignment on the device (SURVEY 8f rank 2).
//
// The reference's callers draw the expert of every hypothesis on the host from the gating distribution and build the
// per-expert histogram that decides which experts run and scales the gating gradient:
//   util.clamp_probs(gating_probs[0], maxexperts)                       util.py:38-48, train_esac.py:130
//   e_hyps = torch.multinomial(gating_probs[0], hypotheses, True)       train_esac.py:133-137, test_esac.py:169-174
//   e_hyps_hist = torch.histc(e_hyps.float(), bins=E, min=0, max=E-1)   train_esac.py:140,  test_esac.py:177
// Here one CTA per image does the three steps without leaving the GPU, so a batch of gating outputs turns into the
// [B, M] assignment that esacb200_forward_batch / esacb200_backward_batch consume.  The draws come from the same
// counter-based generator as the minimal sets (esac_rng.cuh), keyed (seed, image, hypothesis): the oracle
// (oracle/esac_oracle.py: assign_hypotheses) reproduces them bit for bit.  torch.multinomial's own stream is not
// reproduced (it is a property of torch's Philox/mt19937 state, not of the algorithm); the distribution is.
#include "esac_internal.h"
#include "esac_rng.cuh"

namespace esacb200 {

namespace {

constexpr int kMaxExperts = 1024;

// Whether weight a at index ia comes before weight b at index ib in the stable ascending order of torch.sort and
// np.argsort(kind="stable"): NaN above every number (+inf included), equal values and NaNs among themselves by index.
// A plain a < b would give a NaN rank 0, so keep_top would zero it and draw from the rest where torch keeps it and raises.
__device__ __forceinline__ bool sorts_before(float a, int ia, float b, int ib) {
    const bool na = a != a, nb = b != b;
    if (na || nb) return !na || (nb && ia < ib);
    return a < b || (a == b && ia < ib);
}

// weights [B, E] (>= 0, need not sum to 1: multinomial normalises), out_assign [B, M] int64, out_hist [B, E] float.
// keep_top < 0: no clamping; else all but the keep_top largest weights are zeroed first, largest in the stable ascending
// order of sorts_before (ties: the later index wins a place; a NaN is kept before any number, and then flagged below).
// single != 0: one draw per image, repeated M times
// (the "expertselection" mode, train_esac.py:133-135).
// DEV = false: the eager call -- the seed is a parameter and `flags` one int the images OR their error bits into.
// DEV = true: the stream-ordered call -- the seed is read from d_seed when the kernel runs (a graph replays with what the
// tensor holds then) and `flags` is [B]: image b's status (0, 1 or 2) is written, not OR-ed, so no memset precedes it.
template <bool DEV>
__global__ void __launch_bounds__(256) assign_kernel(const float* __restrict__ weights, int E, int M, int keep_top, int single,
                                                     uint64_t seed, const long long* __restrict__ d_seed,
                                                     int64_t* __restrict__ out_assign, float* __restrict__ out_hist,
                                                     int* __restrict__ flags) {
    if constexpr (DEV) seed = (uint64_t)*d_seed;
    __shared__ float w[kMaxExperts];
    __shared__ double cdf[kMaxExperts];
    __shared__ int hist[kMaxExperts];
    __shared__ int last_pos;
    const int b = blockIdx.x;
    for (int e = threadIdx.x; e < E; e += blockDim.x) {
        w[e] = weights[(size_t)b * E + e];
        hist[e] = 0;
    }
    __syncthreads();
    if (keep_top >= 0 && keep_top < E) {
        // rank of entry e in the stable ascending order = #{j: (w[j], j) sorts before (w[e], e)}
        for (int e = threadIdx.x; e < E; e += blockDim.x) {
            const float we = w[e];
            int rank = 0;
            for (int j = 0; j < E; ++j) rank += sorts_before(w[j], j, we, e);
            if (rank < E - keep_top) cdf[e] = 0.;  // remember the verdict; w is still being read by other threads
            else cdf[e] = 1.;
        }
        __syncthreads();
        for (int e = threadIdx.x; e < E; e += blockDim.x)
            if (cdf[e] == 0.) w[e] = 0.f;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        double acc = 0.;
        int lp = -1;
        bool bad = false;
        for (int e = 0; e < E; ++e) {
            const float v = w[e];
            if (!(v >= 0.f) || isinf(v)) bad = true;  // torch.multinomial: "probability tensor contains either inf, nan or element < 0"
            if (v > 0.f) { acc += (double)v; lp = e; }
            cdf[e] = acc;
        }
        if constexpr (DEV) flags[b] = bad ? 1 : (lp < 0 ? 2 : 0);
        else if (bad || lp < 0) atomicOr(flags, bad ? 1 : 2);  // 2: "invalid multinomial distribution (sum of probabilities <= 0)"
        last_pos = lp;
    }
    __syncthreads();
    const int lp = last_pos;
    const double total = lp >= 0 ? cdf[E - 1] : 0.;
    for (int h = threadIdx.x; h < M; h += blockDim.x) {
        const uint32_t k = single ? 0u : (uint32_t)h;
        const uint64_t r = try_state(seed, (uint32_t)b, k);
        const double u = (double)(r >> 11) * 0x1.0p-53 * total;
        // first expert whose cumulative weight exceeds u (experts of zero weight can never be it)
        int lo = 0, hi = E - 1;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (cdf[mid] > u) hi = mid;
            else lo = mid + 1;
        }
        int e = lo;
        if (lp >= 0 && !(cdf[e] > u)) e = lp;  // u rounded up to the total
        if (lp < 0) e = 0;
        out_assign[(size_t)b * M + h] = e;
        atomicAdd(&hist[e], 1);
    }
    __syncthreads();
    if (out_hist)
        for (int e = threadIdx.x; e < E; e += blockDim.x) out_hist[(size_t)b * E + e] = (float)hist[e];
}

}  // namespace

int assign_max_experts() { return kMaxExperts; }

void launch_assign(const float* weights, int B, int E, int M, int keep_top, int single, uint64_t seed, int64_t* out_assign,
                   float* out_hist, int* flags, cudaStream_t stream) {
    assign_kernel<false><<<B, 256, 0, stream>>>(weights, E, M, keep_top, single, seed, nullptr, out_assign, out_hist, flags);
}

void launch_assign_async(const float* weights, int B, int E, int M, int keep_top, int single, const long long* d_seed,
                         int64_t* out_assign, float* out_hist, int* out_status, cudaStream_t stream) {
    assign_kernel<true><<<B, 256, 0, stream>>>(weights, E, M, keep_top, single, 0, d_seed, out_assign, out_hist, out_status);
}

}  // namespace esacb200
