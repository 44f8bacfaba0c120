// What every ESAC call of libesac_b200.so is built from: the problem of an image, the workspace of each stage and the stages
// themselves (upload, prep, sampling, scoring, refinement), the end of a call, the hypotheses of a backward, the context of
// the stream-ordered calls, and the worker contexts of the batched calls.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdio.h>

#include <algorithm>
#include <chrono>
#include <functional>
#include <map>
#include <string>
#include <thread>
#include <vector>

#include "capi_internal.h"
#include "esac_rng.cuh"

using namespace esacb200;
using namespace esacb200::capi;

namespace esacb200::capi {

NcclApi& nccl_api() {
    static NcclApi api;
    static bool tried = false;
    if (tried) return api;
    tried = true;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return api;
    api.GetUniqueId = (int (*)(NcclApi::UniqueId*))dlsym(h, "ncclGetUniqueId");
    api.CommInitRank = (int (*)(void**, int, NcclApi::UniqueId, int))dlsym(h, "ncclCommInitRank");
    api.CommDestroy = (int (*)(void*))dlsym(h, "ncclCommDestroy");
    api.AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(h, "ncclAllGather");
    api.AllReduce = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(h, "ncclAllReduce");
    api.GetErrorString = (const char* (*)(int))dlsym(h, "ncclGetErrorString");
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.AllReduce;
    return api;
}

int fill_problem(esacb200_ctx* ctx, Problem& P, int E, int H, int W, int M, int shiftX, int shiftY, float f, float ppx,
                 float ppy, float tau, float alpha, float beta, float maxReproj, int sub, Draw draw) {
    if (E <= 0 || H <= 0 || W <= 0 || M <= 0) return fail(ctx, ESACB200_ERR_ARG, "empty tensor (E=%d H=%d W=%d M=%d)", E, H, W, M);
    if ((long long)H * W > (1ll << 30)) return fail(ctx, ESACB200_ERR_ARG, "coordinate map too large");
    if (draw != NO_DRAW && (long long)(W - 1) * (H - 1) < 4)
        return fail(ctx, ESACB200_ERR_ARG, "map %dx%d too small to draw 4 distinct cells from [0,W-2]x[0,H-2]", W, H);
    if (draw == DRAWS_INJECTED && ctx->inj_M && ctx->inj_M != M)
        return fail(ctx, ESACB200_ERR_ARG, "injected cells are for M=%d, call has M=%d", ctx->inj_M, M);
    // the sampling kernels gather coords[cy * W + cx] of every injected cell unchecked
    if (draw == DRAWS_INJECTED && ctx->inj_M &&
        (ctx->inj_lo[0] < 0 || ctx->inj_lo[1] < 0 || ctx->inj_hi[0] > W - 1 || ctx->inj_hi[1] > H - 1))
        return fail(ctx, ESACB200_ERR_ARG, "injected cells span x %d..%d, y %d..%d: outside the %dx%d map", ctx->inj_lo[0],
                    ctx->inj_hi[0], ctx->inj_lo[1], ctx->inj_hi[1], W, H);
    P.E = E; P.H = H; P.W = W; P.N = H * W; P.M = M;
    P.shiftX = shiftX; P.shiftY = shiftY; P.sub = sub;
    P.f = f; P.ppx = ppx; P.ppy = ppy; P.tau = tau; P.alpha = alpha; P.beta = beta; P.max_reproj = maxReproj;
    return 0;
}

// The problems of a ragged batch: image b is H[b] x W[b] with entry b of the shift and camera arrays (a null array: 0),
// checked image by image under an "image b:" prefix before any image runs.
int fill_problems(esacb200_ctx* ctx, std::vector<Plan>& plans, int B, int E, const int* H, const int* W, int M, const int* shiftX,
                  const int* shiftY, const float* f, const float* ppx, const float* ppy, float tau, float alpha, float beta,
                  float maxReproj, int sub, Draw draw) {
    plans.resize((size_t)B);
    for (int b = 0; b < B; ++b)
        if (fill_problem(ctx, plans[b].P, E, H[b], W[b], M, shiftX ? shiftX[b] : 0, shiftY ? shiftY[b] : 0, f ? f[b] : 0.f,
                         ppx ? ppx[b] : 0.f, ppy ? ppy[b] : 0.f, tau, alpha, beta, maxReproj, sub, draw))
            return fail(ctx, ESACB200_ERR_ARG, "image %d: %s", b, std::string(ctx->err).c_str());
    return 0;
}

// ---- workspace of the forward pipeline --------------------------------------------------------------------------
// Each stage states the sizes of its buffers in one function that calls `need(buf, bytes)` once per buffer: the stage
// itself grows them (grow), and forward_workspace sizes or checks them for a whole batch before anything is enqueued.
#define NEED(buf, bytes) do { int r__ = need(buf, bytes); if (r__) return r__; } while (0)

int Grow::operator()(DevBuf& b, size_t bytes) const {
    CK(b.ensure(bytes));
    return 0;
}

Grow grow(esacb200_ctx* ctx) { return {ctx}; }

// Input staging: a host coordinate map goes to `cbuf`, host assignments to `abuf` (null: that input is not staged).
template <class Need>
static int input_buffers(const Problem& P, DevBuf* cbuf, DevBuf* abuf, Need&& need) {
    if (cbuf) NEED(*cbuf, (size_t)P.E * 3 * P.N * sizeof(float));
    if (abuf) NEED(*abuf, (size_t)P.M * 8);
    return 0;
}

// Upload (or alias) the inputs.  Host coordinate maps go to `cbuf` on `copy_stream` (pinned memory: asynchronous).
int upload_inputs(esacb200_ctx* ctx, Plan& pl, const float* coords, const int64_t* assign, int64_t stride, DevBuf& cbuf,
                  DevBuf& abuf, cudaStream_t copy_stream, bool allow_split) {
    const Problem& P = pl.P;
    const size_t cbytes = (size_t)P.E * 3 * P.N * sizeof(float);
    const bool dev_coords = is_device_ptr(coords), dev_assign = is_device_ptr(assign);
    int rc = input_buffers(P, dev_coords ? nullptr : &cbuf, dev_assign ? nullptr : &abuf, grow(ctx));
    if (rc) return rc;
    pl.split_e = 0;
    if (dev_coords) {
        pl.d_coords = coords;
    } else if (allow_split && P.E >= 2 && cbytes >= (size_t)(4 << 20) && P.M >= 64 && ctx->aux_stream && ctx->opt.sample_groups > 1 &&
               ctx->opt.upload_split) {
        // Large host maps: two halves on the copy stream, so the first half's experts are sampled while the second half is
        // still on the wire (launch_sample deals its two lanes by expert in this case).
        const int es = (P.E + 1) / 2;
        const size_t first = (size_t)es * 3 * P.N * sizeof(float);
        CK(cudaMemcpyAsync(cbuf.p, coords, first, cudaMemcpyHostToDevice, ctx->copy_stream));
        CK(cudaEventRecord(ctx->ev_copied[0], ctx->copy_stream));
        CK(cudaMemcpyAsync((char*)cbuf.p + first, (const char*)coords + first, cbytes - first, cudaMemcpyHostToDevice, ctx->copy_stream));
        CK(cudaEventRecord(ctx->ev_copied[1], ctx->copy_stream));
        pl.d_coords = cbuf.as<float>();
        pl.split_e = es;
    } else {
        CK(cudaMemcpyAsync(cbuf.p, coords, cbytes, cudaMemcpyHostToDevice, copy_stream));
        pl.d_coords = cbuf.as<float>();
    }
    if (dev_assign) {
        pl.d_assign = (const long long*)assign;
        pl.assign_stride = stride;
    } else {
        std::vector<long long> tmp((size_t)P.M);
        for (int h = 0; h < P.M; ++h) tmp[h] = (long long)assign[(long long)h * stride];
        // pageable source: the copy is staged before cudaMemcpyAsync returns, so tmp may die
        CK(cudaMemcpyAsync(abuf.p, tmp.data(), (size_t)P.M * 8, cudaMemcpyHostToDevice, copy_stream));
        pl.d_assign = abuf.as<long long>();
        pl.assign_stride = 1;
    }
    return 0;
}

// Scoring launch shape (no device work).
static void plan_launch(esacb200_ctx* ctx, Plan& pl) {
    const Problem& P = pl.P;
    // scoring launch shape
    int ppt = 8, hc = 64;
    const int want = 2 * 2 * ctx->sm_count;
    auto items = [&](int ppt_, int hc_) {
        int T = (P.N + score_tile_pixels(ppt_) - 1) / score_tile_pixels(ppt_);
        int nch = (P.M + hc_ - 1) / hc_ + (P.E > 1 ? P.E / 2 : 0);
        return (long long)T * nch;
    };
    if (items(8, 64) < want) { ppt = 4; hc = 32; }
    if (ppt == 4 && items(4, 32) < want) { ppt = 2; hc = 16; }
    const int ppt_opt = ctx->opt.score_ppt_opt, hc_opt = ctx->opt.score_hc_opt;
    if (ppt_opt == 2 || ppt_opt == 4 || ppt_opt == 8) ppt = ppt_opt;
    if (hc_opt > 0) hc = hc_opt < 64 ? hc_opt : 64;
    pl.ppt = ppt;
    pl.hc = hc;
    pl.T = (P.N + score_tile_pixels(ppt) - 1) / score_tile_pixels(ppt);
    const int max_chunks = (P.M + hc - 1) / hc + P.E;
    long long it = (long long)pl.T * max_chunks;
    pl.grid = (int)(it < 2ll * ctx->sm_count ? it : 2ll * ctx->sm_count);
    const int need_align = ppt >= 4 ? 4 : 2;
    pl.vec_ok = (P.N % need_align == 0) && (((uintptr_t)pl.d_coords) % (need_align * 4) == 0);
}

// Prep, scoring and selection: per-hypothesis state and the scoring partials (pl.T: plan_launch first).
template <class Need>
static int prep_buffers(esacb200_ctx* ctx, const Plan& pl, Need&& need) {
    const Problem& P = pl.P;
    NEED(ctx->assign32, (size_t)P.M * 4);
    NEED(ctx->counts, (size_t)P.E * 4);
    NEED(ctx->offsets, (size_t)(P.E + 1) * 4);
    NEED(ctx->perm, (size_t)P.M * 4);
    NEED(ctx->slot_of, (size_t)P.M * 4);
    NEED(ctx->chunks, (size_t)(P.M + P.E) * sizeof(ChunkDesc));
    NEED(ctx->scalars, S_COUNT * 4);
    NEED(ctx->centres, (size_t)P.E * 3 * 4);
    NEED(ctx->poses, (size_t)P.M * sizeof(Pose));
    NEED(ctx->poses_ref, (size_t)P.M * sizeof(Pose));
    NEED(ctx->cells, (size_t)P.M * 8 * 4);
    NEED(ctx->tries, (size_t)P.M * 4);
    NEED(ctx->posepk, (size_t)P.M * sizeof(PosePk));
    NEED(ctx->part, (size_t)P.M * pl.T * 4);
    NEED(ctx->scores, (size_t)P.M * 8);
    NEED(ctx->probs, (size_t)P.M * 8);
    NEED(ctx->stats, sizeof(CallStats));
    NEED(ctx->contrib, (size_t)P.M * 4);
    NEED(ctx->fwd_rec, sizeof(ForwardRecord));
    return 0;
}

// Scoring launch shape, workspace, prep kernel.
int plan_and_prep(esacb200_ctx* ctx, Plan& pl) {
    const Problem& P = pl.P;
    plan_launch(ctx, pl);
    int rc = prep_buffers(ctx, pl, grow(ctx));
    if (rc) return rc;
    int* sc = ctx->scalars.as<int>();
    launch_prep(pl.d_coords, pl.d_assign, pl.assign_stride, P, pl.hc, ctx->assign32.as<int>(), ctx->counts.as<int>(),
                ctx->offsets.as<int>(), ctx->perm.as<int>(), ctx->slot_of.as<int>(), ctx->chunks.as<ChunkDesc>(),
                sc + S_NCHUNKS, sc + S_WORK, ctx->centres.as<float>(), sc + S_FLAGS, pl.split_e ? 1 : 3, ctx->stream);
    ctx->st.kernel_launches += 1;
    mark(ctx, EV_PREP);
    return 0;
}

int stage_inputs(esacb200_ctx* ctx, Plan& pl, const float* coords, const int64_t* assign, int64_t stride, bool allow_split) {
    int rc = upload_inputs(ctx, pl, coords, assign, stride, ctx->coords, ctx->assign64, ctx->stream, allow_split);
    if (rc) return rc;
    mark(ctx, EV_H2D);
    return plan_and_prep(ctx, pl);
}

namespace {

constexpr int kSampleCap = 1 << 19;     // survivors per lane
constexpr int kSampleCapAcc = 1 << 15;  // staged accepts per lane

// Lanes of the sampling stage and its workspace: ints (smp_int) and survivor / staging bytes (smp_surv).
struct SampleSizes {
    int M, G, Mg;
    size_t per_group_ints, int_bytes, per_group_bytes, surv_bytes;
};

// The workspace of G lanes whose work lists hold Mg of the M hypotheses each.
SampleSizes sample_layout(int M, int G, int Mg) {
    SampleSizes z;
    z.M = M;
    z.G = G;
    z.Mg = Mg;
    // ints: [best: 2M] [base: M] [ovf: M] [cut: M] then per group [list: 2*Mg] [counters: SC_COUNT]
    z.per_group_ints = (size_t)2 * z.Mg + SC_COUNT;
    z.int_bytes = ((size_t)M * 5 + G * z.per_group_ints) * 4 + 8;
    z.per_group_bytes = (size_t)kSampleCap * sizeof(int2) + (size_t)kSampleCapAcc * sizeof(Accepted);
    z.surv_bytes = G * z.per_group_bytes;
    return z;
}

SampleSizes sample_sizes(const esacb200_ctx* ctx, const Plan& pl) {
    const Problem& P = pl.P;
    // two lanes pay once a wave's kernels are long enough to overlap (full-resolution maps, or very many hypotheses)
    const int groups = ctx->opt.sample_groups;
    int G = pl.split_e ? 2 : ((groups > 1 && ctx->aux_stream && P.M >= 64 && (P.N >= 65536 || P.M >= 1024)) ? groups : 1);
    if (G > 2 && (!ctx->aux_more[0] || !ctx->aux_more[1] || P.M < 512)) G = 2;
    return sample_layout(P.M, G, pl.split_e ? P.M : (P.M + G - 1) / G);  // Mg: capacity of a lane's work list
}

// Lane g's state in the context's sampling workspace, laid out as z.
SampleState lane_state(const esacb200_ctx* ctx, const SampleSizes& z, int g) {
    SampleState s;
    int* b = ctx->smp_int.as<int>() + 2 * (size_t)z.M;
    s.best = ctx->smp_int.as<unsigned long long>();  // 8-byte aligned: first in the buffer
    s.base = b;
    s.ovf = b + z.M;
    s.cut = b + 2 * (size_t)z.M;
    s.list = b + 3 * (size_t)z.M + g * z.per_group_ints;
    s.counters = s.list + 2 * (size_t)z.Mg;
    char* sb = (char*)ctx->smp_surv.p + g * z.per_group_bytes;
    s.surv = (int2*)sb;
    s.stage = (Accepted*)(sb + (size_t)kSampleCap * sizeof(int2));
    s.cap = kSampleCap;
    s.cap_acc = kSampleCapAcc;
    s.M = z.Mg;
    return s;
}

// Sampling: the lanes' state and the float4 copy of the maps.
template <class Need>
int sample_buffers(esacb200_ctx* ctx, const Plan& pl, Need&& need) {
    const SampleSizes z = sample_sizes(ctx, pl);
    NEED(ctx->smp_int, z.int_bytes);
    NEED(ctx->smp_surv, z.surv_bytes);
    NEED(ctx->coords4, (size_t)pl.P.E * pl.P.N * sizeof(float4));
    return 0;
}

}  // namespace

int run_sample(esacb200_ctx* ctx, const Plan& pl, uint64_t seed) {
    const Problem& P = pl.P;
    const Options& o = ctx->opt;
    const SampleSizes z = sample_sizes(ctx, pl);
    const int G = z.G;
    int rc = sample_buffers(ctx, pl, grow(ctx));
    if (rc) return rc;
    SampleState st[4];
    for (int g = 0; g < G; ++g) st[g] = lane_state(ctx, z, g);
    unsigned long long* trace = nullptr;
    if (o.sample_trace) {  // 4 lanes x 32 waves x 2 kernels x (start, end)
        CK(ctx->smp_trace.ensure(512 * 8));
        CK(cudaMemsetAsync(ctx->smp_trace.p, 0, 512 * 8, ctx->stream));
        trace = ctx->smp_trace.as<unsigned long long>();
        launch_trace_init(trace, 256, ctx->stream);
    }
    const cudaStream_t lane_streams[4] = {ctx->stream, ctx->aux_stream, ctx->aux_more[0], ctx->aux_more[1]};
    const cudaEvent_t lane_joins[4] = {nullptr, ctx->ev_join, ctx->ev_join_more[0], ctx->ev_join_more[1]};
    ctx->st.kernel_launches += launch_sample(pl.d_coords, ctx->coords4.as<float4>(), ctx->assign32.as<int>(), P, seed, o.max_tries,
                                             ctx->inj_M ? ctx->inject.as<int>() : nullptr, ctx->inj_T, st, G, ctx->sm_count,
                                             o.sample_prefilter, o.hyp_offset, o.hyp_stride, ctx->poses.as<Pose>(), ctx->cells.as<int>(),
                                             ctx->tries.as<int>(), lane_streams, ctx->ev_fork, lane_joins,
                                             pl.split_e, ctx->perm.as<int>(), ctx->offsets.as<int>(), ctx->ev_copied,
                                             o.sample_span0, o.sample_window, o.sample_waves, trace, o.sample_tail_boost,
                                             o.sample_prefilter ? o.sample_hint : 0.f, pl.async ? &pl.async->dev : nullptr);
    CK(cudaGetLastError());
    if (pl.split_e) {
        // both halves have landed (the join orders this stream after lane 1, which waited for the second half): plane centres
        int* sc = ctx->scalars.as<int>();
        launch_prep(pl.d_coords, pl.d_assign, pl.assign_stride, P, pl.hc, ctx->assign32.as<int>(), ctx->counts.as<int>(),
                    ctx->offsets.as<int>(), ctx->perm.as<int>(), ctx->slot_of.as<int>(), ctx->chunks.as<ChunkDesc>(),
                    sc + S_NCHUNKS, sc + S_WORK, ctx->centres.as<float>(), sc + S_FLAGS, 2, ctx->stream);
        ctx->st.kernel_launches += 1;
    }
    mark(ctx, EV_SAMPLE);
    return 0;
}

int run_score(esacb200_ctx* ctx, const Plan& pl) {
    const Problem& P = pl.P;
    int* sc = ctx->scalars.as<int>();
    ScoreArgs a;
    score_constants(P, a);
    launch_fold(ctx->poses.as<Pose>(), ctx->perm.as<int>(), ctx->assign32.as<int>(), ctx->centres.as<float>(), P,
                a.fold ? a.k1 : 1.f, ctx->posepk.as<PosePk>(), ctx->stream, pl.async ? &pl.async->dev : nullptr);
    mark(ctx, EV_FOLD);
    a.coords = pl.d_coords;
    a.centres = ctx->centres.as<float>();
    a.poses = ctx->posepk.as<PosePk>();
    a.chunks = ctx->chunks.as<ChunkDesc>();
    a.n_chunks = sc + S_NCHUNKS;
    a.work_counter = sc + S_WORK;
    a.part = ctx->part.as<float>();
    a.P = P;
    a.T = pl.T;
    a.hc = pl.hc;
    a.vec_ok = pl.vec_ok;
    if (pl.async) a.dev = pl.async->dev;
    launch_score(a, pl.ppt, pl.grid, ctx->stream);
    mark(ctx, EV_SCORE);
    launch_select(ctx->part.as<float>(), ctx->slot_of.as<int>(), P, pl.T, ctx->scores.as<double>(), ctx->probs.as<double>(),
                  ctx->stats.as<CallStats>(), sc + S_WINNER, ctx->contrib.as<int>(), sc + S_NCONTRIB, pl.min_prob, ctx->stream);
    mark(ctx, EV_SELECT);
    ctx->st.kernel_launches += 3;
    ctx->st.score_launches += 1;
    ctx->st.score_ppt = pl.ppt;
    ctx->st.score_grid = pl.grid;
    return 0;
}

int pick_group(const esacb200_ctx* ctx, const Problem& P, int jobs_hint) {
    return refine_group_rule(P.N, ctx->refine_coresident, ctx->opt.refine_group_opt, ctx->opt.refine_jobs_per_group, jobs_hint);
}

// Refinement of `n_jobs` (host count, or device scalar when d_njobs != null) hypotheses listed in d_jobs.
namespace {

// Groups of the refinement kernel and its workspace (bytes; clist = 0 when the kernel does not use it).
struct RefineSizes {
    int n_groups, cache;
    size_t masks, rounds, scratch, n_flags, barrier, clist;
};
// group 0: picked on the device from the job count (stream-ordered backward).  The sizes are then the largest of every group
// a count in 1..max_jobs may pick, cache is 1 when any of them caches, and n_groups is the CTA count of the largest launch.
RefineSizes refine_sizes(const esacb200_ctx* ctx, const Problem& P, int max_jobs, int group) {
    RefineSizes z;
    if (group == 0) {
        z = refine_sizes(ctx, P, max_jobs, pick_group(ctx, P, 1));
        z.n_groups *= pick_group(ctx, P, 1);
        for (int n = 2, last = pick_group(ctx, P, 1); n <= max_jobs; ++n) {
            const int g = pick_group(ctx, P, n);
            if (g == last) continue;
            last = g;
            const RefineSizes y = refine_sizes(ctx, P, max_jobs, g);
            z.n_groups = std::max(z.n_groups, y.n_groups * g);
            z.cache = std::max(z.cache, y.cache);
            z.scratch = std::max(z.scratch, y.scratch);
            z.n_flags = std::max(z.n_flags, y.n_flags);
            z.barrier = std::max(z.barrier, y.barrier);
            z.clist = std::max(z.clist, y.clist);
        }
        return z;
    }
    const int words = (P.N + 31) / 32;
    const int n_groups = refine_n_groups(ctx->refine_coresident, group, max_jobs);
    z.n_groups = n_groups;
    z.masks = (size_t)max_jobs * 2 * words * 4;
    z.rounds = (size_t)max_jobs * 2 * 4;
    z.scratch = refine_scratch_doubles(n_groups, group) * 8;
    z.n_flags = refine_flag_words(n_groups, group);
    z.barrier = (z.n_flags + 4) * 4;
    const int wpc = (words + group - 1) / group;
    z.cache = wpc <= refine_cache_words() ? 1 : 0;
    z.clist = (ctx->opt.refine_compact && !z.cache && wpc <= refine_max_compact_words())
                  ? (size_t)n_groups * words * 32 * sizeof(unsigned short) : 0;
    return z;
}

// Refinement (own_masks: the final inlier masks go to the context's workspace).
template <class Need>
int refine_buffers(esacb200_ctx* ctx, const Problem& P, int max_jobs, int group, bool own_masks, Need&& need) {
    const RefineSizes z = refine_sizes(ctx, P, max_jobs, group);
    if (own_masks) NEED(ctx->masks, z.masks);
    NEED(ctx->rounds, z.rounds);
    NEED(ctx->scratch, z.scratch);
    NEED(ctx->barrier, z.barrier);
    if (z.clist) NEED(ctx->clist, z.clist);
    return 0;
}

}  // namespace

// masks_out: where the final inlier masks go ([max_jobs][2][words]); null = the context's workspace.
int run_refine(esacb200_ctx* ctx, const Plan& pl, const Pose* in, Pose* out, const int* d_jobs, const int* d_njobs,
               int n_jobs_host, int max_jobs, int group, uint32_t* masks_out) {
    const Problem& P = pl.P;
    const int words = (P.N + 31) / 32;
    const RefineSizes z = refine_sizes(ctx, P, max_jobs, group);
    const int n_groups = z.n_groups;
    int rc = refine_buffers(ctx, P, max_jobs, group, !masks_out, grow(ctx));
    if (rc) return rc;
    if (!masks_out) masks_out = ctx->masks.as<uint32_t>();
    if (group == 0 && !pl.async) return fail(ctx, ESACB200_ERR_ARG, "refinement group picked on the device outside a stream-ordered call");
    if (group != 1) CK(cudaMemsetAsync(ctx->scratch.p, 0, z.scratch, ctx->stream));  // LL elements: no stale sequence numbers
    const size_t n_flags = z.n_flags;
    CK(cudaMemsetAsync(ctx->barrier.p, 0, z.barrier, ctx->stream));
    RefineArgs a;
    a.coords = pl.d_coords;
    a.centres = ctx->centres.as<float>();
    a.assign32 = ctx->assign32.as<int>();
    a.poses_in = in;
    a.poses_out = out;
    a.jobs = d_jobs;
    a.n_jobs = d_njobs;
    a.n_jobs_host = n_jobs_host;
    a.masks = masks_out;
    a.mask_words = words;
    a.rounds = ctx->rounds.as<int>();
    a.scratch = ctx->scratch.as<double>();
    a.barrier = ctx->barrier.as<unsigned int>();
    a.job_counter = (int*)(ctx->barrier.as<unsigned int>() + n_flags);
    a.group = group;
    a.cache = z.cache;
    a.compact = ctx->opt.refine_compact;
    a.pretest = ctx->opt.refine_pretest;
    a.clist = z.clist ? ctx->clist.as<unsigned short>() : nullptr;
    a.prof = nullptr;
    if (ctx->opt.refine_profile) {
        CK(ctx->prof.ensure(16 * 8));
        CK(cudaMemsetAsync(ctx->prof.p, 0, 16 * 8, ctx->stream));
        a.prof = ctx->prof.as<long long>();
    }
    a.P = P;
    a.max_ref_steps = ctx->opt.max_ref_steps;
    if (pl.async) a.dev = pl.async->dev;
    a.coresident = ctx->refine_coresident;
    a.group_opt = ctx->opt.refine_group_opt;
    a.jobs_per_group = ctx->opt.refine_jobs_per_group;
    a.max_jobs = max_jobs;
    launch_refine(a, n_groups, ctx->stream);
    CK(cudaGetLastError());
    ctx->st.kernel_launches += 1;
    ctx->st.refine_group = group;
    return 0;
}

uint64_t call_seed(esacb200_ctx* ctx) {
    uint64_t s = ctx->opt.fixed_seed ? ctx->seed : mix64(ctx->seed + kGold * ctx->calls);
    if (ctx->calls == 0) s = ctx->seed;
    ++ctx->calls;
    return s;
}

// The backward's tail (bwd_reduce .. bwd_assemble); `losses`: esac.backward's own per-hypothesis losses too.
template <class Need>
int backward_buffers(esacb200_ctx* ctx, const Problem& P, bool losses, Need&& need) {
    if (losses) NEED(ctx->losses, (size_t)P.M * 8);
    NEED(ctx->red, (size_t)P.M * bwd_tiles(P.N) * bwd_red_vals() * 8);
    NEED(ctx->hypgrad, (size_t)P.M * bwd_hypgrad_bytes());
    NEED(ctx->job_of, (size_t)(P.M > P.E ? P.M : P.E) * 4);
    return 0;
}
template int backward_buffers(esacb200_ctx* ctx, const Problem& P, bool losses, Grow&& need);  // the backward entry points

// Sizes every workspace buffer of the forward pipeline (upload, plan_and_prep, sampling, refinement) for the largest of a
// batch's images before the first one is enqueued: DevBuf::ensure growing mid-batch frees the old buffer, and cudaFree
// synchronises the device, which would serialise the copy stream's overlap with the previous image.
// `need(buf, bytes)` is called once per buffer with the largest size any image needs; reserve_forward_batch grows them, the
// stream-ordered forward also checks them.  (host_coords: the images' maps are staged, double-buffered.)  backward: also the
// stream-ordered backward's buffers -- the refinement of up to M jobs with its group picked on the device (every group a
// job count may pick) and backward_buffers.
template <class Need>
static int forward_workspace(esacb200_ctx* ctx, const std::vector<Plan>& plans, bool host_coords, Need&& need, bool backward = false) {
    std::map<DevBuf*, size_t> most;
    auto mx = [&](DevBuf& b, size_t bytes) {
        most[&b] = std::max(most[&b], bytes);
        return 0;
    };
    for (Plan pl : plans) {
        plan_launch(ctx, pl);
        input_buffers(pl.P, host_coords ? &ctx->coords : nullptr, &ctx->assign64, mx);
        input_buffers(pl.P, host_coords ? &ctx->coords_alt : nullptr, &ctx->assign64_alt, mx);
        prep_buffers(ctx, pl, mx);
        sample_buffers(ctx, pl, mx);
        refine_buffers(ctx, pl.P, 1, pick_group(ctx, pl.P, 1), true, mx);
        if (backward) {
            refine_buffers(ctx, pl.P, pl.P.M, 0, true, mx);
            backward_buffers(ctx, pl.P, true, mx);
        }
    }
    for (auto& m : most) NEED(*m.first, m.second);
    return 0;
}

#undef NEED

int reserve_forward_batch(esacb200_ctx* ctx, const std::vector<Plan>& plans, bool host_coords, bool backward) {
    return forward_workspace(ctx, plans, host_coords, grow(ctx), backward);
}

// All B pointers of one argument on the device, or all on the host (a mix is an error).  None may be null.
int pointer_kind(esacb200_ctx* ctx, const void* const* p, int B, const char* what, bool& device) {
    for (int b = 0; b < B; ++b) {
        if (!p[b]) return fail(ctx, ESACB200_ERR_ARG, "image %d: %s is null", b, what);
        const bool d = is_device_ptr(p[b]);
        if (b == 0) device = d;
        else if (d != device)
            return fail(ctx, ESACB200_ERR_ARG, "%s mixes host and device pointers (image 0: %s, image %d: %s)", what,
                        device ? "device" : "host", b, d ? "device" : "host");
    }
    return 0;
}

// The last-call record of a call whose (last) problem `pl` was drawn and scored; `losses`: esac.backward's losses too.
void record_draw(esacb200_ctx* ctx, const Plan& pl, bool losses) {
    const SampleSizes z = sample_sizes(ctx, pl);
    LastCall& l = ctx->last;
    l.M = pl.P.M;
    l.drew = l.scored = true;
    l.lanes = z.G;
    l.lane_cap = z.Mg;
    l.losses = losses;
}

// The end of a call that ran prep .. select on the context and synchronises once: after the copies the caller enqueued,
// read back the scalars and the first `stats_bytes` bytes of the statistics, wait, check the expert indices, fill the
// statistics and the last-call record (`drew`: the call drew `pl`'s hypotheses, and used up any injected cells; `losses`:
// see record_draw) and take the stage times.
int finish_call(esacb200_ctx* ctx, const Plan& pl, size_t stats_bytes, bool drew, bool losses) {
    CK(cudaMemcpyAsync(ctx->pin->scalars, ctx->scalars.p, sizeof(ctx->pin->scalars), cudaMemcpyDeviceToHost, ctx->stream));
    if (stats_bytes) CK(cudaMemcpyAsync(&ctx->pin->stats, ctx->stats.p, stats_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    const int* hs = ctx->pin->scalars;
    if (hs[S_FLAGS]) return fail(ctx, ESACB200_ERR_ARG, "hypAssignment holds an expert index outside [0, %d)", pl.P.E);
    ctx->st.M = pl.P.M;
    ctx->st.winner = hs[S_WINNER];
    ctx->st.n_contrib = hs[S_NCONTRIB];
    if (stats_bytes) ctx->st.entropy = ctx->pin->stats.entropy;
    if (drew) {
        record_draw(ctx, pl, losses);
        ctx->inj_M = ctx->inj_T = 0;
    } else {
        ctx->last.M = pl.P.M;
        ctx->last.scored = true;
    }
    finish_stats(ctx);
    return 0;
}

// Hypothesis-major sharding: the planes that receive gradient on SOME rank (flags after the max-all-reduce, host copy in
// ctx->h_flags) are the only ones whose slices have to be summed over the ranks -- with a peaked gating that is one plane of
// twenty (3.7 of 74 MB at 480x640).  phase 0: zero those slices of the work buffer; phase 1: all-reduce them and add them to dst.
int for_flagged_planes(esacb200_ctx* ctx, int E, size_t plane, float* work, float* dst, int phase) {
    for (int e = 0; e < E;) {
        if (!ctx->h_flags[e]) { ++e; continue; }
        int e1 = e;
        while (e1 < E && ctx->h_flags[e1]) ++e1;
        float* w = work + (size_t)e * plane;
        const size_t n = (size_t)(e1 - e) * plane;
        if (phase == 0) {
            CK(cudaMemsetAsync(w, 0, n * sizeof(float), ctx->stream));
        } else {
            CKN(nccl_api().AllReduce(w, w, n, kNcclFloat32, kNcclSum, ctx->nccl_comm, ctx->stream));
            launch_add_inplace(dst + (size_t)e * plane, w, n, ctx->stream);
            ctx->st.kernel_launches += 2;
        }
        e = e1;
    }
    return 0;
}

// The gradient tensor the kernels accumulate into: `grads` itself on the device, else a copy of the host tensor in the
// workspace (d_grads != grads: the caller copies it back after the kernels).
int stage_grads(esacb200_ctx* ctx, float* grads, size_t bytes, float*& d_grads) {
    d_grads = grads;
    if (is_device_ptr(grads)) return 0;
    CK(ctx->grads.ensure(bytes));
    CK(cudaMemcpyAsync(ctx->grads.p, grads, bytes, cudaMemcpyHostToDevice, ctx->stream));
    d_grads = ctx->grads.as<float>();
    return 0;
}

// The hypotheses of a backward call: stage -> sample -> score -> select [-> exchange 1] -> refHyps = initHyps -> one read-back
// of n_contrib -> refinement of every contributing hypothesis (final inlier masks into `masks`, or the workspace when null).
// esac.backward and the hypotheses node both run it, so they draw, score and refine alike.
int run_hypotheses(esacb200_ctx* ctx, Plan& pl, const float* coords, const int64_t* assign, int64_t assign_stride,
                   const ShardSteps& sh, uint32_t* masks) {
    int rc = stage_inputs(ctx, pl, coords, assign, assign_stride);
    if (rc) return rc;
    const Problem& P = pl.P;
    const int M = P.M, E = P.E;
    int* sc = ctx->scalars.as<int>();
    const uint64_t seed = pl.async ? 0 : call_seed(ctx);
    rc = run_sample(ctx, pl, seed);
    if (rc) return rc;
    rc = run_score(ctx, pl);
    if (rc) return rc;
    if (sh.exchange) {
        // exchange 1 (SURVEY 8e): softmax normalisation over the hypotheses of ALL ranks
        double* x = ctx->pin->exchange;
        CK(cudaMemcpyAsync(x, &ctx->stats.as<CallStats>()->max_score, 2 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        double v[2] = {x[0], x[1]};
        if (sh.exchange(sh.user, 1, v, 2) != 0) return fail(ctx, ESACB200_ERR_ARG, "exchange callback failed (phase 1)");
        launch_rescale_probs(ctx->scores.as<double>(), P, v[0], v[1], ctx->probs.as<double>(), ctx->contrib.as<int>(),
                             sc + S_NCONTRIB, pl.min_prob, ctx->stream);
        ctx->st.kernel_launches += 1;
    } else if (sh.use_nccl) {
        // exchange 1 on the device: all-gather of the (max, sum exp) pairs, merged by the kernel that rebuilds the probabilities
        CK(ctx->gathered.ensure((size_t)ctx->comm_world * 2 * 8));
        CKN(nccl_api().AllGather(&ctx->stats.as<CallStats>()->max_score, ctx->gathered.p, 2, kNcclFloat64, ctx->nccl_comm, ctx->stream));
        launch_rescale_probs_gathered(ctx->scores.as<double>(), P, ctx->gathered.as<double>(), ctx->comm_world, nullptr,
                                      ctx->probs.as<double>(), ctx->contrib.as<int>(), sc + S_NCONTRIB, pl.min_prob, ctx->stream);
        ctx->st.kernel_launches += 2;
    }
    // refHyps = initHyps for everything below the floor (PROB_THRESH: esac.cpp:331-334)
    CK(cudaMemcpyAsync(ctx->poses_ref.p, ctx->poses.p, (size_t)M * sizeof(Pose), cudaMemcpyDeviceToDevice, ctx->stream));
    // Refining many hypotheses is fp64-throughput bound, so every SM should be busy and no CTA should wait at an inter-CTA
    // barrier longer than needed: one 4-byte read-back of the number of contributing hypotheses (a ~20 us stall on a
    // multi-millisecond call) lets the group size be coresident / jobs.  A stream-ordered call (pl.async) reads nothing back:
    // its refinement kernel picks the same group from the same count on the device (group 0).
    int group = 0;
    if (!pl.async) {
        CK(cudaMemcpyAsync(&ctx->pin->n_contrib, sc + S_NCONTRIB, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        if (sh.reduce_grads) {  // which planes receive gradient on some rank: rides on the same host synchronisation
            CK(ctx->eflags.ensure((size_t)E * sizeof(int)));
            launch_expert_flags(ctx->contrib.as<int>(), sc + S_NCONTRIB, ctx->assign32.as<int>(), E, ctx->eflags.as<int>(), ctx->stream);
            CKN(nccl_api().AllReduce(ctx->eflags.p, ctx->eflags.p, (size_t)E, kNcclInt32, kNcclMax, ctx->nccl_comm, ctx->stream));
            CK(cudaMemcpyAsync(ctx->h_flags, ctx->eflags.p, (size_t)E * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
            ctx->st.kernel_launches += 2;
        }
        CK(cudaStreamSynchronize(ctx->stream));
        if (sh.reduce_grads) {
            rc = for_flagged_planes(ctx, E, (size_t)3 * P.N, sh.d_work, sh.d_dst, 0);
            if (rc) return rc;
        }
        int n_jobs_now = ctx->pin->n_contrib;
        if (n_jobs_now < 1) n_jobs_now = 1;
        group = pick_group(ctx, P, n_jobs_now);
    }
    rc = run_refine(ctx, pl, ctx->poses.as<Pose>(), ctx->poses_ref.as<Pose>(), ctx->contrib.as<int>(), sc + S_NCONTRIB, 0, M, group,
                    masks);
    if (rc) return rc;
    mark(ctx, EV_REFINE);
    return 0;
}

// The context of the stream-ordered forward and backward, created on first use with ctx's seed (a capture may not create
// it: that allocates).
// The options are copied from ctx on every call.
// `what`: the entry point, forward_async or backward_async, named in the messages with its reserve call.
int async_context(esacb200_ctx* ctx, bool capturing, const char* what, esacb200_ctx** out) {
    if (!ctx->async) {
        if (capturing)
            return fail(ctx, ESACB200_ERR_ARG, "%s: the first call may not be captured; call reserve_%s (esacb200_reserve_%s) "
                                               "with the largest shape before capturing", what, what, what);
        esacb200_ctx* a = nullptr;
        int rc = esacb200_create(ctx->device, &a);
        if (rc) return fail(ctx, rc, "cannot create the context of the stream-ordered calls");
        a->is_async = true;
        if (a->seed_state.ensure(2 * sizeof(unsigned long long)) != cudaSuccess) {
            esacb200_destroy(a);
            cudaGetLastError();
            return fail(ctx, ESACB200_ERR_CUDA, "cannot allocate the seed state of the stream-ordered calls");
        }
        launch_seed_reset(a->seed_state.as<unsigned long long>(), ctx->seed, ctx->stream);
        ctx->async = a;
    }
    esacb200_ctx* a = ctx->async;
    a->stream = ctx->stream;
    // The two diagnostics stay off here and in the batch workers: they allocate and need a read-back, which a capture cannot
    // do, and their getters read the caller's context, not the one that ran the kernels.
    a->opt = ctx->opt;
    a->opt.refine_profile = a->opt.sample_trace = 0;
    *out = a;
    return 0;
}

int stream_capturing(esacb200_ctx* ctx, bool& capturing) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    CK(cudaStreamIsCapturing(ctx->stream, &cs));
    capturing = cs != cudaStreamCaptureStatusNone;
    return 0;
}

// Makes the async workspace hold `plans`: grows it when no capture has used it yet, else fails without touching it.
// backward: the workspace of the stream-ordered backward (forward_workspace's `backward`), else of the forward.  `name`: the
// entry point named in the message (null: the one of `backward`).
int async_workspace(esacb200_ctx* ctx, esacb200_ctx* a, const std::vector<Plan>& plans, bool capturing, bool backward,
                    const char* name) {
    const bool fits =
        forward_workspace(a, plans, false, [](DevBuf& b, size_t bytes) { return bytes <= b.cap ? 0 : 1; }, backward) == 0;
    if (fits) return 0;
    const Problem& P = plans[0].P;
    const char* what = backward ? "backward_async" : "forward_async";
    if (capturing || a->frozen)
        return fail(ctx, ESACB200_ERR_ARG,
                    "%s: E=%d H=%d W=%d M=%d needs more workspace than %s, and a graph that holds it may still be "
                    "replayed; call reserve_%s (esacb200_reserve_%s) with the largest shape before the "
                    "first capture", name ? name : what, P.E, P.H, P.W, P.M,
                    capturing ? "was reserved before this capture" : "an earlier capture used", what, what);
    int rc = reserve_forward_batch(a, plans, false, backward);
    if (rc) return fail(ctx, rc, "%s", a->err);
    return 0;
}

// The async context of reserve_`what`: a reserve call allocates, so it may not run while the stream is being captured.
int reserve_context(esacb200_ctx* ctx, const char* what, esacb200_ctx** out) {
    bool capturing = false;
    int rc = stream_capturing(ctx, capturing);
    if (rc) return rc;
    if (capturing) return fail(ctx, ESACB200_ERR_ARG, "reserve_%s allocates: call it before the capture", what);
    return async_context(ctx, false, what, out);
}

// The n named arguments are device memory (a null one is an error unless `optional` has its bit set).
int device_args(esacb200_ctx* ctx, const char* what, int n, const void* const* ptrs, const char* const* names, unsigned optional) {
    for (int i = 0; i < n; ++i) {
        if (!ptrs[i]) {
            if (optional >> i & 1) continue;
            return fail(ctx, ESACB200_ERR_ARG, "%s: %s is null", what, names[i]);
        }
        if (!is_device_ptr(ptrs[i])) return fail(ctx, ESACB200_ERR_ARG, "%s takes device pointers only: %s is host memory", what, names[i]);
    }
    return 0;
}

// The async context of a stream-ordered call on images of problem P, with its workspace fitted to them (async_workspace)
// and frozen when the stream is being captured.  backward: the workspace of the stream-ordered backward, else of the
// forward; `name`: the entry point named in the messages (null: the one of `backward`).
int enter_async(esacb200_ctx* ctx, const Problem& P, bool backward, const char* name, esacb200_ctx** out) {
    bool capturing = false;
    int rc = stream_capturing(ctx, capturing);
    if (rc) return rc;
    rc = async_context(ctx, capturing, backward ? "backward_async" : "forward_async", out);
    if (rc) return rc;
    rc = async_workspace(ctx, *out, std::vector<Plan>(1, Plan{P}), capturing, backward, name);
    if (rc) return rc;
    if (capturing) (*out)->frozen = true;
    return 0;
}

// What forward_async and backward_async (`backward`) share for B images of problem P: checks the arguments (the n arrays
// `ptrs`, called `names`, must be device memory), enters the async context and lays out the images.
// `name`: the entry point named in the messages (null: the one of `backward`); hypotheses_forward_async passes its own and
// uses the backward's workspace.
int begin_async(esacb200_ctx* ctx, bool backward, int B, const Problem& P, const float* coords, const int64_t* assign,
                int64_t assign_stride, const int32_t* shifts, const float* cameras, int32_t* out_status, int n,
                const void* const* ptrs, const char* const* names, AsyncCall& call, const char* name) {
    const char* what = name ? name : backward ? "backward_async" : "forward_async";
    int rc = device_args(ctx, what, n, ptrs, names);
    if (rc) return rc;
    rc = enter_async(ctx, P, backward, what, &call.a);
    if (rc) return rc;
    esacb200_ctx* a = call.a;
    // element stride between the assignments of consecutive images: rows of a [B, M] tensor
    const int64_t arow = assign_stride == 0 ? 0 : (int64_t)P.M * assign_stride;
    const size_t cstride = (size_t)P.E * 3 * P.N;
    call.plans.resize((size_t)B);
    call.imgs.resize((size_t)B);
    for (int b = 0; b < B; ++b) {
        Plan& pl = call.plans[b];
        pl.P = P;
        pl.d_coords = coords + (size_t)b * cstride;
        pl.d_assign = (const long long*)assign + b * arow;
        pl.assign_stride = assign_stride;
        AsyncImage& im = call.imgs[b];
        im.dev.shift = shifts + 2 * (size_t)b;
        im.dev.cam = cameras + 3 * (size_t)b;
        im.dev.seed = a->seed_state.as<unsigned long long>();
        im.dev.index = b;
        im.dev.fixed_seed = a->opt.fixed_seed;
        im.status = out_status + b;
        im.advance = b == B - 1 ? B : 0;
        pl.async = &im;
    }
    return 0;
}

// -------------------------------------------------------------------------------------------------
// Batches.  Every image is an independent problem (SURVEY 8e: "images in a batch are fully independent"), so the images
// are dealt round-robin to a few worker contexts, each driven by its own host thread on its own stream: the small kernels of
// one image fill the gaps the host synchronisations of another leave.  Image b has its own map size; with `draws` the seeds
// are fixed per image before the images are dealt (image b draws what the b-th of B consecutive single-image calls would),
// so a worker runs its images largest first and its workspace grows at most once.  `image(w, b)` runs image b on worker
// context w.  Everything the caller queued on its stream (the experts' outputs) is visible to the workers.  The statistics
// of the call are those of the last image, with the wall time and kernel launches of the whole batch.
int run_batch(esacb200_ctx* ctx, int B, const int* H, const int* W, bool draws,
              const std::function<int(esacb200_ctx*, int)>& image) {
    ctx->last = LastCall();  // the per-hypothesis buffers the images write are the workers'
    CK(cudaStreamSynchronize(ctx->stream));
    std::vector<uint64_t> seeds((size_t)B);
    if (draws)
        for (int b = 0; b < B; ++b) seeds[b] = call_seed(ctx);
    const int nw = ctx->opt.batch_workers < B ? ctx->opt.batch_workers : B;
    while ((int)ctx->workers.size() < nw) {
        esacb200_ctx* w = nullptr;
        int rc = esacb200_create(ctx->device, &w);
        if (rc) return fail(ctx, rc, "cannot create batch worker context");
        ctx->workers.push_back(w);
    }
    std::vector<int> rcs((size_t)nw, 0), failed_at((size_t)nw, -1);
    std::vector<esacb200_stats> last((size_t)nw);
    std::vector<unsigned long long> launches((size_t)nw, 0);
    auto work = [&](int wi) {
        try {
        esacb200_ctx* w = ctx->workers[wi];
        cudaSetDevice(ctx->device);
        w->opt = ctx->opt;
        w->opt.fixed_seed = 1;
        w->opt.refine_profile = w->opt.sample_trace = 0;  // as in async_context
        // this worker's images (dealt round-robin), largest first: the workspace grows at most once
        std::vector<int> mine;
        for (int b = wi; b < B; b += nw) mine.push_back(b);
        std::stable_sort(mine.begin(), mine.end(), [&](int a, int c) { return (long long)H[a] * W[a] > (long long)H[c] * W[c]; });
        for (int b : mine) {
            w->seed = seeds[b];
            int rc = image(w, b);
            if (rc) { rcs[wi] = rc; failed_at[wi] = b; return; }
            launches[wi] += w->st.kernel_launches;
            if (b == B - 1) last[wi] = w->st;
        }
        } catch (...) {  // an exception escaping a std::thread would terminate the process
            rcs[wi] = ESACB200_ERR_ARG;
            failed_at[wi] = -1;
            snprintf(ctx->workers[wi]->err, sizeof(ctx->workers[wi]->err), "host-side failure in a batch worker");
        }
    };
    const auto t0 = std::chrono::steady_clock::now();
    if (nw == 1) {
        work(0);
    } else {
        std::vector<std::thread> th;
        for (int wi = 0; wi < nw; ++wi) th.emplace_back(work, wi);
        for (auto& t : th) t.join();
    }
    const double wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    for (int wi = 0; wi < nw; ++wi)
        if (rcs[wi]) return fail(ctx, rcs[wi], "image %d: %s", failed_at[wi], ctx->workers[wi]->err);
    ctx->st = last[(B - 1) % nw];
    unsigned long long total = 0;
    for (int wi = 0; wi < nw; ++wi) total += launches[wi];
    ctx->st.kernel_launches = total;
    ctx->st.ms_total = (float)wall_ms;
    return ESACB200_OK;
}

}  // namespace esacb200::capi

extern "C" {

int esacb200_get_sample_profile(esacb200_ctx* ctx, long long* out8) try {
    if (!ctx || !out8) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    for (int i = 0; i < 8; ++i) out8[i] = 0;
    int rc = last_call_left(ctx, ctx->last.drew, "sampling profile");
    if (rc) return rc;
    const SampleSizes z = sample_layout(ctx->last.M, ctx->last.lanes, ctx->last.lane_cap);
    const int G = z.G;
    CK(cudaStreamSynchronize(ctx->stream));
    for (int g = 0; g < G; ++g) {
        int c[SC_COUNT];
        CK(cudaMemcpy(c, lane_state(ctx, z, g).counters, sizeof(c), cudaMemcpyDeviceToHost));
        out8[0] += (unsigned)c[SC_PREFILTERED];
        out8[1] += (unsigned)c[SC_JUDGED];
        out8[2] = out8[2] > c[SC_WAVES] ? out8[2] : c[SC_WAVES];
        out8[3] += c[SC_UNRESOLVED];
        out8[4] += c[SC_STAGED];
        out8[6] += (unsigned)c[SC_CUT];
        out8[7] += (unsigned)c[SC_HINTS_REJECTED];
    }
    out8[5] = G;
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

}  // extern "C"
