// Host side of libesac_b200.so: context, workspace, stage orchestration, the C ABI of include/esac_b200.h.
//
// Orchestration follows esac_forward (esac.cpp:64-190) and esac_backward (esac.cpp:213-511) stage by
// stage; every stage is a CUDA kernel launched on one stream with no host round trip until the final
// 68-byte (forward) / 8-byte (backward) result copy.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <exception>
#include <functional>
#include <map>
#include <new>
#include <string>
#include <vector>
#include <thread>
#include <chrono>

#include "../../include/esac_b200.h"
#include "../../include/esac_b200_testhooks.h"
#include "esac_internal.h"
#include "esac_p3p_fast.cuh"
#include "esac_rng.cuh"

using namespace esacb200;

namespace {

// A device buffer that owns its memory: freed when the buffer dies (the owner destroys it on its device, after its stream).
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() {
        if (p) cudaFree(p);
    }
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    template <class T>
    T* as() const { return (T*)p; }
};

// The tunables of esacb200_set_option.
struct Options {
    int max_tries = 1000000;
    int max_ref_steps = 100;
    int fixed_seed = 0;
    int refine_group_opt = 0;
    int refine_pretest = 1;    // inlier selection: float pretest with a rounding-error bound, exact arithmetic only where in doubt
    int refine_compact = 1;    // LM evaluations over per-CTA inlier lists instead of predicated passes over all cells
    int refine_profile = 0;    // 1: block 0 of the refinement kernel records phase cycle counts (esacb200_get_refine_profile)
    int refine_jobs_per_group = 3;
    int sample_prefilter = 1;
    int sample_span0 = 256;       // tries per hypothesis in the first wave (a multiple of the 256-try pass of a prefilter CTA)
    float sample_window = 1.25f;  // later waves: window / acceptance rate
    int sample_waves = 6;         // launched unconditionally (empty ones cost ~6 us each); what is left after them goes to tail_kernel
    float sample_tail_boost = 1.f;  // window factor once <= 64 hypotheses are left in a lane (x2 more for <= 8)
    int sample_trace = 0;         // 1: prefilter / exact kernels of waves 0-31 stamp first-CTA-start / last-CTA-end times (esacb200_get_sample_trace)
    int sample_groups = 2;        // lanes of the sampling stage (third and fourth lane: no gain measured)
    int upload_split = 1;
    int hyp_offset = 0, hyp_stride = 1;
    int score_ppt_opt = 0, score_hc_opt = 0;
    int batch_workers = 8;
};

enum { EV_START = 0, EV_H2D, EV_PREP, EV_SAMPLE, EV_FOLD, EV_SCORE, EV_SELECT, EV_REFINE, EV_BWD, EV_END, EV_COUNT };

// What the last call on a context left in its per-hypothesis buffers: the getters read nothing else.  Every call clears it
// (begin_call, run_batch); only the code that writes those buffers sets it.
struct LastCall {
    int M = 0;
    bool drew = false;         // poses, cells, tries, probs, refined poses and the sampling lanes' counters
    int lanes = 0, lane_cap = 0;  // of the sampling stage (sample_sizes: G, Mg)
    bool scored = false;       // scores
    bool losses = false;       // esac.backward's per-hypothesis losses
};

// The context's pinned host memory: a member for each value a call reads back or uploads through it, so no two uses share
// bytes.
struct Pinned {
    ForwardRecord fwd;   // the forward record (esacb200_forward, forward_sharded)
    float gt[16];        // a device ground-truth pose (esac.backward)
    int scalars[8];      // the head of the scalars buffer (finish_call)
    int n_contrib;       // contributing hypotheses before the refinement (run_hypotheses)
    int gating_flags;    // the flags of esacb200_assign
    CallStats stats;     // the call statistics (finish_call; global_loss: backward_sharded_nccl without hypotheses)
    int rounds[2];       // head of the refinement rounds of esacb200_forward
    double exchange[3];  // this rank's contributions to the exchanges of a sharded backward, and their results
    double upload;       // the global expected loss from the exchange callback, on its way to CallStats::global_loss
};

}  // namespace

struct esacb200_ctx {
    int device = 0;
    int sm_count = 0;
    char dev_name[128] = {0};
    cudaStream_t own_stream = nullptr;
    cudaStream_t copy_stream = nullptr;
    cudaStream_t aux_stream = nullptr;   // second lane of the sampling stage
    cudaStream_t aux_more[2] = {nullptr, nullptr};  // third and fourth lane (option sample_groups)
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_join_more[2] = {nullptr, nullptr};
    cudaEvent_t ev_copied[2] = {nullptr, nullptr}, ev_consumed[2] = {nullptr, nullptr};
    cudaStream_t stream = nullptr;
    uint64_t seed = 1305;  // thread_rand.h:103
    uint64_t calls = 0;
    Options opt;
    int* h_flags = nullptr;    // pinned: per-expert "receives gradient on some rank" flags (hypothesis-major sharding)
    int h_flags_cap = 0;
    int refine_coresident = 0;
    char err[512] = {0};
    // workspace
    DevBuf coords, grads, assign64, assign32, counts, offsets, perm, slot_of, chunks, scalars, centres, poses, poses_ref,
        cells, tries, posepk, part, scores, probs, stats, contrib, masks, rounds, scratch, barrier, fwd_rec, inject,
        losses, red, hypgrad, job_of, gt, smp_int, smp_surv, smp_trace, clist, eflags, coords4, coords_alt, assign64_alt, out_batch, prof,
        contrib8, upstream;
    Pinned* pin = nullptr;
    int inj_M = 0, inj_T = 0;
    cudaEvent_t ev[EV_COUNT] = {nullptr};
    bool ev_used[EV_COUNT] = {false};
    esacb200_stats st;
    LastCall last;
    // NCCL communicator of the sharded entry points (esacb200_comm_init); the library is resolved at run time with dlopen
    void* nccl_comm = nullptr;
    int comm_world = 1, comm_rank = 0;
    DevBuf gathered, grads_work;
    std::vector<esacb200_ctx*> workers;  // lazily created contexts of esacb200_backward_batch (own stream + workspace each)
    // Stream-ordered forward and backward (esacb200_forward_async / _backward_async): their own context, so that eager calls
    // never touch the buffers a captured graph holds.  In that context: is_async = true, seed_state = device {base seed,
    // async calls}, and frozen once a capture has used the workspace (from then on nothing in it is freed or reallocated).
    esacb200_ctx* async = nullptr;
    bool is_async = false;
    bool frozen = false;
    DevBuf seed_state;
    // The stream-ordered losses' workspace (esacb200_reproj_loss_async / _coord_loss_async), in the async context: apart from
    // the forward's and the backward's, so that loss graphs and ESAC graphs do not size each other's buffers; loss_frozen
    // once a capture has used it.
    DevBuf loss_ws;
    bool loss_frozen = false;
};

namespace {

// Every entry point works on the context's device and leaves the caller's current device as it found it (torch reads the
// current device with cudaGetDevice: a library that silently switches it redirects the caller's later allocations).
struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int device) {
        if (cudaGetDevice(&prev) != cudaSuccess) { cudaGetLastError(); prev = -1; }
        if (prev != device) cudaSetDevice(device);
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
    DeviceGuard(const DeviceGuard&) = delete;
    DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// ---- NCCL, resolved at run time ---------------------------------------------------------------------------------
// The library must load on machines without NCCL (the CPU test box) and must share the NCCL instance the host process already
// holds (torch bundles its own libnccl.so.2): no link-time dependency, dlopen of the soname instead -- RTLD_NOLOAD first, so an
// already loaded copy is reused.  Only the five entry points below are needed; their prototypes are NCCL's public ABI.
struct NcclApi {
    typedef struct { char internal[128]; } UniqueId;
    int (*GetUniqueId)(UniqueId*) = nullptr;
    int (*CommInitRank)(void**, int, UniqueId, int) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool ok = false;
};
constexpr int kNcclFloat32 = 7;  // ncclFloat
constexpr int kNcclFloat64 = 8;  // ncclDouble
constexpr int kNcclSum = 0;      // ncclSum
constexpr int kNcclInt32 = 2;    // ncclInt32
constexpr int kNcclMax = 2;      // ncclMax

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

int fail(esacb200_ctx* c, int code, const char* fmt, ...);
#define CKN(call)                                                                                              \
    do {                                                                                                       \
        int r__ = (call);                                                                                      \
        if (r__ != 0)                                                                                          \
            return fail(ctx, ESACB200_ERR_CUDA, "%s failed: %s (%s:%d)", #call,                                \
                        nccl_api().GetErrorString ? nccl_api().GetErrorString(r__) : "NCCL error", __FILE__, __LINE__); \
    } while (0)

int fail(esacb200_ctx* c, int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(c->err, sizeof(c->err), fmt, ap);
    va_end(ap);
    return code;
}

#define CK(call)                                                                                          \
    do {                                                                                                  \
        cudaError_t e__ = (call);                                                                         \
        if (e__ != cudaSuccess)                                                                           \
            return fail(ctx, ESACB200_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), \
                        __FILE__, __LINE__);                                                              \
    } while (0)

bool is_device_ptr(const void* p) {
    cudaPointerAttributes a;
    cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

void mark(esacb200_ctx* c, int id) {
    if (c->is_async) return;  // no stage timers for stream-ordered calls: they would need a synchronisation to read
    cudaEventRecord(c->ev[id], c->stream);
    c->ev_used[id] = true;
}

float span(esacb200_ctx* c, int a, int b) {
    if (!c->ev_used[a] || !c->ev_used[b]) return 0.f;
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, c->ev[a], c->ev[b]) != cudaSuccess) {
        cudaGetLastError();
        return 0.f;
    }
    return ms;
}

// scalars buffer layout (ints): [0]=n_chunks [1]=work_counter [2]=flags [3]=winner [4]=n_contrib
enum { S_NCHUNKS = 0, S_WORK, S_FLAGS, S_WINNER, S_NCONTRIB, S_COUNT = 16 };

struct Plan {
    Problem P;
    int T, ppt, hc, grid, vec_ok;
    const float* d_coords = nullptr;
    const long long* d_assign;
    long long assign_stride;
    int split_e = 0;  // > 0: host maps are uploaded in two halves [0, split_e) / [split_e, E) on the copy stream (ev_copied[0/1])
    const struct AsyncImage* async = nullptr;  // stream-ordered call: device parameters and the caller's outputs
    double min_prob = kProbThresh;  // the hypotheses with !(p < min_prob) contribute (the hypotheses node's floor)
};

// One image of a stream-ordered forward or backward: what its kernels read from device memory, and where its results go.
struct AsyncImage {
    DevParams dev;
    float* pose;        // [4,4] (forward)
    long long* expert;  // (forward)
    double* loss;       // (backward) esac.backward's return value
    const float* gt;    // (backward) [4,4] camera->world ground truth
    int* status;
    int advance;        // the last image of an execution: advance the async call counter by B
};

// Whether a call draws hypotheses from its problem, and whether it draws the context's injected cells (esacb200_inject_cells)
// when there are any; a call that draws ignores or clears them otherwise.
enum Draw { NO_DRAW, DRAWS, DRAWS_INJECTED };

int fill_problem(esacb200_ctx* ctx, Problem& P, int E, int H, int W, int M, int shiftX, int shiftY, float f, float ppx,
                 float ppy, float tau, float alpha, float beta, float maxReproj, int sub, Draw draw) {
    if (E <= 0 || H <= 0 || W <= 0 || M <= 0) return fail(ctx, ESACB200_ERR_ARG, "empty tensor (E=%d H=%d W=%d M=%d)", E, H, W, M);
    if ((long long)H * W > (1ll << 30)) return fail(ctx, ESACB200_ERR_ARG, "coordinate map too large");
    if (draw != NO_DRAW && (long long)(W - 1) * (H - 1) < 4)
        return fail(ctx, ESACB200_ERR_ARG, "map %dx%d too small to draw 4 distinct cells from [0,W-2]x[0,H-2]", W, H);
    if (draw == DRAWS_INJECTED && ctx->inj_M && ctx->inj_M != M)
        return fail(ctx, ESACB200_ERR_ARG, "injected cells are for M=%d, call has M=%d", ctx->inj_M, M);
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

auto grow(esacb200_ctx* ctx) {
    return [ctx](DevBuf& b, size_t bytes) -> int {
        CK(b.ensure(bytes));
        return 0;
    };
}

// Input staging: a host coordinate map goes to `cbuf`, host assignments to `abuf` (null: that input is not staged).
template <class Need>
int input_buffers(const Problem& P, DevBuf* cbuf, DevBuf* abuf, Need&& need) {
    if (cbuf) NEED(*cbuf, (size_t)P.E * 3 * P.N * sizeof(float));
    if (abuf) NEED(*abuf, (size_t)P.M * 8);
    return 0;
}

// Upload (or alias) the inputs.  Host coordinate maps go to `cbuf` on `copy_stream` (pinned memory: asynchronous).
int upload_inputs(esacb200_ctx* ctx, Plan& pl, const float* coords, const int64_t* assign, int64_t stride, DevBuf& cbuf,
                  DevBuf& abuf, cudaStream_t copy_stream, bool allow_split = false) {
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
void plan_launch(esacb200_ctx* ctx, Plan& pl) {
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
int prep_buffers(esacb200_ctx* ctx, const Plan& pl, Need&& need) {
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

int stage_inputs(esacb200_ctx* ctx, Plan& pl, const float* coords, const int64_t* assign, int64_t stride, bool allow_split = false) {
    int rc = upload_inputs(ctx, pl, coords, assign, stride, ctx->coords, ctx->assign64, ctx->stream, allow_split);
    if (rc) return rc;
    mark(ctx, EV_H2D);
    return plan_and_prep(ctx, pl);
}

constexpr int kSampleCap = 1 << 19;     // survivors per lane
constexpr int kSampleCapAcc = 1 << 15;  // staged accepts per lane

// Lanes of the sampling stage and its workspace: ints (smp_int) and survivor / staging bytes (smp_surv).
struct SampleSizes {
    int G, Mg;
    size_t per_group_ints, int_bytes, per_group_bytes, surv_bytes;
};
SampleSizes sample_sizes(const esacb200_ctx* ctx, const Plan& pl) {
    const Problem& P = pl.P;
    SampleSizes z;
    // two lanes pay once a wave's kernels are long enough to overlap (full-resolution maps, or very many hypotheses)
    const int groups = ctx->opt.sample_groups;
    int G = pl.split_e ? 2 : ((groups > 1 && ctx->aux_stream && P.M >= 64 && (P.N >= 65536 || P.M >= 1024)) ? groups : 1);
    if (G > 2 && (!ctx->aux_more[0] || !ctx->aux_more[1] || P.M < 512)) G = 2;
    z.G = G;
    z.Mg = pl.split_e ? P.M : (P.M + G - 1) / G;  // capacity of a lane's work list
    // ints: [best: 2M] [base: M] [ovf: M] then per group [list: 2*Mg] [counters: SC_COUNT]
    z.per_group_ints = (size_t)2 * z.Mg + SC_COUNT;
    z.int_bytes = ((size_t)P.M * 4 + G * z.per_group_ints) * 4 + 8;
    z.per_group_bytes = (size_t)kSampleCap * sizeof(int2) + (size_t)kSampleCapAcc * sizeof(Accepted);
    z.surv_bytes = G * z.per_group_bytes;
    return z;
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

int run_sample(esacb200_ctx* ctx, const Plan& pl, uint64_t seed) {
    const Problem& P = pl.P;
    const Options& o = ctx->opt;
    const int cap = kSampleCap;
    const int cap_acc = kSampleCapAcc;
    const SampleSizes z = sample_sizes(ctx, pl);
    const int G = z.G, Mg = z.Mg;
    const size_t per_group_ints = z.per_group_ints, per_group_bytes = z.per_group_bytes;
    int rc = sample_buffers(ctx, pl, grow(ctx));
    if (rc) return rc;
    SampleState st[4];
    int* b = ctx->smp_int.as<int>() + 2 * (size_t)P.M;
    for (int g = 0; g < G; ++g) {
        st[g].best = ctx->smp_int.as<unsigned long long>();  // 8-byte aligned: first in the buffer
        st[g].base = b;
        st[g].ovf = b + P.M;
        st[g].list = b + 2 * (size_t)P.M + g * per_group_ints;
        st[g].counters = st[g].list + 2 * (size_t)Mg;
        char* sb = (char*)ctx->smp_surv.p + g * per_group_bytes;
        st[g].surv = (int2*)sb;
        st[g].stage = (Accepted*)(sb + (size_t)cap * sizeof(int2));
        st[g].cap = cap;
        st[g].cap_acc = cap_acc;
        st[g].M = Mg;
    }
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
                                             pl.async ? &pl.async->dev : nullptr);
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

// masks_out: where the final inlier masks go ([max_jobs][2][words]); null = the context's workspace.
int run_refine(esacb200_ctx* ctx, const Plan& pl, const Pose* in, Pose* out, const int* d_jobs, const int* d_njobs,
               int n_jobs_host, int max_jobs, int group, uint32_t* masks_out = nullptr) {
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

// sample -> score -> select -> refine(winner) -> the forward record (rank aside) into d_rec; no sync.
// A stream-ordered image (pl.async) takes its seed from device memory and writes the caller's arrays instead.
int enqueue_forward_core(esacb200_ctx* ctx, const Plan& pl, ForwardRecord* d_rec) {
    const Problem& P = pl.P;
    int* sc = ctx->scalars.as<int>();
    const uint64_t seed = pl.async ? 0 : call_seed(ctx);
    int rc = run_sample(ctx, pl, seed);
    if (rc) return rc;
    rc = run_score(ctx, pl);
    if (rc) return rc;
    const int group = pick_group(ctx, P, 1);
    rc = run_refine(ctx, pl, ctx->poses.as<Pose>(), ctx->poses_ref.as<Pose>(), sc + S_WINNER, nullptr, 1, 1, group);
    if (rc) return rc;
    mark(ctx, EV_REFINE);
    if (pl.async)
        launch_finish_forward_async(ctx->poses_ref.as<Pose>(), sc + S_WINNER, ctx->assign32.as<int>(), sc + S_FLAGS, pl.async->pose,
                                    pl.async->expert, pl.async->status, ctx->seed_state.as<unsigned long long>(), pl.async->advance,
                                    ctx->stream);
    else
        launch_finish_forward(ctx->poses_ref.as<Pose>(), sc + S_WINNER, ctx->assign32.as<int>(), sc + S_FLAGS, d_rec, ctx->stream);
    ctx->st.kernel_launches += 1;
    return 0;
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

// Sizes every workspace buffer of the forward pipeline (upload, plan_and_prep, sampling, refinement) for the largest of a
// batch's images before the first one is enqueued: DevBuf::ensure growing mid-batch frees the old buffer, and cudaFree
// synchronises the device, which would serialise the copy stream's overlap with the previous image.
// `need(buf, bytes)` is called once per buffer with the largest size any image needs; reserve_forward_batch grows them, the
// stream-ordered forward also checks them.  (host_coords: the images' maps are staged, double-buffered.)  backward: also the
// stream-ordered backward's buffers -- the refinement of up to M jobs with its group picked on the device (every group a
// job count may pick) and backward_buffers.
template <class Need>
int forward_workspace(esacb200_ctx* ctx, const std::vector<Plan>& plans, bool host_coords, Need&& need, bool backward = false) {
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

int reserve_forward_batch(esacb200_ctx* ctx, const std::vector<Plan>& plans, bool host_coords, bool backward = false) {
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

// The B image pointers of a stacked [B, ...] tensor whose images lie `stride` elements apart (a null base: B nulls).
template <class T>
std::vector<T*> slices(T* base, int B, size_t stride) {
    std::vector<T*> p((size_t)B, nullptr);
    for (int b = 0; base && b < B; ++b) p[b] = base + (size_t)b * stride;
    return p;
}

// The tape of a hypotheses forward of problem P: at least tape_bytes large, 16-byte aligned device memory.
int check_tape(esacb200_ctx* ctx, const void* tape, size_t bytes, const Problem& P) {
    const size_t need = tape_bytes(P.M, P.N);
    if (bytes < need) return fail(ctx, ESACB200_ERR_ARG, "tape holds %zu bytes, this call needs %zu", bytes, need);
    if (!is_device_ptr(tape) || ((uintptr_t)tape & 15)) return fail(ctx, ESACB200_ERR_ARG, "tape must be 16-byte aligned device memory");
    return 0;
}

// Offsets of B host images packed into one device buffer, each at a 16-byte aligned offset (so that an image keeps the
// 128-bit load path a single-image call would give it).  Returns the total.
size_t pack_offsets(const std::vector<size_t>& bytes, std::vector<size_t>& off) {
    size_t total = 0;
    off.resize(bytes.size());
    for (size_t b = 0; b < bytes.size(); ++b) {
        off[b] = total;
        total += (bytes[b] + 15) & ~(size_t)15;
    }
    return total;
}

// Copies between B host images and their packed device copies; runs of images that lie back to back on both sides go as
// one copy (a stacked tensor with N % 4 == 0 is a single copy).
int copy_packed(esacb200_ctx* ctx, char* const* host, const std::vector<size_t>& bytes, const std::vector<size_t>& off, char* dev,
                bool to_device, cudaStream_t stream) {
    const size_t B = bytes.size();
    for (size_t b = 0; b < B;) {
        size_t e = b + 1, len = bytes[b];
        while (e < B && host[e] == host[e - 1] + bytes[e - 1] && off[e] == off[e - 1] + bytes[e - 1]) len += bytes[e++];
        if (to_device) CK(cudaMemcpyAsync(dev + off[b], host[b], len, cudaMemcpyHostToDevice, stream));
        else CK(cudaMemcpyAsync(host[b], dev + off[b], len, cudaMemcpyDeviceToHost, stream));
        b = e;
    }
    return 0;
}

// Stages the B images of one argument on the device: device pointers are used as they are; host images are packed into
// `buf` at 16-byte aligned offsets (and copied there when `upload`).  dev[b] receives image b's device address.
template <class T>
int stage_images(esacb200_ctx* ctx, T* const* ptrs, const std::vector<size_t>& bytes, bool device, bool upload, DevBuf& buf,
                 std::vector<T*>& dev, std::vector<size_t>& off) {
    const size_t B = bytes.size();
    dev.resize(B);
    if (device) {
        for (size_t b = 0; b < B; ++b) dev[b] = ptrs[b];
        return 0;
    }
    CK(buf.ensure(pack_offsets(bytes, off)));
    for (size_t b = 0; b < B; ++b) dev[b] = (T*)((char*)buf.p + off[b]);
    if (upload) return copy_packed(ctx, (char* const*)ptrs, bytes, off, (char*)buf.p, true, ctx->stream);
    return 0;
}

// Orders a loss call's per-image records by load path (128-bit first) so that each path is one launch over a contiguous
// slice of the table; returns the bytes of the table.
template <class Rec>
size_t order_by_path(const std::vector<Rec>& recs, const std::vector<char>& vec, std::vector<Rec>& out, int& n_vec, int& max_vec,
                     int& max_sc) {
    out.clear();
    n_vec = max_vec = max_sc = 0;
    for (size_t i = 0; i < recs.size(); ++i)
        if (vec[i]) { out.push_back(recs[i]); ++n_vec; if (recs[i].blocks > max_vec) max_vec = recs[i].blocks; }
    for (size_t i = 0; i < recs.size(); ++i)
        if (!vec[i]) { out.push_back(recs[i]); if (recs[i].blocks > max_sc) max_sc = recs[i].blocks; }
    return out.size() * sizeof(Rec);
}

void begin_call(esacb200_ctx* ctx) {
    memset(&ctx->st, 0, sizeof(ctx->st));
    ctx->last = LastCall();
    for (int i = 0; i < EV_COUNT; ++i) ctx->ev_used[i] = false;
    ctx->err[0] = 0;
    mark(ctx, EV_START);
}

void finish_stats(esacb200_ctx* ctx) {
    esacb200_stats& s = ctx->st;
    s.ms_h2d = span(ctx, EV_START, EV_H2D);
    s.ms_prep = span(ctx, EV_H2D, EV_PREP);
    s.ms_sample = span(ctx, EV_PREP, EV_SAMPLE);
    s.ms_score = span(ctx, EV_FOLD, EV_SCORE);
    s.ms_select = span(ctx, EV_SCORE, EV_SELECT);
    s.ms_refine = span(ctx, EV_SELECT, EV_REFINE);
    s.ms_backward = span(ctx, EV_REFINE, EV_BWD);
    s.ms_total = span(ctx, EV_START, EV_END);
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

// How much of CallStats a call reads back: nothing, what the select kernel wrote (entropy .. n_contrib) or all of it.
constexpr size_t kNoStats = 0, kSelectStats = offsetof(CallStats, unused), kAllStats = sizeof(CallStats);

// The end of a call that ran prep .. select on the context and synchronises once: after the copies the caller enqueued,
// read back the scalars and the first `stats_bytes` bytes of the statistics, wait, check the expert indices, fill the
// statistics and the last-call record (`drew`: the call drew `pl`'s hypotheses, and used up any injected cells; `losses`:
// see record_draw) and take the stage times.
int finish_call(esacb200_ctx* ctx, const Plan& pl, size_t stats_bytes, bool drew, bool losses = false) {
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


}  // namespace

// No C++ exception may cross the C ABI (std::vector / std::thread can throw): every entry point that allocates on the host is
// a function-try-block ending in this handler.
#define ESAC_ABI_CATCH(ctx)                                                                                   \
    catch (const std::exception& e) {                                                                         \
        return (ctx) ? fail((ctx), ESACB200_ERR_ARG, "host-side failure: %s", e.what()) : ESACB200_ERR_ARG;   \
    }                                                                                                         \
    catch (...) {                                                                                             \
        return (ctx) ? fail((ctx), ESACB200_ERR_ARG, "host-side failure (unknown exception)") : ESACB200_ERR_ARG; \
    }

// =================================================================================================
extern "C" {

int esacb200_create(int device, esacb200_ctx** out) {
    if (!out) return ESACB200_ERR_ARG;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) {
        cudaGetLastError();
        return ESACB200_ERR_NO_DEVICE;
    }
    esacb200_ctx* ctx = new (std::nothrow) esacb200_ctx();
    if (!ctx) return ESACB200_ERR_ARG;
    ctx->device = device;
    DeviceGuard device_guard(device);
    if (cudaSetDevice(device) != cudaSuccess) { delete ctx; return ESACB200_ERR_NO_DEVICE; }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { delete ctx; return ESACB200_ERR_CUDA; }
    ctx->sm_count = prop.multiProcessorCount;
    snprintf(ctx->dev_name, sizeof(ctx->dev_name), "%s", prop.name);
    if (cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return ESACB200_ERR_CUDA; }
    ctx->stream = ctx->own_stream;
    cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking);
    {
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        if (cudaStreamCreateWithPriority(&ctx->aux_stream, cudaStreamNonBlocking, hi) != cudaSuccess) { ctx->aux_stream = nullptr; cudaGetLastError(); }
        cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming);
        cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming);
        for (int i = 0; i < 2; ++i) {
            if (cudaStreamCreateWithPriority(&ctx->aux_more[i], cudaStreamNonBlocking, hi) != cudaSuccess) { ctx->aux_more[i] = nullptr; cudaGetLastError(); }
            cudaEventCreateWithFlags(&ctx->ev_join_more[i], cudaEventDisableTiming);
        }
    }
    for (int i = 0; i < 2; ++i) {
        cudaEventCreateWithFlags(&ctx->ev_copied[i], cudaEventDisableTiming);
        cudaEventCreateWithFlags(&ctx->ev_consumed[i], cudaEventDisableTiming);
    }
    for (int i = 0; i < EV_COUNT; ++i) cudaEventCreate(&ctx->ev[i]);
    cudaMallocHost((void**)&ctx->pin, sizeof(Pinned));
    ctx->refine_coresident = refine_max_coresident_blocks(ctx->sm_count);
    if (ctx->refine_coresident < 1) ctx->refine_coresident = 1;
    memset(&ctx->st, 0, sizeof(ctx->st));
    *out = ctx;
    return ESACB200_OK;
}

void esacb200_destroy(esacb200_ctx* ctx) {
    if (!ctx) return;
    for (esacb200_ctx* w : ctx->workers) esacb200_destroy(w);
    ctx->workers.clear();
    if (ctx->async) esacb200_destroy(ctx->async);
    ctx->async = nullptr;
    DeviceGuard device_guard(ctx->device);
    if (ctx->nccl_comm) { cudaStreamSynchronize(ctx->stream); nccl_api().CommDestroy(ctx->nccl_comm); ctx->nccl_comm = nullptr; }
    cudaStreamSynchronize(ctx->stream);
    for (int i = 0; i < EV_COUNT; ++i)
        if (ctx->ev[i]) cudaEventDestroy(ctx->ev[i]);
    if (ctx->pin) cudaFreeHost(ctx->pin);
    if (ctx->h_flags) cudaFreeHost(ctx->h_flags);
    for (int i = 0; i < 2; ++i) {
        if (ctx->ev_copied[i]) cudaEventDestroy(ctx->ev_copied[i]);
        if (ctx->ev_consumed[i]) cudaEventDestroy(ctx->ev_consumed[i]);
    }
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    if (ctx->aux_stream) cudaStreamDestroy(ctx->aux_stream);
    if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
    if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
    for (int i = 0; i < 2; ++i) {
        if (ctx->aux_more[i]) cudaStreamDestroy(ctx->aux_more[i]);
        if (ctx->ev_join_more[i]) cudaEventDestroy(ctx->ev_join_more[i]);
    }
    if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
    delete ctx;  // frees the workspace buffers (still on the context's device, after its stream has drained)
}

const char* esacb200_last_error(const esacb200_ctx* ctx) { return ctx ? ctx->err : "null context"; }

int esacb200_set_stream(esacb200_ctx* ctx, void* s) {
    if (!ctx) return ESACB200_ERR_ARG;
    ctx->stream = s ? (cudaStream_t)s : ctx->own_stream;
    return ESACB200_OK;
}

int esacb200_set_seed(esacb200_ctx* ctx, uint64_t seed) {
    if (!ctx) return ESACB200_ERR_ARG;
    ctx->seed = seed;
    ctx->calls = 0;
    if (ctx->async) {  // the stream-ordered calls' seed and call counter, in stream order
        DeviceGuard device_guard(ctx->device);
        launch_seed_reset(ctx->async->seed_state.as<unsigned long long>(), seed, ctx->stream);
        CK(cudaGetLastError());
    }
    return ESACB200_OK;
}

int esacb200_set_option(esacb200_ctx* ctx, const char* key, double v) {
    if (!ctx || !key) return ESACB200_ERR_ARG;
    Options& o = ctx->opt;
    if (!strcmp(key, "max_tries")) o.max_tries = v < 1 ? 1 : (int)v;
    else if (!strcmp(key, "max_ref_steps")) o.max_ref_steps = v < 0 ? 0 : (int)v;
    else if (!strcmp(key, "fixed_seed")) o.fixed_seed = v != 0;
    else if (!strcmp(key, "refine_group")) o.refine_group_opt = (int)v;
    else if (!strcmp(key, "refine_pretest")) o.refine_pretest = v != 0;
    else if (!strcmp(key, "refine_compact")) o.refine_compact = v != 0;
    else if (!strcmp(key, "refine_profile")) o.refine_profile = v != 0;
    else if (!strcmp(key, "refine_jobs_per_group")) o.refine_jobs_per_group = v < 1 ? 1 : (int)v;
    else if (!strcmp(key, "sample_prefilter")) o.sample_prefilter = v != 0;
    else if (!strcmp(key, "sample_tail_boost")) o.sample_tail_boost = v < 1 ? 1.f : (float)v;
    else if (!strcmp(key, "sample_trace")) o.sample_trace = v != 0;
    else if (!strcmp(key, "sample_span0")) o.sample_span0 = v < 256 ? 256 : ((int)v + 255) / 256 * 256;
    else if (!strcmp(key, "sample_window")) o.sample_window = v < 0.05 ? 0.05f : (float)v;
    else if (!strcmp(key, "sample_waves")) o.sample_waves = v < 0 ? 0 : (v > 64 ? 64 : (int)v);
    else if (!strcmp(key, "upload_split")) o.upload_split = v != 0;  // host maps in two halves, sampling under the second copy
    else if (!strcmp(key, "sample_groups")) o.sample_groups = v >= 4 ? 4 : (v >= 2 ? (int)v : 1);  // interleaved lanes, one stream each
    else if (!strcmp(key, "hyp_offset")) o.hyp_offset = (int)v;  // global index of local hypothesis 0 (sharded runs)
    else if (!strcmp(key, "hyp_stride")) o.hyp_stride = v < 1 ? 1 : (int)v;  // ... of local hypothesis h: offset + h * stride
    else if (!strcmp(key, "score_ppt")) o.score_ppt_opt = (int)v;   // 0 = automatic, else 2 / 4 / 8 cells per thread
    else if (!strcmp(key, "score_hc")) o.score_hc_opt = (int)v;     // 0 = automatic, else hypotheses per chunk (<= 64)
    else if (!strcmp(key, "batch_workers")) o.batch_workers = v < 1 ? 1 : (v > 16 ? 16 : (int)v);  // streams of backward_batch
    else return fail(ctx, ESACB200_ERR_ARG, "unknown option '%s'", key);
    return ESACB200_OK;
}

int esacb200_inject_cells(esacb200_ctx* ctx, const int32_t* cells, int M, int T) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!cells) { ctx->inj_M = ctx->inj_T = 0; return ESACB200_OK; }
    if (M <= 0 || T <= 0) return fail(ctx, ESACB200_ERR_ARG, "inject_cells: M and T must be positive");
    size_t bytes = (size_t)M * T * 8 * 4;
    CK(ctx->inject.ensure(bytes));
    CK(cudaMemcpy(ctx->inject.p, cells, bytes, cudaMemcpyHostToDevice));
    ctx->inj_M = M;
    ctx->inj_T = T;
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_device_info(esacb200_ctx* ctx, int* sm_count, char* name, int name_len) {
    if (!ctx) return ESACB200_ERR_ARG;
    if (sm_count) *sm_count = ctx->sm_count;
    if (name && name_len > 0) snprintf(name, name_len, "%s", ctx->dev_name);
    return ESACB200_OK;
}

// -------------------------------------------------------------------------------------------------
int esacb200_forward(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                     int64_t assign_stride, int M, float* out_pose, int shiftX, int shiftY, float f, float ppx,
                     float ppy, float tau, float alpha, float beta, float maxReproj, int sub, int* out_expert) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !assign || !out_pose) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    Plan pl;
    int rc = fill_problem(ctx, pl.P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS_INJECTED);
    if (rc) return rc;
    begin_call(ctx);
    rc = stage_inputs(ctx, pl, coords, assign, assign_stride, /*allow_split=*/!ctx->inj_M);
    if (rc) return rc;
    rc = enqueue_forward_core(ctx, pl, ctx->fwd_rec.as<ForwardRecord>());
    if (rc) return rc;
    Pinned& h = *ctx->pin;
    CK(cudaMemcpyAsync(&h.fwd, ctx->fwd_rec.p, offsetof(ForwardRecord, bad), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(h.rounds, ctx->rounds.p, sizeof(h.rounds), cudaMemcpyDeviceToHost, ctx->stream));
    if (is_device_ptr(out_pose)) CK(cudaMemcpyAsync(out_pose, ctx->fwd_rec.p, sizeof(h.fwd.pose), cudaMemcpyDeviceToDevice, ctx->stream));
    rc = finish_call(ctx, pl, kSelectStats, true);
    if (rc) return rc;
    if (!is_device_ptr(out_pose)) memcpy(out_pose, h.fwd.pose, sizeof(h.fwd.pose));
    if (out_expert) *out_expert = (int)h.fwd.expert;
    ctx->st.refine_rounds = h.rounds[0];
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
// Local half of a sharded forward: pipeline + record, no synchronisation (shared by forward_pack and forward_sharded).  The
// call begins (begin_record) before the shard's problem is filled, so bad sizes still clear the stats and the last-call
// record; M = 0 is a shard without hypotheses, whose problem is neither filled nor read.
static int begin_record(esacb200_ctx* ctx, int M, int M_pad) {
    if (M_pad < M || M_pad < 1) return fail(ctx, ESACB200_ERR_ARG, "M_pad (%d) must be >= M (%d) and >= 1", M_pad, M);
    begin_call(ctx);
    ctx->inj_M = ctx->inj_T = 0;
    return 0;
}

static int enqueue_forward_record(esacb200_ctx* ctx, const Problem& P, const float* coords, const int64_t* assign,
                                  int64_t assign_stride, int M, int M_pad, int expert_offset, double* pack_out) {
    Plan pl{P};
    if (M > 0) {
        int rc = stage_inputs(ctx, pl, coords, assign, assign_stride);
        if (rc) return rc;
        rc = enqueue_forward_core(ctx, pl, ctx->fwd_rec.as<ForwardRecord>());
        if (rc) return rc;
    } else {
        CK(ctx->scores.ensure(8));
        CK(ctx->fwd_rec.ensure(sizeof(ForwardRecord)));
    }
    launch_pack_forward(ctx->scores.as<double>(), ctx->fwd_rec.as<ForwardRecord>(), M, M_pad, expert_offset, ctx->opt.hyp_offset,
                        ctx->opt.hyp_stride, pack_out, ctx->stream);
    CK(cudaGetLastError());
    ctx->st.kernel_launches += 1;
    ctx->st.M = M;
    if (M > 0) record_draw(ctx, pl, false);
    return ESACB200_OK;
}

int esacb200_forward_pack(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                          int64_t assign_stride, int M, int M_pad, int shiftX, int shiftY, float f, float ppx, float ppy, float tau,
                          float alpha, float beta, float maxReproj, int sub, int expert_offset, double* pack_out) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!pack_out || (M > 0 && (!coords || !assign))) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    if ((M > 0 && (!is_device_ptr(coords) || !is_device_ptr(assign))) || !is_device_ptr(pack_out))
        return fail(ctx, ESACB200_ERR_ARG, "forward_pack takes device pointers only");
    Problem P = {};
    int rc = begin_record(ctx, M, M_pad);
    if (!rc && M > 0) rc = fill_problem(ctx, P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS);
    if (!rc) rc = enqueue_forward_record(ctx, P, coords, assign, assign_stride, M, M_pad, expert_offset, pack_out);
    if (rc) return rc;
    mark(ctx, EV_END);
    return ESACB200_OK;   // stage timers of this call are not collected: that would need the synchronisation
} ESAC_ABI_CATCH(ctx)

// ---- communicator -----------------------------------------------------------------------------------
int esacb200_nccl_unique_id(void* out128) {
    if (!out128) return ESACB200_ERR_ARG;
    NcclApi& n = nccl_api();
    if (!n.ok) return ESACB200_ERR_NO_DEVICE;
    NcclApi::UniqueId id;
    if (n.GetUniqueId(&id) != 0) return ESACB200_ERR_CUDA;
    memcpy(out128, id.internal, 128);
    return ESACB200_OK;
}

int esacb200_comm_init(esacb200_ctx* ctx, int world, int rank, const void* id128) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!id128 || world < 1 || rank < 0 || rank >= world) return fail(ctx, ESACB200_ERR_ARG, "bad communicator arguments");
    NcclApi& n = nccl_api();
    if (!n.ok) return fail(ctx, ESACB200_ERR_NO_DEVICE, "libnccl.so.2 cannot be loaded");
    if (ctx->nccl_comm) { n.CommDestroy(ctx->nccl_comm); ctx->nccl_comm = nullptr; }
    NcclApi::UniqueId id;
    memcpy(id.internal, id128, 128);
    CKN(n.CommInitRank(&ctx->nccl_comm, world, id, rank));
    ctx->comm_world = world;
    ctx->comm_rank = rank;
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_comm_destroy(esacb200_ctx* ctx) {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (ctx->nccl_comm) {
        cudaStreamSynchronize(ctx->stream);
        nccl_api().CommDestroy(ctx->nccl_comm);
        ctx->nccl_comm = nullptr;
    }
    ctx->comm_world = 1;
    ctx->comm_rank = 0;
    return ESACB200_OK;
}

// esac_forward with the experts / hypotheses sharded over the ranks of the communicator (SURVEY 8e): local pipeline ->
// record -> ONE ncclAllGather on the context's stream -> softMax / draw over all records on the device -> one 80-byte
// read-back.  Every rank returns the global winner's pose and expert.  M may be 0 (a shard without hypotheses); M_pad is
// the largest M of any rank (records must have one size).
int esacb200_forward_sharded(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                             int64_t assign_stride, int M, int M_pad, float* out_pose, int shiftX, int shiftY, float f, float ppx,
                             float ppy, float tau, float alpha, float beta, float maxReproj, int sub, int expert_offset,
                             int* out_expert) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!ctx->nccl_comm) return fail(ctx, ESACB200_ERR_ARG, "no communicator: call esacb200_comm_init first");
    if (!out_pose || (M > 0 && (!coords || !assign))) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    const int world = ctx->comm_world;
    const size_t rec = (size_t)M_pad + kPackTail;
    CK(ctx->gathered.ensure((world + 1) * rec * 8));
    double* mine = ctx->gathered.as<double>() + (size_t)world * rec;
    Problem P = {};
    int rc = begin_record(ctx, M, M_pad);
    if (!rc && M > 0) rc = fill_problem(ctx, P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS);
    if (!rc) rc = enqueue_forward_record(ctx, P, coords, assign, assign_stride, M, M_pad, expert_offset, mine);
    if (rc) return rc;
    CKN(nccl_api().AllGather(mine, ctx->gathered.p, rec, kNcclFloat64, ctx->nccl_comm, ctx->stream));
    launch_select_gathered(ctx->gathered.as<double>(), world, M_pad, ctx->fwd_rec.as<ForwardRecord>(), ctx->stream);
    CK(cudaGetLastError());
    ctx->st.kernel_launches += 2;
    Pinned& h = *ctx->pin;
    CK(cudaMemcpyAsync(&h.fwd, ctx->fwd_rec.p, sizeof(ForwardRecord), cudaMemcpyDeviceToHost, ctx->stream));
    if (is_device_ptr(out_pose)) CK(cudaMemcpyAsync(out_pose, ctx->fwd_rec.p, sizeof(h.fwd.pose), cudaMemcpyDeviceToDevice, ctx->stream));
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    if (h.fwd.bad != 0.f) return fail(ctx, ESACB200_ERR_ARG, "a shard's hypAssignment holds an expert index outside its experts");
    if (!is_device_ptr(out_pose)) memcpy(out_pose, h.fwd.pose, sizeof(h.fwd.pose));
    if (out_expert) *out_expert = (int)h.fwd.expert;
    ctx->st.winner = (int)h.fwd.winner;
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
// esac_forward over a batch of B images (BASELINE configs[2]: "batch 8 images").  The reference has no such entry: its
// callers loop over a DataLoader with batch_size=1 (test_esac.py:137).  Images are processed back to back on the compute
// stream with ONE host synchronisation at the end; host coordinate maps are double-buffered and copied on a second stream
// so the copy of image b+1 overlaps the kernels of image b.  Image b runs with its own map size, shift and camera: the
// pipeline of one image reads them from its Problem, so only the loop below sees the arrays.  The workspace is sized for
// the largest image before the first one is enqueued.
int esacb200_forward_ragged(esacb200_ctx* ctx, int B, const float* const* coords, const int* H, const int* W, int E,
                            const int64_t* assign, int64_t assign_stride, int M, float* out_poses, const int* shiftX,
                            const int* shiftY, const float* f, const float* ppx, const float* ppy, float tau, float alpha,
                            float beta, float maxReproj, int sub, int* out_experts) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !H || !W || !assign || !out_poses || B <= 0) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument or empty batch");
    if (!f || !ppx || !ppy) return fail(ctx, ESACB200_ERR_ARG, "null camera array");
    std::vector<Plan> plans;
    int rc = fill_problems(ctx, plans, B, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS);
    if (rc) return rc;
    bool dev_coords = false;
    rc = pointer_kind(ctx, (const void* const*)coords, B, "coords", dev_coords);
    if (rc) return rc;
    const bool host_coords = !dev_coords;
    begin_call(ctx);
    ctx->inj_M = ctx->inj_T = 0;
    rc = reserve_forward_batch(ctx, plans, host_coords);
    if (rc) return rc;
    // element stride between the assignments of consecutive images: rows of a [B, M] tensor
    const int64_t arow = assign_stride == 0 ? 0 : (int64_t)M * assign_stride;
    CK(ctx->out_batch.ensure((size_t)B * sizeof(ForwardRecord)));
    DevBuf* cb[2] = {&ctx->coords, &ctx->coords_alt};
    DevBuf* ab[2] = {&ctx->assign64, &ctx->assign64_alt};
    for (int b = 0; b < B; ++b) {
        const int buf = b & 1;
        Plan& pl = plans[b];
        if (host_coords && b >= 2) CK(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_consumed[buf], 0));
        rc = upload_inputs(ctx, pl, coords[b], assign + (size_t)b * arow, assign_stride, *cb[buf], *ab[buf],
                           host_coords ? ctx->copy_stream : ctx->stream);
        if (rc) return rc;
        if (host_coords) {
            CK(cudaEventRecord(ctx->ev_copied[buf], ctx->copy_stream));
            CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_copied[buf], 0));
        }
        if (b == 0) mark(ctx, EV_H2D);
        rc = plan_and_prep(ctx, pl);
        if (rc) return rc;
        rc = enqueue_forward_core(ctx, pl, ctx->out_batch.as<ForwardRecord>() + b);
        if (rc) return rc;
        if (host_coords) CK(cudaEventRecord(ctx->ev_consumed[buf], ctx->stream));
    }
    std::vector<ForwardRecord> host((size_t)B);
    CK(cudaMemcpyAsync(host.data(), ctx->out_batch.p, host.size() * sizeof(ForwardRecord), cudaMemcpyDeviceToHost, ctx->stream));
    const bool dev_out = is_device_ptr(out_poses);
    const size_t pose_bytes = sizeof(ForwardRecord::pose);
    if (dev_out)
        CK(cudaMemcpy2DAsync(out_poses, pose_bytes, ctx->out_batch.p, sizeof(ForwardRecord), pose_bytes, B, cudaMemcpyDeviceToDevice,
                             ctx->stream));
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    for (int b = 0; b < B; ++b) {
        const ForwardRecord& o = host[b];
        if (o.bad != 0.f) return fail(ctx, ESACB200_ERR_ARG, "image %d: hypAssignment holds an expert index outside [0, %d)", b, E);
        if (!dev_out) memcpy(out_poses + (size_t)b * 16, o.pose, pose_bytes);
        if (out_experts) out_experts[b] = (int)o.expert;
    }
    ctx->st.M = M;
    ctx->st.winner = (int)host[B - 1].winner;
    record_draw(ctx, plans[B - 1], false);  // the buffers hold the last image's hypotheses
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// B images of one shape: the pointer and size arrays of a [B,E,3,H,W] tensor.
int esacb200_forward_batch_cameras(esacb200_ctx* ctx, int B, const float* coords, int E, int H, int W, const int64_t* assign,
                                   int64_t assign_stride, int M, float* out_poses, const int* shiftX, const int* shiftY,
                                   const float* f, const float* ppx, const float* ppy, float tau, float alpha, float beta,
                                   float maxReproj, int sub, int* out_experts) try {
    if (!ctx) return ESACB200_ERR_ARG;
    if (!coords || !assign || !out_poses || B <= 0) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument or empty batch");
    if (!f || !ppx || !ppy) return fail(ctx, ESACB200_ERR_ARG, "null camera array");
    const auto ptrs = slices(coords, B, (size_t)E * 3 * H * W);  // (sizes are checked image by image by the ragged call)
    const std::vector<int> hs((size_t)B, H), ws((size_t)B, W);
    return esacb200_forward_ragged(ctx, B, ptrs.data(), hs.data(), ws.data(), E, assign, assign_stride, M, out_poses, shiftX, shiftY,
                                   f, ppx, ppy, tau, alpha, beta, maxReproj, sub, out_experts);
} ESAC_ABI_CATCH(ctx)

// One camera for the whole batch: broadcast to B entries.
int esacb200_forward_batch(esacb200_ctx* ctx, int B, const float* coords, int E, int H, int W, const int64_t* assign,
                           int64_t assign_stride, int M, float* out_poses, int shiftX, int shiftY, float f, float ppx,
                           float ppy, float tau, float alpha, float beta, float maxReproj, int sub, int* out_experts) try {
    if (!ctx) return ESACB200_ERR_ARG;
    const size_t n = B > 0 ? (size_t)B : 1;  // B <= 0 is rejected by the call below, with its usual message
    const std::vector<int> sx(n, shiftX), sy(n, shiftY);
    const std::vector<float> fs(n, f), cx(n, ppx), cy(n, ppy);
    return esacb200_forward_batch_cameras(ctx, B, coords, E, H, W, assign, assign_stride, M, out_poses, sx.data(), sy.data(),
                                          fs.data(), cx.data(), cy.data(), tau, alpha, beta, maxReproj, sub, out_experts);
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
// Stream-ordered forward.  The pipeline is enqueue_forward_core's, run in the context ctx->async with every image's seed,
// shift and camera read from device memory (AsyncImage), so a CUDA graph that captured the call replays with the values the
// arrays hold at replay time.  Nothing here synchronises, reads back or queries an event, and a call that a capture records
// allocates nothing.

// The context of the stream-ordered forward and backward, created on first use with ctx's seed (a capture may not create
// it: that allocates).
// The options are copied from ctx on every call.
// `what`: the entry point, forward_async or backward_async, named in the messages with its reserve call.
static int async_context(esacb200_ctx* ctx, bool capturing, const char* what, esacb200_ctx** out) {
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

static int stream_capturing(esacb200_ctx* ctx, bool& capturing) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    CK(cudaStreamIsCapturing(ctx->stream, &cs));
    capturing = cs != cudaStreamCaptureStatusNone;
    return 0;
}

// Makes the async workspace hold `plans`: grows it when no capture has used it yet, else fails without touching it.
// backward: the workspace of the stream-ordered backward (forward_workspace's `backward`), else of the forward.  `name`: the
// entry point named in the message (null: the one of `backward`).
static int async_workspace(esacb200_ctx* ctx, esacb200_ctx* a, const std::vector<Plan>& plans, bool capturing, bool backward,
                           const char* name = nullptr) {
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
static int reserve_context(esacb200_ctx* ctx, const char* what, esacb200_ctx** out) {
    bool capturing = false;
    int rc = stream_capturing(ctx, capturing);
    if (rc) return rc;
    if (capturing) return fail(ctx, ESACB200_ERR_ARG, "reserve_%s allocates: call it before the capture", what);
    return async_context(ctx, false, what, out);
}

// reserve_forward_async / reserve_backward_async (`backward`): sizes the async workspace for B images of one shape.
static int reserve_async(esacb200_ctx* ctx, int B, int E, int H, int W, int M, int sub, bool backward) {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = backward ? "backward_async" : "forward_async";
    if (B <= 0) return fail(ctx, ESACB200_ERR_ARG, "reserve_%s: empty batch (B=%d)", what, B);
    std::vector<Plan> plans(1);
    int rc = fill_problem(ctx, plans[0].P, E, H, W, M, 0, 0, 1.f, 0.f, 0.f, 1.f, 1.f, 1.f, 1.f, sub, NO_DRAW);
    if (rc) return rc;
    plans[0].d_coords = nullptr;  // the load path does not change the workspace
    esacb200_ctx* a = nullptr;
    if ((rc = reserve_context(ctx, what, &a))) return rc;
    return async_workspace(ctx, a, plans, false, backward);
}

// The n named arguments are device memory (a null one is an error unless `optional` has its bit set).
static int device_args(esacb200_ctx* ctx, const char* what, int n, const void* const* ptrs, const char* const* names, unsigned optional = 0) {
    for (int i = 0; i < n; ++i) {
        if (!ptrs[i]) {
            if (optional >> i & 1) continue;
            return fail(ctx, ESACB200_ERR_ARG, "%s: %s is null", what, names[i]);
        }
        if (!is_device_ptr(ptrs[i])) return fail(ctx, ESACB200_ERR_ARG, "%s takes device pointers only: %s is host memory", what, names[i]);
    }
    return 0;
}

// A stream-ordered call of B images of one shape: the async context, and per image its Plan and its AsyncImage (whose
// outputs the entry point fills in).
struct AsyncCall {
    esacb200_ctx* a = nullptr;
    std::vector<Plan> plans;
    std::vector<AsyncImage> imgs;
};

// What forward_async and backward_async (`backward`) share for B images of problem P: checks the arguments (the n arrays
// `ptrs`, called `names`, must be device memory), takes the async context, lays out the images and fits the workspace.
// `name`: the entry point named in the messages (null: the one of `backward`); hypotheses_forward_async passes its own and
// uses the backward's workspace.
static int begin_async(esacb200_ctx* ctx, bool backward, int B, const Problem& P, const float* coords, const int64_t* assign,
                       int64_t assign_stride, const int32_t* shifts, const float* cameras, int32_t* out_status, int n,
                       const void* const* ptrs, const char* const* names, AsyncCall& call, const char* name = nullptr) {
    const char* what = name ? name : backward ? "backward_async" : "forward_async";
    int rc = device_args(ctx, what, n, ptrs, names);
    if (rc) return rc;
    bool capturing = false;
    rc = stream_capturing(ctx, capturing);
    if (rc) return rc;
    rc = async_context(ctx, capturing, backward ? "backward_async" : "forward_async", &call.a);
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
    rc = async_workspace(ctx, a, call.plans, capturing, backward, what);
    if (rc) return rc;
    if (capturing) a->frozen = true;
    return 0;
}

int esacb200_reserve_forward_async(esacb200_ctx* ctx, int B, int E, int H, int W, int M, int sub) try {
    return reserve_async(ctx, B, E, H, W, M, sub, false);
} ESAC_ABI_CATCH(ctx)

int esacb200_forward_async(esacb200_ctx* ctx, int B, const float* coords, int E, int H, int W, const int64_t* assign,
                           int64_t assign_stride, int M, const int32_t* shifts, const float* cameras, float tau, float alpha,
                           float beta, float maxReproj, int sub, float* out_poses, int64_t* out_experts, int32_t* out_status) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const void* ptrs[] = {coords, assign, shifts, cameras, out_poses, out_experts, out_status};
    const char* names[] = {"coords", "assign", "shifts", "cameras", "out_poses", "out_experts", "out_status"};
    AsyncCall call;
    Problem P;
    int rc = B <= 0 ? fail(ctx, ESACB200_ERR_ARG, "forward_async: empty batch (B=%d)", B)
                    : fill_problem(ctx, P, E, H, W, M, 0, 0, 0.f, 0.f, 0.f, tau, alpha, beta, maxReproj, sub, DRAWS);
    if (!rc) rc = begin_async(ctx, false, B, P, coords, assign, assign_stride, shifts, cameras, out_status, 7, ptrs, names, call);
    if (rc) return rc;
    for (int b = 0; b < B; ++b) {
        call.imgs[b].pose = out_poses + 16 * (size_t)b;
        call.imgs[b].expert = (long long*)out_experts + b;
        rc = plan_and_prep(call.a, call.plans[b]);
        if (!rc) rc = enqueue_forward_core(call.a, call.plans[b], nullptr);
        if (rc) return fail(ctx, rc, "image %d: %s", b, call.a->err);
    }
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
int esacb200_score_poses(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                         int64_t assign_stride, int M, const double* poses6, int shiftX, int shiftY, float f, float ppx,
                         float ppy, float tau, float alpha, float beta, float maxReproj, int sub, double* out_scores) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !assign || !poses6 || !out_scores) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    Plan pl;
    int rc = fill_problem(ctx, pl.P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, NO_DRAW);
    if (rc) return rc;
    begin_call(ctx);
    rc = stage_inputs(ctx, pl, coords, assign, assign_stride);
    if (rc) return rc;
    CK(cudaMemcpyAsync(ctx->poses.p, poses6, (size_t)M * sizeof(Pose), cudaMemcpyHostToDevice, ctx->stream));
    mark(ctx, EV_SAMPLE);
    rc = run_score(ctx, pl);
    if (rc) return rc;
    CK(cudaMemcpyAsync(out_scores, ctx->scores.p, (size_t)M * 8, cudaMemcpyDeviceToHost, ctx->stream));
    return finish_call(ctx, pl, kNoStats, false);
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
int esacb200_refine_poses(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                          int64_t assign_stride, int M, double* poses6, int shiftX, int shiftY, float f, float ppx,
                          float ppy, float tau, float maxReproj, int sub, int* out_rounds, int* out_inliers) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !assign || !poses6) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    Plan pl;
    int rc = fill_problem(ctx, pl.P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, 100.f, 0.5f, maxReproj, sub, NO_DRAW);
    if (rc) return rc;
    begin_call(ctx);
    rc = stage_inputs(ctx, pl, coords, assign, assign_stride);
    if (rc) return rc;
    CK(cudaMemcpyAsync(ctx->poses.p, poses6, (size_t)M * sizeof(Pose), cudaMemcpyHostToDevice, ctx->stream));
    std::vector<int> jobs((size_t)M);
    for (int i = 0; i < M; ++i) jobs[i] = i;
    CK(cudaMemcpyAsync(ctx->contrib.p, jobs.data(), (size_t)M * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    const int group = pick_group(ctx, pl.P, M);
    mark(ctx, EV_SELECT);
    rc = run_refine(ctx, pl, ctx->poses.as<Pose>(), ctx->poses_ref.as<Pose>(), ctx->contrib.as<int>(), nullptr, M, M, group);
    if (rc) return rc;
    mark(ctx, EV_REFINE);
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    CK(cudaMemcpy(poses6, ctx->poses_ref.p, (size_t)M * sizeof(Pose), cudaMemcpyDeviceToHost));
    std::vector<int> rr((size_t)M * 2);
    CK(cudaMemcpy(rr.data(), ctx->rounds.p, (size_t)M * 8, cudaMemcpyDeviceToHost));
    const int words = (pl.P.N + 31) / 32;
    std::vector<uint32_t> mk;
    if (out_inliers) {
        mk.resize((size_t)M * 2 * words);
        CK(cudaMemcpy(mk.data(), ctx->masks.p, mk.size() * 4, cudaMemcpyDeviceToHost));
    }
    for (int i = 0; i < M; ++i) {
        if (out_rounds) out_rounds[i] = rr[2 * i];
        if (out_inliers) {
            int c = 0;
            if (rr[2 * i] > 0) {
                const uint32_t* m = mk.data() + ((size_t)i * 2 + rr[2 * i + 1]) * words;
                for (int w = 0; w < words; ++w) c += __builtin_popcount(m[w]);
            }
            out_inliers[i] = c;
        }
    }
    ctx->st.M = M;
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)


// Hypothesis-major sharding: the planes that receive gradient on SOME rank (flags after the max-all-reduce, host copy in
// ctx->h_flags) are the only ones whose slices have to be summed over the ranks -- with a peaked gating that is one plane of
// twenty (3.7 of 74 MB at 480x640).  phase 0: zero those slices of the work buffer; phase 1: all-reduce them and add them to dst.
static int ensure_host_flags(esacb200_ctx* ctx, int E) {
    if (ctx->h_flags_cap >= E + 1) return 0;
    if (ctx->h_flags) cudaFreeHost(ctx->h_flags);
    ctx->h_flags = nullptr; ctx->h_flags_cap = 0;
    CK(cudaMallocHost((void**)&ctx->h_flags, (size_t)(E + 1) * sizeof(int)));
    ctx->h_flags_cap = E + 1;
    return 0;
}
static int for_flagged_planes(esacb200_ctx* ctx, int E, size_t plane, float* work, float* dst, int phase) {
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
static int stage_grads(esacb200_ctx* ctx, float* grads, size_t bytes, float*& d_grads) {
    d_grads = grads;
    if (is_device_ptr(grads)) return 0;
    CK(ctx->grads.ensure(bytes));
    CK(cudaMemcpyAsync(ctx->grads.p, grads, bytes, cudaMemcpyHostToDevice, ctx->stream));
    d_grads = ctx->grads.as<float>();
    return 0;
}

// The sharded backward's steps inside the hypotheses prefix (none for a single-GPU call).
struct ShardSteps {
    esacb200_exchange_fn exchange = nullptr;  // host callback: softmax normalisation over all ranks
    void* user = nullptr;
    bool use_nccl = false;      // the same exchange as an all-gather on the device
    bool reduce_grads = false;  // hypothesis-major sharding: zero the work buffer's slices of the planes some rank updates
    float* d_work = nullptr;
    float* d_dst = nullptr;
};

// The hypotheses of a backward call: stage -> sample -> score -> select [-> exchange 1] -> refHyps = initHyps -> one read-back
// of n_contrib -> refinement of every contributing hypothesis (final inlier masks into `masks`, or the workspace when null).
// esac.backward and the hypotheses node both run it, so they draw, score and refine alike.
static int run_hypotheses(esacb200_ctx* ctx, Plan& pl, const float* coords, const int64_t* assign, int64_t assign_stride,
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

// The arguments of launch_backward that come from the context's workspace after run_hypotheses.
static BwdArgs backward_args(esacb200_ctx* ctx, const Plan& pl, float* grads) {
    const Problem& P = pl.P;
    int* sc = ctx->scalars.as<int>();
    BwdArgs b;
    b.coords = pl.d_coords;
    b.grads = grads;
    b.assign32 = ctx->assign32.as<int>();
    b.perm = ctx->perm.as<int>();
    b.counts = ctx->counts.as<int>();
    b.offsets = ctx->offsets.as<int>();
    b.init = ctx->poses.as<Pose>();
    b.ref = ctx->poses_ref.as<Pose>();
    b.cells = ctx->cells.as<int>();
    b.probs = ctx->probs.as<double>();
    b.contrib = ctx->contrib.as<int>();
    b.n_contrib = sc + S_NCONTRIB;
    b.job_of = ctx->job_of.as<int>();
    b.masks = ctx->masks.as<uint32_t>();
    b.mask_words = (P.N + 31) / 32;
    b.rounds = ctx->rounds.as<int>();
    b.losses = ctx->losses.as<double>();
    b.out_loss = &ctx->stats.as<CallStats>()->local_loss;
    b.red = ctx->red.as<double>();
    b.hyp_grad = ctx->hypgrad.p;
    b.P = P;
    b.expected_override = nullptr;
    return b;
}

// -------------------------------------------------------------------------------------------------
// esac.backward on one image of problem P (filled and checked by the caller); `sh`: the steps of a sharded call, whose
// work and destination buffers this fills in.
static int backward_impl(esacb200_ctx* ctx, const Problem& P, const float* coords, const int64_t* assign, int64_t assign_stride,
                         float* grads, const float* gt_pose, float wRot, float wTrans, float cut, ShardSteps sh, double* out_loss) {
    Plan pl{P};
    const int M = P.M, E = P.E;
    begin_call(ctx);
    const size_t cbytes = (size_t)P.E * 3 * P.N * sizeof(float);
    float* d_grads = nullptr;
    int rc = stage_grads(ctx, grads, cbytes, d_grads);
    if (rc) return rc;
    // hypothesis-major sharding: every rank holds all planes and a slice of the hypotheses, so the gradient slices overlap:
    // the local gradient goes to a zeroed work buffer, is summed over the ranks and only then added to the caller's tensor
    float* d_dst = d_grads;
    if (sh.reduce_grads) {
        CK(ctx->grads_work.ensure(cbytes));
        d_grads = ctx->grads_work.as<float>();  // (the slices that will be used are zeroed once they are known, below)
        rc = ensure_host_flags(ctx, E);
        if (rc) return rc;
    }
    sh.d_work = d_grads;
    sh.d_dst = d_dst;
    rc = run_hypotheses(ctx, pl, coords, assign, assign_stride, sh, nullptr);
    if (rc) return rc;
    rc = backward_buffers(ctx, P, true, grow(ctx));
    if (rc) return rc;
    BwdArgs b = backward_args(ctx, pl, d_grads);
    Pinned& h = *ctx->pin;
    CallStats* d_stats = ctx->stats.as<CallStats>();
    if (is_device_ptr(gt_pose)) {
        CK(cudaMemcpyAsync(h.gt, gt_pose, sizeof(h.gt), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        memcpy(b.gt, h.gt, sizeof(h.gt));
    } else {
        memcpy(b.gt, gt_pose, 16 * sizeof(float));
    }
    b.wRot = wRot; b.wTrans = wTrans; b.cut = cut;
    double global_loss = 0;
    if (sh.exchange) {
        // exchange 2: the expectation sum_h p_h loss_h runs over the hypotheses of all ranks (esac.cpp:357-362, esac_derivative.h:372-374)
        launch_backward_losses(b, ctx->stream);
        CK(cudaMemcpyAsync(h.exchange, &d_stats->local_loss, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        double v[1] = {h.exchange[0]};
        if (sh.exchange(sh.user, 2, v, 1) != 0) return fail(ctx, ESACB200_ERR_ARG, "exchange callback failed (phase 2)");
        global_loss = v[0];
        h.upload = v[0];
        CK(cudaMemcpyAsync(&d_stats->global_loss, &h.upload, sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        b.expected_override = &d_stats->global_loss;
        ctx->st.kernel_launches += 1;
    } else if (sh.use_nccl) {
        // exchange 2 on the device: all-reduce of the partial expectations, no host round trip
        launch_backward_losses(b, ctx->stream);
        CKN(nccl_api().AllReduce(&d_stats->local_loss, &d_stats->global_loss, 1, kNcclFloat64, kNcclSum, ctx->nccl_comm, ctx->stream));
        b.expected_override = &d_stats->global_loss;
        ctx->st.kernel_launches += 2;
    }
    launch_backward(b, M, ctx->sm_count, ctx->stream);
    CK(cudaGetLastError());
    ctx->st.kernel_launches += 5;
    if (sh.reduce_grads) {
        rc = for_flagged_planes(ctx, E, (size_t)3 * P.N, d_grads, d_dst, 1);
        if (rc) return rc;
        CK(cudaGetLastError());
        d_grads = d_dst;
    }
    mark(ctx, EV_BWD);
    if (d_grads != grads) CK(cudaMemcpyAsync(grads, d_grads, cbytes, cudaMemcpyDeviceToHost, ctx->stream));
    rc = finish_call(ctx, pl, kAllStats, true, /*losses=*/true);
    if (rc) return rc;
    if (sh.use_nccl) global_loss = h.stats.global_loss;
    ctx->st.expected_loss = (sh.exchange || sh.use_nccl) ? global_loss : h.stats.local_loss;
    if (out_loss) *out_loss = ctx->st.expected_loss;
    return ESACB200_OK;
}

int esacb200_backward(esacb200_ctx* ctx, const float* coords, float* grads, int E, int H, int W, const int64_t* assign,
                      int64_t assign_stride, int M, const float* gt_pose, float wRot, float wTrans, float cut, int shiftX,
                      int shiftY, float f, float ppx, float ppy, float tau, float alpha, float beta, float maxReproj, int sub,
                      double* out_loss) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !assign || !grads || !gt_pose) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    Problem P;
    int rc = fill_problem(ctx, P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS_INJECTED);
    return rc ? rc : backward_impl(ctx, P, coords, assign, assign_stride, grads, gt_pose, wRot, wTrans, cut, ShardSteps(), out_loss);
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
// Stream-ordered backward (esacb200_backward_async): esac.backward with the forward_async contract.  It runs in the same
// context as forward_async (ctx->async) and counts calls with it; the host path is the eager one, with the refinement group
// picked on the device from the number of contributing hypotheses.
int esacb200_reserve_backward_async(esacb200_ctx* ctx, int B, int E, int H, int W, int M, int sub) try {
    return reserve_async(ctx, B, E, H, W, M, sub, true);
} ESAC_ABI_CATCH(ctx)

int esacb200_backward_async(esacb200_ctx* ctx, int B, const float* coords, float* grads, int E, int H, int W,
                            const int64_t* assign, int64_t assign_stride, int M, const float* gt_poses, float wRot, float wTrans,
                            float cut, const int32_t* shifts, const float* cameras, float tau, float alpha, float beta,
                            float maxReproj, int sub, double* out_losses, int32_t* out_status) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const void* ptrs[] = {coords, grads, assign, gt_poses, shifts, cameras, out_losses, out_status};
    const char* names[] = {"coords", "grads", "assign", "gt_poses", "shifts", "cameras", "out_losses", "out_status"};
    AsyncCall call;
    Problem P;
    int rc = B <= 0 ? fail(ctx, ESACB200_ERR_ARG, "backward_async: empty batch (B=%d)", B)
                    : fill_problem(ctx, P, E, H, W, M, 0, 0, 0.f, 0.f, 0.f, tau, alpha, beta, maxReproj, sub, DRAWS);
    if (!rc) rc = begin_async(ctx, true, B, P, coords, assign, assign_stride, shifts, cameras, out_status, 8, ptrs, names, call);
    if (rc) return rc;
    esacb200_ctx* a = call.a;
    const size_t cstride = (size_t)E * 3 * H * W;
    for (int b = 0; b < B; ++b) {
        Plan& pl = call.plans[b];
        AsyncImage& im = call.imgs[b];
        im.loss = out_losses + b;
        im.gt = gt_poses + 16 * (size_t)b;
        rc = run_hypotheses(a, pl, pl.d_coords, (const int64_t*)pl.d_assign, assign_stride, ShardSteps(), nullptr);
        if (!rc) rc = backward_buffers(a, pl.P, true, grow(a));
        if (rc) return fail(ctx, rc, "image %d: %s", b, a->err);
        BwdArgs args = backward_args(a, pl, grads + (size_t)b * cstride);
        args.wRot = wRot; args.wTrans = wTrans; args.cut = cut;
        BwdDev dv;
        dv.gt = im.gt;
        dv.flags = a->scalars.as<int>() + S_FLAGS;
        dv.dev = im.dev;
        launch_backward(args, M, a->sm_count, a->stream, &dv);
        launch_finish_backward_async(a->stats.as<CallStats>(), a->scalars.as<int>() + S_FLAGS, im.loss, im.status,
                                     a->seed_state.as<unsigned long long>(), im.advance, a->stream);
        a->st.kernel_launches += 6;
    }
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
// The hypotheses as an autograd node: a forward that returns scores, refined poses and contributing flags and keeps what its
// backward needs in a caller-owned tape, and a backward that maps upstream gradients of (scores, poses) to the coordinates.
size_t esacb200_hypotheses_tape_bytes(int E, int H, int W, int M) {
    if (E <= 0 || H <= 0 || W <= 0 || M <= 0 || (long long)H * W > (1ll << 30)) return 0;
    return tape_bytes(M, H * W);
}

// The tape header of a hypotheses forward of problem P with probability floor min_prob.
static TapeHead tape_head(const Problem& P, double min_prob) {
    TapeHead head;
    memset(&head, 0, sizeof(head));
    head.magic = kTapeMagic;
    head.M = P.M;
    head.mask_words = (P.N + 31) / 32;
    head.P = P;
    head.min_prob = min_prob;
    return head;
}

static_assert(kProbThresh == ESACB200_PROB_THRESH, "the C ABI's default floor is the reference's PROB_THRESH");

// The hypotheses node's probability floor: a number in [0, 1] (NaN is refused).  `what`: the entry point, or null.
static int check_min_prob(esacb200_ctx* ctx, const char* what, double min_prob) {
    if (min_prob >= 0.0 && min_prob <= 1.0) return 0;
    return fail(ctx, ESACB200_ERR_ARG, "%s%smin_prob must lie in [0, 1], got %g", what ? what : "", what ? ": " : "", min_prob);
}

// The arguments of the tape's record kernel: the hypotheses of problem P that run_hypotheses left in ctx's workspace.
static BwdArgs tape_record_args(esacb200_ctx* ctx, const Problem& P) {
    BwdArgs b;
    memset(&b, 0, sizeof(b));
    b.assign32 = ctx->assign32.as<int>();
    b.init = ctx->poses.as<Pose>();
    b.ref = ctx->poses_ref.as<Pose>();
    b.cells = ctx->cells.as<int>();
    b.contrib = ctx->contrib.as<int>();
    b.n_contrib = ctx->scalars.as<int>() + S_NCONTRIB;
    b.rounds = ctx->rounds.as<int>();
    b.P = P;
    return b;
}

// The hypotheses forward of problem P (filled and checked by the caller, with the tape: check_tape, and the floor).
static int hypotheses_forward_impl(esacb200_ctx* ctx, const Problem& P, double min_prob, const float* coords, const int64_t* assign,
                                   int64_t assign_stride, void* tape, double* out_scores, double* out_poses6, uint8_t* out_contrib) {
    Plan pl{P};
    pl.min_prob = min_prob;
    const int M = P.M;
    begin_call(ctx);
    int rc = run_hypotheses(ctx, pl, coords, assign, assign_stride, ShardSteps(), (uint32_t*)((char*)tape + tape_masks_offset(M)));
    if (rc) return rc;
    CK(ctx->contrib8.ensure((size_t)M));
    CK(cudaMemsetAsync((char*)tape + kTapeTailOffset, 0, sizeof(TapeTail), ctx->stream));  // (a bad assignment fails the call)
    launch_tape_records(tape_record_args(ctx, P), tape_head(P, min_prob), tape, ctx->contrib8.as<unsigned char>(), ctx->stream);
    CK(cudaGetLastError());
    ctx->st.kernel_launches += 1;
    CK(cudaMemcpyAsync(out_scores, ctx->scores.p, (size_t)M * 8, cudaMemcpyDefault, ctx->stream));
    CK(cudaMemcpyAsync(out_poses6, ctx->poses_ref.p, (size_t)M * sizeof(Pose), cudaMemcpyDefault, ctx->stream));
    CK(cudaMemcpyAsync(out_contrib, ctx->contrib8.p, (size_t)M, cudaMemcpyDefault, ctx->stream));
    return finish_call(ctx, pl, kSelectStats, true);
}

int esacb200_hypotheses_forward_floor(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                                      int64_t assign_stride, int M, int shiftX, int shiftY, float f, float ppx, float ppy,
                                      float tau, float alpha, float beta, float maxReproj, int sub, double min_prob, void* tape,
                                      size_t tape_bytes_, double* out_scores, double* out_poses6, uint8_t* out_contrib) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !assign || !tape || !out_scores || !out_poses6 || !out_contrib) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    Problem P;
    int rc = check_min_prob(ctx, nullptr, min_prob);
    if (!rc) rc = fill_problem(ctx, P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS_INJECTED);
    if (!rc) rc = check_tape(ctx, tape, tape_bytes_, P);
    return rc ? rc : hypotheses_forward_impl(ctx, P, min_prob, coords, assign, assign_stride, tape, out_scores, out_poses6, out_contrib);
} ESAC_ABI_CATCH(ctx)

int esacb200_hypotheses_forward(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                                int64_t assign_stride, int M, int shiftX, int shiftY, float f, float ppx, float ppy, float tau,
                                float alpha, float beta, float maxReproj, int sub, void* tape, size_t tape_bytes_,
                                double* out_scores, double* out_poses6, uint8_t* out_contrib) {
    return esacb200_hypotheses_forward_floor(ctx, coords, E, H, W, assign, assign_stride, M, shiftX, shiftY, f, ppx, ppy, tau,
                                             alpha, beta, maxReproj, sub, ESACB200_PROB_THRESH, tape, tape_bytes_, out_scores,
                                             out_poses6, out_contrib);
}

// d_scores / d_poses6 are [rows, M] / [rows, M, 6] arrays (M of the tape) of which row `row` is this tape's upstream.
static int hypotheses_backward_impl(esacb200_ctx* ctx, const void* tape, const float* coords, float* grads, int E, int H, int W,
                                    const double* d_scores, const double* d_poses6, int row) {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!tape || !coords || !grads) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    if (!is_device_ptr(tape) || ((uintptr_t)tape & 15)) return fail(ctx, ESACB200_ERR_ARG, "tape must be 16-byte aligned device memory");
    // the header: problem and hypothesis count of the forward (ordered after the forward on this stream)
    TapeHead head;
    CK(cudaMemcpyAsync(&head, tape, sizeof(head), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (head.magic != kTapeMagic) return fail(ctx, ESACB200_ERR_ARG, "tape holds no hypotheses forward");
    const Problem P = head.P;
    if (P.E != E || P.H != H || P.W != W)
        return fail(ctx, ESACB200_ERR_ARG, "coordinates are [%d,3,%d,%d], the forward saw [%d,3,%d,%d]", E, H, W, P.E, P.H, P.W);
    const int M = head.M;
    if (d_scores) d_scores += (size_t)row * M;
    if (d_poses6) d_poses6 += (size_t)row * M * 6;
    begin_call(ctx);
    const size_t cbytes = (size_t)E * 3 * P.N * sizeof(float);
    const float* d_coords = coords;
    if (!is_device_ptr(coords)) {
        CK(ctx->coords.ensure(cbytes));
        CK(cudaMemcpyAsync(ctx->coords.p, coords, cbytes, cudaMemcpyHostToDevice, ctx->stream));
        d_coords = ctx->coords.as<float>();
    }
    float* d_grads = nullptr;
    int rc = stage_grads(ctx, grads, cbytes, d_grads);
    if (rc) return rc;
    // upstream gradients: [M] of the scores then [M,6] of the poses; an absent one is zero
    CK(ctx->upstream.ensure((size_t)M * 7 * 8));
    double* up = ctx->upstream.as<double>();
    if (d_scores) CK(cudaMemcpyAsync(up, d_scores, (size_t)M * 8, cudaMemcpyDefault, ctx->stream));
    else CK(cudaMemsetAsync(up, 0, (size_t)M * 8, ctx->stream));
    if (d_poses6) CK(cudaMemcpyAsync(up + M, d_poses6, (size_t)M * 6 * 8, cudaMemcpyDefault, ctx->stream));
    else CK(cudaMemsetAsync(up + M, 0, (size_t)M * 6 * 8, ctx->stream));
    mark(ctx, EV_REFINE);
    rc = backward_buffers(ctx, P, false, grow(ctx));
    if (rc) return rc;
    BwdArgs b;
    memset(&b, 0, sizeof(b));
    b.coords = d_coords;
    b.grads = d_grads;
    b.n_contrib = (const int*)((const char*)tape + offsetof(TapeHead, n_contrib));
    b.job_of = ctx->job_of.as<int>();
    b.masks = (const uint32_t*)((const char*)tape + tape_masks_offset(M));
    b.mask_words = head.mask_words;
    b.red = ctx->red.as<double>();
    b.hyp_grad = ctx->hypgrad.p;
    b.P = P;
    launch_backward_upstream(b, tape, up, up + M, M, ctx->sm_count, ctx->stream);
    CK(cudaGetLastError());
    ctx->st.kernel_launches += 5;
    mark(ctx, EV_BWD);
    if (d_grads != grads) CK(cudaMemcpyAsync(grads, d_grads, cbytes, cudaMemcpyDeviceToHost, ctx->stream));
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    ctx->st.M = M;
    ctx->st.n_contrib = head.n_contrib;
    finish_stats(ctx);
    return ESACB200_OK;
}

int esacb200_hypotheses_backward(esacb200_ctx* ctx, const void* tape, const float* coords, float* grads, int E, int H, int W,
                                 const double* d_scores, const double* d_poses6) try {
    return hypotheses_backward_impl(ctx, tape, coords, grads, E, H, W, d_scores, d_poses6, 0);
} ESAC_ABI_CATCH(ctx)

int esacb200_pose_loss_batch(esacb200_ctx* ctx, int B, int M, const double* poses6, const float* gt16, float wRot, float wTrans,
                             float cut, double* out_losses, double* out_dloss6) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!poses6 || !gt16 || !out_losses || !out_dloss6) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    if (M <= 0) return fail(ctx, ESACB200_ERR_ARG, "no poses (M=%d)", M);
    if (B <= 0 || B > 65535) return fail(ctx, ESACB200_ERR_ARG, "batch of %d images outside [1, 65535]", B);
    begin_call(ctx);
    const size_t n = (size_t)B * M;
    // [B,M] poses, [B,M] losses, [B,M,6] dLoss; the ground truths [B,4,4] in their own buffer
    CK(ctx->upstream.ensure(n * 13 * 8));
    CK(ctx->gt.ensure((size_t)B * 16 * sizeof(float)));
    double* buf = ctx->upstream.as<double>();
    CK(cudaMemcpyAsync(buf, poses6, n * sizeof(Pose), cudaMemcpyDefault, ctx->stream));
    CK(cudaMemcpyAsync(ctx->gt.p, gt16, (size_t)B * 16 * sizeof(float), cudaMemcpyDefault, ctx->stream));
    launch_pose_loss((const Pose*)buf, B, M, ctx->gt.as<float>(), wRot, wTrans, cut, buf + 6 * n, buf + 7 * n, ctx->stream);
    CK(cudaGetLastError());
    ctx->st.kernel_launches += 1;
    CK(cudaMemcpyAsync(out_losses, buf + 6 * n, n * 8, cudaMemcpyDefault, ctx->stream));
    CK(cudaMemcpyAsync(out_dloss6, buf + 7 * n, n * 6 * 8, cudaMemcpyDefault, ctx->stream));
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_pose_loss(esacb200_ctx* ctx, int M, const double* poses6, const float* gt16, float wRot, float wTrans, float cut,
                       double* out_losses, double* out_dloss6) {
    return esacb200_pose_loss_batch(ctx, 1, M, poses6, gt16, wRot, wTrans, cut, out_losses, out_dloss6);
}

// -------------------------------------------------------------------------------------------------
// The hypotheses node with the forward_async contract (esacb200_hypotheses_forward_async / _backward_async): the host path is
// the eager one, in the stream-ordered context, with the refinement group picked on the device; the record kernel writes the
// header from device-read values and the caller's outputs, and the backward checks the header on the device.  It uses the
// workspace of backward_async and its rule.

// Bytes between consecutive images' tapes: the tape rounded up to 256 bytes.
static size_t tape_stride(const Problem& P) { return (tape_bytes(P.M, P.N) + 255) & ~(size_t)255; }

// The tapes argument of B images: 16-byte aligned device memory of at least B strides.
static int check_tapes(esacb200_ctx* ctx, const char* what, const void* tapes, size_t bytes, int B, const Problem& P) {
    const size_t need = (size_t)B * tape_stride(P);
    if (bytes < need)
        return fail(ctx, ESACB200_ERR_ARG, "%s: tapes hold %zu bytes, %d image(s) of E=%d H=%d W=%d M=%d need %zu", what, bytes, B,
                    P.E, P.H, P.W, P.M, need);
    if ((uintptr_t)tapes & 15) return fail(ctx, ESACB200_ERR_ARG, "%s: tapes must be 16-byte aligned", what);
    return 0;
}

int esacb200_hypotheses_forward_async_floor(esacb200_ctx* ctx, int B, const float* coords, int E, int H, int W,
                                            const int64_t* assign, int64_t assign_stride, int M, const int32_t* shifts,
                                            const float* cameras, float tau, float alpha, float beta, float maxReproj, int sub,
                                            double min_prob, void* tapes, size_t tapes_bytes, double* out_scores,
                                            double* out_poses6, uint8_t* out_contrib, int32_t* out_status) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "hypotheses_forward_async";
    const void* ptrs[] = {coords, assign, shifts, cameras, tapes, out_scores, out_poses6, out_contrib, out_status};
    const char* names[] = {"coords", "assign", "shifts", "cameras", "tapes", "out_scores", "out_poses6", "out_contrib", "out_status"};
    AsyncCall call;
    Problem P;
    int rc = B <= 0 ? fail(ctx, ESACB200_ERR_ARG, "%s: empty batch (B=%d)", what, B) : check_min_prob(ctx, what, min_prob);
    if (!rc) rc = fill_problem(ctx, P, E, H, W, M, 0, 0, 0.f, 0.f, 0.f, tau, alpha, beta, maxReproj, sub, DRAWS);
    if (!rc) rc = check_tapes(ctx, what, tapes, tapes_bytes, B, P);
    if (!rc) rc = begin_async(ctx, true, B, P, coords, assign, assign_stride, shifts, cameras, out_status, 9, ptrs, names, call, what);
    if (rc) return rc;
    esacb200_ctx* a = call.a;
    const size_t stride = tape_stride(P);
    for (int b = 0; b < B; ++b) {
        Plan& pl = call.plans[b];
        const AsyncImage& im = call.imgs[b];
        char* tape = (char*)tapes + (size_t)b * stride;
        pl.min_prob = min_prob;  // a kernel parameter: a captured graph replays with the floor it was captured with
        rc = run_hypotheses(a, pl, pl.d_coords, (const int64_t*)pl.d_assign, assign_stride, ShardSteps(),
                            (uint32_t*)(tape + tape_masks_offset(M)));
        if (rc) return fail(ctx, rc, "image %d: %s", b, a->err);
        TapeDev td;
        td.dev = im.dev;
        td.flags = a->scalars.as<int>() + S_FLAGS;
        td.scores = a->scores.as<double>();
        td.poses = a->poses_ref.as<Pose>();
        td.out_scores = out_scores + (size_t)b * M;
        td.out_poses6 = out_poses6 + (size_t)b * M * 6;
        td.status = im.status;
        td.seed = a->seed_state.as<unsigned long long>();
        td.advance = im.advance;
        launch_tape_records_async(tape_record_args(a, P), tape_head(P, min_prob), tape, out_contrib + (size_t)b * M, td, a->stream);
        a->st.kernel_launches += 1;
    }
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_hypotheses_forward_async(esacb200_ctx* ctx, int B, const float* coords, int E, int H, int W, const int64_t* assign,
                                      int64_t assign_stride, int M, const int32_t* shifts, const float* cameras, float tau,
                                      float alpha, float beta, float maxReproj, int sub, void* tapes, size_t tapes_bytes,
                                      double* out_scores, double* out_poses6, uint8_t* out_contrib, int32_t* out_status) {
    return esacb200_hypotheses_forward_async_floor(ctx, B, coords, E, H, W, assign, assign_stride, M, shifts, cameras, tau, alpha,
                                                   beta, maxReproj, sub, ESACB200_PROB_THRESH, tapes, tapes_bytes, out_scores,
                                                   out_poses6, out_contrib, out_status);
}

int esacb200_hypotheses_backward_async(esacb200_ctx* ctx, int B, const void* tapes, size_t tapes_bytes, const float* coords,
                                       float* grads, int E, int H, int W, int M, const double* d_scores, const double* d_poses6,
                                       int32_t* out_status) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "hypotheses_backward_async";
    if (B <= 0) return fail(ctx, ESACB200_ERR_ARG, "%s: empty batch (B=%d)", what, B);
    const void* ptrs[] = {tapes, coords, grads, out_status, d_scores, d_poses6};
    const char* names[] = {"tapes", "coords", "grads", "out_status", "d_scores", "d_poses6"};
    int rc = device_args(ctx, what, 6, ptrs, names, 0x30u);  // an absent upstream is zero
    if (rc) return rc;
    std::vector<Plan> plans(1);
    Problem& P = plans[0].P;
    // sub, tau, alpha, beta and maxReproj are the forward's, read from the tape header on the device (BwdDev::prob)
    rc = fill_problem(ctx, P, E, H, W, M, 0, 0, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 1, NO_DRAW);
    if (!rc) rc = check_tapes(ctx, what, tapes, tapes_bytes, B, P);
    if (rc) return rc;
    plans[0].d_coords = coords;
    bool capturing = false;
    rc = stream_capturing(ctx, capturing);
    esacb200_ctx* a = nullptr;
    if (!rc) rc = async_context(ctx, capturing, "backward_async", &a);
    if (!rc) rc = async_workspace(ctx, a, plans, capturing, true, what);
    if (rc) return rc;
    if (capturing) a->frozen = true;
    int* sc = a->scalars.as<int>();
    const size_t cstride = (size_t)E * 3 * P.N, stride = tape_stride(P);
    for (int b = 0; b < B; ++b) {
        const char* tape = (const char*)tapes + (size_t)b * stride;
        BwdArgs args;
        memset(&args, 0, sizeof(args));
        args.coords = coords + (size_t)b * cstride;
        args.grads = grads + (size_t)b * cstride;
        args.n_contrib = sc + S_NCONTRIB;
        args.job_of = a->job_of.as<int>();
        args.masks = (const uint32_t*)(tape + tape_masks_offset(M));
        args.mask_words = (P.N + 31) / 32;
        args.red = a->red.as<double>();
        args.hyp_grad = a->hypgrad.p;
        args.P = P;
        const Problem* hp = (const Problem*)(tape + offsetof(TapeHead, P));
        BwdDev dv;
        dv.flags = sc + S_FLAGS;
        dv.dev.shift = &hp->shiftX;
        dv.dev.cam = &hp->f;
        dv.prob = hp;
        launch_backward_upstream_async(args, tape, d_scores ? d_scores + (size_t)b * M : nullptr,
                                       d_poses6 ? d_poses6 + (size_t)b * M * 6 : nullptr, sc + S_NCONTRIB, sc + S_FLAGS,
                                       out_status + b, dv, M, a->sm_count, a->stream);
        a->st.kernel_launches += 5;
    }
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_pose_loss_async(esacb200_ctx* ctx, int B, int M, const double* poses6, const float* gt16, float wRot, float wTrans,
                             float cut, double* out_losses, double* out_dloss6) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const void* ptrs[] = {poses6, gt16, out_losses, out_dloss6};
    const char* names[] = {"poses6", "gt16", "out_losses", "out_dloss6"};
    const int rc = device_args(ctx, "pose_loss_async", 4, ptrs, names);
    if (rc) return rc;
    if (M <= 0) return fail(ctx, ESACB200_ERR_ARG, "pose_loss_async: no poses (M=%d)", M);
    if (B <= 0 || B > 65535) return fail(ctx, ESACB200_ERR_ARG, "pose_loss_async: batch of %d images outside [1, 65535]", B);
    launch_pose_loss((const Pose*)poses6, B, M, gt16, wRot, wTrans, cut, out_losses, out_dloss6, ctx->stream);
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_backward_sharded(esacb200_ctx* ctx, const float* coords, float* grads, int E, int H, int W, const int64_t* assign,
                              int64_t assign_stride, int M, const float* gt_pose, float wRot, float wTrans, float cut,
                              int shiftX, int shiftY, float f, float ppx, float ppy, float tau, float alpha, float beta,
                              float maxReproj, int sub, esacb200_exchange_fn exchange, void* user, double* out_loss) try {
    if (!exchange) return ctx ? fail(ctx, ESACB200_ERR_ARG, "exchange callback is null") : ESACB200_ERR_ARG;
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !assign || !grads || !gt_pose) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    Problem P;
    int rc = fill_problem(ctx, P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS_INJECTED);
    return rc ? rc : backward_impl(ctx, P, coords, assign, assign_stride, grads, gt_pose, wRot, wTrans, cut, {exchange, user}, out_loss);
} ESAC_ABI_CATCH(ctx)

// esac_backward with the experts / hypotheses sharded over the ranks of the communicator: the two exchanges of the path
// (SURVEY 8e) run as NCCL collectives on the context's stream -- an all-gather of two doubles per rank and an all-reduce of
// one -- with no host callback.  M may be 0: the rank then only takes part in the collectives.
int esacb200_backward_sharded_nccl(esacb200_ctx* ctx, const float* coords, float* grads, int E, int H, int W,
                                   const int64_t* assign, int64_t assign_stride, int M, const float* gt_pose, float wRot,
                                   float wTrans, float cut, int shiftX, int shiftY, float f, float ppx, float ppy, float tau,
                                   float alpha, float beta, float maxReproj, int sub, int reduce_grads, double* out_loss) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!ctx->nccl_comm) return fail(ctx, ESACB200_ERR_ARG, "no communicator: call esacb200_comm_init first");
    if (M > 0) {
        if (!coords || !assign || !grads || !gt_pose) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
        Problem P;
        int rc = fill_problem(ctx, P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS_INJECTED);
        const ShardSteps sh = {nullptr, nullptr, /*use_nccl=*/true, /*reduce_grads=*/reduce_grads != 0};
        return rc ? rc : backward_impl(ctx, P, coords, assign, assign_stride, grads, gt_pose, wRot, wTrans, cut, sh, out_loss);
    }
    // no hypotheses here: neutral contributions to both collectives
    begin_call(ctx);
    CK(ctx->stats.ensure(sizeof(CallStats)));
    CK(ctx->gathered.ensure((size_t)ctx->comm_world * 2 * 8));
    Pinned& h = *ctx->pin;
    CallStats* d_stats = ctx->stats.as<CallStats>();
    h.exchange[0] = 0.; h.exchange[1] = -1e300; h.exchange[2] = 0.;  // local_loss, max_score, sum_exp
    CK(cudaMemcpyAsync(&d_stats->local_loss, h.exchange, sizeof(h.exchange), cudaMemcpyHostToDevice, ctx->stream));
    // the collectives below come in the order backward_impl issues them on the ranks that do hold hypotheses
    CKN(nccl_api().AllGather(&d_stats->max_score, ctx->gathered.p, 2, kNcclFloat64, ctx->nccl_comm, ctx->stream));
    const size_t n = reduce_grads ? (size_t)E * 3 * H * W : 0;
    float* d_dst = grads;
    if (reduce_grads) {  // zero contribution to the gradient sum, then the sum is added to this rank's tensor like everywhere
        if (!grads || E <= 0 || H <= 0 || W <= 0) return fail(ctx, ESACB200_ERR_ARG, "reduce_grads needs the gradient tensor and its shape on every rank");
        CK(ctx->grads_work.ensure(n * 4));
        int rc = ensure_host_flags(ctx, E);
        if (rc) return rc;
        CK(ctx->eflags.ensure((size_t)E * sizeof(int)));
        CK(cudaMemsetAsync(ctx->eflags.p, 0, (size_t)E * sizeof(int), ctx->stream));
        CKN(nccl_api().AllReduce(ctx->eflags.p, ctx->eflags.p, (size_t)E, kNcclInt32, kNcclMax, ctx->nccl_comm, ctx->stream));
        CK(cudaMemcpyAsync(ctx->h_flags, ctx->eflags.p, (size_t)E * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        if (!is_device_ptr(grads)) {
            CK(ctx->grads.ensure(n * 4));
            CK(cudaMemcpyAsync(ctx->grads.p, grads, n * 4, cudaMemcpyHostToDevice, ctx->stream));
            d_dst = ctx->grads.as<float>();
        }
        rc = for_flagged_planes(ctx, E, (size_t)3 * H * W, ctx->grads_work.as<float>(), d_dst, 0);
        if (rc) return rc;
    }
    CKN(nccl_api().AllReduce(&d_stats->local_loss, &d_stats->global_loss, 1, kNcclFloat64, kNcclSum, ctx->nccl_comm, ctx->stream));
    if (reduce_grads) {
        int rc = for_flagged_planes(ctx, E, (size_t)3 * H * W, ctx->grads_work.as<float>(), d_dst, 1);
        if (rc) return rc;
        if (!is_device_ptr(grads)) CK(cudaMemcpyAsync(grads, ctx->grads.p, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaGetLastError());
    }
    CK(cudaMemcpyAsync(&h.stats.global_loss, &d_stats->global_loss, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    if (out_loss) *out_loss = h.stats.global_loss;
    ctx->st.expected_loss = h.stats.global_loss;
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
// Batches.  Every image is an independent problem (SURVEY 8e: "images in a batch are fully independent"), so the images
// are dealt round-robin to a few worker contexts, each driven by its own host thread on its own stream: the small kernels of
// one image fill the gaps the host synchronisations of another leave.  Image b has its own map size; with `draws` the seeds
// are fixed per image before the images are dealt (image b draws what the b-th of B consecutive single-image calls would),
// so a worker runs its images largest first and its workspace grows at most once.  `image(w, b)` runs image b on worker
// context w.  Everything the caller queued on its stream (the experts' outputs) is visible to the workers.  The statistics
// of the call are those of the last image, with the wall time and kernel launches of the whole batch.
static int run_batch(esacb200_ctx* ctx, int B, const int* H, const int* W, bool draws,
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

// esac_backward over a batch, on the worker contexts of run_batch.
int esacb200_backward_ragged(esacb200_ctx* ctx, int B, const float* const* coords, float* const* grads, const int* H, const int* W,
                             int E, const int64_t* assign, int64_t assign_stride, int M, const float* gt_poses, float wRot,
                             float wTrans, float cut, const int* shiftX, const int* shiftY, const float* f, const float* ppx,
                             const float* ppy, float tau, float alpha, float beta, float maxReproj, int sub,
                             double* out_losses) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !grads || !H || !W || !assign || !gt_poses || B <= 0)
        return fail(ctx, ESACB200_ERR_ARG, "null pointer argument or empty batch");
    if (!f || !ppx || !ppy) return fail(ctx, ESACB200_ERR_ARG, "null camera array");
    if (ctx->inj_M) return fail(ctx, ESACB200_ERR_ARG, "injected cells are a single-image test hook");
    if (E <= 0 || M <= 0) return fail(ctx, ESACB200_ERR_ARG, "bad sizes E=%d M=%d", E, M);
    std::vector<Plan> plans;
    int rc = fill_problems(ctx, plans, B, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS);
    if (rc) return rc;
    bool dev_c = false, dev_g = false;
    rc = pointer_kind(ctx, (const void* const*)coords, B, "coords", dev_c);
    if (rc) return rc;
    rc = pointer_kind(ctx, (const void* const*)grads, B, "grads", dev_g);
    if (rc) return rc;
    const int64_t arow = assign_stride == 0 ? 0 : (int64_t)M * assign_stride;
    std::vector<float> gt_host;
    const float* gt = gt_poses;
    if (is_device_ptr(gt_poses)) {  // read back with run_batch's synchronisation
        gt_host.resize((size_t)B * 16);
        CK(cudaMemcpyAsync(gt_host.data(), gt_poses, gt_host.size() * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
        gt = gt_host.data();
    }
    rc = run_batch(ctx, B, H, W, true, [&](esacb200_ctx* w, int b) {
        double loss = 0;
        int rc = backward_impl(w, plans[b].P, coords[b], assign + (size_t)b * arow, assign_stride, grads[b], gt + (size_t)b * 16, wRot,
                               wTrans, cut, ShardSteps(), &loss);
        if (!rc && out_losses) out_losses[b] = loss;
        return rc;
    });
    return rc ? rc : ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// The hypotheses node over a batch, on the worker contexts of run_batch: image b runs the single-image forward / backward
// with row b of the [B,M] outputs / upstreams.
int esacb200_hypotheses_forward_ragged_floor(esacb200_ctx* ctx, int B, const float* const* coords, const int* H, const int* W,
                                             int E, const int64_t* assign, int64_t assign_stride, int M, const int* shiftX,
                                             const int* shiftY, const float* f, const float* ppx, const float* ppy, float tau,
                                             float alpha, float beta, float maxReproj, int sub, double min_prob,
                                             void* const* tapes, const size_t* tape_bytes_, double* out_scores,
                                             double* out_poses6, uint8_t* out_contrib) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !H || !W || !assign || !tapes || !tape_bytes_ || !out_scores || !out_poses6 || !out_contrib || B <= 0)
        return fail(ctx, ESACB200_ERR_ARG, "null pointer argument or empty batch");
    if (check_min_prob(ctx, nullptr, min_prob)) return ESACB200_ERR_ARG;
    if (!f || !ppx || !ppy) return fail(ctx, ESACB200_ERR_ARG, "null camera array");
    if (ctx->inj_M) return fail(ctx, ESACB200_ERR_ARG, "injected cells are a single-image test hook");
    if (E <= 0 || M <= 0) return fail(ctx, ESACB200_ERR_ARG, "bad sizes E=%d M=%d", E, M);
    std::vector<Plan> plans;
    int rc = fill_problems(ctx, plans, B, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS);
    if (rc) return rc;
    bool dev_c = false;
    rc = pointer_kind(ctx, (const void* const*)coords, B, "coords", dev_c);
    if (rc) return rc;
    for (int b = 0; b < B; ++b) {
        if (!tapes[b]) return fail(ctx, ESACB200_ERR_ARG, "image %d: tape is null", b);
        if (check_tape(ctx, tapes[b], tape_bytes_[b], plans[b].P))
            return fail(ctx, ESACB200_ERR_ARG, "image %d: %s", b, std::string(ctx->err).c_str());
    }
    const int64_t arow = assign_stride == 0 ? 0 : (int64_t)M * assign_stride;
    rc = run_batch(ctx, B, H, W, true, [&](esacb200_ctx* w, int b) {
        return hypotheses_forward_impl(w, plans[b].P, min_prob, coords[b], assign + (size_t)b * arow, assign_stride, tapes[b],
                                       out_scores + (size_t)b * M, out_poses6 + (size_t)b * M * 6, out_contrib + (size_t)b * M);
    });
    return rc ? rc : ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_hypotheses_forward_ragged(esacb200_ctx* ctx, int B, const float* const* coords, const int* H, const int* W, int E,
                                       const int64_t* assign, int64_t assign_stride, int M, const int* shiftX, const int* shiftY,
                                       const float* f, const float* ppx, const float* ppy, float tau, float alpha, float beta,
                                       float maxReproj, int sub, void* const* tapes, const size_t* tape_bytes_,
                                       double* out_scores, double* out_poses6, uint8_t* out_contrib) {
    return esacb200_hypotheses_forward_ragged_floor(ctx, B, coords, H, W, E, assign, assign_stride, M, shiftX, shiftY, f, ppx, ppy,
                                                    tau, alpha, beta, maxReproj, sub, ESACB200_PROB_THRESH, tapes, tape_bytes_,
                                                    out_scores, out_poses6, out_contrib);
}

int esacb200_hypotheses_backward_ragged(esacb200_ctx* ctx, int B, const void* const* tapes, const float* const* coords,
                                        float* const* grads, const int* H, const int* W, int E, const double* d_scores,
                                        const double* d_poses6) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!tapes || !coords || !grads || !H || !W || B <= 0) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument or empty batch");
    if (ctx->inj_M) return fail(ctx, ESACB200_ERR_ARG, "injected cells are a single-image test hook");
    if (E <= 0) return fail(ctx, ESACB200_ERR_ARG, "bad size E=%d", E);
    std::vector<Plan> sizes;  // the maps' sizes, checked as those of a forward of one hypothesis (the tapes hold M)
    int rc = fill_problems(ctx, sizes, B, E, H, W, 1, nullptr, nullptr, nullptr, nullptr, nullptr, 0.f, 0.f, 0.f, 0.f, 1, DRAWS);
    if (rc) return rc;
    bool dev_c = false, dev_g = false, dev_t = false;
    rc = pointer_kind(ctx, (const void* const*)coords, B, "coords", dev_c);
    if (rc) return rc;
    rc = pointer_kind(ctx, (const void* const*)grads, B, "grads", dev_g);
    if (rc) return rc;
    rc = pointer_kind(ctx, tapes, B, "tape", dev_t);
    if (rc) return rc;
    rc = run_batch(ctx, B, H, W, false, [&](esacb200_ctx* w, int b) {
        return hypotheses_backward_impl(w, tapes[b], coords[b], grads[b], E, H[b], W[b], d_scores, d_poses6, b);
    });
    return rc ? rc : ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// B images of one shape: the pointer and size arrays of [B,E,3,H,W] tensors.
int esacb200_backward_batch_cameras(esacb200_ctx* ctx, int B, const float* coords, float* grads, int E, int H, int W,
                                    const int64_t* assign, int64_t assign_stride, int M, const float* gt_poses, float wRot,
                                    float wTrans, float cut, const int* shiftX, const int* shiftY, const float* f,
                                    const float* ppx, const float* ppy, float tau, float alpha, float beta, float maxReproj,
                                    int sub, double* out_losses) try {
    if (!ctx) return ESACB200_ERR_ARG;
    if (!coords || !grads || !assign || !gt_poses || B <= 0) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument or empty batch");
    if (!f || !ppx || !ppy) return fail(ctx, ESACB200_ERR_ARG, "null camera array");
    if (ctx->inj_M) return fail(ctx, ESACB200_ERR_ARG, "injected cells are a single-image test hook");
    if (E <= 0 || H <= 0 || W <= 0 || M <= 0) return fail(ctx, ESACB200_ERR_ARG, "bad sizes E=%d H=%d W=%d M=%d", E, H, W, M);
    const size_t cstride = (size_t)E * 3 * H * W;
    const auto cp = slices(coords, B, cstride);
    const auto gp = slices(grads, B, cstride);
    const std::vector<int> hs((size_t)B, H), ws((size_t)B, W);
    return esacb200_backward_ragged(ctx, B, cp.data(), gp.data(), hs.data(), ws.data(), E, assign, assign_stride, M, gt_poses, wRot,
                                    wTrans, cut, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, out_losses);
} ESAC_ABI_CATCH(ctx)

int esacb200_backward_batch(esacb200_ctx* ctx, int B, const float* coords, float* grads, int E, int H, int W,
                            const int64_t* assign, int64_t assign_stride, int M, const float* gt_poses, float wRot,
                            float wTrans, float cut, const int* shiftX, const int* shiftY, float f, float ppx, float ppy,
                            float tau, float alpha, float beta, float maxReproj, int sub, double* out_losses) try {
    if (!ctx) return ESACB200_ERR_ARG;
    const size_t n = B > 0 ? (size_t)B : 1;  // B <= 0 is rejected by the call below, with its usual message
    const std::vector<float> fs(n, f), cx(n, ppx), cy(n, ppy);
    return esacb200_backward_batch_cameras(ctx, B, coords, grads, E, H, W, assign, assign_stride, M, gt_poses, wRot, wTrans, cut,
                                           shiftX, shiftY, fs.data(), cx.data(), cy.data(), tau, alpha, beta, maxReproj, sub,
                                           out_losses);
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
int esacb200_assign_hypotheses(esacb200_ctx* ctx, int B, int E, int M, const float* weights, int keep_top, int single_expert,
                               uint64_t seed, int64_t* out_assign, float* out_hist) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!weights || !out_assign) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    if (B <= 0 || E <= 0 || M <= 0) return fail(ctx, ESACB200_ERR_ARG, "bad sizes B=%d E=%d M=%d", B, E, M);
    if (E > assign_max_experts()) return fail(ctx, ESACB200_ERR_ARG, "E=%d exceeds the %d experts one CTA holds", E, assign_max_experts());
    const bool w_host = !is_device_ptr(weights), a_host = !is_device_ptr(out_assign), h_host = out_hist && !is_device_ptr(out_hist);
    const size_t wb = (size_t)B * E * sizeof(float), ab = (size_t)B * M * sizeof(int64_t);
    // staging layout in `scratch`: [flags int (16 B)] [weights] [hist] [assign]
    const size_t off_w = 16, off_h = off_w + ((wb + 15) & ~(size_t)15), off_a = off_h + ((wb + 15) & ~(size_t)15);
    CK(ctx->scratch.ensure(off_a + ab));
    char* base = (char*)ctx->scratch.p;
    const float* d_w = weights;
    if (w_host) {
        CK(cudaMemcpyAsync(base + off_w, weights, wb, cudaMemcpyHostToDevice, ctx->stream));
        d_w = (const float*)(base + off_w);
    }
    int64_t* d_a = a_host ? (int64_t*)(base + off_a) : out_assign;
    float* d_h = !out_hist ? nullptr : (h_host ? (float*)(base + off_h) : out_hist);
    CK(cudaMemsetAsync(base, 0, 16, ctx->stream));
    launch_assign(d_w, B, E, M, keep_top, single_expert, seed, d_a, d_h, (int*)base, ctx->stream);
    CK(cudaGetLastError());
    if (a_host) CK(cudaMemcpyAsync(out_assign, d_a, ab, cudaMemcpyDeviceToHost, ctx->stream));
    if (h_host) CK(cudaMemcpyAsync(out_hist, d_h, wb, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(&ctx->pin->gating_flags, base, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    const int flags = ctx->pin->gating_flags;
    if (flags & 1) return fail(ctx, ESACB200_ERR_ARG, "probability tensor contains either inf, nan or element < 0");
    if (flags & 2) return fail(ctx, ESACB200_ERR_ARG, "invalid multinomial distribution (sum of probabilities <= 0)");
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
// The two losses' steps that the eager ragged calls and the stream-ordered calls share: the per-image size checks, the
// per-image records, the workspace layout and the launches.

static size_t align64(size_t n) { return (n + 63) & ~(size_t)63; }

// Byte offsets in the loss workspace of a call of B images whose blocks have `parts` partials.
//   reprojection: [tickets B u32] [img B x kReprojImgFloats f32] [records] [losses B f64] [bad B i32] [partials f64 each]
//   coordinates:  [tickets B u32 | counts B u32] [records] [losses B f64] [valid counts B i64] [partials 2 f64 each]
// The eager reprojection loss leaves `bad` unused: a singular ground truth fails it before anything is enqueued.
struct LossLayout {
    size_t img = 0, rec, loss, flags, part, end;
};
static LossLayout reproj_layout(int B, long long parts) {
    LossLayout L;
    L.img = align64((size_t)B * 4);
    L.rec = L.img + align64((size_t)B * kReprojImgFloats * sizeof(float));
    L.loss = L.rec + align64((size_t)B * sizeof(ReprojImage));
    L.flags = L.loss + align64((size_t)B * 8);
    L.part = L.flags + align64((size_t)B * 4);
    L.end = L.part + (size_t)parts * 8;
    return L;
}
static LossLayout coord_layout(int B, long long parts) {
    LossLayout L;
    L.rec = align64((size_t)B * 8);
    L.loss = L.rec + align64((size_t)B * sizeof(CoordImage));
    L.flags = L.loss + align64((size_t)B * 8);
    L.part = L.flags + align64((size_t)B * 8);
    L.end = L.part + (size_t)parts * 2 * 8;
    return L;
}

// The per-image sizes of a reprojection-loss call: positive, at most 2^30 cells.  `what`: the entry point named in front of
// each message, or null.
static int reproj_sizes(esacb200_ctx* ctx, const char* what, int B, const int* H, const int* W) {
    const char* sep = what ? ": " : "";
    if (!what) what = "";
    for (int b = 0; b < B; ++b) {
        if (H[b] <= 0 || W[b] <= 0) return fail(ctx, ESACB200_ERR_ARG, "%s%simage %d: bad size %dx%d", what, sep, b, W[b], H[b]);
        if ((long long)H[b] * W[b] > (1ll << 30))
            return fail(ctx, ESACB200_ERR_ARG, "%s%simage %d: map %dx%d too large", what, sep, b, W[b], H[b]);
    }
    return 0;
}

// The records of a reprojection-loss call on the B images at the device addresses coords[b] and grads[b] (grads, or an
// entry of it, null: no gradient), and per image whether it takes the 128-bit load path.  Returns the blocks' partials.
static long long reproj_records(int B, const float* const* coords, float* const* grads, const int* H, const int* W,
                                std::vector<ReprojImage>& recs, std::vector<char>& vec) {
    recs.resize((size_t)B);
    vec.resize((size_t)B);
    long long parts = 0;
    for (int b = 0; b < B; ++b) {
        ReprojImage& r = recs[b];
        r.coords = coords[b];
        r.grads = grads ? grads[b] : nullptr;
        r.N = H[b] * W[b];
        r.W = W[b];
        r.b = b;
        r.blocks = reproj_blocks_per_image(r.N);
        r.part0 = parts;
        parts += r.blocks;
        vec[b] = reproj_vec_ok(r.coords, r.grads, r.N, r.W);
    }
    return parts;
}

// The reprojection loss's launches, one per load path, on the workspace at `base` laid out as L, whose records are in
// order_by_path's order (n_vec on the 128-bit path first).  They run on run's stream and count in its kernel_launches.
static void reproj_launches(esacb200_ctx* run, char* base, const LossLayout& L, int B, int n_vec, int max_vec, int max_sc,
                            int sub, float cut, float maxReproj, float minDepth) {
    const ReprojImage* rec = (const ReprojImage*)(base + L.rec);
    for (int path = 0; path < 2; ++path) {
        const int n = path == 0 ? n_vec : B - n_vec;
        if (n == 0) continue;
        launch_reproj(path == 0, rec + (path == 0 ? 0 : n_vec), n, path == 0 ? max_vec : max_sc, (const float*)(base + L.img),
                      (float)sub, cut, maxReproj, minDepth, (double*)(base + L.part), (unsigned*)base, (double*)(base + L.loss),
                      run->stream);
        run->st.kernel_launches += 1;
    }
}

// The per-image sizes of a coordinate-loss call: positive, prediction and ground truth at most 1 apart, at most 2^30 cells.
// `what`: the entry point named in front of each message, or null.
static int coord_sizes(esacb200_ctx* ctx, const char* what, int B, const int* Hp, const int* Wp, const int* Hg, const int* Wg) {
    const char* sep = what ? ": " : "";
    if (!what) what = "";
    for (int b = 0; b < B; ++b) {
        if (Hp[b] <= 0 || Wp[b] <= 0 || Hg[b] <= 0 || Wg[b] <= 0)
            return fail(ctx, ESACB200_ERR_ARG, "%s%simage %d: bad sizes prediction %dx%d ground truth %dx%d", what, sep, b, Hp[b],
                        Wp[b], Hg[b], Wg[b]);
        if (abs(Hp[b] - Hg[b]) > 1 || abs(Wp[b] - Wg[b]) > 1)   // util.assert_size tolerates 1 cell
            return fail(ctx, ESACB200_ERR_ARG, "%s%simage %d: size mismatch: prediction %dx%d, ground truth %dx%d (at most 1 apart)",
                        what, sep, b, Hp[b], Wp[b], Hg[b], Wg[b]);
        if ((long long)Hp[b] * Wp[b] > (1ll << 30) || (long long)Hg[b] * Wg[b] > (1ll << 30))
            return fail(ctx, ESACB200_ERR_ARG, "%s%simage %d: map too large", what, sep, b);
    }
    return 0;
}

// The records of a coordinate-loss call on the B images at the device addresses pred[b], gt[b] and grads[b] (grads, or an
// entry of it, null: no gradient), and per image whether it takes the 128-bit load path.  Returns the blocks' partials.
static long long coord_records(int B, const float* const* pred, const float* const* gt, float* const* grads, const int* Hp,
                               const int* Wp, const int* Hg, const int* Wg, std::vector<CoordImage>& recs, std::vector<char>& vec) {
    recs.resize((size_t)B);
    vec.resize((size_t)B);
    long long parts = 0;
    for (int b = 0; b < B; ++b) {
        CoordImage& r = recs[b];
        r.pred = pred[b];
        r.gt = gt[b];
        r.grads = grads ? grads[b] : nullptr;
        vec[b] = coord_image(r, Hp[b], Wp[b], Hg[b], Wg[b]);
        r.b = b;
        r.part0 = parts;
        parts += r.blocks;
    }
    return parts;
}

// The coordinate loss's launches, per load path the count pass (with gradients) and the loss pass, on the workspace at
// `base` laid out as L, whose records are in order_by_path's order.  They run on run's stream and count in its
// kernel_launches.
static void coord_launches(esacb200_ctx* run, char* base, const LossLayout& L, int B, bool grads, int n_vec, int max_vec,
                           int max_sc, float cut) {
    const CoordImage* rec = (const CoordImage*)(base + L.rec);
    for (int path = 0; path < 2; ++path) {
        const int n = path == 0 ? n_vec : B - n_vec;
        if (n == 0) continue;
        for (int pass = grads ? 1 : 2; pass <= 2; ++pass) {
            launch_coord_loss(path == 0, pass, grads, rec + (path == 0 ? 0 : n_vec), n, path == 0 ? max_vec : max_sc, cut,
                              (unsigned*)base + B, (double*)(base + L.part), (unsigned*)base, (double*)(base + L.loss),
                              (long long*)(base + L.flags), run->stream);
            run->st.kernel_launches += 1;
        }
    }
}

// -------------------------------------------------------------------------------------------------
// The reprojection loss over B images, each with its own size: one launch per load path (128-bit / scalar, chosen per
// image as a single-image call would choose it), each image cut into the blocks a single-image call uses.
int esacb200_reproj_loss_ragged(esacb200_ctx* ctx, int B, const float* const* coords, float* const* grads, const int* H,
                                const int* W, const float* gt_poses, const int* shiftX, const int* shiftY, const float* f,
                                const float* ppx, const float* ppy, int sub, float cut, float maxReproj, float minDepth,
                                double* out_losses) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !H || !W || !gt_poses || !out_losses) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    if (!f || !ppx || !ppy) return fail(ctx, ESACB200_ERR_ARG, "null camera array");
    if (B <= 0 || sub <= 0) return fail(ctx, ESACB200_ERR_ARG, "bad sizes B=%d sub=%d", B, sub);
    int rc = reproj_sizes(ctx, nullptr, B, H, W);
    if (rc) return rc;
    bool c_dev = false, g_dev = false;
    if ((rc = pointer_kind(ctx, (const void* const*)coords, B, "coords", c_dev))) return rc;
    if (grads && (rc = pointer_kind(ctx, (const void* const*)grads, B, "grads", g_dev))) return rc;
    begin_call(ctx);
    std::vector<size_t> bytes((size_t)B), c_off, g_off;
    for (int b = 0; b < B; ++b) bytes[b] = (size_t)3 * H[b] * W[b] * sizeof(float);
    std::vector<const float*> d_coords;
    std::vector<float*> d_grads((size_t)B, nullptr);
    rc = stage_images(ctx, coords, bytes, c_dev, true, ctx->coords, d_coords, c_off);
    if (rc) return rc;
    if (grads && (rc = stage_images(ctx, grads, bytes, g_dev, false, ctx->grads, d_grads, g_off))) return rc;
    std::vector<float> gt((size_t)B * 16);
    if (is_device_ptr(gt_poses)) {
        CK(cudaMemcpyAsync(gt.data(), gt_poses, gt.size() * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    } else {
        memcpy(gt.data(), gt_poses, gt.size() * sizeof(float));
    }
    // world->camera rows: inverse of the affine camera->world matrix (torch's .inverse()[0:3,:], ref_expert.py:127)
    std::vector<float> img((size_t)B * kReprojImgFloats, 0.f);
    for (int b = 0; b < B; ++b)
        if (!reproj_img_row(gt.data() + (size_t)b * 16, shiftX ? shiftX[b] : 0, shiftY ? shiftY[b] : 0, f[b], ppx[b], ppy[b],
                            img.data() + (size_t)b * kReprojImgFloats))
            return fail(ctx, ESACB200_ERR_ARG, "image %d: ground-truth pose is singular", b);
    std::vector<ReprojImage> recs, ordered;
    std::vector<char> vec;
    const long long parts = reproj_records(B, d_coords.data(), d_grads.data(), H, W, recs, vec);
    int n_vec, max_vec, max_sc;
    const size_t rec_bytes = order_by_path(recs, vec, ordered, n_vec, max_vec, max_sc);
    const LossLayout L = reproj_layout(B, parts);
    CK(ctx->scratch.ensure(L.end));
    char* base = (char*)ctx->scratch.p;
    std::vector<char> staging(L.rec - L.img + rec_bytes);
    memcpy(staging.data(), img.data(), img.size() * sizeof(float));
    memcpy(staging.data() + (L.rec - L.img), ordered.data(), rec_bytes);
    CK(cudaMemsetAsync(base, 0, L.img, ctx->stream));
    CK(cudaMemcpyAsync(base + L.img, staging.data(), staging.size(), cudaMemcpyHostToDevice, ctx->stream));
    mark(ctx, EV_H2D);
    mark(ctx, EV_FOLD);  // ms_score = the kernels alone
    reproj_launches(ctx, base, L, B, n_vec, max_vec, max_sc, sub, cut, maxReproj, minDepth);
    CK(cudaGetLastError());
    mark(ctx, EV_SCORE);
    if (grads && !g_dev) {
        rc = copy_packed(ctx, (char* const*)grads, bytes, g_off, (char*)ctx->grads.p, false, ctx->stream);
        if (rc) return rc;
    }
    CK(cudaMemcpyAsync(out_losses, base + L.loss, (size_t)B * 8, cudaMemcpyDeviceToHost, ctx->stream));
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// B images of one shape: the pointer and size arrays of a [B,3,H,W] tensor.
int esacb200_reproj_loss_cameras(esacb200_ctx* ctx, int B, const float* coords, float* grads, int H, int W, const float* gt_poses,
                                 const int* shiftX, const int* shiftY, const float* f, const float* ppx, const float* ppy, int sub,
                                 float cut, float maxReproj, float minDepth, double* out_losses) try {
    if (!ctx) return ESACB200_ERR_ARG;
    if (!coords || !gt_poses || !out_losses) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    if (!f || !ppx || !ppy) return fail(ctx, ESACB200_ERR_ARG, "null camera array");
    if (B <= 0 || H <= 0 || W <= 0 || sub <= 0) return fail(ctx, ESACB200_ERR_ARG, "bad sizes B=%d H=%d W=%d sub=%d", B, H, W, sub);
    if ((long long)H * W > (1ll << 30)) return fail(ctx, ESACB200_ERR_ARG, "map %dx%d too large", W, H);
    const size_t n = (size_t)3 * H * W;
    const auto cp = slices(coords, B, n);
    const auto gp = slices(grads, B, n);
    const std::vector<int> hs((size_t)B, H), ws((size_t)B, W);
    return esacb200_reproj_loss_ragged(ctx, B, cp.data(), grads ? gp.data() : nullptr, hs.data(), ws.data(), gt_poses, shiftX, shiftY,
                                       f, ppx, ppy, sub, cut, maxReproj, minDepth, out_losses);
} ESAC_ABI_CATCH(ctx)

int esacb200_reproj_loss(esacb200_ctx* ctx, int B, const float* coords, float* grads, int H, int W, const float* gt_poses,
                         const int* shiftX, const int* shiftY, float f, float ppx, float ppy, int sub, float cut,
                         float maxReproj, float minDepth, double* out_losses) try {
    if (!ctx) return ESACB200_ERR_ARG;
    const size_t n = B > 0 ? (size_t)B : 1;  // B <= 0 is rejected by the call below, with its usual message
    const std::vector<float> fs(n, f), cx(n, ppx), cy(n, ppy);
    return esacb200_reproj_loss_cameras(ctx, B, coords, grads, H, W, gt_poses, shiftX, shiftY, fs.data(), cx.data(), cy.data(), sub,
                                        cut, maxReproj, minDepth, out_losses);
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
// The coordinate loss over B images, each with its own prediction and ground-truth size: one launch per load path and
// pass, each image cut into the blocks a single-image call uses.
int esacb200_coord_loss_ragged(esacb200_ctx* ctx, int B, const float* const* pred, const int* Hp, const int* Wp,
                               const float* const* gt, const int* Hg, const int* Wg, float* const* grads, float cut,
                               double* out_losses, int64_t* out_counts) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!pred || !gt || !Hp || !Wp || !Hg || !Wg || !out_losses) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    if (B <= 0) return fail(ctx, ESACB200_ERR_ARG, "bad sizes B=%d", B);
    int rc = coord_sizes(ctx, nullptr, B, Hp, Wp, Hg, Wg);
    if (rc) return rc;
    bool p_dev = false, q_dev = false, g_dev = false;
    if ((rc = pointer_kind(ctx, (const void* const*)pred, B, "pred", p_dev))) return rc;
    if ((rc = pointer_kind(ctx, (const void* const*)gt, B, "gt", q_dev))) return rc;
    if (grads && (rc = pointer_kind(ctx, (const void* const*)grads, B, "grads", g_dev))) return rc;
    begin_call(ctx);
    std::vector<size_t> pbytes((size_t)B), gbytes((size_t)B), p_off, q_off, g_off;
    for (int b = 0; b < B; ++b) {
        pbytes[b] = (size_t)3 * Hp[b] * Wp[b] * sizeof(float);
        gbytes[b] = (size_t)3 * Hg[b] * Wg[b] * sizeof(float);
    }
    std::vector<const float*> d_pred, d_gt;
    std::vector<float*> d_grads((size_t)B, nullptr);
    if ((rc = stage_images(ctx, pred, pbytes, p_dev, true, ctx->coords, d_pred, p_off))) return rc;
    if ((rc = stage_images(ctx, gt, gbytes, q_dev, true, ctx->coords_alt, d_gt, q_off))) return rc;
    if (grads && (rc = stage_images(ctx, grads, pbytes, g_dev, false, ctx->grads, d_grads, g_off))) return rc;
    std::vector<CoordImage> recs, ordered;
    std::vector<char> vec;
    const long long parts = coord_records(B, d_pred.data(), d_gt.data(), d_grads.data(), Hp, Wp, Hg, Wg, recs, vec);
    int n_vec, max_vec, max_sc;
    const size_t rec_bytes = order_by_path(recs, vec, ordered, n_vec, max_vec, max_sc);
    const LossLayout L = coord_layout(B, parts);
    CK(ctx->scratch.ensure(L.end));
    char* base = (char*)ctx->scratch.p;
    CK(cudaMemsetAsync(base, 0, L.rec, ctx->stream));
    CK(cudaMemcpyAsync(base + L.rec, ordered.data(), rec_bytes, cudaMemcpyHostToDevice, ctx->stream));
    mark(ctx, EV_H2D);
    mark(ctx, EV_FOLD);  // ms_score = the kernels alone
    coord_launches(ctx, base, L, B, grads != nullptr, n_vec, max_vec, max_sc, cut);
    CK(cudaGetLastError());
    mark(ctx, EV_SCORE);
    if (grads && !g_dev) {
        rc = copy_packed(ctx, (char* const*)grads, pbytes, g_off, (char*)ctx->grads.p, false, ctx->stream);
        if (rc) return rc;
    }
    CK(cudaMemcpyAsync(out_losses, base + L.loss, (size_t)B * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (out_counts) CK(cudaMemcpyAsync(out_counts, base + L.flags, (size_t)B * 8, cudaMemcpyDeviceToHost, ctx->stream));
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// B images of one shape: the pointer and size arrays of [B,3,Hp,Wp] / [B,3,Hg,Wg] tensors.
int esacb200_coord_loss(esacb200_ctx* ctx, int B, const float* pred, int Hp, int Wp, const float* gt, int Hg, int Wg,
                        float* grads, float cut, double* out_losses, int64_t* out_counts) try {
    if (!ctx) return ESACB200_ERR_ARG;
    if (!pred || !gt || !out_losses) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    if (B <= 0 || Hp <= 0 || Wp <= 0 || Hg <= 0 || Wg <= 0)
        return fail(ctx, ESACB200_ERR_ARG, "bad sizes B=%d prediction %dx%d ground truth %dx%d", B, Hp, Wp, Hg, Wg);
    if (abs(Hp - Hg) > 1 || abs(Wp - Wg) > 1)   // util.assert_size tolerates 1 cell
        return fail(ctx, ESACB200_ERR_ARG, "size mismatch: prediction %dx%d, ground truth %dx%d (at most 1 apart)", Hp, Wp, Hg, Wg);
    if ((long long)Hp * Wp > (1ll << 30) || (long long)Hg * Wg > (1ll << 30))
        return fail(ctx, ESACB200_ERR_ARG, "map too large");
    const size_t np = (size_t)3 * Hp * Wp;
    const auto pp = slices(pred, B, np), qp = slices(gt, B, (size_t)3 * Hg * Wg);
    const auto gp = slices(grads, B, np);
    const std::vector<int> hp((size_t)B, Hp), wp((size_t)B, Wp), hg((size_t)B, Hg), wg((size_t)B, Wg);
    return esacb200_coord_loss_ragged(ctx, B, pp.data(), hp.data(), wp.data(), qp.data(), hg.data(), wg.data(),
                                      grads ? gp.data() : nullptr, cut, out_losses, out_counts);
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
// Stream-ordered losses.  The eager ragged calls' records and launches, run in the context ctx->async on the caller's device
// arrays: the records reach the workspace as prep-kernel parameters (loss_async.cu), the ground truth, pads and camera are
// read on the device, and a finish kernel writes the caller's outputs.  Nothing here synchronises, reads back or queries an
// event, and a call that a capture records allocates nothing.

// Makes the loss workspace hold `bytes`: grows it when no capture has used it yet, else fails without touching it.
static int loss_workspace(esacb200_ctx* ctx, esacb200_ctx* a, size_t bytes, bool capturing, const char* what) {
    if (bytes <= a->loss_ws.cap) return 0;
    if (capturing || a->loss_frozen)
        return fail(ctx, ESACB200_ERR_ARG,
                    "%s: this call needs %zu bytes of loss workspace, more than %s, and a graph that holds it may still be "
                    "replayed; call reserve_loss_async (esacb200_reserve_loss_async) with the largest batch and map before the "
                    "first capture", what, bytes, capturing ? "was reserved before this capture" : "an earlier capture used");
    CK(a->loss_ws.ensure(bytes));
    return 0;
}

// The B image pointers of one argument are device memory.
static int device_images(esacb200_ctx* ctx, const char* what, const char* name, const void* const* p, int B) {
    for (int b = 0; b < B; ++b) {
        if (!p[b]) return fail(ctx, ESACB200_ERR_ARG, "%s: image %d: %s is null", what, b, name);
        if (!is_device_ptr(p[b]))
            return fail(ctx, ESACB200_ERR_ARG, "%s takes device pointers only: image %d: %s is host memory", what, b, name);
    }
    return 0;
}

// The async context of a loss call, and whether the stream is being captured.
static int begin_loss_async(esacb200_ctx* ctx, esacb200_ctx*& a, bool& capturing) {
    int rc = stream_capturing(ctx, capturing);
    if (!rc) rc = async_context(ctx, capturing, "loss_async", &a);
    return rc;
}

int esacb200_reserve_loss_async(esacb200_ctx* ctx, int B, int H, int W) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (B <= 0 || H <= 0 || W <= 0 || (long long)H * W > (1ll << 30))
        return fail(ctx, ESACB200_ERR_ARG, "reserve_loss_async: bad sizes B=%d H=%d W=%d", B, H, W);
    esacb200_ctx* a = nullptr;
    const int rc = reserve_context(ctx, "loss_async", &a);
    if (rc) return rc;
    const long long parts = (long long)B * reproj_max_blocks(H * W);
    return loss_workspace(ctx, a, std::max(reproj_layout(B, parts).end, coord_layout(B, parts).end), false, "reserve_loss_async");
} ESAC_ABI_CATCH(ctx)

int esacb200_reproj_loss_async(esacb200_ctx* ctx, int B, const float* const* coords, float* const* grads, const int* H,
                               const int* W, const float* gt_poses, const int32_t* shifts, const float* cameras, int sub,
                               float cut, float maxReproj, float minDepth, double* out_losses, int32_t* out_status) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "reproj_loss_async";
    if (!coords || !H || !W) return fail(ctx, ESACB200_ERR_ARG, "%s: null pointer or size array", what);
    if (B <= 0 || B > 65535 || sub <= 0) return fail(ctx, ESACB200_ERR_ARG, "%s: bad sizes B=%d sub=%d", what, B, sub);
    const void* ptrs[] = {gt_poses, shifts, cameras, out_losses, out_status};
    const char* names[] = {"gt_poses", "shifts", "cameras", "out_losses", "out_status"};
    int rc = reproj_sizes(ctx, what, B, H, W);
    if (!rc) rc = device_args(ctx, what, 5, ptrs, names);
    if (!rc) rc = device_images(ctx, what, "coords", (const void* const*)coords, B);
    if (!rc && grads) rc = device_images(ctx, what, "grads", (const void* const*)grads, B);
    if (rc) return rc;
    esacb200_ctx* a = nullptr;
    bool capturing = false;
    if ((rc = begin_loss_async(ctx, a, capturing))) return rc;
    std::vector<ReprojImage> recs, ordered;
    std::vector<char> vec;
    const long long parts = reproj_records(B, coords, grads, H, W, recs, vec);
    int n_vec, max_vec, max_sc;
    order_by_path(recs, vec, ordered, n_vec, max_vec, max_sc);
    const LossLayout L = reproj_layout(B, parts);
    if ((rc = loss_workspace(ctx, a, L.end, capturing, what))) return rc;
    if (capturing) a->loss_frozen = true;
    char* base = (char*)a->loss_ws.p;
    ReprojImage* d_rec = (ReprojImage*)(base + L.rec);
    double* losses = (double*)(base + L.loss);
    int* bad = (int*)(base + L.flags);
    CK(cudaMemsetAsync(base, 0, L.img, a->stream));
    a->st.kernel_launches +=
        launch_reproj_prep(ordered.data(), B, d_rec, gt_poses, shifts, cameras, (float*)(base + L.img), bad, a->stream);
    reproj_launches(a, base, L, B, n_vec, max_vec, max_sc, sub, cut, maxReproj, minDepth);
    launch_reproj_finish(d_rec, B, grads != nullptr, losses, bad, out_losses, out_status, a->stream);
    a->st.kernel_launches += 1;
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_coord_loss_async(esacb200_ctx* ctx, int B, const float* const* pred, const int* Hp, const int* Wp,
                              const float* const* gt, const int* Hg, const int* Wg, float* const* grads, float cut,
                              double* out_losses, int64_t* out_counts) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "coord_loss_async";
    if (!pred || !gt || !Hp || !Wp || !Hg || !Wg) return fail(ctx, ESACB200_ERR_ARG, "%s: null pointer or size array", what);
    if (B <= 0 || B > 65535) return fail(ctx, ESACB200_ERR_ARG, "%s: bad sizes B=%d", what, B);
    const void* ptrs[] = {out_losses, out_counts};
    const char* names[] = {"out_losses", "out_counts"};
    int rc = coord_sizes(ctx, what, B, Hp, Wp, Hg, Wg);
    if (!rc) rc = device_args(ctx, what, 2, ptrs, names, 2u);
    if (!rc) rc = device_images(ctx, what, "pred", (const void* const*)pred, B);
    if (!rc) rc = device_images(ctx, what, "gt", (const void* const*)gt, B);
    if (!rc && grads) rc = device_images(ctx, what, "grads", (const void* const*)grads, B);
    if (rc) return rc;
    esacb200_ctx* a = nullptr;
    bool capturing = false;
    if ((rc = begin_loss_async(ctx, a, capturing))) return rc;
    std::vector<CoordImage> recs, ordered;
    std::vector<char> vec;
    const long long parts = coord_records(B, pred, gt, grads, Hp, Wp, Hg, Wg, recs, vec);
    int n_vec, max_vec, max_sc;
    order_by_path(recs, vec, ordered, n_vec, max_vec, max_sc);
    const LossLayout L = coord_layout(B, parts);
    if ((rc = loss_workspace(ctx, a, L.end, capturing, what))) return rc;
    if (capturing) a->loss_frozen = true;
    char* base = (char*)a->loss_ws.p;
    CK(cudaMemsetAsync(base, 0, L.rec, a->stream));
    a->st.kernel_launches += launch_coord_prep(ordered.data(), B, (CoordImage*)(base + L.rec), a->stream);
    coord_launches(a, base, L, B, grads != nullptr, n_vec, max_vec, max_sc, cut);
    launch_coord_finish(B, (const double*)(base + L.loss), (const long long*)(base + L.flags), out_losses, (long long*)out_counts,
                        a->stream);
    a->st.kernel_launches += 1;
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// The getters below read only what the last call on the context wrote (LastCall).
static int last_call_left(esacb200_ctx* ctx, bool wrote, const char* what) {
    return wrote ? 0 : fail(ctx, ESACB200_ERR_ARG, "the last call on this context left no %s", what);
}

int esacb200_copy_last_scores(esacb200_ctx* ctx, double* dst, int M) try {
    if (!ctx || !dst) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    int rc = last_call_left(ctx, ctx->last.scored, "scores");
    if (rc) return rc;
    if (M != ctx->last.M) return fail(ctx, ESACB200_ERR_ARG, "last call had M=%d, asked for %d", ctx->last.M, M);
    CK(cudaMemcpyAsync(dst, ctx->scores.p, (size_t)M * 8, cudaMemcpyDefault, ctx->stream));
    if (!is_device_ptr(dst)) CK(cudaStreamSynchronize(ctx->stream));
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_get_refine_profile(esacb200_ctx* ctx, long long* out16) try {
    if (!ctx || !out16) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!ctx->prof.p) return fail(ctx, ESACB200_ERR_ARG, "no refinement ran with option refine_profile = 1");
    CK(cudaMemcpy(out16, ctx->prof.p, 16 * 8, cudaMemcpyDeviceToHost));
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_get_stats(esacb200_ctx* ctx, esacb200_stats* out) {
    if (!ctx || !out) return ESACB200_ERR_ARG;
    *out = ctx->st;
    return ESACB200_OK;
}

int esacb200_get_sample_trace(esacb200_ctx* ctx, unsigned long long* out512) try {
    if (!ctx || !out512) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!ctx->smp_trace.p) return fail(ctx, ESACB200_ERR_ARG, "no sampling ran with option sample_trace = 1");
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaMemcpy(out512, ctx->smp_trace.p, 512 * 8, cudaMemcpyDeviceToHost));
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_get_sample_profile(esacb200_ctx* ctx, long long* out8) try {
    if (!ctx || !out8) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    for (int i = 0; i < 8; ++i) out8[i] = 0;
    int rc = last_call_left(ctx, ctx->last.drew, "sampling profile");
    if (rc) return rc;
    const int G = ctx->last.lanes, M = ctx->last.M, Mg = ctx->last.lane_cap;
    CK(cudaStreamSynchronize(ctx->stream));
    const size_t per_group_ints = (size_t)2 * Mg + SC_COUNT;
    for (int g = 0; g < G; ++g) {
        int c[SC_COUNT];
        const int* src = ctx->smp_int.as<int>() + 4 * (size_t)M + g * per_group_ints + 2 * (size_t)Mg;
        CK(cudaMemcpy(c, src, sizeof(c), cudaMemcpyDeviceToHost));
        out8[0] += (unsigned)c[SC_PREFILTERED];
        out8[1] += (unsigned)c[SC_JUDGED];
        out8[2] = out8[2] > c[SC_WAVES] ? out8[2] : c[SC_WAVES];
        out8[3] += c[SC_UNRESOLVED];
        out8[4] += c[SC_STAGED];
    }
    out8[5] = G;
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_get_hypotheses(esacb200_ctx* ctx, double* poses6, int32_t* cells, int32_t* tries, double* scores,
                            double* probs, double* refined6, double* losses) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    int rc = last_call_left(ctx, ctx->last.drew, "hypotheses");
    if (!rc && losses) rc = last_call_left(ctx, ctx->last.losses, "per-hypothesis losses");
    if (rc) return rc;
    const int M = ctx->last.M;
    if (poses6) CK(cudaMemcpy(poses6, ctx->poses.p, (size_t)M * sizeof(Pose), cudaMemcpyDeviceToHost));
    if (cells) CK(cudaMemcpy(cells, ctx->cells.p, (size_t)M * 32, cudaMemcpyDeviceToHost));
    if (tries) CK(cudaMemcpy(tries, ctx->tries.p, (size_t)M * 4, cudaMemcpyDeviceToHost));
    if (scores) CK(cudaMemcpy(scores, ctx->scores.p, (size_t)M * 8, cudaMemcpyDeviceToHost));
    if (probs) CK(cudaMemcpy(probs, ctx->probs.p, (size_t)M * 8, cudaMemcpyDeviceToHost));
    if (refined6) CK(cudaMemcpy(refined6, ctx->poses_ref.p, (size_t)M * sizeof(Pose), cudaMemcpyDeviceToHost));
    if (losses) CK(cudaMemcpy(losses, ctx->losses.p, (size_t)M * 8, cudaMemcpyDeviceToHost));
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

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

}  // extern "C"
