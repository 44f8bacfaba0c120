// The context of libesac_b200.so's C ABI (include/esac_b200.h): its lifecycle, options and getters, and the frame every entry
// point shares -- the error message, the stage timers and the last-call record.
#include <climits>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <new>

#include "capi_internal.h"

using namespace esacb200;
using namespace esacb200::capi;

namespace esacb200::capi {

int fail(esacb200_ctx* c, int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(c->err, sizeof(c->err), fmt, ap);
    va_end(ap);
    return code;
}

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

static float span(esacb200_ctx* c, int a, int b) {
    if (!c->ev_used[a] || !c->ev_used[b]) return 0.f;
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, c->ev[a], c->ev[b]) != cudaSuccess) {
        cudaGetLastError();
        return 0.f;
    }
    return ms;
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

// The getters read only what the last call on the context wrote (LastCall): `wrote` is its flag for `what`.
int last_call_left(esacb200_ctx* ctx, bool wrote, const char* what) {
    return wrote ? 0 : fail(ctx, ESACB200_ERR_ARG, "the last call on this context left no %s", what);
}

}  // namespace esacb200::capi

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
    else if (!strcmp(key, "sample_hint")) o.sample_hint = v > 0 ? (v < 1.99 ? (float)v : 1.99f) : 0.f;  // fraction of tau, < kPrefilterMargin
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
    int lo[2] = {INT_MAX, INT_MAX}, hi[2] = {INT_MIN, INT_MIN};
    for (size_t i = 0; i < (size_t)M * T * 8; ++i) {
        const int c = (int)(i & 1);
        lo[c] = cells[i] < lo[c] ? cells[i] : lo[c];
        hi[c] = cells[i] > hi[c] ? cells[i] : hi[c];
    }
    CK(ctx->inject.ensure(bytes));
    CK(cudaMemcpy(ctx->inject.p, cells, bytes, cudaMemcpyHostToDevice));
    ctx->inj_M = M;
    ctx->inj_T = T;
    for (int c = 0; c < 2; ++c) { ctx->inj_lo[c] = lo[c]; ctx->inj_hi[c] = hi[c]; }
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_device_info(esacb200_ctx* ctx, int* sm_count, char* name, int name_len) {
    if (!ctx) return ESACB200_ERR_ARG;
    if (sm_count) *sm_count = ctx->sm_count;
    if (name && name_len > 0) snprintf(name, name_len, "%s", ctx->dev_name);
    return ESACB200_OK;
}

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

}  // extern "C"
