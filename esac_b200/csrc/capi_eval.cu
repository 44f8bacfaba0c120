// Test-time pose evaluation (include/esac_b200.h: esacb200_eval_poses_async, esacb200_eval_poses).
#include "capi_internal.h"

using namespace esacb200;
using namespace esacb200::capi;

namespace {

// Checks the arguments and enqueues the evaluation kernel on the context's stream; nothing is enqueued on an error.
int eval_enqueue(esacb200_ctx* ctx, const char* what, int B, const float* out_poses, const float* gt_poses,
                 const int64_t* experts, const int64_t* scenes, const float* hist, int E, const int32_t* status,
                 double* records, int64_t capacity, int64_t* state) {
    const void* ptrs[] = {out_poses, gt_poses, experts, scenes, records, state, hist, status};
    const char* names[] = {"out_poses", "gt_poses", "experts", "scenes", "records", "state", "hist", "status"};
    const int rc = device_args(ctx, what, 8, ptrs, names, 0xC0u);
    if (rc) return rc;
    if (B <= 0 || B > (1 << 24)) return fail(ctx, ESACB200_ERR_ARG, "%s: batch of %d images outside [1, %d]", what, B, 1 << 24);
    if (capacity <= 0) return fail(ctx, ESACB200_ERR_ARG, "%s: record capacity %lld must be positive", what, (long long)capacity);
    if (hist && (E <= 0 || E > ESACB200_GATE_MAX))
        return fail(ctx, ESACB200_ERR_ARG, "%s: E=%d outside [1, %d] with a histogram", what, E, ESACB200_GATE_MAX);
    EvalArgs a;
    a.out_poses = out_poses;
    a.gt_poses = gt_poses;
    a.experts = (const long long*)experts;
    a.scenes = (const long long*)scenes;
    a.hist = hist;
    a.status = status;
    a.B = B;
    a.E = hist ? E : 0;
    a.records = (EvalRecord*)records;
    a.capacity = capacity;
    a.state = (EvalState*)state;
    launch_eval_poses(a, ctx->stream);
    CK(cudaGetLastError());
    return ESACB200_OK;
}

}  // namespace

int esacb200_eval_poses_async(esacb200_ctx* ctx, int B, const float* out_poses, const float* gt_poses, const int64_t* experts,
                              const int64_t* scenes, const float* hist, int E, const int32_t* status, double* records,
                              int64_t capacity, int64_t* state) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    return eval_enqueue(ctx, "eval_poses_async", B, out_poses, gt_poses, experts, scenes, hist, E, status, records, capacity,
                        state);
} ESAC_ABI_CATCH(ctx)

int esacb200_eval_poses(esacb200_ctx* ctx, int B, const float* out_poses, const float* gt_poses, const int64_t* experts,
                        const int64_t* scenes, const float* hist, int E, const int32_t* status, double* records,
                        int64_t capacity, int64_t* state) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const int rc = eval_enqueue(ctx, "eval_poses", B, out_poses, gt_poses, experts, scenes, hist, E, status, records, capacity,
                                state);
    if (rc) return rc;
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)
