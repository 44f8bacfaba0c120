// One step of a device-resident image set (include/esac_b200.h: esacb200_data_step_async).
#include <math.h>

#include "capi_internal.h"

using namespace esacb200;
using namespace esacb200::capi;

namespace {

// The device address of set storage: device memory as it is, mapped pinned host memory through its device alias.
int storage_ptr(esacb200_ctx* ctx, const char* what, const char* name, const void* p, const void** out) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        at.type = cudaMemoryTypeUnregistered;
    }
    if (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) {
        *out = p;
        return 0;
    }
    if (at.type == cudaMemoryTypeHost && at.devicePointer) {
        *out = at.devicePointer;
        return 0;
    }
    return fail(ctx, ESACB200_ERR_ARG, "%s: %s is neither device memory nor mapped pinned host memory", what, name);
}

}  // namespace

int esacb200_data_step_async(esacb200_ctx* ctx, const uint8_t* pixels, const float* gt, const esacb200_data_image* images,
                             int64_t n_images, int group, int H, int W, int gt_h, int gt_w, const float* mean,
                             const float* std, int n_attach, const float* const* attach, const int64_t* attach_numel,
                             const esacb200_data_row* plan, int64_t capacity, esacb200_data_state* state, int B,
                             int64_t* work, float* out_image, int32_t* out_shifts, float* out_cameras, float* out_poses,
                             float* out_coords, int64_t* out_scenes, int64_t* out_indices, float* const* out_attach,
                             int32_t* out_status) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "data_step_async";
    if (!pixels || !mean || !std) return fail(ctx, ESACB200_ERR_ARG, "%s: pixels, mean and std must not be null", what);
    if ((gt == nullptr) != (out_coords == nullptr))
        return fail(ctx, ESACB200_ERR_ARG, "%s: gt and out_coords must both be given or both be null", what);
    if (B < 1 || B > ESACB200_DATA_MAX_BATCH)
        return fail(ctx, ESACB200_ERR_ARG, "%s: batch of %d images outside [1, %d]", what, B, ESACB200_DATA_MAX_BATCH);
    if (n_images < 1 || n_images > INT32_MAX)
        return fail(ctx, ESACB200_ERR_ARG, "%s: %lld images outside [1, %d]", what, (long long)n_images, INT32_MAX);
    if (capacity < 1) return fail(ctx, ESACB200_ERR_ARG, "%s: plan capacity %lld must be positive", what, (long long)capacity);
    if (group < 0) return fail(ctx, ESACB200_ERR_ARG, "%s: group %d is negative", what, group);
    if (H < 1 || W < 1 || H > ESACB200_DATA_MAX_SIDE || W > ESACB200_DATA_MAX_SIDE)
        return fail(ctx, ESACB200_ERR_ARG, "%s: image %dx%d, need sides in [1, %d]", what, H, W, ESACB200_DATA_MAX_SIDE);
    if (gt && (gt_h < 1 || gt_w < 1 || gt_h > ESACB200_DATA_MAX_SIDE || gt_w > ESACB200_DATA_MAX_SIDE))
        return fail(ctx, ESACB200_ERR_ARG, "%s: ground truth %dx%d, need sides in [1, %d]", what, gt_h, gt_w,
                    ESACB200_DATA_MAX_SIDE);
    for (int c = 0; c < 3; ++c)
        if (!isfinite(mean[c]) || !isfinite(std[c]) || std[c] == 0.f)
            return fail(ctx, ESACB200_ERR_ARG, "%s: mean[%d] = %g, std[%d] = %g: need finite values and a nonzero std", what,
                        c, mean[c], c, std[c]);
    if (n_attach < 0 || n_attach > ESACB200_DATA_MAX_ATTACH)
        return fail(ctx, ESACB200_ERR_ARG, "%s: %d attachments outside [0, %d]", what, n_attach, ESACB200_DATA_MAX_ATTACH);
    if (n_attach > 0 && (!attach || !attach_numel || !out_attach))
        return fail(ctx, ESACB200_ERR_ARG, "%s: %d attachments but a null attachment array", what, n_attach);
    const void* ptrs[] = {images, plan, state, work, out_image, out_shifts, out_cameras, out_poses, out_scenes, out_indices,
                          out_status, out_coords};
    const char* names[] = {"images", "plan", "state", "work", "out_image", "out_shifts", "out_cameras", "out_poses",
                           "out_scenes", "out_indices", "out_status", "out_coords"};
    int rc = device_args(ctx, what, 12, ptrs, names, 1u << 11);
    if (rc) return rc;
    DataArgs a{};
    const void* p = nullptr;
    if ((rc = storage_ptr(ctx, what, "pixels", pixels, &p))) return rc;
    a.pixels = (const unsigned char*)p;
    a.gt = nullptr;
    if (gt) {
        if ((rc = storage_ptr(ctx, what, "gt", gt, &p))) return rc;
        a.gt = (const float*)p;
    }
    for (int k = 0; k < n_attach; ++k) {
        if (!attach[k] || !out_attach[k] || attach_numel[k] < 1)
            return fail(ctx, ESACB200_ERR_ARG, "%s: attachment %d: null pointer or %lld floats per image", what, k,
                        (long long)attach_numel[k]);
        if ((rc = storage_ptr(ctx, what, "an attachment", attach[k], &p))) return rc;
        a.attach[k] = (const float*)p;
        a.attach_numel[k] = attach_numel[k];
        if (!is_device_ptr(out_attach[k]))
            return fail(ctx, ESACB200_ERR_ARG, "%s takes device pointers only: out_attach[%d] is host memory", what, k);
        a.out_attach[k] = out_attach[k];
    }
    a.images = images;
    a.n_images = n_images;
    a.group = group;
    a.H = H;
    a.W = W;
    a.gt_h = gt ? gt_h : 0;
    a.gt_w = gt ? gt_w : 0;
    for (int c = 0; c < 3; ++c) {
        a.mean[c] = mean[c];
        a.std[c] = std[c];
    }
    a.n_attach = n_attach;
    a.plan = plan;
    a.capacity = capacity;
    a.state = state;
    a.B = B;
    a.sums = (unsigned long long*)work;
    a.image = out_image;
    a.shifts = out_shifts;
    a.cameras = out_cameras;
    a.poses = out_poses;
    a.coords = out_coords;
    a.scenes = (long long*)out_scenes;
    a.indices = (long long*)out_indices;
    a.status = out_status;
    launch_data_step(a, ctx->stream);
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)
