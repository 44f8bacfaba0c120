// Inference of the gating network (include/esac_b200.h: esacb200_gating_packed_floats, _workspace_bytes, _pack,
// _forward_async).
#include "capi_internal.h"

using namespace esacb200;
using namespace esacb200::capi;

namespace {

bool gating_sizes_ok(int B, int E, int capacity, int H, int W) {
    return B >= 1 && B <= ESACB200_EXPERTS_MAX_PAIRS && E >= 1 && E <= ESACB200_EXPERTS_MAX &&
           (capacity == 1 || capacity == 2) && H >= 1 && W >= 1 && H <= ESACB200_EXPERTS_MAX_SIDE &&
           W <= ESACB200_EXPERTS_MAX_SIDE;
}

}  // namespace

int64_t esacb200_gating_packed_floats(int E, int capacity) {
    if (E < 1 || E > ESACB200_EXPERTS_MAX || (capacity != 1 && capacity != 2)) return -1;
    return gating_packed_floats(E, capacity);
}

int64_t esacb200_gating_workspace_bytes(int B, int E, int capacity, int H, int W) {
    if (!gating_sizes_ok(B, E, capacity, H, W)) return -1;
    return experts_hdr_bytes(B) + (long long)B * gating_shape(H, W, capacity).image_floats * 4;
}

int esacb200_gating_pack(esacb200_ctx* ctx, int E, int capacity, const float* const* params, float* packed) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "gating_pack";
    if (E < 1 || E > ESACB200_EXPERTS_MAX)
        return fail(ctx, ESACB200_ERR_ARG, "%s: E=%d outside [1, %d]", what, E, ESACB200_EXPERTS_MAX);
    if (capacity != 1 && capacity != 2) return fail(ctx, ESACB200_ERR_ARG, "%s: capacity %d is not 1 or 2", what, capacity);
    if (!params) return fail(ctx, ESACB200_ERR_ARG, "%s: params is null", what);
    const void* ptrs[] = {packed};
    const char* names[] = {"packed"};
    int rc = device_args(ctx, what, 1, ptrs, names);
    if (rc) return rc;
    if ((uintptr_t)packed % 16) return fail(ctx, ESACB200_ERR_ARG, "%s: packed must be 16-byte aligned", what);
    for (int i = 0; i < ESACB200_GATING_TENSORS; ++i)
        if (!params[i]) return fail(ctx, ESACB200_ERR_ARG, "%s: tensor %d is null", what, i);
    // stage every layer in torch's layout back to back, then permute on the device; the gaps between segments are zero
    std::vector<long long> w_at(kGatingLayers), b_at(kGatingLayers);
    long long total = 0;
    for (int l = 0; l < kGatingLayers; ++l) {
        const GatingLayer d = gating_layer(l, E, capacity);
        w_at[l] = total;
        total += (long long)d.cout * d.cin * d.k * d.k;
        b_at[l] = total;
        total += d.cout;
    }
    DevBuf staged;
    CK(staged.ensure((size_t)total * sizeof(float)));
    CK(cudaMemsetAsync(packed, 0, gating_packed_floats(E, capacity) * sizeof(float), ctx->stream));
    for (int l = 0; l < kGatingLayers; ++l) {
        const GatingLayer d = gating_layer(l, E, capacity);
        CK(cudaMemcpyAsync(staged.as<float>() + w_at[l], params[2 * l], (size_t)d.cout * d.cin * d.k * d.k * sizeof(float),
                           cudaMemcpyDefault, ctx->stream));
        CK(cudaMemcpyAsync(staged.as<float>() + b_at[l], params[2 * l + 1], d.cout * sizeof(float), cudaMemcpyDefault,
                           ctx->stream));
        launch_gating_pack(staged.as<float>(), packed, E, capacity, l, w_at[l], b_at[l], ctx->stream);
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(ctx->stream));  // the staging buffer dies here
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_gating_forward_async(esacb200_ctx* ctx, int B, int E, int capacity, int H, int W, const float* image,
                                  const float* packed, void* workspace, int64_t workspace_bytes, float* out_log_probs,
                                  float* out_probs) {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "gating_forward_async";
    if (!gating_sizes_ok(B, E, capacity, H, W))
        return fail(ctx, ESACB200_ERR_ARG,
                    "%s: B=%d E=%d capacity=%d H=%d W=%d: need B <= %d, E <= %d, capacity 1 or 2 and sides <= %d", what, B,
                    E, capacity, H, W, ESACB200_EXPERTS_MAX_PAIRS, ESACB200_EXPERTS_MAX, ESACB200_EXPERTS_MAX_SIDE);
    const int64_t need = esacb200_gating_workspace_bytes(B, E, capacity, H, W);
    if (workspace_bytes < need)
        return fail(ctx, ESACB200_ERR_ARG, "%s: workspace of %lld bytes, B=%d at %dx%d needs %lld (reserve it first)", what,
                    (long long)workspace_bytes, B, H, W, (long long)need);
    const void* ptrs[] = {image, packed, workspace, out_log_probs, out_probs};
    const char* names[] = {"image", "packed", "workspace", "out_log_probs", "out_probs"};
    const int rc = device_args(ctx, what, 5, ptrs, names, 1u << 4);
    if (rc) return rc;
    if ((uintptr_t)workspace % 256 || (uintptr_t)packed % 16)
        return fail(ctx, ESACB200_ERR_ARG, "%s: workspace must be 256-byte and packed 16-byte aligned", what);
    GatingArgs a{};
    a.B = B;
    a.E = E;
    a.c = capacity;
    a.H = H;
    a.W = W;
    a.image = image;
    a.packed = packed;
    a.ws_hdr = (int*)workspace;
    a.ws_images = (float*)((char*)workspace + experts_hdr_bytes(B));
    a.out_log = out_log_probs;
    a.out_prob = out_probs;
    launch_gating_forward(a, ctx->stream);
    CK(cudaGetLastError());
    return ESACB200_OK;
}
