// Inference of a stack of experts (include/esac_b200.h: esacb200_experts_pack, _workspace_bytes, _forward_async).
#include "capi_internal.h"

using namespace esacb200;
using namespace esacb200::capi;

namespace {

// Sizes one call accepts: grids run one CTA row per (image, expert) pair.
bool experts_sizes_ok(int B, int E, int H, int W) {
    return B >= 1 && E >= 1 && E <= ESACB200_EXPERTS_MAX && H >= 1 && W >= 1 && H <= ESACB200_EXPERTS_MAX_SIDE &&
           W <= ESACB200_EXPERTS_MAX_SIDE && (long long)B * E <= ESACB200_EXPERTS_MAX_PAIRS;
}

}  // namespace

int64_t esacb200_experts_packed_floats(int E) {
    if (E < 1 || E > ESACB200_EXPERTS_MAX) return -1;
    return experts_packed_floats(E);
}

int64_t esacb200_experts_workspace_bytes(int B, int E, int H, int W) {
    if (!experts_sizes_ok(B, E, H, W)) return -1;
    return experts_hdr_bytes(B * E) + (long long)B * E * experts_shape(H, W).pair_floats * 4;
}

int esacb200_experts_pack(esacb200_ctx* ctx, int E, const float* const* params, float* packed) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "experts_pack";
    if (E < 1 || E > ESACB200_EXPERTS_MAX)
        return fail(ctx, ESACB200_ERR_ARG, "%s: E=%d outside [1, %d]", what, E, ESACB200_EXPERTS_MAX);
    if (!params) return fail(ctx, ESACB200_ERR_ARG, "%s: params is null", what);
    const void* ptrs[] = {packed};
    const char* names[] = {"packed"};
    int rc = device_args(ctx, what, 1, ptrs, names);
    if (rc) return rc;
    for (int i = 0; i < E * ESACB200_EXPERT_TENSORS; ++i)
        if (!params[i]) return fail(ctx, ESACB200_ERR_ARG, "%s: tensor %d of expert %d is null", what,
                                    i % ESACB200_EXPERT_TENSORS, i / ESACB200_EXPERT_TENSORS);
    // stage every layer's weights and biases of all experts back to back in torch's layouts, then permute on the device
    std::vector<long long> w_at(kExpertLayers), b_at(kExpertLayers);
    long long total = 0;
    for (int l = 0; l < kExpertLayers; ++l) {
        w_at[l] = total;
        total += E * expert_layer(l).w_count();
        b_at[l] = total;
        total += (long long)E * expert_layer(l).cout;
    }
    DevBuf staged;
    CK(staged.ensure((size_t)total * sizeof(float)));
    // the padding between segments is never read, but the packed weights are one well-defined array: zero it
    CK(cudaMemsetAsync(packed, 0, experts_packed_floats(E) * sizeof(float), ctx->stream));
    for (int l = 0; l < kExpertLayers; ++l) {
        const ExpertLayer d = expert_layer(l);
        for (int e = 0; e < E; ++e) {
            const float* const* t = params + (size_t)e * ESACB200_EXPERT_TENSORS;
            CK(cudaMemcpyAsync(staged.as<float>() + w_at[l] + e * d.w_count(), t[2 * l], d.w_count() * sizeof(float),
                               cudaMemcpyDefault, ctx->stream));
            CK(cudaMemcpyAsync(staged.as<float>() + b_at[l] + (long long)e * d.cout, t[2 * l + 1], d.cout * sizeof(float),
                               cudaMemcpyDefault, ctx->stream));
        }
        launch_experts_pack(staged.as<float>(), packed, E, l, w_at[l], b_at[l], ctx->stream);
        CK(cudaGetLastError());
    }
    for (int e = 0; e < E; ++e)
        CK(cudaMemcpyAsync(packed + expert_mean_off(E) + 3LL * e, params[(size_t)e * ESACB200_EXPERT_TENSORS + 2 * kExpertLayers],
                           3 * sizeof(float), cudaMemcpyDefault, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));  // the staging buffer dies here
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_experts_forward_async(esacb200_ctx* ctx, int B, int E, int H, int W, const float* image, int image_batch,
                                   const float* hist, const float* packed, void* workspace, int64_t workspace_bytes,
                                   float* out) {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "experts_forward_async";
    if (!experts_sizes_ok(B, E, H, W))
        return fail(ctx, ESACB200_ERR_ARG, "%s: B=%d E=%d H=%d W=%d: need E <= %d, sides <= %d and B * E <= %d", what, B, E,
                    H, W, ESACB200_EXPERTS_MAX, ESACB200_EXPERTS_MAX_SIDE, ESACB200_EXPERTS_MAX_PAIRS);
    if (image_batch != 1 && image_batch != B)
        return fail(ctx, ESACB200_ERR_ARG, "%s: %d images for a batch of %d (need 1 or B)", what, image_batch, B);
    const int64_t need = esacb200_experts_workspace_bytes(B, E, H, W);
    if (workspace_bytes < need)
        return fail(ctx, ESACB200_ERR_ARG, "%s: workspace of %lld bytes, B=%d E=%d at %dx%d needs %lld (reserve it first)",
                    what, (long long)workspace_bytes, B, E, H, W, (long long)need);
    const void* ptrs[] = {image, packed, workspace, out, hist};
    const char* names[] = {"image", "packed", "workspace", "out", "hist"};
    const int rc = device_args(ctx, what, 5, ptrs, names, 1u << 4);
    if (rc) return rc;
    if ((uintptr_t)workspace % 256 || (uintptr_t)packed % 16)
        return fail(ctx, ESACB200_ERR_ARG, "%s: workspace must be 256-byte and packed 16-byte aligned", what);
    ExpertsArgs a;
    a.B = B;
    a.E = E;
    a.H = H;
    a.W = W;
    a.image = image;
    a.image_batch = image_batch;
    a.hist = hist;
    a.packed = packed;
    a.ws_hdr = (int*)workspace;
    a.ws_pairs = (float*)((char*)workspace + experts_hdr_bytes(B * E));
    a.pair_floats = experts_shape(H, W).pair_floats;
    a.out = out;
    launch_experts_forward(a, ctx->stream);
    CK(cudaGetLastError());
    return ESACB200_OK;
}
