// Rendering ground-truth scene-coordinate maps from an SfM reconstruction (include/esac_b200.h: esacb200_render_init_maps).
// The call checks all of its arguments, allocates a workspace of its own (not the context's: it holds 16 B per cell and
// 8 B per observation, which the context would otherwise keep for the rest of the process), enqueues the upload and the
// four passes, synchronises once and frees the workspace before it returns.
#include <vector>

#include "capi_internal.h"

using namespace esacb200;
using namespace esacb200::capi;

namespace {

size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }

}  // namespace

int esacb200_render_init_maps(esacb200_ctx* ctx, int C, const float* points, int64_t P, const int64_t* offsets,
                              const int32_t* indices, const float* poses, const float* focal, const float* out_scale,
                              const int32_t* H, const int32_t* W, float* out_maps, float* out_zbuf, int32_t* out_count,
                              int32_t* out_status) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "render_init_maps";
    if (C < 1) return fail(ctx, ESACB200_ERR_ARG, "%s: %d cameras, need at least 1", what, C);
    if (!offsets || !poses || !focal || !out_scale || !H || !W || !out_maps || !out_count || !out_status)
        return fail(ctx, ESACB200_ERR_ARG, "%s: null pointer argument", what);
    if (P < 0 || P > ESACB200_RENDER_MAX_OBS)
        return fail(ctx, ESACB200_ERR_ARG, "%s: P=%lld points outside [0, %d]", what, (long long)P, ESACB200_RENDER_MAX_OBS);
    if (offsets[0] != 0) return fail(ctx, ESACB200_ERR_ARG, "%s: offsets[0]=%lld, need 0", what, (long long)offsets[0]);
    for (int c = 0; c < C; ++c)
        if (offsets[c + 1] < offsets[c])
            return fail(ctx, ESACB200_ERR_ARG, "%s: offsets decrease at camera %d (%lld > %lld)", what, c,
                        (long long)offsets[c], (long long)offsets[c + 1]);
    const int64_t V = offsets[C];
    if (V > ESACB200_RENDER_MAX_OBS)
        return fail(ctx, ESACB200_ERR_ARG, "%s: V=%lld observations, more than %d", what, (long long)V, ESACB200_RENDER_MAX_OBS);
    if (V > 0 && !indices)
        return fail(ctx, ESACB200_ERR_ARG, "%s: %lld observations but indices is null", what, (long long)V);
    if (P > 0 && !points) return fail(ctx, ESACB200_ERR_ARG, "%s: %lld points but points is null", what, (long long)P);
    int64_t cells = 0;
    std::vector<RenderCamera> cams((size_t)C);
    for (int c = 0; c < C; ++c) {
        if (H[c] < 1 || W[c] < 1 || H[c] > ESACB200_RENDER_MAX_SIDE || W[c] > ESACB200_RENDER_MAX_SIDE)
            return fail(ctx, ESACB200_ERR_ARG, "%s: camera %d map is %dx%d, need sides in [1, %d]", what, c, H[c], W[c],
                        ESACB200_RENDER_MAX_SIDE);
        RenderCamera& k = cams[c];
        for (int j = 0; j < 12; ++j) k.pose[j] = poses[(size_t)c * 12 + j];
        k.f = focal[c];
        k.scale = out_scale[c];
        k.half_w = (float)W[c] / 2.f;
        k.half_h = (float)H[c] / 2.f;
        k.H = H[c];
        k.W = W[c];
        k.cell0 = (int)cells;
        k.pad = 0;
        cells += (int64_t)H[c] * W[c];
        if (cells > ESACB200_RENDER_MAX_CELLS)
            return fail(ctx, ESACB200_ERR_ARG, "%s: the maps of cameras 0..%d hold more than %d cells", what, c,
                        ESACB200_RENDER_MAX_CELLS);
    }
    if (!is_device_ptr(out_maps)) return fail(ctx, ESACB200_ERR_ARG, "%s: out_maps is host memory, need device memory", what);
    if (out_zbuf && !is_device_ptr(out_zbuf))
        return fail(ctx, ESACB200_ERR_ARG, "%s: out_zbuf is host memory, need device memory", what);
    const bool dev_points = V > 0 && P > 0 && is_device_ptr(points), dev_indices = V > 0 && is_device_ptr(indices);
    begin_call(ctx);

    // The whole workspace, allocated before anything is enqueued and freed (after the synchronisation) when ws goes out of
    // scope.
    std::vector<int> offs32((size_t)C + 1);
    for (int c = 0; c <= C; ++c) offs32[c] = (int)offsets[c];
    const size_t b_cams = align16((size_t)C * sizeof(RenderCamera)), b_offs = align16(((size_t)C + 1) * sizeof(int)),
                 b_cam_ints = align16((size_t)C * sizeof(int)), b_cell_u64 = align16((size_t)cells * 8),
                 b_cell_i32 = align16((size_t)cells * 4), b_obs = align16((size_t)V * 4),
                 b_points = dev_points || V == 0 ? 0 : align16((size_t)P * 3 * sizeof(float)),
                 b_indices = dev_indices || V == 0 ? 0 : b_obs;
    const size_t total = b_cams + b_offs + 2 * b_cam_ints + b_cell_u64 + 2 * b_cell_i32 + 2 * b_obs + b_points + b_indices;
    DevBuf ws;
    CK(cudaMalloc(&ws.p, total));
    ws.cap = total;
    char* p = (char*)ws.p;
    auto carve = [&p](size_t b) { char* q = p; p += b; return q; };
    RenderArgs a;
    a.cams = (const RenderCamera*)carve(b_cams);
    a.offsets = (const int*)carve(b_offs);
    a.count = (int*)carve(b_cam_ints);
    a.status = (int*)carve(b_cam_ints);
    a.key = (unsigned long long*)carve(b_cell_u64);
    a.first_neg = (unsigned*)carve(b_cell_i32);
    a.last_zero = (int*)carve(b_cell_i32);
    a.obs_cell = (int*)carve(b_obs);
    a.obs_z = (float*)carve(b_obs);
    a.points = dev_points ? points : (const float*)carve(b_points);
    a.indices = dev_indices ? indices : (const int*)carve(b_indices);
    a.C = C;
    a.P = (int)P;
    a.V = (int)V;
    a.cells = (int)cells;
    a.maps = out_maps;
    a.zbuf = out_zbuf;
    CK(cudaMemcpyAsync((void*)a.cams, cams.data(), cams.size() * sizeof(RenderCamera), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync((void*)a.offsets, offs32.data(), offs32.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    if (b_points && P > 0)
        CK(cudaMemcpyAsync((void*)a.points, points, (size_t)P * 3 * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    if (b_indices) CK(cudaMemcpyAsync((void*)a.indices, indices, (size_t)V * 4, cudaMemcpyHostToDevice, ctx->stream));
    mark(ctx, EV_H2D);
    launch_render(a, ctx->stream);
    CK(cudaGetLastError());
    mark(ctx, EV_END);
    CK(cudaMemcpyAsync(out_count, a.count, (size_t)C * sizeof(int), cudaMemcpyDefault, ctx->stream));
    CK(cudaMemcpyAsync(out_status, a.status, (size_t)C * sizeof(int), cudaMemcpyDefault, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)
