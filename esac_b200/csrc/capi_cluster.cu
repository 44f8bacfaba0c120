// Clustering a large environment into experts (include/esac_b200.h: esacb200_cluster_stats_ragged, esacb200_kmeans2,
// esacb200_cluster_targets).  Each call checks all of its arguments before it enqueues anything and synchronises once.
#include <algorithm>
#include <vector>

#include "capi_internal.h"

using namespace esacb200;
using namespace esacb200::capi;

int esacb200_cluster_stats_ragged(esacb200_ctx* ctx, int B, const float* const* maps, const int* H, const int* W,
                                  float* out_median, float* out_mean, int32_t* out_count, int32_t* out_status) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "cluster_stats_ragged";
    if (!maps || !H || !W || !out_median || !out_mean || !out_count || !out_status)
        return fail(ctx, ESACB200_ERR_ARG, "%s: null pointer argument", what);
    if (B < 1) return fail(ctx, ESACB200_ERR_ARG, "%s: batch of %d maps, need at least 1", what, B);
    int max_cells = 1;
    std::vector<size_t> bytes((size_t)B);
    for (int b = 0; b < B; ++b) {
        if (H[b] < 1 || W[b] < 1 || (long long)H[b] * W[b] > (1ll << 30))
            return fail(ctx, ESACB200_ERR_ARG, "%s: map %d is %dx%d, need 1 <= H*W <= 2^30", what, b, H[b], W[b]);
        max_cells = std::max(max_cells, H[b] * W[b]);
        bytes[b] = (size_t)3 * H[b] * W[b] * sizeof(float);
    }
    bool dev = false;
    int rc = pointer_kind(ctx, (const void* const*)maps, B, "maps", dev);
    if (rc) return rc;
    begin_call(ctx);
    std::vector<const float*> d_maps;
    std::vector<size_t> off;
    if ((rc = stage_images(ctx, maps, bytes, dev, true, ctx->coords, d_maps, off))) return rc;
    mark(ctx, EV_H2D);
    std::vector<ClusterMap> recs((size_t)B);
    for (int b = 0; b < B; ++b) recs[b] = {d_maps[b], H[b], W[b]};
    const size_t rec_bytes = recs.size() * sizeof(ClusterMap), out_off = (rec_bytes + 15) & ~(size_t)15,
                 out_bytes = (size_t)B * sizeof(ClusterStats);
    CK(ctx->scratch.ensure(out_off + out_bytes));
    char* base = (char*)ctx->scratch.p;
    ClusterStats* d_out = (ClusterStats*)(base + out_off);
    CK(cudaMemcpyAsync(base, recs.data(), rec_bytes, cudaMemcpyHostToDevice, ctx->stream));
    launch_cluster_stats((const ClusterMap*)base, B, std::min(max_cells, kStatsSmemKeys), d_out, ctx->stream);
    CK(cudaGetLastError());
    std::vector<ClusterStats> h((size_t)B);
    CK(cudaMemcpyAsync(h.data(), d_out, out_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    std::vector<float> med((size_t)B * 3), mean((size_t)B * 3);
    std::vector<int32_t> count((size_t)B), status((size_t)B);
    for (int b = 0; b < B; ++b) {
        for (int c = 0; c < 3; ++c) {
            med[(size_t)b * 3 + c] = h[b].median[c];
            mean[(size_t)b * 3 + c] = h[b].mean[c];
        }
        count[b] = h[b].count;
        status[b] = h[b].status;
    }
    CK(cudaMemcpy(out_median, med.data(), med.size() * sizeof(float), cudaMemcpyDefault));
    CK(cudaMemcpy(out_mean, mean.data(), mean.size() * sizeof(float), cudaMemcpyDefault));
    CK(cudaMemcpy(out_count, count.data(), count.size() * sizeof(int32_t), cudaMemcpyDefault));
    CK(cudaMemcpy(out_status, status.data(), status.size() * sizeof(int32_t), cudaMemcpyDefault));
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_kmeans2(esacb200_ctx* ctx, int n, const float* points, uint64_t seed, int split, int attempts, int max_iter,
                     double eps, int32_t* out_labels, float* out_centres, double* out_compactness) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "kmeans2";
    if (n < 2) return fail(ctx, ESACB200_ERR_ARG, "%s: %d points, need at least 2", what, n);
    if (attempts < 1 || attempts > 4096) return fail(ctx, ESACB200_ERR_ARG, "%s: attempts=%d outside [1, 4096]", what, attempts);
    if (max_iter < 1) return fail(ctx, ESACB200_ERR_ARG, "%s: max_iter=%d, need at least 1", what, max_iter);
    if (!(eps >= 0.)) return fail(ctx, ESACB200_ERR_ARG, "%s: eps=%g, need eps >= 0", what, eps);
    if (split < 0) return fail(ctx, ESACB200_ERR_ARG, "%s: split=%d must not be negative", what, split);
    const void* ptrs[] = {points, out_labels, out_centres, out_compactness};
    const char* names[] = {"points", "labels", "centres", "compactness"};
    int rc = device_args(ctx, what, 4, ptrs, names);
    if (rc) return rc;
    begin_call(ctx);
    CK(ctx->scratch.ensure((size_t)attempts * sizeof(KmeansAttempt)));
    KmeansArgs a;
    a.points = points;
    a.n = n;
    a.attempts = attempts;
    a.max_iter = max_iter;
    a.eps2 = eps * eps;
    a.seed = seed;
    a.split = (unsigned)split;
    a.att = ctx->scratch.as<KmeansAttempt>();
    a.labels = out_labels;
    a.centres = out_centres;
    a.compactness = out_compactness;
    launch_kmeans2(a, ctx->stream);
    CK(cudaGetLastError());
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_cluster_targets(esacb200_ctx* ctx, int N, const float* means, const int64_t* labels, int K, float softness,
                             float* out_centres, float* out_sizes, float* out_probs) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "cluster_targets";
    if (N < 1) return fail(ctx, ESACB200_ERR_ARG, "%s: %d images, need at least 1", what, N);
    if (K < 1 || K > kTargetsMaxClusters)
        return fail(ctx, ESACB200_ERR_ARG, "%s: K=%d outside [1, %d]", what, K, kTargetsMaxClusters);
    if (!(softness > 0.f)) return fail(ctx, ESACB200_ERR_ARG, "%s: softness=%g, need softness > 0", what, (double)softness);
    const void* ptrs[] = {means, labels, out_centres, out_sizes, out_probs};
    const char* names[] = {"means", "labels", "centres", "sizes", "probs"};
    int rc = device_args(ctx, what, 5, ptrs, names);
    if (rc) return rc;
    // every label in [0, K) and every cluster non-empty: checked on the host before the launch
    std::vector<int64_t> h((size_t)N);
    CK(cudaMemcpyAsync(h.data(), labels, h.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    std::vector<int> sizes((size_t)K, 0);
    for (int i = 0; i < N; ++i) {
        if (h[i] < 0 || h[i] >= K)
            return fail(ctx, ESACB200_ERR_ARG, "%s: image %d has label %lld, outside [0, %d)", what, i, (long long)h[i], K);
        ++sizes[h[i]];
    }
    for (int k = 0; k < K; ++k)
        if (!sizes[k]) return fail(ctx, ESACB200_ERR_ARG, "%s: cluster %d has no image", what, k);
    begin_call(ctx);
    ClusterTargetsArgs a;
    a.means = means;
    a.labels = (const long long*)labels;
    a.N = N;
    a.K = K;
    a.softness = softness;
    a.centres = out_centres;
    a.sizes = out_sizes;
    a.probs = out_probs;
    launch_cluster_targets(a, ctx->stream);
    CK(cudaGetLastError());
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)
