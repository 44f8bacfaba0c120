// The kernels around the two loss kernels in the stream-ordered losses (esacb200_reproj_loss_async / _coord_loss_async).
//
// The eager calls build their per-image records on the host and upload them with a copy; a captured copy from host memory
// would read that memory again at every replay, after it is gone.  Here the records travel as kernel parameters of a prep
// kernel, in chunks under the 4 KB parameter limit, so each graph holds its own copy, and the prep kernel writes them into
// the workspace.  The reprojection loss's prep kernel also inverts the image's ground truth there, from the caller's device
// arrays, with the host's arithmetic (reproj_img_row).  The loss kernels themselves are the eager ones, unchanged; a finish
// kernel copies their per-image results to the caller's arrays.
#include <math.h>

#include "esac_internal.h"

namespace esacb200 {

namespace {

template <class Rec>
struct RecChunk {
    Rec r[loss_chunk<Rec>()];
};

// One block per record of this chunk; thread 0 does the work.  Writes the record to recs[blockIdx.x] and image b's row of
// img; a singular or NaN ground truth sets bad[b] and gives the record no blocks, so the loss kernel skips the image.
__global__ void __launch_bounds__(32) reproj_prep_kernel(const RecChunk<ReprojImage> chunk, ReprojImage* __restrict__ recs,
                                                         const float* __restrict__ gt16, const int* __restrict__ shifts,
                                                         const float* __restrict__ cameras, float* __restrict__ img,
                                                         int* __restrict__ bad) {
    if (threadIdx.x != 0) return;
    ReprojImage r = chunk.r[blockIdx.x];
    const int b = r.b;
    float* row = img + (size_t)b * kReprojImgFloats;
    const float* cam = cameras + 3 * (size_t)b;
    const bool ok = reproj_img_row(gt16 + 16 * (size_t)b, shifts[2 * b], shifts[2 * b + 1], cam[0], cam[1], cam[2], row);
    for (int i = 17; i < kReprojImgFloats; ++i) row[i] = 0.f;
    if (!ok) r.blocks = 0;
    bad[b] = ok ? 0 : 1;
    recs[blockIdx.x] = r;
}

// grid = (gblocks, B), row blockIdx.y = record blockIdx.y of image b: block 0 writes the loss (NaN when bad) and the
// status; the blocks of a bad image zero its gradient: elements of type T, each the rounded (0 * s) of a scaled call.
template <class T>
__global__ void __launch_bounds__(256) reproj_finish_kernel(const ReprojImage* __restrict__ recs, const double* __restrict__ losses,
                                                            const int* __restrict__ bad, const float* __restrict__ grad_scale,
                                                            double* __restrict__ out_losses, int* __restrict__ status) {
    const ReprojImage r = recs[blockIdx.y];
    const int b = r.b;
    const bool is_bad = bad[b] != 0;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        out_losses[b] = is_bad ? (double)NAN : losses[b];
        status[b] = is_bad ? 1 : 0;
    }
    if (!is_bad || !r.grads) return;
    const size_t n = 3 * (size_t)r.N;
    const T zero = loss_out<T>(grad_scale ? __fmul_rn(0.f, *grad_scale) : 0.f);
    T* g = static_cast<T*>(r.grads);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) g[i] = zero;
}

// One block: records 0 .. n-1 of this chunk into recs.
__global__ void __launch_bounds__(64) coord_prep_kernel(const RecChunk<CoordImage> chunk, int n, CoordImage* __restrict__ recs) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) recs[i] = chunk.r[i];
}

__global__ void __launch_bounds__(256) coord_finish_kernel(int B, const double* __restrict__ losses, const long long* __restrict__ counts,
                                                           double* __restrict__ out_losses, long long* __restrict__ out_counts) {
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        out_losses[b] = losses[b];
        if (out_counts) out_counts[b] = counts[b];
    }
}

// Blocks per image that zero a bad image's gradient (a rare case: a few per SM keep it short without a grid per size).
constexpr int kZeroBlocks = 32;

}  // namespace

int launch_reproj_prep(const ReprojImage* host_recs, int n, ReprojImage* recs, const float* gt16, const int* shifts,
                       const float* cameras, float* img, int* bad, cudaStream_t st) {
    constexpr int chunk = loss_chunk<ReprojImage>();
    int launches = 0;
    for (int i = 0; i < n; i += chunk, ++launches) {
        RecChunk<ReprojImage> c{};
        const int k = n - i < chunk ? n - i : chunk;
        for (int j = 0; j < k; ++j) c.r[j] = host_recs[i + j];
        reproj_prep_kernel<<<k, 32, 0, st>>>(c, recs + i, gt16, shifts, cameras, img, bad);
    }
    return launches;
}

void launch_reproj_finish(const ReprojImage* recs, int B, bool grads, int dtype, const float* grad_scale, const double* losses,
                          const int* bad, double* out_losses, int* status, cudaStream_t st) {
    const dim3 grid(grads ? kZeroBlocks : 1, B);
    if (dtype == kLossF32)
        reproj_finish_kernel<float><<<grid, 256, 0, st>>>(recs, losses, bad, nullptr, out_losses, status);
    else if (dtype == kLossF16)
        reproj_finish_kernel<__half><<<grid, 256, 0, st>>>(recs, losses, bad, grad_scale, out_losses, status);
    else
        reproj_finish_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(recs, losses, bad, grad_scale, out_losses, status);
}

int launch_coord_prep(const CoordImage* host_recs, int n, CoordImage* recs, cudaStream_t st) {
    constexpr int chunk = loss_chunk<CoordImage>();
    int launches = 0;
    for (int i = 0; i < n; i += chunk, ++launches) {
        RecChunk<CoordImage> c{};
        const int k = n - i < chunk ? n - i : chunk;
        for (int j = 0; j < k; ++j) c.r[j] = host_recs[i + j];
        coord_prep_kernel<<<1, 64, 0, st>>>(c, k, recs + i);
    }
    return launches;
}

void launch_coord_finish(int B, const double* losses, const long long* counts, double* out_losses, long long* out_counts,
                         cudaStream_t st) {
    coord_finish_kernel<<<1, 256, 0, st>>>(B, losses, counts, out_losses, out_counts);
}

}  // namespace esacb200
