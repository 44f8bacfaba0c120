// One step of a device-resident image set (include/esac_b200.h: esacb200_data_step_async): the item path of the reference's
// datasets (room_dataset.py:134-207, cluster_dataset.py:245-275) and util.random_shift (util.py:4-11) for B plan rows, with
// the random draws taken from the plan the host made.  Five launches:
//   head      checks the rows (status), writes the small per-image outputs and clears the contrast sums;
//   contrast  the exact integer sum of L over each contrast row's image as the ops before contrast leave it;
//   compose   jitter, ToTensor + Normalize and the zero-pad shift, one output pixel per thread;
//   gather    the ground-truth map and the attachments;
//   advance   moves the plan position by B.
// Every launch after the head reads the status the head wrote and does nothing unless it is 0; every launch before the
// advance reads the position the head read.  The pixel arithmetic is PIL's ImageEnhance (Image.blend) and torchvision's
// to_tensor / normalize, stated in float32 with round-to-nearest intrinsics so that no multiply-add is contracted.
#include "esac_internal.h"

namespace esacb200 {

namespace {

constexpr int kHeadThreads = 128;
constexpr int kThreads = 256;
constexpr int kMaxGridX = 1024;

// PIL's RGB -> L (Convert.c, rgb2l: ITU-R 601-2 luma in 16-bit fixed point).
__device__ __forceinline__ int luma(int r, int g, int b) { return (19595 * r + 38470 * g + 7471 * b + 0x8000) >> 16; }

// Image.blend(a, b, f) on one channel (Blend.c): a + f (b - a) in float32, truncated when 0 <= f <= 1 (the result then lies
// between a and b), else clipped to [0, 255] first.
__device__ __forceinline__ int blend(int a, int b, float f) {
    const float t = __fadd_rn((float)a, __fmul_rn(f, (float)(b - a)));
    if (f >= 0.f && f <= 1.f) return (int)t;
    return t <= 0.f ? 0 : (t >= 255.f ? 255 : (int)t);
}

// Ops 0 .. n-1 of a row on one pixel; `mean` is the contrast grey (used only when contrast is among them).
__device__ __forceinline__ void jitter(const esacb200_data_row& row, int n, int mean, int& r, int& g, int& b) {
    for (int k = 0; k < n; ++k) {
        const float f = row.factors[k];
        int a = 0;
        if (row.ops[k] == ESACB200_DATA_CONTRAST) a = mean;
        else if (row.ops[k] == ESACB200_DATA_SATURATION) a = luma(r, g, b);
        else if (row.ops[k] != ESACB200_DATA_BRIGHTNESS) continue;
        r = blend(a, r, f);
        g = blend(a, g, f);
        b = blend(a, b, f);
    }
}

__device__ __forceinline__ int row_ops(const esacb200_data_row& row) { return min(max(row.n_ops, 0), 3); }

// The position of the row a contrast op takes, or -1.
__device__ __forceinline__ int contrast_at(const esacb200_data_row& row) {
    const int n = row_ops(row);
    for (int k = 0; k < n; ++k)
        if (row.ops[k] == ESACB200_DATA_CONTRAST) return k;
    return -1;
}

__global__ void __launch_bounds__(kHeadThreads) data_head_kernel(const __grid_constant__ DataArgs a) {
    const long long pos = a.state->position, rows = a.state->rows;
    const bool exhausted = pos < 0 || rows > a.capacity || pos + a.B > rows;  // the same for every thread
    bool bad = false;
    if (!exhausted) {
        for (int b = threadIdx.x; b < a.B; b += blockDim.x) {
            const long long i = a.plan[pos + b].image;
            if (i < 0 || i >= a.n_images) {
                bad = true;
                continue;
            }
            const esacb200_data_image& m = a.images[i];
            bad |= m.group != a.group || m.H != a.H || m.W != a.W || m.gt_h != a.gt_h || m.gt_w != a.gt_w ||
                   (a.coords && m.gt < 0);
        }
    }
    bad = __syncthreads_or(bad);
    const int status = exhausted ? 1 : (bad ? 2 : 0);
    if (threadIdx.x == 0) *a.status = status;
    if (status) return;
    for (int b = threadIdx.x; b < a.B; b += blockDim.x) {
        const esacb200_data_row row = a.plan[pos + b];
        const esacb200_data_image& m = a.images[row.image];
        a.indices[b] = row.image;
        a.scenes[b] = m.scene;
        a.shifts[2 * b] = row.padX;
        a.shifts[2 * b + 1] = row.padY;
        a.cameras[3 * b] = (float)m.focal;
        a.cameras[3 * b + 1] = (float)a.W / 2.f;
        a.cameras[3 * b + 2] = (float)a.H / 2.f;
        for (int j = 0; j < 16; ++j) a.poses[16 * b + j] = m.pose[j];
        a.sums[b] = 0ull;
    }
}

__global__ void __launch_bounds__(kThreads) data_contrast_kernel(const __grid_constant__ DataArgs a) {
    if (*a.status) return;
    const int b = blockIdx.y;
    const esacb200_data_row row = a.plan[a.state->position + b];
    const int k = contrast_at(row);
    if (k < 0) return;
    const unsigned char* __restrict__ src = a.pixels + a.images[row.image].pixels;
    const int N = a.H * a.W;
    unsigned long long s = 0;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        int r = src[3 * p], g = src[3 * p + 1], bl = src[3 * p + 2];
        jitter(row, k, 0, r, g, bl);
        s += (unsigned)luma(r, g, bl);
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    __shared__ unsigned long long warp_sums[kThreads / 32];
    if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (int w = 0; w < kThreads / 32; ++w) t += warp_sums[w];
        atomicAdd(a.sums + b, t);  // integer: the total does not depend on the order the blocks land in
    }
}

__global__ void __launch_bounds__(kThreads) data_compose_kernel(const __grid_constant__ DataArgs a) {
    if (*a.status) return;
    const int b = blockIdx.y;
    const int N = a.H * a.W;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= N) return;
    const esacb200_data_row row = a.plan[a.state->position + b];
    // ImageEnhance.Contrast's grey: int(ImageStat mean + 0.5), the mean an exact int / int division in fp64
    const int mean = contrast_at(row) < 0 ? 0 : (int)((double)a.sums[b] / (double)N + 0.5);
    const int y = p / a.W, x = p - y * a.W;
    const int sy = y - row.padY, sx = x - row.padX;  // nn.ZeroPad2d((padX, -padX, padY, -padY))
    float v[3] = {0.f, 0.f, 0.f};
    if (sy >= 0 && sy < a.H && sx >= 0 && sx < a.W) {
        const unsigned char* __restrict__ src = a.pixels + a.images[row.image].pixels + 3 * ((size_t)sy * a.W + sx);
        int c[3] = {src[0], src[1], src[2]};
        jitter(row, row_ops(row), mean, c[0], c[1], c[2]);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch)
            v[ch] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)c[ch], 255.f), a.mean[ch]), a.std[ch]);
    }
    float* out = a.image + (size_t)b * 3 * N + p;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) out[(size_t)ch * N] = v[ch];
}

__global__ void __launch_bounds__(kThreads) data_gather_kernel(const __grid_constant__ DataArgs a) {
    if (*a.status) return;
    const int b = blockIdx.y, z = blockIdx.z;
    const long long image = a.plan[a.state->position + b].image;
    const float* __restrict__ src;
    float* dst;
    long long n;
    if (z == 0) {
        if (!a.coords) return;
        n = 3ll * a.gt_h * a.gt_w;
        src = a.gt + a.images[image].gt;
        dst = a.coords + b * n;
    } else {
        n = a.attach_numel[z - 1];
        src = a.attach[z - 1] + image * n;
        dst = a.out_attach[z - 1] + b * n;
    }
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        dst[i] = src[i];
}

__global__ void data_advance_kernel(const __grid_constant__ DataArgs a) {
    if (*a.status == 0) a.state->position += a.B;
}

int blocks_for(long long n) { return (int)min((long long)kMaxGridX, max(1ll, (n + kThreads - 1) / kThreads)); }

}  // namespace

void launch_data_step(const DataArgs& a, cudaStream_t st) {
    const int N = a.H * a.W;
    data_head_kernel<<<1, kHeadThreads, 0, st>>>(a);
    data_contrast_kernel<<<dim3(blocks_for((N + 7) / 8), a.B), kThreads, 0, st>>>(a);
    data_compose_kernel<<<dim3((N + kThreads - 1) / kThreads, a.B), kThreads, 0, st>>>(a);
    long long most = a.coords ? 3ll * a.gt_h * a.gt_w : 0;
    for (int k = 0; k < a.n_attach; ++k) most = max(most, a.attach_numel[k]);
    if (most > 0) data_gather_kernel<<<dim3(blocks_for(most), a.B, 1 + a.n_attach), kThreads, 0, st>>>(a);
    data_advance_kernel<<<1, 1, 0, st>>>(a);
}

}  // namespace esacb200
