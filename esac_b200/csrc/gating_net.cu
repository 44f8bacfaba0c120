// Inference of the reference's gating network (code/gating.py: Gating) for B images, one launch per stage:
//
//   experts_active     the image list that experts_conv_kernel walks (every image: the gating runs as one "expert")
//   gating_front       conv1 .. conv3 (3 -> 8 -> 16 -> 32 channels, full resolution to /4) in fp32 FMAs, one 8x8 tile of
//                      conv3's output per CTA: conv1's and conv2's cells of the tile live only in shared memory, so conv3's
//                      NHWC output is the front end's one write to global memory
//   experts_conv       conv4, res1_conv1..3 at /8 (Cin 32 or 64c): the experts' implicit-GEMM kernel, TF32 operands with
//                      fp32 accumulation, fed the gating's layers as data
//   gating_pool        tanh (capacity 1), then fixed-order fp32 sums over chunks of kGatingPoolPixels cells of the /8 map
//   gating_head        the chunks' sums in order over the cell count, fc1, fc2 (ReLU), fc3 and log_softmax in fp32, one CTA
//                      per image; exp(log_p) when asked
//
// No split-K and no atomics: every output of image b is computed by the same threads in the same order whatever the batch,
// so image b's log-probabilities are bitwise those of a call on it alone.
#include "esac_internal.h"

namespace esacb200 {

namespace {

// The front end's tile: kT3 x kT3 cells of conv3's output read kT2 x kT2 cells of conv2's, which read kT1 x kT1 of conv1's,
// which read kT0 x kT0 pixels.
constexpr int kT3 = 8, kT2 = 2 * kT3 + 1, kT1 = 2 * kT2 + 1, kT0 = kT1 + 2;
constexpr int kFrontThreads = 256;
// shared floats: the three layers' weights and biases, conv1's tile, then the image's tile, later conv2's, in one region
constexpr int kW1 = 27 * 8, kW2 = 72 * 16, kW3 = 144 * 32;
constexpr int kFrontW = kW1 + 8 + kW2 + 16 + kW3 + 32;
constexpr int kFrontT1 = 8 * kT1 * kT1;
constexpr int kFrontT02 = 3 * kT0 * kT0 > 16 * kT2 * kT2 ? 3 * kT0 * kT0 : 16 * kT2 * kT2;
constexpr int kFrontSmem = (kFrontW + kFrontT1 + kFrontT02) * (int)sizeof(float);  // 80 KiB: two CTAs per SM
static_assert(kFrontThreads == 4 * kT3 * kT3, "conv3: one thread per cell and 8-channel group");

__device__ __forceinline__ void fma8(float* acc, float v, const float* w) {
    const float4 w0 = *(const float4*)w, w1 = *(const float4*)(w + 4);
    acc[0] = fmaf(w0.x, v, acc[0]);
    acc[1] = fmaf(w0.y, v, acc[1]);
    acc[2] = fmaf(w0.z, v, acc[2]);
    acc[3] = fmaf(w0.w, v, acc[3]);
    acc[4] = fmaf(w1.x, v, acc[4]);
    acc[5] = fmaf(w1.y, v, acc[5]);
    acc[6] = fmaf(w1.z, v, acc[6]);
    acc[7] = fmaf(w1.w, v, acc[7]);
}

__global__ void __launch_bounds__(kFrontThreads, 2) gating_front_kernel(GatingArgs a, GatingShape s) {
    extern __shared__ float4 front_smem4[];
    float* w1 = (float*)front_smem4;
    float* b1 = w1 + kW1;
    float* w2 = b1 + 8;
    float* b2 = w2 + kW2;
    float* w3 = b2 + 16;
    float* b3 = w3 + kW3;
    float* t1 = w1 + kFrontW;   // conv1 [8][kT1 * kT1]
    float* t0 = t1 + kFrontT1;  // image [3][kT0 * kT0]
    float* t2 = t0;             // conv2 [16][kT2 * kT2], once conv1 has read the image
    const int tid = threadIdx.x, b = blockIdx.y;
    const int tiles_x = (s.w[2] + kT3 - 1) / kT3;
    const int Y3 = (blockIdx.x / tiles_x) * kT3, X3 = (blockIdx.x % tiles_x) * kT3;
    const int H = a.H, W = a.W;

    const float* src[6] = {a.packed + a.w_off[0], a.packed + a.b_off[0], a.packed + a.w_off[1],
                           a.packed + a.b_off[1], a.packed + a.w_off[2], a.packed + a.b_off[2]};
    const int len[6] = {kW1, 8, kW2, 16, kW3, 32};
    float* dst = w1;
#pragma unroll
    for (int q = 0; q < 6; ++q) {
        for (int i = tid; i < len[q]; i += kFrontThreads) dst[i] = __ldg(src[q] + i);
        dst += len[q];
    }
    const float* img = a.image + (size_t)b * 3 * H * W;
    for (int i = tid; i < 3 * kT0 * kT0; i += kFrontThreads) {
        const int c = i / (kT0 * kT0), r = i - c * kT0 * kT0;
        const int gy = 4 * Y3 - 4 + r / kT0, gx = 4 * X3 - 4 + r % kT0;
        t0[i] = gy >= 0 && gy < H && gx >= 0 && gx < W ? __ldg(img + ((size_t)c * H + gy) * W + gx) : 0.f;
    }
    __syncthreads();

    // conv1: one cell, 8 channels per item; cells outside the image are conv2's zero padding
    for (int i = tid; i < kT1 * kT1; i += kFrontThreads) {
        const int ty = i / kT1, tx = i - ty * kT1;
        const int gy = 4 * Y3 - 3 + ty, gx = 4 * X3 - 3 + tx;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
#pragma unroll
            for (int tap = 0; tap < 9; ++tap)
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    fma8(acc, t0[c * kT0 * kT0 + (ty + tap / 3) * kT0 + tx + tap % 3], w1 + (tap * 3 + c) * 8);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = fmaxf(acc[j] + b1[j], 0.f);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) t1[j * kT1 * kT1 + i] = acc[j];
    }
    __syncthreads();

    // conv2: one cell and 8 of its 16 channels per item
    for (int it = tid; it < 2 * kT2 * kT2; it += kFrontThreads) {
        const int half = it / (kT2 * kT2), i = it - half * kT2 * kT2;
        const int ty = i / kT2, tx = i - ty * kT2;
        const int gy = 2 * Y3 - 1 + ty, gx = 2 * X3 - 1 + tx;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (gy >= 0 && gy < s.h[1] && gx >= 0 && gx < s.w[1]) {
#pragma unroll
            for (int tap = 0; tap < 9; ++tap)
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    fma8(acc, t1[c * kT1 * kT1 + (2 * ty + tap / 3) * kT1 + 2 * tx + tap % 3], w2 + (tap * 8 + c) * 16 + half * 8);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = fmaxf(acc[j] + b2[half * 8 + j], 0.f);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) t2[(half * 8 + j) * kT2 * kT2 + i] = acc[j];
    }
    __syncthreads();

    // conv3: one cell and 8 of its 32 channels per thread (a warp shares the channel group), NHWC into the workspace
    const int g = tid >> 6, cy = (tid & 63) >> 3, cx = tid & 7;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 3
    for (int tap = 0; tap < 9; ++tap)
#pragma unroll
        for (int c = 0; c < 16; ++c)
            fma8(acc, t2[c * kT2 * kT2 + (2 * cy + tap / 3) * kT2 + 2 * cx + tap % 3], w3 + (tap * 16 + c) * 32 + g * 8);
    const int y3 = Y3 + cy, x3 = X3 + cx;
    if (y3 < s.h[2] && x3 < s.w[2]) {
        float4* out = (float4*)(a.ws_images + (size_t)b * s.image_floats + s.a3 + ((size_t)y3 * s.w[2] + x3) * 32 + g * 8);
        out[0] = make_float4(fmaxf(acc[0] + b3[g * 8], 0.f), fmaxf(acc[1] + b3[g * 8 + 1], 0.f),
                             fmaxf(acc[2] + b3[g * 8 + 2], 0.f), fmaxf(acc[3] + b3[g * 8 + 3], 0.f));
        out[1] = make_float4(fmaxf(acc[4] + b3[g * 8 + 4], 0.f), fmaxf(acc[5] + b3[g * 8 + 5], 0.f),
                             fmaxf(acc[6] + b3[g * 8 + 6], 0.f), fmaxf(acc[7] + b3[g * 8 + 7], 0.f));
    }
}

// One CTA per chunk of kGatingPoolPixels cells of one image: thread t sums channel t % C over the chunk's cells
// t / C, t / C + 256 / C, ... in order; the 256 / C partial sums of a channel are then added in order.
constexpr int kPoolThreads = 256;
__global__ void __launch_bounds__(kPoolThreads) gating_pool_kernel(GatingArgs a, GatingShape s) {
    __shared__ float red[kPoolThreads];
    const int b = blockIdx.y, chunk = blockIdx.x, tid = threadIdx.x;
    const int C = 64 * a.c, G = kPoolThreads / C;
    const int ch = tid % C, r = tid / C;
    const int P = s.h[3] * s.w[3];
    const int p0 = chunk * kGatingPoolPixels, p1 = min(P, p0 + kGatingPoolPixels);
    float* img = a.ws_images + (size_t)b * s.image_floats;
    const float* y = img + s.y;
    float sum = 0.f;
    for (int p = p0 + r; p < p1; p += G) {
        const float v = y[(size_t)p * C + ch];
        sum += a.c == 1 ? tanhf(v) : v;
    }
    red[tid] = sum;
    __syncthreads();
    if (tid < C) {
        float t = red[tid];
        for (int q = 1; q < G; ++q) t += red[q * C + tid];
        img[s.part + (size_t)chunk * C + tid] = t;
    }
}

constexpr int kHeadThreads = 256;
constexpr int kHeadWarps = kHeadThreads / 32;

// Fixed-order block reductions: a shuffle tree in each warp, then warp 0's lanes in order.
template <bool MAX>
__device__ __forceinline__ float head_reduce(float v, float* red) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        const float o = __shfl_xor_sync(0xffffffffu, v, d);
        v = MAX ? fmaxf(v, o) : v + o;
    }
    __syncthreads();  // red may still be read by the previous reduction
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = red[0];
#pragma unroll
    for (int w = 1; w < kHeadWarps; ++w) t = MAX ? fmaxf(t, red[w]) : t + red[w];
    return t;
}

// 64c pooled channels -> fc1 -> fc2 (64c^2, ReLU) -> fc3 (E) -> log_softmax: one CTA per image, one thread per output.
__global__ void __launch_bounds__(kHeadThreads) gating_head_kernel(GatingArgs a, GatingShape s) {
    __shared__ float v0[kHeadThreads], v1[kHeadThreads];
    __shared__ float z[ESACB200_EXPERTS_MAX];
    __shared__ float red[kHeadWarps];
    const int b = blockIdx.x, t = threadIdx.x;
    const int C = 64 * a.c, F = 64 * a.c * a.c, E = a.E;
    const float* part = a.ws_images + (size_t)b * s.image_floats + s.part;
    if (t < C) {
        float sum = 0.f;
        for (int k = 0; k < s.chunks; ++k) sum += part[(size_t)k * C + t];
        v0[t] = sum / (float)(s.h[3] * s.w[3]);
    }
    __syncthreads();
    if (t < F) {
        const float* w = a.packed + a.w_off[7];
        float acc = 0.f;
        for (int i = 0; i < C; ++i) acc = fmaf(w[i * F + t], v0[i], acc);
        v1[t] = fmaxf(acc + a.packed[a.b_off[7] + t], 0.f);
    }
    __syncthreads();
    if (t < F) {
        const float* w = a.packed + a.w_off[8];
        float acc = 0.f;
        for (int i = 0; i < F; ++i) acc = fmaf(w[i * F + t], v1[i], acc);
        v0[t] = fmaxf(acc + a.packed[a.b_off[8] + t], 0.f);
    }
    __syncthreads();
    float m = -INFINITY;
    for (int e = t; e < E; e += kHeadThreads) {
        const float* w = a.packed + a.w_off[9];
        float acc = 0.f;
        for (int i = 0; i < F; ++i) acc = fmaf(w[(size_t)i * E + e], v0[i], acc);
        z[e] = acc + a.packed[a.b_off[9] + e];
        m = fmaxf(m, z[e]);
    }
    m = head_reduce<true>(m, red);
    float sum = 0.f;
    for (int e = t; e < E; e += kHeadThreads) sum += expf(z[e] - m);
    const float lse = logf(head_reduce<false>(sum, red));
    for (int e = t; e < E; e += kHeadThreads) {
        const float lp = (z[e] - m) - lse;
        a.out_log[(size_t)b * E + e] = lp;
        if (a.out_prob) a.out_prob[(size_t)b * E + e] = expf(lp);
    }
}

// Layer l from torch's [Cout][Cin][k][k] into its packed layout (kind 0: [k][k][Cin][Cout]; 1: [Cout][k][k][Cin], TF32;
// 2: [Cin][Cout]).
__global__ void gating_pack_kernel(const float* staged, float* packed, int cin, int cout, int k, int kind, long long w_off,
                                   long long b_off, long long staged_w, long long staged_b) {
    const int kk = k * k;
    const long long n = (long long)cout * cin * kk;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int tap = (int)(i % kk);
        const long long r = i / kk;
        const int ci = (int)(r % cin), co = (int)(r / cin);
        const float v = staged[staged_w + i];
        if (kind == 0) packed[w_off + ((long long)tap * cin + ci) * cout + co] = v;
        else if (kind == 1) packed[w_off + ((long long)co * kk + tap) * cin + ci] = __uint_as_float(to_tf32(v));
        else packed[w_off + (long long)ci * cout + co] = v;
    }
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < cout; i += (long long)gridDim.x * blockDim.x)
        packed[b_off + i] = staged[staged_b + i];
}

}  // namespace

void launch_gating_pack(const float* staged, float* packed, int E, int c, int l, long long staged_w, long long staged_b,
                        cudaStream_t st) {
    const GatingLayer d = gating_layer(l, E, c);
    const int kind = l < 3 ? 0 : l < 7 ? 1 : 2;
    gating_pack_kernel<<<132, 256, 0, st>>>(staged, packed, d.cin, d.cout, d.k, kind, d.w_off, d.b_off, staged_w, staged_b);
}

void launch_gating_forward(GatingArgs a, cudaStream_t st) {
    const GatingShape s = gating_shape(a.H, a.W, a.c);
    for (int l = 0; l < kGatingLayers; ++l) {
        a.w_off[l] = gating_layer(l, a.E, a.c).w_off;
        a.b_off[l] = gating_layer(l, a.E, a.c).b_off;
    }
    ExpertsArgs e{};
    e.B = a.B;
    e.E = 1;
    e.H = a.H;
    e.W = a.W;
    e.packed = a.packed;
    e.ws_hdr = a.ws_hdr;
    e.ws_pairs = a.ws_images;
    e.pair_floats = s.image_floats;
    launch_experts_active(e, st);
    // per call: the attribute belongs to the current device's context, and a process may drive several devices
    cudaFuncSetAttribute(gating_front_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFrontSmem);
    const int tiles = ((s.h[2] + kT3 - 1) / kT3) * ((s.w[2] + kT3 - 1) / kT3);
    gating_front_kernel<<<dim3(tiles, a.B), kFrontThreads, kFrontSmem, st>>>(a, s);
    // conv4 (/4 -> /8), then res1_conv1..3 at /8: (layer, input, output)
    const struct { int l; long long in, out; } steps[] = {{3, s.a3, s.x}, {4, s.x, s.y}, {5, s.y, s.x}, {6, s.x, s.y}};
    for (const auto& q : steps) {
        const GatingLayer d = gating_layer(q.l, a.E, a.c);
        ExpertsConvLayer L;
        L.cin = d.cin;
        L.cout = d.cout;
        L.hin = s.h[q.l == 3 ? 2 : 3];
        L.win = s.w[q.l == 3 ? 2 : 3];
        L.hout = s.h[3];
        L.wout = s.w[3];
        L.in_off = q.in;
        L.out_off = q.out;
        L.res_off = -1;
        L.w_off = d.w_off;
        L.b_off = d.b_off;
        L.relu = true;
        launch_experts_conv(e, L, d.k, d.stride, st);
    }
    gating_pool_kernel<<<dim3(s.chunks, a.B), kPoolThreads, 0, st>>>(a, s);
    gating_head_kernel<<<a.B, kHeadThreads, 0, st>>>(a, s);
}

}  // namespace esacb200
