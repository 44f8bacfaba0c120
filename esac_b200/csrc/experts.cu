// Inference of a stack of E scene-coordinate experts (the reference's Expert FCN, code/expert.py) for B images: only the
// (image, expert) pairs whose hypothesis count is positive run, and every layer of every active pair is one launch.
//
//   experts_active    compacts the active pairs from the [B,E] histogram (all pairs without one)
//   experts_conv1     3 -> 32, 3x3, full resolution: a direct fp32 kernel (Cin = 3 is too narrow for a GEMM)
//   experts_conv      conv2 .. fc2: implicit-GEMM convolution on the tensor cores (mma.sync m16n8k8, TF32 operands,
//                     fp32 accumulation), NHWC activations, fused bias / ReLU / "ReLU then add the residual" epilogues
//   experts_fc3       512 -> 3 plus the expert's mean, into the NCHW [B,E,3,H/8,W/8] prediction; zero planes for the
//                     inactive pairs (a replayed graph reuses the output buffer)
//
// Every tile of a pair is computed the same way whatever the other pairs are: no split-K, no dependence on the pair's slot
// in the active list, so expert e's output for image b does not depend on the active set or on b's place in the batch.
#include "esac_internal.h"

namespace esacb200 {

namespace {

constexpr int kBM = 128, kBN = 128, kBK = 32, kStages = 3, kConvThreads = 256;
constexpr int kConvSmem = kStages * (kBM + kBN) * kBK * (int)sizeof(float);  // 96 KiB: two CTAs per SM

__device__ __forceinline__ void cp_async16(float* dst, const float* src, bool ok) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(ok ? 16 : 0));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }

__device__ __forceinline__ void mma_tf32(float* c, const uint32_t* a, const uint32_t* b) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// Shared-memory tiles hold rows of kBK = 32 floats; the 16-byte chunk c of row r is stored at chunk c ^ (r & 7), so that the
// fragment loads of a warp (8 rows x 4 columns) hit 32 different banks.
__device__ __forceinline__ int swz(int r, int k) { return r * kBK + (k ^ ((r & 7) << 2)); }

__global__ void __launch_bounds__(1024) experts_active_kernel(ExpertsArgs a) {
    __shared__ int warp_n[32];
    __shared__ int base;
    const int n = a.B * a.E;
    int* count = a.ws_hdr;
    int* list = a.ws_hdr + kExpertsHdrList;
    int* flags = list + n;
    if (threadIdx.x == 0) base = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int c0 = 0; c0 < n; c0 += blockDim.x) {
        const int p = c0 + threadIdx.x;
        const bool on = p < n && (!a.hist || a.hist[p] > 0.f);
        const unsigned ballot = __ballot_sync(0xffffffffu, on);
        if (lane == 0) warp_n[warp] = __popc(ballot);
        __syncthreads();
        int off = base;
        for (int w = 0; w < warp; ++w) off += warp_n[w];
        if (p < n) {
            flags[p] = on;
            if (on) list[off + __popc(ballot & ((1u << lane) - 1u))] = p;
        }
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) base = off + __popc(ballot);
        __syncthreads();
    }
    if (threadIdx.x == 0) *count = base;
}

// One thread per output pixel of one active pair, all 32 channels: 27 x 32 FMAs from the weights in shared memory.
__global__ void __launch_bounds__(256) experts_conv1_kernel(ExpertsArgs a) {
    __shared__ float w[32 * 27 + 32];
    const int slot = blockIdx.y;
    if (slot >= a.ws_hdr[0]) return;
    const int p = a.ws_hdr[kExpertsHdrList + slot];
    const int b = p / a.E, e = p % a.E;
    const float* wl = a.packed + expert_layer(0).w_off(a.E) + (size_t)e * 32 * 27;
    const float* bl = a.packed + expert_layer(0).b_off(a.E) + (size_t)e * 32;
    for (int i = threadIdx.x; i < 32 * 27; i += blockDim.x) w[i] = wl[i];
    if (threadIdx.x < 32) w[32 * 27 + threadIdx.x] = bl[threadIdx.x];
    __syncthreads();
    const int H = a.H, W = a.W;
    const int pix = blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= H * W) return;
    const int y = pix / W, x = pix % W;
    const float* img = a.image + (size_t)(a.image_batch == 1 ? 0 : b) * 3 * H * W;
    float in[27];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
            const int iy = y + ky - 1, ix = x + kx - 1;
            const bool ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
#pragma unroll
            for (int c = 0; c < 3; ++c) in[(ky * 3 + kx) * 3 + c] = ok ? __ldg(img + ((size_t)c * H + iy) * W + ix) : 0.f;
        }
    float4* out = (float4*)(a.ws_pairs + (size_t)p * a.pair_floats + (size_t)pix * 32);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int co = q * 4 + j;
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 27; ++k) s = fmaf(w[co * 27 + k], in[k], s);
            v[j] = fmaxf(s + w[32 * 27 + co], 0.f);
        }
        out[q] = make_float4(v[0], v[1], v[2], v[3]);
    }
}

// Implicit GEMM: rows are the output pixels of one active pair (M = Hout * Wout), columns its Cout channels, and the
// reduction runs over (ky, kx, ci) -- one 32-channel slice of one tap per k-tile, since Cin is a multiple of 32.  The
// input is NHWC, the weights [Cout][kh][kw][Cin] (TF32-rounded when packed), so both tiles are rows of 32 contiguous
// floats, brought in with cp.async (zero-filled outside the image) through a three-stage pipeline.  8 warps, 4 along M x
// 2 along N, each a 32 x 64 tile of m16n8k8 TF32 MMAs.
template <int KS, int STRIDE>
__global__ void __launch_bounds__(kConvThreads, 2) experts_conv_kernel(ExpertsArgs a, ExpertsConvLayer L) {
    extern __shared__ float4 smem4[];
    float* sA = (float*)smem4;
    float* sB = sA + kStages * kBM * kBK;
    const int slot = blockIdx.y;
    if (slot >= a.ws_hdr[0]) return;
    const int p = a.ws_hdr[kExpertsHdrList + slot];
    const int e = p % a.E;
    float* pair = a.ws_pairs + (size_t)p * a.pair_floats;
    const float* in = pair + L.in_off;
    float* out = pair + L.out_off;
    const float* res = L.res_off >= 0 ? pair + L.res_off : nullptr;
    const int Cin = L.cin, Cout = L.cout, Ktot = KS * KS * Cin;
    const float* w = a.packed + L.w_off + (size_t)e * Cout * Ktot;
    const float* bias = a.packed + L.b_off + (size_t)e * Cout;
    const int Mtot = L.hout * L.wout;
    const int tiles_n = (Cout + kBN - 1) / kBN;
    const int m0 = (blockIdx.x / tiles_n) * kBM, n0 = (blockIdx.x % tiles_n) * kBN;
    const int tid = threadIdx.x;

    // this thread's four A rows (output pixels) and B rows (output channels), all at chunk tid & 7
    const int chunk = tid & 7;
    int iy0[4], ix0[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + (tid >> 3) + 32 * i;
        const int oy = m / L.wout, ox = m % L.wout;
        iy0[i] = m < Mtot ? oy * STRIDE - KS / 2 : -(1 << 20);
        ix0[i] = ox * STRIDE - KS / 2;
    }
    const int KT = Ktot / kBK;
    auto load = [&](int stage, int kt) {
        const int k0 = kt * kBK;
        const int tap = k0 / Cin, ci0 = k0 - tap * Cin;
        const int ky = tap / KS, kx = tap - ky * KS;
        float* dA = sA + stage * kBM * kBK;
        float* dB = sB + stage * kBN * kBK;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int r = (tid >> 3) + 32 * i;
            const int iy = iy0[i] + ky, ix = ix0[i] + kx;
            const bool ok = iy >= 0 && iy < L.hin && ix >= 0 && ix < L.win;
            const float* src = ok ? in + ((size_t)(iy * L.win + ix) * Cin + ci0 + chunk * 4) : in;
            cp_async16(dA + r * kBK + ((chunk ^ (r & 7)) << 2), src, ok);
            const int co = n0 + r;
            const bool okb = co < Cout;
            cp_async16(dB + r * kBK + ((chunk ^ (r & 7)) << 2), okb ? w + (size_t)co * Ktot + k0 + chunk * 4 : w, okb);
        }
    };

    const int warp = tid >> 5, lane = tid & 31;
    const int wm = warp & 3, wn = warp >> 2;
    const int g = lane >> 2, t = lane & 3;
    const bool busy = n0 + wn * 64 < Cout;  // conv2's 64 channels leave the second column of warps idle
    float acc[2][8][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;

#pragma unroll
    for (int s = 0; s < kStages - 1; ++s) {
        if (s < KT) load(s, s);
        cp_async_commit();
    }
    for (int kt = 0; kt < KT; ++kt) {
        cp_async_wait<kStages - 2>();
        __syncthreads();
        if (kt + kStages - 1 < KT) load((kt + kStages - 1) % kStages, kt + kStages - 1);
        cp_async_commit();
        if (busy) {
            const float* tA = sA + (kt % kStages) * kBM * kBK;
            const float* tB = sB + (kt % kStages) * kBN * kBK;
#pragma unroll
            for (int kk = 0; kk < kBK; kk += 8) {
                uint32_t af[2][4], bf[8][2];
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int r = wm * 32 + i * 16 + g;
                    af[i][0] = to_tf32(tA[swz(r, kk + t)]);
                    af[i][1] = to_tf32(tA[swz(r + 8, kk + t)]);
                    af[i][2] = to_tf32(tA[swz(r, kk + t + 4)]);
                    af[i][3] = to_tf32(tA[swz(r + 8, kk + t + 4)]);
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int r = wn * 64 + j * 8 + g;
                    bf[j][0] = __float_as_uint(tB[swz(r, kk + t)]);
                    bf[j][1] = __float_as_uint(tB[swz(r, kk + t + 4)]);
                }
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int j = 0; j < 8; ++j) mma_tf32(acc[i][j], af[i], bf[j]);
            }
        }
    }
    cp_async_wait<0>();
    if (!busy) return;

    // epilogue: bias, then ReLU, then the residual (read before the store: it may be the output itself)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = m0 + wm * 32 + i * 16 + g + h * 8;
            if (m >= Mtot) continue;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int n = n0 + wn * 64 + j * 8 + 2 * t;
                if (n >= Cout) continue;
                const float2 bv = *(const float2*)(bias + n);
                float v0 = acc[i][j][2 * h] + bv.x, v1 = acc[i][j][2 * h + 1] + bv.y;
                if (L.relu) {
                    v0 = fmaxf(v0, 0.f);
                    v1 = fmaxf(v1, 0.f);
                }
                const size_t o = (size_t)m * Cout + n;
                if (res) {
                    const float2 rv = *(const float2*)(res + o);
                    v0 = rv.x + v0;
                    v1 = rv.y + v1;
                }
                *(float2*)(out + o) = make_float2(v0, v1);
            }
        }
}

// One warp per output pixel of every pair: lanes split the 512 channels, a fixed shuffle tree sums them.  Inactive pairs
// get zero planes.
constexpr int kFc3Warps = 8;
__global__ void __launch_bounds__(kFc3Warps * 32) experts_fc3_kernel(ExpertsArgs a, ExpertsConvLayer L) {
    __shared__ float4 w4[3 * 128];
    const int p = blockIdx.y;
    const int e = p % a.E;
    const int P8 = L.hout * L.wout;
    float* out = a.out + (size_t)p * 3 * P8;
    const int pix = blockIdx.x * kFc3Warps + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (!a.ws_hdr[kExpertsHdrList + a.B * a.E + p]) {
        if (pix < P8 && lane < 3) out[(size_t)lane * P8 + pix] = 0.f;
        return;
    }
    const float4* wl = (const float4*)(a.packed + L.w_off + (size_t)e * 3 * 512);
    for (int i = threadIdx.x; i < 3 * 128; i += blockDim.x) w4[i] = wl[i];
    __syncthreads();
    if (pix >= P8) return;
    const float4* x = (const float4*)(a.ws_pairs + (size_t)p * a.pair_floats + L.in_off + (size_t)pix * 512);
    float s[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const float4 v = x[q * 32 + lane];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float4 wv = w4[c * 128 + q * 32 + lane];
            s[c] = fmaf(wv.x, v.x, fmaf(wv.y, v.y, fmaf(wv.z, v.z, fmaf(wv.w, v.w, s[c]))));
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) s[c] += __shfl_xor_sync(0xffffffffu, s[c], d);
    if (lane < 3) {
        const float bias = a.packed[L.b_off + (size_t)e * 3 + lane];
        const float mean = a.packed[expert_mean_off(a.E) + (size_t)e * 3 + lane];
        out[(size_t)lane * P8 + pix] = (s[lane] + bias) + mean;
    }
}

// Packing: layer l of expert e from torch's [Cout][Cin][kh][kw] (staged back to back, as the state dicts hold them) to
// [Cout][kh][kw][Cin], rounded to TF32 for the layers the tensor cores run.
__global__ void experts_pack_kernel(const float* staged, float* packed, int E, ExpertLayer d, long long w_off, long long b_off,
                                    long long staged_w, long long staged_b) {
    const int kk = d.k * d.k;
    const long long per = (long long)d.cout * d.cin * kk;
    const long long n = (long long)E * per;
    const bool tf32 = d.index != 0 && d.index != kExpertLayers - 1;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int e = (int)(i / per);
        long long r = i - e * per;
        const int ci = (int)(r % d.cin);
        r /= d.cin;
        const int tap = (int)(r % kk);
        const int co = (int)(r / kk);
        const float v = staged[staged_w + e * per + ((long long)co * d.cin + ci) * kk + tap];
        packed[w_off + i] = tf32 ? __uint_as_float(to_tf32(v)) : v;
    }
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)E * d.cout;
         i += (long long)gridDim.x * blockDim.x)
        packed[b_off + i] = staged[staged_b + i];
}

}  // namespace

void launch_experts_pack(const float* staged, float* packed, int E, int l, long long staged_w, long long staged_b,
                         cudaStream_t st) {
    const ExpertLayer d = expert_layer(l);
    experts_pack_kernel<<<264, 256, 0, st>>>(staged, packed, E, d, d.w_off(E), d.b_off(E), staged_w, staged_b);
}

template <int KS, int STRIDE>
static void conv(const ExpertsArgs& a, const ExpertsConvLayer& L, cudaStream_t st) {
    // per call: the attribute belongs to the current device's context, and a process may drive several devices
    cudaFuncSetAttribute(experts_conv_kernel<KS, STRIDE>, cudaFuncAttributeMaxDynamicSharedMemorySize, kConvSmem);
    const int tiles = ((L.hout * L.wout + kBM - 1) / kBM) * ((L.cout + kBN - 1) / kBN);
    experts_conv_kernel<KS, STRIDE><<<dim3(tiles, a.B * a.E), kConvThreads, kConvSmem, st>>>(a, L);
}

void launch_experts_active(const ExpertsArgs& a, cudaStream_t st) { experts_active_kernel<<<1, 1024, 0, st>>>(a); }

void launch_experts_conv(const ExpertsArgs& a, const ExpertsConvLayer& L, int k, int stride, cudaStream_t st) {
    if (k == 1) conv<1, 1>(a, L, st);
    else if (stride == 2) conv<3, 2>(a, L, st);
    else conv<3, 1>(a, L, st);
}

void launch_experts_forward(const ExpertsArgs& a, cudaStream_t st) {
    const ExpertsShape s = experts_shape(a.H, a.W);
    launch_experts_active(a, st);
    experts_conv1_kernel<<<dim3((a.H * a.W + 255) / 256, a.B * a.E), 256, 0, st>>>(a);
    // the layer sequence of Expert.forward: (layer, input, output, residual or -1, ReLU)
    struct Step { int l; long long in, out, res; bool relu; };
    const Step steps[] = {
        {1, s.a0, s.a1, -1, true},  {2, s.a1, s.a2, -1, true},  {3, s.a2, s.r, -1, true},          // conv2 .. conv4
        {4, s.r, s.x, -1, true},    {5, s.x, s.y, -1, true},    {6, s.y, s.r, s.r, true},          // res1: res += x
        {7, s.r, s.x, -1, true},    {8, s.x, s.y, -1, true},    {10, s.r, s.s, -1, false},         // res2, skip
        {9, s.y, s.s, s.s, true},                                                                  // res = skip(res) + x
        {11, s.s, s.x, -1, true},   {12, s.x, s.y, -1, true},   {13, s.y, s.s, s.s, true},         // res3: res += x
        {14, s.s, s.x, -1, true},   {15, s.x, s.y, -1, true}};                                     // fc1, fc2
    for (const Step& q : steps) {
        const ExpertLayer d = expert_layer(q.l);
        ExpertsConvLayer L;
        L.cin = d.cin;
        L.cout = d.cout;
        const int lvl_in = q.l <= 3 ? q.l - 1 : 3, lvl_out = q.l <= 3 ? q.l : 3;
        L.hin = s.h[lvl_in];
        L.win = s.w[lvl_in];
        L.hout = s.h[lvl_out];
        L.wout = s.w[lvl_out];
        L.in_off = q.in;
        L.out_off = q.out;
        L.res_off = q.res;
        L.relu = q.relu;
        L.w_off = d.w_off(a.E);
        L.b_off = d.b_off(a.E);
        launch_experts_conv(a, L, d.k, d.stride, st);
    }
    const ExpertLayer d = expert_layer(kExpertLayers - 1);
    ExpertsConvLayer L{};
    L.cin = d.cin;
    L.cout = d.cout;
    L.hout = s.h[3];
    L.wout = s.w[3];
    L.in_off = s.y;
    L.w_off = d.w_off(a.E);
    L.b_off = d.b_off(a.E);
    experts_fc3_kernel<<<dim3((L.hout * L.wout + kFc3Warps - 1) / kFc3Warps, a.B * a.E), kFc3Warps * 32, 0, st>>>(a, L);
}

}  // namespace esacb200
