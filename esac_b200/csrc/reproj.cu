// Reprojection loss of the expert refinement stage, forward and backward in one pass (SURVEY 8f rank 4).
//
// ref_expert.py:103-146 projects every predicted scene coordinate with the ground-truth pose, takes the pixel distance to
// the cell centre, clamps it to [0, 100] px, applies an L1 / square-root robust loss and lets autograd walk back through
// six elementwise tensors.  It is the scoring kernel's projection with a different epilogue, and purely HBM-bound:
// 12 B read + 12 B written per cell.  One launch covers a batch of maps; each thread handles 4 consecutive cells with
// 128-bit loads/stores; the per-image loss is summed in fp64 in a fixed order (block partials, last block adds them up),
// so the result does not depend on scheduling.
//
//   eye = gtPose^-1[0:3,:] * [X;1]                                   ref_expert.py:127-132
//   px  = K * eye;  px[2].clamp_(min=0.1);  px = px[0:2] / px[2]     :135-137   (numerator keeps the unclamped depth)
//   err = ||px - (cell centre - pad)||, clamp(0, 100)                :140-142
//   loss = (sum_{err<=cut} err + sum_{err>cut} sqrt(cut*err)) / N    :144-148
#include "esac_internal.h"

namespace esacb200 {

namespace {

constexpr int kThreads = 256;
constexpr int kCellsPerThread = 4;

struct CellOut { float gx, gy, gz, loss; };
struct PairOut { float2 gx, gy, gz, loss; };

constexpr float kTiny = 1e-30f;

__device__ __forceinline__ float rcp_fast(float x) {   // MUFU.RCP, <= 1 ulp
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float rsqrt_fast(float x) { // MUFU.RSQ, <= 2 ulp
    float r;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// One cell, fp32 like the torch ops it replaces, arranged so that the kernel stays under the HBM roofline's instruction
// budget (~70 issue slots per cell, 3 MUFU) and loses no accuracy against the original op sequence:
//  * the pixel offset is formed as (nu - tx*zz) / zz with one FMA, so the division only ever scales a small number (the
//    original rounds u = nu/zz at |u| ~ 1e3 px before subtracting);
//  * where the depth clamp is open, d/dzc collapses to -(gxc*xc + gyc*yc)/zz, free of the cx/zz - u/zz cancellation.
// m = rows of the 3x4 world->camera matrix.
__device__ __forceinline__ CellOut reproj_cell(float X, float Y, float Z, const float* __restrict__ m, float f, float cx,
                                               float cy, float tx, float ty, float cut, float max_err, float min_depth,
                                               float inv_n) {
    const float xc = fmaf(m[0], X, fmaf(m[1], Y, fmaf(m[2], Z, m[3])));
    const float yc = fmaf(m[4], X, fmaf(m[5], Y, fmaf(m[6], Z, m[7])));
    const float zc = fmaf(m[8], X, fmaf(m[9], Y, fmaf(m[10], Z, m[11])));
    const float nu = fmaf(f, xc, cx * zc);         // numerator keeps the unclamped depth (ref_expert.py:135-137)
    const float nv = fmaf(f, yc, cy * zc);
    const bool open = zc >= min_depth;             // clamp_ passes the gradient where it did not clamp
    const float zz = open ? zc : min_depth;
    const float iz = rcp_fast(zz);
    const float du = fmaf(-tx, zz, nu) * iz;
    const float dv = fmaf(-ty, zz, nv) * iz;
    const float s2 = fmaf(du, du, dv * dv);
    const float r = rsqrt_fast(fmaxf(s2, kTiny));   // 1/err; at the origin err = s2*r = 0 and the gradient gr*du = 0 (norm backward)
    const float err = s2 * r;
    const float e = fminf(err, max_err);
    const float t = cut * e;
    const float rt = rsqrt_fast(fmaxf(t, kTiny));
    const bool l1 = e <= cut;
    CellOut o;
    o.loss = l1 ? e : t * rt;                       // sqrt(cut * e)
    // d loss / d err; the clamp's gradient is 1 on [0, max_err] (bounds included) and 0 outside
    float g = l1 ? 1.f : 0.5f * cut * rt;
    g = err <= max_err ? g * inv_n : 0.f;
    const float gr = g * r;
    const float fiz = f * iz;
    const float gxc = gr * du * fiz;
    const float gyc = gr * dv * fiz;
    const float gz_open = -(gxc * xc + gyc * yc) * iz;
    const float gz_shut = gr * (du * cx + dv * cy) * iz;
    const float gzc = open ? gz_open : gz_shut;
    o.gx = fmaf(m[0], gxc, fmaf(m[4], gyc, m[8] * gzc));
    o.gy = fmaf(m[1], gxc, fmaf(m[5], gyc, m[9] * gzc));
    o.gz = fmaf(m[2], gxc, fmaf(m[6], gyc, m[10] * gzc));
    if (!(s2 == s2)) {                              // NaN input: in neither branch of the masked sums; gradient NaN as in torch
        o.loss = 0.f;
        o.gx = o.gy = o.gz = s2;
    }
    return o;
}

// Two cells at once as float2 pairs (two IEEE fp32 results per operation -- bitwise what
// reproj_cell computes for each): two independent dependency chains per thread for the scheduler to interleave.
struct PairConst {
    float2 m[12];            // world->camera entries, broadcast
    float2 f, cx, cy, cut, half_cut, inv_n;
    float max_err, min_depth, cut_s;
};

__device__ __forceinline__ float2 bc(float v) { return make_float2(v, v); }
__device__ __forceinline__ float2 neg2(float2 v) { return make_float2(-v.x, -v.y); }

__device__ __forceinline__ PairOut reproj_pair(float2 X, float2 Y, float2 Z, const PairConst& k, float2 tx, float2 ty) {
    const float2 xc = ffma2(k.m[0], X, ffma2(k.m[1], Y, ffma2(k.m[2], Z, k.m[3])));
    const float2 yc = ffma2(k.m[4], X, ffma2(k.m[5], Y, ffma2(k.m[6], Z, k.m[7])));
    const float2 zc = ffma2(k.m[8], X, ffma2(k.m[9], Y, ffma2(k.m[10], Z, k.m[11])));
    const float2 nu = ffma2(k.f, xc, fmul2(k.cx, zc));
    const float2 nv = ffma2(k.f, yc, fmul2(k.cy, zc));
    const bool open0 = zc.x >= k.min_depth, open1 = zc.y >= k.min_depth;
    const float2 zz = make_float2(open0 ? zc.x : k.min_depth, open1 ? zc.y : k.min_depth);
    const float2 iz = make_float2(rcp_fast(zz.x), rcp_fast(zz.y));
    const float2 du = fmul2(ffma2(neg2(tx), zz, nu), iz);
    const float2 dv = fmul2(ffma2(neg2(ty), zz, nv), iz);
    const float2 s2 = ffma2(du, du, fmul2(dv, dv));
    const float2 r = make_float2(rsqrt_fast(fmaxf(s2.x, kTiny)), rsqrt_fast(fmaxf(s2.y, kTiny)));
    const float2 err = fmul2(s2, r);
    const float2 e = make_float2(fminf(err.x, k.max_err), fminf(err.y, k.max_err));
    const float2 t = fmul2(k.cut, e);
    const float2 rt = make_float2(rsqrt_fast(fmaxf(t.x, kTiny)), rsqrt_fast(fmaxf(t.y, kTiny)));
    const float2 sq = fmul2(t, rt);                  // sqrt(cut * e)
    const float2 gs = fmul2(k.half_cut, rt);         // its derivative
    const bool l0 = e.x <= k.cut_s, l1 = e.y <= k.cut_s;
    PairOut o;
    o.loss = make_float2(l0 ? e.x : sq.x, l1 ? e.y : sq.y);
    float2 g = make_float2(l0 ? 1.f : gs.x, l1 ? 1.f : gs.y);
    g = fmul2(g, k.inv_n);
    g = make_float2(err.x <= k.max_err ? g.x : 0.f, err.y <= k.max_err ? g.y : 0.f);
    const float2 gr = fmul2(g, r);
    const float2 fiz = fmul2(k.f, iz);
    const float2 gxc = fmul2(fmul2(gr, du), fiz);
    const float2 gyc = fmul2(fmul2(gr, dv), fiz);
    const float2 go = fmul2(neg2(ffma2(gxc, xc, fmul2(gyc, yc))), iz);
    const float2 gsh = fmul2(fmul2(gr, ffma2(du, k.cx, fmul2(dv, k.cy))), iz);
    const float2 gzc = make_float2(open0 ? go.x : gsh.x, open1 ? go.y : gsh.y);
    o.gx = ffma2(k.m[0], gxc, ffma2(k.m[4], gyc, fmul2(k.m[8], gzc)));
    o.gy = ffma2(k.m[1], gxc, ffma2(k.m[5], gyc, fmul2(k.m[9], gzc)));
    o.gz = ffma2(k.m[2], gxc, ffma2(k.m[6], gyc, fmul2(k.m[10], gzc)));
    if (!(s2.x == s2.x)) { o.loss.x = 0.f; o.gx.x = o.gy.x = o.gz.x = s2.x; }   // NaN input (see reproj_cell)
    if (!(s2.y == s2.y)) { o.loss.y = 0.f; o.gx.y = o.gy.y = o.gz.y = s2.y; }
    return o;
}

// grid = (max blocks, images of this load path).  Row blockIdx.y is image recs[blockIdx.y]; its blocks are blockIdx.x <
// rec.blocks, the others leave at once.  img[b] = kReprojImgFloats floats: 12 matrix entries, padX, padY, f, cx, cy, 3 unused.
// T: the maps' element type (float, __half, __nv_bfloat16), widened on load; SCALE: every gradient times *grad_scale
// (loss_scale) before it is rounded to T.
template <class T, bool VEC, bool SCALE>
__global__ void __launch_bounds__(kThreads, 5) reproj_kernel(const ReprojImage* __restrict__ recs, const float* __restrict__ img,
                                                          float sub, float cut, float max_err, float min_depth,
                                                          const float* __restrict__ grad_scale, double* __restrict__ partial,
                                                          unsigned* __restrict__ tickets, double* __restrict__ losses) {
    __shared__ float m[kReprojImgFloats];
    // The image's geometry sits in shared memory and is re-read where it is used (volatile).  Unlike kernel parameters,
    // loaded values cannot be rematerialised: held in registers across the loop they would push the scalar path over the
    // 48 registers of __launch_bounds__(256, 5).
    __shared__ ReprojImage rec;
    const volatile ReprojImage& vrec = rec;
    if ((int)blockIdx.x >= recs[blockIdx.y].blocks) return;
    if (threadIdx.x == 0) rec = recs[blockIdx.y];
    __syncthreads();
    if (threadIdx.x < kReprojImgFloats) m[threadIdx.x] = img[rec.b * kReprojImgFloats + threadIdx.x];
    __syncthreads();
    const float inv_n = 1.f / (float)rec.N;
    const float half = sub * 0.5f;
    const float padX = m[12], padY = m[13];
    PairConst kc;
    if (VEC) {
#pragma unroll
        for (int i = 0; i < 12; ++i) kc.m[i] = bc(m[i]);
        kc.f = bc(m[14]); kc.cx = bc(m[15]); kc.cy = bc(m[16]);   // this image's camera
        kc.cut = bc(cut); kc.half_cut = bc(0.5f * cut); kc.inv_n = bc(inv_n);
        kc.max_err = max_err; kc.min_depth = min_depth; kc.cut_s = cut;
    }
    double acc = 0.;
    const int per_block = kThreads * kCellsPerThread;
    for (int base = blockIdx.x * per_block; base < vrec.N; base += vrec.blocks * per_block) {
        const int N = vrec.N, W = vrec.W;
        const int p0 = base + threadIdx.x * kCellsPerThread;
        if (p0 >= N) continue;
        float X[4], Y[4], Z[4];
        int n = min(kCellsPerThread, N - p0);
        if (VEC) {
            const T* px = static_cast<const T*>(vrec.coords);
            const T* py = px + N;
            const T* pz = py + N;
            const float4 a = loss_ld4(px + p0);
            const float4 c = loss_ld4(py + p0);
            const float4 d = loss_ld4(pz + p0);
            X[0] = a.x; X[1] = a.y; X[2] = a.z; X[3] = a.w;
            Y[0] = c.x; Y[1] = c.y; Y[2] = c.z; Y[3] = c.w;
            Z[0] = d.x; Z[1] = d.y; Z[2] = d.z; Z[3] = d.w;
        }
        int y = p0 / W, x = p0 - y * W;
        float ox[4], oy[4], oz[4];
        float four = 0.f;   // 4 losses <= 100 each: exact enough in fp32; the long sums run in fp64
        if (VEC) {
            // target pixels of the 4 cells; a row change inside the group moves the later cells to the next row (W >= 4)
            const float xf = (float)x, yf = (float)y;
            float txs[4], tys[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const bool wrap = x + i >= W;
                const float xi = xf + (float)i - (wrap ? (float)W : 0.f);
                const float yi = yf + (wrap ? 1.f : 0.f);
                txs[i] = fmaf(xi, sub, half) - padX;
                tys[i] = fmaf(yi, sub, half) - padY;
            }
#pragma unroll
            for (int i = 0; i < 4; i += 2) {
                const PairOut o = reproj_pair(make_float2(X[i], X[i + 1]), make_float2(Y[i], Y[i + 1]), make_float2(Z[i], Z[i + 1]),
                                              kc, make_float2(txs[i], txs[i + 1]), make_float2(tys[i], tys[i + 1]));
                four += o.loss.x + o.loss.y;
                ox[i] = o.gx.x; ox[i + 1] = o.gx.y;
                oy[i] = o.gy.x; oy[i + 1] = o.gy.y;
                oz[i] = o.gz.x; oz[i + 1] = o.gz.y;
            }
        } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                // each cell is loaded where it is used: four cells of inputs held at once would not fit the register budget
                const T* c = static_cast<const T*>(vrec.coords);
                const bool ok = i < n;
                X[i] = ok ? loss_in(c[p0 + i]) : 0.f;
                Y[i] = ok ? loss_in(c[vrec.N + p0 + i]) : 0.f;
                Z[i] = ok ? loss_in(c[2 * (size_t)vrec.N + p0 + i]) : 1.f;
                const float tx = fmaf((float)x, sub, half) - padX;
                const float ty = fmaf((float)y, sub, half) - padY;
                const CellOut o = reproj_cell(X[i], Y[i], Z[i], m, m[14], m[15], m[16], tx, ty, cut, max_err, min_depth, inv_n);
                if (i < n) {
                    four += o.loss;
                    T* g = static_cast<T*>(vrec.grads);
                    if (g) {   // stored as computed: no gradient array stays live across the four cells
                        const int Nv = vrec.N;
                        const float s = SCALE ? *grad_scale : 1.f;
                        g[p0 + i] = loss_out<T>(loss_scale<SCALE>(o.gx, s));
                        g[Nv + p0 + i] = loss_out<T>(loss_scale<SCALE>(o.gy, s));
                        g[2 * (size_t)Nv + p0 + i] = loss_out<T>(loss_scale<SCALE>(o.gz, s));
                    }
                }
                if (++x == vrec.W) { x = 0; ++y; }
            }
        }
        acc += (double)four;
        T* gx = static_cast<T*>(vrec.grads);
        if (VEC && gx) {
            const float s = SCALE ? *grad_scale : 1.f;
            auto sc = [s](float g) { return loss_scale<SCALE>(g, s); };
            loss_st4(gx + p0, sc(ox[0]), sc(ox[1]), sc(ox[2]), sc(ox[3]));
            loss_st4(gx + N + p0, sc(oy[0]), sc(oy[1]), sc(oy[2]), sc(oy[3]));
            loss_st4(gx + 2 * (size_t)N + p0, sc(oz[0]), sc(oz[1]), sc(oz[2]), sc(oz[3]));
        }
    }
    // block sum in a fixed order, then the last block of the image adds the partials, again in a fixed order
    double total[1] = {acc};
    if (block_image_sum<kThreads>(total, partial, tickets, vrec.b, vrec.blocks, (size_t)vrec.part0))
        losses[vrec.b] = total[0] / (double)vrec.N;
}

}  // namespace

int reproj_blocks_per_image(int N) {
    // Many short CTAs (each a few KB of traffic) rather than one resident wave: the hardware scheduler then keeps every SM
    // streaming to the end, where a persistent grid of sm_count * k CTAs would finish with a ragged tail.  Two passes per CTA
    // on large maps amortise the per-CTA prologue / reduction; the count is a pure function of N (the fixed summation
    // order depends on it).
    const int per_block = kThreads * kCellsPerThread;
    const int need = (N + per_block - 1) / per_block;
    return need < 64 ? need : (need < 256 ? (need + 1) / 2 : (need + 3) / 4);
}

int reproj_max_blocks(int N) {
    // the count rises with N within each of its three ranges and drops where a range starts: the largest is at N or at the
    // end of a range below it
    const int per_block = kThreads * kCellsPerThread;
    int most = reproj_blocks_per_image(N);
    for (int need : {63, 255}) {
        if ((long long)need * per_block >= N) break;
        const int b = reproj_blocks_per_image(need * per_block);
        if (b > most) most = b;
    }
    return most;
}

bool reproj_vec_ok(const void* coords, const void* grads, int N, int W, int esize) {
    const uintptr_t align = 4 * (uintptr_t)esize;
    return (N % 4 == 0) && W >= 4 && ((uintptr_t)coords % align == 0) && (!grads || (uintptr_t)grads % align == 0);
}

template <class T, bool SCALE>
static void launch_reproj_typed(bool vec, dim3 grid, const ReprojImage* recs, const float* img, float sub, float cut,
                                float max_err, float min_depth, const float* grad_scale, double* partial, unsigned* tickets,
                                double* losses, cudaStream_t stream) {
    if (vec)
        reproj_kernel<T, true, SCALE><<<grid, kThreads, 0, stream>>>(recs, img, sub, cut, max_err, min_depth, grad_scale, partial,
                                                                     tickets, losses);
    else
        reproj_kernel<T, false, SCALE><<<grid, kThreads, 0, stream>>>(recs, img, sub, cut, max_err, min_depth, grad_scale, partial,
                                                                      tickets, losses);
}

void launch_reproj(bool vec, int dtype, const ReprojImage* recs, int n, int max_blocks, const float* img, float sub, float cut,
                   float max_err, float min_depth, const float* grad_scale, double* partial, unsigned* tickets, double* losses,
                   cudaStream_t stream) {
    const dim3 grid(max_blocks, n);
    const bool scale = grad_scale != nullptr;
    if (dtype == kLossF32)   // float32 is never scaled in the kernel
        launch_reproj_typed<float, false>(vec, grid, recs, img, sub, cut, max_err, min_depth, nullptr, partial, tickets, losses, stream);
    else if (dtype == kLossF16 && scale)
        launch_reproj_typed<__half, true>(vec, grid, recs, img, sub, cut, max_err, min_depth, grad_scale, partial, tickets, losses, stream);
    else if (dtype == kLossF16)
        launch_reproj_typed<__half, false>(vec, grid, recs, img, sub, cut, max_err, min_depth, nullptr, partial, tickets, losses, stream);
    else if (scale)
        launch_reproj_typed<__nv_bfloat16, true>(vec, grid, recs, img, sub, cut, max_err, min_depth, grad_scale, partial, tickets,
                                                 losses, stream);
    else
        launch_reproj_typed<__nv_bfloat16, false>(vec, grid, recs, img, sub, cut, max_err, min_depth, nullptr, partial, tickets,
                                                  losses, stream);
}

}  // namespace esacb200
