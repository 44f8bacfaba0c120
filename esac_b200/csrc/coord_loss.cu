// Robust scene-coordinate loss of the expert initialisation stage, loss and gradient (init_expert.py:106-135).
//
// init_expert.py crops prediction and ground truth to a common size (:114, util.assert_size, util.py:18-36), drops the cells
// whose ground truth is all zero (:119-121), takes the Euclidean distance per cell, applies the same L1 / square-root robust
// loss as the refinement stage and divides by the number of valid cells (:123-130); autograd then walks back through it.  Four
// boolean-mask indexings each synchronise the host.  Here it is two launches and no host round trip:
//
//   count pass   valid cells per image (12 B read per window cell: the ground truth)
//   loss pass    loss and d loss / d prediction (24 B read + 12 B written per cell), scaled by 1 / count
//
// i.e. 48 B per cell with the gradient; a loss-only call skips the count pass and counts in the loss pass (24 B per cell).
// Per cell, with d = pred - gt in fp32 (the subtraction torch does) and everything after it in fp64:
//   valid  = gt.x != 0 || gt.y != 0 || gt.z != 0        (gt.abs().sum(0) != 0; NaN counts as valid, no flush to zero)
//   n      = ||d||
//   loss   = n <= cut ? n : sqrt(cut * n)
//   grad   = rho'(n) * d / n / count,  rho' = 1 or 0.5 * sqrt(cut / n);  0 at n = 0 (torch's norm backward)
// A NaN cell counts but falls in neither masked sum (loss 0, gradient NaN); an invalid cell has loss and gradient 0, as do
// prediction cells outside the common window.  The per-image loss is summed in fp64 in a fixed order (block partials, the
// image's last block adds them up), so the result does not depend on scheduling.
#include <type_traits>

#include "esac_internal.h"

namespace esacb200 {

namespace {

constexpr int kThreads = 256;
constexpr int kCellsPerThread = 4;

__device__ __forceinline__ bool gt_valid(float x, float y, float z) { return x != 0.f || y != 0.f || z != 0.f; }

// Window cell of prediction cell p (scalar path); -1 outside the window, else the ground-truth index.
__device__ __forceinline__ int gt_index(int y, int x, const CoordImage& g) { return (y < g.H && x < g.W) ? y * g.Wg + x : -1; }

struct CellOut {
    double loss;
    float gx, gy, gz;
};

// One valid cell.  cnt = valid cells of the image (the gradient's normaliser; unused without GRAD).
template <bool GRAD>
__device__ __forceinline__ CellOut coord_cell(float px, float py, float pz, float qx, float qy, float qz, float cut, double cnt) {
    const float dx = px - qx, dy = py - qy, dz = pz - qz;
    const double s2 = fma((double)dx, (double)dx, fma((double)dy, (double)dy, (double)dz * (double)dz));   // exact products
    const double n = sqrt(s2);
    CellOut o;
    double w = 0.;                                    // rho'(n) / n / count
    if (n <= (double)cut) {                           // n == cut is in the L1 branch (loss[loss <= cut])
        o.loss = n;
        if (GRAD) w = 1.0 / (n * cnt);
    } else {
        o.loss = sqrt((double)cut * n);
        if (GRAD) w = 0.5 * o.loss / (s2 * cnt);      // 0.5 sqrt(cut / n) / n = 0.5 sqrt(cut n) / n^2
    }
    if (!(n > 0.)) w = 0.;                            // n = 0: zero gradient
    o.gx = (float)(w * dx);
    o.gy = (float)(w * dy);
    o.gz = (float)(w * dz);
    if (!(n == n)) {                                  // NaN: in neither masked sum, gradient NaN
        o.loss = 0.;
        o.gx = o.gy = o.gz = (float)n;
    }
    return o;
}

// grid = (max blocks, images of this load path): row blockIdx.y is image recs[blockIdx.y], its blocks are blockIdx.x <
// blocks.  counts[b] += valid cells of image b (zeroed before the launch).
template <bool VEC>
__global__ void __launch_bounds__(kThreads) coord_count_kernel(const CoordImage* __restrict__ recs, unsigned* __restrict__ counts) {
    const CoordImage g = recs[blockIdx.y];
    if ((int)blockIdx.x >= g.blocks) return;
    const int b = g.b;
    const float* qx = g.gt;
    const float* qy = qx + g.Ng;
    const float* qz = qy + g.Ng;
    unsigned cnt = 0;
    const int per_block = kThreads * kCellsPerThread;
    for (int base = blockIdx.x * per_block; base < g.Np; base += g.blocks * per_block) {
        const int p0 = base + threadIdx.x * kCellsPerThread;
        if (VEC) {
            if (p0 >= g.N) continue;   // the window is the first N cells of both planes (equal pitch, N % 4 == 0)
            const float4 a = __ldcs(reinterpret_cast<const float4*>(qx + p0));
            const float4 c = __ldcs(reinterpret_cast<const float4*>(qy + p0));
            const float4 d = __ldcs(reinterpret_cast<const float4*>(qz + p0));
            cnt += gt_valid(a.x, c.x, d.x) + gt_valid(a.y, c.y, d.y) + gt_valid(a.z, c.z, d.z) + gt_valid(a.w, c.w, d.w);
        } else {
            if (p0 >= g.Np) continue;
            int y = p0 / g.Wp, x = p0 - y * g.Wp;
            const int n = min(kCellsPerThread, g.Np - p0);
            for (int i = 0; i < n; ++i) {
                const int q = gt_index(y, x, g);
                if (q >= 0) cnt += gt_valid(qx[q], qy[q], qz[q]);
                if (++x == g.Wp) { x = 0; ++y; }
            }
        }
    }
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&counts[b], cnt);
}

// grid as for the count pass, over the prediction's cells.  GRAD: grads overwritten, counts[b] from the count pass.
// losses[b] = loss of image b, out_counts[b] = its valid cells; partial: 2 doubles per block, tickets: zeroed counters
// (left zeroed).  T: the prediction's and gradient's element type, widened on load; SCALE: every gradient (zeros included)
// times *grad_scale (loss_scale) after coord_cell's rounding to float, then rounded to T.
template <class T, bool VEC, bool GRAD, bool SCALE>
__global__ void __launch_bounds__(kThreads) coord_loss_kernel(const CoordImage* __restrict__ recs, float cut,
                                                               const float* __restrict__ grad_scale,
                                                               const unsigned* __restrict__ counts, double* __restrict__ partial,
                                                               unsigned* __restrict__ tickets, double* __restrict__ losses,
                                                               long long* __restrict__ out_counts) {
    const CoordImage g = recs[blockIdx.y];
    if ((int)blockIdx.x >= g.blocks) return;
    const int b = g.b;
    const T* px = static_cast<const T*>(g.pred);
    const T* py = px + g.Np;
    const T* pz = py + g.Np;
    const float* qx = g.gt;
    const float* qy = qx + g.Ng;
    const float* qz = qy + g.Ng;
    T* gx = GRAD ? static_cast<T*>(g.grads) : nullptr;
    const double cnt = GRAD ? (double)counts[b] : 0.;
    const float s = SCALE ? *grad_scale : 1.f;
    double acc = 0.;
    unsigned nvalid = 0;
    const int per_block = kThreads * kCellsPerThread;
    for (int base = blockIdx.x * per_block; base < g.Np; base += g.blocks * per_block) {
        const int p0 = base + threadIdx.x * kCellsPerThread;
        if (p0 >= g.Np) continue;
        if (VEC) {
            float o[3][4] = {};
            if (p0 < g.N) {   // all four cells in the window (N % 4 == 0), else all four outside: zero gradient
                const float4 a = loss_ld4(px + p0);
                const float4 c = loss_ld4(py + p0);
                const float4 d = loss_ld4(pz + p0);
                const float4 e = __ldcs(reinterpret_cast<const float4*>(qx + p0));
                const float4 f = __ldcs(reinterpret_cast<const float4*>(qy + p0));
                const float4 h = __ldcs(reinterpret_cast<const float4*>(qz + p0));
                const float P[3][4] = {{a.x, a.y, a.z, a.w}, {c.x, c.y, c.z, c.w}, {d.x, d.y, d.z, d.w}};
                const float Q[3][4] = {{e.x, e.y, e.z, e.w}, {f.x, f.y, f.z, f.w}, {h.x, h.y, h.z, h.w}};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    if (!gt_valid(Q[0][i], Q[1][i], Q[2][i])) continue;
                    const CellOut r = coord_cell<GRAD>(P[0][i], P[1][i], P[2][i], Q[0][i], Q[1][i], Q[2][i], cut, cnt);
                    acc += r.loss;
                    ++nvalid;
                    o[0][i] = r.gx; o[1][i] = r.gy; o[2][i] = r.gz;
                }
            }
            if (GRAD) {
                auto sc = [s](float v) { return loss_scale<SCALE>(v, s); };
                loss_st4(gx + p0, sc(o[0][0]), sc(o[0][1]), sc(o[0][2]), sc(o[0][3]));
                loss_st4(gx + g.Np + p0, sc(o[1][0]), sc(o[1][1]), sc(o[1][2]), sc(o[1][3]));
                loss_st4(gx + 2 * (size_t)g.Np + p0, sc(o[2][0]), sc(o[2][1]), sc(o[2][2]), sc(o[2][3]));
            }
        } else {
            int y = p0 / g.Wp, x = p0 - y * g.Wp;
            const int n = min(kCellsPerThread, g.Np - p0);
            for (int i = 0; i < n; ++i) {
                const int q = gt_index(y, x, g);
                float rx = 0.f, ry = 0.f, rz = 0.f;
                if (q >= 0) {
                    const float ex = qx[q], ey = qy[q], ez = qz[q];
                    if (gt_valid(ex, ey, ez)) {
                        const CellOut r = coord_cell<GRAD>(loss_in(px[p0 + i]), loss_in(py[p0 + i]), loss_in(pz[p0 + i]), ex, ey,
                                                           ez, cut, cnt);
                        acc += r.loss;
                        ++nvalid;
                        rx = r.gx; ry = r.gy; rz = r.gz;
                    }
                }
                if (GRAD) {
                    gx[p0 + i] = loss_out<T>(loss_scale<SCALE>(rx, s));
                    gx[g.Np + p0 + i] = loss_out<T>(loss_scale<SCALE>(ry, s));
                    gx[2 * (size_t)g.Np + p0 + i] = loss_out<T>(loss_scale<SCALE>(rz, s));
                }
                if (++x == g.Wp) { x = 0; ++y; }
            }
        }
    }
    double total[2] = {acc, (double)nvalid};
    if (block_image_sum<kThreads>(total, partial, tickets, b, g.blocks, (size_t)g.part0)) {
        losses[b] = total[0] / total[1];   // no valid cell: 0 / 0 = NaN, as in torch
        out_counts[b] = (long long)total[1];
    }
}

}  // namespace

bool coord_image(CoordImage& r, int Hp, int Wp, int Hg, int Wg, int esize) {
    r.Np = Hp * Wp; r.Ng = Hg * Wg; r.Wp = Wp; r.Wg = Wg;
    r.H = Hp < Hg ? Hp : Hg;
    r.W = Wp < Wg ? Wp : Wg;
    r.N = r.H * r.W;
    r.blocks = reproj_blocks_per_image(r.Np);
    r.pad = 0;
    // vector path: equal row pitch (the window is then the first N cells of every plane), every plane aligned for a 4-element
    // access (16 bytes for float32, 8 for the 16-bit types; the ground truth is float32)
    const uintptr_t align = 4 * (uintptr_t)esize;
    return Wp == Wg && r.N % 4 == 0 && r.Np % 4 == 0 && r.Ng % 4 == 0 && (uintptr_t)r.pred % align == 0 &&
           (uintptr_t)r.gt % 16 == 0 && (!r.grads || (uintptr_t)r.grads % align == 0);
}

// The loss pass of element type T: loss only, or with gradients (scaled when grad_scale is not null).
template <class T>
static void launch_coord_pass(bool vec, bool grad, dim3 grid, const CoordImage* recs, float cut, const float* grad_scale,
                              unsigned* counts, double* partial, unsigned* tickets, double* losses, long long* out_counts,
                              cudaStream_t stream) {
#define ESAC_COORD_LOSS(V, G, S) \
    coord_loss_kernel<T, V, G, S><<<grid, kThreads, 0, stream>>>(recs, cut, grad_scale, counts, partial, tickets, losses, out_counts)
    if (!grad) {
        if (vec) ESAC_COORD_LOSS(true, false, false);
        else ESAC_COORD_LOSS(false, false, false);
    } else if (!grad_scale) {
        if (vec) ESAC_COORD_LOSS(true, true, false);
        else ESAC_COORD_LOSS(false, true, false);
    } else if constexpr (!std::is_same_v<T, float>) {   // float32 is never scaled in the kernel
        if (vec) ESAC_COORD_LOSS(true, true, true);
        else ESAC_COORD_LOSS(false, true, true);
    }
#undef ESAC_COORD_LOSS
}

void launch_coord_loss(bool vec, int pass, bool grad, int dtype, const CoordImage* recs, int n, int max_blocks, float cut,
                       const float* grad_scale, unsigned* counts, double* partial, unsigned* tickets, double* losses,
                       long long* out_counts, cudaStream_t stream) {
    const dim3 grid(max_blocks, n);
    if (pass == 1) {   // reads the float32 ground truth only: one kernel for every dtype
        if (vec) coord_count_kernel<true><<<grid, kThreads, 0, stream>>>(recs, counts);
        else coord_count_kernel<false><<<grid, kThreads, 0, stream>>>(recs, counts);
    } else if (dtype == kLossF32) {
        launch_coord_pass<float>(vec, grad, grid, recs, cut, nullptr, counts, partial, tickets, losses, out_counts, stream);
    } else if (dtype == kLossF16) {
        launch_coord_pass<__half>(vec, grad, grid, recs, cut, grad_scale, counts, partial, tickets, losses, out_counts, stream);
    } else {
        launch_coord_pass<__nv_bfloat16>(vec, grad, grid, recs, cut, grad_scale, counts, partial, tickets, losses, out_counts,
                                         stream);
    }
}

}  // namespace esacb200
