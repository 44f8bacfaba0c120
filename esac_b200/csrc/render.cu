// Ground-truth scene-coordinate maps rendered from an SfM reconstruction on the device (setup_aachen.py:184-202,
// setup_dubrovnik.py:171-190): every observation of a camera projects its point into the camera's out map, and a cell
// keeps the point that the reference's serial z-test leaves there.  That test, `zbuf == 0 or zbuf > z`, run over a cell's
// observations in file order, leaves:
//   - the nearest point (lowest depth, negative depths first; the earliest on equal depths) among the observations after
//     the last *written* point of depth +-0, which reopens the cell;
//   - else that depth-0 point;
//   - else nothing (the cell stays all-zero).
// A depth-0 point is written unless a negative depth came before it in the cell: a negative z-buffer value is neither 0 nor
// greater than 0, and no later write can lift it back to 0.  So the last written depth-0 point is the last one before the
// cell's first negative depth.  The four passes below find exactly that with commutative atomics (min / max on integers), so
// the result does not depend on the order in which they land.  oracle/render_oracle.py restates the passes in numpy.
#include <limits.h>

#include "esac_internal.h"

namespace esacb200 {

namespace {

constexpr int kThreads = 256;

// The order-preserving integer image of a non-NaN float (unsigned order of keys = numeric order, -0 < +0).
__device__ __forceinline__ unsigned depth_key(float f) {
    const unsigned u = __float_as_uint(f);
    return u ^ ((unsigned)((int)u >> 31) | 0x80000000u);
}

// The camera that owns observation v: the last c with offsets[c] <= v (cameras without observations are skipped over).
__device__ __forceinline__ int camera_of_obs(const int* __restrict__ offsets, int C, int v) {
    int lo = 0, hi = C - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(offsets + mid) <= v) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// The camera that owns packed cell g (every camera has at least one cell).
__device__ __forceinline__ int camera_of_cell(const RenderCamera* __restrict__ cams, int C, int g) {
    int lo = 0, hi = C - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(&cams[mid].cell0) <= g) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// Row r of the pose times [x, y, z, 1] in one stated float32 order, ((r0 x + r1 y) + r2 z) + r3, without contraction.
__device__ __forceinline__ float pose_row(const float* r, float x, float y, float z) {
    return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r[0], x), __fmul_rn(r[1], y)), __fmul_rn(r[2], z)), r[3]);
}

// Pass 1: project each observation once; its cell (-1 when its point index is out of range or its projection is NaN, both
// flagged in the camera's status) and its depth.  Negative depths register with their cell's first_neg.
__global__ void __launch_bounds__(kThreads) render_project_kernel(const RenderArgs a) {
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v >= a.V) return;
    const int c = camera_of_obs(a.offsets, a.C, v);
    const RenderCamera& cam = a.cams[c];
    const int i = __ldg(a.indices + v);
    int cell = -1;
    float z = 0.f;
    if (i < 0 || i >= a.P) {
        atomicOr(&a.status[c], kRenderBadIndex);
    } else {
        const float X = __ldg(a.points + 3 * (size_t)i), Y = __ldg(a.points + 3 * (size_t)i + 1),
                    Z = __ldg(a.points + 3 * (size_t)i + 2);
        float r[12];
#pragma unroll
        for (int k = 0; k < 12; ++k) r[k] = cam.pose[k];
        const float cx = pose_row(r, X, Y, Z), cy = pose_row(r + 4, X, Y, Z);
        z = pose_row(r + 8, X, Y, Z);
        // ((c * f) / z) * scale + w / 2, each op rounded to float32 as torch does with a Python float operand
        const float u = __fadd_rn(__fmul_rn(__fdiv_rn(__fmul_rn(cx, cam.f), z), cam.scale), cam.half_w);
        const float w = __fadd_rn(__fmul_rn(__fdiv_rn(__fmul_rn(cy, cam.f), z), cam.scale), cam.half_h);
        if (isnan(u) || isnan(w)) {
            atomicOr(&a.status[c], kRenderNaN);
        } else {
            // torch.clamp(t, 0, side - 1) then int(): truncation of a value >= 0
            const int col = (int)fminf(fmaxf(u, 0.f), (float)(cam.W - 1));
            const int row = (int)fminf(fmaxf(w, 0.f), (float)(cam.H - 1));
            cell = cam.cell0 + row * cam.W + col;
            if (z < 0.f) atomicMin(&a.first_neg[cell], (unsigned)v);
        }
    }
    a.obs_cell[v] = cell;
    a.obs_z[v] = z;
}

// Pass 2: the last depth-0 observation of each cell that the reference writes (before the cell's first negative depth).
__global__ void __launch_bounds__(kThreads) render_zero_kernel(const RenderArgs a) {
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v >= a.V) return;
    const int cell = a.obs_cell[v];
    if (cell < 0 || a.obs_z[v] != 0.f) return;
    if ((unsigned)v < a.first_neg[cell]) atomicMax(&a.last_zero[cell], v);
}

// Pass 3: the nearest non-zero depth after the cell's last written depth-0 point, the earliest observation on a tie.
__global__ void __launch_bounds__(kThreads) render_nearest_kernel(const RenderArgs a) {
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v >= a.V) return;
    const int cell = a.obs_cell[v];
    if (cell < 0) return;
    const float z = a.obs_z[v];
    if (z == 0.f || v <= a.last_zero[cell]) return;
    atomicMin(&a.key[cell], (unsigned long long)depth_key(z) << 32 | (unsigned)v);
}

// Pass 4: one thread per cell writes the winner's coordinates (zeros for an empty cell), its depth, and counts the written
// cells of each camera (one atomic per camera and warp).
__global__ void __launch_bounds__(kThreads) render_resolve_kernel(const RenderArgs a) {
    const int g = blockIdx.x * kThreads + threadIdx.x;
    const bool in = g < a.cells;
    int c = -1, obs = -1;
    if (in) {
        c = camera_of_cell(a.cams, a.C, g);
        const RenderCamera& cam = a.cams[c];
        const unsigned long long k = a.key[g];
        obs = k != ~0ull ? (int)(unsigned)k : a.last_zero[g];
        float x = 0.f, y = 0.f, zc = 0.f, depth = 0.f;
        if (obs >= 0) {
            const size_t i = (size_t)__ldg(a.indices + obs);
            x = __ldg(a.points + 3 * i);
            y = __ldg(a.points + 3 * i + 1);
            zc = __ldg(a.points + 3 * i + 2);
            depth = a.obs_z[obs];
        }
        const size_t plane = (size_t)cam.H * cam.W, local = (size_t)(g - cam.cell0);
        float* m = a.maps + 3 * (size_t)cam.cell0 + local;
        m[0] = x;
        m[plane] = y;
        m[2 * plane] = zc;
        if (a.zbuf) a.zbuf[g] = depth;
    }
    const bool wrote = in && obs >= 0;
    const unsigned mask = __ballot_sync(0xffffffffu, wrote);
    if (wrote) {
        const unsigned peers = __match_any_sync(mask, c);
        if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&a.count[c], __popc(peers));
    }
}

}  // namespace

void launch_render(const RenderArgs& a, cudaStream_t st) {
    cudaMemsetAsync(a.first_neg, 0xFF, (size_t)a.cells * sizeof(unsigned), st);
    cudaMemsetAsync(a.last_zero, 0xFF, (size_t)a.cells * sizeof(int), st);
    cudaMemsetAsync(a.key, 0xFF, (size_t)a.cells * sizeof(unsigned long long), st);
    cudaMemsetAsync(a.count, 0, (size_t)a.C * sizeof(int), st);
    cudaMemsetAsync(a.status, 0, (size_t)a.C * sizeof(int), st);
    if (a.V > 0) {
        const unsigned grid = (unsigned)(((long long)a.V + kThreads - 1) / kThreads);
        render_project_kernel<<<grid, kThreads, 0, st>>>(a);
        render_zero_kernel<<<grid, kThreads, 0, st>>>(a);
        render_nearest_kernel<<<grid, kThreads, 0, st>>>(a);
    }
    render_resolve_kernel<<<(unsigned)(((long long)a.cells + kThreads - 1) / kThreads), kThreads, 0, st>>>(a);
}

}  // namespace esacb200
