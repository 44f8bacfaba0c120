// The two expert losses in the C ABI of include/esac_b200.h: the reprojection loss (ref_expert.py) and the scene-coordinate
// loss (init_expert.py), eager over stacked or ragged batches and stream-ordered.
#include <cuda_runtime.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "capi_internal.h"

using namespace esacb200;
using namespace esacb200::capi;

namespace esacb200::capi {

// Offsets of B host images packed into one device buffer, each at a 16-byte aligned offset (so that an image keeps the
// 128-bit load path a single-image call would give it).  Returns the total.
size_t pack_offsets(const std::vector<size_t>& bytes, std::vector<size_t>& off) {
    size_t total = 0;
    off.resize(bytes.size());
    for (size_t b = 0; b < bytes.size(); ++b) {
        off[b] = total;
        total += (bytes[b] + 15) & ~(size_t)15;
    }
    return total;
}

// Copies between B host images and their packed device copies; runs of images that lie back to back on both sides go as
// one copy (a stacked tensor with N % 4 == 0 is a single copy).
int copy_packed(esacb200_ctx* ctx, char* const* host, const std::vector<size_t>& bytes, const std::vector<size_t>& off, char* dev,
                bool to_device, cudaStream_t stream) {
    const size_t B = bytes.size();
    for (size_t b = 0; b < B;) {
        size_t e = b + 1, len = bytes[b];
        while (e < B && host[e] == host[e - 1] + bytes[e - 1] && off[e] == off[e - 1] + bytes[e - 1]) len += bytes[e++];
        if (to_device) CK(cudaMemcpyAsync(dev + off[b], host[b], len, cudaMemcpyHostToDevice, stream));
        else CK(cudaMemcpyAsync(host[b], dev + off[b], len, cudaMemcpyDeviceToHost, stream));
        b = e;
    }
    return 0;
}

// Stages the B images of one argument on the device: device pointers are used as they are; host images are packed into
// `buf` at 16-byte aligned offsets (and copied there when `upload`).  dev[b] receives image b's device address.
template <class T>
int stage_images(esacb200_ctx* ctx, T* const* ptrs, const std::vector<size_t>& bytes, bool device, bool upload, DevBuf& buf,
                 std::vector<T*>& dev, std::vector<size_t>& off) {
    const size_t B = bytes.size();
    dev.resize(B);
    if (device) {
        for (size_t b = 0; b < B; ++b) dev[b] = ptrs[b];
        return 0;
    }
    CK(buf.ensure(pack_offsets(bytes, off)));
    for (size_t b = 0; b < B; ++b) dev[b] = (T*)((char*)buf.p + off[b]);
    if (upload) return copy_packed(ctx, (char* const*)ptrs, bytes, off, (char*)buf.p, true, ctx->stream);
    return 0;
}
template int stage_images<const float>(esacb200_ctx*, const float* const*, const std::vector<size_t>&, bool, bool, DevBuf&,
                                       std::vector<const float*>&, std::vector<size_t>&);

}  // namespace esacb200::capi

namespace {

// Orders a loss call's per-image records by load path (128-bit first) so that each path is one launch over a contiguous
// slice of the table; returns the bytes of the table.
template <class Rec>
size_t order_by_path(const std::vector<Rec>& recs, const std::vector<char>& vec, std::vector<Rec>& out, int& n_vec, int& max_vec,
                     int& max_sc) {
    out.clear();
    n_vec = max_vec = max_sc = 0;
    for (size_t i = 0; i < recs.size(); ++i)
        if (vec[i]) { out.push_back(recs[i]); ++n_vec; if (recs[i].blocks > max_vec) max_vec = recs[i].blocks; }
    for (size_t i = 0; i < recs.size(); ++i)
        if (!vec[i]) { out.push_back(recs[i]); if (recs[i].blocks > max_sc) max_sc = recs[i].blocks; }
    return out.size() * sizeof(Rec);
}

}  // namespace

extern "C" {

// -------------------------------------------------------------------------------------------------
// The two losses' steps that the eager ragged calls and the stream-ordered calls share: the per-image size checks, the
// per-image records, the workspace layout and the launches.

static size_t align64(size_t n) { return (n + 63) & ~(size_t)63; }

// Byte offsets in the loss workspace of a call of B images whose blocks have `parts` partials.
//   reprojection: [tickets B u32] [img B x kReprojImgFloats f32] [records] [losses B f64] [bad B i32] [partials f64 each]
//   coordinates:  [tickets B u32 | counts B u32] [records] [losses B f64] [valid counts B i64] [partials 2 f64 each]
// The eager reprojection loss leaves `bad` unused: a singular ground truth fails it before anything is enqueued.
struct LossLayout {
    size_t img = 0, rec, loss, flags, part, end;
};
static LossLayout reproj_layout(int B, long long parts) {
    LossLayout L;
    L.img = align64((size_t)B * 4);
    L.rec = L.img + align64((size_t)B * kReprojImgFloats * sizeof(float));
    L.loss = L.rec + align64((size_t)B * sizeof(ReprojImage));
    L.flags = L.loss + align64((size_t)B * 8);
    L.part = L.flags + align64((size_t)B * 4);
    L.end = L.part + (size_t)parts * 8;
    return L;
}
static LossLayout coord_layout(int B, long long parts) {
    LossLayout L;
    L.rec = align64((size_t)B * 8);
    L.loss = L.rec + align64((size_t)B * sizeof(CoordImage));
    L.flags = L.loss + align64((size_t)B * 8);
    L.part = L.flags + align64((size_t)B * 8);
    L.end = L.part + (size_t)parts * 2 * 8;
    return L;
}

// The per-image sizes of a reprojection-loss call: positive, at most 2^30 cells.  `what`: the entry point named in front of
// each message, or null.
static int reproj_sizes(esacb200_ctx* ctx, const char* what, int B, const int* H, const int* W) {
    const char* sep = what ? ": " : "";
    if (!what) what = "";
    for (int b = 0; b < B; ++b) {
        if (H[b] <= 0 || W[b] <= 0) return fail(ctx, ESACB200_ERR_ARG, "%s%simage %d: bad size %dx%d", what, sep, b, W[b], H[b]);
        if ((long long)H[b] * W[b] > (1ll << 30))
            return fail(ctx, ESACB200_ERR_ARG, "%s%simage %d: map %dx%d too large", what, sep, b, W[b], H[b]);
    }
    return 0;
}

// The records of a reprojection-loss call on the B images at the device addresses coords[b] and grads[b] (grads, or an
// entry of it, null: no gradient) of elements of `esize` bytes, and per image whether it takes the vector load path.
// Returns the blocks' partials.
static long long reproj_records(int B, const void* const* coords, void* const* grads, const int* H, const int* W, int esize,
                                std::vector<ReprojImage>& recs, std::vector<char>& vec) {
    recs.resize((size_t)B);
    vec.resize((size_t)B);
    long long parts = 0;
    for (int b = 0; b < B; ++b) {
        ReprojImage& r = recs[b];
        r.coords = coords[b];
        r.grads = grads ? grads[b] : nullptr;
        r.N = H[b] * W[b];
        r.W = W[b];
        r.b = b;
        r.blocks = reproj_blocks_per_image(r.N);
        r.part0 = parts;
        parts += r.blocks;
        vec[b] = reproj_vec_ok(r.coords, r.grads, r.N, r.W, esize);
    }
    return parts;
}

// The reprojection loss's launches, one per load path, on the workspace at `base` laid out as L, whose records are in
// order_by_path's order (n_vec on the vector path first), for maps of `dtype` with gradients scaled by grad_scale (or not).
// They run on run's stream and count in its kernel_launches.
static void reproj_launches(esacb200_ctx* run, char* base, const LossLayout& L, int B, int n_vec, int max_vec, int max_sc,
                            int sub, float cut, float maxReproj, float minDepth, int dtype, const float* grad_scale) {
    const ReprojImage* rec = (const ReprojImage*)(base + L.rec);
    for (int path = 0; path < 2; ++path) {
        const int n = path == 0 ? n_vec : B - n_vec;
        if (n == 0) continue;
        launch_reproj(path == 0, dtype, rec + (path == 0 ? 0 : n_vec), n, path == 0 ? max_vec : max_sc,
                      (const float*)(base + L.img), (float)sub, cut, maxReproj, minDepth, grad_scale, (double*)(base + L.part),
                      (unsigned*)base, (double*)(base + L.loss), run->stream);
        run->st.kernel_launches += 1;
    }
}

// The per-image sizes of a coordinate-loss call: positive, prediction and ground truth at most 1 apart, at most 2^30 cells.
// `what`: the entry point named in front of each message, or null.
static int coord_sizes(esacb200_ctx* ctx, const char* what, int B, const int* Hp, const int* Wp, const int* Hg, const int* Wg) {
    const char* sep = what ? ": " : "";
    if (!what) what = "";
    for (int b = 0; b < B; ++b) {
        if (Hp[b] <= 0 || Wp[b] <= 0 || Hg[b] <= 0 || Wg[b] <= 0)
            return fail(ctx, ESACB200_ERR_ARG, "%s%simage %d: bad sizes prediction %dx%d ground truth %dx%d", what, sep, b, Hp[b],
                        Wp[b], Hg[b], Wg[b]);
        if (abs(Hp[b] - Hg[b]) > 1 || abs(Wp[b] - Wg[b]) > 1)   // util.assert_size tolerates 1 cell
            return fail(ctx, ESACB200_ERR_ARG, "%s%simage %d: size mismatch: prediction %dx%d, ground truth %dx%d (at most 1 apart)",
                        what, sep, b, Hp[b], Wp[b], Hg[b], Wg[b]);
        if ((long long)Hp[b] * Wp[b] > (1ll << 30) || (long long)Hg[b] * Wg[b] > (1ll << 30))
            return fail(ctx, ESACB200_ERR_ARG, "%s%simage %d: map too large", what, sep, b);
    }
    return 0;
}

// The records of a coordinate-loss call on the B images at the device addresses pred[b], gt[b] and grads[b] (grads, or an
// entry of it, null: no gradient; pred and grads of elements of `esize` bytes), and per image whether it takes the vector
// load path.  Returns the blocks' partials.
static long long coord_records(int B, const void* const* pred, const float* const* gt, void* const* grads, const int* Hp,
                               const int* Wp, const int* Hg, const int* Wg, int esize, std::vector<CoordImage>& recs,
                               std::vector<char>& vec) {
    recs.resize((size_t)B);
    vec.resize((size_t)B);
    long long parts = 0;
    for (int b = 0; b < B; ++b) {
        CoordImage& r = recs[b];
        r.pred = pred[b];
        r.gt = gt[b];
        r.grads = grads ? grads[b] : nullptr;
        vec[b] = coord_image(r, Hp[b], Wp[b], Hg[b], Wg[b], esize);
        r.b = b;
        r.part0 = parts;
        parts += r.blocks;
    }
    return parts;
}

// The coordinate loss's launches, per load path the count pass (with gradients) and the loss pass, on the workspace at
// `base` laid out as L, whose records are in order_by_path's order; dtype and grad_scale as for reproj_launches.  They run
// on run's stream and count in its kernel_launches.
static void coord_launches(esacb200_ctx* run, char* base, const LossLayout& L, int B, bool grads, int n_vec, int max_vec,
                           int max_sc, float cut, int dtype, const float* grad_scale) {
    const CoordImage* rec = (const CoordImage*)(base + L.rec);
    for (int path = 0; path < 2; ++path) {
        const int n = path == 0 ? n_vec : B - n_vec;
        if (n == 0) continue;
        for (int pass = grads ? 1 : 2; pass <= 2; ++pass) {
            launch_coord_loss(path == 0, pass, grads, dtype, rec + (path == 0 ? 0 : n_vec), n, path == 0 ? max_vec : max_sc, cut,
                              grad_scale, (unsigned*)base + B, (double*)(base + L.part), (unsigned*)base,
                              (double*)(base + L.loss), (long long*)(base + L.flags), run->stream);
            run->st.kernel_launches += 1;
        }
    }
}

// The element type of a typed loss call: a known dtype code; grad_scale only with a 16-bit code, and then device memory;
// 16-bit images (device: whether every image argument is device memory) only in device memory.  esize receives the
// element's bytes.  `what`: the entry point named in front of each message, or null.
static int loss_dtype(esacb200_ctx* ctx, const char* what, int dtype, const float* grad_scale, bool device, int& esize) {
    const char* sep = what ? ": " : "";
    if (!what) what = "";
    if (dtype != ESACB200_FLOAT32 && dtype != ESACB200_FLOAT16 && dtype != ESACB200_BFLOAT16)
        return fail(ctx, ESACB200_ERR_ARG, "%s%sunknown dtype code %d", what, sep, dtype);
    esize = loss_elem_bytes(dtype);
    if (dtype == ESACB200_FLOAT32) {
        if (grad_scale) return fail(ctx, ESACB200_ERR_ARG, "%s%sgrad_scale is for float16 / bfloat16 maps only", what, sep);
        return 0;
    }
    if (!device) return fail(ctx, ESACB200_ERR_ARG, "%s%sfloat16 / bfloat16 maps must be device memory", what, sep);
    if (grad_scale && !is_device_ptr(grad_scale))
        return fail(ctx, ESACB200_ERR_ARG, "%s%sgrad_scale must be device memory", what, sep);
    return 0;
}
static_assert(ESACB200_FLOAT32 == kLossF32 && ESACB200_FLOAT16 == kLossF16 && ESACB200_BFLOAT16 == kLossBF16,
              "the C ABI's dtype codes are the kernels' LossDtype");

// -------------------------------------------------------------------------------------------------
// The reprojection loss over B images, each with its own size: one launch per load path (128-bit / scalar, chosen per
// image as a single-image call would choose it), each image cut into the blocks a single-image call uses.
int esacb200_reproj_loss_ragged_typed(esacb200_ctx* ctx, int B, int dtype, const void* const* coords, void* const* grads,
                                      const int* H, const int* W, const float* gt_poses, const int* shiftX, const int* shiftY,
                                      const float* f, const float* ppx, const float* ppy, int sub, float cut, float maxReproj,
                                      float minDepth, const float* grad_scale, double* out_losses) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !H || !W || !gt_poses || !out_losses) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    if (!f || !ppx || !ppy) return fail(ctx, ESACB200_ERR_ARG, "null camera array");
    if (B <= 0 || sub <= 0) return fail(ctx, ESACB200_ERR_ARG, "bad sizes B=%d sub=%d", B, sub);
    int rc = reproj_sizes(ctx, nullptr, B, H, W);
    if (rc) return rc;
    bool c_dev = false, g_dev = false;
    if ((rc = pointer_kind(ctx, (const void* const*)coords, B, "coords", c_dev))) return rc;
    if (grads && (rc = pointer_kind(ctx, (const void* const*)grads, B, "grads", g_dev))) return rc;
    int esize = 0;
    if ((rc = loss_dtype(ctx, nullptr, dtype, grad_scale, c_dev && (!grads || g_dev), esize))) return rc;
    begin_call(ctx);
    std::vector<size_t> bytes((size_t)B), c_off, g_off;
    for (int b = 0; b < B; ++b) bytes[b] = (size_t)3 * H[b] * W[b] * esize;
    std::vector<const void*> d_coords;
    std::vector<void*> d_grads((size_t)B, nullptr);
    rc = stage_images(ctx, coords, bytes, c_dev, true, ctx->coords, d_coords, c_off);
    if (rc) return rc;
    if (grads && (rc = stage_images(ctx, grads, bytes, g_dev, false, ctx->grads, d_grads, g_off))) return rc;
    std::vector<float> gt((size_t)B * 16);
    if (is_device_ptr(gt_poses)) {
        CK(cudaMemcpyAsync(gt.data(), gt_poses, gt.size() * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    } else {
        memcpy(gt.data(), gt_poses, gt.size() * sizeof(float));
    }
    // world->camera rows: inverse of the affine camera->world matrix (torch's .inverse()[0:3,:], ref_expert.py:127)
    std::vector<float> img((size_t)B * kReprojImgFloats, 0.f);
    for (int b = 0; b < B; ++b)
        if (!reproj_img_row(gt.data() + (size_t)b * 16, shiftX ? shiftX[b] : 0, shiftY ? shiftY[b] : 0, f[b], ppx[b], ppy[b],
                            img.data() + (size_t)b * kReprojImgFloats))
            return fail(ctx, ESACB200_ERR_ARG, "image %d: ground-truth pose is singular", b);
    std::vector<ReprojImage> recs, ordered;
    std::vector<char> vec;
    const long long parts = reproj_records(B, d_coords.data(), d_grads.data(), H, W, esize, recs, vec);
    int n_vec, max_vec, max_sc;
    const size_t rec_bytes = order_by_path(recs, vec, ordered, n_vec, max_vec, max_sc);
    const LossLayout L = reproj_layout(B, parts);
    CK(ctx->scratch.ensure(L.end));
    char* base = (char*)ctx->scratch.p;
    std::vector<char> staging(L.rec - L.img + rec_bytes);
    memcpy(staging.data(), img.data(), img.size() * sizeof(float));
    memcpy(staging.data() + (L.rec - L.img), ordered.data(), rec_bytes);
    CK(cudaMemsetAsync(base, 0, L.img, ctx->stream));
    CK(cudaMemcpyAsync(base + L.img, staging.data(), staging.size(), cudaMemcpyHostToDevice, ctx->stream));
    mark(ctx, EV_H2D);
    mark(ctx, EV_FOLD);  // ms_score = the kernels alone
    reproj_launches(ctx, base, L, B, n_vec, max_vec, max_sc, sub, cut, maxReproj, minDepth, dtype, grad_scale);
    CK(cudaGetLastError());
    mark(ctx, EV_SCORE);
    if (grads && !g_dev) {
        rc = copy_packed(ctx, (char* const*)grads, bytes, g_off, (char*)ctx->grads.p, false, ctx->stream);
        if (rc) return rc;
    }
    CK(cudaMemcpyAsync(out_losses, base + L.loss, (size_t)B * 8, cudaMemcpyDeviceToHost, ctx->stream));
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_reproj_loss_ragged(esacb200_ctx* ctx, int B, const float* const* coords, float* const* grads, const int* H,
                                const int* W, const float* gt_poses, const int* shiftX, const int* shiftY, const float* f,
                                const float* ppx, const float* ppy, int sub, float cut, float maxReproj, float minDepth,
                                double* out_losses) {
    return esacb200_reproj_loss_ragged_typed(ctx, B, ESACB200_FLOAT32, (const void* const*)coords, (void* const*)grads, H, W,
                                             gt_poses, shiftX, shiftY, f, ppx, ppy, sub, cut, maxReproj, minDepth, nullptr,
                                             out_losses);
}

// B images of one shape: the pointer and size arrays of a [B,3,H,W] tensor.
int esacb200_reproj_loss_cameras(esacb200_ctx* ctx, int B, const float* coords, float* grads, int H, int W, const float* gt_poses,
                                 const int* shiftX, const int* shiftY, const float* f, const float* ppx, const float* ppy, int sub,
                                 float cut, float maxReproj, float minDepth, double* out_losses) try {
    if (!ctx) return ESACB200_ERR_ARG;
    if (!coords || !gt_poses || !out_losses) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    if (!f || !ppx || !ppy) return fail(ctx, ESACB200_ERR_ARG, "null camera array");
    if (B <= 0 || H <= 0 || W <= 0 || sub <= 0) return fail(ctx, ESACB200_ERR_ARG, "bad sizes B=%d H=%d W=%d sub=%d", B, H, W, sub);
    if ((long long)H * W > (1ll << 30)) return fail(ctx, ESACB200_ERR_ARG, "map %dx%d too large", W, H);
    const size_t n = (size_t)3 * H * W;
    const auto cp = slices(coords, B, n);
    const auto gp = slices(grads, B, n);
    const std::vector<int> hs((size_t)B, H), ws((size_t)B, W);
    return esacb200_reproj_loss_ragged(ctx, B, cp.data(), grads ? gp.data() : nullptr, hs.data(), ws.data(), gt_poses, shiftX, shiftY,
                                       f, ppx, ppy, sub, cut, maxReproj, minDepth, out_losses);
} ESAC_ABI_CATCH(ctx)

int esacb200_reproj_loss(esacb200_ctx* ctx, int B, const float* coords, float* grads, int H, int W, const float* gt_poses,
                         const int* shiftX, const int* shiftY, float f, float ppx, float ppy, int sub, float cut,
                         float maxReproj, float minDepth, double* out_losses) try {
    if (!ctx) return ESACB200_ERR_ARG;
    const size_t n = B > 0 ? (size_t)B : 1;  // B <= 0 is rejected by the call below, with its usual message
    const std::vector<float> fs(n, f), cx(n, ppx), cy(n, ppy);
    return esacb200_reproj_loss_cameras(ctx, B, coords, grads, H, W, gt_poses, shiftX, shiftY, fs.data(), cx.data(), cy.data(), sub,
                                        cut, maxReproj, minDepth, out_losses);
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
// The coordinate loss over B images, each with its own prediction and ground-truth size: one launch per load path and
// pass, each image cut into the blocks a single-image call uses.
int esacb200_coord_loss_ragged_typed(esacb200_ctx* ctx, int B, int dtype, const void* const* pred, const int* Hp, const int* Wp,
                                     const float* const* gt, const int* Hg, const int* Wg, void* const* grads, float cut,
                                     const float* grad_scale, double* out_losses, int64_t* out_counts) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!pred || !gt || !Hp || !Wp || !Hg || !Wg || !out_losses) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    if (B <= 0) return fail(ctx, ESACB200_ERR_ARG, "bad sizes B=%d", B);
    int rc = coord_sizes(ctx, nullptr, B, Hp, Wp, Hg, Wg);
    if (rc) return rc;
    bool p_dev = false, q_dev = false, g_dev = false;
    if ((rc = pointer_kind(ctx, (const void* const*)pred, B, "pred", p_dev))) return rc;
    if ((rc = pointer_kind(ctx, (const void* const*)gt, B, "gt", q_dev))) return rc;
    if (grads && (rc = pointer_kind(ctx, (const void* const*)grads, B, "grads", g_dev))) return rc;
    int esize = 0;
    if ((rc = loss_dtype(ctx, nullptr, dtype, grad_scale, p_dev && (!grads || g_dev), esize))) return rc;
    begin_call(ctx);
    std::vector<size_t> pbytes((size_t)B), gbytes((size_t)B), p_off, q_off, g_off;
    for (int b = 0; b < B; ++b) {
        pbytes[b] = (size_t)3 * Hp[b] * Wp[b] * esize;
        gbytes[b] = (size_t)3 * Hg[b] * Wg[b] * sizeof(float);
    }
    std::vector<const void*> d_pred;
    std::vector<const float*> d_gt;
    std::vector<void*> d_grads((size_t)B, nullptr);
    if ((rc = stage_images(ctx, pred, pbytes, p_dev, true, ctx->coords, d_pred, p_off))) return rc;
    if ((rc = stage_images(ctx, gt, gbytes, q_dev, true, ctx->coords_alt, d_gt, q_off))) return rc;
    if (grads && (rc = stage_images(ctx, grads, pbytes, g_dev, false, ctx->grads, d_grads, g_off))) return rc;
    std::vector<CoordImage> recs, ordered;
    std::vector<char> vec;
    const long long parts = coord_records(B, d_pred.data(), d_gt.data(), d_grads.data(), Hp, Wp, Hg, Wg, esize, recs, vec);
    int n_vec, max_vec, max_sc;
    const size_t rec_bytes = order_by_path(recs, vec, ordered, n_vec, max_vec, max_sc);
    const LossLayout L = coord_layout(B, parts);
    CK(ctx->scratch.ensure(L.end));
    char* base = (char*)ctx->scratch.p;
    CK(cudaMemsetAsync(base, 0, L.rec, ctx->stream));
    CK(cudaMemcpyAsync(base + L.rec, ordered.data(), rec_bytes, cudaMemcpyHostToDevice, ctx->stream));
    mark(ctx, EV_H2D);
    mark(ctx, EV_FOLD);  // ms_score = the kernels alone
    coord_launches(ctx, base, L, B, grads != nullptr, n_vec, max_vec, max_sc, cut, dtype, grad_scale);
    CK(cudaGetLastError());
    mark(ctx, EV_SCORE);
    if (grads && !g_dev) {
        rc = copy_packed(ctx, (char* const*)grads, pbytes, g_off, (char*)ctx->grads.p, false, ctx->stream);
        if (rc) return rc;
    }
    CK(cudaMemcpyAsync(out_losses, base + L.loss, (size_t)B * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (out_counts) CK(cudaMemcpyAsync(out_counts, base + L.flags, (size_t)B * 8, cudaMemcpyDeviceToHost, ctx->stream));
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_coord_loss_ragged(esacb200_ctx* ctx, int B, const float* const* pred, const int* Hp, const int* Wp,
                               const float* const* gt, const int* Hg, const int* Wg, float* const* grads, float cut,
                               double* out_losses, int64_t* out_counts) {
    return esacb200_coord_loss_ragged_typed(ctx, B, ESACB200_FLOAT32, (const void* const*)pred, Hp, Wp, gt, Hg, Wg,
                                            (void* const*)grads, cut, nullptr, out_losses, out_counts);
}

// B images of one shape: the pointer and size arrays of [B,3,Hp,Wp] / [B,3,Hg,Wg] tensors.
int esacb200_coord_loss(esacb200_ctx* ctx, int B, const float* pred, int Hp, int Wp, const float* gt, int Hg, int Wg,
                        float* grads, float cut, double* out_losses, int64_t* out_counts) try {
    if (!ctx) return ESACB200_ERR_ARG;
    if (!pred || !gt || !out_losses) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    if (B <= 0 || Hp <= 0 || Wp <= 0 || Hg <= 0 || Wg <= 0)
        return fail(ctx, ESACB200_ERR_ARG, "bad sizes B=%d prediction %dx%d ground truth %dx%d", B, Hp, Wp, Hg, Wg);
    if (abs(Hp - Hg) > 1 || abs(Wp - Wg) > 1)   // util.assert_size tolerates 1 cell
        return fail(ctx, ESACB200_ERR_ARG, "size mismatch: prediction %dx%d, ground truth %dx%d (at most 1 apart)", Hp, Wp, Hg, Wg);
    if ((long long)Hp * Wp > (1ll << 30) || (long long)Hg * Wg > (1ll << 30))
        return fail(ctx, ESACB200_ERR_ARG, "map too large");
    const size_t np = (size_t)3 * Hp * Wp;
    const auto pp = slices(pred, B, np), qp = slices(gt, B, (size_t)3 * Hg * Wg);
    const auto gp = slices(grads, B, np);
    const std::vector<int> hp((size_t)B, Hp), wp((size_t)B, Wp), hg((size_t)B, Hg), wg((size_t)B, Wg);
    return esacb200_coord_loss_ragged(ctx, B, pp.data(), hp.data(), wp.data(), qp.data(), hg.data(), wg.data(),
                                      grads ? gp.data() : nullptr, cut, out_losses, out_counts);
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
// Stream-ordered losses.  The eager ragged calls' records and launches, run in the context ctx->async on the caller's device
// arrays: the records reach the workspace as prep-kernel parameters (loss_async.cu), the ground truth, pads and camera are
// read on the device, and a finish kernel writes the caller's outputs.  Nothing here synchronises, reads back or queries an
// event, and a call that a capture records allocates nothing.

// Makes the loss workspace hold `bytes`: grows it when no capture has used it yet, else fails without touching it.
static int loss_workspace(esacb200_ctx* ctx, esacb200_ctx* a, size_t bytes, bool capturing, const char* what) {
    if (bytes <= a->loss_ws.cap) return 0;
    if (capturing || a->loss_frozen)
        return fail(ctx, ESACB200_ERR_ARG,
                    "%s: this call needs %zu bytes of loss workspace, more than %s, and a graph that holds it may still be "
                    "replayed; call reserve_loss_async (esacb200_reserve_loss_async) with the largest batch and map before the "
                    "first capture", what, bytes, capturing ? "was reserved before this capture" : "an earlier capture used");
    CK(a->loss_ws.ensure(bytes));
    return 0;
}

// The B image pointers of one argument are device memory.
static int device_images(esacb200_ctx* ctx, const char* what, const char* name, const void* const* p, int B) {
    for (int b = 0; b < B; ++b) {
        if (!p[b]) return fail(ctx, ESACB200_ERR_ARG, "%s: image %d: %s is null", what, b, name);
        if (!is_device_ptr(p[b]))
            return fail(ctx, ESACB200_ERR_ARG, "%s takes device pointers only: image %d: %s is host memory", what, b, name);
    }
    return 0;
}

// The async context of a loss call, and whether the stream is being captured.
static int begin_loss_async(esacb200_ctx* ctx, esacb200_ctx*& a, bool& capturing) {
    int rc = stream_capturing(ctx, capturing);
    if (!rc) rc = async_context(ctx, capturing, "loss_async", &a);
    return rc;
}

int esacb200_reserve_loss_async(esacb200_ctx* ctx, int B, int H, int W) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (B <= 0 || H <= 0 || W <= 0 || (long long)H * W > (1ll << 30))
        return fail(ctx, ESACB200_ERR_ARG, "reserve_loss_async: bad sizes B=%d H=%d W=%d", B, H, W);
    esacb200_ctx* a = nullptr;
    const int rc = reserve_context(ctx, "loss_async", &a);
    if (rc) return rc;
    const long long parts = (long long)B * reproj_max_blocks(H * W);
    return loss_workspace(ctx, a, std::max(reproj_layout(B, parts).end, coord_layout(B, parts).end), false, "reserve_loss_async");
} ESAC_ABI_CATCH(ctx)

int esacb200_reproj_loss_async_typed(esacb200_ctx* ctx, int B, int dtype, const void* const* coords, void* const* grads,
                                     const int* H, const int* W, const float* gt_poses, const int32_t* shifts,
                                     const float* cameras, int sub, float cut, float maxReproj, float minDepth,
                                     const float* grad_scale, double* out_losses, int32_t* out_status) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "reproj_loss_async";
    if (!coords || !H || !W) return fail(ctx, ESACB200_ERR_ARG, "%s: null pointer or size array", what);
    if (B <= 0 || B > 65535 || sub <= 0) return fail(ctx, ESACB200_ERR_ARG, "%s: bad sizes B=%d sub=%d", what, B, sub);
    const void* ptrs[] = {gt_poses, shifts, cameras, out_losses, out_status};
    const char* names[] = {"gt_poses", "shifts", "cameras", "out_losses", "out_status"};
    int rc = reproj_sizes(ctx, what, B, H, W);
    if (!rc) rc = device_args(ctx, what, 5, ptrs, names);
    if (!rc) rc = device_images(ctx, what, "coords", (const void* const*)coords, B);
    if (!rc && grads) rc = device_images(ctx, what, "grads", (const void* const*)grads, B);
    int esize = 0;
    if (!rc) rc = loss_dtype(ctx, what, dtype, grad_scale, true, esize);
    if (rc) return rc;
    esacb200_ctx* a = nullptr;
    bool capturing = false;
    if ((rc = begin_loss_async(ctx, a, capturing))) return rc;
    std::vector<ReprojImage> recs, ordered;
    std::vector<char> vec;
    const long long parts = reproj_records(B, coords, grads, H, W, esize, recs, vec);
    int n_vec, max_vec, max_sc;
    order_by_path(recs, vec, ordered, n_vec, max_vec, max_sc);
    const LossLayout L = reproj_layout(B, parts);
    if ((rc = loss_workspace(ctx, a, L.end, capturing, what))) return rc;
    if (capturing) a->loss_frozen = true;
    char* base = (char*)a->loss_ws.p;
    ReprojImage* d_rec = (ReprojImage*)(base + L.rec);
    double* losses = (double*)(base + L.loss);
    int* bad = (int*)(base + L.flags);
    CK(cudaMemsetAsync(base, 0, L.img, a->stream));
    a->st.kernel_launches +=
        launch_reproj_prep(ordered.data(), B, d_rec, gt_poses, shifts, cameras, (float*)(base + L.img), bad, a->stream);
    reproj_launches(a, base, L, B, n_vec, max_vec, max_sc, sub, cut, maxReproj, minDepth, dtype, grad_scale);
    launch_reproj_finish(d_rec, B, grads != nullptr, dtype, grad_scale, losses, bad, out_losses, out_status, a->stream);
    a->st.kernel_launches += 1;
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_reproj_loss_async(esacb200_ctx* ctx, int B, const float* const* coords, float* const* grads, const int* H,
                               const int* W, const float* gt_poses, const int32_t* shifts, const float* cameras, int sub,
                               float cut, float maxReproj, float minDepth, double* out_losses, int32_t* out_status) {
    return esacb200_reproj_loss_async_typed(ctx, B, ESACB200_FLOAT32, (const void* const*)coords, (void* const*)grads, H, W,
                                            gt_poses, shifts, cameras, sub, cut, maxReproj, minDepth, nullptr, out_losses,
                                            out_status);
}

int esacb200_coord_loss_async_typed(esacb200_ctx* ctx, int B, int dtype, const void* const* pred, const int* Hp, const int* Wp,
                                    const float* const* gt, const int* Hg, const int* Wg, void* const* grads, float cut,
                                    const float* grad_scale, double* out_losses, int64_t* out_counts) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "coord_loss_async";
    if (!pred || !gt || !Hp || !Wp || !Hg || !Wg) return fail(ctx, ESACB200_ERR_ARG, "%s: null pointer or size array", what);
    if (B <= 0 || B > 65535) return fail(ctx, ESACB200_ERR_ARG, "%s: bad sizes B=%d", what, B);
    const void* ptrs[] = {out_losses, out_counts};
    const char* names[] = {"out_losses", "out_counts"};
    int rc = coord_sizes(ctx, what, B, Hp, Wp, Hg, Wg);
    if (!rc) rc = device_args(ctx, what, 2, ptrs, names, 2u);
    if (!rc) rc = device_images(ctx, what, "pred", (const void* const*)pred, B);
    if (!rc) rc = device_images(ctx, what, "gt", (const void* const*)gt, B);
    if (!rc && grads) rc = device_images(ctx, what, "grads", (const void* const*)grads, B);
    int esize = 0;
    if (!rc) rc = loss_dtype(ctx, what, dtype, grad_scale, true, esize);
    if (rc) return rc;
    esacb200_ctx* a = nullptr;
    bool capturing = false;
    if ((rc = begin_loss_async(ctx, a, capturing))) return rc;
    std::vector<CoordImage> recs, ordered;
    std::vector<char> vec;
    const long long parts = coord_records(B, pred, gt, grads, Hp, Wp, Hg, Wg, esize, recs, vec);
    int n_vec, max_vec, max_sc;
    order_by_path(recs, vec, ordered, n_vec, max_vec, max_sc);
    const LossLayout L = coord_layout(B, parts);
    if ((rc = loss_workspace(ctx, a, L.end, capturing, what))) return rc;
    if (capturing) a->loss_frozen = true;
    char* base = (char*)a->loss_ws.p;
    CK(cudaMemsetAsync(base, 0, L.rec, a->stream));
    a->st.kernel_launches += launch_coord_prep(ordered.data(), B, (CoordImage*)(base + L.rec), a->stream);
    coord_launches(a, base, L, B, grads != nullptr, n_vec, max_vec, max_sc, cut, dtype, grad_scale);
    launch_coord_finish(B, (const double*)(base + L.loss), (const long long*)(base + L.flags), out_losses, (long long*)out_counts,
                        a->stream);
    a->st.kernel_launches += 1;
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_coord_loss_async(esacb200_ctx* ctx, int B, const float* const* pred, const int* Hp, const int* Wp,
                              const float* const* gt, const int* Hg, const int* Wg, float* const* grads, float cut,
                              double* out_losses, int64_t* out_counts) {
    return esacb200_coord_loss_async_typed(ctx, B, ESACB200_FLOAT32, (const void* const*)pred, Hp, Wp, gt, Hg, Wg,
                                           (void* const*)grads, cut, nullptr, out_losses, out_counts);
}

}  // extern "C"
