// The hypotheses as an autograd node in the C ABI of include/esac_b200.h -- eager, ragged and stream-ordered forward and
// backward -- and the pose loss a caller may put behind it.
#include <cuda_runtime.h>
#include <string.h>

#include <string>
#include <vector>

#include "capi_internal.h"

using namespace esacb200;
using namespace esacb200::capi;

extern "C" {

// -------------------------------------------------------------------------------------------------
// The hypotheses as an autograd node: a forward that returns scores, refined poses and contributing flags and keeps what its
// backward needs in a caller-owned tape, and a backward that maps upstream gradients of (scores, poses) to the coordinates.
size_t esacb200_hypotheses_tape_bytes(int E, int H, int W, int M) {
    if (E <= 0 || H <= 0 || W <= 0 || M <= 0 || (long long)H * W > (1ll << 30)) return 0;
    return tape_bytes(M, H * W);
}

// The tape header of a hypotheses forward of problem P with probability floor min_prob.
static TapeHead tape_head(const Problem& P, double min_prob) {
    TapeHead head;
    memset(&head, 0, sizeof(head));
    head.magic = kTapeMagic;
    head.M = P.M;
    head.mask_words = (P.N + 31) / 32;
    head.P = P;
    head.min_prob = min_prob;
    return head;
}

static_assert(kProbThresh == ESACB200_PROB_THRESH, "the C ABI's default floor is the reference's PROB_THRESH");

// The hypotheses node's probability floor: a number in [0, 1] (NaN is refused).  `what`: the entry point, or null.
static int check_min_prob(esacb200_ctx* ctx, const char* what, double min_prob) {
    if (min_prob >= 0.0 && min_prob <= 1.0) return 0;
    return fail(ctx, ESACB200_ERR_ARG, "%s%smin_prob must lie in [0, 1], got %g", what ? what : "", what ? ": " : "", min_prob);
}

// The arguments of the tape's record kernel: the hypotheses of problem P that run_hypotheses left in ctx's workspace.
static BwdArgs tape_record_args(esacb200_ctx* ctx, const Problem& P) {
    BwdArgs b;
    memset(&b, 0, sizeof(b));
    b.assign32 = ctx->assign32.as<int>();
    b.init = ctx->poses.as<Pose>();
    b.ref = ctx->poses_ref.as<Pose>();
    b.cells = ctx->cells.as<int>();
    b.contrib = ctx->contrib.as<int>();
    b.n_contrib = ctx->scalars.as<int>() + S_NCONTRIB;
    b.rounds = ctx->rounds.as<int>();
    b.P = P;
    return b;
}

// The arguments of the upstream backward of the hypotheses forward of problem P whose tape is at `tape`: its image's
// coordinates and gradient tensor, the contributing count at n_contrib, and ctx's backward workspace.
static BwdArgs upstream_args(esacb200_ctx* ctx, const Problem& P, const void* tape, const float* coords, float* grads,
                             const int* n_contrib) {
    BwdArgs b;
    memset(&b, 0, sizeof(b));
    b.coords = coords;
    b.grads = grads;
    b.n_contrib = n_contrib;
    b.job_of = ctx->job_of.as<int>();
    b.masks = (const uint32_t*)((const char*)tape + tape_masks_offset(P.M));
    b.mask_words = (P.N + 31) / 32;
    b.red = ctx->red.as<double>();
    b.hyp_grad = ctx->hypgrad.p;
    b.P = P;
    return b;
}

// The tape of a hypotheses forward of problem P: at least tape_bytes large, 16-byte aligned device memory.
static int check_tape(esacb200_ctx* ctx, const void* tape, size_t bytes, const Problem& P) {
    const size_t need = tape_bytes(P.M, P.N);
    if (bytes < need) return fail(ctx, ESACB200_ERR_ARG, "tape holds %zu bytes, this call needs %zu", bytes, need);
    if (!is_device_ptr(tape) || ((uintptr_t)tape & 15)) return fail(ctx, ESACB200_ERR_ARG, "tape must be 16-byte aligned device memory");
    return 0;
}

// The hypotheses forward of problem P (filled and checked by the caller, with the tape: check_tape, and the floor).
static int hypotheses_forward_impl(esacb200_ctx* ctx, const Problem& P, double min_prob, const float* coords, const int64_t* assign,
                                   int64_t assign_stride, void* tape, double* out_scores, double* out_poses6, uint8_t* out_contrib) {
    Plan pl{P};
    pl.min_prob = min_prob;
    const int M = P.M;
    begin_call(ctx);
    int rc = run_hypotheses(ctx, pl, coords, assign, assign_stride, ShardSteps(), (uint32_t*)((char*)tape + tape_masks_offset(M)));
    if (rc) return rc;
    CK(ctx->contrib8.ensure((size_t)M));
    CK(cudaMemsetAsync((char*)tape + kTapeTailOffset, 0, sizeof(TapeTail), ctx->stream));  // (a bad assignment fails the call)
    launch_tape_records(tape_record_args(ctx, P), tape_head(P, min_prob), tape, ctx->contrib8.as<unsigned char>(), ctx->stream);
    CK(cudaGetLastError());
    ctx->st.kernel_launches += 1;
    CK(cudaMemcpyAsync(out_scores, ctx->scores.p, (size_t)M * 8, cudaMemcpyDefault, ctx->stream));
    CK(cudaMemcpyAsync(out_poses6, ctx->poses_ref.p, (size_t)M * sizeof(Pose), cudaMemcpyDefault, ctx->stream));
    CK(cudaMemcpyAsync(out_contrib, ctx->contrib8.p, (size_t)M, cudaMemcpyDefault, ctx->stream));
    return finish_call(ctx, pl, kSelectStats, true);
}

int esacb200_hypotheses_forward_floor(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                                      int64_t assign_stride, int M, int shiftX, int shiftY, float f, float ppx, float ppy,
                                      float tau, float alpha, float beta, float maxReproj, int sub, double min_prob, void* tape,
                                      size_t tape_bytes_, double* out_scores, double* out_poses6, uint8_t* out_contrib) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !assign || !tape || !out_scores || !out_poses6 || !out_contrib) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    Problem P;
    int rc = check_min_prob(ctx, nullptr, min_prob);
    if (!rc) rc = fill_problem(ctx, P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS_INJECTED);
    if (!rc) rc = check_tape(ctx, tape, tape_bytes_, P);
    return rc ? rc : hypotheses_forward_impl(ctx, P, min_prob, coords, assign, assign_stride, tape, out_scores, out_poses6, out_contrib);
} ESAC_ABI_CATCH(ctx)

int esacb200_hypotheses_forward(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                                int64_t assign_stride, int M, int shiftX, int shiftY, float f, float ppx, float ppy, float tau,
                                float alpha, float beta, float maxReproj, int sub, void* tape, size_t tape_bytes_,
                                double* out_scores, double* out_poses6, uint8_t* out_contrib) {
    return esacb200_hypotheses_forward_floor(ctx, coords, E, H, W, assign, assign_stride, M, shiftX, shiftY, f, ppx, ppy, tau,
                                             alpha, beta, maxReproj, sub, ESACB200_PROB_THRESH, tape, tape_bytes_, out_scores,
                                             out_poses6, out_contrib);
}

// d_scores / d_poses6 are [rows, M] / [rows, M, 6] arrays (M of the tape) of which row `row` is this tape's upstream.
static int hypotheses_backward_impl(esacb200_ctx* ctx, const void* tape, const float* coords, float* grads, int E, int H, int W,
                                    const double* d_scores, const double* d_poses6, int row) {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!tape || !coords || !grads) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    if (!is_device_ptr(tape) || ((uintptr_t)tape & 15)) return fail(ctx, ESACB200_ERR_ARG, "tape must be 16-byte aligned device memory");
    // the header: problem and hypothesis count of the forward (ordered after the forward on this stream)
    TapeHead head;
    CK(cudaMemcpyAsync(&head, tape, sizeof(head), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (head.magic != kTapeMagic) return fail(ctx, ESACB200_ERR_ARG, "tape holds no hypotheses forward");
    const Problem P = head.P;
    if (P.E != E || P.H != H || P.W != W)
        return fail(ctx, ESACB200_ERR_ARG, "coordinates are [%d,3,%d,%d], the forward saw [%d,3,%d,%d]", E, H, W, P.E, P.H, P.W);
    const int M = head.M;
    if (d_scores) d_scores += (size_t)row * M;
    if (d_poses6) d_poses6 += (size_t)row * M * 6;
    begin_call(ctx);
    const size_t cbytes = (size_t)E * 3 * P.N * sizeof(float);
    const float* d_coords = coords;
    if (!is_device_ptr(coords)) {
        CK(ctx->coords.ensure(cbytes));
        CK(cudaMemcpyAsync(ctx->coords.p, coords, cbytes, cudaMemcpyHostToDevice, ctx->stream));
        d_coords = ctx->coords.as<float>();
    }
    float* d_grads = nullptr;
    int rc = stage_grads(ctx, grads, cbytes, d_grads);
    if (rc) return rc;
    // upstream gradients: [M] of the scores then [M,6] of the poses; an absent one is zero
    CK(ctx->upstream.ensure((size_t)M * 7 * 8));
    double* up = ctx->upstream.as<double>();
    if (d_scores) CK(cudaMemcpyAsync(up, d_scores, (size_t)M * 8, cudaMemcpyDefault, ctx->stream));
    else CK(cudaMemsetAsync(up, 0, (size_t)M * 8, ctx->stream));
    if (d_poses6) CK(cudaMemcpyAsync(up + M, d_poses6, (size_t)M * 6 * 8, cudaMemcpyDefault, ctx->stream));
    else CK(cudaMemsetAsync(up + M, 0, (size_t)M * 6 * 8, ctx->stream));
    mark(ctx, EV_REFINE);
    rc = backward_buffers(ctx, P, false, grow(ctx));
    if (rc) return rc;
    const BwdArgs b =
        upstream_args(ctx, P, tape, d_coords, d_grads, (const int*)((const char*)tape + offsetof(TapeHead, n_contrib)));
    launch_backward_upstream(b, tape, up, up + M, M, ctx->sm_count, ctx->stream);
    CK(cudaGetLastError());
    ctx->st.kernel_launches += 5;
    mark(ctx, EV_BWD);
    if (d_grads != grads) CK(cudaMemcpyAsync(grads, d_grads, cbytes, cudaMemcpyDeviceToHost, ctx->stream));
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    ctx->st.M = M;
    ctx->st.n_contrib = head.n_contrib;
    finish_stats(ctx);
    return ESACB200_OK;
}

int esacb200_hypotheses_backward(esacb200_ctx* ctx, const void* tape, const float* coords, float* grads, int E, int H, int W,
                                 const double* d_scores, const double* d_poses6) try {
    return hypotheses_backward_impl(ctx, tape, coords, grads, E, H, W, d_scores, d_poses6, 0);
} ESAC_ABI_CATCH(ctx)

int esacb200_pose_loss_batch(esacb200_ctx* ctx, int B, int M, const double* poses6, const float* gt16, float wRot, float wTrans,
                             float cut, double* out_losses, double* out_dloss6) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!poses6 || !gt16 || !out_losses || !out_dloss6) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    if (M <= 0) return fail(ctx, ESACB200_ERR_ARG, "no poses (M=%d)", M);
    if (B <= 0 || B > 65535) return fail(ctx, ESACB200_ERR_ARG, "batch of %d images outside [1, 65535]", B);
    begin_call(ctx);
    const size_t n = (size_t)B * M;
    // [B,M] poses, [B,M] losses, [B,M,6] dLoss; the ground truths [B,4,4] in their own buffer
    CK(ctx->upstream.ensure(n * 13 * 8));
    CK(ctx->gt.ensure((size_t)B * 16 * sizeof(float)));
    double* buf = ctx->upstream.as<double>();
    CK(cudaMemcpyAsync(buf, poses6, n * sizeof(Pose), cudaMemcpyDefault, ctx->stream));
    CK(cudaMemcpyAsync(ctx->gt.p, gt16, (size_t)B * 16 * sizeof(float), cudaMemcpyDefault, ctx->stream));
    launch_pose_loss((const Pose*)buf, B, M, ctx->gt.as<float>(), wRot, wTrans, cut, buf + 6 * n, buf + 7 * n, ctx->stream);
    CK(cudaGetLastError());
    ctx->st.kernel_launches += 1;
    CK(cudaMemcpyAsync(out_losses, buf + 6 * n, n * 8, cudaMemcpyDefault, ctx->stream));
    CK(cudaMemcpyAsync(out_dloss6, buf + 7 * n, n * 6 * 8, cudaMemcpyDefault, ctx->stream));
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_pose_loss(esacb200_ctx* ctx, int M, const double* poses6, const float* gt16, float wRot, float wTrans, float cut,
                       double* out_losses, double* out_dloss6) {
    return esacb200_pose_loss_batch(ctx, 1, M, poses6, gt16, wRot, wTrans, cut, out_losses, out_dloss6);
}

// -------------------------------------------------------------------------------------------------
// The hypotheses node with the forward_async contract (esacb200_hypotheses_forward_async / _backward_async): the host path is
// the eager one, in the stream-ordered context, with the refinement group picked on the device; the record kernel writes the
// header from device-read values and the caller's outputs, and the backward checks the header on the device.  It uses the
// workspace of backward_async and its rule.

// Bytes between consecutive images' tapes: the tape rounded up to 256 bytes.
static size_t tape_stride(const Problem& P) { return (tape_bytes(P.M, P.N) + 255) & ~(size_t)255; }

// The tapes argument of B images: 16-byte aligned device memory of at least B strides.
static int check_tapes(esacb200_ctx* ctx, const char* what, const void* tapes, size_t bytes, int B, const Problem& P) {
    const size_t need = (size_t)B * tape_stride(P);
    if (bytes < need)
        return fail(ctx, ESACB200_ERR_ARG, "%s: tapes hold %zu bytes, %d image(s) of E=%d H=%d W=%d M=%d need %zu", what, bytes, B,
                    P.E, P.H, P.W, P.M, need);
    if ((uintptr_t)tapes & 15) return fail(ctx, ESACB200_ERR_ARG, "%s: tapes must be 16-byte aligned", what);
    return 0;
}

int esacb200_hypotheses_forward_async_floor(esacb200_ctx* ctx, int B, const float* coords, int E, int H, int W,
                                            const int64_t* assign, int64_t assign_stride, int M, const int32_t* shifts,
                                            const float* cameras, float tau, float alpha, float beta, float maxReproj, int sub,
                                            double min_prob, void* tapes, size_t tapes_bytes, double* out_scores,
                                            double* out_poses6, uint8_t* out_contrib, int32_t* out_status) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "hypotheses_forward_async";
    const void* ptrs[] = {coords, assign, shifts, cameras, tapes, out_scores, out_poses6, out_contrib, out_status};
    const char* names[] = {"coords", "assign", "shifts", "cameras", "tapes", "out_scores", "out_poses6", "out_contrib", "out_status"};
    AsyncCall call;
    Problem P;
    int rc = B <= 0 ? fail(ctx, ESACB200_ERR_ARG, "%s: empty batch (B=%d)", what, B) : check_min_prob(ctx, what, min_prob);
    if (!rc) rc = fill_problem(ctx, P, E, H, W, M, 0, 0, 0.f, 0.f, 0.f, tau, alpha, beta, maxReproj, sub, DRAWS);
    if (!rc) rc = check_tapes(ctx, what, tapes, tapes_bytes, B, P);
    if (!rc) rc = begin_async(ctx, true, B, P, coords, assign, assign_stride, shifts, cameras, out_status, 9, ptrs, names, call, what);
    if (rc) return rc;
    esacb200_ctx* a = call.a;
    const size_t stride = tape_stride(P);
    for (int b = 0; b < B; ++b) {
        Plan& pl = call.plans[b];
        const AsyncImage& im = call.imgs[b];
        char* tape = (char*)tapes + (size_t)b * stride;
        pl.min_prob = min_prob;  // a kernel parameter: a captured graph replays with the floor it was captured with
        rc = run_hypotheses(a, pl, pl.d_coords, (const int64_t*)pl.d_assign, assign_stride, ShardSteps(),
                            (uint32_t*)(tape + tape_masks_offset(M)));
        if (rc) return fail(ctx, rc, "image %d: %s", b, a->err);
        TapeDev td;
        td.dev = im.dev;
        td.flags = a->scalars.as<int>() + S_FLAGS;
        td.scores = a->scores.as<double>();
        td.poses = a->poses_ref.as<Pose>();
        td.out_scores = out_scores + (size_t)b * M;
        td.out_poses6 = out_poses6 + (size_t)b * M * 6;
        td.status = im.status;
        td.seed = a->seed_state.as<unsigned long long>();
        td.advance = im.advance;
        launch_tape_records_async(tape_record_args(a, P), tape_head(P, min_prob), tape, out_contrib + (size_t)b * M, td, a->stream);
        a->st.kernel_launches += 1;
    }
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_hypotheses_forward_async(esacb200_ctx* ctx, int B, const float* coords, int E, int H, int W, const int64_t* assign,
                                      int64_t assign_stride, int M, const int32_t* shifts, const float* cameras, float tau,
                                      float alpha, float beta, float maxReproj, int sub, void* tapes, size_t tapes_bytes,
                                      double* out_scores, double* out_poses6, uint8_t* out_contrib, int32_t* out_status) {
    return esacb200_hypotheses_forward_async_floor(ctx, B, coords, E, H, W, assign, assign_stride, M, shifts, cameras, tau, alpha,
                                                   beta, maxReproj, sub, ESACB200_PROB_THRESH, tapes, tapes_bytes, out_scores,
                                                   out_poses6, out_contrib, out_status);
}

int esacb200_hypotheses_backward_async(esacb200_ctx* ctx, int B, const void* tapes, size_t tapes_bytes, const float* coords,
                                       float* grads, int E, int H, int W, int M, const double* d_scores, const double* d_poses6,
                                       int32_t* out_status) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = "hypotheses_backward_async";
    if (B <= 0) return fail(ctx, ESACB200_ERR_ARG, "%s: empty batch (B=%d)", what, B);
    const void* ptrs[] = {tapes, coords, grads, out_status, d_scores, d_poses6};
    const char* names[] = {"tapes", "coords", "grads", "out_status", "d_scores", "d_poses6"};
    int rc = device_args(ctx, what, 6, ptrs, names, 0x30u);  // an absent upstream is zero
    if (rc) return rc;
    Problem P;
    // sub, tau, alpha, beta and maxReproj are the forward's, read from the tape header on the device (BwdDev::prob)
    rc = fill_problem(ctx, P, E, H, W, M, 0, 0, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 1, NO_DRAW);
    if (!rc) rc = check_tapes(ctx, what, tapes, tapes_bytes, B, P);
    esacb200_ctx* a = nullptr;
    if (!rc) rc = enter_async(ctx, P, true, what, &a);
    if (rc) return rc;
    int* sc = a->scalars.as<int>();
    const size_t cstride = (size_t)E * 3 * P.N, stride = tape_stride(P);
    for (int b = 0; b < B; ++b) {
        const char* tape = (const char*)tapes + (size_t)b * stride;
        const BwdArgs args = upstream_args(a, P, tape, coords + (size_t)b * cstride, grads + (size_t)b * cstride, sc + S_NCONTRIB);
        const Problem* hp = (const Problem*)(tape + offsetof(TapeHead, P));
        BwdDev dv;
        dv.flags = sc + S_FLAGS;
        dv.dev.shift = &hp->shiftX;
        dv.dev.cam = &hp->f;
        dv.prob = hp;
        launch_backward_upstream_async(args, tape, d_scores ? d_scores + (size_t)b * M : nullptr,
                                       d_poses6 ? d_poses6 + (size_t)b * M * 6 : nullptr, sc + S_NCONTRIB, sc + S_FLAGS,
                                       out_status + b, dv, M, a->sm_count, a->stream);
        a->st.kernel_launches += 5;
    }
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_pose_loss_async(esacb200_ctx* ctx, int B, int M, const double* poses6, const float* gt16, float wRot, float wTrans,
                             float cut, double* out_losses, double* out_dloss6) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const void* ptrs[] = {poses6, gt16, out_losses, out_dloss6};
    const char* names[] = {"poses6", "gt16", "out_losses", "out_dloss6"};
    const int rc = device_args(ctx, "pose_loss_async", 4, ptrs, names);
    if (rc) return rc;
    if (M <= 0) return fail(ctx, ESACB200_ERR_ARG, "pose_loss_async: no poses (M=%d)", M);
    if (B <= 0 || B > 65535) return fail(ctx, ESACB200_ERR_ARG, "pose_loss_async: batch of %d images outside [1, 65535]", B);
    launch_pose_loss((const Pose*)poses6, B, M, gt16, wRot, wTrans, cut, out_losses, out_dloss6, ctx->stream);
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// The hypotheses node over a batch, on the worker contexts of run_batch: image b runs the single-image forward / backward
// with row b of the [B,M] outputs / upstreams.
int esacb200_hypotheses_forward_ragged_floor(esacb200_ctx* ctx, int B, const float* const* coords, const int* H, const int* W,
                                             int E, const int64_t* assign, int64_t assign_stride, int M, const int* shiftX,
                                             const int* shiftY, const float* f, const float* ppx, const float* ppy, float tau,
                                             float alpha, float beta, float maxReproj, int sub, double min_prob,
                                             void* const* tapes, const size_t* tape_bytes_, double* out_scores,
                                             double* out_poses6, uint8_t* out_contrib) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !H || !W || !assign || !tapes || !tape_bytes_ || !out_scores || !out_poses6 || !out_contrib || B <= 0)
        return fail(ctx, ESACB200_ERR_ARG, "null pointer argument or empty batch");
    if (check_min_prob(ctx, nullptr, min_prob)) return ESACB200_ERR_ARG;
    if (!f || !ppx || !ppy) return fail(ctx, ESACB200_ERR_ARG, "null camera array");
    if (ctx->inj_M) return fail(ctx, ESACB200_ERR_ARG, "injected cells are a single-image test hook");
    if (E <= 0 || M <= 0) return fail(ctx, ESACB200_ERR_ARG, "bad sizes E=%d M=%d", E, M);
    std::vector<Plan> plans;
    int rc = fill_problems(ctx, plans, B, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS);
    if (rc) return rc;
    bool dev_c = false;
    rc = pointer_kind(ctx, (const void* const*)coords, B, "coords", dev_c);
    if (rc) return rc;
    for (int b = 0; b < B; ++b) {
        if (!tapes[b]) return fail(ctx, ESACB200_ERR_ARG, "image %d: tape is null", b);
        if (check_tape(ctx, tapes[b], tape_bytes_[b], plans[b].P))
            return fail(ctx, ESACB200_ERR_ARG, "image %d: %s", b, std::string(ctx->err).c_str());
    }
    const int64_t arow = assign_stride == 0 ? 0 : (int64_t)M * assign_stride;
    rc = run_batch(ctx, B, H, W, true, [&](esacb200_ctx* w, int b) {
        return hypotheses_forward_impl(w, plans[b].P, min_prob, coords[b], assign + (size_t)b * arow, assign_stride, tapes[b],
                                       out_scores + (size_t)b * M, out_poses6 + (size_t)b * M * 6, out_contrib + (size_t)b * M);
    });
    return rc ? rc : ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_hypotheses_forward_ragged(esacb200_ctx* ctx, int B, const float* const* coords, const int* H, const int* W, int E,
                                       const int64_t* assign, int64_t assign_stride, int M, const int* shiftX, const int* shiftY,
                                       const float* f, const float* ppx, const float* ppy, float tau, float alpha, float beta,
                                       float maxReproj, int sub, void* const* tapes, const size_t* tape_bytes_,
                                       double* out_scores, double* out_poses6, uint8_t* out_contrib) {
    return esacb200_hypotheses_forward_ragged_floor(ctx, B, coords, H, W, E, assign, assign_stride, M, shiftX, shiftY, f, ppx, ppy,
                                                    tau, alpha, beta, maxReproj, sub, ESACB200_PROB_THRESH, tapes, tape_bytes_,
                                                    out_scores, out_poses6, out_contrib);
}

int esacb200_hypotheses_backward_ragged(esacb200_ctx* ctx, int B, const void* const* tapes, const float* const* coords,
                                        float* const* grads, const int* H, const int* W, int E, const double* d_scores,
                                        const double* d_poses6) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!tapes || !coords || !grads || !H || !W || B <= 0) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument or empty batch");
    if (ctx->inj_M) return fail(ctx, ESACB200_ERR_ARG, "injected cells are a single-image test hook");
    if (E <= 0) return fail(ctx, ESACB200_ERR_ARG, "bad size E=%d", E);
    std::vector<Plan> sizes;  // the maps' sizes, checked as those of a forward of one hypothesis (the tapes hold M)
    int rc = fill_problems(ctx, sizes, B, E, H, W, 1, nullptr, nullptr, nullptr, nullptr, nullptr, 0.f, 0.f, 0.f, 0.f, 1, DRAWS);
    if (rc) return rc;
    bool dev_c = false, dev_g = false, dev_t = false;
    rc = pointer_kind(ctx, (const void* const*)coords, B, "coords", dev_c);
    if (rc) return rc;
    rc = pointer_kind(ctx, (const void* const*)grads, B, "grads", dev_g);
    if (rc) return rc;
    rc = pointer_kind(ctx, tapes, B, "tape", dev_t);
    if (rc) return rc;
    rc = run_batch(ctx, B, H, W, false, [&](esacb200_ctx* w, int b) {
        return hypotheses_backward_impl(w, tapes[b], coords[b], grads[b], E, H[b], W[b], d_scores, d_poses6, b);
    });
    return rc ? rc : ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

}  // extern "C"
