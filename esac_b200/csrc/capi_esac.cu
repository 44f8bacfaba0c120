// esac.forward and esac.backward in the C ABI of include/esac_b200.h: single image, sharded, batched, ragged and
// stream-ordered, plus scoring and refining given poses.
//
// Orchestration follows esac_forward (esac.cpp:64-190) and esac_backward (esac.cpp:213-511) stage by
// stage; every stage is a CUDA kernel launched on one stream with no host round trip until the final
// 68-byte (forward) / 8-byte (backward) result copy.
#include <cuda_runtime.h>
#include <string.h>

#include <vector>

#include "capi_internal.h"

using namespace esacb200;
using namespace esacb200::capi;

// sample -> score -> select -> refine(winner) -> the forward record (rank aside) into d_rec; no sync.
// A stream-ordered image (pl.async) takes its seed from device memory and writes the caller's arrays instead.
static int enqueue_forward_core(esacb200_ctx* ctx, const Plan& pl, ForwardRecord* d_rec) {
    const Problem& P = pl.P;
    int* sc = ctx->scalars.as<int>();
    const uint64_t seed = pl.async ? 0 : call_seed(ctx);
    int rc = run_sample(ctx, pl, seed);
    if (rc) return rc;
    rc = run_score(ctx, pl);
    if (rc) return rc;
    const int group = pick_group(ctx, P, 1);
    rc = run_refine(ctx, pl, ctx->poses.as<Pose>(), ctx->poses_ref.as<Pose>(), sc + S_WINNER, nullptr, 1, 1, group);
    if (rc) return rc;
    mark(ctx, EV_REFINE);
    if (pl.async)
        launch_finish_forward_async(ctx->poses_ref.as<Pose>(), sc + S_WINNER, ctx->assign32.as<int>(), sc + S_FLAGS, pl.async->pose,
                                    pl.async->expert, pl.async->status, ctx->seed_state.as<unsigned long long>(), pl.async->advance,
                                    ctx->stream);
    else
        launch_finish_forward(ctx->poses_ref.as<Pose>(), sc + S_WINNER, ctx->assign32.as<int>(), sc + S_FLAGS, d_rec, ctx->stream);
    ctx->st.kernel_launches += 1;
    return 0;
}

// The pinned host copy of the per-expert flags of hypothesis-major sharding (for_flagged_planes), for E experts.
static int ensure_host_flags(esacb200_ctx* ctx, int E) {
    if (ctx->h_flags_cap >= E + 1) return 0;
    if (ctx->h_flags) cudaFreeHost(ctx->h_flags);
    ctx->h_flags = nullptr; ctx->h_flags_cap = 0;
    CK(cudaMallocHost((void**)&ctx->h_flags, (size_t)(E + 1) * sizeof(int)));
    ctx->h_flags_cap = E + 1;
    return 0;
}

extern "C" {

// -------------------------------------------------------------------------------------------------
int esacb200_forward(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                     int64_t assign_stride, int M, float* out_pose, int shiftX, int shiftY, float f, float ppx,
                     float ppy, float tau, float alpha, float beta, float maxReproj, int sub, int* out_expert) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !assign || !out_pose) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    Plan pl;
    int rc = fill_problem(ctx, pl.P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS_INJECTED);
    if (rc) return rc;
    begin_call(ctx);
    rc = stage_inputs(ctx, pl, coords, assign, assign_stride, /*allow_split=*/!ctx->inj_M);
    if (rc) return rc;
    rc = enqueue_forward_core(ctx, pl, ctx->fwd_rec.as<ForwardRecord>());
    if (rc) return rc;
    Pinned& h = *ctx->pin;
    CK(cudaMemcpyAsync(&h.fwd, ctx->fwd_rec.p, offsetof(ForwardRecord, bad), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(h.rounds, ctx->rounds.p, sizeof(h.rounds), cudaMemcpyDeviceToHost, ctx->stream));
    if (is_device_ptr(out_pose)) CK(cudaMemcpyAsync(out_pose, ctx->fwd_rec.p, sizeof(h.fwd.pose), cudaMemcpyDeviceToDevice, ctx->stream));
    rc = finish_call(ctx, pl, kSelectStats, true);
    if (rc) return rc;
    if (!is_device_ptr(out_pose)) memcpy(out_pose, h.fwd.pose, sizeof(h.fwd.pose));
    if (out_expert) *out_expert = (int)h.fwd.expert;
    ctx->st.refine_rounds = h.rounds[0];
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
// Local half of a sharded forward: pipeline + record, no synchronisation (shared by forward_pack and forward_sharded).  The
// call begins (begin_record) before the shard's problem is filled, so bad sizes still clear the stats and the last-call
// record; M = 0 is a shard without hypotheses, whose problem is neither filled nor read.
static int begin_record(esacb200_ctx* ctx, int M, int M_pad) {
    if (M_pad < M || M_pad < 1) return fail(ctx, ESACB200_ERR_ARG, "M_pad (%d) must be >= M (%d) and >= 1", M_pad, M);
    begin_call(ctx);
    ctx->inj_M = ctx->inj_T = 0;
    return 0;
}

static int enqueue_forward_record(esacb200_ctx* ctx, const Problem& P, const float* coords, const int64_t* assign,
                                  int64_t assign_stride, int M, int M_pad, int expert_offset, double* pack_out) {
    Plan pl{P};
    if (M > 0) {
        int rc = stage_inputs(ctx, pl, coords, assign, assign_stride);
        if (rc) return rc;
        rc = enqueue_forward_core(ctx, pl, ctx->fwd_rec.as<ForwardRecord>());
        if (rc) return rc;
    } else {
        CK(ctx->scores.ensure(8));
        CK(ctx->fwd_rec.ensure(sizeof(ForwardRecord)));
    }
    launch_pack_forward(ctx->scores.as<double>(), ctx->fwd_rec.as<ForwardRecord>(), M, M_pad, expert_offset, ctx->opt.hyp_offset,
                        ctx->opt.hyp_stride, pack_out, ctx->stream);
    CK(cudaGetLastError());
    ctx->st.kernel_launches += 1;
    ctx->st.M = M;
    if (M > 0) record_draw(ctx, pl, false);
    return ESACB200_OK;
}

int esacb200_forward_pack(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                          int64_t assign_stride, int M, int M_pad, int shiftX, int shiftY, float f, float ppx, float ppy, float tau,
                          float alpha, float beta, float maxReproj, int sub, int expert_offset, double* pack_out) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!pack_out || (M > 0 && (!coords || !assign))) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    if ((M > 0 && (!is_device_ptr(coords) || !is_device_ptr(assign))) || !is_device_ptr(pack_out))
        return fail(ctx, ESACB200_ERR_ARG, "forward_pack takes device pointers only");
    Problem P = {};
    int rc = begin_record(ctx, M, M_pad);
    if (!rc && M > 0) rc = fill_problem(ctx, P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS);
    if (!rc) rc = enqueue_forward_record(ctx, P, coords, assign, assign_stride, M, M_pad, expert_offset, pack_out);
    if (rc) return rc;
    mark(ctx, EV_END);
    return ESACB200_OK;   // stage timers of this call are not collected: that would need the synchronisation
} ESAC_ABI_CATCH(ctx)

// ---- communicator -----------------------------------------------------------------------------------
int esacb200_nccl_unique_id(void* out128) {
    if (!out128) return ESACB200_ERR_ARG;
    NcclApi& n = nccl_api();
    if (!n.ok) return ESACB200_ERR_NO_DEVICE;
    NcclApi::UniqueId id;
    if (n.GetUniqueId(&id) != 0) return ESACB200_ERR_CUDA;
    memcpy(out128, id.internal, 128);
    return ESACB200_OK;
}

int esacb200_comm_init(esacb200_ctx* ctx, int world, int rank, const void* id128) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!id128 || world < 1 || rank < 0 || rank >= world) return fail(ctx, ESACB200_ERR_ARG, "bad communicator arguments");
    NcclApi& n = nccl_api();
    if (!n.ok) return fail(ctx, ESACB200_ERR_NO_DEVICE, "libnccl.so.2 cannot be loaded");
    if (ctx->nccl_comm) { n.CommDestroy(ctx->nccl_comm); ctx->nccl_comm = nullptr; }
    NcclApi::UniqueId id;
    memcpy(id.internal, id128, 128);
    CKN(n.CommInitRank(&ctx->nccl_comm, world, id, rank));
    ctx->comm_world = world;
    ctx->comm_rank = rank;
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_comm_destroy(esacb200_ctx* ctx) {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (ctx->nccl_comm) {
        cudaStreamSynchronize(ctx->stream);
        nccl_api().CommDestroy(ctx->nccl_comm);
        ctx->nccl_comm = nullptr;
    }
    ctx->comm_world = 1;
    ctx->comm_rank = 0;
    return ESACB200_OK;
}

// esac_forward with the experts / hypotheses sharded over the ranks of the communicator (SURVEY 8e): local pipeline ->
// record -> ONE ncclAllGather on the context's stream -> softMax / draw over all records on the device -> one 80-byte
// read-back.  Every rank returns the global winner's pose and expert.  M may be 0 (a shard without hypotheses); M_pad is
// the largest M of any rank (records must have one size).
int esacb200_forward_sharded(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                             int64_t assign_stride, int M, int M_pad, float* out_pose, int shiftX, int shiftY, float f, float ppx,
                             float ppy, float tau, float alpha, float beta, float maxReproj, int sub, int expert_offset,
                             int* out_expert) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!ctx->nccl_comm) return fail(ctx, ESACB200_ERR_ARG, "no communicator: call esacb200_comm_init first");
    if (!out_pose || (M > 0 && (!coords || !assign))) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    const int world = ctx->comm_world;
    const size_t rec = (size_t)M_pad + kPackTail;
    CK(ctx->gathered.ensure((world + 1) * rec * 8));
    double* mine = ctx->gathered.as<double>() + (size_t)world * rec;
    Problem P = {};
    int rc = begin_record(ctx, M, M_pad);
    if (!rc && M > 0) rc = fill_problem(ctx, P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS);
    if (!rc) rc = enqueue_forward_record(ctx, P, coords, assign, assign_stride, M, M_pad, expert_offset, mine);
    if (rc) return rc;
    CKN(nccl_api().AllGather(mine, ctx->gathered.p, rec, kNcclFloat64, ctx->nccl_comm, ctx->stream));
    launch_select_gathered(ctx->gathered.as<double>(), world, M_pad, ctx->fwd_rec.as<ForwardRecord>(), ctx->stream);
    CK(cudaGetLastError());
    ctx->st.kernel_launches += 2;
    Pinned& h = *ctx->pin;
    CK(cudaMemcpyAsync(&h.fwd, ctx->fwd_rec.p, sizeof(ForwardRecord), cudaMemcpyDeviceToHost, ctx->stream));
    if (is_device_ptr(out_pose)) CK(cudaMemcpyAsync(out_pose, ctx->fwd_rec.p, sizeof(h.fwd.pose), cudaMemcpyDeviceToDevice, ctx->stream));
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    // every rank selects from the same records, so every rank refuses alike (esac.forward refuses M = 0 as well)
    if (h.fwd.winner < 0.f) return fail(ctx, ESACB200_ERR_ARG, "no shard holds a hypothesis: hypAssignment is empty on every rank");
    if (h.fwd.bad != 0.f) return fail(ctx, ESACB200_ERR_ARG, "a shard's hypAssignment holds an expert index outside its experts");
    if (!is_device_ptr(out_pose)) memcpy(out_pose, h.fwd.pose, sizeof(h.fwd.pose));
    if (out_expert) *out_expert = (int)h.fwd.expert;
    ctx->st.winner = (int)h.fwd.winner;
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
// esac_forward over a batch of B images (BASELINE configs[2]: "batch 8 images").  The reference has no such entry: its
// callers loop over a DataLoader with batch_size=1 (test_esac.py:137).  Images are processed back to back on the compute
// stream with ONE host synchronisation at the end; host coordinate maps are double-buffered and copied on a second stream
// so the copy of image b+1 overlaps the kernels of image b.  Image b runs with its own map size, shift and camera: the
// pipeline of one image reads them from its Problem, so only the loop below sees the arrays.  The workspace is sized for
// the largest image before the first one is enqueued.
int esacb200_forward_ragged(esacb200_ctx* ctx, int B, const float* const* coords, const int* H, const int* W, int E,
                            const int64_t* assign, int64_t assign_stride, int M, float* out_poses, const int* shiftX,
                            const int* shiftY, const float* f, const float* ppx, const float* ppy, float tau, float alpha,
                            float beta, float maxReproj, int sub, int* out_experts) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !H || !W || !assign || !out_poses || B <= 0) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument or empty batch");
    if (!f || !ppx || !ppy) return fail(ctx, ESACB200_ERR_ARG, "null camera array");
    std::vector<Plan> plans;
    int rc = fill_problems(ctx, plans, B, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS);
    if (rc) return rc;
    bool dev_coords = false;
    rc = pointer_kind(ctx, (const void* const*)coords, B, "coords", dev_coords);
    if (rc) return rc;
    const bool host_coords = !dev_coords;
    begin_call(ctx);
    ctx->inj_M = ctx->inj_T = 0;
    rc = reserve_forward_batch(ctx, plans, host_coords);
    if (rc) return rc;
    // element stride between the assignments of consecutive images: rows of a [B, M] tensor
    const int64_t arow = assign_stride == 0 ? 0 : (int64_t)M * assign_stride;
    CK(ctx->out_batch.ensure((size_t)B * sizeof(ForwardRecord)));
    DevBuf* cb[2] = {&ctx->coords, &ctx->coords_alt};
    DevBuf* ab[2] = {&ctx->assign64, &ctx->assign64_alt};
    for (int b = 0; b < B; ++b) {
        const int buf = b & 1;
        Plan& pl = plans[b];
        if (host_coords && b >= 2) CK(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_consumed[buf], 0));
        rc = upload_inputs(ctx, pl, coords[b], assign + (size_t)b * arow, assign_stride, *cb[buf], *ab[buf],
                           host_coords ? ctx->copy_stream : ctx->stream);
        if (rc) return rc;
        if (host_coords) {
            CK(cudaEventRecord(ctx->ev_copied[buf], ctx->copy_stream));
            CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_copied[buf], 0));
        }
        if (b == 0) mark(ctx, EV_H2D);
        rc = plan_and_prep(ctx, pl);
        if (rc) return rc;
        rc = enqueue_forward_core(ctx, pl, ctx->out_batch.as<ForwardRecord>() + b);
        if (rc) return rc;
        if (host_coords) CK(cudaEventRecord(ctx->ev_consumed[buf], ctx->stream));
    }
    std::vector<ForwardRecord> host((size_t)B);
    CK(cudaMemcpyAsync(host.data(), ctx->out_batch.p, host.size() * sizeof(ForwardRecord), cudaMemcpyDeviceToHost, ctx->stream));
    const bool dev_out = is_device_ptr(out_poses);
    const size_t pose_bytes = sizeof(ForwardRecord::pose);
    if (dev_out)
        CK(cudaMemcpy2DAsync(out_poses, pose_bytes, ctx->out_batch.p, sizeof(ForwardRecord), pose_bytes, B, cudaMemcpyDeviceToDevice,
                             ctx->stream));
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    for (int b = 0; b < B; ++b) {
        const ForwardRecord& o = host[b];
        if (o.bad != 0.f) return fail(ctx, ESACB200_ERR_ARG, "image %d: hypAssignment holds an expert index outside [0, %d)", b, E);
        if (!dev_out) memcpy(out_poses + (size_t)b * 16, o.pose, pose_bytes);
        if (out_experts) out_experts[b] = (int)o.expert;
    }
    ctx->st.M = M;
    ctx->st.winner = (int)host[B - 1].winner;
    record_draw(ctx, plans[B - 1], false);  // the buffers hold the last image's hypotheses
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// B images of one shape: the pointer and size arrays of a [B,E,3,H,W] tensor.
int esacb200_forward_batch_cameras(esacb200_ctx* ctx, int B, const float* coords, int E, int H, int W, const int64_t* assign,
                                   int64_t assign_stride, int M, float* out_poses, const int* shiftX, const int* shiftY,
                                   const float* f, const float* ppx, const float* ppy, float tau, float alpha, float beta,
                                   float maxReproj, int sub, int* out_experts) try {
    if (!ctx) return ESACB200_ERR_ARG;
    if (!coords || !assign || !out_poses || B <= 0) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument or empty batch");
    if (!f || !ppx || !ppy) return fail(ctx, ESACB200_ERR_ARG, "null camera array");
    const auto ptrs = slices(coords, B, (size_t)E * 3 * H * W);  // (sizes are checked image by image by the ragged call)
    const std::vector<int> hs((size_t)B, H), ws((size_t)B, W);
    return esacb200_forward_ragged(ctx, B, ptrs.data(), hs.data(), ws.data(), E, assign, assign_stride, M, out_poses, shiftX, shiftY,
                                   f, ppx, ppy, tau, alpha, beta, maxReproj, sub, out_experts);
} ESAC_ABI_CATCH(ctx)

// One camera for the whole batch: broadcast to B entries.
int esacb200_forward_batch(esacb200_ctx* ctx, int B, const float* coords, int E, int H, int W, const int64_t* assign,
                           int64_t assign_stride, int M, float* out_poses, int shiftX, int shiftY, float f, float ppx,
                           float ppy, float tau, float alpha, float beta, float maxReproj, int sub, int* out_experts) try {
    if (!ctx) return ESACB200_ERR_ARG;
    const size_t n = B > 0 ? (size_t)B : 1;  // B <= 0 is rejected by the call below, with its usual message
    const std::vector<int> sx(n, shiftX), sy(n, shiftY);
    const std::vector<float> fs(n, f), cx(n, ppx), cy(n, ppy);
    return esacb200_forward_batch_cameras(ctx, B, coords, E, H, W, assign, assign_stride, M, out_poses, sx.data(), sy.data(),
                                          fs.data(), cx.data(), cy.data(), tau, alpha, beta, maxReproj, sub, out_experts);
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
// Stream-ordered forward.  The pipeline is enqueue_forward_core's, run in the context ctx->async with every image's seed,
// shift and camera read from device memory (AsyncImage), so a CUDA graph that captured the call replays with the values the
// arrays hold at replay time.  Nothing here synchronises, reads back or queries an event, and a call that a capture records
// allocates nothing.

// reserve_forward_async / reserve_backward_async (`backward`): sizes the async workspace for B images of one shape.
static int reserve_async(esacb200_ctx* ctx, int B, int E, int H, int W, int M, int sub, bool backward) {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const char* what = backward ? "backward_async" : "forward_async";
    if (B <= 0) return fail(ctx, ESACB200_ERR_ARG, "reserve_%s: empty batch (B=%d)", what, B);
    std::vector<Plan> plans(1);
    int rc = fill_problem(ctx, plans[0].P, E, H, W, M, 0, 0, 1.f, 0.f, 0.f, 1.f, 1.f, 1.f, 1.f, sub, NO_DRAW);
    if (rc) return rc;
    plans[0].d_coords = nullptr;  // the load path does not change the workspace
    esacb200_ctx* a = nullptr;
    if ((rc = reserve_context(ctx, what, &a))) return rc;
    return async_workspace(ctx, a, plans, false, backward);
}

int esacb200_reserve_forward_async(esacb200_ctx* ctx, int B, int E, int H, int W, int M, int sub) try {
    return reserve_async(ctx, B, E, H, W, M, sub, false);
} ESAC_ABI_CATCH(ctx)

int esacb200_forward_async(esacb200_ctx* ctx, int B, const float* coords, int E, int H, int W, const int64_t* assign,
                           int64_t assign_stride, int M, const int32_t* shifts, const float* cameras, float tau, float alpha,
                           float beta, float maxReproj, int sub, float* out_poses, int64_t* out_experts, int32_t* out_status) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const void* ptrs[] = {coords, assign, shifts, cameras, out_poses, out_experts, out_status};
    const char* names[] = {"coords", "assign", "shifts", "cameras", "out_poses", "out_experts", "out_status"};
    AsyncCall call;
    Problem P;
    int rc = B <= 0 ? fail(ctx, ESACB200_ERR_ARG, "forward_async: empty batch (B=%d)", B)
                    : fill_problem(ctx, P, E, H, W, M, 0, 0, 0.f, 0.f, 0.f, tau, alpha, beta, maxReproj, sub, DRAWS);
    if (!rc) rc = begin_async(ctx, false, B, P, coords, assign, assign_stride, shifts, cameras, out_status, 7, ptrs, names, call);
    if (rc) return rc;
    for (int b = 0; b < B; ++b) {
        call.imgs[b].pose = out_poses + 16 * (size_t)b;
        call.imgs[b].expert = (long long*)out_experts + b;
        rc = plan_and_prep(call.a, call.plans[b]);
        if (!rc) rc = enqueue_forward_core(call.a, call.plans[b], nullptr);
        if (rc) return fail(ctx, rc, "image %d: %s", b, call.a->err);
    }
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
int esacb200_score_poses(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                         int64_t assign_stride, int M, const double* poses6, int shiftX, int shiftY, float f, float ppx,
                         float ppy, float tau, float alpha, float beta, float maxReproj, int sub, double* out_scores) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !assign || !poses6 || !out_scores) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    Plan pl;
    int rc = fill_problem(ctx, pl.P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, NO_DRAW);
    if (rc) return rc;
    begin_call(ctx);
    rc = stage_inputs(ctx, pl, coords, assign, assign_stride);
    if (rc) return rc;
    CK(cudaMemcpyAsync(ctx->poses.p, poses6, (size_t)M * sizeof(Pose), cudaMemcpyHostToDevice, ctx->stream));
    mark(ctx, EV_SAMPLE);
    rc = run_score(ctx, pl);
    if (rc) return rc;
    CK(cudaMemcpyAsync(out_scores, ctx->scores.p, (size_t)M * 8, cudaMemcpyDeviceToHost, ctx->stream));
    return finish_call(ctx, pl, kNoStats, false);
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
int esacb200_refine_poses(esacb200_ctx* ctx, const float* coords, int E, int H, int W, const int64_t* assign,
                          int64_t assign_stride, int M, double* poses6, int shiftX, int shiftY, float f, float ppx,
                          float ppy, float tau, float maxReproj, int sub, int* out_rounds, int* out_inliers) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !assign || !poses6) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    Plan pl;
    int rc = fill_problem(ctx, pl.P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, 100.f, 0.5f, maxReproj, sub, NO_DRAW);
    if (rc) return rc;
    begin_call(ctx);
    rc = stage_inputs(ctx, pl, coords, assign, assign_stride);
    if (rc) return rc;
    CK(cudaMemcpyAsync(ctx->poses.p, poses6, (size_t)M * sizeof(Pose), cudaMemcpyHostToDevice, ctx->stream));
    std::vector<int> jobs((size_t)M);
    for (int i = 0; i < M; ++i) jobs[i] = i;
    CK(cudaMemcpyAsync(ctx->contrib.p, jobs.data(), (size_t)M * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    const int group = pick_group(ctx, pl.P, M);
    mark(ctx, EV_SELECT);
    rc = run_refine(ctx, pl, ctx->poses.as<Pose>(), ctx->poses_ref.as<Pose>(), ctx->contrib.as<int>(), nullptr, M, M, group);
    if (rc) return rc;
    mark(ctx, EV_REFINE);
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    CK(cudaMemcpy(poses6, ctx->poses_ref.p, (size_t)M * sizeof(Pose), cudaMemcpyDeviceToHost));
    std::vector<int> rr((size_t)M * 2);
    CK(cudaMemcpy(rr.data(), ctx->rounds.p, (size_t)M * 8, cudaMemcpyDeviceToHost));
    const int words = (pl.P.N + 31) / 32;
    std::vector<uint32_t> mk;
    if (out_inliers) {
        mk.resize((size_t)M * 2 * words);
        CK(cudaMemcpy(mk.data(), ctx->masks.p, mk.size() * 4, cudaMemcpyDeviceToHost));
    }
    for (int i = 0; i < M; ++i) {
        if (out_rounds) out_rounds[i] = rr[2 * i];
        if (out_inliers) {
            int c = 0;
            if (rr[2 * i] > 0) {
                const uint32_t* m = mk.data() + ((size_t)i * 2 + rr[2 * i + 1]) * words;
                for (int w = 0; w < words; ++w) c += __builtin_popcount(m[w]);
            }
            out_inliers[i] = c;
        }
    }
    ctx->st.M = M;
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// The arguments of launch_backward that come from the context's workspace after run_hypotheses.
static BwdArgs backward_args(esacb200_ctx* ctx, const Plan& pl, float* grads) {
    const Problem& P = pl.P;
    int* sc = ctx->scalars.as<int>();
    BwdArgs b;
    b.coords = pl.d_coords;
    b.grads = grads;
    b.assign32 = ctx->assign32.as<int>();
    b.perm = ctx->perm.as<int>();
    b.counts = ctx->counts.as<int>();
    b.offsets = ctx->offsets.as<int>();
    b.init = ctx->poses.as<Pose>();
    b.ref = ctx->poses_ref.as<Pose>();
    b.cells = ctx->cells.as<int>();
    b.probs = ctx->probs.as<double>();
    b.contrib = ctx->contrib.as<int>();
    b.n_contrib = sc + S_NCONTRIB;
    b.job_of = ctx->job_of.as<int>();
    b.masks = ctx->masks.as<uint32_t>();
    b.mask_words = (P.N + 31) / 32;
    b.rounds = ctx->rounds.as<int>();
    b.losses = ctx->losses.as<double>();
    b.out_loss = &ctx->stats.as<CallStats>()->local_loss;
    b.red = ctx->red.as<double>();
    b.hyp_grad = ctx->hypgrad.p;
    b.P = P;
    b.expected_override = nullptr;
    return b;
}

// -------------------------------------------------------------------------------------------------
// esac.backward on one image of problem P (filled and checked by the caller); `sh`: the steps of a sharded call, whose
// work and destination buffers this fills in.
static int backward_impl(esacb200_ctx* ctx, const Problem& P, const float* coords, const int64_t* assign, int64_t assign_stride,
                         float* grads, const float* gt_pose, float wRot, float wTrans, float cut, ShardSteps sh, double* out_loss) {
    Plan pl{P};
    const int M = P.M, E = P.E;
    begin_call(ctx);
    const size_t cbytes = (size_t)P.E * 3 * P.N * sizeof(float);
    float* d_grads = nullptr;
    int rc = stage_grads(ctx, grads, cbytes, d_grads);
    if (rc) return rc;
    // hypothesis-major sharding: every rank holds all planes and a slice of the hypotheses, so the gradient slices overlap:
    // the local gradient goes to a zeroed work buffer, is summed over the ranks and only then added to the caller's tensor
    float* d_dst = d_grads;
    if (sh.reduce_grads) {
        CK(ctx->grads_work.ensure(cbytes));
        d_grads = ctx->grads_work.as<float>();  // (the slices that will be used are zeroed once they are known, below)
        rc = ensure_host_flags(ctx, E);
        if (rc) return rc;
    }
    sh.d_work = d_grads;
    sh.d_dst = d_dst;
    rc = run_hypotheses(ctx, pl, coords, assign, assign_stride, sh, nullptr);
    if (rc) return rc;
    rc = backward_buffers(ctx, P, true, grow(ctx));
    if (rc) return rc;
    BwdArgs b = backward_args(ctx, pl, d_grads);
    Pinned& h = *ctx->pin;
    CallStats* d_stats = ctx->stats.as<CallStats>();
    if (is_device_ptr(gt_pose)) {
        CK(cudaMemcpyAsync(h.gt, gt_pose, sizeof(h.gt), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        memcpy(b.gt, h.gt, sizeof(h.gt));
    } else {
        memcpy(b.gt, gt_pose, 16 * sizeof(float));
    }
    b.wRot = wRot; b.wTrans = wTrans; b.cut = cut;
    double global_loss = 0;
    if (sh.exchange) {
        // exchange 2: the expectation sum_h p_h loss_h runs over the hypotheses of all ranks (esac.cpp:357-362, esac_derivative.h:372-374)
        launch_backward_losses(b, ctx->stream);
        CK(cudaMemcpyAsync(h.exchange, &d_stats->local_loss, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        double v[1] = {h.exchange[0]};
        if (sh.exchange(sh.user, 2, v, 1) != 0) return fail(ctx, ESACB200_ERR_ARG, "exchange callback failed (phase 2)");
        global_loss = v[0];
        h.upload = v[0];
        CK(cudaMemcpyAsync(&d_stats->global_loss, &h.upload, sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        b.expected_override = &d_stats->global_loss;
        ctx->st.kernel_launches += 1;
    } else if (sh.use_nccl) {
        // exchange 2 on the device: all-reduce of the partial expectations, no host round trip
        launch_backward_losses(b, ctx->stream);
        CKN(nccl_api().AllReduce(&d_stats->local_loss, &d_stats->global_loss, 1, kNcclFloat64, kNcclSum, ctx->nccl_comm, ctx->stream));
        b.expected_override = &d_stats->global_loss;
        ctx->st.kernel_launches += 2;
    }
    launch_backward(b, M, ctx->sm_count, ctx->stream);
    CK(cudaGetLastError());
    ctx->st.kernel_launches += 5;
    if (sh.reduce_grads) {
        rc = for_flagged_planes(ctx, E, (size_t)3 * P.N, d_grads, d_dst, 1);
        if (rc) return rc;
        CK(cudaGetLastError());
        d_grads = d_dst;
    }
    mark(ctx, EV_BWD);
    if (d_grads != grads) CK(cudaMemcpyAsync(grads, d_grads, cbytes, cudaMemcpyDeviceToHost, ctx->stream));
    rc = finish_call(ctx, pl, kAllStats, true, /*losses=*/true);
    if (rc) return rc;
    if (sh.use_nccl) global_loss = h.stats.global_loss;
    ctx->st.expected_loss = (sh.exchange || sh.use_nccl) ? global_loss : h.stats.local_loss;
    if (out_loss) *out_loss = ctx->st.expected_loss;
    return ESACB200_OK;
}

int esacb200_backward(esacb200_ctx* ctx, const float* coords, float* grads, int E, int H, int W, const int64_t* assign,
                      int64_t assign_stride, int M, const float* gt_pose, float wRot, float wTrans, float cut, int shiftX,
                      int shiftY, float f, float ppx, float ppy, float tau, float alpha, float beta, float maxReproj, int sub,
                      double* out_loss) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !assign || !grads || !gt_pose) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    Problem P;
    int rc = fill_problem(ctx, P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS_INJECTED);
    return rc ? rc : backward_impl(ctx, P, coords, assign, assign_stride, grads, gt_pose, wRot, wTrans, cut, ShardSteps(), out_loss);
} ESAC_ABI_CATCH(ctx)

// -------------------------------------------------------------------------------------------------
// Stream-ordered backward (esacb200_backward_async): esac.backward with the forward_async contract.  It runs in the same
// context as forward_async (ctx->async) and counts calls with it; the host path is the eager one, with the refinement group
// picked on the device from the number of contributing hypotheses.
int esacb200_reserve_backward_async(esacb200_ctx* ctx, int B, int E, int H, int W, int M, int sub) try {
    return reserve_async(ctx, B, E, H, W, M, sub, true);
} ESAC_ABI_CATCH(ctx)

int esacb200_backward_async(esacb200_ctx* ctx, int B, const float* coords, float* grads, int E, int H, int W,
                            const int64_t* assign, int64_t assign_stride, int M, const float* gt_poses, float wRot, float wTrans,
                            float cut, const int32_t* shifts, const float* cameras, float tau, float alpha, float beta,
                            float maxReproj, int sub, double* out_losses, int32_t* out_status) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    const void* ptrs[] = {coords, grads, assign, gt_poses, shifts, cameras, out_losses, out_status};
    const char* names[] = {"coords", "grads", "assign", "gt_poses", "shifts", "cameras", "out_losses", "out_status"};
    AsyncCall call;
    Problem P;
    int rc = B <= 0 ? fail(ctx, ESACB200_ERR_ARG, "backward_async: empty batch (B=%d)", B)
                    : fill_problem(ctx, P, E, H, W, M, 0, 0, 0.f, 0.f, 0.f, tau, alpha, beta, maxReproj, sub, DRAWS);
    if (!rc) rc = begin_async(ctx, true, B, P, coords, assign, assign_stride, shifts, cameras, out_status, 8, ptrs, names, call);
    if (rc) return rc;
    esacb200_ctx* a = call.a;
    const size_t cstride = (size_t)E * 3 * H * W;
    for (int b = 0; b < B; ++b) {
        Plan& pl = call.plans[b];
        AsyncImage& im = call.imgs[b];
        im.loss = out_losses + b;
        im.gt = gt_poses + 16 * (size_t)b;
        rc = run_hypotheses(a, pl, pl.d_coords, (const int64_t*)pl.d_assign, assign_stride, ShardSteps(), nullptr);
        if (!rc) rc = backward_buffers(a, pl.P, true, grow(a));
        if (rc) return fail(ctx, rc, "image %d: %s", b, a->err);
        BwdArgs args = backward_args(a, pl, grads + (size_t)b * cstride);
        args.wRot = wRot; args.wTrans = wTrans; args.cut = cut;
        BwdDev dv;
        dv.gt = im.gt;
        dv.flags = a->scalars.as<int>() + S_FLAGS;
        dv.dev = im.dev;
        launch_backward(args, M, a->sm_count, a->stream, &dv);
        launch_finish_backward_async(a->stats.as<CallStats>(), a->scalars.as<int>() + S_FLAGS, im.loss, im.status,
                                     a->seed_state.as<unsigned long long>(), im.advance, a->stream);
        a->st.kernel_launches += 6;
    }
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_backward_sharded(esacb200_ctx* ctx, const float* coords, float* grads, int E, int H, int W, const int64_t* assign,
                              int64_t assign_stride, int M, const float* gt_pose, float wRot, float wTrans, float cut,
                              int shiftX, int shiftY, float f, float ppx, float ppy, float tau, float alpha, float beta,
                              float maxReproj, int sub, esacb200_exchange_fn exchange, void* user, double* out_loss) try {
    if (!exchange) return ctx ? fail(ctx, ESACB200_ERR_ARG, "exchange callback is null") : ESACB200_ERR_ARG;
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !assign || !grads || !gt_pose) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
    Problem P;
    int rc = fill_problem(ctx, P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS_INJECTED);
    return rc ? rc : backward_impl(ctx, P, coords, assign, assign_stride, grads, gt_pose, wRot, wTrans, cut, {exchange, user}, out_loss);
} ESAC_ABI_CATCH(ctx)

// esac_backward with the experts / hypotheses sharded over the ranks of the communicator: the two exchanges of the path
// (SURVEY 8e) run as NCCL collectives on the context's stream -- an all-gather of two doubles per rank and an all-reduce of
// one -- with no host callback.  M may be 0: the rank then only takes part in the collectives.
int esacb200_backward_sharded_nccl(esacb200_ctx* ctx, const float* coords, float* grads, int E, int H, int W,
                                   const int64_t* assign, int64_t assign_stride, int M, const float* gt_pose, float wRot,
                                   float wTrans, float cut, int shiftX, int shiftY, float f, float ppx, float ppy, float tau,
                                   float alpha, float beta, float maxReproj, int sub, int reduce_grads, double* out_loss) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!ctx->nccl_comm) return fail(ctx, ESACB200_ERR_ARG, "no communicator: call esacb200_comm_init first");
    if (M > 0) {
        if (!coords || !assign || !grads || !gt_pose) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument");
        Problem P;
        int rc = fill_problem(ctx, P, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS_INJECTED);
        const ShardSteps sh = {nullptr, nullptr, /*use_nccl=*/true, /*reduce_grads=*/reduce_grads != 0};
        return rc ? rc : backward_impl(ctx, P, coords, assign, assign_stride, grads, gt_pose, wRot, wTrans, cut, sh, out_loss);
    }
    // no hypotheses here: neutral contributions to both collectives
    begin_call(ctx);
    CK(ctx->stats.ensure(sizeof(CallStats)));
    CK(ctx->gathered.ensure((size_t)ctx->comm_world * 2 * 8));
    Pinned& h = *ctx->pin;
    CallStats* d_stats = ctx->stats.as<CallStats>();
    h.exchange[0] = 0.; h.exchange[1] = -1e300; h.exchange[2] = 0.;  // local_loss, max_score, sum_exp
    CK(cudaMemcpyAsync(&d_stats->local_loss, h.exchange, sizeof(h.exchange), cudaMemcpyHostToDevice, ctx->stream));
    // the collectives below come in the order backward_impl issues them on the ranks that do hold hypotheses
    CKN(nccl_api().AllGather(&d_stats->max_score, ctx->gathered.p, 2, kNcclFloat64, ctx->nccl_comm, ctx->stream));
    const size_t n = reduce_grads ? (size_t)E * 3 * H * W : 0;
    float* d_dst = grads;
    if (reduce_grads) {  // zero contribution to the gradient sum, then the sum is added to this rank's tensor like everywhere
        if (!grads || E <= 0 || H <= 0 || W <= 0) return fail(ctx, ESACB200_ERR_ARG, "reduce_grads needs the gradient tensor and its shape on every rank");
        CK(ctx->grads_work.ensure(n * 4));
        int rc = ensure_host_flags(ctx, E);
        if (rc) return rc;
        CK(ctx->eflags.ensure((size_t)E * sizeof(int)));
        CK(cudaMemsetAsync(ctx->eflags.p, 0, (size_t)E * sizeof(int), ctx->stream));
        CKN(nccl_api().AllReduce(ctx->eflags.p, ctx->eflags.p, (size_t)E, kNcclInt32, kNcclMax, ctx->nccl_comm, ctx->stream));
        CK(cudaMemcpyAsync(ctx->h_flags, ctx->eflags.p, (size_t)E * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        if (!is_device_ptr(grads)) {
            CK(ctx->grads.ensure(n * 4));
            CK(cudaMemcpyAsync(ctx->grads.p, grads, n * 4, cudaMemcpyHostToDevice, ctx->stream));
            d_dst = ctx->grads.as<float>();
        }
        rc = for_flagged_planes(ctx, E, (size_t)3 * H * W, ctx->grads_work.as<float>(), d_dst, 0);
        if (rc) return rc;
    }
    CKN(nccl_api().AllReduce(&d_stats->local_loss, &d_stats->global_loss, 1, kNcclFloat64, kNcclSum, ctx->nccl_comm, ctx->stream));
    if (reduce_grads) {
        int rc = for_flagged_planes(ctx, E, (size_t)3 * H * W, ctx->grads_work.as<float>(), d_dst, 1);
        if (rc) return rc;
        if (!is_device_ptr(grads)) CK(cudaMemcpyAsync(grads, ctx->grads.p, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaGetLastError());
    }
    CK(cudaMemcpyAsync(&h.stats.global_loss, &d_stats->global_loss, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    mark(ctx, EV_END);
    CK(cudaStreamSynchronize(ctx->stream));
    if (out_loss) *out_loss = h.stats.global_loss;
    ctx->st.expected_loss = h.stats.global_loss;
    finish_stats(ctx);
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// esac_backward over a batch, on the worker contexts of run_batch.
int esacb200_backward_ragged(esacb200_ctx* ctx, int B, const float* const* coords, float* const* grads, const int* H, const int* W,
                             int E, const int64_t* assign, int64_t assign_stride, int M, const float* gt_poses, float wRot,
                             float wTrans, float cut, const int* shiftX, const int* shiftY, const float* f, const float* ppx,
                             const float* ppy, float tau, float alpha, float beta, float maxReproj, int sub,
                             double* out_losses) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (!coords || !grads || !H || !W || !assign || !gt_poses || B <= 0)
        return fail(ctx, ESACB200_ERR_ARG, "null pointer argument or empty batch");
    if (!f || !ppx || !ppy) return fail(ctx, ESACB200_ERR_ARG, "null camera array");
    if (ctx->inj_M) return fail(ctx, ESACB200_ERR_ARG, "injected cells are a single-image test hook");
    if (E <= 0 || M <= 0) return fail(ctx, ESACB200_ERR_ARG, "bad sizes E=%d M=%d", E, M);
    std::vector<Plan> plans;
    int rc = fill_problems(ctx, plans, B, E, H, W, M, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, DRAWS);
    if (rc) return rc;
    bool dev_c = false, dev_g = false;
    rc = pointer_kind(ctx, (const void* const*)coords, B, "coords", dev_c);
    if (rc) return rc;
    rc = pointer_kind(ctx, (const void* const*)grads, B, "grads", dev_g);
    if (rc) return rc;
    const int64_t arow = assign_stride == 0 ? 0 : (int64_t)M * assign_stride;
    std::vector<float> gt_host;
    const float* gt = gt_poses;
    if (is_device_ptr(gt_poses)) {  // read back with run_batch's synchronisation
        gt_host.resize((size_t)B * 16);
        CK(cudaMemcpyAsync(gt_host.data(), gt_poses, gt_host.size() * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
        gt = gt_host.data();
    }
    rc = run_batch(ctx, B, H, W, true, [&](esacb200_ctx* w, int b) {
        double loss = 0;
        int rc = backward_impl(w, plans[b].P, coords[b], assign + (size_t)b * arow, assign_stride, grads[b], gt + (size_t)b * 16, wRot,
                               wTrans, cut, ShardSteps(), &loss);
        if (!rc && out_losses) out_losses[b] = loss;
        return rc;
    });
    return rc ? rc : ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

// B images of one shape: the pointer and size arrays of [B,E,3,H,W] tensors.
int esacb200_backward_batch_cameras(esacb200_ctx* ctx, int B, const float* coords, float* grads, int E, int H, int W,
                                    const int64_t* assign, int64_t assign_stride, int M, const float* gt_poses, float wRot,
                                    float wTrans, float cut, const int* shiftX, const int* shiftY, const float* f,
                                    const float* ppx, const float* ppy, float tau, float alpha, float beta, float maxReproj,
                                    int sub, double* out_losses) try {
    if (!ctx) return ESACB200_ERR_ARG;
    if (!coords || !grads || !assign || !gt_poses || B <= 0) return fail(ctx, ESACB200_ERR_ARG, "null pointer argument or empty batch");
    if (!f || !ppx || !ppy) return fail(ctx, ESACB200_ERR_ARG, "null camera array");
    if (ctx->inj_M) return fail(ctx, ESACB200_ERR_ARG, "injected cells are a single-image test hook");
    if (E <= 0 || H <= 0 || W <= 0 || M <= 0) return fail(ctx, ESACB200_ERR_ARG, "bad sizes E=%d H=%d W=%d M=%d", E, H, W, M);
    const size_t cstride = (size_t)E * 3 * H * W;
    const auto cp = slices(coords, B, cstride);
    const auto gp = slices(grads, B, cstride);
    const std::vector<int> hs((size_t)B, H), ws((size_t)B, W);
    return esacb200_backward_ragged(ctx, B, cp.data(), gp.data(), hs.data(), ws.data(), E, assign, assign_stride, M, gt_poses, wRot,
                                    wTrans, cut, shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub, out_losses);
} ESAC_ABI_CATCH(ctx)

int esacb200_backward_batch(esacb200_ctx* ctx, int B, const float* coords, float* grads, int E, int H, int W,
                            const int64_t* assign, int64_t assign_stride, int M, const float* gt_poses, float wRot,
                            float wTrans, float cut, const int* shiftX, const int* shiftY, float f, float ppx, float ppy,
                            float tau, float alpha, float beta, float maxReproj, int sub, double* out_losses) try {
    if (!ctx) return ESACB200_ERR_ARG;
    const size_t n = B > 0 ? (size_t)B : 1;  // B <= 0 is rejected by the call below, with its usual message
    const std::vector<float> fs(n, f), cx(n, ppx), cy(n, ppy);
    return esacb200_backward_batch_cameras(ctx, B, coords, grads, E, H, W, assign, assign_stride, M, gt_poses, wRot, wTrans, cut,
                                           shiftX, shiftY, fs.data(), cx.data(), cy.data(), tau, alpha, beta, maxReproj, sub,
                                           out_losses);
} ESAC_ABI_CATCH(ctx)

}  // extern "C"
