// Host side of libesac_b200.so, shared by its translation units: the context, the frame of every C entry point (device,
// errors, exceptions), the plan of one image, and the helpers that the entry points of more than one file call.
//
//   capi.cu             the context: lifecycle, options, getters
//   capi_pipeline.cu    the stages every ESAC call is built from, the stream-ordered context, the batch workers
//   capi_esac.cu        esac.forward / esac.backward in every form
//   capi_hypotheses.cu  the hypotheses node and the pose loss
//   capi_losses.cu      the two expert losses
//   capi_gate.cu        expert gates and the stream-ordered hypothesis assignment
//   capi_eval.cu        test-time pose evaluation
//   capi_cluster.cu     clustering a large environment into experts
//   capi_render.cu      rendering ground-truth maps from an SfM reconstruction
//   capi_data.cu        one step of a device-resident image set
//   capi_experts.cu     inference of a stack of experts
//   capi_gating_net.cu  inference of the gating network
//   capi_testhooks.cu   include/esac_b200_testhooks.h
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include <exception>
#include <functional>
#include <vector>

#include "../../include/esac_b200.h"
#include "esac_internal.h"

namespace esacb200::capi {

// A device buffer that owns its memory: freed when the buffer dies (the owner destroys it on its device, after its stream).
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() {
        if (p) cudaFree(p);
    }
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    template <class T>
    T* as() const { return (T*)p; }
};

// The tunables of esacb200_set_option.
struct Options {
    int max_tries = 1000000;
    int max_ref_steps = 100;
    int fixed_seed = 0;
    int refine_group_opt = 0;
    int refine_pretest = 1;    // inlier selection: float pretest with a rounding-error bound, exact arithmetic only where in doubt
    int refine_compact = 1;    // LM evaluations over per-CTA inlier lists instead of predicated passes over all cells
    int refine_profile = 0;    // 1: block 0 of the refinement kernel records phase cycle counts (esacb200_get_refine_profile)
    int refine_jobs_per_group = 3;
    int sample_prefilter = 1;
    int sample_span0 = 256;       // tries per hypothesis in the first wave (a multiple of the 256-try pass of a prefilter CTA)
    float sample_window = 1.25f;  // later waves: window / acceptance rate
    int sample_waves = 6;         // launched unconditionally (empty ones cost ~6 us each); what is left after them goes to tail_kernel
    float sample_tail_boost = 1.f;  // window factor once <= 64 hypotheses are left in a lane (x2 more for <= 8)
    int sample_trace = 0;         // 1: prefilter / exact kernels of waves 0-31 stamp first-CTA-start / last-CTA-end times (esacb200_get_sample_trace)
    int sample_groups = 2;        // lanes of the sampling stage (third and fourth lane: no gain measured)
    float sample_hint = 0.95f;    // prefilter no tries of a window beyond one whose 4th point the float path puts within
                                  // this fraction of tau (0: off; below the prefilter's 2 tau band)
    int upload_split = 1;
    int hyp_offset = 0, hyp_stride = 1;
    int score_ppt_opt = 0, score_hc_opt = 0;
    int batch_workers = 8;
};

enum { EV_START = 0, EV_H2D, EV_PREP, EV_SAMPLE, EV_FOLD, EV_SCORE, EV_SELECT, EV_REFINE, EV_BWD, EV_END, EV_COUNT };

// What the last call on a context left in its per-hypothesis buffers: the getters read nothing else.  Every call clears it
// (begin_call, run_batch); only the code that writes those buffers sets it.
struct LastCall {
    int M = 0;
    bool drew = false;         // poses, cells, tries, probs, refined poses and the sampling lanes' counters
    int lanes = 0, lane_cap = 0;  // of the sampling stage (sample_sizes: G, Mg)
    bool scored = false;       // scores
    bool losses = false;       // esac.backward's per-hypothesis losses
};

// The context's pinned host memory: a member for each value a call reads back or uploads through it, so no two uses share
// bytes.
struct Pinned {
    ForwardRecord fwd;   // the forward record (esacb200_forward, forward_sharded)
    float gt[16];        // a device ground-truth pose (esac.backward)
    int scalars[8];      // the head of the scalars buffer (finish_call)
    int n_contrib;       // contributing hypotheses before the refinement (run_hypotheses)
    int gating_flags;    // the flags of esacb200_assign
    CallStats stats;     // the call statistics (finish_call; global_loss: backward_sharded_nccl without hypotheses)
    int rounds[2];       // head of the refinement rounds of esacb200_forward
    double exchange[3];  // this rank's contributions to the exchanges of a sharded backward, and their results
    double upload;       // the global expected loss from the exchange callback, on its way to CallStats::global_loss
};

}  // namespace esacb200::capi

struct esacb200_ctx {
    int device = 0;
    int sm_count = 0;
    char dev_name[128] = {0};
    cudaStream_t own_stream = nullptr;
    cudaStream_t copy_stream = nullptr;
    cudaStream_t aux_stream = nullptr;   // second lane of the sampling stage
    cudaStream_t aux_more[2] = {nullptr, nullptr};  // third and fourth lane (option sample_groups)
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_join_more[2] = {nullptr, nullptr};
    cudaEvent_t ev_copied[2] = {nullptr, nullptr}, ev_consumed[2] = {nullptr, nullptr};
    cudaStream_t stream = nullptr;
    uint64_t seed = 1305;  // thread_rand.h:103
    uint64_t calls = 0;
    esacb200::capi::Options opt;
    int* h_flags = nullptr;    // pinned: per-expert "receives gradient on some rank" flags (hypothesis-major sharding)
    int h_flags_cap = 0;
    int refine_coresident = 0;
    char err[512] = {0};
    // workspace
    esacb200::capi::DevBuf coords, grads, assign64, assign32, counts, offsets, perm, slot_of, chunks, scalars, centres, poses,
        poses_ref, cells, tries, posepk, part, scores, probs, stats, contrib, masks, rounds, scratch, barrier, fwd_rec, inject,
        losses, red, hypgrad, job_of, gt, smp_int, smp_surv, smp_trace, clist, eflags, coords4, coords_alt, assign64_alt, out_batch, prof,
        contrib8, upstream;
    esacb200::capi::Pinned* pin = nullptr;
    int inj_M = 0, inj_T = 0;
    int inj_lo[2] = {0, 0}, inj_hi[2] = {0, 0};  // smallest and largest injected x, y: checked against each call's map
    cudaEvent_t ev[esacb200::capi::EV_COUNT] = {nullptr};
    bool ev_used[esacb200::capi::EV_COUNT] = {false};
    esacb200_stats st;
    esacb200::capi::LastCall last;
    // NCCL communicator of the sharded entry points (esacb200_comm_init); the library is resolved at run time with dlopen
    void* nccl_comm = nullptr;
    int comm_world = 1, comm_rank = 0;
    esacb200::capi::DevBuf gathered, grads_work;
    std::vector<esacb200_ctx*> workers;  // lazily created contexts of esacb200_backward_batch (own stream + workspace each)
    // Stream-ordered forward and backward (esacb200_forward_async / _backward_async): their own context, so that eager calls
    // never touch the buffers a captured graph holds.  In that context: is_async = true, seed_state = device {base seed,
    // async calls}, and frozen once a capture has used the workspace (from then on nothing in it is freed or reallocated).
    esacb200_ctx* async = nullptr;
    bool is_async = false;
    bool frozen = false;
    esacb200::capi::DevBuf seed_state;
    // The stream-ordered losses' workspace (esacb200_reproj_loss_async / _coord_loss_async), in the async context: apart from
    // the forward's and the backward's, so that loss graphs and ESAC graphs do not size each other's buffers; loss_frozen
    // once a capture has used it.
    esacb200::capi::DevBuf loss_ws;
    bool loss_frozen = false;
};

namespace esacb200::capi {

// Every entry point works on the context's device and leaves the caller's current device as it found it (torch reads the
// current device with cudaGetDevice: a library that silently switches it redirects the caller's later allocations).
struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int device) {
        if (cudaGetDevice(&prev) != cudaSuccess) { cudaGetLastError(); prev = -1; }
        if (prev != device) cudaSetDevice(device);
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
    DeviceGuard(const DeviceGuard&) = delete;
    DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// ---- NCCL, resolved at run time ---------------------------------------------------------------------------------
// The library must load on machines without NCCL (the CPU test box) and must share the NCCL instance the host process already
// holds (torch bundles its own libnccl.so.2): no link-time dependency, dlopen of the soname instead -- RTLD_NOLOAD first, so an
// already loaded copy is reused.  Only the five entry points below are needed; their prototypes are NCCL's public ABI.
struct NcclApi {
    typedef struct { char internal[128]; } UniqueId;
    int (*GetUniqueId)(UniqueId*) = nullptr;
    int (*CommInitRank)(void**, int, UniqueId, int) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool ok = false;
};
constexpr int kNcclFloat32 = 7;  // ncclFloat
constexpr int kNcclFloat64 = 8;  // ncclDouble
constexpr int kNcclSum = 0;      // ncclSum
constexpr int kNcclInt32 = 2;    // ncclInt32
constexpr int kNcclMax = 2;      // ncclMax

NcclApi& nccl_api();

// Records the message of a failed call in c->err and returns `code`.
int fail(esacb200_ctx* c, int code, const char* fmt, ...);

#define CKN(call)                                                                                              \
    do {                                                                                                       \
        int r__ = (call);                                                                                      \
        if (r__ != 0)                                                                                          \
            return fail(ctx, ESACB200_ERR_CUDA, "%s failed: %s (%s:%d)", #call,                                \
                        nccl_api().GetErrorString ? nccl_api().GetErrorString(r__) : "NCCL error", __FILE__, __LINE__); \
    } while (0)

#define CK(call)                                                                                          \
    do {                                                                                                  \
        cudaError_t e__ = (call);                                                                         \
        if (e__ != cudaSuccess)                                                                           \
            return fail(ctx, ESACB200_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), \
                        __FILE__, __LINE__);                                                              \
    } while (0)

// No C++ exception may cross the C ABI (std::vector / std::thread can throw): every entry point that allocates on the host is
// a function-try-block ending in this handler.
#define ESAC_ABI_CATCH(ctx)                                                                                   \
    catch (const std::exception& e) {                                                                         \
        return (ctx) ? fail((ctx), ESACB200_ERR_ARG, "host-side failure: %s", e.what()) : ESACB200_ERR_ARG;   \
    }                                                                                                         \
    catch (...) {                                                                                             \
        return (ctx) ? fail((ctx), ESACB200_ERR_ARG, "host-side failure (unknown exception)") : ESACB200_ERR_ARG; \
    }

// scalars buffer layout (ints): [0]=n_chunks [1]=work_counter [2]=flags [3]=winner [4]=n_contrib
enum { S_NCHUNKS = 0, S_WORK, S_FLAGS, S_WINNER, S_NCONTRIB, S_COUNT = 16 };

struct Plan {
    Problem P;
    int T, ppt, hc, grid, vec_ok;
    const float* d_coords = nullptr;
    const long long* d_assign;
    long long assign_stride;
    int split_e = 0;  // > 0: host maps are uploaded in two halves [0, split_e) / [split_e, E) on the copy stream (ev_copied[0/1])
    const struct AsyncImage* async = nullptr;  // stream-ordered call: device parameters and the caller's outputs
    double min_prob = kProbThresh;  // the hypotheses with !(p < min_prob) contribute (the hypotheses node's floor)
};

// One image of a stream-ordered forward or backward: what its kernels read from device memory, and where its results go.
struct AsyncImage {
    DevParams dev;
    float* pose;        // [4,4] (forward)
    long long* expert;  // (forward)
    double* loss;       // (backward) esac.backward's return value
    const float* gt;    // (backward) [4,4] camera->world ground truth
    int* status;
    int advance;        // the last image of an execution: advance the async call counter by B
};

// Whether a call draws hypotheses from its problem, and whether it draws the context's injected cells (esacb200_inject_cells)
// when there are any; a call that draws ignores or clears them otherwise.
enum Draw { NO_DRAW, DRAWS, DRAWS_INJECTED };

// The sharded backward's steps inside the hypotheses prefix (none for a single-GPU call).
struct ShardSteps {
    esacb200_exchange_fn exchange = nullptr;  // host callback: softmax normalisation over all ranks
    void* user = nullptr;
    bool use_nccl = false;      // the same exchange as an all-gather on the device
    bool reduce_grads = false;  // hypothesis-major sharding: zero the work buffer's slices of the planes some rank updates
    float* d_work = nullptr;
    float* d_dst = nullptr;
};

// A stream-ordered call of B images of one shape: the async context, and per image its Plan and its AsyncImage (whose
// outputs the entry point fills in).
struct AsyncCall {
    esacb200_ctx* a = nullptr;
    std::vector<Plan> plans;
    std::vector<AsyncImage> imgs;
};

// How much of CallStats a call reads back (finish_call): nothing, what the select kernel wrote (entropy .. n_contrib) or all
// of it.
constexpr size_t kNoStats = 0, kSelectStats = offsetof(CallStats, unused), kAllStats = sizeof(CallStats);

// The B image pointers of a stacked [B, ...] tensor whose images lie `stride` elements apart (a null base: B nulls).
template <class T>
std::vector<T*> slices(T* base, int B, size_t stride) {
    std::vector<T*> p((size_t)B, nullptr);
    for (int b = 0; base && b < B; ++b) p[b] = base + (size_t)b * stride;
    return p;
}

// ---- capi.cu: the call frame -------------------------------------------------------------------------------------
bool is_device_ptr(const void* p);
void mark(esacb200_ctx* c, int id);
void begin_call(esacb200_ctx* ctx);
void finish_stats(esacb200_ctx* ctx);
int last_call_left(esacb200_ctx* ctx, bool wrote, const char* what);

// ---- capi_pipeline.cu: the stages --------------------------------------------------------------------------------
int fill_problem(esacb200_ctx* ctx, Problem& P, int E, int H, int W, int M, int shiftX, int shiftY, float f, float ppx,
                 float ppy, float tau, float alpha, float beta, float maxReproj, int sub, Draw draw);
int fill_problems(esacb200_ctx* ctx, std::vector<Plan>& plans, int B, int E, const int* H, const int* W, int M, const int* shiftX,
                  const int* shiftY, const float* f, const float* ppx, const float* ppy, float tau, float alpha, float beta,
                  float maxReproj, int sub, Draw draw);

// The `need` of a stage's buffer sizes that grows each buffer to its size (a failed allocation fails the call on ctx).
struct Grow {
    esacb200_ctx* ctx;
    int operator()(DevBuf& b, size_t bytes) const;
};
Grow grow(esacb200_ctx* ctx);
// The backward's tail (bwd_reduce .. bwd_assemble); `losses`: esac.backward's own per-hypothesis losses too.
template <class Need>
int backward_buffers(esacb200_ctx* ctx, const Problem& P, bool losses, Need&& need);

int upload_inputs(esacb200_ctx* ctx, Plan& pl, const float* coords, const int64_t* assign, int64_t stride, DevBuf& cbuf,
                  DevBuf& abuf, cudaStream_t copy_stream, bool allow_split = false);
int plan_and_prep(esacb200_ctx* ctx, Plan& pl);
int stage_inputs(esacb200_ctx* ctx, Plan& pl, const float* coords, const int64_t* assign, int64_t stride, bool allow_split = false);
int run_sample(esacb200_ctx* ctx, const Plan& pl, uint64_t seed);
int run_score(esacb200_ctx* ctx, const Plan& pl);
int pick_group(const esacb200_ctx* ctx, const Problem& P, int jobs_hint);
int run_refine(esacb200_ctx* ctx, const Plan& pl, const Pose* in, Pose* out, const int* d_jobs, const int* d_njobs,
               int n_jobs_host, int max_jobs, int group, uint32_t* masks_out = nullptr);
uint64_t call_seed(esacb200_ctx* ctx);
int reserve_forward_batch(esacb200_ctx* ctx, const std::vector<Plan>& plans, bool host_coords, bool backward = false);
void record_draw(esacb200_ctx* ctx, const Plan& pl, bool losses);
int finish_call(esacb200_ctx* ctx, const Plan& pl, size_t stats_bytes, bool drew, bool losses = false);
int pointer_kind(esacb200_ctx* ctx, const void* const* p, int B, const char* what, bool& device);
int for_flagged_planes(esacb200_ctx* ctx, int E, size_t plane, float* work, float* dst, int phase);
int stage_grads(esacb200_ctx* ctx, float* grads, size_t bytes, float*& d_grads);
int run_hypotheses(esacb200_ctx* ctx, Plan& pl, const float* coords, const int64_t* assign, int64_t assign_stride,
                   const ShardSteps& sh, uint32_t* masks);

// ---- capi_pipeline.cu: the stream-ordered context ----------------------------------------------------------------
int stream_capturing(esacb200_ctx* ctx, bool& capturing);
int async_context(esacb200_ctx* ctx, bool capturing, const char* what, esacb200_ctx** out);
int async_workspace(esacb200_ctx* ctx, esacb200_ctx* a, const std::vector<Plan>& plans, bool capturing, bool backward,
                    const char* name = nullptr);
int enter_async(esacb200_ctx* ctx, const Problem& P, bool backward, const char* name, esacb200_ctx** out);
int reserve_context(esacb200_ctx* ctx, const char* what, esacb200_ctx** out);
int device_args(esacb200_ctx* ctx, const char* what, int n, const void* const* ptrs, const char* const* names, unsigned optional = 0);
int begin_async(esacb200_ctx* ctx, bool backward, int B, const Problem& P, const float* coords, const int64_t* assign,
                int64_t assign_stride, const int32_t* shifts, const float* cameras, int32_t* out_status, int n,
                const void* const* ptrs, const char* const* names, AsyncCall& call, const char* name = nullptr);

// ---- capi_losses.cu: host images of a ragged call ------------------------------------------------------------------
size_t pack_offsets(const std::vector<size_t>& bytes, std::vector<size_t>& off);
int copy_packed(esacb200_ctx* ctx, char* const* host, const std::vector<size_t>& bytes, const std::vector<size_t>& off, char* dev,
                bool to_device, cudaStream_t stream);
template <class T>
int stage_images(esacb200_ctx* ctx, T* const* ptrs, const std::vector<size_t>& bytes, bool device, bool upload, DevBuf& buf,
                 std::vector<T*>& dev, std::vector<size_t>& off);

// ---- capi_pipeline.cu: batches -----------------------------------------------------------------------------------
int run_batch(esacb200_ctx* ctx, int B, const int* H, const int* W, bool draws, const std::function<int(esacb200_ctx*, int)>& image);

}  // namespace esacb200::capi
