// Internal declarations shared by the translation units of libesac_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "esac_geom.cuh"

namespace esacb200 {

#ifdef __CUDACC__
// One stage of warp_reduce_scatter.  O is a template parameter so that every index into w is a constant: with the stage
// width a loop variable (o >>= 1) the inner loops were not unrolled, and w lived in local memory.
template <int O>
__device__ __forceinline__ void reduce_scatter_stage(double* w, int lane) {
    const bool up = (lane & O) != 0;
#pragma unroll
    for (int i = 0; i < O; ++i) {
        const double keep = up ? w[i + O] : w[i];
        const double send = up ? w[i] : w[i + O];
        w[i] = keep + __shfl_xor_sync(0xffffffffu, send, O);
    }
}
// Warp reduce-scatter of NV <= 32 doubles per lane: lane L returns the warp total of value L (0 for L >= NV).
// A transposing butterfly: 31 double shuffles instead of 5*NV.
template <int NV>
__device__ __forceinline__ double warp_reduce_scatter(const double (&v)[NV]) {
    static_assert(NV <= 32, "at most 32 values");
    const int lane = threadIdx.x & 31;
    double w[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) w[i] = i < NV ? v[i] : 0.0;
    reduce_scatter_stage<16>(w, lane);
    reduce_scatter_stage<8>(w, lane);
    reduce_scatter_stage<4>(w, lane);
    reduce_scatter_stage<2>(w, lane);
    reduce_scatter_stage<1>(w, lane);
    return w[0];
}

// Sum of NV doubles per thread over a block of THREADS threads in a fixed order: a butterfly within each warp, then the
// warp totals in warp order.  The totals are valid in thread 0.  Every thread of the block calls it.
template <int THREADS, int NV>
__device__ __forceinline__ void block_sum_fixed(double (&v)[NV]) {
    __shared__ double warp_sum[NV][THREADS / 32];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[i] += __shfl_xor_sync(0xffffffffu, v[i], o);
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int i = 0; i < NV; ++i) warp_sum[i][threadIdx.x >> 5] = v[i];
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        double s = 0.;
        if (threadIdx.x == 0)
            for (int w = 0; w < THREADS / 32; ++w) s += warp_sum[i][w];
        v[i] = s;
    }
}

// Per-image sum over the `blocks` blocks (blockIdx.x = 0 .. blocks-1) of image b, deterministic: every block sums its
// threads' NV values (block_sum_fixed) and stores the totals in partial[part0 + blockIdx.x][NV]; the image's last block to
// take a ticket adds the partials in block order.  Returns true in thread 0 of that block, with the image totals in v;
// tickets[b] (zero before the launch) is left zero for the next one.  The block count and the partial base are the
// image's own, so images of different sizes share one launch and each sums exactly as it would alone.
template <int THREADS, int NV>
__device__ __forceinline__ bool block_image_sum(double (&v)[NV], double* __restrict__ partial, unsigned* __restrict__ tickets,
                                                int b, unsigned blocks, size_t part0) {
    __shared__ bool last;
    block_sum_fixed<THREADS, NV>(v);
    if (threadIdx.x == 0) {
#pragma unroll
        for (int i = 0; i < NV; ++i) partial[(part0 + blockIdx.x) * NV + i] = v[i];
        __threadfence();
        last = atomicAdd(&tickets[b], 1u) == blocks - 1;
    }
    __syncthreads();
    if (!last) return false;
    __threadfence();
#pragma unroll
    for (int i = 0; i < NV; ++i) v[i] = 0.;
    for (unsigned k = threadIdx.x; k < blocks; k += THREADS) {
#pragma unroll
        for (int i = 0; i < NV; ++i) v[i] += __ldcg(&partial[(part0 + k) * NV + i]);
    }
    block_sum_fixed<THREADS, NV>(v);
    if (threadIdx.x == 0) tickets[b] = 0;  // ready for the next launch
    return threadIdx.x == 0;
}
#endif

// Per-call problem description (esac.cpp:64-77 arguments + tensor sizes).
struct Problem {
    int E, H, W, N, M;
    int shiftX, shiftY, sub;
    float f, ppx, ppy;
    float tau, alpha, beta, max_reproj;
};

// What a forward hands back to the host, in one device record that one copy reads (finish_forward_kernel; for a sharded
// forward select_gathered_kernel): the camera->world pose of the winner, its expert, the bad-assignment flag and the
// winning hypothesis, and for a sharded forward the owning rank.
struct ForwardRecord {
    float pose[16];
    float expert, bad, winner, rank;
};
static_assert(sizeof(ForwardRecord) == 20 * sizeof(float), "ForwardRecord is 20 floats");

// Statistics of one call on the device.  The select kernel writes entropy, winner, n_contrib and the local softmax
// normalisation (max_score, sum_exp); the backward writes the expected loss over this rank's hypotheses (local_loss) and,
// sharded, over all ranks (global_loss).
struct CallStats {
    double entropy, winner, n_contrib, unused;
    double local_loss, max_score, sum_exp, global_loss;
};
static_assert(sizeof(CallStats) == 8 * sizeof(double), "CallStats is 8 doubles");
static_assert(offsetof(CallStats, sum_exp) == offsetof(CallStats, max_score) + sizeof(double),
              "(max_score, sum_exp) are all-gathered as two adjacent doubles");

// Tail of the record a shard contributes to the all-gather of a sharded forward, behind its M_pad scores (include/esac_b200.h):
// the camera pose of the local winner, its global expert id (-1 on a bad assignment), the local winner, the shard's M, and
// hyp_offset / hyp_stride (local hypothesis k is hypothesis hyp_offset + k * hyp_stride of the unsharded problem).  With
// M = 0 every field before M is -1.
struct ShardTail {
    double pose[16];
    double expert, winner, M, hyp_offset, hyp_stride;
};
constexpr int kPackTail = sizeof(ShardTail) / sizeof(double);  // doubles behind the M_pad scores of a shard's record
static_assert(kPackTail == 21, "the shard record's tail is the 21 doubles include/esac_b200.h documents");

// Per-image values of a stream-ordered forward or backward (esacb200_forward_async / _backward_async) that the kernels read
// from device memory instead of from Problem / a seed argument, so that a captured graph replays with the values current at
// replay time.  The kernels that take one are templates on a flag DEV; with DEV = false they ignore it and read Problem as
// before.
struct DevParams {
    const int* shift = nullptr;                // [2] shiftX, shiftY
    const float* cam = nullptr;                // [3] f, ppx, ppy
    const unsigned long long* seed = nullptr;  // [0] base seed, [1] async calls before this execution
    int index = 0;                             // image b of the execution: its draws are those of call [1] + b
    int fixed_seed = 0;
};

#ifdef __CUDACC__
// The image's shift and camera: from P, or (DEV) from a.dev, where `a` is the kernel's argument struct.
template <bool DEV, class A> __device__ __forceinline__ int dev_shift_x(const Problem& P, const A& a) {
    if constexpr (DEV) return __ldg(a.dev.shift); else return P.shiftX;
}
template <bool DEV, class A> __device__ __forceinline__ int dev_shift_y(const Problem& P, const A& a) {
    if constexpr (DEV) return __ldg(a.dev.shift + 1); else return P.shiftY;
}
template <bool DEV, class A> __device__ __forceinline__ float dev_f(const Problem& P, const A& a) {
    if constexpr (DEV) return __ldg(a.dev.cam); else return P.f;
}
template <bool DEV, class A> __device__ __forceinline__ float dev_ppx(const Problem& P, const A& a) {
    if constexpr (DEV) return __ldg(a.dev.cam + 1); else return P.ppx;
}
template <bool DEV, class A> __device__ __forceinline__ float dev_ppy(const Problem& P, const A& a) {
    if constexpr (DEV) return __ldg(a.dev.cam + 2); else return P.ppy;
}
#endif

// CTAs per refinement job for `jobs` jobs of an N-cell map (the host's pick_group, and the stream-ordered backward's
// refinement kernel, which knows the job count only on the device): one rule, so the two pick the same group.
ESAC_HD int refine_group_rule(int N, int coresident, int group_opt, int jobs_per_group, int jobs) {
    if (group_opt > 0) return group_opt < coresident ? group_opt : coresident;
    const int words = (N + 31) / 32;
    // ~320 cells per CTA, up to every co-resident CTA: with the warp-parallel slot summation the inter-CTA barrier costs less
    // than the fp64 work it spreads (60x80 -> 16 CTAs, 480x640 -> every co-resident CTA)
    int g = words / 10;
    if (g < 1) g = 1;
    // Jobs are handed out dynamically inside the kernel, so a group may work through several jobs: fewer, larger groups even
    // out the differing job lengths (rounds x LM iterations) -- worth it only while a block's share of the map stays large
    // against the cost of a group exchange (480x640: yes; 60x80: no)
    int waves = jobs >= 8 ? jobs_per_group : 1;
    int concurrent = jobs > 0 ? (jobs + waves - 1) / waves : 1;
    int cap = coresident / concurrent;
    if (waves > 1 && (cap < 1 || N / (cap < 1 ? 1 : cap) < 4096)) cap = coresident / (jobs > 0 ? jobs : 1);
    if (cap < 1) cap = 1;
    if (g > cap) g = cap;
    return g;
}

// Groups of one refinement launch of `group` CTAs each, for at most max_jobs jobs.
ESAC_HD int refine_n_groups(int coresident, int group, int max_jobs) {
    int n_groups = coresident / group;
    if (n_groups > max_jobs) n_groups = max_jobs;
    if (n_groups < 1) n_groups = 1;
    return n_groups;
}

// Hypotheses of one expert are contiguous in "sorted slot" order (stable by hypothesis index);
// a chunk is <= kMaxChunk consecutive slots of one expert: the unit the scoring kernel pairs with a
// pixel tile.
constexpr int kMaxChunk = 64;
struct ChunkDesc {
    int expert;
    int slot0;
    int count;
    int pad;
};

// Folded fp32 pose for the scoring kernel: rows [A_r0 A_r1 A_r2 | b_r] of diag(f,f,1)*R and
// diag(f,f,1)*(R*c + t).
struct PosePk {
    float4 v[3];
};

struct ScoreArgs {
    const float* coords;     // [E,3,N]
    const float* centres;    // [E,3]
    const PosePk* poses;     // [M] sorted slots
    const ChunkDesc* chunks;
    const int* n_chunks;     // device scalar
    int* work_counter;       // device scalar, zeroed by the prep kernel
    float* part;             // [M, T] partial soft-inlier sums (slot-major)
    Problem P;
    int T;                   // pixel tiles per plane
    int hc;                  // hypotheses per chunk used when building the chunk table
    float k1, k0;            // beta*log2(e), -beta*tau*log2(e) (minus kScorePairShift when fold)
    float tmax;              // fold: k1*maxReproj + k0, the exponent of a clamped cell
    float tiny;              // floor of |p|^2: 1e-30, times k1^2 when fold
    int fold;                // k1 folded into the f rows and pixel offsets, one reciprocal per pair of cells
    int vec_ok;              // planes are 16-byte aligned and N % 4 == 0
    DevParams dev;           // dev.shift != null: shift and camera from device memory (stream-ordered forward)
};

// --- score.cu -----------------------------------------------------------------------------
// prep: int64 strided assignment -> int32, per-expert histogram / offsets / stable permutation,
// chunk table, work counter reset, plane centres.  flags[0] != 0 on a bad expert index.
void launch_prep(const float* coords, const long long* assign, long long assign_stride, const Problem& P, int hc,
                 int* assign32, int* counts, int* offsets, int* perm, int* slot_of, ChunkDesc* chunks, int* n_chunks,
                 int* work_counter, float* centres, int* flags, int roles, cudaStream_t st);
// dev: non-null -> f from device memory (stream-ordered forward)
void launch_fold(const Pose* poses, const int* perm, const int* assign32, const float* centres, const Problem& P,
                 float kf, PosePk* out, cudaStream_t st, const DevParams* dev = nullptr);
int score_tile_pixels(int ppt);
// k1, k0, tmax, tiny and fold of the scoring arguments for this problem
void score_constants(const Problem& P, ScoreArgs& a);
void launch_score(const ScoreArgs& a, int ppt, int grid, cudaStream_t st);
// scores[h] = (alpha/W/H) * sum_tiles part ; softmax ; entropy ; argmax ; contributing list (the hypotheses with
// !(p < min_prob), in ascending order; kProbThresh everywhere but the hypotheses node)
// into stats: entropy, winner, n_contrib, max_score, sum_exp
void launch_select(const float* part, const int* slot_of, const Problem& P, int T, double* scores, double* probs,
                   CallStats* stats, int* winner, int* contrib, int* n_contrib, double min_prob, cudaStream_t st);

void launch_rescale_probs(const double* scores, const Problem& P, double gmax, double gsum, double* probs, int* contrib,
                          int* n_contrib, double min_prob, cudaStream_t st);
void launch_rescale_probs_gathered(const double* scores, const Problem& P, const double* pairs, int world, double* norm_out,
                                   double* probs, int* contrib, int* n_contrib, double min_prob, cudaStream_t st);

// --- hyp.cu -------------------------------------------------------------------------------
// Work state of the sampling waves (all device memory, M = hypotheses).
struct Accepted {
    Pose pose;
    int cells[8];
};
struct SampleState {
    unsigned long long* best;  // [M] (lowest accepted try << 32) | staging slot; ~0 = none yet
    Accepted* stage;           // [cap_acc] poses of accepted tries
    int cap_acc;
    int* base;      // [M] first try not judged yet
    int* ovf;       // [M] lowest survivor that did not fit the list in the current wave
    int* list;      // [2M] unresolved hypotheses (second half: scratch for rebuilding)
    int2* surv;     // [cap] (hypothesis, try) pairs that passed the float prefilter
    int cap;
    int* counters;  // [SC_COUNT], indexed by SampleCounter
    int M;
};
// Slots of SampleState::counters.
enum SampleCounter {
    SC_UNRESOLVED = 0,  // hypotheses in the list
    SC_SURVIVORS,       // (hypothesis, try) pairs the prefilter passed in the current wave
    SC_STAGED,          // accepted poses staged
    SC_SPAN,            // tries per hypothesis in the current wave
    SC_TICKET,          // exact_kernel CTAs done with the current wave
    // diagnostics (esacb200_get_sample_profile)
    SC_PREFILTERED,     // tries prefiltered
    SC_JUDGED,          // survivors judged
    SC_WAVES,           // waves that had work
    SC_COUNT
};
// Returns the number of kernel launches it enqueued.
int launch_sample(const float* coords, float4* coords4, const int* assign32, const Problem& P, uint64_t seed, int max_tries,
                  const int* injected, int inj_T, const SampleState* st, int n_lanes, int sm_count, int use_prefilter,
                  int hyp_offset, int hyp_stride, Pose* poses, int* cells, int* tries, const cudaStream_t* lanes,
                  cudaEvent_t ev_fork, const cudaEvent_t* ev_join, int split_e, const int* perm, const int* offsets,
                  const cudaEvent_t* ev_half, int span0, float window, int n_waves,
                  unsigned long long* trace, float tail_boost, const DevParams* dev = nullptr);
void launch_trace_init(unsigned long long* trace, int slots, cudaStream_t st);

// --- refine.cu ----------------------------------------------------------------------------
// Refines poses_in[jobs[j]] -> poses_out[jobs[j]] for j < *n_jobs (device scalar) or n_jobs_host.
// masks: [job][ceil(N/32)] final inlier bit masks (may be null), rounds: [job] accepted rounds.
struct RefineArgs {
    const float* coords;
    const float* centres;    // [E,3] plane centres (prep kernel)
    const int* assign32;
    const Pose* poses_in;
    Pose* poses_out;
    const int* jobs;
    const int* n_jobs;       // device scalar (null -> n_jobs_host)
    int n_jobs_host;
    uint32_t* masks;
    int mask_words;          // words per job
    int* rounds;
    double* scratch;         // cross-CTA reduction slots
    unsigned int* barrier;   // per group: one epoch flag per block + the root's command flag, zeroed before launch
    int* job_counter;        // next job to hand out (dynamic scheduling), zeroed before launch
    int group;               // CTAs cooperating on one job
    int cache;               // 1: every CTA's share of the map fits the shared-memory cell cache
    int compact;             // 1: LM evaluations walk a per-CTA list of the round's inlier cells
    int pretest;             // 1: the inlier selection classifies clear cases in fp32 (error-bounded), exact arithmetic for the rest
    unsigned short* clist;   // [n_groups][words * 32] inlier lists of blocks whose share does not fit shared memory (or null)
    long long* prof;         // diagnostics: 16 cycle counters of block 0 (null = off)
    Problem P;
    int max_ref_steps;
    DevParams dev;           // dev.shift != null: shift and camera from device memory (stream-ordered forward)
    // group == 0 (with dev): refine_group_kernel picks group = refine_group_rule(N, coresident, group_opt, jobs_per_group,
    // max(1, *n_jobs)) and derives n_groups, cache and clist from it as refine_sizes does; the grid is the largest any group
    // needs, and clist (when not null) has room for any of them.
    int coresident = 0, group_opt = 0, jobs_per_group = 0, max_jobs = 0;
};
void launch_refine(const RefineArgs& a, int n_groups, cudaStream_t st);
int refine_max_coresident_blocks(int sm_count);
int refine_cache_words();
int refine_max_compact_words();
size_t refine_scratch_doubles(int n_groups, int group);
size_t refine_flag_words(int n_groups, int group);
// camera->world 4x4 float of poses[*winner], its expert, flags[0] and the winner into rec (all but rec->rank)
void launch_finish_forward(const Pose* poses, const int* winner, const int* assign32, const int* flags, ForwardRecord* rec,
                           cudaStream_t st);

// Stream-ordered forward: camera->world pose of poses[*winner] (NaN on a bad assignment) into pose16, its expert (-1 on a bad
// assignment) into *expert, flags[0] into *status; advance != 0 adds it to seed[1] (the last image of an execution).
void launch_finish_forward_async(const Pose* poses, const int* winner, const int* assign32, const int* flags, float* pose16,
                                 long long* expert, int* status, unsigned long long* seed, int advance, cudaStream_t st);
// seed[0] = base, seed[1] = 0, stream-ordered
void launch_seed_reset(unsigned long long* seed, unsigned long long base, cudaStream_t st);

void launch_pack_forward(const double* scores, const ForwardRecord* fwd, int M, int M_pad, int expert_offset, int hyp_offset,
                         int hyp_stride, double* pack, cudaStream_t st);
void launch_select_gathered(const double* gathered, int world, int M_pad, ForwardRecord* rec, cudaStream_t st);

// --- gating.cu ----------------------------------------------------------------------------
int assign_max_experts();
void launch_assign(const float* weights, int B, int E, int M, int keep_top, int single, uint64_t seed, int64_t* out_assign,
                   float* out_hist, int* flags, cudaStream_t stream);
// The stream-ordered assignment: the seed read from d_seed on the device, image b's status (0 / 1 / 2) written to out_status[b].
void launch_assign_async(const float* weights, int B, int E, int M, int keep_top, int single, const long long* d_seed,
                         int64_t* out_assign, float* out_hist, int* out_status, cudaStream_t stream);

// --- gate.cu ------------------------------------------------------------------------------
// An expert gate's device side: the arm kernel sets the gate's conditional handles from a histogram on the device, and the
// marker kernel, which does nothing, delimits one region in a captured graph.  The host finds both in the graph by their
// function pointers (gate_arm_fn / gate_mark_fn) and reads their single parameter.
constexpr int kGateMax = 1024;
// What finalize leaves for the arm kernel: until `ready`, nothing; then `count` (index, handle) pairs, one per region.
struct GateTable {
    unsigned long long ready;
    unsigned long long count;
    const unsigned long long* pairs;  // [count][2]: the region's index into counts, its conditional handle
};
struct GateArm {
    unsigned gate;  // the gate's id
    int n;
    const float* counts;       // [n]: the regions of index i run where counts[i] > 0
    const GateTable* table;
};
struct GateTag {
    unsigned gate;  // the gate's id
    int serial;     // the region's serial number on its gate (a begin and its end share it; -1: an end without a begin)
    int index;      // the gate's handle the region runs on
    int begin;      // 1: begin marker, 0: end marker
};
const void* gate_arm_fn();
const void* gate_mark_fn();
void launch_gate_arm(const GateArm& a, cudaStream_t stream);
void launch_gate_mark(const GateTag& t, cudaStream_t stream);

// --- the expert losses' element types -------------------------------------------------------
// The predictions and gradients of one loss call share one element type, the C ABI's dtype code (ESACB200_FLOAT32,
// _FLOAT16, _BFLOAT16); the ground truth is always float32.  The kernels widen every prediction to fp32 and compute exactly
// as on a float32 map, and round each gradient to the element type once, after the optional device-side scale s:
// (g * s) as one fp32 multiply, then round to nearest.
enum LossDtype : int { kLossF32 = 0, kLossF16 = 1, kLossBF16 = 2 };
inline int loss_elem_bytes(int dtype) { return dtype == kLossF32 ? 4 : 2; }

#ifdef __CUDACC__
__device__ __forceinline__ float loss_in(float v) { return v; }
__device__ __forceinline__ float loss_in(__half v) { return __half2float(v); }
__device__ __forceinline__ float loss_in(__nv_bfloat16 v) { return __bfloat162float(v); }
template <class T> __device__ __forceinline__ T loss_out(float v);
template <> __device__ __forceinline__ float loss_out<float>(float v) { return v; }
template <> __device__ __forceinline__ __half loss_out<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 loss_out<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// Four consecutive elements, streamed: one 128-bit access for float, one 64-bit access for the 16-bit types (a warp still
// moves 256 contiguous bytes per plane).
__device__ __forceinline__ float4 loss_ld4(const float* p) { return __ldcs(reinterpret_cast<const float4*>(p)); }
template <class T>
__device__ __forceinline__ float4 loss_ld4(const T* p) {
    union { uint2 u; T e[4]; } v;
    v.u = __ldcs(reinterpret_cast<const uint2*>(p));
    return make_float4(loss_in(v.e[0]), loss_in(v.e[1]), loss_in(v.e[2]), loss_in(v.e[3]));
}
__device__ __forceinline__ void loss_st4(float* p, float a, float b, float c, float d) {
    __stcs(reinterpret_cast<float4*>(p), make_float4(a, b, c, d));
}
template <class T>
__device__ __forceinline__ void loss_st4(T* p, float a, float b, float c, float d) {
    union { uint2 u; T e[4]; } v;
    v.e[0] = loss_out<T>(a); v.e[1] = loss_out<T>(b); v.e[2] = loss_out<T>(c); v.e[3] = loss_out<T>(d);
    __stcs(reinterpret_cast<uint2*>(p), v.u);
}
// The gradient's scale: g * s with round to nearest, never contracted into a neighbouring add.
template <bool SCALE>
__device__ __forceinline__ float loss_scale(float g, float s) { return SCALE ? __fmul_rn(g, s) : g; }
#endif

// --- reproj.cu ----------------------------------------------------------------------------
// Blocks of one image in the loss kernels of reproj.cu and coord_loss.cu: a pure function of its cell count N, so an image
// is cut into the same blocks, and summed in the same order, whatever else is in the batch.
int reproj_blocks_per_image(int N);
// One image of a reprojection-loss launch.  The image's blocks are blockIdx.x < blocks of grid row blockIdx.y; its block
// partials are partial[part0 .. part0 + blocks).  The maps hold elements of the call's dtype.
struct ReprojImage {
    const void* coords;    // [3, H, W]
    void* grads;           // [3, H, W] overwritten, or null (loss only)
    int N, W;              // cells, row pitch
    int b;                 // index in the batch: img record, ticket, loss
    int blocks;            // reproj_blocks_per_image(N)
    long long part0;
};
// Vector loads and stores for this image (4 elements of `esize` bytes per access): N % 4 == 0, W >= 4, planes aligned to
// 4 * esize bytes.
bool reproj_vec_ok(const void* coords, const void* grads, int N, int W, int esize);
// img: per image kReprojImgFloats floats = world->camera 3x4 (row major), padX, padY, f, cx, cy, 3 unused.  recs: n device
// records, all on the load path `vec`; max_blocks = their largest block count.  tickets: zeroed counters per batch image
// (left zeroed), losses: a double per batch image.  dtype: the maps' LossDtype; grad_scale: a device float that scales
// every gradient, or null (float32 always null).
constexpr int kReprojImgFloats = 20;
void launch_reproj(bool vec, int dtype, const ReprojImage* recs, int n, int max_blocks, const float* img, float sub, float cut,
                   float max_err, float min_depth, const float* grad_scale, double* partial, unsigned* tickets, double* losses,
                   cudaStream_t stream);

// fp64 products and sums rounded once each, on both sides: nvcc would contract a*b - c*d into an FMA, the host compiler
// (no -march) does not, and the reprojection loss's ground-truth inversion must round alike on the host and the device.
ESAC_HD double mul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
ESAC_HD double add_rn(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
ESAC_HD double sub_rn(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
ESAC_HD double div_rn(double a, double b) {
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

// One image's row of the reprojection loss's `img` table (kReprojImgFloats floats): the world->camera 3x4 inverse of the
// affine camera->world ground truth T [4,4] (torch's .inverse()[0:3,:], ref_expert.py:127; adjugate over determinant),
// then padX, padY, f, cx, cy.  Returns false, with o untouched, when the rotation block is singular or NaN (det == 0 or
// det != det).  The eager call runs it on the host, the stream-ordered call on the device: bitwise the same row.
ESAC_HD bool reproj_img_row(const float* T, int padX, int padY, float f, float cx, float cy, float* o) {
    double A[9], inv[9];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) A[r * 3 + c] = T[r * 4 + c];
    // cofactor (i,j,k,l) = A[i] * A[j] - A[k] * A[l]
    auto cof = [&](int i, int j, int k, int l) { return sub_rn(mul_rn(A[i], A[j]), mul_rn(A[k], A[l])); };
    const double det = add_rn(sub_rn(mul_rn(A[0], cof(4, 8, 5, 7)), mul_rn(A[1], cof(3, 8, 5, 6))), mul_rn(A[2], cof(3, 7, 4, 6)));
    if (det == 0. || !(det == det)) return false;
    inv[0] = div_rn(cof(4, 8, 5, 7), det); inv[1] = div_rn(cof(2, 7, 1, 8), det); inv[2] = div_rn(cof(1, 5, 2, 4), det);
    inv[3] = div_rn(cof(5, 6, 3, 8), det); inv[4] = div_rn(cof(0, 8, 2, 6), det); inv[5] = div_rn(cof(2, 3, 0, 5), det);
    inv[6] = div_rn(cof(3, 7, 4, 6), det); inv[7] = div_rn(cof(1, 6, 0, 7), det); inv[8] = div_rn(cof(0, 4, 1, 3), det);
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) o[r * 4 + c] = (float)inv[r * 3 + c];
        const double t = add_rn(add_rn(mul_rn(inv[r * 3], T[3]), mul_rn(inv[r * 3 + 1], T[7])), mul_rn(inv[r * 3 + 2], T[11]));
        o[r * 4 + 3] = (float)-t;
    }
    o[12] = (float)padX;
    o[13] = (float)padY;
    o[14] = f;
    o[15] = cx;
    o[16] = cy;
    return true;
}

// --- coord_loss.cu ------------------------------------------------------------------------
// One image of a coordinate-loss launch: pred [3,Hp,Wp], gt [3,Hg,Wg] (|Hp-Hg|, |Wp-Wg| <= 1, checked by the caller),
// grads [3,Hp,Wp] overwritten or null (loss only).  blocks = reproj_blocks_per_image(Np), partials part0 .. part0 + blocks
// (2 doubles each), as for ReprojImage.  pred and grads hold elements of the call's dtype, gt float32.
struct CoordImage {
    const void* pred;
    const float* gt;
    void* grads;
    int Np, Ng;   // plane sizes of the prediction / the ground truth (Hp*Wp, Hg*Wg)
    int Wp, Wg;   // their row pitches
    int H, W;     // the common top-left window
    int N;        // H*W
    int b;        // index in the batch: counter, ticket, loss
    int blocks;
    int pad;
    long long part0;
};
// Fills the geometry of r from the two sizes and picks the load path: vector loads when the row pitches are equal (the
// window is then the first N cells of every plane), N, Np, Ng % 4 == 0, the ground truth's planes are 16-byte aligned and
// the prediction's and gradient's planes are aligned to 4 * esize bytes.
bool coord_image(CoordImage& r, int Hp, int Wp, int Hg, int Wg, int esize);
// Both passes run on a (max_blocks, n) grid of 256-thread blocks, 4 cells per thread, as the reprojection loss; recs: n
// device records on load path `vec`.  counts: a zeroed counter per batch image (gradient only), tickets: zeroed counters
// (left zeroed), losses / out_counts: per batch image.  pass 1 = count pass (gradient only), 2 = loss pass.  dtype and
// grad_scale as for launch_reproj.
void launch_coord_loss(bool vec, int pass, bool grad, int dtype, const CoordImage* recs, int n, int max_blocks, float cut,
                       const float* grad_scale, unsigned* counts, double* partial, unsigned* tickets, double* losses,
                       long long* out_counts, cudaStream_t stream);
// The largest reproj_blocks_per_image(n) over n <= N (the count is not monotonic in N): the partials that a workspace for
// maps of at most N cells must hold per image.
int reproj_max_blocks(int N);

// --- loss_async.cu ------------------------------------------------------------------------
// Records per prep-kernel launch of the stream-ordered losses: they travel as a kernel parameter, under the 4 KB limit.
constexpr size_t kLossChunkBytes = 3072;
template <class Rec> constexpr int loss_chunk() { return (int)(kLossChunkBytes / sizeof(Rec)); }
// The n host records (ordered by load path) into recs, in chunks; record i's image b gets its row of img from gt16 [B,4,4]
// camera->world, shifts [B,2] and cameras [B,3] (device), and bad[b] = 1 (and no blocks) when its rotation block is
// singular or NaN.  Returns the launches.
int launch_reproj_prep(const ReprojImage* host_recs, int n, ReprojImage* recs, const float* gt16, const int* shifts,
                       const float* cameras, float* img, int* bad, cudaStream_t st);
// out_losses[b] = losses[b] (NaN when bad[b]), status[b] = bad[b], and the gradient of a bad image zeroed (grads: the call
// has gradients; a zero of the call's dtype, scaled by grad_scale as the loss kernel scales every gradient).  recs: the B
// device records.
void launch_reproj_finish(const ReprojImage* recs, int B, bool grads, int dtype, const float* grad_scale, const double* losses,
                          const int* bad, double* out_losses, int* status, cudaStream_t st);
// The n host records into recs, in chunks.  Returns the launches.
int launch_coord_prep(const CoordImage* host_recs, int n, CoordImage* recs, cudaStream_t st);
// out_losses[b] = losses[b], out_counts[b] = counts[b] (out_counts may be null).
void launch_coord_finish(int B, const double* losses, const long long* counts, double* out_losses, long long* out_counts,
                         cudaStream_t st);

// --- bwd.cu -------------------------------------------------------------------------------
struct BwdArgs {
    const float* coords;
    float* grads;            // [E,3,N] accumulated in place
    const int* assign32;
    const int* perm;         // slot -> hyp
    const int* counts;
    const int* offsets;
    const Pose* init;        // [M]
    const Pose* ref;         // [M] (== init for non-contributing)
    const int* cells;        // [M,4,2]
    const double* probs;     // [M]
    const int* contrib;      // contributing hypothesis ids (ascending)
    const int* n_contrib;    // device scalar
    const int* job_of;       // [M] hypothesis -> job index (or -1)
    const uint32_t* masks;
    int mask_words;
    const int* rounds;       // [job]
    double* losses;          // [M]
    double* out_loss;        // device scalar: expected loss
    double* red;             // [job][tiles][kRedVals] partial reductions
    void* hyp_grad;          // [job] HypGrad records
    float gt[16];
    float wRot, wTrans, cut;
    Problem P;
    const double* expected_override;  // device scalar: global expected loss (multi-GPU), or null
};
// What B1-B5 of the stream-ordered backward (esacb200_backward_async) read from device memory.  The kernels take it as their
// last argument, so the arguments of the eager instantiations keep their places.
struct BwdDev {
    const float* gt = nullptr;   // [4,4] camera->world ground truth (B1), instead of BwdArgs::gt
    const int* flags = nullptr;  // the prep kernel's bad-assignment flag: B5 leaves the gradient untouched when it is set
    DevParams dev;               // shift and camera
    // The stream-ordered hypotheses backward: the forward's problem in the tape header, whose sub, tau, alpha, beta and
    // maxReproj B2-B5 use instead of BwdArgs::P's (the call does not take them); null: BwdArgs::P's.
    const Problem* prob = nullptr;
};
// dev: non-null -> the stream-ordered instantiations, which read *dev
void launch_backward(const BwdArgs& a, int max_jobs, int sm_count, cudaStream_t st, const BwdDev* dev = nullptr);
// Stream-ordered backward: the expected loss stats->local_loss (NaN on a bad assignment) into *loss, flags[0] into *status;
// advance != 0 adds it to seed[1] (the last image of an execution).
void launch_finish_backward_async(const CallStats* stats, const int* flags, double* loss, int* status, unsigned long long* seed,
                                  int advance, cudaStream_t st);
// phase split for the multi-GPU path: losses + local expectation only / everything after the loss exchange
void launch_backward_losses(const BwdArgs& a, cudaStream_t st);
void launch_add_inplace(float* dst, const float* src, size_t n, cudaStream_t st);
void launch_expert_flags(const int* contrib, const int* n_contrib, const int* assign32, int E, int* flags, cudaStream_t st);
size_t bwd_hypgrad_bytes();
int bwd_red_vals();
int bwd_tiles(int N);

// State a hypotheses forward leaves for its backward, in one caller-owned device buffer (the tape):
//   [TapeHead, kTapeHeadBytes] [M per-job records, bwd_hypgrad_bytes() each] [M jobs x 2 x ceil(N/32) words of inlier masks]
// Job j's final inliers are mask (2j + its refinement buffer), the layout the refinement writes and B2-B5 read.
struct TapeHead {
    unsigned magic;
    int n_contrib;  // written on the device by the forward
    int M, mask_words;
    Problem P;
    double min_prob;  // the forward's probability floor: its records are the hypotheses with !(p < min_prob)
};
constexpr unsigned kTapeMagic = 0x45534831u;  // "ESH1"
constexpr size_t kTapeHeadBytes = 256;
// Header fields behind TapeHead (still inside the kTapeHeadBytes): bad = 1 when the forward's assignment held an expert index
// outside [0, E) (stream-ordered forward; the eager forward fails instead and writes 0).
struct TapeTail {
    int bad;
};
constexpr size_t kTapeTailOffset = (sizeof(TapeHead) + 15) & ~(size_t)15;
static_assert(kTapeTailOffset + sizeof(TapeTail) <= kTapeHeadBytes, "the tape header holds TapeHead and TapeTail");
size_t tape_records_offset();
size_t tape_masks_offset(int M);
size_t tape_bytes(int M, int N);
// records, header and per-hypothesis contributing flags [M] from a (init, ref, cells, rounds, contrib, n_contrib, assign32)
void launch_tape_records(const BwdArgs& a, const TapeHead& head, void* tape, unsigned char* contrib_flags, cudaStream_t st);
// the tape's records with dl = d_poses6[h], g = d_scores[h], p = 1 (device arrays of M), then B2-B5 into a.grads
void launch_backward_upstream(const BwdArgs& a, const void* tape, const double* d_scores, const double* d_poses6, int max_jobs,
                              int sm_count, cudaStream_t st);

// Stream-ordered hypotheses forward (esacb200_hypotheses_forward_async): what the record kernel reads from and writes to
// device memory besides the eager kernel's arguments.
struct TapeDev {
    DevParams dev;                   // the shift and camera the forward used (written into the header)
    const int* flags = nullptr;      // the prep kernel's bad-assignment flag
    const double* scores = nullptr;  // [M] the workspace's scores
    const Pose* poses = nullptr;     // [M] the workspace's refined poses
    double* out_scores = nullptr;    // [M] the caller's row (NaN on a bad assignment)
    double* out_poses6 = nullptr;    // [M,6] the caller's row (NaN on a bad assignment)
    int* status = nullptr;           // 0 or 1
    unsigned long long* seed = nullptr;  // the async call counter seed[1], advanced by `advance`
    int advance = 0;
};
// records, header (its shift and camera from td.dev), contributing flags straight into the caller's row, scores, poses and
// status; on a bad assignment no records, n_contrib = 0 and TapeTail::bad = 1.
void launch_tape_records_async(const BwdArgs& a, const TapeHead& head, void* tape, unsigned char* contrib_flags, const TapeDev& td,
                               cudaStream_t st);
// Stream-ordered hypotheses backward (esacb200_hypotheses_backward_async): checks the tape header on the device against
// a.P's E, H, W and M, publishes the job count into *count (a.n_contrib must point there) and the skip flag into *skip
// (dv.flags), writes *status (0, 1 = bad assignment in the forward, 2 = not a tape of this problem), then B2-B5 with
// dv.dev / dv.prob pointing into the header.  d_scores / d_poses6 null: zero.
void launch_backward_upstream_async(const BwdArgs& a, const void* tape, const double* d_scores, const double* d_poses6, int* count,
                                    int* skip, int* status, const BwdDev& dv, int max_jobs, int sm_count, cudaStream_t st);
// loss / dLoss of [B,M] scene poses, image b against camera->world ground truth gt16[b] (device [B,4,4]); outputs [B,M], [B,M,6]
void launch_pose_loss(const Pose* poses, int B, int M, const float* gt16, float wRot, float wTrans, float cut, double* losses,
                      double* dloss6, cudaStream_t st);

// --- eval.cu ------------------------------------------------------------------------------
// One test image's evaluation (test_esac.py:209-247), the row a pose evaluation writes into the caller's record buffer; all
// fp64 (include/esac_b200.h documents the row).  Integers are stored exactly; `active` is NaN when the call has no histogram.
struct EvalRecord {
    double rot_deg;   // rotation error, degrees (exactly 0 in OpenCV's s < 1e-5, c > 0 branch)
    double trans_cm;  // translation error, centimetres
    double correct;   // 1 when expert == scene
    double scene;     // ground-truth scene (expert) index
    double expert;    // the winning expert
    double status;    // the forward's status (0 = counted)
    double active;    // experts that drew a hypothesis
    double q[4];      // qw qx qy qz of the inverted estimate (q_xyz NaN at angle 0, as the reference writes it)
    double t[3];      // tx ty tz of the inverted estimate
};
constexpr int kEvalRecordDoubles = sizeof(EvalRecord) / sizeof(double);
static_assert(kEvalRecordDoubles == 14, "EvalRecord is the 14 doubles include/esac_b200.h documents");
// The record store's device state: rows written so far (slots handed out, including those past the capacity), a flag set
// when a slot fell past the capacity, and the CTA ticket of the launch in flight (zero between launches).
struct EvalState {
    unsigned long long count, overflow, ticket, unused;
};
static_assert(sizeof(EvalState) == 4 * sizeof(long long), "EvalState is 4 int64");
struct EvalArgs {
    const float* out_poses;       // [B,4,4] camera->world estimates
    const float* gt_poses;        // [B,4,4] camera->world ground truths
    const long long* experts;     // [B] winning experts
    const long long* scenes;      // [B] ground-truth scenes
    const float* hist;            // [B,E] hypothesis histogram, or null
    const int* status;            // [B] forward status, or null (0)
    int B, E;
    EvalRecord* records;          // [capacity]
    long long capacity;
    EvalState* state;
};
// Image b of the call goes to slot state->count + b; the launch's last CTA advances count by B.
void launch_eval_poses(const EvalArgs& a, cudaStream_t st);

// --- cluster.cu ---------------------------------------------------------------------------
// Clustering a large environment into experts (cluster_dataset.py:19-140, 219-240).
struct ClusterMap {
    const float* p;  // [3,H,W] ground-truth scene coordinates, device memory
    int H, W;
};
// One map's statistics over its valid cells ((x + y) + z != 0 in float32): lower median and mean per coordinate.
struct ClusterStats {
    float median[3], mean[3];
    int count;   // valid cells
    int status;  // 0 ok, 1 no valid cell, 2 a non-finite median or mean
};
static_assert(sizeof(ClusterStats) == 32, "ClusterStats is 32 bytes");
constexpr int kStatsThreads = 256;
constexpr int kStatsSmemKeys = 8192;  // valid cells per coordinate selected in shared memory; more: from global memory
// One CTA per map; `cap` keys per coordinate of dynamic shared memory (3 * cap * 4 bytes).
void launch_cluster_stats(const ClusterMap* maps, int B, int cap, ClusterStats* out, cudaStream_t st);

// One k-means attempt's result: its fp64 centres, the compactness of its final assignment, and the point its final
// assignment moved into an emptied cluster (-1: none).
struct KmeansAttempt {
    double centre[2][3];
    double compactness;
    int reseed, reseed_label;
};
struct KmeansArgs {
    const float* points;  // [n,3]
    int n, attempts, max_iter;
    double eps2;          // stop when the largest squared centre shift is <= eps2
    unsigned long long seed;
    unsigned split;
    KmeansAttempt* att;   // [attempts] workspace
    int* labels;          // [n] the best attempt's labels
    float* centres;       // [2,3]
    double* compactness;  // [1]
};
constexpr int kKmeansThreads = 256;  // the reduction tree of every k-means sum (oracle/cluster_oracle.py restates it)
// One CTA per attempt, then one pass that picks the best attempt and writes its labels, centres and compactness.
void launch_kmeans2(const KmeansArgs& a, cudaStream_t st);

struct ClusterTargetsArgs {
    const float* means;      // [N,3] image means
    const long long* labels; // [N] in [0, K), every cluster non-empty
    int N, K;
    float softness;
    float* centres;          // [K,3]
    float* sizes;            // [K]
    float* probs;            // [N,K]
};
constexpr int kTargetsMaxClusters = 1024;
void launch_cluster_targets(const ClusterTargetsArgs& a, cudaStream_t st);

// --- render.cu ----------------------------------------------------------------------------
// Ground-truth scene-coordinate maps from an SfM reconstruction (setup_aachen.py:184-202, setup_dubrovnik.py:171-190).
struct RenderCamera {
    float pose[12];        // world -> camera, rows 0-2 of the 4x4, row-major
    float f, scale;        // focal length and out_w / image width, as float32
    float half_w, half_h;  // w / 2, h / 2 of the out map
    int H, W;
    int cell0;             // first cell of this camera in the packed cell numbering (cells of camera c: [cell0, cell0 + H*W))
    int pad;
};
static_assert(sizeof(RenderCamera) == 80, "RenderCamera is 80 bytes");
// Per-camera status bits.
enum { kRenderBadIndex = 1, kRenderNaN = 2 };
struct RenderArgs {
    const float* points;     // [P,3]
    const int* indices;      // [V] point of each observation; camera c owns [offsets[c], offsets[c+1])
    const int* offsets;      // [C+1]
    const RenderCamera* cams;  // [C]
    int C, P, V, cells;      // cells: the sum of H*W over the cameras
    // workspace
    int* obs_cell;           // [V] the cell of each observation, -1 when it takes no part
    float* obs_z;            // [V] its camera-space depth
    unsigned* first_neg;     // [cells] first observation with a negative depth (0xFFFFFFFF: none)
    int* last_zero;          // [cells] last observation with depth +-0 before first_neg (-1: none)
    unsigned long long* key; // [cells] min of (order-preserving depth << 32 | observation) after last_zero
    // outputs
    float* maps;             // camera c: [3,H,W] at 3 * cell0
    float* zbuf;             // camera c: [H,W] at cell0 (may be null)
    int* count;              // [C] cells written
    int* status;             // [C] kRender* bits
};
// Clears the per-cell workspace and the counters, then the four passes; the caller synchronises.
void launch_render(const RenderArgs& a, cudaStream_t st);

}  // namespace esacb200
