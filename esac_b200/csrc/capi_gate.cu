// Expert gates and the stream-ordered hypothesis assignment (include/esac_b200.h): what lets a captured ESAC step run only
// the experts that drew hypotheses, as the reference's loops do.
//
// A gate is armed and its regions are marked while a stream is captured; esacb200_gate_finalize then moves each region
// into the body of an IF conditional node on the gate's handle for it.  Finalize validates every region before it edits
// anything, so a graph it refuses is left as it was captured (its markers are empty kernels: it still runs every region).
// The conditional handles are created by finalize, after it has extracted the regions (cudaGraphClone refuses a graph
// that owns conditional handles), one per region (a handle drives one conditional node), and reach the arm kernel through
// the gate's device table, whose ready flag finalize sets last: until then, and for ever in a refused graph, the arm
// kernel does nothing.
#include <cuda_runtime.h>
#include <stdio.h>

#include <atomic>
#include <set>
#include <unordered_map>
#include <utility>
#include <vector>

#include "capi_internal.h"

using namespace esacb200;
using namespace esacb200::capi;

struct esacb200_gate {
    esacb200_ctx* ctx = nullptr;
    int device = 0;                           // the context's: the gate may outlive its context object
    int n = 0;
    unsigned id = 0;                          // in every arm and marker kernel's parameter: tells this gate's nodes apart
    unsigned long long armed_capture = 0;     // the capture sequence the gate was last armed in (0: none)
    unsigned long long mark_capture = 0;      // the capture sequence of the last marker
    std::vector<std::pair<int, int>> open;    // (serial, index) of the regions begun and not yet ended in mark_capture
    int next_serial = 0;
    DevBuf table;                             // GateTable
    DevBuf pairs;                             // its (index, handle) pairs, one per region
};

namespace {

std::atomic<unsigned> next_gate_id{1};

int check_driver(esacb200_ctx* ctx) {
    int v = 0;
    if (cudaDriverGetVersion(&v) != cudaSuccess) {
        cudaGetLastError();
        v = 0;
    }
    if (v < 12030)
        return fail(ctx, ESACB200_ERR_CUDA, "expert gates need conditional graph nodes, which need a CUDA 12.3 driver or newer "
                    "(this driver supports CUDA %d.%d)", v / 1000, v % 1000 / 10);
    return 0;
}

// The type of a graph node, from the driver (the runtime's getter fails on the nodes of a graph that holds conditional
// nodes); -1 where neither answers.
int node_type(cudaGraphNode_t node) {
    typedef int (*GetType)(cudaGraphNode_t, int*);
    static GetType drv = [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuGraphNodeGetType", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
            cudaGetLastError();
            f = nullptr;
        }
        return (GetType)f;
    }();
    int t = -1;
    if (drv && drv(node, &t) == 0) return t;
    cudaGraphNodeType rt;
    if (cudaGraphNodeGetType(node, &rt) == cudaSuccess) return (int)rt;
    cudaGetLastError();
    return -1;
}

// A failed CUDA call of the gate's host code: its error is reported here, and cleared, so that the caller's next CUDA check
// does not find it.
int gate_fail(esacb200_ctx* ctx, cudaError_t e, const char* what) {
    cudaGetLastError();
    return fail(ctx, ESACB200_ERR_CUDA, "%s failed: %s", what, cudaGetErrorString(e));
}

// The capture sequence `s` belongs to, and its graph; fails unless `s` is being captured.
int capture_of(esacb200_ctx* ctx, cudaStream_t s, const char* what, unsigned long long& id, cudaGraph_t& graph) {
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    cudaError_t e = cudaStreamGetCaptureInfo(s, &st, &id, &graph);
    if (e != cudaSuccess) return gate_fail(ctx, e, "cudaStreamGetCaptureInfo");
    if (st != cudaStreamCaptureStatusActive) return fail(ctx, ESACB200_ERR_ARG, "%s works only while the stream is being captured", what);
    return 0;
}

const char* type_name(cudaGraphNodeType t) {
    switch (t) {
        case cudaGraphNodeTypeKernel: return "kernel";
        case cudaGraphNodeTypeMemcpy: return "memcpy";
        case cudaGraphNodeTypeMemset: return "memset";
        case cudaGraphNodeTypeHost: return "host";
        case cudaGraphNodeTypeGraph: return "child graph";
        case cudaGraphNodeTypeEmpty: return "empty";
        case cudaGraphNodeTypeWaitEvent: return "event wait";
        case cudaGraphNodeTypeEventRecord: return "event record";
        case cudaGraphNodeTypeExtSemaphoreSignal: return "external semaphore signal";
        case cudaGraphNodeTypeExtSemaphoreWait: return "external semaphore wait";
        case cudaGraphNodeTypeMemAlloc: return "memory allocation";
        case cudaGraphNodeTypeMemFree: return "memory free";
        case cudaGraphNodeTypeConditional: return "conditional";
        default: return "unknown";
    }
}

// A memcpy node a conditional body can hold: device memory on both sides.
bool device_memcpy(cudaGraphNode_t node) {
    cudaMemcpy3DParms p = {};
    if (cudaGraphMemcpyNodeGetParams(node, &p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    if (p.kind == cudaMemcpyHostToDevice || p.kind == cudaMemcpyDeviceToHost || p.kind == cudaMemcpyHostToHost) return false;
    return (p.srcArray || is_device_ptr(p.srcPtr.ptr)) && (p.dstArray || is_device_ptr(p.dstPtr.ptr));
}

// Whether `body` fits into the body of an IF conditional node: tried on a scratch graph of its own, so the caller's graph
// gets no handle and no node.
cudaError_t fits_conditional(cudaGraph_t body) {
    cudaGraph_t scratch = nullptr;
    cudaError_t e = cudaGraphCreate(&scratch, 0);
    if (e != cudaSuccess) return e;
    cudaGraphConditionalHandle h = 0;
    e = cudaGraphConditionalHandleCreate(&h, scratch, 0, cudaGraphCondAssignDefault);
    cudaGraphNodeParams p = {};
    p.type = cudaGraphNodeTypeConditional;
    p.conditional.handle = h;
    p.conditional.type = cudaGraphCondTypeIf;
    p.conditional.size = 1;
    cudaGraphNode_t cond = nullptr, child = nullptr;
    if (e == cudaSuccess) e = cudaGraphAddNode(&cond, scratch, nullptr, 0, &p);
    if (e == cudaSuccess) e = cudaGraphAddChildGraphNode(&child, p.conditional.phGraph_out[0], nullptr, 0, body);
    cudaGetLastError();
    cudaGraphDestroy(scratch);
    return e;
}

// A copy of `graph` that keeps only the nodes with keep[v] != 0 (nodes[v] in `graph`), with their parameters, attributes and
// the edges among them.
cudaError_t extract(cudaGraph_t graph, const std::vector<cudaGraphNode_t>& nodes, const std::vector<char>& keep,
                    cudaGraph_t* out, const char** step) {
    *out = nullptr;
    *step = "cudaGraphClone";
    cudaError_t e = cudaGraphClone(out, graph);
    for (size_t v = 0; v < nodes.size() && e == cudaSuccess; ++v) {
        if (keep[v]) continue;
        cudaGraphNode_t c = nullptr;
        *step = "cudaGraphNodeFindInClone";
        e = cudaGraphNodeFindInClone(&c, nodes[v], *out);
        *step = "cudaGraphDestroyNode";
        if (e == cudaSuccess) e = cudaGraphDestroyNode(c);
    }
    if (e != cudaSuccess) {
        cudaGetLastError();
        if (*out) cudaGraphDestroy(*out);
        *out = nullptr;
    }
    return e;
}

struct Region {
    int serial = -1, index = -1, end_index = -1;
    int b = -1, e = -1;           // node indices of the begin and end markers
    std::vector<char> in;         // membership, by node index
    std::vector<int> nodes;       // the members, markers included
};

// Marks every node reachable from `from` along `adj` (from itself excluded) in `seen`.
void reach(int from, const std::vector<std::vector<int>>& adj, std::vector<char>& seen) {
    std::vector<int> stack(adj[from].begin(), adj[from].end());
    while (!stack.empty()) {
        const int v = stack.back();
        stack.pop_back();
        if (seen[v]) continue;
        seen[v] = 1;
        for (int w : adj[v]) if (!seen[w]) stack.push_back(w);
    }
}

}  // namespace

extern "C" {

int esacb200_assign_hypotheses_async(esacb200_ctx* ctx, int B, int E, int M, const float* weights, int keep_top,
                                     int single_expert, const int64_t* seed, int64_t* out_assign, float* out_hist,
                                     int* out_status) try {
    if (!ctx) return ESACB200_ERR_ARG;
    DeviceGuard device_guard(ctx->device);
    if (B <= 0 || E <= 0 || M <= 0) return fail(ctx, ESACB200_ERR_ARG, "assign_hypotheses_async: bad sizes B=%d E=%d M=%d", B, E, M);
    if (E > assign_max_experts())
        return fail(ctx, ESACB200_ERR_ARG, "assign_hypotheses_async: E=%d exceeds the %d experts one CTA holds", E, assign_max_experts());
    const void* ptrs[] = {weights, seed, out_assign, out_hist, out_status};
    const char* names[] = {"weights", "seed", "out_assign", "out_hist", "out_status"};
    int rc = device_args(ctx, "assign_hypotheses_async", 5, ptrs, names, 1u << 3);
    if (rc) return rc;
    launch_assign_async(weights, B, E, M, keep_top, single_expert, (const long long*)seed, out_assign, out_hist, out_status,
                        ctx->stream);
    CK(cudaGetLastError());
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

int esacb200_gate_create(esacb200_ctx* ctx, int n, esacb200_gate** out) try {
    if (!ctx || !out) return ESACB200_ERR_ARG;
    *out = nullptr;
    if (n < 1 || n > ESACB200_GATE_MAX) return fail(ctx, ESACB200_ERR_ARG, "gate_create: n=%d outside [1, %d]", n, ESACB200_GATE_MAX);
    int rc = check_driver(ctx);
    if (rc) return rc;
    DeviceGuard device_guard(ctx->device);
    esacb200_gate* g = new esacb200_gate();
    g->ctx = ctx;
    g->device = ctx->device;
    g->n = n;
    g->id = next_gate_id.fetch_add(1);
    cudaError_t e = g->table.ensure(sizeof(GateTable));
    if (e == cudaSuccess) e = cudaMemset(g->table.p, 0, sizeof(GateTable));
    if (e != cudaSuccess) {
        delete g;
        return gate_fail(ctx, e, "gate_create: the handle table");
    }
    *out = g;
    return ESACB200_OK;
} ESAC_ABI_CATCH(ctx)

void esacb200_gate_destroy(esacb200_gate* gate) {
    if (!gate) return;
    DeviceGuard device_guard(gate->device);
    delete gate;
}

int esacb200_gate_arm(esacb200_gate* gate, const float* counts, void* stream) try {
    if (!gate) return ESACB200_ERR_ARG;
    esacb200_ctx* ctx = gate->ctx;
    if (!counts) return fail(ctx, ESACB200_ERR_ARG, "gate_arm: counts is null");
    DeviceGuard device_guard(ctx->device);
    if (!is_device_ptr(counts)) return fail(ctx, ESACB200_ERR_ARG, "gate_arm takes device pointers only: counts is host memory");
    unsigned long long id = 0;
    cudaGraph_t graph = nullptr;
    int rc = capture_of(ctx, (cudaStream_t)stream, "gate_arm", id, graph);
    if (rc) return rc;
    if (gate->armed_capture == id) return fail(ctx, ESACB200_ERR_ARG, "gate_arm: the gate is already armed in this graph");
    if (gate->armed_capture)
        return fail(ctx, ESACB200_ERR_ARG, "gate_arm: the gate is armed in another graph already (a gate serves one graph)");
    const GateArm a = {gate->id, gate->n, counts, gate->table.as<const GateTable>()};
    launch_gate_arm(a, (cudaStream_t)stream);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return gate_fail(ctx, e, "gate_arm: the arm kernel's launch");
    gate->armed_capture = id;
    return ESACB200_OK;
} ESAC_ABI_CATCH(gate->ctx)

int esacb200_gate_mark(esacb200_gate* gate, int index, int begin, void* stream) try {
    if (!gate) return ESACB200_ERR_ARG;
    esacb200_ctx* ctx = gate->ctx;
    if (index < 0 || index >= gate->n) return fail(ctx, ESACB200_ERR_ARG, "gate_mark: index %d outside [0, %d)", index, gate->n);
    DeviceGuard device_guard(ctx->device);
    unsigned long long id = 0;
    cudaGraph_t graph = nullptr;
    int rc = capture_of(ctx, (cudaStream_t)stream, "gate_mark", id, graph);
    if (rc) return rc;
    if (id != gate->mark_capture) {  // a new capture: whatever an earlier one left open is not this graph's
        gate->open.clear();
        gate->mark_capture = id;
    }
    GateTag t = {gate->id, -1, index, begin ? 1 : 0};
    if (begin) {
        t.serial = gate->next_serial++;
        gate->open.emplace_back(t.serial, index);
    } else if (!gate->open.empty()) {
        t.serial = gate->open.back().first;
        gate->open.pop_back();
    }
    launch_gate_mark(t, (cudaStream_t)stream);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return gate_fail(ctx, e, "gate_mark: the marker's launch");
    return ESACB200_OK;
} ESAC_ABI_CATCH(gate->ctx)

int esacb200_gate_finalize(esacb200_gate* gate, void* graph_ptr) try {
    if (!gate) return ESACB200_ERR_ARG;
    esacb200_ctx* ctx = gate->ctx;
    if (!graph_ptr) return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: graph is null");
    DeviceGuard device_guard(ctx->device);
    cudaGraph_t graph = (cudaGraph_t)graph_ptr;

    // ---- the graph: nodes, edges, the gate's arm node and markers
#define GK(call)                                              \
    do {                                                      \
        cudaError_t e__ = (call);                             \
        if (e__ != cudaSuccess) return gate_fail(ctx, e__, "gate_finalize: " #call); \
    } while (0)
    size_t nn = 0, ne = 0;
    GK(cudaGraphGetNodes(graph, nullptr, &nn));
    std::vector<cudaGraphNode_t> nodes(nn);
    if (nn) GK(cudaGraphGetNodes(graph, nodes.data(), &nn));
    GK(cudaGraphGetEdges_v2(graph, nullptr, nullptr, nullptr, &ne));
    std::vector<cudaGraphNode_t> from(ne), to(ne);
    std::vector<cudaGraphEdgeData> edata(ne);
    if (ne) GK(cudaGraphGetEdges_v2(graph, from.data(), to.data(), edata.data(), &ne));
    std::unordered_map<cudaGraphNode_t, int> at;
    for (size_t i = 0; i < nn; ++i) at[nodes[i]] = (int)i;
    std::vector<std::vector<int>> preds(nn), succs(nn);
    for (size_t k = 0; k < ne; ++k) {
        const int u = at.at(from[k]), v = at.at(to[k]);
        succs[u].push_back(v);
        preds[v].push_back(u);
    }
    std::vector<cudaGraphNodeType> type(nn);
    int arm = -1, arms = 0, armed_n = 0;
    std::vector<Region> regions;
    std::unordered_map<int, int> by_serial;
    int stray_end = -1;  // an end marker with no begin (its index)
    for (size_t i = 0; i < nn; ++i) {
        type[i] = (cudaGraphNodeType)node_type(nodes[i]);
        if (type[i] != cudaGraphNodeTypeKernel) continue;
        cudaKernelNodeParams kp = {};
        if (cudaGraphKernelNodeGetParams(nodes[i], &kp) != cudaSuccess) {  // e.g. a library's driver-API kernel: not ours
            cudaGetLastError();
            continue;
        }
        if (kp.func == gate_arm_fn() && kp.kernelParams) {
            const GateArm& a = *(const GateArm*)kp.kernelParams[0];
            if (a.gate != gate->id) continue;
            arm = (int)i;
            ++arms;
            armed_n = a.n;
        } else if (kp.func == gate_mark_fn() && kp.kernelParams) {
            const GateTag t = *(const GateTag*)kp.kernelParams[0];
            if (t.gate != gate->id) continue;
            if (t.serial < 0) {
                stray_end = t.index;
                continue;
            }
            auto it = by_serial.find(t.serial);
            if (it == by_serial.end()) {
                it = by_serial.emplace(t.serial, (int)regions.size()).first;
                regions.emplace_back();
                regions.back().serial = t.serial;
            }
            Region& r = regions[it->second];
            if (t.begin) {
                r.b = (int)i;
                r.index = t.index;
            } else {
                r.e = (int)i;
                r.end_index = t.index;
            }
        }
    }

    // ---- validate everything before the first edit
    if (stray_end >= 0) return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: an end marker of index %d has no begin marker", stray_end);
    if (regions.empty())
        return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: the graph holds no region of this gate (captured without one, or "
                    "already finalized)");
    for (const Region& r : regions) {
        if (r.b < 0) return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: region %d (index %d) has no begin marker in this graph", r.serial, r.end_index);
        if (r.e < 0) return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: region %d (index %d) has no end marker", r.serial, r.index);
        if (r.index != r.end_index)
            return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: region %d begins on index %d and ends on index %d", r.serial, r.index, r.end_index);
    }
    if (arms == 0) return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: region %d (index %d): the gate was not armed in this graph", regions[0].serial, regions[0].index);
    if (arms > 1) return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: the gate is armed %d times in this graph", arms);
    if (armed_n != gate->n) return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: the graph's arm node holds %d switches, the gate %d", armed_n, gate->n);
    std::vector<int> owner(nn, -1);
    for (size_t ri = 0; ri < regions.size(); ++ri) {
        Region& r = regions[ri];
        std::vector<char> desc_b(nn, 0), anc_e(nn, 0), anc_b(nn, 0), desc_e(nn, 0);
        reach(r.b, succs, desc_b);
        reach(r.e, preds, anc_e);
        reach(r.b, preds, anc_b);
        reach(r.e, succs, desc_e);
        if (!desc_b[r.e])
            return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: region %d (index %d): its end marker does not follow its begin "
                        "marker (the region crosses streams)", r.serial, r.index);
        if (!anc_b[arm])
            return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: region %d (index %d): the gate is not armed upstream of the region",
                        r.serial, r.index);
        r.in.assign(nn, 0);
        for (size_t v = 0; v < nn; ++v)
            if ((int)v == r.b || (int)v == r.e || (desc_b[v] && anc_e[v])) {
                r.in[v] = 1;
                r.nodes.push_back((int)v);
            }
        for (size_t v = 0; v < nn; ++v)
            if (desc_b[v] && !r.in[v] && !desc_e[v])
                return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: region %d (index %d): work downstream of its begin marker "
                            "does not pass through its end marker (a stream forked inside the region must join before it ends)",
                            r.serial, r.index);
        for (int v : r.nodes) {
            if (owner[v] >= 0)
                return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: regions %d and %d nest or overlap", regions[owner[v]].serial, r.serial);
            owner[v] = (int)ri;
            if (v == r.b) continue;
            for (int p : preds[v])
                if (!r.in[p] && !anc_b[p])
                    return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: region %d (index %d) waits on work that does not precede "
                                "its begin marker (a stream joined inside the region)", r.serial, r.index);
            if (v == r.e) continue;
            const cudaGraphNodeType t = type[v];
            const bool ok = t == cudaGraphNodeTypeKernel || t == cudaGraphNodeTypeMemset || t == cudaGraphNodeTypeEmpty ||
                            t == cudaGraphNodeTypeGraph || t == cudaGraphNodeTypeConditional ||
                            (t == cudaGraphNodeTypeMemcpy && device_memcpy(nodes[v]));
            if (!ok)
                return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: region %d (index %d) holds a %s node, which a conditional "
                            "body cannot hold (kernel, memset, device memcpy, empty, child graph and conditional nodes only)",
                            r.serial, r.index, t == cudaGraphNodeTypeMemcpy ? "host memcpy" : type_name(t));
        }
    }

    // ---- extract each region as its own graph: a clone of the whole graph without the nodes outside it (or its markers)
    std::vector<cudaGraph_t> bodies;
    auto drop_bodies = [&]() { for (cudaGraph_t b : bodies) cudaGraphDestroy(b); };
    for (const Region& r : regions) {
        std::vector<char> keep(r.in);
        keep[r.b] = keep[r.e] = 0;
        cudaGraph_t body = nullptr;
        const char* step = "";
        cudaError_t e = extract(graph, nodes, keep, &body, &step);
        if (e == cudaSuccess) {
            bodies.push_back(body);
            if (r.nodes.size() == 2) {  // nothing between the markers: an empty body
                cudaGraphNode_t c = nullptr;
                step = "cudaGraphAddEmptyNode";
                e = cudaGraphAddEmptyNode(&c, body, nullptr, 0);
            }
        }
        if (e != cudaSuccess) {
            cudaGetLastError();
            drop_bodies();
            return fail(ctx, ESACB200_ERR_CUDA, "gate_finalize: extracting region %d: %s failed: %s (the graph is untouched)",
                        r.serial, step, cudaGetErrorString(e));
        }
        if ((e = fits_conditional(body)) == cudaSuccess) continue;
        // name the first node the body cannot hold on its own
        for (int v : r.nodes) {
            if (v == r.b || v == r.e) continue;
            std::vector<char> one(nn, 0);
            one[v] = 1;
            cudaGraph_t single = nullptr;
            if (extract(graph, nodes, one, &single, &step) != cudaSuccess) break;
            const cudaError_t ev = fits_conditional(single);
            cudaGraphDestroy(single);
            if (ev == cudaSuccess) continue;
            const char* fname = nullptr;
            cudaKernelNodeParams kp = {};
            if (type[v] == cudaGraphNodeTypeKernel && cudaGraphKernelNodeGetParams(nodes[v], &kp) == cudaSuccess)
                cudaFuncGetName(&fname, kp.func);
            cudaGetLastError();
            drop_bodies();
            return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: region %d (index %d) holds a %s node%s%s that a conditional body "
                        "refuses (%s; the graph is untouched)", r.serial, r.index, type_name(type[v]), fname ? " of " : "",
                        fname ? fname : "", cudaGetErrorString(ev));
        }
        drop_bodies();
        return fail(ctx, ESACB200_ERR_ARG, "gate_finalize: region %d (index %d) does not fit a conditional body (%s; the graph "
                    "is untouched)", r.serial, r.index, cudaGetErrorString(e));
    }

    // ---- the edits: the handles, a conditional node per region, its wiring, then the regions' nodes go
    std::vector<unsigned long long> pairs(2 * regions.size(), 0ull);
    {
        cudaError_t e = gate->pairs.ensure(pairs.size() * sizeof(unsigned long long));
        for (size_t ri = 0; ri < regions.size() && e == cudaSuccess; ++ri) {
            cudaGraphConditionalHandle h = 0;
            e = cudaGraphConditionalHandleCreate(&h, graph, 0, cudaGraphCondAssignDefault);
            pairs[2 * ri] = (unsigned long long)regions[ri].index;
            pairs[2 * ri + 1] = (unsigned long long)h;
        }
        if (e != cudaSuccess) {
            drop_bodies();
            return gate_fail(ctx, e, "gate_finalize: the conditional handles");
        }
    }
    std::vector<cudaGraphNode_t> cond(regions.size(), nullptr);
    for (size_t ri = 0; ri < regions.size(); ++ri) {
        cudaGraphNodeParams p = {};
        p.type = cudaGraphNodeTypeConditional;
        p.conditional.handle = (cudaGraphConditionalHandle)pairs[2 * ri + 1];
        p.conditional.type = cudaGraphCondTypeIf;
        p.conditional.size = 1;
        cudaError_t e = cudaGraphAddNode(&cond[ri], graph, nullptr, 0, &p);
        cudaGraphNode_t child = nullptr;
        if (e == cudaSuccess) e = cudaGraphAddChildGraphNode(&child, p.conditional.phGraph_out[0], nullptr, 0, bodies[ri]);
        if (e != cudaSuccess) {
            cudaGetLastError();
            drop_bodies();
            return fail(ctx, ESACB200_ERR_CUDA, "gate_finalize: the conditional node of region %d: %s", regions[ri].serial,
                        cudaGetErrorString(e));
        }
    }
    drop_bodies();
    auto outside = [&](int v) { return owner[v] >= 0 ? cond[owner[v]] : nodes[v]; };
    std::set<std::pair<cudaGraphNode_t, cudaGraphNode_t>> wires;
    for (size_t ri = 0; ri < regions.size(); ++ri) {
        for (int p : preds[regions[ri].b]) wires.emplace(outside(p), cond[ri]);
        for (int s : succs[regions[ri].e]) wires.emplace(cond[ri], outside(s));
    }
    for (const auto& w : wires) GK(cudaGraphAddDependencies(graph, &w.first, &w.second, 1));
    for (const Region& r : regions)
        for (int v : r.nodes) GK(cudaGraphDestroyNode(nodes[v]));
    GK(cudaMemcpy(gate->pairs.p, pairs.data(), pairs.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice));
    const GateTable table = {1, regions.size(), gate->pairs.as<const unsigned long long>()};  // ready: the arm kernel runs
    GK(cudaMemcpy(gate->table.p, &table, sizeof(table), cudaMemcpyHostToDevice));
#undef GK
    return ESACB200_OK;
} ESAC_ABI_CATCH(gate->ctx)

}  // extern "C"
