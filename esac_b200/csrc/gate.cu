// Expert gates (include/esac_b200.h: esacb200_gate_*): run a region of a captured CUDA graph only where a histogram on the
// device says so.  The host turns every region between a begin and an end marker into an IF conditional node on one of the
// gate's handles (capi_gate.cu); at run time the arm kernel sets each handle from its count, so a replay runs the experts
// that drew hypotheses and skips the others, as the reference's loops do (train_esac.py:143-145, test_esac.py:179-185).
#include "esac_internal.h"

namespace esacb200 {

namespace {

// One thread per region (a conditional handle drives one conditional node, so every region has its own).  The handles
// start every launch at 0 (cudaGraphCondAssignDefault): a region runs only if its count is positive when this kernel
// runs.  A count of 0.5 counts as positive, NaN does not.  Until finalize has written the table (a graph it refused never
// gets one) the kernel does nothing.
__global__ void __launch_bounds__(256) gate_arm_kernel(const GateArm a) {
    const GateTable* t = a.table;
    if (!t->ready) return;
    for (unsigned long long k = blockIdx.x * blockDim.x + threadIdx.x; k < t->count; k += (unsigned long long)gridDim.x * blockDim.x)
        cudaGraphSetConditional(t->pairs[2 * k + 1], a.counts[t->pairs[2 * k]] > 0.f ? 1u : 0u);
}

// Does nothing: its parameter tells the host which region of which gate it opens or closes.
__global__ void gate_mark_kernel(const GateTag) {}

}  // namespace

const void* gate_arm_fn() { return (const void*)gate_arm_kernel; }
const void* gate_mark_fn() { return (const void*)gate_mark_kernel; }

void launch_gate_arm(const GateArm& a, cudaStream_t stream) {
    gate_arm_kernel<<<(a.n + 255) / 256, 256, 0, stream>>>(a);
}

void launch_gate_mark(const GateTag& t, cudaStream_t stream) { gate_mark_kernel<<<1, 1, 0, stream>>>(t); }

}  // namespace esacb200
