/* Python module `esac_ref`: the reference's two entry points, compiled from the UNMODIFIED sources under
 * code/esac (see oracle/build_ref.py) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Why not the module esac.cpp:513-516 defines itself: that binding keeps the GIL while esac_forward runs, and the
 * reference's OpenMP worker threads would then wait forever for it inside the cv2-forwarding shim.  This file binds the
 * same two functions with the GIL released; nothing else differs (same positional signature, same return values).
 * Additive test hooks: force_init (ThreadRand::forceInit, thread_rand.h:88), irand (thread_rand.cpp:68-71),
 * set_num_threads (omp_set_num_threads), set_native_project / counters of the shim.
 */
#include <torch/extension.h>
#include <omp.h>

#include <atomic>

#include "thread_rand.h"

int esac_forward(at::Tensor sceneCoordinatesSrc, at::Tensor hypAssignmentSrc, at::Tensor outPoseSrc, int shiftX, int shiftY,
                 float focalLength, float ppointX, float ppointY, float inlierThreshold, float inlierAlpha, float inlierBeta,
                 float maxReproj, int subSampling);
double esac_backward(at::Tensor sceneCoordinatesSrc, at::Tensor outGradientsSrc, at::Tensor hypAssignmentSrc, at::Tensor gtPoseSrc,
                     float wLossRot, float wLossTrans, float lossCut, int shiftX, int shiftY, float focalLength, float ppointX,
                     float ppointY, float inlierThreshold, float inlierAlpha, float inlierBeta, float maxReproj, int subSampling);

namespace esac_ref_shim {
extern std::atomic<int> native_project;
extern std::atomic<long> n_solvepnp, n_solvepnp_fail, n_project, n_rodrigues, n_inv, n_cv_error;
}

PYBIND11_MODULE(esac_ref, m) {
    namespace py = pybind11;
    py::module_::import("cv2"); /* resolve the dependency while the GIL is held */
    m.def("forward", &esac_forward, "ESAC forward (reference esac.cpp:64-190)", py::call_guard<py::gil_scoped_release>());
    m.def("backward", &esac_backward, "ESAC backward (reference esac.cpp:213-511)", py::call_guard<py::gil_scoped_release>());
    m.def("force_init", [](unsigned seed) { ThreadRand::forceInit(seed); });
    m.def("irand", [](int incMin, int excMax, int tid) { return irand(incMin, excMax, tid); });
    m.def("set_num_threads", [](int n) { omp_set_num_threads(n); });
    m.def("get_max_threads", []() { return omp_get_max_threads(); });
    m.def("set_native_project", [](bool on) { esac_ref_shim::native_project = on ? 1 : 0; });
    m.def("counters", []() {
        py::dict d;
        d["solvePnP"] = esac_ref_shim::n_solvepnp.load();
        d["solvePnP_failed"] = esac_ref_shim::n_solvepnp_fail.load();
        d["projectPoints"] = esac_ref_shim::n_project.load();
        d["Rodrigues"] = esac_ref_shim::n_rodrigues.load();
        d["inv"] = esac_ref_shim::n_inv.load();
        d["cv_error"] = esac_ref_shim::n_cv_error.load();
        return d;
    });
}
