/* Python module `esac_ref`: the reference's two entry points, compiled from the UNMODIFIED sources under
 * code/esac (see oracle/build_ref.py) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Why not the module esac.cpp:513-516 defines itself: that binding keeps the GIL while esac_forward runs, and the
 * reference's OpenMP worker threads would then wait forever for it inside the cv2-forwarding shim.  This file binds the
 * same two functions with the GIL released; nothing else differs (same positional signature, same return values).
 * Additive test hooks: force_init (ThreadRand::forceInit, thread_rand.h:88), irand (thread_rand.cpp:68-71),
 * set_num_threads (omp_set_num_threads), set_native_project / counters of the shim, and the pose loss pair loss / dLoss
 * (esac_loss.h, compiled into esac.cpp's object; declared here, not included, so that they are defined once).
 */
#include <torch/extension.h>
#include <omp.h>

#include <atomic>

#include "thread_rand.h"
#include "esac_types.h"

int esac_forward(at::Tensor sceneCoordinatesSrc, at::Tensor hypAssignmentSrc, at::Tensor outPoseSrc, int shiftX, int shiftY,
                 float focalLength, float ppointX, float ppointY, float inlierThreshold, float inlierAlpha, float inlierBeta,
                 float maxReproj, int subSampling);
double esac_backward(at::Tensor sceneCoordinatesSrc, at::Tensor outGradientsSrc, at::Tensor hypAssignmentSrc, at::Tensor gtPoseSrc,
                     float wLossRot, float wLossTrans, float lossCut, int shiftX, int shiftY, float focalLength, float ppointX,
                     float ppointY, float inlierThreshold, float inlierAlpha, float inlierBeta, float maxReproj, int subSampling);

namespace esac {
double loss(const trans_t& trans1, const trans_t& trans2, double wRot, double wTrans, double cut);
cv::Mat_<double> dLoss(const pose_t& est, const pose_t& gt, double wRot, double wTrans, double cut);
}

static esac::trans_t trans_of(const std::vector<double>& v) {
    if (v.size() != 16) throw std::invalid_argument("a transform is 16 doubles (4x4, row-major)");
    esac::trans_t t(4, 4);
    for (int i = 0; i < 16; ++i) t(i / 4, i % 4) = v[i];
    return t;
}

static esac::pose_t pose_of(const std::vector<double>& v) {
    if (v.size() != 6) throw std::invalid_argument("a pose is 6 doubles (rvec, tvec)");
    cv::Mat_<double> r(3, 1), t(3, 1);
    for (int i = 0; i < 3; ++i) { r(i, 0) = v[i]; t(i, 0) = v[3 + i]; }
    return esac::pose_t(r, t);
}

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
    m.def("loss", [](const std::vector<double>& T1, const std::vector<double>& T2, double wRot, double wTrans, double cut) {
        return esac::loss(trans_of(T1), trans_of(T2), wRot, wTrans, cut);
    }, "esac_loss.h loss() of two camera->world transforms (16 doubles each, row-major)");
    m.def("d_loss", [](const std::vector<double>& est, const std::vector<double>& gt, double wRot, double wTrans, double cut) {
        cv::Mat_<double> j = esac::dLoss(pose_of(est), pose_of(gt), wRot, wTrans, cut);
        std::vector<double> out(6);
        for (int i = 0; i < 6; ++i) out[i] = j(0, i);
        return out;
    }, "esac_loss.h dLoss() of two scene poses (rvec, tvec: 6 doubles each); returns its 1x6 Jacobian");
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
