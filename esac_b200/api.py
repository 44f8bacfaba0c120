"""Host-side mirror of the reference's `esac` extension module on top of libesac_b200.so.

`forward` / `backward` keep the positional signatures of esac_forward / esac_backward
(code/esac/esac.cpp:64-77, 213-230; bound at esac.cpp:513-516) so
train_esac.py:151-168 and test_esac.py:192-205 run unchanged with `import esac` resolving to the
top-level `esac.py` shim of this repository.  Tensors may be CPU tensors (what the reference's
callers pass) or CUDA tensors (no host round trip), or numpy arrays.

There is no CPU implementation behind this module: if libesac_b200.so is missing or no CUDA device is
visible, calls raise RuntimeError.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import math
import numbers
import os
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "libesac_b200.so"


class Stats(C.Structure):
    _fields_ = [("M", C.c_int), ("winner", C.c_int), ("n_contrib", C.c_int), ("refine_rounds", C.c_int),
                ("entropy", C.c_double), ("expected_loss", C.c_double),
                ("ms_h2d", C.c_float), ("ms_prep", C.c_float), ("ms_sample", C.c_float), ("ms_score", C.c_float),
                ("ms_select", C.c_float), ("ms_refine", C.c_float), ("ms_backward", C.c_float), ("ms_total", C.c_float),
                ("score_launches", C.c_int), ("kernel_launches", C.c_int),
                ("score_ppt", C.c_int), ("score_grid", C.c_int), ("refine_group", C.c_int)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


_lib = None
PACK_TAIL = 21  # doubles behind the M_pad scores of a shard's record (include/esac_b200.h)
# Offsets of the tail's fields from its start (M_pad): camera pose of the local winner (16 doubles), its global expert id
# (-1 on a bad assignment), local winner, the shard's M, hyp_offset, hyp_stride.
TAIL_POSE, TAIL_EXPERT, TAIL_WINNER, TAIL_M, TAIL_HYP_OFFSET, TAIL_HYP_STRIDE = 0, 16, 17, 18, 19, 20
EXCHANGE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_double), C.c_int)


def load_library() -> C.CDLL:
    """dlopen libesac_b200.so and declare the prototypes of include/esac_b200.h."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise RuntimeError(f"{LIB_PATH} is not built: run `python -m esac_b200.build` "
                           "(or __graft_entry__.build()); there is no CPU fallback")
    lib = C.CDLL(str(LIB_PATH))
    vp, i32, i64, f32, f64 = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_double
    lib.esacb200_create.argtypes = [i32, C.POINTER(vp)]
    lib.esacb200_create.restype = i32
    lib.esacb200_destroy.argtypes = [vp]
    lib.esacb200_destroy.restype = None
    lib.esacb200_last_error.argtypes = [vp]
    lib.esacb200_last_error.restype = C.c_char_p
    lib.esacb200_set_stream.argtypes = [vp, vp]
    lib.esacb200_set_seed.argtypes = [vp, C.c_uint64]
    lib.esacb200_set_option.argtypes = [vp, C.c_char_p, f64]
    lib.esacb200_inject_cells.argtypes = [vp, vp, i32, i32]
    cam = [i32, i32, f32, f32, f32, f32, f32, f32, f32, i32]  # shiftX .. subSampling
    lib.esacb200_forward.argtypes = [vp, vp, i32, i32, i32, vp, i64, i32, vp] + cam + [C.POINTER(i32)]
    lib.esacb200_backward.argtypes = [vp, vp, vp, i32, i32, i32, vp, i64, i32, vp, f32, f32, f32] + cam + [C.POINTER(f64)]
    lib.esacb200_forward_batch.argtypes = [vp, i32, vp, i32, i32, i32, vp, i64, i32, vp] + cam + [vp]
    lib.esacb200_forward_batch.restype = i32
    lib.esacb200_forward_pack.argtypes = [vp, vp, i32, i32, i32, vp, i64, i32, i32] + cam + [i32, vp]
    lib.esacb200_forward_pack.restype = i32
    lib.esacb200_nccl_unique_id.argtypes = [vp]
    lib.esacb200_nccl_unique_id.restype = i32
    lib.esacb200_comm_init.argtypes = [vp, i32, i32, vp]
    lib.esacb200_comm_init.restype = i32
    lib.esacb200_comm_destroy.argtypes = [vp]
    lib.esacb200_comm_destroy.restype = i32
    lib.esacb200_forward_sharded.argtypes = [vp, vp, i32, i32, i32, vp, i64, i32, i32, vp] + cam + [i32, C.POINTER(i32)]
    lib.esacb200_forward_sharded.restype = i32
    lib.esacb200_backward_sharded_nccl.argtypes = [vp, vp, vp, i32, i32, i32, vp, i64, i32, vp, f32, f32, f32] + cam + [i32, C.POINTER(f64)]
    lib.esacb200_backward_sharded_nccl.restype = i32
    lib.esacb200_backward_batch.argtypes = ([vp, i32, vp, vp, i32, i32, i32, vp, i64, i32, vp, f32, f32, f32, vp, vp] + cam[2:] +
                                             [vp])
    lib.esacb200_backward_batch.restype = i32
    cams = [vp, vp, vp, vp, vp, f32, f32, f32, f32, i32]  # per-image shiftX, shiftY, f, ppx, ppy; then tau .. subSampling
    lib.esacb200_forward_batch_cameras.argtypes = [vp, i32, vp, i32, i32, i32, vp, i64, i32, vp] + cams + [vp]
    lib.esacb200_forward_batch_cameras.restype = i32
    lib.esacb200_backward_batch_cameras.argtypes = [vp, i32, vp, vp, i32, i32, i32, vp, i64, i32, vp, f32, f32, f32] + cams + [vp]
    lib.esacb200_backward_batch_cameras.restype = i32
    lib.esacb200_assign_hypotheses.argtypes = [vp, i32, i32, i32, vp, i32, i32, C.c_uint64, vp, vp]
    lib.esacb200_assign_hypotheses.restype = i32
    lib.esacb200_assign_hypotheses_async.argtypes = [vp, i32, i32, i32, vp, i32, i32, vp, vp, vp, vp]
    lib.esacb200_assign_hypotheses_async.restype = i32
    lib.esacb200_gate_create.argtypes = [vp, i32, C.POINTER(vp)]
    lib.esacb200_gate_create.restype = i32
    lib.esacb200_gate_destroy.argtypes = [vp]
    lib.esacb200_gate_destroy.restype = None
    lib.esacb200_gate_arm.argtypes = [vp, vp, vp]
    lib.esacb200_gate_arm.restype = i32
    lib.esacb200_gate_mark.argtypes = [vp, i32, i32, vp]
    lib.esacb200_gate_mark.restype = i32
    lib.esacb200_gate_finalize.argtypes = [vp, vp]
    lib.esacb200_gate_finalize.restype = i32
    lib.esacb200_reproj_loss.argtypes = [vp, i32, vp, vp, i32, i32, vp, vp, vp, f32, f32, f32, i32, f32, f32, f32, vp]
    lib.esacb200_reproj_loss.restype = i32
    lib.esacb200_reproj_loss_cameras.argtypes = [vp, i32, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, i32, f32, f32, f32, vp]
    lib.esacb200_reproj_loss_cameras.restype = i32
    lib.esacb200_coord_loss.argtypes = [vp, i32, vp, i32, i32, vp, i32, i32, vp, f32, vp, vp]
    lib.esacb200_coord_loss.restype = i32
    # ragged batches: host arrays of B pointers and of B heights / widths
    lib.esacb200_forward_ragged.argtypes = [vp, i32, vp, vp, vp, i32, vp, i64, i32, vp] + cams + [vp]
    lib.esacb200_forward_ragged.restype = i32
    lib.esacb200_backward_ragged.argtypes = [vp, i32, vp, vp, vp, vp, i32, vp, i64, i32, vp, f32, f32, f32] + cams + [vp]
    lib.esacb200_backward_ragged.restype = i32
    lib.esacb200_reproj_loss_ragged.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, f32, f32, f32, vp]
    lib.esacb200_reproj_loss_ragged.restype = i32
    lib.esacb200_coord_loss_ragged.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, f32, vp, vp]
    lib.esacb200_coord_loss_ragged.restype = i32
    lib.esacb200_backward_sharded.argtypes = ([vp, vp, vp, i32, i32, i32, vp, i64, i32, vp, f32, f32, f32] + cam +
                                               [EXCHANGE_FN, vp, C.POINTER(f64)])
    lib.esacb200_backward_sharded.restype = i32
    lib.esacb200_score_poses.argtypes = [vp, vp, i32, i32, i32, vp, i64, i32, vp] + cam + [vp]
    lib.esacb200_refine_poses.argtypes = [vp, vp, i32, i32, i32, vp, i64, i32, vp, i32, i32, f32, f32, f32, f32, f32, i32, vp, vp]
    lib.esacb200_get_refine_profile.argtypes = [vp, vp]
    lib.esacb200_get_refine_profile.restype = i32
    lib.esacb200_get_sample_trace.argtypes = [vp, vp]
    lib.esacb200_get_sample_trace.restype = i32
    lib.esacb200_get_sample_profile.argtypes = [vp, vp]
    lib.esacb200_get_sample_profile.restype = i32
    lib.esacb200_get_stats.argtypes = [vp, C.POINTER(Stats)]
    lib.esacb200_get_hypotheses.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
    lib.esacb200_device_info.argtypes = [vp, C.POINTER(i32), C.c_char_p, i32]
    lib.esacb200_copy_last_scores.argtypes = [vp, vp, i32]
    lib.esacb200_copy_last_scores.restype = i32
    # the hypotheses as an autograd node
    lib.esacb200_hypotheses_tape_bytes.argtypes = [i32, i32, i32, i32]
    lib.esacb200_hypotheses_tape_bytes.restype = C.c_size_t
    lib.esacb200_hypotheses_forward.argtypes = [vp, vp, i32, i32, i32, vp, i64, i32] + cam + [vp, C.c_size_t, vp, vp, vp]
    lib.esacb200_hypotheses_forward.restype = i32
    lib.esacb200_hypotheses_backward.argtypes = [vp, vp, vp, vp, i32, i32, i32, vp, vp]
    lib.esacb200_hypotheses_backward.restype = i32
    lib.esacb200_pose_loss.argtypes = [vp, i32, vp, vp, f32, f32, f32, vp, vp]
    lib.esacb200_pose_loss.restype = i32
    lib.esacb200_pose_loss_batch.argtypes = [vp, i32, i32, vp, vp, f32, f32, f32, vp, vp]
    lib.esacb200_pose_loss_batch.restype = i32
    lib.esacb200_hypotheses_forward_ragged.argtypes = [vp, i32, vp, vp, vp, i32, vp, i64, i32] + cams + [vp, vp, vp, vp, vp]
    lib.esacb200_hypotheses_forward_ragged.restype = i32
    lib.esacb200_hypotheses_backward_ragged.argtypes = [vp, i32, vp, vp, vp, vp, vp, i32, vp, vp]
    lib.esacb200_hypotheses_backward_ragged.restype = i32
    lib.esacb200_forward_async.argtypes = [vp, i32, vp, i32, i32, i32, vp, i64, i32, vp, vp, f32, f32, f32, f32, i32, vp, vp, vp]
    lib.esacb200_forward_async.restype = i32
    lib.esacb200_reserve_forward_async.argtypes = [vp, i32, i32, i32, i32, i32, i32]
    lib.esacb200_reserve_forward_async.restype = i32
    lib.esacb200_backward_async.argtypes = [vp, i32, vp, vp, i32, i32, i32, vp, i64, i32, vp, f32, f32, f32, vp, vp, f32, f32,
                                            f32, f32, i32, vp, vp]
    lib.esacb200_backward_async.restype = i32
    lib.esacb200_reserve_backward_async.argtypes = [vp, i32, i32, i32, i32, i32, i32]
    lib.esacb200_reserve_backward_async.restype = i32
    lib.esacb200_hypotheses_forward_async.argtypes = [vp, i32, vp, i32, i32, i32, vp, i64, i32, vp, vp, f32, f32, f32, f32, i32,
                                                      vp, C.c_size_t, vp, vp, vp, vp]
    lib.esacb200_hypotheses_forward_async.restype = i32
    # the hypotheses node with a probability floor of the caller's (min_prob after subSampling)
    lib.esacb200_hypotheses_forward_floor.argtypes = [vp, vp, i32, i32, i32, vp, i64, i32] + cam + [f64, vp, C.c_size_t, vp, vp, vp]
    lib.esacb200_hypotheses_forward_floor.restype = i32
    lib.esacb200_hypotheses_forward_ragged_floor.argtypes = ([vp, i32, vp, vp, vp, i32, vp, i64, i32] + cams +
                                                             [f64, vp, vp, vp, vp, vp])
    lib.esacb200_hypotheses_forward_ragged_floor.restype = i32
    lib.esacb200_hypotheses_forward_async_floor.argtypes = [vp, i32, vp, i32, i32, i32, vp, i64, i32, vp, vp, f32, f32, f32, f32,
                                                            i32, f64, vp, C.c_size_t, vp, vp, vp, vp]
    lib.esacb200_hypotheses_forward_async_floor.restype = i32
    lib.esacb200_hypotheses_backward_async.argtypes = [vp, i32, vp, C.c_size_t, vp, vp, i32, i32, i32, i32, vp, vp, vp]
    lib.esacb200_hypotheses_backward_async.restype = i32
    lib.esacb200_pose_loss_async.argtypes = [vp, i32, i32, vp, vp, f32, f32, f32, vp, vp]
    lib.esacb200_pose_loss_async.restype = i32
    lib.esacb200_reproj_loss_async.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, i32, f32, f32, f32, vp, vp]
    lib.esacb200_reproj_loss_async.restype = i32
    lib.esacb200_coord_loss_async.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, f32, vp, vp]
    lib.esacb200_coord_loss_async.restype = i32
    lib.esacb200_reproj_loss_ragged_typed.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, f32, f32, f32,
                                                      vp, vp]
    lib.esacb200_reproj_loss_ragged_typed.restype = i32
    lib.esacb200_coord_loss_ragged_typed.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, f32, vp, vp, vp]
    lib.esacb200_coord_loss_ragged_typed.restype = i32
    lib.esacb200_reproj_loss_async_typed.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, i32, f32, f32, f32, vp, vp, vp]
    lib.esacb200_reproj_loss_async_typed.restype = i32
    lib.esacb200_coord_loss_async_typed.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, f32, vp, vp, vp]
    lib.esacb200_coord_loss_async_typed.restype = i32
    lib.esacb200_reserve_loss_async.argtypes = [vp, i32, i32, i32]
    lib.esacb200_reserve_loss_async.restype = i32
    lib.esacb200_reserve_backward_async.restype = i32
    for name in ("eval_poses", "eval_poses_async"):
        getattr(lib, "esacb200_" + name).argtypes = [vp, i32, vp, vp, vp, vp, vp, i32, vp, vp, i64, vp]
        getattr(lib, "esacb200_" + name).restype = i32
    lib.esacb200_cluster_stats_ragged.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp]
    lib.esacb200_cluster_stats_ragged.restype = i32
    lib.esacb200_kmeans2.argtypes = [vp, i32, vp, C.c_uint64, i32, i32, i32, f64, vp, vp, vp]
    lib.esacb200_kmeans2.restype = i32
    lib.esacb200_cluster_targets.argtypes = [vp, i32, vp, vp, i32, f32, vp, vp, vp]
    lib.esacb200_cluster_targets.restype = i32
    lib.esacb200_render_init_maps.argtypes = [vp, i32, vp, i64, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.esacb200_render_init_maps.restype = i32
    lib.esacb200_data_step_async.argtypes = [vp, vp, vp, vp, i64, i32, i32, i32, i32, i32, vp, vp, i32, vp, vp, vp, i64,
                                             vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.esacb200_data_step_async.restype = i32
    lib.esacb200_experts_packed_floats.argtypes = [i32]
    lib.esacb200_experts_packed_floats.restype = i64
    lib.esacb200_experts_workspace_bytes.argtypes = [i32, i32, i32, i32]
    lib.esacb200_experts_workspace_bytes.restype = i64
    lib.esacb200_experts_pack.argtypes = [vp, i32, vp, vp]
    lib.esacb200_experts_pack.restype = i32
    lib.esacb200_experts_forward_async.argtypes = [vp, i32, i32, i32, i32, vp, i32, vp, vp, vp, i64, vp]
    lib.esacb200_experts_forward_async.restype = i32
    lib.esacb200_gating_packed_floats.argtypes = [i32, i32]
    lib.esacb200_gating_packed_floats.restype = i64
    lib.esacb200_gating_workspace_bytes.argtypes = [i32, i32, i32, i32, i32]
    lib.esacb200_gating_workspace_bytes.restype = i64
    lib.esacb200_gating_pack.argtypes = [vp, i32, i32, vp, vp]
    lib.esacb200_gating_pack.restype = i32
    lib.esacb200_gating_forward_async.argtypes = [vp, i32, i32, i32, i32, i32, vp, vp, vp, i64, vp, vp]
    lib.esacb200_gating_forward_async.restype = i32
    for name in ("set_stream", "set_seed", "set_option", "inject_cells", "forward", "backward", "score_poses",
                 "refine_poses", "get_stats", "get_hypotheses", "device_info"):
        getattr(lib, "esacb200_" + name).restype = i32
    # host test hooks (include/esac_b200_testhooks.h)
    lib.esacb200_host_rodrigues.argtypes = [vp, vp, vp]
    lib.esacb200_host_rodrigues.restype = None
    lib.esacb200_host_rodrigues_inv.argtypes = [vp, vp]
    lib.esacb200_host_rodrigues_inv.restype = None
    lib.esacb200_host_p3p_all.argtypes = [vp, vp, vp, vp]
    lib.esacb200_host_p3p_all.restype = i32
    lib.esacb200_host_p3p_pose.argtypes = [vp, vp, f32, f32, f32, f32, vp, C.POINTER(i32)]
    lib.esacb200_host_p3p_pose.restype = i32
    lib.esacb200_host_try.argtypes = [vp, vp, f32, f32, f32, f32, f32, C.POINTER(i32), C.POINTER(i32)]
    lib.esacb200_host_try.restype = None
    lib.esacb200_host_tries_hint.argtypes = [i32, vp, vp, f32, f32, f32, f32, f32, vp, vp, vp]
    lib.esacb200_host_tries_hint.restype = None
    lib.esacb200_host_try_verdict.argtypes = [vp, vp, f32, f32, f32, f32, C.POINTER(i32), vp]
    lib.esacb200_host_try_verdict.restype = None
    lib.esacb200_host_project.argtypes = [vp, f32, f32, f32, vp, vp, vp, vp]
    lib.esacb200_host_project.restype = None
    lib.esacb200_host_loss.argtypes = [vp, vp, f64, f64, f64]
    lib.esacb200_host_loss.restype = f64
    lib.esacb200_host_dloss.argtypes = [vp, vp, f64, f64, f64, vp]
    lib.esacb200_host_dloss.restype = None
    lib.esacb200_host_pose2trans.argtypes = [vp, vp]
    lib.esacb200_host_pose2trans.restype = None
    lib.esacb200_host_trans2pose.argtypes = [vp, vp]
    lib.esacb200_host_trans2pose.restype = None
    lib.esacb200_host_dprojectdobj.argtypes = [vp, vp, vp, f32, f32, f32, f32, vp]
    lib.esacb200_host_dprojectdobj.restype = None
    lib.esacb200_host_pinv6.argtypes = [vp, vp]
    lib.esacb200_host_pinv6.restype = None
    lib.esacb200_host_draw_cells.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, i32, i32, vp]
    lib.esacb200_host_draw_cells.restype = None
    lib.esacb200_graph_node_types.argtypes = [vp, vp, i32]
    lib.esacb200_graph_node_types.restype = i32
    lib.esacb200_test_experts_conv.argtypes = [vp, i32, i32, vp, vp, i64, i64, i32, i32, i32, i32, i32, i32, i32, vp, i64,
                                               i64, i64, i64, vp]
    lib.esacb200_test_experts_conv.restype = i32
    lib.esacb200_test_gathered.argtypes = [vp, i32, i32, vp, vp, vp, vp, i32, vp, vp, vp, vp]
    lib.esacb200_test_gathered.restype = i32
    _lib = lib
    return lib


# ------------------------------------------------------------------------------------------------
# contexts (one per device) -- the analogue of the reference's static ThreadRand state
# ------------------------------------------------------------------------------------------------
class Context:
    def __init__(self, device: int = 0):
        self.lib = load_library()
        h = C.c_void_p()
        rc = self.lib.esacb200_create(int(device), C.byref(h))
        if rc != 0:
            raise RuntimeError(f"esac_b200: cannot create a context on CUDA device {device} (status {rc}); "
                               "this implementation has no CPU path")
        self.handle = h
        self.device = int(device)
        self.comm_world, self.comm_rank = 1, 0

    def close(self):
        if getattr(self, "handle", None):
            self.lib.esacb200_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check(self, rc: int):
        if rc != 0:
            msg = self.lib.esacb200_last_error(self.handle)
            raise RuntimeError(f"esac_b200 (status {rc}): {msg.decode() if msg else ''}")

    # additive API ------------------------------------------------------------------------------
    def set_seed(self, seed: int):
        """Seeds the draws and resets the call counters.  Once forward_async has run on the context, the reset of its
        device-side seed is enqueued on torch's current stream, ordered with the calls and graph replays there."""
        if getattr(self, "async_used", False):
            import torch
            self.set_stream(torch.cuda.current_stream(self.device).cuda_stream or _CUDA_STREAM_LEGACY)
        self.check(self.lib.esacb200_set_seed(self.handle, C.c_uint64(seed & ((1 << 64) - 1))))

    def set_option(self, key: str, value: float):
        self.check(self.lib.esacb200_set_option(self.handle, key.encode(), float(value)))

    def set_stream(self, stream_ptr: int):
        self.check(self.lib.esacb200_set_stream(self.handle, C.c_void_p(stream_ptr or None)))

    def inject_cells(self, cells):
        if cells is None:
            self.check(self.lib.esacb200_inject_cells(self.handle, None, 0, 0))
            return
        cells = np.ascontiguousarray(cells, np.int32)
        assert cells.ndim == 4 and cells.shape[2:] == (4, 2), "cells must be [M, T, 4, 2] (x, y)"
        self.check(self.lib.esacb200_inject_cells(self.handle, cells.ctypes.data, cells.shape[0], cells.shape[1]))

    def stats(self) -> dict:
        s = Stats()
        self.check(self.lib.esacb200_get_stats(self.handle, C.byref(s)))
        return s.as_dict()

    def comm_init(self, world: int, rank: int, unique_id: bytes):
        """ncclCommInitRank inside the library (collective over all ranks); unique_id from nccl_unique_id() of rank 0."""
        buf = C.create_string_buffer(bytes(unique_id), 128)
        self.check(self.lib.esacb200_comm_init(self.handle, int(world), int(rank), buf))
        self.comm_world, self.comm_rank = int(world), int(rank)

    def comm_destroy(self):
        self.check(self.lib.esacb200_comm_destroy(self.handle))
        self.comm_world, self.comm_rank = 1, 0

    def refine_profile(self) -> np.ndarray:
        """Phase cycle counters of the last refinement (option "refine_profile" = 1), see include/esac_b200.h."""
        out = np.zeros(16, np.int64)
        self.check(self.lib.esacb200_get_refine_profile(self.handle, out.ctypes.data))
        return out

    def sample_profile(self) -> dict:
        out = np.zeros(8, np.int64)
        self.check(self.lib.esacb200_get_sample_profile(self.handle, out.ctypes.data))
        d = {"tries_prefiltered": int(out[0]), "survivors_judged": int(out[1]), "waves": int(out[2]),
             "left_to_tail": int(out[3]), "accepted_staged": int(out[4]), "lanes": int(out[5]),
             "tries_cut": int(out[6]), "hints_rejected": int(out[7])}
        return d

    def sample_trace(self) -> np.ndarray:
        """[lane, wave, kernel (0 prefilter, 1 exact), (start, end)] in ns relative to the first stamp; -1 where nothing ran.
        Waves 32 and later (option sample_waves goes up to 64) run but are not stamped."""
        raw = np.zeros(512, np.uint64)
        self.check(self.lib.esacb200_get_sample_trace(self.handle, raw.ctypes.data))
        t = raw.reshape(4, 32, 2, 2)
        ran = t[..., 0] != np.uint64(0xFFFFFFFFFFFFFFFF)
        t0 = t[..., 0][ran].min() if ran.any() else np.uint64(0)
        out = np.full(t.shape, -1, np.int64)
        out[ran] = (t[ran] - t0).astype(np.int64)
        return out

    def copy_last_scores(self, dst):
        """dst: float64 torch tensor (CUDA or CPU) or numpy array of M elements; stream-ordered copy."""
        n = int(dst.numel()) if _is_torch(dst) else int(np.asarray(dst).size)
        ptr = dst.data_ptr() if _is_torch(dst) else np.asarray(dst).ctypes.data
        self.check(self.lib.esacb200_copy_last_scores(self.handle, ptr, n))

    def device_info(self) -> dict:
        n = C.c_int()
        buf = C.create_string_buffer(128)
        self.check(self.lib.esacb200_device_info(self.handle, C.byref(n), buf, 128))
        return {"sm_count": n.value, "name": buf.value.decode()}

    def hypotheses(self, losses: bool = False) -> dict:
        M = self.stats()["M"]
        out = {"poses": np.zeros((M, 6)), "cells": np.zeros((M, 4, 2), np.int32), "tries": np.zeros(M, np.int32),
               "scores": np.zeros(M), "probs": np.zeros(M), "refined": np.zeros((M, 6))}
        lo = np.zeros(M) if losses else None
        self.check(self.lib.esacb200_get_hypotheses(self.handle, out["poses"].ctypes.data, out["cells"].ctypes.data,
                                                    out["tries"].ctypes.data, out["scores"].ctypes.data,
                                                    out["probs"].ctypes.data, out["refined"].ctypes.data,
                                                    lo.ctypes.data if losses else None))
        if losses:
            out["losses"] = lo
        return out


_contexts: dict[int, Context] = {}


def context(device: int | None = None) -> Context:
    if device is None:
        device = 0
        try:
            import torch
            if torch.cuda.is_available():
                device = torch.cuda.current_device()
        except Exception:
            pass
    if device not in _contexts:
        _contexts[device] = Context(device)
    return _contexts[device]


# ------------------------------------------------------------------------------------------------
# tensor plumbing
# ------------------------------------------------------------------------------------------------
_TORCH_NAMES = {"torch.float32": "Float", "torch.float64": "Double", "torch.float16": "Half", "torch.int64": "Long",
                "torch.int32": "Int", "torch.bfloat16": "BFloat16", "torch.uint8": "Byte", "torch.int16": "Short",
                "torch.int8": "Char", "torch.bool": "Bool"}
_NP_NAMES = {"float32": "Float", "float64": "Double", "float16": "Half", "int64": "Long", "int32": "Int"}


def _is_torch(t) -> bool:
    return type(t).__module__.startswith("torch")


def _dtype_name(t) -> str:
    if _is_torch(t):
        name, names = str(t.dtype), _TORCH_NAMES
    else:
        name, names = str(np.asarray(t).dtype), _NP_NAMES
    return names.get(name, name)


def _check(t, want: str | tuple, rank: int, what: str):
    """Same failure mode as at::Tensor::accessor<T, N>() in the reference (esac.cpp:80-84): RuntimeError.  want: a dtype
    name, or a tuple of the names accepted."""
    have = _dtype_name(t)
    wants = want if isinstance(want, tuple) else (want,)
    if have not in wants:
        raise RuntimeError(f"expected scalar type {' or '.join(wants)} but found {have} ({what})")
    nd = t.dim() if _is_torch(t) else np.asarray(t).ndim
    if nd != rank:
        raise RuntimeError(f"expected {rank} dims but tensor has {nd} ({what})")


class _Arg:
    """Pointer view of a tensor argument; keeps temporaries alive and writes results back."""

    def __init__(self, t, writable=False, need_contig=True):
        self.orig = t
        self.writable = writable
        self.tmp = None
        if _is_torch(t):
            self.is_cuda = t.is_cuda
            self.device = t.device.index if t.is_cuda else None
            v = t
            if need_contig and not t.is_contiguous():
                v = t.contiguous()
                self.tmp = v
            self.view = v
            self.ptr = v.data_ptr()
        else:
            a = np.asarray(t)
            self.is_cuda = False
            self.device = None
            v = a
            if need_contig and not a.flags["C_CONTIGUOUS"]:
                v = np.ascontiguousarray(a)
                self.tmp = v
            self.view = v
            self.ptr = v.ctypes.data

    def finish(self):
        if self.writable and self.tmp is not None:
            if _is_torch(self.orig):
                self.orig.copy_(self.tmp)
            else:
                np.copyto(np.asarray(self.orig), self.tmp)


def _assign_arg(t):
    """hypAssignment: int64 [M], any stride (stride 0 for expert.expand(), test_esac.py:173)."""
    if _is_torch(t):
        M = int(t.shape[0])
        stride = int(t.stride(0)) if M > 0 else 1
        return t.data_ptr(), stride, M, (t.device.index if t.is_cuda else None), t
    a = np.asarray(t)
    M = int(a.shape[0])
    stride = int(a.strides[0] // a.itemsize) if M > 0 else 1
    return a.ctypes.data, stride, M, None, a


def _is_number(v) -> bool:
    """A Python / numpy number or a 0-d array or tensor: one value for the whole batch."""
    if isinstance(v, (list, tuple)):
        return False
    return isinstance(v, (int, float)) or ((v.dim() == 0) if _is_torch(v) else np.ndim(v) == 0)


def _per_image(v, B: int, dtype, what: str) -> np.ndarray:
    """A batch argument as B contiguous host values of `dtype`: a number is broadcast; a sequence, numpy array or tensor
    (CPU or CUDA) must hold B values.  float64 values (a DataLoader's focal lengths) round to float32 exactly as ctypes
    rounds a Python float.  Raises RuntimeError before any context exists, so the check runs without a GPU."""
    if _is_number(v):
        return np.full(B, int(v) if dtype == np.int32 else float(v), dtype)
    if _is_torch(v):
        v = v.detach().cpu().numpy()
    a = np.ascontiguousarray(np.asarray(v).reshape(-1), dtype=dtype)
    if a.shape[0] != B:
        kind = "an int or {} ints" if dtype == np.int32 else "a number or {} numbers"
        raise RuntimeError(f"{what} must be {kind.format(B)}, got {a.shape[0]} values")
    return a


def _cameras(B: int, shiftX, shiftY, focalLength, ppointX, ppointY, shift_names=("shiftX", "shiftY")) -> tuple:
    """The shifts and camera of a batch as five host arrays of B values (int32 shifts, float32 f, ppx, ppy), see _per_image."""
    return (_per_image(shiftX, B, np.int32, shift_names[0]), _per_image(shiftY, B, np.int32, shift_names[1]),
            _per_image(focalLength, B, np.float32, "focalLength"), _per_image(ppointX, B, np.float32, "ppointX"),
            _per_image(ppointY, B, np.float32, "ppointY"))


def _thresholds(inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling) -> tuple:
    """tau, alpha, beta, maxReproj, subSampling as ctypes takes them (the tail of the `cam` / `cams` argtypes)."""
    return float(inlierThreshold), float(inlierAlpha), float(inlierBeta), float(maxReproj), int(subSampling)


def _camera_tail(shiftX, shiftY, focalLength, ppointX, ppointY, *thresholds) -> tuple:
    """The scalar tail of a single-image call, shiftX .. subSampling, as ctypes takes it (the `cam` argtypes)."""
    return (int(shiftX), int(shiftY), float(focalLength), float(ppointX), float(ppointY)) + _thresholds(*thresholds)


@contextlib.contextmanager
def _hypothesis_shard(ctx: Context, hyp_offset: int, hyp_stride: int | None = None):
    """Options hyp_offset (and hyp_stride) on the context for one sharded call, back to 0 (1) when it returns or raises."""
    options = {"hyp_offset": (hyp_offset, 0)}
    if hyp_stride is not None:
        options["hyp_stride"] = (hyp_stride, 1)
    for key, (value, _) in options.items():
        ctx.set_option(key, value)
    try:
        yield
    finally:
        for key, (_, default) in options.items():
            ctx.set_option(key, default)


def _is_list(t) -> bool:
    """A ragged batch: a list or tuple of per-image tensors / arrays (each with its own H x W)."""
    return isinstance(t, (list, tuple))


class _Images:
    """An image-sized argument of a batched entry point as the library's ragged form takes it: a host array of B pointers
    with the B heights and widths.  The argument is one stacked float32 tensor [B, *inner] or a list / tuple of B float32
    tensors of `rank` dims [..., 3, H_b, W_b] (a ragged batch; all CPU / numpy or all CUDA).  A stacked tensor stays one
    buffer (a pinned host tensor stays pinned, and the library copies it in one run) and image b starts b images past its
    base.  `like`: an image argument of the same call that this one must match in kind and number of images.  dtypes: the
    dtype names accepted instead of float32 (_check's `want`); the images of a list share one (self.dtype).  Raises
    RuntimeError before any context exists."""

    def __init__(self, t, rank: int, what: str, writable: bool = False, like: _Images | None = None,
                 dtypes: str | tuple = "Float"):
        self.what = what
        self.ragged = _is_list(t)
        if like is not None and self.ragged != like.ragged:
            kind = "a list or tuple of tensors" if like.ragged else "one stacked tensor"
            owner = like.what + ("'" if like.what.endswith("s") else "'s")
            raise RuntimeError(f"{what} must be {kind}, of {owner} kind")
        if self.ragged:
            if len(t) == 0:
                raise RuntimeError(f"{what} is an empty list")
            for b, x in enumerate(t):
                _check(x, dtypes, rank, f"{what}[{b}]")
            if len({_dtype_name(x) for x in t}) > 1:
                raise RuntimeError(f"{what} mixes dtypes: " + ", ".join(f"{what}[{b}] {_dtype_name(x)}" for b, x in enumerate(t)))
            if len({bool(_is_torch(x) and x.is_cuda) for x in t}) > 1:
                raise RuntimeError(f"{what} mixes CPU and CUDA tensors")
            self.shapes = [tuple(int(v) for v in x.shape) for x in t]
        else:
            _check(t, dtypes, rank + 1, what)
            n, *inner = (int(v) for v in t.shape)
            if n == 0:
                raise RuntimeError(f"{what} is an empty batch")
            self.shapes = [tuple(inner)] * n
        self.B = len(self.shapes)
        self.dtype = _dtype_name(t[0] if self.ragged else t)
        if like is not None and self.B != like.B:
            raise RuntimeError(f"shapes must be of one batch: {what} holds {self.B} {'tensors' if self.ragged else 'images'} "
                               f"for {like.B} images")
        for b, s in enumerate(self.shapes):
            if s[-3] != 3:
                inner = "E,3,H,W" if rank == 4 else "3,H,W"
                raise RuntimeError(f"shapes must be [B,{inner}] or a list of B [{inner}]: {what}[{b}] is {list(s)}")
        if self.ragged:
            self.args = [_Arg(x, writable=writable) for x in t]
            ptrs = [a.ptr for a in self.args]
        else:
            self.args = [_Arg(t, writable=writable)]
            step = self.args[0].view.itemsize * math.prod(self.shapes[0])
            ptrs = [self.args[0].ptr + b * step for b in range(self.B)]
        self.ptrs = (C.c_void_p * self.B)(*ptrs)
        self.hs = (C.c_int * self.B)(*[s[-2] for s in self.shapes])
        self.ws = (C.c_int * self.B)(*[s[-1] for s in self.shapes])
        self.devices = [a.device for a in self.args]

    def require_shapes_of(self, other: _Images):
        """Gradients: image b has the shape of other's image b."""
        for b, (s, o) in enumerate(zip(self.shapes, other.shapes)):
            if s != o:
                raise RuntimeError(f"{self.what} are not of the shape of {other.what}: {self.what}[{b}] is {list(s)}, "
                                   f"{other.what}[{b}] is {list(o)}")

    def finish(self):
        for a in self.args:
            a.finish()


def _check_maps(shapes, what: str) -> int:
    """[E,3,H,W] images with one E, each large enough to draw 4 distinct cells (esac.cpp:110-113); returns E."""
    E = shapes[0][0]
    for b, s in enumerate(shapes):
        if s[0] != E:
            raise RuntimeError(f"{what}[{b}] must be [E,3,H,W] with the E of image 0 ({E}), got {list(s)}")
        if (s[3] - 1) * (s[2] - 1) < 4:
            raise RuntimeError(f"{what}[{b}]: map {s[3]}x{s[2]} too small to draw 4 distinct cells")
    return E


_CUDA_STREAM_LEGACY = 0x1


def _pick_ctx(*devices) -> Context:
    devs = {d for d in devices if d is not None}
    if len(devs) > 1:
        raise RuntimeError(f"esac_b200: tensors live on different CUDA devices {sorted(devs)}")
    ctx = context(next(iter(devs)) if devs else None)
    stream = 0
    if devs:
        # CUDA tensors: run on torch's current stream so that the call is ordered after whatever produced them.  torch
        # reports its default stream as handle 0, which the C ABI reads as "use the context's own stream"; the legacy
        # default stream has the explicit handle cudaStreamLegacy = 0x1.
        import torch
        stream = torch.cuda.current_stream(ctx.device).cuda_stream or _CUDA_STREAM_LEGACY
    ctx.set_stream(stream)
    return ctx


def _pick_ctx_host(device: int | None) -> Context:
    """Context for host-only arguments on an explicit device (sharded entry points: one process per GPU)."""
    ctx = context(device)
    ctx.set_stream(0)
    return ctx


# ------------------------------------------------------------------------------------------------
# the reference's two entry points
# ------------------------------------------------------------------------------------------------
def forward(sceneCoordinates, hypAssignment, outPose, shiftX, shiftY, focalLength, ppointX, ppointY,
            inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling) -> int:
    """esac.forward (esac.cpp:64-190): writes the estimated camera pose into outPose (4x4, in place) and
    returns the index of the winning expert."""
    _check(sceneCoordinates, "Float", 4, "sceneCoordinates")
    _check(hypAssignment, "Long", 1, "hypAssignment")
    _check(outPose, "Float", 2, "outPose")
    if tuple(sceneCoordinates.shape)[1] != 3:
        raise RuntimeError("sceneCoordinates must be [E, 3, H, W]")
    if tuple(outPose.shape) != (4, 4):
        raise RuntimeError("outPose must be [4, 4]")
    co = _Arg(sceneCoordinates)
    op = _Arg(outPose, writable=True)
    aptr, astride, M, adev, _keep = _assign_arg(hypAssignment)
    ctx = _pick_ctx(co.device, op.device, adev)
    E, _, H, W = (int(s) for s in sceneCoordinates.shape)
    expert = C.c_int(-1)
    ctx.check(ctx.lib.esacb200_forward(ctx.handle, co.ptr, E, H, W, aptr, astride, M, op.ptr,
                                       *_camera_tail(shiftX, shiftY, focalLength, ppointX, ppointY, inlierThreshold, inlierAlpha,
                                                     inlierBeta, maxReproj, subSampling), C.byref(expert)))
    op.finish()
    return int(expert.value)


def backward(sceneCoordinates, outGradients, hypAssignment, gtPose, wLossRot, wLossTrans, lossCut, shiftX, shiftY,
             focalLength, ppointX, ppointY, inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling) -> float:
    """esac.backward (esac.cpp:213-511): accumulates d(expected pose loss)/d(sceneCoordinates) into
    outGradients (in place, +=) and returns the expected loss."""
    _check(sceneCoordinates, "Float", 4, "sceneCoordinates")
    _check(outGradients, "Float", 4, "outGradients")
    _check(hypAssignment, "Long", 1, "hypAssignment")
    _check(gtPose, "Float", 2, "gtPose")
    if tuple(sceneCoordinates.shape)[1] != 3 or tuple(outGradients.shape) != tuple(sceneCoordinates.shape):
        raise RuntimeError("sceneCoordinates / outGradients must both be [E, 3, H, W]")
    if tuple(gtPose.shape) != (4, 4):
        raise RuntimeError("gtPose must be [4, 4]")
    co = _Arg(sceneCoordinates)
    gr = _Arg(outGradients, writable=True)
    gt = _Arg(gtPose)
    aptr, astride, M, adev, _keep = _assign_arg(hypAssignment)
    ctx = _pick_ctx(co.device, gr.device, gt.device, adev)
    E, _, H, W = (int(s) for s in sceneCoordinates.shape)
    loss = C.c_double(0.0)
    ctx.check(ctx.lib.esacb200_backward(ctx.handle, co.ptr, gr.ptr, E, H, W, aptr, astride, M, gt.ptr, float(wLossRot),
                                        float(wLossTrans), float(lossCut),
                                        *_camera_tail(shiftX, shiftY, focalLength, ppointX, ppointY, inlierThreshold,
                                                      inlierAlpha, inlierBeta, maxReproj, subSampling), C.byref(loss)))
    gr.finish()
    return float(loss.value)


def backward_sharded(sceneCoordinates, outGradients, hypAssignment, gtPose, wLossRot, wLossTrans, lossCut, shiftX, shiftY,
                     focalLength, ppointX, ppointY, inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling,
                     exchange, hyp_offset=0) -> float:
    """esac.backward on this rank's shard of the experts / hypotheses.  `exchange(phase, values) -> list` performs the two
    cross-rank reductions (see include/esac_b200.h); returns the GLOBAL expected loss."""
    _check(sceneCoordinates, "Float", 4, "sceneCoordinates")
    _check(outGradients, "Float", 4, "outGradients")
    _check(hypAssignment, "Long", 1, "hypAssignment")
    _check(gtPose, "Float", 2, "gtPose")
    co = _Arg(sceneCoordinates)
    gr = _Arg(outGradients, writable=True)
    gt = _Arg(gtPose)
    aptr, astride, M, adev, _keep = _assign_arg(hypAssignment)
    ctx = _pick_ctx(co.device, gr.device, gt.device, adev)
    E, _, H, W = (int(s) for s in sceneCoordinates.shape)
    err = []

    def _cb(user, phase, values, n):
        try:
            out = exchange(int(phase), [values[i] for i in range(n)])
            for i in range(n):
                values[i] = float(out[i])
            return 0
        except Exception as e:  # never let an exception cross the C boundary
            err.append(e)
            return 1

    cb = EXCHANGE_FN(_cb)
    loss = C.c_double(0.0)
    with _hypothesis_shard(ctx, hyp_offset):
        rc = ctx.lib.esacb200_backward_sharded(ctx.handle, co.ptr, gr.ptr, E, H, W, aptr, astride, M, gt.ptr, float(wLossRot),
                                               float(wLossTrans), float(lossCut),
                                               *_camera_tail(shiftX, shiftY, focalLength, ppointX, ppointY, inlierThreshold,
                                                             inlierAlpha, inlierBeta, maxReproj, subSampling),
                                               cb, None, C.byref(loss))
    if err:
        raise err[0]
    ctx.check(rc)
    gr.finish()
    return float(loss.value)


# ------------------------------------------------------------------------------------------------
# additive entry points
# ------------------------------------------------------------------------------------------------
def forward_batch(sceneCoordinates, hypAssignment, outPoses, shiftX, shiftY, focalLength, ppointX, ppointY,
                  inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling) -> list:
    """esac.forward over a batch: sceneCoordinates [B,E,3,H,W] float32, hypAssignment [B,M] int64 (contiguous rows),
    outPoses [B,4,4] float32 written in place.  Returns the winning expert of every image.  One host synchronisation
    for the whole batch; host tensors (pinned) are copied on a second stream while the previous image computes.
    shiftX, shiftY, focalLength, ppointX and ppointY are each a number (one camera for the batch) or B values -- a
    sequence, numpy array or 1-D tensor, e.g. the DataLoader's `focallength` -- giving image b its own shift and camera;
    image b then computes what esac.forward with those values computes.
    sceneCoordinates may also be a list or tuple of B [E,3,H_b,W_b] tensors (CPU, CUDA or numpy), each image with its own
    map size (a ragged batch); image b then computes what esac.forward on that tensor computes."""
    co = _Images(sceneCoordinates, 4, "sceneCoordinates")
    B, E = co.B, _check_maps(co.shapes, "sceneCoordinates")
    _check(hypAssignment, "Long", 2, "hypAssignment")
    _check(outPoses, "Float", 3, "outPoses")
    if tuple(outPoses.shape) != (B, 4, 4) or int(hypAssignment.shape[0]) != B:
        raise RuntimeError(f"a batch of {B} maps needs hypAssignment [{B},M] and outPoses [{B},4,4]")
    cams = _cameras(B, shiftX, shiftY, focalLength, ppointX, ppointY)
    op = _Arg(outPoses, writable=True)
    ha = _Arg(hypAssignment)
    M = int(hypAssignment.shape[1])
    ctx = _pick_ctx(*co.devices, op.device, ha.device)
    experts = (C.c_int * B)()
    ctx.check(ctx.lib.esacb200_forward_ragged(ctx.handle, B, co.ptrs, co.hs, co.ws, E, ha.ptr, 1, M, op.ptr,
                                              *(a.ctypes.data for a in cams),
                                              *_thresholds(inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling),
                                              experts))
    op.finish()
    return [int(e) for e in experts]


def backward_batch(sceneCoordinates, outGradients, hypAssignment, gtPoses, wLossRot, wLossTrans, lossCut, shiftX, shiftY,
                   focalLength, ppointX, ppointY, inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling) -> list:
    """esac.backward over a batch: sceneCoordinates / outGradients [B,E,3,H,W] float32 (gradients accumulated in place),
    hypAssignment [B,M] int64, gtPoses [B,4,4] float32 (camera->world), shiftX / shiftY an int or a sequence of B ints
    (train_esac.py:125 draws one shift per image), focalLength / ppointX / ppointY a number or B values (one camera per
    image, as forward_batch).  Returns the expected loss of every image; equal, image by image, to B consecutive
    esac.backward calls on the same context, each with its image's shift and camera.
    sceneCoordinates and outGradients may also be lists or tuples of B [E,3,H_b,W_b] tensors (a ragged batch, as for
    forward_batch); outGradients[b] has the shape of sceneCoordinates[b]."""
    co = _Images(sceneCoordinates, 4, "sceneCoordinates")
    B, E = co.B, _check_maps(co.shapes, "sceneCoordinates")
    og = _Images(outGradients, 4, "outGradients", writable=True, like=co)
    og.require_shapes_of(co)
    _check(hypAssignment, "Long", 2, "hypAssignment")
    _check(gtPoses, "Float", 3, "gtPoses")
    if tuple(gtPoses.shape) != (B, 4, 4) or int(hypAssignment.shape[0]) != B:
        raise RuntimeError(f"a batch of {B} maps needs hypAssignment [{B},M] and gtPoses [{B},4,4]")
    cams = _cameras(B, shiftX, shiftY, focalLength, ppointX, ppointY)
    ha = _Arg(hypAssignment)
    gt = _Arg(gtPoses)
    M = int(hypAssignment.shape[1])
    ctx = _pick_ctx(*co.devices, *og.devices, ha.device, gt.device)
    losses = np.zeros(B, np.float64)
    ctx.check(ctx.lib.esacb200_backward_ragged(ctx.handle, B, co.ptrs, og.ptrs, co.hs, co.ws, E, ha.ptr, 1, M, gt.ptr,
                                               float(wLossRot), float(wLossTrans), float(lossCut),
                                               *(a.ctypes.data for a in cams),
                                               *_thresholds(inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling),
                                               losses.ctypes.data))
    og.finish()
    return [float(v) for v in losses]


def assign_hypotheses(gatingProbs, hypotheses: int, seed: int, maxExperts: int = -1, expertSelection: bool = False):
    """The callers' hypothesis assignment (util.clamp_probs + torch.multinomial(replacement=True) + torch.histc,
    train_esac.py:130-140, test_esac.py:169-177) for a batch of gating outputs, on the device.  gatingProbs [B,E] float32
    (CPU, CUDA or numpy; need not be normalised).  Returns (e_hyps int64 [B,M], e_hyps_hist float32 [B,E]) of the same
    kind as the input.  A pure function of (seed, image, hypothesis); see oracle.esac_oracle.assign_hypotheses."""
    _check(gatingProbs, "Float", 2, "gatingProbs")
    B, E = (int(v) for v in gatingProbs.shape)
    M = int(hypotheses)
    gp = _Arg(gatingProbs)
    if _is_torch(gatingProbs):
        import torch
        assign = torch.empty((B, M), dtype=torch.int64, device=gatingProbs.device)
        hist = torch.empty((B, E), dtype=torch.float32, device=gatingProbs.device)
        ap, hp = assign.data_ptr(), hist.data_ptr()
    else:
        assign = np.empty((B, M), np.int64)
        hist = np.empty((B, E), np.float32)
        ap, hp = assign.ctypes.data, hist.ctypes.data
    ctx = _pick_ctx(gp.device)
    ctx.check(ctx.lib.esacb200_assign_hypotheses(ctx.handle, B, E, M, gp.ptr, int(maxExperts), int(bool(expertSelection)),
                                                 int(seed) & 0xFFFFFFFFFFFFFFFF, ap, hp))
    return assign, hist


MAX_EXPERTS = 1024  # experts one assignment CTA holds, and handles one ExpertGate holds (include/esac_b200.h)


def assign_hypotheses_async(gatingProbs, hypotheses, seed, outAssign, outHist, outStatus, maxExperts: int = -1,
                            expertSelection: bool = False):
    """assign_hypotheses enqueued on torch's current stream with no host synchronisation, so that a CUDA graph can capture
    the draw.  CUDA tensors only: gatingProbs float32 [B,E] (or [E]), seed int64 [1] (or []), read when the kernel runs --
    a graph can advance it (seed.add_(1) in the capture) or the caller can write a new one before each replay; the results
    go to outAssign int64 [B,M] (M = hypotheses), outHist float32 [B,E] or None and outStatus int32 [B] (0; 1 for a row
    with a negative, NaN or infinite probability; 2 for a row that sums to 0 -- where assign_hypotheses raises; that row's
    draws are then meaningless).  Given the same seed value it draws bitwise what assign_hypotheses draws."""
    call = "assign_hypotheses_async"
    if not _is_torch(gatingProbs):
        raise RuntimeError(f"{call} takes torch CUDA tensors only (gatingProbs is a {type(gatingProbs).__name__})")
    if _dtype_name(gatingProbs) != "Float":
        raise RuntimeError(f"expected scalar type Float but found {_dtype_name(gatingProbs)} (gatingProbs)")
    if gatingProbs.dim() not in (1, 2):
        raise RuntimeError(f"gatingProbs must be [B,E] or [E], got {list(gatingProbs.shape)}")
    lead = tuple(int(v) for v in gatingProbs.shape[:-1])
    B, E, M = (lead[0] if lead else 1), int(gatingProbs.shape[-1]), int(hypotheses)
    if B < 1 or E < 1 or M < 1:
        raise RuntimeError(f"{call}: sizes must be positive, got B={B} E={E} M={M}")
    if E > MAX_EXPERTS:
        raise RuntimeError(f"{call}: E={E} exceeds the {MAX_EXPERTS} experts one CTA holds")
    if not _is_torch(seed) or _dtype_name(seed) != "Long" or int(seed.numel()) != 1:
        raise RuntimeError(f"seed must be an int64 CUDA tensor of one element, got "
                           f"{_dtype_name(seed) if _is_torch(seed) else type(seed).__name__}"
                           f"{list(seed.shape) if _is_torch(seed) else ''}")
    fixed = {"outAssign": (outAssign, "Long", lead + (M,)), "outStatus": (outStatus, "Int", lead)}
    if outHist is not None:
        fixed["outHist"] = (outHist, "Float", lead + (E,))

    def check():
        if not gatingProbs.is_contiguous():
            raise RuntimeError("gatingProbs must be contiguous (a copy would not be captured with the call)")
    ctx = _async_context(call, fixed, [("gatingProbs", gatingProbs), ("seed", seed)], check)
    ctx.check(ctx.lib.esacb200_assign_hypotheses_async(ctx.handle, B, E, M, gatingProbs.data_ptr(), int(maxExperts),
                                                       int(bool(expertSelection)), seed.data_ptr(), outAssign.data_ptr(),
                                                       outHist.data_ptr() if outHist is not None else None,
                                                       outStatus.data_ptr()))


# The C ABI's dtype codes of the typed loss calls (ESACB200_FLOAT32, _FLOAT16, _BFLOAT16), by _dtype_name.
_LOSS_DTYPES = {"Float": 0, "Half": 1, "BFloat16": 2}
_AMP = ("Half", "BFloat16")


def _grad_scale(gradScale, call: str):
    """gradScale of the _amp losses: None (a scale of 1) or a CUDA float32 tensor of one element, read on the device when
    the kernels run.  Returns its (name, tensor) pair for the device checks, or nothing.  Raises before any context exists."""
    if gradScale is None:
        return []
    if not (_is_torch(gradScale) and gradScale.is_cuda and _dtype_name(gradScale) == "Float" and gradScale.numel() == 1):
        kind = (f"a {'CUDA' if gradScale.is_cuda else 'CPU'} {_dtype_name(gradScale)} tensor of {gradScale.numel()} elements"
                if _is_torch(gradScale) else f"a {type(gradScale).__name__}")
        raise RuntimeError(f"{call}: gradScale must be a CUDA float32 tensor of one element or None, got {kind}")
    return [("gradScale", gradScale)]


def _amp_on_cuda(call: str, images, scale):
    """The image arguments (and gradScale) of an eager _amp loss are CUDA tensors (the 16-bit kernels read device memory)."""
    for what, t in _image_tensors(images) + scale:
        if not _is_torch(t):
            raise RuntimeError(f"{call} takes torch CUDA tensors only ({what} is a {type(t).__name__})")
        if not t.is_cuda:
            raise RuntimeError(f"{call} takes CUDA tensors only ({what} is on the CPU)")


def _reproj_loss(call, prediction, gtPoses, focalLength, padX, padY, cutLoss, subSampling, ppointX, ppointY, outGradients,
                 maxReproj, minDepth, gradScale):
    """reproj_loss (call None: float32 maps) or reproj_loss_amp (call "reproj_loss_amp": float16 / bfloat16 CUDA maps)."""
    pr = _Images(prediction, 3, "prediction", dtypes=_AMP if call else "Float")
    B = pr.B
    _check(gtPoses, "Float", 3, "gtPoses")
    if tuple(gtPoses.shape) != (B, 4, 4):
        raise RuntimeError(f"a batch of {B} predictions needs gtPoses [{B},4,4]")
    og = None
    if outGradients is not None:
        og = _Images(outGradients, 3, "outGradients", writable=True, like=pr, dtypes=pr.dtype)
        og.require_shapes_of(pr)
    scale = _grad_scale(gradScale, call) if call else []
    if call:
        _amp_on_cuda(call, [pr] + ([og] if og else []), scale)
    # the default principal point is the centre of each image's own sub*W x sub*H frame
    ppx = [s[2] * subSampling / 2 for s in pr.shapes] if ppointX is None else ppointX
    ppy = [s[1] * subSampling / 2 for s in pr.shapes] if ppointY is None else ppointY
    cams = _cameras(B, padX, padY, focalLength, ppx, ppy, ("padX", "padY"))
    gt = _Arg(gtPoses)
    ctx = _pick_ctx(*pr.devices, *(og.devices if og else ()), gt.device, *(t.device.index for _, t in scale))
    losses = np.zeros(B, np.float64)
    args = (pr.ptrs, og.ptrs if og else None, pr.hs, pr.ws, gt.ptr, *(a.ctypes.data for a in cams), int(subSampling),
            float(cutLoss), float(maxReproj), float(minDepth))
    if call:
        ctx.check(ctx.lib.esacb200_reproj_loss_ragged_typed(ctx.handle, B, _LOSS_DTYPES[pr.dtype], *args,
                                                            gradScale.data_ptr() if scale else None, losses.ctypes.data))
    else:
        ctx.check(ctx.lib.esacb200_reproj_loss_ragged(ctx.handle, B, *args, losses.ctypes.data))
    if og:
        og.finish()
    return [float(v) for v in losses]


def reproj_loss(prediction, gtPoses, focalLength, padX, padY, cutLoss, subSampling=8, ppointX=None, ppointY=None,
                outGradients=None, maxReproj=100.0, minDepth=0.1):
    """The robust reprojection loss of ref_expert.py:103-148 and, when outGradients is given, d loss / d prediction in the
    same pass (what `robust_loss.backward()` hands to the expert, ref_expert.py:150).  prediction [B,3,H,W] float32 (the
    reference has B = 1), gtPoses [B,4,4] float32 camera->world, padX / padY an int or B ints (the random shift),
    outGradients [B,3,H,W] float32 written in place (overwritten) or None.  focalLength, ppointX and ppointY are a number
    or B values (one camera per image, e.g. the DataLoader's `focallength`); the principal point defaults to the centre
    of the sub*W x sub*H image (ref_expert.py:118-119).  Returns the B losses.
    prediction (and outGradients) may also be lists or tuples of B [3,H_b,W_b] tensors (a ragged batch); the default
    principal point is then each image's own centre, and image b gives bitwise the loss and gradient of a call on it alone."""
    return _reproj_loss(None, prediction, gtPoses, focalLength, padX, padY, cutLoss, subSampling, ppointX, ppointY,
                        outGradients, maxReproj, minDepth, None)


def reproj_loss_amp(prediction, gtPoses, focalLength, padX, padY, cutLoss, subSampling=8, ppointX=None, ppointY=None,
                    outGradients=None, maxReproj=100.0, minDepth=0.1, gradScale=None):
    """reproj_loss on a float16 or bfloat16 prediction, as an expert trained under torch.autocast produces it: CUDA tensors
    only, prediction [B,3,H,W] or a list / tuple of B [3,H_b,W_b] tensors of one dtype, outGradients of the prediction's
    dtype, form and shapes (overwritten) or None; gtPoses and the camera as for reproj_loss (float32).  Each loss is
    bitwise reproj_loss's on prediction.float() (for maps on the same load path: aligned alike).  Each gradient is
    reproj_loss's gradient g on prediction.float(), times gradScale (a CUDA float32 tensor of one element, read on the
    device; None = 1) as one float32 multiply, rounded to the prediction's dtype: bitwise what autograd hands a 16-bit
    prediction through prediction.float() when the loss's upstream gradient is gradScale."""
    return _reproj_loss("reproj_loss_amp", prediction, gtPoses, focalLength, padX, padY, cutLoss, subSampling, ppointX,
                        ppointY, outGradients, maxReproj, minDepth, gradScale)


def _coord_loss(call, prediction, gtCoords, cutLoss, outGradients, return_counts, gradScale):
    """coord_loss (call None: float32 maps) or coord_loss_amp (call "coord_loss_amp": float16 / bfloat16 CUDA maps)."""
    pr = _Images(prediction, 3, "prediction", dtypes=_AMP if call else "Float")
    gt = _Images(gtCoords, 3, "gtCoords", like=pr)
    for b, ((_, hp, wp), (_, hg, wg)) in enumerate(zip(pr.shapes, gt.shapes)):
        if abs(hp - hg) > 1 or abs(wp - wg) > 1:
            raise RuntimeError(f"image {b}: tensor size mismatch: prediction {hp}x{wp}, ground truth {hg}x{wg} "
                               "(util.assert_size allows 1)")
    og = None
    if outGradients is not None:
        og = _Images(outGradients, 3, "outGradients", writable=True, like=pr, dtypes=pr.dtype)
        og.require_shapes_of(pr)
    scale = _grad_scale(gradScale, call) if call else []
    if call:
        _amp_on_cuda(call, [pr, gt] + ([og] if og else []), scale)
    ctx = _pick_ctx(*pr.devices, *gt.devices, *(og.devices if og else ()), *(t.device.index for _, t in scale))
    losses = np.zeros(pr.B, np.float64)
    counts = np.zeros(pr.B, np.int64)
    args = (pr.ptrs, pr.hs, pr.ws, gt.ptrs, gt.hs, gt.ws, og.ptrs if og else None, float(cutLoss))
    if call:
        ctx.check(ctx.lib.esacb200_coord_loss_ragged_typed(ctx.handle, pr.B, _LOSS_DTYPES[pr.dtype], *args,
                                                           gradScale.data_ptr() if scale else None, losses.ctypes.data,
                                                           counts.ctypes.data))
    else:
        ctx.check(ctx.lib.esacb200_coord_loss_ragged(ctx.handle, pr.B, *args, losses.ctypes.data, counts.ctypes.data))
    if og:
        og.finish()
    out = [float(v) for v in losses]
    return (out, [int(v) for v in counts]) if return_counts else out


def coord_loss(prediction, gtCoords, cutLoss=100.0, outGradients=None, return_counts=False):
    """The robust scene-coordinate loss of init_expert.py:106-130 and, when outGradients is given, d loss / d prediction in
    the same call (what `robust_loss.backward()` hands to the expert, :132).  prediction [B,3,Hp,Wp] float32 (the reference
    has B = 1), gtCoords [B,3,Hg,Wg] float32; the two may differ by at most 1 in H and in W and are cropped to the common
    top-left window (util.assert_size).  Cells whose ground truth is all zero do not count; the loss of an image is the sum
    over its valid cells divided by their number (NaN if there is none).  outGradients [B,3,Hp,Wp] float32 is overwritten
    (0 outside the window and on invalid cells) or None for the loss alone.  Returns the B losses, and with return_counts
    also the B valid-cell counts.
    prediction, gtCoords (and outGradients) may also all be lists or tuples of B [3,H_b,W_b] tensors (a ragged batch), each
    pair at most 1 apart; image b gives bitwise the loss and gradient of a call on it alone."""
    return _coord_loss(None, prediction, gtCoords, cutLoss, outGradients, return_counts, None)


def coord_loss_amp(prediction, gtCoords, cutLoss=100.0, outGradients=None, return_counts=False, gradScale=None):
    """coord_loss on a float16 or bfloat16 prediction (torch.autocast): CUDA tensors only, prediction [B,3,Hp,Wp] or a list
    / tuple of B [3,H_b,W_b] tensors of one dtype, gtCoords float32 in the prediction's form, outGradients of the
    prediction's dtype, form and shapes (overwritten) or None.  The losses and counts are bitwise coord_loss's on
    prediction.float(); each gradient is coord_loss's gradient on prediction.float(), times gradScale (a CUDA float32
    tensor of one element, read on the device; None = 1) as one float32 multiply, rounded to the prediction's dtype."""
    return _coord_loss("coord_loss_amp", prediction, gtCoords, cutLoss, outGradients, return_counts, gradScale)


def nccl_unique_id() -> bytes:
    """128-byte ncclUniqueId (call on one rank, distribute to the others, then Context.comm_init on every rank)."""
    buf = C.create_string_buffer(128)
    rc = load_library().esacb200_nccl_unique_id(buf)
    if rc != 0:
        raise RuntimeError(f"esac_b200: ncclGetUniqueId failed (status {rc}); is libnccl.so.2 loadable?")
    return buf.raw


def forward_pack(sceneCoordinates, hypAssignment, params, expert_offset: int, pack_out, M_pad: int | None = None):
    """The local half of a sharded forward, enqueued on the current CUDA stream without a host synchronisation
    (esacb200_forward_pack).  sceneCoordinates [E,3,H,W] / hypAssignment [M] are CUDA tensors, params the positional tail of
    esac.forward (shiftX .. subSampling), pack_out a CUDA float64 tensor of M_pad + 21 elements (see include/esac_b200.h);
    M_pad (default M) = the largest M of any shard."""
    _check(sceneCoordinates, "Float", 4, "sceneCoordinates")
    _check(hypAssignment, "Long", 1, "hypAssignment")
    if not (_is_torch(sceneCoordinates) and sceneCoordinates.is_cuda and hypAssignment.is_cuda and pack_out.is_cuda):
        raise RuntimeError("forward_pack takes CUDA tensors")
    co = _Arg(sceneCoordinates)
    aptr, astride, M, adev, _keep = _assign_arg(hypAssignment)
    M_pad = M if M_pad is None else int(M_pad)
    if pack_out.dtype != __import__("torch").float64 or pack_out.numel() != M_pad + PACK_TAIL or not pack_out.is_contiguous():
        raise RuntimeError(f"pack_out must be a contiguous float64 tensor of M_pad + {PACK_TAIL} elements")
    ctx = _pick_ctx(co.device, adev, pack_out.device.index)
    E, _, H, W = (int(v) for v in sceneCoordinates.shape)
    ctx.check(ctx.lib.esacb200_forward_pack(ctx.handle, co.ptr, E, H, W, aptr, astride, M, M_pad, *_camera_tail(*params),
                                            int(expert_offset), pack_out.data_ptr()))


def forward_sharded(sceneCoordinates, hypAssignment, outPose, shiftX, shiftY, focalLength, ppointX, ppointY, inlierThreshold,
                    inlierAlpha, inlierBeta, maxReproj, subSampling, expert_offset: int = 0, M_pad: int | None = None,
                    hyp_offset: int = 0, device: int | None = None, hyp_stride: int = 1) -> int:
    """esac.forward over experts / hypotheses sharded across the ranks of the library's communicator (Context.comm_init):
    this rank's shard in, the GLOBAL winner's pose (outPose, in place) and expert index out, on every rank.  One
    ncclAllGather on the library's stream, no torch collective.  hypAssignment may be empty (M = 0)."""
    _check(sceneCoordinates, "Float", 4, "sceneCoordinates")
    _check(hypAssignment, "Long", 1, "hypAssignment")
    _check(outPose, "Float", 2, "outPose")
    co = _Arg(sceneCoordinates)
    op = _Arg(outPose, writable=True)
    aptr, astride, M, adev, _keep = _assign_arg(hypAssignment)
    M_pad = max(M, 1) if M_pad is None else int(M_pad)
    devs = [d for d in (co.device, op.device, adev) if d is not None]
    ctx = _pick_ctx(*devs) if devs else _pick_ctx_host(device)
    E, _, H, W = (int(s) for s in sceneCoordinates.shape)
    expert = C.c_int(-1)
    with _hypothesis_shard(ctx, hyp_offset, hyp_stride):
        rc = ctx.lib.esacb200_forward_sharded(ctx.handle, co.ptr, E, H, W, aptr, astride, M, M_pad, op.ptr,
                                              *_camera_tail(shiftX, shiftY, focalLength, ppointX, ppointY, inlierThreshold,
                                                            inlierAlpha, inlierBeta, maxReproj, subSampling),
                                              int(expert_offset), C.byref(expert))
    ctx.check(rc)
    op.finish()
    return int(expert.value)


def backward_sharded_nccl(sceneCoordinates, outGradients, hypAssignment, gtPose, wLossRot, wLossTrans, lossCut, shiftX, shiftY,
                          focalLength, ppointX, ppointY, inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling,
                          hyp_offset: int = 0, device: int | None = None, reduce_grads: bool = False, hyp_stride: int = 1) -> float:
    """esac.backward on this rank's shard; the two exchanges run as NCCL collectives inside the library.  Returns the GLOBAL
    expected loss; outGradients receives this shard's gradient slices, or -- reduce_grads, hypothesis-major sharding with all
    planes on every rank -- the gradient summed over all ranks.  hypAssignment may be empty."""
    _check(sceneCoordinates, "Float", 4, "sceneCoordinates")
    _check(outGradients, "Float", 4, "outGradients")
    _check(hypAssignment, "Long", 1, "hypAssignment")
    _check(gtPose, "Float", 2, "gtPose")
    co = _Arg(sceneCoordinates)
    gr = _Arg(outGradients, writable=True)
    gt = _Arg(gtPose)
    aptr, astride, M, adev, _keep = _assign_arg(hypAssignment)
    devs = [d for d in (co.device, gr.device, gt.device, adev) if d is not None]
    ctx = _pick_ctx(*devs) if devs else _pick_ctx_host(device)
    E, _, H, W = (int(s) for s in sceneCoordinates.shape)
    loss = C.c_double(0.0)
    with _hypothesis_shard(ctx, hyp_offset, hyp_stride):
        rc = ctx.lib.esacb200_backward_sharded_nccl(ctx.handle, co.ptr, gr.ptr, E, H, W, aptr, astride, M, gt.ptr, float(wLossRot),
                                                    float(wLossTrans), float(lossCut),
                                                    *_camera_tail(shiftX, shiftY, focalLength, ppointX, ppointY, inlierThreshold,
                                                                  inlierAlpha, inlierBeta, maxReproj, subSampling),
                                                    int(bool(reduce_grads)), C.byref(loss))
    ctx.check(rc)
    gr.finish()
    return float(loss.value)


def score_poses(sceneCoordinates, hypAssignment, poses6, shiftX, shiftY, focalLength, ppointX, ppointY,
                inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling) -> np.ndarray:
    """Soft-inlier scores (getReproErrs + getHypScores) of given scene poses [M, 6] = (rvec, tvec)."""
    _check(sceneCoordinates, "Float", 4, "sceneCoordinates")
    _check(hypAssignment, "Long", 1, "hypAssignment")
    co = _Arg(sceneCoordinates)
    aptr, astride, M, adev, _keep = _assign_arg(hypAssignment)
    poses6 = np.ascontiguousarray(poses6, np.float64)
    assert poses6.shape == (M, 6)
    ctx = _pick_ctx(co.device, adev)
    E, _, H, W = (int(s) for s in sceneCoordinates.shape)
    out = np.zeros(M)
    ctx.check(ctx.lib.esacb200_score_poses(ctx.handle, co.ptr, E, H, W, aptr, astride, M, poses6.ctypes.data,
                                           *_camera_tail(shiftX, shiftY, focalLength, ppointX, ppointY, inlierThreshold,
                                                         inlierAlpha, inlierBeta, maxReproj, subSampling), out.ctypes.data))
    return out


def refine_poses(sceneCoordinates, hypAssignment, poses6, shiftX, shiftY, focalLength, ppointX, ppointY,
                 inlierThreshold, maxReproj, subSampling):
    """refineHyp for every given pose.  Returns (refined [M, 6], accepted rounds [M], final inlier counts [M])."""
    _check(sceneCoordinates, "Float", 4, "sceneCoordinates")
    _check(hypAssignment, "Long", 1, "hypAssignment")
    co = _Arg(sceneCoordinates)
    aptr, astride, M, adev, _keep = _assign_arg(hypAssignment)
    poses6 = np.array(poses6, np.float64, order="C", copy=True)
    assert poses6.shape == (M, 6)
    ctx = _pick_ctx(co.device, adev)
    E, _, H, W = (int(s) for s in sceneCoordinates.shape)
    rounds = np.zeros(M, np.int32)
    inl = np.zeros(M, np.int32)
    ctx.check(ctx.lib.esacb200_refine_poses(ctx.handle, co.ptr, E, H, W, aptr, astride, M, poses6.ctypes.data, int(shiftX),
                                            int(shiftY), float(focalLength), float(ppointX), float(ppointY),
                                            float(inlierThreshold), float(maxReproj), int(subSampling),
                                            rounds.ctypes.data, inl.ctypes.data))
    return poses6, rounds, inl


# ------------------------------------------------------------------------------------------------
# the hypotheses as a differentiable function (the layer under autograd.esac_hypotheses)
# ------------------------------------------------------------------------------------------------
def hypotheses_tape_bytes(E: int, H: int, W: int, M: int) -> int:
    """Bytes of the tape a hypotheses forward of M hypotheses on [E,3,H,W] maps leaves for its backward (no device needed)."""
    return int(load_library().esacb200_hypotheses_tape_bytes(int(E), int(H), int(W), int(M)))


PROB_THRESH = 1e-3  # the reference's probability threshold (ESACB200_PROB_THRESH): the hypotheses node's default floor


def _min_prob(minProb, call: str, name: str = "minProb") -> float:
    """The hypotheses node's probability floor (argument `name` of `call`) as a float in [0, 1], NaN refused; raises
    RuntimeError before any context exists, so the check runs without a GPU."""
    if isinstance(minProb, (bool, np.bool_)) or not isinstance(minProb, numbers.Real):
        raise RuntimeError(f"{call}: {name} must be a number in [0, 1], got a {type(minProb).__name__}")
    v = float(minProb)
    if not 0.0 <= v <= 1.0:
        raise RuntimeError(f"{call}: {name} must lie in [0, 1], got {v}")
    return v


def _floor_entry(lib, name: str, minProb: float):
    """esacb200_`name` and the floor arguments it takes after subSampling: at the default floor the entry point without
    one (which is the _floor entry point with ESACB200_PROB_THRESH), else esacb200_`name`_floor with minProb."""
    if minProb == PROB_THRESH:
        return getattr(lib, "esacb200_" + name), ()
    return getattr(lib, f"esacb200_{name}_floor"), (minProb,)


def _out_device(a: _Arg):
    import torch
    return torch.device("cuda", a.device) if a.is_cuda else torch.device("cpu")


def hypotheses_forward(sceneCoordinates, hypAssignment, shiftX, shiftY, focalLength, ppointX, ppointY, inlierThreshold,
                       inlierAlpha, inlierBeta, maxReproj, subSampling, minProb=PROB_THRESH):
    """The hypotheses of an esac.backward call at the same point of the context's call sequence: the same draws, scores and
    refinements.  Returns torch tensors (scores float64 [M], poses float64 [M,6] = (rvec, tvec), refined where p >=
    minProb and initial elsewhere, contributing bool [M] = p >= minProb) on the coordinates' device (CPU for numpy input),
    and the tape: a CUDA uint8 tensor holding what hypotheses_backward needs.  p is the hypothesis's softmax probability;
    minProb in [0, 1] (default PROB_THRESH, the reference's truncation; 0 = every hypothesis, also those whose p underflows
    to 0).  Runs on torch's current stream."""
    minProb = _min_prob(minProb, "hypotheses_forward")
    _check(sceneCoordinates, "Float", 4, "sceneCoordinates")
    _check(hypAssignment, "Long", 1, "hypAssignment")
    E, three, H, W = (int(s) for s in sceneCoordinates.shape)
    if three != 3:
        raise RuntimeError("sceneCoordinates must be [E, 3, H, W]")
    if (W - 1) * (H - 1) < 4:
        raise RuntimeError(f"sceneCoordinates: map {W}x{H} too small to draw 4 distinct cells")
    if int(hypAssignment.shape[0]) < 1:
        raise RuntimeError("hypAssignment holds no hypothesis")
    import torch
    co = _Arg(sceneCoordinates)
    aptr, astride, M, adev, _keep = _assign_arg(hypAssignment)
    ctx = _pick_ctx(co.device, adev)
    if co.device is None and adev is None:  # the tape is a CUDA tensor: order the call on torch's stream all the same
        ctx.set_stream(torch.cuda.current_stream(ctx.device).cuda_stream or _CUDA_STREAM_LEGACY)
    dev = _out_device(co)
    nbytes = hypotheses_tape_bytes(E, H, W, M)
    tape = torch.empty(nbytes, dtype=torch.uint8, device=torch.device("cuda", ctx.device))
    scores = torch.empty(M, dtype=torch.float64, device=dev)
    poses = torch.empty(M, 6, dtype=torch.float64, device=dev)
    contributing = torch.empty(M, dtype=torch.bool, device=dev)
    fn, floor = _floor_entry(ctx.lib, "hypotheses_forward", minProb)
    ctx.check(fn(ctx.handle, co.ptr, E, H, W, aptr, astride, M,
                 *_camera_tail(shiftX, shiftY, focalLength, ppointX, ppointY, inlierThreshold, inlierAlpha, inlierBeta,
                               maxReproj, subSampling),
                 *floor, tape.data_ptr(), nbytes, scores.data_ptr(), poses.data_ptr(), contributing.data_ptr()))
    return scores, poses, contributing, tape


def hypotheses_backward(tape, sceneCoordinates, outGradients, gradScores=None, gradPoses=None):
    """Accumulates (+=) into outGradients [E,3,H,W] the gradient of the scene coordinates for upstream gradients gradScores
    (float64 [M]) and gradPoses (float64 [M,6]) of a hypotheses_forward's outputs; None counts as zero, and entries of
    hypotheses that do not contribute (p < the forward's minProb) are ignored.  sceneCoordinates must hold the values the forward saw."""
    _check(sceneCoordinates, "Float", 4, "sceneCoordinates")
    _check(outGradients, "Float", 4, "outGradients")
    shape = tuple(int(s) for s in sceneCoordinates.shape)
    if shape[1] != 3 or tuple(int(s) for s in outGradients.shape) != shape:
        raise RuntimeError("sceneCoordinates / outGradients must both be [E, 3, H, W]")
    M = None
    if gradScores is not None:
        _check(gradScores, "Double", 1, "gradScores")
        M = int(gradScores.shape[0])
    if gradPoses is not None:
        _check(gradPoses, "Double", 2, "gradPoses")
        if int(gradPoses.shape[1]) != 6 or (M is not None and int(gradPoses.shape[0]) != M):
            raise RuntimeError(f"gradPoses must be [M, 6] with the M of gradScores, got {list(gradPoses.shape)}")
        M = int(gradPoses.shape[0])
    if not (_is_torch(tape) and tape.is_cuda and str(tape.dtype) == "torch.uint8" and tape.dim() == 1 and tape.is_contiguous()):
        raise RuntimeError("tape must be the contiguous CUDA uint8 tensor hypotheses_forward returned")
    E, _, H, W = shape
    if M is not None and int(tape.numel()) != hypotheses_tape_bytes(E, H, W, M):
        raise RuntimeError(f"the tape is not that of a forward of {M} hypotheses on [{E}, 3, {H}, {W}] maps")
    co = _Arg(sceneCoordinates)
    gr = _Arg(outGradients, writable=True)
    gs = _Arg(gradScores) if gradScores is not None else None
    gp = _Arg(gradPoses) if gradPoses is not None else None
    ctx = _pick_ctx(co.device, gr.device, tape.device.index, gs.device if gs else None, gp.device if gp else None)
    ctx.check(ctx.lib.esacb200_hypotheses_backward(ctx.handle, tape.data_ptr(), co.ptr, gr.ptr, E, H, W,
                                                   gs.ptr if gs else None, gp.ptr if gp else None))
    gr.finish()


def _tape_hypotheses(tape, E: int, H: int, W: int, what: str) -> int:
    """The number of hypotheses a tape of this size holds for [E,3,H,W] maps (tape_bytes is affine in M)."""
    if not (_is_torch(tape) and tape.is_cuda and str(tape.dtype) == "torch.uint8" and tape.dim() == 1 and tape.is_contiguous()):
        raise RuntimeError(f"{what} must be a contiguous CUDA uint8 tensor hypotheses_forward_batch returned")
    one = hypotheses_tape_bytes(E, H, W, 1)
    per = hypotheses_tape_bytes(E, H, W, 2) - one
    n = int(tape.numel()) - (one - per)
    if n < per or n % per:
        raise RuntimeError(f"{what} is not the tape of a forward on [{E}, 3, {H}, {W}] maps")
    return n // per


def hypotheses_forward_batch(sceneCoordinates, hypAssignment, shiftX, shiftY, focalLength, ppointX, ppointY, inlierThreshold,
                             inlierAlpha, inlierBeta, maxReproj, subSampling, minProb=PROB_THRESH):
    """hypotheses_forward over a batch: image b draws, scores and refines what the b-th of B consecutive hypotheses_forward
    (or esac.backward) calls would, with its own shift and camera.  sceneCoordinates [B,E,3,H,W] float32 or a list / tuple of
    B [E,3,H_b,W_b] tensors; hypAssignment int64 [B,M] (a stride-0 [B,1].expand(B,M) included); shiftX, shiftY,
    focalLength, ppointX, ppointY each a number or B values.  Returns scores float64 [B,M], poses float64 [B,M,6],
    contributing bool [B,M] on the coordinates' device (CPU for numpy input), and the B tapes: views into one CUDA uint8
    tensor, each at a 256-byte aligned offset.  minProb: hypotheses_forward's, one floor for every image.  The images run on
    worker streams (option batch_workers) after everything queued on torch's current stream."""
    minProb = _min_prob(minProb, "hypotheses_forward_batch")
    maps = _Images(sceneCoordinates, 4, "sceneCoordinates")
    B, E = maps.B, _check_maps(maps.shapes, "sceneCoordinates")
    _check(hypAssignment, "Long", 2, "hypAssignment")
    if int(hypAssignment.shape[0]) != B:
        raise RuntimeError(f"hypAssignment must be [{B}, M] for {B} images, got {list(hypAssignment.shape)}")
    M = int(hypAssignment.shape[1])
    if M < 1:
        raise RuntimeError("hypAssignment holds no hypothesis")
    cams = _cameras(B, shiftX, shiftY, focalLength, ppointX, ppointY)
    import torch
    ha = _Arg(hypAssignment)
    ctx = _pick_ctx(*maps.devices, ha.device)
    if all(d is None for d in maps.devices) and ha.device is None:  # the tapes are CUDA tensors: follow torch's stream
        ctx.set_stream(torch.cuda.current_stream(ctx.device).cuda_stream or _CUDA_STREAM_LEGACY)
    dev = _out_device(maps.args[0])
    sizes = [hypotheses_tape_bytes(E, h, w, M) for h, w in zip(maps.hs, maps.ws)]
    offsets = np.cumsum([0] + [(n + 255) // 256 * 256 for n in sizes])
    buf = torch.empty(int(offsets[-1]), dtype=torch.uint8, device=torch.device("cuda", ctx.device))
    tapes = [buf[int(o):int(o) + n] for o, n in zip(offsets, sizes)]
    scores = torch.empty(B, M, dtype=torch.float64, device=dev)
    poses = torch.empty(B, M, 6, dtype=torch.float64, device=dev)
    contributing = torch.empty(B, M, dtype=torch.bool, device=dev)
    tape_ptrs = (C.c_void_p * B)(*[t.data_ptr() for t in tapes])
    tape_sizes = (C.c_size_t * B)(*sizes)
    fn, floor = _floor_entry(ctx.lib, "hypotheses_forward_ragged", minProb)
    ctx.check(fn(
        ctx.handle, B, maps.ptrs, maps.hs, maps.ws, E, ha.ptr, 1, M, *(a.ctypes.data for a in cams),
        *_thresholds(inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling), *floor, tape_ptrs, tape_sizes,
        scores.data_ptr(), poses.data_ptr(), contributing.data_ptr()))
    return scores, poses, contributing, tapes


def hypotheses_backward_batch(tapes, sceneCoordinates, outGradients, gradScores=None, gradPoses=None):
    """hypotheses_backward over a batch: accumulates (+=) into outGradients[b] what hypotheses_backward on tapes[b] with
    gradScores[b] / gradPoses[b] would add.  sceneCoordinates / outGradients [B,E,3,H,W] float32 or lists / tuples of B
    [E,3,H_b,W_b] tensors of the forward's shapes; gradScores float64 [B,M] and gradPoses float64 [B,M,6], None = zero."""
    maps = _Images(sceneCoordinates, 4, "sceneCoordinates")
    B, E = maps.B, _check_maps(maps.shapes, "sceneCoordinates")
    grads = _Images(outGradients, 4, "outGradients", writable=True, like=maps)
    grads.require_shapes_of(maps)
    if not (_is_list(tapes) and len(tapes) == B):
        raise RuntimeError(f"tapes must be the list of {B} tapes hypotheses_forward_batch returned")
    Ms = {_tape_hypotheses(t, E, h, w, f"tapes[{b}]") for b, (t, h, w) in enumerate(zip(tapes, maps.hs, maps.ws))}
    if len(Ms) > 1:
        raise RuntimeError(f"the tapes hold different numbers of hypotheses {sorted(Ms)}")
    M = Ms.pop()
    if gradScores is not None:
        _check(gradScores, "Double", 2, "gradScores")
        if tuple(int(s) for s in gradScores.shape) != (B, M):
            raise RuntimeError(f"gradScores must be [{B}, {M}], got {list(gradScores.shape)}")
    if gradPoses is not None:
        _check(gradPoses, "Double", 3, "gradPoses")
        if tuple(int(s) for s in gradPoses.shape) != (B, M, 6):
            raise RuntimeError(f"gradPoses must be [{B}, {M}, 6], got {list(gradPoses.shape)}")
    gs = _Arg(gradScores) if gradScores is not None else None
    gp = _Arg(gradPoses) if gradPoses is not None else None
    ctx = _pick_ctx(*maps.devices, *grads.devices, *(t.device.index for t in tapes), gs.device if gs else None,
                    gp.device if gp else None)
    tape_ptrs = (C.c_void_p * B)(*[t.data_ptr() for t in tapes])
    ctx.check(ctx.lib.esacb200_hypotheses_backward_ragged(ctx.handle, B, tape_ptrs, maps.ptrs, grads.ptrs, maps.hs, maps.ws, E,
                                                          gs.ptr if gs else None, gp.ptr if gp else None))
    grads.finish()


def pose_loss(poses, gtPose, wLossRot, wLossTrans, lossCut):
    """The reference's loss (esac_loss.h) of scene poses float64 [M,6] = (rvec, tvec) against a float32 [4,4] camera->world
    ground truth, and its dLoss, quirks included, with esac.backward's arithmetic.  Returns torch tensors (losses float64
    [M], dloss float64 [M,6]) on the poses' device (CPU for numpy input).  A batch, poses [B,M,6] against ground truths
    [B,4,4], gives losses [B,M] and dloss [B,M,6] in one launch, row b bitwise what [M,6] against gtPose[b] gives."""
    batch = (poses.dim() if _is_torch(poses) else np.ndim(poses)) == 3
    _check(poses, "Double", 3 if batch else 2, "poses")
    _check(gtPose, "Float", 3 if batch else 2, "gtPose")
    lead = tuple(int(s) for s in poses.shape[:-2]) if batch else ()
    if int(poses.shape[-1]) != 6 or int(poses.shape[-2]) < 1 or (batch and lead[0] < 1):
        raise RuntimeError(f"poses must be {'[B, M, 6] with B, M' if batch else '[M, 6] with M'} >= 1, got {list(poses.shape)}")
    if tuple(int(s) for s in gtPose.shape) != lead + (4, 4):
        raise RuntimeError(f"gtPose must be [{lead[0]}, 4, 4] for [B, M, 6] poses" if batch else "gtPose must be [4, 4]")
    import torch
    po = _Arg(poses)
    gt = _Arg(gtPose)
    ctx = _pick_ctx(po.device, gt.device)
    B, M = (lead[0] if batch else 1), int(poses.shape[-2])
    dev = _out_device(po)
    losses = torch.empty(lead + (M,), dtype=torch.float64, device=dev)
    dloss = torch.empty(lead + (M, 6), dtype=torch.float64, device=dev)
    ctx.check(ctx.lib.esacb200_pose_loss_batch(ctx.handle, B, M, po.ptr, gt.ptr, float(wLossRot), float(wLossTrans),
                                               float(lossCut), losses.data_ptr(), dloss.data_ptr()))
    return losses, dloss


def _async_shapes(sceneCoordinates, hypAssignment, shifts, cameras, call="forward_async"):
    """Checks the dtypes and shapes of the inputs forward_async and backward_async (`call`) share (one B) before any
    context exists; returns (B, E, H, W, M).  [E,3,H,W] / [M] / [2] / [3] inputs are one image."""
    for t, what in ((sceneCoordinates, "sceneCoordinates"), (hypAssignment, "hypAssignment"), (shifts, "shifts"),
                    (cameras, "cameras")):
        if not _is_torch(t):
            raise RuntimeError(f"{call} takes torch CUDA tensors only ({what} is a {type(t).__name__})")
    single = sceneCoordinates.dim() == 4
    _check(sceneCoordinates, "Float", 4 if single else 5, "sceneCoordinates")
    _check(hypAssignment, "Long", 1 if single else 2, "hypAssignment")
    _check(shifts, "Int", 1 if single else 2, "shifts")
    _check(cameras, "Float", 1 if single else 2, "cameras")
    lead = () if single else (int(sceneCoordinates.shape[0]),)
    B = lead[0] if lead else 1
    E, three, H, W = (int(v) for v in sceneCoordinates.shape[-4:])
    if three != 3:
        raise RuntimeError("sceneCoordinates must be [B,E,3,H,W] or [E,3,H,W]")
    if B < 1 or E < 1:
        raise RuntimeError("sceneCoordinates holds no image or no expert")
    if (W - 1) * (H - 1) < 4:
        raise RuntimeError(f"sceneCoordinates: map {W}x{H} too small to draw 4 distinct cells")
    M = int(hypAssignment.shape[-1])
    if M < 1:
        raise RuntimeError("hypAssignment holds no hypothesis")
    for t, tail, what in ((hypAssignment, (M,), "hypAssignment"), (shifts, (2,), "shifts"), (cameras, (3,), "cameras")):
        if tuple(int(v) for v in t.shape) != lead + tail:
            want = ", ".join(str(v) for v in lead + tail)
            raise RuntimeError(f"{what} must be [{want}] for {B} image(s), got {list(t.shape)}")
    return B, E, H, W, M


def _async_context(call, fixed, inputs, check_inputs=None):
    """The checks every stream-ordered call (`call`) makes before it takes a context, in this order: every `fixed`
    argument (name -> (tensor, dtype, shape)) is a contiguous torch tensor of that shape; check_inputs(), if given; then
    the inputs ((name, tensor) pairs) and the fixed arguments are CUDA tensors of one device.  Returns the context, on
    torch's current stream."""
    for what, (t, dt, shape) in fixed.items():
        if not _is_torch(t):
            raise RuntimeError(f"{call} takes torch CUDA tensors only ({what} is a {type(t).__name__})")
        _check(t, dt, len(shape), what)
        if tuple(int(v) for v in t.shape) != shape or not t.is_contiguous():
            raise RuntimeError(f"{what} must be a contiguous {list(shape)} tensor, got {list(t.shape)}")
    if check_inputs is not None:
        check_inputs()
    tensors = list(inputs) + [(what, t) for what, (t, _, _) in fixed.items()]
    for what, t in tensors:
        if not t.is_cuda:
            raise RuntimeError(f"{call} takes CUDA tensors only ({what} is on the CPU)")
    devs = {t.device.index for _, t in tensors}
    if len(devs) > 1:
        raise RuntimeError(f"esac_b200: tensors live on different CUDA devices {sorted(devs)}")
    ctx = _pick_ctx(*devs)
    ctx.async_used = True
    return ctx


def _esac_inputs(inputs: dict, lead, M):
    """The stream-ordered ESAC calls' inputs (name -> tensor, hypAssignment among them if the call takes one) are
    contiguous, hypAssignment row by row.  Returns a check for _async_context and the inputs as (name, tensor) pairs."""
    def check():
        for what, t in inputs.items():
            if what != "hypAssignment" and not t.is_contiguous():
                raise RuntimeError(f"{what} must be contiguous (a copy would not be captured with the call)")
        hypAssignment = inputs.get("hypAssignment")
        if hypAssignment is not None and lead and lead[0] > 1 and hypAssignment.stride(0) != M * hypAssignment.stride(-1):
            raise RuntimeError("hypAssignment must hold its rows back to back (row stride M times the element stride)")
    return list(inputs.items()), check


def _reserve_async(call, device, sizes: dict, *rest):
    """esacb200_`call` with the sizes (name -> value, all positive) and `rest`, all as ints, on torch's current stream of
    the device's context."""
    if min(int(v) for v in sizes.values()) < 1:
        raise RuntimeError(f"{call}: sizes must be positive, got " + " ".join(f"{k}={v}" for k, v in sizes.items()))
    ctx = context(device)
    import torch
    ctx.set_stream(torch.cuda.current_stream(ctx.device).cuda_stream or _CUDA_STREAM_LEGACY)
    ctx.async_used = True
    ctx.check(getattr(ctx.lib, "esacb200_" + call)(ctx.handle, *(int(v) for v in (*sizes.values(), *rest))))


def forward_async(sceneCoordinates, hypAssignment, shifts, cameras, inlierThreshold, inlierAlpha, inlierBeta, maxReproj,
                  subSampling, outPoses, outExperts, outStatus):
    """esac.forward enqueued on torch's current stream with no host synchronisation, so it can be captured in a CUDA graph
    (torch.cuda.graph).  CUDA tensors only: sceneCoordinates float32 [B,E,3,H,W], hypAssignment int64 [B,M], shifts int32
    [B,2] (shiftX, shiftY), cameras float32 [B,3] (focal length, ppointX, ppointY); the results go to outPoses float32
    [B,4,4] (camera->world), outExperts int64 [B] and outStatus int32 [B] (0 = OK, 1 = an expert index outside [0,E): pose
    NaN, expert -1).  [E,3,H,W] / [M] / [2] / [3] / [4,4] / [] tensors are one image.  The seed, shift and camera are read
    on the device when the kernels run: a replayed graph uses what the tensors hold then, and image b of the j-th call
    after set_seed(s) draws what the (j*B + b)-th esac.forward after set_seed(s) draws.  Call reserve_forward_async with
    the largest shape before the first capture; once captured, the workspace never grows again."""
    B, E, H, W, M = _async_shapes(sceneCoordinates, hypAssignment, shifts, cameras)
    lead = (B,) if sceneCoordinates.dim() == 5 else ()
    ctx = _async_context("forward_async", {"outPoses": (outPoses, "Float", lead + (4, 4)), "outExperts": (outExperts, "Long", lead),
                                           "outStatus": (outStatus, "Int", lead)},
                         *_esac_inputs({"sceneCoordinates": sceneCoordinates, "hypAssignment": hypAssignment, "shifts": shifts,
                                        "cameras": cameras}, lead, M))
    ctx.check(ctx.lib.esacb200_forward_async(ctx.handle, B, sceneCoordinates.data_ptr(), E, H, W, hypAssignment.data_ptr(),
                                             int(hypAssignment.stride(-1)), M, shifts.data_ptr(), cameras.data_ptr(),
                                             *_thresholds(inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling),
                                             outPoses.data_ptr(), outExperts.data_ptr(), outStatus.data_ptr()))


def reserve_forward_async(B: int, E: int, H: int, W: int, M: int, subSampling: int = 8, device: int | None = None):
    """Sizes forward_async's workspace for this shape; call it before capturing (it allocates)."""
    _reserve_async("reserve_forward_async", device, dict(B=B, E=E, H=H, W=W, M=M), subSampling)


def backward_async(sceneCoordinates, outGradients, hypAssignment, gtPoses, shifts, cameras, wLossRot, wLossTrans, lossCut,
                   inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling, outLosses, outStatus):
    """esac.backward enqueued on torch's current stream with no host synchronisation, so a training step can be captured
    in a CUDA graph (torch.cuda.graph).  CUDA tensors only: sceneCoordinates float32 [B,E,3,H,W], outGradients float32
    [B,E,3,H,W] (accumulated, +=, as esac.backward), hypAssignment int64 [B,M], gtPoses float32 [B,4,4] (camera->world),
    shifts int32 [B,2], cameras float32 [B,3] (focal length, ppointX, ppointY); the results go to outLosses float64 [B]
    (what esac.backward returns) and outStatus int32 [B] (0 = OK, 1 = an expert index outside [0,E): loss NaN, gradient
    slice untouched).  [E,3,H,W] / [M] / [4,4] / [2] / [3] / [] tensors are one image.  The seed, ground truth, shift and
    camera are read on the device when the kernels run.  forward_async and backward_async share one call counter: image b
    of the j-th call after set_seed(s) draws what the (j*B + b)-th esac.forward / esac.backward after set_seed(s) draws,
    and the results are bitwise esac.backward's.  Call reserve_backward_async with the largest shape before the first
    capture; once captured, the workspace never grows again."""
    B, E, H, W, M = _async_shapes(sceneCoordinates, hypAssignment, shifts, cameras, "backward_async")
    lead = (B,) if sceneCoordinates.dim() == 5 else ()
    ctx = _async_context("backward_async", {"outGradients": (outGradients, "Float", lead + (E, 3, H, W)),
                                            "gtPoses": (gtPoses, "Float", lead + (4, 4)), "outLosses": (outLosses, "Double", lead),
                                            "outStatus": (outStatus, "Int", lead)},
                         *_esac_inputs({"sceneCoordinates": sceneCoordinates, "hypAssignment": hypAssignment, "shifts": shifts,
                                        "cameras": cameras}, lead, M))
    ctx.check(ctx.lib.esacb200_backward_async(ctx.handle, B, sceneCoordinates.data_ptr(), outGradients.data_ptr(), E, H, W,
                                              hypAssignment.data_ptr(), int(hypAssignment.stride(-1)), M, gtPoses.data_ptr(),
                                              float(wLossRot), float(wLossTrans), float(lossCut), shifts.data_ptr(),
                                              cameras.data_ptr(),
                                              *_thresholds(inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling),
                                              outLosses.data_ptr(), outStatus.data_ptr()))


def reserve_backward_async(B: int, E: int, H: int, W: int, M: int, subSampling: int = 8, device: int | None = None):
    """Sizes backward_async's workspace (which forward_async shares) for this shape; call it before capturing (it
    allocates)."""
    _reserve_async("reserve_backward_async", device, dict(B=B, E=E, H=H, W=W, M=M), subSampling)


def hypotheses_tape_stride(E: int, H: int, W: int, M: int) -> int:
    """Bytes between consecutive images' tapes in hypotheses_forward_async: hypotheses_tape_bytes rounded up to 256."""
    return (hypotheses_tape_bytes(E, H, W, M) + 255) // 256 * 256


def _check_tapes(tapes, B, E, H, W, M, call):
    if not (_is_torch(tapes) and str(tapes.dtype) == "torch.uint8" and tapes.dim() == 1 and tapes.is_contiguous()):
        raise RuntimeError(f"{call}: tapes must be a contiguous 1-D uint8 torch tensor")
    need = B * hypotheses_tape_stride(E, H, W, M)
    if int(tapes.numel()) < need:
        raise RuntimeError(f"{call}: tapes hold {int(tapes.numel())} bytes, {B} image(s) of [{E}, 3, {H}, {W}] maps with "
                           f"M={M} need {need} (B * hypotheses_tape_stride)")


def hypotheses_forward_async(sceneCoordinates, hypAssignment, shifts, cameras, inlierThreshold, inlierAlpha, inlierBeta,
                             maxReproj, subSampling, tapes, outScores, outPoses, outContributing, outStatus, minProb=PROB_THRESH):
    """hypotheses_forward enqueued on torch's current stream with no host synchronisation, so that a training step with
    a pose loss of the caller's own can be captured in a CUDA graph.  CUDA tensors only: sceneCoordinates float32
    [B,E,3,H,W], hypAssignment int64 [B,M], shifts int32 [B,2], cameras float32 [B,3] (focal length, ppointX, ppointY),
    read on the device when the kernels run; tapes a uint8 tensor of at least B * hypotheses_tape_stride(E,H,W,M) bytes
    (image b's tape at b * stride).  Row b of outScores float64 [B,M], outPoses float64 [B,M,6] and outContributing bool
    [B,M] is what hypotheses_forward returns for the same draws; outStatus int32 [B]: 0 = OK, 1 = an expert index outside
    [0,E) (scores and poses NaN, nothing contributes).  [E,3,H,W] / [M] / [2] / [3] / [M,6] / [] tensors are one image.
    Seeding is forward_async's: image b of the j-th call after set_seed(s) draws what the (j*B + b)-th esac.backward or
    hypotheses_forward after set_seed(s) draws.  The workspace is backward_async's: call reserve_backward_async with the
    largest shape before the first capture.  minProb: hypotheses_forward's; a captured graph keeps the floor it was
    captured with (a training hyperparameter, not per-image data)."""
    call = "hypotheses_forward_async"
    minProb = _min_prob(minProb, call)
    B, E, H, W, M = _async_shapes(sceneCoordinates, hypAssignment, shifts, cameras, call)
    lead = (B,) if sceneCoordinates.dim() == 5 else ()
    if not _is_torch(tapes):
        raise RuntimeError(f"{call} takes torch CUDA tensors only (tapes is a {type(tapes).__name__})")
    _check_tapes(tapes, B, E, H, W, M, call)
    ctx = _async_context(call, {"outScores": (outScores, "Double", lead + (M,)), "outPoses": (outPoses, "Double", lead + (M, 6)),
                                "outContributing": (outContributing, "Bool", lead + (M,)), "outStatus": (outStatus, "Int", lead)},
                         *_esac_inputs({"sceneCoordinates": sceneCoordinates, "hypAssignment": hypAssignment, "shifts": shifts,
                                        "cameras": cameras, "tapes": tapes}, lead, M))
    fn, floor = _floor_entry(ctx.lib, "hypotheses_forward_async", minProb)
    ctx.check(fn(
        ctx.handle, B, sceneCoordinates.data_ptr(), E, H, W, hypAssignment.data_ptr(), int(hypAssignment.stride(-1)), M,
        shifts.data_ptr(), cameras.data_ptr(), *_thresholds(inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling),
        *floor, tapes.data_ptr(), int(tapes.numel()), outScores.data_ptr(), outPoses.data_ptr(), outContributing.data_ptr(),
        outStatus.data_ptr()))


def hypotheses_backward_async(tapes, sceneCoordinates, outGradients, M, gradScores=None, gradPoses=None, outStatus=None):
    """hypotheses_backward enqueued on torch's current stream with no host synchronisation: accumulates (+=) into
    outGradients float32 [B,E,3,H,W] what hypotheses_backward on image b's tape (written by hypotheses_forward_async with
    M hypotheses) with gradScores[b] float64 [B,M] / gradPoses[b] float64 [B,M,6] adds; None counts as zero.  CUDA
    tensors only; [E,3,H,W] / [M] / [M,6] / [] tensors are one image.  outStatus int32 [B] (or None): 0 = OK, 1 = the
    forward's assignment held a bad expert index, 2 = the tape holds no forward of this shape; the gradient slice of a
    non-zero status is left untouched.  Draws nothing and leaves the call counter alone."""
    call = "hypotheses_backward_async"
    for t, what in ((tapes, "tapes"), (sceneCoordinates, "sceneCoordinates"), (outGradients, "outGradients")):
        if not _is_torch(t):
            raise RuntimeError(f"{call} takes torch CUDA tensors only ({what} is a {type(t).__name__})")
    single = sceneCoordinates.dim() == 4
    _check(sceneCoordinates, "Float", 4 if single else 5, "sceneCoordinates")
    lead = () if single else (int(sceneCoordinates.shape[0]),)
    B = lead[0] if lead else 1
    E, three, H, W = (int(v) for v in sceneCoordinates.shape[-4:])
    M = int(M)
    if three != 3 or B < 1 or E < 1 or M < 1:
        raise RuntimeError(f"{call}: sceneCoordinates must be [B,E,3,H,W] or [E,3,H,W] and M >= 1")
    fixed = {"outGradients": (outGradients, "Float", lead + (E, 3, H, W))}
    if gradScores is not None:
        fixed["gradScores"] = (gradScores, "Double", lead + (M,))
    if gradPoses is not None:
        fixed["gradPoses"] = (gradPoses, "Double", lead + (M, 6))
    if outStatus is not None:
        fixed["outStatus"] = (outStatus, "Int", lead)
    _check_tapes(tapes, B, E, H, W, M, call)
    ctx = _async_context(call, fixed, *_esac_inputs({"sceneCoordinates": sceneCoordinates, "tapes": tapes}, lead, M))
    if outStatus is None:
        import torch
        outStatus = torch.empty(lead, dtype=torch.int32, device=sceneCoordinates.device)
    ctx.check(ctx.lib.esacb200_hypotheses_backward_async(
        ctx.handle, B, tapes.data_ptr(), int(tapes.numel()), sceneCoordinates.data_ptr(), outGradients.data_ptr(), E, H, W, M,
        gradScores.data_ptr() if gradScores is not None else None, gradPoses.data_ptr() if gradPoses is not None else None,
        outStatus.data_ptr()))
    return outStatus


def pose_loss_async(poses, gtPose, wLossRot, wLossTrans, lossCut, outLosses=None, outDloss=None):
    """pose_loss launched on torch's current stream on the caller's CUDA tensors, with no staging copy and no host
    synchronisation: poses float64 [B,M,6] (or [M,6]) against gtPose float32 [B,4,4] (or [4,4]).  Returns (losses [B,M],
    dloss [B,M,6]), written into outLosses / outDloss when given; row b is bitwise what pose_loss gives."""
    call = "pose_loss_async"
    for t, what in ((poses, "poses"), (gtPose, "gtPose")):
        if not _is_torch(t):
            raise RuntimeError(f"{call} takes torch CUDA tensors only ({what} is a {type(t).__name__})")
    batch = poses.dim() == 3
    _check(poses, "Double", 3 if batch else 2, "poses")
    lead = (int(poses.shape[0]),) if batch else ()
    M = int(poses.shape[-2])
    if int(poses.shape[-1]) != 6 or M < 1 or (batch and lead[0] < 1):
        raise RuntimeError(f"poses must be {'[B, M, 6]' if batch else '[M, 6]'} with M >= 1, got {list(poses.shape)}")
    import torch
    if outLosses is None:
        outLosses = torch.empty(lead + (M,), dtype=torch.float64, device=poses.device)
    if outDloss is None:
        outDloss = torch.empty(lead + (M, 6), dtype=torch.float64, device=poses.device)
    ctx = _async_context(call, {"gtPose": (gtPose, "Float", lead + (4, 4)), "outLosses": (outLosses, "Double", lead + (M,)),
                                "outDloss": (outDloss, "Double", lead + (M, 6))},
                         *_esac_inputs({"poses": poses}, lead, M))
    B = lead[0] if lead else 1
    ctx.check(ctx.lib.esacb200_pose_loss_async(ctx.handle, B, M, poses.data_ptr(), gtPose.data_ptr(), float(wLossRot),
                                               float(wLossTrans), float(lossCut), outLosses.data_ptr(), outDloss.data_ptr()))
    return outLosses, outDloss


def _loss_images(t, what: str, call: str, writable: bool = False, like: _Images | None = None,
                 dtypes: str | tuple = "Float") -> _Images:
    """An image argument of the stream-ordered losses: torch tensors only, each contiguous (a copy would not be captured
    with the call); then _Images' dtype (dtypes), rank and shape checks.  Raises before any context exists."""
    parts = list(enumerate(t)) if _is_list(t) else [(None, t)]
    for b, x in parts:
        name = what if b is None else f"{what}[{b}]"
        if not _is_torch(x):
            raise RuntimeError(f"{call} takes torch CUDA tensors only ({name} is a {type(x).__name__})")
    im = _Images(t, 3, what, writable=writable, like=like, dtypes=dtypes)
    for b, x in parts:
        if not x.is_contiguous():
            name = what if b is None else f"{what}[{b}]"
            raise RuntimeError(f"{name} must be contiguous (a copy would not be captured with the call)")
    return im


def _image_tensors(images):
    """The (name, tensor) pairs of the stream-ordered losses' image arguments (_loss_images)."""
    return [(im.what, a.orig) for im in images for a in im.args]


def _reproj_loss_async(call, prediction, gtPoses, shifts, cameras, cutLoss, subSampling, outLosses, outStatus, outGradients,
                       maxReproj, minDepth, gradScale):
    """reproj_loss_async (call "reproj_loss_async": float32 maps) or reproj_loss_amp_async (float16 / bfloat16 maps)."""
    amp = call == "reproj_loss_amp_async"
    pr = _loss_images(prediction, "prediction", call, dtypes=_AMP if amp else "Float")
    B = pr.B
    og = None
    if outGradients is not None:
        og = _loss_images(outGradients, "outGradients", call, writable=True, like=pr, dtypes=pr.dtype)
        og.require_shapes_of(pr)
    scale = _grad_scale(gradScale, call) if amp else []
    ctx = _async_context(call, {"gtPoses": (gtPoses, "Float", (B, 4, 4)), "shifts": (shifts, "Int", (B, 2)),
                                "cameras": (cameras, "Float", (B, 3)), "outLosses": (outLosses, "Double", (B,)),
                                "outStatus": (outStatus, "Int", (B,))},
                         _image_tensors([pr] + ([og] if og else [])) + scale)
    args = (pr.ptrs, og.ptrs if og else None, pr.hs, pr.ws, gtPoses.data_ptr(), shifts.data_ptr(), cameras.data_ptr(),
            int(subSampling), float(cutLoss), float(maxReproj), float(minDepth))
    outs = (outLosses.data_ptr(), outStatus.data_ptr())
    if amp:
        ctx.check(ctx.lib.esacb200_reproj_loss_async_typed(ctx.handle, B, _LOSS_DTYPES[pr.dtype], *args,
                                                           gradScale.data_ptr() if scale else None, *outs))
    else:
        ctx.check(ctx.lib.esacb200_reproj_loss_async(ctx.handle, B, *args, *outs))


def reproj_loss_async(prediction, gtPoses, shifts, cameras, cutLoss, subSampling, outLosses, outStatus, outGradients=None,
                      maxReproj=100.0, minDepth=0.1):
    """reproj_loss enqueued on torch's current stream with no host synchronisation, so that a ref_expert.py step can be
    captured in a CUDA graph.  CUDA tensors only: prediction float32 [B,3,H,W] or a list / tuple of B [3,H_b,W_b] tensors,
    gtPoses float32 [B,4,4] camera->world, shifts int32 [B,2] (padX, padY), cameras float32 [B,3] (focal length, ppointX,
    ppointY), all read on the device when the kernels run (the image pointers and sizes are fixed by a capture).
    outGradients (the prediction's form and shapes, overwritten) or None; outLosses float64 [B] and outStatus int32 [B]
    receive, bitwise, reproj_loss's losses and 0, or for an image whose ground-truth rotation is singular or NaN (where
    reproj_loss raises) a NaN loss, a zero gradient and status 1.  Call reserve_loss_async with the largest batch and map
    before the first capture."""
    _reproj_loss_async("reproj_loss_async", prediction, gtPoses, shifts, cameras, cutLoss, subSampling, outLosses, outStatus,
                       outGradients, maxReproj, minDepth, None)


def reproj_loss_amp_async(prediction, gtPoses, shifts, cameras, cutLoss, subSampling, outLosses, outStatus, outGradients=None,
                          maxReproj=100.0, minDepth=0.1, gradScale=None):
    """reproj_loss_async on a float16 or bfloat16 prediction (a list: of one dtype), with reproj_loss_amp's results:
    outGradients of the prediction's dtype receive the float32 gradients times gradScale, rounded (a bad image's gradient:
    a rounded 0 * gradScale).  gradScale (a CUDA float32 tensor of one element, or None = 1) is read on the device when the
    kernels run, so a captured call replays with the scale of the moment."""
    _reproj_loss_async("reproj_loss_amp_async", prediction, gtPoses, shifts, cameras, cutLoss, subSampling, outLosses,
                       outStatus, outGradients, maxReproj, minDepth, gradScale)


def _coord_loss_async(call, prediction, gtCoords, cutLoss, outLosses, outGradients, outCounts, gradScale):
    """coord_loss_async (call "coord_loss_async": float32 maps) or coord_loss_amp_async (float16 / bfloat16 maps)."""
    amp = call == "coord_loss_amp_async"
    pr = _loss_images(prediction, "prediction", call, dtypes=_AMP if amp else "Float")
    gt = _loss_images(gtCoords, "gtCoords", call, like=pr)
    for b, ((_, hp, wp), (_, hg, wg)) in enumerate(zip(pr.shapes, gt.shapes)):
        if abs(hp - hg) > 1 or abs(wp - wg) > 1:
            raise RuntimeError(f"image {b}: tensor size mismatch: prediction {hp}x{wp}, ground truth {hg}x{wg} "
                               "(util.assert_size allows 1)")
    og = None
    if outGradients is not None:
        og = _loss_images(outGradients, "outGradients", call, writable=True, like=pr, dtypes=pr.dtype)
        og.require_shapes_of(pr)
    scale = _grad_scale(gradScale, call) if amp else []
    fixed = {"outLosses": (outLosses, "Double", (pr.B,))}
    if outCounts is not None:
        fixed["outCounts"] = (outCounts, "Long", (pr.B,))
    ctx = _async_context(call, fixed, _image_tensors([pr, gt] + ([og] if og else [])) + scale)
    args = (pr.ptrs, pr.hs, pr.ws, gt.ptrs, gt.hs, gt.ws, og.ptrs if og else None, float(cutLoss))
    outs = (outLosses.data_ptr(), outCounts.data_ptr() if outCounts is not None else None)
    if amp:
        ctx.check(ctx.lib.esacb200_coord_loss_async_typed(ctx.handle, pr.B, _LOSS_DTYPES[pr.dtype], *args,
                                                          gradScale.data_ptr() if scale else None, *outs))
    else:
        ctx.check(ctx.lib.esacb200_coord_loss_async(ctx.handle, pr.B, *args, *outs))


def coord_loss_async(prediction, gtCoords, cutLoss, outLosses, outGradients=None, outCounts=None):
    """coord_loss enqueued on torch's current stream with no host synchronisation, so that an init_expert.py step can be
    captured in a CUDA graph.  CUDA tensors only: prediction float32 [B,3,Hp,Wp] and gtCoords float32 [B,3,Hg,Wg] (at most
    1 apart in H and W), or both lists / tuples of B [3,H_b,W_b] tensors; outGradients (the prediction's form and shapes,
    overwritten) or None.  outLosses float64 [B] and outCounts int64 [B] (or None) receive, bitwise, coord_loss's losses
    and valid-cell counts.  The maps are read on the device when the kernels run (their pointers and sizes are fixed by a
    capture).  Call reserve_loss_async with the largest batch and map before the first capture."""
    _coord_loss_async("coord_loss_async", prediction, gtCoords, cutLoss, outLosses, outGradients, outCounts, None)


def coord_loss_amp_async(prediction, gtCoords, cutLoss, outLosses, outGradients=None, outCounts=None, gradScale=None):
    """coord_loss_async on a float16 or bfloat16 prediction (a list: of one dtype) and a float32 gtCoords, with
    coord_loss_amp's results; gradScale as for reproj_loss_amp_async."""
    _coord_loss_async("coord_loss_amp_async", prediction, gtCoords, cutLoss, outLosses, outGradients, outCounts, gradScale)


def reserve_loss_async(B: int, H: int, W: int, device: int | None = None):
    """Sizes the workspace of reproj_loss_async and coord_loss_async (and of their _amp forms, which use the same) for B
    images of at most H x W cells (the prediction's); call it before capturing (it allocates)."""
    _reserve_async("reserve_loss_async", device, dict(B=B, H=H, W=W))


# The columns of a pose evaluation's record (include/esac_b200.h, esacb200_eval_poses): float64, one row per image.
EVAL_FIELDS = ("rot_deg", "trans_cm", "correct", "scene", "expert", "status", "active", "qw", "qx", "qy", "qz", "tx", "ty", "tz")
EVAL_STATE = 4  # int64 words of a record store's device state: rows handed out, overflow flag, launch ticket, unused


def _eval_context(call, outPoses, gtPoses, experts, gtScenes, hist, status, outRecords, state):
    """The checks of evaluate_poses / evaluate_poses_async before any context exists; returns (ctx, B, E, capacity)."""
    for what, t in (("outPoses", outPoses), ("outRecords", outRecords)):
        if not _is_torch(t):
            raise RuntimeError(f"{call} takes torch CUDA tensors only ({what} is a {type(t).__name__})")
    _check(outPoses, "Float", 3 if outPoses.dim() == 3 else 2, "outPoses")
    lead = tuple(int(v) for v in outPoses.shape[:-2])
    if tuple(int(v) for v in outPoses.shape[-2:]) != (4, 4) or (lead and lead[0] < 1):
        raise RuntimeError(f"outPoses must be [B,4,4] or [4,4], got {list(outPoses.shape)}")
    B = lead[0] if lead else 1
    _check(outRecords, "Double", 2, "outRecords")
    capacity = int(outRecords.shape[0])
    if capacity < 1:
        raise RuntimeError("outRecords holds no row")
    fixed = {"outPoses": (outPoses, "Float", lead + (4, 4)), "gtPoses": (gtPoses, "Float", lead + (4, 4)),
             "experts": (experts, "Long", lead), "gtScenes": (gtScenes, "Long", lead),
             "outRecords": (outRecords, "Double", (capacity, len(EVAL_FIELDS))), "state": (state, "Long", (EVAL_STATE,))}
    E = 0
    if hist is not None:
        if not _is_torch(hist) or hist.dim() != len(lead) + 1:
            raise RuntimeError(f"hist must be a float32 tensor [B,E] or [E], got "
                               f"{list(hist.shape) if _is_torch(hist) else type(hist).__name__}")
        E = int(hist.shape[-1])
        if not 1 <= E <= MAX_EXPERTS:
            raise RuntimeError(f"{call}: hist holds E={E} experts, outside [1, {MAX_EXPERTS}]")
        fixed["hist"] = (hist, "Float", lead + (E,))
    if status is not None:
        fixed["status"] = (status, "Int", lead)
    return _async_context(call, fixed, []), B, E, capacity


def _eval_call(name, ctx, B, E, capacity, outPoses, gtPoses, experts, gtScenes, hist, status, outRecords, state):
    ctx.check(getattr(ctx.lib, name)(ctx.handle, B, outPoses.data_ptr(), gtPoses.data_ptr(), experts.data_ptr(),
                                     gtScenes.data_ptr(), hist.data_ptr() if hist is not None else None, E,
                                     status.data_ptr() if status is not None else None, outRecords.data_ptr(), capacity,
                                     state.data_ptr()))


def evaluate_poses_async(outPoses, gtPoses, experts, gtScenes, outRecords, state, hist=None, status=None):
    """test_esac.py's per-image evaluation (pose errors, correct expert, experts active, pose-file entry) enqueued on torch's
    current stream with no host synchronisation, so that a CUDA graph can capture it.  CUDA tensors only, contiguous:
    outPoses / gtPoses float32 [B,4,4] (or [4,4]) camera->world, experts / gtScenes int64 [B] (or []), hist float32 [B,E]
    (or [E]; assign_hypotheses_async's histogram) or None, status int32 [B] (or []; forward_async's) or None.  Image b's
    record (EVAL_FIELDS, float64) goes to row state[0] + b of outRecords float64 [capacity, 14]; state int64 [4] is the
    store's device state (zero it to start; state[1] becomes 1 when a row falls past capacity, and that row is dropped)."""
    ctx, B, E, capacity = _eval_context("evaluate_poses_async", outPoses, gtPoses, experts, gtScenes, hist, status,
                                        outRecords, state)
    _eval_call("esacb200_eval_poses_async", ctx, B, E, capacity, outPoses, gtPoses, experts, gtScenes, hist, status,
               outRecords, state)


def evaluate_poses(outPoses, gtPoses, experts, gtScenes, hist=None, status=None):
    """evaluate_poses_async into a fresh store, synchronised: returns the records, float64 [B,14] (EVAL_FIELDS) for a batch
    or [14] for one [4,4] pose, on the poses' device."""
    call = "evaluate_poses"
    if not _is_torch(outPoses):
        raise RuntimeError(f"{call} takes torch CUDA tensors only (outPoses is a {type(outPoses).__name__})")
    import torch
    B = int(outPoses.shape[0]) if outPoses.dim() == 3 else 1
    dev = outPoses.device
    records = torch.empty((max(B, 1), len(EVAL_FIELDS)), dtype=torch.float64, device=dev)
    state = torch.zeros(EVAL_STATE, dtype=torch.int64, device=dev)
    ctx, B, E, capacity = _eval_context(call, outPoses, gtPoses, experts, gtScenes, hist, status, records, state)
    _eval_call("esacb200_eval_poses", ctx, B, E, capacity, outPoses, gtPoses, experts, gtScenes, hist, status, records, state)
    return records if outPoses.dim() == 3 else records[0]


# ------------------------------------------------------------------------------------------------
# clustering a large environment into experts (cluster_dataset.py:19-140, 219-240; esac_b200/cluster.py drives these)
# ------------------------------------------------------------------------------------------------
MAX_CLUSTERS = 1024  # clusters one cluster_targets call handles (include/esac_b200.h)


def cluster_statistics(init_maps):
    """Per-image statistics of ground-truth scene-coordinate maps (cluster_dataset.py:52-58, 121-124): init_maps is one
    stacked float32 tensor [B,3,H,W] or a list / tuple of B float32 tensors [3,H_b,W_b] (all CPU / numpy or all CUDA).  A
    cell is valid when the float32 sum (x + y) + z is not 0.  Returns (median float32 [B,3]: torch.median(1)[0] over the
    valid cells, bitwise; mean float32 [B,3]: their fp64 mean rounded once; count int32 [B]: valid cells; status int32
    [B]: 0 ok, 1 no valid cell, 2 a non-finite median or mean), on the maps' device (CPU for host maps)."""
    import torch
    maps = _Images(init_maps, 3, "init_maps")
    ctx = _pick_ctx(*maps.devices)
    dev = torch.device("cuda", maps.devices[0]) if maps.devices[0] is not None else torch.device("cpu")
    median = torch.empty((maps.B, 3), dtype=torch.float32, device=dev)
    mean = torch.empty((maps.B, 3), dtype=torch.float32, device=dev)
    count = torch.empty(maps.B, dtype=torch.int32, device=dev)
    status = torch.empty(maps.B, dtype=torch.int32, device=dev)
    ctx.check(ctx.lib.esacb200_cluster_stats_ragged(ctx.handle, maps.B, maps.ptrs, maps.hs, maps.ws, median.data_ptr(),
                                                    mean.data_ptr(), count.data_ptr(), status.data_ptr()))
    return median, mean, count, status


def _cuda_only(call: str, **tensors):
    """The last check of a CUDA-only call: every tensor lives on the GPU (after the dtype and shape checks, so that those
    run without one)."""
    for what, t in tensors.items():
        if not t.is_cuda:
            raise RuntimeError(f"{call} takes CUDA tensors only ({what} is on the CPU)")


def kmeans2(points, seed: int, attempts: int = 10, max_iter: int = 100, eps: float = 0.1, split: int = 0):
    """One 2-means split, the replacement of cv2.kmeans(points, 2, None, (EPS + MAX_ITER, max_iter, eps), attempts,
    KMEANS_PP_CENTERS) (cluster_dataset.py:65-86) with the repository's own random stream: points a CUDA float32 tensor
    [n,3] (n >= 2); the draws of attempt a are keyed by (seed, split, a), so the splits of one clustering take distinct
    `split` values.  Stops after max_iter iterations or once no centre moves more than eps (OpenCV squares eps too).
    Returns (labels int32 [n] of 0 / 1, centres float32 [2,3], compactness float) of the attempt with the lowest
    compactness; bitwise repeatable.  The numbering of the two clusters is this implementation's, not cv2's."""
    call = "kmeans2"
    if not _is_torch(points):
        raise RuntimeError(f"{call} takes torch CUDA tensors only (points is a {type(points).__name__})")
    _check(points, "Float", 2, "points")
    if int(points.shape[1]) != 3 or not points.is_contiguous():
        raise RuntimeError(f"{call}: points must be a contiguous [n,3], got {list(points.shape)}")
    n = int(points.shape[0])
    if n < 2:
        raise RuntimeError(f"{call}: {n} points, need at least 2")
    if not 1 <= int(attempts) <= 4096:
        raise RuntimeError(f"{call}: attempts={attempts} outside [1, 4096]")
    if int(max_iter) < 1:
        raise RuntimeError(f"{call}: max_iter={max_iter}, need at least 1")
    if not float(eps) >= 0:
        raise RuntimeError(f"{call}: eps={eps}, need eps >= 0")
    if int(split) < 0:
        raise RuntimeError(f"{call}: split={split} must not be negative")
    _cuda_only(call, points=points)
    import torch
    ctx = _pick_ctx(points.device.index)
    labels = torch.empty(n, dtype=torch.int32, device=points.device)
    centres = torch.empty((2, 3), dtype=torch.float32, device=points.device)
    compactness = torch.empty(1, dtype=torch.float64, device=points.device)
    ctx.check(ctx.lib.esacb200_kmeans2(ctx.handle, n, points.data_ptr(), int(seed) & (2**64 - 1), int(split), int(attempts),
                                       int(max_iter), float(eps), labels.data_ptr(), centres.data_ptr(),
                                       compactness.data_ptr()))
    return labels, centres, float(compactness.item())


def cluster_targets(means, labels, K: int, softness: float = 5.0):
    """The cluster centres, sizes and soft gating targets of a clustering (cluster_dataset.py:104-134, 219-240): means a
    CUDA float32 tensor [N,3] (the images' mean scene coordinates), labels a CUDA int64 tensor [N] with every label in
    [0, K) and every cluster non-empty.  Returns (cam_centers float32 [K,3]: the mean of each cluster's image means,
    cam_sizes float32 [K,1]: their mean squared distance to the centre, gating_probs float32 [N,K]:
    exp(-d^2 / size / 2 * softness) / sqrt(2 pi size) normalised by its sum + 1e-7, in the reference's float32 op order)."""
    call = "cluster_targets"
    for what, t in (("means", means), ("labels", labels)):
        if not _is_torch(t):
            raise RuntimeError(f"{call} takes torch CUDA tensors only ({what} is a {type(t).__name__})")
    _check(means, "Float", 2, "means")
    _check(labels, "Long", 1, "labels")
    N = int(means.shape[0])
    if N < 1 or int(means.shape[1]) != 3 or not means.is_contiguous():
        raise RuntimeError(f"{call}: means must be a contiguous [N,3] with N >= 1, got {list(means.shape)}")
    if int(labels.shape[0]) != N or not labels.is_contiguous():
        raise RuntimeError(f"{call}: labels must be a contiguous [{N}], got {list(labels.shape)}")
    K = int(K)
    if not 1 <= K <= MAX_CLUSTERS:
        raise RuntimeError(f"{call}: K={K} outside [1, {MAX_CLUSTERS}]")
    if not float(softness) > 0:
        raise RuntimeError(f"{call}: softness={softness}, need softness > 0")
    import torch
    if means.device != labels.device:
        raise RuntimeError(f"{call}: means and labels live on different devices ({means.device}, {labels.device})")
    lab = labels.cpu().numpy()
    outside = np.flatnonzero((lab < 0) | (lab >= K))
    if len(outside):
        raise RuntimeError(f"{call}: label {int(lab[outside[0]])} of image {int(outside[0])} outside [0, {K})")
    empty = np.flatnonzero(np.bincount(lab, minlength=K) == 0)
    if len(empty):
        raise RuntimeError(f"{call}: cluster {int(empty[0])} has no image")
    _cuda_only(call, means=means, labels=labels)
    ctx = _pick_ctx(means.device.index)
    centres = torch.empty((K, 3), dtype=torch.float32, device=means.device)
    sizes = torch.empty((K, 1), dtype=torch.float32, device=means.device)
    probs = torch.empty((N, K), dtype=torch.float32, device=means.device)
    ctx.check(ctx.lib.esacb200_cluster_targets(ctx.handle, N, means.data_ptr(), labels.data_ptr(), K, float(softness),
                                               centres.data_ptr(), sizes.data_ptr(), probs.data_ptr()))
    return centres, sizes, probs


# ------------------------------------------------------------------------------------------------
# ground-truth maps from an SfM reconstruction (setup_aachen.py:184-202, setup_dubrovnik.py:171-190; esac_b200/prepare.py
# reads the reconstructions and writes the files)
# ------------------------------------------------------------------------------------------------
RENDER_MAX_SIDE = 8192           # out map side (include/esac_b200.h: ESACB200_RENDER_MAX_SIDE)
RENDER_MAX_CELLS = 1 << 30       # cells of all maps of one call
RENDER_MAX_OBS = 2**31 - 256     # observations, and points, of one call
RENDER_STATUS = {1: "a point index out of range", 2: "a NaN projection"}


def _host_values(t) -> np.ndarray:
    if _is_torch(t):
        t = t.detach().cpu().numpy()
    return np.asarray(t)


def render_init_maps(points, offsets, indices, poses, focal, out_scale, out_shapes, zbuffer: bool = False):
    """Renders the ground-truth scene-coordinate maps of C cameras from an SfM reconstruction, as the z-buffer loop of
    setup_aachen.py / setup_dubrovnik.py does, on the GPU.

    points float32 [P,3]; offsets integer [C+1] (0, non-decreasing, ending at V): camera c's observations are
    indices[offsets[c]:offsets[c+1]], int32 point indices in reconstruction file order; poses float32 [C,4,4] or [C,3,4]
    (world -> camera; only rows 0-2 are used); focal and out_scale (out width / image width) C numbers, rounded to float32;
    out_shapes C pairs (h, w), each side in [1, RENDER_MAX_SIDE].  points and indices may be host (numpy / CPU torch) or
    CUDA tensors; the other arguments are read on the host.

    Each projection runs in float32 in one stated order (include/esac_b200.h); off-image points and points behind the
    camera are clamped onto the border and take part in the z-test, as in the reference.  Returns (maps: C float32 views
    [3,h,w] of one CUDA buffer, counts: int32 CPU tensor [C] of the cells written, zbufs: C float32 views [h,w] or None
    unless zbuffer).  Raises RuntimeError naming the cameras with an observation whose point index is out of range or
    whose projection is NaN (cam.z = 0 with cam.x or cam.y = 0: the reference's int(nan)).  Argument errors raise before
    any context exists."""
    call = "render_init_maps"
    _check(points, "Float", 2, "points")
    if int(points.shape[1]) != 3:
        raise RuntimeError(f"{call}: points must be [P,3], got {list(points.shape)}")
    _check(indices, "Int", 1, "indices")
    _check(poses, "Float", 3, "poses")
    offs = _host_values(offsets)
    if offs.ndim != 1 or not np.issubdtype(offs.dtype, np.integer):
        raise RuntimeError(f"{call}: offsets must be a 1-d integer array, got {offs.dtype} of shape {list(offs.shape)}")
    C = int(offs.shape[0]) - 1
    if C < 1:
        raise RuntimeError(f"{call}: {C} cameras, need at least 1 (offsets holds C+1 values)")
    offs = offs.astype(np.int64)
    P, V = int(points.shape[0]), int(indices.shape[0])
    if offs[0] != 0:
        raise RuntimeError(f"{call}: offsets[0]={int(offs[0])}, need 0")
    dec = np.flatnonzero(np.diff(offs) < 0)
    if len(dec):
        raise RuntimeError(f"{call}: offsets decrease at camera {int(dec[0])}")
    if int(offs[-1]) != V:
        raise RuntimeError(f"{call}: offsets end at {int(offs[-1])}, but indices holds {V} observations")
    if V > RENDER_MAX_OBS or P > RENDER_MAX_OBS:
        raise RuntimeError(f"{call}: {V} observations and {P} points, at most {RENDER_MAX_OBS} each")
    if tuple(int(v) for v in poses.shape[1:]) not in ((4, 4), (3, 4)) or int(poses.shape[0]) != C:
        raise RuntimeError(f"{call}: poses must be [{C},4,4] or [{C},3,4], got {list(poses.shape)}")
    f = _per_image(focal, C, np.float32, "focal")
    s = _per_image(out_scale, C, np.float32, "out_scale")
    shp = _host_values(out_shapes)
    if shp.shape != (C, 2) or not np.issubdtype(shp.dtype, np.integer):
        raise RuntimeError(f"{call}: out_shapes must be {C} integer pairs (h, w), got {shp.dtype} of shape {list(shp.shape)}")
    shp = shp.astype(np.int64)
    off_side = np.flatnonzero((shp < 1).any(1) | (shp > RENDER_MAX_SIDE).any(1))
    if len(off_side):
        c = int(off_side[0])
        raise RuntimeError(f"{call}: camera {c} map is {int(shp[c, 0])}x{int(shp[c, 1])}, need sides in [1, {RENDER_MAX_SIDE}]")
    cells = shp[:, 0] * shp[:, 1]
    if int(cells.sum()) > RENDER_MAX_CELLS:
        raise RuntimeError(f"{call}: the maps hold {int(cells.sum())} cells, more than {RENDER_MAX_CELLS}")
    devs = {t.device.index for t in (points, indices) if _is_torch(t) and t.is_cuda}
    if len(devs) > 1:
        raise RuntimeError(f"{call}: points and indices live on different CUDA devices {sorted(devs)}")
    pose34 = np.ascontiguousarray(_host_values(poses)[:, :3, :], np.float32)
    pts, idx = _Arg(points), _Arg(indices)
    import torch
    # Always on torch's current stream of the target device, also for host inputs: the outputs come from torch's caching
    # allocator, which may hand out a block that queued torch work on that stream still writes.
    ctx = _pick_ctx(*devs) if devs else _pick_ctx(torch.cuda.current_device() if torch.cuda.is_available() else None)
    dev = torch.device("cuda", ctx.device)
    buf = torch.empty(int(3 * cells.sum()), dtype=torch.float32, device=dev)
    zb = torch.empty(int(cells.sum()), dtype=torch.float32, device=dev) if zbuffer else None
    count = np.zeros(C, np.int32)
    status = np.zeros(C, np.int32)
    H = np.ascontiguousarray(shp[:, 0], np.int32)
    W = np.ascontiguousarray(shp[:, 1], np.int32)
    ctx.check(ctx.lib.esacb200_render_init_maps(
        ctx.handle, C, pts.ptr if P else None, P, offs.ctypes.data, idx.ptr if V else None, pose34.ctypes.data,
        f.ctypes.data, s.ctypes.data, H.ctypes.data, W.ctypes.data, buf.data_ptr(),
        zb.data_ptr() if zb is not None else None, count.ctypes.data, status.ctypes.data))
    bad = np.flatnonzero(status)
    if len(bad):
        listed = ", ".join(f"{int(c)} (" + " and ".join(m for b, m in RENDER_STATUS.items() if status[c] & b) + ")"
                           for c in bad[:10])
        raise RuntimeError(f"{call}: {len(bad)} camera(s) cannot be rendered: {listed}" + (", ..." if len(bad) > 10 else ""))
    starts = np.concatenate([[0], np.cumsum(cells)])
    maps = [buf[3 * int(starts[c]):3 * int(starts[c + 1])].view(3, int(shp[c, 0]), int(shp[c, 1])) for c in range(C)]
    zbufs = None
    if zb is not None:
        zbufs = [zb[int(starts[c]):int(starts[c + 1])].view(int(shp[c, 0]), int(shp[c, 1])) for c in range(C)]
    return maps, torch.from_numpy(count), zbufs



# ------------------------------------------------------------------------------------------------
# one step of a device-resident image set (esac_b200/data.py: DeviceImageSet drives this)
# ------------------------------------------------------------------------------------------------
# The records include/esac_b200.h names, as numpy dtypes: a plan row, an image of the set, the set's device state.
DATA_ROW = np.dtype([("image", "<i4"), ("padX", "<i4"), ("padY", "<i4"), ("n_ops", "<i4"), ("ops", "<i4", (3,)),
                     ("factors", "<f4", (3,))])
DATA_IMAGE = np.dtype([("pixels", "<i8"), ("gt", "<i8"), ("focal", "<f8"), ("scene", "<i8"), ("pose", "<f4", (16,)),
                       ("group", "<i4"), ("H", "<i4"), ("W", "<i4"), ("gt_h", "<i4"), ("gt_w", "<i4"), ("unused", "<i4")])
DATA_STATE = 2   # int64 words: the next plan row, the rows the plan holds
DATA_BRIGHTNESS, DATA_CONTRAST, DATA_SATURATION = 0, 1, 2
DATA_MAX_ATTACH, DATA_MAX_SIDE, DATA_MAX_BATCH = 8, 8192, 4096
assert DATA_ROW.itemsize == 40 and DATA_IMAGE.itemsize == 120


def _storage_kind(t, what: str, call: str):
    """Set storage lives on a CUDA device or in pinned host memory (which the kernels read through its device alias)."""
    if not (t.is_cuda or t.is_pinned()):
        raise RuntimeError(f"{call}: {what} must be a CUDA tensor or a pinned CPU tensor")


def data_step_async(pixels, images, plan, state, group, mean, std, work, outImage, outShifts, outCameras, outPoses,
                    outScenes, outIndices, outStatus, gt=None, outCoords=None, attachments=(), outAttachments=()):
    """One step of B images of shape group `group` of a device-resident image set, enqueued on torch's current stream with
    no host synchronisation, so that a CUDA graph can capture it (include/esac_b200.h: esacb200_data_step_async).
    Storage (CUDA or pinned CPU tensors): pixels uint8 [bytes] (RGB [H,W,3] per image), gt float32 [floats] or None,
    attachments float32 [N, ...] each.  Device tensors: images uint8 [N, 120] (DATA_IMAGE records), plan int32
    [capacity, 10] (DATA_ROW rows), state int64 [2] (DATA_STATE), work int64 [B].  Outputs (CUDA): outImage float32
    [B,3,H,W], outShifts int32 [B,2], outCameras float32 [B,3], outPoses float32 [B,4,4], outScenes / outIndices int64
    [B], outStatus int32 [1] (0 ok, 1 plan exhausted, 2 a row of another group), outCoords float32 [B,3,h,w] (with gt),
    outAttachments float32 [B, ...] (one per attachment).  mean, std: three numbers each."""
    call = "data_step_async"
    named = {"pixels": pixels, "images": images, "plan": plan, "state": state, "work": work, "outImage": outImage,
             "outShifts": outShifts, "outCameras": outCameras, "outPoses": outPoses, "outScenes": outScenes,
             "outIndices": outIndices, "outStatus": outStatus}
    if (gt is None) != (outCoords is None):
        raise RuntimeError(f"{call}: gt and outCoords must both be given or both be None")
    if gt is not None:
        named.update(gt=gt, outCoords=outCoords)
    for k, (a, o) in enumerate(zip(attachments, outAttachments)):
        named.update({f"attachments[{k}]": a, f"outAttachments[{k}]": o})
    for what, t in named.items():
        if not _is_torch(t):
            raise RuntimeError(f"{call} takes torch tensors only ({what} is a {type(t).__name__})")
    if len(attachments) != len(outAttachments) or len(attachments) > DATA_MAX_ATTACH:
        raise RuntimeError(f"{call}: {len(attachments)} attachments for {len(outAttachments)} outputs "
                           f"(at most {DATA_MAX_ATTACH})")
    if isinstance(group, bool) or not isinstance(group, numbers.Integral) or group < 0:
        raise RuntimeError(f"{call}: group must be a non-negative int, got {group!r}")
    mean, std = (np.ascontiguousarray(np.resize(np.asarray(v, np.float32).reshape(-1), 3) if np.size(v) == 1 else
                                      np.asarray(v, np.float32).reshape(-1)) for v in (mean, std))
    if mean.shape != (3,) or std.shape != (3,) or not np.isfinite(mean).all() or not np.isfinite(std).all() or \
            (std == 0).any():
        raise RuntimeError(f"{call}: mean and std must be three finite numbers each, std nonzero")
    _check(outImage, "Float", 4, "outImage")
    B, three, H, W = (int(v) for v in outImage.shape)
    if three != 3 or not 1 <= B <= DATA_MAX_BATCH or not (1 <= H <= DATA_MAX_SIDE and 1 <= W <= DATA_MAX_SIDE):
        raise RuntimeError(f"outImage must be [B,3,H,W] with B in [1, {DATA_MAX_BATCH}] and sides in [1, {DATA_MAX_SIDE}], "
                           f"got {list(outImage.shape)}")
    _check(images, "Byte", 2, "images")
    N = int(images.shape[0])
    _check(plan, "Int", 2, "plan")
    capacity = int(plan.shape[0])
    if N < 1 or capacity < 1:
        raise RuntimeError(f"{call}: the set holds {N} images and the plan {capacity} rows; both must be positive")
    fixed = {"images": (images, "Byte", (N, DATA_IMAGE.itemsize)), "plan": (plan, "Int", (capacity, DATA_ROW.itemsize // 4)),
             "state": (state, "Long", (DATA_STATE,)), "work": (work, "Long", (B,)), "outImage": (outImage, "Float", (B, 3, H, W)),
             "outShifts": (outShifts, "Int", (B, 2)), "outCameras": (outCameras, "Float", (B, 3)),
             "outPoses": (outPoses, "Float", (B, 4, 4)), "outScenes": (outScenes, "Long", (B,)),
             "outIndices": (outIndices, "Long", (B,)), "outStatus": (outStatus, "Int", (1,))}
    gt_h = gt_w = 0
    if gt is not None:
        _check(gt, "Float", 1, "gt")
        _check(outCoords, "Float", 4, "outCoords")
        _, _, gt_h, gt_w = (int(v) for v in outCoords.shape)
        if not (1 <= gt_h <= DATA_MAX_SIDE and 1 <= gt_w <= DATA_MAX_SIDE):
            raise RuntimeError(f"outCoords must be [B,3,h,w] with sides in [1, {DATA_MAX_SIDE}], got {list(outCoords.shape)}")
        fixed["outCoords"] = (outCoords, "Float", (B, 3, gt_h, gt_w))
    numel = []
    for k, (a, o) in enumerate(zip(attachments, outAttachments)):
        _check(a, "Float", a.dim(), f"attachments[{k}]")
        if a.dim() < 1 or int(a.shape[0]) != N or a.numel() == 0 or not a.is_contiguous():
            raise RuntimeError(f"attachments[{k}] must be a contiguous float32 [{N}, ...] tensor with elements, "
                               f"got {list(a.shape)}")
        fixed[f"outAttachments[{k}]"] = (o, "Float", (B,) + tuple(int(v) for v in a.shape[1:]))
        numel.append(a.numel() // N)
    for what, (t, dt, shape) in fixed.items():
        _check(t, dt, len(shape), what)
        if tuple(int(v) for v in t.shape) != shape or not t.is_contiguous():
            raise RuntimeError(f"{what} must be a contiguous {list(shape)} tensor, got {list(t.shape)}")
    _check(pixels, "Byte", 1, "pixels")
    storage = [("pixels", pixels)] + ([("gt", gt)] if gt is not None else []) + \
        [(f"attachments[{k}]", a) for k, a in enumerate(attachments)]
    for what, t in storage:
        if not t.is_contiguous():
            raise RuntimeError(f"{what} must be contiguous")
        _storage_kind(t, what, call)
    for what, (t, _, _) in fixed.items():
        if not t.is_cuda:
            raise RuntimeError(f"{call} takes CUDA tensors only ({what} is on the CPU)")
    devs = {t.device.index for _, (t, _, _) in fixed.items()} | {t.device.index for _, t in storage if t.is_cuda}
    if len(devs) > 1:
        raise RuntimeError(f"esac_b200: tensors live on different CUDA devices {sorted(devs)}")
    ctx = _pick_ctx(*devs)
    n = len(attachments)
    att = (C.c_void_p * max(n, 1))(*[a.data_ptr() for a in attachments])
    att_out = (C.c_void_p * max(n, 1))(*[o.data_ptr() for o in outAttachments])
    att_numel = (C.c_int64 * max(n, 1))(*numel)
    ctx.check(ctx.lib.esacb200_data_step_async(
        ctx.handle, pixels.data_ptr(), gt.data_ptr() if gt is not None else None, images.data_ptr(), N, int(group), H, W,
        gt_h, gt_w, mean.ctypes.data, std.ctypes.data, n, att, att_numel, plan.data_ptr(), capacity, state.data_ptr(), B,
        work.data_ptr(), outImage.data_ptr(), outShifts.data_ptr(), outCameras.data_ptr(), outPoses.data_ptr(),
        outCoords.data_ptr() if outCoords is not None else None, outScenes.data_ptr(), outIndices.data_ptr(), att_out,
        outStatus.data_ptr()))

def set_seed(seed: int, device: int | None = None):
    context(device).set_seed(seed)


def set_option(key: str, value: float, device: int | None = None):
    context(device).set_option(key, value)


def inject_cells(cells, device: int | None = None):
    context(device).inject_cells(cells)


def last_stats(device: int | None = None) -> dict:
    return context(device).stats()


def last_hypotheses(device: int | None = None, losses: bool = False) -> dict:
    return context(device).hypotheses(losses)
