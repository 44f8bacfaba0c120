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

import ctypes as C
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
             "left_to_tail": int(out[3]), "accepted_staged": int(out[4]), "lanes": int(out[5])}
        return d

    def sample_trace(self) -> np.ndarray:
        """[lane, wave, kernel (0 prefilter, 1 exact), (start, end)] in ns relative to the first stamp; -1 where nothing ran."""
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
        return _TORCH_NAMES.get(str(t.dtype), str(t.dtype))
    return _NP_NAMES.get(str(np.asarray(t).dtype), str(np.asarray(t).dtype))


def _check(t, want: str, rank: int, what: str):
    """Same failure mode as at::Tensor::accessor<T, N>() in the reference (esac.cpp:80-84): RuntimeError."""
    have = _dtype_name(t)
    if have != want:
        raise RuntimeError(f"expected scalar type {want} but found {have} ({what})")
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
    return (v.dim() == 0) if _is_torch(v) else np.ndim(v) == 0


def _per_image(v, B: int, dtype, what: str) -> np.ndarray:
    """A batch argument as B contiguous host values of `dtype`: a number is broadcast; a sequence, numpy array or tensor
    (CPU or CUDA) must hold B values.  float64 values (a DataLoader's focal lengths) round to float32 exactly as ctypes
    rounds a Python float.  Raises RuntimeError before any context exists, so the check runs without a GPU."""
    if _is_number(v):
        v = [int(v) if dtype == np.int32 else float(v)] * B
    elif _is_torch(v):
        v = v.detach().cpu().numpy()
    a = np.ascontiguousarray(np.asarray(v).reshape(-1), dtype=dtype)
    if a.shape[0] != B:
        kind = "an int or {} ints" if dtype == np.int32 else "a number or {} numbers"
        raise RuntimeError(f"{what} must be {kind.format(B)}, got {a.shape[0]} values")
    return a


def _is_list(t) -> bool:
    """A ragged batch: a list or tuple of per-image tensors / arrays (each with its own H x W)."""
    return isinstance(t, (list, tuple))


def _check_list(ts, rank: int, what: str, B: int | None = None) -> list:
    """Checks a ragged argument (float32 elements of `rank` dims, all CPU / numpy or all CUDA, B of them) and returns the
    element shapes.  Raises RuntimeError before any context exists."""
    if not _is_list(ts):
        raise RuntimeError(f"{what} must be a list or tuple of tensors, as the other image arguments")
    if len(ts) == 0:
        raise RuntimeError(f"{what} is an empty list")
    if B is not None and len(ts) != B:
        raise RuntimeError(f"{what} holds {len(ts)} tensors for {B} images")
    for b, t in enumerate(ts):
        _check(t, "Float", rank, f"{what}[{b}]")
    if len({bool(_is_torch(t) and t.is_cuda) for t in ts}) > 1:
        raise RuntimeError(f"{what} mixes CPU and CUDA tensors")
    return [tuple(int(v) for v in t.shape) for t in ts]


def _check_maps(shapes, what: str) -> int:
    """[E,3,H,W] elements with one E, each large enough to draw 4 distinct cells (esac.cpp:110-113); returns E."""
    E = shapes[0][0]
    for b, s in enumerate(shapes):
        if s[1] != 3 or s[0] != E:
            raise RuntimeError(f"{what}[{b}] must be [E,3,H,W] with the E of image 0 ({E}), got {list(s)}")
        if (s[3] - 1) * (s[2] - 1) < 4:
            raise RuntimeError(f"{what}[{b}]: map {s[3]}x{s[2]} too small to draw 4 distinct cells")
    return E


def _ptr_array(args) -> C.Array:
    return (C.c_void_p * len(args))(*[a.ptr for a in args])


def _dims(shapes, axis: int) -> np.ndarray:
    return np.ascontiguousarray([s[axis] for s in shapes], np.int32)


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
    ctx.check(ctx.lib.esacb200_forward(ctx.handle, co.ptr, E, H, W, aptr, astride, M, op.ptr, int(shiftX), int(shiftY),
                                       float(focalLength), float(ppointX), float(ppointY), float(inlierThreshold),
                                       float(inlierAlpha), float(inlierBeta), float(maxReproj), int(subSampling),
                                       C.byref(expert)))
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
                                        float(wLossTrans), float(lossCut), int(shiftX), int(shiftY), float(focalLength),
                                        float(ppointX), float(ppointY), float(inlierThreshold), float(inlierAlpha),
                                        float(inlierBeta), float(maxReproj), int(subSampling), C.byref(loss)))
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
    ctx.set_option("hyp_offset", hyp_offset)
    try:
        rc = ctx.lib.esacb200_backward_sharded(ctx.handle, co.ptr, gr.ptr, E, H, W, aptr, astride, M, gt.ptr, float(wLossRot),
                                               float(wLossTrans), float(lossCut), int(shiftX), int(shiftY), float(focalLength),
                                               float(ppointX), float(ppointY), float(inlierThreshold), float(inlierAlpha),
                                               float(inlierBeta), float(maxReproj), int(subSampling), cb, None, C.byref(loss))
    finally:
        ctx.set_option("hyp_offset", 0)
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
    if _is_list(sceneCoordinates):
        return _forward_ragged(sceneCoordinates, hypAssignment, outPoses, shiftX, shiftY, focalLength, ppointX, ppointY,
                               inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling)
    _check(sceneCoordinates, "Float", 5, "sceneCoordinates")
    _check(hypAssignment, "Long", 2, "hypAssignment")
    _check(outPoses, "Float", 3, "outPoses")
    B, E, C3, H, W = (int(v) for v in sceneCoordinates.shape)
    if C3 != 3 or tuple(outPoses.shape) != (B, 4, 4) or int(hypAssignment.shape[0]) != B:
        raise RuntimeError("shapes must be [B,E,3,H,W], [B,M], [B,4,4]")
    one_camera = all(_is_number(v) for v in (shiftX, shiftY, focalLength, ppointX, ppointY))
    if not one_camera:
        sx, sy = _per_image(shiftX, B, np.int32, "shiftX"), _per_image(shiftY, B, np.int32, "shiftY")
        fs = _per_image(focalLength, B, np.float32, "focalLength")
        cx, cy = _per_image(ppointX, B, np.float32, "ppointX"), _per_image(ppointY, B, np.float32, "ppointY")
    co = _Arg(sceneCoordinates)
    op = _Arg(outPoses, writable=True)
    ha = _Arg(hypAssignment)
    M = int(hypAssignment.shape[1])
    ctx = _pick_ctx(co.device, op.device, ha.device)
    experts = (C.c_int * B)()
    if one_camera:
        rc = ctx.lib.esacb200_forward_batch(ctx.handle, B, co.ptr, E, H, W, ha.ptr, 1, M, op.ptr, int(shiftX), int(shiftY),
                                            float(focalLength), float(ppointX), float(ppointY), float(inlierThreshold),
                                            float(inlierAlpha), float(inlierBeta), float(maxReproj), int(subSampling), experts)
    else:
        rc = ctx.lib.esacb200_forward_batch_cameras(ctx.handle, B, co.ptr, E, H, W, ha.ptr, 1, M, op.ptr, sx.ctypes.data,
                                                    sy.ctypes.data, fs.ctypes.data, cx.ctypes.data, cy.ctypes.data,
                                                    float(inlierThreshold), float(inlierAlpha), float(inlierBeta),
                                                    float(maxReproj), int(subSampling), experts)
    ctx.check(rc)
    op.finish()
    return [int(e) for e in experts]


def _forward_ragged(sceneCoordinates, hypAssignment, outPoses, shiftX, shiftY, focalLength, ppointX, ppointY,
                    inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling) -> list:
    shapes = _check_list(sceneCoordinates, 4, "sceneCoordinates")
    B = len(shapes)
    E = _check_maps(shapes, "sceneCoordinates")
    _check(hypAssignment, "Long", 2, "hypAssignment")
    _check(outPoses, "Float", 3, "outPoses")
    if tuple(outPoses.shape) != (B, 4, 4) or int(hypAssignment.shape[0]) != B:
        raise RuntimeError(f"a list of {B} maps needs hypAssignment [{B},M] and outPoses [{B},4,4]")
    sx, sy = _per_image(shiftX, B, np.int32, "shiftX"), _per_image(shiftY, B, np.int32, "shiftY")
    fs = _per_image(focalLength, B, np.float32, "focalLength")
    cx, cy = _per_image(ppointX, B, np.float32, "ppointX"), _per_image(ppointY, B, np.float32, "ppointY")
    co = [_Arg(t) for t in sceneCoordinates]
    op = _Arg(outPoses, writable=True)
    ha = _Arg(hypAssignment)
    M = int(hypAssignment.shape[1])
    ctx = _pick_ctx(*(a.device for a in co), op.device, ha.device)
    experts = (C.c_int * B)()
    hs, ws = _dims(shapes, 2), _dims(shapes, 3)
    ctx.check(ctx.lib.esacb200_forward_ragged(ctx.handle, B, _ptr_array(co), hs.ctypes.data, ws.ctypes.data, E, ha.ptr, 1, M, op.ptr,
                                              sx.ctypes.data, sy.ctypes.data, fs.ctypes.data, cx.ctypes.data, cy.ctypes.data,
                                              float(inlierThreshold), float(inlierAlpha), float(inlierBeta), float(maxReproj),
                                              int(subSampling), experts))
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
    if _is_list(sceneCoordinates) or _is_list(outGradients):
        return _backward_ragged(sceneCoordinates, outGradients, hypAssignment, gtPoses, wLossRot, wLossTrans, lossCut, shiftX,
                                shiftY, focalLength, ppointX, ppointY, inlierThreshold, inlierAlpha, inlierBeta, maxReproj,
                                subSampling)
    _check(sceneCoordinates, "Float", 5, "sceneCoordinates")
    _check(outGradients, "Float", 5, "outGradients")
    _check(hypAssignment, "Long", 2, "hypAssignment")
    _check(gtPoses, "Float", 3, "gtPoses")
    B, E, C3, H, W = (int(v) for v in sceneCoordinates.shape)
    if (C3 != 3 or tuple(outGradients.shape) != tuple(sceneCoordinates.shape) or tuple(gtPoses.shape) != (B, 4, 4)
            or int(hypAssignment.shape[0]) != B):
        raise RuntimeError("shapes must be [B,E,3,H,W], [B,E,3,H,W], [B,M], [B,4,4]")
    co = _Arg(sceneCoordinates)
    og = _Arg(outGradients, writable=True)
    ha = _Arg(hypAssignment)
    gt = _Arg(gtPoses)
    M = int(hypAssignment.shape[1])
    sx, sy = _per_image(shiftX, B, np.int32, "shiftX"), _per_image(shiftY, B, np.int32, "shiftY")
    one_camera = all(_is_number(v) for v in (focalLength, ppointX, ppointY))
    if not one_camera:
        fs = _per_image(focalLength, B, np.float32, "focalLength")
        cx, cy = _per_image(ppointX, B, np.float32, "ppointX"), _per_image(ppointY, B, np.float32, "ppointY")
    ctx = _pick_ctx(co.device, og.device, ha.device, gt.device)
    losses = np.zeros(B, np.float64)
    head = (ctx.handle, B, co.ptr, og.ptr, E, H, W, ha.ptr, 1, M, gt.ptr, float(wLossRot), float(wLossTrans), float(lossCut),
            sx.ctypes.data, sy.ctypes.data)
    tail = (float(inlierThreshold), float(inlierAlpha), float(inlierBeta), float(maxReproj), int(subSampling), losses.ctypes.data)
    if one_camera:
        rc = ctx.lib.esacb200_backward_batch(*head, float(focalLength), float(ppointX), float(ppointY), *tail)
    else:
        rc = ctx.lib.esacb200_backward_batch_cameras(*head, fs.ctypes.data, cx.ctypes.data, cy.ctypes.data, *tail)
    ctx.check(rc)
    og.finish()
    return [float(v) for v in losses]


def _backward_ragged(sceneCoordinates, outGradients, hypAssignment, gtPoses, wLossRot, wLossTrans, lossCut, shiftX, shiftY,
                     focalLength, ppointX, ppointY, inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling) -> list:
    shapes = _check_list(sceneCoordinates, 4, "sceneCoordinates")
    B = len(shapes)
    E = _check_maps(shapes, "sceneCoordinates")
    gshapes = _check_list(outGradients, 4, "outGradients", B)
    for b in range(B):
        if gshapes[b] != shapes[b]:
            raise RuntimeError(f"outGradients[{b}] is {list(gshapes[b])}, sceneCoordinates[{b}] is {list(shapes[b])}")
    _check(hypAssignment, "Long", 2, "hypAssignment")
    _check(gtPoses, "Float", 3, "gtPoses")
    if tuple(gtPoses.shape) != (B, 4, 4) or int(hypAssignment.shape[0]) != B:
        raise RuntimeError(f"a list of {B} maps needs hypAssignment [{B},M] and gtPoses [{B},4,4]")
    sx, sy = _per_image(shiftX, B, np.int32, "shiftX"), _per_image(shiftY, B, np.int32, "shiftY")
    fs = _per_image(focalLength, B, np.float32, "focalLength")
    cx, cy = _per_image(ppointX, B, np.float32, "ppointX"), _per_image(ppointY, B, np.float32, "ppointY")
    co = [_Arg(t) for t in sceneCoordinates]
    og = [_Arg(t, writable=True) for t in outGradients]
    ha = _Arg(hypAssignment)
    gt = _Arg(gtPoses)
    M = int(hypAssignment.shape[1])
    ctx = _pick_ctx(*(a.device for a in co + og), ha.device, gt.device)
    losses = np.zeros(B, np.float64)
    hs, ws = _dims(shapes, 2), _dims(shapes, 3)
    ctx.check(ctx.lib.esacb200_backward_ragged(ctx.handle, B, _ptr_array(co), _ptr_array(og), hs.ctypes.data, ws.ctypes.data, E,
                                               ha.ptr, 1, M, gt.ptr, float(wLossRot), float(wLossTrans), float(lossCut),
                                               sx.ctypes.data, sy.ctypes.data, fs.ctypes.data, cx.ctypes.data, cy.ctypes.data,
                                               float(inlierThreshold), float(inlierAlpha), float(inlierBeta), float(maxReproj),
                                               int(subSampling), losses.ctypes.data))
    for a in og:
        a.finish()
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
    if _is_list(prediction) or _is_list(outGradients):
        return _reproj_loss_ragged(prediction, gtPoses, focalLength, padX, padY, cutLoss, subSampling, ppointX, ppointY,
                                   outGradients, maxReproj, minDepth)
    _check(prediction, "Float", 4, "prediction")
    _check(gtPoses, "Float", 3, "gtPoses")
    B, C3, H, W = (int(v) for v in prediction.shape)
    if C3 != 3 or tuple(gtPoses.shape) != (B, 4, 4):
        raise RuntimeError("shapes must be [B,3,H,W] and [B,4,4]")
    pr = _Arg(prediction)
    gt = _Arg(gtPoses)
    og = None
    if outGradients is not None:
        _check(outGradients, "Float", 4, "outGradients")
        if tuple(outGradients.shape) != tuple(prediction.shape):
            raise RuntimeError("outGradients must have the shape of prediction")
        og = _Arg(outGradients, writable=True)

    sx, sy = _per_image(padX, B, np.int32, "padX"), _per_image(padY, B, np.int32, "padY")
    ppx = W * subSampling / 2 if ppointX is None else ppointX
    ppy = H * subSampling / 2 if ppointY is None else ppointY
    one_camera = all(_is_number(v) for v in (focalLength, ppx, ppy))
    if not one_camera:
        fs = _per_image(focalLength, B, np.float32, "focalLength")
        cx, cy = _per_image(ppx, B, np.float32, "ppointX"), _per_image(ppy, B, np.float32, "ppointY")
    ctx = _pick_ctx(pr.device, gt.device, og.device if og else None)
    losses = np.zeros(B, np.float64)
    head = (ctx.handle, B, pr.ptr, og.ptr if og else None, H, W, gt.ptr, sx.ctypes.data, sy.ctypes.data)
    tail = (int(subSampling), float(cutLoss), float(maxReproj), float(minDepth), losses.ctypes.data)
    if one_camera:
        rc = ctx.lib.esacb200_reproj_loss(*head, float(focalLength), float(ppx), float(ppy), *tail)
    else:
        rc = ctx.lib.esacb200_reproj_loss_cameras(*head, fs.ctypes.data, cx.ctypes.data, cy.ctypes.data, *tail)
    ctx.check(rc)
    if og:
        og.finish()
    return [float(v) for v in losses]


def _reproj_loss_ragged(prediction, gtPoses, focalLength, padX, padY, cutLoss, subSampling, ppointX, ppointY, outGradients,
                        maxReproj, minDepth):
    shapes = _check_list(prediction, 3, "prediction")
    B = len(shapes)
    for b, s in enumerate(shapes):
        if s[0] != 3:
            raise RuntimeError(f"prediction[{b}] must be [3,H,W], got {list(s)}")
    _check(gtPoses, "Float", 3, "gtPoses")
    if tuple(gtPoses.shape) != (B, 4, 4):
        raise RuntimeError(f"a list of {B} predictions needs gtPoses [{B},4,4]")
    og = None
    if outGradients is not None:
        gshapes = _check_list(outGradients, 3, "outGradients", B)
        for b in range(B):
            if gshapes[b] != shapes[b]:
                raise RuntimeError(f"outGradients[{b}] is {list(gshapes[b])}, prediction[{b}] is {list(shapes[b])}")
        og = [_Arg(t, writable=True) for t in outGradients]
    sx, sy = _per_image(padX, B, np.int32, "padX"), _per_image(padY, B, np.int32, "padY")
    fs = _per_image(focalLength, B, np.float32, "focalLength")
    # the default principal point is the centre of each image's own sub*W x sub*H frame
    ppx = [s[2] * subSampling / 2 for s in shapes] if ppointX is None else ppointX
    ppy = [s[1] * subSampling / 2 for s in shapes] if ppointY is None else ppointY
    cx, cy = _per_image(ppx, B, np.float32, "ppointX"), _per_image(ppy, B, np.float32, "ppointY")
    pr = [_Arg(t) for t in prediction]
    gt = _Arg(gtPoses)
    ctx = _pick_ctx(*(a.device for a in pr + (og or [])), gt.device)
    losses = np.zeros(B, np.float64)
    hs, ws = _dims(shapes, 1), _dims(shapes, 2)
    ctx.check(ctx.lib.esacb200_reproj_loss_ragged(ctx.handle, B, _ptr_array(pr), _ptr_array(og) if og else None, hs.ctypes.data,
                                                  ws.ctypes.data, gt.ptr, sx.ctypes.data, sy.ctypes.data, fs.ctypes.data,
                                                  cx.ctypes.data, cy.ctypes.data, int(subSampling), float(cutLoss),
                                                  float(maxReproj), float(minDepth), losses.ctypes.data))
    for a in og or []:
        a.finish()
    return [float(v) for v in losses]


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
    if _is_list(prediction) or _is_list(gtCoords) or _is_list(outGradients):
        return _coord_loss_ragged(prediction, gtCoords, cutLoss, outGradients, return_counts)
    _check(prediction, "Float", 4, "prediction")
    _check(gtCoords, "Float", 4, "gtCoords")
    B, C3, Hp, Wp = (int(v) for v in prediction.shape)
    Bg, Cg, Hg, Wg = (int(v) for v in gtCoords.shape)
    if C3 != 3 or Cg != 3 or Bg != B:
        raise RuntimeError(f"shapes must be [B,3,Hp,Wp] and [B,3,Hg,Wg], got {list(prediction.shape)} and {list(gtCoords.shape)}")
    if abs(Hp - Hg) > 1 or abs(Wp - Wg) > 1:
        raise RuntimeError(f"tensor size mismatch: prediction {Hp}x{Wp}, ground truth {Hg}x{Wg} (util.assert_size allows 1)")
    og = None
    if outGradients is not None:
        _check(outGradients, "Float", 4, "outGradients")
        if tuple(outGradients.shape) != tuple(prediction.shape):
            raise RuntimeError("outGradients must have the shape of prediction")
        og = _Arg(outGradients, writable=True)
    pr = _Arg(prediction)
    gt = _Arg(gtCoords)
    ctx = _pick_ctx(pr.device, gt.device, og.device if og else None)
    losses = np.zeros(B, np.float64)
    counts = np.zeros(B, np.int64)
    ctx.check(ctx.lib.esacb200_coord_loss(ctx.handle, B, pr.ptr, Hp, Wp, gt.ptr, Hg, Wg, og.ptr if og else None, float(cutLoss),
                                          losses.ctypes.data, counts.ctypes.data))
    if og:
        og.finish()
    out = [float(v) for v in losses]
    return (out, [int(v) for v in counts]) if return_counts else out


def _coord_loss_ragged(prediction, gtCoords, cutLoss, outGradients, return_counts):
    shapes = _check_list(prediction, 3, "prediction")
    B = len(shapes)
    gshapes = _check_list(gtCoords, 3, "gtCoords", B)
    for b in range(B):
        (c, hp, wp), (cg, hg, wg) = shapes[b], gshapes[b]
        if c != 3 or cg != 3:
            raise RuntimeError(f"prediction[{b}] / gtCoords[{b}] must be [3,H,W], got {list(shapes[b])} and {list(gshapes[b])}")
        if abs(hp - hg) > 1 or abs(wp - wg) > 1:
            raise RuntimeError(f"image {b}: tensor size mismatch: prediction {hp}x{wp}, ground truth {hg}x{wg} "
                               "(util.assert_size allows 1)")
    og = None
    if outGradients is not None:
        oshapes = _check_list(outGradients, 3, "outGradients", B)
        for b in range(B):
            if oshapes[b] != shapes[b]:
                raise RuntimeError(f"outGradients[{b}] is {list(oshapes[b])}, prediction[{b}] is {list(shapes[b])}")
        og = [_Arg(t, writable=True) for t in outGradients]
    pr = [_Arg(t) for t in prediction]
    gt = [_Arg(t) for t in gtCoords]
    ctx = _pick_ctx(*(a.device for a in pr + gt + (og or [])))
    losses = np.zeros(B, np.float64)
    counts = np.zeros(B, np.int64)
    hp, wp, hg, wg = _dims(shapes, 1), _dims(shapes, 2), _dims(gshapes, 1), _dims(gshapes, 2)
    ctx.check(ctx.lib.esacb200_coord_loss_ragged(ctx.handle, B, _ptr_array(pr), hp.ctypes.data, wp.ctypes.data, _ptr_array(gt),
                                                 hg.ctypes.data, wg.ctypes.data, _ptr_array(og) if og else None, float(cutLoss),
                                                 losses.ctypes.data, counts.ctypes.data))
    for a in og or []:
        a.finish()
    out = [float(v) for v in losses]
    return (out, [int(v) for v in counts]) if return_counts else out


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
    shiftX, shiftY, f, ppx, ppy, tau, alpha, beta, maxReproj, sub = params
    ctx.check(ctx.lib.esacb200_forward_pack(ctx.handle, co.ptr, E, H, W, aptr, astride, M, M_pad, int(shiftX), int(shiftY), float(f),
                                            float(ppx), float(ppy), float(tau), float(alpha), float(beta), float(maxReproj),
                                            int(sub), int(expert_offset), pack_out.data_ptr()))


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
    ctx.set_option("hyp_offset", hyp_offset)
    ctx.set_option("hyp_stride", hyp_stride)
    try:
        rc = ctx.lib.esacb200_forward_sharded(ctx.handle, co.ptr, E, H, W, aptr, astride, M, M_pad, op.ptr, int(shiftX), int(shiftY),
                                              float(focalLength), float(ppointX), float(ppointY), float(inlierThreshold),
                                              float(inlierAlpha), float(inlierBeta), float(maxReproj), int(subSampling),
                                              int(expert_offset), C.byref(expert))
    finally:
        ctx.set_option("hyp_offset", 0)
        ctx.set_option("hyp_stride", 1)
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
    ctx.set_option("hyp_offset", hyp_offset)
    ctx.set_option("hyp_stride", hyp_stride)
    try:
        rc = ctx.lib.esacb200_backward_sharded_nccl(ctx.handle, co.ptr, gr.ptr, E, H, W, aptr, astride, M, gt.ptr, float(wLossRot),
                                                    float(wLossTrans), float(lossCut), int(shiftX), int(shiftY), float(focalLength),
                                                    float(ppointX), float(ppointY), float(inlierThreshold), float(inlierAlpha),
                                                    float(inlierBeta), float(maxReproj), int(subSampling), int(bool(reduce_grads)),
                                                    C.byref(loss))
    finally:
        ctx.set_option("hyp_offset", 0)
        ctx.set_option("hyp_stride", 1)
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
    ctx.check(ctx.lib.esacb200_score_poses(ctx.handle, co.ptr, E, H, W, aptr, astride, M, poses6.ctypes.data, int(shiftX),
                                           int(shiftY), float(focalLength), float(ppointX), float(ppointY),
                                           float(inlierThreshold), float(inlierAlpha), float(inlierBeta), float(maxReproj),
                                           int(subSampling), out.ctypes.data))
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
