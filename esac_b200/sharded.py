"""Multi-GPU esac.forward / esac.backward: experts (and with them the hypotheses) sharded across ranks, one process per GPU.

Hypotheses are independent through sampling, P3P, scoring, refinement and per-hypothesis gradients; the path has ONE
exchange in forward -- the softmax / argmax over all scores (esac.cpp:153-155) -- and TWO in backward (the softmax
normalisation, then the expectation sum_h p_h loss_h every gradient needs, esac.cpp:357-362, esac_derivative.h:372-374);
SURVEY.md section 8e.  Every rank runs the complete local pipeline on the experts it owns, including the refinement of its
local best hypothesis (the ranks run concurrently, so that costs no latency), and contributes the record
    [ scores (M_pad, -inf beyond its own M) | refined pose of its winner (16) | global expert id | local winner | M |
      hyp_offset | hyp_stride ]
to one all-gather; the first strict maximum in the hypothesis order of the unsharded problem (global index of local
hypothesis k = hyp_offset + k * hyp_stride) is the reference's draw() (esac_util.h:519-523).

Two transports:
  * the library's own NCCL communicator (`init_comm`): esacb200_forward_sharded / esacb200_backward_sharded_nccl issue the
    collectives on the library's stream, select on the device and synchronise once -- the production path;
  * torch.distributed (any backend) around esacb200_forward_pack / the exchange callback of esacb200_backward_sharded --
    kept for the CPU (gloo) tests of the host logic and as a fallback.
Shards may hold different numbers of hypotheses, including none (real gating draws give every expert a different count).
"""
from __future__ import annotations

import numpy as np

from . import api

_NEG_INF = float("-inf")
_lib_comm: dict = {}   # device index -> (world, rank) of the library communicator


def init_comm(group=None, device: int | None = None):
    """Create the library's NCCL communicator over the ranks of `group` (default: the world group): rank 0 draws an
    ncclUniqueId, torch.distributed carries its 128 bytes to the others, every rank calls ncclCommInitRank."""
    import torch
    import torch.distributed as dist
    if device is None:
        device = torch.cuda.current_device()
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    box = [api.nccl_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(box, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
    api.context(device).comm_init(world, rank, box[0])
    _lib_comm[device] = (world, rank)
    return world, rank


def destroy_comm(device: int | None = None):
    import torch
    if device is None:
        device = torch.cuda.current_device()
    if device in _lib_comm:
        api.context(device).comm_destroy()
        del _lib_comm[device]


def max_over_ranks(value: int, group=None, device=None) -> int:
    """M_pad: the largest shard size (one small all-reduce; callers with a fixed layout compute it once)."""
    import torch
    import torch.distributed as dist
    t = torch.tensor([int(value)], dtype=torch.int64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return max(int(t.item()), 1)


def pack_local(scores, pose16, expert_global: int, local_winner: int, M_pad: int | None = None, hyp_offset: int = 0,
               hyp_stride: int = 1):
    """float64 record [M_pad + api.PACK_TAIL] (see the module docstring) from a local result."""
    import torch
    scores = scores.reshape(-1).to(torch.float64)
    M = int(scores.numel())
    M_pad = M if M_pad is None else int(M_pad)
    pad = torch.full((M_pad - M,), _NEG_INF, dtype=torch.float64, device=scores.device)
    if M == 0:
        tail = torch.tensor([-1.0] * api.TAIL_M + [0.0, float(hyp_offset), float(hyp_stride)], dtype=torch.float64,
                            device=scores.device)
        return torch.cat([pad, tail])
    tail = torch.tensor([float(expert_global), float(local_winner), float(M), float(hyp_offset), float(hyp_stride)],
                        dtype=torch.float64, device=scores.device)
    return torch.cat([scores, pad, pose16.reshape(16).to(torch.float64), tail])


def select_global(gathered: np.ndarray, M_pad: int):
    """gathered: [world, M_pad + api.PACK_TAIL].  Returns (winner slot = rank * M_pad + local index, owning rank, pose 4x4 float32,
    expert id, probabilities of all M_pad * world slots) with softMax / draw(training=false) semantics (esac_util.h:461-530):
    the first strict maximum in the hypothesis order of the unsharded problem; padded slots carry -inf and probability 0."""
    world = gathered.shape[0]
    scores = gathered[:, :M_pad].reshape(-1)
    with np.errstate(invalid="ignore"):
        sf = np.exp(scores - scores.max())
    probs = sf / sf.sum()
    # global index of every slot: hyp_offset + k * hyp_stride; draw() keeps the first maximum in that order
    k = np.arange(M_pad)[None, :]
    tail = gathered[:, M_pad:]
    offset, stride = tail[:, api.TAIL_HYP_OFFSET:api.TAIL_HYP_OFFSET + 1], tail[:, api.TAIL_HYP_STRIDE:api.TAIL_HYP_STRIDE + 1]
    gidx = (offset + k * np.maximum(stride, 1)).reshape(-1)
    gidx = np.where(k.repeat(world, 0).reshape(-1) < tail[:, api.TAIL_M].repeat(M_pad), gidx, np.inf)
    if probs.max() >= 1e-8:
        cand = np.flatnonzero(probs == probs.max())
        winner = int(cand[np.argmin(gidx[cand])])
    else:
        winner = 0
    rank = winner // M_pad
    assert rank < world
    pose = tail[rank, api.TAIL_POSE:api.TAIL_EXPERT].reshape(4, 4).astype(np.float32)
    expert = int(tail[rank, api.TAIL_EXPERT])
    return winner, rank, pose, expert, probs


def make_exchange(group=None, device=None):
    """The two reductions of the sharded backward as torch.distributed collectives (NCCL on `device`, gloo on CPU):
    phase 1 all-gathers (max, sum exp) pairs and merges them into the global softmax normalisation, phase 2 sums the
    partial expectations."""
    import torch
    import torch.distributed as dist

    def exchange(phase, values):
        world = dist.get_world_size(group)
        t = torch.tensor(values, dtype=torch.float64, device=device)
        if phase == 1:
            g = torch.empty(world * 2, dtype=torch.float64, device=device)
            dist.all_gather_into_tensor(g, t, group=group)
            g = g.view(world, 2).cpu().numpy()
            gmax = float(g[:, 0].max())
            gsum = float((g[:, 1] * np.exp(g[:, 0] - gmax)).sum())
            return [gmax, gsum]
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
        return [float(v) for v in t.cpu()]

    return exchange


def _device_of(t):
    return t.device.index if getattr(t, "is_cuda", False) else None


def backward_sharded(coords_local, grads_local, assign_local, gt_pose, w_rot, w_trans, cut, params, hyp_offset: int, group=None,
                     device: int | None = None, reduce_grads: bool = False, hyp_stride: int = 1):
    """esac.backward with experts sharded expert-major across ranks: every rank owns its experts' planes and gradient
    slices (no gradient reduction); two KB-sized collectives give every rank the global softmax and the global expected
    loss, which it returns.  `hyp_offset` = number of hypotheses owned by lower ranks.  Uses the library communicator when
    `init_comm` was called for this device, else torch.distributed through the exchange callback.
    reduce_grads (library communicator only): hypothesis-major sharding -- every rank passes ALL planes and a slice of the
    hypotheses; the gradients are summed over the ranks (one ncclAllReduce) and added to grads_local on every rank."""
    dev = _device_of(coords_local)
    if dev is None:
        dev = device
    if dev is None:
        try:
            import torch
            dev = torch.cuda.current_device() if torch.cuda.is_available() else None
        except Exception:
            dev = None
    if dev in _lib_comm:
        return api.backward_sharded_nccl(coords_local, grads_local, assign_local, gt_pose, w_rot, w_trans, cut, *params,
                                         hyp_offset=hyp_offset, device=dev, reduce_grads=reduce_grads, hyp_stride=hyp_stride)
    if reduce_grads:
        raise RuntimeError("reduce_grads needs the library communicator (sharded.init_comm)")
    if int(assign_local.shape[0]) == 0:
        # a shard without hypotheses only takes part in the two reductions
        ex = make_exchange(group, coords_local.device if getattr(coords_local, "is_cuda", False) else None)
        ex(1, [-1e300, 0.0])
        return ex(2, [0.0])[0]
    ex = make_exchange(group, coords_local.device if getattr(coords_local, "is_cuda", False) else None)
    return api.backward_sharded(coords_local, grads_local, assign_local, gt_pose, w_rot, w_trans, cut, *params, exchange=ex,
                                hyp_offset=hyp_offset)


def forward_sharded(coords_local, assign_local, out_pose, params, expert_offset: int, group=None, local_forward=None,
                    hyp_offset: int = 0, M_pad: int | None = None, device: int | None = None, hyp_stride: int = 1):
    """esac.forward over experts sharded across the ranks of `group`.  coords_local [E_local,3,H,W] and
    assign_local [M_local] (expert indices local to the shard; may be empty) live on this rank; out_pose [4,4] receives the
    global winner's camera pose on every rank; returns the global expert index.  M_pad = the largest M_local of any rank
    (computed with one extra all-reduce when not given)."""
    import torch
    import torch.distributed as dist

    M = int(assign_local.shape[0])
    dev = _device_of(coords_local)
    if dev is None:
        dev = device
    if dev is None and local_forward is None:
        dev = torch.cuda.current_device()
    if local_forward is None and dev in _lib_comm:
        if M_pad is None:
            M_pad = max_over_ranks(M, group, torch.device("cuda", dev))
        return api.forward_sharded(coords_local, assign_local, out_pose, *params, expert_offset=expert_offset, M_pad=M_pad,
                                   hyp_offset=hyp_offset, device=dev, hyp_stride=hyp_stride)
    # ---- torch.distributed transport ----
    if local_forward is None:
        if not hasattr(coords_local, "is_cuda"):
            coords_local, assign_local = torch.from_numpy(coords_local), torch.from_numpy(assign_local)
        tdev = coords_local.device if coords_local.is_cuda else torch.device("cuda", dev)
        if M_pad is None:
            M_pad = max_over_ranks(M, group, tdev)
        # host inputs (the reference's callers hold CPU tensors): staged on the current stream, asynchronously if pinned
        coords_local = coords_local.to(tdev, non_blocking=True)
        assign_local = assign_local.to(tdev, non_blocking=True)
        ctx = api.context(tdev.index)
        ctx.set_option("hyp_offset", hyp_offset)
        ctx.set_option("hyp_stride", hyp_stride)
        buf = torch.empty(M_pad + api.PACK_TAIL, dtype=torch.float64, device=tdev)
        try:
            if M > 0:
                api.forward_pack(coords_local, assign_local, params, expert_offset, buf, M_pad=M_pad)   # enqueued, no host sync
            else:
                buf.copy_(pack_local(torch.empty(0, dtype=torch.float64, device=tdev), None, -1, 0, M_pad, hyp_offset, hyp_stride))
        finally:
            ctx.set_option("hyp_offset", 0)
            ctx.set_option("hyp_stride", 1)
    else:
        if M_pad is None:
            M_pad = max_over_ranks(M, group, None)
        if M > 0:
            scores, pose, e_local, lw = local_forward(coords_local, assign_local, params)
            buf = pack_local(scores, pose, expert_offset + e_local, lw, M_pad, hyp_offset, hyp_stride)
        else:
            buf = pack_local(torch.empty(0, dtype=torch.float64), None, -1, 0, M_pad, hyp_offset, hyp_stride)
    world = dist.get_world_size(group)
    rec = M_pad + api.PACK_TAIL
    gathered = torch.empty(world * rec, dtype=torch.float64, device=buf.device)
    dist.all_gather_into_tensor(gathered, buf, group=group)
    g = gathered.view(world, rec)
    if g.is_cuda:
        # selection on the device: first maximum = draw(training=false) -- in rank-major order, which is the order of the
        # unsharded problem for contiguous shards (this fallback transport does not support hyp_stride > 1 tie-breaking);
        # ONE read-back of the winner's pose and expert (the only host sync of the step)
        w = torch.argmax(g[:, :M_pad].reshape(-1))
        tail = g.reshape(-1)[(w // M_pad) * rec + M_pad + torch.arange(api.TAIL_WINNER, device=g.device)]
        if hasattr(out_pose, "is_cuda") and out_pose.is_cuda:
            out_pose.copy_(tail[api.TAIL_POSE:api.TAIL_EXPERT].reshape(4, 4))
            expert = int(tail[api.TAIL_EXPERT].item())
            if expert < 0:
                raise RuntimeError("hypAssignment holds an expert index outside the shard's experts")
            return expert
        small = tail.cpu().numpy()
        gpose, expert = small[api.TAIL_POSE:api.TAIL_EXPERT].reshape(4, 4).astype(np.float32), int(small[api.TAIL_EXPERT])
        if expert < 0:
            raise RuntimeError("hypAssignment holds an expert index outside the shard's experts")
    else:
        _, _, gpose, expert, _ = select_global(g.numpy(), M_pad)
    if hasattr(out_pose, "copy_"):
        out_pose.copy_(torch.from_numpy(gpose))
    else:
        out_pose[:, :] = gpose
    return expert
