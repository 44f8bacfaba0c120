"""torch.autograd wrapper around esac.backward (SURVEY.md section 8f, rank 1).

The reference's trainer calls the extension, then builds the gating gradient by hand and feeds both gradients to
torch.autograd.backward (train_esac.py:151-180).  EsacLoss packages exactly that: its forward returns the expected
pose loss, its backward hands d loss / d sceneCoordinates (from the extension) and the REINFORCE-style gating
gradient to autograd -- loss * histogram(e_hyps) in the default mode (train_esac.py:174-176), or, in the trainer's
`expertselection` mode (one expert drawn and expanded to all hypotheses, train_esac.py:133-135), `loss` at the drawn
expert only (train_esac.py:171-173).  CUDA tensors stay on the device."""
from __future__ import annotations

import operator

import torch

from . import api


class EsacLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, scene_coordinates, gating_log_probs, hyp_assignment, gt_pose, w_rot, w_trans, loss_cut, shift_x,
                shift_y, focal_length, ppoint_x, ppoint_y, inlier_threshold, inlier_alpha, inlier_beta, max_reproj,
                sub_sampling, expert_selection=None):
        grads = torch.zeros_like(scene_coordinates)
        loss = api.backward(scene_coordinates.detach(), grads, hyp_assignment, gt_pose, w_rot, w_trans, loss_cut, shift_x,
                            shift_y, focal_length, ppoint_x, ppoint_y, inlier_threshold, inlier_alpha, inlier_beta,
                            max_reproj, sub_sampling)
        E = scene_coordinates.shape[0]
        if expert_selection is None:
            # expert.expand(M) (train_esac.py:135-136) is a stride-0 view: that is the expertselection branch
            expert_selection = hyp_assignment.dim() == 1 and hyp_assignment.shape[0] > 1 and hyp_assignment.stride(0) == 0
        if expert_selection:
            g_gating = torch.zeros(E)
            g_gating[int(hyp_assignment[0])] = loss                                      # train_esac.py:171-173
        else:
            hist = torch.histc(hyp_assignment.float().cpu(), bins=E, min=0, max=E - 1)   # train_esac.py:140
            g_gating = loss * hist                                                        # train_esac.py:174-176
        ctx.save_for_backward(grads, g_gating.to(gating_log_probs.device).reshape(gating_log_probs.shape))
        return scene_coordinates.new_tensor(loss)

    @staticmethod
    def backward(ctx, grad_out):
        g_coords, g_gating = ctx.saved_tensors
        return (g_coords * grad_out, g_gating * grad_out) + (None,) * 16


def esac_loss(scene_coordinates, gating_log_probs, hyp_assignment, gt_pose, *params, expert_selection=None):
    """params: wLossRot, wLossTrans, lossCut, shiftX, shiftY, focalLength, ppointX, ppointY, inlierThreshold,
    inlierAlpha, inlierBeta, maxReproj, subSampling -- the positional tail of esac.backward.
    expert_selection: True = the trainer's `expertselection` gating gradient (loss at the drawn expert), False = loss *
    histogram, None = decide from the assignment tensor (a stride-0 `expert.expand(M)` view means expert selection)."""
    return EsacLoss.apply(scene_coordinates, gating_log_probs, hyp_assignment, gt_pose, *params, expert_selection)


def _as_inputs(images):
    """The images of a batched node as trailing autograd inputs, so that autograd sees every one of them: the stacked
    tensor alone, or the B tensors of a list / tuple.  Also returns `form`, which turns such a sequence of tensors (the
    inputs, or tensors made like them) back into the api's argument: the one tensor, or a list."""
    if api._is_list(images):
        return tuple(images), list
    return (images,), operator.itemgetter(0)


def _gating_rows(losses, hyp_assignment, E, expert_selection):
    rows = []
    for b, loss in enumerate(losses):
        if expert_selection:
            g = torch.zeros(E)
            g[int(hyp_assignment[b, 0])] = loss                                          # train_esac.py:171-173
        else:
            hist = torch.histc(hyp_assignment[b].float().cpu(), bins=E, min=0, max=E - 1)   # train_esac.py:140
            g = loss * hist                                                               # train_esac.py:174-176
        rows.append(g)
    return torch.stack(rows)


class EsacLossBatch(torch.autograd.Function):
    """EsacLoss over a batch of images, on api.backward_batch: forward returns the B expected pose losses, backward hands
    d loss_b / d scene_coordinates[b] and row b of the gating gradient -- loss_b * histogram(e_hyps[b]), or loss_b at the
    drawn expert in expert-selection mode -- to autograd, each computed exactly as EsacLoss computes it for one image.
    The maps come last (_as_inputs); `meta` holds the non-differentiable arguments."""

    @staticmethod
    def forward(ctx, meta, gating_log_probs, *scene_coordinates):
        form, hyp_assignment, gt_poses, params, expert_selection = meta
        grads = [torch.zeros_like(c) for c in scene_coordinates]
        losses = api.backward_batch(form([c.detach() for c in scene_coordinates]), form(grads), hyp_assignment, gt_poses,
                                    *params)
        if expert_selection is None:
            # [B,1].expand(B,M): a stride-0 row per image, the batched form of expert.expand(M)
            expert_selection = hyp_assignment.dim() == 2 and hyp_assignment.shape[1] > 1 and hyp_assignment.stride(1) == 0
        E = scene_coordinates[0].shape[-4]
        g_gating = _gating_rows(losses, hyp_assignment, E, expert_selection)
        ctx.save_for_backward(g_gating.to(gating_log_probs.device).reshape(gating_log_probs.shape), *grads)
        return scene_coordinates[0].new_tensor(losses)

    @staticmethod
    def backward(ctx, grad_out):
        g_gating, *g_coords = ctx.saved_tensors
        B = grad_out.shape[0]
        # the factor of each input: [B,1,1,1,1] for a stacked gradient [B,E,3,H,W], [1,1,1,1] for image b's [E,3,H,W]
        w = grad_out.reshape((len(g_coords), -1) + (1,) * (g_coords[0].dim() - 1))
        return ((None, g_gating * grad_out.reshape((B,) + (1,) * (g_gating.dim() - 1))) +
                tuple(g * wb for g, wb in zip(g_coords, w)))


def esac_loss_batch(scene_coordinates, gating_log_probs, hyp_assignment, gt_poses, *params, expert_selection=None):
    """The batched counterpart of esac_loss (one train_esac.py step on B images, each with its own camera):
    scene_coordinates [B,E,3,H,W], gating_log_probs [B,E], hyp_assignment [B,M], gt_poses [B,4,4]; params the positional
    tail of api.backward_batch (wLossRot, wLossTrans, lossCut, shiftX, shiftY, focalLength, ppointX, ppointY,
    inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling), where shifts and camera may be per image.
    Returns the B expected losses; image b draws the minimal sets of the b-th of B consecutive esac_loss calls.
    expert_selection as for esac_loss, decided for the whole batch (None: a stride-0 [B,1].expand(B,M) assignment).
    scene_coordinates may also be a list or tuple of B [E,3,H_b,W_b] tensors of different sizes; every element then
    receives its own gradient."""
    inputs, form = _as_inputs(scene_coordinates)
    return EsacLossBatch.apply((form, hyp_assignment, gt_poses, params, expert_selection), gating_log_probs, *inputs)


def _gating_grad(losses, hyp_assignment, E, expert_selection):
    """The gating gradient of esac_loss / esac_loss_batch computed on the assignment's device, with no host round trip:
    losses float64 [B], hyp_assignment int64 [B,M].  Row b is loss_b at the drawn expert (expert selection), or loss_b
    times the histogram of row b.  Rounded as esac_loss rounds: the float64 loss becomes a float32 first, and the product
    with the float32 histogram is a float32 product (torch multiplies a float32 tensor by a Python float in float32).
    Indices outside [0, E) (an image backward_async flags, whose loss is NaN) are counted nowhere."""
    loss32 = losses.float()[:, None]
    valid = (hyp_assignment >= 0) & (hyp_assignment < E)
    index = torch.where(valid, hyp_assignment, torch.zeros_like(hyp_assignment))
    g = torch.zeros(hyp_assignment.shape[0], E, device=hyp_assignment.device)
    if expert_selection:
        return g.scatter_(1, index[:, :1], loss32)                                           # train_esac.py:171-173
    counts = g.scatter_add_(1, index, valid.float())                                         # train_esac.py:140
    return loss32 * counts                                                                    # train_esac.py:174-176


class EsacLossAsync(torch.autograd.Function):
    """esac_loss / esac_loss_batch on api.backward_async: no host synchronisation in the forward or the backward, so the
    node, and loss.backward() through it, can be captured in a CUDA graph.  The forward returns the expected losses as
    float32, as esac_loss does; `meta` holds the non-differentiable arguments."""

    @staticmethod
    def forward(ctx, meta, gating_log_probs, scene_coordinates):
        hyp_assignment, gt_poses, shifts, cameras, params, expert_selection, status = meta
        grads = torch.zeros_like(scene_coordinates)
        lead = scene_coordinates.shape[:-4]
        losses = torch.empty(lead, dtype=torch.float64, device=scene_coordinates.device)
        if status is None:
            status = torch.empty(lead, dtype=torch.int32, device=scene_coordinates.device)
        w_rot, w_trans, loss_cut, tau, alpha, beta, max_reproj, sub = params
        api.backward_async(scene_coordinates.detach(), grads, hyp_assignment, gt_poses, shifts, cameras, w_rot, w_trans,
                           loss_cut, tau, alpha, beta, max_reproj, sub, losses, status)
        E = scene_coordinates.shape[-4]
        M = hyp_assignment.shape[-1]
        if expert_selection is None:
            # a stride-0 `expert.expand(M)` view (one image: the batched form needs its rows back to back)
            expert_selection = hyp_assignment.dim() == 1 and M > 1 and hyp_assignment.stride(0) == 0
        g_gating = _gating_grad(losses.reshape(-1), hyp_assignment.reshape(-1, M), E, expert_selection)
        ctx.save_for_backward(g_gating.reshape(gating_log_probs.shape), grads)
        return losses.float()

    @staticmethod
    def backward(ctx, grad_out):
        g_gating, g_coords = ctx.saved_tensors
        w = grad_out.reshape(grad_out.shape + (1,) * 4)
        return None, g_gating * grad_out.reshape(grad_out.shape + (1,) * (g_gating.dim() - grad_out.dim())), g_coords * w


def esac_loss_async(scene_coordinates, gating_log_probs, hyp_assignment, gt_poses, shifts, cameras, w_rot, w_trans, loss_cut,
                    tau, alpha, beta, max_reproj, sub_sampling, expert_selection=None, status=None):
    """esac_loss (one image: scene_coordinates [E,3,H,W], hyp_assignment [M], gt_poses [4,4], shifts [2], cameras [3]) or
    esac_loss_batch (scene_coordinates [B,E,3,H,W], gating_log_probs [B,E], hyp_assignment [B,M], gt_poses [B,4,4], shifts
    [B,2] int32, cameras [B,3] = focal length, ppointX, ppointY) on api.backward_async, for training steps captured in a CUDA
    graph: CUDA tensors only, the shifts, cameras and ground truth read on the device at replay time.  The losses,
    coordinate gradients and gating gradients are bitwise those of esac_loss for the same draws; image b of the j-th call
    draws what the (j*B + b)-th esac_loss call draws.  expert_selection as for esac_loss (None: a stride-0 one-image
    assignment means expert selection).  status: an int32 CUDA tensor [B] (or [] for one image) that receives
    backward_async's per-image status (1 = a bad expert index: that loss is NaN, its gradients are NaN or zero); None
    keeps it internal."""
    meta = (hyp_assignment, gt_poses, shifts, cameras, (w_rot, w_trans, loss_cut, tau, alpha, beta, max_reproj, sub_sampling),
            expert_selection, status)
    return EsacLossAsync.apply(meta, gating_log_probs, scene_coordinates)


class ReprojLoss(torch.autograd.Function):
    """ref_expert.py:103-150 as one autograd node: forward = the robust reprojection loss of a batch of predictions
    (mean over the batch of the per-image losses; the reference has one image per step), backward = its gradient, both
    from the single fused kernel behind api.reproj_loss.  The predictions come last (_as_inputs)."""

    @staticmethod
    def forward(ctx, meta, *prediction):
        form, args = meta
        grads = [torch.empty_like(p) for p in prediction]
        losses = api.reproj_loss(form([p.detach() for p in prediction]), *args, outGradients=form(grads))
        ctx.save_for_backward(*grads)
        ctx.batch = len(losses)
        return prediction[0].new_tensor(sum(losses) / len(losses))

    @staticmethod
    def backward(ctx, grad_out):
        return (None,) + tuple(g * (grad_out / ctx.batch) for g in ctx.saved_tensors)


def reproj_loss(prediction, gt_poses, focal_length, pad_x, pad_y, cut_loss, sub_sampling=8, ppoint_x=None, ppoint_y=None):
    """Drop-in for the loss block of ref_expert.py: `robust_loss = reproj_loss(prediction, gt_pose, f, padX, padY,
    opt.cutloss)` followed by `robust_loss.backward()`.  prediction [B,3,H,W] (CUDA), gt_poses [B,4,4] camera->world.
    focal_length, pad_x / pad_y and the principal point are a number or B values, so a batch may mix cameras.
    prediction may also be a list or tuple of B [3,H_b,W_b] tensors of different sizes."""
    inputs, form = _as_inputs(prediction)
    args = (gt_poses, focal_length, pad_x, pad_y, cut_loss, sub_sampling, ppoint_x, ppoint_y)
    return ReprojLoss.apply((form, args), *inputs)


class CoordLoss(torch.autograd.Function):
    """init_expert.py:106-132 as one autograd node: forward = the robust scene-coordinate loss of a batch of predictions
    (mean over the batch of the per-image losses; the reference has one image per step), backward = its gradient, both
    from the fused kernels behind api.coord_loss.  The predictions come last (_as_inputs)."""

    @staticmethod
    def forward(ctx, meta, *prediction):
        form, gt_coords, cut_loss = meta
        grads = [torch.empty_like(p) for p in prediction]
        losses = api.coord_loss(form([p.detach() for p in prediction]), gt_coords, cut_loss, outGradients=form(grads))
        ctx.save_for_backward(*grads)
        ctx.batch = len(losses)
        return prediction[0].new_tensor(sum(losses) / len(losses))

    @staticmethod
    def backward(ctx, grad_out):
        return (None,) + tuple(g * (grad_out / ctx.batch) for g in ctx.saved_tensors)


def coord_loss(prediction, gt_coords, cut_loss=100.0):
    """Drop-in for the loss block of init_expert.py: `prediction, gt_coords = util.assert_size(...)` through the robust loss
    (:114-130) become `robust_loss = coord_loss(prediction, gt_coords, opt.cutloss)`, followed by `robust_loss.backward()`.
    prediction [B,3,Hp,Wp] (CUDA), gt_coords [B,3,Hg,Wg], at most 1 apart in H and W; or both lists or tuples of B
    [3,H_b,W_b] tensors of different sizes."""
    inputs, form = _as_inputs(prediction)
    return CoordLoss.apply((form, gt_coords, cut_loss), *inputs)


def _batch_mean(losses):
    """sum(losses) / len(losses) of ReprojLoss / CoordLoss taken on the device: the float64 losses added left to right, then
    one float64 division (by a tensor: torch multiplies by the reciprocal of a Python divisor), rounded to float32 as
    new_tensor rounds it.  No host synchronisation."""
    total = losses[0]
    for b in range(1, losses.shape[0]):
        total = total + losses[b]
    return (total / torch.full((), float(losses.shape[0]), dtype=torch.float64, device=losses.device)).float()


class ReprojLossAsync(torch.autograd.Function):
    """ReprojLoss on api.reproj_loss_async: no host synchronisation in the forward or the backward, so the node, and
    loss.backward() through it, can be captured in a CUDA graph.  The predictions come last (_as_inputs)."""

    @staticmethod
    def forward(ctx, meta, *prediction):
        form, gt_poses, shifts, cameras, cut_loss, sub_sampling, max_reproj, min_depth, status = meta
        grads = [torch.empty_like(p) for p in prediction]
        B = len(prediction) if form is list else prediction[0].shape[0]
        dev = prediction[0].device
        losses = torch.empty(B, dtype=torch.float64, device=dev)
        if status is None:
            status = torch.empty(B, dtype=torch.int32, device=dev)
        api.reproj_loss_async(form([p.detach() for p in prediction]), gt_poses, shifts, cameras, cut_loss, sub_sampling, losses,
                              status, outGradients=form(grads), maxReproj=max_reproj, minDepth=min_depth)
        ctx.save_for_backward(*grads)
        ctx.batch = B
        return _batch_mean(losses)

    @staticmethod
    def backward(ctx, grad_out):
        return (None,) + tuple(g * (grad_out / ctx.batch) for g in ctx.saved_tensors)


def reproj_loss_async(prediction, gt_poses, shifts, cameras, cut_loss, sub_sampling=8, max_reproj=100.0, min_depth=0.1,
                      status=None):
    """reproj_loss for training steps captured in a CUDA graph (ref_expert.py as one graph): CUDA tensors only, prediction
    [B,3,H,W] or a list / tuple of B [3,H_b,W_b] tensors, gt_poses float32 [B,4,4] camera->world, shifts int32 [B,2] (padX,
    padY), cameras float32 [B,3] (focal length, ppointX, ppointY), all read on the device at replay time.  The loss (the
    batch mean, float32) and the gradients are bitwise those of reproj_loss.  status: an int32 CUDA tensor [B] that receives
    the per-image status (1 = a singular ground truth: that loss is NaN, its gradient zero); None keeps it internal.  Call
    api.reserve_loss_async with the largest batch and map before the first capture."""
    inputs, form = _as_inputs(prediction)
    meta = (form, gt_poses, shifts, cameras, cut_loss, sub_sampling, max_reproj, min_depth, status)
    return ReprojLossAsync.apply(meta, *inputs)


class CoordLossAsync(torch.autograd.Function):
    """CoordLoss on api.coord_loss_async: no host synchronisation in the forward or the backward, so the node, and
    loss.backward() through it, can be captured in a CUDA graph.  The predictions come last (_as_inputs)."""

    @staticmethod
    def forward(ctx, meta, *prediction):
        form, gt_coords, cut_loss, counts = meta
        grads = [torch.empty_like(p) for p in prediction]
        B = len(prediction) if form is list else prediction[0].shape[0]
        losses = torch.empty(B, dtype=torch.float64, device=prediction[0].device)
        api.coord_loss_async(form([p.detach() for p in prediction]), gt_coords, cut_loss, losses, outGradients=form(grads),
                             outCounts=counts)
        ctx.save_for_backward(*grads)
        ctx.batch = B
        return _batch_mean(losses)

    @staticmethod
    def backward(ctx, grad_out):
        return (None,) + tuple(g * (grad_out / ctx.batch) for g in ctx.saved_tensors)


def coord_loss_async(prediction, gt_coords, cut_loss=100.0, counts=None):
    """coord_loss for training steps captured in a CUDA graph (init_expert.py as one graph): CUDA tensors only, prediction
    [B,3,Hp,Wp] and gt_coords [B,3,Hg,Wg], or both lists / tuples of B [3,H_b,W_b] tensors, read on the device at replay
    time.  The loss (the batch mean, float32) and the gradients are bitwise those of coord_loss.  counts: an int64 CUDA
    tensor [B] that receives the valid cells per image, or None.  Call api.reserve_loss_async with the largest batch and
    map before the first capture."""
    inputs, form = _as_inputs(prediction)
    return CoordLossAsync.apply((form, gt_coords, cut_loss, counts), *inputs)


# ------------------------------------------------------------------------------------------------
# The hypotheses as an autograd node: any pose loss written in torch
# ------------------------------------------------------------------------------------------------
class EsacHypotheses(torch.autograd.Function):
    """Scores and poses of the hypotheses of an esac.backward call, differentiable with respect to the scene coordinates."""

    @staticmethod
    def forward(ctx, scene_coordinates, hyp_assignment, *params):
        scores, poses, contributing, tape = api.hypotheses_forward(scene_coordinates.detach(), hyp_assignment, *params)
        # the coordinates are passed to the backward again; autograd's version counter catches an in-place change
        ctx.save_for_backward(scene_coordinates, tape)
        ctx.mark_non_differentiable(contributing)
        ctx.set_materialize_grads(False)
        ctx.n_params = len(params)
        return scores, poses, contributing

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_scores, grad_poses, _grad_contributing):
        coords, tape = ctx.saved_tensors
        grads = torch.zeros_like(coords)
        api.hypotheses_backward(tape, coords, grads, grad_scores, grad_poses)
        return (grads, None) + (None,) * ctx.n_params


def esac_hypotheses(scene_coordinates, hyp_assignment, shift_x, shift_y, focal_length, ppoint_x, ppoint_y,
                    inlier_threshold, inlier_alpha, inlier_beta, max_reproj, sub_sampling):
    """The hypotheses of esac.backward as a differentiable function, so that a trainer can write its own pose loss in torch.

    scene_coordinates [E,3,H,W] float32 (CPU or CUDA), hyp_assignment [M] int64; the other arguments are esac.forward's.
    Returns, on the coordinates' device:
      scores        float64 [M]    the soft-inlier scores (softmax(scores) are the hypothesis probabilities),
      poses         float64 [M,6]  scene pose (rvec, tvec) per hypothesis: refined where p >= PROB_THRESH, else initial,
      contributing  bool [M]       p >= PROB_THRESH.
    It draws what an esac.backward call at the same point of the context's call sequence would draw, so with the option
    fixed_seed and the same seed its hypotheses, scores and refined poses are bitwise those of esac.backward.

    The backward gives d L / d scene_coordinates from the gradients of `scores` and `poses` (either may be absent, which
    counts as zero).  As in the reference, only contributing hypotheses are differentiated: gradients reaching hypotheses
    with p < PROB_THRESH are ignored, and a refined pose is differentiated through its refinement's linearisation, with the
    reference's > 10 clamps.  The node is once differentiable.  With
        L = (softmax(scores) * reference_pose_loss(poses, gt_pose, w_rot, w_trans, cut)).sum()
    L and its gradient are those of esac.backward / esac_loss."""
    return EsacHypotheses.apply(scene_coordinates, hyp_assignment, shift_x, shift_y, focal_length, ppoint_x, ppoint_y,
                                inlier_threshold, inlier_alpha, inlier_beta, max_reproj, sub_sampling)


class EsacHypothesesBatch(torch.autograd.Function):
    """EsacHypotheses over a batch of images (api.hypotheses_forward_batch).  The maps come last (_as_inputs); `meta` holds
    the non-differentiable arguments."""

    @staticmethod
    def forward(ctx, meta, *scene_coordinates):
        form, hyp_assignment, params = meta
        scores, poses, contributing, tapes = api.hypotheses_forward_batch(form([c.detach() for c in scene_coordinates]),
                                                                          hyp_assignment, *params)
        # the coordinates are passed to the backward again; autograd's version counter catches an in-place change
        ctx.save_for_backward(*scene_coordinates, *tapes)
        ctx.mark_non_differentiable(contributing)
        ctx.set_materialize_grads(False)
        ctx.form, ctx.n = form, len(scene_coordinates)
        return scores, poses, contributing

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_scores, grad_poses, _grad_contributing):
        saved = ctx.saved_tensors
        coords, tapes = saved[:ctx.n], list(saved[ctx.n:])
        grads = [torch.zeros_like(c) for c in coords]
        api.hypotheses_backward_batch(tapes, ctx.form(coords), ctx.form(grads), grad_scores, grad_poses)
        return (None,) + tuple(grads)


def esac_hypotheses_batch(scene_coordinates, hyp_assignment, shift_x, shift_y, focal_length, ppoint_x, ppoint_y,
                          inlier_threshold, inlier_alpha, inlier_beta, max_reproj, sub_sampling):
    """esac_hypotheses over a batch of images, each with its own shift and camera: scene_coordinates [B,E,3,H,W] float32 or
    a list / tuple of B [E,3,H_b,W_b] tensors of different sizes (every element then receives its own gradient),
    hyp_assignment [B,M] int64; shift_x, shift_y, focal_length, ppoint_x, ppoint_y a number or B values.  Returns scores
    float64 [B,M], poses float64 [B,M,6] and contributing bool [B,M]; row b is what the b-th of B consecutive esac_hypotheses
    calls would return, and the backward gives each image the gradient esac_hypotheses would.  The images run on the worker
    streams of api.backward_batch.  With
        L = (softmax(scores, 1) * reference_pose_loss(poses, gt_poses, w_rot, w_trans, cut)).sum(1)
    L and its gradient are those of esac_loss_batch."""
    params = (shift_x, shift_y, focal_length, ppoint_x, ppoint_y, inlier_threshold, inlier_alpha, inlier_beta, max_reproj,
              sub_sampling)
    inputs, form = _as_inputs(scene_coordinates)
    return EsacHypothesesBatch.apply((form, hyp_assignment, params), *inputs)


class EsacHypothesesAsync(torch.autograd.Function):
    """EsacHypotheses / EsacHypothesesBatch on api.hypotheses_forward_async / hypotheses_backward_async: no host
    synchronisation in the forward or the backward, so a training step with a pose loss of the caller's own can be
    captured in a CUDA graph.  The tapes are allocated by torch in the forward (inside a capture: in the graph's pool) and
    live on the autograd context.  `meta` holds the non-differentiable arguments."""

    @staticmethod
    def forward(ctx, meta, scene_coordinates):
        hyp_assignment, shifts, cameras, params, status = meta
        lead = tuple(scene_coordinates.shape[:-4])
        E, _, H, W = (int(v) for v in scene_coordinates.shape[-4:])
        M = int(hyp_assignment.shape[-1])
        B = lead[0] if lead else 1
        dev = scene_coordinates.device
        tapes = torch.empty(B * api.hypotheses_tape_stride(E, H, W, M), dtype=torch.uint8, device=dev)
        scores = torch.empty(lead + (M,), dtype=torch.float64, device=dev)
        poses = torch.empty(lead + (M, 6), dtype=torch.float64, device=dev)
        contributing = torch.empty(lead + (M,), dtype=torch.bool, device=dev)
        if status is None:
            status = torch.empty(lead, dtype=torch.int32, device=dev)
        api.hypotheses_forward_async(scene_coordinates.detach(), hyp_assignment, shifts, cameras, *params, tapes, scores, poses,
                                     contributing, status)
        # the coordinates are passed to the backward again; autograd's version counter catches an in-place change
        ctx.save_for_backward(scene_coordinates, tapes)
        ctx.mark_non_differentiable(contributing)
        ctx.set_materialize_grads(False)
        ctx.M = M
        return scores, poses, contributing

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_scores, grad_poses, _grad_contributing):
        coords, tapes = ctx.saved_tensors
        grads = torch.zeros_like(coords)
        api.hypotheses_backward_async(tapes, coords, grads, ctx.M,
                                      grad_scores.contiguous() if grad_scores is not None else None,
                                      grad_poses.contiguous() if grad_poses is not None else None)
        return None, grads


def esac_hypotheses_async(scene_coordinates, hyp_assignment, shifts, cameras, tau, alpha, beta, max_reproj, sub, status=None):
    """esac_hypotheses (one image: scene_coordinates [E,3,H,W], hyp_assignment [M], shifts [2], cameras [3]) or
    esac_hypotheses_batch on a stacked batch (scene_coordinates [B,E,3,H,W], hyp_assignment [B,M], shifts [B,2] int32,
    cameras [B,3] = focal length, ppointX, ppointY) on the stream-ordered node, for training steps captured in a CUDA
    graph: CUDA tensors only, the shifts and cameras read on the device at replay time.  Returns scores float64 [B,M],
    poses float64 [B,M,6] and contributing bool [B,M] (or [M], [M,6], [M] for one image), bitwise those of esac_hypotheses
    for the same draws: image b of the j-th call draws what the (j*B + b)-th esac_hypotheses call draws.  Once
    differentiable; an absent upstream gradient counts as zero.  status: an int32 CUDA tensor [B] (or []) that receives the
    forward's per-image status (1 = a bad expert index: scores and poses NaN, no gradient); None keeps it internal.  Call
    api.reserve_backward_async with the largest shape before the first capture."""
    meta = (hyp_assignment, shifts, cameras, (tau, alpha, beta, max_reproj, sub), status)
    return EsacHypothesesAsync.apply(meta, scene_coordinates)


class ReferencePoseLossAsync(torch.autograd.Function):
    @staticmethod
    def forward(ctx, poses, gt_pose, w_rot, w_trans, cut):
        losses, dloss = api.pose_loss_async(poses.detach(), gt_pose, w_rot, w_trans, cut)
        ctx.save_for_backward(dloss)
        return losses

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_losses):
        (dloss,) = ctx.saved_tensors
        return grad_losses[..., None] * dloss, None, None, None, None


def reference_pose_loss_async(poses, gt_pose, w_rot, w_trans, cut):
    """reference_pose_loss on api.pose_loss_async: CUDA tensors only, no host synchronisation, so it can be captured in a
    CUDA graph.  poses [M,6] / [B,M,6] float64 against gt_pose [4,4] / [B,4,4] float32; the same values and gradients."""
    return ReferencePoseLossAsync.apply(poses, gt_pose, w_rot, w_trans, cut)


class ReferencePoseLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, poses, gt_pose, w_rot, w_trans, cut):
        losses, dloss = api.pose_loss(poses.detach(), gt_pose, w_rot, w_trans, cut)
        ctx.save_for_backward(dloss)
        return losses

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_losses):
        (dloss,) = ctx.saved_tensors
        return grad_losses.to(dloss.device)[..., None] * dloss, None, None, None, None


def reference_pose_loss(poses, gt_pose, w_rot, w_trans, cut):
    """The reference's pose loss (esac_loss.h `loss`) of scene poses [M,6] = (rvec, tvec) float64 against a float32 [4,4]
    camera->world ground truth: wRot * angle(deg) + wTrans * |t_est - t_gt|, above `cut` sqrt(cut * l), at most 1e7.
    Its gradient is the reference's dLoss, bug for bug: above the cut it is scaled as the derivative of sqrt(l) (not of
    sqrt(cut * l)), the angle uses CV_PI where the loss uses 3.1415926, and it is zero on NaN, on errors below 1e-8 and at
    the 1e7 cap.  Both come from the device functions esac.backward uses.  Returns float64 [M].  Poses [B,M,6] against
    ground truths [B,4,4] give [B,M] in one launch, row b bitwise what [M,6] against gt_pose[b] gives."""
    return ReferencePoseLoss.apply(poses, gt_pose, w_rot, w_trans, cut)


def _skew(r):
    z = torch.zeros_like(r[..., 0])
    return torch.stack([torch.stack([z, -r[..., 2], r[..., 1]], -1),
                        torch.stack([r[..., 2], z, -r[..., 0]], -1),
                        torch.stack([-r[..., 1], r[..., 0], z], -1)], -2)


def pose_to_transform(poses):
    """pose2trans (esac_util.h) in differentiable torch: scene poses [M,6] = (rvec, tvec), world->camera, to camera->world
    transforms [M,4,4] = [R^T | -R^T t].  R = I + a K + b K^2 with K = [r]x, a = sin(th)/th, b = (1 - cos(th))/th^2; below
    th = 1e-3 a and b are their Taylor series in th^2, so th = 0 has a finite gradient."""
    r, t = poses[..., :3], poses[..., 3:]
    th2 = (r * r).sum(-1)
    small = th2 < 1e-6
    th2_safe = torch.where(small, torch.ones_like(th2), th2)
    th = torch.sqrt(th2_safe)
    a = torch.where(small, 1 - th2 / 6 + th2 * th2 / 120, torch.sin(th) / th)
    b = torch.where(small, 0.5 - th2 / 24 + th2 * th2 / 720, (1 - torch.cos(th)) / th2_safe)
    K = _skew(r)
    eye = torch.eye(3, dtype=poses.dtype, device=poses.device).expand(K.shape)
    R = eye + a[..., None, None] * K + b[..., None, None] * (K @ K)
    Rt = R.transpose(-1, -2)
    bottom = torch.cat([torch.zeros_like(t[..., None, :]), torch.ones_like(t[..., None, :1])], -1)
    return torch.cat([torch.cat([Rt, -(Rt @ t[..., None])], -1), bottom], -2)
