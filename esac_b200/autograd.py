"""torch.autograd wrapper around esac.backward (SURVEY.md section 8f, rank 1).

The reference's trainer calls the extension, then builds the gating gradient by hand and feeds both gradients to
torch.autograd.backward (train_esac.py:151-180).  EsacLoss packages exactly that: its forward returns the expected
pose loss, its backward hands d loss / d sceneCoordinates (from the extension) and the REINFORCE-style gating
gradient to autograd -- loss * histogram(e_hyps) in the default mode (train_esac.py:174-176), or, in the trainer's
`expertselection` mode (one expert drawn and expanded to all hypotheses, train_esac.py:133-135), `loss` at the drawn
expert only (train_esac.py:171-173).  CUDA tensors stay on the device."""
from __future__ import annotations

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


class EsacLossBatch(torch.autograd.Function):
    """EsacLoss over a batch of images, on api.backward_batch: forward returns the B expected pose losses, backward hands
    d loss_b / d scene_coordinates[b] and row b of the gating gradient -- loss_b * histogram(e_hyps[b]), or loss_b at the
    drawn expert in expert-selection mode -- to autograd, each computed exactly as EsacLoss computes it for one image."""

    @staticmethod
    def forward(ctx, scene_coordinates, gating_log_probs, hyp_assignment, gt_poses, w_rot, w_trans, loss_cut, shift_x,
                shift_y, focal_length, ppoint_x, ppoint_y, inlier_threshold, inlier_alpha, inlier_beta, max_reproj,
                sub_sampling, expert_selection=None):
        grads = torch.zeros_like(scene_coordinates)
        losses = api.backward_batch(scene_coordinates.detach(), grads, hyp_assignment, gt_poses, w_rot, w_trans, loss_cut,
                                    shift_x, shift_y, focal_length, ppoint_x, ppoint_y, inlier_threshold, inlier_alpha,
                                    inlier_beta, max_reproj, sub_sampling)
        E = scene_coordinates.shape[1]
        if expert_selection is None:
            # [B,1].expand(B,M): a stride-0 row per image, the batched form of expert.expand(M)
            expert_selection = hyp_assignment.dim() == 2 and hyp_assignment.shape[1] > 1 and hyp_assignment.stride(1) == 0
        rows = []
        for b, loss in enumerate(losses):
            if expert_selection:
                g = torch.zeros(E)
                g[int(hyp_assignment[b, 0])] = loss                                      # train_esac.py:171-173
            else:
                hist = torch.histc(hyp_assignment[b].float().cpu(), bins=E, min=0, max=E - 1)   # train_esac.py:140
                g = loss * hist                                                           # train_esac.py:174-176
            rows.append(g)
        g_gating = torch.stack(rows).to(gating_log_probs.device).reshape(gating_log_probs.shape)
        ctx.save_for_backward(grads, g_gating)
        return scene_coordinates.new_tensor(losses)

    @staticmethod
    def backward(ctx, grad_out):
        g_coords, g_gating = ctx.saved_tensors
        B = grad_out.shape[0]
        return (g_coords * grad_out.reshape((B,) + (1,) * (g_coords.dim() - 1)),
                g_gating * grad_out.reshape((B,) + (1,) * (g_gating.dim() - 1))) + (None,) * 16


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


class EsacLossRagged(torch.autograd.Function):
    """EsacLossBatch on a list of B maps [E,3,H_b,W_b] of different sizes (api.backward_batch on a list).  The maps come
    last so that autograd sees every one of them; `meta` holds the non-differentiable arguments."""

    @staticmethod
    def forward(ctx, meta, gating_log_probs, *scene_coordinates):
        hyp_assignment, gt_poses, params, expert_selection = meta
        grads = [torch.zeros_like(c) for c in scene_coordinates]
        losses = api.backward_batch([c.detach() for c in scene_coordinates], grads, hyp_assignment, gt_poses, *params)
        if expert_selection is None:
            expert_selection = hyp_assignment.dim() == 2 and hyp_assignment.shape[1] > 1 and hyp_assignment.stride(1) == 0
        E = scene_coordinates[0].shape[0]
        g_gating = _gating_rows(losses, hyp_assignment, E, expert_selection)
        ctx.save_for_backward(g_gating.to(gating_log_probs.device).reshape(gating_log_probs.shape), *grads)
        return scene_coordinates[0].new_tensor(losses)

    @staticmethod
    def backward(ctx, grad_out):
        g_gating, *g_coords = ctx.saved_tensors
        B = grad_out.shape[0]
        return ((None, g_gating * grad_out.reshape((B,) + (1,) * (g_gating.dim() - 1))) +
                tuple(g * grad_out[b] for b, g in enumerate(g_coords)))


def esac_loss_batch(scene_coordinates, gating_log_probs, hyp_assignment, gt_poses, *params, expert_selection=None):
    """The batched counterpart of esac_loss (one train_esac.py step on B images, each with its own camera):
    scene_coordinates [B,E,3,H,W], gating_log_probs [B,E], hyp_assignment [B,M], gt_poses [B,4,4]; params the positional
    tail of api.backward_batch (wLossRot, wLossTrans, lossCut, shiftX, shiftY, focalLength, ppointX, ppointY,
    inlierThreshold, inlierAlpha, inlierBeta, maxReproj, subSampling), where shifts and camera may be per image.
    Returns the B expected losses; image b draws the minimal sets of the b-th of B consecutive esac_loss calls.
    expert_selection as for esac_loss, decided for the whole batch (None: a stride-0 [B,1].expand(B,M) assignment).
    scene_coordinates may also be a list or tuple of B [E,3,H_b,W_b] tensors of different sizes; every element then
    receives its own gradient."""
    if isinstance(scene_coordinates, (list, tuple)):
        return EsacLossRagged.apply((hyp_assignment, gt_poses, params, expert_selection), gating_log_probs, *scene_coordinates)
    return EsacLossBatch.apply(scene_coordinates, gating_log_probs, hyp_assignment, gt_poses, *params, expert_selection)


class ReprojLoss(torch.autograd.Function):
    """ref_expert.py:103-150 as one autograd node: forward = the robust reprojection loss of a batch of predictions
    (mean over the batch of the per-image losses; the reference has one image per step), backward = its gradient, both
    from the single fused kernel behind api.reproj_loss."""

    @staticmethod
    def forward(ctx, prediction, gt_poses, focal_length, pad_x, pad_y, cut_loss, sub_sampling, ppoint_x, ppoint_y):
        grads = torch.empty_like(prediction)
        losses = api.reproj_loss(prediction.detach(), gt_poses, focal_length, pad_x, pad_y, cut_loss, sub_sampling, ppoint_x,
                                 ppoint_y, outGradients=grads)
        ctx.save_for_backward(grads)
        ctx.batch = len(losses)
        return prediction.new_tensor(sum(losses) / len(losses))

    @staticmethod
    def backward(ctx, grad_out):
        (grads,) = ctx.saved_tensors
        return (grads * (grad_out / ctx.batch),) + (None,) * 8


class ReprojLossRagged(torch.autograd.Function):
    """ReprojLoss on a list of B predictions [3,H_b,W_b]: the batch mean of the per-image losses, a gradient per element."""

    @staticmethod
    def forward(ctx, meta, *prediction):
        grads = [torch.empty_like(p) for p in prediction]
        losses = api.reproj_loss([p.detach() for p in prediction], *meta, outGradients=grads)
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
    if isinstance(prediction, (list, tuple)):
        meta = (gt_poses, focal_length, pad_x, pad_y, cut_loss, sub_sampling, ppoint_x, ppoint_y)
        return ReprojLossRagged.apply(meta, *prediction)
    return ReprojLoss.apply(prediction, gt_poses, focal_length, pad_x, pad_y, cut_loss, sub_sampling, ppoint_x, ppoint_y)


class CoordLoss(torch.autograd.Function):
    """init_expert.py:106-132 as one autograd node: forward = the robust scene-coordinate loss of a batch of predictions
    (mean over the batch of the per-image losses; the reference has one image per step), backward = its gradient, both
    from the fused kernels behind api.coord_loss."""

    @staticmethod
    def forward(ctx, prediction, gt_coords, cut_loss):
        grads = torch.empty_like(prediction)
        losses = api.coord_loss(prediction.detach(), gt_coords, cut_loss, outGradients=grads)
        ctx.save_for_backward(grads)
        ctx.batch = len(losses)
        return prediction.new_tensor(sum(losses) / len(losses))

    @staticmethod
    def backward(ctx, grad_out):
        (grads,) = ctx.saved_tensors
        return (grads * (grad_out / ctx.batch),) + (None,) * 2


class CoordLossRagged(torch.autograd.Function):
    """CoordLoss on lists of B predictions [3,Hp_b,Wp_b] and ground truths: the batch mean, a gradient per prediction."""

    @staticmethod
    def forward(ctx, meta, *prediction):
        gt_coords, cut_loss = meta
        grads = [torch.empty_like(p) for p in prediction]
        losses = api.coord_loss([p.detach() for p in prediction], gt_coords, cut_loss, outGradients=grads)
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
    if isinstance(prediction, (list, tuple)):
        return CoordLossRagged.apply((gt_coords, cut_loss), *prediction)
    return CoordLoss.apply(prediction, gt_coords, cut_loss)


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
    """EsacHypotheses over a batch of images of one shape (api.hypotheses_forward_batch on [B,E,3,H,W] maps)."""

    @staticmethod
    def forward(ctx, scene_coordinates, hyp_assignment, *params):
        scores, poses, contributing, tapes = api.hypotheses_forward_batch(scene_coordinates.detach(), hyp_assignment, *params)
        ctx.save_for_backward(scene_coordinates, *tapes)
        ctx.mark_non_differentiable(contributing)
        ctx.set_materialize_grads(False)
        ctx.n_params = len(params)
        return scores, poses, contributing

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_scores, grad_poses, _grad_contributing):
        coords, *tapes = ctx.saved_tensors
        grads = torch.zeros_like(coords)
        api.hypotheses_backward_batch(tapes, coords, grads, grad_scores, grad_poses)
        return (grads, None) + (None,) * ctx.n_params


class EsacHypothesesRagged(torch.autograd.Function):
    """EsacHypothesesBatch on a list of B maps [E,3,H_b,W_b].  The maps come last so that autograd sees every one of them;
    `meta` holds the non-differentiable arguments."""

    @staticmethod
    def forward(ctx, meta, *scene_coordinates):
        hyp_assignment, params = meta
        scores, poses, contributing, tapes = api.hypotheses_forward_batch([c.detach() for c in scene_coordinates],
                                                                          hyp_assignment, *params)
        ctx.save_for_backward(*scene_coordinates, *tapes)
        ctx.mark_non_differentiable(contributing)
        ctx.set_materialize_grads(False)
        ctx.B = len(scene_coordinates)
        return scores, poses, contributing

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_scores, grad_poses, _grad_contributing):
        saved = ctx.saved_tensors
        coords, tapes = list(saved[:ctx.B]), list(saved[ctx.B:])
        grads = [torch.zeros_like(c) for c in coords]
        api.hypotheses_backward_batch(tapes, coords, grads, grad_scores, grad_poses)
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
    if isinstance(scene_coordinates, (list, tuple)):
        return EsacHypothesesRagged.apply((hyp_assignment, params), *scene_coordinates)
    return EsacHypothesesBatch.apply(scene_coordinates, hyp_assignment, *params)


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
