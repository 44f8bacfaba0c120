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
