"""Oracle for the expert-refinement reprojection loss (SURVEY 8f rank 4).  TEST INFRASTRUCTURE ONLY.

A restatement of ref_expert.py:84-89 (target grid) and :103-148 (projection, clamps, robust loss) as one function of
(prediction, gt_pose, focal length, pad, cut, clamps) built from the same torch ops in the same order, so that torch's own
autograd provides the reference gradient.  It runs on the CPU in float32 (what the original computes in, on its GPU) or,
with dtype=torch.float64, as the higher-precision yardstick that the tolerance of the fp32 comparison is judged by.

Parity status: the reference ships no fixture for this loss ("parity unpinned" in the sense of the task contract); the
restatement is the reference's own op sequence, and tests/test_oracle.py pins it against an independent closed-form
gradient in float64.

Only tests/ may import this module; the product path (esac_b200/csrc/reproj.cu) never does.
"""
from __future__ import annotations

import torch


def reproj_errors(prediction: torch.Tensor, gt_pose: torch.Tensor, focallength: float, pad_x: float, pad_y: float,
                  subsample: int = 8, image_w: float | None = None, image_h: float | None = None,
                  dtype=torch.float32, max_reproj: float = 100.0, min_depth: float = 0.1) -> torch.Tensor:
    """Per-cell reprojection error clamped to [0, max_reproj] px, flat [h*w] (ref_expert.py:103-142, where
    max_reproj = 100 and the depth clamp min_depth = 0.1).
    prediction [1 or none,3,h,w] scene coordinates (requires_grad allowed), gt_pose [4,4] camera->world.
    image_w/h: size of the (padded) input image; default sub*w, sub*h -> principal point at the map centre
    (ref_expert.py:118-119)."""
    if prediction.dim() == 3:
        prediction = prediction.unsqueeze(0)
    prediction = prediction.to(dtype)
    h, w = prediction.size(2), prediction.size(3)
    # ref_expert.py:84-89: target pixel of every cell
    xs = torch.arange(w, dtype=dtype) * subsample + subsample / 2
    ys = torch.arange(h, dtype=dtype) * subsample + subsample / 2
    grid = torch.stack((xs.unsqueeze(0).expand(h, w), ys.unsqueeze(1).expand(h, w)))
    grid = grid.clone().view(2, -1)
    grid[0] -= pad_x                                     # :110
    grid[1] -= pad_y                                     # :111
    cam_mat = torch.eye(3, dtype=dtype)                  # :115-119
    cam_mat[0, 0] = focallength
    cam_mat[1, 1] = focallength
    cam_mat[0, 2] = (image_w if image_w is not None else w * subsample) / 2
    cam_mat[1, 2] = (image_h if image_h is not None else h * subsample) / 2
    ones = torch.ones((prediction.size(0), 1, h, w), dtype=dtype)   # :123-125
    pred = torch.cat((prediction, ones), 1)
    pose = gt_pose.to(dtype).inverse()[0:3, :]           # :127
    pred = pred[0].view(4, -1)                           # :131
    eye = torch.mm(pose, pred)                           # :132
    px = torch.mm(cam_mat, eye)                          # :135
    px[2].clamp_(min=min_depth)                          # :136
    px = px[0:2] / px[2]                                 # :137
    px = px - grid                                       # :140
    px = px.norm(2, 0)                                   # :141
    return px.clamp(0, max_reproj)                       # :142


def reproj_loss(prediction: torch.Tensor, gt_pose: torch.Tensor, focallength: float, pad_x: float, pad_y: float,
                cutloss: float, subsample: int = 8, image_w: float | None = None, image_h: float | None = None,
                dtype=torch.float32, max_reproj: float = 100.0, min_depth: float = 0.1) -> torch.Tensor:
    """The robust loss of ref_expert.py:144-148 over reproj_errors()."""
    px = reproj_errors(prediction, gt_pose, focallength, pad_x, pad_y, subsample, image_w, image_h, dtype, max_reproj,
                       min_depth)
    loss_l1 = px[px <= cutloss]                          # :144
    loss_sqrt = px[px > cutloss]                         # :145
    loss_sqrt = torch.sqrt(cutloss * loss_sqrt)          # :146
    return (loss_l1.sum() + loss_sqrt.sum()) / float(px.size(0))   # :148


def reproj_loss_and_grad(prediction, gt_pose, focallength, pad_x, pad_y, cutloss, subsample=8, image_w=None, image_h=None,
                         dtype=torch.float32, max_reproj=100.0, min_depth=0.1):
    """(loss, d loss / d prediction [3,h,w]) through torch autograd, as `robust_loss.backward()` (ref_expert.py:150)."""
    p = torch.as_tensor(prediction).detach().clone().to(dtype).requires_grad_(True)
    loss = reproj_loss(p, torch.as_tensor(gt_pose), focallength, pad_x, pad_y, cutloss, subsample, image_w, image_h, dtype,
                       max_reproj, min_depth)
    loss.backward()
    g = p.grad
    return float(loss.detach()), (g[0] if g.dim() == 4 else g)
