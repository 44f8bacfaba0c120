"""The scene-coordinate loss of the expert initialisation stage without a GPU: the oracle's known answers, and the argument
checks of api.coord_loss, which run before any CUDA context exists."""
import numpy as np
import pytest
import torch

from oracle.coord_loss_oracle import coord_loss_and_grad


def known_answer_maps():
    """Four valid cells at cut = 100 -- d = 0, a NaN prediction, n = 100 exactly, n = 400 -- and one invalid cell.
    Loss (0 + 0 + 100 + sqrt(100 * 400)) / 4 = 75; gradients on z 0, NaN, 1/4, 0.5 * sqrt(100 / 400) / 4."""
    gt = np.zeros((3, 1, 5), np.float32)
    pred = np.zeros((3, 1, 5), np.float32)
    gt[:, 0, 0] = pred[:, 0, 0] = [1.0, 2.0, 3.0]
    gt[:, 0, 1] = [1.0, 2.0, 3.0]
    pred[:, 0, 1] = np.nan
    gt[2, 0, 2], pred[2, 0, 2] = 5.0, 105.0
    gt[2, 0, 3], pred[2, 0, 3] = 5.0, 405.0
    pred[:, 0, 4] = 7.0
    return pred, gt


KNOWN_LOSS = 75.0
KNOWN_GZ = [0.0, np.nan, 0.25, 0.0625, 0.0]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_oracle_known_answer(dtype):
    pred, gt = known_answer_maps()
    loss, g = coord_loss_and_grad(torch.from_numpy(pred), torch.from_numpy(gt), 100.0, dtype)
    assert loss == KNOWN_LOSS
    np.testing.assert_array_equal(g[2, 0].numpy(), np.array(KNOWN_GZ))
    assert torch.isnan(g[:, 0, 1]).all()
    assert (g[:2, 0, [0, 2, 3, 4]] == 0).all()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_oracle_image_without_valid_cells(dtype):
    pred = torch.randn(3, 6, 7)
    loss, g = coord_loss_and_grad(pred, torch.zeros(3, 6, 7), 100.0, dtype)
    assert np.isnan(loss)
    assert (g == 0).all()


def test_oracle_mask_counts_subnormal_and_nan_ground_truth():
    """gt.abs().sum(0) != 0: one nonzero component suffices, a subnormal one too, and NaN is valid."""
    gt = torch.zeros(3, 1, 4)
    gt[0, 0, 0] = 1e-40          # subnormal x only
    gt[1, 0, 1] = 2.0            # y only
    gt[2, 0, 2] = float("nan")   # NaN z
    pred = torch.ones(3, 1, 4)
    loss, g = coord_loss_and_grad(pred, gt, 100.0, torch.float32)
    assert loss == pytest.approx((np.sqrt(3.0) + np.sqrt(3.0)) / 3, rel=1e-6)
    assert (g[:, 0, 3] == 0).all() and torch.isnan(g[:, 0, 2]).all() and (g[:, 0, :2] != 0).all()


def test_oracle_crop_and_size_mismatch():
    from oracle.coord_loss_oracle import coord_loss
    pred = torch.randn(3, 61, 81)
    gt = torch.randn(3, 60, 80)
    loss, g = coord_loss_and_grad(pred, gt, 100.0, torch.float64)
    assert (g[:, 60, :] == 0).all() and (g[:, :, 80] == 0).all()
    assert loss == pytest.approx(float(coord_loss(pred[:, :60, :80], gt, 100.0, torch.float64)), rel=1e-15)
    with pytest.raises(RuntimeError, match="size mismatch"):
        coord_loss(torch.randn(3, 62, 80), gt, 100.0)


P = np.zeros((2, 3, 6, 8), np.float32)
G = np.ones((2, 3, 6, 8), np.float32)
BAD = [
    ("dtype", (P.astype(np.float64), G), {}, "expected scalar type Float but found Double"),
    ("gt dtype", (P, G.astype(np.float64)), {}, "expected scalar type Float but found Double"),
    ("rank", (P[0], G[0]), {}, "expected 4 dims"),
    ("gt rank", (P, G[:, :, :, :, None]), {}, "expected 4 dims"),
    ("channels", (P[:, :2], G[:, :2]), {}, "shapes must be"),
    ("gt channels", (P, np.ones((2, 4, 6, 8), np.float32)), {}, "shapes must be"),
    ("batch", (P, G[:1]), {}, "shapes must be"),
    ("height", (P, np.ones((2, 3, 8, 8), np.float32)), {}, "size mismatch"),
    ("width", (np.zeros((2, 3, 6, 10), np.float32), G), {}, "size mismatch"),
    ("grad dtype", (P, G), {"outGradients": np.zeros_like(P, np.float64)}, "expected scalar type Float but found Double"),
    ("grad shape", (P, G), {"outGradients": np.zeros((2, 3, 6, 9), np.float32)}, "shape of prediction"),
]


@pytest.mark.parametrize("args,kw,msg", [b[1:] for b in BAD], ids=[b[0] for b in BAD])
def test_coord_loss_rejects_bad_arguments_before_any_context(args, kw, msg):
    import esac_b200.api as api
    with pytest.raises(RuntimeError, match=msg):
        api.coord_loss(*args, **kw)


def test_coord_loss_has_no_cpu_path(lib):
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    import esac_b200.api as api
    with pytest.raises(RuntimeError, match="no CPU path"):
        api.coord_loss(P, G)
    # a difference of one cell in either direction is accepted, so the call reaches the (missing) device
    with pytest.raises(RuntimeError, match="no CPU path"):
        api.coord_loss(torch.zeros(1, 3, 61, 81), torch.ones(1, 3, 60, 80), 100.0, outGradients=torch.zeros(1, 3, 61, 81))
