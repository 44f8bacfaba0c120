"""Argument errors of the 16-bit losses (api.reproj_loss_amp, coord_loss_amp and their _async forms): raised before any
context exists, so they run without a GPU (the tensors here are CPU tensors; the dtype, shape and gradScale checks come
before the device check)."""
import pytest
import torch

import esac_b200.api as api

B, H, W = 2, 6, 8
F16 = torch.float16


def _call(name, dtype=F16, **kw):
    """Entry point `name` on default arguments of `dtype`, with the arguments in kw replaced."""
    pred = torch.zeros(B, 3, H, W, dtype=dtype)
    a = dict(prediction=pred, outGradients=torch.zeros_like(pred), gradScale=None)
    if name.startswith("reproj"):
        a.update(gtPoses=torch.eye(4).repeat(B, 1, 1), shifts=torch.zeros(B, 2, dtype=torch.int32), cameras=torch.ones(B, 3),
                 outLosses=torch.zeros(B, dtype=torch.float64), outStatus=torch.zeros(B, dtype=torch.int32))
    else:
        a.update(gtCoords=torch.zeros(B, 3, H, W), outLosses=torch.zeros(B, dtype=torch.float64),
                 outCounts=torch.zeros(B, dtype=torch.int64))
    a.update(kw)
    if name == "reproj_loss_amp":
        api.reproj_loss_amp(a["prediction"], a["gtPoses"], 500.0, 0, 0, 10.0, outGradients=a["outGradients"],
                            gradScale=a["gradScale"])
    elif name == "reproj_loss_amp_async":
        api.reproj_loss_amp_async(a["prediction"], a["gtPoses"], a["shifts"], a["cameras"], 10.0, 8, a["outLosses"],
                                  a["outStatus"], outGradients=a["outGradients"], gradScale=a["gradScale"])
    elif name == "coord_loss_amp":
        api.coord_loss_amp(a["prediction"], a["gtCoords"], 10.0, outGradients=a["outGradients"], gradScale=a["gradScale"])
    else:
        api.coord_loss_amp_async(a["prediction"], a["gtCoords"], 10.0, a["outLosses"], outGradients=a["outGradients"],
                                 outCounts=a["outCounts"], gradScale=a["gradScale"])


CALLS = ["reproj_loss_amp", "reproj_loss_amp_async", "coord_loss_amp", "coord_loss_amp_async"]


@pytest.fixture(autouse=True)
def no_context():
    """Every refusal comes before a context is created (earlier tests of a GPU run may have created some)."""
    before = dict(api._contexts)
    yield
    assert api._contexts == before


@pytest.mark.parametrize("name", CALLS)
def test_float32_is_refused(name):
    with pytest.raises(RuntimeError, match=r"expected scalar type Half or BFloat16 but found Float \(prediction\)"):
        _call(name, dtype=torch.float32)
    with pytest.raises(RuntimeError, match=r"expected scalar type Half or BFloat16 but found Double \(prediction\)"):
        _call(name, dtype=torch.float64)


@pytest.mark.parametrize("name", CALLS)
def test_a_list_is_of_one_dtype(name):
    pred = [torch.zeros(3, H, W, dtype=F16), torch.zeros(3, H, W, dtype=torch.bfloat16)]
    extra = {"gtCoords": [torch.zeros(3, H, W)] * 2} if name.startswith("coord") else {}
    with pytest.raises(RuntimeError, match=r"prediction mixes dtypes: prediction\[0\] Half, prediction\[1\] BFloat16"):
        _call(name, prediction=pred, outGradients=None, **extra)
    with pytest.raises(RuntimeError, match=r"expected scalar type Half or BFloat16 but found Float \(prediction\[1\]\)"):
        _call(name, prediction=[pred[0], torch.zeros(3, H, W)], outGradients=None, **extra)


@pytest.mark.parametrize("name", CALLS)
@pytest.mark.parametrize("grad_dtype", [torch.bfloat16, torch.float32])
def test_gradients_have_the_prediction_dtype(name, grad_dtype):
    msg = rf"expected scalar type Half but found {api._TORCH_NAMES[str(grad_dtype)]} \(outGradients\)"
    with pytest.raises(RuntimeError, match=msg):
        _call(name, outGradients=torch.zeros(B, 3, H, W, dtype=grad_dtype))
    # a bfloat16 prediction wants bfloat16 gradients
    with pytest.raises(RuntimeError, match=r"expected scalar type BFloat16 but found Half \(outGradients\)"):
        _call(name, dtype=torch.bfloat16, outGradients=torch.zeros(B, 3, H, W, dtype=F16))


@pytest.mark.parametrize("name", ["coord_loss_amp", "coord_loss_amp_async"])
@pytest.mark.parametrize("gt_dtype", [F16, torch.bfloat16, torch.float64])
def test_ground_truth_stays_float32(name, gt_dtype):
    with pytest.raises(RuntimeError, match=r"expected scalar type Float but found \w+ \(gtCoords\)"):
        _call(name, gtCoords=torch.zeros(B, 3, H, W, dtype=gt_dtype))


@pytest.mark.parametrize("name", ["reproj_loss_amp", "reproj_loss_amp_async"])
def test_poses_stay_float32(name):
    with pytest.raises(RuntimeError, match=r"expected scalar type Float but found Half \(gtPoses\)"):
        _call(name, gtPoses=torch.eye(4, dtype=F16).repeat(B, 1, 1))


@pytest.mark.parametrize("name", CALLS)
def test_cpu_tensors_are_refused(name):
    with pytest.raises(RuntimeError, match=rf"{name} takes CUDA tensors only \(prediction is on the CPU\)"):
        _call(name)
    with pytest.raises(RuntimeError, match=rf"{name} takes CUDA tensors only \(prediction is on the CPU\)"):
        _call(name, dtype=torch.bfloat16, outGradients=None)


@pytest.mark.parametrize("name", CALLS)
@pytest.mark.parametrize("scale,kind", [
    (torch.ones(1), "a CPU Float tensor of 1 elements"),
    (torch.ones((), dtype=torch.float64), "a CPU Double tensor of 1 elements"),
    (torch.ones(2), "a CPU Float tensor of 2 elements"),
    (1.0, "a float"),
])
def test_grad_scale_is_one_cuda_float32(name, scale, kind):
    with pytest.raises(RuntimeError, match=rf"{name}: gradScale must be a CUDA float32 tensor of one element or None, "
                                           rf"got {kind}"):
        _call(name, gradScale=scale)


def test_the_float32_calls_keep_their_contract():
    # the float32 entry points still refuse 16-bit maps: the 16-bit ones are separate names
    with pytest.raises(RuntimeError, match=r"expected scalar type Float but found Half \(prediction\)"):
        api.reproj_loss(torch.zeros(B, 3, H, W, dtype=F16), torch.eye(4).repeat(B, 1, 1), 500.0, 0, 0, 10.0)
    with pytest.raises(RuntimeError, match=r"expected scalar type Float but found BFloat16 \(prediction\)"):
        api.coord_loss(torch.zeros(B, 3, H, W, dtype=torch.bfloat16), torch.zeros(B, 3, H, W))
