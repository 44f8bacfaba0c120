"""Argument errors of api.render_init_maps and its C entry point: the Python checks raise before any context exists, and
the C entry point refuses a null context before it reads anything, so all of this runs without a GPU.  The C entry
point's other refusals (inconsistent offsets, sides, null or host outputs) need a context, which needs a device: they are
checked in test_gpu_render.py (test_c_entry_refuses_inconsistent_arguments)."""
import re
from pathlib import Path

import numpy as np
import pytest
import torch

import esac_b200.api as api


def base():
    return dict(points=torch.zeros(4, 3), offsets=np.array([0, 2, 3]), indices=torch.tensor([0, 1, 3], dtype=torch.int32),
                poses=torch.eye(4).repeat(2, 1, 1), focal=[500.0, 400.0], out_scale=[0.1, 0.1],
                out_shapes=[(60, 80), (80, 60)])


BAD = [
    (dict(points=torch.zeros(4, 3, dtype=torch.float64)), "found Double"),
    (dict(points=torch.zeros(4, 2)), r"points must be \[P,3\]"),
    (dict(indices=torch.tensor([0, 1, 3])), "expected scalar type Int but found Long"),
    (dict(poses=torch.eye(4).repeat(2, 1, 1).double()), "found Double"),
    (dict(poses=torch.eye(4).repeat(3, 1, 1)), r"poses must be \[2,4,4\] or \[2,3,4\]"),
    (dict(poses=torch.zeros(2, 2, 4)), r"poses must be"),
    (dict(offsets=np.array([0])), "0 cameras, need at least 1"),
    (dict(offsets=np.array([1, 2, 3])), r"offsets\[0\]=1, need 0"),
    (dict(offsets=np.array([0, 3, 2, 3]), focal=[1.0] * 3, out_scale=[1.0] * 3, poses=torch.eye(4).repeat(3, 1, 1),
          out_shapes=[(4, 4)] * 3), "offsets decrease at camera 1"),
    (dict(offsets=np.array([0, 2, 4])), "offsets end at 4, but indices holds 3"),
    (dict(offsets=np.array([0.0, 2.0, 3.0])), "offsets must be a 1-d integer array"),
    (dict(focal=[1.0]), "focal must be a number or 2 numbers"),
    (dict(out_scale=[1.0, 2.0, 3.0]), "out_scale must be a number or 2 numbers"),
    (dict(out_shapes=[(60, 80)]), r"out_shapes must be 2 integer pairs"),
    (dict(out_shapes=[(60, 0), (80, 60)]), r"camera 0 map is 60x0, need sides in \[1, 8192\]"),
    (dict(out_shapes=[(60, 80), (8193, 60)]), r"camera 1 map is 8193x60"),
    (dict(offsets=np.r_[0, np.full(17, 3)], poses=torch.eye(4).repeat(17, 1, 1), focal=1.0, out_scale=1.0,
          out_shapes=[(8192, 8192)] * 17), "more than 1073741824"),
]


@pytest.mark.parametrize("change, match", BAD, ids=[str(i) for i in range(len(BAD))])
def test_render_refuses_before_any_context(change, match):
    a = base()
    a.update(change)
    with pytest.raises(RuntimeError, match=match):
        api.render_init_maps(**a)
    assert not api._contexts


def test_c_entry_refuses_a_null_context(lib):
    assert lib.esacb200_render_init_maps(None, 1, None, 0, None, None, None, None, None, None, None, None, None, None,
                                         None) == -2


def test_entry_point_is_declared():
    header = (Path(__file__).resolve().parents[1] / "include" / "esac_b200.h").read_text()
    assert re.search(r"int esacb200_render_init_maps\(esacb200_ctx\* ctx, int C,", header)
    assert "#define ESACB200_RENDER_MAX_SIDE 8192" in header
