"""The packed weights of ExpertStack and GatingNet are fully defined, padding included: a buffer the caching allocator
hands back with stale contents still packs bitwise to the oracle's array (zero between segments)."""
import numpy as np
import pytest
import torch

from esac_b200.experts import ExpertStack
from esac_b200.gating_net import GatingNet
from oracle import expert_oracle as XO
from oracle import gating_oracle as GO

pytestmark = pytest.mark.gpu


def _dirty(floats: int):
    """Leaves a freed block of at least `floats` NaN floats in torch's caching allocator."""
    junk = torch.full((floats,), float("nan"), device="cuda")
    del junk


def test_expert_stack_pack_over_stale_memory():
    sds = [XO.kaiming_state_dict(200 + e) for e in range(3)]
    _dirty(XO.packed_floats(3))
    got = ExpertStack(sds, "cuda").packed.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), XO.pack(sds).view(np.uint32))


@pytest.mark.parametrize("E, c", [(7, 1), (10, 2)])
def test_gating_pack_over_stale_memory(E, c):
    sd = GO.kaiming_state_dict(300 + E, E, c)
    _dirty(GO.packed_floats(E, c))
    got = GatingNet(sd, "cuda").packed.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), GO.pack(sd, c).view(np.uint32))
