"""esac_b200.networks: Expert and Gating as trainable torch modules.  Their state dicts are the reference's (the keys and
shapes the device paths take), model files load into them and theirs into the restated reference modules with
strict=True, and their float64 forward is the oracles' to 1e-12."""
import pytest
import torch

from esac_b200 import experts as X
from esac_b200 import gating_net as G
from esac_b200.networks import Expert, Gating, init_adam_state
from oracle import expert_oracle as XO
from oracle import gating_oracle as GO
from test_experts_oracle import Expert as RestatedExpert


def shapes(module) -> dict:
    return {k: tuple(v.shape) for k, v in module.state_dict().items()}


def test_expert_state_dict_is_the_layer_tables():
    m = Expert(torch.tensor([1.0, 2.0, 3.0]))
    assert shapes(m) == X.state_dict_shapes()
    assert torch.equal(m.mean, torch.tensor([1.0, 2.0, 3.0]))
    assert [k for k, _ in m.named_buffers()] == ["mean"]


@pytest.mark.parametrize("E, c", [(1, 1), (7, 1), (19, 1), (2, 2), (10, 2)])
def test_gating_state_dict_is_the_layer_tables(E, c):
    m = Gating(E, c)
    assert shapes(m) == G.state_dict_shapes(E, c)
    assert G.network_size(m.state_dict()) == (E, c)


def test_gating_refuses_other_capacities():
    with pytest.raises(ValueError, match="capacity"):
        Gating(3, 3)


def test_model_files_load_both_ways():
    sd = XO.kaiming_state_dict(5, mean=(0.5, -1.0, 2.0))
    m = Expert(torch.zeros(3))
    m.load_state_dict(sd, strict=True)
    assert torch.equal(m.mean, sd["mean"])
    RestatedExpert().load_state_dict(m.state_dict(), strict=True)
    for E, c in ((3, 1), (4, 2)):
        gsd = GO.kaiming_state_dict(9, E, c)
        g = Gating(E, c)
        g.load_state_dict(gsd, strict=True)
        GO.make_gating_class()(E, c).load_state_dict(g.state_dict(), strict=True)
        with pytest.raises(RuntimeError):
            Gating(E + 1, c).load_state_dict(gsd, strict=True)


@pytest.mark.parametrize("hw", [(37, 53), (64, 48)])
def test_expert_forward_is_the_oracle(hw):
    sd = XO.kaiming_state_dict(3, mean=(0.3, -0.5, 2.5))
    m = Expert(torch.zeros(3)).double()
    m.load_state_dict(sd)
    img = torch.randn((2, 3) + hw, generator=torch.Generator().manual_seed(hw[0]), dtype=torch.float64)
    with torch.no_grad():
        got = m(img)
    want = XO.forward(img, sd)
    assert got.shape == want.shape == (2, 3, -(-hw[0] // 8), -(-hw[1] // 8))
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("E, c, hw", [(3, 1, (40, 56)), (7, 1, (64, 48)), (2, 2, (48, 64)), (5, 2, (37, 53))])
def test_gating_forward_is_the_oracle(E, c, hw):
    sd = GO.kaiming_state_dict(E + c, E, c)
    m = Gating(E, c).double()
    m.load_state_dict(sd)
    img = torch.randn((2, 3) + hw, generator=torch.Generator().manual_seed(E), dtype=torch.float64)
    with torch.no_grad():
        got = m(img)
    want = GO.forward(img, sd, c)
    assert got.shape == want.shape == (2, E)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)


def test_expert_output_is_differentiable():
    m = Expert(torch.tensor([1.0, 0.0, -1.0]))
    out = m(torch.randn(1, 3, 16, 24, generator=torch.Generator().manual_seed(0)))
    out.sum().backward()
    assert all(p.grad is not None for p in m.parameters()) and m.mean.grad is None


def test_init_adam_state_is_adams_first_state():
    m = Gating(3, 1)
    made = torch.optim.Adam(m.parameters(), lr=1e-3)
    init_adam_state(made)
    for p in m.parameters():
        st = made.state[p]
        assert st["step"].dtype == torch.float32 and float(st["step"]) == 0.0
        assert torch.equal(st["exp_avg"], torch.zeros_like(p)) and torch.equal(st["exp_avg_sq"], torch.zeros_like(p))
    kept = {p: made.state[p]["exp_avg"] for p in m.parameters()}
    init_adam_state(made)                                   # a second call keeps what is there
    assert all(made.state[p]["exp_avg"] is kept[p] for p in m.parameters())
