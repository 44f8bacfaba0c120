"""The expert stack's oracle (oracle/expert_oracle.py) on the CPU: the packed layout round-trips to the state dicts (the
tensor-core layers' weights to their TF32 rounding, everything else exactly), the TF32 rounding itself, and the float64
layer sequence against an independent nn.Module built here from the reference's layer table."""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import expert_oracle as O


def test_tf32_rounding():
    x = np.array([1.0, 1.0 + 2.0 ** -11, 1.0 + 2.0 ** -10, 1.0 + 3 * 2.0 ** -11, -(1.0 + 2.0 ** -11), 1.0 + 2.0 ** -12,
                  0.0, -0.0, 3.0e-39], np.float32)
    want = np.array([1.0, 1.0 + 2.0 ** -10, 1.0 + 2.0 ** -10, 1.0 + 2.0 ** -9, -(1.0 + 2.0 ** -10), 1.0, 0.0, -0.0,
                     np.float32(3.0e-39).view(np.uint32) & 0xFFFFE000], np.float64)
    want[-1] = np.array([int(want[-1])], np.uint32).view(np.float32)[0]
    got = O.tf32(x)
    assert np.array_equal(got.view(np.uint32)[:-1], want[:-1].astype(np.float32).view(np.uint32))
    assert got[-1] == np.float32(want[-1])
    r = np.random.default_rng(0).normal(size=10000).astype(np.float32)
    t = O.tf32(r)
    assert not (t.view(np.uint32) & 0x1FFF).any()
    assert np.all(np.abs(t - r) <= np.abs(r) * 2.0 ** -11)


def test_pack_round_trip():
    sds = [O.kaiming_state_dict(s, mean=(1.0 + s, -2.0, 0.25)) for s in range(3)]
    packed = O.pack(sds)
    assert packed.size == O.packed_floats(3)
    back = O.unpack(packed, 3)
    for sd, got in zip(sds, back):
        assert list(got) == list(sd)
        for k, v in sd.items():
            want = v.numpy()
            if k.endswith(".weight") and not k.startswith(("conv1.", "fc3.")):
                want = O.tf32(want)
            assert got[k].shape == want.shape and np.array_equal(got[k].view(np.uint32), want.view(np.uint32)), k


class Expert(nn.Module):
    """The reference's Expert from its layer table, as modules (float64 here)."""

    def __init__(self):
        super().__init__()
        c = lambda i, o, k, s: nn.Conv2d(i, o, k, s, k // 2)  # noqa: E731
        self.conv1, self.conv2, self.conv3, self.conv4 = c(3, 32, 3, 1), c(32, 64, 3, 2), c(64, 128, 3, 2), c(128, 256, 3, 2)
        self.res1_conv1, self.res1_conv2, self.res1_conv3 = c(256, 256, 3, 1), c(256, 256, 1, 1), c(256, 256, 3, 1)
        self.res2_conv1, self.res2_conv2, self.res2_conv3 = c(256, 512, 3, 1), c(512, 512, 1, 1), c(512, 512, 3, 1)
        self.res2_skip = c(256, 512, 1, 1)
        self.res3_conv1, self.res3_conv2, self.res3_conv3 = c(512, 512, 1, 1), c(512, 512, 1, 1), c(512, 512, 1, 1)
        self.fc1, self.fc2, self.fc3 = c(512, 512, 1, 1), c(512, 512, 1, 1), c(512, 3, 1, 1)
        self.register_buffer("mean", torch.zeros(3))

    def forward(self, x):
        x = F.relu(self.conv3(F.relu(self.conv2(F.relu(self.conv1(x))))))
        res = F.relu(self.conv4(x))
        res = res + F.relu(self.res1_conv3(F.relu(self.res1_conv2(F.relu(self.res1_conv1(res))))))
        res = self.res2_skip(res) + F.relu(self.res2_conv3(F.relu(self.res2_conv2(F.relu(self.res2_conv1(res))))))
        res = res + F.relu(self.res3_conv3(F.relu(self.res3_conv2(F.relu(self.res3_conv1(res))))))
        x = self.fc3(F.relu(self.fc2(F.relu(self.fc1(res)))))
        return x + self.mean.view(1, 3, 1, 1)


def test_oracle_matches_module():
    sd = O.kaiming_state_dict(4, mean=(0.5, -1.5, 3.0))
    m = Expert().double()
    m.load_state_dict({k: v.double() for k, v in sd.items()})
    assert set(m.state_dict()) == set(sd)
    g = torch.Generator().manual_seed(1)
    for H, W in ((37, 53), (64, 80)):
        img = torch.randn((2, 3, H, W), generator=g, dtype=torch.float64)
        with torch.no_grad():
            want = m(img)
        got = O.forward(img, sd)
        assert got.dtype == torch.float64 and got.shape == (2, 3, -(-H // 8), -(-W // 8))
        assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)
