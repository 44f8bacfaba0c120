"""The reference's networks as trainable torch modules, written from the layer tables of this library.

Expert(mean) is code/expert.py's Expert and Gating(num_experts, capacity) is code/gating.py's Gating: the same layers, the
same forward, and the same state-dict keys and shapes (experts.state_dict_shapes(), gating_net.state_dict_shapes(E,
capacity)), so the reference's model files load into them with load_state_dict(strict=True) and theirs into the
reference's.  They are what the training command (esac_b200.train) differentiates and steps with torch.optim.Adam; the
device inference paths (experts.ExpertStack, gating_net.GatingNet) take their state dicts as they are.

    gating, expert = Gating(E, 1).cuda(), Expert(torch.zeros(3)).cuda()
    gating.load_state_dict(torch.load('gating_scene.net'))
    expert.load_state_dict(torch.load('expert_e0_scene.net'))
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from .experts import LAYERS
from .gating_net import layers


def _convs(module: nn.Module, table):
    for name, cin, cout, k, s in table:
        setattr(module, name, nn.Conv2d(cin, cout, k, s, k // 2))


class Expert(nn.Module):
    """The scene-coordinate FCN: image [B,3,H,W] -> scene coordinates [B,3,ceil(H/8),ceil(W/8)], plus the buffer `mean`
    (the expert's scene centre, 3 values) added to the output."""

    def __init__(self, mean):
        super().__init__()
        self.register_buffer("mean", torch.as_tensor(mean, dtype=torch.float32).detach().clone().reshape(3))
        _convs(self, LAYERS)

    def forward(self, inputs):
        x = F.relu(self.conv1(inputs))
        x = F.relu(self.conv2(x))
        x = F.relu(self.conv3(x))
        res = F.relu(self.conv4(x))
        x = F.relu(self.res1_conv1(res))
        x = F.relu(self.res1_conv2(x))
        x = F.relu(self.res1_conv3(x))
        res = res + x
        x = F.relu(self.res2_conv1(res))
        x = F.relu(self.res2_conv2(x))
        x = F.relu(self.res2_conv3(x))
        res = self.res2_skip(res) + x
        x = F.relu(self.res3_conv1(res))
        x = F.relu(self.res3_conv2(x))
        x = F.relu(self.res3_conv3(x))
        res = res + x
        x = F.relu(self.fc1(res))
        x = F.relu(self.fc2(x))
        return self.fc3(x) + self.mean.view(1, 3, 1, 1)


class Gating(nn.Module):
    """The gating network: image [B,3,H,W] -> log-probabilities [B,num_experts] over the experts.  capacity 1 for room
    environments (a tanh before the pooling), 2 for clustered ones (twice the channels, no tanh)."""

    def __init__(self, num_experts: int, capacity: int = 1):
        super().__init__()
        if capacity not in (1, 2):
            raise ValueError(f"Gating: capacity must be 1 or 2, got {capacity}")
        self.capacity = capacity
        _convs(self, layers(num_experts, capacity))

    def forward(self, inputs):
        x = inputs
        for name in ("conv1", "conv2", "conv3", "conv4", "res1_conv1", "res1_conv2", "res1_conv3"):
            x = F.relu(getattr(self, name)(x))
        if self.capacity == 1:
            x = torch.tanh(x)
        x = F.avg_pool2d(x, x.size()[2:])
        x = F.relu(self.fc1(x))
        x = F.relu(self.fc2(x))
        x = F.log_softmax(self.fc3(x), dim=1)
        return x[:, :, 0, 0]


def init_adam_state(opt):
    """Creates now the state torch.optim.Adam(capturable=True) creates at its first step: zero moments, step 0 on the
    parameter's device.  A captured step must not create it, least of all inside a region of a graph that a replay may
    skip (gate.ExpertGate), so every optimiser of a captured training step is prepared with this before the warm-up."""
    for group in opt.param_groups:
        for p in group["params"]:
            st = opt.state[p]
            if not st:
                st["step"] = torch.zeros((), dtype=torch.float32, device=p.device)
                st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
