"""`networks.cnn` of the drop-in: the two CNN approximators of DSAC-T (reference networks/cnn.py:151-240 `StochaPolicy`,
:383-461 `ActionValueDistri`), with the reference's class names, constructor kwargs and parameter names, so `state_dict()`
keeps the shipped schema (`policy.conv.0.weight`, `policy.mean.0.weight`, `q1.log_std.6.bias`, ...).

As in `networks.mlp`, these modules are containers + the plain-torch forward used by the CPU sampler and the evaluator;
during training their parameters are views into the CUDA engine's flat buffers and the update runs in libdsact.so
(`dsact_step` on a head-wise handle).  The reference's other classes of this file (DetermPolicy, ActionValue, the discrete variants) are
not on the DSAC-T path and are not mirrored.
"""
__all__ = ["StochaPolicy", "ActionValueDistri", "CONV_TYPES"]

import torch
import torch.nn as nn

from dsact_host import ActionDistributionMixin
from networks.mlp import _activation

# reference networks/cnn.py:163-170 (type_1) and :201-216 (type_2): kernel sizes, channels, strides, head widths
CONV_TYPES = {
    "type_1": dict(kernels=(8, 4, 3), channels=(32, 64, 64), strides=(4, 2, 1), heads=(512, 256)),
    "type_2": dict(kernels=(4, 3, 3, 3, 3, 3), channels=(8, 16, 32, 64, 128, 256), strides=(2, 2, 2, 2, 1, 1), heads=(256, 256, 256)),
}


def build_cnn(kernels, channels, strides, in_channels):
    """Conv2d / ReLU pairs (reference networks/cnn.py:30-53); even indices are the convolutions."""
    mods, cin = [], in_channels
    for k, c, s in zip(kernels, channels, strides):
        mods += [nn.Conv2d(cin, c, k, s), nn.ReLU()]
        cin = c
    return nn.Sequential(*mods)


def build_head(sizes, hidden_activation, output_activation):
    hidden, out = _activation(hidden_activation), _activation(output_activation)
    mods, last = [], len(sizes) - 2
    for j, (n_in, n_out) in enumerate(zip(sizes[:-1], sizes[1:])):
        mods += [nn.Linear(n_in, n_out), out() if j == last else hidden()]
    return nn.Sequential(*mods)


def _encoder(kwargs):
    if kwargs["conv_type"] not in CONV_TYPES:
        raise NotImplementedError(kwargs["conv_type"])
    t = CONV_TYPES[kwargs["conv_type"]]
    obs_dim = tuple(kwargs["obs_dim"])
    conv = build_cnn(t["kernels"], t["channels"], t["strides"], obs_dim[0])
    with torch.no_grad():
        feat = conv(torch.ones(obs_dim).unsqueeze(0)).reshape(1, -1).shape[-1]
    return conv, feat, list(t["heads"])


class StochaPolicy(nn.Module, ActionDistributionMixin):
    """image -> cat(mean, std); conv encoder + separate `mean` and `log_std` heads."""

    def __init__(self, **kwargs):
        super().__init__()
        act_dim = kwargs["act_dim"]
        self.conv, feat, heads = _encoder(kwargs)
        self.mean = build_head([feat, *heads, act_dim], kwargs["hidden_activation"], kwargs["output_activation"])
        self.log_std = build_head([feat, *heads, act_dim], kwargs["hidden_activation"], kwargs["output_activation"])
        self.min_log_std, self.max_log_std = kwargs["min_log_std"], kwargs["max_log_std"]
        self.register_buffer("act_high_lim", torch.from_numpy(kwargs["act_high_lim"]))
        self.register_buffer("act_low_lim", torch.from_numpy(kwargs["act_low_lim"]))
        self.action_distribution_cls = kwargs["action_distribution_cls"]

    def forward(self, obs):
        img = self.conv(obs)
        feature = img.view(img.size(0), -1)
        std = torch.clamp(self.log_std(feature), self.min_log_std, self.max_log_std).exp()
        return torch.cat((self.mean(feature), std), dim=-1)


class ActionValueDistri(nn.Module):
    """(image, act) -> cat(mean, softplus(std)); the action joins the flattened feature (reference :454-461)."""

    def __init__(self, **kwargs):
        super().__init__()
        act_dim = kwargs["act_dim"]
        self.conv, feat, heads = _encoder(kwargs)
        self.mean = build_head([feat + act_dim, *heads, 1], kwargs["hidden_activation"], kwargs["output_activation"])
        self.log_std = build_head([feat + act_dim, *heads, 1], kwargs["hidden_activation"], kwargs["output_activation"])

    def forward(self, obs, act):
        img = self.conv(obs)
        feature = torch.cat([img.view(img.size(0), -1), act], -1)
        return torch.cat((self.mean(feature), nn.functional.softplus(self.log_std(feature))), dim=-1)
