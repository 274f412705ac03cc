"""Python owner of one handle of libdsact's head-wise fp32 engine (`dsact_cnn_create`, include/dsact.h): the update with
the reference's CNN approximators (BASELINE config 5; reference networks/cnn.py), the policy std types the MLP engine
does not implement, and DSAC_V1.  Everything but the configuration, the state_dict schema and the image-shaped
minibatches is `engine.Engine`'s: the same buffers, and the same dsact_* calls on the handle.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import torch

from . import _lib
from ._lib import Batch, CnnConfig
from .engine import Engine


def make_cnn_config(obs_shape: Sequence[int], act_dim: int, kernels: Sequence[int], channels: Sequence[int],
                    strides: Sequence[int], hidden: Sequence[int], *, max_batch: int, act_hidden: str = "gelu", gamma=0.99,
                    tau=0.005, tau_b=None, delay_update=2, auto_alpha=True, alpha=0.2, lr_q=1e-4, lr_pi=1e-4, lr_alpha=3e-4,
                    min_log_std=-20.0, max_log_std=0.5, q_heads: int = 2, pi_std: str = "head",
                    act_dist: str = "TanhGaussDistribution", algo: str = "DSAC_V2", bound: bool = True,
                    td_bound: float = 20.0) -> CnnConfig:
    """`q_heads` / `pi_std` select the head wiring: (2, "head") = networks/cnn.py; with no conv layers and
    obs_shape = (obs_dim, 1, 1): (1, "head") = networks/mlp.py with policy std_type "mlp_separated", (1, "row") = "parameter"."""
    if len(kernels) > _lib.MAX_CONV or len(hidden) > _lib.MAX_HIDDEN:
        raise ValueError("too many layers")
    c = CnnConfig()
    c.abi_version = _lib.ABI_VERSION
    c.channels, c.height, c.width = (int(x) for x in obs_shape)
    c.act_dim, c.n_conv, c.n_hidden = int(act_dim), len(kernels), len(hidden)
    for j, (k, ch, st) in enumerate(zip(kernels, channels, strides)):
        c.conv_kernel[j], c.conv_channels[j], c.conv_stride[j] = int(k), int(ch), int(st)
    for j, v in enumerate(hidden):
        c.hidden[j] = int(v)
    c.act_hidden = _lib.ACTIVATIONS[act_hidden]
    c.max_batch, c.auto_alpha, c.delay_update = int(max_batch), int(bool(auto_alpha)), int(delay_update)
    c.gamma, c.tau, c.tau_b = float(gamma), float(tau), float(tau if tau_b is None else tau_b)
    c.alpha_fixed = float(alpha)
    c.lr_q, c.lr_pi, c.lr_alpha = float(lr_q), float(lr_pi), float(lr_alpha)
    c.min_log_std, c.max_log_std = float(min_log_std), float(max_log_std)
    c.adam_beta1, c.adam_beta2, c.adam_eps = 0.9, 0.999, 1e-8
    c.q_heads, c.pi_std = int(q_heads), {"head": 0, "row": 1, "shared": 2}[pi_std]
    c.algo, c.v1_bound, c.td_bound = {"DSAC_V2": 0, "DSAC_V1": 1}[algo], int(bool(bound)), float(td_bound)
    c.act_dist = _lib.ACT_DISTS[act_dist]
    return c


def make_heads_config(obs_dim: int, act_dim: int, hidden: Sequence[int], std_type: str, **kw) -> CnnConfig:
    """The MLP approximators on the head-wise fp32 engine: no encoder, one two-output head per critic, the policy with any
    of the reference's std types (networks/mlp.py:43-72).  DSAC-T with "mlp_shared" normally runs on `engine.Engine`
    (wgmma); this entry is for "mlp_separated" / "parameter" and for `algo="DSAC_V1"`."""
    return make_cnn_config((int(obs_dim), 1, 1), act_dim, (), (), (), hidden, q_heads=1,
                           pi_std={"mlp_separated": "head", "parameter": "row", "mlp_shared": "shared"}[std_type], **kw)


class CnnEngine(Engine):
    """A head-wise engine handle bound to flat torch-owned buffers on one CUDA device.  Minibatches are copied to the
    device by torch (image observations [B, C, H, W], host or device tensors); the MLP engine's host-staging path, its
    replay-fused steps, `profile_step` and `test_gemm` raise `DsactError`."""

    _query, _create = "dsact_cnn_query_layout", "dsact_cnn_create"
    _step_host = None   # _batch copies host minibatches to the device

    @property
    def obs_elems(self) -> int:
        return self.cfg.channels * self.cfg.height * self.cfg.width

    # ---- flat layout in the reference's state_dict schema (include/dsact.h) --------------------------------------------
    def _schema(self):
        c = self.cfg
        out, off = [], 0
        shapes = []
        cin, hh, ww = c.channels, c.height, c.width
        for j in range(c.n_conv):
            k, co, st = c.conv_kernel[j], c.conv_channels[j], c.conv_stride[j]
            shapes.append((f"conv.{2 * j}", (co, cin, k, k), (co,)))
            cin, hh, ww = co, (hh - k) // st + 1, (ww - k) // st + 1
        feat = cin * hh * ww
        hidden = [c.hidden[j] for j in range(c.n_hidden)]

        def leaf(net, name, shape):
            nonlocal off
            n = 1
            for d in shape:
                n *= int(d)
            out.append((f"{net}.{name}", f"{net}_target.{name}", off, n, shape))
            off += n

        def mlp(net, head, sizes):
            for j in range(len(sizes) - 1):
                leaf(net, f"{head}.{2 * j}.weight", (sizes[j + 1], sizes[j]))
                leaf(net, f"{head}.{2 * j}.bias", (sizes[j + 1],))

        critics = ("q",) if c.algo == 1 else ("q1", "q2")   # dsac_v1.ApproxContainer holds ONE critic named `q`
        for net, extra, width in tuple((n, c.act_dim, 1) for n in critics) + (("policy", 0, c.act_dim),):
            for name, wshape, bshape in shapes:
                leaf(net, f"{name}.weight", wshape)
                leaf(net, f"{name}.bias", bshape)
            if net != "policy" and c.q_heads == 1:          # networks/mlp.py ActionValueDistri: self.q
                mlp(net, "q", [feat + extra] + hidden + [2])
            elif net == "policy" and c.pi_std == 2:         # networks/mlp.py std_type "mlp_shared": self.policy, 2A outputs
                mlp(net, "policy", [feat] + hidden + [2 * width])
            elif net == "policy" and c.pi_std == 1:         # the module's own parameter precedes its children's
                leaf(net, "log_std", (1, width))
                mlp(net, "mean", [feat] + hidden + [width])
            else:
                for head in ("mean", "log_std"):
                    mlp(net, head, [feat + extra] + hidden + [width])
        return out, off

    def _batch(self, data: Dict[str, torch.Tensor]) -> Batch:
        """ctypes batch of a minibatch; the device copies stay referenced until the next call, which is after the kernels
        reading them were enqueued."""
        t = {k: data[k].to(device=self.device, dtype=torch.float32).contiguous() for k in ("obs", "act", "rew", "obs2", "done")}
        B = t["obs"].shape[0]
        if t["obs"][0].numel() != self.obs_elems or t["obs2"].shape != t["obs"].shape or t["act"].shape != (B, self.cfg.act_dim):
            raise ValueError("minibatch shapes do not match the configured observation / action shape")
        self._keep = t
        return Batch(t["obs"].data_ptr(), t["act"].data_ptr(), t["rew"].data_ptr(), t["obs2"].data_ptr(), t["done"].data_ptr(), B, None)

    def replay_sample(self, batch: int, size: int, idx: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        out = super().replay_sample(batch, size, idx)
        if self.cfg.n_conv:   # image observations
            shape = (int(batch), self.cfg.channels, self.cfg.height, self.cfg.width)
            out["obs"], out["obs2"] = out["obs"].view(shape), out["obs2"].view(shape)
        return out
