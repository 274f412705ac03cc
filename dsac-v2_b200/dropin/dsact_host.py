"""Host-side helpers shared by the drop-in modules (`dsac_v2`, `networks.mlp`,
`training.*`): kwargs plumbing, the action distributions the CPU sampler and
evaluator call, and the TensorBoard tag names.  None of this is on the update
path; the update itself runs in libdsact.so.
"""
from __future__ import annotations

import math
import os
import sys
import time
from collections.abc import Mapping

import numpy as np
import torch

_REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if _REPO not in sys.path:
    sys.path.append(_REPO)  # for the `dsac_v2_b200` import shim at the repo root

EPS = 1e-6  # reference utils/act_distribution_cls.py:3

# tag names of reference utils/tensorboard_setup.py:142-153 that the update path emits
try:  # a DSAC-v2 checkout on sys.path provides the full table
    from utils.tensorboard_setup import tb_tags as TB_TAGS  # type: ignore
except Exception:  # standalone
    TB_TAGS = {
        "loss_actor": "Loss/Actor loss-RL iter",
        "loss_critic": "Loss/Critic loss-RL iter",
        "alg_time": "Time/Algorithm time [ms]-RL iter",
        "sampler_time": "Time/Sampler time [ms]-RL iter",
        "TAR of RL iteration": "Evaluation/1. TAR-RL iter",
        "TAR of total time": "Evaluation/2. TAR-Total time [s]",
        "TAR of collected samples": "Evaluation/3. TAR-Collected samples",
        "TAR of replay samples": "Evaluation/4. TAR-Replay samples",
        "Buffer RAM of RL iteration": "RAM/RAM [MB]-RL iter",
    }


class _DiagGaussBase:
    """Shared pieces of the two diagonal-Gaussian action distributions
    (reference utils/act_distribution_cls.py:21-116).  `logits` = cat(mean, std)."""

    def __init__(self, logits: torch.Tensor):
        self.logits = logits
        self.mean, self.std = torch.chunk(logits, 2, dim=-1)
        self.act_high_lim = torch.tensor([1.0])
        self.act_low_lim = torch.tensor([-1.0])

    def _gauss_logp(self, x):
        z = (x - self.mean) / self.std
        return (-0.5 * z * z - self.std.log() - 0.5 * math.log(2 * math.pi)).sum(-1)

    def _draw(self, reparam: bool):
        noise = torch.randn_like(self.mean)
        x = self.mean + self.std * noise
        return x if reparam else x.detach()

    def entropy(self):
        return (0.5 + 0.5 * math.log(2 * math.pi) + self.std.log()).sum(-1)

    def kl_divergence(self, other):
        var_ratio = (self.std / other.std) ** 2
        t1 = ((self.mean - other.mean) / other.std) ** 2
        return (0.5 * (var_ratio + t1 - 1 - var_ratio.log())).sum(-1)


class TanhGaussDistribution(_DiagGaussBase):
    """a = scale*tanh(u)+shift, u ~ N(mean, std) (reference :21-79)."""

    def _squash(self, u):
        scale = (self.act_high_lim - self.act_low_lim) / 2
        shift = (self.act_high_lim + self.act_low_lim) / 2
        logp = self._gauss_logp(u) - torch.log(1 + EPS - torch.tanh(u) ** 2).sum(-1) - torch.log(scale).sum(-1)
        return scale * torch.tanh(u) + shift, logp

    def sample(self):
        return self._squash(self._draw(False))

    def rsample(self):
        return self._squash(self._draw(True))

    def log_prob(self, action_limited):
        span = self.act_high_lim - self.act_low_lim
        u = torch.atanh((1 - EPS) * (2 * action_limited - (self.act_high_lim + self.act_low_lim)) / span)
        return self._gauss_logp(u) - torch.log(span * (1 + EPS - torch.tanh(u) ** 2)).sum(-1)

    def mode(self):
        scale = (self.act_high_lim - self.act_low_lim) / 2
        return scale * torch.tanh(self.mean) + (self.act_high_lim + self.act_low_lim) / 2


class GaussDistribution(_DiagGaussBase):
    """Unsquashed variant (reference :82-116); not used by the DSAC-T update engine."""

    def sample(self):
        x = self._draw(False)
        return x, self._gauss_logp(x)

    def rsample(self):
        x = self._draw(True)
        return x, self._gauss_logp(x)

    def log_prob(self, action):
        return self._gauss_logp(action)

    def mode(self):
        return torch.clamp(self.mean, self.act_low_lim, self.act_high_lim)


DISTRIBUTIONS = {"TanhGaussDistribution": TanhGaussDistribution, "GaussDistribution": GaussDistribution}


class ActionDistributionMixin:
    """`get_act_dist(logits)` of reference utils/act_distribution_cls.py:9-18."""

    def get_act_dist(self, logits):
        dist = self.action_distribution_cls(logits)
        if hasattr(self, "act_high_lim"):
            dist.act_high_lim = self.act_high_lim
            dist.act_low_lim = self.act_low_lim
        return dist


FULL_STATE_FORMAT = "dsact-full-state-1"


def full_state_dict(networks) -> dict:
    """Everything a bit-for-bit resume needs beyond `networks.state_dict()`: Adam moments and step counters, the
    mean_std EMA pair, the device generator's seed/counter.  `networks` is an `ApproxContainer` of `dsac_v2` or
    `dsac_v1`; both engines keep these in the same state slots (include/dsact.h)."""
    eng = networks.engine()
    st = eng.state.detach().cpu()
    ints = st[:16].view(torch.int32)
    return {
        "format": FULL_STATE_FORMAT,
        "networks": networks.state_dict(),
        "adam_m": eng.adam_m.detach().cpu().clone(),
        "adam_v": eng.adam_v.detach().cpu().clone(),
        "mean_std": [float(st[0]), float(st[1])],
        "adam_steps": [int(ints[8]), int(ints[9])],
        "rng_counter": int(ints[10]) & 0xFFFFFFFF,
        "rng_seed": int(eng._seed),
    }


def load_full_state_dict(networks, state: dict) -> None:
    """Restore what `full_state_dict` saved into the networks' engine."""
    if state.get("format") != FULL_STATE_FORMAT:
        raise ValueError("not a dsact full-state checkpoint")
    networks.load_state_dict(state["networks"])
    eng = networks.engine()
    with torch.no_grad():
        eng.adam_m.copy_(state["adam_m"])
        eng.adam_v.copy_(state["adam_v"])
        ints = eng.state[:16].view(torch.int32)
        ints[10] = int(state["rng_counter"]) - (1 << 32 if int(state["rng_counter"]) >= (1 << 31) else 0)
    eng.set_carry(state["mean_std"][0], state["mean_std"][1], state["adam_steps"][0], state["adam_steps"][1])
    eng.seed(state["rng_seed"])


def net_kwargs(kind: str, kwargs: dict) -> dict:
    """Per-network constructor arguments out of the flat kwargs dict; same keys and
    defaults as reference utils/common_utils.py:48-89 (MLP branch)."""
    func_type = kwargs[kind + "_func_type"]
    if func_type not in ("MLP", "CNN"):
        raise NotImplementedError(f"{kind}_func_type={func_type!r}: MLP and CNN networks run on the CUDA engine (not CNN_SHARED)")
    if kwargs.get("action_type", "continu") != "continu":
        raise NotImplementedError("DSAC don't support discrete action space!")
    dist = kwargs.get("policy_act_distribution", "TanhGaussDistribution")
    cls = dist if isinstance(dist, type) else DISTRIBUTIONS.get(dist)
    if cls is None:
        raise NotImplementedError(f"unknown action distribution {dist!r}")
    extra = dict(hidden_sizes=list(kwargs[kind + "_hidden_sizes"])) if func_type == "MLP" else dict(conv_type=kwargs[kind + "_conv_type"])
    return dict(
        apprfunc=func_type,
        name=kwargs[kind + "_func_name"],
        obs_dim=kwargs["obsv_dim"],
        act_dim=kwargs["action_dim"],
        **extra,
        hidden_activation=kwargs[kind + "_hidden_activation"],
        output_activation=kwargs[kind + "_output_activation"],
        min_log_std=kwargs.get(kind + "_min_log_std", -20.0),
        max_log_std=kwargs.get(kind + "_max_log_std", 2.0),
        std_type=kwargs.get(kind + "_std_type", "mlp_shared"),
        act_high_lim=np.array(kwargs["action_high_limit"], dtype=np.float32),
        act_low_lim=np.array(kwargs["action_low_limit"], dtype=np.float32),
        action_distribution_cls=cls,
    )


# ---- n replay-fed updates per call (DSAC_V2.replay_updates / DSAC_V1.replay_updates) --------------------------------
def host_draws(buffer, batch: int, n: int, noise_fn):
    """The host draws of n rounds of `buffer.sample_batch(batch)` + `local_update`, in that order: per round the replay
    indices (numpy's global generator, index_source "numpy"; else None) then the update's noise (`noise_fn(batch)`, torch's
    CPU generator; None for device noise).  Returns (idx [n, batch] or None, (eps1, eps2, z3, z4) stacked over rounds or
    None)."""
    idx, noise = [], []
    for _ in range(n):
        idx.append(buffer.sample_indices(batch))
        noise.append(noise_fn(batch))
    idx = None if idx[0] is None else torch.stack([torch.as_tensor(i) for i in idx])
    noise = None if noise[0] is None else tuple(torch.stack([z[j] for z in noise]) for j in range(4))
    return idx, noise


class LazyStatsRow(Mapping):
    """tb_info of update k of a replay_updates call: the [n, 16] statistics block is copied to pinned host memory once
    (asynchronously, at the call) and read on the first access to any of its rows.  `keys`: (tag, column) pairs."""

    class Block:
        def __init__(self, dev_stats: torch.Tensor):
            self.host = torch.empty(dev_stats.shape, dtype=torch.float32).pin_memory()
            self.host.copy_(dev_stats, non_blocking=True)
            self.event = torch.cuda.Event()
            self.event.record(torch.cuda.current_stream(dev_stats.device))
            self.rows = None

        def get(self):
            if self.rows is None:
                self.event.synchronize()
                self.rows = self.host.tolist()
            return self.rows

    def __init__(self, block: "LazyStatsRow.Block", k: int, keys, alg_ms: float):
        self._block, self._k, self._keys, self._alg_ms, self._vals = block, k, keys, alg_ms, None

    def _materialise(self) -> dict:
        if self._vals is None:
            row = self._block.get()[self._k]
            if row[14] != 0.0:   # include/dsact.h: tb_info slot 14 = 1 + rank of a peer that never arrived
                from dsac_v2_b200._lib import DsactError
                raise DsactError(f"data-parallel exchange timed out waiting for rank {int(row[14]) - 1}")
            vals = {tag: row[c] for tag, c in self._keys}
            vals[TB_TAGS["alg_time"]] = self._alg_ms
            self._vals, self._block = vals, None
        return self._vals

    def __getitem__(self, k):
        return self._materialise()[k]

    def __iter__(self):
        return iter(self._materialise())

    def __len__(self):
        return len(self._keys) + 1


def replay_updates_on_engine(eng, buffer, batch: int, iteration: int, n: int, noise_fn, keys, global_batch=None) -> list:
    """replay_updates on the MLP engine: the host draws of n rounds, one Engine.replay_steps call (with `global_batch`:
    one Engine.dp_replay_steps call over that many rows of every rank), one lazy tb_info mapping per update (`keys`: (tag,
    column of the 16 statistics) pairs)."""
    t0 = time.time()
    if buffer.engine is not eng:
        raise ValueError("the replay buffer is not attached to this algorithm's engine")
    if buffer.size == 0:
        raise ValueError("cannot sample from an empty replay buffer")
    buffer.flush()
    idx, noise = host_draws(buffer, batch, n, noise_fn)
    if global_batch is None:
        stats = eng.replay_steps(n, batch, buffer.size, iteration, idx=idx, noise=noise)
    else:
        stats = eng.dp_replay_steps(n, batch, buffer.size, iteration, global_batch, idx=idx, noise=noise)
    block = LazyStatsRow.Block(stats)
    alg_ms = (time.time() - t0) * 1000 / n
    return [LazyStatsRow(block, k, keys, alg_ms) for k in range(n)]
