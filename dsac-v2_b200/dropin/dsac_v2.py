"""`dsac_v2` of the drop-in: `ApproxContainer` and `DSAC_V2` with the reference's
names, kwargs and return values (reference dsac_v2.py:19-62, 66-347), backed by
the CUDA engine (libdsact.so) instead of eager PyTorch.

* `ApproxContainer` stays an `nn.Module` with the reference's parameter names and
  53-key `state_dict`; once on a CUDA device its parameters are views into the
  engine's flat buffers (params / targets), and Adam moments live beside them.
* `DSAC_V2.local_update(data, iteration) -> tb_info` runs the whole update
  (losses, three backward passes, Adam, delayed Polyak) in the CUDA library.
  There is no CPU fallback: on a CPU module it raises.
* `value_output_activation` / `policy_output_activation` (any hidden-activation
  name) end the networks as in the reference, on every engine the module picks.
* `get_remote_update_info` / `remote_update` keep the gradient-message seam
  (reference :107-138); with `torch.distributed` initialised the step is
  data-parallel (all-reduce of the two critic-std sums and of the flat gradients).

Extra kwargs (all optional): `dsact_noise` = "device" (Philox on the GPU, default)
or "reference" (draw the 8 normals of one update from torch's CPU generator in the
reference's order, SURVEY Appendix B — same seed, same numbers as the reference);
`dsact_gemm` = "bf16x3" (wgmma split-precision, default) | "fp32" | "bf16" (outside the parity gate); `dsact_graph` = True; `dsact_max_batch`.
"""
__all__ = ["ApproxContainer", "DSAC_V2"]

import time
import weakref
from collections.abc import Mapping
from copy import deepcopy
from typing import Dict, Tuple

import torch
import torch.nn as nn

from dsact_host import TB_TAGS as tb_tags
from dsact_host import full_state_dict as _full_state
from dsact_host import replay_updates_on_engine
from dsact_host import load_full_state_dict as _load_full_state
from dsact_route import EngineContainer, network_classes

from dsac_v2_b200 import _lib, dp
from dsac_v2_b200.engine import STAT_KEYS


class ApproxContainer(EngineContainer):
    """Six networks + log_alpha (reference dsac_v2.py:19-62)."""

    algorithm, critics = "DSAC_V2", ("q1", "q2")

    def __init__(self, **kwargs):
        super().__init__()
        q_args, pi_args, q_cls, pi_cls = network_classes(self.algorithm, kwargs)
        # construction order q1, q2, policy = the reference's consumption of torch's RNG (:31-39)
        self.q1 = q_cls(**q_args)
        self.q2 = q_cls(**q_args)
        self.q1_target = deepcopy(self.q1)
        self.q2_target = deepcopy(self.q2)
        self.policy = pi_cls(**pi_args)
        self.policy_target = deepcopy(self.policy)
        for net in (self.policy_target, self.q1_target, self.q2_target):
            for p in net.parameters():
                p.requires_grad = False
        self.log_alpha = nn.Parameter(torch.tensor(1, dtype=torch.float32))
        self._route(kwargs)

    def device_seed(self) -> int:
        """64-bit seed of the engine's Philox generator: splitmix64 of (user seed, data-parallel rank), so that seeds and
        ranks draw independent streams."""
        rank = 0
        try:
            import torch.distributed as dist
            if dist.is_available() and dist.is_initialized():
                rank = dist.get_rank()
        except Exception:   # noqa: BLE001
            rank = 0
        z = (super().device_seed() * 0x9E3779B97F4A7C15 + (rank + 1) * 0xBF58476D1CE4E5B9) & (2 ** 64 - 1)
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & (2 ** 64 - 1)
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & (2 ** 64 - 1)
        return z ^ (z >> 31)


class _LazyTbInfo(Mapping):
    """tb_info whose 14 device-computed scalars are fetched on first access (one event wait),
    so a training loop that only logs every N iterations never stalls on `.item()`."""

    def __init__(self, slot, event, alg_ms):
        self._slot, self._event, self._alg_ms, self._vals = slot, event, alg_ms, None

    def _materialise(self):
        if self._vals is None:
            self._event.synchronize()
            err = float(self._slot[14])
            if err != 0.0:   # include/dsact.h: tb_info slot 14 = 1 + rank of a peer that never arrived
                raise _lib.DsactError(f"data-parallel exchange timed out waiting for rank {int(err) - 1}")
            vals = dict(zip(STAT_KEYS, self._slot.tolist()))
            vals[tb_tags["alg_time"]] = self._alg_ms
            self._vals, self._slot = vals, None
        return self._vals

    def __getitem__(self, k):
        return self._materialise()[k]

    def __iter__(self):
        return iter(self._materialise())

    def __len__(self):
        return len(STAT_KEYS) + 1


class DSAC_V2:
    """DSAC-T (arXiv 2310.05858) on the CUDA engine; interface of reference dsac_v2.py:66-138."""

    _RING = 32

    def __init__(self, **kwargs):
        self.networks = ApproxContainer(**kwargs)
        self.gamma = kwargs["gamma"]
        self.tau = kwargs["tau"]
        self.target_entropy = -kwargs["action_dim"]
        self.auto_alpha = kwargs["auto_alpha"]
        self.alpha = kwargs.get("alpha", 0.2)
        self.delay_update = kwargs["delay_update"]
        self.tau_b = kwargs.get("tau_b", self.tau)
        self.act_dim = kwargs["action_dim"]
        self.noise_source = kwargs.get("dsact_noise", "device")
        if self.noise_source not in ("device", "reference"):
            raise ValueError("dsact_noise must be 'device' or 'reference'")
        self.data_parallel = kwargs.get("dsact_data_parallel", True)
        # "peer": exchanges inside the step's kernels over NVLink peer memory (falls back to NCCL if the ranks cannot
        # map each other's buffers); "nccl": torch.distributed all-reduces between three graph launches
        self.dp_transport = kwargs.get("dsact_dp_transport", "peer")
        if self.networks.route.engine == "mlp" and kwargs.get("policy_std_type", "mlp_shared") != "mlp_shared":
            self.dp_transport = "nccl"   # the MLP engine's peer-memory step serves mlp_shared only (dsact_dp_step refuses)
        self._peer_dp, self._peer_eng = None, None
        self._slots, self._owners, self._cursor = None, [None] * self._RING, 0

    @property
    def adjustable_parameters(self):
        return ("gamma", "tau", "auto_alpha", "alpha", "delay_update")

    @property
    def mean_std1(self):
        return float(self.networks.engine().state[0])

    @property
    def mean_std2(self):
        return float(self.networks.engine().state[1])

    # ---- helpers ------------------------------------------------------------------
    def _noise(self, batch: int):
        if self.noise_source == "device":
            return None
        A = self.act_dim
        eps1 = torch.empty(batch, A).normal_()   # rsample of pi(obs),        reference :160
        eps2 = torch.empty(batch, A).normal_()   # rsample of pi_target(obs2), reference :228
        z = [torch.normal(torch.zeros(batch), torch.ones(batch)) for _ in range(6)]  # __q_evaluate x6
        return eps1, eps2, z[2], z[3]

    def _world(self):
        return dp.world() if self.data_parallel else (None, 1)

    def _peers(self, eng, dist) -> bool:
        """True when `eng`'s data-parallel updates run over peer memory.  The first data-parallel update (or the first
        after the engine was rebuilt) maps the exchange buffers: a collective call."""
        if self._peer_dp is None or self._peer_eng is not eng:
            self._peer_dp = self.dp_transport != "nccl" and dp.connect_peers(eng, dist)
            self._peer_eng = eng
        return self._peer_dp

    def _stats(self, eng, global_batch, t0):
        if self._slots is None:
            self._slots = [torch.zeros(_lib.NUM_STATS, dtype=torch.float32).pin_memory() for _ in range(self._RING)]
        i = self._cursor
        self._cursor = (i + 1) % self._RING
        prev = self._owners[i]() if self._owners[i] is not None else None
        if prev is not None:
            prev._materialise()  # its pinned slot is about to be reused
        eng.read_stats_async(global_batch, out=self._slots[i])
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(eng.device))
        info = _LazyTbInfo(self._slots[i], ev, (time.time() - t0) * 1000)
        self._owners[i] = weakref.ref(info)
        return info

    def _gradients(self, data, eng):
        """Everything up to (and including) the gradients; returns the global batch size."""
        B = data["obs"].shape[0]
        noise = self._noise(B)
        dist, world = self._world()
        if world == 1:
            eng.compute_grads(data, noise)
            return B
        # every rank holds `B` rows of the global minibatch (the trainer samples B per rank)
        return dp.data_parallel_gradients(eng, data, noise, dist, B, B * world)

    # ---- full training state (SURVEY §8f rank 3; the reference saves weights only, training/trainer.py:137-152) ----
    def full_state_dict(self) -> dict:
        """Everything a bit-for-bit resume needs beyond the 53-key `networks.state_dict()`: Adam moments and step
        counters, the mean_std EMA pair, the device generator's seed/counter."""
        return _full_state(self.networks)

    def load_full_state_dict(self, state: dict) -> None:
        _load_full_state(self.networks, state)

    # ---- reference interface ------------------------------------------------------
    def local_update(self, data: Dict, iteration: int) -> dict:
        t0 = time.time()
        B = data["obs"].shape[0]
        eng = self.networks.engine(B)
        dist, world = self._world()
        if world == 1:
            eng.step(data, iteration, self._noise(B))
            return self._stats(eng, B, t0)
        if self._peers(eng, dist):   # one graph launch; exchanges inside the step's kernels over NVLink peer memory
            eng.dp_step(data, iteration, B * world, self._noise(B))
            return self._stats(eng, B * world, t0)
        gb = self._gradients(data, eng)
        eng.apply(iteration)
        return self._stats(eng, gb, t0)

    def replay_updates(self, buffer, batch_size: int, iteration: int, n: int) -> list:
        """n rounds of `local_update(buffer.sample_batch(batch_size), iteration + k)`, k = 0 .. n-1, as ONE engine call
        (Engine.replay_steps) where the engine has one: the same host draws in the same order (numpy indices, torch CPU
        noise), the same results.  Device draws take one generator counter per update (as replay_step), not two as a
        sample_batch + local_update round does: same distribution, other numbers.  Returns the n tb_info mappings; their
        values are fetched with one copy of the [n, 16] block on first access.
        Under torch.distributed with the peer transport the call is one Engine.dp_replay_steps on every rank, each rank
        drawing `batch_size` rows from its own buffer, with the same rules: host draws give the results of the n
        data-parallel rounds, device draws take one generator counter per update.  The "nccl" transport and the head-wise
        engine take the n rounds one by one."""
        eng = self.networks.engine(batch_size)
        dist, world = self._world()
        keys = list(zip(STAT_KEYS, range(14)))
        if self.networks.route.engine != "mlp":
            return self._rounds(buffer, batch_size, iteration, n)
        if world == 1:
            return replay_updates_on_engine(eng, buffer, batch_size, iteration, n, self._noise, keys)
        if not self._peers(eng, dist):
            return self._rounds(buffer, batch_size, iteration, n)
        return replay_updates_on_engine(eng, buffer, batch_size, iteration, n, self._noise, keys,
                                        global_batch=batch_size * world)

    def _rounds(self, buffer, batch_size: int, iteration: int, n: int) -> list:
        return [self.local_update(buffer.sample_batch(batch_size), iteration + k) for k in range(n)]

    def get_remote_update_info(self, data: Dict, iteration: int) -> Tuple[dict, dict]:
        t0 = time.time()
        eng = self.networks.engine(data["obs"].shape[0])
        gb = self._gradients(data, eng)
        g = self.networks.grad_views()
        update_info = {"q1_grad": g["q1"], "q2_grad": g["q2"], "policy_grad": g["policy"], "iteration": iteration}
        if self.auto_alpha:
            update_info["log_alpha_grad"] = g["log_alpha"]
        return self._stats(eng, gb, t0), update_info

    def remote_update(self, update_info: dict):
        eng = self.networks.engine()
        g = self.networks.grad_views()
        with torch.no_grad():
            for key, name in (("q1_grad", "q1"), ("q2_grad", "q2"), ("policy_grad", "policy")):
                for dst, src in zip(g[name], update_info[key]):
                    if src.data_ptr() != dst.data_ptr():
                        dst.copy_(src)
            if self.auto_alpha and update_info["log_alpha_grad"].data_ptr() != g["log_alpha"].data_ptr():
                g["log_alpha"].copy_(update_info["log_alpha_grad"])
        eng.apply(update_info["iteration"])
