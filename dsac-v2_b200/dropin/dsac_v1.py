"""`dsac_v1` of the drop-in: `ApproxContainer` and `DSAC_V1` with the reference's names, kwargs and `tb_info` keys
(reference dsac_v1.py:17-52, 56-273) — the older algorithm (one distributional critic, fixed TD bound; selectable with
`--algorithm DSAC_V1`), backed by libdsact.so: by default the head-wise fp32 engine (`dsact_cnn_create` with `algo = 1`);
with `dsact_gemm` the MLP engine (`dsact_v1_create`: wgmma layer chains or fp32 SIMT GEMMs, captured steps).

* `ApproxContainer`: `q`, `q_target`, `policy`, `policy_target` (the same `networks.mlp` / `networks.cnn` classes as
  DSAC-T) + `log_alpha`; on a CUDA device the parameters are views into the engine's flat buffers [q | policy | log_alpha].
  Approximators: MLP with policy std_type "mlp_shared" / "mlp_separated" / "parameter", or CNN (`type_1` / `type_2`,
  one conv_type for both networks, as in example_train/dsacv1_cnn_carracing_offasync.py).
  `value_output_activation` / `policy_output_activation` end the networks as in the reference, on either engine.
* `DSAC_V1.local_update(data, iteration) -> tb_info` runs the whole update in the CUDA library; no CPU fallback.
  `get_remote_update_info` / `remote_update` (the gradient-message seam of the reference's asynchronous trainers) are not
  part of this engine and raise.
* `full_state_dict` / `load_full_state_dict`: weights, Adam moments and counters, the device generator's state, in the
  "dsact-full-state-1" format of `dsac_v2.DSAC_V2` (what `OffSerialTrainer` writes with `dsact_full_checkpoint`).

Extra kwargs: `dsact_noise` = "device" (default) | "reference" (draw eps1, eps2 and the three z's of one update from torch's
CPU generator in the reference's order), `dsact_max_batch`, `seed`.
`dsact_gemm` = "fp32" | "bf16x3" | "bf16" (as in `dsac_v2`) selects the MLP engine in that arithmetic, and `dsact_graph`
(default True) its captured steps.  It takes MLP approximators with the policy std_type "mlp_shared" (critic and policy may
then differ in hidden_sizes and activation); any other approximator raises NotImplementedError with `dsact_gemm`.  Without
`dsact_gemm` every configuration runs on the head-wise fp32 engine.
"""
__all__ = ["ApproxContainer", "DSAC_V1"]

import time
from copy import deepcopy
from typing import Dict

import torch
import torch.nn as nn

from dsact_host import TB_TAGS as tb_tags
from dsact_host import full_state_dict as _full_state
from dsact_host import load_full_state_dict as _load_full_state
from dsact_host import replay_updates_on_engine
from dsact_route import EngineContainer, network_classes

# where the engine's 16-slot statistics carry DSAC_V1's tb_info (dsac_v1.py:172-181)
_V1_KEYS = (("DSAC/critic_avg_q-RL iter", 0), ("DSAC/critic_avg_std-RL iter", 2), (tb_tags["loss_actor"], 6),
            ("DSAC/policy_mean-RL iter", 8), ("DSAC/policy_std-RL iter", 9), ("DSAC/entropy-RL iter", 10),
            ("DSAC/alpha-RL iter", 11))


class ApproxContainer(EngineContainer):
    """One critic, one policy, their targets and log_alpha (reference dsac_v1.py:17-52)."""

    algorithm, critics = "DSAC_V1", ("q",)

    def __init__(self, **kwargs):
        super().__init__()
        q_args, pi_args, q_cls, pi_cls = network_classes(self.algorithm, kwargs)
        self.q = q_cls(**q_args)                      # construction order = the reference's RNG consumption (:28-34)
        self.q_target = deepcopy(self.q)
        self.policy = pi_cls(**pi_args)
        self.policy_target = deepcopy(self.policy)
        for net in (self.policy_target, self.q_target):
            for p in net.parameters():
                p.requires_grad = False
        self.log_alpha = nn.Parameter(torch.tensor(1, dtype=torch.float32))
        self._route(kwargs)


class DSAC_V1:
    """DSAC (IEEE TNNLS 2021) on the CUDA engine; interface of reference dsac_v1.py:56-135."""

    def __init__(self, **kwargs):
        self.networks = ApproxContainer(**kwargs)
        self.gamma = kwargs["gamma"]
        self.tau = kwargs["tau"]
        self.target_entropy = -kwargs["action_dim"]
        self.auto_alpha = kwargs["auto_alpha"]
        self.alpha = kwargs.get("alpha", 0.2)
        self.TD_bound = kwargs.get("TD_bound", 20)
        self.bound = kwargs.get("bound", True)
        self.delay_update = kwargs["delay_update"]
        self.act_dim = kwargs["action_dim"]
        self.noise_source = kwargs.get("dsact_noise", "device")
        if self.noise_source not in ("device", "reference"):
            raise ValueError("dsact_noise must be 'device' or 'reference'")

    @property
    def adjustable_parameters(self):
        return ("gamma", "tau", "auto_alpha", "alpha", "TD_bound", "bound", "delay_update")

    def _noise(self, batch: int):
        if self.noise_source == "device":
            return None
        A = self.act_dim
        eps1 = torch.empty(batch, A).normal_()   # rsample of pi(obs),         reference :147
        eps2 = torch.empty(batch, A).normal_()   # rsample of pi_target(obs2),  reference :205
        z = [torch.normal(torch.zeros(batch), torch.ones(batch)) for _ in range(3)]   # __q_evaluate x3 (:207-210, :245)
        return eps1, eps2, z[1], z[1]            # only the target critic's draw enters the update

    def local_update(self, data: Dict, iteration: int) -> dict:
        t0 = time.time()
        B = data["obs"].shape[0]
        eng = self.networks.engine(B)
        eng.step(data, iteration, self._noise(B))
        s = eng.read_stats(B)
        vals = list(s.values())
        tb = {k: vals[i] for k, i in _V1_KEYS}
        tb[tb_tags["alg_time"]] = (time.time() - t0) * 1000
        return tb

    def replay_updates(self, buffer, batch_size: int, iteration: int, n: int) -> list:
        """n rounds of `local_update(buffer.sample_batch(batch_size), iteration + k)`, k = 0 .. n-1, as ONE engine call
        (Engine.replay_steps) on the MLP engine: the same host draws in the same order, the same results.  Returns the n
        tb_info mappings, fetched with one copy of the [n, 16] block on first access.  The head-wise engine takes the n
        rounds one by one."""
        eng = self.networks.engine(batch_size)
        if self.networks.route.engine != "mlp":
            return [self.local_update(buffer.sample_batch(batch_size), iteration + k) for k in range(n)]
        return replay_updates_on_engine(eng, buffer, batch_size, iteration, n, self._noise, _V1_KEYS)

    # ---- full training state (the reference saves weights only, training/trainer.py:137-152) ----
    def full_state_dict(self) -> dict:
        """Everything a bit-for-bit resume needs beyond `networks.state_dict()`: Adam moments and step counters, the
        device generator's seed/counter."""
        return _full_state(self.networks)

    def load_full_state_dict(self, state: dict) -> None:
        _load_full_state(self.networks, state)

    def get_remote_update_info(self, data: Dict, iteration: int):
        raise NotImplementedError("DSAC_V1 on the CUDA engine: local_update only (no gradient-message seam)")

    def remote_update(self, update_info: dict):
        raise NotImplementedError("DSAC_V1 on the CUDA engine: local_update only (no gradient-message seam)")
