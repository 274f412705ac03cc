"""Which engine a drop-in configuration runs on, and the `nn.Module` base of `dsac_v2.ApproxContainer` and
`dsac_v1.ApproxContainer` that owns that engine.

`route(algorithm, kwargs)` is the one place that reads the reference's kwargs to pick the engine (INTEGRATION.md §2, "Which
engine a configuration lands on"; pinned row by row by tests/test_dropin_route.py): the MLP engine (`engine.Engine`:
`dsact_create` / `dsact_v1_create`), the head-wise engine without an encoder ("heads") or with the CNN encoders ("cnn",
both `engine_cnn.CnnEngine`), and the configuration it is built from.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Optional, Tuple

import torch
import torch.nn as nn

import networks.cnn as _cnn
import networks.mlp as _mlp
from dsact_host import net_kwargs

from dsac_v2_b200 import _lib
from dsac_v2_b200.engine import Engine, make_config, make_v1_options
from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config, make_heads_config


@dataclass(frozen=True)
class Route:
    engine: str                    # "mlp" | "heads" | "cnn"
    cfg_args: dict                 # everything of the config but max_batch
    make: Callable                 # make_config | make_heads_config | make_cnn_config
    v1: Optional[_lib.V1Options]   # DSAC_V1 on the MLP engine (dsact_v1_create), else None
    out_acts: Tuple[str, str]      # (value, policy) output activations
    regrow: bool                   # engine(batch) may rebuild the engine for a batch above max_batch

    def config(self, max_batch: int):
        return self.make(max_batch=max_batch, **self.cfg_args)

    def new_engine(self, device, act_high, act_low, max_batch: int) -> Engine:
        cls = Engine if self.engine == "mlp" else CnnEngine
        return cls(self.config(max_batch), device, act_high, act_low, v1=self.v1, output_activations=self.out_acts)


def network_classes(algorithm: str, kwargs: dict):
    """(value kwargs, policy kwargs, value class, policy class): the refusals that come before the networks are built."""
    if algorithm == "DSAC_V2" and kwargs.get("cnn_shared", False):
        raise NotImplementedError("cnn_shared feature nets are not part of the CUDA update path")
    q_args, pi_args = net_kwargs("value", kwargs), net_kwargs("policy", kwargs)
    if q_args["apprfunc"] != pi_args["apprfunc"]:
        raise NotImplementedError("value and policy approximators must be of the same type (both MLP or both CNN)")
    mod = _cnn if q_args["apprfunc"] == "CNN" else _mlp
    q_cls, pi_cls = getattr(mod, q_args["name"], None), getattr(mod, pi_args["name"], None)
    if q_cls is None or pi_cls is None:
        raise NotImplementedError("This apprfunc is not properly defined")
    return q_args, pi_args, q_cls, pi_cls


def route(algorithm: str, kwargs: dict) -> Route:
    """The engine and configuration of `algorithm` ("DSAC_V2" or "DSAC_V1") for the reference's `kwargs`; raises what the
    container raises for a configuration no engine takes.  Pure: no device and no module."""
    q, pi, _, _ = network_classes(algorithm, kwargs)
    act_dist = pi["action_distribution_cls"].__name__
    if act_dist not in _lib.ACT_DISTS:
        raise NotImplementedError("the CUDA engine implements TanhGaussDistribution and GaussDistribution")
    v1, cnn, shared = algorithm == "DSAC_V1", q["apprfunc"] == "CNN", pi["std_type"] == "mlp_shared"
    same = lambda *keys: all(q[k] == pi[k] for k in keys)
    if v1:   # dsact_gemm selects the MLP engine, which takes MLP networks with the mlp_shared policy only
        gemm = kwargs.get("dsact_gemm", None)
        if gemm is not None and (cnn or not shared):
            raise NotImplementedError(
                "dsact_gemm: DSAC_V1 runs on the MLP engine with MLP approximators and the policy std_type 'mlp_shared' "
                "(TanhGaussDistribution or GaussDistribution) only; drop dsact_gemm for the head-wise fp32 engine")
        if gemm is not None and gemm not in _lib.GEMM_MODES:
            raise ValueError(f"dsact_gemm must be one of {sorted(_lib.GEMM_MODES)}, got {gemm!r}")
        engine = "mlp" if gemm is not None else "cnn" if cnn else "heads"
        if engine != "mlp" and not same("hidden_activation"):
            raise NotImplementedError("the head-wise engine takes one hidden activation for critic and policy")
        if engine == "cnn" and not same("conv_type"):
            raise NotImplementedError("the CNN engine takes one conv_type for critic and policy")
        if engine == "heads" and not same("hidden_sizes"):
            raise NotImplementedError("the head-wise engine takes one hidden_sizes list for critic and policy")
    else:    # CNN networks ignore dsact_gemm; the other std types run head-wise unless dsact_gemm names the MLP engine
        engine = "cnn" if cnn else "heads" if not shared and "dsact_gemm" not in kwargs else "mlp"
        if engine == "cnn" and not same("conv_type", "hidden_activation"):
            raise NotImplementedError("the CNN engine takes one conv_type / head activation for critics and policy")
        if engine == "heads" and not same("hidden_sizes", "hidden_activation"):
            raise NotImplementedError("policy std_type != 'mlp_shared': critics and policy take one hidden_sizes / activation")

    # the reference's hyperparameter names -> config kwargs
    args = dict(gamma=kwargs.get("gamma", 0.99), tau=kwargs.get("tau", 0.005), delay_update=kwargs.get("delay_update", 2),
                auto_alpha=kwargs.get("auto_alpha", True), alpha=kwargs.get("alpha", 0.2), lr_q=kwargs["value_learning_rate"],
                lr_pi=kwargs["policy_learning_rate"], lr_alpha=kwargs["alpha_learning_rate"], min_log_std=pi["min_log_std"],
                max_log_std=pi["max_log_std"], act_dist=act_dist)
    if not v1:   # DSAC-T's own kwarg; DSAC_V1's configs keep the default tau_b = tau
        args.update(tau_b=kwargs.get("tau_b", None))
    if engine == "mlp":
        args.update(obs_dim=q["obs_dim"], act_dim=q["act_dim"], hidden_q=q["hidden_sizes"], hidden_pi=pi["hidden_sizes"],
                    act_q=q["hidden_activation"], act_pi=pi["hidden_activation"], gemm_mode=kwargs.get("dsact_gemm", "bf16x3"),
                    use_graph=kwargs.get("dsact_graph", True), policy_std=pi["std_type"])
    elif engine == "cnn":
        t = _cnn.CONV_TYPES[q["conv_type"]]
        args.update(obs_shape=tuple(q["obs_dim"]), act_dim=q["act_dim"], kernels=t["kernels"], channels=t["channels"],
                    strides=t["strides"], hidden=t["heads"], act_hidden=q["hidden_activation"])
    else:
        args.update(obs_dim=q["obs_dim"], act_dim=q["act_dim"], hidden=q["hidden_sizes"], std_type=pi["std_type"],
                    act_hidden=q["hidden_activation"])
    bound, td_bound = kwargs.get("bound", True), kwargs.get("TD_bound", 20)
    if v1 and engine != "mlp":
        args.update(algo="DSAC_V1", bound=bound, td_bound=td_bound)
    return Route(engine, args, {"mlp": make_config, "heads": make_heads_config, "cnn": make_cnn_config}[engine],
                 make_v1_options(bound, td_bound) if v1 and engine == "mlp" else None,
                 (q["output_activation"], pi["output_activation"]), regrow=engine == "mlp" and not v1)


class EngineContainer(nn.Module):
    """The networks of one algorithm + log_alpha; on a CUDA device every parameter is a view into the flat buffers of the
    engine `self.route` picks (include/dsact.h layout).  A subclass builds its networks (the reference's order, which is
    its consumption of torch's RNG) and then calls `_route`; `critics` names its critic networks."""

    algorithm: str
    critics: Tuple[str, ...]

    # the route under the containers' earlier attribute names, read-only, for code written against them
    _cfg_args = property(lambda self: self.route.cfg_args)
    _make = property(lambda self: self.route.make)
    _cnn = property(lambda self: self.route.engine != "mlp")
    _heads_std = property(lambda self: self.route.cfg_args["std_type"] if self.route.engine == "heads" else None)

    def _route(self, kwargs: dict):
        self.route = route(self.algorithm, kwargs)
        self._max_batch = int(kwargs.get("dsact_max_batch", kwargs.get("replay_batch_size", 256)))
        self._engine = None
        self._user_seed = kwargs.get("seed", None)
        self._attachments = []   # objects holding a reference to the engine (ReplayBuffer): re-bound when the engine is rebuilt
        self._register_state_dict_hook(_detach_state_dict)

    def create_action_distributions(self, logits):
        return self.policy.get_act_dist(logits)

    def device_seed(self) -> int:
        """64-bit seed of the engine's Philox generator (noise + replay indices): the run's `seed` kwarg (reference
        utils/init_args.py seeds torch / numpy with it)."""
        return 0x5DEECE66D if self._user_seed is None else int(self._user_seed)

    # ---- flat-buffer plumbing -----------------------------------------------------
    def _flat_groups(self):
        """(trainable parameters, target parameters), each in layout order."""
        nets = self.critics + ("policy",)
        train = [p for n in nets for p in getattr(self, n).parameters()] + [self.log_alpha]
        targ = [p for n in nets for p in getattr(self, n + "_target").parameters()]
        return train, targ

    def _apply(self, fn, recurse=True):
        super()._apply(fn, recurse)
        if self.log_alpha.device.type == "cuda":
            self._attach(self.log_alpha.device)
        return self

    def _attach(self, device):
        """Make every parameter a view into the engine's flat buffers on `device`."""
        eng = self._engine
        if eng is not None and eng.device != torch.device(device):
            self._engine = eng = None  # moved to another GPU: rebuild there
        if eng is None:
            eng = self._engine = self.route.new_engine(device, self.policy.act_high_lim, self.policy.act_low_lim, self._max_batch)
            eng.seed(self.device_seed())
        train, targ = self._flat_groups()
        with torch.no_grad():
            for flat, group in ((eng.params, train), (eng.targets, targ)):
                off = 0
                for p in group:
                    n = p.numel()
                    view = flat[off:off + n].view(p.shape)
                    if p.data.data_ptr() != view.data_ptr():
                        view.copy_(p.data)
                        p.data = view
                    off += n
                assert off == flat.numel(), "flat layout does not match the module"

    def engine(self, batch: int = 0) -> Engine:
        """The bound engine; raises when the module is not on a CUDA device."""
        if self.log_alpha.device.type != "cuda" or self._engine is None:
            raise _lib.DsactError(
                f"{self.algorithm}'s update path runs only on the CUDA engine (libdsact.so, sm_90a); "
                "move the networks to the GPU first (`alg.networks.cuda()`). There is no CPU fallback.")
        if batch > self._max_batch and not self.route.regrow:
            why = " (the CNN engine does not regrow)" if self.algorithm == "DSAC_V2" else ""
            raise ValueError(f"batch {batch} > dsact_max_batch / replay_batch_size {self._max_batch}{why}")
        if batch > self._max_batch:  # grow the activation arena, keep weights / Adam state / carry
            old = self._engine
            self._max_batch = int(batch)
            new = self.route.new_engine(old.device, self.policy.act_high_lim, self.policy.act_low_lim, self._max_batch)
            with torch.no_grad():
                for name in ("params", "targets", "adam_m", "adam_v", "state"):
                    getattr(new, name).copy_(getattr(old, name))
            new.seed(old._seed)            # a seed restored by load_full_state_dict survives the rebuild
            self._engine = new
            for p in self.parameters():  # force re-pointing
                p.data = p.data.clone()
            self._attach(old.device)
            for ref in list(self._attachments):   # replay rings move with their rows; peers reconnect on the next update
                obj = ref()
                if obj is not None:
                    obj.rebind(old, new)
            old.close()
        return self._engine

    def grad_views(self):
        """Per-parameter views of the flat gradient buffer, grouped like get_remote_update_info."""
        eng = self.engine()
        out, off = {}, 0
        for name in self.critics + ("policy",):
            views = []
            for p in getattr(self, name).parameters():
                views.append(eng.grads[off:off + p.numel()].view(p.shape))
                off += p.numel()
            out[name] = views
        out["log_alpha"] = eng.grads[off]
        return out


def _detach_state_dict(module, state_dict, prefix, local_metadata):
    # checkpoints must not alias the flat buffers (torch.save would serialise the whole storage per view)
    for k, v in list(state_dict.items()):
        if isinstance(v, torch.Tensor):
            state_dict[k] = v.detach().clone()
    return state_dict
