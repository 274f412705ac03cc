"""The CPU oracles of `oracle.dsact_oracle` / `oracle.dsact_oracle_v1_heads` with the reference's output activations.

Every network of the reference passes `output_activation` to its last layer (networks/mlp.py: StochaPolicy, all three
std types, and ActionValueDistri; networks/cnn.py: every mean / log_std head), chosen by the kwargs
`value_output_activation` / `policy_output_activation` (utils/common_utils.get_activation_func, the same names as the
hidden layers).  The classes here restate `policy_logits` / `q_dist` of each oracle with that activation on the network
outputs; the update (losses, Adam, Polyak) is the oracle's own.  With both activations "linear" they compute what the
oracles compute.  Builders: `build(cfg, over)` from a golden case's config and overrides.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import dsact_oracle as O
from oracle import dsact_oracle_v1_heads as OV1


class _OutAct:
    def __init__(self, *args, value_output_activation="linear", policy_output_activation="linear", **hyper):
        self.out_q, self.out_pi = O._ACT[value_output_activation], O._ACT[policy_output_activation]
        super().__init__(*args, **hyper)


class _Mlp(_OutAct):
    def policy_logits(self, layers, obs):
        """StochaPolicy.forward, std_type "mlp_shared" (networks/mlp.py:85-100): the activation on all 2A outputs."""
        out = self.out_pi(O.mlp_forward(layers, obs, self.act_pi, self.linear))
        mean, log_std = torch.chunk(out, 2, dim=-1)
        return mean, torch.clamp(log_std, self.min_log_std, self.max_log_std).exp()

    def q_dist(self, layers, obs, act):
        """ActionValueDistri.forward (networks/mlp.py:122-127): the activation on both outputs, softplus on the std."""
        out = self.out_q(O.mlp_forward(layers, torch.cat([obs, act], dim=-1), self.act_q, self.linear))
        return out[..., 0], F.softplus(out[..., 1])


class _Std(_Mlp):
    def policy_logits(self, layers, obs):
        """std_type "mlp_separated" (both networks activated) / "parameter" (the mean network only)."""
        w = dict(zip(self.names["policy"], layers))

        def head(name):
            ls, j = [], 0
            while f"{name}.{2 * j}.weight" in w:
                ls += [w[f"{name}.{2 * j}.weight"], w[f"{name}.{2 * j}.bias"]]
                j += 1
            return self.out_pi(O.mlp_forward(ls, obs, self.act_pi, self.linear))

        mean = head("mean")
        log_std = head("log_std") if self.std_type == "mlp_separated" else w["log_std"] + torch.zeros_like(mean)
        return mean, torch.clamp(log_std, self.min_log_std, self.max_log_std).exp()


class _Cnn(_OutAct):
    def policy_logits(self, layers, obs):
        """networks/cnn.py:233-240 with the activation on both heads."""
        w = dict(zip(self.names["policy"], layers))
        f = self._features(w, obs)
        mean = self.out_pi(self._head(w, "mean", f, self.act_pi))
        log_std = self.out_pi(self._head(w, "log_std", f, self.act_pi))
        return mean, torch.clamp(log_std, self.min_log_std, self.max_log_std).exp()

    def q_dist(self, layers, obs, act):
        """networks/cnn.py:454-461 with the activation on both heads."""
        w = dict(zip(self.names["q1"], layers))
        f = torch.cat([self._features(w, obs), act], dim=-1)
        return self.out_q(self._head(w, "mean", f, self.act_q))[..., 0], \
            F.softplus(self.out_q(self._head(w, "log_std", f, self.act_q))[..., 0])


class OracleDSACT(_Mlp, O.OracleDSACT):
    pass


class OracleDSACTStd(_Std, O.OracleDSACTStd):
    pass


class OracleDSACTCNN(_Cnn, O.OracleDSACTCNN):
    pass


class OracleDSACV1(_Mlp, O.OracleDSACV1):
    pass


class OracleDSACV1Std(_Std, OV1.OracleDSACV1Std):
    pass


class OracleDSACV1CNN(_Cnn, OV1.OracleDSACV1CNN):
    pass


def build(cfg: dict, over: dict, weights=None, **extra):
    """The oracle of a golden case: `cfg` a synth config, `over` the case's overrides (the algorithm, std type and action
    distribution pick the class; the rest are hyperparameters), on `weights` (default: synth's weights of the case's
    schema).  Returns (oracle, weights)."""
    from dsac_v2_b200 import synth
    hyper = dict(synth.HYPER)
    hyper.update(over)
    hyper.update(extra)
    v1 = hyper.pop("algorithm", "DSAC_V2") == "DSAC_V1"
    std_type = hyper.pop("policy_std_type", "mlp_shared")
    lim = [cfg["act_lim"]] * cfg["act_dim"]
    lims = (lim, [-x for x in lim])
    if "conv_type" in cfg:
        w = weights if weights is not None else synth.make_cnn_weights_v1(cfg) if v1 else synth.make_cnn_weights(cfg)
        cls = OracleDSACV1CNN if v1 else OracleDSACTCNN
        return cls(cfg["obs_dim"], cfg["act_dim"], synth.CONV_TYPES[cfg["conv_type"]]["strides"], *lims, w, **hyper), w
    if "hidden_activation" not in hyper:
        act_q, act_pi = synth.activations(cfg)
        hyper = dict(dict(value_hidden_activation=act_q, policy_hidden_activation=act_pi), **hyper)
    if std_type != "mlp_shared":   # critics and policy may differ in shape (std_mlp_common.std_weights)
        from std_mlp_common import std_weights
        w = weights if weights is not None else synth.to_v1_schema(std_weights(cfg, std_type)) if v1 else std_weights(cfg, std_type)
        cls = OracleDSACV1Std if v1 else OracleDSACTStd
        return cls(cfg["obs_dim"], cfg["act_dim"], *synth.hidden_sizes(cfg), *lims, w, std_type=std_type, **hyper), w
    w = weights if weights is not None else synth.make_weights_v1(cfg) if v1 else synth.make_weights(cfg)
    cls = OracleDSACV1 if v1 else OracleDSACT
    return cls(cfg["obs_dim"], cfg["act_dim"], *synth.hidden_sizes(cfg), *lims, w, **hyper), w
