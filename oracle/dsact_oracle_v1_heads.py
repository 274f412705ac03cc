"""CPU oracle for DSAC_V1 (reference dsac_v1.py) on the reference's other networks.  TEST INFRASTRUCTURE, NOT PRODUCT;
the same import rule as `dsact_oracle` applies.

`OracleDSACV1` of `dsact_oracle` restates DSAC_V1's update (loss, target, TD bound, Adam / Polyak on
[q | policy | log_alpha]) on the MLP networks with policy std_type "mlp_shared".  The classes here run that same update on
the network code of `OracleDSACTCNN` (the CNN approximators, networks/cnn.py) and of `OracleDSACTStd` (policy std types
"mlp_separated" / "parameter", networks/mlp.py:42-100): the update comes from `OracleDSACV1`, the network pieces
(weight loading, `policy_logits`, `q_dist`, state_dict schema) from the DSAC-T class.

Parity status: PINNED on tests/golden/v1_cnn_carracing_b4.npz, v1_cnn_type1_b5.npz, v1_std_separated.npz and
v1_std_parameter.npz (tests/test_oracle_golden_v1_heads.py; fixtures from tests/golden/make_golden_v1_heads.py).
"""
from __future__ import annotations

from oracle.dsact_oracle import OracleDSACTCNN, OracleDSACTStd, OracleDSACV1


class OracleDSACV1CNN(OracleDSACV1, OracleDSACTCNN):
    """DSAC_V1 with the CNN critic `q` (ActionValueDistri) and policy (StochaPolicy) of networks/cnn.py, as in the
    reference's example_train/dsacv1_cnn_carracing_offasync.py.  Weights in the schema of `synth.make_cnn_weights_v1`."""

    state_dict = OracleDSACTCNN.state_dict
    grad_dict = OracleDSACTCNN.grad_dict

    def _load_weights(self, weights, nq, npi):
        OracleDSACTCNN._load_weights(self, weights, nq, npi)   # one entry per net of NETS = ("q", "policy")
        self.names["q1"] = self.names["q"]                     # OracleDSACTCNN.q_dist reads the critic's names under "q1"


class OracleDSACV1Std(OracleDSACV1, OracleDSACTStd):
    """DSAC_V1 with one MLP critic `q.q.*` and the policy std type "mlp_separated" / "parameter".  Weights in the schema
    of `synth.make_weights_std_v1`."""

    state_dict = OracleDSACTStd.state_dict
    grad_dict = OracleDSACTStd.grad_dict

    def _load_weights(self, weights, nq, npi):
        # OracleDSACTStd loads the twin critics `q1`, `q2` and the policy: hand it the one critic under both names and
        # keep one copy
        w = dict(weights)
        for k, v in weights.items():
            if k.startswith("q.") or k.startswith("q_target."):
                w["q1" + k[1:]] = w["q2" + k[1:]] = v
        OracleDSACTStd._load_weights(self, w, nq, npi)
        self.p = {"q": self.p["q1"], "policy": self.p["policy"]}
        self.t = {"q": self.t["q1"], "policy": self.t["policy"]}


def v1_cnn_from_config(cfg: dict, weights: dict, **hyper) -> OracleDSACV1CNN:
    """Build from a `synth.CNN_CONFIGS` entry with weights of `synth.make_cnn_weights_v1`."""
    from dsac_v2_b200.synth import CONV_TYPES
    lim = [cfg["act_lim"]] * cfg["act_dim"]
    return OracleDSACV1CNN(cfg["obs_dim"], cfg["act_dim"], CONV_TYPES[cfg["conv_type"]]["strides"], lim, [-x for x in lim],
                           weights, **hyper)


def v1_std_from_config(cfg: dict, weights: dict, std_type: str, **hyper) -> OracleDSACV1Std:
    """Build from a `synth.CONFIGS` entry with weights of `synth.make_weights_std_v1`."""
    lim = [cfg["act_lim"]] * cfg["act_dim"]
    return OracleDSACV1Std(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], lim, [-x for x in lim], weights,
                           std_type=std_type, **hyper)
