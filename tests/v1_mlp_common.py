"""Shared pieces of the DSAC_V1 tests on the MLP engine (`dsact_v1_create`): the float64-capable oracle for critics and
policy of different shapes, the golden fixtures' configurations, and the engine built from them."""
from __future__ import annotations

import ast
import os

import numpy as np

from dsac_v2_b200 import synth

# columns of the engine's 16 statistics that carry DSAC_V1's tb_info (dsac_v1.py:172-181), in V1_TB_KEYS order
V1_COLS = [0, 2, 6, 8, 9, 10, 11]
# DSAC_V1 fixtures of the reference on MLP approximators with the "mlp_shared" policy (make_golden.py,
# make_golden_v1_heads.py, make_golden_v1_mlp.py)
GOLDENS = ["v1_tiny_b16", "v1_ragged_tight", "v1_tiny_nll", "v1_tiny_gauss", "v1_pendulum_b64", "v1_asym_b70",
           "v1_deep_pi_b70", "v1_layered_pi_b70", "v1_layered_q_b70", "v1_hopper_b256"]
NEW_GOLDENS = GOLDENS[5:]


def v1_oracle(cfg: dict, weights: dict, **hyper):
    """`oracle.dsact_oracle.OracleDSACV1` with the config's own critic / policy widths and activations
    (`synth.hidden_sizes`, `synth.activations`) unless the overrides name the activations."""
    from oracle.dsact_oracle import OracleDSACV1
    lim = [cfg["act_lim"]] * cfg["act_dim"]
    if "hidden_activation" not in hyper:
        act_q, act_pi = synth.activations(cfg)
        hyper = dict(dict(value_hidden_activation=act_q, policy_hidden_activation=act_pi), **hyper)
    return OracleDSACV1(cfg["obs_dim"], cfg["act_dim"], *synth.hidden_sizes(cfg), lim, [-x for x in lim], weights, **hyper)


def golden(golden_dir: str, name: str):
    """(fixture, cfg, batch, steps, hyperparameters incl. the fixture's overrides, without `algorithm`)."""
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg_name, batch, steps, over = z["meta"]
    over = dict(ast.literal_eval(str(over)))
    assert over.pop("algorithm") == "DSAC_V1"
    hyper = dict(synth.HYPER)
    hyper.update(over)
    return z, synth.mlp_config(str(cfg_name)), int(batch), int(steps), hyper


def engine_config(cfg: dict, max_batch: int, hyper: dict, gemm: str = "fp32", graph: bool = True):
    """(dsact_config, dsact_v1_options) of a DSAC_V1 MLP-engine handle for a synth configuration."""
    from dsac_v2_b200.engine import make_config, make_v1_options
    act_q, act_pi = synth.activations(cfg)
    c = make_config(cfg["obs_dim"], cfg["act_dim"], *synth.hidden_sizes(cfg), max_batch=max_batch, act_q=act_q, act_pi=act_pi,
                    gamma=hyper["gamma"], tau=hyper["tau"], delay_update=hyper["delay_update"], auto_alpha=hyper["auto_alpha"],
                    alpha=hyper["alpha"], lr_q=hyper["value_learning_rate"], lr_pi=hyper["policy_learning_rate"],
                    lr_alpha=hyper["alpha_learning_rate"], min_log_std=hyper["policy_min_log_std"],
                    max_log_std=hyper["policy_max_log_std"], gemm_mode=gemm, use_graph=graph,
                    act_dist=hyper.get("policy_act_distribution", "TanhGaussDistribution"))
    return c, make_v1_options(hyper.get("bound", True), hyper.get("TD_bound", 20))


def make_engine(cfg: dict, max_batch: int, hyper: dict, gemm: str = "fp32", graph: bool = True, workspace_fill: float = 0.0):
    import torch
    from dsac_v2_b200.engine import Engine
    c, v1 = engine_config(cfg, max_batch, hyper, gemm, graph)
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    eng = Engine(c, torch.device("cuda", 0), lim, -lim, workspace_fill=workspace_fill, v1=v1)
    eng.load_weights(synth.make_weights_v1(cfg))
    return eng


def engine_noise(n):
    """The four noise arrays a DSAC_V1 step consumes of synth.make_noise's eight: eps1, eps2, the target critic's z (twice)."""
    return tuple(n[i] for i in (0, 1, 3, 3))
