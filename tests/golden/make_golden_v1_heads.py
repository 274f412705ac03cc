#!/usr/bin/env python
"""Generate the DSAC_V1 golden vectors on the reference's other networks by running the UNMODIFIED reference.

    python tests/golden/make_golden_v1_heads.py [case name ...]

With names, only those cases are (re)generated.  Each case runs `make_golden.run_case` (the reference's `DSAC_V1`, the
noise feed, the recorded tb_info / digests / states) unchanged.  What differs is the weights: run_case loads the V1 schema
through `synth.make_weights_v1` (MLP, "mlp_shared") and `synth.make_cnn_weights` (CNN, DSAC-T schema), so for these cases
both builders answer with the case's V1-schema weights: `synth.make_cnn_weights_v1` for the CNN networks,
`synth.make_weights_std_v1` for the policy std types, `synth.make_weights_v1` otherwise.
"""
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden  # noqa: E402  (imports the reference from DSAC_REFERENCE)

synth = make_golden.synth

# name, config, batch, steps, full-state snapshot steps, hyper overrides (as make_golden.CASES)
CASES = [
    # the reference's DSAC_V1 CarRacing example (example_train/dsacv1_cnn_carracing_offasync.py: type_2, 3x96x96); digests only
    ("v1_cnn_carracing_b4", "carracing", 4, 6, (), {"algorithm": "DSAC_V1"}),
    ("v1_cnn_type1_b5", "small_t1", 5, 4, (), {"algorithm": "DSAC_V1"}),   # type_1 encoder (8x8 stride 4 first layer)
    # the policy's other std types (networks/mlp.py:42-72): two policy heads / a learnable log_std row
    ("v1_std_separated", "tiny", 16, 10, (10,), {"algorithm": "DSAC_V1", "policy_std_type": "mlp_separated"}),
    ("v1_std_parameter", "tiny", 16, 10, (10,), {"algorithm": "DSAC_V1", "policy_std_type": "parameter"}),
    # the plain Gaussian action distribution (utils/act_distribution_cls.py:82-116)
    ("v1_tiny_gauss", "tiny", 16, 8, (8,), {"algorithm": "DSAC_V1", "policy_act_distribution": "GaussDistribution"}),
    # act_dim 1: the logged policy_std = logits[..., 1] is the std itself (dsac_v1.py:142-143); digests only
    ("v1_pendulum_b64", "pendulum", 64, 10, (), {"algorithm": "DSAC_V1"}),
]


def v1_weights(cfg_name, over):
    if cfg_name in synth.CNN_CONFIGS:
        return synth.make_cnn_weights_v1(synth.CNN_CONFIGS[cfg_name])
    cfg, std_type = synth.CONFIGS[cfg_name], over.get("policy_std_type", "mlp_shared")
    return synth.make_weights_v1(cfg) if std_type == "mlp_shared" else synth.make_weights_std_v1(cfg, std_type)


def run_case(name, cfg_name, batch, steps, snaps, over):
    w = v1_weights(cfg_name, over)
    proxy = types.ModuleType("synth_v1")
    proxy.__dict__.update(synth.__dict__)
    proxy.make_weights_v1 = proxy.make_cnn_weights = lambda cfg: w
    make_golden.synth = proxy
    try:
        make_golden.run_case(name, cfg_name, batch, steps, snaps, over)
    finally:
        make_golden.synth = synth


if __name__ == "__main__":
    make_golden.torch.set_num_threads(4)
    only = set(sys.argv[1:])
    for case in CASES:
        if not only or case[0] in only:
            run_case(*case)
