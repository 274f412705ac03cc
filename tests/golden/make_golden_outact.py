#!/usr/bin/env python
"""Generate golden vectors for non-linear output activations by running the UNMODIFIED reference.

    python tests/golden/make_golden_outact.py [case name ...]

The reference's networks pass `value_output_activation` / `policy_output_activation` to their last layer (networks/mlp.py,
networks/cnn.py).  Each case runs `make_golden.run_case` (DSAC_V2) or `make_golden_v1_heads.run_case` (DSAC_V1, any
network) unchanged, with the two activations among the case's overrides: the same weights, minibatches, noise feed and
recorded tb_info / digests / states as the linear fixtures.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden  # noqa: E402  (imports the reference from DSAC_REFERENCE)
import make_golden_v1_heads  # noqa: E402


def acts(q, pi):
    return {"value_output_activation": q, "policy_output_activation": pi}


V1 = {"algorithm": "DSAC_V1"}

# name, config, batch, steps, full-state snapshot steps, hyper overrides (as make_golden.CASES)
CASES = [
    ("outact_tiny_tanh", "tiny", 16, 12, (1, 12), acts("tanh", "tanh")),
    # a kink: relu on the policy, whose log_std half sits at 0 for every negative pre-activation
    ("outact_tiny_relu_pi", "tiny", 16, 10, (10,), acts("linear", "relu")),
    # saturation: sigmoid on the critics (the std column is softplus(sigmoid(z)))
    ("outact_ragged_sigmoid_q", "ragged", 37, 10, (10,), acts("sigmoid", "linear")),
    ("outact_std_separated", "tiny", 16, 10, (10,), dict(acts("gelu", "tanh"), policy_std_type="mlp_separated")),
    # "parameter": the learnable log_std row is not activated
    ("outact_std_parameter", "tiny", 16, 10, (10,), dict(acts("tanh", "elu"), policy_std_type="parameter")),
    ("outact_gauss", "tiny", 16, 10, (10,), dict(acts("tanh", "tanh"), policy_act_distribution="GaussDistribution")),
    ("outact_cnn_type1", "small_t1", 5, 4, (), acts("tanh", "tanh")),
    # DSAC_V1: bounded loss (MLP engine and head-wise engine), a separated policy (head-wise engine), CNN
    ("outact_v1_tiny", "tiny", 16, 10, (10,), dict(V1, **acts("tanh", "tanh"))),
    ("outact_v1_std_separated", "tiny", 16, 8, (8,), dict(V1, policy_std_type="mlp_separated", **acts("selu", "tanh"))),
    ("outact_v1_cnn_type1", "small_t1", 5, 4, (), dict(V1, **acts("tanh", "tanh"))),
]


if __name__ == "__main__":
    make_golden.torch.set_num_threads(4)
    only = set(sys.argv[1:])
    for case in CASES:
        if not only or case[0] in only:
            run = make_golden_v1_heads.run_case if case[5].get("algorithm") == "DSAC_V1" else make_golden.run_case
            run(*case)
