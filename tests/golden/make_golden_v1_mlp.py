#!/usr/bin/env python
"""Generate the DSAC_V1 golden vectors of the MLP engine's shapes by running the UNMODIFIED reference.

    python tests/golden/make_golden_v1_mlp.py [case name ...]

With names, only those cases are (re)generated.  Each case runs `make_golden.run_case` (the reference's `DSAC_V1`, the
noise feed, the recorded tb_info / digests / states) unchanged, with `synth.make_weights_v1` weights: critics and policy
of different depths, widths and activations (`synth.ASYM_CONFIGS`), and the shape of the reference's Hopper example
(`synth.EXAMPLE_CONFIGS["hopper"]`, example_train/dsacv1_mlp_hopper_offserial.py: 256x3 GELU, TD_bound 10, gamma 0.999,
batch 256).  Digests only, the full state for the smallest case.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden  # noqa: E402  (imports the reference from DSAC_REFERENCE)

synth = make_golden.synth

# name, config, batch, steps, full-state snapshot steps, hyper overrides (as make_golden.CASES)
CASES = [
    (f"v1_{cfg}_b70", cfg, 70, 10, (1,) if cfg == "layered_q" else (), {"algorithm": "DSAC_V1"}) for cfg in synth.ASYM_CONFIGS
] + [
    ("v1_hopper_b256", "hopper", 256, 10, (), {"algorithm": "DSAC_V1", "TD_bound": 10.0, "gamma": 0.999}),
]


if __name__ == "__main__":
    make_golden.torch.set_num_threads(4)
    only = set(sys.argv[1:])
    for case in CASES:
        if not only or case[0] in only:
            make_golden.run_case(*case)
