"""Pin the CPU oracle to the reference: fixtures in tests/golden/*.npz were
produced by the unmodified reference (tests/golden/make_golden.py)."""
import ast
import os

import numpy as np
import pytest
import torch

from dsac_v2_b200 import synth
from oracle.dsact_oracle import TB_KEYS, V1_TB_KEYS, cnn_from_config, from_config, std_from_config, v1_from_config

CASES = ["tiny_b16", "ragged_b37", "tiny_fixed_alpha", "pendulum_b256", "halfcheetah_b512",
         "humanoid_b256", "humanoid_b4096",
         # the reference's other hidden activations (utils/common_utils.py:16-43)
         "tiny_relu", "tiny_tanh", "ragged_elu", "ragged_selu", "tiny_sigmoid", "tiny_gauss",
         # the policy's other std types (oracle-level groundwork for SURVEY.md 8f rank 4)
         "tiny_std_separated", "tiny_std_parameter",
         # CNN approximators (BASELINE config 5; oracle-level groundwork for SURVEY.md 8f rank 1)
         "cnn_carracing_b4", "cnn_type1_b5", "v1_tiny_b16", "v1_ragged_tight", "v1_tiny_nll",
         # critics and policy of different depths, widths and activations (synth.ASYM_CONFIGS)
         "asym_b70", "deep_pi_b70", "layered_pi_b70", "layered_q_b70"]
MAX_STEPS = {"humanoid_b256": 100, "pendulum_b256": 100}


def load(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg_name, batch, steps, over = z["meta"]
    cfg = synth.CNN_CONFIGS[str(cfg_name)] if str(cfg_name) in synth.CNN_CONFIGS else synth.mlp_config(str(cfg_name))
    return z, cfg, int(batch), int(steps), dict(ast.literal_eval(str(over)))


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference(golden_dir, name):
    torch.set_num_threads(4)
    z, cfg, batch, steps, over = load(golden_dir, name)
    v1 = over.get("algorithm") == "DSAC_V1"   # the older algorithm (dsac_v1.py): its own oracle class and tb_info keys
    tb_keys = V1_TB_KEYS if v1 else TB_KEYS
    assert list(z["tb_keys"]) == tb_keys
    hyper = dict(synth.HYPER)
    hyper.update(over)
    hyper.pop("algorithm", None)
    cnn = "conv_type" in cfg
    std_type = hyper.pop("policy_std_type", "mlp_shared")
    if v1:
        orc = v1_from_config(cfg, synth.make_weights_v1(cfg), **hyper)
    elif std_type != "mlp_shared":
        orc = std_from_config(cfg, synth.make_weights_std(cfg, std_type), std_type, **hyper)
    elif cnn:
        orc = cnn_from_config(cfg, synth.make_cnn_weights(cfg), **hyper)
    else:
        orc = from_config(cfg, synth.make_weights(cfg), **hyper)
    make_batch = synth.make_cnn_batch if cnn else synth.make_batch
    names = [str(n) for n in z["param_names"]]
    trainable = [str(n) for n in z["trainable_names"]]
    for it in range(steps):
        tb = orc.update(make_batch(cfg, batch, it), synth.make_noise(cfg, batch, it), it)
        got = np.array([tb[k] for k in tb_keys])
        # same ATen ops in the same order: expect (near) bitwise agreement
        np.testing.assert_allclose(got, z["tb"][it], rtol=2e-6, atol=1e-7, err_msg=f"{name} step {it}")
        sd = orc.state_dict()
        if f"pdigest_{it + 1}" in z:
            dig = z[f"pdigest_{it + 1}"]
            for row, k in zip(dig, names):
                d = sd[k].double().reshape(-1)
                # digest = (sum, abs-sum, sq-sum, first 8 entries); the plain sum cancels, so scale its atol
                np.testing.assert_allclose(d.sum().item(), row[0], rtol=1e-6, atol=1e-7 * row[1] + 1e-9,
                                           err_msg=f"{name} {k} after step {it + 1}")
                np.testing.assert_allclose(d.abs().sum().item(), row[1], rtol=1e-6, atol=1e-9,
                                           err_msg=f"{name} {k} after step {it + 1}")
                np.testing.assert_allclose(d[:8].numpy(), row[3:3 + min(8, d.numel())], rtol=1e-5, atol=1e-8,
                                           err_msg=f"{name} {k} after step {it + 1}")
        if it in (0, 1) and f"gdigest_{it}" in z:
            gd = orc.grad_dict()
            for row, k in zip(z[f"gdigest_{it}"], trainable):
                if k in gd:
                    d = gd[k].double().reshape(-1)
                    np.testing.assert_allclose(d.abs().sum().item(), row[1], rtol=1e-5, atol=1e-9,
                                               err_msg=f"{name} grad {k} step {it}")
        if f"state_{it + 1}/{names[0]}" in z:
            for k in names:
                np.testing.assert_allclose(sd[k].numpy(), z[f"state_{it + 1}/{k}"], rtol=1e-6, atol=1e-8,
                                           err_msg=f"{name} {k} after step {it + 1}")
            gd = orc.grad_dict()
            for k in trainable:
                if f"grad_{it}/{k}" in z:
                    ref = z[f"grad_{it}/{k}"]
                    np.testing.assert_allclose(gd[k].numpy(), ref, rtol=1e-5, atol=1e-6 * np.abs(ref).max(),
                                               err_msg=f"{name} grad {k} step {it}")


def test_oracle_fp64_close_to_fp32(golden_dir):
    """fp32 round-off of the path is ~1e-6, two orders below the 1e-4 parity gate."""
    z, cfg, batch, steps, over = load(golden_dir, "tiny_b16")
    orc = from_config(cfg, synth.make_weights(cfg), dtype=torch.float64, **synth.HYPER)
    for it in range(steps):
        tb = orc.update(synth.make_batch(cfg, batch, it), synth.make_noise(cfg, batch, it), it)
        got = np.array([tb[k] for k in TB_KEYS])
        np.testing.assert_allclose(got, z["tb"][it], rtol=5e-5, atol=1e-6)
