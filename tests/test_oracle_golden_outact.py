"""Pin the output-activation oracles (tests/outact_oracle.py) to the reference: fixtures tests/golden/outact_*.npz were
produced by the unmodified reference (tests/golden/make_golden_outact.py).  Tolerances as tests/test_oracle_golden.py."""
import numpy as np
import pytest
import torch

import outact_oracle
from dsac_v2_b200 import synth
from oracle.dsact_oracle import TB_KEYS, V1_TB_KEYS
from test_oracle_golden import load

CASES = ["outact_tiny_tanh", "outact_tiny_relu_pi", "outact_ragged_sigmoid_q", "outact_std_separated", "outact_std_parameter",
         "outact_gauss", "outact_cnn_type1", "outact_v1_tiny", "outact_v1_std_separated", "outact_v1_cnn_type1"]


@pytest.mark.parametrize("name", CASES)
def test_outact_oracle_matches_reference(golden_dir, name):
    torch.set_num_threads(4)
    z, cfg, batch, steps, over = load(golden_dir, name)
    assert over["value_output_activation"] != "linear" or over["policy_output_activation"] != "linear"
    tb_keys = V1_TB_KEYS if over.get("algorithm") == "DSAC_V1" else TB_KEYS
    assert list(z["tb_keys"]) == tb_keys
    orc, _ = outact_oracle.build(cfg, over)
    make_batch = synth.make_cnn_batch if "conv_type" in cfg else synth.make_batch
    names = [str(n) for n in z["param_names"]]
    trainable = [str(n) for n in z["trainable_names"]]
    for it in range(steps):
        tb = orc.update(make_batch(cfg, batch, it), synth.make_noise(cfg, batch, it), it)
        np.testing.assert_allclose(np.array([tb[k] for k in tb_keys]), z["tb"][it], rtol=2e-6, atol=1e-7,
                                   err_msg=f"{name} step {it}")
        sd = orc.state_dict()
        if f"pdigest_{it + 1}" in z:
            for row, k in zip(z[f"pdigest_{it + 1}"], names):
                d = sd[k].double().reshape(-1)
                np.testing.assert_allclose(d.sum().item(), row[0], rtol=1e-6, atol=1e-7 * row[1] + 1e-9, err_msg=f"{name} {k}")
                np.testing.assert_allclose(d.abs().sum().item(), row[1], rtol=1e-6, atol=1e-9, err_msg=f"{name} {k}")
                np.testing.assert_allclose(d[:8].numpy(), row[3:3 + min(8, d.numel())], rtol=1e-5, atol=1e-8,
                                           err_msg=f"{name} {k}")
        if it in (0, 1) and f"gdigest_{it}" in z:
            gd = orc.grad_dict()
            for row, k in zip(z[f"gdigest_{it}"], trainable):
                if k in gd:
                    np.testing.assert_allclose(gd[k].double().abs().sum().item(), row[1], rtol=1e-5, atol=1e-9,
                                               err_msg=f"{name} grad {k} step {it}")
        if f"state_{it + 1}/{names[0]}" in z:
            for k in names:
                np.testing.assert_allclose(sd[k].numpy(), z[f"state_{it + 1}/{k}"], rtol=1e-6, atol=1e-8,
                                           err_msg=f"{name} {k} after step {it + 1}")


@pytest.mark.parametrize("name", ["tiny_b16", "tiny_std_parameter", "cnn_type1_b5", "v1_tiny_b16"])
def test_linear_output_activations_compute_what_the_oracle_computes(golden_dir, name):
    """With both activations linear the restated networks are the oracles' own: the linear fixtures hold at the same
    tolerance."""
    z, cfg, batch, steps, over = load(golden_dir, name)
    tb_keys = V1_TB_KEYS if over.get("algorithm") == "DSAC_V1" else TB_KEYS
    orc, _ = outact_oracle.build(cfg, over, value_output_activation="linear", policy_output_activation="linear")
    make_batch = synth.make_cnn_batch if "conv_type" in cfg else synth.make_batch
    for it in range(min(steps, 4)):
        tb = orc.update(make_batch(cfg, batch, it), synth.make_noise(cfg, batch, it), it)
        np.testing.assert_allclose(np.array([tb[k] for k in tb_keys]), z["tb"][it], rtol=2e-6, atol=1e-7,
                                   err_msg=f"{name} step {it}")
