"""Pin the DSAC_V1 oracle on the CNN approximators, the policy std types "mlp_separated" / "parameter", the plain
Gaussian and act_dim 1 to the reference: tests/golden/v1_{cnn_*,std_*,tiny_gauss,pendulum_b64}.npz were produced by the
unmodified reference (tests/golden/make_golden_v1_heads.py), at the tolerances of test_oracle_golden.py."""
import ast
import os

import numpy as np
import pytest
import torch

from dsac_v2_b200 import synth
from oracle.dsact_oracle import V1_TB_KEYS, v1_from_config
from oracle.dsact_oracle_v1_heads import v1_cnn_from_config, v1_std_from_config

CASES = ["v1_cnn_carracing_b4", "v1_cnn_type1_b5", "v1_std_separated", "v1_std_parameter", "v1_tiny_gauss", "v1_pendulum_b64"]


def v1_oracle(golden_dir, name):
    """(fixture, cfg, batch, steps, oracle built from the fixture's config and hyper-parameter overrides)."""
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg_name, batch, steps, over = z["meta"]
    over = dict(ast.literal_eval(str(over)))
    assert over.pop("algorithm") == "DSAC_V1"
    hyper = dict(synth.HYPER)
    hyper.update(over)
    std_type = hyper.pop("policy_std_type", "mlp_shared")
    if str(cfg_name) in synth.CNN_CONFIGS:
        cfg = synth.CNN_CONFIGS[str(cfg_name)]
        orc = v1_cnn_from_config(cfg, synth.make_cnn_weights_v1(cfg), **hyper)
    elif std_type != "mlp_shared":
        cfg = synth.CONFIGS[str(cfg_name)]
        orc = v1_std_from_config(cfg, synth.make_weights_std_v1(cfg, std_type), std_type, **hyper)
    else:
        cfg = synth.CONFIGS[str(cfg_name)]
        orc = v1_from_config(cfg, synth.make_weights_v1(cfg), **hyper)
    return z, cfg, int(batch), int(steps), orc


@pytest.mark.parametrize("name", CASES)
def test_v1_oracle_matches_reference(golden_dir, name):
    torch.set_num_threads(4)
    z, cfg, batch, steps, orc = v1_oracle(golden_dir, name)
    assert list(z["tb_keys"]) == V1_TB_KEYS
    names = [str(n) for n in z["param_names"]]
    trainable = [str(n) for n in z["trainable_names"]]
    assert set(names) == set(orc.state_dict())
    make_batch = synth.make_cnn_batch if "conv_type" in cfg else synth.make_batch
    for it in range(steps):
        tb = orc.update(make_batch(cfg, batch, it), synth.make_noise(cfg, batch, it), it)
        got = np.array([tb[k] for k in V1_TB_KEYS])
        np.testing.assert_allclose(got, z["tb"][it], rtol=2e-6, atol=1e-7, err_msg=f"{name} step {it}")
        sd = orc.state_dict()
        if f"pdigest_{it + 1}" in z:
            for row, k in zip(z[f"pdigest_{it + 1}"], names):
                d = sd[k].double().reshape(-1)
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

