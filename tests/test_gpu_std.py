"""The policy's other std types (reference networks/mlp.py:43-72: "mlp_separated" = two MLPs, "parameter" = mean MLP +
learnable log_std row) through the C ABI: the head-wise fp32 engine (`dsact_cnn_create` with no encoder, one two-output head
per critic) against the goldens produced by the unmodified reference (tests/golden/tiny_std_*.npz), against the pinned
oracle on a ragged batch with gradients, and through the drop-in `DSAC_V2` (state_dict schema, `local_update`)."""
import ast
import os

import numpy as np
import pytest
import torch

from dsac_v2_b200 import synth

pytestmark = pytest.mark.gpu
RTOL = 1e-4


def make_engine(cfg, batch, std_type, act="gelu"):
    from dsac_v2_b200.engine_cnn import CnnEngine, make_heads_config
    h = synth.HYPER
    c = make_heads_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], std_type, max_batch=batch, act_hidden=act,
                          gamma=h["gamma"], tau=h["tau"], delay_update=h["delay_update"], auto_alpha=h["auto_alpha"], alpha=h["alpha"],
                          lr_q=h["value_learning_rate"], lr_pi=h["policy_learning_rate"], lr_alpha=h["alpha_learning_rate"],
                          min_log_std=h["policy_min_log_std"], max_log_std=h["policy_max_log_std"])
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    eng = CnnEngine(c, torch.device("cuda", 0), lim, -lim)
    eng.load_weights(synth.make_weights_std(cfg, std_type))
    return eng


def feed(cfg, batch, it):
    b = {k: torch.from_numpy(v).cuda() for k, v in synth.make_batch(cfg, batch, it).items()}
    n = synth.make_noise(cfg, batch, it)
    return b, tuple(torch.from_numpy(n[i]).cuda() for i in (0, 1, 4, 5))


@pytest.mark.parametrize("name", ["tiny_std_separated", "tiny_std_parameter"])
def test_std_type_update_matches_reference_golden(golden_dir, name):
    from dsac_v2_b200.engine import STAT_KEYS
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg_name, batch, steps, over = z["meta"]
    cfg, batch, steps = synth.CONFIGS[str(cfg_name)], int(batch), int(steps)
    std_type = dict(ast.literal_eval(str(over)))["policy_std_type"]
    eng = make_engine(cfg, batch, std_type)
    names = [str(n) for n in z["param_names"]]
    for it in range(steps):
        b, n = feed(cfg, batch, it)
        eng.step(b, it, n)
        s = eng.read_stats()
        np.testing.assert_allclose([s[k] for k in STAT_KEYS], z["tb"][it], rtol=RTOL, atol=1e-6, err_msg=f"{name} tb_info at step {it}")
        if f"pdigest_{it + 1}" in z:
            w = eng.export_weights()
            for row, k in zip(z[f"pdigest_{it + 1}"], names):
                d = w[k].double().reshape(-1)
                np.testing.assert_allclose(d.abs().sum().item(), row[1], rtol=RTOL, err_msg=f"{name} {k} step {it + 1}")
                np.testing.assert_allclose(d[:8].numpy(), row[3:3 + min(8, d.numel())], rtol=RTOL, atol=1e-7, err_msg=f"{name} {k} step {it + 1}")
        if f"state_{it + 1}/{names[0]}" in z:
            w = eng.export_weights()
            for k in names:
                ref = z[f"state_{it + 1}/{k}"]
                np.testing.assert_allclose(w[k].numpy(), ref, rtol=RTOL, atol=1e-6 * max(1e-3, np.abs(ref).max()), err_msg=f"{name} {k} after step {it + 1}")
    eng.close()


@pytest.mark.parametrize("std_type,cfg_name,batch", [("mlp_separated", "ragged", 37), ("parameter", "ragged", 50), ("mlp_separated", "tiny", 1)])
def test_std_type_update_matches_oracle(std_type, cfg_name, batch):
    """Ragged widths and batches, full post-update state and the gradients of the last step against the pinned oracle."""
    from dsac_v2_b200.engine import STAT_KEYS
    from oracle.dsact_oracle import TB_KEYS, std_from_config
    cfg = synth.CONFIGS[cfg_name]
    eng = make_engine(cfg, batch, std_type)
    orc = std_from_config(cfg, synth.make_weights_std(cfg, std_type), std_type, **synth.HYPER)
    assert STAT_KEYS == TB_KEYS
    for it in range(4):
        ref = orc.update(synth.make_batch(cfg, batch, it), synth.make_noise(cfg, batch, it), it)
        b, n = feed(cfg, batch, it)
        eng.step(b, it, n)
        s = eng.read_stats()
        np.testing.assert_allclose([s[k] for k in TB_KEYS], [ref[k] for k in TB_KEYS], rtol=RTOL, atol=1e-6, err_msg=f"step {it}")
    g, gref = eng.export_weights(grads=True), orc.grad_dict()
    for k, v in gref.items():
        np.testing.assert_allclose(g[k].numpy(), v.numpy(), rtol=1e-3, atol=2e-6 * float(v.abs().max()) + 1e-12, err_msg=f"grad {k}")
    w, sd = eng.export_weights(), orc.state_dict()
    for k, v in sd.items():
        np.testing.assert_allclose(w[k].numpy(), v.numpy(), rtol=RTOL, atol=1e-5, err_msg=k)
    eng.close()


@pytest.mark.parametrize("std_type", ["mlp_separated", "parameter"])
def test_std_type_dropin_local_update(golden_dir, std_type):
    """`dsac_v2.DSAC_V2(policy_std_type=...)`: the reference's state_dict keys, parameters as views of the engine's flat
    buffers in the module's own parameter order, `local_update` on the GPU."""
    import dsac_v2
    from dsac_v2_b200.engine import STAT_KEYS
    name = {"mlp_separated": "tiny_std_separated", "parameter": "tiny_std_parameter"}[std_type]
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg, B = synth.CONFIGS["tiny"], int(z["meta"][1])
    kw = synth.reference_kwargs(cfg, policy_std_type=std_type, replay_batch_size=B)
    alg = dsac_v2.DSAC_V2(**kw)
    sd = alg.networks.state_dict()
    ref_w = synth.make_weights_std(cfg, std_type)
    assert {k for k in sd if not k.endswith("_lim")} == set(ref_w) | {"log_alpha"}
    assert [k for k, _ in alg.networks.named_parameters()] == [str(n) for n in z["param_names"]]   # the reference's order
    for k, v in ref_w.items():
        sd[k] = torch.from_numpy(v)
    alg.networks.load_state_dict(sd)
    alg.networks.cuda()
    eng = alg.networks.engine(B)
    for it in range(3):
        b, n = feed(cfg, B, it)
        eng.step(b, it, n)
        s = eng.read_stats()
        np.testing.assert_allclose([s[k] for k in STAT_KEYS], z["tb"][it], rtol=RTOL, atol=1e-6)
    key = "policy.log_std" if std_type == "parameter" else "policy.log_std.0.weight"
    assert not torch.equal(alg.networks.state_dict()[key].cpu(), torch.from_numpy(ref_w[key]))   # views: the module sees the update
    tb = alg.local_update(feed(cfg, B, 7)[0], 3)
    assert np.isfinite(tb["Loss/Critic loss-RL iter"]) and np.isfinite(tb["Loss/Actor loss-RL iter"])
    # the CPU-side forward of the module (sampler / evaluator) agrees with the engine's view of the weights
    obs = torch.from_numpy(synth.make_batch(cfg, B, 0)["obs"])
    import copy
    out = copy.deepcopy(alg.networks.policy).cpu()(obs)
    assert out.shape == (B, 2 * cfg["act_dim"]) and torch.isfinite(out).all()


def test_gauss_distribution_dropin(golden_dir):
    """`policy_act_distribution="GaussDistribution"` (reference utils/act_distribution_cls.py:82-116) through the drop-in:
    the engine samples without squashing; tb_info follows the reference golden (the engine-level parity of this case, fp32
    and bf16x3, is in test_gpu_parity.py)."""
    import dsac_v2
    from dsac_v2_b200.engine import STAT_KEYS
    z = np.load(os.path.join(golden_dir, "tiny_gauss.npz"))
    cfg, B = synth.CONFIGS["tiny"], int(z["meta"][1])
    kw = synth.reference_kwargs(cfg, policy_act_distribution="GaussDistribution", replay_batch_size=B, dsact_gemm="fp32")
    alg = dsac_v2.DSAC_V2(**kw)
    sd = alg.networks.state_dict()
    for k, v in synth.make_weights(cfg).items():
        sd[k] = torch.from_numpy(v)
    alg.networks.load_state_dict(sd)
    alg.networks.cuda()
    eng = alg.networks.engine(B)
    assert eng.cfg.act_dist == 1
    for it in range(3):
        b = {k: torch.from_numpy(v).cuda() for k, v in synth.make_batch(cfg, B, it).items()}
        n = synth.make_noise(cfg, B, it)
        eng.step(b, it, tuple(torch.from_numpy(n[i]).cuda() for i in (0, 1, 4, 5)))
        s = eng.read_stats()
        np.testing.assert_allclose([s[k] for k in STAT_KEYS], z["tb"][it], rtol=RTOL, atol=1e-6)
    # the host-side distribution the sampler acts with is the plain Gaussian too
    dist = alg.networks.create_action_distributions(torch.zeros(2, 2 * cfg["act_dim"]).add_(0.5))
    assert type(dist).__name__ == "GaussDistribution"
