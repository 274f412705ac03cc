"""The CUDA update path, called through the C ABI, against (a) golden vectors produced by the
unmodified reference and (b) the CPU oracle on the same seeded inputs.

Tolerance: north_star asks for 1e-4 relative on the first 100 losses; fp32 kernels land ~1e-6."""
import ast
import os

import numpy as np
import pytest
import torch

from dsac_v2_b200 import synth

pytestmark = pytest.mark.gpu

RTOL = 1e-4


def load(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg_name, batch, steps, over = z["meta"]
    return z, synth.mlp_config(str(cfg_name)), int(batch), int(steps), dict(ast.literal_eval(str(over)))


def make_engine(cfg, batch, over=None, **kw):
    from dsac_v2_b200.engine import Engine, make_config
    hyper = dict(synth.HYPER)
    hyper.update(over or {})
    if "policy_act_distribution" in hyper:   # golden of the plain Gaussian action distribution
        kw.setdefault("act_dist", hyper.pop("policy_act_distribution"))
    act_q, act_pi = synth.activations(cfg)   # goldens of the reference's other activations override the config's
    kw.setdefault("act_q", hyper.pop("value_hidden_activation", act_q))
    kw.setdefault("act_pi", hyper.pop("policy_hidden_activation", act_pi))
    c = make_config(cfg["obs_dim"], cfg["act_dim"], *synth.hidden_sizes(cfg), max_batch=batch,
                    gamma=hyper["gamma"], tau=hyper["tau"], tau_b=hyper.get("tau_b"), delay_update=hyper["delay_update"],
                    auto_alpha=hyper["auto_alpha"], alpha=hyper["alpha"], lr_q=hyper["value_learning_rate"],
                    lr_pi=hyper["policy_learning_rate"], lr_alpha=hyper["alpha_learning_rate"],
                    min_log_std=hyper["policy_min_log_std"], max_log_std=hyper["policy_max_log_std"], **kw)
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    eng = Engine(c, torch.device("cuda", 0), lim, -lim)
    eng.load_weights(synth.make_weights(cfg))
    return eng


def feed(cfg, batch, it):
    b = {k: torch.from_numpy(v).cuda() for k, v in synth.make_batch(cfg, batch, it).items()}
    n = synth.make_noise(cfg, batch, it)
    return b, tuple(torch.from_numpy(n[i]).cuda() for i in (0, 1, 4, 5))


def stats_vec(eng):
    from dsac_v2_b200.engine import STAT_KEYS
    s = eng.read_stats()
    return np.array([s[k] for k in STAT_KEYS])


# critics and policy of different depths, widths and activations (synth.ASYM_CONFIGS)
ASYM_CASES = ["asym_b70", "deep_pi_b70", "layered_pi_b70", "layered_q_b70"]
CASES = ["tiny_b16", "ragged_b37", "tiny_fixed_alpha", "pendulum_b256", "halfcheetah_b512", "humanoid_b256",
         "humanoid_b4096", "tiny_relu", "tiny_tanh", "ragged_elu", "ragged_selu", "tiny_sigmoid", "tiny_gauss"] + ASYM_CASES


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("name", CASES)
def test_update_matches_reference_golden(golden_dir, name, use_graph):
    if use_graph and name in ("pendulum_b256", "halfcheetah_b512"):
        pytest.skip("graph replay covered by the other cases")
    z, cfg, batch, steps, over = load(golden_dir, name)
    eng = make_engine(cfg, batch, over, use_graph=use_graph)
    names = [str(n) for n in z["param_names"]]
    for it in range(steps):
        b, n = feed(cfg, batch, it)
        eng.step(b, it, n)
        got = stats_vec(eng)
        np.testing.assert_allclose(got, z["tb"][it], rtol=RTOL, atol=1e-6, err_msg=f"{name} tb_info at step {it}")
        if f"pdigest_{it + 1}" in z:
            w = eng.export_weights()
            for row, k in zip(z[f"pdigest_{it + 1}"], names):
                d = w[k].double().reshape(-1)
                np.testing.assert_allclose(d.abs().sum().item(), row[1], rtol=RTOL, err_msg=f"{name} {k} step {it + 1}")
                np.testing.assert_allclose(d[:8].numpy(), row[3:3 + min(8, d.numel())], rtol=RTOL, atol=1e-7,
                                           err_msg=f"{name} {k} step {it + 1}")
        if f"state_{it + 1}/{names[0]}" in z:
            w = eng.export_weights()
            for k in names:
                ref = z[f"state_{it + 1}/{k}"]
                np.testing.assert_allclose(w[k].numpy(), ref, rtol=RTOL, atol=1e-6 * max(1e-3, np.abs(ref).max()),
                                           err_msg=f"{name} {k} after step {it + 1}")
    eng.close()


@pytest.mark.parametrize("name", ["tiny_b16", "ragged_b37"])
def test_gradients_match_reference_golden(golden_dir, name):
    z, cfg, batch, steps, over = load(golden_dir, name)
    eng = make_engine(cfg, batch, over, use_graph=False)
    trainable = [str(n) for n in z["trainable_names"]]
    for it in (0, 1):
        b, n = feed(cfg, batch, it)
        eng.compute_grads(b, n)
        g = eng.export_weights(grads=True)
        for k in trainable:
            ref = z[f"grad_{it}/{k}"]
            np.testing.assert_allclose(g[k].numpy(), ref, rtol=RTOL, atol=2e-6 * np.abs(ref).max() + 1e-12,
                                       err_msg=f"{name} grad {k} step {it}")
        eng.apply(it)
    eng.close()


@pytest.mark.parametrize("cfg_name,batch,act", [("ragged", 50, "relu"), ("tiny", 33, "tanh"), ("tiny", 8, "elu"),
                                                 ("ragged", 19, "selu"), ("tiny", 64, "sigmoid"), ("tiny", 1, "gelu")])
def test_update_matches_oracle_other_activations(cfg_name, batch, act):
    from oracle.dsact_oracle import TB_KEYS, from_config
    cfg = synth.CONFIGS[cfg_name]
    eng = make_engine(cfg, batch, use_graph=False, act_q=act, act_pi=act)
    orc = from_config(cfg, synth.make_weights(cfg), hidden_activation=act, **synth.HYPER)
    for it in range(4):
        hb, hn = synth.make_batch(cfg, batch, it), synth.make_noise(cfg, batch, it)
        ref = orc.update(hb, hn, it)
        b, n = feed(cfg, batch, it)
        eng.step(b, it, n)
        got = stats_vec(eng)
        np.testing.assert_allclose(got, [ref[k] for k in TB_KEYS], rtol=RTOL, atol=2e-6, err_msg=f"{act} step {it}")
    w, sd = eng.export_weights(), orc.state_dict()
    for k, v in sd.items():
        np.testing.assert_allclose(w[k].numpy(), v.numpy(), rtol=RTOL, atol=1e-6, err_msg=k)
    eng.close()


def test_split_api_equals_fused_step():
    """phase1 + phase2 + apply (the data-parallel seam) == dsact_step, bit for bit up to atomics order."""
    cfg, B = synth.CONFIGS["ragged"], 37
    a, b_ = make_engine(cfg, B, use_graph=False), make_engine(cfg, B, use_graph=True)
    for it in range(5):
        b, n = feed(cfg, B, it)
        a.step(b, it, n)
        b_.grad_phase1(b, n)
        b_.grad_phase2(B)
        b_.apply(it)
        np.testing.assert_allclose(stats_vec(b_), stats_vec(a), rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(a.params, b_.params, rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(a.targets, b_.targets, rtol=1e-5, atol=1e-7)
    a.close(); b_.close()


def test_device_noise_statistics():
    """Philox/Box-Muller draws used when no host noise is supplied: moments and reproducibility."""
    cfg, B = synth.CONFIGS["humanoid"], 4096
    eng = make_engine(cfg, B, use_graph=False)
    eng.seed(1234)
    b, _ = feed(cfg, B, 0)
    eng.step(b, 0, None)
    s1 = stats_vec(eng)
    assert np.all(np.isfinite(s1))
    # same seed + same counter -> same update
    eng2 = make_engine(cfg, B, use_graph=False)
    eng2.seed(1234)
    eng2.step(b, 0, None)
    np.testing.assert_allclose(stats_vec(eng2), s1, rtol=1e-5)
    # the generated noise itself sits in the arena: N(0,1)
    eps1 = eng.arena_views(B)["eps1"]
    assert abs(eps1.mean().item()) < 0.02 and abs(eps1.std().item() - 1.0) < 0.02
    assert abs((eps1 ** 4).mean().item() - 3.0) < 0.2
    eng.close(); eng2.close()


# ---- tensor-core (wgmma) paths -------------------------------------------------------------------------------------
TC_CASES = ["tiny_b16", "ragged_b37", "halfcheetah_b512", "humanoid_b256", "humanoid_b4096",
            # the generic-activation branch of the fused chain epilogue (GELU and ReLU have their own)
            "tiny_relu", "tiny_tanh", "ragged_elu", "ragged_selu", "tiny_sigmoid", "tiny_gauss"] + ASYM_CASES


@pytest.mark.parametrize("name", TC_CASES)
def test_bf16x3_tensor_core_path_matches_reference_golden(golden_dir, name):
    """Split-precision bf16 (hi*hi + hi*lo + lo*hi) on wgmma: still inside the 1e-4 gate on 100 losses."""
    z, cfg, batch, steps, over = load(golden_dir, name)
    eng = make_engine(cfg, batch, over, use_graph=True, gemm_mode="bf16x3")
    worst = 0.0
    for it in range(steps):
        b, n = feed(cfg, batch, it)
        eng.step(b, it, n)
        got = stats_vec(eng)
        ref = z["tb"][it]
        worst = max(worst, float(np.max(np.abs(got - ref) / np.maximum(np.abs(ref), 1e-2))))
        np.testing.assert_allclose(got, ref, rtol=RTOL, atol=1e-5, err_msg=f"{name} tb_info at step {it}")
    names = [str(n) for n in z["param_names"]]
    last = max(int(k.split("_")[1]) for k in z.files if k.startswith("pdigest_"))
    if last == steps:
        w = eng.export_weights()
        for row, k in zip(z[f"pdigest_{last}"], names):
            d = w[k].double().reshape(-1)
            np.testing.assert_allclose(d.abs().sum().item(), row[1], rtol=RTOL, err_msg=f"{name} {k}")
    print(f"{name}: worst relative tb_info deviation over {steps} steps = {worst:.2e}")
    eng.close()


# a hidden layer wider than 256: the chain kernel does not take it, so the tensor-core modes run the per-layer GEMM path
WIDE = dict(obs_dim=7, act_dim=3, hidden=(264, 40), act_lim=1.0)


@pytest.mark.parametrize("mode", ["bf16x3", "fp32"])
@pytest.mark.parametrize("cfg_name,batch,steps", [("humanoid", 65536, 2), ("halfcheetah", 8192, 3), ("wide", 40, 3)])
def test_large_batches_match_oracle(cfg_name, batch, steps, mode):
    """The largest configurations of BASELINE.json (config 4's 65536-row sweep point; config 3's 8192 rows per GPU):
    multi-wave chain launches and the bounded weight-gradient launches, against the pinned oracle on the same inputs.
    `wide` (WIDE) is the per-layer tensor-core step, which shapes outside the chain kernel's range take."""
    from oracle.dsact_oracle import TB_KEYS, from_config
    cfg = WIDE if cfg_name == "wide" else synth.CONFIGS[cfg_name]
    eng = make_engine(cfg, batch, use_graph=True, gemm_mode=mode)
    orc = from_config(cfg, synth.make_weights(cfg), **synth.HYPER)
    torch.set_num_threads(min(16, os.cpu_count() or 4))
    try:
        for it in range(steps):
            hb, hn = synth.make_batch(cfg, batch, it), synth.make_noise(cfg, batch, it)
            ref = orc.update(hb, hn, it)
            b = {k: torch.from_numpy(v).cuda() for k, v in hb.items()}
            n = tuple(torch.from_numpy(hn[i]).cuda() for i in (0, 1, 4, 5))
            eng.step(b, it, n)
            got = stats_vec(eng)
            np.testing.assert_allclose(got, [ref[k] for k in TB_KEYS], rtol=RTOL, atol=1e-5, err_msg=f"{cfg_name} B={batch} step {it}")
    finally:
        torch.set_num_threads(4)
    w, sd = eng.export_weights(), orc.state_dict()
    for k, v in sd.items():   # digests: |.|-sum and the first elements of every tensor
        a, r = w[k].double().reshape(-1), v.double().reshape(-1)
        np.testing.assert_allclose(a.abs().sum().item(), r.abs().sum().item(), rtol=RTOL, err_msg=k)
        np.testing.assert_allclose(a[:8].numpy(), r[:8].numpy(), rtol=RTOL, atol=1e-6, err_msg=k)
    eng.close()


def test_bf16x3_gradients_match_reference_golden(golden_dir):
    z, cfg, batch, steps, over = load(golden_dir, "ragged_b37")
    eng = make_engine(cfg, batch, over, use_graph=False, gemm_mode="bf16x3")
    trainable = [str(n) for n in z["trainable_names"]]
    for it in (0, 1):
        b, n = feed(cfg, batch, it)
        eng.compute_grads(b, n)
        g = eng.export_weights(grads=True)
        for k in trainable:
            ref = z[f"grad_{it}/{k}"]
            np.testing.assert_allclose(g[k].numpy(), ref, rtol=1e-3, atol=3e-5 * np.abs(ref).max() + 1e-12,
                                       err_msg=f"grad {k} step {it}")
        eng.apply(it)
    eng.close()


def test_bf16_single_pass_is_close_but_outside_the_parity_gate(golden_dir):
    """Throughput mode: operands rounded to bf16 once.  It must track the reference loosely; it is NOT a parity mode."""
    z, cfg, batch, steps, over = load(golden_dir, "humanoid_b256")
    eng = make_engine(cfg, batch, over, use_graph=True, gemm_mode="bf16")
    dev = []
    for it in range(30):
        b, n = feed(cfg, batch, it)
        eng.step(b, it, n)
        got = stats_vec(eng)
        assert np.all(np.isfinite(got))
        dev.append(abs(got[7] - z["tb"][it][7]) / abs(z["tb"][it][7]))
    assert max(dev) < 5e-2, max(dev)
    print(f"bf16 single pass: max critic-loss deviation over 30 steps = {max(dev):.2e}")
    eng.close()
