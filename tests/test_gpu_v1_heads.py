"""DSAC_V1 (reference dsac_v1.py) on the head-wise fp32 engine beyond the MLP / "mlp_shared" configuration: the CNN
approximators (example_train/dsacv1_cnn_carracing_offasync.py), the policy std types "mlp_separated" / "parameter", the
plain Gaussian and act_dim 1.  Through the C ABI against the goldens of the unmodified reference (tests/golden/v1_cnn_*,
v1_std_*, v1_tiny_gauss, v1_pendulum_b64) and against the pinned oracle on ragged shapes; through the drop-in
`dsac_v1.DSAC_V1`; and the trainer's full-state checkpoint / resume on the head-wise engine."""
import ast
import os

import numpy as np
import pytest
import torch

from dsac_v2_b200 import synth

pytestmark = pytest.mark.gpu
RTOL = 1e-4
# columns of the engine's 16 statistics that carry DSAC_V1's tb_info (dsac_v1.py:172-181), in V1_TB_KEYS order
V1_COLS = [0, 2, 6, 8, 9, 10, 11]
GOLDENS = ["v1_cnn_carracing_b4", "v1_cnn_type1_b5", "v1_std_separated", "v1_std_parameter", "v1_tiny_gauss", "v1_pendulum_b64"]


def v1_weights(cfg, std_type="mlp_shared"):
    if "conv_type" in cfg:
        return synth.make_cnn_weights_v1(cfg)
    return synth.make_weights_v1(cfg) if std_type == "mlp_shared" else synth.make_weights_std_v1(cfg, std_type)


def make_engine(cfg, batch, over):
    from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config, make_heads_config
    h = dict(synth.HYPER)
    h.update(over)
    common = dict(max_batch=batch, algo="DSAC_V1", bound=h.get("bound", True), td_bound=h.get("TD_bound", 20), gamma=h["gamma"],
                  tau=h["tau"], delay_update=h["delay_update"], auto_alpha=h["auto_alpha"], alpha=h["alpha"],
                  lr_q=h["value_learning_rate"], lr_pi=h["policy_learning_rate"], lr_alpha=h["alpha_learning_rate"],
                  min_log_std=h["policy_min_log_std"], max_log_std=h["policy_max_log_std"],
                  act_dist=h.get("policy_act_distribution", "TanhGaussDistribution"))
    std_type = h.get("policy_std_type", "mlp_shared")
    if "conv_type" in cfg:
        t = synth.CONV_TYPES[cfg["conv_type"]]
        c = make_cnn_config(cfg["obs_dim"], cfg["act_dim"], t["kernels"], t["channels"], t["strides"], t["heads"], **common)
    else:
        c = make_heads_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], std_type, **common)
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    eng = CnnEngine(c, torch.device("cuda", 0), lim, -lim)
    eng.load_weights(v1_weights(cfg, std_type))
    return eng


def make_batch(cfg, batch, it):
    return (synth.make_cnn_batch if "conv_type" in cfg else synth.make_batch)(cfg, batch, it)


def feed(cfg, batch, it):
    b = {k: torch.from_numpy(v).cuda() for k, v in make_batch(cfg, batch, it).items()}
    n = synth.make_noise(cfg, batch, it)
    return b, tuple(torch.from_numpy(n[i]).cuda() for i in (0, 1, 3, 3))   # eps1, eps2, the target critic's z (twice)


def stats_v1(eng):
    from dsac_v2_b200.engine import STAT_KEYS
    s = eng.read_stats()
    v = [s[k] for k in STAT_KEYS]
    return np.array([v[i] for i in V1_COLS])


def load_golden(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg_name, batch, steps, over = z["meta"]
    cfg = synth.CNN_CONFIGS[str(cfg_name)] if str(cfg_name) in synth.CNN_CONFIGS else synth.CONFIGS[str(cfg_name)]
    over = dict(ast.literal_eval(str(over)))
    assert over.pop("algorithm") == "DSAC_V1"
    return z, cfg, int(batch), int(steps), over


@pytest.mark.parametrize("name", GOLDENS)
def test_v1_heads_update_matches_reference_golden(golden_dir, name):
    z, cfg, batch, steps, over = load_golden(golden_dir, name)
    eng = make_engine(cfg, batch, over)
    names = [str(n) for n in z["param_names"]]
    # the flat layout [q | policy] in the reference's named_parameters order
    assert [key for key, *_ in eng._schema()[0]] == [k for k in names if "_target." not in k and k != "log_alpha"]
    for it in range(steps):
        b, n = feed(cfg, batch, it)
        eng.step(b, it, n)
        np.testing.assert_allclose(stats_v1(eng), z["tb"][it], rtol=RTOL, atol=1e-6, err_msg=f"{name} tb_info at step {it}")
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
                np.testing.assert_allclose(w[k].numpy().reshape(ref.shape), ref, rtol=RTOL, atol=1e-6 * max(1e-3, np.abs(ref).max()),
                                           err_msg=f"{name} {k} after step {it + 1}")
    eng.close()


ORACLE_CASES = [("carracing", 3, {}), ("carracing", 32, {}), ("small_t1", 7, {}), ("odd", 9, {}), ("odd", 200, {})] + [
    ("ragged", 50, dict(over, policy_std_type=std)) for std in ("mlp_separated", "parameter")
    for over in ({"TD_bound": 0.5}, {"bound": False})]


@pytest.mark.parametrize("cfg_name,batch,over", ORACLE_CASES)
def test_v1_heads_update_matches_oracle(cfg_name, batch, over):
    """Ragged batch sizes against every tile size, the three encoders, both std types with a TD bound that clips and with
    the Gaussian NLL: tb_info of every step, the gradients of the last step, the full post-update state."""
    from oracle.dsact_oracle import V1_TB_KEYS
    from oracle.dsact_oracle_v1_heads import v1_cnn_from_config, v1_std_from_config
    cnn = cfg_name in synth.CNN_CONFIGS
    cfg = synth.CNN_CONFIGS[cfg_name] if cnn else synth.CONFIGS[cfg_name]
    eng = make_engine(cfg, batch, over)
    hyper = dict(synth.HYPER)
    hyper.update(over)
    std_type = hyper.pop("policy_std_type", "mlp_shared")
    orc = v1_cnn_from_config(cfg, v1_weights(cfg), **hyper) if cnn else \
        v1_std_from_config(cfg, v1_weights(cfg, std_type), std_type, **hyper)
    for it in range(3):
        ref = orc.update(make_batch(cfg, batch, it), synth.make_noise(cfg, batch, it), it)
        b, n = feed(cfg, batch, it)
        eng.step(b, it, n)
        np.testing.assert_allclose(stats_v1(eng), [ref[k] for k in V1_TB_KEYS], rtol=RTOL, atol=1e-6, err_msg=f"step {it}")
    g, gref = eng.export_weights(grads=True), orc.grad_dict()
    for k, v in gref.items():
        np.testing.assert_allclose(g[k].numpy().reshape(v.shape), v.numpy(), rtol=1e-3, atol=2e-6 * float(v.abs().max()) + 1e-12,
                                   err_msg=f"grad {k}")
    w, sd = eng.export_weights(), orc.state_dict()
    for k, v in sd.items():   # (Adam turns a 1e-7 gradient difference on a near-zero gradient into up to a few 1e-6 of weight)
        np.testing.assert_allclose(w[k].numpy().reshape(v.shape), v.numpy(), rtol=RTOL, atol=1e-5, err_msg=k)
    eng.close()


def _load_into(alg, weights):
    sd = alg.networks.state_dict()
    assert {k for k in sd if not k.endswith("_lim")} == set(weights) | {"log_alpha"}   # (+ act_high/low_lim buffers)
    for k, v in weights.items():
        sd[k] = torch.from_numpy(v)
    alg.networks.load_state_dict(sd)


def test_v1_cnn_dropin_local_update(golden_dir):
    """`dsac_v1.DSAC_V1(**cnn_reference_kwargs)`: the reference's state_dict keys and parameter order, the golden's values
    through the module's engine, `local_update` on a host image minibatch with device noise and with the reference's noise
    order (checked against the oracle fed the same torch draws)."""
    import dsac_v1
    from oracle.dsact_oracle import V1_TB_KEYS
    from oracle.dsact_oracle_v1_heads import v1_cnn_from_config
    z, cfg, B, _steps, _over = load_golden(golden_dir, "v1_cnn_carracing_b4")
    kw = synth.cnn_reference_kwargs(cfg, algorithm="DSAC_V1", replay_batch_size=B)
    alg = dsac_v1.DSAC_V1(**kw)
    assert [k for k, _ in alg.networks.named_parameters()] == [str(n) for n in z["param_names"]]
    ref_w = synth.make_cnn_weights_v1(cfg)
    _load_into(alg, ref_w)
    alg.networks.cuda()
    eng = alg.networks.engine(B)
    for it in range(2):
        b, n = feed(cfg, B, it)
        eng.step(b, it, n)
        np.testing.assert_allclose(stats_v1(eng), z["tb"][it], rtol=RTOL, atol=1e-6)
    # parameters are views of the flat buffers: the module sees the update, in the reference's schema
    sd, w = alg.networks.state_dict(), eng.export_weights()
    assert not torch.equal(sd["policy.conv.0.weight"].cpu(), torch.from_numpy(ref_w["policy.conv.0.weight"]))
    for k in ref_w:
        assert torch.equal(sd[k].cpu(), w[k]), k
    tb = alg.local_update({k: torch.from_numpy(v) for k, v in make_batch(cfg, B, 5).items()}, 2)   # host minibatch, device noise
    assert set(V1_TB_KEYS) <= set(tb) and all(np.isfinite(tb[k]) for k in V1_TB_KEYS)
    with pytest.raises(NotImplementedError):
        alg.get_remote_update_info({}, 0)

    # reference noise order: eps1, eps2 and three z's from torch's CPU generator; the target critic's draw is the second z
    alg = dsac_v1.DSAC_V1(**dict(kw, dsact_noise="reference"))
    _load_into(alg, ref_w)
    alg.networks.cuda()
    orc = v1_cnn_from_config(cfg, ref_w, **synth.HYPER)
    for it in range(2):
        data = make_batch(cfg, B, it)
        torch.manual_seed(100 + it)
        tb = alg.local_update({k: torch.from_numpy(v) for k, v in data.items()}, it)
        torch.manual_seed(100 + it)
        A = cfg["act_dim"]
        noise = [torch.empty(B, A).normal_(), torch.empty(B, A).normal_()] + [torch.normal(torch.zeros(B), torch.ones(B)) for _ in range(3)]
        ref = orc.update(data, noise, it)
        np.testing.assert_allclose([tb[k] for k in V1_TB_KEYS], [ref[k] for k in V1_TB_KEYS], rtol=RTOL, atol=1e-6, err_msg=f"step {it}")


@pytest.mark.parametrize("std_type", ["mlp_separated", "parameter"])
def test_v1_std_type_dropin(golden_dir, std_type):
    """`dsac_v1.DSAC_V1(policy_std_type=...)`: named_parameters in the reference's order (the learnable log_std row of
    "parameter" before the mean MLP), the module's views line up with the engine's flat layout, golden values."""
    import dsac_v1
    name = {"mlp_separated": "v1_std_separated", "parameter": "v1_std_parameter"}[std_type]
    z, cfg, B, steps, _over = load_golden(golden_dir, name)
    alg = dsac_v1.DSAC_V1(**synth.reference_kwargs(cfg, algorithm="DSAC_V1", policy_std_type=std_type, replay_batch_size=B))
    names = [str(n) for n in z["param_names"]]
    assert [k for k, _ in alg.networks.named_parameters()] == names
    _load_into(alg, synth.make_weights_std_v1(cfg, std_type))
    alg.networks.cuda()
    eng = alg.networks.engine(B)
    for it in range(steps):
        b, n = feed(cfg, B, it)
        eng.step(b, it, n)
        np.testing.assert_allclose(stats_v1(eng), z["tb"][it], rtol=RTOL, atol=1e-6, err_msg=f"step {it}")
    sd = alg.networks.state_dict()
    for k in names:
        ref = z[f"state_{steps}/{k}"]
        np.testing.assert_allclose(sd[k].cpu().numpy(), ref, rtol=RTOL, atol=1e-6 * max(1e-3, np.abs(ref).max()), err_msg=k)


# ---- the drop-in trainer on the head-wise engine ---------------------------------------------------------------------
VARIANTS = {
    "v1_mlp": ("DSAC_V1", "tiny", {}),
    "v1_cnn": ("DSAC_V1", "small_t1", {}),
    "v2_separated": ("DSAC_V2", "tiny", {"policy_std_type": "mlp_separated"}),
}


def make_trainer(variant, folder, **extra):
    """An `OffSerialTrainer` with a stub sampler (the CPU mirror of the policy acting on a random walk of observations;
    images for the CNN variant) and a stub evaluator.  Loss records of every local_update land in the returned list."""
    import dsac_v1
    import dsac_v2
    from training.replay_buffer import ReplayBuffer
    from training.trainer import create_trainer
    algo, cfg_name, over = VARIANTS[variant]
    mod = dsac_v1 if algo == "DSAC_V1" else dsac_v2
    cnn = cfg_name in synth.CNN_CONFIGS
    cfg = synth.CNN_CONFIGS[cfg_name] if cnn else synth.CONFIGS[cfg_name]
    np.random.seed(3)
    torch.manual_seed(3)
    kw = (synth.cnn_reference_kwargs if cnn else synth.reference_kwargs)(cfg, algorithm=algo, replay_batch_size=16, seed=11, **over)
    kw = dict(kw, buffer_max_size=400, additional_info={}, buffer_name="replay_buffer", buffer_warm_size=60, max_iteration=16,
              log_save_interval=1000, apprfunc_save_interval=8, eval_interval=1000, save_folder=str(folder), ini_network_dir=None,
              use_gpu=True, dsact_tensorboard=False, **extra)
    alg = (mod.DSAC_V1 if algo == "DSAC_V1" else mod.DSAC_V2)(**kw)
    shape = tuple(cfg["obs_dim"]) if cnn else (cfg["obs_dim"],)

    class Sampler:
        def __init__(self):
            self.networks = mod.ApproxContainer(**kw)
            self.n, self.g = 0, np.random.default_rng(0)
            self.obs = self.g.random(shape).astype(np.float32)

        def sample(self):
            out = []
            for _ in range(20):
                logits = self.networks.policy(torch.from_numpy(self.obs[None]))
                act, logp = self.networks.create_action_distributions(logits).sample()
                nxt = np.clip(0.9 * self.obs + 0.1 * self.g.random(shape), 0, 1).astype(np.float32)
                out.append((self.obs.copy(), {}, act.detach()[0].numpy(), float(-np.abs(nxt - 0.5).mean()), nxt.copy(), False,
                            logp.detach()[0].numpy(), {}))
                self.obs = nxt
            self.n += 20
            return out, {}

        def get_total_sample_number(self):
            return self.n

    class Evaluator:
        networks, calls = None, 0

        def run_evaluation(self, it):
            self.calls += 1
            return 0.0

    rec = []
    inner = alg.local_update

    def local_update(data, it):
        tb = inner(data, it)
        rec.append((it, float(tb["Loss/Actor loss-RL iter"])))
        return tb

    alg.local_update = local_update
    return create_trainer(alg, Sampler(), ReplayBuffer(**kw), Evaluator(), **kw), alg, rec


def test_v1_cnn_trainer_with_image_replay_ring(tmp_path):
    """`OffSerialTrainer` around DSAC_V1 with CNN networks: image rows in the device replay ring, the CPU policy mirror
    tracks the trained GPU policy."""
    trainer, alg, rec = make_trainer("v1_cnn", tmp_path, sample_interval=4)
    assert tuple(trainer.buffer.engine.replay["obs"].shape) == (400, int(np.prod(synth.CNN_CONFIGS["small_t1"]["obs_dim"])))
    first = alg.networks.policy.conv[0].weight.detach().clone()
    trainer.train()
    assert trainer.iteration == 16 and [it for it, _ in rec] == list(range(16))
    assert all(np.isfinite(v) for _, v in rec)
    now = alg.networks.policy.conv[0].weight.detach()
    assert not torch.equal(first, now)
    trainer.refresh_policy_mirror()
    torch.testing.assert_close(trainer.sampler.networks.policy.conv[0].weight.detach(), now.cpu(), rtol=0, atol=0)
    assert os.path.exists(tmp_path / "apprfunc" / "apprfunc_16.pkl")


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_trainer_full_checkpoint_resume_is_bit_identical(tmp_path, variant):
    """`dsact_full_checkpoint` inside iteration 8, a second trainer resumed from it with `dsact_resume_dir`: the same
    updates 9..15 as the uninterrupted run and bit-identical final weights, targets, log_alpha and Adam moments."""
    full, alg_full, rec_full = make_trainer(variant, tmp_path / "full", dsact_full_checkpoint=True, sample_interval=1000)
    full.train()
    assert [it for it, _ in rec_full] == list(range(16))
    ck = tmp_path / "full" / "apprfunc" / "trainstate_8.pkl"      # written inside iteration 8, after its update
    assert torch.load(ck, weights_only=False)["iteration"] == 9
    resumed, alg_res, rec_res = make_trainer(variant, tmp_path / "resumed", dsact_full_checkpoint=True, sample_interval=1000,
                                             dsact_resume_dir=str(ck))
    assert resumed.iteration == 9
    resumed.train()
    assert [it for it, _ in rec_res] == list(range(9, 16))
    assert [v for _, v in rec_res] == [v for _, v in rec_full[9:]]
    sd_full, sd_res = alg_full.networks.state_dict(), alg_res.networks.state_dict()
    assert list(sd_full) == list(sd_res)
    for k in sd_full:
        assert torch.equal(sd_full[k], sd_res[k]), k
    ef, er = alg_full.networks.engine(), alg_res.networks.engine()
    for name in ("params", "targets", "adam_m", "adam_v"):
        assert torch.equal(getattr(ef, name), getattr(er, name)), name
