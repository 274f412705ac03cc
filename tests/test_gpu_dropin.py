"""The host-side mirror of the reference interface (dsac_v2.DSAC_V2 / ApproxContainer,
training.replay_buffer.ReplayBuffer, training.trainer.OffSerialTrainer) on the GPU."""
import os

import numpy as np
import pytest
import torch

from dsac_v2_b200 import synth

pytestmark = pytest.mark.gpu


def build_alg(cfg, batch, **over):
    import dsac_v2
    kw = synth.reference_kwargs(cfg, replay_batch_size=batch, **over)
    alg = dsac_v2.DSAC_V2(**kw)
    sd = alg.networks.state_dict()
    for k, v in synth.make_weights(cfg).items():
        sd[k] = torch.from_numpy(v)
    alg.networks.load_state_dict(sd)
    return alg, kw


def test_local_update_same_seed_as_reference_rng_order():
    """dsact_noise='reference': the 8 normal draws come from torch's CPU generator in the reference's
    order (SURVEY Appendix B), so an oracle consuming the same stream must agree step for step."""
    check_local_update_against_oracle(synth.CONFIGS["halfcheetah"], 64)


@pytest.mark.parametrize("name,gemm", [("asym", "bf16x3"), ("layered_pi", "fp32")])
def test_local_update_with_different_critic_and_policy_networks(name, gemm):
    """value_hidden_sizes / value_hidden_activation differ from the policy_* ones: the fused layer chain (asym) and the
    per-layer path (layered_pi) against the oracle of the same configuration.  layered_pi runs in fp32: its ReLU critic
    has weight-gradient entries near zero, whose first Adam steps (about lr * sign) bf16x3 rounding can flip."""
    check_local_update_against_oracle(synth.ASYM_CONFIGS[name], 70, dsact_gemm=gemm)


def check_local_update_against_oracle(cfg, B, **over):
    from oracle.dsact_oracle import TB_KEYS, from_config
    alg, _ = build_alg(cfg, B, dsact_noise="reference", **over)
    alg.networks.cuda()
    orc = from_config(cfg, synth.make_weights(cfg), **synth.HYPER)
    A = cfg["act_dim"]
    for it in range(6):
        batch = {k: torch.from_numpy(v) for k, v in synth.make_batch(cfg, B, it).items()}
        torch.manual_seed(100 + it)
        noise = [torch.empty(B, A).normal_(), torch.empty(B, A).normal_()] + \
                [torch.normal(torch.zeros(B), torch.ones(B)) for _ in range(6)]
        ref = orc.update(batch, noise, it)
        torch.manual_seed(100 + it)
        tb = alg.local_update({k: v.cuda() for k, v in batch.items()}, it)
        for k in TB_KEYS:
            assert abs(tb[k] - ref[k]) <= 1e-4 * max(1.0, abs(ref[k])), (it, k, tb[k], ref[k])
        assert "Time/Algorithm time [ms]-RL iter" in tb and len(tb) == 15
    sd = alg.networks.state_dict()
    for k, v in orc.state_dict().items():
        np.testing.assert_allclose(sd[k].cpu().numpy(), v.numpy(), rtol=1e-4, atol=1e-6, err_msg=k)


def test_state_dict_schema_and_checkpoint_roundtrip(tmp_path):
    cfg = synth.CONFIGS["pendulum"]
    alg, kw = build_alg(cfg, 32)
    net = alg.networks
    keys_cpu = list(net.state_dict())
    net.cuda()
    sd = net.state_dict()
    assert list(sd) == keys_cpu and len(sd) == 53  # the shipped checkpoint schema (SURVEY §4)
    for want in ("log_alpha", "q1.q.0.weight", "q2.q.6.bias", "q1_target.q.4.weight", "policy.act_high_lim",
                 "policy.policy.6.weight", "policy_target.policy.0.bias", "policy_target.act_low_lim"):
        assert want in sd
    # parameters are views into the flat buffers, checkpoints are not
    eng = net.engine()
    assert net.q1.q[0].weight.data_ptr() == eng.params.data_ptr()
    assert sd["q1.q.0.weight"].data_ptr() != eng.params.data_ptr()
    path = tmp_path / "apprfunc_0.pkl"
    torch.save(sd, path)
    assert os.path.getsize(path) < 4 * sum(v.numel() for v in sd.values()) + 65536
    b = {k: torch.from_numpy(v).cuda() for k, v in synth.make_batch(cfg, 32, 0).items()}
    alg.local_update(b, 0)
    changed = net.state_dict()
    assert not torch.equal(changed["q1.q.0.weight"], sd["q1.q.0.weight"])
    net.load_state_dict(torch.load(path, weights_only=True))
    torch.testing.assert_close(net.state_dict()["q1.q.0.weight"], sd["q1.q.0.weight"], rtol=0, atol=0)
    assert net.q1.q[0].weight.data_ptr() == eng.params.data_ptr()  # still bound after load
    # a CPU container (what run_policy / the sampler build) loads the same file
    import dsac_v2
    cpu_net = dsac_v2.ApproxContainer(**kw)
    cpu_net.load_state_dict(torch.load(path, weights_only=True))
    out = cpu_net.policy(torch.zeros(1, cfg["obs_dim"]))
    assert out.shape == (1, 2 * cfg["act_dim"])
    act = cpu_net.create_action_distributions(out).mode()
    assert act.abs().max() <= cfg["act_lim"] + 1e-6


def test_module_device_round_trip_keeps_training_state():
    """ModuleOnDevice-style cuda -> cpu -> cuda (reference trainer.py:64) must not lose weights."""
    cfg, B = synth.CONFIGS["tiny"], 16
    alg, _ = build_alg(cfg, B)
    alg.networks.cuda()
    b = {k: torch.from_numpy(v).cuda() for k, v in synth.make_batch(cfg, B, 0).items()}
    alg.local_update(b, 0)
    before = {k: v.clone() for k, v in alg.networks.state_dict().items()}
    alg.networks.to("cpu")
    assert next(alg.networks.parameters()).device.type == "cpu"
    with pytest.raises(Exception):
        alg.local_update(b, 1)
    alg.networks.to("cuda")
    for k, v in alg.networks.state_dict().items():
        torch.testing.assert_close(v, before[k], rtol=0, atol=0)
    alg.local_update(b, 1)


def test_remote_update_seam_equals_local_update():
    cfg, B = synth.CONFIGS["tiny"], 16
    a, _ = build_alg(cfg, B, dsact_noise="reference")
    b, _ = build_alg(cfg, B, dsact_noise="reference")
    a.networks.cuda(); b.networks.cuda()
    for it in range(4):
        batch = {k: torch.from_numpy(v).cuda() for k, v in synth.make_batch(cfg, B, it).items()}
        torch.manual_seed(it)
        tb_a = a.local_update(batch, it)
        torch.manual_seed(it)
        tb_b, info = b.get_remote_update_info(batch, it)
        assert set(info) == {"q1_grad", "q2_grad", "policy_grad", "iteration", "log_alpha_grad"}
        assert [g.shape for g in info["q1_grad"]] == [p.shape for p in b.networks.q1.parameters()]
        msg = {k: ([g.clone() for g in v] if isinstance(v, list) else (v.clone() if torch.is_tensor(v) else v))
               for k, v in info.items()}
        b.remote_update(msg)
        assert abs(tb_a["Loss/Critic loss-RL iter"] - tb_b["Loss/Critic loss-RL iter"]) < 1e-5
    for (k, va), vb in zip(a.networks.state_dict().items(), b.networks.state_dict().values()):
        torch.testing.assert_close(va, vb, rtol=1e-5, atol=1e-7, msg=k)


def test_replay_ring_store_wrap_and_gather_are_bit_exact():
    from training.replay_buffer import ReplayBuffer
    cfg = synth.CONFIGS["ragged"]
    alg, kw = build_alg(cfg, 64)
    alg.networks.cuda()
    cap, O, A = 50, cfg["obs_dim"], cfg["act_dim"]
    buf = ReplayBuffer(**dict(kw, buffer_max_size=cap, additional_info={}, dsact_index_source="numpy"))
    g = np.random.default_rng(3)
    rows = []
    for i in range(70):  # wraps past capacity; first 7 stored before the engine is attached
        if i == 7:
            buf.attach(alg.networks.engine())
        row = (g.standard_normal(O).astype(np.float32), {}, g.standard_normal(A).astype(np.float32), float(i),
               g.standard_normal(O).astype(np.float32), bool(i % 5 == 0), np.float32(-i), {})
        rows.append(row)
        buf.add_batch([row])
        if i % 13 == 12:
            buf.flush()
    assert len(buf) == cap and buf.size == cap
    assert buf.__get_RAM__() > 0
    np.random.seed(0)
    out = buf.sample_batch(64)
    np.random.seed(0)
    idx = np.random.randint(0, cap, size=64)
    ring = {}
    for i, r in enumerate(rows):
        ring[i % cap] = r
    for j, src in enumerate(idx):
        r = ring[int(src)]
        assert np.array_equal(out["obs"][j].cpu().numpy(), r[0])
        assert np.array_equal(out["act"][j].cpu().numpy(), r[2])
        assert out["rew"][j].item() == r[3]
        assert np.array_equal(out["obs2"][j].cpu().numpy(), r[4])
        assert out["done"][j].item() == float(r[5])
        assert out["logp"][j].item() == float(r[6])
    assert set(out) == {"obs", "obs2", "act", "rew", "done", "logp"}
    # device-side index generation: in range, roughly uniform
    buf.index_source = "device"
    alg.networks.engine().seed(5)
    seen = torch.zeros(cap)
    for _ in range(50):
        rew = buf.sample_batch(64)["rew"].cpu()
        vals = rew.long()
        assert ((vals >= 20) & (vals < 70)).all()  # surviving rows are i = 20..69
        seen += torch.bincount(vals - 20, minlength=cap)
    assert seen.min() > 20 and seen.max() < 120  # mean 64
    with pytest.raises(Exception):
        ReplayBuffer(**dict(kw, buffer_max_size=8, additional_info={})).sample_batch(4)


class _StubEnvSampler:
    """Stands in for training.off_sampler.OffSampler: same attributes the trainer touches."""

    def __init__(self, kw, cfg):
        import dsac_v2
        self.networks = dsac_v2.ApproxContainer(**kw)
        self.cfg, self.n, self.g = cfg, 0, np.random.default_rng(0)
        self.obs = self.g.standard_normal(cfg["obs_dim"]).astype(np.float32)

    def sample(self):
        out = []
        for _ in range(20):
            logits = self.networks.policy(torch.from_numpy(self.obs[None]))
            act, logp = self.networks.create_action_distributions(logits).sample()
            nxt = (0.9 * self.obs + 0.1 * self.g.standard_normal(self.cfg["obs_dim"])).astype(np.float32)
            out.append((self.obs.copy(), {}, act.detach()[0].numpy(), float(-np.abs(nxt).mean()), nxt.copy(), False,
                        logp.detach()[0].numpy(), {}))
            self.obs = nxt
        self.n += 20
        return out, {"Time/Sampler time [ms]-RL iter": 0.0}

    def get_total_sample_number(self):
        return self.n


class _StubEvaluator:
    def __init__(self):
        self.networks, self.calls = None, 0

    def run_evaluation(self, it):
        self.calls += 1
        out = self.networks.policy(torch.zeros(1, self.networks.policy.policy[0].in_features))
        return float(out.sum())


def test_trainer_loop_runs_and_mirrors_policy(tmp_path):
    from training.replay_buffer import ReplayBuffer
    from training.trainer import create_trainer
    cfg = synth.CONFIGS["tiny"]
    alg, kw = build_alg(cfg, 32)
    kw = dict(kw, buffer_max_size=1000, additional_info={}, buffer_name="replay_buffer", buffer_warm_size=100,
              max_iteration=30, log_save_interval=10, apprfunc_save_interval=20, eval_interval=10,
              save_folder=str(tmp_path), ini_network_dir=None, use_gpu=True, dsact_tensorboard=False)
    sampler, evaluator = _StubEnvSampler(kw, cfg), _StubEvaluator()
    buf = ReplayBuffer(**kw)
    trainer = create_trainer(alg, sampler, buf, evaluator, **kw)
    assert buf.size >= 100
    w0 = alg.networks.state_dict()["policy.policy.0.weight"].clone()
    trainer.train()
    assert trainer.iteration == 30 and evaluator.calls == 3
    files = sorted(os.listdir(tmp_path / "apprfunc"))
    assert "apprfunc_0.pkl" in files and "apprfunc_20.pkl" in files and "apprfunc_30.pkl" in files
    w1 = alg.networks.state_dict()["policy.policy.0.weight"]
    assert not torch.equal(w0, w1)
    # the CPU mirror the sampler acts with tracks the trained GPU policy
    trainer.refresh_policy_mirror()
    torch.testing.assert_close(sampler.networks.policy.policy[0].weight.detach(), w1.cpu(), rtol=0, atol=0)
    tb = trainer.last_tb
    assert np.isfinite(tb["Loss/Critic loss-RL iter"])
    ck = torch.load(tmp_path / "apprfunc" / "apprfunc_30.pkl", weights_only=True)
    assert len(ck) == 41


def test_full_state_checkpoint_resumes_exactly(tmp_path):
    """SURVEY §8f rank 3: weights + Adam moments + EMA + counters + generator + replay ring -> identical continuation."""
    from training.replay_buffer import ReplayBuffer
    cfg, B = synth.CONFIGS["tiny"], 32

    def make():
        alg, kw = build_alg(cfg, B)
        alg.networks.cuda()
        eng = alg.networks.engine()
        eng.seed(99)
        buf = ReplayBuffer(**dict(kw, buffer_max_size=500, additional_info={}))
        buf.attach(eng)
        return alg, buf

    g = np.random.default_rng(0)
    rows = [(g.standard_normal(5).astype(np.float32), {}, g.uniform(-1, 1, 2).astype(np.float32), float(g.standard_normal()),
             g.standard_normal(5).astype(np.float32), False, np.float32(0), {}) for _ in range(300)]
    a, buf_a = make()
    buf_a.add_batch(rows)
    for it in range(6):
        a.local_update(buf_a.sample_batch(B), it)
    path = tmp_path / "trainstate.pkl"
    torch.save({"alg": a.full_state_dict(), "buffer": buf_a.state_dict()}, path)
    cont_a = [a.local_update(buf_a.sample_batch(B), it)["Loss/Critic loss-RL iter"] for it in range(6, 12)]

    b, buf_b = make()
    st = torch.load(path, weights_only=False)
    b.load_full_state_dict(st["alg"])
    buf_b.load_state_dict(st["buffer"])
    assert (buf_b.size, buf_b.ptr) == (300, 300)
    cont_b = [b.local_update(buf_b.sample_batch(B), it)["Loss/Critic loss-RL iter"] for it in range(6, 12)]
    np.testing.assert_allclose(cont_b, cont_a, rtol=2e-5)   # same device indices and noise, same Adam state
    for (k, va), vb in zip(a.networks.state_dict().items(), b.networks.state_dict().values()):
        torch.testing.assert_close(va, vb, rtol=2e-5, atol=1e-7, msg=k)


def test_async_sampler_feeds_buffer_while_training(tmp_path):
    from training.replay_buffer import ReplayBuffer
    from training.trainer import create_trainer
    cfg = synth.CONFIGS["tiny"]
    alg, kw = build_alg(cfg, 32)
    kw = dict(kw, buffer_max_size=5000, additional_info={}, buffer_name="replay_buffer", buffer_warm_size=100,
              max_iteration=200, log_save_interval=1000, apprfunc_save_interval=1000, eval_interval=1000,
              save_folder=str(tmp_path), ini_network_dir=None, use_gpu=True, dsact_tensorboard=False,
              dsact_async_sampler=True, dsact_full_checkpoint=True)
    sampler, evaluator = _StubEnvSampler(kw, cfg), _StubEvaluator()
    buf = ReplayBuffer(**kw)
    trainer = create_trainer(alg, sampler, buf, evaluator, **kw)
    size0 = buf.size
    trainer.train()
    assert trainer.iteration == 200 and trainer._thread is None
    assert buf.size > size0                      # transitions arrived from the background thread
    assert sampler.get_total_sample_number() >= buf.size - 0
    assert np.isfinite(trainer.last_tb["Loss/Critic loss-RL iter"])
    assert os.path.exists(tmp_path / "apprfunc" / "trainstate_200.pkl")


def test_trainer_checkpoint_resumes_at_the_next_iteration(tmp_path):
    """A trainer restored from an in-step trainstate continues with the NEXT iteration: the interrupted run and the
    uninterrupted one produce the same critic losses and the same final weights (no repeated update)."""
    from training.replay_buffer import ReplayBuffer
    from training.trainer import create_trainer
    cfg = synth.CONFIGS["tiny"]

    def make(folder, **extra):
        np.random.seed(3); torch.manual_seed(3)
        alg, kw = build_alg(cfg, 32, seed=11)
        kw = dict(kw, buffer_max_size=2000, additional_info={}, buffer_name="replay_buffer", buffer_warm_size=100,
                  max_iteration=16, log_save_interval=1000, apprfunc_save_interval=8, eval_interval=1000,
                  save_folder=str(folder), ini_network_dir=None, use_gpu=True, dsact_tensorboard=False,
                  dsact_full_checkpoint=True, sample_interval=1000, **extra)   # no new transitions after the warm-up
        sampler, evaluator = _StubEnvSampler(kw, cfg), _StubEvaluator()
        buf = ReplayBuffer(**kw)
        rec = []
        inner = alg.local_update

        def local_update(data, it):
            tb = inner(data, it)
            rec.append((it, tb["Loss/Critic loss-RL iter"]))
            return tb

        alg.local_update = local_update
        return create_trainer(alg, sampler, buf, evaluator, **kw), alg, rec

    full, alg_full, rec_full = make(tmp_path / "full")
    full.train()
    assert [it for it, _ in rec_full] == list(range(16))
    ck = tmp_path / "full" / "apprfunc" / "trainstate_8.pkl"      # written inside iteration 8, after its update
    assert torch.load(ck, weights_only=False)["iteration"] == 9
    resumed, alg_res, rec_res = make(tmp_path / "resumed", dsact_resume_dir=str(ck))
    assert resumed.iteration == 9
    resumed.train()
    assert [it for it, _ in rec_res] == list(range(9, 16))
    np.testing.assert_allclose([v for _, v in rec_res], [v for _, v in rec_full[9:]], rtol=2e-5)
    for (k, va), vb in zip(alg_full.networks.state_dict().items(), alg_res.networks.state_dict().values()):
        torch.testing.assert_close(va, vb, rtol=2e-5, atol=1e-7, msg=k)


def test_device_generator_is_seeded_from_the_run_seed():
    """Two seeds draw different device noise and replay indices; the same seed reproduces them."""
    cfg, B = synth.CONFIGS["tiny"], 64
    outs = []
    for seed in (1, 2, 1):
        alg, kw = build_alg(cfg, B, seed=seed)
        alg.networks.cuda()
        eng = alg.networks.engine()
        data = {k: torch.from_numpy(v).cuda() for k, v in synth.make_batch(cfg, B, 0).items()}
        alg.local_update(data, 0)
        torch.cuda.synchronize()
        outs.append(eng.arena_views(B)["eps1"].clone())
    assert not torch.equal(outs[0], outs[1])
    assert torch.equal(outs[0], outs[2])
