"""DSAC_V1 on the MLP engine (`dsact_v1_create`: one critic, flat layout [q | policy | log_alpha]) in its three arithmetics:
against the reference's DSAC_V1 goldens, against the float64 oracle with gates checked for their own power, against the
head-wise fp32 engine on the same inputs, through the replay-fed step and the device generator, on a poisoned workspace,
and through the drop-in `dsac_v1.DSAC_V1(dsact_gemm=...)` and its trainer."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

import gradcheck64 as gc
from dsac_v2_b200 import _lib, synth
from v1_mlp_common import GOLDENS, V1_COLS, engine_noise, golden, make_engine, v1_oracle

pytestmark = pytest.mark.gpu
RTOL = 1e-4


def stats_v1(eng):
    from dsac_v2_b200.engine import STAT_KEYS
    s = eng.read_stats()
    v = [s[k] for k in STAT_KEYS]
    return np.array([v[i] for i in V1_COLS])


def feed(cfg, batch, it):
    b = {k: torch.from_numpy(v).cuda() for k, v in synth.make_batch(cfg, batch, it).items()}
    return b, tuple(torch.from_numpy(x).cuda() for x in engine_noise(synth.make_noise(cfg, batch, it)))


def rel_l2(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / max(float(b.norm()), 1e-30))


# ---- 1. the reference's goldens ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode,graph", [("fp32", True), ("fp32", False), ("bf16x3", True)])
@pytest.mark.parametrize("name", GOLDENS)
def test_v1_mlp_matches_reference_golden(golden_dir, name, mode, graph):
    z, cfg, batch, steps, hyper = golden(golden_dir, name)
    eng = make_engine(cfg, batch, hyper, mode, graph)
    names = [str(n) for n in z["param_names"]]
    atol = 1e-6 if mode == "fp32" else 1e-5
    for it in range(steps):
        b, n = feed(cfg, batch, it)
        eng.step(b, it, n)
        np.testing.assert_allclose(stats_v1(eng), z["tb"][it], rtol=RTOL, atol=atol, err_msg=f"{name} {mode} tb_info at step {it}")
        if f"pdigest_{it + 1}" in z:
            w = eng.export_weights()
            for row, k in zip(z[f"pdigest_{it + 1}"], names):
                d = w[k].double().reshape(-1)
                np.testing.assert_allclose(d.abs().sum().item(), row[1], rtol=RTOL, err_msg=f"{name} {k} step {it + 1}")
                if mode == "fp32":
                    np.testing.assert_allclose(d[:8].numpy(), row[3:3 + min(8, d.numel())], rtol=RTOL, atol=1e-7,
                                               err_msg=f"{name} {k} step {it + 1}")
        if mode == "fp32" and f"state_{it + 1}/{names[0]}" in z:
            w = eng.export_weights()
            for k in names:
                ref = z[f"state_{it + 1}/{k}"]
                np.testing.assert_allclose(w[k].numpy(), ref, rtol=RTOL, atol=1e-6 * max(1e-3, np.abs(ref).max()),
                                           err_msg=f"{name} {k} after step {it + 1}")
    eng.close()


# ---- 2. the float64 oracle ---------------------------------------------------------------------------------------------
def _v1_case(name, cfg_name, batch, hyper=(), bf16x3_scale=1.0):
    return gc.Case(name, "mlp", cfg_name, batch, algo="DSAC_V1", hyper=tuple(hyper), bf16x3_scale=bf16x3_scale)


HOPPER_HYPER = (("TD_bound", 10.0), ("gamma", 0.999))
# ragged at the tile edges and multi-tile, the reference example's shape, critics and policy of different shapes, and a
# TD bound that clips (v1_ragged_tight's), and asym at a batch whose chain launches all run on the ping-pong kernel.
# layered_q's six tanh critic layers: bf16x3 gates doubled, as in gradcheck64.
F64_CASES = {c.name: c for c in [_v1_case(f"v1mlp_ragged_b{b}", "ragged", b) for b in (63, 65, 129, 1000)] + [
    _v1_case("v1mlp_hopper_b256", "hopper", 256, HOPPER_HYPER)] + [
    _v1_case(f"v1mlp_{n}_b200", n, 200, bf16x3_scale=2.0 if n == "layered_q" else 1.0) for n in synth.ASYM_CONFIGS] + [
    _v1_case("v1mlp_tight_ragged_b129", "ragged", 129, (("TD_bound", 0.5), ("delay_update", 3))),
    # one critic: launches of 3, 2 and 2 passes, each more than one wave of row tiles at B = 4300 (the ping-pong kernel)
    _v1_case("v1mlp_asym_b4300", "asym", 4300)]}


def _oracle_grads(case, dtype, rows=None):
    w, b, n = gc.inputs(case)
    orc = v1_oracle(case.cfg, w, **dict(case.hyperparameters, dtype=dtype, policy_act_distribution=case.act_dist))
    if rows is not None:
        b, n = {k: v[:rows] for k, v in b.items()}, [x[:rows] for x in n]
    tb = orc.compute_gradients(b, n)
    return {k: g.detach().double() for k, g in orc.grad_dict().items()}, tb


@functools.lru_cache(maxsize=None)
def reference(name):
    """gradcheck64.reference for the cases of this file (float64 yardstick, float32 oracle, float64 without the last tile)."""
    case = F64_CASES[name]
    g64, tb64 = _oracle_grads(case, torch.float64)
    g32, tb32 = _oracle_grads(case, torch.float32)
    cut = gc.TILE * ((case.batch - 1) // gc.TILE)
    gcut = _oracle_grads(case, torch.float64, rows=cut)[0] if cut > 0 else None
    ref = {k: gc.rel(g32[k], g64[k]) for k in g64}
    signal = {k: (gc.rel(gcut[k], g64[k]) if gcut is not None else 1.0) for k in g64}
    return gc.Reference(g64, tb64, tb32, ref, signal)


def gates(name, mode):
    c, floor = gc.GATES[mode]
    scale = F64_CASES[name].bf16x3_scale if mode == "bf16x3" else 1.0
    return {k: scale * max(c * r, floor) for k, r in reference(name).ref.items()}


def engine_grads(case, mode):
    """One whole step (DSAC_V1 has no gradient-message seam): the gradient buffer holds the step's gradients."""
    from dsac_v2_b200.engine import Engine
    from v1_mlp_common import engine_config
    w, b, n = gc.inputs(case)
    c, v1 = engine_config(case.cfg, case.batch, dict(case.hyperparameters, policy_act_distribution=case.act_dist), mode, False)
    lim = torch.full((case.cfg["act_dim"],), case.cfg["act_lim"])
    eng = Engine(c, torch.device("cuda", 0), lim, -lim, v1=v1)
    try:
        eng.load_weights(w)
        eng.step({k: torch.from_numpy(v).cuda() for k, v in b.items()}, 0, tuple(torch.from_numpy(x).cuda() for x in engine_noise(n)))
        g = eng.export_weights(grads=True)
        s = stats_v1(eng)
    finally:
        eng.close()
    from oracle.dsact_oracle import V1_TB_KEYS
    return g, dict(zip(V1_TB_KEYS, s))


@pytest.mark.parametrize("mode", ["fp32", "bf16x3"])
@pytest.mark.parametrize("name", list(F64_CASES))
def test_v1_mlp_gradients_against_float64(name, mode):
    r = reference(name)
    gate = gates(name, mode)
    weak = {k: (g, r.signal[k]) for k, g in gate.items() if not g <= r.signal[k] / gc.POWER}
    assert not weak, f"gates that would not notice a lost row tile: {weak}"
    g, tb = engine_grads(F64_CASES[name], mode)
    bad = {k: (gc.rel(g[k], r.g64[k]), gate[k]) for k in r.g64 if not gc.rel(g[k], r.g64[k]) <= gate[k]}
    worst = max(gc.rel(g[k], r.g64[k]) / gate[k] for k in r.g64)
    print(f"{name} {mode}: largest err_k / gate_k = {worst:.2f}")
    assert not bad, bad
    c = gc.GATES[mode][0]
    for k, want in r.tb64.items():
        tol = max(gc.TB_RTOL * max(1.0, abs(want)), c * abs(r.tb32[k] - want))
        assert abs(tb[k] - want) <= tol, (k, tb[k], want, tol)


# ---- 3. the head-wise engine on the same inputs --------------------------------------------------------------------------
def _heads_engine(cfg, B, hyper):
    from dsac_v2_b200.engine_cnn import CnnEngine, make_heads_config
    c = make_heads_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], "mlp_shared", max_batch=B, algo="DSAC_V1",
                          bound=hyper.get("bound", True), td_bound=hyper.get("TD_bound", 20), gamma=hyper["gamma"], tau=hyper["tau"],
                          delay_update=hyper["delay_update"], auto_alpha=hyper["auto_alpha"], alpha=hyper["alpha"],
                          lr_q=hyper["value_learning_rate"], lr_pi=hyper["policy_learning_rate"], lr_alpha=hyper["alpha_learning_rate"],
                          min_log_std=hyper["policy_min_log_std"], max_log_std=hyper["policy_max_log_std"])
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    eng = CnnEngine(c, torch.device("cuda", 0), lim, -lim)
    eng.load_weights(synth.make_weights_v1(cfg))
    return eng


def test_v1_mlp_fp32_equals_the_head_wise_engine():
    """20 steps with the same weights, host noise and minibatches: parameters, targets, Adam moments and statistics agree to
    ~1e-6.  Both engines draw device noise with the same generator (noise_body at the same seed and counter), so one more
    step with device noise must see the same draws, bit for bit, and stay within the same agreement."""
    cfg, B, hyper = synth.CONFIGS["ragged"], 100, dict(synth.HYPER)
    a, b = make_engine(cfg, B, hyper, "fp32", True), _heads_engine(cfg, B, hyper)
    a.seed(77)
    b.seed(77)
    for it in range(20):
        bt = {k: torch.from_numpy(v) for k, v in synth.make_batch(cfg, B, it).items()}
        nz = engine_noise(synth.make_noise(cfg, B, it))
        a.step({k: v.cuda() for k, v in bt.items()}, it, tuple(torch.from_numpy(x) for x in nz))
        b.step(bt, it, tuple(torch.from_numpy(x) for x in nz))
        np.testing.assert_allclose(stats_v1(a), stats_v1(b), rtol=2e-6, atol=1e-7, err_msg=f"step {it}")
    torch.cuda.synchronize()
    for k in ("params", "targets", "adam_m", "adam_v"):
        assert rel_l2(getattr(a, k), getattr(b, k)) <= 1e-6, (k, rel_l2(getattr(a, k), getattr(b, k)))
    bt = {k: torch.from_numpy(v).cuda() for k, v in synth.make_batch(cfg, B, 20).items()}
    a.step(bt, 20, None)
    b.step(bt, 20, None)
    va, vb = a.arena_views(B), b.arena_views(B)
    for k in ("eps1", "eps2", "z3"):
        assert torch.equal(va[k], vb[k]), k
    np.testing.assert_allclose(stats_v1(a), stats_v1(b), rtol=2e-6, atol=1e-7)
    for k in ("params", "targets", "adam_m", "adam_v"):
        assert rel_l2(getattr(a, k), getattr(b, k)) <= 1e-6, k
    a.close(); b.close()


# ---- 4. the replay-fed step -----------------------------------------------------------------------------------------
def _ring(cfg, cap, seed=11):
    g = np.random.default_rng(seed)
    O, A, lim = cfg["obs_dim"], cfg["act_dim"], cfg["act_lim"]
    return {"obs": g.standard_normal((cap, O)).astype(np.float32), "obs2": g.standard_normal((cap, O)).astype(np.float32),
            "act": g.uniform(-lim, lim, (cap, A)).astype(np.float32), "rew": g.standard_normal(cap).astype(np.float32),
            "done": (g.random(cap) < 0.05).astype(np.float32), "logp": g.standard_normal(cap).astype(np.float32)}


def _bind(eng, host):
    cap = host["obs"].shape[0]
    eng.bind_replay(cap)
    eng.replay_add({k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in host.items()}, cap, 0)


def _rows(host, idx):
    return {k: host[k][idx] for k in ("obs", "act", "rew", "obs2", "done")}


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("mode", list(_lib.GEMM_MODES))
def test_v1_replay_step_equals_step_on_the_gathered_rows(mode, graph):
    cfg, B, hyper = synth.CONFIGS["ragged"], 16, dict(synth.HYPER)
    a, b = make_engine(cfg, B, hyper, mode, graph), make_engine(cfg, B, hyper, mode, graph)
    cap = 50
    host = _ring(cfg, cap)
    _bind(a, host)
    g = np.random.default_rng(5)
    for it in range(3):
        idx = g.integers(0, cap, B)
        nz = tuple(torch.from_numpy(x) for x in engine_noise(synth.make_noise(cfg, B, it)))
        a.replay_step(B, cap, it, idx=torch.from_numpy(idx), noise=nz)
        b.step({k: torch.from_numpy(v).cuda() for k, v in _rows(host, idx).items()}, it, nz)
        np.testing.assert_array_equal(stats_v1(a), stats_v1(b), err_msg=f"stats step {it}")
    torch.cuda.synchronize()
    for k in ("params", "targets", "adam_m", "adam_v"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k
    a.close(); b.close()


@pytest.mark.parametrize("mode", ["fp32", "bf16x3"])
def test_v1_replay_draws_equal_the_restatement(mode):
    """Device-drawn indices bit for bit and device noise within a few ulps of oracle/dsact_rng.py, the step against the
    oracle on the restated draws, and a replayed graph that follows a changed ring size."""
    from oracle.dsact_oracle import V1_TB_KEYS
    from oracle.dsact_rng import device_noise, replay_indices
    cfg, B, hyper, seed = synth.CONFIGS["ragged"], 37, dict(synth.HYPER), 0x0123456789ABCDEF
    eng = make_engine(cfg, B, hyper, mode, True)
    eng.seed(seed)
    cap = 90
    host = _ring(cfg, cap)
    _bind(eng, host)
    orc = v1_oracle(cfg, synth.make_weights_v1(cfg), **hyper)
    for it, size in enumerate((cap - 5, cap - 5, 20, cap - 5)):
        torch.cuda.synchronize()
        c = int(eng.state.view(torch.int32)[10].item()) & 0xFFFFFFFF
        eng.replay_step(B, size, it)
        idx = replay_indices(seed, c, B, size)
        np.testing.assert_array_equal(eng.arena_views(B)["idx"].cpu().numpy(), idx)
        eps1, eps2, z3, _ = device_noise(seed, c, B, cfg["act_dim"])
        v = eng.arena_views(B)
        for k, r in (("eps1", eps1), ("eps2", eps2), ("z3", z3)):
            np.testing.assert_allclose(v[k].cpu().numpy(), r, rtol=1e-5, atol=1e-6, err_msg=k)
        f = lambda x: np.asarray(x, dtype=np.float32)
        z = np.zeros_like(f(z3))
        ref = orc.update(_rows(host, idx), [f(eps1), f(eps2), z, f(z3), z], it)
        np.testing.assert_allclose(stats_v1(eng), [ref[k] for k in V1_TB_KEYS], rtol=RTOL, atol=1e-5, err_msg=f"step {it}")
    eng.close()


# ---- 5. a poisoned workspace -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("mode", list(_lib.GEMM_MODES))
def test_v1_poisoned_workspace_changes_nothing(mode, graph):
    """NaN and +-1e30 over the whole workspace (but the slabs dsact_bind zeroes) before every call: the same results as a
    clean run.  Then a small step after the large ones."""
    from test_gpu_workspace import poison_workspace
    cfg, hyper = synth.CONFIGS["ragged"], dict(synth.HYPER)
    runs = []
    for poison in (None, float("nan"), 1e30, -1e30):
        eng = make_engine(cfg, 200, hyper, mode, graph)
        stats = []
        for it, B in enumerate((200, 130, 200, 7)):
            if poison is not None:
                poison_workspace(eng, poison)
            b, n = feed(cfg, B, it)
            eng.step(b, it, n)
            stats.append(stats_v1(eng))
        torch.cuda.synchronize()
        runs.append((np.array(stats), eng))
    (s0, e0) = runs[0]
    assert np.all(np.isfinite(s0))
    for s, e in runs[1:]:
        # above 16 rows the float atomics of the bias gradients may sum in another order
        np.testing.assert_allclose(s, s0, rtol=1e-5 if mode != "bf16" else 1e-4, atol=1e-7)
        for k in ("params", "targets", "adam_m", "adam_v"):
            assert torch.isfinite(getattr(e, k)).all(), k
            assert rel_l2(getattr(e, k), getattr(e0, k)) <= (1e-6 if mode != "bf16" else 1e-4), k
    for _, e in runs:
        e.close()


# ---- 6. the drop-in ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", list(_lib.GEMM_MODES))
def test_v1_dropin_on_the_mlp_engine(golden_dir, mode):
    import dsac_v1
    from dsac_v2_b200.engine import Engine
    from oracle.dsact_oracle import V1_TB_KEYS
    z, cfg, B, steps, hyper = golden(golden_dir, "v1_tiny_b16")
    kw = synth.reference_kwargs(cfg, algorithm="DSAC_V1", replay_batch_size=B, dsact_gemm=mode)
    alg = dsac_v1.DSAC_V1(**kw)
    sd = alg.networks.state_dict()
    ref_w = synth.make_weights_v1(cfg)
    assert {k for k in sd if not k.endswith("_lim")} == set(ref_w) | {"log_alpha"}
    assert [k for k, _ in alg.networks.named_parameters()] == [str(n) for n in z["param_names"]]
    for k, v in ref_w.items():
        assert tuple(sd[k].shape) == v.shape, k
        sd[k] = torch.from_numpy(v)
    alg.networks.load_state_dict(sd)
    alg.networks.cuda()
    eng = alg.networks.engine(B)
    assert type(eng) is Engine and eng.v1 is not None
    # the parameters are views of the flat buffers
    ptrs = {p.data_ptr() for p in alg.networks.parameters()}
    assert eng.params.data_ptr() in ptrs and eng.targets.data_ptr() in ptrs
    assert alg.networks.log_alpha.data_ptr() == eng.params[-1:].data_ptr()
    for it in range(3):
        b, n = feed(cfg, B, it)
        eng.step(b, it, n)
        if mode != "bf16":
            np.testing.assert_allclose(stats_v1(eng), z["tb"][it], rtol=RTOL, atol=1e-5)
    for it, data in ((3, {k: torch.from_numpy(v) for k, v in synth.make_batch(cfg, B, 9).items()}),                 # host
                     (4, {k: torch.from_numpy(v).cuda() for k, v in synth.make_batch(cfg, B, 10).items()})):       # device
        tb = alg.local_update(data, it)
        assert set(V1_TB_KEYS) <= set(tb) and all(np.isfinite(tb[k]) for k in V1_TB_KEYS)
    with pytest.raises(NotImplementedError):
        alg.get_remote_update_info({}, 0)
    with pytest.raises(NotImplementedError):
        alg.remote_update({})


def test_v1_dropin_without_dsact_gemm_stays_head_wise():
    import dsac_v1
    from dsac_v2_b200.engine_cnn import CnnEngine
    alg = dsac_v1.DSAC_V1(**synth.reference_kwargs(synth.CONFIGS["tiny"], algorithm="DSAC_V1", replay_batch_size=8))
    alg.networks.cuda()
    assert isinstance(alg.networks.engine(), CnnEngine)


def test_v1_dropin_with_different_critic_and_policy():
    """An ASYM_CONFIGS shape through the drop-in: a host-minibatch local_update against the oracle."""
    import dsac_v1
    from oracle.dsact_oracle import V1_TB_KEYS
    cfg, B = synth.ASYM_CONFIGS["asym"], 70
    alg = dsac_v1.DSAC_V1(**synth.reference_kwargs(cfg, algorithm="DSAC_V1", replay_batch_size=B, dsact_gemm="fp32",
                                                   dsact_noise="reference"))
    sd = alg.networks.state_dict()
    w = synth.make_weights_v1(cfg)
    sd.update({k: torch.from_numpy(v) for k, v in w.items()})
    alg.networks.load_state_dict(sd)
    alg.networks.cuda()
    torch.manual_seed(0)
    tb = alg.local_update({k: torch.from_numpy(v) for k, v in synth.make_batch(cfg, B, 0).items()}, 0)
    torch.manual_seed(0)   # the same five draws the drop-in made, in the reference's order
    A = cfg["act_dim"]
    noise = [torch.empty(B, A).normal_().numpy(), torch.empty(B, A).normal_().numpy()] + \
            [torch.normal(torch.zeros(B), torch.ones(B)).numpy() for _ in range(3)]
    ref = v1_oracle(cfg, w, **synth.HYPER).update(synth.make_batch(cfg, B, 0), noise, 0)
    np.testing.assert_allclose([tb[k] for k in V1_TB_KEYS], [ref[k] for k in V1_TB_KEYS], rtol=RTOL, atol=1e-6)


@pytest.mark.parametrize("mode", ["fp32", "bf16x3"])
def test_v1_trainer_on_the_mlp_engine(tmp_path, mode):
    """`OffSerialTrainer` (replay ring attached to the engine, `ReplayBuffer.sample_batch`) for a few dozen iterations."""
    from test_gpu_v1_heads import make_trainer
    trainer, alg, rec = make_trainer("v1_mlp", tmp_path, sample_interval=4, dsact_gemm=mode)
    trainer.max_iteration = 36
    from dsac_v2_b200.engine import Engine
    assert type(alg.networks.engine()) is Engine
    assert trainer.buffer.engine is alg.networks.engine()
    first = next(iter(alg.networks.policy.parameters())).detach().clone()
    trainer.train()
    assert trainer.iteration == 36 and [it for it, _ in rec] == list(range(36))
    assert all(np.isfinite(v) for _, v in rec)
    now = next(iter(alg.networks.policy.parameters())).detach()
    assert not torch.equal(first, now)
    trainer.refresh_policy_mirror()
    torch.testing.assert_close(next(iter(trainer.sampler.networks.policy.parameters())).detach(), now.cpu(), rtol=0, atol=0)


@pytest.mark.parametrize("mode", ["fp32", "bf16x3"])
def test_v1_trainer_resume_is_bit_identical(tmp_path, mode):
    from test_gpu_v1_heads import make_trainer
    full, alg_full, rec_full = make_trainer("v1_mlp", tmp_path / "full", dsact_full_checkpoint=True, sample_interval=1000,
                                            dsact_gemm=mode)
    full.train()
    ck = tmp_path / "full" / "apprfunc" / "trainstate_8.pkl"
    resumed, alg_res, rec_res = make_trainer("v1_mlp", tmp_path / "resumed", dsact_full_checkpoint=True, sample_interval=1000,
                                             dsact_resume_dir=str(ck), dsact_gemm=mode)
    assert resumed.iteration == 9
    resumed.train()
    assert [v for _, v in rec_res] == [v for _, v in rec_full[9:]]
    sd_full, sd_res = alg_full.networks.state_dict(), alg_res.networks.state_dict()
    for k in sd_full:
        assert torch.equal(sd_full[k], sd_res[k]), k
    ef, er = alg_full.networks.engine(), alg_res.networks.engine()
    for name in ("params", "targets", "adam_m", "adam_v"):
        assert torch.equal(getattr(ef, name), getattr(er, name)), name


# ---- 7. refused calls ------------------------------------------------------------------------------------------------
def test_v1_mlp_refuses_the_split_and_data_parallel_calls():
    from dsac_v2_b200._lib import Batch
    cfg, B = synth.CONFIGS["tiny"], 8
    eng = make_engine(cfg, B, dict(synth.HYPER), "bf16x3", True)
    lib, h = eng.lib, eng.h
    b, n = feed(cfg, B, 0)
    bt = Batch(b["obs"].data_ptr(), b["act"].data_ptr(), b["rew"].data_ptr(), b["obs2"].data_ptr(), b["done"].data_ptr(), B, None)
    s = eng._stream()
    eng.bind_replay(32)
    buf = C.create_string_buffer(_lib.IPC_HANDLE_BYTES)
    calls = [lambda: lib.dsact_grad_phase1(h, C.byref(bt), None, s), lambda: lib.dsact_grad_phase2(h, B, s),
             lambda: lib.dsact_compute_grads(h, C.byref(bt), None, s), lambda: lib.dsact_apply(h, 0, s),
             lambda: lib.dsact_dp_export(h, buf, None), lambda: lib.dsact_dp_connect(h, 0, 2, buf.raw * 2),
             lambda: lib.dsact_dp_step(h, C.byref(bt), None, 2 * B, 0, s),
             lambda: lib.dsact_dp_replay_step(h, B, 32, None, None, 2 * B, 0, s)]
    for i, call in enumerate(calls):
        rc = call()
        assert rc == -1, (i, rc)
        assert b"DSAC_V1" in lib.dsact_last_error(), (i, lib.dsact_last_error())
    eng.step(b, 0, n)   # the handle still steps
    assert np.all(np.isfinite(stats_v1(eng)))
    eng.close()
