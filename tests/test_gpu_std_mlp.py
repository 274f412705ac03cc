"""The policy's "mlp_separated" / "parameter" std types (reference networks/mlp.py:43-72) on the MLP engine, through the
C ABI: against the goldens of the unmodified reference, against the pinned oracle on shapes that take every lowering (the
layer chain in its 64- and 128-row modes, per-layer wgmma groups, SIMT groups; aligned and unaligned head columns), against
the head-wise fp32 engine on the same inputs, and every entry point against `step`."""
import ast
import os

import numpy as np
import pytest
import torch

from dsac_v2_b200 import synth
from std_mlp_common import STD_TYPES, feed, make_engine, make_oracle, std_weights

pytestmark = pytest.mark.gpu
RTOL = 1e-4   # the gate of test_gpu_std.py (fp32) and of the bf16x3 golden tests
GOLDEN = {"mlp_separated": "tiny_std_separated", "parameter": "tiny_std_parameter"}


def stats_vec(eng, gb=None):
    from dsac_v2_b200.engine import STAT_KEYS
    s = eng.read_stats(gb)
    return [s[k] for k in STAT_KEYS]


def state_of(eng):
    torch.cuda.synchronize()
    return [getattr(eng, k).clone() for k in ("params", "targets", "adam_m", "adam_v")] + [eng.state[:6].clone()]


def assert_same_bits(a, b, what):
    for x, y, k in zip(a, b, ("params", "targets", "adam_m", "adam_v", "state")):
        assert torch.equal(x, y), f"{what}: {k} differs (max |d| = {(x - y).abs().max().item():.3e})"


# ---- the reference's goldens ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode,graph", [("fp32", True), ("fp32", False), ("bf16x3", True)])
@pytest.mark.parametrize("std_type", STD_TYPES)
def test_update_matches_reference_golden(golden_dir, std_type, mode, graph):
    z = np.load(os.path.join(golden_dir, GOLDEN[std_type] + ".npz"))
    cfg_name, batch, steps, over = z["meta"]
    cfg, batch, steps = synth.CONFIGS[str(cfg_name)], int(batch), int(steps)
    assert dict(ast.literal_eval(str(over)))["policy_std_type"] == std_type
    eng = make_engine(cfg, batch, std_type, mode, graph)
    names = [str(n) for n in z["param_names"]]
    atol = 1e-6 if mode == "fp32" else 1e-5
    for it in range(steps):
        eng.step(*feed(cfg, batch, it)[:1], it, feed(cfg, batch, it)[1])
        np.testing.assert_allclose(stats_vec(eng), z["tb"][it], rtol=RTOL, atol=atol, err_msg=f"tb_info at step {it}")
        if f"pdigest_{it + 1}" in z:
            w = eng.export_weights()
            for row, k in zip(z[f"pdigest_{it + 1}"], names):
                d = w[k].double().reshape(-1)
                np.testing.assert_allclose(d.abs().sum().item(), row[1], rtol=RTOL, err_msg=f"{k} step {it + 1}")
                np.testing.assert_allclose(d[:8].numpy(), row[3:3 + min(8, d.numel())], rtol=RTOL, atol=10 * atol, err_msg=f"{k} step {it + 1}")
        if f"state_{it + 1}/{names[0]}" in z:
            w = eng.export_weights()
            for k in names:
                ref = z[f"state_{it + 1}/{k}"]
                np.testing.assert_allclose(w[k].numpy(), ref, rtol=RTOL, atol=atol * max(1e-3, np.abs(ref).max()) * (1 if mode == "fp32" else 10),
                                           err_msg=f"{k} after step {it + 1}")
    eng.close()


# ---- the oracle, on every lowering ---------------------------------------------------------------------------------
WIDE_A8 = dict(obs_dim=20, act_dim=8, hidden=(300, 64), act_lim=1.5)    # a layer wider than 256: per-layer wgmma groups; A % 8 == 0
ODD_PER_LAYER = dict(obs_dim=9, act_dim=5, hidden=(100, 36), act_lim=1.0)   # a hidden width off the multiples of 8: per-layer groups, odd A
ONE_ACT = dict(obs_dim=6, act_dim=1, hidden=(32, 16), act_lim=2.0)      # act_dim 1
ORACLE_CASES = [
    ("ragged", 37, 3), ("ragged", 50, 3), ("tiny", 1, 3), ("tiny", 65, 2), ("tiny", 129, 2), ("tiny", 1000, 2),
    ("humanoid", 4096, 2),                 # act_dim 17 (odd); the policy launches past one wave: 128 rows per chain CTA
    ("asym", 70, 2), ("deep_pi", 70, 2),   # critics deeper than the policy and the reverse (act_dim 96: A % 8 == 0)
    (WIDE_A8, 70, 2), (ONE_ACT, 33, 3),
    ("ragged", 63, 2), ("ragged", 64, 2),  # the last row tile full but for a row, and full
    (ODD_PER_LAYER, 70, 2),
]
# (statistics rtol / atol, parameter atol, gradient atol as a fraction of the tensor's largest entry).  Parameters in the
# tensor-core modes: Adam's first steps move an element by up to lr = 1e-4 whatever its gradient's size, so an element
# whose gradient sits at the arithmetic's noise floor may differ by a step
# (two steps here).  Gradients: a tensor's smallest entries carry the summation-order noise of its largest (fp32: 1e-5 of
# the largest entry; bf16x3 through up to seven layers: 3e-4); single-pass bf16 is not a parity mode and is held loosely.
GATES = {"fp32": (RTOL, 2e-6, 1e-5, 1e-5), "bf16x3": (RTOL, 1e-5, 2e-4, 3e-4), "bf16": (5e-2, 3e-2, 4e-4, 2e-1)}


@pytest.mark.parametrize("mode", list(GATES))
@pytest.mark.parametrize("std_type", STD_TYPES)
@pytest.mark.parametrize("cfg_name,batch,steps", ORACLE_CASES, ids=[f"{c if isinstance(c, str) else 'A%d' % c['act_dim']}-{b}" for c, b, _ in ORACLE_CASES])
def test_update_and_gradients_match_oracle(cfg_name, batch, steps, std_type, mode):
    from oracle.dsact_oracle import TB_KEYS
    cfg = synth.mlp_config(cfg_name) if isinstance(cfg_name, str) else cfg_name
    s_rtol, s_atol, p_atol, g_frac = GATES[mode]
    eng = make_engine(cfg, batch, std_type, mode)
    orc = make_oracle(cfg, std_type)
    worst = 0.0
    for it in range(steps):
        ref = orc.update(synth.make_batch(cfg, batch, it), synth.make_noise(cfg, batch, it), it)
        eng.step(*feed(cfg, batch, it)[:1], it, feed(cfg, batch, it)[1])
        got, want = np.array(stats_vec(eng)), np.array([ref[k] for k in TB_KEYS])
        worst = max(worst, float(np.max(np.abs(got - want) / (s_atol + s_rtol * np.abs(want)))))
        np.testing.assert_allclose(got, want, rtol=s_rtol, atol=s_atol, err_msg=f"step {it}")
    g, gref = eng.export_weights(grads=True), orc.grad_dict()
    for k, v in gref.items():
        np.testing.assert_allclose(g[k].numpy(), v.numpy(), rtol=1e-3 if mode != "bf16" else 1e-1,
                                   atol=g_frac * float(v.abs().max()) + 1e-12, err_msg=f"grad {k}")
    w = eng.export_weights()
    for k, v in orc.state_dict().items():
        np.testing.assert_allclose(w[k].numpy(), v.numpy(), rtol=RTOL if mode != "bf16" else 1e-2, atol=p_atol, err_msg=k)
    print(f"[std_mlp] {std_type} {mode} B={batch}: largest statistics err/gate = {worst:.3f}")
    eng.close()


def test_gauss_distribution_matches_oracle():
    cfg, B = synth.CONFIGS["ragged"], 37
    for std_type in STD_TYPES:
        eng = make_engine(cfg, B, std_type, "bf16x3", act_dist="GaussDistribution")
        orc = make_oracle(cfg, std_type, policy_act_distribution="GaussDistribution")
        from oracle.dsact_oracle import TB_KEYS
        for it in range(3):
            ref = orc.update(synth.make_batch(cfg, B, it), synth.make_noise(cfg, B, it), it)
            eng.step(*feed(cfg, B, it)[:1], it, feed(cfg, B, it)[1])
            np.testing.assert_allclose(stats_vec(eng), [ref[k] for k in TB_KEYS], rtol=RTOL, atol=1e-5)
        eng.close()


@pytest.mark.parametrize("mode", ["fp32", "bf16x3"])
def test_clamped_log_std_row_has_zero_gradient_in_the_clamped_columns(mode):
    """A "parameter" row with entries below, inside and above [min_log_std, max_log_std]: the row's gradient (the log_std
    half's bias-gradient target) is exactly zero where the clamp is active, and the oracle's elsewhere."""
    cfg, B = synth.CONFIGS["ragged"], 50
    A = cfg["act_dim"]
    row = np.linspace(-0.9, 0.4, A).astype(np.float32)
    row[0], row[-1] = -25.0, 0.75
    w = std_weights(cfg, "parameter", row=row)
    eng = make_engine(cfg, B, "parameter", mode, weights=w)
    orc = make_oracle(cfg, "parameter", weights=w)
    orc.update(synth.make_batch(cfg, B, 0), synth.make_noise(cfg, B, 0), 0)
    b, n = feed(cfg, B, 0)
    eng.compute_grads(b, n)
    g, ref = eng.export_weights(grads=True)["policy.log_std"].reshape(-1), orc.grad_dict()["policy.log_std"].reshape(-1)
    assert g[0].item() == 0.0 and g[-1].item() == 0.0 and (g[1:-1] != 0).all()
    np.testing.assert_allclose(g.numpy(), ref.numpy(), rtol=1e-3, atol=3e-5 * float(ref.abs().max()))
    eng.close()


# ---- the two engines agree -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("std_type", STD_TYPES)
def test_mlp_engine_fp32_agrees_with_the_head_wise_engine(std_type):
    from test_gpu_std import make_engine as make_heads
    cfg, B = synth.CONFIGS["ragged"], 50
    a, h = make_engine(cfg, B, std_type, "fp32"), make_heads(cfg, B, std_type)
    for it in range(3):   # delay_update 2: iterations 0 and 2 update the policy, 1 does not
        b, n = feed(cfg, B, it)
        a.step(b, it, n)
        h.step(b, it, n)
        np.testing.assert_allclose(stats_vec(a), stats_vec(h), rtol=1e-5, atol=1e-7)
    for k in ("params", "targets", "adam_m", "adam_v"):
        x, y = getattr(a, k).double(), getattr(h, k).double()
        assert ((x - y).norm() / y.norm()).item() <= 1e-6, k
    a.close(), h.close()


# ---- every entry point against `step` ------------------------------------------------------------------------------
ROWS = 16   # at most two blocks per reduction: sums do not depend on timing, results are the same bits on every run


@pytest.mark.parametrize("mode", ["fp32", "bf16x3"])
@pytest.mark.parametrize("std_type", STD_TYPES)
def test_entry_points_equal_step(std_type, mode):
    cfg, cap = synth.CONFIGS["ragged"], 40
    ring = {k: torch.from_numpy(v).cuda() for k, v in synth.make_batch(cfg, cap, 99).items()}
    idx = torch.from_numpy(np.random.default_rng(3).integers(0, cap, (6, ROWS)))
    noise = [feed(cfg, ROWS, it)[1] for it in range(6)]
    rows = lambda k: {key: v[idx[k].cuda()].contiguous() for key, v in ring.items()}

    def fresh(fill=0.0):
        from dsac_v2_b200.engine import Engine
        from std_mlp_common import std_config
        lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
        e = Engine(std_config(cfg, std_type, 64, mode), torch.device("cuda", 0), lim, -lim, workspace_fill=fill)
        e.load_weights(std_weights(cfg, std_type))
        e.bind_replay(cap)
        e.replay_add(ring, cap, 0)
        return e

    ref = fresh()
    ref_states, ref_stats = [], []
    for k in range(6):   # across delayed-update boundaries
        ref.step(rows(k), k, noise[k])
        ref_states.append(state_of(ref))
        ref_stats.append(stats_vec(ref))
    ref.close()

    e = fresh(float("nan"))   # a poisoned workspace changes nothing
    for k in range(6):
        e.replay_step(ROWS, cap, k, idx=idx[k], noise=noise[k])
        assert_same_bits(state_of(e), ref_states[k], f"replay_step {k}")
        assert stats_vec(e) == ref_stats[k]
    e.close()

    e = fresh(1e30)
    for k in range(2):
        e.step({key: v.cpu() for key, v in rows(k).items()}, k, noise[k])   # host minibatch: dsact_step_host
        assert_same_bits(state_of(e), ref_states[k], f"step_host {k}")
    e.close()

    e = fresh()
    e.replay_step(ROWS, cap, 0, idx=idx[0], noise=noise[0])
    stack = lambda i: torch.stack([noise[k][i] for k in range(1, 6)])
    out = e.replay_steps(5, ROWS, cap, 1, idx=idx[1:6], noise=tuple(stack(i) for i in range(4)))
    assert_same_bits(state_of(e), ref_states[5], "replay_steps(5)")   # update k + 1 reads the row update k's apply wrote
    np.testing.assert_array_equal(out[:, :14].cpu().numpy(), np.array(ref_stats[1:6], dtype=np.float32))
    e.close()

    e = fresh(-1e30)   # the split calls
    for k in range(3):
        if k % 2:
            e.compute_grads(rows(k), noise[k])
        else:
            e.grad_phase1(rows(k), noise[k])
            e.grad_phase2(ROWS)
        e.apply(k)
        for x, y, name in zip(state_of(e), ref_states[k], ("params", "targets", "adam_m", "adam_v", "state")):
            torch.testing.assert_close(x, y, rtol=1e-5, atol=1e-7, msg=lambda m: f"split update {k} {name}: {m}")
    e.close()


@pytest.mark.parametrize("std_type", STD_TYPES)
def test_small_batch_after_a_large_one_equals_a_fresh_workspace(std_type):
    cfg = synth.CONFIGS["ragged"]
    a, b = make_engine(cfg, 300, std_type, "bf16x3"), make_engine(cfg, 300, std_type, "bf16x3")
    big, nb = feed(cfg, 300, 0)
    a.step(big, 0, nb)
    a.load_weights(std_weights(cfg, std_type))
    for e in (a, b):
        for k in ("adam_m", "adam_v", "state"):
            getattr(e, k).zero_()
        e.set_carry()
        small, ns = feed(cfg, ROWS, 1)
        e.step(small, 0, ns)
    assert_same_bits(state_of(a), state_of(b), "small after large")
    a.close(), b.close()


# ---- the schedule --------------------------------------------------------------------------------------------------
def step_flops(cfg, std_type, B):
    """Per class (forward, dgrad, weight gradient): 2 M N K over the GEMM problems of one step, from the shapes alone."""
    O, A = cfg["obs_dim"], cfg["act_dim"]
    hq, hp = synth.hidden_sizes(cfg)
    q, p = [O + A] + list(hq) + [2], [O] + list(hp) + [A]
    mac = lambda s, j0=0: sum(s[j] * s[j + 1] for j in range(j0, len(s) - 1))
    heads = 2 if std_type == "mlp_separated" else 1
    fwd = 6 * mac(q) + 2 * heads * mac(p)
    dgrad = 4 * mac(q, 1) + 2 * A * q[1] + heads * mac(p, 1)
    wgrad = 2 * mac(q) + heads * mac(p)
    return [2 * B * x for x in (fwd, dgrad, wgrad)]


CALLS = ("step", "step_device_noise", "replay_step", "replay_step_device_draws", "compute_grads", "apply", "grad_phase1",
         "grad_phase2", "apply_after_phases")
# (std_type, config, mode, graph) -> (launches per call of CALLS, profiled launches per class).  mlp_separated's wave A is two
# chain launches (the four policy passes, then the critics); "parameter" adds the log_std row launch to every prologue.
SCHEDULE = {
    ("mlp_separated", "humanoid", "fp32", True): ((23, 24, 24, 25, 23, 1, 10, 13, 1), [5, 8, 7, 3]),
    ("mlp_separated", "humanoid", "bf16x3", True): ((14, 14, 15, 15, 14, 1, 6, 8, 1), [6, 3, 2, 2]),
    ("mlp_separated", "humanoid", "bf16x3", False): ((13, 13, 14, 14, 14, 1, 6, 8, 1), [6, 3, 2, 2]),
    ("mlp_separated", "ragged", "bf16x3", True): ((14, 14, 15, 15, 14, 1, 6, 8, 1), [6, 3, 2, 2]),
    ("mlp_separated", "layered_q", "bf16x3", True): ((30, 30, 31, 31, 31, 1, 17, 14, 1), [6, 14, 8, 2]),
    ("parameter", "humanoid", "fp32", True): ((24, 25, 25, 26, 24, 1, 11, 13, 1), [6, 8, 7, 3]),
    ("parameter", "humanoid", "bf16x3", True): ((13, 13, 14, 14, 13, 1, 5, 8, 1), [6, 2, 2, 2]),
    ("parameter", "humanoid", "bf16x3", False): ((12, 12, 13, 13, 13, 1, 5, 8, 1), [6, 2, 2, 2]),
    ("parameter", "ragged", "bf16x3", True): ((13, 13, 14, 14, 13, 1, 5, 8, 1), [6, 2, 2, 2]),
    ("parameter", "layered_q", "bf16x3", True): ((31, 31, 32, 32, 32, 1, 18, 14, 1), [7, 14, 8, 2]),
}


@pytest.mark.parametrize("case", sorted(SCHEDULE), ids=["-".join(map(str, c)) for c in sorted(SCHEDULE)])
def test_step_schedule_is_pinned(case):
    from test_gpu_step_schedule import B, run_schedule
    std_type, cfg_name, mode, graph = case
    cfg = synth.mlp_config(cfg_name)
    eng = make_engine(cfg, B, std_type, mode, graph)
    try:
        calls, launches, flops = run_schedule(eng, cfg)
    finally:
        eng.close()
    want_calls, want_launches = SCHEDULE[case]
    assert calls == dict(zip(CALLS, want_calls))
    assert launches == want_launches
    assert flops == [0] + step_flops(cfg, std_type, B)


# ---- the drop-in ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("std_type", STD_TYPES)
def test_dropin_on_the_mlp_engine(golden_dir, std_type):
    """`DSAC_V2(policy_std_type=..., dsact_gemm="bf16x3")`: the MLP engine, the reference's goldens through `local_update`
    on host minibatches, parameters as views, `replay_updates(n)` = n rounds, and the full-state round trip."""
    import dsac_v2
    from dsac_v2_b200.engine import STAT_KEYS, Engine
    from dsac_v2_b200.engine_cnn import CnnEngine
    z = np.load(os.path.join(golden_dir, GOLDEN[std_type] + ".npz"))
    cfg, B = synth.CONFIGS["tiny"], int(z["meta"][1])
    ref_w = std_weights(cfg, std_type)

    def build():
        kw = synth.reference_kwargs(cfg, policy_std_type=std_type, replay_batch_size=B, dsact_gemm="bf16x3", dsact_noise="reference")
        alg = dsac_v2.DSAC_V2(**kw)
        sd = alg.networks.state_dict()
        assert [k for k, _ in alg.networks.named_parameters()] == [str(n) for n in z["param_names"]]
        for k, v in ref_w.items():
            sd[k] = torch.from_numpy(v)
        alg.networks.load_state_dict(sd)
        alg.networks.cuda()
        return alg

    alg = build()
    eng = alg.networks.engine(B)
    assert type(eng) is Engine and not isinstance(eng, CnnEngine) and eng.cfg.gemm_mode == 1
    for it in range(3):
        b, n = feed(cfg, B, it, device="cpu")
        eng.step(b, it, n)   # a host minibatch: host staging
        s = eng.read_stats()
        np.testing.assert_allclose([s[k] for k in STAT_KEYS], z["tb"][it], rtol=RTOL, atol=1e-5)
    key = "policy.log_std" if std_type == "parameter" else "policy.log_std.0.weight"
    assert not torch.equal(alg.networks.state_dict()[key].cpu(), torch.from_numpy(ref_w[key]))   # views see the update
    tb = alg.local_update(feed(cfg, B, 7, device="cpu")[0], 3)
    assert np.isfinite(tb["Loss/Critic loss-RL iter"]) and np.isfinite(tb["Loss/Actor loss-RL iter"])

    state = alg.full_state_dict()
    other = build()
    other.load_full_state_dict(state)
    b, n = feed(cfg, B, 9, device="cpu")
    for a in (alg, other):
        a.networks.engine(B).step(b, 4, n)
    assert_same_bits(state_of(other.networks.engine()), state_of(alg.networks.engine()), "full_state_dict round trip")


@pytest.mark.parametrize("std_type", STD_TYPES)
def test_dropin_replay_updates_is_one_engine_call_equal_to_n_rounds(std_type):
    from test_gpu_replay_steps import _alg_and_buffer, _ring, rel_l2
    kw = synth.reference_kwargs(synth.CONFIGS["tiny"], replay_batch_size=ROWS, policy_std_type=std_type, dsact_gemm="bf16x3",
                                dsact_noise="reference", seed=5)
    n, it = 5, 3
    ring = _ring(kw, 3 * ROWS + 11)
    a, abuf = _alg_and_buffer(kw, ring)
    b, bbuf = _alg_and_buffer(kw, ring)
    np.random.seed(21), torch.manual_seed(22)
    want = [dict(a.local_update(abuf.sample_batch(ROWS), it + k)) for k in range(n)]
    np.random.seed(21), torch.manual_seed(22)
    before = b.networks.engine().launch_count()
    got = b.replay_updates(bbuf, ROWS, it, n)
    eng = b.networks.engine()
    assert eng.launch_count() - before <= eng.last_call_launches() + 4   # one dsact_replay_steps call (+ counter syncs)
    for k in range(n):
        for key in want[k]:
            if "time" not in key.lower():
                np.testing.assert_allclose(got[k][key], want[k][key], rtol=1e-6, atol=1e-7, err_msg=f"update {k}: {key}")
    torch.cuda.synchronize()
    for k in ("params", "targets", "adam_m", "adam_v"):
        assert rel_l2(getattr(eng, k), getattr(a.networks.engine(), k)) <= 1e-6, k


# ---- the float64 gradient gate (tests/gradcheck64.py's rule) -------------------------------------------------------
def _f64_case(std_type, batch, clamp):
    """(weights, minibatch, noise, hyperparameter overrides).  `clamp`: log_std held above max_log_std in every row in
    component 0, below min_log_std in component 1 and across the upper bound in component 2 (gradcheck64's regime; for
    "parameter" the row's entries themselves, so component 2 stays inside)."""
    import gradcheck64 as gc
    cfg = synth.CONFIGS["ragged"]
    if not clamp:
        return std_weights(cfg, std_type), synth.make_batch(cfg, batch, 0), synth.make_noise(cfg, batch, 0), {}
    hyper = dict(gc.REGIME_HYPER["log_std_clamp"])
    if std_type == "mlp_separated":
        w, b, n = gc.inputs(gc.Case("clamp", "heads", "ragged", batch, std_type=std_type, regime="log_std_clamp"))
        return w, b, n, hyper
    row = np.array([30.0, -40.0, 0.3], dtype=np.float32)
    return std_weights(cfg, std_type, row=row), synth.make_batch(cfg, batch, 0), synth.make_noise(cfg, batch, 0), hyper


def f64_engine_grads(std_type, batch, clamp, mode):
    """The engine's step-0 gradients of one F64_CASES entry (the gradient-message seam, no graph)."""
    cfg = synth.CONFIGS["ragged"]
    w, b, n, hyper = _f64_case(std_type, batch, clamp)
    eng = make_engine(cfg, batch, std_type, mode, graph=False, weights=w,
                      **({"min_log_std": hyper["policy_min_log_std"]} if hyper else {}))
    try:
        eng.compute_grads({k: torch.from_numpy(v).cuda() for k, v in b.items()},
                          tuple(torch.from_numpy(n[i]).cuda() for i in (0, 1, 4, 5)))
        return eng.export_weights(grads=True)
    finally:
        eng.close()


# B = 2200: the four policy passes run as one ping-pong chain launch (4 x 35 row tiles, more than one wave), their heads
# writing the [B, 2A] logits at a pitch
F64_CASES = [(s, b, False) for s in STD_TYPES for b in (200, 1000, 2200)] + [(s, 1000, True) for s in STD_TYPES]
# "parameter" at B = 200 in bf16x3: the mean network's first-layer weight gradient comes out at 1.09 x the 1e-5 floor on an
# H100 (its ref_k is far below the floor, so the floor is the gate).  The same case in fp32, which runs the same pass
# table, pitches and bias-gradient targets, stays at 0.3 of a floor five times tighter, so the excess is the split-bf16
# operand rounding carried through the three dgrad GEMMs above that layer, as for gradcheck64's layered_q; that case's
# bf16x3 gates are doubled like layered_q's, and the power rule still has to hold for the doubled gate.  At B = 2200 the
# same tensor comes out at 1.03 x the floor, and the float64 oracle with every GEMM restated as split-bf16 products at
# 0.94 x (at B = 200: 1.07 x against the engine's 1.09 x; tests/test_grad_rounded.py recomputes both); its gates are
# doubled too.
F64_BF16X3_SCALE = {("parameter", 200, False): 2.0, ("parameter", 2200, False): 2.0}


@pytest.mark.parametrize("mode", ["fp32", "bf16x3"])
@pytest.mark.parametrize("std_type,batch,clamp", F64_CASES)
def test_gradients_within_the_float64_gate(std_type, batch, clamp, mode):
    """err_k <= max(c ref_k, floor) for every gradient tensor, with gate_k <= signal_k / 5 (a lost row tile would show)."""
    import gradcheck64 as gc
    cfg = synth.CONFIGS["ragged"]
    w, b, n, hyper = _f64_case(std_type, batch, clamp)

    def oracle_grads(dtype, rows=None):
        orc = make_oracle(cfg, std_type, weights=w, dtype=dtype, **hyper)
        bb, nn = (b, n) if rows is None else ({k: v[:rows] for k, v in b.items()}, [x[:rows] for x in n])
        orc.compute_gradients(bb, nn)
        return {k: g.detach().double() for k, g in orc.grad_dict().items()}

    g64, g32 = oracle_grads(torch.float64), oracle_grads(torch.float32)
    gcut = oracle_grads(torch.float64, gc.TILE * ((batch - 1) // gc.TILE))
    g = f64_engine_grads(std_type, batch, clamp, mode)
    c, floor = gc.GATES[mode]
    worst = 0.0
    for k in g64:
        scale = F64_BF16X3_SCALE.get((std_type, batch, clamp), 1.0) if mode == "bf16x3" else 1.0
        err, gate, signal = gc.rel(g[k], g64[k]), scale * max(c * gc.rel(g32[k], g64[k]), floor), gc.rel(gcut[k], g64[k])
        assert err <= gate, (k, err, gate)
        assert gate <= signal / gc.POWER, (k, gate, signal)
        worst = max(worst, err / gate)
    print(f"[std_mlp f64] {std_type} {mode} B={batch} clamp={clamp}: largest err/gate = {worst:.2f}")
    if clamp:   # the clamped components' gradient is exactly zero
        key = "policy.log_std" if std_type == "parameter" else gc.log_std_bias(gc.Case("c", "heads", "ragged", batch, std_type=std_type))[0]
        v = g[key].reshape(-1)
        assert v[gc.CLAMPED_HIGH].item() == 0.0 and v[gc.CLAMPED_LOW].item() == 0.0 and v[2].item() != 0.0


# ---- kernel level --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["bf16x3", "bf16"])
@pytest.mark.parametrize("A,M", [(17, 200), (8, 65), (1, 64), (17, 2200)])
def test_chain_head_store_at_a_pitch_leaves_the_other_columns_alone(A, M, mode):
    """One launch of the layer-chain kernel with the same input three times: the head stored contiguously, into columns
    [0, A) and into columns [A, 2A) of NaN-filled [M, 2A] rows.  The three results are the same bits and the columns a head
    does not own stay NaN.  Four passes of 2200 rows are 140 CTAs of 64 rows, past one wave of an H100's 132 SMs, where the
    kernel carries 128 rows per CTA."""
    cfg = synth.CONFIGS["tiny"]
    eng = make_engine(cfg, 4, "mlp_separated", mode)
    g = torch.Generator().manual_seed(A * 1000 + M)
    sizes = [11, 40, 72, A]
    params = torch.cat([torch.randn(sizes[j + 1] * sizes[j] + sizes[j + 1], generator=g) / sizes[j] ** 0.5 for j in range(3)]).cuda()
    x = torch.randn(M, sizes[0], generator=g).cuda()
    nan = float("nan")
    dense = torch.full((M, A), nan, device="cuda")
    left, right, both = (torch.full((M, 2 * A), nan, device="cuda") for _ in range(3))
    passes = [dict(M=M, x0=x, out=dense), dict(M=M, x0=x, out=left, out_ld=2 * A), dict(M=M, x0=x, out=right[:, A:], out_ld=2 * A),
              dict(M=M, x0=x, out=both[:, A:], out_ld=2 * A)]
    eng.test_chain(False, sizes, sizes[0], 0, 0, 2, params, passes)
    eng.test_chain(False, sizes, sizes[0], 0, 0, 2, params, [dict(M=M, x0=x, out=both, out_ld=2 * A)])
    torch.cuda.synchronize()
    assert torch.isfinite(dense).all()
    assert dense.abs().max() > 0
    assert torch.equal(left[:, :A], dense) and torch.isnan(left[:, A:]).all()
    assert torch.equal(right[:, A:], dense) and torch.isnan(right[:, :A]).all()
    assert torch.equal(both, torch.cat([dense, dense], 1))
    eng.close()


@pytest.mark.parametrize("mode", ["bf16x3", "bf16"])
def test_policy_grad_split_images_are_the_halves_of_the_whole_image(mode):
    """policy_grad_kernel through dsact_test_rows: the mean and log_std images it writes for two policy heads are, bit for
    bit, columns [0, A) and [A, 2A) of the one image it writes for mlp_shared; with a log_std row only the mean image is
    written; the fp32 gradient and the bias-gradient targets are the same in all three."""
    cfg, B = synth.CONFIGS["humanoid"], 200
    A = cfg["act_dim"]
    eng = make_engine(cfg, B, "mlp_separated", mode)
    g = torch.Generator().manual_seed(5)
    logits = torch.randn(B, 2 * A, generator=g).cuda()
    logits[::5, A] = 1.0      # above max_log_std: a clamped entry
    eps, d1, d2 = (torch.randn(B, A, generator=g).cuda() for _ in range(3))
    pa, pw = (A + 7) // 8 * 8, (2 * A + 7) // 8 * 8
    poison = lambda *shape: torch.full(shape, float("nan"), dtype=torch.bfloat16, device="cuda")

    def run(**img):
        out = dict(d=torch.full((B, 2 * A), float("nan"), device="cuda"), gb=torch.zeros(A, device="cuda"), gl=torch.zeros(A, device="cuda"))
        eng.test_rows("policy_grad", B, logits=[logits, None], eps=[eps, None], d_act=[d1, d2], d_logits=out["d"],
                      gbias_pi=out["gb"], gbias_ls=out["gl"], **img)
        torch.cuda.synchronize()
        return out

    whole, mean, ls, mean_only = poison(2, B, pw), poison(2, B, pa), poison(2, B, pa), poison(2, B, pa)
    a = run(img_dlogits=whole)
    b = run(img_dlogits=mean, img_dlogits_ls=ls, split_dlogits=1)
    c = run(img_dlogits=mean_only, split_dlogits=1)
    planes = 2 if mode == "bf16x3" else 1
    bits = lambda t: t.view(torch.int16)
    assert torch.equal(bits(mean[:planes, :, :A]), bits(whole[:planes, :, :A]))
    assert torch.equal(bits(ls[:planes, :, :A]), bits(whole[:planes, :, A:2 * A]))
    assert torch.equal(bits(mean_only[:planes, :, :A]), bits(whole[:planes, :, :A]))
    assert torch.isnan(mean[:, :, A:]).all() and torch.isnan(ls[:, :, A:]).all()   # nothing past a head's A columns
    hi = whole[0, :, :2 * A].float()
    assert torch.equal(hi, a["d"].bfloat16().float())                                 # round-to-nearest split of the fp32 gradient
    for o in (b, c):
        assert torch.equal(o["d"], a["d"])
        torch.testing.assert_close(o["gb"], a["gb"], rtol=1e-5, atol=1e-7)
        torch.testing.assert_close(o["gl"], a["gl"], rtol=1e-5, atol=1e-7)
    assert (a["d"][::5, A] == 0).all()
    eng.close()


def test_peer_data_parallel_calls_refuse_these_std_types():
    """dsact_dp_* on the MLP engine serve mlp_shared; the drop-in takes the all-reduce transport for the other std types."""
    from dsac_v2_b200._lib import DsactError
    for std_type in STD_TYPES:
        eng = make_engine(synth.CONFIGS["tiny"], 4, std_type)
        with pytest.raises(DsactError, match="mlp_shared"):
            eng.dp_export()
        eng.close()
