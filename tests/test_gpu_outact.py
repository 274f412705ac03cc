"""Non-linear output activations (the reference's value_output_activation / policy_output_activation) on the GPU.

- The goldens of tests/golden/make_golden_outact.py (the unmodified reference) on every engine route the drop-in takes:
  the MLP engine in fp32 and bf16x3, with captured graphs and eagerly; the head-wise engine for the std types without
  `dsact_gemm`, for the CNN approximators and for DSAC_V1; DSAC_V1 on the MLP engine.  Gates as tests/test_gpu_parity.py.
- Step-0 gradients at a ragged multi-tile batch against the float64 oracle (tests/gradcheck64.py's gates and power rule).
- At <= 16 rows, bit for bit: replay_steps(n) = n replay_step calls, compute_grads + apply = step, one W = 2 dsact_dp_step
  on one device = the split API with host exchanges, and an explicit linear dsact_set_output_activations = no call.
- dsact_set_output_activations' refusals.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import gradcheck64 as G
import outact_oracle
from dsac_v2_b200 import _lib, synth
from dsac_v2_b200.engine import STAT_KEYS
from test_gpu_replay_step import SEED, bind_ring, ring_rows
from test_oracle_golden import load

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL = 1e-4
V1_COLS = [0, 2, 6, 8, 9, 10, 11]

# golden -> routes: ("mlp", gemm, graph) = the MLP engine through `dsact_gemm`; ("heads",) = the head-wise engine
MLP_ROUTES = [("mlp", "fp32", True), ("mlp", "fp32", False), ("mlp", "bf16x3", True), ("mlp", "bf16x3", False)]
# (the std types: the head-wise engine without `dsact_gemm`, the MLP engine with it)
GOLDEN_ROUTES = [(g, r) for g in ("outact_tiny_tanh", "outact_tiny_relu_pi", "outact_ragged_sigmoid_q", "outact_gauss",
                                  "outact_std_separated", "outact_std_parameter")
                 for r in MLP_ROUTES] + [
    ("outact_std_separated", ("heads",)), ("outact_std_parameter", ("heads",)), ("outact_cnn_type1", ("heads",)),
    ("outact_v1_tiny", ("heads",)), ("outact_v1_tiny", ("mlp", "fp32", True)), ("outact_v1_tiny", ("mlp", "fp32", False)),
    ("outact_v1_tiny", ("mlp", "bf16x3", True)), ("outact_v1_std_separated", ("heads",)), ("outact_v1_cnn_type1", ("heads",))]


def _dropin(cfg, B, over, route, **extra):
    """DSAC_V2 / DSAC_V1 of the drop-in from the reference's kwargs, on `route`, with the case's weights, on cuda:0."""
    import dsac_v1
    import dsac_v2
    v1 = over.get("algorithm") == "DSAC_V1"
    kw = (synth.cnn_reference_kwargs if "conv_type" in cfg else synth.reference_kwargs)(cfg, replay_batch_size=B, **over, **extra)
    if route[0] == "mlp":
        kw.update(dsact_gemm=route[1], dsact_graph=route[2])
    alg = (dsac_v1.DSAC_V1 if v1 else dsac_v2.DSAC_V2)(**kw)
    _, w = outact_oracle.build(cfg, over)
    sd = alg.networks.state_dict()
    for k, v in w.items():
        sd[k] = torch.from_numpy(v)
    alg.networks.load_state_dict(sd)
    alg.networks.cuda()
    return alg, kw


def _feed(cfg, B, it, v1):
    b = {k: torch.from_numpy(v).cuda() for k, v in (synth.make_cnn_batch if "conv_type" in cfg else synth.make_batch)(cfg, B, it).items()}
    n = synth.make_noise(cfg, B, it)
    return b, tuple(torch.from_numpy(n[i]).cuda() for i in ((0, 1, 3, 3) if v1 else (0, 1, 4, 5)))


def _stats(eng, v1):
    s = eng.read_stats()
    v = np.array([s[k] for k in STAT_KEYS])
    return v[V1_COLS] if v1 else v


@pytest.mark.parametrize("name,route", GOLDEN_ROUTES, ids=[f"{g}-{'-'.join(map(str, r))}" for g, r in GOLDEN_ROUTES])
def test_outact_golden_on_every_route(golden_dir, name, route):
    z, cfg, B, steps, over = load(golden_dir, name)
    v1 = over.get("algorithm") == "DSAC_V1"
    alg, _ = _dropin(cfg, B, over, route)
    eng = alg.networks.engine(B)
    assert eng.output_activations == (over["value_output_activation"], over["policy_output_activation"])
    assert type(eng).__name__ == ("Engine" if route[0] == "mlp" else "CnnEngine")
    atol = 1e-5 if route[0] == "mlp" and route[1] == "bf16x3" else 1e-6
    names = [str(n) for n in z["param_names"]]
    for it in range(steps):
        b, n = _feed(cfg, B, it, v1)
        eng.step(b, it, n)
        np.testing.assert_allclose(_stats(eng, v1), z["tb"][it], rtol=RTOL, atol=atol, err_msg=f"{name} {route} tb_info step {it}")
        w = None
        if f"pdigest_{it + 1}" in z:
            w = eng.export_weights()
            for row, k in zip(z[f"pdigest_{it + 1}"], names):
                np.testing.assert_allclose(w[k].double().abs().sum().item(), row[1], rtol=RTOL, err_msg=f"{name} {k} step {it + 1}")
        # every parameter where the golden holds the full state; in bf16x3 the digests only, as the linear goldens' bf16x3 gate
        # (tests/test_gpu_parity.py): Adam's first steps move a weight by about lr * sign(g), and a gradient entry near zero
        # can change sign under the split-bf16 operands
        if f"state_{it + 1}/{names[0]}" in z and atol == 1e-6:
            w = eng.export_weights() if w is None else w
            for k in names:
                ref = z[f"state_{it + 1}/{k}"]
                np.testing.assert_allclose(w[k].numpy().reshape(ref.shape), ref, rtol=RTOL,
                                           atol=max(atol, 1e-6 * np.abs(ref).max()), err_msg=f"{name} {k} after step {it + 1}")


# ---- float64 gradient gates at a ragged multi-tile batch ------------------------------------------------------------
F64_CASES = [("tanh", "tanh"), ("gelu", "gelu"), ("sigmoid", "relu")]


def _f64_inputs(B):
    cfg = synth.CONFIGS["ragged"]
    return cfg, synth.make_weights(cfg), synth.make_batch(cfg, B, 0), synth.make_noise(cfg, B, 0)


def _f64_grads(acts, B, dtype, rows=None):
    cfg, w, b, n = _f64_inputs(B)
    if rows is not None:
        b, n = {k: v[:rows] for k, v in b.items()}, [x[:rows] for x in n]
    orc, _ = outact_oracle.build(cfg, {}, value_output_activation=acts[0], policy_output_activation=acts[1], dtype=dtype)
    orc.compute_gradients(b, n)
    return {k: g.detach().double() for k, g in orc.grad_dict().items()}


@pytest.mark.parametrize("mode", ["bf16x3", "fp32"])
@pytest.mark.parametrize("acts", F64_CASES, ids=["-".join(a) for a in F64_CASES])
def test_ragged_step0_gradients_meet_the_float64_gates(acts, mode):
    """250 rows (three full 64-row tiles and a ragged one): err_k <= max(c ref_k, floor) for every gradient tensor, with
    every gate at least POWER times below what losing the last row tile moves."""
    from dsac_v2_b200.engine import Engine, make_config
    B = 250
    g64, g32 = _f64_grads(acts, B, torch.float64), _f64_grads(acts, B, torch.float32)
    gcut = _f64_grads(acts, B, torch.float64, rows=G.TILE * ((B - 1) // G.TILE))
    c, floor = G.GATES[mode]
    cfg, w, b, n = _f64_inputs(B)
    h = synth.HYPER
    eng = Engine(make_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], max_batch=B, gemm_mode=mode, use_graph=False,
                             act_q=synth.activations(cfg)[0], act_pi=synth.activations(cfg)[1], gamma=h["gamma"], tau=h["tau"],
                             delay_update=h["delay_update"], auto_alpha=h["auto_alpha"], alpha=h["alpha"],
                             lr_q=h["value_learning_rate"], lr_pi=h["policy_learning_rate"], lr_alpha=h["alpha_learning_rate"],
                             min_log_std=h["policy_min_log_std"], max_log_std=h["policy_max_log_std"]),
                 torch.device("cuda", 0), torch.full((cfg["act_dim"],), cfg["act_lim"]), -torch.full((cfg["act_dim"],), cfg["act_lim"]),
                 output_activations=acts)
    eng.load_weights(w)
    eng.compute_grads({k: torch.from_numpy(v).cuda() for k, v in b.items()}, tuple(torch.from_numpy(n[i]).cuda() for i in (0, 1, 4, 5)))
    g = eng.export_weights(grads=True)
    eng.close()
    fails, weak, worst = {}, {}, 0.0
    for k in g64:
        gate = max(c * G.rel(g32[k], g64[k]), floor)
        sig = G.rel(gcut[k], g64[k])
        err = G.rel(g[k], g64[k])
        worst = max(worst, err / gate)
        if not sig >= G.POWER * gate:
            weak[k] = (gate, sig)
        if not err <= gate:
            fails[k] = (err, gate)
    print(f"\nGRADF64 outact {acts} {mode}: max err/gate {worst:.3g}")
    assert not weak, weak
    assert not fails, fails


# ---- bit for bit at <= 16 rows ---------------------------------------------------------------------------------------
ACTS = ("tanh", "gelu")


def _mlp_engine(cfg, B, mode, acts=ACTS, graph=True, cls=None):
    from dsac_v2_b200.engine import Engine, make_config
    h = synth.HYPER
    c = make_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], max_batch=B, gemm_mode=mode, use_graph=graph,
                    gamma=h["gamma"], tau=h["tau"], delay_update=h["delay_update"], auto_alpha=h["auto_alpha"], alpha=h["alpha"],
                    lr_q=h["value_learning_rate"], lr_pi=h["policy_learning_rate"], lr_alpha=h["alpha_learning_rate"],
                    min_log_std=h["policy_min_log_std"], max_log_std=h["policy_max_log_std"])
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    eng = (cls or Engine)(c, torch.device("cuda", 0), lim, -lim, output_activations=acts)
    eng.load_weights(synth.make_weights(cfg))
    eng.seed(SEED)
    return eng


def _same(a, b, what):
    torch.cuda.synchronize()
    for k in ("params", "targets", "adam_m", "adam_v"):
        assert torch.equal(getattr(a, k), getattr(b, k)), (what, k)
    assert torch.equal(a.state[:16], b.state[:16]), (what, "state")
    sa, sb = a.read_stats_async(), b.read_stats_async()
    torch.cuda.synchronize()
    assert torch.equal(sa, sb), (what, "stats")


@pytest.mark.parametrize("mode", ["bf16x3", "fp32"])
def test_replay_steps_equal_single_calls_bit_for_bit(mode):
    cfg, B = synth.CONFIGS["tiny"], 16
    host = ring_rows(cfg, 40)
    a, b = _mlp_engine(cfg, B, mode), _mlp_engine(cfg, B, mode)
    bind_ring(a, host)
    bind_ring(b, host)
    for k in range(5):
        a.replay_step(B, 40, 1 + k)
    b.replay_steps(5, B, 40, 1)
    _same(a, b, "replay_steps(5)")
    a.close(); b.close()


@pytest.mark.parametrize("mode", ["bf16x3", "fp32"])
def test_compute_grads_and_apply_equal_step_bit_for_bit(mode):
    cfg, B = synth.CONFIGS["tiny"], 13
    a, b = _mlp_engine(cfg, B, mode), _mlp_engine(cfg, B, mode)
    for it in range(3):
        bt, n = _feed(cfg, B, it, False)
        a.step(bt, it, n)
        b.compute_grads(bt, n)
        b.apply(it)
        _same(a, b, f"iteration {it}")
    a.close(); b.close()


def test_explicit_linear_setter_equals_no_call_bit_for_bit():
    """An explicit linear `dsact_set_output_activations` leaves every step as it is without the call (MLP engine in both
    arithmetics, head-wise engine)."""
    from dsac_v2_b200.engine import Engine
    from dsac_v2_b200.engine_cnn import CnnEngine, make_heads_config

    def explicit(base):
        class Explicit(base):
            def _bind(self):
                _lib.check(self.lib.dsact_set_output_activations(self.h, 0, 0))
                super()._bind()
        return Explicit

    cfg, B = synth.CONFIGS["tiny"], 16
    for mode in ("bf16x3", "fp32"):
        a = _mlp_engine(cfg, B, mode, acts=("linear", "linear"))
        b = _mlp_engine(cfg, B, mode, acts=("linear", "linear"), cls=explicit(Engine))
        for it in range(3):
            bt, n = _feed(cfg, B, it, False)
            a.step(bt, it, n)
            b.step(bt, it, n)
        _same(a, b, mode)
        a.close(); b.close()
    h = synth.HYPER
    c = make_heads_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], "parameter", max_batch=B, gamma=h["gamma"], tau=h["tau"])
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    e = [cls(c, torch.device("cuda", 0), lim, -lim) for cls in (CnnEngine, explicit(CnnEngine))]
    for x in e:
        x.load_weights(synth.make_weights_std(cfg, "parameter"))
    for it in range(3):
        bt, n = _feed(cfg, B, it, False)
        for x in e:
            x.step(bt, it, n)
    _same(e[0], e[1], "heads parameter")


def test_dp_step_equals_split_api_bit_for_bit():
    """One W = 2 data-parallel step on one device (tests/test_gpu_dp_one_device.py's child, with output activations)."""
    paths = [REPO, os.path.join(REPO, "dsac-v2_b200", "dropin"), os.path.join(REPO, "tests")]
    env = dict(os.environ, CUDA_MODULE_LOADING="EAGER", DSACT_DP_TIMEOUT_MS="5000", PYTHONPATH=os.pathsep.join(paths))
    p = subprocess.run([sys.executable, os.path.abspath(__file__), "dp"], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert p.returncode == 0, f"child exited with {p.returncode}:\n{p.stdout[-4000:]}\n{p.stderr[-6000:]}"
    print(p.stdout[-2000:])


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_setter_refusals():
    from dsac_v2_b200.engine import make_config, make_v1_options
    from dsac_v2_b200.engine_cnn import make_heads_config
    lib = _lib.load()
    cfg = synth.CONFIGS["tiny"]
    creates = [
        lambda h: lib.dsact_create(C.byref(make_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], max_batch=8)), 0, C.byref(h)),
        lambda h: lib.dsact_v1_create(C.byref(make_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], max_batch=8)),
                                      C.byref(make_v1_options()), 0, C.byref(h)),
        lambda h: lib.dsact_cnn_create(C.byref(make_heads_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], "parameter", max_batch=8)),
                                       0, C.byref(h)),
    ]
    for create in creates:
        h = C.c_void_p()
        assert create(h) == 0
        try:
            for bad in ((7, 0), (0, 7), (-1, 3)):
                assert lib.dsact_set_output_activations(h, *bad) == -1, bad   # DSACT_EINVAL
            assert lib.dsact_set_output_activations(h, 3, 2) == 0
            assert lib.dsact_set_output_activations(h, 0, 0) == 0
        finally:
            lib.dsact_destroy(h)
    assert lib.dsact_set_output_activations(None, 0, 0) == -1
    eng = _mlp_engine(cfg, 8, "fp32")
    assert lib.dsact_set_output_activations(eng.h, 0, 0) == -3                         # DSACT_ESTATE after bind
    eng.close()
    with pytest.raises(ValueError):
        _mlp_engine(cfg, 8, "fp32", acts=("tanh", "swish"))


# ---- the data-parallel child ---------------------------------------------------------------------------------------
def _child_dp():
    from dsac_v2_b200.engine import Engine
    import test_gpu_dp_one_device as D
    init = Engine.__init__

    def with_acts(self, *a, **k):   # every engine the child builds (CnnEngine inherits it)
        init(self, *a, **dict(k, output_activations=ACTS))
    Engine.__init__ = with_acts
    for variant in ("bf16x3_eager", "fp32_eager", "parameter"):
        D.child_exact(variant, 2)


if __name__ == "__main__":
    if sys.argv[1:] == ["dp"]:
        _child_dp()
