"""Step-0 gradients of the CUDA engines against a float64 oracle, with gates that are checked for their own power.

For one case (engine, configuration, batch, an optional edit of weights or minibatch that forces a branch of the loss or
sampling arithmetic), the oracle runs three times on the CPU: float64 on the whole batch (the yardstick), float32 on the
whole batch (what the reference's own arithmetic achieves), and float64 without the last 64-row tile.  Per gradient
tensor k of `grad_dict()`:

    err_k    = |g_cuda - g64| / |g64|
    ref_k    = |g32 - g64| / |g64|
    signal_k = |g64(batch without its last row tile) - g64| / |g64|
    gate_k   = max(c * ref_k, floor)          one (c, floor) pair per arithmetic (GATES)

A case passes when err_k <= gate_k for every k, and a gate is only admissible if gate_k <= signal_k / POWER: a gate loose
enough to let a lost tile of rows through fails by itself.  `tests/test_grad_gate_power.py` checks the power rule and
the regimes' engagement on the CPU; `tests/test_gpu_grad_f64.py` runs the engines.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from dsac_v2_b200 import synth

TILE = 64          # rows per tile of the MLP engine's chain / weight-gradient kernels
POWER = 5.0        # every gate must sit at least this factor below the signal of a lost row tile
# (c, floor) per arithmetic: "heads" is the fp32 head-wise engine (CNN, policy std types, DSAC_V1).  bf16x3 is set from
# its error on an H100 at these cases (operands carried to about 2^-17 instead of fp32's 2^-24): largest err_k / gate_k
# 0.91, smallest signal_k / gate_k 5.7 (the log_alpha gradient at halfcheetah B=8192).  layered_q's six tanh critic
# layers carry the split-bf16 rounding through six dgrad GEMMs into the first layer's weight gradient: there err_k reaches
# 1.15 x the floor on an H100, and the float64 oracle with its GEMMs restated as hi*hi + hi*lo + lo*hi of bf16 splits
# reaches 1.19 x.  That case's bf16x3 gates are doubled; its smallest signal_k / gate_k stays above 80.  deep_pi at
# B = 2200 in bf16x3: q1.q.0.weight, the gradient of the first critic layer (109 inputs: 13 observation and 96 action
# columns), comes out at 9.59 x the floor on an H100, and the float64 oracle with every GEMM restated as split-bf16
# products reaches 9.59 x as well (the other tensors stay below 0.52 x).  Only that tensor's gate is widened, 12 x: its
# signal_k / gate_k is 467, while a case-wide factor would leave log_alpha's lost-tile signal (5.4 x its gate) unseen.
# The restated oracle is tests/gradcheck_rounded.py; tests/test_grad_rounded.py recomputes both widenings' numbers.
GATES = {"fp32": (4.0, 2e-6), "heads": (4.0, 2e-6), "bf16x3": (8.0, 1e-5)}
BF16_LIMIT = 5e-2  # the single-pass bf16 mode is not a parity mode: finite gradients within this relative error
TB_RTOL = 1e-4
ORACLE_THREADS = 4   # torch CPU threads of the oracle runs (tests/conftest.py)

# a hidden layer wider than 256: the tensor-core modes run the per-layer GEMM path (tests/test_gpu_parity.py)
WIDE = dict(obs_dim=7, act_dim=3, hidden=(264, 40), act_lim=1.0)
V1_COLS = [0, 2, 6, 8, 9, 10, 11]   # columns of the engine's statistics that carry DSAC_V1's tb_info


@dataclass(frozen=True)
class Case:
    name: str
    engine: str                    # "mlp" (engine.Engine) or "heads" (engine_cnn.CnnEngine, with or without an encoder)
    cfg_name: str
    batch: int
    std_type: str = "mlp_shared"   # policy std type on the head-wise engine
    algo: str = "DSAC_V2"
    act_dist: str = "TanhGaussDistribution"
    regime: Optional[str] = None   # key of REGIMES
    hyper: Tuple[Tuple[str, float], ...] = ()   # overrides of synth.HYPER
    fp32_only: bool = False        # MLP engine: skip the bf16x3 mode (see REGIME_CASES)
    bf16x3_scale: float = 1.0      # widens this case's bf16x3 gates (see SHAPE_CASES)
    bf16x3_keys: Tuple[Tuple[str, float], ...] = ()   # widens the bf16x3 gates of single tensors instead (see SHAPE_CASES)

    @property
    def cnn(self) -> bool:
        return self.cfg_name in synth.CNN_CONFIGS

    @property
    def cfg(self) -> dict:
        return synth.CNN_CONFIGS[self.cfg_name] if self.cnn else (WIDE if self.cfg_name == "wide" else synth.mlp_config(self.cfg_name))

    @property
    def hyperparameters(self) -> dict:
        return dict(synth.HYPER, **dict(self.hyper))

    @property
    def modes(self) -> Tuple[str, ...]:
        if self.engine != "mlp":
            return ("heads",)
        return ("fp32",) if self.fp32_only else ("fp32", "bf16x3")


# ---- the case table -------------------------------------------------------------------------------------------------
# multi-tile batches and the benchmarked shapes (ragged 63..129 sit on tile edges: at 65 and 129 the last tile holds a row)
SHAPE_CASES = [Case(f"ragged_b{b}", "mlp", "ragged", b) for b in (63, 64, 65, 129, 1000)] + [
    Case("humanoid_b4096", "mlp", "humanoid", 4096),
    Case("halfcheetah_b8192", "mlp", "halfcheetah", 8192),
    Case("pendulum_b256", "mlp", "pendulum", 256),
    Case("wide_b200", "mlp", "wide", 200),
] + [Case(f"{name}_b200", "mlp", name, 200, bf16x3_scale=2.0 if name == "layered_q" else 1.0)
      for name in synth.ASYM_CONFIGS] + [   # critics and policy of different shapes
    # B = 2200: a four-pass chain launch has 4 x 35 row tiles, more than one wave of 132 CTAs, so both forward chains and
    # the critic dgrad chain run on the ping-pong kernel, with ELU, SELU and tanh, six-layer critics and policies, the
    # narrow ragged widths, and a last CTA holding one ragged 24-row tile
    Case(f"{name}_b2200", "mlp", name, 2200, bf16x3_keys=(("q1.q.0.weight", 12.0),) if name == "deep_pi" else ())
    for name in ("asym", "deep_pi", "ragged")] + [
    Case("separated_ragged_b1000", "heads", "ragged", 1000, std_type="mlp_separated"),
    Case("parameter_ragged_b1000", "heads", "ragged", 1000, std_type="parameter"),
    Case("gauss_tiny_b1000", "heads", "tiny", 1000, act_dist="GaussDistribution"),
    Case("v1_pendulum_b4096", "heads", "pendulum", 4096, algo="DSAC_V1"),
    Case("cnn_carracing_b256", "heads", "carracing", 256),
    Case("v1_cnn_carracing_b256", "heads", "carracing", 256, algo="DSAC_V1"),
    Case("cnn_carracing_b1024", "heads", "carracing", 1024),
]

# regime -> {probe: minimum engaged fraction measured by the float64 oracle}
REGIMES = {
    "log_std_clamp": {"log_std_above_max": 0.25, "log_std_below_min": 0.25},
    "tanh_saturation": {"abs_u_above_4": 0.05},
    "huber_linear": {"abs_q_minus_y_above_50": 0.20},
    "ratio_clamp": {"ratio_above_10": 0.10, "ratio_below_0.1": 0.10, "std_raw_above_20": 0.10},
    "ties": {"target_q_tie": 1.0},
    "done_half": {"done": 0.5},
}
# log_std clamp and tanh saturation also run on the head-wise engine's separate log_std head.
# Both are as deep as fp32 arithmetic allows a float64 yardstick to go.  The log_std clamp case raises the lower bound
# from -20 to -2.5: at std = e^-20 the rsample's u - mean (= std * eps) cancels completely in fp32, in the reference's
# arithmetic and the kernel's alike, so the yardstick would measure that cancellation, not the clamp's derivative.  In the
# tanh case 1 - tanh(u)^2 loses a digit per unit of |u| in fp32: with mean biases of +-2.6 (|u| > 4 in 6 % of the
# components) the fp32 oracle's policy gradient stays 5x inside what a lost row tile moves; at +-3 the separate-head
# policy no longer does, and at |u| > 5 in 20 % of the components (biases of +-5.3) the fp32 error exceeds that
# signal itself.  So at |u| ~ 4, 1 - tanh(u)^2 ~ 1e-3 stays far above TG_EPS = 1e-6: the case exercises the squashing's
# derivative near saturation, not the regime where TG_EPS in the log-prob and its gradient matters.
# The ratio clamp case runs the MLP engine in fp32 only: with the critics' std output row scaled by ~1400 the bf16x3
# GEMMs' error grows with the fp32 oracle's (up to 270x it, against <= 55x elsewhere) and no single bf16x3 gate both holds
# there and sees a lost tile at halfcheetah B=8192.  The loss kernel whose branches the case forces is the same code in
# both modes.
REGIME_HYPER = {"log_std_clamp": (("policy_min_log_std", -2.5),)}
REGIME_CASES = [Case(f"{r}_ragged_b1000", "mlp", "ragged", 1000, regime=r, hyper=REGIME_HYPER.get(r, ()),
                     fp32_only=r == "ratio_clamp") for r in REGIMES] + [
    Case(f"{r}_separated_ragged_b1000", "heads", "ragged", 1000, std_type="mlp_separated", regime=r, hyper=REGIME_HYPER.get(r, ()))
    for r in ("log_std_clamp", "tanh_saturation")]

CASES = {c.name: c for c in SHAPE_CASES + REGIME_CASES}
# the action component of the log_std clamp case held above the upper bound / below the lower bound in every row
CLAMPED_HIGH, CLAMPED_LOW = 0, 1


# ---- inputs ---------------------------------------------------------------------------------------------------------
def _weights(case: Case) -> dict:
    cfg = case.cfg
    if case.cnn:
        return synth.make_cnn_weights_v1(cfg) if case.algo == "DSAC_V1" else synth.make_cnn_weights(cfg)
    if case.std_type == "mlp_shared":
        return synth.make_weights_v1(cfg) if case.algo == "DSAC_V1" else synth.make_weights(cfg)
    return synth.make_weights_std_v1(cfg, case.std_type) if case.algo == "DSAC_V1" else synth.make_weights_std(cfg, case.std_type)


def _policy_out_bias(case: Case, w: dict, half: str) -> np.ndarray:
    """Views of the policy's output-layer bias entries for the action mean or log_std, in every weight set."""
    L = 2 * len(synth.hidden_sizes(case.cfg)[1])
    A = case.cfg["act_dim"]
    if case.std_type == "mlp_shared":
        return [w[f"{net}.policy.{L}.bias"][(slice(0, A) if half == "mean" else slice(A, 2 * A))] for net in ("policy", "policy_target")]
    return [w[f"{net}.{half}.{L}.bias"] for net in ("policy", "policy_target")]


def log_std_bias(case: Case) -> Tuple[str, int]:
    """(gradient key, offset of component 0) of the policy's output-layer log_std bias."""
    L = 2 * len(synth.hidden_sizes(case.cfg)[1])
    if case.std_type == "mlp_shared":
        return f"policy.policy.{L}.bias", case.cfg["act_dim"]
    return f"policy.log_std.{L}.bias", 0


def inputs(case: Case):
    """(weights, minibatch, noise) of the case, with its regime edit applied: all numpy float32, edited identically for the
    engine and the oracle (online and target networks alike)."""
    cfg, B = case.cfg, case.batch
    w = {k: v.copy() for k, v in _weights(case).items()}
    b = (synth.make_cnn_batch if case.cnn else synth.make_batch)(cfg, B, 0)
    n = synth.make_noise(cfg, B, 0)
    r = case.regime
    L = 2 * len(synth.hidden_sizes(cfg)[0]) if not case.cnn else None   # the critics' output layer
    if r == "log_std_clamp":        # one component above max_log_std in every row, one below min_log_std, one across max
        for v in _policy_out_bias(case, w, "log_std"):
            v[CLAMPED_HIGH] += 30.0
            v[CLAMPED_LOW] -= 40.0
            v[2] += 0.45
    elif r == "tanh_saturation":    # two of the three action means pushed towards +-1 after the squashing
        for v in _policy_out_bias(case, w, "mean"):
            v[0] += 2.6
            v[1] -= 2.6
    elif r == "huber_linear":
        b["rew"] *= 200.0
    elif r == "ratio_clamp":        # the raw std output of both critics spread as N(-10, 30^2) over the batch
        for net in ("q1", "q2"):
            f = _std_output_features(case, w, net, b)
            scale = 30.0 / float(f.std())
            bias = -10.0 - scale * float(f.mean())
            for k in (net, net + "_target"):
                w[f"{k}.q.{L}.weight"][1] *= scale
                w[f"{k}.q.{L}.bias"][1] = bias
    elif r == "ties":               # q2 = q1, online and target: the target's choice of critic ties in every row
        # (checks that choice, which picks z4's sample over z3's, and that neither critic is counted twice; the 0.5 split of
        # min(q1p, q2p) stays unseen: with identical critics the policy gradient only sees the sum of the two shares)
        for k in [k for k in w if k.startswith("q1")]:
            w["q2" + k[2:]] = w[k].copy()
    elif r == "done_half":
        b["done"][::2] = 1.0
    return w, b, n


def _std_output_features(case: Case, w: dict, net: str, b: dict) -> torch.Tensor:
    """W[1] . h of a critic's std output over the batch (its raw std without the bias), in float64."""
    from oracle.dsact_oracle import _ACT, mlp_forward
    L = len(synth.hidden_sizes(case.cfg)[0])
    layers = [torch.as_tensor(w[f"{net}.q.{2 * j}.{leaf}"], dtype=torch.float64) for j in range(L) for leaf in ("weight", "bias")]
    x = torch.cat([torch.as_tensor(b["obs"], dtype=torch.float64), torch.as_tensor(b["act"], dtype=torch.float64)], -1)
    h = _ACT["gelu"](mlp_forward(layers, x, "gelu"))
    return h @ torch.as_tensor(w[f"{net}.q.{2 * L}.weight"][1], dtype=torch.float64)


def noise_for_engine(case: Case, n):
    """The four noise arrays the engine consumes, in the order of its `dsact_noise`."""
    return tuple(n[i] for i in ((0, 1, 3, 3) if case.algo == "DSAC_V1" else (0, 1, 4, 5)))


# ---- oracle ---------------------------------------------------------------------------------------------------------
def make_oracle(case: Case, w: dict, dtype):
    from oracle.dsact_oracle import cnn_from_config, from_config, std_from_config, v1_from_config
    from oracle.dsact_oracle_v1_heads import v1_cnn_from_config, v1_std_from_config
    cfg, hyper = case.cfg, dict(case.hyperparameters, dtype=dtype, policy_act_distribution=case.act_dist)
    if case.cnn:
        return (v1_cnn_from_config if case.algo == "DSAC_V1" else cnn_from_config)(cfg, w, **hyper)
    if case.std_type == "mlp_shared":
        return (v1_from_config if case.algo == "DSAC_V1" else from_config)(cfg, w, **hyper)
    return (v1_std_from_config if case.algo == "DSAC_V1" else std_from_config)(cfg, w, case.std_type, **hyper)


def _oracle_grads(case, w, b, n, dtype, rows=None):
    orc = make_oracle(case, w, dtype)
    if rows is not None:
        b, n = {k: v[:rows] for k, v in b.items()}, [x[:rows] for x in n]
    tb = orc.compute_gradients(b, n)
    return {k: g.detach().double() for k, g in orc.grad_dict().items()}, tb


def rel(a: torch.Tensor, b: torch.Tensor) -> float:
    """|a - b| / |b| (L2 over the whole tensor), in float64."""
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    den = float(b.norm())
    num = float((a.reshape(b.shape) - b).norm())
    if den == 0.0:
        return 0.0 if num == 0.0 else float("inf")
    return num / den


@dataclass
class Reference:
    g64: Dict[str, torch.Tensor]
    tb64: Dict[str, float]
    tb32: Dict[str, float]
    ref: Dict[str, float]       # fp32 oracle vs float64
    signal: Dict[str, float]    # float64 without the last row tile vs float64


@functools.lru_cache(maxsize=None)
def reference(name: str) -> Reference:
    case = CASES[name]
    w, b, n = inputs(case)
    # the fp32 oracle's rounding sets the gates: it runs on the thread count tests/conftest.py pins, on every host
    assert torch.get_num_threads() == ORACLE_THREADS, torch.get_num_threads()
    g64, tb64 = _oracle_grads(case, w, b, n, torch.float64)
    g32, tb32 = _oracle_grads(case, w, b, n, torch.float32)
    cut = TILE * ((case.batch - 1) // TILE)
    gcut = _oracle_grads(case, w, b, n, torch.float64, rows=cut)[0] if cut > 0 else None
    ref = {k: rel(g32[k], g64[k]) for k in g64}
    # with one tile the batch without it is empty: no gradient at all
    signal = {k: (rel(gcut[k], g64[k]) if gcut is not None else 1.0) for k in g64}
    return Reference(g64, tb64, tb32, ref, signal)


def gates(name: str, mode: str) -> Dict[str, float]:
    c, floor = GATES[mode]
    case = CASES[name]
    keys = dict(case.bf16x3_keys)
    scale = lambda k: keys.get(k, case.bf16x3_scale) if mode == "bf16x3" else 1.0
    return {k: scale(k) * max(c * r, floor) for k, r in reference(name).ref.items()}


def power_violations(name: str, mode: str) -> Dict[str, Tuple[float, float]]:
    """{k: (gate_k, signal_k)} for every tensor whose gate could not notice the loss of the last row tile."""
    r = reference(name)
    return {k: (g, r.signal[k]) for k, g in gates(name, mode).items() if not g <= r.signal[k] / POWER}


# ---- regime probes (float64 oracle) ---------------------------------------------------------------------------------
def engagement(name: str) -> Dict[str, float]:
    """Fraction of rows (or row x action components) in which each branch of the case's regime engages, measured on the
    float64 oracle's own forward pieces at step 0."""
    case = CASES[name]
    assert case.algo == "DSAC_V2" and not case.cnn
    w, b, n = inputs(case)
    orc = make_oracle(case, w, torch.float64)
    t = lambda x: torch.as_tensor(x, dtype=torch.float64)
    obs, act, rew, obs2, done = (t(b[k]) for k in ("obs", "act", "rew", "obs2", "done"))
    eps1, eps2 = t(n[0]), t(n[1])
    P, T = orc.p, orc.t
    with torch.no_grad():
        mean, std = orc.policy_logits(P["policy"], obs)
        ls = std.log()
        u = mean + std * eps1
        mean2, std2 = orc.policy_logits(T["policy"], obs2)
        act2, logp2 = orc.tanh_gauss_rsample(mean2, std2, eps2)
        q1n, _ = orc.q_dist(T["q1"], obs2, act2)
        q2n, _ = orc.q_dist(T["q2"], obs2, act2)
        y = rew + (1 - done) * orc.gamma * (torch.min(q1n, q2n) - orc.alpha() * logp2)
        q1, s1 = orc.q_dist(P["q1"], obs, act)
        ratio = s1.mean() ** 2 / (s1 ** 2 + 0.1)     # at step 0 mean_std is the batch mean of the critic std
    frac = lambda m: float(m.double().mean())
    return {
        "log_std_above_max": frac(ls >= orc.max_log_std - 1e-9),
        "log_std_below_min": frac(ls <= orc.min_log_std + 1e-9),
        "abs_u_above_4": frac(u.abs() > 4),
        "abs_q_minus_y_above_50": frac((q1 - y).abs() > 50),
        "ratio_above_10": frac(ratio > 10),
        "ratio_below_0.1": frac(ratio < 0.1),
        "std_raw_above_20": frac(s1 > 20),          # softplus(raw) = raw above 20 (torch's threshold)
        "target_q_tie": frac(q1n == q2n),
        "done": frac(done > 0),
    }


# ---- the CUDA side --------------------------------------------------------------------------------------------------
def make_engine(case: Case, mode: str, use_graph: bool = False):
    """The case's engine on cuda:0; `use_graph`: the MLP engine captures its steps in CUDA graphs."""
    cfg, B, h = case.cfg, case.batch, case.hyperparameters
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    common = dict(max_batch=B, gamma=h["gamma"], tau=h["tau"], delay_update=h["delay_update"], auto_alpha=h["auto_alpha"],
                  alpha=h["alpha"], lr_q=h["value_learning_rate"], lr_pi=h["policy_learning_rate"],
                  lr_alpha=h["alpha_learning_rate"], min_log_std=h["policy_min_log_std"], max_log_std=h["policy_max_log_std"],
                  act_dist=case.act_dist)
    if case.engine == "mlp":
        from dsac_v2_b200.engine import Engine, make_config
        if case.std_type != "mlp_shared" or case.algo != "DSAC_V2":
            # this builder makes DSAC-T mlp_shared handles only; tests/gradmatrix.py builds the others through the drop-in's route
            raise ValueError(f"{case.name}: the MLP-engine case builder takes DSAC_V2 with std_type 'mlp_shared' only, "
                             f"not {case.algo} / {case.std_type!r}")
        act_q, act_pi = synth.activations(cfg)
        c = make_config(cfg["obs_dim"], cfg["act_dim"], *synth.hidden_sizes(cfg), act_q=act_q, act_pi=act_pi, gemm_mode=mode,
                        use_graph=use_graph, **common)
        return Engine(c, torch.device("cuda", 0), lim, -lim)
    from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config, make_heads_config
    if case.cnn:
        t = synth.CONV_TYPES[cfg["conv_type"]]
        c = make_cnn_config(cfg["obs_dim"], cfg["act_dim"], t["kernels"], t["channels"], t["strides"], t["heads"], algo=case.algo, **common)
    else:
        c = make_heads_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], case.std_type, algo=case.algo, **common)
    return CnnEngine(c, torch.device("cuda", 0), lim, -lim)


def engine_grads(name, mode: str):
    """(gradients in the schema of the oracle's grad_dict, tb_info) of one step-0 gradient computation on cuda:0 for the
    case named `name` (or the Case itself).  DSAC-T runs the gradient-message seam (`compute_grads`); DSAC_V1 has none, so
    it runs one whole step, which leaves the step's gradients in the gradient buffer and the statistics of its forward
    pass."""
    case = name if isinstance(name, Case) else CASES[name]
    w, b, n = inputs(case)
    return step0_grads(make_engine(case, "fp32" if mode == "heads" else mode), case.algo, w, b, noise_for_engine(case, n))


def step0_grads(eng, algo: str, w: dict, b: dict, noise):
    """(gradients, tb_info) of `eng` (closed on return) loaded with `w`, for the minibatch `b` and the engine's four noise
    arrays: engine_grads on an engine built elsewhere."""
    from dsac_v2_b200.engine import STAT_KEYS
    try:
        eng.load_weights(w)
        bt = {k: torch.from_numpy(v).cuda() for k, v in b.items()}
        nz = tuple(torch.from_numpy(x).cuda() for x in noise)
        if algo == "DSAC_V1":
            eng.step(bt, 0, nz)
        else:
            eng.compute_grads(bt, nz)
        g = eng.export_weights(grads=True)
        s = eng.read_stats(len(b["rew"]))
    finally:
        eng.close()
    if algo == "DSAC_V1":
        from oracle.dsact_oracle import V1_TB_KEYS
        vals = [s[k] for k in STAT_KEYS]
        tb = {k: vals[c] for k, c in zip(V1_TB_KEYS, V1_COLS)}
    else:
        tb = {k: s[k] for k in STAT_KEYS[:14]}
    return g, tb


def tb_deviations(r: Reference, tb: Dict[str, float], mode: str):
    """The engine's tb_info entries [(key, got, want, tol)] farther from float64 than the fp32 oracle, up to the factor of
    the mode's gate; never tighter than TB_RTOL."""
    c = GATES[mode][0]
    bad = []
    for k, want in r.tb64.items():
        tol = max(TB_RTOL * max(1.0, abs(want)), c * abs(r.tb32[k] - want))
        if not abs(tb[k] - want) <= tol:
            bad.append((k, tb[k], want, tol))
    return bad


def compare(name: str, mode: str):
    """{k: (err_k, gate_k, ref_k, signal_k)}, the engine's gradients, and the tb_info deviations [(key, got, want, tol)]
    that exceed the tolerance."""
    r = reference(name)
    g, tb = engine_grads(name, mode)
    gate = gates(name, mode)
    out = {k: (rel(g[k], r.g64[k]), gate[k], r.ref[k], r.signal[k]) for k in r.g64}
    return out, g, tb_deviations(r, tb, mode)
