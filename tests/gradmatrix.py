"""Step-0 gradients against float64 across the feature matrix: algorithm, engine route, policy std type, action
distribution, value / policy output activations, network shape and batch class, crossed in one case table.

Each axis reached the engines on its own and has its own float64 gate (tests/gradcheck64.py and the tests built on it).
What this table checks is the plumbing between them: every pair of axis values that some configuration allows meets in
at least one case, and every value of every other axis meets the bf16x3 MLP engine at a batch past one wave of row tiles,
where the layer chains run on the ping-pong kernel.

- A case is valid exactly when the drop-in's `dsact_route.route` accepts its kwargs and lands on the engine the case names;
  the engine is built through that route (`Route.new_engine`), so there is no second list of constraints.
- The oracle is `outact_oracle.build` (every class with output activations) on the same weights; minibatch and noise as
  gradcheck64.  DSAC-T runs the gradient seam (`compute_grads`), DSAC_V1 one whole step, as gradcheck64 does.
- Gates and power rule are gradcheck64's (`GATES`, `POWER`, the tb_info rule): MLP fp32 -> "fp32", MLP bf16x3 ->
  "bf16x3", head-wise and CNN -> "heads".  A bf16x3 gate is widened only for a tensor that the oracle with
  gradcheck_rounded's split-bf16 GEMMs moves as far (WIDENED: one tensor of one case); on the CNN route ref_k also
  covers the encoders' ReLU units at their kink (KINK_EPS).
- FAULTS: float64 oracles that each emulate a subtle wiring bug of one combination; tests/test_grad_matrix_table.py checks
  that every case where a fault's feature is active sees it through its gates.

CASES is the committed table, written out from `cover()` (a deterministic greedy covering; `python tests/gradmatrix.py`
prints it again).  tests/test_grad_matrix_table.py recomputes the coverage requirement from `route()` over the full
product; tests/test_gpu_grad_matrix.py runs the engines.
"""
from __future__ import annotations

import functools
import itertools
import os
import sys
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import numpy as np
import torch

import gradcheck64 as G
import outact_oracle as OA
from dsac_v2_b200 import synth
from oracle import dsact_oracle as O

# ---- the axes ---------------------------------------------------------------------------------------------------------
AXES = {
    "algo": ("DSAC_V2", "DSAC_V1"),
    "route": ("mlp_fp32", "mlp_bf16x3", "heads", "cnn"),
    "std": ("mlp_shared", "mlp_separated", "parameter"),
    "dist": ("TanhGaussDistribution", "GaussDistribution"),
    "out_q": ("linear", "tanh", "sigmoid", "gelu"),
    "out_pi": ("linear", "tanh", "relu", "elu"),
    # ragged: fused layer chains; asym: critics and policy of different shapes; wide: a 264-wide layer, per-layer GEMM
    # groups; small_t1: the reference's type_1 encoder on a 2 x 44 x 44 image, the only shape of the "cnn" route (synth's
    # "odd" encoder is no reference conv_type, so the drop-in's route refuses it)
    "shape": ("ragged", "asym", "wide", "small_t1"),
    # one: 1000 rows, 16 row tiles (multi-tile within one wave); past: more 64-row tiles per chain launch than an H100 has
    # SMs, for every pass count of the algorithm's chains (DSAC_V1's chains have fewer passes, so it needs more rows)
    "wave": ("one", "past"),
}
ONE_WAVE = 1000
PAST_WAVE = {"DSAC_V2": 2200, "DSAC_V1": 4300}
ENGINE = {"mlp_fp32": "mlp", "mlp_bf16x3": "mlp", "heads": "heads", "cnn": "cnn"}   # the engine each route names
MODE = {"mlp_fp32": "fp32", "mlp_bf16x3": "bf16x3", "heads": "heads", "cnn": "heads"}   # its gate (gradcheck64.GATES)
SHORT = {"DSAC_V2": "v2", "DSAC_V1": "v1", "mlp_fp32": "fp32", "mlp_bf16x3": "bf16x3", "mlp_shared": "shared",
         "mlp_separated": "separated", "TanhGaussDistribution": "tg", "GaussDistribution": "gauss"}


@dataclass(frozen=True)
class Case:
    algo: str
    route: str
    std: str
    dist: str
    out_q: str
    out_pi: str
    shape: str
    wave: str

    @property
    def name(self) -> str:
        parts = [SHORT.get(v, v) for v in (self.algo, self.route, self.std, self.dist, self.out_q, self.out_pi, self.shape)]
        return "_".join(parts) + f"_b{self.batch}"

    @property
    def batch(self) -> int:
        return ONE_WAVE if self.wave == "one" else PAST_WAVE[self.algo]

    @property
    def cnn(self) -> bool:
        return self.shape == "small_t1"

    @property
    def cfg(self) -> dict:
        if self.cnn:
            return synth.CNN_CONFIGS["small_t1"]
        return G.WIDE if self.shape == "wide" else synth.mlp_config(self.shape)

    @property
    def mode(self) -> str:
        return MODE[self.route]

    @property
    def over(self) -> dict:
        """The reference's kwargs that set the case's algorithm, std type, distribution and output activations."""
        return dict(algorithm=self.algo, policy_std_type=self.std, policy_act_distribution=self.dist,
                    value_output_activation=self.out_q, policy_output_activation=self.out_pi)

    def kwargs(self) -> dict:
        """The drop-in's kwargs: the reference's, the route's `dsact_gemm` on the MLP engine, no graphs, max_batch = B."""
        extra = dict(dsact_graph=False, dsact_max_batch=self.batch)
        if ENGINE[self.route] == "mlp":
            extra["dsact_gemm"] = self.route[len("mlp_"):]
        make = synth.cnn_reference_kwargs if self.cnn else synth.reference_kwargs
        return make(self.cfg, **self.over, **extra)


def _route_fn():
    if "dsact_route" not in sys.modules:   # the drop-in's modules import each other by their bare names
        d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dsac-v2_b200", "dropin")
        if d not in sys.path:
            sys.path.insert(0, d)
    from dsact_route import route
    return route


def routed(case: Case):
    """The drop-in's Route of the case, or None when `route()` refuses its kwargs or lands on another engine (or, on the
    MLP engine, another arithmetic)."""
    try:
        r = _route_fn()(case.algo, case.kwargs())
    except (NotImplementedError, ValueError):
        return None
    if r.engine != ENGINE[case.route]:
        return None
    if r.engine == "mlp" and r.cfg_args["gemm_mode"] != case.route[len("mlp_"):]:
        return None
    return r


def product():
    return [Case(*v) for v in itertools.product(*AXES.values())]


# ---- coverage ---------------------------------------------------------------------------------------------------------
def items(case: Case):
    """What one case covers: every pair of its axis values, and with (mlp_bf16x3, past) its shape and, when that shape
    runs layer chains (all but "wide"), the value of every other axis: the values that reach the ping-pong kernel."""
    vals = list(zip(AXES, (getattr(case, a) for a in AXES)))
    out = {("pair",) + p + q for p, q in itertools.combinations(vals, 2)}
    if case.route == "mlp_bf16x3" and case.wave == "past":
        out |= {("pingpong",) + v for v in vals if v[0] == "shape" or (v[0] not in ("route", "wave") and case.shape != "wide")}
    return out


def required(valid):
    """Every item some valid full assignment covers."""
    return set().union(*(items(c) for c in valid))


def cover(valid, admissible=lambda c: True):
    """A deterministic greedy covering of `required(valid)`: the valid assignment (in product order) that covers the most
    uncovered items, until none is left.  A pick that fails `admissible` (the generator passes the power rule) is
    dropped from the candidates instead."""
    need, table, cand = required(valid), [], list(valid)
    while need:
        best = max(cand, key=lambda c: len(items(c) & need))   # max keeps the first of equals
        cand.remove(best)
        if admissible(best):
            table.append(best)
            need -= items(best)
    return table


# ---- the table (written out from cover(); see the module docstring) ----------------------------------------------------
def _c(algo, route, std, dist, out_q, out_pi, shape, wave):
    return Case(algo, route, std, dist, out_q, out_pi, shape, wave)


TABLE = [
    _c('DSAC_V2', 'mlp_bf16x3', 'mlp_shared', 'TanhGaussDistribution', 'linear', 'linear', 'ragged', 'past'),
    _c('DSAC_V2', 'mlp_bf16x3', 'mlp_separated', 'GaussDistribution', 'tanh', 'tanh', 'asym', 'past'),
    _c('DSAC_V1', 'mlp_fp32', 'mlp_shared', 'GaussDistribution', 'sigmoid', 'relu', 'wide', 'one'),
    _c('DSAC_V2', 'cnn', 'parameter', 'TanhGaussDistribution', 'gelu', 'elu', 'small_t1', 'one'),
    _c('DSAC_V1', 'heads', 'mlp_separated', 'TanhGaussDistribution', 'linear', 'tanh', 'ragged', 'one'),
    _c('DSAC_V2', 'mlp_bf16x3', 'parameter', 'TanhGaussDistribution', 'sigmoid', 'relu', 'asym', 'past'),
    _c('DSAC_V1', 'mlp_bf16x3', 'mlp_shared', 'GaussDistribution', 'gelu', 'elu', 'asym', 'past'),
    _c('DSAC_V1', 'heads', 'parameter', 'GaussDistribution', 'tanh', 'linear', 'wide', 'one'),
    _c('DSAC_V1', 'cnn', 'mlp_separated', 'GaussDistribution', 'linear', 'relu', 'small_t1', 'past'),
    _c('DSAC_V2', 'mlp_fp32', 'mlp_separated', 'TanhGaussDistribution', 'linear', 'elu', 'wide', 'past'),
    _c('DSAC_V2', 'heads', 'mlp_separated', 'GaussDistribution', 'gelu', 'relu', 'ragged', 'past'),
    _c('DSAC_V2', 'cnn', 'mlp_shared', 'TanhGaussDistribution', 'tanh', 'tanh', 'small_t1', 'one'),
    _c('DSAC_V2', 'mlp_fp32', 'mlp_separated', 'TanhGaussDistribution', 'sigmoid', 'linear', 'asym', 'one'),
    _c('DSAC_V2', 'mlp_fp32', 'parameter', 'TanhGaussDistribution', 'tanh', 'tanh', 'ragged', 'one'),
    _c('DSAC_V1', 'heads', 'mlp_shared', 'TanhGaussDistribution', 'sigmoid', 'elu', 'ragged', 'one'),
    _c('DSAC_V2', 'mlp_bf16x3', 'mlp_shared', 'TanhGaussDistribution', 'gelu', 'tanh', 'wide', 'one'),
    _c('DSAC_V2', 'cnn', 'mlp_shared', 'TanhGaussDistribution', 'sigmoid', 'linear', 'small_t1', 'one'),
    _c('DSAC_V2', 'mlp_fp32', 'mlp_shared', 'TanhGaussDistribution', 'gelu', 'linear', 'ragged', 'one'),
    _c('DSAC_V2', 'mlp_fp32', 'parameter', 'TanhGaussDistribution', 'linear', 'linear', 'asym', 'one'),
    _c('DSAC_V2', 'mlp_bf16x3', 'mlp_shared', 'TanhGaussDistribution', 'tanh', 'relu', 'wide', 'past'),
    _c('DSAC_V2', 'mlp_fp32', 'mlp_shared', 'TanhGaussDistribution', 'tanh', 'elu', 'ragged', 'one'),
    _c('DSAC_V2', 'mlp_fp32', 'mlp_shared', 'TanhGaussDistribution', 'sigmoid', 'tanh', 'ragged', 'one'),
]
CASES = {c.name: c for c in TABLE}

# case -> {gradient key: factor} of bf16x3 gates widened after the oracle with gradcheck_rounded's split-bf16 GEMMs
# (`Rounded("bf16x3")` as its dense layer) reached the same excess.  DSAC_V1 asym at B = 4300 with Gauss and gelu / elu
# outputs: policy.policy.0.weight, the policy's first layer (64 observation columns), came out at 1.08 x its gate on an
# H100 and the restatement reaches 1.04 x (every other tensor of the bf16x3 cases stays below 0.94 x there).  Only that
# tensor is widened, 1.5 x: its signal_k / gate_k stays above 3000.  case -> {key: (factor, the restatement's move in
# unwidened gates)}; tests/test_grad_matrix_table.py recomputes the move (`widening`).
WIDENED: Dict[str, Dict[str, Tuple[float, float]]] = {
    "v1_bf16x3_shared_gauss_gelu_elu_asym_b4300": {"policy.policy.0.weight": (1.5, 1.04)}}


def _case(c) -> Case:
    return c if isinstance(c, Case) else CASES[c]


# ---- oracle -----------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _inputs(c: Case):
    _, w = OA.build(c.cfg, c.over)
    b = (synth.make_cnn_batch if c.cnn else synth.make_batch)(c.cfg, c.batch, 0)
    return (_centred_heads(c, w, b) if c.cnn else w), b, synth.make_noise(c.cfg, c.batch, 0)


def inputs(c):
    """(weights, minibatch, noise) of a case (Case or name): the oracle builder's weights, gradcheck64's minibatch and
    noise streams.  The CNN heads' output biases are centred on the batch (`_centred_heads`)."""
    return _inputs(_case(c))


def _centred_heads(c: Case, w: dict, b: dict) -> dict:
    """`w` with the CNN head outputs moved to set batch means, online and target networks alike: the policy's mean and
    log_std components alternately to 0 (rows on both sides of relu's and elu's kink) and to -0.75 (where act' of tanh,
    relu and elu is far from 1), each critic's mean and std output to -0.5.  With synth's weights on U(0, 1) images
    every head output lies in a narrow positive band near 0: relu and elu would run their linear branch only and tanh'
    would be 1 to four digits, so a missing or misplaced act' would stay unseen."""
    orc, _ = OA.build(c.cfg, c.over, weights=w, dtype=torch.float64)
    t = lambda x: torch.as_tensor(x, dtype=torch.float64)
    L = 2 * len(synth.CONV_TYPES[c.cfg["conv_type"]]["heads"])
    A = c.cfg["act_dim"]
    want = {"policy": torch.where(torch.arange(A) % 2 == 0, 0.0, -0.75).double()}
    out = {k: v.copy() for k, v in w.items()}
    with torch.no_grad():
        for net in type(orc).NETS:
            pre = (_policy_pre(orc, orc.p[net], t(b["obs"])) if net == "policy"
                   else _q_pre(orc, orc.p[net], t(b["obs"]), t(b["act"])))
            for head, x in zip(("mean", "log_std"), pre):
                d = (want.get(net, torch.tensor(-0.5, dtype=torch.float64)) - x.mean(0)).numpy()
                for k in (net, net + "_target"):
                    out[f"{k}.{head}.{L}.bias"] += d.astype(np.float32)
    return out


def noise_for_engine(case: Case, n):
    return tuple(n[i] for i in ((0, 1, 3, 3) if case.algo == "DSAC_V1" else (0, 1, 4, 5)))


def make_oracle(c, dtype, fault: Optional[str] = None, linear=None, kink_seed=False):
    """The case's oracle in `dtype`; `fault`: a key of FAULTS, emulated; `linear`: the dense layer (gradcheck_rounded's
    `Rounded` restates the tensor-core GEMMs); `kink_seed` (CNN only): None or a seed of KINK_SEEDS, the encoders'
    near-kink ReLU units taken to the other side of the kink in the backward (`_FlippedKinks`)."""
    c = _case(c)
    orc, _ = OA.build(c.cfg, c.over, weights=inputs(c)[0], dtype=dtype)
    if fault is not None:
        orc.__class__ = type(f"{fault}_{type(orc).__name__}", (FAULTS[fault][0], type(orc)), {})
    if kink_seed is not False:
        orc.__class__ = type(f"kinks_{type(orc).__name__}", (_FlippedKinks, type(orc)), {})
        orc.kink_seed = kink_seed
    if linear is not None:
        orc.linear = linear
    return orc


def oracle_grads(c, dtype, rows: Optional[int] = None, fault: Optional[str] = None, linear=None, kink_seed=False):
    _, b, n = inputs(c)
    if rows is not None:
        b, n = {k: v[:rows] for k, v in b.items()}, [x[:rows] for x in n]
    orc = make_oracle(c, dtype, fault, linear, kink_seed)
    tb = orc.compute_gradients(b, n)
    return {k: g.detach().double() for k, g in orc.grad_dict().items()}, tb


@functools.lru_cache(maxsize=None)
def _reference(c: Case) -> G.Reference:
    assert torch.get_num_threads() == G.ORACLE_THREADS, torch.get_num_threads()
    g64, tb64 = oracle_grads(c, torch.float64)
    g32, tb32 = oracle_grads(c, torch.float32)
    gcut = oracle_grads(c, torch.float64, rows=G.TILE * ((c.batch - 1) // G.TILE))[0]
    ref = {k: G.rel(g32[k], g64[k]) for k in g64}
    signal = {k: G.rel(gcut[k], g64[k]) for k in g64}
    if c.cnn:   # an encoder unit at its ReLU kink may land on either side in fp32 (KINK_EPS)
        for seed in KINK_SEEDS:
            gk = oracle_grads(c, torch.float64, kink_seed=seed)[0]
            ref = {k: max(ref[k], G.rel(gk[k], g64[k])) for k in g64}
    return G.Reference(g64, tb64, tb32, ref, signal)


def reference(c) -> G.Reference:
    """gradcheck64.reference of a matrix case: float64 and float32 on the whole batch, float64 without the last row tile;
    on the CNN route ref_k also covers the encoders' near-kink ReLU units (KINK_EPS)."""
    return _reference(_case(c))


def gates(c) -> Dict[str, float]:
    c = _case(c)
    k_c, floor = G.GATES[c.mode]
    wide = WIDENED.get(c.name, {}) if c.mode == "bf16x3" else {}
    return {k: wide.get(k, (1.0,))[0] * max(k_c * r, floor) for k, r in reference(c).ref.items()}


def widening(c) -> Dict[str, float]:
    """{k: |g64R - g64| / |g64| / common_k}: how far the float64 oracle with split-bf16 GEMMs (gradcheck_rounded's
    `Rounded("bf16x3")`) moves each gradient from plain float64, in the case's unwidened bf16x3 gates common_k."""
    from gradcheck_rounded import Rounded
    c = _case(c)
    k_c, floor = G.GATES["bf16x3"]
    r = reference(c)
    g64r = oracle_grads(c, torch.float64, linear=Rounded("bf16x3"))[0]
    return {k: G.rel(g64r[k], r.g64[k]) / max(k_c * r.ref[k], floor) for k in r.g64}


def power_violations(c) -> Dict[str, Tuple[float, float]]:
    """{k: (gate_k, signal_k)} for every tensor whose gate could not notice the loss of the last row tile."""
    r = reference(c)
    return {k: (g, r.signal[k]) for k, g in gates(c).items() if not g <= r.signal[k] / G.POWER}


# ---- ReLU units at their kink (CNN encoders) --------------------------------------------------------------------------
# A conv pre-activation z within fp32 rounding of 0 is on either side of the ReLU kink depending on the summation order:
# the engine's direct convolutions and the fp32 oracle's conv2d each pick one, and a unit that picks the other side than
# float64 passes its whole dz (or none of it) to the layers below.  The type_1 encoders of these cases hold units with |z|
# down to 4e-9 .. 2e-8 of the magnitude sum(|x| |w|) + |b| of their terms (fp32's unit roundoff is 6e-8), and one such
# unit among the 3.2 million of the first layer at B = 1000 moves the gradients of the layers below it by 1e-5 to 1e-4
# (relative).  On an H100 that was what separated the engine from plain float64: the encoders holding the units nearest
# their kink (q2 at B = 1000, the DSAC_V1 policy at B = 4300) had their conv.0 / conv.2 gradients 4 to 30 gates away, the
# others within 0.31.  So on the CNN route ref_k is also the largest move of the float64 oracle's gradients when such
# units (|z| < KINK_EPS x magnitude, two unit roundoffs) take the other side, all of them (seed None) or the pseudo-random
# half a seed picks, as gradcheck_rounded.FLIP_EPS does for bf16 rounding midpoints.  The forward values stay float64's:
# only a unit's backward mask flips (its ReLU output is within its rounding of 0 either way).
KINK_EPS = 2.0 ** -23
KINK_SEEDS = (None, 1, 2, 3)


def _relu_mask(z: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """relu(z) with `mask` as the backward's derivative."""
    through = torch.where(mask, z, torch.zeros_like(z))
    return torch.relu(z).detach() + (through - through.detach())


class _FlippedKinks:
    """The CNN encoders with every near-kink ReLU unit (or the half `kink_seed` picks) on the other side in the backward."""
    kink_seed = None

    def _features(self, w, obs):
        import torch.nn.functional as F
        x, j = obs, 0
        while f"conv.{2 * j}.weight" in w:
            wt, bs, st = w[f"conv.{2 * j}.weight"], w[f"conv.{2 * j}.bias"], self.conv_strides[j]
            z = F.conv2d(x, wt, bs, stride=st)
            with torch.no_grad():
                near = z.abs() < KINK_EPS * F.conv2d(x.abs(), wt.abs(), bs.abs(), stride=st)
                if self.kink_seed is not None:
                    g = torch.Generator().manual_seed(1000 * self.kink_seed + j)
                    near &= torch.rand(z.shape, generator=g, dtype=torch.float64) < 0.5
            x = _relu_mask(z, (z > 0) ^ near)
            j += 1
        return x.reshape(x.shape[0], -1)


# ---- emulated faults --------------------------------------------------------------------------------------------------
def _identity_grad(act):
    """act's value with the identity's derivative: the activation applied, its act' left out of the backward."""
    return lambda z: z + (act(z) - z).detach()


def _policy_pre(o, layers, obs):
    """(mean, log_std) of the policy before its output activation; log_std None for the "parameter" row."""
    if isinstance(o, OA._Cnn):
        w = dict(zip(o.names["policy"], layers))
        f = o._features(w, obs)
        return o._head(w, "mean", f, o.act_pi), o._head(w, "log_std", f, o.act_pi)
    if isinstance(o, OA._Std):
        w = dict(zip(o.names["policy"], layers))

        def head(name):
            n = sum(k.startswith(name + ".") and k.endswith(".weight") for k in w)
            return O.mlp_forward([w[f"{name}.{2 * j}.{leaf}"] for j in range(n) for leaf in ("weight", "bias")], obs,
                                 o.act_pi, o.linear)
        return head("mean"), (head("log_std") if o.std_type == "mlp_separated" else None)
    return torch.chunk(O.mlp_forward(layers, obs, o.act_pi, o.linear), 2, dim=-1)


def _q_pre(o, layers, obs, act):
    """(mean, raw std) of a critic before its output activation."""
    if isinstance(o, OA._Cnn):
        w = dict(zip(o.names["q1"], layers))
        f = torch.cat([o._features(w, obs), act], dim=-1)
        return o._head(w, "mean", f, o.act_q)[..., 0], o._head(w, "log_std", f, o.act_q)[..., 0]
    out = O.mlp_forward(layers, torch.cat([obs, act], dim=-1), o.act_q, o.linear)
    return out[..., 0], out[..., 1]


def _policy(o, layers, obs, act_log_std, act_row):
    mean, log_std = _policy_pre(o, layers, obs)
    if log_std is None:
        log_std = act_row(dict(zip(o.names["policy"], layers))["log_std"]) + torch.zeros_like(mean)
    else:
        log_std = act_log_std(log_std)
    return o.out_pi(mean), torch.clamp(log_std, o.min_log_std, o.max_log_std).exp()


class _GaussSquashed:
    """GaussDistribution: the action squashed by tanh and the limits as TanhGauss does, the log-prob still Gaussian."""

    def tanh_gauss_rsample(self, mean, std, eps):
        a, logp = super().tanh_gauss_rsample(mean, std, eps)
        if not self.gauss_only:
            return a, logp
        return (self.hi - self.lo) / 2 * torch.tanh(a) + (self.hi + self.lo) / 2, logp


class _LogStdNoDeriv:
    """act' of the policy output activation left out on the log_std outputs (the log_std half or network)."""

    def policy_logits(self, layers, obs):
        return _policy(self, layers, obs, _identity_grad(self.out_pi), lambda x: x)


class _RowActivated:
    """The policy output activation applied to the "parameter" std type's learnable log_std row as well."""

    def policy_logits(self, layers, obs):
        return _policy(self, layers, obs, self.out_pi, self.out_pi)


class _QStdNoDeriv:
    """act' of the value output activation left out on the critics' std output."""

    def q_dist(self, layers, obs, act):
        mean, std = _q_pre(self, layers, obs, act)
        return self.out_q(mean), torch.nn.functional.softplus(_identity_grad(self.out_q)(std))


class _QMeanOnly:
    """The value output activation applied to the critic's mean output only."""

    def q_dist(self, layers, obs, act):
        mean, std = _q_pre(self, layers, obs, act)
        return self.out_q(mean), torch.nn.functional.softplus(std)


# fault -> (oracle mixin, the cases where the fault's feature is active)
FAULTS = {
    "gauss_squashed": (_GaussSquashed, lambda c: c.dist == "GaussDistribution"),
    "log_std_no_act_grad": (_LogStdNoDeriv, lambda c: c.out_pi != "linear" and (c.cnn or c.std != "parameter")),
    "q_std_no_act_grad": (_QStdNoDeriv, lambda c: c.out_q != "linear"),
    "parameter_row_activated": (_RowActivated, lambda c: c.out_pi != "linear" and c.std == "parameter" and not c.cnn),
    "v1_q_mean_only": (_QMeanOnly, lambda c: c.out_q != "linear" and c.algo == "DSAC_V1"),
}


def fault_factor(c, fault: str) -> Tuple[float, str]:
    """(max_k |g_fault - g64| / gate_k, its key): how far the emulated fault moves the case's gradients, in gates."""
    r, gt = reference(c), gates(c)
    g = oracle_grads(c, torch.float64, fault=fault)[0]
    m = {k: G.rel(g[k], r.g64[k]) / gt[k] for k in gt}
    k = max(m, key=m.get)
    return m[k], k


# ---- the CUDA side ----------------------------------------------------------------------------------------------------
def make_engine(c):
    """The case's engine on cuda:0, built by the drop-in's route from the case's kwargs."""
    c = _case(c)
    r = routed(c)
    assert r is not None, f"{c.name}: route() does not put this case on the {c.route} engine"
    lim = torch.full((c.cfg["act_dim"],), c.cfg["act_lim"])
    eng = r.new_engine(torch.device("cuda", 0), lim, -lim, c.batch)
    assert eng.output_activations == (c.out_q, c.out_pi)
    return eng


def engine_grads(c):
    """(gradients, tb_info) of one step-0 gradient computation of the case's engine (gradcheck64.step0_grads)."""
    c = _case(c)
    w, b, n = inputs(c)
    return G.step0_grads(make_engine(c), c.algo, w, b, noise_for_engine(c, n))


def compare(c):
    """{k: (err_k, gate_k, ref_k, signal_k)}, the engine's gradients, and the tb_info deviations beyond tolerance."""
    c = _case(c)
    r = reference(c)
    g, tb = engine_grads(c)
    gate = gates(c)
    out = {k: (G.rel(g[k], r.g64[k]), gate[k], r.ref[k], r.signal[k]) for k in r.g64}
    return out, g, G.tb_deviations(r, tb, c.mode)


if __name__ == "__main__":   # print the covering table
    torch.set_num_threads(G.ORACLE_THREADS)
    valid = [c for c in product() if routed(c) is not None]
    for c in cover(valid, lambda c: not power_violations(c)):
        print(f"    _c{tuple(getattr(c, a) for a in AXES)!r},")
