"""Step-0 gradients of the MLP engine's tensor-core modes against a float64 oracle whose every GEMM multiplies the
operands the kernels multiply.

The tensor-core modes multiply bf16 images of every GEMM operand (tests/tc_ref.py: hi = bf16_rn(x), lo = bf16_rn(x - hi);
bf16x3 sums hi*hi + hi*lo + lo*hi, bf16 hi*hi).  The step imaged by the engine (csrc/engine.cu) rounds them all the
same way, whichever lowering runs a GEMM (the layer chains, the per-layer groups of a layer wider than 256, the weight
gradient kernel) and whatever the layer's width (a two-column critic head included):

    forward           y  = planes(x) . planes(W)^T + b      x: obs, obs2, act, the sampled actions, hidden activations
    input gradient    dx = planes(dz) . planes(W)            dz: the loss kernels' dL/d(output) and each dgrad's dL/dz
    weight gradient   dW = planes(dz)^T . planes(x)          the same images of dz and x the other two GEMMs read
    bias gradient     db = sum over rows of dz               fp32 column sums, taken before dz is imaged

`Rounded` is that dense layer, handed to the oracle (`OracleDSACT.linear`) in place of `F.linear`; every other piece
of the oracle's arithmetic is unchanged.  Against this yardstick what separates the engine is its fp32 accumulation and
fp32 elementwise arithmetic (and, in bf16, which way a value near a rounding midpoint images), so gradcheck64's gate
scheme applies, power rule included (GATES; in bf16 refR_k also covers those flips):

    g64R     the float64 restatement on the whole batch          g32R  the float32 restatement (its own fp32
    refR_k   = |g32R - g64R| / |g64R|                                   activations rounded as the kernels round them)
    signal_k = |g64R(batch without its last row tile) - g64R| / |g64R|
    gateR_k  = max(c * refR_k, floor)        one (c, floor) pair for the mode, gateR_k <= signal_k / POWER

`tests/test_grad_rounded.py` checks the restatement against tc_ref's layer reference, the power rule and the gates'
sight of emulated wiring faults on the CPU; `tests/test_gpu_grad_rounded.py` runs the engine.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

import gradcheck64 as G
import std_mlp_common as S
import tc_ref as R
import v1_mlp_common as V
from dsac_v2_b200 import synth

MODES = ("bf16x3", "bf16")
# (c, floor) per mode.  bf16x3: the fp32 pair (4, 2e-6) does not hold on an H100: the engine's fp32 accumulation lands up
# to 4.04 of those gates from g64R (halfcheetah B = 8192, q1.q.4.weight: err 8.1e-6, 21.5 x refR; humanoid B = 4096
# 1.59, DSAC_V1 asym B = 4300 1.85), so bf16x3 keeps gradcheck64's bf16x3 pair, without any per-case or per-tensor factor.
# bf16: its images keep 8 bits, so a computed value (hidden activation, dz, sampled action) that the engine's fp32
# arithmetic and the restatement's put on opposite sides of a bf16 rounding midpoint images one bf16 ulp apart.  On an
# H100 that accounted for every bf16 case beyond (4, 2e-6) of refR alone: at ragged_b63 one dz element 1.1e-7 (relative)
# from its midpoint moved q2.q.0.weight by 77 gates, at wide_b200 two first-layer activations 1.8e-7 and 2.7e-7 from
# theirs moved policy.policy.4.weight by 42; with those elements rounded the other way both cases sit inside 1.03 gates.
# So the bf16 gate takes refR_k from the float32 restatement or from restatements that round such near-midpoint values
# (within FLIP_EPS) the other way, whichever is larger (`reference`).
GATES = {"bf16x3": (8.0, 1e-5), "bf16": (4.0, 2e-6)}
FLIP_EPS = 2.0 ** -20     # relative distance from a bf16 rounding midpoint within which a computed value may image either way
FLIP_SEEDS = (None, 1, 2, 3)   # None: every such value rounded the other way; a seed: a pseudo-random half of them
GATED = tuple(GATES)
POWER = G.POWER
PAIRS = {"bf16x3": ((0, 0), (1, 0), (0, 1)), "bf16": ((0, 0),)}   # (plane of the first operand, plane of the second)

# wiring faults the restatement emulates as if it were the engine (test_grad_rounded.py)
FAULTS = ("trunc_w",        # the weight images split by truncation instead of round-to-nearest
          "trunc_act",      # the activation images (obs, act, sampled actions, hidden layers)
          "trunc_dz",       # the dz images
          "drop_hilo",      # bf16x3 without its hi * lo product
          "one_plane",      # bf16x3 run with the hi planes only
          "fp32_dz_wgrad",  # the weight gradient reads dz in fp32 instead of its image
          "lost_row_tile")  # the batch's last 64-row tile never reaches the gradients


class _RoundedLinear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, arith):
        ctx.save_for_backward(x, w)
        ctx.arith = arith
        y = arith.mm(arith.planes(x, "act"), [p.t() for p in arith.planes(w, "w")])
        return y if b is None else y + b

    @staticmethod
    def backward(ctx, dz):
        x, w = ctx.saved_tensors
        a = ctx.arith
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = a.mm(a.planes(dz, "dz"), a.planes(w, "w"))
        if ctx.needs_input_grad[1]:
            dw = a.mm([p.t() for p in a.planes(dz, "dz_wgrad")], a.planes(x, "act"))
        if ctx.needs_input_grad[2]:
            db = dz.sum(0)
        return dx, dw, db, None


class Rounded:
    """`linear(x, W, b)` with the tensor-core kernels' operand planes in `mode` ("bf16x3" or "bf16"), in the dtype of
    its arguments (the oracle's).  `fault`: one of FAULTS but lost_row_tile (None: the engine as it should be)."""

    def __init__(self, mode: str, fault: Optional[str] = None, flip_eps: float = 0.0, flip_seed: Optional[int] = None):
        """`flip_eps` > 0 (bf16): computed values within that relative distance of a bf16 rounding midpoint image to
        the other neighbour, all of them (`flip_seed` None) or the pseudo-random half `flip_seed` picks."""
        assert mode in MODES and fault in (None,) + FAULTS[:-1], (mode, fault)
        assert flip_eps == 0.0 or mode == "bf16"
        self.mode, self.fault, self.flip_eps, self.flip_seed = mode, fault, flip_eps, flip_seed
        pairs = PAIRS["bf16" if fault == "one_plane" else mode]
        self.pairs = pairs[:2] if (fault == "drop_hilo" and mode == "bf16x3") else pairs

    def planes(self, t: torch.Tensor, role: str):
        """The planes of `t` a GEMM multiplies: tc_ref.operands (role "w", "act", "dz"; "dz_wgrad": dz as the weight
        gradient reads it)."""
        t = t.detach()
        if role == "dz_wgrad":
            if self.fault == "fp32_dz_wgrad":   # unrounded: one fp32 plane (and a zero lo plane in bf16x3)
                return [t, torch.zeros_like(t)] if self.mode == "bf16x3" else [t]
            role = "dz"
        planes = [p.to(t.dtype) for p in R.operands(t, self.mode, trunc=self.fault == "trunc_" + role)]
        if self.flip_eps > 0.0 and role != "w" and t.dtype == torch.float64:
            planes[0] = self._flipped(t, planes[0])
        return planes

    def _flipped(self, t, hi):
        """hi with the near-midpoint computed values of `t` rounded to the other bf16 neighbour.  Weights, obs and act
        are fp32 numbers the engine images exactly as the restatement does: only values that are not (float64 results
        of the restatement's own arithmetic) can flip.  The pick depends on the value alone, so every GEMM that reads
        one image sees the same flips."""
        f = t.float()
        down = R.bf16_rn(f, trunc=True)
        up = down + torch.sign(f.double()) * R.ulp(down)
        mid = (down + up) / 2
        near = (t != f.double()) & (down != 0) & ((f.double() - mid).abs() < self.flip_eps * f.double().abs())
        if self.flip_seed is not None:
            bits = f.view(torch.int32).long()
            near &= ((bits * 2654435761 + self.flip_seed * 40503) >> 11) % 2 == 1
        return torch.where(near, torch.where(hi == down, up, down), hi)

    def mm(self, a, b):
        """sum over the mode's plane pairs of a[i] @ b[j]"""
        return sum(a[i] @ b[j] for i, j in self.pairs)

    def __call__(self, x, w, b=None):
        y = _RoundedLinear.apply(x.reshape(-1, x.shape[-1]), w, b, self)
        return y.reshape(*x.shape[:-1], w.shape[0])


# ---- the case table -------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class RCase:
    name: str
    kind: str                  # "dsact" (gradcheck64's inputs), "std" (std_mlp_common's), "v1" (DSAC_V1, v1_mlp_common)
    case: G.Case               # configuration, batch, std type, algorithm
    prefix: str = ""           # compare only the gradients whose key starts with this


def _std(std_type, batch):
    return RCase(f"{std_type}_ragged_b{batch}", "std", G.Case(f"{std_type}_ragged_b{batch}", "mlp", "ragged", batch,
                                                               std_type=std_type))


# gradcheck64's MLP-engine shapes (ragged tile edges, the benchmarked shapes, the per-layer path, critics and policies of
# different shapes, the ping-pong kernel at B = 2200); the two other policy std types at B = 1000 and 2200 (ping-pong);
# DSAC_V1 at B = 4300 (ping-pong, one critic); and B = 8500, where the policy's single-pass dgrad chain runs on the
# ping-pong kernel: as in test_gpu_pingpong_steps.py only its policy.* gradients are compared (a lost row tile moves some
# critic-bias and log_alpha gradients by less than a floor there)
CASES = {c.name: c for c in
         [RCase(c.name, "dsact", c) for c in G.SHAPE_CASES if c.engine == "mlp"] +
         [_std(s, b) for s in S.STD_TYPES for b in (1000, 2200)] +
         [RCase("v1mlp_asym_b4300", "v1", G.Case("v1mlp_asym_b4300", "mlp", "asym", 4300, algo="DSAC_V1"))] +
         [RCase(f"{n}_b8500", "dsact", G.Case(f"{n}_b8500", "mlp", n, 8500), prefix="policy.")
          for n in ("asym", "deep_pi", "ragged")]}

# (case, mode) -> {key: why}: tensors the power rule cannot hold for, left out of that case's comparison (none so far)
EXCLUDED: Dict[Tuple[str, str], Dict[str, str]] = {}

# The bf16x3 gates of the float64 tests (gradcheck64 (8, 1e-5) against the plain float64 oracle) that are widened:
# case -> (the tensor the widening is for, None: the whole case; the factor; how far the split-bf16 operand rounding
# alone moves the most-moved of those tensors, in unwidened gates).  test_grad_rounded.py recomputes the last number
# (widening()) and checks it stays inside the widened gate.  parameter at B = 2200 stays inside the common gate by the
# rounding alone: the engine's 1.03 there is that 0.94 plus its fp32 arithmetic, which test_gpu_grad_rounded.py bounds.
WIDENED = {"layered_q_b200": (None, 2.0, 1.19),                      # gradcheck64.SHAPE_CASES, bf16x3_scale
           "deep_pi_b2200": ("q1.q.0.weight", 12.0, 9.59),           # gradcheck64.SHAPE_CASES, bf16x3_keys
           "parameter_ragged_b200": (None, 2.0, 1.07),               # test_gpu_std_mlp.F64_BF16X3_SCALE
           "parameter_ragged_b2200": (None, 2.0, 0.94)}
_AUX = {"parameter_ragged_b200": _std("parameter", 200)}      # cases only the widening checks use


def case(name: str) -> RCase:
    return CASES[name] if name in CASES else _AUX[name]


@functools.lru_cache(maxsize=None)
def inputs(name: str):
    rc = case(name)
    if rc.kind == "std":
        cfg, B = rc.case.cfg, rc.case.batch
        return S.std_weights(cfg, rc.case.std_type), synth.make_batch(cfg, B, 0), synth.make_noise(cfg, B, 0)
    return G.inputs(rc.case)


def make_oracle(name: str, dtype, linear=F.linear):
    rc = case(name)
    c = rc.case
    w = inputs(name)[0]
    if rc.kind == "std":
        orc = S.make_oracle(c.cfg, c.std_type, weights=w, dtype=dtype)
    elif rc.kind == "v1":
        orc = V.v1_oracle(c.cfg, w, **dict(c.hyperparameters, dtype=dtype, policy_act_distribution=c.act_dist))
    else:
        orc = G.make_oracle(c, w, dtype)
    orc.linear = linear
    return orc


def oracle_grads(name: str, dtype, linear=F.linear, rows: Optional[int] = None) -> Dict[str, torch.Tensor]:
    _, b, n = inputs(name)
    if rows is not None:
        b, n = {k: v[:rows] for k, v in b.items()}, [x[:rows] for x in n]
    orc = make_oracle(name, dtype, linear)
    orc.compute_gradients(b, n)
    return {k: g.detach().double() for k, g in orc.grad_dict().items()}


def cut_rows(name: str) -> int:
    return G.TILE * ((case(name).case.batch - 1) // G.TILE)


@dataclass
class Reference:
    g64: Dict[str, torch.Tensor]   # g64R
    ref: Dict[str, float]          # refR_k
    signal: Dict[str, float]
    gate: Dict[str, float]         # gateR_k of the compared keys


@functools.lru_cache(maxsize=None)
def reference(name: str, mode: str) -> Reference:
    assert torch.get_num_threads() == G.ORACLE_THREADS, torch.get_num_threads()
    lin = Rounded(mode)
    g64 = oracle_grads(name, torch.float64, lin)
    g32 = oracle_grads(name, torch.float32, lin)
    cut = cut_rows(name)
    gcut = oracle_grads(name, torch.float64, lin, rows=cut) if cut > 0 else None
    ref = {k: G.rel(g32[k], g64[k]) for k in g64}
    # with one tile the batch without it is empty: no gradient at all
    signal = {k: (G.rel(gcut[k], g64[k]) if gcut is not None else 1.0) for k in g64}
    if mode == "bf16":   # the engine may image a value near a bf16 rounding midpoint either way (GATES)
        for seed in FLIP_SEEDS:
            gf = oracle_grads(name, torch.float64, Rounded(mode, flip_seed=seed, flip_eps=FLIP_EPS))
            ref = {k: max(ref[k], G.rel(gf[k], g64[k])) for k in g64}
    c, floor = GATES[mode]
    gate = {k: max(c * ref[k], floor) for k in keys(name, mode, g64)}
    return Reference(g64, ref, signal, gate)


def keys(name: str, mode: str, g: Dict[str, torch.Tensor]):
    """The compared gradient keys of a case: its prefix's, without the excluded ones."""
    out = EXCLUDED.get((name, mode), {})
    return [k for k in g if k.startswith(case(name).prefix) and k not in out]


def power_violations(name: str, mode: str) -> Dict[str, Tuple[float, float]]:
    r = reference(name, mode)
    return {k: (g, r.signal[k]) for k, g in r.gate.items() if not g <= r.signal[k] / POWER}


def fault_margin(name: str, mode: str, fault: str) -> Tuple[float, str]:
    """(max_k |g_fault - g64R| / gateR_k, its key): how far the emulated fault moves the compared gradients, in gates."""
    r = reference(name, mode)
    if fault == "lost_row_tile":
        if cut_rows(name) == 0:   # the whole batch lost: every gradient is zero
            return max(1.0 / gt for gt in r.gate.values()), "(all)"
        g = oracle_grads(name, torch.float64, Rounded(mode), rows=cut_rows(name))
    else:
        g = oracle_grads(name, torch.float64, Rounded(mode, fault))
    m = {k: G.rel(g[k], r.g64[k]) / gt for k, gt in r.gate.items()}
    k = max(m, key=m.get)
    return m[k], k



@functools.lru_cache(maxsize=None)
def widening(name: str) -> Dict[str, float]:
    """{k: |g64R - g64| / |g64| / common_k} in bf16x3, common_k = max(8 |g32 - g64| / |g64|, 1e-5) the unwidened bf16x3
    gate of the float64 tests against the plain oracle: how far the split-bf16 operand rounding alone moves each
    gradient, in those gates."""
    c, floor = G.GATES["bf16x3"]
    g64, g32 = oracle_grads(name, torch.float64), oracle_grads(name, torch.float32)
    g64r = oracle_grads(name, torch.float64, Rounded("bf16x3"))
    return {k: G.rel(g64r[k], g64[k]) / max(c * G.rel(g32[k], g64[k]), floor) for k in g64}
