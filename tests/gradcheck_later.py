"""Whole single-call updates of both engines against float64 from states that are not step 0.

Every step-0 gate (tests/gradcheck64.py, tests/gradmatrix.py) starts from targets equal to the online networks, an unset
mean_std, Adam at t = 0 and iteration 0.  There a target pass that reads the online weights, or a target image one Polyak
step stale, computes the same numbers as a correct one, and the carried mean_std, the Adam counters and the delayed
iterations never enter a gated value.  This module gates the update `step` / `replay_step` makes from a later state:

- State: the engine's whole state between two updates (`State`: parameters and targets, Adam moments, log_alpha, the
  carried mean_std pair and both Adam counters), exported from an engine (`export_state`), loaded into an engine
  (`load_state`) or into the oracles (`OracleDSACT.load_state`).
- Two kinds of start: `synthetic_state` (targets = online + an independent perturbation of TARGET_SCALE x each tensor's
  RMS, Adam moments of the state's own gradients with v > 0, counters and iteration of SYNTH, mean_std off the batch
  mean by MEAN_STD_OFF, log_alpha at LOG_ALPHA), and the engine's own state after n replay-fed updates with
  its graphs captured (`trajectory`, TRAJ_N), which is where an image or stamp left over from an earlier graph replay
  would show.
- At the gated update k, from the same state: (1) the gradients the single-call step leaves in `grads` against float64
  under gradcheck64's rule (err_k <= max(c ref_k, floor), ref_k from the fp32 oracle from that state, and the power rule
  against a lost 64-row tile); (2) parameters, targets, moments, the committed mean_std and the counters against
  step_ref.apply_ref fed the engine's own step-k gradients and its pre-step state, element by element under step_ref's
  gates, with the policy, its moments, log_alpha and every target bit-unchanged on odd k; (3) tb_info through
  gradcheck64.tb_deviations.
- FAULTS: wiring faults emulated in the float64 oracle (or in apply_ref for the update's own arithmetic); every one must
  move some compared gradient or update element by POWER gates in every case where it applies
  (tests/test_grad_later_power.py).  tests/test_gpu_grad_later.py runs the engines.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import numpy as np
import torch

import gradcheck64 as G
import gradmatrix as GM
import step_ref as S
from dsac_v2_b200 import synth

POWER = G.POWER
# synthetic later states: parity -> (iteration k, critics' Adam counter, policy / temperature counter).  k = 1000 follows
# 1000 updates of which 500 were delayed; k = 7 follows seven, four of them delayed.  Odd k runs the critics only.
SYNTH = {"even": (1000, 1000, 500), "odd": (7, 7, 4)}
# Target perturbation, in units of each tensor's RMS.  A target one Polyak step stale differs from the right one by
# tau / (1 - tau) of it, so that fault sets its size: at 0.1 it moves humanoid B = 4096's gradients by 2.0 gates only, at
# 0.5 every fault of FAULTS clears POWER gates in every case (tests/test_grad_later_power.py prints the margins, DESIGN.md
# §5 records them).
TARGET_SCALE = 0.5
MOMENT_NOISE = 0.5         # Adam's m = the state's gradient + this x its RMS of noise (see synthetic_state)
MEAN_STD_OFF = (1.3, 0.8)  # carried mean_std = these factors x the batch mean of each critic's std at the gated update
# log_alpha of the synthetic states (the weights start at 1.0).  alpha = 0.14 lets the critics' part of the policy
# gradient show: at log_alpha = -1 a policy backward through critics the early apply already moved is 4.5 gates away at
# DSAC_V1 asym bf16x3, at -2 it clears POWER everywhere while alpha's own faults still do.
LOG_ALPHA = -2.0
TRAJ_N = (1, 6)             # engine updates before the gated one in the real-trajectory states (k = n: odd and even)


@dataclass(frozen=True)
class Case:
    name: str
    base: object                # a gradcheck64.Case or a gradmatrix.Case (built through the drop-in's route)
    replay: bool = False        # the gated update through replay_step with given indices (the benchmarked call)
    trajectory: bool = False    # also the states after TRAJ_N engine updates, graphs captured

    @property
    def matrix(self) -> bool:
        return isinstance(self.base, GM.Case)

    @property
    def algo(self) -> str:
        return self.base.algo

    @property
    def v1(self) -> bool:
        return self.algo == "DSAC_V1"

    @property
    def batch(self) -> int:
        return self.base.batch

    @property
    def cfg(self) -> dict:
        return self.base.cfg

    @property
    def modes(self) -> Tuple[str, ...]:
        return (self.base.mode,) if self.matrix else self.base.modes

    @property
    def hyper(self) -> dict:
        return dict(synth.HYPER) if self.matrix else self.base.hyperparameters

    def inputs(self):
        """(weights, minibatch, noise) of the base case at step 0."""
        return GM.inputs(self.base) if self.matrix else G.inputs(self.base)

    def noise_for_engine(self, n):
        return G.noise_for_engine(self.base, n) if not self.matrix else GM.noise_for_engine(self.base, n)

    def oracle(self, dtype, state: "State"):
        orc = GM.make_oracle(self.base, dtype) if self.matrix else G.make_oracle(self.base, self.inputs()[0], dtype)
        orc.load_state(state.params, state.m, state.v, state.mean_std, state.tq, state.tp)
        return orc

    def make_engine(self, mode: str, use_graph: bool = False):
        if self.matrix:
            return GM.make_engine(self.base)
        return G.make_engine(self.base, "fp32" if mode == "heads" else mode, use_graph=use_graph)


def _m(algo, route, std, shape):
    return GM.Case(algo, route, std, "TanhGaussDistribution", "linear", "linear", shape, "one")


_MLP = [Case("ragged_b1000", G.CASES["ragged_b1000"], trajectory=True),
        Case("asym_b2200", G.CASES["asym_b2200"]),
        Case("humanoid_b4096", G.CASES["humanoid_b4096"], replay=True, trajectory=True),
        Case("wide_b200", G.CASES["wide_b200"])]
_ROUTED = [Case(f"{tag}_{route[4:]}_b1000", _m(algo, route, std, shape))
           for tag, algo, std, shape in (("v1_asym", "DSAC_V1", "mlp_shared", "asym"),
                                         ("separated_ragged", "DSAC_V2", "mlp_separated", "ragged"),
                                         ("parameter_ragged", "DSAC_V2", "parameter", "ragged"))
           for route in ("mlp_fp32", "mlp_bf16x3")]
_HEADS = [Case("cnn_carracing_b256", G.CASES["cnn_carracing_b256"]),
          Case("v1_pendulum_b4096", G.CASES["v1_pendulum_b4096"]),
          Case("heads_separated_ragged_b1000", G.CASES["separated_ragged_b1000"])]
CASES = {c.name: c for c in _MLP + _ROUTED + _HEADS}


# ---- state ------------------------------------------------------------------------------------------------------------
@dataclass
class State:
    """Everything one update carries to the next (float32 CPU tensors in the state_dict schema)."""
    params: Dict[str, torch.Tensor]   # online, *_target and log_alpha
    m: Dict[str, torch.Tensor]        # online keys and log_alpha
    v: Dict[str, torch.Tensor]
    mean_std: Tuple[float, float]     # < 0: unset (always so on DSAC_V1)
    tq: int                           # Adam steps of the critics' optimizers
    tp: int                           # Adam steps of the policy and temperature optimizers


def _unflat(eng, flat: torch.Tensor) -> Dict[str, torch.Tensor]:
    schema, n = eng._schema()
    out = {key: flat[off:off + cnt].view(shape).clone() for key, _, off, cnt, shape in schema}
    out["log_alpha"] = flat[n].clone()
    return out


def flat(eng, d: Dict[str, torch.Tensor], targets: bool = False) -> torch.Tensor:
    """The engine's flat buffer (params layout, or with `targets` the targets') of a state_dict-schema dict, float64."""
    schema, n = eng._schema()
    out = torch.zeros(n if targets else n + 1, dtype=torch.float64)
    for key, tkey, off, cnt, shape in schema:
        out[off:off + cnt] = torch.as_tensor(d[tkey if targets else key]).reshape(-1).double()
    if not targets:
        out[n] = float(d["log_alpha"])
    return out


def _ints(eng) -> torch.Tensor:
    return eng.state.detach().cpu().view(torch.int32)


def export_state(eng) -> State:
    torch.cuda.synchronize(eng.device)
    st, ints = eng.state.detach().cpu(), _ints(eng)
    return State(eng.export_weights(), _unflat(eng, eng.adam_m.detach().cpu()), _unflat(eng, eng.adam_v.detach().cpu()),
                 (float(st[0]), float(st[1])), int(ints[8]), int(ints[9]))


def load_state(eng, s: State) -> None:
    eng.load_weights(s.params)
    with torch.no_grad():
        eng.adam_m.copy_(flat(eng, s.m).float())
        eng.adam_v.copy_(flat(eng, s.v).float())
    eng.set_carry(s.mean_std[0], s.mean_std[1], s.tq, s.tp)


def _online(params: dict) -> Dict[str, torch.Tensor]:
    return {k: v for k, v in params.items() if "_target." not in k and k != "log_alpha"}


def _target_key(k: str) -> str:
    net, rest = k.split(".", 1)
    return f"{net}_target.{rest}"


@functools.lru_cache(maxsize=None)
def synthetic_state(name: str, parity: str) -> State:
    """The synthetic later state of a case (see the module docstring), deterministic per (case, parity)."""
    case = CASES[name]
    w, b, n = case.inputs()
    k, tq, tp = SYNTH[parity]
    g = np.random.default_rng([sum(map(ord, name)), k])
    f32 = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float32))
    online = {key: torch.as_tensor(np.asarray(w[key], dtype=np.float32)) for key in w
              if "_target." not in key and key != "log_alpha"}
    params = dict(online)
    for key, x in online.items():
        rms = float(x.double().pow(2).mean().sqrt()) or 1.0
        params[_target_key(key)] = f32(x.numpy() + TARGET_SCALE * rms * g.standard_normal(x.shape))
    params["log_alpha"] = f32(LOG_ALPHA)
    # moments as a run would leave them after t steps of its optimizer: bias corrections 1 - beta^t times m' = the
    # state's own gradient g (fp32 oracle) plus MOMENT_NOISE x its RMS of independent noise and v' = m'^2 +
    # (rms x U(0.25, 0.75))^2 > 0.  So |m^| / sqrt(v^) < 1 at any t, and each Adam step moves its tensor coherently by
    # about lr per element, as the early critic apply moves the critics that the policy backward must not see
    zeros = {k2: torch.zeros_like(x) for k2, x in _m_keys(online).items()}
    o = case.oracle(torch.float32, State(params, zeros, zeros, (-1.0, -1.0), 0, 0))
    tb = o.compute_gradients(b, n)
    grads = {key: gr.detach().double().numpy() for key, gr in o.grad_dict().items()}
    if "log_alpha" not in grads:
        grads["log_alpha"] = np.array(1.0)
    m, v = {}, {}
    for key, gr in grads.items():
        rms = float(np.sqrt(np.mean(gr ** 2))) or 1e-3
        t = tq if not (key.startswith("policy") or key == "log_alpha") else tp
        mm = gr + MOMENT_NOISE * rms * g.standard_normal(gr.shape)
        m[key] = f32((1 - 0.9 ** t) * mm)
        v[key] = f32((1 - 0.999 ** t) * (mm ** 2 + (rms * g.uniform(0.25, 0.75, gr.shape)) ** 2))
    if case.v1:
        ms = (-1.0, -1.0)
    else:
        ms = tuple(float(np.float32(f * tb[f"DSAC2/mean_std{i + 1}"])) for i, f in enumerate(MEAN_STD_OFF))
    return State(params, m, v, ms, tq, tp)


def _m_keys(online: dict) -> Dict[str, torch.Tensor]:
    d = dict(online)
    d["log_alpha"] = torch.tensor(0.0)
    return d


# ---- the float64 yardstick from a state --------------------------------------------------------------------------------
def oracle_grads(case: Case, state: State, b, n, dtype, rows: Optional[int] = None, fault: Optional[str] = None):
    """(gradients in float64, tb_info) of the case's oracle from `state`; `fault`: a gradient fault of FAULTS."""
    if rows is not None:
        b, n = {k: v[:rows] for k, v in b.items()}, [x[:rows] for x in n]
    if fault is not None:
        return FAULTS[fault][0](case, state, b, n, dtype)
    orc = case.oracle(dtype, state)
    tb = orc.compute_gradients(b, n)
    return {k: g.detach().double() for k, g in orc.grad_dict().items()}, tb


def reference(case: Case, state: State, b, n) -> G.Reference:
    assert torch.get_num_threads() == G.ORACLE_THREADS, torch.get_num_threads()
    g64, tb64 = oracle_grads(case, state, b, n, torch.float64)
    g32, tb32 = oracle_grads(case, state, b, n, torch.float32)
    gcut = oracle_grads(case, state, b, n, torch.float64, rows=G.TILE * ((case.batch - 1) // G.TILE))[0]
    return G.Reference(g64, tb64, tb32, {k: G.rel(g32[k], g64[k]) for k in g64}, {k: G.rel(gcut[k], g64[k]) for k in g64})


def gated_rows(case: Case, k: int):
    """(minibatch, noise) of the gated update k of a synthetic state: gradcheck64's step-0 rows and noise streams (as
    the replay ring's rows, drawn in the order of `replay_idx` when the case runs replay_step)."""
    _, b, n = case.inputs()
    if case.replay:
        idx = replay_idx(case.batch, case.batch, k)
        b = {key: v[idx] for key, v in b.items()}
    return b, n


def replay_idx(batch: int, capacity: int, k: int) -> np.ndarray:
    return np.random.default_rng([91, k]).integers(0, capacity, size=batch).astype(np.int64)


@functools.lru_cache(maxsize=None)
def synthetic_reference(name: str, parity: str) -> G.Reference:
    case = CASES[name]
    b, n = gated_rows(case, SYNTH[parity][0])
    return reference(case, synthetic_state(name, parity), b, n)


def gates(case: Case, r: G.Reference, mode: str) -> Dict[str, float]:
    c, floor = G.GATES[mode]
    return {k: max(c * x, floor) for k, x in r.ref.items()}


def power_violations(case: Case, r: G.Reference, mode: str):
    return {k: (g, r.signal[k]) for k, g in gates(case, r, mode).items() if not g <= r.signal[k] / POWER}


# ---- the update against step_ref.apply_ref ----------------------------------------------------------------------------
def apply_hyper(case: Case) -> dict:
    h = case.hyper
    return dict(tau=h["tau"], lr_q=h["value_learning_rate"], lr_pi=h["policy_learning_rate"], lr_alpha=h["alpha_learning_rate"],
                adam_beta1=0.9, adam_beta2=0.999, adam_eps=1e-8)


def expected_update(case: Case, eng, pre: State, grads: Dict[str, torch.Tensor], k: int, fault: Optional[str] = None,
                    delayed: Optional[bool] = None):
    """step_ref.apply_ref on the engine's flat buffers: {"w", "m", "v", "t"} as (value, gate), from the pre-step state
    and the step's gradients (`grads` in the state_dict schema, log_alpha's included)."""
    hy = apply_hyper(case)
    h = case.hyper
    delayed = (k % h["delay_update"] == 0) if delayed is None else delayed
    nq2 = int(eng.layout.n_q) * (1 if case.v1 else 2)
    sh = S.adam_step_sizes(hy, pre.tq, pre.tp, fault="bc_t" if fault == "bc_t" else None)
    f = lambda d, t=False: S.f32(flat(eng, d, t))
    return S.apply_ref(f(pre.params), f(grads), f(pre.m), f(pre.v), f(pre.params, True), [], nq2, hy, sh,
                       torch.tensor(bool(delayed)), bool(h["auto_alpha"]))


def update_deviations(case: Case, eng, pre: State, post: State, grads, k: int):
    """[(what, worst |got - want| / gate, index)] of every update element outside its gate, and the bit-unchanged checks."""
    exp = expected_update(case, eng, pre, grads, k)
    got = {"w": flat(eng, post.params), "m": flat(eng, post.m), "v": flat(eng, post.v), "t": flat(eng, post.params, True)}
    bad = []
    for key, (val, gate) in exp.items():
        if key == "g":
            continue
        d = (got[key] - val).abs() / gate
        d = torch.where(torch.isnan(d), torch.full_like(d, torch.inf), d)
        if not bool((d <= 1.0).all()):
            i = int(d.argmax())
            bad.append((key, float(d[i]), i))
    h = case.hyper
    delayed = k % h["delay_update"] == 0
    nq2 = int(eng.layout.n_q) * (1 if case.v1 else 2)
    if not delayed:   # the policy, its moments, log_alpha and every target bit-unchanged
        for key, a, b_ in (("w", post.params, pre.params), ("m", post.m, pre.m), ("v", post.v, pre.v)):
            if not torch.equal(flat(eng, a)[nq2:], flat(eng, b_)[nq2:]):
                bad.append((f"{key} of policy / log_alpha changed on odd k", float("inf"), -1))
        if not torch.equal(flat(eng, post.params, True), flat(eng, pre.params, True)):
            bad.append(("targets changed on odd k", float("inf"), -1))
    if (post.tq, post.tp) != (pre.tq + 1, pre.tp + int(delayed)):
        bad.append((f"counters {(post.tq, post.tp)} after {(pre.tq, pre.tp)}", float("inf"), -1))
    return bad


def mean_std_deviation(case: Case, eng, pre: State, gb: int):
    """The committed mean_std pair against the EMA restated from the step's own std sums (step_ref.mean_std_of):
    [(critic, got, want, gate)] outside the gate."""
    if case.v1:
        return []
    st = eng.state.detach().cpu()
    sc = {"tau_b": S.c32(case.hyper.get("tau_b", case.hyper["tau"]))}
    bad = []
    for i in range(2):
        t = S.Track()
        y = S.mean_std_of(t, sc, float(st[4 + i]), pre.mean_std[i], gb, (1,))
        want, gate = float(y.detach()[0]), float(t.gate(y)[0])
        if not abs(float(st[i]) - want) <= gate:
            bad.append((i, float(st[i]), want, gate))
    return bad


# ---- emulated faults ---------------------------------------------------------------------------------------------------
def _with_targets(state: State, targets) -> State:
    p = dict(state.params)
    p.update(targets)
    return State(p, state.m, state.v, state.mean_std, state.tq, state.tp)


def _f_target_online(case, state, b, n, dtype):
    on = _online(state.params)
    return oracle_grads(case, _with_targets(state, {_target_key(k): v for k, v in on.items()}), b, n, dtype)


def _f_target_stale(case, state, b, n, dtype):
    """The targets one Polyak step back: T = polyak T' + (1 - polyak) P  =>  T' = (T - tau P) / (1 - tau)."""
    tau = case.hyper["tau"]
    on = _online(state.params)
    old = {_target_key(k): (state.params[_target_key(k)].double() - tau * v.double()) / (1 - tau) for k, v in on.items()}
    return oracle_grads(case, _with_targets(state, old), b, n, dtype)


def _f_mean_std_batch(case, state, b, n, dtype):
    return oracle_grads(case, State(state.params, state.m, state.v, (-1.0, -1.0), state.tq, state.tp), b, n, dtype)


def _f_mean_std_no_ema(case, state, b, n, dtype):
    orc = case.oracle(dtype, state)
    orc.tau_b = 0.0
    tb = orc.compute_gradients(b, n)
    return {k: g.detach().double() for k, g in orc.grad_dict().items()}, tb


def _f_alpha_previous(case, state, b, n, dtype):
    """exp of log_alpha before the last temperature step (that step undone from the state's moments)."""
    t = state.tp
    bc1, bc2 = 1 - 0.9 ** t, 1 - 0.999 ** t
    lr = case.hyper["alpha_learning_rate"]
    m, v = float(state.m["log_alpha"]), float(state.v["log_alpha"])
    prev = float(state.params["log_alpha"]) + lr / bc1 * m / (v ** 0.5 / bc2 ** 0.5 + 1e-8)
    p = dict(state.params)
    p["log_alpha"] = torch.tensor(prev, dtype=torch.float64)
    g, tb = oracle_grads(case, State(p, state.m, state.v, state.mean_std, state.tq, state.tp), b, n, dtype)
    g["log_alpha"] = oracle_grads(case, state, b, n, dtype)[0]["log_alpha"]   # the temperature's own gradient keeps its value
    return g, tb


def _f_policy_after_critic_adam(case, state, b, n, dtype):
    """The policy gradient through the critics this update's Adam has already moved."""
    orc = case.oracle(dtype, state)
    tb = orc.compute_gradients(b, n)
    g = {k: x.detach().double() for k, x in orc.grad_dict().items()}
    for net in orc.NETS:
        if net != "policy":
            orc._adam(net, orc.p[net], orc.grads[net])
    moved = {k: v for k, v in orc.state_dict().items() if not k.startswith("policy") and "_target." not in k}
    p = dict(state.params)
    p.update(moved)
    g2 = oracle_grads(case, State(p, state.m, state.v, state.mean_std, state.tq, state.tp), b, n, dtype)[0]
    g.update({k: x for k, x in g2.items() if k.startswith("policy.")})
    return g, tb


# fault -> (gradient fault: oracle function, or None for an update fault; applies to (case, parity))
FAULTS = {
    "target_reads_online": (_f_target_online, lambda c, p: True),
    "target_one_polyak_stale": (_f_target_stale, lambda c, p: True),
    "mean_std_batch_mean": (_f_mean_std_batch, lambda c, p: not c.v1),
    "mean_std_without_ema": (_f_mean_std_no_ema, lambda c, p: not c.v1),
    "alpha_previous_log_alpha": (_f_alpha_previous, lambda c, p: bool(c.hyper["auto_alpha"])),
    "policy_grad_after_critic_adam": (_f_policy_after_critic_adam, lambda c, p: True),
    "polyak_on_odd_iteration": (None, lambda c, p: p == "odd"),
    "adam_bias_correction_at_t": (None, lambda c, p: True),
}


class _Layout:
    """What `expected_update` needs of an engine, without one: the flat schema and the critics' span."""

    def __init__(self, case: Case):
        self._case = case
        w = case.inputs()[0]
        self._keys = [(k, _target_key(k), tuple(np.shape(w[k]))) for k in w if "_target." not in k and k != "log_alpha"]
        crit = ("q.",) if case.v1 else ("q1.", "q2.")
        self.layout = type("L", (), {})()
        self.layout.n_q = sum(int(np.prod(s)) for k, _, s in self._keys if k.startswith(crit[0]))

    def _schema(self):
        out, off = [], 0
        critics = [x for x in self._keys if not x[0].startswith("policy.")]
        for key, tkey, shape in critics + [x for x in self._keys if x[0].startswith("policy.")]:
            cnt = int(np.prod(shape))
            out.append((key, tkey, off, cnt, shape))
            off += cnt
        return out, off


def fault_margin(name: str, parity: str, fault: str) -> Tuple[float, str]:
    """(largest move / gate over the compared elements, where): how far the emulated fault moves the gated update of a
    synthetic state, in the gates of the case's loosest mode."""
    case = CASES[name]
    state = synthetic_state(name, parity)
    r = synthetic_reference(name, parity)
    fn = FAULTS[fault][0]
    k = SYNTH[parity][0]
    if fn is not None:
        b, n = gated_rows(case, k)
        g = fn(case, state, b, n, torch.float64)[0]
        per_mode = []   # the loosest mode decides
        for mode in case.modes:
            m = {key: G.rel(g[key], r.g64[key]) / gt for key, gt in gates(case, r, mode).items()}
            key = max(m, key=m.get)
            per_mode.append((m[key], key))
        return min(per_mode)
    lay = _Layout(case)
    grads = {key: x.float() for key, x in r.g64.items()}
    if "log_alpha" not in grads:
        grads["log_alpha"] = torch.tensor(0.0)
    base = expected_update(case, lay, state, grads, k)
    moved = (expected_update(case, lay, state, grads, k, delayed=True) if fault == "polyak_on_odd_iteration"
             else expected_update(case, lay, state, grads, k, fault="bc_t"))
    best = (0.0, "")
    for key in ("t",) if fault == "polyak_on_odd_iteration" else ("w", "m", "v", "t"):   # Polyak alone: the targets
        d = float(((moved[key][0] - base[key][0]).abs() / base[key][1]).max())
        if d > best[0]:
            best = (d, key)
    return best


# ---- the CUDA side ----------------------------------------------------------------------------------------------------
def tb_of(eng, algo: str, B: int) -> Dict[str, float]:
    from dsac_v2_b200.engine import STAT_KEYS
    s = eng.read_stats(B)
    if algo == "DSAC_V1":
        from oracle.dsact_oracle import V1_TB_KEYS
        vals = [s[k] for k in STAT_KEYS]
        return {k: vals[c] for k, c in zip(V1_TB_KEYS, G.V1_COLS)}
    return {k: s[k] for k in STAT_KEYS[:14]}


def _device(b):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in b.items()}


def bind_ring(eng, rows: dict) -> int:
    """A flat replay ring holding `rows` (numpy, as a minibatch), logp zero; its capacity."""
    cap = len(rows["rew"])
    eng.bind_replay(cap)
    d = _device(rows)
    d["logp"] = torch.zeros(cap, device=d["rew"].device)
    eng.replay_add(d, cap, 0)
    return cap


def gated_step(case: Case, eng, k: int, b, nz, ring: Optional[int] = None, idx=None):
    """The single-call update k on the engine: replay_step over the bound ring with `idx`, or step on device rows."""
    if ring is not None:
        eng.replay_step(case.batch, ring, k, idx=idx, noise=nz)
    else:
        eng.step(_device(b), k, tuple(torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in nz))
    torch.cuda.synchronize()


def run_synthetic(case: Case, mode: str, parity: str):
    """The engine's gated update from the synthetic state: (pre-state, post-state, gradients, tb_info, engine), the engine
    still open (the caller closes it)."""
    k = SYNTH[parity][0]
    state = synthetic_state(case.name, parity)
    eng = case.make_engine(mode, use_graph=case.replay)
    _, b0, n = case.inputs()
    nz = case.noise_for_engine(n)
    ring, idx = None, None
    if case.replay:
        ring = bind_ring(eng, b0)
        idx = torch.from_numpy(replay_idx(case.batch, ring, k)).cuda()
    load_state(eng, state)
    gated_step(case, eng, k, b0, nz, ring, idx)
    return state, export_state(eng), eng.export_weights(grads=True), tb_of(eng, case.algo, case.batch), eng


def trajectory(case: Case, mode: str, n_updates: int):
    """n_updates replay-fed engine updates (graphs captured, given indices, host noise) from the case's step-0 weights,
    then the gated update n_updates.  The ring holds the case's step-0 minibatch (rows 0 .. B-1) and B rows more; the
    earlier updates draw from all of it, the gated one takes the step-0 rows in order with the step-0 noise, where the
    power rule of gradcheck64's case holds (humanoid B = 4096 in bf16x3: log_alpha's lost-tile signal 10.8 gates at step
    0, 2.2 to 3.7 gates for rows drawn at random).  Returns (state before it, its minibatch and noise, post-state,
    gradients, tb_info, engine)."""
    B = case.batch
    w, b0, n0 = case.inputs()
    more = synth.make_batch(case.cfg, B, 0, seed=321)
    rows = {key: np.concatenate([b0[key], more[key]]) for key in b0}
    eng = case.make_engine(mode, use_graph=True)
    eng.load_weights(w)
    ring = bind_ring(eng, rows)
    idx_dev = torch.zeros(B, dtype=torch.int64, device="cuda")   # one buffer: every update replays the captured graph
    for k in range(n_updates):
        idx_dev.copy_(torch.from_numpy(replay_idx(B, ring, k)))
        eng.replay_step(B, ring, k, idx=idx_dev, noise=case.noise_for_engine(synth.make_noise(case.cfg, B, 100 + k)))
    pre = export_state(eng)
    idx_dev.copy_(torch.arange(B))
    eng.replay_step(B, ring, n_updates, idx=idx_dev, noise=case.noise_for_engine(n0))
    torch.cuda.synchronize()
    return pre, b0, n0, export_state(eng), eng.export_weights(grads=True), tb_of(eng, case.algo, B), eng
