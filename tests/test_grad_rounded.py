"""CPU guard of the rounded-operand float64 oracle (tests/gradcheck_rounded.py, run against the engine by
tests/test_gpu_grad_rounded.py): its dense layer is tc_ref's layer reference, the hook it enters the oracle by changes
nothing when it is F.linear, its gates can see a lost row tile and the wiring faults it emulates, and the bf16x3 gates
the float64 tests widen are widened by the operand rounding itself."""
import math

import pytest
import torch
import torch.nn.functional as F

import gradcheck64 as G
import gradcheck_rounded as GR
import tc_ref as R


# ---- the rounded dense layer is tc_ref's ------------------------------------------------------------------------------
def _layer_outputs(case, x, mode):
    """tc_ref.layer_ref's checked value of `case`, computed through GR.Rounded's forward or autograd backward."""
    lin = GR.Rounded(mode)
    v = case["variant"]
    if v == "fwd":
        A = torch.cat([x["A0"], x["A1"]], 1) if case["K1"] else x["A0"]
        return R.act(lin(A.double(), x["B"].double(), x["bias"].double()), case["act"])
    if v == "dgrad":   # dz = A0 [M, K], the layer's weight B [K, N]: dx = dz . W, times act'
        dz, W = x["A0"].double(), x["B"].double().requires_grad_(False)
        xin = torch.zeros(dz.shape[0], W.shape[1], dtype=torch.float64, requires_grad=True)
        lin(xin, W, None).backward(dz)
        return xin.grad * x["D"].double()
    dz, xin = x["A0"].double(), x["B"].double()   # wgrad: dz [batch, M], the layer input [batch, N]: dW = dz^T . x
    W = torch.zeros(dz.shape[1], xin.shape[1], dtype=torch.float64, requires_grad=True)
    lin(xin, W, None).backward(dz)
    return x["C0"].double() + W.grad


@pytest.mark.parametrize("mode", GR.MODES)
@pytest.mark.parametrize("name", ["fwd_seg_376_17", "fwd_seg_11_3", "fwd_n45", "dgrad_gelu", "dgrad_n45", "wgrad_odd",
                                  "wgrad_64wide"])
def test_rounded_linear_is_the_layer_reference(name, mode):
    """Forward (two K segments included), input gradient and weight gradient equal tc_ref.layer_ref to float64 rounding."""
    case = R.LAYER_CASES[name]
    x = R.layer_inputs(case)
    want = R.layer_ref(case, x, mode)["C"][0]
    got = _layer_outputs(case, x, mode)
    assert float((got - want).abs().max()) <= 1e-12 * max(1.0, float(want.abs().max())), name


# ---- the hook ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["ragged_b65", "layered_q_b200", "mlp_separated_ragged_b1000", "parameter_ragged_b1000",
                                  "v1mlp_asym_b4300"])
def test_linear_hook_is_inert(name):
    """The oracle with `linear` handed F.linear (or a wrapper around it, counted, so the hook is seen to carry every dense
    layer) gives the plain oracle's gradients bit for bit, in float64 and float32."""
    calls = []

    def wrapped(x, w, b):
        calls.append(w.shape)
        return F.linear(x, w, b)

    w, b, n = GR.inputs(name)
    for dtype in (torch.float64, torch.float32):
        plain = GR.make_oracle(name, dtype)
        assert plain.linear is F.linear   # the default path
        plain.compute_gradients(b, n)
        want = plain.grad_dict()
        for lin in (F.linear, wrapped):
            got = GR.oracle_grads(name, dtype, lin)
            assert set(got) == set(want)
            for k in want:
                assert torch.equal(got[k], want[k].detach().double()), (name, dtype, k)
    assert calls


# ---- the power rule ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", GR.GATED)
@pytest.mark.parametrize("name", list(GR.CASES))
def test_rounded_gates_can_see_a_lost_row_tile(name, mode):
    r = GR.reference(name, mode)
    assert r.gate and set(r.g64) == set(r.ref) == set(r.signal)
    bad = GR.power_violations(name, mode)
    assert not bad, {k: f"gate {g:.3g} > signal {s:.3g} / {GR.POWER}" for k, (g, s) in bad.items()}
    w = min(r.gate, key=lambda k: r.signal[k] / r.gate[k])
    print(f"\n{name} {mode}: min signal/gate {r.signal[w] / r.gate[w]:.3g} ({w}), max refR {max(r.ref.values()):.3g}")


def test_case_table_covers_the_issue_shapes():
    names = set(GR.CASES)
    assert {c.name for c in G.SHAPE_CASES if c.engine == "mlp"} <= names
    assert {"mlp_separated_ragged_b1000", "mlp_separated_ragged_b2200", "parameter_ragged_b1000", "parameter_ragged_b2200",
            "v1mlp_asym_b4300", "asym_b8500", "deep_pi_b8500", "ragged_b8500"} <= names


# ---- emulated faults --------------------------------------------------------------------------------------------------
# Per mode: faults every case sees on its own, and faults only some cases see (the suite as a whole sees them).  A
# truncating split moves a bf16x3 product by lo * lo-sized terms only (tc_ref.power), and an unrounded dz in the
# weight gradient differs from hi + lo by about 2^-17 of dz: bf16x3 sees those in few cases or none, bf16 in every one.
EVERY_CASE = {"bf16x3": ("drop_hilo", "one_plane", "lost_row_tile"),
              "bf16": ("trunc_w", "trunc_act", "trunc_dz", "lost_row_tile")}
SOME_CASE = {"bf16x3": ("trunc_w", "trunc_act", "trunc_dz"), "bf16": ("fp32_dz_wgrad",)}


def test_fault_table_is_complete():
    """Every fault is seen in some mode; bf16x3-only faults are the two that single-pass bf16 cannot have."""
    seen = {f for m in GR.GATED for f in EVERY_CASE[m] + SOME_CASE[m]}
    assert seen == set(GR.FAULTS)
    assert set(GR.FAULTS) - set(EVERY_CASE["bf16"] + SOME_CASE["bf16"]) == {"drop_hilo", "one_plane"}


@pytest.mark.parametrize("fault,mode", [(f, m) for m in GR.GATED for f in EVERY_CASE[m] + SOME_CASE[m]])
def test_gates_see_the_emulated_faults(fault, mode):
    m = {name: GR.fault_margin(name, mode, fault) for name in GR.CASES}
    lo = min(m, key=lambda n: m[n][0])
    hi = max(m, key=lambda n: m[n][0])
    print(f"\nfault {fault} {mode}: smallest margin {m[lo][0]:.3g} gates ({lo}, {m[lo][1]}), "
          f"largest {m[hi][0]:.3g} ({hi}, {m[hi][1]})")
    if fault in EVERY_CASE[mode]:
        assert m[lo][0] >= GR.POWER, (lo, m[lo])
    else:
        assert m[hi][0] >= GR.POWER, (hi, m[hi])


# ---- the near-midpoint flips of the bf16 gate -------------------------------------------------------------------------
def test_flips_touch_only_computed_values_near_a_midpoint():
    """Rounded(flip_eps) moves a value's bf16 image to the other neighbour only when the value is a float64 result (not
    an fp32 number: weights, obs and act image identically in the engine) within flip_eps of a rounding midpoint, and
    gives every use of one value the same image."""
    lin = GR.Rounded("bf16", flip_eps=GR.FLIP_EPS)
    mid = 1.0 + 2.0 ** -8                                   # the midpoint between bf16 1 and 1 + 2^-7
    x = torch.tensor([[mid + 2.0 ** -30, mid - 2.0 ** -30, mid + 2.0 ** -12, 0.3]], dtype=torch.float64)
    hi = R.bf16_rn(x)
    got = lin.planes(x, "act")[0]
    assert float(hi[0, 0]) == 1.0 and float(got[0, 0]) == 1.0 + 2.0 ** -7   # fp32 rounds it to the midpoint, a tie
    assert torch.equal(got[0, 2:], hi[0, 2:])                              # far from a midpoint / not near one
    exact = x.float().double()                                             # fp32 numbers: never flipped
    assert torch.equal(lin.planes(exact, "act")[0], R.bf16_rn(exact))
    assert torch.equal(lin.planes(x, "w")[0], hi)                           # weights: never flipped
    assert torch.equal(lin.planes(x, "dz")[0], lin.planes(x, "dz_wgrad")[0])
    half = GR.Rounded("bf16", flip_eps=GR.FLIP_EPS, flip_seed=1)
    assert torch.equal(half.planes(x, "act")[0], half.planes(x, "dz")[0])


# ---- the widened bf16x3 gates of the float64 tests --------------------------------------------------------------------
@pytest.mark.parametrize("name", list(GR.WIDENED))
def test_widened_bf16x3_gates_are_the_rounding_s_doing(name):
    """|g64R - g64| / |g64| of the widened tensors, in unwidened gates: what DESIGN.md §5 and the comments quote, inside
    the widened gate, and (but for parameter at B = 2200) beyond the common one."""
    key, factor, measured = GR.WIDENED[name]
    w = GR.widening(name)
    covered = {key: w[key]} if key else w
    k = max(covered, key=covered.get)
    print(f"\n{name}: the rounding alone moves {k} by {covered[k]:.3g} common bf16x3 gates (widened {factor:g} x)")
    assert math.isclose(covered[k], measured, rel_tol=0.02), (k, covered[k], measured)
    assert max(covered.values()) <= factor
    if measured > 1.0:
        assert covered[k] > 1.0
    if key:   # a single tensor widened: the rest of the case needs no widening
        assert max(v for kk, v in w.items() if kk != key) < 1.0
