"""CPU checks of the float64 layer reference (tests/tc_ref.py) that tests/test_gpu_layer_kernels.py holds the tensor-core and
fp32 layer kernels to: the split is the kernels' split, and every gate is narrow enough to see the faults a layer kernel
can make (the rule tests/test_grad_gate_power.py enforces for the gradient gates)."""
import math

import pytest
import torch

import tc_ref as R


def test_split_invariants():
    g = torch.Generator().manual_seed(0)
    x = torch.cat([torch.randn(20000, generator=g) * 10.0 ** torch.randint(-6, 6, (20000,), generator=g).float(),
                   torch.tensor([0.0, -0.0, 1.0, -1.0, 3.0e38, 1e-38, 0.1, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -9])])
    hi, lo = R.split(x)
    assert R.split_ok(hi, lo)
    assert not R.split_ok(*R.split(x, trunc=True))
    # round to nearest even at a tie: 1 + 2^-8 lies halfway between 1 and 1 + 2^-7
    assert float(R.bf16_rn(torch.tensor([1.0 + 2.0 ** -8]))) == 1.0
    assert float(R.bf16_rn(torch.tensor([1.0 + 3 * 2.0 ** -8]))) == 1.0 + 2.0 ** -6
    # the truncating split is another split, and further from x
    th, _ = R.split(x, trunc=True)
    assert bool(((th - x.double()).abs() >= (hi - x.double()).abs()).all())


def test_bf16x3_product_is_within_2e_16():
    g = torch.Generator().manual_seed(1)
    A, W = torch.randn(64, 300, generator=g), torch.randn(40, 300, generator=g)
    exact = A.double() @ W.double().t()
    v, ab = R.mm(A, W, "bf16x3")
    assert float(((v - exact).abs() / ab).max()) <= 2.0 ** -16
    v1, _ = R.mm(A, W, "bf16")
    assert float(((v1 - exact).abs() / ab).max()) > 2.0 ** -12   # single pass carries the operand rounding


def test_reference_activations_match_torch():
    z = torch.linspace(-15, 15, 3001, dtype=torch.float64)
    mods = {"relu": torch.nn.ReLU(), "gelu": torch.nn.GELU(), "tanh": torch.nn.Tanh(), "sigmoid": torch.nn.Sigmoid(),
            "elu": torch.nn.ELU(), "selu": torch.nn.SELU()}
    for a, m in mods.items():
        zz = z.clone().requires_grad_(True)
        y = m(zz)
        (d,) = torch.autograd.grad(y.sum(), zz)
        torch.testing.assert_close(R.act(z, a), y.detach(), rtol=1e-13, atol=1e-13)
        ok = z != 0
        torch.testing.assert_close(R.dact(z, a)[ok], d[ok], rtol=1e-13, atol=1e-13)
        # the Lipschitz bounds the gates use hold
        L1, L2 = R.LIP[a]
        assert float(R.dact(z, a).abs().max()) <= L1
        dd = (R.dact(z[1:], a) - R.dact(z[:-1], a)).abs() / (z[1] - z[0])
        jump = (z[1:] > 0) & (z[:-1] <= 0) if a in R.KINK else torch.zeros_like(dd, dtype=torch.bool)
        assert float(dd[~jump].max()) <= L2 * 1.01, a


def test_case_table_covers_the_layer_edges():
    fwd = [c for c in R.LAYER_CASES.values() if c["variant"] == "fwd"]
    assert {1, 3, 45, 129, 192, 256, 300, 520} <= {c["N"] for c in fwd}
    assert {1, 63, 64, 65, 4096} <= {c["M"] for c in fwd}
    assert set(R.ACTS) <= {c["act"] for c in fwd}
    assert {(11, 3), (64, 5), (376, 17)} <= {(c["K0"], c["K1"]) for c in fwd}
    w = [c for c in R.LAYER_CASES.values() if c["variant"] == "wgrad"]
    # both sides of the 64 / 128-wide weight-gradient tile choice (64-wide when 4 slabs of 128-wide tiles fill <= 66 SMs)
    ctas = [((c["M"] + 63) // 64) * ((c["N"] + 127) // 128) * 4 for c in w]
    assert min(ctas) * 2 <= 132 < max(ctas) * 2


@pytest.mark.parametrize("mode", ["fp32", "bf16x3", "bf16"])
@pytest.mark.parametrize("name", list(R.LAYER_CASES))
def test_gates_see_every_fault(name, mode):
    case = R.LAYER_CASES[name]
    x = R.layer_inputs(case)
    weak = {}
    for f in R.FAULTS:
        if R.fault_applies(case, mode, f):
            p = R.power(case, x, mode, f)
            if not p >= R.POWER:
                weak[f] = p
    assert not weak, {f: f"moves the outputs by {p:.3g} gates < {R.POWER}" for f, p in weak.items()}


@pytest.mark.parametrize("mode", ["fp32", "bf16x3", "bf16"])
def test_correct_reference_is_inside_its_own_gate(mode):
    for name, case in R.LAYER_CASES.items():
        if case["M"] * case["N"] > 300000:
            continue
        x = R.layer_inputs(case)
        out = R.layer_ref(case, x, mode)
        for k, (v, g, _) in out.items():
            assert bool(torch.isfinite(v).all()) and bool((g >= 0).all()), (name, k)


def test_bf16_gates_are_as_tight_as_bf16x3():
    """The single-pass mode's gates are those of bf16x3 (the operand rounding is inside the reference), not the loose
    relative tolerances of a comparison with the unrounded product."""
    case = R.LAYER_CASES["fwd_gelu"]
    x = R.layer_inputs(case)
    g3 = R.layer_ref(case, x, "bf16x3")["C"][1]
    g1 = R.layer_ref(case, x, "bf16")["C"][1]
    assert float((g1 / g3.clamp_min(1e-300)).max()) < 1.5
    assert float(g1.max()) < 1e-4
