"""CPU guard of the float64 gradient comparison (tests/gradcheck64.py, run on the GPU by tests/test_gpu_grad_f64.py):
with the oracle alone, every case's gates must be able to see the loss of the batch's last 64-row tile, and every regime
case must engage its branch.  A change to `synth`, the oracle, a regime edit or a gate that would quietly disarm a GPU
case fails here, on machines without a GPU."""
import pytest

import gradcheck64 as G


@pytest.mark.parametrize("name", list(G.CASES))
def test_gates_can_see_a_lost_row_tile(name):
    r = G.reference(name)
    assert set(r.g64) == set(r.ref) == set(r.signal) and r.g64
    for mode in G.CASES[name].modes:
        bad = G.power_violations(name, mode)
        assert not bad, {k: f"gate {g:.3g} > signal {s:.3g} / {G.POWER}" for k, (g, s) in bad.items()}


@pytest.mark.parametrize("name", [c.name for c in G.REGIME_CASES])
def test_regime_engages_its_branch(name):
    case = G.CASES[name]
    e = G.engagement(name)
    for probe, least in G.REGIMES[case.regime].items():
        assert e[probe] >= least, (probe, e[probe], least)


@pytest.mark.parametrize("name", [c.name for c in G.REGIME_CASES if c.regime == "log_std_clamp"])
def test_clamped_log_std_gets_no_gradient_in_float64(name):
    """The exact zero the GPU test demands of the engine is what float64 autograd produces."""
    case = G.CASES[name]
    g = G.reference(name).g64
    key, off = G.log_std_bias(case)
    for j in (G.CLAMPED_HIGH, G.CLAMPED_LOW):
        assert float(g[key][off + j]) == 0.0
    assert float(g[key][off + 2].abs()) > 0.0   # the component that crosses the bound in some rows still learns


def test_multi_tile_cases_span_more_than_one_tile():
    """The MLP engine's row tiles are 64 rows: the shape table must keep batches on both sides of the tile edges."""
    batches = {c.batch for c in G.SHAPE_CASES if c.engine == "mlp" and c.cfg_name == "ragged"}
    assert {63, 64, 65, 129} <= batches
    assert any(c.batch > 4 * G.TILE for c in G.SHAPE_CASES if c.engine == "mlp")

