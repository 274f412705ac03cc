"""Step-0 gradients of both engines against the float64 oracle (tests/gradcheck64.py) at multi-tile batches, at the
benchmarked shapes and in the clamped / saturated / tied regimes of the loss and sampling arithmetic.

Every gradient tensor must be as close to float64 as the fp32 oracle, up to the factor of its arithmetic's gate, and every
gate must be able to see the loss of the batch's last 64-row tile.  Each test prints one `GRADF64` line: the largest
err_k / ref_k and the smallest signal_k / gate_k of the case."""
import numpy as np
import pytest
import torch

import gradcheck64 as G

pytestmark = pytest.mark.gpu

PARITY = [(c.name, m) for c in G.CASES.values() for m in c.modes]


def _report(name, mode, res):
    worst = max(res, key=lambda k: res[k][0] / max(res[k][2], 1e-30))
    weakest = min(res, key=lambda k: res[k][3] / res[k][1])
    tightest = max(res, key=lambda k: res[k][0] / res[k][1])
    e, g, r, s = res[worst]
    print(f"\nGRADF64 {name} {mode} max_err/ref {e / max(r, 1e-30):.3g} ({worst}: err {e:.3g}, ref {r:.3g}) "
          f"max_err/gate {res[tightest][0] / res[tightest][1]:.3g} ({tightest}) "
          f"min_signal/gate {res[weakest][3] / res[weakest][1]:.3g} ({weakest})")


@pytest.mark.parametrize("name,mode", PARITY)
def test_step0_gradients_match_float64(name, mode):
    case = G.CASES[name]
    assert not G.power_violations(name, mode), "a gate too loose to see a lost row tile"
    res, g, bad_tb = G.compare(name, mode)
    _report(name, mode, res)
    for k, v in g.items():
        assert torch.isfinite(v).all(), k
    fails = {k: f"err {e:.3g} > gate {gt:.3g} (ref {r:.3g}, signal {s:.3g})" for k, (e, gt, r, s) in res.items() if not e <= gt}
    assert not fails, fails
    assert not bad_tb, bad_tb
    if case.regime == "log_std_clamp":   # components clamped in every row: no gradient reaches their log_std output at all
        key, off = G.log_std_bias(case)
        for j in (G.CLAMPED_HIGH, G.CLAMPED_LOW):
            assert float(g[key][off + j]) == 0.0, (key, j, float(g[key][off + j]))


@pytest.mark.parametrize("name", [c.name for c in G.SHAPE_CASES if c.engine == "mlp"])
def test_bf16_single_pass_gradients_are_close(name):
    """bf16 operands rounded once: not a parity mode, but its gradients must be finite and near float64."""
    r = G.reference(name)
    g, _ = G.engine_grads(name, "bf16")
    errs = {k: G.rel(g[k], r.g64[k]) for k in r.g64}
    for k, v in g.items():
        assert torch.isfinite(v).all(), k
    worst = max(errs, key=errs.get)
    print(f"\nGRADF64 {name} bf16 max_err {errs[worst]:.3g} ({worst})")
    assert errs[worst] <= G.BF16_LIMIT, (worst, errs[worst])
