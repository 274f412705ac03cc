"""Step-0 gradients of the MLP engine's tensor-core modes, bf16x3 and single-pass bf16, against the float64 oracle with
every GEMM operand rounded as the kernels round it (tests/gradcheck_rounded.py).

Against that yardstick the engine differs by its fp32 accumulation and fp32 elementwise arithmetic only (in bf16 also by
which way a value near a rounding midpoint images), so every gradient tensor must be as close to it as the float32
restatement (bf16: or the near-midpoint flips), up to the mode's (c, floor) pair, and every gate must
be able to see the loss of the batch's last 64-row tile.  Each test prints one `GRADF64` line: the largest
err_k / refR_k, the largest err_k / gateR_k and the smallest signal_k / gateR_k of the case."""
import pytest
import torch

import gradcheck64 as G
import gradcheck_rounded as GR

pytestmark = pytest.mark.gpu


def engine_grads(name, mode):
    rc = GR.CASES[name]
    if rc.kind == "std":
        import test_gpu_std_mlp as S
        return S.f64_engine_grads(rc.case.std_type, rc.case.batch, False, mode)
    if rc.kind == "v1":
        import test_gpu_v1_mlp as V
        return V.engine_grads(rc.case, mode)[0]
    return G.engine_grads(rc.case, mode)[0]


@pytest.mark.parametrize("mode", GR.GATED)
@pytest.mark.parametrize("name", list(GR.CASES))
def test_step0_gradients_match_the_rounded_float64_oracle(name, mode):
    assert not GR.power_violations(name, mode), "a gate too loose to see a lost row tile"
    r = GR.reference(name, mode)
    g = engine_grads(name, mode)
    res = {k: (G.rel(g[k], r.g64[k]), gt, r.ref[k], r.signal[k]) for k, gt in r.gate.items()}
    worst = max(res, key=lambda k: res[k][0] / max(res[k][2], 1e-30))
    tightest = max(res, key=lambda k: res[k][0] / res[k][1])
    weakest = min(res, key=lambda k: res[k][3] / res[k][1])
    e, _, rf, _ = res[worst]
    print(f"\nGRADF64 {name} {mode} rounded max_err/ref {e / max(rf, 1e-30):.3g} ({worst}) "
          f"max_err/gate {res[tightest][0] / res[tightest][1]:.3g} ({tightest}) "
          f"min_signal/gate {res[weakest][3] / res[weakest][1]:.3g} ({weakest})")
    for k in r.gate:
        assert torch.isfinite(g[k]).all(), k
    fails = {k: f"err {e:.3g} > gate {gt:.3g} (ref {rf:.3g}, signal {s:.3g})" for k, (e, gt, rf, s) in res.items() if not e <= gt}
    assert not fails, fails
