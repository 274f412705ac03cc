"""The single-call update (`step`, and `replay_step` as the benchmark runs it) of both engines against float64 from states
that are not step 0 (tests/gradcheck_later.py): synthetic later states at an even and an odd iteration, and the engine's
own state after 1 and 6 replay-fed updates with its graphs captured.

At the gated update: the gradients the step leaves in `grads` within gradcheck64's gates of float64 (every gate able to
see a lost row tile), parameters, targets, moments, the committed mean_std and the counters within step_ref's gates of
the restated Adam / Polyak fed the step's own gradients, and tb_info within gradcheck64's rule.  Each test prints one
`GRADLATER` line: the largest err_k / gate_k and the smallest signal_k / gate_k of the case."""
import pytest
import torch

import gradcheck64 as G
import gradcheck_later as L

pytestmark = pytest.mark.gpu

SYNTHETIC = [(c.name, m, p) for c in L.CASES.values() for m in c.modes for p in ("even", "odd")]
TRAJECTORIES = [(c.name, m, n) for c in L.CASES.values() if c.trajectory for m in c.modes for n in L.TRAJ_N]


def _check(case, mode, label, r, pre, post, g, tb, eng, k):
    gate = L.gates(case, r, mode)
    res = {key: (G.rel(g[key], r.g64[key]), gate[key], r.signal[key]) for key in r.g64}
    tight = max(res, key=lambda key: res[key][0] / res[key][1])
    weak = min(res, key=lambda key: res[key][2] / res[key][1])
    print(f"\nGRADLATER {case.name} {mode} {label} max_err/gate {res[tight][0] / res[tight][1]:.3g} ({tight}) "
          f"min_signal/gate {res[weak][2] / res[weak][1]:.3g} ({weak})")
    for key, x in g.items():
        assert torch.isfinite(x).all(), key
    assert not L.power_violations(case, r, mode), "a gate too loose to see a lost row tile"
    fails = {key: f"err {e:.3g} > gate {gt:.3g} (signal {s:.3g})" for key, (e, gt, s) in res.items() if not e <= gt}
    assert not fails, fails
    bad = L.update_deviations(case, eng, pre, post, g, k)
    assert not bad, bad
    bad_ms = L.mean_std_deviation(case, eng, pre, case.batch)
    assert not bad_ms, bad_ms
    assert int(L._ints(eng)[11]) == k + 1   # the iteration the next apply will use
    bad_tb = G.tb_deviations(r, tb, mode)
    assert not bad_tb, bad_tb


@pytest.mark.parametrize("name,mode,parity", SYNTHETIC)
def test_update_from_a_synthetic_later_state(name, mode, parity):
    case = L.CASES[name]
    r = L.synthetic_reference(name, parity)
    k = L.SYNTH[parity][0]
    pre, post, g, tb, eng = L.run_synthetic(case, mode, parity)
    try:
        _check(case, mode, f"{parity} k={k}", r, pre, post, g, tb, eng, k)
    finally:
        eng.close()


def _trajectory(name, mode, n):
    case = L.CASES[name]
    pre, b, nz, post, g, tb, eng = L.trajectory(case, mode, n)
    return pre, post, g, tb, eng, L.reference(case, pre, b, nz)


@pytest.mark.parametrize("name,mode,n", TRAJECTORIES)
def test_update_after_engine_updates(name, mode, n):
    """Update n + 1 (iteration n) after n graph-replayed updates of the engine itself, from the state they left."""
    case = L.CASES[name]
    pre, post, g, tb, eng, r = _trajectory(name, mode, n)
    try:
        assert pre.tq == n and pre.tp == (n + 1) // 2
        assert case.v1 or min(pre.mean_std) > 0
        _check(case, mode, f"after {n} updates", r, pre, post, g, tb, eng, n)
    finally:
        eng.close()
