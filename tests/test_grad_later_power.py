"""CPU guard of the later-state update gates (tests/gradcheck_later.py, run on the GPU by tests/test_gpu_grad_later.py):
with the oracle alone, every gate of every synthetic later state must see the loss of the batch's last 64-row tile, every
emulated wiring fault must move some compared gradient or update element by POWER gates wherever it applies, and the
state must survive its round trip through the oracle."""
import pytest
import torch

import gradcheck_later as L

PARITIES = ("even", "odd")


@pytest.mark.parametrize("parity", PARITIES)
@pytest.mark.parametrize("name", list(L.CASES))
def test_later_gates_can_see_a_lost_row_tile(name, parity):
    case = L.CASES[name]
    r = L.synthetic_reference(name, parity)
    assert set(r.g64) == set(r.ref) == set(r.signal) and r.g64
    for mode in case.modes:
        bad = L.power_violations(case, r, mode)
        assert not bad, {k: f"gate {g:.3g} > signal {s:.3g} / {L.POWER}" for k, (g, s) in bad.items()}


@pytest.mark.parametrize("fault", list(L.FAULTS))
def test_every_fault_clears_the_gates(fault):
    applies = L.FAULTS[fault][1]
    margins = {(name, p): L.fault_margin(name, p, fault) for name, c in L.CASES.items() for p in PARITIES if applies(c, p)}
    assert margins
    (name, p), (x, where) = min(margins.items(), key=lambda kv: kv[1][0])
    print(f"\nGRADLATER_FAULT {fault} smallest margin {x:.3g} gates ({name} {p}, {where}) over {len(margins)} cases")
    weak = {k: f"{v[0]:.3g} ({v[1]})" for k, v in margins.items() if not v[0] >= L.POWER}
    assert not weak, weak


@pytest.mark.parametrize("name", ["ragged_b1000", "v1_asym_fp32_b1000", "parameter_ragged_fp32_b1000",
                                  "cnn_carracing_b256", "v1_pendulum_b4096"])
def test_state_round_trip_through_the_oracle(name):
    """load_state, then the oracle's state_dict and moments give back the state bit for bit (float32 oracle), and its
    counters, log_alpha and mean_std are the state's."""
    case = L.CASES[name]
    s = L.synthetic_state(name, "even")
    orc = case.oracle(torch.float32, s)
    sd = orc.state_dict()
    assert set(sd) == set(s.params)
    for k, v in s.params.items():
        assert torch.equal(sd[k].reshape(v.shape), v), k
    m, v = orc.moments()
    for got, want in ((m, s.m), (v, s.v)):
        assert set(got) == set(want)
        for k in want:
            assert torch.equal(got[k].reshape(want[k].shape), want[k]), k
    for net in orc.NETS:
        assert orc.steps[net] == (s.tp if net == "policy" else s.tq)
    assert orc.steps["log_alpha"] == s.tp
    if case.v1:
        assert orc.mean_std == [None, None]
    else:
        assert [float(x) for x in orc.mean_std] == list(s.mean_std)
    # the state is a later one: targets off the online networks, moments and counters non-zero, mean_std carried
    on = L._online(s.params)
    assert all(not torch.equal(s.params[L._target_key(k)], x) for k, x in on.items())
    assert all(bool((x > 0).all()) for x in s.v.values())
    assert s.tq > 0 and s.tp > 0 and float(s.params["log_alpha"]) != 1.0
    assert case.v1 or min(s.mean_std) > 0


def test_update_restatement_moves_what_each_parity_moves():
    """apply_ref from a later state: odd k leaves the policy, log_alpha and every target as they were, even k moves them
    all; both advance the critics."""
    name = "ragged_b1000"
    case = L.CASES[name]
    lay = L._Layout(case)
    for parity in PARITIES:
        s = L.synthetic_state(name, parity)
        k = L.SYNTH[parity][0]
        g = {key: x.float() for key, x in L.synthetic_reference(name, parity).g64.items()}
        out = L.expected_update(case, lay, s, g, k)
        w0, t0 = L.flat(lay, s.params), L.flat(lay, s.params, True)
        nq2 = 2 * int(lay.layout.n_q)
        assert not torch.equal(out["w"][0][:nq2], w0[:nq2])
        odd = k % 2 == 1
        assert torch.equal(out["w"][0][nq2:], w0[nq2:]) == odd
        assert torch.equal(out["t"][0], t0) == odd
