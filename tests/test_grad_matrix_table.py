"""CPU guard of the feature-matrix gradient table (tests/gradmatrix.py, run on the GPU by tests/test_gpu_grad_matrix.py):
every case lands where it says through the drop-in's route, the table covers what the full product of the axes allows,
every gate can see a lost row tile, and every emulated wiring fault of a new combination moves some gradient past its
gate on every case where the fault's feature is active.  No GPU."""
import pytest

import gradcheck64 as G
import gradmatrix as M


@pytest.mark.parametrize("name", list(M.CASES))
def test_case_lands_on_its_engine(name):
    c = M.CASES[name]
    r = M.routed(c)
    assert r is not None, f"route() refuses {name} or puts it on another engine"
    assert r.engine == M.ENGINE[c.route] and r.out_acts == (c.out_q, c.out_pi)
    cfg = r.config(c.batch)
    assert cfg.max_batch == c.batch
    if r.engine == "mlp":
        assert r.cfg_args["gemm_mode"] == c.route[len("mlp_"):] and r.cfg_args["use_graph"] is False
        assert r.cfg_args["policy_std"] == c.std and (r.v1 is not None) == (c.algo == "DSAC_V1")
    assert r.cfg_args["act_dist"] == c.dist


def test_table_covers_every_allowed_pair_and_the_pingpong_values():
    valid = [c for c in M.product() if M.routed(c) is not None]
    need = M.required(valid)
    got = set().union(*(M.items(c) for c in M.CASES.values()))
    print(f"\n{len(M.product())} assignments, {len(valid)} valid, {len(need)} required combinations "
          f"({sum(i[0] == 'pingpong' for i in need)} with bf16x3 past one wave), {len(M.CASES)} cases")
    assert len(M.CASES) == len(M.TABLE), "two cases of one name"
    assert not need - got, sorted(need - got)
    # every value of every other axis reaches bf16x3 past one wave; all but the shapes on a chain-lowered shape
    for axis, values in M.AXES.items():
        if axis not in ("route", "wave"):
            allowed = {i[2] for i in need if i[:2] == ("pingpong", axis)}
            assert allowed == set(values) - ({"small_t1"} if axis == "shape" else set()), (axis, allowed)


@pytest.mark.parametrize("name", list(M.CASES))
def test_gates_can_see_a_lost_row_tile(name):
    r = M.reference(name)
    assert set(r.g64) == set(r.ref) == set(r.signal) and r.g64
    bad = M.power_violations(name)
    assert not bad, {k: f"gate {g:.3g} > signal {s:.3g} / {G.POWER}" for k, (g, s) in bad.items()}


@pytest.mark.parametrize("name", list(M.WIDENED))
def test_widened_gates_are_the_operand_rounding(name):
    """A widened bf16x3 gate: the split-bf16 restatement moves the tensor past its common gate by the recorded amount,
    and stays inside the widened one."""
    assert M.CASES[name].mode == "bf16x3"
    move = M.widening(name)
    for key, (factor, recorded) in M.WIDENED[name].items():
        print(f"\nWIDENED {name} {key}: restatement {move[key]:.3g} common gates (recorded {recorded}), factor {factor}")
        assert 1.0 < move[key] <= factor, (key, move[key], factor)
        assert abs(move[key] - recorded) <= 0.02 * recorded, (key, move[key], recorded)


FAULT_CASES = [(f, n) for f, (_, active) in M.FAULTS.items() for n, c in M.CASES.items() if active(c)]


def test_every_fault_is_active_somewhere():
    assert {f for f, _ in FAULT_CASES} == set(M.FAULTS)


@pytest.mark.parametrize("fault,name", FAULT_CASES)
def test_emulated_fault_exceeds_a_gate(fault, name):
    factor, key = M.fault_factor(name, fault)
    print(f"\nFAULT {fault} {name}: {factor:.3g} gates ({key})")
    assert factor > 1.0, (fault, name, factor, key)
