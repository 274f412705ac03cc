"""Whole steps whose layer-chain launches run on the ping-pong kernel (tc_pingpong_kernel: launches of more than one wave
of 64-row tiles), against the float64 oracle of tests/gradcheck64.py, and the kernel each of those launches selects.

- Policy gradients at B = 8500: the policy's dgrad chain is one pass, so only from B = 8449 on (133 tiles) does it run on
  the ping-pong kernel.  At that batch, losing one 64-row tile moves some critic-bias and log_alpha gradients by less than
  the bf16x3 floor, so the power rule cannot hold for every key: the test compares the `policy.*` gradients, with
  gradcheck64's gates, and asserts the power rule on exactly those keys.
- Kernel selection: with DSACT_TC_DEBUG set, `launch_chain` prints one `[chain_debug] class C passes P grid G ... <kernel>`
  line per launch (class 1: forward, 2: dgrad; G: 64-row tiles).  A child process runs one gradient computation of every
  step case that is meant to reach the ping-pong kernel, and each launch must have run the ping-pong kernel exactly when
  G exceeds the device's SMs (the column split keeps one resident CTA per SM)."""
import os
import re
import subprocess
import sys

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if __name__ == "__main__":   # the kernel-selection child process
    sys.path[:0] = [REPO, os.path.join(REPO, "dsac-v2_b200", "dropin")]

import gradcheck64 as G  # noqa: E402

pytestmark = pytest.mark.gpu

MODE = "bf16x3"
POLICY_CASES = [G.Case(f"{name}_b8500", "mlp", name, 8500) for name in ("asym", "deep_pi", "ragged")]
# the step cases of the suite that reach the ping-pong kernel: (kind, name)
STEP_CASES = ([("dsact", f"{n}_b2200") for n in ("asym", "deep_pi", "ragged")] +
              [("std", f"{s}_b2200") for s in ("mlp_separated", "parameter")] +
              [("v1", "v1mlp_asym_b4300")] +
              [("dsact", c.name) for c in POLICY_CASES])
LINE = re.compile(r"^\[chain_debug\] class (\d+) passes (\d+) grid (\d+) span \S+ us (ping-pong|column split)$")


@pytest.fixture(scope="module")
def policy_cases():
    """POLICY_CASES registered in gradcheck64's table while this module runs (they are not in its power-rule guard)."""
    G.CASES.update({c.name: c for c in POLICY_CASES})
    yield
    for c in POLICY_CASES:
        G.CASES.pop(c.name, None)


@pytest.mark.parametrize("name", [c.name for c in POLICY_CASES])
def test_policy_gradients_at_a_single_pass_pingpong_batch(policy_cases, name):
    gates = {k: g for k, g in G.gates(name, MODE).items() if k.startswith("policy.")}
    assert gates
    r = G.reference(name)
    weak = {k: (g, r.signal[k]) for k, g in gates.items() if not g <= r.signal[k] / G.POWER}
    assert not weak, f"gates that would not notice a lost row tile: {weak}"
    g, _ = G.engine_grads(name, MODE)
    res = {k: (G.rel(g[k], r.g64[k]), gates[k], r.ref[k], r.signal[k]) for k in gates}
    tightest = max(res, key=lambda k: res[k][0] / res[k][1])
    weakest = min(res, key=lambda k: res[k][3] / res[k][1])
    print(f"\nGRADF64 {name} {MODE} policy.* max_err/gate {res[tightest][0] / res[tightest][1]:.3g} ({tightest}) "
          f"min_signal/gate {res[weakest][3] / res[weakest][1]:.3g} ({weakest})")
    for k in gates:
        assert torch.isfinite(g[k]).all(), k
    fails = {k: f"err {e:.3g} > gate {gt:.3g} (ref {rf:.3g}, signal {s:.3g})" for k, (e, gt, rf, s) in res.items() if not e <= gt}
    assert not fails, fails


def _child():
    """One bf16x3 gradient computation of every STEP_CASES entry (no graphs), each preceded by a `[case]` line on stderr."""
    torch.set_num_threads(4)
    import test_gpu_std_mlp as S
    import test_gpu_v1_mlp as V
    G.CASES.update({c.name: c for c in POLICY_CASES})
    for kind, name in STEP_CASES:
        print(f"[case] {name}", file=sys.stderr, flush=True)
        if kind == "dsact":
            G.engine_grads(name, MODE)
        elif kind == "std":
            std_type, batch = name.rsplit("_b", 1)
            S.f64_engine_grads(std_type, int(batch), False, MODE)
        else:
            V.engine_grads(V.F64_CASES[name], MODE)
        torch.cuda.synchronize()
    print("[case] done", file=sys.stderr, flush=True)


def test_step_cases_run_their_chains_on_the_pingpong_kernel():
    env = dict(os.environ, DSACT_TC_DEBUG="1")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), "select"], env=env, cwd=REPO, capture_output=True,
                       text=True, timeout=1800)
    assert p.returncode == 0, f"child exited with {p.returncode}:\n{p.stdout[-4000:]}\n{p.stderr[-6000:]}"
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    launches, case = {}, None
    for line in p.stderr.splitlines():
        if line.startswith("[case] "):
            case = line[len("[case] "):]
            launches[case] = []
        elif line.startswith("[chain_debug]"):
            print(case, line)
            m = LINE.match(line)
            assert m and case is not None, line
            launches[case].append((int(m.group(1)), int(m.group(2)), int(m.group(3)), m.group(4)))
    assert list(launches) == [n for _, n in STEP_CASES] + ["done"], list(launches)
    for name in launches:
        if name == "done":
            continue
        ls = launches[name]
        for cls, passes, grid, kernel in ls:
            want = "ping-pong" if grid > sms else "column split"
            assert kernel == want, (name, cls, passes, grid, kernel, sms)
        for cls in (1, 2):
            assert any(c == cls and k == "ping-pong" for c, _, _, k in ls), (name, cls, ls)
        if name.endswith("_b8500"):
            assert all(k == "ping-pong" for *_, k in ls), (name, ls)


if __name__ == "__main__":
    if sys.argv[1] == "select":
        _child()
