"""Step-0 gradients of every feature-matrix case (tests/gradmatrix.py) against float64, on the engine the drop-in's route
builds for it, and the layer-chain kernel each bf16x3 case past one wave runs.

- Every gradient tensor within its gate (gradcheck64's (c, floor) of the case's arithmetic, power rule included), finite,
  and tb_info within gradcheck64's tolerance.  Each test prints one `GRADF64` line (test_gpu_grad_f64._report).
- Kernel selection: with DSACT_TC_DEBUG set, `launch_chain` prints one `[chain_debug] class C passes P grid G ... <kernel>`
  line per launch (class 1: forward, 2: dgrad; G: 64-row tiles).  A child process runs one gradient computation of each
  bf16x3 case past one wave: on a chain-lowered shape both classes must run the ping-pong kernel, every launch exactly
  when G exceeds the device's SMs; on the "wide" shape (per-layer GEMM groups) no chain launches at all."""
import os
import re
import subprocess
import sys

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if __name__ == "__main__":   # the kernel-selection child process
    sys.path[:0] = [REPO, os.path.join(REPO, "dsac-v2_b200", "dropin"), os.path.join(REPO, "tests")]

import gradmatrix as M  # noqa: E402
from test_gpu_grad_f64 import _report  # noqa: E402

pytestmark = pytest.mark.gpu

PAST = [n for n, c in M.CASES.items() if c.route == "mlp_bf16x3" and c.wave == "past"]
LINE = re.compile(r"^\[chain_debug\] class (\d+) passes (\d+) grid (\d+) span \S+ us (ping-pong|column split)$")


@pytest.mark.parametrize("name", list(M.CASES))
def test_step0_gradients_match_float64(name):
    mode = M.CASES[name].mode
    assert not M.power_violations(name), "a gate too loose to see a lost row tile"
    res, g, bad_tb = M.compare(name)
    _report(name, mode, res)
    for k, v in g.items():
        assert torch.isfinite(v).all(), k
    fails = {k: f"err {e:.3g} > gate {gt:.3g} (ref {r:.3g}, signal {s:.3g})" for k, (e, gt, r, s) in res.items() if not e <= gt}
    assert not fails, fails
    assert not bad_tb, bad_tb


def _child():
    """One gradient computation of every PAST case, each preceded by a `[case]` line on stderr."""
    torch.set_num_threads(4)
    for name in PAST:
        print(f"[case] {name}", file=sys.stderr, flush=True)
        M.engine_grads(name)
        torch.cuda.synchronize()
    print("[case] done", file=sys.stderr, flush=True)


def test_past_one_wave_cases_run_the_pingpong_kernel():
    assert PAST
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
    assert list(launches) == PAST + ["done"], list(launches)
    for name in PAST:
        ls = launches[name]
        if M.CASES[name].shape == "wide":
            assert not ls, (name, ls)
            continue
        for cls, passes, grid, kernel in ls:
            assert kernel == ("ping-pong" if grid > sms else "column split"), (name, cls, passes, grid, kernel, sms)
        for cls in (1, 2):
            assert any(c == cls and k == "ping-pong" for c, _, _, k in ls), (name, cls, ls)


if __name__ == "__main__":
    if sys.argv[1] == "select":
        _child()
