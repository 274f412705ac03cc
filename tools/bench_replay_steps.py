"""n replay-fed updates per call (Engine.replay_steps) against n replay_step calls, alternating in one process.

One JSON line per shape, mode and n: median updates/s over timed windows of each path, their spread (max - min over
the windows, relative to the median), the gain, and the largest relative L2 difference between the two paths' outputs
(params, targets, Adam moments, per-update statistics) from one start state.  Every line carries the card name, its
power limit and SM clocks, read in the same run.  --trace writes a torch.profiler kernel timeline of one captured 2-update
call under --out.

    python tools/bench_replay_steps.py [--windows 5] [--window-s 0.5] [--ns 1,2,4,8,16,32] [--trace] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))

from dsac_v2_b200 import synth  # noqa: E402

# (label, algorithm, config, batch, modes)
SHAPES = [("humanoid_b4096", "t", synth.CONFIGS["humanoid"], 4096, ("bf16x3", "bf16")),
          ("humanoid_b256", "t", synth.CONFIGS["humanoid"], 256, ("bf16x3",)),
          ("hopper_b256", "t", synth.EXAMPLE_CONFIGS["hopper"], 256, ("bf16x3", "fp32")),
          ("v1_hopper_b256", "v1", synth.EXAMPLE_CONFIGS["hopper"], 256, ("bf16x3",))]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, plim, sm, smmax = [x.strip() for x in q[0].split(",")] if q else ["?"] * 4
    return {"card": name, "power_limit": plim, "sm_clock": sm, "sm_clock_max": smmax}


def engine(algo, cfg, B, mode):
    from test_gpu_parity import make_engine
    import v1_mlp_common as v1c
    e = v1c.make_engine(cfg, B, dict(synth.HYPER), gemm=mode) if algo == "v1" else make_engine(cfg, B, gemm_mode=mode)
    e.seed(1234)
    cap = 4 * B + 100
    g = np.random.default_rng(1)
    O, A = cfg["obs_dim"], cfg["act_dim"]
    ring = {"obs": g.standard_normal((cap, O)), "obs2": g.standard_normal((cap, O)), "act": g.uniform(-1, 1, (cap, A)),
            "rew": g.standard_normal(cap), "done": (g.random(cap) < 0.05) * 1.0, "logp": g.standard_normal(cap)}
    e.bind_replay(cap)
    e.replay_add({k: torch.from_numpy(v.astype(np.float32)).cuda() for k, v in ring.items()}, cap, 0)
    return e, cap - 50


def rate(run, per_call, window_s):
    """updates/s of `run` (one call = per_call updates) over one window of >= window_s seconds."""
    torch.cuda.synchronize()
    t0, calls = time.perf_counter(), 0
    while True:
        for _ in range(8):
            run()
        calls += 8
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if dt >= window_s:
            return calls * per_call / dt


def out_diff(algo, cfg, B, mode, n):
    """Largest relative L2 difference of n single calls vs one n-call from one start state."""
    a, size = engine(algo, cfg, B, mode)
    b, _ = engine(algo, cfg, B, mode)
    for e in (a, b):
        e.replay_step(B, size, 0)
    rows = []
    for k in range(n):
        a.replay_step(B, size, 1 + k)
        out = a.read_stats_async(B)
        torch.cuda.synchronize()
        rows.append(out.clone())
    got = b.replay_steps(n, B, size, 1)
    torch.cuda.synchronize()
    rl2 = lambda x, y: float((x.double() - y.double()).norm() / max(float(y.double().norm()), 1e-30))  # noqa: E731
    d = max(rl2(getattr(b, k), getattr(a, k)) for k in ("params", "targets", "adam_m", "adam_v"))
    d = max(d, rl2(got.cpu()[:, :14], torch.stack(rows)[:, :14]))
    a.close(); b.close()
    return d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--window-s", type=float, default=0.5)
    ap.add_argument("--ns", default="1,2,4,8,16,32")
    ap.add_argument("--shapes", default=",".join(s[0] for s in SHAPES))
    ap.add_argument("--trace", action="store_true")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "bench_replay_steps"),
                    help="directory of the --trace timeline (default: a directory under the system's temporary directory)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    ns = [int(x) for x in args.ns.split(",")]
    want = set(args.shapes.split(","))
    if args.trace:
        from torch.profiler import ProfilerActivity, profile
        e, size = engine("t", synth.CONFIGS["humanoid"], 256, "bf16x3")
        for _ in range(3):
            e.replay_steps(2, 256, size, 0)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as p:
            e.replay_steps(2, 256, size, 0)
            torch.cuda.synchronize()
        os.makedirs(args.out, exist_ok=True)
        path = os.path.join(args.out, "replay_steps_trace.json")
        p.export_chrome_trace(path)
        ev = sorted([x for x in p.events() if x.device_type.name == "CUDA"], key=lambda x: x.time_range.start)
        gathers = [x for x in ev if "gather_kernel" in x.name]
        applies = [x for x in ev if "apply_kernel" in x.name]
        print(json.dumps({"trace": path, "gather_starts_us": [g.time_range.start for g in gathers],
                          "apply_ends_us": [a.time_range.end for a in applies],
                          "second_gather_before_first_apply_ends": bool(len(gathers) > 1 and applies and
                                                                        gathers[1].time_range.start < applies[0].time_range.end)}))
        e.close()
        return
    for label, algo, cfg, B, modes in SHAPES:
        if label not in want:
            continue
        for mode in modes:
            e, size = engine(algo, cfg, B, mode)
            it = [0]

            def singles(n):
                def run():
                    for _ in range(n):
                        e.replay_step(B, size, it[0]); it[0] += 1
                return run

            def multi(n):
                def run():
                    e.replay_steps(n, B, size, it[0], stats=False); it[0] += n
                return run
            for n in ns:   # warm-up: every graph of the timed windows
                singles(n)(); multi(n)()
            info = card()
            for n in ns:
                rs, rm = [], []
                for _ in range(args.windows):
                    rs.append(rate(singles(n), n, args.window_s))
                    rm.append(rate(multi(n), n, args.window_s))
                ms, mm = float(np.median(rs)), float(np.median(rm))
                print(json.dumps({"shape": label, "mode": mode, "n": n, "single_updates_per_s": round(ms, 1),
                                  "multi_updates_per_s": round(mm, 1), "gain": round(mm / ms - 1, 4),
                                  "single_spread": round((max(rs) - min(rs)) / ms, 4),
                                  "multi_spread": round((max(rm) - min(rm)) / mm, 4),
                                  "out_max_rel_l2": out_diff(algo, cfg, B, mode, n), **info}), flush=True)
            e.close()


if __name__ == "__main__":
    main()
