"""Replay-fed update rate with linear, tanh and gelu output activations, alternating in one process.

The output activations run in the step's row kernels only (sampling, losses, policy gradient), a small part of a step,
so the question is whether a non-linear output moves the update rate beyond the run-to-run spread.  Shapes: the
benchmarked Humanoid step (B = 4096, bf16x3) and the reference's Hopper example (B = 256, bf16x3).  One JSON line per
shape and activation: the median updates/s over --windows timed windows (each of >= --window-s seconds of captured
replay_step calls), the spread (max - min over the windows, relative to the median) and the change against linear.
Every line carries the card name, its power limit and SM clocks, read in the same run.

    python tools/bench_outact.py [--windows 7] [--window-s 0.5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from dsac_v2_b200 import synth  # noqa: E402

SHAPES = [("humanoid_b4096", synth.CONFIGS["humanoid"], 4096), ("hopper_b256", synth.EXAMPLE_CONFIGS["hopper"], 256)]
ACTS = ("linear", "tanh", "gelu")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, plim, sm, smmax = [x.strip() for x in q[0].split(",")] if q else ["?"] * 4
    return {"card": name, "power_limit": plim, "sm_clock": sm, "sm_clock_max": smmax}


def engine(cfg, B, act):
    from dsac_v2_b200.engine import Engine, make_config
    h = synth.HYPER
    act_q, act_pi = synth.activations(cfg)
    c = make_config(cfg["obs_dim"], cfg["act_dim"], *synth.hidden_sizes(cfg), max_batch=B, act_q=act_q, act_pi=act_pi,
                    gemm_mode="bf16x3", gamma=h["gamma"], tau=h["tau"], delay_update=h["delay_update"], lr_q=h["value_learning_rate"],
                    lr_pi=h["policy_learning_rate"], lr_alpha=h["alpha_learning_rate"])
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    e = Engine(c, torch.device("cuda", 0), lim, -lim, output_activations=(act, act))
    e.load_weights(synth.make_weights(cfg))
    e.seed(1234)
    cap = 4 * B + 100
    g = np.random.default_rng(1)
    O, A = cfg["obs_dim"], cfg["act_dim"]
    ring = {"obs": g.standard_normal((cap, O)), "obs2": g.standard_normal((cap, O)), "act": g.uniform(-1, 1, (cap, A)),
            "rew": g.standard_normal(cap), "done": (g.random(cap) < 0.05) * 1.0, "logp": g.standard_normal(cap)}
    e.bind_replay(cap)
    e.replay_add({k: torch.from_numpy(v.astype(np.float32)).cuda() for k, v in ring.items()}, cap, 0)
    return e, cap - 50


def rate(e, B, size, it, window_s):
    """updates/s of replay_step calls over one window of >= window_s seconds"""
    torch.cuda.synchronize()
    t0, n = time.perf_counter(), 0
    while True:
        for _ in range(16):
            e.replay_step(B, size, it[0])
            it[0] += 1
        n += 16
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if dt >= window_s:
            return n / dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--window-s", type=float, default=0.5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    for label, cfg, B in SHAPES:
        engs = {a: engine(cfg, B, a) for a in ACTS}
        its = {a: [0] for a in ACTS}
        for a, (e, size) in engs.items():   # warm-up: capture every graph the windows replay
            for _ in range(8):
                e.replay_step(B, size, its[a][0])
                its[a][0] += 1
        rates = {a: [] for a in ACTS}
        for _ in range(args.windows):   # alternating windows: the same host and clock conditions for every activation
            for a, (e, size) in engs.items():
                rates[a].append(rate(e, B, size, its[a], args.window_s))
        info = card()
        base = float(np.median(rates["linear"]))
        for a in ACTS:
            med = float(np.median(rates[a]))
            print(json.dumps({"shape": label, "mode": "bf16x3", "output_activation": a, "updates_per_s": round(med, 1),
                              "step_ms": round(1e3 / med, 4), "spread": round((max(rates[a]) - min(rates[a])) / med, 4),
                              "vs_linear": round(med / base - 1, 4), **info}), flush=True)
            engs[a][0].close()


if __name__ == "__main__":
    main()
