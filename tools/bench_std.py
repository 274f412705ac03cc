"""DSAC-T with the policy's "mlp_separated" / "parameter" std types on the H100: the head-wise fp32 engine against the
MLP engine in fp32, bf16x3 and bf16.

    python tools/bench_std.py [--seconds S] [--warmup W] [--repeats R] [--shapes ...] [--arms heads,fp32,bf16x3,bf16]
                              [--std mlp_separated,parameter]

Shapes: Humanoid-shaped (obs 376, act 17, 256x3 GELU) at batch 4096 and 256, and the Hopper example shape (obs 11, act 3,
256x3 GELU) at batch 256.  Per std type, shape and arm, two timings, each the median of R windows of at least S seconds
after W warm-up steps (every graph the window replays is captured in the warm-up):
  replay   the device-resident replay-fed step: dsact_replay_step on the MLP engine; replay_sample + step on the arena
           views on the head-wise engine, which has no fused replay step
  e2e      DSAC_V2.local_update on pinned host minibatches (what OffSerialTrainer calls), tb_info read back every step
One JSON line each, with the card's name, power limit and SM clocks read in the same run.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [REPO, os.path.join(REPO, "dsac-v2_b200", "dropin")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from dsac_v2_b200 import synth  # noqa: E402

SHAPES = {   # (configuration, batch, replay ring rows)
    "humanoid_b4096": (synth.CONFIGS["humanoid"], 4096, 100_000),
    "humanoid_b256": (synth.CONFIGS["humanoid"], 256, 100_000),
    "hopper_b256": (synth.EXAMPLE_CONFIGS["hopper"], 256, 200_000),
}
ARMS = {"heads": None, "fp32": "fp32", "bf16x3": "bf16x3", "bf16": "bf16"}


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"name": out[0], "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2]), "sm_mhz_idle": float(out[3])}
    except Exception as e:   # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "error": repr(e)}


def make_alg(cfg, B, std_type, gemm):
    import dsac_v2
    kw = synth.reference_kwargs(cfg, policy_std_type=std_type, replay_batch_size=B)
    if gemm is not None:
        kw["dsact_gemm"] = gemm
    alg = dsac_v2.DSAC_V2(**kw)
    alg.networks.cuda()
    return alg


def timed(fn, seconds, warmup, repeats):
    """Steps per second of `fn(it)` over `repeats` windows of at least `seconds` each, every window ending in a device
    synchronise; the window's step count comes from a timed probe after the warm-up."""
    it = 0
    for _ in range(warmup):
        fn(it); it += 1
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(50):
        fn(it); it += 1
    torch.cuda.synchronize()
    steps = max(50, int(1.2 * seconds * 50 / (time.perf_counter() - t0)))
    rates = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        for _ in range(steps):
            fn(it); it += 1
        torch.cuda.synchronize()
        rates.append(steps / (time.perf_counter() - t0))
    return {"steps_per_s": statistics.median(rates), "min": min(rates), "max": max(rates), "windows": len(rates),
            "steps_per_window": steps}


def run(std_type, shape, arm, args, gpu):
    cfg, B, cap = SHAPES[shape]
    alg = make_alg(cfg, B, std_type, ARMS[arm])
    eng = alg.networks.engine(B)
    eng.seed(1234)
    g = np.random.default_rng(0)
    O, A, lim = cfg["obs_dim"], cfg["act_dim"], cfg["act_lim"]
    eng.bind_replay(cap)
    chunk = 20_000
    for p in range(0, cap, chunk):
        n = min(chunk, cap - p)
        rows = {"obs": g.standard_normal((n, O)), "obs2": g.standard_normal((n, O)), "act": g.uniform(-lim, lim, (n, A)),
                "rew": g.standard_normal(n), "done": (g.random(n) < 0.01), "logp": np.zeros(n)}
        eng.replay_add({k: torch.from_numpy(np.asarray(v, dtype=np.float32)).cuda() for k, v in rows.items()}, n, p)
    torch.cuda.synchronize()

    if arm == "heads":
        def replay(it):
            eng.step(eng.replay_sample(B, cap), it)
    else:
        def replay(it):
            eng.replay_step(B, cap, it)
    with ClockSampler(0) as clk:
        r = timed(replay, args.seconds, args.warmup, args.repeats)
    r["clocks"] = clk.summary()
    assert np.all(np.isfinite(list(eng.read_stats().values())[:14]))

    host = [{k: torch.from_numpy(v).pin_memory() for k, v in synth.make_batch(cfg, B, s).items()} for s in range(4)]
    with ClockSampler(0) as clk:
        e = timed(lambda it: alg.local_update(host[it % 4], it), args.seconds, args.warmup, args.repeats)
    e["clocks"] = clk.summary()
    out = {"bench": "dsact_std_mlp", "std_type": std_type, "shape": shape, "obs_dim": O, "act_dim": A, "hidden": list(cfg["hidden"]), "batch": B,
           "arm": arm, "engine": "head-wise fp32" if arm == "heads" else f"MLP {arm}",
           "replay_step": r, "e2e_local_update_host": e, "gpu": gpu}
    print(json.dumps(out), flush=True)
    del alg, eng
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--arms", default=",".join(ARMS))
    ap.add_argument("--std", default="mlp_separated,parameter")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_std measures the H100 engines: no CUDA device")
    gpu = card()
    for std_type in args.std.split(","):
        for shape in args.shapes.split(","):
            for arm in args.arms.split(","):
                run(std_type, shape, arm, args, gpu)


if __name__ == "__main__":
    main()
