"""DSAC_V1 with MLP approximators on the H100: the head-wise fp32 engine against the MLP engine in fp32 and in bf16x3.

    python tools/bench_v1.py [--steps K] [--warmup W] [--repeats R] [--shapes hopper,humanoid] [--arms heads,fp32,bf16x3]

Shapes: the reference's example (example_train/dsacv1_mlp_hopper_offserial.py: obs 11, act 3, 256x3 GELU critic and
policy, batch 256, TD_bound 10) and a Humanoid-shaped one (obs 376, act 17, 256x3 GELU, batch 4096).  Per arm, two
timings, each R windows of K steps after W warm-up steps:
  replay   the device-resident replay-fed step: dsact_replay_step on the MLP engine; replay_sample + step on the arena
           views on the head-wise engine, which has no fused replay step
  e2e      DSAC_V1.local_update on pinned host minibatches (what OffSerialTrainer calls), tb_info read back every step
One JSON line per arm and shape, with the card's name, power limit and SM clocks read in the same run.  Needs a GPU.
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

SHAPES = {
    "hopper": (synth.EXAMPLE_CONFIGS["hopper"], 256, {"TD_bound": 10.0, "gamma": 0.999}, 200_000),
    "humanoid": (synth.CONFIGS["humanoid"], 4096, {"TD_bound": 10.0}, 100_000),
}
ARMS = {"heads": None, "fp32": "fp32", "bf16x3": "bf16x3"}
V1_COLS = [0, 2, 6, 8, 9, 10, 11]   # the statistics that carry DSAC_V1's tb_info (include/dsact.h)


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"name": out[0], "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2]), "sm_mhz_idle": float(out[3])}
    except Exception as e:   # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "error": repr(e)}


def make_alg(cfg, B, over, gemm):
    import dsac_v1
    kw = synth.reference_kwargs(cfg, algorithm="DSAC_V1", replay_batch_size=B, **over)
    if gemm is not None:
        kw["dsact_gemm"] = gemm
    alg = dsac_v1.DSAC_V1(**kw)
    alg.networks.cuda()
    return alg


def timed(fn, steps, warmup, repeats):
    """Steps per second of `fn(it)` over `repeats` windows of `steps` calls, each ending in a device synchronise."""
    it = 0
    for _ in range(warmup):
        fn(it); it += 1
    torch.cuda.synchronize()
    rates = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        for _ in range(steps):
            fn(it); it += 1
        torch.cuda.synchronize()
        rates.append(steps / (time.perf_counter() - t0))
    return {"steps_per_s": statistics.median(rates), "min": min(rates), "max": max(rates), "windows": len(rates)}


def run(shape, arm, args, gpu):
    cfg, B, over, cap = SHAPES[shape]
    alg = make_alg(cfg, B, over, ARMS[arm])
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
        r = timed(replay, args.steps, args.warmup, args.repeats)
    r["clocks"] = clk.summary()
    assert np.all(np.isfinite([list(eng.read_stats().values())[c] for c in V1_COLS]))

    host = [{k: torch.from_numpy(v).pin_memory() for k, v in synth.make_batch(cfg, B, s).items()} for s in range(4)]
    with ClockSampler(0) as clk:
        e = timed(lambda it: alg.local_update(host[it % 4], it), args.steps, args.warmup, args.repeats)
    e["clocks"] = clk.summary()
    out = {"bench": "dsac_v1_mlp", "shape": shape, "obs_dim": O, "act_dim": A, "hidden": list(cfg["hidden"]), "batch": B,
           "arm": arm, "engine": "head-wise fp32" if arm == "heads" else f"MLP {arm}",
           "replay_step": r, "e2e_local_update_host": e, "gpu": gpu}
    print(json.dumps(out), flush=True)
    del alg, eng
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--shapes", default="hopper,humanoid")
    ap.add_argument("--arms", default="heads,fp32,bf16x3")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_v1 measures the H100 engines: no CUDA device")
    gpu = card()
    for shape in args.shapes.split(","):
        for arm in args.arms.split(","):
            run(shape, arm, args, gpu)


if __name__ == "__main__":
    main()
