"""The frame replay ring (`ReplayBuffer(dsact_replay_frames=K)`) against the flat ring: device bytes, gather time per
call and the DSAC_V1 CNN update rate, on one GPU.  One JSON line per measurement; every line carries the card name, its
power limit and SM clocks, read in the same run.

- ring bytes: the frame ring filled through the drop-in ReplayBuffer with synthetic episodes (CarRacing-raw 3x96x96
  with K = 1, obs_t = obs2_{t-1}; stacked CarRacing 4x96x96 with K = 4, obs2 = obs shifted by one frame), computed from
  the planner and measured as the torch.cuda.memory_allocated delta; the flat ring measured at the largest of the
  requested capacities that fits (its bytes do not depend on what it holds) and computed at the requested one.
- gather: dsact_replay_sample with device-drawn indices, the two rings alternating in timed windows (median per call).
- update rate: replay_sample + step of DSAC_V1 with the CarRacing CNN networks at B = 256, alternating.

    python tools/bench_frame_replay.py [--rows 200000] [--windows 5] [--skip-bytes]
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
sys.path[:0] = [REPO, os.path.join(REPO, "dsac-v2_b200", "dropin")]

from dsac_v2_b200 import synth  # noqa: E402
from dsac_v2_b200.engine import Engine, make_config  # noqa: E402
from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config  # noqa: E402

DEV = torch.device("cuda", 0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, plim, sm, smmax = [x.strip() for x in q[0].split(",")] if q else ["?"] * 4
    return {"card": name, "power_limit": plim, "sm_clock": sm, "sm_clock_max": smmax}


def emit(**kw):
    print(json.dumps({**kw, **card()}), flush=True)


def vec_engine(obs_dim, act_dim, batch, hidden=(64,)):
    lim = torch.ones(act_dim)
    return Engine(make_config(obs_dim, act_dim, hidden, hidden, max_batch=batch, gemm_mode="fp32"), DEV, lim, -lim)


def fill(buf, shape, K, rows, seed=0):
    """Synthetic episodes of 1000 steps: K = 1, obs_t = obs2_{t-1}; K > 1, stacked frames (obs2 = obs shifted by one)."""
    g = np.random.default_rng(seed)
    fshape = (shape[0] // K,) + tuple(shape[1:])
    pool = g.random((64,) + fshape, dtype=np.float32)   # frame contents: a pool, perturbed per frame
    n = 0
    while n < rows:
        stack = [pool[g.integers(64)] + np.float32(n)] * K
        for t in range(min(1000, rows - n)):
            stack_next = stack[1:] + [pool[g.integers(64)] + np.float32(n + t + 1)]
            buf.store(np.concatenate(stack), {}, np.zeros(3, np.float32), 0.0, np.concatenate(stack_next), t == 999, 0.0, {})
            stack = stack_next
        n += 1000
    buf.flush()
    torch.cuda.synchronize()


def ring_bytes(rows):
    from training.replay_buffer import ReplayBuffer
    for label, shape, K in (("carracing_raw_k1", (3, 96, 96), 1), ("carracing_stacked_k4", (4, 96, 96), 4)):
        O = int(np.prod(shape))
        eng = vec_engine(O, 3, 8)
        base = torch.cuda.memory_allocated(DEV)
        buf = ReplayBuffer(obsv_dim=shape, action_dim=3, buffer_max_size=rows, dsact_replay_frames=K)
        t0 = time.perf_counter()
        buf.attach(eng)
        fill(buf, shape, K, rows)
        pl = buf.planner
        frame_alloc = torch.cuda.memory_allocated(DEV) - base
        held = int(buf.__get_RAM__() * 1e6)
        fill_s = time.perf_counter() - t0
        del buf
        eng.replay = None
        torch.cuda.empty_cache()
        flat_rows, flat_alloc = None, None
        for cap in (rows, rows // 2, rows // 4, rows // 8):
            try:
                base = torch.cuda.memory_allocated(DEV)
                eng.bind_replay(cap)
                flat_rows, flat_alloc = cap, torch.cuda.memory_allocated(DEV) - base
                eng.replay = None
                torch.cuda.empty_cache()
                break
            except torch.OutOfMemoryError:
                eng.replay = None
                torch.cuda.empty_cache()
        flat_row = 4 * (2 * O + 3 + 3)
        emit(what="ring_bytes", shape=label, rows=rows, K=K, frames_held=pl.held(), frame_capacity=pl.frame_capacity,
             frame_ring_held_GB=held / 1e9, frame_ring_allocated_GB=frame_alloc / 1e9, flat_ring_computed_GB=flat_row * rows / 1e9,
             flat_ring_measured_rows=flat_rows, flat_ring_allocated_GB=None if flat_alloc is None else flat_alloc / 1e9,
             flat_ring_allocated_scaled_GB=None if flat_alloc is None else flat_alloc * rows / flat_rows / 1e9, fill_s=fill_s)
        eng.close()
        del eng
        torch.cuda.empty_cache()


def bind_pair(make, cap):
    """Two engines: a flat ring and a K = 1 frame ring (row r: obs = frame r, obs2 = frame r + 1), random contents."""
    flat, fr = make(), make()
    for e in (flat, fr):
        e.seed(1234)
    flat.bind_replay(cap)
    for k in ("obs", "obs2", "act", "rew", "done", "logp"):
        flat.replay[k].uniform_()
    fr.bind_replay_frames(cap, cap + 1, 1)
    fr.replay["frames"].uniform_()
    for k in ("act", "rew", "done", "logp"):
        fr.replay[k].uniform_()
    ids = torch.arange(cap, dtype=torch.int32, device=DEV)[:, None]
    fr.replay["obs_frames"].copy_(ids)
    fr.replay["obs2_frames"].copy_(ids + 1)
    torch.cuda.synchronize()
    return flat, fr


def alternate(fns, n, windows):
    """Median seconds per call of each fn over `windows` alternating windows of n calls."""
    for f in fns:
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    times = [[] for _ in fns]
    for _ in range(windows):
        for i, f in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(n):
                f()
            b.record()
            b.synchronize()
            times[i].append(a.elapsed_time(b) / 1e3 / n)
    return [(float(np.median(t)), float((max(t) - min(t)) / np.median(t))) for t in times]


def gathers(windows):
    for label, O, A, B, cap in (("carracing_raw_b256", 3 * 96 * 96, 3, 256, 20000),
                                ("carracing_raw_b1024", 3 * 96 * 96, 3, 1024, 20000),
                                ("humanoid_b4096", 376, 17, 4096, 1000000)):
        flat, fr = bind_pair(lambda: vec_engine(O, A, B), cap)
        (tf, sf), (tr, sr) = alternate([lambda: flat.replay_sample(B, cap), lambda: fr.replay_sample(B, cap)], 200, windows)
        emit(what="gather", shape=label, batch=B, ring_rows=cap, flat_us=tf * 1e6, frame_us=tr * 1e6, flat_spread=sf,
             frame_spread=sr, frame_over_flat=tr / tf)
        for e in (flat, fr):
            e.close()
        del flat, fr
        torch.cuda.empty_cache()


def update_rate(windows):
    cfg = synth.CNN_CONFIGS["carracing"]
    t = synth.CONV_TYPES[cfg["conv_type"]]
    B, cap = 256, 20000
    c = make_cnn_config(cfg["obs_dim"], cfg["act_dim"], t["kernels"], t["channels"], t["strides"], t["heads"], max_batch=B,
                        algo="DSAC_V1")
    lim = torch.ones(cfg["act_dim"])
    w = synth.make_cnn_weights_v1(cfg)

    def make():
        e = CnnEngine(c, DEV, lim, -lim)
        e.load_weights(w)
        return e
    flat, fr = bind_pair(make, cap)
    it = [0, 0]

    def step(i, e):
        e.step(e.replay_sample(B, cap), it[i])
        it[i] += 1
    (tf, sf), (tr, sr) = alternate([lambda: step(0, flat), lambda: step(1, fr)], 20, windows)
    emit(what="update_rate", shape="v1_cnn_carracing_b256", batch=B, flat_steps_per_s=1 / tf, frame_steps_per_s=1 / tr,
         flat_spread=sf, frame_spread=sr, frame_over_flat=tf / tr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=200000)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--skip-bytes", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    gathers(a.windows)
    update_rate(a.windows)
    if not a.skip_bytes:
        ring_bytes(a.rows)


if __name__ == "__main__":
    main()
