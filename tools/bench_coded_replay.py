"""The coded frame ring (`ReplayBuffer(dsact_replay_frames=K, dsact_replay_codes=True)`) against the fp32 frame ring and
the flat ring on CarRacing-raw observations (3x96x96, rgb / 255: 256 distinct values): device bytes, gather time per
call and the CNN replay-fed update rate, on one GPU.  One JSON line per measurement; every line carries the card name,
its power limit and SM clocks, read in the same run.

- ring bytes: each ring bound at --rows rows (K = 1) through the drop-in ReplayBuffer and fed --fill rows of 1000-step
  episodes (obs_t = obs2_{t-1}), measured as the torch.cuda.memory_allocated delta.  With such episodes the frame store
  never grows past its initial capacity, so the allocation at --rows rows is the ring's footprint at that size.
- gather: dsact_replay_sample with device-drawn indices at B = 256 and 1024 from rings of 20 000 rows holding the same
  observations (checked equal once), the three rings alternating in timed windows (median per call).
- update rate: replay_sample + step of tools/bench_cnn.py's configuration (DSAC-T, carracing type_2 encoder, B = 1024),
  alternating.

    python tools/bench_coded_replay.py [--rows 200000] [--fill 20000] [--windows 5] [--skip-bytes]
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
SHAPE = (3, 96, 96)
LEVELS = np.asarray(np.arange(256) / 255, dtype=np.float32)   # gym_carracingraw: rgb.transpose(2, 0, 1) / 255
KINDS = ("flat", "frames", "coded")


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


def fill(buf, rows, seed=0):
    """Episodes of 1000 steps, obs_t = obs2_{t-1}: CarRacing-raw frames from a pool of 64 uint8 images, shifted by the
    step so that no two frames are equal."""
    g = np.random.default_rng(seed)
    pool = g.integers(0, 256, (64,) + SHAPE)
    frame = lambda n: LEVELS[(pool[g.integers(64)] + n) % 256]
    n = 0
    while n < rows:
        obs = frame(n)
        for t in range(min(1000, rows - n)):
            nxt = frame(n + t + 1)
            buf.store(obs, {}, np.zeros(3, np.float32), 0.0, nxt, t == 999, 0.0, {})
            obs = nxt
        n += 1000
    buf.flush()
    torch.cuda.synchronize()


def ring_bytes(rows, fill_rows):
    from training.replay_buffer import ReplayBuffer
    O = int(np.prod(SHAPE))
    eng = vec_engine(O, 3, 8)
    for kind in KINDS:
        kw = {} if kind == "flat" else {"dsact_replay_frames": 1}
        if kind == "coded":
            kw["dsact_replay_codes"] = True
        base = torch.cuda.memory_allocated(DEV)
        buf = ReplayBuffer(obsv_dim=SHAPE, action_dim=3, buffer_max_size=rows, **kw)
        t0 = time.perf_counter()
        buf.attach(eng)
        fill(buf, fill_rows)
        alloc = torch.cuda.memory_allocated(DEV) - base
        pl = buf.planner
        emit(what="ring_bytes", ring=kind, shape="carracing_raw_k1", rows=rows, rows_filled=fill_rows, allocated_GB=alloc / 1e9,
             held_GB=buf.__get_RAM__() / 1e3, frame_capacity=None if pl is None else pl.frame_capacity,
             codes=None if buf.coder is None else buf.coder.n, fill_s=time.perf_counter() - t0)
        del buf
        eng.replay = None
        torch.cuda.empty_cache()
    eng.close()


def bind_triple(make, cap, seed=1234):
    """Three engines holding the same cap rows of CarRacing-raw observations (row r: obs = frame r, obs2 = frame r + 1):
    a flat ring, a K = 1 fp32 frame ring and a K = 1 coded frame ring."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    codes = torch.randint(0, 256, (cap + 1, int(np.prod(SHAPE))), dtype=torch.uint8, device=DEV, generator=g)
    table = torch.from_numpy(LEVELS).to(DEV)
    rows = {k: torch.rand(cap, *s, device=DEV, generator=g) for k, s in (("act", (3,)), ("rew", ()), ("done", ()), ("logp", ()))}
    ids = torch.arange(cap, dtype=torch.int32, device=DEV)[:, None]
    engines = [make() for _ in KINDS]
    for e, kind in zip(engines, KINDS):
        e.seed(seed)
        if kind == "flat":
            e.bind_replay(cap)
            e.replay["obs"].copy_(table[codes[:-1].long()])
            e.replay["obs2"].copy_(table[codes[1:].long()])
        else:
            e.bind_replay_frames(cap, cap + 1, 1, coded=kind == "coded")
            e.replay["frames"].copy_(codes if kind == "coded" else table[codes.long()])
            if kind == "coded":
                e.replay["table"].copy_(table)
            e.replay["obs_frames"].copy_(ids)
            e.replay["obs2_frames"].copy_(ids + 1)
        for k, v in rows.items():
            e.replay[k].copy_(v)
    torch.cuda.synchronize()
    idx = torch.randint(0, cap, (64,), generator=torch.Generator().manual_seed(seed))
    out = [{k: v.clone() for k, v in e.replay_sample(64, cap, idx).items()} for e in engines]
    for o in out[1:]:
        assert all(torch.equal(o[k].view(torch.int32), out[0][k].view(torch.int32)) for k in o), "the rings gather differently"
    return engines


def alternate(fns, n, windows):
    """Median seconds per call of each fn over `windows` alternating windows of n calls, and the spread (max - min) /
    median."""
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
    O, cap = int(np.prod(SHAPE)), 20000
    for B in (256, 1024):
        engines = bind_triple(lambda: vec_engine(O, 3, B), cap)
        res = alternate([lambda e=e: e.replay_sample(B, cap) for e in engines], 200, windows)
        (tf, sf), (tr, sr), (tc, sc) = res
        emit(what="gather", shape="carracing_raw", batch=B, ring_rows=cap, flat_us=tf * 1e6, frame_us=tr * 1e6,
             coded_us=tc * 1e6, flat_spread=sf, frame_spread=sr, coded_spread=sc, coded_over_flat=tc / tf,
             coded_over_frame=tc / tr)
        for e in engines:
            e.close()
        del engines
        torch.cuda.empty_cache()


def update_rate(windows, B=1024):
    cfg = synth.CNN_CONFIGS["carracing"]
    t = synth.CONV_TYPES[cfg["conv_type"]]
    cap = 20000
    c = make_cnn_config(cfg["obs_dim"], cfg["act_dim"], t["kernels"], t["channels"], t["strides"], t["heads"], max_batch=B)
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    w = synth.make_cnn_weights(cfg)

    def make():
        e = CnnEngine(c, DEV, lim, -lim)
        e.load_weights(w)
        return e
    engines = bind_triple(make, cap)
    it = [0] * len(engines)

    def step(i):
        e = engines[i]
        e.step(e.replay_sample(B, cap), it[i])
        it[i] += 1
    (tf, sf), (tr, sr), (tc, sc) = alternate([lambda i=i: step(i) for i in range(len(engines))], 10, windows)
    emit(what="update_rate", shape="dsact_cnn_carracing_type2", batch=B, flat_steps_per_s=1 / tf, frame_steps_per_s=1 / tr,
         coded_steps_per_s=1 / tc, flat_spread=sf, frame_spread=sr, coded_spread=sc, coded_over_flat=tf / tc)
    for e in engines:
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=200000)
    ap.add_argument("--fill", type=int, default=20000)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--skip-bytes", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    gathers(a.windows)
    update_rate(a.windows)
    if not a.skip_bytes:
        ring_bytes(a.rows, min(a.fill, a.rows))


if __name__ == "__main__":
    main()
