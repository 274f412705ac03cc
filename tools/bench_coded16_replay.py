"""The 16-bit coded frame ring (`ReplayBuffer(dsact_replay_frames=4, dsact_replay_codes=16)`) on `gym_carracing`'s
observations: 4 stacked grey 96x96 frames, dot(rgb, [0.299, 0.587, 0.114]) / 128 - 1 (BASELINE config 5).  Device
bytes, gather time per call and the CNN replay-fed update rate, on one GPU.  One JSON line per measurement; every line
carries the card name, its power limit and SM clocks, read in the same run.

- ring bytes: the fp32 frame ring and the 16-bit ring bound at --rows rows (K = 4) through the drop-in ReplayBuffer and
  fed --fill rows of 1000-step stacked episodes, measured as the torch.cuda.memory_allocated delta.  Stacked rows store
  one new frame each, so the frame store never grows past its initial capacity: the allocation at --rows rows is the
  ring's footprint at that size.
- gather: dsact_replay_sample with device-drawn indices at B = 256 and 1024 from rings of 20 000 rows (K = 4, one new
  frame per row) holding the same observations (checked equal once): the fp32 frame ring against the 16-bit ring, in
  alternating timed windows (median per call and spread).  Two streams: one of 3000 grey values (12 KiB of the table
  in use) and one of 60 000 (234 KiB: more than L1 keeps).  --other-build PATH adds the same gathers on a second build
  of libdsact.so (another decode design), alternating with the others.
- update rate: replay_sample + step of DSAC-T with the carracing type_2 encoder on 4x96x96 input at B = 1024, flat ring
  against the 16-bit ring, alternating.

    python tools/bench_coded16_replay.py [--rows 200000] [--fill 20000] [--windows 5] [--other-build PATH] [--skip-bytes]
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

from dsac_v2_b200 import _lib, synth  # noqa: E402
from dsac_v2_b200.engine import Engine, make_config  # noqa: E402
from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config  # noqa: E402

DEV = torch.device("cuda", 0)
K = 4
SHAPE = (K, 96, 96)
F = 96 * 96
# BASELINE config 5: gym_carracing (4 stacked grey frames) with the carracing type_2 encoder
STACKED4 = dict(obs_dim=SHAPE, act_dim=3, act_lim=1.0, conv_type="type_2")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, plim, sm, smmax = [x.strip() for x in q[0].split(",")] if q else ["?"] * 4
    return {"card": name, "power_limit": plim, "sm_clock": sm, "sm_clock_max": smmax}


def emit(**kw):
    print(json.dumps({**kw, **card()}), flush=True)


def grey_levels(n, seed=0):
    """n distinct grey values of the reference's rgb2gray, in random order."""
    g = np.random.default_rng(seed)
    rgb = g.integers(0, 256, (4 * n, 3))
    v = np.unique(np.asarray(np.dot(rgb, [0.299, 0.587, 0.114]) / 128.0 - 1.0, dtype=np.float32).view(np.uint32))
    assert len(v) >= n
    g.shuffle(v)
    return v[:n].view(np.float32)


def vec_engine(obs_dim, act_dim, batch, hidden=(64,)):
    lim = torch.ones(act_dim)
    return Engine(make_config(obs_dim, act_dim, hidden, hidden, max_batch=batch, gemm_mode="fp32"), DEV, lim, -lim)


def on_build(path, make):
    """make() with every entry point of the engines it creates bound to another build of libdsact.so."""
    saved = _lib._lib, _lib.LIB_PATH
    _lib._lib, _lib.LIB_PATH = None, path
    try:
        return make()
    finally:
        _lib._lib, _lib.LIB_PATH = saved


def fill(buf, rows, levels, seed=0):
    """Stacked episodes of 1000 steps (obs2 = obs shifted by one frame): grey frames drawn from `levels`."""
    g = np.random.default_rng(seed)
    pool = g.integers(0, len(levels), (64, 96, 96))
    frame = lambda n: levels[(pool[g.integers(64)] + n) % len(levels)]
    n = 0
    while n < rows:
        stack = [frame(n)] * K
        for t in range(min(1000, rows - n)):
            nxt = stack[1:] + [frame(n + t + 1)]
            buf.store(np.stack(stack), {}, np.zeros(3, np.float32), 0.0, np.stack(nxt), t == 999, 0.0, {})
            stack = nxt
        n += 1000
    buf.flush()
    torch.cuda.synchronize()


def ring_bytes(rows, fill_rows):
    from training.replay_buffer import ReplayBuffer
    eng = vec_engine(int(np.prod(SHAPE)), 3, 8)
    levels = grey_levels(3000)
    for kind in ("frames", "coded16"):
        kw = {"dsact_replay_frames": K}
        if kind == "coded16":
            kw["dsact_replay_codes"] = 16
        base = torch.cuda.memory_allocated(DEV)
        buf = ReplayBuffer(obsv_dim=SHAPE, action_dim=3, buffer_max_size=rows, **kw)
        t0 = time.perf_counter()
        buf.attach(eng)
        fill(buf, fill_rows, levels)
        alloc = torch.cuda.memory_allocated(DEV) - base
        emit(what="ring_bytes", ring=kind, shape="carracing_stacked_k4", rows=rows, rows_filled=fill_rows,
             allocated_GB=alloc / 1e9, held_GB=buf.__get_RAM__() / 1e3, frame_capacity=buf.planner.frame_capacity,
             codes=None if buf.coder is None else buf.coder.n, fill_s=time.perf_counter() - t0)
        del buf
        eng.replay = None
        torch.cuda.empty_cache()
    eng.close()


def bind(engines, kinds, cap, levels, seed=1234):
    """The same cap rows of stacked frames in every engine (row r: obs = frames r..r+3, obs2 = frames r+1..r+4): a flat
    ring, a K = 4 fp32 frame ring or a K = 4 16-bit ring, by kind."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    nf = cap + K
    codes = torch.randint(0, len(levels), (nf, F), dtype=torch.int32, device=DEV, generator=g)
    table = torch.from_numpy(levels).to(DEV)
    rows = {k: torch.rand(cap, *s, device=DEV, generator=g) for k, s in (("act", (3,)), ("rew", ()), ("done", ()), ("logp", ()))}
    ids = torch.arange(cap, dtype=torch.int32, device=DEV)[:, None] + torch.arange(K, dtype=torch.int32, device=DEV)
    for e, kind in zip(engines, kinds):
        e.seed(seed)
        if kind == "flat":
            e.bind_replay(cap)
            vals = table[codes.long()]
            e.replay["obs"].copy_(vals[ids.long()].reshape(cap, -1))
            e.replay["obs2"].copy_(vals[ids.long() + 1].reshape(cap, -1))
            del vals
        else:
            coded = kind == "coded16"
            e.bind_replay_frames(cap, nf, K, coded=coded, code_bits=16)
            if coded:
                e.replay["frames"].copy_(codes.to(torch.int16))
                e.replay["table"][:len(levels)].copy_(table)
            else:
                e.replay["frames"].copy_(table[codes.long()])
            e.replay["obs_frames"].copy_(ids)
            e.replay["obs2_frames"].copy_(ids + 1)
        for k, v in rows.items():
            e.replay[k].copy_(v)
    torch.cuda.synchronize()
    idx = torch.randint(0, cap, (64,), generator=torch.Generator().manual_seed(seed))
    out = [{k: v.clone() for k, v in e.replay_sample(64, cap, idx).items()} for e in engines]
    for o in out[1:]:
        assert all(torch.equal(o[k].view(torch.int32), out[0][k].view(torch.int32)) for k in o), "the rings gather differently"


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


def gathers(windows, other):
    O, cap = int(np.prod(SHAPE)), 20000
    for n_values in (3000, 60000):
        levels = grey_levels(n_values)
        for B in (256, 1024):
            kinds = ["frames", "coded16"]
            engines = [vec_engine(O, 3, B) for _ in kinds]
            if other:
                kinds.append("coded16")
                engines.append(on_build(other, lambda: vec_engine(O, 3, B)))
            bind(engines, kinds, cap, levels)
            res = alternate([lambda e=e: e.replay_sample(B, cap) for e in engines], 100, windows)
            line = dict(what="gather", shape="carracing_stacked_k4", distinct_values=n_values, batch=B, ring_rows=cap,
                        frame_us=res[0][0] * 1e6, coded16_us=res[1][0] * 1e6, frame_spread=res[0][1],
                        coded16_spread=res[1][1], coded16_over_frame=res[1][0] / res[0][0])
            if other:
                line.update(other_build=other, other_us=res[2][0] * 1e6, other_spread=res[2][1],
                            other_over_coded16=res[2][0] / res[1][0])
            emit(**line)
            for e in engines:
                e.close()
            del engines
            torch.cuda.empty_cache()


def update_rate(windows, B=1024):
    cfg = STACKED4
    t = synth.CONV_TYPES[cfg["conv_type"]]
    cap = 20000
    c = make_cnn_config(cfg["obs_dim"], cfg["act_dim"], t["kernels"], t["channels"], t["strides"], t["heads"], max_batch=B)
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    w = synth.make_cnn_weights(cfg)

    def make():
        e = CnnEngine(c, DEV, lim, -lim)
        e.load_weights(w)
        return e
    kinds = ("flat", "coded16")
    engines = [make() for _ in kinds]
    bind(engines, kinds, cap, grey_levels(3000))
    it = [0] * len(engines)

    def step(i):
        e = engines[i]
        e.step(e.replay_sample(B, cap), it[i])
        it[i] += 1
    (tf, sf), (tc, sc) = alternate([lambda i=i: step(i) for i in range(len(engines))], 10, windows)
    emit(what="update_rate", shape="dsact_cnn_carracing_stacked_type2", batch=B, flat_steps_per_s=1 / tf,
         coded16_steps_per_s=1 / tc, flat_spread=sf, coded16_spread=sc, coded16_over_flat=tf / tc)
    for e in engines:
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=200000)
    ap.add_argument("--fill", type=int, default=20000)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--other-build", default=None, help="a second build of libdsact.so to time the gathers on as well")
    ap.add_argument("--skip-bytes", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    gathers(a.windows, a.other_build and os.path.abspath(a.other_build))
    update_rate(a.windows)
    if not a.skip_bytes:
        ring_bytes(a.rows, min(a.fill, a.rows))


if __name__ == "__main__":
    main()
