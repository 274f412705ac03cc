#!/usr/bin/env python
"""BASELINE.json config 5: gym_carracing-shaped CNN encoder + DSAC-T heads (reference networks/cnn.py `type_2`, 3x96x96
observations) at a fixed global batch (default 1024).  --gpus N > 1 spawns one process per GPU; each holds a shard of the
batch and runs the peer-memory data-parallel step (`CnnEngine.dp_step`).  Device-resident minibatches; prints one JSON line
with steps/s, the card's name, power limit and the clocks during the timed region, and whether the replicas ended
bit-identical (checksums all-gathered, as bench.py's replica check does).  With --cpu (one GPU only), the oracle port on
the host cores for the same step.  --algorithm DSAC_V1 times the older algorithm's update (one critic, fixed TD bound;
the reference's example_train/dsacv1_cnn_carracing_offasync.py) with the same encoder and heads, on one GPU: DSAC_V1 has
no data-parallel step.

    python tools/bench_cnn.py [--algorithm DSAC_V2|DSAC_V1] [--gpus 1] [--batch 1024] [--steps 20] [--warmup 3] [--cpu]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from dsac_v2_b200 import dp, synth  # noqa: E402
from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config  # noqa: E402


def card(index):
    """Name, power limit and maximum SM clock of GPU `index`, read in the same run as the measurement."""
    out = {"name": torch.cuda.get_device_name(index)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", str(index)],
                           capture_output=True, text=True, timeout=20).stdout.strip().split(",")
        out.update({"power_limit_w": float(r[0]), "sm_max_mhz": float(r[1])})
    except Exception:   # noqa: BLE001
        out.update({"power_limit_w": None, "sm_max_mhz": None})
    return out


def run(rank, world, a, out_path):
    cfg = synth.CNN_CONFIGS["carracing"]
    t = synth.CONV_TYPES[cfg["conv_type"]]
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    dist = None
    if world > 1:
        import torch.distributed as dist
        os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(a.port)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    lo, hi = dp.shard_rows(a.batch, rank, world)
    B = hi - lo
    v1 = a.algorithm == "DSAC_V1"
    c = make_cnn_config(cfg["obs_dim"], cfg["act_dim"], t["kernels"], t["channels"], t["strides"], t["heads"], max_batch=B,
                        algo=a.algorithm)
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    eng = CnnEngine(c, dev, lim, -lim)
    eng.load_weights(synth.make_cnn_weights_v1(cfg) if v1 else synth.make_cnn_weights(cfg))
    if dist is not None and not dp.connect_peers(eng, dist):
        raise SystemExit("the ranks could not map each other's exchange buffers (peer transport unavailable)")
    g = torch.Generator(device=dev).manual_seed(3 + rank)
    data = {"obs": torch.rand((B,) + tuple(cfg["obs_dim"]), device=dev, generator=g),
            "obs2": torch.rand((B,) + tuple(cfg["obs_dim"]), device=dev, generator=g),
            "act": (torch.rand(B, cfg["act_dim"], device=dev, generator=g) * 2 - 1) * cfg["act_lim"],
            "rew": torch.randn(B, device=dev, generator=g), "done": torch.zeros(B, device=dev)}
    step = (lambda it: eng.step(data, it)) if dist is None else (lambda it: eng.dp_step(data, it, a.batch))
    it = 0
    for _ in range(a.warmup):
        step(it); it += 1
    torch.cuda.synchronize(dev)
    if dist is not None:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ClockSampler(rank) as clocks:
        e0.record()
        for _ in range(a.steps):
            step(it); it += 1
        e1.record()
        torch.cuda.synchronize(dev)
        time.sleep(max(0.0, 1.2 - e0.elapsed_time(e1) / 1000))
    ms = e0.elapsed_time(e1) / a.steps
    stats = eng.read_stats(a.batch)   # raises if a peer never arrived (tb_info slot 14)
    parts = [eng.params, eng.targets, eng.adam_m, eng.adam_v]
    cs = torch.stack([p.double().sum() for p in parts] + [p.double().abs().sum() for p in parts])
    identical = True
    if dist is not None:
        gathered = [torch.zeros_like(cs) for _ in range(world)]
        dist.all_gather(gathered, cs)
        identical = all(bool(torch.equal(x, gathered[0])) for x in gathered)
    if rank == 0:
        name = "DSAC_V1" if v1 else "DSAC-T"
        out = {"metric": "%s gradient-steps/sec, CNN encoder (carracing type_2, 3x96x96), global batch %d on %d GPU(s)" % (name, a.batch, world),
               "value": 1000.0 / ms, "unit": "steps/s", "ms_per_step": ms, "steps": a.steps, "warmup": a.warmup, "dtype": "f32",
               "algorithm": a.algorithm, "data": "synthetic", "gpus": world, "transport": "peer" if world > 1 else None,
               "config": {"workload": "gym_carracing shapes, conv(4,3,3,3,3,3)/(8..256) + mean/log_std heads [256,256,256], fp32 direct convolutions",
                          "batch": a.batch, "shard_rows": [dp.shard_rows(a.batch, r, world)[1] - dp.shard_rows(a.batch, r, world)[0] for r in range(world)]},
               "card": card(0), "clocks_rank0": clocks.summary(), "finite": bool(all(v == v for v in stats.values())),
               "replicas_bit_identical": identical}
        if a.cpu:   # the CPU arm lives in bench.py (the one place outside tests/ and smoke() that may execute oracle/)
            import bench
            out["cpu_baseline"] = bench.time_cnn_cpu_port(cfg, a.batch, {k: v.cpu().numpy() for k, v in data.items()})
        with open(out_path, "w") as f:
            json.dump(out, f)
    eng.close()
    if dist is not None:
        dist.barrier()
        dist.destroy_process_group()


def _spawned(rank, world, a, out_path):
    run(rank, world, a, out_path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--algorithm", choices=("DSAC_V2", "DSAC_V1"), default="DSAC_V2")
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--batch", type=int, default=1024, help="global batch (split over the GPUs)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--port", type=int, default=29400 + os.getpid() % 1000)
    a = ap.parse_args()
    if a.algorithm == "DSAC_V1" and a.gpus > 1:
        raise SystemExit("--algorithm DSAC_V1 runs on one GPU: DSAC_V1 has no data-parallel step (use --gpus 1)")
    if a.gpus < 1 or a.gpus > torch.cuda.device_count():
        raise SystemExit(f"--gpus {a.gpus}: this host has {torch.cuda.device_count()} CUDA device(s)")
    if a.cpu and a.gpus > 1:
        raise SystemExit("--cpu compares against one GPU: use it with --gpus 1")
    if a.algorithm == "DSAC_V1" and a.cpu:
        raise SystemExit("--cpu times the DSAC-T step only: use it without --algorithm DSAC_V1")
    with tempfile.TemporaryDirectory() as tmp:
        out_path = os.path.join(tmp, "result.json")
        if a.gpus == 1:
            run(0, 1, a, out_path)
        else:
            import torch.multiprocessing as mp
            mp.spawn(_spawned, args=(a.gpus, a, out_path), nprocs=a.gpus, join=True)
        print(open(out_path).read())


if __name__ == "__main__":
    main()
