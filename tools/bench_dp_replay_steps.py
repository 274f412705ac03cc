"""n data-parallel replay-fed updates per call (Engine.dp_replay_steps) against n dp_replay_step calls, one process per
GPU, the exchanges over NVLink peer memory, alternating the two paths window by window in one run.

For each world size (2, 4, 8 up to the GPUs the machine has), shape and n, rank 0 prints one JSON line: the median
updates/s over the timed windows of each path, their spread (max - min over the windows, relative to the median), the
gain, and whether the replicas' parameters were bit-identical afterwards.  Every line carries the card name, its power
limit and SM clocks, read in the same run.  All ranks run the same number of calls per window (rank 0 sizes the window
after the warm-up and broadcasts it): a data-parallel call waits for every peer.  Needs two or more GPUs; with fewer it
measures nothing and exits with an error.

    python tools/bench_dp_replay_steps.py [--windows 5] [--window-s 0.5] [--ns 8,32] [--worlds 2,4,8]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.multiprocessing as mp

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

# (label, config name, rows per rank, modes)
SHAPES = [("humanoid_b4096", "humanoid", 4096, ("bf16x3",)),
          ("humanoid_b256", "humanoid", 256, ("bf16x3",))]


def card(device):
    q = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    name, plim, sm, smmax = [x.strip() for x in q[0].split(",")] if q else ["?"] * 4
    return {"card": name, "power_limit": plim, "sm_clock": sm, "sm_clock_max": smmax}


def engine(cfg, B, mode, device):
    from dsac_v2_b200 import synth
    from dsac_v2_b200.engine import Engine, make_config
    h = synth.HYPER
    c = make_config(cfg["obs_dim"], cfg["act_dim"], *synth.hidden_sizes(cfg), max_batch=B, gemm_mode=mode, gamma=h["gamma"],
                    tau=h["tau"], delay_update=h["delay_update"], auto_alpha=h["auto_alpha"], alpha=h["alpha"],
                    lr_q=h["value_learning_rate"], lr_pi=h["policy_learning_rate"], lr_alpha=h["alpha_learning_rate"],
                    min_log_std=h["policy_min_log_std"], max_log_std=h["policy_max_log_std"])
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    e = Engine(c, device, lim, -lim)
    e.load_weights(synth.make_weights(cfg))
    e.seed(1234 + device.index)
    cap = 4 * B + 100
    g = np.random.default_rng(1 + device.index)
    O, A = cfg["obs_dim"], cfg["act_dim"]
    ring = {"obs": g.standard_normal((cap, O)), "obs2": g.standard_normal((cap, O)), "act": g.uniform(-1, 1, (cap, A)),
            "rew": g.standard_normal(cap), "done": (g.random(cap) < 0.05) * 1.0, "logp": g.standard_normal(cap)}
    e.bind_replay(cap)
    e.replay_add({k: torch.from_numpy(v.astype(np.float32)).to(device) for k, v in ring.items()}, cap, 0)
    return e, cap - 50


def _worker(rank, world, port, args):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from dsac_v2_b200 import dp, synth
    ns = [int(x) for x in args.ns.split(",")]
    for label, cfg_name, B, modes in SHAPES:
        cfg = synth.CONFIGS[cfg_name]
        for mode in modes:
            e, size = engine(cfg, B, mode, dev)
            if not dp.connect_peers(e, dist):
                raise SystemExit(f"rank {rank}: the ranks could not map each other's exchange buffers")
            it = [0]
            gb = B * world

            def singles(n):
                def run():
                    for _ in range(n):
                        e.dp_replay_step(B, size, it[0], gb); it[0] += 1
                return run

            def multi(n):
                def run():
                    e.dp_replay_steps(n, B, size, it[0], gb, stats=False); it[0] += n
                return run

            def window(run, per_call, calls):
                dist.barrier()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(calls):
                    run()
                torch.cuda.synchronize()
                return calls * per_call / (time.perf_counter() - t0)

            for n in ns:   # warm-up: every graph of the timed windows
                for _ in range(2):
                    singles(n)(); multi(n)()
            info = card(rank)
            for n in ns:
                # calls per window: sized on rank 0 from a warm run of the single calls, the same on every rank
                sized = [max(1, int(np.ceil(args.window_s / (n / window(singles(n), n, 4)))))]
                dist.broadcast_object_list(sized, src=0)
                rs, rm = [], []
                for _ in range(args.windows):
                    rs.append(window(singles(n), n, sized[0]))
                    rm.append(window(multi(n), n, sized[0]))
                if int(e.state[:16].view(torch.int32)[7]) != 0:
                    raise SystemExit(f"rank {rank}: an exchange timed out (slot 14 = {int(e.state[:16].view(torch.int32)[7])})")
                digest = hashlib.sha256(e.params.cpu().numpy().tobytes()).hexdigest()
                digests = [None] * world
                dist.all_gather_object(digests, digest)
                ms, mm = float(np.median(rs)), float(np.median(rm))
                if rank == 0:
                    print(json.dumps({"shape": label, "mode": mode, "world": world, "rows_per_rank": B, "n": n,
                                      "single_updates_per_s": round(ms, 1), "multi_updates_per_s": round(mm, 1),
                                      "gain": round(mm / ms - 1, 4), "single_spread": round((max(rs) - min(rs)) / ms, 4),
                                      "multi_spread": round((max(rm) - min(rm)) / mm, 4),
                                      "replicas_identical": len(set(digests)) == 1, **info}), flush=True)
            dist.barrier()
            e.close()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--window-s", type=float, default=0.5)
    ap.add_argument("--ns", default="8,32")
    ap.add_argument("--worlds", default="2,4,8")
    args = ap.parse_args()
    n_dev = torch.cuda.device_count()
    if n_dev < 2:
        raise SystemExit(f"needs two or more CUDA devices, found {n_dev}: nothing measured")
    for world in (int(w) for w in args.worlds.split(",")):
        if world > n_dev:
            continue
        mp.spawn(_worker, args=(world, 29500 + (os.getpid() + world) % 1000, args), nprocs=world, join=True)


if __name__ == "__main__":
    main()
