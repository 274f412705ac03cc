"""Data-parallel update on 2 to 8 GPUs (ragged shards) == single-GPU update on the concatenated minibatch, for both transports:
"peer" (exchanges inside the step's kernels over NVLink peer memory, one graph per rank: dsact_dp_step) and "nccl"
(torch.distributed all-reduces between the phase launches).  Needs >= 2 CUDA devices; world sizes above the device count are skipped."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, out_dir, gemm, transport):
    sys.path.insert(0, REPO)
    sys.path.insert(0, os.path.join(REPO, "dsac-v2_b200", "dropin"))
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import dsac_v2
    from dsac_v2_b200 import dp, synth
    cfg, B = synth.CONFIGS["halfcheetah"], GLOBAL_ROWS
    kw = synth.reference_kwargs(cfg, replay_batch_size=(B + world - 1) // world, dsact_gemm=gemm)
    alg = dsac_v2.DSAC_V2(**kw)
    sd = alg.networks.state_dict()
    for k, v in synth.make_weights(cfg).items():
        sd[k] = torch.from_numpy(v)
    alg.networks.load_state_dict(sd)
    alg.networks.cuda()
    eng = alg.networks.engine()
    if transport == "peer":
        assert dp.connect_peers(eng, dist), "the ranks could not map each other's exchange buffers"
    tbs = []
    for it in range(5):
        full, noise = synth.make_batch(cfg, B, it), synth.make_noise(cfg, B, it)
        lo, hi = dp.shard_rows(B, rank, world)
        shard = {k: torch.from_numpy(v[lo:hi]).cuda() for k, v in full.items()}
        nz = tuple(torch.from_numpy(noise[i][lo:hi]).cuda() for i in (0, 1, 4, 5))
        # the engine-level sequence DSAC_V2.local_update runs under torch.distributed, with explicit noise
        if transport == "peer":
            eng.dp_step(shard, it, B, nz)
            gb = B
        else:
            gb = dp.data_parallel_gradients(eng, shard, nz, dist, hi - lo, B)
            eng.apply(it)
        tbs.append([eng.read_stats(gb)[k] for k in ("Loss/Critic loss-RL iter", "Loss/Actor loss-RL iter",
                                                    "DSAC2/critic_avg_min_std1-RL iter", "DSAC2/mean_std1")])
    assert int(eng.state[:16].view(torch.int32)[7]) == 0, "a peer timed out"
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), params=eng.params.cpu().numpy(), targets=eng.targets.cpu().numpy(),
             grads=eng.grads.cpu().numpy(), tb=np.array(tbs))
    dist.destroy_process_group()


GLOBAL_ROWS = 250   # not a multiple of 4 or 8: the ranks hold shards of different sizes (dp.shard_rows)


@pytest.mark.parametrize("world", [2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("transport", ["peer", "nccl"])
@pytest.mark.parametrize("gemm", ["fp32", "bf16x3"])
def test_data_parallel_equals_single_gpu(tmp_path, gemm, transport, world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    port = 29600 + (os.getpid() + 13 * world + (7 if transport == "peer" else 0)) % 1000
    mp.spawn(_worker, args=(world, port, str(tmp_path), gemm, transport), nprocs=world, join=True)
    ranks = [np.load(tmp_path / f"rank{r}.npz") for r in range(world)]
    r0 = ranks[0]
    for r in ranks[1:]:
        np.testing.assert_array_equal(r0["params"], r["params"])   # replicas stay bit-identical
        np.testing.assert_array_equal(r0["targets"], r["targets"])
        np.testing.assert_array_equal(r0["grads"], r["grads"])     # every rank holds the global gradient
    # single GPU on the full minibatch
    sys.path.insert(0, os.path.join(REPO, "dsac-v2_b200", "dropin"))
    from dsac_v2_b200 import synth
    from dsac_v2_b200.engine import Engine, make_config
    cfg, B = synth.CONFIGS["halfcheetah"], GLOBAL_ROWS
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    eng = Engine(make_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], max_batch=B, gemm_mode=gemm),
                 torch.device("cuda", 0), lim, -lim)
    eng.load_weights(synth.make_weights(cfg))
    tbs = []
    for it in range(5):
        full, noise = synth.make_batch(cfg, B, it), synth.make_noise(cfg, B, it)
        eng.step({k: torch.from_numpy(v).cuda() for k, v in full.items()}, it,
                 tuple(torch.from_numpy(noise[i]).cuda() for i in (0, 1, 4, 5)))
        s = eng.read_stats()
        tbs.append([s[k] for k in ("Loss/Critic loss-RL iter", "Loss/Actor loss-RL iter",
                                   "DSAC2/critic_avg_min_std1-RL iter", "DSAC2/mean_std1")])
    tol = 2e-5 if gemm == "fp32" else 1e-4
    np.testing.assert_allclose(r0["tb"], np.array(tbs), rtol=tol, atol=1e-6)
    # parameters after 5 Adam steps (each moves a weight by <= 1e-4): Adam's normalisation turns the split-precision
    # summation-order noise on near-zero gradients into up to a few 1e-6 of weight, more with more shards
    atol = 2e-6 if gemm == "fp32" else 1e-5
    diff = np.abs(r0["params"] - eng.params.cpu().numpy())
    print(f"{gemm} {transport} world {world}: max |param diff| vs one GPU = {diff.max():.2e}")
    np.testing.assert_allclose(r0["params"], eng.params.cpu().numpy(), rtol=tol, atol=atol)
