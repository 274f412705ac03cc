"""Data-parallel updates of the head-wise engine on 2 to 8 GPUs (ragged shards) == one GPU on the concatenated
minibatch, for the CNN approximators (config `odd`) and the policy std types "mlp_separated" / "parameter", over both
transports: "peer" (`dsact_dp_step` on head-wise handles, exchanges inside the step's kernels over NVLink peer memory) and "nccl"
(`dp.data_parallel_gradients`: torch.distributed all-reduces between the split-API calls).  Each spawn also runs
`DSAC_V2(**cnn_reference_kwargs).local_update` under torch.distributed.  World sizes above the device count are skipped."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GLOBAL_ROWS = 250   # not a multiple of 4 or 8: the ranks hold shards of different sizes (dp.shard_rows)
CASES = ["odd", "mlp_separated", "parameter"]
STEPS = 5


def make_engine(case, max_batch, device):
    from dsac_v2_b200 import synth
    from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config, make_heads_config
    h = synth.HYPER
    hyper = dict(gamma=h["gamma"], tau=h["tau"], delay_update=h["delay_update"], auto_alpha=h["auto_alpha"], alpha=h["alpha"],
                 lr_q=h["value_learning_rate"], lr_pi=h["policy_learning_rate"], lr_alpha=h["alpha_learning_rate"],
                 min_log_std=h["policy_min_log_std"], max_log_std=h["policy_max_log_std"])
    if case == "odd":
        cfg = synth.CNN_CONFIGS[case]
        t = synth.CONV_TYPES[cfg["conv_type"]]
        c = make_cnn_config(cfg["obs_dim"], cfg["act_dim"], t["kernels"], t["channels"], t["strides"], t["heads"], max_batch=max_batch, **hyper)
        weights, make_batch = synth.make_cnn_weights(cfg), synth.make_cnn_batch
    else:
        cfg = synth.CONFIGS["ragged"]
        c = make_heads_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], case, max_batch=max_batch, **hyper)
        weights, make_batch = synth.make_weights_std(cfg, case), synth.make_batch
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    eng = CnnEngine(c, device, lim, -lim)
    eng.load_weights(weights)
    return eng, cfg, make_batch


def _worker(rank, world, port, out_dir, transport):
    sys.path.insert(0, REPO)
    sys.path.insert(0, os.path.join(REPO, "dsac-v2_b200", "dropin"))
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from dsac_v2_b200 import dp, synth
    from dsac_v2_b200.engine import STAT_KEYS
    B = GLOBAL_ROWS
    lo, hi = dp.shard_rows(B, rank, world)
    for case in CASES:
        eng, cfg, make_batch = make_engine(case, hi - lo, dev)
        if transport == "peer":
            assert dp.connect_peers(eng, dist), "the ranks could not map each other's exchange buffers"
        tbs = []
        for it in range(STEPS):
            full, noise = make_batch(cfg, B, it), synth.make_noise(cfg, B, it)
            shard = {k: torch.from_numpy(v[lo:hi]).cuda() for k, v in full.items()}
            nz = tuple(torch.from_numpy(noise[i][lo:hi]).cuda() for i in (0, 1, 4, 5))
            if transport == "peer":
                eng.dp_step(shard, it, B, nz)
            else:
                dp.data_parallel_gradients(eng, shard, nz, dist, hi - lo, B)
                eng.apply(it)
            s = eng.read_stats(B)   # raises if slot 14 (a peer never arrived) is set
            tbs.append([s[k] for k in STAT_KEYS])
        assert int(eng.state[:16].view(torch.int32)[7]) == 0, "a peer timed out"
        np.savez(os.path.join(out_dir, f"{case}_rank{rank}.npz"), params=eng.params.cpu().numpy(), targets=eng.targets.cpu().numpy(),
                 grads=eng.grads.cpu().numpy(), tb=np.array(tbs))
        dist.barrier()   # no rank reads a peer's exchange buffer any more: free them
        eng.close()
    # the reference-facing path: DSAC_V2 with CNN approximators under torch.distributed (every rank holds `rows` rows)
    import dsac_v2
    cfg, rows = synth.CNN_CONFIGS["carracing"], 4   # (the drop-in's networks.cnn builds the reference's conv types only)
    alg = dsac_v2.DSAC_V2(**synth.cnn_reference_kwargs(cfg, replay_batch_size=rows, dsact_dp_transport=transport))
    sd = alg.networks.state_dict()
    for k, v in synth.make_cnn_weights(cfg).items():
        sd[k] = torch.from_numpy(v)
    alg.networks.load_state_dict(sd)
    alg.networks.cuda()
    for it in range(2):
        shard = {k: torch.from_numpy(v[rank * rows:(rank + 1) * rows]).cuda() for k, v in synth.make_cnn_batch(cfg, rows * world, it).items()}
        tb = alg.local_update(shard, it)
        assert np.isfinite(tb["Loss/Critic loss-RL iter"]) and np.isfinite(tb["Loss/Actor loss-RL iter"])
    assert (alg._peer_dp is True) == (transport == "peer")
    eng = alg.networks.engine()
    np.savez(os.path.join(out_dir, f"dropin_rank{rank}.npz"), params=eng.params.cpu().numpy(), targets=eng.targets.cpu().numpy())
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("transport", ["peer", "nccl"])
def test_data_parallel_equals_single_gpu(tmp_path, transport, world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    port = 31600 + (os.getpid() + 13 * world + (7 if transport == "peer" else 0)) % 1000
    mp.spawn(_worker, args=(world, port, str(tmp_path), transport), nprocs=world, join=True)
    sys.path.insert(0, os.path.join(REPO, "dsac-v2_b200", "dropin"))
    from dsac_v2_b200 import synth
    from dsac_v2_b200.engine import STAT_KEYS
    dropin = [np.load(tmp_path / f"dropin_rank{r}.npz") for r in range(world)]
    for r in dropin[1:]:
        np.testing.assert_array_equal(dropin[0]["params"], r["params"], err_msg="DSAC_V2.local_update: replicas diverged")
        np.testing.assert_array_equal(dropin[0]["targets"], r["targets"])
    B = GLOBAL_ROWS
    for case in CASES:
        ranks = [np.load(tmp_path / f"{case}_rank{r}.npz") for r in range(world)]
        r0 = ranks[0]
        for r in ranks[1:]:
            np.testing.assert_array_equal(r0["params"], r["params"], err_msg=f"{case}: replicas diverged")   # bit-identical
            np.testing.assert_array_equal(r0["targets"], r["targets"], err_msg=case)
            np.testing.assert_array_equal(r0["grads"], r["grads"], err_msg=case)     # every rank holds the global gradient
        # one GPU on the full minibatch
        eng, cfg, make_batch = make_engine(case, B, torch.device("cuda", 0))
        tbs = []
        for it in range(STEPS):
            full, noise = make_batch(cfg, B, it), synth.make_noise(cfg, B, it)
            eng.step({k: torch.from_numpy(v).cuda() for k, v in full.items()}, it,
                     tuple(torch.from_numpy(noise[i]).cuda() for i in (0, 1, 4, 5)))
            s = eng.read_stats()
            tbs.append([s[k] for k in STAT_KEYS])
        np.testing.assert_allclose(r0["tb"], np.array(tbs), rtol=2e-5, atol=1e-6, err_msg=case)
        diff = np.abs(r0["params"] - eng.params.cpu().numpy())
        print(f"{case} {transport} world {world}: max |param diff| vs one GPU = {diff.max():.2e}")
        np.testing.assert_allclose(r0["params"], eng.params.cpu().numpy(), rtol=2e-5, atol=2e-6, err_msg=case)
        eng.close()
