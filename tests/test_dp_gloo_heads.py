"""World-size-2 CPU test (gloo) of the data-parallel seam for the head-wise engine's configurations: the collective
sequence of `dsac_v2_b200.dp.data_parallel_gradients`, driven by the CPU oracles of the CNN approximators
(`OracleDSACTCNN`) and of the policy std types "mlp_separated" / "parameter" (`OracleDSACTStd`), on ragged shards, must
reproduce the single-process full-batch update and keep the replicas identical."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_dp_gloo import OracleShardEngine

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = {   # name: global batch (odd: the ranks hold 5 + 4 and 19 + 18 rows)
    "cnn_odd": 9,
    "mlp_separated": 37,
    "parameter": 37,
}


def _oracle(case):
    from dsac_v2_b200 import synth
    from oracle.dsact_oracle import cnn_from_config, std_from_config
    if case == "cnn_odd":
        cfg = synth.CNN_CONFIGS["odd"]
        return cnn_from_config(cfg, synth.make_cnn_weights(cfg), **synth.HYPER), cfg, synth.make_cnn_batch
    cfg = synth.CONFIGS["ragged"]
    return std_from_config(cfg, synth.make_weights_std(cfg, case), case, **synth.HYPER), cfg, synth.make_batch


def _worker(rank, world, port, out_dir, case):
    sys.path.insert(0, REPO)
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from dsac_v2_b200 import dp, synth
    orc, cfg, make_batch = _oracle(case)
    eng, B = OracleShardEngine(orc), CASES[case]
    d, w = dp.world()
    assert w == world
    for it in range(4):
        full, noise = make_batch(cfg, B, it), synth.make_noise(cfg, B, it)
        lo, hi = dp.shard_rows(B, rank, world)
        shard = {k: torch.from_numpy(v[lo:hi]) for k, v in full.items()}
        nshard = [torch.from_numpy(n[lo:hi]) for n in noise]
        rows = dp.global_rows(d, hi - lo, torch.device("cpu"))
        assert rows == B
        dp.data_parallel_gradients(eng, shard, nshard, d, hi - lo, rows)
        eng.scatter_grads()
        eng.orc.apply(it)
    sd = {k: v.numpy() for k, v in eng.orc.state_dict().items()}
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **sd)
    dist.destroy_process_group()


@pytest.mark.parametrize("case", list(CASES))
def test_two_rank_shards_equal_full_batch(tmp_path, case):
    from dsac_v2_b200 import synth
    port = 30300 + (os.getpid() + 101 * list(CASES).index(case)) % 1500
    mp.spawn(_worker, args=(2, port, str(tmp_path), case), nprocs=2, join=True)
    ref, cfg, make_batch = _oracle(case)
    B = CASES[case]
    for it in range(4):
        ref.update(make_batch(cfg, B, it), synth.make_noise(cfg, B, it), it)
    r0, r1 = np.load(tmp_path / "rank0.npz"), np.load(tmp_path / "rank1.npz")
    sd = ref.state_dict()
    assert set(r0.files) == set(sd)
    for k, v in sd.items():
        np.testing.assert_array_equal(r0[k], r1[k], err_msg=f"replicas diverged: {k}")
        np.testing.assert_allclose(r0[k], v.numpy(), rtol=2e-5, atol=1e-7, err_msg=k)
