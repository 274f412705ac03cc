"""DSAC_V2.replay_updates under torch.distributed on 2 to 8 GPUs with the peer transport: one captured
dsact_dp_replay_steps graph per rank and call.  Every rank draws its own minibatches from its own replay buffer (numpy
indices, the reference's torch CPU noise).  After every call the replicas must be bit-identical, and every update must
equal, within the gates of tests/test_gpu_dp.py, one GPU's update on the concatenation of the ranks' minibatches and
noise.  Needs >= 2 CUDA devices; world sizes above the device count are skipped."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, CAP = 64, 300                  # rows per rank and update; rows of every rank's replay buffer
CALLS = ((0, 2), (2, 2), (4, 1))  # (first iteration, n): the second call replays the first call's captured graph
KEYS = ("Loss/Critic loss-RL iter", "Loss/Actor loss-RL iter", "DSAC2/critic_avg_min_std1-RL iter", "DSAC2/mean_std1")


def _ring_rows(cfg, n):
    """The rows every rank's buffer holds (ReplayBuffer.add_batch samples)."""
    g = np.random.default_rng(4)
    O, A = cfg["obs_dim"], cfg["act_dim"]
    return [(g.standard_normal(O).astype(np.float32), {}, g.uniform(-1, 1, A).astype(np.float32), float(g.standard_normal()),
             g.standard_normal(O).astype(np.float32), bool(i % 7 == 0), np.float32(-1.0), {}) for i in range(n)]


def _worker(rank, world, port, out_dir, gemm):
    sys.path.insert(0, REPO)
    sys.path.insert(0, os.path.join(REPO, "dsac-v2_b200", "dropin"))
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import dsac_v2
    from dsact_host import host_draws
    from training.replay_buffer import ReplayBuffer
    from dsac_v2_b200 import synth
    cfg = synth.CONFIGS["halfcheetah"]
    kw = synth.reference_kwargs(cfg, replay_batch_size=B, dsact_gemm=gemm, dsact_noise="reference", dsact_index_source="numpy")
    alg = dsac_v2.DSAC_V2(**kw)
    sd = alg.networks.state_dict()
    for k, v in synth.make_weights(cfg).items():
        sd[k] = torch.from_numpy(v)
    alg.networks.load_state_dict(sd)
    alg.networks.cuda()
    eng = alg.networks.engine(B)
    buf = ReplayBuffer(**dict(kw, buffer_max_size=CAP, additional_info={}))
    buf.attach(eng)
    buf.add_batch(_ring_rows(cfg, CAP))
    buf.flush()
    ring = {k: v.cpu().numpy() for k, v in eng.replay.items()}
    calls = []
    steps = eng.dp_replay_steps
    eng.dp_replay_steps = lambda *a, **k: (calls.append(a[0]), steps(*a, **k))[1]
    out = dict(ring_obs=ring["obs"], ring_obs2=ring["obs2"], ring_act=ring["act"], ring_rew=ring["rew"], ring_done=ring["done"])
    tbs, idx, noise = [], [], []
    for c, (it, n) in enumerate(CALLS):
        seed = 1000 * c + rank
        np.random.seed(seed); torch.manual_seed(seed)
        i, nz = host_draws(buf, B, n, alg._noise)   # what the call will draw
        idx.append(i.numpy()); noise.append([x.numpy() for x in nz])
        np.random.seed(seed); torch.manual_seed(seed)
        infos = alg.replay_updates(buf, B, it, n)
        tbs.extend([info[k] for k in KEYS] for info in infos)
        torch.cuda.synchronize()
        for k in ("params", "targets", "adam_m", "adam_v"):
            out[f"{k}_{c}"] = getattr(eng, k).cpu().numpy()
    assert alg._peer_dp, "the ranks could not map each other's exchange buffers"
    assert calls == [n for _, n in CALLS], f"replay_updates made the dp_replay_steps calls {calls}"
    assert int(eng.state[:16].view(torch.int32)[7]) == 0, "a peer timed out"
    out.update(tb=np.array(tbs), idx=np.concatenate(idx), **{f"noise{j}": np.concatenate([z[j] for z in noise]) for j in range(4)})
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **out)
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("gemm", ["fp32", "bf16x3"])
def test_replay_updates_under_torch_distributed_equal_single_gpu(tmp_path, gemm, world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    port = 29600 + (os.getpid() + 13 * world + 3) % 1000
    mp.spawn(_worker, args=(world, port, str(tmp_path), gemm), nprocs=world, join=True)
    ranks = [np.load(tmp_path / f"rank{r}.npz") for r in range(world)]
    r0 = ranks[0]
    for c in range(len(CALLS)):
        for r, x in enumerate(ranks[1:], 1):
            for k in ("params", "targets", "adam_m", "adam_v"):   # replicas stay bit-identical
                np.testing.assert_array_equal(x[f"{k}_{c}"], r0[f"{k}_{c}"], err_msg=f"call {c} rank {r} {k}")
    # one GPU on the concatenation of the ranks' minibatches and noise, update by update
    from dsac_v2_b200 import synth
    from dsac_v2_b200.engine import Engine, make_config
    cfg = synth.CONFIGS["halfcheetah"]
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    eng = Engine(make_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], max_batch=B * world, gemm_mode=gemm),
                 torch.device("cuda", 0), lim, -lim)
    eng.load_weights(synth.make_weights(cfg))
    tol = 2e-5 if gemm == "fp32" else 1e-4
    atol = 2e-6 if gemm == "fp32" else 1e-5   # as tests/test_gpu_dp.py: Adam turns summation-order noise into weight
    u = 0
    for c, (it0, n) in enumerate(CALLS):
        tbs = []
        for k in range(n):
            rows = {key: np.concatenate([x[f"ring_{key}"][x["idx"][u]] for x in ranks]) for key in ("obs", "act", "rew", "obs2", "done")}
            nz = tuple(torch.from_numpy(np.concatenate([x[f"noise{j}"][u] for x in ranks])).cuda() for j in range(4))
            eng.step({key: torch.from_numpy(v).cuda() for key, v in rows.items()}, it0 + k, nz)
            s = eng.read_stats()
            tbs.append([s[key] for key in KEYS])
            u += 1
        np.testing.assert_allclose(r0["tb"][u - n:u], np.array(tbs), rtol=tol, atol=1e-6, err_msg=f"call {c} statistics")
        diff = np.abs(r0[f"params_{c}"] - eng.params.cpu().numpy())
        print(f"{gemm} world {world} call {c}: max |param diff| vs one GPU = {diff.max():.2e}")
        np.testing.assert_allclose(r0[f"params_{c}"], eng.params.cpu().numpy(), rtol=tol, atol=atol, err_msg=f"call {c} params")
    eng.close()
