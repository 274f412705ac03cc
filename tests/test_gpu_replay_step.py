"""The replay-fed step (`dsact_replay_step`, what bench.py times) and the device generator it draws from.

Every draw is checked against the host restatement in oracle/dsact_rng.py: the replay indices bit for bit, the noise to a
few float32 ulps (`logf` and `sincospif` are not correctly rounded).  The reference minibatch is always the HOST copy of
the ring indexed by those draws: in the fused tensor-core modes the gather writes only the bf16 images, so the arena's
fp32 copy of obs / obs2 / act is stale by design."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from dsac_v2_b200 import synth
from oracle.dsact_rng import device_noise, replay_indices
from test_gpu_parity import RTOL, WIDE, make_engine, stats_vec

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# obs 520 = 130 float4 columns: the gather's float4 loop takes a second trip (c0 += 96 passes 96 < 130); act 40 > 32: the
# act loop takes a second trip; B = 10000 > 8 * 132 * 8 rows: the grid-stride loop of the gather takes a second pass
GATHERWIDE = dict(obs_dim=520, act_dim=40, hidden=(64, 64), act_lim=1.0)
SHAPES = {"tiny": (synth.CONFIGS["tiny"], 16), "ragged": (synth.CONFIGS["ragged"], 37),
          "humanoid": (synth.CONFIGS["humanoid"], 4096), "gatherwide": (GATHERWIDE, 10000), "wide": (WIDE, 40)}
MODES = ["fp32", "bf16x3", "bf16"]
SEED = 0x0123456789ABCDEF

# Device noise vs the float64 restatement, in float32 ulps of the restated value.  Measured on one H100 80GB HBM3 (400 W):
# at most 2.6 ulps over every shape and mode of this file (logf, sqrtf, sincospif and the products each round once).
NOISE_ULPS = 4


def ring_rows(cfg, cap, seed=11):
    g = np.random.default_rng(seed)
    O, A, lim = cfg["obs_dim"], cfg["act_dim"], cfg["act_lim"]
    return {"obs": g.standard_normal((cap, O)).astype(np.float32), "obs2": g.standard_normal((cap, O)).astype(np.float32),
            "act": g.uniform(-lim, lim, (cap, A)).astype(np.float32), "rew": g.standard_normal(cap).astype(np.float32),
            "done": (g.random(cap) < 0.05).astype(np.float32), "logp": g.standard_normal(cap).astype(np.float32)}


def bind_ring(eng, host):
    cap = host["obs"].shape[0]
    eng.bind_replay(cap)
    eng.replay_add({k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in host.items()}, cap, 0)


def counter(eng) -> int:
    torch.cuda.synchronize()
    return int(eng.state.view(torch.int32)[10].item()) & 0xFFFFFFFF


def rows(host, idx):
    return {k: host[k][idx] for k in ("obs", "act", "rew", "obs2", "done")}


def oracle_noise(eps1, eps2, z3, z4):
    """The 8-draw list oracle.update takes; only eps1, eps2, z3 and z4 (positions 0, 1, 4, 5) enter the update."""
    f = lambda x: np.asarray(x, dtype=np.float32)
    z = np.zeros_like(f(z3))
    return [f(eps1), f(eps2), z, z, f(z3), f(z4), z, z]


def noise_ulps(eng, B, A, ctr):
    """Largest distance, in float32 ulps, between the arena's noise slots and the restated draws at counter `ctr`."""
    ref = device_noise(SEED, ctr, B, A)
    v = eng.arena_views(B)
    worst = 0.0
    for k, r in zip(("eps1", "eps2", "z3", "z4"), ref):
        got = v[k].double().cpu().numpy()
        worst = max(worst, float(np.max(np.abs(got - r) / np.spacing(np.abs(r).astype(np.float32)))))
    return worst


def fused(cfg, mode):
    return mode != "fp32" and cfg is not WIDE


def setup(name, mode, use_graph, extra=5):
    cfg, B = SHAPES[name]
    eng = make_engine(cfg, B, use_graph=use_graph, gemm_mode=mode)
    eng.seed(SEED)
    cap = B + 3 * B // 4 + 8
    host = ring_rows(cfg, cap)
    bind_ring(eng, host)
    return cfg, B, eng, host, cap - extra


def poison_arena_inputs(eng, cfg, B):
    """NaN over the arena's fp32 obs / obs2 / act (the first three arena slots, Arena::build): a fused step must not read them."""
    r64 = lambda n: (n + 63) // 64 * 64
    n = 2 * r64(B * cfg["obs_dim"]) + r64(B * cfg["act_dim"])
    eng._ws_view[:n].fill_(float("nan"))


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(SHAPES))
def test_replay_draws_equal_the_restatement(name, mode, use_graph):
    cfg, B, eng, host, size = setup(name, mode, use_graph)
    A = cfg["act_dim"]
    g = np.random.default_rng(3)
    worst = 0.0

    # replay_sample without indices: the gather draws them, records them and the counter steps once
    c = counter(eng)
    got = eng.replay_sample(B, size)
    ref_idx = replay_indices(SEED, c, B, size)
    np.testing.assert_array_equal(eng.arena_views(B)["idx"].cpu().numpy(), ref_idx)
    assert counter(eng) == c + 1
    for k in ("obs", "obs2", "act", "rew", "done", "logp"):   # replay_sample always writes the fp32 copy
        np.testing.assert_array_equal(got[k].cpu().numpy(), host[k][ref_idx], err_msg=k)

    it = 0
    for give_idx in (False, True):
        for give_noise in (False, True):
            c = counter(eng)
            idx = g.integers(0, size, B) if give_idx else None
            nz = tuple(torch.from_numpy(x.astype(np.float32)) for x in device_noise(99, it, B, A)) if give_noise else None
            eng.replay_step(B, size, it, idx=None if idx is None else torch.from_numpy(idx), noise=nz)
            drew = not (give_idx and give_noise)
            assert counter(eng) == c + (1 if drew else 0), (give_idx, give_noise)
            if not give_idx:
                np.testing.assert_array_equal(eng.arena_views(B)["idx"].cpu().numpy(), replay_indices(SEED, c, B, size))
            if not give_noise:
                worst = max(worst, noise_ulps(eng, B, A, c))
            assert np.all(np.isfinite(stats_vec(eng)))
            it += 1

    # step() on a device minibatch with device noise (the fp32 noise kernel, or the tensor-core prologue)
    c = counter(eng)
    idx = g.integers(0, size, B)
    eng.step({k: torch.from_numpy(v).cuda() for k, v in rows(host, idx).items()}, it, None)
    assert counter(eng) == c + 1
    worst = max(worst, noise_ulps(eng, B, A, c))
    it += 1

    # the ring size lives in device state, outside the graph key: a replayed graph must draw from the new size
    for s in (size, max(1, size // 3), size):
        c = counter(eng)
        eng.replay_step(B, s, it)
        np.testing.assert_array_equal(eng.arena_views(B)["idx"].cpu().numpy(), replay_indices(SEED, c, B, s))
        worst = max(worst, noise_ulps(eng, B, A, c))
        assert counter(eng) == c + 1
        it += 1
    print(f"{name} {mode} graph={use_graph}: device noise within {worst:.1f} float32 ulps of the restatement")
    assert worst <= NOISE_ULPS, worst
    eng.close()


def check_against_oracle(eng, mode, it, ref):
    from oracle.dsact_oracle import TB_KEYS
    got = stats_vec(eng)
    assert np.all(np.isfinite(got)), got
    want = np.array([ref[k] for k in TB_KEYS])
    if mode == "bf16":   # single-pass bf16: loose, like test_bf16_single_pass_is_close_but_outside_the_parity_gate
        assert abs(got[7] - want[7]) <= 5e-2 * abs(want[7]), (it, got[7], want[7])
        return
    np.testing.assert_allclose(got, want, rtol=RTOL, atol=1e-5, err_msg=f"step {it}")


def check_digests(eng, orc, mode):
    w = eng.export_weights()
    for k, v in orc.state_dict().items():
        a, r = w[k].double().reshape(-1), v.double().reshape(-1)
        assert torch.isfinite(a).all(), k
        if mode == "bf16":
            continue
        np.testing.assert_allclose(a.abs().sum().item(), r.abs().sum().item(), rtol=RTOL, err_msg=k)
        np.testing.assert_allclose(a[:8].numpy(), r[:8].numpy(), rtol=RTOL, atol=1e-6, err_msg=k)


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(SHAPES))
def test_replay_step_matches_oracle(name, mode, use_graph):
    """Device-drawn indices and noise, 3 steps, against the oracle on the restated draws.  In the fused modes the arena's
    fp32 obs / obs2 / act are NaN before every call: the step must read only the images the gather wrote."""
    from oracle.dsact_oracle import from_config
    cfg, B, eng, host, size = setup(name, mode, use_graph)
    orc = from_config(cfg, synth.make_weights(cfg), **synth.HYPER)
    torch.set_num_threads(min(16, os.cpu_count() or 4))
    try:
        for it in range(3):
            c = counter(eng)
            if fused(cfg, mode):
                poison_arena_inputs(eng, cfg, B)
            eng.replay_step(B, size, it)
            idx = replay_indices(SEED, c, B, size)
            ref = orc.update(rows(host, idx), oracle_noise(*device_noise(SEED, c, B, cfg["act_dim"])), it)
            check_against_oracle(eng, mode, it, ref)
    finally:
        torch.set_num_threads(4)
    check_digests(eng, orc, mode)
    eng.close()


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / max(float(b.norm()), 1e-30))


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(SHAPES))
def test_replay_step_equals_step_on_the_gathered_rows(name, mode, use_graph):
    """replay_step(idx, noise) and step(ring[idx], noise) on twin engines: the gather's bf16 images and the prologue's must
    round the same way.  Bit-identical up to 16 rows; above that the float atomics of the bias gradients may sum in another
    order (DESIGN §9, item 6)."""
    cfg, B, a, host, size = setup(name, mode, use_graph)
    b = make_engine(cfg, B, use_graph=use_graph, gemm_mode=mode)
    g = np.random.default_rng(5)
    # single-pass bf16 rounds every activation once: a last-bit difference from the atomics' order can flip a rounding,
    # which moves a logged mean by up to ~1e-5 relative (measured 1.3e-5 on humanoid B = 4096)
    tol = 1e-4 if mode == "bf16" else 1e-6
    for it in range(3):
        idx = g.integers(0, size, B)
        n = synth.make_noise(cfg, B, it)
        nz = tuple(torch.from_numpy(n[i]) for i in (0, 1, 4, 5))
        a.replay_step(B, size, it, idx=torch.from_numpy(idx), noise=nz)
        b.step({k: torch.from_numpy(v).cuda() for k, v in rows(host, idx).items()}, it, nz)
        sa, sb = stats_vec(a), stats_vec(b)
        if B <= 16:
            np.testing.assert_array_equal(sa, sb, err_msg=f"stats step {it}")
        else:
            np.testing.assert_allclose(sa, sb, rtol=tol, atol=1e-7, err_msg=f"stats step {it}")
    torch.cuda.synchronize()
    for k in ("params", "targets", "adam_m", "adam_v"):
        ta, tb = getattr(a, k), getattr(b, k)
        if B <= 16:
            assert torch.equal(ta, tb), k
        else:
            assert rel_l2(ta, tb) <= tol, (k, rel_l2(ta, tb))
    a.close(); b.close()


def test_replay_sample_then_step_reads_the_gathered_images():
    """replay_sample -> step on the arena views (take_arena_images: the step reuses the gather's images) in bf16x3 at
    humanoid B = 256, device-drawn indices, against the oracle."""
    from oracle.dsact_oracle import from_config
    cfg, B = synth.CONFIGS["humanoid"], 256
    eng = make_engine(cfg, B, use_graph=True, gemm_mode="bf16x3")
    eng.seed(SEED)
    host = ring_rows(cfg, 1000)
    bind_ring(eng, host)
    orc = from_config(cfg, synth.make_weights(cfg), **synth.HYPER)
    for it in range(3):
        c = counter(eng)
        data = eng.replay_sample(B, 900)
        idx = replay_indices(SEED, c, B, 900)
        n = synth.make_noise(cfg, B, it)
        eng.step(data, it, tuple(torch.from_numpy(n[i]).cuda() for i in (0, 1, 4, 5)))
        ref = orc.update(rows(host, idx), n, it)
        check_against_oracle(eng, "bf16x3", it, ref)
    check_digests(eng, orc, "bf16x3")
    eng.close()


@pytest.mark.parametrize("use_graph", [False, True])
def test_step_on_sampled_views_after_a_profiled_step_images_them_again(use_graph):
    """replay_sample, then profile_step on another minibatch, then step on the sampled arena views, in bf16x3 at B = 16.
    The profiled step wrote its own rows' images into the arena's input image slots, so the step must image the views
    again: its parameters, targets, Adam moments and state equal, bit for bit, a twin engine's step on a copy of the
    sampled rows (up to 16 rows an update is bit-reproducible, DESIGN §9 item 6)."""
    cfg, B, a, host, size = setup("tiny", "bf16x3", use_graph)
    b = make_engine(cfg, B, use_graph=use_graph, gemm_mode="bf16x3")
    b.seed(SEED)
    bind_ring(b, host)
    other = {k: torch.from_numpy(v).cuda() for k, v in synth.make_batch(cfg, B, 7).items()}
    noise = [tuple(torch.from_numpy(n[i]).cuda() for i in (0, 1, 4, 5)) for n in (synth.make_noise(cfg, B, it) for it in (0, 1))]
    views = a.replay_sample(B, size)
    copy = {k: v.clone() for k, v in views.items()}
    b.replay_sample(B, size)   # the same draws: the generator counters stay equal
    for e in (a, b):
        e.profile_step(other, 0, noise[0])
    a.step(views, 1, noise[1])
    b.step(copy, 1, noise[1])
    torch.cuda.synchronize()
    for k in ("params", "targets", "adam_m", "adam_v", "state"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k
    a.close(); b.close()


def test_headwise_replay_sample_draws_and_gathers_exactly():
    """The head-wise engine's gather on carracing rows (27648 floats: many float4 trips per row)."""
    from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config
    ccfg = synth.CNN_CONFIGS["carracing"]
    t = synth.CONV_TYPES[ccfg["conv_type"]]
    B, cap, size = 64, 300, 257
    lim = torch.full((ccfg["act_dim"],), ccfg["act_lim"])
    eng = CnnEngine(make_cnn_config(ccfg["obs_dim"], ccfg["act_dim"], t["kernels"], t["channels"], t["strides"], t["heads"],
                                    max_batch=B), torch.device("cuda", 0), lim, -lim)
    eng.seed(SEED)
    O = int(np.prod(ccfg["obs_dim"]))
    host = ring_rows(dict(obs_dim=O, act_dim=ccfg["act_dim"], act_lim=1.0), cap)
    bind_ring(eng, host)
    for _ in range(2):
        c = counter(eng)
        got = eng.replay_sample(B, size)
        idx = replay_indices(SEED, c, B, size)
        np.testing.assert_array_equal(eng.arena_views(B)["idx"].cpu().numpy(), idx)
        assert counter(eng) == c + 1
        for k in ("obs", "obs2", "act", "rew", "done", "logp"):
            np.testing.assert_array_equal(got[k].reshape(B, -1).cpu().numpy().reshape(host[k][idx].shape), host[k][idx],
                                          err_msg=k)
    # the head-wise engine's device noise lands in the slots arena_views names
    c = counter(eng)
    eng.step({k: v.clone() for k, v in got.items()}, 0, None)
    assert counter(eng) == c + 1
    ref = device_noise(SEED, c, B, ccfg["act_dim"])
    v = eng.arena_views(B)
    for k, r in zip(("eps1", "eps2", "z3", "z4"), ref):
        d = np.abs(v[k].double().cpu().numpy() - r) / np.spacing(np.abs(r).astype(np.float32))
        assert d.max() <= NOISE_ULPS, (k, d.max())
    eng.close()


# ---- data-parallel replay step ------------------------------------------------------------------------------------------
DP_CFG, DP_ROWS = "halfcheetah", 96   # rows per rank


def _dp_worker(rank, world, port, out_dir, gemm):
    sys.path.insert(0, REPO)
    sys.path.insert(0, os.path.join(REPO, "tests"))
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from dsac_v2_b200 import dp
    from dsac_v2_b200.engine import Engine, make_config
    cfg, B = synth.CONFIGS[DP_CFG], DP_ROWS
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    eng = Engine(make_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], max_batch=B, gemm_mode=gemm),
                 torch.device("cuda", rank), lim, -lim)
    eng.load_weights(synth.make_weights(cfg))
    eng.seed(1000 + rank)   # as bench.py seeds its ranks
    host = ring_rows(cfg, 400, seed=50 + rank)
    with torch.cuda.device(rank):
        eng.bind_replay(400)
        eng.replay_add({k: torch.from_numpy(v).cuda(rank) for k, v in host.items()}, 400, 0)
    assert dp.connect_peers(eng, dist), "the ranks could not map each other's exchange buffers"
    ctrs, tbs = [], []
    for it in range(3):
        torch.cuda.synchronize(rank)
        ctrs.append(int(eng.state.view(torch.int32)[10].item()))
        eng.dp_replay_step(B, 390, it, B * world)
        s = eng.read_stats(B * world)
        tbs.append([s["Loss/Critic loss-RL iter"], s["Loss/Actor loss-RL iter"]])
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), params=eng.params.cpu().numpy(), targets=eng.targets.cpu().numpy(),
             tb=np.array(tbs), ctrs=np.array(ctrs), **{f"ring_{k}": v for k, v in host.items()})
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("gemm", ["fp32", "bf16x3"])
def test_dp_replay_step_equals_single_gpu(tmp_path, gemm, world):
    """dp_replay_step with device draws on every rank == one GPU's step on the concatenation of every rank's ring[idx] and
    noise, restated from each rank's seed and counter."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    port = 29700 + (os.getpid() + 17 * world) % 1000
    mp.spawn(_dp_worker, args=(world, port, str(tmp_path), gemm), nprocs=world, join=True)
    ranks = [np.load(tmp_path / f"rank{r}.npz") for r in range(world)]
    for r in ranks[1:]:
        np.testing.assert_array_equal(ranks[0]["params"], r["params"])
        np.testing.assert_array_equal(ranks[0]["targets"], r["targets"])
    cfg, B = synth.CONFIGS[DP_CFG], DP_ROWS
    A = cfg["act_dim"]
    streams = [[replay_indices(1000 + r, int(ranks[r]["ctrs"][it]), B, 390) for it in range(3)] for r in range(world)]
    for r in range(world):
        for q in range(r + 1, world):
            assert not np.array_equal(streams[r][0], streams[q][0]), (r, q)
    lim = torch.full((A,), cfg["act_lim"])
    from dsac_v2_b200.engine import Engine, make_config
    one = Engine(make_config(cfg["obs_dim"], A, cfg["hidden"], cfg["hidden"], max_batch=B * world, gemm_mode=gemm),
                 torch.device("cuda", 0), lim, -lim)
    one.load_weights(synth.make_weights(cfg))
    tbs = []
    for it in range(3):
        parts, noises = [], []
        for r in range(world):
            ring = {k[5:]: ranks[r][k] for k in ranks[r].files if k.startswith("ring_")}
            parts.append(rows(ring, streams[r][it]))
            noises.append(device_noise(1000 + r, int(ranks[r]["ctrs"][it]), B, A))
        full = {k: torch.from_numpy(np.concatenate([p[k] for p in parts])).cuda() for k in parts[0]}
        nz = tuple(torch.from_numpy(np.concatenate([n[i] for n in noises]).astype(np.float32)).cuda() for i in range(4))
        one.step(full, it, nz)
        s = one.read_stats()
        tbs.append([s["Loss/Critic loss-RL iter"], s["Loss/Actor loss-RL iter"]])
    tol = 2e-5 if gemm == "fp32" else 1e-4
    np.testing.assert_allclose(ranks[0]["tb"], np.array(tbs), rtol=tol, atol=1e-6)
    atol = 2e-6 if gemm == "fp32" else 1e-5
    np.testing.assert_allclose(ranks[0]["params"], one.params.cpu().numpy(), rtol=tol, atol=atol)
    one.close()
