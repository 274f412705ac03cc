"""The frame replay ring (dsact_frame_replay, `ReplayBuffer(dsact_replay_frames=K)`) against the flat ring on the same
stream of transitions: the same minibatches bit for bit on every engine, the same replay-fed steps (single, n per call,
data-parallel), the same trainer runs and resumes, and the refusals of the C entry points."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if __name__ == "__main__":   # the data-parallel child process
    sys.path[:0] = [REPO, os.path.join(REPO, "dsac-v2_b200", "dropin")]

from dsac_v2_b200 import _lib, synth  # noqa: E402

pytestmark = pytest.mark.gpu

SEED = 0x0123456789ABCDEF
VEC = dict(obs_dim=24, act_dim=3, hidden=(64, 64), act_lim=1.0)
HUMANOID = synth.CONFIGS["humanoid"]


# ---- streams and rings ------------------------------------------------------------------------------------------------
def transitions(kind, K, O, A, n, seed):
    """n transitions of random episodes (lengths 1-50).  kind: "stacked" (obs2 = obs shifted by one of its K frames),
    "shift" (obs_t = obs2_{t-1}), "none" (nothing shared), "mixed" (all three, episode by episode)."""
    g = np.random.default_rng(seed)
    F = O // K
    out = []
    while len(out) < n:
        k = kind if kind != "mixed" else ("stacked", "shift", "none")[g.integers(3)]
        length = int(g.integers(1, 51))
        frames = [g.standard_normal(F).astype(np.float32) for _ in range(1 if g.integers(2) else K)]
        stack = frames * K if len(frames) == 1 else frames    # a reset stack [f0] * K, or K distinct frames
        obs = np.concatenate(stack)
        for t in range(length):
            if k == "stacked":
                stack = stack[1:] + [g.standard_normal(F).astype(np.float32)]
                obs2 = np.concatenate(stack)
            else:
                obs2 = g.standard_normal(O).astype(np.float32)
            out.append((obs, g.uniform(-1, 1, A).astype(np.float32), float(g.standard_normal()), obs2,
                        float(t == length - 1), float(g.standard_normal())))
            obs = obs2 if k != "none" else g.standard_normal(O).astype(np.float32)
    return out[:n]


def ring_pair(new_engine, obs_shape, A, cap, K, rows):
    """A flat-ring and a frame-ring ReplayBuffer on two fresh engines, both fed `rows`."""
    from training.replay_buffer import ReplayBuffer
    bufs = []
    for frames in (None, K):
        eng = new_engine()
        eng.seed(SEED)
        kw = dict(obsv_dim=obs_shape, action_dim=A, buffer_max_size=cap)
        if frames is not None:
            kw["dsact_replay_frames"] = frames
        b = ReplayBuffer(**kw)
        b.attach(eng)
        for o, a, r, o2, d, lp in rows:
            b.store(o.reshape(obs_shape), {}, a, r, o2.reshape(obs_shape), d, lp, {})
        b.flush()
        bufs.append(b)
    torch.cuda.synchronize()
    return bufs


def bits(t):
    return t.detach().contiguous().view(torch.int32).cpu().numpy()


def same(a, b, what):
    x, y = bits(a), bits(b)
    bad = np.flatnonzero(x.ravel() != y.ravel())
    assert bad.size == 0, f"{what}: {bad.size} of {x.size} words differ, first at {bad[:6]}"


# ---- 1. the same stream into both rings: the same minibatches ----------------------------------------------------------
def mlp_engine(mode, max_batch, cfg=VEC, use_graph=True):
    from dsac_v2_b200.engine import Engine, make_config
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    c = make_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], max_batch=max_batch, gemm_mode=mode,
                    use_graph=use_graph)
    w = synth.make_weights(cfg)

    def new():
        e = Engine(c, torch.device("cuda", 0), lim, -lim)
        e.load_weights(w)
        return e
    return new


def heads_engine(kind, max_batch):
    from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config, make_heads_config
    if kind == "small_t1":
        cfg = synth.CNN_CONFIGS["small_t1"]
        t = synth.CONV_TYPES[cfg["conv_type"]]
        c = make_cnn_config(cfg["obs_dim"], cfg["act_dim"], t["kernels"], t["channels"], t["strides"], t["heads"],
                            max_batch=max_batch)
        shape, A = tuple(cfg["obs_dim"]), cfg["act_dim"]
    else:
        c = make_heads_config(VEC["obs_dim"], VEC["act_dim"], VEC["hidden"], "mlp_separated", max_batch=max_batch)
        shape, A = (VEC["obs_dim"],), VEC["act_dim"]
    lim = torch.full((A,), 1.0)
    return (lambda: CnnEngine(c, torch.device("cuda", 0), lim, -lim)), shape, A


ENGINES = ["fp32", "bf16x3", "bf16", "small_t1", "heads"]
# (stream, K): F = 24 / K floats per frame on the vector engines (F % 4 = 0 at K = 1 and 2, 6 at K = 4: the scalar path),
# F = 44 * 44 or twice that on the CNN engine
STREAMS = [("stacked", 2), ("stacked", 4), ("shift", 1), ("none", 2), ("mixed", 2)]


@pytest.mark.parametrize("stream,K", STREAMS)
@pytest.mark.parametrize("engine", ENGINES)
def test_frame_ring_gathers_the_flat_rings_minibatches(engine, stream, K):
    Bmax, cap = 1025, 150
    if engine in ("small_t1", "heads"):
        new, shape, A = heads_engine(engine, Bmax)
        if engine == "small_t1" and K == 4:
            K = 1   # two channels: one frame per observation
    else:
        new, shape, A = mlp_engine(engine, Bmax), (VEC["obs_dim"],), VEC["act_dim"]
    O = int(np.prod(shape))
    rows = transitions(stream, K, O, A, 3 * cap + 61, seed=K)   # wraps the ring three times
    flat, fr = ring_pair(new, shape, A, cap, K, rows)
    pl = fr.planner
    if stream in ("none", "mixed"):
        assert pl.frame_capacity > min(cap + cap // 16 + 2 * K, pl.max_frames), "the frame store never grew"
    ef, er = flat.engine, fr.engine
    g = np.random.default_rng(7)
    for B in (1, 7, 64, 1025):
        for draw in ("host", "device"):
            idx = torch.from_numpy(g.integers(0, cap, B)) if draw == "host" else None
            a = ef.replay_sample(B, cap, idx)
            b = er.replay_sample(B, cap, idx)
            torch.cuda.synchronize()
            tag = f"{engine} {stream} K={K} B={B} {draw}"
            for k in ("obs", "obs2", "act", "rew", "done", "logp"):
                same(a[k], b[k], f"{tag} {k}")
            same(ef.arena_views(B)["idx"], er.arena_views(B)["idx"], f"{tag} recorded indices")
            same(ef._ws_view, er._ws_view, f"{tag} workspace (arena rows and bf16 images)")
            if draw == "host":   # and against the rows stored
                want = np.stack([rows[len(rows) - cap + ((i - len(rows)) % cap)][0] for i in idx.numpy()])
                np.testing.assert_array_equal(a["obs"].reshape(B, -1).cpu().numpy(), want)


# ---- 2. whole replay-fed steps on the MLP engine ------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["fp32", "bf16x3"])
@pytest.mark.parametrize("K", [2, 4])   # F = 188 (float4 path) and 94 (scalar path)
def test_replay_steps_on_the_frame_ring_equal_the_flat_ring(mode, K):
    B, cap = 16, 120
    new = mlp_engine(mode, B, HUMANOID)
    rows = transitions("mixed", K, HUMANOID["obs_dim"], HUMANOID["act_dim"], 3 * cap + 5, seed=3)
    flat, fr = ring_pair(new, (HUMANOID["obs_dim"],), HUMANOID["act_dim"], cap, K, rows)
    ef, er = flat.engine, fr.engine
    g = np.random.default_rng(1)
    it = 0
    for rep in range(3):
        idx = torch.from_numpy(g.integers(0, cap, B)) if rep == 1 else None
        for e in (ef, er):
            e.replay_step(B, cap, it, idx=idx)
        it += 1
    idx8 = torch.from_numpy(g.integers(0, cap, (8, B)))
    for idx in (None, idx8):
        outs = [e.replay_steps(8, B, cap, it, idx=idx) for e in (ef, er)]
        torch.cuda.synchronize()
        same(outs[0], outs[1], f"K={K} {mode} replay_steps statistics")
        it += 8
    torch.cuda.synchronize()
    for k in ("params", "targets", "adam_m", "adam_v", "state"):
        same(getattr(ef, k), getattr(er, k), f"K={K} {mode} {k}")


def test_dp_replay_step_on_the_frame_ring_equals_the_flat_ring():
    env = dict(os.environ, CUDA_MODULE_LOADING="EAGER", DSACT_DP_TIMEOUT_MS="5000")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), "dp"], env=env, cwd=REPO, capture_output=True, text=True,
                       timeout=900)
    assert p.returncode == 0, f"child exited with {p.returncode}:\n{p.stdout[-4000:]}\n{p.stderr[-6000:]}"


def child_dp(W=2, K=4):
    """Two eager ranks on one device (dsact_test_dp_attach), twice: one world on the flat ring, one on the frame ring.
    Humanoid's observation and action with the small `ragged` layers: the ranks' spinning kernels must fit on the device
    side by side."""
    B, cap = 16, 100
    cfg = dict(synth.CONFIGS["ragged"], obs_dim=HUMANOID["obs_dim"], act_dim=HUMANOID["act_dim"])
    new = mlp_engine("bf16x3", B, cfg, use_graph=False)
    rows = transitions("mixed", K, cfg["obs_dim"], cfg["act_dim"], 3 * cap + 5, seed=9)
    worlds = [[], []]
    for r in range(W):
        flat, fr = ring_pair(new, (cfg["obs_dim"],), cfg["act_dim"], cap, K, rows)
        worlds[0].append(flat.engine)
        worlds[1].append(fr.engine)
    for w in worlds:
        for e in w:
            e.dp_export()
        for r, e in enumerate(w):
            e.test_dp_attach(r, w)
    streams = [torch.cuda.Stream() for _ in range(W)]
    g = np.random.default_rng(2)
    for it in range(3):
        idx = [torch.from_numpy(g.integers(0, cap, B)).cuda() for _ in range(W)]
        for w in worlds:
            torch.cuda.synchronize()
            for e, s, i in zip(w, streams, idx):
                with torch.cuda.stream(s):
                    e.dp_replay_step(B, cap, it, W * B, idx=i)
            torch.cuda.synchronize()
            assert all(int(e.state[:16].view(torch.int32)[7]) == 0 for e in w), "an exchange timed out"
        for r in range(W):
            for k in ("params", "targets", "adam_m", "adam_v", "grads"):
                same(getattr(worlds[0][r], k), getattr(worlds[1][r], k), f"dp iteration {it} rank {r} {k}")
    print("dp_replay_step on the frame ring == on the flat ring")


# ---- 3. through the drop-in trainer -------------------------------------------------------------------------------------
TRAINERS = {"v1_cnn": ("DSAC_V1", "small_t1", 2), "v2_mlp": ("DSAC_V2", "humanoid", 4)}


def make_trainer(variant, folder, frames, **extra):
    """An `OffSerialTrainer` fed by a frame-stacking stand-in sampler: each observation is K frames, the next one drops
    the oldest and appends a new frame; episodes of 13 steps start from a reset stack."""
    import dsac_v1
    import dsac_v2
    from training.replay_buffer import ReplayBuffer
    from training.trainer import create_trainer
    algo, cfg_name, K = TRAINERS[variant]
    mod = dsac_v1 if algo == "DSAC_V1" else dsac_v2
    cnn = cfg_name in synth.CNN_CONFIGS
    cfg = synth.CNN_CONFIGS[cfg_name] if cnn else synth.CONFIGS[cfg_name]
    np.random.seed(3)
    torch.manual_seed(3)
    kw = (synth.cnn_reference_kwargs if cnn else synth.reference_kwargs)(cfg, algorithm=algo, replay_batch_size=16, seed=11)
    kw = dict(kw, buffer_max_size=400, additional_info={}, buffer_name="replay_buffer", buffer_warm_size=60, max_iteration=16,
              log_save_interval=1000, apprfunc_save_interval=8, eval_interval=1000, save_folder=str(folder), ini_network_dir=None,
              use_gpu=True, dsact_tensorboard=False, **extra)
    if frames:
        kw["dsact_replay_frames"] = K
    alg = (mod.DSAC_V1 if algo == "DSAC_V1" else mod.DSAC_V2)(**kw)
    shape = tuple(cfg["obs_dim"]) if cnn else (cfg["obs_dim"],)
    fshape = (shape[0] // K,) + shape[1:]

    class Sampler:
        def __init__(self):
            self.networks = mod.ApproxContainer(**kw)
            self.n, self.t, self.g = 0, 0, np.random.default_rng(0)
            self.reset()

        def reset(self):
            self.stack = [self.g.random(fshape).astype(np.float32)] * K

        def sample(self):
            out = []
            for _ in range(20):
                obs = np.concatenate(self.stack)
                logits = self.networks.policy(torch.from_numpy(obs[None]))
                act, logp = self.networks.create_action_distributions(logits).sample()
                self.stack = self.stack[1:] + [np.clip(0.9 * self.stack[-1] + 0.1 * self.g.random(fshape), 0, 1).astype(np.float32)]
                nxt = np.concatenate(self.stack)
                self.t += 1
                done = self.t % 13 == 0
                out.append((obs, {}, act.detach()[0].numpy(), float(-np.abs(nxt - 0.5).mean()), nxt, done,
                            logp.detach()[0].numpy(), {}))
                if done:
                    self.reset()
            self.n += 20
            return out, {}

        def get_total_sample_number(self):
            return self.n

    class Evaluator:
        networks, calls = None, 0

        def run_evaluation(self, it):
            self.calls += 1
            return 0.0

    rec = []
    inner = alg.local_update

    def local_update(data, it):
        tb = inner(data, it)
        rec.append((it, sorted((k, float(v)) for k, v in tb.items() if "loss" in k.lower())))
        return tb

    alg.local_update = local_update
    return create_trainer(alg, Sampler(), ReplayBuffer(**kw), Evaluator(), **kw), alg, rec


def same_runs(alg_a, alg_b, what):
    sa, sb = alg_a.networks.state_dict(), alg_b.networks.state_dict()
    assert list(sa) == list(sb)
    for k in sa:
        assert torch.equal(sa[k], sb[k]), f"{what}: {k}"
    ea, eb = alg_a.networks.engine(), alg_b.networks.engine()
    for name in ("params", "targets", "adam_m", "adam_v"):
        same(getattr(ea, name), getattr(eb, name), f"{what}: {name}")


@pytest.mark.parametrize("variant", list(TRAINERS))
def test_trainer_on_the_frame_ring_equals_the_flat_ring(tmp_path, variant):
    # one run after the other: the samplers draw their actions from torch's global generator, seeded by make_trainer
    flat, alg_flat, rec_flat = make_trainer(variant, tmp_path / "flat", False, sample_interval=4)
    flat.train()
    fr, alg_fr, rec_fr = make_trainer(variant, tmp_path / "frames", True, sample_interval=4)
    fr.train()
    assert len(rec_fr) == 16 and rec_fr == rec_flat
    same_runs(alg_flat, alg_fr, variant)
    assert fr.buffer.__get_RAM__() < 0.75 * flat.buffer.__get_RAM__()


@pytest.mark.parametrize("variant", list(TRAINERS))
def test_frame_ring_full_checkpoint_resume_is_bit_identical(tmp_path, variant):
    full, alg_full, rec_full = make_trainer(variant, tmp_path / "full", True, dsact_full_checkpoint=True, sample_interval=1000)
    full.train()
    ck = tmp_path / "full" / "apprfunc" / "trainstate_8.pkl"
    resumed, alg_res, rec_res = make_trainer(variant, tmp_path / "resumed", True, dsact_full_checkpoint=True,
                                             sample_interval=1000, dsact_resume_dir=str(ck))
    assert resumed.iteration == 9
    resumed.train()
    assert rec_res == rec_full[9:]
    same_runs(alg_full, alg_res, variant)


# ---- 4. refusals ----------------------------------------------------------------------------------------------------------
def test_refusals_before_any_copy():
    lib = _lib.load()
    e = mlp_engine("fp32", 8)()
    O, A = VEC["obs_dim"], VEC["act_dim"]
    with pytest.raises(ValueError):
        e.bind_replay_frames(10, 40, 5)    # 5 does not divide 24
    with pytest.raises(ValueError):
        e.bind_replay_frames(10, 3, 4)     # frame_capacity < K
    dev = lambda *s: torch.zeros(*s, device="cuda")
    keep = [dev(40, 6), torch.zeros(10, 4, dtype=torch.int32, device="cuda"), torch.zeros(10, 4, dtype=torch.int32, device="cuda"),
            dev(10, A), dev(10), dev(10), dev(10)]
    ptrs = [t.data_ptr() for t in keep]

    def bind(K=4, fc=40, cap=10, null=None):
        p = list(ptrs)
        if null is not None:
            p[null] = None
        return lib.dsact_replay_bind_frames(e.h, C.byref(_lib.FrameReplay(*p, cap, fc, K)))
    assert bind(K=5) == -1 and b"divide" in lib.dsact_last_error()
    assert bind(K=65) == -1 and bind(K=0) == -1
    assert bind(fc=3) == -1 and b"frame_capacity" in lib.dsact_last_error()
    assert bind(fc=2 ** 31) == -1
    for i in range(7):
        assert bind(null=i) == -1 and b"null" in lib.dsact_last_error()
    assert bind() == 0
    frames = torch.full((2, 6), 7.0, device="cuda")
    rows = dict(act=dev(1, A), rew=dev(1), done=dev(1), logp=dev(1))
    good = torch.zeros(1, 4, dtype=torch.int32)
    for bad in ([0, 1, 40, 2], [0, -1, 0, 0]):
        ids = torch.tensor([bad], dtype=torch.int32)
        for which in ("obs_frames", "obs2_frames"):
            t = dict(rows, obs_frames=good, obs2_frames=good)
            t[which] = ids
            with pytest.raises(_lib.DsactError, match="frame-id table"):
                e.replay_add_frames(frames, 2, 0, t, 1, 0)
    # device-resident id tables are refused too: their ids cannot be checked before the copy
    rc = lib.dsact_replay_add_frames(e.h, frames.data_ptr(), 2, 0, keep[1].data_ptr(), keep[2].data_ptr(),
                                     *(rows[k].data_ptr() for k in ("act", "rew", "done", "logp")), 1, 0, None)
    assert rc == -1 and b"host memory" in lib.dsact_last_error()
    torch.cuda.synchronize()
    assert not keep[0].any(), "a refused call copied frames"
    assert lib.dsact_replay_add(e.h, *([keep[3].data_ptr()] * 6), 1, 0, None) == -3   # the flat entry point on a frame ring
    e.replay_add_frames(frames, 2, 39, dict(rows, obs_frames=good, obs2_frames=good), 1, 9)   # wraps: slots 39 and 0
    torch.cuda.synchronize()
    assert keep[0][39].eq(7).all() and keep[0][0].eq(7).all() and not keep[0][1:39].any()


if __name__ == "__main__":
    if sys.argv[1] == "dp":
        child_dp()
