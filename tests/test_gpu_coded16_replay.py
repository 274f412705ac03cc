"""The 16-bit coded frame ring (dsact_replay_bind_coded16_frames, `ReplayBuffer(dsact_replay_frames=K,
dsact_replay_codes=16)`) against the flat ring and the fp32 frame ring on the same stream of stacked-grey CarRacing
values (the reference's rgb2gray over a palette of RGB colours: more than 256 and at most 65 536 distinct values): the
same minibatches bit for bit (fp32 rows and bf16 images, 8-code and scalar gather paths, codes from the table's first
and later entries), the same replay-fed updates on the MLP engine, the same CNN updates of DSAC-T type_2 on
4x96x96 stacked frames and of DSAC_V1 type_1 on poisoned workspaces, a captured replay step that stays valid while the
table grows, the checkpoint round trip and its refusal across ring kinds, and the refusals of the C entry points."""
import ctypes as C

import numpy as np
import pytest
import torch

from dsac_v2_b200 import _lib, synth
from test_gpu_coded_replay import close, mlp_engine, quantise, ring_copy, vec_cfg
from test_gpu_frame_replay import SEED, heads_engine, same, transitions
from test_gpu_workspace import poison_workspace

pytestmark = pytest.mark.gpu

FAR = 4096   # codes from here on are table entries past the first 16 KiB of its 256 KiB
# BASELINE config 5's source: gym_carracing, 4 stacked grey 96x96 frames, with the carracing type_2 encoder
STACKED4 = dict(obs_dim=(4, 96, 96), act_dim=3, act_lim=1.0, conv_type="type_2")


def grey(rgb):
    """The reference's rgb2gray (env_gym/gym_carracing_data.py): dot(rgb, [0.299, 0.587, 0.114]) / 128 - 1, float64,
    stored as float32 by the replay buffer."""
    return np.asarray(np.dot(rgb, [0.299, 0.587, 0.114]) / 128.0 - 1.0, dtype=np.float32)


def grey_levels(colours, seed=0):
    """The distinct grey values of a palette of `colours` random RGB colours, in random order, with both zeros."""
    g = np.random.default_rng(seed)
    v = np.unique(grey(g.integers(0, 256, (colours, 3))).view(np.uint32))
    v = np.concatenate([v[(v != 0) & (v != 0x80000000)], np.uint32([0, 0x80000000])])
    g.shuffle(v)
    return v.view(np.float32)


GREY = grey_levels(6000)
assert FAR < len(GREY) <= 65536


def rings(new_engine, obs_shape, A, cap, K, rows, kinds=("flat", "frames", "coded16")):
    """ReplayBuffers of the given kinds on fresh engines, all fed `rows`."""
    from training.replay_buffer import ReplayBuffer
    bufs = []
    for kind in kinds:
        eng = new_engine()
        eng.seed(SEED)
        kw = dict(obsv_dim=obs_shape, action_dim=A, buffer_max_size=cap)
        if kind != "flat":
            kw["dsact_replay_frames"] = K
        if kind == "coded16":
            kw["dsact_replay_codes"] = 16
        elif kind == "coded8":
            kw["dsact_replay_codes"] = True
        b = ReplayBuffer(**kw)
        b.attach(eng)
        for o, a, r, o2, d, lp in rows:
            b.store(o.reshape(obs_shape), {}, a, r, o2.reshape(obs_shape), d, lp, {})
        b.flush()
        bufs.append(b)
    torch.cuda.synchronize()
    return bufs


def codes_of(buf, x):
    codes, new = buf.coder.encode(x.cpu().numpy())
    assert len(new) == 0, "a gathered value the table does not hold"
    return codes


# ---- 1. the same stream into all three rings: the same minibatches ---------------------------------------------------------
# obs 64: F = 64 and 16 at K = 1 and 4 (8-code loads); obs 24: F = 24 (8-code loads) and 6 (scalar path); small_t1:
# 2x44x44, F = 3872 at K = 1 (8-code loads); heads: the head-wise engine on 24 floats
ENGINES = [("fp32", 64), ("bf16x3", 64), ("bf16", 64), ("bf16x3", 24), ("small_t1", None), ("heads", None)]
STREAMS = [("shift", 1), ("stacked", 4), ("mixed", 1), ("mixed", 4)]


@pytest.mark.parametrize("stream,K", STREAMS)
@pytest.mark.parametrize("engine,obs", ENGINES)
def test_coded16_ring_gathers_the_flat_and_frame_rings_minibatches(engine, obs, stream, K):
    Bmax, cap = 1025, 150
    if engine in ("small_t1", "heads"):
        new, shape, A = heads_engine(engine, Bmax)
        if engine == "small_t1" and K == 4:
            K = 1
    else:
        new, shape, A = mlp_engine(engine, Bmax, vec_cfg(obs)), (obs,), 3
    O = int(np.prod(shape))
    rows = quantise(transitions(stream, K, O, A, 3 * cap + 61, seed=K), GREY)   # wraps the ring three times
    flat, fr, cr = rings(new, shape, A, cap, K, rows)
    assert 256 < cr.coder.n <= 65536 and cr.engine.replay["frames"].dtype == torch.int16
    assert cr.coder.n > FAR or O < 64, "a stream that should bring more than FAR values"
    if stream == "mixed":
        assert cr.planner.frame_capacity > min(cap + cap // 16 + 2 * K, cr.planner.max_frames), "the frame store never grew"
    engines = [b.engine for b in (flat, fr, cr)]
    g = np.random.default_rng(7)
    for B in (1, 7, 64, 1025):
        for draw in ("host", "device"):
            idx = torch.from_numpy(g.integers(0, cap, B)) if draw == "host" else None
            out = [e.replay_sample(B, cap, idx) for e in engines]
            torch.cuda.synchronize()
            tag = f"{engine}/{obs} {stream} K={K} B={B} {draw}"
            for ref, name in ((0, "flat"), (1, "frame")):
                for k in ("obs", "obs2", "act", "rew", "done", "logp"):
                    same(out[ref][k], out[2][k], f"{tag} {k} against the {name} ring")
                same(engines[ref].arena_views(B)["idx"], engines[2].arena_views(B)["idx"], f"{tag} indices ({name})")
                same(engines[ref]._ws_view, engines[2]._ws_view, f"{tag} workspace: arena rows and bf16 images ({name})")
            if B == 1025 and cr.coder.n > FAR:
                c = codes_of(cr, torch.cat([out[2]["obs"], out[2]["obs2"]]))
                assert c.min() < FAR <= c.max(), f"{tag}: codes on one side of {FAR} only"
    # two bytes per frame value against four, and the table
    held = cr.planner.F * cr.planner.held()
    assert fr.planner.held() == cr.planner.held()
    assert cr.__get_RAM__() == pytest.approx(fr.__get_RAM__() - (2 * held - 4 * 65536) / 1e6)


# ---- 2. whole replay-fed updates on the MLP engine, poisoned workspace ----------------------------------------------------
@pytest.mark.parametrize("mode", ["fp32", "bf16x3"])
@pytest.mark.parametrize("K", [1, 4])
def test_replay_steps_on_the_coded16_ring_equal_the_flat_ring(mode, K):
    B, cap = 16, 120
    cfg = vec_cfg(64)
    new = mlp_engine(mode, B, cfg, fill=float("nan"))
    rows = quantise(transitions("mixed", K, cfg["obs_dim"], cfg["act_dim"], 3 * cap + 5, seed=3), GREY)
    flat, cr = rings(new, (cfg["obs_dim"],), cfg["act_dim"], cap, K, rows, kinds=("flat", "coded16"))
    assert cr.coder.n > FAR
    ef, ec = flat.engine, cr.engine
    g = np.random.default_rng(1)
    it = 0
    for rep in range(3):
        idx = torch.from_numpy(g.integers(0, cap, B)) if rep == 1 else None
        for e in (ef, ec):
            poison_workspace(e, float("nan"))
            e.replay_step(B, cap, it, idx=idx)
        it += 1
    idx8 = torch.from_numpy(g.integers(0, cap, (8, B)))
    for idx in (None, idx8):
        for e in (ef, ec):
            poison_workspace(e, float("nan"))
        outs = [e.replay_steps(8, B, cap, it, idx=idx) for e in (ef, ec)]
        torch.cuda.synchronize()
        same(outs[0], outs[1], f"K={K} {mode} replay_steps statistics")
        assert torch.isfinite(outs[1]).all()
        it += 8
    torch.cuda.synchronize()
    for k in ("params", "targets", "adam_m", "adam_v", "state"):
        same(getattr(ef, k), getattr(ec, k), f"K={K} {mode} {k}")


# ---- 3. a captured replay step stays valid while the table grows --------------------------------------------------------
def test_captured_replay_step_after_the_table_grows_equals_the_flat_ring():
    B, cap, K = 16, 100, 1   # (up to ~16 rows an update repeats bit for bit; larger ones differ in the last bits)
    cfg = vec_cfg(64)
    new = mlp_engine("bf16x3", B, cfg, fill=float("nan"))
    first = quantise(transitions("shift", K, 64, 3, cap, seed=11), GREY[:300])       # codes below 300
    flat, cr = rings(new, (64,), 3, cap, K, first, kinds=("flat", "coded16"))
    assert cr.coder.n <= 300
    ef, ec = flat.engine, cr.engine
    for e in (ef, ec):
        e.replay_step(B, cap, 0)   # captured here
        e.replay_step(B, cap, 1)
    torch.cuda.synchronize()
    frame_capacity = cr.planner.frame_capacity
    more = quantise(transitions("shift", K, 64, 3, 2 * cap, seed=12), GREY)          # overwrites every row
    for b in (flat, cr):
        for o, a, r, o2, d, lp in more:
            b.store(o, {}, a, r, o2, d, lp, {})
        b.flush()
    assert cr.coder.n > FAR and cr.planner.frame_capacity == frame_capacity, "the ring was bound again"
    for it in range(2, 6):
        for e in (ef, ec):
            poison_workspace(e, float("nan"))
            e.replay_step(B, cap, it)
        torch.cuda.synchronize()
        # (bf16x3 steps gather only the bf16 images: the rows come from the flat ring)
        idx = ec.arena_views(B)["idx"].cpu()
        same(idx, ef.arena_views(B)["idx"], f"step {it} indices")
        assert ((idx >= 0) & (idx < cap)).all(), idx
        c = codes_of(cr, torch.cat([ef.replay["obs"].cpu()[idx], ef.replay["obs2"].cpu()[idx]]))
        assert c.max() >= FAR, "the replayed step gathered no code the table gained after its capture"
    for k in ("params", "targets", "adam_m", "adam_v", "state"):
        same(getattr(ef, k), getattr(ec, k), f"after the table grew: {k}")


# ---- 4. CNN updates of DSAC-T type_2 on 4x96x96 stacked grey frames, and DSAC_V1 type_1, poisoned workspace ------------------
def stacked_grey_rows(shape, A, n, seed, colours=3000):
    """Episodes of stacked grey frames as the reference's CarRacing wrapper makes them: frames of a palette's colours
    through rgb2gray, obs2 = obs shifted by one frame, a reset stack [f0] * K every 9 steps."""
    g = np.random.default_rng(seed)
    Kc, H, W = shape
    pal = g.integers(0, 256, (colours, 3))
    frame = lambda: grey(pal[g.integers(0, colours, (H, W))])
    out, stack = [], [frame()] * Kc
    for t in range(n):
        nxt = stack[1:] + [frame()]
        out.append((np.stack(stack), g.uniform(-1, 1, A).astype(np.float32), float(g.standard_normal()), np.stack(nxt),
                    float(t % 9 == 8), float(g.standard_normal())))
        stack = nxt if t % 9 != 8 else [frame()] * Kc
    return out


# type_2 on 96x96 images: two engines' updates on the same minibatch differ in the last bits (float atomics); the small
# type_1 encoder's updates repeat bit for bit
@pytest.mark.parametrize("variant,exact", [("dsact_type2", False), ("v1_type1", True)])
def test_cnn_updates_on_the_coded16_ring_equal_the_flat_ring(variant, exact):
    from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config
    cfg, algo, K = (STACKED4, "DSAC_T", 4) if variant == "dsact_type2" else (synth.CNN_CONFIGS["small_t1"], "DSAC_V1", 2)
    t = synth.CONV_TYPES[cfg["conv_type"]]
    B, cap = 8, 40
    kw = {} if algo == "DSAC_T" else {"algo": "DSAC_V1"}
    c = make_cnn_config(cfg["obs_dim"], cfg["act_dim"], t["kernels"], t["channels"], t["strides"], t["heads"], max_batch=B, **kw)
    w = synth.make_cnn_weights(cfg) if algo == "DSAC_T" else synth.make_cnn_weights_v1(cfg)
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])

    def new():
        e = CnnEngine(c, torch.device("cuda", 0), lim, -lim, workspace_fill=float("nan"))
        e.load_weights(w)
        return e
    shape, A = tuple(cfg["obs_dim"]), cfg["act_dim"]
    rows = stacked_grey_rows(shape, A, cap + 13, seed=5)
    flat, cr = rings(new, shape, A, cap, K, rows, kinds=("flat", "coded16"))
    assert 256 < cr.coder.n <= 65536
    ef, ec = flat.engine, cr.engine
    g = np.random.default_rng(4)
    for it in range(4):
        idx = torch.from_numpy(g.integers(0, cap, B)) if it % 2 else None
        noise = synth.make_noise(cfg, B, it)
        nz = tuple(torch.from_numpy(noise[i]).cuda() for i in (0, 1, 4, 5))
        data = []
        for e in (ef, ec):
            poison_workspace(e, float("nan"))
            data.append(e.replay_sample(B, cap, idx))
        for k in data[0]:   # the update's whole input
            same(data[0][k], data[1][k], f"{variant} update {it} minibatch {k}")
        for e, d in zip((ef, ec), data):
            e.step(d, it, nz)
        torch.cuda.synchronize()
        sf, sc = (np.array(list(e.read_stats(B).values()), np.float32) for e in (ef, ec))
        close(sf, sc, exact, f"{variant} update {it} statistics")
        assert np.all(np.isfinite(sc if algo == "DSAC_T" else sc[[0, 2, 6, 8, 9, 10, 11]])), sc
    for k in ("params", "targets", "adam_m", "adam_v"):
        close(getattr(ef, k), getattr(ec, k), exact, f"{variant} {k}")


# ---- 5. the drop-in buffer: checkpoint round trip and ring kinds ------------------------------------------------------------
def buffer(cap, K, rows, codes=16):
    from training.replay_buffer import ReplayBuffer
    e = mlp_engine("bf16x3", 64, vec_cfg(64))()
    e.seed(SEED)
    kw = {} if codes is None else dict(dsact_replay_frames=K)
    if codes not in (None, "frames"):
        kw["dsact_replay_codes"] = codes
    b = ReplayBuffer(obsv_dim=(64,), action_dim=3, buffer_max_size=cap, **kw)
    b.attach(e)
    for o, a, r, o2, d, lp in rows:
        b.store(o, {}, a, r, o2, d, lp, {})
    b.flush()
    torch.cuda.synchronize()
    return b


def test_state_dict_restores_codes_and_table_exactly():
    cap, K = 90, 4
    rows = quantise(transitions("mixed", K, 64, 3, 2 * cap + 17, seed=8), GREY)
    a = buffer(cap, K, rows)
    st = a.state_dict()
    assert st["data"]["frames"].dtype == torch.int16 and len(st["frame_coder"]["bits"]) == a.coder.n > FAR
    b = buffer(cap, K, [])
    b.load_state_dict(st)
    torch.cuda.synchronize()
    assert b.coder.n == a.coder.n and np.array_equal(b.coder.bits, a.coder.bits)
    same(a.engine.replay["table"], b.engine.replay["table"], "device table")
    idx = torch.from_numpy(np.random.default_rng(3).integers(0, cap, 64))
    x, y = a.engine.replay_sample(64, cap, idx), b.engine.replay_sample(64, cap, idx)
    for k in ("obs", "obs2", "act", "rew", "done", "logp"):
        same(x[k], y[k], f"restored ring {k}")
    more = quantise(transitions("mixed", K, 64, 3, 30, seed=9), GREY[::-1])
    for buf in (a, b):
        for o, act, r, o2, d, lp in more:
            buf.store(o, {}, act, r, o2, d, lp, {})
        buf.flush()
    x, y = a.engine.replay_sample(64, cap, idx), b.engine.replay_sample(64, cap, idx)
    for k in ("obs", "obs2"):
        same(x[k], y[k], f"after more rows {k}")


def test_checkpoints_are_refused_across_ring_kinds():
    cap, K = 30, 4
    rows = quantise(transitions("stacked", K, 64, 3, 20, seed=4), GREY[:200])   # values every coded ring can hold
    kinds = (None, "frames", True, 16)
    states = {k: buffer(cap, K, rows, codes=k).state_dict() for k in kinds}
    for mine in kinds:
        b = buffer(cap, K, [], codes=mine)
        before = ring_copy(b)
        for theirs in kinds:
            if (mine == 16) == (theirs == 16) or 16 not in (mine, theirs):
                continue
            with pytest.raises(ValueError, match="ring kind"):
                b.load_state_dict(states[theirs])
            for k, v in ring_copy(b).items():
                same(before[k], v, f"{mine} buffer after refusing a {theirs} checkpoint: {k}")
            assert (b.ptr, len(b)) == (0, 0)
        b.load_state_dict(states[mine])
        assert len(b) == 20


def test_a_65537th_value_leaves_the_ring_as_it_was():
    cap, K = 40, 1
    levels = np.arange(65536, dtype=np.float32) / 7
    b = buffer(cap, K, [])
    fill = levels.reshape(-1, 64)
    for i in range(0, len(fill) - 1, 2):
        b.store(fill[i], {}, np.zeros(3), 0.0, fill[i + 1], 0.0, 0.0, {})
    b.flush()
    torch.cuda.synchronize()
    assert b.coder.n == 65536
    before, st = ring_copy(b), (b.ptr, len(b), b.coder.n, b.coder.bits.copy(), b.planner.state_dict())
    bad = fill[-1].copy()
    bad[5] = -7.25
    with pytest.raises(ValueError, match="-7.25"):
        b.store(fill[-1], {}, np.zeros(3), 0.0, bad, 0.0, 0.0, {})
    b.flush()
    after = ring_copy(b)
    for k in before:
        same(before[k], after[k], f"ring {k} after the refused row")
    assert (b.ptr, len(b), b.coder.n) == st[:3] and np.array_equal(b.coder.bits, st[3])
    assert b.planner.state_dict()["next"] == st[4]["next"]


# ---- 6. refusals of the C entry points --------------------------------------------------------------------------------------
def test_refusals_before_any_copy():
    lib = _lib.load()
    e = mlp_engine("fp32", 8, vec_cfg(24))()
    A = 3
    dev = lambda *s: torch.zeros(*s, device="cuda")
    codes = torch.zeros(40, 6, dtype=torch.int16, device="cuda")
    table = dev(65536)
    keep = [codes, torch.zeros(10, 4, dtype=torch.int32, device="cuda"), torch.zeros(10, 4, dtype=torch.int32, device="cuda"),
            dev(10, A), dev(10), dev(10), dev(10)]
    rb = _lib.FrameReplay(*(t.data_ptr() for t in keep), 10, 40, 4)
    assert lib.dsact_replay_bind_coded16_frames(e.h, C.byref(rb), None) == -1 and b"null table" in lib.dsact_last_error()
    bad_rb = _lib.FrameReplay(*(t.data_ptr() for t in keep), 10, 40, 5)
    assert lib.dsact_replay_bind_coded16_frames(e.h, C.byref(bad_rb), table.data_ptr()) == -1
    assert b"divide" in lib.dsact_last_error()
    assert lib.dsact_replay_bind_coded16_frames(e.h, C.byref(rb), table.data_ptr()) == 0
    host_tab = np.arange(65536, dtype=np.float32) + 1
    good = torch.zeros(1, 4, dtype=torch.int32)
    rows = dict(act=dev(1, A), rew=dev(1), done=dev(1), logp=dev(1), obs_frames=good, obs2_frames=good)
    args = lambda: (good.data_ptr(), good.data_ptr(), *(rows[k].data_ptr() for k in ("act", "rew", "done", "logp")), 1, 0,
                    None)

    def add(c, n_frames, n_codes, tab=host_tab, frame_ptr=0, fn=lib.dsact_replay_add_coded16_frames):
        return fn(e.h, c.data_ptr(), n_frames, frame_ptr, None if tab is None else tab.ctypes.data, n_codes, *args())
    staged = torch.full((41, 6), 3, dtype=torch.int16)
    big = staged.clone()
    big.view(torch.uint16).view(-1)[7] = 65535   # the largest code
    for pos in range(12):   # each staged code at or above n_codes
        s = staged.clone()
        s.view(-1)[pos] = 4
        assert add(s, 2, 4) == -1 and b"n_codes" in lib.dsact_last_error(), pos
    assert add(staged, 2, 3) == -1                        # every code is 3
    assert add(big, 2, 65535) == -1 and b"65535" in lib.dsact_last_error()
    assert add(staged, 2, 4, tab=None) == -1 and b"null table" in lib.dsact_last_error()
    assert add(staged, 2, 65537) == -1 and add(staged, 2, -1) == -1
    assert add(staged, 41, 4) == -1 and b"n_frames" in lib.dsact_last_error()   # more frames than the store holds
    assert add(staged.cuda(), 2, 4) == -1 and b"host memory" in lib.dsact_last_error()
    torch.cuda.synchronize()
    assert not codes.any() and not table.any() and not keep[3].any(), "a refused call copied something"
    # every other ring kind's add refuses a 16-bit ring
    f32 = torch.zeros(2, 6, device="cuda")
    assert lib.dsact_replay_add_frames(e.h, f32.data_ptr(), 2, 0, *args()) == -3
    assert b"dsact_replay_add_coded16_frames" in lib.dsact_last_error()
    assert add(staged.to(torch.uint8), 2, 4, fn=lib.dsact_replay_add_coded_frames) == -3
    assert lib.dsact_replay_add(e.h, *([keep[3].data_ptr()] * 6), 1, 0, None) == -3
    torch.cuda.synchronize()
    assert not codes.any() and not table.any() and not keep[3].any(), "a refused call copied something"
    assert add(big, 2, 65536, frame_ptr=39) == 0   # wraps: slots 39 and 0; the whole table
    torch.cuda.synchronize()
    assert codes[39].eq(3).all() and codes[0].view(torch.uint16).view(-1).tolist() == [3, 65535, 3, 3, 3, 3]
    assert not codes[1:39].any() and table.cpu().numpy().tolist() == host_tab.tolist()
    # and a 16-bit add refuses every other ring kind
    e.bind_replay_frames(10, 40, 4)
    assert add(staged, 2, 4) == -3 and b"16-bit coded" in lib.dsact_last_error()
    e.bind_replay_frames(10, 40, 4, coded=True)
    assert add(staged, 2, 4) == -3 and b"16-bit coded" in lib.dsact_last_error()
    e.bind_replay(10)
    assert add(staged, 2, 4) == -3
    assert not e.replay["obs"].any()
