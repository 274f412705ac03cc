"""The coded frame ring (dsact_replay_bind_coded_frames, `ReplayBuffer(dsact_replay_frames=K, dsact_replay_codes=True)`)
against the flat ring and the fp32 frame ring on the same stream of 8-bit quantised transitions: the same minibatches
bit for bit (fp32 rows and bf16 images, 16-code and scalar gather paths), the same replay-fed updates on the MLP engine
and the same CNN updates of DSAC-T type_2 and DSAC_V1 on poisoned workspaces, the checkpoint round trip, a refused
257th value, and the refusals of the C entry points."""
import ctypes as C

import numpy as np
import pytest
import torch

from dsac_v2_b200 import _lib, synth
from test_gpu_frame_replay import SEED, bits, heads_engine, same, transitions
from test_gpu_workspace import poison_workspace

pytestmark = pytest.mark.gpu

CARRACING_RAW = np.asarray(np.arange(256) / 255, dtype=np.float32)   # rgb / 255 of gym_carracingraw
# 256 values with both zeros: codes are matched on bit patterns
SIGNED = np.concatenate([np.linspace(-3, 3, 255, dtype=np.float32), np.float32([-0.0])])
assert len(np.unique(SIGNED.view(np.uint32))) == 256


def quantise(rows, levels):
    """The same transitions with every value replaced by one of `levels`, elementwise and deterministically, so that
    frames equal before stay equal."""
    q = lambda x: levels[(np.abs(x.astype(np.float64)) * 1e4).astype(np.int64) % len(levels)]
    return [(q(o), a, r, q(o2), d, lp) for o, a, r, o2, d, lp in rows]


def ring_triple(new_engine, obs_shape, A, cap, K, rows):
    """A flat ring, an fp32 frame ring and a coded frame ring ReplayBuffer on three fresh engines, all fed `rows`."""
    from training.replay_buffer import ReplayBuffer
    bufs = []
    for kind in ("flat", "frames", "coded"):
        eng = new_engine()
        eng.seed(SEED)
        kw = dict(obsv_dim=obs_shape, action_dim=A, buffer_max_size=cap)
        if kind != "flat":
            kw["dsact_replay_frames"] = K
        if kind == "coded":
            kw["dsact_replay_codes"] = True
        b = ReplayBuffer(**kw)
        b.attach(eng)
        for o, a, r, o2, d, lp in rows:
            b.store(o.reshape(obs_shape), {}, a, r, o2.reshape(obs_shape), d, lp, {})
        b.flush()
        bufs.append(b)
    torch.cuda.synchronize()
    return bufs


def vec_cfg(obs_dim):
    return dict(obs_dim=obs_dim, act_dim=3, hidden=(64, 64), act_lim=1.0)


def mlp_engine(mode, max_batch, cfg, fill=0.0, use_graph=True):
    from dsac_v2_b200.engine import Engine, make_config
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    c = make_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], max_batch=max_batch, gemm_mode=mode,
                    use_graph=use_graph)
    w = synth.make_weights(cfg)

    def new():
        e = Engine(c, torch.device("cuda", 0), lim, -lim, workspace_fill=fill)
        e.load_weights(w)
        return e
    return new


# ---- 1. the same stream into all three rings: the same minibatches ---------------------------------------------------------
# obs 64: F = 64 / K floats per frame, a multiple of 16 at K = 1 and 4 (16-code loads); obs 24: F = 24 and 6 (scalar path);
# small_t1: 2x44x44, F = 3872 at K = 1 (16-code loads)
ENGINES = [("fp32", 64), ("bf16x3", 64), ("bf16", 64), ("bf16x3", 24), ("small_t1", None), ("heads", None)]
STREAMS = [("shift", 1), ("stacked", 4), ("mixed", 1), ("mixed", 4)]


@pytest.mark.parametrize("stream,K", STREAMS)
@pytest.mark.parametrize("engine,obs", ENGINES)
def test_coded_ring_gathers_the_flat_and_frame_rings_minibatches(engine, obs, stream, K):
    Bmax, cap = 1025, 150
    if engine in ("small_t1", "heads"):
        new, shape, A = heads_engine(engine, Bmax)
        if engine == "small_t1" and K == 4:
            K = 1
    else:
        new, shape, A = mlp_engine(engine, Bmax, vec_cfg(obs)), (obs,), 3
    O = int(np.prod(shape))
    levels = CARRACING_RAW if engine == "small_t1" else SIGNED
    rows = quantise(transitions(stream, K, O, A, 3 * cap + 61, seed=K), levels)   # wraps the ring three times
    flat, fr, cr = ring_triple(new, shape, A, cap, K, rows)
    assert cr.coder.n <= 256 and cr.engine.replay["frames"].dtype == torch.uint8
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
    assert cr.__get_RAM__() < fr.__get_RAM__()


# ---- 2. whole replay-fed updates on the MLP engine, poisoned workspace ----------------------------------------------------
@pytest.mark.parametrize("mode", ["fp32", "bf16x3"])
@pytest.mark.parametrize("K", [1, 4])
def test_replay_steps_on_the_coded_ring_equal_the_flat_ring(mode, K):
    B, cap = 16, 120
    cfg = vec_cfg(64)
    new = mlp_engine(mode, B, cfg, fill=float("nan"))
    rows = quantise(transitions("mixed", K, cfg["obs_dim"], cfg["act_dim"], 3 * cap + 5, seed=3), SIGNED)
    flat, _, cr = ring_triple(new, (cfg["obs_dim"],), cfg["act_dim"], cap, K, rows)
    assert cr.coder.n > 200
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


# ---- 3. CNN updates of DSAC-T type_2 and DSAC_V1 on CarRacing-raw frames, poisoned workspace ----------------------------------
def carracing_raw_rows(shape, A, n, seed):
    """Episodes of CarRacing-raw observations made as the reference makes them: uint8 rgb -> float64 / 255 -> float32;
    obs_t = obs2_{t-1} within an episode of 7 steps."""
    g = np.random.default_rng(seed)
    C, H, W = shape
    frame = lambda: np.asarray(g.integers(0, 256, (H, W, C), dtype=np.uint8).transpose(2, 0, 1) / 255, dtype=np.float32)
    out, obs = [], frame()
    for t in range(n):
        nxt = frame()
        out.append((obs, g.uniform(-1, 1, A).astype(np.float32), float(g.standard_normal()), nxt, float(t % 7 == 6),
                    float(g.standard_normal())))
        obs = nxt if t % 7 != 6 else frame()
    return out


def close(a, b, exact, what):
    """Bit for bit, or (exact = False) to 1e-6 relative L2: the convolutions' weight gradients are block sums added by
    float atomics (csrc/conv.cuh), in an order that may differ between two engines on the same minibatch."""
    a, b = (torch.as_tensor(x).float().cpu() for x in (a, b))
    if exact:
        same(a, b, what)
        return
    a, b = a.double(), b.double()
    err = float((a - b).norm() / max(float(b.norm()), 1e-30))
    assert err <= 1e-6, (what, err)


# type_2 on 96x96 images: two engines' updates on the same minibatch differ in the last bits (float atomics); the small
# type_1 encoder's updates repeat bit for bit (test_gpu_frame_replay.py's trainer runs rely on that too)
@pytest.mark.parametrize("variant,exact", [("dsact_type2", False), ("v1_type1", True)])
def test_cnn_updates_on_the_coded_ring_equal_the_flat_ring(variant, exact):
    from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config
    name, algo = ("carracing", "DSAC_T") if variant == "dsact_type2" else ("small_t1", "DSAC_V1")
    cfg = synth.CNN_CONFIGS[name]
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
    rows = carracing_raw_rows(shape, A, cap + 13, seed=5)
    flat, _, cr = ring_triple(new, shape, A, cap, 1, rows)
    assert cr.coder.n == 256
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
        # DSAC_V1's tb_info is carried in 7 of the 16 slots; the others keep their cleared values (e.g. +inf minima)
        assert np.all(np.isfinite(sc if algo == "DSAC_T" else sc[[0, 2, 6, 8, 9, 10, 11]])), sc
    for k in ("params", "targets", "adam_m", "adam_v"):
        close(getattr(ef, k), getattr(ec, k), exact, f"{variant} {k}")


# ---- 4. the drop-in buffer: checkpoint round trip, a refused 257th value ------------------------------------------------------
def coded_buffer(cap, K, rows):
    from training.replay_buffer import ReplayBuffer
    e = mlp_engine("bf16x3", 64, vec_cfg(64))()
    e.seed(SEED)
    b = ReplayBuffer(obsv_dim=(64,), action_dim=3, buffer_max_size=cap, dsact_replay_frames=K, dsact_replay_codes=True)
    b.attach(e)
    for o, a, r, o2, d, lp in rows:
        b.store(o, {}, a, r, o2, d, lp, {})
    b.flush()
    torch.cuda.synchronize()
    return b


def ring_copy(b):
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in b.engine.replay.items()}


def test_state_dict_restores_codes_and_table_exactly():
    cap, K = 90, 4
    rows = quantise(transitions("mixed", K, 64, 3, 2 * cap + 17, seed=8), SIGNED)
    a = coded_buffer(cap, K, rows)
    st = a.state_dict()
    assert st["data"]["frames"].dtype == torch.uint8 and len(st["frame_coder"]["bits"]) == a.coder.n
    b = coded_buffer(cap, K, [])
    b.load_state_dict(st)
    torch.cuda.synchronize()
    assert b.coder.n == a.coder.n and np.array_equal(b.coder.bits, a.coder.bits)
    same(a.engine.replay["table"], b.engine.replay["table"], "device table")
    idx = torch.from_numpy(np.random.default_rng(3).integers(0, cap, 64))
    x, y = a.engine.replay_sample(64, cap, idx), b.engine.replay_sample(64, cap, idx)
    for k in ("obs", "obs2", "act", "rew", "done", "logp"):
        same(x[k], y[k], f"restored ring {k}")
    # and both go on coding the same way
    more = quantise(transitions("mixed", K, 64, 3, 30, seed=9), SIGNED)
    for buf in (a, b):
        for o, act, r, o2, d, lp in more:
            buf.store(o, {}, act, r, o2, d, lp, {})
        buf.flush()
    x, y = a.engine.replay_sample(64, cap, idx), b.engine.replay_sample(64, cap, idx)
    for k in ("obs", "obs2"):
        same(x[k], y[k], f"after more rows {k}")


def test_a_257th_value_leaves_the_ring_as_it_was():
    cap, K = 40, 1
    rows = quantise(transitions("shift", K, 64, 3, 60, seed=2), SIGNED)
    b = coded_buffer(cap, K, rows)
    assert b.coder.n == 256
    before, st = ring_copy(b), (b.ptr, len(b), b.coder.n, b.coder.bits.copy(), b.planner.state_dict())
    o, a, r, o2, d, lp = rows[-1]
    bad = o2.copy()
    bad[5] = 7.25
    with pytest.raises(ValueError, match="7.25"):
        b.store(o2, {}, a, r, bad, d, lp, {})
    b.flush()
    after = ring_copy(b)
    for k in before:
        same(before[k], after[k], f"ring {k} after the refused row")
    assert (b.ptr, len(b), b.coder.n) == st[:3] and np.array_equal(b.coder.bits, st[3])
    assert b.planner.state_dict()["next"] == st[4]["next"]


# ---- 5. refusals of the C entry points --------------------------------------------------------------------------------------
def test_refusals_before_any_copy():
    lib = _lib.load()
    e = mlp_engine("fp32", 8, vec_cfg(24))()
    A = 3
    dev = lambda *s: torch.zeros(*s, device="cuda")
    codes = torch.zeros(40, 6, dtype=torch.uint8, device="cuda")
    table = dev(256)
    keep = [codes, torch.zeros(10, 4, dtype=torch.int32, device="cuda"), torch.zeros(10, 4, dtype=torch.int32, device="cuda"),
            dev(10, A), dev(10), dev(10), dev(10)]
    rb = _lib.FrameReplay(*(t.data_ptr() for t in keep), 10, 40, 4)
    assert lib.dsact_replay_bind_coded_frames(e.h, C.byref(rb), None) == -1 and b"null table" in lib.dsact_last_error()
    bad_rb = _lib.FrameReplay(*(t.data_ptr() for t in keep), 10, 40, 5)
    assert lib.dsact_replay_bind_coded_frames(e.h, C.byref(bad_rb), table.data_ptr()) == -1
    assert b"divide" in lib.dsact_last_error()
    assert lib.dsact_replay_bind_coded_frames(e.h, C.byref(rb), table.data_ptr()) == 0
    host_tab = np.arange(256, dtype=np.float32) + 1
    good = torch.zeros(1, 4, dtype=torch.int32)
    rows = dict(act=dev(1, A), rew=dev(1), done=dev(1), logp=dev(1), obs_frames=good, obs2_frames=good)

    def add(c, n_frames, n_codes, tab=host_tab, frame_ptr=0):
        return lib.dsact_replay_add_coded_frames(e.h, c.data_ptr(), n_frames, frame_ptr,
                                                 None if tab is None else tab.ctypes.data, n_codes,
                                                 good.data_ptr(), good.data_ptr(),
                                                 *(rows[k].data_ptr() for k in ("act", "rew", "done", "logp")), 1, 0, None)
    staged = torch.full((41, 6), 3, dtype=torch.uint8)
    # each staged code at or above n_codes
    for pos in range(12):
        s = staged.clone()
        s.view(-1)[pos] = 4
        assert add(s, 2, 4) == -1 and b"n_codes" in lib.dsact_last_error(), pos
    assert add(staged, 2, 3) == -1                        # every code is 3
    assert add(staged, 2, 4, tab=None) == -1 and b"null table" in lib.dsact_last_error()
    assert add(staged, 2, 257) == -1 and add(staged, 2, -1) == -1
    assert add(staged, 41, 4) == -1 and b"n_frames" in lib.dsact_last_error()   # more frames than the store holds
    assert add(staged.cuda(), 2, 4) == -1 and b"host memory" in lib.dsact_last_error()
    torch.cuda.synchronize()
    assert not codes.any() and not table.any() and not keep[3].any(), "a refused call copied something"
    # the other rings' entry points refuse a coded ring, and a coded add refuses the other rings
    f32 = torch.zeros(2, 6, device="cuda")
    assert lib.dsact_replay_add_frames(e.h, f32.data_ptr(), 2, 0, good.data_ptr(), good.data_ptr(),
                                       *(rows[k].data_ptr() for k in ("act", "rew", "done", "logp")), 1, 0, None) == -3
    assert lib.dsact_replay_add(e.h, *([keep[3].data_ptr()] * 6), 1, 0, None) == -3
    assert add(staged, 2, 4, frame_ptr=39) == 0   # wraps: slots 39 and 0; table entries 0..3
    torch.cuda.synchronize()
    assert codes[39].eq(3).all() and codes[0].eq(3).all() and not codes[1:39].any()
    assert table[:4].tolist() == [1.0, 2.0, 3.0, 4.0] and not table[4:].any()
    e.bind_replay_frames(10, 40, 4)
    assert add(staged, 2, 4) == -3 and b"coded" in lib.dsact_last_error()
