"""Every step reads only workspace it wrote.  Engine P binds a workspace filled with poison and is poisoned again before
every call that starts an update; engine A runs the same calls on a zero-filled workspace.  P must match A and stay finite.
NaN shows any read of unwritten memory that reaches a result; +-1e30 shows the reads that comparisons or fminf would mask.
A stale-data pass runs a step at max_batch and then a smaller ragged step, against a fresh workspace running only the
small step from the same state: rows past B and image padding of the larger batch must not leak into the smaller one."""
import numpy as np
import pytest
import torch

from dsac_v2_b200 import synth
from test_gpu_parity import WIDE, make_engine, stats_vec
from test_gpu_replay_step import bind_ring, ring_rows, rows

pytestmark = pytest.mark.gpu

POISONS = [float("nan"), 1e30, -1e30]
SHAPES = {"tiny": (synth.CONFIGS["tiny"], 16), "ragged": (synth.CONFIGS["ragged"], 37),
          "humanoid": (synth.CONFIGS["humanoid"], 100), "wide": (WIDE, 40),
          # critics and policy of different shapes: arena slots sized from the wrong network read unwritten memory
          "asym": (synth.ASYM_CONFIGS["asym"], 70), "layered_q": (synth.ASYM_CONFIGS["layered_q"], 70)}
STATE = ("params", "targets", "adam_m", "adam_v")


def same(a, b, B, what):
    """Bit-identical up to 16 rows; above that the float atomics of the bias gradients may sum in another order."""
    if B <= 16:
        assert torch.equal(a, b) if torch.is_tensor(a) else np.array_equal(a, b), what
        return
    a = torch.as_tensor(a).double().cpu()
    b = torch.as_tensor(b).double().cpu()
    err = float((a - b).norm() / max(float(b.norm()), 1e-30))
    assert err <= 1e-6, (what, err)


def poison_workspace(eng, value):
    """Everything but the weight-gradient slabs, which dsact_bind zeroes and the steps keep (their bias entries are
    never written)."""
    ws, slabs = eng._ws_view, eng.arena_views()["slabs"]
    lo = slabs.data_ptr() - ws.data_ptr()
    ws[:lo // 4].fill_(value)
    ws[lo // 4 + slabs.numel():].fill_(value)


def run_mlp(eng, cfg, B, path, poison, host, size):
    """Three updates through `path`, the workspace poisoned before each call that starts one."""
    g = np.random.default_rng(9)
    stats = []
    for it in range(3):
        idx = g.integers(0, size, B)
        n = synth.make_noise(cfg, B, it)
        nz = tuple(torch.from_numpy(n[i]) for i in (0, 1, 4, 5))
        if poison is not None:
            poison_workspace(eng, poison)
        if path == "step":
            eng.step({k: torch.from_numpy(v).cuda() for k, v in rows(host, idx).items()}, it, nz)
        elif path == "replay_step":       # device-drawn indices and noise
            eng.replay_step(B, size, it)
        else:                             # replay_sample, then the step that consumes its minibatch and images
            data = eng.replay_sample(B, size)
            eng.step(data, it, tuple(x.cuda() for x in nz))
        stats.append(stats_vec(eng))
    torch.cuda.synchronize()
    return np.array(stats)


def mlp_engine(cfg, B, mode, use_graph, fill=0.0):
    from dsac_v2_b200.engine import Engine
    e = make_engine(cfg, B, use_graph=use_graph, gemm_mode=mode)
    if fill == 0.0:
        return e
    # the same configuration and weights, bound to a poisoned workspace
    p = Engine(e.cfg, e.device, e.act_high, e.act_low, workspace_fill=fill)
    p.load_weights(synth.make_weights(cfg))
    e.close()
    return p


@pytest.mark.parametrize("path", ["step", "replay_step", "sample"])
@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("mode", ["fp32", "bf16x3", "bf16"])
@pytest.mark.parametrize("name", list(SHAPES))
def test_poisoned_workspace_changes_nothing(name, mode, use_graph, path):
    cfg, B = SHAPES[name]
    host = ring_rows(cfg, 3 * B)
    size = 3 * B - 2
    engines = []
    for poison in [None] + POISONS:
        e = mlp_engine(cfg, B, mode, use_graph, 0.0 if poison is None else poison)
        e.seed(77)
        bind_ring(e, host)
        engines.append((poison, e, run_mlp(e, cfg, B, path, poison, host, size)))
    _, a, sa = engines[0]
    for poison, p, sp in engines[1:]:
        assert np.all(np.isfinite(sp)), (poison, sp)
        same(sp, sa, B, f"stats, poison {poison}")
        for k in STATE:
            assert torch.isfinite(getattr(p, k)).all(), (poison, k)
            same(getattr(p, k), getattr(a, k), B, f"{k}, poison {poison}")
    for _, e, _ in engines:
        e.close()


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("mode", ["fp32", "bf16x3", "bf16"])
@pytest.mark.parametrize("name,small", [("tiny", 9), ("ragged", 13), ("humanoid", 37), ("wide", 21)])
def test_smaller_batch_ignores_the_previous_larger_one(name, small, mode, use_graph):
    cfg, B = SHAPES[name]
    stale = make_engine(cfg, B, use_graph=use_graph, gemm_mode=mode)
    big = synth.make_batch(cfg, B, 0)
    n = synth.make_noise(cfg, B, 0)
    stale.step({k: torch.from_numpy(v).cuda() for k, v in big.items()}, 0, tuple(torch.from_numpy(n[i]) for i in (0, 1, 4, 5)))
    torch.cuda.synchronize()
    fresh = make_engine(cfg, B, use_graph=use_graph, gemm_mode=mode)
    for k in STATE + ("state",):
        getattr(fresh, k).copy_(getattr(stale, k))
    sb, sn = synth.make_batch(cfg, small, 1), synth.make_noise(cfg, small, 1)
    for e in (stale, fresh):
        e.step({k: torch.from_numpy(v).cuda() for k, v in sb.items()}, 1, tuple(torch.from_numpy(sn[i]) for i in (0, 1, 4, 5)))
    s_stale, s_fresh = stats_vec(stale), stats_vec(fresh)
    assert np.all(np.isfinite(s_stale))
    same(s_stale, s_fresh, small, "stats")
    for k in STATE:
        same(getattr(stale, k), getattr(fresh, k), small, k)
    stale.close(); fresh.close()


# ---- the head-wise engine ----------------------------------------------------------------------------------------------
def cnn_case(kind, B, fill):
    from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config, make_heads_config
    if kind == "cnn":
        cfg = synth.CNN_CONFIGS["small_t1"]
        t = synth.CONV_TYPES[cfg["conv_type"]]
        c = make_cnn_config(cfg["obs_dim"], cfg["act_dim"], t["kernels"], t["channels"], t["strides"], t["heads"], max_batch=B)
        w, batch = synth.make_cnn_weights(cfg), synth.make_cnn_batch
    else:
        cfg = synth.CONFIGS["ragged"]
        if kind == "separated":
            c = make_heads_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], "mlp_separated", max_batch=B)
        else:
            c = make_heads_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], "mlp_shared", max_batch=B, algo="DSAC_V1")
        w, batch = None, synth.make_batch
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    e = CnnEngine(c, torch.device("cuda", 0), lim, -lim, workspace_fill=fill)
    if w is None:   # the head-wise schema's weights: the engine's own initial parameters, made reproducible
        g = torch.Generator().manual_seed(4)
        init = (torch.rand(e.params.numel(), generator=g) - 0.5) * 0.2
        e.params.copy_(init)
        e.targets.copy_(init[:e.targets.numel()])
    else:
        e.load_weights(w)
    return cfg, e, batch


@pytest.mark.parametrize("kind,B", [("cnn", 5), ("cnn", 37), ("separated", 37), ("v1", 16), ("v1", 37)])
def test_headwise_poisoned_workspace_changes_nothing(kind, B):
    results = []
    for poison in [None] + POISONS:
        cfg, e, batch = cnn_case(kind, B, 0.0 if poison is None else poison)
        stats = []
        for it in range(3):
            n = synth.make_noise(cfg, B, it)
            if poison is not None:
                e.workspace.fill_(poison)
            e.step({k: torch.from_numpy(v) for k, v in batch(cfg, B, it).items()}, it, (n[0], n[1], n[4], n[5]))
            stats.append(list(e.read_stats().values()))
        if kind == "v1":   # the slots that carry DSAC_V1's tb_info; the others keep their cleared values (e.g. +inf minima)
            stats = [[row[c] for c in (0, 2, 6, 8, 9, 10, 11)] for row in stats]
        results.append((poison, e, np.array(stats)))
    _, a, sa = results[0]
    for poison, p, sp in results[1:]:
        assert np.all(np.isfinite(sp)), (poison, sp)
        same(sp, sa, B, f"stats, poison {poison}")
        for k in STATE:
            assert torch.isfinite(getattr(p, k)).all(), (poison, k)
            same(getattr(p, k), getattr(a, k), B, f"{k}, poison {poison}")
    for _, e, _ in results:
        e.close()


def test_headwise_bind_rejects_an_unaligned_workspace():
    import ctypes as C
    from dsac_v2_b200 import _lib
    _, e, _ = cnn_case("separated", 8, 0.0)
    ptrs = [t.data_ptr() for t in (e.params, e.targets, e.grads, e.adam_m, e.adam_v, e.act_high, e.act_low, e.state)]
    assert e.lib.dsact_bind(e.h, C.byref(_lib.Buffers(*ptrs, e._ws_view.data_ptr() + 4))) == -1
    assert b"256-byte aligned" in e.lib.dsact_last_error()
    e.close()
