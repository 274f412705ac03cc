"""n replay-fed updates in one call (`dsact_replay_steps`, Engine.replay_steps) against n single calls, the oracle and the
host restatement of the device generator; its graph reuse, workspace independence, refusals and the drop-in's
replay_updates.

Consecutive updates of one call alternate between two minibatch input sets and gather the next minibatch beside the
current backward; none of that may change a result: up to 16 rows the n-call is bit-identical to n single calls, above
that the float atomics of the bias gradients may sum in another order (the tolerances test_gpu_replay_step.py uses)."""
import os

import numpy as np
import pytest
import torch

from dsac_v2_b200 import _lib, synth
from oracle.dsact_rng import device_noise, replay_indices
from test_gpu_parity import RTOL, make_engine
from test_gpu_replay_step import SEED, bind_ring, counter, oracle_noise, rel_l2, ring_rows, rows
from test_gpu_workspace import poison_workspace
import v1_mlp_common as v1c

pytestmark = pytest.mark.gpu

MODES = ["fp32", "bf16x3", "bf16"]
NS = (1, 2, 3, 8)
# (algorithm, config, batch)
CASES = {"tiny": ("t", synth.CONFIGS["tiny"], 16), "ragged": ("t", synth.CONFIGS["ragged"], 37),
         "humanoid": ("t", synth.CONFIGS["humanoid"], 4096), "asym": ("t", synth.mlp_config("asym"), 70),
         "v1_hopper": ("v1", synth.EXAMPLE_CONFIGS["hopper"], 256), "v1_asym": ("v1", synth.mlp_config("asym"), 70)}
STATE_WORDS = (0, 1, 8, 9, 10, 11)   # mean_std1/2, Adam counters, Philox counter, iteration


def new_engine(case, mode, use_graph):
    algo, cfg, B = CASES[case]
    if algo == "v1":
        eng = v1c.make_engine(cfg, B, dict(synth.HYPER), gemm=mode, graph=use_graph)
    else:
        eng = make_engine(cfg, B, use_graph=use_graph, gemm_mode=mode)
    eng.seed(SEED)
    return eng


def twin(case, mode, use_graph):
    """Two engines from the same start state on the same ring."""
    _, cfg, B = CASES[case]
    host = ring_rows(cfg, B + 3 * B // 4 + 8)
    a, b = new_engine(case, mode, use_graph), new_engine(case, mode, use_graph)
    bind_ring(a, host)
    bind_ring(b, host)
    return cfg, B, a, b, host, host["obs"].shape[0] - 5


def raw_stats(eng, B):
    out = eng.read_stats_async(B)
    torch.cuda.synchronize()
    return out.clone().numpy()


def state_words(eng):
    torch.cuda.synchronize()
    return eng.state.view(torch.int32)[list(STATE_WORDS)].cpu().numpy()


def compare(a, b, B, mode, what):
    tol = 1e-4 if mode == "bf16" else 1e-6
    torch.cuda.synchronize()
    for k in ("params", "targets", "adam_m", "adam_v"):
        ta, tb = getattr(a, k), getattr(b, k)
        if B <= 16:
            assert torch.equal(ta, tb), (what, k)
        else:
            assert rel_l2(ta, tb) <= tol, (what, k, rel_l2(ta, tb))
    wa, wb = state_words(a), state_words(b)
    np.testing.assert_array_equal(wa[2:], wb[2:], err_msg=f"{what}: counters / iteration")
    if B <= 16:
        np.testing.assert_array_equal(wa[:2], wb[:2], err_msg=f"{what}: mean_std")
    else:
        np.testing.assert_allclose(a.state[:2].cpu().numpy(), b.state[:2].cpu().numpy(), rtol=tol, err_msg=what)


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(CASES))
def test_replay_steps_equal_n_single_calls(case, mode, use_graph):
    """Device-drawn indices and noise, delay_update = 2 from an odd iteration: params, targets, Adam moments, the state
    words, the off_idx slot and every statistics row of one n-call against n replay_step calls from the same state."""
    cfg, B, a, b, host, size = twin(case, mode, use_graph)
    tol = 1e-4 if mode == "bf16" else 1e-6
    a.replay_step(B, size, 0)   # start at iteration 1
    b.replay_step(B, size, 0)
    it = 1
    for n in NS:
        singles = []
        for k in range(n):
            a.replay_step(B, size, it + k)
            singles.append(raw_stats(a, B))
        got = b.replay_steps(n, B, size, it)
        torch.cuda.synchronize()
        rows_b = got.cpu().numpy()
        assert rows_b.shape == (n, _lib.NUM_STATS)
        if B <= 16:
            np.testing.assert_array_equal(np.array(singles), rows_b, err_msg=f"n={n} stats rows")
        else:   # relative L2 per row: a logged value near zero moves by more than `tol` of itself.  DSAC_V1 leaves the
            # minima it does not log at +inf
            for k in range(n):
                fin = np.isfinite(singles[k][:14])
                np.testing.assert_array_equal(np.isfinite(rows_b[k, :14]), fin)
                assert rel_l2(torch.from_numpy(rows_b[k, :14][fin]), torch.from_numpy(singles[k][:14][fin])) <= tol, (n, k)
        np.testing.assert_array_equal(a.arena_views(B)["idx"].cpu().numpy(), b.arena_views(B)["idx"].cpu().numpy())
        compare(a, b, B, mode, f"n={n}")
        # dsact_read_stats after the n-call: the last update's statistics
        np.testing.assert_array_equal(raw_stats(b, B), rows_b[-1])
        if n == 1 and B <= 16:   # n = 1 is replay_step exactly
            np.testing.assert_array_equal(singles[0], rows_b[0])
        it += n
    a.close(); b.close()


@pytest.mark.parametrize("mode", ["fp32", "bf16x3"])
@pytest.mark.parametrize("case", ["tiny", "humanoid", "v1_hopper"])
def test_replay_steps_match_the_oracle(case, mode):
    """Host idx [n, B] and host noise [n, ...] through one 4-update call against the oracle on the ring's rows; then a
    device-drawn 3-update call against the oracle on the restated draws, its last indices and its counter."""
    from oracle.dsact_oracle import TB_KEYS, V1_TB_KEYS, from_config
    algo, cfg, B = CASES[case]
    B = min(B, 256)
    eng = v1c.make_engine(cfg, B, dict(synth.HYPER), gemm=mode) if algo == "v1" else make_engine(cfg, B, gemm_mode=mode)
    eng.seed(SEED)
    host = ring_rows(cfg, 400)
    bind_ring(eng, host)
    size = 390
    if algo == "v1":
        orc, keys, cols = v1c.v1_oracle(cfg, synth.make_weights_v1(cfg), **synth.HYPER), V1_TB_KEYS, [0, 2, 6, 8, 9, 10, 11]
    else:
        orc, keys, cols = from_config(cfg, synth.make_weights(cfg), **synth.HYPER), TB_KEYS, list(range(14))
    torch.set_num_threads(min(16, os.cpu_count() or 4))
    g = np.random.default_rng(7)
    n, it = 4, 0
    idx = g.integers(0, size, (n, B))
    ns = [synth.make_noise(cfg, B, 100 + k) for k in range(n)]
    pick = (0, 1, 3, 3) if algo == "v1" else (0, 1, 4, 5)
    nz = tuple(torch.from_numpy(np.stack([x[i] for x in ns])) for i in pick)
    got = eng.replay_steps(n, B, size, it, idx=torch.from_numpy(idx), noise=nz).cpu().numpy()
    for k in range(n):
        noise = ns[k] if algo == "t" else ns[k]
        ref = orc.update(rows(host, idx[k]), noise, it + k)
        np.testing.assert_allclose(got[k][cols], [ref[key] for key in keys], rtol=RTOL, atol=1e-5, err_msg=f"host draws, update {k}")
    it += n
    c0, n = counter(eng), 3
    got = eng.replay_steps(n, B, size, it).cpu().numpy()
    assert counter(eng) == c0 + n
    A = cfg["act_dim"]
    for k in range(n):
        ridx = replay_indices(SEED, c0 + k, B, size)
        e1, e2, z3, z4 = device_noise(SEED, c0 + k, B, A)
        noise = oracle_noise(e1, e2, z3, z4)
        if algo == "v1":   # DSAC_V1's oracle takes the target critic's draw at position 3
            noise[3] = noise[4]
        ref = orc.update(rows(host, ridx), noise, it + k)
        np.testing.assert_allclose(got[k][cols], [ref[key] for key in keys], rtol=RTOL, atol=1e-5, err_msg=f"device draws, update {k}")
        if k == n - 1:
            np.testing.assert_array_equal(eng.arena_views(B)["idx"].cpu().numpy(), ridx)
    torch.set_num_threads(4)
    eng.close()


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("mode", ["fp32", "bf16x3"])
def test_graph_reuse_size_iteration_and_launch_counts(mode, use_graph):
    """A second call continues counters and iteration; a replayed graph follows a changed ring size and start iteration;
    the launches of one n-call are those of n replay_step calls plus one statistics kernel per update."""
    _, cfg, B = CASES["ragged"]
    cfg, B, a, b, host, size = twin("ragged", mode, use_graph)
    a.replay_step(B, size, 0)
    single = a.last_call_launches()
    n = 3
    for s, it in ((size, 1), (size, 4), (size // 3, 7), (size, 20), (size // 3, 3)):   # same graph key throughout
        c = counter(b)
        out = b.replay_steps(n, B, s, it)
        assert b.last_call_launches() == n * single + n, (b.last_call_launches(), single)
        assert counter(b) == c + n
        assert int(b.state.view(torch.int32)[11].item()) == it + n
        np.testing.assert_array_equal(b.arena_views(B)["idx"].cpu().numpy(), replay_indices(SEED, c + n - 1, B, s))
        assert np.all(np.isfinite(out.cpu().numpy()[:, :14]))
    b.replay_steps(n, B, size, 30, stats=False)
    assert b.last_call_launches() == n * single
    a.close(); b.close()


@pytest.mark.parametrize("mode", ["fp32", "bf16x3"])
def test_poisoned_workspace_and_small_after_large(mode):
    """The caller's workspace NaN / +-1e30 before every call changes nothing (to the run-to-run spread of 256-row updates);
    a 16-row call after a 256-row one (the second input set holds the large call's rows) equals, bit for bit, a fresh
    handle's call from the same state."""
    _, cfg, B = CASES["humanoid"]
    B = 256
    host = ring_rows(cfg, 600)
    engs = []
    for poison in (None, float("nan"), 1e30, -1e30):
        e = make_engine(cfg, B, gemm_mode=mode)
        e.seed(SEED)
        bind_ring(e, host)
        if poison is not None:
            poison_workspace(e, poison)
        r = [e.replay_steps(3, B, 590, 0).clone()]
        if poison is not None:
            poison_workspace(e, poison)
        r.append(e.replay_steps(2, 16, 590, 3).clone())
        torch.cuda.synchronize()
        engs.append((e, torch.cat(r).cpu()))
    e0, r0 = engs[0]
    for e, r in engs[1:]:
        assert torch.isfinite(r[:, :14]).all()
        assert rel_l2(r[:, :14], r0[:, :14]) <= 1e-6
        assert rel_l2(e.params, e0.params) <= 1e-6
    # small after large vs a fresh handle fed the same small call from the same state
    f = make_engine(cfg, B, gemm_mode=mode)
    f.seed(SEED)
    bind_ring(f, host)
    f.replay_steps(3, B, 590, 0)
    torch.cuda.synchronize()
    g = make_engine(cfg, B, gemm_mode=mode)
    g.seed(SEED)
    bind_ring(g, host)
    for k in ("params", "targets", "adam_m", "adam_v", "state"):
        getattr(g, k).copy_(getattr(f, k))
    ra = f.replay_steps(2, 16, 590, 3).cpu().numpy()
    rb = g.replay_steps(2, 16, 590, 3).cpu().numpy()
    np.testing.assert_array_equal(ra, rb)
    for e, _ in engs:
        e.close()
    f.close(); g.close()


def test_refusals():
    from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config
    _, cfg, B = CASES["tiny"]
    eng = make_engine(cfg, B, gemm_mode="bf16x3")
    with pytest.raises(_lib.DsactError, match="not bound"):
        eng.replay_steps(2, B, 10, 0)
    bind_ring(eng, ring_rows(cfg, 40))
    for n in (0, 65):
        with pytest.raises(_lib.DsactError, match="n_steps"):
            eng.replay_steps(n, B, 30, 0)
    eng.replay_steps(64, B, 30, 0, stats=False)
    eng.close()
    ccfg = synth.CNN_CONFIGS["small_t1"]
    t = synth.CONV_TYPES[ccfg["conv_type"]]
    lim = torch.full((ccfg["act_dim"],), ccfg["act_lim"])
    h = CnnEngine(make_cnn_config(ccfg["obs_dim"], ccfg["act_dim"], t["kernels"], t["channels"], t["strides"], t["heads"], max_batch=5),
                  torch.device("cuda", 0), lim, -lim)
    with pytest.raises(_lib.DsactError, match="head-wise"):
        h.replay_steps(2, 5, 10, 0)
    h.close()


# ---- drop-in ------------------------------------------------------------------------------------------------------------
def _alg_and_buffer(kw, rows_):
    """An algorithm (initial weights from torch's generator seeded with 0) on the GPU and a ring holding `rows_`."""
    import dsac_v1
    import dsac_v2
    from training.replay_buffer import ReplayBuffer
    torch.manual_seed(0)
    alg = (dsac_v1.DSAC_V1 if kw["algorithm"] == "DSAC_V1" else dsac_v2.DSAC_V2)(**kw)
    alg.networks.cuda()
    buf = ReplayBuffer(**dict(kw, buffer_max_size=len(rows_), additional_info={}))
    buf.attach(alg.networks.engine())
    buf.add_batch(rows_)
    buf.flush()
    return alg, buf


def _ring(kw, n_rows):
    g = np.random.default_rng(4)
    O, A = kw["obsv_dim"], kw["action_dim"]
    shape = (O,) if np.isscalar(O) else tuple(O)
    draw = (lambda: g.random(shape).astype(np.float32)) if len(shape) > 1 else (lambda: g.standard_normal(shape).astype(np.float32))
    return [(draw(), {}, g.uniform(-1, 1, A).astype(np.float32), float(g.standard_normal()), draw(), bool(i % 7 == 0),
             np.float32(-1.0), {}) for i in range(n_rows)]


# (With device draws a round of sample_batch + local_update takes two generator counters, one for the indices and one for
# the noise, and a replay_updates update one, as dsact_replay_step does: the same distribution, other numbers.
# test_replay_steps_equal_n_single_calls covers that stream.)
DROPIN = {
    "mlp_reference": lambda: synth.reference_kwargs(synth.CONFIGS["tiny"], replay_batch_size=16, seed=5, dsact_noise="reference"),
    "mlp_numpy_idx": lambda: synth.reference_kwargs(synth.CONFIGS["ragged"], replay_batch_size=37, seed=5,
                                                    dsact_index_source="numpy", dsact_gemm="fp32"),
    "v1_mlp_reference": lambda: synth.reference_kwargs(synth.EXAMPLE_CONFIGS["hopper"], replay_batch_size=16, algorithm="DSAC_V1",
                                                       dsact_gemm="bf16x3", dsact_noise="reference", seed=5),
    "mlp_separated": lambda: synth.reference_kwargs(synth.CONFIGS["tiny"], replay_batch_size=16, policy_std_type="mlp_separated",
                                                    dsact_noise="reference"),
    "cnn_small_t1": lambda: synth.cnn_reference_kwargs(synth.CNN_CONFIGS["small_t1"], replay_batch_size=5, dsact_noise="reference"),
}


@pytest.mark.parametrize("name", list(DROPIN))
def test_dropin_replay_updates_equal_sample_and_local_update(name):
    """replay_updates(buffer, B, it, n) == n rounds of sample_batch + local_update from the same seeds: every update's
    tb_info and the final weights (the head-wise engine runs the rounds itself)."""
    kw = DROPIN[name]()
    B, n, it = kw["replay_batch_size"], 5, 3
    ring = _ring(kw, 3 * B + 11)
    a, abuf = _alg_and_buffer(kw, ring)
    b, bbuf = _alg_and_buffer(kw, ring)
    np.random.seed(21); torch.manual_seed(22)
    want = [dict(a.local_update(abuf.sample_batch(B), it + k)) for k in range(n)]
    np.random.seed(21); torch.manual_seed(22)
    got = b.replay_updates(bbuf, B, it, n)
    assert len(got) == n
    alg_time = "Time/Algorithm time [ms]-RL iter"
    for k in range(n):
        w, g = dict(want[k]), dict(got[k])
        assert set(w) == set(g), (k, set(w) ^ set(g))
        for key in w:
            if "Algorithm time" in key or key == alg_time:
                continue
            np.testing.assert_allclose(g[key], w[key], rtol=1e-6, atol=1e-7, err_msg=f"update {k}: {key}")
    ea, eb = a.networks.engine(), b.networks.engine()
    torch.cuda.synchronize()
    for k in ("params", "targets", "adam_m", "adam_v"):
        assert rel_l2(getattr(eb, k), getattr(ea, k)) <= 1e-6, k
