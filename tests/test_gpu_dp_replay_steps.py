"""n data-parallel replay-fed updates in one call (dsact_dp_replay_steps, Engine.dp_replay_steps) on one device: W = 2..8
handles on cuda:0 attached to each other's exchange buffers (dsact_test_dp_attach), each rank on its own stream, with the
harness of tests/test_gpu_dp_one_device.py (eager engines in a child process, eager module loading, a 5 s exchange
timeout, every input on the device before the first rank is enqueued, every rank's error slot 0 afterwards).  The
second input set of the n-update call is allocated when a handle is attached, and the statistics blocks before the
enqueues: an allocation between the ranks' enqueues lets CUDA hold back the later ranks' work behind the earlier ranks'
spinning kernels.

- At <= 16 rows per rank, dp_replay_steps(n) for n = 1, 2, 5 equals n dp_replay_step calls bit for bit: parameters,
  targets, Adam moments, the whole state (exchange epoch, error flag, generator counter, iteration), the arrival flags of
  the exchange buffer, and every statistics row against dsact_read_stats after the matching single call.  With host
  indices and noise, and with device draws.  W = 2..8 covers the one-shot and the two-shot gradient exchange.
- On 250 ragged global rows, the step-0 gradients meet the float64 oracle's gates (tests/gradcheck64.py), the replicas
  stay bit-identical, and the statistics rows match one handle stepping the whole batch.
- Every refusal of the call returns its siblings' message and launches nothing."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORLDS = list(range(2, 9))
CALLS = (1, 2, 5)    # consecutive calls: iterations 0, 1-2, 3-7 (delay_update = 2: both phases of the delayed update)
DP_FLAG_WORDS = 96   # the exchange buffer's arrival flags (csrc/dp_peer.cuh); word 96 is the reduce-scatter's ticket


def _run_child(what, variant, worlds):
    env = dict(os.environ, CUDA_MODULE_LOADING="EAGER", DSACT_DP_TIMEOUT_MS="5000")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), what, variant, ",".join(map(str, worlds))], env=env, cwd=REPO,
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, f"child {what} {variant} exited with {p.returncode}:\n{p.stdout[-4000:]}\n{p.stderr[-6000:]}"
    print(p.stdout[-3000:])


@pytest.mark.parametrize("variant", ["fp32_eager", "bf16x3_eager"])
def test_dp_replay_steps_equal_n_dp_replay_step_calls_bit_for_bit(variant):
    _run_child("exact", variant, WORLDS)


@pytest.mark.parametrize("mode", ["fp32", "bf16x3"])
def test_ragged_dp_replay_steps_meet_the_float64_gates(mode):
    _run_child("ragged", mode, WORLDS)


def test_refusals_launch_nothing():
    import torch
    from dsac_v2_b200 import _lib, synth
    from dsac_v2_b200.engine import Engine, make_config, make_v1_options
    from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config
    cfg, B = synth.CONFIGS["tiny"], 8
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    dev = torch.device("cuda", 0)

    def mk(policy_std="mlp_shared", v1=None):
        c = make_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], max_batch=B, gemm_mode="bf16x3",
                        use_graph=False, policy_std=policy_std)
        return Engine(c, dev, lim, -lim, v1=v1)

    def refused(e, match, *args, **kw):
        before = e.launch_count()
        with pytest.raises(_lib.DsactError, match=match):
            e.dp_replay_steps(*args, **kw)
        assert e.launch_count() == before, f"a refused call ({match}) launched {e.launch_count() - before} kernels"

    ccfg = synth.CNN_CONFIGS["small_t1"]
    t = synth.CONV_TYPES[ccfg["conv_type"]]
    clim = torch.full((ccfg["act_dim"],), ccfg["act_lim"])
    heads = CnnEngine(make_cnn_config(ccfg["obs_dim"], ccfg["act_dim"], t["kernels"], t["channels"], t["strides"], t["heads"], max_batch=5),
                      dev, clim, -clim)
    refused(heads, "head-wise", 2, 5, 10, 0, 10)
    heads.close()
    engs = {"v1": mk(v1=make_v1_options()), "separated": mk("mlp_separated"), "plain": mk()}
    for e in engs.values():
        e.bind_replay(32)
    refused(engs["v1"], "DSAC_V1", 2, B, 32, 0, 2 * B)
    refused(engs["separated"], "mlp_shared", 2, B, 32, 0, 2 * B)
    refused(engs["plain"], "dsact_dp_connect has not been called", 2, B, 32, 0, 2 * B)
    # a connected pair: the argument checks
    pair = [mk(), mk()]
    for e in pair:
        e.bind_replay(32)
        e.dp_export()
    for r, e in enumerate(pair):
        e.test_dp_attach(r, pair)
    for n in (0, 65):
        refused(pair[0], "n_steps", n, B, 32, 0, 2 * B)
    refused(pair[0], "global_batch", 2, B, 32, 0, B - 1)
    for e in list(engs.values()) + pair:
        e.close()


# ---- the child process ----------------------------------------------------------------------------------------------
def _world(new, weights, W, cap, ring):
    """W attached ranks with the ring bound and filled, each seeded with its own generator key; their exchange buffers."""
    import torch
    engs = [new() for _ in range(W)]
    for r, e in enumerate(engs):
        e.load_weights(weights)
        e.seed(1000 + r)
        e.dp_export()
        e.bind_replay(cap)
        e.replay_add({k: torch.from_numpy(v).cuda() for k, v in ring.items()}, cap, 0)
    bufs = [e.test_dp_attach(r, engs) for r, e in enumerate(engs)]
    return engs, bufs


def _stats_blocks(engs, n):
    """The [n, 16] statistics blocks dp_replay_steps writes, allocated before the ranks are enqueued (an allocation
    between the W enqueues could wait on the device while the ranks already enqueued spin on the later ones)."""
    import torch
    from dsac_v2_b200 import _lib
    for e in engs:
        e.__dict__.setdefault("_steps_stats", {}).setdefault(n, torch.zeros(n, _lib.NUM_STATS, device=e.device))


def child_exact(variant, W):
    import torch
    from test_gpu_dp_one_device import _check_no_timeout, _make, _rows, _same, _stats
    from dsac_v2_b200 import synth
    rows = _rows(16 * W - W // 2, W)   # ragged shards of 16 and 15 rows
    gb = sum(rows)
    new, cfg, make_batch, w = _make(variant, 16)
    cap, A = 64, cfg["act_dim"]
    ring = make_batch(cfg, cap, 99)
    streams = [torch.cuda.Stream() for _ in range(W)]
    for draws in ("host", "device"):
        (a, abufs), (b, bbufs) = _world(new, w, W, cap, ring), _world(new, w, W, cap, ring)
        g = np.random.default_rng(W)
        it = 0
        for n in CALLS:
            idx, nzs = [None] * W, [None] * W
            if draws == "host":
                idx = [torch.from_numpy(g.integers(0, cap, (n, m))).cuda() for m in rows]
                noise = [synth.make_noise(cfg, gb, it + k) for k in range(n)]
                nzs, lo = [], 0
                for m in rows:
                    nzs.append(tuple(torch.from_numpy(np.ascontiguousarray(np.stack([z[i][lo:lo + m] for z in noise]))).cuda()
                                     for i in (0, 1, 4, 5)))
                    lo += m
            _stats_blocks(a, n)
            torch.cuda.synchronize()
            out = []
            for e, s, i, nz, m in zip(a, streams, idx, nzs, rows):
                with torch.cuda.stream(s):
                    out.append(e.dp_replay_steps(n, m, cap, it, gb, idx=i, noise=nz))
            _check_no_timeout(a, f"{draws} dp_replay_steps({n}) from iteration {it}")
            got_rows = [o.cpu().numpy().copy() for o in out]
            want_rows = [[] for _ in range(W)]
            for k in range(n):
                for e, s, i, nz, m in zip(b, streams, idx, nzs, rows):
                    with torch.cuda.stream(s):
                        e.dp_replay_step(m, cap, it + k, gb, idx=None if i is None else i[k],
                                         noise=None if nz is None else tuple(x[k] for x in nz))
                _check_no_timeout(b, f"{draws} dp_replay_step iteration {it + k}")
                for r, e in enumerate(b):
                    want_rows[r].append(_stats(e, gb))
            for r in range(W):
                tag = f"{variant} {draws} W={W} dp_replay_steps({n}) from iteration {it} rank {r}"
                _same(got_rows[r], np.stack(want_rows[r]), f"{tag} statistics rows")
                assert got_rows[r][:, 14].max() == 0.0, f"{tag}: slot 14 {got_rows[r][:, 14]}"
                _stats(a[r], gb)   # the statistics slots of the state, as the single calls' last read_stats left them
                for k in ("params", "targets", "adam_m", "adam_v", "state"):
                    _same(getattr(a[r], k).cpu().numpy(), getattr(b[r], k).cpu().numpy(), f"{tag} {k}")
                _same(getattr(a[r], "params").cpu().numpy(), getattr(a[0], "params").cpu().numpy(), f"{tag} params against rank 0")
                _same(abufs[r][:DP_FLAG_WORDS].cpu().numpy(), bbufs[r][:DP_FLAG_WORDS].cpu().numpy(), f"{tag} arrival flags")
            it += n
        for e in a + b:
            e.close()
    print(f"exact {variant} W={W}: dp_replay_steps(1, 2, 5) == single dp_replay_step calls, host and device draws")


def child_ragged(mode, W):
    import torch
    import gradcheck64 as G
    from test_gpu_dp_one_device import _check_no_timeout, _rows, _same, _stats
    from dsac_v2_b200 import synth
    from dsac_v2_b200.engine import STAT_KEYS, Engine, make_config
    torch.set_num_threads(G.ORACLE_THREADS)
    name = "dp_ragged_b250"
    G.CASES[name] = G.Case(name, "mlp", "ragged", 250)
    case = G.CASES[name]
    assert not G.power_violations(name, mode), G.power_violations(name, mode)
    w, _, _ = G.inputs(case)
    B, cfg, h = case.batch, case.cfg, case.hyperparameters
    rows = _rows(B, W)
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    hyper = dict(gamma=h["gamma"], tau=h["tau"], delay_update=h["delay_update"], auto_alpha=h["auto_alpha"], alpha=h["alpha"],
                 lr_q=h["value_learning_rate"], lr_pi=h["policy_learning_rate"], lr_alpha=h["alpha_learning_rate"],
                 min_log_std=h["policy_min_log_std"], max_log_std=h["policy_max_log_std"])
    dev = torch.device("cuda", 0)
    n_it = 3
    fulls = [synth.make_batch(cfg, B, it) for it in range(n_it)]
    noises = [synth.make_noise(cfg, B, it) for it in range(n_it)]
    # rank r's ring: its shard of iteration 0's global batch, then of iteration 1's, ...; update k reads the k-th shard
    engs, idx, nzs, lo = [], [], [], 0
    for r, m in enumerate(rows):
        e = Engine(make_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], max_batch=max(rows), gemm_mode=mode,
                               use_graph=False, **hyper), dev, lim, -lim)
        e.load_weights(w)
        e.dp_export()
        e.bind_replay(n_it * m)
        e.replay_add({k: torch.from_numpy(np.ascontiguousarray(np.concatenate([f[k][lo:lo + m] for f in fulls]))).cuda()
                      for k in fulls[0]}, n_it * m, 0)
        idx.append(torch.arange(n_it * m, dtype=torch.int64, device=dev).view(n_it, m))
        nzs.append(tuple(torch.from_numpy(np.ascontiguousarray(np.stack([z[i][lo:lo + m] for z in noises]))).cuda()
                         for i in (0, 1, 4, 5)))
        engs.append(e)
        lo += m
    for r, e in enumerate(engs):
        e.test_dp_attach(r, engs)
    one = Engine(make_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], max_batch=B, gemm_mode=mode, **hyper),
                 dev, lim, -lim)
    one.load_weights(w)
    streams = [torch.cuda.Stream() for _ in range(W)]
    keys = [STAT_KEYS.index(k) for k in ("Loss/Critic loss-RL iter", "Loss/Actor loss-RL iter",
                                         "DSAC2/critic_avg_min_std1-RL iter", "DSAC2/mean_std1")]
    tol = 2e-5 if mode == "fp32" else 1e-4
    got = []
    for first, n in ((0, 1), (1, n_it - 1)):   # the step-0 gradients are gated after the first call
        _stats_blocks(engs, n)
        torch.cuda.synchronize()
        out = []
        for e, s, i, nz, m in zip(engs, streams, idx, nzs, rows):
            with torch.cuda.stream(s):
                out.append(e.dp_replay_steps(n, m, n_it * m, first, B, idx=i[first:first + n],
                                             noise=tuple(x[first:first + n] for x in nz)))
        _check_no_timeout(engs, f"dp_replay_steps({n}) from iteration {first}")
        if first == 0:
            r64 = G.reference(name)
            gates = G.gates(name, mode)
            g = engs[0].export_weights(grads=True)
            bad = {k: (G.rel(g[k], r64.g64[k]), gates[k]) for k in r64.g64 if not G.rel(g[k], r64.g64[k]) <= gates[k]}
            assert not bad, f"{mode} W={W}: step-0 gradients outside their float64 gates: {bad}"
        rows_k = [o.cpu().numpy().copy() for o in out]
        for r in range(1, W):
            _same(rows_k[r], rows_k[0], f"{mode} W={W} statistics rows of rank {r}")
            for k in ("params", "targets", "grads", "adam_m", "adam_v"):
                _same(getattr(engs[r], k).cpu().numpy(), getattr(engs[0], k).cpu().numpy(), f"{mode} W={W} replica {r} {k}")
        got.extend(rows_k[0])
    for it in range(n_it):
        one.step({k: torch.from_numpy(v).cuda() for k, v in fulls[it].items()}, it,
                 tuple(torch.from_numpy(noises[it][i]).cuda() for i in (0, 1, 4, 5)))
        want = _stats(one, B)
        for c in keys:
            assert abs(got[it][c] - want[c]) <= tol * abs(want[c]) + 1e-6, (mode, W, it, c, got[it][c], want[c])
    for e in engs + [one]:
        e.close()
    print(f"ragged {mode} W={W} rows {rows}: step-0 gradients within the float64 gates, replicas identical, statistics "
          f"rows match one handle")


if __name__ == "__main__":
    for p in (REPO, os.path.join(REPO, "dsac-v2_b200", "dropin"), os.path.join(REPO, "tests")):
        sys.path.insert(0, p)
    what, variant = sys.argv[1], sys.argv[2]
    for W in map(int, sys.argv[3].split(",")):
        {"exact": child_exact, "ragged": child_ragged}[what](variant, W)
