"""Whole data-parallel updates of W = 2..8 ranks on one device: W handles on cuda:0 attached to each other's exchange
buffers (dsact_test_dp_attach), each rank's dsact_dp_step / dsact_dp_replay_step on its own stream.

- At <= 16 rows per rank every rank must equal, bit for bit, the split API on W more handles with the exchanges restated
  on the host in rank order (float32 sums of the std sums, the gradients and the 16 logged sums, minimum of the 2 minima).
- dsact_dp_replay_step equals dsact_dp_step on the rows at its indices, bit for bit.
- On 250 ragged global rows, the step-0 gradients meet the float64 oracle's gates (tests/gradcheck64.py) and the
  statistics match one handle on the whole batch.

The ranks' kernels spin on each other's flags, so the ranks must run concurrently on one device, which CUDA does not
promise.  Each case runs in a child process with eager module loading (a lazily loaded kernel can wait for the running,
spinning ones) and a 5 s exchange timeout; all inputs are on the device before the first rank is enqueued, nothing
between the W enqueues synchronises or runs a torch kernel, and every rank's error slot must be 0 afterwards."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORLDS = list(range(2, 9))
ST_STDSUM, ST_DP_ERR, ST_ACC = 4, 7, 16
# The MLP engine runs eagerly here: with captured graphs, a rank whose step needed a new graph did not start while the
# earlier ranks' graphs spun on its flags (their exchanges timed out naming it), so W captured ranks cannot share one device.
EXACT_VARIANTS = ["fp32_eager", "bf16x3_eager", "cnn_odd", "parameter"]


def _run_child(what, variant, worlds):
    """One child process runs `what` for every world size in `worlds` (one CUDA context, one torch import)."""
    env = dict(os.environ, CUDA_MODULE_LOADING="EAGER", DSACT_DP_TIMEOUT_MS="5000")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), what, variant, ",".join(map(str, worlds))], env=env, cwd=REPO,
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, f"child {what} {variant} exited with {p.returncode}:\n{p.stdout[-4000:]}\n{p.stderr[-6000:]}"
    print(p.stdout[-3000:])


@pytest.mark.parametrize("variant", EXACT_VARIANTS)
def test_dp_step_equals_the_split_api_with_host_exchanges_bit_for_bit(variant):
    _run_child("exact", variant, WORLDS)


def test_dp_replay_step_equals_dp_step_on_the_gathered_rows():
    _run_child("replay", "bf16x3_eager", [2, 5, 8])


@pytest.mark.parametrize("mode", ["fp32", "bf16x3"])
def test_ragged_dp_step_meets_the_float64_gates(mode):
    _run_child("ragged", mode, WORLDS)


# ---- the child process ----------------------------------------------------------------------------------------------
def _bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.int32)


def _same(a, b, what):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    bad = np.flatnonzero(_bits(a) != _bits(b))
    assert bad.size == 0, f"{what}: {bad.size} of {a.size} differ, first at {bad[:6]}: {a.ravel()[bad[:3]]} vs {b.ravel()[bad[:3]]}"


def _stats(e, gb):
    """The 16 statistics over gb rows (dsact_read_stats), read once the copy has landed."""
    import torch
    out = e.read_stats_async(gb)
    torch.cuda.synchronize()
    return out.numpy().copy()


def _rank_sum(xs):
    acc = np.array(xs[0], np.float32)
    for x in xs[1:]:
        acc = (acc + np.asarray(x, np.float32)).astype(np.float32)
    return acc


def _make(variant, max_batch):
    """(engine factory, config, batch maker) of one variant; the MLP engine's with graphs unless `_eager`."""
    import torch
    from dsac_v2_b200 import synth
    from dsac_v2_b200.engine import Engine, make_config
    from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config, make_heads_config
    h = synth.HYPER
    hyper = dict(gamma=h["gamma"], tau=h["tau"], delay_update=h["delay_update"], auto_alpha=h["auto_alpha"], alpha=h["alpha"],
                 lr_q=h["value_learning_rate"], lr_pi=h["policy_learning_rate"], lr_alpha=h["alpha_learning_rate"],
                 min_log_std=h["policy_min_log_std"], max_log_std=h["policy_max_log_std"])
    dev = torch.device("cuda", 0)
    if variant == "cnn_odd":
        cfg = synth.CNN_CONFIGS["odd"]
        t = synth.CONV_TYPES[cfg["conv_type"]]
        c = make_cnn_config(cfg["obs_dim"], cfg["act_dim"], t["kernels"], t["channels"], t["strides"], t["heads"], max_batch=max_batch, **hyper)
        lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
        w = synth.make_cnn_weights(cfg)
        new = lambda: CnnEngine(c, dev, lim, -lim)
        return new, cfg, synth.make_cnn_batch, w
    cfg = synth.CONFIGS["ragged"]
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    if variant == "parameter":
        c = make_heads_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], "parameter", max_batch=max_batch, **hyper)
        w = synth.make_weights_std(cfg, "parameter")
        return (lambda: CnnEngine(c, dev, lim, -lim)), cfg, synth.make_batch, w
    mode = variant.replace("_eager", "")
    c = make_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], max_batch=max_batch, gemm_mode=mode,
                    use_graph=not variant.endswith("_eager"), **hyper)
    return (lambda: Engine(c, dev, lim, -lim)), cfg, synth.make_batch, synth.make_weights(cfg)


def _world(new, weights, W):
    engs = [new() for _ in range(W)]
    for e in engs:
        e.load_weights(weights)
        e.dp_export()
    for r, e in enumerate(engs):
        e.test_dp_attach(r, engs)
    return engs


def _check_no_timeout(engs, what):
    import torch
    torch.cuda.synchronize()
    errs = [int(e.state[:16].view(torch.int32)[ST_DP_ERR]) for e in engs]
    if any(errs):
        raise AssertionError(f"{what}: an exchange timed out; slot 14 of every rank (1 + the rank it waited for, or 1 + world "
                             f"in the two-shot apply): {errs}")


def _dp_updates(engs, inputs, gb, it, streams):
    """Every rank's dp_step of iteration `it`, each on its own stream, with nothing in between; then one synchronise."""
    import torch
    for e, s, (shard, nz) in zip(engs, streams, inputs):
        with torch.cuda.stream(s):
            e.dp_step(shard, it, gb, nz)
    _check_no_timeout(engs, f"iteration {it}")


def _rows(B, W):
    from dsac_v2_b200 import dp
    return [hi - lo for lo, hi in (dp.shard_rows(B, r, W) for r in range(W))]


def _shards(make_batch, cfg, W, rows, it):
    """Ragged shards of the global batch: (device inputs per rank, global rows)."""
    import torch
    from dsac_v2_b200 import synth
    B = sum(rows)
    full, noise = make_batch(cfg, B, it), synth.make_noise(cfg, B, it)
    out, lo = [], 0
    for n in rows:
        shard = {k: torch.from_numpy(np.ascontiguousarray(v[lo:lo + n])).cuda() for k, v in full.items()}
        nz = tuple(torch.from_numpy(np.ascontiguousarray(noise[i][lo:lo + n])).cuda() for i in (0, 1, 4, 5))
        out.append((shard, nz))
        lo += n
    assert _rows(B, len(rows)) == list(rows)
    return out, B


def child_exact(variant, W):
    import torch
    rows = _rows(16 * W - W // 2, W)   # ragged shards of 16 and 15 rows
    new, cfg, make_batch, w = _make(variant, 16)
    engs = _world(new, w, W)
    refs = [new() for _ in range(W)]
    for e in refs:
        e.load_weights(w)
    streams = [torch.cuda.Stream() for _ in range(W)]
    for it in range(3):   # delay_update = 2: the policy and the targets move at iterations 0 and 2
        inputs, gb = _shards(make_batch, cfg, W, rows, it)
        torch.cuda.synchronize()
        _dp_updates(engs, inputs, gb, it, streams)
        # the reference: the split API on every shard with the exchanges restated on the host
        for e, (shard, nz) in zip(refs, inputs):
            e.grad_phase1(shard, nz)
        std = _rank_sum([e.state[ST_STDSUM:ST_STDSUM + 2].cpu().numpy() for e in refs])
        for e in refs:
            e.state[ST_STDSUM:ST_STDSUM + 2] = torch.from_numpy(std).cuda()
            e.grad_phase2(gb)
        grads = _rank_sum([e.grads.cpu().numpy() for e in refs])
        sums = _rank_sum([e.state[ST_ACC:ST_ACC + 16].cpu().numpy() for e in refs])
        mins = np.stack([e.state[ST_ACC + 16:ST_ACC + 18].cpu().numpy() for e in refs])
        mins = np.minimum.reduce(mins, axis=0).astype(np.float32)
        for e in refs:
            e.grads.copy_(torch.from_numpy(grads))
            e.state[ST_ACC:ST_ACC + 16] = torch.from_numpy(sums).cuda()
            e.state[ST_ACC + 16:ST_ACC + 18] = torch.from_numpy(mins).cuda()
            e.apply(it)
        want_stats = _stats(refs[0], gb)
        for r, (e, ref) in enumerate(zip(engs, refs)):
            tag = f"{variant} W={W} iteration {it} rank {r}"
            for k in ("params", "targets", "adam_m", "adam_v", "grads"):
                _same(getattr(e, k).cpu().numpy(), getattr(ref, k).cpu().numpy(), f"{tag} {k}")
                _same(getattr(e, k).cpu().numpy(), getattr(engs[0], k).cpu().numpy(), f"{tag} {k} against rank 0")
            _same(_stats(e, gb), want_stats, f"{tag} read_stats")
    print(f"exact {variant} W={W}: 3 updates bit-identical to the split API with host exchanges")


def child_replay(variant, W):
    import torch
    rows = _rows(16 * W - W // 2, W)
    new, cfg, make_batch, w = _make(variant, 16)
    a, b = _world(new, w, W), _world(new, w, W)
    cap = 64
    ring = make_batch(cfg, cap, 99)
    for e in a:
        e.bind_replay(cap)
        e.replay_add({k: torch.from_numpy(v).cuda() for k, v in ring.items()}, cap, 0)
    streams = [torch.cuda.Stream() for _ in range(W)]
    g = np.random.default_rng(W)
    for it in range(3):
        gb = sum(rows)
        noise = synth_noise(cfg, gb, it)
        idx = [torch.from_numpy(g.integers(0, cap, n)).cuda() for n in rows]
        nzs, lo = [], 0
        for n in rows:
            nzs.append(tuple(torch.from_numpy(np.ascontiguousarray(noise[i][lo:lo + n])).cuda() for i in (0, 1, 4, 5)))
            lo += n
        gathered = [({k: torch.from_numpy(np.ascontiguousarray(v[i.cpu().numpy()])).cuda() for k, v in ring.items()}, nz)
                    for i, nz in zip(idx, nzs)]
        torch.cuda.synchronize()
        for e, s, i, nz, n in zip(a, streams, idx, nzs, rows):
            with torch.cuda.stream(s):
                e.dp_replay_step(n, cap, it, gb, idx=i, noise=nz)
        _check_no_timeout(a, f"dp_replay_step iteration {it}")
        _dp_updates(b, gathered, gb, it, streams)
        for r, (x, y) in enumerate(zip(a, b)):
            tag = f"replay {variant} W={W} iteration {it} rank {r}"
            for k in ("params", "targets", "adam_m", "adam_v", "grads"):
                _same(getattr(x, k).cpu().numpy(), getattr(y, k).cpu().numpy(), f"{tag} {k}")
            _same(_stats(x, gb), _stats(y, gb), f"{tag} read_stats")
    print(f"replay {variant} W={W}: dp_replay_step == dp_step on the gathered rows")


def synth_noise(cfg, B, it):
    from dsac_v2_b200 import synth
    return synth.make_noise(cfg, B, it)


def child_ragged(mode, W):
    import torch
    import gradcheck64 as G
    from dsac_v2_b200.engine import Engine, make_config
    torch.set_num_threads(G.ORACLE_THREADS)
    name = "dp_ragged_b250"
    G.CASES[name] = G.Case(name, "mlp", "ragged", 250)
    case = G.CASES[name]
    assert not G.power_violations(name, mode), G.power_violations(name, mode)
    w, _, _ = G.inputs(case)
    B = case.batch
    rows = _rows(B, W)
    cfg = case.cfg
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    h = case.hyperparameters
    c = make_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], max_batch=max(rows), gemm_mode=mode, use_graph=False,
                    gamma=h["gamma"], tau=h["tau"], delay_update=h["delay_update"], auto_alpha=h["auto_alpha"], alpha=h["alpha"],
                    lr_q=h["value_learning_rate"], lr_pi=h["policy_learning_rate"], lr_alpha=h["alpha_learning_rate"],
                    min_log_std=h["policy_min_log_std"], max_log_std=h["policy_max_log_std"])
    engs = _world(lambda: Engine(c, torch.device("cuda", 0), lim, -lim), w, W)
    one = Engine(make_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], max_batch=B, gemm_mode=mode,
                             gamma=h["gamma"], tau=h["tau"], delay_update=h["delay_update"], auto_alpha=h["auto_alpha"],
                             alpha=h["alpha"], lr_q=h["value_learning_rate"], lr_pi=h["policy_learning_rate"],
                             lr_alpha=h["alpha_learning_rate"], min_log_std=h["policy_min_log_std"],
                             max_log_std=h["policy_max_log_std"]), torch.device("cuda", 0), lim, -lim)
    one.load_weights(w)
    streams = [torch.cuda.Stream() for _ in range(W)]
    from dsac_v2_b200 import synth
    keys = ("Loss/Critic loss-RL iter", "Loss/Actor loss-RL iter", "DSAC2/critic_avg_min_std1-RL iter", "DSAC2/mean_std1")
    tol = 2e-5 if mode == "fp32" else 1e-4
    for it in range(3):
        inputs, gb = _shards(synth.make_batch, cfg, W, rows, it)
        full, noise = synth.make_batch(cfg, B, it), synth.make_noise(cfg, B, it)
        whole = ({k: torch.from_numpy(v).cuda() for k, v in full.items()}, tuple(torch.from_numpy(noise[i]).cuda() for i in (0, 1, 4, 5)))
        torch.cuda.synchronize()
        _dp_updates(engs, inputs, gb, it, streams)
        if it == 0:   # every rank holds the global step-0 gradient
            r64 = G.reference(name)
            gates = G.gates(name, mode)
            got = engs[0].export_weights(grads=True)
            bad = {k: (G.rel(got[k], r64.g64[k]), gates[k]) for k in r64.g64 if not G.rel(got[k], r64.g64[k]) <= gates[k]}
            assert not bad, f"{mode} W={W}: step-0 gradients outside their float64 gates: {bad}"
        for e in engs[1:]:
            for k in ("params", "targets", "grads"):
                _same(getattr(e, k).cpu().numpy(), getattr(engs[0], k).cpu().numpy(), f"{mode} W={W} it {it} replica {k}")
        one.step(*whole[:1], it, whole[1])
        s1, sd = one.read_stats(), engs[0].read_stats(gb)
        for k in keys:
            assert abs(sd[k] - s1[k]) <= tol * abs(s1[k]) + 1e-6, (mode, W, it, k, sd[k], s1[k])
    print(f"ragged {mode} W={W} rows {rows}: gradients within the float64 gates, statistics match one handle")


if __name__ == "__main__":
    for p in (REPO, os.path.join(REPO, "dsac-v2_b200", "dropin"), os.path.join(REPO, "tests")):
        sys.path.insert(0, p)
    what, variant = sys.argv[1], sys.argv[2]
    for W in map(int, sys.argv[3].split(",")):
        {"exact": child_exact, "replay": child_replay, "ragged": child_ragged}[what](variant, W)
