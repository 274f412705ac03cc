"""The peer-memory data-parallel exchange kernels (csrc/dp_peer.cuh, apply_kernel<2>) with every rank of a world on one
device, against exact host restatements.  dsact_test_dp_attach points W handles of this process at each other's exchange
buffers; dsact_test_dp runs one operation through the step's own launch code.  Every sum the kernels form runs in a
fixed rank (or slab) order, so each result is restated in numpy float32 in that order and compared bit for bit.  Memory
a kernel must not write is poisoned first and checked afterwards."""
import numpy as np
import pytest
import torch

from step_ref import adam_layouts

pytestmark = pytest.mark.gpu

DP_FLAGS, DP_TICKET, DP_SMALL_OFF, DP_SMALL, DP_GRADS_OFF, MAX_RANKS = 128, 96, 128, 32, 2048, 8
ST_STDSUM, ST_DP_ERR, ST_TICKET, ST_DP_EPOCH, ST_ACC, ST_ADAM_SC = 4, 7, 14, 15, 16, 64
ACC_LOGP = 8
WORLDS = list(range(2, 9))
POISON = float("nan")


def bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.int32)


def assert_bits(got, want, msg=""):
    g, w = bits(got), bits(want)
    bad = np.flatnonzero(g != w)
    assert bad.size == 0, f"{msg}: {bad.size} elements differ, first at {bad[:8]}: got {np.asarray(got).ravel()[bad[:4]]}, " \
                          f"want {np.asarray(want).ravel()[bad[:4]]}"


def rank_sum(blocks):
    """float32 sum in rank order, one rounding per addition (the kernels' order)."""
    acc = np.array(blocks[0], dtype=np.float32)
    for b in blocks[1:]:
        acc = (acc + np.asarray(b, dtype=np.float32)).astype(np.float32)
    return acc


def rank_min(blocks):
    acc = np.array(blocks[0], dtype=np.float32)
    for b in blocks[1:]:
        acc = np.fmin(acc, np.asarray(b, dtype=np.float32))
    return acc


def mlp_engine(obs=5, act=2, hidden=(32, 32), **kw):
    from dsac_v2_b200.engine import Engine, make_config
    lim = torch.ones(act)
    return Engine(make_config(obs, act, list(hidden), list(hidden), max_batch=16, gemm_mode="fp32", use_graph=False, **kw),
                  torch.device("cuda", 0), lim, -lim)


def heads_engine(**kw):
    from dsac_v2_b200 import synth
    from dsac_v2_b200.engine_cnn import CnnEngine, make_heads_config
    cfg = synth.CONFIGS["ragged"]
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    return CnnEngine(make_heads_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], "parameter", max_batch=16, **kw),
                     torch.device("cuda", 0), lim, -lim)


def world(W, make):
    """W handles on cuda:0 attached to each other; (engines, their exchange buffers as float32 views)."""
    engs = [make() for _ in range(W)]
    for e in engs:
        e.dp_export()
    bufs = [e.test_dp_attach(r, engs) for r, e in enumerate(engs)]
    torch.cuda.synchronize()
    return engs, bufs


def small_slot(kind, par, src):
    return DP_SMALL_OFF + ((kind * 2 + par) * MAX_RANKS + src) * DP_SMALL


def set_int(state, slot, value):
    state.view(torch.int32)[slot] = int(np.array(value, dtype=np.uint32).view(np.int32))


def get_uint(t, slot):
    return int(t[slot:slot + 1].cpu().numpy().view(np.uint32)[0])


# ---- dp_exchange_kernel ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("start", [None, 0x7FFFFFFE, 0xFFFFFFFE])
@pytest.mark.parametrize("W", WORLDS)
def test_exchange_sums_and_minima_in_rank_order_across_epoch_wraparound(W, start):
    engs, bufs = world(W, mlp_engine)
    g = np.random.default_rng(1000 * W + (start or 0) % 997)
    e0 = 0 if start is None else start
    if start is not None:   # as if the ranks had completed exchanges up to epoch `start`
        for e, b in zip(engs, bufs):
            set_int(e.state, ST_DP_EPOCH, start)
            for slot in range(3 * 16):
                set_int(b, slot, start if slot % 16 < W else 0)
    for step in range(3):
        for kind in (0, 1):
            e = (e0 + step + 1) & 0xFFFFFFFF
            par, n = e & 1, (2 if kind == 0 else 18)
            src = ST_STDSUM if kind == 0 else ST_ACC
            pay = []
            for r, (eng, b) in enumerate(zip(engs, bufs)):
                st = g.standard_normal(80).astype(np.float32)
                st[src:src + n] = g.standard_normal(n).astype(np.float32) * 10.0 ** g.integers(-3, 4, n)
                if kind == 1:
                    st[ST_ACC + 16:ST_ACC + 18] = np.abs(st[ST_ACC + 16:ST_ACC + 18])   # minima of positive stds
                keep = eng.state.cpu().numpy()
                for slot in (ST_DP_ERR, ST_DP_EPOCH):
                    st[slot] = keep[slot]
                eng.state.copy_(torch.from_numpy(st))
                pay.append(st[src:src + n].copy())
                for s in range(MAX_RANKS):   # the other parity's payloads must be neither read nor written
                    b[small_slot(kind, 1 - par, s):small_slot(kind, 1 - par, s) + DP_SMALL] = float("nan")
            before = [(eng.state.cpu().numpy().copy(), b[:DP_GRADS_OFF].cpu().numpy().copy()) for eng, b in zip(engs, bufs)]
            engs[0].test_dp("exchange", kind=kind)
            want = rank_sum(pay)
            if kind == 1:
                want[16:18] = rank_min([p[16:18] for p in pay])
            for r, (eng, b) in enumerate(zip(engs, bufs)):
                st0, hd0 = before[r]
                st, hd = eng.state.cpu().numpy(), b[:DP_GRADS_OFF].cpu().numpy()
                tag = f"W={W} start={start} step {step} kind {kind} rank {r}"
                assert_bits(st[src:src + n], want, tag + " result")
                opened = (int(st0[ST_DP_EPOCH:ST_DP_EPOCH + 1].view(np.uint32)[0]) + (kind == 0)) & 0xFFFFFFFF
                assert get_uint(eng.state, ST_DP_EPOCH) == opened == e, tag + " epoch: +1 after kind 0, kept by kind 1"
                assert eng.state.view(torch.int32)[ST_DP_ERR].item() == 0, tag
                other = np.ones(80, bool)
                other[src:src + n] = False
                other[ST_DP_EPOCH] = False
                assert_bits(st[other], st0[other], tag + " other state slots")
                # every rank's payload and flag, in this rank's buffer
                for s in range(W):
                    assert_bits(hd[small_slot(kind, par, s):small_slot(kind, par, s) + n], pay[s], tag + f" payload of {s}")
                    assert get_uint(b, kind * 16 + s) == e, tag + f" flag of {s}"
                expect = hd0.copy()
                for s in range(W):
                    expect[small_slot(kind, par, s):small_slot(kind, par, s) + n] = pay[s]
                    expect.view(np.uint32)[kind * 16 + s] = e
                assert_bits(hd, expect, tag + " header outside this exchange's payloads and flags")
    for e in engs:
        e.close()


# ---- dp_grad_fold_kernel --------------------------------------------------------------------------------------------
def log_alpha_grad(acc_logp, rows, act_dim, global_batch):
    """-(acc + rows * te) * inv as the kernels form it: nvcc contracts rows * te + acc into one FFMA, then one FFMA with
    -0 forms the product with -inv (SASS of dp_grad_fold_kernel and phase2_tail_kernel).  The sum is exact in float64
    here (te = -act_dim, rows small), so rounding it once to float32 is the fused result."""
    inner = np.float32(float(rows) * float(np.float32(-act_dim)) + float(np.float32(acc_logp)))
    return np.float32(-inner) * np.float32(1.0 / global_batch)


@pytest.mark.parametrize("aligned", [True, False])
@pytest.mark.parametrize("tail", [True, False])
def test_fold_sums_slabs_in_order_and_forms_log_alpha(tail, aligned):
    engs, bufs = world(2, mlp_engine)
    eng, buf = engs[0], bufs[0]
    N = int(eng.layout.n_params)
    g = np.random.default_rng(7 + 2 * tail + aligned)
    eng.state[ST_ACC + ACC_LOGP] = float(np.float32(g.standard_normal() * 30))
    off = 0 if aligned else 1   # a grads / slab base one float off 16 bytes: every element takes the scalar path
    for nslabs in range(5):
        for n in (1, 2, 3, 4, 5, 6, 7, 1029, 1030, 1031, 1032, N - 3, N - 2, N - 1, N):
            stride = n + (-n % 4) + (4 if nslabs % 2 else 0) + (0 if aligned else 1)
            grads = torch.from_numpy(g.standard_normal(n + off).astype(np.float32)).cuda()
            slabs = torch.from_numpy(g.standard_normal(max(nslabs, 1) * stride + off).astype(np.float32)).cuda()
            buf.fill_(POISON)
            rows, gb = 16, 64
            eng.test_dp("fold", grads=grads[off:], slabs=slabs[off:], nslabs=nslabs, slab_stride=stride, n=n,
                        tail_rows=rows if tail else 0, global_batch=gb)
            gr, sl = grads[off:].cpu().numpy(), slabs[off:].cpu().numpy()
            want = rank_sum([gr] + [sl[k * stride:k * stride + n] for k in range(nslabs)])
            if tail:
                want[n - 1] = log_alpha_grad(eng.state[ST_ACC + ACC_LOGP].item(), rows, eng.cfg.act_dim, gb)
            got = buf.cpu().numpy()
            tag = f"nslabs {nslabs} n {n} stride {stride} tail {tail} aligned {aligned}"
            assert_bits(got[DP_GRADS_OFF:DP_GRADS_OFF + n], want, tag)
            assert np.isnan(got[:DP_GRADS_OFF]).all() and np.isnan(got[DP_GRADS_OFF + n:]).all(), tag + ": wrote outside [0, n)"
    for e in engs:
        e.close()


def test_fold_log_alpha_matches_the_split_steps_tail_kernel():
    """The data-parallel fold and phase2_tail_kernel (the split API's end of backward) give the same log_alpha gradient,
    bit for bit, on the same logged sum."""
    from dsac_v2_b200 import synth
    cfg = synth.CONFIGS["tiny"]
    engs, bufs = world(2, lambda: mlp_engine(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"]))
    eng = engs[0]
    B = 13
    batch = {k: torch.from_numpy(v).cuda() for k, v in synth.make_batch(cfg, B, 0).items()}
    noise = synth.make_noise(cfg, B, 0)
    nz = tuple(torch.from_numpy(noise[i]).cuda() for i in (0, 1, 4, 5))
    eng.load_weights(synth.make_weights(cfg))
    eng.grad_phase1(batch, nz)
    eng.grad_phase2(40)
    N = int(eng.layout.n_params)
    eng.test_dp("fold", grads=eng.grads, n=N, tail_rows=B, global_batch=40)
    torch.cuda.synchronize()
    assert_bits(bufs[0][DP_GRADS_OFF + N - 1:DP_GRADS_OFF + N].cpu().numpy(), eng.grads[N - 1:].cpu().numpy(), "log_alpha")
    want = log_alpha_grad(eng.state[ST_ACC + ACC_LOGP].item(), B, cfg["act_dim"], 40)
    assert_bits(eng.grads[N - 1:].cpu().numpy(), np.array([want]), "restated log_alpha")
    for e in engs:
        e.close()


# ---- dp_reduce_scatter_kernel ---------------------------------------------------------------------------------------
def slices(npad, W):
    """enqueue_dp_reduce_scatter's host slicing, in float4 groups: [lo, hi) of every rank (may be empty)."""
    groups = npad // 4
    per = (groups + W - 1) // W
    out = []
    for r in range(W):
        lo = per * r
        hi = lo + per if lo + per < groups else groups
        out.append((min(lo, groups), hi))
    return out


def test_reduce_scatter_host_slicing_has_empty_and_partial_slices():
    assert slices(36, 7) == [(0, 2), (2, 4), (4, 6), (6, 8), (8, 9), (9, 9), (9, 9)]
    assert slices(36, 8) == [(0, 2), (2, 4), (4, 6), (6, 8), (8, 9), (9, 9), (9, 9), (9, 9)]
    for W in WORLDS:
        s = slices(702760, W)
        assert s[0][0] == 0 and s[-1][1] == 702760 // 4 and all(a[1] == b[0] for a, b in zip(s, s[1:]))


@pytest.mark.parametrize("order", ["rank", "reverse"])
@pytest.mark.parametrize("W", WORLDS)
@pytest.mark.parametrize("net", ["smallest", "humanoid"])
def test_reduce_scatter_sums_every_slice_in_rank_order(net, W, order):
    if net == "smallest":   # 35 parameters: 9 float4 groups, so slices are partial or empty from 5 ranks up
        make = lambda: mlp_engine(1, 1, (2,))
    else:                   # 702759 parameters: several blocks per slice, each taking grid-stride trips
        make = lambda: mlp_engine(376, 17, (256, 256, 256))
    engs, bufs = world(W, make)
    n = int(engs[0].layout.n_params)
    npad = (n + 3) // 4 * 4
    red = DP_GRADS_OFF + npad
    sl = slices(npad, W)
    g = np.random.default_rng(W * 31 + (order == "reverse"))
    for epoch in (3, 4, 5):
        blocks = [g.standard_normal(npad).astype(np.float32) * np.float32(10.0 ** g.integers(-2, 3)) for _ in range(W)]
        for e, b, blk in zip(engs, bufs, blocks):
            set_int(e.state, ST_DP_EPOCH, epoch)
            b[DP_GRADS_OFF:red] = torch.from_numpy(blk).cuda()
            b[red:] = POISON
        torch.cuda.synchronize()
        want = rank_sum(blocks)
        done = np.zeros(npad // 4, bool)
        for r in (range(W) if order == "rank" else reversed(range(W))):
            engs[r].test_dp("reduce_scatter")
            lo, hi = sl[r]
            done[lo:hi] = True
            written = ~np.isnan(bufs[(r + 1) % W][red:].cpu().numpy().reshape(-1, 4)).any(axis=1)
            assert np.array_equal(written, done), f"W={W} rank {r}: the slice written is not [{lo}, {hi})"
        for r, b in enumerate(bufs):
            got = b.cpu().numpy()
            tag = f"{net} W={W} {order} epoch {epoch} rank {r}"
            assert_bits(got[red:], want, tag + " reduced block")
            for s in range(W):
                assert get_uint(b, 2 * 16 + s) == epoch, tag + f" kind-2 flag of {s}"
            assert get_uint(b, DP_TICKET) == 0, tag + " ticket"
            assert_bits(got[DP_GRADS_OFF:red], blocks[r], tag + " gradient block")
            assert engs[r].state.view(torch.int32)[ST_DP_ERR].item() == 0
    for e in engs:
        e.close()


# ---- apply_kernel<2> ------------------------------------------------------------------------------------------------
def _apply_layouts():
    return sorted({k[1]: v for k, v in adam_layouts().items() if not v[2]}.values())


def _apply_case(engine, layout, auto_alpha):
    if engine == "mlp":
        obs, h = layout[0], layout[1]
        return lambda: mlp_engine(obs, 2, (h,), auto_alpha=auto_alpha)
    return lambda: heads_engine(auto_alpha=auto_alpha)


@pytest.mark.parametrize("auto_alpha", [True, False])
@pytest.mark.parametrize("W", WORLDS)
@pytest.mark.parametrize("case", [("mlp", i) for i in range(4)] + [("heads", 0)], ids=lambda c: f"{c[0]}{c[1]}")
def test_apply_on_the_rank_ordered_sum_equals_apply_on_the_summed_gradients(case, W, auto_alpha):
    """apply_kernel<2> as the step builds it (one-shot below 6 ranks; from 6 up the reduced block, after every rank's
    reduce-scatter) against apply_kernel<0> (dsact_test_apply) on a twin handle whose grads hold the rank-ordered sum."""
    engine, li = case
    make = _apply_case(engine, _apply_layouts()[li] if engine == "mlp" else None, auto_alpha)
    engs, bufs = world(W, make)
    twin = make()
    n = int(twin.layout.n_params)
    npad = (n + 3) // 4 * 4
    g = np.random.default_rng(97 * W + li + 11 * auto_alpha)
    init = {k: g.standard_normal(getattr(twin, k).numel()).astype(np.float32) for k in ("params", "targets", "adam_m")}
    init["adam_m"] *= np.float32(1e-3)
    init["adam_v"] = (np.abs(g.standard_normal(n)) * 1e-4).astype(np.float32)
    for e in engs + [twin]:
        for k, v in init.items():
            getattr(e, k).copy_(torch.from_numpy(v))
    rows, gb = 16, 16 * W
    for it in range(3):   # delay_update = 2: iterations 0 and 2 update the policy and the targets, 1 only the critics
        st = twin.state.cpu().numpy().copy()
        st[ST_ACC:ST_ACC + 32] = np.float32(0)
        st[ST_ACC + ACC_LOGP] = np.float32(g.integers(-40, 30))   # (not 32 = rows * act_dim: a nonzero gradient)
        st[ST_ADAM_SC:ST_ADAM_SC + 5] = np.array([1e-3, 0.03, 2e-3, 3e-3, 0.04], np.float32) * np.float32(1 + it)
        st[ST_STDSUM:ST_STDSUM + 2] = np.abs(g.standard_normal(2)).astype(np.float32) * gb
        blocks = [(g.standard_normal(npad) * 1e-2).astype(np.float32) for _ in range(W)]
        if engine == "mlp":
            # element n - 1: shares whose rank-ordered sum is exactly the log_alpha gradient the twin forms from the
            # logged sum.  In units of v's ulp: the other ranks' shares have v's sign and rank 0 holds the rest, so every
            # partial sum lies between 0 and v and is exact.
            v = log_alpha_grad(st[ST_ACC + ACC_LOGP], rows, 2, gb)
            ulp = float(np.spacing(np.abs(v)))
            m = int(float(v) / ulp)
            parts = [int(x) * (1 if m > 0 else -1) for x in g.integers(0, 1000, W - 1)]
            for r, p in enumerate([m - sum(parts)] + parts):
                blocks[r][n - 1] = np.float32(p * ulp)
            assert rank_sum([b[n - 1:n] for b in blocks])[0] == v
        for e in engs + [twin]:
            e.state.copy_(torch.from_numpy(st))
            set_int(e.state, ST_DP_EPOCH, 10 + it)
        for b, blk in zip(bufs, blocks):
            b[DP_GRADS_OFF:DP_GRADS_OFF + npad] = torch.from_numpy(blk).cuda()
            b[DP_GRADS_OFF + npad:] = POISON
        twin.grads.copy_(torch.from_numpy(rank_sum(blocks)[:n]))
        for e in engs:
            e.grads.fill_(POISON)
        torch.cuda.synchronize()
        if W >= 6:
            for e in engs:
                e.test_dp("reduce_scatter")
        for e in engs:
            e.test_dp("apply", tail_rows=rows, global_batch=gb)
        twin.test_apply(part=0, scalars_ready=2 if engine == "mlp" else 1, tail_rows=rows if engine == "mlp" else 0,
                        global_batch=gb)
        torch.cuda.synchronize()
        for r, e in enumerate(engs):
            tag = f"{engine}{li} W={W} auto_alpha={auto_alpha} iteration {it} rank {r}"
            for k in ("params", "targets", "adam_m", "adam_v", "grads"):
                assert_bits(getattr(e, k).cpu().numpy(), getattr(twin, k).cpu().numpy(), f"{tag} {k}")
            assert_bits(e.state.cpu().numpy(), twin.state.cpu().numpy(), f"{tag} state")
            assert e.state.view(torch.int32)[ST_TICKET].item() == 0 and e.state.view(torch.int32)[ST_DP_ERR].item() == 0
    for e in engs + [twin]:
        e.close()


# ---- the hooks' own checks ------------------------------------------------------------------------------------------
def test_hooks_refuse_bad_handles_before_any_launch():
    import ctypes as C

    from dsac_v2_b200 import _lib
    from dsac_v2_b200.engine import Engine, make_config, make_v1_options
    engs, _ = world(2, mlp_engine)
    with pytest.raises(_lib.DsactError, match="outside"):
        engs[0].test_dp_attach(2, engs)
    lone = mlp_engine()
    with pytest.raises(_lib.DsactError, match="dsact_dp_export"):
        lone.test_dp_attach(0, [lone, engs[1]])
    lone.dp_export()
    lone._dp_peers = engs
    with pytest.raises(_lib.DsactError, match="not attached"):
        lone.test_dp("reduce_scatter")
    with pytest.raises(_lib.DsactError, match="not rank 1"):   # ranks of another world
        engs[0]._dp_peers = [engs[0], lone]
        engs[0].test_dp("exchange")
    lib = engs[0].lib
    assert lib.dsact_test_dp(engs[0].h, 9, C.byref(_lib.TestDpIo()), None) != 0
    assert b"unknown op" in lib.dsact_last_error()
    sep = mlp_engine(policy_std="mlp_separated")
    with pytest.raises(_lib.DsactError, match="mlp_shared"):
        sep.test_dp_attach(0, [sep, engs[1]])
    lim = torch.ones(2)
    v1 = Engine(make_config(5, 2, [32], [32], max_batch=16), torch.device("cuda", 0), lim, -lim, v1=make_v1_options())
    with pytest.raises(_lib.DsactError, match="DSAC_V1"):
        v1.test_dp_attach(0, [v1, engs[1]])
    for e in engs + [lone, sep, v1]:
        e.close()
