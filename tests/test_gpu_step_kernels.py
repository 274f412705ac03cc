"""The step kernels between the networks (sample, loss, DSAC_V1's loss, policy gradient, finalize, Adam / Polyak) row by
row against the float64 restatement of tests/step_ref.py, through dsact_test_rows / dsact_test_apply, which launch them
with the step's own launch code on caller buffers.  Outputs start as NaN and carry sentinel rows past `batch` that must
stay untouched; inputs past `batch` are NaN, so a kernel that reads past its rows poisons its sums.  Every batch mixes
ordinary rows with the regime rows of step_ref.row_inputs (log_std on its bounds, saturated tanh, raw std at -120 / 20 /
60, z on its clamp, done, exact critic ties, Huber's linear region, both ends of the ratio and ys - q clamps)."""
import math

import numpy as np
import pytest
import torch

import step_ref as R
import tc_ref
from dsac_v2_b200 import _lib

pytestmark = pytest.mark.gpu

HY = dict(gamma=0.99, tau=0.005, tau_b=0.005, alpha=0.2, min_log_std=-20.0, max_log_std=0.5, lr_q=1e-4, lr_pi=1e-4,
          lr_alpha=3e-4, delay_update=2)
NAN = float("nan")
SENT = 3   # sentinel rows past the batch
ST_ACC, ST_STDSUM, ST_MS, ST_ALPHA_USED = 16, 4, 0, 2
ST_ADAM_Q, ST_ADAM_PI, ST_ITER, ST_TICKET, ST_SC = 8, 9, 11, 14, 64


def _report(kernel, case, ratios):
    for k, r in ratios.items():
        print(f"ERR/GATE {kernel} {case} {k} {r:.4g}")
    bad = {k: r for k, r in ratios.items() if not r <= 1.0}
    assert not bad, bad


def _ratio(got, ref, mask=None):
    v, g = ref
    got = got.double().cpu().reshape(v.shape)
    e = (got - v).abs() / g
    e = torch.where((got == v) | (torch.isinf(v) & (got == v)), torch.zeros_like(e), e)
    if mask is not None:
        e = e[mask]
    return float(e.max()) if e.numel() else 0.0


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- engines ---------------------------------------------------------------------------------------------------------
def _engine(kind, A, max_batch, mode="fp32", auto=True, bound=True, obs=5, hidden=(16,)):
    from dsac_v2_b200.engine import Engine, make_config, make_v1_options
    from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config, make_heads_config
    hi = R.f32(1.0 + 0.25 * (torch.arange(A) % 3)).float()
    lo = R.f32(-1.0 + 0.125 * (torch.arange(A) % 2)).float()
    kw = dict(max_batch=max_batch, auto_alpha=auto, gamma=HY["gamma"], tau=HY["tau"], alpha=HY["alpha"])
    dev = torch.device("cuda", 0)
    if kind in ("mlp", "v1", "mlp_gauss"):
        dist = "GaussDistribution" if kind == "mlp_gauss" else "TanhGaussDistribution"
        cfg = make_config(obs, A, hidden, hidden, gemm_mode=mode, act_dist=dist, **kw)
        return Engine(cfg, dev, hi, lo, v1=make_v1_options(bound) if kind == "v1" else None)
    if kind == "separated":   # separate mean / std heads of the critics and the policy
        return CnnEngine(make_cnn_config((obs, 1, 1), A, (), (), (), hidden, q_heads=2, pi_std="head", **kw), dev, hi, lo)
    if kind == "parameter":
        return CnnEngine(make_heads_config(obs, A, hidden, "parameter", **kw), dev, hi, lo)
    if kind == "gauss":
        return CnnEngine(make_heads_config(obs, A, hidden, "mlp_separated", act_dist="GaussDistribution", **kw), dev, hi, lo)
    if kind == "heads_v1":
        return CnnEngine(make_heads_config(obs, A, hidden, "mlp_shared", algo="DSAC_V1", bound=bound, **kw), dev, hi, lo)
    raise ValueError(kind)


def _dev(t, rows, B):
    """t [B, ...] on the device with `rows` rows: the first B the values, the rest NaN."""
    out = torch.full((rows,) + tuple(t.shape[1:]), NAN, dtype=torch.float32, device="cuda")
    out[:B] = t.float().cuda()
    return out


def _nan(rows, *shape):
    return torch.full((rows,) + shape, NAN, dtype=torch.float32, device="cuda")


def _img(B, width):
    """An image [2][B][pitch] as dsact_test_rows lays it out (planes B * pitch elements apart)."""
    return torch.full((2, B, (width + 7) // 8 * 8), NAN, dtype=torch.bfloat16, device="cuda")


def _check_img(img, vals, B, planes):
    """The image's first B rows hold the round-to-nearest split of the kernel's own fp32 `vals`, bit for bit."""
    img = img.cpu()
    w = vals.shape[1]
    hi, lo = tc_ref.split(vals[:B].cpu())
    assert torch.equal(img[0, :B, :w].double(), hi), "hi plane"
    if planes == 2:
        assert torch.equal(img[1, :B, :w].double(), lo), "lo plane"


@pytest.mark.parametrize("name", list(R.ROW_CASES))
def test_row_kernels_against_float64(name):
    kind, A, B, mode, auto, carried, bound, cap, gbf = R.ROW_CASES[name]
    if B == "grid":   # one row past the largest natural grid (loss_kernel: 4 blocks of 64 rows per SM)
        B = 4 * _sm_count() * 64 + 1
    gb = B * gbf
    v1 = kind in ("v1", "heads_v1")
    gauss = kind in R.GAUSS_KINDS
    nq = 1 if v1 else 2
    hy = dict(HY, td_bound=20.0)
    sc = R.scalars(hy)
    eng = _engine(kind, A, max(B, 16), mode, auto, bound)
    planes = {"fp32": 0, "bf16x3": 2, "bf16": 1}[mode] if kind in ("mlp", "v1", "mlp_gauss") else 0
    x = R.case_inputs(name, B, hy)
    rows = B + SENT
    log_alpha = R.c32(-1.3)
    eng.params[-1] = log_alpha
    st = eng.state
    ms = R.case_mean_std(carried)
    st.zero_()
    st[ST_MS], st[ST_MS + 1] = ms[0], ms[1]
    st[ST_ACC + 16:ST_ACC + 32] = math.inf
    ctr0 = int(st.view(torch.int32)[10])

    # ---- sample (its logp outputs feed the loss, as in the step)
    d = {k: [_dev(t, rows, B) for t in x[k]] for k in ("logits", "eps", "out_q")}
    act, logp = [_nan(rows, A), _nan(rows, A)], [_nan(rows), _nan(rows)]
    img_act = [_img(B, A), _img(B, A)] if planes else [None, None]
    eng.test_rows("sample", B, gb, cap, advance_rng=True, logits=d["logits"], eps=d["eps"], act=act, logp=logp,
                  out_q=d["out_q"], img_act=img_act)
    torch.cuda.synchronize()
    ratios = {}
    acc_ref = {}
    for w in range(2):
        ref = R.sample_ref({"logits": x["logits"][w], "eps": x["eps"][w], "hi": x["hi"], "lo": x["lo"]}, sc, gauss, v1)
        ratios[f"act{w}"] = _ratio(act[w][:B], ref["act"])
        ratios[f"logp{w}"] = _ratio(logp[w][:B], ref["logp"])
        assert torch.isnan(act[w][B:]).all() and torch.isnan(logp[w][B:]).all(), "a sentinel row was written"
        if planes:
            _check_img(img_act[w], act[w], B, planes)
        if w == 0:
            if v1:
                tm, sd = (ref["tm"][0][:, 0], ref["tm"][1][:, 0]), ref["v1_std"]
            else:
                tm = (ref["tm"][0].reshape(-1), ref["tm"][1].reshape(-1))
                sd = (ref["sd"][0].reshape(-1), ref["sd"][1].reshape(-1))
            n = tm[0].numel()
            acc_ref["tanh_mean"] = R.sum_gate(tm[0], tm[1], n + 1)
            acc_ref["pi_std"] = R.sum_gate(sd[0], sd[1], n + 1)
    for k in range(nq):
        sp = R.stdsum_ref(x["out_q"][k][:, 1])
        acc_ref[f"stdsum{k}"] = R.sum_gate(sp[0], sp[1], B + 1)
    got = st.double().cpu()
    ratios["acc_tanh_mean"] = _ratio(got[ST_ACC + 6], acc_ref["tanh_mean"])
    ratios["acc_pi_std"] = _ratio(got[ST_ACC + 7], acc_ref["pi_std"])
    for k in range(nq):
        ratios[f"stdsum{k}"] = _ratio(got[ST_STDSUM + k], acc_ref[f"stdsum{k}"])
    assert int(st.view(torch.int32)[10]) == ctr0 + 1, "the generator counter advances once"
    _report("sample", name, ratios)

    # ---- loss
    x["logp_new"], x["logp2"] = logp[0][:B].double().cpu(), logp[1][:B].double().cpu()
    stdsum = [float(st[ST_STDSUM]), float(st[ST_STDSUM + 1])]
    sep_raw = kind == "separated"
    lrow = {k: _dev(x[k], rows, B) for k in ("rew", "done", "z3", "z4")}
    dq, dqa = [_nan(rows, 2) for _ in range(2)], [_nan(rows, 2) for _ in range(2)]
    gbias = torch.full((4,), 0.5, device="cuda")
    graw = torch.full((2,), -0.25, device="cuda")
    img_q = [_img(B, 2) for _ in range(2)] if planes else [None, None]
    img_qa = [_img(B, 2) for _ in range(2)] if planes else [None, None]
    eng.test_rows("loss", B, gb, cap, logp=[_dev(x["logp_new"], rows, B), _dev(x["logp2"], rows, B)], out_q=d["out_q"],
                  d_out_q=dq, d_out_qa=dqa, gbias_q=[gbias[0:], gbias[2:]],
                  gbias_q_raw=[graw[0:], graw[1:]] if sep_raw else [None, None], img_q=img_q, img_qa=img_qa, **lrow)
    torch.cuda.synchronize()
    if v1:
        o, amb, sides = R.loss_v1_ref(x, sc, gb, auto, log_alpha, bound)
    else:
        o, amb, sides = R.loss_ref(x, sc, dict(stdsum=stdsum, mean_std=ms), gb, auto, log_alpha)
    assert int(amb.sum()) <= 0.01 * B + 1, f"{int(amb.sum())} of {B} rows within their gate of a computed branch"
    keep = ~amb
    ratios = {}
    for k in range(nq):
        ratios[f"g_mean{k}"] = _ratio(dq[k][:B, 0], o[f"g_mean{k}"], keep)
        ratios[f"g_raw{k}"] = _ratio(dq[k][:B, 1], o[f"g_raw{k}"], keep)
        ratios[f"g_pa{k}"] = _ratio(dqa[k][:B, 0], o[f"g_pa{k}"])
        assert bool((dqa[k][:B, 1] == 0).all()), "the raw-std component of dL/d Q(s,a~) is zero"
        assert torch.isnan(dq[k][B:]).all() and torch.isnan(dqa[k][B:]).all(), "a sentinel row was written"
        if planes:
            _check_img(img_q[k], dq[k], B, planes)
            _check_img(img_qa[k], dqa[k], B, planes)
    # sums over the rows: the accumulators and the bias gradients (+= onto the targets' start values)
    full = lambda name: (o[name][0], o[name][1])
    acc = st.double().cpu()
    sums = {"q": (ST_ACC + 0, "q0"), "s": (ST_ACC + 2, "sd0"), "loss_pi": (ST_ACC + 4, "loss_pi"), "logp": (ST_ACC + 8, "logp_new")}
    if not v1:
        sums.update({"q2": (ST_ACC + 1, "q1"), "s2": (ST_ACC + 3, "sd1"), "loss_q": (ST_ACC + 5, "loss_q")})
    for name_, (slot, key) in sums.items():
        if keep.all() or key in ("q0", "q1", "sd0", "sd1", "logp_new"):
            ratios[f"acc_{name_}"] = _ratio(acc[slot], R.sum_gate(*full(key), B + 1))
    for k in range(0 if v1 else 2):   # (DSAC_V1 logs no minimum std)
        sdv, sdg = o[f"sd{k}"]
        i = int(torch.argmin(sdv))
        ratios[f"min_std{k}"] = _ratio(acc[ST_ACC + 16 + k], (sdv[i], sdg[i]))
    gb_got = gbias.double().cpu()
    if keep.all():
        for k in range(nq):
            gm, gr = R.sum_gate(*full(f"g_mean{k}"), B + 2), R.sum_gate(*full(f"g_raw{k}"), B + 2)
            ratios[f"gbias_mean{k}"] = _ratio(gb_got[2 * k], (gm[0] + 0.5, gm[1]))
            raw_got = graw.double().cpu()[k] if sep_raw else gb_got[2 * k + 1]
            ratios[f"gbias_raw{k}"] = _ratio(raw_got, (gr[0] + (-0.25 if sep_raw else 0.5), gr[1]))
    _report("loss", name, ratios)

    # ---- policy gradient
    dl = _nan(rows, 2 * A)
    gpi = torch.full((2 * A,), 0.5, device="cuda")
    gls = torch.full((A,), -0.25, device="cuda") if kind in ("separated", "parameter", "gauss") else None
    img_dl = _img(B, 2 * A) if planes else None
    d_act = [_dev(x["d_act"][0], rows, B), _dev(x["d_act"][1], rows, B)]
    eng.test_rows("policy_grad", B, gb, cap, logits=[d["logits"][0], None], eps=[d["eps"][0], None], d_act=d_act,
                  d_logits=dl, gbias_pi=gpi, gbias_ls=gls, img_dlogits=img_dl)
    torch.cuda.synchronize()
    one = kind == "v1"
    gu, gl = R.pgrad_ref({"logits": x["logits"][0], "eps": x["eps"][0], "d_act1": x["d_act"][0],
                          "d_act2": None if one else x["d_act"][1], "hi": x["hi"], "lo": x["lo"]}, sc, gb, auto, log_alpha, gauss)
    ratios = {"d_mean": _ratio(dl[:B, :A], gu), "d_log_std": _ratio(dl[:B, A:], gl)}
    assert torch.isnan(dl[B:]).all(), "a sentinel row was written"
    if planes:
        _check_img(img_dl, dl, B, planes)
    bm, bl = R.sum_gate(gu[0], gu[1], B + 9), R.sum_gate(gl[0], gl[1], B + 9)
    ratios["gbias_mean"] = _ratio(gpi.cpu()[:A], (bm[0] + 0.5, bm[1]))
    ratios["gbias_log_std"] = _ratio((gls if gls is not None else gpi[A:]).cpu(),
                                     (bl[0] + (-0.25 if gls is not None else 0.5), bl[1]))
    _report("policy_grad", name, ratios)

    # ---- finalize: tb_info from the accumulators over global_batch rows
    out = torch.full((16,), NAN, device="cuda")
    st[ST_ALPHA_USED] = 0.375
    eng.test_rows("stats", B, gb, stats_out=out)
    torch.cuda.synchronize()
    a = st.double().cpu()
    ref = R.stats_ref(a[ST_ACC:ST_ACC + 16], a[ST_ACC + 16:ST_ACC + 18], 0.375, (a[0], a[1]), 0, gb, A, v1)
    _report("stats", name, {"tb_info": _ratio(out, ref)})


# ---- Adam / Polyak ---------------------------------------------------------------------------------------------------
def _adam_engine(obs, h, v1, auto, mode="fp32", max_batch=16, heads=False):
    from dsac_v2_b200.engine import Engine, make_config, make_v1_options
    from dsac_v2_b200.engine_cnn import CnnEngine, make_heads_config
    dev = torch.device("cuda", 0)
    if heads:   # the head-wise engine (std type "parameter")
        return CnnEngine(make_heads_config(obs, 2, [h], "parameter", max_batch=max_batch, auto_alpha=auto, tau=HY["tau"]), dev,
                         torch.ones(2), -torch.ones(2))
    cfg = make_config(obs, 2, [h], [h], max_batch=max_batch, gemm_mode=mode, auto_alpha=auto, tau=HY["tau"])
    return Engine(cfg, dev, torch.ones(2), -torch.ones(2), v1=make_v1_options() if v1 else None)


def _fill(eng, seed, big=False):
    """step_ref.adam_inputs into the bound buffers; returns them (float64 on the host)."""
    x = R.adam_inputs(eng.params.numel(), seed, big)
    for k, b in (("w", "params"), ("t", "targets"), ("g", "grads"), ("m", "adam_m"), ("v", "adam_v")):
        getattr(eng, b).copy_(x[k].float().cuda())
    return x


def _snapshot(eng):
    return {k: getattr(eng, k).double().cpu().clone() for k in ("params", "grads", "adam_m", "adam_v", "targets", "state")}


def _nq2(eng):
    return eng.layout.n_q * (1 if getattr(eng, "v1", None) is not None else 2)


def _adam_ref(eng, s0, auto, delayed, sh, slabs=(), part=0):
    n = s0["params"].numel()
    nq2 = _nq2(eng)
    lo, hi = 0, n
    if part == 1:
        hi = nq2 // 4 * 4
    elif part == 2:
        lo = nq2 // 4 * 4
    return R.apply_ref(s0["params"], s0["grads"], s0["adam_m"], s0["adam_v"], s0["targets"], slabs, nq2, R.ADAM_HY, sh,
                       torch.tensor(bool(delayed)), auto, lo=lo, hi=hi)


def _check_adam(eng, ref, case, frozen):
    got = _snapshot(eng)
    ratios = {k: _ratio(got[b], ref[k]) for k, b in (("w", "params"), ("m", "adam_m"), ("v", "adam_v"), ("t", "targets"))}
    _report("apply", case, ratios)
    for k, mask in frozen.items():   # elements the launch must leave bit-unchanged
        assert torch.equal(got[k][mask], ref[{"params": "w", "adam_m": "m", "adam_v": "v", "targets": "t"}[k]][0][mask]), (case, k)


def _trips(n_params, max_blocks):
    """Grid-stride trips of apply_kernel's threads: one 4-element group per thread and trip, 256 threads per block."""
    groups = (n_params + 3) // 4
    return -(-groups // (256 * max_blocks))


def _apply_run(eng, t, delayed, auto, ready, slots, seed, max_blocks=0, big=False):
    """One of step_ref.APPLY_RUNS on `eng`: set the counters, iteration and slots, launch, check element by element."""
    _fill(eng, seed, big)
    st = eng.state.view(torch.int32)
    tq, tp, sh, written = R.apply_run_sizes(t, slots)
    st[ST_ADAM_Q], st[ST_ADAM_PI], st[ST_ITER] = tq, tp, 0 if delayed else 1
    if written is not None:
        eng.state[ST_SC:ST_SC + 5] = torch.tensor(written)
    if ready == 2:   # the stamp: the counters it was formed for (stale: other ones)
        st[ST_SC + 5], st[ST_SC + 6], st[ST_SC + 7] = (tq, tp, 0x5ca1ab1e) if slots == "valid" else (tq + 1, tq, 0x5ca1ab1e)
    s0 = _snapshot(eng)
    eng.test_apply(scalars_ready=ready, max_blocks=max_blocks)
    torch.cuda.synchronize()
    ref = _adam_ref(eng, s0, auto, delayed, sh)
    n, nq2 = s0["params"].numel(), _nq2(eng)
    idx = torch.arange(n)
    frozen = {}
    if not delayed:
        frozen = {"params": idx >= nq2, "adam_m": idx >= nq2, "adam_v": idx >= nq2, "targets": torch.ones(n - 1, dtype=torch.bool)}
    elif not auto:
        frozen = {"params": idx == n - 1, "adam_m": idx == n - 1, "adam_v": idx == n - 1}
    _check_adam(eng, ref, f"n{n}_t{t}_d{int(delayed)}_a{int(auto)}_s{ready}{slots or ''}_cap{max_blocks}", frozen)
    si = eng.state.view(torch.int32).cpu()
    assert (int(si[ST_ADAM_Q]), int(si[ST_ADAM_PI]), int(si[ST_ITER]), int(si[ST_TICKET])) == \
        (tq + 1, tp + int(delayed), (0 if delayed else 1) + 1, 0)


@pytest.mark.parametrize("residue", sorted(R.adam_layouts()))
@pytest.mark.parametrize("t", R.ADAM_T)
def test_apply_against_float64(residue, t):
    obs, h, v1, _, _ = R.adam_layouts()[residue]
    for delayed, auto, ready, slots in R.APPLY_RUNS:
        eng = _adam_engine(obs, h, v1, auto)
        _apply_run(eng, t, delayed, auto, ready, slots, t + 17 * residue[0] + residue[1], big=(t == 1))
        eng.close()


WIDE = dict(obs=6, h=96)   # 3177 parameters on the MLP engine, 2985 on the head-wise one: several trips of one or two blocks


@pytest.mark.parametrize("heads", [False, True])
@pytest.mark.parametrize("max_blocks", [1, 2])
def test_apply_grid_stride_trips(heads, max_blocks):
    """A block cap over a buffer several blocks wide: every thread takes several grid-stride trips, and with more than one
    block the last to finish (the ticket) closes the step.  On both engines."""
    for delayed, auto, ready, slots in R.APPLY_RUNS:
        eng = _adam_engine(WIDE["obs"], WIDE["h"], False, auto, heads=heads)
        n = eng.params.numel()
        assert _trips(n, max_blocks) >= (3 if max_blocks == 1 else 2), (n, max_blocks)
        _apply_run(eng, 2, delayed, auto, ready, slots, 40 + max_blocks, max_blocks=max_blocks)
        eng.close()


@pytest.mark.parametrize("residue", sorted(R.adam_layouts()))
def test_apply_parts_equal_the_whole(residue):
    """Part 1 (the critics, beside the policy backward) then part 2 give the bits of one whole launch."""
    obs, h, v1, _, _ = R.adam_layouts()[residue]
    res = []
    for parts in ((0,), (1, 2)):
        eng = _adam_engine(obs, h, v1, True)
        _fill(eng, 5)
        eng.state.view(torch.int32)[ST_ITER] = 0
        for p in parts:
            eng.test_apply(part=p)
        torch.cuda.synchronize()
        res.append(_snapshot(eng))
        eng.close()
    for k in res[0]:
        assert torch.equal(res[0][k], res[1][k]), k


@pytest.mark.parametrize("max_blocks", [1, 2])
@pytest.mark.parametrize("nslabs", [1, 2, 3, 4])
def test_apply_folds_the_weight_gradient_slabs(nslabs, max_blocks):
    eng = _adam_engine(WIDE["obs"], WIDE["h"], False, True, mode="bf16x3", max_batch=1024)
    _fill(eng, nslabs)
    n = eng.params.numel()
    assert _trips(n, max_blocks) >= 2
    slabs = eng.arena_views()["slabs"]
    stride = (n + 3) // 4 * 4   # slabs are n_params rounded up to 4 apart (float4 access to every slab)
    g = torch.Generator().manual_seed(nslabs)
    slabs.copy_((torch.randn(slabs.numel(), generator=g) * 1e-3).float().cuda())
    st = eng.state.view(torch.int32)
    st[ST_ITER] = 0
    s0 = _snapshot(eng)
    sl = [slabs[k * stride:k * stride + n].double().cpu() for k in range(nslabs)]
    eng.test_apply(fold_slabs=nslabs, max_blocks=max_blocks)
    torch.cuda.synchronize()
    ref = _adam_ref(eng, s0, True, True, R.adam_step_sizes(R.ADAM_HY, 0, 0), slabs=sl)
    _check_adam(eng, ref, f"slabs{nslabs}_cap{max_blocks}", {})
    _report("apply", f"slabs{nslabs}_cap{max_blocks}", {"grads": _ratio(eng.grads, ref["g"])})
    assert int(eng.state.view(torch.int32)[ST_TICKET]) == 0
    eng.close()


@pytest.mark.parametrize("auto", [True, False])
def test_apply_closes_the_step(auto):
    """The finishing block with the step's tail: the log_alpha gradient over `rows` of global_batch, the temperature the
    step used, the mean_std EMA commit, the counters and (fp32 mode) the next step's stamped Adam scalars."""
    hy = dict(HY, **R.ADAM_HY)
    eng = _adam_engine(6, 8, False, auto)
    _fill(eng, 3)
    A = 2
    st, si = eng.state, eng.state.view(torch.int32)
    st[ST_ACC + 8], st[ST_STDSUM], st[ST_STDSUM + 1], st[0], st[1] = -37.5, 12.0, 9.0, 1.25, -1.0
    si[ST_ADAM_Q], si[ST_ADAM_PI], si[ST_ITER] = 4, 2, 6
    s0 = _snapshot(eng)
    la0 = float(s0["params"][-1])
    eng.test_apply(tail_rows=24, global_batch=40, scalars_ready=0)
    torch.cuda.synchronize()
    gv, gg = R.log_alpha_grad(-37.5, 24, 40, A)
    got = eng.grads.double().cpu()
    ratios = {"grad_log_alpha": float(abs(got[-1] - gv) / gg)}
    sc = R.scalars(hy)
    t = R.Track()
    alpha = float(R.alpha_of(t, sc, auto, la0, (1,)).detach()[0])
    ratios["alpha_used"] = abs(float(st[ST_ALPHA_USED]) - alpha) / (abs(alpha) * 4 * R.ULP + R.TINY)
    for k, (ss, old) in enumerate(((12.0, 1.25), (9.0, -1.0))):
        t = R.Track()
        m = R.mean_std_of(t, sc, ss, old, 40, (1,))
        ratios[f"mean_std{k}"] = _ratio(st[k], (m.detach()[0], t.gate(m)[0]))
    s_mid = dict(s0)
    s_mid["grads"] = got
    ref = _adam_ref(eng, s_mid, auto, True, R.adam_step_sizes(R.ADAM_HY, 4, 2))
    _check_adam(eng, ref, f"tail_auto{int(auto)}", {})
    _report("apply", f"tail_auto{int(auto)}", ratios)
    assert (int(si[ST_ADAM_Q]), int(si[ST_ADAM_PI]), int(si[ST_ITER]), int(si[ST_TICKET])) == (5, 3, 7, 0)
    stamp = [int(si[ST_SC + 5]), int(si[ST_SC + 6]), int(si[ST_SC + 7]) & 0xffffffff]
    assert stamp == [5, 3, 0x5ca1ab1e]
    assert np.allclose(st[ST_SC:ST_SC + 5].cpu().numpy(), R.adam_step_sizes(R.ADAM_HY, 5, 3), rtol=0, atol=0)
    eng.close()


def test_hooks_refuse_bad_arguments():
    eng = _engine("mlp", 2, 16)
    x = torch.zeros(64, device="cuda")
    for kw in (dict(kernel="sample", batch=17), dict(kernel="sample", batch=0), dict(kernel="loss", batch=4)):
        with pytest.raises(_lib.DsactError):
            eng.test_rows(kw["kernel"], kw["batch"])
    with pytest.raises(_lib.DsactError):
        eng.test_rows("sample", 4, img_act=[torch.zeros(2, 4, 8, dtype=torch.bfloat16, device="cuda"), None],
                      logits=[x, x], eps=[x, x], act=[x, x], logp=[x, x], out_q=[x, x])
    for kw in (dict(part=3), dict(part=-1), dict(fold_slabs=1), dict(scalars_ready=3), dict(tail_rows=5, global_batch=4)):
        with pytest.raises(_lib.DsactError):
            eng.test_apply(**kw)
    eng.close()
