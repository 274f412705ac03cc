"""The sampling, loss and policy-gradient kernels with non-linear output activations, row by row against float64, through
dsact_test_rows (the step's own launch code on caller buffers).

The kernels read y = act(z) of the networks' linear outputs z and multiply every output gradient by act'(z).  The
reference is tests/step_ref.py's float64 restatement of the linear kernels evaluated at y = act(z) in float64, its
gradients multiplied by act'(z) in float64.  The kernel's own fp32 act / act' carry a few ulps (gelu's 1 + erf cancels to
an absolute error of about |z| 2^-22): each output's tolerance is twice its step_ref gate plus what moving every
activated input, one column at a time, and every act' by its error bound moves the float64 reference.  Sums over rows
(std sums, logged sums, bias gradients) take the sum of their terms' tolerances plus their summation depth.

Every non-linear code runs on the critics and, with another code, on the policy, for each row-kernel route: DSAC-T on the
MLP engine (fp32; bf16x3, whose bf16 images must hold the split of the kernel's own fp32 outputs; the mlp_separated and
"parameter" std types), DSAC_V1 on the MLP engine, and the head-wise engine with separate critic / policy heads, the
"parameter" std type, the plain Gaussian (on both engines, in fp32 and bf16x3 on the MLP engine), and DSAC_V1 with the bounded and the Gaussian NLL loss.  With "parameter" (on
either engine) the log_std half is the learnable row, which is not activated.  The rows put z at 0 and below (the
relu kink, act' = 0), saturate tanh / sigmoid, push the activated log_std past both clamp bounds, and lift the activated
raw std above softplus's threshold of 20.  Outputs start as NaN and sentinel rows past the batch must stay untouched."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import step_ref as R
from test_gpu_step_kernels import SENT, _check_img, _dev, _img, _nan

pytestmark = pytest.mark.gpu

HY = dict(gamma=0.99, tau=0.005, tau_b=0.005, alpha=0.2, min_log_std=-0.8, max_log_std=0.5, lr_q=1e-4, lr_pi=1e-4,
          lr_alpha=3e-4, delay_update=2, td_bound=20.0)
CODES = ["relu", "gelu", "tanh", "sigmoid", "elu", "selu"]
KINDS = ["mlp", "mlp_bf16x3", "v1", "mlp_separated", "mlp_parameter", "separated", "parameter", "gauss", "heads_v1",
         "heads_v1_nll", "mlp_gauss", "mlp_gauss_bf16x3"]
CASES = [(k, q, CODES[(i + 1) % len(CODES)]) for k in KINDS for i, q in enumerate(CODES)]
A, B = 3, 37
U = 2.0 ** -23
ST_STDSUM, ST_ACC = 4, 16
_F = {"relu": F.relu, "gelu": F.gelu, "tanh": torch.tanh, "sigmoid": torch.sigmoid, "elu": F.elu, "selu": F.selu,
      "linear": lambda x: x}


def act64(z, name):
    return _F[name](z)


def dact64(z, name):
    """torch's derivative (relu'(0) = 0, elu'(0) = 1, selu'(0) = 1.0507 * 1.6733), the kernels' act_bwd"""
    zz = z.clone().requires_grad_(True)
    g, = torch.autograd.grad(_F[name](zz).sum(), zz)
    return g


def act_err(z, name):
    """bound on |act_fwd(z) - act(z)| of the kernel's fp32 act_fwd"""
    if name in ("linear", "relu"):
        return torch.zeros_like(z)
    y = act64(z, name).abs()
    return 8 * U * y + (2 * U * z.abs() if name == "gelu" else 0.0)


def dact_err(z, name):
    if name in ("linear", "relu"):
        return torch.zeros_like(z)
    return 8 * U * dact64(z, name).abs() + 4 * U


def _engine(kind, acts):
    from dsac_v2_b200.engine import Engine, make_config, make_v1_options
    from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config, make_heads_config
    hi = R.f32(1.0 + 0.25 * (torch.arange(A) % 3)).float()
    lo = R.f32(-1.0 + 0.125 * (torch.arange(A) % 2)).float()
    kw = dict(max_batch=B, auto_alpha=True, gamma=HY["gamma"], tau=HY["tau"], alpha=HY["alpha"], min_log_std=HY["min_log_std"],
              max_log_std=HY["max_log_std"])
    dev, oa = torch.device("cuda", 0), dict(output_activations=acts)
    if kind in ("mlp", "mlp_bf16x3", "v1", "mlp_separated", "mlp_parameter", "mlp_gauss", "mlp_gauss_bf16x3"):
        std = {"mlp_separated": "mlp_separated", "mlp_parameter": "parameter"}.get(kind, "mlp_shared")
        dist = "GaussDistribution" if kind.startswith("mlp_gauss") else "TanhGaussDistribution"
        cfg = make_config(5, A, (16,), (16,), gemm_mode="bf16x3" if kind.endswith("bf16x3") else "fp32", policy_std=std,
                          act_dist=dist, **kw)
        return Engine(cfg, dev, hi, lo, v1=make_v1_options(True) if kind == "v1" else None, **oa), hi, lo
    if kind == "separated":
        return CnnEngine(make_cnn_config((5, 1, 1), A, (), (), (), (16,), q_heads=2, pi_std="head", **kw), dev, hi, lo, **oa), hi, lo
    if kind == "parameter":
        return CnnEngine(make_heads_config(5, A, (16,), "parameter", **kw), dev, hi, lo, **oa), hi, lo
    if kind == "gauss":
        return CnnEngine(make_heads_config(5, A, (16,), "mlp_separated", act_dist="GaussDistribution", **kw), dev, hi, lo, **oa), hi, lo
    return CnnEngine(make_heads_config(5, A, (16,), "mlp_shared", algo="DSAC_V1", bound=kind == "heads_v1", **kw), dev, hi, lo,
                     **oa), hi, lo


def _inputs(seed):
    g = torch.Generator().manual_seed(seed)
    n = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    logits = [n(B, 2 * A) * 1.5 for _ in range(2)]
    for L in logits:   # the kink, below it, saturation both ways, the log_std clamp both ways after the activation
        L[0] = 0.0
        L[1] = -4.0
        L[2] = 12.0
        L[3] = -12.0
        L[4, A:] = torch.tensor([0.6, -0.9, 2.0])[:A]
    out_q = [n(B, 2) * 2.0 for _ in range(6)]
    for q in out_q:    # raw std (column 1) at the kink, above softplus's threshold after relu / elu / selu / gelu, saturated
        q[0] = 0.0
        q[1] = torch.tensor([-4.0, 25.0])
        q[2] = torch.tensor([12.0, -30.0])
        q[3] = torch.tensor([-12.0, 21.0])
        q[4] = torch.tensor([3.0, 40.0])
    x = {"logits": logits, "eps": [n(B, A), n(B, A)], "out_q": out_q, "rew": n(B), "done": (torch.arange(B) % 5 == 0).double(),
         "z3": n(B) * 1.6, "z4": n(B) * 1.6, "logp_new": n(B) * 2.0, "logp2": n(B) * 2.0, "d_act": [n(B, A) * 0.3, n(B, A) * 0.3]}
    return {k: ([R.f32(t) for t in v] if isinstance(v, list) else R.f32(v)) for k, v in x.items()}


def _tolerances(ref_fn, groups):
    """ref_fn(perturbation) -> {name: (v, gate)}; groups: perturbations (callables of a sign).  Returns {name: (v, tol)}."""
    base = ref_fn(None)
    spread = {k: torch.zeros_like(v) for k, (v, _) in base.items()}
    for grp in groups:
        moved = [ref_fn(grp(s)) for s in (1.0, -1.0)]
        for k, (v, _) in base.items():
            spread[k] = spread[k] + torch.maximum((moved[0][k][0] - v).abs(), (moved[1][k][0] - v).abs()).nan_to_num(0.0, 0.0, 0.0)
    return {k: (v, 2 * g + 2 * spread[k] + 8 * U * v.abs() + R.TINY) for k, (v, g) in base.items()}


def _check(errs, what, got, ref, mask=None):
    v, tol = ref
    got = got.double().cpu().reshape(v.shape)
    e = (got - v).abs() / tol
    e = torch.where(got == v, torch.zeros_like(e), e)
    if mask is not None:
        e = e[mask]
    errs[what] = float(e.max()) if e.numel() else 0.0


def _sum(ref, start=0.0, mask=None):
    v, tol = ref
    if mask is not None:
        v, tol = v[mask], tol[mask]
    return (v.sum() + start, tol.sum() + 2 * (B + 10) * U * v.abs().sum() + R.TINY)


@pytest.mark.parametrize("kind,act_q,act_pi", CASES)
def test_row_kernels_with_output_activations(kind, act_q, act_pi):
    eng, hi, lo = _engine(kind, (act_q, act_pi))
    act_ls = "linear" if kind in ("parameter", "mlp_parameter") else act_pi
    v1 = kind in ("v1", "heads_v1", "heads_v1_nll")
    gauss = kind in ("gauss", "mlp_gauss", "mlp_gauss_bf16x3")
    nq = 1 if v1 else 2
    planes = 2 if kind.endswith("bf16x3") else 0
    sc = R.scalars(HY)
    x = _inputs(7 + CODES.index(act_q))
    x["hi"], x["lo"] = R.f32(hi), R.f32(lo)
    rows = B + SENT
    log_alpha = R.c32(-1.3)
    eng.params[-1] = log_alpha
    st = eng.state
    st.zero_()
    ms = [R.c32(0.8), R.c32(1.1)]
    st[0], st[1] = ms[0], ms[1]
    st[ST_ACC + 16:ST_ACC + 32] = float("inf")
    d = {k: [_dev(t, rows, B) for t in x[k]] for k in ("logits", "eps", "out_q")}

    def act_logits(L, pert=None):
        y = torch.cat([act64(L[:, :A], act_pi), act64(L[:, A:], act_ls)], 1)
        err = torch.cat([act_err(L[:, :A], act_pi), act_err(L[:, A:], act_ls)], 1)
        return y if pert is None else y + pert * err

    def col(j):   # perturbation of one column of the (mean | log_std) row: a [B, 2A] mask
        m = torch.zeros(B, 2 * A, dtype=torch.float64)
        m[:, j] = 1.0
        return m
    dpi = torch.cat([dact64(x["logits"][0][:, :A], act_pi), dact64(x["logits"][0][:, A:], act_ls)], 1)
    dpi_err = torch.cat([dact_err(x["logits"][0][:, :A], act_pi), dact_err(x["logits"][0][:, A:], act_ls)], 1)

    # ---- sample
    act, logp = [_nan(rows, A), _nan(rows, A)], [_nan(rows), _nan(rows)]
    img_act = [_img(B, A), _img(B, A)] if planes else [None, None]
    eng.test_rows("sample", B, B, 0, logits=d["logits"], eps=d["eps"], act=act, logp=logp, out_q=d["out_q"], img_act=img_act)
    torch.cuda.synchronize()
    errs = {}
    for w in range(2):
        def ref_fn(p, w=w):
            r = R.sample_ref({"logits": act_logits(x["logits"][w], p), "eps": x["eps"][w], "hi": x["hi"], "lo": x["lo"]}, sc, gauss, v1)
            out = {"act": r["act"], "logp": r["logp"], "tm": r["tm"], "sd": r["sd"]}
            if v1:
                out["v1_std"] = r["v1_std"]
            return out
        ref = _tolerances(ref_fn, [lambda s, j=j: s * col(j) for j in range(2 * A)])
        _check(errs, f"act{w}", act[w][:B], ref["act"])
        _check(errs, f"logp{w}", logp[w][:B], ref["logp"])
        assert torch.isnan(act[w][B:]).all() and torch.isnan(logp[w][B:]).all(), "a sentinel row was written"
        if planes:
            _check_img(img_act[w], act[w], B, planes)
        if w == 0:
            got = st.double().cpu()
            tm = (ref["tm"][0][:, 0], ref["tm"][1][:, 0]) if v1 else (ref["tm"][0].reshape(-1), ref["tm"][1].reshape(-1))
            sd = ref["v1_std"] if v1 else (ref["sd"][0].reshape(-1), ref["sd"][1].reshape(-1))
            _check(errs, "acc_tanh_mean", got[ST_ACC + 6], _sum(tm))
            _check(errs, "acc_pi_std", got[ST_ACC + 7], _sum(sd))
    for k in range(nq):
        raw = x["out_q"][k][:, 1]
        ref = _tolerances(lambda p: {"sp": R.stdsum_ref(act64(raw, act_q) + (0.0 if p is None else p * act_err(raw, act_q)))},
                          [lambda s: s])
        _check(errs, f"stdsum{k}", st.double().cpu()[ST_STDSUM + k], _sum(ref["sp"]))

    # ---- loss
    stdsum = [R.c32(0.9 * B), R.c32(1.3 * B)]
    st[ST_STDSUM], st[ST_STDSUM + 1] = stdsum[0], stdsum[1]
    lrow = {k: _dev(x[k], rows, B) for k in ("rew", "done", "z3", "z4")}
    dq, dqa = [_nan(rows, 2) for _ in range(2)], [_nan(rows, 2) for _ in range(2)]
    gbias = torch.full((4,), 0.5, device="cuda")
    graw = torch.full((2,), -0.25, device="cuda")
    sep_raw = kind == "separated"
    img_q = [_img(B, 2) for _ in range(2)] if planes else [None, None]
    img_qa = [_img(B, 2) for _ in range(2)] if planes else [None, None]
    eng.test_rows("loss", B, B, 0, logp=[_dev(x["logp_new"], rows, B), _dev(x["logp2"], rows, B)], out_q=d["out_q"],
                  d_out_q=dq, d_out_qa=dqa, gbias_q=[gbias[0:], gbias[2:]], gbias_q_raw=[graw[0:], graw[1:]] if sep_raw else [None, None],
                  img_q=img_q, img_qa=img_qa, **lrow)
    torch.cuda.synchronize()
    oq = x["out_q"]
    dq64 = [dact64(q, act_q) for q in oq]
    dq_err = [dact_err(q, act_q) for q in oq]
    amb_rows = []

    def loss_fn(p):
        yq = [act64(q, act_q) for q in oq]
        dd = [t.clone() for t in dq64]
        if p is not None:
            kind_, i, c, s = p
            if kind_ == "y":
                yq[i] = yq[i].clone()
                yq[i][:, c] += s * act_err(oq[i][:, c], act_q)
            else:
                dd = [t + s * e for t, e in zip(dd, dq_err)]
        xx = dict(x, out_q=yq)
        if v1:
            o, amb, _ = R.loss_v1_ref(xx, sc, B, True, log_alpha, kind != "heads_v1_nll")
        else:
            o, amb, _ = R.loss_ref(xx, sc, dict(stdsum=stdsum, mean_std=ms), B, True, log_alpha)
        if p is None:
            amb_rows.append(amb)
        scale = lambda vg, t: (vg[0] * t, vg[1] * t.abs())
        out = {}
        for k in range(nq):
            out[f"g_mean{k}"] = scale(o[f"g_mean{k}"], dd[k][:, 0])
            out[f"g_raw{k}"] = scale(o[f"g_raw{k}"], dd[k][:, 1])
            out[f"g_pa{k}"] = scale(o[f"g_pa{k}"], dd[4 + k][:, 0])
            out[f"q{k}"], out[f"sd{k}"] = o[f"q{k}"], o[f"sd{k}"]
        out["loss_pi"] = o["loss_pi"]
        return out
    groups = [lambda s, i=i, c=c: ("y", i, c, s) for i in range(6) for c in range(2)] + [lambda s: ("d", 0, 0, s)]
    ref = _tolerances(loss_fn, groups)
    keep = ~amb_rows[0]
    assert int((~keep).sum()) <= 2, f"{int((~keep).sum())} rows within their gate of a computed branch"
    for k in range(nq):
        _check(errs, f"g_mean{k}", dq[k][:B, 0], ref[f"g_mean{k}"], keep)
        _check(errs, f"g_raw{k}", dq[k][:B, 1], ref[f"g_raw{k}"], keep)
        _check(errs, f"g_pa{k}", dqa[k][:B, 0], ref[f"g_pa{k}"])
        assert bool((dqa[k][:B, 1] == 0).all()), "the raw-std component of dL/d Q(s,a~) is zero"
        assert torch.isnan(dq[k][B:]).all() and torch.isnan(dqa[k][B:]).all(), "a sentinel row was written"
        if planes:
            _check_img(img_q[k], dq[k], B, planes)
            _check_img(img_qa[k], dqa[k], B, planes)
        acc = st.double().cpu()
        _check(errs, f"acc_q{k}", acc[ST_ACC + k], _sum(ref[f"q{k}"]))
        _check(errs, f"acc_s{k}", acc[ST_ACC + 2 + k], _sum(ref[f"sd{k}"]))
        if bool(keep.all()):
            gb = gbias.double().cpu()
            _check(errs, f"gbias_mean{k}", gb[2 * k], _sum(ref[f"g_mean{k}"], 0.5))
            _check(errs, f"gbias_raw{k}", graw.double().cpu()[k] if sep_raw else gb[2 * k + 1],
                   _sum(ref[f"g_raw{k}"], -0.25 if sep_raw else 0.5))
    _check(errs, "acc_loss_pi", st.double().cpu()[ST_ACC + 4], _sum(ref["loss_pi"]))

    # ---- policy gradient
    dl = _nan(rows, 2 * A)
    gpi = torch.full((2 * A,), 0.5, device="cuda")
    gls = torch.full((A,), -0.25, device="cuda") if kind in ("separated", "parameter", "gauss", "mlp_separated", "mlp_parameter") else None
    img_dl = _img(B, 2 * A) if planes else None
    d_act = [_dev(x["d_act"][0], rows, B), _dev(x["d_act"][1], rows, B)]
    eng.test_rows("policy_grad", B, B, 0, logits=[d["logits"][0], None], eps=[d["eps"][0], None], d_act=d_act, d_logits=dl,
                  gbias_pi=gpi, gbias_ls=gls, img_dlogits=img_dl)
    torch.cuda.synchronize()

    def pg_fn(p):
        y = act_logits(x["logits"][0], p if isinstance(p, torch.Tensor) else None)
        dd = dpi + (p[1] * dpi_err if isinstance(p, tuple) else 0.0)
        gu, gl = R.pgrad_ref({"logits": y, "eps": x["eps"][0], "d_act1": x["d_act"][0], "d_act2": None if kind == "v1" else x["d_act"][1],
                              "hi": x["hi"], "lo": x["lo"]}, sc, B, True, log_alpha, gauss)
        return {"gu": (gu[0] * dd[:, :A], gu[1] * dd[:, :A].abs()), "gls": (gl[0] * dd[:, A:], gl[1] * dd[:, A:].abs())}
    ref = _tolerances(pg_fn, [lambda s, j=j: s * col(j) for j in range(2 * A)] + [lambda s: ("d", s)])
    _check(errs, "d_mean", dl[:B, :A], ref["gu"])
    _check(errs, "d_log_std", dl[:B, A:], ref["gls"])
    assert torch.isnan(dl[B:]).all(), "a sentinel row was written"
    if planes:
        _check_img(img_dl, dl, B, planes)
    gp = gpi.double().cpu()
    for j in range(A):
        _check(errs, f"gbias_mean{j}", gp[j], _sum((ref["gu"][0][:, j], ref["gu"][1][:, j]), 0.5))
        got_ls = gls.double().cpu()[j] if gls is not None else gp[A + j]
        _check(errs, f"gbias_log_std{j}", got_ls, _sum((ref["gls"][0][:, j], ref["gls"][1][:, j]), -0.25 if gls is not None else 0.5))
    eng.close()
    for k, r in errs.items():
        print(f"ERR/TOL outact {kind} {act_q}/{act_pi} {k} {r:.4g}")
    bad = {k: r for k, r in errs.items() if not r <= 1.0}
    assert not bad, bad
