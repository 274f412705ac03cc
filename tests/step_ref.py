"""float64 restatement of the step kernels between the networks (csrc/kernels.cuh): sample_kernel, loss_kernel,
loss_v1_kernel, policy_grad_kernel, apply_kernel (Adam / Polyak) and finalize_stats_kernel, one row (one element for
Adam) at a time, from the exact fp32 inputs a kernel is given and in its operation order.

Every output comes with a gate, a first-order running-error bound computed by the same code: each fp32 operation of the
kernel is written x (1 + d) with d = 0, and float64 autograd gives dy/dd.  gate(y) = 2 sum |dy/dd_i| u_i + FLOOR ulps of
|y|, with u = 2^-24 for + - * / and sqrtf (the build uses no fast-math: they are correctly rounded; an FMA contraction
only removes a rounding) and, for the transcendentals, CUDA's documented maximum errors (2 ulp expf / tanhf, 1 ulp
logf / log1pf; one ulp is at most 2^-23 relative).  The gate follows the conditioning: it is wide where 1 + TG_EPS - th^2
cancels and tight everywhere else.

Branches on inputs (the log_std clamp and its gradient mask, softplus's `> 20`, the z clamp, the critic picks) are
taken exactly as the kernel takes them.  Branches on computed values (Huber's |d| <= 50, the ys - q clamp, the ratio
clamp, DSAC_V1's TD clamp) are undecidable within the gate of their argument: `ambiguous` marks such rows, which the
value checks skip.  Sums (accumulators, bias gradients, std sums) are bounded by their depth in the kernel's summation
order times sum |terms|, plus the terms' own gates.

`fault` arguments emulate the kernel faults tests/test_step_ref.py requires every gate to see (ROW_FAULTS, ADAM_FAULTS
there).  ROW_CASES / case_inputs and adam_layouts / adam_inputs / APPLY_RUNS are the cases tests/test_gpu_step_kernels.py
runs, so that the power of every gate is measured on the inputs the kernels are checked on."""
from __future__ import annotations

import math

import numpy as np
import torch

U = 2.0 ** -24
ULP = 2.0 ** -23                 # one ulp, relative, at most
U_EXP, U_TANH, U_LOG, U_LOG1P = 2 * ULP, 2 * ULP, ULP, ULP
FLOOR = 4.0                      # ulps of |y| every gate allows
TINY = 2.0 ** -140               # absolute floor: fp32 underflow (expf(-120) = 0 against float64's 8e-53)
FLT_MAX = float(np.finfo(np.float32).max)
POWER = 5.0                      # every emulated fault must move some checked output by this many gates


_exact = False


def c32(x) -> float:
    """The fp32 value of a scalar, as a Python float (the float64 value itself under `exact_constants`)."""
    return float(x) if _exact else float(np.float32(x))


TG_EPS = c32(1e-6)
C1 = c32(np.float32(1.0) + np.float32(TG_EPS))   # 1.f + TG_EPS
HUBER = 50.0
STD_BIAS = c32(0.1)
HALF_LOG_2PI = c32(0.91893853320467274)
R_LO, R_HI = c32(0.1), 10.0      # the ratio clamp


class exact_constants:
    """Within: every constant and scalar in float64, as the float64 oracle forms them (the restatement's formulas can
    then be compared with the oracle's to float64 rounding)."""

    def __enter__(self):
        global _exact, TG_EPS, C1, STD_BIAS, HALF_LOG_2PI, R_LO
        self.saved = (TG_EPS, C1, STD_BIAS, HALF_LOG_2PI, R_LO)
        _exact, TG_EPS, C1, STD_BIAS, HALF_LOG_2PI, R_LO = True, 1e-6, 1 + 1e-6, 0.1, math.log(math.sqrt(2 * math.pi)), 0.1

    def __exit__(self, *a):
        global _exact, TG_EPS, C1, STD_BIAS, HALF_LOG_2PI, R_LO
        _exact = False
        TG_EPS, C1, STD_BIAS, HALF_LOG_2PI, R_LO = self.saved


def f32(x) -> torch.Tensor:
    """float64 tensor of the fp32 values of x."""
    return torch.as_tensor(x).float().double()


class Track:
    """Running-error bookkeeping: r(x) marks one fp32 rounding of x."""

    def __init__(self):
        self.ds = []

    def r(self, x, u=U):
        d = torch.zeros_like(x, requires_grad=True)
        self.ds.append((d, u))
        return x * (1 + d)

    def exp(self, x):
        return self.r(torch.exp(x), U_EXP)

    def tanh(self, x):
        return self.r(torch.tanh(x), U_TANH)

    def log(self, x):
        return self.r(torch.log(x), U_LOG)

    def softplus(self, x, fault=None):
        """softplus_f: x > 20 ? x : log1pf(expf(x))."""
        big = x >= 20 if fault == "softplus_ge20" else x > 20
        return torch.where(big, x, self.r(torch.log1p(self.exp(torch.where(big, torch.zeros_like(x), x))), U_LOG1P))

    def gate(self, y):
        """2 sum |dy/dd_i| u_i + the floor, per element of y (every rounding of a row feeds only that row's outputs)."""
        ds = [d for d, _ in self.ds]
        acc = torch.zeros(y.shape, dtype=torch.float64)
        if not y.requires_grad:   # an input passed through: exact
            return acc + TINY
        gs = torch.autograd.grad(y.sum(), ds, retain_graph=True, allow_unused=True)
        for (d, u), g in zip(self.ds, gs):
            if g is None:
                continue
            # (NaN: an infinity times a zero sensitivity, as through m / inf where (1 - beta2) g g overflowed)
            g = g.abs().nan_to_num(0.0, math.inf, math.inf) * u
            while g.dim() > y.dim():
                g = g.sum(-1)
            if g.shape != y.shape:   # the targets: element i of the (one longer) parameter buffer feeds target i
                g = g[tuple(slice(0, s) for s in y.shape)]
            acc = acc + g
        yv = y.detach()
        return 2 * acc + FLOOR * ULP * yv.abs().nan_to_num(0.0, 0.0, 0.0) + TINY


def out(t: Track, y):
    """(value, gate) of one output."""
    return y.detach().clone(), t.gate(y)


def sum_gate(terms, gates, depth, dim=0):
    """Value and gate of a sum of `terms` (with per-term `gates`) added at most `depth` deep."""
    return terms.sum(dim), 2 * depth * U * terms.abs().sum(dim) + gates.sum(dim) + TINY


def near(arg, gate, thr):
    """Rows whose computed branch argument lies within its gate of a threshold."""
    return (arg - thr).abs() <= gate


# ---- hyperparameters as the kernels receive them -----------------------------------------------------------------------
def scalars(hy: dict) -> dict:
    """fp32 scalars of a handle's configuration (`hy` as make_config's keywords, plus act_dim)."""
    return dict(gamma=c32(hy["gamma"]), tau=c32(hy["tau"]), tau_b=c32(hy["tau_b"]), alpha_fixed=c32(hy["alpha"]),
                min_ls=c32(hy["min_log_std"]), max_ls=c32(hy["max_log_std"]), td=c32(hy.get("td_bound", 20.0)))


def inv_gb(gb) -> float:
    return c32(1.0 / gb)


def alpha_of(t: Track, sc, auto, log_alpha, shape):
    """step_alpha, evaluated per element of `shape` (every row evaluates it itself)."""
    if not auto:
        return torch.full(shape, sc["alpha_fixed"], dtype=torch.float64)
    return t.exp(torch.full(shape, float(log_alpha), dtype=torch.float64))


def mean_std_of(t: Track, sc, stdsum, old, gb, shape):
    """step_mean_std per element of `shape`."""
    mean = t.r(torch.full(shape, float(stdsum), dtype=torch.float64) * inv_gb(gb))
    if old < 0:
        return mean
    a = c32(np.float32(1.0) - np.float32(sc["tau_b"]))
    return t.r(t.r(torch.full(shape, a * float(old), dtype=torch.float64)) + t.r(sc["tau_b"] * mean))


# ---- sample_kernel ---------------------------------------------------------------------------------------------------
def sample_ref(x: dict, sc: dict, gauss=False, v1=False, fault=None):
    """One policy (which = 0 or 1) of sample_kernel: x holds logits [B, 2A], eps [B, A], hi, lo [A] (fp32 values as float64).
    Returns {"act": (v, g), "logp": (v, g), "tm": ..., "sd": ...} per element / row, and the stat terms."""
    t = Track()
    L, eps = x["logits"].clone(), x["eps"]
    if fault == "neighbour":
        L = torch.roll(L, -1, 0)
    B, A2 = L.shape
    A = A2 // 2
    mean, ls = L[:, :A], L[:, A:]
    ls_c = ls if fault == "no_clamp_sample" else ls.clamp(sc["min_ls"], sc["max_ls"])
    sd = t.exp(ls_c)
    u = t.r(mean + t.r(sd * eps))
    d = t.r(u - mean)
    gterm = t.r(t.r(-t.r(d * d) / t.r(2 * sd * sd)) - t.log(sd))
    gterm = t.r(gterm - HALF_LOG_2PI)
    tm = t.tanh(mean)
    hi, lo = x["hi"].expand(B, A), x["lo"].expand(B, A)
    if gauss and fault != "gauss_squash":
        act, lp = u, gterm
    else:
        th = t.tanh(u)
        scale, shift = 0.5 * t.r(hi - lo), 0.5 * t.r(hi + lo)
        act = t.r(t.r(scale * th) + shift)
        c1 = 1.0 if fault == "tg_eps_logp" else C1
        lp = t.r(gterm - t.log(t.r(c1 - t.r(th * th))))
        lp = t.r(lp - t.log(scale))
    res = {"act": out(t, act)}
    lpv, lpg = out(t, lp)
    res["logp"] = sum_gate(lpv, lpg, (A + 31) // 32 + 5, dim=-1)
    res["tm"], res["sd"] = out(t, tm), out(t, sd)
    if v1:   # dsac_v1.py:142-143: entry 1 of cat(mean, std): the raw logit of mean 1, or (A == 1) the std itself
        if (A == 1) != (fault == "v1_stats_pick"):
            res["v1_std"] = (res["sd"][0][:, 0], res["sd"][1][:, 0])
        else:
            res["v1_std"] = (L[:, 1].clone(), torch.full((B,), TINY, dtype=torch.float64))
    return res


def stdsum_ref(raw, fault=None):
    """The y = 1 half's softplus(raw std) terms of one critic [B] (value, gate)."""
    t = Track()
    return out(t, t.softplus(raw, fault))


# ---- loss_kernel -----------------------------------------------------------------------------------------------------
def _huber(t, d):
    a = d.abs()
    return torch.where(a <= HUBER, t.r(0.5 * t.r(d * d)), t.r(HUBER * t.r(a - 0.5 * HUBER)))


def loss_ref(x: dict, sc: dict, st: dict, gb, auto, log_alpha, fault=None):
    """loss_kernel per row.  x: rew, done, z3, z4, logp_new, logp2 [B], out_q [6][B, 2].  st: stdsum[2], mean_std[2]
    (the carried state).  Returns outputs {name: (v, g)}, the rows `ambiguous` and the branch sides the checked rows took."""
    t = Track()
    B = x["rew"].shape[0]
    sh = (B,)
    invB = inv_gb(gb)
    m = [mean_std_of(t, sc, st["stdsum"][k], st["mean_std"][k], gb, sh) for k in range(2)]
    alpha = alpha_of(t, sc, auto, log_alpha, sh)
    oq = [q.clone() for q in x["out_q"]]
    if fault == "neighbour":
        oq[2] = torch.roll(oq[2], -1, 0)
    q1n, q2n = oq[2][:, 0], oq[3][:, 0]
    s1n, s2n = t.softplus(oq[2][:, 1], fault), t.softplus(oq[3][:, 1], fault)
    clampz = (lambda z: z) if fault == "no_zclamp" else (lambda z: z.clamp(-3.0, 3.0))
    zc3, zc4 = clampz(x["z3"]), clampz(x["z4"])
    pick1 = q1n <= q2n if fault == "tie_target_c1" else q1n < q2n
    qn = torch.where(q1n < q2n, q1n, q2n)
    qn_s = torch.where(pick1, t.r(q1n + t.r(zc3 * s1n)), t.r(q2n + t.r(zc4 * s2n)))
    done = torch.zeros_like(x["done"]) if fault == "done_ignored" else x["done"]
    nd = t.r(t.r(1.0 - done) * sc["gamma"])
    alp2 = t.r(alpha * x["logp2"])
    y = t.r(x["rew"] + t.r(nd * t.r(qn - alp2)))
    ys = t.r(x["rew"] + t.r(nd * t.r(qn_s - alp2)))
    amb = torch.zeros(sh, dtype=torch.bool)
    sides = {}
    res = {}
    loss_q = 0.0
    args = []
    for k in range(2):
        q, raw = oq[k][:, 0], oq[k][:, 1]
        sd = t.softplus(raw, fault)
        b3 = t.r(3.0 * m[k])
        dys = t.r(ys - q)
        yb = t.r(q + torch.minimum(torch.maximum(dys, -b3), b3))
        w0 = t.r(t.r(m[k] * m[k]) / t.r(t.r(sd * sd) + STD_BIAS))
        w = w0 if fault == "no_ratio_clamp" else w0.clamp(R_LO, R_HI)
        dq = t.r(q - y)
        dqb = t.r(q - yb)
        sterm = t.r(t.r(t.r(sd * sd) - _huber(t, dqb)) / t.r(sd + STD_BIAS))
        loss_q = t.r(loss_q + t.r(w * t.r(_huber(t, dq) + t.r(sd * sterm))))
        dqc = dq if fault == "huber_unclamped" else dq.clamp(-HUBER, HUBER)
        res[f"g_mean{k}"] = t.r(t.r(w * dqc) * invB)
        big = raw >= 20 if fault == "dsoft_ge20" else raw > 20
        dsoft = torch.where(big, torch.ones_like(raw),
                            t.r(1.0 / t.r(1.0 + t.exp(-torch.where(big, torch.zeros_like(raw), raw)))))
        res[f"g_raw{k}"] = t.r(t.r(t.r(w * sterm) * invB) * dsoft)
        res[f"q{k}"], res[f"sd{k}"] = q, sd
        args += [(f"huber{k}", dq, (HUBER,)), (f"huber_b{k}", dqb, (HUBER,)), (f"yb{k}", (dys, b3), None),
                 (f"ratio{k}", w0, (R_LO, R_HI))]
    q1p, q2p = oq[4][:, 0], oq[5][:, 0]
    alpn = t.r(alpha * x["logp_new"])
    res["loss_pi"] = t.r(alpn - torch.where(q1p < q2p, q1p, q2p))
    res["loss_q"] = loss_q
    half = c32(0.5 * invB)
    tie = q1p == q2p
    g0 = torch.where(q1p < q2p, -invB, torch.where(tie, -half, 0.0))
    g1 = torch.where(q2p < q1p, -invB, torch.where(tie, -half, 0.0))
    if fault == "tie_gpa_one":
        g0, g1 = torch.where(tie, -invB, g0), torch.where(tie, 0.0, g1)
    outs = {k: out(t, v) for k, v in res.items()}
    outs["g_pa0"], outs["g_pa1"] = (g0.double(), torch.full(sh, TINY)), (g1.double(), torch.full(sh, TINY))
    outs["logp_new"] = (x["logp_new"].clone(), torch.full(sh, TINY))
    for name, a, thr in args:
        if thr is None:   # |ys - q| against 3 m
            d, b = a
            gd, gb3 = t.gate(d), t.gate(b)
            amb |= ((d.detach().abs() - b.detach()).abs() <= gd + gb3)
            sides[name] = (d.detach() > b.detach(), d.detach() < -b.detach(), d.detach().abs() < b.detach())
            continue
        g = t.gate(a)
        av = a.detach()
        for th in thr:
            amb |= near(av.abs() if name.startswith("huber") else av, g, th)
        if name.startswith("huber"):
            sides[name] = (av.abs() <= HUBER, av.abs() > HUBER)
        else:
            sides[name] = (av < R_LO, av > R_HI, (av > R_LO) & (av < R_HI))
    return outs, amb, sides


# ---- loss_v1_kernel --------------------------------------------------------------------------------------------------
def loss_v1_ref(x: dict, sc: dict, gb, auto, log_alpha, bound=True, fault=None):
    t = Track()
    B = x["rew"].shape[0]
    sh = (B,)
    invB = inv_gb(gb)
    alpha = alpha_of(t, sc, auto, log_alpha, sh)
    oq = [q.clone() for q in x["out_q"]]
    if fault == "neighbour":
        oq[2] = torch.roll(oq[2], -1, 0)
    qn, sn = oq[2][:, 0], t.softplus(oq[2][:, 1], fault)
    zc = x["z3"] if fault == "no_zclamp" else x["z3"].clamp(-3.0, 3.0)
    done = torch.zeros_like(x["done"]) if fault == "done_ignored" else x["done"]
    inner = t.r(t.r(qn + t.r(zc * sn)) - t.r(alpha * x["logp2"]))
    target = t.r(x["rew"] + t.r(t.r(t.r(1.0 - done) * sc["gamma"]) * inner))
    q, raw = oq[0][:, 0], oq[0][:, 1]
    sd = t.softplus(raw, fault)
    td = sc["td"]
    amb = torch.zeros(sh, dtype=torch.bool)
    sides = {}
    dtq = t.r(target - q)
    if bound:
        sdd = sd.clamp(min=0.0)
        tq = dtq if fault == "v1_no_td_clamp" else dtq.clamp(-td, td)
        tb = t.r(q + tq)
        g_mean = t.r(t.r(-dtq / t.r(t.r(sdd * sdd) + STD_BIAS)) * invB)
        qtb = t.r(q - tb)
        g_sd = t.r(t.r(-t.r(t.r(qtb * qtb) - t.r(sdd * sdd)) / t.r(t.r(t.r(sdd * sdd) * sdd) + STD_BIAS)) * invB)
        if fault == "v1_gsd_sign":
            g_sd = -g_sd
        g = t.gate(dtq)
        amb |= near(dtq.detach().abs(), g, td)
        sides["td"] = (dtq.detach().abs() < td, dtq.detach().abs() > td)
    else:
        g_mean = t.r(t.r(-dtq / t.r(sd * sd)) * invB)
        dd = t.r(dtq * dtq)
        g_sd = t.r(t.r(t.r(1.0 / sd) - t.r(dd / t.r(t.r(sd * sd) * sd))) * invB)
        if fault == "v1_gsd_sign":
            g_sd = -g_sd
    big = raw >= 20 if fault == "dsoft_ge20" else raw > 20
    dsoft = torch.where(big, torch.ones_like(raw), t.r(1.0 / t.r(1.0 + t.exp(-torch.where(big, torch.zeros_like(raw), raw)))))
    g_raw = t.r(g_sd * dsoft)
    lp = x["logp_new"]
    res = {"g_mean0": g_mean, "g_raw0": g_raw, "q0": q, "sd0": sd, "loss_pi": t.r(t.r(alpha * lp) - oq[4][:, 0])}
    outs = {k: out(t, v) for k, v in res.items()}
    outs["g_pa0"] = (torch.full(sh, -invB, dtype=torch.float64), torch.full(sh, TINY))
    outs["logp_new"] = (lp.clone(), torch.full(sh, TINY))
    return outs, amb, sides


# ---- policy_grad_kernel ----------------------------------------------------------------------------------------------
def pgrad_ref(x: dict, sc: dict, gb, auto, log_alpha, gauss=False, fault=None):
    """policy_grad_kernel per element: x holds logits [B, 2A], eps, d_act1 (and d_act2) [B, A], hi, lo [A].
    Returns (gu, gls) as (v, g) [B, A]."""
    t = Track()
    L = x["logits"].clone()
    if fault == "neighbour":
        L = torch.roll(L, -1, 0)
    B, A2 = L.shape
    A = A2 // 2
    mean, ls, e = L[:, :A], L[:, A:], x["eps"]
    lo_, hi_ = sc["min_ls"], sc["max_ls"]
    inside = (ls > lo_) & (ls < hi_) if fault == "clamp_mask_exclusive" else (ls >= lo_) & (ls <= hi_)
    sd = t.exp(ls.clamp(lo_, hi_))
    da = x["d_act1"] if x.get("d_act2") is None else t.r(x["d_act1"] + x["d_act2"])
    coef = t.r(alpha_of(t, sc, auto, log_alpha, (B, A)) * inv_gb(gb))
    if gauss:
        gu = da
        gls = torch.where(inside, t.r(t.r(t.r(gu * e) - t.r(coef / sd)) * sd), 0.0)
    else:
        scale = 0.5 * t.r(x["hi"].expand(B, A) - x["lo"].expand(B, A))
        th = t.tanh(t.r(mean + t.r(sd * e)))
        # th * th is written twice; nvcc forms it once or contracts both subtractions into FMAs (no rounding): one
        # rounding shared by 1 - th^2 and 1 + TG_EPS - th^2 bounds either
        th2 = t.r(th * th)
        om = t.r(1.0 - th2)
        c1 = 1.0 if fault == "tg_eps_grad" else C1
        gu = t.r(t.r(t.r(da * scale) * om) + t.r(coef * t.r(t.r(2 * th * om) / t.r(c1 - th2))))
        gsd = t.r(t.r(gu * e) - t.r(coef / sd))
        gls = torch.where(inside, t.r(gsd * sd), 0.0)
    return out(t, gu), out(t, gls)


# ---- apply_kernel ----------------------------------------------------------------------------------------------------
def adam_step_sizes(hy: dict, tq: int, tp: int, fault=None):
    """adam_scalars: {lr_q / bc1q, sqrt(bc2q), lr_pi / bc1p, lr_alpha / bc1p, sqrt(bc2p)} for the counters (tq, tp) the
    state holds, in double, rounded to fp32."""
    o = 0 if fault == "bc_t" else 1
    b1, b2 = hy.get("adam_beta1", 0.9), hy.get("adam_beta2", 0.999)
    tq, tp = tq + o, tp + o
    div = lambda a, b: a / b if b != 0 else math.inf
    return [c32(div(hy["lr_q"], 1 - b1 ** tq)), c32(math.sqrt(1 - b2 ** tq)), c32(div(hy["lr_pi"], 1 - b1 ** tp)),
            c32(div(hy["lr_alpha"], 1 - b1 ** tp)), c32(math.sqrt(1 - b2 ** tp))]


def _ovf(x):
    """fp32 overflow of a rounded result (|x| past the largest finite float rounds to infinity)."""
    lim = FLT_MAX * (1 + 2.0 ** -25)
    return torch.where(x.abs() >= lim, torch.sign(x) * math.inf, x)


def apply_ref(w, g, m, v, tg, slabs, n_q2, hy, sh, delayed, auto, fault=None, lo=None, hi=None):
    """apply_kernel on elements [lo, hi) (default all) of the flat buffers (fp32 values as float64): w params, g grads
    (the log_alpha element already formed), m, v, tg targets (one shorter), slabs [n][len] folded first, `sh` the five
    step sizes in use.  Returns {"w", "m", "v", "t", "g"}: (v, g) of the whole buffers (untouched elements exact)."""
    n = w.shape[0]
    lo = 0 if lo is None else lo
    hi = n if hi is None else hi
    idx = torch.arange(n)
    sel = (idx >= lo) & (idx < hi)
    t = Track()
    gg = g.clone()
    for s in slabs:
        gg = torch.where(sel, t.r(gg + s[:n]), gg)
    omb1, b2f, omb2 = c32(1 - hy.get("adam_beta1", 0.9)), c32(hy.get("adam_beta2", 0.999)), c32(1 - hy.get("adam_beta2", 0.999))
    eps, tau = c32(hy.get("adam_eps", 1e-8)), c32(hy["tau"])
    critic = idx < n_q2
    is_alpha = idx == n - 1
    upd = sel & (critic | (delayed if fault != "policy_nondelayed" else torch.ones_like(critic)))
    upd &= ~(is_alpha & (not auto if fault != "alpha_fixed_update" else False))
    f = lambda v: torch.tensor(v, dtype=torch.float64)
    step = torch.where(critic, f(sh[0]), torch.where(is_alpha, f(sh[3]), f(sh[2])))
    bc2 = torch.where(critic, f(sh[1]), f(sh[4]))
    m2 = t.r(m + t.r(t.r(gg - m) * omb1))
    gsq = _ovf(t.r(_ovf(t.r(omb2 * gg)) * gg))
    v2 = _ovf(t.r(t.r(v * b2f) + gsq))
    # sqrt with a finite derivative at v = 0 (g = 0 elements), where its rounding contributes nothing
    sqrt = lambda a: torch.where(a > 0, torch.sqrt(torch.where(a > 0, a, torch.ones_like(a))), torch.zeros_like(a))
    if fault == "eps_in_sqrt":
        denom = t.r(t.r(sqrt(t.r(v2 + eps))) / bc2)
    else:
        denom = t.r(t.r(t.r(sqrt(v2)) / bc2) + eps)
    w2 = t.r(w - t.r(step * t.r(m2 / denom)))
    w2 = torch.where(upd, w2, w)
    m2, v2 = torch.where(upd, m2, m), torch.where(upd, v2, v)
    polyak = c32(1 - tau)
    a, b = (c32(1 - polyak), polyak) if fault == "polyak_swap" else (polyak, c32(1 - polyak))
    tw = w2[:n - 1]
    t2 = t.r(t.r(tg * a) + t.r(b * tw))
    tsel = sel[:n - 1] & (torch.ones_like(critic[:n - 1]) & delayed)
    t2 = torch.where(tsel, t2, tg)
    return {"w": out(t, w2), "m": out(t, m2), "v": out(t, v2), "t": out(t, t2), "g": out(t, gg)}


def log_alpha_grad(acc_logp, rows, gb, act_dim, fault=None):
    """tail_grad_log_alpha: -(ACC_LOGP + rows * target_entropy) * inv_global_batch (value, gate)."""
    t = Track()
    r = gb if fault == "logalpha_rows" else rows
    te = -float(act_dim)
    y = -t.r(t.r(torch.tensor([float(acc_logp)], dtype=torch.float64) + t.r(torch.tensor([r * te], dtype=torch.float64)))
             ) * inv_gb(gb)
    y = t.r(y)
    return y.detach()[0], t.gate(y)[0]


# ---- finalize_stats_kernel -------------------------------------------------------------------------------------------
def stats_ref(acc16, mins2, alpha_used, ms, dp_err, gb, A, v1=False):
    """The 16 tb_info floats from the accumulators (fp32 values): every entry one product with its scale, or a copy."""
    ib = inv_gb(gb)
    ip = c32(1.0 / (gb if v1 else gb * A))
    a = [float(x) for x in acc16]
    v = [a[0] * ib, a[1] * ib, a[2] * ib, a[3] * ib, mins2[0], mins2[1], a[4] * ib, a[5] * ib, a[6] * ip, a[7] * ip,
         -a[8] * ib, alpha_used, ms[0], ms[1], float(dp_err), 0.0]
    g = [abs(x) * ULP + TINY for x in v]
    return torch.tensor(v, dtype=torch.float64), torch.tensor(g, dtype=torch.float64)


# ---- inputs: ordinary rows and the regime rows every batch carries ---------------------------------------------------
def nextafter(x, d):
    return float(np.nextafter(np.float32(x), np.float32(d)))


def row_inputs(A: int, B: int, seed: int, hy: dict):
    """fp32 inputs (float64 tensors) of every per-row kernel for B rows: row r is ordinary when r % 3 == 0, else a regime
    row (kind r // 3 cycling): log_std below / at / one step inside / outside both bounds; |u| up to 12 of both signs;
    raw std at -120, 20, nextafter(20), 60; z at +-3 and beyond; done 0 and 1; exact ties q1n == q2n and q1p == q2p;
    Huber's linear region; both ends of the ratio and ys - q clamps."""
    g = torch.Generator().manual_seed(seed)
    n = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    lo_ls, hi_ls = c32(hy["min_log_std"]), c32(hy["max_log_std"])
    mean, ls, eps = n(B, A), -2.5 + 2.5 * torch.rand(B, A, generator=g, dtype=torch.float64), n(B, A)
    ls_vals = [lo_ls - 1, lo_ls, nextafter(lo_ls, 0), nextafter(lo_ls, -100), hi_ls, nextafter(hi_ls, 0),
               nextafter(hi_ls, 100), hi_ls + 1]
    u_vals = [2.0, -2.0, 4.0, -4.0, 6.0, -6.0, 8.0, -8.0, 10.0, -10.0, 12.0, -12.0]
    raw_vals = [-120.0, 20.0, nextafter(20.0, 100), 60.0, nextafter(20.0, 0)]
    z_vals = [3.0, -3.0, nextafter(3.0, 100), nextafter(-3.0, -100), 5.0, -5.0, nextafter(3.0, 0)]
    oq = [torch.stack([2.0 * n(B), n(B)], 1) for _ in range(6)]
    z3, z4 = n(B), n(B)
    done = (torch.rand(B, generator=g) < 0.3).double()
    rew = n(B)
    for r in range(B):
        if r % 3 == 0:
            continue
        k = r // 3
        ls[r] = torch.tensor([ls_vals[(k + j) % len(ls_vals)] for j in range(A)], dtype=torch.float64)
        if k % 2:   # a saturating action: small std, |u| large
            mean[r] = torch.tensor([u_vals[(k + j) % len(u_vals)] for j in range(A)], dtype=torch.float64)
            ls[r] = -6.0
        kind = k % 8
        p = k % len(raw_vals)
        oq[k % 6][r, 1] = raw_vals[p]
        oq[(k + 3) % 6][r, 1] = raw_vals[(p + 2) % len(raw_vals)]
        z3[r], z4[r] = z_vals[k % len(z_vals)], z_vals[(k + 3) % len(z_vals)]
        done[r] = float(k % 2)
        if kind == 0:
            oq[3][r, 0] = oq[2][r, 0]                 # q1n == q2n: the target takes critic 2's sample
        elif kind == 1:
            oq[5][r, 0] = oq[4][r, 0]                 # q1p == q2p: the actor gradient splits
        elif kind == 2:
            oq[0][r, 0], oq[1][r, 0] = 300.0, -300.0  # Huber's linear region, the ys - q clamp at both ends
        elif kind == 3:
            oq[0][r, 1], oq[1][r, 1] = 60.0, -120.0   # ratio clamp: 0.1 (large std) and 10 (zero std)
        elif kind == 4:
            oq[2][r, 0], oq[3][r, 0] = 80.0, 90.0
    x = {"logits": [f32(torch.cat([mean, ls], 1)), f32(torch.cat([n(B, A), ls.flip(0)], 1))],
         "eps": [f32(eps), f32(n(B, A))], "hi": f32(1.0 + 0.25 * (torch.arange(A) % 3)),
         "lo": f32(-1.0 + 0.125 * (torch.arange(A) % 2)), "rew": f32(rew), "done": done, "z3": f32(z3), "z4": f32(z4),
         "out_q": [f32(q) for q in oq], "logp_new": f32(3 * n(B)), "logp2": f32(3 * n(B)),
         "d_act": [f32(0.01 * n(B, A)), f32(0.01 * n(B, A))]}
    return x


# kind, A, B, mode, auto_alpha, mean_std carried (else unset), bound, max_blocks, global batch factor
ROW_CASES = {}
GAUSS_KINDS = ("gauss", "mlp_gauss")   # the row kinds whose policy samples the plain Gaussian
for _A in (1, 2, 3, 17, 32, 33, 96):
    ROW_CASES[f"mlp_fp32_A{_A}"] = ("mlp", _A, 65, "fp32", _A % 2 == 1, _A % 3 == 0, True, 0, 1)
for _B in (1, 7, 8, 9, 63, 64):
    ROW_CASES[f"mlp_fp32_B{_B}"] = ("mlp", 3, _B, "fp32", _B % 2 == 0, _B % 3 == 0, True, 0, 1)
ROW_CASES.update({
    "mlp_bf16x3": ("mlp", 3, 65, "bf16x3", True, True, True, 0, 1),
    "mlp_bf16x3_A33": ("mlp", 33, 9, "bf16x3", False, False, True, 0, 2),
    "mlp_bf16": ("mlp", 17, 64, "bf16", True, True, True, 0, 1),
    "mlp_capped": ("mlp", 3, 200, "fp32", True, True, True, 1, 1),
    "mlp_wide_ms": ("mlp", 2, 65, "fp32", True, "wide", True, 0, 1),
    "v1_bf16x3_A1": ("v1", 1, 65, "bf16x3", True, False, True, 0, 1),
    "v1_bf16x3": ("v1", 3, 64, "bf16x3", False, False, True, 0, 1),
    "v1_fp32_nll": ("v1", 2, 63, "fp32", True, False, False, 0, 1),
    "separated": ("separated", 3, 65, "fp32", True, True, True, 0, 1),
    "parameter": ("parameter", 2, 63, "fp32", False, False, True, 0, 1),
    "gauss": ("gauss", 3, 65, "fp32", True, True, True, 0, 1),
    # the plain Gaussian on MLP-engine handles (the log_std half in the policy's 2A outputs; bf16x3 images of the rows)
    "mlp_gauss": ("mlp_gauss", 3, 65, "fp32", True, True, True, 0, 1),
    "mlp_gauss_bf16x3": ("mlp_gauss", 17, 63, "bf16x3", False, False, True, 0, 2),
    "heads_v1_bound": ("heads_v1", 3, 65, "fp32", True, False, True, 0, 1),
    "heads_v1_nll": ("heads_v1", 3, 9, "fp32", False, False, False, 2, 1),
    "mlp_past_grid": ("mlp", 2, "grid", "fp32", True, True, True, 0, 1),
})


def case_inputs(name: str, B: int, hy: dict):
    """The inputs of ROW_CASES[name] at B rows (its own B, or the grid-derived one): row_inputs, with the zero-std rows
    moved to raw std -10 where the Gaussian NLL of DSAC_V1 divides by the std."""
    kind, A, _, _, _, _, bound, _, _ = ROW_CASES[name]
    x = row_inputs(A, B, 7 + A + B, hy)
    if kind in ("v1", "heads_v1") and not bound:
        for q in x["out_q"]:
            q[:, 1] = torch.where(q[:, 1] < -50, torch.full_like(q[:, 1], -10.0), q[:, 1])
    return x


def case_mean_std(carried):
    """The carried mean_std pair of a case: wide (3 m past Huber's 50), ordinary, or unset."""
    return [20.0, 20.5] if carried == "wide" else ([1.25, 0.75] if carried else [-1.0, -1.0])


# ---- Adam / Polyak cases ---------------------------------------------------------------------------------------------
ADAM_HY = dict(tau=0.005, lr_q=1e-4, lr_pi=1e-4, lr_alpha=3e-4, adam_beta1=0.9, adam_beta2=0.999, adam_eps=1e-8)
ADAM_T = (0, 1, 2, 10 ** 6)   # the critics' counter; the policy's is one less (at least 0)
# (delayed, auto_alpha, scalars_ready, slots): the step sizes formed in the kernel; read from the slots; read over a stamp
# that matches the counters (slots hold 1.5x the formed values, which the kernel must use); a stale stamp (slots hold 7,
# which the kernel must not use)
APPLY_RUNS = ((True, True, 0, None), (False, True, 2, "stale"), (True, False, 1, "slots"), (False, False, 0, None),
              (True, True, 2, "valid"))


def adam_layouts():
    """fp32-mode DSAC-T and DSAC_V1 shapes (obs, hidden, v1) whose critic span n_q2 and n_params take every residue mod 4,
    and n_params of each."""
    from dsac_v2_b200.engine import make_config, make_v1_options, query_layout
    got = {}
    for obs in range(3, 12):
        for h in (5, 6, 7, 8):
            for v1 in (False, True):
                lay = query_layout(make_config(obs, 2, [h], [h], max_batch=16), make_v1_options() if v1 else None)
                nq2 = lay.n_q * (1 if v1 else 2)
                got.setdefault((nq2 % 4, lay.n_params % 4), (obs, h, v1, int(lay.n_params), int(nq2)))
    return got


def adam_inputs(n: int, seed: int, big=False):
    """fp32 values (float64) of params, targets, grads, exp_avg, exp_avg_sq for n parameters: g = 0 (and v = 0) on every
    7th element, and with `big` g = 3e21 on every 11th, where (1 - beta2) g g overflows fp32 in the kernel's order."""
    g = torch.Generator().manual_seed(seed)
    r = lambda s=1.0: (torch.randn(n, generator=g) * s).float().double()
    w, t, gr = r(), r()[:-1], r(1e-2)
    gr[::7] = 0.0
    if big:
        gr[3::11] = 3e21
    m, v = r(1e-3), r(1e-4).abs()
    v[::7] = 0.0
    return dict(w=w, t=t, g=gr, m=m, v=v)


def apply_run_sizes(t: int, slots):
    """(tq, tp) and the step sizes the kernel must use in one of APPLY_RUNS, and the slot values the test writes."""
    tq, tp = t, max(t - 1, 0)
    sh = adam_step_sizes(ADAM_HY, tq, tp)
    written = None
    if slots in ("slots", "valid"):
        sh = [c32(x * 1.5) for x in sh]
        written = sh
    elif slots == "stale":
        written = [7.0] * 5
    return tq, tp, sh, written

