"""CPU checks of the float64 restatement (tests/step_ref.py) that tests/test_gpu_step_kernels.py holds the step kernels to:
composed with the networks it reproduces the float64 oracle's gradients and Adam / Polyak update, the GPU cases take
both sides of every branch on a computed value, and every gate is narrow enough to see each emulated kernel fault by at
least step_ref.POWER gates."""
import math

import pytest
import torch

import step_ref as R
from dsac_v2_b200 import synth
from oracle.dsact_oracle import from_config, mlp_forward

HY = dict(gamma=0.99, tau=0.005, tau_b=0.005, alpha=0.2, min_log_std=-20.0, max_log_std=0.5, lr_q=1e-4, lr_pi=1e-4,
          lr_alpha=3e-4, td_bound=20.0, adam_beta1=0.9, adam_beta2=0.999, adam_eps=1e-8)


def test_cases_take_both_sides_of_every_computed_branch():
    sc = R.scalars(HY)
    seen = {}
    for name, (kind, A, B, mode, auto, carried, bound, cap, gbf) in R.ROW_CASES.items():
        if B == "grid" or kind in ("v1", "heads_v1"):
            continue
        x = R.row_inputs(A, B, 7 + A + B, HY)
        _, amb, sides = R.loss_ref(x, sc, dict(stdsum=[0.9 * B, 1.1 * B], mean_std=R.case_mean_std(carried)), B * gbf, auto, -1.3)
        assert int(amb.sum()) <= 0.01 * B + 1, name
        for k, s in sides.items():
            key = k.rstrip("01")
            prev = seen.get(key, [False] * len(s))
            seen[key] = [a or bool((m & ~amb).any()) for a, m in zip(prev, s)]
    x = R.row_inputs(3, 65, 75, HY)
    _, amb, sides = R.loss_v1_ref(x, R.scalars(HY), 65, True, -1.3)
    seen["td"] = [bool((m & ~amb).any()) for m in sides["td"]]
    assert all(all(v) for v in seen.values()), seen


def test_regime_rows_sit_on_the_input_branches():
    x = R.row_inputs(3, 90, 1, HY)
    ls = x["logits"][0][:, 3:]
    lo, hi = R.c32(HY["min_log_std"]), R.c32(HY["max_log_std"])
    assert bool((ls == lo).any()) and bool((ls == hi).any()) and bool((ls < lo).any()) and bool((ls > hi).any())
    raws = torch.cat([q[:, 1] for q in x["out_q"]])
    assert {-120.0, 20.0, R.nextafter(20.0, 100), 60.0} <= set(raws.tolist())
    assert {3.0, -3.0} <= set(x["z3"].tolist()) | set(x["z4"].tolist())
    assert bool((x["out_q"][2][:, 0] == x["out_q"][3][:, 0]).any()) and bool((x["out_q"][4][:, 0] == x["out_q"][5][:, 0]).any())
    assert {0.0, 1.0} == set(x["done"].tolist())


# ---- the restatement against the float64 oracle ------------------------------------------------------------------------
def test_restatement_composed_with_the_networks_is_the_float64_oracle():
    """Per-row restated gradients, pulled back through the networks by autograd, are the float64 oracle's parameter
    gradients; the restated Adam / Polyak is its update."""
    cfg = synth.CONFIGS["tiny"]
    B, A = 16, cfg["act_dim"]
    w = synth.make_weights(cfg)
    orc = from_config(cfg, w, dtype=torch.float64, **synth.HYPER)
    batch = {k: torch.from_numpy(v).double() for k, v in synth.make_batch(cfg, B, 0).items()}
    noise = [torch.from_numpy(n).double() for n in synth.make_noise(cfg, B, 0)]
    orc.compute_gradients(batch, noise)
    hy = dict(HY, **{k: synth.HYPER[k] for k in ("gamma", "tau") if k in synth.HYPER})
    hy["tau_b"] = synth.HYPER.get("tau_b", hy["tau"])
    hy["alpha"] = synth.HYPER.get("alpha", 0.2)
    with R.exact_constants():
        sc = R.scalars(hy)
        P = {k: [p.detach().clone().requires_grad_(True) for p in v] for k, v in orc.p.items()}
        T = orc.t
        lim = torch.full((A,), float(cfg["act_lim"]), dtype=torch.float64)
        la = float(orc.log_alpha.detach())
        logits = mlp_forward(P["policy"], batch["obs"], orc.act_pi)
        logitsT = mlp_forward(T["policy"], batch["obs2"], orc.act_pi).detach()
        s0 = R.sample_ref({"logits": logits.detach(), "eps": noise[0], "hi": lim, "lo": -lim}, sc)
        s1 = R.sample_ref({"logits": logitsT, "eps": noise[1], "hi": lim, "lo": -lim}, sc)
        new_act = s0["act"][0].requires_grad_(True)
        qf = lambda net, o, a: mlp_forward(net, torch.cat([o, a], -1), orc.act_q)
        oq = [qf(P["q1"], batch["obs"], batch["act"]), qf(P["q2"], batch["obs"], batch["act"]),
              qf(T["q1"], batch["obs2"], s1["act"][0]).detach(), qf(T["q2"], batch["obs2"], s1["act"][0]).detach(),
              qf([p.detach() for p in P["q1"]], batch["obs"], new_act), qf([p.detach() for p in P["q2"]], batch["obs"], new_act)]
        x = {"rew": batch["rew"], "done": batch["done"], "z3": noise[4], "z4": noise[5], "logp_new": s0["logp"][0],
             "logp2": s1["logp"][0], "out_q": [q.detach() for q in oq]}
        stdsum = [float(torch.nn.functional.softplus(oq[k][:, 1].detach()).sum()) for k in range(2)]
        o, _, _ = R.loss_ref(x, sc, dict(stdsum=stdsum, mean_std=[-1.0, -1.0]), B, True, la)
        for k, net in enumerate(("q1", "q2")):
            d = torch.stack([o[f"g_mean{k}"][0], o[f"g_raw{k}"][0]], 1)
            g = torch.autograd.grad(oq[k], P[net], d)
            for a, b in zip(g, orc.grads[net]):
                torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-14)
        d_act = [torch.autograd.grad(oq[4 + k], new_act, torch.stack([o[f"g_pa{k}"][0], torch.zeros(B, dtype=torch.float64)], 1),
                                     retain_graph=True)[0] for k in range(2)]
        gu, gl = R.pgrad_ref({"logits": logits.detach(), "eps": noise[0], "d_act1": d_act[0], "d_act2": d_act[1], "hi": lim,
                              "lo": -lim}, sc, B, True, la)
        g = torch.autograd.grad(logits, P["policy"], torch.cat([gu[0], gl[0]], 1))
        for a, b in zip(g, orc.grads["policy"]):
            torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-14)
        gla, _ = R.log_alpha_grad(float(s0["logp"][0].sum()), B, B, A)
        torch.testing.assert_close(torch.tensor(float(gla), dtype=torch.float64), orc.grads["log_alpha"][0].reshape(()), rtol=1e-12, atol=1e-14)

        # Adam / Polyak of one delayed iteration, against the oracle's _adam / apply
        flat = lambda d: torch.cat([t.reshape(-1) for n in ("q1", "q2", "policy") for t in d[n]])
        wv = torch.cat([flat(orc.p).detach(), orc.log_alpha.detach().reshape(1)])
        gv = torch.cat([flat(orc.grads), orc.grads["log_alpha"][0].reshape(1)])
        tv = flat(orc.t).detach()
        zeros = torch.zeros_like(wv)
        nq2 = sum(t.numel() for n in ("q1", "q2") for t in orc.p[n])
        ref = R.apply_ref(wv, gv, zeros, zeros, tv, (), nq2, hy, R.adam_step_sizes(hy, 0, 0), torch.tensor(True), True)
        orc.apply(0)
        torch.testing.assert_close(ref["w"][0], torch.cat([flat(orc.p).detach(), orc.log_alpha.detach().reshape(1)]),
                                   rtol=1e-12, atol=1e-15)
        torch.testing.assert_close(ref["t"][0], flat(orc.t).detach(), rtol=1e-12, atol=1e-15)


# ---- power: every fault moves a checked output by POWER gates in the GPU test's cases --------------------------------------
GPU_HY = dict(HY)   # the hyperparameters tests/test_gpu_step_kernels.py gives its handles
LOG_ALPHA = R.c32(-1.3)
_ok = {}


def _row_outputs(name, fault=None):
    """The outputs test_row_kernels_against_float64 checks in case `name`, restated ({name: (value, gate)}; the loss only
    on the rows it does not skip), with the loss fed the restated sample and std sums as the kernels feed it."""
    kind, A, B, mode, auto, carried, bound, cap, gbf = R.ROW_CASES[name]
    gb = B * gbf
    v1, gauss = kind in ("v1", "heads_v1"), kind in R.GAUSS_KINDS
    sc = R.scalars(GPU_HY)
    x = R.case_inputs(name, B, GPU_HY)
    res = {}
    for w in range(2):
        s = R.sample_ref({"logits": x["logits"][w], "eps": x["eps"][w], "hi": x["hi"], "lo": x["lo"]}, sc, gauss, v1, fault)
        res[f"act{w}"], res[f"logp{w}"] = s["act"], s["logp"]
        if w == 0:
            tm = (s["tm"][0][:, 0], s["tm"][1][:, 0]) if v1 else (s["tm"][0].reshape(-1), s["tm"][1].reshape(-1))
            sd = s["v1_std"] if v1 else (s["sd"][0].reshape(-1), s["sd"][1].reshape(-1))
            res["acc_tanh_mean"] = R.sum_gate(*tm, tm[0].numel() + 1)
            res["acc_pi_std"] = R.sum_gate(*sd, sd[0].numel() + 1)
    x["logp_new"], x["logp2"] = res["logp0"][0], res["logp1"][0]
    stdsum = []
    for k in range(1 if v1 else 2):
        sp = R.stdsum_ref(x["out_q"][k][:, 1], fault)
        res[f"stdsum{k}"] = R.sum_gate(*sp, B + 1)
        stdsum.append(float(res[f"stdsum{k}"][0]))
    if v1:
        o, amb, _ = R.loss_v1_ref(x, sc, gb, auto, LOG_ALPHA, bound, fault)
    else:
        o, amb, _ = R.loss_ref(x, sc, dict(stdsum=stdsum, mean_std=R.case_mean_std(carried)), gb, auto, LOG_ALPHA, fault)
    for k, v in o.items():
        if k.startswith("g_"):
            res[k] = (v[0][~amb], v[1][~amb])
    gu, gl = R.pgrad_ref({"logits": x["logits"][0], "eps": x["eps"][0], "d_act1": x["d_act"][0],
                          "d_act2": None if kind == "v1" else x["d_act"][1], "hi": x["hi"], "lo": x["lo"]}, sc, gb, auto,
                         LOG_ALPHA, gauss, fault)
    res["d_mean"], res["d_log_std"] = gu, gl
    return res


def _margin(ok, bad):
    """max over the outputs of |faulty - correct| / gate (a NaN or infinite faulty value counts as infinite)."""
    best = 0.0
    for k, (v, g) in ok.items():
        fv = bad[k][0]
        if fv.shape != v.shape:
            return math.inf
        d = (fv - v).abs() / g
        d = torch.where(torch.isnan(fv) & ~torch.isnan(v), torch.full_like(d, math.inf), d)
        d = torch.where(fv == v, torch.zeros_like(d), d)
        best = max(best, float(d.nan_to_num(0.0, math.inf).max()) if d.numel() else 0.0)
    return best


_DSACT = ("mlp", "separated", "parameter", "gauss", "mlp_gauss")
_V1 = ("v1", "heads_v1")
ROW_FAULTS = {   # fault: (emulated fault, the cases of ROW_CASES it applies to)
    "tg_eps_logp": ("tg_eps_logp", lambda c: c[0] not in R.GAUSS_KINDS),
    "tg_eps_grad": ("tg_eps_grad", lambda c: c[0] not in R.GAUSS_KINDS),
    "clamp_mask_exclusive": ("clamp_mask_exclusive", lambda c: True),
    "no_clamp_sample": ("no_clamp_sample", lambda c: True),
    "tie_gpa_one": ("tie_gpa_one", lambda c: c[0] in _DSACT),
    "tie_target_c1": ("tie_target_c1", lambda c: c[0] in _DSACT),
    "no_zclamp": ("no_zclamp", lambda c: True),
    "done_ignored": ("done_ignored", lambda c: True),
    "huber_unclamped": ("huber_unclamped", lambda c: c[0] in _DSACT),
    "no_ratio_clamp": ("no_ratio_clamp", lambda c: c[0] in _DSACT),
    "neighbour": ("neighbour", lambda c: True),
    "v1_no_td_clamp": ("v1_no_td_clamp", lambda c: c[0] in _V1 and c[6]),
    "v1_gsd_sign_bound": ("v1_gsd_sign", lambda c: c[0] in _V1 and c[6]),
    "v1_gsd_sign_nll": ("v1_gsd_sign", lambda c: c[0] in _V1 and not c[6]),
    "gauss_squash": ("gauss_squash", lambda c: c[0] in R.GAUSS_KINDS),
    "v1_stats_pick_A1": ("v1_stats_pick", lambda c: c[0] in _V1 and c[1] == 1),
    "v1_stats_pick_A2plus": ("v1_stats_pick", lambda c: c[0] in _V1 and c[1] >= 2),
}


@pytest.mark.parametrize("fault", list(ROW_FAULTS))
def test_row_gates_see_every_fault(fault):
    """The largest move, over the GPU test's cases the fault applies to (all but the one sized from the device's SM
    count), of some checked output, in gates."""
    f, applies = ROW_FAULTS[fault]
    best, where = 0.0, None
    for name, case in R.ROW_CASES.items():
        if case[2] == "grid" or not applies(case):
            continue
        if name not in _ok:
            _ok[name] = _row_outputs(name)
        m = _margin(_ok[name], _row_outputs(name, f))
        if m > best:
            best, where = m, name
    print(f"POWER {fault} {best:.3g} ({where})")
    assert best >= R.POWER, f"{fault} moves the checked outputs by {best:.3g} gates < {R.POWER}"


def test_lost_grid_stride_trip_is_seen():
    """A trip lost in the capped case (one block: 8 rows a trip in sample / policy gradient, 64 in the loss) leaves its
    rows' outputs unwritten (NaN, as the outputs start) and their terms out of every sum."""
    name = "mlp_capped"
    _, A, B, _, _, _, _, cap, _ = R.ROW_CASES[name]
    ok = _ok.get(name) or _row_outputs(name)
    bad = {k: (v.clone(), g) for k, (v, g) in ok.items()}
    for k in ("act0", "logp0", "d_mean"):
        bad[k][0][B - 8:] = math.nan
    assert _margin({k: ok[k] for k in ("act0", "logp0", "d_mean")}, bad) >= R.POWER
    x = R.case_inputs(name, B, GPU_HY)
    s = R.sample_ref({"logits": x["logits"][0][:B - 8], "eps": x["eps"][0][:B - 8], "hi": x["hi"], "lo": x["lo"]},
                     R.scalars(GPU_HY))
    part = s["sd"][0].reshape(-1).sum()
    m = float((part - ok["acc_pi_std"][0]).abs() / ok["acc_pi_std"][1])
    print(f"POWER lost_trip {m:.3g}")
    assert m >= R.POWER


ADAM_FAULTS = ["bc_t", "eps_in_sqrt", "polyak_swap", "policy_nondelayed", "alpha_fixed_update", "stale_stamp",
               "valid_stamp_refused"]


def _adam_margin(fault):
    """The largest move, over the GPU test's Adam cases (the residue layouts, counters and runs), of some checked
    element, in gates."""
    best = 0.0
    for residue, (obs, h, v1, n, nq2) in sorted(R.adam_layouts().items()):
        for t in R.ADAM_T:
            x = R.adam_inputs(n, t + 17 * residue[0] + residue[1], big=(t == 1))
            for delayed, auto, ready, slots in R.APPLY_RUNS:
                tq, tp, sh, written = R.apply_run_sizes(t, slots)
                formed = ready == 0 or slots == "stale"
                f, sh_bad = fault, sh
                if fault == "bc_t":
                    if not formed:
                        continue
                    f, sh_bad = None, R.adam_step_sizes(R.ADAM_HY, tq, tp, "bc_t")
                elif fault == "stale_stamp":
                    if slots != "stale":
                        continue
                    f, sh_bad = None, written
                elif fault == "valid_stamp_refused":
                    if slots != "valid":
                        continue
                    f, sh_bad = None, R.adam_step_sizes(R.ADAM_HY, tq, tp)
                args = (x["w"], x["g"], x["m"], x["v"], x["t"], (), nq2, R.ADAM_HY)
                ok = R.apply_ref(*args, sh, torch.tensor(delayed), auto)
                bad = R.apply_ref(*args, sh_bad, torch.tensor(delayed), auto, fault=f)
                best = max(best, _margin({k: ok[k] for k in ("w", "m", "v", "t")}, bad))
    return best


@pytest.mark.parametrize("fault", ADAM_FAULTS)
def test_adam_gates_see_every_fault(fault):
    best = _adam_margin(fault)
    print(f"POWER {fault} {best:.3g}")
    assert best >= R.POWER


def test_log_alpha_gradient_over_rows_is_seen():
    v, g = R.log_alpha_grad(-37.5, 24, 40, 2)
    vb, _ = R.log_alpha_grad(-37.5, 24, 40, 2, fault="logalpha_rows")
    m = float(abs(vb - v) / g)
    print(f"POWER logalpha_rows {m:.3g}")
    assert m >= R.POWER


def test_adam_overflow_leaves_the_weight():
    """(1 - beta2) g g past the fp32 range in the kernel's order: v = inf, the step m / denom = 0, w unchanged."""
    obs, h, v1, n, nq2 = R.adam_layouts()[(0, 1)]
    x = R.adam_inputs(n, 1, big=True)
    out = R.apply_ref(x["w"], x["g"], x["m"], x["v"], x["t"], (), nq2, R.ADAM_HY, R.adam_step_sizes(R.ADAM_HY, 1, 0),
                      torch.tensor(True), True)
    big = x["g"] == 3e21
    assert bool(big.any()) and bool(torch.isinf(out["v"][0][big]).all()) and torch.equal(out["w"][0][big], x["w"][big])
