"""The dense-layer kernels one by one (dsact_test_gemm) and the fused layer chain (dsact_test_chain) against the float64
reference of tests/tc_ref.py, which rounds the operands the way the kernels do: the gates hold only the fp32
accumulation, the epilogue's rounding and the activation approximation, in all three modes.  Outputs start as NaN, so an
element a kernel fails to write fails its check; images are read back whole, padding included."""
import math

import pytest
import torch

import tc_ref as R
from dsac_v2_b200 import _lib

pytestmark = pytest.mark.gpu

MODES = ["fp32", "bf16x3", "bf16"]
ACT = _lib.ACTIVATIONS
VARIANT = {"fwd": 0, "dgrad": 1, "wgrad": 2}
EPI = {"fwd": 1, "dgrad": 2, "wgrad": 0}
NAN = float("nan")


def _engine(mode):
    from dsac_v2_b200.engine import Engine, make_config
    lim = torch.ones(2)
    e = Engine(make_config(5, 2, [32, 32], [32, 32], max_batch=16, gemm_mode=mode), torch.device("cuda", 0), lim, -lim)
    e.mode = mode
    return e


@pytest.fixture(scope="module", params=MODES)
def eng(request):
    e = _engine(request.param)
    yield e
    e.close()


@pytest.fixture(scope="module", params=["bf16x3", "bf16"])
def tc_eng(request):
    e = _engine(request.param)
    yield e
    e.close()


def _report(mode, what, ratios):
    """The largest err / gate of each checked output (printed for DESIGN.md §5), then the gate."""
    for k, r in ratios.items():
        print(f"ERR/GATE {mode} {what} {k} {r:.4g}")
    bad = {k: r for k, r in ratios.items() if not r <= 1.0}
    assert not bad, bad


def _planes(mode):
    return 2 if mode == "bf16x3" else 1


def _nan_img(M, N):
    return torch.full((2, M, (N + 7) // 8 * 8), NAN, dtype=torch.bfloat16, device="cuda")


def _check_image(img, want, mode):
    """img (device, [2, M, pitch]) holds the round-to-nearest split of the fp32 values `want` [M, N], bit for bit, and
    zeros in its padding columns."""
    img = img.cpu()
    N = want.shape[1]
    R.check_split(img[:_planes(mode)], N, _planes(mode))
    hi, lo = R.split(want.cpu())
    assert torch.equal(img[0, :, :N].double(), hi), "hi plane"
    if mode == "bf16x3":
        assert torch.equal(img[1, :, :N].double(), lo), "lo plane"


# ---- per-layer kernels -----------------------------------------------------------------------------------------------
def _layer_problems(case, x, mode, with_img=True):
    """dsact_test_layer dicts of one case: the checked problem, and in the tensor-core modes a copy that stores the
    output image instead (forward / dgrad)."""
    v, M, N = case["variant"], case["M"], case["N"]
    d = lambda t: None if t is None else t.cuda()
    out = {}
    if v == "wgrad":
        out["C"] = x["C0"].clone().cuda()
        return [dict(M=M, N=N, K0=case["K0"], A0=d(x["A0"]), B=d(x["B"]), C=out["C"])], out
    p = dict(M=M, N=N, K0=case["K0"], K1=case["K1"], kB1=case["kB1"], A0=d(x["A0"]), B=d(x["B"]), epi=EPI[v],
             act=ACT[case["act"]])
    if case["K1"]:
        p["A1"] = d(x["A1"])
    out["C"] = torch.full((M, N), NAN, device="cuda")
    if v == "fwd":
        out["Zout"] = torch.full((M, N), NAN, device="cuda")
        p.update(bias=d(x["bias"]), Zout=out["Zout"])
    else:
        out["colsum"] = x["colsum0"].clone().cuda()
        p.update(Zin=d(x["Z"] if mode == "fp32" else x["D"]), colsum=out["colsum"])
    probs = [dict(p, C=out["C"])]
    if mode != "fp32" and with_img:
        out["img"] = _nan_img(M, N)
        q = dict(p, img=out["img"])
        q.pop("Zout", None)
        q.pop("colsum", None)
        probs.append(q)
    return probs, out


def _check_layer(mode, case, x, out):
    ref = R.layer_ref(case, x, mode)
    ratios = {k: R.ratio(out[k].cpu(), v, g, m) for k, (v, g, m) in ref.items()}
    if "img" in out:
        _check_image(out["img"], out["C"], mode)
    return ratios


@pytest.mark.parametrize("name", list(R.LAYER_CASES))
def test_layer_against_float64(eng, name):
    case = R.LAYER_CASES[name]
    x = R.layer_inputs(case)
    probs, out = _layer_problems(case, x, eng.mode)
    eng.test_layers(VARIANT[case["variant"]], probs)
    torch.cuda.synchronize()
    _report(eng.mode, name, _check_layer(eng.mode, case, x, out))


def test_group_of_more_than_eight_problems(eng):
    """Ten forward problems in one group: in fp32 mode the SIMT lowering issues two launches."""
    names = ["fwd_linear", "fwd_relu", "fwd_gelu", "fwd_tanh", "fwd_sigmoid", "fwd_elu", "fwd_selu", "fwd_n3", "fwd_n45",
             "fwd_seg_11_3"]
    cases = [R.LAYER_CASES[n] for n in names]
    xs = [R.layer_inputs(c) for c in cases]
    probs, outs = [], []
    for c, x in zip(cases, xs):
        p, o = _layer_problems(c, x, eng.mode, with_img=False)
        probs += p
        outs.append(o)
    assert len(probs) == 10
    eng.test_layers(0, probs)
    torch.cuda.synchronize()
    ratios = {}
    for n, c, x, o in zip(names, cases, xs, outs):
        for k, r in _check_layer(eng.mode, c, x, o).items():
            ratios[f"{n}.{k}"] = r
    _report(eng.mode, "group10", ratios)


def test_launches_of_bounded_size(tc_eng):
    """max_ctas slices a group into several launches with per-launch first tiles; the result is the same bits."""
    cases = [R.LAYER_CASES[n] for n in ("fwd_m4096", "fwd_n520", "fwd_seg_376_17")]
    xs = [R.layer_inputs(c) for c in cases]
    res = []
    for max_ctas in (0, 7):
        probs, outs = [], []
        for c, x in zip(cases, xs):
            p, o = _layer_problems(c, x, tc_eng.mode)
            probs += p
            outs.append(o)
        tc_eng.test_layers(0, probs, max_ctas=max_ctas)
        torch.cuda.synchronize()
        res.append(outs)
    for a, b in zip(*res):
        for k in a:
            assert torch.equal(a[k].view(torch.int16) if a[k].dtype == torch.bfloat16 else a[k],
                               b[k].view(torch.int16) if b[k].dtype == torch.bfloat16 else b[k]), k


@pytest.mark.parametrize("variant", ["fwd", "dgrad"])
def test_paired_and_single_accesses_give_the_same_bits(eng, variant):
    """Even leading dimensions on 8-byte aligned bases take the epilogue's 8-byte loads and stores, odd ones or 4-byte
    offset bases the 4-byte ones: the arithmetic must not differ."""
    case = R.LAYER_CASES["fwd_n45" if variant == "fwd" else "dgrad_n45"]
    case = dict(case, N=46)
    x = R.layer_inputs(case)
    M, N = case["M"], case["N"]
    res = []
    for ld, off in ((N, 0), (N + 1, 1), (N + 2, 1), (N + 1, 0)):
        big = lambda: torch.full((M * ld + 8,), NAN, device="cuda")[off:off + M * ld].view(M, ld)
        C = big()
        p = dict(M=M, N=N, K0=case["K0"], A0=x["A0"].cuda(), B=x["B"].cuda(), epi=EPI[variant], act=ACT[case["act"]], C=C)
        if variant == "fwd":
            bias = torch.zeros(N + 1, device="cuda")[off:off + N]
            bias.copy_(x["bias"])
            p.update(bias=bias, Zout=big())
        else:
            Z = big()
            Z[:, :N].copy_((x["Z"] if eng.mode == "fp32" else x["D"]).cuda())
            p.update(Zin=Z, ldz=ld)
        eng.test_layers(VARIANT[variant], [p])
        torch.cuda.synchronize()
        res.append([C[:, :N].clone()] + ([p["Zout"][:, :N].clone()] if variant == "fwd" else []))
    for r in res[1:]:
        for a, b in zip(res[0], r):
            assert torch.equal(a, b)


# ---- fused layer chains ----------------------------------------------------------------------------------------------
def chain_case(name, hidden, K0, head, M, act, K1=0, kB1=0, passes=1):
    return dict(name=name, hidden=hidden, K0=K0, K1=K1, kB1=kB1, head=head, M=M, act=act, passes=passes)


CHAIN_CASES = {c["name"]: c for c in [
    chain_case("w8_64_256", [8, 64, 256], 5, 2, 65, "gelu"),
    chain_case("w56_72_136", [56, 72, 136], 64, 34, 63, "relu"),
    chain_case("w128_192_200_248", [128, 192, 200, 248], 376, 192, 200, "tanh"),
    chain_case("deep256", [256] * 6, 11, 2, 4096, "gelu", K1=3, kB1=64),
    chain_case("w192_m1", [192], 64, 1, 1, "elu", K1=5, kB1=64),
    chain_case("w136_8", [136, 8], 376, 2, 64, "selu", K1=17, kB1=384),
    chain_case("w64x5", [64] * 5, 5, 2, 65, "sigmoid"),
    chain_case("w256_4pass_m8192", [256, 256], 376, 2, 8192, "gelu", K1=17, kB1=384, passes=4),
    chain_case("w248_40_linear", [248, 40], 120, 2, 97, "linear"),
    # six hidden layers whose ring items per tile (k-blocks x column halves) mix odd and even: 1, 2, 3, 2, 4, 4, then 3 for
    # the head; the ping-pong kernel's turns and parity waits go through many ring phases
    chain_case("ring_parity6", [64, 192, 8, 256, 72, 136], 5, 2, 1000, "elu"),
]}
# tiling: None selects the kernel by launch shape, 0 forces the column split, 1 the ping-pong kernel
TILINGS = {"by_shape": None, "column_split": 0, "pingpong": 1}
# the passes the ping-pong runs add: 161 rows (two full tiles, the kind bodies; then a CTA whose only tile is ragged) and
# 97 rows (a CTA whose second tile is ragged)
PP_EXTRA_ROWS = [161, 97]
MAX_PASSES = 4


def chain_rows(case, tiling):
    """The rows of each pass of one launch of the case: its own passes, and under the ping-pong kernel PP_EXTRA_ROWS from
    the second pass on (at most MAX_PASSES passes)."""
    rows = [case["M"]] * case["passes"]
    if tiling == 1:
        rows = (rows[:1] + PP_EXTRA_ROWS + rows[1:])[:MAX_PASSES]
    return rows


def pp_ctas(M):
    """The kinds of ping-pong CTA a pass of M rows has: "full" (a tile of 64 rows), "ragged2" (a second tile below 64
    rows), "missing2" (no second tile)."""
    tiles = (M + 63) // 64
    kinds = {"full"} if M >= 64 else set()
    kinds.add("missing2" if tiles % 2 else ("ragged2" if M % 64 else "full"))
    return kinds


def _chain_params(sizes, g):
    """Flat [W_0 | b_0 | ...]: weights ~ 1/sqrt(fan-in); every bias starts with 0, +-4, +-12."""
    parts = []
    for j in range(len(sizes) - 1):
        parts.append(torch.randn(sizes[j + 1], sizes[j], generator=g) / math.sqrt(sizes[j]))
        b = torch.randn(sizes[j + 1], generator=g) * 0.5
        fixed = torch.tensor([0.0, 4.0, -4.0, 12.0, -12.0])
        b[:min(5, b.numel())] = fixed[:min(5, b.numel())]
        parts.append(b)
    return parts


def _chain_setup(case, seed):
    sizes = [case["K0"] + case["K1"]] + case["hidden"] + [case["head"]]
    g = torch.Generator().manual_seed(seed)
    parts = _chain_params(sizes, g)
    return sizes, parts, torch.cat([p.reshape(-1) for p in parts]).cuda(), g


def _fwd_pass(case, sizes, g, M, zout=True, img=True):
    x = torch.randn(M, sizes[0], generator=g)
    x[3::7] = 0.0
    L = len(sizes) - 2
    p = dict(M=M, x0=x[:, :case["K0"]].contiguous().cuda(), out=torch.full((M, sizes[-1]), NAN, device="cuda"))
    if case["K1"]:
        p["x1"] = x[:, case["K0"]:].contiguous().cuda()
    p["Zout"] = [torch.full((M, sizes[j + 1]), NAN, device="cuda") for j in range(L)] if zout else None
    p["img"] = [_nan_img(M, sizes[j + 1]) for j in range(L)] if img else None
    return x, p


def _img_value(img, width, mode):
    """hi + lo of a hidden image, and half an ulp of its last plane: the fp32 value it was split from lies that close."""
    v = R.check_split(img.cpu()[:_planes(mode)], width, _planes(mode))
    last = img.cpu()[_planes(mode) - 1, :, :width].double()
    return v, R.ulp(last) / 2


def _check_fwd_chain(mode, case, sizes, parts, x, p):
    L = len(sizes) - 2
    planes = R.operands(x, mode)
    ratios = {}
    for j in range(L + 1):
        W, b = parts[2 * j], parts[2 * j + 1]
        acc, ab = R.mm_planes(planes, R.operands(W, mode))
        gate = R.mm_gate(ab, sizes[j])
        if j == L:
            z = acc + b.double()
            ratios["head"] = R.ratio(p["out"].cpu(), z, gate + R.U * z.abs())
            break
        e = R.epilogue(acc, gate, case["act"], mode, b)
        ratios[f"Zout{j}"] = R.ratio(p["Zout"][j].cpu(), *e["d"], e["kink"])
        v, half = _img_value(p["img"][j], sizes[j + 1], mode)
        ratios[f"img{j}"] = R.ratio(v, *e["y"], slack=half)
        # teacher forcing: the next layer multiplies the kernel's own image
        hi = p["img"][j].cpu()[0, :, :sizes[j + 1]].double()
        planes = [hi, p["img"][j].cpu()[1, :, :sizes[j + 1]].double()] if mode == "bf16x3" else [hi]
    return ratios


@pytest.mark.parametrize("tiling", list(TILINGS.values()), ids=list(TILINGS))
@pytest.mark.parametrize("name", list(CHAIN_CASES))
def test_forward_chain_against_float64(tc_eng, name, tiling):
    case = CHAIN_CASES[name]
    sizes, parts, params, g = _chain_setup(case, 7)
    runs = [_fwd_pass(case, sizes, g, M) for M in chain_rows(case, tiling)]
    tc_eng.test_chain(False, sizes, case["K0"], case["K1"], case["kB1"], ACT[case["act"]], params, [p for _, p in runs],
                      tiling=tiling)
    torch.cuda.synchronize()
    ratios = {}
    for i, (x, p) in enumerate(runs):
        for k, r in _check_fwd_chain(tc_eng.mode, case, sizes, parts, x, p).items():
            ratios[f"p{i}.{k}"] = r
    _report(tc_eng.mode, f"chain_fwd.{name}", ratios)


@pytest.mark.parametrize("tiling", list(TILINGS.values()), ids=list(TILINGS))
def test_forward_pass_is_the_same_alone_in_a_group_and_without_stores(tc_eng, tiling):
    """One pass gives the same bits run alone, as the second of 4 passes of different lengths, and without its act' and
    image stores."""
    case = dict(CHAIN_CASES["w128_192_200_248"], K1=17, kB1=384, K0=64)
    sizes, parts, params, g = _chain_setup(case, 11)
    runs = [_fwd_pass(case, sizes, g, m) for m in (65, 200, 1, 130)]
    act = ACT[case["act"]]
    tc_eng.test_chain(False, sizes, case["K0"], case["K1"], case["kB1"], act, params, [p for _, p in runs], tiling=tiling)
    x, p = runs[1]
    alone = dict(p, out=torch.full_like(p["out"], NAN), Zout=[torch.full_like(z, NAN) for z in p["Zout"]],
                 img=[torch.full_like(i, NAN) for i in p["img"]])
    bare = dict(p, out=torch.full_like(p["out"], NAN), Zout=None, img=None)
    tc_eng.test_chain(False, sizes, case["K0"], case["K1"], case["kB1"], act, params, [alone], tiling=tiling)
    tc_eng.test_chain(False, sizes, case["K0"], case["K1"], case["kB1"], act, params, [bare], tiling=tiling)
    torch.cuda.synchronize()
    assert torch.equal(p["out"], alone["out"]) and torch.equal(p["out"], bare["out"])
    for a, b in zip(p["Zout"], alone["Zout"]):
        assert torch.equal(a, b)
    for a, b in zip(p["img"], alone["img"]):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    _report(tc_eng.mode, "chain_fwd.group_of_4", _check_fwd_chain(tc_eng.mode, case, sizes, parts, x, p))


@pytest.mark.parametrize("tiling", list(TILINGS.values()), ids=list(TILINGS))
@pytest.mark.parametrize("name", list(CHAIN_CASES))
def test_dgrad_chain_against_float64(tc_eng, name, tiling):
    """dz_{j-1} = (dz_j W_j) * act'(z_{j-1}) down the hidden layers, the bias gradients (accumulated onto non-zero
    values) and the action columns' gradient read through the dact window at the step's column kB1 of W_0's image."""
    case = CHAIN_CASES[name]
    mode = tc_eng.mode
    sizes, parts, params, g = _chain_setup(case, 13)
    L = len(sizes) - 2
    runs = []
    for M in chain_rows(case, tiling):
        dout = torch.randn(M, sizes[-1], generator=g)
        dout[3::7] = 0.0
        D = [torch.rand(M, sizes[j + 1], generator=g) * 2.0 - 0.25 for j in range(L)]
        cs0 = [torch.randn(sizes[j + 1], generator=g) for j in range(L)]
        p = dict(M=M, x0=dout.cuda(), Zin=[d.cuda() for d in D], colsum=[c.clone().cuda() for c in cs0],
                 img=[_nan_img(M, sizes[j + 1]) for j in range(L)])
        if case["K1"]:
            p["out"] = torch.full((M, case["K1"]), NAN, device="cuda")
        runs.append((dout, D, cs0, p))
    tc_eng.test_chain(True, sizes, case["K0"], case["K1"], case["kB1"], ACT[case["act"]], params, [r[3] for r in runs],
                      tiling=tiling)
    torch.cuda.synchronize()
    ratios = {}
    for i, (dout, D, cs0, p) in enumerate(runs):
        planes = R.operands(dout, mode)
        for j in range(L, 0, -1):
            acc, ab = R.mm_planes(planes, R.operands(parts[2 * j].t().contiguous(), mode))
            gate = R.mm_gate(ab, sizes[j + 1])
            d = D[j - 1].double()
            y = acc * d
            gy = gate * d.abs() + R.U * y.abs()
            v, half = _img_value(p["img"][j - 1], sizes[j], mode)
            ratios[f"p{i}.dz{j - 1}"] = R.ratio(v, y, gy, slack=half)
            cs = cs0[j - 1].double() + y.sum(0)
            gcs = gy.sum(0) + (y.shape[0] / 64 + 8) * R.U * (y.abs().sum(0) + cs0[j - 1].abs().double())
            ratios[f"p{i}.colsum{j - 1}"] = R.ratio(p["colsum"][j - 1].cpu(), cs, gcs)
            im = p["img"][j - 1].cpu()
            hi = im[0, :, :sizes[j]].double()
            planes = [hi, im[1, :, :sizes[j]].double()] if mode == "bf16x3" else [hi]
        if case["K1"]:
            W0a = parts[0][:, case["K0"]:].t().contiguous()
            acc, ab = R.mm_planes(planes, R.operands(W0a, mode))
            ratios[f"p{i}.dact"] = R.ratio(p["out"].cpu(), acc, R.mm_gate(ab, sizes[1]) + R.U * acc.abs())
    _report(mode, f"chain_dgrad.{name}", ratios)


def test_chain_case_table_covers_the_layer_bodies():
    widths = {w for c in CHAIN_CASES.values() for w in c["hidden"]}
    assert {8, 56, 64, 72, 128, 136, 192, 200, 248, 256} <= widths
    assert set(range(1, _lib.MAX_HIDDEN + 1)) <= {len(c["hidden"]) for c in CHAIN_CASES.values()}
    assert {1, 2, 34, 192} <= {c["head"] for c in CHAIN_CASES.values()}
    assert {(5, 0), (64, 0), (376, 0), (11, 3), (64, 5), (376, 17)} <= {(c["K0"], c["K1"]) for c in CHAIN_CASES.values()}
    assert {1, 63, 64, 65, 200, 4096, 8192} <= {c["M"] for c in CHAIN_CASES.values()}
    assert set(ACT) == {c["act"] for c in CHAIN_CASES.values()}
    # under the ping-pong kernel every activation meets a full tile, a CTA whose second tile is ragged and one whose
    # second tile is missing
    for act in ACT:
        kinds = {k for c in CHAIN_CASES.values() if c["act"] == act for M in chain_rows(c, 1) for k in pp_ctas(M)}
        assert kinds == {"full", "ragged2", "missing2"}, (act, kinds)
    assert all(len(chain_rows(c, t)) <= MAX_PASSES for c in CHAIN_CASES.values() for t in TILINGS.values())
