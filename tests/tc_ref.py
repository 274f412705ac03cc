"""Float64 restatement of the dense-layer kernels (gemm_tc.cuh, chain_tc.cuh, gemm_simt.cuh) with the operands rounded
the way the kernels round them, and the gates the GPU tests hold the kernels to.

The tensor-core modes multiply bf16 "images": hi = bf16_rn(x), lo = bf16_rn(x - hi) (image_kernel / split_pack2); bf16x3
sums hi*hi + hi*lo + lo*hi, bf16 hi*hi.  Every rounding of the operands is done here, so what separates a kernel from
`mm` is the fp32 accumulation, the fp32 epilogue and the activation approximation.  Matmul gate:

    gate = c(K) * 2^-24 * (|A_e| @ |W_e|^T)        c(K) = C_MM * sqrt(max(K, 16))

over the absolute values of the products the kernel sums (the same for all three modes).  The floor of 16: a wgmma
sums a whole k16 step (48 products in bf16x3) however few of them are non-zero, so a reduction over K = 2 (the gradient
of a two-output head) rounds like one over 16.  Hopper's wgmma accumulation
order and rounding are not documented, so C_MM is set from measurements on an H100 (DESIGN.md §5).
"""
import math

import torch

U = 2.0 ** -24                      # fp32 unit roundoff
C_MM = 2.0                          # c(K) / sqrt(max(K, 16)), DESIGN.md §5
GELU_TC = 3e-7                      # A&S 7.1.26 GELU of the tensor-core epilogue: error on Phi
ACTS = ("linear", "relu", "gelu", "tanh", "sigmoid", "elu", "selu")
SELU_L, SELU_A = 1.0507009873554805, 1.6732632423543772
# |act'| and |act''| bounds (Lipschitz constants of act and act')
LIP = {"linear": (1.0, 0.0), "relu": (1.0, 0.0), "gelu": (1.13, 0.8), "tanh": (1.0, 0.77), "sigmoid": (0.25, 0.1),
       "elu": (1.0, 1.0), "selu": (SELU_L * SELU_A, SELU_L * SELU_A)}
KINK = {"relu", "selu"}             # act' jumps at z = 0
POWER = 5.0                         # every emulated fault must move some checked output by this many gates


def bf16_rn(x, trunc=False):
    """fp32 -> bf16 (round to nearest even, or toward zero), as float64."""
    x = x.float()
    if trunc:
        return (x.view(torch.int32) & -65536).view(torch.float32).double()
    return x.to(torch.bfloat16).double()


def split(x, trunc=False):
    """hi, lo of the bf16 image of fp32 `x` (float64 tensors): hi = bf16(x), lo = bf16(x - hi), x - hi exact in fp32."""
    x = x.float()
    hi = bf16_rn(x, trunc)
    lo = bf16_rn((x.double() - hi).float(), trunc)
    return hi, lo


def operands(x, mode, trunc=False):
    """The planes of `x` the kernel multiplies: [x] (fp32), [hi, lo] (bf16x3), [hi] (bf16)."""
    if mode == "fp32":
        return [x.double()]
    hi, lo = split(x, trunc)
    return [hi, lo] if mode == "bf16x3" else [hi]


def mm_planes(a, w, drop_hilo=False):
    """sum of the plane products the kernel forms for out = A W^T (a, w: plane lists), and |A_e| @ |W_e|^T."""
    if len(a) == 1:
        pairs = [(0, 0)]
    else:
        pairs = [(0, 0), (1, 0)] + ([] if drop_hilo else [(0, 1)])
    val = sum(a[i] @ w[j].t() for i, j in pairs)
    ab = sum(a[i].abs() @ w[j].abs().t() for i, j in pairs)
    return val, ab


def mm(A, W, mode, **kw):
    """out = A W^T in float64 of the rounded operands (A [M, K], W [N, K] fp32), and the |products| sum."""
    return mm_planes(operands(A, mode), operands(W, mode), **kw)


def mm_gate(ab, K):
    return C_MM * math.sqrt(max(K, 16)) * U * ab


def act(z, a):
    z = z.double()
    if a == "linear":
        return z.clone()
    if a == "relu":
        return z.clamp_min(0.0)
    if a == "gelu":
        return 0.5 * z * (1.0 + torch.erf(z / math.sqrt(2.0)))
    if a == "tanh":
        return torch.tanh(z)
    if a == "sigmoid":
        return torch.sigmoid(z)
    if a == "elu":
        return torch.where(z > 0, z, torch.expm1(z))
    return SELU_L * torch.where(z > 0, z, SELU_A * torch.expm1(z))


def dact(z, a):
    z = z.double()
    if a == "linear":
        return torch.ones_like(z)
    if a == "relu":
        return (z > 0).double()
    if a == "gelu":
        return 0.5 * (1.0 + torch.erf(z / math.sqrt(2.0))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi)
    if a == "tanh":
        return 1.0 - torch.tanh(z) ** 2
    if a == "sigmoid":
        s = torch.sigmoid(z)
        return s * (1.0 - s)
    if a == "elu":
        return torch.where(z > 0, torch.ones_like(z), torch.exp(z))
    return SELU_L * torch.where(z > 0, torch.ones_like(z), SELU_A * torch.exp(z))


def act_approx(z, a, mode):
    """What the fp32 evaluation of act / act' may add beyond rounding of its argument: the A&S GELU of the tensor-core
    modes, a few ulps of the libm functions otherwise."""
    e = GELU_TC if (a == "gelu" and mode != "fp32") else 0.0
    return (e + 8 * U) * (1.0 + z.abs())


def epilogue(acc, acc_gate, a, mode, bias=None):
    """Forward epilogue of a hidden layer on the float64 product `acc`: z = acc + bias, y = act(z), d = act'(z), each with
    its gate; `kink`: elements whose d the check skips (z within its gate of a jump of act')."""
    z = acc + (bias.double() if bias is not None else 0.0)
    gz = acc_gate + U * z.abs()
    L1, L2 = LIP[a]
    y, d = act(z, a), dact(z, a)
    gy = L1 * gz + act_approx(z, a, mode) + U * y.abs()
    gd = L2 * gz + act_approx(z, a, mode) + U * d.abs()
    kink = (z.abs() <= gz) if a in KINK else torch.zeros_like(z, dtype=torch.bool)
    return dict(z=(z, gz), y=(y, gy), d=(d, gd), kink=kink)


def ratio(got, ref, gate, mask=None, slack=None):
    """max |got - ref| / gate (0 / 0 counts as 0: an exact result where the gate is zero).  `slack`: half-width of the
    interval `got` stands for (a bf16 image holds the fp32 value it was split from to within half an ulp of its last
    plane); the error is the distance from `ref` to that interval."""
    err = (got.double() - ref).abs()
    if slack is not None:
        err = (err - slack).clamp_min(0.0)
    r = torch.where(err == 0, torch.zeros_like(err), err / gate.clamp_min(1e-300))
    if mask is not None:
        r = torch.where(mask, torch.zeros_like(r), r)
    return float(r.max()) if r.numel() else 0.0


def check_split(img, width, planes):
    """The bf16 image planes [planes, M, pitch] (as stored) are a split: hi == bf16_rn(hi + lo), |lo| <= ulp(hi) / 2;
    columns [width, pitch) are +0.  Returns the float64 value hi + lo of the first `width` columns."""
    hi = img[0].double()
    pad = img[:, :, width:]
    assert bool((pad.view(torch.int16) == 0).all()), "image padding is not +0"
    hi = hi[:, :width]
    if planes == 2:
        lo = img[1, :, :width].double()
        assert split_ok(hi, lo), "the planes are not a round-to-nearest split"
        return hi + lo
    return hi


def ulp(hi):
    """bf16 ulp of the (bf16-valued) float64 tensor `hi`."""
    return torch.where(hi == 0, torch.zeros_like(hi), 2.0 ** (torch.floor(torch.log2(hi.abs().clamp_min(1e-38))) - 7))


def split_ok(hi, lo):
    """hi == bf16_rn(hi + lo) and |lo| <= ulp(hi) / 2 (at |lo| == ulp(hi) / 2, a tie, hi + lo may round to hi's even
    neighbour).  Both hold for (hi, lo) = split(x) and fail for a truncating split of about half of all x."""
    half = lo.abs() == ulp(hi) / 2
    return bool(((bf16_rn((hi + lo).float()) == hi) | half).all()) and bool((lo.abs() <= ulp(hi) / 2).all())


# ---- the per-layer cases the GPU tests run and the CPU tests hold to the power rule -----------------------------------
def layer_case(name, M, N, K0, K1=0, kB1=0, variant="fwd", act="gelu", seed=0):
    return dict(name=name, M=M, N=N, K0=K0, K1=K1, kB1=kB1, variant=variant, act=act, seed=seed)


def _layer_cases():
    c = []
    for a in ACTS:
        c.append(layer_case(f"fwd_{a}", 65, 136, 72, act=a, seed=1))
    for n in (1, 3, 45, 129, 192, 256, 300, 520):
        c.append(layer_case(f"fwd_n{n}", 65, n, 40, act="gelu", seed=2))
    for m in (1, 63, 64, 65, 4096):
        c.append(layer_case(f"fwd_m{m}", m, 129, 56, act="tanh", seed=3))
    c.append(layer_case("fwd_seg_11_3", 200, 64, 11, 3, 64, act="relu", seed=4))
    c.append(layer_case("fwd_seg_64_5", 65, 256, 64, 5, 64, act="elu", seed=5))
    c.append(layer_case("fwd_seg_376_17", 130, 256, 376, 17, 384, act="gelu", seed=6))
    for a in ("gelu", "relu", "selu", "sigmoid"):
        c.append(layer_case(f"dgrad_{a}", 200, 192, 256, variant="dgrad", act=a, seed=7))
    for n in (1, 45, 300):
        c.append(layer_case(f"dgrad_n{n}", 65, n, 129, variant="dgrad", act="gelu", seed=8))
    c.append(layer_case("dgrad_m4096", 4096, 64, 256, variant="dgrad", act="tanh", seed=9))
    c.append(layer_case("wgrad_64wide", 64, 256, 300, variant="wgrad", seed=10))
    c.append(layer_case("wgrad_128wide", 1024, 256, 512, variant="wgrad", seed=11))
    c.append(layer_case("wgrad_odd", 45, 17, 65, variant="wgrad", seed=12))
    return {x["name"]: x for x in c}


LAYER_CASES = _layer_cases()


def layer_inputs(case):
    """Seeded fp32 inputs of a case: operands with all-zero rows (their pre-activations equal the bias exactly), biases
    that include 0, +-4 and +-12 (the activation tails and kinks with no matmul error in front of them)."""
    g = torch.Generator().manual_seed(1000 + case["seed"])
    M, N, K0, K1 = case["M"], case["N"], case["K0"], case["K1"]
    r = lambda *s: torch.randn(*s, generator=g)
    v = case["variant"]
    if v == "wgrad":   # C[M, N] += A0[K0, M]^T B[K0, N]
        return dict(A0=r(K0, M), B=r(K0, N), C0=r(M, N))
    A0 = r(M, K0) / math.sqrt(K0 + K1)
    A0[3::7] = 0.0
    A1 = r(M, K1) / math.sqrt(K0 + K1) if K1 else None
    if K1:
        A1[3::7] = 0.0
    out = dict(A0=A0, A1=A1)
    if v == "fwd":
        out["B"] = r(N, K0 + K1)
        b = r(N)
        fixed = torch.tensor([0.0, 4.0, -4.0, 12.0, -12.0])
        b[:min(N, 5)] = fixed[:min(N, 5)]
        out["bias"] = b
    else:
        out["B"] = r(K0, N)
        out["D"] = torch.rand(M, N, generator=g) * 2.0 - 0.25   # act'(z) fed to the tensor-core epilogue
        out["Z"] = r(M, N) * 3.0                                  # z fed to the fp32 one
        out["colsum0"] = r(N)
    return out


FAULTS = ("trunc_split", "drop_hilo", "lost_k16", "lost_col_block", "lost_row_tile", "neighbour_epi", "wrong_act",
          "pad_nonzero")
OTHER_ACT = {"linear": "relu", "relu": "gelu", "gelu": "relu", "tanh": "sigmoid", "sigmoid": "tanh", "elu": "selu",
             "selu": "elu"}


def layer_ref(case, x, mode, fault=None):
    """float64 outputs of one per-layer case and their gates: {name: (value, gate, skip-mask or None)}.
    fwd: C (bias + act), Zout (z in fp32 mode, act'(z) otherwise); dgrad: C (product * act'), colsum (+= column sums);
    wgrad: C (+= product).  `fault` emulates one of FAULTS (None: the correct kernel)."""
    v, a = case["variant"], case["act"]
    M, N, K0, K1 = case["M"], case["N"], case["K0"], case["K1"]
    trunc = fault == "trunc_split"
    drop = fault == "drop_hilo" and mode == "bf16x3"
    if v == "fwd":
        A = torch.cat([x["A0"], x["A1"]], 1) if K1 else x["A0"]
        W = x["B"]
    elif v == "dgrad":
        A, W = x["A0"], x["B"].t()
    else:
        A, W = x["A0"].t(), x["B"].t()
    A, W = A.clone(), W.clone()
    if fault == "lost_k16":   # k16 step 1 of the first k-block (step 0 when K <= 16)
        k = slice(16, 32) if A.shape[1] > 16 else slice(0, 16)
        A[:, k] = 0.0
    val, ab = mm_planes(operands(A, mode, trunc), operands(W, mode, trunc), drop_hilo=drop)
    gate = mm_gate(ab, A.shape[1])
    out = {}
    if v == "fwd":
        bias = x["bias"].double()
        aa = OTHER_ACT[a] if fault == "wrong_act" else a
        if fault == "neighbour_epi" and N > 1:
            bias = torch.cat([bias[1:], bias[-1:]])
        e = epilogue(val, gate, aa, mode, bias)
        e0 = epilogue(val, gate, a, mode, x["bias"])   # gates and kink mask are the correct kernel's
        out["C"] = (e["y"][0], e0["y"][1], None)
        out["Zout"] = (e["z"][0], e0["z"][1], None) if mode == "fp32" else (e["d"][0], e0["d"][1], e0["kink"])
    elif v == "dgrad":
        if mode == "fp32":
            d = dact(x["Z"], a)
            gd = act_approx(x["Z"], a, mode) + U * d.abs()
            kink = (x["Z"].abs() == 0) if a in KINK else None
        else:
            d, gd, kink = x["D"].double(), torch.zeros(M, N, dtype=torch.float64), None
        dd = torch.cat([d[:, 1:], d[:, -1:]], 1) if (fault == "neighbour_epi" and N > 1) else d
        y = val * dd
        gy = gate * d.abs() + val.abs() * gd + U * y.abs()
        out["C"] = (y, gy, kink)
        cs = x["colsum0"].double() + y.sum(0)
        gcs = gy.sum(0) + (M / 64 + 8) * U * (y.abs().sum(0) + x["colsum0"].abs().double())
        out["colsum"] = (cs, gcs, None)
    else:
        y = x["C0"].double() + val
        out["C"] = (y, gate + U * y.abs() * 4, None)
    if fault == "lost_row_tile":   # the last 64-row tile of every output leaves unwritten (zeros)
        for k in ("C", "Zout"):
            if k in out:
                t = out[k][0].clone()
                t[(M - 1) // 64 * 64:] = 0.0
                out[k] = (t,) + out[k][1:]
        if "colsum" in out:
            c, g, _ = out["colsum"]
            out["colsum"] = (c - y[(M - 1) // 64 * 64:].sum(0), g, None)
    if fault == "lost_col_block" and N > 64:   # columns 64..127 not written, as when warpgroup 1 is idle
        for k in ("C", "Zout"):
            if k in out:
                t = out[k][0].clone()
                t[:, 64:128] = 0.0
                out[k] = (t,) + out[k][1:]
    return out


def fault_applies(case, mode, fault):
    v, N = case["variant"], case["N"]
    if fault == "drop_hilo":
        return mode == "bf16x3"
    if fault == "trunc_split":
        return mode != "fp32"
    if fault == "lost_col_block":
        return N > 64
    if fault == "neighbour_epi":
        return v != "wgrad" and N > 1
    if fault == "wrong_act":
        return v == "fwd"
    if fault == "pad_nonzero":
        return mode != "fp32" and v != "wgrad" and N % 8 != 0
    return True


def power(case, x, mode, fault):
    """max over the checked outputs of |faulty - correct| / gate.  Image padding is checked for exact zeros, and image
    planes for the round-to-nearest split bit for bit (split_ok): operands and output images are both formed by
    split_pack2, so a non-zero padding word or a truncating split fails the image checks of every tensor-core forward
    and dgrad case, whatever the value gates see (in bf16x3 a truncating split moves a product by lo*lo-sized terms
    only, a few gates at K >= 300)."""
    if fault == "pad_nonzero" or (fault == "trunc_split" and mode != "fp32"):
        return math.inf
    good, bad = layer_ref(case, x, mode), layer_ref(case, x, mode, fault)
    return max(ratio(bad[k][0], good[k][0], good[k][1], good[k][2]) for k in good)
