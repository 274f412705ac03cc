"""The ping-pong layer-chain kernel (two 64-row tiles per CTA, one per MMA warpgroup) against the column split (one tile per
CTA, each warpgroup with half of a layer's columns): the same chain group through both kernels must give the same bits in
the outputs, act' and images, and the column sums up to the order of their float atomics.  Every output lies inside a
NaN-poisoned buffer, so an element either kernel writes outside it shows up.  The step selects the ping-pong kernel by
launch shape; dsact_test_chain_tiling runs a chosen kernel on any shape.

Also the SASS of the ping-pong kernel (no GPU needed): stmatrix and TMA stores, no wgmma serialisation, no spills."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

from dsac_v2_b200 import _lib
from test_gpu_layer_kernels import ACT, NAN, _chain_setup, tc_eng  # noqa: F401  (tc_eng: the fixture)

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(REPO, "dsac-v2_b200", "libdsact.so")
GUARD = 64   # poisoned elements on each side of every output

# name: dgrad, hidden widths, K0, K1, kB1, head.  The widths take every layer body: 64 (one 64-column block), 128 (two),
# 136 (three: a 64-column second half), 200 / 256 (four), and 8 (a 16-column tile).
CASES = {
    "fwd_wide": (False, [256, 256, 256], 376, 17, 384, 2),
    "fwd_mixed": (False, [64, 136, 200, 128], 11, 3, 64, 34),
    "fwd_head192": (False, [128], 64, 0, 0, 192),
    "dgrad_wide": (True, [256, 256, 256], 376, 17, 384, 2),
    "dgrad_mixed": (True, [64, 136, 200, 128], 14, 0, 0, 2),
    "dgrad_narrow": (True, [8, 72, 256, 248], 5, 0, 0, 34),
    # five and six hidden layers; the six-layer chain's ring items per tile mix odd and even counts (forward: 1, 2, 3, 2,
    # 4, 4, then 3 for the head), so the warpgroups' turns and the ring's parity waits go through many phases
    "fwd_deep5": (False, [256, 64, 128, 200, 136], 14, 3, 16, 2),
    "fwd_parity6": (False, [64, 192, 8, 256, 72, 136], 5, 0, 0, 2),
    "dgrad_deep5": (True, [256, 64, 128, 200, 136], 14, 3, 16, 2),
    "dgrad_parity6": (True, [64, 192, 8, 256, 72, 136], 5, 0, 0, 2),
}
# the rows of each pass of one launch: one tile, a full and a partial CTA, a CTA whose second tile is missing (129, 8449)
PASS_SETS = {
    "p1_m1": [1],
    "p2": [63, 8449],
    "p3": [65, 4097, 129],
    "p4": [64, 127, 2, 8449],
}


def _guarded(shape, dtype=torch.float32):
    """A NaN buffer with GUARD poisoned elements on each side, and the output view inside it."""
    n = 1
    for s in shape:
        n *= s
    buf = torch.full((n + 2 * GUARD,), NAN, dtype=dtype, device="cuda")
    return buf, buf[GUARD:GUARD + n].view(*shape)


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _build(case, Ms, seed):
    """Inputs and poisoned outputs of every pass, as dicts for test_chain (built twice from the same seed)."""
    dgrad, hidden, K0, K1, kB1, head = case
    sizes, parts, params, g = _chain_setup(dict(K0=K0, K1=K1, kB1=kB1, hidden=hidden, head=head), seed)
    passes, bufs = [], []
    for M in Ms:
        img = [_guarded((2, M, (w + 7) // 8 * 8), torch.bfloat16) for w in hidden]
        p = dict(M=M, img=[v for _, v in img])
        if dgrad:
            dout = torch.randn(M, head, generator=g)
            dout[3::7] = 0.0
            p["x0"] = dout.cuda()
            p["Zin"] = [(torch.rand(M, w, generator=g) * 2.0 - 0.25).cuda() for w in hidden]
            cs = [_guarded((w,)) for w in hidden]
            for (_, v), w in zip(cs, hidden):
                v.copy_(torch.randn(w, generator=g))
            p["colsum"] = [v for _, v in cs]
            outs = [b for b, _ in img]
            if K1:
                o = _guarded((M, K1))
                p["out"] = o[1]
                outs.append(o[0])
            bufs.append((outs, [b for b, _ in cs]))
        else:
            x = torch.randn(M, K0 + K1, generator=g)
            x[3::7] = 0.0
            p["x0"] = x[:, :K0].contiguous().cuda()
            if K1:
                p["x1"] = x[:, K0:].contiguous().cuda()
            o = _guarded((M, head))
            z = [_guarded((M, w)) for w in hidden]
            p["out"] = o[1]
            p["Zout"] = [v for _, v in z]
            bufs.append(([b for b, _ in img] + [o[0]] + [b for b, _ in z], []))
        passes.append(p)
    return sizes, params, passes, bufs


@pytest.mark.gpu
@pytest.mark.parametrize("act", list(ACT))
@pytest.mark.parametrize("pset", list(PASS_SETS))
@pytest.mark.parametrize("name", list(CASES))
def test_pingpong_gives_the_column_split_bits(tc_eng, name, pset, act):
    case = CASES[name]
    dgrad, hidden, K0, K1, kB1 = case[:5]
    Ms = PASS_SETS[pset]
    res = []
    for tiling in (0, 1):
        sizes, params, passes, bufs = _build(case, Ms, 23)
        tc_eng.test_chain(dgrad, sizes, K0, K1, kB1, ACT[act], params, passes, tiling=tiling)
        torch.cuda.synchronize()
        res.append(bufs)
    for i, ((exact0, sums0), (exact1, sums1)) in enumerate(zip(*res)):
        M = Ms[i]
        for k, (a, b) in enumerate(zip(exact0, exact1)):
            a, b = a.cpu(), b.cpu()
            assert torch.equal(_bits(a), _bits(b)), f"pass {i} (M = {M}) output {k}: bits differ"
            assert bool(a[:GUARD].isnan().all()) and bool(a[-GUARD:].isnan().all()), f"pass {i} output {k}: written outside"
            assert bool(b[:GUARD].isnan().all()) and bool(b[-GUARD:].isnan().all()), f"pass {i} output {k}: written outside"
        for k, (a, b) in enumerate(zip(sums0, sums1)):
            a, b = a.cpu().double(), b.cpu().double()
            assert bool(b[:GUARD].isnan().all()) and bool(b[-GUARD:].isnan().all()), f"pass {i} colsum {k}: written outside"
            a, b = a[GUARD:-GUARD], b[GUARD:-GUARD]
            # the same partial sums added in another order: a few ulps of the sum of magnitudes
            img = exact0[k][GUARD:-GUARD].view(2, M, -1)[:, :, :hidden[k]].cpu().double()
            mag = (img[0] + (img[1] if tc_eng.mode == "bf16x3" else 0)).abs().sum(0) + a.abs()
            tol = (M / 16 + 16) * 2.0 ** -23 * mag
            assert bool(((a - b).abs() <= tol).all()), f"pass {i} colsum {k}: {(a - b).abs().max().item()}"


@pytest.mark.gpu
def test_step_shapes_select_by_wave(tc_eng):
    """By shape, a launch that fits one wave runs the column split and one that does not runs the ping-pong kernel; both
    are the same bits as the forced kernels."""
    case = CASES["fwd_wide"]
    K0, K1, kB1 = case[2:5]
    for Ms in ([64] * 4, [4096] * 4):
        res = []
        for tiling in (None, 0, 1):
            sizes, params, passes, bufs = _build(case, Ms, 5)
            tc_eng.test_chain(False, sizes, K0, K1, kB1, ACT["gelu"], params, passes, tiling=tiling)
            torch.cuda.synchronize()
            res.append([b.cpu() for outs, _ in bufs for b in outs])
        for a, b, c in zip(*res):
            assert torch.equal(_bits(a), _bits(b)) and torch.equal(_bits(a), _bits(c))


def test_tiling_hook_refuses_an_unknown_kernel():
    lib = _lib.load()
    sizes = (C.c_int32 * 3)(4, 8, 2)
    assert lib.dsact_test_chain_tiling(None, 2, 0, 1, sizes, 4, 0, 0, 2, None, None, 1, None) == -1   # DSACT_EINVAL
    assert b"tiling" in lib.dsact_last_error()


# ---- SASS -------------------------------------------------------------------------------------------------------------
def _cuobjdump():
    for d in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if d and os.path.exists(os.path.join(d, "bin", "cuobjdump")):
            return os.path.join(d, "bin", "cuobjdump")
    return shutil.which("cuobjdump")


@pytest.fixture(scope="module")
def pp_sass():
    tool = _cuobjdump()
    if not os.path.exists(LIB) or tool is None:
        pytest.skip("needs the built libdsact.so and the CUDA toolkit's cuobjdump")
    text = subprocess.run([tool, "-sass", LIB], check=True, capture_output=True, text=True).stdout
    funcs = {}
    for chunk in re.split(r"\n\s*Function : ", text)[1:]:
        name, body = chunk.split("\n", 1)
        if "tc_pingpong_kernel" in name:
            funcs[name.strip()] = [m.group(1).strip() for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)]
    assert len(funcs) == 4, sorted(funcs)   # 2 plane counts x 2 B orientations
    return funcs


def _count(ins, op):
    return sum(1 for s in ins if re.search(r"(^|\s)" + op + r"(\.|\s|$)", s))


def test_pingpong_stores_by_stmatrix_and_tma(pp_sass):
    for name, ins in pp_sass.items():
        assert _count(ins, "STSM") > 0, f"{name}: no STSM"
        assert _count(ins, "UTMASTG") > 0, f"{name}: no UTMASTG"


def test_pingpong_keeps_wgmma_in_flight(pp_sass):
    # as tests/test_sass.py: a full wait between two HGMMAs only where a new ring item begins (after its mbarrier wait)
    for name, ins in pp_sass.items():
        hg = [i for i, s in enumerate(ins) if s.startswith("HGMMA") or " HGMMA" in s]
        assert hg, f"{name}: no HGMMA"
        bad = 0
        for a, b in zip(hg, hg[1:]):
            between = ins[a + 1:b]
            if any("DEPBAR.LE gsb0, 0x0" in s for s in between) and not any("SYNCS.PHASECHK" in s for s in between):
                bad += 1
        assert bad == 0, f"{name}: {bad} of {len(hg)} HGMMAs wait for all MMAs before the next one issues"
        assert any("DEPBAR.LE gsb0, 0x1" in s for s in ins), f"{name}: no wgmma.wait_group 1"


def test_pingpong_has_no_local_memory(pp_sass):
    for name, ins in pp_sass.items():
        assert _count(ins, "STL") == 0 and _count(ins, "LDL") == 0, f"{name}: local memory (spills)"
