"""The layer chain stores a hidden layer's bf16 image as TMA stores of its operand buffer.  Into NaN-poisoned buffers, the
images of forward and dgrad chains at ragged batch sizes hold the values the float64 reference checks accept, with zero
padding, and nothing outside rows < M, columns < (N + 7) / 8 * 8 and the mode's planes is written."""
import pytest
import torch

import tc_ref as R
from test_gpu_layer_kernels import (ACT, NAN, _chain_setup, _check_fwd_chain, _fwd_pass, _img_value, _report, chain_case,
                                    tc_eng)  # noqa: F401  (tc_eng: the fixture)

pytestmark = pytest.mark.gpu

HIDDEN = [64, 72, 200, 256]
MS = [1, 63, 65, 4097, 8449]
GUARD = 64   # poisoned elements before an image; 64 poisoned rows follow it


def _poisoned(M, N):
    """A NaN buffer and the [2, M, pitch] image inside it (the layout dsact_test_chain gives an image)."""
    pitch = (N + 7) // 8 * 8
    buf = torch.full((GUARD + (2 * M + 64) * pitch,), NAN, dtype=torch.bfloat16, device="cuda")
    return buf, buf[GUARD:GUARD + 2 * M * pitch].view(2, M, pitch)


def _check_untouched(bufs, mode):
    for buf, img in bufs:
        M, pitch = img.shape[1], img.shape[2]
        b = buf.cpu()
        assert bool(b[:GUARD].isnan().all()), "written before the image"
        assert bool(b[GUARD + 2 * M * pitch:].isnan().all()), "written past row M of the last plane"
        if mode == "bf16":
            assert bool(img[1].cpu().isnan().all()), "the lo plane written in bf16 mode"


@pytest.mark.parametrize("M", MS)
def test_forward_chain_images(tc_eng, M):
    case = chain_case("img_fwd", HIDDEN, 11, 2, M, "gelu", K1=3, kB1=64)
    sizes, parts, params, g = _chain_setup(case, 17)
    x, p = _fwd_pass(case, sizes, g, M)
    bufs = [_poisoned(M, w) for w in HIDDEN]
    p["img"] = [img for _, img in bufs]
    tc_eng.test_chain(False, sizes, case["K0"], case["K1"], case["kB1"], ACT[case["act"]], params, [p])
    torch.cuda.synchronize()
    _check_untouched(bufs, tc_eng.mode)
    _report(tc_eng.mode, f"chain_img_fwd.M{M}", _check_fwd_chain(tc_eng.mode, case, sizes, parts, x, p))


@pytest.mark.parametrize("M", MS)
def test_dgrad_chain_images(tc_eng, M):
    """Without action columns the last layer (dz_0) has no next layer in the chain; its image is staged all the same."""
    mode = tc_eng.mode
    case = chain_case("img_dgrad", HIDDEN, 14, 2, M, "tanh")
    sizes, parts, params, g = _chain_setup(case, 19)
    L = len(HIDDEN)
    dout = torch.randn(M, sizes[-1], generator=g)
    D = [torch.rand(M, w, generator=g) * 2.0 - 0.25 for w in HIDDEN]
    bufs = [_poisoned(M, w) for w in HIDDEN]
    p = dict(M=M, x0=dout.cuda(), Zin=[d.cuda() for d in D], img=[img for _, img in bufs])
    tc_eng.test_chain(True, sizes, case["K0"], 0, 0, ACT[case["act"]], params, [p])
    torch.cuda.synchronize()
    _check_untouched(bufs, mode)
    ratios = {}
    planes = R.operands(dout, mode)
    for j in range(L, 0, -1):
        acc, ab = R.mm_planes(planes, R.operands(parts[2 * j].t().contiguous(), mode))
        d = D[j - 1].double()
        y = acc * d
        v, half = _img_value(p["img"][j - 1], sizes[j], mode)
        ratios[f"dz{j - 1}"] = R.ratio(v, y, R.mm_gate(ab, sizes[j + 1]) * d.abs() + R.U * y.abs(), slack=half)
        im = p["img"][j - 1].cpu()
        planes = [im[0].double(), im[1].double()] if mode == "bf16x3" else [im[0].double()]
    _report(mode, f"chain_img_dgrad.M{M}", ratios)
