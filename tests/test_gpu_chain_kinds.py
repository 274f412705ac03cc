"""The ping-pong kernel's epilogue kinds (straight-line bodies for the full tiles of forward GELU / ReLU hidden layers with
and without act' stores, and of dgrad hidden layers with and without column sums) against the column split, which runs
the runtime epilogue everywhere: the same bits in the outputs, act' and images, the column sums up to the order of their
float atomics, and nothing written outside the NaN-poisoned outputs.  The passes mix full tiles with a ragged last tile
and a CTA whose second tile is missing, and the widths take every layer body (64, 128, 192 and 256 columns)."""
import pytest
import torch

from test_gpu_chain_pingpong import GUARD, _bits, _build
from test_gpu_layer_kernels import ACT, tc_eng  # noqa: F401  (tc_eng: the fixture)

HIDDEN = [256, 192, 128, 64]
MS = [4096, 8449, 100]


def _run(tc_eng, dgrad, act, drop):
    """Both kernels on the same inputs, without the per-layer outputs named in `drop` (Zout or colsum)."""
    case = (dgrad, HIDDEN, 120, 0, 0, 34)
    res = []
    for tiling in (0, 1):
        sizes, params, passes, bufs = _build(case, MS, 11)
        for p in passes:
            if drop:
                p[drop] = None
        tc_eng.test_chain(dgrad, sizes, case[2], 0, 0, ACT[act], params, passes, tiling=tiling)
        torch.cuda.synchronize()
        res.append(bufs)
    for i, ((exact0, sums0), (exact1, sums1)) in enumerate(zip(*res)):
        for k, (a, b) in enumerate(zip(exact0, exact1)):
            a, b = a.cpu(), b.cpu()
            assert torch.equal(_bits(a), _bits(b)), f"pass {i} (M = {MS[i]}) output {k}: bits differ"
            assert bool(b[:GUARD].isnan().all()) and bool(b[-GUARD:].isnan().all()), f"pass {i} output {k}: written outside"
        if drop == "colsum":
            continue
        for k, (a, b) in enumerate(zip(sums0, sums1)):
            a, b = a.cpu().double(), b.cpu().double()
            assert bool(b[:GUARD].isnan().all()) and bool(b[-GUARD:].isnan().all()), f"pass {i} colsum {k}: written outside"
            a, b = a[GUARD:-GUARD], b[GUARD:-GUARD]
            img = exact0[k][GUARD:-GUARD].view(2, MS[i], -1)[:, :, :HIDDEN[k]].cpu().double()
            mag = (img[0] + (img[1] if tc_eng.mode == "bf16x3" else 0)).abs().sum(0) + a.abs()
            tol = (MS[i] / 16 + 16) * 2.0 ** -23 * mag
            assert bool(((a - b).abs() <= tol).all()), f"pass {i} colsum {k}: {(a - b).abs().max().item()}"


@pytest.mark.gpu
@pytest.mark.parametrize("zout", [True, False])
@pytest.mark.parametrize("act", ["gelu", "relu"])
def test_forward_kinds_give_the_column_split_bits(tc_eng, act, zout):
    _run(tc_eng, False, act, None if zout else "Zout")


@pytest.mark.gpu
@pytest.mark.parametrize("colsum", [True, False])
@pytest.mark.parametrize("act", ["gelu", "relu"])
def test_dgrad_kinds_give_the_column_split_bits(tc_eng, act, colsum):
    _run(tc_eng, True, act, None if colsum else "colsum")
