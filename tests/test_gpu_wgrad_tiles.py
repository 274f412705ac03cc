"""The tensor-core weight gradient (dsact_test_gemm, variant wgrad) at the batch sizes and widths where its tiles and
batch splits have edges, under several grid bounds.

The persistent kernel walks a static tile list, so a bound on its grid changes which CTA computes a tile and in which
order, but not the sum a tile forms: every split ("slab") must come out as the same bits under every bound.  The hook
reduces the four slabs into C in a fixed order, over slab scratch filled with NaN before the launch, so C shows both
properties: equal bits across bounds, and every slab element written (a batch of fewer than four k-blocks leaves splits
with no k-blocks, which must store zeros).  C must also lie within the float64 gate of tests/tc_ref.py, which rounds the
operands the way the kernel does."""
import pytest
import torch

import tc_ref as R

pytestmark = pytest.mark.gpu

BATCHES = (1, 63, 64, 65, 1000, 4096, 8449)
# (M, N): every width of the list; rows below, at and above one warpgroup's 64 and one CTA's 128, and the critic and
# policy output layers (2 and 34 rows) whose second warpgroup has no rows
SHAPES = ((2, 256), (34, 256), (65, 17), (130, 34), (256, 120), (256, 376))
CAPS = (0, 1, 7, 68)   # 0: one CTA per SM


@pytest.fixture(scope="module", params=["bf16x3", "bf16"])
def tc_eng(request):
    from dsac_v2_b200.engine import Engine, make_config
    lim = torch.ones(2)
    e = Engine(make_config(5, 2, [32, 32], [32, 32], max_batch=16, gemm_mode=request.param), torch.device("cuda", 0),
               lim, -lim)
    e.mode = request.param
    yield e
    e.close()


@pytest.mark.parametrize("B", BATCHES)
def test_slabs_equal_under_every_grid_bound_and_within_the_float64_gate(tc_eng, B):
    cases = [R.layer_case(f"wgrad_{M}x{N}", M, N, B, variant="wgrad", seed=20 + i) for i, (M, N) in enumerate(SHAPES)]
    xs = [R.layer_inputs(c) for c in cases]
    got = {}
    for cap in CAPS:
        outs = [x["C0"].clone().cuda() for x in xs]
        probs = [dict(M=c["M"], N=c["N"], K0=B, A0=x["A0"].cuda(), B=x["B"].cuda(), C=o) for c, x, o in zip(cases, xs, outs)]
        tc_eng.test_layers(2, probs, max_ctas=cap)
        torch.cuda.synchronize()
        got[cap] = [o.cpu() for o in outs]
    for cap in CAPS[1:]:
        for c, a, b in zip(cases, got[CAPS[0]], got[cap]):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (c["name"], cap)
    for c, x, o in zip(cases, xs, got[CAPS[0]]):
        val, gate, mask = R.layer_ref(c, x, tc_eng.mode)["C"]
        assert bool(torch.isfinite(o).all()), f"{c['name']}: a slab element was not written"
        r = R.ratio(o, val, gate, mask)
        assert r <= 1.0, (c["name"], r)
