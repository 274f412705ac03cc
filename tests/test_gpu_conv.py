"""The head-wise engine's convolution kernels one layer at a time (`dsact_cnn_test_conv`: the dispatch the engine itself
runs, `conv_layer_fwd` / `_wgrad` / `_dgrad` of csrc/cnn_engine.cuh), with every kernel variant forced at small sizes and
the engine's own choice on both sides of its thresholds, against float64 `conv2d`, `conv2d_weight` and `conv2d_input`
(the dgrad masked by x > 0 like the ReLU of the layer below).

Forward and dgrad: relative L2 error <= 1e-6.  Weight gradient (a sum over up to millions of rows): within WGRAD_C times
the error of torch's fp32 CPU weight gradient at the same shape, and never above 1e-6 from that rule alone."""
import pytest
import torch
import torch.nn.functional as F

from dsac_v2_b200 import _lib

pytestmark = pytest.mark.gpu

FWD, WGRAD, DGRAD = 0, 1, 2
TOL = 1e-6
WGRAD_C, WGRAD_FLOOR = 8.0, 1e-6
WAVE = 2 * 132 * 128            # conv_fwd8's launch wave on 132 SMs: R = 2 from 2 waves of rows, R = 4 from 4


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm())


def layer(B, cin, h, w, cout, k, s, seed=0):
    """x >= 0 with about half its entries 0 (a ReLU output), weights and bias ~ U(+-1/sqrt(fan_in)), dy ~ N(0, 1)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(B, cin, h, w, generator=g))
    bound = (cin * k * k) ** -0.5
    wt = (torch.rand(cout, cin, k, k, generator=g) * 2 - 1) * bound
    b = (torch.rand(cout, generator=g) * 2 - 1) * bound
    ho, wo = (h - k) // s + 1, (w - k) // s + 1
    dy = torch.randn(B, cout, ho, wo, generator=g)
    return x, wt, b, dy


def run(op, x, wt, b, dy, s, r=0, cob=0, slabs=0, channels=0):
    """(return code, output(s)) of one dsact_cnn_test_conv call on cuda:0."""
    B, cin, h, w = x.shape
    cout, k = wt.shape[0], wt.shape[2]
    xd, wd, bd, dyd = (t.cuda().contiguous() for t in (x, wt, b, dy))
    out = torch.full(x.shape if op == DGRAD else dy.shape, float("nan"), device="cuda")
    dw, db = torch.zeros_like(wd), torch.zeros_like(bd)
    rc = _lib.load().dsact_cnn_test_conv(op, B, cin, h, w, cout, k, s, xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), dyd.data_ptr(),
                                         out.data_ptr(), dw.data_ptr(), db.data_ptr(), r, cob, slabs, channels,
                                         torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, (out, dw, db)


def check(op, x, wt, b, dy, s, **pick):
    rc, (out, dw, db) = run(op, x, wt, b, dy, s, **pick)
    assert rc == 0, _lib.load().dsact_last_error().decode()
    X, Wt, Bb, Dy = (t.double() for t in (x, wt, b, dy))
    if op == FWD:
        e = rel(out, torch.relu(F.conv2d(X, Wt, Bb, stride=s)))
        assert e <= TOL, e
    elif op == DGRAD:
        e = rel(out, torch.nn.grad.conv2d_input(X.shape, Wt, Dy, stride=s) * (X > 0))
        assert e <= TOL, e
    else:
        ref_w = torch.nn.grad.conv2d_weight(X, Wt.shape, Dy, stride=s)
        ref_b = Dy.sum((0, 2, 3))
        f32_w = torch.nn.grad.conv2d_weight(x, wt.shape, dy, stride=s)
        f32_b = dy.sum((0, 2, 3))
        for got, ref, f32 in ((dw, ref_w, f32_w), (db, ref_b, f32_b)):
            e, gate = rel(got, ref), max(WGRAD_C * rel(f32, ref), WGRAD_FLOOR)
            assert e <= gate, (e, gate)


# (B, Cin, H, W, Cout, K, S): every window and stride, S > K (input pixels no window covers get dx = 0), (H - K) % S != 0
# (unused trailing rows and columns), non-square maps, channel counts with and without a factor of 8
SHAPES = [
    (3, 8, 9, 7, 16, 1, 1), (2, 5, 10, 9, 8, 1, 2), (2, 8, 11, 13, 6, 1, 4),
    (2, 8, 12, 11, 16, 2, 1), (3, 6, 13, 10, 8, 2, 3), (2, 16, 14, 9, 12, 2, 2),
    (2, 8, 14, 13, 8, 3, 2), (2, 3, 17, 12, 16, 3, 4), (3, 16, 9, 11, 24, 3, 1), (2, 10, 15, 14, 9, 3, 3),
    (2, 8, 15, 12, 16, 4, 2), (2, 3, 18, 13, 8, 4, 3), (2, 8, 10, 11, 4, 4, 1), (2, 12, 19, 17, 20, 4, 4),
    (2, 8, 21, 19, 8, 8, 4), (2, 3, 20, 17, 16, 8, 3), (2, 4, 17, 18, 5, 8, 2), (1, 8, 16, 12, 8, 8, 1),
]


def ids(p):
    return "B{}_c{}_{}x{}_o{}_k{}_s{}".format(*p)


@pytest.mark.parametrize("shape", SHAPES, ids=ids)
@pytest.mark.parametrize("op", [FWD, WGRAD, DGRAD], ids=["fwd", "wgrad", "dgrad"])
def test_engine_choice_matches_float64(shape, op):
    B, cin, h, w, cout, k, s = shape
    check(op, *layer(B, cin, h, w, cout, k, s), s)


@pytest.mark.parametrize("shape", SHAPES, ids=ids)
def test_every_variant_matches_float64(shape):
    """Each forward R and channel count, each dgrad channel count, each COB and slab count the kernels have for this shape;
    combinations without a kernel return DSACT_EINVAL and write nothing."""
    B, cin, h, w, cout, k, s = shape
    t = layer(B, cin, h, w, cout, k, s)
    for r in (1, 2, 4):
        ok = cout % 8 == 0 and (k != 8 or r == 1)
        rc = run(FWD, *t, s, r=r, channels=8)[0]
        assert (rc == 0) == ok, (r, rc)
        if ok:
            check(FWD, *t, s, r=r, channels=8)
    check(FWD, *t, s, channels=1)
    if cin % 8 == 0:
        check(DGRAD, *t, s, channels=8)
    else:
        assert run(DGRAD, *t, s, channels=8)[0] == -1
    check(DGRAD, *t, s, channels=1)
    for cob in (1, 4, 8):
        ok = cout % cob == 0 and not (k == 4 and cob == 8) and not (k == 8 and cob != 1)
        for slabs in (1, 9, 88):
            rc, (_, dw, _) = run(WGRAD, *t, s, cob=cob, slabs=slabs)
            assert (rc == 0) == ok, (cob, slabs, rc)
            if ok:
                check(WGRAD, *t, s, cob=cob, slabs=slabs)
            else:
                assert not dw.any()


def test_forward_and_dgrad_fall_back_at_the_shared_memory_limits():
    """Cin*K*K*32 B just above 48 KiB: the forward takes one channel per thread; Cout*K*K*32 B just above 96 KiB: so does
    the dgrad.  Just below, the eight-channel kernels run; above, forcing them is an error."""
    for cin, fits in ((170, True), (171, False)):          # 170 * 9 * 32 B = 47.8 KiB, 171 * 9 * 32 B = 48.1 KiB
        t = layer(2, cin, 7, 6, 8, 3, 1)
        check(FWD, *t, 1)
        assert (run(FWD, *t, 1, channels=8)[0] == 0) == fits
    for cout, fits in ((192, True), (193, False)):         # 192 * 16 * 32 B = 96 KiB, 193 * 16 * 32 B = 96.5 KiB
        t = layer(2, 8, 9, 8, cout, 4, 1)
        check(DGRAD, *t, 1)
        assert (run(DGRAD, *t, 1, channels=8)[0] == 0) == fits


@pytest.mark.parametrize("rows", [2 * WAVE - 3, 2 * WAVE + 39, 4 * WAVE - 3, 4 * WAVE + 39])
def test_forward_positions_per_thread_around_the_engine_thresholds(rows):
    """Row counts on both sides of the R = 2 and R = 4 thresholds and no multiple of 128 * R (1 x 1 windows on 3 x 1 maps:
    rows = 3 B)."""
    assert rows % 3 == 0
    t = layer(rows // 3, 8, 3, 1, 8, 1, 1, seed=1)
    check(FWD, *t, 1)
    for r in (1, 2, 4):
        check(FWD, *t, 1, r=r, channels=8)


def test_weight_gradient_slabs_beyond_the_engine_choice():
    """Slab counts of 1, 9, 88 and 131 over a row count that no slab size divides."""
    t = layer(37, 8, 29, 23, 16, 3, 2, seed=2)
    for slabs in (1, 9, 88, 131):
        for cob in (4, 8):
            check(WGRAD, *t, 2, cob=cob, slabs=slabs)


ENCODERS = {   # (Cin, H, W) of each layer's input at 3 x 96 x 96 images; (Cout, K, S)
    "type_2": [(3, 96, 96, 8, 4, 2), (8, 47, 47, 16, 3, 2), (16, 23, 23, 32, 3, 2), (32, 11, 11, 64, 3, 2),
               (64, 5, 5, 128, 3, 1), (128, 3, 3, 256, 3, 1)],
    "type_1": [(3, 96, 96, 32, 8, 4), (32, 23, 23, 64, 4, 2), (64, 10, 10, 64, 3, 1)],
}


@pytest.mark.parametrize("enc,j", [(e, j) for e, ls in ENCODERS.items() for j in range(len(ls))])
def test_encoder_layers_at_batch_1024(enc, j):
    """The layer shapes of the reference's encoders at the CNN benchmark's batch, in the engine's own choice of kernels
    (type_2's first layer: R = 4 forward, 88 weight-gradient slabs on 132 SMs; its last: the GEMM of a linear layer)."""
    cin, h, w, cout, k, s = ENCODERS[enc][j]
    t = layer(1024, cin, h, w, cout, k, s, seed=3 + j)
    for op in (FWD, WGRAD) + ((DGRAD,) if j > 0 else ()):
        check(op, *t, s)
