"""Dense-layer kernels through the C ABI (`dsact_test_gemm`) against torch fp32."""
import pytest
import torch

pytestmark = pytest.mark.gpu


# per-mode (rtol, atol per sqrt(K)): fp32 FFMA; bf16 split-precision on wgmma (products good to ~2^-16);
# single-pass bf16 on wgmma (operands rounded to 8 bits)
TOL = {"fp32": (2e-5, 2e-5), "bf16x3": (1e-4, 6e-5), "bf16": (3e-2, 2.5e-2)}


@pytest.fixture(scope="module", params=["fp32", "bf16x3", "bf16"])
def eng(request):
    from dsac_v2_b200.engine import Engine, make_config
    lim = torch.ones(2)
    e = Engine(make_config(5, 2, [32, 32], [32, 32], max_batch=16, gemm_mode=request.param), torch.device("cuda", 0), lim, -lim)
    e.mode = request.param
    yield e
    e.close()


SHAPES = [(1, 1, 1), (16, 32, 7), (37, 40, 14), (64, 64, 64), (100, 34, 256), (256, 256, 376), (300, 2, 256),
          (1000, 256, 17), (4096, 256, 256), (129, 257, 31),
          # N or K in 129..192: the three-block (192-column) accumulator of the tensor-core kernels
          (70, 150, 129), (200, 192, 160), (64, 129, 192)]


def _ref(a, b):
    return (a.double() @ b.double()).float()


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_forward_xwT_bias(eng, M, N, K):
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    A = torch.randn(M, K, device="cuda", generator=g)
    W = torch.randn(N, K, device="cuda", generator=g)
    bias = torch.randn(N, device="cuda", generator=g)
    C = torch.full((M, N), float("nan"), device="cuda")
    eng.test_gemm(0, A, W, bias, C, M, N, K)
    ref = _ref(A, W.t()) + bias
    r, a = TOL[eng.mode]
    torch.testing.assert_close(C, ref, rtol=r, atol=a * K ** 0.5)


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_dgrad_dy_w(eng, M, N, K):
    g = torch.Generator(device="cuda").manual_seed(M + N * 5 + K * 11)
    dY = torch.randn(M, K, device="cuda", generator=g)
    W = torch.randn(K, N, device="cuda", generator=g)
    C = torch.full((M, N), float("nan"), device="cuda")
    eng.test_gemm(1, dY, W, None, C, M, N, K)
    r, a = TOL[eng.mode]
    torch.testing.assert_close(C, _ref(dY, W), rtol=r, atol=a * K ** 0.5)


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_wgrad_dyT_x_accumulates(eng, M, N, K):
    g = torch.Generator(device="cuda").manual_seed(M * 13 + N + K * 2)
    dY = torch.randn(K, M, device="cuda", generator=g)  # K = batch (reduction), M = layer outputs
    X = torch.randn(K, N, device="cuda", generator=g)
    C = torch.ones(M, N, device="cuda")               # split-K epilogue accumulates into C
    eng.test_gemm(2, dY, X, None, C, M, N, K)
    r, a = TOL[eng.mode]
    torch.testing.assert_close(C, _ref(dY.t(), X) + 1.0, rtol=r, atol=1.5 * a * K ** 0.5)


def test_strided_operands(eng):
    """Leading dimensions larger than the logical width (column slices of cat(obs, act) weights)."""
    g = torch.Generator(device="cuda").manual_seed(5)
    Wfull = torch.randn(256, 393, device="cuda", generator=g)
    A = torch.randn(77, 17, device="cuda", generator=g)
    C = torch.empty(77, 256, device="cuda")
    r, a = TOL[eng.mode]
    eng.test_gemm(0, A, Wfull[:, 376:], None, C, 77, 256, 17)     # unaligned base + ld 393
    torch.testing.assert_close(C, _ref(A, Wfull[:, 376:].t()), rtol=r, atol=5 * a)
    dZ = torch.randn(77, 256, device="cuda", generator=g)
    D = torch.empty(77, 17, device="cuda")
    eng.test_gemm(1, dZ, Wfull[:, 376:], None, D, 77, 17, 256)
    torch.testing.assert_close(D, _ref(dZ, Wfull[:, 376:]), rtol=r, atol=20 * a)
