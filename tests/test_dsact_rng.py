"""The host restatement of the device generator (oracle/dsact_rng.py): Random123's known-answer vectors, the replay-index
draw and the noise layout, and the statistics a correct generator must show.  CPU only; every seed is fixed."""
import numpy as np
import pytest
from scipy import stats

from oracle.dsact_rng import box_muller, device_noise, philox4x32_10, replay_indices, u01

SIZES = [1, 2, 3, 7, 1000, 10 ** 6, 2 ** 32 + 15]
N_ROWS = 200_000


def test_philox_known_answers():
    """Random123's published philox4x32-10 vectors (kat_vectors): zero counter and key, all-ones counter and key."""
    assert [int(v) for v in philox4x32_10((0, 0, 0, 0), (0, 0))] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    m = 0xFFFFFFFF
    assert [int(v) for v in philox4x32_10((m, m, m, m), (m, m))] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]


def test_philox_vectorised_equals_scalar():
    ctr = np.arange(5, dtype=np.uint64) * 0x10001 + 7
    vec = philox4x32_10((ctr, 3, 0x49445853, 0), (11, 12))
    for i, c in enumerate(ctr):
        one = philox4x32_10((int(c), 3, 0x49445853, 0), (11, 12))
        assert [int(v[i]) for v in vec] == [int(v) for v in one]


def test_u01_is_the_kernels_float32_map():
    assert u01(0).dtype == np.float32
    assert float(u01(0)) == 2.0 ** -33                  # never 0: log stays finite
    assert float(u01(0xFFFFFFFF)) == 1.0                # 2^32 - 1 rounds to 2^32 in float32
    assert float(u01(1 << 24 | 1)) == float((np.float32(1 << 24) + np.float32(0.5)) * np.float32(2.0 ** -32))
    n0, n1 = box_muller(np.uint32(0), np.uint32(0))     # the largest radius the generator can produce
    assert abs(float(n0)) == pytest.approx(np.sqrt(66 * np.log(2.0)))
    assert float(n1) == pytest.approx(np.sqrt(66 * np.log(2.0)) * np.sin(2 * np.pi * 2.0 ** -33))


def test_replay_index_words_and_product():
    """Row r: block r >> 1, (x, y) for even rows and (z, w) for odd rows, high half of the 128-bit product with size."""
    seed, ctr, size = 0x123456789ABCDEF, 41, 2 ** 32 + 15
    got = replay_indices(seed, ctr, 6, size)
    for r in range(6):
        x, y, z, w = (int(v) for v in philox4x32_10((r >> 1, ctr, 0x49445853, 0), (seed & 0xFFFFFFFF, seed >> 32)))
        a = (z << 32 | w) if r & 1 else (x << 32 | y)
        assert int(got[r]) == (a * size) >> 64


@pytest.mark.parametrize("size", SIZES)
def test_replay_indices_in_range_and_uniform(size):
    idx = replay_indices(2024, 5, N_ROWS, size)
    assert idx.dtype == np.int64 and idx.min() >= 0 and idx.max() < size
    if size == 1:
        assert not idx.any()
        return
    k = min(size, 1000)
    bins = idx * k // size if size > k else idx
    counts = np.bincount(bins, minlength=k)
    assert stats.chisquare(counts).pvalue > 1e-4, (size, counts[:16])
    # rows 2i and 2i+1 share one Philox block: their joint table must be uniform as well
    j = min(size, 16)
    pb = idx * j // size if size > j else idx
    table = np.bincount(pb[0::2] * j + pb[1::2], minlength=j * j)
    assert stats.chisquare(table).pvalue > 1e-4, (size, table.reshape(j, j))


@pytest.mark.parametrize("size", SIZES[1:])
def test_replay_indices_of_consecutive_counters_are_independent(size):
    """A reused counter would repeat the previous call's rows: positional matches must stay at the 1/size rate."""
    a, b = replay_indices(77, 9, N_ROWS, size), replay_indices(77, 10, N_ROWS, size)
    same = int((a == b).sum())
    expect = N_ROWS / size
    assert same <= expect + 6 * np.sqrt(expect) + 1, (size, same, expect)
    # and a different seed at the same counter is another stream
    c = replay_indices(78, 9, N_ROWS, size)
    assert int((a == c).sum()) <= expect + 6 * np.sqrt(expect) + 1


# odd B and odd B*A: the last pair of eps1, eps2, z3 and z4 each drops its second value
NB, NA = 200_001, 5


@pytest.fixture(scope="module")
def noise():
    return device_noise(31337, 4, NB, NA)


def test_noise_shapes_and_range(noise):
    eps1, eps2, z3, z4 = noise
    assert eps1.shape == (NB, NA) and eps2.shape == (NB, NA) and z3.shape == (NB,) and z4.shape == (NB,)
    for x in noise:
        assert np.all(np.isfinite(x))
        assert np.abs(x).max() <= 6.8


def test_noise_is_standard_normal(noise):
    for name, x in zip(("eps1", "eps2", "z3", "z4"), noise):
        p = stats.kstest(x.reshape(-1), "norm").pvalue
        assert p > 1e-4, (name, p)


def test_noise_streams_are_uncorrelated(noise):
    eps1, eps2, z3, z4 = (x.reshape(-1) for x in noise)
    n = eps1.size
    assert abs(np.corrcoef(eps1, eps2)[0, 1]) < 5 / np.sqrt(n)
    assert abs(np.corrcoef(z3, z4)[0, 1]) < 5 / np.sqrt(z3.size)
    nxt = device_noise(31337, 5, NB, NA)          # the next counter
    oth = device_noise(31338, 4, NB, NA)          # the next seed
    for a, b, m in zip(noise, nxt, ("eps1", "eps2", "z3", "z4")):
        a, b = a.reshape(-1), b.reshape(-1)
        assert abs(np.corrcoef(a, b)[0, 1]) < 5 / np.sqrt(a.size), ("counter", m)
    for a, b, m in zip(noise, oth, ("eps1", "eps2", "z3", "z4")):
        a, b = a.reshape(-1), b.reshape(-1)
        assert abs(np.corrcoef(a, b)[0, 1]) < 5 / np.sqrt(a.size), ("seed", m)


@pytest.mark.parametrize("B,A", [(1, 1), (3, 3), (4, 3), (5, 2), (37, 6)])
def test_noise_pair_layout(B, A):
    """Every tensor starts on a pair of its own: with n = ceil(B*A/2) pairs per eps tensor, eps2 starts at value 2n of the
    normal stream, z3 at 4n and z4 at 4n + 2 ceil(B/2); no value appears in two tensors."""
    eps1, eps2, z3, z4 = device_noise(5, 0, B, A)
    n_ea, n_z = (B * A + 1) // 2, (B + 1) // 2
    m = 4 * n_ea + 4 * n_z
    big = device_noise(5, 0, m, 1)[0].reshape(-1)   # B = m (even), A = 1: eps1 is the first m values of the stream
    assert np.array_equal(eps1.reshape(-1), big[:B * A])
    assert np.array_equal(eps2.reshape(-1), big[2 * n_ea:2 * n_ea + B * A])
    assert np.array_equal(z3, big[4 * n_ea:4 * n_ea + B])
    assert np.array_equal(z4, big[4 * n_ea + 2 * n_z:4 * n_ea + 2 * n_z + B])
    vals = np.concatenate([eps1.reshape(-1), eps2.reshape(-1), z3, z4])
    assert np.unique(vals).size == vals.size
