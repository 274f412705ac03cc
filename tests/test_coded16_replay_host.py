"""The 16-bit coded frame ring's host side, without a GPU: the 16-bit coder (dsac_v2_b200/frame_plan.py
FrameCoder(16)) against a dictionary coder, on signed zeros and NaN payloads, its refusal of a 65 537th value and its
state round trip; the drop-in kwarg, refusals and checkpoint kinds; a synthetic stacked-grey CarRacing source that the
8-bit ring refuses and the 16-bit ring takes; and the C entry points' declarations and refusals."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from dsac_v2_b200 import _lib
from dsac_v2_b200.frame_plan import FrameCoder

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def stacked_grey(g, palette, n, shape=(96, 96)):
    """n grey frames of `gym_carracing` made from a palette of RGB colours: the reference's rgb2gray,
    dot(rgb, [0.299, 0.587, 0.114]) / 128 - 1 (float64), stored as float32 by the replay buffer."""
    rgb = palette[g.integers(0, len(palette), (n,) + shape)]
    return np.asarray(np.dot(rgb, [0.299, 0.587, 0.114]) / 128.0 - 1.0, dtype=np.float32)


def palette(g, colours):
    return g.integers(0, 256, (colours, 3)).astype(np.uint8)


def test_the_default_coder_is_the_8_bit_coder():
    c = FrameCoder()
    assert c.code_bits == 8 and c.N == 256 and c.bits.shape == (256,) and c.bits.dtype == np.uint32
    codes, _ = c.encode(np.float32([0.5, 0.25, 0.5]))
    assert codes.dtype == np.uint8 and codes.tolist() == [0, 1, 0]
    w = FrameCoder(16)
    assert w.N == 65536 and w.bits.shape == (65536,) and w.table.dtype == np.float32
    for bad in (0, 12, 32):
        with pytest.raises(ValueError, match="8- or 16-bit"):
            FrameCoder(bad)


@pytest.mark.parametrize("seed", range(3))
def test_codes_equal_a_dictionary_coder_on_random_bit_patterns(seed):
    # up to all 65 536 codes, in batches that bring few or many new patterns
    g = np.random.default_rng(seed)
    pats = np.unique(g.integers(0, 2 ** 32, 70000, dtype=np.uint64).astype(np.uint32))[:65536]
    g.shuffle(pats)
    coder, ref = FrameCoder(16), {}
    for step in range(50):
        hi = len(pats) if step == 49 else min(len(pats), 16 + 2 * len(ref) + int(g.integers(0, 4000)))
        x = pats[g.integers(0, hi, int(g.integers(1, 12000)))]
        if step == 49:
            x = np.concatenate([x, pats])   # every pattern: the table fills
        codes, new = coder.encode(x.view(np.float32))
        coder.commit(new)
        want = [ref.setdefault(int(v), len(ref)) for v in x]
        assert codes.dtype == np.uint16 and codes.tolist() == want
        assert coder.n == len(ref)
    assert coder.n == 65536
    assert np.array_equal(coder.bits, np.array(sorted(ref, key=ref.get), np.uint32))
    np.testing.assert_array_equal(coder.table[coder.encode(pats.view(np.float32))[0]].view(np.uint32), pats)


def test_codes_follow_first_appearance_and_bit_patterns():
    nan_a = np.array([0x7FC00001], np.uint32).view(np.float32)[0]
    nan_b = np.array([0xFFC00002], np.uint32).view(np.float32)[0]
    v = np.array([0.5, -0.0, 0.0, 0.5, nan_a, nan_b, -0.0, nan_a], np.float32)
    coder = FrameCoder(16)
    codes, new = coder.encode(v.reshape(2, 4))
    assert coder.n == 0, "encode changed the table"
    coder.commit(new)
    assert codes.shape == (2, 4) and codes.reshape(-1).tolist() == [0, 1, 2, 0, 3, 4, 1, 3]
    np.testing.assert_array_equal(coder.table[codes].view(np.uint32).reshape(-1), v.view(np.uint32))
    codes, new = coder.encode(np.array([0.0, 0.25, nan_b, -1.0, 0.25], np.float32))
    coder.commit(new)
    assert codes.tolist() == [2, 5, 4, 6, 5] and coder.n == 7


def test_the_65537th_value_is_refused_and_nothing_changes():
    coder = FrameCoder(16)
    _, new = coder.encode(np.arange(65536, dtype=np.float32))
    coder.commit(new)
    bits = coder.bits.copy()
    with pytest.raises(ValueError, match="65536"):
        coder.encode(np.array([3.0, 1e6 + 0.5, 2.0], np.float32))
    assert coder.n == 65536 and np.array_equal(coder.bits, bits)
    with pytest.raises(ValueError, match="1000000.5"):   # the message names the value
        coder.encode(np.array([1e6 + 0.5], np.float32))
    codes, new = coder.encode(np.array([65535.0, 0.0], np.float32))   # and still codes what it holds
    assert codes.tolist() == [65535, 0] and len(new) == 0


def test_coder_state_round_trips_and_keeps_its_width():
    g = np.random.default_rng(1)
    pal = palette(g, 3000)
    a = FrameCoder(16)
    _, new = a.encode(stacked_grey(g, pal, 2))
    a.commit(new)
    assert 256 < a.n <= 3000
    b = FrameCoder(16)
    b.load_state_dict(a.state_dict())
    assert b.n == a.n and np.array_equal(a.bits, b.bits)
    x = stacked_grey(g, palette(g, 4000), 1)
    ca, na = a.encode(x)
    cb, nb = b.encode(x)
    assert np.array_equal(ca, cb) and np.array_equal(na, nb)
    with pytest.raises(ValueError, match="16-bit"):
        FrameCoder(8).load_state_dict(a.state_dict())
    with pytest.raises(ValueError, match="8-bit"):
        FrameCoder(16).load_state_dict(FrameCoder(8).state_dict())
    with pytest.raises(ValueError):
        b.load_state_dict({"bits": np.zeros(2, np.uint32), "code_bits": 16})   # a repeated pattern: not a code table


# ---- the drop-in buffer -------------------------------------------------------------------------------------------------
def buffer(**kw):
    from training.replay_buffer import ReplayBuffer
    return ReplayBuffer(obsv_dim=(4, 64, 64), action_dim=2, buffer_max_size=10, dsact_replay_frames=4, **kw)


def test_codes_kwarg():
    assert buffer(dsact_replay_codes=16).coder.code_bits == 16
    assert buffer(dsact_replay_codes=True).coder.code_bits == 8
    assert buffer(dsact_replay_codes=False).coder is None and buffer().coder is None
    for bad in (8, 12, 32, "16", 1.5):
        with pytest.raises(ValueError, match="dsact_replay_codes"):
            buffer(dsact_replay_codes=bad)
    from training.replay_buffer import ReplayBuffer
    with pytest.raises(ValueError, match="dsact_replay_frames"):
        ReplayBuffer(obsv_dim=(4, 8, 8), action_dim=3, buffer_max_size=10, dsact_replay_codes=16)


def test_drop_in_buffer_refuses_a_65537th_value_and_stays_as_it_was():
    b = buffer(dsact_replay_codes=16)
    levels = np.arange(65536, dtype=np.float32) / 7
    obs = levels.reshape(4, 4, 64, 64)
    b.store(obs[0], {}, np.zeros(2), 0.0, obs[1], 0.0, 0.0, {})
    b.store(obs[2], {}, np.zeros(2), 0.0, obs[3], 0.0, 0.0, {})
    assert b.coder.n == 65536 and len(b) == 2
    before = (len(b), len(b._pending), b.coder.n, b.coder.bits.copy(), b.planner.state_dict())
    bad = obs[3].copy()
    bad[1, 2, 3] = -1.0
    with pytest.raises(ValueError, match="-1.0"):
        b.store(obs[3], {}, np.zeros(2), 0.0, bad, 0.0, 0.0, {})
    after = (len(b), len(b._pending), b.coder.n, b.coder.bits, b.planner.state_dict())
    assert before[:3] == after[:3] and np.array_equal(before[3], after[3])
    assert before[4]["next"] == after[4]["next"] and np.array_equal(before[4]["serials"], after[4]["serials"])


def test_stacked_grey_frames_are_refused_by_the_8_bit_ring_and_taken_by_the_16_bit_ring():
    """A stacked-grey source (4 x 96 x 96, obs2[k] = obs[k + 1]) over a palette of 3000 RGB colours: more than 256 and
    at most 65 536 distinct float32 values."""
    from training.replay_buffer import ReplayBuffer
    g = np.random.default_rng(5)
    frames = stacked_grey(g, palette(g, 3000), 8)
    n = len(np.unique(frames.view(np.uint32)))
    assert 256 < n <= 65536
    kw = dict(obsv_dim=(4, 96, 96), action_dim=3, buffer_max_size=8, dsact_replay_frames=4)
    b8, b16 = ReplayBuffer(**kw, dsact_replay_codes=True), ReplayBuffer(**kw, dsact_replay_codes=16)
    rows = [(frames[t:t + 4], np.zeros(3), 0.0, frames[t + 1:t + 5], 0.0, 0.0) for t in range(4)]
    with pytest.raises(ValueError, match="256"):
        for o, a, r, o2, d, lp in rows:
            b8.store(o, {}, a, r, o2, d, lp, {})
    for o, a, r, o2, d, lp in rows:
        b16.store(o, {}, a, r, o2, d, lp, {})
    assert len(b16) == 4 and b16.coder.n == n
    for o, *_ in rows:
        codes, new = b16.coder.encode(o)
        assert len(new) == 0 and codes.dtype == np.uint16
        np.testing.assert_array_equal(b16.coder.table[codes].view(np.uint32), o.view(np.uint32))


# ---- C ABI --------------------------------------------------------------------------------------------------------------
def _prototype_params(name):
    header = open(os.path.join(REPO, "include", "dsact.h")).read()
    m = re.search(r"\b%s\s*\(([^)]*)\)" % name, header)
    assert m, name
    return [re.sub(r"\s+", " ", p.strip()) for p in m.group(1).split(",")]


def test_coded16_entry_points_match_the_header_and_the_8_bit_calls():
    bind = _prototype_params("dsact_replay_bind_coded16_frames")
    assert bind == _prototype_params("dsact_replay_bind_coded_frames")
    add, add8 = _prototype_params("dsact_replay_add_coded16_frames"), _prototype_params("dsact_replay_add_coded_frames")
    assert add[1] == "const uint16_t *codes" and add[4] == "const float *table" and add[5] == "int32_t n_codes"
    assert add[:1] + add[2:] == add8[:1] + add8[2:], "the 8-bit call's argument order"
    for name, params, twin in (("dsact_replay_bind_coded16_frames", bind, "dsact_replay_bind_coded_frames"),
                               ("dsact_replay_add_coded16_frames", add, "dsact_replay_add_coded_frames")):
        restype, argtypes = _lib.SYMBOLS[name]
        assert len(argtypes) == len(params), name
        assert _lib.SYMBOLS[name] == _lib.SYMBOLS[twin], name


def test_coded16_entry_points_refuse_without_a_handle():
    lib = _lib.load()
    rb = _lib.FrameReplay()
    assert lib.dsact_replay_bind_coded16_frames(None, C.byref(rb), None) == -1
    assert b"null" in lib.dsact_last_error()
    assert lib.dsact_replay_add_coded16_frames(None, None, 0, 0, None, 0, None, None, None, None, None, None, 0, 0,
                                               None) == -3
    assert b"16-bit coded frame replay ring not bound" in lib.dsact_last_error()
