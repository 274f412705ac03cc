"""The coded frame ring's host side, without a GPU: the bit-pattern coder (dsac_v2_b200/frame_plan.py FrameCoder) on
CarRacing-raw observations made as the reference makes them, on signed zeros and NaN payloads, its refusal of a 257th
value, its state round trip; the drop-in kwarg; and the C entry points' declarations and refusals."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from dsac_v2_b200 import _lib
from dsac_v2_b200.frame_plan import FrameCoder

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def carracing_raw(g, n):
    """n observations of `gym_carracingraw`: uint8 rgb [96, 96, 3] -> rgb.transpose(2, 0, 1) / 255 (float64), stored as
    float32 by the replay buffer."""
    rgb = g.integers(0, 256, (n, 96, 96, 3), dtype=np.uint8)
    return np.stack([np.asarray(x.transpose(2, 0, 1) / 255, dtype=np.float32) for x in rgb])


def decode(coder, codes):
    return coder.table[codes]


def test_carracing_raw_frames_code_losslessly_in_at_most_256_values():
    g = np.random.default_rng(0)
    coder = FrameCoder()
    for _ in range(3):
        obs = carracing_raw(g, 2)
        codes, new = coder.encode(obs)
        coder.commit(new)
        assert codes.dtype == np.uint8 and codes.shape == obs.shape
        np.testing.assert_array_equal(decode(coder, codes).view(np.uint32), obs.view(np.uint32))
    assert coder.n == 256
    want = np.asarray(np.arange(256) / 255, dtype=np.float32)
    assert set(coder.table[:coder.n].view(np.uint32).tolist()) == set(want.view(np.uint32).tolist())
    # a source that only shows some of the 256 levels takes only those
    small = FrameCoder()
    dark = np.asarray(g.integers(0, 40, (3, 96, 96)) / 255, dtype=np.float32)
    codes, new = small.encode(dark)
    small.commit(new)
    assert small.n == len(np.unique(dark))
    np.testing.assert_array_equal(decode(small, codes).view(np.uint32), dark.view(np.uint32))


def test_codes_follow_first_appearance_and_bit_patterns():
    nan_a = np.array([0x7FC00001], np.uint32).view(np.float32)[0]
    nan_b = np.array([0x7FC00002], np.uint32).view(np.float32)[0]
    v = np.array([0.5, -0.0, 0.0, 0.5, nan_a, nan_b, -0.0, nan_a], np.float32)
    coder = FrameCoder()
    codes, new = coder.encode(v)
    assert coder.n == 0, "encode changed the table"
    coder.commit(new)
    assert codes.tolist() == [0, 1, 2, 0, 3, 4, 1, 3]
    assert coder.n == 5
    np.testing.assert_array_equal(decode(coder, codes).view(np.uint32), v.view(np.uint32))
    # known values take their codes again; new ones are appended
    codes, new = coder.encode(np.array([0.0, 0.25, nan_b], np.float32))
    coder.commit(new)
    assert codes.tolist() == [2, 5, 4] and coder.n == 6


@pytest.mark.parametrize("seed", range(4))
def test_codes_equal_a_dictionary_coder_on_random_bit_patterns(seed):
    # 256 random patterns (hash collisions among them force other multipliers), fed in random batches
    g = np.random.default_rng(seed)
    pats = np.unique(g.integers(0, 2 ** 32, 300, dtype=np.uint64).astype(np.uint32))[:256]
    g.shuffle(pats)
    coder, ref = FrameCoder(), {}
    for _ in range(40):
        x = pats[g.integers(0, min(len(pats), 8 + 8 * len(ref)), int(g.integers(1, 500)))]
        codes, new = coder.encode(x.view(np.float32))
        coder.commit(new)
        want = [ref.setdefault(int(v), len(ref)) for v in x]
        assert codes.tolist() == want
        assert coder.n == len(ref)
    assert np.array_equal(coder.bits[:coder.n], np.array(sorted(ref, key=ref.get), np.uint32))


def test_the_257th_value_is_refused_and_nothing_changes():
    coder = FrameCoder()
    _, new = coder.encode(np.arange(256, dtype=np.float32))
    coder.commit(new)
    bits = coder.bits.copy()
    with pytest.raises(ValueError, match="256"):
        coder.encode(np.array([3.0, 1000.5, 2.0], np.float32))
    assert coder.n == 256 and np.array_equal(coder.bits, bits)
    with pytest.raises(ValueError, match="1000.5"):   # the message names the value
        coder.encode(np.array([1000.5], np.float32))


def test_drop_in_buffer_refuses_an_uncodable_row_and_stays_as_it_was():
    from training.replay_buffer import ReplayBuffer
    b = ReplayBuffer(obsv_dim=(2, 4, 4), action_dim=2, buffer_max_size=10, dsact_replay_frames=2, dsact_replay_codes=True)
    levels = np.arange(256, dtype=np.float32) / 7
    rows = [levels[i * 64:(i + 1) * 64].reshape(2, 2, 4, 4) for i in range(4)]
    for i in range(2):
        b.store(rows[2 * i][0], {}, np.zeros(2), 0.0, rows[2 * i + 1][0], 0.0, 0.0, {})
        b.store(rows[2 * i][1], {}, np.zeros(2), 0.0, rows[2 * i + 1][1], 0.0, 0.0, {})
    assert b.coder.n == 256 and len(b) == 4
    before = (len(b), len(b._pending), b.coder.n, b.coder.bits.copy(), b.planner.state_dict())
    bad = rows[0][0].copy()
    bad[1, 2, 3] = -1.0
    with pytest.raises(ValueError, match="-1.0"):
        b.store(rows[0][0], {}, np.zeros(2), 0.0, bad, 0.0, 0.0, {})
    after = (len(b), len(b._pending), b.coder.n, b.coder.bits, b.planner.state_dict())
    assert before[:3] == after[:3] and np.array_equal(before[3], after[3])
    assert before[4]["next"] == after[4]["next"] and np.array_equal(before[4]["serials"], after[4]["serials"])


def test_coder_state_round_trips():
    g = np.random.default_rng(1)
    a = FrameCoder()
    _, new = a.encode(carracing_raw(g, 1)[0, :, :5])
    a.commit(new)
    b = FrameCoder()
    b.load_state_dict(a.state_dict())
    assert b.n == a.n and np.array_equal(a.bits, b.bits)
    x = carracing_raw(g, 1)
    ca, na = a.encode(x)
    cb, nb = b.encode(x)
    assert np.array_equal(ca, cb) and np.array_equal(na, nb)
    with pytest.raises(ValueError):
        b.load_state_dict({"bits": np.zeros(2, np.uint32)})   # a repeated pattern: not a code table


def test_codes_kwarg_needs_the_frame_ring():
    from training.replay_buffer import ReplayBuffer
    with pytest.raises(ValueError, match="dsact_replay_frames"):
        ReplayBuffer(obsv_dim=(3, 8, 8), action_dim=3, buffer_max_size=10, dsact_replay_codes=True)
    assert ReplayBuffer(obsv_dim=(3, 8, 8), action_dim=3, buffer_max_size=10).coder is None


# ---- C ABI --------------------------------------------------------------------------------------------------------------
def _prototype_params(name):
    header = open(os.path.join(REPO, "include", "dsact.h")).read()
    m = re.search(r"\b%s\s*\(([^)]*)\)" % name, header)
    assert m, name
    return [p.strip() for p in m.group(1).split(",")]


def test_coded_ring_entry_points_match_the_header():
    bind = _prototype_params("dsact_replay_bind_coded_frames")
    assert bind == ["dsact_handle *h", "const dsact_frame_replay *rb", "const float *table"]
    add = _prototype_params("dsact_replay_add_coded_frames")
    assert add[1] == "const uint8_t *codes" and add[4] == "const float *table" and add[5] == "int32_t n_codes"
    for name, params in (("dsact_replay_bind_coded_frames", bind), ("dsact_replay_add_coded_frames", add)):
        restype, argtypes = _lib.SYMBOLS[name]
        assert len(argtypes) == len(params), name
    # the ring is described by the frame ring's struct
    assert _lib.SYMBOLS["dsact_replay_bind_coded_frames"][1][1] == C.POINTER(_lib.FrameReplay)
    assert [t for t in _lib.SYMBOLS["dsact_replay_add_coded_frames"][1]][5] is C.c_int32


def test_coded_ring_entry_points_refuse_without_a_handle():
    lib = _lib.load()
    rb = _lib.FrameReplay()
    assert lib.dsact_replay_bind_coded_frames(None, C.byref(rb), None) == -1
    assert b"null" in lib.dsact_last_error()
    assert lib.dsact_replay_add_coded_frames(None, None, 0, 0, None, 0, None, None, None, None, None, None, 0, 0, None) == -3
    assert b"not bound" in lib.dsact_last_error()
