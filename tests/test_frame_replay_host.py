"""The frame ring's host planner (dsac_v2_b200/frame_plan.py) on random episode streams, with a numpy frame store that
follows its writes and growths: every live row rebuilds bit for bit, no frame a live row refers to is overwritten, the
store grows within the flat ring's size, stacked streams hold about one frame per row, and the state round-trips."""
import numpy as np
import pytest

from dsac_v2_b200.frame_plan import FramePlanner

F = 5   # floats per frame: odd, as the gather's scalar path takes


def episode_rows(g, kind, K, length, reset_stack):
    """(obs, obs2, done) rows of one episode of `length` steps.  kind: "shift" (obs_t = obs2_{t-1}, K frames per
    observation drawn together), "stacked" (obs2 = obs shifted by one frame), "none" (nothing shared)."""
    frame = lambda: g.standard_normal(F).astype(np.float32)
    if kind == "stacked":
        stack = [frame()] * K if reset_stack else [frame() for _ in range(K)]
        for t in range(length):
            nxt = stack[1:] + [frame()]
            yield np.concatenate(stack), np.concatenate(nxt), float(t == length - 1)
            stack = nxt
    elif kind == "shift":
        obs = np.concatenate([frame()] * K) if reset_stack else g.standard_normal(K * F).astype(np.float32)
        for t in range(length):
            nxt = g.standard_normal(K * F).astype(np.float32)
            yield obs, nxt, float(t == length - 1)
            obs = nxt
    else:
        for t in range(length):
            yield g.standard_normal(K * F).astype(np.float32), g.standard_normal(K * F).astype(np.float32), 0.0


def stream(seed, K, kinds, n_rows):
    """Rows of random episodes (lengths 1-50) of the given kinds, with a flag on each episode's first row."""
    g = np.random.default_rng(seed)
    n = 0
    while n < n_rows:
        kind = kinds[g.integers(len(kinds))]
        for t, (o, o2, d) in enumerate(episode_rows(g, kind, K, int(g.integers(1, 51)), bool(g.integers(2)))):
            yield o, o2, d, t == 0
            n += 1


class Store:
    """A numpy frame store that follows the planner: its writes, its growths, and which serial each slot holds."""

    def __init__(self, pl):
        self.pl = pl
        self.frames = np.full((pl.frame_capacity, pl.F), np.nan, np.float32)
        self.holds = np.full(pl.frame_capacity, -1, np.int64)
        self.grown = 0

    def store(self, obs, obs2):
        pl = self.pl
        p = pl.plan(obs, obs2)
        if p.need > pl.frame_capacity:
            cap = pl.grown_capacity(p.need)
            assert p.need <= cap <= pl.max_frames
            src, dst = pl.moves(cap)
            frames, holds = np.full((cap, pl.F), np.nan, np.float32), np.full(cap, -1, np.int64)
            frames[dst], holds[dst] = self.frames[src], self.holds[src]
            self.frames, self.holds = frames, holds
            pl.frame_capacity = cap
            self.grown += 1
        keep = min(pl.size, pl.capacity - 1)
        live = {int(s) for r in range(1, keep + 1) for s in pl.serials[(pl.ptr - r) % pl.capacity]} | set(p.serials.tolist())
        row, slots, new, frame_ptr = pl.commit(p)
        for i, f in enumerate(new):
            slot = (frame_ptr + i) % pl.frame_capacity
            assert self.holds[slot] not in live, "a frame a live row refers to was overwritten"
            self.frames[slot], self.holds[slot] = f, pl.next - len(new) + i
        assert np.array_equal(slots % pl.frame_capacity, slots)
        return row

    def rebuild(self, row):
        K = self.pl.K
        slots = self.pl.slots()[row]
        return self.frames[slots[:K]].reshape(-1), self.frames[slots[K:]].reshape(-1)


def run(pl, rows, check_every=1):
    st = Store(pl)
    held_rows = {}
    for n, (o, o2, d, first) in enumerate(rows):
        row = st.store(o, o2)
        held_rows[row] = (o, o2, first)
        if n % check_every == 0:
            for r, (a, b, _) in held_rows.items():
                ra, rb = st.rebuild(r)
                assert ra.view(np.uint32).tolist() == a.view(np.uint32).tolist(), (n, r)
                assert rb.view(np.uint32).tolist() == b.view(np.uint32).tolist(), (n, r)
        assert pl.frame_capacity <= 2 * pl.K * pl.capacity and pl.held() <= pl.frame_capacity
    return st, held_rows


@pytest.mark.parametrize("kinds", [("shift",), ("stacked",), ("none",), ("shift", "stacked", "none")])
@pytest.mark.parametrize("K", [1, 2, 4])
def test_rows_rebuild_bit_for_bit_while_the_ring_wraps(K, kinds):
    pl = FramePlanner(37, K, K * F)
    st, _ = run(pl, stream(K * 7 + len(kinds), K, kinds, 600))
    assert pl.size == 37 and pl.next > 2 * pl.frame_capacity   # wrapped many times
    if "none" in kinds:
        assert st.grown >= 1


@pytest.mark.parametrize("K", [1, 2, 4])
def test_stacked_stream_holds_about_one_frame_per_row(K):
    pl = FramePlanner(37, K, K * F)
    st = Store(pl)
    firsts = {}
    for n, (o, o2, d, first) in enumerate(stream(5 + K, K, ("stacked",), 900)):
        row = st.store(o, o2)
        firsts[row] = first
        starts = sum(firsts.values())
        # each episode start stores its first stack (at most K frames) and the oldest live row reaches back at most K + 1
        assert pl.held() <= pl.size + (K + 2) * (starts + 1), (n, pl.held(), pl.size, starts)


def test_no_sharing_grows_to_the_flat_size_and_no_further():
    pl = FramePlanner(37, 2, 2 * F)
    st, _ = run(pl, stream(1, 2, ("none",), 300), check_every=7)
    assert pl.frame_capacity == pl.max_frames == 2 * 2 * 37 and st.grown >= 1


def test_a_frame_repeated_forever_is_stored_again_rather_than_outgrowing_the_ring():
    """obs = [X, a_t], obs2 = [X, a_{t+1}]: every row would refer to the first X ever stored; a row may reach back only 2K
    serials minus what it stores, so X is stored again now and then and the store stays within 2K per row."""
    g = np.random.default_rng(0)
    X = g.standard_normal(F).astype(np.float32)
    a = [g.standard_normal(F).astype(np.float32) for _ in range(501)]
    pl = FramePlanner(37, 2, 2 * F)
    run(pl, ((np.concatenate([X, a[t]]), np.concatenate([X, a[t + 1]]), 0.0, t == 0) for t in range(500)), check_every=5)
    assert pl.frame_capacity <= pl.max_frames


def test_frames_are_compared_bit_for_bit():
    pl = FramePlanner(4, 1, 3)
    z = np.zeros(3, np.float32)
    p = pl.plan(z, -z)   # 0.0 and -0.0 compare equal as floats, not as stored bits
    assert len(p.new) == 2
    pl.commit(p)
    p = pl.plan(-z, np.ones(3, np.float32))   # obs == the last row's obs2
    assert len(p.new) == 1 and p.serials[0] == 1


def test_state_round_trips():
    K = 4
    rows = list(stream(9, K, ("stacked", "shift", "none"), 400))
    a = FramePlanner(37, K, K * F)
    sa = Store(a)
    for r in rows[:250]:
        sa.store(*r[:2])
    b = FramePlanner(37, K, K * F)
    b.load_state_dict(a.state_dict())
    sb = Store(b)
    sb.frames, sb.holds = sa.frames.copy(), sa.holds.copy()
    for r in rows[250:]:
        assert sa.store(*r[:2]) == sb.store(*r[:2])
        assert np.array_equal(a.slots(), b.slots()) and a.frame_capacity == b.frame_capacity
    assert np.array_equal(sa.frames, sb.frames, equal_nan=True)


@pytest.mark.parametrize("K, O", [(0, 8), (3, 8), (65, 65 * 2)])
def test_refuses_a_frame_count_that_does_not_divide_the_observation(K, O):
    with pytest.raises(ValueError):
        FramePlanner(8, K, O)
