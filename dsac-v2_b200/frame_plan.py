"""Host planner of the frame replay ring (dsact_frame_replay, include/dsact.h): decides, row by row, which observation
frames are stored and which are shared, and where every frame lives.  Pure numpy; it touches no device.

An observation of O floats is K frames of F = O / K floats.  A frame of a new row is stored only if it does not equal,
bit for bit, a frame of the previous row's obs2 or a frame earlier in the same row; otherwise the row refers to that
frame.  This catches obs_t == obs2_{t-1}, stacked frames (obs2[k] == obs[k+1]) and reset stacks ([f0] * K) with at most
4K^2 frame compares per row and no hashing.

Frames take consecutive serial numbers and go into slot serial % frame_capacity.  Each row records the oldest serial it
refers to (its `first`); `first` never decreases from one row to the next, so the frames still needed are exactly the
serials from the oldest live row's `first` on, and a slot may be reused once its old serial is older than that.  A row
may reach back at most 2K - (frames it stores) serials before its own, which keeps the live serial span within 2K per
live row: the flat ring's size, the most the frame store ever needs.  When a row needs more than the current
frame_capacity, the caller grows the store (`grown_capacity`, `moves`) before committing the row.
"""
from __future__ import annotations

from typing import Optional

import numpy as np


class FramePlan:
    """One planned row: its 2K frame serials (obs then obs2), the frames it stores and the capacity it needs."""
    __slots__ = ("serials", "new", "need", "bits")

    def __init__(self, serials, new, need, bits):
        self.serials, self.new, self.need, self.bits = serials, new, need, bits


class FramePlanner:
    def __init__(self, capacity: int, frames_per_obs: int, obs_elems: int, frame_capacity: Optional[int] = None):
        K, C = int(frames_per_obs), int(capacity)
        if C < 1 or not 1 <= K <= 64 or obs_elems % K:
            raise ValueError(f"frames_per_obs {K} must be in [1, 64] and divide the observation's {obs_elems} floats")
        self.K, self.F, self.capacity = K, int(obs_elems) // K, C
        self.max_frames = 2 * K * C
        self.frame_capacity = min(C + C // 16 + 2 * K, self.max_frames) if frame_capacity is None else int(frame_capacity)
        self.next = 0                       # serial of the next stored frame
        self.ptr, self.size = 0, 0          # ring row of the next row, rows held
        self.serials = np.zeros((C, 2 * K), np.int64)   # per row: serials of obs frames, then of obs2 frames
        self.first = np.zeros(C, np.int64)
        self.prev_bits = None               # uint32 [K, F]: the last row's obs2 frames, and their serials
        self.prev_serials = None

    # ---- planning ---------------------------------------------------------------------------------------------------
    def plan(self, obs: np.ndarray, obs2: np.ndarray) -> FramePlan:
        """Plan the next row (changes nothing).  `obs`, `obs2`: O float32 values each."""
        K, S = self.K, self.next
        frames = np.concatenate([np.asarray(obs, np.float32).reshape(K, self.F),
                                 np.asarray(obs2, np.float32).reshape(K, self.F)])
        bits = frames.view(np.uint32)
        # the compares, once: the first equal frame earlier in this row, else the first equal frame of the last obs2
        dup = np.full(2 * K, -1)
        hit = np.full(2 * K, -1)
        for j in range(2 * K):
            for i in range(j):
                if dup[i] < 0 and np.array_equal(bits[i], bits[j]):
                    dup[j] = i
                    break
            if dup[j] < 0 and self.prev_bits is not None:
                for k in range(K):
                    if np.array_equal(self.prev_bits[k], bits[j]):
                        hit[j] = k
                        break
        floor = -1   # serials below `floor` are not referred to: the frame is stored again
        while True:
            ser = np.empty(2 * K, np.int64)
            new = []
            for j in range(2 * K):
                if dup[j] >= 0:
                    ser[j] = ser[dup[j]]
                elif hit[j] >= 0 and self.prev_serials[hit[j]] >= floor:
                    ser[j] = self.prev_serials[hit[j]]
                else:
                    ser[j] = S + len(new)
                    new.append(j)
            lo = int(ser.min())
            if lo >= S or S - lo <= 2 * K - len(new):
                break
            floor = lo + 1
        keep = min(self.size, self.capacity - 1)   # rows that stay live beside this one
        live = lo if keep == 0 else min(lo, int(self.first[(self.ptr - keep) % self.capacity]))
        return FramePlan(ser, np.asarray(new, np.int64), S + len(new) - live, bits)

    def live_first(self) -> int:
        """Oldest serial a row held now refers to (`next` when no row is held)."""
        return self.next if self.size == 0 else int(self.first[(self.ptr - self.size) % self.capacity])

    def grown_capacity(self, need: int) -> int:
        """Frame capacity to grow to for a row that needs `need` frames."""
        return min(max(need, self.frame_capacity + self.frame_capacity // 2), self.max_frames)

    def moves(self, new_capacity: int):
        """(old slots, new slots) of every frame rows held now refer to, for growing the store to `new_capacity`."""
        s = np.arange(self.live_first(), self.next, dtype=np.int64)
        return s % self.frame_capacity, s % new_capacity

    def commit(self, p: FramePlan):
        """Store the planned row: returns (row, int32 slots [2K], new frames float32 [m, F], slot of the first of them)."""
        if p.need > self.frame_capacity:
            raise RuntimeError(f"the row needs {p.need} frames; grow the frame store first ({self.frame_capacity})")
        K, row = self.K, self.ptr
        self.serials[row] = p.serials
        self.first[row] = p.serials.min()
        frame_ptr = self.next % self.frame_capacity
        self.next += len(p.new)
        self.prev_bits, self.prev_serials = p.bits[K:].copy(), p.serials[K:].copy()
        self.ptr = (row + 1) % self.capacity
        self.size = min(self.size + 1, self.capacity)
        return row, (p.serials % self.frame_capacity).astype(np.int32), p.bits[p.new].view(np.float32), frame_ptr

    def slots(self) -> np.ndarray:
        """int32 [capacity, 2K]: every row's frame slots at the current capacity."""
        return (self.serials % self.frame_capacity).astype(np.int32)

    def held(self) -> int:
        """Frames the rows held refer to, and the frames between them: what the store must keep."""
        return self.next - self.live_first()

    # ---- checkpoint -----------------------------------------------------------------------------------------------------
    def state_dict(self) -> dict:
        return {"K": self.K, "F": self.F, "capacity": self.capacity, "frame_capacity": self.frame_capacity,
                "next": self.next, "ptr": self.ptr, "size": self.size, "serials": self.serials.copy(),
                "first": self.first.copy(),
                "prev_bits": None if self.prev_bits is None else self.prev_bits.copy(),
                "prev_serials": None if self.prev_serials is None else self.prev_serials.copy()}

    def load_state_dict(self, st: dict) -> None:
        if (st["K"], st["F"], st["capacity"]) != (self.K, self.F, self.capacity):
            raise ValueError("frame planner state of a different ring shape")
        self.frame_capacity, self.next = int(st["frame_capacity"]), int(st["next"])
        self.ptr, self.size = int(st["ptr"]), int(st["size"])
        self.serials, self.first = np.array(st["serials"], np.int64), np.array(st["first"], np.int64)
        self.prev_bits = None if st["prev_bits"] is None else np.array(st["prev_bits"], np.uint32)
        self.prev_serials = None if st["prev_serials"] is None else np.array(st["prev_serials"], np.int64)


class FrameCoder:
    """Host coder of the coded frame rings (dsact_replay_bind_coded_frames, dsact_replay_bind_coded16_frames): float32
    values -> codes of `code_bits` bits (8: uint8, up to 256 values; 16: uint16, up to 65 536) through a table.  Values
    are matched on their bit patterns (so -0.0 and 0.0, and NaNs of different payloads, are different values) and take
    codes in order of first appearance.  The table is a bijection between codes and the bit patterns seen, so comparing
    codes is comparing values.

    Lookup, with no Python loop over values.  8 bits: a multiplicative hash (bits * mul mod 2^32) >> 16 into 65536 slots,
    with `mul` chosen so that no two table entries share a slot; a value is known when its slot holds its own bit
    pattern.  16 bits: a table that large cannot be placed collision-free in such a hash, so a binary search
    (np.searchsorted) over the patterns held, kept sorted beside their codes."""
    _SHIFT = 16

    def __init__(self, code_bits: int = 8):
        if code_bits not in (8, 16):
            raise ValueError(f"code_bits {code_bits!r}: the coded frame rings take 8- or 16-bit codes")
        self.code_bits = code_bits
        self.N = 1 << code_bits
        self.dtype = np.uint8 if code_bits == 8 else np.uint16
        self.bits = np.zeros(self.N, np.uint32)   # table: code -> bit pattern
        self.n = 0
        if code_bits == 8:
            self._mul = np.uint32(0x9E3779B1)
            self._used = np.zeros(1 << (32 - self._SHIFT), bool)    # slot -> (holds an entry, its pattern, its code)
            self._slot_bits = np.zeros(1 << (32 - self._SHIFT), np.uint32)
            self._slot_code = np.zeros(1 << (32 - self._SHIFT), np.uint8)
        else:
            self._sorted = np.zeros(0, np.uint32)        # the patterns held, ascending, and their codes
            self._sorted_code = np.zeros(0, np.uint16)

    @property
    def table(self) -> np.ndarray:
        """float32 [N]: code -> value (entries from n on are unused)."""
        return self.bits.view(np.float32)

    def _slots(self, flat: np.ndarray, mul) -> np.ndarray:
        return (flat * mul) >> np.uint32(self._SHIFT)

    def _find(self, flat: np.ndarray):
        """(known: bool per value, codes: a writable code array, valid where known)."""
        if self.code_bits == 8:
            s = self._slots(flat, self._mul)
            return self._used[s] & (self._slot_bits[s] == flat), self._slot_code[s]
        if self.n == 0:
            return np.zeros(flat.shape, bool), np.zeros(flat.shape, np.uint16)
        i = np.minimum(np.searchsorted(self._sorted, flat), self.n - 1)
        return self._sorted[i] == flat, self._sorted_code[i]

    def encode(self, values: np.ndarray):
        """(codes of `values`' shape, bit patterns the table does not hold yet, in order of first appearance).
        Changes nothing; ValueError when the table would need more than N entries."""
        b = np.ascontiguousarray(values, np.float32).view(np.uint32)
        flat = b.reshape(-1)
        known, codes = self._find(flat)
        if known.all():
            return codes.reshape(b.shape), flat[:0]
        miss = ~known
        uniq, first, inv = np.unique(flat[miss], return_index=True, return_inverse=True)
        order = np.argsort(first)
        new = uniq[order]
        if self.n + len(new) > self.N:
            v = new[self.N - self.n]
            raise ValueError(f"the {self.code_bits}-bit coded replay ring holds at most {self.N} distinct observation "
                             f"values; {np.array(v, np.uint32).view(np.float32).item()!r} (bits 0x{int(v):08x}) would be "
                             f"value {self.N + 1}: the observations are not {self.code_bits}-bit quantised")
        rank = np.empty(len(uniq), np.int64)
        rank[order] = np.arange(len(uniq))
        codes[miss] = (self.n + rank[inv.reshape(-1)]).astype(self.dtype)
        return codes.reshape(b.shape), new

    def commit(self, new: np.ndarray) -> None:
        """Append the patterns `encode` returned to the table."""
        if len(new) == 0:
            return
        start = self.n
        self.bits[self.n:self.n + len(new)] = new
        self.n += len(new)
        if self.code_bits == 16:
            o = np.argsort(new)
            pos = np.searchsorted(self._sorted, new[o])
            self._sorted = np.insert(self._sorted, pos, new[o])
            self._sorted_code = np.insert(self._sorted_code, pos, (start + o).astype(np.uint16))
            return
        bits = self.bits[:self.n]
        mul, g = self._mul, np.random.default_rng(self.n)
        while len(np.unique(self._slots(bits, mul))) != self.n:   # a collision: another odd multiplier
            mul = np.uint32(int(g.integers(0, 2 ** 31)) * 2 + 1)
        self._mul = mul
        s = self._slots(bits, mul)
        self._used[:] = False
        self._used[s] = True
        self._slot_bits[s] = bits
        self._slot_code[s] = np.arange(self.n).astype(np.uint8)

    def state_dict(self) -> dict:
        st = {"bits": self.bits[:self.n].copy()}
        if self.code_bits != 8:   # (8-bit states keep the form they always had)
            st["code_bits"] = self.code_bits
        return st

    def load_state_dict(self, st: dict) -> None:
        if st.get("code_bits", 8) != self.code_bits:
            raise ValueError(f"frame coder state of {st.get('code_bits', 8)}-bit codes, not {self.code_bits}-bit")
        bits = np.asarray(st["bits"], np.uint32)
        if len(bits) > self.N or len(np.unique(bits)) != len(bits):
            raise ValueError(f"frame coder state: not a table of at most {self.N} distinct values")
        self.bits[:] = 0
        self.n = 0
        if self.code_bits == 16:
            self._sorted, self._sorted_code = self._sorted[:0], self._sorted_code[:0]
        self.commit(bits)
