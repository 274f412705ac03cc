"""`training.replay_buffer` of the drop-in: the reference's `ReplayBuffer`
interface (reference training/replay_buffer.py:15-90) over a DEVICE-resident ring
buffer.  Transitions are staged in pinned host memory and copied to the GPU
asynchronously; `sample_batch` is a coalesced row gather on the GPU
(libdsact `dsact_replay_sample`), so no H2D copy sits on the update step.

Uniform sampling with replacement, like `np.random.randint` (reference :86).
`index_source="numpy"` draws the indices from numpy's global generator exactly as
the reference does (same seed -> same minibatch rows); the default "device" draws
them with Philox on the GPU.

`dsact_replay_frames=K` stores each observation frame once instead (the frame ring, include/dsact.h): an observation
is K frames of obs_elems / K floats (an NCHW image with K = C: one channel each; K = 1: the whole observation), and a
row refers to the frames of the previous row's obs2 or of its own obs that it repeats (dsac_v2_b200/frame_plan.py).
The minibatches are bit for bit those of the flat ring; the device memory is about half of it (K = 1, obs2_t = obs_{t+1})
or less (stacked frames: one new frame per row).

`dsact_replay_codes=True` (with `dsact_replay_frames`) stores the frames as 8-bit codes into a table of at most 256
float32 values (the coded frame ring): a quarter of the frame bytes, for observations with at most 256 distinct values
(8-bit images scaled to floats, such as `gym_carracingraw`'s rgb / 255).  Values are matched bit for bit; a store that
brings a 257th distinct value raises ValueError and leaves the buffer as it was.  The minibatches are still bit for bit
those of the flat ring.

`dsact_replay_codes=16` (with `dsact_replay_frames`) stores 16-bit codes into a table of at most 65 536 values: half the
frame bytes, for sources such as `gym_carracing`'s stacked grey frames (`dot(rgb, [0.299, 0.587, 0.114]) / 128 - 1`)
whose stream uses at most 65 536 distinct values.  A store that brings a 65 537th value is refused the same way.
"""
__all__ = ["ReplayBuffer"]

import numpy as np
import torch

from dsac_v2_b200.frame_plan import FrameCoder, FramePlanner


class ReplayBuffer:
    _STAGE_ROWS = 4096
    _STAGES = 4

    def __init__(self, index=0, **kwargs):
        self.obsv_dim = kwargs["obsv_dim"]
        self.act_dim = kwargs["action_dim"]
        self.max_size = int(kwargs["buffer_max_size"])
        if not np.isscalar(self.act_dim):
            raise NotImplementedError("the device ring buffer stores flat action vectors")
        # image observations (CNN path, BASELINE config 5): rows hold the flattened [C*H*W] image
        self.obs_shape = None if np.isscalar(self.obsv_dim) else tuple(int(x) for x in self.obsv_dim)
        self.obs_elems = int(self.obsv_dim) if self.obs_shape is None else int(np.prod(self.obs_shape))
        if kwargs.get("additional_info"):
            raise NotImplementedError("additional_info fields are not supported by the device ring buffer")
        self.index_source = kwargs.get("dsact_index_source",
                                       "numpy" if kwargs.get("dsact_noise") == "reference" else "device")
        self.frames_per_obs = kwargs.get("dsact_replay_frames")
        self.planner = None
        if self.frames_per_obs is not None:
            self.planner = FramePlanner(self.max_size, int(self.frames_per_obs), self.obs_elems)
        self.coder = None
        codes = kwargs.get("dsact_replay_codes")
        if codes is not None and codes is not False:
            if codes is not True and (isinstance(codes, bool) or codes != 16):
                raise ValueError(f"dsact_replay_codes={codes!r}: True (8-bit codes) or 16 (16-bit codes)")
            if self.planner is None:
                raise ValueError("dsact_replay_codes codes the frames of the frame ring: it needs dsact_replay_frames")
            self.coder = FrameCoder(8 if codes is True else 16)
        self.ptr, self.size = 0, 0
        self.engine = None
        self._stage = None      # pinned staging buffers
        self._events = None
        self._cur, self._fill, self._flushed = 0, 0, 0
        self._pending = []      # transitions stored before an engine was attached

    # ---- wiring -------------------------------------------------------------------
    def attach(self, engine):
        """Bind the ring storage to an engine (done by the trainer once the networks are on the GPU)."""
        eng_obs = getattr(engine, "obs_elems", None) or engine.cfg.obs_dim
        if eng_obs != self.obs_elems or engine.cfg.act_dim != self.act_dim:
            raise ValueError("replay buffer and engine disagree on obs/act dimensions")
        self.engine = engine
        O, A = self.obs_elems, self.act_dim
        R = min(self._STAGE_ROWS if self.obs_shape is None else max(8, self._STAGE_ROWS * 400 // O), self.max_size)   # ~6 MB per staging set
        self._rows = R
        pin = lambda *s: torch.zeros(*s, dtype=torch.float32).pin_memory()
        if self.planner is None:
            engine.bind_replay(self.max_size)
            self._stage = [dict(obs=pin(R, O), obs2=pin(R, O), act=pin(R, A), rew=pin(R), done=pin(R), logp=pin(R))
                           for _ in range(self._STAGES)]
        else:
            pl = self.planner
            self._bind_frames(engine, pl.frame_capacity)
            ids = lambda: torch.zeros(R, pl.K, dtype=torch.int32).pin_memory()
            # up to 2K new frames per row: the same bytes as the flat ring's obs + obs2 staging (a quarter with 8-bit codes,
            # a half with 16-bit codes, held in int16 and written through a uint16 view)
            fdt = {None: torch.float32, 8: torch.uint8, 16: torch.int16}[self._code_bits()]
            self._stage = [dict(frames=torch.zeros(2 * R * pl.K, pl.F, dtype=fdt).pin_memory(), obs_frames=ids(),
                                obs2_frames=ids(), act=pin(R, A), rew=pin(R), done=pin(R), logp=pin(R))
                           for _ in range(self._STAGES)]
            self._nframes, self._frame_ptr = 0, 0
        self._np = [{k: v.numpy().view(np.uint16) if v.dtype == torch.int16 else v.numpy() for k, v in s.items()}
                    for s in self._stage]
        self._events = [None] * self._STAGES
        pending, self._pending = self._pending, []
        for row in pending:
            self._store_row(*row)

    def rebind(self, old, new):
        """The engine was rebuilt (larger activation arena): give the new one a ring and move the stored rows."""
        if self.engine is not old:
            return
        self.flush()
        torch.cuda.current_stream(old.device).synchronize()
        if self.planner is None:
            new.bind_replay(self.max_size)
        else:
            self._bind_frames(new, self.planner.frame_capacity)
        for k, v in old.replay.items():
            new.replay[k].copy_(v)
        self.engine = new

    def _code_bits(self):
        return None if self.coder is None else self.coder.code_bits

    def _bind_frames(self, eng, frame_capacity: int):
        eng.bind_replay_frames(self.max_size, frame_capacity, self.planner.K, coded=self.coder is not None,
                               code_bits=self._code_bits() or 8)

    def _require_engine(self):
        if self.engine is None:
            raise RuntimeError("ReplayBuffer is not attached to the CUDA engine: call buffer.attach(alg.networks.engine()) "
                               "(training.trainer.OffSerialTrainer does this). There is no CPU sampling path.")

    def __len__(self):
        return self.size

    def __get_RAM__(self):
        """MB of device memory holding valid transitions (frame ring: the frames they refer to, and their frame ids; coded
        frame rings: one or two bytes per frame value, and the table)."""
        if self.planner is not None:
            pl = self.planner
            c = self.coder
            frames = 4 * pl.F * pl.held() if c is None else c.code_bits // 8 * pl.F * pl.held() + 4 * c.N
            return (frames + 4 * (2 * pl.K + self.act_dim + 3) * self.size) / 1e6
        row_bytes = 4 * (2 * self.obs_elems + self.act_dim + 3)
        return row_bytes * self.size / 1e6

    # ---- store ----------------------------------------------------------------------
    def _store_row(self, obs, act, rew, next_obs, done, logp):
        if self.planner is not None:
            plan = self.planner.plan(obs, next_obs)
            if self.coder is not None:   # (raises before anything changes)
                codes, new_values = self.coder.encode(plan.bits[plan.new].view(np.float32))
            if plan.need > self.planner.frame_capacity:
                self._grow(self.planner.grown_capacity(plan.need))
            # a flush copies at most frame_capacity frames: no two of its frames share a slot
            if self._fill and self._nframes + len(plan.new) > self.planner.frame_capacity:
                self.flush()
        if self._fill == self._rows:
            self.flush()
        if self._fill == 0 and self._events[self._cur] is not None:
            self._events[self._cur].synchronize()  # the async copy out of this staging buffer has finished
        s, i = self._np[self._cur], self._fill
        if self.planner is None:
            s["obs"][i] = obs.reshape(-1)
            s["obs2"][i] = next_obs.reshape(-1)
        else:
            _, slots, new, frame_ptr = self.planner.commit(plan)
            K, m = self.planner.K, len(new)
            if self._fill == 0:
                self._frame_ptr = frame_ptr
            if self.coder is not None:
                self.coder.commit(new_values)
                new = codes
            s["frames"][self._nframes:self._nframes + m] = new
            self._nframes += m
            s["obs_frames"][i], s["obs2_frames"][i] = slots[:K], slots[K:]
        s["act"][i] = act
        s["rew"][i] = rew
        s["done"][i] = done
        s["logp"][i] = logp
        self._fill += 1

    def store(self, obs, info, act, rew, next_obs, done, logp, next_info):
        row = (np.asarray(obs, dtype=np.float32), np.asarray(act, dtype=np.float32), float(rew),
               np.asarray(next_obs, dtype=np.float32), float(done), float(np.asarray(logp)))
        if self.engine is None:
            if self.coder is not None:   # refuse an uncodable row now, not when the buffer is attached
                _, new_values = self.coder.encode(np.concatenate([row[0].reshape(-1), row[3].reshape(-1)]))
                self.coder.commit(new_values)
            self._pending.append(row)
        else:
            self._store_row(*row)
        self.size = min(self.size + 1, self.max_size)

    def add_batch(self, samples: list):
        for sample in samples:
            self.store(*sample)

    def flush(self):
        """Enqueue the async H2D copy of the staged rows into the ring."""
        if self.engine is None or self._fill == 0:
            return
        n = self._fill
        if self.planner is None:
            self.engine.replay_add(self._stage[self._cur], n, self.ptr)
        else:
            st = self._stage[self._cur]
            if self.coder is None:
                self.engine.replay_add_frames(st["frames"], self._nframes, self._frame_ptr, st, n, self.ptr)
            else:
                e = self.engine
                add = e.replay_add_coded_frames if self.coder.code_bits == 8 else e.replay_add_coded16_frames
                add(st["frames"], self._nframes, self._frame_ptr, self.coder.table, self.coder.n, st, n, self.ptr)
            self._nframes = 0
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.engine.device))
        self._events[self._cur] = ev
        self.ptr = (self.ptr + n) % self.max_size
        self._cur = (self._cur + 1) % self._STAGES
        self._fill = 0

    def _grow(self, frame_capacity: int):
        """Move the frame store to `frame_capacity` slots: every live frame to its new slot, every row's ids rewritten."""
        self.flush()
        eng, pl = self.engine, self.planner
        with torch.cuda.device(eng.device):
            old = eng.replay
            src, dst = (torch.from_numpy(x).to(eng.device) for x in pl.moves(frame_capacity))
            self._bind_frames(eng, frame_capacity)
            eng.replay["frames"][dst] = old["frames"][src]
            for k in ("act", "rew", "done", "logp") + (("table",) if self.coder is not None else ()):
                eng.replay[k].copy_(old[k])
            pl.frame_capacity = frame_capacity
            self._put_ids()
            torch.cuda.current_stream(eng.device).synchronize()   # `old` may go

    def _put_ids(self):
        slots = torch.from_numpy(self.planner.slots())
        K = self.planner.K
        self.engine.replay["obs_frames"].copy_(slots[:, :K])
        self.engine.replay["obs2_frames"].copy_(slots[:, K:])

    # ---- full-state checkpoint (SURVEY §8f rank 3) ---------------------------------------
    def state_dict(self, with_data: bool = True) -> dict:
        """ptr/size (+ the valid transitions, fetched from the device ring) for an exact resume.  Frame ring: the planner's
        state and the frames its rows refer to, in serial order, instead of obs / obs2 rows.  Coded frame ring: those
        frames' codes, and the coder's table."""
        self.flush()
        out = {"ptr": self.ptr, "size": self.size, "max_size": self.max_size}
        if self.planner is not None:
            out["frame_planner"] = self.planner.state_dict()
        if self.coder is not None:
            out["frame_coder"] = self.coder.state_dict()
        if with_data and self.engine is not None:
            torch.cuda.current_stream(self.engine.device).synchronize()
            if self.planner is None:
                out["data"] = {k: v[:self.size].cpu().clone() for k, v in self.engine.replay.items()}
            else:
                r = self.engine.replay
                src, _ = self.planner.moves(self.planner.frame_capacity)
                out["data"] = {k: r[k][:self.size].cpu().clone() for k in ("act", "rew", "done", "logp")}
                out["data"]["frames"] = r["frames"][torch.from_numpy(src).to(r["frames"].device)].cpu()
        return out

    def load_state_dict(self, state: dict) -> None:
        self._require_engine()
        if state["max_size"] != self.max_size:
            raise ValueError("replay capacity differs from the checkpoint")
        coder = state.get("frame_coder")
        if ("frame_planner" in state, None if coder is None else coder.get("code_bits", 8)) != \
                (self.planner is not None, self._code_bits()):
            raise ValueError("the checkpoint's replay ring kind (flat / frame / 8-bit or 16-bit coded frame ring) differs "
                             "from this buffer's")
        self.ptr, self.size, self._fill = int(state["ptr"]), int(state["size"]), 0
        if self.planner is not None:
            pl = self.planner
            pl.load_state_dict(state["frame_planner"])
            eng = self.engine
            if eng.replay["frames"].shape[0] != pl.frame_capacity:
                self._bind_frames(eng, pl.frame_capacity)
            self._nframes = 0
            self._put_ids()
            if self.coder is not None:
                self.coder.load_state_dict(state["frame_coder"])
                eng.replay["table"].copy_(torch.from_numpy(self.coder.table.copy()))
            if "data" in state:
                _, dst = pl.moves(pl.frame_capacity)
                eng.replay["frames"][torch.from_numpy(dst).to(eng.device)] = state["data"]["frames"].to(eng.device)
                for k in ("act", "rew", "done", "logp"):
                    eng.replay[k][:self.size].copy_(state["data"][k])
            return
        if "data" in state:
            for k, v in state["data"].items():
                self.engine.replay[k][:self.size].copy_(v)

    # ---- sample -----------------------------------------------------------------------
    def sample_indices(self, batch_size: int):
        if self.index_source == "numpy":
            return torch.from_numpy(np.random.randint(0, self.size, size=batch_size))
        return None

    def sample_batch(self, batch_size: int):
        """dict of DEVICE fp32 tensors (views of the engine's minibatch arena, valid until the next sample)."""
        self._require_engine()
        if self.size == 0:
            raise ValueError("cannot sample from an empty replay buffer")
        self.flush()
        return self.engine.replay_sample(batch_size, self.size, self.sample_indices(batch_size))
