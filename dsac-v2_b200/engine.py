"""Python owner of one libdsact handle: allocates the flat device buffers with
torch (the library only borrows pointers), and exposes the update path.

This is plumbing around the C ABI (include/dsact.h); all arithmetic of the
path runs in the CUDA library.
"""
from __future__ import annotations

import ctypes as C
import weakref
from typing import Dict, Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import Batch, Buffers, Config, Layout, Noise, Replay, V1Options, check

STAT_KEYS = [
    "DSAC2/critic_avg_q1-RL iter",
    "DSAC2/critic_avg_q2-RL iter",
    "DSAC2/critic_avg_std1-RL iter",
    "DSAC2/critic_avg_std2-RL iter",
    "DSAC2/critic_avg_min_std1-RL iter",
    "DSAC2/critic_avg_min_std2-RL iter",
    "Loss/Actor loss-RL iter",
    "Loss/Critic loss-RL iter",
    "DSAC2/policy_mean-RL iter",
    "DSAC2/policy_std-RL iter",
    "DSAC2/entropy-RL iter",
    "DSAC2/alpha-RL iter",
    "DSAC2/mean_std1",
    "DSAC2/mean_std2",
]


def make_config(obs_dim: int, act_dim: int, hidden_q: Sequence[int], hidden_pi: Sequence[int], *, max_batch: int,
                act_q: str = "gelu", act_pi: str = "gelu", gamma=0.99, tau=0.005, tau_b=None, delay_update=2,
                auto_alpha=True, alpha=0.2, lr_q=1e-4, lr_pi=1e-4, lr_alpha=3e-4, min_log_std=-20.0,
                max_log_std=0.5, gemm_mode="fp32", use_graph=True, act_dist="TanhGaussDistribution",
                policy_std="mlp_shared") -> Config:
    """`policy_std`: the policy's std_type (networks/mlp.py:43-72), "mlp_shared", "mlp_separated" or "parameter"; the
    last two on DSAC-T handles only."""
    if len(hidden_q) > _lib.MAX_HIDDEN or len(hidden_pi) > _lib.MAX_HIDDEN:
        raise ValueError(f"at most {_lib.MAX_HIDDEN} hidden layers")
    for name in (act_q, act_pi):
        if name not in _lib.ACTIVATIONS:
            raise ValueError(f"unsupported activation {name!r}")
    c = Config()
    c.abi_version = _lib.ABI_VERSION
    c.obs_dim, c.act_dim = int(obs_dim), int(act_dim)
    c.n_hidden_q, c.n_hidden_pi = len(hidden_q), len(hidden_pi)
    for j, v in enumerate(hidden_q):
        c.hidden_q[j] = int(v)
    for j, v in enumerate(hidden_pi):
        c.hidden_pi[j] = int(v)
    c.act_q, c.act_pi = _lib.ACTIVATIONS[act_q], _lib.ACTIVATIONS[act_pi]
    c.max_batch = int(max_batch)
    c.auto_alpha, c.delay_update = int(bool(auto_alpha)), int(delay_update)
    c.gemm_mode, c.use_graph = _lib.GEMM_MODES[gemm_mode], int(bool(use_graph))
    c.act_dist = _lib.ACT_DISTS[act_dist]
    c.policy_std = _lib.POLICY_STDS[policy_std]
    c.gamma, c.tau = float(gamma), float(tau)
    c.tau_b = float(tau if tau_b is None else tau_b)
    c.alpha_fixed = float(alpha)
    c.lr_q, c.lr_pi, c.lr_alpha = float(lr_q), float(lr_pi), float(lr_alpha)
    c.min_log_std, c.max_log_std = float(min_log_std), float(max_log_std)
    c.adam_beta1, c.adam_beta2, c.adam_eps = 0.9, 0.999, 1e-8
    return c


def make_v1_options(bound: bool = True, td_bound: float = 20.0) -> V1Options:
    """DSAC_V1's settings (reference dsac_v1.py:79-80) for an MLP-engine handle: `bound` selects the bounded critic loss
    (else the Gaussian NLL), `td_bound` is `TD_bound`."""
    v = V1Options()
    v.abi_version, v.bound, v.td_bound = _lib.ABI_VERSION, int(bool(bound)), float(td_bound)
    return v


def query_layout(cfg: Config, v1: Optional[V1Options] = None) -> Layout:
    out = Layout()
    if v1 is None:
        check(_lib.load().dsact_query_layout(C.byref(cfg), C.byref(out)))
    else:
        check(_lib.load().dsact_v1_query_layout(C.byref(cfg), C.byref(v1), C.byref(out)))
    return out


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _f32c(t: torch.Tensor, device) -> torch.Tensor:
    if t.dtype != torch.float32 or t.device != device or not t.is_contiguous():
        t = t.to(device=device, dtype=torch.float32).contiguous()
    return t


class Engine:
    """One handle bound to flat torch-owned buffers on one CUDA device."""

    # the entry points that turn a configuration into its layout and a handle; every other call is shared by both engines
    _query, _create = "dsact_query_layout", "dsact_create"

    def __init__(self, cfg: Config, device: torch.device, act_high: torch.Tensor, act_low: torch.Tensor, *,
                 workspace_fill: float = 0.0, v1: Optional[V1Options] = None,
                 output_activations: Sequence[str] = ("linear", "linear")):
        """`workspace_fill`: the value the scratch workspace holds when it is bound.  No step depends on it: every region a
        step reads is written first by that step, or by dsact_bind (arena_views()["slabs"]).
        `v1` (`make_v1_options`): a DSAC_V1 handle of the MLP engine (dsact_v1_create): one critic, flat layout
        [q | policy | log_alpha], the reference's `dsac_v1.ApproxContainer` names.
        `output_activations`: (value, policy) names of `_lib.ACTIVATIONS`, the reference's value_output_activation /
        policy_output_activation: the activation of the critics' and the policy's last layer (with policy std_type
        "parameter" the learnable log_std row is not activated; dsact_set_output_activations in include/dsact.h)."""
        out_q, out_pi = output_activations
        for name in (out_q, out_pi):
            if name not in _lib.ACTIVATIONS:
                raise ValueError(f"unsupported output activation {name!r}")
        self.output_activations = (out_q, out_pi)
        if not torch.cuda.is_available():
            raise _lib.DsactError("the DSAC-T update engine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.lib = _lib.load()
        self.cfg = cfg
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.DsactError(f"engine device must be CUDA, got {self.device}")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.v1 = v1
        self.layout = L = Layout()
        if v1 is None:
            check(getattr(self.lib, self._query)(C.byref(cfg), C.byref(L)))
        else:
            check(self.lib.dsact_v1_query_layout(C.byref(cfg), C.byref(v1), C.byref(L)))
        with torch.cuda.device(self.device):
            z = lambda n: torch.zeros(int(n), dtype=torch.float32, device=self.device)
            self.params, self.targets = z(L.n_params), z(L.n_targets)
            self.grads, self.adam_m, self.adam_v = z(L.n_params), z(L.n_params), z(L.n_params)
            self.state = z(L.state_floats)
            self.workspace = torch.full((int(L.workspace_bytes) // 4 + 64,), float(workspace_fill), dtype=torch.float32,
                                        device=self.device)
            self.act_high = _f32c(torch.as_tensor(act_high).reshape(-1), self.device).clone()
            self.act_low = _f32c(torch.as_tensor(act_low).reshape(-1), self.device).clone()
            h = C.c_void_p()
            if v1 is None:
                check(getattr(self.lib, self._create)(C.byref(cfg), self.device.index, C.byref(h)))
            else:
                check(self.lib.dsact_v1_create(C.byref(cfg), C.byref(v1), self.device.index, C.byref(h)))
            self.h = h
            if self.output_activations != ("linear", "linear"):
                check(self.lib.dsact_set_output_activations(h, _lib.ACTIVATIONS[out_q], _lib.ACTIVATIONS[out_pi]))
            self._stats_host = torch.zeros(_lib.NUM_STATS, dtype=torch.float32).pin_memory()
            self._bind()
            check(self.lib.dsact_set_carry(self.h, -1.0, -1.0, 0, 0, self._stream()))
        self.replay = None
        self.last_batch = 0
        self.dp_world = 0          # > 1 once dp_connect has mapped the peers
        self._seed = 0x5DEECE66D   # the library's default (csrc/engine.cu)
        self._staged = False
        self._keep_host = [None, None]
        self._keep = None  # tensors referenced by the last enqueued call

    def _bind(self):
        ws = self.workspace
        off = (-ws.data_ptr() % 256) // 4  # 256-byte aligned view
        self._ws_view = ws[off:]
        b = Buffers(self.params.data_ptr(), self.targets.data_ptr(), self.grads.data_ptr(), self.adam_m.data_ptr(),
                    self.adam_v.data_ptr(), self.act_high.data_ptr(), self.act_low.data_ptr(), self.state.data_ptr(),
                    self._ws_view.data_ptr())
        check(self.lib.dsact_bind(self.h, C.byref(b)))

    def close(self):
        if getattr(self, "h", None):
            self.lib.dsact_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    # ---- argument marshalling ------------------------------------------------
    def _host_batch(self, data) -> Batch:
        """ctypes view of a HOST minibatch (contiguous fp32 CPU tensors; pinned ones copy at full PCIe rate)."""
        t = {}
        for k in ("obs", "act", "rew", "obs2", "done"):
            v = data[k]
            if v.dtype != torch.float32 or not v.is_contiguous():
                v = v.to(torch.float32).contiguous()
            t[k] = v
        B = t["obs"].shape[0]
        O, A = self.cfg.obs_dim, self.cfg.act_dim
        if B > self.cfg.max_batch:
            raise ValueError(f"batch {B} > max_batch {self.cfg.max_batch}")
        if t["obs"].shape != (B, O) or t["obs2"].shape != (B, O) or t["act"].shape != (B, A) \
                or t["rew"].numel() != B or t["done"].numel() != B:
            raise ValueError("minibatch shapes do not match the configured obs_dim/act_dim")
        # the async copies read these tensors after the call returns: keep the last two sets alive
        self._keep_host = (getattr(self, "_keep_host", None) or [None, None])[1:] + [t]
        return Batch(t["obs"].data_ptr(), t["act"].data_ptr(), t["rew"].data_ptr(), t["obs2"].data_ptr(),
                     t["done"].data_ptr(), B, None)

    def _stage_in(self, data) -> Batch:
        """Host minibatch -> one of the library's two device staging sets, copied on its private copy stream so that the
        H2D transfer of call k+1 overlaps the kernels of call k (`dsact_stage_host`, include/dsact.h)."""
        hb = self._host_batch(data)
        dev = Batch()
        check(self.lib.dsact_stage_host(self.h, C.byref(hb), C.byref(dev), self._stream()))
        self._staged = True
        return dev

    def _mark_staged_done(self):
        """The kernels reading the current staging set have been enqueued: the set may be refilled after them."""
        if getattr(self, "_staged", False):
            check(self.lib.dsact_stage_release(self.h, self._stream()))
            self._staged = False

    def _batch(self, data: Dict[str, torch.Tensor]) -> Batch:
        if data["obs"].device.type == "cpu":
            b = self._stage_in(data)
            self._keep = None
            return b
        t = {k: _f32c(data[k], self.device) for k in ("obs", "act", "rew", "obs2", "done")}
        B = t["obs"].shape[0]
        O, A = self.cfg.obs_dim, self.cfg.act_dim
        if t["obs"].shape != (B, O) or t["obs2"].shape != (B, O) or t["act"].shape != (B, A) \
                or t["rew"].numel() != B or t["done"].numel() != B:
            raise ValueError("minibatch shapes do not match the configured obs_dim/act_dim")
        self._keep = t
        return Batch(t["obs"].data_ptr(), t["act"].data_ptr(), t["rew"].data_ptr(), t["obs2"].data_ptr(),
                     t["done"].data_ptr(), B, None)

    def arena_views(self, batch: Optional[int] = None) -> Dict[str, torch.Tensor]:
        """Views of the arena slots the device generator writes, for the first `batch` rows (default max_batch): `idx`
        (int64 [B], the replay indices the last index-drawing gather recorded) and the noise `eps1`, `eps2` [B, A],
        `z3`, `z4` [B] (device noise, or host noise staged there); and `slabs`, the one region dsact_bind initialises
        (empty in fp32 mode and on the head-wise engine).  Offsets are the ones the library reports (dsact_layout)."""
        L, A, v = self.layout, self.cfg.act_dim, self._ws_view
        B = int(L.max_batch) if batch is None else int(batch)
        return {"idx": v[L.off_idx:L.off_idx + 2 * B].view(torch.int64),
                "eps1": v[L.off_eps1:L.off_eps1 + B * A].view(B, A), "eps2": v[L.off_eps2:L.off_eps2 + B * A].view(B, A),
                "z3": v[L.off_z3:L.off_z3 + B], "z4": v[L.off_z4:L.off_z4 + B],
                "slabs": v[L.off_slabs:L.off_slabs + L.slab_floats]}

    def _noise_slots(self, B):
        v = self.arena_views(B)
        return [v[k] for k in ("eps1", "eps2", "z3", "z4")]

    def _noise(self, noise, B):
        if noise is None:
            return None, None
        noise = [torch.as_tensor(x) for x in noise]
        if all(x.device.type == "cpu" for x in noise):  # stage into the arena's noise slots: stable pointers
            slots = self._noise_slots(B)
            for dst, src in zip(slots, noise):
                dst.copy_(src.reshape(dst.shape), non_blocking=True)
            noise = slots
        eps1, eps2, z3, z4 = (_f32c(x, self.device) for x in noise)
        A = self.cfg.act_dim
        if eps1.shape != (B, A) or eps2.shape != (B, A) or z3.numel() != B or z4.numel() != B:
            raise ValueError("noise shapes must be eps1/eps2 [B,A], z3/z4 [B]")
        keep = (eps1, eps2, z3, z4)
        return C.byref(Noise(eps1.data_ptr(), eps2.data_ptr(), z3.data_ptr(), z4.data_ptr())), keep

    def _update(self, fn: str, data=None, noise=None, *, replay=None, args=(), out=None, host_fn=None, release=True):
        """One update call `fn` of the C ABI: its rows (the minibatch `data`, or with `replay` = (batch, size, idx) the
        replay gather's), `noise`, the other arguments `args`, the stream, then `out` if given.  `host_fn`: the entry point
        that takes a host minibatch itself (`data` on the CPU).  `release`: no later call reads a staged host minibatch."""
        with torch.cuda.device(self.device):
            if replay is not None:
                B, size, idx = replay
                if idx is not None:
                    idx = idx.to(device=self.device, dtype=torch.int64).contiguous()
                    self._keep_idx = idx
                rows = (int(B), int(size), _ptr(idx))
            else:
                if host_fn is not None and data["obs"].device.type == "cpu":
                    b, fn = self._host_batch(data), host_fn
                else:
                    b = self._batch(data)
                B, rows = b.batch, (C.byref(b),)
            n, self._keep_noise = self._noise(noise, int(B))
            check(getattr(self.lib, fn)(self.h, *rows, n, *args, self._stream(), *(() if out is None else (out,))))
            if release:
                self._mark_staged_done()
        self.last_batch = int(B)

    # ---- the path ---------------------------------------------------------------
    # the step on a host minibatch in one C call (None: the minibatch goes through _batch)
    _step_host = "dsact_step_host"

    def step(self, data, iteration: int, noise=None):
        """DSAC_V2.local_update (reference dsac_v2.py:102-105), or DSAC_V1's, on a host or device minibatch."""
        self._update("dsact_step", data, noise, args=(int(iteration),), host_fn=self._step_host)

    def profile_step(self, data, iteration: int, noise=None) -> dict:
        """One eager step with per-launch CUDA events (bench.py's roofline leg)."""
        out = _lib.Profile()
        self._update("dsact_profile_step", data, noise, args=(int(iteration),), out=C.byref(out))
        names = ("other", "gemm_fwd", "gemm_dgrad", "gemm_wgrad")
        return {"total_ms": out.total_ms,
                **{k: {"ms": out.ms[i], "flops": out.flops[i], "launches": out.launches[i]} for i, k in enumerate(names)}}

    def compute_grads(self, data, noise=None):
        self._update("dsact_compute_grads", data, noise)

    def grad_phase1(self, data, noise=None):
        self._update("dsact_grad_phase1", data, noise, release=False)   # grad_phase2 reads the rows as well

    def grad_phase2(self, global_batch: int):
        with torch.cuda.device(self.device):
            check(self.lib.dsact_grad_phase2(self.h, int(global_batch), self._stream()))
            self._mark_staged_done()

    def apply(self, iteration: int):
        with torch.cuda.device(self.device):
            check(self.lib.dsact_apply(self.h, int(iteration), self._stream()))

    def read_stats_async(self, global_batch: Optional[int] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Enqueue finalisation + D2H of the 16 tb_info floats; caller synchronises before reading."""
        out = self._stats_host if out is None else out
        with torch.cuda.device(self.device):
            check(self.lib.dsact_read_stats(self.h, int(global_batch or self.last_batch), out.data_ptr(), self._stream()))
        return out

    def read_stats(self, global_batch: Optional[int] = None) -> Dict[str, float]:
        out = self.read_stats_async(global_batch)
        torch.cuda.current_stream(self.device).synchronize()
        if float(out[14]) != 0.0:   # include/dsact.h: slot 14 = 1 + rank of a peer that never arrived (dsact_dp_step)
            raise _lib.DsactError(f"data-parallel exchange timed out waiting for rank {int(out[14]) - 1}")
        return {k: float(out[i]) for i, k in enumerate(STAT_KEYS)}

    def set_carry(self, mean_std1=-1.0, mean_std2=-1.0, adam_steps_q=0, adam_steps_pi=0):
        """The state one update carries to the next besides weights and Adam moments: the mean_std EMA pair (-1 = not
        started; unused by DSAC_V1) and the Adam step counters of the critic and policy optimizers."""
        with torch.cuda.device(self.device):
            check(self.lib.dsact_set_carry(self.h, float(mean_std1), float(mean_std2), int(adam_steps_q),
                                           int(adam_steps_pi), self._stream()))

    def seed(self, seed: int):
        self._seed = int(seed) & (2 ** 64 - 1)
        check(self.lib.dsact_seed(self.h, self._seed))

    # ---- replay ring buffer -------------------------------------------------------
    @property
    def obs_elems(self) -> int:
        """Floats of one observation (a replay row of obs / obs2)."""
        return self.cfg.obs_dim

    def bind_replay(self, capacity: int):
        O, A = self.obs_elems, self.cfg.act_dim
        with torch.cuda.device(self.device):
            z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)
            self.replay = dict(obs=z(capacity, O), obs2=z(capacity, O), act=z(capacity, A), rew=z(capacity),
                               done=z(capacity), logp=z(capacity))
            r = self.replay
            rb = Replay(r["obs"].data_ptr(), r["obs2"].data_ptr(), r["act"].data_ptr(), r["rew"].data_ptr(),
                        r["done"].data_ptr(), r["logp"].data_ptr(), int(capacity))
            check(self.lib.dsact_replay_bind(self.h, C.byref(rb)))
        self.capacity = int(capacity)

    def bind_replay_frames(self, capacity: int, frame_capacity: int, frames_per_obs: int, coded: bool = False,
                           code_bits: int = 8):
        """Bind a frame ring (dsact_replay_bind_frames): `capacity` rows whose obs / obs2 are `frames_per_obs` (K) frame
        ids each into a store of `frame_capacity` frames of obs_elems / K floats.  `replay` then holds `frames`,
        `obs_frames`, `obs2_frames` (int32 [capacity, K]), `act`, `rew`, `done`, `logp`.
        coded: a coded frame ring, `frames` holding codes of `code_bits` bits and `table` (2^code_bits floats, zeros until
        an add fills them) their values.  code_bits 8 (dsact_replay_bind_coded_frames): uint8 codes; 16
        (dsact_replay_bind_coded16_frames): uint16 codes, held in an int16 tensor."""
        O, A, K = self.obs_elems, self.cfg.act_dim, int(frames_per_obs)
        capacity, frame_capacity = int(capacity), int(frame_capacity)
        if not 1 <= K <= 64 or O % K:
            raise ValueError(f"frames_per_obs {K} must be in [1, 64] and divide the observation's {O} floats")
        if not K <= frame_capacity <= 2 ** 31 - 1 or capacity < 1:
            raise ValueError(f"frame_capacity {frame_capacity} outside [{K}, 2^31 - 1] or capacity {capacity} < 1")
        if coded and code_bits not in (8, 16):
            raise ValueError(f"code_bits {code_bits!r}: the coded frame rings take 8- or 16-bit codes")
        with torch.cuda.device(self.device):
            z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)
            ids = lambda: torch.zeros(capacity, K, dtype=torch.int32, device=self.device)
            frames = (torch.zeros(frame_capacity, O // K, dtype=torch.uint8 if code_bits == 8 else torch.int16,
                                  device=self.device) if coded else z(frame_capacity, O // K))
            self.replay = dict(frames=frames, obs_frames=ids(), obs2_frames=ids(), act=z(capacity, A),
                               rew=z(capacity), done=z(capacity), logp=z(capacity))
            if coded:
                self.replay["table"] = z(1 << code_bits)
            r = self.replay
            rb = _lib.FrameReplay(*(r[k].data_ptr() for k in ("frames", "obs_frames", "obs2_frames", "act", "rew", "done",
                                                              "logp")), capacity, frame_capacity, K)
            if coded:
                bind = self.lib.dsact_replay_bind_coded_frames if code_bits == 8 else self.lib.dsact_replay_bind_coded16_frames
                check(bind(self.h, C.byref(rb), r["table"].data_ptr()))
            else:
                check(self.lib.dsact_replay_bind_frames(self.h, C.byref(rb)))
        self.capacity = capacity

    def bind_replay_coded_frames(self, capacity: int, frame_capacity: int, frames_per_obs: int):
        """Bind a coded frame ring (dsact_replay_bind_coded_frames): bind_replay_frames with uint8 codes for frames."""
        self.bind_replay_frames(capacity, frame_capacity, frames_per_obs, coded=True)

    def replay_add_coded_frames(self, codes: Optional[torch.Tensor], n_frames: int, frame_ptr: int, table: np.ndarray,
                                n_codes: int, rows: Dict[str, torch.Tensor], n: int, ptr: int):
        """dsact_replay_add_coded_frames: `n_frames` frames of codes (contiguous uint8 HOST tensor) -> frame slots
        (frame_ptr + i) % frame_capacity, table[:n_codes] (float32, host) -> the device table; the rows as in
        replay_add_frames."""
        self._add_coded(self.lib.dsact_replay_add_coded_frames, (torch.uint8,), codes, n_frames, frame_ptr, table, n_codes,
                        rows, n, ptr)

    def replay_add_coded16_frames(self, codes: Optional[torch.Tensor], n_frames: int, frame_ptr: int, table: np.ndarray,
                                  n_codes: int, rows: Dict[str, torch.Tensor], n: int, ptr: int):
        """dsact_replay_add_coded16_frames: replay_add_coded_frames with 16-bit codes (a contiguous int16 or uint16 HOST
        tensor holding the uint16 codes) and up to 65 536 table entries."""
        self._add_coded(self.lib.dsact_replay_add_coded16_frames, (torch.int16, torch.uint16), codes, n_frames, frame_ptr,
                        table, n_codes, rows, n, ptr)

    def _add_coded(self, fn, code_dtypes, codes, n_frames, frame_ptr, table, n_codes, rows, n, ptr):
        r = rows
        for k, dts, t in (("codes", code_dtypes, codes), ("obs_frames", (torch.int32,), r["obs_frames"]),
                          ("obs2_frames", (torch.int32,), r["obs2_frames"])):
            if t is not None and (t.device.type != "cpu" or t.dtype not in dts or not t.is_contiguous()):
                raise ValueError(f"{k} must be a contiguous {' or '.join(map(str, dts))} host tensor")
        table = np.ascontiguousarray(table, np.float32)
        with torch.cuda.device(self.device):
            check(fn(self.h, _ptr(codes), int(n_frames), int(frame_ptr), table.ctypes.data, int(n_codes),
                     r["obs_frames"].data_ptr(), r["obs2_frames"].data_ptr(), r["act"].data_ptr(), r["rew"].data_ptr(),
                     r["done"].data_ptr(), r["logp"].data_ptr(), int(n), int(ptr), self._stream()))

    def replay_add_frames(self, frames: Optional[torch.Tensor], n_frames: int, frame_ptr: int, rows: Dict[str, torch.Tensor],
                          n: int, ptr: int):
        """dsact_replay_add_frames: `n_frames` frames (contiguous fp32, host or device) -> frame slots
        (frame_ptr + i) % frame_capacity; rows' `obs_frames` / `obs2_frames` (contiguous int32 HOST tensors [n, K]) and
        `act`, `rew`, `done`, `logp` (host or device) -> rows (ptr + i) % capacity."""
        r = rows
        for k in ("obs_frames", "obs2_frames"):
            if r[k].device.type != "cpu" or r[k].dtype != torch.int32 or not r[k].is_contiguous():
                raise ValueError(f"{k} must be a contiguous int32 host tensor")
        with torch.cuda.device(self.device):
            check(self.lib.dsact_replay_add_frames(self.h, _ptr(frames), int(n_frames), int(frame_ptr),
                                                   r["obs_frames"].data_ptr(), r["obs2_frames"].data_ptr(),
                                                   r["act"].data_ptr(), r["rew"].data_ptr(), r["done"].data_ptr(),
                                                   r["logp"].data_ptr(), int(n), int(ptr), self._stream()))

    def replay_add(self, staging: Dict[str, torch.Tensor], n: int, ptr: int):
        """Rows of contiguous fp32 staging tensors (pinned host or device) -> ring rows (ptr+i) % capacity."""
        s = staging
        with torch.cuda.device(self.device):
            check(self.lib.dsact_replay_add(self.h, s["obs"].data_ptr(), s["obs2"].data_ptr(), s["act"].data_ptr(),
                                            s["rew"].data_ptr(), s["done"].data_ptr(), s["logp"].data_ptr(),
                                            int(n), int(ptr), self._stream()))

    def arena_batch(self, b: Batch) -> Dict[str, torch.Tensor]:
        """Torch views of the engine's gathered-minibatch arena (no copies)."""
        O, A, B = self.obs_elems, self.cfg.act_dim, b.batch
        base = self._ws_view.data_ptr()

        def view(ptr, n, shape):
            off = (ptr - base) // 4
            return self._ws_view[off:off + n].view(shape)

        return {"obs": view(b.obs, B * O, (B, O)), "act": view(b.act, B * A, (B, A)), "rew": view(b.rew, B, (B,)),
                "obs2": view(b.obs2, B * O, (B, O)), "done": view(b.done, B, (B,)), "logp": view(b.logp, B, (B,))}

    def replay_sample(self, batch: int, size: int, idx: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        out = Batch()
        with torch.cuda.device(self.device):
            if idx is not None:
                idx = idx.to(device=self.device, dtype=torch.int64).contiguous()
                self._keep_idx = idx
            check(self.lib.dsact_replay_sample(self.h, int(batch), int(size), _ptr(idx), C.byref(out), self._stream()))
        return self.arena_batch(out)

    def replay_step(self, batch: int, size: int, iteration: int, idx: Optional[torch.Tensor] = None, noise=None):
        self._update("dsact_replay_step", noise=noise, replay=(batch, size, idx), args=(int(iteration),))

    def _steps_buffer(self, name: str, src: torch.Tensor, dtype) -> torch.Tensor:
        """`src` as a contiguous device tensor.  Host data is staged into a buffer kept per name and shape, so that a
        repeated call hands the library the same pointers (they are part of the captured graph's key)."""
        if src.device == self.device and src.dtype == dtype and src.is_contiguous():
            return src
        if src.device.type != "cpu":
            return src.to(device=self.device, dtype=dtype).contiguous()
        bufs = self.__dict__.setdefault("_steps_bufs", {})
        key = (name, tuple(src.shape))
        if key not in bufs:
            bufs[key] = torch.empty(src.shape, dtype=dtype, device=self.device)
        buf = bufs[key]
        buf.copy_(src.to(dtype).contiguous(), non_blocking=True)
        return buf

    def replay_steps(self, n: int, batch: int, size: int, iteration: int, idx: Optional[torch.Tensor] = None, noise=None,
                     stats: bool = True) -> Optional[torch.Tensor]:
        """n replay_step calls in one submission (dsact_replay_steps): updates for iterations iteration .. iteration+n-1.
        `idx`: None (device draws) or int64 [n, batch]; `noise`: None or (eps1, eps2 [n, batch, A], z3, z4 [n, batch]).
        Returns the [n, 16] device tensor of per-update tb_info rows (valid until the next call with the same n), or None
        with stats=False."""
        return self._replay_steps("dsact_replay_steps", n, batch, size, iteration, idx, noise, stats)

    def _replay_steps(self, fn: str, n: int, batch: int, size: int, iteration: int, idx, noise, stats: bool, dp_args=()):
        """replay_steps through entry point `fn`, whose `dp_args` follow the noise."""
        n, B, A = int(n), int(batch), self.cfg.act_dim
        with torch.cuda.device(self.device):
            if idx is not None:
                idx = self._steps_buffer("idx", torch.as_tensor(idx), torch.int64)
                if idx.shape != (n, B):
                    raise ValueError(f"idx must be [n, batch] = [{n}, {B}], got {tuple(idx.shape)}")
            nz = None
            if noise is not None:
                shapes = ((n, B, A), (n, B, A), (n, B), (n, B))
                ts = [self._steps_buffer(k, torch.as_tensor(x).reshape(s), torch.float32)
                      for k, x, s in zip(("eps1", "eps2", "z3", "z4"), noise, shapes)]
                nz = C.byref(Noise(*(t.data_ptr() for t in ts)))
                self._keep_noise = ts
            out = None
            if stats:
                outs = self.__dict__.setdefault("_steps_stats", {})
                if n not in outs:
                    outs[n] = torch.zeros(n, _lib.NUM_STATS, dtype=torch.float32, device=self.device)
                out = outs[n]
            self._keep_idx = idx
            check(getattr(self.lib, fn)(self.h, n, B, int(size), _ptr(idx), nz, *dp_args, _ptr(out), int(iteration),
                                        self._stream()))
        self.last_batch = B
        return out

    # ---- data-parallel replicas over NVLink peer memory (include/dsact.h) ---------------------
    def dp_export(self) -> bytes:
        """Allocate this rank's exchange buffer; its CUDA IPC handle (to be handed to every other rank)."""
        buf = C.create_string_buffer(_lib.IPC_HANDLE_BYTES)
        n = C.c_int64(0)
        with torch.cuda.device(self.device):
            check(self.lib.dsact_dp_export(self.h, buf, C.byref(n)))
        return buf.raw

    def dp_connect(self, rank: int, handles: Sequence[bytes]):
        """Map every rank's exchange buffer (`handles` in rank order, one per rank including this one)."""
        blob = b"".join(handles)
        if len(blob) != _lib.IPC_HANDLE_BYTES * len(handles):
            raise ValueError("malformed IPC handle list")
        with torch.cuda.device(self.device):
            check(self.lib.dsact_dp_connect(self.h, int(rank), len(handles), blob))
        self.dp_world = len(handles)

    def dp_step(self, data, iteration: int, global_batch: int, noise=None):
        """dsact_step on this rank's shard with the exchanges done in-kernel over peer memory."""
        self._update("dsact_dp_step", data, noise, args=(int(global_batch), int(iteration)))

    def dp_replay_step(self, batch: int, size: int, iteration: int, global_batch: int, idx: Optional[torch.Tensor] = None,
                       noise=None):
        self._update("dsact_dp_replay_step", noise=noise, replay=(batch, size, idx), args=(int(global_batch), int(iteration)))

    def dp_replay_steps(self, n: int, batch: int, size: int, iteration: int, global_batch: int,
                        idx: Optional[torch.Tensor] = None, noise=None, stats: bool = True) -> Optional[torch.Tensor]:
        """n dp_replay_step calls in one submission (dsact_dp_replay_steps): replay_steps with every update's exchanges
        over the peers, over `global_batch` rows.  The same `idx` / `noise` layouts, staging buffers and [n, 16] return
        as replay_steps; row k's statistics are over `global_batch` rows, slot 14 the peer-timeout flag."""
        return self._replay_steps("dsact_dp_replay_steps", n, batch, size, iteration, idx, noise, stats,
                                  dp_args=(int(global_batch),))

    # ---- weights in the reference's state_dict schema -----------------------------------
    def _schema(self):
        """[(key, flat name, offset, shape)] for every tensor of the flat layout (include/dsact.h).  DSAC_V1 handles walk
        the one critic `q` (dsac_v1.ApproxContainer) instead of `q1`, `q2`.  The policy span follows `policy_std`
        (DSACT_STD_*): `policy.policy.*`, or `policy.mean.*` then `policy.log_std.*`, or the row `policy.log_std` then
        `policy.mean.*`."""
        c = self.cfg
        q_sizes = [c.obs_dim + c.act_dim] + [c.hidden_q[j] for j in range(c.n_hidden_q)] + [2]
        pi_in = [c.obs_dim] + [c.hidden_pi[j] for j in range(c.n_hidden_pi)]
        out, off = [], 0

        def leaf(net, name, shape):
            nonlocal off
            n = 1
            for d in shape:
                n *= d
            out.append((f"{net}.{name}", f"{net}_target.{name}", off, n, shape))
            off += n

        def mlp(net, inner, sizes):
            for j in range(len(sizes) - 1):
                leaf(net, f"{inner}.{2 * j}.weight", (sizes[j + 1], sizes[j]))
                leaf(net, f"{inner}.{2 * j}.bias", (sizes[j + 1],))

        for net in ("q",) if getattr(self, "v1", None) is not None else ("q1", "q2"):
            mlp(net, "q", q_sizes)
        if c.policy_std == _lib.POLICY_STDS["mlp_separated"]:
            mlp("policy", "mean", pi_in + [c.act_dim])
            mlp("policy", "log_std", pi_in + [c.act_dim])
        elif c.policy_std == _lib.POLICY_STDS["parameter"]:
            leaf("policy", "log_std", (1, c.act_dim))
            mlp("policy", "mean", pi_in + [c.act_dim])
        else:
            mlp("policy", "policy", pi_in + [2 * c.act_dim])
        return out, off

    def load_weights(self, weights: dict):
        """Fill params/targets from a dict keyed like the reference's state_dict."""
        schema, n = self._schema()
        assert n == self.layout.n_targets, (n, self.layout.n_targets)
        with torch.no_grad():
            for key, tkey, off, cnt, shape in schema:
                self.params[off:off + cnt].copy_(torch.as_tensor(weights[key]).reshape(-1))
                self.targets[off:off + cnt].copy_(torch.as_tensor(weights.get(tkey, weights[key])).reshape(-1))
            self.params[n] = float(weights.get("log_alpha", 1.0))

    def export_weights(self, grads: bool = False) -> dict:
        schema, n = self._schema()
        src = self.grads if grads else self.params
        host, thost = src.detach().cpu(), self.targets.detach().cpu()
        out = {"log_alpha": host[n].clone()}
        for key, tkey, off, cnt, shape in schema:
            out[key] = host[off:off + cnt].view(shape).clone()
            if not grads:
                out[tkey] = thost[off:off + cnt].view(shape).clone()
        return out

    # ---- test hooks ----------------------------------------------------------------
    def launch_count(self) -> int:
        return int(self.lib.dsact_launch_count(self.h))

    def last_call_launches(self) -> int:
        return int(self.lib.dsact_last_call_launches(self.h))

    def test_gemm(self, variant: int, A: torch.Tensor, B: torch.Tensor, bias: Optional[torch.Tensor], C_out: torch.Tensor,
                  M: int, N: int, K: int):
        """One plain problem (store epilogue) of `test_layers`."""
        self.test_layers(variant, [dict(M=M, N=N, K0=K, A0=A, B=B, bias=bias, C=C_out)])

    def test_layers(self, variant: int, probs, max_ctas: int = 0):
        """dsact_test_gemm: one group of problems, each a dict of dsact_test_layer fields with tensors for the pointers
        (leading dimensions default to the tensors' row strides; `img` is a [2, M, pitch] bf16 tensor)."""
        arr = (_lib.TestLayer * len(probs))()
        for t, p in zip(arr, probs):
            for k, v in p.items():
                if k == "img":
                    t.img, t.img_pitch, t.img_plane = v.data_ptr(), v.stride(1), v.stride(0)
                elif isinstance(v, torch.Tensor):
                    setattr(t, k, v.data_ptr())
                    ld = {"A0": "lda0", "A1": "lda1", "B": "ldb", "Zin": "ldz", "C": "ldc"}.get(k)
                    if ld and ld not in p:
                        setattr(t, ld, v.stride(0))
                elif v is not None:
                    setattr(t, k, v)
        with torch.cuda.device(self.device):
            check(self.lib.dsact_test_gemm(self.h, variant, arr, len(probs), max_ctas, self._stream()))

    def test_chain(self, dgrad: bool, sizes, K0: int, K1: int, kB1: int, act: int, params: torch.Tensor, passes,
                   tiling: Optional[int] = None):
        """dsact_test_chain: one launch of the layer-chain kernel; `passes` are dicts of dsact_test_chain_pass fields
        (Zout / Zin / img / colsum: lists per hidden layer, entries may be None; `img` entries [2, M, pitch] bf16).
        `tiling` (dsact_test_chain_tiling): 0 = the column-split kernel, 1 = the ping-pong kernel, None = by shape."""
        arr = (_lib.TestChainPass * len(passes))()
        for t, p in zip(arr, passes):
            t.M = p["M"]
            for k in ("x0", "x1", "out"):
                setattr(t, k, _ptr(p.get(k)))
            t.out_ld = int(p.get("out_ld", 0))
            for k in ("Zout", "Zin", "img", "colsum"):
                for j, v in enumerate(p.get(k) or []):
                    getattr(t, k)[j] = _ptr(v)
        sz = (C.c_int32 * len(sizes))(*sizes)
        with torch.cuda.device(self.device):
            if tiling is None:
                check(self.lib.dsact_test_chain(self.h, int(dgrad), len(sizes) - 2, sz, K0, K1, kB1, act, params.data_ptr(),
                                                arr, len(passes), self._stream()))
            else:
                check(self.lib.dsact_test_chain_tiling(self.h, int(tiling), int(dgrad), len(sizes) - 2, sz, K0, K1, kB1, act,
                                                       params.data_ptr(), arr, len(passes), self._stream()))

    def test_rows(self, kernel: str, batch: int, global_batch: Optional[int] = None, max_blocks: int = 0,
                  advance_rng: bool = False, **arrays):
        """dsact_test_rows: one step kernel ("sample", "loss", "policy_grad", "stats") on caller tensors.  `arrays` are
        dsact_test_row_io fields: a tensor, None, or for the array fields a list of them (images [2, batch, pitch] bf16)."""
        t = _lib.TestRowIo()
        t.kernel, t.batch = _lib.TEST_KERNELS[kernel], int(batch)
        t.global_batch = int(batch if global_batch is None else global_batch)
        t.max_blocks, t.advance_rng = int(max_blocks), int(bool(advance_rng))
        for k, v in arrays.items():
            if isinstance(v, (list, tuple)):
                for i, x in enumerate(v):
                    getattr(t, k)[i] = _ptr(x)
            else:
                setattr(t, k, v if isinstance(v, int) else _ptr(v))
        with torch.cuda.device(self.device):
            check(self.lib.dsact_test_rows(self.h, C.byref(t), self._stream()))

    def test_apply(self, part: int = 0, fold_slabs: int = 0, scalars_ready: int = 0, tail_rows: int = 0,
                   global_batch: int = 1, max_blocks: int = 0):
        """dsact_test_apply: one Adam / Polyak launch on the bound buffers, built as a single-call step builds it."""
        with torch.cuda.device(self.device):
            check(self.lib.dsact_test_apply(self.h, int(part), int(fold_slabs), int(scalars_ready), int(tail_rows),
                                            int(global_batch), int(max_blocks), self._stream()))

    def test_dp_attach(self, rank: int, peers: Sequence["Engine"]) -> torch.Tensor:
        """dsact_test_dp_attach: make this handle rank `rank` of `peers` (engines of this process and device, in rank order,
        each exported with dp_export).  Returns a float32 view of this rank's whole exchange buffer (header, gradient
        block, reduced block; csrc/dp_peer.cuh)."""
        arr = (C.c_void_p * len(peers))(*(p.h.value for p in peers))
        buf, n = C.c_void_p(), C.c_int64()
        with torch.cuda.device(self.device):
            check(self.lib.dsact_test_dp_attach(self.h, int(rank), len(peers), arr, C.byref(buf), C.byref(n)))
        self.dp_world = len(peers)
        # weak references: the peers hold this engine too, and a reference cycle would leave a closed world's handles to
        # the cyclic garbage collector, whose dsact_destroy (cudaFree synchronises the device) can then run in the middle
        # of another world's rank enqueues while their kernels wait on each other
        self._dp_peers = [weakref.proxy(p) for p in peers]
        return _device_view(buf.value, int(n.value), self.device)   # the library owns it: valid while this handle lives

    def test_dp(self, op: str, kind: int = 0, grads: Optional[torch.Tensor] = None, slabs: Optional[torch.Tensor] = None,
                nslabs: int = 0, slab_stride: int = 0, n: int = 0, tail_rows: int = 0, global_batch: int = 1):
        """dsact_test_dp: one exchange operation ("exchange", "fold", "reduce_scatter", "apply") on an attached handle.
        "exchange" runs every rank of the world attached with test_dp_attach."""
        t = _lib.TestDpIo()
        t.kind, t.grads, t.slabs, t.nslabs = int(kind), _ptr(grads), _ptr(slabs), int(nslabs)
        t.slab_stride, t.n, t.tail_rows, t.global_batch = int(slab_stride), int(n), int(tail_rows), int(global_batch)
        ranks = (C.c_void_p * len(self._dp_peers))(*(p.h.value for p in self._dp_peers))
        t.ranks = C.cast(ranks, C.POINTER(C.c_void_p))
        with torch.cuda.device(self.device):
            check(self.lib.dsact_test_dp(self.h, _lib.TEST_DP_OPS[op], C.byref(t), self._stream()))


def _device_view(ptr: int, n: int, device: torch.device) -> torch.Tensor:
    """A float32 tensor over n floats of device memory at `ptr` that torch does not own (through
    __cuda_array_interface__, no copy)."""
    class _Mem:
        __cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 3, "strides": None}
    with torch.cuda.device(device):
        return torch.as_tensor(_Mem(), device=device)
