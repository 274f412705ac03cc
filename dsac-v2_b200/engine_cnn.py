"""Python owner of one libdsact CNN handle (`dsact_cnn_*`, include/dsact.h): the DSAC-T update with the reference's CNN
approximators (BASELINE config 5; reference networks/cnn.py).  Same division of labour as `engine.Engine`: torch owns the
flat device buffers, every arithmetic step runs in the CUDA library; there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Sequence

import torch

from . import _lib
from ._lib import Batch, Buffers, CnnConfig, Layout, Noise, Replay, check
from .engine import STAT_KEYS


def make_cnn_config(obs_shape: Sequence[int], act_dim: int, kernels: Sequence[int], channels: Sequence[int],
                    strides: Sequence[int], hidden: Sequence[int], *, max_batch: int, act_hidden: str = "gelu", gamma=0.99,
                    tau=0.005, tau_b=None, delay_update=2, auto_alpha=True, alpha=0.2, lr_q=1e-4, lr_pi=1e-4, lr_alpha=3e-4,
                    min_log_std=-20.0, max_log_std=0.5, q_heads: int = 2, pi_std: str = "head",
                    act_dist: str = "TanhGaussDistribution", algo: str = "DSAC_V2", bound: bool = True,
                    td_bound: float = 20.0) -> CnnConfig:
    """`q_heads` / `pi_std` select the head wiring: (2, "head") = networks/cnn.py; with no conv layers and
    obs_shape = (obs_dim, 1, 1): (1, "head") = networks/mlp.py with policy std_type "mlp_separated", (1, "row") = "parameter"."""
    if len(kernels) > _lib.MAX_CONV or len(hidden) > _lib.MAX_HIDDEN:
        raise ValueError("too many layers")
    c = CnnConfig()
    c.abi_version = _lib.ABI_VERSION
    c.channels, c.height, c.width = (int(x) for x in obs_shape)
    c.act_dim, c.n_conv, c.n_hidden = int(act_dim), len(kernels), len(hidden)
    for j, (k, ch, st) in enumerate(zip(kernels, channels, strides)):
        c.conv_kernel[j], c.conv_channels[j], c.conv_stride[j] = int(k), int(ch), int(st)
    for j, v in enumerate(hidden):
        c.hidden[j] = int(v)
    c.act_hidden = _lib.ACTIVATIONS[act_hidden]
    c.max_batch, c.auto_alpha, c.delay_update = int(max_batch), int(bool(auto_alpha)), int(delay_update)
    c.gamma, c.tau, c.tau_b = float(gamma), float(tau), float(tau if tau_b is None else tau_b)
    c.alpha_fixed = float(alpha)
    c.lr_q, c.lr_pi, c.lr_alpha = float(lr_q), float(lr_pi), float(lr_alpha)
    c.min_log_std, c.max_log_std = float(min_log_std), float(max_log_std)
    c.adam_beta1, c.adam_beta2, c.adam_eps = 0.9, 0.999, 1e-8
    c.q_heads, c.pi_std = int(q_heads), {"head": 0, "row": 1, "shared": 2}[pi_std]
    c.algo, c.v1_bound, c.td_bound = {"DSAC_V2": 0, "DSAC_V1": 1}[algo], int(bool(bound)), float(td_bound)
    c.act_dist = _lib.ACT_DISTS[act_dist]
    return c


def make_heads_config(obs_dim: int, act_dim: int, hidden: Sequence[int], std_type: str, **kw) -> CnnConfig:
    """The MLP approximators on the head-wise fp32 engine: no encoder, one two-output head per critic, the policy with any
    of the reference's std types (networks/mlp.py:43-72).  DSAC-T with "mlp_shared" normally runs on `engine.Engine`
    (wgmma); this entry is for "mlp_separated" / "parameter" and for `algo="DSAC_V1"`."""
    return make_cnn_config((int(obs_dim), 1, 1), act_dim, (), (), (), hidden, q_heads=1,
                           pi_std={"mlp_separated": "head", "parameter": "row", "mlp_shared": "shared"}[std_type], **kw)


class CnnEngine:
    """One `dsact_cnn_handle` bound to flat torch-owned buffers on one CUDA device."""

    def __init__(self, cfg: CnnConfig, device, act_high, act_low, *, workspace_fill: float = 0.0):
        """`workspace_fill`: the value the scratch workspace holds when it is bound (see `engine.Engine`)."""
        if not torch.cuda.is_available():
            raise _lib.DsactError("the DSAC-T update engine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.lib, self.cfg = _lib.load(), cfg
        self.device = torch.device(device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        lay = Layout()
        check(self.lib.dsact_cnn_query_layout(C.byref(cfg), C.byref(lay)))
        self.layout = lay
        with torch.cuda.device(self.device):
            z = lambda n: torch.zeros(int(n), dtype=torch.float32, device=self.device)
            self.params, self.targets = z(lay.n_params), z(lay.n_targets)
            self.grads, self.adam_m, self.adam_v = z(lay.n_params), z(lay.n_params), z(lay.n_params)
            self.state = z(lay.state_floats)
            self.workspace = torch.full((int(lay.workspace_bytes) // 4 + 64,), float(workspace_fill), dtype=torch.float32,
                                        device=self.device)
            off = (-self.workspace.data_ptr() % 256) // 4
            self._ws_view = self.workspace[off:]
            self.act_high = torch.as_tensor(act_high, dtype=torch.float32).reshape(-1).to(self.device).clone()
            self.act_low = torch.as_tensor(act_low, dtype=torch.float32).reshape(-1).to(self.device).clone()
            h = C.c_void_p()
            check(self.lib.dsact_cnn_create(C.byref(cfg), self.device.index, C.byref(h)))
            self.h = h
            b = Buffers(self.params.data_ptr(), self.targets.data_ptr(), self.grads.data_ptr(), self.adam_m.data_ptr(),
                        self.adam_v.data_ptr(), self.act_high.data_ptr(), self.act_low.data_ptr(), self.state.data_ptr(),
                        self._ws_view.data_ptr())
            check(self.lib.dsact_cnn_bind(self.h, C.byref(b)))
            check(self.lib.dsact_cnn_set_carry(self.h, -1.0, -1.0, 0, 0, self._stream()))
            self._stats_host = torch.zeros(_lib.NUM_STATS, dtype=torch.float32).pin_memory()
        self.last_batch = 0
        self.dp_world = 0          # > 1 once dp_connect has mapped the peers

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def close(self):
        if getattr(self, "h", None):
            self.lib.dsact_cnn_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:   # noqa: BLE001
            pass

    # ---- flat layout in the reference's state_dict schema (include/dsact.h) --------------------------------------------
    def _schema(self):
        c = self.cfg
        out, off = [], 0
        shapes = []
        cin, hh, ww = c.channels, c.height, c.width
        for j in range(c.n_conv):
            k, co, st = c.conv_kernel[j], c.conv_channels[j], c.conv_stride[j]
            shapes.append((f"conv.{2 * j}", (co, cin, k, k), (co,)))
            cin, hh, ww = co, (hh - k) // st + 1, (ww - k) // st + 1
        feat = cin * hh * ww
        hidden = [c.hidden[j] for j in range(c.n_hidden)]

        def leaf(net, name, shape):
            nonlocal off
            n = 1
            for d in shape:
                n *= int(d)
            out.append((f"{net}.{name}", f"{net}_target.{name}", off, n, shape))
            off += n

        def mlp(net, head, sizes):
            for j in range(len(sizes) - 1):
                leaf(net, f"{head}.{2 * j}.weight", (sizes[j + 1], sizes[j]))
                leaf(net, f"{head}.{2 * j}.bias", (sizes[j + 1],))

        critics = ("q",) if c.algo == 1 else ("q1", "q2")   # dsac_v1.ApproxContainer holds ONE critic named `q`
        for net, extra, width in tuple((n, c.act_dim, 1) for n in critics) + (("policy", 0, c.act_dim),):
            for name, wshape, bshape in shapes:
                leaf(net, f"{name}.weight", wshape)
                leaf(net, f"{name}.bias", bshape)
            if net != "policy" and c.q_heads == 1:          # networks/mlp.py ActionValueDistri: self.q
                mlp(net, "q", [feat + extra] + hidden + [2])
            elif net == "policy" and c.pi_std == 2:         # networks/mlp.py std_type "mlp_shared": self.policy, 2A outputs
                mlp(net, "policy", [feat] + hidden + [2 * width])
            elif net == "policy" and c.pi_std == 1:         # the module's own parameter precedes its children's
                leaf(net, "log_std", (1, width))
                mlp(net, "mean", [feat] + hidden + [width])
            else:
                for head in ("mean", "log_std"):
                    mlp(net, head, [feat + extra] + hidden + [width])
        return out, off

    def load_weights(self, weights: dict):
        schema, n = self._schema()
        assert n == self.layout.n_targets, (n, self.layout.n_targets)
        with torch.no_grad():
            for key, tkey, off, cnt, shape in schema:
                self.params[off:off + cnt].copy_(torch.as_tensor(weights[key]).reshape(-1))
                self.targets[off:off + cnt].copy_(torch.as_tensor(weights.get(tkey, weights[key])).reshape(-1))
            self.params[n] = float(weights.get("log_alpha", 1.0))

    def export_weights(self, grads: bool = False) -> dict:
        schema, n = self._schema()
        src = (self.grads if grads else self.params).detach().cpu()
        tgt = self.targets.detach().cpu()
        out = {"log_alpha": src[n].clone()}
        for key, tkey, off, cnt, shape in schema:
            out[key] = src[off:off + cnt].view(shape).clone()
            if not grads:
                out[tkey] = tgt[off:off + cnt].view(shape).clone()
        return out

    # ---- the path -------------------------------------------------------------------------------------------------------
    def _args(self, data: Dict[str, torch.Tensor], noise):
        """ctypes batch / noise of a minibatch (image observations [B, C, H, W]); the device copies stay referenced until
        the next call, which is after the kernels reading them were enqueued."""
        t = {k: data[k].to(device=self.device, dtype=torch.float32).contiguous() for k in ("obs", "act", "rew", "obs2", "done")}
        B = t["obs"].shape[0]
        c = self.cfg
        if t["obs"][0].numel() != self.obs_elems or t["obs2"].shape != t["obs"].shape or t["act"].shape != (B, c.act_dim):
            raise ValueError("minibatch shapes do not match the configured observation / action shape")
        b = Batch(t["obs"].data_ptr(), t["act"].data_ptr(), t["rew"].data_ptr(), t["obs2"].data_ptr(), t["done"].data_ptr(), B, None)
        n = None
        if noise is not None:
            nz = [torch.as_tensor(x).to(device=self.device, dtype=torch.float32).contiguous() for x in noise]
            n = C.byref(Noise(*(x.data_ptr() for x in nz)))
            self._keep_noise = nz
        self._keep = t
        return b, n

    def step(self, data: Dict[str, torch.Tensor], iteration: int, noise=None):
        """DSAC_V2.local_update (reference dsac_v2.py:102-105) with image observations [B, C, H, W] on the device."""
        with torch.cuda.device(self.device):
            b, n = self._args(data, noise)
            check(self.lib.dsact_cnn_step(self.h, C.byref(b), n, int(iteration), self._stream()))
        self.last_batch = b.batch

    # ---- split form (get_remote_update_info / remote_update) and data parallelism: the signatures of engine.Engine ------
    def compute_grads(self, data, noise=None):
        with torch.cuda.device(self.device):
            b, n = self._args(data, noise)
            check(self.lib.dsact_cnn_compute_grads(self.h, C.byref(b), n, self._stream()))
        self.last_batch = b.batch

    def grad_phase1(self, data, noise=None):
        with torch.cuda.device(self.device):
            b, n = self._args(data, noise)
            check(self.lib.dsact_cnn_grad_phase1(self.h, C.byref(b), n, self._stream()))
        self.last_batch = b.batch

    def grad_phase2(self, global_batch: int):
        with torch.cuda.device(self.device):
            check(self.lib.dsact_cnn_grad_phase2(self.h, int(global_batch), self._stream()))

    def apply(self, iteration: int):
        with torch.cuda.device(self.device):
            check(self.lib.dsact_cnn_apply(self.h, int(iteration), self._stream()))

    def dp_export(self) -> bytes:
        """Allocate this rank's exchange buffer; its CUDA IPC handle (to be handed to every other rank)."""
        buf = C.create_string_buffer(_lib.IPC_HANDLE_BYTES)
        n = C.c_int64(0)
        with torch.cuda.device(self.device):
            check(self.lib.dsact_cnn_dp_export(self.h, buf, C.byref(n)))
        return buf.raw

    def dp_connect(self, rank: int, handles: Sequence[bytes]):
        """Map every rank's exchange buffer (`handles` in rank order, one per rank including this one)."""
        blob = b"".join(handles)
        if len(blob) != _lib.IPC_HANDLE_BYTES * len(handles):
            raise ValueError("malformed IPC handle list")
        with torch.cuda.device(self.device):
            check(self.lib.dsact_cnn_dp_connect(self.h, int(rank), len(handles), blob))
        self.dp_world = len(handles)

    def dp_step(self, data, iteration: int, global_batch: int, noise=None):
        """dsact_cnn_step on this rank's shard with the exchanges done in-kernel over peer memory."""
        with torch.cuda.device(self.device):
            b, n = self._args(data, noise)
            check(self.lib.dsact_cnn_dp_step(self.h, C.byref(b), n, int(global_batch), int(iteration), self._stream()))
        self.last_batch = b.batch

    # ---- device replay ring (flattened image rows) ---------------------------------------------------------------------
    @property
    def obs_elems(self) -> int:
        return self.cfg.channels * self.cfg.height * self.cfg.width

    def bind_replay(self, capacity: int):
        O, A = self.obs_elems, self.cfg.act_dim
        with torch.cuda.device(self.device):
            z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)
            self.replay = dict(obs=z(capacity, O), obs2=z(capacity, O), act=z(capacity, A), rew=z(capacity), done=z(capacity), logp=z(capacity))
            r = self.replay
            rb = Replay(r["obs"].data_ptr(), r["obs2"].data_ptr(), r["act"].data_ptr(), r["rew"].data_ptr(), r["done"].data_ptr(),
                        r["logp"].data_ptr(), int(capacity))
            check(self.lib.dsact_cnn_replay_bind(self.h, C.byref(rb)))
        self.capacity = int(capacity)

    def replay_add(self, staging: Dict[str, torch.Tensor], n: int, ptr: int):
        s = staging
        with torch.cuda.device(self.device):
            check(self.lib.dsact_cnn_replay_add(self.h, s["obs"].data_ptr(), s["obs2"].data_ptr(), s["act"].data_ptr(), s["rew"].data_ptr(),
                                                s["done"].data_ptr(), s["logp"].data_ptr(), int(n), int(ptr), self._stream()))

    def replay_sample(self, batch: int, size: int, idx: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        out = Batch()
        with torch.cuda.device(self.device):
            if idx is not None:
                idx = idx.to(device=self.device, dtype=torch.int64).contiguous()
                self._keep_idx = idx
            check(self.lib.dsact_cnn_replay_sample(self.h, int(batch), int(size), None if idx is None else idx.data_ptr(), C.byref(out),
                                                   self._stream()))
        base, c, B, A = self._ws_view.data_ptr(), self.cfg, int(batch), self.cfg.act_dim

        def view(ptr, n, shape):
            off = (ptr - base) // 4
            return self._ws_view[off:off + n].view(shape)

        img = (B, c.channels, c.height, c.width) if c.n_conv else (B, self.obs_elems)
        return {"obs": view(out.obs, B * self.obs_elems, img), "obs2": view(out.obs2, B * self.obs_elems, img),
                "act": view(out.act, B * A, (B, A)), "rew": view(out.rew, B, (B,)), "done": view(out.done, B, (B,)),
                "logp": view(out.logp, B, (B,))}

    def arena_views(self, batch: Optional[int] = None) -> Dict[str, torch.Tensor]:
        """Views of the arena slots the device generator writes, for the first `batch` rows (default max_batch): `idx`
        (int64 [B]) and `eps1`, `eps2` [B, A], `z3`, `z4` [B].  Offsets follow dsact_cnn_handle::layout
        (csrc/cnn_engine.cuh), counted back from the end of the workspace: the replay minibatch and its indices come last,
        and between them and the noise lie the critic outputs, the action gradients, the feature gradients and the two
        conv-backward buffers."""
        c, r64 = self.cfg, lambda n: (n + 63) // 64 * 64
        mb, A, O = c.max_batch, c.act_dim, self.obs_elems
        B = mb if batch is None else int(batch)
        cin, hh, ww, big = c.channels, c.height, c.width, 0
        for j in range(c.n_conv):
            k, st = c.conv_kernel[j], c.conv_stride[j]
            cin, hh, ww = c.conv_channels[j], (hh - k) // st + 1, (ww - k) // st + 1
            big = max(big, cin * hh * ww)
        F = cin * hh * ww
        end = int(self.layout.workspace_bytes) // 4
        idx = end - r64(2 * mb)
        r_obs = idx - 3 * r64(mb) - r64(mb * A) - 2 * r64(mb * O)
        z4 = r_obs - 2 * r64(mb * big) - 2 * r64(mb * (F + A)) - 3 * r64(mb * F) - 2 * r64(mb * A) - 12 * r64(2 * mb) - r64(mb)
        z3 = z4 - r64(mb)
        eps2 = z3 - r64(mb * A)
        eps1 = eps2 - r64(mb * A)
        v = self._ws_view
        return {"idx": v[idx:idx + 2 * B].view(torch.int64), "eps1": v[eps1:eps1 + B * A].view(B, A),
                "eps2": v[eps2:eps2 + B * A].view(B, A), "z3": v[z3:z3 + B], "z4": v[z4:z4 + B]}

    def set_carry(self, mean_std1=-1.0, mean_std2=-1.0, adam_steps_q=0, adam_steps_pi=0):
        """The state one update carries to the next besides weights and Adam moments: the mean_std EMA pair (-1 = not
        started; unused by DSAC_V1) and the Adam step counters of the critic and policy optimizers."""
        with torch.cuda.device(self.device):
            check(self.lib.dsact_cnn_set_carry(self.h, float(mean_std1), float(mean_std2), int(adam_steps_q),
                                               int(adam_steps_pi), self._stream()))

    def seed(self, seed: int):
        self._seed = int(seed) & (2 ** 64 - 1)
        check(self.lib.dsact_cnn_seed(self.h, self._seed))

    def read_stats_async(self, global_batch: Optional[int] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        out = self._stats_host if out is None else out
        with torch.cuda.device(self.device):
            check(self.lib.dsact_cnn_read_stats(self.h, int(global_batch or self.last_batch), out.data_ptr(), self._stream()))
        return out

    def read_stats(self, global_batch: Optional[int] = None) -> Dict[str, float]:
        with torch.cuda.device(self.device):
            check(self.lib.dsact_cnn_read_stats(self.h, int(global_batch or self.last_batch), self._stats_host.data_ptr(), self._stream()))
            torch.cuda.current_stream(self.device).synchronize()
        if float(self._stats_host[14]) != 0.0:   # include/dsact.h: slot 14 = 1 + rank of a peer that never arrived (dp_step)
            raise _lib.DsactError(f"data-parallel exchange timed out waiting for rank {int(self._stats_host[14]) - 1}")
        return dict(zip(STAT_KEYS, self._stats_host.tolist()))
