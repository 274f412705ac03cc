"""CPU checks of the data-parallel n-update call: `dsact_dp_replay_steps` is declared as include/dsact.h declares it and
refuses a null handle; `DSAC_V2.replay_updates` under torch.distributed makes one `Engine.dp_replay_steps` call with the
peer transport and takes the n rounds with the "nccl" transport, when the peers cannot be mapped, and on the head-wise
engine; the lazy statistics rows surface a peer timeout.  Fake engines, buffers and process groups: no GPU."""
import ctypes as C
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dsac_v2_b200 import _lib, synth

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_the_symbol_is_declared_as_the_header_declares_it():
    header = re.sub(r"\s+", " ", open(os.path.join(REPO, "include", "dsact.h")).read())
    proto = re.search(r"int dsact_dp_replay_steps\(([^)]*)\);", header).group(1)
    kinds = {"dsact_handle *h": C.c_void_p, "int32_t": C.c_int32, "int64_t": C.c_int64, "const int64_t *idx": C.c_void_p,
             "const dsact_noise *noise": C.POINTER(_lib.Noise), "float *stats_out": C.c_void_p, "void *stream": C.c_void_p}
    want = [kinds.get(a.strip(), kinds.get(a.strip().split(" ")[0])) for a in proto.split(",")]
    assert len(want) == 10 and None not in want, proto
    res, args = _lib.SYMBOLS["dsact_dp_replay_steps"]
    assert res is C.c_int and args == want, (args, want)


def test_a_null_handle_is_refused():
    lib = _lib.load()
    rc = lib.dsact_dp_replay_steps(None, 2, 8, 32, None, None, 16, None, 0, None)
    assert rc == -3, rc   # DSACT_ESTATE
    assert b"not bound" in lib.dsact_last_error()


# ---- which path replay_updates takes ---------------------------------------------------------------------------------
class _Dist:
    """What dp.world hands the algorithm: a live process group of `world` ranks (never reached: connect_peers is faked)."""


def _alg(monkeypatch, kw, world, connects=True):
    import dsac_v2
    alg = dsac_v2.DSAC_V2(**kw)
    eng = SimpleNamespace(name="engine")
    alg.networks = SimpleNamespace(engine=lambda batch=None: eng, route=alg.networks.route)
    log = SimpleNamespace(connect=[], steps=[], rounds=[])

    def connect(e, dist):
        log.connect.append(e)
        return connects

    def on_engine(e, buffer, batch, iteration, n, noise_fn, keys, global_batch=None):
        log.steps.append((e, batch, iteration, n, global_batch, noise_fn == alg._noise))
        return ["row"] * n

    monkeypatch.setattr(dsac_v2.dp, "world", lambda dist_module=None: (_Dist(), world) if world > 1 else (None, 1))
    monkeypatch.setattr(dsac_v2.dp, "connect_peers", connect)
    monkeypatch.setattr(dsac_v2, "replay_updates_on_engine", on_engine)
    alg.local_update = lambda data, iteration: log.rounds.append((data, iteration)) or "info"
    buf = SimpleNamespace(sample_batch=lambda b: ("minibatch", b))
    return alg, eng, buf, log


def _mlp_kw(**over):
    return synth.reference_kwargs(synth.CONFIGS["tiny"], replay_batch_size=8, **over)


def test_peer_transport_makes_one_dp_replay_steps_call(monkeypatch):
    alg, eng, buf, log = _alg(monkeypatch, _mlp_kw(), 4)
    assert alg.replay_updates(buf, 8, 10, 5) == ["row"] * 5
    assert alg.replay_updates(buf, 8, 15, 3) == ["row"] * 3
    assert log.connect == [eng]   # mapped once, by the first call
    assert log.steps == [(eng, 8, 10, 5, 32, True), (eng, 8, 15, 3, 32, True)]
    assert log.rounds == []


@pytest.mark.parametrize("why", ["nccl", "no_peer_access"])
def test_nccl_transport_takes_the_rounds(monkeypatch, why):
    kw = _mlp_kw(dsact_dp_transport="nccl") if why == "nccl" else _mlp_kw()
    alg, eng, buf, log = _alg(monkeypatch, kw, 2, connects=why != "no_peer_access")
    # (the rounds' local_update is faked here: it would decide the transport itself, the same way)
    assert alg.replay_updates(buf, 8, 4, 3) == ["info"] * 3
    assert log.steps == []
    assert log.rounds == [(("minibatch", 8), 4), (("minibatch", 8), 5), (("minibatch", 8), 6)]
    assert log.connect == ([] if why == "nccl" else [eng])


def test_separated_std_takes_the_rounds(monkeypatch):
    alg, eng, buf, log = _alg(monkeypatch, _mlp_kw(policy_std_type="mlp_separated", dsact_gemm="bf16x3"), 2)
    assert alg.networks.route.engine == "mlp"
    assert alg.dp_transport == "nccl"
    alg.replay_updates(buf, 8, 0, 2)
    assert log.steps == [] and len(log.rounds) == 2 and log.connect == []


def test_head_wise_engine_takes_the_rounds(monkeypatch):
    kw = synth.cnn_reference_kwargs(synth.CNN_CONFIGS["small_t1"], replay_batch_size=5)
    for world in (1, 2):
        alg, eng, buf, log = _alg(monkeypatch, kw, world)
        assert alg.networks.route.engine != "mlp"
        alg.replay_updates(buf, 5, 0, 2)
        assert log.steps == [] and len(log.rounds) == 2 and log.connect == []


def test_one_gpu_makes_one_replay_steps_call(monkeypatch):
    alg, eng, buf, log = _alg(monkeypatch, _mlp_kw(), 1)
    alg.replay_updates(buf, 8, 2, 4)
    assert log.steps == [(eng, 8, 2, 4, None, True)] and log.rounds == [] and log.connect == []


# ---- replay_updates_on_engine with a global batch ---------------------------------------------------------------------
class _Block:
    """LazyStatsRow.Block without the pinned copy and the CUDA event: the rows as the device wrote them."""

    def __init__(self, dev_stats):
        self.rows = dev_stats.tolist()

    def get(self):
        return self.rows


def test_replay_updates_on_engine_calls_dp_replay_steps(monkeypatch):
    import dsact_host
    monkeypatch.setattr(dsact_host.LazyStatsRow, "Block", _Block)
    stats = torch.arange(3 * _lib.NUM_STATS, dtype=torch.float32).view(3, _lib.NUM_STATS)
    stats[:, 14] = 0.0
    stats[2, 14] = 3.0   # update 2: the peer of rank 2 never arrived
    calls = []

    class Eng:
        def dp_replay_steps(self, *a, **k):
            calls.append(("dp", a, k))
            return stats

        def replay_steps(self, *a, **k):
            calls.append(("one", a, k))
            return stats

    eng = Eng()
    buf = SimpleNamespace(engine=eng, size=40, flush=lambda: None,
                          sample_indices=lambda b: torch.from_numpy(np.random.randint(0, 40, size=b)))
    noise_fn = lambda b: (torch.zeros(b, 2), torch.ones(b, 2), torch.zeros(b), torch.ones(b))   # noqa: E731
    keys = [("a", 0), ("b", 13)]
    rows = dsact_host.replay_updates_on_engine(eng, buf, 8, 7, 3, noise_fn, keys, global_batch=24)
    kind, a, k = calls[-1]
    assert kind == "dp" and a == (3, 8, 40, 7, 24)
    assert k["idx"].shape == (3, 8) and [x.shape for x in k["noise"]] == [(3, 8, 2), (3, 8, 2), (3, 8), (3, 8)]
    assert rows[0]["a"] == 0.0 and rows[1]["b"] == float(_lib.NUM_STATS + 13)
    with pytest.raises(_lib.DsactError, match="waiting for rank 2"):
        rows[2]["a"]
    dsact_host.replay_updates_on_engine(eng, buf, 8, 7, 1, noise_fn, keys)
    assert calls[-1][0] == "one"
