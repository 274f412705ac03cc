"""The MLP engine's step schedule: how many kernels every entry point launches, and dsact_profile_step's launch count and
FLOPs per class (other, forward GEMM, dgrad GEMM, weight-gradient GEMM).  The values are pinned, so that a change to how
the step lowers its network passes (layer chains or per-layer GEMM groups, the forked side branches) shows up here even
where it leaves every result within tolerance.

Shapes: humanoid (the benchmark's) and ragged (no width a multiple of a tile), in fp32 (SIMT GEMM groups) and bf16x3 (layer
chains); layered_q, whose 6-layer critic is outside the layer-chain kernel's range and takes per-layer wgmma groups; and a
DSAC_V1 handle (one critic).  200 rows: several 64-row tiles and a ragged last one."""
import numpy as np
import pytest
import torch

from dsac_v2_b200 import synth

pytestmark = pytest.mark.gpu

B = 200
CAP = 300   # replay ring rows
# Humanoid: 2*M*N*K summed over every GEMM problem of one step, per sample (DESIGN.md section 4)
HUMANOID_FLOP_PER_SAMPLE = 6_480_896


def make_handle(cfg, mode, graph, v1=False, batch=B):
    """A DSAC-T (or DSAC_V1) MLP-engine handle of synth configuration `cfg` with its synth weights."""
    from dsac_v2_b200.engine import Engine, make_config
    if v1:
        from v1_mlp_common import make_engine
        return make_engine(cfg, batch, dict(synth.HYPER), mode, graph)
    act_q, act_pi = synth.activations(cfg)
    c = make_config(cfg["obs_dim"], cfg["act_dim"], *synth.hidden_sizes(cfg), max_batch=batch, act_q=act_q, act_pi=act_pi,
                    gemm_mode=mode, use_graph=graph)
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    eng = Engine(c, torch.device("cuda", 0), lim, -lim)
    eng.load_weights(synth.make_weights(cfg))
    return eng


def run_schedule(eng, cfg, v1=False, batch=B):
    """Every entry point of the handle once or twice on seeded inputs: {call: launches} and the profiled step's
    (launches, FLOPs) per class.  DSAC_V1 handles have no split update (compute_grads, phases, apply)."""
    pick = (0, 1, 3, 3) if v1 else (0, 1, 4, 5)

    def data(it):
        b = {k: torch.from_numpy(v).cuda() for k, v in synth.make_batch(cfg, batch, it).items()}
        n = synth.make_noise(cfg, batch, it)
        return b, tuple(torch.from_numpy(n[i]).cuda() for i in pick)

    calls = {}

    def call(name, fn):
        fn()
        calls[name] = eng.last_call_launches()

    b, n = data(0)
    call("step", lambda: eng.step(b, 0, n))
    b1, _ = data(1)
    call("step_device_noise", lambda: eng.step(b1, 1))
    eng.bind_replay(CAP)
    eng.replay_add({k: torch.from_numpy(v).cuda() for k, v in synth.make_batch(cfg, CAP, 99).items()}, CAP, 0)
    idx = torch.from_numpy(np.random.default_rng(1).integers(0, CAP, batch))
    _, n2 = data(2)
    call("replay_step", lambda: eng.replay_step(batch, CAP, 2, idx=idx, noise=n2))
    call("replay_step_device_draws", lambda: eng.replay_step(batch, CAP, 3))
    it = 4
    if not v1:
        b4, n4 = data(4)
        call("compute_grads", lambda: eng.compute_grads(b4, n4))
        call("apply", lambda: eng.apply(4))
        b5, n5 = data(5)
        call("grad_phase1", lambda: eng.grad_phase1(b5, n5))
        call("grad_phase2", lambda: eng.grad_phase2(batch))
        call("apply_after_phases", lambda: eng.apply(5))
        it = 6
    bp, np_ = data(it)
    prof = eng.profile_step(bp, it, np_)
    torch.cuda.synchronize()
    classes = ("other", "gemm_fwd", "gemm_dgrad", "gemm_wgrad")
    return calls, [prof[k]["launches"] for k in classes], [prof[k]["flops"] for k in classes]


# The entry points run_schedule calls, in order (DSAC_V1 handles: the first four)
CALLS = ("step", "step_device_noise", "replay_step", "replay_step_device_draws", "compute_grads", "apply", "grad_phase1",
         "grad_phase2", "apply_after_phases")
# Recorded before the step's network passes were described once in csrc/engine.cu: (config, mode, graph, v1) ->
# (launches per call of CALLS, profiled launches per class, profiled FLOPs per class)
EXPECTED = {
    ("humanoid", "fp32", True, False): ((23, 24, 24, 25, 23, 1, 10, 13, 1), [5, 8, 7, 3], [0, 746086400, 269926400, 280166400]),
    ("humanoid", "fp32", False, False): ((23, 24, 24, 25, 23, 1, 10, 13, 1), [5, 8, 7, 3], [0, 746086400, 269926400, 280166400]),
    ("humanoid", "bf16x3", True, False): ((12, 12, 13, 13, 12, 1, 4, 8, 1), [5, 2, 2, 2], [0, 746086400, 269926400, 280166400]),
    ("humanoid", "bf16x3", False, False): ((11, 11, 12, 12, 12, 1, 4, 8, 1), [5, 2, 2, 2], [0, 746086400, 269926400, 280166400]),
    ("ragged", "fp32", True, False): ((23, 24, 24, 25, 23, 1, 10, 13, 1), [5, 8, 7, 3], [0, 10988800, 5875200, 4137600]),
    ("ragged", "fp32", False, False): ((23, 24, 24, 25, 23, 1, 10, 13, 1), [5, 8, 7, 3], [0, 10988800, 5875200, 4137600]),
    ("ragged", "bf16x3", True, False): ((12, 12, 13, 13, 12, 1, 4, 8, 1), [5, 2, 2, 2], [0, 10988800, 5875200, 4137600]),
    ("ragged", "bf16x3", False, False): ((11, 11, 12, 12, 12, 1, 4, 8, 1), [5, 2, 2, 2], [0, 10988800, 5875200, 4137600]),
    ("layered_q", "bf16x3", True, False): ((30, 30, 31, 31, 31, 1, 17, 14, 1), [6, 14, 8, 2], [0, 26468000, 14152000, 9724000]),
    ("layered_q", "bf16x3", False, False): ((30, 30, 31, 31, 31, 1, 17, 14, 1), [6, 14, 8, 2], [0, 26468000, 14152000, 9724000]),
    ("hopper", "bf16x3", True, True): ((12, 12, 13, 13), [5, 2, 2, 2], [0, 270540800, 158617600, 108236800]),
    ("hopper", "bf16x3", False, True): ((11, 11, 12, 12), [5, 2, 2, 2], [0, 270540800, 158617600, 108236800]),
}
CASES = sorted(EXPECTED)


@pytest.mark.parametrize("case", CASES, ids=["-".join(map(str, c)) for c in CASES])
def test_step_schedule_is_pinned(case):
    cfg_name, mode, graph, v1 = case
    cfg = synth.mlp_config(cfg_name)
    eng = make_handle(cfg, mode, graph, v1)
    try:
        calls, launches, flops = run_schedule(eng, cfg, v1)
    finally:
        eng.close()
    want_calls, want_launches, want_flops = EXPECTED[case]
    assert calls == dict(zip(CALLS, want_calls))
    assert launches == want_launches
    assert flops == want_flops
    if cfg_name == "humanoid":
        assert sum(flops) == HUMANOID_FLOP_PER_SAMPLE * B
