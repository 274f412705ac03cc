#!/usr/bin/env python
"""Generate golden vectors by running the UNMODIFIED reference update path.

Run once in the build container (needs /root/reference, which does not exist
on the GPU box):

    python tests/golden/make_golden.py

For every case in CASES it builds the reference's `DSAC_V2` (dsac_v2.py:66),
loads the deterministic numpy weights of `synth.make_weights`, and calls
`local_update(batch, it)` (dsac_v2.py:102) N times on `synth.make_batch`
minibatches.  The eight normal draws per update (SURVEY.md Appendix B) are
served from `synth.make_noise` by intercepting `Tensor.normal_`/`torch.normal`,
so no value in the fixture depends on torch's RNG stream.  Outputs: the 14
deterministic `tb_info` scalars per step, parameter/gradient digests, and for
the small cases the complete post-step state.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("DSAC_REFERENCE", "/root/reference")

sys.path.insert(0, REPO)
from dsac_v2_b200 import synth  # noqa: E402

sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(HERE, "gymstub"))
import torch  # noqa: E402
import utils  # noqa: E402,F401  (reference utils/__init__ puts utils/ on sys.path)
import dsac_v2 as ref_dsac  # noqa: E402
import dsac_v1 as ref_dsac_v1  # noqa: E402

assert os.path.realpath(ref_dsac.__file__).startswith(os.path.realpath(REF)), ref_dsac.__file__

# name, config, batch, steps, full-state snapshot steps, hyper overrides
CASES = [
    ("tiny_b16", "tiny", 16, 20, (1, 2, 3, 20), {}),
    ("ragged_b37", "ragged", 37, 20, (1, 2, 20), {}),
    ("pendulum_b256", "pendulum", 256, 100, (), {}),
    ("halfcheetah_b512", "halfcheetah", 512, 40, (), {}),
    ("humanoid_b256", "humanoid", 256, 100, (), {}),
    ("humanoid_b4096", "humanoid", 4096, 100, (), {}),   # the benchmarked configuration: the north_star gate is the first 100 losses
    # fixed temperature + different delay / tau_b: exercises the non-default branches
    ("tiny_fixed_alpha", "tiny", 16, 12, (1, 12), {"auto_alpha": False, "alpha": 0.2, "delay_update": 3, "tau_b": 0.05}),
    # the policy's other std types (networks/mlp.py:42-72)
    ("tiny_std_separated", "tiny", 16, 10, (10,), {"policy_std_type": "mlp_separated"}),
    ("tiny_std_parameter", "tiny", 16, 10, (10,), {"policy_std_type": "parameter"}),
    # the plain Gaussian action distribution (utils/act_distribution_cls.py:82-116)
    ("tiny_gauss", "tiny", 16, 10, (1, 2, 10), {"policy_act_distribution": "GaussDistribution"}),
    # CNN approximators (example_train/dsacv2_cnn_carracing_offasync.py: type_2 encoder, 3x96x96 observations); digests only
    ("cnn_carracing_b4", "carracing", 4, 6, (), {}),
    ("cnn_type1_b5", "small_t1", 5, 4, (), {}),   # type_1 encoder (8x8 stride 4 first layer)
    # the older algorithm (dsac_v1.py): bounded loss with the default TD bound, a tight bound that clips, the Gaussian NLL
    ("v1_tiny_b16", "tiny", 16, 12, (1, 2, 12), {"algorithm": "DSAC_V1"}),
    ("v1_ragged_tight", "ragged", 37, 8, (8,), {"algorithm": "DSAC_V1", "TD_bound": 0.5, "delay_update": 3}),
    ("v1_tiny_nll", "tiny", 16, 8, (8,), {"algorithm": "DSAC_V1", "bound": False}),
] + [
    # the reference's other hidden activations (utils/common_utils.py:16-43), same one in critics and policy
    (f"{cfg}_{act}", cfg, batch, 10, (10,), {"value_hidden_activation": act, "policy_hidden_activation": act})
    for cfg, batch, act in (("tiny", 16, "relu"), ("tiny", 33, "tanh"), ("ragged", 19, "elu"), ("ragged", 37, "selu"),
                            ("tiny", 8, "sigmoid"))
] + [
    # critics and policy of different depths, widths and activations (synth.ASYM_CONFIGS): two row tiles of 64, the last
    # ragged; the full state only for the smallest
    (f"{cfg}_b70", cfg, 70, 10, (1,) if cfg == "layered_q" else (), {}) for cfg in synth.ASYM_CONFIGS
]

V1_TB_KEYS = ["DSAC/critic_avg_q-RL iter", "DSAC/critic_avg_std-RL iter", "Loss/Actor loss-RL iter", "DSAC/policy_mean-RL iter",
              "DSAC/policy_std-RL iter", "DSAC/entropy-RL iter", "DSAC/alpha-RL iter"]   # dsac_v1.py:172-181
TB_KEYS = [
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

DIGEST_STEPS = (1, 2, 10, 50, 100)


class NoiseFeed:
    """Replaces the reference's normal draws with a prepared queue."""

    def __init__(self):
        self.queue = []
        self._normal_ = torch.Tensor.normal_
        self._normal = torch.normal

    def install(self):
        feed = self

        def normal_(t, *a, **k):
            src = feed.queue.pop(0)
            assert tuple(t.shape) == src.shape, (t.shape, src.shape)
            return t.copy_(torch.from_numpy(src))

        def normal(mean, std, *a, **k):
            src = feed.queue.pop(0)
            assert tuple(mean.shape) == src.shape
            return mean + std * torch.from_numpy(src)

        torch.Tensor.normal_ = normal_
        torch.normal = normal

    def remove(self):
        torch.Tensor.normal_ = self._normal_
        torch.normal = self._normal


def digest(t) -> np.ndarray:
    if t is None:  # log_alpha when auto_alpha is off
        return np.zeros(11)
    d = t.detach().double().reshape(-1)
    head = d[:8].numpy()
    head = np.pad(head, (0, 8 - head.size))
    return np.concatenate([[d.sum().item(), d.abs().sum().item(), (d * d).sum().item()], head])


def run_case(name, cfg_name, batch, steps, snaps, over):
    cnn = cfg_name in synth.CNN_CONFIGS   # BASELINE config 5: conv encoder + separate heads (networks/cnn.py)
    cfg = synth.CNN_CONFIGS[cfg_name] if cnn else synth.mlp_config(cfg_name)
    torch.manual_seed(0)
    v1 = over.get("algorithm") == "DSAC_V1"
    tb_keys = V1_TB_KEYS if v1 else TB_KEYS
    kw = synth.cnn_reference_kwargs(cfg, **over) if cnn else synth.reference_kwargs(cfg, **over)
    alg = ref_dsac_v1.DSAC_V1(**kw) if v1 else ref_dsac.DSAC_V2(**kw)
    sd = alg.networks.state_dict()
    std_type = over.get("policy_std_type", "mlp_shared")
    weights = synth.make_cnn_weights(cfg) if cnn else synth.make_weights_v1(cfg) if v1 else \
        (synth.make_weights(cfg) if std_type == "mlp_shared" else synth.make_weights_std(cfg, std_type))
    for k, v in weights.items():
        assert tuple(sd[k].shape) == v.shape, k
        sd[k] = torch.from_numpy(v)
    alg.networks.load_state_dict(sd)
    names = [k for k, _ in alg.networks.named_parameters()]
    trainable = [k for k, p in alg.networks.named_parameters() if p.requires_grad]

    feed = NoiseFeed()
    feed.install()
    out = {"tb": np.zeros((steps, len(tb_keys)))}
    try:
        for it in range(steps):
            data = {k: torch.from_numpy(v) for k, v in (synth.make_cnn_batch if cnn else synth.make_batch)(cfg, batch, it).items()}
            feed.queue = synth.make_noise(cfg, batch, it)[:5 if v1 else 8]   # DSAC_V1 draws eps1, eps2 and three z's
            tb = alg.local_update(data, it)
            assert not feed.queue
            out["tb"][it] = [float(tb[k]) for k in tb_keys]
            params = dict(alg.networks.named_parameters())
            if it + 1 in DIGEST_STEPS and it + 1 <= steps:
                out[f"pdigest_{it + 1}"] = np.stack([digest(params[k]) for k in names])
            if it in (0, 1):
                out[f"gdigest_{it}"] = np.stack([digest(params[k].grad) for k in trainable])
            if it + 1 in snaps:
                for k in names:
                    out[f"state_{it + 1}/{k}"] = params[k].detach().numpy().copy()
                if it in (0, 1):
                    for k in trainable:
                        if params[k].grad is not None:
                            out[f"grad_{it}/{k}"] = params[k].grad.detach().numpy().copy()
    finally:
        feed.remove()
    out["param_names"] = np.array(names)
    out["trainable_names"] = np.array(trainable)
    out["tb_keys"] = np.array(tb_keys)
    out["meta"] = np.array([cfg_name, str(batch), str(steps), repr(sorted(over.items()))])
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    col = 2 if v1 else 7   # actor loss (DSAC_V1 does not log the critic loss) / critic loss
    print(f"{name}: {steps} steps, loss {out['tb'][0, col]:.6f} -> {out['tb'][-1, col]:.6f}, "
          f"{os.path.getsize(os.path.join(HERE, name + '.npz')) / 1024:.0f} KiB")


if __name__ == "__main__":
    torch.set_num_threads(4)
    only = set(sys.argv[1:])
    for case in CASES:
        if not only or case[0] in only:
            run_case(*case)
