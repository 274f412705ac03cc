"""Deterministic synthetic inputs for the DSAC-T update path (numpy only).

Everything the parity tests, the golden-vector generator, ``smoke()`` and
``bench.py`` feed to the update step comes from here, so that the reference
run (``tests/golden/make_golden.py``, executed once in the build container)
and the CUDA run (on the GPU box, where the reference does not exist) see
bit-identical weights, minibatches and noise.  Streams are numpy PCG64
(`numpy.random.default_rng`), whose output is stable across platforms.

Shapes follow SURVEY.md §8(d): obs/obs2 ~ N(0,1) [B,O], act ~ U(lo,hi) [B,A],
rew ~ N(0,1) [B], done ~ Bernoulli(0.01) [B]; noise = the eight normal draws
one `DSAC_V2.local_update` consumes (reference dsac_v2.py:160,228,212 — see
SURVEY.md Appendix B).
"""
from __future__ import annotations

import numpy as np

# Named problem shapes of BASELINE.json `configs` (P, H, C) plus a tiny one
# whose complete state fits in a golden fixture.
CONFIGS = {
    "tiny": dict(obs_dim=5, act_dim=2, hidden=(32, 32), act_lim=1.0),
    "pendulum": dict(obs_dim=3, act_dim=1, hidden=(256, 256, 256), act_lim=2.0),
    "halfcheetah": dict(obs_dim=17, act_dim=6, hidden=(256, 256), act_lim=1.0),
    "humanoid": dict(obs_dim=376, act_dim=17, hidden=(256, 256, 256), act_lim=0.4),
    # ragged: nothing is a multiple of the GEMM tile or of the vector width
    "ragged": dict(obs_dim=11, act_dim=3, hidden=(40, 24, 72), act_lim=1.5),
}

# Critics and policy of different depths, widths and activations (`hidden_q` / `act_q` for the critics, `hidden_pi` /
# `act_pi` for the policy), the way the reference's value_* / policy_* kwargs build them.  Kept out of CONFIGS, whose
# entries size both networks from one `hidden`.  Widths that are multiples of 8 and at most 256 run the layer-chain kernel.
ASYM_CONFIGS = {
    # chain widths in all four 64-column blocks, off the 16- and 64-grids, an 8-wide bottleneck; obs_dim = 64 puts the
    # critic's action segment at the start of a k-block; six critic layers, a one-layer policy
    "asym": dict(obs_dim=64, act_dim=5, hidden_q=(152, 104, 8, 192, 256, 72), act_q="elu", hidden_pi=(136,), act_pi="tanh",
                 act_lim=1.0),
    # the policy deeper than the critics; its 2A = 192 output and a 96-column action segment over two k-blocks
    "deep_pi": dict(obs_dim=13, act_dim=96, hidden_q=(200,), act_q="selu", hidden_pi=(256, 24, 128, 200, 64, 248),
                    act_pi="gelu", act_lim=1.0),
    # widths the chain kernel does not take: the per-layer path, with pi.L > q.L and with q.L > pi.L
    "layered_pi": dict(obs_dim=7, act_dim=3, hidden_q=(300, 40), act_q="relu", hidden_pi=(48, 48, 48, 48), act_pi="sigmoid",
                       act_lim=1.0),
    "layered_q": dict(obs_dim=9, act_dim=2, hidden_q=(45, 40, 40, 40, 40, 40), act_q="tanh", hidden_pi=(520,), act_pi="gelu",
                      act_lim=1.0),
}

# The reference's DSAC_V1 MLP example (example_train/dsacv1_mlp_hopper_offserial.py): Hopper's observation and action
# sizes, 256x3 GELU critic and policy.  Kept out of CONFIGS, whose entries the DSAC-T tests walk.
EXAMPLE_CONFIGS = {
    "hopper": dict(obs_dim=11, act_dim=3, hidden=(256, 256, 256), act_lim=1.0),
}

# BASELINE.json config 5 (gym_carracingraw, SURVEY.md §8f rank 1): conv encoder `type_2` + separate mean / log_std
# heads (csrc/cnn_engine.cuh; oracle/dsact_oracle.py:OracleDSACTCNN, tests/golden/cnn_carracing_b4.npz).
CNN_CONFIGS = {
    "carracing": dict(obs_dim=(3, 96, 96), act_dim=3, act_lim=1.0, conv_type="type_2"),
    # the reference's other encoder (networks/cnn.py:173-186: 8x8/4, 4x4/2, 3x3/1, heads 512-256) on a smaller image
    "small_t1": dict(obs_dim=(2, 44, 44), act_dim=2, act_lim=1.0, conv_type="type_1"),
    "odd": dict(obs_dim=(3, 13, 11), act_dim=2, act_lim=1.0, conv_type="test_odd"),
}
# reference networks/cnn.py:201-216 (type_2) and :163-170 (type_1): kernel sizes, channels, strides, head widths
CONV_TYPES = {
    "type_1": dict(kernels=(8, 4, 3), channels=(32, 64, 64), strides=(4, 2, 1), heads=(512, 256)),
    "type_2": dict(kernels=(4, 3, 3, 3, 3, 3), channels=(8, 16, 32, 64, 128, 256), strides=(2, 2, 2, 2, 1, 1), heads=(256, 256, 256)),
    # not a reference type: channel counts that are no multiples of 4 / 8 and 2x2 / 1x1 windows, for the one-channel-per-thread
    # kernels of conv.cuh (tests only; checked against the oracle)
    "test_odd": dict(kernels=(3, 2, 1), channels=(6, 10, 12), strides=(2, 1, 1), heads=(24,)),
}

HYPER = dict(
    gamma=0.99,
    tau=0.005,
    delay_update=2,
    auto_alpha=True,
    alpha=0.2,
    value_learning_rate=1e-4,
    policy_learning_rate=1e-4,
    alpha_learning_rate=3e-4,
    policy_min_log_std=-20.0,
    policy_max_log_std=0.5,
)


def _rng(*key) -> np.random.Generator:
    return np.random.default_rng([int(k) for k in key])


def mlp_config(name: str) -> dict:
    """A named MLP configuration of CONFIGS, ASYM_CONFIGS or EXAMPLE_CONFIGS."""
    if name in CONFIGS:
        return CONFIGS[name]
    return ASYM_CONFIGS[name] if name in ASYM_CONFIGS else EXAMPLE_CONFIGS[name]


def hidden_sizes(cfg: dict) -> tuple:
    """(hidden_q, hidden_pi): the critics' and the policy's hidden widths of a CONFIGS or ASYM_CONFIGS entry."""
    if "hidden" in cfg:
        return tuple(cfg["hidden"]), tuple(cfg["hidden"])
    return tuple(cfg["hidden_q"]), tuple(cfg["hidden_pi"])


def activations(cfg: dict) -> tuple:
    """(act_q, act_pi): the critics' and the policy's hidden activations (the reference's default GELU unless given)."""
    return cfg.get("act_q", "gelu"), cfg.get("act_pi", "gelu")


def net_shapes(obs_dim, act_dim, hidden_q, hidden_pi=None):
    """(q_sizes, pi_sizes) layer-size lists, reference networks/mlp.py:58,116; the policy takes the critics' hidden
    widths unless `hidden_pi` is given."""
    q = [obs_dim + act_dim] + list(hidden_q) + [2]
    pi = [obs_dim] + list(hidden_q if hidden_pi is None else hidden_pi) + [2 * act_dim]
    return q, pi


def make_weights(cfg: dict, seed: int = 0) -> dict:
    """state_dict-shaped fp32 arrays for q1, q2, policy (targets = copies).

    U(-1/sqrt(fan_in), 1/sqrt(fan_in)) like nn.Linear's default init; keys use
    the reference's schema (`q1.q.{0,2,..}.weight`, `policy.policy.{0,2,..}.bias`).
    """
    q_sizes, pi_sizes = net_shapes(cfg["obs_dim"], cfg["act_dim"], *hidden_sizes(cfg))
    out = {}
    for n, (name, inner, sizes) in enumerate(
        (("q1", "q", q_sizes), ("q2", "q", q_sizes), ("policy", "policy", pi_sizes))
    ):
        g = _rng(seed, 11, n)
        for j in range(len(sizes) - 1):
            bound = 1.0 / np.sqrt(sizes[j])
            out[f"{name}.{inner}.{2 * j}.weight"] = g.uniform(
                -bound, bound, size=(sizes[j + 1], sizes[j])
            ).astype(np.float32)
            out[f"{name}.{inner}.{2 * j}.bias"] = g.uniform(
                -bound, bound, size=(sizes[j + 1],)
            ).astype(np.float32)
    for src, dst in (("q1", "q1_target"), ("q2", "q2_target"), ("policy", "policy_target")):
        for k in [k for k in out if k.startswith(src + ".")]:
            out[dst + k[len(src):]] = out[k].copy()
    return out


def make_batch(cfg: dict, batch: int, step: int, seed: int = 123) -> dict:
    g = _rng(seed, 22, step)
    O, A, lim = cfg["obs_dim"], cfg["act_dim"], cfg["act_lim"]
    return {
        "obs": g.standard_normal((batch, O)).astype(np.float32),
        "act": g.uniform(-lim, lim, size=(batch, A)).astype(np.float32),
        "rew": g.standard_normal(batch).astype(np.float32),
        "obs2": g.standard_normal((batch, O)).astype(np.float32),
        "done": (g.random(batch) < 0.01).astype(np.float32),
        "logp": np.zeros(batch, dtype=np.float32),
    }


def make_noise(cfg: dict, batch: int, step: int, seed: int = 7) -> list:
    """The 8 standard-normal draws of one update, in the reference's order:
    eps1 [B,A], eps2 [B,A], z1..z6 [B] (z3,z4 are the two that matter)."""
    g = _rng(seed, 33, step)
    A = cfg["act_dim"]
    out = [g.standard_normal((batch, A)).astype(np.float32) for _ in range(2)]
    out += [g.standard_normal(batch).astype(np.float32) for _ in range(6)]
    return out


def reference_kwargs(cfg: dict, **over) -> dict:
    """The kwargs dict the reference threads through DSAC_V2 / ApproxContainer
    (what example_train/main.py + utils/init_args.py would have produced)."""
    lim = np.full(cfg["act_dim"], cfg["act_lim"], dtype=np.float32)
    hidden_q, hidden_pi = hidden_sizes(cfg)
    act_q, act_pi = activations(cfg)
    kw = dict(
        algorithm="DSAC_V2",
        obsv_dim=cfg["obs_dim"],
        action_dim=cfg["act_dim"],
        action_type="continu",
        action_high_limit=lim,
        action_low_limit=-lim,
        value_func_name="ActionValueDistri",
        value_func_type="MLP",
        value_hidden_sizes=list(hidden_q),
        value_hidden_activation=act_q,
        value_output_activation="linear",
        policy_func_name="StochaPolicy",
        policy_func_type="MLP",
        policy_act_distribution="TanhGaussDistribution",
        policy_hidden_sizes=list(hidden_pi),
        policy_hidden_activation=act_pi,
        policy_output_activation="linear",
        cnn_shared=False,
    )
    kw.update(HYPER)
    kw.update(over)
    return kw


# ---- CNN variant (config 5) -----------------------------------------------------------------------------------------
def conv_feature_dim(cfg: dict) -> int:
    c, h, w = cfg["obs_dim"]
    t = CONV_TYPES[cfg["conv_type"]]
    for k, s_ in zip(t["kernels"], t["strides"]):
        h, w = (h - k) // s_ + 1, (w - k) // s_ + 1
    return t["channels"][-1] * h * w


def make_cnn_weights(cfg: dict, seed: int = 0) -> dict:
    """state_dict-shaped fp32 arrays in the schema of the reference's CNN `StochaPolicy` / `ActionValueDistri`
    (networks/cnn.py:151-240, 383-461): `{net}.conv.{0,2,..}.{weight,bias}`, `{net}.mean.{0,2,..}`, `{net}.log_std.{0,2,..}`;
    U(-1/sqrt(fan_in), 1/sqrt(fan_in)) like the torch defaults; targets are copies."""
    t = CONV_TYPES[cfg["conv_type"]]
    feat, A = conv_feature_dim(cfg), cfg["act_dim"]
    out = {}
    for n, (net, extra, width) in enumerate((("q1", A, 1), ("q2", A, 1), ("policy", 0, A))):
        g = _rng(seed, 44, n)
        cin = cfg["obs_dim"][0]
        for j, (k, cout) in enumerate(zip(t["kernels"], t["channels"])):
            bound = 1.0 / np.sqrt(cin * k * k)
            out[f"{net}.conv.{2 * j}.weight"] = g.uniform(-bound, bound, (cout, cin, k, k)).astype(np.float32)
            out[f"{net}.conv.{2 * j}.bias"] = g.uniform(-bound, bound, (cout,)).astype(np.float32)
            cin = cout
        sizes = [feat + extra] + list(t["heads"]) + [width]
        for head in ("mean", "log_std"):
            for j in range(len(sizes) - 1):
                bound = 1.0 / np.sqrt(sizes[j])
                out[f"{net}.{head}.{2 * j}.weight"] = g.uniform(-bound, bound, (sizes[j + 1], sizes[j])).astype(np.float32)
                out[f"{net}.{head}.{2 * j}.bias"] = g.uniform(-bound, bound, (sizes[j + 1],)).astype(np.float32)
    for src, dst in (("q1", "q1_target"), ("q2", "q2_target"), ("policy", "policy_target")):
        for k in [k for k in out if k.startswith(src + ".")]:
            out[dst + k[len(src):]] = out[k].copy()
    return out


def make_cnn_batch(cfg: dict, batch: int, step: int, seed: int = 123) -> dict:
    """Image minibatch: obs/obs2 ~ U(0,1) [B,C,H,W] (pixel-like), the rest as `make_batch`."""
    g = _rng(seed, 55, step)
    A, lim = cfg["act_dim"], cfg["act_lim"]
    shape = (batch,) + tuple(cfg["obs_dim"])
    return {
        "obs": g.random(shape, dtype=np.float32),
        "act": g.uniform(-lim, lim, size=(batch, A)).astype(np.float32),
        "rew": g.standard_normal(batch).astype(np.float32),
        "obs2": g.random(shape, dtype=np.float32),
        "done": (g.random(batch) < 0.01).astype(np.float32),
    }


def cnn_reference_kwargs(cfg: dict, **over) -> dict:
    """kwargs of example_train/dsacv2_cnn_carracing_offasync.py:53-79 for `DSAC_V2` / `ApproxContainer`."""
    kw = reference_kwargs(dict(obs_dim=0, act_dim=cfg["act_dim"], act_lim=cfg["act_lim"], hidden=()))
    for k in ("value_hidden_sizes", "policy_hidden_sizes"):
        kw.pop(k)
    kw.update(obsv_dim=tuple(cfg["obs_dim"]), value_func_type="CNN", policy_func_type="CNN",
              value_conv_type=cfg["conv_type"], policy_conv_type=cfg["conv_type"])
    kw.update(over)
    return kw


# ---- other policy std types (reference networks/mlp.py:42-72; SURVEY.md §8f rank 4) ---------------------------------
def make_weights_std(cfg: dict, std_type: str, seed: int = 0) -> dict:
    """`make_weights` with the policy in the schema of `std_type`:
    "mlp_separated": `policy.mean.{0,2,..}` and `policy.log_std.{0,2,..}` (two MLPs ending in act_dim outputs),
    "parameter": `policy.mean.{0,2,..}` and the learnable row `policy.log_std` [1, act_dim] (= -0.5)."""
    out = {k: v for k, v in make_weights(cfg, seed).items() if not k.startswith("policy")}
    sizes = [cfg["obs_dim"]] + list(cfg["hidden"]) + [cfg["act_dim"]]
    g = _rng(seed, 66, {"mlp_separated": 0, "parameter": 1}[std_type])
    heads = ("mean", "log_std") if std_type == "mlp_separated" else ("mean",)
    for head in heads:
        for j in range(len(sizes) - 1):
            bound = 1.0 / np.sqrt(sizes[j])
            out[f"policy.{head}.{2 * j}.weight"] = g.uniform(-bound, bound, (sizes[j + 1], sizes[j])).astype(np.float32)
            out[f"policy.{head}.{2 * j}.bias"] = g.uniform(-bound, bound, (sizes[j + 1],)).astype(np.float32)
    if std_type == "parameter":
        out["policy.log_std"] = np.full((1, cfg["act_dim"]), -0.5, dtype=np.float32)
    for k in [k for k in out if k.startswith("policy.")]:
        out["policy_target" + k[len("policy"):]] = out[k].copy()
    return out


# ---- DSAC_V1 (reference dsac_v1.py; SURVEY.md §8f rank 4) --------------------------------------------------------------
def to_v1_schema(weights: dict) -> dict:
    """DSAC-T weights in the schema of `dsac_v1.ApproxContainer` (:17-52): critic `q1` (and its target) becomes the one
    critic `q`, `q2` is dropped, the policy and its target are kept."""
    out = {}
    for k, v in weights.items():
        if k.startswith("q1"):
            out["q" + k[2:]] = v.copy()
        elif k.startswith("policy"):
            out[k] = v.copy()
    return out


def make_weights_v1(cfg: dict, seed: int = 0) -> dict:
    """`make_weights` in the V1 schema: one critic `q.q.*`, `policy.policy.*`, targets."""
    return to_v1_schema(make_weights(cfg, seed))


def make_cnn_weights_v1(cfg: dict, seed: int = 0) -> dict:
    """`make_cnn_weights` in the V1 schema: `q.conv.*`, `q.mean.*`, `q.log_std.*`, the CNN policy, targets."""
    return to_v1_schema(make_cnn_weights(cfg, seed))


def make_weights_std_v1(cfg: dict, std_type: str, seed: int = 0) -> dict:
    """`make_weights_std` in the V1 schema: one critic `q.q.*`, the policy of `std_type`, targets."""
    return to_v1_schema(make_weights_std(cfg, std_type, seed))
