"""Shared by test_std_mlp.py and test_gpu_std_mlp.py: MLP-engine handles, weights and the oracle for the policy's
"mlp_separated" / "parameter" std types, on configurations whose critics and policy may differ in shape."""
import numpy as np
import torch

from dsac_v2_b200 import synth

STD_TYPES = ("mlp_separated", "parameter")


def std_config(cfg, std_type, batch, mode="fp32", graph=True, **over):
    """dsact_config of synth configuration `cfg` (CONFIGS or ASYM_CONFIGS entry) with the policy of `std_type`."""
    from dsac_v2_b200.engine import make_config
    h = synth.HYPER
    act_q, act_pi = synth.activations(cfg)
    kw = dict(max_batch=batch, act_q=act_q, act_pi=act_pi, gemm_mode=mode, use_graph=graph, policy_std=std_type,
              gamma=h["gamma"], tau=h["tau"], delay_update=h["delay_update"], auto_alpha=h["auto_alpha"], alpha=h["alpha"],
              lr_q=h["value_learning_rate"], lr_pi=h["policy_learning_rate"], lr_alpha=h["alpha_learning_rate"],
              min_log_std=h["policy_min_log_std"], max_log_std=h["policy_max_log_std"])
    kw.update(over)
    return make_config(cfg["obs_dim"], cfg["act_dim"], *synth.hidden_sizes(cfg), **kw)


def std_weights(cfg, std_type, seed=0, row=None):
    """`synth.make_weights_std` for any configuration: the critics of `synth.make_weights`, the policy's mean (and
    log_std) networks with the policy's own hidden widths.  `row`: the "parameter" log_std row (default -0.5)."""
    if "hidden" in cfg:
        out = synth.make_weights_std(cfg, std_type, seed)
    else:
        out = {k: v for k, v in synth.make_weights(cfg, seed).items() if not k.startswith("policy")}
        sizes = [cfg["obs_dim"]] + list(synth.hidden_sizes(cfg)[1]) + [cfg["act_dim"]]
        g = np.random.default_rng([seed, 67, STD_TYPES.index(std_type)])
        for head in ("mean", "log_std") if std_type == "mlp_separated" else ("mean",):
            for j in range(len(sizes) - 1):
                bound = 1.0 / np.sqrt(sizes[j])
                for leaf, shape in (("weight", (sizes[j + 1], sizes[j])), ("bias", (sizes[j + 1],))):
                    out[f"policy.{head}.{2 * j}.{leaf}"] = g.uniform(-bound, bound, shape).astype(np.float32)
        if std_type == "parameter":
            out["policy.log_std"] = np.full((1, cfg["act_dim"]), -0.5, dtype=np.float32)
        for k in [k for k in out if k.startswith("policy.")]:
            out["policy_target." + k[len("policy."):]] = out[k].copy()
    if row is not None:
        out["policy.log_std"] = np.asarray(row, dtype=np.float32).reshape(1, -1)
        out["policy_target.log_std"] = out["policy.log_std"].copy()
    return out


def make_engine(cfg, batch, std_type, mode="fp32", graph=True, weights=None, **over):
    from dsac_v2_b200.engine import Engine
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    eng = Engine(std_config(cfg, std_type, batch, mode, graph, **over), torch.device("cuda", 0), lim, -lim)
    eng.load_weights(std_weights(cfg, std_type) if weights is None else weights)
    return eng


def make_oracle(cfg, std_type, weights=None, dtype=torch.float32, **over):
    from oracle.dsact_oracle import OracleDSACTStd
    lim = [cfg["act_lim"]] * cfg["act_dim"]
    act_q, act_pi = synth.activations(cfg)
    hyper = dict(synth.HYPER, value_hidden_activation=act_q, policy_hidden_activation=act_pi, **over)
    hyper.pop("hidden_activation", None)
    return OracleDSACTStd(cfg["obs_dim"], cfg["act_dim"], *synth.hidden_sizes(cfg), lim, [-x for x in lim],
                          std_weights(cfg, std_type) if weights is None else weights, std_type=std_type, dtype=dtype, **hyper)


def feed(cfg, batch, it, device="cuda"):
    b = {k: torch.from_numpy(v).to(device) for k, v in synth.make_batch(cfg, batch, it).items()}
    n = synth.make_noise(cfg, batch, it)
    return b, tuple(torch.from_numpy(n[i]).to(device) for i in (0, 1, 4, 5))
