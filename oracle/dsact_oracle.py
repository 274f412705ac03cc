"""CPU oracle for the DSAC-T update path.  TEST INFRASTRUCTURE, NOT PRODUCT.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s CPU-baseline /
`--impl reference` legs may import this module; the product path
(`dsac-v2_b200/`) never does and fails loudly without its CUDA library.

What it is: a restatement, in plain torch-CPU tensor algebra (fp32 by default,
fp64 on request), of what one `DSAC_V2.local_update(data, iteration)` of the
reference computes.  Each function cites the reference lines it follows
(paths relative to the reference checkout).  Gradients come from torch
autograd on the restated losses, exactly as the reference obtains them; the
Adam/Polyak arithmetic is written out by hand (the reference delegates it to
`torch.optim.Adam`, dsac_v2.py:54-59 — not vendored; formulas below are the
single-tensor path of torch 2.11 `optim/adam.py`).

Parity status: PINNED.  `tests/test_oracle_golden.py` checks this oracle
against fixtures produced by running the unmodified reference in the build
container (`tests/golden/make_golden.py`): all 14 deterministic `tb_info`
scalars for up to 100 consecutive updates, gradient and parameter digests, and
for the small cases every parameter of the post-update state.

Noise is an explicit input: `noise = [eps1[B,A], eps2[B,A], z1..z6[B]]`, the
eight standard-normal draws one update consumes (dsac_v2.py:160,228 and the
six `__q_evaluate` calls at :230,:231,:245,:249,:306,:307).
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence

import torch
import torch.nn.functional as F

EPS = 1e-6  # utils/act_distribution_cls.py:3
HUBER_DELTA = 50.0  # dsac_v2.py:282-287
STD_BIAS = 0.1  # dsac_v2.py:277
ADAM_B1, ADAM_B2, ADAM_EPS = 0.9, 0.999, 1e-8  # torch.optim.Adam defaults (dsac_v2.py:54-59)

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

_ACT = {
    "gelu": F.gelu,  # nn.GELU() exact erf, utils/common_utils.py:26-27
    "relu": F.relu,
    "elu": F.elu,
    "selu": F.selu,
    "sigmoid": torch.sigmoid,
    "tanh": torch.tanh,
    "linear": lambda x: x,
}


def mlp_forward(layers: Sequence[torch.Tensor], x: torch.Tensor, act: str, linear=F.linear) -> torch.Tensor:
    """networks/mlp.py:15-20 — Linear+act per hidden layer, Identity on the last.  `linear(x, W, b)`: the dense layer
    (tests/gradcheck_rounded.py restates it with the tensor-core kernels' bf16 operands)."""
    n = len(layers) // 2
    for j in range(n):
        x = linear(x, layers[2 * j], layers[2 * j + 1])
        if j < n - 1:
            x = _ACT[act](x)
    return x


def huber(x: torch.Tensor, y: torch.Tensor, delta: float = HUBER_DELTA) -> torch.Tensor:
    """torch.nn.functional.huber_loss(reduction='none') as used at dsac_v2.py:282-287."""
    d = x - y
    a = d.abs()
    return torch.where(a <= delta, 0.5 * d * d, delta * (a - 0.5 * delta))


class OracleDSACT:
    """State + one-update arithmetic of the reference's ApproxContainer/DSAC_V2."""

    NETS = ("q1", "q2", "policy")

    def __init__(self, obs_dim: int, act_dim: int, hidden_q, hidden_pi, act_high, act_low,
                 weights: Dict[str, "torch.Tensor"], *, gamma=0.99, tau=0.005, tau_b=None,
                 delay_update=2, auto_alpha=True, alpha=0.2, value_learning_rate=1e-4,
                 policy_learning_rate=1e-4, alpha_learning_rate=3e-4,
                 policy_min_log_std=-20.0, policy_max_log_std=0.5, hidden_activation="gelu",
                 value_hidden_activation=None, policy_hidden_activation=None,
                 policy_act_distribution="TanhGaussDistribution", dtype=torch.float32, linear=F.linear, **_ignored):
        self.O, self.A = int(obs_dim), int(act_dim)
        self.dtype = dtype
        self.linear = linear   # every dense layer of every network (mlp_forward); F.linear is the reference's nn.Linear
        # critics / policy: the reference's value_* / policy_* kwargs, else `hidden_activation` for both networks
        self.act_q = value_hidden_activation or hidden_activation
        self.act_pi = policy_hidden_activation or hidden_activation
        assert policy_act_distribution in ("TanhGaussDistribution", "GaussDistribution")
        self.gauss_only = policy_act_distribution == "GaussDistribution"   # utils/act_distribution_cls.py:82-116
        self.gamma, self.tau = float(gamma), float(tau)
        self.tau_b = float(tau if tau_b is None else tau_b)  # dsac_v2.py:90
        self.delay_update = int(delay_update)
        self.auto_alpha, self.alpha_fixed = bool(auto_alpha), float(alpha)
        self.target_entropy = -float(act_dim)  # dsac_v2.py:84
        self.lr = {"q1": value_learning_rate, "q2": value_learning_rate,
                   "policy": policy_learning_rate, "log_alpha": alpha_learning_rate}
        self.min_log_std, self.max_log_std = float(policy_min_log_std), float(policy_max_log_std)
        self.hi = torch.as_tensor(act_high, dtype=dtype).reshape(-1)
        self.lo = torch.as_tensor(act_low, dtype=dtype).reshape(-1)
        self._load_weights(weights, len(hidden_q) + 1, len(hidden_pi) + 1)
        la = weights.get("log_alpha", 1.0)  # dsac_v2.py:51
        self.log_alpha = torch.as_tensor(la, dtype=dtype).reshape(()).clone()
        for group in self.p.values():
            for w in group:
                w.requires_grad_(True)
        self.log_alpha.requires_grad_(True)
        # Adam state (exp_avg, exp_avg_sq, step) per optimizer, dsac_v2.py:54-59
        self.m = {k: [torch.zeros_like(w) for w in v] for k, v in self.p.items()}
        self.v = {k: [torch.zeros_like(w) for w in v] for k, v in self.p.items()}
        self.m["log_alpha"], self.v["log_alpha"] = [torch.zeros((), dtype=dtype)], [torch.zeros((), dtype=dtype)]
        self.steps = {"q1": 0, "q2": 0, "policy": 0, "log_alpha": 0}
        self.mean_std = [None, None]  # dsac_v2.py:88-89 (-1.0 sentinel)
        self.grads: Dict[str, List[torch.Tensor]] = {}
        self.device = torch.device("cpu")

    def to(self, device) -> "OracleDSACT":
        """Move every tensor of the state to `device`.  The same ATen ops then run there: on a CUDA device this is what
        the reference's eager PyTorch path does on that GPU (bench.py's `cuda_eager_baseline` leg); parity tests stay on CPU."""
        self.device = torch.device(device)
        mv = lambda w: w.detach().to(self.device).requires_grad_(w.requires_grad)
        self.p = {k: [mv(w) for w in v] for k, v in self.p.items()}
        self.t = {k: [mv(w) for w in v] for k, v in self.t.items()}
        self.m = {k: [mv(w) for w in v] for k, v in self.m.items()}
        self.v = {k: [mv(w) for w in v] for k, v in self.v.items()}
        self.log_alpha, self.hi, self.lo = mv(self.log_alpha), mv(self.hi), mv(self.lo)
        self.mean_std = [None if x is None else x.to(self.device) for x in self.mean_std]
        return self

    def _load_weights(self, weights, nq, npi):
        """Parameter lists per network, in the reference's named_parameters order."""
        inner = {"q1": "q", "q2": "q", "policy": "policy"}

        def grab(net, n_layers):
            out = []
            for j in range(n_layers):
                for leaf in ("weight", "bias"):
                    w = weights[f"{net}.{inner[net.replace('_target', '')]}.{2 * j}.{leaf}"]
                    out.append(torch.as_tensor(w).detach().clone().to(self.dtype))
            return out

        self.p = {"q1": grab("q1", nq), "q2": grab("q2", nq), "policy": grab("policy", npi)}
        self.t = {"q1": grab("q1_target", nq), "q2": grab("q2_target", nq),
                  "policy": grab("policy_target", npi)}

    # ---- network pieces -------------------------------------------------
    def policy_logits(self, layers, obs):
        """StochaPolicy.forward, std_type='mlp_shared' (networks/mlp.py:85-100)."""
        out = mlp_forward(layers, obs, self.act_pi, self.linear)
        mean, log_std = torch.chunk(out, 2, dim=-1)
        return mean, torch.clamp(log_std, self.min_log_std, self.max_log_std).exp()

    def q_dist(self, layers, obs, act):
        """ActionValueDistri.forward (networks/mlp.py:122-127): mean, softplus(std)."""
        out = mlp_forward(layers, torch.cat([obs, act], dim=-1), self.act_q, self.linear)
        return out[..., 0], F.softplus(out[..., 1])

    def tanh_gauss_rsample(self, mean, std, eps):
        """TanhGaussDistribution.rsample (utils/act_distribution_cls.py:44-54); GaussDistribution.rsample (:97-100) when
        the policy's action distribution is the plain Gaussian (no squashing, no limits in the update)."""
        u = mean + std * eps
        gauss = (-((u - mean) ** 2) / (2 * std ** 2) - std.log() - math.log(math.sqrt(2 * math.pi))).sum(-1)
        if self.gauss_only:
            return u, gauss
        t = torch.tanh(u)
        scale, shift = (self.hi - self.lo) / 2, (self.hi + self.lo) / 2
        logp = gauss - torch.log(1 + EPS - t.pow(2)).sum(-1) - torch.log(scale).sum(-1)
        return scale * t + shift, logp

    def alpha(self) -> float:
        """__get_alpha(requires_grad=False), dsac_v2.py:140-148."""
        return float(self.log_alpha.detach().exp()) if self.auto_alpha else self.alpha_fixed

    # ---- one update -----------------------------------------------------
    def compute_gradients(self, batch: Dict[str, torch.Tensor], noise, *, global_batch=None,
                          std_sum_hook=None) -> Dict[str, float]:
        """__compute_gradient (dsac_v2.py:150-206) with explicit noise.

        `global_batch` / `std_sum_hook` restate the same arithmetic for a data-parallel shard
        (SURVEY.md §8e): batch means become sums over the local rows divided by the global row
        count, and the two critic-std sums pass through the hook (an all-reduce) before the
        mean_std EMA.  With the defaults this is exactly the single-process update."""
        c = lambda x: torch.as_tensor(x).to(device=self.device, dtype=self.dtype)
        obs, act, rew, obs2, done = (c(batch[k]) for k in ("obs", "act", "rew", "obs2", "done"))
        eps1, eps2, _z1, _z2, z3, z4 = (c(n) for n in noise[:6])
        B = obs.shape[0]
        GB = B if global_batch is None else int(global_batch)
        gmean = (lambda x: x.mean()) if GB == B else (lambda x: x.sum() / GB)
        P, T = self.p, self.t
        alpha = self.alpha()

        # actor sample (dsac_v2.py:154-161)
        mean, std = self.policy_logits(P["policy"], obs)
        new_act, new_logp = self.tanh_gauss_rsample(mean, std, eps1)

        # ---- critic loss (__compute_loss_q, dsac_v2.py:218-290)
        with torch.no_grad():
            mean2, std2 = self.policy_logits(T["policy"], obs2)
            act2, logp2 = self.tanh_gauss_rsample(mean2, std2, eps2)
        q1, s1 = self.q_dist(P["q1"], obs, act)
        q2, s2 = self.q_dist(P["q2"], obs, act)
        sums = [s1.detach().sum(), s2.detach().sum()]
        if std_sum_hook is not None:
            sums = std_sum_hook(sums)
        for k, s in enumerate((s1, s2)):  # dsac_v2.py:233-241
            batch_mean = s.detach().mean() if (GB == B and std_sum_hook is None) else sums[k] / GB
            self.mean_std[k] = batch_mean if self.mean_std[k] is None else \
                (1 - self.tau_b) * self.mean_std[k] + self.tau_b * batch_mean
        with torch.no_grad():
            q1n, s1n = self.q_dist(T["q1"], obs2, act2)
            q2n, s2n = self.q_dist(T["q2"], obs2, act2)
            q1n_s = q1n + torch.clamp(z3, -3, 3) * s1n  # __q_evaluate, dsac_v2.py:208-216
            q2n_s = q2n + torch.clamp(z4, -3, 3) * s2n
            qn = torch.min(q1n, q2n)
            qn_s = torch.where(q1n < q2n, q1n_s, q2n_s)  # dsac_v2.py:252-253
            # __compute_target_q, dsac_v2.py:292-302
            y = rew + (1 - done) * self.gamma * (qn - alpha * logp2)
            y_s = rew + (1 - done) * self.gamma * (qn_s - alpha * logp2)
        loss_q = 0.0
        for q, s, m in ((q1, s1, self.mean_std[0]), (q2, s2, self.mean_std[1])):
            qd = q.detach()
            yb = qd + torch.clamp(y_s - qd, -3 * m, 3 * m)
            sd = torch.clamp(s, min=0.0).detach()
            ratio = (m.pow(2) / (sd.pow(2) + STD_BIAS)).clamp(min=0.1, max=10)  # dsac_v2.py:279-280
            loss_q = loss_q + gmean(ratio * (huber(q, y) + s * (sd.pow(2) - huber(qd, yb)) / (sd + STD_BIAS)))
        gq = torch.autograd.grad(loss_q, P["q1"] + P["q2"])
        n1 = len(P["q1"])
        self.grads = {"q1": list(gq[:n1]), "q2": list(gq[n1:])}

        # ---- actor loss (__compute_loss_policy, dsac_v2.py:304-310); no grad to Q params (:168-181)
        q1p, _ = self.q_dist([w.detach() for w in P["q1"]], obs, new_act)
        q2p, _ = self.q_dist([w.detach() for w in P["q2"]], obs, new_act)
        loss_pi = gmean(alpha * new_logp - torch.min(q1p, q2p))
        self.grads["policy"] = list(torch.autograd.grad(loss_pi, P["policy"]))
        entropy = -new_logp.detach().mean()

        # ---- temperature loss (__compute_loss_alpha, dsac_v2.py:312-318)
        if self.auto_alpha:
            loss_alpha = -self.log_alpha * gmean(new_logp.detach() + self.target_entropy)
            self.grads["log_alpha"] = list(torch.autograd.grad(loss_alpha, [self.log_alpha]))

        vals = [q1.detach().mean(), q2.detach().mean(), s1.detach().mean(), s2.detach().mean(),
                s1.detach().min(), s2.detach().min(), loss_pi.detach(), loss_q.detach(),
                torch.tanh(mean).mean().detach(), std.mean().detach(), entropy, alpha,
                self.mean_std[0], self.mean_std[1]]  # dsac_v2.py:188-202
        return {k: float(v) for k, v in zip(TB_KEYS, vals)}

    def _adam(self, name, params, grads):
        """torch.optim.Adam single-tensor step (amsgrad/weight_decay off)."""
        self.steps[name] += 1
        t = self.steps[name]
        bc1, bc2 = 1 - ADAM_B1 ** t, 1 - ADAM_B2 ** t
        step_size, bc2_sqrt = self.lr[name] / bc1, math.sqrt(bc2)
        with torch.no_grad():
            for w, g, m, v in zip(params, grads, self.m[name], self.v[name]):
                m.lerp_(g, 1 - ADAM_B1)
                v.mul_(ADAM_B2).addcmul_(g, g, value=1 - ADAM_B2)
                denom = (v.sqrt() / bc2_sqrt).add_(ADAM_EPS)
                w.addcdiv_(m, denom, value=-step_size)

    def apply(self, iteration: int) -> None:
        """__update (dsac_v2.py:320-347)."""
        self._adam("q1", self.p["q1"], self.grads["q1"])
        self._adam("q2", self.p["q2"], self.grads["q2"])
        if iteration % self.delay_update == 0:
            self._adam("policy", self.p["policy"], self.grads["policy"])
            if self.auto_alpha:
                self._adam("log_alpha", [self.log_alpha], self.grads["log_alpha"])
            with torch.no_grad():
                polyak = 1 - self.tau
                for net in self.NETS:
                    for w, wt in zip(self.p[net], self.t[net]):
                        wt.mul_(polyak)
                        wt.add_((1 - polyak) * w)

    def update(self, batch, noise, iteration: int) -> Dict[str, float]:
        """local_update (dsac_v2.py:102-105)."""
        tb = self.compute_gradients(batch, noise)
        self.apply(iteration)
        return tb

    # ---- the whole state between two updates -----------------------------
    def _online_keys(self) -> Dict[str, List[str]]:
        """{net: the state_dict keys of its parameters, in the order of self.p[net]}."""
        sd = list(self.state_dict())
        return {net: [k for k in sd if k.startswith(net + ".")] for net in self.NETS}

    def load_state(self, params, m, v, mean_std, steps_q: int, steps_pi: int) -> None:
        """Replace the state one update starts from: `params` in the state_dict schema (online, `*_target` and
        log_alpha), the Adam moments `m` / `v` keyed like the online parameters plus "log_alpha", the carried mean_std
        pair (None or a negative value: unset, as dsac_v2.py:88-89) and the step counters of the critics' optimizers and
        of the policy and temperature optimizers (they step together, dsac_v2.py:327-333)."""
        c = lambda x: torch.as_tensor(x).detach().clone().to(device=self.device, dtype=self.dtype)
        for net, keys in self._online_keys().items():
            tkeys = [net + "_target" + k[len(net):] for k in keys]
            self.p[net] = [c(params[k]).requires_grad_(True) for k in keys]
            self.t[net] = [c(params[k]) for k in tkeys]
            self.m[net], self.v[net] = [c(m[k]) for k in keys], [c(v[k]) for k in keys]
            self.steps[net] = int(steps_pi if net == "policy" else steps_q)
        self.log_alpha = c(params["log_alpha"]).reshape(()).requires_grad_(True)
        self.m["log_alpha"], self.v["log_alpha"] = [c(m["log_alpha"]).reshape(())], [c(v["log_alpha"]).reshape(())]
        self.steps["log_alpha"] = int(steps_pi)
        self.mean_std = [None if x is None or float(x) < 0 else c(float(x)).reshape(()) for x in mean_std]

    def moments(self):
        """(m, v): the Adam moments in the schema `load_state` takes."""
        out = []
        for mv in (self.m, self.v):
            d = {k: mv[net][i].detach() for net, keys in self._online_keys().items() for i, k in enumerate(keys)}
            d["log_alpha"] = mv["log_alpha"][0].detach()
            out.append(d)
        return tuple(out)

    # ---- views in the reference's state_dict schema ----------------------
    def state_dict(self) -> Dict[str, torch.Tensor]:
        inner = {"q1": "q", "q2": "q", "policy": "policy"}
        out = {"log_alpha": self.log_alpha.detach()}
        for net in self.NETS:
            for group, suffix in ((self.p, ""), (self.t, "_target")):
                for i, w in enumerate(group[net]):
                    leaf = "weight" if i % 2 == 0 else "bias"
                    out[f"{net}{suffix}.{inner[net]}.{2 * (i // 2)}.{leaf}"] = w.detach()
        return out

    def grad_dict(self) -> Dict[str, torch.Tensor]:
        inner = {"q1": "q", "q2": "q", "policy": "policy"}
        out = {}
        for net in self.NETS:
            for i, g in enumerate(self.grads[net]):
                leaf = "weight" if i % 2 == 0 else "bias"
                out[f"{net}.{inner[net]}.{2 * (i // 2)}.{leaf}"] = g
        if "log_alpha" in self.grads:
            out["log_alpha"] = self.grads["log_alpha"][0]
        return out


class OracleDSACTStd(OracleDSACT):
    """The same update with the policy's other `std_type`s (reference networks/mlp.py:42-100; SURVEY.md §8f rank 4):
    "mlp_separated" — two MLPs `mean` and `log_std`; "parameter" — one MLP `mean` and a learnable row `log_std` [1, A]
    broadcast over the batch (:95-99).  Critics, losses, Adam and Polyak are inherited unchanged.

    Parity status: PINNED on `tests/golden/tiny_std_separated.npz` / `tiny_std_parameter.npz`.  No CUDA path yet."""

    def __init__(self, *args, std_type="mlp_separated", **hyper):
        assert std_type in ("mlp_separated", "parameter")
        self.std_type, self.names = std_type, {}
        super().__init__(*args, **hyper)

    def _load_weights(self, weights, nq, npi):
        super_w = dict(weights)
        # critics through the base schema; the policy by name, in the reference's named_parameters order:
        # "mlp_separated": mean.*, log_std.* (attribute order); "parameter": mean.*, then log_std (nn.Parameter set last)
        inner = {"q1": "q", "q2": "q"}

        def grab_q(net):
            return [torch.as_tensor(super_w[f"{net}.{inner[net.replace('_target', '')]}.{2 * j}.{leaf}"]).detach().clone().to(self.dtype)
                    for j in range(nq) for leaf in ("weight", "bias")]

        def grab_pi(net):
            keys = [k for k in weights if k.startswith(net + ".")]
            order = {"mean": 0, "log_std": 1}

            def rank(k):
                parts = k.split(".")
                return (order[parts[1]], int(parts[2]) if len(parts) > 2 else 0, len(parts) > 3 and parts[3] == "bias")
            keys.sort(key=rank)
            self.names["policy"] = [k[len(net) + 1:] for k in keys]
            return [torch.as_tensor(weights[k]).detach().clone().to(self.dtype) for k in keys]

        self.p = {"q1": grab_q("q1"), "q2": grab_q("q2"), "policy": grab_pi("policy")}
        self.t = {"q1": grab_q("q1_target"), "q2": grab_q("q2_target"), "policy": grab_pi("policy_target")}

    def policy_logits(self, layers, obs):
        w = dict(zip(self.names["policy"], layers))

        def head(name):
            ls, j = [], 0
            while f"{name}.{2 * j}.weight" in w:
                ls += [w[f"{name}.{2 * j}.weight"], w[f"{name}.{2 * j}.bias"]]
                j += 1
            return mlp_forward(ls, obs, self.act_pi, self.linear)

        mean = head("mean")
        log_std = head("log_std") if self.std_type == "mlp_separated" else w["log_std"] + torch.zeros_like(mean)
        return mean, torch.clamp(log_std, self.min_log_std, self.max_log_std).exp()

    def _named(self, net, group):
        if net == "policy":
            return list(zip(self.names["policy"], group))
        return [(f"q.{2 * (i // 2)}.{'weight' if i % 2 == 0 else 'bias'}", w) for i, w in enumerate(group)]

    def state_dict(self):
        out = {"log_alpha": self.log_alpha.detach()}
        for net in self.NETS:
            for group, suffix in ((self.p, ""), (self.t, "_target")):
                for name, w in self._named(net, group[net]):
                    out[f"{net}{suffix}.{name}"] = w.detach()
        return out

    def grad_dict(self):
        out = {}
        for net in self.NETS:
            for name, g in self._named(net, self.grads[net]):
                out[f"{net}.{name}"] = g
        if "log_alpha" in self.grads:
            out["log_alpha"] = self.grads["log_alpha"][0]
        return out


class OracleDSACTCNN(OracleDSACT):
    """The same update with the reference's CNN approximators (BASELINE config 5, SURVEY.md §8f rank 1): a private conv
    encoder per network (`CNN()`, networks/cnn.py:30-53, ReLU between convs) followed by two separate MLP heads `mean`
    and `log_std` (StochaPolicy networks/cnn.py:151-240; ActionValueDistri :383-461, which concatenates the action to
    the flattened feature, :455-456).  Loss, Adam and Polyak arithmetic are inherited unchanged.

    Parity status: PINNED on `tests/golden/cnn_carracing_b4.npz` (tests/test_oracle_golden.py).  No CUDA path yet."""

    def __init__(self, obs_dim, act_dim, conv_strides, act_high, act_low, weights, **hyper):
        self.conv_strides = tuple(int(x) for x in conv_strides)
        self.names = {}
        super().__init__(0, act_dim, (), (), act_high, act_low, weights, **hyper)
        self.O = tuple(obs_dim)

    def _load_weights(self, weights, nq, npi):
        order = {"conv": 0, "mean": 1, "log_std": 2}   # attribute order of the reference modules = named_parameters order

        def grab(net):
            keys = [k for k in weights if k.startswith(net + ".")]
            keys.sort(key=lambda k: (order[k.split(".")[1]], int(k.split(".")[2]), k.split(".")[3] == "bias"))
            self.names[net.replace("_target", "")] = [k[len(net) + 1:] for k in keys]
            return [torch.as_tensor(weights[k]).detach().clone().to(self.dtype) for k in keys]

        self.p = {n: grab(n) for n in self.NETS}
        self.t = {n: grab(n + "_target") for n in self.NETS}

    def _features(self, w, obs):
        x, j = obs, 0
        while f"conv.{2 * j}.weight" in w:   # Conv2d + ReLU per layer, networks/cnn.py:41-52
            x = F.relu(F.conv2d(x, w[f"conv.{2 * j}.weight"], w[f"conv.{2 * j}.bias"], stride=self.conv_strides[j]))
            j += 1
        return x.reshape(x.shape[0], -1)     # img.view(img.size(0), -1), networks/cnn.py:234-235

    def _head(self, w, head, x, act):
        layers, j = [], 0
        while f"{head}.{2 * j}.weight" in w:
            layers += [w[f"{head}.{2 * j}.weight"], w[f"{head}.{2 * j}.bias"]]
            j += 1
        return mlp_forward(layers, x, act, self.linear)

    def policy_logits(self, layers, obs):
        """StochaPolicy.forward (networks/cnn.py:233-240): mean head, exp(clamp(log_std head))."""
        w = dict(zip(self.names["policy"], layers))
        f = self._features(w, obs)
        return self._head(w, "mean", f, self.act_pi), \
            torch.clamp(self._head(w, "log_std", f, self.act_pi), self.min_log_std, self.max_log_std).exp()

    def q_dist(self, layers, obs, act):
        """ActionValueDistri.forward (networks/cnn.py:454-461): heads on cat(feature, act); softplus on the std head."""
        w = dict(zip(self.names["q1"], layers))
        f = torch.cat([self._features(w, obs), act], dim=-1)
        return self._head(w, "mean", f, self.act_q)[..., 0], F.softplus(self._head(w, "log_std", f, self.act_q)[..., 0])

    def state_dict(self):
        out = {"log_alpha": self.log_alpha.detach()}
        for net in self.NETS:
            for group, suffix in ((self.p, ""), (self.t, "_target")):
                for name, w in zip(self.names[net], group[net]):
                    out[f"{net}{suffix}.{name}"] = w.detach()
        return out

    def grad_dict(self):
        out = {}
        for net in self.NETS:
            for name, g in zip(self.names[net], self.grads[net]):
                out[f"{net}.{name}"] = g
        if "log_alpha" in self.grads:
            out["log_alpha"] = self.grads["log_alpha"][0]
        return out


def std_from_config(cfg: dict, weights: dict, std_type: str, **hyper) -> OracleDSACTStd:
    """Build from a `synth.CONFIGS` entry with weights of `synth.make_weights_std`."""
    lim = [cfg["act_lim"]] * cfg["act_dim"]
    return OracleDSACTStd(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], lim, [-x for x in lim], weights,
                          std_type=std_type, **hyper)


def cnn_from_config(cfg: dict, weights: dict, **hyper) -> OracleDSACTCNN:
    """Build from a `synth.CNN_CONFIGS` entry."""
    from dsac_v2_b200.synth import CONV_TYPES
    lim = [cfg["act_lim"]] * cfg["act_dim"]
    return OracleDSACTCNN(cfg["obs_dim"], cfg["act_dim"], CONV_TYPES[cfg["conv_type"]]["strides"], lim, [-x for x in lim],
                          weights, **hyper)


def from_config(cfg: dict, weights: dict, **hyper) -> OracleDSACT:
    """Build from a `synth.CONFIGS` or `synth.ASYM_CONFIGS` entry (+ `synth.HYPER`-style overrides).  The networks'
    activations are the config's unless the overrides name `hidden_activation` (both networks) or the reference's
    `value_hidden_activation` / `policy_hidden_activation`."""
    from dsac_v2_b200.synth import activations, hidden_sizes
    lim = [cfg["act_lim"]] * cfg["act_dim"]
    if "hidden_activation" not in hyper:
        act_q, act_pi = activations(cfg)
        hyper = dict(dict(value_hidden_activation=act_q, policy_hidden_activation=act_pi), **hyper)
    return OracleDSACT(cfg["obs_dim"], cfg["act_dim"], *hidden_sizes(cfg), lim, [-x for x in lim], weights, **hyper)


# ---- DSAC_V1 (reference dsac_v1.py; SURVEY.md §8f rank 4): one critic, fixed TD bound ---------------------------------
V1_TB_KEYS = [
    "DSAC/critic_avg_q-RL iter",
    "DSAC/critic_avg_std-RL iter",
    "Loss/Actor loss-RL iter",
    "DSAC/policy_mean-RL iter",
    "DSAC/policy_std-RL iter",
    "DSAC/entropy-RL iter",
    "DSAC/alpha-RL iter",
]
V1_STD_BIAS = 0.1  # dsac_v1.py:224


class OracleDSACV1(OracleDSACT):
    """State + one-update arithmetic of the reference's older algorithm (`dsac_v1.ApproxContainer` :17-52, `DSAC_V1` :56-273):
    networks q, q_target, policy, policy_target (the same MLP classes as DSAC-T, std_type mlp_shared) + log_alpha."""

    NETS = ("q", "policy")

    def __init__(self, *args, TD_bound=20.0, bound=True, **hyper):
        self.TD_bound, self.bound = float(TD_bound), bool(bound)
        super().__init__(*args, **hyper)
        self.lr = {"q": self.lr["q1"], "policy": self.lr["policy"], "log_alpha": self.lr["log_alpha"]}
        self.steps = {"q": 0, "policy": 0, "log_alpha": 0}

    def _load_weights(self, weights, nq, npi):
        inner = {"q": "q", "policy": "policy"}

        def grab(net, n_layers):
            out = []
            for j in range(n_layers):
                for leaf in ("weight", "bias"):
                    w = weights[f"{net}.{inner[net.replace('_target', '')]}.{2 * j}.{leaf}"]
                    out.append(torch.as_tensor(w).detach().clone().to(self.dtype))
            return out

        self.p = {"q": grab("q", nq), "policy": grab("policy", npi)}
        self.t = {"q": grab("q_target", nq), "policy": grab("policy_target", npi)}

    def compute_gradients(self, batch, noise, **_unused) -> Dict[str, float]:
        """__compute_gradient (dsac_v1.py:137-183).  `noise` = (eps1, eps2, z_q, z_next, z_pi): the normal draws in the
        reference's order; only z_next enters the arithmetic (the other two samples are computed and dropped there)."""
        c = lambda x: torch.as_tensor(x).to(device=self.device, dtype=self.dtype)
        obs, act, rew, obs2, done = (c(batch[k]) for k in ("obs", "act", "rew", "obs2", "done"))
        eps1, eps2, z_next = c(noise[0]), c(noise[1]), c(noise[3])
        P, T = self.p, self.t
        alpha = self.alpha()
        mean, std = self.policy_logits(P["policy"], obs)
        logits = torch.cat((mean, std), dim=-1)
        new_act, new_logp = self.tanh_gauss_rsample(mean, std, eps1)
        # __compute_loss_q (dsac_v1.py:195-233)
        with torch.no_grad():
            mean2, std2 = self.policy_logits(T["policy"], obs2)
            act2, logp2 = self.tanh_gauss_rsample(mean2, std2, eps2)
            qn, sn = self.q_dist(T["q"], obs2, act2)
            qn_s = qn + torch.clamp(z_next, -3, 3) * sn                      # __q_evaluate :185-193
        q, s = self.q_dist(P["q"], obs, act)
        with torch.no_grad():                                                # __compute_target_q :235-241
            target = rew + (1 - done) * self.gamma * (qn_s - alpha * logp2)
            target_bound = q.detach() + torch.clamp(target - q.detach(), -self.TD_bound, self.TD_bound)
        if self.bound:
            sd = torch.clamp(s, min=0.0).detach()
            loss_q = torch.mean(-(target - q).detach() / (sd.pow(2) + V1_STD_BIAS) * q
                                - ((q.detach() - target_bound).pow(2) - sd.pow(2)) / (sd.pow(3) + V1_STD_BIAS) * s)
        else:
            loss_q = -torch.distributions.Normal(q, s).log_prob(target).mean()
        self.grads = {"q": list(torch.autograd.grad(loss_q, P["q"]))}
        # __compute_loss_policy (:243-248); the critic is frozen (:155-163)
        qp, _ = self.q_dist([w.detach() for w in P["q"]], obs, new_act)
        loss_pi = (alpha * new_logp - qp).mean()
        self.grads["policy"] = list(torch.autograd.grad(loss_pi, P["policy"]))
        entropy = -new_logp.detach().mean()
        if self.auto_alpha:                                                  # __compute_loss_alpha :250-256
            loss_alpha = -self.log_alpha * (new_logp.detach() + self.target_entropy).mean()
            self.grads["log_alpha"] = list(torch.autograd.grad(loss_alpha, [self.log_alpha]))
        # tb_info (:172-181); policy_mean / policy_std index the LOGITS at [..., 0] and [..., 1] (:142-143)
        vals = [q.detach().mean(), s.detach().mean(), loss_pi.detach(), torch.tanh(logits[..., 0]).mean().detach(),
                logits[..., 1].mean().detach(), entropy, alpha]
        return {k: float(v) for k, v in zip(V1_TB_KEYS, vals)}

    def apply(self, iteration: int) -> None:
        """__update (dsac_v1.py:258-273)."""
        self._adam("q", self.p["q"], self.grads["q"])
        if iteration % self.delay_update == 0:
            self._adam("policy", self.p["policy"], self.grads["policy"])
            if self.auto_alpha:
                self._adam("log_alpha", [self.log_alpha], self.grads["log_alpha"])
            with torch.no_grad():
                polyak = 1 - self.tau
                for net in self.NETS:
                    for w, wt in zip(self.p[net], self.t[net]):
                        wt.mul_(polyak)
                        wt.add_((1 - polyak) * w)

    def state_dict(self) -> Dict[str, torch.Tensor]:
        inner = {"q": "q", "policy": "policy"}
        out = {"log_alpha": self.log_alpha.detach()}
        for net in self.NETS:
            for group, suffix in ((self.p, ""), (self.t, "_target")):
                for i, w in enumerate(group[net]):
                    leaf = "weight" if i % 2 == 0 else "bias"
                    out[f"{net}{suffix}.{inner[net]}.{2 * (i // 2)}.{leaf}"] = w.detach()
        return out

    def grad_dict(self) -> Dict[str, torch.Tensor]:
        inner = {"q": "q", "policy": "policy"}
        out = {}
        for net in self.NETS:
            for i, g in enumerate(self.grads[net]):
                leaf = "weight" if i % 2 == 0 else "bias"
                out[f"{net}.{inner[net]}.{2 * (i // 2)}.{leaf}"] = g
        if "log_alpha" in self.grads:
            out["log_alpha"] = self.grads["log_alpha"][0]
        return out


def v1_from_config(cfg: dict, weights: dict, **hyper) -> OracleDSACV1:
    """Build from a `synth.CONFIGS` entry with weights of `synth.make_weights_v1`."""
    lim = [cfg["act_lim"]] * cfg["act_dim"]
    return OracleDSACV1(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], cfg["hidden"], lim, [-x for x in lim], weights, **hyper)
