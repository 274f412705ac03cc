"""The drop-in's engine choice, `dsact_route.route(algorithm, kwargs)`, row by row of INTEGRATION.md §2's "Which engine a
configuration lands on": the engine, the config struct fields of the table's third column, the `dsact_v1_options`,
whether `engine(batch)` may regrow the engine, and every configuration the containers refuse.  No GPU: configs only."""
import pytest

from dsac_v2_b200 import _lib, synth

RAGGED, ASYM, TINY = synth.CONFIGS["ragged"], synth.ASYM_CONFIGS["asym"], synth.CONFIGS["tiny"]
T1, T2 = synth.CNN_CONFIGS["small_t1"], synth.CNN_CONFIGS["carracing"]


def _mlp(cfg, alg="DSAC_V2", **over):
    return alg, synth.reference_kwargs(cfg, algorithm=alg, replay_batch_size=4, **over)


def _cnn(cfg, alg="DSAC_V2", **over):
    return alg, synth.cnn_reference_kwargs(cfg, algorithm=alg, replay_batch_size=4, **over)


def _conv(cfg):
    t = synth.CONV_TYPES[cfg["conv_type"]]
    return dict(n_conv=len(t["kernels"]), conv_kernel=t["kernels"], conv_channels=t["channels"], conv_stride=t["strides"],
                channels=cfg["obs_dim"][0], height=cfg["obs_dim"][1], width=cfg["obs_dim"][2], hidden=t["heads"])


def _heads(cfg):
    return dict(n_conv=0, channels=cfg["obs_dim"], height=1, width=1, q_heads=1, hidden=cfg["hidden"])


# (id, (algorithm, kwargs), engine, config fields, dsact_v1_options (bound, td_bound) or None, regrow)
ROWS = [
    # MLP networks, policy_std_type "mlp_shared": the MLP engine, bf16x3 unless dsact_gemm names another arithmetic
    ("v2_mlp_shared", _mlp(RAGGED), "mlp", dict(gemm_mode=1, act_dist=0, policy_std=0, use_graph=1), None, True),
    ("v2_mlp_shared_gauss_fp32", _mlp(RAGGED, policy_act_distribution="GaussDistribution", dsact_gemm="fp32"), "mlp",
     dict(gemm_mode=0, act_dist=1, policy_std=0), None, True),
    ("v2_mlp_shared_asym_bf16", _mlp(ASYM, dsact_gemm="bf16", dsact_graph=False), "mlp",
     dict(gemm_mode=2, n_hidden_q=6, n_hidden_pi=1, act_q=_lib.ACTIVATIONS["elu"], act_pi=_lib.ACTIVATIONS["tanh"],
          use_graph=0), None, True),
    ("v2_mlp_shared_tau_b", _mlp(RAGGED, tau_b=0.25), "mlp", dict(tau=0.005, tau_b=0.25), None, True),
    # CNN networks: the head-wise engine with the encoder; dsact_gemm is ignored
    ("v2_cnn_type1", _cnn(T1), "cnn", dict(_conv(T1), q_heads=2, pi_std=0, algo=0), None, False),
    ("v2_cnn_type2_gemm", _cnn(T2, dsact_gemm="bf16", tau_b=0.25), "cnn", dict(_conv(T2), q_heads=2, pi_std=0, tau_b=0.25),
     None, False),
    # MLP networks, the other std types: the head-wise engine without an encoder ...
    ("v2_separated", _mlp(RAGGED, policy_std_type="mlp_separated"), "heads", dict(_heads(RAGGED), pi_std=0, algo=0), None,
     False),
    ("v2_parameter", _mlp(RAGGED, policy_std_type="parameter", tau_b=0.25), "heads", dict(_heads(RAGGED), pi_std=1, tau_b=0.25),
     None, False),
    # ... or, with dsact_gemm, the MLP engine (critics and policy may differ)
    ("v2_separated_gemm", _mlp(ASYM, policy_std_type="mlp_separated", dsact_gemm="fp32"), "mlp",
     dict(policy_std=1, gemm_mode=0, n_hidden_q=6, n_hidden_pi=1), None, True),
    ("v2_parameter_gemm", _mlp(RAGGED, policy_std_type="parameter", dsact_gemm="bf16x3"), "mlp", dict(policy_std=2, gemm_mode=1),
     None, True),
    # DSAC_V1: the head-wise engine for every approximator; tau_b stays tau; cnn_shared is not read
    ("v1_mlp_shared", _mlp(RAGGED, "DSAC_V1", tau_b=0.25, cnn_shared=True), "heads",
     dict(_heads(RAGGED), pi_std=2, algo=1, v1_bound=1, td_bound=20.0, tau_b=0.005), None, False),
    ("v1_separated", _mlp(RAGGED, "DSAC_V1", policy_std_type="mlp_separated"), "heads", dict(_heads(RAGGED), pi_std=0, algo=1),
     None, False),
    ("v1_parameter_nll", _mlp(RAGGED, "DSAC_V1", policy_std_type="parameter", bound=False, TD_bound=3.5), "heads",
     dict(_heads(RAGGED), pi_std=1, algo=1, v1_bound=0, td_bound=3.5), None, False),
    ("v1_cnn_type1", _cnn(T1, "DSAC_V1"), "cnn", dict(_conv(T1), q_heads=2, pi_std=0, algo=1), None, False),
    ("v1_cnn_type2_gauss", _cnn(T2, "DSAC_V1", policy_act_distribution="GaussDistribution"), "cnn",
     dict(_conv(T2), act_dist=1, algo=1), None, False),
    # DSAC_V1 + dsact_gemm: the MLP engine (dsact_v1_create), critic and policy may differ
    ("v1_gemm", _mlp(RAGGED, "DSAC_V1", dsact_gemm="bf16x3", tau_b=0.25), "mlp", dict(gemm_mode=1, policy_std=0, tau_b=0.005),
     (1, 20.0), False),
    ("v1_gemm_asym_nll", _mlp(ASYM, "DSAC_V1", dsact_gemm="fp32", bound=False, TD_bound=3.5), "mlp",
     dict(gemm_mode=0, n_hidden_q=6, n_hidden_pi=1), (0, 3.5), False),
]


@pytest.mark.parametrize("row", ROWS, ids=[r[0] for r in ROWS])
def test_route_table(row):
    import dsac_v1
    import dsac_v2
    from dsact_route import route
    _, (alg, kw), engine, fields, v1, regrow = row
    r = route(alg, kw)
    assert (r.engine, r.regrow) == (engine, regrow)
    assert r.out_acts == ("linear", "linear")
    for mb in (4, 300):
        c = r.config(mb)
        assert isinstance(c, _lib.Config if engine == "mlp" else _lib.CnnConfig) and c.max_batch == mb
        for k, want in fields.items():
            got = getattr(c, k)
            got = list(got)[:len(want)] if isinstance(want, tuple) else got
            assert got == (list(want) if isinstance(want, tuple) else want), k
    assert (r.v1 is None) == (v1 is None)
    if v1 is not None:
        assert (r.v1.abi_version, r.v1.bound, r.v1.td_bound) == (_lib.ABI_VERSION, *v1)
    net = (dsac_v1 if alg == "DSAC_V1" else dsac_v2).ApproxContainer(**kw)   # the container takes this route
    assert net.route.engine == r.engine and net.route.cfg_args == r.cfg_args and bytes(net.route.config(4)) == bytes(r.config(4))


def test_route_takes_the_output_activations():
    from dsact_route import route
    for alg in ("DSAC_V2", "DSAC_V1"):
        _, kw = _mlp(TINY, alg, value_output_activation="relu", policy_output_activation="sigmoid")
        assert route(alg, kw).out_acts == ("relu", "sigmoid")


def test_v2_checks_dsact_gemm_only_when_it_builds_the_config():
    from dsact_route import route
    r = route(*_mlp(TINY, dsact_gemm="bogus"))
    assert r.engine == "mlp"
    with pytest.raises(KeyError):
        r.config(4)
    assert route(*_cnn(T1, dsact_gemm="bogus")).engine == "cnn"   # CNN networks ignore it


OtherDist = type("OtherDist", (), {})

# (id, (algorithm, kwargs), exception type, message fragment); the cases that fail two checks pin which one comes first
REFUSALS = [
    ("v2_cnn_shared", _mlp(TINY, cnn_shared=True, value_func_type="CNN"), NotImplementedError, "cnn_shared"),
    ("v2_apprfunc_mismatch", _mlp(TINY, value_func_type="CNN", value_conv_type="type_1"), NotImplementedError, "same type"),
    ("v1_apprfunc_mismatch", _mlp(TINY, "DSAC_V1", value_func_type="CNN", value_conv_type="type_1", dsact_gemm="fp32"),
     NotImplementedError, "same type"),
    ("v2_unknown_class", _mlp(TINY, value_func_name="Nope"), NotImplementedError, "not properly defined"),
    ("v1_unknown_class", _cnn(T1, "DSAC_V1", policy_func_name="Nope"), NotImplementedError, "not properly defined"),
    ("v2_distribution", _cnn(T1, policy_act_distribution=OtherDist, policy_conv_type="type_2"), NotImplementedError,
     "implements TanhGaussDistribution and GaussDistribution"),
    ("v1_distribution", _mlp(TINY, "DSAC_V1", policy_act_distribution=OtherDist, dsact_gemm="bogus"), NotImplementedError,
     "implements TanhGaussDistribution and GaussDistribution"),
    ("v2_cnn_conv_type", _cnn(T2, policy_conv_type="type_1", dsact_gemm="fp32"), NotImplementedError,
     "one conv_type / head activation"),
    ("v2_cnn_activation", _cnn(T1, policy_hidden_activation="tanh"), NotImplementedError, "one conv_type / head activation"),
    ("v2_heads_hidden_sizes", _mlp(ASYM, policy_std_type="parameter", policy_hidden_activation="elu"), NotImplementedError,
     "one hidden_sizes / activation"),
    ("v2_heads_activation", _mlp(RAGGED, policy_std_type="mlp_separated", policy_hidden_activation="tanh"), NotImplementedError,
     "one hidden_sizes / activation"),
    ("v1_heads_activation", _cnn(T1, "DSAC_V1", policy_hidden_activation="tanh", policy_conv_type="type_2"),
     NotImplementedError, "one hidden activation for critic and policy"),
    ("v1_cnn_conv_type", _cnn(T1, "DSAC_V1", policy_conv_type="type_2"), NotImplementedError,
     "one conv_type for critic and policy"),
    ("v1_heads_hidden_sizes", _mlp(ASYM, "DSAC_V1", policy_hidden_activation="elu"), NotImplementedError,
     "one hidden_sizes list"),
    ("v1_gemm_cnn", _cnn(T1, "DSAC_V1", dsact_gemm="bogus", policy_conv_type="type_2"), NotImplementedError, "'mlp_shared'"),
    ("v1_gemm_separated", _mlp(ASYM, "DSAC_V1", policy_std_type="mlp_separated", dsact_gemm="fp32"), NotImplementedError,
     "'mlp_shared'"),
    ("v1_gemm_parameter", _mlp(RAGGED, "DSAC_V1", policy_std_type="parameter", dsact_gemm="bf16"), NotImplementedError,
     "'mlp_shared'"),
    ("v1_gemm_unknown", _mlp(ASYM, "DSAC_V1", dsact_gemm="bogus"), ValueError, "dsact_gemm must be one of"),
]


@pytest.mark.parametrize("case", REFUSALS, ids=[c[0] for c in REFUSALS])
def test_route_refusals(case):
    from dsact_route import route
    _, (alg, kw), exc, fragment = case
    with pytest.raises(exc) as e:
        route(alg, kw)
    assert fragment in str(e.value)


@pytest.mark.parametrize("case", [c for c in REFUSALS if c[0] in ("v2_cnn_shared", "v1_unknown_class", "v2_cnn_conv_type",
                                                                   "v1_heads_hidden_sizes", "v1_gemm_unknown")],
                         ids=lambda c: c[0])
def test_containers_refuse_with_the_routes_checks(case):
    import dsac_v1
    import dsac_v2
    _, (alg, kw), exc, fragment = case
    with pytest.raises(exc, match=fragment):
        (dsac_v1 if alg == "DSAC_V1" else dsac_v2).ApproxContainer(**kw)
