"""CPU checks of DSAC_V1 on the MLP engine (`dsact_v1_query_layout`, no GPU needed): the flat layout is the drop-in
`dsac_v1.ApproxContainer(dsact_gemm=...)`'s parameter order and sizes and what `Engine._schema` walks; the workspace slots;
the validation of the DSAC_V1 options; the oracle pinned to the reference's DSAC_V1 goldens of the MLP engine's shapes."""
import ctypes as C

import numpy as np
import pytest
import torch

from dsac_v2_b200 import _lib, synth
from dsac_v2_b200.engine import Engine, make_config, make_v1_options, query_layout
from test_abi import _check_slots
from v1_mlp_common import NEW_GOLDENS, engine_config, golden, v1_oracle

MLP_CONFIGS = list(synth.CONFIGS) + list(synth.ASYM_CONFIGS)


def _container(name, gemm):
    import dsac_v1
    cfg = synth.mlp_config(name)
    return dsac_v1.ApproxContainer(**synth.reference_kwargs(cfg, algorithm="DSAC_V1", replay_batch_size=4, dsact_gemm=gemm))


@pytest.mark.parametrize("mode", list(_lib.GEMM_MODES))
@pytest.mark.parametrize("name", MLP_CONFIGS)
def test_v1_layout_matches_the_dropin_module(name, mode):
    cfg = synth.mlp_config(name)
    net = _container(name, mode)
    train, targ = net._flat_groups()

    class Probe:   # _schema only reads the config and whether the handle is DSAC_V1
        cfg = None
        v1 = make_v1_options()
    for mb in (1, 256, 1000):
        c, v1 = engine_config(cfg, mb, synth.HYPER, mode)
        lay = query_layout(c, v1)
        assert lay.n_params == sum(p.numel() for p in train) and lay.n_targets == sum(p.numel() for p in targ)
        assert lay.n_params == lay.n_q + lay.n_pi + 1 and lay.n_targets == lay.n_q + lay.n_pi
        Probe.cfg = c
        schema, n = Engine._schema(Probe)
        assert n == lay.n_targets
        names = [k for k, p in net.named_parameters() if p.requires_grad and k != "log_alpha"]
        assert [e[0] for e in schema] == names
        sizes = dict(net.named_parameters())
        assert all(tuple(sizes[e[0]].shape) == tuple(e[4]) and sizes[e[0]].numel() == e[3] for e in schema)
        assert [e[1] for e in schema] == [k for k, p in net.named_parameters() if not p.requires_grad]
        off = 0
        for e in schema:
            assert e[2] == off
            off += e[3]


@pytest.mark.parametrize("mode", list(_lib.GEMM_MODES))
@pytest.mark.parametrize("name", MLP_CONFIGS)
def test_v1_workspace_slots(name, mode):
    cfg = synth.mlp_config(name)
    for mb in (1, 256, 1000):
        c, v1 = engine_config(cfg, mb, synth.HYPER, mode)
        lay = query_layout(c, v1)
        _check_slots(lay, cfg["act_dim"], mode != "fp32")
        # one critic: a smaller arena than the DSAC-T handle of the same networks
        assert lay.workspace_bytes < query_layout(c).workspace_bytes


def test_v1_options_are_validated_with_a_message():
    lib = _lib.load()
    c = make_config(5, 2, [8], [8], max_batch=4)
    out = _lib.Layout()
    h = C.c_void_p()
    for mutate in (lambda v: setattr(v, "bound", 2), lambda v: setattr(v, "bound", -1), lambda v: setattr(v, "td_bound", 0.0),
                   lambda v: setattr(v, "td_bound", -1.0), lambda v: setattr(v, "td_bound", float("nan")),
                   lambda v: setattr(v, "td_bound", float("inf")), lambda v: setattr(v, "abi_version", 99)):
        v = make_v1_options(True, 10.0)
        mutate(v)
        assert lib.dsact_v1_query_layout(C.byref(c), C.byref(v), C.byref(out)) == -1
        assert lib.dsact_last_error()
        # rejected before any device is touched
        assert lib.dsact_v1_create(C.byref(c), C.byref(v), 0, C.byref(h)) == -1
        assert lib.dsact_last_error()
    assert lib.dsact_v1_query_layout(C.byref(c), None, C.byref(out)) == -1
    bad = make_config(5, 2, [8], [8], max_batch=4)
    bad.max_batch = 0
    assert lib.dsact_v1_query_layout(C.byref(bad), C.byref(make_v1_options()), C.byref(out)) == -1
    assert lib.dsact_v1_query_layout(C.byref(c), C.byref(make_v1_options(False, 0.5)), C.byref(out)) == 0


@pytest.mark.parametrize("kw", [dict(value_func_type="CNN", policy_func_type="CNN"), dict(policy_std_type="mlp_separated"),
                                dict(policy_std_type="parameter")])
def test_dsact_gemm_refuses_what_the_mlp_engine_does_not_run(kw):
    import dsac_v1
    cfg = synth.CONFIGS["tiny"]
    if "value_func_type" in kw:
        cfg = synth.CNN_CONFIGS["small_t1"]
        args = synth.cnn_reference_kwargs(cfg, algorithm="DSAC_V1", replay_batch_size=4, dsact_gemm="fp32")
    else:
        args = synth.reference_kwargs(cfg, algorithm="DSAC_V1", replay_batch_size=4, dsact_gemm="fp32", **kw)
    with pytest.raises(NotImplementedError, match="mlp_shared"):
        dsac_v1.ApproxContainer(**args)
    args.pop("dsact_gemm")
    dsac_v1.ApproxContainer(**args)   # the head-wise engine takes them


def test_dsact_gemm_takes_different_critic_and_policy_networks():
    import dsac_v1
    kw = synth.reference_kwargs(synth.ASYM_CONFIGS["asym"], algorithm="DSAC_V1", replay_batch_size=4)
    with pytest.raises(NotImplementedError):   # the head-wise engine: one hidden_sizes / activation
        dsac_v1.ApproxContainer(**kw)
    net = dsac_v1.ApproxContainer(**dict(kw, dsact_gemm="bf16x3", dsact_graph=False))
    assert net.route.cfg_args["gemm_mode"] == "bf16x3" and net.route.cfg_args["use_graph"] is False


@pytest.mark.parametrize("name", NEW_GOLDENS)
def test_v1_oracle_matches_reference(golden_dir, name):
    """The oracle (critic and policy of the config's own shapes) against the unmodified reference
    (tests/golden/make_golden_v1_mlp.py), at the tolerances of test_oracle_golden_v1_heads.py."""
    from oracle.dsact_oracle import V1_TB_KEYS
    torch.set_num_threads(4)
    z, cfg, batch, steps, hyper = golden(golden_dir, name)
    orc = v1_oracle(cfg, synth.make_weights_v1(cfg), **hyper)
    assert list(z["tb_keys"]) == V1_TB_KEYS
    names = [str(n) for n in z["param_names"]]
    trainable = [str(n) for n in z["trainable_names"]]
    assert set(names) == set(orc.state_dict())
    for it in range(steps):
        tb = orc.update(synth.make_batch(cfg, batch, it), synth.make_noise(cfg, batch, it), it)
        np.testing.assert_allclose([tb[k] for k in V1_TB_KEYS], z["tb"][it], rtol=2e-6, atol=1e-7, err_msg=f"{name} step {it}")
        sd = orc.state_dict()
        if f"pdigest_{it + 1}" in z:
            for row, k in zip(z[f"pdigest_{it + 1}"], names):
                d = sd[k].double().reshape(-1)
                np.testing.assert_allclose(d.sum().item(), row[0], rtol=1e-6, atol=1e-7 * row[1] + 1e-9, err_msg=f"{name} {k}")
                np.testing.assert_allclose(d.abs().sum().item(), row[1], rtol=1e-6, atol=1e-9, err_msg=f"{name} {k}")
                np.testing.assert_allclose(d[:8].numpy(), row[3:3 + min(8, d.numel())], rtol=1e-5, atol=1e-8, err_msg=f"{name} {k}")
        if it in (0, 1) and f"gdigest_{it}" in z:
            gd = orc.grad_dict()
            for row, k in zip(z[f"gdigest_{it}"], trainable):
                if k in gd:
                    np.testing.assert_allclose(gd[k].double().abs().sum().item(), row[1], rtol=1e-5, atol=1e-9,
                                               err_msg=f"{name} grad {k} step {it}")
        if f"state_{it + 1}/{names[0]}" in z:
            for k in names:
                np.testing.assert_allclose(sd[k].numpy(), z[f"state_{it + 1}/{k}"], rtol=1e-6, atol=1e-8, err_msg=f"{name} {k}")


def test_v1_oracle_is_the_existing_one_on_symmetric_configs():
    """On CONFIGS entries (one width list, GELU) the oracle with per-network shapes is `v1_from_config` exactly."""
    from oracle.dsact_oracle import V1_TB_KEYS, v1_from_config
    cfg = synth.CONFIGS["ragged"]
    w = synth.make_weights_v1(cfg)
    a, b = v1_oracle(cfg, w, **synth.HYPER), v1_from_config(cfg, w, **synth.HYPER)
    for it in range(2):
        ta = a.update(synth.make_batch(cfg, 20, it), synth.make_noise(cfg, 20, it), it)
        tb = b.update(synth.make_batch(cfg, 20, it), synth.make_noise(cfg, 20, it), it)
        assert [ta[k] for k in V1_TB_KEYS] == [tb[k] for k in V1_TB_KEYS]
    for k, v in a.state_dict().items():
        assert torch.equal(v, b.state_dict()[k]), k
