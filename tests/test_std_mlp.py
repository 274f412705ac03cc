"""The policy's "mlp_separated" / "parameter" std types on the MLP engine, as far as a host without a GPU can check: the
new configuration field leaves the struct layout alone, the flat layout is the head-wise engine's (so weights, views and
checkpoints carry over), `Engine._schema` walks it in the drop-in modules' parameter order, bad values are refused with a
message, and the drop-in picks the MLP engine exactly when `dsact_gemm` is given."""
import ctypes as C

import pytest

from dsac_v2_b200 import _lib, synth
from dsac_v2_b200.engine import Engine, make_v1_options, query_layout
from std_mlp_common import STD_TYPES, make_oracle, std_config, std_weights
from test_abi import _check_slots


def test_policy_std_sits_in_the_former_padding():
    assert C.sizeof(_lib.Config) == 200
    assert _lib.Config.policy_std.offset == 100 and _lib.Config.act_dist.offset == 96 and _lib.Config.gamma.offset == 104
    assert _lib.ABI_VERSION == 4 == _lib.load().dsact_abi_version()


@pytest.mark.parametrize("std_type", STD_TYPES)
@pytest.mark.parametrize("name", ["tiny", "ragged"])
def test_layout_is_the_head_wise_engines(name, std_type):
    from dsac_v2_b200.engine_cnn import make_heads_config
    cfg = synth.CONFIGS[name]
    lay = query_layout(std_config(cfg, std_type, 4))
    ref = _lib.Layout()
    heads = make_heads_config(cfg["obs_dim"], cfg["act_dim"], cfg["hidden"], std_type, max_batch=4)
    assert _lib.load().dsact_cnn_query_layout(C.byref(heads), C.byref(ref)) == 0
    assert (lay.n_q, lay.n_pi, lay.n_params, lay.n_targets) == (ref.n_q, ref.n_pi, ref.n_params, ref.n_targets)


@pytest.mark.parametrize("std_type", STD_TYPES)
@pytest.mark.parametrize("name", ["ragged", "asym", "deep_pi"])
def test_schema_names_every_float_once_in_the_modules_order(name, std_type):
    import dsac_v2
    cfg = synth.mlp_config(name)
    net = dsac_v2.ApproxContainer(**synth.reference_kwargs(cfg, policy_std_type=std_type, replay_batch_size=4, dsact_gemm="fp32"))
    assert net.route.engine == "mlp"   # the MLP engine, with the networks' own shapes
    c = net.route.config(4)
    lay = query_layout(c)

    class Probe:   # _schema only reads the config
        cfg, v1 = c, None
    schema, n = Engine._schema(Probe)
    assert n == lay.n_targets == lay.n_params - 1
    spans = sorted((e[2], e[3]) for e in schema)
    assert spans[0][0] == 0 and all(a + k == b for (a, k), (b, _) in zip(spans, spans[1:])) and sum(spans[-1]) == n
    assert [e[0] for e in schema] == [k for k, p in net.named_parameters() if p.requires_grad and k != "log_alpha"]
    assert [e[1] for e in schema] == [k for k, p in net.named_parameters() if not p.requires_grad]
    sizes = dict(net.named_parameters())
    assert all(tuple(sizes[e[0]].shape) == tuple(e[4]) for e in schema)
    assert set(std_weights(cfg, std_type)) == {k for e in schema for k in e[:2]}
    first = "policy.log_std" if std_type == "parameter" else "policy.mean.0.weight"
    assert [e[0] for e in schema if e[0].startswith("policy.")][0] == first


def test_without_dsact_gemm_the_head_wise_engine_is_still_chosen():
    import dsac_v2
    cfg = synth.CONFIGS["ragged"]
    for std_type in STD_TYPES:
        net = dsac_v2.ApproxContainer(**synth.reference_kwargs(cfg, policy_std_type=std_type, replay_batch_size=4))
        assert net.route.engine == "heads" and net.route.cfg_args["std_type"] == std_type
    with pytest.raises(NotImplementedError):   # the head-wise engine takes one shape for critics and policy
        dsac_v2.ApproxContainer(**synth.reference_kwargs(synth.mlp_config("asym"), policy_std_type="parameter", replay_batch_size=4))


def test_bad_policy_std_is_refused_with_a_message():
    lib, out, cfg = _lib.load(), _lib.Layout(), synth.CONFIGS["tiny"]
    c = std_config(cfg, "parameter", 4)
    c.policy_std = 3
    assert lib.dsact_query_layout(C.byref(c), C.byref(out)) == -1 and b"policy_std" in lib.dsact_last_error()
    c.policy_std = -1
    assert lib.dsact_query_layout(C.byref(c), C.byref(out)) == -1
    v1 = make_v1_options()
    for std_type in STD_TYPES:   # DSAC_V1 runs these policies on the head-wise engine
        c = std_config(cfg, std_type, 4)
        assert lib.dsact_v1_query_layout(C.byref(c), C.byref(v1), C.byref(out)) == -1 and b"mlp_shared" in lib.dsact_last_error()
        h = C.c_void_p()
        assert lib.dsact_v1_create(C.byref(c), C.byref(v1), 0, C.byref(h)) == -1
    assert lib.dsact_v1_query_layout(C.byref(std_config(cfg, "mlp_shared", 4)), C.byref(v1), C.byref(out)) == 0


@pytest.mark.parametrize("mode", list(_lib.GEMM_MODES))
@pytest.mark.parametrize("std_type", STD_TYPES)
@pytest.mark.parametrize("name", ["tiny", "ragged", "humanoid", "asym", "layered_pi"])
def test_reported_workspace_slots(name, std_type, mode):
    cfg = synth.mlp_config(name)
    for mb in (1, 256, 1000):
        _check_slots(query_layout(std_config(cfg, std_type, mb, mode)), cfg["act_dim"], mode != "fp32")


def test_mlp_shared_layout_is_what_it_was():
    """The default std type keeps its parameter counts and takes none of the log_std network's arena slots: the
    mlp_separated workspace of the same networks is larger, with the shared leading slots where they were."""
    cfg = synth.CONFIGS["humanoid"]
    lay = query_layout(std_config(cfg, "mlp_shared", 4096, "bf16x3"))
    assert (lay.n_pi, lay.n_params) == (236834, 702759)
    two = query_layout(std_config(cfg, "mlp_separated", 4096, "bf16x3"))
    assert two.workspace_bytes > lay.workspace_bytes and two.off_eps1 == lay.off_eps1


@pytest.mark.parametrize("std_type", STD_TYPES)
def test_oracle_takes_each_networks_own_shape(std_type):
    """The oracle the GPU tests compare against, on critics and policy of different depths, widths and activations: one
    update runs and moves every policy tensor."""
    cfg = synth.mlp_config("asym")
    orc = make_oracle(cfg, std_type)
    before = {k: v.clone() for k, v in orc.state_dict().items()}
    for it in range(2):
        orc.update(synth.make_batch(cfg, 9, it), synth.make_noise(cfg, 9, it), it)
    after = orc.state_dict()
    moved = [k for k in before if k.startswith("policy.") and not (after[k] == before[k]).all()]
    assert moved == [k for k in before if k.startswith("policy.")]


def test_dropin_takes_the_all_reduce_transport_for_these_std_types():
    """The MLP engine's peer-memory data-parallel step serves mlp_shared only (dsact_dp_* refuse the other std types);
    under torch.distributed the drop-in then reduces between the split calls."""
    import dsac_v2
    cfg = synth.CONFIGS["tiny"]
    for std_type in STD_TYPES:
        alg = dsac_v2.DSAC_V2(**synth.reference_kwargs(cfg, policy_std_type=std_type, replay_batch_size=4, dsact_gemm="bf16x3"))
        assert alg.dp_transport == "nccl"
    assert dsac_v2.DSAC_V2(**synth.reference_kwargs(cfg, replay_batch_size=4)).dp_transport == "peer"
    assert dsac_v2.DSAC_V2(**synth.reference_kwargs(cfg, policy_std_type="parameter", replay_batch_size=4)).dp_transport == "peer"
