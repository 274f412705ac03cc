"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol the
header declares, and the size/validation entry points (which need no GPU) behave."""
import ctypes as C
import os
import re

import pytest

from dsac_v2_b200 import _lib, synth
from dsac_v2_b200.engine import make_config, query_layout

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_symbols_are_exported_and_bound():
    header = open(os.path.join(REPO, "include", "dsact.h")).read()
    declared = set(re.findall(r"\b(dsact_[a-z0-9_]+)\s*\(", header))
    assert declared, "no prototypes found"
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/dsact.h but not exported"
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    assert lib.dsact_abi_version() == _lib.ABI_VERSION


def test_struct_sizes_match_header_layout():
    # 5 + 12 + 8 int32 = 25 int32 (100 B, padded to 104 for the doubles) + 12 doubles
    assert C.sizeof(_lib.Config) == 104 + 12 * 8
    assert C.sizeof(_lib.Batch) == 5 * 8 + 8 + 8
    assert C.sizeof(_lib.Buffers) == 9 * 8
    assert C.sizeof(_lib.Layout) == 14 * 8


MLP_CONFIGS = list(synth.CONFIGS) + list(synth.ASYM_CONFIGS)


@pytest.mark.parametrize("name", MLP_CONFIGS)
def test_layout_matches_network_shapes(name):
    cfg = synth.mlp_config(name)
    q, pi = synth.net_shapes(cfg["obs_dim"], cfg["act_dim"], *synth.hidden_sizes(cfg))
    count = lambda s: sum(s[j] * s[j + 1] + s[j + 1] for j in range(len(s) - 1))
    lay = query_layout(make_config(cfg["obs_dim"], cfg["act_dim"], *synth.hidden_sizes(cfg), max_batch=256))
    assert lay.n_q == count(q) and lay.n_pi == count(pi)
    assert lay.n_params == 2 * count(q) + count(pi) + 1
    assert lay.n_targets == lay.n_params - 1
    assert lay.workspace_bytes > 0 and lay.workspace_bytes % 256 == 0


def test_humanoid_parameter_count_is_the_surveyed_one():
    cfg = synth.CONFIGS["humanoid"]
    lay = query_layout(make_config(376, 17, cfg["hidden"], cfg["hidden"], max_batch=4096))
    assert (lay.n_q, lay.n_pi, lay.n_params) == (232962, 236834, 702759)  # SURVEY.md §8 a1


def test_invalid_configs_are_rejected_with_a_message():
    lib = _lib.load()
    out = _lib.Layout()
    for mutate in (lambda c: setattr(c, "obs_dim", 0), lambda c: setattr(c, "n_hidden_q", 0),
                   lambda c: setattr(c, "delay_update", 0), lambda c: setattr(c, "abi_version", 99),
                   lambda c: setattr(c, "act_q", 42), lambda c: setattr(c, "max_batch", 0)):
        c = make_config(5, 2, [8], [8], max_batch=4)
        mutate(c)
        assert lib.dsact_query_layout(C.byref(c), C.byref(out)) == -1
        assert lib.dsact_last_error()


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("needs a CUDA-less host")
    from dsac_v2_b200.engine import Engine
    with pytest.raises(_lib.DsactError):
        Engine(make_config(5, 2, [8], [8], max_batch=4), torch.device("cuda", 0), torch.ones(2), -torch.ones(2))
    import dsac_v2
    alg = dsac_v2.DSAC_V2(**synth.reference_kwargs(synth.CONFIGS["tiny"]))
    with pytest.raises(_lib.DsactError):
        alg.local_update({"obs": torch.zeros(4, 5)}, 0)


def _check_slots(lay, act_dim, slabs):
    """The workspace slots the library reports: 64-float aligned, inside the workspace for max_batch rows, disjoint; the
    weight-gradient slabs are the last region and are empty exactly when `slabs` is false."""
    mb, end = int(lay.max_batch), int(lay.workspace_bytes) // 4
    regions = [(lay.off_idx, 2 * mb), (lay.off_eps1, mb * act_dim), (lay.off_eps2, mb * act_dim), (lay.off_z3, mb),
               (lay.off_z4, mb), (lay.off_slabs, lay.slab_floats)]
    for off, n in regions:
        assert off % 64 == 0 and 0 <= off and off + n <= end, (off, n, end)
    spans = sorted(regions)
    assert all(a + n <= b for (a, n), (b, _) in zip(spans, spans[1:])), spans
    assert lay.off_slabs + lay.slab_floats == end and all(off + n <= lay.off_slabs for off, n in regions[:-1])
    assert (lay.slab_floats > 0) == slabs


@pytest.mark.parametrize("mode", list(_lib.GEMM_MODES))
@pytest.mark.parametrize("name", MLP_CONFIGS)
def test_reported_workspace_slots(name, mode):
    cfg = synth.mlp_config(name)
    for mb in (1, 256, 1000):
        lay = query_layout(make_config(cfg["obs_dim"], cfg["act_dim"], *synth.hidden_sizes(cfg), max_batch=mb, gemm_mode=mode))
        _check_slots(lay, cfg["act_dim"], mode != "fp32")


HEAD_WISE = ["cnn_type2", "cnn_type1", "mlp_separated", "parameter", "v1_mlp"]


def _head_wise(variant):
    """(drop-in ApproxContainer, dsact_cnn_config) of one head-wise variant at max_batch 4."""
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [os.path.join(root, "dsac-v2_b200", "dropin")]
    import dsac_v1
    import dsac_v2
    if variant.startswith("cnn"):
        cfg = synth.CNN_CONFIGS["small_t1" if variant != "cnn_type2" else "carracing"]
        kw = synth.cnn_reference_kwargs(cfg, replay_batch_size=4)
    else:
        cfg = synth.CONFIGS["ragged"]
        over = {"algorithm": "DSAC_V1"} if variant == "v1_mlp" else {"policy_std_type": variant}
        kw = synth.reference_kwargs(cfg, replay_batch_size=4, **over)
    net = (dsac_v1 if variant.startswith("v1") else dsac_v2).ApproxContainer(**kw)
    return net, net.route.config(4)


@pytest.mark.parametrize("variant", HEAD_WISE)
def test_head_wise_workspace_slots(variant):
    from dsac_v2_b200._lib import Layout
    _, c = _head_wise(variant)
    lay = Layout()
    assert _lib.load().dsact_cnn_query_layout(C.byref(c), C.byref(lay)) == 0
    _check_slots(lay, c.act_dim, False)


@pytest.mark.parametrize("variant", HEAD_WISE)
def test_head_wise_layouts_match_the_dropin_modules(variant):
    """The flat layout the head-wise engine reports (`dsact_cnn_query_layout`, no GPU needed) and the state_dict schema
    `CnnEngine._schema` walks are those of the drop-in modules' own parameter order, for every variant it serves."""
    from dsac_v2_b200.engine_cnn import CnnEngine
    from dsac_v2_b200._lib import Layout
    net, c = _head_wise(variant)
    lay = Layout()
    assert _lib.load().dsact_cnn_query_layout(C.byref(c), C.byref(lay)) == 0
    train, targ = net._flat_groups()
    assert lay.n_params == sum(p.numel() for p in train) and lay.n_targets == sum(p.numel() for p in targ)

    class Probe:   # _schema only reads the config
        cfg = c
    schema, n = CnnEngine._schema(Probe)
    assert n == lay.n_targets
    names = [k for k, p in net.named_parameters() if p.requires_grad and k != "log_alpha"]
    assert [e[0] for e in schema] == names
    sizes = dict(net.named_parameters())
    assert all(tuple(sizes[e[0]].shape) == tuple(e[4]) and sizes[e[0]].numel() == e[3] for e in schema)
    assert [e[1] for e in schema] == [k for k, p in net.named_parameters() if not p.requires_grad]


def test_conv_test_hook_rejects_bad_arguments_before_touching_a_device():
    lib = _lib.load()
    null = None
    for op, shape in ((3, (2, 8, 9, 9, 8, 3, 1)), (0, (2, 8, 2, 9, 8, 3, 1)), (1, (0, 8, 9, 9, 8, 3, 1))):
        assert lib.dsact_cnn_test_conv(op, *shape, null, null, null, null, null, null, null, 0, 0, 0, 0, null) == -1
        assert lib.dsact_last_error()


def test_dp_test_hooks_reject_bad_arguments_before_touching_a_device():
    lib = _lib.load()
    io = _lib.TestDpIo()
    peers = (C.c_void_p * 2)()
    for rank, world, want in ((0, 1, b"outside"), (0, 9, b"outside"), (2, 2, b"outside"), (-1, 2, b"outside"),
                              (0, 2, b"not bound")):
        assert lib.dsact_test_dp_attach(None, rank, world, peers, None, None) != 0
        assert want in lib.dsact_last_error(), (rank, world, lib.dsact_last_error())
    assert lib.dsact_test_dp_attach(None, 0, 2, None, None, None) != 0 and b"null peers" in lib.dsact_last_error()
    for op, want in ((-1, b"unknown op"), (4, b"unknown op"), (0, b"not bound"), (3, b"not bound")):
        assert lib.dsact_test_dp(None, op, C.byref(io), None) != 0
        assert want in lib.dsact_last_error(), (op, lib.dsact_last_error())
    assert lib.dsact_test_dp(None, 1, None, None) != 0 and b"null io" in lib.dsact_last_error()
