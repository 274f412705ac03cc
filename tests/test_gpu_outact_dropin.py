"""The drop-in's `DSAC_V2` / `DSAC_V1` with the reference's value_output_activation / policy_output_activation on every
engine route: they construct from the reference's kwargs, train through `OffSerialTrainer`, keep the reference's
state_dict keys and the full-state round trip, and an engine regrown for a larger batch keeps the activations."""
import numpy as np
import pytest
import torch

import test_gpu_v1_heads as H
from dsac_v2_b200 import synth

pytestmark = pytest.mark.gpu

ACTS = dict(value_output_activation="tanh", policy_output_activation="tanh")
# variant -> (algorithm, config, overrides): the routes the drop-in takes
ROUTES = {
    "v2_mlp_bf16x3": ("DSAC_V2", "tiny", {}),
    "v2_mlp_fp32_eager": ("DSAC_V2", "tiny", {"dsact_gemm": "fp32", "dsact_graph": False}),
    "v2_separated": ("DSAC_V2", "tiny", {"policy_std_type": "mlp_separated"}),
    "v2_parameter": ("DSAC_V2", "tiny", {"policy_std_type": "parameter"}),
    "v2_separated_mlp_engine": ("DSAC_V2", "tiny", {"policy_std_type": "mlp_separated", "dsact_gemm": "bf16x3"}),
    "v2_parameter_mlp_engine": ("DSAC_V2", "tiny", {"policy_std_type": "parameter", "dsact_gemm": "fp32"}),
    "v2_cnn": ("DSAC_V2", "small_t1", {}),
    "v1_heads": ("DSAC_V1", "tiny", {}),
    "v1_mlp_bf16x3": ("DSAC_V1", "tiny", {"dsact_gemm": "bf16x3"}),
    "v1_cnn": ("DSAC_V1", "small_t1", {}),
}


@pytest.mark.parametrize("route", list(ROUTES))
def test_trainer_trains_with_output_activations(tmp_path, monkeypatch, route):
    monkeypatch.setitem(H.VARIANTS, route, ROUTES[route])
    trainer, alg, rec = H.make_trainer(route, tmp_path / "run", sample_interval=4, **ACTS)
    eng = alg.networks.engine()
    assert eng.output_activations == ("tanh", "tanh")
    _, linear, _ = H.make_trainer(route, tmp_path / "linear", sample_interval=4)
    assert list(alg.networks.state_dict()) == list(linear.networks.state_dict())
    first = [p.detach().clone() for p in alg.networks.parameters()]
    trainer.train()
    assert trainer.iteration == 16 and [it for it, _ in rec] == list(range(16))
    assert all(np.isfinite(v) for _, v in rec)
    assert any(not torch.equal(a, b.detach()) for a, b in zip(first, alg.networks.parameters()))
    # the CPU mirror the sampler acts with: the reference's network, with the same output activations, holds the weights
    trainer.refresh_policy_mirror()
    for a, b in zip(trainer.sampler.networks.policy.parameters(), alg.networks.policy.parameters()):
        assert torch.equal(a.detach(), b.detach().cpu())

    # full-state round trip: a second algorithm loaded from the first one's full state continues bit for bit
    _, twin, _ = H.make_trainer(route, tmp_path / "twin", sample_interval=4, **ACTS)
    twin.networks.cuda()
    twin.load_full_state_dict(alg.full_state_dict())
    e0, e1 = alg.networks.engine(), twin.networks.engine()
    assert e1.output_activations == ("tanh", "tanh")
    for name in ("params", "targets", "adam_m", "adam_v"):
        assert torch.equal(getattr(e0, name), getattr(e1, name)), name
    cfg_name = ROUTES[route][1]
    cnn = cfg_name in synth.CNN_CONFIGS
    data = {k: torch.from_numpy(v) for k, v in (synth.make_cnn_batch(synth.CNN_CONFIGS[cfg_name], 16, 99) if cnn
                                                 else synth.make_batch(synth.CONFIGS[cfg_name], 16, 99)).items()}
    tb0, tb1 = dict(alg.local_update(data, 16)), dict(twin.local_update(data, 16))
    for k in tb0:
        if "time" not in k.lower():
            assert tb0[k] == tb1[k], k
    for name in ("params", "targets", "adam_m", "adam_v"):
        assert torch.equal(getattr(e0, name), getattr(e1, name)), name


def test_regrown_engine_keeps_output_activations():
    """A batch larger than dsact_max_batch rebuilds the MLP engine: the new one keeps the output activations and updates as
    an engine built at that size from the same state."""
    import dsac_v2
    cfg = synth.CONFIGS["tiny"]
    kw = synth.reference_kwargs(cfg, replay_batch_size=16, dsact_gemm="fp32", value_output_activation="sigmoid",
                                policy_output_activation="gelu")
    small, big = dsac_v2.DSAC_V2(**kw), dsac_v2.DSAC_V2(**dict(kw, replay_batch_size=40))
    big.networks.load_state_dict(small.networks.state_dict())
    small.networks.cuda()
    big.networks.cuda()
    data = {k: torch.from_numpy(v) for k, v in synth.make_batch(cfg, 40, 0).items()}
    for a in (small, big):
        a.noise_source = "reference"
    torch.manual_seed(3)
    tb_small = dict(small.local_update(data, 0))
    torch.manual_seed(3)
    tb_big = dict(big.local_update(data, 0))
    eng = small.networks.engine()
    assert eng.cfg.max_batch == 40 and eng.output_activations == ("sigmoid", "gelu")
    for k in tb_big:
        if "time" not in k.lower():
            assert abs(tb_small[k] - tb_big[k]) <= 1e-5 * max(1.0, abs(tb_big[k])), (k, tb_small[k], tb_big[k])
    np.testing.assert_allclose(eng.params.cpu().numpy(), big.networks.engine().params.cpu().numpy(), rtol=1e-5, atol=1e-7)
