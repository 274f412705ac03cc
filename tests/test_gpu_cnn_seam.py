"""The split gradient API on a head-wise handle (`dsact_grad_phase1` / `_grad_phase2` / `dsact_compute_grads` /
`dsact_apply`) on one GPU, for the CNN approximators and the policy std types "mlp_separated" / "parameter": gradients and
post-update state against the pinned oracle, and the drop-in's gradient-message seam (`DSAC_V2.get_remote_update_info` /
`remote_update`, reference dsac_v2.py:107-138) against `local_update`."""
import ctypes as C

import numpy as np
import pytest
import torch

from dsac_v2_b200 import synth

pytestmark = pytest.mark.gpu
RTOL = 1e-4
CASES = ["odd", "mlp_separated", "parameter"]   # CNN config `odd`; the std types on the `ragged` MLP shapes


def _setup(case, batch):
    """(engine factory, oracle factory, batch maker, config, weights) of one case."""
    from oracle.dsact_oracle import cnn_from_config, std_from_config
    if case in synth.CNN_CONFIGS:
        from test_gpu_cnn import make_engine
        cfg = synth.CNN_CONFIGS[case]
        w = synth.make_cnn_weights(cfg)
        return (lambda: make_engine(cfg, batch)), (lambda: cnn_from_config(cfg, w, **synth.HYPER)), synth.make_cnn_batch, cfg, w
    from test_gpu_std import make_engine
    cfg = synth.CONFIGS["ragged"]
    w = synth.make_weights_std(cfg, case)
    return (lambda: make_engine(cfg, batch, case)), (lambda: std_from_config(cfg, w, case, **synth.HYPER)), synth.make_batch, cfg, w


def _feed(make_batch, cfg, batch, it):
    b = {k: torch.from_numpy(v).cuda() for k, v in make_batch(cfg, batch, it).items()}
    n = synth.make_noise(cfg, batch, it)
    return b, tuple(torch.from_numpy(n[i]).cuda() for i in (0, 1, 4, 5))


def _assert_grads(eng, orc, what):
    g, gref = eng.export_weights(grads=True), orc.grad_dict()
    assert set(gref) <= set(g)
    for k, v in gref.items():   # the tolerances of test_cnn_update_matches_oracle / test_std_type_update_matches_oracle
        np.testing.assert_allclose(g[k].numpy(), v.numpy(), rtol=1e-3, atol=2e-6 * float(v.abs().max()) + 1e-12, err_msg=f"{what}: grad {k}")


@pytest.mark.parametrize("case", CASES)
def test_split_gradients_and_apply_match_oracle(case):
    from dsac_v2_b200.engine import STAT_KEYS
    from oracle.dsact_oracle import TB_KEYS
    B = 9 if case == "odd" else 37
    make_eng, make_orc, make_batch, cfg, _ = _setup(case, B)
    whole, split, orc = make_eng(), make_eng(), make_orc()
    assert STAT_KEYS == TB_KEYS
    for it in range(3):
        ref = orc.compute_gradients(make_batch(cfg, B, it), synth.make_noise(cfg, B, it))
        b, n = _feed(make_batch, cfg, B, it)
        whole.compute_grads(b, n)
        split.grad_phase1(b, n)
        split.grad_phase2(B)
        if it == 0:   # same weights on all three: the gradients themselves (later steps compare the updated state below)
            _assert_grads(whole, orc, "compute_grads")
            _assert_grads(split, orc, "grad_phase1 + grad_phase2")
        g, gs = whole.grads.cpu().numpy(), split.grads.cpu().numpy()
        np.testing.assert_allclose(gs, g, rtol=1e-3, atol=2e-6 * float(np.abs(g).max()), err_msg=f"phases vs compute_grads, step {it}")
        orc.apply(it)
        whole.apply(it)
        split.apply(it)
        for eng, what in ((whole, "compute_grads"), (split, "phases")):
            s = eng.read_stats(B)
            np.testing.assert_allclose([s[k] for k in TB_KEYS], [ref[k] for k in TB_KEYS], rtol=RTOL, atol=1e-6, err_msg=f"{what} step {it}")
    sd = orc.state_dict()
    for eng, what in ((whole, "compute_grads + apply"), (split, "phases + apply")):
        w = eng.export_weights()
        for k, v in sd.items():   # (Adam turns a 1e-7 gradient difference on a near-zero gradient into up to a few 1e-6 of weight)
            np.testing.assert_allclose(w[k].numpy(), v.numpy(), rtol=RTOL, atol=1e-5, err_msg=f"{what}: {k}")
        eng.close()


def test_split_api_argument_checks():
    from dsac_v2_b200 import _lib
    from dsac_v2_b200.engine_cnn import CnnEngine, make_heads_config
    make_eng, _, make_batch, cfg, _ = _setup("mlp_separated", 8)
    eng = make_eng()
    with pytest.raises(_lib.DsactError, match="without a preceding"):
        eng.grad_phase2(8)
    b, n = _feed(make_batch, cfg, 8, 0)
    eng.grad_phase1(b, n)
    with pytest.raises(_lib.DsactError, match="global_batch"):
        eng.grad_phase2(7)
    with pytest.raises(_lib.DsactError, match="dp_connect"):
        eng.dp_step(b, 0, 8, n)
    # the calls only the MLP engine implements refuse a head-wise handle with a message
    lib, stream, hb = eng.lib, eng._stream(), eng._batch(b)
    for rc in (lib.dsact_step_host(eng.h, C.byref(hb), None, 0, stream), lib.dsact_replay_step(eng.h, 8, 8, None, None, 0, stream),
               lib.dsact_profile_step(eng.h, C.byref(hb), None, 0, stream, C.byref(_lib.Profile()))):
        assert rc == -1 and b"head-wise" in lib.dsact_last_error()
    with pytest.raises(_lib.DsactError, match="head-wise"):
        eng.profile_step(b, 0, n)
    assert eng._seed == 0x5DEECE66D   # unseeded: the library's default generator seed
    before = eng.launch_count()
    eng.step(b, 0, n)
    assert eng.launch_count() > before and eng.last_call_launches() > 0
    eng.close()
    tiny = synth.CONFIGS["tiny"]
    lim = torch.full((tiny["act_dim"],), tiny["act_lim"])
    v1 = CnnEngine(make_heads_config(tiny["obs_dim"], tiny["act_dim"], tiny["hidden"], "mlp_shared", max_batch=4, algo="DSAC_V1"),
                   torch.device("cuda", 0), lim, -lim)
    bt = {k: torch.from_numpy(v).cuda() for k, v in synth.make_batch(tiny, 4, 0).items()}
    for call in (lambda: v1.compute_grads(bt), lambda: v1.grad_phase1(bt), lambda: v1.grad_phase2(4), lambda: v1.apply(0),
                 lambda: v1.dp_export(), lambda: v1.dp_step(bt, 0, 4)):
        with pytest.raises(_lib.DsactError, match="DSAC_V1"):
            call()
    v1.close()


def _dropin(case, B):
    import dsac_v2
    _, _, _, cfg, w = _setup(case, B)
    if case in synth.CNN_CONFIGS:
        kw = synth.cnn_reference_kwargs(cfg, replay_batch_size=B, dsact_noise="reference")
    else:
        kw = synth.reference_kwargs(cfg, policy_std_type=case, replay_batch_size=B, dsact_noise="reference")
    alg = dsac_v2.DSAC_V2(**kw)
    sd = alg.networks.state_dict()
    for k, v in w.items():
        sd[k] = torch.from_numpy(v)
    alg.networks.load_state_dict(sd)
    alg.networks.cuda()
    return alg


@pytest.mark.parametrize("case", ["carracing", "mlp_separated", "parameter"])
def test_remote_update_seam_equals_local_update(case):
    """Twin `DSAC_V2` instances: `get_remote_update_info` + `remote_update` (a cloned message) on one equals
    `local_update` on the other, with the reference's update_info keys and per-parameter gradient shapes.  (The drop-in's
    `networks.cnn` builds the reference's conv types only: the CNN case is `type_2`, CarRacing-shaped.)"""
    B = 4 if case in synth.CNN_CONFIGS else 16
    _, _, make_batch, cfg, _ = _setup(case, B)
    a, b = _dropin(case, B), _dropin(case, B)
    for it in range(4):
        batch = {k: torch.from_numpy(v).cuda() for k, v in make_batch(cfg, B, it).items()}
        torch.manual_seed(it)
        tb_a = a.local_update(batch, it)
        torch.manual_seed(it)
        tb_b, info = b.get_remote_update_info(batch, it)
        assert set(info) == {"q1_grad", "q2_grad", "policy_grad", "iteration", "log_alpha_grad"}
        for key, net in (("q1_grad", b.networks.q1), ("q2_grad", b.networks.q2), ("policy_grad", b.networks.policy)):
            assert [g.shape for g in info[key]] == [p.shape for p in net.parameters()], key
        assert info["log_alpha_grad"].shape == b.networks.log_alpha.shape
        msg = {k: ([g.clone() for g in v] if isinstance(v, list) else (v.clone() if torch.is_tensor(v) else v))
               for k, v in info.items()}
        b.remote_update(msg)
        assert abs(tb_a["Loss/Critic loss-RL iter"] - tb_b["Loss/Critic loss-RL iter"]) < 1e-5
    for (k, va), vb in zip(a.networks.state_dict().items(), b.networks.state_dict().values()):
        torch.testing.assert_close(va, vb, rtol=1e-5, atol=1e-7, msg=k)
