"""BASELINE config 5 (CNN encoder + DSAC-T heads, reference networks/cnn.py) through the C ABI (a `dsact_cnn_create` handle):
the CUDA path against the golden produced by the unmodified reference (tests/golden/cnn_carracing_b4.npz) and against
the pinned oracle on a second batch size, gradients included.  fp32 direct convolutions + fp32 GEMMs: tolerance 1e-4
relative (north_star's gate); observed ~1e-6."""
import ast
import os

import numpy as np
import pytest
import torch

from dsac_v2_b200 import synth

pytestmark = pytest.mark.gpu
RTOL = 1e-4


def make_engine(cfg, batch):
    from dsac_v2_b200.engine_cnn import CnnEngine, make_cnn_config
    t = synth.CONV_TYPES[cfg["conv_type"]]
    h = synth.HYPER
    c = make_cnn_config(cfg["obs_dim"], cfg["act_dim"], t["kernels"], t["channels"], t["strides"], t["heads"], max_batch=batch,
                        gamma=h["gamma"], tau=h["tau"], delay_update=h["delay_update"], auto_alpha=h["auto_alpha"], alpha=h["alpha"],
                        lr_q=h["value_learning_rate"], lr_pi=h["policy_learning_rate"], lr_alpha=h["alpha_learning_rate"],
                        min_log_std=h["policy_min_log_std"], max_log_std=h["policy_max_log_std"])
    lim = torch.full((cfg["act_dim"],), cfg["act_lim"])
    eng = CnnEngine(c, torch.device("cuda", 0), lim, -lim)
    eng.load_weights(synth.make_cnn_weights(cfg))
    return eng


def feed(cfg, batch, it):
    b = {k: torch.from_numpy(v).cuda() for k, v in synth.make_cnn_batch(cfg, batch, it).items()}
    n = synth.make_noise(cfg, batch, it)
    return b, tuple(torch.from_numpy(n[i]).cuda() for i in (0, 1, 4, 5))


@pytest.mark.parametrize("name", ["cnn_carracing_b4", "cnn_type1_b5"])
def test_cnn_update_matches_reference_golden(golden_dir, name):
    from dsac_v2_b200.engine import STAT_KEYS
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg_name, batch, steps, over = z["meta"]
    cfg, batch, steps = synth.CNN_CONFIGS[str(cfg_name)], int(batch), int(steps)
    assert dict(ast.literal_eval(str(over))) == {}
    eng = make_engine(cfg, batch)
    names = [str(n) for n in z["param_names"]]
    for it in range(steps):
        b, n = feed(cfg, batch, it)
        eng.step(b, it, n)
        s = eng.read_stats()
        got = np.array([s[k] for k in STAT_KEYS])
        np.testing.assert_allclose(got, z["tb"][it], rtol=RTOL, atol=1e-6, err_msg=f"tb_info at step {it}")
        if f"pdigest_{it + 1}" in z:
            w = eng.export_weights()
            for row, k in zip(z[f"pdigest_{it + 1}"], names):
                d = w[k].double().reshape(-1)
                np.testing.assert_allclose(d.abs().sum().item(), row[1], rtol=RTOL, err_msg=f"{k} after step {it + 1}")
                np.testing.assert_allclose(d[:8].numpy(), row[3:3 + min(8, d.numel())], rtol=RTOL, atol=1e-7, err_msg=f"{k} after step {it + 1}")
    eng.close()


@pytest.mark.parametrize("cfg_name,batch", [("carracing", 3), ("carracing", 32), ("small_t1", 7), ("odd", 9), ("odd", 200)])
def test_cnn_update_matches_oracle(cfg_name, batch):
    """Other batch sizes (ragged against every tile size) and encoders — type_1 (8x8 first layer) and a stack whose channel
    counts force the one-channel-per-thread kernels —, full post-update state and the gradients of the last step."""
    from dsac_v2_b200.engine import STAT_KEYS
    from oracle.dsact_oracle import TB_KEYS, cnn_from_config
    cfg = synth.CNN_CONFIGS[cfg_name]
    eng = make_engine(cfg, batch)
    orc = cnn_from_config(cfg, synth.make_cnn_weights(cfg), **synth.HYPER)
    assert STAT_KEYS == TB_KEYS
    for it in range(3):
        ref = orc.update(synth.make_cnn_batch(cfg, batch, it), synth.make_noise(cfg, batch, it), it)
        b, n = feed(cfg, batch, it)
        eng.step(b, it, n)
        s = eng.read_stats()
        np.testing.assert_allclose([s[k] for k in TB_KEYS], [ref[k] for k in TB_KEYS], rtol=RTOL, atol=1e-6, err_msg=f"step {it}")
    g, gref = eng.export_weights(grads=True), orc.grad_dict()
    for k, v in gref.items():
        np.testing.assert_allclose(g[k].numpy(), v.numpy(), rtol=1e-3, atol=2e-6 * float(v.abs().max()) + 1e-12, err_msg=f"grad {k}")
    w, sd = eng.export_weights(), orc.state_dict()
    for k, v in sd.items():   # (Adam turns a 1e-7 gradient difference on a near-zero gradient into up to a few 1e-6 of weight)
        np.testing.assert_allclose(w[k].numpy(), v.numpy(), rtol=RTOL, atol=1e-5, err_msg=k)
    eng.close()


def test_cnn_dropin_local_update_and_replay_ring():
    """The reference-facing path: `dsac_v2.DSAC_V2(**kwargs with value_func_type="CNN")`, networks with the reference's
    173-key state_dict, `local_update` on image minibatches (reference noise order), and the device replay ring with
    image rows (store -> gather is bit exact)."""
    import dsac_v2
    from training.replay_buffer import ReplayBuffer
    cfg, B = synth.CNN_CONFIGS["carracing"], 4
    kw = synth.cnn_reference_kwargs(cfg, replay_batch_size=B, dsact_noise="reference", buffer_max_size=64, additional_info={})
    alg = dsac_v2.DSAC_V2(**kw)
    sd = alg.networks.state_dict()
    ref_w = synth.make_cnn_weights(cfg)
    assert {k for k in sd if not k.endswith("_lim")} == set(ref_w) | {"log_alpha"}   # (+ the act_high/low_lim buffers, as in the reference)
    for k, v in ref_w.items():
        sd[k] = torch.from_numpy(v)
    alg.networks.load_state_dict(sd)
    alg.networks.cuda()
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cnn_carracing_b4.npz"))
    from dsac_v2_b200.engine import STAT_KEYS
    # the golden's noise through torch's CPU generator order is not reproducible here; feed the engine directly for the values
    eng = alg.networks.engine(B)
    for it in range(2):
        b, n = feed(cfg, B, it)
        eng.step(b, it, n)
        s = eng.read_stats()
        np.testing.assert_allclose([s[k] for k in STAT_KEYS], z["tb"][it], rtol=RTOL, atol=1e-6)
    # parameters are views of the flat buffers: the module sees the update
    w = alg.networks.state_dict()["policy.conv.0.weight"]
    assert not torch.equal(w.cpu(), torch.from_numpy(ref_w["policy.conv.0.weight"]))
    # local_update with device noise runs and returns finite tb_info
    tb = alg.local_update({k: v for k, v in feed(cfg, B, 5)[0].items()}, 2)
    assert np.isfinite(tb["Loss/Critic loss-RL iter"]) and np.isfinite(tb["Loss/Actor loss-RL iter"])
    # replay ring with image rows
    buf = ReplayBuffer(**kw)
    buf.attach(eng)
    g = np.random.default_rng(0)
    rows = [(g.random(cfg["obs_dim"], dtype=np.float32), {}, g.uniform(-1, 1, cfg["act_dim"]).astype(np.float32), float(i),
             g.random(cfg["obs_dim"], dtype=np.float32), False, np.float32(0), {}) for i in range(10)]
    buf.add_batch(rows)
    idx = torch.tensor([3, 0, 9, 3])
    buf.index_source = "numpy"
    buf.sample_indices = lambda n: idx
    got = buf.sample_batch(4)
    assert tuple(got["obs"].shape) == (4,) + tuple(cfg["obs_dim"])
    for j, i in enumerate(idx.tolist()):
        np.testing.assert_array_equal(got["obs"][j].cpu().numpy(), rows[i][0])
        np.testing.assert_array_equal(got["obs2"][j].cpu().numpy(), rows[i][4])
        assert float(got["rew"][j]) == float(i)
