"""CPU check of the host draws of the drop-in's replay_updates: n rounds drawn up front must be the numbers n interleaved
rounds of `buffer.sample_batch` (numpy indices) + `local_update` (torch CPU noise) would have drawn, in order."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch


class _Buffer:
    """What host_draws reads of training.replay_buffer.ReplayBuffer with dsact_index_source="numpy"."""

    def __init__(self, size, numpy_indices=True):
        self.size, self.numpy_indices = size, numpy_indices

    def sample_indices(self, batch):
        return torch.from_numpy(np.random.randint(0, self.size, size=batch)) if self.numpy_indices else None


@pytest.mark.parametrize("algo", ["DSAC_V2", "DSAC_V1"])
@pytest.mark.parametrize("numpy_indices,noise", [(True, "reference"), (True, "device"), (False, "reference"), (False, "device")])
def test_host_draws_equal_interleaved_rounds(algo, numpy_indices, noise):
    import dsac_v1
    import dsac_v2
    from dsact_host import host_draws
    cls = dsac_v1.DSAC_V1 if algo == "DSAC_V1" else dsac_v2.DSAC_V2
    alg = SimpleNamespace(noise_source=noise, act_dim=3)
    noise_fn = lambda b: cls._noise(alg, b)   # noqa: E731
    buf, B, n = _Buffer(50, numpy_indices), 7, 4

    np.random.seed(3); torch.manual_seed(4)
    want_idx, want_noise = [], []
    for _ in range(n):   # sample_batch, then local_update
        want_idx.append(buf.sample_indices(B))
        want_noise.append(noise_fn(B))

    np.random.seed(3); torch.manual_seed(4)
    idx, nz = host_draws(buf, B, n, noise_fn)
    if numpy_indices:
        assert idx.shape == (n, B) and idx.dtype == torch.int64
        for k in range(n):
            assert torch.equal(idx[k], want_idx[k])
    else:
        assert idx is None
    if noise == "reference":
        shapes = [(n, B, 3), (n, B, 3), (n, B), (n, B)]
        for j in range(4):
            assert nz[j].shape == shapes[j]
            for k in range(n):
                assert torch.equal(nz[j][k], want_noise[k][j]), (j, k)
    else:
        assert nz is None
