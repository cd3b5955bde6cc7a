"""Shared by tests/golden/make_golden_priv.py and the num_privileged_obs tests: the seeded inputs of tests/golden/ppo_priv.npz.
They are re-created from numpy's PCG64 stream (platform- and version-independent) instead of being stored (the histories alone are 3 MB)."""
import numpy as np

N, T, NOBS, NH, NA = 16, 24, 70, 2100, 12       # 16 envs x 24 steps: 4 minibatches of 96 rows (>= 64: the fused first-layer path)
E_MAX = 45
CASES = {"e5": (5, False), "e18": (18, False), "e45": (45, False), "e45sel": (45, True)}     # name: (num_privileged_obs, selective loss)


def inputs(seed=23):
    """One rollout's inputs, shared by every case; a case with E privileged observations reads priv[..., :E]."""
    rng = np.random.default_rng(seed)
    f = lambda *s, scale=1.0: (rng.standard_normal(s) * scale).astype(np.float32)
    out = {"in/obs": f(T, N, NOBS), "in/hist": f(T, N, NH, scale=0.3), "in/priv": f(T, N, E_MAX), "in/eps": f(T, N, NA), "in/rew": f(T, N),
           "last/hist": f(N, NH, scale=0.3), "last/priv": f(N, E_MAX)}
    out["in/done"] = rng.random((T, N)) < 0.1
    out["in/perm"] = rng.permutation(N * T).astype(np.int64)
    return out


def sample_stride(numel):
    """Stride of the parameter samples stored per tensor (about 512 samples each)."""
    return max(1, numel // 512)
