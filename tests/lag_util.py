"""Shared by tests/golden/make_golden_lag.py and the lag_timesteps tests: the cases and seeded inputs of tests/golden/lag.npz.
The inputs are re-created from numpy's PCG64 stream (platform- and version-independent) instead of being stored."""
import numpy as np

N, T = 8, 4             # 8 envs, 4 policy steps of `decimation` control substeps each
# name: (lag_timesteps, control_type, decimation)
CASES = {f"L{L}": (L, "actuator_net", 4) for L in (0, 1, 3, 4, 5, 7, 8, 13, 32)}
CASES["L5_P"] = (5, "P", 4)
CASES["L3_d2"] = (3, "actuator_net", 2)


def inputs(case, default_dof_pos, seed=31):
    """Initial state of one case.  `default_dof_pos` [12] float32; "fifo" holds the L live slots, oldest first."""
    L, _, _ = CASES[case]
    rng = np.random.default_rng([seed, list(CASES).index(case)])
    f = lambda lo, hi, *s: rng.uniform(lo, hi, s).astype(np.float32)
    return {"dof_pos": np.asarray(default_dof_pos, dtype=np.float32) + f(-0.6, 0.6, N, 12), "dof_vel": f(-6, 6, N, 12),
            "actions": f(-3, 3, T, N, 12), "fifo": f(-0.6, 0.6, L, N, 12),
            "joint_pos_err_last": f(-0.5, 0.5, N, 12), "joint_pos_err_last_last": f(-0.5, 0.5, N, 12),
            "joint_vel_last": f(-6, 6, N, 12), "joint_vel_last_last": f(-6, 6, N, 12),
            "motor_offsets": f(-0.02, 0.02, N, 12), "motor_strengths": f(0.9, 1.1, N)}
