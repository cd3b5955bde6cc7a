"""Cfg.domain_rand.lag_timesteps (the action FIFO depth L) on the CPU: oracle/env_oracle.py against vectors produced by the reference's
own LeggedRobot._compute_torques (tests/golden/lag.npz), and the range build_sim_config accepts."""
import os

import numpy as np
import pytest
import torch

import lag_util as U
from env_golden_util import HERE, train_sim_config
from oracle import env_oracle as eo


def lag_config(n, L, control_type="actuator_net", decimation=4, **dr):
    return train_sim_config(n, cfg_overrides={"domain_rand": dict(lag_timesteps=L, **dr),
                                              "control": {"control_type": control_type, "decimation": decimation}})


def load_lag_gold():
    return np.load(os.path.join(HERE, "golden", "lag.npz"))


@pytest.mark.parametrize("case", list(U.CASES))
def test_oracle_matches_reference(case):
    g = load_lag_gold()
    L, control_type, decimation = U.CASES[case]
    Cfg, c, info = lag_config(U.N, L, control_type, decimation)
    P = eo.params_from_sim_config(c, info["active_reward_scales"], info["dt"])
    x = {k: torch.from_numpy(v) for k, v in U.inputs(case, np.array(c.default_dof_pos, dtype=np.float32)).items()}
    s = {k: x[k].clone() for k in ("dof_pos", "dof_vel", "joint_pos_err_last", "joint_pos_err_last_last", "joint_vel_last",
                                   "joint_vel_last_last", "motor_offsets")}
    s.update(motor_strengths=x["motor_strengths"][:, None].repeat(1, 12), Kp_factors=torch.ones(U.N, 12), Kd_factors=torch.ones(U.N, 12),
             lag_buffer=[torch.zeros(U.N, 12)] + [x["fifo"][i].clone() for i in range(L)])
    net = eo.ActuatorNet()
    k = 0
    for t in range(U.T):
        s["actions"] = x["actions"][t].clone()
        for _ in range(decimation):
            tq = eo.compute_torques(s, P, net)
            assert np.array_equal(s["joint_pos_target"].numpy(), g[f"{case}/target"][k]), (case, k)
            assert np.allclose(tq.numpy(), g[f"{case}/torque"][k], rtol=1e-5, atol=2e-5), (case, k)
            fifo = torch.stack(s["lag_buffer"][1:]).numpy() if L else np.zeros((0, U.N, 12), np.float32)
            assert np.array_equal(fifo, g[f"{case}/fifo"][k]), (case, k)
            k += 1
    assert k == g[f"{case}/target"].shape[0]


def test_build_sim_config_accepts_the_range():
    from go1_b200 import capi
    assert capi.MAX_LAG_TIMESTEPS == 32
    for L in range(0, 33):
        _, c, _ = lag_config(16, L)
        assert c.use_lag == 1 and c.lag_timesteps == L
    for L in (-1, 33, 2.5):
        with pytest.raises(ValueError, match=r"0\.\.32"):
            lag_config(16, L)


def test_lag_timesteps_changes_only_its_own_field():
    _, c6, _ = lag_config(16, 6)
    assert c6.use_lag == 1 and c6.lag_timesteps == 6
    for L in (0, 13, 32):
        _, c, _ = lag_config(16, L)
        c.lag_timesteps = 6
        assert bytes(c) == bytes(c6), L


def test_without_randomize_lag_timesteps_no_fifo_is_used():
    # the reference never reads its FIFO then, whatever lag_timesteps says (legged_robot.py:921-926)
    for L in (6, 50):
        _, c, _ = lag_config(16, L, randomize_lag_timesteps=False)
        assert c.use_lag == 0 and c.lag_timesteps == 0
