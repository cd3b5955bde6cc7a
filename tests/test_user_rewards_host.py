"""Reward containers on the host: the registry, and how config.reward_tables sorts the nonzero scales of Cfg.reward_scales into
kernel terms, user terms and missing terms (legged_robot.py:1385-1429)."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200"))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))


def _cfg(**scales):
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    apply_train_config(Cfg)
    for k, v in scales.items():
        setattr(Cfg.reward_scales, k, v)
    return Cfg


def test_registry_and_markers():
    from go1_b200 import capi
    from go1_gym.envs.rewards import REWARD_CONTAINERS, BuiltinReward, CoRLRewards
    assert REWARD_CONTAINERS["CoRLRewards"] is CoRLRewards
    for name in capi.REWARD_TERMS:
        m = getattr(CoRLRewards, "_reward_" + name)
        assert isinstance(m, BuiltinReward) and m.builtin_term == name and not callable(m)
    with pytest.raises(KeyError):
        REWARD_CONTAINERS["NoSuchContainer"]


def test_unknown_container_name_raises_at_env_construction():
    cfg = _cfg()
    cfg.rewards.reward_container_name = "NoSuchContainer"
    from go1_gym.envs.base.legged_robot import LeggedRobot
    env = LeggedRobot.__new__(LeggedRobot)
    env.cfg, env.eval_cfg, env.rank_seed_offset = cfg, None, 0
    env.num_envs = env.num_train_envs = 8
    env.num_eval_envs, env.device = 0, "cpu"
    cfg.terrain.mesh_type = "plane"
    with pytest.raises(KeyError):
        env.create_sim()


def _container():
    from go1_gym.envs.rewards import CoRLRewards

    class Mine(CoRLRewards):
        def _reward_hop(self):
            return None

        def _reward_lin_vel_z(self):          # override of a built-in
            return None

    return Mine


def test_classification_scaling_and_order(capsys):
    from go1_b200 import capi
    from go1_b200.config import build_sim_config, cfg_dict
    Mine = _container()
    cfg = _cfg(hop=2.0, lin_vel_z=-0.5, nowhere=1.0, dof_pos=0.0)
    c, info = build_sim_config(cfg, num_envs=8, reward_container=Mine)
    dt = info["dt"]
    assert "Warning: reward _reward_nowhere has nonzero coefficient but was not found!" in capsys.readouterr().out
    nonzero = [k for k, v in cfg_dict(cfg.reward_scales).items() if v != 0]
    assert list(info["active_reward_scales"]) == nonzero                       # dict order kept
    assert list(info["user_reward_scales"]) == [k for k in nonzero if k in ("hop", "lin_vel_z")]
    assert info["user_reward_scales"]["hop"] == 2.0 * dt and info["user_reward_scales"]["lin_vel_z"] == -0.5 * dt
    table = np.array(c.reward_scale)
    assert table[capi.REWARD_TERMS.index("lin_vel_z")] == 0.0                 # the override is zeroed in the kernel table
    order = list(c.reward_order)[:c.num_active_rewards]
    assert capi.REWARD_TERMS.index("lin_vel_z") not in order
    plain, pinfo = build_sim_config(_cfg(hop=2.0, lin_vel_z=-0.5, nowhere=1.0, dof_pos=0.0), num_envs=8)
    want = np.array(plain.reward_scale)
    want[capi.REWARD_TERMS.index("lin_vel_z")] = 0.0
    assert np.array_equal(table, want) and pinfo["user_reward_scales"] == {}
    assert "_reward_hop has nonzero coefficient" in capsys.readouterr().out   # without a container: not found


def test_container_without_a_builtin_drops_it_with_the_warning(capsys):
    from go1_b200 import capi
    from go1_b200.config import build_sim_config

    class Bare:
        def __init__(self, env):
            self.env = env

    c, info = build_sim_config(_cfg(lin_vel_z=-0.5), num_envs=8, reward_container=Bare)
    assert "Warning: reward _reward_lin_vel_z has nonzero coefficient but was not found!" in capsys.readouterr().out
    assert c.reward_scale[capi.REWARD_TERMS.index("lin_vel_z")] == 0.0 and info["user_reward_scales"] == {}


@pytest.mark.parametrize("name", ["tracking_lin_vel", "tracking_ang_vel", "tracking_contacts_shaped_force", "tracking_contacts_shaped_vel"])
def test_task_term_override_raises(name):
    from go1_b200.config import build_sim_config
    from go1_gym.envs.rewards import CoRLRewards
    Task = type("Task", (CoRLRewards,), {"_reward_" + name: lambda self: None})
    with pytest.raises(ValueError, match="command_sums"):
        build_sim_config(_cfg(**{name: 1.0}), num_envs=8, reward_container=Task)
