"""Sim-to-sim acceptance (SURVEY.md §8c(7), the scripts/play.py:89-139 scenario): the policy shipped with the reference
(runs/.../ac_weights_last.pt, stored here as fp16 in slices below 1 MB: tests/golden/pretrained_policy_fp16.part*.npz), trained in Isaac Gym, is
rolled out in THIS simulator with a 1.5 m/s, 3 Hz trot command for 250 steps.  It must walk forward without falling —
the only end-to-end check available for the new rigid-body step (PhysX parity is unpinned)."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))


def _play_env(n):
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    apply_train_config(Cfg)
    dr = Cfg.domain_rand       # play.py:48-61 turns the randomisation off
    for k in ("push_robots", "randomize_friction", "randomize_gravity", "randomize_restitution", "randomize_motor_offset",
              "randomize_motor_strength", "randomize_base_mass", "randomize_Kd_factor", "randomize_Kp_factor", "randomize_com_displacement"):
        setattr(dr, k, False)
    Cfg.env.num_envs = n
    Cfg.domain_rand.lag_timesteps = 6
    Cfg.domain_rand.randomize_lag_timesteps = True
    Cfg.control.control_type = "actuator_net"
    return HistoryWrapper(VelocityTrackingEasyEnv(sim_device="cuda:0", headless=True, cfg=Cfg))


def _load_policy():
    """name -> float32 array, reassembled from the flattened slices `name@offset` (+ `name@shape`) of the part files."""
    import glob
    flat, shape = {}, {}
    for fn in sorted(glob.glob(os.path.join(HERE, "golden", "pretrained_policy_fp16.part*.npz"))):
        z = np.load(fn)
        for key in z.files:
            name, tag = key.rsplit("@", 1)
            if tag == "shape":
                shape[name] = tuple(int(v) for v in z[key])
            else:
                flat.setdefault(name, {})[int(tag)] = z[key]
    out = {}
    for name, chunks in flat.items():
        a = np.concatenate([chunks[o] for o in sorted(chunks)]).astype(np.float32)
        assert a.size == int(np.prod(shape[name])), name
        out[name] = a.reshape(shape[name])
    return out


def test_shipped_policy_trots_forward_in_this_simulator():
    from go1_gym_learn.ppo_cse import ActorCritic
    n = 32
    env = _play_env(n)
    w = _load_policy()
    assert len(w) == 15
    ac = ActorCritic(env.num_obs, env.num_privileged_obs, env.num_obs_history, env.num_actions).to("cuda:0")
    sd = ac.state_dict()
    for k in w:
        sd[k] = torch.from_numpy(w[k])
    ac.load_state_dict(sd)
    obs = env.reset()
    vx, resets = [], 0
    for i in range(250):
        with torch.no_grad():
            actions = ac.act_student(obs["obs_history"]).clone()
        c = env.commands
        c[:, 0] = 1.5; c[:, 1] = 0.0; c[:, 2] = 0.0; c[:, 3] = 0.0; c[:, 4] = 3.0
        c[:, 5] = 0.5; c[:, 6] = 0.0; c[:, 7] = 0.0; c[:, 8] = 0.5; c[:, 9] = 0.08; c[:, 10] = 0.0; c[:, 11] = 0.0; c[:, 12] = 0.25
        obs, rew, done, info = env.step(actions)
        vx.append(env.base_lin_vel[:, 0].clone())
        if i > 20:
            resets += int(done.sum())
    vx = torch.stack(vx)
    mean_v = float(vx[150:].mean())
    z = env.base_pos[:, 2]
    print(f"mean forward velocity over the last 100 steps: {mean_v:.3f} m/s (commanded 1.5); resets after step 20: {resets}; base z {float(z.mean()):.3f}")
    assert resets <= n // 8, f"robots fell: {resets} resets"
    assert 1.0 < mean_v < 1.9, mean_v
    assert 0.2 < float(z.mean()) < 0.4
