"""Cfg.domain_rand.lag_timesteps (the action FIFO depth L, 0..32 substeps) on the H100: the fused step kernel against vectors produced
by the reference's own LeggedRobot._compute_torques (tests/golden/lag.npz), the reset kernel, the C-ABI range check, and whole-env
rollouts.  FIFO rows and joint targets are compared bit for bit, torques with test_sim_gpu.py's tolerance."""
import os
import sys

import numpy as np
import pytest
import torch

import lag_util as U
from test_lag_oracle import lag_config, load_lag_gold
from oracle import env_oracle as eo

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SENTINEL = 7.25


def _sim(n, L, control_type="actuator_net", decimation=4):
    from go1_b200.sim import SimCore
    _, c, info = lag_config(n, L, control_type, decimation)
    c.rand_interval = 0
    return c, info, SimCore(c, inject_noise=True, inject_reset_rand=True)


def _fifo(sim, L):
    """The L live slots as [L][N][12] (slot i = rows 3i..3i+2)."""
    return sim.leg("lag_buffer")[:3 * L].reshape(L, 3, sim.N, 4).permute(0, 2, 3, 1).reshape(L, sim.N, 12).cpu().numpy()


def _set_fifo(sim, fifo):
    lag = sim.leg("lag_buffer")
    for i in range(fifo.shape[0]):
        lag[3 * i:3 * i + 3].copy_(fifo[i].reshape(sim.N, 4, 3).permute(2, 0, 1))


def _load_case(sim, c, case):
    L = U.CASES[case][0]
    x = {k: torch.from_numpy(v).cuda() for k, v in U.inputs(case, np.array(c.default_dof_pos, dtype=np.float32)).items()}
    for k in ("dof_pos", "dof_vel", "joint_pos_err_last", "joint_pos_err_last_last", "joint_vel_last", "joint_vel_last_last", "motor_offsets"):
        sim.set_joint_aos(k, x[k])
    sim.env("motor_strengths")[0].copy_(x["motor_strengths"])
    sim.leg("lag_buffer")[3 * L:].fill_(SENTINEL)
    _set_fifo(sim, x["fifo"])
    return x


def _sentinel_intact(sim, L):
    return bool((sim.leg("lag_buffer")[3 * L:] == SENTINEL).all())


@pytest.mark.parametrize("case", list(U.CASES))
def test_single_substeps_match_reference(case):
    """mode 1: one control substep per call (no physics), so targets, torques and the FIFO are checked after every substep."""
    g = load_lag_gold()
    L, control_type, decimation = U.CASES[case]
    c, info, sim = _sim(U.N, L, control_type, decimation)
    x = _load_case(sim, c, case)
    k = 0
    for t in range(U.T):
        for _ in range(decimation):
            sim.step(x["actions"][t].contiguous(), mode=1)
            torch.cuda.synchronize()
            assert np.array_equal(sim.joint_aos("joint_pos_target").cpu().numpy(), g[f"{case}/target"][k]), (case, k)
            assert np.allclose(sim.joint_aos("torques").cpu().numpy(), g[f"{case}/torque"][k], rtol=1e-5, atol=5e-5), (case, k)
            assert np.array_equal(_fifo(sim, L), g[f"{case}/fifo"][k]), (case, k)
            assert _sentinel_intact(sim, L), (case, k)
            k += 1


@pytest.mark.parametrize("case", list(U.CASES))
def test_full_steps_match_reference(case):
    """mode 0: `decimation` substeps with physics per call.  The FIFO and the targets do not depend on the physics, so the FIFO and
    the last substep's target after every policy step are bit-exact against the reference."""
    g = load_lag_gold()
    L, control_type, decimation = U.CASES[case]
    c, info, sim = _sim(U.N, L, control_type, decimation)
    x = _load_case(sim, c, case)
    sim.env("root_pos")[2].fill_(0.32)
    for t in range(U.T):
        sim.step(x["actions"][t].contiguous(), common_step=t, mode=0)
        torch.cuda.synchronize()
        k = (t + 1) * decimation - 1
        assert np.array_equal(sim.joint_aos("joint_pos_target").cpu().numpy(), g[f"{case}/target"][k]), (case, t)
        assert np.array_equal(_fifo(sim, L), g[f"{case}/fifo"][k]), (case, t)
        assert _sentinel_intact(sim, L), (case, t)


@pytest.mark.parametrize("L", [0, 1, 6, 13, 32])
def test_reset_zeroes_exactly_the_live_slots(L):
    n = 8
    c, info, sim = _sim(n, L)
    before = torch.rand(3 * 32, n, 4, generator=torch.Generator().manual_seed(L)).cuda() + 1.0
    sim.leg("lag_buffer").copy_(before)
    ids = np.array([1, 4, 6])
    sim.reset_idx(ids, np.zeros((len(ids), 15), np.float32))
    torch.cuda.synchronize()
    want = before.clone()
    want[:3 * L, torch.from_numpy(ids).cuda()] = 0.0
    assert torch.equal(sim.leg("lag_buffer"), want)


def test_without_use_lag_no_kernel_touches_the_fifo():
    """A C caller may leave lag_timesteps set with use_lag = 0: the step and reset kernels then neither read nor write the FIFO rows."""
    from go1_b200.sim import SimCore
    n = 8
    _, c, _ = lag_config(n, 6, randomize_lag_timesteps=False)
    c.rand_interval, c.lag_timesteps = 0, 6
    sim = SimCore(c, inject_noise=True, inject_reset_rand=True)
    before = torch.rand(3 * 32, n, 4, generator=torch.Generator().manual_seed(3)).cuda() + 1.0
    sim.leg("lag_buffer").copy_(before)
    sim.env("root_pos")[2].fill_(0.32)
    actions = torch.rand(n, 12, generator=torch.Generator().manual_seed(4)).cuda()
    sim.step(actions, mode=1)
    torch.cuda.synchronize()
    want = actions.cpu() * c.action_scale               # the target is this step's action, not a FIFO slot
    want[:, 0::3] *= c.hip_scale_reduction
    want += torch.tensor(list(c.default_dof_pos))
    assert np.array_equal(sim.joint_aos("joint_pos_target").cpu().numpy(), want.numpy())
    sim.step(actions, mode=0)
    sim.reset_idx(np.array([1, 4, 6]), np.zeros((3, 15), np.float32))
    torch.cuda.synchronize()
    assert torch.equal(sim.leg("lag_buffer"), before)


def test_abi_rejects_out_of_range_lag_before_any_launch():
    from go1_b200 import capi
    from go1_b200.sim import SimCore
    lib = capi.lib()
    _, c, _ = lag_config(16, 6)
    n0 = lib.go1_kernel_launch_count()
    for bad in (33, -1):
        c.lag_timesteps = bad
        with pytest.raises(capi.Go1Error, match=r"lag_timesteps .* 0\.\.32"):
            SimCore(c)
    c.lag_timesteps = 6
    sim = SimCore(c)
    for bad in (33, -1):
        sim.cfg.lag_timesteps = bad
        with pytest.raises(capi.Go1Error, match=r"lag_timesteps .* 0\.\.32"):
            sim.update_config()
    torch.cuda.synchronize()
    assert lib.go1_kernel_launch_count() == n0


def _env(n, **dr):
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    apply_train_config(Cfg)
    Cfg.env.num_envs = n
    for k, v in dr.items():
        setattr(Cfg.domain_rand, k, v)
    torch.manual_seed(0)            # creation-time domain randomisation draws from torch's global generators
    torch.cuda.manual_seed_all(0)
    return VelocityTrackingEasyEnv(sim_device="cuda:0", headless=True, cfg=Cfg)


def test_zero_lag_equals_no_lag_rollout():
    """lag_timesteps = 0 is the reference's randomize_lag_timesteps = False: every observation, reward and reset agrees bit for bit."""
    N, T = 256, 50
    envs = [_env(N, randomize_lag_timesteps=True, lag_timesteps=0), _env(N, randomize_lag_timesteps=False)]
    assert envs[0].core.cfg.use_lag == 1 and envs[1].core.cfg.use_lag == 0
    g = torch.Generator().manual_seed(5)
    ep0 = torch.randint(0, 1001, (N,), generator=g)
    for e in envs:
        e.reset()
        e.episode_length_buf = ep0.clone()
    n_reset = 0
    for t in range(T):
        a = (torch.randn(N, 12, generator=g) * (2.5 if t % 7 else 6.0)).cuda()
        outs = [e.step(a.clone()) for e in envs]
        torch.cuda.synchronize()
        for name, i in (("obs", 0), ("rew", 1), ("reset", 2)):
            assert torch.equal(outs[0][i], outs[1][i]), (t, name)
        assert torch.equal(envs[0].core.env_f32, envs[1].core.env_f32), t
        n_reset += int(outs[0][2].sum())
    assert n_reset > 10


@pytest.mark.parametrize("L", [2, 13, 32])
def test_control_rollout_with_resets_matches_oracle(L):
    """20 policy steps of 4 control substeps (mode 1) with random actions, and random envs reset after every step: the kernel's FIFO
    and targets equal the CPU oracle's (oracle/env_oracle.py, FIFO of L + 1 entries, zeroed for reset envs) bit for bit."""
    N, T = 64, 20
    c, info, sim = _sim(N, L)
    P = eo.params_from_sim_config(c, info["active_reward_scales"], info["dt"])
    net = eo.ActuatorNet()
    rng = np.random.default_rng(100 + L)
    f = lambda lo, hi, *s: torch.from_numpy(rng.uniform(lo, hi, s).astype(np.float32))
    sim.reset_rand.copy_(f(0, 1, N, 48))
    s = dict(dof_pos=torch.tensor(list(c.default_dof_pos)) + f(-0.5, 0.5, N, 12), dof_vel=f(-5, 5, N, 12),
             lag_buffer=[torch.zeros(N, 12)] + [f(-0.6, 0.6, N, 12) for _ in range(L)])
    for k in ("joint_pos_err_last", "joint_pos_err_last_last", "joint_vel_last", "joint_vel_last_last", "motor_offsets"):
        s[k] = torch.zeros(N, 12)
    s["motor_strengths"], s["Kp_factors"], s["Kd_factors"] = torch.ones(N, 12), torch.ones(N, 12), torch.ones(N, 12)
    sim.set_joint_aos("dof_pos", s["dof_pos"].cuda()); sim.set_joint_aos("dof_vel", s["dof_vel"].cuda())
    _set_fifo(sim, torch.stack(s["lag_buffer"][1:]).cuda())
    n_reset = 0
    for t in range(T):
        a = f(-3, 3, N, 12)
        s["actions"] = a.clone()
        for sub in range(c.decimation):
            sim.step(a.cuda(), mode=1)
            tq = eo.compute_torques(s, P, net)
            torch.cuda.synchronize()
            assert np.array_equal(sim.joint_aos("joint_pos_target").cpu().numpy(), s["joint_pos_target"].numpy()), (L, t, sub)
            assert np.allclose(sim.joint_aos("torques").cpu().numpy(), tq.numpy(), rtol=1e-5, atol=5e-5), (L, t, sub)
            assert np.array_equal(_fifo(sim, L), torch.stack(s["lag_buffer"][1:]).numpy()), (L, t, sub)
        ids = np.sort(rng.choice(N, size=int(rng.integers(1, N // 4)), replace=False))
        n_reset += len(ids)
        sim.reset_idx(ids, np.zeros((len(ids), 15), np.float32), common_step=t)
        torch.cuda.synchronize()
        for b in s["lag_buffer"]:
            b[torch.from_numpy(ids)] = 0.0
        # the reset kernel's own draws (dof state, motor DR; pinned by test_dr_gpu.py) continue the oracle's state
        s["dof_pos"], s["dof_vel"] = sim.joint_aos("dof_pos").cpu(), sim.joint_aos("dof_vel").cpu()
        s["motor_offsets"] = sim.joint_aos("motor_offsets").cpu()
        s["motor_strengths"] = sim.env("motor_strengths")[0].cpu()[:, None].repeat(1, 12)
    assert n_reset > 100
    assert np.array_equal(_fifo(sim, L), torch.stack(s["lag_buffer"][1:]).numpy())


def _runner_env(tmp_path, n, L):
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    from ml_logger import logger
    apply_train_config(Cfg)
    Cfg.env.num_envs = n
    Cfg.domain_rand.lag_timesteps = L
    logger.configure(prefix="run", root=str(tmp_path))
    return HistoryWrapper(VelocityTrackingEasyEnv(sim_device="cuda:0", headless=True, cfg=Cfg))


def test_graph_replayed_rollout_equals_eager_at_lag_13(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    keep = (RunnerArgs.num_steps_per_env, RunnerArgs.resume)
    out = []
    try:
        for graphed in (False, True):
            torch.manual_seed(0); np.random.seed(0)
            env = _runner_env(tmp_path, 256, 13)
            assert env.env.core.cfg.lag_timesteps == 13
            RunnerArgs.num_steps_per_env, RunnerArgs.resume = 24, False
            runner = Runner(env, device="cuda:0")
            runner.step_graph = graphed
            if not graphed:       # launch by launch, and without the policy-only graph (its capture warm-up draws from the action-noise stream)
                runner.alg.use_cuda_graph = False
            env.episode_length_buf = torch.randint(0, 1001, (256,), generator=torch.Generator().manual_seed(1))
            od = env.get_observations()
            state = (od["obs"], od["privileged_obs"], od["obs_history"])
            snaps = []
            for it in range(2):                  # the second rollout replays graphs captured during the first
                state = runner.rollout(*state)[:3]
                torch.cuda.synchronize()
                st = runner.alg.storage
                snaps.append({k: getattr(st, k).clone() for k in ("observations", "actions", "rewards", "dones", "values")})
                snaps[-1]["env_f32"], snaps[-1]["leg_f32"] = env.env.core.env_f32.clone(), env.env.core.leg_f32.clone()
                runner.alg.storage.clear()
            out.append(snaps)
    finally:
        RunnerArgs.num_steps_per_env, RunnerArgs.resume = keep
    for it in range(2):
        assert int(out[0][it]["dones"].sum()) > 0
        for k in out[0][it]:
            assert torch.equal(out[0][it][k], out[1][it][k]), (it, k)


def test_runner_learn_at_lag_13(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    env = _runner_env(tmp_path, 256, 13)
    keep = (RunnerArgs.num_steps_per_env, RunnerArgs.save_interval, RunnerArgs.log_freq, RunnerArgs.save_video_interval, RunnerArgs.resume)
    RunnerArgs.num_steps_per_env, RunnerArgs.save_interval, RunnerArgs.log_freq, RunnerArgs.save_video_interval, RunnerArgs.resume = 8, 100, 1, 100, False
    try:
        runner = Runner(env, device="cuda:0")
        w0 = runner.alg.actor_critic.flat_params.clone()
        runner.learn(num_learning_iterations=2, init_at_random_ep_len=True, eval_freq=100)
    finally:
        RunnerArgs.num_steps_per_env, RunnerArgs.save_interval, RunnerArgs.log_freq, RunnerArgs.save_video_interval, RunnerArgs.resume = keep
    ac = runner.alg.actor_critic
    assert torch.isfinite(ac.flat_params).all() and not torch.equal(ac.flat_params, w0)
    assert np.isfinite(runner.alg._acc.cpu().numpy()).all()
    assert torch.isfinite(env.env.core.leg_f32).all()
