"""User reward terms (go1_gym/envs/rewards) on the device: the deferred step kernel, the finish kernel and the reset fold against
the fused kernel's built-in terms and a torch restatement of compute_reward (legged_robot.py:263-300)."""
import os
import sys
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200"))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))
sys.path.insert(0, HERE)

RE_EXPRESSED = {"lin_vel_z": -0.02, "dof_acc": -2.5e-7, "action_rate": -0.01, "action_smoothness_2": -0.1}


def _fresh_cfg(n, episode_s=0.6, combo="ji22", scales=None, container=None):
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    apply_train_config(Cfg)
    Cfg.env.num_envs = n
    Cfg.env.episode_length_s = episode_s             # timeouts within the test's steps
    Cfg.rewards.only_positive_rewards = combo == "clip"
    Cfg.rewards.only_positive_rewards_ji22_style = combo == "ji22"
    for k, v in (scales or {}).items():
        setattr(Cfg.reward_scales, k, v)
    if container is not None:
        from go1_gym.envs.rewards import REWARD_CONTAINERS
        REWARD_CONTAINERS[container.__name__] = container
        Cfg.rewards.reward_container_name = container.__name__
    return Cfg


def _env(cfg, eval_cfg=None):
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    torch.manual_seed(0); np.random.seed(0)          # creation-time randomisation draws from the global generators
    return VelocityTrackingEasyEnv(sim_device="cuda:0", headless=True, cfg=cfg, eval_cfg=eval_cfg)


def _containers():
    from go1_gym.envs.rewards import CoRLRewards

    class ReExpressed(CoRLRewards):
        def _reward_lin_vel_z_u(self):
            return torch.square(self.env.base_lin_vel[:, 2])

        def _reward_dof_acc_u(self):
            return torch.sum(torch.square((self.env.last_dof_vel - self.env.dof_vel) / self.env.dt), dim=1)

        def _reward_action_rate_u(self):
            return torch.sum(torch.square(self.env.last_actions - self.env.actions), dim=1)

        def _reward_action_smoothness_2_u(self):
            e = self.env
            d = e.joint_pos_target[:, :12] - 2 * e.last_joint_pos_target[:, :12] + e.last_last_joint_pos_target[:, :12]
            return torch.sum(torch.square(d) * (e.last_actions != 0) * (e.last_last_actions != 0), dim=1)

    class Override(CoRLRewards):
        def _reward_lin_vel_z(self):
            return torch.square(self.env.base_lin_vel[:, 2])

    return ReExpressed, Override


def _run(env, steps, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    env.reset()
    out = []
    for _ in range(steps):
        a = 2.0 * torch.randn(env.num_envs, 12, device="cuda", generator=g)
        obs, rew, reset, ex = env.step(a)
        ep = dict(ex["train/episode"]) if "train/episode" in ex else {}
        out.append(dict(obs=obs.clone(), rew=rew.clone(), pos=env.rew_buf_pos.clone(), neg=env.rew_buf_neg.clone(),
                        reset=reset.clone(), dof=env.dof_pos.clone(), ep={k: torch.as_tensor(v).float().cpu() for k, v in ep.items()}))
    return out


def test_reexpressed_builtins_match_the_kernel():
    """Four built-ins restated as user terms (they read last_actions / last_dof_vel / last_*_joint_pos_target, so they need the pre-roll
    state) give the same rewards as the kernel; the state does not depend on rewards and stays bit-identical."""
    ReExpressed, _ = _containers()
    plain = _env(_fresh_cfg(256, scales=RE_EXPRESSED))
    a = _run(plain, 60)
    user_scales = {k: 0 for k in RE_EXPRESSED}
    user_scales.update({k + "_u": v for k, v in RE_EXPRESSED.items()})
    env = _env(_fresh_cfg(256, scales=user_scales, container=ReExpressed))
    assert env.user_reward_names == [k + "_u" for k in RE_EXPRESSED]
    b = _run(env, 60)
    assert sum(int(x["reset"].sum()) for x in a) > 256       # episodes ended during the run
    for x, y in zip(a, b):
        assert torch.equal(x["obs"], y["obs"]) and torch.equal(x["dof"], y["dof"]) and torch.equal(x["reset"], y["reset"])
        for k in ("rew", "pos", "neg"):
            torch.testing.assert_close(y[k], x[k], rtol=1e-5, atol=1e-6)
        for k in RE_EXPRESSED:
            if "rew_" + k in x["ep"]:
                torch.testing.assert_close(y["ep"]["rew_" + k + "_u"], x["ep"]["rew_" + k], rtol=1e-5, atol=1e-6)
        if "rew_total" in x["ep"]:
            torch.testing.assert_close(y["ep"]["rew_total"], x["ep"]["rew_total"], rtol=1e-5, atol=1e-6)


def test_override_of_a_builtin_matches_the_kernel():
    _, Override = _containers()
    plain = _run(_env(_fresh_cfg(128, scales={"lin_vel_z": -0.02})), 30)
    env = _env(_fresh_cfg(128, scales={"lin_vel_z": -0.02}, container=Override))
    assert env.user_reward_names == ["lin_vel_z"] and env.sim_cfg.reward_scale[2] == 0.0
    over = _run(env, 30)
    for x, y in zip(plain, over):
        assert torch.equal(x["obs"], y["obs"])
        for k in ("rew", "pos", "neg"):
            torch.testing.assert_close(y[k], x[k], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("combo", ["ji22", "clip", "sum"])
def test_dynamic_sign_and_combination(combo):
    """A user term whose batch sum changes sign from step to step goes to rew_buf_pos or rew_buf_neg by that sum's sign; rew_buf follows
    the configured combination.  The built-in side comes from a twin env with the same single built-in term and the plain sum."""
    from go1_gym.envs.rewards import CoRLRewards
    seen = []

    class Signed(CoRLRewards):
        def _reward_wobble(self):
            c = 0.3 if len(seen) % 3 else -0.4
            r = self.env.base_lin_vel[:, 0] + c
            seen.append(r.clone())
            return r

    only = {"tracking_lin_vel": 0, "tracking_ang_vel": 0, "termination": 0}
    cfg = _fresh_cfg(200, combo="sum", scales=only)
    from go1_b200.config import cfg_dict
    keep = [k for k, v in cfg_dict(cfg.reward_scales).items() if v != 0]
    zero = {k: 0 for k in keep if k != "orientation"}
    zero["orientation"] = -5.0
    twin = _run(_env(_fresh_cfg(200, combo="sum", scales={**only, **zero})), 12)
    env = _env(_fresh_cfg(200, combo=combo, scales={**only, **zero, "wobble": 0.5}, container=Signed))
    sigma = env.cfg.rewards.sigma_rew_neg
    seen.clear()
    got = _run(env, 12)
    sc = env.reward_scales["wobble"]
    signs = set()
    for t, (x, y) in enumerate(zip(twin, got)):
        r = seen[t + 1] * np.float32(sc)             # seen[0]: the step inside env.reset()
        s = r.double().sum().item()
        signs.add(s >= 0)
        pos = x["pos"] + (r if s >= 0 else 0)
        neg = x["neg"] + (r if s < 0 else 0)
        rew = x["rew"] + r
        if combo == "clip":
            rew = rew.clamp(min=0)
        elif combo == "ji22":
            rew = pos * torch.exp(neg / sigma)
        torch.testing.assert_close(y["pos"], pos, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(y["neg"], neg, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(y["rew"], rew, rtol=1e-5, atol=1e-6)
    assert signs == {True, False}


def _runner(n, container, scales, graph, monkeypatch, tmp_path, policy_graph=True):
    monkeypatch.setenv("GO1_STEP_GRAPH", "1" if graph else "0")
    cfg = _fresh_cfg(n, episode_s=20.0, scales=scales, container=container)
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    from ml_logger import logger
    logger.configure(prefix="run", root=str(tmp_path))
    RunnerArgs.num_steps_per_env, RunnerArgs.resume, RunnerArgs.save_video_interval, RunnerArgs.log_freq = 8, False, 100, 1
    RunnerArgs.save_interval = 100
    env = HistoryWrapper(_env(cfg))
    runner = Runner(env, device="cuda:0")
    runner.alg.use_cuda_graph = policy_graph      # the policy-only graph's capture warm-up draws from the action-noise stream
    return env, runner, logger


def _rollout_rewards(env, runner):
    """Stored rewards of two rollouts (the second replays the graphs captured in the first)."""
    g = torch.Generator().manual_seed(1)
    env.episode_length_buf = torch.randint(0, int(env.env.max_episode_length), (env.num_envs,), generator=g)
    od = env.get_observations()
    state, out = (od["obs"], od["privileged_obs"], od["obs_history"]), []
    for _ in range(2):
        obs, priv, hist, _ = runner.rollout(*state)
        state = (obs, priv, hist)
        out.append(runner.alg.storage.rewards.clone())
        runner.alg.storage.clear()
    return torch.stack(out)


def test_graph_replay_matches_eager_and_falls_back_on_host_sync(monkeypatch, tmp_path):
    from go1_gym.envs.rewards import CoRLRewards

    class Cheap(CoRLRewards):
        def _reward_upright(self):
            return self.env.projected_gravity[:, 2] ** 2

        def _reward_action_rate_u(self):        # this step's actions and the pre-roll last_actions
            return torch.sum(torch.square(self.env.last_actions - self.env.actions), dim=1)

    class Syncs(CoRLRewards):
        def _reward_upright(self):
            if self.env.projected_gravity[:, 2].sum().item() > 1e30:
                raise AssertionError
            return self.env.projected_gravity[:, 2] ** 2

    scales = {"upright": 0.3}
    cheap_scales = {"upright": 0.3, "action_rate": 0, "action_rate_u": -0.01}
    env, runner, _ = _runner(64, Cheap, cheap_scales, True, monkeypatch, tmp_path)
    graphed = _rollout_rewards(env, runner)
    assert runner._sg is not None and runner._sg["graphs"], "the rollout was not graph-replayed"
    assert float(env.env.episode_sums["action_rate_u"].abs().sum()) > 0
    env, runner, _ = _runner(64, Cheap, cheap_scales, False, monkeypatch, tmp_path, policy_graph=False)
    eager = _rollout_rewards(env, runner)
    assert torch.equal(graphed, eager)
    # the same term as the kernel's built-in action_rate: graph-replayed rollouts agree with the kernel within rounding
    env, runner, _ = _runner(64, Cheap, {"upright": 0.3, "action_rate": -0.01}, True, monkeypatch, tmp_path)
    torch.testing.assert_close(_rollout_rewards(env, runner), graphed, rtol=1e-5, atol=1e-6)
    env, runner, _ = _runner(64, Syncs, scales, False, monkeypatch, tmp_path)
    eager_sync = _rollout_rewards(env, runner)
    env, runner, _ = _runner(64, Syncs, scales, True, monkeypatch, tmp_path)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        synced = _rollout_rewards(env, runner)
    assert len([x for x in w if "cannot be captured" in str(x.message)]) == 1
    assert runner._sg is None
    assert torch.equal(synced, eager_sync)


def test_eval_envs_keep_their_first_episode():
    from env_golden_util import clone_cfg
    from go1_gym.envs.rewards import CoRLRewards
    seen = []

    class Counted(CoRLRewards):
        def _reward_height(self):
            r = self.env.base_pos[:, 2].clone()
            seen.append(r)
            return r

    cfg = _fresh_cfg(48, episode_s=0.3, scales={"height": 0.2}, container=Counted)
    ecfg = clone_cfg(cfg, "EvalCfg")
    ecfg.env.num_envs = 16
    env = _env(cfg, ecfg)
    assert env.num_eval_envs == 16
    sc = np.float32(env.reward_scales["height"])
    env.reset()
    env._user_sums_eval.fill_(-1.0)          # env.reset() filed the empty episodes; start the record from here
    seen.clear()
    running = env.episode_sums["height"].clone()
    first = torch.full((env.num_envs,), -1.0, device="cuda")
    for _ in range(40):
        env.step(torch.randn(env.num_envs, 12, device="cuda"))
        running += seen[-1] * sc
        done = env.reset_buf
        first = torch.where(done & (first == -1), running, first)
        running = torch.where(done, torch.zeros_like(running), running)
    ev = env.num_train_envs
    assert (first[ev:] != -1).all()
    torch.testing.assert_close(env.episode_sums_eval["height"][ev:], first[ev:], rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(env.episode_sums["height"], running, rtol=1e-5, atol=1e-6)


def test_training_logs_user_terms(monkeypatch, tmp_path):
    from go1_gym.envs.rewards import CoRLRewards

    class Cheap(CoRLRewards):
        def _reward_upright(self):
            return self.env.projected_gravity[:, 2] ** 2

    monkeypatch.chdir(tmp_path)
    env, runner, logger = _runner(64, Cheap, {"upright": 0.3}, True, monkeypatch, tmp_path)
    runner.learn(num_learning_iterations=2, init_at_random_ep_len=True)
    assert torch.isfinite(runner.alg.actor_critic.flat_params).all()
    assert any("train/episode/rew_upright/mean" in row for row in logger.summaries)


def _kernel_trace(env, steps=3):
    """Distinct kernel names in the profiler's list over `steps` env steps, and the library's count of its launches in them."""
    from go1_b200 import capi
    from torch.profiler import ProfilerActivity, profile
    L = capi.lib()
    env.reset()
    a = torch.zeros(env.num_envs, 12, device="cuda")
    env.step(a)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        n0 = L.go1_kernel_launch_count()
        for _ in range(steps):
            env.step(a)
        n = L.go1_kernel_launch_count() - n0
        torch.cuda.synchronize()
    names = {e.name for e in p.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memset" not in e.name and "Memcpy" not in e.name}
    return names, n


def test_no_user_term_launches_what_the_kernel_alone_launches():
    from go1_gym.envs.rewards import CoRLRewards

    class ZeroScale(CoRLRewards):
        def _reward_unused(self):
            raise AssertionError("a zero-scale term must not run")

    _kernel_trace(_env(_fresh_cfg(64)))          # the first profiled window of a process also initialises the tracer
    base, n_base = _kernel_trace(_env(_fresh_cfg(64)))
    assert any("go1_step_kernel<false, false>" in n for n in base)
    for cls, scales in ((CoRLRewards, {}), (ZeroScale, {"unused": 0.0})):
        env = _env(_fresh_cfg(64, scales=scales, container=type(cls.__name__ + "Only", (cls,), {})))
        assert env.user_reward_names == []
        names, n = _kernel_trace(env)
        assert names == base and n == n_base
        assert not any(k in x for x in names for k in ("reward_finish", "reward_partials", "user_reward_fold", "true>"))
