"""The self-collision instantiation of the step kernel against the fp64 self-collision oracle, the default kernel against it at
nominal poses, and the rule that the model is fixed once the sim has stepped."""
import numpy as np
import pytest
import torch

from env_golden_util import train_sim_config

pytestmark = pytest.mark.gpu


def _self_cfg(on=True):
    from go1_b200 import capi
    import self_collision_oracle as so
    sc = capi.Go1SelfCollision()
    sc.enabled = int(on)
    sc.k, sc.c = so.DEFAULTS["k"], so.DEFAULTS["c"]
    sc.thigh_radius, sc.calf_radius, sc.foot_radius = so.DEFAULTS["thigh_radius"], so.DEFAULTS["calf_radius"], so.DEFAULTS["foot_radius"]
    return sc


def _crossed_states(n, seed):
    """Free-flight states (2 m up) with the front and rear legs adducted towards each other and closing at a few rad/s."""
    from oracle import physics as ph
    rng = np.random.default_rng(seed)
    q = np.tile(ph.DEFAULT_DOF_POS, (n, 1))
    for j, sgn in ((0, -1), (3, 1), (6, -1), (9, 1)):
        q[:, j] = sgn * rng.uniform(0.25, 0.4, n)
    qd = rng.uniform(-0.5, 0.5, (n, 12))
    for j, sgn in ((0, -1), (3, 1), (6, -1), (9, 1)):
        qd[:, j] += sgn * 3.0
    return dict(pos=np.stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), np.full(n, 2.0)], 1), quat=np.tile([0, 0, 0, 1.0], (n, 1)),
                linvel=rng.uniform(-0.2, 0.2, (n, 3)), angvel=rng.uniform(-0.2, 0.2, (n, 3)), q=q, qd=qd,
                friction=rng.uniform(0.5, 1.25, n), restitution=np.zeros(n), payload=np.zeros(n)), rng


def _run(st, n, steps, sc, g):
    from go1_b200.sim import SimCore
    from test_sim_gpu import _load_phys_state
    Cfg, c, info = train_sim_config(n, cfg_overrides={"control": {"control_type": "P"}})
    c.rand_interval = 0
    sim = SimCore(c, inject_noise=True, inject_reset_rand=True, self_collision=sc)
    _load_phys_state(sim, st)
    sim.set_gravity(g, [0, 0, -1])
    actions = torch.zeros(n, 12, device="cuda")
    for t in range(steps):
        sim.step(actions, common_step=t, mode=0)
    torch.cuda.synchronize()
    got = dict(pos=sim.env("root_pos").t().cpu().numpy(), quat=sim.env("root_quat").t().cpu().numpy(),
               linvel=sim.env("root_lin_vel").t().cpu().numpy(), angvel=sim.env("root_ang_vel").t().cpu().numpy(),
               q=sim.joint_aos("dof_pos").cpu().numpy(), qd=sim.joint_aos("dof_vel").cpu().numpy())
    return sim, c, info, got


FEET, THIGH, CALF = [4, 8, 12, 16], [2, 6, 10, 14], [3, 7, 11, 15]
TOL = dict(pos=2e-4, quat=3e-4, linvel=5e-3, angvel=2e-2, q=1e-3, qd=5e-2)      # test_sim_gpu.physics_vs_oracle's


def _rows(sim):
    """The kernel's reported contact rows in Isaac Gym body order [n][17][3] (base, then hip, thigh, calf, foot per leg; hips 0)."""
    n = sim.N
    out = np.zeros((n, 17, 3))
    out[:, 0] = sim.foot_aos("base_contact_forces_part").cpu().numpy().sum(1)
    for rows, name in ((THIGH, "thigh_contact_forces"), (CALF, "calf_contact_forces"), (FEET, "foot_contact_forces")):
        out[:, rows] = sim.foot_aos(name).cpu().numpy()
    return out


def _state(sim):
    return dict(pos=sim.env("root_pos").t().cpu().numpy(), quat=sim.env("root_quat").t().cpu().numpy(),
                linvel=sim.env("root_lin_vel").t().cpu().numpy(), angvel=sim.env("root_ang_vel").t().cpu().numpy(),
                q=sim.joint_aos("dof_pos").cpu().numpy(), qd=sim.joint_aos("dof_vel").cpu().numpy())


def _actions_for(c, q_target):
    """Actions whose joint targets are q_target (P control: target = default + action_scale * action, hips also x hip_scale_reduction)."""
    scale = np.full(12, c.action_scale)
    scale[[0, 3, 6, 9]] *= c.hip_scale_reduction
    return ((q_target - np.array(list(c.default_dof_pos))) / scale).astype(np.float32)


def _kernel_vs_oracle(st, steps, q_target=None, no_limits=False, unactuated=False):
    """`steps` policy steps of the kernel (P control, zero actions, no gravity) and of the fp64 oracle from the same state.  After
    every step: the state within TOL (95 % of envs, median below TOL / 10) and the thigh, calf, foot and base rows of the last
    substep within 0.5 N for 90 % of envs.  Returns (envs with a self-contact, per-step row maxima of the oracle, kernel states)."""
    from go1_b200.sim import SimCore
    from oracle import physics as ph
    from oracle import env_oracle as eo
    import self_collision_oracle as so
    from test_sim_gpu import _load_phys_state
    n = len(st["pos"])
    Cfg, c, info = train_sim_config(n, cfg_overrides={"control": {"control_type": "P"}})
    c.rand_interval = 0
    if no_limits:
        c.limit_k = c.limit_c = 0.0
    act = np.zeros((n, 12), dtype=np.float32) if q_target is None else _actions_for(c, q_target)
    assert np.abs(act).max() < c.clip_actions
    sim = SimCore(c, inject_noise=True, inject_reset_rand=True, self_collision=_self_cfg())
    _load_phys_state(sim, st)
    if unactuated:
        sim.env("motor_strengths")[0].fill_(0.0)
    sim.set_gravity([0.0, 0.0, 0.0], [0, 0, -1])
    P = eo.params_from_sim_config(c, info["active_reward_scales"], info["dt"])
    s = dict(actions=torch.from_numpy(act), dof_pos=torch.tensor(st["q"], dtype=torch.float32), dof_vel=torch.tensor(st["qd"], dtype=torch.float32),
             lag_buffer=[torch.zeros(n, 12) for _ in range(7)], motor_offsets=torch.zeros(n, 12),
             motor_strengths=torch.zeros(n, 12) if unactuated else torch.ones(n, 12),
             Kp_factors=torch.ones(n, 12), Kd_factors=torch.ones(n, 12))
    for k in ("joint_pos_err_last", "joint_pos_err_last_last", "joint_vel_last", "joint_vel_last_last"):
        s[k] = torch.zeros(n, 12)
    pp = ph.default_params()
    pp.gravity[2] = 0.0
    if no_limits:
        pp.limit_k = pp.limit_c = 0.0
    states = [ph.make_state(st["pos"][i], st["quat"][i], st["linvel"][i], st["angvel"][i], st["q"][i], st["qd"][i]) for i in range(n)]
    drs = [ph.make_dr(st["friction"][i], 0.0, 0.0) for i in range(n)]
    touched = np.zeros(n, dtype=bool)
    row_max, kstates = [], []
    for step in range(steps):
        sim.step(torch.from_numpy(act).cuda(), common_step=step, mode=0)
        for sub in range(4):
            tau = eo.compute_torques(s, P).numpy().astype(np.float64)
            cf = np.zeros((n, 17, 3))
            for i in range(n):
                cf[i], h = so.substep(pp, drs[i], states[i], tau[i], so.DEFAULTS)
                touched[i] |= h > 0
            s["dof_pos"] = torch.tensor(np.array([np.array(x.q) for x in states]), dtype=torch.float32)
            s["dof_vel"] = torch.tensor(np.array([np.array(x.qd) for x in states]), dtype=torch.float32)
        torch.cuda.synchronize()
        got = _state(sim)
        want = {k: np.array([np.array(getattr(x, k)) for x in states]) for k in got}
        for k in want:
            err = np.abs(got[k] - want[k]).max(axis=1)
            assert (err < TOL[k]).mean() >= 0.95, (step, k, np.sort(err)[-5:])
            assert np.median(err) < 0.1 * TOL[k], (step, k, np.median(err))
        rows = [0] + THIGH + CALF + FEET
        kr = _rows(sim)
        errf = np.abs(kr[:, rows] - cf[:, rows]).reshape(n, -1).max(axis=1)
        assert (errf < 0.5).mean() >= 0.9, (step, np.sort(errf)[-8:])
        row_max.append({name: np.abs(cf[:, r]).reshape(n, -1).max(axis=1) for name, r in (("base", [0]), ("thigh", THIGH), ("calf", CALF), ("foot", FEET))})
        kstates.append(got)
    return touched, row_max, kstates


@pytest.mark.parametrize("steps", [1, 5])
def test_self_collision_kernel_matches_fp64_oracle(steps):
    """Crossed-leg free flight (gravity 0, 2 m up): trajectories and contact rows against the oracle over 1 and 5 policy steps;
    at least half of the envs touch, and within 5 steps the calf and foot rows carry self-contact forces at a step's end."""
    n = 96
    st, rng = _crossed_states(n, 5)
    q_target = st["q"].copy()                  # PD targets past the crossing: the legs stay pressed together
    q_target[:, [0, 6]], q_target[:, [3, 9]] = -0.6, 0.6
    touched, row_max, _ = _kernel_vs_oracle(st, steps, q_target)
    assert touched.mean() >= 0.5, touched.mean()
    if steps == 5:                              # the legs close again after the first contacts: by then calf and foot rows carry force
        hit = {k: max((m[k] > 0.2).sum() for m in row_max) for k in ("calf", "foot")}
        assert min(hit.values()) > 0, hit


def test_knee_into_trunk_rows_match_oracle():
    """The knee probe against the trunk (FL hip rolled under the body, thigh at 1.18 rad and closing; no pose inside the URDF limits
    brings the knee to the trunk, so the joint limits and motors are off): the base and thigh rows carry the contact, in the kernel
    as in the oracle."""
    from oracle import physics as ph
    n = 32
    rng = np.random.default_rng(7)
    q = np.tile(ph.DEFAULT_DOF_POS, (n, 1))
    q[:, 0], q[:, 1], q[:, 2] = -2.6166666666666667 + rng.uniform(-0.01, 0.01, n), 1.1775, -2.7
    qd = np.zeros((n, 12)); qd[:, 1] = rng.uniform(0.2, 0.5, n)
    st = dict(pos=np.stack([np.zeros(n), np.zeros(n), np.full(n, 2.0)], 1), quat=np.tile([0, 0, 0, 1.0], (n, 1)),
              linvel=np.zeros((n, 3)), angvel=np.zeros((n, 3)), q=q, qd=qd, friction=np.ones(n), restitution=np.zeros(n), payload=np.zeros(n))
    touched, row_max, _ = _kernel_vs_oracle(st, 1, no_limits=True, unactuated=True)
    assert touched.all()
    assert (row_max[0]["base"] > 0.2).mean() >= 0.5 and (row_max[0]["thigh"] > 0.2).mean() >= 0.5, row_max[0]


def test_kernel_momentum_change_matches_oracle():
    """The explicit penalty at dt = 5 ms does not conserve momentum exactly (semi-implicit Euler on stiff contacts: both the kernel
    and the oracle drift by up to ~0.3 kg m/s over 5 policy steps of legs colliding at 3 rad/s).  The kernel's spatial-force route
    must change the linear and angular momentum as the oracle's joint-torque route does: a missing reaction, a wrong moment arm or
    frame would not."""
    from oracle import physics as ph
    from test_physics_oracle import momentum_energy
    n = 64
    st, _ = _crossed_states(n, 11)
    _, _, ks = _kernel_vs_oracle(st, 5)
    # the oracle's states after 5 steps are what _kernel_vs_oracle compared against; recompute them here from its own run
    import self_collision_oracle as so
    from oracle import env_oracle as eo
    Cfg, c, info = train_sim_config(n, cfg_overrides={"control": {"control_type": "P"}})
    P = eo.params_from_sim_config(c, info["active_reward_scales"], info["dt"])
    s = dict(actions=torch.zeros(n, 12), dof_pos=torch.tensor(st["q"], dtype=torch.float32), dof_vel=torch.tensor(st["qd"], dtype=torch.float32),
             lag_buffer=[torch.zeros(n, 12) for _ in range(7)], motor_offsets=torch.zeros(n, 12), motor_strengths=torch.ones(n, 12),
             Kp_factors=torch.ones(n, 12), Kd_factors=torch.ones(n, 12))
    for k in ("joint_pos_err_last", "joint_pos_err_last_last", "joint_vel_last", "joint_vel_last_last"):
        s[k] = torch.zeros(n, 12)
    pp = ph.default_params()
    pp.gravity[2] = 0.0
    states = [ph.make_state(st["pos"][i], st["quat"][i], st["linvel"][i], st["angvel"][i], st["q"][i], st["qd"][i]) for i in range(n)]
    m0 = [momentum_energy(x)[:2] for x in states]
    for sub in range(20):
        tau = eo.compute_torques(s, P).numpy().astype(np.float64)
        for i in range(n):
            so.substep(pp, ph.make_dr(st["friction"][i], 0.0, 0.0), states[i], tau[i], so.DEFAULTS)
        s["dof_pos"] = torch.tensor(np.array([np.array(x.q) for x in states]), dtype=torch.float32)
        s["dof_vel"] = torch.tensor(np.array([np.array(x.qd) for x in states]), dtype=torch.float32)
    got = ks[-1]
    err = []
    for i in range(n):
        Pk, Lk, _, _ = momentum_energy(ph.make_state(*(got[k][i].astype(np.float64) for k in ("pos", "quat", "linvel", "angvel", "q", "qd"))))
        Po, Lo, _, _ = momentum_energy(states[i])
        dk, do = (Pk - m0[i][0], Lk - m0[i][1]), (Po - m0[i][0], Lo - m0[i][1])
        err.append((np.abs(dk[0] - do[0]).max(), np.abs(dk[1] - do[1]).max(), np.abs(do[0]).max()))
    err = np.array(err)
    assert (err[:, 2] > 0.05).sum() >= 5                     # the motion does move momentum
    assert (err[:, 0] < 0.02).mean() >= 0.95 and (err[:, 1] < 0.02).mean() >= 0.95, np.sort(err, axis=0)[-5:]


def test_nominal_standing_is_unchanged_by_the_switch():
    from oracle import physics as ph
    n = 128
    rng = np.random.default_rng(1)
    st = dict(pos=np.stack([np.zeros(n), np.zeros(n), np.full(n, 0.32)], 1), quat=np.tile([0, 0, 0, 1.0], (n, 1)),
              linvel=np.zeros((n, 3)), angvel=np.zeros((n, 3)), q=ph.DEFAULT_DOF_POS + rng.uniform(-0.05, 0.05, (n, 12)),
              qd=np.zeros((n, 12)), friction=np.ones(n), restitution=np.zeros(n), payload=np.zeros(n))
    _, _, _, on = _run(st, n, 5, _self_cfg(True), [0.0, 0.0, -9.8])
    _, _, _, off = _run(st, n, 5, None, [0.0, 0.0, -9.8])
    for k in on:
        assert np.abs(on[k] - off[k]).max() < 1e-5, (k, np.abs(on[k] - off[k]).max())


def test_set_self_collision_after_first_step_fails():
    from go1_b200 import capi
    from go1_b200.sim import SimCore
    import ctypes as C
    Cfg, c, info = train_sim_config(32)
    sim = SimCore(c)
    sim.step(torch.zeros(32, 12, device="cuda"))
    rc = sim.L.go1_sim_set_self_collision(sim._handle, C.byref(_self_cfg()))
    assert rc != 0 and b"cannot change after the first go1_sim_step" in sim.L.go1_last_error()
    with pytest.raises(capi.Go1Error):
        capi.check(rc, "go1_sim_set_self_collision")


def _make_env(tmp_path, n, on):
    import sys
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    from ml_logger import logger
    apply_train_config(Cfg)
    Cfg.env.num_envs = n
    if on is not None:
        Cfg.asset.model_self_collisions = on
    logger.configure(prefix="run", root=str(tmp_path))
    return HistoryWrapper(VelocityTrackingEasyEnv(sim_device="cuda:0", headless=True, cfg=Cfg))


def test_graph_replayed_rollout_equals_eager_rollout_with_self_collisions(tmp_path, monkeypatch):
    """As test_runner_gpu.test_graph_replayed_rollout_equals_eager_rollout, with the self-collision kernel captured in the graphs."""
    monkeypatch.chdir(tmp_path)
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    out = []
    for graphed in (False, True):
        torch.manual_seed(0); np.random.seed(0)
        env = _make_env(tmp_path, 256, True)
        assert env.env.core.self_collision.enabled == 1
        RunnerArgs.num_steps_per_env, RunnerArgs.resume = 24, False
        runner = Runner(env, device="cuda:0")
        runner.step_graph = graphed
        if not graphed:
            runner.alg.use_cuda_graph = False
        g = torch.Generator().manual_seed(1)
        env.episode_length_buf = torch.randint(0, 1001, (256,), generator=g)
        od = env.get_observations()
        state = (od["obs"], od["privileged_obs"], od["obs_history"])
        snaps = []
        for it in range(2):
            obs, priv, hist, infos = runner.rollout(*state)
            state = (obs, priv, hist)
            torch.cuda.synchronize()
            st = runner.alg.storage
            snaps.append({k: getattr(st, k).clone() for k in ("observations", "privileged_observations", "observation_histories", "actions",
                                                              "rewards", "dones", "values")})
            snaps[-1]["env_f32"] = env.env.core.env_f32.clone(); snaps[-1]["leg_f32"] = env.env.core.leg_f32.clone()
            runner.alg.storage.clear()
        sg = runner.__dict__.get("_sg")
        assert (sg is not None and len(sg["graphs"]) == 2) if graphed else (not sg or not sg["graphs"])
        out.append(snaps)
    for it in range(2):
        for k in out[0][it]:
            assert torch.equal(out[0][it][k], out[1][it][k]), (it, k)


def test_runner_learn_with_self_collisions(tmp_path, monkeypatch):
    """GO1_SELF_COLLISIONS=1 reaches the step kernel through Cfg -> build_sim_config -> LeggedRobot -> SimCore; two iterations of
    Runner.learn at 1024 envs stay finite, and the logged episode terms include the collision penalty."""
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv("GO1_SELF_COLLISIONS", "1")
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    env = _make_env(tmp_path, 1024, None)
    assert env.env.core.self_collision.enabled == 1
    RunnerArgs.num_steps_per_env, RunnerArgs.save_interval, RunnerArgs.log_freq, RunnerArgs.save_video_interval = 24, 100, 1, 100
    RunnerArgs.resume = False
    runner = Runner(env, device="cuda:0")
    w0 = runner.alg.actor_critic.flat_params.clone()
    runner.learn(num_learning_iterations=2, init_at_random_ep_len=True, eval_freq=100)
    ac = runner.alg.actor_critic
    assert torch.isfinite(ac.flat_params).all() and not torch.equal(ac.flat_params, w0)
    od = env.get_observations()
    obs, priv, hist, infos = runner.rollout(od["obs"], od["privileged_obs"], od["obs_history"])
    runner.alg.compute_returns(hist, priv)
    losses = runner.alg.update()
    assert all(np.isfinite(losses))
    assert any("collision" in k for k in infos["train/episode"]), list(infos["train/episode"])
    assert torch.isfinite(env.env.core.env_f32).all() and torch.isfinite(env.env.core.leg_f32).all()
