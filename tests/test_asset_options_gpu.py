"""Cfg.asset in the fused step kernel (go1_sim_set_asset_options): the Go1 defaults leave every kernel bit-identical, contact-body
sets drive termination and the collision term exactly, a welded base holds the root and moves the joints as the fp64 restatement
(tests/fixed_base_oracle.py) does, with armature and with gravity off, and training runs with the options."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from env_golden_util import train_sim_config

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
LEGS = ("FL", "FR", "RL", "RR")


def _sim(n, asset=None, overrides=None, self_collision=None, **asset_cfg):
    from go1_b200.config import asset_config
    from go1_b200.sim import SimCore
    ov = {k: dict(v) for k, v in (overrides or {}).items()}
    ov.setdefault("asset", {}).update(asset_cfg)
    Cfg, c, info = train_sim_config(n, cfg_overrides=ov)
    c.rand_interval = 0
    opts = asset_config(Cfg) if asset == "cfg" else asset
    return SimCore(c, self_collision=self_collision, asset=opts), c, info


def _standing(sim, c, z=0.32, seed=0):
    n = sim.N
    g = torch.Generator(device="cuda").manual_seed(seed)
    sim.env("root_pos")[2].fill_(z)
    sim.env("root_pos")[:2].copy_(torch.rand(2, n, device="cuda", generator=g) * 4 - 2)
    sim.set_joint_aos("dof_pos", torch.tensor(list(c.default_dof_pos), device="cuda").repeat(n, 1))
    sim.env("commands")[4].fill_(3.0); sim.env("commands")[8].fill_(0.5)


def _rows(sim):
    """[N][17][3] contact rows in BODY_NAMES order; the base row summed as the kernel's 4-lane all-reduce: (p0 + p1) + (p2 + p3)."""
    from go1_b200.config import BODY_NAMES
    p = sim.foot_aos("base_contact_forces_part")
    out = torch.zeros(sim.N, 17, 3, device="cuda")
    out[:, 0] = (p[:, 0] + p[:, 1]) + (p[:, 2] + p[:, 3])
    for part in ("hip", "thigh", "calf", "foot"):
        out[:, [BODY_NAMES.index(f"{l}_{part}") for l in LEGS]] = sim.foot_aos(f"{part}_contact_forces")
    return out


def _snapshot(sim):
    return [t.clone() for t in (sim.env_f32, sim.leg_f32, sim.env_i32, sim.obs, sim.priv_obs, sim.rew, sim.reset_u8, sim.timeout_u8)]


@pytest.mark.parametrize("kernel", ["default", "self", "deferred"])
def test_go1_defaults_through_the_setter_are_bit_identical(kernel):
    """A sim that sets the Go1 options explicitly computes exactly what a sim that never calls the setter computes."""
    from go1_b200 import capi
    n, steps = 384, 50
    snaps = []
    for explicit in (False, True):
        sim, c, info = _sim(n, asset="cfg" if explicit else None)
        if kernel == "self":
            sc = info["self_collision"]
            sc.enabled = 1
            capi.check(sim.L.go1_sim_set_self_collision(sim._handle, ctypes.byref(sc)), "set_self_collision")
        _standing(sim, c)
        sim.episode_length_buf[: n // 8] = c.max_episode_length - 5
        g = torch.Generator(device="cuda").manual_seed(1)
        pre = torch.zeros(capi.PRE_ROLL_ROWS, 4 * n, device="cuda")
        ended = torch.zeros(n, dtype=torch.int32, device="cuda")
        for t in range(steps):
            a = torch.randn(n, 12, device="cuda", generator=g) * 3.0
            if kernel == "deferred":
                sim.step_deferred(a, pre, common_step=t)
            else:
                sim.step(a, common_step=t)
            ended += sim.reset_u8 * (1 - sim.timeout_u8)
        torch.cuda.synchronize()
        snaps.append(_snapshot(sim) + [pre, ended])
        if explicit:
            assert sim.asset is not None
        sim.close()
    for x, y in zip(*snaps):
        assert torch.equal(x, y)
    assert int(snaps[0][-1].sum()) > 0                        # episodes ended by termination, not time-out


def test_contact_sets_drive_termination_and_collision_exactly():
    """terminate_after_contacts_on = [base, thigh], penalize_contacts_on = [thigh, calf, hip, FL] under flailing actions: every
    step, reset == any(|F[idx]| > 1) | time_out | body_height < terminal, recomputed from the reported rows, and the collision
    episode sum grows by sum_idx [|F| > 0.1] * scale * dt: the count exactly, the sum to the rounding of one add."""
    from go1_b200 import capi
    n, steps = 320, 50
    sim, c, info = _sim(n, asset="cfg", terminate_after_contacts_on=["base", "thigh"], penalize_contacts_on=["thigh", "calf", "hip", "FL"])
    bodies = info["contact_bodies"]
    assert bin(sim.asset.termination_mask).count("1") == 5 and len(bodies["penalised"]) == 16
    _standing(sim, c)
    sim.episode_length_buf[: n // 8] = c.max_episode_length - 5           # some envs time out inside the window
    term_idx = torch.tensor(bodies["termination"], device="cuda")
    pen_idx = torch.tensor(bodies["penalised"], device="cuda")
    cid = capi.REWARD_TERMS.index("collision")
    scale = torch.tensor(c.reward_scale[cid], dtype=torch.float32, device="cuda")
    assert float(scale) != 0.0
    g = torch.Generator(device="cuda").manual_seed(2)
    thigh_hits = hip_or_fl = 0
    for t in range(steps):
        ep = sim.episode_length_buf.clone()
        prev = sim.env("episode_sums")[cid].clone()
        sim.step(torch.randn(n, 12, device="cuda", generator=g) * 3.0, common_step=t)
        F = _rows(sim)
        norm = torch.norm(F, dim=-1)
        contact_term = (norm[:, term_idx] > 1.0).any(1)
        time_out = (ep + 1) > c.max_episode_length
        want = contact_term | time_out
        if c.use_terminal_body_height:
            want |= sim.env("root_pos")[2] < c.terminal_body_height
        assert torch.equal(sim.reset_u8.bool(), want), t
        assert torch.equal(sim.timeout_u8.bool(), time_out), t
        raw = (norm[:, pen_idx] > 0.1).float().sum(1)
        new = sim.env("episode_sums")[cid]
        assert torch.equal(torch.round((new - prev) / scale), raw), t
        assert torch.allclose(new, prev + raw * scale, rtol=0, atol=1e-6 + 1e-6 * float(new.abs().max())), t
        thigh_hits += int((norm[:, [2, 6, 10, 14]] > 1.0).any(1).sum())
        hip_or_fl += int((norm[:, [1, 5, 9, 13, 4]] > 0.1).any(1).sum())
    assert thigh_hits > 0 and hip_or_fl > 0                    # the added bodies were exercised


def _hanging(sim, c, rng, z=1.2):
    n = sim.N
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()
    yaw = rng.uniform(-np.pi, np.pi, n)
    quat = np.stack([np.zeros(n), np.zeros(n), np.sin(yaw / 2), np.cos(yaw / 2)], 1)
    D = c.dr[0]                # inside the tile grid's teleport box, so that no teleport moves the root
    cx = 0.5 * (D.teleport_x_lo + D.teleport_x_hi) if D.teleport_robots else 0.0
    cy = 0.5 * (D.teleport_y_lo + D.teleport_y_hi) if D.teleport_robots else 0.0
    sim.env("root_pos").copy_(T(np.stack([cx + rng.uniform(-1, 1, n), cy + rng.uniform(-1, 1, n), np.full(n, z)], 1)).t())
    sim.env("root_quat").copy_(T(quat).t())
    sim.env("root_lin_vel").copy_(T(rng.uniform(-0.5, 0.5, (n, 3))).t())           # a reset's draw: the welded base ignores it
    sim.env("root_ang_vel").copy_(T(rng.uniform(-0.5, 0.5, (n, 3))).t())
    q = np.tile(np.array(list(c.default_dof_pos)), (n, 1)) + rng.uniform(-0.3, 0.3, (n, 12))
    qd = rng.uniform(-1.5, 1.5, (n, 12))
    sim.set_joint_aos("dof_pos", T(q)); sim.set_joint_aos("dof_vel", T(qd))
    return sim.env_aos("root_pos").clone(), sim.env_aos("root_quat").clone(), quat, q, qd


# One policy step (4 substeps) of fp32 articulated-body kernel vs the fp64 joint-space restatement: rounding only (no contacts, no
# limits), far tighter than test_sim_gpu.physics_vs_oracle's floating-base tolerances (q 1e-3, qd 5e-2).
TOL_Q, TOL_QD = 2e-5, 2e-3


@pytest.mark.parametrize("armature", [0.0, 0.01])
def test_fixed_base_holds_the_root_and_matches_the_fp64_restatement(armature):
    import fixed_base_oracle as fb
    n = 256
    sim, c, info = _sim(n, asset="cfg", overrides={"control": {"control_type": "P"}}, fix_base_link=True, armature=armature)
    assert sim.asset.fix_base == 1 and abs(sim.asset.armature - armature) < 1e-9
    rng = np.random.default_rng(3)
    pos0, quat0, quat, q0, qd0 = _hanging(sim, c, rng)
    grav = [0.0, 0.0, -9.8]
    actions = torch.zeros(n, 12, device="cuda")
    sim.step(actions, common_step=0)
    torch.cuda.synchronize()
    q1, qd1 = sim.joint_aos("dof_pos").cpu().numpy(), sim.joint_aos("dof_vel").cpu().numpy()
    kp, kd, lim = c.kp, c.kd, c.torque_limit
    target = np.array(list(c.default_dof_pos))           # zero actions and an empty action FIFO: the default pose
    assert (np.abs(_rows(sim).cpu().numpy()) == 0).all()  # nothing touches: the feet hang free
    worst_q = worst_qd = 0.0
    for e in range(n):
        R0 = fb.quat_to_R(sim.env_aos("root_quat")[e].double().cpu().numpy())
        tq = lambda q, qd: np.clip(kp * (target - q) - kd * qd, -lim, lim)
        qe, qde = fb.policy_step(R0, q0[e].astype(np.float32).astype(np.float64), qd0[e].astype(np.float32).astype(np.float64), tq, grav,
                                 float(np.float32(c.sim_dt)), c.decimation, armature)
        worst_q, worst_qd = max(worst_q, np.abs(q1[e] - qe).max()), max(worst_qd, np.abs(qd1[e] - qde).max())
    assert worst_q < TOL_Q and worst_qd < TOL_QD, (worst_q, worst_qd)
    assert np.abs(qd1 - qd0).max() > 0.1                   # the joints did move
    for t in range(1, 50):
        sim.step(actions, common_step=t)
    torch.cuda.synchronize()
    assert torch.equal(sim.env_aos("root_pos"), pos0) and torch.equal(sim.env_aos("root_quat"), quat0)
    assert (sim.env("root_lin_vel") == 0).all() and (sim.env("root_ang_vel") == 0).all() and (sim.env("base_lin_vel") == 0).all()
    assert torch.isfinite(sim.leg_f32).all()


def test_armature_slows_the_joints():
    """Under the same torques a heavier joint-space inertia gives smaller joint accelerations."""
    speeds = []
    for arm in (0.0, 0.05):
        sim, c, _ = _sim(256, asset="cfg", overrides={"control": {"control_type": "P"}}, fix_base_link=True, armature=arm)
        _hanging(sim, c, np.random.default_rng(4))
        qd0 = sim.joint_aos("dof_vel").clone()
        sim.step(torch.zeros(256, 12, device="cuda"))
        speeds.append(float((sim.joint_aos("dof_vel") - qd0).abs().mean()))
        sim.close()
    assert speeds[1] < 0.8 * speeds[0], speeds


def _unactuated():
    return {"control": {"control_type": "P", "stiffness": {"joint": 0.0}, "damping": {"joint": 0.0}}}


def test_gravity_off_welded_joints_stay_at_rest():
    """disable_gravity + zero joint torque on a welded base: nothing moves, whatever gravity the randomisation sets."""
    n = 256
    sim, c, _ = _sim(n, asset="cfg", overrides=_unactuated(), fix_base_link=True, disable_gravity=True)
    assert c.kp == 0.0 and c.kd == 0.0
    _hanging(sim, c, np.random.default_rng(5))
    sim.set_joint_aos("dof_vel", torch.zeros(n, 12, device="cuda"))
    sim.set_gravity([1.5, -2.0, -12.0], [0.12, -0.16, -0.98])
    q0 = sim.joint_aos("dof_pos").clone()
    for t in range(50):
        sim.step(torch.randn(n, 12, device="cuda"), common_step=t)
    torch.cuda.synchronize()
    assert torch.equal(sim.joint_aos("dof_pos"), q0) and (sim.joint_aos("dof_vel") == 0).all()
    # projected_gravity still follows gravity_vec, as in the reference
    assert (sim.env("projected_gravity").abs().sum(0) > 0.5).all()


def test_gravity_off_free_base_keeps_its_velocity():
    """disable_gravity + zero joint torque, base free and in the air, moving without rotation and joints at rest: no external
    force, so the whole robot translates rigidly and the base's (= the robot's) centre-of-mass velocity stays constant."""
    n = 256
    sim, c, _ = _sim(n, asset="cfg", overrides=_unactuated(), disable_gravity=True)
    rng = np.random.default_rng(6)
    _hanging(sim, c, rng, z=3.0)
    v0 = torch.from_numpy(rng.uniform(-1, 1, (n, 3)).astype(np.float32)).cuda()
    sim.env("root_lin_vel").copy_(v0.t()); sim.env("root_ang_vel").zero_()
    sim.set_joint_aos("dof_vel", torch.zeros(n, 12, device="cuda"))
    z0 = sim.env("root_pos")[2].clone()
    for t in range(50):
        sim.step(torch.zeros(n, 12, device="cuda"), common_step=t)
    torch.cuda.synchronize()
    # fp32 rounding of the coupled base / leg recursion over 200 substeps moves the base by ~1e-4 m/s; gravity would add 9.8 m/s
    assert torch.allclose(sim.env("root_lin_vel").t(), v0, rtol=0, atol=1e-3)
    assert sim.env("root_ang_vel").abs().max() < 1e-3 and sim.joint_aos("dof_vel").abs().max() < 1e-3
    dt = 50 * c.decimation * float(np.float32(c.sim_dt))
    assert torch.allclose(sim.env("root_pos")[2], z0 + v0[:, 2] * dt, atol=1e-3)      # no fall


def test_setter_rejects_bad_input_and_late_calls():
    from go1_b200 import capi
    from go1_b200.config import asset_config
    sim, c, info = _sim(32)
    L, h = sim.L, sim._handle
    good = info["asset"]
    assert L.go1_sizeof_asset_options() == ctypes.sizeof(capi.Go1AssetOptions)
    assert L.go1_sim_set_asset_options(h, None) != 0
    for mutate in (lambda o: o.penalty_weight.__setitem__(3, -1.0), lambda o: o.penalty_weight.__setitem__(0, float("nan")),
                   lambda o: o.penalty_weight.__setitem__(16, float("inf")), lambda o: setattr(o, "termination_mask", 1 << 17),
                   lambda o: setattr(o, "armature", -0.5), lambda o: setattr(o, "armature", float("nan"))):
        o = capi.Go1AssetOptions.from_buffer_copy(good)
        mutate(o)
        assert L.go1_sim_set_asset_options(h, ctypes.byref(o)) != 0
        assert b"go1_sim_set_asset_options" in L.go1_last_error()
    assert L.go1_sim_set_asset_options(h, ctypes.byref(good)) == 0
    sim.step(torch.zeros(32, 12, device="cuda"))
    assert L.go1_sim_set_asset_options(h, ctypes.byref(good)) != 0
    assert b"after the first go1_sim_step" in L.go1_last_error()


def _runner(tmp_path, n, graphed):
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    from ml_logger import logger
    apply_train_config(Cfg)
    Cfg.env.num_envs = n
    Cfg.asset.fix_base_link = True
    Cfg.asset.armature = 0.005
    Cfg.asset.terminate_after_contacts_on = ["base", "calf"]
    Cfg.asset.penalize_contacts_on = ["thigh", "hip", "FR"]
    logger.configure(prefix="run_asset", root=str(tmp_path))
    env = HistoryWrapper(VelocityTrackingEasyEnv(sim_device="cuda:0", headless=True, cfg=Cfg))
    RunnerArgs.num_steps_per_env, RunnerArgs.resume = 24, False
    runner = Runner(env, device="cuda:0")
    runner.step_graph = graphed
    if not graphed:
        runner.alg.use_cuda_graph = False
    return env, runner


def test_runner_trains_a_welded_robot_graph_equals_eager(tmp_path, monkeypatch):
    """fix_base_link with non-default contact sets: graph-replayed and eager rollouts store bit-identical rewards and dones
    (the second rollout replays the graphs captured in the first), then two training iterations stay finite."""
    monkeypatch.chdir(tmp_path)
    n = 256
    out = []
    for graphed in (False, True):
        torch.manual_seed(0); np.random.seed(0)
        env, runner = _runner(tmp_path, n, graphed)
        core = env.env.core
        assert core.asset.fix_base == 1 and env.env.penalised_contact_indices.tolist() == [2, 6, 10, 14, 1, 5, 9, 13, 5, 6, 7, 8]
        assert env.env.termination_contact_indices.tolist() == [0, 3, 7, 11, 15]
        env.episode_length_buf = torch.randint(0, 1001, (n,), generator=torch.Generator().manual_seed(1))
        od = env.get_observations()
        state = (od["obs"], od["privileged_obs"], od["obs_history"])
        snaps = []
        for it in range(2):
            obs, priv, hist, infos = runner.rollout(*state)
            state = (obs, priv, hist)
            torch.cuda.synchronize()
            st = runner.alg.storage
            snaps.append(dict(rewards=st.rewards.clone(), dones=st.dones.clone()))
            runner.alg.storage.clear()
        out.append(snaps)
        if graphed:
            for it in range(2):                   # two training iterations
                obs, priv, hist, infos = runner.rollout(*state)
                state = (obs, priv, hist)
                with torch.inference_mode():
                    runner.alg.compute_returns(hist[:env.num_train_envs], priv[:env.num_train_envs])
                losses = runner.alg.update()
                torch.cuda.synchronize()
                assert all(np.isfinite(losses)), losses
                assert torch.isfinite(core.env_f32).all() and torch.isfinite(core.leg_f32).all()
                assert torch.isfinite(runner.alg.actor_critic.flat_params).all()
            # welded: every root sits where its last reset put it, at rest
            assert (core.env("root_lin_vel") == 0).all() and (core.env("root_ang_vel") == 0).all()
        del runner, env
        torch.cuda.empty_cache()
    assert int(out[0][0]["dones"].sum() + out[0][1]["dones"].sum()) > 0
    for it in range(2):
        for k in ("rewards", "dones"):
            assert torch.equal(out[0][it][k], out[1][it][k]), (it, k)
