"""Cfg tree -> Go1SimConfig (the resolved, flat configuration the CUDA step kernel consumes).

Mirrors the host-side derivations the reference performs once at start-up:
  _parse_cfg (legged_robot.py:1716-1732), _get_noise_scale_vec (:1053-1120), _init_buffers' commands_scale
  and default_dof_pos (:1193-1236), _process_dof_props' soft limits (:593-607), _prepare_reward_function
  (:1385-1429), get_scale_shift (go1_gym/utils/math_utils.py:35-38).
"""
import json
import os

import numpy as np

from . import capi

_PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DOF_NAMES = [f"{leg}_{part}_joint" for leg in ("FL", "FR", "RL", "RR") for part in ("hip", "thigh", "calf")]
# The 17 rigid bodies in Isaac Gym order (go1.urdf with collapse_fixed_joints: trunk and imu_link merge into base, each
# *_thigh_shoulder into its hip): the body axis of LeggedRobot.contact_forces, of the contact-index sets and of Go1AssetOptions.
BODY_NAMES = ["base"] + [f"{leg}_{part}" for leg in ("FL", "FR", "RL", "RR") for part in ("hip", "thigh", "calf", "foot")]


def load_model():
    with open(os.path.join(_PKG, "resources", "go1_model.json")) as f:
        return json.load(f)


def load_actuator_weights():
    w = np.fromfile(os.path.join(_PKG, "resources", "actuator_net_go1.bin"), dtype=np.float32)
    assert w.size == 1313
    return w


def cfg_dict(node):
    """vars() of a config class as a clean dict (works for params_proto and plain classes)."""
    return {k: v for k, v in vars(node).items() if not k.startswith("_")}


def get_scale_shift(rng):
    scale = 2. / (rng[1] - rng[0])
    shift = (rng[1] + rng[0]) / 2.
    return scale, shift


def derive(cfg):
    """Derived quantities of _parse_cfg; returns a dict and (like the reference) writes them back into cfg."""
    # gymapi.SimParams.dt is a C float: the reference's self.dt = decimation * float32(0.005) = 0.0199999995..., which is
    # what makes max_episode_length 1001 and the DR intervals 201/401/397 in the shipped parameters.pkl
    sim_dt = float(np.float32(cfg.sim.dt))
    dt = cfg.control.decimation * sim_dt
    if cfg.terrain.mesh_type not in ['heightfield', 'trimesh']:
        cfg.terrain.curriculum = False
    cfg.env.max_episode_length = np.ceil(cfg.env.episode_length_s / dt)
    cfg.domain_rand.push_interval = np.ceil(cfg.domain_rand.push_interval_s / dt)
    cfg.domain_rand.rand_interval = np.ceil(cfg.domain_rand.rand_interval_s / dt)
    cfg.domain_rand.gravity_rand_interval = np.ceil(cfg.domain_rand.gravity_rand_interval_s / dt)
    cfg.domain_rand.gravity_rand_duration = np.ceil(
        cfg.domain_rand.gravity_rand_interval * cfg.domain_rand.gravity_impulse_duration)
    return dict(dt=dt, sim_dt=sim_dt)


def default_dof_pos(cfg):
    return np.array([cfg.init_state.default_joint_angles[n] for n in DOF_NAMES], dtype=np.float32)


def pd_gains(cfg):
    kp = kd = 0.0
    for name in DOF_NAMES:
        for key in cfg.control.stiffness.keys():
            if key in name:
                kp, kd = cfg.control.stiffness[key], cfg.control.damping[key]
    return float(kp), float(kd)


def soft_limits(cfg, model):
    lo, hi = [], []
    for leg in range(4):
        for part in ("hip", "thigh", "calf"):
            d = model[part][leg]
            # computed in float32 like the reference's torch buffers (legged_robot.py:598-607)
            l, u = np.float32(d["lower"]), np.float32(d["upper"])
            m = (l + u) / np.float32(2)
            r = u - l
            lo.append(m - np.float32(0.5) * r * np.float32(cfg.rewards.soft_dof_pos_limit))
            hi.append(m + np.float32(0.5) * r * np.float32(cfg.rewards.soft_dof_pos_limit))
    return np.array(lo, dtype=np.float32), np.array(hi, dtype=np.float32)


def commands_scale(cfg):
    s = cfg.obs_scales
    return np.array([s.lin_vel, s.lin_vel, s.ang_vel, s.body_height_cmd, s.gait_freq_cmd, s.gait_phase_cmd,
                     s.gait_phase_cmd, s.gait_phase_cmd, s.gait_phase_cmd, s.footswing_height_cmd, s.body_pitch_cmd,
                     s.body_roll_cmd, s.stance_width_cmd, s.stance_length_cmd, s.aux_reward_cmd],
                    dtype=np.float32)[:cfg.commands.num_commands]


def noise_scale_vec(cfg):
    """legged_robot.py:1053-1120, same concatenation order."""
    ns, lvl, os_ = cfg.noise_scales, cfg.noise.noise_level, cfg.obs_scales
    e = cfg.env
    ndof = e.num_actions
    v = [np.ones(3) * ns.gravity * lvl]
    if e.observe_command:
        v.append(np.zeros(cfg.commands.num_commands))
    v += [np.ones(ndof) * ns.dof_pos * lvl * os_.dof_pos, np.ones(ndof) * ns.dof_vel * lvl * os_.dof_vel, np.zeros(ndof)]
    if e.observe_two_prev_actions:
        v.append(np.zeros(ndof))
    if e.observe_timing_parameter:
        v.append(np.zeros(1))
    if e.observe_clock_inputs:
        v.append(np.zeros(4))
    if e.observe_vel:
        v = [np.ones(3) * ns.lin_vel * lvl * os_.lin_vel, np.ones(3) * ns.ang_vel * lvl * os_.ang_vel] + v
    if e.observe_only_lin_vel:
        v = [np.ones(3) * ns.lin_vel * lvl * os_.lin_vel] + v
    if e.observe_yaw:
        v.append(np.zeros(1))
    if e.observe_contact_states:
        v.append(np.ones(4) * ns.contact_states * lvl)
    return np.concatenate(v).astype(np.float32)


TASK_TERMS = ("tracking_lin_vel", "tracking_ang_vel", "tracking_contacts_shaped_force", "tracking_contacts_shaped_vel")


def reward_tables(cfg, dt, container=None):
    """_prepare_reward_function: drop zero scales, multiply by dt, keep dict order (legged_robot.py:1394-1412).

    With a reward container class, each nonzero term is built-in when its `_reward_<name>` is the BuiltinReward marker of that
    name (the kernel table), a user term when it is a plain method (`user`: name -> scale, in order; a built-in of that name is
    left out of the table), and unknown when there is no such attribute.  Without one, the names of capi.REWARD_TERMS are the
    built-ins.  Returns (active, order, table, unknown, user)."""
    scales = cfg_dict(cfg.reward_scales)
    order, table = [], np.zeros(capi.NUM_REWARD_TERMS, dtype=np.float32)
    active = {}
    for name, sc in scales.items():
        if sc == 0:
            continue
        active[name] = sc * dt
    unknown, user = [], {}
    for name, sc in active.items():
        fn = getattr(container, "_reward_" + name, None) if container is not None else None
        marker = getattr(fn, "builtin_term", None)
        if name not in capi.REWARD_TERMS or (container is not None and marker != name):
            if container is not None and marker is None and callable(fn):
                if name in TASK_TERMS or name == "termination":
                    raise ValueError(f"_reward_{name} cannot be overridden: "
                                     + ("it feeds the command curriculum's command_sums" if name in TASK_TERMS
                                        else "the termination term is added after the combination of the others"))
                user[name] = sc
            else:
                unknown.append(name)
            continue
        tid = capi.REWARD_TERMS.index(name)
        table[tid] = np.float32(sc)
        if name != "termination":
            order.append(tid)
    if len(user) > capi.MAX_USER_REWARDS:
        raise ValueError(f"{len(user)} user reward terms: at most {capi.MAX_USER_REWARDS}")
    return active, order, table, unknown, user


def _lo_span(rng):
    """{low, float32(high - low)}: the reference evaluates torch.rand(...) * (high - low) + low with the difference taken in
    Python double precision (legged_robot.py:611-665)."""
    lo, hi = float(rng[0]), float(rng[1])
    return [lo, float(np.float32(hi - lo))]


def fill_domain_rand(D, cfg, dt):
    """One Go1DomainRand from a Cfg tree (the train cfg or the eval cfg): everything _call_train_eval switches."""
    dr, t = cfg.domain_rand, cfg.terrain
    g = lambda name, default: getattr(dr, name, default)
    D.randomize_motor_strength = int(bool(dr.randomize_motor_strength))
    D.randomize_motor_offset = int(bool(g("randomize_motor_offset", False)))
    D.randomize_Kp_factor = int(bool(dr.randomize_Kp_factor))
    D.randomize_Kd_factor = int(bool(dr.randomize_Kd_factor))
    D.motor_strength_range[:] = _lo_span(dr.motor_strength_range)
    D.motor_offset_range[:] = _lo_span(g("motor_offset_range", [0., 0.]))
    D.Kp_factor_range[:] = _lo_span(dr.Kp_factor_range)
    D.Kd_factor_range[:] = _lo_span(dr.Kd_factor_range)
    D.randomize_rigids_after_start = int(bool(g("randomize_rigids_after_start", False)))
    D.randomize_base_mass = int(bool(dr.randomize_base_mass))
    D.randomize_com_displacement = int(bool(g("randomize_com_displacement", False)))
    D.randomize_friction = int(bool(dr.randomize_friction))
    D.randomize_restitution = int(bool(g("randomize_restitution", False)))
    D.added_mass_range[:] = _lo_span(dr.added_mass_range)
    D.com_displacement_range[:] = _lo_span(g("com_displacement_range", [0., 0.]))
    D.friction_range[:] = _lo_span(dr.friction_range)
    D.restitution_range[:] = _lo_span(g("restitution_range", [0., 0.]))
    D.push_robots = int(bool(dr.push_robots))
    D.push_interval = int(np.ceil(dr.push_interval_s / dt))            # _parse_cfg (legged_robot.py:1727)
    D.max_push_vel_xy = float(dr.max_push_vel_xy)
    # _teleport_robots (legged_robot.py:1028-1051); thresholds rounded to float32 like the scalar side of the tensor compare
    tiles = t.mesh_type in ["heightfield", "trimesh"]
    D.teleport_robots = int(bool(t.teleport_robots) and tiles)
    if D.teleport_robots:
        thresh = t.teleport_thresh
        x_offset = int(getattr(t, "x_offset", 0) * t.horizontal_scale)
        D.teleport_x_lo = float(np.float32(thresh + x_offset))
        D.teleport_x_hi = float(np.float32(t.terrain_length * t.num_rows - thresh + x_offset))
        D.teleport_dx = float(np.float32(t.terrain_length * (t.num_rows - 1)))
        D.teleport_y_lo = float(np.float32(thresh))
        D.teleport_y_hi = float(np.float32(t.terrain_width * t.num_cols - thresh))
        D.teleport_dy = float(np.float32(t.terrain_width * (t.num_cols - 1)))
    D.x_init_range, D.y_init_range, D.yaw_init_range = t.x_init_range, t.y_init_range, t.yaw_init_range
    D.x_init_offset, D.y_init_offset = t.x_init_offset, t.y_init_offset


SELF_K, SELF_C = 5000.0, 20.0      # self-contact penalty stiffness (N/m) and damping (N s/m), DESIGN.md §3


def self_collision_config(cfg, k=SELF_K, c=SELF_C):
    """Go1SelfCollision of `cfg`: on iff Cfg.asset.model_self_collisions (unset = the GO1_SELF_COLLISIONS=1 environment switch)
    and bit 0 of Cfg.asset.self_collisions is clear (the reference's "1 to disable, 0 to enable")."""
    on = getattr(cfg.asset, "model_self_collisions", os.environ.get("GO1_SELF_COLLISIONS") == "1")
    sc = capi.Go1SelfCollision()
    sc.enabled = int(bool(on) and (int(getattr(cfg.asset, "self_collisions", 0)) & 1) == 0)
    sc.k, sc.c = float(k), float(c)
    sc.thigh_radius, sc.calf_radius, sc.foot_radius = 0.017, 0.008, 0.02
    return sc


# Cfg.asset options that the compiled Go1 model does not simulate, with the base Cfg's values (legged_robot_config.py): a
# different value is reported once per build_sim_config.  density, thickness, flip_visual_attachments and
# replace_cylinder_with_capsule change nothing for this model (its masses and inertias are compiled in, its collision shapes are
# spheres, capsules and a box, meshes are never loaded), so they are accepted silently.
_WARN_ONLY = dict(linear_damping=0., angular_damping=0., max_linear_velocity=1000., max_angular_velocity=1000.,
                  default_dof_drive_mode=3, collapse_fixed_joints=True)


def _asset_get(asset, key, default):
    """An attribute of Cfg.asset, which is a config class or, restored from parameters.pkl, possibly a plain dict."""
    return asset.get(key, default) if isinstance(asset, dict) else getattr(asset, key, default)


def contact_bodies(cfg):
    """Body indices (BODY_NAMES) that Cfg.asset selects, as the reference builds them (legged_robot.py:1521-1527, 1580-1590):
    every body whose name contains an entry, entry by entry, so a body that several entries select is listed once per entry.
    Returns dict(penalised=[...], termination=[...], feet=[...]); feet must be exactly the four *_foot bodies."""
    a = cfg.asset
    pick = lambda names: [i for n in names for i, b in enumerate(BODY_NAMES) if str(n) in b]
    foot = str(_asset_get(a, "foot_name", "None"))
    feet = pick([foot])
    want = [i for i, b in enumerate(BODY_NAMES) if b.endswith("_foot")]
    if feet != want:
        raise ValueError(f"Cfg.asset.foot_name = {foot!r} selects {[BODY_NAMES[i] for i in feet]}: the simulated Go1's feet terms and "
                         f"contact states are defined over exactly {[BODY_NAMES[i] for i in want]}")
    return dict(penalised=pick(_asset_get(a, "penalize_contacts_on", [])),
                termination=pick(_asset_get(a, "terminate_after_contacts_on", [])), feet=feet)


def asset_config(cfg, warn=True, bodies=None):
    """Go1AssetOptions of Cfg.asset: collision-penalty weight per body (the number of penalize_contacts_on entries its name
    contains), termination bits (terminate_after_contacts_on), fix_base_link, disable_gravity and armature.  With `warn`, prints
    one warning per option the compiled Go1 model does not simulate (_WARN_ONLY, or a `file` other than go1.urdf).  `bodies`:
    contact_bodies(cfg) when the caller has resolved it already."""
    a = cfg.asset
    bodies = contact_bodies(cfg) if bodies is None else bodies
    o = capi.Go1AssetOptions()
    for i in bodies["penalised"]:
        o.penalty_weight[i] += 1.0
    mask = 0
    for i in bodies["termination"]:
        mask |= 1 << i
    o.termination_mask = mask
    o.fix_base = int(bool(_asset_get(a, "fix_base_link", False)))
    o.disable_gravity = int(bool(_asset_get(a, "disable_gravity", False)))
    arm = _asset_get(a, "armature", 0.)
    try:
        armf = float(arm)
    except (TypeError, ValueError):
        armf = float("nan")
    if not (np.isfinite(armf) and armf >= 0.):
        raise ValueError(f"Cfg.asset.armature = {arm!r}: must be a finite float >= 0 (kg m^2 added to every joint's inertia)")
    o.armature = armf
    if warn:
        f = str(_asset_get(a, "file", ""))
        if not f.endswith("go1.urdf"):
            print(f"Warning: Cfg.asset.file = {f!r} is not go1.urdf: the compiled Go1 model is simulated")
        for k, default in _WARN_ONLY.items():
            v = _asset_get(a, k, default)
            if v != default:
                print(f"Warning: Cfg.asset.{k} = {v!r} differs from {default!r} and is not simulated: the compiled Go1 model ignores it")
    return o


def build_sim_config(cfg, num_envs=None, num_train_envs=None, seed=0, physics=None, eval_cfg=None, reward_container=None):
    """Resolve `cfg` (a Cfg-like class tree) into a Go1SimConfig.  `physics` overrides solver parameters; `eval_cfg` is the
    second Cfg tree of the train/eval split (its randomisation / reset ranges apply to envs >= num_train_envs);
    `reward_container` is the reward container class whose user terms run beside the kernel (reward_tables)."""
    d = derive(cfg)
    if eval_cfg is not None:
        derive(eval_cfg)
    model = load_model()
    c = capi.Go1SimConfig()
    n = int(num_envs if num_envs is not None else cfg.env.num_envs)
    c.num_envs = n
    c.num_train_envs = int(num_train_envs if num_train_envs is not None else n)
    c.sim_dt = cfg.sim.dt
    c.decimation = int(cfg.control.decimation)
    c.clip_actions = cfg.normalization.clip_actions
    c.clip_obs = cfg.normalization.clip_observations
    ct = cfg.control.control_type
    if ct not in ("actuator_net", "P"):
        raise NameError(f"Unknown controller type: {ct}")          # legged_robot.py:943
    c.control_type = 0 if ct == "actuator_net" else 1
    c.action_scale = cfg.control.action_scale
    c.hip_scale_reduction = cfg.control.hip_scale_reduction
    c.kp, c.kd = pd_gains(cfg)
    c.use_lag = int(bool(cfg.domain_rand.randomize_lag_timesteps))
    # without randomize_lag_timesteps the reference never reads its FIFO (legged_robot.py:921-926), so it needs no rows here
    if c.use_lag:
        lag = cfg.domain_rand.lag_timesteps
        if int(lag) != lag or not 0 <= lag <= capi.MAX_LAG_TIMESTEPS:
            raise ValueError(f"Cfg.domain_rand.lag_timesteps ({lag!r}) must be an integer in 0..{capi.MAX_LAG_TIMESTEPS}: "
                             "the fused step kernel reserves that many action FIFO slots")
        c.lag_timesteps = int(lag)
    c.default_dof_pos[:] = default_dof_pos(cfg).tolist()
    lo, hi = soft_limits(cfg, model)
    c.soft_limit_lo[:] = lo.tolist()
    c.soft_limit_hi[:] = hi.tolist()
    c.torque_limit = model["hip"][0]["effort"]
    c.num_commands = int(cfg.commands.num_commands)
    e = cfg.env
    c.observe_gait_commands = int(bool(e.observe_gait_commands))
    c.pacing_offset = int(bool(cfg.commands.pacing_offset))
    c.kappa_gait_probs = cfg.rewards.kappa_gait_probs
    for f in ("observe_vel", "observe_only_ang_vel", "observe_only_lin_vel", "observe_command", "observe_two_prev_actions",
              "observe_timing_parameter", "observe_clock_inputs", "observe_yaw", "observe_contact_states"):
        setattr(c, f, int(bool(getattr(e, f))))
    c.num_obs = int(e.num_observations)
    c.num_priv_obs = int(e.num_privileged_obs)
    c.add_noise = int(bool(cfg.noise.add_noise))
    cs = commands_scale(cfg)
    c.commands_scale[:len(cs)] = cs.tolist()
    c.obs_scale_lin_vel, c.obs_scale_ang_vel = cfg.obs_scales.lin_vel, cfg.obs_scales.ang_vel
    c.obs_scale_dof_pos, c.obs_scale_dof_vel = cfg.obs_scales.dof_pos, cfg.obs_scales.dof_vel
    nv = noise_scale_vec(cfg)
    if len(nv) != c.num_obs:
        raise ValueError(f"num_observations ({c.num_obs}) does not match the observe_* flags ({len(nv)})")
    c.noise_scale_vec[:len(nv)] = nv.tolist()
    for unsupported in ("priv_observe_ground_friction", "priv_observe_ground_friction_per_foot"):
        if getattr(e, unsupported, False):
            raise NotImplementedError(f"{unsupported}: _get_ground_frictions is undefined in the reference as well (legged_robot.py:394)")
    pmap = dict(priv_friction="priv_observe_friction", priv_restitution="priv_observe_restitution",
                priv_base_mass="priv_observe_base_mass", priv_com_displacement="priv_observe_com_displacement",
                priv_motor_strength="priv_observe_motor_strength", priv_motor_offset="priv_observe_motor_offset",
                priv_body_height="priv_observe_body_height", priv_body_velocity="priv_observe_body_velocity",
                priv_gravity="priv_observe_gravity", priv_clock_inputs="priv_observe_clock_inputs",
                priv_desired_contact_states="priv_observe_desired_contact_states")
    for k, src in pmap.items():
        setattr(c, k, int(bool(getattr(e, src, False))))
    nm = cfg.normalization
    for k, rng in (("friction_ss", nm.friction_range), ("restitution_ss", nm.restitution_range), ("mass_ss", nm.added_mass_range),
                   ("com_ss", nm.com_displacement_range), ("motor_strength_ss", nm.motor_strength_range),
                   ("motor_offset_ss", nm.motor_offset_range), ("body_height_ss", nm.body_height_range),
                   ("body_velocity_ss", nm.body_velocity_range), ("gravity_ss", nm.gravity_range)):
        sc, sh = get_scale_shift(rng)
        getattr(c, k)[:] = [sc, sh]
    active, order, table, unknown, user = reward_tables(cfg, d["dt"], reward_container)
    for name in unknown:
        print(f"Warning: reward {'_reward_' + name} has nonzero coefficient but was not found!")   # legged_robot.py:1409
    c.reward_scale[:] = table.tolist()
    c.reward_order[:len(order)] = order
    c.num_active_rewards = len(order)
    r = cfg.rewards
    c.only_positive_rewards = int(bool(r.only_positive_rewards))
    c.only_positive_rewards_ji22_style = int(bool(r.only_positive_rewards_ji22_style))
    c.sigma_rew_neg, c.tracking_sigma, c.tracking_sigma_yaw = r.sigma_rew_neg, r.tracking_sigma, r.tracking_sigma_yaw
    c.gait_force_sigma, c.gait_vel_sigma = r.gait_force_sigma, r.gait_vel_sigma
    c.base_height_target, c.max_contact_force = r.base_height_target, r.max_contact_force
    c.use_terminal_body_height = int(bool(r.use_terminal_body_height))
    c.max_episode_length = int(cfg.env.max_episode_length)
    c.terminal_body_height = r.terminal_body_height
    fill_domain_rand(c.dr[0], cfg, d["dt"])
    fill_domain_rand(c.dr[1], eval_cfg if eval_cfg is not None else cfg, d["dt"])
    c.rand_interval = int(cfg.domain_rand.rand_interval)
    c.resampling_interval = int(cfg.commands.resampling_time / d["dt"])
    ist = cfg.init_state
    c.base_init_state[:] = list(ist.pos) + list(ist.rot) + list(ist.lin_vel) + list(ist.ang_vel)
    t = cfg.terrain
    c.custom_origins = int(t.mesh_type in ["heightfield", "trimesh"])
    px = cfg.sim.physx            # a config class, or the plain dict scripts/play.py restores from parameters.pkl
    pxg = (lambda k: px[k]) if isinstance(px, dict) else (lambda k: getattr(px, k))
    c.erp, c.cfm, c.pgs_iters = 0.2, 1e-4, 8
    c.max_depen_vel = pxg("max_depenetration_velocity")
    c.contact_margin = pxg("contact_offset")
    c.bounce_threshold = pxg("bounce_threshold_velocity")
    c.terrain_friction, c.terrain_restitution = t.static_friction, t.restitution
    c.pen_k[:] = [20000., 20000., 5000., 5000.]
    c.pen_c[:] = [150., 150., 30., 30.]
    c.pen_mt, c.limit_k, c.limit_c = 0.2, 300., 3.
    physics = dict(physics or {})
    sc = self_collision_config(cfg, physics.pop("self_k", SELF_K), physics.pop("self_c", SELF_C))
    bodies = contact_bodies(cfg)
    asset = asset_config(cfg, bodies=bodies)
    if physics:
        for k, v in physics.items():
            if hasattr(v, "__len__"):
                getattr(c, k)[:] = list(v)
            else:
                setattr(c, k, v)
    c.hf = None                                  # set by LeggedRobot.create_sim once the Terrain exists
    mh = bool(getattr(t, "measure_heights", False)) and t.mesh_type in ("heightfield", "trimesh")
    px, py = list(getattr(t, "measured_points_x", [])), list(getattr(t, "measured_points_y", []))
    if mh and (len(px) > 32 or len(py) > 32):
        raise ValueError("at most 32 x 32 measured height points")
    c.measure_heights = int(mh)
    c.num_height_points_x, c.num_height_points_y = (len(px), len(py)) if mh else (0, 0)
    if mh:
        c.height_points_x[:len(px)] = px
        c.height_points_y[:len(py)] = py
    c.seed = int(seed)
    return c, dict(active_reward_scales=active, user_reward_scales=user, dt=d["dt"], noise_scale_vec=nv, self_collision=sc,
                   asset=asset, contact_bodies=bodies)
