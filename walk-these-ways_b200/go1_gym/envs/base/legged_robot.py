"""LeggedRobot — the reference's vectorised Go1 env (go1_gym/envs/base/legged_robot.py:19-1806) with the
simulator, torque model, rewards, observations, termination and resets running in the fused CUDA kernels of
libgo1b200.so.  What stays on the host is exactly what the reference keeps on the host: the numpy command
curriculum (legged_robot.py:710-824) and the global gravity randomisation (:546-561, 701-705).

Per step:   [commands of envs due for the periodic resample -> go1_sim_set_commands]
            go1_sim_step (one fused launch: control x4, physics x4, post-physics, rewards, obs)
            one D2H read of the event list (reset envs + next step's resample envs, with their command sums)
            host curriculum update/sample for the reset envs
            go1_sim_reset_idx (sparse: re-initialise those envs and write their observations)

With user reward terms (go1_gym/envs/rewards) the step launch is go1_sim_step_deferred, the terms (torch) and
go1_sim_reward_finish, and go1_sim_user_reward_fold follows the reset launch.

Public attributes keep the reference's names and AoS shapes; they are views/copies of the SoA device state."""
import ctypes

import numpy as np
import torch

from go1_b200 import capi
from go1_b200.config import BODY_NAMES, build_sim_config, cfg_dict
from go1_b200.sim import SimCore
from go1_gym.envs.base.base_task import BaseTask
from go1_gym.utils.terrain import Terrain
from .legged_robot_config import Cfg

_TASK_KEYS = ["tracking_lin_vel", "tracking_ang_vel", "tracking_contacts_shaped_force", "tracking_contacts_shaped_vel"]
_LOCAL_RANGE = np.array([0.55, 0.55, 0.55, 0.55, 0.35, 0.25, 0.25, 0.25, 0.25, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0])


class LazyExtras(dict):
    """dict whose expensive entries (device->host copies) are produced on first access."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self._lazy = {}

    def lazy(self, key, thunk):
        self._lazy[key] = thunk
        dict.pop(self, key, None)

    def __missing__(self, key):
        if key in self._lazy:
            v = self._lazy[key]()
            return v
        raise KeyError(key)

    def __contains__(self, key):
        return dict.__contains__(self, key) or key in self._lazy

    def get(self, key, default=None):
        try:
            return self[key]
        except KeyError:
            return default


class _LazyDict(dict):
    """A dict that fills itself from `build()` the first time it is read (keys(), items(), [], **, len, in)."""

    def __init__(self, build):
        super().__init__()
        self._build = build

    def _fill(self):
        if self._build is not None:
            b, self._build = self._build, None
            dict.update(self, b())

    def keys(self):
        self._fill(); return dict.keys(self)

    def items(self):
        self._fill(); return dict.items(self)

    def values(self):
        self._fill(); return dict.values(self)

    def __getitem__(self, k):
        self._fill(); return dict.__getitem__(self, k)

    def __iter__(self):
        self._fill(); return dict.__iter__(self)

    def __len__(self):
        self._fill(); return dict.__len__(self)

    def __contains__(self, k):
        self._fill(); return dict.__contains__(self, k)

    def setdefault(self, k, d=None):
        self._fill(); return dict.setdefault(self, k, d)

    def __setitem__(self, k, v):
        self._fill(); dict.__setitem__(self, k, v)

    def __reduce__(self):          # pickles (logger.save_pkl of the curriculum distribution) as the plain dict it stands for
        self._fill()
        return (dict, (dict(self),))


def measured_heights_at(base_quat, base_pos, height_samples, terrain_cfg):
    """_get_heights of the reference (legged_robot.py:1790-1806) as a pure function: the measured_points grid rotated by the
    base YAW (quat_apply_yaw, go1_gym/utils/math_utils.py:12-16) and shifted to the base position; per point the minimum of
    the three height samples at the truncated cell index (x, y), (x+1, y), (x, y+1).  Returns [n, len(px)*len(py)] metres."""
    t = terrain_cfg
    dev = base_quat.device
    gx, gy = torch.meshgrid(torch.tensor(t.measured_points_x, device=dev), torch.tensor(t.measured_points_y, device=dev), indexing="ij")
    lx, ly = gx.reshape(1, -1), gy.reshape(1, -1)
    yn = torch.rsqrt(base_quat[:, 2] ** 2 + base_quat[:, 3] ** 2)
    yz, yw = base_quat[:, 2] * yn, base_quat[:, 3] * yn
    cy, sy = (yw * yw - yz * yz)[:, None], (2 * yw * yz)[:, None]
    wx = cy * lx - sy * ly + base_pos[:, 0:1] + t.border_size
    wy = sy * lx + cy * ly + base_pos[:, 1:2] + t.border_size
    ix = torch.clip((wx / t.horizontal_scale).long(), 0, height_samples.shape[0] - 2)
    iy = torch.clip((wy / t.horizontal_scale).long(), 0, height_samples.shape[1] - 2)
    hs = height_samples
    h = torch.min(torch.min(hs[ix, iy], hs[ix + 1, iy]), hs[ix, iy + 1])
    return h.float() * t.vertical_scale


class PreRollEnv:
    """A reward container's `self.env`: the env, except that the fields the step rolls after compute_reward (legged_robot.py:126-131)
    read as they were before this step's roll, from the slab go1_sim_step_deferred writes ([N, 12] copies, Isaac DOF order).
    Those values are the ones of the last step; outside a step's user terms they are stale."""

    _ROWS = {name: 3 * i for i, name in enumerate(capi.PRE_ROLL_FIELDS)}

    def __init__(self, env, slab):
        object.__setattr__(self, "_env", env)
        object.__setattr__(self, "_slab", slab)

    def __getattr__(self, name):
        r = PreRollEnv._ROWS.get(name)
        if r is None:
            return getattr(self._env, name)
        n = self._env.num_envs
        return self._slab[r:r + 3].view(3, n, 4).permute(1, 2, 0).reshape(n, 12)

    def __setattr__(self, name, value):
        setattr(self._env, name, value)


class LeggedRobot(BaseTask):
    def __init__(self, cfg: Cfg, sim_params, physics_engine, sim_device, headless, eval_cfg=None, initial_dynamics_dict=None):
        self.cfg = cfg
        self.eval_cfg = eval_cfg
        # one process per GPU: every rank draws its device randomness (observation noise, reset / DR / push draws) and its
        # command curriculum from its own streams, otherwise env i of every rank would see identical noise and commands
        self.rank_seed_offset = 0
        self.shared_curriculum = False
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            import os
            self.rank_seed_offset = int(torch.distributed.get_rank())
            # SURVEY.md §8e(4): ONE command curriculum for the envs of all ranks (replayed identically on every rank from the
            # all-gathered event records) instead of one per rank; needs the device curriculum
            self.shared_curriculum = torch.distributed.get_world_size() > 1 and self.device_curriculum and not os.environ.get("GO1_HOST_CURRICULUM") \
                and os.environ.get("GO1_SHARED_CURRICULUM", "1") != "0"
        self.sim_params = sim_params
        self.height_samples = None
        self.debug_viz = False
        self.init_done = False
        self.initial_dynamics_dict = initial_dynamics_dict
        super().__init__(self.cfg, sim_params, physics_engine, sim_device, headless, self.eval_cfg)

        self._init_command_distribution(np.arange(self.num_envs))
        self._init_buffers()
        self._prepare_reward_function()
        self.init_done = True
        self.record_now = False
        self.record_eval_now = False
        self.collecting_evaluation = False
        self.num_still_evaluating = 0

    # ------------------------------------------------------------------ construction
    def create_sim(self):
        """Replaces create_sim/_create_envs (legged_robot.py:493-515, 1481-1609): build the resolved kernel
        configuration, allocate the SoA state, place the env origins, draw the creation-time randomisation."""
        cfg, ecfg = self.cfg, self.eval_cfg
        seed = int(getattr(cfg, "seed", 0)) if hasattr(cfg, "seed") else 0
        seed += 1000 * self.rank_seed_offset
        mesh_type = cfg.terrain.mesh_type
        if mesh_type in ['heightfield', 'trimesh']:     # before the kernel config: Terrain sets the x_offset the teleport reads
            if ecfg is not None:
                self.terrain = Terrain(cfg.terrain, self.num_train_envs, ecfg.terrain, self.num_eval_envs)
            else:
                self.terrain = Terrain(cfg.terrain, self.num_train_envs)
        elif mesh_type not in (None, 'plane'):
            raise ValueError("Terrain mesh type not recognised. Allowed types are [None, plane, heightfield, trimesh]")
        from go1_gym.envs.rewards import REWARD_CONTAINERS
        self._reward_container_cls = REWARD_CONTAINERS[cfg.rewards.reward_container_name]
        self.sim_cfg, info = build_sim_config(cfg, num_envs=self.num_envs, num_train_envs=self.num_train_envs, seed=seed, eval_cfg=ecfg,
                                              reward_container=self._reward_container_cls)
        self.dt = info["dt"]
        self.reward_scales = dict(info["active_reward_scales"])
        self._user_reward_scales = dict(info["user_reward_scales"])
        self.obs_scales = cfg.obs_scales
        self.curriculum_thresholds = cfg_dict(cfg.curriculum_thresholds)
        cfg.command_ranges = cfg_dict(cfg.commands)
        if ecfg is not None:
            ecfg.command_ranges = cfg_dict(ecfg.commands)
        self.max_episode_length = cfg.env.max_episode_length
        self.up_axis_idx = 2
        if mesh_type in ['heightfield', 'trimesh']:
            self._bind_height_field()
        self.core = SimCore(self.sim_cfg, device=self.device, self_collision=info["self_collision"], asset=info["asset"])
        self.num_dof = self.num_dofs = self.num_actuated_dof = 12
        self.num_bodies = len(BODY_NAMES)
        self.dof_names = [f"{l}_{p}_joint" for l in ("FL", "FR", "RL", "RR") for p in ("hip", "thigh", "calf")]
        bodies = info["contact_bodies"]            # Cfg.asset's sets (legged_robot.py:1521-1527, 1580-1590), as the kernel applies them
        self.feet_indices = torch.tensor(bodies["feet"], device=self.device)
        self.penalised_contact_indices = torch.tensor(bodies["penalised"], dtype=torch.long, device=self.device)
        self.termination_contact_indices = torch.tensor(bodies["termination"], dtype=torch.long, device=self.device)
        self.env_origins = torch.zeros(self.num_envs, 3, device=self.device)
        self.terrain_levels = torch.zeros(self.num_envs, device=self.device, dtype=torch.long)
        self.terrain_types = torch.zeros(self.num_envs, device=self.device, dtype=torch.long)
        self._call_train_eval(self._get_env_origins, torch.arange(self.num_envs, device=self.device))
        self.core.env("env_origins").copy_(self.env_origins.t())
        self._init_custom_buffers__()
        self._call_train_eval(self._randomize_rigid_body_props, torch.arange(self.num_envs, device=self.device))
        self.core.sync_rigid_props()          # the bodies are created with these payloads / com displacements (legged_robot.py:667-673)
        if self.num_eval_envs > 0:
            self.core.enable_eval_sums()
        self.common_step_counter = 0
        self._randomize_gravity()

    def _bind_height_field(self):
        """_create_heightfield / _create_trimesh (legged_robot.py:1442-1479): the int16 samples go to the device once and the
        step kernel samples them (bilinear) for every contact point; world (x, y) = (row, col) * horizontal_scale - border_size."""
        t, tc = self.terrain, self.cfg.terrain
        self.height_samples = torch.tensor(t.heightsamples).view(t.tot_rows, t.tot_cols).to(self.device)
        c = self.sim_cfg
        if t.is_flat:
            c.hf = None                      # flat tiles (scripts/train.py): the analytic z = 0 plane
            return
        self._hf_dev = self.height_samples.contiguous()
        c.hf, c.hf_rows, c.hf_cols = self._hf_dev.data_ptr(), int(t.tot_rows), int(t.tot_cols)
        c.hf_hscale, c.hf_vscale, c.hf_border = float(tc.horizontal_scale), float(tc.vertical_scale), float(tc.border_size)

    def _get_heights(self, env_ids, cfg=None):
        """legged_robot.py:1772-1806 (reference-shaped helper; the step kernel evaluates the same expression itself for the
        body-height termination)."""
        cfg = cfg or self.cfg
        t = cfg.terrain
        n_pts = len(t.measured_points_x) * len(t.measured_points_y)
        env_ids = torch.as_tensor(env_ids, device=self.device, dtype=torch.long)
        if t.mesh_type == 'plane' or getattr(self, "height_samples", None) is None:
            return torch.zeros(len(env_ids), n_pts, device=self.device)
        return measured_heights_at(self.base_quat[env_ids], self.base_pos[env_ids], self.height_samples, t)

    @property
    def measured_heights(self):
        if not self.cfg.terrain.measure_heights:
            return 0
        return self._get_heights(torch.arange(self.num_envs, device=self.device))

    def _call_train_eval(self, func, env_ids):
        """legged_robot.py:531-544: `func(ids, cfg)` for the train envs, `func(ids, eval_cfg)` for the eval envs."""
        train, ev = env_ids[env_ids < self.num_train_envs], env_ids[env_ids >= self.num_train_envs]
        ret = ret_eval = None
        if len(train) > 0:
            ret = func(train, self.cfg)
        if len(ev) > 0:
            ret_eval = func(ev, self.eval_cfg)
            if ret is not None and ret_eval is not None:
                ret = torch.cat((ret, ret_eval), axis=-1)
        return ret

    def _get_env_origins(self, env_ids, cfg):
        """legged_robot.py:1675-1714."""
        n, dev = len(env_ids), self.device
        if cfg.terrain.mesh_type in ["heightfield", "trimesh"]:
            self.custom_origins = True
            t = cfg.terrain
            max_init, min_init = t.max_init_terrain_level, t.min_init_terrain_level
            if not t.curriculum:
                max_init, min_init = t.num_rows - 1, 0
            if t.center_robots:
                lo_l, hi_l = t.num_rows // 2 - t.center_span, t.num_rows // 2 + t.center_span - 1
                lo_t, hi_t = t.num_cols // 2 - t.center_span, t.num_cols // 2 + t.center_span - 1
                self.terrain_levels[env_ids] = torch.randint(lo_l, hi_l + 1, (n,), device=dev)
                self.terrain_types[env_ids] = torch.randint(lo_t, hi_t + 1, (n,), device=dev)
            else:
                self.terrain_levels[env_ids] = torch.randint(min_init, max_init + 1, (n,), device=dev)
                self.terrain_types[env_ids] = torch.div(torch.arange(n, device=dev), (n / t.num_cols), rounding_mode='floor').to(torch.long)
            t.max_terrain_level = t.num_rows
            t.terrain_origins = torch.from_numpy(t.env_origins).to(dev).to(torch.float)
            self.env_origins[env_ids] = t.terrain_origins[self.terrain_levels[env_ids], self.terrain_types[env_ids]]
        else:
            self.custom_origins = False
            num_cols = np.floor(np.sqrt(n))
            num_rows = np.ceil(self.num_envs / num_cols)
            xx, yy = torch.meshgrid(torch.arange(num_rows), torch.arange(num_cols), indexing="ij")
            sp = cfg.env.env_spacing
            self.env_origins[env_ids, 0] = sp * xx.flatten()[:n].to(dev)
            self.env_origins[env_ids, 1] = sp * yy.flatten()[:n].to(dev)
            self.env_origins[env_ids, 2] = 0.

    def _init_custom_buffers__(self):
        """legged_robot.py:1260-1297: DR defaults (the SimCore constructor already set 1.0 where needed)."""
        c = self.core
        c.env("friction_coeffs").fill_(1.0)       # default asset friction
        c.env("restitutions").fill_(0.0)
        if self.initial_dynamics_dict is not None:
            for k, v in self.initial_dynamics_dict.items():
                if k in ("friction_coeffs", "restitutions"):
                    c.env(k)[0].copy_(v.to(self.device).reshape(self.num_envs, -1)[:, 0])
                elif k == "payloads":
                    c.env(k)[0].copy_(v.to(self.device))
                elif k == "com_displacements":
                    c.env(k).copy_(v.to(self.device).t())
                elif k in ("motor_strengths", "Kp_factors", "Kd_factors"):
                    c.env(k)[0].copy_(v.to(self.device).reshape(self.num_envs, -1)[:, 0])
        self.gravities = torch.zeros(self.num_envs, 3, dtype=torch.float, device=self.device)
        self.gravity_vec = torch.tensor([0., 0., -1.], device=self.device).repeat((self.num_envs, 1))

    def _randomize_rigid_body_props(self, env_ids, cfg):
        """legged_robot.py:611-633 (creation-time draw; randomize_rigids_after_start is False in train.py)."""
        dr, c, n, dev = cfg.domain_rand, self.core, len(env_ids), self.device
        U = lambda lo, hi, *s: torch.rand(*s, dtype=torch.float, device=dev) * (hi - lo) + lo
        if dr.randomize_base_mass:
            c.env("payloads")[0, env_ids] = U(*dr.added_mass_range, n)
        if dr.randomize_com_displacement:
            c.env("com_displacements")[:, env_ids] = U(*dr.com_displacement_range, n, 3).t()
        if dr.randomize_friction:
            c.env("friction_coeffs")[0, env_ids] = U(*dr.friction_range, n)
        if dr.randomize_restitution:
            c.env("restitutions")[0, env_ids] = U(*dr.restitution_range, n)

    def _randomize_gravity(self, external_force=None):
        """legged_robot.py:546-561: one global gravity offset for all envs (kept on the host: it is a kernel argument)."""
        if external_force is not None:
            g0 = torch.as_tensor(external_force, dtype=torch.float).cpu()
        elif self.cfg.domain_rand.randomize_gravity:
            lo, hi = self.cfg.domain_rand.gravity_range
            g0 = torch.rand(3, dtype=torch.float) * (hi - lo) + lo
        else:
            g0 = getattr(self, "_gravity_host", torch.zeros(3))
        self._gravity_host = g0
        self.gravities[:, :] = g0.to(self.device).unsqueeze(0)
        gravity = g0 + torch.tensor([0., 0., -9.8])
        gv = gravity / torch.norm(gravity)
        self.gravity_vec[:, :] = gv.to(self.device).unsqueeze(0)
        self.core.set_gravity(gravity.tolist(), gv.tolist())

    def _init_command_distribution(self, env_ids):
        """legged_robot.py:1299-1383."""
        from .curriculum import RewardThresholdCurriculum
        c = self.cfg.commands
        self.category_names = ['pronk', 'trot', 'pace', 'bound'] if c.gaitwise_curricula else ['nominal']
        if c.curriculum_type != "RewardThresholdCurriculum":
            raise NotImplementedError(c.curriculum_type)
        dims = [("x_vel", "vel_x"), ("y_vel", "vel_y"), ("yaw_vel", "vel_yaw"), ("body_height", "body_height"),
                ("gait_frequency", "gait_frequency"), ("gait_phase", "gait_phase"), ("gait_offset", "gait_offset"),
                ("gait_bounds", "gait_bound"), ("gait_duration", "gait_duration"), ("footswing_height", "footswing_height"),
                ("body_pitch", "body_pitch"), ("body_roll", "body_roll"), ("stance_width", "stance_width"),
                ("stance_length", "stance_length"), ("aux_reward_coef", "aux_reward_coef")]
        kw = {name: (getattr(c, f"limit_{key}")[0], getattr(c, f"limit_{key}")[1], getattr(c, f"num_bins_{key}")) for name, key in dims}
        # per-rank curricula get per-rank streams; the shared curriculum must start identical everywhere
        cur_seed = c.curriculum_seed + (0 if getattr(self, "shared_curriculum", False) else 1000 * getattr(self, "rank_seed_offset", 0))
        self.curricula = [RewardThresholdCurriculum(seed=cur_seed, **kw) for _ in self.category_names]
        self.env_command_bins = np.zeros(len(env_ids), dtype=int)
        self.env_command_categories = np.zeros(len(env_ids), dtype=int)
        from go1_b200.curriculum_dev import SplitMix64
        self._cat_rng = SplitMix64(cur_seed + 1)      # category draws (torch.rand on the device in the reference)
        rng_keys = ["lin_vel_x", "lin_vel_y", "ang_vel_yaw", "body_height_cmd", "gait_frequency_cmd_range", "gait_phase_cmd_range",
                    "gait_offset_cmd_range", "gait_bound_cmd_range", "gait_duration_cmd_range", "footswing_height_range",
                    "body_pitch_range", "body_roll_range", "stance_width_range", "stance_length_range", "aux_reward_coef_range"]
        low = np.array([getattr(c, k)[0] for k in rng_keys])
        high = np.array([getattr(c, k)[1] for k in rng_keys])
        for cur in self.curricula:
            cur.set_to(low=low, high=high)

    def _init_buffers(self):
        """legged_robot.py:1123-1258 — everything is a view of (or lives in) the SoA device state."""
        self.extras = LazyExtras()
        self.noise_scale_vec = torch.tensor(list(self.sim_cfg.noise_scale_vec)[:self.num_obs], device=self.device)
        self.add_noise = self.cfg.noise.add_noise
        self.default_dof_pos = torch.tensor(list(self.sim_cfg.default_dof_pos), device=self.device).unsqueeze(0)
        self.commands_scale = torch.tensor(list(self.sim_cfg.commands_scale)[:self.cfg.commands.num_commands], device=self.device)
        self.torque_limits = torch.full((12,), self.sim_cfg.torque_limit, device=self.device)
        self.dof_pos_limits = torch.stack((torch.tensor(list(self.sim_cfg.soft_limit_lo)), torch.tensor(list(self.sim_cfg.soft_limit_hi))), 1).to(self.device)
        self._pending_interval = (np.zeros(0, dtype=np.int64), np.zeros((0, 4), dtype=np.float32))
        self._ep_len_dirty = False
        self._time_outs = torch.zeros(self.num_train_envs, dtype=torch.bool, device=self.device)
        self._env_bins_dev = torch.zeros(self.num_train_envs, device=self.device)
        self._env_bins_host = [torch.zeros(self.num_train_envs).pin_memory() for _ in range(2)]      # ping-pong upload staging
        self._env_bins_host_np = [t.numpy() for t in self._env_bins_host]
        self._env_bins_flip = 0
        self._env_bins_dirty = True
        self.actions = torch.zeros(self.num_envs, self.num_actions, device=self.device)
        self.lag_timesteps = self.cfg.domain_rand.lag_timesteps

    def _prepare_reward_function(self):
        """legged_robot.py:1385-1429: the reward container and the names of the active terms.  The kernel owns the arithmetic of the
        built-in terms; user terms (plain `_reward_<name>` methods of the container, config.reward_tables) run in torch beside it."""
        user = self._user_reward_scales
        sc = self.sim_cfg.reward_scale
        kernel = {n for i, n in enumerate(capi.REWARD_TERMS) if sc[i] != 0}
        self.reward_names = [n for n in self.reward_scales if n != "termination" and (n in kernel or n in user)]
        self.user_reward_names = list(user)
        K, N, dev = len(user), self.num_envs, self.device
        if K == 0:
            self.reward_container = self._reward_container_cls(self)
            return
        self._pre_roll = torch.zeros(capi.PRE_ROLL_ROWS, 4 * N, device=dev)
        self.reward_container = self._reward_container_cls(PreRollEnv(self, self._pre_roll))
        self._user_fns = [getattr(self.reward_container, "_reward_" + n) for n in user]
        self._user_scales = (ctypes.c_float * K)(*user.values())
        self._user_raw = torch.zeros(K, N, device=dev)
        self._user_sums = torch.zeros(K, N, device=dev)
        self._user_sums_eval = torch.full((K, N), -1.0, device=dev) if self.num_eval_envs > 0 else None
        self._reward_ws = torch.zeros(max(1, int(capi.lib().go1_reward_finish_workspace(N, K))), device=dev)

    def _eval_user_rewards(self):
        """compute_reward's loop for the user terms (legged_robot.py:270-279): raw values into _user_raw."""
        for k, fn in enumerate(self._user_fns):
            r = fn()
            if not isinstance(r, torch.Tensor) or r.shape != (self.num_envs,):
                raise ValueError(f"_reward_{self.user_reward_names[k]} must return a [num_envs] tensor, got "
                                 f"{tuple(r.shape) if isinstance(r, torch.Tensor) else type(r).__name__}")
            self._user_raw[k].copy_(r)

    def _sim_step(self, actions, common_step):
        """The step launch: go1_sim_step, or with user terms the deferred step, the terms and go1_sim_reward_finish."""
        core = self.core
        if not self.user_reward_names:
            core.step(actions, common_step=common_step, mode=0)
            return
        core.step_deferred(actions, self._pre_roll, common_step=common_step)
        self._eval_user_rewards()
        core.reward_finish(self._user_raw, self._user_scales, self._user_sums, self._reward_ws)

    def _user_rewards_capturable(self):
        """Whether the user terms can run inside a captured CUDA graph (no host synchronisation, ...): a trial capture of the
        terms alone, which executes nothing."""
        g = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(g):
                self._eval_user_rewards()
            return True
        except Exception as e:
            import warnings
            warnings.warn(f"user reward terms cannot be captured in a CUDA graph ({type(e).__name__}: {e}); the rollout runs "
                          "launch by launch instead")
            torch.cuda.synchronize()
            return False

    # ------------------------------------------------------------------ reference attribute surface (views / copies)
    obs_buf = property(lambda s: s.core.obs)
    privileged_obs_buf = property(lambda s: s.core.priv_obs)
    rew_buf = property(lambda s: s.core.rew)
    reset_buf = property(lambda s: s.core.reset_u8.bool())
    time_out_buf = property(lambda s: s.core.timeout_u8.bool())
    rew_buf_pos = property(lambda s: s.core.env("rew_buf_pos")[0])
    rew_buf_neg = property(lambda s: s.core.env("rew_buf_neg")[0])
    commands = property(lambda s: s.core.env_aos("commands")[:, :s.cfg.commands.num_commands])      # writable view [N, num_commands]
    gait_indices = property(lambda s: s.core.env("gait_indices")[0])
    base_lin_vel = property(lambda s: s.core.env_aos("base_lin_vel"))
    base_ang_vel = property(lambda s: s.core.env_aos("base_ang_vel"))
    projected_gravity = property(lambda s: s.core.env_aos("projected_gravity"))
    base_pos = property(lambda s: s.core.env_aos("root_pos"))
    base_quat = property(lambda s: s.core.env_aos("root_quat"))
    dof_pos = property(lambda s: s.core.joint_aos("dof_pos"))
    dof_vel = property(lambda s: s.core.joint_aos("dof_vel"))
    torques = property(lambda s: s.core.joint_aos("torques"))
    joint_pos_target = property(lambda s: s.core.joint_aos("joint_pos_target"))
    last_actions = property(lambda s: s.core.joint_aos("last_actions"))
    last_last_actions = property(lambda s: s.core.joint_aos("last_last_actions"))
    last_dof_vel = property(lambda s: s.core.joint_aos("last_dof_vel"))
    foot_positions = property(lambda s: s.core.foot_aos("foot_positions"))
    foot_velocities = property(lambda s: s.core.foot_aos("foot_velocities"))
    clock_inputs = property(lambda s: s.core.leg("clock_inputs")[0])
    desired_contact_states = property(lambda s: s.core.leg("desired_contact_states")[0])
    foot_indices = property(lambda s: s.core.leg("foot_indices")[0])
    friction_coeffs = property(lambda s: s.core.env("friction_coeffs")[0].unsqueeze(1).repeat(1, 4))
    restitutions = property(lambda s: s.core.env("restitutions")[0].unsqueeze(1).repeat(1, 4))
    payloads = property(lambda s: s.core.env("payloads")[0])
    com_displacements = property(lambda s: s.core.env_aos("com_displacements"))
    motor_strengths = property(lambda s: s.core.env("motor_strengths")[0].unsqueeze(1).repeat(1, 12))
    motor_offsets = property(lambda s: s.core.joint_aos("motor_offsets"))

    @property
    def root_states(self):
        c = self.core
        return torch.cat((c.env_aos("root_pos"), c.env_aos("root_quat"), c.env_aos("root_lin_vel"), c.env_aos("root_ang_vel")), 1)

    @property
    def contact_forces(self):
        """[N, 17, 3] in Isaac Gym body order (BODY_NAMES: base; per leg hip, thigh, calf, foot)."""
        c = self.core
        out = torch.zeros(self.num_envs, len(BODY_NAMES), 3, device=self.device)
        out[:, BODY_NAMES.index("base")] = c.foot_aos("base_contact_forces_part").sum(1)
        for part in ("hip", "thigh", "calf", "foot"):
            out[:, [BODY_NAMES.index(f"{leg}_{part}") for leg in ("FL", "FR", "RL", "RR")]] = c.foot_aos(f"{part}_contact_forces")
        return out

    @property
    def episode_sums(self):
        es = self.core.env("episode_sums")
        d = {n: es[capi.REWARD_TERMS.index(n)] for n in self.reward_scales if n in capi.REWARD_TERMS}
        for i, n in enumerate(self.user_reward_names):
            d[n] = self._user_sums[i]
        d["total"] = es[capi.NUM_REWARD_TERMS]
        return d

    @property
    def episode_sums_eval(self):
        """legged_robot.py:1420-1424: the first finished episode of every eval env (-1 = none yet; "total" starts at 0)."""
        ev = self.core.episode_sums_eval
        if ev is None:
            return {}
        d = {n: ev[capi.REWARD_TERMS.index(n)] for n in self.reward_scales if n in capi.REWARD_TERMS}
        for i, n in enumerate(self.user_reward_names):
            d[n] = self._user_sums_eval[i]
        d["total"] = ev[capi.NUM_REWARD_TERMS]
        return d

    @property
    def command_sums(self):
        cs = self.core.env("command_sums")
        d = {n: cs[capi.REWARD_TERMS.index(n)] for n in self.reward_scales if n in capi.REWARD_TERMS}
        for i, k in enumerate(capi.COMMAND_SUM_EXTRAS):
            d[k] = cs[capi.NUM_REWARD_TERMS + i]
        return d

    @property
    def episode_length_buf(self):
        return self.core.episode_length_buf

    @episode_length_buf.setter
    def episode_length_buf(self, value):
        """The Runner overwrites this with random episode lengths (ppo_cse/__init__.py:114-116)."""
        self.core.episode_length_buf.copy_(value.to(self.device).to(torch.int32))
        self._ep_len_dirty = True

    @property
    def actions(self):
        """The last actions clipped to +-clip_actions (legged_robot.py:64-65); the kernel clips its own copy."""
        a = self.__dict__.get("_raw_actions")
        clip = self.cfg.normalization.clip_actions
        return None if a is None else torch.clip(a, -clip, clip)

    @actions.setter
    def actions(self, value):
        self._raw_actions = value

    # ------------------------------------------------------------------ stepping
    def step(self, actions):
        """legged_robot.py:60-88."""
        core = self.core
        actions = actions.to(self.device, dtype=torch.float32).contiguous()
        self._raw_actions = actions                 # `self.actions` (the clipped copy, legged_robot.py:64-65) is produced on read
        self.common_step_counter += 1
        dc = self._device_curriculum()
        if dc is not None:
            return self._step_device(dc, actions)
        self._apply_pending_interval_resample()
        self._sim_step(actions, self.common_step_counter)
        rid, rsum, iid, isum = core.fetch_events()
        self._pending_interval = (iid, isum)
        self._post_physics_step_callback_host()
        if len(rid):
            self._reset_sorted(rid, rsum, True, actions)
        return self.obs_buf, self.privileged_obs_buf, self.rew_buf, self.reset_buf, self.extras

    # ------------------------------------------------------------------ device-resident curriculum (no host round trip)
    device_curriculum = True        # class switch; GO1_HOST_CURRICULUM=1 in the environment forces the host path

    def _device_curriculum(self):
        dc = self.__dict__.get("_dev_cur", False)
        if dc is False:
            import os
            dc = None
            if self.device_curriculum and not os.environ.get("GO1_HOST_CURRICULUM") and self.core.noise is None and self.core.reset_rand is None:
                from go1_b200.curriculum_dev import DeviceCurriculum
                dc = DeviceCurriculum(self, _LOCAL_RANGE, _TASK_KEYS, torch.distributed.group.WORLD if self.shared_curriculum else None)
            self._dev_cur = dc
        return dc

    def _curriculum_to_host(self, keep_device=False):
        dc = self.__dict__.get("_dev_cur")
        if dc:
            dc.to_host(keep_device=keep_device)

    def _step_device(self, dc, actions):
        """step() with the curriculum on the device: five stream-ordered launches, no synchronisation.
        [resample list 1 (envs marked last step)] -> [step kernel] -> [resample list 0] -> [reset kernel]."""
        core = self.core
        if self._ep_len_dirty:
            self._sync_interval_events_after_ep_len_write()
        dc.to_device()
        dc.resample(1)
        self._sim_step(actions, self.common_step_counter)
        dc.gather()
        self._post_physics_step_callback_host()
        acc = torch.zeros(capi.NUM_EPISODE_SUMS + 1, device=self.device)
        dc.resample(0)
        dc.reset_envs(actions, True, self.common_step_counter, acc)
        # a step without a reset carries the last non-empty sums forward (the reference's extras entry just stays in place)
        prev = self.__dict__.get("_episode_acc_prev")
        if prev is not None:
            torch.where(acc[capi.NUM_EPISODE_SUMS:] > 0, acc, prev, out=acc)
        self._episode_acc_prev = acc
        user_acc = None
        if self.user_reward_names:
            K = len(self.user_reward_names)
            user_acc = torch.empty(K + 1, device=self.device)
            core.user_reward_fold(dc.out_ids, dc.out_count, 0, self._user_sums, self._user_sums_eval, user_acc)
            prev = self.__dict__.get("_user_acc_prev")
            if prev is not None:
                torch.where(user_acc[K:] > 0, user_acc, prev, out=user_acc)
            self._user_acc_prev = user_acc
        ex = self.extras
        ex["train/episode"] = _LazyDict(self._episode_builder(acc, may_be_empty=True, user_acc=user_acc))
        if self.cfg.commands.command_curriculum:
            ex["env_bins"] = dc.env_bins_f32
            ex["curriculum/distribution"] = _LazyDict(self._distribution_builder())
        if self.cfg.env.send_timeouts:
            ex["time_outs"] = dc.time_outs
        if self.num_eval_envs > 0:
            ex["eval/episode"] = {}            # legged_robot.py:188-195: the entry carries no values (the sums go to episode_sums_eval)
        return self.obs_buf, self.privileged_obs_buf, self.rew_buf, self.reset_buf, self.extras

    def _sync_interval_events_after_ep_len_write(self):
        """Episode lengths were overwritten from outside (Runner: init_at_random_ep_len): rebuild the device-side list of envs
        due for the periodic command resample at the next step."""
        core = self.core
        interval = int(self.sim_cfg.resampling_interval)
        ep = core.episode_length_buf
        ids = torch.nonzero((ep + 1) % interval == 0).squeeze(1) if interval > 0 else ep.new_zeros(0, dtype=torch.long)
        k = int(ids.numel())
        if k:
            rows = [capi.REWARD_TERMS.index(key) for key in _TASK_KEYS]
            core.events[1, :k, 0] = ids.float()
            core.events[1, :k, 1:5] = core.env("command_sums")[rows][:, ids].t()
        core.event_count[1] = k
        self._ep_len_dirty = False
        dc = self.__dict__.get("_dev_cur")
        if dc:
            dc.gather()           # cross-rank replay: every rank needs every rank's rebuilt list

    def _apply_pending_interval_resample(self):
        """legged_robot.py:683-686: envs whose episode length hits a multiple of resampling_time/dt."""
        if self._ep_len_dirty:          # episode lengths were overwritten from outside: rebuild the pending list
            ep = self.core.episode_length_buf.cpu().numpy()
            interval = int(self.sim_cfg.resampling_interval)
            ids = np.nonzero((ep + 1) % interval == 0)[0] if interval > 0 else np.zeros(0, dtype=np.int64)
            cs = self.core.env("command_sums")[[capi.REWARD_TERMS.index(k) for k in _TASK_KEYS]][:, torch.as_tensor(ids, device=self.device, dtype=torch.long)]
            self._pending_interval = (ids, cs.t().cpu().numpy())
            self._ep_len_dirty = False
        ids, sums = self._pending_interval
        if len(ids) == 0:
            return
        cmds = self._resample_commands_host(ids, sums)
        self.core.set_commands(ids, cmds)
        self._env_bins_dirty = True
        self._pending_interval = (np.zeros(0, dtype=np.int64), np.zeros((0, 4), dtype=np.float32))

    def _post_physics_step_callback_host(self):
        """The host part of legged_robot.py:701-705 (global gravity impulses)."""
        dr = self.cfg.domain_rand
        if self.common_step_counter % int(dr.gravity_rand_interval) == 0:
            self._randomize_gravity()
        if int(self.common_step_counter - dr.gravity_rand_duration) % int(dr.gravity_rand_interval) == 0:
            self._randomize_gravity(torch.tensor([0., 0., 0.]))

    def post_physics_step(self):
        raise NotImplementedError("fused into go1_sim_step; see step()")

    # ------------------------------------------------------------------ commands / resets
    def _resample_constants(self):
        """(ep_len float32, columns of the 4 task sums that have an active reward, their float32 success thresholds)."""
        hc = self.__dict__.get("_resample_consts")
        if hc is None:
            cfg = self.cfg
            timesteps = int(cfg.commands.resampling_time / self.dt)
            ep_len = min(cfg.env.max_episode_length, timesteps)
            present = [key for key in _TASK_KEYS if key in self.reward_scales]
            cols = [_TASK_KEYS.index(key) for key in present]
            thr = np.array([self.curriculum_thresholds[key] * self.reward_scales[key] for key in present], dtype=np.float32)
            hc = self._resample_consts = (np.float32(ep_len), cols, thr)
        return hc

    def _resample_commands_host(self, env_ids, task_sums):
        """legged_robot.py:710-824 for env ids (numpy, ascending) whose 4 task command sums are `task_sums`.
        Returns the new commands [k, 15]; updates curricula, env_command_bins/categories.  Runs on the critical path
        between the event D2H and the reset launch, so it is written for few numpy calls at k ~ 5; bit-exactness
        against the reference is pinned by tests/test_resample_host.py."""
        cfg = self.cfg
        k = len(env_ids)
        ep_len, cols, thr = self._resample_constants()
        ncat = len(self.category_names)
        nc = cfg.commands.num_commands
        if len(cols) > 0:
            # success = every task reward above its threshold, in float32 like the reference's torch comparison
            ok = (task_sums[:, cols].astype(np.float32, copy=False) / ep_len > thr).all(axis=1)
            if ok.any():
                ok_ids = env_ids[ok]
                ok_bins, ok_cats = self.env_command_bins[ok_ids], self.env_command_categories[ok_ids]
                for i in (range(ncat) if ncat > 1 else (0,)):
                    m = ok_cats == i
                    if m.any():
                        self.curricula[i].apply_successes(ok_bins[m], _LOCAL_RANGE)
        # new categories: host RNG (the reference draws torch.rand on the device; only the distribution matters)
        r = self._cat_rng.random(k)
        if ncat in (1, 2, 4, 8):       # p = 1/ncat is exact: p*i <= r < p*(i+1)  <=>  floor(r * ncat) == i
            cat = (r * ncat).astype(np.intp)
        else:
            p = 1. / ncat
            cat = np.full(k, -1, dtype=np.intp)
            for i in range(ncat):
                cat[np.logical_and(p * i <= r, r < p * (i + 1))] = i
        c = np.zeros((k, capi.NUM_COMMANDS), dtype=np.float32)
        new_bins = self.env_command_bins[env_ids]
        new_cats = self.env_command_categories[env_ids]
        members = [None] * ncat
        for i in range(ncat):
            m = np.flatnonzero(cat == i) if ncat > 1 else np.arange(k)
            members[i] = m
            if len(m) == 0:
                continue
            cmds, bins = self.curricula[i].sample(batch_size=len(m))
            new_bins[m] = bins
            new_cats[m] = i
            c[m, :nc] = cmds[:, :nc]            # float64 -> float32 on assignment, like torch.Tensor(new_commands)
        self.env_command_bins[env_ids] = new_bins
        self.env_command_categories[env_ids] = new_cats
        q = np.float32(0.25)
        if nc > 5:
            if cfg.commands.gaitwise_curricula:
                for category, m in zip(self.category_names, members):
                    if len(m) == 0:
                        continue
                    if category == "pronk":
                        c[m, 5:8] = np.mod(c[m, 5:8] / 2 - q, 1)
                    elif category == "trot":
                        c[m, 5] = c[m, 5] / 2 + q; c[m, 6:8] = 0
                    elif category == "pace":
                        c[m, 6] = c[m, 6] / 2 + q; c[m, 5] = 0; c[m, 7] = 0
                    elif category == "bound":
                        c[m, 7] = c[m, 7] / 2 + q; c[m, 5:7] = 0
            elif cfg.commands.exclusive_phase_offset:
                r2 = self._cat_rng.random(k)
                trot, pace, bound = r2 < 0.34, np.logical_and(0.34 <= r2, r2 < 0.67), 0.67 <= r2
                c[pace, 5] = 0; c[bound, 5] = 0; c[trot, 6] = 0; c[bound, 6] = 0; c[trot, 7] = 0; c[pace, 7] = 0
            elif cfg.commands.balance_gait_distribution:
                r2 = self._cat_rng.random(k)
                pronk, trot = r2 <= 0.25, np.logical_and(0.25 <= r2, r2 < 0.50)
                pace, bound = np.logical_and(0.50 <= r2, r2 < 0.75), 0.75 <= r2
                for j in (5, 6, 7):
                    c[pronk, j] = np.mod(c[pronk, j] / 2 - q, 1)
                c[trot, 6] = 0; c[trot, 7] = 0; c[pace, 5] = 0; c[pace, 7] = 0; c[bound, 5] = 0; c[bound, 6] = 0
                c[trot, 5] = c[trot, 5] / 2 + q; c[pace, 6] = c[pace, 6] / 2 + q
                c[bound, 7] = c[bound, 7] / 2 + q
            if cfg.commands.binary_phases:
                c[:, 5:8] = np.mod(np.round(2 * c[:, 5:8]) / np.float32(2.0), 1)     # torch.round == np.round (half to even)
        x, y = c[:, 0], c[:, 1]
        c[:, :2] *= (np.sqrt(x * x + y * y) > np.float32(0.2))[:, None]          # torch.norm(...) > 0.2 in float32
        return c

    def _resample_commands(self, env_ids):
        """Reference-shaped entry point (legged_robot.py:710): env_ids is a tensor."""
        ids = np.sort(np.asarray(env_ids.cpu() if hasattr(env_ids, "cpu") else env_ids, dtype=np.int64))
        if len(ids) == 0:
            return
        if self.shared_curriculum:
            raise NotImplementedError("shared (cross-rank) curriculum: _resample_commands on the host would desynchronise the ranks")
        self._curriculum_to_host()
        idx = torch.as_tensor(ids, device=self.device)
        cs = self.core.env("command_sums")[[capi.REWARD_TERMS.index(k) for k in _TASK_KEYS]][:, idx].t().cpu().numpy()
        self.core.set_commands(ids, self._resample_commands_host(ids, cs))
        self._env_bins_dirty = True

    def reset_idx(self, env_ids, _sums=None, _post_step=False, _actions=None):
        """legged_robot.py:150-239."""
        if len(env_ids) == 0:
            return
        ids = np.sort(np.asarray(env_ids.cpu() if hasattr(env_ids, "cpu") else env_ids, dtype=np.int64))
        self._curriculum_to_host()
        if _sums is None:
            idx = torch.as_tensor(ids, device=self.device)
            _sums = self.core.env("command_sums")[[capi.REWARD_TERMS.index(k) for k in _TASK_KEYS]][:, idx].t().cpu().numpy()
        self._reset_sorted(ids, _sums, _post_step, _actions)

    def _resample_commands_host_all_ranks(self, sums):
        """The host twin for ALL envs of ALL ranks at once (env.reset() under the shared curriculum): every rank replays the
        single-process call reset_idx(arange(world * N)) -- same successes, same category draws, same RandomState words -- and
        keeps its own slice, so the curricula stay identical everywhere.  Collective: every rank must call it."""
        import torch.distributed as dist
        W, r, N = dist.get_world_size(), dist.get_rank(), self.num_envs
        dev = self.device

        def gather(a, dtype):
            loc = torch.as_tensor(np.ascontiguousarray(a), device=dev).to(dtype)
            out = torch.empty((W * loc.shape[0],) + tuple(loc.shape[1:]), device=dev, dtype=dtype)      # concatenated along dim 0
            dist.all_gather_into_tensor(out, loc)
            return out.cpu().numpy()
        sums_g = gather(sums, torch.float32)
        bins_l, cats_l = self.env_command_bins, self.env_command_categories
        self.env_command_bins, self.env_command_categories = gather(bins_l, torch.int64), gather(cats_l, torch.int64)
        try:
            cmds = self._resample_commands_host(np.arange(W * N), sums_g)
            bins_l[:] = self.env_command_bins[r * N:(r + 1) * N]
            cats_l[:] = self.env_command_categories[r * N:(r + 1) * N]
        finally:
            self.env_command_bins, self.env_command_categories = bins_l, cats_l
        return cmds[r * N:(r + 1) * N]

    def _reset_sorted(self, ids, sums, post_step, actions):
        """reset_idx for ascending numpy ids whose task command sums are already on the host (the step() path)."""
        core = self.core
        if self.shared_curriculum:
            if len(ids) != self.num_envs:
                raise NotImplementedError("shared (cross-rank) curriculum: host-side reset_idx is collective and resets ALL envs of every rank; "
                                          "partial resets happen on the device inside step()")
            cmds = self._resample_commands_host_all_ranks(sums)
        else:
            cmds = self._resample_commands_host(ids, sums)
        core.episode_acc.zero_()
        core.reset_idx(ids, cmds, actions=actions, post_step=post_step, common_step=self.common_step_counter)
        self._user_acc = None
        if self.user_reward_names:
            self._user_acc = torch.empty(len(self.user_reward_names) + 1, device=self.device)
            ids_dev = torch.as_tensor(ids, dtype=torch.int32).to(self.device)
            core.user_reward_fold(ids_dev, None, len(ids), self._user_sums, self._user_sums_eval, self._user_acc)
        self._env_bins_dirty = True
        self._fill_extras(ids)

    def _episode_builder(self, acc, may_be_empty=False, user_acc=None):
        """extras["train/episode"] of legged_robot.py:180-229 from one snapshot `acc` of the device accumulators
        (episode sums of the envs reset in that step + their count; `user_acc` the same for the user terms).  may_be_empty: no env
        has reset yet -> no entries."""
        core, env = self.core, self
        user = {n: i for i, n in enumerate(self.user_reward_names)}

        def build_episode():
            if may_be_empty and float(acc[capi.NUM_EPISODE_SUMS]) == 0.0:
                return {}
            means = acc[:capi.NUM_EPISODE_SUMS] / acc[capi.NUM_EPISODE_SUMS].clamp(min=1.0)
            ep = {}
            for name in list(env.reward_scales) + ["total"]:
                if name == "total":
                    ep["rew_total"] = means[capi.NUM_REWARD_TERMS]
                elif name in user:
                    if user_acc is not None:
                        ep["rew_" + name] = user_acc[user[name]] / user_acc[len(user)].clamp(min=1.0)
                elif name in capi.REWARD_TERMS:
                    ep["rew_" + name] = means[capi.REWARD_TERMS.index(name)]
            if env.cfg.terrain.curriculum:
                ep["terrain_level"] = torch.mean(env.terrain_levels[:env.num_train_envs].float())
            if env.cfg.commands.command_curriculum:
                env._curriculum_to_host(keep_device=True)
                cmd = core.env("commands")
                mins, maxs = cmd.min(dim=1).values, cmd.max(dim=1).values
                for idx, nm in ((8, "duration"), (7, "bound"), (6, "offset"), (5, "phase"), (4, "freq"), (0, "x_vel"), (1, "y_vel"), (2, "yaw_vel")):
                    ep[f"min_command_{nm}"] = mins[idx]
                    ep[f"max_command_{nm}"] = maxs[idx]
                if env.cfg.commands.num_commands > 9:
                    ep["min_command_swing_height"] = mins[9]
                    ep["max_command_swing_height"] = maxs[9]
                for curriculum, category in zip(env.curricula, env.category_names):
                    ep[f"command_area_{category}"] = np.sum(curriculum.weights) / curriculum.weights.shape[0]
                ep["min_action"] = torch.min(env.actions)
                ep["max_action"] = torch.max(env.actions)
            return ep
        return build_episode

    def _distribution_builder(self):
        def build():
            self._curriculum_to_host(keep_device=True)
            return {**{f"weights_{c}": cur.weights for cur, c in zip(self.curricula, self.category_names)},
                    **{f"grid_{c}": cur.grid for cur, c in zip(self.curricula, self.category_names)}}
        return build

    def _fill_extras(self, ids):
        """legged_robot.py:180-234.  Everything the logger consumes is produced lazily from ONE snapshot of the device
        accumulators taken here (a clone, no host sync); the dict values are materialised when somebody reads them."""
        core, ex = self.core, self.extras
        if (ids < self.num_train_envs).any():
            ex["train/episode"] = _LazyDict(self._episode_builder(core.episode_acc.clone(), user_acc=self.__dict__.get("_user_acc")))
        if (ids >= self.num_train_envs).any():
            ex["eval/episode"] = {}
        if self.cfg.commands.command_curriculum:
            if self._env_bins_dirty:
                f = self._env_bins_flip = self._env_bins_flip ^ 1
                self._env_bins_host_np[f][:] = self.env_command_bins[:self.num_train_envs]
                self._env_bins_dev.copy_(self._env_bins_host[f], non_blocking=True)
                self._env_bins_dirty = False
                core.h2d_bytes += 4 * self.num_train_envs
            ex["env_bins"] = self._env_bins_dev
            ex["curriculum/distribution"] = _LazyDict(self._distribution_builder())
        if self.cfg.env.send_timeouts:
            self._time_outs = core.timeout_u8[:self.num_train_envs].bool()      # a copy taken at reset time (legged_robot.py:234)
            ex["time_outs"] = self._time_outs

    def set_idx_pose(self, env_ids, dof_pos, base_state):
        """legged_robot.py:241-261."""
        if len(env_ids) == 0:
            return
        c, ids = self.core, env_ids.to(self.device).long()
        if dof_pos is not None:
            q = c.joint_aos("dof_pos"); q[ids] = dof_pos.to(self.device); c.set_joint_aos("dof_pos", q)
            v = c.joint_aos("dof_vel"); v[ids] = 0.; c.set_joint_aos("dof_vel", v)
        b = base_state.to(self.device).reshape(-1, 13)
        c.env("root_pos")[:, ids] = b[:, 0:3].t(); c.env("root_quat")[:, ids] = b[:, 3:7].t()
        c.env("root_lin_vel")[:, ids] = b[:, 7:10].t(); c.env("root_ang_vel")[:, ids] = b[:, 10:13].t()

    # ------------------------------------------------------------------ recording API (rendering is out of scope)
    def start_recording(self):
        self.record_now = True

    def start_recording_eval(self):
        self.record_eval_now = True

    def pause_recording(self):
        self.record_now = False

    def pause_recording_eval(self):
        self.record_eval_now = False

    def get_complete_frames(self):
        return []

    def get_complete_frames_eval(self):
        return []

    def render(self, mode="rgb_array"):
        raise NotImplementedError("no renderer: SURVEY.md §2 row 1 marks rendering out of scope")
