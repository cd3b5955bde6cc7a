"""SimCore — owns the torch-allocated device buffers of one sim instance and drives libgo1b200.so.

State lives in three SoA slabs (`env_f32 [rows][N]`, `leg_f32 [rows][4N]`, `env_i32 [rows][N]`); the row
offsets are queried from the library by field name, so this file has no layout knowledge of its own.
Accessors return torch views in the reference's AoS shapes (writes go through where the view is a true
view; `aos()` helpers return copies).
"""
import ctypes as C

import numpy as np
import torch

from . import capi
from .config import load_actuator_weights


class SimCore:
    def __init__(self, sim_cfg: capi.Go1SimConfig, device="cuda:0", inject_noise=False, inject_reset_rand=False, self_collision=None,
                 asset=None):
        if not torch.cuda.is_available():
            raise capi.Go1Error("SimCore needs a CUDA device: the Go1 step kernel has no CPU fallback")
        self.L = capi.lib()
        self.device = torch.device(device)
        self.dev_index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.cfg = sim_cfg
        self.N = N = int(sim_cfg.num_envs)
        self.num_obs, self.num_priv = int(sim_cfg.num_obs), int(sim_cfg.num_priv_obs)
        dev = self.device
        self.n_env_rows = self.L.go1_sim_num_rows(0)
        self.n_leg_rows = self.L.go1_sim_num_rows(1)
        self.env_f32 = torch.zeros(self.n_env_rows, N, device=dev)
        self.leg_f32 = torch.zeros(self.n_leg_rows, 4 * N, device=dev)
        self.env_i32 = torch.zeros(self.L.go1_sim_num_rows(2), N, dtype=torch.int32, device=dev)
        self.obs = torch.zeros(N, self.num_obs, device=dev)
        self._priv_store = torch.zeros(N, max(self.num_priv, 1), device=dev)
        self.priv_obs = self._priv_store[:, :self.num_priv] if self.num_priv else self._priv_store[:, :0]
        self.rew = torch.zeros(N, device=dev)
        self.reset_u8 = torch.ones(N, dtype=torch.uint8, device=dev)       # base_task.py:61 (reset_buf init ones)
        self.timeout_u8 = torch.zeros(N, dtype=torch.uint8, device=dev)
        self.event_count = torch.zeros(2, dtype=torch.int32, device=dev)
        self.events = torch.zeros(2, N, capi.EVENT_STRIDE, device=dev)
        self.episode_acc = torch.zeros(capi.NUM_EPISODE_SUMS + 1, device=dev)
        self.noise = torch.zeros(N, self.num_obs, device=dev) if inject_noise else None
        self.reset_rand = torch.zeros(N, capi.RESET_RAND_STRIDE, device=dev) if inject_reset_rand else None
        self.episode_sums_eval = None
        # pinned staging for the per-step host round trip (event list down, new commands up)
        self.h_count = torch.zeros(2, dtype=torch.int32).pin_memory()
        self.h_events = torch.zeros(2, N, capi.EVENT_STRIDE).pin_memory()
        # upload staging, one slot per call site (0 = reset_idx, 1 = set_commands): [k int32 ids][k x 15 float commands]
        # packed back to back so that one H2D copy of 64*k bytes carries both; a slot is rewritten only after the event
        # recorded behind its previous copy has completed
        W = 1 + capi.NUM_COMMANDS
        self._h_stage = [torch.zeros(N * W).pin_memory() for _ in range(2)]
        self._h_stage_f32 = [t.numpy() for t in self._h_stage]
        self._h_stage_i32 = [a.view(np.int32) for a in self._h_stage_f32]
        self._d_stage = [torch.zeros(N * W, device=dev) for _ in range(2)]
        self._d_stage_ptr = [t.data_ptr() for t in self._d_stage]
        self._stage_event = [torch.cuda.Event() for _ in range(2)]
        self._stage_used = [False, False]
        self.h2d_bytes = self.d2h_bytes = 0            # host<->device traffic of the step path (bench.py reports it)
        self.iters_counted = 1
        self.gravity = (C.c_float * 3)(0.0, 0.0, -9.8)
        self.gravity_vec = (C.c_float * 3)(0.0, 0.0, -1.0)
        # gravity and the step counter also live in device memory (the kernels read them from there), so that a captured CUDA
        # graph of the env step follows _randomize_gravity and the Philox streams keep advancing across replays
        self.gravity_dev = torch.tensor([0.0, 0.0, -9.8, 0.0, 0.0, -1.0], device=dev)
        self.step_dev = torch.zeros(1, dtype=torch.int64, device=dev)

        w = load_actuator_weights()
        self._handle = C.c_void_p()
        with torch.cuda.device(self.dev_index):
            capi.check(self.L.go1_sim_create(C.byref(sim_cfg), w.ctypes.data_as(C.c_void_p), self.dev_index, C.byref(self._handle)),
                       "go1_sim_create")
        self.self_collision = self_collision
        if self_collision is not None and self_collision.enabled:     # only before the first step (captured graphs keep the kernel)
            capi.check(self.L.go1_sim_set_self_collision(self._handle, C.byref(self_collision)), "go1_sim_set_self_collision")
        self.asset = asset                                             # Go1AssetOptions; None keeps the Go1 values of go1_sim_create
        if asset is not None:                                          # also only before the first step (graphs keep kernel arguments)
            capi.check(self.L.go1_sim_set_asset_options(self._handle, C.byref(asset)), "go1_sim_set_asset_options")
        self._bind()
        # DR defaults (legged_robot.py:1260-1278)
        self.env("motor_strengths").fill_(1.0)
        self.env("Kp_factors").fill_(1.0)
        self.env("Kd_factors").fill_(1.0)
        self.env("friction_coeffs").fill_(1.0)
        self.env("root_quat")[3].fill_(1.0)

    def _bind(self):
        b = capi.Go1SimBuffers()
        b.env_f32, b.leg_f32, b.env_i32 = self.env_f32.data_ptr(), self.leg_f32.data_ptr(), self.env_i32.data_ptr()
        b.obs, b.priv_obs = self.obs.data_ptr(), self._priv_store.data_ptr()
        b.rew, b.reset, b.time_out = self.rew.data_ptr(), self.reset_u8.data_ptr(), self.timeout_u8.data_ptr()
        b.event_count, b.events, b.episode_acc = self.event_count.data_ptr(), self.events.data_ptr(), self.episode_acc.data_ptr()
        b.noise = self.noise.data_ptr() if self.noise is not None else None
        b.reset_rand = self.reset_rand.data_ptr() if self.reset_rand is not None else None
        b.episode_sums_eval = self.episode_sums_eval.data_ptr() if self.episode_sums_eval is not None else None
        b.gravity_dev, b.step_dev = self.gravity_dev.data_ptr(), self.step_dev.data_ptr()
        if self.num_priv and self._priv_store.shape[1] != self.num_priv:
            raise AssertionError
        capi.check(self.L.go1_sim_bind(self._handle, C.byref(b)), "go1_sim_bind")

    def sync_rigid_props(self):
        """The rigid bodies take their mass / centre of mass from `payloads` / `com_displacements` as they are NOW (Isaac Gym
        applies them once at actor creation, legged_robot.py:667-673); later re-draws only change the observed buffers."""
        self.env("rigid_payload").copy_(self.env("payloads"))
        self.env("rigid_com").copy_(self.env("com_displacements"))

    def enable_eval_sums(self):
        """LeggedRobot.episode_sums_eval (legged_robot.py:1420-1424): [NUM_EPISODE_SUMS][N], -1 = not yet recorded."""
        self.episode_sums_eval = torch.full((capi.NUM_EPISODE_SUMS, self.N), -1.0, device=self.device)
        self.episode_sums_eval[capi.NUM_REWARD_TERMS].zero_()     # "total" starts at 0 in the reference (:1423): never recorded
        self._bind()

    def close(self):
        if self._handle:
            self.L.go1_sim_destroy(self._handle)
            self._handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ views
    def env(self, name, width=None):
        """[width][N] view of a per-env field."""
        r = capi.row(0, name)
        w = width if width is not None else self._width(0, name)
        return self.env_f32[r:r + w]

    def leg(self, name, width=None):
        """[width][N][4] view of a per-leg field (leg order FL,FR,RL,RR)."""
        r = capi.row(1, name)
        w = width if width is not None else self._width(1, name)
        return self.leg_f32[r:r + w].view(w, self.N, 4)

    _WIDTHS = {}

    def _width(self, kind, name):
        key = (kind, name)
        if key not in self._WIDTHS:
            names = _FIELD_NAMES[kind]
            rows = sorted((capi.row(kind, n), n) for n in names)
            total = self.L.go1_sim_num_rows(kind)
            for i, (r, n) in enumerate(rows):
                nxt = rows[i + 1][0] if i + 1 < len(rows) else total
                self._WIDTHS[(kind, n)] = nxt - r
        return self._WIDTHS[key]

    def env_aos(self, name):
        """[N][width] writable transposed view (e.g. commands [N,15])."""
        return self.env(name).t()

    def joint_aos(self, name):
        """[N][12] copy in Isaac DOF order (FL hip,thigh,calf, FR ..., RL ..., RR ...)."""
        return self.leg(name).permute(1, 2, 0).reshape(self.N, 12)

    def set_joint_aos(self, name, value):
        self.leg(name).copy_(value.reshape(self.N, 4, 3).permute(2, 0, 1))

    def foot_aos(self, name):
        """[N][4][3] copy of a 3-vector-per-foot field."""
        return self.leg(name).permute(1, 2, 0).contiguous()

    def set_foot_aos(self, name, value):
        self.leg(name).copy_(value.reshape(self.N, 4, 3).permute(2, 0, 1))

    @property
    def episode_length_buf(self):
        return self.env_i32[0]

    # ------------------------------------------------------------------ calls
    def set_gravity(self, g, gvec):
        self.gravity[:] = [float(x) for x in g]
        self.gravity_vec[:] = [float(x) for x in gvec]
        self.gravity_dev.copy_(torch.tensor(list(self.gravity) + list(self.gravity_vec), dtype=torch.float32))    # stream-ordered; ~1 call / 400 steps

    def step(self, actions, common_step=0, mode=0):
        assert actions.is_cuda and actions.dtype == torch.float32 and actions.is_contiguous() and actions.shape == (self.N, 12)
        capi.check(self.L.go1_sim_step(self._handle, capi.ptr(actions), C.byref(self.gravity), C.byref(self.gravity_vec),
                                       int(common_step), int(mode), capi.stream_ptr()), "go1_sim_step")

    def step_deferred(self, actions, pre_roll, common_step=0):
        """step() for a step with user reward terms: the pre-roll last_* values go to `pre_roll` [PRE_ROLL_ROWS][4N], and rew /
        rew_buf_pos / rew_buf_neg hold the built-in terms only until reward_finish()."""
        assert actions.is_cuda and actions.dtype == torch.float32 and actions.is_contiguous() and actions.shape == (self.N, 12)
        assert pre_roll.shape == (capi.PRE_ROLL_ROWS, 4 * self.N) and pre_roll.is_contiguous()
        capi.check(self.L.go1_sim_step_deferred(self._handle, capi.ptr(actions), C.byref(self.gravity), C.byref(self.gravity_vec),
                                                int(common_step), capi.ptr(pre_roll), capi.stream_ptr()), "go1_sim_step_deferred")

    def reward_finish(self, raw, scales, user_sums, workspace):
        """The user terms' values raw [K][N] into rew / rew_buf_pos / rew_buf_neg / the episode sums (go1_sim_reward_finish).
        scales: ctypes float array of K."""
        capi.check(self.L.go1_sim_reward_finish(self._handle, capi.ptr(raw), scales, raw.shape[0], capi.ptr(user_sums), capi.ptr(workspace),
                                                capi.stream_ptr()), "go1_sim_reward_finish")

    def user_reward_fold(self, ids, k_dev, k, user_sums, user_sums_eval, acc, acc_hist=None, slot=None):
        """User episode sums of the reset envs `ids` (int32; count k or k_dev) -> acc [K+1] (+ acc_hist[slot]), then zeroed."""
        T = acc_hist.shape[0] if acc_hist is not None else 0
        capi.check(self.L.go1_sim_user_reward_fold(self._handle, capi.ptr(ids), capi.ptr(k_dev), int(k), user_sums.shape[0], capi.ptr(user_sums),
                                                   capi.ptr(user_sums_eval), capi.ptr(acc), capi.ptr(acc_hist), T, capi.ptr(slot),
                                                   capi.stream_ptr()), "go1_sim_user_reward_fold")

    EVENT_PREFIX = 48      # records per list copied speculatively together with the counters

    def fetch_events(self):
        """The synchronising D2H of the event lists written by the last step: counters + the first EVENT_PREFIX records of
        both lists in one sync; a second copy only when a list is longer.
        Returns (reset_ids, reset_sums[k,4], interval_ids, interval_sums[k,4]) sorted by env id."""
        P = min(self.EVENT_PREFIX, self.N)
        self.h_count.copy_(self.event_count, non_blocking=True)
        self.h_events[:, :P].copy_(self.events[:, :P], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self.d2h_bytes += 8 + 2 * P * capi.EVENT_STRIDE * 4
        out = []
        for lst in range(2):
            k = int(self.h_count[lst])
            if k == 0:
                out += [np.zeros(0, dtype=np.int64), np.zeros((0, 4), dtype=np.float32)]
                continue
            if k > P:
                self.h_events[lst, P:k].copy_(self.events[lst, P:k], non_blocking=True)
                torch.cuda.current_stream().synchronize()
                self.d2h_bytes += (k - P) * capi.EVENT_STRIDE * 4
            ev = self.h_events[lst, :k].numpy()
            ids = ev[:, 0].astype(np.int64)
            order = np.argsort(ids, kind="stable")
            out += [ids[order], ev[order, 1:5].copy()]
        return tuple(out)

    def _upload(self, slot, ids, cmds):
        """ids (int, ascending) + commands [k,15] float32 -> device staging of `slot`; returns (k, ids_ptr, cmds_ptr)."""
        k = len(ids)
        if k == 0:
            return 0, None, None
        if self._stage_used[slot] and not self._stage_event[slot].query():
            self._stage_event[slot].synchronize()
        n = k * capi.NUM_COMMANDS
        self._h_stage_i32[slot][:k] = ids
        self._h_stage_f32[slot][k:k + n] = np.asarray(cmds, dtype=np.float32).reshape(-1)
        self._d_stage[slot][:k + n].copy_(self._h_stage[slot][:k + n], non_blocking=True)
        self._stage_event[slot].record()
        self._stage_used[slot] = True
        self.h2d_bytes += 4 * (k + n)
        base = self._d_stage_ptr[slot]
        return k, C.c_void_p(base), C.c_void_p(base + 4 * k)

    def reset_idx(self, ids, new_commands, actions=None, post_step=False, common_step=0):
        k, pi, pc = self._upload(0, ids, new_commands)
        if k == 0:
            return
        capi.check(self.L.go1_sim_reset_idx(self._handle, pi, k, pc, capi.ptr(actions) if actions is not None else None,
                                            int(bool(post_step)), int(common_step), capi.stream_ptr()), "go1_sim_reset_idx")

    def set_commands(self, ids, new_commands):
        k, pi, pc = self._upload(1, ids, new_commands)
        if k == 0:
            return
        capi.check(self.L.go1_sim_set_commands(self._handle, pi, k, pc, capi.stream_ptr()), "go1_sim_set_commands")

    def update_config(self):
        capi.check(self.L.go1_sim_update_config(self._handle, C.byref(self.cfg), capi.stream_ptr()), "go1_sim_update_config")


_FIELD_NAMES = {
    0: ["root_pos", "root_quat", "root_lin_vel", "root_ang_vel", "commands", "gait_indices", "friction_coeffs", "restitutions",
        "payloads", "com_displacements", "motor_strengths", "Kp_factors", "Kd_factors", "env_origins", "rigid_payload", "rigid_com", "base_lin_vel",
        "base_ang_vel", "projected_gravity", "rew_buf_pos", "rew_buf_neg", "episode_sums", "command_sums"],
    1: ["dof_pos", "dof_vel", "last_dof_vel", "actions", "last_actions", "last_last_actions", "joint_pos_target",
        "last_joint_pos_target", "last_last_joint_pos_target", "lag_buffer", "joint_pos_err_last", "joint_pos_err_last_last",
        "joint_vel_last", "joint_vel_last_last", "motor_offsets", "torques", "clock_inputs", "doubletime_clock_inputs",
        "halftime_clock_inputs", "desired_contact_states", "foot_indices", "foot_positions", "foot_velocities",
        "prev_foot_velocities", "foot_contact_forces", "hip_contact_forces", "thigh_contact_forces", "calf_contact_forces",
        "base_contact_forces_part", "last_contacts"],
    2: ["episode_length_buf"],
}
