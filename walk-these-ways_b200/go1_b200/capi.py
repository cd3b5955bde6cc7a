"""ctypes binding of libgo1b200.so (include/go1_b200.h).

The product has no CPU fallback: importing this module works anywhere (so the build can be checked
on a CPU box), but every compute call goes through the CUDA library and raises Go1Error if the
library is missing or no CUDA device is present.
"""
import contextlib
import ctypes as C
import os

_PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(_PKG, "lib", "libgo1b200.so")

NUM_DOF = 12
NUM_COMMANDS = 15
MAX_OBS = 128
MAX_PRIV_OBS = 48
EVENT_STRIDE = 6
XR_STRIDE = 8

REWARD_TERMS = [
    "tracking_lin_vel", "tracking_ang_vel", "lin_vel_z", "ang_vel_xy", "orientation", "torques", "dof_acc",
    "action_rate", "collision", "dof_pos_limits", "jump", "tracking_contacts_shaped_force",
    "tracking_contacts_shaped_vel", "dof_pos", "dof_vel", "action_smoothness_1", "action_smoothness_2",
    "feet_slip", "feet_contact_vel", "feet_contact_forces", "feet_clearance_cmd_linear", "feet_impact_vel",
    "orientation_control", "raibert_heuristic", "termination",
]
NUM_REWARD_TERMS = len(REWARD_TERMS)
NUM_EPISODE_SUMS = NUM_REWARD_TERMS + 1
NUM_COMMAND_SUMS = NUM_REWARD_TERMS + 5
COMMAND_SUM_EXTRAS = ["lin_vel_raw", "ang_vel_raw", "lin_vel_residual", "ang_vel_residual", "ep_timesteps"]

def row_pitch(width):
    """Row pitch (floats) of a buffer whose rows are `width` floats wide and that a tensor-core product reads or writes through TMA, which
    needs row strides that are multiples of 16 bytes: widths that are multiples of 4 floats keep their natural pitch, the others are
    rounded up to a multiple of 32 floats (128-byte aligned rows).  Holders expose the width as a [:, :width] view."""
    width = int(width)
    return width if width % 4 == 0 else (width + 31) // 32 * 32


def history_pitch(width):
    """Row pitch (floats) of observation-history rows `width` = num_observations x num_observation_history wide, for every buffer that
    holds them (HistoryWrapper's ping-pong buffers, RolloutStorage's history slab).  TMA, through which the learner's tensor-core
    products read the histories, needs row strides that are multiples of 16 bytes: widths that are multiples of 4 floats keep their
    natural pitch, the others are rounded up to a multiple of 32 floats (128-byte aligned rows, as RolloutStorage.hist_pitch)."""
    return row_pitch(width)


def bf16_pitch(width):
    """Row pitch (elements) of a BF16 buffer that a tensor-core product reads or writes through TMA (AC_Args.gemm_impl = 2): row strides must
    be multiples of 16 bytes, 8 elements.  Widths that are multiples of 8 keep their natural pitch, the others are rounded up to a multiple
    of 64 elements (128-byte aligned rows, the width of one TMA box row).  Holders expose the width as a [:, :width] view."""
    width = int(width)
    return width if width % 8 == 0 else (width + 63) // 64 * 64


RESET_RAND_STRIDE = 48
MAX_LAG_TIMESTEPS = 32
MAX_USER_REWARDS = 32
PRE_ROLL_FIELDS = ["last_actions", "last_last_actions", "last_dof_vel", "last_joint_pos_target", "last_last_joint_pos_target"]   # 3 rows each
PRE_ROLL_ROWS = 3 * len(PRE_ROLL_FIELDS)
_i, _f = C.c_int32, C.c_float


class Go1DomainRand(C.Structure):
    _fields_ = [
        ("randomize_motor_strength", _i), ("randomize_motor_offset", _i), ("randomize_Kp_factor", _i), ("randomize_Kd_factor", _i),
        ("motor_strength_range", _f * 2), ("motor_offset_range", _f * 2), ("Kp_factor_range", _f * 2), ("Kd_factor_range", _f * 2),
        ("randomize_rigids_after_start", _i), ("randomize_base_mass", _i), ("randomize_com_displacement", _i),
        ("randomize_friction", _i), ("randomize_restitution", _i),
        ("added_mass_range", _f * 2), ("com_displacement_range", _f * 2), ("friction_range", _f * 2), ("restitution_range", _f * 2),
        ("push_robots", _i), ("push_interval", _i), ("max_push_vel_xy", _f),
        ("teleport_robots", _i),
        ("teleport_x_lo", _f), ("teleport_x_hi", _f), ("teleport_dx", _f), ("teleport_y_lo", _f), ("teleport_y_hi", _f), ("teleport_dy", _f),
        ("x_init_range", _f), ("y_init_range", _f), ("yaw_init_range", _f), ("x_init_offset", _f), ("y_init_offset", _f),
    ]


class Go1SimConfig(C.Structure):
    _fields_ = [
        ("num_envs", _i), ("num_train_envs", _i), ("sim_dt", _f), ("decimation", _i),
        ("clip_actions", _f), ("clip_obs", _f), ("control_type", _i),
        ("action_scale", _f), ("hip_scale_reduction", _f), ("kp", _f), ("kd", _f), ("use_lag", _i), ("lag_timesteps", _i),
        ("default_dof_pos", _f * NUM_DOF), ("soft_limit_lo", _f * NUM_DOF), ("soft_limit_hi", _f * NUM_DOF),
        ("torque_limit", _f),
        ("num_commands", _i), ("observe_gait_commands", _i), ("pacing_offset", _i), ("kappa_gait_probs", _f),
        ("observe_vel", _i), ("observe_only_ang_vel", _i), ("observe_only_lin_vel", _i), ("observe_command", _i),
        ("observe_two_prev_actions", _i), ("observe_timing_parameter", _i), ("observe_clock_inputs", _i),
        ("observe_yaw", _i), ("observe_contact_states", _i),
        ("num_obs", _i), ("num_priv_obs", _i), ("add_noise", _i),
        ("commands_scale", _f * NUM_COMMANDS),
        ("obs_scale_lin_vel", _f), ("obs_scale_ang_vel", _f), ("obs_scale_dof_pos", _f), ("obs_scale_dof_vel", _f),
        ("noise_scale_vec", _f * MAX_OBS),
        ("priv_friction", _i), ("priv_restitution", _i), ("priv_base_mass", _i), ("priv_com_displacement", _i),
        ("priv_motor_strength", _i), ("priv_motor_offset", _i), ("priv_body_height", _i), ("priv_body_velocity", _i),
        ("priv_gravity", _i), ("priv_clock_inputs", _i), ("priv_desired_contact_states", _i),
        ("friction_ss", _f * 2), ("restitution_ss", _f * 2), ("mass_ss", _f * 2), ("com_ss", _f * 2),
        ("motor_strength_ss", _f * 2), ("motor_offset_ss", _f * 2), ("body_height_ss", _f * 2),
        ("body_velocity_ss", _f * 2), ("gravity_ss", _f * 2),
        ("reward_scale", _f * NUM_REWARD_TERMS), ("reward_order", _i * NUM_REWARD_TERMS),
        ("num_active_rewards", _i), ("only_positive_rewards", _i), ("only_positive_rewards_ji22_style", _i),
        ("sigma_rew_neg", _f), ("tracking_sigma", _f), ("tracking_sigma_yaw", _f), ("gait_force_sigma", _f),
        ("gait_vel_sigma", _f), ("base_height_target", _f), ("max_contact_force", _f),
        ("use_terminal_body_height", _i), ("max_episode_length", _i), ("terminal_body_height", _f),
        ("dr", Go1DomainRand * 2), ("rand_interval", _i), ("resampling_interval", _i),
        ("base_init_state", _f * 13),
        ("custom_origins", _i),
        ("erp", _f), ("cfm", _f), ("max_depen_vel", _f), ("contact_margin", _f), ("bounce_threshold", _f),
        ("pgs_iters", _i), ("terrain_friction", _f), ("terrain_restitution", _f),
        ("pen_k", _f * 4), ("pen_c", _f * 4), ("pen_mt", _f), ("limit_k", _f), ("limit_c", _f),
        ("hf", C.c_void_p), ("hf_rows", _i), ("hf_cols", _i), ("hf_hscale", _f), ("hf_vscale", _f), ("hf_border", _f),
        ("measure_heights", _i), ("num_height_points_x", _i), ("num_height_points_y", _i),
        ("height_points_x", _f * 32), ("height_points_y", _f * 32),
        ("seed", C.c_uint64),
    ]


class Go1SimBuffers(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "env_f32", "leg_f32", "env_i32", "obs", "priv_obs", "rew", "reset", "time_out", "event_count", "events",
        "episode_acc", "noise", "reset_rand", "gravity_dev", "step_dev", "episode_sums_eval")]


class Go1SelfCollision(C.Structure):
    """Self-collision model of a sim (go1_sim_set_self_collision); enabled = 0 keeps the default step kernel."""
    _fields_ = [("enabled", _i), ("k", _f), ("c", _f), ("thigh_radius", _f), ("calf_radius", _f), ("foot_radius", _f)]


NUM_BODIES = 17


class Go1AssetOptions(C.Structure):
    """Asset options of a sim (go1_sim_set_asset_options): per-body collision-penalty weights and termination bits in Isaac Gym body
    order (config.BODY_NAMES), a welded base, the gravity switch and the joint armature."""
    _fields_ = [("penalty_weight", _f * NUM_BODIES), ("termination_mask", C.c_uint32), ("fix_base", _i), ("disable_gravity", _i),
                ("armature", _f)]


CUR_MAX_CATEGORIES = 8


class Go1CurriculumConfig(C.Structure):
    _fields_ = [("num_categories", _i), ("category_kind", _i * CUR_MAX_CATEGORIES), ("num_bins", _i), ("num_dims", _i), ("num_commands", _i),
                ("num_task_keys", _i), ("task_col", _i * 4), ("threshold", _f * 4), ("ep_len", _f),
                ("gaitwise_curricula", _i), ("exclusive_phase_offset", _i), ("balance_gait_distribution", _i), ("binary_phases", _i),
                ("num_train_envs", _i), ("snapshot_time_outs", _i), ("xr_world", _i), ("xr_rank", _i), ("xr_cap", _i)]


class Go1CurriculumBuffers(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "weights", "grid", "half_bins", "local_range", "mt", "cat_rng", "env_bins", "env_categories", "env_bins_f32", "time_outs_snapshot",
        "cdf", "cdf_valid", "scratch_i32", "scratch_u32", "scratch_f64", "out_count", "out_ids", "out_commands",
        "xr_send", "xr_events", "xr_ids", "xr_commands")]


# enum Go1Activation (include/go1_b200.h), keyed by the names AC_Args.activation accepts (the reference maps crelu to nn.ReLU too)
ACTIVATIONS = {"elu": 0, "selu": 1, "relu": 2, "crelu": 2, "lrelu": 3, "tanh": 4, "sigmoid": 5}


def act_arg(kind, mode):
    """GO1_ACT(kind, mode): the `act` argument of the entry points that take a bare int."""
    return (kind << 8) | mode


class Go1GemmEpilogue(C.Structure):
    _fields_ = [("bias", C.c_void_p), ("act", _i), ("accumulate", _i), ("extra", C.c_void_p), ("ld_extra", _i), ("w_extra", C.c_void_p),
                ("ld_w_extra", _i), ("num_extra", _i), ("dact_y", C.c_void_p), ("ld_dact_y", _i), ("lead_cols", _i), ("colsum", C.c_void_p),
                ("bwd_extra", C.c_void_p), ("bwd_w_extra", C.c_void_p), ("g_w_extra", C.c_void_p), ("d_extra", C.c_void_p),
                ("ld_bwd_extra", _i), ("ld_bwd_w_extra", _i), ("ld_g_w_extra", _i), ("ld_d_extra", _i), ("num_bwd_extra", _i), ("act_kind", _i),
                ("store_transposed", _i), ("out_bf16", C.c_void_p), ("ld_out_bf16", _i)]


class Go1TailProblem(C.Structure):
    _fields_ = [("x", C.c_void_p), ("ldx", _i), ("W2", C.c_void_p), ("b2", C.c_void_p), ("y2", C.c_void_p), ("ldy2", _i),
                ("W3", C.c_void_p), ("b3", C.c_void_p), ("y3", C.c_void_p), ("ldy3", _i), ("Wh", C.c_void_p), ("bh", C.c_void_p), ("nh", _i),
                ("out", C.c_void_p), ("ldout", _i), ("act_kind", _i), ("ldw2", _i), ("ldw3", _i)]


class Go1CopySeg(C.Structure):
    _fields_ = [("src", C.c_void_p), ("lds", _i), ("dst", C.c_void_p), ("ldd", _i), ("rows", _i), ("cols", _i)]


def copy_segments(pairs):
    """dst.copy_(src) for up to 8 (dst, src) pairs of 2-D float32 CUDA tensors (unit inner stride) in ONE launch (go1_copy_segments)."""
    n = len(pairs)
    arr = (Go1CopySeg * n)()
    for sg, (dst, src) in zip(arr, pairs):
        assert dst.shape == src.shape and dst.dim() == 2 and dst.stride(1) == 1 and src.stride(1) == 1
        sg.src, sg.lds, sg.dst, sg.ldd, sg.rows, sg.cols = src.data_ptr(), src.stride(0), dst.data_ptr(), dst.stride(0), dst.shape[0], dst.shape[1]
    check(lib().go1_copy_segments(arr, n, stream_ptr()), "go1_copy_segments")


class Go1Bf16Seg(C.Structure):
    _fields_ = [("src", C.c_void_p), ("lds", _i), ("dst", C.c_void_p), ("ldd", _i), ("rows", _i), ("cols", _i)]


def convert_bf16_segments(pairs):
    """dst.copy_(src.to(torch.bfloat16)) for (dst, src) pairs -- BF16 dst, float32 src, 2-D CUDA tensors with unit inner stride -- in one
    go1_convert_bf16_segments launch per 16 pairs."""
    for k0 in range(0, len(pairs), 16):
        chunk = pairs[k0:k0 + 16]
        arr = (Go1Bf16Seg * len(chunk))()
        for sg, (dst, src) in zip(arr, chunk):
            assert dst.shape == src.shape and dst.dim() == 2 and dst.stride(1) == 1 and src.stride(1) == 1
            sg.src, sg.lds, sg.dst, sg.ldd, sg.rows, sg.cols = src.data_ptr(), src.stride(0), dst.data_ptr(), dst.stride(0), dst.shape[0], dst.shape[1]
        check(lib().go1_convert_bf16_segments(arr, len(chunk), stream_ptr()), "go1_convert_bf16_segments")


class Go1Error(RuntimeError):
    pass


_lib = None


def lib():
    """Load libgo1b200.so (built by __graft_entry__.build() / csrc/Makefile). Fails loudly if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise Go1Error(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                       f"(nvcc, sm_90a). There is no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    L.go1_last_error.restype = C.c_char_p
    vp, ip, i64 = C.c_void_p, C.c_int, C.c_int64
    sig = {
        "go1_version": ([], ip), "go1_device_count": ([], ip), "go1_sizeof_config": ([], ip), "go1_sizeof_buffers": ([], ip),
        "go1_kernel_launch_count": ([], C.c_longlong), "go1_kernel_launch_add": ([C.c_longlong], None),
        "go1_gemm_timing": ([ip, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_longlong)], ip),
        "go1_sim_num_rows": ([ip], ip), "go1_sim_row": ([ip, C.c_char_p], ip),
        "go1_sim_create": ([C.POINTER(Go1SimConfig), vp, ip, C.POINTER(vp)], ip),
        "go1_sim_destroy": ([vp], ip), "go1_sim_bind": ([vp, C.POINTER(Go1SimBuffers)], ip),
        "go1_sim_update_config": ([vp, C.POINTER(Go1SimConfig), vp], ip),
        "go1_sim_step": ([vp, vp, C.POINTER(_f * 3), C.POINTER(_f * 3), i64, ip, vp], ip),
        "go1_sim_reset_idx": ([vp, vp, ip, vp, vp, ip, i64, vp], ip),
        "go1_sim_step_deferred": ([vp, vp, C.POINTER(_f * 3), C.POINTER(_f * 3), i64, vp, vp], ip),
        "go1_reward_finish_workspace": ([ip, ip], i64),
        "go1_sim_reward_finish": ([vp, vp, vp, ip, vp, vp, vp], ip),
        "go1_sim_user_reward_fold": ([vp, vp, vp, ip, ip, vp, vp, vp, vp, ip, vp, vp], ip),
        "go1_sim_set_commands": ([vp, vp, ip, vp, vp], ip),
        "go1_sim_set_step_block": ([ip], None),
        "go1_sizeof_self_collision": ([], ip), "go1_sim_set_self_collision": ([vp, C.POINTER(Go1SelfCollision)], ip),
        "go1_sizeof_asset_options": ([], ip), "go1_sim_set_asset_options": ([vp, C.POINTER(Go1AssetOptions)], ip),
        "go1_sizeof_curriculum": ([ip], ip), "go1_curriculum_set_grouped": ([ip], None),
        "go1_set_deterministic": ([ip], None), "go1_deterministic": ([], ip), "go1_deterministic_workspace_bytes": ([], i64),
        "go1_deterministic_reserve": ([vp], ip),
        "go1_curriculum_resample": ([vp, C.POINTER(Go1CurriculumConfig), C.POINTER(Go1CurriculumBuffers), ip, vp], ip),
        "go1_curriculum_pack": ([vp, C.POINTER(Go1CurriculumConfig), C.POINTER(Go1CurriculumBuffers), vp], ip),
        "go1_sim_reset_idx_dev": ([vp, vp, vp, vp, vp, ip, i64, vp, vp], ip),
        "go1_history_roll": ([vp, vp, vp, ip, ip, ip, vp], ip),
        "go1_history_roll_pitched": ([vp, ip, vp, vp, ip, ip, ip, ip, vp], ip),
        "go1_ppo_gae": ([vp, vp, vp, vp, vp, vp, vp, ip, ip, _f, _f, vp], ip),
        "go1_ppo_normalize_advantages": ([vp, vp, i64, i64, vp], ip),
        "go1_gemm": ([ip, ip, ip, ip, ip, vp, ip, vp, ip, vp, ip, vp, ip, ip, ip, vp], ip),
        "go1_gemm_ex": ([ip, ip, ip, ip, ip, vp, ip, vp, ip, vp, ip, C.POINTER(Go1GemmEpilogue), ip, vp], ip),
        "go1_mlp_tail_forward_grouped": ([C.POINTER(Go1TailProblem), ip, ip, ip, ip, ip, vp], ip),
        "go1_mlp_tail_forward": ([vp, ip, ip, ip, vp, vp, ip, vp, ip, vp, vp, ip, vp, ip, vp, vp, ip, vp, ip, vp], ip),
        "go1_transpose": ([vp, ip, vp, ip, ip, ip, vp], ip),
        "go1_elu_backward": ([vp, ip, vp, ip, vp, ip, ip, ip, vp], ip),
        "go1_act_backward": ([vp, ip, vp, ip, vp, ip, ip, ip, ip, vp], ip),
        "go1_mlp_extra_forward": ([vp, ip, vp, ip, vp, ip, ip, ip, ip, ip, vp], ip),
        "go1_mlp_extra_backward": ([vp, ip, ip, vp, ip, vp, ip, vp, ip, vp, ip, ip, ip, ip, ip, vp], ip),
        "go1_skinny_dgrad": ([vp, ip, vp, ip, vp, ip, vp, ip, ip, ip, ip, vp], ip),
        "go1_skinny_dgrad_ex": ([vp, ip, vp, ip, vp, ip, vp, ip, vp, ip, ip, ip, vp], ip),
        "go1_skinny_dgrad_act": ([vp, ip, vp, ip, vp, ip, vp, ip, vp, ip, ip, ip, ip, vp], ip),
        "go1_skinny_wgrad_ex": ([vp, ip, vp, ip, vp, ip, vp, ip, ip, ip, ip, vp], ip),
        "go1_gemm_bf16_ex": ([ip, ip, ip, ip, ip, vp, ip, vp, ip, vp, ip, C.POINTER(Go1GemmEpilogue), vp], ip),
        "go1_convert_bf16": ([vp, ip, vp, ip, ip, ip, vp], ip),
        "go1_gather_rows_bf16": ([vp, ip, vp, vp, ip, i64, ip, vp], ip),
        "go1_rollout_store_rows_bf16": ([vp, ip, vp, ip, vp, ip, ip, vp], ip),
        "go1_transpose_to_bf16": ([vp, ip, vp, ip, ip, ip, vp], ip),
        "go1_transpose_bf16": ([vp, ip, vp, ip, ip, ip, vp], ip),
        "go1_gemm_grouped": ([ip, ip, ip, ip, ip, ip, C.POINTER(vp), ip, C.POINTER(vp), ip, C.POINTER(vp), ip, ip, vp], ip),
        "go1_gemm_bf16_mn": ([ip, ip, ip, ip, ip, vp, ip, vp, ip, vp, ip, ip, C.POINTER(Go1GemmEpilogue), vp], ip),
        "go1_gemm_bf16_grouped": ([ip, ip, ip, ip, ip, ip, C.POINTER(vp), ip, C.POINTER(vp), ip, C.POINTER(vp), ip, ip, vp], ip),
        "go1_convert_bf16_segments": ([C.POINTER(Go1Bf16Seg), ip, vp], ip),
        "go1_skinny_dgrad_act_bf16": ([vp, ip, vp, ip, vp, ip, vp, ip, vp, ip, ip, ip, ip, vp], ip),
        "go1_copy_segments": ([C.POINTER(Go1CopySeg), ip, vp], ip),
        "go1_skinny_forward": ([vp, ip, vp, ip, vp, vp, ip, ip, ip, ip, vp], ip),
        "go1_skinny_wgrad": ([vp, ip, vp, ip, vp, ip, ip, ip, ip, ip, vp], ip),
        "go1_colsum": ([vp, ip, vp, ip, ip, ip, vp], ip),
        "go1_ppo_sample_actions": ([vp, ip, vp, vp, C.c_uint64, C.c_uint64, vp, vp, vp, ip, ip, vp], ip),
        "go1_ppo_loss": ([vp, ip, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, ip, vp, vp, vp, ip, ip, _f, _f, _f, ip, _f, vp], ip),
        "go1_ppo_mse": ([vp, ip, vp, ip, vp, ip, vp, ip, ip, ip, vp], ip),
        "go1_ppo_grad_sqnorm": ([vp, i64, vp, vp], ip),
        "go1_ppo_adam_step": ([vp, vp, vp, vp, i64, vp, _f, _f, vp, _f, _f, _f, ip, vp], ip),
        "go1_ppo_adaptive_lr": ([vp, vp, _f, _f, _f, vp], ip),
        "go1_store_transition": ([vp, vp, vp, vp, vp, ip, ip, ip, ip, ip, _f, vp], ip),
        "go1_store_observations": ([vp, vp, vp, vp, ip, ip, ip, vp], ip),
        "go1_rollout_store_observations": ([vp, vp, vp, vp, vp, ip, ip, ip, vp], ip),
        "go1_rollout_store_transition": ([vp, vp, vp, vp, vp, vp, ip, ip, ip, ip, ip, _f, vp], ip),
        "go1_rollout_advance": ([vp, vp, ip, ip, vp, vp, vp], ip),
        "go1_gather_rows": ([vp, vp, vp, i64, ip, ip, vp], ip),
    }
    for name, (args, res) in sig.items():
        fn = getattr(L, name)          # AttributeError here = header/library mismatch: fail loudly
        fn.argtypes = args
        fn.restype = res
    if L.go1_sizeof_config() != C.sizeof(Go1SimConfig):
        raise Go1Error(f"Go1SimConfig mirror out of date: C {L.go1_sizeof_config()} vs ctypes {C.sizeof(Go1SimConfig)}")
    if L.go1_sizeof_buffers() != C.sizeof(Go1SimBuffers):
        raise Go1Error("Go1SimBuffers mirror out of date")
    if L.go1_sizeof_self_collision() != C.sizeof(Go1SelfCollision):
        raise Go1Error("Go1SelfCollision mirror out of date")
    if L.go1_sizeof_asset_options() != C.sizeof(Go1AssetOptions):
        raise Go1Error("Go1AssetOptions mirror out of date")
    if L.go1_sizeof_curriculum(0) != C.sizeof(Go1CurriculumConfig) or L.go1_sizeof_curriculum(1) != C.sizeof(Go1CurriculumBuffers):
        raise Go1Error("Go1Curriculum* mirrors out of date")
    _lib = L
    return L


@contextlib.contextmanager
def deterministic(on):
    """The library's deterministic mode (go1_set_deterministic) set to `on` for the launches inside the block and restored afterwards.  Nothing
    is called when the library is already in that mode, nor to keep the default mode before the library has been loaded."""
    on = 1 if on else 0
    if _lib is None and not on:
        yield
        return
    L = lib()
    prev = L.go1_deterministic()
    if prev == on:
        yield
        return
    L.go1_set_deterministic(on)
    try:
        yield
    finally:
        L.go1_set_deterministic(prev)


def check(rc, what=""):
    if rc != 0:
        raise Go1Error(f"{what} failed ({rc}): {lib().go1_last_error().decode()}")


def exported_symbols():
    """Names every entry point include/go1_b200.h declares (used by the CPU-side ABI test)."""
    import re
    hdr = os.path.join(os.path.dirname(_PKG), "include", "go1_b200.h")
    txt = open(hdr).read()
    return sorted(set(re.findall(r"\b(go1_[a-z0-9_]+)\s*\(", txt)))


def row(kind, name):
    r = lib().go1_sim_row(kind, name.encode())
    if r < 0:
        raise KeyError(name)
    return r


def ptr(t):
    """Raw device pointer of a torch tensor (or None)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr():
    """cudaStream_t of torch's CURRENT stream on the current device (raw C query: ~1 us, honours torch.cuda.stream())."""
    import torch
    return C.c_void_p(torch._C._cuda_getCurrentRawStream(torch._C._cuda_getDevice()))
