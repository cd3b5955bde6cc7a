/*
 * go1_b200.h — C-ABI of libgo1b200.so: the H100-native (sm_90a) replacement for the hot path of
 * Improbable-AI/walk-these-ways (LeggedRobot.step() + the ppo_cse learner).
 *
 * Conventions (SURVEY.md §8b):
 *   - plain pointers and sizes only; every device buffer is allocated and owned by the caller
 *     (torch on the Python side), the library only borrows pointers;
 *   - every call returns 0 on success, non-zero on failure; the message is in go1_last_error();
 *   - calls are stream-ordered on the cudaStream_t passed as `void* stream` and never synchronise
 *     the device themselves (except go1_sim_create / *_destroy);
 *   - no CPU fallback: without a CUDA device every compute entry point fails with an error.
 *
 * Each entry point cites the reference interface it replaces (paths relative to the reference root).
 */
#ifndef GO1_B200_H
#define GO1_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define GO1_NUM_DOF 12
#define GO1_NUM_COMMANDS 15
#define GO1_MAX_OBS 128
#define GO1_MAX_PRIV_OBS 48
#define GO1_EVENT_STRIDE 6        /* floats per event record */
#define GO1_RESET_RAND_STRIDE 48  /* injected uniform draws per env (Go1SimBuffers.reset_rand) */
#define GO1_MAX_LAG_TIMESTEPS 32  /* action FIFO slots reserved per leg in leg_f32 (3 rows each, "lag_buffer") */
#define GO1_MAX_USER_REWARDS 32   /* user reward terms (go1_gym/envs/rewards) per go1_sim_reward_finish call */
/* rows of the pre-roll slab of go1_sim_step_deferred: [GO1_PRE_ROLL_ROWS][4N] in leg_f32 layout, 3 rows (joints) per field */
enum Go1PreRollRow {
    GO1_PRE_ROLL_LAST_ACTIONS = 0, GO1_PRE_ROLL_LAST_LAST_ACTIONS = 3, GO1_PRE_ROLL_LAST_DOF_VEL = 6,
    GO1_PRE_ROLL_LAST_JOINT_POS_TARGET = 9, GO1_PRE_ROLL_LAST_LAST_JOINT_POS_TARGET = 12, GO1_PRE_ROLL_ROWS = 15
};

/* reward term ids: one per CoRLRewards._reward_<name> (go1_gym/envs/rewards/corl_rewards.py:15-201) */
enum Go1RewardTerm {
    GO1_REW_TRACKING_LIN_VEL = 0, GO1_REW_TRACKING_ANG_VEL, GO1_REW_LIN_VEL_Z, GO1_REW_ANG_VEL_XY,
    GO1_REW_ORIENTATION, GO1_REW_TORQUES, GO1_REW_DOF_ACC, GO1_REW_ACTION_RATE, GO1_REW_COLLISION,
    GO1_REW_DOF_POS_LIMITS, GO1_REW_JUMP, GO1_REW_TRACKING_CONTACTS_SHAPED_FORCE,
    GO1_REW_TRACKING_CONTACTS_SHAPED_VEL, GO1_REW_DOF_POS, GO1_REW_DOF_VEL, GO1_REW_ACTION_SMOOTHNESS_1,
    GO1_REW_ACTION_SMOOTHNESS_2, GO1_REW_FEET_SLIP, GO1_REW_FEET_CONTACT_VEL, GO1_REW_FEET_CONTACT_FORCES,
    GO1_REW_FEET_CLEARANCE_CMD_LINEAR, GO1_REW_FEET_IMPACT_VEL, GO1_REW_ORIENTATION_CONTROL,
    GO1_REW_RAIBERT_HEURISTIC, GO1_REW_TERMINATION, GO1_NUM_REWARD_TERMS
};

/* The part of Cfg that LeggedRobot._call_train_eval (legged_robot.py:531-544) switches between `cfg` (envs
 * < num_train_envs) and `eval_cfg` (the rest): per-episode / periodic domain randomisation (:611-665), reset ranges
 * (:965-1001), pushes (:1017-1026) and edge teleports (:1028-1051). */
typedef struct Go1DomainRand {
    int32_t randomize_motor_strength, randomize_motor_offset, randomize_Kp_factor, randomize_Kd_factor;
    float motor_strength_range[2], motor_offset_range[2], Kp_factor_range[2], Kd_factor_range[2];
    /* _randomize_rigid_body_props again at reset / every rand_interval steps (legged_robot.py:164-166, 706-708) */
    int32_t randomize_rigids_after_start, randomize_base_mass, randomize_com_displacement, randomize_friction, randomize_restitution;
    float added_mass_range[2], com_displacement_range[2], friction_range[2], restitution_range[2];
    /* _push_robots: every push_interval steps the base xy velocity is redrawn in [-max_push_vel_xy, max_push_vel_xy] */
    int32_t push_robots, push_interval;
    float max_push_vel_xy;
    /* _teleport_robots: x < x_lo -> x += dx; then x > x_hi -> x -= dx; same for y (thresholds as float32, like the tensor compare) */
    int32_t teleport_robots;
    float teleport_x_lo, teleport_x_hi, teleport_dx, teleport_y_lo, teleport_y_hi, teleport_dy;
    /* _reset_root_states */
    float x_init_range, y_init_range, yaw_init_range, x_init_offset, y_init_offset;
} Go1DomainRand;

/* Resolved configuration of the env hot path.  Field-by-field mirror of what LeggedRobot reads from
 * Cfg (go1_gym/envs/base/legged_robot_config.py) after _parse_cfg (legged_robot.py:1716-1732). */
typedef struct Go1SimConfig {
    int32_t num_envs, num_train_envs;
    float sim_dt;                       /* Cfg.sim.dt (0.005) */
    int32_t decimation;                 /* Cfg.control.decimation (4) */
    float clip_actions, clip_obs;       /* Cfg.normalization */
    int32_t control_type;               /* 0 = actuator_net, 1 = P   (legged_robot.py:928-943) */
    float action_scale, hip_scale_reduction, kp, kd;
    int32_t use_lag;                    /* Cfg.domain_rand.randomize_lag_timesteps */
    int32_t lag_timesteps;              /* Cfg.domain_rand.lag_timesteps: depth L of the action FIFO in physics substeps,
                                         * 0..GO1_MAX_LAG_TIMESTEPS (legged_robot.py:922-924); ignored when use_lag = 0 */
    float default_dof_pos[GO1_NUM_DOF];
    float soft_limit_lo[GO1_NUM_DOF], soft_limit_hi[GO1_NUM_DOF];   /* legged_robot.py:603-607 */
    float torque_limit;
    /* gait clock (legged_robot.py:826-905) */
    int32_t num_commands, observe_gait_commands, pacing_offset;
    float kappa_gait_probs;
    /* observations (legged_robot.py:302-376) */
    int32_t observe_vel, observe_only_ang_vel, observe_only_lin_vel, observe_command, observe_two_prev_actions,
            observe_timing_parameter, observe_clock_inputs, observe_yaw, observe_contact_states;
    int32_t num_obs, num_priv_obs, add_noise;
    float commands_scale[GO1_NUM_COMMANDS];
    float obs_scale_lin_vel, obs_scale_ang_vel, obs_scale_dof_pos, obs_scale_dof_vel;
    float noise_scale_vec[GO1_MAX_OBS]; /* legged_robot.py:1053-1120 */
    /* privileged observations (legged_robot.py:378-491); scale/shift from get_scale_shift */
    int32_t priv_friction, priv_restitution, priv_base_mass, priv_com_displacement, priv_motor_strength,
            priv_motor_offset, priv_body_height, priv_body_velocity, priv_gravity, priv_clock_inputs,
            priv_desired_contact_states;
    float friction_ss[2], restitution_ss[2], mass_ss[2], com_ss[2], motor_strength_ss[2], motor_offset_ss[2],
          body_height_ss[2], body_velocity_ss[2], gravity_ss[2];
    /* rewards (legged_robot.py:263-300, 1385-1429) */
    float reward_scale[GO1_NUM_REWARD_TERMS];   /* already multiplied by dt; 0 = inactive */
    int32_t reward_order[GO1_NUM_REWARD_TERMS]; /* active term ids in the reference's iteration order */
    int32_t num_active_rewards, only_positive_rewards, only_positive_rewards_ji22_style;
    float sigma_rew_neg, tracking_sigma, tracking_sigma_yaw, gait_force_sigma, gait_vel_sigma,
          base_height_target, max_contact_force;
    /* termination (legged_robot.py:138-148) */
    int32_t use_terminal_body_height, max_episode_length;
    float terminal_body_height;
    /* domain randomisation: dr[0] for train envs, dr[1] for eval envs (= dr[0] without an eval_cfg); the interval of the
     * periodic re-randomisation is the TRAIN cfg's for all envs (legged_robot.py:697-699); command resampling interval (:684-686) */
    Go1DomainRand dr[2];
    int32_t rand_interval, resampling_interval;
    /* reset (legged_robot.py:948-1001) */
    float base_init_state[13];
    int32_t custom_origins;
    /* rigid-body solver (our algorithm, DESIGN.md §3; PhysX parameters legged_robot_config.py:402-421) */
    float erp, cfm, max_depen_vel, contact_margin, bounce_threshold;
    int32_t pgs_iters;
    float terrain_friction, terrain_restitution;
    float pen_k[4], pen_c[4], pen_mt, limit_k, limit_c;
    /* heightfield terrain (NULL/0 = flat): int16 samples [rows][cols] in device memory */
    const int16_t* hf; int32_t hf_rows, hf_cols; float hf_hscale, hf_vscale, hf_border;
    /* measured terrain heights under the base (legged_robot.py:689-691, 1772-1806): a num_x x num_y grid of points in the
     * yaw frame; only the body-height termination consumes them (legged_robot.py:146) */
    int32_t measure_heights, num_height_points_x, num_height_points_y;
    float height_points_x[32], height_points_y[32];
    uint64_t seed;                      /* Philox key for device-side randomisation */
} Go1SimConfig;

/* Device buffers borrowed from the caller.  State is SoA: row-major [rows][num_envs] for per-env rows
 * and [rows][4*num_envs] (index env*4+leg, legs FL,FR,RL,RR) for per-leg rows; row indices are
 * queried by name with go1_sim_row().  obs/priv_obs are the reference's AoS outputs. */
typedef struct Go1SimBuffers {
    float* env_f32;      /* [go1_sim_num_rows(0)][N]  */
    float* leg_f32;      /* [go1_sim_num_rows(1)][4N] */
    int32_t* env_i32;    /* [go1_sim_num_rows(2)][N]  */
    float* obs;          /* [N][num_obs]       LeggedRobot.obs_buf */
    float* priv_obs;     /* [N][num_priv_obs]  LeggedRobot.privileged_obs_buf */
    float* rew;          /* [N]                LeggedRobot.rew_buf */
    uint8_t* reset;      /* [N]                LeggedRobot.reset_buf (bool after check_termination) */
    uint8_t* time_out;   /* [N]                LeggedRobot.time_out_buf */
    int32_t* event_count;/* [2]  number of records in `events` (reset envs, interval-resample envs) */
    float* events;       /* [2][N][GO1_EVENT_STRIDE]: env id + 4 curriculum command_sums + ep_len */
    float* episode_acc;  /* [GO1_NUM_REWARD_TERMS+2] sum of episode_sums over envs reset this step, + count */
    const float* noise;  /* optional [N][num_obs] uniform(0,1) draws injected for parity tests, or NULL */
    const float* reset_rand; /* optional [N][GO1_RESET_RAND_STRIDE] uniform(0,1) draws injected for reset/DR/push parity tests, or NULL.
                              * slots: 0-11 dof pos, 12-14 x y yaw, 15-20 base twist, 21 motor strength, 22 Kp, 23 Kd, 24-35 motor offsets,
                              * 36-37 push xy, 38 payload, 39-41 com displacement, 42 friction, 43 restitution */
    const float* gravity_dev;/* optional [6] in device memory: gravity[3], gravity_vec[3].  When set, go1_sim_step / go1_sim_reset_idx* read
                              * gravity from here instead of their host arguments, so a captured CUDA graph of the env step sees later
                              * _randomize_gravity calls (legged_robot.py:546-561) */
    const int64_t* step_dev; /* optional [1] in device memory: added to the `common_step` argument (device-side common_step_counter of a
                              * graph-replayed rollout, advanced by go1_rollout_advance) */
    float* episode_sums_eval;/* optional [GO1_NUM_REWARD_TERMS+1][N], -1 = unset: LeggedRobot.episode_sums_eval (legged_robot.py:188-195), or NULL */
} Go1SimBuffers;

typedef struct Go1Sim Go1Sim;

const char* go1_last_error(void);
int go1_version(void);
int go1_device_count(void);
/* sizeof(Go1SimConfig) / sizeof(Go1SimBuffers) as compiled, so FFI bindings can verify their struct mirrors */
int go1_sizeof_config(void);
int go1_sizeof_buffers(void);
/* number of CUDA kernels this library has launched in this process (bench.py reports it as gpu_launches) */
long long go1_kernel_launch_count(void);

/* Layout queries: kind 0 = env_f32, 1 = leg_f32, 2 = env_i32. go1_sim_row returns the first row of the
 * named field or -1. */
int go1_sim_num_rows(int kind);
int go1_sim_row(int kind, const char* name);

/* Replaces BaseTask.__init__/create_sim/_init_buffers (base_task.py:16-86, legged_robot.py:1123-1258):
 * uploads the model/actuator/config table.  actuator_weights: 1313 floats
 * (W1[32x6] b1[32] W2[32x32] b2[32] W3[32] b3[1]) of resources/actuator_nets/unitree_go1.pt. */
int go1_sim_create(const Go1SimConfig* cfg, const float* actuator_weights, int device, Go1Sim** out);
int go1_sim_destroy(Go1Sim* sim);
int go1_sim_bind(Go1Sim* sim, const Go1SimBuffers* bufs);
/* Re-upload a changed config (e.g. reward scales after Cfg mutation) */
int go1_sim_update_config(Go1Sim* sim, const Go1SimConfig* cfg, void* stream);

/* Replaces LeggedRobot.step + post_physics_step for all envs that do not reset this step
 * (legged_robot.py:60-136): clip actions, 4x{_compute_torques -> rigid-body substep}, base-frame
 * quantities, _step_contact_targets, check_termination, compute_reward, compute_observations, history
 * of last_* buffers; envs that terminate are recorded in `events[0]`, envs due for the periodic
 * command resample next step in `events[1]`.  gravity = Cfg gravity + randomised offset
 * (legged_robot.py:546-561); gravity_vec = normalised gravity used for projected_gravity.
 * mode: 0 = full step; 1 = torques only (test hook for _compute_torques: one substep of control,
 * no dynamics); 2 = post-physics only (test hook: physics outputs already in the buffers). */
int go1_sim_step(Go1Sim* sim, const float* actions /*[N][12]*/, const float gravity[3],
                 const float gravity_vec[3], int64_t common_step, int mode, void* stream);

/* ---- user reward terms (go1_gym/envs/rewards, DESIGN.md §4) ------------------------------------------------------------
 * A step with K > 0 user terms is three launches instead of one: go1_sim_step_deferred, the user terms (torch, writing
 * raw[K][N]), go1_sim_reward_finish.  The reset launches follow as usual, then go1_sim_user_reward_fold.
 *
 * go1_sim_step_deferred: go1_sim_step (mode 0) with two differences.  It also writes the values that last_actions,
 * last_last_actions, last_dof_vel, last_joint_pos_target and last_last_joint_pos_target had before this step's rolls
 * (legged_robot.py:126-131) to `pre_roll` ([GO1_PRE_ROLL_ROWS][4N]), which is what compute_reward sees.  It leaves rew = the
 * plain sum of the built-in terms and rew_buf_pos / rew_buf_neg = their split; the combination, the termination term and
 * the "total" episode sum are left to go1_sim_reward_finish. */
int go1_sim_step_deferred(Go1Sim* sim, const float* actions /*[N][12]*/, const float gravity[3], const float gravity_vec[3],
                          int64_t common_step, float* pre_roll, void* stream);

/* Scratch floats go1_sim_reward_finish needs for `num_envs` envs and K user terms. */
int64_t go1_reward_finish_workspace(int num_envs, int K);

/* Finishes compute_reward (legged_robot.py:263-300) after go1_sim_step_deferred and the user terms.  raw: [K][N] user term
 * values (before scaling), scales: K host floats (already multiplied by dt).  Each user term r = raw * scale is added to rew
 * and to user_sums[k] ([K][N] episode sums), and to rew_buf_pos if its sum over all N envs is >= 0, else to rew_buf_neg if
 * it is <= 0 (neither when the sum is NaN).  That sum is taken in a fixed order (per-CTA partials in `workspace`, summed in
 * CTA order), so the sign does not depend on scheduling.  Then the combination of the config (only_positive_rewards /
 * ji22 style / plain), the termination term and the "total" episode sum, as go1_sim_step does them.  Two launches. */
int go1_sim_reward_finish(Go1Sim* sim, const float* raw, const float* scales, int K, float* user_sums, float* workspace, void* stream);

/* The user-term part of reset_idx's episode bookkeeping (legged_robot.py:181-195) for the reset list `env_ids` (count k, or
 * *k_dev when k_dev != NULL, as go1_sim_reset_idx_dev): acc[0..K-1] = sum of user_sums[k] over the reset train envs and acc[K] =
 * their count (written, not added; fixed summation order); for reset eval envs, user_sums_eval[k] ([K][N], -1 = unset) keeps
 * the first finished episode; the reset envs' user_sums are zeroed.  With acc_hist != NULL the result is also filed in
 * acc_hist[*slot_dev] ([T][K+1]; a step without a reset train env carries the previous row forward, as go1_rollout_advance
 * does for the built-in accumulator).  One CTA, no host synchronisation. */
int go1_sim_user_reward_fold(Go1Sim* sim, const int32_t* env_ids, const int32_t* k_dev, int k, int K, float* user_sums,
                             float* user_sums_eval, float* acc, float* acc_hist, int T, const int32_t* slot_dev, void* stream);

/* Self-collisions between the robot's own links (DESIGN.md §3), the counterpart of Isaac Gym's
 * asset_options.self_collisions / PhysX's self-collision filter.  Thigh and calf are capsules (thigh joint -> knee, knee -> foot),
 * the foot a sphere, the trunk the box GO1_BASE_BOX_HALF.  Tested pairs: thigh/calf/foot of one leg against thigh/calf/foot of
 * every other leg, and each leg's knee, calf midpoint and foot (as spheres of the thigh, calf and foot radius) against the
 * trunk.  Explicit penalty law: normal force max(k depth - c v_n, 0), friction clamped as for the ground penalty contacts
 * with the env's robot friction.  The forces are added to the reported thigh, calf, foot and base contact forces. */
typedef struct Go1SelfCollision {
    int32_t enabled;                    /* 0 = off (default): the step kernel is the one without self-collisions */
    float k, c;                         /* N/m, N s/m */
    float thigh_radius, calf_radius, foot_radius;   /* m */
} Go1SelfCollision;
int go1_sizeof_self_collision(void);
/* Store the self-collision model of `sim`.  Only before the first go1_sim_step: a captured step graph keeps the kernel that
 * was chosen when it was captured, so a later change fails (and leaves the setting as it was). */
int go1_sim_set_self_collision(Go1Sim* sim, const Go1SelfCollision* sc);

/* Asset options of the simulated Go1 (Cfg.asset, DESIGN.md §3).  Bodies are numbered in Isaac Gym order:
 * 0 base, then hip, thigh, calf, foot of FL (1-4), FR (5-8), RL (9-12), RR (13-16). */
#define GO1_NUM_BODIES 17
typedef struct Go1AssetOptions {
    float penalty_weight[GO1_NUM_BODIES]; /* collision term: sum_b penalty_weight[b] * (|F_b| > 0.1); Go1: 1 on thighs and calves */
    uint32_t termination_mask;          /* bit b: |F_b| > 1 ends the episode; Go1: 1 (the base) */
    int32_t fix_base;                   /* 1: the base is welded to the world (root pose held, root twist zero) */
    int32_t disable_gravity;            /* 1: no gravity acceleration on any body */
    float armature;                     /* kg m^2 added to every joint's diagonal of the joint-space inertia; >= 0 */
} Go1AssetOptions;
int go1_sizeof_asset_options(void);
/* Store the asset options of `sim` (go1_sim_create sets the Go1 values above).  Weights must be finite and >= 0, the mask
 * below 2^17, armature finite and >= 0.  Only before the first go1_sim_step: captured step graphs keep their kernel
 * arguments, so a later call fails (and leaves the options as they were). */
int go1_sim_set_asset_options(Go1Sim* sim, const Go1AssetOptions* opt);

/* Threads per CTA of the step kernel: 32, 64 or 128; 0 (default) = 32 up to 16384 envs, 128 above (tuning knob). */
void go1_sim_set_step_block(int threads);

/* Replaces LeggedRobot.reset_idx (+ _resample_commands' device part, _randomize_dof_props,
 * _reset_dofs, _reset_root_states; legged_robot.py:150-239, 645-665, 948-1001) for `k` envs, followed —
 * when post_step != 0 — by compute_observations and the last_* rolls for those envs
 * (legged_robot.py:124-131).  new_commands: [k][15] sampled by the host curriculum. */
int go1_sim_reset_idx(Go1Sim* sim, const int32_t* env_ids, int k, const float* new_commands,
                      const float* actions, int post_step, int64_t common_step, void* stream);

/* Replaces the device part of LeggedRobot._resample_commands for the periodic resample
 * (legged_robot.py:684-686, 756-824): write new commands, zero command_sums. */
int go1_sim_set_commands(Go1Sim* sim, const int32_t* env_ids, int k, const float* new_commands, void* stream);

/* ---- device-resident command curriculum ---------------------------------------------------------------------
 * Replaces the HOST work of LeggedRobot._resample_commands (legged_robot.py:710-824) and of
 * RewardThresholdCurriculum.update / Curriculum.sample (go1_gym/envs/base/curriculum.py:67-89, 135-154): success
 * test on the 4 task command sums, bin-weight updates with neighbour bumps, category draw, numpy
 * RandomState(MT19937)-exact bin + in-cell sampling (cdf, searchsorted, uniform), gait-category remap of commands
 * 5-7, binary phases, zeroing of small xy commands.  One CTA consumes the event list the step kernel wrote
 * (`events[list]`, ids sorted ascending like the reference's env_ids) so the rollout needs no host round trip. */
#define GO1_CUR_MAX_CATEGORIES 8
typedef struct Go1CurriculumConfig {
    int32_t num_categories;                          /* 1 ('nominal') or 4 (gaitwise_curricula) */
    int32_t category_kind[GO1_CUR_MAX_CATEGORIES];   /* 0 nominal, 1 pronk, 2 trot, 3 pace, 4 bound */
    int32_t num_bins, num_dims;                      /* bins per curriculum, command dimensions of the grid (15) */
    int32_t num_commands;                            /* Cfg.commands.num_commands */
    int32_t num_task_keys, task_col[4];              /* active task rewards: column of the 4 event sums */
    float threshold[4];                              /* curriculum_thresholds[key] * reward_scales[key], float32 */
    float ep_len;                                    /* min(max_episode_length, resampling_time / dt) */
    int32_t gaitwise_curricula, exclusive_phase_offset, balance_gait_distribution, binary_phases;
    int32_t num_train_envs, snapshot_time_outs;
    /* cross-rank replay (SURVEY.md §8e(4)): with xr_world > 1 the call consumes the event records of ALL ranks (gathered into
     * Go1CurriculumBuffers.xr_events) in ascending GLOBAL env id = xr_rank * num_envs + local id, exactly as one process owning
     * xr_world * num_envs envs would: every rank applies the same weight updates and draws the same RandomState words, so the
     * curricula stay identical everywhere; only the envs of this rank receive their commands / bins. */
    int32_t xr_world, xr_rank, xr_cap;
} Go1CurriculumConfig;

typedef struct Go1CurriculumBuffers {
    double* weights;             /* [num_categories][num_bins]   Curriculum.weights */
    const double* grid;          /* [num_bins][num_dims]         bin centroids (Curriculum.grid.T) */
    const double* half_bins;     /* [num_dims]                   bin_sizes / 2 */
    const double* local_range;   /* [num_dims]                   neighbour range of the weight update */
    uint32_t* mt;                /* [num_categories][625]        RandomState key[624] + pos, one per curriculum */
    uint64_t* cat_rng;           /* [1]                          splitmix64 state of the category draws */
    int32_t* env_bins;           /* [N]                          LeggedRobot.env_command_bins */
    int32_t* env_categories;     /* [N]                          LeggedRobot.env_command_categories */
    float* env_bins_f32;         /* [num_train_envs]             extras["env_bins"] */
    uint8_t* time_outs_snapshot; /* [num_train_envs]             extras["time_outs"] (copied when list 0 is not empty) */
    double* cdf;                 /* [num_categories][num_bins]   cached sampling cdf */
    int32_t* cdf_valid;          /* [num_categories]             0 after a weight change */
    int32_t* scratch_i32;        /* [8N + 64], zero on first use */
    uint32_t* scratch_u32;       /* [2 (num_dims + 1) max(N, 1024)] */
    double* scratch_f64;         /* [(num_dims + 2) max(N, 1024)] */
    int32_t* out_count;          /* [1]   number of envs processed (k for go1_sim_reset_idx_dev) */
    int32_t* out_ids;            /* [N]   their ids, ascending */
    float* out_commands;         /* [N][15] their new commands */
    /* cross-rank replay only (xr_world > 1; NULL otherwise).  Scratch sizes above then scale with xr_world * N instead of N. */
    float* xr_send;              /* [2][1 + xr_cap * GO1_XR_STRIDE]  this rank's records of both lists, written by go1_curriculum_pack */
    const float* xr_events;      /* [xr_world][2][1 + xr_cap * GO1_XR_STRIDE]  all ranks' xr_send blocks (an all-gather of xr_send) */
    int32_t* xr_ids;             /* [xr_world * N]      working list of global ids */
    float* xr_commands;          /* [xr_world * N][15]  working list of sampled commands */
} Go1CurriculumBuffers;
#define GO1_XR_STRIDE 8           /* floats per gathered record: global env id, 4 task command sums, ep_len, old bin, old category */

/* sizeof(Go1CurriculumConfig) (which = 0) / sizeof(Go1CurriculumBuffers) (which = 1) as compiled */
int go1_sizeof_curriculum(int which);

/* list 0: envs that terminated this step -> out_ids / out_commands / out_count feed go1_sim_reset_idx_dev.
 * list 1: envs due for the periodic resample -> commands written and command_sums zeroed in place
 *         (go1_sim_set_commands semantics). */
int go1_curriculum_resample(Go1Sim* sim, const Go1CurriculumConfig* cfg, const Go1CurriculumBuffers* bufs, int list, void* stream);

/* Cross-rank replay, step 1: pack this rank's two event lists (after go1_sim_step) into bufs->xr_send with global ids and the
 * envs' current bins / categories; the caller all-gathers xr_send into xr_events (one collective per env step, NCCL) before
 * the go1_curriculum_resample calls of the step (list 0) and of the next step (list 1). */
int go1_curriculum_pack(Go1Sim* sim, const Go1CurriculumConfig* cfg, const Go1CurriculumBuffers* bufs, void* stream);

/* 1 (default): calls with <= 256 events process the (independent) categories concurrently, one 256-thread group each; 0: one
 * category after the other.  Same arithmetic either way. */
void go1_curriculum_set_grouped(int on);

/* Deterministic learner (AC_Args.deterministic).  1: every learner entry point launched from then on sums its cross-CTA reductions
 * (split-K partial tiles, column sums, trailing-input terms, loss / statistics scalars, weight gradients of the narrow layers) in a
 * fixed order: per-CTA partials are stored to a workspace with plain stores and added up by a separate launch, so identical inputs
 * give bit-identical outputs on the same build, GPU model and launch configuration.  0 (default): the atomics of the default mode.
 * The mode is library-wide and read at launch; the workspace is one buffer per stream, grown outside CUDA graph capture only (a
 * launch that needs more during capture fails) and never freed, so captured graphs keep valid pointers. */
void go1_set_deterministic(int on);
int go1_deterministic(void);
/* Bytes held by the deterministic-mode workspaces of all streams. */
int64_t go1_deterministic_workspace_bytes(void);
/* Grows the workspace of `stream` to the size of the largest one: called before a CUDA graph is captured on a stream of its own, after the
 * captured work ran eagerly on another stream (the capture then finds the workspace it needs). */
int go1_deterministic_reserve(void* stream);

/* go1_sim_reset_idx with the env count read from device memory (*k_dev <= num_envs) and an optional per-call
 * accumulator for extras["train/episode"] (NULL = the bound episode_acc). */
int go1_sim_reset_idx_dev(Go1Sim* sim, const int32_t* env_ids, const int32_t* k_dev, const float* new_commands,
                          const float* actions, int post_step, int64_t common_step, float* episode_acc, void* stream);

/* Replaces HistoryWrapper.step's torch.cat roll (go1_gym/envs/wrappers/history_wrapper.py:23):
 * hist_out[n] = concat(hist_in[n][num_obs:], obs[n]). */
int go1_history_roll(const float* hist_in, const float* obs, float* hist_out, int n, int num_obs,
                     int history_len, void* stream);

/* The same roll on rows with a pitch: hist_out[n][0:K0] = concat(hist_in[n][num_obs:K0], obs[n]), K0 = num_obs * history_len,
 * with row strides ld_in / ld_out (floats, >= K0 and multiples of 4) and 16-byte aligned hist_in / hist_out; obs is contiguous
 * [n][num_obs].  Columns K0..ld_out-1 of hist_out are not written.  HistoryWrapper keeps histories whose K0 is not a multiple of
 * 4 floats at such a pitch (go1_b200.capi.history_pitch) so that the learner's tensor-core products read them in place. */
int go1_history_roll_pitched(const float* hist_in, int ld_in, const float* obs, float* hist_out, int ld_out, int n,
                             int num_obs, int history_len, void* stream);

/* ------------------------------------------------------------------ ppo_cse learner ---------- */

/* Replaces RolloutStorage.compute_returns (go1_gym_learn/ppo_cse/rollout_storage.py:74-88): GAE scan
 * over T steps for n envs ([T][n] row-major), then advantage normalisation (global mean / unbiased std).
 * dones: uint8.  stats (device, 2 doubles) receives sum and sum of squares of the raw advantages so that
 * multi-GPU callers can all-reduce before go1_ppo_normalize_advantages. */
int go1_ppo_gae(const float* rewards, const uint8_t* dones, const float* values, const float* last_values,
                float* returns, float* advantages, double* stats, int T, int n, float gamma, float lam,
                void* stream);
int go1_ppo_normalize_advantages(float* advantages, const double* stats, int64_t global_count, int64_t local_count,
                                 void* stream);

/* Hidden-layer activation of ActorCritic's MLPs (AC_Args.activation; the reference's get_activation, actor_critic.py:149-166, maps
 * `crelu` to nn.ReLU as well).  ELU is 0: zero-initialised structs and callers that predate the other kinds mean ELU(alpha = 1).
 * selu: lambda = 1.0507009873554805, alpha = 1.6732632423543772; lrelu: slope 0.01 (nn.LeakyReLU() default).  All backward kernels
 * compute the derivative from the SAVED OUTPUT y = f(v): elu y > 0 ? 1 : y + 1; selu y > 0 ? lambda : y + lambda alpha; relu y > 0 ? 1 : 0;
 * lrelu y > 0 ? 1 : 0.01; tanh 1 - y^2; sigmoid y (1 - y).  An unknown kind makes the entry point return non-zero before any launch. */
typedef enum Go1Activation { GO1_ACT_ELU = 0, GO1_ACT_SELU, GO1_ACT_RELU, GO1_ACT_LRELU, GO1_ACT_TANH, GO1_ACT_SIGMOID } Go1Activation;
/* `act` argument of the entry points that take a bare int: mode (0 none, 1 activation, 2 times its derivative) in bits 0..7, the
 * Go1Activation in bits 8.. (so the plain modes 0 / 1 / 2 keep meaning ELU). */
#define GO1_ACT(kind, mode) (((kind) << 8) | (mode))

/* GEMM primitive behind every nn.Linear of ActorCritic (actor_critic.py:38-77; replaces the cuBLAS sgemm
 * calls issued by F.linear and its autograd): C[M][N] (+)= opA(A) opB(B) (+ bias[n]), optional ELU.
 *   transA == 0: A is row-major [M][K] (row stride lda);  transA == 1: A is [K][M]
 *   transB == 0: B is row-major [K][N] (row stride ldb);  transB == 1: B is [N][K] (torch Linear weight)
 * forward  y  = act(x W^T + b):  go1_gemm(0,1, M,N,K, x,ldx, W,ldw, y,ldy, b, act, 0, impl)
 * dgrad    dx = dz W          :  go1_gemm(0,0, M,K,N, dz,lddz, W,ldw, dx,lddx, NULL,0, acc, impl)
 * wgrad    dW = dz^T x        :  go1_gemm(1,0, N,K,M, dz,lddz, x,ldx, dW,lddw, NULL,0, acc, impl)
 * Row strides let a layer read/write column slices of wider buffers, so cat(obs_history, latent)
 * (actor_critic.py:115) is never materialised.  accumulate: add into C instead of overwriting
 * (bias/act are applied after the accumulation).  act: 0 none, 1 ELU(alpha=1), GO1_ACT(kind, 1) another activation.
 * impl: 0 = fp32 CUDA cores (exact-fp32 path), 1 = wgmma TF32 tensor cores with fp32 accumulation (BF16 operands: go1_gemm_bf16_ex). */
int go1_gemm(int transA, int transB, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
             float* C, int ldc, const float* bias, int act, int accumulate, int impl, void* stream);
/* Same product with the full fused epilogue, applied in this order to each output element v = sum_k a*b:
 *   v += C_old (accumulate);  v += sum_e extra[m][e] * w_extra[n][e]  (num_extra <= 4: the E trailing input columns of
 *   the actor/critic first layer, i.e. cat(obs_history, latent) without the cat; a wider E is added after the product by
 *   go1_mlp_extra_forward);  v += bias[n];
 *   act 1: v = f(v);  act 2: v *= f'(z) computed from the saved activation dact_y[m][n] (the autograd of the activation module
 *   fused into the dgrad GEMM);  f = the Go1Activation act_kind (0 = ELU). */
typedef struct Go1GemmEpilogue {
    const float* bias; int32_t act, accumulate;
    const float* extra; int32_t ld_extra; const float* w_extra; int32_t ld_w_extra, num_extra;
    const float* dact_y; int32_t ld_dact_y;
    int32_t lead_cols;   /* > 0: the extra columns and the activation apply to output columns < lead_cols only (the rest gets
                          * bias only): lets several first layers that share their input run as ONE product (impl 1) */
    float* colsum;       /* optional [N] (impl 1): colsum[n] += sum_m C[m][n] of the FINAL values this call writes -- the bias gradient
                          * of the layer whose dz this dgrad product produces, reduced in the epilogue (atomic adds: zero it first) */
    /* optional (impl 1): C is the dz of a first layer with `num_bwd_extra` (<= 4; a wider E goes through go1_mlp_extra_backward) trailing
     * inputs (go1_mlp_extra_backward's job done in
     * this epilogue, atomic adds into zeroed outputs):  g_w_extra[n][t] += sum_m C[m][n] bwd_extra[m][t];
     * d_extra[m][t] += sum_n C[m][n] bwd_w_extra[n][t]  (d_extra may be NULL; g_w_extra may be NULL when d_extra is given) */
    const float* bwd_extra; const float* bwd_w_extra; float* g_w_extra; float* d_extra;
    int32_t ld_bwd_extra, ld_bwd_w_extra, ld_g_w_extra, ld_d_extra, num_bwd_extra;
    int32_t act_kind;    /* Go1Activation behind act 1 / 2 (0 = ELU) */
    int32_t store_transposed;   /* impl 1: C is stored as its transpose, [N][M] with row stride ldc (the fused terms above still see
                                 * C[m][n]); gives the next product a K-major operand: the first-layer dz of the weight-gradient product.
                                 * Needs M >= 32, accumulate 0, a 16-byte aligned C and ldc % 4 == 0.  The TMA store writes whole 16-byte
                                 * chunks: when M % 4 != 0, row padding columns M .. (M rounded up to 4) - 1 may be overwritten. */
    uint16_t* out_bf16;  /* optional, with store_transposed: the transposed result goes here as BF16 (round to nearest even of the fp32 value
                          * the fp32 store would write) instead of to C, which is then not written and may be NULL.  [N][M] with row stride
                          * ld_out_bf16 elements (>= M, a multiple of 8), 16-byte aligned.  The column sums and trailing-input terms above still
                          * see the fp32 values.  The A operand of a go1_gemm_bf16_ex weight gradient.  As above, whole 16-byte chunks are
                          * written: when M % 8 != 0, row padding columns M .. (M rounded up to 8) - 1 may be overwritten. */
    int32_t ld_out_bf16;
} Go1GemmEpilogue;
int go1_gemm_ex(int transA, int transB, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
                float* C, int ldc, const Go1GemmEpilogue* ep, int impl, void* stream);
/* The same product with BF16 operands (bit patterns of torch.bfloat16, leading dimensions in elements) on the wgmma BF16 tensor-core path,
 * fp32 accumulation, fp32 output and the full fused epilogue above: the first-layer products of AC_Args.gemm_impl = 2, which reduce over the
 * observation history.  Both operands K-major: transA = 0 (A [M][K]) and transB = 1 (B [N][K]); 16-byte aligned, lda / ldb multiples of 8.
 * Any other layout returns non-zero before any launch. */
int go1_gemm_bf16_ex(int transA, int transB, int M, int N, int K, const uint16_t* A, int lda, const uint16_t* B, int ldb,
                     float* C, int ldc, const Go1GemmEpilogue* ep, void* stream);
/* Conversions to BF16 for those products, each rounding once to nearest even (torch's .to(torch.bfloat16)); columns of dst beyond the
 * copied width (row pitch padding) are not written.
 *   go1_convert_bf16:       dst[r][c] = bf16(src[r][c])                  rows x cols, row strides lds / ldd (elements)
 *   go1_gather_rows_bf16:   dst[i][c] = src[idx[i]][c], c < width        BF16 source (the rollout's BF16 history slab: no rounding)
 *   go1_rollout_store_rows_bf16: slab[slot][r][c] = src[r][c]           BF16 rows into slot *slot_dev (slot 0 if NULL) of a [T][rows][ldd]
 *                           slab: the history the policy evaluated, stored by the captured env step (go1_rollout_store_transition then
 *                           takes in_f32[2] = NULL)
 *   go1_transpose_to_bf16:  dst[c][r] = bf16(src[r][c])                  fp32 source
 *   go1_transpose_bf16:     dst[c][r] = src[r][c]                        BF16 source (no rounding) */
int go1_convert_bf16(const float* src, int lds, uint16_t* dst, int ldd, int rows, int cols, void* stream);
int go1_gather_rows_bf16(const uint16_t* src, int lds, const int64_t* idx, uint16_t* dst, int ldd, int64_t rows, int width, void* stream);
int go1_rollout_store_rows_bf16(const uint16_t* src, int lds, uint16_t* dst_base, int ldd, const int32_t* slot_dev, int rows, int cols, void* stream);
int go1_transpose_to_bf16(const float* src, int lds, uint16_t* dst, int ldd, int rows, int cols, void* stream);
int go1_transpose_bf16(const uint16_t* src, int lds, uint16_t* dst, int ldd, int rows, int cols, void* stream);
/* Up to 16 go1_convert_bf16 copies in ONE launch, dst[r][c] = bf16(src[r][c]) per segment: the BF16 copies of the hidden-layer outputs that
 * the weight gradients of AC_Args.bf16_backward read and of the hidden weights its dgrads read, made once per minibatch forward.  A bad segment returns non-zero before any launch. */
typedef struct Go1Bf16Seg { const float* src; int32_t lds; uint16_t* dst; int32_t ldd; int32_t rows, cols; } Go1Bf16Seg;
int go1_convert_bf16_segments(const Go1Bf16Seg* segs, int n, void* stream);
/* go1_gemm_bf16_ex with BF16 operands in EITHER major (transA / transB as go1_gemm), read in place: an MN-major operand ([K][M] A, [K][N] B,
 * the dgrad's W and both operands of a weight gradient) reaches the tensor core as 128B-swizzled TMA boxes through the transpose immediates
 * of BF16 wgmma, without the shared-to-shared transposition of the TF32 kernel.  The full Go1GemmEpilogue, out_bf16 included.
 *   c_bf16 = 0: C is fp32 [M][N] (row stride ldc floats), as go1_gemm_bf16_ex.
 *   c_bf16 = 1: C is a row-major BF16 matrix (uint16_t*, ldc elements, a multiple of 8, >= N, 16-byte aligned): every value is rounded once
 *               to nearest even after all fp32 terms (the column sums and trailing-input terms see fp32 values, as with out_bf16).  Whole
 *               16-byte chunks are written: when N % 8 != 0, row padding columns N .. (N rounded up to 8) - 1 may be overwritten.  Not
 *               with accumulate, store_transposed or out_bf16.
 * A / B 16-byte aligned with lda / ldb multiples of 8 elements (TMA); anything else returns non-zero before any launch.  Used by the
 * hidden-layer dgrads and weight gradients of AC_Args.bf16_backward. */
int go1_gemm_bf16_mn(int transA, int transB, int M, int N, int K, const uint16_t* A, int lda, const uint16_t* B, int ldb,
                     void* C, int ldc, int c_bf16, const Go1GemmEpilogue* ep, void* stream);
/* go1_gemm_grouped with BF16 operands in either major (go1_gemm_bf16_mn's kernels, fp32 C): the equal-shape weight gradients of
 * AC_Args.bf16_backward in one grid. */
int go1_gemm_bf16_grouped(int transA, int transB, int M, int N, int K, int nprob, const uint16_t* const* A, int lda, const uint16_t* const* B, int ldb,
                          float* const* C, int ldc, int accumulate, void* stream);
/* nprob (<= 4) wgmma products of the SAME shape and operand strides in one grid: C[p] (+)= op(A[p]) op(B[p]) (impl 1 only, no fused
 * epilogue operands).  Used for the equal-shape split-K wgrads of the three MLPs (nn.Linear weight gradients, actor_critic.py:38-77). */
int go1_gemm_grouped(int transA, int transB, int M, int N, int K, int nprob, const float* const* A, int lda, const float* const* B, int ldb,
                     float* const* C, int ldc, int accumulate, void* stream);
/* The layers BEHIND a first layer of one of ActorCritic's MLPs in one launch (impl 1, wgmma; actor_critic.py:38-77, 113-144):
 *   y2 = ELU(x W2^T + b2) [M][N2];   y3 = ELU(y2 W3^T + b3) [M][N3]  (N3 = 0: skipped);   out = y_last Wh^T + bh [M][nh], nh <= 16.
 * x is the first layer's activated output (K1 columns, row stride ldx); W* are torch nn.Linear weights [out][in], contiguous; y2 / y3 are
 * kept for the backward pass.  Any K1 >= 1, N2 = 1..256, N3 = 0..128: 512-256-128 (actor / critic bodies of scripts/train.py) and 256-128-0
 * (adaptation module) run on exact-width kernels, every other shape on kernels whose tiles cover N2 / N3 (64, 128 or 256 columns), with the
 * rows and columns beyond the widths read as zeros (the y2 stores write whole 16-byte chunks: when N2 % 4 != 0, row padding columns
 * N2 .. (N2 rounded up to 4) - 1 may be overwritten); the activations between the layers never leave the SM (wgmma accumulators in
 * registers -> shared memory -> tensor core). */
int go1_mlp_tail_forward(const float* x, int ldx, int M, int K1, const float* W2, const float* b2, int N2, float* y2, int ldy2,
                         const float* W3, const float* b3, int N3, float* y3, int ldy3, const float* Wh, const float* bh, int nh,
                         float* out, int ldout, void* stream);
/* The same (ELU, or the problems' act_kind) for up to two problems of equal shape in ONE grid (the actor and critic bodies: one CTA per SM
 * walks the 64-row blocks of both problems, instead of two launches that each end in a partly filled round).  nh <= 12 per problem. */
typedef struct Go1TailProblem {
    const float* x; int32_t ldx; const float* W2; const float* b2; float* y2; int32_t ldy2;
    const float* W3; const float* b3; float* y3; int32_t ldy3; const float* Wh; const float* bh; int32_t nh; float* out; int32_t ldout;
    int32_t act_kind;    /* Go1Activation in place of ELU (0 = ELU); the problems of one launch share it */
    int32_t ldw2, ldw3;  /* row strides of W2 / W3 in floats, multiples of 4 (0: contiguous, K1 / N2) */
} Go1TailProblem;
int go1_mlp_tail_forward_grouped(const Go1TailProblem* probs, int nprob, int M, int K1, int N2, int N3, void* stream);

/* Per-launch timing of the impl-1 (wgmma) products for the roofline report: on = 1 starts collecting (CUDA events on the launch
 * stream around every call that is not being graph-captured), on = 0 stops and returns the summed kernel time, flops and count. */
int go1_gemm_timing(int on, double* total_ms, double* total_flop, long long* launches);
/* number of kernels replayed through CUDA graphs, added to go1_kernel_launch_count() by the caller that replays them */
void go1_kernel_launch_add(long long n);
/* dst[c][r] = src[r][c] (rows x cols fp32, row strides lds/ldd).  impl 1 reads operands in either major, but an MN-major one is
 * transposed on the SM every k-block: the learner stages the K-major copy of the minibatch history for its first-layer weight gradients. */
int go1_transpose(const float* src, int lds, float* dst, int ldd, int rows, int cols, void* stream);
/* dz = dy * ELU'(z) computed from the saved layer output y (autograd of nn.ELU). dz may alias dy. */
int go1_elu_backward(const float* y, int ldy, const float* dy, int lddy, float* dz, int lddz, int M, int N, void* stream);
/* The same for any Go1Activation: dz = dy * f'(z) from the saved output y (go1_elu_backward is kind GO1_ACT_ELU of this kernel). */
int go1_act_backward(const float* y, int ldy, const float* dy, int lddy, float* dz, int lddz, int M, int N, int kind, void* stream);
/* Finishes a first layer whose trailing-input term was left out of the product: y = act(y + extra[m][:E] . w_extra[n][:E])
 * in place (1 <= E <= 64, the privileged-observation widths: at most 45; act 0 / 1 / GO1_ACT(kind, 1)).  Row strides: ldy >= o,
 * ldex >= E, ldw >= E.  A bad argument returns non-zero before any launch. */
int go1_mlp_extra_forward(float* y, int ldy, const float* extra, int ldex, const float* w_extra, int ldw, int M, int o, int E, int act,
                          void* stream);
/* Backward of the E (1..64) trailing input columns of a first layer (the `latent` / privileged columns of
 * cat(obs_history, .), actor_critic.py:115,143), bandwidth-bound passes over dz:
 *   g_w_extra[j][t] (+)= sum_m dz[m][j] extra[m][t]  (if g_w_extra != NULL; needs dz_transposed 0);
 *   dextra[m][t] = sum_j dz[m][j] w_extra[j][t]      (if dextra != NULL).
 * dz_transposed 0: dz is [M][o] (lddz >= o);  1: dz is stored as [o][M] (lddz >= M), the first-layer dz a store_transposed dgrad
 * epilogue writes.  At least one output; a bad argument returns non-zero before any launch. */
int go1_mlp_extra_backward(const float* dz, int lddz, int dz_transposed, const float* extra, int ldex, const float* w_extra, int ldw,
                           float* g_w_extra, int ldgw, float* dextra, int ldde, int M, int o, int E, int accumulate, void* stream);
/* Forward of a narrow (o <= 16) output layer, the 12 / 2 / 1-wide heads of ActorCritic (actor_critic.py:52,64,76):
 *   out[m][t] = b[t] + sum_k x[m][k] W[t][k]   (W row-major [o][K], K % 4 == 0, x rows 16-byte aligned; b may be NULL). */
int go1_skinny_forward(const float* x, int ldx, const float* W, int ldw, const float* b, float* out, int ldo, int M, int o, int K, void* stream);
/* dgrad through a narrow (o <= 16) output layer, with the previous layer's ELU' fused (y_prev may be NULL):
 *   dprev[m][c] = (sum_t dz[m][t] W[t][c]) * ELU'(y_prev[m][c]),  W row-major [o][n]. */
int go1_skinny_dgrad(const float* dz, int lddz, const float* W, int ldw, const float* y_prev, int ldy, float* dprev, int lddp,
                     int M, int o, int n, void* stream);
/* go1_skinny_dgrad + the column sums of the values written, colsum[c] += sum_m dprev[m][c] (atomics into a zeroed buffer; may be NULL):
 * the bias gradient of the layer below (nn.Linear backward), reduced while dprev is produced. */
int go1_skinny_dgrad_ex(const float* dz, int lddz, const float* W, int ldw, const float* y_prev, int ldy, float* dprev, int lddp,
                        float* colsum, int M, int o, int n, void* stream);
/* go1_skinny_dgrad_ex with the derivative of any Go1Activation in place of ELU'. */
int go1_skinny_dgrad_act(const float* dz, int lddz, const float* W, int ldw, const float* y_prev, int ldy, float* dprev, int lddp,
                         float* colsum, int M, int o, int n, int kind, void* stream);
/* go1_skinny_dgrad_act whose dprev is BF16 (uint16_t, lddp elements), each value rounded once to nearest even after the fp32 column sum:
 * the head dgrad of AC_Args.bf16_backward.  n, ldw, lddp and ldy multiples of 4, W / y_prev 16-byte and dprev 8-byte aligned. */
int go1_skinny_dgrad_act_bf16(const float* dz, int lddz, const float* W, int ldw, const float* y_prev, int ldy, uint16_t* dprev, int lddp,
                              float* colsum, int M, int o, int n, int kind, void* stream);
/* go1_skinny_wgrad + the layer's bias gradient gb[j] (+)= sum_m dz[m][j] (may be NULL; needs K % 4 == 0 and 16-byte aligned x rows). */
int go1_skinny_wgrad_ex(const float* dz, int lddz, const float* x, int ldx, float* gW, int ldg, float* gb, int M, int o, int K, int accumulate, void* stream);
/* wgrad of a narrow (o <= 16) output layer (the 12 / 2 / 1-wide heads): gW[j][k] (+)= sum_m dz[m][j] x[m][k]. */
int go1_skinny_wgrad(const float* dz, int lddz, const float* x, int ldx, float* gW, int ldg, int M, int o, int K, int accumulate, void* stream);
/* Up to 8 strided 2-D copies dst[r][c] = src[r][c] in ONE launch: builds the packed first-layer weight block / bias / trailing-input
 * weights that the fused first-layer product of ActorCritic reads (actor_critic.py:113-144 evaluates the three MLPs on the same
 * obs_history), and brings the fused wgrad's output back into the flat gradient buffer. */
typedef struct Go1CopySeg { const float* src; int32_t lds; float* dst; int32_t ldd; int32_t rows, cols; } Go1CopySeg;
int go1_copy_segments(const Go1CopySeg* segs, int n, void* stream);
/* out[n] (+)= sum_m x[m][n]: bias gradient of nn.Linear. */
int go1_colsum(const float* x, int ldx, float* out, int M, int N, int accumulate, void* stream);

/* Replaces the Normal(mean,std) sample + log-prob of ActorCritic.act / get_actions_log_prob
 * (actor_critic.py:113-126): actions = mean + std*eps (eps ~ N(0,1) from Philox(seed,counter) or the
 * injected `eps` for parity tests), logp = sum_j log N(a_j).  counter_dev (optional, device memory): added to `counter` and
 * incremented by the call, so that a CUDA graph holding this call draws fresh noise on every replay. */
int go1_ppo_sample_actions(const float* mean, int ldm, const float* std, const float* eps, uint64_t seed,
                           uint64_t counter, uint64_t* counter_dev, float* actions, float* logp, int n, int num_actions,
                           void* stream);

/* Replaces the loss block of PPO.update (ppo.py:113-152): from the minibatch forward outputs computes the
 * clipped surrogate, clipped value loss, entropy bonus, their gradients w.r.t. mean / value / std, and the
 * KL(old||new) mean used by the adaptive LR schedule.  scalars (device, 8 floats): surrogate_loss,
 * value_loss, entropy_mean, kl_mean, ... ; inv_count = 1/global minibatch size. */
int go1_ppo_loss(const float* mean, int ldm, const float* std, const float* value, const float* actions,
                 const float* old_logp, const float* old_mean, const float* old_std, const float* advantages,
                 const float* returns, const float* old_values, float* dmean, int lddm, float* dvalue,
                 float* dstd, float* scalars, int n, int num_actions, float clip_param,
                 float value_loss_coef, float entropy_coef, int use_clipped_value_loss, float inv_count,
                 void* stream);

/* Replaces F.mse_loss(adaptation_pred[:num_train], target[:num_train]) fwd+bwd and the test-split loss
 * (ppo.py:168-186). scalars: [0] train loss, [1] test loss. */
int go1_ppo_mse(const float* pred, int ldp, const float* target, int ldt, float* dpred, int lddp, float* scalars,
                int n, int num_train, int dim, void* stream);

/* Replaces nn.utils.clip_grad_norm_ + Adam.step over one flat parameter/gradient buffer
 * (ppo.py:155-158, 187-189).  grad_sq (device double) = sum of squared gradients (computed by
 * go1_ppo_grad_sqnorm, all-reducible).  max_grad_norm <= 0 disables clipping. */
int go1_ppo_grad_sqnorm(const float* grad, int64_t count, double* grad_sq, void* stream);
int go1_ppo_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t count,
                      const double* grad_sq, float max_grad_norm, float lr, const float* lr_dev, float beta1, float beta2,
                      float eps, int step, void* stream);
/* Replaces the adaptive-KL learning-rate schedule of PPO.update (ppo.py:118-132) without a host sync:
 * lr_dev <- max(lr_min, lr/1.5) if kl > 2*desired_kl; min(lr_max, lr*1.5) if 0 < kl < desired_kl/2.
 * kl = scalars[3] written by go1_ppo_loss (all-reduced first on multi-GPU).  go1_ppo_adam_step reads the
 * learning rate from lr_dev when it is non-NULL. */
int go1_ppo_adaptive_lr(const float* scalars, float* lr_dev, float desired_kl, float lr_min, float lr_max, void* stream);

/* Replaces RolloutStorage.add_transitions (rollout_storage.py:55-69) and the time-out bootstrap of
 * PPO.process_env_step (ppo.py:84-86: rewards += gamma * values * time_outs) in one launch.
 * in_f32[10]  = {obs[n][nobs] or NULL, priv[n][npriv] or NULL, obs_history[n][nhist], actions[n][nact], rewards[n], values[n], log_prob[n],
 *                action_mean[n][nact], std[nact], env_bins[n] or NULL};  dones/time_outs: uint8 [n] (time_outs may be NULL)
 * out_f32[10] = the slot `step` of the storage slabs in the same order (sigma[n][nact] for std);  s_dones: uint8 [n].
 * obs_history may be NULL: the history is then not stored (a BF16 slab, filled by go1_rollout_store_rows_bf16). */
int go1_store_transition(const float* const* in_f32, const uint8_t* dones, const uint8_t* time_outs, float* const* out_f32, uint8_t* s_dones,
                         int n, int nobs, int npriv, int nhist, int nact, float gamma, void* stream);

/* The observation half of RolloutStorage.add_transitions (rollout_storage.py:58-59), done when PPO.act records the transition
 * (ppo.py:73-76): s_obs[n][nobs] <- obs, s_priv[n][npriv] <- priv.  The env's observation buffers are overwritten in place by
 * the next go1_sim_step, so the copy cannot wait for process_env_step; go1_store_transition then takes in_f32[0] = in_f32[1] = NULL. */
int go1_store_observations(const float* obs, const float* priv, float* s_obs, float* s_priv, int n, int nobs, int npriv, void* stream);

/* The two stores above with the slot index `*slot_dev` read on the device and slab BASE pointers ([T][n][.]) as outputs, so that ONE
 * captured CUDA graph of a whole env step (policy, sim step, curriculum, reset, history roll, stores) is replayed for every step of the
 * rollout (ppo_cse/__init__.py:138-147); go1_rollout_advance closes a step: it files the step's extras["train/episode"] accumulator
 * `acc[W]` (last element = number of train envs reset; 0 -> the previous slot's entry is carried forward, like the reference's extras
 * entry that stays in place) into acc_hist[T][W], then *slot_dev = (*slot_dev + 1) % T and *step_dev += 1 (Go1SimBuffers.step_dev). */
int go1_rollout_store_observations(const float* obs, const float* priv, float* s_obs_base, float* s_priv_base, const int32_t* slot_dev,
                                   int n, int nobs, int npriv, void* stream);
int go1_rollout_store_transition(const float* const* in_f32, const uint8_t* dones, const uint8_t* time_outs, float* const* out_base_f32,
                                 uint8_t* s_dones_base, const int32_t* slot_dev, int n, int nobs, int npriv, int nhist, int nact, float gamma,
                                 void* stream);
int go1_rollout_advance(const float* acc, float* acc_hist, int W, int T, int32_t* slot_dev, int64_t* step_dev, void* stream);

/* Replaces the fancy-index gathers of RolloutStorage.mini_batch_generator (rollout_storage.py:98-137):
 * dst[i][0:width] = src[idx[i]][0:width]; ldd = row stride of dst in floats (>= width). */
int go1_gather_rows(const float* src, const int64_t* idx, float* dst, int64_t rows, int width, int ldd, void* stream);

#ifdef __cplusplus
}
#endif
#endif
