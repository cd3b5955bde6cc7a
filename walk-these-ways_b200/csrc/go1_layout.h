// Internal SoA row layout of the sim state (shared by the kernels and the C-ABI row query).
// Per-env rows: [row][N]; per-leg rows: [row][4N] with index env*4+leg (legs FL,FR,RL,RR); a
// "3-wide" per-leg field holds the leg's hip/thigh/calf joint values in 3 consecutive rows.
#pragma once
#include "../../include/go1_b200.h"

#define GO1_NUM_EPISODE_SUMS (GO1_NUM_REWARD_TERMS + 1)   // + "total"        (legged_robot.py:1415-1419)
#define GO1_NUM_COMMAND_SUMS (GO1_NUM_REWARD_TERMS + 5)   // + 5 raw sums     (legged_robot.py:1425-1429)

#define GO1_ENV_F32_FIELDS(X) \
    X(root_pos, 3) X(root_quat, 4) X(root_lin_vel, 3) X(root_ang_vel, 3) \
    X(commands, GO1_NUM_COMMANDS) X(gait_indices, 1) \
    X(friction_coeffs, 1) X(restitutions, 1) X(payloads, 1) X(com_displacements, 3) \
    X(motor_strengths, 1) X(Kp_factors, 1) X(Kd_factors, 1) X(env_origins, 3) X(rigid_payload, 1) X(rigid_com, 3) \
    X(base_lin_vel, 3) X(base_ang_vel, 3) X(projected_gravity, 3) X(rew_buf_pos, 1) X(rew_buf_neg, 1) \
    X(episode_sums, GO1_NUM_EPISODE_SUMS) X(command_sums, GO1_NUM_COMMAND_SUMS)

#define GO1_LEG_F32_FIELDS(X) \
    X(dof_pos, 3) X(dof_vel, 3) X(last_dof_vel, 3) X(actions, 3) X(last_actions, 3) X(last_last_actions, 3) \
    X(joint_pos_target, 3) X(last_joint_pos_target, 3) X(last_last_joint_pos_target, 3) X(lag_buffer, 3 * GO1_MAX_LAG_TIMESTEPS) \
    X(joint_pos_err_last, 3) X(joint_pos_err_last_last, 3) X(joint_vel_last, 3) X(joint_vel_last_last, 3) \
    X(motor_offsets, 3) X(torques, 3) \
    X(clock_inputs, 1) X(doubletime_clock_inputs, 1) X(halftime_clock_inputs, 1) \
    X(desired_contact_states, 1) X(foot_indices, 1) \
    X(foot_positions, 3) X(foot_velocities, 3) X(prev_foot_velocities, 3) X(foot_contact_forces, 3) X(hip_contact_forces, 3) \
    X(thigh_contact_forces, 3) X(calf_contact_forces, 3) X(base_contact_forces_part, 3) X(last_contacts, 1)

#define GO1_ENV_I32_FIELDS(X) X(episode_length_buf, 1)

// compile-time row offsets (running-sum enum: each field starts after the previous field's last row)
enum Go1EnvF32Rows {
#define X(name, n) EROW_##name, EROW_##name##_end = EROW_##name + (n) - 1,
    GO1_ENV_F32_FIELDS(X)
#undef X
    GO1_ENV_F32_ROWS
};
enum Go1LegF32Rows {
#define X(name, n) LROW_##name, LROW_##name##_end = LROW_##name + (n) - 1,
    GO1_LEG_F32_FIELDS(X)
#undef X
    GO1_LEG_F32_ROWS
};
#define EROW(name) EROW_##name
#define LROW(name) LROW_##name
#define IROW_episode_length_buf 0
#define GO1_ENV_I32_ROWS 1

// ---- table staged into shared memory by one TMA bulk copy per CTA ----
struct alignas(16) Go1LegModel {
    float r_hip[3], r_thigh[3], r_calf[3], r_foot[3];      // joint origins in parent frame, foot in calf frame
    float I_hip[10], I_thigh[10], I_calf[10];              // rigid inertia about link origin: Ixx,Ixy,Ixz,Iyy,Iyz,Izz, hx,hy,hz (=m*c), m
    float lim_lo[3], lim_hi[3], vmax[3];
    float hip_coll[3];                                      // hip collision sphere centre (hip frame)
    float sx, sy;                                           // +1 front / left
};

struct alignas(16) Go1DevTable {
    // actuator network (legged_robot.py:1238-1251): W1[32][8] (6 used, padded), b1[32], W2T[32][32] (k-major), b2[32], W3[32], b3
    float act_W1[32 * 8];
    float act_b1[32];
    float act_W2T[32 * 32];
    float act_b2[32];
    float act_W3[32];
    float act_b3[4];
    Go1LegModel leg[4];
    float base_mass, base_Icom[6], base_box[3], foot_radius, hip_coll_radius, knee_radius, calf_radius;
    Go1SimConfig cfg;
};
