// capi.cu — C-ABI of libgo1b200.so (declared in include/go1_b200.h): handle management, table upload,
// error reporting.  No torch types, no hidden allocations after create, no CPU fallback.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <string>
#include "go1_layout.h"
#include "go1_model_generated.h"

extern "C" int go1_launch_step(const Go1SimBuffers*, const Go1DevTable*, const Go1SelfCollision*, const Go1AssetOptions*, const float*, const float*, const float*, long long, int, int, float*, cudaStream_t);
extern "C" int go1_launch_reward_finish(const Go1SimBuffers*, const Go1SimConfig*, const float*, const float*, int, float*, float*, int, cudaStream_t);
extern "C" int go1_launch_user_reward_fold(const int*, const int*, int, int, float*, float*, float*, float*, int, const int*, int, int, cudaStream_t);
extern "C" long long go1_reward_finish_workspace_floats(int, int);
extern "C" int go1_launch_reset(const Go1SimBuffers*, const Go1DevTable*, const int*, int, const float*, const float*, int, long long, const float*, int, int, cudaStream_t);
extern "C" int go1_launch_set_commands(const Go1SimBuffers*, const int*, int, const float*, int, cudaStream_t);
extern "C" int go1_launch_reset_dev(const Go1SimBuffers*, const Go1DevTable*, const int*, const int*, const float*, const float*, int, long long, const float*, float*, int, int, cudaStream_t);
extern "C" int go1_launch_curriculum(const Go1SimBuffers*, const Go1CurriculumConfig*, const Go1CurriculumBuffers*, int, int, cudaStream_t);
extern "C" int go1_launch_curriculum_pack(const Go1SimBuffers*, const Go1CurriculumConfig*, const Go1CurriculumBuffers*, int, cudaStream_t);
extern "C" int go1_launch_history_roll(const float*, const float*, float*, int, int, int, cudaStream_t);
extern "C" int go1_launch_history_roll_pitched(const float*, int, const float*, float*, int, int, int, int, cudaStream_t);

static thread_local std::string g_err;
static int fail(const std::string& m) { g_err = m; return 1; }
static int cuda_fail(const char* what, int e) {
    g_err = std::string(what) + ": " + cudaGetErrorString((cudaError_t)e);
    return e ? e : 1;
}
int go1_set_error(const char* m) { return fail(m); }
#include <atomic>
static std::atomic<long long> g_launches{0};
void go1_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
extern "C" long long go1_kernel_launch_count(void) { return g_launches.load(); }
extern "C" void go1_kernel_launch_add(long long n) { g_launches += n; }

struct Go1Sim {
    Go1SimConfig cfg;
    Go1DevTable* d_tab;
    Go1DevTable h_tab;
    Go1SimBuffers bufs;
    int bound;
    int device;
    float gravity[3];
    Go1SelfCollision self;   // enabled = 0 unless go1_sim_set_self_collision turned it on
    Go1AssetOptions asset;   // the Go1 values (go1_asset_defaults) unless go1_sim_set_asset_options replaced them
    int stepped;             // go1_sim_step has been called: the kernel choice is fixed
};

extern "C" const char* go1_last_error(void) { return g_err.c_str(); }
extern "C" int go1_version(void) { return 100; }
extern "C" int go1_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

extern "C" int go1_sizeof_config(void) { return (int)sizeof(Go1SimConfig); }
extern "C" int go1_sizeof_buffers(void) { return (int)sizeof(Go1SimBuffers); }
extern "C" int go1_sizeof_self_collision(void) { return (int)sizeof(Go1SelfCollision); }
extern "C" int go1_sizeof_asset_options(void) { return (int)sizeof(Go1AssetOptions); }

// config_go1's asset section (go1_gym/envs/go1/go1_config.py): penalize_contacts_on = ["thigh", "calf"],
// terminate_after_contacts_on = ["base"], a floating base under gravity, no armature
static void go1_asset_defaults(Go1AssetOptions* o) {
    memset(o, 0, sizeof(*o));
    for (int leg = 0; leg < 4; leg++) { o->penalty_weight[1 + 4 * leg + 1] = 1.f; o->penalty_weight[1 + 4 * leg + 2] = 1.f; }
    o->termination_mask = 1u;
}

extern "C" int go1_sim_num_rows(int kind) {
    return kind == 0 ? (int)GO1_ENV_F32_ROWS : (kind == 1 ? (int)GO1_LEG_F32_ROWS : (kind == 2 ? GO1_ENV_I32_ROWS : -1));
}
extern "C" int go1_sim_row(int kind, const char* name) {
    if (!name) return -1;
    if (kind == 0) {
#define X(n, c) if (!strcmp(name, #n)) return (int)EROW_##n;
        GO1_ENV_F32_FIELDS(X)
#undef X
    } else if (kind == 1) {
#define X(n, c) if (!strcmp(name, #n)) return (int)LROW_##n;
        GO1_LEG_F32_FIELDS(X)
#undef X
    } else if (kind == 2) {
        if (!strcmp(name, "episode_length_buf")) return IROW_episode_length_buf;
    }
    return -1;
}

static void rigid_inertia_row(double m, const double c[3], const double Ic[9], float out[10]) {
    double cc = c[0] * c[0] + c[1] * c[1] + c[2] * c[2];
    double A[3][3];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) A[i][j] = Ic[3 * i + j] + m * ((i == j ? cc : 0.0) - c[i] * c[j]);
    out[0] = (float)A[0][0]; out[1] = (float)A[0][1]; out[2] = (float)A[0][2]; out[3] = (float)A[1][1]; out[4] = (float)A[1][2]; out[5] = (float)A[2][2];
    out[6] = (float)(m * c[0]); out[7] = (float)(m * c[1]); out[8] = (float)(m * c[2]); out[9] = (float)m;
}

static int build_table(const Go1SimConfig* cfg, const float* aw, Go1DevTable* T) {
    memset(T, 0, sizeof(*T));
    if (aw) {
        // W1[32][6] -> padded [32][8]
        for (int k = 0; k < 32; k++) for (int m = 0; m < 6; m++) T->act_W1[k * 8 + m] = aw[k * 6 + m];
        const float* p = aw + 192;
        for (int k = 0; k < 32; k++) T->act_b1[k] = p[k];
        p += 32;
        // W2[out i][in k] -> W2T[k][i]
        for (int i = 0; i < 32; i++) for (int k = 0; k < 32; k++) T->act_W2T[k * 32 + i] = p[i * 32 + k];
        p += 1024;
        for (int k = 0; k < 32; k++) T->act_b2[k] = p[k];
        p += 32;
        for (int k = 0; k < 32; k++) T->act_W3[k] = p[k];
        p += 32;
        T->act_b3[0] = p[0];
    } else if (cfg->control_type == 0) {
        return fail("control_type actuator_net needs actuator_weights");
    }
    for (int L = 0; L < 4; L++) {
        Go1LegModel& M = T->leg[L];
        for (int k = 0; k < 3; k++) {
            M.r_hip[k] = (float)GO1_HIP_ORIGIN[L][k]; M.r_thigh[k] = (float)GO1_THIGH_ORIGIN[L][k];
            M.r_calf[k] = (float)GO1_CALF_ORIGIN[L][k]; M.r_foot[k] = (float)GO1_FOOT_OFFSET[L][k];
            M.hip_coll[k] = (float)GO1_HIP_COLL_OFFSET[L][k];
        }
        rigid_inertia_row(GO1_HIP_MASS[L], GO1_HIP_COM[L], GO1_HIP_INERTIA_COM[L], M.I_hip);
        rigid_inertia_row(GO1_THIGH_MASS[L], GO1_THIGH_COM[L], GO1_THIGH_INERTIA_COM[L], M.I_thigh);
        rigid_inertia_row(GO1_CALF_MASS[L], GO1_CALF_COM[L], GO1_CALF_INERTIA_COM[L], M.I_calf);
        M.lim_lo[0] = (float)GO1_HIP_LIMITS[L][0]; M.lim_hi[0] = (float)GO1_HIP_LIMITS[L][1];
        M.lim_lo[1] = (float)GO1_THIGH_LIMITS[L][0]; M.lim_hi[1] = (float)GO1_THIGH_LIMITS[L][1];
        M.lim_lo[2] = (float)GO1_CALF_LIMITS[L][0]; M.lim_hi[2] = (float)GO1_CALF_LIMITS[L][1];
        M.vmax[0] = (float)GO1_HIP_VEL_LIMIT; M.vmax[1] = (float)GO1_THIGH_VEL_LIMIT; M.vmax[2] = (float)GO1_CALF_VEL_LIMIT;
        M.sx = (L < 2) ? 1.f : -1.f; M.sy = (L % 2 == 0) ? 1.f : -1.f;
    }
    T->base_mass = (float)GO1_BASE_MASS;
    const double* I = GO1_BASE_INERTIA_COM;
    T->base_Icom[0] = (float)I[0]; T->base_Icom[1] = (float)I[1]; T->base_Icom[2] = (float)I[2];
    T->base_Icom[3] = (float)I[4]; T->base_Icom[4] = (float)I[5]; T->base_Icom[5] = (float)I[8];
    for (int k = 0; k < 3; k++) T->base_box[k] = (float)GO1_BASE_BOX_HALF[k];
    T->foot_radius = (float)GO1_FOOT_RADIUS; T->hip_coll_radius = (float)GO1_HIP_COLL_RADIUS;
    T->knee_radius = 0.017f; T->calf_radius = 0.008f;
    T->cfg = *cfg;
    return 0;
}

static int check_cfg(const Go1SimConfig* c) {
    if (!c) return fail("null config");
    if (c->num_envs <= 0) return fail("num_envs must be positive");
    if (c->num_obs <= 0 || c->num_obs > GO1_MAX_OBS) return fail("num_obs out of range");
    if (c->num_priv_obs < 0 || c->num_priv_obs > GO1_MAX_PRIV_OBS) return fail("num_priv_obs out of range");
    if (c->num_commands < 3 || c->num_commands > GO1_NUM_COMMANDS) return fail("num_commands out of range");
    if (c->decimation <= 0 || c->sim_dt <= 0.f) return fail("bad sim_dt/decimation");
    if (c->lag_timesteps < 0 || c->lag_timesteps > GO1_MAX_LAG_TIMESTEPS) {
        char b[96]; snprintf(b, sizeof b, "lag_timesteps (%d) must be in 0..%d", c->lag_timesteps, GO1_MAX_LAG_TIMESTEPS); return fail(b);
    }
    if (c->num_active_rewards < 0 || c->num_active_rewards > GO1_NUM_REWARD_TERMS) return fail("bad num_active_rewards");
    for (int i = 0; i < c->num_active_rewards; i++)
        if (c->reward_order[i] < 0 || c->reward_order[i] >= GO1_NUM_REWARD_TERMS) return fail("bad reward_order entry");
    // observation width implied by the flags (legged_robot.py:302-376) must match num_obs
    int w = 3 + 12 + 12 + 12;
    if (c->observe_command) w += c->num_commands;
    if (c->observe_two_prev_actions) w += 12;
    if (c->observe_timing_parameter) w += 1;
    if (c->observe_clock_inputs) w += 4;
    if (c->observe_vel) w += 6;
    if (c->observe_only_ang_vel) w += 3;
    if (c->observe_only_lin_vel) w += 3;
    if (c->observe_yaw) w += 1;
    if (c->observe_contact_states) w += 4;
    if (w != c->num_obs) { char b[128]; snprintf(b, sizeof b, "num_obs (%d) != width implied by observe_* flags (%d)", c->num_obs, w); return fail(b); }
    int p = 0;
    p += c->priv_friction + c->priv_restitution + c->priv_base_mass + 3 * c->priv_com_displacement + 12 * c->priv_motor_strength +
         12 * c->priv_motor_offset + c->priv_body_height + 3 * c->priv_body_velocity + 3 * c->priv_gravity + 4 * c->priv_clock_inputs +
         4 * c->priv_desired_contact_states;
    if (p != c->num_priv_obs) { char b[128]; snprintf(b, sizeof b, "num_privileged_obs (%d) != the number of privileged observations (%d)", c->num_priv_obs, p); return fail(b); }
    return 0;
}

extern "C" int go1_sim_create(const Go1SimConfig* cfg, const float* actuator_weights, int device, Go1Sim** out) {
    if (!out) return fail("null out");
    *out = nullptr;
    if (int e = check_cfg(cfg)) return e;
    int n = 0;
    cudaError_t ce = cudaGetDeviceCount(&n);
    if (ce != cudaSuccess || n == 0) { cudaGetLastError(); return fail("no CUDA device: libgo1b200 has no CPU fallback"); }
    if (device < 0 || device >= n) return fail("bad device index");
    if ((ce = cudaSetDevice(device)) != cudaSuccess) return cuda_fail("cudaSetDevice", ce);
    Go1Sim* s = new Go1Sim();
    memset(&s->bufs, 0, sizeof(s->bufs));
    s->cfg = *cfg; s->bound = 0; s->device = device; s->d_tab = nullptr;
    memset(&s->self, 0, sizeof(s->self)); s->stepped = 0;
    go1_asset_defaults(&s->asset);
    if (int e = build_table(cfg, actuator_weights, &s->h_tab)) { delete s; return e; }
    if ((ce = cudaMalloc(&s->d_tab, sizeof(Go1DevTable))) != cudaSuccess) { delete s; return cuda_fail("cudaMalloc table", ce); }
    if ((ce = cudaMemcpy(s->d_tab, &s->h_tab, sizeof(Go1DevTable), cudaMemcpyHostToDevice)) != cudaSuccess) { cudaFree(s->d_tab); delete s; return cuda_fail("upload table", ce); }
    *out = s;
    return 0;
}

extern "C" int go1_sim_destroy(Go1Sim* s) {
    if (!s) return 0;
    cudaSetDevice(s->device);
    if (s->d_tab) cudaFree(s->d_tab);
    delete s;
    return 0;
}

extern "C" int go1_sim_bind(Go1Sim* s, const Go1SimBuffers* b) {
    if (!s || !b) return fail("null argument");
    if (!b->env_f32 || !b->leg_f32 || !b->env_i32 || !b->obs || !b->rew || !b->reset || !b->time_out || !b->event_count || !b->events || !b->episode_acc)
        return fail("go1_sim_bind: a required buffer is NULL");
    if (s->cfg.num_priv_obs > 0 && !b->priv_obs) return fail("go1_sim_bind: priv_obs is NULL");
    s->bufs = *b; s->bound = 1;
    return 0;
}

extern "C" int go1_sim_update_config(Go1Sim* s, const Go1SimConfig* cfg, void* stream) {
    if (!s) return fail("null sim");
    if (int e = check_cfg(cfg)) return e;
    if (cfg->num_envs != s->cfg.num_envs) return fail("num_envs cannot change");
    s->cfg = *cfg; s->h_tab.cfg = *cfg;
    cudaError_t ce = cudaMemcpyAsync(&s->d_tab->cfg, &s->h_tab.cfg, sizeof(Go1SimConfig), cudaMemcpyHostToDevice, (cudaStream_t)stream);
    if (ce != cudaSuccess) return cuda_fail("update config", ce);
    return 0;
}

extern "C" int go1_sim_set_self_collision(Go1Sim* s, const Go1SelfCollision* sc) {
    if (!s || !sc) return fail("go1_sim_set_self_collision: null argument");
    if (s->stepped) return fail("go1_sim_set_self_collision: the self-collision model cannot change after the first go1_sim_step");
    if (sc->enabled && !(sc->k >= 0.f && sc->c >= 0.f && sc->thigh_radius > 0.f && sc->calf_radius > 0.f && sc->foot_radius > 0.f))
        return fail("go1_sim_set_self_collision: k and c must be >= 0 and the radii > 0");
    s->self = *sc;
    return 0;
}

extern "C" int go1_sim_set_asset_options(Go1Sim* s, const Go1AssetOptions* o) {
    if (!s || !o) return fail("go1_sim_set_asset_options: null argument");
    if (s->stepped) return fail("go1_sim_set_asset_options: the asset options cannot change after the first go1_sim_step");
    for (int b = 0; b < GO1_NUM_BODIES; b++)
        if (!(isfinite(o->penalty_weight[b]) && o->penalty_weight[b] >= 0.f)) return fail("go1_sim_set_asset_options: penalty weights must be finite and >= 0");
    if (o->termination_mask >> GO1_NUM_BODIES) return fail("go1_sim_set_asset_options: termination_mask has bits above body 16");
    if (!(isfinite(o->armature) && o->armature >= 0.f)) return fail("go1_sim_set_asset_options: armature must be finite and >= 0");
    s->asset = *o;
    s->asset.fix_base = o->fix_base ? 1 : 0; s->asset.disable_gravity = o->disable_gravity ? 1 : 0;
    return 0;
}

extern "C" int go1_sim_step(Go1Sim* s, const float* actions, const float gravity[3], const float gravity_vec[3],
                            int64_t common_step, int mode, void* stream) {
    if (!s || !s->bound) return fail("go1_sim_step: sim not bound");
    if (!actions) return fail("go1_sim_step: null actions");
    if (mode < 0 || mode > 2) return fail("go1_sim_step: bad mode");
    for (int k = 0; k < 3; k++) s->gravity[k] = gravity[k];
    s->stepped = 1;
    int e = go1_launch_step(&s->bufs, s->d_tab, &s->self, &s->asset, actions, gravity, gravity_vec, (long long)common_step, mode, s->cfg.num_envs, nullptr, (cudaStream_t)stream);
    return e ? cuda_fail("go1_sim_step launch", e) : 0;
}

extern "C" int go1_sim_step_deferred(Go1Sim* s, const float* actions, const float gravity[3], const float gravity_vec[3],
                                     int64_t common_step, float* pre_roll, void* stream) {
    if (!s || !s->bound) return fail("go1_sim_step_deferred: sim not bound");
    if (!actions || !pre_roll) return fail("go1_sim_step_deferred: null actions / pre_roll");
    for (int k = 0; k < 3; k++) s->gravity[k] = gravity[k];
    s->stepped = 1;
    int e = go1_launch_step(&s->bufs, s->d_tab, &s->self, &s->asset, actions, gravity, gravity_vec, (long long)common_step, 0, s->cfg.num_envs, pre_roll, (cudaStream_t)stream);
    return e ? cuda_fail("go1_sim_step_deferred launch", e) : 0;
}

extern "C" int64_t go1_reward_finish_workspace(int num_envs, int K) {
    return (num_envs <= 0 || K < 0) ? 0 : (int64_t)go1_reward_finish_workspace_floats(num_envs, K);
}

extern "C" int go1_sim_reward_finish(Go1Sim* s, const float* raw, const float* scales, int K, float* user_sums, float* workspace, void* stream) {
    if (!s || !s->bound) return fail("go1_sim_reward_finish: sim not bound");
    if (K < 1 || K > GO1_MAX_USER_REWARDS) return fail("go1_sim_reward_finish: K must be in 1..GO1_MAX_USER_REWARDS");
    if (!raw || !scales || !user_sums || !workspace) return fail("go1_sim_reward_finish: null argument");
    int e = go1_launch_reward_finish(&s->bufs, &s->cfg, raw, scales, K, user_sums, workspace, s->cfg.num_envs, (cudaStream_t)stream);
    return e ? cuda_fail("go1_sim_reward_finish launch", e) : 0;
}

extern "C" int go1_sim_user_reward_fold(Go1Sim* s, const int32_t* env_ids, const int32_t* k_dev, int k, int K, float* user_sums,
                                        float* user_sums_eval, float* acc, float* acc_hist, int T, const int32_t* slot_dev, void* stream) {
    if (!s || !s->bound) return fail("go1_sim_user_reward_fold: sim not bound");
    if (K < 1 || K > GO1_MAX_USER_REWARDS) return fail("go1_sim_user_reward_fold: K must be in 1..GO1_MAX_USER_REWARDS");
    if (!env_ids || !user_sums || !acc || (!k_dev && (k < 0 || k > s->cfg.num_envs))) return fail("go1_sim_user_reward_fold: bad arguments");
    if (acc_hist && (T <= 0 || !slot_dev)) return fail("go1_sim_user_reward_fold: acc_hist needs T > 0 and slot_dev");
    int e = go1_launch_user_reward_fold(env_ids, k_dev, k, K, user_sums, user_sums_eval, acc, acc_hist, T, slot_dev,
                                        s->cfg.num_train_envs, s->cfg.num_envs, (cudaStream_t)stream);
    return e ? cuda_fail("go1_sim_user_reward_fold launch", e) : 0;
}

extern "C" int go1_sim_reset_idx(Go1Sim* s, const int32_t* env_ids, int k, const float* new_commands, const float* actions,
                                 int post_step, int64_t common_step, void* stream) {
    if (!s || !s->bound) return fail("go1_sim_reset_idx: sim not bound");
    if (k < 0 || k > s->cfg.num_envs) return fail("go1_sim_reset_idx: bad k");
    if (k == 0) return 0;
    if (!env_ids || !new_commands) return fail("go1_sim_reset_idx: null ids/commands");
    int e = go1_launch_reset(&s->bufs, s->d_tab, env_ids, k, new_commands, actions, post_step, (long long)common_step, s->gravity, s->asset.fix_base, s->cfg.num_envs, (cudaStream_t)stream);
    return e ? cuda_fail("go1_sim_reset_idx launch", e) : 0;
}

extern "C" int go1_sim_set_commands(Go1Sim* s, const int32_t* env_ids, int k, const float* new_commands, void* stream) {
    if (!s || !s->bound) return fail("go1_sim_set_commands: sim not bound");
    if (k == 0) return 0;
    if (k < 0 || !env_ids || !new_commands) return fail("go1_sim_set_commands: bad arguments");
    int e = go1_launch_set_commands(&s->bufs, env_ids, k, new_commands, s->cfg.num_envs, (cudaStream_t)stream);
    return e ? cuda_fail("go1_sim_set_commands launch", e) : 0;
}

extern "C" int go1_sizeof_curriculum(int which) { return which == 0 ? (int)sizeof(Go1CurriculumConfig) : (int)sizeof(Go1CurriculumBuffers); }

extern "C" int go1_curriculum_resample(Go1Sim* s, const Go1CurriculumConfig* cfg, const Go1CurriculumBuffers* cb, int list, void* stream) {
    if (!s || !s->bound) return fail("go1_curriculum_resample: sim not bound");
    if (!cfg || !cb || list < 0 || list > 1) return fail("go1_curriculum_resample: bad arguments");
    if (cfg->num_categories < 1 || cfg->num_categories > GO1_CUR_MAX_CATEGORIES || cfg->num_bins < 1 || cfg->num_dims < 1 ||
        cfg->num_task_keys < 0 || cfg->num_task_keys > 4 || cfg->num_commands < 1 || cfg->num_commands > GO1_NUM_COMMANDS)
        return fail("go1_curriculum_resample: bad curriculum config");
    if (!cb->weights || !cb->grid || !cb->half_bins || !cb->local_range || !cb->mt || !cb->cat_rng || !cb->env_bins || !cb->env_categories ||
        !cb->env_bins_f32 || !cb->cdf || !cb->cdf_valid || !cb->scratch_i32 || !cb->scratch_u32 || !cb->scratch_f64 || !cb->out_count ||
        !cb->out_ids || !cb->out_commands || (cfg->snapshot_time_outs && !cb->time_outs_snapshot))
        return fail("go1_curriculum_resample: null buffer");
    if (cfg->xr_world > 1) {
        if (cfg->xr_world > GO1_CUR_MAX_CATEGORIES || cfg->xr_rank < 0 || cfg->xr_rank >= cfg->xr_world || cfg->xr_cap < s->cfg.num_envs)
            return fail("go1_curriculum_resample: bad cross-rank configuration (xr_world <= 8, 0 <= xr_rank < xr_world, xr_cap >= num_envs)");
        if (!cb->xr_events || !cb->xr_ids || !cb->xr_commands) return fail("go1_curriculum_resample: cross-rank replay needs xr_events / xr_ids / xr_commands");
    }
    int e = go1_launch_curriculum(&s->bufs, cfg, cb, list, s->cfg.num_envs, (cudaStream_t)stream);
    return e ? cuda_fail("go1_curriculum_resample launch", e) : 0;
}

extern "C" int go1_curriculum_pack(Go1Sim* s, const Go1CurriculumConfig* cfg, const Go1CurriculumBuffers* cb, void* stream) {
    if (!s || !s->bound) return fail("go1_curriculum_pack: sim not bound");
    if (!cfg || !cb || cfg->xr_world < 2 || !cb->xr_send || !cb->env_bins || !cb->env_categories || cfg->xr_cap < s->cfg.num_envs)
        return fail("go1_curriculum_pack: bad arguments");
    int e = go1_launch_curriculum_pack(&s->bufs, cfg, cb, s->cfg.num_envs, (cudaStream_t)stream);
    return e ? cuda_fail("go1_curriculum_pack launch", e) : 0;
}

extern "C" int go1_sim_reset_idx_dev(Go1Sim* s, const int32_t* env_ids, const int32_t* k_dev, const float* new_commands, const float* actions,
                                     int post_step, int64_t common_step, float* episode_acc, void* stream) {
    if (!s || !s->bound) return fail("go1_sim_reset_idx_dev: sim not bound");
    if (!env_ids || !k_dev || !new_commands) return fail("go1_sim_reset_idx_dev: null ids/count/commands");
    int e = go1_launch_reset_dev(&s->bufs, s->d_tab, env_ids, k_dev, new_commands, actions, post_step, (long long)common_step, s->gravity,
                                 episode_acc, s->asset.fix_base, s->cfg.num_envs, (cudaStream_t)stream);
    return e ? cuda_fail("go1_sim_reset_idx_dev launch", e) : 0;
}

extern "C" int go1_history_roll(const float* hist_in, const float* obs, float* hist_out, int n, int num_obs, int history_len, void* stream) {
    if (!hist_in || !obs || !hist_out || n <= 0 || num_obs <= 0 || history_len <= 0) return fail("go1_history_roll: bad arguments");
    int e = go1_launch_history_roll(hist_in, obs, hist_out, n, num_obs, history_len, (cudaStream_t)stream);
    return e ? cuda_fail("go1_history_roll launch", e) : 0;
}

extern "C" int go1_history_roll_pitched(const float* hist_in, int ld_in, const float* obs, float* hist_out, int ld_out, int n, int num_obs,
                                        int history_len, void* stream) {
    if (!hist_in || !obs || !hist_out) return fail("go1_history_roll_pitched: null pointer");
    if (n <= 0 || num_obs <= 0 || history_len <= 0 || (long long)num_obs * history_len > (1 << 30))
        return fail("go1_history_roll_pitched: n, num_obs and history_len must be positive (num_obs * history_len <= 2^30)");
    const int nhist = num_obs * history_len;
    if (ld_in < nhist || ld_out < nhist || (ld_in & 3) || (ld_out & 3)) {
        char b[160];
        snprintf(b, sizeof b, "go1_history_roll_pitched: row pitches (ld_in %d, ld_out %d) must be >= num_obs * history_len (%d) and multiples of 4",
                 ld_in, ld_out, nhist);
        return fail(b);
    }
    if ((((uintptr_t)hist_in) | ((uintptr_t)hist_out)) & 15) return fail("go1_history_roll_pitched: hist_in and hist_out must be 16-byte aligned");
    int e = go1_launch_history_roll_pitched(hist_in, ld_in, obs, hist_out, ld_out, n, num_obs, history_len, (cudaStream_t)stream);
    return e ? cuda_fail("go1_history_roll_pitched launch", e) : 0;
}
