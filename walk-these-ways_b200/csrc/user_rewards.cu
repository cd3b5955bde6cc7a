// user_rewards.cu — the kernels around user reward terms (go1_gym/envs/rewards, DESIGN.md §4).  A step with user terms runs
// go1_step_kernel<SELF, true> (sim_step_defer.cu), the terms in torch, then the two kernels of go1_launch_reward_finish here; after
// the reset launches, go1_user_reward_fold_kernel files and clears the user episode sums of the reset envs.
#include <cuda_runtime.h>
#include <math.h>
#include "go1_layout.h"
void go1_count_launch(int n);

namespace {

constexpr int kThreads = 256;

struct FinishArgs {
    Go1SimBuffers b;
    const float* raw;           // [K][N] user term values
    float* user_sums;           // [K][N] their episode sums
    float* partials;            // [blocks][K] per-CTA sums of raw * scale
    int N, K;
    int only_positive, ji22;
    float sigma_rew_neg, term_scale;
    float scale[GO1_MAX_USER_REWARDS];
};

// Sum of v over the CTA in a fixed order (warp tree, then the warps in index order); the result is valid in thread 0.
__device__ float block_sum(float v, float* s_warp) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();            // s_warp may still be read by the previous call
    if (lane == 0) s_warp[warp] = v;
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x == 0)
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) t += s_warp[w];
    return t;
}

// The sign test of legged_robot.py:275-278 needs each user term's sum over all envs: one partial per CTA and term.
__global__ void __launch_bounds__(kThreads) go1_reward_partials_kernel(const FinishArgs a) {
    __shared__ float s_warp[kThreads / 32];
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    for (int k = 0; k < a.K; k++) {
        const float v = env < a.N ? __fmul_rn(a.raw[(size_t)k * a.N + env], a.scale[k]) : 0.f;
        const float t = block_sum(v, s_warp);
        if (threadIdx.x == 0) a.partials[(size_t)blockIdx.x * a.K + k] = t;
    }
}

// Every CTA sums the partials in CTA order (so all agree on the signs), then finishes compute_reward for its envs.
__global__ void __launch_bounds__(kThreads) go1_reward_finish_kernel(const FinishArgs a) {
    __shared__ int s_sign[GO1_MAX_USER_REWARDS];
    const int nblk = gridDim.x;
    if ((int)threadIdx.x < a.K) {
        float s = 0.f;
        for (int j = 0; j < nblk; j++) s += a.partials[(size_t)j * a.K + threadIdx.x];
        s_sign[threadIdx.x] = (s >= 0.f) ? 1 : ((s <= 0.f) ? -1 : 0);     // NaN: neither
    }
    __syncthreads();
    const int env = blockIdx.x * blockDim.x + threadIdx.x, N = a.N;
    if (env >= N) return;
    float* ef = a.b.env_f32;
    float& pos_ref = ef[(size_t)EROW(rew_buf_pos) * N + env];
    float& neg_ref = ef[(size_t)EROW(rew_buf_neg) * N + env];
    float rew = a.b.rew[env], pos = pos_ref, neg = neg_ref;
    for (int k = 0; k < a.K; k++) {
        const float r = __fmul_rn(a.raw[(size_t)k * N + env], a.scale[k]);
        rew += r;
        if (s_sign[k] > 0) pos += r;
        else if (s_sign[k] < 0) neg += r;
        a.user_sums[(size_t)k * N + env] += r;
    }
    if (a.only_positive) rew = fmaxf(rew, 0.f);
    else if (a.ji22) rew = pos * expf(neg / a.sigma_rew_neg);
    const float total_for_sum = rew;
    if (a.term_scale != 0.f) {
        const float r = ((a.b.reset[env] && !a.b.time_out[env]) ? 1.f : 0.f) * a.term_scale;
        rew += r;
        ef[(size_t)(EROW(episode_sums) + GO1_REW_TERMINATION) * N + env] += r;
        ef[(size_t)(EROW(command_sums) + GO1_REW_TERMINATION) * N + env] += r;
    }
    ef[(size_t)(EROW(episode_sums) + GO1_NUM_REWARD_TERMS) * N + env] += total_for_sum;      // "total"
    pos_ref = pos; neg_ref = neg;
    a.b.rew[env] = rew;
}

// One CTA over the reset list: fixed summation order, and the per-step history row needs no grid-wide completion.
__global__ void __launch_bounds__(kThreads) go1_user_reward_fold_kernel(const int* ids, const int* k_dev, int k, int K, float* user_sums,
                                                                        float* user_sums_eval, float* acc, float* acc_hist, int T,
                                                                        const int* slot_dev, int num_train, int N) {
    __shared__ float s_warp[kThreads / 32];
    __shared__ float s_acc[GO1_MAX_USER_REWARDS + 1];
    const int n = k_dev ? *k_dev : k;
    for (int t = 0; t <= K; t++) {
        float v = 0.f;
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const int env = ids[i];
            if (t == K) { v += env < num_train ? 1.f : 0.f; continue; }
            float* s = user_sums + (size_t)t * N + env;
            if (env < num_train) v += *s;
            else if (user_sums_eval) {          // the first finished episode of an eval env is kept (legged_robot.py:188-195)
                float* e = user_sums_eval + (size_t)t * N + env;
                if (*e == -1.0f) *e = *s;
            }
            *s = 0.f;
        }
        const float tot = block_sum(v, s_warp);
        if (threadIdx.x == 0) s_acc[t] = tot;
    }
    __syncthreads();
    if ((int)threadIdx.x <= K) {
        const float v = s_acc[threadIdx.x];
        acc[threadIdx.x] = v;
        if (acc_hist) {
            const int slot = *slot_dev, W = K + 1;
            acc_hist[(size_t)slot * W + threadIdx.x] = s_acc[K] == 0.f ? acc_hist[(size_t)((slot + T - 1) % T) * W + threadIdx.x] : v;
        }
    }
}

}  // namespace

extern "C" long long go1_reward_finish_workspace_floats(int N, int K) { return (long long)((N + kThreads - 1) / kThreads) * K; }

extern "C" int go1_launch_reward_finish(const Go1SimBuffers* b, const Go1SimConfig* cfg, const float* raw, const float* scales, int K,
                                        float* user_sums, float* workspace, int N, cudaStream_t st) {
    FinishArgs a;
    a.b = *b; a.raw = raw; a.user_sums = user_sums; a.partials = workspace; a.N = N; a.K = K;
    a.only_positive = cfg->only_positive_rewards; a.ji22 = cfg->only_positive_rewards_ji22_style;
    a.sigma_rew_neg = cfg->sigma_rew_neg; a.term_scale = cfg->reward_scale[GO1_REW_TERMINATION];
    for (int k = 0; k < GO1_MAX_USER_REWARDS; k++) a.scale[k] = k < K ? scales[k] : 0.f;
    const int blocks = (N + kThreads - 1) / kThreads;
    go1_reward_partials_kernel<<<blocks, kThreads, 0, st>>>(a); go1_count_launch(1);
    go1_reward_finish_kernel<<<blocks, kThreads, 0, st>>>(a); go1_count_launch(1);
    return (int)cudaGetLastError();
}

extern "C" int go1_launch_user_reward_fold(const int* ids, const int* k_dev, int k, int K, float* user_sums,
                                           float* user_sums_eval, float* acc, float* acc_hist, int T, const int* slot_dev, int num_train,
                                           int N, cudaStream_t st) {
    go1_user_reward_fold_kernel<<<1, kThreads, 0, st>>>(ids, k_dev, k, K, user_sums, user_sums_eval, acc, acc_hist, T, slot_dev, num_train, N);
    go1_count_launch(1);
    return (int)cudaGetLastError();
}
