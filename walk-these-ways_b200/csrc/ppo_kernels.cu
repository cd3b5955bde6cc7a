// ppo_kernels.cu — learner-side kernels of go1_gym_learn/ppo_cse for sm_90a:
//   GAE warp-scan (rollout_storage.py:74-88), fp32 CUDA-core GEMM with fused bias/activation epilogue (the
//   exact-fp32 path next to the wgmma TF32 path in gemm_tf32.cu), activation backward, column sums, Normal
//   sampling/log-prob (actor_critic.py:113-126), PPO loss + gradients (ppo.py:113-152), MSE
//   (ppo.py:168-186), global grad-norm + clip + Adam (ppo.py:155-158), row gather
//   (rollout_storage.py:98-137).
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "../../include/go1_b200.h"
#include "sim_math.cuh"
#include "activation.cuh"
#include "deterministic.cuh"
void go1_count_launch(int n);

extern int go1_set_error(const char* m);
static int cuda_rc(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) return 0;
    char buf[256];
    snprintf(buf, sizeof buf, "%s: %s", what, cudaGetErrorString(e));
    go1_set_error(buf);
    return (int)e;
}

// ---------------------------------------------------------------------------------------------
// GAE: A_t = delta_t + c_t A_{t+1} is a scan over affine maps x -> b + a x.  One warp per env, lanes = time
// steps (reversed), composed with a 5-step Kogge-Stone shuffle scan; tiles of 32 envs are staged through
// shared memory so global loads/stores stay coalesced along the env axis.  T <= 32 per pass; longer
// rollouts chain passes through the carry.
// ---------------------------------------------------------------------------------------------
// DET (deterministic mode, go1_set_deterministic): stats is the workspace, and the block's two statistics go to stats[2 blockIdx.x ..]
template <bool DET>
__global__ void __launch_bounds__(1024) gae_kernel(const float* __restrict__ rew, const uint8_t* __restrict__ done,
                                                   const float* __restrict__ val, const float* __restrict__ last_val,
                                                   float* __restrict__ ret, float* __restrict__ adv, double* __restrict__ stats,
                                                   int T, int n, float gamma, float lam) {
    __shared__ float s_a[32][33], s_b[32][33], s_v[32][33];
    __shared__ double s_red[2][32];
    const int lane = threadIdx.x, w = threadIdx.y;        // block = (32, 32)
    const int env0 = blockIdx.x * 32;
    double lsum = 0.0, lsq = 0.0;
    float carry = 0.f;                                     // A_{t+1} entering the current chunk (per env = per warp)
    for (int t_hi = T; t_hi > 0; t_hi -= 32) {
        const int t_lo = max(t_hi - 32, 0), len = t_hi - t_lo;
        // load: thread (lane = env offset, w = time offset) -> coalesced over envs
        {
            const int t = t_lo + w, e = env0 + lane;
            float a = 0.f, b = 0.f, v = 0.f;
            if (w < len && e < n) {
                const size_t i = (size_t)t * n + e;
                v = val[i];
                const float nv = (t == T - 1) ? last_val[e] : val[i + n];
                const float nt = 1.0f - (float)done[i];
                b = rew[i] + nt * gamma * nv - v;          // delta_t
                a = nt * gamma * lam;                      // c_t
            }
            s_a[w][lane] = a; s_b[w][lane] = b; s_v[w][lane] = v;
        }
        __syncthreads();
        // scan: warp w = env offset, lane j = reversed time (j = 0 is the last step of the chunk)
        {
            const int tt = len - 1 - lane;
            float a = (lane < len) ? s_a[tt][w] : 1.f, b = (lane < len) ? s_b[tt][w] : 0.f;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const float ap = __shfl_up_sync(0xffffffffu, a, d), bp = __shfl_up_sync(0xffffffffu, b, d);
                if (lane >= d) { b = b + a * bp; a = a * ap; }
            }
            const float A = b + a * carry;                 // advantage at time t_lo + tt
            if (lane < len) s_b[tt][w] = A;
            carry = __shfl_sync(0xffffffffu, A, len - 1);  // A at t_lo feeds the next (earlier) chunk
        }
        __syncthreads();
        {
            const int t = t_lo + w, e = env0 + lane;
            if (w < len && e < n) {
                const size_t i = (size_t)t * n + e;
                const float A = s_b[w][lane];
                ret[i] = A + s_v[w][lane];
                adv[i] = A;                                // == returns - values (rollout_storage.py:87)
                lsum += (double)A; lsq += (double)A * (double)A;
            }
        }
        __syncthreads();
    }
    // block reduce of the statistics
    for (int d = 16; d > 0; d >>= 1) { lsum += __shfl_xor_sync(0xffffffffu, lsum, d); lsq += __shfl_xor_sync(0xffffffffu, lsq, d); }
    if (lane == 0) { s_red[0][w] = lsum; s_red[1][w] = lsq; }
    __syncthreads();
    if (w == 0) {
        double a = s_red[0][lane], b = s_red[1][lane];
        for (int d = 16; d > 0; d >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, d); b += __shfl_xor_sync(0xffffffffu, b, d); }
        if (lane == 0) {
            if constexpr (DET) { stats[2 * blockIdx.x] = a; stats[2 * blockIdx.x + 1] = b; }
            else { atomicAdd(stats, a); atomicAdd(stats + 1, b); }
        }
    }
}
__global__ void normalize_adv_kernel(float* __restrict__ adv, const double* __restrict__ stats, long long global_count, long long local_count) {
    const double mean = stats[0] / (double)global_count;
    const double var = (stats[1] - (double)global_count * mean * mean) / (double)(global_count - 1);   // unbiased (torch.std)
    const float m = (float)mean, inv = 1.0f / ((float)sqrt(fmax(var, 0.0)) + 1e-8f);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < local_count; i += (long long)gridDim.x * blockDim.x)
        adv[i] = (adv[i] - m) * inv;
}

extern "C" int go1_ppo_gae(const float* rewards, const uint8_t* dones, const float* values, const float* last_values,
                           float* returns, float* advantages, double* stats, int T, int n, float gamma, float lam, void* stream) {
    if (!rewards || !dones || !values || !last_values || !returns || !advantages || !stats || T <= 0 || n <= 0) return go1_set_error("go1_ppo_gae: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    const int nb = (n + 31) / 32;
    const bool det = go1_det_on();     // deterministic mode: the blocks' statistics meet in stats in block order
    double* out = go1_det_out(det, st, 2 * (size_t)nb, stats);
    if (det && !out) return 1;
    if (!det) cudaMemsetAsync(stats, 0, 2 * sizeof(double), st);
    (det ? gae_kernel<true> : gae_kernel<false>)<<<nb, dim3(32, 32), 0, st>>>(rewards, dones, values, last_values, returns, advantages, out, T, n, gamma, lam);
    go1_count_launch(1);
    if (int e = cuda_rc("go1_ppo_gae")) return e;
    return det ? go1_det_sum64(out, nb, 2, stats, 2, 0, st) : 0;
}
extern "C" int go1_ppo_normalize_advantages(float* advantages, const double* stats, int64_t global_count, int64_t local_count, void* stream) {
    if (!advantages || !stats || global_count < 2 || local_count <= 0) return go1_set_error("go1_ppo_normalize_advantages: bad arguments");
    normalize_adv_kernel<<<296, 256, 0, (cudaStream_t)stream>>>(advantages, stats, global_count, local_count); go1_count_launch(1);
    return cuda_rc("go1_ppo_normalize_advantages");
}

// ---------------------------------------------------------------------------------------------
// fp32 CUDA-core GEMM: C[M][N] (+)= opA(A) opB(B) (+ bias[n]) with optional activation (Go1Activation `kind`, activation.cuh).
//   TA == 0: A is [M][K] (lda), TA == 1: A is [K][M];  TB == 0: B is [K][N] (ldb), TB == 1: B is [N][K].
// 128x128x8 tiles, 256 threads, 8x8 register micro-tiles; split-K over gridDim.z with atomicAdd.
// ---------------------------------------------------------------------------------------------
// The exact-fp32 kernels apply the activation per element inside unrolled loops: ELU stays inline (the configured default), the other
// kinds share one out-of-line copy of their libm code.
__device__ __noinline__ float act_exact_other(int kind, float v) {
    GO1_ACT_SWITCH(kind, KD, return act_exact<KD>(v);)
    return v;
}
DI float act_exact_rt(int kind, float v) { return kind == GO1_ACT_ELU ? act_exact<GO1_ACT_ELU>(v) : act_exact_other(kind, v); }
DI float act_deriv_rt(int kind, float y) {
    GO1_ACT_SWITCH(kind, KD, return act_deriv<KD>(y);)
    return 1.0f;
}
// entry points that take a bare `int act`: mode in bits 0..7, Go1Activation above (GO1_ACT)
static inline int act_mode(int act) { return act & 0xff; }
static inline int act_kind(int act) { return act >> 8; }

struct SgemmEp { const float* ex; const float* wex; const float* aux; int ldex, ldwex, nex, ldaux; };

// DET: a split's partial tile goes to part[split][M][N] (plain stores; go1_det_sum adds the splits into C)
template <int TA, int TB, bool DET>
__global__ void __launch_bounds__(256) sgemm_kernel(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb,
                                                    float* __restrict__ Cm, int ldc, const float* __restrict__ bias,
                                                    int M, int N, int K, int act, int kind, int accumulate, int kchunk, const SgemmEp ep, float* __restrict__ part) {
    constexpr int BM = 128, BN = 128, BK = 8;
    __shared__ float As[2][BK][BM + 4], Bs[2][BK][BN + 4];
    const int tid = threadIdx.x;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int kbeg = blockIdx.z * kchunk, kend = min(K, kbeg + kchunk);
    const int tx = tid & 15, ty = tid >> 4;                 // 16 x 16 threads, each 8 (m) x 8 (n)
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < 8; j++) acc[i][j] = 0.f;

    auto load_tile = [&](int buf, int k0) {
        // A tile: BM x BK
        if (TA == 0) {      // A[m][k]: thread -> (m = tid/2, k half = tid%2 * 4 .. +4)
            const int m = tid >> 1, kk = (tid & 1) * 4;
            const int gm = m0 + m;
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const int gk = k0 + kk + c;
                As[buf][kk + c][m] = (gm < M && gk < kend) ? A[(size_t)gm * lda + gk] : 0.f;
            }
        } else {            // A[k][m]: thread -> (k = tid/32, m = (tid%32)*4 .. +4), coalesced over m
            const int kk = tid >> 5, m = (tid & 31) * 4;
            const int gk = k0 + kk;
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const int gm = m0 + m + c;
                As[buf][kk][m + c] = (gm < M && gk < kend) ? A[(size_t)gk * lda + gm] : 0.f;
            }
        }
        if (TB == 1) {      // B[n][k]
            const int n = tid >> 1, kk = (tid & 1) * 4;
            const int gn = n0 + n;
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const int gk = k0 + kk + c;
                Bs[buf][kk + c][n] = (gn < N && gk < kend) ? B[(size_t)gn * ldb + gk] : 0.f;
            }
        } else {            // B[k][n]
            const int kk = tid >> 5, n = (tid & 31) * 4;
            const int gk = k0 + kk;
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const int gn = n0 + n + c;
                Bs[buf][kk][n + c] = (gn < N && gk < kend) ? B[(size_t)gk * ldb + gn] : 0.f;
            }
        }
    };

    int buf = 0;
    if (kbeg < kend) load_tile(0, kbeg);
    __syncthreads();
    for (int k0 = kbeg; k0 < kend; k0 += BK) {
        if (k0 + BK < kend) load_tile(buf ^ 1, k0 + BK);
#pragma unroll
        for (int kk = 0; kk < BK; kk++) {
            float a[8], b[8];
            const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
            a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
            b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
#pragma unroll
            for (int i = 0; i < 8; i++)
#pragma unroll
                for (int j = 0; j < 8; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
        buf ^= 1;
    }
    const bool split = gridDim.z > 1;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int gm = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
        if (gm >= M) continue;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int gn = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
            if (gn >= N) continue;
            float* c = Cm + (size_t)gm * ldc + gn;
            float v = acc[i][j];
            if (split) {
                if (DET) part[((size_t)blockIdx.z * M + gm) * N + gn] = v;
                else atomicAdd(c, v);      // caller pre-initialised C (zero or accumulate target)
                continue;
            }
            if (accumulate) v += *c;
            for (int t = 0; t < ep.nex; t++) v = fmaf(ep.ex[(size_t)gm * ep.ldex + t], ep.wex[(size_t)gn * ep.ldwex + t], v);
            if (bias) v += bias[gn];
            if (act == 1) v = act_exact_rt(kind, v);
            else if (act == 2) { const float y = ep.aux[(size_t)gm * ep.ldaux + gn]; v *= act_deriv_rt(kind, y); }
            *c = v;
        }
    }
}

__global__ void bias_act_kernel(float* __restrict__ Cm, int ldc, const float* __restrict__ bias, int M, int N, int act, int kind) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)M * N) return;
    const int m = (int)(i / N), n = (int)(i - (size_t)m * N);
    float v = Cm[(size_t)m * ldc + n];
    if (bias) v += bias[n];
    if (act == 1) v = act_exact_rt(kind, v);
    Cm[(size_t)m * ldc + n] = v;
}
__global__ void zero_strided_kernel(float* __restrict__ Cm, int ldc, int M, int N) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)M * N) return;
    const int m = (int)(i / N), n = (int)(i - (size_t)m * N);
    Cm[(size_t)m * ldc + n] = 0.f;
}

extern "C" int go1_gemm_tf32(int transA, int transB, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
                             float* Cm, int ldc, const Go1GemmEpilogue* ep, cudaStream_t st);

extern "C" int go1_gemm_ex(int transA, int transB, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
                           float* Cm, int ldc, const Go1GemmEpilogue* epi, int impl, void* stream) {
    if (!A || !B || !epi || (!Cm && !epi->out_bf16) || M <= 0 || N <= 0 || K <= 0) return go1_set_error("go1_gemm: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    if (epi->act < 0 || epi->act > 2) return go1_set_error("go1_gemm_ex: act must be 0, 1 or 2");
    if (!go1_act_kind_ok(epi->act_kind)) return go1_set_error("go1_gemm_ex: unknown activation kind (Go1Activation)");
    if (impl == 1) return go1_gemm_tf32(transA, transB, M, N, K, A, lda, B, ldb, Cm, ldc, epi, st);
    if (impl != 0) return go1_set_error("go1_gemm: unknown impl");
    if (epi->lead_cols > 0) return go1_set_error("go1_gemm_ex: lead_cols is implemented by impl 1 only");
    if (epi->colsum || epi->num_bwd_extra > 0) return go1_set_error("go1_gemm_ex: the fused column sum / trailing-input backward are implemented by impl 1 only");
    if (epi->store_transposed || epi->out_bf16) return go1_set_error("go1_gemm_ex: store_transposed / out_bf16 are implemented by impl 1 only");
    const float* bias = epi->bias; const int act = epi->act, kind = epi->act_kind, accumulate = epi->accumulate;
    SgemmEp ep; ep.ex = epi->extra; ep.wex = epi->w_extra; ep.aux = epi->dact_y; ep.ldex = epi->ld_extra; ep.ldwex = epi->ld_w_extra;
    ep.nex = epi->extra ? epi->num_extra : 0; ep.ldaux = epi->ld_dact_y;
    if (ep.nex < 0 || ep.nex > 4) return go1_set_error("go1_gemm_ex: num_extra must be 0..4");
    if (act == 2 && !ep.aux) return go1_set_error("go1_gemm_ex: act 2 needs dact_y");
    const bool fused = ep.nex > 0 || act == 2;
    const int tiles = ((M + 127) / 128) * ((N + 127) / 128);
    int splitk = 1;
    if (tiles < 132 && K >= 2048 && !fused) { splitk = min((132 * 2 + tiles - 1) / tiles, (K + 255) / 256); if (splitk < 1) splitk = 1; }
    int kchunk = ((K + splitk - 1) / splitk + 7) / 8 * 8;
    splitk = (K + kchunk - 1) / kchunk;
    dim3 grid((N + 127) / 128, (M + 127) / 128, splitk);
    const bool det = splitk > 1 && go1_det_on();      // deterministic mode: the splits' partial tiles meet in C in split order
    float* part = go1_det_out<float>(det, st, (size_t)splitk * M * N, nullptr);
    if (det && !part) return 1;
    if (splitk > 1 && !accumulate && !det) {
        const size_t tot = (size_t)M * N;
        zero_strided_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(Cm, ldc, M, N); go1_count_launch(1);
    }
#define LAUNCH(TA, TB) (det ? sgemm_kernel<TA, TB, true> : sgemm_kernel<TA, TB, false>)<<<grid, 256, 0, st>>>(A, lda, B, ldb, Cm, ldc, bias, M, N, K, act, kind, accumulate, kchunk, ep, part)
    if (!transA && !transB) LAUNCH(0, 0); else if (!transA && transB) LAUNCH(0, 1); else if (transA && !transB) LAUNCH(1, 0); else LAUNCH(1, 1);
    go1_count_launch(1);
#undef LAUNCH
    if (det) {
        if (int e = cuda_rc("go1_gemm")) return e;
        if (int e = go1_det_sum(part, splitk, (size_t)M * N, Cm, M, N, ldc, accumulate, st)) return e;
    }
    if (splitk > 1 && (bias || act)) {
        const size_t tot = (size_t)M * N;
        bias_act_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(Cm, ldc, bias, M, N, act, kind); go1_count_launch(1);
    }
    return cuda_rc("go1_gemm");
}
extern "C" int go1_gemm(int transA, int transB, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
                        float* Cm, int ldc, const float* bias, int act, int accumulate, int impl, void* stream) {
    Go1GemmEpilogue ep;
    memset(&ep, 0, sizeof ep);
    if (act < 0) return go1_set_error("go1_gemm: bad act");
    ep.bias = bias; ep.act = act_mode(act); ep.act_kind = act_kind(act); ep.accumulate = accumulate;
    return go1_gemm_ex(transA, transB, M, N, K, A, lda, B, ldb, Cm, ldc, &ep, impl, stream);
}

// y = act(y + extra . w_extra^T) in place: the deferred trailing-input term + activation of a first layer.
// float4 variant (o % 4 == 0, 16-byte aligned rows): one thread = 4 consecutive columns, 4 row-strided elements in flight per thread;
// it finishes a wgmma product, so it uses the branch-free activations of that path (act_fast).  KIND < 0: no activation.
template <int KIND>
__global__ void __launch_bounds__(256) extra_fwd4_kernel(float* __restrict__ y, int ldy, const float* __restrict__ ex, int ldex, const float* __restrict__ wex, int ldw,
                                                         int M, int o4, int E, int rows_per_pass) {
    // blockDim.x = 256 threads = (256 / o4) rows x o4 column groups (o4 divides 256) or one row segment
    const int cg = threadIdx.x % o4, rsub = threadIdx.x / o4, rpb = blockDim.x / o4;
    float w[4][4];
#pragma unroll
    for (int c = 0; c < 4; c++)
#pragma unroll
        for (int t = 0; t < 4; t++) w[c][t] = t < E ? __ldg(wex + (size_t)(4 * cg + c) * ldw + t) : 0.f;
    for (int m0 = blockIdx.x * rpb * 4 + rsub; m0 < M; m0 += gridDim.x * rpb * 4) {
        float4 v[4]; float e[4][4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int m = m0 + u * rpb;
            if (m < M) {
                v[u] = *reinterpret_cast<const float4*>(y + (size_t)m * ldy + 4 * cg);
#pragma unroll
                for (int t = 0; t < 4; t++) e[u][t] = t < E ? __ldg(ex + (size_t)m * ldex + t) : 0.f;
            }
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int m = m0 + u * rpb;
            if (m < M) {
                float r[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    float a = r[c];
#pragma unroll
                    for (int t = 0; t < 4; t++) a = fmaf(e[u][t], w[c][t], a);
                    r[c] = KIND >= 0 ? act_fast<(KIND >= 0 ? KIND : 0)>(a) : a;
                }
                *reinterpret_cast<float4*>(y + (size_t)m * ldy + 4 * cg) = make_float4(r[0], r[1], r[2], r[3]);
            }
        }
    }
}
// generic variant: grid (column blocks of 256, row blocks of 8): each thread keeps its column's E weights in registers and walks 8 rows
__global__ void __launch_bounds__(256) extra_fwd_kernel(float* __restrict__ y, int ldy, const float* __restrict__ ex, int ldex, const float* __restrict__ wex, int ldw,
                                                        int M, int o, int E, int act, int kind) {
    const int n = blockIdx.x * 256 + threadIdx.x;
    if (n >= o) return;
    float w[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int t = 0; t < 4; t++) if (t < E) w[t] = __ldg(wex + (size_t)n * ldw + t);
    const int m0 = blockIdx.y * 8, m1 = min(M, m0 + 8);
#pragma unroll 8
    for (int m = m0; m < m1; m++) {
        float acc = 0.f;
#pragma unroll
        for (int t = 0; t < 4; t++) if (t < E) acc = fmaf(__ldg(ex + (size_t)m * ldex + t), w[t], acc);
        float v = y[(size_t)m * ldy + n] + acc;
        if (act == 1) v = act_exact_rt(kind, v);
        y[(size_t)m * ldy + n] = v;
    }
}
// Wide variant (4 < E <= 64, the privileged-observation widths): the CTA stages its 128-column tile of w_extra, transposed to [E][128],
// in shared memory once, and copies of its 32-row chunks of extra.  A warp walks rows (4 in flight), a lane owns 4 consecutive columns and
// reads the row's E extra values as shared-memory broadcasts.  VEC: float4 rows and act_fast, as extra_fwd4_kernel; otherwise scalar
// accesses and the libm forms, as extra_fwd_kernel.  KIND < 0: no activation.
constexpr int XWIDE_MAX_E = 64, XWIDE_COLS = 128, XWIDE_ROWS = 32;
template <int KIND, bool VEC>
__global__ void __launch_bounds__(256) extra_fwd_wide_kernel(float* __restrict__ y, int ldy, const float* __restrict__ ex, int ldex, const float* __restrict__ wex,
                                                             int ldw, int M, int o, int E) {
    __shared__ __align__(16) float ws[XWIDE_MAX_E][XWIDE_COLS];
    __shared__ float xs[XWIDE_ROWS][XWIDE_MAX_E + 1];
    const int n0 = blockIdx.x * XWIDE_COLS, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < E * XWIDE_COLS; i += blockDim.x) {
        const int c = i / E, t = i - c * E;         // consecutive threads read consecutive t of one w_extra row
        ws[t][c] = n0 + c < o ? __ldg(wex + (size_t)(n0 + c) * ldw + t) : 0.f;
    }
    const int c0 = n0 + 4 * lane;
    for (int r0 = blockIdx.y * XWIDE_ROWS; r0 < M; r0 += gridDim.y * XWIDE_ROWS) {
        const int rows = min(XWIDE_ROWS, M - r0);
        __syncthreads();                            // ws complete / the previous chunk's xs consumed
        for (int i = threadIdx.x; i < rows * E; i += blockDim.x) {
            const int r = i / E, t = i - r * E;
            xs[r][t] = __ldg(ex + (size_t)(r0 + r) * ldex + t);
        }
        __syncthreads();
        if (c0 >= o) continue;
        float a[4][4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int r = warp + 8 * u;
            if (r < rows) {
                const float* yr = y + (size_t)(r0 + r) * ldy + c0;
                if (VEC) {
                    const float4 v = *reinterpret_cast<const float4*>(yr);
                    a[u][0] = v.x; a[u][1] = v.y; a[u][2] = v.z; a[u][3] = v.w;
                } else {
#pragma unroll
                    for (int c = 0; c < 4; c++) a[u][c] = c0 + c < o ? yr[c] : 0.f;
                }
            }
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int r = warp + 8 * u;
            if (r >= rows) continue;
#pragma unroll 4
            for (int t = 0; t < E; t++) {
                const float e = xs[r][t];
                const float4 w = *reinterpret_cast<const float4*>(&ws[t][4 * lane]);
                a[u][0] = fmaf(e, w.x, a[u][0]); a[u][1] = fmaf(e, w.y, a[u][1]); a[u][2] = fmaf(e, w.z, a[u][2]); a[u][3] = fmaf(e, w.w, a[u][3]);
            }
            constexpr int K = KIND >= 0 ? KIND : 0;
#pragma unroll
            for (int c = 0; c < 4; c++) a[u][c] = KIND < 0 ? a[u][c] : (VEC ? act_fast<K>(a[u][c]) : act_exact<K>(a[u][c]));
            float* yr = y + (size_t)(r0 + r) * ldy + c0;
            if (VEC) {
                *reinterpret_cast<float4*>(yr) = make_float4(a[u][0], a[u][1], a[u][2], a[u][3]);
            } else {
#pragma unroll
                for (int c = 0; c < 4; c++) if (c0 + c < o) yr[c] = a[u][c];
            }
        }
    }
}
extern "C" int go1_mlp_extra_forward(float* y, int ldy, const float* extra, int ldex, const float* w_extra, int ldw, int M, int o, int E, int act,
                                     void* stream) {
    if (!y || !extra || !w_extra || M <= 0 || o <= 0 || act < 0 || act_mode(act) > 1) return go1_set_error("go1_mlp_extra_forward: bad arguments");
    if (E < 1 || E > XWIDE_MAX_E) return go1_set_error("go1_mlp_extra_forward: E (trailing input columns) must be 1..64");
    if (ldy < o || ldex < E || ldw < E) return go1_set_error("go1_mlp_extra_forward: row strides must be >= o (y) and >= E (extra, w_extra)");
    const int kind = act_kind(act);
    act = act_mode(act);
    if (!go1_act_kind_ok(kind)) return go1_set_error("go1_mlp_extra_forward: unknown activation kind (Go1Activation)");
    if (E > 4) {
        const bool vec = (o & 3) == 0 && (ldy & 3) == 0 && (((uintptr_t)y) & 15) == 0;
        const int gx = (o + XWIDE_COLS - 1) / XWIDE_COLS;
        const int gy = min((M + XWIDE_ROWS - 1) / XWIDE_ROWS, max(1, (132 * 4 + gx - 1) / gx));
        const dim3 grid(gx, gy);
#define LAUNCH(KD, V) extra_fwd_wide_kernel<KD, V><<<grid, 256, 0, (cudaStream_t)stream>>>(y, ldy, extra, ldex, w_extra, ldw, M, o, E)
        if (act == 0) { if (vec) LAUNCH(-1, true); else LAUNCH(-1, false); }
        else if (vec) { GO1_ACT_SWITCH(kind, KD, LAUNCH(KD, true);) }
        else { GO1_ACT_SWITCH(kind, KD, LAUNCH(KD, false);) }
#undef LAUNCH
        go1_count_launch(1);
        return cuda_rc("go1_mlp_extra_forward");
    }
    const int o4 = o / 4;
    if ((o & 3) == 0 && (ldy & 3) == 0 && (((uintptr_t)y) & 15) == 0 && o4 <= 256 && 256 % o4 == 0) {
        const int rpb = 256 / o4;
        int grid = (M + 4 * rpb - 1) / (4 * rpb);
        if (grid > 132 * 16) grid = 132 * 16;
#define LAUNCH(KD) extra_fwd4_kernel<KD><<<grid, 256, 0, (cudaStream_t)stream>>>(y, ldy, extra, ldex, w_extra, ldw, M, o4, E, 4 * rpb)
        if (act == 0) LAUNCH(-1);
        else { GO1_ACT_SWITCH(kind, KD, LAUNCH(KD);) }
#undef LAUNCH
        go1_count_launch(1);
        return cuda_rc("go1_mlp_extra_forward");
    }
    dim3 grid((o + 255) / 256, (M + 7) / 8);
    extra_fwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(y, ldy, extra, ldex, w_extra, ldw, M, o, E, act, kind); go1_count_launch(1);
    return cuda_rc("go1_mlp_extra_forward");
}

// dz = dy * f'(z) from the saved output y (act_deriv, activation.cuh; ELU, alpha = 1: 1 for y > 0 else y + 1)
__global__ void act_bwd_kernel(const float* __restrict__ y, int ldy, const float* __restrict__ dy, int lddy, float* __restrict__ dz, int lddz, int M, int N, int kind) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)M * N) return;
    const int m = (int)(i / N), n = (int)(i - (size_t)m * N);
    const float yv = y[(size_t)m * ldy + n];
    dz[(size_t)m * lddz + n] = dy[(size_t)m * lddy + n] * act_deriv_rt(kind, yv);
}
extern "C" int go1_act_backward(const float* y, int ldy, const float* dy, int lddy, float* dz, int lddz, int M, int N, int kind, void* stream) {
    if (!y || !dy || !dz || M <= 0 || N <= 0) return go1_set_error("go1_act_backward: bad arguments");
    if (!go1_act_kind_ok(kind)) return go1_set_error("go1_act_backward: unknown activation kind (Go1Activation)");
    const size_t tot = (size_t)M * N;
    act_bwd_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, (cudaStream_t)stream>>>(y, ldy, dy, lddy, dz, lddz, M, N, kind); go1_count_launch(1);
    return cuda_rc("go1_act_backward");
}
extern "C" int go1_elu_backward(const float* y, int ldy, const float* dy, int lddy, float* dz, int lddz, int M, int N, void* stream) {
    return go1_act_backward(y, ldy, dy, lddy, dz, lddz, M, N, GO1_ACT_ELU, stream);
}

// wgrad of a narrow (o <= 16) output layer: gW[j][k] (+)= sum_m dz[m][j] x[m][k].  One thread per input column k keeps the o
// partial sums in registers over a 64-row slab (x read once, coalesced; dz rows broadcast), then o atomics.
// DET: the slab's sums go to part[blockIdx.y][o][K] instead of gW (plain stores; go1_det_sum adds the slabs)
template <int O, bool DET>
__global__ void __launch_bounds__(128) skinny_wgrad_kernel(const float* __restrict__ dz, int lddz, const float* __restrict__ x, int ldx,
                                                           float* __restrict__ gW, int ldg, int M, int o, int K, int rows_per_block, float* __restrict__ part) {
    const int k = blockIdx.x * 128 + threadIdx.x;
    const int r0 = blockIdx.y * rows_per_block, r1 = min(M, r0 + rows_per_block);
    if (k >= K) return;
    float acc[O];
#pragma unroll
    for (int j = 0; j < O; j++) acc[j] = 0.f;
#pragma unroll 4
    for (int m = r0; m < r1; m++) {
        const float xv = x[(size_t)m * ldx + k];
#pragma unroll
        for (int j = 0; j < O; j++) if (j < o) acc[j] = fmaf(__ldg(dz + (size_t)m * lddz + j), xv, acc[j]);
    }
#pragma unroll
    for (int j = 0; j < O; j++) {
        if (j < o) {
            if (DET) part[((size_t)blockIdx.y * o + j) * K + k] = acc[j];
            else atomicAdd(gW + (size_t)j * ldg + k, acc[j]);
        }
    }
}
// float4 variant: a warp owns rows (stride 8 inside a row slab), lanes own 4 consecutive input columns; the o gradients of
// a row are fetched by the first o lanes and shuffle-broadcast.  Per-block partial sums meet in shared memory, then one
// set of global atomics per block.
// DET: the warps add their sums into s_acc one after the other, the bias-gradient sums meet in s_gb in warp order, and the block's
// results go to part[blockIdx.y][o][K] and (gb: only whether there is one) part_gb[blockIdx.y][o] (plain stores; go1_det_sum adds the slabs)
template <int O, bool DET>
__global__ void __launch_bounds__(256) skinny_wgrad4_kernel(const float* __restrict__ dz, int lddz, const float* __restrict__ x, int ldx,
                                                            float* __restrict__ gW, int ldg, float* __restrict__ gb, int M, int o, int K, int rows_per_block,
                                                            float* __restrict__ part, float* __restrict__ part_gb) {
    __shared__ float s_acc[O][128];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int k = blockIdx.x * 128 + lane * 4;
    const int r0 = blockIdx.y * rows_per_block, r1 = min(M, r0 + rows_per_block);
    for (int i = threadIdx.x; i < O * 128; i += 256) (&s_acc[0][0])[i] = 0.f;
    __syncthreads();
    float acc[O][4];
#pragma unroll
    for (int j = 0; j < O; j++) { acc[j][0] = 0.f; acc[j][1] = 0.f; acc[j][2] = 0.f; acc[j][3] = 0.f; }
    float dsum = 0.f;          // lane j < o: sum over this warp's rows of dz[m][j] (the layer's bias gradient, reduced by the column-block-0 CTAs)
#pragma unroll 2
    for (int m = r0 + w; m < r1; m += 8) {
        const float4 xv = k < K ? *reinterpret_cast<const float4*>(x + (size_t)m * ldx + k) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float dl = lane < o ? __ldg(dz + (size_t)m * lddz + lane) : 0.f;
        dsum += dl;
#pragma unroll
        for (int j = 0; j < O; j++) {
            const float d = __shfl_sync(0xffffffffu, dl, j);
            acc[j][0] = fmaf(d, xv.x, acc[j][0]); acc[j][1] = fmaf(d, xv.y, acc[j][1]);
            acc[j][2] = fmaf(d, xv.z, acc[j][2]); acc[j][3] = fmaf(d, xv.w, acc[j][3]);
        }
    }
    if constexpr (DET) {
        __shared__ float s_gb[8][16];
        for (int ww = 0; ww < 8; ww++) {
            if (w == ww) {
#pragma unroll
                for (int j = 0; j < O; j++)
#pragma unroll
                    for (int c = 0; c < 4; c++) s_acc[j][lane * 4 + c] += acc[j][c];
            }
            __syncthreads();
        }
        if (lane < 16) s_gb[w][lane] = dsum;
        __syncthreads();
        for (int i = threadIdx.x; i < o * 128; i += 256) {
            const int j = i >> 7, kk = blockIdx.x * 128 + (i & 127);
            if (kk < K) part[((size_t)blockIdx.y * o + j) * K + kk] = s_acc[j][i & 127];
        }
        if (gb && blockIdx.x == 0 && threadIdx.x < o) {
            float t = s_gb[0][threadIdx.x];
            for (int k = 1; k < 8; k++) t += s_gb[k][threadIdx.x];
            part_gb[(size_t)blockIdx.y * o + threadIdx.x] = t;
        }
    } else {
#pragma unroll
        for (int j = 0; j < O; j++)
#pragma unroll
            for (int c = 0; c < 4; c++) atomicAdd(&s_acc[j][lane * 4 + c], acc[j][c]);
        __syncthreads();
        for (int i = threadIdx.x; i < o * 128; i += 256) {
            const int j = i >> 7, kk = blockIdx.x * 128 + (i & 127);
            if (kk < K) atomicAdd(gW + (size_t)j * ldg + kk, s_acc[j][i & 127]);
        }
        if (gb && blockIdx.x == 0 && lane < o) atomicAdd(gb + lane, dsum);
    }
}
extern "C" int go1_skinny_wgrad_ex(const float* dz, int lddz, const float* x, int ldx, float* gW, int ldg, float* gb, int M, int o, int K, int accumulate, void* stream) {
    if (!dz || !x || !gW || M <= 0 || o < 1 || o > 16 || K <= 0 || ldg < K) return go1_set_error("go1_skinny_wgrad: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    if (gb && !((K & 3) == 0 && (ldx & 3) == 0 && (((uintptr_t)x) & 15) == 0)) return go1_set_error("go1_skinny_wgrad_ex: the fused bias gradient needs K % 4 == 0 and 16-byte aligned x rows");
    if (!accumulate) {
        if (ldg == K) cudaMemsetAsync(gW, 0, sizeof(float) * (size_t)o * K, st);
        else cudaMemset2DAsync(gW, sizeof(float) * ldg, 0, sizeof(float) * K, o, st);
        if (gb) cudaMemsetAsync(gb, 0, sizeof(float) * (size_t)o, st);
    }
    const bool det = go1_det_on();     // deterministic mode: the row slabs' sums meet in gW / gb in slab order
    const bool vec = (K & 3) == 0 && (ldx & 3) == 0 && (((uintptr_t)x) & 15) == 0;
    int rpb = 64;
    if (vec) {
        rpb = (M * ((K + 127) / 128) + 131) / 132;       // about one block per SM (the per-block reduction and atomics dominate with more)
        rpb = (rpb + 7) / 8 * 8; if (rpb < 8) rpb = 8;
    }
    const dim3 grid((K + 127) / 128, (M + rpb - 1) / rpb);
    const size_t nw = (size_t)grid.y * o * K;
    float* part = go1_det_out<float>(det, st, nw + (vec ? (size_t)grid.y * o : 0), nullptr);
    if (det && !part) return 1;
    float* const part_gb = det ? part + nw : nullptr;
#define LAUNCH(O)                                                                                                                                      \
    if (vec) (det ? skinny_wgrad4_kernel<O, true> : skinny_wgrad4_kernel<O, false>)<<<grid, 256, 0, st>>>(dz, lddz, x, ldx, gW, ldg, gb, M, o, K, rpb, part, part_gb); \
    else (det ? skinny_wgrad_kernel<O, true> : skinny_wgrad_kernel<O, false>)<<<grid, 128, 0, st>>>(dz, lddz, x, ldx, gW, ldg, M, o, K, rpb, part)
    if (o <= 2) { LAUNCH(2); } else if (o <= 4) { LAUNCH(4); } else { LAUNCH(16); }
#undef LAUNCH
    go1_count_launch(1);
    if (int e = cuda_rc("go1_skinny_wgrad")) return e;
    if (!det) return 0;
    if (int e = go1_det_sum(part, grid.y, (size_t)o * K, gW, o, K, ldg, 1, st)) return e;
    return gb ? go1_det_sum(part_gb, grid.y, o, gb, 1, o, o, 1, st) : 0;
}

extern "C" int go1_skinny_wgrad(const float* dz, int lddz, const float* x, int ldx, float* gW, int ldg, int M, int o, int K, int accumulate, void* stream) {
    return go1_skinny_wgrad_ex(dz, lddz, x, ldx, gW, ldg, nullptr, M, o, K, accumulate, stream);
}

// Up to 8 strided 2-D copies in ONE launch (dst[r][c] = src[r][c]): the packed first-layer weight block / bias / trailing-input
// weights the fused first-layer product reads, and the way back from the fused wgrad's output into the flat gradient buffer.
// Rows of the ActorCritic first layers are 2102 floats long (8-byte aligned), so the vector width is 8 bytes.
struct CopySegs { Go1CopySeg s[8]; int n; };
__global__ void __launch_bounds__(256) copy_segments_kernel(const CopySegs a) {
    for (int si = 0; si < a.n; si++) {
        const Go1CopySeg& sg = a.s[si];
        const bool v2 = ((sg.cols & 1) == 0) && ((sg.lds & 1) == 0) && ((sg.ldd & 1) == 0) && (((uintptr_t)sg.src | (uintptr_t)sg.dst) & 7) == 0;
        if (v2) {
            const int c2 = sg.cols >> 1;
            const long long total = (long long)sg.rows * c2;
            for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
                const int r = (int)(i / c2), c = (int)(i - (long long)r * c2);
                reinterpret_cast<float2*>(sg.dst + (size_t)r * sg.ldd)[c] = __ldg(reinterpret_cast<const float2*>(sg.src + (size_t)r * sg.lds) + c);
            }
        } else {
            const long long total = (long long)sg.rows * sg.cols;
            for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
                const int r = (int)(i / sg.cols), c = (int)(i - (long long)r * sg.cols);
                sg.dst[(size_t)r * sg.ldd + c] = __ldg(sg.src + (size_t)r * sg.lds + c);
            }
        }
    }
}
extern "C" int go1_copy_segments(const Go1CopySeg* segs, int n, void* stream) {
    if (!segs || n < 1 || n > 8) return go1_set_error("go1_copy_segments: 1..8 segments");
    CopySegs a; a.n = n;
    long long work = 0;
    for (int i = 0; i < n; i++) {
        if (!segs[i].src || !segs[i].dst || segs[i].rows <= 0 || segs[i].cols <= 0 || segs[i].lds < segs[i].cols || segs[i].ldd < segs[i].cols)
            return go1_set_error("go1_copy_segments: bad segment");
        a.s[i] = segs[i];
        const long long w = (long long)segs[i].rows * segs[i].cols / 2;
        if (w > work) work = w;
    }
    long long blocks = (work + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (blocks < 1) blocks = 1;
    copy_segments_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(a); go1_count_launch(1);
    return cuda_rc("go1_copy_segments");
}

// out[n] (+)= sum_m x[m][n]   (bias gradients).  DET (both variants): the slab's sums go to out[blockIdx.y][N] (plain stores, partials for go1_det_sum)
template <bool DET>
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ x, int ldx, float* __restrict__ out, int M, int N, int rows_per_block) {
    __shared__ float s[8][33];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int n = blockIdx.x * 32 + lane;
    const int r0 = blockIdx.y * rows_per_block, r1 = min(M, r0 + rows_per_block);
    float acc = 0.f;
    if (n < N) for (int m = r0 + w; m < r1; m += 8) acc += x[(size_t)m * ldx + n];
    s[w][lane] = acc;
    __syncthreads();
    if (w == 0 && n < N) {
        float t = 0.f;
#pragma unroll
        for (int k = 0; k < 8; k++) t += s[k][lane];
        if (DET) out[(size_t)blockIdx.y * N + n] = t;
        else atomicAdd(out + n, t);
    }
}
// wide variant: one float4 column group per lane (128 columns per warp row), 4 independent rows in flight per thread
template <bool DET>
__global__ void __launch_bounds__(256) colsum4_kernel(const float* __restrict__ x, int ldx, float* __restrict__ out, int M, int N, int rows_per_block) {
    __shared__ float4 s[8][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int n = blockIdx.x * 128 + lane * 4;
    const int r0 = blockIdx.y * rows_per_block, r1 = min(M, r0 + rows_per_block);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (n < N) {
        int m = r0 + w;
        for (; m + 24 < r1; m += 32) {
            const float4 a = *reinterpret_cast<const float4*>(x + (size_t)m * ldx + n);
            const float4 b = *reinterpret_cast<const float4*>(x + (size_t)(m + 8) * ldx + n);
            const float4 c = *reinterpret_cast<const float4*>(x + (size_t)(m + 16) * ldx + n);
            const float4 d = *reinterpret_cast<const float4*>(x + (size_t)(m + 24) * ldx + n);
            acc.x += (a.x + b.x) + (c.x + d.x); acc.y += (a.y + b.y) + (c.y + d.y);
            acc.z += (a.z + b.z) + (c.z + d.z); acc.w += (a.w + b.w) + (c.w + d.w);
        }
        for (; m < r1; m += 8) {
            const float4 a = *reinterpret_cast<const float4*>(x + (size_t)m * ldx + n);
            acc.x += a.x; acc.y += a.y; acc.z += a.z; acc.w += a.w;
        }
    }
    s[w][lane] = acc;
    __syncthreads();
    if (w == 0 && n < N) {
        float4 t = s[0][lane];
#pragma unroll
        for (int k = 1; k < 8; k++) { t.x += s[k][lane].x; t.y += s[k][lane].y; t.z += s[k][lane].z; t.w += s[k][lane].w; }
        if (DET) *reinterpret_cast<float4*>(out + (size_t)blockIdx.y * N + n) = t;
        else { atomicAdd(out + n, t.x); atomicAdd(out + n + 1, t.y); atomicAdd(out + n + 2, t.z); atomicAdd(out + n + 3, t.w); }
    }
}
extern "C" int go1_colsum(const float* x, int ldx, float* out, int M, int N, int accumulate, void* stream) {
    if (!x || !out || M <= 0 || N <= 0) return go1_set_error("go1_colsum: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    const bool vec = N >= 64 && (N & 3) == 0 && (ldx & 3) == 0 && (((uintptr_t)x) & 15) == 0;
    const bool det = go1_det_on();     // deterministic mode: the row slabs' sums meet in out in slab order
    const int rpb = vec ? 128 : 512;
    const dim3 grid(vec ? (N + 127) / 128 : (N + 31) / 32, (M + rpb - 1) / rpb);
    float* dst = go1_det_out(det, st, (size_t)grid.y * N, out);
    if (det && !dst) return 1;
    if (!accumulate && !det) cudaMemsetAsync(out, 0, sizeof(float) * N, st);
    if (vec) (det ? colsum4_kernel<true> : colsum4_kernel<false>)<<<grid, 256, 0, st>>>(x, ldx, dst, M, N, rpb);
    else (det ? colsum_kernel<true> : colsum_kernel<false>)<<<grid, 256, 0, st>>>(x, ldx, dst, M, N, rpb);
    go1_count_launch(1);
    if (int e = cuda_rc("go1_colsum")) return e;
    return det ? go1_det_sum(dst, grid.y, N, out, 1, N, N, accumulate, st) : 0;
}

// ---------------------------------------------------------------------------------------------
// Normal(mean, std): sample + log-prob  (actor_critic.py:113-126)
// ---------------------------------------------------------------------------------------------
__global__ void sample_actions_kernel(const float* __restrict__ mean, int ldm, const float* __restrict__ std, const float* __restrict__ eps,
                                      uint64_t seed, uint64_t counter, const unsigned long long* __restrict__ counter_dev,
                                      float* __restrict__ actions, float* __restrict__ logp, int n, int na) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (counter_dev) counter += *counter_dev;
    float lp = 0.f;
    for (int j = 0; j < na; j++) {
        float e;
        if (eps) e = eps[(size_t)i * na + j];
        else {   // Box-Muller on two Philox uniforms
            float u1 = philox_uniform(seed, (uint32_t)i, counter, 2u * j), u2 = philox_uniform(seed, (uint32_t)i, counter, 2u * j + 1u);
            u1 = fmaxf(u1, 5.9604645e-8f);
            e = sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
        }
        const float mu = mean[(size_t)i * ldm + j], sd = std[j];
        const float a = mu + sd * e;
        actions[(size_t)i * na + j] = a;
        const float d = a - mu;
        lp += -(d * d) / (2.0f * sd * sd) - logf(sd) - 0.91893853320467274178f;
    }
    logp[i] = lp;
}
__global__ void bump_counter_kernel(unsigned long long* c) { *c += 1ull; }
extern "C" int go1_ppo_sample_actions(const float* mean, int ldm, const float* std, const float* eps, uint64_t seed, uint64_t counter,
                                      uint64_t* counter_dev, float* actions, float* logp, int n, int num_actions, void* stream) {
    if (!mean || !std || !actions || !logp || n <= 0 || num_actions <= 0) return go1_set_error("go1_ppo_sample_actions: bad arguments");
    sample_actions_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(mean, ldm, std, eps, seed, counter, (const unsigned long long*)counter_dev, actions, logp, n, num_actions);
    if (counter_dev) { bump_counter_kernel<<<1, 1, 0, (cudaStream_t)stream>>>((unsigned long long*)counter_dev); go1_count_launch(1); } go1_count_launch(1);
    return cuda_rc("go1_ppo_sample_actions");
}

// ---------------------------------------------------------------------------------------------
// PPO loss + gradients (ppo.py:113-152).  scalars[0..3] += inv_count * {surrogate, value loss, entropy, kl} sums.
// ---------------------------------------------------------------------------------------------
#define PPO_MAX_ACT 16
// DET: the block's PPO_MAX_ACT dstd sums and three scalars go to part[blockIdx.x][PPO_MAX_ACT + 3] (partials for go1_det_sum)
template <bool DET>
__global__ void __launch_bounds__(256) ppo_loss_kernel(const float* __restrict__ mean, int ldm, const float* __restrict__ std, const float* __restrict__ value,
        const float* __restrict__ actions, const float* __restrict__ old_logp, const float* __restrict__ old_mean, const float* __restrict__ old_std,
        const float* __restrict__ adv, const float* __restrict__ returns, const float* __restrict__ old_values,
        float* __restrict__ dmean, int lddm, float* __restrict__ dvalue, float* __restrict__ dstd, float* __restrict__ scalars,
        int n, int na, float clip, float vcoef, float ecoef, int clipped_v, float inv_count, float* __restrict__ part) {
    __shared__ float s_red[8][PPO_MAX_ACT + 4];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float dsd[PPO_MAX_ACT];
#pragma unroll
    for (int j = 0; j < PPO_MAX_ACT; j++) dsd[j] = 0.f;
    float surr = 0.f, vloss = 0.f, kl = 0.f;
    if (i < n) {
        float lp = 0.f;
        for (int j = 0; j < na; j++) {
            const float mu = mean[(size_t)i * ldm + j], sd = std[j], a = actions[(size_t)i * na + j];
            const float d = a - mu;
            lp += -(d * d) / (2.0f * sd * sd) - logf(sd) - 0.91893853320467274178f;
            const float om = old_mean[(size_t)i * na + j], os = old_std[(size_t)i * na + j];
            kl += logf(sd / os + 1.e-5f) + (os * os + (om - mu) * (om - mu)) / (2.0f * sd * sd) - 0.5f;
        }
        const float A = adv[i];
        const float ratio = expf(lp - old_logp[i]);
        const float s1 = -A * ratio, s2 = -A * fminf(fmaxf(ratio, 1.0f - clip), 1.0f + clip);
        surr = fmaxf(s1, s2);
        const bool inside = ratio >= 1.0f - clip && ratio <= 1.0f + clip;
        // d max(s1,s2)/d ratio (torch: ties split evenly; inside the clip range both branches carry -A)
        float gr = (s1 > s2) ? -A : ((s1 == s2) ? (inside ? -A : -0.5f * A) : (inside ? -A : 0.f));
        const float glp = gr * ratio * inv_count;
        for (int j = 0; j < na; j++) {
            const float mu = mean[(size_t)i * ldm + j], sd = std[j], a = actions[(size_t)i * na + j];
            const float d = a - mu;
            dmean[(size_t)i * lddm + j] = glp * d / (sd * sd);
            dsd[j] = glp * (d * d / (sd * sd * sd) - 1.0f / sd);
        }
        const float v = value[i], R = returns[i];
        float gv;
        if (clipped_v) {
            const float vt = old_values[i];
            const float dv = v - vt;
            const float vc = vt + fminf(fmaxf(dv, -clip), clip);
            const float l1 = (v - R) * (v - R), l2 = (vc - R) * (vc - R);
            vloss = fmaxf(l1, l2);
            const float g1 = 2.0f * (v - R), g2 = (dv >= -clip && dv <= clip) ? 2.0f * (vc - R) : 0.f;
            gv = (l1 > l2) ? g1 : ((l1 == l2) ? 0.5f * (g1 + g2) : g2);
        } else { vloss = (R - v) * (R - v); gv = 2.0f * (v - R); }
        dvalue[i] = vcoef * gv * inv_count;
    }
    // reductions: 12 dstd partials + 3 scalars
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    float red[PPO_MAX_ACT + 3];
#pragma unroll
    for (int j = 0; j < PPO_MAX_ACT; j++) red[j] = dsd[j];
    red[PPO_MAX_ACT] = surr; red[PPO_MAX_ACT + 1] = vloss; red[PPO_MAX_ACT + 2] = kl;
#pragma unroll
    for (int j = 0; j < PPO_MAX_ACT + 3; j++) {
        float v = red[j];
        for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
        if (lane == 0) s_red[w][j] = v;
    }
    __syncthreads();
    if (threadIdx.x < PPO_MAX_ACT + 3) {
        float t = 0.f;
        for (int k = 0; k < 8; k++) t += s_red[k][threadIdx.x];
        const int j = threadIdx.x;
        if (DET) part[(size_t)blockIdx.x * (PPO_MAX_ACT + 3) + j] = j < PPO_MAX_ACT ? t : t * inv_count;
        else if (j < PPO_MAX_ACT) { if (j < na) atomicAdd(dstd + j, t); }
        else atomicAdd(scalars + (j == PPO_MAX_ACT ? 0 : (j == PPO_MAX_ACT + 1 ? 1 : 3)), t * inv_count);
    }
}
__global__ void ppo_entropy_kernel(const float* __restrict__ std, float* __restrict__ dstd, float* __restrict__ scalars, int na, float ecoef, float local_frac) {
    // entropy of Normal(mean, std) summed over actions is the same for every sample: sum_j 0.5 + 0.5 log(2 pi) + log std_j
    const int j = threadIdx.x;
    float h = 0.f;
    if (j < na) { h = 1.4189385332046727f + logf(std[j]); atomicAdd(dstd + j, -ecoef * local_frac / std[j]); }
    for (int d = 16; d > 0; d >>= 1) h += __shfl_xor_sync(0xffffffffu, h, d);
    if (j == 0) atomicAdd(scalars + 2, h * local_frac);
}
extern "C" int go1_ppo_loss(const float* mean, int ldm, const float* std, const float* value, const float* actions,
                            const float* old_logp, const float* old_mean, const float* old_std, const float* advantages,
                            const float* returns, const float* old_values, float* dmean, int lddm, float* dvalue,
                            float* dstd, float* scalars, int n, int num_actions, float clip_param,
                            float value_loss_coef, float entropy_coef, int use_clipped_value_loss, float inv_count, void* stream) {
    if (!mean || !std || !value || !actions || !old_logp || !old_mean || !old_std || !advantages || !returns || !old_values || !dmean || !dvalue || !dstd || !scalars)
        return go1_set_error("go1_ppo_loss: null argument");
    if (n <= 0 || num_actions <= 0 || num_actions > PPO_MAX_ACT) return go1_set_error("go1_ppo_loss: bad sizes");
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(dstd, 0, sizeof(float) * num_actions, st);
    cudaMemsetAsync(scalars, 0, sizeof(float) * 8, st);
    const bool det = go1_det_on();     // deterministic mode: the blocks' sums meet in dstd / scalars in block order, then the entropy kernel adds its terms
    const int nb = (n + 255) / 256;
    constexpr int W = PPO_MAX_ACT + 3;
    float* part = go1_det_out<float>(det, st, (size_t)nb * W, nullptr);
    if (det && !part) return 1;
    (det ? ppo_loss_kernel<true> : ppo_loss_kernel<false>)<<<nb, 256, 0, st>>>(mean, ldm, std, value, actions, old_logp, old_mean, old_std, advantages, returns,
                                                                               old_values, dmean, lddm, dvalue, dstd, scalars, n, num_actions, clip_param,
                                                                               value_loss_coef, entropy_coef, use_clipped_value_loss, inv_count, part);
    go1_count_launch(1);
    if (det) {
        if (int e = cuda_rc("go1_ppo_loss")) return e;
        if (int e = go1_det_sum(part, nb, W, dstd, 1, num_actions, num_actions, 0, st)) return e;
        if (int e = go1_det_sum(part + PPO_MAX_ACT, nb, W, scalars, 1, 2, 2, 0, st)) return e;         // surrogate, value loss
        if (int e = go1_det_sum(part + PPO_MAX_ACT + 2, nb, W, scalars + 3, 1, 1, 1, 0, st)) return e;  // kl
    }
    ppo_entropy_kernel<<<1, 32, 0, st>>>(std, dstd, scalars, num_actions, entropy_coef, (float)n * inv_count); go1_count_launch(1);
    return cuda_rc("go1_ppo_loss");
}

// MSE (ppo.py:168-186): train split [0, num_train) gets loss + gradient, the rest only the test loss.  DET: scalars is the workspace, and
// the block's two losses go to scalars[2 blockIdx.x ..]
template <bool DET>
__global__ void __launch_bounds__(256) mse_kernel(const float* __restrict__ pred, int ldp, const float* __restrict__ tgt, int ldt, float* __restrict__ dpred, int lddp,
                                                  float* __restrict__ scalars, int n, int num_train, int dim) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float ltr = 0.f, lte = 0.f;
    if (i < n) {
        const bool train = i < num_train;
        const float inv_tr = 1.0f / ((float)num_train * dim);
        for (int j = 0; j < dim; j++) {
            const float d = pred[(size_t)i * ldp + j] - tgt[(size_t)i * ldt + j];
            if (train) { ltr += d * d; dpred[(size_t)i * lddp + j] = 2.0f * d * inv_tr; }
            else { lte += d * d; dpred[(size_t)i * lddp + j] = 0.f; }
        }
    }
    __shared__ float s[2][8];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int d = 16; d > 0; d >>= 1) { ltr += __shfl_xor_sync(0xffffffffu, ltr, d); lte += __shfl_xor_sync(0xffffffffu, lte, d); }
    if (lane == 0) { s[0][w] = ltr; s[1][w] = lte; }
    __syncthreads();
    if (threadIdx.x < 2) {
        float t = 0.f;
        for (int k = 0; k < 8; k++) t += s[threadIdx.x][k];
        const float cnt = threadIdx.x == 0 ? (float)num_train * dim : (float)(n - num_train) * dim;
        if constexpr (DET) scalars[2 * blockIdx.x + threadIdx.x] = cnt > 0.f ? t / cnt : 0.f;
        else if (cnt > 0.f) atomicAdd(scalars + threadIdx.x, t / cnt);
    }
}
extern "C" int go1_ppo_mse(const float* pred, int ldp, const float* target, int ldt, float* dpred, int lddp, float* scalars,
                           int n, int num_train, int dim, void* stream) {
    if (!pred || !target || !dpred || !scalars || n <= 0 || dim <= 0 || num_train < 0 || num_train > n) return go1_set_error("go1_ppo_mse: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    const bool det = go1_det_on();     // deterministic mode: the blocks' losses meet in scalars in block order
    const int nb = (n + 255) / 256;
    float* out = go1_det_out(det, st, 2 * (size_t)nb, scalars);
    if (det && !out) return 1;
    if (!det) cudaMemsetAsync(scalars, 0, sizeof(float) * 2, st);
    (det ? mse_kernel<true> : mse_kernel<false>)<<<nb, 256, 0, st>>>(pred, ldp, target, ldt, dpred, lddp, out, n, num_train, dim); go1_count_launch(1);
    if (int e = cuda_rc("go1_ppo_mse")) return e;
    return det ? go1_det_sum(out, nb, 2, scalars, 1, 2, 2, 0, st) : 0;
}

// ---------------------------------------------------------------------------------------------
// clip_grad_norm_ + Adam over a flat buffer (ppo.py:155-158)
// ---------------------------------------------------------------------------------------------
// DET: the block's sum goes to out[blockIdx.x] (partials for go1_det_sum64)
template <bool DET>
__global__ void __launch_bounds__(256) sqnorm_kernel(const float* __restrict__ g, long long count, double* __restrict__ out) {
    double acc = 0.0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) { const float v = g[i]; acc += (double)v * (double)v; }
    __shared__ double s[8];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int d = 16; d > 0; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
    if (lane == 0) s[w] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0; for (int k = 0; k < 8; k++) t += s[k];
        if (DET) out[blockIdx.x] = t;
        else atomicAdd(out, t);
    }
}
extern "C" int go1_ppo_grad_sqnorm(const float* grad, int64_t count, double* grad_sq, void* stream) {
    if (!grad || !grad_sq || count <= 0) return go1_set_error("go1_ppo_grad_sqnorm: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    const bool det = go1_det_on();     // deterministic mode: the 296 blocks' sums meet in grad_sq in block order
    double* out = go1_det_out(det, st, 296, grad_sq);
    if (det && !out) return 1;
    if (!det) cudaMemsetAsync(grad_sq, 0, sizeof(double), st);
    (det ? sqnorm_kernel<true> : sqnorm_kernel<false>)<<<296, 256, 0, st>>>(grad, count, out); go1_count_launch(1);
    if (int e = cuda_rc("go1_ppo_grad_sqnorm")) return e;
    return det ? go1_det_sum64(out, 296, 1, grad_sq, 1, 0, st) : 0;
}
__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long long count,
                                                   const double* __restrict__ grad_sq, float max_norm, float lr, const float* __restrict__ lr_dev, float b1, float b2, float eps, float bc1, float bc2_sqrt) {
    if (lr_dev) lr = *lr_dev;
    float coef = 1.0f;
    if (max_norm > 0.f && grad_sq) {
        const float total = (float)sqrt(*grad_sq);
        coef = fminf(max_norm / (total + 1e-6f), 1.0f);
    }
    const float step_size = lr / bc1;
    if ((count & 3) == 0 && ((((uintptr_t)p) | ((uintptr_t)g) | ((uintptr_t)m) | ((uintptr_t)v)) & 15) == 0) {      // same arithmetic, 16-byte accesses
        float4* p4 = reinterpret_cast<float4*>(p); const float4* g4 = reinterpret_cast<const float4*>(g);
        float4* m4 = reinterpret_cast<float4*>(m); float4* v4 = reinterpret_cast<float4*>(v);
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count / 4; i += (long long)gridDim.x * blockDim.x) {
            float4 pp = p4[i], mm = m4[i], vv = v4[i]; const float4 gg = g4[i];
            float* pa = &pp.x; float* ma = &mm.x; float* va = &vv.x; const float* ga = &gg.x;
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const float gi = ga[c] * coef;
                const float mi = b1 * ma[c] + (1.0f - b1) * gi;
                const float vi = b2 * va[c] + (1.0f - b2) * gi * gi;
                ma[c] = mi; va[c] = vi;
                const float denom = sqrtf(vi) / bc2_sqrt + eps;
                pa[c] -= step_size * (mi / denom);
            }
            p4[i] = pp; m4[i] = mm; v4[i] = vv;
        }
        return;
    }
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
        const float gi = g[i] * coef;
        const float mi = b1 * m[i] + (1.0f - b1) * gi;
        const float vi = b2 * v[i] + (1.0f - b2) * gi * gi;
        m[i] = mi; v[i] = vi;
        const float denom = sqrtf(vi) / bc2_sqrt + eps;
        p[i] -= step_size * (mi / denom);
    }
}
__global__ void adaptive_lr_kernel(const float* __restrict__ scalars, float* __restrict__ lr, float desired_kl, float lo, float hi) {
    const float kl = scalars[3];
    float v = *lr;
    if (kl > desired_kl * 2.0f) v = fmaxf(lo, v / 1.5f);
    else if (kl < desired_kl / 2.0f && kl > 0.0f) v = fminf(hi, v * 1.5f);
    *lr = v;
}
extern "C" int go1_ppo_adaptive_lr(const float* scalars, float* lr_dev, float desired_kl, float lr_min, float lr_max, void* stream) {
    if (!scalars || !lr_dev) return go1_set_error("go1_ppo_adaptive_lr: bad arguments");
    adaptive_lr_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(scalars, lr_dev, desired_kl, lr_min, lr_max); go1_count_launch(1);
    return cuda_rc("go1_ppo_adaptive_lr");
}
extern "C" int go1_ppo_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t count, const double* grad_sq,
                                 float max_grad_norm, float lr, const float* lr_dev, float beta1, float beta2, float eps, int step, void* stream) {
    if (!param || !grad || !exp_avg || !exp_avg_sq || count <= 0 || step <= 0) return go1_set_error("go1_ppo_adam_step: bad arguments");
    const float bc1 = 1.0f - powf(beta1, (float)step), bc2 = 1.0f - powf(beta2, (float)step);
    adam_kernel<<<296, 256, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, count, grad_sq, max_grad_norm, lr, lr_dev, beta1, beta2, eps, bc1, sqrtf(bc2)); go1_count_launch(1);
    return cuda_rc("go1_ppo_adam_step");
}

// ---------------------------------------------------------------------------------------------
// row gather: dst[i][0:width] = src[idx[i]][0:width]   (dst row stride ldd)
// ---------------------------------------------------------------------------------------------
__global__ void gather_rows_kernel(const float* __restrict__ src, const long long* __restrict__ idx, float* __restrict__ dst, long long rows, int width, int ldd) {
    const long long r = blockIdx.x;
    if (r >= rows) return;
    const float* s = src + (size_t)idx[r] * width;
    float* d = dst + (size_t)r * ldd;
    if ((width & 3) == 0 && (ldd & 3) == 0 && (((uintptr_t)src | (uintptr_t)dst) & 15) == 0) {
        const int w4 = width / 4;
        if (w4 <= 5 * (int)blockDim.x) {        // long rows (the 2100-float histories): all of a thread's loads in flight before its stores
            float4 v[5];
#pragma unroll
            for (int k = 0; k < 5; k++) { const int c = threadIdx.x + k * blockDim.x; if (c < w4) v[k] = __ldg(reinterpret_cast<const float4*>(s) + c); }
#pragma unroll
            for (int k = 0; k < 5; k++) { const int c = threadIdx.x + k * blockDim.x; if (c < w4) reinterpret_cast<float4*>(d)[c] = v[k]; }
        } else {
            for (int c = threadIdx.x; c < w4; c += blockDim.x) reinterpret_cast<float4*>(d)[c] = reinterpret_cast<const float4*>(s)[c];
        }
    } else {
        for (int c = threadIdx.x; c < width; c += blockDim.x) d[c] = s[c];
    }
}
extern "C" int go1_gather_rows(const float* src, const int64_t* idx, float* dst, int64_t rows, int width, int ldd, void* stream) {
    if (!src || !idx || !dst || rows <= 0 || width <= 0 || ldd < width) return go1_set_error("go1_gather_rows: bad arguments");
    const int threads = width >= 1024 ? 128 : (width >= 128 ? 64 : 32);
    gather_rows_kernel<<<(unsigned)rows, threads, 0, (cudaStream_t)stream>>>(src, (const long long*)idx, dst, rows, width, ldd); go1_count_launch(1);
    return cuda_rc("go1_gather_rows");
}

// ---------------------------------------------------------------------------------------------
// skinny pieces of the MLP backward that are pure bandwidth (one pass over dz), kept off the GEMM kernels:
//   extra columns of a first layer:  dextra[m][t] = sum_j dz[m][j] We[j][t];   gWe[j][t] (+)= sum_m dz[m][j] extra[m][t]
//   dgrad through a <=4-wide output: dprev[m][c] = (sum_t dz[m][t] W[t][c]) * f'(y_prev[m][c])   (f' from the saved output: act_deriv)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) extra_dinput_kernel(const float* __restrict__ dz, int lddz, const float* __restrict__ We, int ldw,
                                                           float* __restrict__ dextra, int ldde, int M, int o, int E) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= M) return;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const float* row = dz + (size_t)warp * lddz;
#pragma unroll 4
    for (int j = lane; j < o; j += 32) {
        const float d = row[j];
#pragma unroll
        for (int t = 0; t < 4; t++) if (t < E) acc[t] = fmaf(d, __ldg(We + (size_t)j * ldw + t), acc[t]);      // static indices: acc stays in registers
    }
#pragma unroll
    for (int t = 0; t < 4; t++) {
        float v = acc[t];
        for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
        if (lane == 0 && t < E) dextra[(size_t)warp * ldde + t] = v;
    }
}
// DET (this kernel and extra_wgrad_wide): the slab's sums go to part[blockIdx.y][o][E] (plain stores; go1_det_sum adds the slabs into gWe)
template <bool DET>
__global__ void __launch_bounds__(256) extra_wgrad_kernel(const float* __restrict__ dz, int lddz, const float* __restrict__ extra, int ldex,
                                                          float* __restrict__ gWe, int ldgw, int M, int o, int E, int rows_per_block, float* __restrict__ part) {
    const int r0 = blockIdx.y * rows_per_block, r1 = min(M, r0 + rows_per_block);
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= o) return;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 8
    for (int m = r0; m < r1; m++) {
        const float d = dz[(size_t)m * lddz + j];
#pragma unroll
        for (int t = 0; t < 4; t++) if (t < E) acc[t] = fmaf(d, __ldg(extra + (size_t)m * ldex + t), acc[t]);
    }
#pragma unroll
    for (int t = 0; t < 4; t++) {
        if (t < E) {
            if (DET) part[((size_t)blockIdx.y * o + j) * E + t] = acc[t];
            else atomicAdd(gWe + (size_t)j * ldgw + t, acc[t]);
        }
    }
}
__global__ void zero_small_kernel(float* p, int ld, int rows, int cols) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < rows * cols) p[(size_t)(i / cols) * ld + (i % cols)] = 0.f;
}
// Wide variants (E up to EB = 8 / 16 / 32 / 64; also every E of a transposed dz).
// d(extra): one thread per row m with its EB sums in registers; w_extra is staged in shared memory 64 rows at a time (zero beyond E) and
// read as broadcasts.  DZT: dz is [o][M] (the transposed first-layer dz the dgrad epilogue stores; coalesced along m), else [M][o].
template <int EB, bool DZT>
__global__ void __launch_bounds__(128) extra_dinput_wide_kernel(const float* __restrict__ dz, int lddz, const float* __restrict__ We, int ldw,
                                                                float* __restrict__ dextra, int ldde, int M, int o, int E) {
    __shared__ __align__(16) float ws[64][EB];
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    float acc[EB];
#pragma unroll
    for (int t = 0; t < EB; t++) acc[t] = 0.f;
    for (int j0 = 0; j0 < o; j0 += 64) {
        const int nj = min(64, o - j0);
        __syncthreads();
        for (int i = threadIdx.x; i < 64 * EB; i += blockDim.x) {
            const int jj = i / EB, t = i - jj * EB;
            ws[jj][t] = jj < nj && t < E ? __ldg(We + (size_t)(j0 + jj) * ldw + t) : 0.f;
        }
        __syncthreads();
        if (m >= M) continue;
        const float* p = DZT ? dz + (size_t)j0 * lddz + m : dz + (size_t)m * lddz + j0;
        const size_t step = DZT ? (size_t)lddz : 1;
#pragma unroll 4
        for (int jj = 0; jj < nj; jj++, p += step) {
            const float d = *p;
#pragma unroll
            for (int t = 0; t < EB; t += 4) {
                const float4 w = *reinterpret_cast<const float4*>(&ws[jj][t]);
                acc[t] = fmaf(d, w.x, acc[t]); acc[t + 1] = fmaf(d, w.y, acc[t + 1]); acc[t + 2] = fmaf(d, w.z, acc[t + 2]); acc[t + 3] = fmaf(d, w.w, acc[t + 3]);
            }
        }
    }
    if (m >= M) return;
#pragma unroll
    for (int t = 0; t < EB; t++) if (t < E) dextra[(size_t)m * ldde + t] = acc[t];
}
// weight gradient: one thread per column j with its EB sums in registers over the CTA's row slab; the slab's extra rows are staged in
// shared memory 32 at a time (zero beyond E) and read as broadcasts; E atomics per thread at the end.
template <int EB, bool DET>
__global__ void __launch_bounds__(128) extra_wgrad_wide_kernel(const float* __restrict__ dz, int lddz, const float* __restrict__ extra, int ldex,
                                                               float* __restrict__ gWe, int ldgw, int M, int o, int E, int rows_per_block, float* __restrict__ part) {
    __shared__ __align__(16) float xs[32][EB];
    const int r0 = blockIdx.y * rows_per_block, r1 = min(M, r0 + rows_per_block);
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    float acc[EB];
#pragma unroll
    for (int t = 0; t < EB; t++) acc[t] = 0.f;
    for (int m0 = r0; m0 < r1; m0 += 32) {
        const int nr = min(32, r1 - m0);
        __syncthreads();
        for (int i = threadIdx.x; i < 32 * EB; i += blockDim.x) {
            const int r = i / EB, t = i - r * EB;
            xs[r][t] = r < nr && t < E ? __ldg(extra + (size_t)(m0 + r) * ldex + t) : 0.f;
        }
        __syncthreads();
        if (j >= o) continue;
#pragma unroll 4
        for (int r = 0; r < nr; r++) {
            const float d = dz[(size_t)(m0 + r) * lddz + j];
#pragma unroll
            for (int t = 0; t < EB; t += 4) {
                const float4 x = *reinterpret_cast<const float4*>(&xs[r][t]);
                acc[t] = fmaf(d, x.x, acc[t]); acc[t + 1] = fmaf(d, x.y, acc[t + 1]); acc[t + 2] = fmaf(d, x.z, acc[t + 2]); acc[t + 3] = fmaf(d, x.w, acc[t + 3]);
            }
        }
    }
    if (j >= o) return;
#pragma unroll
    for (int t = 0; t < EB; t++) {
        if (t < E) {
            if (DET) part[((size_t)blockIdx.y * o + j) * E + t] = acc[t];
            else atomicAdd(gWe + (size_t)j * ldgw + t, acc[t]);
        }
    }
}
#define XWIDE_EB_SWITCH(E, EBV, ...)                                                   \
    if ((E) <= 8) { constexpr int EBV = 8; __VA_ARGS__ }                               \
    else if ((E) <= 16) { constexpr int EBV = 16; __VA_ARGS__ }                        \
    else if ((E) <= 32) { constexpr int EBV = 32; __VA_ARGS__ }                        \
    else { constexpr int EBV = 64; __VA_ARGS__ }
extern "C" int go1_mlp_extra_backward(const float* dz, int lddz, int dz_transposed, const float* extra, int ldex, const float* w_extra, int ldw,
                                      float* g_w_extra, int ldgw, float* dextra, int ldde, int M, int o, int E, int accumulate, void* stream) {
    if (!dz || M <= 0 || o <= 0) return go1_set_error("go1_mlp_extra_backward: bad arguments");
    if (E < 1 || E > XWIDE_MAX_E) return go1_set_error("go1_mlp_extra_backward: E (trailing input columns) must be 1..64");
    if (!g_w_extra && !dextra) return go1_set_error("go1_mlp_extra_backward: nothing to compute (g_w_extra and dextra are NULL)");
    if (dextra && (!w_extra || ldw < E || ldde < E)) return go1_set_error("go1_mlp_extra_backward: dextra needs w_extra, ldw >= E and ldde >= E");
    if (g_w_extra && (!extra || ldex < E || ldgw < E)) return go1_set_error("go1_mlp_extra_backward: g_w_extra needs extra, ldex >= E and ldgw >= E");
    if (g_w_extra && dz_transposed) return go1_set_error("go1_mlp_extra_backward: the weight gradient takes dz as [M][o] (dz_transposed 0)");
    if (lddz < (dz_transposed ? M : o)) return go1_set_error("go1_mlp_extra_backward: lddz must be >= o ([M][o] dz) or >= M ([o][M] dz)");
    cudaStream_t st = (cudaStream_t)stream;
    const bool narrow = E <= 4 && !dz_transposed;      // the E <= 4 kernels, else the wide ones
    if (dextra) {
        if (narrow) extra_dinput_kernel<<<(M * 32 + 255) / 256, 256, 0, st>>>(dz, lddz, w_extra, ldw, dextra, ldde, M, o, E);
        else {
            const unsigned grid = (unsigned)((M + 127) / 128);
            if (dz_transposed) { XWIDE_EB_SWITCH(E, EB, extra_dinput_wide_kernel<EB, true><<<grid, 128, 0, st>>>(dz, lddz, w_extra, ldw, dextra, ldde, M, o, E);) }
            else { XWIDE_EB_SWITCH(E, EB, extra_dinput_wide_kernel<EB, false><<<grid, 128, 0, st>>>(dz, lddz, w_extra, ldw, dextra, ldde, M, o, E);) }
        }
        go1_count_launch(1);
    }
    if (g_w_extra) {
        if (!accumulate) { zero_small_kernel<<<(o * E + 255) / 256, 256, 0, st>>>(g_w_extra, ldgw, o, E); go1_count_launch(1); }
        int rpb = 64;
        dim3 grid((o + 255) / 256, (M + rpb - 1) / rpb);
        if (!narrow) {
            const int gx = (o + 127) / 128;
            const int gy = min((M + 31) / 32, max(1, (132 * 4 + gx - 1) / gx));     // ~4 CTAs per SM; fewer slabs, fewer atomics
            rpb = ((M + gy - 1) / gy + 31) / 32 * 32;
            grid = dim3(gx, (M + rpb - 1) / rpb);
        }
        const bool det = go1_det_on();     // deterministic mode: the row slabs' sums meet in g_w_extra in slab order
        float* part = go1_det_out<float>(det, st, (size_t)grid.y * o * E, nullptr);
        if (det && !part) return 1;
        if (narrow) (det ? extra_wgrad_kernel<true> : extra_wgrad_kernel<false>)<<<grid, 256, 0, st>>>(dz, lddz, extra, ldex, g_w_extra, ldgw, M, o, E, rpb, part);
        else { XWIDE_EB_SWITCH(E, EB, (det ? extra_wgrad_wide_kernel<EB, true> : extra_wgrad_wide_kernel<EB, false>)<<<grid, 128, 0, st>>>(dz, lddz, extra, ldex, g_w_extra, ldgw, M, o, E, rpb, part);) }
        go1_count_launch(1);
        if (det) {
            if (int e = cuda_rc("go1_mlp_extra_backward")) return e;
            if (int e = go1_det_sum(part, grid.y, (size_t)o * E, g_w_extra, o, E, ldgw, 1, st)) return e;
        }
    }
    return cuda_rc("go1_mlp_extra_backward");
}
__global__ void skinny_dgrad_kernel(const float* __restrict__ dz, int lddz, const float* __restrict__ W, int ldw, const float* __restrict__ y, int ldy,
                                    float* __restrict__ dprev, int lddp, int M, int o, int n, int kind) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)M * n) return;
    const int m = (int)(idx / n), c = (int)(idx - (size_t)m * n);
    float v = 0.f;
#pragma unroll
    for (int t = 0; t < 16; t++) if (t < o) v = fmaf(__ldg(dz + (size_t)m * lddz + t), __ldg(W + (size_t)t * ldw + c), v);
    if (y) { const float yy = y[(size_t)m * ldy + c]; v *= act_deriv_rt(kind, yy); }
    dprev[(size_t)m * lddp + c] = v;
}
// float4 variant: a warp owns rows (stride 8 inside the block's row slab), a lane owns 4 consecutive columns of a 128-column group and keeps
// its O x 4 weights in registers; the row's o output gradients are fetched by the first o lanes and shuffle-broadcast.  Optionally the
// column sums of the values written (= the bias gradient of the layer below) are reduced here as well: per-lane partial sums, one
// shared-memory reduction per block, one set of atomics per block.  OUT16: dprev is a BF16 matrix (uint16_t, lddp elements) that gets the
// values rounded to nearest even; the column sums see the fp32 values (go1_skinny_dgrad_act_bf16).  DET: colsum is the workspace, and the
// block's column sums go to colsum[blockIdx.y][n] (plain stores; go1_det_sum adds the slabs)
template <int O, int KIND, bool OUT16, bool DET>
__global__ void __launch_bounds__(256) skinny_dgrad4_kernel(const float* __restrict__ dz, int lddz, const float* __restrict__ W, int ldw, const float* __restrict__ y, int ldy,
                                                            float* __restrict__ dprev, int lddp, float* __restrict__ colsum, int M, int o, int n, int rows_per_block) {
    __shared__ float4 s_sum[8][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int c = blockIdx.x * 128 + lane * 4;
    const bool col_ok = c < n;
    float wr[O][4];
#pragma unroll
    for (int t = 0; t < O; t++) {
        const float4 ww = (t < o && col_ok) ? __ldg(reinterpret_cast<const float4*>(W + (size_t)t * ldw + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
        wr[t][0] = ww.x; wr[t][1] = ww.y; wr[t][2] = ww.z; wr[t][3] = ww.w;
    }
    const int r0 = blockIdx.y * rows_per_block, r1 = min(M, r0 + rows_per_block);
    float4 cs = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 2
    for (int m = r0 + w; m < r1; m += 8) {
        const float dl = lane < o ? __ldg(dz + (size_t)m * lddz + lane) : 0.f;
        float4 yy = make_float4(1.f, 1.f, 1.f, 1.f);
        if (y && col_ok) yy = __ldg(reinterpret_cast<const float4*>(y + (size_t)m * ldy + c));
        float v0 = 0.f, v1 = 0.f, v2 = 0.f, v3 = 0.f;
#pragma unroll
        for (int t = 0; t < O; t++) {
            const float d = __shfl_sync(0xffffffffu, dl, t);
            v0 = fmaf(d, wr[t][0], v0); v1 = fmaf(d, wr[t][1], v1); v2 = fmaf(d, wr[t][2], v2); v3 = fmaf(d, wr[t][3], v3);
        }
        if (y) { v0 *= act_deriv<KIND>(yy.x); v1 *= act_deriv<KIND>(yy.y); v2 *= act_deriv<KIND>(yy.z); v3 *= act_deriv<KIND>(yy.w); }
        if (OUT16) {
            if (col_ok) {
                uint16_t* d16 = reinterpret_cast<uint16_t*>(dprev) + (size_t)m * lddp + c;
                *reinterpret_cast<uint2*>(d16) = make_uint2((uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(v0)) | ((uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(v1)) << 16),
                                                            (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(v2)) | ((uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(v3)) << 16));
            }
        } else if (col_ok) *reinterpret_cast<float4*>(dprev + (size_t)m * lddp + c) = make_float4(v0, v1, v2, v3);
        cs.x += v0; cs.y += v1; cs.z += v2; cs.w += v3;
    }
    if (DET || colsum) {
        s_sum[w][lane] = cs;
        __syncthreads();
        if (w == 0 && col_ok) {
            float4 t = s_sum[0][lane];
#pragma unroll
            for (int k = 1; k < 8; k++) { t.x += s_sum[k][lane].x; t.y += s_sum[k][lane].y; t.z += s_sum[k][lane].z; t.w += s_sum[k][lane].w; }
            if constexpr (DET) *reinterpret_cast<float4*>(colsum + (size_t)blockIdx.y * n + c) = t;
            else { atomicAdd(colsum + c, t.x); atomicAdd(colsum + c + 1, t.y); atomicAdd(colsum + c + 2, t.z); atomicAdd(colsum + c + 3, t.w); }
        }
    }
}
// the launch of skinny_dgrad4 shared by go1_skinny_dgrad_act and its BF16 variant; deterministic mode: the column sums of the row slabs
// meet in colsum in slab order
template <bool OUT16>
static int launch_skinny_dgrad4(const float* dz, int lddz, const float* W, int ldw, const float* y_prev, int ldy, float* dprev, int lddp,
                                float* colsum, int M, int o, int n, int kind, cudaStream_t st, const char* what) {
    const int cb = (n + 127) / 128;
    int rpb = (M * cb + 2 * 132 - 1) / (2 * 132);           // about two blocks per SM
    rpb = (rpb + 7) / 8 * 8; if (rpb < 8) rpb = 8;
    dim3 grid(cb, (M + rpb - 1) / rpb);
    const bool det = colsum && go1_det_on();
    float* cs = go1_det_out(det, st, (size_t)grid.y * n, colsum);
    if (det && !cs) return 1;
#define LAUNCH(O, KD) (det ? skinny_dgrad4_kernel<O, KD, OUT16, true> : skinny_dgrad4_kernel<O, KD, OUT16, false>)<<<grid, 256, 0, st>>>(dz, lddz, W, ldw, y_prev, ldy, dprev, lddp, cs, M, o, n, rpb)
    GO1_ACT_SWITCH(kind, KD, if (o <= 2) LAUNCH(2, KD); else if (o <= 4) LAUNCH(4, KD); else LAUNCH(16, KD);)
#undef LAUNCH
    go1_count_launch(1);
    if (int e = cuda_rc(what)) return e;
    return det ? go1_det_sum(cs, grid.y, n, colsum, 1, n, n, 1, st) : 0;
}
extern "C" int go1_skinny_dgrad_act(const float* dz, int lddz, const float* W, int ldw, const float* y_prev, int ldy, float* dprev, int lddp,
                                    float* colsum, int M, int o, int n, int kind, void* stream) {
    if (!dz || !W || !dprev || M <= 0 || o <= 0 || o > 16 || n <= 0) return go1_set_error("go1_skinny_dgrad: bad arguments");
    if (!go1_act_kind_ok(kind)) return go1_set_error("go1_skinny_dgrad: unknown activation kind (Go1Activation)");
    cudaStream_t st = (cudaStream_t)stream;
    const bool vec = (n & 3) == 0 && (ldw & 3) == 0 && (lddp & 3) == 0 && (!y_prev || (ldy & 3) == 0) &&
                     ((((uintptr_t)W) | ((uintptr_t)dprev) | ((uintptr_t)(y_prev ? y_prev : W))) & 15) == 0;
    if (vec) return launch_skinny_dgrad4<false>(dz, lddz, W, ldw, y_prev, ldy, dprev, lddp, colsum, M, o, n, kind, st, "go1_skinny_dgrad");
    if (colsum) return go1_set_error("go1_skinny_dgrad_ex: the fused column sum needs 16-byte aligned operands with n % 4 == 0");
    const size_t tot = (size_t)M * n;
    skinny_dgrad_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(dz, lddz, W, ldw, y_prev, ldy, dprev, lddp, M, o, n, kind); go1_count_launch(1);
    return cuda_rc("go1_skinny_dgrad");
}
// go1_skinny_dgrad_act with a BF16 dprev (AC_Args.bf16_backward: the head's dgrad stores the hidden dz the BF16 products read)
extern "C" int go1_skinny_dgrad_act_bf16(const float* dz, int lddz, const float* W, int ldw, const float* y_prev, int ldy, uint16_t* dprev, int lddp,
                                         float* colsum, int M, int o, int n, int kind, void* stream) {
    if (!dz || !W || !dprev || M <= 0 || o <= 0 || o > 16 || n <= 0) return go1_set_error("go1_skinny_dgrad_act_bf16: bad arguments");
    if (!go1_act_kind_ok(kind)) return go1_set_error("go1_skinny_dgrad_act_bf16: unknown activation kind (Go1Activation)");
    if ((n & 3) || (ldw & 3) || (lddp & 3) || lddp < n || (y_prev && (ldy & 3)) || ((((uintptr_t)W) | ((uintptr_t)(y_prev ? y_prev : W))) & 15) || (((uintptr_t)dprev) & 7))
        return go1_set_error("go1_skinny_dgrad_act_bf16: n, ldw, lddp, ldy multiples of 4; W / y_prev 16-byte and dprev 8-byte aligned");
    return launch_skinny_dgrad4<true>(dz, lddz, W, ldw, y_prev, ldy, reinterpret_cast<float*>(dprev), lddp, colsum, M, o, n, kind, (cudaStream_t)stream, "go1_skinny_dgrad_act_bf16");
}
extern "C" int go1_skinny_dgrad_ex(const float* dz, int lddz, const float* W, int ldw, const float* y_prev, int ldy, float* dprev, int lddp,
                                   float* colsum, int M, int o, int n, void* stream) {
    return go1_skinny_dgrad_act(dz, lddz, W, ldw, y_prev, ldy, dprev, lddp, colsum, M, o, n, GO1_ACT_ELU, stream);
}
extern "C" int go1_skinny_dgrad(const float* dz, int lddz, const float* W, int ldw, const float* y_prev, int ldy, float* dprev, int lddp,
                                int M, int o, int n, void* stream) {
    return go1_skinny_dgrad_ex(dz, lddz, W, ldw, y_prev, ldy, dprev, lddp, nullptr, M, o, n, stream);
}

// Forward of a narrow output layer (the 12 / 2 / 1-wide heads, actor_critic.py:52,64,76): out[m][t] = b[t] + sum_k x[m][k] W[t][k], o <= 16.
// One bandwidth-bound pass over x (8 lanes per row, 16-byte loads; W and b in shared memory) instead of a padded 128 x 32 tensor-core tile.
__global__ void __launch_bounds__(256) skinny_forward_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ W, int ldw, const float* __restrict__ b,
                                                             float* __restrict__ out, int ldo, int M, int o, int K) {
    extern __shared__ float s_w[];              // [o][K] then [16] bias
    float* s_b = s_w + (size_t)o * K;
    for (int i = threadIdx.x; i < o * K; i += blockDim.x) s_w[i] = __ldg(W + (size_t)(i / K) * ldw + (i % K));
    if (threadIdx.x < 16) s_b[threadIdx.x] = (threadIdx.x < o && b) ? __ldg(b + threadIdx.x) : 0.f;
    __syncthreads();
    const int sub = threadIdx.x & 7;            // lane within the row's group of 8
    const int K4 = K >> 2;
    for (int m = blockIdx.x * (blockDim.x >> 3) + (threadIdx.x >> 3); m < M; m += gridDim.x * (blockDim.x >> 3)) {
        float acc[16];
#pragma unroll
        for (int t = 0; t < 16; t++) acc[t] = 0.f;
        const float4* xr = reinterpret_cast<const float4*>(x + (size_t)m * ldx);
        for (int c = sub; c < K4; c += 8) {
            const float4 v = __ldg(xr + c);
#pragma unroll
            for (int t = 0; t < 16; t++) {
                if (t < o) {
                    const float4 w = *reinterpret_cast<const float4*>(s_w + (size_t)t * K + 4 * c);
                    acc[t] = fmaf(v.x, w.x, fmaf(v.y, w.y, fmaf(v.z, w.z, fmaf(v.w, w.w, acc[t]))));
                }
            }
        }
#pragma unroll
        for (int t = 0; t < 16; t++) {
            if (t < o) {
                float a = acc[t];
                a += __shfl_xor_sync(0xffffffffu, a, 1); a += __shfl_xor_sync(0xffffffffu, a, 2); a += __shfl_xor_sync(0xffffffffu, a, 4);
                if (sub == (t & 7)) out[(size_t)m * ldo + t] = a + s_b[t];
            }
        }
    }
}
extern "C" int go1_skinny_forward(const float* x, int ldx, const float* W, int ldw, const float* b, float* out, int ldo, int M, int o, int K, void* stream) {
    if (!x || !W || !out || M <= 0 || o <= 0 || o > 16 || K <= 0 || (K & 3) || (ldx & 3) || (((uintptr_t)x) & 15) || (size_t)(o * K + 16) * 4 > 48 * 1024)
        return go1_set_error("go1_skinny_forward: bad arguments (o <= 16, K % 4 == 0, x 16-byte aligned rows)");
    const int rows_per_block = 32;
    int grid = (M + rows_per_block - 1) / rows_per_block;
    if (grid > 132 * 8) grid = 132 * 8;
    skinny_forward_kernel<<<grid, 256, (size_t)(o * K + 16) * 4, (cudaStream_t)stream>>>(x, ldx, W, ldw, b, out, ldo, M, o, K); go1_count_launch(1);
    return cuda_rc("go1_skinny_forward");
}

// ---------------------------------------------------------------------------------------------
// RolloutStorage.add_transitions (rollout_storage.py:55-69) + the time-out bootstrap of PPO.process_env_step
// (ppo.py:84-86) in one launch: the 2100-wide history row is the bulk (float4 copy), the small fields ride along.
// ---------------------------------------------------------------------------------------------
struct StoreArgs {
    const float *obs, *priv, *hist, *actions, *rewards, *values, *logp, *mean, *std, *env_bins;
    const uint8_t *dones, *time_outs;
    float *s_obs, *s_priv, *s_hist, *s_actions, *s_rewards, *s_values, *s_logp, *s_mu, *s_sigma, *s_env_bins;
    uint8_t* s_dones;
    const int* slot_dev;          // optional: the output pointers are slab BASES and the slot index is read from device memory
    int n, nobs, npriv, nhist, nact; float gamma;
};
__global__ void __launch_bounds__(256) store_transition_kernel(StoreArgs a) {
    const int e = blockIdx.x;
    if (e >= a.n) return;
    const int t = threadIdx.x;
    if (a.slot_dev) {
        const size_t off = (size_t)(*a.slot_dev) * a.n;
        a.s_obs += off * a.nobs; a.s_priv += off * a.npriv; if (a.hist) a.s_hist += off * a.nhist; a.s_actions += off * a.nact; a.s_rewards += off;
        a.s_values += off; a.s_logp += off; a.s_mu += off * a.nact; a.s_sigma += off * a.nact; a.s_env_bins += off; a.s_dones += off;
    }
    if (!a.hist) {
        // (the history is stored by go1_rollout_store_rows_bf16: AC_Args.gemm_impl = 2 keeps a BF16 slab)
    } else if ((a.nhist & 3) == 0) {
        const float4* src = reinterpret_cast<const float4*>(a.hist + (size_t)e * a.nhist);
        float4* dst = reinterpret_cast<float4*>(a.s_hist + (size_t)e * a.nhist);
        for (int c = t; c < a.nhist / 4; c += blockDim.x) dst[c] = src[c];
    } else {
        for (int c = t; c < a.nhist; c += blockDim.x) a.s_hist[(size_t)e * a.nhist + c] = a.hist[(size_t)e * a.nhist + c];
    }
    if (a.obs) for (int c = t; c < a.nobs; c += blockDim.x) a.s_obs[(size_t)e * a.nobs + c] = a.obs[(size_t)e * a.nobs + c];
    if (a.priv && t < a.npriv) a.s_priv[(size_t)e * a.npriv + t] = a.priv[(size_t)e * a.npriv + t];
    if (t < a.nact) {
        a.s_actions[(size_t)e * a.nact + t] = a.actions[(size_t)e * a.nact + t];
        a.s_mu[(size_t)e * a.nact + t] = a.mean[(size_t)e * a.nact + t];
        a.s_sigma[(size_t)e * a.nact + t] = a.std[t];
    }
    if (t == 0) {
        const float v = a.values[e];
        float r = a.rewards[e];
        // rewards += gamma * (values * time_outs): a rounded product, then a rounded add (ppo.py:84-86), never an FMA
        if (a.time_outs) r = __fadd_rn(r, __fmul_rn(a.gamma, a.time_outs[e] ? v : 0.0f));
        a.s_rewards[e] = r; a.s_values[e] = v; a.s_logp[e] = a.logp[e]; a.s_dones[e] = a.dones[e] ? 1 : 0;
        a.s_env_bins[e] = a.env_bins ? a.env_bins[e] : 0.f;
    }
}
// obs / privileged obs of the step the policy is ABOUT to act on: copied at act() time, before env.step overwrites the env's buffers
__global__ void store_observations_kernel(const float* __restrict__ obs, const float* __restrict__ priv, float* __restrict__ s_obs,
                                          float* __restrict__ s_priv, size_t n_obs, size_t n_priv, const int* __restrict__ slot_dev) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t slot = slot_dev ? (size_t)*slot_dev : 0;
    if (i < n_obs) s_obs[slot * n_obs + i] = obs[i];
    if (i < n_priv) s_priv[slot * n_priv + i] = priv[i];
}
extern "C" int go1_store_observations(const float* obs, const float* priv, float* s_obs, float* s_priv, int n, int nobs, int npriv, void* stream) {
    if (!obs || !s_obs || n <= 0 || nobs <= 0 || npriv < 0 || (npriv > 0 && (!priv || !s_priv))) return go1_set_error("go1_store_observations: bad arguments");
    const size_t n_obs = (size_t)n * nobs, n_priv = (size_t)n * npriv;
    store_observations_kernel<<<(unsigned)((n_obs + 255) / 256), 256, 0, (cudaStream_t)stream>>>(obs, priv, s_obs, s_priv, n_obs, n_priv, nullptr); go1_count_launch(1);
    return cuda_rc("go1_store_observations");
}

// ---- the same two stores with the slot index in device memory: one captured CUDA graph serves every step of the rollout ----
extern "C" int go1_rollout_store_observations(const float* obs, const float* priv, float* s_obs_base, float* s_priv_base, const int32_t* slot_dev,
                                              int n, int nobs, int npriv, void* stream) {
    if (!obs || !s_obs_base || !slot_dev || n <= 0 || nobs <= 0 || npriv < 0 || (npriv > 0 && (!priv || !s_priv_base)))
        return go1_set_error("go1_rollout_store_observations: bad arguments");
    const size_t n_obs = (size_t)n * nobs, n_priv = (size_t)n * npriv;
    store_observations_kernel<<<(unsigned)((n_obs + 255) / 256), 256, 0, (cudaStream_t)stream>>>(obs, priv, s_obs_base, s_priv_base, n_obs, n_priv, slot_dev);
    go1_count_launch(1);
    return cuda_rc("go1_rollout_store_observations");
}

// Ends one env step of a graph-replayed rollout: files the step's extras["train/episode"] accumulator (episode sums of the envs reset in
// this step + their count; a step without a reset carries the previous entry forward, like the reference's extras entry that just
// stays in place) under the step's slot, then advances the slot index and the device-side common_step_counter.
__global__ void rollout_advance_kernel(const float* __restrict__ acc, float* __restrict__ acc_hist, int W, int T, int* slot_dev, long long* step_dev) {
    const int t = *slot_dev;
    const int i = threadIdx.x;
    if (acc && acc_hist && i < W) {
        float v = acc[i];
        if (acc[W - 1] == 0.0f) v = acc_hist[(size_t)((t + T - 1) % T) * W + i];
        acc_hist[(size_t)t * W + i] = v;
    }
    __syncthreads();
    if (i == 0) { *slot_dev = (t + 1) % T; if (step_dev) *step_dev += 1; }
}
extern "C" int go1_rollout_advance(const float* acc, float* acc_hist, int W, int T, int32_t* slot_dev, int64_t* step_dev, void* stream) {
    if (!slot_dev || T <= 0 || W < 0 || W > 256) return go1_set_error("go1_rollout_advance: bad arguments");
    rollout_advance_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(acc, acc_hist, W, T, slot_dev, (long long*)step_dev); go1_count_launch(1);
    return cuda_rc("go1_rollout_advance");
}

extern "C" int go1_store_transition(const float* const* in_f32, const uint8_t* dones, const uint8_t* time_outs, float* const* out_f32, uint8_t* s_dones,
                                    int n, int nobs, int npriv, int nhist, int nact, float gamma, void* stream) {
    if (!in_f32 || !out_f32 || !dones || !s_dones || n <= 0 || nact > 256 || npriv > 256) return go1_set_error("go1_store_transition: bad arguments");
    StoreArgs a;
    a.obs = in_f32[0]; a.priv = in_f32[1]; a.hist = in_f32[2]; a.actions = in_f32[3]; a.rewards = in_f32[4]; a.values = in_f32[5];
    a.logp = in_f32[6]; a.mean = in_f32[7]; a.std = in_f32[8]; a.env_bins = in_f32[9];
    a.dones = dones; a.time_outs = time_outs;
    a.s_obs = out_f32[0]; a.s_priv = out_f32[1]; a.s_hist = out_f32[2]; a.s_actions = out_f32[3]; a.s_rewards = out_f32[4]; a.s_values = out_f32[5];
    a.s_logp = out_f32[6]; a.s_mu = out_f32[7]; a.s_sigma = out_f32[8]; a.s_env_bins = out_f32[9]; a.s_dones = s_dones;
    a.n = n; a.nobs = nobs; a.npriv = npriv; a.nhist = nhist; a.nact = nact; a.gamma = gamma; a.slot_dev = nullptr;
    for (int i = 3; i < 9; i++) if (!in_f32[i] || !out_f32[i]) return go1_set_error("go1_store_transition: null tensor");
    if (in_f32[2] && !out_f32[2]) return go1_set_error("go1_store_transition: null tensor");
    if ((in_f32[0] && !out_f32[0]) || (in_f32[1] && !out_f32[1])) return go1_set_error("go1_store_transition: null tensor");
    if (!out_f32[9]) return go1_set_error("go1_store_transition: null tensor");
    store_transition_kernel<<<n, 256, 0, (cudaStream_t)stream>>>(a); go1_count_launch(1);
    return cuda_rc("go1_store_transition");
}
extern "C" int go1_rollout_store_transition(const float* const* in_f32, const uint8_t* dones, const uint8_t* time_outs, float* const* out_base_f32,
                                            uint8_t* s_dones_base, const int32_t* slot_dev, int n, int nobs, int npriv, int nhist, int nact, float gamma,
                                            void* stream) {
    if (!in_f32 || !out_base_f32 || !dones || !s_dones_base || !slot_dev || n <= 0 || nact > 256 || npriv > 256)
        return go1_set_error("go1_rollout_store_transition: bad arguments");
    StoreArgs a;
    a.obs = in_f32[0]; a.priv = in_f32[1]; a.hist = in_f32[2]; a.actions = in_f32[3]; a.rewards = in_f32[4]; a.values = in_f32[5];
    a.logp = in_f32[6]; a.mean = in_f32[7]; a.std = in_f32[8]; a.env_bins = in_f32[9];
    a.dones = dones; a.time_outs = time_outs;
    a.s_obs = out_base_f32[0]; a.s_priv = out_base_f32[1]; a.s_hist = out_base_f32[2]; a.s_actions = out_base_f32[3]; a.s_rewards = out_base_f32[4];
    a.s_values = out_base_f32[5]; a.s_logp = out_base_f32[6]; a.s_mu = out_base_f32[7]; a.s_sigma = out_base_f32[8]; a.s_env_bins = out_base_f32[9];
    a.s_dones = s_dones_base; a.slot_dev = slot_dev;
    a.n = n; a.nobs = nobs; a.npriv = npriv; a.nhist = nhist; a.nact = nact; a.gamma = gamma;
    for (int i = 3; i < 9; i++) if (!in_f32[i] || !out_base_f32[i]) return go1_set_error("go1_rollout_store_transition: null tensor");
    if (in_f32[2] && !out_base_f32[2]) return go1_set_error("go1_rollout_store_transition: null tensor");
    if (!out_base_f32[9] || (in_f32[0] && !out_base_f32[0]) || (in_f32[1] && !out_base_f32[1])) return go1_set_error("go1_rollout_store_transition: null tensor");
    store_transition_kernel<<<n, 256, 0, (cudaStream_t)stream>>>(a); go1_count_launch(1);
    return cuda_rc("go1_rollout_store_transition");
}
