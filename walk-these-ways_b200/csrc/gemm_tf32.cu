// gemm_tf32.cu — hand-written wgmma TF32 GEMM for sm_90a (the dense layers of ppo_cse's ActorCritic).
//
//   C[M][N] (+)= A[M][K] * B[N][K]^T (+ bias[n]) (activation)   fp32 in HBM, TF32 multiply, fp32 accumulate
//
// The forward products read both operands K-major (A = activations row-major, B = torch.nn.Linear weight [out][in]).
// dgrad (B = W as [K][N]) and wgrad (A = dz as [K][M], B = activations as [K][N]) have MN-major operands, and TF32 wgmma
// multiplies K-major shared-memory tiles only: their TMA boxes ([32 k-rows][tile width], unswizzled) are transposed by the
// consumer warps from shared memory to shared memory (into the 128B-swizzled K-major form, double-buffered so that the
// transposition of k-block i + 1 overlaps the tensor-core work on k-block i).  That costs 64 KB of shared-memory traffic per
// 128 x 128 k-block on top of 80 KB of TMA writes and wgmma reads, plus a wait and a barrier per k-block.  The two largest
// wgrads, the first layers' (1280 x 2105 and 256 x 2101 over M = 24576), read K-major copies instead: the history transposed once
// per update (go1_transpose, [2105][24576] per minibatch: 207 MB each, 830 MB for the four minibatches at 4096 envs) and dz stored
// transposed by the dgrad epilogue that produces it (store_transposed).  On an H100 SXM (700 W): 1299 -> 565 us and
// 206 -> 137 us per launch.  The dgrads' W and the layer-2/3 wgrads are still transposed on the SM in TF32; with BF16 operands
// (gemm_bf16_mn_wgmma, AC_Args.bf16_backward) they are read in place as 128B-swizzled MN-major boxes through wgmma's transpose immediates.
// Structure (persistent CTAs, one per SM, 384 threads, walking 128 x BN output tiles):
//   warps 0-7   two consumer warpgroups, 64 rows x BN columns each: wgmma.mma_async m64nBNk8 (4 per k-block) with the accumulator
//               in registers, then the epilogue: accumulator -> swizzled shared memory -> one 32 x 32 block per warp at a time,
//               a row per lane -> bias / activation / its derivative / column sums / trailing-input terms -> the same block -> one TMA store
//               (staged epilogue), red.global.add.v4 when split-K partitions the reduction
//   warp 8      TMA producer: cp.async.bulk.tensor 2D loads of the A and B boxes of a k-block into a ring of 3-8 stages guarded by
//               full / empty mbarriers; it runs ahead into the next tile while the consumers are in their epilogue
// The long-K products with K-major operands (the first layers' forward and weight gradient) run as clusters of two CTAs working
// adjacent tiles: each CTA loads half of the operand box the pair shares and multicasts it to both, so the pair reads 24 KB instead
// of 32 KB per k-block from L2 (full-chip, these products are bound by the L2-to-SM operand stream, not by the tensor cores).
// mlp_tail_fwd_kernel chains two such products and a CUDA-core head for the layers behind a first layer.
#include <cuda_runtime.h>
#include <cuda.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <mutex>
#include <unordered_map>
#include <stdlib.h>
#include "../../include/go1_b200.h"
#include "wgmma_tf32.cuh"
#include "activation.cuh"
#include "deterministic.cuh"

extern int go1_set_error(const char* m);
void go1_count_launch(int n);

namespace {

constexpr int BM = 128, BK = 32;          // BK fp32 = 128 bytes = one swizzle-128B row
constexpr int NCONS = 8, EPI_G = 2;       // consumer warps; column groups of the epilogue (warp = (32-row block, column group))

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done = 0;
    const uint32_t a = smem_u32(bar);
    while (!done) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(a), "r"(parity) : "memory");
    }
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// the same box delivered to the same shared-memory offset and mbarrier of every CTA of the cluster in cta_mask
__device__ __forceinline__ void tma_load_2d_multicast(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, uint16_t cta_mask) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask) : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// every thread of every CTA of the cluster (threads may arrive from different places in the code)
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `rank` of the cluster.  Default (.release.cta) semantics.  The only
// ordering this arrive provides is read-before-write: the caller's wgmma.wait_group has retired the tensor core's (async-proxy) reads of
// the stage before the peer's TMA overwrites it.  It publishes no generic-proxy writes to the peer at cluster scope, and nothing may come
// to rely on it doing so.  (A .release.cluster arrive would also wait for the thread's outstanding global writes, once per k-block.)
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(rank));
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
// named barriers of the consumer warps (the producer warp never joins them): 1 = both warpgroups, 2 / 3 = one warpgroup
__device__ __forceinline__ void cons_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void wg_sync(int wgi) { asm volatile("bar.sync %0, 128;" ::"r"(2 + wgi) : "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// MN-major operand box as TMA delivers it, raw[32 k][W mn], -> the K-major tile wgmma reads: dst[mn][32 k], 128-byte rows whose
// 16-byte chunks are XOR-swizzled by row % 8.  All 256 consumer threads; a warp reads 32 consecutive mn of one k (conflict-free)
// and writes 32 rows x 16 bytes that cover every bank group four times (the minimum for 512 bytes).
template <int W>
__device__ __forceinline__ void transpose_tile(const float* __restrict__ raw, uint8_t* dst, const int ctid) {
#pragma unroll
    for (int it = 0; it < W * 8 / 256; it++) {
        const int idx = ctid + 256 * it;
        const int mn = idx % W, kq = idx / W;
        const float* r = raw + (size_t)(4 * kq) * W + mn;
        *reinterpret_cast<float4*>(dst + mn * 128 + ((kq ^ (mn & 7)) << 4)) = make_float4(r[0], r[W], r[2 * W], r[3 * W]);
    }
}

// Accumulator fragment of a 64 x (8 NJ) warpgroup tile -> shared memory as [32-column chunk][64 rows][128 bytes], swizzled like a
// TMA box: every 32 x 32 block of it is 4 KB that a TMA store can send and that the tensor core can read as a K-major k-block.
// f(v, column) is applied to every value on the way; column = first column of the pair.
template <int NJ, typename F>
__device__ __forceinline__ void store_fragment(const float (&acc)[4 * NJ], uint8_t* tile, const int col_base, const int w, const int lane, F f) {
    const int rb = 16 * w + (lane >> 2);
#pragma unroll
    for (int j = 0; j < NJ; j++) {
        const int col = col_base + 8 * j + 2 * (lane & 3);
        uint8_t* p = tile + (size_t)(col >> 5) * (64 * 128) + rb * 128 + ((((col & 31) >> 2) ^ (rb & 7)) << 4) + (lane & 1) * 8;
        *reinterpret_cast<float2*>(p) = f(make_float2(acc[4 * j], acc[4 * j + 1]), col, 0);
        *reinterpret_cast<float2*>(p + 8 * 128) = f(make_float2(acc[4 * j + 2], acc[4 * j + 3]), col, 1);
    }
}

// The activations are act_fast / act_deriv of activation.cuh: their results feed TF32 products (relative operand rounding 5e-4) and the
// derivative-from-output forms of the backward pass.  The kind is a warp-uniform kernel argument; GO1_ACT_SWITCH dispatches on it around
// each unrolled loop.  The kernels whose register budget is full (the persistent GEMM, the fused tails) exist twice: ANYKIND = false
// is the ELU-only code (the switch folds away), ANYKIND = true carries the switch and serves the other kinds.

struct GemmArgs {
    float* C; const float* bias;
    int M, N, K, ldc, act, kind, accumulate, kb_per_split;      // kind: Go1Activation behind act 1 / 2
    const float* ex; const float* wex; const float* aux;      // fused epilogue operands (see Go1GemmEpilogue)
    int ldex, ldwex, nex, ldaux;
    int lead;                // > 0: extra columns + activation only for output columns < lead
    int amn, bmn;            // operand is MN-major in HBM (A given as [K][M], B given as [K][N]); persistent kernel only
    int ct;                  // C is stored transposed, element (m, n) at C[n * ldc + m]: staged epilogue only (tma_store)
    int c16;                 // with ct: the transposed blocks leave as BF16 (round to nearest even) through a BF16 map of the output
    float* colsum;           // optional [N]: += column sums of the values written (bias gradient fused into the dgrad epilogue)
    const float* bx; const float* bwx; float* gwx; float* dx;     // fused trailing-input backward (see Go1GemmEpilogue)
    int ldbx, ldbwx, ldgwx, lddx, nbx;
    int tma_store, tma_aux;  // staged epilogue: C blocks leave / derivative operand blocks arrive through shared memory by TMA
    // grouped launch (persistent kernel): nprob problems of the same shape and operand strides in one grid; tile t belongs to problem
    // t / tiles_per_prob, whose operands are maps.a/b[p] and whose output is Cg[p] (no per-problem epilogue operands: split-K wgrads)
    float* Cg[4]; int nprob, tiles_per_prob;
};
constexpr int GEMM_MAXP = 4;
// Deterministic mode (go1_set_deterministic): where the plain kernels add into their targets with atomics, the DET instantiations store
// partials to the stream's workspace and go1_det_sum adds them in a fixed order:
//   split    [problem][split][M][ldc]  the split-K partial tiles (slab = M x ldc floats)
//   cs       [M / 32][N]               colsum: the column sums of each 32-row block
//   gwx      [M / 32][N][nbx]          the trailing-input weight gradient of each 32-row block
//   dx       [N / 32][M][nbx]          the trailing-input gradient of each 32-column chunk
struct DetArgs { float* split; size_t slab; int nsplit; float* cs; float* gwx; float* dx; };
// half: the 64-row box of the operand a CTA pair shares (cluster launches: see gemm_tf32_wgmma)
struct GemmMaps { CUtensorMap a[GEMM_MAXP], b[GEMM_MAXP], half; };

// Per-warp shared-memory staging of the staged epilogue.  A row-per-lane float4 store touches 32 different 128-byte lines per
// instruction (8 x the LSU wavefronts of a coalesced store), which bounds every short-K product.  Staged: the warp's
// 32 x 32 block is written to shared memory (128B-swizzled: conflict-free 16-byte accesses) and ONE thread hands it to the TMA unit.
struct EpiStage {
    uint8_t* out;            // 4 KB, 1024-byte aligned: the block the values came from, or nullptr: direct global stores
    const CUtensorMap* mapC;
    const uint8_t* aux;      // 4 KB block of the derivative operand (the saved activation), fetched by TMA and already waited for, or nullptr
};
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1) : "memory");
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    return (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(lo)) | ((uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(hi)) << 16);
}

// act == 2 of one chunk: v[j] *= f'(z) from the saved activation, wherever this chunk's 32 values of it are (see epilogue_chunk)
template <typename D>
__device__ __forceinline__ void epilogue_dact(const D dact, const GemmArgs& g, float (&v)[32], const int row, const int col0, const int ncols, const int lane,
                                              const float4 (&ypre)[8], const bool have_pre, const EpiStage& es) {
    const float* arow = g.aux + (size_t)row * g.ldaux + col0;
    if (es.aux) {          // the operand block sits in shared memory (TMA, 128B swizzle: 16-byte chunk j of row l at (j ^ (l & 7)))
        const uint8_t* srow = es.aux + lane * 128;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const float4 y = *reinterpret_cast<const float4*>(srow + ((j ^ (lane & 7)) << 4));
            v[4 * j] *= dact(y.x); v[4 * j + 1] *= dact(y.y); v[4 * j + 2] *= dact(y.z); v[4 * j + 3] *= dact(y.w);
        }
    } else if (have_pre) { // the operand was fetched before the accumulator was ready (epilogue_prefetch)
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const float4 y = ypre[j];
            v[4 * j] *= dact(y.x); v[4 * j + 1] *= dact(y.y); v[4 * j + 2] *= dact(y.z); v[4 * j + 3] *= dact(y.w);
        }
    } else if (ncols == 32 && (g.ldaux & 3) == 0 && ((((uintptr_t)g.aux) & 15) == 0) && ((col0 & 3) == 0)) {
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const float4 y = __ldg(reinterpret_cast<const float4*>(arow) + j);
            v[4 * j] *= dact(y.x); v[4 * j + 1] *= dact(y.y); v[4 * j + 2] *= dact(y.z); v[4 * j + 3] *= dact(y.w);
        }
    } else {
#pragma unroll
        for (int j = 0; j < 32; j++) if (j < ncols) v[j] *= dact(__ldg(arow + j));
    }
}

// Column sums of a 32 x 32 block held one row per lane (sred[j] = column j; overwritten) by a transpose-reduce: 31 shuffles for 32
// columns (each halving step trades half of the columns for the partner's partial sums).  Lane l ends up with column l.
__device__ __forceinline__ float transpose_reduce32(float (&sred)[32], const int lane) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        const bool upper = (lane & off) != 0;
#pragma unroll
        for (int j = 0; j < off; j++) {
            const float send = upper ? sred[j] : sred[j + off];
            const float keep = upper ? sred[j + off] : sred[j];
            sred[j] = keep + __shfl_xor_sync(0xffffffffu, send, off);
        }
    }
    return sred[0];
}

// Epilogue of one 32-column chunk held in registers (thread = output row, r[j] = column col0 + j).  Called by all 32 lanes
// of an epilogue warp (the per-column operands -- bias, extra-input weights -- are loaded once per lane and broadcast
// with shuffles instead of 32 x per-thread global loads, which made the rank-2 term the slowest part of the kernel).
template <bool ANYKIND, bool ROW16 = false, bool DET = false>
__device__ __forceinline__ void epilogue_chunk(const GemmArgs& g, float* const Cbase, uint32_t (&r)[32], const int row, const int col0, const bool split, const int lane,
                                               const float4 (&ypre)[8], const bool have_pre, const EpiStage& es, const DetArgs* det = nullptr) {
    if (col0 >= g.N) return;                                    // warp-uniform
    const int ncols = min(32, g.N - col0);
    const bool row_ok = row < g.M;
    float* crow = Cbase + (size_t)(row_ok ? row : 0) * g.ldc + col0;
    if constexpr (DET) {
        if (split) {        // split-K partial tile: stored into this split's slab of the workspace (Cbase)
            if (row_ok) {
                if ((ncols == 32) && ((g.ldc & 3) == 0) && ((((uintptr_t)Cbase) & 15) == 0) && ((col0 & 3) == 0)) {
#pragma unroll
                    for (int j = 0; j < 8; j++)
                        reinterpret_cast<float4*>(crow)[j] = make_float4(__uint_as_float(r[4 * j]), __uint_as_float(r[4 * j + 1]), __uint_as_float(r[4 * j + 2]),
                                                                         __uint_as_float(r[4 * j + 3]));
                } else {
#pragma unroll
                    for (int j = 0; j < 32; j++) if (j < ncols) crow[j] = __uint_as_float(r[j]);
                }
            }
            return;
        }
    }
    if (split) {            // split-K partial tile: reduce into C; 16-byte vector reductions cut the L2 atomic operations 4x
        if (row_ok) {
            if ((ncols == 32) && ((g.ldc & 3) == 0) && ((((uintptr_t)Cbase) & 15) == 0) && ((col0 & 3) == 0)) {
#pragma unroll
                for (int j = 0; j < 8; j++)
                    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(crow + 4 * j), "f"(__uint_as_float(r[4 * j])), "f"(__uint_as_float(r[4 * j + 1])),
                                 "f"(__uint_as_float(r[4 * j + 2])), "f"(__uint_as_float(r[4 * j + 3])) : "memory");
            } else {
#pragma unroll
                for (int j = 0; j < 32; j++) if (j < ncols) atomicAdd(crow + j, __uint_as_float(r[j]));
            }
        }
        return;
    }
    const bool vec = (ncols == 32) && ((g.ldc & 3) == 0) && ((((uintptr_t)Cbase) & 15) == 0) && ((col0 & 3) == 0);
    float v[32];
#pragma unroll
    for (int j = 0; j < 32; j++) v[j] = __uint_as_float(r[j]);
    if (g.accumulate && row_ok) {
        if (vec) {
#pragma unroll
            for (int j = 0; j < 8; j++) { const float4 o = reinterpret_cast<const float4*>(crow)[j]; v[4 * j] += o.x; v[4 * j + 1] += o.y; v[4 * j + 2] += o.z; v[4 * j + 3] += o.w; }
        } else {
#pragma unroll
            for (int j = 0; j < 32; j++) if (j < ncols) v[j] += crow[j];
        }
    }
    const int cj = col0 + lane;                                  // the column whose per-column operands this lane fetches
    const bool lead_j = cj < g.N && (g.lead <= 0 || cj < g.lead);
    if (g.nex > 0) {        // rank-nex update from the trailing input columns (cat(obs_history, latent))
        float e[4], wl[4];
#pragma unroll
        for (int t = 0; t < 4; t++) {
            e[t] = (t < g.nex && row_ok) ? __ldg(g.ex + (size_t)row * g.ldex + t) : 0.f;
            wl[t] = (t < g.nex && lead_j) ? __ldg(g.wex + (size_t)cj * g.ldwex + t) : 0.f;
        }
        if (g.nex <= 2) {
#pragma unroll
            for (int j = 0; j < 32; j++)
                v[j] += fmaf(e[1], __shfl_sync(0xffffffffu, wl[1], j), e[0] * __shfl_sync(0xffffffffu, wl[0], j));
        } else {
#pragma unroll
            for (int j = 0; j < 32; j++) {
                float a = e[0] * __shfl_sync(0xffffffffu, wl[0], j);
                a = fmaf(e[1], __shfl_sync(0xffffffffu, wl[1], j), a);
                a = fmaf(e[2], __shfl_sync(0xffffffffu, wl[2], j), a);
                v[j] += fmaf(e[3], __shfl_sync(0xffffffffu, wl[3], j), a);
            }
        }
    }
    if (g.bias) {
        const float bl = cj < g.N ? __ldg(g.bias + cj) : 0.f;
#pragma unroll
        for (int j = 0; j < 32; j++) v[j] += __shfl_sync(0xffffffffu, bl, j);
    }
    const int kind = ANYKIND ? g.kind : (int)GO1_ACT_ELU;
    if (row_ok) {
    if (g.act == 1) {
        const int nlead = g.lead <= 0 ? 32 : max(0, min(32, g.lead - col0));      // leading columns of this chunk that get the activation
        GO1_ACT_SWITCH(kind, KD,
            _Pragma("unroll")
            for (int j = 0; j < 32; j++) if (j < nlead) v[j] = act_fast<KD>(v[j]);)
    } else if (g.act == 2) {   // multiply by f'(z) from the saved activation y (ELU: 1 if y > 0 else y + 1)
        if (ANYKIND) epilogue_dact(act_deriv_coefficients(kind), g, v, row, col0, ncols, lane, ypre, have_pre, es);
        else epilogue_dact([](float y) { return act_deriv<GO1_ACT_ELU>(y); }, g, v, row, col0, ncols, lane, ypre, have_pre, es);
    }
    }
    if (g.colsum) {         // warp-uniform.  Column sums over the warp's 32 rows, then one atomic per lane
        float sred[32];
#pragma unroll
        for (int j = 0; j < 32; j++) sred[j] = (row_ok && j < ncols) ? v[j] : 0.f;
        const float s = transpose_reduce32(sred, lane);
        // (DET: a 32-row block that starts at or beyond M -- the last tile's, when M % 128 is 1..96 -- has no slot among the M / 32 partials)
        if constexpr (DET) { if (lane < ncols && row - lane < g.M) det->cs[(size_t)(row >> 5) * g.N + col0 + lane] = s; }
        else if (lane < ncols) atomicAdd(g.colsum + col0 + lane, s);
    }
    if (g.nbx > 0) {        // warp-uniform.  C is the dz of a first layer with nbx trailing inputs: their weight gradient (column sums weighted by the
        const int cjx = col0 + lane;                     // row's trailing inputs) and input gradient (row dots with the trailing-input weights)
#pragma unroll
        for (int t = 0; t < 4; t++) {
            if (t < g.nbx) {
                if (g.gwx) {        // (NULL: the caller gets this weight gradient elsewhere -- from augmented input columns of the first-layer wgrad)
                const float e = row_ok ? __ldg(g.bx + (size_t)row * g.ldbx + t) : 0.f;
                float sred[32];
#pragma unroll
                for (int j = 0; j < 32; j++) sred[j] = (row_ok && j < ncols) ? v[j] * e : 0.f;
                const float s = transpose_reduce32(sred, lane);
                if constexpr (DET) { if (lane < ncols && row - lane < g.M) det->gwx[((size_t)(row >> 5) * g.N + cjx) * g.nbx + t] = s; }
                else if (lane < ncols) atomicAdd(g.gwx + (size_t)cjx * g.ldgwx + t, s);
                }
                if (g.dx) {
                    const float wl = lane < ncols ? __ldg(g.bwx + (size_t)cjx * g.ldbwx + t) : 0.f;
                    float acc = 0.f;
#pragma unroll
                    for (int j = 0; j < 32; j++) acc = fmaf(v[j], __shfl_sync(0xffffffffu, wl, j), acc);      // wl = 0 beyond ncols
                    if constexpr (DET) { if (row_ok) det->dx[((size_t)(col0 >> 5) * g.M + row) * g.nbx + t] = acc; }
                    else if (row_ok) atomicAdd(g.dx + (size_t)row * g.lddx + t, acc);
                }
            }
        }
    }
    if (ROW16 && g.c16 && !g.ct) {      // row-major BF16 C (C is then a uint16_t matrix with row stride ldc elements): rounded after every term above
        if (es.out) {       // the block as 32 rows of 64 bytes, 64B-swizzled (chunk j of row l at j ^ ((l / 2) % 4): conflict-free), one TMA store
            __syncwarp();   // (it overlays the fp32 rows of the block: every lane has read its row)
            uint8_t* srow = es.out + lane * 64;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                uint4 o;
                o.x = pack_bf16x2(v[8 * j], v[8 * j + 1]); o.y = pack_bf16x2(v[8 * j + 2], v[8 * j + 3]);
                o.z = pack_bf16x2(v[8 * j + 4], v[8 * j + 5]); o.w = pack_bf16x2(v[8 * j + 6], v[8 * j + 7]);
                *reinterpret_cast<uint4*>(srow + ((j ^ ((lane >> 1) & 3)) << 4)) = o;
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) {
                tma_store_2d(es.mapC, es.out, col0, row);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        } else if (row_ok) {
            uint16_t* c16 = reinterpret_cast<uint16_t*>(Cbase) + (size_t)row * g.ldc + col0;
#pragma unroll
            for (int j = 0; j < 32; j++) if (j < ncols) c16[j] = __bfloat16_as_ushort(__float2bfloat16_rn(v[j]));
        }
        return;
    }
    if (es.out) {           // warp-uniform: all 32 lanes stage their row (rows / columns beyond M / N are clipped by the TMA store)
        if (g.ct && g.c16) {    // BF16 block of C^T, unswizzled 64-byte rows: store j writes row j, 32 lanes x 2 consecutive bytes (conflict-free)
            __syncwarp();
#pragma unroll
            for (int j = 0; j < 32; j++) *reinterpret_cast<__nv_bfloat16*>(es.out + j * 64 + lane * 2) = __float2bfloat16_rn(v[j]);
        } else if (g.ct) {  // the block of C^T: this lane's row becomes column `lane`; store j writes row j of the block, 32 lanes x 4 bytes of
            __syncwarp();   // one 128-byte row (swizzled chunk (lane / 4) ^ (j % 8): conflict-free).  Every lane has read its row of the block.
#pragma unroll
            for (int j = 0; j < 32; j++)
                *reinterpret_cast<float*>(es.out + j * 128 + ((((lane >> 2) ^ (j & 7)) << 4) | ((lane & 3) << 2))) = v[j];
        } else {
            uint8_t* srow = es.out + lane * 128;
#pragma unroll
            for (int j = 0; j < 8; j++)
                *reinterpret_cast<float4*>(srow + ((j ^ (lane & 7)) << 4)) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy writes -> visible to the TMA (async proxy) read
        __syncwarp();
        if (lane == 0) {
            if (g.ct) tma_store_2d(es.mapC, es.out, row, col0);          // lane 0's row is the block's first row (the map is over C^T)
            else tma_store_2d(es.mapC, es.out, col0, row);
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
        return;
    }
    if (!row_ok) return;
    if (vec) {
#pragma unroll
        for (int j = 0; j < 8; j++) reinterpret_cast<float4*>(crow)[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
    } else {
#pragma unroll
        for (int j = 0; j < 32; j++) if (j < ncols) crow[j] = v[j];
    }
}

// derivative operand (the saved activation) of one 32-column chunk (act == 2), fetched into registers BEFORE the wait on the accumulator so that the HBM / L2
// latency of these row-per-lane loads overlaps the main loop of the tile.  Warp-uniform result; rows beyond M read row 0 (ignored).
__device__ __forceinline__ bool epilogue_prefetch(const GemmArgs& g, const int row, const int col0, const bool split, float4 (&ypre)[8]) {
    if (g.act != 2 || split || col0 + 32 > g.N || (g.ldaux & 3) != 0 || ((((uintptr_t)g.aux) & 15) != 0) || (col0 & 3) != 0) return false;
    const float4* arow = reinterpret_cast<const float4*>(g.aux + (size_t)(row < g.M ? row : 0) * g.ldaux + col0);
#pragma unroll
    for (int j = 0; j < 8; j++) ypre[j] = __ldg(arow + j);
    return true;
}

// ---------------------------------------------------------------------------------------------------------------
// Persistent kernel: grid = min(#tiles, #SMs); every CTA walks tiles t = blockIdx.x + i * gridDim.x (n fastest, so the CTAs of
// one wave share A tiles through L2).  Shared memory: [ring: stages x (A | B)][X: 64 KB][derivative operand staging 8 x 4 KB][barriers].
// X serves the main loop as the double-buffered transposed tiles of MN-major operands (A 2 x 16 KB, B 2 x 16 KB) and the epilogue
// as the accumulator / output staging (32 KB per warpgroup).
// CL = 2 (K-major operands, one problem, BN = 128): clusters of two CTAs walk pairs of adjacent tiles, paired along N when tiles_n is
// even (the pair shares its A box) and along M otherwise (tiles_m even: the pair shares its B box).  Per k-block each CTA loads its
// own box of the other operand and rank r's 64-row half of the shared box, multicast into both CTAs at byte offset r x 8 KB of the
// shared operand's slot (the 128B swizzle repeats every 1 KB, so the two halves form the same tile one 128-row box forms).  Both
// producers write every stage of both rings: empty[s] counts the consumer warps of both CTAs, and each consumer warp releases a
// stage in its own CTA and in its peer.  Cluster barriers after the mbarrier initialisation and before any thread exits keep a CTA
// alive while its peer may still multicast into it or arrive on its barriers.
// ---------------------------------------------------------------------------------------------------------------
// BF16 = true: the operands are BF16 (K-major only), a k-block is 64 of them (the same 128-byte rows, boxes, ring and multicast as 32
// floats) and the tensor core runs m64nBNk16 BF16 instructions; the epilogue is the same fp32 code.
// BF16 with AMN / BMN (gemm_bf16_mn_wgmma, go1_gemm_bf16_mn): an MN-major operand arrives as [64 k][64 mn] boxes, 128B-swizzled (BN = 32:
// one [64 k][32 n] box, 64B-swizzled), two boxes per 128-wide tile 8 KB apart, and the tensor core reads them in place through its
// transpose immediates: no shared-to-shared transposition.  ROW16: the epilogue can also store C row-major in BF16 (c16 without ct).
constexpr int X_BYTES = 65536;
template <int BN, bool ANYKIND, int CL, bool BF16, int AMN, int BMN, bool ROW16, bool DET>
__device__ __forceinline__ void gemm_wgmma_body(const GemmMaps& gm, const CUtensorMap& mapC, const CUtensorMap& mapY, const GemmArgs& g,
                                                const int tiles_m, const int tiles_n, const int total_tiles, const int stages, const DetArgs* det) {
    static_assert(CL == 1 || (CL == 2 && BN == BM), "CTA pairs share 128-row operand boxes");
    static_assert((AMN == 0 && BMN == 0 && !ROW16) || (BF16 && CL == 1), "MN-major BF16 operands and the row-major BF16 store: one CTA per tile");
    constexpr int G = EPI_G;
    constexpr int A_BYTES = BM * BK * 4, STAGE_BYTES = (BM + BN) * BK * 4;
    constexpr int MAX_STAGES = 8;
    constexpr int KE = BF16 ? 2 * BK : BK;       // operand elements per k-block
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* base = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* ring = base;
    uint8_t* xreg = base + (size_t)stages * STAGE_BYTES;
    uint8_t* stage_aux = xreg + X_BYTES;
    uint64_t* full = (uint64_t*)(stage_aux + (g.tma_aux ? NCONS * 4096 : 0));
    uint64_t* empty = full + MAX_STAGES;
    uint64_t* aux_bar = empty + MAX_STAGES;      // [NCONS]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_kb_total = (g.K + KE - 1) / KE;

    if (threadIdx.x == 0) {
        for (int p = 0; p < g.nprob; p++) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&gm.a[p]) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&gm.b[p]) : "memory");
        }
        if (g.tma_store) asm volatile("prefetch.tensormap [%0];" ::"l"(&mapC) : "memory");
        if (g.tma_aux) asm volatile("prefetch.tensormap [%0];" ::"l"(&mapY) : "memory");
        if (CL > 1) asm volatile("prefetch.tensormap [%0];" ::"l"(&gm.half) : "memory");
        for (int s = 0; s < stages; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], CL * NCONS); }
        for (int w = 0; w < NCONS; w++) mbar_init(&aux_bar[w], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (CL > 1) cluster_sync();      // the peer's barriers are initialised before any multicast or remote arrive reaches them
    else __syncthreads();

    // the work of this CTA: (pair-)tiles pt = first(), first() + step(), ... < npt; tile t = cta_tile(pt).  The block / cluster indices
    // are read where they are used: held in registers across the whole kernel they cost the consumers spill slots.
    const int npt = total_tiles / CL;
    auto first = [] { return (int)blockIdx.x / CL; };
    auto step = [] { return (int)gridDim.x / CL; };
    auto rank = [] { return CL > 1 ? cluster_ctarank() : 0u; };
    auto pair_n = [&] { return (tiles_n & 1) == 0; };
    auto cta_tile = [&](int pt) -> int {
        if (CL == 1) return pt;
        if (pair_n()) return 2 * pt + (int)rank();                    // tiles (2 j, 2 j + 1) along N of one row of tiles
        const int tn = pt % tiles_n, r = pt / tiles_n, hm = tiles_m / 2;
        return ((r / hm) * tiles_m + 2 * (r % hm) + (int)rank()) * tiles_n + tn;     // tiles (2 j, 2 j + 1) along M of one split
    };
    // tile -> (m0, n0, k-block range); grouped launches: tile t of problem t / tiles_per_prob
    auto tile_coords = [&](int t, int& m0, int& n0, int& kb0, int& nkb) {
        if (CL == 1 && g.nprob > 1) t %= g.tiles_per_prob;
        const int tn = t % tiles_n; t /= tiles_n;
        const int tm = t % tiles_m; const int z = t / tiles_m;
        m0 = tm * BM; n0 = tn * BN; kb0 = z * g.kb_per_split; nkb = min(g.kb_per_split, num_kb_total - kb0);
    };

    if (warp == NCONS) {
        // ===== TMA producer =====
        if (elect_one()) {
            int s = 0, ph = 0;      // ring position of this CTA's k-block stream
            for (int pt = first(); pt < npt; pt += step()) {
                const int t = cta_tile(pt);
                int m0, n0, kb0, nkb; tile_coords(t, m0, n0, kb0, nkb);
                const int p = CL == 1 && g.nprob > 1 ? t / g.tiles_per_prob : 0;
                const CUtensorMap* mapA = &gm.a[p];
                const CUtensorMap* mapB = &gm.b[p];
                for (int i = 0; i < nkb; i++) {
                    mbar_wait(&empty[s], ph ^ 1);
                    mbar_expect_tx(&full[s], STAGE_BYTES);
                    uint8_t* a = ring + (size_t)s * STAGE_BYTES;
                    uint8_t* b = a + A_BYTES;
                    if (CL > 1) {           // K-major: this CTA's half of the shared box to both CTAs, its own box of the other operand
                        const int kc = (kb0 + i) * KE;
                        if (pair_n()) {
                            tma_load_2d_multicast(&gm.half, &full[s], a + rank() * (A_BYTES / 2), kc, m0 + (int)rank() * (BM / 2), 0x3);
                            tma_load_2d(mapB, &full[s], b, kc, n0);
                        } else {
                            tma_load_2d(mapA, &full[s], a, kc, m0);
                            tma_load_2d_multicast(&gm.half, &full[s], b + rank() * (A_BYTES / 2), kc, n0 + (int)rank() * (BN / 2), 0x3);
                        }
                    } else if (AMN || BMN) {        // BF16: MN-major operands as 64-wide boxes (see above)
                        const int kc = (kb0 + i) * KE;
                        if (AMN) { tma_load_2d(mapA, &full[s], a, m0, kc); tma_load_2d(mapA, &full[s], a + A_BYTES / 2, m0 + BM / 2, kc); }
                        else tma_load_2d(mapA, &full[s], a, kc, m0);
                        if (BMN) {
                            tma_load_2d(mapB, &full[s], b, n0, kc);
                            if (BN == 128) tma_load_2d(mapB, &full[s], b + A_BYTES / 2, n0 + 64, kc);
                        } else tma_load_2d(mapB, &full[s], b, kc, n0);
                    } else {
                        if (g.amn) tma_load_2d(mapA, &full[s], a, m0, (kb0 + i) * KE);        // box [32 k-rows][128 m]
                        else tma_load_2d(mapA, &full[s], a, (kb0 + i) * KE, m0);              // box [128 m-rows][32 k]
                        if (g.bmn) tma_load_2d(mapB, &full[s], b, n0, (kb0 + i) * KE);
                        else tma_load_2d(mapB, &full[s], b, (kb0 + i) * KE, n0);
                    }
                    if (++s == stages) { s = 0; ph ^= 1; }
                }
            }
        }
        if (CL > 1) cluster_sync();
        return;
    }
    if (warp > NCONS) {
        if (CL > 1) cluster_sync();
        return;
    }

    // ===== consumers: warpgroup wgi owns rows [64 wgi, 64 wgi + 64) of the tile =====
    const int wgi = warp >> 2, w = warp & 3, ctid = threadIdx.x;
    const int q = 2 * wgi + (w & 1), grp = w >> 1;      // epilogue: 32-row block q of the tile, column group grp
    const bool tr = !BF16 && CL == 1 && (g.amn || g.bmn);        // pairs read K-major operands only, one problem; BF16: K-major only
    const bool split = g.kb_per_split < num_kb_total;
    const bool st_out = g.tma_store, st_aux = CL == 1 && g.tma_aux;      // pairs: no derivative operand (act 2)
    uint8_t* xwg = xreg + wgi * (X_BYTES / 2);          // this warpgroup's accumulator staging: [chunk][64 rows][128 B]
    uint8_t* my_aux = stage_aux + warp * 4096;
    uint64_t* my_bar = &aux_bar[warp];
    // derivative operand blocks run one chunk ahead of the epilogue: cursor (pt, pc) = the next chunk of this warp whose block has not been requested yet
    int pt = first(), pc = grp - G;
    auto next_chunk = [&]() -> bool {
        for (;;) {
            pc += G;
            if (pc >= BN / 32) { pt += step(); pc = grp; }
            if (pt >= npt) return false;
            if (pc < BN / 32 && (cta_tile(pt) % tiles_n) * BN + 32 * pc < g.N) return true;
        }
    };
    // stage s has been read: it returns to the producer of this CTA and, in a pair, to the peer's (whose half of it this CTA received)
    auto release = [&](int s) {
        if (lane == 0) {
            mbar_arrive(&empty[s]);
            if (CL > 1) mbar_arrive_cluster(&empty[s], rank() ^ 1);
        }
    };
    auto request_aux = [&]() {
        if (next_chunk() && lane == 0) {
            int m0, n0, kb0, nkb; tile_coords(cta_tile(pt), m0, n0, kb0, nkb);
            mbar_expect_tx(my_bar, 4096);
            tma_load_2d(&mapY, my_bar, my_aux, n0 + 32 * pc, m0 + 32 * q);
        }
    };
    if (st_aux) request_aux();
    uint32_t aux_phase = 0;
    int s = 0, ph = 0;
    float acc[BN / 2];
    for (int tp = first(); tp < npt; tp += step()) {
        const int t = cta_tile(tp);
        int m0, n0, kb0, nkb; tile_coords(t, m0, n0, kb0, nkb);
        // X is about to be rewritten: the TMA stores of the previous tile have read it
        if (st_out && lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        cons_sync();
        int prev = -1;
        for (int i = 0; i < nkb; i++) {
            mbar_wait(&full[s], ph);
            const uint8_t* a = ring + (size_t)s * STAGE_BYTES;
            const uint8_t* b = a + A_BYTES;
            if (tr) {
                if (g.amn) { uint8_t* ta = xreg + (i & 1) * A_BYTES; transpose_tile<BM>((const float*)a, ta, ctid); a = ta; }
                if (g.bmn) { uint8_t* tb = xreg + 2 * A_BYTES + (i & 1) * A_BYTES; transpose_tile<BN>((const float*)b, tb, ctid); b = tb; }
                if (prev >= 0) {        // k-block i - 1 is done: its stage returns to the producer, and its transposed tiles may be rewritten next round
                    wg::wait<0>();
                    release(prev);
                }
                fence_async_smem();     // generic-proxy writes -> visible to the tensor core (async proxy)
                cons_sync();
            }
            wg::fence();
            if constexpr (AMN || BMN) {
                const uint64_t da = AMN ? wg::desc_mn128(a + (size_t)wgi * 64 * 128, 8192) : wg::desc(a + (size_t)wgi * 64 * 128);
                const uint64_t db = BMN ? (BN == 32 ? wg::desc_mn64(b) : wg::desc_mn128(b, 8192)) : wg::desc(b);
                wg::mma_kblock_bf16<BN, AMN, BMN>(acc, da, db, i > 0);
            } else {
                wg::mma_kblock<BN, BF16>(acc, a + (size_t)wgi * 64 * 128, b, i > 0);
            }
            wg::commit();
            if (!tr && prev >= 0) {
                wg::wait<1>();
                release(prev);
            }
            prev = s;
            if (++s == stages) { s = 0; ph ^= 1; }
        }
        wg::wait<0>();
        release(prev);
        if (tr) cons_sync();            // both warpgroups are done with the transposed tiles that the staging overlays

        const int row = m0 + 32 * q + lane;
        float* Cbase = CL == 1 && g.nprob > 1 ? g.Cg[t / g.tiles_per_prob] : g.C;
        if constexpr (DET) {    // split-K: the slab of (problem, split) in the workspace
            if (split) Cbase = det->split + (size_t)((CL == 1 && g.nprob > 1 ? t / g.tiles_per_prob : 0) * det->nsplit + kb0 / g.kb_per_split) * det->slab;
        }
        float4 ypre[8];
        const bool have_pre = CL == 1 && !st_aux && (grp < BN / 32) && epilogue_prefetch(g, row, n0 + 32 * grp, split, ypre);
        store_fragment<BN / 8>(acc, xwg, 0, w, lane, [](float2 v, int, int) { return v; });
        wg_sync(wgi);
#pragma unroll 1
        for (int c = grp; c < BN / 32; c += G) {
            if (n0 + 32 * c >= g.N) break;                           // warp-uniform
            uint8_t* blk = xwg + (size_t)c * (64 * 128) + (w & 1) * 4096;
            uint32_t r[32];
            const uint8_t* srow = blk + lane * 128;
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const uint4 x = *reinterpret_cast<const uint4*>(srow + ((j ^ (lane & 7)) << 4));
                r[4 * j] = x.x; r[4 * j + 1] = x.y; r[4 * j + 2] = x.z; r[4 * j + 3] = x.w;
            }
            EpiStage es;
            es.out = st_out ? blk : nullptr; es.mapC = &mapC; es.aux = st_aux ? my_aux : nullptr;
            if (st_aux) { mbar_wait(my_bar, aux_phase); aux_phase ^= 1; }
            epilogue_chunk<ANYKIND, ROW16, DET>(g, Cbase, r, row, n0 + 32 * c, split, lane, ypre, have_pre && c == grp, es, det);
            if (st_aux) { __syncwarp(); request_aux(); }             // every lane has read the operand block: fetch the next one into it
        }
    }
    if (st_out && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");      // all stores of this warp have completed
    if (CL > 1) cluster_sync();
}

// DET (deterministic mode): the cross-CTA sums go to the workspace regions of det (DetArgs), left to go1_det_sum; the default instantiation
// receives an empty det and adds into its targets
template <int BN, bool ANYKIND, int CL, bool BF16, bool DET>
__global__ void __launch_bounds__(32 * NCONS + 128, 1) gemm_tf32_wgmma(const __grid_constant__ GemmMaps gm,
                                                                      const __grid_constant__ CUtensorMap mapC, const __grid_constant__ CUtensorMap mapY, const GemmArgs g,
                                                                      const int tiles_m, const int tiles_n, const int total_tiles, const int stages, const DetArgs det) {
    gemm_wgmma_body<BN, ANYKIND, CL, BF16, 0, 0, false, DET>(gm, mapC, mapY, g, tiles_m, tiles_n, total_tiles, stages, &det);
}
// BF16 operands in the majors AMN / BMN (1: MN-major), fp32 or row-major BF16 output (go1_gemm_bf16_mn / go1_gemm_bf16_grouped)
template <int BN, bool ANYKIND, int AMN, int BMN, bool DET>
__global__ void __launch_bounds__(32 * NCONS + 128, 1) gemm_bf16_mn_wgmma(const __grid_constant__ GemmMaps gm,
                                                                         const __grid_constant__ CUtensorMap mapC, const __grid_constant__ CUtensorMap mapY, const GemmArgs g,
                                                                         const int tiles_m, const int tiles_n, const int total_tiles, const int stages, const DetArgs det) {
    gemm_wgmma_body<BN, ANYKIND, 1, true, AMN, BMN, true, DET>(gm, mapC, mapY, g, tiles_m, tiles_n, total_tiles, stages, &det);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;
std::once_flag g_once;

int sm_count() {
    static int sms = 0;
    if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); if (sms <= 0) sms = 132; }
    return sms;
}

int make_map_uncached(CUtensorMap* map, const void* ptr, int rows, int cols, int ld, int box_rows, int box_cols, CUtensorMapSwizzle swz, int esize);
// Encoding a tensor map costs about a microsecond of host time and the learner issues the same few hundred (pointer, shape) combinations
// every update: keep them.
struct MapKey { const void* ptr; int rows, cols, ld, box_rows, box_cols, swz, esize; bool operator==(const MapKey& o) const { return ptr == o.ptr && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows && box_cols == o.box_cols && swz == o.swz && esize == o.esize; } };
struct MapKeyHash { size_t operator()(const MapKey& k) const { size_t h = (size_t)k.ptr; h = h * 1000003u ^ (size_t)k.rows; h = h * 1000003u ^ (size_t)k.cols; h = h * 1000003u ^ (size_t)k.ld; h = h * 1000003u ^ (size_t)((k.box_rows * 8 + k.swz) * 8 + k.esize); h = h * 1000003u ^ (size_t)k.box_cols; return h; } };
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_map_cache;
std::mutex g_map_mutex;
// rows x cols fp32 matrix with row stride ld; box = box_rows x box_cols.  K-major operand tiles and 32 x 32 output blocks: 32-float (128-byte)
// box rows, 128B-swizzled.  MN-major operand boxes ([32 k-rows][tile width]): unswizzled, transposed on the SM.  esize 2: a BF16 matrix
// (ld and box_cols in elements; K-major operand boxes are 64 wide, the same 128-byte rows).
int make_map(CUtensorMap* map, const void* ptr, int rows, int cols, int ld, int box_rows, int box_cols = BK, CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B,
             int esize = 4) {
    const MapKey key{ptr, rows, cols, ld, box_rows, box_cols, (int)swz, esize};
    {
        std::lock_guard<std::mutex> lk(g_map_mutex);
        auto it = g_map_cache.find(key);
        if (it != g_map_cache.end()) { *map = it->second; return 0; }
    }
    if (int e = make_map_uncached(map, ptr, rows, cols, ld, box_rows, box_cols, swz, esize)) return e;
    std::lock_guard<std::mutex> lk(g_map_mutex);
    if (g_map_cache.size() > 8192) g_map_cache.clear();
    g_map_cache.emplace(key, *map);
    return 0;
}
int make_map_mn(CUtensorMap* map, const float* ptr, int k_rows, int mn_cols, int ld, int width) {
    return make_map(map, ptr, k_rows, mn_cols, ld, BK, width, CU_TENSOR_MAP_SWIZZLE_NONE);
}
int make_map_uncached(CUtensorMap* map, const void* ptr, int rows, int cols, int ld, int box_rows, int box_cols, CUtensorMapSwizzle swz, int esize) {
    std::call_once(g_once, [] {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) g_encode = (EncodeTiledFn)fn;
    });
    if (!g_encode) return go1_set_error("cuTensorMapEncodeTiled unavailable");
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * esize};
    cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = g_encode(map, esize == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { char b[96]; snprintf(b, sizeof b, "cuTensorMapEncodeTiled failed (%d)", (int)r); return go1_set_error(b); }
    return 0;
}

// Split count of a plain product: the s (with at least min_kb k-blocks per split) that minimises the wave-quantised makespan
// ceil(tiles s / SMs) x (ceil(num_kb / s) + SPLIT_TILE_KB) in k-block times, where a tile costs about SPLIT_TILE_KB k-blocks besides its
// main loop (pipeline fill, accumulator staging, the reduction into C).  Ties go to the smaller s (less reduction traffic).  The fused
// first-layer weight gradient (170 tiles x 768 k-blocks) gets s = 3: 510 tiles, 3.86 of 4 waves, where s = 1 ran 1.29 waves as 2.
int split_count(int tiles, int num_kb, int min_kb, int sms) {
    constexpr int SPLIT_TILE_KB = 4;
    int best = 1;
    long long best_cost = -1;
    for (int s = 1; s <= num_kb / (min_kb > 0 ? min_kb : 1); s++) {
        const int kb = (num_kb + s - 1) / s;
        if ((num_kb + kb - 1) / kb != s) continue;                  // some split would be empty
        const long long cost = (long long)(((long long)tiles * s + sms - 1) / sms) * (kb + SPLIT_TILE_KB);
        if (best_cost < 0 || cost < best_cost) { best = s; best_cost = cost; }
    }
    return best;
}

__global__ void zero_strided(float* C, int ldc, int M, int N) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)M * N) return;
    C[(i / N) * ldc + (i % N)] = 0.f;
}
__global__ void bias_act_strided(float* C, int ldc, const float* bias, int M, int N, int act, int kind) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)M * N) return;
    float* c = C + (i / N) * ldc + (i % N);
    float v = *c;
    if (bias) v += bias[i % N];
    if (act == 1) { GO1_ACT_SWITCH(kind, KD, v = act_exact<KD>(v);) }
    *c = v;
}

// MN < 0: gemm_tf32_wgmma<BN, ANYKIND, CL, BF16, DET>; MN = 0..3: gemm_bf16_mn_wgmma<BN, ANYKIND, MN & 1, MN >> 1, DET> (CL 1, BF16)
template <int BN, bool ANYKIND, int CL, bool BF16, int MN, bool DET>
int launch_gemm(const GemmMaps& gm, const CUtensorMap& mc, const CUtensorMap& my, GemmArgs& g, int splits, cudaStream_t st, const DetArgs& det) {
    constexpr int STAGE_BYTES = (BM + BN) * BK * 4;
    const size_t staging = X_BYTES + (g.tma_aux ? (size_t)NCONS * 4096 : 0);
    const size_t fixed = staging + (2 * 8 + NCONS) * 8 + 16 + 1024;
    const size_t budget = 227 * 1024;
    int stages = (int)((budget - fixed) / STAGE_BYTES);
    if (stages > 8) stages = 8;
    if (stages < 2) return go1_set_error("go1_gemm impl=1: no room for the operand ring");
    const size_t smem = (size_t)stages * STAGE_BYTES + fixed;
    static_assert(MN < 0 || (CL == 1 && BF16), "the MN-major BF16 kernel runs one CTA per tile");
    auto kernel = [] {
        if constexpr (MN < 0) return gemm_tf32_wgmma<BN, ANYKIND, CL, BF16, DET>;
        else return gemm_bf16_mn_wgmma<BN, ANYKIND, (MN & 1), (MN >> 1), DET>;
    }();
    const int tiles_m = (g.M + BM - 1) / BM, tiles_n = (g.N + BN - 1) / BN;
    g.tiles_per_prob = tiles_m * tiles_n * splits;
    const int total = g.tiles_per_prob * (g.nprob > 1 ? g.nprob : 1);
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CL; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.blockDim = dim3(32 * NCONS + 128); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cfg.attrs = attr; cfg.numAttrs = 1;
    static bool configured = false;
    static int slots = 0;        // CTAs (clusters of CL) resident at once: one per SM, as far as the GPCs can place the clusters
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)budget);
        if (e != cudaSuccess) return go1_set_error(cudaGetErrorString(e));
        slots = sm_count();
        if (CL > 1) {
            cfg.gridDim = dim3(CL * sm_count());
            int clusters = 0;
            e = cudaOccupancyMaxActiveClusters(&clusters, kernel, &cfg);
            if (e != cudaSuccess) return go1_set_error(cudaGetErrorString(e));
            if (clusters < 1) return go1_set_error("go1_gemm impl=1: no CTA pair of the persistent GEMM fits a GPC");
            slots = clusters;
        }
        configured = true;
    }
    // persistent grid: one CTA per SM (the ring and the staging fill its shared memory), CL x (pair-)tile slots for clusters
    const int units = total / CL;
    cfg.gridDim = dim3(CL * (units < slots ? units : slots));
    if (CL == 1) kernel<<<cfg.gridDim, cfg.blockDim, smem, st>>>(gm, mc, my, g, tiles_m, tiles_n, total, stages, det);
    else {
        cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, gm, mc, my, g, tiles_m, tiles_n, total, stages, det);
        if (e != cudaSuccess) return go1_set_error(cudaGetErrorString(e));
    }
    go1_count_launch(1);
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Fused MLP tail, forward: the layers behind a first layer of ActorCritic's MLPs (actor_critic.py:38-77) in ONE launch,
//     y2 = f(x W2^T + b2)     [M][N2]        x = the first layer's activated output, K1 wide (a column slice of the fused first-layer product)
//     y3 = f(y2 W3^T + b3)    [M][N3]        (N3 = 0: two-layer tail, the head reads y2)
//     out = y_last Wh^T + bh  [M][nh]        nh <= 12 (12 action means / 1 value / 2 latents): CUDA cores, from registers
// (f = the launch's Go1Activation, ELU by default)
// for up to two problems of the same shape (actor and critic bodies) in one grid.  One CTA (384 threads) owns a 64-row block:
//   warps 0-7   two consumer warpgroups; warpgroup g computes columns [g N2 / 2, (g + 1) N2 / 2) of y2 and [g N3 / 2, (g + 1) N3 / 2) of y3
//               for all 64 rows (wgmma, accumulators in registers).  y2 = f(acc + b2) goes from the registers to shared memory once,
//               K-major and 128B-swizzled, and from there BOTH to the tensor core (A operand of product 2) and to global memory (one TMA
//               store per 32 x 32 block: the backward pass needs y2); y3 is stored from registers; the head's partial dot products
//               are taken on the accumulator fragments, reduced over the four lanes that share a row, and the two warpgroups' halves
//               meet in shared memory.
//   warp 8      TMA producer: ring 1 streams x and W2 k-blocks, ring 2 the W3 k-blocks; it runs ahead into the next block's product 1
//               while the consumers are in product 2 and the head.
// ---------------------------------------------------------------------------------------------------------------
constexpr int TAIL_MAXP = 2, TAIL_HPW = 12, TAIL_BM = 64;
struct TailProb { const float* b2; const float* b3; const float* Wh; const float* bh; float* y3; float* out; int ldy3, ldout, nh, wh_row0; };
struct TailArgs { TailProb p[TAIL_MAXP]; int nprob, M, tiles_per_prob, tiles, kind; };
struct TailMaps { CUtensorMap x[TAIL_MAXP], w2[TAIL_MAXP], w3[TAIL_MAXP], y2[TAIL_MAXP]; };

template <int K1, int N2, int N3>
struct TailSmem {
    static constexpr int S1 = (N3 > 0) ? 2 : 3, S2 = (N3 > 0) ? 2 : 0;
    static constexpr int KB1 = K1 / BK, KB2 = N2 / BK;
    static constexpr int STAGE1 = (TAIL_BM + N2) * BK * 4;
    static constexpr int Y2TILE = KB2 * TAIL_BM * BK * 4;
    static constexpr int STAGE2 = (N3 > 0 ? N3 : 8) * BK * 4;
    static constexpr int NL = (N3 > 0) ? N3 : N2;
    static constexpr int PARAMS = (TAIL_MAXP * (N2 + N3) + 16 * NL + TAIL_MAXP * 16) * 4;
    static constexpr int HP = TAIL_HPW * TAIL_BM * 4;
    static constexpr int BARS = (2 * S1 + 2 * (S2 > 0 ? S2 : 1)) * 8 + 16;
    static constexpr int TOTAL = S1 * STAGE1 + Y2TILE + S2 * STAGE2 + PARAMS + HP + BARS + 1024;
};

// partial dot products of the head on an accumulator fragment: hp[r][n] += sum over this thread's columns of v[row r][col] * Wh[n][col]
template <int NJ>
__device__ __forceinline__ void head_partial(const float (&v)[4 * NJ], const float* wh, const int NL, const int nh, const int col_base, const int lane, float (&hp)[2][TAIL_HPW]) {
#pragma unroll
    for (int n = 0; n < TAIL_HPW; n++) {
        if (n < nh) {
            const float* wr = wh + n * NL + col_base + 2 * (lane & 3);
            float a0 = hp[0][n], a1 = hp[1][n];
#pragma unroll
            for (int j = 0; j < NJ; j++) {
                const float2 ww = *reinterpret_cast<const float2*>(wr + 8 * j);
                a0 = fmaf(v[4 * j], ww.x, a0); a0 = fmaf(v[4 * j + 1], ww.y, a0);
                a1 = fmaf(v[4 * j + 2], ww.x, a1); a1 = fmaf(v[4 * j + 3], ww.y, a1);
            }
            hp[0][n] = a0; hp[1][n] = a1;
        }
    }
}

// The true widths of a ragged tail (mlp_tail_fwd_ragged_kernel): k1 any, n2 <= N2, n3 <= N3 (0 with N3), where N2 / N3 are the
// instantiated tile widths.  TMA reads the W rows and columns beyond them as zeros and clips the y2 stores; the biases and head weights of
// the padded columns are zero in shared memory, so those columns add nothing whatever f(0) is.
struct TailDims { int k1, n2, n3; };

template <int K1, int N2, int N3, bool ANYKIND, bool RAGGED>
__device__ __forceinline__ void mlp_tail_fwd_body(const TailMaps& maps, const TailArgs& g, const TailDims d) {
    const int kind = ANYKIND ? g.kind : (int)GO1_ACT_ELU;
    using L = TailSmem<K1, N2, N3>;
    constexpr int S1 = L::S1, S2 = (L::S2 > 0 ? L::S2 : 1), KB2 = L::KB2, STAGE1 = L::STAGE1, STAGE2 = L::STAGE2, NL = L::NL;
    const int KB1 = RAGGED ? (d.k1 + BK - 1) / BK : L::KB1;
    const int n2 = RAGGED ? d.n2 : N2, n3 = RAGGED ? d.n3 : N3, nl = RAGGED ? (N3 > 0 ? d.n3 : d.n2) : NL;
    constexpr int NH2 = N2 / 2, NH3 = (N3 > 0 ? N3 : 64) / 2;      // columns per warpgroup
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* base = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* r1 = base;
    uint8_t* y2t = r1 + S1 * STAGE1;                         // [KB2][64 rows][128 B]
    uint8_t* r2 = y2t + L::Y2TILE;
    float* s_b2 = (float*)(r2 + L::S2 * STAGE2);             // [MAXP][N2]
    float* s_b3 = s_b2 + TAIL_MAXP * N2;                     // [MAXP][N3]
    float* s_wh = s_b3 + TAIL_MAXP * N3;                     // [16][NL]: the head rows of all problems (problem p starts at row wh_row0)
    float* s_bh = s_wh + 16 * NL;                            // [MAXP][16]
    float* s_hp = s_bh + TAIL_MAXP * 16;                     // [HPW][64]: head partial sums of warpgroup 1
    uint64_t* full1 = (uint64_t*)(s_hp + TAIL_HPW * TAIL_BM);
    uint64_t* empty1 = full1 + S1;
    uint64_t* full2 = empty1 + S1;
    uint64_t* empty2 = full2 + S2;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int p = 0; p < g.nprob; p++) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.x[p]) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.w2[p]) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.y2[p]) : "memory");
            if (N3 > 0) asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.w3[p]) : "memory");
        }
        for (int s = 0; s < S1; s++) { mbar_init(&full1[s], 1); mbar_init(&empty1[s], NCONS); }
        for (int s = 0; s < S2; s++) { mbar_init(&full2[s], 1); mbar_init(&empty2[s], NCONS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // biases and head weights: read by every consumer thread for every row -> shared memory
    for (int i = threadIdx.x; i < TAIL_MAXP * N2; i += blockDim.x) { const int p = i / N2; s_b2[i] = (p < g.nprob && g.p[p].b2 && i - p * N2 < n2) ? __ldg(g.p[p].b2 + (i - p * N2)) : 0.f; }
    if (N3 > 0) for (int i = threadIdx.x; i < TAIL_MAXP * N3; i += blockDim.x) { const int p = i / (N3 > 0 ? N3 : 1); s_b3[i] = (p < g.nprob && g.p[p].b3 && i - p * N3 < n3) ? __ldg(g.p[p].b3 + (i - p * N3)) : 0.f; }
    for (int i = threadIdx.x; i < 16 * NL; i += blockDim.x) {
        const int n = i / NL, k = i - n * NL;
        float v = 0.f;
        if (k < nl)
            for (int p = 0; p < g.nprob; p++) { const int r = n - g.p[p].wh_row0; if (r >= 0 && r < g.p[p].nh) v = __ldg(g.p[p].Wh + (size_t)r * nl + k); }
        s_wh[i] = v;
    }
    if (threadIdx.x < TAIL_MAXP * 16) { const int p = threadIdx.x >> 4, n = threadIdx.x & 15; s_bh[threadIdx.x] = (p < g.nprob && n < g.p[p].nh && g.p[p].bh) ? __ldg(g.p[p].bh + n) : 0.f; }
    __syncthreads();

    if (warp == NCONS) {
        // ===== TMA producer =====
        if (elect_one()) {
            int it1 = 0, it2 = 0;
            for (int t = blockIdx.x; t < g.tiles; t += gridDim.x) {
                const int p = t / g.tiles_per_prob, m0 = (t - p * g.tiles_per_prob) * TAIL_BM;
                for (int i = 0; i < KB1; i++, it1++) {
                    const int s = it1 % S1, ph = (it1 / S1) & 1;
                    mbar_wait(&empty1[s], ph ^ 1);
                    mbar_expect_tx(&full1[s], STAGE1);
                    tma_load_2d(&maps.x[p], &full1[s], r1 + (size_t)s * STAGE1, i * BK, m0);
                    tma_load_2d(&maps.w2[p], &full1[s], r1 + (size_t)s * STAGE1 + TAIL_BM * BK * 4, i * BK, 0);
                }
                if (N3 > 0) {
                    for (int i = 0; i < KB2; i++, it2++) {
                        const int s = it2 % S2, ph = (it2 / S2) & 1;
                        mbar_wait(&empty2[s], ph ^ 1);
                        mbar_expect_tx(&full2[s], STAGE2);
                        tma_load_2d(&maps.w3[p], &full2[s], r2 + (size_t)s * STAGE2, i * BK, 0);
                    }
                }
            }
        }
        return;
    }
    if (warp > NCONS) return;

    // ===== consumers =====
    const int wgi = warp >> 2, w = warp & 3;
    const int rA = 16 * w + (lane >> 2);                     // this thread's fragment rows: rA and rA + 8
    int it1 = 0, it2 = 0;
    for (int t = blockIdx.x; t < g.tiles; t += gridDim.x) {
        const int p = t / g.tiles_per_prob, m0 = (t - p * g.tiles_per_prob) * TAIL_BM;
        const TailProb& pr = g.p[p];
        const bool ok0 = m0 + rA < g.M, ok1 = m0 + rA + 8 < g.M;
        float hp[2][TAIL_HPW];
#pragma unroll
        for (int n = 0; n < TAIL_HPW; n++) hp[0][n] = hp[1][n] = 0.f;
        const float* wh = s_wh + (size_t)pr.wh_row0 * NL;
        {
            // ---- product 1 and y2
            float acc[NH2 / 2];
            int prev = -1;
            for (int i = 0; i < KB1; i++, it1++) {
                const int s = it1 % S1, ph = (it1 / S1) & 1;
                mbar_wait(&full1[s], ph);
                const uint8_t* a = r1 + (size_t)s * STAGE1;
                wg::fence();
                wg::mma_kblock<NH2>(acc, a, a + TAIL_BM * BK * 4 + (size_t)wgi * NH2 * 128, i > 0);
                wg::commit();
                if (prev >= 0) { wg::wait<1>(); if (lane == 0) mbar_arrive(&empty1[prev]); }
                prev = s;
            }
            wg::wait<0>();
            if (lane == 0) mbar_arrive(&empty1[prev]);
            const float* b2 = s_b2 + p * N2;
            // rows beyond M stay 0 by the guard, not by f(0): they are operand rows of product 2 and sigmoid(0) = 0.5
            GO1_ACT_SWITCH(kind, KD,
                _Pragma("unroll")
                for (int j = 0; j < NH2 / 8; j++) {
                    const float2 bb = *reinterpret_cast<const float2*>(b2 + wgi * NH2 + 8 * j + 2 * (lane & 3));
                    acc[4 * j] = ok0 ? act_fast<KD>(acc[4 * j] + bb.x) : 0.f; acc[4 * j + 1] = ok0 ? act_fast<KD>(acc[4 * j + 1] + bb.y) : 0.f;
                    acc[4 * j + 2] = ok1 ? act_fast<KD>(acc[4 * j + 2] + bb.x) : 0.f; acc[4 * j + 3] = ok1 ? act_fast<KD>(acc[4 * j + 3] + bb.y) : 0.f;
                })
            // (the previous block's readers of the y2 tile -- product 2 and the TMA stores -- were waited for at the end of that block)
            store_fragment<NH2 / 8>(acc, y2t, wgi * NH2, w, lane, [](float2 v, int, int) { return v; });
            if (N3 == 0) head_partial<NH2 / 8>(acc, wh, NL, pr.nh, wgi * NH2, lane, hp);       // two-layer tail: the head reads y2
        }
        fence_async_smem();                                  // generic-proxy stores -> visible to the async proxy (tensor core, TMA store)
        cons_sync();
        if (lane == 0) {
            for (int b = warp; b < 2 * KB2; b += NCONS)      // rows beyond M (and columns beyond n2) are clipped
                if (!RAGGED || 32 * (b >> 1) < n2) tma_store_2d(&maps.y2[p], y2t + (size_t)b * 4096, 32 * (b >> 1), m0 + 32 * (b & 1));
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
        if (N3 > 0) {
            // ---- product 2 (A = the y2 tile), y3 and the head
            float acc[NH3 / 2];
            int prev = -1;
            for (int i = 0; i < KB2; i++, it2++) {
                const int s = it2 % S2, ph = (it2 / S2) & 1;
                mbar_wait(&full2[s], ph);
                wg::fence();
                wg::mma_kblock<NH3>(acc, y2t + (size_t)i * (TAIL_BM * 128), r2 + (size_t)s * STAGE2 + (size_t)wgi * NH3 * 128, i > 0);
                wg::commit();
                if (prev >= 0) { wg::wait<1>(); if (lane == 0) mbar_arrive(&empty2[prev]); }
                prev = s;
            }
            wg::wait<0>();
            if (lane == 0) mbar_arrive(&empty2[prev]);
            const float* b3 = s_b3 + p * N3;
            GO1_ACT_SWITCH(kind, KD,
                _Pragma("unroll")
                for (int j = 0; j < NH3 / 8; j++) {
                    const int col = wgi * NH3 + 8 * j + 2 * (lane & 3);
                    const float2 bb = *reinterpret_cast<const float2*>(b3 + col);
                    acc[4 * j] = act_fast<KD>(acc[4 * j] + bb.x); acc[4 * j + 1] = act_fast<KD>(acc[4 * j + 1] + bb.y);
                    acc[4 * j + 2] = act_fast<KD>(acc[4 * j + 2] + bb.x); acc[4 * j + 3] = act_fast<KD>(acc[4 * j + 3] + bb.y);
                    if (!RAGGED || col + 1 < n3) {
                        if (ok0) *reinterpret_cast<float2*>(pr.y3 + (size_t)(m0 + rA) * pr.ldy3 + col) = make_float2(acc[4 * j], acc[4 * j + 1]);
                        if (ok1) *reinterpret_cast<float2*>(pr.y3 + (size_t)(m0 + rA + 8) * pr.ldy3 + col) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
                    } else if (col < n3) {
                        if (ok0) pr.y3[(size_t)(m0 + rA) * pr.ldy3 + col] = acc[4 * j];
                        if (ok1) pr.y3[(size_t)(m0 + rA + 8) * pr.ldy3 + col] = acc[4 * j + 2];
                    }
                })
            head_partial<NH3 / 8>(acc, wh, NL, pr.nh, wgi * NH3, lane, hp);
        }
        // the head: sum over the four lanes that share a row, then warpgroup 1's half meets warpgroup 0's in shared memory
#pragma unroll
        for (int n = 0; n < TAIL_HPW; n++) {
            if (n < pr.nh) {
#pragma unroll
                for (int r = 0; r < 2; r++) {
                    float a = hp[r][n];
                    a += __shfl_xor_sync(0xffffffffu, a, 1);
                    a += __shfl_xor_sync(0xffffffffu, a, 2);
                    hp[r][n] = a;
                }
                if (wgi == 1 && (lane & 3) == 0) { s_hp[n * TAIL_BM + rA] = hp[0][n]; s_hp[n * TAIL_BM + rA + 8] = hp[1][n]; }
            }
        }
        cons_sync();
        if (wgi == 0 && (lane & 3) == 0) {
            const float* bh = s_bh + p * 16;
#pragma unroll
            for (int n = 0; n < TAIL_HPW; n++) {
                if (n < pr.nh) {
                    if (ok0) pr.out[(size_t)(m0 + rA) * pr.ldout + n] = hp[0][n] + s_hp[n * TAIL_BM + rA] + bh[n];
                    if (ok1) pr.out[(size_t)(m0 + rA + 8) * pr.ldout + n] = hp[1][n] + s_hp[n * TAIL_BM + rA + 8] + bh[n];
                }
            }
        }
        // the y2 tile and the head exchange are rewritten by the next block: the TMA stores have read the tile, every warp is past its reads
        if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        cons_sync();
    }
    if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// the tails of scripts/train.py's shapes (512-256-128 and 256-128), every width a compile-time constant
template <int K1, int N2, int N3, bool ANYKIND>
__global__ void __launch_bounds__(32 * NCONS + 128, 1) mlp_tail_fwd_kernel(const __grid_constant__ TailMaps maps, const TailArgs g) {
    mlp_tail_fwd_body<K1, N2, N3, ANYKIND, false>(maps, g, TailDims{K1, N2, N3});
}
// any other tail: K1 streamed at run time, N2 / N3 the tile widths that cover n2 / n3 (N2 64, 128 or 256; N3 0 (two-layer tail), 64 or
// 128: a 256-wide N3 would need 237 KB of shared memory with two W3 stages, and spills 1.2 KB with one)
template <int N2, int N3, bool ANYKIND>
__global__ void __launch_bounds__(32 * NCONS + 128, 1) mlp_tail_fwd_ragged_kernel(const __grid_constant__ TailMaps maps, const TailArgs g, const TailDims d) {
    mlp_tail_fwd_body<BK, N2, N3, ANYKIND, true>(maps, g, d);
}

template <int K1, int N2, int N3, bool ANYKIND>
int launch_tail(const TailMaps& maps, const TailArgs& g, cudaStream_t st) {
    using L = TailSmem<K1, N2, N3>;
    static_assert(L::TOTAL <= 227 * 1024, "fused tail: shared memory budget");
    const size_t smem = L::TOTAL;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(mlp_tail_fwd_kernel<K1, N2, N3, ANYKIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return go1_set_error(cudaGetErrorString(e));
        configured = true;
    }
    const int sms = sm_count();
    const int grid = g.tiles < sms ? g.tiles : sms;
    mlp_tail_fwd_kernel<K1, N2, N3, ANYKIND><<<grid, 32 * NCONS + 128, smem, st>>>(maps, g);
    go1_count_launch(1);
    return 0;
}

template <int N2, int N3, bool ANYKIND>
int launch_tail_ragged(const TailMaps& maps, const TailArgs& g, const TailDims d, cudaStream_t st) {
    using L = TailSmem<BK, N2, N3>;      // (K1 only sets the k-block count, which the ragged kernel takes at run time)
    static_assert(L::TOTAL <= 227 * 1024, "fused tail: shared memory budget");
    const size_t smem = L::TOTAL;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(mlp_tail_fwd_ragged_kernel<N2, N3, ANYKIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return go1_set_error(cudaGetErrorString(e));
        configured = true;
    }
    const int sms = sm_count();
    const int grid = g.tiles < sms ? g.tiles : sms;
    mlp_tail_fwd_ragged_kernel<N2, N3, ANYKIND><<<grid, 32 * NCONS + 128, smem, st>>>(maps, g, d);
    go1_count_launch(1);
    return 0;
}

// the ragged instantiation whose tiles cover (n2, n3)
template <bool ANYKIND>
int launch_tail_ragged_any(const TailMaps& maps, const TailArgs& g, const TailDims d, cudaStream_t st) {
    const int w2 = d.n2 <= 64 ? 64 : d.n2 <= 128 ? 128 : 256, w3 = d.n3 == 0 ? 0 : d.n3 <= 64 ? 64 : d.n3 <= 128 ? 128 : -1;
#define GO1_TAIL_CASE(A, B) if (w2 == A && w3 == B) return launch_tail_ragged<A, B, ANYKIND>(maps, g, d, st);
    GO1_TAIL_CASE(64, 0) GO1_TAIL_CASE(64, 64) GO1_TAIL_CASE(64, 128)
    GO1_TAIL_CASE(128, 0) GO1_TAIL_CASE(128, 64) GO1_TAIL_CASE(128, 128)
    GO1_TAIL_CASE(256, 0) GO1_TAIL_CASE(256, 64) GO1_TAIL_CASE(256, 128)
#undef GO1_TAIL_CASE
    return go1_set_error("go1_mlp_tail_forward: tail widths N2 1..256, N3 0..128");
}

}  // namespace

// ---- optional per-launch timing of the tensor-core GEMM (bench.py's roofline): CUDA events on the launch stream around every
// go1_gemm impl=1 call between go1_gemm_timing(1, ..) and go1_gemm_timing(0, ..)
#include <vector>
static bool g_time_on = false;
static std::vector<cudaEvent_t> g_time_events;
static size_t g_time_used = 0;
static double g_time_flop = 0.0;
// what each timed launch was (GO1_GEMM_TIMING_CSV dump).  Fused tails: N = N2, K = K1, n3 = N3 (0: two-layer tail), heads = the head
// columns of all problems, problems = the problems in the grid (M counts the rows of all of them)
struct TimeRec { int M, N, K, amn, bmn, act, nex, splits, kern, colsum, cluster, n3, heads, problems, bf16; };
static std::vector<TimeRec> g_time_recs;
static cudaEvent_t timing_event() {
    if (g_time_used == g_time_events.size()) { cudaEvent_t e; cudaEventCreate(&e); g_time_events.push_back(e); }
    return g_time_events[g_time_used++];
}
extern "C" int go1_gemm_timing(int on, double* total_ms, double* total_flop, long long* launches) {
    if (on) { g_time_on = true; g_time_used = 0; g_time_flop = 0.0; g_time_recs.clear(); return 0; }
    g_time_on = false;
    double ms = 0.0;
    FILE* csv = getenv("GO1_GEMM_TIMING_CSV") ? fopen(getenv("GO1_GEMM_TIMING_CSV"), "w") : nullptr;
    if (csv) fprintf(csv, "M,N,K,a_mn_major,b_mn_major,act,num_extra,splits,kernel,colsum,us,n3,heads,problems,bf16\n");
    for (size_t i = 0; i + 1 < g_time_used; i += 2) {
        if (cudaEventSynchronize(g_time_events[i + 1]) != cudaSuccess) return go1_set_error("go1_gemm_timing: event sync failed");
        float t = 0.f;
        if (cudaEventElapsedTime(&t, g_time_events[i], g_time_events[i + 1]) != cudaSuccess) return go1_set_error("go1_gemm_timing: elapsed time failed");
        ms += t;
        if (csv && i / 2 < g_time_recs.size()) {
            const TimeRec& r = g_time_recs[i / 2];
            fprintf(csv, "%d,%d,%d,%d,%d,%d,%d,%d,%s,%d,%.2f,%d,%d,%d,%d\n", r.M, r.N, r.K, r.amn, r.bmn, r.act, r.nex, r.splits,
                    r.kern >= 1000 ? (r.kern == 1003 ? "tail3" : "tail2") : (r.kern == 128 ? (r.cluster == 2 ? "p128c2" : "p128") : (r.kern == 64 ? "p64" : "p32")),
                    r.colsum, 1e3 * t, r.n3, r.heads, r.problems, r.bf16);
        }
    }
    if (csv) fclose(csv);
    if (total_ms) *total_ms = ms;
    if (total_flop) *total_flop = g_time_flop;
    if (launches) *launches = (long long)(g_time_used / 2);
    return 0;
}

// the MN-major BF16 kernel of layout mn (bit 0: A MN-major, bit 1: B MN-major)
template <int BN, bool ANYKIND, bool DET>
int launch_gemm_mn(int mn, const GemmMaps& gm, const CUtensorMap& mc, const CUtensorMap& my, GemmArgs& g, int splits, cudaStream_t st, const DetArgs& det) {
    switch (mn) {
        case 0: return launch_gemm<BN, ANYKIND, 1, true, 0, DET>(gm, mc, my, g, splits, st, det);
        case 1: return launch_gemm<BN, ANYKIND, 1, true, 1, DET>(gm, mc, my, g, splits, st, det);
        case 2: return launch_gemm<BN, ANYKIND, 1, true, 2, DET>(gm, mc, my, g, splits, st, det);
        default: return launch_gemm<BN, ANYKIND, 1, true, 3, DET>(gm, mc, my, g, splits, st, det);
    }
}
// the kernel of (mnk, cluster, BN, any) in the default or the deterministic instantiation
template <bool BF16, bool DET>
int launch_gemm_any(int mnk, int cluster, int BN, bool any, const GemmMaps& gm, const CUtensorMap& mc, const CUtensorMap& my, GemmArgs& g, int splits, cudaStream_t st,
                    const DetArgs& det) {
    if (mnk >= 0) {
        if constexpr (BF16) {
            if (BN == 128) return any ? launch_gemm_mn<128, true, DET>(mnk, gm, mc, my, g, splits, st, det) : launch_gemm_mn<128, false, DET>(mnk, gm, mc, my, g, splits, st, det);
            if (BN == 64) return any ? launch_gemm_mn<64, true, DET>(mnk, gm, mc, my, g, splits, st, det) : launch_gemm_mn<64, false, DET>(mnk, gm, mc, my, g, splits, st, det);
            return any ? launch_gemm_mn<32, true, DET>(mnk, gm, mc, my, g, splits, st, det) : launch_gemm_mn<32, false, DET>(mnk, gm, mc, my, g, splits, st, det);
        }
        return go1_set_error("go1_gemm: MN-major BF16 layout without BF16 operands");
    }
    if (cluster == 2) return any ? launch_gemm<128, true, 2, BF16, -1, DET>(gm, mc, my, g, splits, st, det) : launch_gemm<128, false, 2, BF16, -1, DET>(gm, mc, my, g, splits, st, det);
    if (BN == 128) return any ? launch_gemm<128, true, 1, BF16, -1, DET>(gm, mc, my, g, splits, st, det) : launch_gemm<128, false, 1, BF16, -1, DET>(gm, mc, my, g, splits, st, det);
    if (BN == 64) return any ? launch_gemm<64, true, 1, BF16, -1, DET>(gm, mc, my, g, splits, st, det) : launch_gemm<64, false, 1, BF16, -1, DET>(gm, mc, my, g, splits, st, det);
    return any ? launch_gemm<32, true, 1, BF16, -1, DET>(gm, mc, my, g, splits, st, det) : launch_gemm<32, false, 1, BF16, -1, DET>(gm, mc, my, g, splits, st, det);
}

// T = float: TF32 products (operands in either major); T = uint16_t: BF16 products, K-major operands only (go1_gemm_bf16_ex), or with
// mn (go1_gemm_bf16_mn / go1_gemm_bf16_grouped) in either major, read in place, and with row16 a row-major BF16 C (Cs[0] is then a
// uint16_t matrix, ldc in elements).  One code path for all: only the operand maps, the k-block width and the tensor-core instruction differ.
template <typename T>
static int gemm_wgmma_impl(int transA, int transB, int M, int N, int K, int nprob, const T* const* As, int lda, const T* const* Bs, int ldb,
                           float* const* Cs, int ldc, const Go1GemmEpilogue* ep, cudaStream_t st, bool mn = false, bool row16 = false) {
    constexpr bool BF16 = sizeof(T) == 2;
    constexpr int ES = sizeof(T), KE = 128 / ES;      // operand element size, operand elements per k-block (one 128-byte row)
    float* Cm = Cs[0];
    const float* bias = ep->bias; const int act = ep->act, accumulate = ep->accumulate;
    if (act < 0 || act > 2) return go1_set_error("go1_gemm_ex: act must be 0, 1 or 2");
    if (!go1_act_kind_ok(ep->act_kind)) return go1_set_error("go1_gemm_ex: unknown activation kind (Go1Activation)");
    const int amn = transA ? 1 : 0, bmn = transB ? 0 : 1;     // A given as [K][M] / B given as [K][N]: MN-major operands
    if (BF16 && !mn && (amn || bmn)) return go1_set_error("go1_gemm_bf16_ex: both operands must be K-major (transA = 0, transB = 1)");
    const bool c16 = ep->out_bf16 != nullptr;
    if (row16 && (c16 || ep->store_transposed || accumulate || nprob != 1 || (ldc & 7) || ldc < N || (((uintptr_t)Cm) & 15)))
        return go1_set_error("go1_gemm_bf16_mn: c_bf16 needs a 16-byte aligned C with ldc >= N, a multiple of 8, no accumulate, no store_transposed and no out_bf16");
    if (c16 && (!ep->store_transposed || (ep->ld_out_bf16 & 7) || ep->ld_out_bf16 < M || (((uintptr_t)ep->out_bf16) & 15)))
        return go1_set_error("go1_gemm_ex: out_bf16 needs store_transposed, a 16-byte aligned output and ld_out_bf16 >= M, a multiple of 8");
    for (int p = 0; p < nprob; p++)
        if (((lda * ES) & 15) || ((ldb * ES) & 15) || (((uintptr_t)As[p] | (uintptr_t)Bs[p]) & 15) || (!Cs[p] && !c16))
            return go1_set_error(BF16 ? (mn ? "go1_gemm_bf16_mn: A/B must be 16-byte aligned with row strides that are multiples of 8 elements (TMA)"
                                            : "go1_gemm_bf16_ex: A/B must be 16-byte aligned with row strides that are multiples of 8 elements (TMA)")
                                      : "go1_gemm impl=1: A/B must be 16-byte aligned with row strides that are multiples of 4 floats (TMA)");
    GemmArgs g;
    g.nprob = nprob; g.tiles_per_prob = 0;
    for (int p = 0; p < GEMM_MAXP; p++) g.Cg[p] = Cs[p < nprob ? p : 0];
    g.C = Cm; g.bias = bias; g.M = M; g.N = N; g.K = K; g.ldc = ldc; g.act = act; g.kind = ep->act_kind; g.accumulate = accumulate;
    g.ex = ep->extra; g.ldex = ep->ld_extra; g.wex = ep->w_extra; g.ldwex = ep->ld_w_extra; g.nex = ep->extra ? ep->num_extra : 0;
    g.aux = ep->dact_y; g.ldaux = ep->ld_dact_y;
    g.amn = amn; g.bmn = bmn; g.lead = ep->lead_cols; g.colsum = ep->colsum; g.ct = ep->store_transposed ? 1 : 0; g.c16 = (c16 || row16) ? 1 : 0;
    g.nbx = ep->num_bwd_extra; g.bx = ep->bwd_extra; g.bwx = ep->bwd_w_extra; g.gwx = ep->g_w_extra; g.dx = ep->d_extra;
    g.ldbx = ep->ld_bwd_extra; g.ldbwx = ep->ld_bwd_w_extra; g.ldgwx = ep->ld_g_w_extra; g.lddx = ep->ld_d_extra;
    if (g.nbx < 0 || g.nbx > 4 || (g.nbx > 0 && ((g.gwx && !g.bx) || (!g.gwx && !g.dx) || (g.dx && !g.bwx)))) return go1_set_error("go1_gemm_ex: bad fused trailing-input backward arguments");
    if (g.nex < 0 || g.nex > 4) return go1_set_error("go1_gemm_ex: num_extra must be 0..4");
    if (act == 2 && !g.aux) return go1_set_error("go1_gemm_ex: act 2 needs dact_y");
    if (g.ct && (nprob != 1 || accumulate || M < 32 || (!c16 && ((ldc & 3) || (((uintptr_t)Cm) & 15)))))      // the transposed blocks leave by TMA store only
        return go1_set_error("go1_gemm_ex: store_transposed needs M >= 32, no accumulate and a 16-byte aligned C with ldc a multiple of 4");
    const int num_kb = (K + KE - 1) / KE;
    // Tile selection: 128 x BN tiles, BN = the smallest of 32 / 64 / 128 that covers N (128 beyond).  Plain products (no fused epilogue) with a
    // long reduction are split along K (partial tiles meet in C by vector reductions).
    constexpr int SPLIT_MIN_KB = 16;          // least k-blocks per split
    const int BN = (N > 64) ? 128 : (N > 32 ? 64 : 32);
    const int tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN) * nprob;
    const bool plain = g.nex == 0 && act != 2 && g.lead <= 0 && !g.colsum && g.nbx == 0 && !g.ct && !row16;
    const int splits = plain ? split_count(tiles, num_kb, SPLIT_MIN_KB, sm_count()) : 1;
    g.kb_per_split = (num_kb + splits - 1) / splits;
    GemmMaps gm;
    // K-major: rows = M (or N), cols = K, box BK x tile rows.  MN-major: rows = K, cols = M (or N), box tile width x BK k-rows; BF16:
    // 64 k-rows x 64 mn, 128B-swizzled (BN = 32: 64 k-rows x 32 n, 64B-swizzled), read in place by the tensor core.
    for (int p = 0; p < nprob; p++) {
        int e = 0;
        if (BF16 && amn) e = make_map(&gm.a[p], As[p], K, M, lda, KE, BM / 2, CU_TENSOR_MAP_SWIZZLE_128B, ES);
        else e = amn ? make_map_mn(&gm.a[p], (const float*)As[p], K, M, lda, BM) : make_map(&gm.a[p], As[p], M, K, lda, BM, KE, CU_TENSOR_MAP_SWIZZLE_128B, ES);
        if (e) return e;
        if (BF16 && bmn) e = make_map(&gm.b[p], Bs[p], K, N, ldb, KE, BN == 32 ? 32 : 64, BN == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, ES);
        else e = bmn ? make_map_mn(&gm.b[p], (const float*)Bs[p], K, N, ldb, BN) : make_map(&gm.b[p], Bs[p], N, K, ldb, BN, KE, CU_TENSOR_MAP_SWIZZLE_128B, ES);
        if (e) return e;
    }
    const int mnk = BF16 && (amn || bmn || row16) ? (amn | (bmn << 1)) : -1;      // >= 0: gemm_bf16_mn_wgmma of that layout
    for (int p = nprob; p < GEMM_MAXP; p++) { gm.a[p] = gm.a[0]; gm.b[p] = gm.b[0]; }
    const CUtensorMap& ma = gm.a[0];
    // CTA pairs (cluster of 2) share one operand box of every k-block by multicast: K-major operands, one problem, 128 x 128 tiles and an
    // even tile count along N (pairs share A) or else along M (pairs share B).  Same tiles, instructions and order of the sums as one CTA.
    // No derivative operand (act 2, the dgrads, whose W is MN-major anyway): without its prefetch registers the pair kernels spill less.
    const int tiles_m = (M + BM - 1) / BM, tiles_n = (N + BN - 1) / BN;
    const int cluster = (mnk < 0 && !amn && !bmn && nprob == 1 && act != 2 && BN == 128 && (tiles_n % 2 == 0 || tiles_m % 2 == 0)) ? 2 : 1;
    gm.half = ma;
    if (cluster == 2) {
        if (int e = tiles_n % 2 == 0 ? make_map(&gm.half, As[0], M, K, lda, BM / 2, KE, CU_TENSOR_MAP_SWIZZLE_128B, ES)
                                     : make_map(&gm.half, Bs[0], N, K, ldb, BN / 2, KE, CU_TENSOR_MAP_SWIZZLE_128B, ES)) return e;
    }
    // deterministic mode: the launches whose CTAs add into shared targets run their DET kernels, whose partials go to the stream's workspace
    const bool det = go1_det_on() && (splits > 1 || g.colsum || (g.nbx > 0 && (g.gwx || g.dx)));
    DetArgs da = {};
    if (det) {
        const size_t nrb = (size_t)(M + 31) / 32, ncb = (size_t)(N + 31) / 32;
        const size_t r4 = 3;        // region sizes rounded up to 16 bytes
        const size_t n_split = splits > 1 ? ((size_t)nprob * splits * M * ldc + r4) & ~r4 : 0, n_cs = g.colsum ? (nrb * N + r4) & ~r4 : 0;
        const size_t n_gwx = g.nbx > 0 && g.gwx ? (nrb * N * g.nbx + r4) & ~r4 : 0, n_dx = g.nbx > 0 && g.dx ? (ncb * M * g.nbx + r4) & ~r4 : 0;
        float* ws = (float*)go1_det_workspace(st, sizeof(float) * (n_split + n_cs + n_gwx + n_dx));
        if (!ws) return 1;
        da.split = ws; da.slab = (size_t)M * ldc; da.nsplit = splits;
        da.cs = ws + n_split; da.gwx = da.cs + n_cs; da.dx = da.gwx + n_gwx;
    }
    if (splits > 1) {
        if (!accumulate && !det)
            for (int p = 0; p < nprob; p++) { const size_t tot = (size_t)M * N; zero_strided<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(Cs[p], ldc, M, N); go1_count_launch(1); }
        g.bias = nullptr; g.act = 0;
    }
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    const bool timed = g_time_on && cudaStreamIsCapturing(st, &cap) == cudaSuccess && cap == cudaStreamCaptureStatusNone;
    if (timed) {
        cudaEventRecord(timing_event(), st); g_time_flop += 2.0 * (double)M * (double)N * (double)K * nprob;
        g_time_recs.push_back({M * nprob, N, K, amn, bmn, act, g.nex, splits, BN, g.colsum ? 1 : 0, cluster, 0, 0, nprob, BF16 ? (mn ? 2 : 1) : 0});
    }
    int e;
    // staged epilogue: C blocks leave the accumulator staging by TMA store, the derivative operand arrives through TMA loads.  The direct
    // row-per-lane stores serve the rest: split-K partial tiles, accumulate, grouped launches, N < 32 and a misaligned C.
    CUtensorMap mc = ma, my = ma;
    g.tma_store = g.tma_aux = 0;
    if (row16) {        // row-major BF16 C: 32 x 32 blocks of 64-byte rows, 64B-swizzled (N < 32: direct stores)
        if (N >= 32) {
            if (int e2 = make_map(&mc, Cm, M, N, ldc, 32, 32, CU_TENSOR_MAP_SWIZZLE_64B, 2)) return e2;
            g.tma_store = 1;
        }
    } else if (c16) {   // (a BF16 transposed store: checked above) 32 x 32 blocks of 64-byte rows, unswizzled
        if (int e2 = make_map(&mc, ep->out_bf16, N, M, ep->ld_out_bf16, 32, 32, CU_TENSOR_MAP_SWIZZLE_NONE, 2)) return e2;
        g.tma_store = 1;
    } else if (nprob == 1 && splits == 1 && !accumulate && (g.ct ? M : N) >= 32 && (ldc & 3) == 0 && (((uintptr_t)Cm) & 15) == 0) {
        if (int e2 = g.ct ? make_map(&mc, Cm, N, M, ldc, 32) : make_map(&mc, Cm, M, N, ldc, 32)) return e2;
        g.tma_store = 1;
    }
    if (g.tma_store) {
        if (g.act == 2 && (g.ldaux & 3) == 0 && (((uintptr_t)g.aux) & 15) == 0) {
            if (int e2 = make_map(&my, g.aux, M, N, g.ldaux, 32)) return e2;
            g.tma_aux = 1;
        }
    }
    const bool any = g.act != 0 && g.kind != GO1_ACT_ELU;
    e = det ? launch_gemm_any<BF16, true>(mnk, cluster, BN, any, gm, mc, my, g, splits, st, da)
            : launch_gemm_any<BF16, false>(mnk, cluster, BN, any, gm, mc, my, g, splits, st, da);
    if (e) return e;
    if (det) {      // the partials, in a fixed order, into C (split-K: overwriting it unless accumulate) and the epilogue's targets (adding)
        if (splits > 1)
            for (int p = 0; p < nprob; p++)
                if (int e2 = go1_det_sum(da.split + (size_t)p * splits * da.slab, splits, da.slab, Cs[p], M, N, ldc, accumulate, st, ldc)) return e2;
        const int nrb = (M + 31) / 32, ncb = (N + 31) / 32;
        if (g.colsum) { if (int e2 = go1_det_sum(da.cs, nrb, N, g.colsum, 1, N, N, 1, st)) return e2; }
        if (g.nbx > 0 && g.gwx) { if (int e2 = go1_det_sum(da.gwx, nrb, (size_t)N * g.nbx, g.gwx, N, g.nbx, g.ldgwx, 1, st)) return e2; }
        if (g.nbx > 0 && g.dx) { if (int e2 = go1_det_sum(da.dx, ncb, (size_t)M * g.nbx, g.dx, M, g.nbx, g.lddx, 1, st)) return e2; }
    }
    if (splits > 1 && (bias || act))
        for (int p = 0; p < nprob; p++) { const size_t tot = (size_t)M * N; bias_act_strided<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(Cs[p], ldc, bias, M, N, act, ep->act_kind); go1_count_launch(1); }
    if (timed) cudaEventRecord(timing_event(), st);
    cudaError_t ce = cudaGetLastError();
    if (ce != cudaSuccess) return go1_set_error(cudaGetErrorString(ce));
    return 0;
}

extern "C" int go1_gemm_tf32(int transA, int transB, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
                             float* Cm, int ldc, const Go1GemmEpilogue* ep, cudaStream_t st) {
    return gemm_wgmma_impl<float>(transA, transB, M, N, K, 1, &A, lda, &B, ldb, &Cm, ldc, ep, st);
}
// BF16 operands, fp32 accumulation and output, the full fused epilogue of go1_gemm_ex impl 1 (include/go1_b200.h)
extern "C" int go1_gemm_bf16_ex(int transA, int transB, int M, int N, int K, const uint16_t* A, int lda, const uint16_t* B, int ldb,
                                float* Cm, int ldc, const Go1GemmEpilogue* ep, void* stream) {
    if (!A || !B || !ep || M <= 0 || N <= 0 || K <= 0) return go1_set_error("go1_gemm_bf16_ex: bad arguments");
    if (!ep->out_bf16 && (!Cm || ldc < N)) return go1_set_error("go1_gemm_bf16_ex: bad output");
    return gemm_wgmma_impl<uint16_t>(transA, transB, M, N, K, 1, &A, lda, &B, ldb, &Cm, ldc, ep, (cudaStream_t)stream);
}
// BF16 operands in either major, read in place (MN-major ones through the tensor core's transpose immediates); C fp32, or with c_bf16 a
// row-major BF16 matrix (uint16_t, ldc elements); the full fused epilogue (include/go1_b200.h)
extern "C" int go1_gemm_bf16_mn(int transA, int transB, int M, int N, int K, const uint16_t* A, int lda, const uint16_t* B, int ldb,
                                void* Cm, int ldc, int c_bf16, const Go1GemmEpilogue* ep, void* stream) {
    if (!A || !B || !ep || M <= 0 || N <= 0 || K <= 0 || (transA & ~1) || (transB & ~1) || (c_bf16 & ~1)) return go1_set_error("go1_gemm_bf16_mn: bad arguments");
    if (!ep->out_bf16 && (!Cm || ldc < (ep->store_transposed ? M : N))) return go1_set_error("go1_gemm_bf16_mn: bad output");
    float* C = (float*)Cm;
    return gemm_wgmma_impl<uint16_t>(transA, transB, M, N, K, 1, &A, lda, &B, ldb, &C, ldc, ep, (cudaStream_t)stream, true, c_bf16 != 0);
}
// go1_gemm_grouped with BF16 operands in either major (the equal-shape weight gradients of AC_Args.bf16_backward)
extern "C" int go1_gemm_bf16_grouped(int transA, int transB, int M, int N, int K, int nprob, const uint16_t* const* A, int lda, const uint16_t* const* B, int ldb,
                                     float* const* C, int ldc, int accumulate, void* stream) {
    if (!A || !B || !C || nprob < 1 || nprob > GEMM_MAXP || M <= 0 || N <= 0 || K <= 0 || (transA & ~1) || (transB & ~1))
        return go1_set_error("go1_gemm_bf16_grouped: 1..4 problems");
    for (int p = 0; p < nprob; p++) if (!A[p] || !B[p] || !C[p]) return go1_set_error("go1_gemm_bf16_grouped: bad arguments");
    if (ldc < N) return go1_set_error("go1_gemm_bf16_grouped: bad output");
    Go1GemmEpilogue ep = {};
    ep.accumulate = accumulate;
    return gemm_wgmma_impl<uint16_t>(transA, transB, M, N, K, nprob, A, lda, B, ldb, C, ldc, &ep, (cudaStream_t)stream, true, false);
}
// nprob (<= 4) products of the same shape and operand strides in ONE grid: C[p] (+)= op(A[p]) op(B[p]).  Meant for the equal-shape
// split-K wgrads of the three MLPs (128 x 256 x 24576 three times, 256 x 512 x 24576 twice per optimizer step): one launch fills the
// SMs that a single two-tile product leaves idle.  No fused epilogue operands.
extern "C" int go1_gemm_grouped(int transA, int transB, int M, int N, int K, int nprob, const float* const* A, int lda, const float* const* B, int ldb,
                                float* const* C, int ldc, int accumulate, void* stream) {
    if (!A || !B || !C || nprob < 1 || nprob > GEMM_MAXP || M <= 0 || N <= 0 || K <= 0) return go1_set_error("go1_gemm_grouped: 1..4 problems");
    Go1GemmEpilogue ep = {};
    ep.accumulate = accumulate;
    return gemm_wgmma_impl<float>(transA, transB, M, N, K, nprob, A, lda, B, ldb, C, ldc, &ep, (cudaStream_t)stream);
}

// dst[c][r] = src[r][c]  (32x32 smem tiles)
__global__ void transpose_kernel(const float* __restrict__ src, int lds, float* __restrict__ dst, int ldd, int rows, int cols) {
    __shared__ float t[32][33];
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        t[i][threadIdx.x] = (r < rows && c < cols) ? src[(size_t)r * lds + c] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int c = c0 + i, r = r0 + threadIdx.x;
        if (c < cols && r < rows) dst[(size_t)c * ldd + r] = t[threadIdx.x][i];
    }
}
extern "C" int go1_transpose(const float* src, int lds, float* dst, int ldd, int rows, int cols, void* stream) {
    if (!src || !dst || rows <= 0 || cols <= 0 || lds < cols || ldd < rows) return go1_set_error("go1_transpose: bad arguments");
    dim3 grid((cols + 31) / 32, (rows + 31) / 32);
    transpose_kernel<<<grid, dim3(32, 8), 0, (cudaStream_t)stream>>>(src, lds, dst, ldd, rows, cols);
    go1_count_launch(1);
    cudaError_t ce = cudaGetLastError();
    if (ce != cudaSuccess) return go1_set_error(cudaGetErrorString(ce));
    return 0;
}


// ---- fused MLP tail (forward), see mlp_tail_fwd_kernel
extern "C" int go1_mlp_tail_forward_grouped(const Go1TailProblem* probs, int nprob, int M, int K1, int N2, int N3, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (!probs || nprob < 1 || nprob > TAIL_MAXP || M <= 0) return go1_set_error("go1_mlp_tail_forward: 1 or 2 problems of the same shape");
    if (K1 < 1 || N2 < 1 || N2 > 256 || N3 < 0 || N3 > 128) return go1_set_error("go1_mlp_tail_forward: tail widths N2 1..256, N3 0..128 (K1 >= 1)");
    // scripts/train.py's two tails on their exact-width kernels, every other shape on the ragged ones
    bool shape_a = (K1 == 512 && N2 == 256 && N3 == 128), shape_b = (K1 == 256 && N2 == 128 && N3 == 0);
    for (int p = 0; p < nprob; p++)
        if ((probs[p].ldw2 != 0 && probs[p].ldw2 != K1) || (N3 > 0 && probs[p].ldw3 != 0 && probs[p].ldw3 != N2)) shape_a = shape_b = false;
    TailMaps maps;
    TailArgs g;
    g.nprob = nprob; g.M = M; g.tiles_per_prob = (M + TAIL_BM - 1) / TAIL_BM; g.tiles = g.tiles_per_prob * nprob;
    g.kind = probs[0].act_kind;
    if (!go1_act_kind_ok(g.kind)) return go1_set_error("go1_mlp_tail_forward: unknown activation kind (Go1Activation)");
    int rows = 0;
    for (int p = 0; p < nprob; p++) {
        const Go1TailProblem& q = probs[p];
        if (q.act_kind != g.kind) return go1_set_error("go1_mlp_tail_forward: the problems of one launch share their activation kind");
        if (!q.x || !q.W2 || !q.y2 || !q.Wh || !q.out || q.nh < 1 || q.nh > TAIL_HPW || q.ldout < q.nh) return go1_set_error("go1_mlp_tail_forward: bad arguments (head width 1..12)");
        if (N3 > 0 && (!q.W3 || !q.y3)) return go1_set_error("go1_mlp_tail_forward: the three-layer tail needs W3 / y3");
        const int ldw2 = q.ldw2 ? q.ldw2 : K1, ldw3 = q.ldw3 ? q.ldw3 : N2;
        if ((q.ldx & 3) || (q.ldy2 & 3) || (N3 > 0 && (q.ldy3 & 3)) || (ldw2 & 3) || ldw2 < K1 || (N3 > 0 && ((ldw3 & 3) || ldw3 < N2)) ||
            ((((uintptr_t)q.x | (uintptr_t)q.W2 | (uintptr_t)q.y2 | (uintptr_t)(N3 > 0 ? (const void*)q.W3 : (const void*)q.W2) |
               (uintptr_t)(N3 > 0 ? (const void*)q.y3 : (const void*)q.y2)) & 15) != 0))
            return go1_set_error("go1_mlp_tail_forward: operands must be 16-byte aligned with row strides that are multiples of 4 floats");
        if (int e = make_map(&maps.x[p], q.x, M, K1, q.ldx, TAIL_BM)) return e;
        // boxes of the tile widths: the rows beyond N2 / N3 of a ragged tail read as zeros
        const int t2 = N2 <= 64 ? 64 : N2 <= 128 ? 128 : 256, t3 = N3 <= 64 ? 64 : 128;
        if (int e = make_map(&maps.w2[p], q.W2, N2, K1, ldw2, t2)) return e;
        if (N3 > 0) { if (int e = make_map(&maps.w3[p], q.W3, N3, N2, ldw3, t3)) return e; } else maps.w3[p] = maps.w2[p];
        if (int e = make_map(&maps.y2[p], q.y2, M, N2, q.ldy2, 32)) return e;
        TailProb& d = g.p[p];
        d.b2 = q.b2; d.b3 = q.b3; d.Wh = q.Wh; d.bh = q.bh; d.y3 = q.y3; d.out = q.out; d.ldy3 = q.ldy3; d.ldout = q.ldout; d.nh = q.nh; d.wh_row0 = rows;
        rows += q.nh;
    }
    if (rows > 16) return go1_set_error("go1_mlp_tail_forward: the head rows of all problems must fit 16");
    for (int p = nprob; p < TAIL_MAXP; p++) { maps.x[p] = maps.x[0]; maps.w2[p] = maps.w2[0]; maps.w3[p] = maps.w3[0]; maps.y2[p] = maps.y2[0]; g.p[p] = g.p[0]; }
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    const bool timed = g_time_on && cudaStreamIsCapturing(st, &cap) == cudaSuccess && cap == cudaStreamCaptureStatusNone;
    if (timed) {
        cudaEventRecord(timing_event(), st);
        double fl = 0.0;
        for (int p = 0; p < nprob; p++) fl += 2.0 * (double)M * ((double)K1 * N2 + (double)N2 * N3 + (double)(N3 > 0 ? N3 : N2) * probs[p].nh);
        g_time_flop += fl;
        g_time_recs.push_back({M * nprob, N2, K1, 0, 0, 1, 0, 1, N3 > 0 ? 1003 : 1002, 0, 1, N3, rows, nprob});
    }
    int e;
    const bool any = g.kind != GO1_ACT_ELU;
    if (shape_a) e = any ? launch_tail<512, 256, 128, true>(maps, g, st) : launch_tail<512, 256, 128, false>(maps, g, st);
    else if (shape_b) e = any ? launch_tail<256, 128, 0, true>(maps, g, st) : launch_tail<256, 128, 0, false>(maps, g, st);
    else e = any ? launch_tail_ragged_any<true>(maps, g, TailDims{K1, N2, N3}, st) : launch_tail_ragged_any<false>(maps, g, TailDims{K1, N2, N3}, st);
    if (e) return e;
    if (timed) cudaEventRecord(timing_event(), st);
    cudaError_t ce = cudaGetLastError();
    if (ce != cudaSuccess) return go1_set_error(cudaGetErrorString(ce));
    return 0;
}
extern "C" int go1_mlp_tail_forward(const float* x, int ldx, int M, int K1, const float* W2, const float* b2, int N2, float* y2, int ldy2,
                                    const float* W3, const float* b3, int N3, float* y3, int ldy3, const float* Wh, const float* bh, int nh,
                                    float* out, int ldout, void* stream) {
    Go1TailProblem q = {};
    q.x = x; q.ldx = ldx; q.W2 = W2; q.b2 = b2; q.y2 = y2; q.ldy2 = ldy2; q.W3 = W3; q.b3 = b3; q.y3 = y3; q.ldy3 = ldy3; q.Wh = Wh; q.bh = bh; q.nh = nh; q.out = out; q.ldout = ldout;
    return go1_mlp_tail_forward_grouped(&q, 1, M, K1, N2, N3, stream);
}
