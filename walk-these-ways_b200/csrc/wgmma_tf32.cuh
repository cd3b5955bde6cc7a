// wgmma_tf32.cuh — sm_90a warpgroup MMA (wgmma.mma_async, TF32 or BF16 operands from shared memory, fp32 accumulators in registers).
//
// One TF32 instruction multiplies a 64 x 8 slice of A by an 8 x N slice of B (BF16: 64 x 16 by 16 x N), both K-major in shared memory
// (TF32 wgmma has no transposed-operand form: MN-major data must be brought to K-major first; BF16 reads MN-major tiles through its transpose
// immediates: mma_kblock_bf16).  Accumulator fragment of thread t of the warpgroup
// (warp w = t / 32, lane l): d[4 j + 0 / 1] = C[16 w + l / 4][8 j + 2 (l % 4) + 0 / 1], d[4 j + 2 / 3] = the same columns of row + 8.
#pragma once
#include <stdint.h>

namespace wg {

__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// K-major operand tile with 128-byte rows, 128B-swizzled (what TMA writes with CU_TENSOR_MAP_SWIZZLE_128B): 8-row groups 1024 B apart.
// Advancing by one instruction along K (8 floats or 16 bf16 = 32 bytes) adds 2 to the descriptor.
__device__ __forceinline__ uint64_t desc(const void* smem) {
    uint64_t d = 0;
    d |= (uint64_t)(((uint32_t)__cvta_generic_to_shared(smem) >> 4) & 0x3FFF);      // start address
    d |= (uint64_t)1 << 16;                                                         // leading byte offset (unused for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;                                               // stride byte offset
    d |= (uint64_t)1 << 62;                                                         // SWIZZLE_128B
    return d;
}

// TF32 instructions (k8: 8 floats = 32 bytes of a 128-byte row) and BF16 ones (k16: 16 bf16 = the same 32 bytes), both operands K-major
// (the BF16 form's transpose immediates are 0).  The k-block is one 128-byte swizzle row either way: 32 floats or 64 bf16.
#define GO1_WG_D16 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
#define GO1_WG_D32 GO1_WG_D16, "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
#define GO1_WG_D64 GO1_WG_D32, "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
    "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define GO1_WG_R16 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}"
#define GO1_WG_R32 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define GO1_WG_R64 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, " \
    "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
// INSTR: the instruction with its shape and types; R: the accumulator registers; A, B, P: the operand numbers of the two descriptors
// and of `accumulate`; TAIL: the immediates behind scale-d (scale-a, scale-b, and for 16-bit operands the two transpose flags); then
// the accumulator operand list
#define GO1_WG_MMA(INSTR, R, A, B, P, TAIL, ...) \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" P ", 0;\n\t" INSTR " " R ", %" A ", %" B ", p, " TAIL ";\n\t}" \
                 : __VA_ARGS__ : "l"(da), "l"(db), "r"(accumulate))

template <int N, bool BF16> __device__ __forceinline__ void mma(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate);
#define GO1_WG_SPEC(N, BF16, INSTR, R, A, B, P, TAIL, ...) \
    template <> __device__ __forceinline__ void mma<N, BF16>(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate) { GO1_WG_MMA(INSTR, R, A, B, P, TAIL, __VA_ARGS__); }
GO1_WG_SPEC(32, false, "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32", GO1_WG_R16, "16", "17", "18", "1, 1", GO1_WG_D16)
GO1_WG_SPEC(64, false, "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32", GO1_WG_R32, "32", "33", "34", "1, 1", GO1_WG_D32)
GO1_WG_SPEC(128, false, "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32", GO1_WG_R64, "64", "65", "66", "1, 1", GO1_WG_D64)
GO1_WG_SPEC(32, true, "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16", GO1_WG_R16, "16", "17", "18", "1, 1, 0, 0", GO1_WG_D16)
GO1_WG_SPEC(64, true, "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16", GO1_WG_R32, "32", "33", "34", "1, 1, 0, 0", GO1_WG_D32)
GO1_WG_SPEC(128, true, "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16", GO1_WG_R64, "64", "65", "66", "1, 1, 0, 0", GO1_WG_D64)
#undef GO1_WG_SPEC

// One k-block (one 128-byte swizzle row: 32 floats or 64 bf16) of a 64 x N product: four instructions.
template <int N, bool BF16 = false> __device__ __forceinline__ void mma_kblock(float (&d)[N / 2], const void* a, const void* b, bool accumulate) {
    const uint64_t da = desc(a), db = desc(b);
#pragma unroll
    for (int k = 0; k < 4; k++) mma<N, BF16>(d, da + 2 * k, db + 2 * k, (accumulate || k > 0) ? 1u : 0u);
}

// MN-major 16-bit operand tiles, as TMA writes a [64 k][64 mn] box with CU_TENSOR_MAP_SWIZZLE_128B (128-byte rows along MN, 16-byte
// chunks XOR-swizzled by k % 8).  PTX ISA's MN-major canonical layout: the 8-k-row groups are the stride byte offset apart (1024 B) and the
// next 64 mn (the next box) the leading byte offset apart (lbo).  One k16 instruction step is 16 k-rows = 2048 B: +128 in the descriptor.
__device__ __forceinline__ uint64_t desc_mn128(const void* smem, uint32_t lbo) {
    uint64_t d = 0;
    d |= (uint64_t)(((uint32_t)__cvta_generic_to_shared(smem) >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;                                                         // SWIZZLE_128B
    return d;
}
// The 32-wide form, a [64 k][32 mn] box with CU_TENSOR_MAP_SWIZZLE_64B (64-byte rows): 8-k-row groups 512 B apart, a k16 step is 1024 B (+64).
__device__ __forceinline__ uint64_t desc_mn64(const void* smem) {
    uint64_t d = 0;
    d |= (uint64_t)(((uint32_t)__cvta_generic_to_shared(smem) >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(512 >> 4) << 32;
    d |= (uint64_t)2 << 62;                                                         // SWIZZLE_64B
    return d;
}

// BF16 instructions with the transpose immediates TA / TB (1: that operand is MN-major in shared memory)
#define GO1_WG_MMAT(INSTR, R, A, B, P, TA, TB, ...) \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" P ", 0;\n\t" INSTR " " R ", %" A ", %" B ", p, 1, 1, %" TA ", %" TB ";\n\t}" \
                 : __VA_ARGS__ : "l"(da), "l"(db), "r"(accumulate), "n"(TRA), "n"(TRB))
template <int N> struct MmaBf16T;
template <> struct MmaBf16T<32> { template <int TRA, int TRB> static __device__ __forceinline__ void run(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
    GO1_WG_MMAT("wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16", GO1_WG_R16, "16", "17", "18", "19", "20", GO1_WG_D16); } };
template <> struct MmaBf16T<64> { template <int TRA, int TRB> static __device__ __forceinline__ void run(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
    GO1_WG_MMAT("wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16", GO1_WG_R32, "32", "33", "34", "35", "36", GO1_WG_D32); } };
template <> struct MmaBf16T<128> { template <int TRA, int TRB> static __device__ __forceinline__ void run(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    GO1_WG_MMAT("wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16", GO1_WG_R64, "64", "65", "66", "67", "68", GO1_WG_D64); } };
#undef GO1_WG_MMAT

// One BF16 k-block (64 k) of a 64 x N product whose operands are K-major (TA / TB = 0: da / db from desc, +2 per k16) or MN-major
// (1: da from desc_mn128, db from desc_mn128 or, N = 32, desc_mn64; +128 / +64 per k16).
template <int N, int TA, int TB>
__device__ __forceinline__ void mma_kblock_bf16(float (&d)[N / 2], const uint64_t da, const uint64_t db, bool accumulate) {
    constexpr uint32_t sa = TA ? 128 : 2, sb = TB ? (N == 32 ? 64 : 128) : 2;
#pragma unroll
    for (int k = 0; k < 4; k++) MmaBf16T<N>::template run<TA, TB>(d, da + sa * k, db + sb * k, (accumulate || k > 0) ? 1u : 0u);
}

}  // namespace wg
