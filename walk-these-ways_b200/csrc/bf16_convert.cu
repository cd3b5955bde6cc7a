// bf16_convert.cu — data movement into BF16 for the products of AC_Args.gemm_impl = 2 (go1_gemm_bf16_ex, whose operands reduce over the
// observation history): the packed first-layer weights and the policy's input history (go1_convert_bf16), its store into the rollout's
// BF16 history slab (go1_rollout_store_rows_bf16), the minibatch gather from that slab (go1_gather_rows_bf16) and the K-major copy [history | 1 | priv | latent]^T of the first-layer weight gradients (go1_transpose_*);
// for AC_Args.bf16_backward the hidden-layer outputs of a minibatch forward, several matrices in one launch (go1_convert_bf16_segments).
// Every fp32 value is rounded once, to nearest even (__float2bfloat16_rn, bit-identical to torch's .to(torch.bfloat16)); BF16 sources
// are copied.  Only the listed columns of a destination row are written: pitch padding stays as it was.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include "../../include/go1_b200.h"

extern int go1_set_error(const char* m);
void go1_count_launch(int n);

namespace {

__device__ __forceinline__ uint16_t to_bf16(float v) { return __bfloat16_as_ushort(__float2bfloat16_rn(v)); }
__device__ __forceinline__ uint16_t to_bf16(uint16_t v) { return v; }

int launch_rc() {
    go1_count_launch(1);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : go1_set_error(cudaGetErrorString(e));
}

// one CTA per destination row (src row = idx[r] or r); four columns per thread per step, vector loads where the source allows them.
// slot_dev (optional): dst is the base of a slab of such blocks, slot_stride elements apart, and the block is slab[*slot_dev]
template <typename S>
__global__ void rows_to_bf16_kernel(const S* __restrict__ src, int lds, const long long* __restrict__ idx, uint16_t* __restrict__ dst, int ldd, int cols,
                                    const int* __restrict__ slot_dev, size_t slot_stride) {
    const long long r = blockIdx.x;
    const S* s = src + (size_t)(idx ? idx[r] : r) * lds;
    if (slot_dev) dst += (size_t)(*slot_dev) * slot_stride;
    uint16_t* d = dst + (size_t)r * ldd;
    const bool vec = (lds & 3) == 0 && (ldd & 3) == 0 && (((uintptr_t)src) & (4 * sizeof(S) - 1)) == 0 && (((uintptr_t)dst) & 7) == 0;
    if (vec) {
        const int c4 = cols / 4;
        for (int c = threadIdx.x; c < c4; c += blockDim.x) {
            uint2 o;
            if constexpr (sizeof(S) == 4) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(s) + c);
                o = make_uint2((uint32_t)to_bf16(v.x) | ((uint32_t)to_bf16(v.y) << 16), (uint32_t)to_bf16(v.z) | ((uint32_t)to_bf16(v.w) << 16));
            } else {
                o = __ldg(reinterpret_cast<const uint2*>(s) + c);
            }
            reinterpret_cast<uint2*>(d)[c] = o;
        }
        for (int c = 4 * c4 + threadIdx.x; c < cols; c += blockDim.x) d[c] = to_bf16(s[c]);
    } else {
        for (int c = threadIdx.x; c < cols; c += blockDim.x) d[c] = to_bf16(s[c]);
    }
}

// dst[c][r] = bf16(src[r][c]) through a 32 x 32 shared-memory tile (as go1_transpose)
template <typename S>
__global__ void transpose_bf16_kernel(const S* __restrict__ src, int lds, uint16_t* __restrict__ dst, int ldd, int rows, int cols) {
    __shared__ uint16_t t[32][34];
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        t[i][threadIdx.x] = (r < rows && c < cols) ? to_bf16(src[(size_t)r * lds + c]) : (uint16_t)0;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int c = c0 + i, r = r0 + threadIdx.x;
        if (c < cols && r < rows) dst[(size_t)c * ldd + r] = t[threadIdx.x][i];
    }
}

template <typename S>
int transpose(const S* src, int lds, uint16_t* dst, int ldd, int rows, int cols, void* stream, const char* what) {
    if (!src || !dst || rows <= 0 || cols <= 0 || lds < cols || ldd < rows) return go1_set_error(what);
    dim3 grid((cols + 31) / 32, (rows + 31) / 32);
    if (grid.y > 65535) return go1_set_error(what);
    transpose_bf16_kernel<S><<<grid, dim3(32, 8), 0, (cudaStream_t)stream>>>(src, lds, dst, ldd, rows, cols);
    return launch_rc();
}

int rows_threads(int cols) { return cols >= 1024 ? 256 : (cols >= 128 ? 64 : 32); }

// go1_convert_bf16_segments: a grid-stride loop over work items of four columns each; the items of segment s are
// item0[s] .. item0[s + 1] - 1, row-major over its rows x q[s] = ceil(cols / 4) column quads (one CTA per row left most threads of the
// 128- and 256-wide hidden rows idle and ran ~170K CTAs per minibatch).  vec[s]: 16-byte loads / 8-byte stores where the segment allows.
constexpr int BF16_MAX_SEGS = 16;
struct Bf16Segs { Go1Bf16Seg s[BF16_MAX_SEGS]; long long item0[BF16_MAX_SEGS + 1]; int q[BF16_MAX_SEGS]; int vec[BF16_MAX_SEGS]; int n; };
__global__ void __launch_bounds__(256) segments_to_bf16_kernel(const __grid_constant__ Bf16Segs a) {
    const long long total = a.item0[a.n];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int si = 0;
        while (si + 1 < a.n && i >= a.item0[si + 1]) si++;
        const Go1Bf16Seg& sg = a.s[si];
        const long long j = i - a.item0[si];
        const int r = (int)(j / a.q[si]), c = 4 * (int)(j - (long long)r * a.q[si]);
        const float* src = sg.src + (size_t)r * sg.lds + c;
        uint16_t* dst = sg.dst + (size_t)r * sg.ldd + c;
        if (a.vec[si] && c + 4 <= sg.cols) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(src));
            *reinterpret_cast<uint2*>(dst) = make_uint2((uint32_t)to_bf16(v.x) | ((uint32_t)to_bf16(v.y) << 16), (uint32_t)to_bf16(v.z) | ((uint32_t)to_bf16(v.w) << 16));
        } else {
            for (int k = 0; k < 4 && c + k < sg.cols; k++) dst[k] = to_bf16(src[k]);
        }
    }
}

}  // namespace

extern "C" int go1_convert_bf16(const float* src, int lds, uint16_t* dst, int ldd, int rows, int cols, void* stream) {
    if (!src || !dst || rows <= 0 || cols <= 0 || lds < cols || ldd < cols) return go1_set_error("go1_convert_bf16: bad arguments");
    rows_to_bf16_kernel<float><<<(unsigned)rows, rows_threads(cols), 0, (cudaStream_t)stream>>>(src, lds, nullptr, dst, ldd, cols, nullptr, 0);
    return launch_rc();
}

extern "C" int go1_gather_rows_bf16(const uint16_t* src, int lds, const int64_t* idx, uint16_t* dst, int ldd, int64_t rows, int width, void* stream) {
    if (!src || !idx || !dst || rows <= 0 || width <= 0 || lds < width || ldd < width) return go1_set_error("go1_gather_rows_bf16: bad arguments");
    rows_to_bf16_kernel<uint16_t><<<(unsigned)rows, rows_threads(width), 0, (cudaStream_t)stream>>>(src, lds, (const long long*)idx, dst, ldd, width, nullptr, 0);
    return launch_rc();
}

extern "C" int go1_rollout_store_rows_bf16(const uint16_t* src, int lds, uint16_t* dst_base, int ldd, const int32_t* slot_dev, int rows, int cols, void* stream) {
    if (!src || !dst_base || rows <= 0 || cols <= 0 || lds < cols || ldd < cols) return go1_set_error("go1_rollout_store_rows_bf16: bad arguments");
    rows_to_bf16_kernel<uint16_t><<<(unsigned)rows, rows_threads(cols), 0, (cudaStream_t)stream>>>(src, lds, nullptr, dst_base, ldd, cols, slot_dev,
                                                                                                 (size_t)rows * ldd);
    return launch_rc();
}

extern "C" int go1_transpose_to_bf16(const float* src, int lds, uint16_t* dst, int ldd, int rows, int cols, void* stream) {
    return transpose(src, lds, dst, ldd, rows, cols, stream, "go1_transpose_to_bf16: bad arguments");
}

extern "C" int go1_transpose_bf16(const uint16_t* src, int lds, uint16_t* dst, int ldd, int rows, int cols, void* stream) {
    return transpose(src, lds, dst, ldd, rows, cols, stream, "go1_transpose_bf16: bad arguments");
}

extern "C" int go1_convert_bf16_segments(const Go1Bf16Seg* segs, int n, void* stream) {
    if (!segs || n < 1 || n > BF16_MAX_SEGS) return go1_set_error("go1_convert_bf16_segments: 1..16 segments");
    Bf16Segs a;
    a.n = n;
    long long items = 0;
    for (int i = 0; i < n; i++) {
        const Go1Bf16Seg& sg = segs[i];
        if (!sg.src || !sg.dst || sg.rows <= 0 || sg.cols <= 0 || sg.lds < sg.cols || sg.ldd < sg.cols) return go1_set_error("go1_convert_bf16_segments: bad segment");
        a.s[i] = sg;
        a.q[i] = (sg.cols + 3) / 4;
        a.vec[i] = (sg.lds & 3) == 0 && (sg.ldd & 3) == 0 && (((uintptr_t)sg.src) & 15) == 0 && (((uintptr_t)sg.dst) & 7) == 0;
        a.item0[i] = items;
        items += (long long)sg.rows * a.q[i];
    }
    a.item0[n] = items;
    static int sms = 0;
    if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); if (sms <= 0) sms = 132; }
    const long long want = (items + 255) / 256, cap = 8LL * sms;
    segments_to_bf16_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, (cudaStream_t)stream>>>(a);
    return launch_rc();
}
