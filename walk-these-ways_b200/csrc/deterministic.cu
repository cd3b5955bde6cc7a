// deterministic.cu — the deterministic learner mode (go1_set_deterministic, AC_Args.deterministic): the library-wide switch, the per-stream
// workspace that holds per-CTA partial sums, and the fixed-order reduction that adds them into their targets.
//
// Every reduction site of the learner kernels has a deterministic variant that stores its per-CTA (per split, per 32-row block, per row
// slab) partials to the workspace with plain stores instead of adding them into the target with atomics; det_sum then adds the partials
// of each target element in an order fixed by the launch configuration alone.  No CTA waits for another.
#include <cuda_runtime.h>
#include <stdint.h>
#include <atomic>
#include <mutex>
#include <unordered_map>
#include <vector>
#include "../../include/go1_b200.h"
#include "deterministic.cuh"

extern int go1_set_error(const char* m);
void go1_count_launch(int n);

static std::atomic<int> g_det{0};
extern "C" void go1_set_deterministic(int on) { g_det.store(on ? 1 : 0); }
extern "C" int go1_deterministic(void) { return g_det.load(); }
bool go1_det_on() { return g_det.load() != 0; }

// One buffer per stream: the launches of one stream are ordered, so consecutive entry points reuse it; two streams never share one.
// A buffer that is outgrown stays allocated (a captured CUDA graph may hold its address), so growth doubles.
// The key is the raw stream handle, and a CUDA graph keeps the buffer of the stream it was captured on while it is replayed on another.
// The capture streams of the learner (PPO._act_graphed, Runner's step graph) come from torch's round-robin stream pool, so the same
// handle may later serve eager work, e.g. ActorCritic's update side stream.  That is safe only while those replays and that eager work
// never overlap on the device, as now (rollout and update alternate on the main stream); work that overlaps them needs a stream of its own.
namespace {
struct Ws { void* p = nullptr; size_t bytes = 0; };
std::mutex g_ws_mutex;
std::unordered_map<cudaStream_t, Ws> g_ws;
std::vector<void*> g_ws_retired;
size_t g_ws_total = 0;
}

void* go1_det_workspace(cudaStream_t st, size_t bytes) {
    bytes = (bytes + 255) & ~(size_t)255;
    std::lock_guard<std::mutex> lk(g_ws_mutex);
    Ws& w = g_ws[st];
    if (w.bytes >= bytes) return w.p;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cap) != cudaSuccess || cap != cudaStreamCaptureStatusNone) {
        go1_set_error("deterministic mode: the stream's workspace is too small during CUDA graph capture (run the work once on the capturing stream before capture)");
        return nullptr;
    }
    const size_t want = bytes > 2 * w.bytes ? bytes : 2 * w.bytes;
    void* p = nullptr;
    if (cudaMalloc(&p, want) != cudaSuccess) { cudaGetLastError(); go1_set_error("deterministic mode: workspace allocation failed"); return nullptr; }
    if (w.p) g_ws_retired.push_back(w.p);
    w.p = p; w.bytes = want;
    g_ws_total += want;
    return p;
}
extern "C" int go1_deterministic_reserve(void* stream) {
    size_t most = 0;
    {
        std::lock_guard<std::mutex> lk(g_ws_mutex);
        for (const auto& kv : g_ws) most = kv.second.bytes > most ? kv.second.bytes : most;
    }
    return most == 0 || go1_det_workspace((cudaStream_t)stream, most) ? 0 : 1;
}
extern "C" int64_t go1_deterministic_workspace_bytes(void) {
    std::lock_guard<std::mutex> lk(g_ws_mutex);
    return (int64_t)g_ws_total;
}

// out[r][c] (+)= sum over p of parts[p * pstride + r * ldp + c].  A block covers EPB = 256 / G consecutive elements; thread (g, e) sums
// the parts p = g, g + G, g + 2G, ... in that order, and thread (0, e) adds the G group sums in group order: the order depends on
// (nparts, G) only, and G on the shape only (det_groups).
template <typename T>
__global__ void __launch_bounds__(256) det_sum_kernel(const T* __restrict__ parts, int nparts, long long pstride, long long ldp, T* __restrict__ out, int rows,
                                                      int cols, long long ldo, int accumulate, int G) {
    __shared__ T s[256];
    const int epb = 256 / G, e = threadIdx.x % epb, g = threadIdx.x / epb;
    const long long i = (long long)blockIdx.x * epb + e;
    const bool ok = i < (long long)rows * cols;
    const int r = ok ? (int)(i / cols) : 0, c = ok ? (int)(i - (long long)r * cols) : 0;
    T acc = 0;
    if (ok) {
        const T* p = parts + (size_t)r * ldp + c;
#pragma unroll 4
        for (int q = g; q < nparts; q += G) acc += p[(size_t)q * pstride];
    }
    s[threadIdx.x] = acc;
    __syncthreads();
    if (g == 0 && ok) {
        T t = s[e];
        for (int k = 1; k < G; k++) t += s[k * epb + e];
        T* o = out + (size_t)r * ldo + c;
        *o = accumulate ? *o + t : t;
    }
}

static int det_groups(int nparts, long long elems) {
    if (nparts <= 4) return 1;
    if (elems >= 65536) return 4;
    return nparts >= 256 ? 32 : 8;
}

template <typename T>
static int det_sum_t(const T* parts, int nparts, size_t pstride, long long ldp, T* out, int rows, int cols, long long ldo, int accumulate, cudaStream_t st) {
    const long long elems = (long long)rows * cols;
    if (elems <= 0 || nparts <= 0) return 0;
    const int G = det_groups(nparts, elems);
    const long long blocks = (elems + 256 / G - 1) / (256 / G);
    det_sum_kernel<T><<<(unsigned)blocks, 256, 0, st>>>(parts, nparts, (long long)pstride, ldp, out, rows, cols, ldo, accumulate, G);
    go1_count_launch(1);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : go1_set_error(cudaGetErrorString(e));
}
int go1_det_sum(const float* parts, int nparts, size_t pstride, float* out, int rows, int cols, long long ldo, int accumulate, cudaStream_t st, long long ldp) {
    return det_sum_t<float>(parts, nparts, pstride, ldp > 0 ? ldp : cols, out, rows, cols, ldo, accumulate, st);
}
int go1_det_sum64(const double* parts, int nparts, size_t pstride, double* out, int n, int accumulate, cudaStream_t st) {
    return det_sum_t<double>(parts, nparts, pstride, n, out, 1, n, n, accumulate, st);
}
