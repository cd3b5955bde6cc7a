// deterministic.cuh — the deterministic learner mode inside the library (deterministic.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

// the library-wide mode (go1_set_deterministic), read by every learner entry point at launch
bool go1_det_on();
// `bytes` of workspace private to stream st, valid until the next call for st; nullptr (error set) if it would have to grow during capture
void* go1_det_workspace(cudaStream_t st, size_t bytes);
// where a reduction site's kernel puts its per-CTA sums: with det, `count` Ts of st's workspace (nullptr, error set, if it cannot be had);
// else `dflt` (the target the kernel adds into, or nullptr for a kernel that takes its partials beside the target)
template <typename T>
T* go1_det_out(bool det, cudaStream_t st, size_t count, T* dflt) {
    return det ? static_cast<T*>(go1_det_workspace(st, sizeof(T) * count)) : dflt;
}
// out[r * ldo + c] = (accumulate ? out[r * ldo + c] : 0) + the sum over p < nparts of parts[p * pstride + r * ldp + c] (ldp 0: cols), in an
// order fixed by (nparts, rows, cols)
int go1_det_sum(const float* parts, int nparts, size_t pstride, float* out, int rows, int cols, long long ldo, int accumulate, cudaStream_t st, long long ldp = 0);
// the same over n doubles (rows = 1)
int go1_det_sum64(const double* parts, int nparts, size_t pstride, double* out, int n, int accumulate, cudaStream_t st);
