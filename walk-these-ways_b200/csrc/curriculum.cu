// curriculum.cu — the command curriculum of LeggedRobot._resample_commands on the device (one CTA per call).
//
// What the reference does on the host for every env that resets or hits the 10 s resample mark
// (legged_robot.py:710-824 + curriculum.py:67-89,135-154) is sequential by construction: a numpy RandomState
// (MT19937) stream per curriculum, weight updates applied success by success, cdf = cumsum(w / w.sum()).  This kernel
// reproduces that arithmetic bit for bit (fp64, numpy's pairwise summation, genrand_res53 doubles, separate mul/add
// instead of fma) so that the rollout never has to stop for a host round trip:
//   A  sort the event list by env id (counting sort through a mark array: ids are unique)
//   B  success test per env (float32 division + compare, as torch does it)
//   C  per category: +0.2 on the successful bins (from the old values), then one neighbour bump per successful env
//   D  category draw per env (splitmix64 stream shared with the host implementation)
//   E  per category: (re)build the cdf if the weights changed, pull 2(1+D) n_i MT words collectively (parallel
//      tempering, 3-phase parallel twist), searchsorted + in-cell uniform
//   F  gait-category remap, binary phases, small-command zeroing, bookkeeping, output
// Host twin: go1_gym/envs/base/legged_robot.py::_resample_commands_host (pinned to the reference by
// tests/test_resample_host.py); tests/test_curriculum_gpu.py pins this kernel to the host twin.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include "go1_layout.h"

void go1_count_launch(int n);

namespace {

constexpr int CT = 1024;
constexpr int S = GO1_EVENT_STRIDE;

struct CurArgs {
    Go1SimBuffers b;
    Go1CurriculumConfig c;
    Go1CurriculumBuffers cb;
    int list, N, grouped;
};

// numpy's DOUBLE_pairwise_sum (contiguous): <8 plain loop, <=128 eight partial sums, else split at n/2 rounded down to
// a multiple of 8 and add the two halves.  The recursion is unrolled over an explicit frame stack (depth log2(n/128)).
__device__ double pairwise_leaf(const double* a, int n) {
    if (n < 8) {
        double r = 0.0;
        for (int i = 0; i < n; i++) r = __dadd_rn(r, a[i]);
        return r;
    }
    double r[8];
    for (int j = 0; j < 8; j++) r[j] = a[j];
    int i = 8;
    for (; i < n - (n % 8); i += 8)
        for (int j = 0; j < 8; j++) r[j] = __dadd_rn(r[j], a[i + j]);
    double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])), __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
    for (; i < n; i++) res = __dadd_rn(res, a[i]);
    return res;
}
__device__ double pairwise_sum(const double* a, int n) {
    struct Frame { int off, n, stage; double left; };
    Frame st[28];
    int sp = 0;
    st[sp++] = {0, n, 0, 0.0};
    double ret = 0.0;
    while (sp > 0) {
        Frame& f = st[sp - 1];
        if (f.n <= 128) { ret = pairwise_leaf(a + f.off, f.n); sp--; continue; }
        int n2 = f.n / 2;
        n2 -= n2 % 8;
        if (f.stage == 0) { f.stage = 1; st[sp++] = {f.off, n2, 0, 0.0}; }
        else if (f.stage == 1) { f.left = ret; f.stage = 2; st[sp++] = {f.off + n2, f.n - n2, 0, 0.0}; }
        else { ret = __dadd_rn(f.left, ret); sp--; }
    }
    return ret;
}

__device__ __forceinline__ double clip01(double x) { return fmin(fmax(x, 0.0), 1.0); }

__device__ __forceinline__ uint32_t mt_temper(uint32_t y) {
    y ^= (y >> 11);
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= (y >> 18);
    return y;
}
__device__ __forceinline__ uint32_t mt_mix(uint32_t u, uint32_t v) {
    const uint32_t y = (u & 0x80000000u) | (v & 0x7fffffffu);
    return (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}
// barrier among `nthr` threads: the whole CTA (id 0, __syncthreads) or one category group (named barrier id > 0)
__device__ __forceinline__ void sync_threads(int bar_id, int nthr) {
    if (bar_id == 0) __syncthreads();
    else asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "r"(nthr) : "memory");
}
// mt19937_gen over key[624] in shared memory, by `nthr` >= 227 threads (tid = 0..nthr-1).  The sequential recurrence
//   key[i] = key[(i + 397) % 624] ^ mix(key[i], key[i + 1])
// only looks 397 ahead / 227 behind, so it splits into three parallel sweeps ([0,227) reads old words only,
// [227,454) reads the new [0,227), [454,623) reads the new [227,396)) plus the last word.
__device__ void mt_twist(uint32_t* key, int tid, int nthr, int bar_id) {
    uint32_t v = 0;
    if (tid < 227) v = key[tid + 397] ^ mt_mix(key[tid], key[tid + 1]);
    sync_threads(bar_id, nthr);
    if (tid < 227) key[tid] = v;
    sync_threads(bar_id, nthr);
    if (tid < 227) v = key[tid] ^ mt_mix(key[tid + 227], key[tid + 228]);          // word tid + 227 in [227, 454)
    sync_threads(bar_id, nthr);
    if (tid < 227) key[tid + 227] = v;
    sync_threads(bar_id, nthr);
    if (tid < 169) v = key[tid + 227] ^ mt_mix(key[tid + 454], key[tid + 455]);    // word tid + 454 in [454, 623)
    sync_threads(bar_id, nthr);
    if (tid < 169) key[tid + 454] = v;
    sync_threads(bar_id, nthr);
    if (tid == 0) key[623] = key[396] ^ mt_mix(key[623], key[0]);
    sync_threads(bar_id, nthr);
}
// out[0..need) = the next `need` tempered words of the stream (uniform control flow across the participating threads)
__device__ void mt_draw(uint32_t* key, int* pos_sh, uint32_t* out, int need, int tid, int nthr, int bar_id) {
    int done = 0;
    while (done < need) {
        int pos = *pos_sh;
        sync_threads(bar_id, nthr);
        if (pos >= 624) {
            mt_twist(key, tid, nthr, bar_id);
            pos = 0;
        }
        const int take = min(624 - pos, need - done);
        for (int i = tid; i < take; i += nthr) out[done + i] = mt_temper(key[pos + i]);
        sync_threads(bar_id, nthr);
        if (tid == 0) *pos_sh = pos + take;
        sync_threads(bar_id, nthr);
        done += take;
    }
}

__device__ __forceinline__ double splitmix_next(uint64_t& st) {
    st += 0x9E3779B97F4A7C15ull;
    uint64_t z = st;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z = z ^ (z >> 31);
    return (double)(z >> 11) * (1.0 / 9007199254740992.0);
}

// numpy remainder for float32 with divisor 1 (npy_divmodf): fmod, then the sign of the result follows the divisor
__device__ __forceinline__ float mod1(float a) {
    float m = fmodf(a, 1.0f);
    if (m != 0.0f) { if (m < 0.0f) m = __fadd_rn(m, 1.0f); }
    else m = 0.0f;
    return m;
}
__device__ __forceinline__ float half_plus_quarter(float x) { return __fadd_rn(__fdiv_rn(x, 2.0f), 0.25f); }
__device__ __forceinline__ float half_minus_quarter_mod1(float x) { return mod1(__fsub_rn(__fdiv_rn(x, 2.0f), 0.25f)); }

__global__ void __launch_bounds__(CT, 1) go1_curriculum_kernel(const CurArgs A) {
    __shared__ uint32_t s_key4[4][624];  // MT19937 words: [0] on the sequential path, one per category group on the grouped path
    __shared__ int s_pos4[4];
    __shared__ int s_scan[CT];           // block scan (sequential path) / four 256-entry index lists (grouped path)
    __shared__ int s_n4[4];
    __shared__ double s_d4[4][2];
    uint32_t* const s_key = s_key4[0];
    int& s_pos = s_pos4[0];
    int& s_n = s_n4[0];
    double* const s_d = s_d4[0];
    const int t = threadIdx.x;
    const int N = A.N;
    const Go1CurriculumConfig& c = A.c;
    const Go1CurriculumBuffers& cb = A.cb;
    const int L = c.num_bins, D = c.num_dims, ncat = c.num_categories, nc = c.num_commands;
    // cross-rank replay: the records of every rank (gathered), walked in ascending GLOBAL id; NT = envs of all ranks
    const bool xr = c.xr_world > 1;
    const int NT = xr ? N * c.xr_world : N;
    __shared__ int s_xcnt[GO1_CUR_MAX_CATEGORIES + 2];          // exclusive prefix of the per-rank record counts (xr_world <= 8)
    const size_t xr_block = 1 + (size_t)c.xr_cap * GO1_XR_STRIDE;
    if (xr) {
        if (t == 0) {
            int acc = 0;
            for (int r = 0; r < c.xr_world; r++) { s_xcnt[r] = acc; acc += (int)cb.xr_events[((size_t)r * 2 + A.list) * xr_block]; }
            s_xcnt[c.xr_world] = acc;
        }
        __syncthreads();
    }
    const int n = xr ? s_xcnt[c.xr_world] : A.b.event_count[A.list];
    if (t == 0 && A.list == 0) cb.out_count[0] = xr ? 0 : n;
    if (n <= 0) return;
    const float* ev = A.b.events + (size_t)A.list * N * S;
    // record i of the (unsorted) list: [env id, 4 task command sums, ep_len (, old bin, old category when gathered)]
    auto rec = [&](int i) -> const float* {
        if (!xr) return ev + (size_t)i * S;
        int r = 0;
        while (i >= s_xcnt[r + 1]) r++;
        return cb.xr_events + ((size_t)r * 2 + A.list) * xr_block + 1 + (size_t)(i - s_xcnt[r]) * GO1_XR_STRIDE;
    };
    int* const w_ids = xr ? cb.xr_ids : cb.out_ids;              // working lists: global ids / commands of all n records
    float* const w_cmd = xr ? cb.xr_commands : cb.out_commands;

    // the usual call handles a handful of envs: then every per-env array lives in shared memory and the index lists are
    // built by counting predecessors in parallel; the global-scratch path (n > SMALL) keeps the simple serial builders
    constexpr int SMALL = 512;
    __shared__ int s_arr[7][SMALL];
    __shared__ double s_cdf4[4][512];    // cdf staging: flat [2048] on the sequential path, one row per category group otherwise
    double* const s_cdf = &s_cdf4[0][0];
    const bool small = n <= SMALL;
    int* mark = cb.scratch_i32;          // [NT], all zero between calls
    int* order = small ? s_arr[0] : mark + NT;               // [n] event slot of the p-th smallest env id
    int* a_cat_old = small ? s_arr[1] : mark + 2 * (size_t)NT;
    int* a_bin_old = small ? s_arr[2] : mark + 3 * (size_t)NT;
    int* a_ok = small ? s_arr[3] : mark + 4 * (size_t)NT;
    int* a_cat_new = small ? s_arr[4] : mark + 5 * (size_t)NT;
    int* a_bin_new = small ? s_arr[5] : mark + 6 * (size_t)NT;
    int* a_list = small ? s_arr[6] : mark + 7 * (size_t)NT;  // [n] per-phase index list (successful bins / category members)
    double* dd = cb.scratch_f64;         // [(D + 1) NT] doubles of the current category
    double* r2 = dd + (size_t)(D + 1) * NT;   // [NT] second category draw (exclusive / balanced gait modes)

    // =============================================================================================================
    // Grouped path (the usual call: a handful of envs).  The categories are independent -- own weights, own cdf, own
    // RandomState -- so phases C and E run for all of them at once, one 256-thread group per category with a named
    // barrier, instead of one category after the other; everything lives in shared memory.  Same arithmetic, same order
    // inside every category, hence the same bits (tests/test_curriculum_gpu.py runs both paths).
    // =============================================================================================================
    constexpr int GS = 256, NSM = 256;
    if (A.grouped && !xr && n <= NSM && ncat <= 4 && L <= 512) {      // scratch: >= 4 x 2(D+1) x 256 words and 4 x (D+1) x 256 doubles (curriculum_dev.py)
        const int g = t / GS, gt = t % GS, bar = 1 + g;
        int* ord = s_arr[0]; int* cat_old = s_arr[1]; int* bin_old = s_arr[2]; int* okf = s_arr[3];
        int* cat_new = s_arr[4]; int* bin_new = s_arr[5]; int* ids = s_arr[6];
        int* glist = s_scan + g * NSM;                      // this group's index list
        // A: rank sort of the (unique) ids
        if (t < n) ids[t] = (int)ev[(size_t)t * S];
        __syncthreads();
        if (t < n) {
            const int me = ids[t];
            int rank = 0;
            for (int q = 0; q < n; q++) rank += ids[q] < me;
            ord[rank] = t;
        }
        __syncthreads();
        // B: success test, old bin / category
        if (t < n) {
            const float* e = ev + (size_t)ord[t] * S;
            const int id = (int)e[0];
            bool ok = c.num_task_keys > 0;
            for (int q = 0; q < c.num_task_keys; q++) ok = ok && (__fdiv_rn(e[1 + c.task_col[q]], c.ep_len) > c.threshold[q]);
            cb.out_ids[t] = id;
            okf[t] = ok ? 1 : 0;
            cat_old[t] = cb.env_categories[id];
            bin_old[t] = cb.env_bins[id];
        }
        __syncthreads();
        // C: curriculum update of category g by group g
        if (g < ncat) {
            if (gt == 0) s_n4[g] = 0;
            sync_threads(bar, GS);
            if (gt < n && okf[gt] && cat_old[gt] == g) {
                int pos = 0;
                for (int q = 0; q < gt; q++) pos += (okf[q] && cat_old[q] == g);
                glist[pos] = bin_old[gt];
                atomicAdd(&s_n4[g], 1);
            }
            sync_threads(bar, GS);
            const int ns = s_n4[g];
            if (ns > 0) {
                double* w = cb.weights + (size_t)g * L;
                double nv = 0.0;
                if (gt < ns) nv = clip01(__dadd_rn(w[glist[gt]], 0.2));                 // from the OLD weights
                sync_threads(bar, GS);
                if (gt < ns) w[glist[gt]] = nv;
                sync_threads(bar, GS);
                for (int sidx = 0; sidx < ns; sidx++) {
                    const int bsel = glist[sidx];
                    for (int j = gt; j < L; j += GS) {
                        bool adj = true;
                        for (int d = 0; d < D; d++) {
                            const double gg = cb.grid[(size_t)j * D + d], ce = cb.grid[(size_t)bsel * D + d], r = cb.local_range[d];
                            adj = adj && (gg >= __dsub_rn(ce, r)) && (gg <= __dadd_rn(ce, r));
                        }
                        if (adj) w[j] = clip01(__dadd_rn(w[j], 0.2));
                    }
                    sync_threads(bar, GS);
                }
                if (gt == 0) cb.cdf_valid[g] = 0;
            }
        }
        __syncthreads();
        // D: new categories (one splitmix64 stream, env order)
        if (t == 0) {
            uint64_t st = cb.cat_rng[0];
            const bool pow2 = (ncat & (ncat - 1)) == 0;
            const double pc = 1.0 / (double)ncat;
            for (int p = 0; p < n; p++) {
                const double r = splitmix_next(st);
                int cat = -1;
                if (pow2) cat = (int)(r * (double)ncat);
                else
                    for (int i = 0; i < ncat; i++)
                        if (pc * i <= r && r < pc * (i + 1)) cat = i;
                cat_new[p] = cat;
                bin_new[p] = bin_old[p];
            }
            cb.cat_rng[0] = st;
        }
        if (t < n)
            for (int d = 0; d < GO1_NUM_COMMANDS; d++) cb.out_commands[(size_t)t * GO1_NUM_COMMANDS + d] = 0.0f;
        __syncthreads();
        // E: category g's members sampled by group g
        if (g < ncat) {
            if (gt == 0) s_n4[g] = 0;
            sync_threads(bar, GS);
            if (gt < n && cat_new[gt] == g) {
                int pos = 0;
                for (int q = 0; q < gt; q++) pos += cat_new[q] == g;
                glist[pos] = gt;
                atomicAdd(&s_n4[g], 1);
            }
            sync_threads(bar, GS);
            const int ni = s_n4[g];
            if (ni > 0) {
                double* w = cb.weights + (size_t)g * L;
                double* cdf = cb.cdf + (size_t)g * L;
                if (!cb.cdf_valid[g]) {
                    if (gt == 0) s_d4[g][0] = __dadd_rn(0.0, pairwise_sum(w, L));
                    sync_threads(bar, GS);
                    const double tot = s_d4[g][0];
                    for (int j = gt; j < L; j += GS) cdf[j] = __ddiv_rn(w[j], tot);
                    sync_threads(bar, GS);
                    if (gt == 0) {
                        double acc = cdf[0];
                        for (int j = 1; j < L; j++) { acc = __dadd_rn(acc, cdf[j]); cdf[j] = acc; }
                        s_d4[g][1] = acc;
                    }
                    sync_threads(bar, GS);
                    const double last = s_d4[g][1];
                    for (int j = gt; j < L; j += GS) cdf[j] = __ddiv_rn(cdf[j], last);
                    sync_threads(bar, GS);
                    if (gt == 0) cb.cdf_valid[g] = 1;
                }
                uint32_t* mt = cb.mt + (size_t)g * 625;
                uint32_t* key = s_key4[g];
                double* cdf_s = s_cdf4[g];
                for (int j = gt; j < 624; j += GS) key[j] = mt[j];
                if (gt == 0) s_pos4[g] = (int)mt[624];
                for (int j = gt; j < L; j += GS) cdf_s[j] = cdf[j];
                sync_threads(bar, GS);
                const int nd = (D + 1) * ni;
                uint32_t* words = cb.scratch_u32 + (size_t)g * 2 * (D + 1) * NSM;
                double* ddg = dd + (size_t)g * (D + 1) * NSM;
                mt_draw(key, &s_pos4[g], words, 2 * nd, gt, GS, bar);
                for (int j = gt; j < 624; j += GS) mt[j] = key[j];
                if (gt == 0) mt[624] = (uint32_t)s_pos4[g];
                for (int q = gt; q < nd; q += GS) {
                    const uint32_t a = words[2 * q] >> 5, bb = words[2 * q + 1] >> 6;
                    ddg[q] = __ddiv_rn(__dadd_rn(__dmul_rn((double)a, 67108864.0), (double)bb), 9007199254740992.0);
                }
                sync_threads(bar, GS);
                if (gt < ni) {
                    const int p = glist[gt];
                    const double u = ddg[gt];
                    int lo = 0, hi = L;
                    while (lo < hi) {
                        const int mid = (lo + hi) >> 1;
                        if (cdf_s[mid] <= u) lo = mid + 1; else hi = mid;
                    }
                    const int idx = min(lo, L - 1);
                    bin_new[p] = idx;
                    for (int d = 0; d < D; d++) {
                        const double ce = cb.grid[(size_t)idx * D + d];
                        const double lo_ = __dadd_rn(ce, cb.half_bins[d]), hi_ = __dsub_rn(ce, cb.half_bins[d]);
                        const double val = __dadd_rn(lo_, __dmul_rn(__dsub_rn(hi_, lo_), ddg[ni + (size_t)gt * D + d]));
                        if (d < nc && d < GO1_NUM_COMMANDS) cb.out_commands[(size_t)p * GO1_NUM_COMMANDS + d] = __double2float_rn(val);
                    }
                }
            }
        }
        __syncthreads();
        // hand over to the common tail (second category draw, phase F) with the arrays it expects
        order = ord; a_cat_old = cat_old; a_bin_old = bin_old; a_ok = okf; a_cat_new = cat_new; a_bin_new = bin_new;
        goto tail;
    }

    // ---- A: ascending env order --------------------------------------------------------------------------------
    if (small) {             // rank of every id among the n ids (ids are unique)
        int* ids = a_list;
        for (int i = t; i < n; i += CT) ids[i] = (int)rec(i)[0];
        __syncthreads();
        for (int i = t; i < n; i += CT) {
            const int me = ids[i];
            int rank = 0;
            for (int q = 0; q < n; q++) rank += ids[q] < me;
            order[rank] = i;
        }
    } else {
    for (int i = t; i < n; i += CT) mark[(int)rec(i)[0]] = i + 1;
    __syncthreads();
    {
        const int chunk = (NT + CT - 1) / CT;
        const int lo = min(t * chunk, NT), hi = min(lo + chunk, NT);
        int cnt = 0;
        for (int e = lo; e < hi; e++) cnt += mark[e] != 0;
        s_scan[t] = cnt;
        __syncthreads();
        for (int off = 1; off < CT; off <<= 1) {        // inclusive Hillis-Steele scan
            const int v = (t >= off) ? s_scan[t - off] : 0;
            __syncthreads();
            s_scan[t] += v;
            __syncthreads();
        }
        int base = s_scan[t] - cnt;
        for (int e = lo; e < hi; e++)
            if (mark[e]) { order[base++] = mark[e] - 1; mark[e] = 0; }
    }
    }
    __syncthreads();

    // ---- B: success test (legged_robot.py:727-732; curriculum.py:136-139), old bin / category ---------------------
    for (int p = t; p < n; p += CT) {
        const float* e = rec(order[p]);
        const int id = (int)e[0];
        bool ok = c.num_task_keys > 0;
        for (int q = 0; q < c.num_task_keys; q++) ok = ok && (__fdiv_rn(e[1 + c.task_col[q]], c.ep_len) > c.threshold[q]);
        w_ids[p] = id;
        a_ok[p] = ok ? 1 : 0;
        a_cat_old[p] = xr ? (int)e[7] : cb.env_categories[id];      // gathered records carry the owner's bin / category
        a_bin_old[p] = xr ? (int)e[6] : cb.env_bins[id];
    }
    __syncthreads();

    // ---- C: curriculum update, category by category (curriculum.py:141-154) --------------------------------------
    for (int i = 0; i < ncat; i++) {
        if (small) {            // position = number of earlier successes of this category
            if (t == 0) s_n = 0;
            __syncthreads();
            for (int p = t; p < n; p += CT)
                if (a_ok[p] && a_cat_old[p] == i) {
                    int pos = 0;
                    for (int q = 0; q < p; q++) pos += (a_ok[q] && a_cat_old[q] == i);
                    a_list[pos] = a_bin_old[p];
                    atomicAdd(&s_n, 1);
                }
        } else if (t == 0) {
            int ns = 0;
            for (int p = 0; p < n; p++)
                if (a_ok[p] && a_cat_old[p] == i) a_list[ns++] = a_bin_old[p];
            s_n = ns;
        }
        __syncthreads();
        const int ns = s_n;
        if (ns > 0) {
            double* w = cb.weights + (size_t)i * L;
            for (int s = t; s < ns; s += CT) dd[s] = clip01(__dadd_rn(w[a_list[s]], 0.2));     // from the OLD weights
            __syncthreads();
            for (int s = t; s < ns; s += CT) w[a_list[s]] = dd[s];
            __syncthreads();
            for (int s = 0; s < ns; s++) {
                const int bsel = a_list[s];
                for (int j = t; j < L; j += CT) {
                    bool adj = true;
                    for (int d = 0; d < D; d++) {
                        const double g = cb.grid[(size_t)j * D + d], ce = cb.grid[(size_t)bsel * D + d], r = cb.local_range[d];
                        adj = adj && (g >= __dsub_rn(ce, r)) && (g <= __dadd_rn(ce, r));
                    }
                    if (adj) w[j] = clip01(__dadd_rn(w[j], 0.2));
                }
                __syncthreads();
            }
            if (t == 0) cb.cdf_valid[i] = 0;
        }
        __syncthreads();
    }

    // ---- D: new categories (legged_robot.py:742-746) -----------------------------------------------------------------
    if (t == 0) {
        uint64_t st = cb.cat_rng[0];
        const bool pow2 = (ncat & (ncat - 1)) == 0;
        const double pc = 1.0 / (double)ncat;
        for (int p = 0; p < n; p++) {
            const double r = splitmix_next(st);
            int cat = -1;
            if (pow2) cat = (int)(r * (double)ncat);
            else
                for (int i = 0; i < ncat; i++)
                    if (pc * i <= r && r < pc * (i + 1)) cat = i;
            a_cat_new[p] = cat;
            a_bin_new[p] = a_bin_old[p];
        }
        cb.cat_rng[0] = st;
    }
    __syncthreads();
    for (int p = t; p < n; p += CT)
        for (int d = 0; d < GO1_NUM_COMMANDS; d++) w_cmd[(size_t)p * GO1_NUM_COMMANDS + d] = 0.0f;
    __syncthreads();

    // ---- E: sample each category's members from its curriculum (curriculum.py:67-89) ---------------------------------
    for (int i = 0; i < ncat; i++) {
        if (small) {
            if (t == 0) s_n = 0;
            __syncthreads();
            for (int p = t; p < n; p += CT)
                if (a_cat_new[p] == i) {
                    int pos = 0;
                    for (int q = 0; q < p; q++) pos += a_cat_new[q] == i;
                    a_list[pos] = p;
                    atomicAdd(&s_n, 1);
                }
        } else if (t == 0) {
            int ni = 0;
            for (int p = 0; p < n; p++)
                if (a_cat_new[p] == i) a_list[ni++] = p;
            s_n = ni;
        }
        __syncthreads();
        const int ni = s_n;
        if (ni == 0) { __syncthreads(); continue; }
        double* w = cb.weights + (size_t)i * L;
        double* cdf = cb.cdf + (size_t)i * L;
        if (!cb.cdf_valid[i]) {                 // p = w / w.sum(); cdf = p.cumsum(); cdf /= cdf[-1]
            if (t == 0) s_d[0] = __dadd_rn(0.0, pairwise_sum(w, L));
            __syncthreads();
            const double tot = s_d[0];
            for (int j = t; j < L; j += CT) cdf[j] = __ddiv_rn(w[j], tot);
            __syncthreads();
            if (t == 0) {
                double acc = cdf[0];
                for (int j = 1; j < L; j++) { acc = __dadd_rn(acc, cdf[j]); cdf[j] = acc; }
                s_d[1] = acc;
            }
            __syncthreads();
            const double last = s_d[1];
            for (int j = t; j < L; j += CT) cdf[j] = __ddiv_rn(cdf[j], last);
            __syncthreads();
            if (t == 0) cb.cdf_valid[i] = 1;
        }
        // the RandomState stream: ni doubles for the bins, then ni x D for the in-cell positions (C order)
        uint32_t* mt = cb.mt + (size_t)i * 625;
        for (int j = t; j < 624; j += CT) s_key[j] = mt[j];
        if (t == 0) s_pos = (int)mt[624];
        __syncthreads();
        const int nd = (D + 1) * ni;
        mt_draw(s_key, &s_pos, cb.scratch_u32, 2 * nd, t, CT, 0);
        for (int j = t; j < 624; j += CT) mt[j] = s_key[j];
        if (t == 0) mt[624] = (uint32_t)s_pos;
        for (int q = t; q < nd; q += CT) {
            const uint32_t a = cb.scratch_u32[2 * q] >> 5, bb = cb.scratch_u32[2 * q + 1] >> 6;
            dd[q] = __ddiv_rn(__dadd_rn(__dmul_rn((double)a, 67108864.0), (double)bb), 9007199254740992.0);
        }
        const double* cdf_s = cdf;
        if (L <= 1024) {
            for (int j = t; j < L; j += CT) s_cdf[j] = cdf[j];
            cdf_s = s_cdf;
        }
        __syncthreads();
        for (int m = t; m < ni; m += CT) {
            const int p = a_list[m];
            const double u = dd[m];
            int lo = 0, hi = L;                 // searchsorted(cdf, u, side='right')
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (cdf_s[mid] <= u) lo = mid + 1; else hi = mid;
            }
            const int idx = min(lo, L - 1);
            a_bin_new[p] = idx;
            for (int d = 0; d < D; d++) {
                const double ce = cb.grid[(size_t)idx * D + d];
                const double lo_ = __dadd_rn(ce, cb.half_bins[d]), hi_ = __dsub_rn(ce, cb.half_bins[d]);
                const double val = __dadd_rn(lo_, __dmul_rn(__dsub_rn(hi_, lo_), dd[ni + (size_t)m * D + d]));
                if (d < nc && d < GO1_NUM_COMMANDS) w_cmd[(size_t)p * GO1_NUM_COMMANDS + d] = __double2float_rn(val);
            }
        }
        __syncthreads();
    }

tail:
    // second category draw of the two non-gaitwise gait modes (legged_robot.py:783, 795)
    const bool need_r2 = nc > 5 && !c.gaitwise_curricula && (c.exclusive_phase_offset || c.balance_gait_distribution);
    if (need_r2) {
        if (t == 0) {
            uint64_t st = cb.cat_rng[0];
            for (int p = 0; p < n; p++) r2[p] = splitmix_next(st);
            cb.cat_rng[0] = st;
        }
        __syncthreads();
    }

    // ---- F: gait remap (legged_robot.py:762-817), small-command zeroing (:820), bookkeeping, output ---------------------
    for (int p = t; p < n; p += CT) {
        float* cm = w_cmd + (size_t)p * GO1_NUM_COMMANDS;
        const int id = xr ? w_ids[p] - c.xr_rank * N : w_ids[p];       // local env id; other ranks' envs fall outside [0, N)
        const bool mine = id >= 0 && id < N;
        const int cat = a_cat_new[p];
        if (nc > 5) {
            if (c.gaitwise_curricula) {
                const int kind = cat >= 0 ? c.category_kind[cat] : 0;
                if (kind == 1) { for (int j = 5; j < 8; j++) cm[j] = half_minus_quarter_mod1(cm[j]); }
                else if (kind == 2) { cm[5] = half_plus_quarter(cm[5]); cm[6] = 0.f; cm[7] = 0.f; }
                else if (kind == 3) { cm[6] = half_plus_quarter(cm[6]); cm[5] = 0.f; cm[7] = 0.f; }
                else if (kind == 4) { cm[7] = half_plus_quarter(cm[7]); cm[5] = 0.f; cm[6] = 0.f; }
            } else if (c.exclusive_phase_offset) {
                const double r = r2[p];
                const bool trot = r < 0.34, pace = 0.34 <= r && r < 0.67, bound = 0.67 <= r;
                if (pace || bound) cm[5] = 0.f;
                if (trot || bound) cm[6] = 0.f;
                if (trot || pace) cm[7] = 0.f;
            } else if (c.balance_gait_distribution) {
                const double r = r2[p];
                const bool pronk = r <= 0.25, trot = 0.25 <= r && r < 0.50, pace = 0.50 <= r && r < 0.75, bound = 0.75 <= r;
                if (pronk) for (int j = 5; j < 8; j++) cm[j] = half_minus_quarter_mod1(cm[j]);
                if (trot) { cm[6] = 0.f; cm[7] = 0.f; }
                if (pace) { cm[5] = 0.f; cm[7] = 0.f; }
                if (bound) { cm[5] = 0.f; cm[6] = 0.f; }
                if (trot) cm[5] = half_plus_quarter(cm[5]);
                if (pace) cm[6] = half_plus_quarter(cm[6]);
                if (bound) cm[7] = half_plus_quarter(cm[7]);
            }
            if (c.binary_phases)
                for (int j = 5; j < 8; j++) cm[j] = mod1(__fdiv_rn(rintf(__fmul_rn(2.0f, cm[j])), 2.0f));
        }
        const float nrm = __fsqrt_rn(__fadd_rn(__fmul_rn(cm[0], cm[0]), __fmul_rn(cm[1], cm[1])));
        const float keep = nrm > 0.2f ? 1.0f : 0.0f;
        cm[0] = __fmul_rn(cm[0], keep); cm[1] = __fmul_rn(cm[1], keep);
        if (mine && cat >= 0) { cb.env_bins[id] = a_bin_new[p]; cb.env_categories[id] = cat; }
        if (mine && A.list == 1) {      // periodic resample: commands take effect here (go1_sim_set_commands)
            for (int d = 0; d < GO1_NUM_COMMANDS; d++) A.b.env_f32[(size_t)(EROW(commands) + d) * N + id] = cm[d];
            for (int d = 0; d < GO1_NUM_COMMAND_SUMS; d++) A.b.env_f32[(size_t)(EROW(command_sums) + d) * N + id] = 0.f;
        }
    }
    // cross-rank replay: hand this rank's envs (a contiguous run of the sorted list) to the reset kernel as local ids + commands
    if (xr && A.list == 0) {
        __shared__ int s_before, s_mine;
        if (t == 0) { s_before = 0; s_mine = 0; }
        __syncthreads();
        const int g0 = c.xr_rank * N;
        int before = 0, mine_cnt = 0;
        for (int p = t; p < n; p += CT) { before += w_ids[p] < g0; mine_cnt += (w_ids[p] >= g0 && w_ids[p] < g0 + N); }
        if (before) atomicAdd(&s_before, before);
        if (mine_cnt) atomicAdd(&s_mine, mine_cnt);
        __syncthreads();
        const int p0 = s_before, k = s_mine;
        for (int q = t; q < k; q += CT) {
            cb.out_ids[q] = w_ids[p0 + q] - g0;
            for (int d = 0; d < GO1_NUM_COMMANDS; d++) cb.out_commands[(size_t)q * GO1_NUM_COMMANDS + d] = w_cmd[(size_t)(p0 + q) * GO1_NUM_COMMANDS + d];
        }
        if (t == 0) cb.out_count[0] = k;
    }
    // extras["env_bins"] / extras["time_outs"] are snapshots taken inside reset_idx (legged_robot.py:231-234): refreshed
    // only by a step in which some env reset, and then for ALL train envs
    if (A.list == 0) {
        __syncthreads();
        for (int e = t; e < c.num_train_envs; e += CT) {
            cb.env_bins_f32[e] = (float)cb.env_bins[e];
            if (c.snapshot_time_outs) cb.time_outs_snapshot[e] = A.b.time_out[e];
        }
    }
}

// cross-rank replay: this rank's two event lists with global ids and the envs' current bins / categories
__global__ void go1_curriculum_pack_kernel(const Go1SimBuffers b, const Go1CurriculumConfig c, const Go1CurriculumBuffers cb, int N) {
    const int list = blockIdx.y;
    const int n = b.event_count[list];
    float* out = cb.xr_send + (size_t)list * (1 + (size_t)c.xr_cap * GO1_XR_STRIDE);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) out[0] = (float)n;
    if (i >= n || i >= c.xr_cap) return;
    const float* e = b.events + ((size_t)list * N + i) * S;
    const int id = (int)e[0];
    float* o = out + 1 + (size_t)i * GO1_XR_STRIDE;
    o[0] = (float)(c.xr_rank * N + id);
    for (int k = 1; k < S; k++) o[k] = e[k];
    o[6] = (float)cb.env_bins[id];
    o[7] = (float)cb.env_categories[id];
}

}  // namespace

extern "C" int go1_launch_curriculum_pack(const Go1SimBuffers* b, const Go1CurriculumConfig* cfg, const Go1CurriculumBuffers* cb, int N, cudaStream_t st) {
    dim3 grid((N + 255) / 256, 2);
    go1_curriculum_pack_kernel<<<grid, 256, 0, st>>>(*b, *cfg, *cb, N);
    go1_count_launch(1);
    return (int)cudaGetLastError();
}

// The category-parallel grouped path is ON by default (bit-exact against the host twin in all four curriculum modes:
// tests/test_curriculum_gpu.py::test_grouped_path_matches_host_twin); GO1_CUR_GROUPED=0 or
// go1_curriculum_set_grouped(0) select the category-by-category path.
static int g_cur_grouped = -1;
extern "C" void go1_curriculum_set_grouped(int on) { g_cur_grouped = on ? 1 : 0; }

extern "C" int go1_launch_curriculum(const Go1SimBuffers* b, const Go1CurriculumConfig* cfg, const Go1CurriculumBuffers* cb, int list, int N,
                                     cudaStream_t st) {
    CurArgs a;
    a.b = *b; a.c = *cfg; a.cb = *cb; a.list = list; a.N = N;
    a.grouped = g_cur_grouped < 0 ? (g_cur_grouped = getenv("GO1_CUR_GROUPED") ? atoi(getenv("GO1_CUR_GROUPED")) : 1) : g_cur_grouped;
    go1_curriculum_kernel<<<1, CT, 0, st>>>(a);
    go1_count_launch(1);
    return (int)cudaGetLastError();
}
