// residual_resample (filterpy/monte_carlo/resampling.py:27-76) on the device, bit for bit.
//
//   num_copies = floor(N * w).astype(int)                 :57   -> k_counts / k_scan_counts / k_expand
//   indexes[0:k] = repeat(arange(N), num_copies)          :58-62
//   residual = w - num_copies                             :69   (NOT N*w - num_copies: negative for every
//   residual /= sum(residual)                             :70    particle with a copy, so the cumulative sum
//   cumulative_sum = np.cumsum(residual); [-1] = 1.       :71-72 below is not monotone)
//   indexes[k:N] = np.searchsorted(cumulative_sum, random(N - k))   :74
//
// Two pieces are order-dependent and are reproduced in the reference's order:
//  * `sum(residual)` (the Python builtin: 0 + r0 + r1 + ..., one fp64 add at a time) and `np.cumsum` of
//    a MIXED-SIGN array: the parity-map scan of resample.cu needs non-negative terms, so one warp walks
//    the array (k_residual_seq): all lanes form the residuals of the next 1024 particles while lane 0
//    runs the dependent adds out of shared memory (one DADD per particle on the critical path).
//  * np.searchsorted on a non-monotone array: NumPy's bisection (npy_binsearch, side='left') carries its
//    bracket from key to key — key i starts from [r[i-1], N) if key[i-1] < key[i], else from
//    [0, r[i-1] + 1) — so the answer for key i depends on the answer for key i-1.  The state carried is
//    the single integer r[i-1], hence r is the fixed point of r[i] = search(key[i]; bracket(r[i-1])) with
//    r[0] searched over [0, N).  k_bisect_sweep evaluates that map for every key in parallel from the
//    previous sweep's values; after t sweeps the first t+1 answers are final, and a sweep that changes
//    nothing proves the whole array (the brackets only differ where the array is locally non-monotone,
//    so two or three sweeps are typical).  The host repeats sweeps until `changed` stays 0.
#include "residual_rules.cuh"

namespace bke {
namespace rr {

constexpr int RB = 256;                 // threads per CTA
constexpr int RIPT = 8;                 // particles per thread
constexpr int RTILE = RB * RIPT;        // 2048 particles per tile
constexpr int SEQ_CHUNK = 1024;         // particles per step of the sequential warp (32 per lane)

struct RWs {
    i64 *tile_cnt;      // [T] copies made by the tile
    i64 *tile_off;      // [T] exclusive prefix of tile_cnt
    int T;
};

__host__ __device__ inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

static size_t ws_bytes(i64 n)
{
    const i64 T = (n + RTILE - 1) / RTILE;
    return 2 * align256((size_t)(T > 0 ? T : 1) * sizeof(i64)) + 256;
}

static void carve(i64 n, unsigned char *base, RWs *ws)
{
    const i64 T = (n + RTILE - 1) / RTILE;
    unsigned char *p = base + ((256 - (reinterpret_cast<uintptr_t>(base) & 255)) & 255);
    ws->tile_cnt = reinterpret_cast<i64 *>(p); p += align256((size_t)(T > 0 ? T : 1) * sizeof(i64));
    ws->tile_off = reinterpret_cast<i64 *>(p);
    ws->T = (int)T;
}

__device__ __forceinline__ i64 block_sum_i64(i64 v, i64 *sh)
{
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(FULL, v, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    i64 t = 0;
    for (int i = 0; i < RB / 32; i++) t += sh[i];
    __syncthreads();
    return t;
}

__global__ void __launch_bounds__(RB) k_counts(i64 n, const double *__restrict__ w, RWs ws)
{
    __shared__ i64 sh[RB / 32];
    const double Nd = (double)n;
    for (int t = blockIdx.x; t < ws.T; t += gridDim.x) {
        const i64 base = (i64)t * RTILE;
        i64 c = 0;
#pragma unroll
        for (int i = 0; i < RIPT; i++) {
            const i64 j = base + i * RB + threadIdx.x;
            if (j < n) c += copies_made(Nd, w[j]);
        }
        const i64 tot = block_sum_i64(c, sh);
        if (threadIdx.x == 0) ws.tile_cnt[t] = tot;
    }
}

// exclusive scan of the tile counts, one CTA (integer sums: any order is exact)
__global__ void __launch_bounds__(1024) k_scan_counts(RWs ws, i64 *k_out)
{
    __shared__ i64 wtot[32];
    __shared__ i64 carry_sh;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) carry_sh = 0;
    __syncthreads();
    for (int b = 0; b < ws.T; b += 1024) {
        const int t = b + tid;
        const i64 v = t < ws.T ? ws.tile_cnt[t] : 0;
        i64 inc = v;
        for (int o = 1; o < 32; o <<= 1) { const i64 y = __shfl_up_sync(FULL, inc, o); if (lane >= o) inc += y; }
        if (lane == 31) wtot[wid] = inc;
        __syncthreads();
        i64 ex = inc - v, all = 0;
        for (int i = 0; i < 32; i++) { const i64 x = wtot[i]; if (i < wid) ex += x; all += x; }
        const i64 carry = carry_sh;
        if (t < ws.T) ws.tile_off[t] = carry + ex;
        __syncthreads();
        if (tid == 0) carry_sh = carry + all;
        __syncthreads();
    }
    if (tid == 0) *k_out = carry_sh;
}

// indexes[off + q] = the particle that owns the q-th copy of the tile (resampling.py:58-62)
__global__ void __launch_bounds__(RB) k_expand(i64 n, const double *__restrict__ w, RWs ws, int *__restrict__ idx)
{
    __shared__ i64 pre[RTILE];          // inclusive prefix of the copies inside the tile
    __shared__ i64 wtot[RB / 32];
    const double Nd = (double)n;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int t = blockIdx.x; t < ws.T; t += gridDim.x) {
        const i64 cnt = ws.tile_cnt[t];
        if (cnt == 0) continue;                         // uniform over the CTA
        const i64 base = (i64)t * RTILE, off = ws.tile_off[t];
        i64 c[RIPT], acc = 0;
#pragma unroll
        for (int i = 0; i < RIPT; i++) {
            const i64 j = base + tid * RIPT + i;
            acc += (j < n) ? copies_made(Nd, w[j]) : 0;
            c[i] = acc;
        }
        i64 inc = acc;
        for (int o = 1; o < 32; o <<= 1) { const i64 y = __shfl_up_sync(FULL, inc, o); if (lane >= o) inc += y; }
        if (lane == 31) wtot[wid] = inc;
        __syncthreads();
        i64 ex = inc - acc;
        for (int i = 0; i < wid; i++) ex += wtot[i];
#pragma unroll
        for (int i = 0; i < RIPT; i++) pre[tid * RIPT + i] = c[i] + ex;
        __syncthreads();
        for (i64 q = tid; q < cnt; q += RB) {
            int lo = 0, hi = RTILE;                     // first particle whose inclusive prefix exceeds q
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (pre[mid] > q) hi = mid; else lo = mid + 1; }
            if (off + q < n) idx[off + q] = (int)(base + lo);        // k > N: the reference raises IndexError (:61)
        }
        __syncthreads();
    }
}

// sum(residual) and np.cumsum(residual / sum) in the reference's order; cumulative_sum[-1] = 1.
__global__ void __launch_bounds__(32, 1) k_residual_seq(i64 n, const double *__restrict__ w, double *__restrict__ c_out,
                                                        double *__restrict__ sum_out)
{
    __shared__ double buf[SEQ_CHUNK];
    const int lane = threadIdx.x;
    const double Nd = (double)n;
    constexpr int PER = SEQ_CHUNK / 32;
    double r[PER];
    auto fetch = [&](i64 base) {
#pragma unroll
        for (int i = 0; i < PER; i++) { const i64 j = base + i * 32 + lane; r[i] = (j < n) ? w[j] : 0.0; }
    };
    // ---- pass 1: s = 0 + r0 + r1 + ... (resampling.py:70, builtin sum)
    double s = 0.0;
    fetch(0);
    for (i64 base = 0; base < n; base += SEQ_CHUNK) {
#pragma unroll
        for (int i = 0; i < PER; i++) buf[i * 32 + lane] = residual_of(Nd, r[i]);
        __syncwarp();
        if (base + SEQ_CHUNK < n) fetch(base + SEQ_CHUNK);      // in flight during the serial part
        if (lane == 0) {
            const int m = (int)((n - base < SEQ_CHUNK) ? (n - base) : SEQ_CHUNK);
            if (m == SEQ_CHUNK) {
#pragma unroll 16
                for (int j = 0; j < SEQ_CHUNK; j++) s = __dadd_rn(s, buf[j]);
            } else {
                for (int j = 0; j < m; j++) s = __dadd_rn(s, buf[j]);
            }
        }
        __syncwarp();
    }
    s = __shfl_sync(FULL, s, 0);
    if (lane == 0 && sum_out) *sum_out = s;
    // ---- pass 2: c[j] = c[j-1] + r[j] / s (resampling.py:70-71), c[N-1] = 1 (:72)
    double c = 0.0;
    fetch(0);
    for (i64 base = 0; base < n; base += SEQ_CHUNK) {
#pragma unroll
        for (int i = 0; i < PER; i++) buf[i * 32 + lane] = __ddiv_rn(residual_of(Nd, r[i]), s);
        __syncwarp();
        if (base + SEQ_CHUNK < n) fetch(base + SEQ_CHUNK);
        if (lane == 0) {
            const int m = (int)((n - base < SEQ_CHUNK) ? (n - base) : SEQ_CHUNK);
            int j0 = 0;
            if (base == 0) { c = buf[0]; j0 = 1; }              // np.cumsum starts from the first element itself
            if (m == SEQ_CHUNK && j0 == 0) {
#pragma unroll 16
                for (int j = 0; j < SEQ_CHUNK; j++) { c = __dadd_rn(c, buf[j]); buf[j] = c; }
            } else {
                for (int j = j0; j < m; j++) { c = __dadd_rn(c, buf[j]); buf[j] = c; }
            }
        }
        __syncwarp();
#pragma unroll
        for (int i = 0; i < PER; i++) {
            const i64 j = base + i * 32 + lane;
            if (j < n) c_out[j] = (j == n - 1) ? 1.0 : buf[i * 32 + lane];
        }
        __syncwarp();
    }
}

// one sweep of the bracket recurrence (see the header of this file); prev == nullptr: every key over [0, n)
__global__ void __launch_bounds__(256) k_bisect_sweep(i64 n, const double *__restrict__ arr, i64 m, const double *__restrict__ keys,
                                                      const i64 *__restrict__ prev, i64 *__restrict__ next,
                                                      int *__restrict__ idx32, int *changed)
{
    int any = 0;
    for (i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (i64)gridDim.x * blockDim.x) {
        const double key = keys[i];
        i64 lo = 0, hi = n;
        if (prev && i > 0) {
            const i64 rp = prev[i - 1];
            if (np_lt(keys[i - 1], key)) { lo = rp; hi = n; }
            else { lo = 0; hi = rp < n ? rp + 1 : n; }
        }
        while (lo < hi) {
            const i64 mid = lo + ((hi - lo) >> 1);
            if (np_lt(arr[mid], key)) lo = mid + 1; else hi = mid;
        }
        if (prev && prev[i] != lo) any = 1;
        next[i] = lo;
        if (idx32) idx32[i] = (int)lo;
    }
    if (any) *changed = 1;
}

}  // namespace rr
}  // namespace bke

using namespace bke;

extern "C" {

size_t bke_residual_workspace_bytes(int64_t n) { return rr::ws_bytes(n > 0 ? n : 0); }

int bke_residual_prepare(int64_t n, const double *weights, int32_t *indexes, double *cumsum_out, int64_t *n_copies_out,
                         double *residual_sum_out, void *workspace, size_t workspace_bytes, void *stream)
{
    if (n < 0) { set_error("n < 0"); return BKE_ERR_BAD_ARG; }
    if (!n_copies_out) { set_error("n_copies_out is NULL"); return BKE_ERR_BAD_ARG; }
    cudaStream_t s = (cudaStream_t)stream;
    if (n == 0) return check_cuda(cudaMemsetAsync(n_copies_out, 0, sizeof(int64_t), s), "memset n_copies");
    if (n > 0x7fffffffLL) { set_error("residual_resample: n must fit int32 indexes"); return BKE_ERR_BAD_ARG; }
    if (!weights || !indexes || !cumsum_out || !workspace) { set_error("NULL argument"); return BKE_ERR_BAD_ARG; }
    if (workspace_bytes < rr::ws_bytes(n)) { set_error("workspace too small: %zu < %zu", workspace_bytes, rr::ws_bytes(n)); return BKE_ERR_BAD_ARG; }
    rr::RWs ws;
    rr::carve(n, (unsigned char *)workspace, &ws);
    const int grid = ws.T < sm_count() * 8 ? ws.T : sm_count() * 8;
    rr::k_counts<<<grid, rr::RB, 0, s>>>(n, weights, ws);
    rr::k_scan_counts<<<1, 1024, 0, s>>>(ws, (rr::i64 *)n_copies_out);
    rr::k_expand<<<grid, rr::RB, 0, s>>>(n, weights, ws, indexes);
    rr::k_residual_seq<<<1, 32, 0, s>>>(n, weights, cumsum_out, residual_sum_out);
    return check_cuda(cudaGetLastError(), "residual_prepare launch");
}

int bke_searchsorted_bracket_sweep(int64_t n, const double *arr, int64_t n_keys, const double *keys, const int64_t *prev,
                                   int64_t *next, int32_t *indexes32, int32_t *changed, void *stream)
{
    if (n < 0 || n_keys < 0) { set_error("negative length"); return BKE_ERR_BAD_ARG; }
    if (n_keys == 0) return BKE_OK;
    if ((n > 0 && !arr) || !keys || !next || !changed) { set_error("NULL argument"); return BKE_ERR_BAD_ARG; }
    int64_t blocks = (n_keys + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 32;
    if (blocks > cap) blocks = cap;
    rr::k_bisect_sweep<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(n, arr, n_keys, keys, (const rr::i64 *)prev,
                                                                           (rr::i64 *)next, indexes32, changed);
    return check_cuda(cudaGetLastError(), "searchsorted_bracket_sweep launch");
}

}  // extern "C"
