// resample_bank.cu — systematic / stratified resampling of a BANK of particle sets in one launch:
// row b of weights[B, M] is one set, resampled exactly as the reference resamples one weight vector
// (filterpy/monte_carlo/resampling.py:117-150 systematic, :80-114 stratified).
//
// With B independent sets the parallelism comes from the sets, so each set can run the reference's
// own arithmetic literally: one thread per set forms the strictly sequential fp64 cumsum (:142,
// c_0 = w_0, c_j = fl(c_{j-1} + w_j)) and walks the two-pointer merge of :144-149
//
//     while i < M:  if pos_i < c_j: indexes[i] = j; i += 1   else: j += 1   (j == M: IndexError, :145)
//
// with pos_i = fl(fl(u + i) / M) (:139) or fl(fl(U_i + i) / M) (:103).  That is the reference for
// every input — negative, NaN, infinite, signed-zero and subnormal weights, uniforms outside [0, 1)
// or out of order — with no verification pass and no fallback.
//
// A thread walking its own row would load and store uncoalesced (rows are M elements apart), so
// each CTA stages a window of COLS elements of every one of its ROWS sets in shared memory: the
// weights at the merge's j, the positions and the output indexes at its i.  The CTA alternates
//   run    every set advances its merge until it leaves its weight window or fills its output window;
//   move   a warp per set moves 32 consecutive elements: it writes back a full (or final) output
//          window, loads the next weight window, and loads the next uniforms and forms the positions
//          (so the fp64 divisions run in parallel over the window, off the sequential path).
// Each round consumes at least one window per unfinished set, so a set of M particles finishes in at
// most 2M / COLS + 1 rounds.  Global traffic: weights (and uniforms) read once, indexes written once,
// all as 256-byte / 128-byte row segments.
//
// Below k_resample_bank: multinomial (resampling.py:153-176) and residual (:27-76) resampling of a bank.
// Both end in np.searchsorted(c, keys) (side='left') over a per-set array c, which NumPy bisects with a
// bracket carried from key to key ([r[i-1], M) if key[i-1] < key[i], else [0, r[i-1] + 1), NaN last;
// csrc/residual.cu).  One warp per set:
//   k_prepare_bank   the strictly sequential parts literally: builtin sum(residual) and np.cumsum, one
//                    __dadd_rn per element, the chain fed by a warp shuffle of 32 coalesced loads; c goes
//                    to the workspace with c[-1] = 1.  Residual also writes the copies repeat(arange(M),
//                    num_copies) as coalesced 32-wide segments, and k.  The set is marked for the exact
//                    search unless c[0..M-2] is nondecreasing in NaN-last order and c[M-2] <= 1: then the
//                    whole c is sorted, less(c[i], key) holds on a prefix for every key, any bracket NumPy
//                    carries contains that prefix's end, and every key can be searched on its own.
//   k_search_bank    32 keys per round, one per lane.  A sorted set takes one bisection per key.  Any other
//                    set runs the carried-bracket recurrence as a fixed point inside the round: each lane
//                    re-bisects from the bracket its left neighbour's current answer gives (lane 0: the
//                    previous round's last key and answer, which are final), until a sweep changes no lane.
//                    After t sweeps the first t lanes are final, so a round takes at most 33 sweeps; on
//                    residual's sets two or three are typical.
#include <type_traits>

#include "bke_internal.cuh"
#include "residual_rules.cuh"

namespace bke {
namespace rsb {

typedef long long i64;

constexpr int ROWS = 64;        // sets per CTA, one thread each
constexpr int COLS = 32;        // elements of one set per window (one warp-wide segment)
constexpr int PAD = COLS + 1;   // row pitch in shared memory: consecutive sets start in different banks

struct Shared {
    double w[ROWS][PAD];        // weights[kj .. kj + COLS) of each set
    double pos[ROWS][PAD];      // positions[ki .. ki + COLS)
    int out[ROWS][PAD];         // indexes[ki .. ki + COLS), written back when full or final
    int kj[ROWS], ki[ROWS];     // window bases to load in the next move, in units of COLS
    int fbase[ROWS];            // output window to write back, in units of COLS
    double u[ROWS];             // systematic offset of each set
    int nflush[ROWS];           // outputs to write back (0: none)
    int load_w[ROWS], load_p[ROWS];
};

// The CTA's sets are b0 .. b0 + ROWS - 1, or, with a RowList, list.rows[b0 ..] of the *list.count listed sets
// (the gated epoch below resamples only those).  NoList is an empty trailing argument, so the plain
// instances keep their parameter offsets and their code.
struct NoList {};
struct RowList { const int *rows; const int *count; };

template <bool STRAT, typename L = NoList>
__global__ void __launch_bounds__(ROWS) k_resample_bank(i64 n_sets, i64 M, const double *__restrict__ w,
                                                        const double *__restrict__ u, const double *__restrict__ U,
                                                        int *__restrict__ idx, int *__restrict__ status, L list = L())
{
    constexpr bool LISTED = std::is_same<L, RowList>::value;
    __shared__ Shared sh;
    const int r = threadIdx.x;
    const i64 b0 = (i64)blockIdx.x * ROWS;
    i64 rem = n_sets - b0;
    if constexpr (LISTED) {
        rem = (i64)*list.count - b0;
        if (rem <= 0) return;                     // the whole CTA: past the listed sets
    }
    const int rows = rem < ROWS ? (int)rem : ROWS;
    const double Md = (double)M;

    bool active = r < rows;
    i64 ki = 0, kj = 0;             // window bases of this thread's set
    int ii = 0, jj = 0;             // merge pointers within the windows: i = ki + ii, j = kj + jj
    double c = 0.0;                 // cumsum(w)[j]
    bool fresh_w = true;            // the weight window was just loaded: c still lacks w[kj]
    i64 set = 0;                    // the listed set of this thread (plain instances: b0 + r)
    if constexpr (LISTED) set = active ? (i64)list.rows[b0 + r] : 0;
    sh.kj[r] = 0; sh.ki[r] = 0; sh.fbase[r] = 0; sh.nflush[r] = 0;
    sh.load_w[r] = active; sh.load_p[r] = active;
    sh.u[r] = (!STRAT && active) ? u[LISTED ? set : b0 + r] : 0.0;
    bool more = active;

    while (__syncthreads_or(more)) {
        // ---- move: a warp per set, a lane per column
#pragma unroll 4
        for (int e = r; e < ROWS * COLS; e += ROWS) {
            const int q = e / COLS, t = e % COLS;
            i64 qset = b0 + q;
            if constexpr (LISTED) qset = q < rows ? (i64)list.rows[b0 + q] : 0;
            const i64 row = qset * M;
            if (t < sh.nflush[q]) idx[row + (i64)sh.fbase[q] * COLS + t] = sh.out[q][t];
            if (sh.load_w[q]) {
                const i64 k = (i64)sh.kj[q] * COLS + t;
                if (k < M) sh.w[q][t] = __ldg(w + row + k);
            }
            if (sh.load_p[q]) {
                const i64 k = (i64)sh.ki[q] * COLS + t;
                if (k < M) {
                    const double a = STRAT ? __ldg(U + row + k) : sh.u[q];
                    sh.pos[q][t] = __ddiv_rn(__dadd_rn(a, (double)k), Md);       // resampling.py:139 / :103
                }
            }
        }
        __syncthreads();

        // ---- run: the reference's merge until a window is used up
        int nflush = 0, need_w = 0, need_p = 0;
        const i64 fbase = ki;
        if (active) {
            if (fresh_w) {                                   // np.cumsum: c_0 = w_0, then one add per element
                c = (kj == 0) ? sh.w[r][0] : __dadd_rn(c, sh.w[r][0]);
                fresh_w = false;
            }
            const int ilim = (M - ki) < COLS ? (int)(M - ki) : COLS;
            const int jlim = (M - kj) < COLS ? (int)(M - kj) : COLS;
            const int jbase = (int)kj;
            for (;;) {
                if (sh.pos[r][ii] < c) {                      // :146
                    sh.out[r][ii] = jbase + jj;
                    if (++ii == ilim) break;
                } else {
                    if (++jj == jlim) break;
                    c = __dadd_rn(c, sh.w[r][jj]);
                }
            }
            if (ii == ilim) {
                nflush = ii;
                if (ki + ii == M) {                           // every position placed
                    active = false;
                    if (status) status[LISTED ? set : b0 + r] = 0;
                } else { need_p = 1; ki += COLS; ii = 0; }
            } else if (kj + jj == M) {                        // j ran off the end: the reference's IndexError (:145)
                nflush = ii;
                active = false;
                if (status) status[LISTED ? set : b0 + r] = 1;
            } else { need_w = 1; kj += COLS; jj = 0; fresh_w = true; }
        }
        sh.nflush[r] = nflush; sh.fbase[r] = (int)(fbase / COLS);
        sh.load_w[r] = need_w; sh.kj[r] = (int)(kj / COLS);
        sh.load_p[r] = need_p; sh.ki[r] = (int)(ki / COLS);
        more = active || nflush > 0;
    }
}

// ---------------------------------------------------------------------- gated epoch
// A particle filter's epoch over a bank: normalise every row, take its effective sample size, and resample
// and gather only the sets below the threshold.  Three launches:
//   k_gated_stats      one warp per set: S = np.sum(w), w /= S in place, neff = 1 / np.sum(np.square(w)), the
//                      gate; a gated set appends itself to the row list in the workspace;
//   k_resample_bank    <STRAT, RowList>: the merge above on the listed sets only, so its rounds are paid per
//                      resampled set and not per CTA of 64 sets of which a few are live;
//   k_gather_reset     one CTA per listed set: particles[b] <- particles[b][indexes[b]] through shared
//                      memory, weights[b] <- 1 / M.
//
// np.sum of a contiguous fp64 row is fl(+0.0 + pw(a)), pw NumPy's pairwise_sum (numpy/_core/src/umath/
// loops_utils.h.src, PW_BLOCKSIZE = 128): n < 8 a sequential sum from 0; n <= 128 eight strided accumulators
// r[k] += a[i + k], combined ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the n % 8 rest in order; above 128 the
// sum of the two halves split at n / 2 - (n / 2) % 8.  The tree depends only on M, so the warp walks it
// uniformly: a leaf is staged in shared memory by coalesced loads, lane k (mod 8) runs accumulator k, a xor
// butterfly over 1, 2, 4 forms the bracketing above (fp add commutes), and the pending right halves and left
// sums of the path to the root sit one per lane (the tree is at most 25 deep for M < 2^31).
constexpr int GW = 8;           // sets per CTA of k_gated_stats, one warp each
constexpr int PW_BLOCK = 128;   // NumPy's PW_BLOCKSIZE

__device__ __forceinline__ double pw_leaf(const double *s, int n, int lane)
{
    if (n < 8) {
        double r = 0.0;
        for (int i = 0; i < n; i++) r = __dadd_rn(r, s[i]);
        return r;
    }
    const int k = lane & 7, n8 = n - (n & 7);
    double r = s[k];
    for (int i = 8; i < n8; i += 8) r = __dadd_rn(r, s[i + k]);
    r = __dadd_rn(r, __shfl_xor_sync(FULL, r, 1));
    r = __dadd_rn(r, __shfl_xor_sync(FULL, r, 2));
    r = __dadd_rn(r, __shfl_xor_sync(FULL, r, 4));
    for (int i = n8; i < n; i++) r = __dadd_rn(r, s[i]);
    return r;
}

// NORMALISE = false: pw(row).  true: row <- row / S in place, and pw(square(row)).  Every lane returns it.
template <bool NORMALISE>
__device__ double pw_row(double *row, int M, double S, double *sm, int lane)
{
    int off = 0, n = M, sp = 0;
    int st_off = 0, st_n = 0;             // stack level `lane`: the right half still to sum
    bool st_left = false;                 // ... and whether its left half's sum is in st_sum
    double st_sum = 0.0;
    for (;;) {
        while (n > PW_BLOCK) {
            const int n2 = n / 2 - (n / 2) % 8;
            if (lane == sp) { st_off = off + n2; st_n = n - n2; st_left = false; }
            ++sp;
            n = n2;
        }
        for (int i = lane; i < n; i += 32) {
            double x = row[off + i];
            if (NORMALISE) {
                x = __ddiv_rn(x, S);
                row[off + i] = x;
                x = __dmul_rn(x, x);
            }
            sm[i] = x;
        }
        __syncwarp();
        double v = pw_leaf(sm, n, lane);
        __syncwarp();
        for (;;) {
            if (sp == 0) return v;
            const int top = sp - 1;
            if (!__shfl_sync(FULL, st_left, top)) {
                if (lane == top) { st_left = true; st_sum = v; }
                off = __shfl_sync(FULL, st_off, top);
                n = __shfl_sync(FULL, st_n, top);
                break;
            }
            v = __dadd_rn(__shfl_sync(FULL, st_sum, top), v);
            --sp;
        }
    }
}

__global__ void __launch_bounds__(32 * GW) k_gated_stats(i64 n_sets, int M, double *w, double threshold,
                                                         double *__restrict__ neff, uint8_t *__restrict__ resampled,
                                                         int *__restrict__ status, int *count, int *__restrict__ list)
{
    __shared__ double sm[GW][PW_BLOCK];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const i64 b = (i64)blockIdx.x * GW + wid;
    if (b >= n_sets) return;                                  // whole warps leave
    double *row = w + b * M;
    const double S = __dadd_rn(0.0, pw_row<false>(row, M, 0.0, sm[wid], lane));
    const double q = __dadd_rn(0.0, pw_row<true>(row, M, S, sm[wid], lane));
    const double ne = __ddiv_rn(1.0, q);
    const bool gate = ne < threshold;
    if (lane == 0) {
        neff[b] = ne;
        resampled[b] = gate;
        status[b] = 0;
        if (gate) list[atomicAdd(count, 1)] = (int)b;        // the order only decides which sets share a CTA
    }
}

// particles[b] <- particles[b][indexes[b]] and weights[b] <- 1 / M for the listed sets that did not fail; the
// set's row of M * cpp chunks of V is staged in dynamic shared memory, so the gather runs in place.
template <typename V>
__global__ void __launch_bounds__(256) k_gather_reset(int M, int cpp, V *parts, const int *__restrict__ idx,
                                                      double *w, const int *__restrict__ list, const int *count,
                                                      const int *__restrict__ status)
{
    extern __shared__ uint4 stage_raw[];
    V *stage = reinterpret_cast<V *>(stage_raw);
    const int n = *count, total = M * cpp;
    const double inv = __ddiv_rn(1.0, (double)M);
    for (int t = blockIdx.x; t < n; t += gridDim.x) {
        const i64 b = list[t];
        if (status[b]) continue;                              // the reference raised: keep the row as it is
        V *row = parts + b * (i64)total;
        for (int e = threadIdx.x; e < total; e += blockDim.x) stage[e] = row[e];
        __syncthreads();
        const int *ir = idx + b * M;
        for (int e = threadIdx.x; e < total; e += blockDim.x) {
            const int i = e / cpp, c = e - i * cpp;
            row[e] = stage[ir[i] * cpp + c];
        }
        double *wr = w + b * M;
        for (int i = threadIdx.x; i < M; i += blockDim.x) wr[i] = inv;
        __syncthreads();                                      // the next set overwrites the stage
    }
}

// ---------------------------------------------------------------------- multinomial / residual
constexpr int MR_WARPS = 8;                    // sets per CTA, one warp each
constexpr int ST_FAIL = 1;                     // status bit: the reference raises IndexError (residual: k > M)
constexpr int ST_EXACT = 2;                    // status bit: the set takes the carried-bracket search

__device__ __forceinline__ int warp_incl_scan(int v, int lane)
{
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(FULL, v, o); if (lane >= o) v += y; }
    return v;
}

// c = np.cumsum(w) (multinomial, :173) or np.cumsum(residual / sum(residual)) (residual, :69-71), c[-1] = 1;
// residual also writes indexes[b, :k] and k[b].  status[b] = ST_FAIL where k > M, else ST_EXACT or 0.
template <bool RESIDUAL>
__global__ void __launch_bounds__(32 * MR_WARPS) k_prepare_bank(i64 n_sets, int M, const double *__restrict__ w,
                                                                 double *__restrict__ cws, int *__restrict__ idx,
                                                                 i64 *__restrict__ k_out, int *__restrict__ status)
{
    const int lane = threadIdx.x & 31;
    const i64 b = (i64)blockIdx.x * MR_WARPS + (threadIdx.x >> 5);
    if (b >= n_sets) return;                                  // whole warps leave
    const double *wr = w + b * M;
    double *cr = cws + b * M;
    const double Md = (double)M;
    double s = 0.0;
    if (RESIDUAL) {
        // k (copies, saturated at M + 1) and s = 0 + r0 + r1 + ... (:70, the builtin sum)
        i64 k = 0;
        for (int j0 = 0; j0 < M; j0 += 32) {
            const int j = j0 + lane, n = M - j0 < 32 ? M - j0 : 32;
            const double x = j < M ? __ldg(wr + j) : 0.0;
            const double r = rr::residual_of(Md, x);
            i64 cnt = j < M ? rr::copies_made(Md, x) : 0;
            cnt = cnt > (i64)M + 1 ? (i64)M + 1 : cnt;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(FULL, cnt, o);
            k = k + cnt > (i64)M + 1 ? (i64)M + 1 : k + cnt;
            for (int t = 0; t < n; t++) s = __dadd_rn(s, __shfl_sync(FULL, r, t));
        }
        if (lane == 0) k_out[b] = k;
        if (k > M) {                                          // indexes[k] = i runs off the end (:61)
            if (lane == 0) status[b] = ST_FAIL;
            return;
        }
    }
    double acc = 0.0;                                         // c[j0 - 1]
    bool unsorted = false;
    int off = 0;                                              // copies written so far
    int *ir = RESIDUAL ? idx + b * M : nullptr;
    for (int j0 = 0; j0 < M; j0 += 32) {
        const int j = j0 + lane, n = M - j0 < 32 ? M - j0 : 32;
        const double x = j < M ? __ldg(wr + j) : 0.0;
        const double v = RESIDUAL ? __ddiv_rn(rr::residual_of(Md, x), s) : x;
        const double before = acc;
        double mine = 0.0;
        for (int t = 0; t < n; t++) {                         // np.cumsum: c_0 = v_0, then one add per element
            const double y = __shfl_sync(FULL, v, t);
            acc = (j0 == 0 && t == 0) ? y : __dadd_rn(acc, y);
            if (lane == t) mine = acc;
        }
        double left = __shfl_up_sync(FULL, mine, 1);
        if (lane == 0) left = before;
        if (j >= 1 && j <= M - 2 && rr::np_lt(mine, left)) unsorted = true;
        if (j == M - 2 && rr::np_lt(1.0, mine)) unsorted = true;   // c[-1] = 1 would end the sort
        if (j < M) cr[j] = j == M - 1 ? 1.0 : mine;                // :174 / :72
        if (RESIDUAL) {                                       // repeat(arange(M), num_copies) (:58-62), in order
            const int cnt = j < M ? (int)rr::copies_made(Md, x) : 0;
            const int inc = warp_incl_scan(cnt, lane);
            const int tot = __shfl_sync(FULL, inc, 31);
            for (int q0 = 0; q0 < tot; q0 += 32) {
                const int q = q0 + lane;
                int lo = 0, hi = 31;                          // the first lane whose inclusive count exceeds q
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (__shfl_sync(FULL, inc, mid) > q) hi = mid; else lo = mid + 1;
                }
                if (q < tot) ir[off + q] = j0 + lo;
            }
            off += tot;
        }
    }
    unsorted = __any_sync(FULL, unsorted);
    if (lane == 0) status[b] = unsorted ? ST_EXACT : 0;
}

// np.searchsorted(c, key) over [lo, hi): NumPy's left bisection in NaN-last order
__device__ __forceinline__ int bisect(const double *__restrict__ c, double key, int lo, int hi)
{
    while (lo < hi) {
        const int mid = lo + ((hi - lo) >> 1);
        if (rr::np_lt(__ldg(c + mid), key)) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// indexes[b, k_b + q] = searchsorted(c_b, keys[b, q]) for q < M - k_b (multinomial: k_b = 0)
template <bool RESIDUAL, typename I>
__global__ void __launch_bounds__(32 * MR_WARPS) k_search_bank(i64 n_sets, int M, const double *__restrict__ cws,
                                                                const double *__restrict__ U,
                                                                const i64 *__restrict__ k_in,
                                                                const int *__restrict__ status, I *__restrict__ idx)
{
    const int lane = threadIdx.x & 31;
    const i64 b = (i64)blockIdx.x * MR_WARPS + (threadIdx.x >> 5);
    if (b >= n_sets) return;
    const int st = status[b];
    if (st & ST_FAIL) return;
    const int k = RESIDUAL ? (int)k_in[b] : 0;
    const int n = M - k;
    const double *c = cws + b * M, *keys = U + b * M;
    I *out = idx + b * M + k;
    const bool exact = st & ST_EXACT;
    double ck = 0.0;                                          // the previous round's last key and answer
    int cr = 0;
    for (int q0 = 0; q0 < n; q0 += 32) {
        const int q = q0 + lane;
        const bool valid = q < n;
        const double key = valid ? __ldg(keys + q) : 0.0;
        int r = bisect(c, key, 0, M);
        if (exact) {
            for (;;) {
                double pk = __shfl_up_sync(FULL, key, 1);
                int pr = __shfl_up_sync(FULL, r, 1);
                if (lane == 0) { pk = ck; pr = cr; }
                int lo = 0, hi = M;                           // the first key: [0, M)
                if (q > 0) {
                    if (rr::np_lt(pk, key)) lo = pr;
                    else hi = pr < M ? pr + 1 : M;
                }
                const int nr = bisect(c, key, lo, hi);
                const bool changed = valid && nr != r;
                r = nr;
                if (!__any_sync(FULL, changed)) break;
            }
            const int last = n - q0 < 32 ? n - q0 - 1 : 31;
            ck = __shfl_sync(FULL, key, last);
            cr = __shfl_sync(FULL, r, last);
        }
        if (valid) out[q] = (I)r;
    }
}

static size_t mr_ws_bytes(i64 B, i64 M)
{
    if (B <= 0 || M <= 0) return 0;
    if (B > (i64)(SIZE_MAX / 8) / M) return SIZE_MAX;
    return (size_t)B * (size_t)M * sizeof(double);
}

// the checks every multinomial / residual bank call shares; *done = 1: nothing to compute
static int mr_check(i64 B, i64 M, const void *ws, size_t ws_bytes, int *done)
{
    *done = 0;
    if (B < 0 || M < 0) { set_error("n_sets and n_particles must be >= 0"); return BKE_ERR_BAD_ARG; }
    if (M >= ((i64)1 << 31)) { set_error("n_particles must be < 2^31"); return BKE_ERR_BAD_ARG; }
    if (B == 0 || M == 0) { *done = 1; return BKE_OK; }
    if ((B + MR_WARPS - 1) / MR_WARPS >= ((i64)1 << 31) || mr_ws_bytes(B, M) == SIZE_MAX) {
        set_error("n_sets too large"); return BKE_ERR_BAD_ARG;
    }
    if (!ws || (reinterpret_cast<uintptr_t>(ws) & 7)) { set_error("workspace must be non-NULL and 8-byte aligned"); return BKE_ERR_BAD_ARG; }
    if (ws_bytes < mr_ws_bytes(B, M)) {
        set_error("workspace too small: %zu < %zu", ws_bytes, mr_ws_bytes(B, M)); return BKE_ERR_BAD_ARG;
    }
    return BKE_OK;
}

}  // namespace rsb
}  // namespace bke

using namespace bke;

extern "C" {

int bke_resample_bank(const bke_resample_bank_args *a, void *stream)
{
    if (!a) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    if (a->n_sets < 0 || a->n_particles < 0) { set_error("n_sets and n_particles must be >= 0"); return BKE_ERR_BAD_ARG; }
    if (a->n_particles >= ((int64_t)1 << 31)) { set_error("n_particles must be < 2^31 (indexes are int32, resampling.py:141)"); return BKE_ERR_BAD_ARG; }
    if ((a->u == nullptr) == (a->uniforms == nullptr)) { set_error("give exactly one of u (systematic) and uniforms (stratified)"); return BKE_ERR_BAD_ARG; }
    if (a->n_sets == 0 || a->n_particles == 0) return BKE_OK;
    if (!a->weights || !a->indexes) { set_error("weights and indexes must be non-NULL"); return BKE_ERR_BAD_ARG; }
    const int64_t blocks = (a->n_sets + rsb::ROWS - 1) / rsb::ROWS;
    if (blocks >= ((int64_t)1 << 31)) { set_error("n_sets too large"); return BKE_ERR_BAD_ARG; }
    cudaStream_t s = (cudaStream_t)stream;
    if (a->uniforms)
        rsb::k_resample_bank<true><<<(unsigned)blocks, rsb::ROWS, 0, s>>>(a->n_sets, a->n_particles, a->weights, nullptr,
                                                                         a->uniforms, a->indexes, a->status);
    else
        rsb::k_resample_bank<false><<<(unsigned)blocks, rsb::ROWS, 0, s>>>(a->n_sets, a->n_particles, a->weights, a->u,
                                                                          nullptr, a->indexes, a->status);
    return check_cuda(cudaGetLastError(), "resample bank launch");
}

size_t bke_resample_bank_gated_workspace_bytes(int64_t n_sets)
{
    return n_sets <= 0 ? 0 : 16 + (size_t)n_sets * sizeof(int32_t);      // the counter, padded, then the list
}

// the checks _stats and _apply share; *done = 1: nothing to compute
static int gated_check(const bke_resample_bank_gated_args *a, int *done)
{
    *done = 0;
    if (!a) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    if (a->n_sets < 0 || a->n_particles < 0) { set_error("n_sets and n_particles must be >= 0"); return BKE_ERR_BAD_ARG; }
    if (a->n_particles >= ((int64_t)1 << 31)) { set_error("n_particles must be < 2^31"); return BKE_ERR_BAD_ARG; }
    if (a->n_sets >= ((int64_t)1 << 31)) { set_error("n_sets must be < 2^31"); return BKE_ERR_BAD_ARG; }
    if (a->n_sets == 0 || a->n_particles == 0) { *done = 1; return BKE_OK; }
    if (!a->weights || !a->neff || !a->resampled || !a->status) {
        set_error("weights, neff, resampled and status must be non-NULL"); return BKE_ERR_BAD_ARG;
    }
    if (!a->workspace || (reinterpret_cast<uintptr_t>(a->workspace) & 3)) {
        set_error("workspace must be non-NULL and 4-byte aligned"); return BKE_ERR_BAD_ARG;
    }
    const size_t need = bke_resample_bank_gated_workspace_bytes(a->n_sets);
    if (a->workspace_bytes < need) { set_error("workspace too small: %zu < %zu", a->workspace_bytes, need); return BKE_ERR_BAD_ARG; }
    return BKE_OK;
}

int bke_resample_bank_gated_stats(const bke_resample_bank_gated_args *a, void *stream)
{
    int done, rc = gated_check(a, &done);
    if (rc != BKE_OK || done) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    int *count = (int *)a->workspace;
    int *list = (int *)((char *)a->workspace + 16);
    if (check_cuda(cudaMemsetAsync(count, 0, sizeof(int), s), "gated bank counter reset")) return BKE_ERR_CUDA;
    const unsigned blocks = (unsigned)((a->n_sets + rsb::GW - 1) / rsb::GW);
    rsb::k_gated_stats<<<blocks, 32 * rsb::GW, 0, s>>>(a->n_sets, (int)a->n_particles, a->weights, a->threshold,
                                                       a->neff, a->resampled, a->status, count, list);
    return check_cuda(cudaGetLastError(), "gated bank statistics launch");
}

// what _apply needs beyond gated_check, the shared-memory cap last (it asks the device)
static int gated_apply_check(const bke_resample_bank_gated_args *a)
{
    if ((a->u == nullptr) == (a->uniforms == nullptr)) { set_error("give exactly one of u (systematic) and uniforms (stratified)"); return BKE_ERR_BAD_ARG; }
    if (!a->particles || !a->indexes) { set_error("particles and indexes must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if (a->particle_bytes <= 0) { set_error("particle_bytes must be > 0"); return BKE_ERR_BAD_ARG; }
    int dev = 0, cap = 0;
    if (check_cuda(cudaGetDevice(&dev), "cudaGetDevice") ||
        check_cuda(cudaDeviceGetAttribute(&cap, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev), "cudaDeviceGetAttribute"))
        return BKE_ERR_CUDA;
    if (a->particle_bytes > cap || a->n_particles > cap / a->particle_bytes) {
        set_error("a set's particle row of %lld x %lld bytes exceeds the %d bytes of shared memory one CTA can stage "
                  "(the device's opt-in maximum per block)", (long long)a->n_particles, (long long)a->particle_bytes, cap);
        return BKE_ERR_BAD_ARG;
    }
    return BKE_OK;
}

int bke_resample_bank_gated_apply(const bke_resample_bank_gated_args *a, void *stream)
{
    int done, rc = gated_check(a, &done);
    if (rc != BKE_OK || done) return rc;
    if ((rc = gated_apply_check(a)) != BKE_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const rsb::RowList rl{(const int *)((const char *)a->workspace + 16), (const int *)a->workspace};
    const unsigned blocks = (unsigned)((a->n_sets + rsb::ROWS - 1) / rsb::ROWS);
    if (a->uniforms)
        rsb::k_resample_bank<true, rsb::RowList><<<blocks, rsb::ROWS, 0, s>>>(
            a->n_sets, a->n_particles, a->weights, nullptr, a->uniforms, a->indexes, a->status, rl);
    else
        rsb::k_resample_bank<false, rsb::RowList><<<blocks, rsb::ROWS, 0, s>>>(
            a->n_sets, a->n_particles, a->weights, a->u, nullptr, a->indexes, a->status, rl);
    if (check_cuda(cudaGetLastError(), "gated bank resample launch")) return BKE_ERR_CUDA;

    const int M = (int)a->n_particles;
    const uintptr_t al = reinterpret_cast<uintptr_t>(a->particles) | (uintptr_t)a->particle_bytes;
    const size_t smem = (size_t)a->n_particles * (size_t)a->particle_bytes;
    const int64_t cap_blocks = (int64_t)sm_count() * 8;
    const unsigned grid = (unsigned)(a->n_sets < cap_blocks ? a->n_sets : cap_blocks);
#define BKE_GATHER_RESET(V) do {                                                                             \
        auto kern = rsb::k_gather_reset<V>;                                                                  \
        if (check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),   \
                       "cudaFuncSetAttribute")) return BKE_ERR_CUDA;                                         \
        kern<<<grid, 256, smem, s>>>(M, (int)(a->particle_bytes / (int64_t)sizeof(V)), (V *)a->particles,   \
                                     a->indexes, a->weights, rl.rows, rl.count, a->status);                  \
    } while (0)
    if ((al & 15) == 0) BKE_GATHER_RESET(uint4);
    else if ((al & 7) == 0) BKE_GATHER_RESET(uint2);
    else if ((al & 3) == 0) BKE_GATHER_RESET(unsigned);
    else BKE_GATHER_RESET(unsigned char);
#undef BKE_GATHER_RESET
    return check_cuda(cudaGetLastError(), "gated bank gather launch");
}

int bke_resample_bank_gated(const bke_resample_bank_gated_args *a, void *stream)
{
    int done, rc = gated_check(a, &done);
    if (rc != BKE_OK || done) return rc;
    if ((rc = gated_apply_check(a)) != BKE_OK) return rc;             // before the weights are normalised
    rc = bke_resample_bank_gated_stats(a, stream);
    return rc != BKE_OK ? rc : bke_resample_bank_gated_apply(a, stream);
}

size_t bke_multinomial_resample_bank_workspace_bytes(int64_t n_sets, int64_t n_particles)
{
    return rsb::mr_ws_bytes(n_sets, n_particles);
}

size_t bke_residual_resample_bank_workspace_bytes(int64_t n_sets, int64_t n_particles)
{
    return rsb::mr_ws_bytes(n_sets, n_particles);
}

int bke_multinomial_resample_bank(const bke_multinomial_resample_bank_args *a, void *stream)
{
    if (!a) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    int done, rc = rsb::mr_check(a->n_sets, a->n_particles, a->workspace, a->workspace_bytes, &done);
    if (rc != BKE_OK || done) return rc;
    if (!a->weights || !a->uniforms || !a->indexes || !a->status) {
        set_error("weights, uniforms, indexes and status must be non-NULL"); return BKE_ERR_BAD_ARG;
    }
    const unsigned blocks = (unsigned)((a->n_sets + rsb::MR_WARPS - 1) / rsb::MR_WARPS);
    const int M = (int)a->n_particles;
    double *c = (double *)a->workspace;
    cudaStream_t s = (cudaStream_t)stream;
    rsb::k_prepare_bank<false><<<blocks, 32 * rsb::MR_WARPS, 0, s>>>(a->n_sets, M, a->weights, c, nullptr, nullptr,
                                                                     a->status);
    rsb::k_search_bank<false, long long><<<blocks, 32 * rsb::MR_WARPS, 0, s>>>(
        a->n_sets, M, c, a->uniforms, nullptr, a->status, (long long *)a->indexes);
    return check_cuda(cudaGetLastError(), "multinomial bank launch");
}

int bke_residual_resample_bank_prepare(const bke_residual_resample_bank_args *a, void *stream)
{
    if (!a) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    int done, rc = rsb::mr_check(a->n_sets, a->n_particles, a->workspace, a->workspace_bytes, &done);
    if (rc != BKE_OK || done) return rc;
    if (!a->weights || !a->indexes || !a->n_copies || !a->status) {
        set_error("weights, indexes, n_copies and status must be non-NULL"); return BKE_ERR_BAD_ARG;
    }
    const unsigned blocks = (unsigned)((a->n_sets + rsb::MR_WARPS - 1) / rsb::MR_WARPS);
    rsb::k_prepare_bank<true><<<blocks, 32 * rsb::MR_WARPS, 0, (cudaStream_t)stream>>>(
        a->n_sets, (int)a->n_particles, a->weights, (double *)a->workspace, a->indexes, (rsb::i64 *)a->n_copies,
        a->status);
    return check_cuda(cudaGetLastError(), "residual bank prepare launch");
}

int bke_residual_resample_bank_search(const bke_residual_resample_bank_args *a, void *stream)
{
    if (!a) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    int done, rc = rsb::mr_check(a->n_sets, a->n_particles, a->workspace, a->workspace_bytes, &done);
    if (rc != BKE_OK || done) return rc;
    if (!a->uniforms || !a->indexes || !a->n_copies || !a->status) {
        set_error("uniforms, indexes, n_copies and status must be non-NULL"); return BKE_ERR_BAD_ARG;
    }
    const unsigned blocks = (unsigned)((a->n_sets + rsb::MR_WARPS - 1) / rsb::MR_WARPS);
    rsb::k_search_bank<true, int><<<blocks, 32 * rsb::MR_WARPS, 0, (cudaStream_t)stream>>>(
        a->n_sets, (int)a->n_particles, (const double *)a->workspace, a->uniforms, (const rsb::i64 *)a->n_copies,
        a->status, a->indexes);
    return check_cuda(cudaGetLastError(), "residual bank search launch");
}

}  // extern "C"
