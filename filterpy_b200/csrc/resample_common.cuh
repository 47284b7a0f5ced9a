// resample_common.cuh — device primitives of the resampling kernels (csrc/resample.cu): parity maps
// of the exact sequential fp64 cumulative sum
// (filterpy/monte_carlo/resampling.py:142), warp scans, the position count of :139 / :103.
#pragma once
#include "bke_internal.cuh"

namespace bke {
namespace rs {

constexpr int BLOCK = 256;
constexpr int IPT = 16;
constexpr int TILE = BLOCK * IPT;        // 4096 particles per tile
constexpr int RMAX = 64;                 // raw elements per tile before giving up
constexpr int UMAX = 2048;               // tiles with raw elements before giving up
constexpr int EXPAND = 8192;             // outputs expanded per shared-memory pass
constexpr int INLINE_MAX = 64;           // copies of one particle a thread writes itself (more: general expansion)
constexpr int BIGRUN = 2 * EXPAND;       // runs this long go to the fill kernel
constexpr int CHAIN_THREADS = 1024;
constexpr int CHAIN_BATCH = 8;           // unclean tiles staged in shared memory per round of the chain
constexpr int SEQMAX = 256;             // fully sequential tiles (dense raw zones) before giving up
constexpr int SLOT_SEQ = -2;            // tile_slot code: every element of the tile is applied by a true add
constexpr int SLOT_FAST = -3;           // tile_slot code: clean tile, tie-free, one binade -> plain int64 sums
constexpr int K_ID = -2;                 // identity (only zero weights so far)
constexpr int K_POISON = -3;             // elements of different binades were mixed (never expected)

typedef long long i64;
typedef unsigned long long u64;

// Parity map: d = d0, t = d1 - d0 in {-1,0,1}; cnt = raw elements seen; k = binade of the map.
struct SM { i64 d; int t; int cnt; int k; };

__device__ __forceinline__ int merge_k(int a, int b)
{
    if (a == K_ID) return b;
    if (b == K_ID) return a;
    return a == b ? a : K_POISON;
}

// a applied first, then b.  A raw element (cnt > 0) restarts the map.
__device__ __forceinline__ SM combine(SM a, SM b)
{
    if (b.cnt > 0) { b.cnt += a.cnt; return b; }
    SM r;
    r.cnt = a.cnt;
    r.k = merge_k(a.k, b.k);
    if ((a.t | b.t) == 0) { r.d = a.d + b.d; r.t = 0; }
    else {
        const i64 a1 = a.d + a.t;
        const i64 h0 = a.d + b.d + ((a.d & 1) ? b.t : 0);
        const i64 h1 = a1 + b.d + (((a1 + 1) & 1) ? b.t : 0);
        r.d = h0; r.t = (int)(h1 - h0);
    }
    return r;
}

__device__ __forceinline__ SM sm_identity() { return SM{0, 0, 0, K_ID}; }

// exact state (bit pattern of a non-negative double) advanced by a parity map of binade e
__device__ __forceinline__ i64 apply_bits(i64 sb, i64 d, int t, int e, int *bad)
{
    if ((int)(sb >> 52) != e) { *bad = 1; return sb; }
    const i64 r = sb + d + ((sb & 1) ? t : 0);
    if ((int)(r >> 52) != e) { *bad = 1; return sb; }
    return r;
}

// parity map of adding w (> 0) to a state in binade e: two IEEE adds on the binade base
__device__ __forceinline__ SM elem_map(double w, int e)
{
    const i64 base = (i64)e << 52;
    const i64 d0 = __double_as_longlong(__dadd_rn(__longlong_as_double(base), w)) - base;
    const i64 d1 = __double_as_longlong(__dadd_rn(__longlong_as_double(base + 1), w)) - (base + 1);
    return SM{d0, (int)(d1 - d0), 0, e};
}

// ------------------------------------------------------------------ warp / block primitives
__device__ __forceinline__ SM shfl_up_sm(SM v, int o)
{
    SM r;
    r.d = __shfl_up_sync(FULL, v.d, o);
    r.t = __shfl_up_sync(FULL, v.t, o);
    r.cnt = __shfl_up_sync(FULL, v.cnt, o);
    r.k = __shfl_up_sync(FULL, v.k, o);
    return r;
}
__device__ __forceinline__ SM shfl_sm(SM v, int src)
{
    SM r;
    r.d = __shfl_sync(FULL, v.d, src);
    r.t = __shfl_sync(FULL, v.t, src);
    r.cnt = __shfl_sync(FULL, v.cnt, src);
    r.k = __shfl_sync(FULL, v.k, src);
    return r;
}
__device__ __forceinline__ SM warp_incl_scan_sm(SM v, int lane)
{
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        SM t = shfl_up_sm(v, o);
        if (lane >= o) v = combine(t, v);
    }
    return v;
}
__device__ __forceinline__ double warp_incl_scan_d(double v, int lane)
{
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        double t = __shfl_up_sync(FULL, v, o);
        if (lane >= o) v += t;
    }
    return v;
}

// exclusive block scan of doubles (BLOCK threads); *total = block aggregate.
// sh needs BLOCK/32 + 1 entries.  The 8 warp totals are scanned by warp 0 only.
__device__ __forceinline__ double block_excl_scan_d(double v, double *total, double *sh)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const double inc = warp_incl_scan_d(v, lane);
    if (lane == 31) sh[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        const double a = (lane < BLOCK / 32) ? sh[lane] : 0.0;
        const double ai = warp_incl_scan_d(a, lane);
        if (lane < BLOCK / 32) sh[lane] = ai - a;
        if (lane == BLOCK / 32 - 1) sh[BLOCK / 32] = ai;
    }
    __syncthreads();
    const double base = sh[wid];
    *total = sh[BLOCK / 32];
    __syncthreads();
    return base + (inc - v);
}

__device__ __forceinline__ i64 warp_incl_scan_i64(i64 v, int lane)
{
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const i64 t = __shfl_up_sync(FULL, v, o);
        if (lane >= o) v += t;
    }
    return v;
}

// exclusive block scan of int64 (plain sums: the tie-free fast path); sh needs BLOCK/32 + 1 entries
__device__ __forceinline__ i64 block_excl_scan_i64(i64 v, i64 *total, i64 *sh)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const i64 inc = warp_incl_scan_i64(v, lane);
    if (lane == 31) sh[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        const i64 a = (lane < BLOCK / 32) ? sh[lane] : 0;
        const i64 ai = warp_incl_scan_i64(a, lane);
        if (lane < BLOCK / 32) sh[lane] = ai - a;
        if (lane == BLOCK / 32 - 1) sh[BLOCK / 32] = ai;
    }
    __syncthreads();
    const i64 base = sh[wid];
    *total = sh[BLOCK / 32];
    __syncthreads();
    return base + (inc - v);
}

// exclusive block scan of parity maps; *total = block aggregate; sh needs BLOCK/32 + 1 entries
__device__ __forceinline__ SM block_excl_scan_sm(SM v, SM *total, SM *sh)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const SM inc = warp_incl_scan_sm(v, lane);
    if (lane == 31) sh[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        const SM a = (lane < BLOCK / 32) ? sh[lane] : sm_identity();
        const SM ai = warp_incl_scan_sm(a, lane);
        SM ex = shfl_up_sm(ai, 1);
        if (lane == 0) ex = sm_identity();
        if (lane < BLOCK / 32) sh[lane] = ex;
        if (lane == BLOCK / 32 - 1) sh[BLOCK / 32] = ai;
    }
    __syncthreads();
    const SM base = sh[wid];
    *total = sh[BLOCK / 32];
    __syncthreads();
    SM prev = shfl_up_sm(inc, 1);
    if (lane == 0) prev = sm_identity();
    return combine(base, prev);
}

struct Run { i64 lo, hi; int j; int pad; };

// Is the add "state `before` -> `after`" safely inside ONE binade?  The exact running sum lies
// within eb ulps of the approximate one, so both ends must be that far inside binade e.
// Fast test on the high words (eb < 2^33 for n < 2^31), exact 64-bit test only near the edges.
__device__ __forceinline__ bool clean_add(double before, double after, i64 eb, int *e_out)
{
    const int hb = __double2hiint(before), ha = __double2hiint(after);
    const int e = hb >> 20;
    *e_out = e;
    if ((ha >> 20) != e) return false;
    const int mb = hb & 0xFFFFF, ma = ha & 0xFFFFF;
    if (mb >= 2 && ma <= 0xFFFFD) return true;
    const i64 MANT = (1ll << 52) - 1;
    const i64 bb = __double_as_longlong(before), ab = __double_as_longlong(after);
    return ((bb & MANT) >= eb) && ((MANT + 1 - (ab & MANT)) > eb);
}

// ------------------------------------------------------------------ positions
__device__ __forceinline__ double pos_sys(i64 i, double u, double Nd) { return __ddiv_rn(__dadd_rn(u, (double)i), Nd); }

// number of positions strictly below c (systematic): #{ i in [0,N) : fl(fl(u+i)/N) < c }.
// Away from an integer (by tau, which dominates every rounding error of v and of pos_i) this is
// floor(c N - u) + 1; within tau of an integer the positions are evaluated exactly.
__device__ __forceinline__ i64 count_below_sys(double c, double u, i64 N, double Nd, double tau)
{
    const double v = __dadd_rn(__dmul_rn(c, Nd), -u);
    const double r = rint(v);
    if (fabs(v - r) > tau && fabs(v) < 4.0e15) {
        const i64 g = (i64)r + (r > v ? 0 : 1);            // floor(v) + 1
        return g < 0 ? 0 : (g > N ? N : g);
    }
    double g0d = floor(v) + 1.0;
    if (!(g0d > 0.0)) g0d = 0.0;
    if (g0d > Nd) g0d = Nd;
    i64 g = (i64)g0d;
    while (g < N && pos_sys(g, u, Nd) < c) g++;
    while (g > 0 && !(pos_sys(g - 1, u, Nd) < c)) g--;
    return g;
}

__device__ __forceinline__ double pos_str(i64 i, const double *U, double Nd) { return __ddiv_rn(__dadd_rn(U[i], (double)i), Nd); }

// number of positions strictly below c (stratified; positions are non-decreasing in i)
__device__ __forceinline__ i64 count_below_str(double c, const double *U, i64 N, double Nd)
{
    double v = floor(__dmul_rn(c, Nd));
    if (!(v > 1.0)) v = 1.0;
    if (v > Nd) v = Nd;
    i64 g = (i64)v - 1;                      // candidates start two below the real-valued crossing
    if (g < 0) g = 0;
    while (g < N && pos_str(g, U, Nd) < c) g++;
    while (g > 0 && !(pos_str(g - 1, U, Nd) < c)) g--;
    return g;
}

}  // namespace rs
}  // namespace bke
