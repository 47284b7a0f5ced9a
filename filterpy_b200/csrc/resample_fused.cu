// resample_fused.cu — systematic / stratified resampling of a whole array of weights, normalised on
// the fly, as ONE single-pass kernel: every weight is read from HBM once (8 B in, 4 B out per
// particle).  It is the engine of bke_resample_normalized.
//
//   indexes[i] = #{ j : c_j <= pos_i },  c_j = fl(c_{j-1} + w_j)   (filterpy/monte_carlo/resampling.py:141-149)
//   pos_i = fl(fl(u + i) / N) (:139)  or  fl(fl(U_i + i) / N) (:103)
//
// The running sum is reproduced EXACTLY (resample_common.cuh: inside one binade adding w is the
// integer map bits(S) -> bits(S) + d[parity]); what is new here is how the tiles are chained:
// a decoupled look-back in TWO stages, both on one 64-bit status word per tile.
//
//   stage 1 (producer warp)  approximate fp64 tile sum -> approximate prefix `tp`  (which binade
//            the tile lives in, and which adds might leave it)
//   stage 2 (consumer warps) the tile's parity map D computed in that binade -> exact state S_in
//            (bit pattern of the reference's running sum before the tile), then every c_j,
//            the output range of every particle and the index expansion.
//
// CTA = NW consumer warps + 1 producer warp, persistent, tiles handed out by an atomic counter
// (so a tile only ever waits for tiles that are already running).  The producer warp claims the
// next tile, pulls its 16*NW*32 weights into shared memory with ONE 2-D TMA copy (128-byte
// swizzle: thread t reads its 16 consecutive weights with conflict-free LDS.128), sums them,
// publishes / resolves stage 1 and hands the stage over while the consumers still work on the
// previous tile: HBM latency and the first look-back are off the consumers' critical path.
// A tile that is not "clean" (a possible binade crossing, ties) takes slow_tile(): the old
// raw-element / segment walk, started before S_in arrives so that only the short walk is serial.
//
// Expansion: each particle with >= 1 copies stores (local index + 1) at its first output slot of
// a zeroed shared-memory window; a max-scan over the slots fills the runs (no divergent copy
// loop), and every thread leaves with 16-byte stores of 20 consecutive indexes.
//
// Everything is verified with the exact values (tile start / end inside the assumed binade); a
// failed check or a negative / non-finite weight switches to the literal sequential kernel.
#include <cuda.h>
#include "resample_common.cuh"
#include "resample_fused.cuh"

namespace bke {
namespace rs {

// ------------------------------------------------------------------ status words
// st1[i], st2[i] describe tile i-1; entry 0 is the empty sum before the first tile (INCLUSIVE).
//   st1: bits of an fp64 sum with the two lowest mantissa bits replaced by the flag
//        (1 = this tile's sum, 2 = sum of everything up to and including this tile)
//   st2: bit 63 = INCLUSIVE: bits 0..62 = exact running sum after the tile (a non-negative double)
//        bit 62 = AGGREGATE: bits 0..59 = d0 of the tile's parity map, bits 60..61 = t + 1
constexpr u64 ST1_AGG = 1, ST1_INCL = 2;
constexpr u64 ST2_INCL = 1ull << 63, ST2_AGG = 1ull << 62;
constexpr int SPIN_LIMIT = 1 << 22;

__device__ __forceinline__ u64 st2_pack_agg(i64 d, int t) { return ST2_AGG | ((u64)(t + 1) << 60) | ((u64)d & ((1ull << 60) - 1)); }

// Look-back windows: every round a warp fetches 32 * LBK status words at once (ONE L2 round trip),
// walks them in groups of 32 from the nearest predecessor outwards and stops at the nearest
// INCLUSIVE word.  All tiles of a persistent grid start together, so a tile is typically a few
// hundred tiles ahead of the inclusive frontier: the width of the window, not the number of
// resident CTAs, sets how many round trips a look-back costs.
constexpr int LBK = 4;

// a blocked round (an unpublished word in front of the nearest inclusive one): poll again, and give up
// after SPIN_LIMIT rounds or once any look-back has given up (the result then comes from the fallback)
__device__ __forceinline__ bool f_blocked(FHeader *hdr, int &spins)
{
    spins++;
    if ((spins & 1023) == 0 && *reinterpret_cast<volatile int *>(&hdr->timeout)) return true;
    if (spins >= SPIN_LIMIT) { hdr->timeout = 1; hdr->fallback = 1; return true; }
    return false;
}

// stage 1: approximate sum of everything before tile t (all 32 lanes of the producer warp)
__device__ __forceinline__ double f_lookback_sum(const FParams &p, int t, int lane)
{
    double part = 0.0;                                     // this lane's share; reduced once at the end
    int idx = t - lane;                                    // st1 index of tile t-1-lane (group 0 of the round)
    int spins = 0;
    bool done = false;
    while (!done) {
        u64 v[LBK];
#pragma unroll
        for (int j = 0; j < LBK; j++) {
            const int i = idx - 32 * j;
            v[j] = ST1_INCL;                               // before entry 0: 0.0, inclusive
            if (i >= 0) v[j] = f_ld(p.st1 + i);
        }
        bool blocked = false;
#pragma unroll
        for (int j = 0; j < LBK; j++) {
            if (!done && !blocked) {
                const unsigned incl = __ballot_sync(FULL, (v[j] & 3) == ST1_INCL);
                const unsigned empty = __ballot_sync(FULL, (v[j] & 3) == 0);
                const int first = incl ? __ffs(incl) - 1 : 32;
                const unsigned closer = first >= 32 ? FULL : ((1u << first) - 1u);
                if (empty & closer) blocked = true;
                else {
                    if (lane <= first) part += __longlong_as_double((i64)(v[j] & ~3ull));
                    if (incl) done = true; else idx -= 32;
                }
            }
        }
        if (blocked && f_blocked(p.hdr, spins)) break;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(FULL, part, o);
    return part;
}

// stage 2: exact state before tile t (all 32 lanes of a warp).  The aggregates between the nearest
// inclusive predecessor and this tile are composed in tile order; with tie-free maps (t = 0, the
// normal case) that is a plain int64 sum, kept per lane and reduced once.
__device__ __forceinline__ i64 f_lookback_state(const FParams &p, int t, int lane)
{
    i64 part = 0;                                          // tie-free mode: this lane's share of the sum
    bool general = false;                                  // a map with ties was met: ordered composition from here on
    i64 acc_d = 0; int acc_t = 0;                          // general mode: composite of everything nearer (applied LAST)
    i64 S = 0;
    int idx = t - lane;
    int spins = 0;
    bool done = false;
    while (!done) {
        u64 v[LBK];
#pragma unroll
        for (int j = 0; j < LBK; j++) {
            const int i = idx - 32 * j;
            v[j] = ST2_INCL;
            if (i >= 0) v[j] = f_ld(p.st2 + i);
        }
        bool blocked = false;
#pragma unroll
        for (int j = 0; j < LBK; j++) {
            if (!done && !blocked) {
                const unsigned incl = __ballot_sync(FULL, (v[j] & ST2_INCL) != 0);
                const unsigned empty = __ballot_sync(FULL, (v[j] & (ST2_INCL | ST2_AGG)) == 0);
                const int first = incl ? __ffs(incl) - 1 : 32;
                const unsigned closer = first >= 32 ? FULL : ((1u << first) - 1u);
                if (empty & closer) { blocked = true; continue; }
                i64 d = 0; int tt = 0;
                if (lane < first) { d = (i64)(v[j] & ((1ull << 60) - 1)); tt = (int)((v[j] >> 60) & 3) - 1; }
                const unsigned ties = __ballot_sync(FULL, tt != 0);
                if (!general && ties == 0) part += d;
                else {
                    if (!general) {
                        general = true;
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(FULL, part, o);
                        acc_d = part; acc_t = 0;
                    }
                    // ordered: lane L holds tile (..)-L, i.e. higher lanes are applied first
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const i64 pd = __shfl_down_sync(FULL, d, o);
                        const int pt = __shfl_down_sync(FULL, tt, o);
                        if (lane + o < 32) {
                            const SM r = combine(SM{pd, pt, 0, K_ID}, SM{d, tt, 0, K_ID});
                            d = r.d; tt = r.t;
                        }
                    }
                    d = __shfl_sync(FULL, d, 0); tt = __shfl_sync(FULL, tt, 0);
                    const SM r = combine(SM{d, tt, 0, K_ID}, SM{acc_d, acc_t, 0, K_ID});   // this group lies before everything nearer
                    acc_d = r.d; acc_t = r.t;
                }
                if (incl) { S = (i64)(__shfl_sync(FULL, v[j], first) & ~ST2_INCL); done = true; }
                else idx -= 32;
            }
        }
        if (blocked && f_blocked(p.hdr, spins)) break;
    }
    if (!general) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(FULL, part, o);
        acc_d = part; acc_t = 0;
    }
    return S + acc_d + ((S & 1) ? acc_t : 0);
}

// ------------------------------------------------------------------ shared memory
enum { TM_FAST = 0, TM_SLOW = 1, TM_BAD = 2 };                       // what the consumers do with a tile at emit time
enum { TK_CLEAN = 0, TK_CROSS = 1, TK_TIES = 2, TK_BAD = 3 };        // what stage 1 found out about it
constexpr int MAX_CROSS = 24;                                        // crossing rows resolved by the chain warp
constexpr int RING = 8;                                              // tiles a CTA has between "fronted" and "emitted"
// NW consumer warps per CTA (+ 4 helper warps), F_CTAS CTAs per SM (what the shared memory allows),
// and the emit runs DELTA tiles of the CTA behind the front
constexpr int NW = 8, NT = NW * 32, F_TILE = NT * F_IPT, WIN = NT * F_SPT;
constexpr int F_CTAS = 2, DELTA = 3;
static_assert(DELTA + 2 <= RING, "ring too small");

// one tile of this CTA on its way from front (sum + map) to emit
struct FSlot {
    int t;                  // tile, -1 = end of work
    int eg;                 // binade the front formed its map in (a guess: the binade the chain saw last)
    int bad, tie;           // front: invalid weights / an exact tie somewhere
    double tot;             // front: approximate sum of the tile
    i64 D;                  // front (or C1, when the guess was wrong): tie-free parity map of the tile in binade eg / e0
    i64 D1; int tie1, pad1; // front: the same in binade eg + 1 (a running sum only ever moves up)
    int kind, e0;           // C1
    int mode, good, cross;  // C2: what emit does; verified; per-row start states are in the crossing pool
    int pad;
    i64 S_in, lo, cnt;      // C2: exact state before the tile, its output range
};

struct FSmem {
    double wf[F_TILE];                 // front buffer  \\ TMA destinations (128-byte swizzle): must stay first,
    double we[F_TILE];                 // emit buffer   /  1024-aligned
    int win[WIN];                      // output window (all zero between tiles)
    i64 xrow[NT];                      // crossing pool: exact state before every row of ONE tile that leaves its binade
    unsigned xmask[NT / 32];           // ... and the rows (consumer threads) that are walked with true adds
    struct FPart { double tot; i64 D; i64 D1; int tie; int tie1; int bad; int pad; } fpart[2][NW];      // front: per-warp partials (double buffered)
    i64 warp_i[NW];
    double warp_d[NW];
    SM warp_sm[NW];
    int warp_max[NW];
    uint64_t full_f, empty_f, full_e, empty_e, xfree;
    uint64_t claimed[RING], fronted[RING], mapped[RING], resolved[RING], freed[RING];
    FSlot ring[RING];
    int e_last;                        // binade of the last tile the chain resolved (the front's guess)
    i64 bc_S_in, bc_lo, bc_cnt;
    int bc_ok, bc_skip;
    // slow path (tiles with ties)
    i64 segstate[RMAX + 1];
    i64 segd[RMAX + 1];
    double wraw[RMAX];
    int segk[RMAX + 1];
    int segt[RMAX + 1];
    int first_raw[NT + 1];
    i64 tstart[NT];
};


__device__ __forceinline__ double f_scan_d(double v, double *total, double *sh, int lane, int wid)
{
    const double inc = warp_incl_scan_d(v, lane);
    if (lane == 31) sh[wid] = inc;
    f_bar<NT>();
    double base = 0.0, tot = 0.0;
#pragma unroll
    for (int i = 0; i < NW; i++) { const double x = sh[i]; if (i < wid) base += x; tot += x; }
    f_bar<NT>();
    *total = tot;
    return base + (inc - v);
}

__device__ __forceinline__ SM f_scan_sm(SM v, SM *total, SM *sh, int lane, int wid)
{
    const SM inc = warp_incl_scan_sm(v, lane);
    if (lane == 31) sh[wid] = inc;
    f_bar<NT>();
    SM base = sm_identity(), tot = sm_identity();
    for (int i = 0; i < NW; i++) { const SM x = sh[i]; if (i < wid) base = combine(base, x); tot = combine(tot, x); }
    f_bar<NT>();
    *total = tot;
    SM prev = shfl_up_sm(inc, 1);
    if (lane == 0) prev = sm_identity();
    return combine(base, prev);
}

template <int MODE>
__device__ __forceinline__ i64 f_count_below(const FParams &p, double c)
{
    const double Ngd = (double)p.n;
    return (MODE == F_STRAT) ? count_below_str(c, p.U, p.n, Ngd) : count_below_sys(c, p.u, p.n, Ngd, p.tau);
}

__device__ __forceinline__ void f_put_index(const FParams &p, i64 out_begin, i64 o, int value)
{
    const i64 rel = o - out_begin;
    if (rel >= 0 && rel < p.n) p.idx[rel] = value;
    else p.hdr->cap_overflow = 1;
}

// one lane, after the tile's exact end state is known and published: the tile's output range
// [lo, lo + cnt) and, for the last tile, the call's bookkeeping
template <int MODE>
__device__ __forceinline__ void f_finish_tile(const FParams &p, int t, i64 S_in, i64 S_out, int &good, i64 &lo, i64 &cnt)
{
    lo = 0; cnt = 0;
    if (good) {
        lo = f_count_below<MODE>(p, __longlong_as_double(S_in));
        cnt = f_count_below<MODE>(p, __longlong_as_double(S_out)) - lo;
        if (cnt < 0) { cnt = 0; good = 0; }
    }
    if (!good) { p.hdr->fallback = 1; p.hdr->chain_bad = 1; }
    if (t == p.T - 1) {
        if (p.cumsum_last) *p.cumsum_last = __longlong_as_double(S_out);
        i64 O1 = lo + cnt;
        if (O1 < p.n) {                                    // resampling.py:145 would raise IndexError
            p.hdr->overflow = (int)(p.n - O1 > 0x7fffffff ? 0x7fffffff : p.n - O1);
            const int r = atomicAdd(&p.hdr->n_runs, 1);
            if (r < p.max_runs) p.runs[r] = Run{O1, p.n, (int)(p.n - 1), 0};
            O1 = p.n;
        }
        p.hdr->out_end = O1;
    }
}

// ------------------------------------------------------------------ slow path: ties, raw elements, dense raw zones
// Leaves the exact c_j (bit patterns) of the tile in the stage buffer, at the positions of the
// weights they belong to; returns 1 if the tile verified.  Everything up to the segment export
// runs BEFORE the exact start state is known; only the walk over <= RMAX segments is serial.
template <int MODE>
__device__ __noinline__ int f_slow_tile(const FParams &p, FSmem &sm, int t, i64 S_in_known)
{
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    unsigned char *sb = reinterpret_cast<unsigned char *>(sm.we);
    double w[F_IPT];
#pragma unroll
    for (int c = 0; c < F_IPT / 2; c++) {
        const double2 v = *reinterpret_cast<const double2 *>(sb + f_swz(tid, c));
        w[2 * c] = v.x; w[2 * c + 1] = v.y;
    }
    double ssum = 0.0;
#pragma unroll
    for (int k = 0; k < F_IPT; k++) ssum += w[k];
    double tot;
    // the exact state before the tile is known (chain warp C2): it is the "approximate" prefix of the classification
    double before = __longlong_as_double(S_in_known) + f_scan_d(ssum, &tot, sm.warp_d, lane, wid);
    SM inc[F_IPT];
    int ek[F_IPT];
    SM run = sm_identity();
#pragma unroll
    for (int k = 0; k < F_IPT; k++) {
        const double after = before + w[k];
        SM el;
        if (w[k] == 0.0) { el = sm_identity(); ek[k] = K_ID; }          // fl(S + 0) = S in every binade
        else {
            int e;
            if (clean_add(before, after, p.eb, &e)) { el = elem_map(w[k], e); ek[k] = e; }
            else { el = SM{0, 0, 1, K_ID}; ek[k] = -1; }
        }
        run = combine(run, el);
        inc[k] = run;
        before = after;
    }
    SM total;
    const SM excl = f_scan_sm(run, &total, sm.warp_sm, lane, wid);
#pragma unroll
    for (int k = 0; k < F_IPT; k++) inc[k] = combine(excl, inc[k]);
    const int nraw = total.cnt;
    int bad = 0;
    if (nraw > 0 && nraw <= RMAX) {
        sm.first_raw[tid] = (ek[0] == -1);
        if (tid == 0) sm.first_raw[NT] = 1;                 // the tile end closes the last segment
        for (int q = tid; q <= RMAX; q += NT) { sm.segk[q] = -1; sm.segt[q] = 0; sm.segd[q] = 0; }
        f_bar<NT>();
#pragma unroll
        for (int k = 0; k < F_IPT; k++) {
            const int seg = inc[k].cnt;
            if (ek[k] == -1) {
                sm.wraw[seg - 1] = w[k];                    // the raw element that opens segment `seg`
            } else {
                const bool next_raw = (k + 1 < F_IPT) ? (ek[k + 1] == -1) : (sm.first_raw[tid + 1] != 0);
                if (next_raw) {
                    if (inc[k].k == K_POISON) bad = 1;
                    sm.segk[seg] = inc[k].k == K_ID ? -1 : inc[k].k;    // identity segments are skipped
                    sm.segt[seg] = inc[k].t;
                    sm.segd[seg] = inc[k].d;
                }
            }
        }
    }
    f_bar<NT>();
    if (wid == 0) {
        const i64 S_in = S_in_known;
        if (lane == 0) {
            int wbad = 0;
            i64 S_out;
            if (nraw == 0) {
                S_out = total.k >= 0 ? apply_bits(S_in, total.d, total.t, total.k, &wbad) : S_in;
                if (total.k == K_POISON) wbad = 1;
                sm.segstate[0] = S_in;
            } else if (nraw <= RMAX) {
                i64 S = S_in;
                for (int q = 0; q <= nraw; q++) {
                    sm.segstate[q] = S;
                    if (sm.segk[q] >= 0) S = apply_bits(S, sm.segd[q], sm.segt[q], sm.segk[q], &wbad);
                    if (q < nraw) S = __double_as_longlong(__dadd_rn(__longlong_as_double(S), sm.wraw[q]));
                }
                S_out = S;
                atomicAdd(&p.hdr->n_unclean, 1);
            } else {
                // a dense zone of raw elements (tiny weights next to a binade boundary): true adds, one by one
                double acc = __longlong_as_double(S_in);
                for (int th = 0; th < NT; th++) {
                    sm.tstart[th] = __double_as_longlong(acc);
#pragma unroll
                    for (int c = 0; c < F_IPT / 2; c++) {
                        const double2 v = *reinterpret_cast<const double2 *>(sb + f_swz(th, c));
                        acc = __dadd_rn(acc, v.x);
                        acc = __dadd_rn(acc, v.y);
                    }
                }
                S_out = __double_as_longlong(acc);
                atomicAdd(&p.hdr->n_seq, 1);
            }
            f_st(p.st2 + t + 1, ST2_INCL | (u64)S_out);
            atomicAdd(&p.hdr->n_slow, 1);
            int good = !wbad;
            i64 lo, cnt;
            f_finish_tile<MODE>(p, t, S_in, S_out, good, lo, cnt);
            sm.bc_S_in = S_in; sm.bc_lo = lo; sm.bc_cnt = cnt; sm.bc_ok = good;
        }
    }
    f_bar<NT>();
    i64 cb[F_IPT];
    if (nraw > RMAX) {
        double acc = __longlong_as_double(sm.tstart[tid]);
#pragma unroll
        for (int k = 0; k < F_IPT; k++) { acc = __dadd_rn(acc, w[k]); cb[k] = __double_as_longlong(acc); }
    } else {
#pragma unroll
        for (int k = 0; k < F_IPT; k++) {
            const i64 S0 = sm.segstate[inc[k].cnt];
            if (inc[k].k == K_POISON) bad = 1;
            // a raw element: the segment it opens starts at its own result; only zeros so far: unchanged
            cb[k] = (ek[k] == -1 || inc[k].k < 0) ? S0 : apply_bits(S0, inc[k].d, inc[k].t, inc[k].k, &bad);
        }
    }
    if (bad) { p.hdr->fallback = 1; p.hdr->chain_bad = 2; }
#pragma unroll
    for (int c = 0; c < F_IPT / 2; c++)
        *reinterpret_cast<longlong2 *>(sb + f_swz(tid, c)) = make_longlong2(cb[2 * c], cb[2 * c + 1]);
    f_fence_proxy_async();                // generic-proxy writes to a stage the TMA engine will refill
    return f_bar_and<NT>(!bad && sm.bc_ok);
}

// read this thread's F_SPT window slots (and clear them), running maximum, block max-scan:
// m[i] = marker (local particle index + 1) of the particle that owns slot tid*F_SPT + i
__device__ __forceinline__ void f_window_scan(FSmem &sm, int tid, int lane, int wid, int (&m)[F_SPT])
{
    int4 *wv = reinterpret_cast<int4 *>(sm.win) + tid * (F_SPT / 4);
#pragma unroll
    for (int i = 0; i < F_SPT / 4; i++) {
        const int4 q = wv[i];
        m[4 * i] = q.x; m[4 * i + 1] = q.y; m[4 * i + 2] = q.z; m[4 * i + 3] = q.w;
    }
#pragma unroll
    for (int i = 0; i < F_SPT / 4; i++) wv[i] = make_int4(0, 0, 0, 0);
#pragma unroll
    for (int i = 1; i < F_SPT; i++) m[i] = max(m[i], m[i - 1]);
    int incm = m[F_SPT - 1];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(FULL, incm, o); if (lane >= o) incm = max(incm, y); }
    int basem = __shfl_up_sync(FULL, incm, 1);
    if (lane == 0) basem = 0;
    if (lane == 31) sm.warp_max[wid] = incm;
    f_bar<NT>();
#pragma unroll
    for (int i = 0; i < NW; i++) { const int x = sm.warp_max[i]; if (i < wid) basem = max(basem, x); }
#pragma unroll
    for (int i = 0; i < F_SPT; i++) m[i] = max(m[i], basem);
}

// Row sums of the tie-free parity map of tile t in binade e, read from GLOBAL memory (the rare paths
// of the chain warps: a wrong binade guess, a tile that leaves its binade).  Lane L owns rows
// L, L + 32, ...: rs[i] belongs to row 32 i + L (0 for rows < r0); bit i of the result is set when
// that row holds an exact tie.
__device__ __noinline__ unsigned f_row_sums_g(const FParams &p, int t, int e, int r0, int lane, double divisor, i64 (&rs)[NW])
{
    const i64 base = (i64)e << 52;
    const double B0 = __longlong_as_double(base), B1 = __longlong_as_double(base + 1);
    unsigned ties = 0;
#pragma unroll
    for (int i = 0; i < NW; i++) {
        const int r = i * 32 + lane;
        i64 racc = 0;
        unsigned tie = 0;
        if (r >= r0) {
            const i64 j0 = (i64)t * (NW * 32 * F_IPT) + (i64)r * F_IPT;
            double vv[F_IPT];
#pragma unroll
            for (int k = 0; k < F_IPT; k++) vv[k] = (j0 + k < p.n) ? p.w[j0 + k] : 0.0;
#pragma unroll
            for (int k = 0; k < F_IPT; k++) {
                double v = vv[k];
                if (p.div) v = __ddiv_rn(v, divisor);
                const i64 x0 = __double_as_longlong(__dadd_rn(B0, v)), x1 = __double_as_longlong(__dadd_rn(B1, v));
                tie |= ((unsigned)x0 + 1u) ^ (unsigned)x1;             // d1 != d0: an exact tie
                racc += x0 - base;
            }
        }
        rs[i] = racc;
        if (tie) ties |= 1u << i;
    }
    return ties;
}

// A tile that may leave its binade, resolved from the EXACT state before it (chain warp C2, weights
// read from global memory): rows whose adds all stay in the binade of their start state are integer
// maps; the row that leaves it is walked with true adds; the rows after it are maps of the next
// binade, and so on.  On success sm.xrow[r] = exact state before row r, sm.xmask marks the walked
// rows, *S_out = state after the tile.  false: a tie in a mapped row, or more than MAX_CROSS crossings.
__device__ __noinline__ bool f_resolve_exact(const FParams &p, FSmem &sm, int t, i64 S_in, i64 *S_out, int lane, double divisor)
{
    if (lane < NT / 32) sm.xmask[lane] = 0;
    __syncwarp();
    int r0 = 0;
    i64 S = S_in;
    for (int round = 0; r0 < NT; round++) {
        if (round > MAX_CROSS) return false;
        const int e = (int)(S >> 52);
        i64 rsum[NW];
        const unsigned ties = f_row_sums_g(p, t, e, r0, lane, divisor, rsum);
        i64 carry = S;                                     // state before row 32 i (rows < r0 contribute 0)
        int found = -1;
        i64 S_row = 0;
        bool tie_used = false;
#pragma unroll
        for (int i = 0; i < NW; i++) {
            if (found >= 0) continue;
            const int r = i * 32 + lane;
            const i64 rs = rsum[i];
            const i64 inc = warp_incl_scan_i64(rs, lane);
            const i64 end_state = carry + inc, start_state = end_state - rs;
            const bool leaves = r >= r0 && (int)(end_state >> 52) != e;
            const unsigned m = __ballot_sync(FULL, leaves);
            const int fc = m ? __ffs(m) - 1 : 32;
            if (r >= r0 && lane <= fc) sm.xrow[r] = start_state;       // rows up to and including the leaving one start here
            if (r >= r0 && lane < fc && ((ties >> i) & 1)) tie_used = true;   // a tie in a row that is applied as a map
            if (m) { found = i * 32 + fc; S_row = __shfl_sync(FULL, start_state, fc); }
            carry = __shfl_sync(FULL, end_state, 31);
        }
        if (__any_sync(FULL, tie_used)) return false;
        if (found < 0) { *S_out = carry; return true; }
        // the row that leaves the binade: true adds, one by one
        double acc = __longlong_as_double(S_row);
        {
            const i64 j0 = (i64)t * (NT * F_IPT) + (i64)found * F_IPT;
#pragma unroll 4
            for (int k = 0; k < F_IPT; k++) {
                double v = (j0 + k < p.n) ? p.w[j0 + k] : 0.0;
                if (p.div) v = __ddiv_rn(v, divisor);
                acc = __dadd_rn(acc, v);
            }
        }
        if (lane == 0) sm.xmask[found >> 5] |= 1u << (found & 31);
        __syncwarp();
        S = __double_as_longlong(acc);
        r0 = found + 1;
    }
    *S_out = S;
    return true;
}

// ------------------------------------------------------------------ the kernel
// Roles inside a CTA (NW consumer warps + 3 helper warps):
//   consumers  iteration k: FRONT tile k of this CTA (sum, validation, parity map in the guessed
//              binade -> stage-1 AGGREGATE published at once), then EMIT tile k - DELTA (by then the
//              chain has resolved its exact start state; its weights come back from L2, not HBM)
//   L          claims tiles, TMA-loads the front buffer (from HBM) and the emit buffer (from L2)
//   C1         stage-1 look-back: approximate prefix -> binade -> stage-2 AGGREGATE
//   C2         stage-2 look-back: exact state before the tile -> INCLUSIVE; tiles that leave their binade
// The chain (C1, C2) runs DELTA tiles per CTA — several hundred tiles of the grid — ahead of the
// emit front, so a look-back never stalls the warps that do the work.
template <int MODE>
__global__ void __launch_bounds__(NT + 128, F_CTAS)
k_fused(const __grid_constant__ CUtensorMap wmap, const FParams p)
{
    extern __shared__ __align__(1024) unsigned char f_smem_raw[];
    FSmem &sm = *reinterpret_cast<FSmem *>(f_smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;

    if (tid == 0) {
        f_mbar_init(&sm.full_f, 1); f_mbar_init(&sm.empty_f, NW); f_mbar_init(&sm.full_e, 1); f_mbar_init(&sm.empty_e, NW);
        f_mbar_init(&sm.xfree, NW);
        for (int i = 0; i < RING; i++) {
            f_mbar_init(&sm.claimed[i], 1); f_mbar_init(&sm.fronted[i], 1); f_mbar_init(&sm.mapped[i], 1); f_mbar_init(&sm.resolved[i], 1); f_mbar_init(&sm.freed[i], NW);
        }
        sm.e_last = 1022;              // binade [0.5, 1): where a normalised running sum spends most of its life
        f_fence_mbar_init();
    }
    for (int q = tid; q < WIN; q += NT + 128) sm.win[q] = 0;
    __syncthreads();

    const double divisor = p.div ? *p.div : 1.0;
    const bool tail_generic = (p.n & 15) != 0;             // the last tile of a ragged array is staged by hand

    if (wid == NW || wid == NW + 3) {
        // ============================================================ loader warps: LF (front buffer, from HBM; claims the tiles)
        // and LE (emit buffer: the same tiles again DELTA iterations later, from L2).  Both block on mbarriers only.
        auto load_tile = [&](int t, double *dst, uint64_t *full) {
            if (p.use_tma && !(tail_generic && t == p.T - 1)) {
                if (lane == 0) { f_mbar_expect_tx(full, F_TILE * 8); f_tma_load_2d(dst, &wmap, 0, t * NT, full); }
            } else {
                unsigned char *sb = reinterpret_cast<unsigned char *>(dst);
                const i64 j0 = (i64)t * F_TILE;
                for (int i = lane; i < F_TILE; i += 32) {
                    const i64 j = j0 + i;
                    const double v = (j < p.n) ? p.w[j] : 0.0;
                    *reinterpret_cast<double *>(sb + f_swz(i >> 4, (i >> 1) & 7) + (i & 1) * 8) = v;
                }
                f_fence_proxy_async();                     // generic-proxy writes to a buffer the TMA engine also fills
                __syncwarp();
                if (lane == 0) f_mbar_arrive(full);
            }
        };
        if (wid == NW) {
            for (int kf = 0;; kf++) {
                // front load kf: its ring slot must be free, the front buffer consumed
                const int slot = kf % RING, use = kf / RING;
                if (use > 0) f_mbar_wait(&sm.freed[slot], (use - 1) & 1);
                if (kf > 0) f_mbar_wait(&sm.empty_f, (kf - 1) & 1);
                int t = 0;
                if (lane == 0) t = atomicAdd(&p.hdr->tile_counter, 1);
                t = __shfl_sync(FULL, t, 0);
                if (t >= p.T) t = -1;
                if (lane == 0) {
                    sm.ring[slot].eg = *reinterpret_cast<volatile int *>(&sm.e_last);
                    sm.ring[slot].t = t;
                }
                __syncwarp();
                if (lane == 0) f_mbar_arrive(&sm.claimed[slot]);       // LE may read the slot's tile
                if (t < 0) { if (lane == 0) f_mbar_arrive(&sm.full_f); break; }      // end of work travels down the pipeline
                load_tile(t, sm.wf, &sm.full_f);
            }
        } else {
            for (int ke = 0;; ke++) {
                const int slot = ke % RING, use = ke / RING;
                f_mbar_wait(&sm.claimed[slot], use & 1);
                const int t = sm.ring[slot].t;
                if (t < 0) break;
                if (ke > 0) f_mbar_wait(&sm.empty_e, (ke - 1) & 1);
                load_tile(t, sm.we, &sm.full_e);
            }
        }
        return;
    }
    if (wid == NW + 1) {
        // ============================================================ chain warp C1 (stage 1)
        // approximate prefix -> which binade the tile lives in -> for a tile deep inside one binade the
        // stage-2 AGGREGATE (its parity map D), published right away (C1 never waits for stage 2)
        for (int k = 0;; k++) {
            const int si = k % RING, use = k / RING;
            FSlot &sl = sm.ring[si];
            f_mbar_wait(&sm.fronted[si], use & 1);
            const int t = sl.t;
            if (t < 0) {
                if (lane == 0) f_mbar_arrive(&sm.mapped[si]);
                break;
            }
            const double tot = sl.tot;
            const int bad = sl.bad, eg = sl.eg;
            int any_tie = sl.tie;
            i64 D = sl.D;
            const double tp = f_lookback_sum(p, t, lane);
            if (lane == 0) f_st(p.st1 + t + 1, ((u64)__double_as_longlong(tp + tot) & ~3ull) | ST1_INCL);
            int e0;
            const bool ca = clean_add(tp, tp + tot, p.eb, &e0);
            int kind = bad ? TK_BAD : ((ca || tot == 0.0) ? TK_CLEAN : TK_CROSS);
            if (kind == TK_CLEAN) {
                if (tot == 0.0) { D = 0; any_tie = 0; }
                else if (e0 == eg + 1) { D = sl.D1; any_tie = sl.tie1; }      // the front's second candidate
                else if (e0 != eg) {
                    // the front's guess was wrong (first tiles, a new binade): the map again, in binade e0
                    i64 rsum[NW];
                    any_tie = f_row_sums_g(p, t, e0, 0, lane, divisor, rsum) != 0;
                    any_tie = __any_sync(FULL, any_tie);
                    D = 0;
#pragma unroll
                    for (int i = 0; i < NW; i++) D += rsum[i];
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) D += __shfl_xor_sync(FULL, D, o);
                }
                if (tot != 0.0 && lane == 0) sm.e_last = e0;
                if (any_tie) kind = TK_TIES;               // ties: the general parity maps of the slow path
            }
            if (kind == TK_CLEAN && lane == 0) f_st(p.st2 + t + 1, st2_pack_agg(D, 0));
            if (lane == 0) { sl.kind = kind; sl.e0 = e0; sl.D = D; }
            __syncwarp();
            if (lane == 0) f_mbar_arrive(&sm.mapped[si]);
        }
        return;
    }
    if (wid == NW + 2) {
        // ============================================================ chain warp C2 (stage 2)
        // exact state before the tile; tiles that may leave their binade are resolved here, exactly,
        // from that state (no margins)
        int xuse = 0;
        for (int k = 0;; k++) {
            const int si = k % RING, use = k / RING;
            FSlot &sl = sm.ring[si];
            f_mbar_wait(&sm.mapped[si], use & 1);
            const int t = sl.t;
            if (t < 0) {
                if (lane == 0) f_mbar_arrive(&sm.resolved[si]);
                break;
            }
            const int kind = sl.kind, e0 = sl.e0;
            const double tot = sl.tot;
            const i64 D = sl.D;
            const i64 S_in = f_lookback_state(p, t, lane);
            int mode, good = 1, cross = 0;
            i64 S_out = S_in, lo = 0, cnt = 0;
            if (kind == TK_CLEAN) {
                S_out = S_in + D;
                good = (tot == 0.0) || ((int)(S_in >> 52) == e0 && (int)(S_out >> 52) == e0);
                mode = TM_FAST;
            } else if (kind == TK_BAD) {
                mode = TM_BAD;                             // invalid weights: the sequential kernel will produce the result
            } else {
                mode = TM_SLOW;                            // ties / too many crossings: the consumers' general path publishes
                if (kind == TK_CROSS) {
                    if (xuse > 0) f_mbar_wait(&sm.xfree, (xuse - 1) & 1);       // the pool's previous tile has been emitted
                    if (f_resolve_exact(p, sm, t, S_in, &S_out, lane, divisor)) {
                        mode = TM_FAST; cross = 1; xuse++;
                        if (lane == 0) { atomicAdd(&p.hdr->n_unclean, 1); sm.e_last = (int)(S_out >> 52); }
                    }
                }
            }
            // a failed resolve leaves the pool unused: keep xfree's phase in step by not counting the use
            if (lane == 0) {
                if (mode != TM_SLOW) f_st(p.st2 + t + 1, ST2_INCL | (u64)S_out);
                if (mode == TM_FAST) f_finish_tile<MODE>(p, t, S_in, S_out, good, lo, cnt);
                sl.mode = mode; sl.good = good; sl.cross = cross; sl.S_in = S_in; sl.lo = lo; sl.cnt = cnt;
            }
            __syncwarp();
            if (lane == 0) f_mbar_arrive(&sm.resolved[si]);
        }
        return;
    }

    // ================================================================ consumer warps
    const i64 out_begin = p.hdr->out_begin;
    const double Nd = (double)p.n;
    bool front_done = false;
    for (int k = 0;; k++) {
        // ------------------------------------------------------------ FRONT tile k of this CTA
        if (!front_done) {
            f_mbar_wait(&sm.full_f, k & 1);
            FSlot &sl = sm.ring[k % RING];
            const int t = sl.t;
            if (t < 0) {
                front_done = true;
                if (tid == 0) f_mbar_arrive(&sm.fronted[k % RING]);
            } else {
                const unsigned char *sb = reinterpret_cast<const unsigned char *>(sm.wf);
                double w[F_IPT];
#pragma unroll
                for (int c = 0; c < F_IPT / 2; c++) {
                    const double2 v = *reinterpret_cast<const double2 *>(sb + f_swz(tid, c));
                    w[2 * c] = v.x; w[2 * c + 1] = v.y;
                }
                const int eg = sl.eg;
                const i64 gbase = (i64)eg << 52, hbase = (i64)(eg + 1) << 52;
                const double G0 = __longlong_as_double(gbase), G1 = __longlong_as_double(gbase + 1);
                const double H0 = __longlong_as_double(hbase), H1 = __longlong_as_double(hbase + 1);
                double a0 = 0.0, a1 = 0.0;
                i64 d = 0, dh = 0;
                unsigned mx = 0, tie = 0, tieh = 0;
#pragma unroll
                for (int i = 0; i < F_IPT; i++) {
                    if (p.div) w[i] = __ddiv_rn(w[i], divisor);        // fused normalisation: w / S (IEEE division, as NumPy's w / w.sum())
                    if (i & 1) a1 += w[i]; else a0 += w[i];
                    mx = max(mx, (unsigned)__double2hiint(w[i]));
                    const i64 x0 = __double_as_longlong(__dadd_rn(G0, w[i])), x1 = __double_as_longlong(__dadd_rn(G1, w[i]));
                    tie |= ((unsigned)x0 + 1u) ^ (unsigned)x1;         // d1 != d0: an exact tie
                    d += x0 - gbase;
                    const i64 y0 = __double_as_longlong(__dadd_rn(H0, w[i])), y1 = __double_as_longlong(__dadd_rn(H1, w[i]));
                    tieh |= ((unsigned)y0 + 1u) ^ (unsigned)y1;
                    dh += y0 - hbase;
                }
                // the front buffer is free once every lane of this warp has its weights
                __syncwarp();
                if (lane == 0) f_mbar_arrive(&sm.empty_f);
                int bad = 0;
                if (mx >= 0x7FF00000u) {                   // negative, inf or nan (or a harmless -0.0)
#pragma unroll
                    for (int i = 0; i < F_IPT; i++) if (!(w[i] >= 0.0) || isinf(w[i])) bad = 1;
                }
                double tot = a0 + a1;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    tot += __shfl_xor_sync(FULL, tot, o);
                    d += __shfl_xor_sync(FULL, d, o);
                    dh += __shfl_xor_sync(FULL, dh, o);
                }
                const int wtie = __any_sync(FULL, tie != 0), wtieh = __any_sync(FULL, tieh != 0), wbad = __any_sync(FULL, bad);
                if (lane == 0) {
                    sm.fpart[k & 1][wid].tot = tot; sm.fpart[k & 1][wid].D = d; sm.fpart[k & 1][wid].D1 = dh;
                    sm.fpart[k & 1][wid].tie = wtie; sm.fpart[k & 1][wid].tie1 = wtieh; sm.fpart[k & 1][wid].bad = wbad;
                }
                f_bar<NT>();
                if (tid == 0) {
                    double tt = 0.0; i64 D = 0, Dh = 0; int ttie = 0, ttieh = 0, tbad = 0;
#pragma unroll
                    for (int i = 0; i < NW; i++) {
                        tt += sm.fpart[k & 1][i].tot; D += sm.fpart[k & 1][i].D; Dh += sm.fpart[k & 1][i].D1;
                        ttie |= sm.fpart[k & 1][i].tie; ttieh |= sm.fpart[k & 1][i].tie1; tbad |= sm.fpart[k & 1][i].bad;
                    }
                    if (tbad) { tt = 0.0; p.hdr->fallback = 1; }
                    f_st(p.st1 + t + 1, ((u64)__double_as_longlong(tt) & ~3ull) | ST1_AGG);
                    sl.tot = tt; sl.D = D; sl.tie = ttie; sl.D1 = Dh; sl.tie1 = ttieh; sl.bad = tbad;
                    f_mbar_arrive(&sm.fronted[k % RING]);
                }
            }
        }
        if (k < DELTA) continue;
        // ------------------------------------------------------------ EMIT tile k - DELTA of this CTA
        const int m_idx = k - DELTA, si = m_idx % RING;
        FSlot &sl = sm.ring[si];
        f_mbar_wait(&sm.resolved[si], (m_idx / RING) & 1);
        const int t = sl.t;
        if (t < 0) break;
        f_mbar_wait(&sm.full_e, m_idx & 1);
        const int mode = sl.mode, cross = sl.cross;
        int good = sl.good;
        const i64 S_in = sl.S_in;
        i64 tile_lo = sl.lo, tile_cnt = sl.cnt;
        unsigned char *sb = reinterpret_cast<unsigned char *>(sm.we);
        const i64 jthread = (i64)t * F_TILE + (i64)tid * F_IPT;       // first particle of this thread (local numbering)
        i64 cb[F_IPT];
        i64 thread_start = 0;                               // exact state before this thread's first particle
        if (mode == TM_BAD) {
            __syncwarp();
            if (lane == 0) { f_mbar_arrive(&sm.empty_e); f_mbar_arrive(&sm.freed[si]); }
            continue;
        }
        if (mode == TM_FAST) {
            double w[F_IPT];
#pragma unroll
            for (int c = 0; c < F_IPT / 2; c++) {
                const double2 v = *reinterpret_cast<const double2 *>(sb + f_swz(tid, c));
                w[2 * c] = v.x; w[2 * c + 1] = v.y;
            }
            if (p.div) {
#pragma unroll
                for (int i = 0; i < F_IPT; i++) w[i] = __ddiv_rn(w[i], divisor);
                if (p.wnorm_out) {
                    double *o = p.wnorm_out + jthread;
                    if (jthread + F_IPT <= p.n && (reinterpret_cast<uintptr_t>(o) & 15) == 0) {
#pragma unroll
                        for (int i = 0; i < F_IPT; i += 2) *reinterpret_cast<double2 *>(o + i) = make_double2(w[i], w[i + 1]);
                    } else {
#pragma unroll
                        for (int i = 0; i < F_IPT; i++) if (jthread + i < p.n) o[i] = w[i];
                    }
                }
            }
            if (!cross) {
                // every add of the tile stays in the binade of S_in: bits(S) += d0; block scan of the thread totals
                const i64 base = (S_in >> 52) << 52;
                const double B0 = __longlong_as_double(base);
                i64 acc = 0;
#pragma unroll
                for (int i = 0; i < F_IPT; i++) {
                    acc += __double_as_longlong(__dadd_rn(B0, w[i])) - base;
                    cb[i] = acc;
                }
                const i64 inc = warp_incl_scan_i64(acc, lane);
                if (lane == 31) sm.warp_i[wid] = inc;
                __syncwarp();
                if (lane == 0) { f_mbar_arrive(&sm.empty_e); f_mbar_arrive(&sm.freed[si]); }
                f_bar<NT>();
                i64 ex = inc - acc;
#pragma unroll
                for (int i = 0; i < NW; i++) { const i64 v = sm.warp_i[i]; if (i < wid) ex += v; }
                thread_start = S_in + ex;
#pragma unroll
                for (int i = 0; i < F_IPT; i++) cb[i] += thread_start;
            } else {
                // the chain left the exact state before every row in the crossing pool
                thread_start = sm.xrow[tid];
                const bool walk = (sm.xmask[wid] >> lane) & 1;
                __syncwarp();
                if (lane == 0) { f_mbar_arrive(&sm.empty_e); f_mbar_arrive(&sm.freed[si]); f_mbar_arrive(&sm.xfree); }
                i64 c = thread_start;
                if (walk) {
                    // this row's adds leave the binade of its start state: true adds
#pragma unroll
                    for (int i = 0; i < F_IPT; i++) { c = __double_as_longlong(__dadd_rn(__longlong_as_double(c), w[i])); cb[i] = c; }
                } else {
                    const i64 base = (thread_start >> 52) << 52;
                    const double B0 = __longlong_as_double(base);
#pragma unroll
                    for (int i = 0; i < F_IPT; i++) { c += __double_as_longlong(__dadd_rn(B0, w[i])) - base; cb[i] = c; }
                }
            }
        } else {
            // general path (ties): needs the normalised weights in the buffer
            if (p.div) {
#pragma unroll
                for (int c = 0; c < F_IPT / 2; c++) {
                    double2 v = *reinterpret_cast<const double2 *>(sb + f_swz(tid, c));
                    v.x = __ddiv_rn(v.x, divisor); v.y = __ddiv_rn(v.y, divisor);
                    *reinterpret_cast<double2 *>(sb + f_swz(tid, c)) = v;
                    if (p.wnorm_out) {
                        if (jthread + 2 * c < p.n) p.wnorm_out[jthread + 2 * c] = v.x;
                        if (jthread + 2 * c + 1 < p.n) p.wnorm_out[jthread + 2 * c + 1] = v.y;
                    }
                }
                f_bar<NT>();
            }
            good = f_slow_tile<MODE>(p, sm, t, S_in);
#pragma unroll
            for (int c = 0; c < F_IPT / 2; c++) {
                const longlong2 v = *reinterpret_cast<const longlong2 *>(sb + f_swz(tid, c));
                cb[2 * c] = v.x; cb[2 * c + 1] = v.y;
            }
            // state before the thread's first particle = the previous particle's c (the tile's S_in for thread 0)
            {
                const longlong2 v = *reinterpret_cast<const longlong2 *>(sb + f_swz(tid > 0 ? tid - 1 : 0, 7));
                thread_start = tid > 0 ? v.y : sm.bc_S_in;
            }
            tile_lo = sm.bc_lo; tile_cnt = sm.bc_cnt;
            __syncwarp();
            if (lane == 0) { f_fence_proxy_async(); f_mbar_arrive(&sm.empty_e); f_mbar_arrive(&sm.freed[si]); }
        }
        if (!good) { f_bar<NT>(); continue; }

        // ---- output range end of every particle, relative to tile_lo: hv[k] = #{positions < c_k} - tile_lo
        int hv[F_IPT], hv_prev;
        if (MODE == F_SYS) {
            // branch-free: floor(c N - u) + 1 away from integers; the rare near-integer cases are redone exactly
            const double u = p.u, half_m = 0.5 - p.tau;
            const int n_m1 = (int)p.n - 1, lo_m1 = (int)tile_lo - 1;
            unsigned slow = 0;
            auto count1 = [&](i64 cbits, unsigned bit) -> int {
                const double v = fma(__longlong_as_double(cbits), Nd, -u);    // >= -u > -1
                const double fl = floor(v);
                const double fr = v - fl;                                     // exact, in [0, 1)
                if (!(fabs(fr - 0.5) < half_m)) slow |= bit;                  // within tau of an integer
                return min(__double2int_rz(fl), n_m1) - lo_m1;                // floor(v) + 1 - tile_lo
            };
#pragma unroll
            for (int i = 0; i < F_IPT; i++) hv[i] = count1(cb[i], 1u << i);
            hv_prev = count1(thread_start, 1u << F_IPT);
            if (slow) {
#pragma unroll
                for (int i = 0; i < F_IPT; i++)
                    if (slow & (1u << i)) hv[i] = (int)(f_count_below<MODE>(p, __longlong_as_double(cb[i])) - tile_lo);
                if (slow & (1u << F_IPT)) hv_prev = (int)(f_count_below<MODE>(p, __longlong_as_double(thread_start)) - tile_lo);
            }
        } else {
#pragma unroll
            for (int i = 0; i < F_IPT; i++) hv[i] = (int)(f_count_below<MODE>(p, __longlong_as_double(cb[i])) - tile_lo);
            hv_prev = (int)(f_count_below<MODE>(p, __longlong_as_double(thread_start)) - tile_lo);
        }

        // ---- expansion
        const int base_j = (int)((i64)t * F_TILE) - 1;                        // markers are local index + 1
        const i64 rel_lo = tile_lo - out_begin;
        const int mis = (int)(((reinterpret_cast<uintptr_t>(p.idx) >> 2) + (uintptr_t)rel_lo) & 3);
        if (tile_cnt + 3 <= WIN && rel_lo >= 0 && rel_lo + tile_cnt <= p.n) {
            // one window; slot 0 is 16-byte aligned in the index array, the tile's first output is slot `mis`
            const int total = (int)tile_cnt + mis;
            int l = hv_prev + mis;
#pragma unroll
            for (int i = 0; i < F_IPT; i++) {
                const int h = hv[i] + mis;
                if (h > l) sm.win[l] = tid * F_IPT + i + 1;
                l = h;
            }
            f_bar<NT>();
            int m[F_SPT];
            f_window_scan(sm, tid, lane, wid, m);
            const int s0 = tid * F_SPT;
            int *dst = p.idx + (rel_lo - mis) + s0;
            if (s0 >= mis && s0 + F_SPT <= total) {
#pragma unroll
                for (int i = 0; i < F_SPT; i += 4)
                    *reinterpret_cast<int4 *>(dst + i) = make_int4(base_j + m[i], base_j + m[i + 1], base_j + m[i + 2], base_j + m[i + 3]);
            } else if (s0 < total) {
#pragma unroll
                for (int i = 0; i < F_SPT; i++)
                    if (s0 + i >= mis && s0 + i < total) dst[i] = base_j + m[i];
            }
            continue;      // the next barrier separates these window reads from the next tile's marker writes
        }
        // general expansion: several windows, runs of BIGRUN or more copies go to the fill kernel
        if (tid == 0) atomicAdd(&p.hdr->n_general, 1);
        const int cnt = (int)tile_cnt;
        int cs = 0;
        while (cs < cnt) {
            if (tid == 0) sm.bc_skip = -1;
            f_bar<NT>();
            {
                int l = hv_prev;
#pragma unroll
                for (int i = 0; i < F_IPT; i++) {
                    const int h = hv[i];
                    if (l <= cs && cs < h && h - cs >= BIGRUN) {
                        sm.bc_skip = h;
                        const int r = atomicAdd(&p.hdr->n_runs, 1);
                        if (r < p.max_runs) p.runs[r] = Run{tile_lo + cs, tile_lo + h, base_j + tid * F_IPT + i + 1, 0};
                        else p.hdr->fallback = 1;
                    }
                    l = h;
                }
            }
            f_bar<NT>();
            const int skip = sm.bc_skip;
            if (skip >= 0) { cs = skip; f_bar<NT>(); continue; }
            const int ce = (cnt - cs > WIN) ? cs + WIN : cnt;
            {
                int l = hv_prev;
#pragma unroll
                for (int i = 0; i < F_IPT; i++) {
                    const int h = hv[i];
                    const int a0 = max(l, cs);
                    if (h > a0 && a0 < ce) sm.win[a0 - cs] = tid * F_IPT + i + 1;
                    l = h;
                }
            }
            f_bar<NT>();
            int m[F_SPT];
            f_window_scan(sm, tid, lane, wid, m);
#pragma unroll
            for (int i = 0; i < F_SPT; i++) {
                const int sl2 = tid * F_SPT + i;
                if (sl2 < ce - cs) f_put_index(p, out_begin, tile_lo + cs + sl2, base_j + m[i]);
            }
            f_bar<NT>();
            cs = ce;
        }
        f_bar<NT>();
    }
}

// ------------------------------------------------------------------ init / epilogue kernels
__global__ void __launch_bounds__(256) k_finit(FParams p)
{
    const i64 nst = (i64)p.T + 1;
    for (i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x + 1; i < nst; i += (i64)gridDim.x * blockDim.x) { p.st1[i] = 0; p.st2[i] = 0; }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        FHeader h;
        memset(&h, 0, sizeof(h));
        const double Ngd = (double)p.n;
        h.out_begin = p.U ? count_below_str(0.0, p.U, p.n, Ngd) : count_below_sys(0.0, p.u, p.n, Ngd, p.tau);
        *p.hdr = h;
        p.st1[0] = ST1_INCL;                       // the sums before the first tile: 0.0
        p.st2[0] = ST2_INCL;
    }
}

// long runs (one particle copied >= BIGRUN times), then — only if something failed — the literal
// sequential transcription of resampling.py:141-149, and the info block
__global__ void __launch_bounds__(256) k_fepilogue(FParams p)
{
    FHeader *hdr = p.hdr;
    if (!hdr->fallback) {
        int nr = hdr->n_runs;
        if (nr > p.max_runs) nr = p.max_runs;
        const i64 ob = hdr->out_begin;
        for (int r = 0; r < nr; r++) {
            const Run run = p.runs[r];
            for (i64 i = run.lo + (i64)blockIdx.x * blockDim.x + threadIdx.x; i < run.hi; i += (i64)gridDim.x * blockDim.x) {
                const i64 rel = i - ob;
                if (rel >= 0 && rel < p.n) p.idx[rel] = run.j;
                else hdr->cap_overflow = 1;
            }
        }
    }
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    auto write_info = [&](int overflow, int fb) {
        if (p.info) {
            p.info[0] = overflow; p.info[1] = fb; p.info[2] = hdr->n_unclean; p.info[3] = hdr->n_runs;
            p.info[4] = hdr->chain_bad | (hdr->timeout << 4); p.info[5] = hdr->n_seq; p.info[6] = hdr->cap_overflow; p.info[7] = hdr->n_slow;
        }
    };
    if (!hdr->fallback) { write_info(hdr->overflow, 0); return; }
    const double S = p.div ? *p.div : 1.0;
    auto W = [&](i64 q) { return p.div ? __ddiv_rn(p.w[q], S) : p.w[q]; };
    if (p.div && p.wnorm_out) for (i64 q = 0; q < p.n; q++) p.wnorm_out[q] = W(q);
    // resampling.py:141-149 — cumulative sum and two-pointer merge, one element at a time, over the
    // positions from count_below(0.0)
    const double Ngd = (double)p.n;
    const double carry = 0.0;
    auto pos = [&](i64 i) { return p.U ? pos_str(i, p.U, Ngd) : pos_sys(i, p.u, Ngd); };
    i64 lo = 0, hi = p.n;                        // first i with pos_i >= carry (positions are non-decreasing)
    while (lo < hi) {
        const i64 mid = (lo + hi) >> 1;
        if (pos(mid) < carry) lo = mid + 1; else hi = mid;
    }
    const i64 ob = lo;
    hdr->out_begin = ob;
    hdr->cap_overflow = 0;
    i64 i = ob, j = 0;
    double c = W(0);
    int overflow = 0;
    while (i < p.n) {
        if (pos(i) < c) {
            if (i - ob < p.n) p.idx[i - ob] = (int)j; else hdr->cap_overflow = 1;
            i++;
        } else {
            j++;
            if (j >= p.n) {
                overflow = (int)(p.n - i);
                for (; i < p.n; i++) { if (i - ob < p.n) p.idx[i - ob] = (int)(p.n - 1); else hdr->cap_overflow = 1; }
                break;
            }
            c = __dadd_rn(c, W(j));
        }
    }
    for (i64 q = j + 1; q < p.n; q++) c = __dadd_rn(c, W(q));
    if (p.cumsum_last) *p.cumsum_last = c;
    hdr->out_end = i;
    write_info(overflow, 1);
}

// ------------------------------------------------------------------ host side
namespace {

typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                             const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                             CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn f_get_encode()
{
    static EncodeFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (EncodeFn)ptr;
    }
    return fn;
}

// the weights as rows of 16 doubles (128 bytes); a tile is a box of `box_rows` rows
bool f_make_map(CUtensorMap *m, const double *base, int64_t rows, int box_rows)
{
    EncodeFn enc = f_get_encode();
    if (!enc || rows < 1) return false;
    cuuint64_t gdim[2] = {16, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {128};
    cuuint32_t box[2] = {16, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, const_cast<double *>(base), gdim, gstride, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace

bool f_weights_map(const double *w, int64_t n, int box_rows, CUtensorMap *out)
{
    static thread_local CUtensorMap map;
    static thread_local const void *map_ptr = nullptr;
    static thread_local int64_t map_n = -1;
    static thread_local int map_rows = 0;
    if ((reinterpret_cast<uintptr_t>(w) & 15) != 0 || (n >> 4) < 1 || f_get_encode() == nullptr) return false;
    if (!(map_ptr == w && map_n == n && map_rows == box_rows)) {
        if (!f_make_map(&map, w, n >> 4, box_rows)) { map_ptr = nullptr; return false; }
        map_ptr = w; map_n = n; map_rows = box_rows;
    }
    *out = map;
    return true;
}

namespace {

template <int MODE>
int f_launch(const CUtensorMap &map, const FParams &p, cudaStream_t s)
{
    auto kern = k_fused<MODE>;
    const int smem = (int)sizeof(FSmem);
    static bool configured[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !configured[dev]) {
        if (check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem), "cudaFuncSetAttribute")) return BKE_ERR_CUDA;
        if (dev >= 0 && dev < 64) configured[dev] = true;
    }
    int grid = sm_count() * F_CTAS;
    if (grid > p.T) grid = p.T;
    kern<<<grid, NT + 128, smem, s>>>(map, p);
    return check_cuda(cudaGetLastError(), "k_fused launch");
}

}  // namespace

size_t f_carve(int64_t n, unsigned char *base, FParams *p)
{
    const int64_t Tmax = (n + F_TILE - 1) / F_TILE;
    size_t off = 0;
    auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
    auto take = [&](size_t bytes) { size_t o = off; off += al(bytes); return base ? base + o : nullptr; };
    unsigned char *q;
    q = take(sizeof(FHeader));               if (p) p->hdr = (FHeader *)q;
    q = take(sizeof(u64) * (Tmax + 1));      if (p) p->st1 = (u64 *)q;
    q = take(sizeof(u64) * (Tmax + 1));      if (p) p->st2 = (u64 *)q;
    const int64_t max_runs = n / BIGRUN + 8;
    q = take(sizeof(Run) * max_runs);        if (p) { p->runs = (Run *)q; p->max_runs = (int)max_runs; }
    return off;
}

int f_run(const FRunArgs &a, cudaStream_t s)
{
    const i64 n = a.n;
    if (n < 0) { set_error("bad particle counts"); return BKE_ERR_BAD_ARG; }
    if (n == 0) return BKE_OK;
    if (n >= ((i64)1 << 31)) { set_error("n must be < 2^31 (indexes are int32, resampling.py:141)"); return BKE_ERR_BAD_ARG; }
    if (!a.w || !a.idx || !a.workspace) { set_error("weights, indexes and workspace must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if (!a.U && !(a.u >= 0.0 && a.u < 1.0)) { set_error("u must be in [0, 1)"); return BKE_ERR_BAD_ARG; }
    const size_t need = f_carve(n, nullptr, nullptr);
    if (a.ws_bytes < need) { set_error("workspace too small: %zu < %zu", a.ws_bytes, need); return BKE_ERR_BAD_ARG; }
    if (reinterpret_cast<uintptr_t>(a.workspace) & 255) { set_error("workspace must be 256-byte aligned"); return BKE_ERR_BAD_ARG; }
    FParams p;
    memset(&p, 0, sizeof(p));
    f_carve(n, (unsigned char *)a.workspace, &p);
    p.w = a.w; p.n = n;
    p.u = a.u; p.U = a.U; p.idx = a.idx; p.info = a.info; p.cumsum_last = a.cumsum_last;
    p.div = a.div; p.wnorm_out = a.wnorm_out;
    p.T = (int)((n + F_TILE - 1) / F_TILE);
    // |exact sequential sum - approximate sum| in ulps of the running sum: N adds of the reference,
    // the tree sums inside a tile, the T sequential adds and the 2 flag bits per published word of
    // the look-back (and the division of a normalised call); doubled, plus slack.
    const i64 Tg = n / F_TILE + 2;
    p.eb = 2 * (n + 16 * Tg + 2 * F_TILE) + (n >> 4);
    const double tau = ldexp((double)n, -46);
    p.tau = tau > 1e-6 ? tau : 1e-6;
    // TMA path: 16-byte aligned base and at least one full row of 16 weights
    CUtensorMap map;
    memset(&map, 0, sizeof(map));
    p.use_tma = f_weights_map(a.w, n, NT, &map);
    const int init_blocks = (int)((p.T + 1 + 255) / 256) < 64 ? (int)((p.T + 1 + 255) / 256) : 64;
    k_finit<<<init_blocks, 256, 0, s>>>(p);
    const int rc = a.U ? f_launch<F_STRAT>(map, p, s) : f_launch<F_SYS>(map, p, s);
    if (rc != BKE_OK) return rc;
    k_fepilogue<<<sm_count() * 4, 256, 0, s>>>(p);
    return check_cuda(cudaGetLastError(), "resample launch");
}

}  // namespace rs
}  // namespace bke
