// resample.cu — systematic / stratified particle resampling, bit-exact against the reference's
// strictly sequential fp64 cumsum (filterpy/monte_carlo/resampling.py:117-150, :80-114).
//
//   indexes[i] = #{ j : c_j <= pos_i },   c_j = fl(c_{j-1} + w_j)  (np.cumsum, :142),
//   pos_i = fl(fl(u + i) / N)  (systematic, :139)   or   fl(fl(U_i + i) / N)  (stratified, :103)
//
// A parallel fp64 scan rounds in a different order than np.cumsum and flips output indices, so the
// running sum is reproduced EXACTLY instead.  While the running sum S stays inside one binade
// (exponent field e) it is an integer multiple of the binade's ulp q, its int64 BIT PATTERN is
// linear in units of q, and adding a weight w is the integer map
//       bits(S) -> bits(S) + d[parity(bits(S))],      d0 = rne(w/q) for an even mantissa,
// d1 for an odd one; d1 != d0 only for an exact tie (round-half-even).  d0 and d1 come from two IEEE
// adds on the binade base: d0 = bits(2^e + w) - bits(2^e), d1 = bits(nextafter(2^e) + w) - bits(..).
// Such parity maps compose associatively ((f;g)[p] = f[p] + g[(p + f[p]) & 1]), so a parallel scan
// over them reproduces the sequential rounding.  Zero weights are identities in every binade.  The
// few elements whose addition may leave the binade ("raw" elements, found with an approximate
// scan and a rigorous error margin) are applied by a true fp64 add in a tiny sequential chain.
// Every mapped segment is VERIFIED with the exact values (start and end inside the assumed
// binade); if a check fails, or the weights contain negative / non-finite entries, a literal
// single-thread transcription of the reference loop produces the result instead (info[1] = 1), so
// the output is always the reference's.  tests/test_resample_parity_map_model.py checks this
// arithmetic on the CPU against np.cumsum bit for bit.
//
// Passes (all on one stream, no host sync):
//   A  tile sums (approximate, fp64 tree), input validation      reads w (coalesced 16-byte loads)
//   B  exclusive scan of the tile sums                           1 CTA, warp-striped
//   C  per-tile parity maps / raw-element lists                  reads w
//   D  exact chain over tiles                                    1 CTA: segmented scan + short walk
//   E  exact c_j, output ranges, shared-memory index expansion   reads w, writes indexes (coalesced)
//   F  long runs (one particle copied >= 8192 times)             writes indexes
//   G  sequential fallback (normally exits at once), info
#include "resample_common.cuh"
#include "ptx.cuh"

namespace bke {
namespace rs {


// ------------------------------------------------------------------ workspace
struct Header {
    int fallback;       // 1 -> the sequential kernel must produce the result
    int n_unclean;      // tiles with raw elements
    int n_runs;         // long runs queued for the fill kernel
    int overflow;       // positions >= cumsum[-1]
    int chain_bad;      // a verified assumption failed
    int n_seq;          // tiles walked element by element (more than RMAX raw elements)
    int cap_overflow;   // outputs that did not fit the caller's index buffer (sharded calls)
    int n_slow;         // tiles on the slow list
    i64 out_begin;      // first global output position owned by this call
    i64 out_end;        // one past the last
};

struct Slot {           // one tile with raw elements
    int tile;
    int nraw;
    int segk[RMAX + 1];         // binade of segment s, -1 = empty / identity segment
    int segt[RMAX + 1];
    i64 segd[RMAX + 1];
    double wraw[RMAX];
};


struct Ws {
    Header *hdr;
    double *tile_sum;       // [T]
    double *tile_prefix;    // [T+1] approximate exclusive prefix
    i64 *S_in;              // [T+1] exact state (bit pattern) before each tile
    i64 *tile_d;            // [T]   tile map (clean tiles)
    int *tile_t;            // [T]
    int *tile_k;            // [T]   binade, K_ID for an all-zero tile
    int *tile_slot;         // [T]   -1 clean, >= 0 slot of a tile with raw elements, SLOT_SEQ sequential
    i64 *run_d;             // [T]   composite of the clean tiles since the last unclean tile
    int *run_t;             // [T]
    int *run_cnt;           // [T]
    int *run_k;             // [T]
    Slot *slots;            // [UMAX]
    i64 *S_run;             // [UMAX+SEQMAX+1]
    int *ord2tile;          // [UMAX+SEQMAX]
    Run *runs;              // [max_runs]
    int *slow_list;         // [T] tiles that did not qualify for the fast path (order irrelevant)
    SM *ctot;               // [CHAIN_CTAS] composite of each chain CTA's tile range
    int max_runs;
    int T;
};

size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }
constexpr int CHAIN_CTAS = 8;           // pass D runs as one thread-block cluster of this many CTAs

size_t carve(int64_t n, unsigned char *base, Ws *w)
{
    const int64_t T = (n + TILE - 1) / TILE;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += align256(bytes); return base ? base + o : nullptr; };
    unsigned char *p;
    p = take(sizeof(Header));                 if (w) w->hdr = (Header *)p;
    p = take(sizeof(SM) * CHAIN_CTAS);        if (w) w->ctot = (SM *)p;
    p = take(sizeof(double) * T);             if (w) w->tile_sum = (double *)p;
    p = take(sizeof(double) * (T + 1));       if (w) w->tile_prefix = (double *)p;
    p = take(sizeof(i64) * (T + 1));          if (w) w->S_in = (i64 *)p;
    p = take(sizeof(i64) * T);                if (w) w->tile_d = (i64 *)p;
    p = take(sizeof(int) * T);                if (w) w->tile_t = (int *)p;
    p = take(sizeof(int) * T);                if (w) w->tile_k = (int *)p;
    p = take(sizeof(int) * T);                if (w) w->tile_slot = (int *)p;
    p = take(sizeof(i64) * T);                if (w) w->run_d = (i64 *)p;
    p = take(sizeof(int) * T);                if (w) w->run_t = (int *)p;
    p = take(sizeof(int) * T);                if (w) w->run_cnt = (int *)p;
    p = take(sizeof(int) * T);                if (w) w->run_k = (int *)p;
    p = take(sizeof(Slot) * UMAX);            if (w) w->slots = (Slot *)p;
    p = take(sizeof(i64) * (UMAX + SEQMAX + 1)); if (w) w->S_run = (i64 *)p;
    p = take(sizeof(int) * (UMAX + SEQMAX));  if (w) w->ord2tile = (int *)p;
    p = take(sizeof(int) * T);                if (w) w->slow_list = (int *)p;
    int64_t max_runs = n / BIGRUN + 8;
    p = take(sizeof(Run) * max_runs);         if (w) { w->runs = (Run *)p; w->max_runs = (int)max_runs; w->T = (int)T; }
    return off;
}

struct Params {
    const double *w;
    i64 n;                 // particles in this call (this shard)
    i64 ng;                // particles of the whole set: positions are (u + i) / ng
    i64 j0;                // global index of this call's first particle
    i64 cap;               // capacity of idx
    int is_last;           // this call holds the end of the particle set
    const double *carry_approx;   // device: approximate sum of the earlier shards (NULL = 0)
    const double *carry_exact;    // device: exact running sum before this shard (NULL = 0)
    i64 *out_range;        // device int64[2] (NULL ok): global output positions [begin, end) owned by this call
    double u;              // systematic offset
    const double *U;       // stratified uniforms (NULL = systematic)
    int *idx;
    i64 eb;                // classification margin in ulps of the running sum
    double tau;            // fast-path margin of the position search
    int aligned16;         // weights pointer is 16-byte aligned
    int *info;             // user info[8] or NULL
    double *cumsum_last;   // or NULL
    double *cumsum_out;    // non-NULL: write the exact np.cumsum(w) here instead of emitting indexes
    int last_one;          // cumsum mode: store 1.0 as the last element (resampling.py:174)
    int scan_done;         // the segmented scan of the tile maps (chain_scan) has been run by k_compose
    Ws ws;
    const double *div;     // NORM instances: every weight is divided by *div where it is read
    double *wnorm_out;     // NORM instances, optional: pass A writes the divided weights here
};

// A normalised call (bke_resample_normalized) resamples w / S: its kernels are the NORM = true instances,
// which read d = *p.div once and divide every weight they load, __ddiv_rn(w, d) as NumPy's w / w.sum().
// Everything downstream, validation included, sees the divided values.  NORM = false reads w as it is.
template <bool NORM> __device__ __forceinline__ double divisor(const Params &p) { return NORM ? *p.div : 1.0; }
template <bool NORM> __device__ __forceinline__ double wdiv(double w, double d) { return NORM ? __ddiv_rn(w, d) : w; }
template <bool NORM> __device__ __forceinline__ void normalise(double2 (&g)[IPT / 2], double d)
{
#pragma unroll
    for (int i = 0; i < IPT / 2; i++) { g[i].x = wdiv<NORM>(g[i].x, d); g[i].y = wdiv<NORM>(g[i].y, d); }
}

// ------------------------------------------------------------------ pass A: tile sums
// (NORM: also writes the divided weights to p.wnorm_out when it is non-NULL)
template <bool NORM>
__global__ void __launch_bounds__(BLOCK) k_tile_sums(Params p)
{
    __shared__ double sh[BLOCK / 32 + 1];
    const int t = blockIdx.x;
    const i64 base = (i64)t * TILE;
    const double d = divisor<NORM>(p);
    double s = 0.0;
    bool bad = false;
    if (p.aligned16 && base + TILE <= p.n) {
        const double2 *src = reinterpret_cast<const double2 *>(p.w + base);
#pragma unroll
        for (int i = 0; i < IPT / 2; i++) {
            double2 v = src[i * BLOCK + threadIdx.x];
            if (NORM) {
                v.x = wdiv<NORM>(v.x, d); v.y = wdiv<NORM>(v.y, d);
                if (p.wnorm_out) {
                    double *o = p.wnorm_out + base + 2 * (i * BLOCK + threadIdx.x);
                    if ((reinterpret_cast<uintptr_t>(o) & 15) == 0) *reinterpret_cast<double2 *>(o) = v;
                    else { o[0] = v.x; o[1] = v.y; }
                }
            }
            if (!(v.x >= 0.0) || !(v.y >= 0.0) || isinf(v.x) || isinf(v.y)) bad = true;
            s += v.x + v.y;
        }
    } else {
#pragma unroll
        for (int i = 0; i < IPT; i++) {
            const i64 j = base + i * BLOCK + threadIdx.x;
            const double w = (j < p.n) ? wdiv<NORM>(p.w[j], d) : 0.0;
            if (NORM && p.wnorm_out && j < p.n) p.wnorm_out[j] = w;
            if (!(w >= 0.0) || isinf(w)) bad = true;
            s += w;
        }
    }
    double tot;
    block_excl_scan_d(s, &tot, sh);
    if (threadIdx.x == 0) p.ws.tile_sum[t] = tot;
    if (bad) p.ws.hdr->fallback = 1;
}

// ------------------------------------------------------------------ pass B: scan of tile sums
// Warp w owns the contiguous range [w*per, (w+1)*per); it walks it 32 tiles at a time (coalesced)
// with a warp scan and a running carry; the 32 warp totals are scanned by warp 0.
__global__ void __launch_bounds__(CHAIN_THREADS) k_scan_tiles(Params p)
{
    __shared__ double wtot[CHAIN_THREADS / 32];
    const int T = p.ws.T;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int per = ((T + CHAIN_THREADS - 1) / CHAIN_THREADS) * 32;      // tiles per warp, multiple of 32
    const int a = min(T, wid * per), b = min(T, a + per);
    double carry = 0.0;
    constexpr int PF = 8;                                    // rows fetched ahead (hides the load latency)
    for (int t0 = a; t0 < b; t0 += 32 * PF) {
        double v[PF];
#pragma unroll
        for (int r = 0; r < PF; r++) { const int t = t0 + r * 32 + lane; v[r] = (t < b) ? p.ws.tile_sum[t] : 0.0; }
#pragma unroll
        for (int r = 0; r < PF; r++) {
            const int t = t0 + r * 32 + lane;
            const double inc = warp_incl_scan_d(v[r], lane);
            if (t < b) p.ws.tile_prefix[t] = carry + (inc - v[r]);       // warp-local exclusive prefix
            carry += __shfl_sync(FULL, inc, 31);
        }
    }
    if (lane == 0) wtot[wid] = carry;
    __syncthreads();
    if (wid == 0) {
        const double v = wtot[lane];
        const double inc = warp_incl_scan_d(v, lane);
        wtot[lane] = inc - v;
        if (lane == 31) p.ws.tile_prefix[T] = inc;
    }
    __syncthreads();
    __threadfence_block();
    const double c0 = p.carry_approx ? *p.carry_approx : 0.0;
    const double off = wtot[wid] + c0;
#pragma unroll 8
    for (int t = a + lane; t < b; t += 32) p.ws.tile_prefix[t] += off;
    if (threadIdx.x == 0 && c0 != 0.0) p.ws.tile_prefix[T] += c0;
}

// ------------------------------------------------------------------ shared tile analysis (C and E)
struct TileAn {
    double w[IPT];
    SM inc[IPT];           // inclusive segmented parity map at each element
    int ek[IPT];           // binade of the element (clean), K_ID (zero weight) or -1 (raw)
};

// Tile loads: fetch_tile() issues the coalesced 16-byte global loads of a tile into registers (the
// persistent kernels call it one tile AHEAD, so the HBM latency overlaps the previous tile's
// arithmetic); to_blocked() transposes through shared memory so that thread t owns elements
// [8t, 8t+8).  The 16-byte chunks are XOR-swizzled: both the row-major writes and the
// 64-byte-strided reads are bank-conflict-free.
__device__ __forceinline__ void fetch_tile(const Params &p, int t, double2 (&g)[IPT / 2])
{
    const i64 base = (i64)t * TILE;
#pragma unroll
    for (int i = 0; i < IPT / 2; i++) {
        const i64 j = base + 2 * (i64)(i * BLOCK + threadIdx.x);
        if (p.aligned16 && j + 1 < p.n) g[i] = *reinterpret_cast<const double2 *>(p.w + j);
        else { g[i].x = (j < p.n) ? p.w[j] : 0.0; g[i].y = (j + 1 < p.n) ? p.w[j + 1] : 0.0; }
    }
}
__device__ __forceinline__ void to_blocked(const double2 (&g)[IPT / 2], double (&v)[IPT], double2 *buf /*[TILE/2]*/)
{
    constexpr int CH = IPT / 2;                           // 16-byte chunks per thread row (4 or 8)
    static_assert(CH == 4 || CH == 8, "swizzle written for 64- or 128-byte rows");
    const int tid = threadIdx.x;
#pragma unroll
    for (int i = 0; i < CH; i++) {
        const int c16 = i * BLOCK + tid;                  // 16-byte chunk index in the tile
        const int r = c16 / CH, c = c16 % CH;
        const int sw = (CH == 4) ? ((r >> 1) & 3) : (r & 7);
        buf[r * CH + (c ^ sw)] = g[i];
    }
    __syncthreads();
    const int swt = (CH == 4) ? ((tid >> 1) & 3) : (tid & 7);
#pragma unroll
    for (int c = 0; c < CH; c++) {
        const double2 val = buf[tid * CH + (c ^ swt)];
        v[2 * c] = val.x; v[2 * c + 1] = val.y;
    }
    __syncthreads();
}


// classify the thread's elements and build their maps; returns the thread-local aggregate
__device__ __forceinline__ SM classify(const Params &p, TileAn &an, double before)
{
    SM run = sm_identity();
#pragma unroll
    for (int k = 0; k < IPT; k++) {
        const double after = before + an.w[k];
        SM el;
        if (an.w[k] == 0.0) {             // fl(S + 0) = S in every binade
            el = sm_identity();
            an.ek[k] = K_ID;
        } else {
            int e;
            if (clean_add(before, after, p.eb, &e)) { el = elem_map(an.w[k], e); an.ek[k] = e; }
            else { el = SM{0, 0, 1, K_ID}; an.ek[k] = -1; }
        }
        run = combine(run, el);
        an.inc[k] = run;
        before = after;
    }
    return run;
}

// Fast path test + data: every non-zero element of the thread is a clean, tie-free add in binade
// e0 (the binade of the tile's start state).  pre[k] = inclusive sum of the d0's.
__device__ __forceinline__ bool classify_fast(const Params &p, const double (&w)[IPT], double before, int e0,
                                              i64 (&pre)[IPT], bool *nonzero)
{
    bool ok = true, nz = false;
    i64 acc = 0;
    const i64 base = (i64)e0 << 52;
    const double B0 = __longlong_as_double(base), B1 = __longlong_as_double(base + 1);
#pragma unroll
    for (int k = 0; k < IPT; k++) {
        const double after = before + w[k];
        if (w[k] != 0.0) {
            nz = true;
            int e;
            const bool cl = clean_add(before, after, p.eb, &e);
            const i64 d0 = __double_as_longlong(__dadd_rn(B0, w[k])) - base;
            const i64 d1 = __double_as_longlong(__dadd_rn(B1, w[k])) - (base + 1);
            ok = ok && cl && (e == e0) && (d0 == d1);
            acc += d0;
        }
        pre[k] = acc;
        before = after;
    }
    *nonzero = nz;
    return ok;
}

__device__ __forceinline__ int pad32(int i) { return i + (i >> 5); }

struct TileShared {
    double shd[BLOCK / 32 + 1];
    SM shm[BLOCK / 32 + 1];
    i64 shi[BLOCK / 32 + 1];
    int first_raw[BLOCK + 1];    // raw flag of each thread's first element (+ sentinel)
};

// record segment-end maps and raw weights (tiles with raw elements)
__device__ __forceinline__ void export_segments(const TileAn &an, const TileShared &sm, int *segk, int *segt, i64 *segd,
                                                double *wraw, int *poison)
{
#pragma unroll
    for (int k = 0; k < IPT; k++) {
        const int seg = an.inc[k].cnt;
        if (an.ek[k] == -1) {
            wraw[seg - 1] = an.w[k];                  // the raw element that opens segment `seg`
        } else {
            const bool next_raw = (k + 1 < IPT) ? (an.ek[k + 1] == -1) : (sm.first_raw[threadIdx.x + 1] != 0);
            if (next_raw) {
                if (an.inc[k].k == K_POISON) *poison = 1;
                segk[seg] = an.inc[k].k == K_ID ? -1 : an.inc[k].k;      // identity segments are skipped
                segt[seg] = an.inc[k].t;
                segd[seg] = an.inc[k].d;
            }
        }
    }
}

// sequential walk through one tile with raw elements; returns the exact state after the tile.
// segstate (optional) receives the state at the start of every segment.
__device__ i64 walk_slot(const int *segk, const int *segt, const i64 *segd, const double *wraw, int nraw, i64 S,
                         int *bad, i64 *segstate)
{
    for (int s = 0; s <= nraw; s++) {
        if (segstate) segstate[s] = S;
        if (segk[s] >= 0) S = apply_bits(S, segd[s], segt[s], segk[s], bad);
        if (s < nraw) S = __double_as_longlong(__dadd_rn(__longlong_as_double(S), wraw[s]));
    }
    return S;
}

// ------------------------------------------------------------------ pass C: per-tile maps
struct MapsShared {
    TileShared ts;
    double2 buf[TILE / 2];
    int slot;
};

// Fast kernel: every tile whose adds are all clean and tie-free in ONE binade (decided from the two
// approximate tile prefixes and the elements themselves) gets its map as a plain int64 sum, straight
// from the striped registers.  Everything else is queued for the general kernel.  One tile per CTA and no
// register double-buffer: few registers, many resident CTAs — the way pass A reaches the HBM roofline.
template <bool NORM>
__global__ void __launch_bounds__(BLOCK, 5) k_tile_maps_fast1(Params p)
{
    __shared__ i64 shi[BLOCK / 32 + 1];
    const int t = blockIdx.x;
    const double d = divisor<NORM>(p);
    const double tp = p.ws.tile_prefix[t], tp_next = p.ws.tile_prefix[t + 1];
    double2 g[IPT / 2];
    fetch_tile(p, t, g);
    if (p.ws.hdr->fallback) return;
    normalise<NORM>(g, d);
    int e0;
    const bool tile_clean = clean_add(tp, tp_next, p.eb, &e0);
    const i64 base = (i64)e0 << 52;
    const double B0 = __longlong_as_double(base), B1 = __longlong_as_double(base + 1);
    i64 acc = 0;
    bool ok = tile_clean, nz = false;
#pragma unroll
    for (int i = 0; i < IPT / 2; i++) {
        const double w2[2] = {g[i].x, g[i].y};
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const i64 d0 = __double_as_longlong(__dadd_rn(B0, w2[h])) - base;
            const i64 d1 = __double_as_longlong(__dadd_rn(B1, w2[h])) - (base + 1);
            ok = ok && (d0 == d1);
            nz = nz || (w2[h] != 0.0);
            acc += d0;
        }
    }
    if (__syncthreads_and(ok)) {
        i64 total;
        block_excl_scan_i64(acc, &total, shi);
        const int any_nz = __syncthreads_or(nz);
        if (threadIdx.x == 0) {
            p.ws.tile_k[t] = any_nz ? e0 : K_ID; p.ws.tile_d[t] = total; p.ws.tile_t[t] = 0;
            p.ws.tile_slot[t] = SLOT_FAST;
        }
    } else if (threadIdx.x == 0) {
        p.ws.slow_list[atomicAdd(&p.ws.hdr->n_slow, 1)] = t;
    }
}

// General kernel over the slow list: ties, raw elements, sequential tiles.
template <bool NORM>
__global__ void __launch_bounds__(BLOCK, 2) k_tile_maps(Params p)
{
    __shared__ MapsShared sm;
    if (p.ws.hdr->fallback) return;
    const double d = divisor<NORM>(p);
    const int n_slow = p.ws.hdr->n_slow;
    for (int li = blockIdx.x; li < n_slow; li += gridDim.x) {
        const int t = p.ws.slow_list[li];
        const double tp = p.ws.tile_prefix[t];
        double2 g[IPT / 2];
        fetch_tile(p, t, g);
        normalise<NORM>(g, d);
        TileAn an;
        to_blocked(g, an.w, sm.buf);
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < IPT; k++) s += an.w[k];
        double tot;
        const double before = tp + block_excl_scan_d(s, &tot, sm.ts.shd);
        const SM run = classify(p, an, before);
        const int any_raw = __syncthreads_or(run.cnt > 0);
        if (!any_raw) {
            SM total;
            block_excl_scan_sm(run, &total, sm.ts.shm);
            if (threadIdx.x == 0) {
                if (total.k == K_POISON) p.ws.hdr->fallback = 1;
                p.ws.tile_k[t] = total.k; p.ws.tile_d[t] = total.d; p.ws.tile_t[t] = total.t;
                p.ws.tile_slot[t] = -1;
            }
            continue;
        }
        SM total;
        const SM excl = block_excl_scan_sm(run, &total, sm.ts.shm);
#pragma unroll
        for (int k = 0; k < IPT; k++) an.inc[k] = combine(excl, an.inc[k]);
        if (threadIdx.x == 0) {
            int s2 = -1;
            if (total.cnt <= RMAX) {
                s2 = atomicAdd(&p.ws.hdr->n_unclean, 1);
                if (s2 >= UMAX) { s2 = -1; p.ws.hdr->fallback = 1; }
                p.ws.tile_slot[t] = s2 < 0 ? 0 : s2;
            } else {
                // a dense zone of raw elements (tiny weights next to a binade boundary, e.g. the tail of
                // a degenerate weight vector approaching 1.0): the whole tile is walked with true adds
                if (atomicAdd(&p.ws.hdr->n_seq, 1) >= SEQMAX) p.ws.hdr->fallback = 1;
                p.ws.tile_slot[t] = SLOT_SEQ;
            }
            sm.slot = s2;
            p.ws.tile_k[t] = -1;
        }
        sm.ts.first_raw[threadIdx.x] = (an.ek[0] == -1);
        if (threadIdx.x == 0) sm.ts.first_raw[BLOCK] = 1;       // the tile end closes the last segment
        __syncthreads();
        const int s2 = sm.slot;
        if (s2 >= 0) {
            Slot *sl = &p.ws.slots[s2];
            for (int q = threadIdx.x; q <= RMAX; q += BLOCK) { sl->segk[q] = -1; sl->segt[q] = 0; sl->segd[q] = 0; }
            if (threadIdx.x == 0) { sl->tile = t; sl->nraw = total.cnt; }
            __syncthreads();
            int poison = 0;
            export_segments(an, sm.ts, sl->segk, sl->segt, sl->segd, sl->wraw, &poison);
            if (poison) p.ws.hdr->fallback = 1;
        }
        __syncthreads();
    }
}


// ------------------------------------------------------------------ pass D: exact chain over tiles
__device__ __forceinline__ SM tile_el(const Ws &ws, int t)
{
    const int slot = ws.tile_slot[t];                 // all four loads are issued together
    const SM m = SM{ws.tile_d[t], ws.tile_t[t], 0, ws.tile_k[t]};
    if (slot >= 0 || slot == SLOT_SEQ) return SM{0, 0, 1, K_ID};     // unclean tile: restart marker
    return m;
}

// Segmented exclusive scan of the tile maps (restart after every unclean tile): afterwards
// run_*[t] = composite of the clean tiles since the last unclean tile before t, run_cnt[t] = number of
// unclean tiles before t, ord2tile[i] = i-th unclean tile.  NC CTAs of CHAIN_THREADS threads (one
// thread-block cluster when NC > 1; csync() is its barrier): CTA `rank` owns a contiguous range of
// tiles, the CTA totals meet in ws.ctot.
struct ChainRange { int a, b; };
__device__ __forceinline__ ChainRange chain_range(int T, int rank, int NC)
{
    const int wid = threadIdx.x >> 5;
    const int per = ((T + CHAIN_THREADS * NC - 1) / (CHAIN_THREADS * NC)) * 32;      // tiles per warp, multiple of 32
    const i64 a64 = (i64)(rank * (CHAIN_THREADS / 32) + wid) * per;
    const int a = (int)(a64 < T ? a64 : T);
    return ChainRange{a, min(T, a + per)};
}

// the CTA whose range holds tile T-1
__device__ __forceinline__ bool chain_owns_last(int T, int rank, int NC)
{
    const int per = ((T + CHAIN_THREADS * NC - 1) / (CHAIN_THREADS * NC)) * 32;
    return (T - 1) / (per * (CHAIN_THREADS / 32)) == rank;
}

template <typename Sync>
__device__ __forceinline__ void chain_scan(const Ws &ws, SM *wtot, int &bad, int rank, int NC, Sync csync)
{
    const int T = ws.T;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const ChainRange cr = chain_range(T, rank, NC);
    const int a = cr.a, b = cr.b;
    SM carry_m = sm_identity();
    constexpr int PF = 4;                                    // rows fetched ahead (hides the load latency)
    for (int t0 = a; t0 < b; t0 += 32 * PF) {
        SM v[PF];
#pragma unroll
        for (int r = 0; r < PF; r++) { const int t = t0 + r * 32 + lane; v[r] = (t < b) ? tile_el(ws, t) : sm_identity(); }
#pragma unroll
        for (int r = 0; r < PF; r++) {
            const int t = t0 + r * 32 + lane;
            const SM inc = warp_incl_scan_sm(v[r], lane);
            SM prev = shfl_up_sm(inc, 1);
            if (lane == 0) prev = sm_identity();
            const SM ex = combine(carry_m, prev);             // warp-local exclusive value at tile t
            if (t < b) { ws.run_d[t] = ex.d; ws.run_t[t] = ex.t; ws.run_cnt[t] = ex.cnt; ws.run_k[t] = ex.k; }
            carry_m = combine(carry_m, shfl_sm(inc, 31));
        }
    }
    if (lane == 0) wtot[wid] = carry_m;
    __syncthreads();
    if (wid == 0) {
        const SM v = wtot[lane];
        const SM inc = warp_incl_scan_sm(v, lane);
        SM prev = shfl_up_sm(inc, 1);
        if (lane == 0) prev = sm_identity();
        wtot[lane] = prev;                                    // exclusive prefix of the warp ranges
        if (NC > 1 && lane == 31) { ws.ctot[rank] = inc; __threadfence(); }      // this CTA's composite
    }
    if (NC > 1) csync(); else __syncthreads();
    SM woff = wtot[wid];
    if (NC > 1) {
        SM coff = sm_identity();
        for (int c = 0; c < rank; c++) coff = combine(coff, ws.ctot[c]);
        woff = combine(coff, woff);
    }
    for (int t0 = a + lane; t0 < b; t0 += 32 * PF) {
        SM loc[PF];
        int slot[PF];
#pragma unroll
        for (int r = 0; r < PF; r++) {
            const int t = t0 + r * 32;
            if (t < b) { loc[r] = SM{ws.run_d[t], ws.run_t[t], ws.run_cnt[t], ws.run_k[t]}; slot[r] = ws.tile_slot[t]; }
        }
#pragma unroll
        for (int r = 0; r < PF; r++) {
            const int t = t0 + r * 32;
            if (t < b) {
                const SM ex = combine(woff, loc[r]);
                if (ex.k == K_POISON) bad = 1;
                ws.run_d[t] = ex.d; ws.run_t[t] = ex.t; ws.run_cnt[t] = ex.cnt; ws.run_k[t] = ex.k;
                if ((slot[r] >= 0 || slot[r] == SLOT_SEQ) && ex.cnt < UMAX + SEQMAX) ws.ord2tile[ex.cnt] = t;
            }
        }
    }
    __threadfence();
    if (NC > 1) csync(); else __syncthreads();
}

// NC = 1: one CTA; NC = CHAIN_CTAS: one thread-block cluster, every CTA scans / finishes its own range of
// tiles (the single CTA was bound by what one SM can move: ~4.6 MB of tile records at 2^26), CTA 0 walks
// the tiles with raw elements while the others wait at the cluster barrier.
template <bool STRAT, int NC, bool NORM>
__device__ __forceinline__ void chain_body(const Params &p, int rank)
{
    auto csync = [] {
        if (NC > 1) {
            asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
            asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
        }
    };
    __shared__ SM wtot[CHAIN_THREADS / 32];
    __shared__ Slot s_slots[CHAIN_BATCH];
    __shared__ double s_w[TILE];
    __shared__ SM s_rm[CHAIN_BATCH];
    __shared__ i64 s_S;
    __shared__ int s_bad;
    const Ws &ws = p.ws;
    if (ws.hdr->fallback) return;
    const double d = divisor<NORM>(p);
    const int T = ws.T;
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) s_bad = 0;
    int bad = 0;
    if (!p.scan_done) chain_scan(ws, wtot, bad, rank, NC, csync);     // (k_compose has run it already in the staged multi-GPU sequence)
    constexpr int PF = 4;
    const ChainRange cr = chain_range(T, rank, NC);
    const int a = cr.a, b = cr.b;
    // ---- sequential part: one thread walks the tiles that contain raw elements.  Their slot data
    // is staged into shared memory by the whole block first (a dependent chain of global loads
    // would cost ~1 us per hop), CHAIN_BATCH tiles at a time.
    if (rank == 0) {
        const int U = min(ws.hdr->n_unclean, UMAX) + min(ws.hdr->n_seq, SEQMAX);
        if (threadIdx.x == 0) {
            const double carry = p.carry_exact ? *p.carry_exact : 0.0;
            s_S = __double_as_longlong(carry); ws.S_run[0] = s_S;
            const double Ngd = (double)p.ng;
            ws.hdr->out_begin = STRAT ? count_below_str(carry, p.U, p.ng, Ngd) : count_below_sys(carry, p.u, p.ng, Ngd, p.tau);
        }
        constexpr int SLOT_INTS = (int)(sizeof(Slot) / sizeof(int));
        int i0 = 0;
        while (i0 < U) {
            const int t_first = ws.ord2tile[i0];
            __syncthreads();
            if (ws.tile_slot[t_first] == SLOT_SEQ) {
                // sequential tile: stage its weights, one thread adds them one by one
                const i64 base = (i64)t_first * TILE;
                for (int q = threadIdx.x; q < TILE; q += CHAIN_THREADS) s_w[q] = (base + q < p.n) ? wdiv<NORM>(p.w[base + q], d) : 0.0;
                if (threadIdx.x == 0) s_rm[0] = SM{ws.run_d[t_first], ws.run_t[t_first], 0, ws.run_k[t_first]};
                __syncthreads();
                if (threadIdx.x == 0) {
                    i64 S = s_S;
                    if (s_rm[0].k >= 0) S = apply_bits(S, s_rm[0].d, s_rm[0].t, s_rm[0].k, &bad);
                    double acc = __longlong_as_double(S);
                    for (int q = 0; q < TILE; q++) acc = __dadd_rn(acc, s_w[q]);
                    S = __double_as_longlong(acc);
                    ws.S_run[i0 + 1] = S;
                    s_S = S;
                }
                i0 += 1;
                continue;
            }
            int nb = 1;                                       // consecutive slot-type tiles
            while (nb < CHAIN_BATCH && i0 + nb < U && ws.tile_slot[ws.ord2tile[i0 + nb]] != SLOT_SEQ) nb++;
            for (int q = threadIdx.x; q < nb * SLOT_INTS; q += CHAIN_THREADS) {
                const int bb = q / SLOT_INTS, o = q % SLOT_INTS;
                const int t = ws.ord2tile[i0 + bb];
                reinterpret_cast<int *>(&s_slots[bb])[o] = reinterpret_cast<const int *>(&ws.slots[ws.tile_slot[t]])[o];
            }
            if (threadIdx.x < nb) {
                const int t = ws.ord2tile[i0 + threadIdx.x];
                s_rm[threadIdx.x] = SM{ws.run_d[t], ws.run_t[t], 0, ws.run_k[t]};
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                i64 S = s_S;
                for (int bb = 0; bb < nb; bb++) {
                    if (s_rm[bb].k >= 0) S = apply_bits(S, s_rm[bb].d, s_rm[bb].t, s_rm[bb].k, &bad);
                    const Slot *sl = &s_slots[bb];
                    S = walk_slot(sl->segk, sl->segt, sl->segd, sl->wraw, sl->nraw, S, &bad, nullptr);
                    ws.S_run[i0 + bb + 1] = S;
                }
                s_S = S;
            }
            i0 += nb;
        }
    }
    __threadfence();
    if (NC > 1) csync(); else __syncthreads();
    // ---- parallel part: exact state before every tile, with verification of the clean tiles ---
    {
        const int U = min(ws.hdr->n_unclean, UMAX) + min(ws.hdr->n_seq, SEQMAX);
        i64 *s_run = reinterpret_cast<i64 *>(s_w);            // the staging buffer is free now
        const int cap = TILE;                                 // entries that fit (U + 1 <= 2305 may exceed it)
        for (int q = threadIdx.x; q <= U && q < cap; q += CHAIN_THREADS) s_run[q] = ws.S_run[q];
        __syncthreads();
        for (int t0 = a + lane; t0 < b; t0 += 32 * PF) {
            int rc[PF], rk[PF], rt[PF], tk[PF], tt[PF], slot[PF];
            i64 rd[PF], td[PF];
#pragma unroll
            for (int r = 0; r < PF; r++) {
                const int t = t0 + r * 32;
                if (t < b) {
                    rc[r] = ws.run_cnt[t]; rk[r] = ws.run_k[t]; rt[r] = ws.run_t[t]; rd[r] = ws.run_d[t];
                    slot[r] = ws.tile_slot[t]; tk[r] = ws.tile_k[t]; tt[r] = ws.tile_t[t]; td[r] = ws.tile_d[t];
                }
            }
#pragma unroll
            for (int r = 0; r < PF; r++) {
                const int t = t0 + r * 32;
                if (t < b) {
                    i64 S = rc[r] < cap ? s_run[rc[r]] : ws.S_run[rc[r]];
                    if (rk[r] >= 0) S = apply_bits(S, rd[r], rt[r], rk[r], &bad);
                    ws.S_in[t] = S;
                    if (slot[r] == -1 || slot[r] == SLOT_FAST) {
                        const i64 E = tk[r] >= 0 ? apply_bits(S, td[r], tt[r], tk[r], &bad) : S;
                        if (t == T - 1) ws.S_in[T] = E;
                    } else if (t == T - 1) {
                        ws.S_in[T] = ws.S_run[rc[r] + 1];
                    }
                }
            }
        }
    }
    if (bad) s_bad = 1;
    __threadfence_block();
    __syncthreads();
    if (threadIdx.x == 0) {
        if (s_bad) { ws.hdr->fallback = 1; ws.hdr->chain_bad = 1; }
        // exact sum after this call's particles: written by the CTA that owns the last tile (the sequential
        // kernel rewrites it when any CTA raised the fallback flag)
        else if (p.cumsum_last && chain_owns_last(T, rank, NC)) *p.cumsum_last = __longlong_as_double(ws.S_in[T]);
    }
}

template <bool STRAT, bool NORM>
__global__ void __launch_bounds__(CHAIN_THREADS) k_chain(Params p) { chain_body<STRAT, 1, NORM>(p, 0); }

template <bool STRAT, bool NORM>
__global__ void __cluster_dims__(CHAIN_CTAS, 1, 1) __launch_bounds__(CHAIN_THREADS) k_chain_cluster(Params p)
{
    chain_body<STRAT, CHAIN_CTAS, NORM>(p, (int)blockIdx.x);
}

// ------------------------------------------------------------------ multi-GPU: the shard's composite
// What a LATER shard needs from this one is the map "exact running sum before the shard -> exact
// running sum after it".  It is not a single parity map (the shard may cross binades), but a short
// list: MAP entries (composites of clean stretches) and RAW entries (elements applied by a true
// add), in order.  It depends only on passes A-C (approximate carry), so every rank forms it at
// once; an all-gather of the lists lets rank r derive its exact carry locally — no rank waits for
// another rank's chain.
constexpr int COMP_MAX = 1000;
struct CompEntry { int type; int k; int t; int pad; i64 d; };      // type 0 = MAP (k, t, d), 1 = RAW (d = bits of w)
struct Composite { int n; int bad; int pad[2]; CompEntry e[COMP_MAX]; };

__global__ void __launch_bounds__(CHAIN_THREADS) k_compose(Params p, Composite *out)
{
    __shared__ SM wtot[CHAIN_THREADS / 32];
    const Ws &ws = p.ws;
    if (threadIdx.x == 0) { out->n = 0; out->bad = ws.hdr->fallback ? 1 : 0; }
    if (ws.hdr->fallback) return;
    int bad = 0;
    chain_scan(ws, wtot, bad, 0, 1, [] {});
    __threadfence_block();
    __syncthreads();
    if (threadIdx.x != 0) return;
    const int T = ws.T;
    const int U = ws.hdr->n_unclean + ws.hdr->n_seq;
    int n = 0;
    bool cbad = ws.hdr->n_unclean > UMAX || ws.hdr->n_seq > 0;       // dense raw zones cannot be summarised: serial hand-over
    auto push_map = [&](int k, int t, i64 d) {
        if (k == K_ID) return;
        if (k == K_POISON || n >= COMP_MAX) { cbad = true; return; }
        out->e[n++] = CompEntry{0, k, t, 0, d};
    };
    for (int i = 0; i < U && !cbad; i++) {
        const int tile = ws.ord2tile[i];
        push_map(ws.run_k[tile], ws.run_t[tile], ws.run_d[tile]);
        const Slot *sl = &ws.slots[ws.tile_slot[tile]];
        for (int q = 0; q <= sl->nraw && !cbad; q++) {
            if (sl->segk[q] >= 0) push_map(sl->segk[q], sl->segt[q], sl->segd[q]);
            if (q < sl->nraw) {
                if (n >= COMP_MAX) cbad = true;
                else out->e[n++] = CompEntry{1, 0, 0, 0, __double_as_longlong(sl->wraw[q])};
            }
        }
    }
    if (!cbad) {
        const SM el = tile_el(ws, T - 1);
        if (el.cnt == 0) {                                   // the shard ends with clean tiles
            const SM tail = combine(SM{ws.run_d[T - 1], ws.run_t[T - 1], 0, ws.run_k[T - 1]}, el);
            push_map(tail.k, tail.t, tail.d);
        }
    }
    out->n = n;
    out->bad = (cbad || bad) ? 1 : 0;
}

// exact running sum before shard `n_before`: the composites of the earlier shards applied in order to 0
__global__ void k_compose_carry(int n_before, const Composite *comps, double *carry, int *status)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    i64 S = 0;
    int bad = 0;
    for (int r = 0; r < n_before; r++) {
        const Composite *c = comps + r;
        if (c->bad) bad = 1;
        for (int i = 0; i < c->n && !bad; i++) {
            const CompEntry e = c->e[i];
            if (e.type == 0) S = apply_bits(S, e.d, e.t, e.k, &bad);
            else S = __double_as_longlong(__dadd_rn(__longlong_as_double(S), __longlong_as_double(e.d)));
        }
    }
    *carry = __longlong_as_double(S);
    if (status) *status = bad;
}

// ------------------------------------------------------------------ pass E: emit indexes
struct EmitShared {
    TileShared ts;
    int hi[TILE + TILE / 32];     // output end (exclusive) of every element, relative to tile_lo; index via pad32()
    union { int ebuf[EXPAND + EXPAND / 32]; double2 buf[TILE / 2]; double wd[TILE]; };   // ebuf index via pad32()
    i64 segstate[RMAX + 1];
    int segk[RMAX + 1];
    int segt[RMAX + 1];
    i64 segd[RMAX + 1];
    double wraw[RMAX];
    int warp_max[BLOCK / 32];
};

template <bool STRAT>
__device__ __forceinline__ i64 count_below(const Params &p, double c)
{
    const double Ngd = (double)p.ng;
    return STRAT ? count_below_str(c, p.U, p.ng, Ngd) : count_below_sys(c, p.u, p.ng, Ngd, p.tau);
}

// store one index (global output position o) into the caller's buffer
__device__ __forceinline__ void put_index(const Params &p, i64 o, int value)
{
    const i64 rel = o - p.ws.hdr->out_begin;
    if (rel >= 0 && rel < p.cap) p.idx[rel] = value;
    else p.ws.hdr->cap_overflow = 1;
}

// cumsum mode: the exact running sums leave as they are (each thread owns IPT consecutive elements = one 128-byte line)
__device__ __forceinline__ void store_cumsum(const Params &p, int t, const i64 (&cbits)[IPT])
{
    const i64 j = (i64)t * TILE + (i64)threadIdx.x * IPT;
    double *o = p.cumsum_out + j;
    if (j + IPT <= p.n && (reinterpret_cast<uintptr_t>(o) & 15) == 0 && !(p.last_one && j + IPT == p.n)) {
#pragma unroll
        for (int k = 0; k < IPT; k += 2)
            *reinterpret_cast<double2 *>(o + k) = make_double2(__longlong_as_double(cbits[k]), __longlong_as_double(cbits[k + 1]));
    } else {
#pragma unroll
        for (int k = 0; k < IPT; k++)
            if (j + k < p.n) o[k] = (p.last_one && j + k == p.n - 1) ? 1.0 : __longlong_as_double(cbits[k]);
    }
}

// Common tail of the emit kernels: cbits[k] = exact c_j (bit pattern) of the thread's 8 elements.
// Computes every element's output range end, then expands the tile's outputs through shared memory
// (coalesced stores); particles copied >= BIGRUN times are queued for the fill kernel.
template <bool STRAT>
__device__ __forceinline__ void emit_tile(const Params &p, EmitShared &sm, int t, i64 S_in, const i64 (&cbits)[IPT])
{
    const Ws &ws = p.ws;
    const int tid = threadIdx.x;
    const i64 tile_lo = count_below<STRAT>(p, __longlong_as_double(S_in));       // every thread: no broadcast needed
    const i64 jbase = (i64)t * TILE + (i64)tid * IPT;
    static_assert(32 % IPT == 0 || IPT % 32 == 0, "pad32 of a thread's elements assumed to share one pad offset");
    const int hbase = pad32(tid * IPT);                    // pad32(tid*IPT + k) == hbase + k for k < IPT (IPT divides 32)
    int hv[IPT];                                           // output range end of each element, relative to tile_lo
    const bool full_tile = (i64)(t + 1) * TILE <= p.n;
    if (!STRAT && full_tile) {
        // branch-free fast evaluation of #{positions < c}: floor(c N - u) + 1 away from integers;
        // the rare near-integer cases are collected and redone exactly below
        // (10 instructions per element: v, floor, fraction, |fraction - 1/2| against the margin, one
        // conversion, integer clamp and offset — the first version spent 19 on fp64 selects and clamps)
        const double Nd = (double)p.ng, u = p.u, half_m = 0.5 - p.tau;
        const int n_m1 = (int)p.ng - 1, lo_m1 = (int)tile_lo - 1;
        unsigned slow = 0;
#pragma unroll
        for (int k = 0; k < IPT; k++) {
            const double v = fma(__longlong_as_double(cbits[k]), Nd, -u);     // >= -u > -1
            const double fl = floor(v);
            const double fr = v - fl;                                         // exact, in [0, 1)
            if (!(fabs(fr - 0.5) < half_m)) slow |= 1u << k;                  // within tau of an integer
            const int g = min(__double2int_rz(fl), n_m1);                     // floor(v), clamped (the conversion saturates)
            hv[k] = g - lo_m1;                                                // floor(v) + 1 - tile_lo
        }
        if (slow) {
#pragma unroll
            for (int k = 0; k < IPT; k++)
                if (slow & (1u << k)) hv[k] = (int)(count_below<STRAT>(p, __longlong_as_double(cbits[k])) - tile_lo);
        }
    } else {
#pragma unroll
        for (int k = 0; k < IPT; k++) {
            hv[k] = -1;                       // padding elements own no output (fixed below)
            if (jbase + k < p.n) hv[k] = (int)(count_below<STRAT>(p, __longlong_as_double(cbits[k])) - tile_lo);
        }
    }
#pragma unroll
    for (int k = 0; k < IPT; k++) sm.hi[hbase + k] = hv[k];
    __syncthreads();
    if (!full_tile) {
        const i64 last_real = p.n - 1 - (i64)t * TILE;      // padding inherits the end of the last real element
        const int hvl = sm.hi[pad32((int)last_real)];
        __syncthreads();
        for (int q = tid; q < TILE; q += BLOCK) if (q > last_real) sm.hi[pad32(q)] = hvl;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < IPT; k++) hv[k] = sm.hi[hbase + k];
    }
    const int tile_cnt = sm.hi[pad32(TILE - 1)];            // outputs owned by this tile
    if (t == ws.T - 1 && tid == 0) {
        i64 O1 = tile_lo + tile_cnt;
        if (p.is_last && O1 < p.ng) {                       // resampling.py:145 would raise IndexError
            ws.hdr->overflow = (int)(p.ng - O1 > 0x7fffffff ? 0x7fffffff : p.ng - O1);
            const int r = atomicAdd(&ws.hdr->n_runs, 1);
            if (r < ws.max_runs) ws.runs[r] = Run{O1, p.ng, (int)(p.ng - 1), 0};
            O1 = p.ng;
        }
        ws.hdr->out_end = O1;
        if (p.out_range) { p.out_range[0] = ws.hdr->out_begin; p.out_range[1] = O1; }
    }
    // this thread's elements own the contiguous outputs [hv_prev, hv[IPT-1]) (relative to tile_lo)
    const int hv_prev = (tid == 0) ? 0 : sm.hi[pad32(tid * IPT - 1)];
    int maxc = hv[0] - hv_prev;
#pragma unroll
    for (int k = 1; k < IPT; k++) maxc = max(maxc, hv[k] - hv[k - 1]);
    const int any_big = __syncthreads_or(maxc > INLINE_MAX);
    const int base_j = (int)(p.j0 + (i64)t * TILE);
    if (!any_big) {
        // direct expansion: every thread writes the few copies of its own particles into the staging
        // window (0, 1 or 2 copies without a loop), then the window leaves with coalesced stores
        for (int cs = 0; cs < tile_cnt; cs += EXPAND) {
            const int ce = min(tile_cnt, cs + EXPAND);
            int l = hv_prev;
#pragma unroll
            for (int k = 0; k < IPT; k++) {
                const int h = hv[k];
                const int a0 = max(l, cs), a1 = min(h, ce);
                if (a1 > a0) {
                    const int val = tid * IPT + k;
                    sm.ebuf[pad32(a0 - cs)] = val;
                    if (a1 > a0 + 1) {
                        sm.ebuf[pad32(a0 + 1 - cs)] = val;
                        for (int o = a0 + 2; o < a1; o++) sm.ebuf[pad32(o - cs)] = val;
                    }
                }
                l = h;
            }
            __syncthreads();
            const i64 rel0 = tile_lo + cs - ws.hdr->out_begin;
            if (rel0 >= 0 && rel0 + (ce - cs) <= p.cap) {
                // pad32(tid + BLOCK k) = pad32(tid) + (BLOCK + BLOCK/32) k: fixed strides on both sides,
                // so the unrolled loop is LDS / IADD / STG with immediate offsets
                int *dst = p.idx + rel0 + tid;
                const int *src = sm.ebuf + pad32(tid);
                const int n_out = ce - cs - tid;                                // outputs at and after this thread's first
#pragma unroll 4
                for (int kk = 0; kk * BLOCK < n_out; kk++) dst[kk * BLOCK] = base_j + src[kk * (BLOCK + BLOCK / 32)];
            } else {
                for (int q = tid; q < ce - cs; q += BLOCK) put_index(p, tile_lo + cs + q, base_j + sm.ebuf[pad32(q)]);
            }
            __syncthreads();
        }
        return;
    }
    // general expansion (a particle with many copies in this tile): start markers + max-scan;
    // runs of BIGRUN or more copies are queued for the fill kernel
    int cs = 0;
    while (cs < tile_cnt) {
        int lo_s = 0, hi_s = TILE - 1;                      // owner of output cs: first element with hi > cs
        while (lo_s < hi_s) {
            const int mid = (lo_s + hi_s) >> 1;
            if (sm.hi[pad32(mid)] > cs) hi_s = mid; else lo_s = mid + 1;
        }
        const int owner = lo_s;
        const int owner_end = sm.hi[pad32(owner)];
        if (owner_end - cs >= BIGRUN) {
            if (tid == 0) {
                const int r = atomicAdd(&ws.hdr->n_runs, 1);
                if (r < ws.max_runs) ws.runs[r] = Run{tile_lo + cs, tile_lo + owner_end, base_j + owner, 0};
                else ws.hdr->fallback = 1;
            }
            cs = owner_end;
            continue;
        }
        const int ce = min(tile_cnt, cs + EXPAND);
        for (int q = tid; q < EXPAND + EXPAND / 32; q += BLOCK) sm.ebuf[q] = 0;
        __syncthreads();
        {
            int l = hv_prev;
#pragma unroll
            for (int k = 0; k < IPT; k++) {
                const int h = hv[k];
                if (h > l && h > cs && l < ce) sm.ebuf[pad32((l > cs ? l : cs) - cs)] = tid * IPT + k + 1;
                l = h;
            }
        }
        __syncthreads();
        {   // inclusive max-scan over ebuf: 16 consecutive entries per thread
            constexpr int PER = EXPAND / BLOCK;
            int v[PER];
            int m = 0;
#pragma unroll
            for (int q = 0; q < PER; q++) { const int x = sm.ebuf[pad32(tid * PER + q)]; m = x > m ? x : m; v[q] = m; }
            const int lane = tid & 31, wid = tid >> 5;
            int inc = m;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(FULL, inc, o); if (lane >= o) inc = y > inc ? y : inc; }
            if (lane == 31) sm.warp_max[wid] = inc;
            __syncthreads();
            int basem = 0;
            for (int k2 = 0; k2 < wid; k2++) basem = max(basem, sm.warp_max[k2]);
            int prev = __shfl_up_sync(FULL, inc, 1);
            if (lane == 0) prev = 0;
            basem = max(basem, prev);
#pragma unroll
            for (int q = 0; q < PER; q++) sm.ebuf[pad32(tid * PER + q)] = max(v[q], basem);
        }
        __syncthreads();
        const i64 rel0 = tile_lo + cs - ws.hdr->out_begin;
        if (rel0 >= 0 && rel0 + (ce - cs) <= p.cap) {
            for (int q = tid; q < ce - cs; q += BLOCK) p.idx[rel0 + q] = base_j - 1 + sm.ebuf[pad32(q)];
        } else {
            for (int q = tid; q < ce - cs; q += BLOCK) put_index(p, tile_lo + cs + q, base_j - 1 + sm.ebuf[pad32(q)]);
        }
        __syncthreads();
        cs = ce;
    }
    __syncthreads();
}

// Fast emit: the tiles pass C marked SLOT_FAST (clean, tie-free, one binade):
// c_j = S_in + prefix sum of rne(w_j / ulp), one IEEE add per element.
template <bool STRAT, bool NORM>
__global__ void __launch_bounds__(BLOCK, 2) k_emit_fast(Params p)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    EmitShared &sm = *reinterpret_cast<EmitShared *>(smem_raw);
    const Ws &ws = p.ws;
    if (ws.hdr->fallback) return;
    const double d = divisor<NORM>(p);
    double2 g[IPT / 2];
    if ((int)blockIdx.x < ws.T) fetch_tile(p, blockIdx.x, g);
    for (int t = blockIdx.x; t < ws.T; t += gridDim.x) {
        double w[IPT];
        normalise<NORM>(g, d);
        to_blocked(g, w, sm.buf);
        if (t + (int)gridDim.x < ws.T) fetch_tile(p, t + gridDim.x, g);      // next tile's loads fly during this tile
        if (ws.tile_slot[t] != SLOT_FAST) continue;                           // the general kernel owns this tile
        const i64 S_in = ws.S_in[t];
        const int tk = ws.tile_k[t];
        const i64 base = (i64)(tk >= 0 ? tk : 0) << 52;
        const double B0 = __longlong_as_double(base);
        i64 cbits[IPT];
        i64 acc = 0;
#pragma unroll
        for (int k = 0; k < IPT; k++) {
            acc += __double_as_longlong(__dadd_rn(B0, w[k])) - base;
            cbits[k] = acc;
        }
        i64 total_d;
        const i64 ex = block_excl_scan_i64(acc, &total_d, sm.ts.shi);
#pragma unroll
        for (int k = 0; k < IPT; k++) cbits[k] += S_in + ex;
        if (p.cumsum_out) { store_cumsum(p, t, cbits); continue; }
        emit_tile<STRAT>(p, sm, t, S_in, cbits);
    }
}


// ------------------------------------------------------------------ pass E, second generation: TMA-staged marker / max-scan emit
// The tiles pass C marked SLOT_FAST (clean, tie-free, one binade): c_j = S_in + prefix sum of
// rne(w_j / ulp).  CTA = 8 consumer warps + 1 loader warp; the loader pulls the next tile into shared
// memory with ONE 2-D TMA copy (128-byte swizzle: thread t reads its 16 consecutive weights with
// conflict-free LDS.128) while the consumers work on the current one.  Expansion: every particle with
// >= 1 copies stores (local index + 1) at its first output slot of a zeroed window, a max-scan over the
// slots fills the runs (no divergent copy loop) and every thread leaves with 16-byte stores of 20
// consecutive indexes.  Two 32 KB stages, 96 registers, two CTAs per SM.
constexpr int E2_NW = 8, E2_NT = E2_NW * 32, E2_SPT = 20, E2_WIN = E2_NT * E2_SPT, E2_STAGES = 2, E2_CTAS = 2;
static_assert(E2_NT * IPT == TILE, "the second-generation emit uses the tile size of passes A-D");

// named barrier 1 of the first NT threads (the consumer warps; the loader warp never joins it)
template <int NT> __device__ __forceinline__ void bar_sync()
{
    asm volatile("barrier.cta.sync 1, %0;" ::"n"(NT) : "memory");
}

// byte offset of weight (row r = owning thread, 16-byte chunk c) inside a swizzled stage
__device__ __forceinline__ uint32_t swz(int r, int c) { return (uint32_t)r * 128u + (uint32_t)((c ^ (r & 7)) << 4); }

namespace {

typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                             const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                             CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn get_encode()
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
bool make_weights_map(CUtensorMap *m, const double *base, int64_t rows, int box_rows)
{
    EncodeFn enc = get_encode();
    if (!enc || rows < 1) return false;
    cuuint64_t gdim[2] = {16, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {128};
    cuuint32_t box[2] = {16, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, const_cast<double *>(base), gdim, gstride, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// tensor map of the weights as rows of 16 doubles with a box of `box_rows` rows (cached per thread);
// false when the driver entry point is missing or the pointer / size does not qualify for TMA
bool weights_map(const double *w, int64_t n, int box_rows, CUtensorMap *out)
{
    static thread_local CUtensorMap map;
    static thread_local const void *map_ptr = nullptr;
    static thread_local int64_t map_n = -1;
    static thread_local int map_rows = 0;
    if ((reinterpret_cast<uintptr_t>(w) & 15) != 0 || (n >> 4) < 1 || get_encode() == nullptr) return false;
    if (!(map_ptr == w && map_n == n && map_rows == box_rows)) {
        if (!make_weights_map(&map, w, n >> 4, box_rows)) { map_ptr = nullptr; return false; }
        map_ptr = w; map_n = n; map_rows = box_rows;
    }
    *out = map;
    return true;
}

}  // namespace

struct Emit2Shared {
    double w[E2_STAGES][TILE];         // TMA destinations (128-byte swizzle): must stay first, 1024-aligned
    int win[E2_WIN];                   // output window (all zero between tiles)
    i64 warp_tot[E2_NW];
    int warp_max[E2_NW];
    uint64_t full[E2_STAGES], empty[E2_STAGES];
    int skip;
};

template <bool STRAT, bool NORM>
__global__ void __launch_bounds__(E2_NT + 32, E2_CTAS) k_emit2(const __grid_constant__ CUtensorMap wmap, Params p)
{
    constexpr int NT = E2_NT, NW = E2_NW, WIN = E2_WIN, SPT = E2_SPT;
    extern __shared__ __align__(1024) unsigned char e2_smem[];
    Emit2Shared &sm = *reinterpret_cast<Emit2Shared *>(e2_smem);
    const Ws &ws = p.ws;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) {
        for (int s = 0; s < E2_STAGES; s++) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], NW); }
        fence_mbar_init();
    }
    for (int q = tid; q < WIN; q += NT + 32) sm.win[q] = 0;
    __syncthreads();
    if (ws.hdr->fallback) return;
    const int T = ws.T;
    if (wid == NW) {
        // loader warp: tiles blockIdx.x, blockIdx.x + gridDim.x, ... ; tiles of the slow list are not loaded
        int q = 0;
        for (int t = blockIdx.x; t < T; t += gridDim.x) {
            if (ws.tile_slot[t] != SLOT_FAST) continue;
            const int s = q % E2_STAGES, use = q / E2_STAGES;
            if (use > 0) while (!mbar_try(&sm.empty[s], (use - 1) & 1)) {}
            if (lane == 0) { mbar_expect_tx(&sm.full[s], TILE * 8); tma_load_2d(sm.w[s], &wmap, 0, t * NT, &sm.full[s]); }
            q++;
        }
        return;
    }
    const i64 out_begin = ws.hdr->out_begin;
    const double Nd = (double)p.ng;
    const double d = divisor<NORM>(p);
    int q = 0;
    for (int t = blockIdx.x; t < T; t += gridDim.x) {
        if (ws.tile_slot[t] != SLOT_FAST) continue;                           // the general kernel owns this tile
        const int s = q % E2_STAGES, use = q / E2_STAGES;
        q++;
        const i64 S_in = ws.S_in[t];
        const int tk = ws.tile_k[t];
        while (!mbar_try(&sm.full[s], use & 1)) {}
        const unsigned char *sb = reinterpret_cast<const unsigned char *>(sm.w[s]);
        const i64 base = (i64)(tk >= 0 ? tk : 0) << 52;
        const double B0 = __longlong_as_double(base);
        i64 cb[IPT];
        i64 acc = 0;
#pragma unroll
        for (int c = 0; c < IPT / 2; c++) {
            const double2 v = *reinterpret_cast<const double2 *>(sb + swz(tid, c));
            acc += __double_as_longlong(__dadd_rn(B0, wdiv<NORM>(v.x, d))) - base; cb[2 * c] = acc;
            acc += __double_as_longlong(__dadd_rn(B0, wdiv<NORM>(v.y, d))) - base; cb[2 * c + 1] = acc;
        }
        const i64 inc = warp_incl_scan_i64(acc, lane);
        if (lane == 31) sm.warp_tot[wid] = inc;
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.empty[s]);                           // this warp holds its weights in registers
        bar_sync<NT>();
        i64 ex = inc - acc, D = 0;
#pragma unroll
        for (int i = 0; i < NW; i++) { const i64 v = sm.warp_tot[i]; if (i < wid) ex += v; D += v; }
        const i64 thread_start = S_in + ex;
#pragma unroll
        for (int i = 0; i < IPT; i++) cb[i] += thread_start;
        // the tile's output range (every thread: the values are uniform, no broadcast needed)
        const i64 tile_lo = count_below<STRAT>(p, __longlong_as_double(S_in));
        const i64 tile_cnt = count_below<STRAT>(p, __longlong_as_double(S_in + D)) - tile_lo;
        if (t == T - 1 && tid == 0) {
            i64 O1 = tile_lo + tile_cnt;
            if (p.is_last && O1 < p.ng) {                       // resampling.py:145 would raise IndexError
                ws.hdr->overflow = (int)(p.ng - O1 > 0x7fffffff ? 0x7fffffff : p.ng - O1);
                const int r = atomicAdd(&ws.hdr->n_runs, 1);
                if (r < ws.max_runs) ws.runs[r] = Run{O1, p.ng, (int)(p.ng - 1), 0};
                O1 = p.ng;
            }
            ws.hdr->out_end = O1;
            if (p.out_range) { p.out_range[0] = out_begin; p.out_range[1] = O1; }
        }
        // ---- output range end of every particle, relative to tile_lo: hv[k] = #{positions < c_k} - tile_lo
        int hv[IPT], hv_prev;
        if (!STRAT) {
            // branch-free: floor(c N - u) + 1 away from integers; the rare near-integer cases are redone exactly
            const double u = p.u, half_m = 0.5 - p.tau;
            const int n_m1 = (int)p.ng - 1, lo_m1 = (int)tile_lo - 1;
            unsigned slow = 0;
            auto count1 = [&](i64 cbits, unsigned bit) -> int {
                const double v = fma(__longlong_as_double(cbits), Nd, -u);    // >= -u > -1
                const double fl = floor(v);
                const double fr = v - fl;                                     // exact, in [0, 1)
                if (!(fabs(fr - 0.5) < half_m)) slow |= bit;                  // within tau of an integer
                return min(__double2int_rz(fl), n_m1) - lo_m1;                // floor(v) + 1 - tile_lo
            };
#pragma unroll
            for (int i = 0; i < IPT; i++) hv[i] = count1(cb[i], 1u << i);
            hv_prev = count1(thread_start, 1u << IPT);
            if (slow) {
#pragma unroll
                for (int i = 0; i < IPT; i++)
                    if (slow & (1u << i)) hv[i] = (int)(count_below<STRAT>(p, __longlong_as_double(cb[i])) - tile_lo);
                if (slow & (1u << IPT)) hv_prev = (int)(count_below<STRAT>(p, __longlong_as_double(thread_start)) - tile_lo);
            }
        } else {
#pragma unroll
            for (int i = 0; i < IPT; i++) hv[i] = (int)(count_below<STRAT>(p, __longlong_as_double(cb[i])) - tile_lo);
            hv_prev = (int)(count_below<STRAT>(p, __longlong_as_double(thread_start)) - tile_lo);
        }
        // ---- expansion
        auto window_scan = [&](int (&m)[SPT]) {
            // read this thread's SPT window slots (and clear them), running maximum, block max-scan
            int4 *wv = reinterpret_cast<int4 *>(sm.win) + tid * (SPT / 4);
#pragma unroll
            for (int i = 0; i < SPT / 4; i++) { const int4 v = wv[i]; m[4 * i] = v.x; m[4 * i + 1] = v.y; m[4 * i + 2] = v.z; m[4 * i + 3] = v.w; }
#pragma unroll
            for (int i = 0; i < SPT / 4; i++) wv[i] = make_int4(0, 0, 0, 0);
#pragma unroll
            for (int i = 1; i < SPT; i++) m[i] = max(m[i], m[i - 1]);
            int incm = m[SPT - 1];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(FULL, incm, o); if (lane >= o) incm = max(incm, y); }
            int basem = __shfl_up_sync(FULL, incm, 1);
            if (lane == 0) basem = 0;
            if (lane == 31) sm.warp_max[wid] = incm;
            bar_sync<NT>();
#pragma unroll
            for (int i = 0; i < NW; i++) { const int x = sm.warp_max[i]; if (i < wid) basem = max(basem, x); }
#pragma unroll
            for (int i = 0; i < SPT; i++) m[i] = max(m[i], basem);
        };
        const int base_j = (int)(p.j0 + (i64)t * TILE) - 1;                   // markers are local index + 1
        const i64 rel_lo = tile_lo - out_begin;
        const int mis = (int)(((reinterpret_cast<uintptr_t>(p.idx) >> 2) + (uintptr_t)rel_lo) & 3);
        if (tile_cnt + 3 <= WIN && rel_lo >= 0 && rel_lo + tile_cnt <= p.cap) {
            // one window; slot 0 is 16-byte aligned in the index array, the tile's first output is slot `mis`
            const int total = (int)tile_cnt + mis;
            int l = hv_prev + mis;
#pragma unroll
            for (int i = 0; i < IPT; i++) {
                const int h = hv[i] + mis;
                if (h > l) sm.win[l] = tid * IPT + i + 1;
                l = h;
            }
            bar_sync<NT>();
            int m[SPT];
            window_scan(m);
            const int s0 = tid * SPT;
            int *dst = p.idx + (rel_lo - mis) + s0;
            if (s0 >= mis && s0 + SPT <= total) {
#pragma unroll
                for (int i = 0; i < SPT; i += 4)
                    *reinterpret_cast<int4 *>(dst + i) = make_int4(base_j + m[i], base_j + m[i + 1], base_j + m[i + 2], base_j + m[i + 3]);
            } else if (s0 < total) {
#pragma unroll
                for (int i = 0; i < SPT; i++)
                    if (s0 + i >= mis && s0 + i < total) dst[i] = base_j + m[i];
            }
            continue;      // the next tile's barrier separates these window reads from its marker writes
        }
        // general expansion: several windows, runs of BIGRUN or more copies go to the fill kernel
        const int cnt = (int)tile_cnt;
        int cs = 0;
        while (cs < cnt) {
            if (tid == 0) sm.skip = -1;
            bar_sync<NT>();
            {
                int l = hv_prev;
#pragma unroll
                for (int i = 0; i < IPT; i++) {
                    const int h = hv[i];
                    if (l <= cs && cs < h && h - cs >= BIGRUN) {
                        sm.skip = h;
                        const int r = atomicAdd(&ws.hdr->n_runs, 1);
                        if (r < ws.max_runs) ws.runs[r] = Run{tile_lo + cs, tile_lo + h, base_j + tid * IPT + i + 1, 0};
                        else ws.hdr->fallback = 1;
                    }
                    l = h;
                }
            }
            bar_sync<NT>();
            const int skip = sm.skip;
            if (skip >= 0) { cs = skip; bar_sync<NT>(); continue; }
            const int ce = (cnt - cs > WIN) ? cs + WIN : cnt;
            {
                int l = hv_prev;
#pragma unroll
                for (int i = 0; i < IPT; i++) {
                    const int h = hv[i];
                    const int a0 = max(l, cs);
                    if (h > a0 && a0 < ce) sm.win[a0 - cs] = tid * IPT + i + 1;
                    l = h;
                }
            }
            bar_sync<NT>();
            int m[SPT];
            window_scan(m);
#pragma unroll
            for (int i = 0; i < SPT; i++) {
                const int sl = tid * SPT + i;
                if (sl < ce - cs) put_index(p, tile_lo + cs + sl, base_j + m[i]);
            }
            bar_sync<NT>();
            cs = ce;
        }
        bar_sync<NT>();
    }
}

// General emit over the slow list: ties, raw elements, sequential tiles.
template <bool STRAT, bool NORM>
__global__ void __launch_bounds__(BLOCK, 2) k_emit_slow(Params p)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    EmitShared &sm = *reinterpret_cast<EmitShared *>(smem_raw);
    const Ws &ws = p.ws;
    if (ws.hdr->fallback) return;
    const double d = divisor<NORM>(p);
    const int tid = threadIdx.x;
    const int n_slow = ws.hdr->n_slow;
    for (int li = blockIdx.x; li < n_slow; li += gridDim.x) {
        const int t = ws.slow_list[li];
        double2 g[IPT / 2];
        fetch_tile(p, t, g);
        normalise<NORM>(g, d);
        TileAn an;
        to_blocked(g, an.w, sm.buf);
        const i64 S_in = ws.S_in[t];
        int bad = 0;
        i64 cbits[IPT];
        if (ws.tile_slot[t] == SLOT_SEQ) {
            // every element by a true add: thread 0 walks the tile once to get each thread's start state
            double *wd = sm.wd;
            i64 *tstart = reinterpret_cast<i64 *>(sm.hi);
#pragma unroll
            for (int k = 0; k < IPT; k++) wd[tid * IPT + k] = an.w[k];
            __syncthreads();
            if (tid == 0) {
                double acc = __longlong_as_double(S_in);
                for (int th = 0; th < BLOCK; th++) {
                    tstart[th] = __double_as_longlong(acc);
                    for (int k = 0; k < IPT; k++) acc = __dadd_rn(acc, wd[th * IPT + k]);
                }
            }
            __syncthreads();
            double acc = __longlong_as_double(tstart[tid]);
            __syncthreads();
#pragma unroll
            for (int k = 0; k < IPT; k++) { acc = __dadd_rn(acc, an.w[k]); cbits[k] = __double_as_longlong(acc); }
        } else {
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < IPT; k++) s += an.w[k];
            double tot;
            const double before = ws.tile_prefix[t] + block_excl_scan_d(s, &tot, sm.ts.shd);
            const SM run = classify(p, an, before);
            SM total;
            const SM excl = block_excl_scan_sm(run, &total, sm.ts.shm);
#pragma unroll
            for (int k = 0; k < IPT; k++) an.inc[k] = combine(excl, an.inc[k]);
            if (total.cnt > 0) {      // segment start states (exact)
                sm.ts.first_raw[tid] = (an.ek[0] == -1);
                if (tid == 0) sm.ts.first_raw[BLOCK] = 1;
                for (int q = tid; q <= RMAX; q += BLOCK) { sm.segk[q] = -1; sm.segt[q] = 0; sm.segd[q] = 0; }
                __syncthreads();
                int poison = 0;
                export_segments(an, sm.ts, sm.segk, sm.segt, sm.segd, sm.wraw, &poison);
                __syncthreads();
                if (tid == 0) walk_slot(sm.segk, sm.segt, sm.segd, sm.wraw, total.cnt, S_in, &bad, sm.segstate);
            } else if (tid == 0) {
                sm.segstate[0] = S_in;
            }
            __syncthreads();
#pragma unroll
            for (int k = 0; k < IPT; k++) {
                const i64 S0 = sm.segstate[an.inc[k].cnt];
                // a raw element: the segment it opens starts at its own result; only zeros so far: unchanged
                cbits[k] = (an.ek[k] == -1 || an.inc[k].k < 0) ? S0 : apply_bits(S0, an.inc[k].d, an.inc[k].t, an.inc[k].k, &bad);
            }
            if (bad) ws.hdr->chain_bad = 2;      // cannot happen after pass D verified the tile; recorded for tests
        }
        if (p.cumsum_out) { store_cumsum(p, t, cbits); __syncthreads(); continue; }
        emit_tile<STRAT>(p, sm, t, S_in, cbits);
    }
}

// ------------------------------------------------------------------ pass F: long runs
__global__ void __launch_bounds__(256) k_fill_runs(Params p)
{
    const Ws &ws = p.ws;
    if (ws.hdr->fallback) return;
    int nr = ws.hdr->n_runs;
    if (nr > ws.max_runs) nr = ws.max_runs;
    const i64 ob = ws.hdr->out_begin;
    for (int r = 0; r < nr; r++) {
        const Run run = ws.runs[r];
        for (i64 i = run.lo + (i64)blockIdx.x * blockDim.x + threadIdx.x; i < run.hi; i += (i64)gridDim.x * blockDim.x) {
            const i64 rel = i - ob;
            if (rel >= 0 && rel < p.cap) p.idx[rel] = run.j;
            else ws.hdr->cap_overflow = 1;
        }
    }
}

// ------------------------------------------------------------------ pass G: literal sequential fallback
template <bool STRAT, bool NORM>
__global__ void k_sequential(Params p)
{
    const Ws &ws = p.ws;
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const double d = divisor<NORM>(p);
    auto W = [&](i64 q) { return wdiv<NORM>(p.w[q], d); };
    auto write_info = [&](int overflow, int fb) {
        if (p.info) {
            p.info[0] = overflow; p.info[1] = fb; p.info[2] = ws.hdr->n_unclean; p.info[3] = ws.hdr->n_runs;
            p.info[4] = ws.hdr->chain_bad; p.info[5] = ws.hdr->n_seq; p.info[6] = ws.hdr->cap_overflow; p.info[7] = ws.hdr->n_slow;
        }
    };
    if (!ws.hdr->fallback) { write_info(ws.hdr->overflow, 0); return; }
    if (p.cumsum_out) {                          // cumsum mode: np.cumsum, one add at a time
        double c = 0.0;
        for (i64 q = 0; q < p.n; q++) { c = (q == 0) ? W(0) : __dadd_rn(c, W(q)); p.cumsum_out[q] = c; }
        if (p.cumsum_last) *p.cumsum_last = c;
        if (p.last_one) p.cumsum_out[p.n - 1] = 1.0;
        write_info(0, 1);
        return;
    }
    // resampling.py:141-149 — cumulative sum and two-pointer merge, one element at a time.
    // A shard starts from the exact running sum of the earlier shards and owns the positions from
    // count_below(carry) up to count_below(its last cumulative sum).
    const double Ngd = (double)p.ng;
    const double carry = p.carry_exact ? *p.carry_exact : 0.0;
    i64 lo = 0, hi = p.ng;                       // first i with pos_i >= carry (positions are non-decreasing)
    while (lo < hi) {
        const i64 mid = (lo + hi) >> 1;
        const double pm = STRAT ? pos_str(mid, p.U, Ngd) : pos_sys(mid, p.u, Ngd);
        if (pm < carry) lo = mid + 1; else hi = mid;
    }
    const i64 ob = lo;
    ws.hdr->out_begin = ob;
    ws.hdr->cap_overflow = 0;
    i64 i = ob, j = 0;
    double c = (carry == 0.0) ? W(0) : __dadd_rn(carry, W(0));
    int overflow = 0;
    while (i < p.ng) {
        const double pos = STRAT ? pos_str(i, p.U, Ngd) : pos_sys(i, p.u, Ngd);
        if (pos < c) {
            if (i - ob < p.cap) p.idx[i - ob] = (int)(p.j0 + j); else ws.hdr->cap_overflow = 1;
            i++;
        } else {
            j++;
            if (j >= p.n) {
                if (p.is_last) {
                    overflow = (int)(p.ng - i);
                    for (; i < p.ng; i++) { if (i - ob < p.cap) p.idx[i - ob] = (int)(p.ng - 1); else ws.hdr->cap_overflow = 1; }
                }
                break;
            }
            c = __dadd_rn(c, W(j));
        }
    }
    for (i64 q = j + 1; q < p.n; q++) c = __dadd_rn(c, W(q));
    if (p.cumsum_last) *p.cumsum_last = c;
    ws.hdr->out_end = i;
    if (p.out_range) { p.out_range[0] = ob; p.out_range[1] = i; }
    write_info(overflow, 1);
}

// ------------------------------------------------------------------ weight sum / scale
__global__ void __launch_bounds__(BLOCK) k_scale(i64 n, const double *w, const double *div, double *out)
{
    const double d = *div;
    for (i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (i64)gridDim.x * blockDim.x)
        out[i] = __ddiv_rn(w[i], d);
}

__global__ void __launch_bounds__(CHAIN_THREADS) k_sum_tiles(const double *tile_sum, int T, double *out)
{
    __shared__ double sh[CHAIN_THREADS];
    double s = 0.0;
    for (int t = threadIdx.x; t < T; t += CHAIN_THREADS) s += tile_sum[t];
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = CHAIN_THREADS / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = sh[0];
}

// ------------------------------------------------------------------ searchsorted / gather
// np.searchsorted(a, keys, side): one key per thread.  The top levels of the search hit the same
// few cache lines for every key (L2 / L1 resident); the last ~7 levels stay inside one 1 KB span.
template <bool RIGHT>
__global__ void __launch_bounds__(256) k_searchsorted(i64 n, const double *__restrict__ a, i64 nk,
                                                      const double *__restrict__ keys, i64 *__restrict__ out)
{
    for (i64 q = (i64)blockIdx.x * blockDim.x + threadIdx.x; q < nk; q += (i64)gridDim.x * blockDim.x) {
        const double key = keys[q];
        i64 lo = 0, hi = n;
        while (lo < hi) {
            const i64 mid = lo + ((hi - lo) >> 1);
            const double v = __ldg(a + mid);
            const bool go_right = RIGHT ? !(key < v) : (v < key);
            if (go_right) lo = mid + 1; else hi = mid;
        }
        out[q] = lo;
    }
}

// multinomial: np.searchsorted(cs, keys) (side='left') with a bracket from a lookup table.
// lut[b] = #{j : c_j <= b / n} is a systematic resample with u = 0 of the same weights; a key in
// [b/n, (b+1)/n) has its answer between lut[b-1] and lut[b+1], a span of a particle or two for
// weights that are not degenerate.  The bracket is verified against cs and widened to the whole
// array when it does not hold, so the result never depends on the table being right.
__global__ void __launch_bounds__(256) k_searchsorted_lut(i64 n, const double *__restrict__ cs, const int *__restrict__ lut,
                                                          const double *__restrict__ keys, i64 *__restrict__ out)
{
    const double nd = (double)n;
    for (i64 q = (i64)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (i64)gridDim.x * blockDim.x) {
        const double key = keys[q];
        i64 lo = 0, hi = n;
        if (key >= 0.0 && key < 1.0) {
            i64 b = (i64)(key * nd);
            if (b >= n) b = n - 1;
            lo = b >= 2 ? (i64)__ldg(lut + b - 2) : 0;              // one bucket of slack for the rounding of key * n
            hi = b + 2 < n ? (i64)__ldg(lut + b + 2) : n;
            if (lo > hi) { lo = 0; hi = n; }
            if (lo > 0 && !(__ldg(cs + lo - 1) < key)) lo = 0;     // everything left of lo must be < key
            if (hi < n && (__ldg(cs + hi) < key)) hi = n;          // cs[hi] must not be < key
        }
        while (lo < hi) {
            const i64 mid = lo + ((hi - lo) >> 1);
            if (__ldg(cs + mid) < key) lo = mid + 1; else hi = mid;
        }
        out[q] = lo;
    }
}

// dst[r, :] = src[idx[r], :] for rows of `cpr` chunks of type V (the particle gather that follows a
// resample, docs/monte_carlo/resampling.rst:4-8).  Consecutive threads move consecutive chunks of a row.
// set_len > 0: a bank of sets of set_len rows each, indexes count within the set of the output row.
template <typename V, typename I>
__global__ void __launch_bounds__(256) k_gather_rows(i64 n_out, i64 n_src, i64 cpr, const V *__restrict__ src,
                                                     const I *__restrict__ idx, V *__restrict__ dst, int *err, i64 set_len)
{
    const i64 total = n_out * cpr;
    const i64 lim = set_len ? set_len : n_src;
    for (i64 c = (i64)blockIdx.x * blockDim.x + threadIdx.x; c < total; c += (i64)gridDim.x * blockDim.x) {
        const i64 r = c / cpr, within = c - r * cpr;
        i64 j = (i64)idx[r];
        if (j < 0 || j >= lim) { if (err) *err = 1; continue; }
        if (set_len) j += r - r % set_len;
        dst[c] = src[j * cpr + within];
    }
}

template <typename V, typename I>
int launch_gather(i64 n_out, i64 n_src, i64 row_bytes, const void *src, const void *idx, void *dst, int *err, cudaStream_t s,
                  i64 set_len = 0)
{
    const i64 cpr = row_bytes / (i64)sizeof(V);
    const i64 total = n_out * cpr;
    i64 blocks = (total + 256 * 4 - 1) / (256 * 4);
    const i64 cap = (i64)sm_count() * 16;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    k_gather_rows<V, I><<<(unsigned)blocks, 256, 0, s>>>(n_out, n_src, cpr, (const V *)src, (const I *)idx, (V *)dst, err, set_len);
    return check_cuda(cudaGetLastError(), "gather launch");
}

struct RunArgs {
    i64 n, ng, j0, cap;
    const double *w, *U;
    double u;
    int *idx;
    void *workspace; size_t ws_bytes;
    int *info; double *cumsum_last;
    const double *carry_approx, *carry_exact;
    i64 *out_range;
    int is_last;
    double *cumsum_out; int last_one;
    int phase;           // bit 0: passes A-C (need carry_approx), bit 1: pass D chain (needs carry_exact), bit 2: passes E-G
    const double *div;   // non-NULL: resample w / *div (the NORM instances)
    double *wnorm_out;   // with div, optional: receives w / *div
};

// The passes a.phase selects.
template <bool NORM>
int launch(const RunArgs &a, const Params &p, cudaStream_t s)
{
    const i64 n = a.n;
    const int T = p.ws.T;
    const int emit_smem = (int)sizeof(EmitShared);
    const int sms = sm_count();
    const int slow_grid = T < sms * 2 ? T : sms * 2;
    if (a.phase & 1) {
        if (!(a.phase & 8)) {                       // bit 8: the header reset and pass A have run already (bke_resample_shard_stage)
            if (check_cuda(cudaMemsetAsync(p.ws.hdr, 0, sizeof(Header), s), "memset header")) return BKE_ERR_CUDA;
            k_tile_sums<NORM><<<T, BLOCK, 0, s>>>(p);
        }
        k_scan_tiles<<<1, CHAIN_THREADS, 0, s>>>(p);
        k_tile_maps_fast1<NORM><<<T, BLOCK, 0, s>>>(p);
        k_tile_maps<NORM><<<slow_grid, BLOCK, 0, s>>>(p);
    }
    if (a.phase & 2) {
        // a cluster of CHAIN_CTAS CTAs once there are enough tiles to share out
        if (T >= 2048) {
            if (a.U) k_chain_cluster<true, NORM><<<CHAIN_CTAS, CHAIN_THREADS, 0, s>>>(p);
            else k_chain_cluster<false, NORM><<<CHAIN_CTAS, CHAIN_THREADS, 0, s>>>(p);
        } else if (a.U) k_chain<true, NORM><<<1, CHAIN_THREADS, 0, s>>>(p);
        else k_chain<false, NORM><<<1, CHAIN_THREADS, 0, s>>>(p);
    }
    if (a.phase & 4) {
        const int fast_grid = T < sms * 2 ? T : sms * 2;
        // second-generation emit (TMA-staged, marker / max-scan expansion) whenever the weights qualify for
        // TMA and indexes are produced; otherwise the first-generation kernel
        CUtensorMap wmap;
        const bool emit2 = !a.cumsum_out && (n % 16) == 0 && weights_map(a.w, n, E2_NT, &wmap);
        if (emit2) {
            const auto kern = a.U ? k_emit2<true, NORM> : k_emit2<false, NORM>;
            const int smem2 = (int)sizeof(Emit2Shared);
            if (check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem2), "cudaFuncSetAttribute")) return BKE_ERR_CUDA;
            const int g = T < sms * E2_CTAS ? T : sms * E2_CTAS;
            kern<<<g, E2_NT + 32, smem2, s>>>(wmap, p);
            if (a.U) k_emit_slow<true, NORM><<<slow_grid, BLOCK, emit_smem, s>>>(p);
            else k_emit_slow<false, NORM><<<slow_grid, BLOCK, emit_smem, s>>>(p);
        } else if (a.U) {
            k_emit_fast<true, NORM><<<fast_grid, BLOCK, emit_smem, s>>>(p);
            k_emit_slow<true, NORM><<<slow_grid, BLOCK, emit_smem, s>>>(p);
        } else {
            k_emit_fast<false, NORM><<<fast_grid, BLOCK, emit_smem, s>>>(p);
            k_emit_slow<false, NORM><<<slow_grid, BLOCK, emit_smem, s>>>(p);
        }
        k_fill_runs<<<sms * 4, 256, 0, s>>>(p);
        if (a.U) k_sequential<true, NORM><<<1, 32, 0, s>>>(p);
        else k_sequential<false, NORM><<<1, 32, 0, s>>>(p);
    }
    return check_cuda(cudaGetLastError(), "resample launch");
}

int run(const RunArgs &a, cudaStream_t s)
{
    const i64 n = a.n;
    if (n < 0 || a.ng < n || a.j0 < 0) { set_error("bad particle counts"); return BKE_ERR_BAD_ARG; }
    if (n == 0) return BKE_OK;
    if (a.ng >= ((i64)1 << 31)) { set_error("n must be < 2^31 (indexes are int32, resampling.py:141)"); return BKE_ERR_BAD_ARG; }
    if (!a.w || !(a.idx || a.cumsum_out) || !a.workspace) { set_error("weights, indexes and workspace must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if (!a.U && !(a.u >= 0.0 && a.u < 1.0)) { set_error("u must be in [0, 1)"); return BKE_ERR_BAD_ARG; }
    const size_t need = carve(n, nullptr, nullptr);
    if (a.ws_bytes < need) { set_error("workspace too small: %zu < %zu", a.ws_bytes, need); return BKE_ERR_BAD_ARG; }
    if (reinterpret_cast<uintptr_t>(a.workspace) & 255) { set_error("workspace must be 256-byte aligned"); return BKE_ERR_BAD_ARG; }
    Params p;
    carve(n, (unsigned char *)a.workspace, &p.ws);
    p.w = a.w; p.n = n; p.ng = a.ng; p.j0 = a.j0; p.cap = a.cap; p.is_last = a.is_last;
    p.carry_approx = a.carry_approx; p.carry_exact = a.carry_exact; p.out_range = a.out_range;
    p.u = a.u; p.U = a.U; p.idx = a.idx; p.info = a.info; p.cumsum_last = a.cumsum_last;
    p.cumsum_out = a.cumsum_out; p.last_one = a.last_one;
    p.scan_done = (a.phase & 16) ? 1 : 0;
    p.div = a.div; p.wnorm_out = a.wnorm_out;
    // |exact sequential sum - approximate tree sum| <= (N + 4096) * 2^-53 relative (non-negative
    // terms), i.e. less than (N + 4096) ulps of the running sum; doubled, plus slack.
    p.eb = 2 * (a.ng + 4096) + (a.ng >> 4);
    const double tau = ldexp((double)a.ng, -46);
    p.tau = tau > 1e-6 ? tau : 1e-6;
    p.aligned16 = (reinterpret_cast<uintptr_t>(a.w) & 15) == 0;
    static bool configured[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !configured[dev]) {
        for (const void *k : {(const void *)k_emit_fast<false, false>, (const void *)k_emit_fast<true, false>,
                              (const void *)k_emit_slow<false, false>, (const void *)k_emit_slow<true, false>,
                              (const void *)k_emit_fast<false, true>, (const void *)k_emit_fast<true, true>,
                              (const void *)k_emit_slow<false, true>, (const void *)k_emit_slow<true, true>})
            if (check_cuda(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(EmitShared)), "cudaFuncSetAttribute")) return BKE_ERR_CUDA;
        if (dev >= 0 && dev < 64) configured[dev] = true;
    }
    return a.div ? launch<true>(a, p, s) : launch<false>(a, p, s);
}

}  // namespace rs
}  // namespace bke

using namespace bke;

extern "C" {

size_t bke_resample_workspace_bytes(int64_t n)
{
    if (n <= 0) return 256;
    return rs::carve(n, nullptr, nullptr);
}

static rs::RunArgs whole_array(int64_t n, const double *weights, double u, const double *U, int32_t *indexes,
                               void *workspace, size_t workspace_bytes, int32_t *info, double *cumsum_last)
{
    rs::RunArgs a;
    a.n = n; a.ng = n; a.j0 = 0; a.cap = n; a.w = weights; a.U = U; a.u = u; a.idx = indexes;
    a.workspace = workspace; a.ws_bytes = workspace_bytes; a.info = info; a.cumsum_last = cumsum_last;
    a.carry_approx = nullptr; a.carry_exact = nullptr; a.out_range = nullptr; a.is_last = 1; a.phase = 7;
    a.cumsum_out = nullptr; a.last_one = 0; a.div = nullptr; a.wnorm_out = nullptr;
    return a;
}

int bke_systematic_resample(int64_t n, const double *weights, double u, int32_t *indexes, void *workspace,
                            size_t workspace_bytes, int32_t *info, double *cumsum_last, void *stream)
{
    return rs::run(whole_array(n, weights, u, nullptr, indexes, workspace, workspace_bytes, info, cumsum_last), (cudaStream_t)stream);
}

int bke_stratified_resample(int64_t n, const double *weights, const double *uniforms, int32_t *indexes,
                            void *workspace, size_t workspace_bytes, int32_t *info, double *cumsum_last, void *stream)
{
    if (n > 0 && !uniforms) { set_error("uniforms is NULL"); return BKE_ERR_BAD_ARG; }
    return rs::run(whole_array(n, weights, 0.0, uniforms, indexes, workspace, workspace_bytes, info, cumsum_last), (cudaStream_t)stream);
}

int bke_resample_normalized(int64_t n, const double *weights, double u, const double *uniforms, int32_t *indexes,
                            double *weights_out, double *sum_out, void *workspace, size_t workspace_bytes,
                            int32_t *info, double *cumsum_last, void *stream)
{
    if (n < 0 || !sum_out) { set_error("bad arguments"); return BKE_ERR_BAD_ARG; }
    if (n == 0) return BKE_OK;
    // the sum S first (the only quantity a multi-GPU caller all-reduces), then the passes on w / S, each
    // dividing the weights it reads: the oracle is systematic_resample(w / S) with this S
    int rc = bke_weights_sum(n, weights, sum_out, workspace, workspace_bytes, stream);
    if (rc != BKE_OK) return rc;
    rs::RunArgs a = whole_array(n, weights, u, uniforms, indexes, workspace, workspace_bytes, info, cumsum_last);
    a.div = sum_out; a.wnorm_out = weights_out;
    return rs::run(a, (cudaStream_t)stream);
}

namespace bke { namespace rs {
__global__ void k_carry_approx(int n_before, const double *sums, double *out)
{
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        double c = 0.0;
        for (int r = 0; r < n_before; r++) c += sums[r];      // left to right: every rank forms the same value
        *out = c;
    }
}
} }

size_t bke_resample_composite_bytes(void) { return sizeof(rs::Composite); }

int bke_resample_shard_stage(const bke_resample_shard_args *args, const bke_resample_shard_ext *ext, int32_t stage, void *stream)
{
    if (!args || !ext) { set_error("NULL argument"); return BKE_ERR_BAD_ARG; }
    cudaStream_t s = (cudaStream_t)stream;
    if (args->n_local <= 0) { set_error("empty shards are not supported by the staged call"); return BKE_ERR_BAD_ARG; }
    if (rs::carve(args->n_local, nullptr, nullptr) > args->workspace_bytes) { set_error("workspace too small"); return BKE_ERR_BAD_ARG; }
    bke_resample_shard_args a = *args;
    if (stage == 1) {
        // header reset, pass A (tile sums, validation), the shard's approximate sum
        if (!ext->shard_sum_out) { set_error("shard_sum_out is NULL"); return BKE_ERR_BAD_ARG; }
        rs::Params p;
        rs::carve(a.n_local, (unsigned char *)a.workspace, &p.ws);
        p.w = a.weights; p.n = a.n_local;
        p.aligned16 = (reinterpret_cast<uintptr_t>(a.weights) & 15) == 0;
        if (check_cuda(cudaMemsetAsync(p.ws.hdr, 0, sizeof(rs::Header), s), "memset header")) return BKE_ERR_CUDA;
        rs::k_tile_sums<false><<<p.ws.T, rs::BLOCK, 0, s>>>(p);
        rs::k_sum_tiles<<<1, rs::CHAIN_THREADS, 0, s>>>(p.ws.tile_sum, p.ws.T, ext->shard_sum_out);
        return check_cuda(cudaGetLastError(), "shard stage 1 launch");
    }
    if (stage == 2) {
        // approximate carry from the all-gathered sums, passes B and C, the shard's composite
        if (!ext->shard_sums_all || !ext->carry_approx_buf || !ext->composite_out) { set_error("stage 2 buffers missing"); return BKE_ERR_BAD_ARG; }
        rs::k_carry_approx<<<1, 32, 0, s>>>(ext->shard_rank, ext->shard_sums_all, ext->carry_approx_buf);
        a.carry_approx = ext->carry_approx_buf;
        a.phase = 1 | 8;
        int rc = bke_resample_shard(&a, stream);
        if (rc != BKE_OK) return rc;
        return bke_resample_shard_compose(&a, ext->composite_out, stream);
    }
    if (stage == 3) {
        // exact carry from the all-gathered composites, exact chain, emit
        if (!ext->composites_all || !ext->carry_exact_buf || !ext->carry_approx_buf) { set_error("stage 3 buffers missing"); return BKE_ERR_BAD_ARG; }
        int rc = bke_resample_compose_carry(ext->shard_rank, ext->composites_all, ext->carry_exact_buf, ext->compose_status, stream);
        if (rc != BKE_OK) return rc;
        a.carry_approx = ext->carry_approx_buf;
        a.carry_exact = ext->carry_exact_buf;
        a.phase = 2 | 16;                                  // 16: k_compose has left the scanned tile maps in the workspace
        rc = bke_resample_shard(&a, stream);
        if (rc != BKE_OK) return rc;
        a.phase = 4;
        return bke_resample_shard(&a, stream);
    }
    set_error("stage must be 1, 2 or 3");
    return BKE_ERR_BAD_ARG;
}

int bke_resample_shard_compose(const bke_resample_shard_args *args, void *composite_out, void *stream)
{
    if (!args || !composite_out) { set_error("NULL argument"); return BKE_ERR_BAD_ARG; }
    if (args->n_local <= 0) { return check_cuda(cudaMemsetAsync(composite_out, 0, 16, (cudaStream_t)stream), "memset"); }
    rs::Params p;
    if (rs::carve(args->n_local, nullptr, nullptr) > args->workspace_bytes) { set_error("workspace too small"); return BKE_ERR_BAD_ARG; }
    rs::carve(args->n_local, (unsigned char *)args->workspace, &p.ws);
    p.n = args->n_local;
    rs::k_compose<<<1, rs::CHAIN_THREADS, 0, (cudaStream_t)stream>>>(p, (rs::Composite *)composite_out);
    return check_cuda(cudaGetLastError(), "compose launch");
}

int bke_resample_compose_carry(int32_t n_shards_before, const void *composites, double *carry_exact, int32_t *status,
                               void *stream)
{
    if (n_shards_before < 0 || !carry_exact || (n_shards_before > 0 && !composites)) { set_error("bad arguments"); return BKE_ERR_BAD_ARG; }
    rs::k_compose_carry<<<1, 32, 0, (cudaStream_t)stream>>>(n_shards_before, (const rs::Composite *)composites, carry_exact, status);
    return check_cuda(cudaGetLastError(), "compose carry launch");
}

int bke_resample_shard(const bke_resample_shard_args *args, void *stream)
{
    if (!args) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    if (!(args->phase & 7)) { set_error("phase selects nothing"); return BKE_ERR_BAD_ARG; }
    if ((args->phase & 8) && !(args->phase & 1)) { set_error("phase bit 8 modifies phase 1"); return BKE_ERR_BAD_ARG; }
    rs::RunArgs a;
    a.n = args->n_local; a.ng = args->n_global; a.j0 = args->j_offset; a.cap = args->capacity;
    a.w = args->weights; a.U = args->uniforms; a.u = args->u; a.idx = args->indexes;
    a.workspace = args->workspace; a.ws_bytes = args->workspace_bytes; a.info = args->info; a.cumsum_last = args->carry_out;
    a.carry_approx = args->carry_approx; a.carry_exact = args->carry_exact; a.out_range = reinterpret_cast<rs::i64 *>(args->out_range);
    a.is_last = args->is_last; a.phase = args->phase; a.cumsum_out = nullptr; a.last_one = 0;
    a.div = nullptr; a.wnorm_out = nullptr;
    if (a.j0 + a.n > a.ng) { set_error("shard exceeds the global particle count"); return BKE_ERR_BAD_ARG; }
    return rs::run(a, (cudaStream_t)stream);
}

int bke_weights_sum(int64_t n, const double *weights, double *sum_out, void *workspace, size_t workspace_bytes,
                    void *stream)
{
    if (n < 0 || !sum_out) { set_error("bad arguments"); return BKE_ERR_BAD_ARG; }
    cudaStream_t s = (cudaStream_t)stream;
    if (n == 0) return check_cuda(cudaMemsetAsync(sum_out, 0, sizeof(double), s), "memset");
    if (!weights || !workspace) { set_error("weights and workspace must be non-NULL"); return BKE_ERR_BAD_ARG; }
    const size_t need = rs::carve(n, nullptr, nullptr);
    if (workspace_bytes < need) { set_error("workspace too small: %zu < %zu", workspace_bytes, need); return BKE_ERR_BAD_ARG; }
    rs::Params p;
    rs::carve(n, (unsigned char *)workspace, &p.ws);
    p.w = weights; p.n = n;
    p.aligned16 = (reinterpret_cast<uintptr_t>(weights) & 15) == 0;
    if (check_cuda(cudaMemsetAsync(p.ws.hdr, 0, sizeof(rs::Header), s), "memset header")) return BKE_ERR_CUDA;
    rs::k_tile_sums<false><<<p.ws.T, rs::BLOCK, 0, s>>>(p);
    rs::k_sum_tiles<<<1, rs::CHAIN_THREADS, 0, s>>>(p.ws.tile_sum, p.ws.T, sum_out);
    return check_cuda(cudaGetLastError(), "weights_sum launch");
}

int bke_weights_scale(int64_t n, const double *weights, const double *divisor, double *weights_out, void *stream)
{
    if (n < 0) { set_error("n < 0"); return BKE_ERR_BAD_ARG; }
    if (n == 0) return BKE_OK;
    if (!weights || !divisor || !weights_out) { set_error("NULL argument"); return BKE_ERR_BAD_ARG; }
    int64_t blocks = (n + rs::BLOCK * 8 - 1) / (rs::BLOCK * 8);
    int64_t cap = (int64_t)sm_count() * 16;
    rs::k_scale<<<(unsigned)(blocks < cap ? blocks : cap), rs::BLOCK, 0, (cudaStream_t)stream>>>(n, weights, divisor, weights_out);
    return check_cuda(cudaGetLastError(), "weights_scale launch");
}

int bke_cumsum_exact(int64_t n, const double *weights, double *cumsum_out, int32_t last_one, void *workspace,
                     size_t workspace_bytes, int32_t *info, void *stream)
{
    if (n > 0 && !cumsum_out) { set_error("cumsum_out is NULL"); return BKE_ERR_BAD_ARG; }
    rs::RunArgs a = whole_array(n, weights, 0.0, nullptr, nullptr, workspace, workspace_bytes, info, nullptr);
    a.cumsum_out = cumsum_out; a.last_one = last_one ? 1 : 0;
    return rs::run(a, (cudaStream_t)stream);
}

int bke_searchsorted(int64_t n, const double *sorted, int64_t n_keys, const double *keys, int32_t side_right,
                     int64_t *indexes, void *stream)
{
    if (n < 0 || n_keys < 0) { set_error("negative length"); return BKE_ERR_BAD_ARG; }
    if (n_keys == 0) return BKE_OK;
    if ((n > 0 && !sorted) || !keys || !indexes) { set_error("NULL argument"); return BKE_ERR_BAD_ARG; }
    int64_t blocks = (n_keys + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 32;
    if (blocks > cap) blocks = cap;
    if (side_right) rs::k_searchsorted<true><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(n, sorted, n_keys, keys, (rs::i64 *)indexes);
    else rs::k_searchsorted<false><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(n, sorted, n_keys, keys, (rs::i64 *)indexes);
    return check_cuda(cudaGetLastError(), "searchsorted launch");
}

int bke_multinomial_resample(int64_t n, const double *weights, const double *uniforms, int64_t *indexes,
                             double *cumsum_scratch, int32_t *lut_scratch, void *workspace, size_t workspace_bytes,
                             int32_t *info, void *stream)
{
    if (n < 0) { set_error("n < 0"); return BKE_ERR_BAD_ARG; }
    if (n == 0) return BKE_OK;
    if (!uniforms || !indexes || !cumsum_scratch) { set_error("NULL argument"); return BKE_ERR_BAD_ARG; }
    int rc = bke_cumsum_exact(n, weights, cumsum_scratch, 1, workspace, workspace_bytes, info, stream);
    if (rc != BKE_OK) return rc;
    if (!lut_scratch || n < 4096) return bke_searchsorted(n, cumsum_scratch, n, uniforms, 0, indexes, stream);
    // bracket table: systematic resample with u = 0 (its overflow flag is irrelevant here: info is
    // rewritten by nobody after this call, so keep the cumsum's info by passing NULL)
    rc = bke_systematic_resample(n, weights, 0.0, lut_scratch, workspace, workspace_bytes, nullptr, nullptr, stream);
    if (rc != BKE_OK) return rc;
    int64_t blocks = (n + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 32;
    if (blocks > cap) blocks = cap;
    rs::k_searchsorted_lut<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(n, cumsum_scratch, lut_scratch, uniforms, (rs::i64 *)indexes);
    return check_cuda(cudaGetLastError(), "multinomial launch");
}

static int gather_rows(int64_t n_out, int64_t n_src, int64_t row_bytes, const void *src, const void *indexes,
                       int32_t index_is_64, void *dst, int32_t *err, int64_t set_len, void *stream)
{
    if (n_out < 0 || n_src < 0 || row_bytes <= 0) { set_error("bad sizes"); return BKE_ERR_BAD_ARG; }
    if (n_out == 0) return BKE_OK;
    if (!src || !indexes || !dst) { set_error("NULL argument"); return BKE_ERR_BAD_ARG; }
    if (src == dst) { set_error("gather cannot run in place"); return BKE_ERR_BAD_ARG; }
    cudaStream_t s = (cudaStream_t)stream;
    const uintptr_t al = reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst) | (uintptr_t)row_bytes;
#define BKE_GATHER(V) (index_is_64 ? rs::launch_gather<V, long long>(n_out, n_src, row_bytes, src, indexes, dst, err, s, set_len) \
                                   : rs::launch_gather<V, int>(n_out, n_src, row_bytes, src, indexes, dst, err, s, set_len))
    if ((al & 15) == 0) return BKE_GATHER(uint4);
    if ((al & 7) == 0) return BKE_GATHER(uint2);
    if ((al & 3) == 0) return BKE_GATHER(unsigned);
    return BKE_GATHER(unsigned char);
#undef BKE_GATHER
}

int bke_gather_rows(int64_t n_out, int64_t n_src, int64_t row_bytes, const void *src, const void *indexes,
                    int32_t index_is_64, void *dst, int32_t *err, void *stream)
{
    return gather_rows(n_out, n_src, row_bytes, src, indexes, index_is_64, dst, err, 0, stream);
}

int bke_gather_rows_bank(int64_t n_sets, int64_t set_len, int64_t row_bytes, const void *src, const void *indexes,
                         int32_t index_is_64, void *dst, int32_t *err, void *stream)
{
    if (n_sets < 0 || set_len < 0) { set_error("bad sizes"); return BKE_ERR_BAD_ARG; }
    if (set_len > 0 && n_sets > INT64_MAX / set_len) { set_error("n_sets * set_len overflows"); return BKE_ERR_BAD_ARG; }
    const int64_t n = n_sets * set_len;
    return gather_rows(n, n, row_bytes, src, indexes, index_is_64, dst, err, set_len, stream);
}

}  // extern "C"
