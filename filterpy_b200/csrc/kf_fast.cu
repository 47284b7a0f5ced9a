// kf_fast.cu — specialised fused predict+update for the benchmark shape (dim_x=4, dim_z=2, fp32).
//
// Mapping (H100 / sm_90a):
//   * persistent CTAs of 128 threads; one CTA processes tiles of 128 consecutive filters;
//   * per tile, ONE elected thread issues 7 1-D bulk copies (cp.async.bulk, SASS UBLKCP) that pull
//     the tile's x, P, F, Q, H, R, z blocks — contiguous byte ranges of the dense AoS arrays the API
//     is handed — into a shared-memory stage and complete on an mbarrier; a 2-stage ring keeps the
//     next tiles' 33 KB in flight while the current tile computes (HBM latency is hidden by the
//     ring, not by occupancy); the ragged last tile copies only its own bytes;
//   * each thread then owns one filter: it reads its rows of the linear stage with LDS.128 in a
//     rotated, bank-conflict-free chunk order (lds_row), the
//     whole predict+update runs in registers (kf_regtile.cuh), results are written with 16-byte
//     stores;
//   * consecutive launches overlap at their edges (programmatic dependent launch): a CTA's
//     prologue runs before griddepcontrol.wait, every global access after it, and a CTA releases
//     the next launch once it has issued the loads of its last tile;
//   * the CTAs walk the tiles in a launch order (tile = blockIdx.x + k gridDim.x) that maps to the bank
//     first to last, or last to first with BKE_REVERSE_TILES: a caller that alternates the two starts
//     every step on the tiles the previous step finished, whose state and models are still in L2.
//     The fused ring may take the order from a device word instead (bke_kf_args.tile_order): the parity
//     of a launch count the kernel itself advances, so that one captured launch alternates across replays.
// Shared models (stride 0) are read once per thread through the read-only path instead of TMA.
// A bank whose per-filter Q and R are exactly symmetric may instead hand over a packed copy of their
// upper triangles (bke_kf_pack_sym_models, REC == 1): one bulk copy per tile replaces the two of
// Q and R, 52 instead of 80 B per filter, and the lower triangles are rebuilt in registers.
// Such a bank may go further and hand over only the model words that differ between its filters
// (bke_kf_scan_models + bke_kf_pack_models, REC == 2): one bulk copy per tile brings those planes,
// and every word the whole bank shares rides in the launch parameters (40 instead of 148 B of
// models per filter for the kf_bank_cv2d template).  A plane the scan found to be a copy of an earlier
// plane in every filter (map.duplicate) is not copied: the step reads the earlier plane in its place,
// so a tile's record comes in one bulk copy per run of consecutive planes the launch reads (20 B per
// filter for the kf_bank_cv2d template, whose two axes share dt, q and r).
//
// Reference arithmetic: filterpy/kalman/kalman_filter.py:471-478, 533-556 (see kf_regtile.cuh).
#include <string.h>
#include "bke_internal.cuh"
#include "kf_regtile.cuh"
#include "ptx.cuh"

namespace bke {
namespace {

// L2 eviction priorities (bulk_load_hint, st_hint): the state x, P is re-read by the NEXT step and, for
// banks whose state is at most 38 MB (about 498 k filters; a bound scaled from an earlier target, not
// measured on the H100), fits the 50 MB L2 -> evict_last; the models and measurements
// stream through once per step -> evict_first, so that they do not push the state out.
__device__ __forceinline__ void st_hint(float *addr, float4 v, uint64_t pol)
{
    asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;"
                 ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}

// the tile-order word of the fused ring (FastP::order): a relaxed read at GPU scope (never a stale L1 line), and
// the acq_rel arrival of a CTA
__device__ __forceinline__ uint32_t ld_relaxed_gpu(const uint32_t *addr)
{
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(addr) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t atom_add_acq_rel_gpu(uint32_t *addr, uint32_t v)
{
    uint32_t old;
    asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], %2;" : "=r"(old) : "l"(addr), "r"(v) : "memory");
    return old;
}

// ---------------------------------------------------------------------------- tile geometry
constexpr int TILE = 128;       // filters per tile == threads per CTA

// The packed symmetric models of a 4/2 bank: one record per tile of TILE filters, structure of arrays,
// plane k holding word k of every filter: Q00 Q01 Q02 Q03 Q11 Q12 Q13 Q22 Q23 Q33 | R00 R01 R11.
// Thread t reads word t of each plane (no bank conflicts); a tile's record is SYM_PLANES * TILE * 4 =
// 6656 B, and the record of the whole bank is padded to whole tiles, so every copy has the same size.
constexpr int SYM_Q_PLANES = 10, SYM_PLANES = 13;

// The packed model words of a 4/2 bank (REC == 2): the 37 words of a filter's models, in this order
// (bit e of a map's `varying` stands for word e):
//   F 0..15 (row-major) | Q 16..25 (upper triangle, as above) | H 26..33 (row-major) | R 34..36 (R00 R01 R11).
// The record holds only the words that differ between filters, tile-major like the one above with
// k = popcount(varying) planes per tile.  A launch copies only the planes it reads (those of its MODE's words,
// a copy replaced by its representative) into the same place of the stage, in at most REC_RUNS bulk copies.
constexpr int WORDS = BKE_KF42_MODEL_WORDS, W_F = 0, W_Q = 16, W_H = 26, W_R = 34;
constexpr uint64_t PREDICT_WORDS = (1ull << W_H) - 1;      // F and Q
constexpr int REC_RUNS = (WORDS + 1) / 2;                  // runs of consecutive planes, at most every other one
// the word of Q[i][j] (upper triangle, row by row)
constexpr int q_word(int i, int j)
{
    const int r = i < j ? i : j, c = i < j ? j : i;
    return W_Q + r * 4 - r * (r - 1) / 2 + (c - r);
}

// The structural words an instance of the fused ring is built for: bit e of ZERO = word e is +0 (bit pattern 0)
// in every filter, of ONE = word e is 1.0f in every filter.  The ring takes them as constants and drops or
// folds the products with them (reg_predict_pat, reg_update_pat; F0 .. R0 are those functions' view).
template <uint64_t Z, uint64_t O>
struct WordPattern {
    static constexpr uint64_t ZERO = Z, ONE = O;
    static constexpr bool any = (ZERO | ONE) != 0;
    static constexpr bool structural(int e) { return ((Z | O) >> e) & 1; }
    static constexpr uint32_t F0(int i) { return (uint32_t)(Z >> (W_F + 4 * i)) & 15u; }
    static constexpr uint32_t F1(int i) { return (uint32_t)(O >> (W_F + 4 * i)) & 15u; }
    static constexpr uint32_t H0(int a) { return (uint32_t)(Z >> (W_H + 4 * a)) & 15u; }
    static constexpr uint32_t H1(int a) { return (uint32_t)(O >> (W_H + 4 * a)) & 15u; }
    static constexpr bool Q0(int i, int j) { return (Z >> q_word(i, j)) & 1; }
    static constexpr bool R0(int a, int b) { return (Z >> (W_R + a + b)) & 1; }
    // row a of H is +0 outside block b (A = {0, 1}, B = {2, 3}); the block it touches
    static constexpr bool h_in(int a, int b) { return (H0(a) & blk_other(2 * b)) == blk_other(2 * b); }
    static constexpr int HB(int a) { return h_in(a, 0) ? 0 : 1; }
    // the structural +0 words make F, Q, H and R block-diagonal over A and B: the cross words of F and Q are +0,
    // each row of H touches one block, the two rows different ones, and R01 is +0.  Such an instance runs a warp
    // whose filters have zeros in the cross words of P on the two blocks (reg_predict_blk, reg_update_blk).
    static constexpr bool blocks()
    {
        for (int i = 0; i < 4; i++)
            for (int k = 0; k < 4; k++)
                if (blk_cross(i, k) && !(((Z >> (W_F + 4 * i + k)) & 1) && Q0(i, k))) return false;
        const bool rows = (h_in(0, 0) && h_in(1, 1)) || (h_in(0, 1) && h_in(1, 0));
        return rows && R0(0, 1);
    }
};
// every word as it comes: the generic kernels
struct NoPattern : WordPattern<0, 0> {};
// the constant-velocity 2-D model of kf_bank_cv2d: F = I + dt (E01 + E23) (ten +0, four 1 on the diagonal),
// Q block-diagonal (Q02 Q03 Q12 Q13 +0), H = [e0; e2] (six +0, two 1), R diagonal (R01 +0)
struct Cv2dPattern : WordPattern<
    // F 2 3 4 6 7 8 9 12 13 14 | Q02 Q03 Q12 Q13 | H 27 28 29 30 31 33 | R01
    (1ull << 2) | (1ull << 3) | (1ull << 4) | (1ull << 6) | (1ull << 7) | (1ull << 8) | (1ull << 9) | (1ull << 12) |
        (1ull << 13) | (1ull << 14) | (1ull << q_word(0, 2)) | (1ull << q_word(0, 3)) | (1ull << q_word(1, 2)) |
        (1ull << q_word(1, 3)) | (1ull << 27) | (1ull << 28) | (1ull << 29) | (1ull << 30) | (1ull << 31) |
        (1ull << 33) | (1ull << (W_R + 1)),
    // F 0 5 10 15 | H 26 32
    (1ull << 0) | (1ull << 5) | (1ull << 10) | (1ull << 15) | (1ull << 26) | (1ull << 32)> {};

// REC: 0 = dense models, 1 = the packed Q / R record, 2 = the packed model words (stage sized for all 37)
// ZS: measurement blocks per stage (the fused ring stages one per step)
template <typename T, int N, int M, bool SHARED = false, int REC = 0, int ZS = 1>
struct Stage {
    // byte sizes of one tile of each array
    static constexpr int XB = TILE * N * sizeof(T);
    static constexpr int PB = TILE * N * N * sizeof(T);
    static constexpr int HB = TILE * M * N * sizeof(T);
    static constexpr int RB = TILE * M * M * sizeof(T);
    static constexpr int ZB = TILE * M * sizeof(T);
    static constexpr int QB = REC == 1 ? TILE * SYM_PLANES * sizeof(T) : REC == 2 ? TILE * WORDS * sizeof(T) : PB;
    // offsets (bulk-copy destinations must be 16-byte aligned; 128 keeps every block on its own lines)
    static constexpr int align_up(int v) { return (v + 127) & ~127; }
    // (a bank that shares its models stages only P, x, z: a third of the bytes, so more stages and CTAs fit)
    static constexpr int OP = 0;
    static constexpr int OF = OP + align_up(PB);
    static constexpr int OQ = OF + (SHARED || REC == 2 ? 0 : align_up(PB));     // Q, or the record
    static constexpr int OH = OQ + (SHARED ? 0 : align_up(QB));
    static constexpr int OX = OH + (SHARED || REC == 2 ? 0 : align_up(HB));
    static constexpr int OR_ = OX + align_up(XB);
    static constexpr int OZ = OR_ + (SHARED || REC ? 0 : align_up(RB));
    static constexpr int BYTES = OZ + ZS * align_up(ZB);
};

// read the 16-byte chunk c of row `row` (ROWB bytes per row) from a linear tile
template <int ROWB>
__device__ __forceinline__ float4 lds_chunk(const unsigned char *base, int row, int c)
{
    return *reinterpret_cast<const float4 *>(base + row * ROWB + c * 16);
}

// Read the whole row `row` of a linear tile with rows of ROWS 16-byte chunks (4: P, F, Q; 2: H) into
// m[ROWS][4].  Read in order, the 8 threads served by one LDS.128 wavefront would land on 2 (4) of
// the 8 16-byte bank groups: a 4-way (2-way) conflict.  Thread t starts instead at chunk
// r = (t / (8 / ROWS)) mod ROWS, which spreads the 8 threads over all 8 groups, and rotates the
// chunks back into place with selects (two rotation steps for 4 chunks, one for 2).
template <int ROWS>
__device__ __forceinline__ void lds_row(const unsigned char *base, int row, float (&m)[ROWS][4])
{
    const int r = (row / (8 / ROWS)) & (ROWS - 1);
    float4 v[ROWS];
#pragma unroll
    for (int c = 0; c < ROWS; c++)
        v[c] = *reinterpret_cast<const float4 *>(base + row * ROWS * 16 + ((c + r) & (ROWS - 1)) * 16);
    // v[c] holds chunk (c + r) mod ROWS; chunk i is v[(i - r) mod ROWS]
#pragma unroll
    for (int step = 1; step < ROWS; step <<= 1) {
        const bool rot = r & step;
        float4 w[ROWS];
#pragma unroll
        for (int i = 0; i < ROWS; i++) {
            const float4 a = v[i], b = v[(i - step) & (ROWS - 1)];
            w[i] = make_float4(rot ? b.x : a.x, rot ? b.y : a.y, rot ? b.z : a.z, rot ? b.w : a.w);
        }
#pragma unroll
        for (int i = 0; i < ROWS; i++) v[i] = w[i];
    }
#pragma unroll
    for (int i = 0; i < ROWS; i++) { m[i][0] = v[i].x; m[i][1] = v[i].y; m[i][2] = v[i].z; m[i][3] = v[i].w; }
}

template <int N, int M>
struct FastP {
    int64_t N_filters;
    int num_tiles;
    int l2_hints;                   // 1: keep x, P in L2 between steps (evict_last), stream the rest (evict_first)
    int reverse;                    // 1: the launch's tile t is the bank's tile num_tiles - 1 - t
    float alpha_sq;
    const float *x, *P, *z;         // the prior state and the measurements (dense AoS)
    const float *F, *Q, *H, *R;     // per-filter models (SHARED == 0) or the bank's one model (SHARED == 1)
    const float *rec;               // REC: the packed record (replaces Q, R; with REC == 2 F and H as well)
    float Fh[N * N], Qh[N * N], Hh[M * N], Rh[M * M];   // used when SHARED == 2: the shared models ride in the launch
                                                        // parameters, so every product with them reads the constant bank;
                                                        // REC == 2: the words the whole bank shares
    float *x_out, *P_out;
    const uint8_t *valid;
    float *x_prior, *P_prior, *K, *y, *S, *SI, *ll;
    int32_t *status;
    int sticky;                       // BKE_STATUS_STICKY: write status only on failure
    uint64_t varying;               // REC == 2: bit e set = word e is read from the record...
    int slot_off[WORDS];            // ...at this byte offset into a tile's record (its plane * TILE * 4)
    int rec_planes;                 // REC == 2: planes per tile of the record,
    int rec_copy;                   // how many of them this launch copies,
    int rec_runs;                   // in this many runs of consecutive planes:
    int run_first[REC_RUNS], run_len[REC_RUNS];
    const float *zs[BKE_KF42_MAX_RING];     // RING: the measurements of step k (p.z is not read),
    int n_steps;                            // for k < n_steps
    int ring_ox, ring_oz, ring_stage;       // RING: the stage laid out for this launch (ring_layout)
    uint32_t *order;                        // RING: the bank's tile-order word {epoch, arrived} (device), or
                                            // NULL: `reverse` decides (last, so no other field moves)
};

// MODE: 3 = predict+update, 1 = predict only, 2 = update only
// SHARED: 0 = per-filter models (staged by bulk copies), 1 = one model for the bank read from device
// memory, 2 = one model for the bank carried in the kernel parameters
// REC (SHARED == 0 only): 1 = Q and R come from the packed record p.rec instead of p.Q, p.R;
// 2 = every model word the bank's filters differ in comes from p.rec, the others from p.Fh .. p.Rh
// Each CTA keeps STAGES tiles in flight.  Resident CTAs per SM: 3 with per-filter models (33 KB per
// stage, 29.5 KB with either record), 4 with one shared model (11 KB per stage), 5 when that model
// rides in the launch parameters.
// RING (MODE 3, REC 2, no EXTRAS): 0 = one step; BKE_KF42_MAX_RING = the fused ring: each thread loads x, P and
// the model words once, runs p.n_steps predict+update pairs on the measurements p.zs[0 .. n_steps) back to
// back in registers and stores x, P once.  Its stage is laid out per launch (ring_layout): P, the record's
// planes, x and one 1 KB measurement block per step, so a launch stages only what it reads (19 KB per
// stage for the kf_bank_cv2d template at 4 steps) and up to 4 CTAs, the register limit, fit an SM.
constexpr int STAGES = 2;
constexpr int kf42_ctas_per_sm(int shared, int ring = 0) { return ring ? 4 : shared == 2 ? 5 : (shared ? 4 : 3); }

// PAT (the fused ring only): the structural words the instance takes as constants (WordPattern)
template <int MODE, int SHARED, bool EXTRAS, int REC = 0, int RING = 0, class PAT = NoPattern>
__global__ void __launch_bounds__(TILE, kf42_ctas_per_sm(SHARED, RING))
kf42_f32_kernel(const __grid_constant__ FastP<4, 2> p)
{
    constexpr int N = 4, M = 2;
    static_assert(!(REC && SHARED), "the packed records hold per-filter models");
    static_assert(!RING || (MODE == 3 && REC == 2 && !EXTRAS), "the fused ring steps the packed model words");
    static_assert(!PAT::any || RING, "a pattern instance is a fused ring");
    constexpr int ZS = RING ? RING : 1;
    using St = Stage<float, N, M, SHARED != 0, REC, ZS>;
    // REC == 1: the part of a tile's record this MODE reads (the Q planes, the R planes or both)
    constexpr int SYM_FIRST = (MODE & 1) ? 0 : SYM_Q_PLANES;
    constexpr int SYM_LAST = (MODE & 2) ? SYM_PLANES : SYM_Q_PLANES;
    constexpr uint32_t SYM_BYTES = (SYM_LAST - SYM_FIRST) * TILE * 4;
    constexpr bool DO_P = MODE & 1, DO_U = MODE & 2;
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) uint64_t full[STAGES];

    const int tid = threadIdx.x;
    const int stage_bytes = RING ? p.ring_stage : St::BYTES, off_x = RING ? p.ring_ox : St::OX,
              off_z = RING ? p.ring_oz : St::OZ;

    const uint64_t pol_first = policy_evict_first(), pol_last = policy_evict_last();
    // the tile's blocks are contiguous byte ranges; a ragged last tile copies only its own filters
    // (z: 8 B per filter, rounded down to the 16-byte granule; an odd last filter reads its own z)
    // (tile: the bank's tile, not the position in the launch order)
    auto issue = [&](int tile, int stage) {
        unsigned char *sb = smem + stage * stage_bytes;
        uint64_t *bar = &full[stage];
        const int64_t f0 = (int64_t)tile * TILE;
        const int64_t left = p.N_filters - f0;
        const uint32_t nf = left < TILE ? (uint32_t)left : (uint32_t)TILE;
        const uint32_t zb = (nf * M * 4) & ~15u;
        uint32_t tx = nf * (N + N * N) * 4;
        if (!SHARED && REC != 2 && DO_P) tx += nf * (REC ? 1 : 2) * N * N * 4;
        if (!SHARED && REC != 2 && DO_U) tx += nf * (M * N + (REC ? 0 : M * M)) * 4;
        // the records are padded to whole tiles: always the full planes
        if (REC == 1) tx += SYM_BYTES;
        if (REC == 2) tx += (uint32_t)p.rec_copy * TILE * 4;
        if (DO_U) tx += RING ? p.n_steps * zb : zb;
        mbar_expect_tx(bar, tx);
        auto load = [&](int off, const float *src, int per_filter, uint32_t bytes, uint64_t pol) {
            if (p.l2_hints) bulk_load_hint(sb + off, src + f0 * per_filter, bytes, bar, pol);
            else bulk_load(sb + off, src + f0 * per_filter, bytes, bar);
        };
        load(St::OP, p.P, N * N, nf * N * N * 4, pol_last);
        load(off_x, p.x, N, nf * N * 4, pol_last);
        if (!SHARED && REC != 2 && DO_P) {
            load(St::OF, p.F, N * N, nf * N * N * 4, pol_first);
            if (!REC) load(St::OQ, p.Q, N * N, nf * N * N * 4, pol_first);
        }
        if (!SHARED && REC != 2 && DO_U) {
            load(St::OH, p.H, M * N, nf * M * N * 4, pol_first);
            if (!REC) load(St::OR_, p.R, M * M, nf * M * M * 4, pol_first);
        }
        if (REC == 1) load(St::OQ + SYM_FIRST * TILE * 4, p.rec + SYM_FIRST * TILE, SYM_PLANES, SYM_BYTES, pol_first);
        if (REC == 2)
            for (int r = 0; r < p.rec_runs; r++)
                load(St::OQ + p.run_first[r] * TILE * 4, p.rec + p.run_first[r] * TILE, p.rec_planes,
                     p.run_len[r] * TILE * 4, pol_first);
        if (!RING && DO_U && zb) load(St::OZ, p.z, M, zb, pol_first);
        if (RING && zb)
            for (int k = 0; k < p.n_steps; k++) load(off_z + k * St::align_up(St::ZB), p.zs[k], M, zb, pol_first);
    };

    // prologue: nothing here touches global memory, so it may overlap the previous launch
    if (tid == 0) {
        for (int s = 0; s < STAGES; s++) mbar_init(&full[s], 1);
        fence_mbar_init();
    }
    float F[N][N], Q[N][N], H[M][N], R[M][M];
    if (SHARED == 2) {
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int j = 0; j < N; j++) { F[i][j] = p.Fh[i * N + j]; Q[i][j] = p.Qh[i * N + j]; }
#pragma unroll
        for (int a = 0; a < M; a++) {
#pragma unroll
            for (int j = 0; j < N; j++) H[a][j] = p.Hh[a * N + j];
#pragma unroll
            for (int b = 0; b < M; b++) R[a][b] = p.Rh[a * M + b];
        }
    }
    // Every read and write of global memory comes after this point: the previous kernel on the
    // stream (the previous step, or whatever produced z) may have written any of it, and only
    // griddepcontrol.wait makes those writes visible.
    griddep_wait();
    // RING with an order word: the launch walks the bank last to first when the bank's count of such launches
    // (epoch) is odd, so that consecutive launches alternate whether they come from one graph replay or from
    // two.  Read once per CTA, after the wait (the previous launch may have advanced it), and shared.
    __shared__ uint32_t order_epoch;
    if (RING && p.order && tid == 0) order_epoch = ld_relaxed_gpu(p.order);
    __syncthreads();
    // Launch-order tile t stands for the bank's tile base + sign t; both are formed once from the
    // parameters (or the order word), so that the per-tile address arithmetic stays uniform.
    const int reverse = RING && p.order ? (int)(order_epoch & 1u) : p.reverse;
    const int base = reverse ? p.num_tiles - 1 : 0, sign = reverse ? -1 : 1;
    if (tid == 0) {
        for (int s = 0; s < STAGES; s++) {
            int tile = blockIdx.x + s * gridDim.x;
            if (tile < p.num_tiles) issue(base + sign * tile, s);
        }
    }
    if (SHARED == 1) {
        if (DO_P) {
#pragma unroll
            for (int i = 0; i < N; i++)
#pragma unroll
                for (int j = 0; j < N; j++) { F[i][j] = __ldg(p.F + i * N + j); Q[i][j] = __ldg(p.Q + i * N + j); }
        }
        if (DO_U) {
#pragma unroll
            for (int a = 0; a < M; a++) {
#pragma unroll
                for (int j = 0; j < N; j++) H[a][j] = __ldg(p.H + a * N + j);
#pragma unroll
                for (int b = 0; b < M; b++) R[a][b] = __ldg(p.R + a * M + b);
            }
        }
    }

    int it = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, it++) {
        const int stage = it % STAGES;
        const uint32_t parity = (it / STAGES) & 1;
        const unsigned char *sb = smem + stage * stage_bytes;
        mbar_wait(&full[stage], parity);

        float x[N], P[N][N], z[ZS][M];
        {
            float4 v = lds_chunk<16>(sb + off_x, tid, 0);
            x[0] = v.x; x[1] = v.y; x[2] = v.z; x[3] = v.w;
        }
        lds_row<N>(sb + St::OP, tid, P);
        // REC: word `tid` of a plane of the record (no bank conflicts); the lower triangles are the same
        // registers.  REC == 1 holds all 13 Q / R words, in order; REC == 2 the words in p.varying, and
        // the others are the bank's shared values.  (The shared values are run-time parameters, so the
        // arithmetic is the same instructions as with a dense model: nothing is folded away.  A pattern
        // instance's structural words are constants instead, and its arithmetic drops or folds them.)
        const unsigned char *rec = sb + St::OQ + tid * 4;
        auto word = [&](int e, float shared) -> float {
            if (PAT::structural(e)) return (PAT::ONE >> e) & 1 ? 1.f : 0.f;
            if (REC == 1) return *reinterpret_cast<const float *>(rec + (e < W_H ? e - W_Q : e - W_R + SYM_Q_PLANES) * TILE * 4);
            return (p.varying >> e) & 1 ? *reinterpret_cast<const float *>(rec + p.slot_off[e]) : shared;
        };
        if (!SHARED && DO_P) {
            if (REC == 2) {
#pragma unroll
                for (int i = 0; i < N; i++)
#pragma unroll
                    for (int j = 0; j < N; j++) F[i][j] = word(W_F + i * N + j, p.Fh[i * N + j]);
            } else {
                lds_row<N>(sb + St::OF, tid, F);
            }
            if (REC) {
                int k = W_Q;
#pragma unroll
                for (int i = 0; i < N; i++)
#pragma unroll
                    for (int j = i; j < N; j++, k++) Q[i][j] = Q[j][i] = word(k, p.Qh[i * N + j]);
            } else {
                lds_row<N>(sb + St::OQ, tid, Q);
            }
        }
        if (!SHARED && DO_U) {
            if (REC == 2) {
#pragma unroll
                for (int a = 0; a < M; a++)
#pragma unroll
                    for (int j = 0; j < N; j++) H[a][j] = word(W_H + a * N + j, p.Hh[a * N + j]);
            } else {
                lds_row<M>(sb + St::OH, tid, H);
            }
            if (REC) {
                R[0][0] = word(W_R, p.Rh[0]);
                R[0][1] = R[1][0] = word(W_R + 1, p.Rh[1]);
                R[1][1] = word(W_R + 2, p.Rh[3]);
            } else {
                float4 r = lds_chunk<16>(sb + St::OR_, tid, 0);
                R[0][0] = r.x; R[0][1] = r.y; R[1][0] = r.z; R[1][1] = r.w;
            }
        }
        const int64_t f = (int64_t)(base + sign * tile) * TILE + tid;
        const bool live = f < p.N_filters;
        if (DO_U) {
            // the stage holds z up to the last whole 16 bytes: only an odd last filter misses its own
            const bool own = live && (p.N_filters & 1) && f == p.N_filters - 1;
            if (!RING) {
                float2 v = own ? *reinterpret_cast<const float2 *>(p.z + f * M)
                               : *reinterpret_cast<const float2 *>(sb + St::OZ + tid * 8);
                z[0][0] = v.x; z[0][1] = v.y;
            }
            // the ring: every step's measurement into registers now, so that nothing reads the stage after
            // the barrier below (unrolled to the longest ring under a uniform guard: no run-time index
            // into z[][])
#pragma unroll
            for (int k = 0; k < RING; k++) {
                float2 v = make_float2(0.f, 0.f);
                if (k < p.n_steps)
                    v = own ? *reinterpret_cast<const float2 *>(p.zs[k] + f * M)
                            : *reinterpret_cast<const float2 *>(sb + off_z + k * St::align_up(St::ZB) + tid * 8);
                z[k][0] = v.x; z[k][1] = v.y;
            }
        }
        // The stage is about to be handed back to the TMA engine (async proxy).  A plain barrier
        // does not order the generic-proxy LDS above against that: the loads may still sit in the
        // LSU queue when the barrier releases, and a TMA refill served from L2 can land first
        // (observed in round 1: a few filters per launch picked up rows of the NEXT tile).  Two
        // fixes were measured: a cross-proxy fence (MEMBAR.ALL.CTA + FENCE.VIEW.ASYNC, which also
        // waits for the previous tile's global stores) and the one used here: fold every loaded
        // register into the predicate of the barrier itself (BAR.RED), so the barrier instruction
        // cannot issue before all LDS results have returned.
        unsigned acc = 0;
#pragma unroll
        for (int i = 0; i < N; i++) {
            acc ^= __float_as_uint(x[i]);
#pragma unroll
            for (int j = 0; j < N; j++) acc ^= __float_as_uint(P[i][j]);
        }
        // (REC: each loaded word once; folding a mirrored pair would cancel it out of the predicate.
        // REC == 2 folds every model word: a shared one is a launch parameter and harmless in it; a
        // structural word of PAT is a constant and is left out)
        if (!SHARED && DO_P) {
#pragma unroll
            for (int i = 0; i < N; i++)
#pragma unroll
                for (int j = 0; j < N; j++) {
                    if (!PAT::structural(W_F + i * N + j)) acc ^= __float_as_uint(F[i][j]);
                    if ((!REC || j >= i) && !PAT::structural(q_word(i, j))) acc ^= __float_as_uint(Q[i][j]);
                }
        }
        if (!SHARED && DO_U) {
#pragma unroll
            for (int a = 0; a < M; a++) {
#pragma unroll
                for (int j = 0; j < N; j++)
                    if (!PAT::structural(W_H + a * N + j)) acc ^= __float_as_uint(H[a][j]);
#pragma unroll
                for (int b = 0; b < M; b++)
                    if ((!REC || b >= a) && !PAT::structural(W_R + a + b)) acc ^= __float_as_uint(R[a][b]);
            }
        }
        if (DO_U) {
#pragma unroll
            for (int k = 0; k < ZS; k++) acc ^= __float_as_uint(z[k][0]) ^ __float_as_uint(z[k][1]);
        }
        const int never = __syncthreads_and(acc == 0x7fc0beefu);     // every thread has drained the stage
        if (never && p.num_tiles < 0) p.x_out[0] = 0.f;              // keeps `acc` alive; cannot happen
        const int nt = tile + STAGES * gridDim.x;
        if (nt < p.num_tiles) {
            if (tid == 0) issue(base + sign * nt, stage);
        } else {
            // this CTA has issued the loads of its last tile: the next launch on the stream may
            // take the SM slots this grid frees and run its prologue (it waits before touching memory)
            griddep_launch_dependents();
        }

        int st = BKE_STATUS_OK;
        if (RING) {
            // PAT: the structural words' products are dropped, which is exact for finite operands only
            // (0 Inf is NaN).  nf = the sum of 0 v over every word v the ring reads and every word it writes
            // is NaN when any of them is not finite; such a filter runs the dense ring again (below).
            float nf = 0.f;
            auto check = [&](float v) { nf = __fmaf_rn(0.f, v, nf); };
            if (PAT::any) {
                check(p.alpha_sq);
#pragma unroll
                for (int i = 0; i < N; i++) {
                    check(x[i]);
#pragma unroll
                    for (int j = 0; j < N; j++) {
                        check(P[i][j]);
                        if (!PAT::structural(W_F + i * N + j)) check(F[i][j]);
                        if (j >= i && !PAT::structural(q_word(i, j))) check(Q[i][j]);
                    }
                }
#pragma unroll
                for (int a = 0; a < M; a++) {
#pragma unroll
                    for (int j = 0; j < N; j++)
                        if (!PAT::structural(W_H + a * N + j)) check(H[a][j]);
#pragma unroll
                    for (int b = a; b < M; b++)
                        if (!PAT::structural(W_R + a + b)) check(R[a][b]);
                }
#pragma unroll
                for (int k = 0; k < ZS; k++) { check(z[k][0]); check(z[k][1]); }
            }
            // the steps of the ring, back to back on the registers; the loop stays rolled and the
            // measurements rotate through z[0] instead of being indexed
            // PAT::blocks: a warp whose filters all enter with zeros (of either sign) in the 8 cross words of P runs
            // the two axis blocks.  They leave every step with zeros there again (reg_update_blk), so the choice
            // holds for the whole ring.  A lane past the bank's end stores nothing and does not hold its warp back.
            bool blk = false;
            if constexpr (PAT::blocks()) {
                uint32_t c = 0;
#pragma unroll
                for (int i = 0; i < N; i++)
#pragma unroll
                    for (int j = 0; j < N; j++)
                        if (blk_cross(i, j)) c |= __float_as_uint(P[i][j]);
                blk = __all_sync(FULL, !live || (c & 0x7fffffffu) == 0);
                if (blk) {
#pragma unroll 1
                    for (int k = 0; k < p.n_steps; k++) {
                        reg_predict_blk<PAT, N>(x, P, F, Q, p.alpha_sq);
                        reg_update_blk<PAT, N, M>(x, P, H, R, z[0]);
#pragma unroll
                        for (int j = 0; j + 1 < ZS; j++) { z[j][0] = z[j + 1][0]; z[j][1] = z[j + 1][1]; }
                    }
                }
            }
            // the steps of the ring, back to back on the registers; the loop stays rolled and the
            // measurements rotate through z[0] instead of being indexed
#pragma unroll 1
            for (int k = 0; k < (blk ? 0 : p.n_steps); k++) {       // (none left after the block path)
                if (PAT::any) {
                    reg_predict_pat<PAT, N>(x, P, F, Q, p.alpha_sq);
                    reg_update_pat<PAT, N, M>(x, P, H, R, z[0]);
                } else {
                    reg_predict<float, N>(x, P, F, Q, p.alpha_sq);
                    KfUpdateOut<float, N, M> o;
                    reg_update<float, N, M>(x, P, H, R, z[0], o);
                }
#pragma unroll
                for (int j = 0; j + 1 < ZS; j++) { z[j][0] = z[j + 1][0]; z[j][1] = z[j + 1][1]; }
            }
            if (PAT::any) {
#pragma unroll
                for (int i = 0; i < N; i++) {
                    check(x[i]);
#pragma unroll
                    for (int j = 0; j < N; j++) check(P[i][j]);
                }
            }
            if (PAT::any && live && nf != 0.f) {
                // The dense ring on this filter's inputs, as the generic instance runs it.  They are still in
                // global memory: the ring steps in place, only this thread writes filter f (below), and no z
                // overlaps the state.  A structural word is the bank's shared value (a launch parameter).
                const float *rec = p.rec + (int64_t)(base + sign * tile) * p.rec_planes * TILE + tid;
                auto gword = [&](int e, float shared) -> float {
                    if (PAT::structural(e)) return shared;
                    return (p.varying >> e) & 1 ? rec[p.slot_off[e] / 4] : shared;
                };
                float Fd[N][N], Qd[N][N], Hd[M][N], Rd[M][M];
#pragma unroll
                for (int i = 0, e = W_Q; i < N; i++) {
#pragma unroll
                    for (int j = 0; j < N; j++) Fd[i][j] = gword(W_F + i * N + j, p.Fh[i * N + j]);
#pragma unroll
                    for (int j = i; j < N; j++, e++) Qd[i][j] = Qd[j][i] = gword(e, p.Qh[i * N + j]);
                }
#pragma unroll
                for (int a = 0; a < M; a++)
#pragma unroll
                    for (int j = 0; j < N; j++) Hd[a][j] = gword(W_H + a * N + j, p.Hh[a * N + j]);
                Rd[0][0] = gword(W_R, p.Rh[0]);
                Rd[0][1] = Rd[1][0] = gword(W_R + 1, p.Rh[1]);
                Rd[1][1] = gword(W_R + 2, p.Rh[3]);
                const float4 vx = *reinterpret_cast<const float4 *>(p.x + f * N);
                x[0] = vx.x; x[1] = vx.y; x[2] = vx.z; x[3] = vx.w;
#pragma unroll
                for (int i = 0; i < N; i++) {
                    const float4 v = *reinterpret_cast<const float4 *>(p.P + f * N * N + i * N);
                    P[i][0] = v.x; P[i][1] = v.y; P[i][2] = v.z; P[i][3] = v.w;
                }
#pragma unroll 1
                for (int k = 0; k < p.n_steps; k++) {
                    const float2 v = *reinterpret_cast<const float2 *>(p.zs[k] + f * M);
                    const float zk[M] = {v.x, v.y};
                    reg_predict<float, N>(x, P, Fd, Qd, p.alpha_sq);
                    KfUpdateOut<float, N, M> o;
                    reg_update<float, N, M>(x, P, Hd, Rd, zk, o);
                }
            }
        }
        if (!RING && DO_P) {
            reg_predict<float, N>(x, P, F, Q, p.alpha_sq);
            if (EXTRAS && live) {
                if (p.x_prior) *reinterpret_cast<float4 *>(p.x_prior + f * N) = make_float4(x[0], x[1], x[2], x[3]);
                if (p.P_prior) {
#pragma unroll
                    for (int i = 0; i < N; i++)
                        *reinterpret_cast<float4 *>(p.P_prior + f * N * N + i * N) = make_float4(P[i][0], P[i][1], P[i][2], P[i][3]);
                }
            }
        }
        if (!RING && DO_U) {
            bool has_z = true;
            if (p.valid != nullptr && live) has_z = p.valid[f] != 0;
            KfUpdateOut<float, N, M> o;
            if (has_z) {
                reg_update<float, N, M>(x, P, H, R, z[0], o);
                if (!o.ok) st = BKE_STATUS_SINGULAR_S;
            }
            if (EXTRAS && live) {
                if (!has_z) {
                    if (p.y) *reinterpret_cast<float2 *>(p.y + f * M) = make_float2(0.f, 0.f);
                } else {
                    if (p.S) *reinterpret_cast<float4 *>(p.S + f * M * M) = make_float4(o.S[0][0], o.S[0][1], o.S[1][0], o.S[1][1]);
                    if (o.ok) {
                        if (p.y) *reinterpret_cast<float2 *>(p.y + f * M) = make_float2(o.y[0], o.y[1]);
                        if (p.SI) *reinterpret_cast<float4 *>(p.SI + f * M * M) = make_float4(o.SI[0][0], o.SI[0][1], o.SI[1][0], o.SI[1][1]);
                        if (p.K) {
                            *reinterpret_cast<float4 *>(p.K + f * N * M) = make_float4(o.K[0][0], o.K[0][1], o.K[1][0], o.K[1][1]);
                            *reinterpret_cast<float4 *>(p.K + f * N * M + 4) = make_float4(o.K[2][0], o.K[2][1], o.K[3][0], o.K[3][1]);
                        }
                        if (p.ll) {
                            float q = 0.f;
#pragma unroll
                            for (int a = 0; a < M; a++) {
                                float s = 0.f;
#pragma unroll
                                for (int b = 0; b < M; b++) s += o.SI[a][b] * o.y[b];
                                q += o.y[a] * s;
                            }
                            p.ll[f] = -0.5f * (q + o.logdet + float(M) * float(LOG_2PI));
                        }
                    }
                }
            }
        }
        if (live) {
            if (p.l2_hints) {
                st_hint(p.x_out + f * N, make_float4(x[0], x[1], x[2], x[3]), pol_last);
#pragma unroll
                for (int i = 0; i < N; i++)
                    st_hint(p.P_out + f * N * N + i * N, make_float4(P[i][0], P[i][1], P[i][2], P[i][3]), pol_last);
            } else {
                *reinterpret_cast<float4 *>(p.x_out + f * N) = make_float4(x[0], x[1], x[2], x[3]);
#pragma unroll
                for (int i = 0; i < N; i++)
                    *reinterpret_cast<float4 *>(p.P_out + f * N * N + i * N) = make_float4(P[i][0], P[i][1], P[i][2], P[i][3]);
            }
            if (EXTRAS && p.status && (st != BKE_STATUS_OK || !p.sticky)) p.status[f] = st;
        }
    }
    // Advance the order word: every CTA arrives once, after its read of epoch; the last to arrive resets the
    // count and bumps epoch.  No CTA of this launch reads epoch after that, and the next launch reads it only
    // after its griddepcontrol.wait, which sees every write of this one.
    if (RING && p.order && tid == 0) {
        if (atom_add_acq_rel_gpu(p.order + 1, 1u) == gridDim.x - 1) {
            p.order[1] = 0u;
            p.order[0] = order_epoch + 1u;
        }
    }
}

// ---------------------------------------------------------------------------- host side
template <int MODE, int SHARED, bool EXTRAS, int REC = 0, int RING = 0, class PAT = NoPattern>
int launch_variant(const FastP<4, 2> &p, cudaStream_t s)
{
    using St = Stage<float, 4, 2, SHARED != 0, REC, RING ? RING : 1>;
    auto kern = kf42_f32_kernel<MODE, SHARED, EXTRAS, REC, RING, PAT>;
    // (the ring's stage is laid out per launch and never exceeds St::BYTES)
    const int smem = STAGES * (RING ? p.ring_stage : St::BYTES);
    static bool configured[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !configured[dev]) {
        if (check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, STAGES * St::BYTES),
                       "cudaFuncSetAttribute")) return BKE_ERR_CUDA;
        if (dev >= 0 && dev < 64) configured[dev] = true;
    }
    int ctas = kf42_ctas_per_sm(SHARED, RING);
    if (RING) {
        // the resident CTAs at this launch's shared memory, per device and stage size (a stage is a whole
        // number of 512 B units); the first launch of a shape queries it, so a captured launch finds it
        constexpr int UNITS = STAGES * St::BYTES / 512 + 1;
        static int resident[64][UNITS] = {};
        const int unit = smem / 512;
        int *r = dev >= 0 && dev < 64 && unit < UNITS ? &resident[dev][unit] : nullptr;
        if (!r || *r == 0) {
            int n = 0;
            if (check_cuda(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, TILE, smem), "cudaOccupancyMaxActiveBlocksPerMultiprocessor"))
                return BKE_ERR_CUDA;
            if (n < 1) n = 1;
            if (r) *r = n;
            ctas = n;
        } else {
            ctas = *r;
        }
    }
    int grid = sm_count() * ctas;
    if (grid > p.num_tiles) grid = p.num_tiles;
    // programmatic stream serialization: this launch may start while the previous kernel on the
    // stream drains (the kernel waits with griddepcontrol.wait before it touches memory); under
    // stream capture it becomes a programmatic edge of the graph
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(TILE);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return check_cuda(cudaLaunchKernelEx(&cfg, kern, p), "kf42_f32_kernel launch");
}

// Pack the per-filter Q [N,4,4] and R [N,2,2] of a bank into the record described at SYM_PLANES, one
// thread per filter slot (the padding of the last tile is written with zeros), and set *asym when a
// filter's Q or R differs from its transpose in any bit.
__global__ void __launch_bounds__(256)
kf42_pack_sym_kernel(int64_t n_filters, int64_t slots, const float4 *__restrict__ Q, const float4 *__restrict__ R,
                     float *__restrict__ rec, int32_t *asym)
{
    for (int64_t f = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; f < slots; f += (int64_t)gridDim.x * blockDim.x) {
        float v[SYM_PLANES] = {};
        bool bad = false;
        if (f < n_filters) {
            float q[4][4];
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const float4 r = Q[f * 4 + i];
                q[i][0] = r.x; q[i][1] = r.y; q[i][2] = r.z; q[i][3] = r.w;
            }
            const float4 r = R[f];
            int k = 0;
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = i; j < 4; j++, k++) {
                    v[k] = q[i][j];
                    bad |= __float_as_uint(q[i][j]) != __float_as_uint(q[j][i]);
                }
            v[SYM_Q_PLANES] = r.x; v[SYM_Q_PLANES + 1] = r.y; v[SYM_Q_PLANES + 2] = r.w;
            bad |= __float_as_uint(r.y) != __float_as_uint(r.z);
        }
        float *out = rec + (f / TILE) * (SYM_PLANES * TILE) + (f % TILE);
#pragma unroll
        for (int k = 0; k < SYM_PLANES; k++) out[k * TILE] = v[k];
        if (bad) *asym = 1;
    }
}

// The 37 model words of filter f (order at WORDS) from the dense F [N,4,4], Q [N,4,4], H [N,2,4], R [N,2,2];
// *asym is set when Q or R differs from its transpose in any bit.
__device__ __forceinline__ void kf42_model_words(const float4 *__restrict__ F, const float4 *__restrict__ Q,
                                                 const float4 *__restrict__ H, const float4 *__restrict__ R,
                                                 int64_t f, float (&w)[WORDS], bool &asym)
{
    float q[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const float4 a = F[f * 4 + i], b = Q[f * 4 + i];
        w[W_F + 4 * i] = a.x; w[W_F + 4 * i + 1] = a.y; w[W_F + 4 * i + 2] = a.z; w[W_F + 4 * i + 3] = a.w;
        q[i][0] = b.x; q[i][1] = b.y; q[i][2] = b.z; q[i][3] = b.w;
    }
    asym = false;
    int k = W_Q;
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = i; j < 4; j++, k++) {
            w[k] = q[i][j];
            asym |= __float_as_uint(q[i][j]) != __float_as_uint(q[j][i]);
        }
#pragma unroll
    for (int a = 0; a < 2; a++) {
        const float4 h = H[f * 2 + a];
        w[W_H + 4 * a] = h.x; w[W_H + 4 * a + 1] = h.y; w[W_H + 4 * a + 2] = h.z; w[W_H + 4 * a + 3] = h.w;
    }
    const float4 r = R[f];
    w[W_R] = r.x; w[W_R + 1] = r.y; w[W_R + 2] = r.w;
    asym |= __float_as_uint(r.y) != __float_as_uint(r.z);
}

// Scan pass: OR into map->varying the words in which a filter differs from filter 0 (as bits), and set
// map->asymmetric when one is asymmetric; block 0 also writes filter 0's words.  The caller zeroed both.
__global__ void __launch_bounds__(256)
kf42_scan_models_kernel(int64_t n_filters, const float4 *__restrict__ F, const float4 *__restrict__ Q,
                        const float4 *__restrict__ H, const float4 *__restrict__ R, bke_kf_model_map *map)
{
    float w0[WORDS], w[WORDS];
    bool asym = false, a;
    kf42_model_words(F, Q, H, R, 0, w0, a);
    uint32_t lo = 0, hi = 0;
    for (int64_t f = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; f < n_filters; f += (int64_t)gridDim.x * blockDim.x) {
        kf42_model_words(F, Q, H, R, f, w, a);
        asym |= a;
#pragma unroll
        for (int e = 0; e < WORDS; e++) {
            const uint32_t d = __float_as_uint(w[e]) != __float_as_uint(w0[e]);
            if (e < 32) lo |= d << e;
            else hi |= d << (e - 32);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
#pragma unroll
        for (int e = 0; e < WORDS; e++) map->words[e] = w0[e];
    }
    __shared__ uint32_t red[3][8];
    lo = __reduce_or_sync(FULL, lo);
    hi = __reduce_or_sync(FULL, hi);
    const uint32_t as = __reduce_or_sync(FULL, asym ? 1u : 0u);
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    if (lane == 0) { red[0][warp] = lo; red[1][warp] = hi; red[2][warp] = as; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < (int)blockDim.x / 32; i++) { lo |= red[0][i]; hi |= red[1][i]; }
        uint32_t as_all = 0;
        for (int i = 0; i < (int)blockDim.x / 32; i++) as_all |= red[2][i];
        const unsigned long long v = (unsigned long long)hi << 32 | lo;
        if (v) atomicOr(reinterpret_cast<unsigned long long *>(&map->varying), v);
        if (as_all) atomicOr(&map->asymmetric, 1);
    }
}

// Second scan pass, after kf42_scan_models_kernel on the same stream (which wrote map->varying and
// map->words): AND into map->duplicate, which the caller set to all ones, the slots s < 32 that have a
// candidate c(s) (the rule at bke_kf_model_map) and whose word equals the candidate's, as bits, in every
// filter the block covers.  Each thread keeps its filter's words in its own column of shared memory, so
// the candidate pairs are read at run-time indices without a local-memory array.
__global__ void __launch_bounds__(256)
kf42_scan_duplicates_kernel(int64_t n_filters, const float4 *__restrict__ F, const float4 *__restrict__ Q,
                            const float4 *__restrict__ H, const float4 *__restrict__ R, bke_kf_model_map *map)
{
    __shared__ float col[WORDS][256];
    __shared__ uint8_t pair_e[32], pair_c[32], pair_s[32];
    __shared__ int n_pairs;
    __shared__ uint32_t cand;
    __shared__ uint32_t red[8];
    const int tid = threadIdx.x;
    if (tid == 0) {
        const uint64_t v = map->varying;
        int slot_word[32], n = 0;
        uint32_t c = 0;
        for (int e = 0, s = 0; e < WORDS && s < 32; e++) {
            if (!((v >> e) & 1)) continue;
            slot_word[s] = e;
            for (int t = 0; t < s; t++)
                if (__float_as_uint(map->words[slot_word[t]]) == __float_as_uint(map->words[e])) {
                    pair_e[n] = e; pair_c[n] = slot_word[t]; pair_s[n] = s; n++;
                    c |= 1u << s;
                    break;
                }
            s++;
        }
        n_pairs = n;
        cand = c;
    }
    __syncthreads();
    const int n = n_pairs;
    uint32_t differs = 0;
    if (n) {
        for (int64_t f = blockIdx.x * (int64_t)blockDim.x + tid; f < n_filters; f += (int64_t)gridDim.x * blockDim.x) {
            float w[WORDS];
            bool a;
            kf42_model_words(F, Q, H, R, f, w, a);
#pragma unroll
            for (int e = 0; e < WORDS; e++) col[e][tid] = w[e];
            for (int i = 0; i < n; i++)
                differs |= (uint32_t)(__float_as_uint(col[pair_e[i]][tid]) != __float_as_uint(col[pair_c[i]][tid])) << pair_s[i];
        }
    }
    differs = __reduce_or_sync(FULL, differs);
    if (tid % 32 == 0) red[tid / 32] = differs;
    __syncthreads();
    if (tid == 0) {
        for (int i = 1; i < (int)blockDim.x / 32; i++) differs |= red[i];
        atomicAnd(&map->duplicate, cand & ~differs);
    }
}

// Pack pass: the words in `varying` of every filter slot into the record described at WORDS (the
// padding of the last tile is written with zeros), one thread per slot.
__global__ void __launch_bounds__(256)
kf42_pack_models_kernel(int64_t n_filters, int64_t slots, const float4 *__restrict__ F, const float4 *__restrict__ Q,
                        const float4 *__restrict__ H, const float4 *__restrict__ R, uint64_t varying, int planes,
                        float *__restrict__ rec)
{
    for (int64_t f = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; f < slots; f += (int64_t)gridDim.x * blockDim.x) {
        float w[WORDS] = {};
        bool a;
        if (f < n_filters) kf42_model_words(F, Q, H, R, f, w, a);
        float *out = rec + (f / TILE) * ((int64_t)planes * TILE) + (f % TILE);
        int s = 0;
#pragma unroll
        for (int e = 0; e < WORDS; e++)
            if ((varying >> e) & 1) out[(s++) * TILE] = w[e];
    }
}

bool misaligned16(const void *p) { return p != nullptr && (reinterpret_cast<uintptr_t>(p) & 15u) != 0; }

}  // namespace

size_t kf_sym_models_bytes(int64_t n_filters)
{
    if (n_filters <= 0) return 0;
    return (size_t)((n_filters + TILE - 1) / TILE) * SYM_PLANES * TILE * sizeof(float);
}

int launch_kf_pack_sym(int64_t n_filters, const void *Q, const void *R, void *record, int32_t *asym, cudaStream_t s)
{
    if (n_filters >= (int64_t)1 << 30) { set_error("the packed symmetric models take at most 2^30 filters"); return BKE_ERR_UNSUPPORTED; }
    if (misaligned16(Q) || misaligned16(R) || misaligned16(record)) {
        set_error("Q, R and record must be 16-byte aligned");
        return BKE_ERR_UNSUPPORTED;
    }
    if (check_cuda(cudaMemsetAsync(asym, 0, sizeof(int32_t), s), "cudaMemsetAsync")) return BKE_ERR_CUDA;
    const int64_t slots = (n_filters + TILE - 1) / TILE * TILE;
    if (slots == 0) return BKE_OK;
    int64_t grid = (slots + 255) / 256;
    if (grid > (int64_t)sm_count() * 16) grid = (int64_t)sm_count() * 16;
    kf42_pack_sym_kernel<<<(int)grid, 256, 0, s>>>(n_filters, slots, (const float4 *)Q, (const float4 *)R,
                                                   (float *)record, asym);
    return check_cuda(cudaGetLastError(), "kf42_pack_sym_kernel launch");
}

size_t kf_packed_models_bytes(int64_t n_filters, uint64_t varying)
{
    if (n_filters <= 0 || (varying >> WORDS) != 0) return 0;
    return (size_t)((n_filters + TILE - 1) / TILE) * __builtin_popcountll(varying) * TILE * sizeof(float);
}

static int check_models(int64_t n_filters, const void *F, const void *Q, const void *H, const void *R, const void *out)
{
    if (n_filters >= (int64_t)1 << 30) { set_error("the packed models take at most 2^30 filters"); return BKE_ERR_UNSUPPORTED; }
    if (misaligned16(F) || misaligned16(Q) || misaligned16(H) || misaligned16(R) || misaligned16(out)) {
        set_error("F, Q, H, R and the map or record must be 16-byte aligned");
        return BKE_ERR_UNSUPPORTED;
    }
    return BKE_OK;
}

static int64_t pass_grid(int64_t threads)
{
    const int64_t grid = (threads + 255) / 256;
    return grid < (int64_t)sm_count() * 16 ? grid : (int64_t)sm_count() * 16;
}

int launch_kf_scan_models(int64_t n_filters, const void *F, const void *Q, const void *H, const void *R,
                          bke_kf_model_map *map, cudaStream_t s)
{
    int rc = check_models(n_filters, F, Q, H, R, map);
    if (rc) return rc;
    // varying and asymmetric start at zero, duplicate (for a bank of filters) at all ones; filter 0's words
    // are written by the first kernel
    if (check_cuda(cudaMemsetAsync(map, 0, sizeof(bke_kf_model_map), s), "cudaMemsetAsync")) return BKE_ERR_CUDA;
    if (n_filters == 0) return BKE_OK;
    if (check_cuda(cudaMemsetAsync(&map->duplicate, 0xff, sizeof(map->duplicate), s), "cudaMemsetAsync")) return BKE_ERR_CUDA;
    const int grid = (int)pass_grid(n_filters);
    kf42_scan_models_kernel<<<grid, 256, 0, s>>>(n_filters, (const float4 *)F, (const float4 *)Q, (const float4 *)H,
                                                 (const float4 *)R, map);
    if (check_cuda(cudaGetLastError(), "kf42_scan_models_kernel launch")) return BKE_ERR_CUDA;
    kf42_scan_duplicates_kernel<<<grid, 256, 0, s>>>(n_filters, (const float4 *)F, (const float4 *)Q, (const float4 *)H,
                                                     (const float4 *)R, map);
    return check_cuda(cudaGetLastError(), "kf42_scan_duplicates_kernel launch");
}

int kf_model_planes(const bke_kf_model_map &map, int (&plane)[WORDS])
{
    const int k = __builtin_popcountll(map.varying);
    if (k < 32 && (map.duplicate >> k) != 0) {
        set_error("duplicate flags slot %d, but only %d words vary", 31 - __builtin_clz(map.duplicate), k);
        return BKE_ERR_BAD_ARG;
    }
    int slot_word[WORDS];
    for (int e = 0, s = 0; e < WORDS; e++) {
        plane[e] = -1;
        if (!((map.varying >> e) & 1)) continue;
        slot_word[s] = e;
        plane[e] = s;
        if (s < 32 && ((map.duplicate >> s) & 1)) {
            uint32_t we, wt;
            memcpy(&we, &map.words[e], 4);
            int t = 0;
            for (; t < s; t++) {
                memcpy(&wt, &map.words[slot_word[t]], 4);
                if (wt == we) break;
            }
            if (t == s) {
                set_error("duplicate flags slot %d (word %d), but no earlier slot has the same filter-0 word", s, e);
                return BKE_ERR_BAD_ARG;
            }
            plane[e] = t;
        }
        s++;
    }
    return BKE_OK;
}

int launch_kf_pack_models(int64_t n_filters, const void *F, const void *Q, const void *H, const void *R, uint64_t varying,
                          void *record, cudaStream_t s)
{
    int rc = check_models(n_filters, F, Q, H, R, record);
    if (rc) return rc;
    const int64_t slots = (n_filters + TILE - 1) / TILE * TILE;
    if (slots == 0 || varying == 0) return BKE_OK;
    kf42_pack_models_kernel<<<(int)pass_grid(slots), 256, 0, s>>>(n_filters, slots, (const float4 *)F, (const float4 *)Q,
                                                                  (const float4 *)H, (const float4 *)R, varying,
                                                                  __builtin_popcountll(varying), (float *)record);
    return check_cuda(cudaGetLastError(), "kf42_pack_models_kernel launch");
}

int launch_kf_fast(const bke_kf_args &a, cudaStream_t s, const void *rec, const bke_kf_model_map *map,
                   const void *const *zs, int n_steps)
{
    const bool packed = map != nullptr, sym = rec != nullptr && !packed;
    const bool ring = zs != nullptr;        // bke_kf_steps_packed, which has checked what only the ring refuses
    if (misaligned16(rec)) { set_error("record must be 16-byte aligned"); return BKE_ERR_UNSUPPORTED; }
    if (packed && map->asymmetric) { set_error("the map reports an asymmetric Q or R: the bank runs on bke_kf_step"); return BKE_ERR_UNSUPPORTED; }
    if (!(a.dtype == BKE_F32 && a.dim_x == 4 && a.dim_z == 2)) return BKE_ERR_UNSUPPORTED;
    if (a.B != nullptr && a.u != nullptr) return BKE_ERR_UNSUPPORTED;
    if (a.flags & BKE_UPDATE_FIRST) return BKE_ERR_UNSUPPORTED;
    const bool dp = a.flags & BKE_DO_PREDICT, du = a.flags & BKE_DO_UPDATE;
    // every model either per-filter or shared, not a mixture
    bool all_shared = true, all_dense = true;
    if (dp) { all_shared &= (a.F_stride == 0 && a.Q_stride == 0); all_dense &= (a.F_stride != 0 && a.Q_stride != 0); }
    if (du) { all_shared &= (a.H_stride == 0 && a.R_stride == 0); all_dense &= (a.H_stride != 0 && a.R_stride != 0); }
    if (!all_shared && !all_dense) return BKE_ERR_UNSUPPORTED;
    if ((sym || packed) && !all_dense) return BKE_ERR_UNSUPPORTED;
    if (a.n_filters >= (int64_t)1 << 30) return BKE_ERR_UNSUPPORTED;
    // bulk copies and the 16-byte stores need 16-byte aligned global bases
    const auto mis = misaligned16;
    if (mis(a.x) || mis(a.P) || mis(a.F) || mis(a.Q) || mis(a.H) || mis(a.R) || mis(a.z) || mis(a.x_out) || mis(a.P_out) ||
        mis(a.x_prior) || mis(a.P_prior) || mis(a.K) || mis(a.S) || mis(a.SI) || (a.y && (reinterpret_cast<uintptr_t>(a.y) & 7u)))
        return BKE_ERR_UNSUPPORTED;

    const int64_t N = a.n_filters;
    FastP<4, 2> p;
    p.N_filters = N;
    p.num_tiles = (int)((N + TILE - 1) / TILE);
    p.alpha_sq = (float)a.alpha_sq;
    // keep-the-state-in-L2 hints pay off when x, P fit the L2 together with the streaming traffic
    p.l2_hints = (N * 80 <= (int64_t)38 << 20) && a.x_out == a.x && a.P_out == a.P;
    // a bank whose state stays in L2 between steps (l2_hints) has nothing to gain from the order: it
    // keeps walking first to last (a ring given an order word follows the word, which is harmless there)
    p.reverse = (a.flags & BKE_REVERSE_TILES) && !p.l2_hints;
    p.order = ring ? a.tile_order : nullptr;
    p.x = (const float *)a.x; p.P = (const float *)a.P; p.z = (const float *)a.z;
    p.F = (const float *)a.F; p.Q = (const float *)a.Q; p.H = (const float *)a.H; p.R = (const float *)a.R;
    p.rec = (const float *)rec;
    p.x_out = (float *)a.x_out; p.P_out = (float *)a.P_out;
    p.valid = a.z_valid;
    p.x_prior = (float *)a.x_prior; p.P_prior = (float *)a.P_prior; p.K = (float *)a.K; p.y = (float *)a.y;
    p.S = (float *)a.S; p.SI = (float *)a.SI; p.ll = (float *)a.log_likelihood; p.status = a.status;
    p.sticky = (a.flags & BKE_STATUS_STICKY) ? 1 : 0;
    // host copies of the shared models (optional): carried in the launch parameters
    const bool host_models = all_shared && a.F_host && a.Q_host && a.H_host && a.R_host;
    if (host_models) {
        memcpy(p.Fh, a.F_host, sizeof(p.Fh)); memcpy(p.Qh, a.Q_host, sizeof(p.Qh));
        memcpy(p.Hh, a.H_host, sizeof(p.Hh)); memcpy(p.Rh, a.R_host, sizeof(p.Rh));
    }
    if (packed) {
        // the shared words ride in the launch parameters (lower triangles mirrored), the others are
        // read from the record at their plane
        const float *w = map->words;
        memcpy(p.Fh, w + W_F, sizeof(p.Fh));
        memcpy(p.Hh, w + W_H, sizeof(p.Hh));
        for (int i = 0, k = W_Q; i < 4; i++)
            for (int j = i; j < 4; j++, k++) p.Qh[i * 4 + j] = p.Qh[j * 4 + i] = w[k];
        p.Rh[0] = w[W_R]; p.Rh[1] = p.Rh[2] = w[W_R + 1]; p.Rh[3] = w[W_R + 2];
        p.varying = map->varying;
        int plane[WORDS];
        if (int rc = kf_model_planes(*map, plane)) return rc;
        // the planes this MODE reads, copied in runs of consecutive planes
        const uint64_t words = map->varying & ((dp ? PREDICT_WORDS : 0) | (du ? ~PREDICT_WORDS : 0));
        uint64_t read = 0;
        for (int e = 0; e < WORDS; e++) {
            p.slot_off[e] = plane[e] < 0 ? 0 : plane[e] * TILE * 4;
            if ((words >> e) & 1) read |= 1ull << plane[e];
        }
        p.rec_planes = __builtin_popcountll(map->varying);
        p.rec_copy = __builtin_popcountll(read);
        p.rec_runs = 0;
        for (int k = 0; k < p.rec_planes; k++) {
            if (!((read >> k) & 1)) continue;
            if (k == 0 || !((read >> (k - 1)) & 1)) {
                p.run_first[p.rec_runs] = k;
                p.run_len[p.rec_runs++] = 0;
            }
            p.run_len[p.rec_runs - 1]++;
        }
    }
    const bool extras = a.x_prior || a.P_prior || a.K || a.y || a.S || a.SI || a.log_likelihood || a.status;
    if (ring) {
        if (!packed || !all_dense || !(dp && du) || extras || a.z_valid) return BKE_ERR_UNSUPPORTED;
        for (int k = 0; k < n_steps; k++) p.zs[k] = (const float *)zs[k];
        p.n_steps = n_steps;
        // the stage: P, the record's planes (each copied plane sits at its place in the record), x, and
        // one measurement block per step
        using St = Stage<float, 4, 2, false, 2, BKE_KF42_MAX_RING>;
        p.ring_ox = St::OQ + p.rec_planes * TILE * 4;
        p.ring_oz = p.ring_ox + St::align_up(St::XB);
        p.ring_stage = p.ring_oz + n_steps * St::align_up(St::ZB);
        // the pattern instance when every one of its structural words is, in every filter, the same bits
        // (+0, not -0; exactly 1) and so a word the scan found shared
        uint64_t zero = 0, one = 0;
        for (int e = 0; e < WORDS; e++) {
            uint32_t v;
            memcpy(&v, &map->words[e], 4);
            if ((map->varying >> e) & 1) continue;
            if (v == 0u) zero |= 1ull << e;
            if (v == 0x3f800000u) one |= 1ull << e;
        }
        if ((zero & Cv2dPattern::ZERO) == Cv2dPattern::ZERO && (one & Cv2dPattern::ONE) == Cv2dPattern::ONE)
            return launch_variant<3, 0, false, 2, BKE_KF42_MAX_RING, Cv2dPattern>(p, s);
        return launch_variant<3, 0, false, 2, BKE_KF42_MAX_RING>(p, s);
    }

#define BKE_DISPATCH(MODE)                                                                   \
    do {                                                                                     \
        if (host_models) return extras ? launch_variant<MODE, 2, true>(p, s)           \
                                       : launch_variant<MODE, 2, false>(p, s);         \
        if (all_shared) return extras ? launch_variant<MODE, 1, true>(p, s)            \
                                      : launch_variant<MODE, 1, false>(p, s);          \
        if (packed) return extras ? launch_variant<MODE, 0, true, 2>(p, s)             \
                                  : launch_variant<MODE, 0, false, 2>(p, s);           \
        if (sym) return extras ? launch_variant<MODE, 0, true, 1>(p, s)                \
                               : launch_variant<MODE, 0, false, 1>(p, s);              \
        return extras ? launch_variant<MODE, 0, true>(p, s)                            \
                      : launch_variant<MODE, 0, false>(p, s);                          \
    } while (0)
    if (dp && du) BKE_DISPATCH(3);
    if (dp) BKE_DISPATCH(1);
    BKE_DISPATCH(2);
#undef BKE_DISPATCH
}

}  // namespace bke
