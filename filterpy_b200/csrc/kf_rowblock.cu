// kf_rowblock.cu — fused predict+update for shapes whose covariance does not fit one thread's
// registers (BASELINE config 3: dim_x=9, dim_z=3, fp64; also 9/3 fp32, 6/3 fp64, 16/4 and 16/2 in both
// dtypes, 32/4 fp32): a sub-warp of G lanes owns one filter, each lane owns RPL consecutive ROWS of every
// n x n matrix.
//
//   * every row-block product C[r,:] = sum_k A[r,k] * B[k,:] keeps A's rows and C's rows in the
//     owning lane's registers and reads B from shared memory — the same address for the G lanes of
//     a filter (broadcast), 8-byte words of different filters fall into different banks;
//   * per warp, FPW = 32/G filters form a tile; ONE lane pulls the tile's x, P, F, Q, H, R, z blocks
//     (contiguous byte ranges of the dense AoS arrays) with 1-D bulk TMA copies
//     (cp.async.bulk.shared::cluster.global, SASS UBLKCP) into its own stage with an mbarrier; every
//     warp runs on its own (no block barriers anywhere);
//   * intermediates reuse the stage: P' overwrites P, (I-KH) overwrites F, K / PH' overwrite Q;
//   * the posterior rows overwrite the stage's x / P slots and leave with bulk TMA stores
//     (cp.async.bulk.global.shared::cta); the cross-proxy fence that publishes them also orders
//     every earlier shared-memory read before the stage is handed back to the TMA engine.
//
// Arithmetic per filter: filterpy/kalman/kalman_filter.py:471-478 (predict) and :533-556 (update,
// Joseph form), reference @ 3b51149.  Algorithmic bytes per filter-step (9/3 fp64): 3048.
#include <type_traits>
#include "bke_internal.cuh"
#include "kf_regtile.cuh"
#include "ptx.cuh"

namespace bke {
namespace {

template <typename T>
struct RbP {
    int64_t N;                 // filters handled by this launch (a multiple of FPW)
    T alpha_sq;
    const T *x, *P, *F, *Q, *H, *R, *z;
    T *x_out, *P_out;
    const uint8_t *valid;
    int32_t *status;
    int sticky;                       // BKE_STATUS_STICKY: write status only on failure
    T *x_prior, *P_prior, *K, *y, *S, *SI, *ll;     // optional outputs (NULL = not wanted)
};


// filters per warp tile: as many as fit 32 lanes, lowered until every array's tile is a multiple of
// 16 bytes (what a bulk copy moves): 9/3 fp32 gets 8 filters (24 lanes busy) instead of 10
template <typename T, int N, int M>
constexpr int pick_fpw(int g)
{
    for (int f = 32 / g; f >= 1; f--) {
        const int sz = f * (int)sizeof(T);
        if ((sz * N) % 16 == 0 && (sz * N * N) % 16 == 0 && (sz * M * N) % 16 == 0 && (sz * M * M) % 16 == 0 && (sz * M) % 16 == 0)
            return f;
    }
    return 0;
}

// One stage per warp and 8 warps per CTA, one CTA per SM: on 9/3 fp64 two warps per scheduler (the FP64
// pipe of one warp's dependent DFMA chains is covered by the other) beat a 2-stage ring with 4 warps.
// (9 warps fit the shared memory but cap the kernel at 168 registers.)
constexpr int RB_STAGES = 1, RB_WARPS = 8;

template <typename T, int N, int M, int RPL>
struct RbGeom {
    static constexpr int G = N / RPL;                 // lanes per filter
    static constexpr int FPW = pick_fpw<T, N, M>(G);  // filters per warp tile
    static constexpr int XB = FPW * N * sizeof(T);
    static constexpr int PB = FPW * N * N * sizeof(T);
    static constexpr int HB = FPW * M * N * sizeof(T);
    static constexpr int RBY = FPW * M * M * sizeof(T);
    static constexpr int ZB = FPW * M * sizeof(T);
    static constexpr int a16(int v) { return (v + 15) & ~15; }
    static constexpr int OX = 0;
    static constexpr int OP = OX + a16(XB);
    static constexpr int OF = OP + a16(PB);
    static constexpr int OQ = OF + a16(PB);
    static constexpr int OH = OQ + a16(PB);
    static constexpr int OR_ = OH + a16(HB);
    static constexpr int OZ = OR_ + a16(RBY);
    static constexpr int STAGE = a16(OZ + a16(ZB));
    // the posterior is staged in the stage's own x / P slots
    static constexpr int WARP_BYTES = RB_STAGES * STAGE;
    // one copy of F, Q, H, R per warp for banks that share their models (kept for the whole launch)
    static constexpr int SH_ELEMS = 2 * N * N + M * N + M * M;
    static constexpr int SH_BYTES = a16(SH_ELEMS * (int)sizeof(T));
    // optional outputs (EXTRAS instances): K, y, S, SI, log-likelihood of the warp's FPW filters, staged
    // contiguously so that they leave with bulk stores like the posterior
    static constexpr int LLB = FPW * (int)sizeof(T);
    static constexpr bool LL_BULK = LLB % 16 == 0;
    static constexpr int EK = 0;
    static constexpr int EY = EK + a16(HB);          // K[N][M] has H's size
    static constexpr int ES = EY + a16(ZB);
    static constexpr int ESI = ES + a16(RBY);
    static constexpr int ELL = ESI + a16(RBY);
    static constexpr int EX_BYTES = a16(ELL + a16(LLB));
    static constexpr uint32_t TX = XB + 3 * PB + HB + RBY + ZB;
    static_assert(N % RPL == 0 && G >= 1 && G <= 32 && FPW >= 1, "bad row-block shape");
    static_assert(XB % 16 == 0 && PB % 16 == 0 && HB % 16 == 0 && RBY % 16 == 0 && ZB % 16 == 0, "bulk copies need 16-byte multiples");
    static_assert(2 * N * M <= N * N, "K and PH' are parked in the Q slot");
};

// EXTRAS: compile the optional outputs in (kept out of the plain instantiation: their branches and
// live ranges cost the C3 kernel 9 % when they were run-time tests)
// MODE: 3 = fused predict+update, 1 = predict only, 2 = update only (what is not needed is neither
// loaded nor computed)
// SHARED: F, H, Q, R are one matrix each for the whole bank (stride 0): every warp keeps a copy in
// shared memory for the launch and the tiles carry only x, P, z
template <typename T, int N, int M, int RPL, bool EXTRAS, int MODE, bool SHARED>
__global__ void __launch_bounds__(RB_WARPS * 32, 1) kf_rowblock_kernel(RbP<T> p)
{
    using Gm = RbGeom<T, N, M, RPL>;
    constexpr int G = Gm::G, FPW = Gm::FPW;
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) uint64_t bars[RB_WARPS];

    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    constexpr int WB = Gm::WARP_BYTES + (EXTRAS ? Gm::EX_BYTES : 0);
    unsigned char *wbase = smem + (size_t)wib * WB;
    unsigned char *exb = wbase + Gm::WARP_BYTES;             // EXTRAS: staging of K, y, S, SI, log-likelihood
    uint64_t *bar = &bars[wib];
    const bool active = lane < FPW * G;
    const int fl = active ? lane / G : FPW - 1;            // filter within the tile (idle lanes mirror the last one)
    const int rb = active ? lane % G : 0;
    const int r0 = rb * RPL;

    const int64_t tiles = p.N / FPW;
    const int64_t wglobal = (int64_t)blockIdx.x * RB_WARPS + wib;
    const int64_t wstride = (int64_t)gridDim.x * RB_WARPS;

    auto issue = [&](int64_t tile, int stage) {
        unsigned char *sb = wbase + stage * Gm::STAGE;
        const int64_t f0 = tile * FPW;
        constexpr uint32_t tx = Gm::XB + Gm::PB + ((MODE & 1) && !SHARED ? 2 * Gm::PB : 0) +
                                ((MODE & 2) ? (SHARED ? 0 : Gm::HB + Gm::RBY) + Gm::ZB : 0);
        mbar_expect_tx(&bar[stage], tx);
        bulk_load(sb + Gm::OX, p.x + f0 * N, Gm::XB, &bar[stage]);
        bulk_load(sb + Gm::OP, p.P + f0 * N * N, Gm::PB, &bar[stage]);
        if constexpr ((MODE & 1) && !SHARED) {
            bulk_load(sb + Gm::OF, p.F + f0 * N * N, Gm::PB, &bar[stage]);
            bulk_load(sb + Gm::OQ, p.Q + f0 * N * N, Gm::PB, &bar[stage]);
        }
        if constexpr ((MODE & 2) && !SHARED) {
            bulk_load(sb + Gm::OH, p.H + f0 * M * N, Gm::HB, &bar[stage]);
            bulk_load(sb + Gm::OR_, p.R + f0 * M * M, Gm::RBY, &bar[stage]);
        }
        if constexpr (MODE & 2) bulk_load(sb + Gm::OZ, p.z + f0 * M, Gm::ZB, &bar[stage]);
    };

    // the shared models of this warp: after all warps' stages (generic-proxy loads and stores only)
    T *shF = reinterpret_cast<T *>(smem + (size_t)RB_WARPS * WB + (size_t)wib * Gm::SH_BYTES);
    T *shQ = shF + N * N, *shH = shQ + N * N, *shR = shH + M * N;
    if constexpr (SHARED) {
        for (int e = lane; e < N * N; e += 32) {
            if (MODE & 1) { shF[e] = p.F[e]; shQ[e] = p.Q[e]; }
        }
        if (MODE & 2) {
            for (int e = lane; e < M * N; e += 32) shH[e] = p.H[e];
            for (int e = lane; e < M * M; e += 32) shR[e] = p.R[e];
        }
        __syncwarp();
    }
    if (lane == 0) {
        for (int s = 0; s < RB_STAGES; s++) mbar_init(&bar[s], 1);
        fence_mbar_init();
    }
    __syncwarp();
    if (lane == 0) {
        for (int s = 0; s < RB_STAGES; s++) {
            const int64_t tile = wglobal + s * wstride;
            if (tile < tiles) issue(tile, s);
        }
    }

    int it = 0;
    for (int64_t tile = wglobal; tile < tiles; tile += wstride, it++) {
        const int stage = it % RB_STAGES;
        const uint32_t parity = (it / RB_STAGES) & 1;
        unsigned char *sb = wbase + stage * Gm::STAGE;
        mbar_wait(&bar[stage], parity);

        T *sx = reinterpret_cast<T *>(sb + Gm::OX) + fl * N;
        T *sP = reinterpret_cast<T *>(sb + Gm::OP) + fl * N * N;
        T *sF = reinterpret_cast<T *>(sb + Gm::OF) + fl * N * N;
        T *sQ = reinterpret_cast<T *>(sb + Gm::OQ) + fl * N * N;
        const T *sH = SHARED ? shH : reinterpret_cast<const T *>(sb + Gm::OH) + fl * M * N;
        const T *sR = SHARED ? shR : reinterpret_cast<const T *>(sb + Gm::OR_) + fl * M * M;
        const T *rF = SHARED ? shF : sF;            // the MODELS F, Q (sF / sQ are also scratch for I - K H, K, P H')
        const T *rQ = SHARED ? shQ : sQ;
        const T *sz = reinterpret_cast<const T *>(sb + Gm::OZ) + fl * M;
        unsigned char *out_x = sb + Gm::OX;
        unsigned char *out_P = sb + Gm::OP;
        T *ox = reinterpret_cast<T *>(out_x) + fl * N;
        T *oP = reinterpret_cast<T *>(out_P) + fl * N * N;
        const int64_t f = tile * FPW + fl;

        // ---------------- predict: x' = F x ; P' = alpha^2 (F P) F' + Q -----------------------
        T A[RPL][N];                 // this lane's rows of the left operand
        T C[RPL][N];                 // this lane's rows of the result
        T xr[RPL];
        if constexpr (!(MODE & 1)) {                  // update only: this lane's rows of P and x as they were loaded
#pragma unroll
            for (int i = 0; i < RPL; i++) {
                xr[i] = sx[r0 + i];
#pragma unroll
                for (int k = 0; k < N; k++) A[i][k] = sP[(r0 + i) * N + k];
            }
        } else {
#pragma unroll
        for (int i = 0; i < RPL; i++)
#pragma unroll
            for (int k = 0; k < N; k++) A[i][k] = rF[(r0 + i) * N + k];
#pragma unroll
        for (int i = 0; i < RPL; i++) {
            T s = T(0);
#pragma unroll
            for (int k = 0; k < N; k++) s += A[i][k] * sx[k];
            xr[i] = s;
        }
        // C = F P (own rows)
#pragma unroll
        for (int i = 0; i < RPL; i++)
#pragma unroll
            for (int j = 0; j < N; j++) C[i][j] = T(0);
#pragma unroll
        for (int k = 0; k < N; k++) {
            T b[N];
#pragma unroll
            for (int j = 0; j < N; j++) b[j] = sP[k * N + j];
#pragma unroll
            for (int i = 0; i < RPL; i++)
#pragma unroll
                for (int j = 0; j < N; j++) C[i][j] += A[i][k] * b[j];
        }
        // A = alpha^2 * C F' + Q (own rows of P')
#pragma unroll
        for (int j = 0; j < N; j++) {
            T b[N];
#pragma unroll
            for (int k = 0; k < N; k++) b[k] = rF[j * N + k];
#pragma unroll
            for (int i = 0; i < RPL; i++) {
                T s = T(0);
#pragma unroll
                for (int k = 0; k < N; k++) s += C[i][k] * b[k];
                A[i][j] = p.alpha_sq * s + rQ[(r0 + i) * N + j];
            }
        }
        __syncwarp();                               // every lane is done reading x, P (and F rows it needed as B)
        if (active) {
#pragma unroll
            for (int i = 0; i < RPL; i++) {
                sx[r0 + i] = xr[i];
#pragma unroll
                for (int j = 0; j < N; j++) sP[(r0 + i) * N + j] = A[i][j];          // P' overwrites P
            }
        }
        if (EXTRAS && (p.x_prior || p.P_prior)) {
            // optional outputs: the prior sits in the stage exactly as x_prior / P_prior want it (FPW filters,
            // dense) — two bulk stores; they have the whole update to read the stage before the posterior
            // overwrites it
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) {
                const int64_t f0 = tile * FPW;
                if (p.x_prior) bulk_store(p.x_prior + f0 * N, sb + Gm::OX, Gm::XB);
                if (p.P_prior) bulk_store(p.P_prior + f0 * N * N, sb + Gm::OP, Gm::PB);
                bulk_commit();
            }
        }
        __syncwarp();
        }   // MODE & 1

        // ---------------- update ------------------------------------------------------------
        const bool has_z = (MODE & 2) && ((p.valid == nullptr) || (p.valid[f] != 0));
        const unsigned um = __ballot_sync(FULL, has_z);
        int st = BKE_STATUS_OK;
        T xo[RPL];
#pragma unroll
        for (int i = 0; i < RPL; i++) xo[i] = xr[i];
        // A holds this lane's rows of P'; they become the output unless the update succeeds
        if (has_z) {
            // H in registers while it is at most 64 of them; larger (16/4 fp64) it is read from shared memory
            // where it is used (the lanes of a filter read the same address: a broadcast)
            constexpr bool H_IN_REGS = M * N * (int)sizeof(T) <= 256;
            T Hreg[H_IN_REGS ? M : 1][H_IN_REGS ? N : 1];
            if constexpr (H_IN_REGS) {
#pragma unroll
                for (int a = 0; a < M; a++)
#pragma unroll
                    for (int k = 0; k < N; k++) Hreg[a][k] = sH[a * N + k];
            }
            auto Hm = [&](int a, int k) -> T { if constexpr (H_IN_REGS) return Hreg[a][k]; else return sH[a * N + k]; };
            T y[M];
#pragma unroll
            for (int a = 0; a < M; a++) {
                T s = T(0);
#pragma unroll
                for (int k = 0; k < N; k++) s += Hm(a, k) * sx[k];
                y[a] = sz[a] - s;
            }
            // own rows of P H'  -> parked in the Q slot (offset 0)
            T PHT[RPL][M];
#pragma unroll
            for (int i = 0; i < RPL; i++)
#pragma unroll
                for (int a = 0; a < M; a++) {
                    T s = T(0);
#pragma unroll
                    for (int k = 0; k < N; k++) s += A[i][k] * Hm(a, k);
                    PHT[i][a] = s;
                }
            T *sPHT = sQ;                     // [N][M]
            T *sK = sQ + N * M;               // [N][M]   (needs 2*N*M <= N*N)
            __syncwarp(um);                   // Q rows were consumed above
            if (active) {
#pragma unroll
                for (int i = 0; i < RPL; i++)
#pragma unroll
                    for (int a = 0; a < M; a++) sPHT[(r0 + i) * M + a] = PHT[i][a];
            }
            __syncwarp(um);
            KfUpdateOut<T, N, M> o;
#pragma unroll
            for (int a = 0; a < M; a++)
#pragma unroll
                for (int b = 0; b < M; b++) {
                    T s = sR[a * M + b];
#pragma unroll
                    for (int k = 0; k < N; k++) s += Hm(a, k) * sPHT[k * M + b];
                    o.S[a][b] = s;
                }
            o.ok = reg_inverse<T, M>(o.S, o.SI, o.logdet);
            if (!o.ok) {
                st = BKE_STATUS_SINGULAR_S;
            }
            // K rows, x, (I - K H) rows
            T Kr[RPL][M];
#pragma unroll
            for (int i = 0; i < RPL; i++)
#pragma unroll
                for (int a = 0; a < M; a++) {
                    T s = T(0);
#pragma unroll
                    for (int b = 0; b < M; b++) s += PHT[i][b] * o.SI[b][a];
                    Kr[i][a] = s;
                }
#pragma unroll
            for (int i = 0; i < RPL; i++) {
                T s = xr[i];
#pragma unroll
                for (int a = 0; a < M; a++) s += Kr[i][a] * y[a];
                if (o.ok) xo[i] = s;
            }
#pragma unroll
            for (int i = 0; i < RPL; i++)
#pragma unroll
                for (int j = 0; j < N; j++) {
                    T s = ((r0 + i) == j) ? T(1) : T(0);
#pragma unroll
                    for (int a = 0; a < M; a++) s -= Kr[i][a] * Hm(a, j);
                    C[i][j] = s;                                   // own rows of I - K H
                }
            if (EXTRAS && active && (p.K || p.y || p.S || p.SI || p.ll)) {
                // optional outputs (kalman_filter.py:533-544 attributes) -> the warp's staging area; S always,
                // the rest when S was invertible (else what the arrays held stays: it is staged from there)
                T *eK = reinterpret_cast<T *>(exb + Gm::EK) + fl * N * M, *eY = reinterpret_cast<T *>(exb + Gm::EY) + fl * M;
                T *eS = reinterpret_cast<T *>(exb + Gm::ES) + fl * M * M, *eSI = reinterpret_cast<T *>(exb + Gm::ESI) + fl * M * M;
                T *eLL = reinterpret_cast<T *>(exb + Gm::ELL) + fl;
                if (rb == 0) {
#pragma unroll
                    for (int a = 0; a < M; a++)
#pragma unroll
                        for (int b = 0; b < M; b++) eS[a * M + b] = o.S[a][b];
                }
                if (o.ok) {
#pragma unroll
                    for (int i = 0; i < RPL; i++)
#pragma unroll
                        for (int a = 0; a < M; a++) eK[(r0 + i) * M + a] = Kr[i][a];
                    if (rb == 0) {
#pragma unroll
                        for (int a = 0; a < M; a++) eY[a] = y[a];
#pragma unroll
                        for (int a = 0; a < M; a++)
#pragma unroll
                            for (int b = 0; b < M; b++) eSI[a * M + b] = o.SI[a][b];
                        T q = T(0);
#pragma unroll
                        for (int a = 0; a < M; a++) {
                            T sq = T(0);
#pragma unroll
                            for (int b = 0; b < M; b++) sq += o.SI[a][b] * y[b];
                            q += y[a] * sq;
                        }
                        const T llv = T(-0.5) * (q + o.logdet + T(M) * T(LOG_2PI));
                        if (Gm::LL_BULK) *eLL = llv; else if (p.ll) p.ll[f] = llv;
                    }
                } else {
                    for (int i = 0; i < RPL; i++)
                        for (int a = 0; a < M; a++) eK[(r0 + i) * M + a] = p.K ? p.K[f * N * M + (r0 + i) * M + a] : T(0);
                    if (rb == 0) {
                        for (int a = 0; a < M; a++) eY[a] = p.y ? p.y[f * M + a] : T(0);
                        for (int e = 0; e < M * M; e++) eSI[e] = p.SI ? p.SI[f * M * M + e] : T(0);
                        if (Gm::LL_BULK) *eLL = p.ll ? p.ll[f] : T(0);
                    }
                }
            }
            if (active) {
#pragma unroll
                for (int i = 0; i < RPL; i++) {
#pragma unroll
                    for (int j = 0; j < N; j++) sF[(r0 + i) * N + j] = C[i][j];     // (I-KH) overwrites F
#pragma unroll
                    for (int a = 0; a < M; a++) sK[(r0 + i) * M + a] = Kr[i][a];
                }
            }
            __syncwarp(um);
            // T1 = (I-KH) P'  (own rows, into A2), then P = T1 (I-KH)' + (K R) K'
            T T1[RPL][N];
#pragma unroll
            for (int i = 0; i < RPL; i++)
#pragma unroll
                for (int j = 0; j < N; j++) T1[i][j] = T(0);
#pragma unroll
            for (int k = 0; k < N; k++) {
                T b[N];
#pragma unroll
                for (int j = 0; j < N; j++) b[j] = sP[k * N + j];
#pragma unroll
                for (int i = 0; i < RPL; i++)
#pragma unroll
                    for (int j = 0; j < N; j++) T1[i][j] += C[i][k] * b[j];
            }
            T KR[RPL][M];
#pragma unroll
            for (int i = 0; i < RPL; i++)
#pragma unroll
                for (int b = 0; b < M; b++) {
                    T s = T(0);
#pragma unroll
                    for (int a = 0; a < M; a++) s += Kr[i][a] * sR[a * M + b];
                    KR[i][b] = s;
                }
#pragma unroll
            for (int j = 0; j < N; j++) {
                T b[N], kb[M];
#pragma unroll
                for (int k = 0; k < N; k++) b[k] = sF[j * N + k];
#pragma unroll
                for (int a = 0; a < M; a++) kb[a] = sK[j * M + a];
#pragma unroll
                for (int i = 0; i < RPL; i++) {
                    T s = T(0);
#pragma unroll
                    for (int k = 0; k < N; k++) s += T1[i][k] * b[k];
#pragma unroll
                    for (int a = 0; a < M; a++) s += KR[i][a] * kb[a];
                    if (o.ok) A[i][j] = s;
                }
            }
        }
        if (EXTRAS && (MODE & 2) && !has_z && active && (p.K || p.y || p.S || p.SI || p.ll)) {
            // z is None: y = 0, K / S / SI / log-likelihood keep their values (kalman_filter.py:515-520) — staged
            // from the arrays so that the tile's bulk stores write them back unchanged
            T *eK = reinterpret_cast<T *>(exb + Gm::EK) + fl * N * M, *eY = reinterpret_cast<T *>(exb + Gm::EY) + fl * M;
            T *eS = reinterpret_cast<T *>(exb + Gm::ES) + fl * M * M, *eSI = reinterpret_cast<T *>(exb + Gm::ESI) + fl * M * M;
            for (int i = 0; i < RPL; i++)
                for (int a = 0; a < M; a++) eK[(r0 + i) * M + a] = p.K ? p.K[f * N * M + (r0 + i) * M + a] : T(0);
            if (rb == 0) {
                for (int a = 0; a < M; a++) eY[a] = T(0);
                for (int e = 0; e < M * M; e++) { eS[e] = p.S ? p.S[f * M * M + e] : T(0); eSI[e] = p.SI ? p.SI[f * M * M + e] : T(0); }
                if (Gm::LL_BULK) reinterpret_cast<T *>(exb + Gm::ELL)[fl] = p.ll ? p.ll[f] : T(0);
            }
        }
        // ---------------- posterior rows -> staging -> bulk TMA store ---------------------------
        // the prior's stores (optional outputs) have read the stage slots the posterior is about to overwrite
        if (lane == 0 && EXTRAS) bulk_wait_read<0>();
        __syncwarp();                                       // every lane is done with P', (I-KH), K in the stage
        if (active) {
#pragma unroll
            for (int i = 0; i < RPL; i++) {
                ox[r0 + i] = xo[i];
#pragma unroll
                for (int j = 0; j < N; j++) oP[(r0 + i) * N + j] = A[i][j];
            }
            if (p.status && rb == 0 && (st != BKE_STATUS_OK || !p.sticky)) p.status[f] = st;
        }
        fence_proxy_async();      // publishes the staging buffer to the async proxy AND completes every earlier LDS of the stage
        __syncwarp();
        if (lane == 0) {
            const int64_t f0 = tile * FPW;
            bulk_store(p.x_out + f0 * N, out_x, Gm::XB);
            bulk_store(p.P_out + f0 * N * N, out_P, Gm::PB);
            if (EXTRAS && (MODE & 2)) {
                if (p.K) bulk_store(p.K + f0 * N * M, exb + Gm::EK, Gm::HB);
                if (p.y) bulk_store(p.y + f0 * M, exb + Gm::EY, Gm::ZB);
                if (p.S) bulk_store(p.S + f0 * M * M, exb + Gm::ES, Gm::RBY);
                if (p.SI) bulk_store(p.SI + f0 * M * M, exb + Gm::ESI, Gm::RBY);
                if (Gm::LL_BULK && p.ll) bulk_store(p.ll + f0, exb + Gm::ELL, Gm::LLB);
            }
            bulk_commit();
            // the stores have read the stage (and the staging area of the optional outputs): it may be refilled
            bulk_wait_read<0>();
            const int64_t nt = tile + RB_STAGES * wstride;
            if (nt < tiles) issue(nt, stage);
        }
        __syncwarp();
    }
    if (lane == 0) bulk_wait_all();
}

template <typename T, int N, int M, int RPL>
int launch_rb(const bke_kf_args &a, cudaStream_t s)
{
    const int mode = (int)(a.flags & (BKE_DO_PREDICT | BKE_DO_UPDATE));
    using Gm = RbGeom<T, N, M, RPL>;
    const int64_t Nmain = (a.n_filters / Gm::FPW) * Gm::FPW;
    const int64_t rem = a.n_filters - Nmain;
    if (Nmain > 0) {
        RbP<T> p;
        p.N = Nmain; p.alpha_sq = (T)a.alpha_sq;
        p.x = (const T *)a.x; p.P = (const T *)a.P; p.F = (const T *)a.F; p.Q = (const T *)a.Q;
        p.H = (const T *)a.H; p.R = (const T *)a.R; p.z = (const T *)a.z;
        p.x_out = (T *)a.x_out; p.P_out = (T *)a.P_out; p.valid = a.z_valid; p.status = a.status; p.sticky = (a.flags & BKE_STATUS_STICKY) ? 1 : 0;
        p.x_prior = (T *)a.x_prior; p.P_prior = (T *)a.P_prior; p.K = (T *)a.K; p.y = (T *)a.y;
        p.S = (T *)a.S; p.SI = (T *)a.SI; p.ll = (T *)a.log_likelihood;
        const bool extras = a.x_prior || a.P_prior || a.K || a.y || a.S || a.SI || a.log_likelihood;
        // every model the call reads is shared by the bank (stride 0)?  (a mix goes to the catch-all kernel)
        const bool dp = a.flags & BKE_DO_PREDICT, du = a.flags & BKE_DO_UPDATE;
        const bool shared = (!dp || (a.F_stride == 0 && a.Q_stride == 0)) && (!du || (a.H_stride == 0 && a.R_stride == 0));
        auto kern = extras ? kf_rowblock_kernel<T, N, M, RPL, true, 3, false>
                           : kf_rowblock_kernel<T, N, M, RPL, false, 3, false>;
        if (mode == 1) kern = kf_rowblock_kernel<T, N, M, RPL, true, 1, false>;     // the single-mode and the
        if (mode == 2) kern = kf_rowblock_kernel<T, N, M, RPL, true, 2, false>;     // shared-model kernels always
        if (shared) {                                                                                     // carry the optional outputs
            // fp32 dim_x = 16 / 32: the tensor-core tile (kf_tc.cu) takes every shared-model predict, alone or fused
            if constexpr (sizeof(T) == 4 && (N == 16 || N == 32)) {
                if (mode != 2) return BKE_ERR_UNSUPPORTED;
                kern = kf_rowblock_kernel<T, N, M, RPL, true, 2, true>;
            } else {
                kern = kf_rowblock_kernel<T, N, M, RPL, true, 3, true>;
                if (mode == 1) kern = kf_rowblock_kernel<T, N, M, RPL, true, 1, true>;
                if (mode == 2) kern = kf_rowblock_kernel<T, N, M, RPL, true, 2, true>;
            }
        }
        const bool kern_extras = extras || mode != 3 || shared;      // the instance selected above carries them
        const int smem = RB_WARPS * (Gm::WARP_BYTES + (kern_extras ? Gm::EX_BYTES : 0) + (shared ? Gm::SH_BYTES : 0));
        const int cfg = (mode == 3 ? (int)extras : 1 + mode) + (shared ? 4 : 0);
        static bool configured[8][64] = {{false}};
        int dev = 0;
        cudaGetDevice(&dev);
        if (dev < 0 || dev >= 64 || !configured[cfg][dev]) {
            if (check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem), "cudaFuncSetAttribute")) return BKE_ERR_CUDA;
            if (dev >= 0 && dev < 64) configured[cfg][dev] = true;
        }
        const int64_t tiles = Nmain / Gm::FPW;
        int64_t grid = (tiles + RB_WARPS - 1) / RB_WARPS;
        if (grid > sm_count()) grid = sm_count();
        kern<<<(unsigned)grid, RB_WARPS * 32, smem, s>>>(p);
        if (check_cuda(cudaGetLastError(), "kf_rowblock_kernel launch")) return BKE_ERR_CUDA;
    }
    if (rem > 0) {       // ragged tail (< one warp tile): the catch-all kernel on the last few filters
        bke_kf_args t = a;
        const size_t es = sizeof(T);
        auto off = [&](const void *ptr, int64_t per) { return ptr ? (const void *)((const char *)ptr + (size_t)Nmain * per * es) : nullptr; };
        t.n_filters = rem;
        t.x = off(a.x, N); t.P = off(a.P, N * N); t.x_out = (void *)off(a.x_out, N); t.P_out = (void *)off(a.P_out, N * N);
        t.F = a.F_stride ? off(a.F, N * N) : a.F; t.Q = a.Q_stride ? off(a.Q, N * N) : a.Q;      // shared models are not offset
        t.H = a.H_stride ? off(a.H, M * N) : a.H; t.R = a.R_stride ? off(a.R, M * M) : a.R;
        t.z = off(a.z, M);
        t.x_prior = (void *)off(a.x_prior, N); t.P_prior = (void *)off(a.P_prior, N * N); t.K = (void *)off(a.K, N * M);
        t.y = (void *)off(a.y, M); t.S = (void *)off(a.S, M * M); t.SI = (void *)off(a.SI, M * M);
        t.log_likelihood = (void *)off(a.log_likelihood, 1);
        t.z_valid = a.z_valid ? a.z_valid + Nmain : nullptr;
        t.status = a.status ? a.status + Nmain : nullptr;
        return launch_kf_generic(t, s);
    }
    return BKE_OK;
}

bool al16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace

int launch_kf_rowblock(const bke_kf_args &a, cudaStream_t s)
{
    // fused predict+update, per-filter dense models, no control input
    if ((a.flags & BKE_UPDATE_FIRST) || !(a.flags & (BKE_DO_PREDICT | BKE_DO_UPDATE))) return BKE_ERR_UNSUPPORTED;
    const bool dp = a.flags & BKE_DO_PREDICT, du = a.flags & BKE_DO_UPDATE;
    if (a.B && a.u) return BKE_ERR_UNSUPPORTED;
    {   // the models the call reads are either all per-filter or all shared; a mix goes to the catch-all kernel
        int dense = 0, shared = 0;
        if (dp) { (a.F_stride ? dense : shared)++; (a.Q_stride ? dense : shared)++; }
        if (du) { (a.H_stride ? dense : shared)++; (a.R_stride ? dense : shared)++; }
        if (dense && shared) return BKE_ERR_UNSUPPORTED;
    }
    if (!(al16(a.x) && al16(a.P) && al16(a.x_out) && al16(a.P_out))) return BKE_ERR_UNSUPPORTED;
    if (dp && a.F_stride && !(al16(a.F) && al16(a.Q))) return BKE_ERR_UNSUPPORTED;
    if (du && a.H_stride && !(al16(a.H) && al16(a.R))) return BKE_ERR_UNSUPPORTED;
    if (du && !al16(a.z)) return BKE_ERR_UNSUPPORTED;
    // the optional outputs leave with bulk stores too
    if (!(al16(a.x_prior) && al16(a.P_prior) && al16(a.K) && al16(a.y) && al16(a.S) && al16(a.SI) && al16(a.log_likelihood))) return BKE_ERR_UNSUPPORTED;
    const int n = a.dim_x, m = a.dim_z;
    if (a.dtype == BKE_F64) {
        if (n == 9 && m == 3) return launch_rb<double, 9, 3, 3>(a, s);
        if (n == 6 && m == 3) return launch_rb<double, 6, 3, 3>(a, s);
        // dim_x = 16: one row per lane, 16 lanes per filter, 2 filters per warp tile
        if (n == 16 && m == 4) return launch_rb<double, 16, 4, 1>(a, s);
        if (n == 16 && m == 2) return launch_rb<double, 16, 2, 1>(a, s);
    } else {
        if (n == 16 && m == 4) return launch_rb<float, 16, 4, 2>(a, s);   // two rows per lane, 4 filters per warp tile
        if (n == 16 && m == 2) return launch_rb<float, 16, 2, 2>(a, s);
        // dim_x = 32: one row per lane, the whole warp on one filter (the update half of the tensor-core predict, kf_tc.cu)
        if (n == 32 && m == 4) return launch_rb<float, 32, 4, 1>(a, s);
        if (n == 9 && m == 3) return launch_rb<float, 9, 3, 3>(a, s);        // 8 filters per warp tile (see pick_fpw)
    }
    return BKE_ERR_UNSUPPORTED;
}

}  // namespace bke
