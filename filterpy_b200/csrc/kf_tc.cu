// kf_tc.cu — the tensor-core tile of the linear Kalman filter: covariance propagation
//     x <- F x,   P <- alpha^2 F P F' + Q          (filterpy/kalman/kalman_filter.py:471-478)
// for banks with dim_x = 16 or 32, fp32, whose F and Q are SHARED by the bank (stride 0 — one motion
// model for every track, the usual way a bank is built), on Hopper's warpgroup MMA (wgmma.mma_async,
// accumulators in registers).
//
// Why only here.  A tile is 128 rows deep (two m64 wgmma's).  With per-filter models every 16 x 16 product
// has its own left AND right operand, so a 128-row tile could only be filled block-diagonally (8x wasted
// multiplies, and the operands would have to be re-laid-out per filter).  With a shared F the stacked
// rows of 128 / n covariances ARE one 128 x n operand in the layout they have in HBM:
//     D1[(i,r)][c] = sum_k P_i[r][k] F[c][k]        = (P_i F')[r][c]          A = the P rows, B = F (K-major)
//     D2[(i,c)][j] = sum_k (P_i F')[k][c] F[j][k]   = (F P_i F')[c][j]        A = D1's n x n blocks transposed
// (P symmetric: (P F')' = F P), i.e. both products of the sandwich have the bank on the M side and the
// one shared matrix on the N side.  Below dim_x = 16 nothing fills an MMA fragment (north_star), at
// dim_x >= 16 the CUDA cores fall behind HBM (fp32: 2 x 2 n^3 = 16 k flop per 2 KB of covariance at
// n = 16, 131 k per 8 KB at n = 32) and this kernel takes the predict of the shared-model banks.
//
// Precision.  tf32 reads 10 mantissa bits, north_star asks for 1e-3 relative on P: one TF32 pass per
// product would sit right at that bound, so every product is the usual three-term split
//     a b ~ a_hi b_hi + a_hi b_lo + a_lo b_hi,   a_hi = a rounded to TF32, a_lo = a - a_hi rounded to TF32
// accumulated in fp32 (relative error ~ 2^-20 per term).  The split is made by the CUDA cores while the
// tile is written into the operand layout, so it costs no extra pass.
//
// One CTA = one warpgroup (4 warps) = one 128-row tile at a time (8 filters at n = 16, 4 at n = 32),
// persistent over the tiles; several CTAs per SM overlap each other's loads, MMAs and stores.  Both
// operands come from shared memory in the no-swizzle K-major canonical layout (8-row x 16-byte core
// matrices; descriptors with LBO = distance between the two 16-byte K chunks of an instruction, SBO =
// distance between 8-row groups), so no tensor map is needed and the hi / lo split happens on the way in.
// The accumulator fragment of the first product is written straight back as the (transposed, split)
// A operand of the second; the second goes through a padded scratch so that thread t holds row t.
#include "bke_internal.cuh"
#include "kf_regtile.cuh"
#include "ptx.cuh"

namespace bke {
namespace tc {

template <int NX>
struct Geom {
    static constexpr int FPT = 128 / NX;            // filters per tile
    static constexpr int KC = NX / 4;               // 16-byte chunks along K
    static constexpr int KS = NX / 8;               // wgmma steps along K (8 tf32 = 32 bytes each)
    static constexpr int A_LBO = 128 * 16;          // bytes between consecutive K chunks of the 128-row operand
    static constexpr int A_BYTES = 128 * NX * 4;
    static constexpr int B_LBO = NX * 16;           // the same for the NX-row operand (F)
    static constexpr int B_BYTES = NX * NX * 4;
    static constexpr int SBO = 128;                 // bytes between 8-row groups (core matrices are contiguous)
    static constexpr int ACC = NX / 2;              // fp32 accumulator registers per thread of one m64nNXk8 product
    // shared memory: A_hi | A_lo | F_hi | F_lo | F (plain, rows padded to NX + 1 words: x' = F x reads row r in
    // thread r) | Q (rows padded to NX + 4 words: conflict-free 16-byte reads) | x of the tile's filters.  The
    // scratch [128][NX + 1] of the second product lies over A_hi | A_lo (free once that product has completed).
    static constexpr int FP = NX + 1, QP = NX + 4;
    static constexpr int O_AHI = 0, O_ALO = O_AHI + A_BYTES, O_FHI = O_ALO + A_BYTES, O_FLO = O_FHI + B_BYTES;
    static constexpr int O_F = O_FLO + B_BYTES, O_Q = O_F + ((NX * FP * 4 + 15) & ~15), O_T = O_AHI;
    static constexpr int O_X = O_Q + NX * QP * 4;
    // fused update (shared H, R; dim_z <= 4): H and R plain, for the CUDA-core part
    static constexpr int O_H = O_X + 128 * 4, O_R = O_H + 4 * NX * 4;
    static constexpr int SMEM = O_R + 64;
    static_assert(128 * FP * 4 <= 2 * A_BYTES, "the scratch fits the two operand buffers");
};

// byte offset of element (row, k) of a K-major operand with `lbo` bytes between K chunks
__device__ __forceinline__ int op_off(int row, int k, int lbo) { return (k >> 2) * lbo + (row >> 3) * 128 + (row & 7) * 16 + (k & 3) * 4; }

// wgmma shared-memory matrix descriptor: start address >> 4 in bits [0,14), leading byte offset >> 4 in [16,30),
// stride byte offset >> 4 in [32,46), base offset 0, layout type 0 (no swizzle) in [62,64)
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo)
{
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32);
}

// D (64 x NX, fp32, registers) = A (64 x 8, tf32, smem) B' (NX x 8, tf32, smem) + (accumulate ? D : 0); both operands K-major
template <int NX> __device__ __forceinline__ void wgmma_tf32(float (&d)[NX / 2], uint64_t adesc, uint64_t bdesc, int accumulate);
template <> __device__ __forceinline__ void wgmma_tf32<16>(float (&d)[8], uint64_t adesc, uint64_t bdesc, int accumulate)
{
    asm volatile("{\n"
                 ".reg .pred p;\n"
                 "setp.ne.b32 p, %10, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n"
                 "}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <> __device__ __forceinline__ void wgmma_tf32<32>(float (&d)[16], uint64_t adesc, uint64_t bdesc, int accumulate)
{
    asm volatile("{\n"
                 ".reg .pred p;\n"
                 "setp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, "
                 "%12, %13, %14, %15}, %16, %17, p, 1, 1;\n"
                 "}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// accumulator fragment of m64nNk8 (fp32): register 4 q + 2 h + e of thread (warp w, lane l) holds
// row 16 w + l / 4 + 8 h, column 8 q + 2 (l % 4) + e of the 64-row half
__device__ __forceinline__ int frag_row(int warp, int lane, int reg) { return warp * 16 + (lane >> 2) + ((reg >> 1) & 1) * 8; }
__device__ __forceinline__ int frag_col(int lane, int reg) { return (reg >> 2) * 8 + (lane & 3) * 2 + (reg & 1); }

// round to TF32 (10 mantissa bits, round to nearest, ties away): the tensor core reads exactly these bits, the low 13 are 0
__device__ __forceinline__ float tf32_hi(float v)
{
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
    return __uint_as_float(u);
}
// the remainder v - hi is exact in fp32 (|.| <= 2^-11 |v|); rounded to TF32 itself it leaves 2^-22 |v|
__device__ __forceinline__ float tf32_lo(float v, float hi) { return tf32_hi(v - hi); }

struct TcP {
    int64_t N;                       // filters
    float alpha_sq;
    const float *x, *P, *F, *Q;      // F, Q shared by the bank
    float *x_out, *P_out, *x_prior, *P_prior;
    int32_t *status;
    int sticky;
    // fused update (kf_cov_tc_kernel<NX, M> with M > 0): H [M, NX] and R [M, M] shared by the bank
    const float *H, *R, *z;
    const uint8_t *valid;
    float *K, *y, *S, *SI, *ll;
};

// M = 0: predict only.  M = dim_z in 1 .. 4: the update of kalman_filter.py:533-556 follows in the same launch (H, R shared).
// CTAs per SM the register budget is planned for: the accumulators live in registers, and the update's pieces need more
// of them (dim_z x dim_z ones above all at dim_z >= 3).  Not tuned on the H100: ptxas reports small spills (4-80 B per
// thread) in the fused instances and in the 16/0 predict at these caps.
constexpr int tc_ctas(int nx, int m) { return nx == 16 ? (m >= 3 ? 4 : (m >= 1 ? 6 : 8)) : (m >= 1 ? 3 : 4); }

template <int NX, int M>
__global__ void __launch_bounds__(128, tc_ctas(NX, M)) kf_cov_tc_kernel(TcP p)
{
    using G = Geom<NX>;
    extern __shared__ __align__(1024) unsigned char smem[];
    float *Fs = reinterpret_cast<float *>(smem + G::O_F), *Qs = reinterpret_cast<float *>(smem + G::O_Q);
    float *xs = reinterpret_cast<float *>(smem + G::O_X);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    // ---- one-time setup: the shared model in both forms
    for (int e = tid; e < NX * NX; e += 128) {
        const float f = p.F[e];
        const int n = e / NX, k = e % NX;
        const float hi = tf32_hi(f);
        *reinterpret_cast<float *>(smem + G::O_FHI + op_off(n, k, G::B_LBO)) = hi;
        *reinterpret_cast<float *>(smem + G::O_FLO + op_off(n, k, G::B_LBO)) = tf32_lo(f, hi);
        Fs[n * G::FP + k] = f;
        Qs[n * G::QP + k] = p.Q[e];
    }
    float *Hs = reinterpret_cast<float *>(smem + G::O_H), *Rs = reinterpret_cast<float *>(smem + G::O_R);
    if constexpr (M > 0) {
        for (int e = tid; e < M * NX; e += 128) Hs[e] = p.H[e];
        if (tid < M * M) Rs[tid] = p.R[tid];
    }

    const uint32_t a_hi = smem_u32(smem + G::O_AHI), a_lo = smem_u32(smem + G::O_ALO);
    const uint32_t f_hi = smem_u32(smem + G::O_FHI), f_lo = smem_u32(smem + G::O_FLO);
    // D[half] = A_lo F_hi' + A_hi F_lo' + A_hi F_hi'   (small terms first), rows 64 half .. 64 half + 63, K = NX in steps of 8
    auto product = [&](float (&d)[2][G::ACC]) {
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; h++) {
#pragma unroll
            for (int term = 0; term < 3; term++) {
                const uint32_t a = (term == 0 ? a_lo : a_hi) + h * 8 * G::SBO, b = term == 1 ? f_lo : f_hi;
#pragma unroll
                for (int ks = 0; ks < G::KS; ks++)
                    wgmma_tf32<NX>(d[h], smem_desc(a + ks * 2 * G::A_LBO, G::A_LBO, G::SBO),
                                   smem_desc(b + ks * 2 * G::B_LBO, G::B_LBO, G::SBO), term + ks > 0);
            }
        }
        wgmma_commit();
    };

    const int64_t rows = p.N * NX;
    const int64_t tiles = (rows + 127) / 128;
    const int i_in_tile = tid / NX, r = tid % NX;         // this thread's row of the tile: filter i, matrix row r
    // this thread's row of the NEXT tile is fetched while the current tile's products run
    float4 pre[G::KC];
    float xpre = 0.f;                 // x[(tile * FPT + i) * NX + r] = x[tile * 128 + tid]: the thread's own component, coalesced
    auto fetch_row = [&](int64_t tile) {
        const int64_t row = tile * 128 + tid;
        const float4 *src = reinterpret_cast<const float4 *>(p.P + row * NX);
#pragma unroll
        for (int kc = 0; kc < G::KC; kc++) pre[kc] = (row < rows) ? src[kc] : make_float4(0.f, 0.f, 0.f, 0.f);
        xpre = (row < rows) ? p.x[row] : 0.f;
    };
    if ((int64_t)blockIdx.x < tiles) fetch_row(blockIdx.x);
    for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int64_t row = tile * 128 + tid;
        const bool live = row < rows;
        const int64_t f = tile * G::FPT + i_in_tile;
        // ---- 1. this thread's row of P -> hi / lo parts in the A-operand layout; x' = F x (own component)
        float xr = 0.f;
        {
#pragma unroll
            for (int kc = 0; kc < G::KC; kc++) {
                const float4 v = pre[kc];
                const float4 h = make_float4(tf32_hi(v.x), tf32_hi(v.y), tf32_hi(v.z), tf32_hi(v.w));
                const int off = kc * G::A_LBO + (tid >> 3) * 128 + (tid & 7) * 16;
                *reinterpret_cast<float4 *>(smem + G::O_AHI + off) = h;
                *reinterpret_cast<float4 *>(smem + G::O_ALO + off) = make_float4(tf32_lo(v.x, h.x), tf32_lo(v.y, h.y), tf32_lo(v.z, h.z), tf32_lo(v.w, h.w));
            }
            xs[tid] = xpre;
            if (tile + gridDim.x < tiles) fetch_row(tile + gridDim.x);
        }
        fence_proxy_async();          // generic-proxy writes of the operands -> visible to the tensor core (async proxy)
        __syncthreads();
        // ---- 2. D1 = P F'  (rows (i,r), columns c)
        float d[2][G::ACC];
        product(d);
        {   // x' = F x from the staged state while the tensor core works (the barrier above published xs)
            const float *xf = xs + i_in_tile * NX;
#pragma unroll
            for (int k = 0; k < NX; k++) xr += Fs[r * G::FP + k] * xf[k];
        }
        wgmma_wait_all();
        __syncthreads();              // every warp's share of the first product has read the operands
        // ---- 3. transpose every filter's block on the way back: A2[(i,c)][k] = Y_i[k][c], straight from the fragment
#pragma unroll
        for (int h = 0; h < 2; h++) {
#pragma unroll
            for (int q = 0; q < G::ACC; q++) {
                const int rt = h * 64 + frag_row(warp, lane, q), c = frag_col(lane, q);     // tile row (i, k), column c
                const int off = op_off((rt / NX) * NX + c, rt % NX, G::A_LBO);
                const float hi = tf32_hi(d[h][q]);
                *reinterpret_cast<float *>(smem + G::O_AHI + off) = hi;
                *reinterpret_cast<float *>(smem + G::O_ALO + off) = tf32_lo(d[h][q], hi);
            }
        }
        fence_proxy_async();
        __syncthreads();
        // ---- 4. D2 = (F P) F'  (rows (i,c), columns j)
        product(d);
        wgmma_wait_all();
        __syncthreads();
        float pp[NX];                                   // this thread's row of the prior covariance P' = alpha^2 F P F' + Q
        {
            float *Ts = reinterpret_cast<float *>(smem + G::O_T);          // over A_hi | A_lo: the second product has read them
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
                for (int q = 0; q < G::ACC; q++) Ts[(h * 64 + frag_row(warp, lane, q)) * G::FP + frag_col(lane, q)] = d[h][q];
            __syncthreads();
#pragma unroll
            for (int kc = 0; kc < G::KC; kc++) {
                const float4 q = *reinterpret_cast<const float4 *>(Qs + r * G::QP + kc * 4);
                const float *v = Ts + tid * G::FP + kc * 4;
                pp[kc * 4 + 0] = fmaf(p.alpha_sq, v[0], q.x); pp[kc * 4 + 1] = fmaf(p.alpha_sq, v[1], q.y);
                pp[kc * 4 + 2] = fmaf(p.alpha_sq, v[2], q.z); pp[kc * 4 + 3] = fmaf(p.alpha_sq, v[3], q.w);
            }
            __syncthreads();                            // every row is in registers: the scratch may go
        }
        if (live) {
            if (p.P_prior) {
                float4 *dst2 = reinterpret_cast<float4 *>(p.P_prior + row * NX);
#pragma unroll
                for (int kc = 0; kc < G::KC; kc++) dst2[kc] = make_float4(pp[kc * 4], pp[kc * 4 + 1], pp[kc * 4 + 2], pp[kc * 4 + 3]);
            }
            if (p.x_prior) p.x_prior[row] = xr;
        }
        float xo = xr;                                  // posterior := prior unless the update succeeds
        int st = BKE_STATUS_OK;
        if constexpr (M > 0) {
            // ---- 5. update (kalman_filter.py:533-556) with H, R shared, on the CUDA cores: everything is dim_z-sized per
            // filter and the filter's NX threads sit in one warp.  Row r of P' H' is a thin product (NX x dim_z FMAs per
            // thread, H broadcast from shared memory) — in plain fp32 from the row the thread already holds, so that K, S
            // and the covariance correction are mutually consistent to fp32 rounding
            float pht[M];
#pragma unroll
            for (int a = 0; a < M; a++) {
                float sacc = 0.f;
#pragma unroll
                for (int j = 0; j < NX; j++) sacc = fmaf(pp[j], Hs[a * NX + j], sacc);
                pht[a] = sacc;
            }
            const bool vz = live && (p.valid == nullptr || p.valid[f] != 0);
            // S = H (P' H') + R and H x' : this thread's terms, summed over the filter's NX lanes (xor butterfly)
            float Sm[M][M], hx[M];
#pragma unroll
            for (int a = 0; a < M; a++) {
                const float h = Hs[a * NX + r];
                hx[a] = h * xr;
#pragma unroll
                for (int b = 0; b < M; b++) Sm[a][b] = h * pht[b];
            }
#pragma unroll
            for (int o = NX / 2; o > 0; o >>= 1) {
#pragma unroll
                for (int a = 0; a < M; a++) {
                    hx[a] += __shfl_xor_sync(FULL, hx[a], o);
#pragma unroll
                    for (int b = 0; b < M; b++) Sm[a][b] += __shfl_xor_sync(FULL, Sm[a][b], o);
                }
            }
            float yv[M];
#pragma unroll
            for (int a = 0; a < M; a++) {
                yv[a] = (vz ? p.z[f * M + a] : 0.f) - hx[a];
#pragma unroll
                for (int b = 0; b < M; b++) Sm[a][b] += Rs[a * M + b];
            }
            float SI[M][M], logdet;
            const bool inv_ok = reg_inverse<float, M>(Sm, SI, logdet);
            if (vz && !inv_ok) st = BKE_STATUS_SINGULAR_S;
            const bool upd = vz && inv_ok;
            float Kr[M];                                 // row r of K = P' H' S^-1
#pragma unroll
            for (int a = 0; a < M; a++) {
                float sk = 0.f;
#pragma unroll
                for (int b = 0; b < M; b++) sk += pht[b] * SI[b][a];
                Kr[a] = sk;
            }
            if (upd) {
#pragma unroll
                for (int a = 0; a < M; a++) xo += Kr[a] * yv[a];
            }
            // rows of K and P' H' of the filter's other lanes: through this thread's OWN first two operand chunks (only
            // its warp reads them, the second product is complete) — 16 bytes each, dim_z <= 4
            {
                float4 kq = make_float4(0.f, 0.f, 0.f, 0.f), pq = kq;
                float *kf4 = reinterpret_cast<float *>(&kq), *pf4 = reinterpret_cast<float *>(&pq);
#pragma unroll
                for (int a = 0; a < M; a++) { kf4[a] = Kr[a]; pf4[a] = pht[a]; }
                const int off = (tid >> 3) * 128 + (tid & 7) * 16;
                *reinterpret_cast<float4 *>(smem + G::O_AHI + off) = kq;
                *reinterpret_cast<float4 *>(smem + G::O_AHI + G::A_LBO + off) = pq;
            }
            __syncwarp();
            if (upd) {
                // Joseph form in the reference's order, with thin products (kalman_filter.py:555-556):
                //   T1 = (I - K H) P' = P' - K (P'H')'          row r: P'[r][j] - sum_a K[r][a] (P'H')[j][a]
                //   P  = T1 (I - K H)' + (K R) K'               row r: T1[r][j] + sum_a ((K R)[r][a] - (T1 H')[r][a]) K[j][a]
                // errors of K enter quadratically, as in the reference — not linearly as in P' - K S K'
                const int t0 = tid - r;                   // first thread of this filter
#pragma unroll
                for (int j = 0; j < NX; j++) {
                    const int tj = t0 + j;
                    const float4 pq = *reinterpret_cast<const float4 *>(smem + G::O_AHI + G::A_LBO + (tj >> 3) * 128 + (tj & 7) * 16);
                    const float *pj = reinterpret_cast<const float *>(&pq);
                    float acc = pp[j];
#pragma unroll
                    for (int a = 0; a < M; a++) acc = fmaf(-Kr[a], pj[a], acc);
                    pp[j] = acc;
                }
                float g[M];                               // (K R)[r][a] - (T1 H')[r][a]
#pragma unroll
                for (int a = 0; a < M; a++) {
                    float t1h = 0.f, kr = 0.f;
#pragma unroll
                    for (int j = 0; j < NX; j++) t1h = fmaf(pp[j], Hs[a * NX + j], t1h);
#pragma unroll
                    for (int b = 0; b < M; b++) kr = fmaf(Kr[b], Rs[b * M + a], kr);
                    g[a] = kr - t1h;
                }
#pragma unroll
                for (int j = 0; j < NX; j++) {
                    const int tj = t0 + j;
                    const float4 kq = *reinterpret_cast<const float4 *>(smem + G::O_AHI + (tj >> 3) * 128 + (tj & 7) * 16);
                    const float *kj = reinterpret_cast<const float *>(&kq);
                    float acc = pp[j];
#pragma unroll
                    for (int a = 0; a < M; a++) acc = fmaf(g[a], kj[a], acc);
                    pp[j] = acc;
                }
            }
            __syncwarp();                               // the chunks are rewritten by the next tile's operand rows
            if (live) {
                // optional outputs (kalman_filter.py:533-544 attributes): y always (0 when z is None), S when there is a
                // measurement, K / SI / log-likelihood when S was invertible; otherwise the arrays keep their values
                if (p.y && r == 0) {
#pragma unroll
                    for (int a = 0; a < M; a++) p.y[f * M + a] = vz ? yv[a] : 0.f;
                }
                if (vz && r == 0 && p.S) {
#pragma unroll
                    for (int a = 0; a < M; a++)
#pragma unroll
                        for (int b = 0; b < M; b++) p.S[f * M * M + a * M + b] = Sm[a][b];
                }
                if (upd) {
                    if (p.K) {
#pragma unroll
                        for (int a = 0; a < M; a++) p.K[(f * NX + r) * M + a] = Kr[a];
                    }
                    if (r == 0) {
                        if (p.SI) {
#pragma unroll
                            for (int a = 0; a < M; a++)
#pragma unroll
                                for (int b = 0; b < M; b++) p.SI[f * M * M + a * M + b] = SI[a][b];
                        }
                        if (p.ll) {
                            float q = 0.f;
#pragma unroll
                            for (int a = 0; a < M; a++) {
                                float sq = 0.f;
#pragma unroll
                                for (int b = 0; b < M; b++) sq += SI[a][b] * yv[b];
                                q += yv[a] * sq;
                            }
                            p.ll[f] = -0.5f * (q + logdet + float(M) * float(LOG_2PI));
                        }
                    }
                }
            }
        }
        if (live) {
            float4 *dst = reinterpret_cast<float4 *>(p.P_out + row * NX);
#pragma unroll
            for (int kc = 0; kc < G::KC; kc++) dst[kc] = make_float4(pp[kc * 4], pp[kc * 4 + 1], pp[kc * 4 + 2], pp[kc * 4 + 3]);
            // every thread of the filter has read x (staged before the first barrier of this tile): in place is safe
            p.x_out[row] = xo;
            if (p.status && r == 0 && (st != BKE_STATUS_OK || !p.sticky)) p.status[f] = st;
        }
        // no barrier here: the operand buffers are free (both products were awaited), the scratch was read before the
        // last barrier, the update's chunks are rewritten only by their own warp (after its __syncwarp), and xs was read
        // before this tile's second barrier
    }
}

template <int NX, int M>
int launch_t(const TcP &p, cudaStream_t s)
{
    using G = Geom<NX>;
    static bool configured[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !configured[dev]) {
        if (check_cuda(cudaFuncSetAttribute(kf_cov_tc_kernel<NX, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, G::SMEM), "cudaFuncSetAttribute")) return BKE_ERR_CUDA;
        if (dev >= 0 && dev < 64) configured[dev] = true;
    }
    const int64_t tiles = (p.N * NX + 127) / 128;
    // CTAs per SM: registers (launch bounds) and shared memory (+1 KB the runtime reserves per CTA)
    int occ = tc_ctas(NX, M);
    if (occ > (227 * 1024) / (G::SMEM + 1024)) occ = (227 * 1024) / (G::SMEM + 1024);
    const int64_t cap = (int64_t)sm_count() * occ;
    kf_cov_tc_kernel<NX, M><<<(unsigned)(tiles < cap ? tiles : cap), 128, G::SMEM, s>>>(p);
    return check_cuda(cudaGetLastError(), "kf_cov_tc_kernel launch");
}

template <int NX>
int launch_m(const TcP &p, int m, cudaStream_t s)
{
    switch (m) {
    case 0: return launch_t<NX, 0>(p, s);
    case 1: return launch_t<NX, 1>(p, s);
    case 2: return launch_t<NX, 2>(p, s);
    case 3: return launch_t<NX, 3>(p, s);
    default: return launch_t<NX, 4>(p, s);
    }
}

}  // namespace tc

static bool al16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// Eligible: fp32, dim_x 16 / 32, F and Q shared, no control input.  A fused predict+update whose H and R are shared too
// and whose dim_z <= 4 runs entirely in this kernel; any other fused step runs its predict here and its update through
// launch_kf_any on the prior left in x_out / P_out.
int launch_kf_tc(const bke_kf_args &a, cudaStream_t s)
{
    if (a.dtype != BKE_F32 || !(a.dim_x == 16 || a.dim_x == 32)) return BKE_ERR_UNSUPPORTED;
    if (!(a.flags & BKE_DO_PREDICT) || (a.flags & BKE_UPDATE_FIRST)) return BKE_ERR_UNSUPPORTED;
    if (a.F_stride != 0 || a.Q_stride != 0 || (a.B && a.u)) return BKE_ERR_UNSUPPORTED;
    if (!(al16(a.x) && al16(a.P) && al16(a.x_out) && al16(a.P_out) && al16(a.x_prior) && al16(a.P_prior))) return BKE_ERR_UNSUPPORTED;
    const bool fused = (a.flags & BKE_DO_UPDATE) != 0;
    const bool fused_here = fused && a.H_stride == 0 && a.R_stride == 0 && a.dim_z >= 1 && a.dim_z <= 4 && a.z;
    // a 16/4 or 16/2 fused step this kernel does not take whole is faster as ONE row-block launch than as
    // predict-here + update-there
    if (fused && !fused_here && a.dim_x == 16 && (a.dim_z == 4 || a.dim_z == 2)) return BKE_ERR_UNSUPPORTED;
    // x_out may alias x and P_out may alias P (each tile reads its rows before it writes them); nothing else may overlap
    tc::TcP p;
    p.N = a.n_filters; p.alpha_sq = (float)a.alpha_sq;
    p.x = (const float *)a.x; p.P = (const float *)a.P; p.F = (const float *)a.F; p.Q = (const float *)a.Q;
    p.x_out = (float *)a.x_out; p.P_out = (float *)a.P_out; p.x_prior = (float *)a.x_prior; p.P_prior = (float *)a.P_prior;
    p.status = (fused && !fused_here) ? nullptr : a.status;      // the update that follows owns the status of a two-launch step
    p.sticky = (a.flags & BKE_STATUS_STICKY) ? 1 : 0;
    p.H = (const float *)a.H; p.R = (const float *)a.R; p.z = (const float *)a.z; p.valid = a.z_valid;
    p.K = (float *)a.K; p.y = (float *)a.y; p.S = (float *)a.S; p.SI = (float *)a.SI; p.ll = (float *)a.log_likelihood;
    const int m_here = fused_here ? a.dim_z : 0;
    int rc = a.dim_x == 16 ? tc::launch_m<16>(p, m_here, s) : tc::launch_m<32>(p, m_here, s);
    if (rc != BKE_OK || !fused || fused_here) return rc;
    // two-launch fused step: the update runs on the prior this launch left in x_out / P_out (stream order)
    bke_kf_args u = a;
    u.flags = (a.flags & ~(uint32_t)BKE_DO_PREDICT);
    u.x = a.x_out; u.P = a.P_out;
    u.x_prior = nullptr; u.P_prior = nullptr;         // written above
    return launch_kf_any(u, s);
}

}  // namespace bke
