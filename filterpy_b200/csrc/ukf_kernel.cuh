// ukf_kernel.cuh — device code of the unscented Kalman filter bank (see ukf.cu for the host side).
// Free of host headers: the same text is compiled by nvcc into libbke.so (closed set of fx / hx models)
// and by NVRTC around user-supplied fx / hx device functions (ukf_rtc.cu, bke_ukf_model_compile).
//
// Per filter (filterpy/kalman/UKF.py:364-411 predict, :413-491 update; sigma_points.py:160-177;
// unscented_transform.py:99-128; reference @ 3b51149):
//   U  = chol_upper((n+lambda) P)            rows of U are the sigma offsets (sigma_points.py:168-175)
//   Xs = {x, x + U[k,:], x - U[k,:]}         2n+1 points, propagated through fx
//   x- = sum Wm fx(Xs),  P- = sum Wc (fx(Xs)-x-)(..)' + Q           (unscented_transform.py:104-126)
//   Xs = sigma_points(x-, P-)                 REGENERATED from the prior (UKF.py:407)
//   Zs = hx(Xs);  z^ = sum Wm Zs;  S = sum Wc dz dz' + R;  Pxz = sum Wc dx dz'   (UKF.py:462-473)
//   K = Pxz S^-1;  x = x- + K (z - z^);  P = P- - K S K'                        (UKF.py:476-481)
//
// Register plan: the covariance accumulators (P-, then S and Pxz), U and the means live in
// registers; the 2n+1 propagated points are NOT stored — the cheap process models are evaluated
// twice (mean pass, covariance pass) — while the measurement-space points (which may cost a sqrt
// and two atan2 each) are parked in a conflict-free [point][component][thread] slab of shared
// memory.  F / H of the linear models sit in shared memory too (broadcast when shared by the bank).
// fx / hx are Python callables in the reference; here they come from the closed set in bke.h.
#pragma once
#include "bke_internal.cuh"
#include "kf_regtile.cuh"

namespace bke {
namespace ukfk {

constexpr int UB = 128;      // threads (= filters) per CTA

#ifndef BKE_UKF_HX_UNROLL
#define BKE_UKF_HX_UNROLL 1   // unroll factor of the run-time hx loop of the fp64 kernels
#endif

template <typename T>
struct UkfP {
    int64_t N;
    unsigned flags;
    T dt;
    T scale;                 // n + lambda
    T wm0, wc0, wi;          // Merwe weights (sigma_points.py:180-192)
    const T *x, *P, *Q, *R, *F, *H, *z;
    int64_t sQ, sR, sF, sH;
    const uint8_t *valid;
    T *x_out, *P_out, *x_prior, *P_prior, *K, *y, *S, *SI, *ll;
    int32_t *status;
    const T *fx_args, *hx_args;     // BKE_FX_USER / BKE_HX_USER: parameter vectors handed to the user's functions
    int64_t s_fx_args, s_hx_args;   // 0 = one vector for the bank, else elements per filter
};

// User-supplied process / measurement functions (run-time compiled instances, ukf_rtc.cu): the program
// text specialises these two for its element type; the pre-built instances never reference them.
template <typename T> __device__ void bke_user_fx(const T *x, T *out, T dt, const T *args);
template <typename T> __device__ void bke_user_hx(const T *x, T *z, const T *args);

// The reference's mean / residual / state-add hooks (UKF.py:97-140; x_mean_fn, z_mean_fn, residual_x,
// residual_z, state_add): BKE_UKF_HOOKS is the BKE_HOOK_* mask of the user functions the program text
// supplies.  Only run-time compiled instances define it (ukf_rtc.cu), so every hook below sits behind
// `if constexpr` and the pre-built instances compile to the code they had without hooks.
#ifndef BKE_UKF_HOOKS
#define BKE_UKF_HOOKS 0u
#endif
constexpr unsigned HOOKS = BKE_UKF_HOOKS;
template <typename T> __device__ void bke_hook_x_mean(const T *sigmas, const T *Wm, T *out);     // sigmas [2n+1][n]
template <typename T> __device__ void bke_hook_z_mean(const T *sigmas, const T *Wm, T *out);     // sigmas [2n+1][m]
template <typename T> __device__ void bke_hook_residual_x(const T *a, const T *b, T *out);
template <typename T> __device__ void bke_hook_residual_z(const T *a, const T *b, T *out);
template <typename T> __device__ void bke_hook_state_add(const T *a, const T *b, T *out);

template <int S> struct IntC { static constexpr int value = S; };

// upper Cholesky factor of A (upper triangle of A is read, like scipy.linalg.cholesky):
// U'U = A, U upper triangular (rows N.. of a taller U are left alone).  Returns false if A is not positive definite.
template <typename T, int N, int NR = N>
__device__ __forceinline__ bool chol_upper(const T (&A)[N][N], T (&U)[NR][N])
{
    bool ok = true;
#pragma unroll
    for (int j = 0; j < N; j++) {
        T d = A[j][j];
#pragma unroll
        for (int k = 0; k < j; k++) d -= U[k][j] * U[k][j];
        ok = ok && (d > T(0));
        // 1/sqrt(d) once, then the diagonal as d * (1/sqrt(d)): a reciprocal square root and a product
        // instead of a square root followed by a division on the critical path (both within ~1 ulp)
        T inv = rsqrt(d);
        T r = d * inv;
        U[j][j] = r;
#pragma unroll
        for (int i = j + 1; i < N; i++) {
            T s = A[j][i];
#pragma unroll
            for (int k = 0; k < j; k++) s -= U[k][j] * U[k][i];
            U[j][i] = s * inv;
        }
    }
    return ok;
}

// sigma point s of (x, U): x, x + U[k,:], x - U[k,:]   (sigma_points.py:171-175)
template <typename T, int N, int S>
__device__ __forceinline__ void sigma_point(const T (&x)[N], const T (&U)[N][N], T (&sp)[N])
{
    if constexpr (S == 0) {
#pragma unroll
        for (int i = 0; i < N; i++) sp[i] = x[i];
    } else if constexpr (S <= N) {
        constexpr int k = S - 1;
#pragma unroll
        for (int i = 0; i < N; i++) sp[i] = (i >= k) ? x[i] + U[k][i] : x[i];
    } else {
        constexpr int k = S - 1 - N;
#pragma unroll
        for (int i = 0; i < N; i++) sp[i] = (i >= k) ? x[i] - U[k][i] : x[i];
    }
}

// SimplexSigmaPoints (sigma_points.py:499-513): U = chol_upper(P) unscaled, Xi_j = x + D_j with
// D = (U' sqrt(n) Istar)'.  In closed form, with c_d = sqrt(n / (lambda d (d+1))) = sqrt((n+1) / (d (d+1)))
// and the suffix sums S_j = sum_{k >= j} c_{k+1} U[k,:]:
//     D_0 = -c_1 U[0,:] + S_1,   D_1 = c_1 U[0,:] + S_1,   D_j = -j c_j U[j-1,:] + S_j  (j >= 2).
// D_j (j >= 1) is zero left of column j-1, like row j-1 of U, and overwrites that row (j = n down to 1,
// with a running S); D_0 is dense and goes to the extra row U[n].  No simplex point equals x.
template <typename T>
__device__ __forceinline__ T simplex_coef(int n, int d)
{
    return T(sqrt(double(n + 1) / double(d * (d + 1))));
}

template <typename T, int N>
__device__ __forceinline__ void simplex_offsets(T (&U)[N + 1][N])
{
    T S[N];
#pragma unroll
    for (int i = 0; i < N; i++) S[i] = T(0);
#pragma unroll
    for (int j = N; j >= 2; j--) {
        const T c = simplex_coef<T>(N, j);
#pragma unroll
        for (int i = j - 1; i < N; i++) {
            const T u = U[j - 1][i];
            U[j - 1][i] = T(-j) * c * u + S[i];
            S[i] += c * u;
        }
    }
    const T c1 = simplex_coef<T>(N, 1);
#pragma unroll
    for (int i = 0; i < N; i++) {
        const T u = U[0][i];
        U[N][i] = S[i] - c1 * u;
        U[0][i] = S[i] + c1 * u;
    }
}

// sigma point S of the point set: Merwe's (U is [N][N]), or x + D_S of the simplex set (U is [N+1][N]: D_S in
// row S-1, D_0 in row N)
template <typename T, int N, int S, int NR>
__device__ __forceinline__ void point(const T (&x)[N], const T (&U)[NR][N], T (&sp)[N])
{
    if constexpr (NR == N) {
        sigma_point<T, N, S>(x, U, sp);
    } else if constexpr (S == 0) {
#pragma unroll
        for (int i = 0; i < N; i++) sp[i] = x[i] + U[N][i];
    } else {
        constexpr int k = S - 1;
#pragma unroll
        for (int i = 0; i < N; i++) sp[i] = (i >= k) ? x[i] + U[k][i] : x[i];
    }
}

template <typename T, int N, int FX>
__device__ __forceinline__ void apply_fx(const T (&s)[N], T (&f)[N], T dt, const T *Fs, int fstride, const T *uargs)
{
    if constexpr (FX == BKE_FX_USER) {
        bke_user_fx<T>(s, f, dt, uargs);
    } else if constexpr (FX == BKE_FX_LINEAR) {
#pragma unroll
        for (int i = 0; i < N; i++) {
            T a = Fs[(i * N) * fstride] * s[0];
#pragma unroll
            for (int j = 1; j < N; j++) a += Fs[(i * N + j) * fstride] * s[j];
            f[i] = a;
        }
    } else {   // BKE_FX_CONST_VEL
#pragma unroll
        for (int i = 0; i < N; i += 2) { f[i] = s[i] + dt * s[i + 1]; f[i + 1] = s[i + 1]; }
    }
}

template <typename T, int N, int M, int HX>
__device__ __forceinline__ void apply_hx(const T (&s)[N], T (&h)[M], const T *Hs, int hstride, const T *uargs)
{
    if constexpr (HX == BKE_HX_USER) {
        bke_user_hx<T>(s, h, uargs);
    } else if constexpr (HX == BKE_HX_LINEAR) {
#pragma unroll
        for (int a = 0; a < M; a++) {
            T v = Hs[(a * N) * hstride] * s[0];
#pragma unroll
            for (int j = 1; j < N; j++) v += Hs[(a * N + j) * hstride] * s[j];
            h[a] = v;
        }
    } else if constexpr (HX == BKE_HX_RANGE_AZ_EL) {
        T px = s[0], py = s[2], pz = s[4];
        T rho2 = px * px + py * py;
        h[0] = sqrt(rho2 + pz * pz);
        h[1] = atan2(py, px);
        h[2] = atan2(pz, sqrt(rho2));
    } else {   // BKE_HX_RANGE_BEARING
        T px = s[0], py = s[2];
        h[0] = sqrt(px * px + py * py);
        h[1] = atan2(py, px);
    }
}

// position of (i, j), i <= j, in a packed upper triangle
template <int N>
__device__ __forceinline__ constexpr int tri_index(int i, int j) { return i * N - i * (i - 1) / 2 + (j - i); }

// true when sigma offset row k (non-zero in the components >= k) leaves every input of hx unchanged,
// so hx(x +- U[k,:]) == hx(x) bit for bit
template <int HX, int N>
__device__ __forceinline__ constexpr bool hx_ignores_row(int k)
{
    return HX == BKE_HX_RANGE_AZ_EL ? k > 4 : (HX == BKE_HX_RANGE_BEARING ? k > 2 : false);
}

// the transcendental models from the position components alone (same arithmetic as apply_hx)
template <typename T, int M, int HX>
__device__ __forceinline__ void hx_positions(const T (&pos)[M], T (&h)[M])
{
    if constexpr (HX == BKE_HX_RANGE_AZ_EL) {
        const T px = pos[0], py = pos[1], pz = pos[2];
        const T rho2 = px * px + py * py;
        h[0] = sqrt(rho2 + pz * pz);
        h[1] = atan2(py, px);
        h[2] = atan2(pz, sqrt(rho2));
    } else {   // BKE_HX_RANGE_BEARING
        const T px = pos[0], py = pos[1];
        h[0] = sqrt(px * px + py * py);
        h[1] = atan2(py, px);
    }
}

// Angles of a sigma point relative to the mean point.  The sigma points sit within a few standard
// deviations of the mean, so the angle between the two position vectors is small and
//     atan2(py, px) = atan2(py0, px0) + atan2(px0 py - py0 px, px0 px + py0 py)
// (exact geometry: the second term is the signed angle from the mean direction to the point) needs
// only a short odd series for its arctangent: for |t| < 1/16 the series through t^13 (fp64) /
// t^5 (fp32) is below half an ulp of the sum.  Wider angles take the library atan2.  The result is
// wrapped into (-pi, pi] like atan2's.  A full fp64 atan2 is ~150 instructions; 2n of the 2n+1
// evaluations per angle become a division and a 7-term polynomial.
template <typename T>
__device__ __forceinline__ bool atan_small(T cross, T dot, T &delta)
{
    if (!(fabs(cross) < T(0.0625) * dot)) return false;            // also false for dot <= 0 and NaN
    const T t = cross / dot, t2 = t * t;
    T pl;
    if constexpr (sizeof(T) == 8) {
        pl = T(1.0 / 13.0);
        pl = pl * t2 - T(1.0 / 11.0);
        pl = pl * t2 + T(1.0 / 9.0);
        pl = pl * t2 - T(1.0 / 7.0);
        pl = pl * t2 + T(1.0 / 5.0);
        pl = pl * t2 - T(1.0 / 3.0);
    } else {
        pl = T(1.0 / 5.0);
        pl = pl * t2 - T(1.0 / 3.0);
    }
    delta = t + t * (t2 * pl);
    return true;
}

template <typename T>
__device__ __forceinline__ T wrap_pi(T a)
{
    const T pi = T(3.14159265358979323846);
    if (a > pi) a -= T(2) * pi;
    else if (a <= -pi) a += T(2) * pi;
    return a;
}

// hx of a sigma point given the mean point's positions pos0 (and its horizontal range rho0) and hx(mean) = h0
template <typename T, int M, int HX>
__device__ __forceinline__ void hx_positions_rel(const T (&pos)[M], const T (&pos0)[M], T rho0, const T (&h0)[M], T (&h)[M])
{
    const T px = pos[0], py = pos[1], px0 = pos0[0], py0 = pos0[1];
    const T rho2 = px * px + py * py;
    T d;
    if constexpr (HX == BKE_HX_RANGE_AZ_EL) {
        const T pz = pos[2], pz0 = pos0[2];
        h[0] = sqrt(rho2 + pz * pz);
        h[1] = atan_small<T>(px0 * py - py0 * px, px0 * px + py0 * py, d) ? wrap_pi<T>(h0[1] + d) : atan2(py, px);
        const T rho = sqrt(rho2);
        h[2] = atan_small<T>(rho0 * pz - pz0 * rho, rho0 * rho + pz0 * pz, d) ? h0[2] + d : atan2(pz, rho);
    } else {   // BKE_HX_RANGE_BEARING
        h[0] = sqrt(rho2);
        h[1] = atan_small<T>(px0 * py - py0 * px, px0 * px + py0 * py, d) ? wrap_pi<T>(h0[1] + d) : atan2(py, px);
    }
}

// compile-time loop over the 2N+1 sigma points
template <int S, int END, typename Fn>
__device__ __forceinline__ void for_sigma(Fn &&fn)
{
    if constexpr (S < END) {
        fn(IntC<S>{});
        for_sigma<S + 1, END>(fn);
    }
}

// Cooperative, coalesced movement of a tile's [filters][PER] block between global memory and a
// shared-memory slab whose per-filter stride PAD is odd: the strided per-thread accesses of the
// owning threads are then bank-conflict-free (a thread-per-filter LDG of AoS data would touch one
// cache line per lane per instruction).
template <typename T, int PER, int PAD>
__device__ __forceinline__ void slab_load(T *slab, const T *g, int cnt)
{
    if (cnt == UB) {
        // full tile: all PER loads of a thread are in flight before the first store (a plain loop
        // exposed one global-load latency per few iterations: the top long-scoreboard stall)
        constexpr int CH = PER % 12 == 0 ? 12 : (PER % 9 == 0 ? 9 : (PER % 4 == 0 ? 4 : 1));
#pragma unroll
        for (int k0 = 0; k0 < PER; k0 += CH) {
            T v[CH];
#pragma unroll
            for (int k = 0; k < CH; k++) v[k] = g[threadIdx.x + (k0 + k) * UB];
#pragma unroll
            for (int k = 0; k < CH; k++) {
                const int e = threadIdx.x + (k0 + k) * UB;
                slab[(e / PER) * PAD + (e % PER)] = v[k];
            }
        }
        return;
    }
    for (int e = threadIdx.x; e < cnt * PER; e += UB) slab[(e / PER) * PAD + (e % PER)] = g[e];
}
template <typename T, int PER, int PAD>
__device__ __forceinline__ void slab_store(T *g, const T *slab, int cnt)
{
    for (int e = threadIdx.x; e < cnt * PER; e += UB) g[e] = slab[(e / PER) * PAD + (e % PER)];
}

// The measurement half of the update (UKF.py:407, 462-473): sigma points of (x, P) (U: the Cholesky rows, or
// the simplex offsets), hx of every point into the slab zs ([NS*M][UB]), z^ = zm (or z_mean_fn), S = Sc
// (residual_z, then + R) and its inverse.  Returns false where S is singular; a failed Cholesky sets
// st = BKE_STATUS_NOT_PD.  p is the kernel's parameter block (its scale, wm0, wc0 and wi are read).  The fused step
// and the measurement scores (ukf_score_kernel.cuh) share it:
//   after_chol()           once U is drawn (the step parks P there)
//   prefetch(Rv)           loads R [M][M] ahead of the covariance pass (the step fetches z with it)
//   cross(IntC<S>, w, dz)  every point's weighted residual dz (the step accumulates Pxz)
template <typename T, int N, int M, int HX, bool SPX, typename PP, typename AfterChol, typename Prefetch, typename Cross>
__device__ __forceinline__ bool meas_ut(const PP &p, const T (&x)[N], const T (&P)[N][N], T (&U)[SPX ? N + 1 : N][N], T *zs, int tid,
                                        const T *Hp, int hstride, const T *hxa, int &st, T (&zm)[M], T (&Sc)[M][M], T (&SI)[M][M], T &logdet, AfterChol &&after_chol, Prefetch &&prefetch,
                                        Cross &&cross)
{
    constexpr int NS = SPX ? N + 1 : 2 * N + 1;
    // sigma points regenerated from the prior (UKF.py:407); scipy's cholesky reads the upper triangle
    {
        T A[N][N];
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int j = i; j < N; j++) A[i][j] = p.scale * P[i][j];
        if (!chol_upper<T, N>(A, U)) st = BKE_STATUS_NOT_PD;
        if constexpr (SPX) simplex_offsets<T, N>(U);
    }
    after_chol();
#pragma unroll
    for (int a = 0; a < M; a++) zm[a] = T(0);
    if constexpr (HX == BKE_HX_LINEAR || HX == BKE_HX_USER) {
        for_sigma<0, NS>([&](auto sc) {
            constexpr int S = decltype(sc)::value;
            T sp[N], h[M];
            point<T, N, S>(x, U, sp);
            apply_hx<T, N, M, HX>(sp, h, Hp, hstride, hxa);
            const T w = (S == 0) ? p.wm0 : p.wi;
#pragma unroll
            for (int a = 0; a < M; a++) { zm[a] += w * h[a]; zs[(S * M + a) * UB + tid] = h[a]; }
        });
    } else if constexpr (SPX) {
        // The transcendental models on the simplex set: as below, the positions are parked and a
        // run-time loop evaluates hx in place, but no point equals x, so hx(x) (weight 0) is the
        // reference direction of the relative angles.  D_j with j - 1 past the last position
        // component leaves the positions of x unchanged: that point's hx is hx(x).
        for_sigma<0, NS>([&](auto sc) {
            constexpr int S = decltype(sc)::value;
            T sp[N];
            point<T, N, S>(x, U, sp);
#pragma unroll
            for (int a = 0; a < M; a++) zs[(S * M + a) * UB + tid] = sp[2 * a];
        });
        T h0[M], pos0[M];
#pragma unroll
        for (int a = 0; a < M; a++) pos0[a] = x[2 * a];
        hx_positions<T, M, HX>(pos0, h0);
        const T rho0 = sqrt(pos0[0] * pos0[0] + pos0[1] * pos0[1]);
#pragma unroll 1
        for (int s = 0; s < NS; s++) {
            T h[M];
            if (s >= 2 && hx_ignores_row<HX, N>(s - 1)) {
#pragma unroll
                for (int a = 0; a < M; a++) h[a] = h0[a];
            } else {
                T pa[M];
#pragma unroll
                for (int a = 0; a < M; a++) pa[a] = zs[(s * M + a) * UB + tid];
                hx_positions_rel<T, M, HX>(pa, pos0, rho0, h0, h);
            }
#pragma unroll
            for (int a = 0; a < M; a++) { zm[a] += p.wi * h[a]; zs[(s * M + a) * UB + tid] = h[a]; }
        }
    } else {
        // Transcendental measurement models: the inputs hx reads (M position components per
        // sigma point) are parked in the slab first, then a run-time loop over the n offset
        // rows evaluates hx in place for the +row / -row pair (two independent chains per
        // iteration).  Unrolling 2n+1 inlined atan2/sqrt bodies made the fp64 kernel 117 KB of
        // code (instruction-cache hit rate 83 %, `no_instruction` the second largest stall).
        for_sigma<0, NS>([&](auto sc) {
            constexpr int S = decltype(sc)::value;
            T sp[N];
            sigma_point<T, N, S>(x, U, sp);
#pragma unroll
            for (int a = 0; a < M; a++) zs[(S * M + a) * UB + tid] = sp[2 * a];      // positions sit at 0, 2, 4
        });
        T h0[M], pos0[M];
        {
#pragma unroll
            for (int a = 0; a < M; a++) pos0[a] = zs[a * UB + tid];
            hx_positions<T, M, HX>(pos0, h0);
#pragma unroll
            for (int a = 0; a < M; a++) { zm[a] += p.wm0 * h0[a]; zs[a * UB + tid] = h0[a]; }
        }
        const T rho0 = sqrt(pos0[0] * pos0[0] + pos0[1] * pos0[1]);
#pragma unroll 1
        for (int k = 0; k < N; k++) {
            const int sa = k + 1, sb = k + 1 + N;
            T ha[M], hb[M];
            if (hx_ignores_row<HX, N>(k)) {               // this offset row leaves the positions alone
#pragma unroll
                for (int a = 0; a < M; a++) { ha[a] = h0[a]; hb[a] = h0[a]; }
            } else {
                T pa[M], pb[M];
#pragma unroll
                for (int a = 0; a < M; a++) { pa[a] = zs[(sa * M + a) * UB + tid]; pb[a] = zs[(sb * M + a) * UB + tid]; }
                hx_positions_rel<T, M, HX>(pa, pos0, rho0, h0, ha);
                hx_positions_rel<T, M, HX>(pb, pos0, rho0, h0, hb);
            }
#pragma unroll
            for (int a = 0; a < M; a++) {
                zm[a] += p.wi * ha[a]; zm[a] += p.wi * hb[a];
                zs[(sa * M + a) * UB + tid] = ha[a]; zs[(sb * M + a) * UB + tid] = hb[a];
            }
        }
    }
    if constexpr (HOOKS & BKE_HOOK_Z_MEAN) {                // z_mean_fn(sigmas_h, Wm) (UKF.py:469)
        T sh[NS * M], Wm[NS];
#pragma unroll
        for (int s = 0; s < NS; s++) {
            Wm[s] = (s == 0) ? p.wm0 : p.wi;
#pragma unroll
            for (int a = 0; a < M; a++) sh[s * M + a] = zs[(s * M + a) * UB + tid];
        }
        bke_hook_z_mean<T>(sh, Wm, zm);
    }
    // R is needed after the covariance pass below: fetch it now so that its latency hides behind it (with z
    // in the step, they were the largest long-scoreboard stalls of the update)
    T Rv[M][M];
    prefetch(Rv);
#pragma unroll
    for (int a = 0; a < M; a++)
#pragma unroll
        for (int b = a; b < M; b++) Sc[a][b] = T(0);
    for_sigma<0, NS>([&](auto sc) {
        constexpr int S = decltype(sc)::value;
        T dz[M];
        if constexpr (HOOKS & BKE_HOOK_RESIDUAL_Z) {
            T h[M];
#pragma unroll
            for (int a = 0; a < M; a++) h[a] = zs[(S * M + a) * UB + tid];
            bke_hook_residual_z<T>(h, zm, dz);
        } else {
#pragma unroll
            for (int a = 0; a < M; a++) dz[a] = zs[(S * M + a) * UB + tid] - zm[a];
        }
        const T w = (S == 0) ? p.wc0 : p.wi;
#pragma unroll
        for (int a = 0; a < M; a++) {
            T wd = w * dz[a];
#pragma unroll
            for (int b = a; b < M; b++) Sc[a][b] += wd * dz[b];
        }
        cross(sc, w, dz);
    });
#pragma unroll
    for (int a = 0; a < M; a++)
#pragma unroll
        for (int b = a; b < M; b++) {
            const T sab = Sc[a][b];
            Sc[a][b] = sab + Rv[a][b];
            if (b > a) Sc[b][a] = sab + Rv[b][a];
        }
    return reg_inverse<T, M>(Sc, SI, logdet);
}

// UKF_EXTRAS: the optional outputs (priors, K, y, S, SI, log-likelihood) are compiled in; the plain
// instantiation is 2-4 % faster without their tests and live ranges.
// SPX: the simplex point set (n + 1 points, p.scale = 1, every weight 1/(n+1)) instead of Merwe's.
template <typename T, int N, int M, int FX, int HX, int OCC, bool UKF_EXTRAS, bool SPX = false>
__global__ void __launch_bounds__(UB, OCC) ukf_kernel(UkfP<T> p)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int NS = SPX ? N + 1 : 2 * N + 1;
    constexpr int PADP = (N * N) | 1;                        // odd per-filter stride of the P / Q slab
    constexpr int NT = N * (N + 1) / 2;
    constexpr int SLAB = (NS * M + NT > PADP ? NS * M + NT : PADP) * UB;
    T *zs = reinterpret_cast<T *>(smem_raw);                 // [NS*M][UB]; doubles as the staging slab for P, Q, P_out
    T *park = zs + NS * M * UB;                              // [NT][UB]: the prior covariance while the update works
    T *Fs = zs + SLAB;                                       // [N*N] or [N*N][UB]
    const bool do_p = p.flags & BKE_DO_PREDICT, do_u = p.flags & BKE_DO_UPDATE;
    const int tid = threadIdx.x;
    const int64_t f = (int64_t)blockIdx.x * UB + tid;
    const bool live = f < p.N;
    const int64_t fc = live ? f : p.N - 1;                   // clamp: dead threads redo the last filter

    // stage F / H (linear models) in shared memory
    int fstride = 1, foff = 0;
    T *Hs = Fs;
    if (FX == BKE_FX_LINEAR && do_p) {
        if (p.sF == 0) { for (int e = tid; e < N * N; e += UB) Fs[e] = p.F[e]; Hs = Fs + N * N; }
        else {
            for (int e = 0; e < N * N; e++) Fs[e * UB + tid] = p.F[fc * p.sF + e];
            fstride = UB; foff = tid; Hs = Fs + N * N * UB;
        }
    }
    int hstride = 1, hoff = 0;
    if (HX == BKE_HX_LINEAR && do_u) {
        if (p.sH == 0) { for (int e = tid; e < M * N; e += UB) Hs[e] = p.H[e]; }
        else {
            for (int e = 0; e < M * N; e++) Hs[e * UB + tid] = p.H[fc * p.sH + e];
            hstride = UB; hoff = tid;
        }
    }
    __syncthreads();
    const T *Fp = Fs + foff, *Hp = Hs + hoff;
    const T *fxa = (FX == BKE_FX_USER && p.fx_args) ? p.fx_args + ((f < p.N) ? f : p.N - 1) * p.s_fx_args : nullptr;
    const T *hxa = (HX == BKE_HX_USER && p.hx_args) ? p.hx_args + ((f < p.N) ? f : p.N - 1) * p.s_hx_args : nullptr;

    const int64_t tile0 = (int64_t)blockIdx.x * UB;
    const int cnt = (int)((p.N - tile0) < UB ? (p.N - tile0) : UB);
    const int tl = live ? tid : cnt - 1;                     // slab row of this thread's filter
    T x[N], P[N][N];
#pragma unroll
    for (int i = 0; i < N; i++) x[i] = p.x[fc * N + i];
    slab_load<T, N * N, PADP>(zs, p.P + tile0 * N * N, cnt);
    __syncthreads();
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = 0; j < N; j++) P[i][j] = zs[tl * PADP + i * N + j];
    __syncthreads();
    const bool q_dense = do_p && p.sQ != 0;
    if (q_dense) slab_load<T, N * N, PADP>(zs, p.Q + tile0 * N * N, cnt);     // parked until the end of predict
    __syncthreads();
    int st = BKE_STATUS_OK;
    T U[SPX ? N + 1 : N][N];                                 // the simplex set keeps its offset D_0 in row N

    if (do_p) {
        T A[N][N];
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int j = 0; j < N; j++) A[i][j] = p.scale * P[i][j];
        if (!chol_upper<T, N>(A, U)) st = BKE_STATUS_NOT_PD;
        if constexpr (SPX) simplex_offsets<T, N>(U);
        // pass 1: mean of the propagated points
        T xm[N];
#pragma unroll
        for (int i = 0; i < N; i++) xm[i] = T(0);
        // x_mean_fn sees every propagated point at once (UKF.py:403): only that instance stages them
        T sf[(HOOKS & BKE_HOOK_X_MEAN) ? NS : 1][N];
        if constexpr (HOOKS & BKE_HOOK_X_MEAN) {
            T Wm[NS];
            for_sigma<0, NS>([&](auto sc) {
                constexpr int S = decltype(sc)::value;
                T sp[N];
                point<T, N, S>(x, U, sp);
                apply_fx<T, N, FX>(sp, sf[S], p.dt, Fp, fstride, fxa);
                Wm[S] = (S == 0) ? p.wm0 : p.wi;
            });
            bke_hook_x_mean<T>(&sf[0][0], Wm, xm);
        } else {
            for_sigma<0, NS>([&](auto sc) {
                constexpr int S = decltype(sc)::value;
                T sp[N], fs[N];
                point<T, N, S>(x, U, sp);
                apply_fx<T, N, FX>(sp, fs, p.dt, Fp, fstride, fxa);
                const T w = (S == 0) ? p.wm0 : p.wi;
#pragma unroll
                for (int i = 0; i < N; i++) xm[i] += w * fs[i];
            });
        }
        // pass 2: covariance (upper triangle; mirrored when Q is added)
        T Pm[N][N];
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int j = i; j < N; j++) Pm[i][j] = T(0);
        for_sigma<0, NS>([&](auto sc) {
            constexpr int S = decltype(sc)::value;
            T sp[N], fs[N];
            if constexpr (HOOKS & BKE_HOOK_X_MEAN) {
#pragma unroll
                for (int i = 0; i < N; i++) fs[i] = sf[S][i];
            } else {
                point<T, N, S>(x, U, sp);
                apply_fx<T, N, FX>(sp, fs, p.dt, Fp, fstride, fxa);
            }
            const T w = (S == 0) ? p.wc0 : p.wi;
            T d[N];
            if constexpr (HOOKS & BKE_HOOK_RESIDUAL_X) {
                bke_hook_residual_x<T>(fs, xm, d);
            } else {
#pragma unroll
                for (int i = 0; i < N; i++) d[i] = fs[i] - xm[i];
            }
#pragma unroll
            for (int i = 0; i < N; i++) {
                T wd = w * d[i];
#pragma unroll
                for (int j = i; j < N; j++) Pm[i][j] += wd * d[j];
            }
        });
#pragma unroll
        for (int i = 0; i < N; i++) {
            x[i] = xm[i];
#pragma unroll
            for (int j = i; j < N; j++) {
                P[i][j] = Pm[i][j] + (q_dense ? zs[tl * PADP + i * N + j] : p.Q[i * N + j]);
                if (j > i) P[j][i] = Pm[i][j] + (q_dense ? zs[tl * PADP + j * N + i] : p.Q[j * N + i]);
            }
        }
        if (UKF_EXTRAS && live) {
            if (p.x_prior) for (int i = 0; i < N; i++) p.x_prior[f * N + i] = x[i];
            if (p.P_prior) for (int i = 0; i < N; i++) for (int j = 0; j < N; j++) p.P_prior[f * N * N + i * N + j] = P[i][j];
        }
    }

    __syncthreads();                                         // Q has been consumed: the slab now holds hx(sigma points)
    if (do_u) {
        const bool has_z = (p.valid == nullptr) || (p.valid[fc] != 0);
        if (has_z && st == BKE_STATUS_OK) {
            bool asym = false;
            T zm[M];
            KfUpdateOut<T, N, M> o;
            T Pxz[N][M], zv[M];
            o.ok = meas_ut<T, N, M, HX, SPX>(p, x, P, U, zs, tid, Hp, hstride, hxa, st, zm, o.S, o.SI, o.logdet,
                [&] {
                    // P is not needed again until the posterior: park its upper triangle in shared memory and
                    // free the registers.  A (never expected) non-symmetric P keeps its lower triangle in P_out.
#pragma unroll
                    for (int i = 0; i < N; i++)
#pragma unroll
                        for (int j = i; j < N; j++) {
                            park[tri_index<N>(i, j) * UB + tid] = P[i][j];
                            if (j > i) asym = asym || (P[j][i] != P[i][j]);
                        }
                    if (asym && live) {
#pragma unroll
                        for (int i = 0; i < N; i++)
#pragma unroll
                            for (int j = 0; j < i; j++) p.P_out[f * N * N + i * N + j] = P[i][j];
                    }
                },
                [&](T (&Rv)[M][M]) {
                    // z is needed after the covariance pass too: it comes with R
                    const T *Rf = p.R + fc * p.sR;
#pragma unroll
                    for (int a = 0; a < M; a++) {
                        zv[a] = p.z[fc * M + a];
#pragma unroll
                        for (int b = 0; b < M; b++) Rv[a][b] = Rf[a * M + b];
                    }
#pragma unroll
                    for (int i = 0; i < N; i++)
#pragma unroll
                        for (int a = 0; a < M; a++) Pxz[i][a] = T(0);
                },
                [&](auto sc, T w, const T (&dz)[M]) {
                    constexpr int S = decltype(sc)::value;
                    if constexpr (HOOKS & BKE_HOOK_RESIDUAL_X) {
                        // dx = residual_x(sigma, x) (UKF.py:501): the point itself, not the offset row
                        T sp[N], dx[N];
                        point<T, N, S>(x, U, sp);
                        bke_hook_residual_x<T>(sp, x, dx);
#pragma unroll
                        for (int i = 0; i < N; i++) {
                            T wd = w * dx[i];
#pragma unroll
                            for (int a = 0; a < M; a++) Pxz[i][a] += wd * dz[a];
                        }
                    } else if constexpr (SPX) {
                        // dx = sigma - x = D_S: row N of U, or row S-1 (zero left of column S-1)
                        constexpr int k = S == 0 ? 0 : S - 1, row = S == 0 ? N : S - 1;
#pragma unroll
                        for (int i = k; i < N; i++) {
                            T wd = w * U[row][i];
#pragma unroll
                            for (int a = 0; a < M; a++) Pxz[i][a] += wd * dz[a];
                        }
                    } else if constexpr (S > 0) {
                        // dx = sigma - x is the sigma offset itself: row k of +-U, zero left of the diagonal
                        constexpr int k = (S - 1) % N;
                        const T ws = (S <= N) ? w : -w;
#pragma unroll
                        for (int i = k; i < N; i++) {
                            T wd = ws * U[k][i];
#pragma unroll
                            for (int a = 0; a < M; a++) Pxz[i][a] += wd * dz[a];
                        }
                    }
                });
            if (!o.ok) st = BKE_STATUS_SINGULAR_S;
            const bool good = o.ok && st == BKE_STATUS_OK;
            T SK[M][N];
            if (good) {
#pragma unroll
                for (int i = 0; i < N; i++)
#pragma unroll
                    for (int a = 0; a < M; a++) {
                        T s = Pxz[i][0] * o.SI[0][a];
#pragma unroll
                        for (int b = 1; b < M; b++) s += Pxz[i][b] * o.SI[b][a];
                        o.K[i][a] = s;
                    }
                if constexpr (HOOKS & BKE_HOOK_RESIDUAL_Z) {
                    bke_hook_residual_z<T>(zv, zm, o.y);                  // UKF.py:477
                } else {
#pragma unroll
                    for (int a = 0; a < M; a++) o.y[a] = zv[a] - zm[a];
                }
                if constexpr (HOOKS & BKE_HOOK_STATE_ADD) {
                    T ky[N], xn[N];                                        // state_add(x, K y) (UKF.py:480)
#pragma unroll
                    for (int i = 0; i < N; i++) {
                        T s = o.K[i][0] * o.y[0];
#pragma unroll
                        for (int a = 1; a < M; a++) s += o.K[i][a] * o.y[a];
                        ky[i] = s;
                    }
                    bke_hook_state_add<T>(x, ky, xn);
#pragma unroll
                    for (int i = 0; i < N; i++) x[i] = xn[i];
                } else {
#pragma unroll
                    for (int i = 0; i < N; i++) {
                        T s = x[i];
#pragma unroll
                        for (int a = 0; a < M; a++) s += o.K[i][a] * o.y[a];
                        x[i] = s;
                    }
                }
                // optional outputs leave now, while S, SI, y are still in registers
                if (UKF_EXTRAS && live) {
                    if (p.K) for (int i = 0; i < N; i++) for (int a = 0; a < M; a++) p.K[f * N * M + i * M + a] = o.K[i][a];
                    if (p.y) for (int a = 0; a < M; a++) p.y[f * M + a] = o.y[a];
                    if (p.S) for (int a = 0; a < M; a++) for (int b = 0; b < M; b++) p.S[f * M * M + a * M + b] = o.S[a][b];
                    if (p.SI) for (int a = 0; a < M; a++) for (int b = 0; b < M; b++) p.SI[f * M * M + a * M + b] = o.SI[a][b];
                    if (p.ll) {
                        T q = T(0);
#pragma unroll
                        for (int a = 0; a < M; a++) {
                            T s = T(0);
#pragma unroll
                            for (int b = 0; b < M; b++) s += o.SI[a][b] * o.y[b];
                            q += o.y[a] * s;
                        }
                        p.ll[f] = T(-0.5) * (q + o.logdet + T(M) * T(LOG_2PI));
                    }
                }
                // S K' for P = P - K (S K')
#pragma unroll
                for (int a = 0; a < M; a++)
#pragma unroll
                    for (int j = 0; j < N; j++) {
                        T s = o.S[a][0] * o.K[j][0];
#pragma unroll
                        for (int b = 1; b < M; b++) s += o.S[a][b] * o.K[j][b];
                        SK[a][j] = s;
                    }
            }
            // the prior covariance comes back from its parking place
#pragma unroll
            for (int i = 0; i < N; i++)
#pragma unroll
                for (int j = i; j < N; j++) { P[i][j] = park[tri_index<N>(i, j) * UB + tid]; P[j][i] = P[i][j]; }
            if (asym && live) {
#pragma unroll
                for (int i = 0; i < N; i++)
#pragma unroll
                    for (int j = 0; j < i; j++) P[i][j] = p.P_out[f * N * N + i * N + j];
            }
            if (good) {
#pragma unroll
                for (int i = 0; i < N; i++)
#pragma unroll
                    for (int j = i; j < N; j++) {
                        T s = o.K[i][0] * SK[0][j];
#pragma unroll
                        for (int a = 1; a < M; a++) s += o.K[i][a] * SK[a][j];
                        P[i][j] -= s;
                        if (j > i) P[j][i] -= s;
                    }
            }
        }
    }
    __syncthreads();                                         // the slab is free again: stage the posterior covariance
    if (live) {
#pragma unroll
        for (int i = 0; i < N; i++) p.x_out[f * N + i] = x[i];
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int j = 0; j < N; j++) zs[tid * PADP + i * N + j] = P[i][j];
        if (p.status) p.status[f] = st;
    }
    __syncthreads();
    slab_store<T, N * N, PADP>(p.P_out + tile0 * N * N, zs, cnt);
}

}  // namespace ukfk
}  // namespace bke
