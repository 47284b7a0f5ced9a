// ukf_rts_kernel.cuh — device code of the UKF RTS smoother (host side: ukf_rts.cu); free of host headers,
// compiled by nvcc for the built-in process models and by NVRTC around a user-supplied fx (ukf_rtc.cu).
//
// Per filter, backwards over the epochs k = T-2 .. 0 (UKF.py:708-737):
//     sigmas   = sigma_points(xs[k], Ps[k])                      (Merwe, sigma_points.py:160-177)
//     sigmas_f = fx(sigmas, dts[k])
//     xb, Pb   = unscented_transform(sigmas_f, Wm, Wc, Q)        (self.Q — the Qs argument is not used, :715)
//     Pxb      = sum Wc[i] outer(sigmas[i] - Xs[k], sigmas_f[i] - xb)
//     K        = Pxb inv(Pb)
//     xs[k]   += K (xs[k+1] - xb);   Ps[k] += K (Ps[k+1] - Pb) K'
// One thread per filter, thread-private arrays, any dim_x <= UR_MAXN: the correctness path for this
// §8f row (the per-step state — two covariances, a Cholesky factor, 2n+1 propagated points, an n x n
// inverse — does not fit a register tile at n = 6 in fp64).  Layout [T,N,...] as batch_filter writes it.
#pragma once
#include "bke_internal.cuh"
#include "ukf_kernel.cuh"

namespace bke {

constexpr int UR_MAXN = 8;

template <typename T>
struct UrP {
    int64_t N, Tn;
    int n, fx;
    T scale, wm0, wc0, wi, dt;
    const T *Xs, *Ps, *Q, *F;
    int64_t sQ, sF;
    const double *dts;
    T *x_out, *P_out, *K;
    int32_t *status;
    const T *fx_args;              // USER_FX instances: the parameter vector of the user's fx
    int64_t s_fx_args;             // 0 = one vector for the bank, else elements per filter
};

// the simplex offsets of ukfk::simplex_offsets for a run-time n: row j-1 of U (n x n, zero below the
// diagonal) becomes D_j, D0 receives D_0
template <typename T>
__device__ __forceinline__ void simplex_offsets_rt(int n, T *U, T *D0)
{
    T S[UR_MAXN];
    for (int i = 0; i < n; i++) S[i] = T(0);
    for (int j = n; j >= 2; j--) {
        const T c = ukfk::simplex_coef<T>(n, j);
        for (int i = j - 1; i < n; i++) {
            const T u = U[(j - 1) * n + i];
            U[(j - 1) * n + i] = T(-j) * c * u + S[i];
            S[i] += c * u;
        }
    }
    const T c1 = ukfk::simplex_coef<T>(n, 1);
    for (int i = 0; i < n; i++) {
        const T u = U[i];
        D0[i] = S[i] - c1 * u;
        U[i] = S[i] + c1 * u;
    }
}

// USER_FX: the process function is the user's (run-time compiled instance, ukf_rtc.cu); see ukf_kernel.cuh.
// SPX: the simplex point set (n + 1 points x + D_s, p.scale = 1, every weight 1/(n+1)).
template <typename T, bool USER_FX, bool SPX = false>
__global__ void __launch_bounds__(64) ukf_rts_kernel(UrP<T> p)
{
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= p.N) return;
    const int n = p.n, ns = SPX ? n + 1 : 2 * n + 1;
    T xs[UR_MAXN], Ps[UR_MAXN * UR_MAXN];                 // smoothed epoch k+1
    T xk[UR_MAXN], Pk[UR_MAXN * UR_MAXN];
    T U[UR_MAXN * UR_MAXN], Pb[UR_MAXN * UR_MAXN], Pxb[UR_MAXN * UR_MAXN], PbI[UR_MAXN * UR_MAXN], Kk[UR_MAXN * UR_MAXN];
    T sf[(2 * UR_MAXN + 1) * UR_MAXN], xb[UR_MAXN], tmp[UR_MAXN * UR_MAXN];
    T D0[SPX ? UR_MAXN : 1];                              // the simplex offset D_0
    const T *Q = p.Q + f * p.sQ;
    const T *F = p.F ? p.F + f * p.sF : nullptr;
    int64_t tf = (p.Tn - 1) * p.N + f;
    for (int i = 0; i < n; i++) { xs[i] = p.Xs[tf * n + i]; p.x_out[tf * n + i] = xs[i]; }
    for (int i = 0; i < n * n; i++) {
        Ps[i] = p.Ps[tf * n * n + i];
        p.P_out[tf * n * n + i] = Ps[i];
        if (p.K) p.K[tf * n * n + i] = T(0);
    }
    int st = BKE_STATUS_OK;
    for (int64_t k = p.Tn - 2; k >= 0; k--) {
        tf -= p.N;
        for (int i = 0; i < n; i++) xk[i] = p.Xs[tf * n + i];
        for (int i = 0; i < n * n; i++) Pk[i] = p.Ps[tf * n * n + i];
        bool ok = st == BKE_STATUS_OK;
        if (ok) {
            // U = chol_upper((n + lambda) Pk), upper triangle read (scipy.linalg.cholesky)
            for (int i = 0; i < n * n; i++) U[i] = T(0);
            for (int j = 0; j < n && ok; j++) {
                T d = p.scale * Pk[j * n + j];
                for (int q = 0; q < j; q++) d -= U[q * n + j] * U[q * n + j];
                if (!(d > T(0))) { ok = false; st = BKE_STATUS_NOT_PD; break; }
                const T r = sqrt(d), inv = T(1) / r;
                U[j * n + j] = r;
                for (int i = j + 1; i < n; i++) {
                    T s = p.scale * Pk[j * n + i];
                    for (int q = 0; q < j; q++) s -= U[q * n + j] * U[q * n + i];
                    U[j * n + i] = s * inv;
                }
            }
            if constexpr (SPX) {
                if (ok) simplex_offsets_rt<T>(n, U, D0);
            }
        }
        if (ok) {
            const T dt = p.dts ? (T)p.dts[k] : p.dt;
            // propagate the sigma points; xb = sum Wm f(sigma)
            for (int i = 0; i < n; i++) xb[i] = T(0);
            for (int s = 0; s < ns; s++) {
                T sp[UR_MAXN];
                const int row = s == 0 ? 0 : (s - 1) % n;
                const T sign = s == 0 ? T(0) : (s <= n ? T(1) : T(-1));
                if constexpr (SPX) {
                    for (int i = 0; i < n; i++) sp[i] = xk[i] + (s == 0 ? D0[i] : U[(s - 1) * n + i]);
                } else {
                    for (int i = 0; i < n; i++) sp[i] = (s == 0) ? xk[i] : xk[i] + sign * U[row * n + i];
                }
                T *fo = sf + s * n;
                if constexpr (USER_FX) {
                    ukfk::bke_user_fx<T>(sp, fo, dt, p.fx_args ? p.fx_args + f * p.s_fx_args : nullptr);
                } else if (p.fx == BKE_FX_LINEAR) {
                    for (int i = 0; i < n; i++) {
                        T a = T(0);
                        for (int j = 0; j < n; j++) a += F[i * n + j] * sp[j];
                        fo[i] = a;
                    }
                } else {
                    for (int i = 0; i < n; i += 2) { fo[i] = sp[i] + dt * sp[i + 1]; fo[i + 1] = sp[i + 1]; }
                }
                const T w = s == 0 ? p.wm0 : p.wi;
                for (int i = 0; i < n; i++) xb[i] += w * fo[i];
            }
            if constexpr (ukfk::HOOKS & BKE_HOOK_X_MEAN) {            // xb = x_mean_fn(sigmas_f, Wm) (:720-722)
                T Wm[2 * UR_MAXN + 1];
                for (int s = 0; s < ns; s++) Wm[s] = s == 0 ? p.wm0 : p.wi;
                ukfk::bke_hook_x_mean<T>(sf, Wm, xb);
            }
            // Pb = sum Wc y y' + Q ;  Pxb = sum Wc z y'   (z = sigma - Xs[k] = +-U row, y = f(sigma) - xb)
            for (int i = 0; i < n * n; i++) { Pb[i] = T(0); Pxb[i] = T(0); }
            for (int s = 0; s < ns; s++) {
                const T w = s == 0 ? p.wc0 : p.wi;
                const int row = s == 0 ? 0 : (s - 1) % n;
                const T sign = s == 0 ? T(0) : (s <= n ? T(1) : T(-1));
                T y[UR_MAXN];
                if constexpr (ukfk::HOOKS & BKE_HOOK_RESIDUAL_X) {
                    // y = residual_x(sigmas_f[i], xb), z = residual_x(sigmas[i], Xs[k]) (:727-728)
                    T sp[UR_MAXN], z[UR_MAXN];
                    ukfk::bke_hook_residual_x<T>(sf + s * n, xb, y);
                    if constexpr (SPX) {
                        for (int i = 0; i < n; i++) sp[i] = xk[i] + (s == 0 ? D0[i] : U[(s - 1) * n + i]);
                    } else {
                        for (int i = 0; i < n; i++) sp[i] = (s == 0) ? xk[i] : xk[i] + sign * U[row * n + i];
                    }
                    ukfk::bke_hook_residual_x<T>(sp, xk, z);
                    for (int i = 0; i < n; i++) {
                        const T wy = w * y[i], wz = w * z[i];
                        for (int j = 0; j < n; j++) { Pb[i * n + j] += wy * y[j]; Pxb[i * n + j] += wz * y[j]; }
                    }
                    continue;
                }
                for (int i = 0; i < n; i++) y[i] = sf[s * n + i] - xb[i];
                for (int i = 0; i < n; i++) {
                    const T wy = w * y[i];
                    for (int j = 0; j < n; j++) Pb[i * n + j] += wy * y[j];
                    if constexpr (SPX) {
                        // every simplex point is off x: (x + D_s) - x, formed as the reference does (:722)
                        const T z = (xk[i] + (s == 0 ? D0[i] : U[(s - 1) * n + i])) - xk[i];
                        const T wz = w * z;
                        for (int j = 0; j < n; j++) Pxb[i * n + j] += wz * y[j];
                    } else if (s > 0) {
                        // the reference forms (x + U) - x in floating point (:722); so does this
                        const T z = (xk[i] + sign * U[row * n + i]) - xk[i];
                        const T wz = w * z;
                        for (int j = 0; j < n; j++) Pxb[i * n + j] += wz * y[j];
                    }
                }
            }
            for (int i = 0; i < n * n; i++) Pb[i] += Q[i];
            // PbI = inv(Pb): Gauss-Jordan with partial pivoting on a copy
            for (int i = 0; i < n * n; i++) tmp[i] = Pb[i];
            for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) PbI[i * n + j] = (i == j) ? T(1) : T(0);
            for (int c = 0; c < n && ok; c++) {
                int pr = c;
                T best = fabs(tmp[c * n + c]);
                for (int r = c + 1; r < n; r++) { const T v = fabs(tmp[r * n + c]); if (v > best) { best = v; pr = r; } }
                if (best == T(0)) { ok = false; st = BKE_STATUS_SINGULAR_S; break; }
                if (pr != c)
                    for (int j = 0; j < n; j++) {
                        T t0 = tmp[c * n + j]; tmp[c * n + j] = tmp[pr * n + j]; tmp[pr * n + j] = t0;
                        T t1 = PbI[c * n + j]; PbI[c * n + j] = PbI[pr * n + j]; PbI[pr * n + j] = t1;
                    }
                const T d = T(1) / tmp[c * n + c];
                for (int j = 0; j < n; j++) { tmp[c * n + j] *= d; PbI[c * n + j] *= d; }
                for (int r = 0; r < n; r++) {
                    if (r == c) continue;
                    const T fm = tmp[r * n + c];
                    for (int j = 0; j < n; j++) { tmp[r * n + j] -= fm * tmp[c * n + j]; PbI[r * n + j] -= fm * PbI[c * n + j]; }
                }
            }
        }
        if (ok) {
            for (int i = 0; i < n; i++)
                for (int j = 0; j < n; j++) {
                    T s = T(0);
                    for (int q = 0; q < n; q++) s += Pxb[i * n + q] * PbI[q * n + j];
                    Kk[i * n + j] = s;
                }
            if constexpr (ukfk::HOOKS & BKE_HOOK_RESIDUAL_X) {
                T r[UR_MAXN];                                      // residual_x(xs[k+1], xb) (:735; no state_add)
                ukfk::bke_hook_residual_x<T>(xs, xb, r);
                for (int i = 0; i < n; i++) {
                    T s = T(0);
                    for (int q = 0; q < n; q++) s += Kk[i * n + q] * r[q];
                    xk[i] += s;
                }
            } else {
                for (int i = 0; i < n; i++) {
                    T s = T(0);
                    for (int q = 0; q < n; q++) s += Kk[i * n + q] * (xs[q] - xb[q]);
                    xk[i] += s;
                }
            }
            for (int i = 0; i < n; i++)
                for (int j = 0; j < n; j++) {
                    T s = T(0);
                    for (int q = 0; q < n; q++) s += Kk[i * n + q] * (Ps[q * n + j] - Pb[q * n + j]);
                    tmp[i * n + j] = s;
                }
            for (int i = 0; i < n; i++)
                for (int j = 0; j < n; j++) {
                    T s = T(0);
                    for (int q = 0; q < n; q++) s += tmp[i * n + q] * Kk[j * n + q];
                    Pk[i * n + j] += s;
                }
        } else {
            for (int i = 0; i < n * n; i++) Kk[i] = T(0);
        }
        for (int i = 0; i < n; i++) { xs[i] = xk[i]; p.x_out[tf * n + i] = xk[i]; }
        for (int i = 0; i < n * n; i++) {
            Ps[i] = Pk[i];
            p.P_out[tf * n * n + i] = Pk[i];
            if (p.K) p.K[tf * n * n + i] = Kk[i];
        }
    }
    if (p.status) p.status[f] = st;
}

}  // namespace bke
