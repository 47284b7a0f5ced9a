// kf_regtile.cuh — one filter's predict/update held entirely in registers (thread-per-filter
// tile used by the specialised kernels in kf_fast.cu).  Fully unrolled for compile-time (N, M);
// every array index is a constant so nothing touches local memory.
//
// Arithmetic (filterpy/kalman/kalman_filter.py, reference @ 3b51149):
//   predict :471-478   x = F x ;  P = alpha_sq * (F P) F' + Q
//   update  :533-556   y = z - H x ; PHT = P H' ; S = H PHT + R ; SI = S^-1 ; K = PHT SI ;
//                      x = x + K y ; P = (I-KH) P (I-KH)' + (K R) K'
#pragma once
#include "bke_internal.cuh"

namespace bke {

template <typename T, int N, int M>
struct KfRegs {
    T x[N];
    T P[N][N];
};

template <typename T, int N>
__device__ __forceinline__ void reg_predict(T (&x)[N], T (&P)[N][N], const T (&F)[N][N], const T (&Q)[N][N], T alpha_sq)
{
    T xn[N];
#pragma unroll
    for (int i = 0; i < N; i++) {
        T s = F[i][0] * x[0];
#pragma unroll
        for (int k = 1; k < N; k++) s += F[i][k] * x[k];
        xn[i] = s;
    }
    T FP[N][N];
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = 0; j < N; j++) {
            T s = F[i][0] * P[0][j];
#pragma unroll
            for (int k = 1; k < N; k++) s += F[i][k] * P[k][j];
            FP[i][j] = s;
        }
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = 0; j < N; j++) {
            T s = FP[i][0] * F[j][0];
#pragma unroll
            for (int k = 1; k < N; k++) s += FP[i][k] * F[j][k];
            P[i][j] = alpha_sq * s + Q[i][j];
        }
#pragma unroll
    for (int i = 0; i < N; i++) x[i] = xn[i];
}

// In-register inverse of a small M x M matrix: closed form for M <= 2, Gauss-Jordan with partial
// pivoting for M >= 3 (an indefinite but non-singular S — numerical drift of P, a user R that is not
// PD — inverts exactly where np.linalg.inv does).  Returns false on a zero pivot = singular S.
// logdet = log |det S|.
template <typename T, int M>
__device__ __forceinline__ bool reg_inverse(const T (&S)[M][M], T (&SI)[M][M], T &logdet)
{
    if constexpr (M == 1) {
        logdet = log(fabs(S[0][0]));
        SI[0][0] = T(1) / S[0][0];
        return S[0][0] != T(0);
    } else if constexpr (M == 2) {
        T det = S[0][0] * S[1][1] - S[0][1] * S[1][0];
        T r = T(1) / det;
        SI[0][0] = S[1][1] * r; SI[0][1] = -S[0][1] * r;
        SI[1][0] = -S[1][0] * r; SI[1][1] = S[0][0] * r;
        logdet = log(fabs(det));
        return det != T(0);
    } else {
        T A[M][M];
        bool ok = true;
        T ld = T(0);
#pragma unroll
        for (int i = 0; i < M; i++)
#pragma unroll
            for (int j = 0; j < M; j++) { A[i][j] = S[i][j]; SI[i][j] = (i == j) ? T(1) : T(0); }
#pragma unroll
        for (int c = 0; c < M; c++) {
            // partial pivoting, as np.linalg.inv (LU, kalman_filter.py:541): the largest |entry| of
            // column c at or below the diagonal is bubbled into row c with predicated row swaps of
            // [A | SI] (row operations on both sides leave SI = S^-1; |det| is unchanged)
            T best = fabs(A[c][c]);
#pragma unroll
            for (int r = c + 1; r < M; r++) {
                const T cand = fabs(A[r][c]);
                const bool sw = cand > best;
                best = sw ? cand : best;
#pragma unroll
                for (int j = 0; j < M; j++) {
                    const T a0 = A[c][j], a1 = A[r][j], s0 = SI[c][j], s1 = SI[r][j];
                    A[c][j] = sw ? a1 : a0; A[r][j] = sw ? a0 : a1;
                    SI[c][j] = sw ? s1 : s0; SI[r][j] = sw ? s0 : s1;
                }
            }
            T piv = A[c][c];
            ok = ok && (piv != T(0));
            ld += log(fabs(piv));
            T d = T(1) / piv;
#pragma unroll
            for (int j = 0; j < M; j++) { A[c][j] *= d; SI[c][j] *= d; }
#pragma unroll
            for (int r = 0; r < M; r++) {
                if (r != c) {
                    T f = A[r][c];
#pragma unroll
                    for (int j = 0; j < M; j++) { A[r][j] -= f * A[c][j]; SI[r][j] -= f * SI[c][j]; }
                }
            }
        }
        logdet = ld;
        return ok;
    }
}

template <typename T, int N, int M>
struct KfUpdateOut {
    T y[M];
    T K[N][M];
    T S[M][M];
    T SI[M][M];
    T logdet;
    bool ok;
};

// RECIP: the one-row block of update_sequential (kalman_filter.py:806-807), K = PH' (1 / S): a zero S gives
// inf, never LinAlgError, so the update runs on (o.ok is still false for a zero S)
template <typename T, int N, int M, bool RECIP = false>
__device__ __forceinline__ void reg_update(T (&x)[N], T (&P)[N][N], const T (&H)[M][N], const T (&R)[M][M],
                                           const T (&z)[M], KfUpdateOut<T, N, M> &o)
{
    static_assert(!RECIP || M == 1, "the reciprocal gain is the one-row block's");
#pragma unroll
    for (int a = 0; a < M; a++) {
        T s = H[a][0] * x[0];
#pragma unroll
        for (int k = 1; k < N; k++) s += H[a][k] * x[k];
        o.y[a] = z[a] - s;
    }
    T PHT[N][M];
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int a = 0; a < M; a++) {
            T s = P[i][0] * H[a][0];
#pragma unroll
            for (int k = 1; k < N; k++) s += P[i][k] * H[a][k];
            PHT[i][a] = s;
        }
#pragma unroll
    for (int a = 0; a < M; a++)
#pragma unroll
        for (int b = 0; b < M; b++) {
            T s = H[a][0] * PHT[0][b];
#pragma unroll
            for (int k = 1; k < N; k++) s += H[a][k] * PHT[k][b];
            o.S[a][b] = s + R[a][b];
        }
    o.ok = reg_inverse<T, M>(o.S, o.SI, o.logdet);
    if (!RECIP && !o.ok) return;      // np.linalg.inv would raise; state stays at the prior
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int a = 0; a < M; a++) {
            T s = PHT[i][0] * o.SI[0][a];
#pragma unroll
            for (int b = 1; b < M; b++) s += PHT[i][b] * o.SI[b][a];
            o.K[i][a] = s;
        }
#pragma unroll
    for (int i = 0; i < N; i++) {
        T s = x[i];
#pragma unroll
        for (int a = 0; a < M; a++) s += o.K[i][a] * o.y[a];
        x[i] = s;
    }
    T IKH[N][N];
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = 0; j < N; j++) {
            T s = (i == j) ? T(1) : T(0);
#pragma unroll
            for (int a = 0; a < M; a++) s -= o.K[i][a] * H[a][j];
            IKH[i][j] = s;
        }
    T T1[N][N];
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = 0; j < N; j++) {
            T s = IKH[i][0] * P[0][j];
#pragma unroll
            for (int k = 1; k < N; k++) s += IKH[i][k] * P[k][j];
            T1[i][j] = s;
        }
    T KR[N][M];
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int b = 0; b < M; b++) {
            T s = o.K[i][0] * R[0][b];
#pragma unroll
            for (int a = 1; a < M; a++) s += o.K[i][a] * R[a][b];
            KR[i][b] = s;
        }
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = 0; j < N; j++) {
            T s = T1[i][0] * IKH[j][0];
#pragma unroll
            for (int k = 1; k < N; k++) s += T1[i][k] * IKH[j][k];
#pragma unroll
            for (int a = 0; a < M; a++) s += KR[i][a] * o.K[j][a];
            P[i][j] = s;
        }
}

// update_correlated (kalman_filter.py:730-748), process noise correlated with the measurement noise by Mc[N][M]:
//   y = z - H x ; PHT = P H' ; S = H PHT + H Mc + Mc' H' + R ; SI = S^-1 ; K = (PHT + Mc) SI ; x = x + K y ;
//   P = P - K (H P + Mc')          (not the Joseph form, and not symmetrised: the reference's arithmetic)
template <typename T, int N, int M>
__device__ __forceinline__ void reg_update_correlated(T (&x)[N], T (&P)[N][N], const T (&H)[M][N], const T (&R)[M][M],
                                                      const T (&Mc)[N][M], const T (&z)[M], KfUpdateOut<T, N, M> &o)
{
#pragma unroll
    for (int a = 0; a < M; a++) {
        T s = H[a][0] * x[0];
#pragma unroll
        for (int k = 1; k < N; k++) s += H[a][k] * x[k];
        o.y[a] = z[a] - s;
    }
    T PHT[N][M], HM[M][M];
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int a = 0; a < M; a++) {
            T s = P[i][0] * H[a][0];
#pragma unroll
            for (int k = 1; k < N; k++) s += P[i][k] * H[a][k];
            PHT[i][a] = s;
        }
#pragma unroll
    for (int a = 0; a < M; a++)
#pragma unroll
        for (int b = 0; b < M; b++) {
            T s = H[a][0] * Mc[0][b];
#pragma unroll
            for (int k = 1; k < N; k++) s += H[a][k] * Mc[k][b];
            HM[a][b] = s;
        }
#pragma unroll
    for (int a = 0; a < M; a++)
#pragma unroll
        for (int b = 0; b < M; b++) {
            T s = H[a][0] * PHT[0][b];
#pragma unroll
            for (int k = 1; k < N; k++) s += H[a][k] * PHT[k][b];
            o.S[a][b] = s + HM[a][b] + HM[b][a] + R[a][b];      // (M' H')[a][b] = (H M)[b][a]
        }
    o.ok = reg_inverse<T, M>(o.S, o.SI, o.logdet);
    if (!o.ok) return;
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int a = 0; a < M; a++) {
            T s = (PHT[i][0] + Mc[i][0]) * o.SI[0][a];
#pragma unroll
            for (int b = 1; b < M; b++) s += (PHT[i][b] + Mc[i][b]) * o.SI[b][a];
            o.K[i][a] = s;
        }
#pragma unroll
    for (int i = 0; i < N; i++) {
        T s = x[i];
#pragma unroll
        for (int a = 0; a < M; a++) s += o.K[i][a] * o.y[a];
        x[i] = s;
    }
    T G[M][N];      // H P + Mc'
#pragma unroll
    for (int a = 0; a < M; a++)
#pragma unroll
        for (int j = 0; j < N; j++) {
            T s = H[a][0] * P[0][j];
#pragma unroll
            for (int k = 1; k < N; k++) s += H[a][k] * P[k][j];
            G[a][j] = s + Mc[j][a];
        }
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = 0; j < N; j++) {
            T s = o.K[i][0] * G[0][j];
#pragma unroll
            for (int a = 1; a < M; a++) s += o.K[i][a] * G[a][j];
            P[i][j] -= s;
        }
}

// ---------------------------------------------------------------------------- structural model words
// reg_predict_pat / reg_update_pat: reg_predict / reg_update for a bank whose models hold structural words,
// +0 (bit pattern 0) or 1 in every filter, named at compile time by PAT:
//   PAT::F0(i), PAT::F1(i)   row i of F: bit k set = F[i][k] is +0 / is 1
//   PAT::H0(a), PAT::H1(a)   row a of H, likewise
//   PAT::Q0(i, j), PAT::R0(a, b)   Q[i][j], R[a][b] is +0
// The structural entries of F, Q, H, R are not read.  For finite inputs whose arithmetic stays finite they
// give the bits of the dense functions as compiled, with the products by a structural word dropped or folded.
//
// The dense chain  s = a0 b0;  s += a1 b1; ...  compiles to FMUL of product 1, FFMA of product 0 onto it, then
// FFMA of products 2, 3, ... in order.  A product a b with a = +0 and b finite is a zero of b's sign, and
// adding a zero changes only the sign of a zero partial sum: fma(+0, b, s) is s, or -0 when s is -0 and b's
// sign bit is set.  So a run of dropped products adds the zero whose sign is the AND of the run's sign bits:
// 0 * w, with w the AND of the run's bit patterns (finite, as every b is).  A run ahead of the first kept
// product is the addend of its FFMA (the FMUL becomes an FFMA); a later run costs one FFMA(0, w, s),
// since a kept product or partial sum may round to -0.  A run of one is the dense FFMA itself.
// A factor 1: 1 b is b, fma(1, b, s) is s + b; a product 1 b ahead of every kept product is b, and the run
// ahead of it is added together with the run after it (b + z1 + z2 = b + (z1 + z2) for any b).

// The product a b of a zero (of either sign) and a finite factor is the zero of sign s_a ^ s_b, and the bit
// pattern a ^ b is then the finite float +-(the other factor) with that sign.  So a run of such products (a
// structural +0 a[k] is the case a ^ b = b) adds the zero 0 w, w = the AND of the run's a ^ b: a finite float
// whose sign is the AND of the products' signs.
template <int L>
__device__ __forceinline__ float and_bits(const float (&a)[L], const float (&b)[L], uint32_t D, uint32_t X)
{
    uint32_t m = ~0u;
#pragma unroll
    for (int k = 0; k < L; k++)
        if ((D >> k) & 1) m &= (X >> k) & 1 ? __float_as_uint(a[k]) ^ __float_as_uint(b[k]) : __float_as_uint(b[k]);
    return __uint_as_float(m);
}

// sum_k a[k] b[k] in the dense chain's order and bits, for a[k] = +0 (bit k of Z) or 1 (bit k of O) in every
// filter.  X (the block path): products known to be zeros, a[k] or b[k] a +-0 data word and the other finite;
// they are dropped like the structural ones, each carrying its sign s_a ^ s_b.  A run of one product is the
// dense instruction itself.  !SIGNED: the caller maps a zero result of either sign to the same value, so the
// zero's sign is not tracked and the dropped products cost nothing.
// (Z, O, X and SIGNED are constants wherever it is inlined: the loop unrolls to the kept instructions)
template <int L>
__device__ __forceinline__ float pat_chain(uint32_t Z, uint32_t O, bool SIGNED, const float (&a)[L], const float (&b)[L],
                                           uint32_t X = 0)
{
    float s = 0.f;
    bool have = false;      // s holds a partial sum
    uint32_t d = 0;         // dropped products not yet added
    // the two factors of the zero a run adds: 0 w, or a single product of X as it stands
    auto ra = [&](uint32_t r) {
        float v = 0.f;
#pragma unroll
        for (int k = 0; k < L; k++)
            if (r == (1u << k) && (X >> k) & 1) v = a[k];
        return v;
    };
    auto rb = [&](uint32_t r) {
        float v = and_bits(a, b, r, X);
#pragma unroll
        for (int k = 0; k < L; k++)
            if (r == (1u << k) && (X >> k) & 1) v = b[k];
        return v;
    };
#pragma unroll
    for (int p = 0; p < L; p++) {
        const int k = L > 1 && p < 2 ? 1 - p : p;       // the product evaluated p-th
        if (((Z | X) >> k) & 1) {
            if (SIGNED) d |= 1u << k;
            continue;
        }
        const bool one = (O >> k) & 1;
        if (!have) {
            have = true;
            if (one) { s = b[k]; continue; }            // d is added with the next run
            s = d ? __fmaf_rn(a[k], b[k], __fmul_rn(ra(d), rb(d))) : __fmul_rn(a[k], b[k]);
            d = 0;
            continue;
        }
        if (d) { s = __fmaf_rn(ra(d), rb(d), s); d = 0; }
        s = one ? __fadd_rn(s, b[k]) : __fmaf_rn(a[k], b[k], s);
    }
    if (d) s = have ? __fmaf_rn(ra(d), rb(d), s) : __fmul_rn(ra(d), rb(d));
    return s;
}

// sum_k a[k] b[k] when every product is a zero (a zero factor, the other finite): the dense chain of zeros
// is -0 exactly when every product is -0, so the sum is the zero whose sign is the AND of the s_a ^ s_b
template <int L>
__device__ __forceinline__ float zero_chain(const float (&a)[L], const float (&b)[L])
{
    uint32_t m = ~0u;
#pragma unroll
    for (int k = 0; k < L; k++) m &= __float_as_uint(a[k]) ^ __float_as_uint(b[k]);
    return __uint_as_float(m & 0x80000000u);
}

template <class PAT, int N>
__device__ __forceinline__ void reg_predict_pat(float (&x)[N], float (&P)[N][N], const float (&F)[N][N],
                                                const float (&Q)[N][N], float alpha_sq)
{
    float xn[N];
#pragma unroll
    for (int i = 0; i < N; i++) xn[i] = pat_chain(PAT::F0(i), PAT::F1(i), true, F[i], x);
    float FP[N][N];
#pragma unroll
    for (int j = 0; j < N; j++) {
        float col[N];
#pragma unroll
        for (int k = 0; k < N; k++) col[k] = P[k][j];
#pragma unroll
        for (int i = 0; i < N; i++) FP[i][j] = pat_chain(PAT::F0(i), PAT::F1(i), true, F[i], col);
    }
    // alpha_sq s + (+0) is +0 for a zero s of either sign: those entries need no sign of s
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = 0; j < N; j++)
            P[i][j] = __fmaf_rn(alpha_sq, pat_chain(PAT::F0(j), PAT::F1(j), !PAT::Q0(i, j), F[j], FP[i]), Q[i][j]);
#pragma unroll
    for (int i = 0; i < N; i++) x[i] = xn[i];
}

// the columns of H whose entries are all structural (any), or all +0 (!any)
template <class PAT, int M>
__host__ __device__ constexpr uint32_t pat_cols(bool any)
{
    uint32_t c = ~0u;
    for (int a = 0; a < M; a++) c &= any ? PAT::H0(a) | PAT::H1(a) : PAT::H0(a);
    return c;
}

// false when S is singular (the state is left at the prior, as reg_update leaves it)
template <class PAT, int N, int M>
__device__ __forceinline__ bool reg_update_pat(float (&x)[N], float (&P)[N][N], const float (&H)[M][N],
                                               const float (&R)[M][M], const float (&z)[M])
{
    float y[M];
#pragma unroll
    for (int a = 0; a < M; a++) y[a] = __fadd_rn(z[a], -pat_chain(PAT::H0(a), PAT::H1(a), true, H[a], x));
    float PHT[N][M];
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int a = 0; a < M; a++) PHT[i][a] = pat_chain(PAT::H0(a), PAT::H1(a), true, H[a], P[i]);
    float S[M][M], SI[M][M], logdet;
#pragma unroll
    for (int b = 0; b < M; b++) {
        float col[N];
#pragma unroll
        for (int k = 0; k < N; k++) col[k] = PHT[k][b];
        // s + (+0) is +0 for a zero s of either sign
#pragma unroll
        for (int a = 0; a < M; a++) S[a][b] = __fadd_rn(pat_chain(PAT::H0(a), PAT::H1(a), !PAT::R0(a, b), H[a], col), R[a][b]);
    }
    if (!reg_inverse<float, M>(S, SI, logdet)) return false;
    float K[N][M];
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int a = 0; a < M; a++) {
            float s = PHT[i][0] * SI[0][a];
#pragma unroll
            for (int b = 1; b < M; b++) s += PHT[i][b] * SI[b][a];
            K[i][a] = s;
        }
#pragma unroll
    for (int i = 0; i < N; i++) {
        float s = x[i];
#pragma unroll
        for (int a = 0; a < M; a++) s += K[i][a] * y[a];
        x[i] = s;
    }
    // IKH = I - K H.  A column j of H whose entries are all structural (HS): IKH[i][j] = delta_ij - K[i][a] over
    // the a with H[a][j] = 1, in order (delta - K is never -0, and nor is a difference of it, so the dropped
    // products change nothing); with none such (HZ), IKH[:, j] is the constant delta_ij, a structural word of T1
    // and P.  A column with any other entry runs the dense chain.
    constexpr uint32_t HS = pat_cols<PAT, M>(true), HZ = pat_cols<PAT, M>(false);
    float IKH[N][N];
#pragma unroll
    for (int j = 0; j < N; j++) {
#pragma unroll
        for (int i = 0; i < N; i++) {
            float s = i == j ? 1.f : 0.f;
            if ((HS >> j) & 1) {
#pragma unroll
                for (int a = 0; a < M; a++)
                    if ((PAT::H1(a) >> j) & 1) s = __fadd_rn(s, -K[i][a]);
            } else {
#pragma unroll
                for (int a = 0; a < M; a++) s = __fmaf_rn(-K[i][a], H[a][j], s);
            }
            IKH[i][j] = s;
        }
    }
    float T1[N][N];
#pragma unroll
    for (int j = 0; j < N; j++) {
        float col[N];
#pragma unroll
        for (int k = 0; k < N; k++) col[k] = P[k][j];
#pragma unroll
        for (int i = 0; i < N; i++) T1[i][j] = pat_chain(HZ & ~(1u << i), HZ & (1u << i), true, IKH[i], col);
    }
    float KR[N][M];
#pragma unroll
    for (int b = 0; b < M; b++) {
        float col[M];
        uint32_t rz = 0;
#pragma unroll
        for (int a = 0; a < M; a++) { col[a] = R[a][b]; rz |= PAT::R0(a, b) ? 1u << a : 0u; }
#pragma unroll
        for (int i = 0; i < N; i++) KR[i][b] = pat_chain(rz, 0u, true, col, K[i]);
    }
    // P = T1 IKH' + KR K', one chain of N + M products per entry
#pragma unroll
    for (int j = 0; j < N; j++) {
        float a[N + M];
#pragma unroll
        for (int k = 0; k < N; k++) a[k] = IKH[j][k];
#pragma unroll
        for (int k = 0; k < M; k++) a[N + k] = K[j][k];
#pragma unroll
        for (int i = 0; i < N; i++) {
            float b[N + M];
#pragma unroll
            for (int k = 0; k < N; k++) b[k] = T1[i][k];
#pragma unroll
            for (int k = 0; k < M; k++) b[N + k] = KR[i][k];
            P[i][j] = pat_chain(HZ & ~(1u << j), HZ & (1u << j), true, a, b);
        }
    }
    return true;
}

// ---------------------------------------------------------------------------- the two axis blocks
// reg_predict_blk / reg_update_blk: reg_predict_pat / reg_update_pat for a PAT whose structural +0 words make F, Q,
// H and R block-diagonal over the index blocks A = {0, 1} and B = {2, 3} (PAT::blocks: the cross words of F and Q
// are +0, row a of H touches block PAT::HB(a) only, the two rows different blocks, and R01 is +0), on a P whose
// cross words (P[i][j], i and j in different blocks) are zeros of either sign.  Under finite arithmetic every
// product that feeds a cross word of any intermediate has a zero factor, so a cross word is a zero whose sign
// zero_chain gives (or a +0 known from the code, below), and a filter leaves the step with zeros in the cross
// words of P again.  Every in-block word runs the operations of reg_*_pat in the same order, the products with a
// cross word dropped into pat_chain's runs (X), and so has the same bits.
__host__ __device__ constexpr bool blk_cross(int i, int j) { return (i >> 1) != (j >> 1); }
// the indices k outside i's block
__host__ __device__ constexpr uint32_t blk_other(int i) { return (i >> 1) ? 3u : 12u; }

template <class PAT, int N>
__device__ __forceinline__ void reg_predict_blk(float (&x)[N], float (&P)[N][N], const float (&F)[N][N],
                                                const float (&Q)[N][N], float alpha_sq)
{
    static_assert(N == 4, "two blocks of two");
    float xn[N];
#pragma unroll
    for (int i = 0; i < N; i++) xn[i] = pat_chain(PAT::F0(i), PAT::F1(i), true, F[i], x);
    // FP = F P: in-block, F[i][k] is +0 wherever P[k][j] is a cross word (structural: the pat chain); cross,
    // F[i][k] P[k][j] is a cross word of P (k in i's block) or of F (k in j's block)
    float FP[N][N];
#pragma unroll
    for (int j = 0; j < N; j++) {
        float col[N];
#pragma unroll
        for (int k = 0; k < N; k++) col[k] = P[k][j];
#pragma unroll
        for (int i = 0; i < N; i++)
            FP[i][j] = blk_cross(i, j) ? zero_chain(F[i], col) : pat_chain(PAT::F0(i), PAT::F1(i), true, F[i], col);
    }
    // cross: alpha_sq (+-0) + Q[i][j] (structural +0) is +0
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = 0; j < N; j++)
            P[i][j] = blk_cross(i, j) ? 0.f
                                      : __fmaf_rn(alpha_sq, pat_chain(PAT::F0(j), PAT::F1(j), !PAT::Q0(i, j), F[j], FP[i]), Q[i][j]);
#pragma unroll
    for (int i = 0; i < N; i++) x[i] = xn[i];
}

// false when S is singular (the state is left at the prior, as reg_update_pat leaves it).  Inlined after
// reg_predict_blk, P's cross words are the constant +0 and the compiler folds what follows from that (PHT's,
// T1's and, for the kf_bank_cv2d pattern, P's cross words come out the constant +0).
template <class PAT, int N, int M>
__device__ __forceinline__ bool reg_update_blk(float (&x)[N], float (&P)[N][N], const float (&H)[M][N],
                                               const float (&R)[M][M], const float (&z)[M])
{
    static_assert(N == 4 && M == 2, "two blocks of two, one measurement row each");
    float y[M];
#pragma unroll
    for (int a = 0; a < M; a++) y[a] = __fadd_rn(z[a], -pat_chain(PAT::H0(a), PAT::H1(a), true, H[a], x));
    // PHT[i][a] is a cross word when i is outside H row a's block: H[a][k] P[i][k] has a cross word of P
    // (k in the row's block) or a structural +0 of H
    auto hx = [](int i, int a) { return (i >> 1) != PAT::HB(a); };
    float PHT[N][M];
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int a = 0; a < M; a++)
            PHT[i][a] = hx(i, a) ? zero_chain(H[a], P[i]) : pat_chain(PAT::H0(a), PAT::H1(a), true, H[a], P[i]);
    // S01, S10: a chain of zeros (H[a][k] PHT[k][b] is a cross word of PHT or a structural +0 of H) plus the
    // structural R01 = +0 is +0
    float S[M][M], SI[M][M], logdet;
#pragma unroll
    for (int b = 0; b < M; b++) {
        float col[N];
#pragma unroll
        for (int k = 0; k < N; k++) col[k] = PHT[k][b];
#pragma unroll
        for (int a = 0; a < M; a++)
            S[a][b] = a != b ? 0.f : __fadd_rn(pat_chain(PAT::H0(a), PAT::H1(a), !PAT::R0(a, b), H[a], col), R[a][b]);
    }
    // (S couples the blocks through det: reg_inverse as reg_update_pat runs it; SI01 = -(+0) r, SI10 likewise)
    if (!reg_inverse<float, M>(S, SI, logdet)) return false;
    // K[i][a] = PHT[i][0] SI[0][a] + PHT[i][1] SI[1][a] (the dense chain's order); the product with b != a has the
    // cross word SI[b][a], and, when i is outside row a's block, the other has the cross word PHT[i][a]
    float K[N][M];
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int a = 0; a < M; a++) {
            const float col[M] = {SI[0][a], SI[1][a]};
            K[i][a] = hx(i, a) ? zero_chain(PHT[i], col) : pat_chain(0u, 0u, true, PHT[i], col, 3u & ~(1u << a));
        }
    // (a cross word of K adds a zero: the dense FFMA, as in reg_update_pat)
#pragma unroll
    for (int i = 0; i < N; i++) {
        float s = x[i];
#pragma unroll
        for (int a = 0; a < M; a++) s += K[i][a] * y[a];
        x[i] = s;
    }
    // IKH = I - K H as in reg_update_pat.  Cross: delta_ij = +0 minus zeros (K[i][a] H[a][j] has the cross word
    // K[i][a] where H[a][j] is not a structural +0) is +0
    constexpr uint32_t HS = pat_cols<PAT, M>(true), HZ = pat_cols<PAT, M>(false);
    float IKH[N][N];
#pragma unroll
    for (int j = 0; j < N; j++) {
#pragma unroll
        for (int i = 0; i < N; i++) {
            float s = i == j ? 1.f : 0.f;
            if (blk_cross(i, j)) {
            } else if ((HS >> j) & 1) {
#pragma unroll
                for (int a = 0; a < M; a++)
                    if ((PAT::H1(a) >> j) & 1) s = __fadd_rn(s, -K[i][a]);
            } else {
#pragma unroll
                for (int a = 0; a < M; a++) s = __fmaf_rn(-K[i][a], H[a][j], s);
            }
            IKH[i][j] = s;
        }
    }
    // T1 = IKH P: IKH[i][k] P[k][j] has a cross word of P (k in i's block) or of IKH
    float T1[N][N];
#pragma unroll
    for (int j = 0; j < N; j++) {
        float col[N];
#pragma unroll
        for (int k = 0; k < N; k++) col[k] = P[k][j];
#pragma unroll
        for (int i = 0; i < N; i++)
            T1[i][j] = blk_cross(i, j) ? zero_chain(IKH[i], col)
                                       : pat_chain(HZ & ~(1u << i), HZ & (1u << i), true, IKH[i], col, blk_other(i) & ~HZ);
    }
    // KR = K R: R[a][b] K[i][a] has the structural R01 = +0 or, when i is outside row b's block, the cross word K[i][b]
    float KR[N][M];
#pragma unroll
    for (int b = 0; b < M; b++) {
        float col[M];
        uint32_t rz = 0;
#pragma unroll
        for (int a = 0; a < M; a++) { col[a] = R[a][b]; rz |= PAT::R0(a, b) ? 1u << a : 0u; }
#pragma unroll
        for (int i = 0; i < N; i++) KR[i][b] = hx(i, b) ? zero_chain(col, K[i]) : pat_chain(rz, 0u, true, col, K[i]);
    }
    // P = T1 IKH' + KR K': T1[i][k] IKH[j][k] has a cross word of IKH (k outside j's block) or of T1 (k outside
    // i's), KR[i][a] K[j][a] one of K (row a's block not j's) or of KR (not i's)
#pragma unroll
    for (int j = 0; j < N; j++) {
        float a[N + M];
#pragma unroll
        for (int k = 0; k < N; k++) a[k] = IKH[j][k];
#pragma unroll
        for (int k = 0; k < M; k++) a[N + k] = K[j][k];
        uint32_t xj = blk_other(j) & ~HZ;
#pragma unroll
        for (int k = 0; k < M; k++) xj |= hx(j, k) ? 1u << (N + k) : 0u;
#pragma unroll
        for (int i = 0; i < N; i++) {
            float b[N + M];
#pragma unroll
            for (int k = 0; k < N; k++) b[k] = T1[i][k];
#pragma unroll
            for (int k = 0; k < M; k++) b[N + k] = KR[i][k];
            P[i][j] = blk_cross(i, j) ? zero_chain(a, b) : pat_chain(HZ & ~(1u << j), HZ & (1u << j), true, a, b, xj);
        }
    }
    return true;
}


}  // namespace bke
