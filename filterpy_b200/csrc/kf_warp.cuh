// Warp-per-filter helpers of the catch-all kernels (kf_generic.cu, srkf.cu, information.cu): one warp owns one filter,
// its matrices sit in the warp's slice of shared memory, the 32 lanes split the work and synchronise
// with __syncwarp() only.
#pragma once
#include "bke_internal.cuh"

namespace bke {

// C[r,c] = A[r,k] * B (B is [k,c], or [c,k] when TB), result handed to epi(e, i, j, value)
template <bool TB, typename T, typename Epi>
__device__ __forceinline__ void warp_mm(const T *A, const T *B, int r, int k, int c, int lane, Epi epi)
{
    for (int e = lane; e < r * c; e += 32) {
        int i = e / c, j = e - i * c;
        T s = T(0);
        for (int q = 0; q < k; q++) s += A[i * k + q] * (TB ? B[j * k + q] : B[q * c + j]);
        epi(e, i, j, s);
    }
}

template <typename T>
__device__ __forceinline__ void warp_copy_in(T *dst, const T *src, int cnt, int lane)
{
    for (int e = lane; e < cnt; e += 32) dst[e] = src[e];
}

// sum of v over the warp, returned to every lane
template <typename T>
__device__ __forceinline__ T warp_sum(T v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}

// Gauss-Jordan inverse with partial pivoting of the m x m matrix A (destroyed) into Ai.
// Returns false when a pivot is exactly zero (np.linalg.inv raises LinAlgError).
// logdet receives log|det A|.
template <typename T>
__device__ bool warp_inverse(T *A, T *Ai, T *col, int m, int lane, T &logdet)
{
    for (int e = lane; e < m * m; e += 32) Ai[e] = (e / m == e % m) ? T(1) : T(0);
    __syncwarp();
    T ld = T(0);
    for (int c = 0; c < m; c++) {
        // pivot search (every lane scans; m is tiny)
        int p = c;
        T best = fabs(A[c * m + c]);
        for (int r = c + 1; r < m; r++) {
            T v = fabs(A[r * m + c]);
            if (v > best) { best = v; p = r; }
        }
        if (!(best > T(0))) return false;
        __syncwarp();
        if (p != c) {
            for (int j = lane; j < m; j += 32) {
                T t = A[c * m + j]; A[c * m + j] = A[p * m + j]; A[p * m + j] = t;
                t = Ai[c * m + j]; Ai[c * m + j] = Ai[p * m + j]; Ai[p * m + j] = t;
            }
            __syncwarp();
        }
        T piv = A[c * m + c];
        ld += log(fabs(piv));
        T d = T(1) / piv;
        __syncwarp();
        for (int j = lane; j < m; j += 32) { A[c * m + j] *= d; Ai[c * m + j] *= d; }
        for (int r = lane; r < m; r += 32) col[r] = A[r * m + c];
        __syncwarp();
        for (int e = lane; e < m * m; e += 32) {
            int r = e / m, j = e - r * m;
            if (r != c) {
                T f = col[r];
                A[e] -= f * A[c * m + j];
                Ai[e] -= f * Ai[c * m + j];
            }
        }
        __syncwarp();
    }
    logdet = ld;
    return true;
}

}  // namespace bke
