// Warp-per-filter helpers of the catch-all kernels (kf_generic.cu, srkf.cu): one warp owns one filter,
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

}  // namespace bke
