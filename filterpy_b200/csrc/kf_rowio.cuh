// Thread-per-filter row loads and stores of the register-tile kernels: every thread reads its own rows
// of the AoS arrays with 16-byte accesses when a row is a whole number of 16-byte vectors, so every
// fetched sector is used.
#pragma once
#include <type_traits>
#include "bke_internal.cuh"

namespace bke {

template <typename T, int CNT>
__device__ __forceinline__ void ldv(T *dst, const T *src)
{
    constexpr int VEC = 16 / sizeof(T);
    if constexpr (CNT % VEC == 0) {
        using V = typename std::conditional<sizeof(T) == 4, float4, double2>::type;
#pragma unroll
        for (int i = 0; i < CNT / VEC; i++) *reinterpret_cast<V *>(dst + i * VEC) = __ldg(reinterpret_cast<const V *>(src) + i);
    } else {
#pragma unroll
        for (int i = 0; i < CNT; i++) dst[i] = __ldg(src + i);
    }
}
// plain (coherent) loads: for x and P, which alias x_out / P_out in the in-place call — ld.global.nc
// requires memory that nobody writes during the kernel
template <typename T, int CNT>
__device__ __forceinline__ void ldv_rw(T *dst, const T *src)
{
    constexpr int VEC = 16 / sizeof(T);
    if constexpr (CNT % VEC == 0) {
        using V = typename std::conditional<sizeof(T) == 4, float4, double2>::type;
#pragma unroll
        for (int i = 0; i < CNT / VEC; i++) *reinterpret_cast<V *>(dst + i * VEC) = reinterpret_cast<const V *>(src)[i];
    } else {
#pragma unroll
        for (int i = 0; i < CNT; i++) dst[i] = src[i];
    }
}
template <typename T, int CNT>
__device__ __forceinline__ void stv(T *dst, const T *src)
{
    constexpr int VEC = 16 / sizeof(T);
    if constexpr (CNT % VEC == 0) {
        using V = typename std::conditional<sizeof(T) == 4, float4, double2>::type;
#pragma unroll
        for (int i = 0; i < CNT / VEC; i++) reinterpret_cast<V *>(dst)[i] = *reinterpret_cast<const V *>(src + i * VEC);
    } else {
#pragma unroll
        for (int i = 0; i < CNT; i++) dst[i] = src[i];
    }
}

// element by element, for rows with no 16-byte alignment guarantee
template <typename T, int CNT>
__device__ __forceinline__ void ld_scalar(T *dst, const T *src)
{
#pragma unroll
    for (int i = 0; i < CNT; i++) dst[i] = src[i];
}
template <typename T, int CNT>
__device__ __forceinline__ void st_scalar(T *dst, const T *src)
{
#pragma unroll
    for (int i = 0; i < CNT; i++) dst[i] = src[i];
}

// 16-byte vector accesses are used for the arrays whose row is a multiple of 16 bytes: their base
// pointers and per-filter strides must be 16-byte aligned (otherwise the catch-all kernel runs)
template <typename T, int CNT>
bool vec_ok(const void *p, int64_t stride_elems = CNT)
{
    constexpr int VEC = 16 / sizeof(T);
    if (CNT % VEC != 0 || p == nullptr) return true;
    return (reinterpret_cast<uintptr_t>(p) & 15u) == 0 && (stride_elems * (int64_t)sizeof(T)) % 16 == 0;
}

}  // namespace bke
