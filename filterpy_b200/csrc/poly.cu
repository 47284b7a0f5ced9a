// poly.cu — banks of polynomial trackers (bke_poly_filter): GHFilter, GHKFilter, GHFilterOrder, LeastSquaresFilter
// and FadingMemoryFilter.  One thread per filter runs all n_steps epochs with the state and the parameters in
// registers: per epoch it reads z[t, f] and writes results[t+1, f, :] / predictions[t, f], coalesced across the warp.
//
// fp64 reproduces the reference bit for bit.  Every expression is evaluated in the reference's operation order with
// explicitly rounded operations (__dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn), which the compiler never contracts
// into an FMA, and every constant the reference derives from its scalars (dt**2, h / dt, the beta powers) arrives
// from the caller, computed with the reference's own expression.  fp32 runs the same sequence in fp32.
#include "bke_internal.cuh"

namespace bke {
namespace {

constexpr int kPolyBlock = 256;

__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dvd(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float dvd(float a, float b) { return __fdiv_rn(a, b); }
// 1 / a, correctly rounded like dvd(1, a), without the division's slow-path call
__device__ __forceinline__ double rcp(double a) { return __drcp_rn(a); }
__device__ __forceinline__ float rcp(float a) { return __frcp_rn(a); }

// Python's int -> float conversion: round to nearest, ties to even
template <typename T> __device__ __forceinline__ T from_int(long long v);
template <> __device__ __forceinline__ double from_int<double>(long long v) { return __ll2double_rn(v); }
template <> __device__ __forceinline__ float from_int<float>(long long v) { return __ll2float_rn(v); }

template <typename T> __device__ __forceinline__ T param(const void *p, int64_t stride, int64_t f)
{
    return p ? static_cast<const T *>(p)[f * stride] : T(0);
}

// the state width of an instance, and the width of its results rows
template <int FAM, int ORD> struct PolyShape {
    static constexpr int state = FAM == BKE_POLY_GH ? 2 : FAM == BKE_POLY_GHK ? 3 : ORD + 1;
    static constexpr int rows = (FAM == BKE_POLY_GH || FAM == BKE_POLY_GHK) ? 2 : ORD + 1;
};

// FAM / ORD / BATCH select the recursion at compile time; GHK's batch_filter runs on the GH instance
template <int FAM, int ORD, bool BATCH, typename T>
__global__ void __launch_bounds__(kPolyBlock) poly_kernel(const bke_poly_args a)
{
    using S = PolyShape<FAM, ORD>;
    const int64_t f = (int64_t)blockIdx.x * kPolyBlock + threadIdx.x;
    const int64_t N = a.n_filters;
    if (f >= N) return;
    constexpr bool GHF = FAM == BKE_POLY_GH || FAM == BKE_POLY_GHK;

    T s[3] = {T(0), T(0), T(0)};
    if (GHF) {
        s[0] = static_cast<const T *>(a.x)[f];
        s[1] = static_cast<const T *>(a.dx)[f];
        if (FAM == BKE_POLY_GHK && !BATCH) s[2] = static_cast<const T *>(a.ddx)[f];
    } else {
#pragma unroll
        for (int j = 0; j < S::state; ++j) s[j] = static_cast<const T *>(a.x)[f * S::state + j];
    }
    const T g = param<T>(a.g, a.g_stride, f), h = param<T>(a.h, a.h_stride, f), k = param<T>(a.k, a.k_stride, f);
    const T dt = param<T>(a.dt, a.dt_stride, f), dt2 = param<T>(a.dt2, a.dt2_stride, f);
    const T hdt2 = param<T>(a.hdt2, a.hdt2_stride, f);
    long long n = FAM == BKE_POLY_LSQ ? (long long)a.n[f] : 0;

    const T *Z = static_cast<const T *>(a.z);
    T *res = static_cast<T *>(a.results);
    T *pred = static_cast<T *>(a.predictions);
    if (res) {
#pragma unroll
        for (int j = 0; j < S::rows; ++j) res[f * S::rows + j] = s[j];
    }
    T y = T(0), xp = T(0), dxp = T(0), ddxp = T(0);
    T K[3] = {T(0), T(0), T(0)};
    const T half = T(0.5), two = T(2);

    for (int64_t t = 0; t < a.n_steps; ++t) {
        const T z = Z[t * N + f];
        const T x = s[0], dx = s[1], ddx = s[2];
        if (FAM == BKE_POLY_GH && BATCH) {
            // gh_filter.py:437-442 (GHKFilter.batch_filter :733-738 is the same recursion: k and ddx are ignored).
            // h arrives as h_dt = h / dt (:433) times the residual, where update() rounds h * y / dt (:374)
            const T x_est = add(x, mul(dx, dt));
            const T r = sub(z, x_est);
            s[1] = add(dx, mul(h, r));
            s[0] = add(x_est, mul(g, r));
            if (pred) pred[t * N + f] = x_est;
        } else if (FAM == BKE_POLY_GH) {
            // gh_filter.py:369-375
            dxp = dx;
            xp = add(x, mul(dx, dt));
            y = sub(z, xp);
            s[1] = add(dxp, dvd(mul(h, y), dt));
            s[0] = add(xp, mul(g, y));
        } else if (FAM == BKE_POLY_GHK) {
            // gh_filter.py:667-678; dt2 = dt**2 (:667)
            ddxp = ddx;
            dxp = add(dx, mul(ddx, dt));
            xp = add(add(x, mul(dx, dt)), mul(mul(half, ddx), dt2));
            y = sub(z, xp);
            s[2] = add(ddxp, dvd(mul(mul(two, k), y), dt2));
            s[1] = add(dxp, dvd(mul(h, y), dt));
            s[0] = add(xp, mul(g, y));
        } else if (FAM == BKE_POLY_GH_ORDER) {
            if (ORD == 0) {                                          // gh_filter.py:145-146
                y = sub(z, x);
                s[0] = add(x, mul(g, y));
            } else if (ORD == 1) {                                   // :153-159 (z is stored for order 1 only, :161)
                const T dxdt = mul(dx, dt);
                y = sub(z, add(x, dxdt));
                s[0] = add(add(x, dxdt), mul(g, y));
                s[1] = add(dx, dvd(mul(h, y), dt));
            } else {                                                 // :171-181; dt2 = dt**2. (:175) = dt**2 (:181)
                const T dxdt = mul(dx, dt);
                const T p = add(add(x, dxdt), mul(mul(half, ddx), dt2));
                y = sub(z, p);
                s[0] = add(p, mul(g, y));
                s[1] = add(add(dx, mul(ddx, dt)), dvd(mul(h, y), dt));
                s[2] = add(ddx, dvd(mul(mul(two, k), y), dt2));
            }
        } else if (FAM == BKE_POLY_LSQ) {
            // least_squares.py:122-154.  The gains come from the int64 counter as Python computes them: exact integer
            // products, one round-to-nearest conversion where an int meets a float, then the float operations.
            // The residual is a local (:132, :139, :150): self.y is never written.
            n += 1;
            if (ORD == 0) {
                // :131-133: y = z - x is the whole (one-element) vector and x[0] takes K[0] * y from it
                K[0] = rcp(from_int<T>(n));                 // 1. / n
                const T r = sub(z, x);
                s[0] = add(x, mul(K[0], r));
            } else if (ORD == 1) {
                const long long nn1 = n * (n + 1);
                K[0] = dvd(mul(two, from_int<T>(2 * n - 1)), from_int<T>(nn1));          // :136
                K[1] = dvd(T(6), mul(from_int<T>(nn1), dt));                            // :137
                const T r = sub(sub(z, x), mul(dt, dx));                                // :139
                s[0] = add(x, add(mul(K[0], r), mul(dt, dx)));                          // :141
                s[1] = add(dx, mul(K[1], r));                                           // :142
            } else {
                const long long den = n * (n + 1) * (n + 2);                            // :145
                K[0] = dvd(mul(T(3), from_int<T>(3 * n * n - 3 * n + 2)), from_int<T>(den));
                K[1] = dvd(mul(T(18), from_int<T>(2 * n - 1)), mul(from_int<T>(den), dt));
                K[2] = dvd(T(60), mul(from_int<T>(den), dt2));                          // :148, dt2 = dt**2
                // :150-154, hdt2 = 0.5 * dt**2
                const T r = sub(sub(sub(z, x), mul(dt, dx)), mul(hdt2, ddx));
                s[0] = add(x, add(add(mul(K[0], r), mul(dx, dt)), mul(hdt2, ddx)));
                s[1] = add(dx, add(mul(K[1], r), mul(ddx, dt)));
                s[2] = add(ddx, mul(K[2], r));
            }
        } else {
            // fading_memory.py:164-194: G, H and K depend on the order (g = G, h = H / dt, k = 2*K / dt**2)
            if (ORD == 0) {
                s[0] = add(x, mul(g, sub(z, x)));                                       // :165-166
            } else if (ORD == 1) {
                const T dxdt = mul(dx, dt);                                             // :173-177
                const T r = sub(z, add(x, dxdt));
                s[0] = add(add(x, dxdt), mul(g, r));
                s[1] = add(dx, mul(h, r));
            } else {
                const T dxdt = mul(dx, dt);                                             // :187-194, dt2 = dt**2.
                const T p = add(add(x, dxdt), mul(mul(half, ddx), dt2));
                const T r = sub(z, p);
                s[0] = add(p, mul(g, r));
                s[1] = add(add(dx, mul(ddx, dt)), mul(h, r));
                s[2] = add(ddx, mul(k, r));
            }
        }
        if (res) {
            T *row = res + ((t + 1) * N + f) * S::rows;
#pragma unroll
            for (int j = 0; j < S::rows; ++j) row[j] = s[j];
        }
    }

    if (BATCH || a.mode == BKE_POLY_BATCH) return;               // batch_filter modifies no member (:385-391)
    if (GHF) {
        static_cast<T *>(a.x)[f] = s[0];
        static_cast<T *>(a.dx)[f] = s[1];
        if (FAM == BKE_POLY_GHK) static_cast<T *>(a.ddx)[f] = s[2];
        if (a.x_prediction) static_cast<T *>(a.x_prediction)[f] = xp;
        if (a.dx_prediction) static_cast<T *>(a.dx_prediction)[f] = dxp;
        if (FAM == BKE_POLY_GHK && a.ddx_prediction) static_cast<T *>(a.ddx_prediction)[f] = ddxp;
    } else {
#pragma unroll
        for (int j = 0; j < S::state; ++j) static_cast<T *>(a.x)[f * S::state + j] = s[j];
    }
    if (a.y && FAM != BKE_POLY_LSQ && FAM != BKE_POLY_FADING) static_cast<T *>(a.y)[f] = y;
    if (FAM == BKE_POLY_LSQ) {
        a.n[f] = n;
        if (a.K) {
#pragma unroll
            for (int j = 0; j < S::state; ++j) static_cast<T *>(a.K)[f * S::state + j] = K[j];
        }
    }
}

template <int FAM, int ORD, bool BATCH, typename T>
int launch_one(const bke_poly_args &a, cudaStream_t s)
{
    const unsigned grid = (unsigned)((a.n_filters + kPolyBlock - 1) / kPolyBlock);
    bke_poly_args p = a;
    return launch_kernel((const void *)poly_kernel<FAM, ORD, BATCH, T>, grid, kPolyBlock, 0, &p, s, "poly_kernel");
}

template <typename T>
int launch_typed(const bke_poly_args &a, cudaStream_t s)
{
    const bool batch = a.mode == BKE_POLY_BATCH;
    switch (a.family) {
    case BKE_POLY_GH:
    case BKE_POLY_GHK:
        if (batch) return launch_one<BKE_POLY_GH, 1, true, T>(a, s);
        return a.family == BKE_POLY_GH ? launch_one<BKE_POLY_GH, 1, false, T>(a, s) : launch_one<BKE_POLY_GHK, 2, false, T>(a, s);
    case BKE_POLY_GH_ORDER:
        return a.order == 0 ? launch_one<BKE_POLY_GH_ORDER, 0, false, T>(a, s)
             : a.order == 1 ? launch_one<BKE_POLY_GH_ORDER, 1, false, T>(a, s) : launch_one<BKE_POLY_GH_ORDER, 2, false, T>(a, s);
    case BKE_POLY_LSQ:
        return a.order == 0 ? launch_one<BKE_POLY_LSQ, 0, false, T>(a, s)
             : a.order == 1 ? launch_one<BKE_POLY_LSQ, 1, false, T>(a, s) : launch_one<BKE_POLY_LSQ, 2, false, T>(a, s);
    default:
        return a.order == 0 ? launch_one<BKE_POLY_FADING, 0, false, T>(a, s)
             : a.order == 1 ? launch_one<BKE_POLY_FADING, 1, false, T>(a, s) : launch_one<BKE_POLY_FADING, 2, false, T>(a, s);
    }
}

}  // namespace

int launch_poly(const bke_poly_args &a, cudaStream_t s)
{
    return a.dtype == BKE_F64 ? launch_typed<double>(a, s) : launch_typed<float>(a, s);
}

}  // namespace bke
