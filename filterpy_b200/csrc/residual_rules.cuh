// residual_rules.cuh — the per-element rules of residual_resample (filterpy/monte_carlo/resampling.py:57-69)
// and NumPy's ordering of doubles in searchsorted, shared by the single-set path (csrc/residual.cu) and the
// bank path (csrc/resample_bank.cu).
#pragma once
#include "bke_internal.cuh"

namespace bke {
namespace rr {

typedef long long i64;

// resampling.py:57 — floor(N * w).astype(int) (N * w is one fp64 multiply of float(N) and w).  NumPy's
// float -> int64 cast is the x86-64 conversion, which yields INT64_MIN for NaN and for every value outside
// [-2^63, 2^63) (+inf included); __double2ll_rz would saturate +inf and huge values to INT64_MAX instead.
__device__ __forceinline__ i64 num_copies(double Nd, double w)
{
    const double f = floor(__dmul_rn(Nd, w));
    return f < 9223372036854775808.0 ? __double2ll_rz(f) : (i64)0x8000000000000000ULL;
}
// resampling.py:69 — w - num_copies (int64 -> fp64 is exact below 2^53)
__device__ __forceinline__ double residual_of(double Nd, double w) { return __dsub_rn(w, (double)num_copies(Nd, w)); }
// range(num_copies[i]) is empty for a negative count (resampling.py:60)
__device__ __forceinline__ i64 copies_made(double Nd, double w) { const i64 c = num_copies(Nd, w); return c > 0 ? c : 0; }

// NumPy's ordering of doubles in searchsorted (NaN sorts last): npy_sort.h DOUBLE_LT
__device__ __forceinline__ bool np_lt(double a, double b) { return a < b || (b != b && a == a); }

}  // namespace rr
}  // namespace bke
