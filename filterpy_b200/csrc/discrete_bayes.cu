// discrete_bayes.cu — banks of 1-D discrete Bayes (histogram) filters: predict, update and normalize
// (filterpy/discrete_bayes/discrete_bayes.py) of every row of pdf[B, M] in one call, bit for bit per row.
//
// What the reference computes, per row:
//   predict   wrap:      convolve(np.roll(pdf, offset), kernel, mode='wrap')
//             constant:  convolve(shift(pdf, offset, cval=cval), kernel, mode='constant', cval=cval)
//             scipy's convolve is a correlation with the reversed kernel kr = kernel[::-1], its window
//             starting c = (K - 1) // 2 bins left of the output bin (the origin rule that moves an even
//             kernel's window by one), summed in fp64 in window order from 0.0, one __dmul_rn and one
//             __dadd_rn per term.  scipy drops every weight with |w| <= DBL_EPSILON (NaN included) from the
//             footprint, so those terms are skipped, not added as x * 0.  The result is rounded once to the
//             pdf's dtype.  For an integer offset, shift equals the exact shift up to its spline's roundoff:
//             bins shifted in hold (T)cval, bins outside the row hold cval.
//   update    prior * likelihood in the dtype, then normalize.
//   normalize pdf /= sum(np.asarray(pdf, dtype=float)): the builtin sum, 0 + p0 + p1 + ... in fp64, and an
//             fp64 division rounded once to the dtype.
//
// Two paths, chosen from M and the dtype:
//   single pass  rows whose pdf and posterior fit in one CTA's shared memory (2 M sizeof(T) <= 226 KB): one
//                CTA per row stages the pdf with coalesced loads, its threads form several bins each, and one
//                warp walks the sequential sum, fed 32 bins at a time by a shuffle.  out may be pdf: the row is
//                staged before anything is written.
//   multi-pass   longer rows, one at a time: a parallel predict x likelihood pass into an fp64 workspace row,
//                the exact sequential sum of that row by the parity-map scan of bke_cumsum_exact
//                (cumsum_exact in resample.cu), and a scale pass into out.
#include <float.h>

#include "bke_internal.cuh"

namespace bke {
namespace db {

typedef long long i64;

constexpr int NT = 128;                          // threads per CTA of both paths
constexpr size_t STAGE_BYTES = 226 * 1024;       // sm_90's 227 KB of opt-in shared memory per CTA, less the static

struct Row {
    const double *kr;    // the kernel of the row (read reversed), or NULL: no predict
    i64 K, off;          // wrap: off in [0, M); constant: off clamped to [-M, M]
};

template <typename T>
struct Params {
    i64 B, M;
    const T *pdf;
    const T *lik;
    T *out;
    const double *kernel;
    i64 K, kernel_stride;
    const i64 *offsets;
    i64 offset;
    double cval;
    int wrap, normalize;
    double *sums;
};

template <typename T>
__device__ __forceinline__ Row row_of(const Params<T> &p, i64 b)
{
    Row r;
    r.kr = p.kernel ? p.kernel + b * p.kernel_stride : nullptr;
    r.K = p.K;
    const i64 o = p.offsets ? p.offsets[b] : p.offset;
    if (p.wrap) r.off = ((o % p.M) + p.M) % p.M;
    else r.off = o > p.M ? p.M : o < -p.M ? -p.M : o;
    return r;
}

template <typename T> __device__ __forceinline__ T mul_rn(T a, T b);
template <> __device__ __forceinline__ float mul_rn<float>(float a, float b) { return __fmul_rn(a, b); }
template <> __device__ __forceinline__ double mul_rn<double>(double a, double b) { return __dmul_rn(a, b); }
template <typename T> __device__ __forceinline__ T to_t(double v);
template <> __device__ __forceinline__ float to_t<float>(double v) { return __double2float_rn(v); }
template <> __device__ __forceinline__ double to_t<double>(double v) { return v; }

// the prior of bin i: the reference's correlation over the rolled (wrap) or shifted (constant) row `src`
template <typename T, bool WRAP>
__device__ __forceinline__ T prior_at(const T *src, i64 i, i64 M, const Row &r, double cval)
{
    const i64 c = (r.K - 1) / 2;
    double acc = 0.0;
    if (WRAP) {
        i64 q = ((i - c - r.off) % M + M) % M;                   // rolled[i + j - c] = pdf[(i + j - c - off) mod M]
        for (i64 j = 0; j < r.K; j++) {
            const double w = r.kr[r.K - 1 - j];
            if (fabs(w) > DBL_EPSILON) acc = __dadd_rn(acc, __dmul_rn((double)src[q], w));
            if (++q == M) q = 0;
        }
    } else {
        const T fill = (T)cval;
        for (i64 j = 0; j < r.K; j++) {
            const double w = r.kr[r.K - 1 - j];
            if (!(fabs(w) > DBL_EPSILON)) continue;
            const i64 q = i + j - c, s = q - r.off;
            const double x = (q < 0 || q >= M) ? cval : (s < 0 || s >= M) ? (double)fill : (double)src[s];
            acc = __dadd_rn(acc, __dmul_rn(x, w));
        }
    }
    return to_t<T>(acc);
}

// prior (predicted or the pdf itself) times the likelihood when there is one
template <typename T, bool WRAP>
__device__ __forceinline__ T posterior_at(const Params<T> &p, const T *src, const T *lik_row, i64 i, const Row &r)
{
    const T prior = r.kr ? prior_at<T, WRAP>(src, i, p.M, r, p.cval) : src[i];
    return lik_row ? mul_rn<T>(prior, lik_row[i]) : prior;
}

// ---------------------------------------------------------------------- single pass: one CTA per row
template <typename T, bool WRAP>
__global__ void __launch_bounds__(NT) k_db_row(Params<T> p)
{
    extern __shared__ double stage_raw[];
    T *s_pdf = reinterpret_cast<T *>(stage_raw);
    T *s_post = s_pdf + p.M;
    __shared__ double s_sum;
    const i64 b = blockIdx.x, M = p.M;
    const T *src = p.pdf + b * M;
    for (i64 i = threadIdx.x; i < M; i += NT) s_pdf[i] = src[i];
    __syncthreads();                                             // out may be pdf: every read precedes every write
    const Row r = row_of(p, b);
    const T *lik = p.lik ? p.lik + b * M : nullptr;
    T *dst = p.out + b * M;
    for (i64 i = threadIdx.x; i < M; i += NT) {
        const T v = posterior_at<T, WRAP>(p, s_pdf, lik, i, r);
        if (p.normalize) s_post[i] = v; else dst[i] = v;
    }
    if (!p.normalize) return;
    __syncthreads();
    if (threadIdx.x < 32) {                                      // the builtin sum: 0 + p0 + p1 + ..., one add per bin
        const int lane = threadIdx.x;
        double acc = 0.0;
        for (i64 j0 = 0; j0 < M; j0 += 32) {
            const double v = j0 + lane < M ? (double)s_post[j0 + lane] : 0.0;
            if (M - j0 >= 32) {
#pragma unroll
                for (int t = 0; t < 32; t++) acc = __dadd_rn(acc, __shfl_sync(FULL, v, t));
            } else {
                for (int t = 0; t < (int)(M - j0); t++) acc = __dadd_rn(acc, __shfl_sync(FULL, v, t));
            }
        }
        if (lane == 0) {
            s_sum = acc;
            if (p.sums) p.sums[b] = acc;
        }
    }
    __syncthreads();
    const double s = s_sum;
    for (i64 i = threadIdx.x; i < M; i += NT) dst[i] = to_t<T>(__ddiv_rn((double)s_post[i], s));
}

// ---------------------------------------------------------------------- multi-pass: one row at a time
template <typename T, bool WRAP>
__global__ void __launch_bounds__(NT) k_db_posterior(Params<T> p, i64 b, double *post)
{
    const i64 M = p.M;
    const Row r = row_of(p, b);
    const T *src = p.pdf + b * M;
    const T *lik = p.lik ? p.lik + b * M : nullptr;
    for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < M; i += (i64)gridDim.x * NT)
        post[i] = (double)posterior_at<T, WRAP>(p, src, lik, i, r);
}

// out[b] = post / (0 + S) (or post itself without normalize); S is np.cumsum's last element, which differs from the
// builtin sum's 0 + ... only for an all -0.0 row
template <typename T>
__global__ void __launch_bounds__(NT) k_db_scale(Params<T> p, i64 b, const double *post, const double *total)
{
    const i64 M = p.M;
    T *dst = p.out + b * M;
    if (!p.normalize) {
        for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < M; i += (i64)gridDim.x * NT) dst[i] = (T)post[i];
        return;
    }
    const double s = __dadd_rn(0.0, *total);
    if (p.sums && blockIdx.x == 0 && threadIdx.x == 0) p.sums[b] = s;
    for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < M; i += (i64)gridDim.x * NT)
        dst[i] = to_t<T>(__ddiv_rn(post[i], s));
}

static size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

bool single_pass(int64_t M, int32_t dtype) { return 2 * (uint64_t)M * (dtype == BKE_F32 ? 4 : 8) <= STAGE_BYTES; }

// multi-pass workspace: the posterior row, np.cumsum's scratch row, the row's sum, then the scan's own workspace
size_t workspace_bytes(int64_t M, int32_t dtype)
{
    if (M <= 0 || single_pass(M, dtype)) return 0;
    return 2 * align256((size_t)M * 8) + 256 + cumsum_workspace_bytes(M);
}

template <typename T>
int launch(const bke_db_args &a, cudaStream_t s)
{
    Params<T> p;
    p.B = a.n_rows; p.M = a.n_bins;
    p.pdf = (const T *)a.pdf; p.lik = (const T *)a.likelihood; p.out = (T *)a.out;
    p.kernel = a.kernel; p.K = a.kernel_len; p.kernel_stride = a.kernel_stride;
    p.offsets = (const i64 *)a.offsets; p.offset = a.offset; p.cval = a.cval;
    p.wrap = !(a.flags & BKE_DB_CONSTANT); p.normalize = (a.flags & BKE_DB_NORMALIZE) != 0;
    p.sums = a.sums;
    if (single_pass(a.n_bins, a.dtype)) {
        const size_t smem = 2 * (size_t)a.n_bins * sizeof(T);
        const void *kern = p.wrap ? (const void *)k_db_row<T, true> : (const void *)k_db_row<T, false>;
        return launch_kernel(kern, (unsigned)a.n_rows, NT, smem, &p, s, "discrete Bayes row launch");
    }
    unsigned char *ws = (unsigned char *)a.workspace;
    double *post = (double *)ws;
    double *scratch = (double *)(ws + align256((size_t)a.n_bins * 8));
    double *total = (double *)(ws + 2 * align256((size_t)a.n_bins * 8));
    void *scan_ws = ws + 2 * align256((size_t)a.n_bins * 8) + 256;
    const size_t scan_bytes = a.workspace_bytes - (2 * align256((size_t)a.n_bins * 8) + 256);
    const i64 want = (a.n_bins + NT * 8 - 1) / (NT * 8), cap = (i64)sm_count() * 16;
    const unsigned grid = (unsigned)(want < cap ? want : cap);
    for (i64 b = 0; b < a.n_rows; b++) {
        if (p.wrap) k_db_posterior<T, true><<<grid, NT, 0, s>>>(p, b, post);
        else k_db_posterior<T, false><<<grid, NT, 0, s>>>(p, b, post);
        if (check_cuda(cudaGetLastError(), "discrete Bayes posterior launch")) return BKE_ERR_CUDA;
        if (p.normalize) {
            const int rc = cumsum_exact(a.n_bins, post, scratch, 0, total, scan_ws, scan_bytes, nullptr, s);
            if (rc != BKE_OK) return rc;
        }
        k_db_scale<T><<<grid, NT, 0, s>>>(p, b, post, total);
        if (check_cuda(cudaGetLastError(), "discrete Bayes scale launch")) return BKE_ERR_CUDA;
    }
    return BKE_OK;
}

}  // namespace db

int launch_db(const bke_db_args &a, cudaStream_t s)
{
    return a.dtype == BKE_F32 ? db::launch<float>(a, s) : db::launch<double>(a, s);
}

size_t db_workspace_bytes(int64_t n_bins, int32_t dtype) { return db::workspace_bytes(n_bins, dtype); }

}  // namespace bke
