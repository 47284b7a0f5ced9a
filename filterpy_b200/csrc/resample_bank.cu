// resample_bank.cu — systematic / stratified resampling of a BANK of particle sets in one launch:
// row b of weights[B, M] is one set, resampled exactly as the reference resamples one weight vector
// (filterpy/monte_carlo/resampling.py:117-150 systematic, :80-114 stratified).
//
// With B independent sets the parallelism comes from the sets, so each set can run the reference's
// own arithmetic literally: one thread per set forms the strictly sequential fp64 cumsum (:142,
// c_0 = w_0, c_j = fl(c_{j-1} + w_j)) and walks the two-pointer merge of :144-149
//
//     while i < M:  if pos_i < c_j: indexes[i] = j; i += 1   else: j += 1   (j == M: IndexError, :145)
//
// with pos_i = fl(fl(u + i) / M) (:139) or fl(fl(U_i + i) / M) (:103).  That is the reference for
// every input — negative, NaN, infinite, signed-zero and subnormal weights, uniforms outside [0, 1)
// or out of order — with no verification pass and no fallback.
//
// A thread walking its own row would load and store uncoalesced (rows are M elements apart), so
// each CTA stages a window of COLS elements of every one of its ROWS sets in shared memory: the
// weights at the merge's j, the positions and the output indexes at its i.  The CTA alternates
//   run    every set advances its merge until it leaves its weight window or fills its output window;
//   move   a warp per set moves 32 consecutive elements: it writes back a full (or final) output
//          window, loads the next weight window, and loads the next uniforms and forms the positions
//          (so the fp64 divisions run in parallel over the window, off the sequential path).
// Each round consumes at least one window per unfinished set, so a set of M particles finishes in at
// most 2M / COLS + 1 rounds.  Global traffic: weights (and uniforms) read once, indexes written once,
// all as 256-byte / 128-byte row segments.
#include "bke_internal.cuh"

namespace bke {
namespace rsb {

typedef long long i64;

constexpr int ROWS = 64;        // sets per CTA, one thread each
constexpr int COLS = 32;        // elements of one set per window (one warp-wide segment)
constexpr int PAD = COLS + 1;   // row pitch in shared memory: consecutive sets start in different banks

struct Shared {
    double w[ROWS][PAD];        // weights[kj .. kj + COLS) of each set
    double pos[ROWS][PAD];      // positions[ki .. ki + COLS)
    int out[ROWS][PAD];         // indexes[ki .. ki + COLS), written back when full or final
    int kj[ROWS], ki[ROWS];     // window bases to load in the next move, in units of COLS
    int fbase[ROWS];            // output window to write back, in units of COLS
    double u[ROWS];             // systematic offset of each set
    int nflush[ROWS];           // outputs to write back (0: none)
    int load_w[ROWS], load_p[ROWS];
};

template <bool STRAT>
__global__ void __launch_bounds__(ROWS) k_resample_bank(i64 n_sets, i64 M, const double *__restrict__ w,
                                                        const double *__restrict__ u, const double *__restrict__ U,
                                                        int *__restrict__ idx, int *__restrict__ status)
{
    __shared__ Shared sh;
    const int r = threadIdx.x;
    const i64 b0 = (i64)blockIdx.x * ROWS;
    const i64 rem = n_sets - b0;
    const int rows = rem < ROWS ? (int)rem : ROWS;
    const double Md = (double)M;

    bool active = r < rows;
    i64 ki = 0, kj = 0;             // window bases of this thread's set
    int ii = 0, jj = 0;             // merge pointers within the windows: i = ki + ii, j = kj + jj
    double c = 0.0;                 // cumsum(w)[j]
    bool fresh_w = true;            // the weight window was just loaded: c still lacks w[kj]
    sh.kj[r] = 0; sh.ki[r] = 0; sh.fbase[r] = 0; sh.nflush[r] = 0;
    sh.load_w[r] = active; sh.load_p[r] = active;
    sh.u[r] = (!STRAT && active) ? u[b0 + r] : 0.0;
    bool more = active;

    while (__syncthreads_or(more)) {
        // ---- move: a warp per set, a lane per column
#pragma unroll 4
        for (int e = r; e < ROWS * COLS; e += ROWS) {
            const int q = e / COLS, t = e % COLS;
            const i64 row = (b0 + q) * M;
            if (t < sh.nflush[q]) idx[row + (i64)sh.fbase[q] * COLS + t] = sh.out[q][t];
            if (sh.load_w[q]) {
                const i64 k = (i64)sh.kj[q] * COLS + t;
                if (k < M) sh.w[q][t] = __ldg(w + row + k);
            }
            if (sh.load_p[q]) {
                const i64 k = (i64)sh.ki[q] * COLS + t;
                if (k < M) {
                    const double a = STRAT ? __ldg(U + row + k) : sh.u[q];
                    sh.pos[q][t] = __ddiv_rn(__dadd_rn(a, (double)k), Md);       // resampling.py:139 / :103
                }
            }
        }
        __syncthreads();

        // ---- run: the reference's merge until a window is used up
        int nflush = 0, need_w = 0, need_p = 0;
        const i64 fbase = ki;
        if (active) {
            if (fresh_w) {                                   // np.cumsum: c_0 = w_0, then one add per element
                c = (kj == 0) ? sh.w[r][0] : __dadd_rn(c, sh.w[r][0]);
                fresh_w = false;
            }
            const int ilim = (M - ki) < COLS ? (int)(M - ki) : COLS;
            const int jlim = (M - kj) < COLS ? (int)(M - kj) : COLS;
            const int jbase = (int)kj;
            for (;;) {
                if (sh.pos[r][ii] < c) {                      // :146
                    sh.out[r][ii] = jbase + jj;
                    if (++ii == ilim) break;
                } else {
                    if (++jj == jlim) break;
                    c = __dadd_rn(c, sh.w[r][jj]);
                }
            }
            if (ii == ilim) {
                nflush = ii;
                if (ki + ii == M) {                           // every position placed
                    active = false;
                    if (status) status[b0 + r] = 0;
                } else { need_p = 1; ki += COLS; ii = 0; }
            } else if (kj + jj == M) {                        // j ran off the end: the reference's IndexError (:145)
                nflush = ii;
                active = false;
                if (status) status[b0 + r] = 1;
            } else { need_w = 1; kj += COLS; jj = 0; fresh_w = true; }
        }
        sh.nflush[r] = nflush; sh.fbase[r] = (int)(fbase / COLS);
        sh.load_w[r] = need_w; sh.kj[r] = (int)(kj / COLS);
        sh.load_p[r] = need_p; sh.ki[r] = (int)(ki / COLS);
        more = active || nflush > 0;
    }
}

}  // namespace rsb
}  // namespace bke

using namespace bke;

extern "C" {

int bke_resample_bank(const bke_resample_bank_args *a, void *stream)
{
    if (!a) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    if (a->n_sets < 0 || a->n_particles < 0) { set_error("n_sets and n_particles must be >= 0"); return BKE_ERR_BAD_ARG; }
    if (a->n_particles >= ((int64_t)1 << 31)) { set_error("n_particles must be < 2^31 (indexes are int32, resampling.py:141)"); return BKE_ERR_BAD_ARG; }
    if ((a->u == nullptr) == (a->uniforms == nullptr)) { set_error("give exactly one of u (systematic) and uniforms (stratified)"); return BKE_ERR_BAD_ARG; }
    if (a->n_sets == 0 || a->n_particles == 0) return BKE_OK;
    if (!a->weights || !a->indexes) { set_error("weights and indexes must be non-NULL"); return BKE_ERR_BAD_ARG; }
    const int64_t blocks = (a->n_sets + rsb::ROWS - 1) / rsb::ROWS;
    if (blocks >= ((int64_t)1 << 31)) { set_error("n_sets too large"); return BKE_ERR_BAD_ARG; }
    cudaStream_t s = (cudaStream_t)stream;
    if (a->uniforms)
        rsb::k_resample_bank<true><<<(unsigned)blocks, rsb::ROWS, 0, s>>>(a->n_sets, a->n_particles, a->weights, nullptr,
                                                                         a->uniforms, a->indexes, a->status);
    else
        rsb::k_resample_bank<false><<<(unsigned)blocks, rsb::ROWS, 0, s>>>(a->n_sets, a->n_particles, a->weights, a->u,
                                                                          nullptr, a->indexes, a->status);
    return check_cuda(cudaGetLastError(), "resample bank launch");
}

}  // extern "C"
