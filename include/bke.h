/* bke.h — C-ABI of the H100 batched state-estimation engine ("bke").
 *
 * This is the drop-in boundary for the hot path of rlabbe/filterpy (reference @ 3b51149,
 * v1.4.5).  The reference is pure Python and has no FFI of its own: the interface each entry
 * point replaces is the Python call surface cited beside it (paths relative to the reference
 * root).  INTEGRATION.md shows the ctypes binding a filterpy maintainer would add.
 *
 * Conventions
 *   - every array pointer is a DEVICE pointer unless the name ends in _host; arrays are dense,
 *     row-major, with a leading filter (bank) axis: x[N,n]  P[N,n,n]  F[N,n,n]  H[N,m,n]
 *     Q[N,n,n]  R[N,m,m]  z[N,m]  (n = dim_x, m = dim_z);
 *   - a model array may be shared by the whole bank: pass its *_stride = 0 (stride is the
 *     element distance between consecutive filters, n*n for a per-filter F, and so on);
 *   - dtype is BKE_F32 or BKE_F64 and applies to every floating-point array of the call;
 *   - `stream` is a cudaStream_t passed as void*; calls are asynchronous, stream-ordered,
 *     re-entrant, never allocate and never synchronise the host;
 *   - return value: BKE_OK or an error code; bke_last_error() gives the text for the calling
 *     thread.  Per-filter numerical failures (singular S, non-PD P) do not fail the call: they
 *     are reported in the optional int32 `status[N]` array (0 = ok), the way LAPACK's `info` is.
 *   - there is NO CPU fallback: on a machine without an sm_90 device the compute entry
 *     points return BKE_ERR_CUDA.
 */
#ifndef BKE_H_
#define BKE_H_

#ifndef __CUDACC_RTC__
#include <stddef.h>
#include <stdint.h>
#else   /* NVRTC (run-time compiled UKF models, bke_ukf_model_compile) has no libc headers */
typedef signed char int8_t; typedef unsigned char uint8_t; typedef int int32_t; typedef unsigned int uint32_t;
typedef long long int64_t; typedef unsigned long long uint64_t; typedef unsigned long size_t;
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define BKE_ABI_VERSION 1

/* dtypes */
#define BKE_F32 0
#define BKE_F64 1

/* return codes */
#define BKE_OK 0
#define BKE_ERR_BAD_ARG 1
#define BKE_ERR_UNSUPPORTED 2
#define BKE_ERR_CUDA 3

/* per-filter status codes written to status[N] */
#define BKE_STATUS_OK 0
#define BKE_STATUS_SINGULAR_S 1      /* np.linalg.inv would raise LinAlgError (kalman_filter.py:541) */
#define BKE_STATUS_NOT_PD 2          /* scipy.linalg.cholesky would raise LinAlgError (sigma_points.py:168) */

/* what a kf/ukf step does */
#define BKE_DO_PREDICT 1u            /* KalmanFilter.predict   kalman_filter.py:437-482 */
#define BKE_DO_UPDATE 2u             /* KalmanFilter.update    kalman_filter.py:485-561 */
#define BKE_UPDATE_FIRST 4u          /* batch_filter(update_first=True) order, kalman_filter.py:966-978 */
#define BKE_STATUS_STICKY 8u         /* status[f] is only written when the step FAILS (the caller zeroed it): an
                                        error of an earlier step survives.  bke_kf_batch_filter's status is
                                        sticky over all epochs on every path. */
#define BKE_REVERSE_TILES 16u        /* scheduling hint, no result depends on it: the 4/2 fp32 step (bke_kf_step,
                                        bke_kf_step_sym, bke_kf_step_packed) walks the bank last tile to first.
                                        A caller stepping a bank larger than L2 in place sets it on every other
                                        step, so that each step starts on the filters the previous one finished
                                        while their x, P and models are still in L2.  Other kernels ignore it,
                                        and so does the 4/2 step of a bank whose state fits L2 anyway (at
                                        most 38 MiB of x, P, stepped in place).  bke_kf_steps_packed given
                                        a tile-order word (bke_kf_args.tile_order) ignores it too: the word
                                        alternates the order across launches on the device, where a flag
                                        frozen into a captured launch cannot. */

int bke_abi_version(void);
const char *bke_last_error(void);
/* number of CUDA devices usable by the library (0 on a CPU-only box; never fails) */
int bke_device_count(void);

/* ------------------------------------------------------------------------------------------
 * Linear Kalman filter bank.
 * Replaces, for N independent filters at once:
 *   KalmanFilter.predict(u, B, F, Q)      filterpy/kalman/kalman_filter.py:437-482
 *   KalmanFilter.update(z, R, H)          filterpy/kalman/kalman_filter.py:485-561
 *   (and their procedural twins predict()/update(), kalman_filter.py:1571-1621 / 1401-1508)
 * Arithmetic per filter, in this order (flags = BKE_DO_PREDICT | BKE_DO_UPDATE):
 *   x <- F x (+ B u);  P <- alpha_sq * F P F' + Q;                       [x_prior, P_prior]
 *   y = z - H x;  S = H P H' + R;  SI = S^-1;  K = P H' SI;  x <- x + K y;
 *   P <- (I - K H) P (I - K H)' + K R K'                                  (Joseph form, :555-556)
 * z_valid[i] == 0 means "z is None" for filter i: the update is skipped and the posterior is
 * the prior (kalman_filter.py:515-520).  z_valid == NULL means every filter has a measurement.
 * For such a filter the step writes y = 0 and leaves K, S, SI and log_likelihood unchanged.  The
 * reference's log-likelihood is then log N(0; 0, S) of the kept S (-inf while S is still zero);
 * the caller computes it (KalmanFilter.update does).
 * Optional outputs (NULL = not wanted): x_prior, P_prior, K[N,n,m], y[N,m], S[N,m,m],
 * SI[N,m,m], log_likelihood[N] (log N(y; 0, S), kalman_filter.py:1203-1210), status[N].
 * x_out/P_out may alias x/P (in-place update).
 * Kernels behind this call (same arithmetic, picked by shape; DESIGN.md §3): 4/2 fp32 TMA register tile, register tiles
 * with direct loads (4/2 fp64, 1/1 .. 4/4, 6/3 fp32), row blocks (9/3, 16/4, 16/2, 6/3 fp64, 32/4 fp32), a catch-all for any
 * shape, and — fp32 banks with dim_x = 16 or 32 whose F and Q are shared (stride 0) — the wgmma tile: F P F' as
 * three-term TF32 products accumulated in fp32 (everything else of the
 * step in plain fp32), the whole predict+update in one launch when H and R are shared too and dim_z <= 4.
 */
typedef struct bke_kf_args {
    int64_t n_filters;
    int32_t dim_x, dim_z, dim_u;     /* dim_u may be 0 */
    int32_t dtype;                   /* BKE_F32 | BKE_F64 */
    uint32_t flags;                  /* BKE_DO_* */
    uint32_t reserved;
    double alpha_sq;                 /* fading-memory factor, kalman_filter.py:478 (1.0 = none) */
    const void *x, *P;               /* in  */
    void *x_out, *P_out;             /* out */
    const void *F; int64_t F_stride;
    const void *H; int64_t H_stride;
    const void *Q; int64_t Q_stride;
    const void *R; int64_t R_stride;
    const void *B; int64_t B_stride; /* [N,n,dim_u] or NULL */
    const void *u; int64_t u_stride; /* [N,dim_u]   or NULL */
    const void *z;                   /* [N,m]; may be NULL when BKE_DO_UPDATE is not set */
    const uint8_t *z_valid;          /* [N] or NULL */
    void *x_prior, *P_prior;
    void *K, *y, *S, *SI, *log_likelihood;
    int32_t *status;
    /* Optional HOST copies of models that are shared by the bank (stride 0), in `dtype`: when all
     * four are given (and equal the device copies) a kernel may carry them in its launch parameters
     * instead of loading them from device memory.  NULL = not available. */
    const void *F_host, *Q_host, *H_host, *R_host;
    /* Optional DEVICE tile-order word of the bank, two uint32 {epoch, arrived}, zeroed once by the caller,
     * 4-byte aligned; read by bke_kf_steps_packed only (every other call ignores it).  A launch walks the
     * bank last tile to first when epoch is odd (BKE_REVERSE_TILES is then ignored), and leaves epoch one
     * higher and arrived at 0 when it ends, so consecutive launches on one word alternate, including the
     * replays of a captured graph of one launch.  Launches that share a word must run in stream order.
     * NULL = not used. */
    uint32_t *tile_order;
} bke_kf_args;

int bke_kf_step(const bke_kf_args *args, void *stream);

/* KalmanFilter.update_correlated(z, R, H)      filterpy/kalman/kalman_filter.py:670-752
 * bke_kf_step with process noise correlated with the measurement noise by M [N,n,m] (M_stride = n*m) or
 * [n,m] shared (M_stride = 0).  flags = BKE_DO_UPDATE, optionally | BKE_DO_PREDICT (the predict runs first,
 * as in bke_kf_step) and BKE_STATUS_STICKY.  Per filter with a measurement:
 *   y = z - H x;  S = H P H' + H M + M' H' + R;  SI = S^-1;  K = (P H' + M) SI;  x <- x + K y;
 *   P <- P - K (H P + M')                       (not the Joseph form, and not symmetrised: :748)
 * z_valid, status and the optional outputs are those of bke_kf_step (a filter without a measurement gets
 * y = 0 and keeps K, S, SI and log_likelihood).  A NULL M, or a stride that is neither 0 nor n*m, is
 * BKE_ERR_BAD_ARG. */
int bke_kf_step_correlated(const bke_kf_args *args, const void *M, int64_t M_stride, void *stream);

/* KalmanFilter.update_sequential(start, z_i, R_i, H_i)      filterpy/kalman/kalman_filter.py:754-824
 * The update with the block of rows start .. start+rows-1 (L = rows) of z, H and R.  step.dim_z is the bank's
 * full m, 1 <= L and start + L <= m.  step.z is z_i [N,L].  H_i [.,L,n] and R_i [.,L,L] are per filter
 * (stride L*n, L*L) or shared (stride 0); a NULL one is read in place from the block of step.H / step.R (the
 * bank's [.,m,n] / [.,m,m], strides as in bke_kf_step), without a copy.  Per filter with a measurement:
 *   y_i = z_i - H_i x;  S_i = H_i P H_i' + R_i;  K_i = P H_i' S_i^-1, or P H_i' (1 / S_i) when L = 1;
 *   x <- x + K_i y_i;  P <- (I - K_i H_i) P (I - K_i H_i)' + K_i R_i K_i'        (Joseph form, :819)
 * and y[N,m] rows, K[N,n,m] columns and z_record[N,m] rows start .. start+L-1 receive y_i, K_i and z_i (each
 * may be NULL); everything else of them keeps its value, and so does a filter with z_valid[f] = 0, which gets
 * only the predict of BKE_DO_PREDICT.  For L = 1 a zero S_i gives inf (the reference's reciprocal): status
 * stays BKE_STATUS_OK.  For L > 1 a singular S_i is BKE_STATUS_SINGULAR_S and the filter keeps the prior.
 * flags, B / u, x_prior / P_prior and status are those of bke_kf_step; S, SI and log_likelihood are not
 * written by this update (non-NULL is BKE_ERR_BAD_ARG).  A block outside 0 .. m-1 or a bad H_i / R_i stride is
 * BKE_ERR_BAD_ARG. */
typedef struct bke_kf_rows_args {
    bke_kf_args step;
    int32_t start, rows;
    const void *H_i; int64_t H_i_stride;     /* [N,L,n] / [L,n], or NULL: rows of step.H */
    const void *R_i; int64_t R_i_stride;     /* [N,L,L] / [L,L], or NULL: the block of step.R */
    void *z_record;                          /* [N,m] or NULL */
} bke_kf_rows_args;

int bke_kf_update_rows(const bke_kf_rows_args *args, void *stream);

/* Packed symmetric models of a dim_x = 4, dim_z = 2, BKE_F32 bank (per-filter Q and R).
 * Q and R are covariances: when every filter's Q and R equal their transposes bit for bit, a step
 * only needs their upper triangles, 52 instead of 80 B per filter.  The record holds them tile-major,
 * one tile of 128 filters after the other, each tile 13 planes of 128 floats (Q00 Q01 Q02 Q03 Q11
 * Q12 Q13 Q22 Q23 Q33 R00 R01 R11, plane k holding word k of each filter of the tile), padded to a
 * whole last tile.
 *   bke_kf_sym_models_bytes  the size of the record of n_filters filters (the caller allocates it,
 *                            16-byte aligned);
 *   bke_kf_pack_sym_models   fills `record` from the dense Q[N,4,4] and R[N,2,2] and sets the device
 *                            int32 *asymmetric to 0 when every filter is exactly symmetric, 1 when
 *                            one is not (compared as bits: -0.0 against +0.0 or two NaN payloads
 *                            count as asymmetric); only in the first case may the record be used;
 *   bke_kf_step_sym          bke_kf_step with the record standing in for args->Q and args->R (which
 *                            must still be the per-filter arrays it was packed from, unchanged since);
 *                            the results are bit-identical to bke_kf_step's.
 * Both calls return BKE_ERR_UNSUPPORTED for other shapes, dtypes, shared models or misaligned pointers;
 * bke_kf_step is then the call to make. */
size_t bke_kf_sym_models_bytes(int64_t n_filters);
int bke_kf_pack_sym_models(int64_t n_filters, int32_t dim_x, int32_t dim_z, int32_t dtype, const void *Q,
                           const void *R, void *record, int32_t *asymmetric, void *stream);
int bke_kf_step_sym(const bke_kf_args *args, const void *record, void *stream);

/* Packed model words of a dim_x = 4, dim_z = 2, BKE_F32 bank whose F, Q, H and R are all per filter.
 * Banks built from a template and a few per-filter parameters (dt, q, r) repeat most model words bit for
 * bit in every filter; a step then only needs the words that differ, and the others ride in the launch
 * parameters (40 instead of 148 B of models per filter for a constant-velocity bank with per-filter dt,
 * q and r).  A filter's models are 37 words, in this order (word e = bit e of `varying`):
 *   F 0..15 (row-major) | Q 16..25 (upper triangle: Q00 Q01 Q02 Q03 Q11 Q12 Q13 Q22 Q23 Q33) |
 *   H 26..33 (row-major) | R 34..36 (R00 R01 R11).
 *   bke_kf_scan_models          fills the map (DEVICE memory, 16-byte aligned) from the dense F[N,4,4],
 *                               Q[N,4,4], H[N,2,4], R[N,2,2]: bit e of `varying` is set when word e of
 *                               some filter differs from filter 0's in any bit (-0.0 against +0.0 and two
 *                               NaN payloads differ), `words` are filter 0's, `asymmetric` is 1 when a
 *                               filter's Q or R differs from its transpose in any bit (the record may only
 *                               be used when it is 0).  With v_0 < v_1 < ... the varying words (slot s
 *                               of the record holds word v_s), let c(s) be the lowest slot t < s whose
 *                               filter-0 word has the same bits as v_s's; bit s (s < 32) of `duplicate`
 *                               is set when c(s) exists and word v_s equals word v_c(s) bit for bit in
 *                               every filter, so plane s is a copy of plane c(s) (which is never flagged
 *                               itself).  The rule is conservative: a copy it misses is read from its own
 *                               plane.  A zero `duplicate` means "no copies";
 *   bke_kf_packed_models_bytes  the size of the record of n_filters filters for a `varying` mask (0 for a
 *                               mask with bits above 36); the caller allocates it, 16-byte aligned;
 *   bke_kf_pack_models          fills the record: one tile of 128 filters after the other, each tile
 *                               k = popcount(varying) planes of 128 floats, plane s holding the s-th
 *                               varying word (in the order above) of each filter of the tile, padded with
 *                               zeros to a whole last tile;
 *   bke_kf_step_packed          bke_kf_step with the record and a HOST copy of the map standing in for
 *                               args->F, Q, H and R (which must still be the per-filter arrays they were
 *                               scanned and packed from, unchanged since); the results are bit-identical
 *                               to bke_kf_step's.  The record may be NULL when no word varies.  A plane
 *                               flagged in the map's `duplicate` is not read: the step reads its
 *                               representative plane c(s) instead (40 -> 20 B of models per filter for the
 *                               constant-velocity bank above, which has the same dt, q and r on both
 *                               axes).  A `duplicate` bit at or above popcount(varying), or whose slot has
 *                               no c(s), is refused with BKE_ERR_BAD_ARG;
 *   bke_kf_steps_packed         n_steps consecutive predict+update steps in ONE launch: the same x_out and
 *                               P_out, bit for bit, as n_steps calls of bke_kf_step_packed with args->z =
 *                               zs[k] in turn (args->z itself is ignored).  Every thread keeps its filter's x
 *                               and P in registers between the steps, so the state is read and written once
 *                               per call instead of once per step (212 B per filter and call with 4 steps
 *                               of the constant-velocity bank above, against 4 x 188); between the steps
 *                               x and P exist nowhere in memory.  zs is a HOST array of n_steps device
 *                               pointers, each [N,2], 16-byte aligned and clear of x and P; the same pointer
 *                               may appear more than once.  It takes flags = BKE_DO_PREDICT | BKE_DO_UPDATE
 *                               (BKE_REVERSE_TILES is honoured as in a single step when args->tile_order
 *                               is NULL; with a tile-order word the word decides, and a word that is not
 *                               4-byte aligned is refused with BKE_ERR_BAD_ARG), an in-place state
 *                               (x_out = x, P_out = P), 1 <= n_steps <= BKE_KF42_MAX_RING, and neither
 *                               z_valid, B / u, status nor any optional output: anything else returns
 *                               BKE_ERR_UNSUPPORTED.
 * The calls return BKE_ERR_UNSUPPORTED for other shapes, dtypes, shared models, an asymmetric map or
 * misaligned pointers; bke_kf_step is then the call to make. */
#define BKE_KF42_MODEL_WORDS 37
#define BKE_KF42_MAX_RING 8
typedef struct bke_kf_model_map {
    uint64_t varying;                       /* bit e: word e differs between filters */
    int32_t asymmetric;                     /* 1: some Q or R is not exactly symmetric */
    uint32_t duplicate;                     /* bit s: plane s is a copy of plane c(s) in every filter */
    float words[BKE_KF42_MODEL_WORDS];      /* filter 0's words */
} bke_kf_model_map;

int bke_kf_scan_models(int64_t n_filters, int32_t dim_x, int32_t dim_z, int32_t dtype, const void *F, const void *Q,
                       const void *H, const void *R, bke_kf_model_map *map, void *stream);
size_t bke_kf_packed_models_bytes(int64_t n_filters, uint64_t varying);
int bke_kf_pack_models(int64_t n_filters, int32_t dim_x, int32_t dim_z, int32_t dtype, const void *F, const void *Q,
                       const void *H, const void *R, uint64_t varying, void *record, void *stream);
int bke_kf_step_packed(const bke_kf_args *args, const void *record, const bke_kf_model_map *host_map, void *stream);
int bke_kf_steps_packed(const bke_kf_args *args, const void *record, const bke_kf_model_map *host_map,
                        const void *const *zs, int32_t n_steps, void *stream);

/* The number of nodes of the graph `stream` is capturing into (*n_nodes; HOST).  A caller that captures its own
 * launches can tell from it whether anything else went into the graph.  BKE_ERR_BAD_ARG when the stream is not
 * capturing. */
int bke_capture_node_count(void *stream, int64_t *n_nodes);

/* KalmanFilter.batch_filter over T epochs for a bank (kalman_filter.py:826-993; procedural
 * twin :1664-1788): the time loop runs inside one kernel with the models resident on chip.
 *   zs[T,N,m], zs_valid[T,N] (or NULL)
 *   means[T,N,n]  covariances[T,N,n,n]  means_p[T,N,n]  covariances_p[T,N,n,n]  (any may be NULL)
 * Models are constant in time here (Fs/Qs/Hs/Rs = None in the reference); the host side loops
 * bke_kf_step for per-epoch models.  The final state is written to x_out/P_out.
 * `step` carries everything else (flags selects update_first; its z/x_prior/... are ignored). */
typedef struct bke_kf_batch_args {
    bke_kf_args step;
    int64_t n_steps;
    const void *zs;
    const uint8_t *zs_valid;
    void *means, *covariances, *means_p, *covariances_p;
} bke_kf_batch_args;

int bke_kf_batch_filter(const bke_kf_batch_args *args, void *stream);

/* FixedLagSmoother.smooth / smooth_batch for a bank (filterpy/kalman/fixed_lag_smoother.py:133-215 /
 * :217-311): T epochs of fixed-lag smoothing with lag N, continuing a run that has taken `count` epochs.
 * Per filter, epoch k = count + t:
 *   x_pre = F x (+ B u);  P = F P F' + Q;  y = z - H x_pre;  S = H P H' + R;  SI = S^-1;  K = P H' SI;
 *   x = x_pre + K y;  P = (I - K H) P (I - K H)' + K R K'   (no fading factor)          [xhat[t] = x]
 *   row k of the history = x_pre;  if k < N: row k = x;  else, with g = H' SI y and A = (F - K H)':
 *   row k - i += P A^i g  for i = 0 .. N-1      (the reference's P (F - K H)'^i H' SI y, reassociated)
 * After epoch k, rows k-N+2 .. k can still change; every row <= k-N+1 is final.
 *   xs_smooth   the history, row r at r * n_filters * dim_x: the call reads the live rows count-N+1 ..
 *               count-1 and writes rows up to count+T-1 (the caller provides room for them);
 *   zs[T,N,m], us[T,N,dim_u] (NULL: no control input; else step.B and dim_u >= 1), xhat[T,N,n] (or NULL);
 *   step        n_filters, dims, dtype, x / P, the models and strides, B, x_out / P_out (the state after the
 *               last epoch; may alias x / P) and the optional status[N], y[N,m] and S[N,m,m] of the last
 *               epoch.  Its flags, alpha_sq, z, z_valid, u, x_prior, P_prior, K, SI, log_likelihood are ignored.
 * Every measurement is present (the reference has no missing-measurement rule: z = None raises TypeError).
 * Where the reference's inv(S) raises LinAlgError, status[f] = BKE_STATUS_SINGULAR_S (sticky over the call's
 * epochs), that filter keeps its prior for the epoch (x = x_pre, P = the predicted P), its row k is x_pre
 * and no row is corrected; y and S are still the epoch's z - H x_pre and H P H' + R, on both paths.
 * The workspace (bke_fls_workspace_bytes, 16-byte aligned) is only needed when the call runs the per-epoch
 * path: the size is 0 when the fused kernel covers the shape.  Fused (DESIGN.md §3.4b): 1/1, 2/1 and 4/2,
 * fp32 and fp64, without control input, lag <= BKE_FLS_FUSED_MAX_LAG; the lag window stays in shared memory
 * and each history row is stored once.  Every other call runs bke_kf_step's kernels once per epoch and a
 * lag-correction kernel on the history in HBM. */
#define BKE_FLS_FUSED_MAX_LAG 16
typedef struct bke_fls_args {
    bke_kf_args step;
    int64_t n_steps;                 /* T >= 1 */
    int64_t lag;                     /* N >= 0 */
    int64_t count;                   /* epochs already taken (>= 0) */
    const void *zs;
    const void *us;
    void *xs_smooth;
    void *xhat;
    void *workspace; size_t workspace_bytes;
} bke_fls_args;

size_t bke_fls_workspace_bytes(int64_t n_filters, int32_t dim_x, int32_t dim_z, int32_t dim_u, int32_t dtype, int64_t lag);
int bke_fls_smooth(const bke_fls_args *args, void *stream);

/* ------------------------------------------------------------------------------------------
 * Unscented Kalman filter bank (Merwe scaled sigma points).
 * Replaces UnscentedKalmanFilter.predict / update (filterpy/kalman/UKF.py:364-411, 413-491),
 * MerweScaledSigmaPoints.sigma_points / _compute_weights (sigma_points.py:124-192) and
 * unscented_transform (unscented_transform.py:99-128) for N filters at once.
 * fx / hx are Python callables in the reference (UKF.py:521-522, 463-464); a device cannot call
 * back into Python, so the process and measurement functions come from a closed set:
 */
#define BKE_FX_LINEAR 0          /* x' = F x                      (F[n,n], F_stride 0 or n*n) */
#define BKE_FX_CONST_VEL 1       /* state (p0,v0,p1,v1,...): p_i += dt * v_i */
#define BKE_HX_LINEAR 0          /* z = H x                       (H[m,n]) */
#define BKE_HX_RANGE_AZ_EL 1     /* n=6 (x,vx,y,vy,z,vz) -> (range, azimuth, elevation), m=3 */
#define BKE_HX_RANGE_BEARING 2   /* n=4 (x,vx,y,vy) -> (range, bearing), m=2 */
#define BKE_FX_USER 100          /* device function supplied as source text: bke_ukf_model_compile (below) */
#define BKE_HX_USER 100

/* flag of bke_ukf_args.flags and bke_ukf_rts_args.flags: SimplexSigmaPoints(n) (sigma_points.py:386-534) instead
 * of MerweScaledSigmaPoints: n + 1 points x + D_j, D = (chol_upper(P)' sqrt(n) Istar)', Wm = Wc = 1/(n+1);
 * alpha, beta and kappa are ignored */
#define BKE_UKF_SIMPLEX 32u

typedef struct bke_ukf_args {
    int64_t n_filters;
    int32_t dim_x, dim_z;
    int32_t dtype;
    uint32_t flags;                  /* BKE_DO_PREDICT | BKE_DO_UPDATE (update alone re-draws the
                                        sigma points from (x,P), UKF.py:407), | BKE_UKF_SIMPLEX */
    int32_t fx_model, hx_model;
    double dt;
    double alpha, beta, kappa;       /* MerweScaledSigmaPoints(n, alpha, beta, kappa) */
    const void *x, *P;
    void *x_out, *P_out;
    const void *Q; int64_t Q_stride;
    const void *R; int64_t R_stride;
    const void *F; int64_t F_stride; /* BKE_FX_LINEAR only */
    const void *H; int64_t H_stride; /* BKE_HX_LINEAR only */
    const void *z;
    const uint8_t *z_valid;
    void *x_prior, *P_prior;
    void *K, *y, *S, *SI, *log_likelihood;
    int32_t *status;
} bke_ukf_args;

int bke_ukf_step(const bke_ukf_args *args, void *stream);

/* User-supplied process / measurement functions.
 * The reference's UnscentedKalmanFilter takes fx(x, dt, **fx_args) and hx(x, **hx_args) as Python
 * callables (filterpy/kalman/UKF.py:284-288; called once per sigma point at :521-522 and :463-464).  The
 * drop-in takes them as CUDA C++ source text and compiles a kernel instance around them at run time
 * (NVRTC, sm_90a; the same kernel text as the pre-built instances).  `source` defines, for the element
 * type `real` (a typedef of float / double the program text provides; BKE_DIM_X / BKE_DIM_Z are
 * #defined):
 *     __device__ void fx(const real *x, real *x_out, real dt, const real *args);     when fx_model == BKE_FX_USER
 *     __device__ void hx(const real *x, real *z_out, const real *args);              when hx_model == BKE_HX_USER
 * The other function may be one of the built-ins (BKE_FX_LINEAR, BKE_FX_CONST_VEL, BKE_HX_LINEAR).
 * `include_dirs`: ':'-separated directories holding the engine's kernel headers (filterpy_b200/csrc).
 * `args` of bke_ukf_step_model: device vectors handed to fx / hx (the keyword arguments of the reference's
 * callables), one for the bank (stride 0) or one per filter (stride = elements per filter); may be NULL.
 * A source that does not compile returns BKE_ERR_BAD_ARG with the compiler log in bke_last_error(). */
typedef struct bke_ukf_model bke_ukf_model;
int bke_ukf_model_compile(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, const char *source,
                          const char *include_dirs, bke_ukf_model **out);
const char *bke_ukf_model_log(const bke_ukf_model *model);                 /* NVRTC's log (warnings) */
int bke_ukf_model_registers(const bke_ukf_model *model, int32_t extras);   /* registers per thread of the instance */
void bke_ukf_model_free(bke_ukf_model *model);
int bke_ukf_step_model(const bke_ukf_args *args, const bke_ukf_model *model, const void *fx_args, int64_t fx_args_stride,
                       const void *hx_args, int64_t hx_args_stride, void *stream);
/* the NVRTC half alone (needs no GPU): size of the sm_90a cubin, 0 on failure (log in bke_last_error()) */
size_t bke_debug_ukf_model_cubin_bytes(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model,
                                       const char *source, const char *include_dirs);

/* The reference's mean / residual / state-add hooks (UKF.py:97-140: x_mean_fn, z_mean_fn, residual_x,
 * residual_z, state_add), e.g. to wrap angles and take circular means, cross as source text too.  `hooks`
 * is a mask of the functions `source` defines (n = BKE_DIM_X, m = BKE_DIM_Z, BKE_N_SIGMAS = 2n + 1):
 *     __device__ void x_mean_fn(const real *sigmas, const real *Wm, real *out);   sigmas[BKE_N_SIGMAS][n]  BKE_HOOK_X_MEAN
 *     __device__ void z_mean_fn(const real *sigmas, const real *Wm, real *out);   sigmas[BKE_N_SIGMAS][m]  BKE_HOOK_Z_MEAN
 *     __device__ void residual_x(const real *a, const real *b, real *out);        out = a - b, n           BKE_HOOK_RESIDUAL_X
 *     __device__ void residual_z(const real *a, const real *b, real *out);        out = a - b, m           BKE_HOOK_RESIDUAL_Z
 *     __device__ void state_add(const real *a, const real *b, real *out);         out = a + b, n           BKE_HOOK_STATE_ADD
 * With hooks != 0 any fx / hx model may be compiled, built-in or user; the handle also carries the RTS
 * smoother (bke_ukf_rts_smoother_model), which calls x_mean_fn and residual_x as UKF.py:720-735 does.
 * Hooks need dim_x <= 8 (BKE_ERR_UNSUPPORTED otherwise).  hooks == 0 is bke_ukf_model_compile exactly.
 * The handle is launched with bke_ukf_step_model. */
#define BKE_HOOK_X_MEAN 1u
#define BKE_HOOK_Z_MEAN 2u
#define BKE_HOOK_RESIDUAL_X 4u
#define BKE_HOOK_RESIDUAL_Z 8u
#define BKE_HOOK_STATE_ADD 16u
int bke_ukf_model_compile_hooks(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, uint32_t hooks,
                                const char *source, const char *include_dirs, bke_ukf_model **out);
size_t bke_debug_ukf_model_hooks_cubin_bytes(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model,
                                             uint32_t hooks, const char *source, const char *include_dirs);

/* The same for a chosen point set: points = 0 (MerweScaledSigmaPoints: bke_ukf_model_compile_hooks exactly) or
 * BKE_UKF_SIMPLEX (SimplexSigmaPoints; the text sees BKE_N_SIGMAS = n + 1, hooks or not).  The handle remembers
 * its point set: bke_ukf_step_model and bke_ukf_rts_smoother_model refuse args whose flags ask for the other
 * set (BKE_ERR_BAD_ARG). */
int bke_ukf_model_compile_points(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, uint32_t hooks,
                                 uint32_t points, const char *source, const char *include_dirs, bke_ukf_model **out);
size_t bke_debug_ukf_model_points_cubin_bytes(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model,
                                              uint32_t hooks, uint32_t points, const char *source, const char *include_dirs);

/* ------------------------------------------------------------------------------------------
 * Cubature Kalman filter bank.
 * Replaces CubatureKalmanFilter.predict / update (filterpy/kalman/CubatureKalmanFilter.py:292-327,
 * 329-389; spherical_radial_sigmas :52-61, ckf_transform :87-98) for N filters at once, with the fx / hx
 * models of the UKF above (the closed set, or user source through bke_ckf_model_compile below).
 * Per filter, m = 2n points, no centre point:
 *   U = cholesky(P) * sqrt(n) (upper);  points x + U[k,:], x - U[k,:];  f_k = fx(point_k)   (:56-59, :320-321)
 *   x- = sum f_k / m;  P- = sum (f_k - x-)(f_k - x-)' / m + Q                              [x_prior, P_prior]
 *   Z_k = hx(f_k) (the propagated points, not redrawn, :362-363);  z^ = sum Z_k / m;
 *   S = sum (Z_k - z^)(..)' / m + R;  Pxz = sum (f_k - x)(Z_k - z^)' / m  (:366-373);
 *   K = Pxz S^-1;  y = z - z^;  x <- x + K y;  P <- P - K S K'                               (:375-379)
 * The covariances are formed centred; the reference's ckf_transform forms them as raw second moments
 * (sum f f' - m x x'), the same mathematics with more cancellation.
 * sigmas_f[N,2n,n] (may be NULL) holds the propagated points, the reference's self.sigmas_f: a call with
 * BKE_DO_PREDICT writes them when it is non-NULL, an update-only call reads them (and needs it non-NULL:
 * the reference's update without predict reuses the points of the last predict).  z_valid, the optional
 * outputs and status[N] behave as in bke_ukf_args. */
typedef struct bke_ckf_args {
    int64_t n_filters;
    int32_t dim_x, dim_z;
    int32_t dtype;
    uint32_t flags;                  /* BKE_DO_PREDICT | BKE_DO_UPDATE */
    int32_t fx_model, hx_model;
    double dt;
    const void *x, *P;
    void *x_out, *P_out;
    const void *Q; int64_t Q_stride;
    const void *R; int64_t R_stride;
    const void *F; int64_t F_stride; /* BKE_FX_LINEAR only */
    const void *H; int64_t H_stride; /* BKE_HX_LINEAR only */
    const void *z;
    const uint8_t *z_valid;
    void *x_prior, *P_prior;
    void *K, *y, *S, *SI, *log_likelihood;
    int32_t *status;
    void *sigmas_f;                  /* [N,2n,n] or NULL */
} bke_ckf_args;

int bke_ckf_step(const bke_ckf_args *args, void *stream);

/* User-supplied fx / hx for the CKF: the reference calls fx(x, dt, *fx_args) and hx(x, *hx_args)
 * (CubatureKalmanFilter.py:314-321, :354-363).  Source text, include_dirs and the args vectors follow
 * bke_ukf_model_compile / bke_ukf_step_model; the positional arguments are args[0..] in order.  The handle
 * is a bke_ukf_model built for the CKF kernel (bke_ukf_model_log / _registers / _free apply to it);
 * bke_ckf_step_model refuses a UKF handle and bke_ukf_step_model a CKF handle (BKE_ERR_BAD_ARG). */
int bke_ckf_model_compile(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, const char *source,
                          const char *include_dirs, bke_ukf_model **out);
int bke_ckf_step_model(const bke_ckf_args *args, const bke_ukf_model *model, const void *fx_args, int64_t fx_args_stride,
                       const void *hx_args, int64_t hx_args_stride, void *stream);
/* the NVRTC half alone (needs no GPU): size of the sm_90a cubin, 0 on failure (log in bke_last_error()) */
size_t bke_debug_ckf_model_cubin_bytes(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model,
                                       const char *source, const char *include_dirs);
/* The CKF with hooks: the reference's CKF calls residual_z only (y = residual_z(z, z^), :376), so `hooks`
 * is 0 or BKE_HOOK_RESIDUAL_Z; otherwise as bke_ukf_model_compile_hooks. */
int bke_ckf_model_compile_hooks(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, uint32_t hooks,
                                const char *source, const char *include_dirs, bke_ukf_model **out);
size_t bke_debug_ckf_model_hooks_cubin_bytes(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model,
                                             uint32_t hooks, const char *source, const char *include_dirs);

/* ------------------------------------------------------------------------------------------
 * Ensemble Kalman filter bank.
 * Replaces EnsembleKalmanFilter.initialize / predict / update (filterpy/kalman/ensemble_kalman_filter.py:
 * 187-215, 275-290, 218-273) for N filters of n_members members each, with the fx / hx models of the UKF
 * above (the closed set, or user source through bke_enkf_model_compile below).  sigmas[N, n_members, n].
 * Per filter (flags = BKE_DO_PREDICT | BKE_DO_UPDATE; a fused call runs the predict first):
 *   predict:  s_i <- fx(s_i, dt) + e_i, e_i ~ N(0, Q);  x <- mean(s);  P <- sum (s_i - x)(..)' / (n_members - 1)
 *             [x_prior, P_prior]
 *   update:   h_i = hx(s_i);  z^ = mean(h);  S = sum (h_i - z^)(..)' / (n_members - 1) + R;
 *             Pxz = sum (s_i - x)(h_i - z^)' / (n_members - 1) with the x held before the update (:256-257);
 *             SI = S^-1;  K = Pxz SI;  s_i <- s_i + K (z + r_i - h_i), r_i ~ N(0, R);  x <- mean(s);
 *             P <- P - K S K'  (not the ensemble covariance, as in the reference, :268)      [K, S, SI]
 * Noise: standard normals xi from Philox4x32-10 keyed with (seed, filter index) and counted with
 * (component / 2, member, draw call, filter index >> 32); Box-Muller on uniforms in (0, 1] (DESIGN.md §3.5d).
 * Each of initialize, predict and update is one draw call: a predict draws with call index `counter`, the
 * update of the same launch with counter + 1, an update-only launch with `counter`.  The caller advances
 * the counter by the number of draws of each launch.  A correlated draw is L xi with L L' = C lower, C's
 * Cholesky factor in which a pivot <= 16 n eps max(diag C) zeroes its column (rank-deficient C, C = 0).
 * status[f] = BKE_STATUS_NOT_PD when Q, R or the P of initialize is clearly indefinite (the reference's
 * multivariate_normal only warns) and BKE_STATUS_SINGULAR_S when S is singular; the filter then keeps the
 * state it had before the failing half.  z_valid[f] == 0 skips the update of filter f (no draws, members,
 * x and P unchanged).  x_out / P_out may alias x / P and sigmas_out may alias sigmas. */
typedef struct bke_enkf_args {
    int64_t n_filters;
    int32_t dim_x, dim_z;            /* dim_x <= 16 */
    int32_t n_members;               /* >= 2 */
    int32_t dtype;
    uint32_t flags;                  /* BKE_DO_PREDICT | BKE_DO_UPDATE */
    int32_t fx_model, hx_model;
    uint32_t seed, counter;          /* noise key and the draw-call index of the launch's first draw */
    uint32_t reserved;
    double dt;
    const void *x, *P;
    void *x_out, *P_out;
    const void *sigmas;              /* [N,n_members,n] in */
    void *sigmas_out;                /* [N,n_members,n] out */
    const void *Q; int64_t Q_stride;
    const void *R; int64_t R_stride;
    const void *F; int64_t F_stride; /* BKE_FX_LINEAR only */
    const void *H; int64_t H_stride; /* BKE_HX_LINEAR only */
    const void *z;
    const uint8_t *z_valid;
    void *x_prior, *P_prior;
    void *K, *S, *SI;
    int32_t *status;
} bke_enkf_args;

/* initialize (:206): sigmas[f, i] = x[f] + L_P xi_i with draw call `counter`; x and P are not changed.
 * 1 <= dim_x <= 16.  status[N] (may be NULL): BKE_STATUS_NOT_PD for a clearly indefinite P, whose members
 * are then all x[f]. */
int bke_enkf_initialize(int64_t n_filters, int32_t dim_x, int32_t n_members, int32_t dtype, uint32_t seed, uint32_t counter,
                        const void *x, const void *P, void *sigmas, int32_t *status, void *stream);
int bke_enkf_step(const bke_enkf_args *args, void *stream);

/* User-supplied fx / hx for the EnKF (the reference calls fx(s, dt) and hx(s), :251, :280): source text,
 * include_dirs and args vectors as for bke_ukf_model_compile / bke_ukf_step_model.  The handle is a
 * bke_ukf_model built for the EnKF kernel; the UKF and CKF step calls refuse it and bke_enkf_step_model
 * refuses theirs (BKE_ERR_BAD_ARG). */
int bke_enkf_model_compile(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, const char *source,
                           const char *include_dirs, bke_ukf_model **out);
int bke_enkf_step_model(const bke_enkf_args *args, const bke_ukf_model *model, const void *fx_args, int64_t fx_args_stride,
                        const void *hx_args, int64_t hx_args_stride, void *stream);
size_t bke_debug_enkf_model_cubin_bytes(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model,
                                        const char *source, const char *include_dirs);

/* ------------------------------------------------------------------------------------------
 * Square-root Kalman filter bank.
 * Replaces SquareRootKalmanFilter.predict / update (filterpy/kalman/square_root.py:226-248, 172-224) for N
 * filters at once.  The state is x[N,n] and the lower-triangular factor L[N,n,n] of P = L L' (P1_2), stored
 * dense with explicit zeros above the diagonal; Lq[N,n,n] and Lr[N,m,m] are the factors of Q and R (Q1_2,
 * R1_2).  Per filter, in this order (flags = BKE_DO_PREDICT | BKE_DO_UPDATE):
 *   x <- F x (+ B u);  R~ = qr([F L | Lq]')[1] (2n x n);  L <- R~[:n,:n]'                   [x_prior, L_prior]
 *   M = [[Lr', 0], [(H L)', L']];  r = qr(M)[1];  S1_2 = r[:m,:m]';  SI1_2 = S1_2^-1;
 *   K = r[:m,m:]' SI1_2;  y = z - H x;  x <- x + K y;  L <- r[m:,m:]'
 * The QR is LAPACK's dgeqr2 (what scipy.linalg.qr runs at these sizes), with its signs: a column whose
 * sub-column is exactly zero is left as it is (tau = 0), otherwise its diagonal becomes
 * -copysign(norm, alpha).  So L itself, not only L L', is the reference's.  Lr is read as the full matrix
 * (update(z, R2) passes any square root); L and Lq as well.
 * Deviation: the reference inverts S1_2 with pinv.  Here a zero diagonal entry of S1_2 sets status[f] =
 * BKE_STATUS_SINGULAR_S, K = 0, SI1_2 = 0, and the posterior is the prior.  For S1_2 = 0 (e.g. H = 0 with
 * Lr = 0) that is the reference's result; for a partially singular S1_2 pinv would give a non-zero gain.
 * z_valid[i] == 0 means "z is None" for filter i (:189-193): x and L are not changed and the optional update
 * outputs of that filter are not written.  Optional outputs (NULL = not wanted): x_prior, L_prior (written by
 * a predict), K[N,n,m], y[N,m], S1_2[N,m,m], SI1_2[N,m,m], status[N].  x_out / L_out may alias x / L.
 * Kernels (picked by shape, DESIGN.md §3.5c): a register tile per thread for 1/1, 2/2, 3/1, 4/1 and 4/2
 * without control input, a warp per filter for every other shape. */
typedef struct bke_srkf_args {
    int64_t n_filters;
    int32_t dim_x, dim_z, dim_u;     /* dim_u may be 0 */
    int32_t dtype;
    uint32_t flags;                  /* BKE_DO_PREDICT | BKE_DO_UPDATE */
    uint32_t reserved;
    const void *x, *L;               /* in  */
    void *x_out, *L_out;             /* out */
    const void *F; int64_t F_stride;
    const void *H; int64_t H_stride;
    const void *Lq; int64_t Lq_stride;
    const void *Lr; int64_t Lr_stride;
    const void *B; int64_t B_stride; /* [N,n,dim_u] or NULL */
    const void *u; int64_t u_stride; /* [N,dim_u]   or NULL */
    const void *z;                   /* [N,m]; may be NULL when BKE_DO_UPDATE is not set */
    const uint8_t *z_valid;          /* [N] or NULL */
    void *x_prior, *L_prior;
    void *K, *y, *S1_2, *SI1_2;
    int32_t *status;
} bke_srkf_args;

int bke_srkf_step(const bke_srkf_args *args, void *stream);

/* The setters' factorisation: L[N,k,k] = scipy.linalg.cholesky(A, lower=True) per filter
 * (square_root.py:288, :314, :330).  Only the lower triangle of A is read; L is written dense with zeros
 * above the diagonal.  A[f] is at A + f * stride (stride 0: one matrix for every filter, k*k: per filter).
 * status[N] (may be NULL) = BKE_STATUS_NOT_PD where cholesky would raise LinAlgError.
 * k = 1 .. BKE_CHOLESKY_MAX_DIM (BKE_ERR_UNSUPPORTED above). */
#define BKE_CHOLESKY_MAX_DIM 16
int bke_cholesky_lower(int64_t n_filters, int32_t k, int32_t dtype, const void *A, int64_t stride, void *L,
                       int32_t *status, void *stream);

/* ------------------------------------------------------------------------------------------
 * Information filter bank.
 * Replaces InformationFilter.predict / update (filterpy/kalman/information_filter.py:245-289, 178-243) for N
 * filters at once.  The state is x[N,n], the information matrix P_inv[N,n,n] and the flag no_information[N]
 * (uint8, read and written; 0 at construction).  The models are F, F_inv (inv(F) as the F setter last
 * computed it: an in-place edit of F does not refresh it), Q[n,n], H[m,n], R_inv[m,m] and B / u, each per
 * filter or shared (stride 0).  Per filter, in this order (flags = BKE_DO_PREDICT | BKE_DO_UPDATE):
 *   predict  A = F_inv' P_inv F_inv.  A invertible:  if no_information: x <- inv(P_inv) x (0 x when P_inv is
 *            singular), no_information <- 0;  x <- F x (+ B u);  P_inv <- inv(inv(A) + Q)     [x_prior, P_inv_prior]
 *            A singular:  no_information <- 1;  FTI = inv(F');  AQI = inv(A + Q);
 *            x <- FTI ((I - P_inv F_inv) AQI) (FTI x);  P_inv unchanged                 [x_prior, P_inv_prior = AQI]
 *   update   no_information set:  x <- P_inv x + H' R_inv z;  P_inv <- P_inv + H' R_inv H;
 *                                  log_likelihood = log(DBL_MIN); y, K, S unchanged
 *            otherwise:  y = z - H x;  S = P_inv + H' R_inv H (n x n);  K = inv(S) H' R_inv;  x <- x + K y;
 *                        P_inv <- S;  log_likelihood per ll_mode (BKE_IF_LL_*)
 * "inv fails" is a pivot of the partially pivoted elimination that is exactly zero (LAPACK's dgetrf2
 * decision for n = 2 in the register tile).  A singular A is a branch.  A singular inv(A) + Q, F', A + Q
 * or S is where the reference's np.linalg.inv raises: status[f] = BKE_STATUS_SINGULAR_S and the filter stops there with what the
 * reference has set by then (a failed predict keeps P_inv, skips the update and writes no prior; a failed
 * update keeps x and P_inv and writes y and S but not K).
 * z_valid[i] == 0 means "z is None" (:194-198): nothing of that filter changes in the update.  Optional
 * outputs (NULL = not wanted): x_prior, P_inv_prior (written by a predict), K[N,n,m], y[N,m], S[N,n,n],
 * log_likelihood[N], status[N] (only written on failure with BKE_STATUS_STICKY).  x_out / P_inv_out may
 * alias x / P_inv.  ll_mode other than BKE_IF_LL_NONE needs log_likelihood and the m it names.
 * Kernels (picked by shape, DESIGN.md §3.5e): a register tile per thread for 1/1, 2/1, 2/2, 3/1, 4/1, 4/2,
 * 4/4 and (fp32) 6/3 without control input, a warp per filter for every other shape. */
#define BKE_IF_LL_NONE 0             /* log_likelihood is not computed by an informed update */
#define BKE_IF_LL_FULL 1             /* m == n: log N(y; 0, S) (stats.py logpdf, information_filter.py:235) */
#define BKE_IF_LL_BROADCAST 2        /* m == 1: log N([y, .., y]; 0, S), scipy's broadcast of y over n */
typedef struct bke_if_args {
    int64_t n_filters;
    int32_t dim_x, dim_z, dim_u;     /* dim_u may be 0 */
    int32_t dtype;
    uint32_t flags;                  /* BKE_DO_PREDICT | BKE_DO_UPDATE | BKE_STATUS_STICKY */
    int32_t ll_mode;                 /* BKE_IF_LL_* */
    const void *x, *P_inv;           /* in  */
    void *x_out, *P_inv_out;         /* out */
    uint8_t *no_information;         /* [N], read and written */
    const void *F; int64_t F_stride;
    const void *F_inv; int64_t F_inv_stride;
    const void *Q; int64_t Q_stride;
    const void *H; int64_t H_stride;
    const void *R_inv; int64_t R_inv_stride;
    const void *B; int64_t B_stride; /* [N,n,dim_u] or NULL */
    const void *u; int64_t u_stride; /* [N,dim_u]   or NULL */
    const void *z;                   /* [N,m]; may be NULL when BKE_DO_UPDATE is not set */
    const uint8_t *z_valid;          /* [N] or NULL */
    void *x_prior, *P_inv_prior;
    void *K, *y, *S, *log_likelihood;
    int32_t *status;
} bke_if_args;

int bke_if_step(const bke_if_args *args, void *stream);

/* np.linalg.inv per filter, for the InformationFilter's F setter (F_inv) and P property:
 * Ai[N,k,k] = inv(A[f]), A[f] at A + f * stride (stride 0: one matrix for every filter, k*k: per filter).
 * status[N] (may be NULL) = BKE_STATUS_SINGULAR_S where a pivot is exactly zero (Ai is then undefined).
 * k >= 1; BKE_ERR_UNSUPPORTED when a k x k pair does not fit a warp's shared memory. */
int bke_inverse(int64_t n_filters, int32_t k, int32_t dtype, const void *A, int64_t stride, void *Ai,
                int32_t *status, void *stream);

/* ------------------------------------------------------------------------------------------
 * Polynomial tracker banks: the g-h family, the expanding-memory least-squares filter and the fading-memory
 * filter, n_steps epochs of N filters in one launch (one thread per filter, the time loop inside the kernel).
 *   BKE_POLY_GH        GHFilter.update / batch_filter        filterpy/gh/gh_filter.py:363-377, 421-455
 *   BKE_POLY_GHK       GHKFilter.update / batch_filter       gh_filter.py:659-680, 717-748
 *   BKE_POLY_GH_ORDER  GHFilterOrder.update, order 0..2      gh_filter.py:142-181
 *   BKE_POLY_LSQ       LeastSquaresFilter.update, order 0..2 filterpy/leastsq/least_squares.py:122-155
 *   BKE_POLY_FADING    FadingMemoryFilter.update, order 0..2 filterpy/memory/fading_memory.py:164-194
 * State: GH / GHK keep x[N], dx[N] (and ddx[N] for GHK; order is ignored); the others keep x[N, order+1].
 * mode BKE_POLY_UPDATE runs n_steps calls of update() on z[t, :] and writes the state back (LSQ: n[N] and K
 * [N, order+1] too).  mode BKE_POLY_BATCH reads the state and leaves it alone: GH and GHK run batch_filter's
 * recursion (GHKFilter.batch_filter is GHFilter's: k and ddx are not read), the others run update()'s.
 * Parameters, each per filter (stride 1) or shared (stride 0), in the state's dtype.  Every constant the
 * reference derives from its scalars is computed by the caller with the reference's expression:
 *   g    GH, GHK, GH_ORDER: g                      FADING: G (1 - beta, 1 - beta**2, 1 - beta**3 by order)
 *   h    GH, GHK, GH_ORDER 1-2 (update): h         GH, GHK (batch): h / dt      FADING 1-2: H / dt
 *   k    GHK (update), GH_ORDER 2: k               FADING 2: 2*K / dt**2
 *   dt   every family but the order-0 filters
 *   dt2  dt**2: GHK (update), GH_ORDER 2, LSQ 2, FADING 2
 *   hdt2 0.5 * dt**2: LSQ 2
 * A parameter the instance does not read may be NULL.  LSQ reads and advances n[N] (int64; its gains come from
 * the counter by exact int64 arithmetic and round-to-nearest conversions, as Python's do); n_max is an upper
 * bound of n[] on entry, and the call is refused when the counter's products (n, n(n+1), n(n+1)(n+2) for
 * order 0, 1, 2) could overflow int64 within n_steps.
 * Optional outputs (NULL = not wanted):
 *   results[T+1, N, W]   the state before the first and after every epoch: W = 2 (x, dx) for GH / GHK,
 *                        order+1 otherwise
 *   predictions[T, N]    batch_filter's x_est: GH / GHK batch only
 *   y[N]                 the last residual: GH, GHK, GH_ORDER update only
 *   x_prediction, dx_prediction [N]: GH / GHK update;  ddx_prediction[N]: GHK update
 *   K[N, order+1]        the last gains: LSQ update only
 * An output the family and mode do not have is refused with BKE_ERR_BAD_ARG. */
#define BKE_POLY_GH 0
#define BKE_POLY_GHK 1
#define BKE_POLY_GH_ORDER 2
#define BKE_POLY_LSQ 3
#define BKE_POLY_FADING 4
#define BKE_POLY_UPDATE 0
#define BKE_POLY_BATCH 1
typedef struct bke_poly_args {
    int64_t n_filters;
    int64_t n_steps;                 /* T >= 1 */
    int32_t family, order;           /* BKE_POLY_*; order 0..2 (GH_ORDER, LSQ, FADING) */
    int32_t dtype;
    int32_t mode;                    /* BKE_POLY_UPDATE or BKE_POLY_BATCH */
    void *x, *dx, *ddx;              /* read, and written by BKE_POLY_UPDATE */
    const void *g; int64_t g_stride;
    const void *h; int64_t h_stride;
    const void *k; int64_t k_stride;
    const void *dt; int64_t dt_stride;
    const void *dt2; int64_t dt2_stride;
    const void *hdt2; int64_t hdt2_stride;
    int64_t *n;                      /* LSQ: [N] */
    int64_t n_max;                   /* LSQ: max(n) on entry */
    const void *z;                   /* [T, N] */
    void *results, *predictions, *y;
    void *x_prediction, *dx_prediction, *ddx_prediction;
    void *K;
} bke_poly_args;

int bke_poly_filter(const bke_poly_args *args, void *stream);

/* ------------------------------------------------------------------------------------------
 * Measurement scoring: N tracks against K candidates each, without stepping anything.  Replaces, per pair:
 *   stats.mahalanobis(z, mean, S)                 filterpy/stats/stats.py:64-109
 *   stats.log_likelihood / likelihood(z, x, P, H, R)   stats.py:112-128 (S = H P H' + R)
 *   stats.logpdf(z, mean, S)                      stats.py:131-154
 *   stats.NEES(xs, est_xs, ps)                    stats.py:1138-1179 (d2 with z = xs, mean = est_xs, S = ps)
 *   KalmanFilter.log_likelihood_of / residual_of / measurement_of_state   kalman_filter.py:1252-1260, 1175-1201
 * Per track i, once:  zhat = H x (x when H is NULL), or the given mean;  S = H P H' + R (P + R when H is NULL),
 * or the given S;  SI = S^-1 and log|det S| by the step kernels' inverse (a zero pivot of the partially pivoted
 * elimination is a singular S).  Per pair (i, k), with z_ik at z + i * z_track_stride + k * z_cand_stride:
 *   y = z_ik - zhat;  d2 = y' SI y;  mahalanobis = sqrt(d2);  log_likelihood = -0.5 (d2 + log|det S| + m log 2pi);
 *   likelihood = exp(log_likelihood) (no floor, as stats.likelihood)
 * A pair with z_valid == 0 is "z is None": y = d2 = mahalanobis = 0, log_likelihood = log(DBL_MIN)
 * (kalman_filter.py:1258-1259, 515-520), whatever S is.  Where S is singular, status[i] = BKE_STATUS_SINGULAR_S and
 * the track's valid pairs get NaN in d2, mahalanobis, log_likelihood and likelihood (y is still written).
 * Inputs: exactly one of x[N,n] and mean[N,m]; at most one of P[N,n,n] (with R) and S; H and R with x or P only.
 * H, R and S are per track (stride m*n, m*m) or shared (stride 0); z's strides are any element strides >= 0
 * ([N,K,m]: K*m and m;  one scan [K,m] shared by every track: 0 and m).  dim_x is not read when neither x nor P
 * is given.  Outputs (NULL = not wanted, at least one): zhat[N,m], y[N,K,m], d2, mahalanobis, log_likelihood,
 * likelihood [N,K], status[N].  The covariance is needed by every output but zhat and y, z by every output but
 * zhat and status.  N = 0 or K = 0 launches nothing (zhat and status are then not written either).  The call allocates
 * nothing, so it can be captured.
 * Kernels (DESIGN.md §3.5g): a CTA per tile of tracks computes each track's zhat, SI and log|det S| into shared
 * memory (a register tile per thread for the shapes 1/1, 2/1, 2/2, 3/1, 3/3, 4/1, 4/2, 4/4 and 6/3, a warp per
 * track otherwise), then sweeps the tile's N_tile * K pairs with its threads in pair order. */
typedef struct bke_score_args {
    int64_t n_tracks;                /* N */
    int64_t n_candidates;            /* K */
    int32_t dim_x, dim_z;            /* n, m */
    int32_t dtype;
    int32_t reserved;
    const void *x;                   /* [N,n] or NULL */
    const void *mean;                /* [N,m] or NULL */
    const void *P;                   /* [N,n,n] or NULL */
    const void *S; int64_t S_stride; /* [N,m,m] or NULL */
    const void *H; int64_t H_stride; /* [N,m,n] or NULL = identity (n == m) */
    const void *R; int64_t R_stride; /* [N,m,m]; with P only */
    const void *z; int64_t z_track_stride, z_cand_stride;
    const uint8_t *z_valid;          /* [N,K] or NULL */
    void *zhat, *y, *d2, *mahalanobis, *log_likelihood, *likelihood;
    int32_t *status;
} bke_score_args;

int bke_score_measurements(const bke_score_args *args, void *stream);

/* Measurement scoring against UKF banks: N tracks against K candidates each, without stepping anything.  Per
 * track i and candidate z_ik, what UnscentedKalmanFilter reports as log_likelihood and mahalanobis right after
 * update(z_ik) from the track's current (x, P) (UKF.py:459-477, 742-777):
 *   sigma points of (x, P) (Merwe, or the simplex set with BKE_UKF_SIMPLEX: UKF.py:407);  Zs = hx(Xs);
 *   (zhat, S) = UT(Zs, Wm, Wc, R) with z_mean_fn / residual_z where a run-time model has them;
 *   y = residual_z(z_ik, zhat);  d2 = y' S^-1 y;  mahalanobis = sqrt(d2);
 *   log_likelihood = -0.5 (d2 + log|det S| + m log 2pi);  likelihood = exp(log_likelihood)
 * with S^-1 and log|det S| from the step kernels' inverse.  Every field shared with bke_score_args has its meaning,
 * shape and NULL rule there: a pair with z_valid == 0 scores y = d2 = mahalanobis = 0 and log(DBL_MIN); a singular S
 * is status[i] = BKE_STATUS_SINGULAR_S and a P whose Cholesky fails BKE_STATUS_NOT_PD, and the track's valid pairs
 * then get NaN scores.  x[N,n], P[N,n,n], R[N,m,m] (stride m*m or 0) and, for BKE_HX_LINEAR, H (stride m*n or 0)
 * are read and nothing else is touched.  hx_model is one of the pre-built models (BKE_HX_*, in the dim_x / dim_z
 * instances bke_ukf_step has); bke_ukf_score_model runs a handle of bke_ukf_model_compile[_hooks|_points] (its
 * dim_x, dim_z, dtype, hx_model and point set must match; hx_args as for bke_ukf_step_model) and refuses a CKF or
 * EnKF handle.  A CTA of 128 tracks holds the hx of their sigma points and 128 slots of m + m^2 + 1 words in shared
 * memory: the pre-built instances need 2.5-73 KB; a run-time model whose score needs more than 227 KB (large dim_z,
 * e.g. dim_x = 4, dim_z = 12 in fp64: 265 KB, where the step needs 118 KB) returns BKE_ERR_UNSUPPORTED from
 * bke_ukf_score_model even where it can step.
 * N = 0 or K = 0 launches nothing.  The call allocates nothing, so it can be captured.
 * Kernel (DESIGN.md §3.5h): a CTA per tile of 128 tracks runs the step's measurement half into shared memory, then
 * sweeps the tile's pairs as bke_score_measurements does. */
typedef struct bke_ukf_score_args {
    int64_t n_filters;               /* N */
    int64_t n_candidates;            /* K */
    int32_t dim_x, dim_z;            /* n, m */
    int32_t dtype;
    uint32_t flags;                  /* 0 or BKE_UKF_SIMPLEX */
    int32_t hx_model;
    int32_t reserved;
    double alpha, beta, kappa;       /* MerweScaledSigmaPoints(n, alpha, beta, kappa); ignored with BKE_UKF_SIMPLEX */
    const void *x, *P;               /* [N,n], [N,n,n] */
    const void *R; int64_t R_stride; /* [N,m,m] */
    const void *H; int64_t H_stride; /* [N,m,n]; BKE_HX_LINEAR only */
    const void *z; int64_t z_track_stride, z_cand_stride;
    const uint8_t *z_valid;          /* [N,K] or NULL */
    void *zhat, *y, *d2, *mahalanobis, *log_likelihood, *likelihood;
    int32_t *status;
} bke_ukf_score_args;

int bke_ukf_score(const bke_ukf_score_args *args, void *stream);
int bke_ukf_score_model(const bke_ukf_score_args *args, const bke_ukf_model *model, const void *hx_args, int64_t hx_args_stride,
                        void *stream);
/* A handle compiles its score kernel (NVRTC, its own program) on its first bke_ukf_score_model call with N, K > 0; make
 * that call before capturing one.  The NVRTC half alone (needs no GPU): cubin size of that program, 0 on failure. */
size_t bke_debug_ukf_score_model_cubin_bytes(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model,
                                              uint32_t hooks, uint32_t points, const char *source, const char *include_dirs);

/* Stand-alone pieces of the unscented path for callers that use them directly:
 *   MerweScaledSigmaPoints.sigma_points(x, P)   filterpy/kalman/sigma_points.py:124-177
 *       x[N,n], P[N,n,n] -> sigmas[N,2n+1,n]; status[N] = BKE_STATUS_NOT_PD where scipy's cholesky
 *       would raise (only the upper triangle of P is read, as scipy does);
 *   unscented_transform(sigmas, Wm, Wc, noise_cov)   filterpy/kalman/unscented_transform.py:22-128
 *       sigmas[N,k,n], Wm[k], Wc[k], noise_cov[n,n] (noise_stride 0) / [N,n,n] (n*n) / NULL
 *       -> x_out[N,n], P_out[N,n,n]   (default mean / residual functions). */
int bke_merwe_sigma_points(int64_t n_filters, int32_t dim_x, int32_t dtype, double alpha, double beta, double kappa,
                           const void *x, const void *P, void *sigmas, int32_t *status, void *stream);
/*   SimplexSigmaPoints.sigma_points(x, P)   filterpy/kalman/sigma_points.py:454-513
 *       x[N,n], P[N,n,n] -> sigmas[N,n+1,n] (Xi_0 .. Xi_n); bounds and status as bke_merwe_sigma_points. */
int bke_simplex_sigma_points(int64_t n_filters, int32_t dim_x, int32_t dtype, const void *x, const void *P, void *sigmas,
                             int32_t *status, void *stream);
int bke_unscented_transform(int64_t n_filters, int32_t n_sigmas, int32_t dim, int32_t dtype, const void *sigmas,
                            const void *Wm, const void *Wc, const void *noise_cov, int64_t noise_stride,
                            void *x_out, void *P_out, void *stream);

/* ------------------------------------------------------------------------------------------
 * Particle resampling.
 * Replaces systematic_resample(weights) / stratified_resample(weights)
 * (filterpy/monte_carlo/resampling.py:117-150 / :80-114).  indexes[i] = number of j with
 * cumsum(weights)[j] <= positions[i], where cumsum is the strictly sequential fp64
 * accumulation np.cumsum performs (:142) — reproduced bit for bit, not approximated — and
 * positions[i] = (u + i) / N  (systematic, :139)  or  (U[i] + i) / N  (stratified, :103).
 * The uniforms are drawn by the caller (the reference uses the global NumPy RandomState).
 *
 *   weights[N] fp64, indexes[N] int32 (np.zeros(N, 'i'), :141)
 *   info[8] int32 (device, optional): [0] overflow = number of positions >= cumsum[-1]
 *       (the reference raises IndexError there, :145; such outputs are set to N-1),
 *       [1] 1 if the weights held a negative / non-finite entry and the literal sequential
 *       kernel was used, [2] number of binade-crossing tiles, [3] number of long runs.
 *   cumsum_last (device double, optional): cumsum(weights)[-1] as the reference would see it.
 *       [5] tiles walked sequentially, [6] outputs that did not fit `capacity` (shards),
 *       [7] tiles that needed the general (tie / raw element) path.
 */
size_t bke_resample_workspace_bytes(int64_t n);

int bke_systematic_resample(int64_t n, const double *weights, double u, int32_t *indexes,
                            void *workspace, size_t workspace_bytes,
                            int32_t *info, double *cumsum_last, void *stream);

int bke_stratified_resample(int64_t n, const double *weights, const double *uniforms,
                            int32_t *indexes, void *workspace, size_t workspace_bytes,
                            int32_t *info, double *cumsum_last, void *stream);

/* Fused normalise + resample: S = sum(weights) (tree order, written to sum_out), then the resampling
 * passes on w / S — systematic_resample(weights / S) (resampling.py:117-150; stratified when
 * `uniforms` != NULL, :80-114).  Every pass that reads the weights divides them by S as it reads them
 * (IEEE division, what NumPy's `w / w.sum()` computes given S): the sum and passes A, C and E read the
 * un-normalised weights.  No normalised array is written unless weights_out (optional) is given; it
 * then receives w / S.  info and cumsum_last as for bke_systematic_resample, on w / S. */
int bke_resample_normalized(int64_t n, const double *weights, double u, const double *uniforms,
                            int32_t *indexes, double *weights_out, double *sum_out,
                            void *workspace, size_t workspace_bytes,
                            int32_t *info, double *cumsum_last, void *stream);

/* One contiguous SHARD of a particle set that is spread over several GPUs (rank r holds particles
 * [j_offset, j_offset + n_local) of n_global).  The result equals the single-array call bit for
 * bit: shard r produces exactly the indexes of the global output positions
 * [out_range[0], out_range[1]) — those whose position falls into this shard's span of the
 * cumulative sum — with GLOBAL particle numbers, written to indexes[0 .. out_end - out_begin).
 *   phase bit 1 (passes A-C; independent on every rank) needs `carry_approx`: the approximate
 *           (tree-ordered, all-gathered) sum of all earlier shards, device double;
 *   phase bit 2 (exact chain) needs `carry_exact`: the exact running sum the previous rank's chain
 *           wrote to its `carry_out` (device double; NULL on rank 0) and writes this shard's
 *           `carry_out` — the only serial dependency between ranks;
 *   phase bit 4 (emit, long runs, info) can run after the hand-off has been sent on.
 *   Everything is stream-ordered, no host sync.
 * `uniforms` (stratified) is the GLOBAL uniform array [n_global], replicated; NULL = systematic.
 * `is_last` = 1 on the shard holding the end of the set (positions beyond the last cumulative sum
 * are then reported in info[0] and filled with n_global - 1, as in the single-array call). */
typedef struct bke_resample_shard_args {
    int64_t n_local, n_global, j_offset, capacity;
    const double *weights;
    const double *uniforms;
    double u;
    const double *carry_approx;
    const double *carry_exact;
    int32_t *indexes;
    int64_t *out_range;          /* device int64[2] */
    double *carry_out;           /* device double */
    void *workspace; size_t workspace_bytes;
    int32_t *info;               /* device int32[8] or NULL */
    int32_t is_last;
    int32_t phase;               /* bit mask of 1, 2, 4 (7 = everything); 8 with 1: the header reset and pass A
                                    have already run (bke_resample_shard_stage) */
} bke_resample_shard_args;

int bke_resample_shard(const bke_resample_shard_args *args, void *stream);

/* Multi-GPU without a serial hand-over: after phase 1 every rank summarises its shard as a
 * COMPOSITE — the ordered list of parity maps and true adds that takes the exact running sum from
 * the start of the shard to its end (it depends on the approximate carry only) — of
 * bke_resample_composite_bytes() bytes.  The ranks all-gather their composites (NCCL), and
 * bke_resample_compose_carry applies those of the n_shards_before earlier shards, in order, to 0:
 * the exact carry of this rank, on the device, to be passed as `carry_exact` of phases 2 and 4.
 * *status != 0: a composite could not be formed (a dense zone of tiny weights next to a binade
 * boundary) — use the rank-to-rank hand-over of `carry_out` instead. */
size_t bke_resample_composite_bytes(void);

/* The same sequence with one call per exchange (what filterpy_b200.distributed.ShardedResamplePlan
 * issues; everything stream-ordered):
 *   stage 1  header reset, pass A, this shard's approximate sum -> *shard_sum_out
 *            [ all-gather shard_sum_out -> shard_sums_all ]
 *   stage 2  approximate carry = shard_sums_all[0] + ... + shard_sums_all[shard_rank - 1], passes B
 *            and C, the shard's composite -> composite_out
 *            [ all-gather composite_out -> composites_all ]
 *   stage 3  exact carry from composites_all (*compose_status != 0: see above), exact chain, emit.
 * `carry_approx` / `carry_exact` of `args` are ignored (the two scratch doubles of `ext` are used). */
typedef struct bke_resample_shard_ext {
    double *shard_sum_out;
    const double *shard_sums_all;
    void *composite_out;
    const void *composites_all;
    double *carry_approx_buf;
    double *carry_exact_buf;
    int32_t *compose_status;
    int32_t shard_rank, n_shards;
} bke_resample_shard_ext;
int bke_resample_shard_stage(const bke_resample_shard_args *args, const bke_resample_shard_ext *ext,
                             int32_t stage, void *stream);
int bke_resample_shard_compose(const bke_resample_shard_args *args, void *composite_out, void *stream);
int bke_resample_compose_carry(int32_t n_shards_before, const void *composites, double *carry_exact,
                               int32_t *status, void *stream);

/* A BANK of independent particle sets in one launch: row b of weights[n_sets, n_particles] (fp64, dense)
 * is one set, and row b of indexes[n_sets, n_particles] (int32) is, bit for bit, what the reference's
 * systematic_resample / stratified_resample returns for that row (resampling.py:141-149 / :105-113,
 * literally, for ANY values: negative, NaN, infinite, -0.0 and subnormal weights, and any u / uniforms,
 * including values outside [0, 1) and out of order) with positions
 *   (u[b] + arange(M)) / M          systematic, u[n_sets]               (:139)
 *   (uniforms[b] + arange(M)) / M   stratified, uniforms[n_sets, M]     (:103)
 * Give exactly one of u and uniforms.  status[b] (optional) = 1 where the positions run past
 * cumsum(weights[b])[-1] (the reference's IndexError, :145; that row's indexes are unspecified), else 0.
 * n_sets = 0 or n_particles = 0 does nothing; n_particles < 2^31.  No workspace, no allocation, no host
 * sync: the call can be captured in a CUDA graph. */
typedef struct bke_resample_bank_args {
    int64_t n_sets, n_particles;
    const double *weights;       /* [n_sets, n_particles] */
    const double *u;             /* [n_sets] (systematic) or NULL */
    const double *uniforms;      /* [n_sets, n_particles] (stratified) or NULL */
    int32_t *indexes;            /* [n_sets, n_particles] */
    int32_t *status;             /* [n_sets] or NULL */
} bke_resample_bank_args;

int bke_resample_bank(const bke_resample_bank_args *args, void *stream);

/* One particle-filter epoch of a bank, resampling only the sets that degenerated.  For every row b of
 * weights[n_sets, n_particles] (fp64, dense), independently:
 *   1. w_b <- w_b / np.sum(w_b), in place, with NumPy's pairwise summation order;
 *   2. neff[b] = 1. / np.sum(np.square(w_b)) over the normalised row (pairwise again);
 *   3. resampled[b] = neff[b] < threshold (strict; a NaN neff does not resample);
 *   4. where resampled[b]: indexes[b] is systematic_resample(w_b) for u[b] or stratified_resample(w_b) for
 *      uniforms[b], exactly as bke_resample_bank computes it; particles[b] <- particles[b][indexes[b]] in
 *      place; weights[b] <- 1. / n_particles everywhere;
 *   5. status[b] = 1 where the positions run past the normalised row's cumsum (the reference's IndexError,
 *      resampling.py:145): that row keeps its particles and its normalised weights.  Otherwise 0.
 * Rows that do not resample have their particles neither read nor written, and their indexes are
 * unspecified.  Give exactly one of u and uniforms; only the rows of resampled sets are read.
 *
 * A particle is particle_bytes bytes of any type.  A set's particle row (n_particles * particle_bytes) is
 * staged in one CTA's shared memory, so it must not exceed the device's opt-in shared memory per block
 * (227 KB on the H100); a larger row returns BKE_ERR_BAD_ARG.  n_sets < 2^31, n_particles < 2^31;
 * n_sets = 0 or n_particles = 0 does nothing.
 *
 * workspace: bke_resample_bank_gated_workspace_bytes(n_sets) bytes, 4-byte aligned; it holds the list of
 * sets to resample and its counter.  Three launches and a memset, no allocation, no host sync: the call
 * can be captured in a CUDA graph.  The two halves are callable on their own, in stream order on the same
 * args: _stats runs steps 1-3 (u / uniforms are not read, and may both be NULL), _apply runs steps 4-5 on
 * the sets _stats listed, so a caller can read `resampled` back and draw uniforms only for those sets. */
typedef struct bke_resample_bank_gated_args {
    int64_t n_sets, n_particles;
    double *weights;             /* [n_sets, n_particles] in: raw weights; out: normalised, or 1/M where resampled */
    const double *u;             /* [n_sets] (systematic) or NULL */
    const double *uniforms;      /* [n_sets, n_particles] (stratified) or NULL */
    double threshold;
    void *particles;             /* [n_sets, n_particles] particles of particle_bytes each, any type; in place */
    int64_t particle_bytes;
    int32_t *indexes;            /* [n_sets, n_particles] */
    double *neff;                /* [n_sets] */
    uint8_t *resampled;          /* [n_sets], 0 or 1 */
    int32_t *status;             /* [n_sets] */
    void *workspace;
    size_t workspace_bytes;
} bke_resample_bank_gated_args;

size_t bke_resample_bank_gated_workspace_bytes(int64_t n_sets);
int bke_resample_bank_gated(const bke_resample_bank_gated_args *args, void *stream);
int bke_resample_bank_gated_stats(const bke_resample_bank_gated_args *args, void *stream);
int bke_resample_bank_gated_apply(const bke_resample_bank_gated_args *args, void *stream);

/* multinomial_resample (resampling.py:153-176) of every row of weights[n_sets, n_particles] (fp64, dense):
 *   indexes[b] = np.searchsorted(c_b, uniforms[b]),  c_b = np.cumsum(weights[b]), c_b[-1] = 1
 * bit for bit for ANY values (negative, NaN, infinite, -0.0 and subnormal weights; uniforms outside [0, 1),
 * NaN or out of order), NumPy's bracket-carrying bisection included.  indexes are int64 like
 * np.searchsorted's.  status[b] = 0 where every key was bisected on its own (c_b is sorted), 2 where the set
 * took the carried-bracket search; bit 0 is never set (multinomial cannot fail once n_particles > 0).
 * workspace: bke_multinomial_resample_bank_workspace_bytes(n_sets, n_particles) bytes, 8-byte aligned (it
 * holds c).  n_sets = 0 or n_particles = 0 does nothing; n_particles < 2^31.  No allocation, no host sync:
 * the call can be captured in a CUDA graph. */
typedef struct bke_multinomial_resample_bank_args {
    int64_t n_sets, n_particles;
    const double *weights;       /* [n_sets, n_particles] */
    const double *uniforms;      /* [n_sets, n_particles] */
    int64_t *indexes;            /* [n_sets, n_particles] */
    int32_t *status;             /* [n_sets] */
    void *workspace;
    size_t workspace_bytes;
} bke_multinomial_resample_bank_args;

size_t bke_multinomial_resample_bank_workspace_bytes(int64_t n_sets, int64_t n_particles);
int bke_multinomial_resample_bank(const bke_multinomial_resample_bank_args *args, void *stream);

/* residual_resample (resampling.py:27-76) of every row of weights[n_sets, n_particles], in two stream-ordered
 * calls on the same args, bit for bit for ANY weights (the sums in the reference's order, NumPy's
 * bracket-carrying bisection over the non-monotone cumulative sum):
 *   _prepare  reads weights; writes indexes[b, :k_b] = repeat(arange(M), max(floor(M w), 0)), n_copies[b] =
 *             k_b, cumsum(residual / sum(residual)) with [-1] = 1 into the workspace, and status[b]: 1 where
 *             k_b > M (the reference's IndexError, :61; that row's indexes are unspecified and n_copies[b] is
 *             some value > M), else 0 or 2 (2: the set takes the carried-bracket search, the usual case).
 *   _search   reads uniforms[b, :M - k_b] (the reference's random(M - k_b); the rest of the row is not
 *             read), n_copies, status and the workspace; writes indexes[b, k_b:] (int32); skips status-1 rows.
 * workspace: bke_residual_resample_bank_workspace_bytes(n_sets, n_particles) bytes, 8-byte aligned.  The
 * caller can read n_copies between the calls to draw exactly M - k_b uniforms per row.  n_sets = 0 or
 * n_particles = 0 does nothing; n_particles < 2^31.  No allocation, no host sync: graph-capturable. */
typedef struct bke_residual_resample_bank_args {
    int64_t n_sets, n_particles;
    const double *weights;       /* [n_sets, n_particles] (_prepare) */
    const double *uniforms;      /* [n_sets, n_particles] (_search) */
    int32_t *indexes;            /* [n_sets, n_particles] */
    int64_t *n_copies;           /* [n_sets]: k_b */
    int32_t *status;             /* [n_sets] */
    void *workspace;
    size_t workspace_bytes;
} bke_residual_resample_bank_args;

size_t bke_residual_resample_bank_workspace_bytes(int64_t n_sets, int64_t n_particles);
int bke_residual_resample_bank_prepare(const bke_residual_resample_bank_args *args, void *stream);
int bke_residual_resample_bank_search(const bke_residual_resample_bank_args *args, void *stream);

/* sum of weights (fp64, deterministic tree order) — the quantity that is all-reduced across
 * GPUs before a distributed resample; also used to normalise: weights_out[i] = weights[i] / sum
 * (IEEE division, the same elementwise operation as NumPy's `w / w.sum()` given that sum). */
int bke_weights_sum(int64_t n, const double *weights, double *sum_out, void *workspace,
                    size_t workspace_bytes, void *stream);
int bke_weights_scale(int64_t n, const double *weights, const double *divisor, double *weights_out,
                      void *stream);

/* ---- RTS smoother over batch_filter's outputs ---------------------------------------------------
 *
 * KalmanFilter.rts_smoother filterpy/kalman/kalman_filter.py:995-1074 and the procedural
 * rts_smoother :1792-1858 for a bank: Xs[T,N,n], Ps[T,N,n,n] are batch_filter's `means` and
 * `covariances`; outputs x_out[T,N,n], P_out[T,N,n,n], K[T,N,n,n], Pp[T,N,n,n] (K, Pp may be NULL).
 * The model of recursion step k is F[(k + model_shift) * F_step_stride + i * F_stride] — the method
 * uses Fs[k+1] (:1068, model_shift = 1), the procedural form Fs[k] (:1852, model_shift = 0);
 * step strides of 0 mean one model for every epoch, filter strides of 0 one model for the bank.
 * status[i] = BKE_STATUS_SINGULAR_S where np.linalg.inv(Pp) would raise. */
typedef struct {
    int64_t n_filters, n_steps;
    int32_t dim_x, dtype;
    int32_t model_shift, reserved;
    const void *Xs, *Ps;
    const void *F; int64_t F_stride, F_step_stride;
    const void *Q; int64_t Q_stride, Q_step_stride;
    void *x_out, *P_out, *K, *Pp;
    int32_t *status;
} bke_rts_args;

int bke_kf_rts_smoother(const bke_rts_args *args, void *stream);

/* UnscentedKalmanFilter.rts_smoother filterpy/kalman/UKF.py:634-739 for a bank; same layout as
 * bke_kf_rts_smoother.  Q is the filter's own Q (the reference never reads its Qs argument, :715);
 * dts is a DEVICE array of n_steps doubles (step k uses dts[k], :712) or NULL = dt for every step;
 * fx_model / F as in bke_ukf_args.  K may be NULL.  flags: 0 (Merwe points from alpha, beta, kappa) or
 * BKE_UKF_SIMPLEX (simplex points; alpha, beta, kappa ignored). */
typedef struct {
    int64_t n_filters, n_steps;
    int32_t dim_x, dtype, fx_model;
    uint32_t flags;
    double alpha, beta, kappa;
    double dt;
    const double *dts;
    const void *Xs, *Ps;
    const void *Q; int64_t Q_stride;
    const void *F; int64_t F_stride;
    void *x_out, *P_out, *K;
    int32_t *status;
} bke_ukf_rts_args;

int bke_ukf_rts_smoother(const bke_ukf_rts_args *args, void *stream);
/* the same around a user-supplied fx (fx_model = BKE_FX_USER, a model from bke_ukf_model_compile; dim_x <= 8), or
 * around any fx of a model from bke_ukf_model_compile_hooks (x_mean_fn / residual_x as UKF.py:720-735).  The
 * reference calls self.fx(sigma, dts[k]) WITHOUT keyword arguments here (UKF.py:712): fx_args are the values its
 * callable would default to. */
int bke_ukf_rts_smoother_model(const bke_ukf_rts_args *args, const bke_ukf_model *model, const void *fx_args,
                               int64_t fx_args_stride, void *stream);

/* ---- bank-level model mixing: IMMEstimator / MMAEFilterBank -----------------------------------
 *
 * N tracks, each followed by the same n_models filters; model j's states are the bank arrays
 * x[j][N,n], P[j][N,n,n] (dtype), its per-track log-likelihoods log_likelihood[j][N] (dtype, what
 * bke_kf_step writes).  mu[N,M], cbar[N,M], omega[N,M,M], trans[M,M] are fp64.
 *   bke_mm_probabilities  filterpy/kalman/IMM.py:178-184 and :239-247: mu = cbar * L, normalised;
 *                         cbar = mu . trans; omega[i,j] = trans[i,j] mu[i] / cbar[j], with
 *                         L = exp(log_likelihood) floored at DBL_MIN (kalman_filter.py:1213-1223).
 *                         With BKE_MM_MMAE: mu = mu * L, normalised (filterpy/kalman/mmae.py:180-184).
 *   bke_mm_mix            IMM.py:201-213: x_out[i], P_out[i] = mixed initial conditions of model i
 *                         from omega (weights_stride = M*M per track, 0 = one omega for the bank).
 *   bke_mm_estimate       IMM.py:228-237: x_out[0], P_out[0] = combined estimate from mu
 *                         (weights_stride = M per track, 0 = shared).  With BKE_MM_MMAE the covariance
 *                         follows mmae.py:197-199 literally: term j uses y = x_j - x[j] (component j of
 *                         the mixed state, a scalar) and only min(dim_x, M) terms are summed.
 * Outputs must not alias inputs. */
#define BKE_MM_MAX_MODELS 8
#define BKE_MM_MMAE 1u
#define BKE_MM_FROM_MU 2u   /* bke_mm_probabilities: keep mu as given (no likelihood step), only cbar and omega */
typedef struct {
    int64_t n_tracks;
    int32_t dim_x, n_models, dtype;
    uint32_t flags;
    const void *x[BKE_MM_MAX_MODELS], *P[BKE_MM_MAX_MODELS];
    const void *log_likelihood[BKE_MM_MAX_MODELS];
    void *x_out[BKE_MM_MAX_MODELS], *P_out[BKE_MM_MAX_MODELS];
    double *mu, *cbar, *omega;
    const double *trans;
    int64_t weights_stride;
} bke_mm_args;

int bke_mm_probabilities(const bke_mm_args *args, void *stream);
int bke_mm_mix(const bke_mm_args *args, void *stream);
int bke_mm_estimate(const bke_mm_args *args, void *stream);

/* IMMEstimator.batch_filter: n_steps epochs of IMMEstimator.predict(); update(z) (filterpy/kalman/IMM.py:160-226)
 * for N tracks of M = n_models linear Kalman filters, in ONE launch.  Per track and epoch:
 *   mix (IMM.py:201-213, omega from mu and cbar) -> every model's predict (x = F x, P = alpha_sq[j] F P F' + Q)
 *   -> combined prior (:228-237) -> every model's update with its log-likelihood -> mu, cbar, omega (:178-184,
 *   :239-247, L = max(exp(ll), DBL_MIN)) -> combined posterior,
 * with the formulas and the order of summation of bke_mm_* and bke_kf_step.  A track without a measurement
 * (zs_valid[t,i] == 0) behaves as update(None): each model keeps its prior, y = 0, and its log-likelihood is
 * log N(0; 0, S) of the S of its last real update (-inf where det S <= 0; S is 0 before the first).  A model
 * whose S is singular keeps its prior and its previous log-likelihood; its S is still stored, and status is
 * BKE_STATUS_SINGULAR_S for that epoch.
 *   Per model j: x[j] [N,n], P[j] [N,n,n] (read, then the posterior of the last epoch), F/Q [N,n,n], H [N,m,n],
 *   R [N,m,m] per track or shared (stride 0), alpha_sq[j], and the filter's diagnostics, read at the start
 *   and written at the end as the loop leaves them: S[j] (the kept S), log_likelihood[j] [N], K[j] [N,n,m],
 *   y[j] [N,m], SI[j] [N,m,m], x_prior[j] / P_prior[j] (the last epoch's predicted state, written only) and
 *   status[j] [N] (int32, written only: the last epoch's, or with BKE_STATUS_STICKY the worst of the call's).
 *   mu [N,M] and cbar [N,M] (fp64) are read and written; omega [N,M,M] (fp64) is written (it is derived from
 *   mu and cbar); trans [M,M] (fp64).  zs [T,N,m], zs_valid [T,N] (uint8, NULL = every track measured).
 *   Outputs: means [T,N,n], covariances [T,N,n,n] (combined posteriors), means_p, covariances_p (combined
 *   priors), mus [T,N,M] (fp64, mu after each update).
 * A bad size, stride, dtype, flag or model count (2 .. BKE_MM_MAX_MODELS), a NULL pointer the call reads or
 * writes, or an output that overlaps another array is BKE_ERR_BAD_ARG; a shape without a fused instance
 * ((n, m) other than 2/1 and 3/1 in fp32 and fp64, and 4/2 in fp32), or a state, diagnostic or output array that
 * is not 16-byte aligned, is BKE_ERR_UNSUPPORTED (the caller then runs the separate launches).  Both before any
 * device is touched.
 * The call allocates nothing and can be captured in a graph. */
typedef struct bke_imm_batch_args {
    int64_t n_tracks;
    int32_t dim_x, dim_z, n_models, dtype;
    int64_t n_steps;
    uint32_t flags;                                  /* 0 or BKE_STATUS_STICKY */
    uint32_t reserved;
    void *x[BKE_MM_MAX_MODELS], *P[BKE_MM_MAX_MODELS];
    const void *F[BKE_MM_MAX_MODELS]; int64_t F_stride[BKE_MM_MAX_MODELS];
    const void *Q[BKE_MM_MAX_MODELS]; int64_t Q_stride[BKE_MM_MAX_MODELS];
    const void *H[BKE_MM_MAX_MODELS]; int64_t H_stride[BKE_MM_MAX_MODELS];
    const void *R[BKE_MM_MAX_MODELS]; int64_t R_stride[BKE_MM_MAX_MODELS];
    double alpha_sq[BKE_MM_MAX_MODELS];
    void *S[BKE_MM_MAX_MODELS], *log_likelihood[BKE_MM_MAX_MODELS];
    void *K[BKE_MM_MAX_MODELS], *y[BKE_MM_MAX_MODELS], *SI[BKE_MM_MAX_MODELS];
    void *x_prior[BKE_MM_MAX_MODELS], *P_prior[BKE_MM_MAX_MODELS];
    int32_t *status[BKE_MM_MAX_MODELS];
    double *mu, *cbar, *omega;
    const double *trans;
    const void *zs;
    const uint8_t *zs_valid;
    void *means, *covariances, *means_p, *covariances_p;
    double *mus;
} bke_imm_batch_args;

int bke_imm_batch_filter(const bke_imm_batch_args *args, void *stream);

/* ---- the callers either side of a resample -----------------------------------------------------
 *
 * bke_cumsum_exact: cumsum_out[j] = np.cumsum(weights)[j] bit for bit (the strictly sequential fp64
 *   accumulation, reproduced by the same parity-map scan as the resamplers); last_one != 0 stores 1.0
 *   in the last element (filterpy/monte_carlo/resampling.py:174 `cumulative_sum[-1] = 1.`).
 * bke_searchsorted: np.searchsorted(sorted, keys, side='left' | 'right') -> int64.
 * bke_multinomial_resample: filterpy/monte_carlo/resampling.py:153-176 given the caller's uniforms
 *   (`random(len(weights))`, :176); indexes are int64 like np.searchsorted's result; cumsum_scratch
 *   is n doubles of device scratch; lut_scratch is n int32 of device scratch (or NULL): with it every
 *   bisection starts from a bracket looked up in a systematic resample (u = 0) of the same weights —
 *   same result, ~10x less random DRAM traffic.
 * bke_gather_rows: dst[r, :] = src[indexes[r], :] for rows of row_bytes bytes — the
 *   `particles[:] = particles[indexes]` that follows every resample (docs/monte_carlo/resampling.rst:4-8);
 *   indexes int32 (systematic / stratified) or int64 (multinomial); *err is set to 1 if an index is
 *   outside [0, n_src) (that row is left untouched).  src and dst must not alias.
 * bke_gather_rows_bank: the same per set of a bank, dst[b, i, :] = src[b, indexes[b, i], :] for
 *   n_sets sets of set_len rows each (the gather after bke_resample_bank); *err is set to 1 if an index is
 *   outside [0, set_len). */
int bke_cumsum_exact(int64_t n, const double *weights, double *cumsum_out, int32_t last_one, void *workspace,
                     size_t workspace_bytes, int32_t *info, void *stream);
int bke_searchsorted(int64_t n, const double *sorted, int64_t n_keys, const double *keys, int32_t side_right,
                     int64_t *indexes, void *stream);
int bke_multinomial_resample(int64_t n, const double *weights, const double *uniforms, int64_t *indexes,
                             double *cumsum_scratch, int32_t *lut_scratch, void *workspace, size_t workspace_bytes,
                             int32_t *info, void *stream);
int bke_gather_rows(int64_t n_out, int64_t n_src, int64_t row_bytes, const void *src, const void *indexes,
                    int32_t index_is_64, void *dst, int32_t *err, void *stream);
int bke_gather_rows_bank(int64_t n_sets, int64_t set_len, int64_t row_bytes, const void *src, const void *indexes,
                         int32_t index_is_64, void *dst, int32_t *err, void *stream);

/* ---- residual_resample (filterpy/monte_carlo/resampling.py:27-76) --------------------------------
 *
 * bke_residual_prepare: everything of residual_resample that does not need the uniforms —
 *   num_copies = floor(N*w) (:57), indexes[0:k] = repeat(arange(N), num_copies) (:58-62; int32 like the
 *   reference's np.zeros(N, 'i')), *n_copies_out = k, residual = w - num_copies (:69),
 *   *residual_sum_out = sum(residual) in the builtin's left-to-right fp64 order (:70) and
 *   cumsum_out = np.cumsum(residual / sum) with the last element set to 1 (:71-72), bit for bit.
 *   The caller draws random(N - k) (:74) after reading k.  workspace: bke_residual_workspace_bytes(n).
 * bke_searchsorted_bracket_sweep: np.searchsorted(arr, keys) (side='left') for an array that need NOT
 *   be sorted — residual's cumulative sum is not monotone, and NumPy's bisection carries its bracket
 *   from one key to the next (npy_binsearch: [r[i-1], n) if key[i-1] < key[i], else [0, r[i-1]+1)), so
 *   result i depends on result i-1.  One call evaluates that recurrence for all keys in parallel from
 *   the previous sweep's results `prev` (NULL for the first sweep: every key over [0, n)), writes `next`
 *   (and int32 copies to indexes32 when given) and sets *changed to 1 if any entry differs from prev.
 *   Repeat with prev/next swapped until *changed stays 0 (caller zeroes it before each sweep): the
 *   fixed point is NumPy's result, reached after at most n_keys sweeps, two or three in practice. */
size_t bke_residual_workspace_bytes(int64_t n);
int bke_residual_prepare(int64_t n, const double *weights, int32_t *indexes, double *cumsum_out, int64_t *n_copies_out,
                         double *residual_sum_out, void *workspace, size_t workspace_bytes, void *stream);
int bke_searchsorted_bracket_sweep(int64_t n, const double *arr, int64_t n_keys, const double *keys, const int64_t *prev,
                                   int64_t *next, int32_t *indexes32, int32_t *changed, void *stream);

/* ---- discrete Bayes filter banks (filterpy/discrete_bayes/discrete_bayes.py) ----------------------
 *
 * bke_db_step: any subset of predict, update and normalize on every row of pdf[n_rows, n_bins] (one 1-D
 *   histogram filter per row), fp32 or fp64, bit for bit per row:
 *     predict (kernel != NULL)      wrap: convolve(np.roll(pdf, offset), kernel, mode='wrap') (:124-125);
 *                                   BKE_DB_CONSTANT: convolve(shift(pdf, offset, cval=cval), kernel,
 *                                   mode='constant', cval=cval) (:127-128) for an integer offset, which is the
 *                                   exact shift where the reference's spline shift is so up to its roundoff;
 *                                   fp64 sums in scipy's window order, weights |w| <= DBL_EPSILON skipped as
 *                                   scipy skips them, rounded once to the dtype;
 *     update (likelihood != NULL)   prior * likelihood in the dtype (:88);
 *     normalize (BKE_DB_NORMALIZE)  p / sum(p) with the builtin sum's sequential fp64 chain 0 + p0 + p1 + ...
 *                                   and an fp64 division rounded once to the dtype (:47); sums[n_rows] (fp64,
 *                                   or NULL) receives each row's sum.
 *   kernel [kernel_len] shared (kernel_stride 0) or [n_rows, kernel_len] (kernel_stride kernel_len), fp64 as
 *   scipy converts it; offsets[n_rows] (int64) per row, or NULL for `offset` on every row.  Any offset is
 *   legal, as is kernel_len > n_bins.  out[n_rows, n_bins] may be pdf itself; no other array may overlap
 *   out, sums or the workspace.  Rows of up to 28928 fp32 / 14464 fp64 bins run one CTA per row; longer
 *   rows run one at a time in three passes, the sum by bke_cumsum_exact's parity-map scan, and need
 *   bke_db_workspace_bytes(n_bins, dtype) bytes of 256-byte aligned device workspace (0 for short rows).
 *   A bad size, flag, dtype, stride or pointer is BKE_ERR_BAD_ARG before any device is touched.  The call
 *   allocates nothing and can be captured in a graph. */
#define BKE_DB_NORMALIZE 1u
#define BKE_DB_CONSTANT 2u
typedef struct {
    int64_t n_rows, n_bins;
    int32_t dtype;
    uint32_t flags;                                  /* BKE_DB_NORMALIZE | BKE_DB_CONSTANT */
    const double *kernel;                            /* NULL: no predict */
    int64_t kernel_len, kernel_stride;
    const int64_t *offsets;                          /* NULL: `offset` for every row */
    int64_t offset;
    double cval;                                     /* BKE_DB_CONSTANT only */
    const void *pdf, *likelihood;                    /* likelihood NULL: no update */
    void *out;
    double *sums;                                    /* NULL or [n_rows], with BKE_DB_NORMALIZE */
    void *workspace;
    size_t workspace_bytes;
} bke_db_args;

size_t bke_db_workspace_bytes(int64_t n_bins, int32_t dtype);
int bke_db_step(const bke_db_args *args, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* BKE_H_ */
