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
 * Optional outputs (NULL = not wanted): x_prior, P_prior, K[N,n,m], y[N,m], S[N,m,m],
 * SI[N,m,m], log_likelihood[N] (log N(y; 0, S), kalman_filter.py:1203-1210), status[N].
 * x_out/P_out may alias x/P (in-place update).
 * Kernels behind this call (same arithmetic, picked by shape; DESIGN.md §3): 4/2 fp32 TMA register tile, register tiles
 * with direct loads (4/2 fp64, 1/1 .. 4/4, 6/3 fp32), row blocks (9/3, 6/3, 16/4, 16/2, 32/4 fp32), a catch-all for any
 * shape, and — fp32 banks with dim_x = 16 or 32 whose F and Q are shared (stride 0) — the wgmma tile: F P F' as
 * three-term TF32 products accumulated in fp32 (everything else of the
 * step in plain fp32), the whole predict+update in one launch when H and R are shared too and dim_z <= 4.
 * Environment switches (measurements): BKE_KF_TC=0 keeps those banks on the CUDA cores.
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
} bke_kf_args;

int bke_kf_step(const bke_kf_args *args, void *stream);

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
 * Both calls return BKE_ERR_UNSUPPORTED for other shapes, dtypes, shared models or misaligned pointers,
 * and when the environment sets BKE_KF_SYM=0; bke_kf_step is then the call to make. */
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
 *                               be used when it is 0);
 *   bke_kf_packed_models_bytes  the size of the record of n_filters filters for a `varying` mask (0 for a
 *                               mask with bits above 36); the caller allocates it, 16-byte aligned;
 *   bke_kf_pack_models          fills the record: one tile of 128 filters after the other, each tile
 *                               k = popcount(varying) planes of 128 floats, plane s holding the s-th
 *                               varying word (in the order above) of each filter of the tile, padded with
 *                               zeros to a whole last tile;
 *   bke_kf_step_packed          bke_kf_step with the record and a HOST copy of the map standing in for
 *                               args->F, Q, H and R (which must still be the per-filter arrays they were
 *                               scanned and packed from, unchanged since); the results are bit-identical
 *                               to bke_kf_step's.  The record may be NULL when no word varies.
 * The calls return BKE_ERR_UNSUPPORTED for other shapes, dtypes, shared models, an asymmetric map,
 * misaligned pointers, and when the environment sets BKE_KF_SYM=0; bke_kf_step is then the call to make. */
#define BKE_KF42_MODEL_WORDS 37
typedef struct bke_kf_model_map {
    uint64_t varying;                       /* bit e: word e differs between filters */
    int32_t asymmetric;                     /* 1: some Q or R is not exactly symmetric */
    int32_t reserved;
    float words[BKE_KF42_MODEL_WORDS];      /* filter 0's words */
} bke_kf_model_map;

int bke_kf_scan_models(int64_t n_filters, int32_t dim_x, int32_t dim_z, int32_t dtype, const void *F, const void *Q,
                       const void *H, const void *R, bke_kf_model_map *map, void *stream);
size_t bke_kf_packed_models_bytes(int64_t n_filters, uint64_t varying);
int bke_kf_pack_models(int64_t n_filters, int32_t dim_x, int32_t dim_z, int32_t dtype, const void *F, const void *Q,
                       const void *H, const void *R, uint64_t varying, void *record, void *stream);
int bke_kf_step_packed(const bke_kf_args *args, const void *record, const bke_kf_model_map *host_map, void *stream);

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

typedef struct bke_ukf_args {
    int64_t n_filters;
    int32_t dim_x, dim_z;
    int32_t dtype;
    uint32_t flags;                  /* BKE_DO_PREDICT | BKE_DO_UPDATE (update alone re-draws the
                                        sigma points from (x,P), UKF.py:407) */
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

/* Stand-alone pieces of the unscented path for callers that use them directly:
 *   MerweScaledSigmaPoints.sigma_points(x, P)   filterpy/kalman/sigma_points.py:124-177
 *       x[N,n], P[N,n,n] -> sigmas[N,2n+1,n]; status[N] = BKE_STATUS_NOT_PD where scipy's cholesky
 *       would raise (only the upper triangle of P is read, as scipy does);
 *   unscented_transform(sigmas, Wm, Wc, noise_cov)   filterpy/kalman/unscented_transform.py:22-128
 *       sigmas[N,k,n], Wm[k], Wc[k], noise_cov[n,n] (noise_stride 0) / [N,n,n] (n*n) / NULL
 *       -> x_out[N,n], P_out[N,n,n]   (default mean / residual functions). */
int bke_merwe_sigma_points(int64_t n_filters, int32_t dim_x, int32_t dtype, double alpha, double beta, double kappa,
                           const void *x, const void *P, void *sigmas, int32_t *status, void *stream);
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
 * fx_model / F as in bke_ukf_args.  K may be NULL. */
typedef struct {
    int64_t n_filters, n_steps;
    int32_t dim_x, dtype, fx_model, reserved;
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
/* the same around a user-supplied fx (fx_model = BKE_FX_USER, a model from bke_ukf_model_compile; dim_x <= 8).  The
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
 *   outside [0, n_src) (that row is left untouched).  src and dst must not alias. */
int bke_cumsum_exact(int64_t n, const double *weights, double *cumsum_out, int32_t last_one, void *workspace,
                     size_t workspace_bytes, int32_t *info, void *stream);
int bke_searchsorted(int64_t n, const double *sorted, int64_t n_keys, const double *keys, int32_t side_right,
                     int64_t *indexes, void *stream);
int bke_multinomial_resample(int64_t n, const double *weights, const double *uniforms, int64_t *indexes,
                             double *cumsum_scratch, int32_t *lut_scratch, void *workspace, size_t workspace_bytes,
                             int32_t *info, void *stream);
int bke_gather_rows(int64_t n_out, int64_t n_src, int64_t row_bytes, const void *src, const void *indexes,
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

#ifdef __cplusplus
}
#endif
#endif /* BKE_H_ */
