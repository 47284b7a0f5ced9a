// kf42_ceiling.cu — the memory-only twin of the 4/2 fp32 bank step (kf42_f32_kernel<3,0,false,*>).
//
// It moves exactly the step's traffic and does nothing else: per filter it reads x (16 B), P, F, Q
// (64 B each), H (32 B), R (16 B) and z (8 B) and writes x and P back in place, 264 B read and 80 B
// written.  With mode 1, Q and R are replaced by one stream of 52 B per filter (the packed upper
// triangles a symmetric bank's step reads, bke_kf_pack_sym_models): 236 B read, 316 B in all.  With
// mode 2, F, Q, H and R are replaced by one stream of 40 B per filter (the 10 model words that differ
// between the filters of the bench bank, bke_kf_pack_models): 128 B read, 208 B in all.  With mode 3,
// that stream is 20 B per filter (the 5 distinct planes among those 10 words, the planes the step reads
// when the scan has flagged the copies): 108 B read, 188 B in all.
// Every array is read and written with flat, fully coalesced 16-byte accesses.  A CTA of
// 256 threads covers 64 filters: every thread moves one 16-byte chunk of P, F, Q, the first 128
// threads one of H, the first 64 one of x and R, the first 32 one of z, so the read/write mix is the
// step's at every point of the sweep.  Its bandwidth is the ceiling the step can reach on the card.
//
// Built by scripts/kf42_ceiling.py (nvcc -shared) and driven through ctypes.
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

constexpr int CHUNK = 64;           // filters per CTA iteration
constexpr int THREADS = 256;        // = CHUNK * 64 B / 16 B
constexpr int SYM_CHUNKS = CHUNK * 52 / 16;     // 16-byte chunks of the packed Q / R stream per CTA iteration
constexpr int WORD_CHUNKS = CHUNK * 40 / 16;    // 16-byte chunks of the packed model-word stream per CTA iteration
constexpr int DISTINCT_CHUNKS = CHUNK * 20 / 16;    // the same for its distinct planes only

__global__ void __launch_bounds__(THREADS)
kf42_traffic_kernel(float4 *x, float4 *P, const float4 *F, const float4 *Q, const float4 *H, const float4 *R,
                    const float4 *z, int64_t n_chunks, int mode)
{
    const int t = threadIdx.x;
    for (int64_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
        const int64_t p16 = c * THREADS + t;            // 16-byte chunk of P, F, Q (4 per filter)
        float4 vp = P[p16];
        float4 vh = make_float4(0.f, 0.f, 0.f, 0.f), vf = vh, vq = vh, vx = vh, vr = vh, vz = vh;
        if (mode == 2) {
            if (t < WORD_CHUNKS) vq = __ldg(Q + c * WORD_CHUNKS + t);
        } else if (mode == 3) {
            if (t < DISTINCT_CHUNKS) vq = __ldg(Q + c * DISTINCT_CHUNKS + t);
        } else {
            vf = __ldg(F + p16);
            if (mode == 1) {
                if (t < SYM_CHUNKS) vq = __ldg(Q + c * SYM_CHUNKS + t);
            } else {
                vq = __ldg(Q + p16);
                if (t < THREADS / 4) vr = __ldg(R + c * (THREADS / 4) + t);
            }
            if (t < THREADS / 2) vh = __ldg(H + c * (THREADS / 2) + t);
        }
        if (t < THREADS / 4) vx = x[c * (THREADS / 4) + t];
        if (t < THREADS / 8) vz = __ldg(z + c * (THREADS / 8) + t);
        // the stores depend on every load (bit-wise, no floating-point work), so none is dropped
        const uint32_t k = __float_as_uint(vf.x) | __float_as_uint(vq.y) | __float_as_uint(vh.z) |
                           __float_as_uint(vr.w) | __float_as_uint(vz.x);
        vp.x = __uint_as_float(__float_as_uint(vp.x) | k);
        P[p16] = vp;
        if (t < THREADS / 4) {
            vx.x = __uint_as_float(__float_as_uint(vx.x) | k);
            x[c * (THREADS / 4) + t] = vx;
        }
    }
}

}  // namespace

extern "C" {

// One launch over n_filters (a multiple of 64); returns a cudaError_t.  mode 1: Q is the 52 B-per-filter
// stream and R is not read; mode 2 (3): Q is the 40 (20) B-per-filter stream and F, H, R are not read.
int kf42_traffic(void *x, void *P, const void *F, const void *Q, const void *H, const void *R, const void *z,
                 int64_t n_filters, int grid, int mode, void *stream)
{
    kf42_traffic_kernel<<<grid, THREADS, 0, (cudaStream_t)stream>>>(
        (float4 *)x, (float4 *)P, (const float4 *)F, (const float4 *)Q, (const float4 *)H, (const float4 *)R,
        (const float4 *)z, n_filters / CHUNK, mode);
    return (int)cudaGetLastError();
}

}
