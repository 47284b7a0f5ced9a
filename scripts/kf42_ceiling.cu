// kf42_ceiling.cu — the memory-only twin of the 4/2 fp32 bank step (kf42_f32_kernel<3,0,false,*>).
//
// It moves exactly the step's traffic and does nothing else: per filter it reads x (16 B), P, F, Q
// (64 B each), H (32 B), R (16 B) and z (8 B) and writes x and P back in place, 264 B read and 80 B
// written.  With mode 1, Q and R are replaced by one stream of 52 B per filter (the packed upper
// triangles a symmetric bank's step reads, bke_kf_pack_sym_models): 236 B read, 316 B in all.  With
// mode 2, F, Q, H and R are replaced by one stream of 40 B per filter (the 10 model words that differ
// between the filters of the bench bank, bke_kf_pack_models): 128 B read, 208 B in all.  With mode 3,
// that stream is 20 B per filter (the 5 distinct planes among those 10 words, the planes the step reads
// when the scan has flagged the copies): 108 B read, 188 B in all.  The twin of the fused ring
// (bke_kf_steps_packed, kf42_ring_traffic below) is mode 3 with n_z measurement streams instead of one: the
// state and the 20 B of models once, 8 B of z per fused step, 180 + 8 n_z B per filter and launch.
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

// L2 cache-policy loads and stores (the accesses of the hinted variant below)
__device__ __forceinline__ float4 ld_hint(const float4 *a, uint64_t pol)
{
    float4 v;
    asm volatile("ld.global.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(a), "l"(pol) : "memory");
    return v;
}
__device__ __forceinline__ void st_hint(float4 *a, float4 v, uint64_t pol)
{
    asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;"
                 ::"l"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}

// Order and L2 policy of one launch.  The CTAs walk the chunks in launch order c = blockIdx.x + k gridDim.x;
// chunk c is the bank's chunk c (forward) or n_chunks - 1 - c (reverse).  With HINTS: z is read with
// evict_first when z_first is set, the first `head` chunks of the launch order are read and written with
// evict_first (they are the previous launch's tail, demoted), the last `tail` chunks with evict_last (kept
// for the next launch, which walks the other way and starts on them); the rest with the default policy.
struct Order {
    int reverse, z_first;
    int64_t head, tail;
};

template <bool HINTS>
__global__ void __launch_bounds__(THREADS)
kf42_traffic_kernel(float4 *x, float4 *P, const float4 *F, const float4 *Q, const float4 *H, const float4 *R,
                    const float4 *z, int64_t n_chunks, int mode, Order o, int n_z)
{
    const int t = threadIdx.x;
    uint64_t pol_first = 0, pol_last = 0, pol_normal = 0;
    if (HINTS) {
        asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol_first));
        asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol_last));
        asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol_normal));
    }
    for (int64_t k = blockIdx.x; k < n_chunks; k += gridDim.x) {
        const int64_t c = o.reverse ? n_chunks - 1 - k : k;
        const uint64_t pol = k < o.head ? pol_first : k >= n_chunks - o.tail ? pol_last : pol_normal;
        const uint64_t pol_z = o.z_first ? pol_first : pol;
        auto ld = [&](const float4 *a, uint64_t pl) { return HINTS ? ld_hint(a, pl) : __ldg(a); };
        const int64_t p16 = c * THREADS + t;            // 16-byte chunk of P, F, Q (4 per filter)
        float4 vp = HINTS ? ld_hint(P + p16, pol) : P[p16];
        float4 vh = make_float4(0.f, 0.f, 0.f, 0.f), vf = vh, vq = vh, vx = vh, vr = vh, vz = vh;
        if (mode == 2) {
            if (t < WORD_CHUNKS) vq = ld(Q + c * WORD_CHUNKS + t, pol);
        } else if (mode == 3) {
            if (t < DISTINCT_CHUNKS) vq = ld(Q + c * DISTINCT_CHUNKS + t, pol);
        } else {
            vf = ld(F + p16, pol);
            if (mode == 1) {
                if (t < SYM_CHUNKS) vq = ld(Q + c * SYM_CHUNKS + t, pol);
            } else {
                vq = ld(Q + p16, pol);
                if (t < THREADS / 4) vr = ld(R + c * (THREADS / 4) + t, pol);
            }
            if (t < THREADS / 2) vh = ld(H + c * (THREADS / 2) + t, pol);
        }
        if (t < THREADS / 4) vx = HINTS ? ld_hint(x + c * (THREADS / 4) + t, pol) : x[c * (THREADS / 4) + t];
        if (t < THREADS / 8) {
            // (stream j of the ring's twin is the j-th [N,2] array behind z)
            for (int j = 0; j < n_z; j++) {
                const float4 v = ld(z + (j * n_chunks + c) * (THREADS / 8) + t, pol_z);
                vz.x = __uint_as_float(__float_as_uint(vz.x) | __float_as_uint(v.x) | __float_as_uint(v.w));
            }
        }
        // the stores depend on every load (bit-wise, no floating-point work), so none is dropped
        const uint32_t kk = __float_as_uint(vf.x) | __float_as_uint(vq.y) | __float_as_uint(vh.z) |
                            __float_as_uint(vr.w) | __float_as_uint(vz.x);
        vp.x = __uint_as_float(__float_as_uint(vp.x) | kk);
        if (HINTS) st_hint(P + p16, vp, pol);
        else P[p16] = vp;
        if (t < THREADS / 4) {
            vx.x = __uint_as_float(__float_as_uint(vx.x) | kk);
            if (HINTS) st_hint(x + c * (THREADS / 4) + t, vx, pol);
            else x[c * (THREADS / 4) + t] = vx;
        }
    }
}

}  // namespace

extern "C" {

// One launch over n_filters (a multiple of 64); returns a cudaError_t.  mode 1: Q is the 52 B-per-filter
// stream and R is not read; mode 2 (3): Q is the 40 (20) B-per-filter stream and F, H, R are not read.
// reverse: walk the chunks last to first.  z_first, head_filters, tail_filters: the L2 policy of the
// hinted variant (Order above; head and tail in filters, rounded down to whole chunks); all zero and
// hints == 0: plain accesses with the default policy.
int kf42_traffic(void *x, void *P, const void *F, const void *Q, const void *H, const void *R, const void *z,
                 int64_t n_filters, int grid, int mode, void *stream, int reverse, int hints, int z_first,
                 int64_t head_filters, int64_t tail_filters)
{
    const Order o = {reverse, z_first, head_filters / CHUNK, tail_filters / CHUNK};
    if (hints)
        kf42_traffic_kernel<true><<<grid, THREADS, 0, (cudaStream_t)stream>>>(
            (float4 *)x, (float4 *)P, (const float4 *)F, (const float4 *)Q, (const float4 *)H, (const float4 *)R,
            (const float4 *)z, n_filters / CHUNK, mode, o, 1);
    else
        kf42_traffic_kernel<false><<<grid, THREADS, 0, (cudaStream_t)stream>>>(
            (float4 *)x, (float4 *)P, (const float4 *)F, (const float4 *)Q, (const float4 *)H, (const float4 *)R,
            (const float4 *)z, n_filters / CHUNK, mode, o, 1);
    return (int)cudaGetLastError();
}

// The twin of one fused ring of n_z steps: x, P read and written in place, Q the 20 B-per-filter stream,
// z the n_z consecutive [n_filters, 2] measurement arrays.
int kf42_ring_traffic(void *x, void *P, const void *Q, const void *z, int64_t n_filters, int grid, int n_z, void *stream)
{
    kf42_traffic_kernel<false><<<grid, THREADS, 0, (cudaStream_t)stream>>>(
        (float4 *)x, (float4 *)P, nullptr, (const float4 *)Q, nullptr, nullptr, (const float4 *)z, n_filters / CHUNK, 3,
        Order{0, 0, 0, 0}, n_z);
    return (int)cudaGetLastError();
}

}
