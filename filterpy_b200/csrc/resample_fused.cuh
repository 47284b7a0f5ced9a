// resample_fused.cuh — interface of the single-pass resampling kernel behind bke_resample_normalized
// (csrc/resample_fused.cu), and the PTX wrappers the multi-pass emit kernel shares with it.
#pragma once
#include <cuda.h>
#include "resample_common.cuh"

namespace bke {
namespace rs {

constexpr int F_IPT = 16;        // particles per consumer thread and tile
constexpr int F_SPT = 20;        // output-window slots per consumer thread (5 x 16 bytes)
constexpr int F_STAGES = 2;      // shared-memory tiles per CTA (one in flight while one is processed)
enum { F_SYS = 0, F_STRAT = 1 };

struct FHeader {
    int fallback;       // 1 -> the sequential kernel must produce the result
    int n_unclean;      // tiles with raw elements
    int n_runs;         // long runs queued for the fill pass
    int overflow;       // positions >= cumsum[-1]
    int chain_bad;      // a verified assumption failed
    int n_seq;          // tiles walked element by element
    int cap_overflow;   // outputs that did not fit the index buffer (never expected)
    int n_slow;         // tiles that took the slow path (ties / raw elements)
    int tile_counter;   // next tile to hand out
    int timeout;        // a look-back gave up waiting (never expected)
    int n_general;      // tiles expanded through more than one window
    int pad;
    i64 out_begin;      // first output position owned by this call (0)
    i64 out_end;        // one past the last
};

struct FParams {
    const double *w;
    i64 n;                 // particles: positions are (u + i) / n, idx holds n indexes
    int use_tma;           // weights are 16-byte aligned: tiles arrive by TMA
    double u;              // systematic offset
    const double *U;       // stratified uniforms (NULL = systematic)
    int *idx;
    i64 eb;                // classification margin in ulps of the running sum
    double tau;            // fast-path margin of the position search
    int *info;             // user info[8] or NULL
    double *cumsum_last;   // or NULL
    const double *div;     // non-NULL: every weight is divided by *div first (fused normalisation)
    double *wnorm_out;     // optional: the normalised weights
    FHeader *hdr;
    u64 *st1, *st2;        // [T + 1] status words of the two look-back stages
    Run *runs;
    int max_runs;
    int T;
};

struct FRunArgs {
    i64 n;
    const double *w, *U;
    double u;
    int *idx;
    void *workspace; size_t ws_bytes;
    int *info; double *cumsum_last;
    const double *div; double *wnorm_out;
};

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t f_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void f_mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(f_smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void f_fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void f_fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void f_mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(f_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void f_mbar_arrive(uint64_t *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(f_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool f_mbar_try(uint64_t *bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
                 : "=r"(ok) : "r"(f_smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void f_mbar_wait(uint64_t *bar, uint32_t parity)
{
    while (!f_mbar_try(bar, parity)) {}
}
__device__ __forceinline__ void f_tma_load_2d(void *dst, const CUtensorMap *map, int c0, int c1, uint64_t *bar)
{
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(f_smem_u32(dst)), "l"(map), "r"(f_smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// named barriers of the consumer warps (the producer warp never joins them)
template <int NT> __device__ __forceinline__ void f_bar()
{
    asm volatile("barrier.cta.sync 1, %0;" ::"n"(NT) : "memory");
}
template <int NT> __device__ __forceinline__ int f_bar_and(int pred)
{
    int out;
    asm volatile("{\n.reg .pred p, q;\nsetp.ne.b32 p, %1, 0;\nbarrier.cta.red.and.pred q, 1, %2, p;\nselp.b32 %0, 1, 0, q;\n}\n"
                 : "=r"(out) : "r"(pred), "n"(NT) : "memory");
    return out;
}
__device__ __forceinline__ u64 f_ld(const u64 *p)
{
    u64 v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void f_st(u64 *p, u64 v)
{
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// byte offset of weight (row r = owning thread, 16-byte chunk c) inside a swizzled stage
__device__ __forceinline__ uint32_t f_swz(int r, int c) { return (uint32_t)r * 128u + (uint32_t)((c ^ (r & 7)) << 4); }

// tensor map of the weights as rows of 16 doubles with a box of `box_rows` rows (cached per thread);
// false when the driver entry point is missing or the pointer / size does not qualify for TMA
bool f_weights_map(const double *w, int64_t n, int box_rows, CUtensorMap *out);

size_t f_carve(int64_t n, unsigned char *base, FParams *p);
int f_run(const FRunArgs &a, cudaStream_t s);

}  // namespace rs
}  // namespace bke
