// rpk_device.cuh -- device-side primitives shared by the kernels: programmatic dependent launch, mbarrier +
// bulk async copy (TMA, SASS UBLKCP), the 16-byte split of a result slice, the look-back over CTA counts.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rpk {
namespace dev {

// Programmatic dependent launch (PDL): a kernel launched with the programmatic-serialization attribute may start
// while its stream predecessor is still running; wait() blocks until the predecessor has completed and its writes
// are visible, trigger() in the predecessor lets the dependent be scheduled early.  No-ops without the attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

// A slice of n int32 at src, copied in 16-byte units: `head` elements up to src's first 16-byte boundary, `nvec` units,
// then the elements from `tail0` on.  Source and destinations share the 16-byte phase, so one split fits all of them.
struct SliceSplit { uint32_t head, nvec, tail0; };
__device__ __forceinline__ SliceSplit slice_split(const int32_t* src, uint32_t n) {
    const uint32_t mis = (uint32_t)((reinterpret_cast<uintptr_t>(src) & 15u) >> 2);
    SliceSplit s;
    s.head = min(n, (4u - mis) & 3u);
    s.nvec = (n - s.head) >> 2;
    s.tail0 = s.head + (s.nvec << 2);
    return s;
}
// The <= 3 + 3 elements off the 16-byte grid of the slice src[off, off + n), by the caller's threads t < 3: loaded once
// (ld.global.cg: the source was written by a grid still running or just finished) and stored at the same offset of
// dst(o) for every o < n_dst except o = skip.
template <typename Dst>
__device__ __forceinline__ void copy_slice_edges(const int32_t* src, uint32_t off, uint32_t n, const SliceSplit& s, uint32_t t, int n_dst,
                                                 int skip, Dst dst) {
    int32_t hv = 0, tv = 0;
    if (t < s.head) hv = __ldcg(src + off + t);
    if (t < n - s.tail0) tv = __ldcg(src + off + s.tail0 + t);
    for (int o = 0; o < n_dst; ++o) {
        if (o == skip) continue;
        if (t < s.head) dst(o)[off + t] = hv;
        if (t < n - s.tail0) dst(o)[off + s.tail0 + t] = tv;
    }
}

#define kFlagAgg (1ull << 32)
#define kFlagMask (3ull << 32)

// Decoupled look-back over the CTAs before `id` (one warp): returns the exclusive prefix.  There is at most one CTA
// per SM, and they all finish at about the same time, so walking back window by window would cost one L2 round trip
// per 32 predecessors.  Every CTA publishes its count once (kFlagAgg | count; an entry without a flag bit is not there
// yet) and sums ALL entries before it in one pass of independent loads, retrying only the ones that are not there yet.
// Ids come from a scheduling ticket, so every CTA waited for has started.  Used by the status sweep and the pending list.
__device__ __forceinline__ uint32_t sum_before(volatile unsigned long long* st, uint32_t id, uint32_t total, uint32_t lane) {
    if (lane == 0) st[id] = kFlagAgg | total;
    uint32_t acc = 0;
    for (uint32_t base = 0; base < id; base += 128) {  // four independent loads per lane and pass
        unsigned long long v[4];
        bool need[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) { const uint32_t i = base + (uint32_t)k * 32 + lane; need[k] = i < id; v[k] = need[k] ? st[i] : kFlagAgg; }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t i = base + (uint32_t)k * 32 + lane;
            while (need[k] && (v[k] & kFlagMask) == 0) v[k] = st[i];
            acc += (uint32_t)v[k];
        }
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) acc += __shfl_xor_sync(0xFFFFFFFFu, acc, d);
    return acc;
}

}  // namespace dev
}  // namespace rpk
