// select.cu -- the P pods x G offers grid: Client.GetGPUTypes evaluated for every pod row at once
// (reference runpod_client.go:465-509, called per pod from :1281).
//
// Data flow per call (all on one stream):
//   k_select_fused    kind 4 (bit-sliced view), batches up to kFusedRowsMax rows and empty tables: one launch, one
//                     lane per row; larger batches take the persistent kernel (select_persist.cu).
//   k_pod_prep        kinds 3..1: pod columns -> per-row threshold word (rank compression), rows grouped by (cloud
//                     view, vcpu constrains, ram constrains), pos[] = none
//   k_select_packed   kinds 3/2: one u32 of rank fields per offer, R rows per warp in registers, lanes stride
//                     over offers, row argmin by redux.sync.min over lanes.
//   k_select_wide     kind 1: int32 compares on (mem, vcpu, ram) for tables that do not rank-pack.
//   (packed / wide)   grid = (row tile) x (offer segment); atomicMin merges segments; the last CTA of a row tile
//                     applies price < maxPrice to the winner (the bound is a prefix of the sorted order) and stores
//                     the offer index into every peer's assignment vector (the fused all-gather).
//   k_select_top5*    optional: the whole <=5 gpuTypeIds list per row (runpod_client.go:502-509).
//   k_pod_reselect_top5  the pending results' reselect: gather + thresholds + top-5 over a list whose length is read
//                     on the device (rpk_select_pending_changed, _gather and _device_gather)
//   k_gather_push     several output vectors: copies the finished slice to the peers (a second launch copies the top-5
//                     lists' slice for rpk_select_device_gather_top5); k_peer_signal (select_persist.cu) then signals a
//                     bound peer group.
#include <math_constants.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "rpk_device.cuh"
#include "rpk_internal.cuh"

namespace rpk {
using namespace dev;

// ---------------------------------------------------------------------------------------------------------
// K0: per-row preparation
// ---------------------------------------------------------------------------------------------------------
// Rows are grouped so that a tile is homogeneous in (cloud view, "vcpu request constrains", "ram request
// constrains"): group g = cloud*4 + needs_vcpu*2 + needs_ram.  A request whose rank threshold is 0 is met by
// every offer, so tiles of such rows never read that column's masks (for pods without vcpu/ram requests this
// is literally the reference's predicate, which has no such columns: runpod_client.go:478).
__global__ void __launch_bounds__(1024) k_pod_prep(SelectArgs a) {
    pdl_trigger();  // the grid kernel may be scheduled now; it waits (pdl_wait) before it reads anything written here
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31;
    const bool valid = p < a.P;
    uint32_t grp = kGroups;  // none
    if (valid) {
        uint8_t c = a.cloud ? a.cloud[p] : (uint8_t)RPK_CLOUD_SECURE;
        a.pos[p] = kNone;
        uint32_t need = 3;  // kernels without rank thresholds always test both extension columns
        if (a.pk.bits) {
            uint32_t tm = lower_bound_i32(a.distinct[0], a.D[0], a.req_mem[p]) + 1;
            uint32_t tv = lower_bound_i32(a.distinct[1], a.D[1], a.req_vcpu ? a.req_vcpu[p] : 0);
            uint32_t tr = lower_bound_i32(a.distinct[2], a.D[2], a.req_ram ? a.req_ram[p] : 0);
            need = (tv != 0 ? 2u : 0u) | (tr != 0 ? 1u : 0u);
            a.rw[p] = (tm << a.pk.sh_mem) | (tv << a.pk.sh_vcpu) | (tr << a.pk.sh_ram);
        }
        if (c <= 1) grp = c * 4u + need;
        else finish_row_no_cloud(a, p);
    }
    // one atomic per (group, 1024-row block): the counters are shared by the whole grid
    __shared__ uint32_t s_cnt[kGroups][32], s_base[kGroups];
    const uint32_t warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    uint32_t my_mask = 0;
#pragma unroll
    for (uint32_t g = 0; g < kGroups; ++g) {
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, grp == g);
        if (grp == g) my_mask = m;
        if (lane == 0) s_cnt[g][warp] = __popc(m);
    }
    __syncthreads();
    if (warp < kGroups) {  // warp g scans group g's per-warp counts
        const uint32_t c = lane < nwarps ? s_cnt[warp][lane] : 0u;
        uint32_t inc = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t n = __shfl_up_sync(0xFFFFFFFFu, inc, d); if ((int)lane >= d) inc += n; }
        if (lane < nwarps) s_cnt[warp][lane] = inc - c;
        if (lane == 31) s_base[warp] = inc ? atomicAdd(&a.counts[warp], inc) : 0u;
    }
    __syncthreads();
    if (grp < kGroups)
        a.order[(size_t)grp * a.P + s_base[grp] + s_cnt[grp][warp] + __popc(my_mask & ((1u << lane) - 1))] = p;
}

// ---------------------------------------------------------------------------------------------------------
// row-tile decoding shared by the packed and wide kernels
// ---------------------------------------------------------------------------------------------------------
struct TileInfo { int cloud; uint32_t group; uint32_t row_base; uint32_t nrows; uint32_t total_tiles; bool valid; };

__device__ __forceinline__ TileInfo decode_tile(const SelectArgs& a, uint32_t tile, uint32_t rpc) {
    TileInfo t;
    t.valid = false; t.cloud = 0; t.group = 0; t.row_base = 0; t.nrows = 0;
    uint32_t first = 0;
    // tiles are handed out heaviest group first (3 mask words per (row, chunk), then 2, then 1): the CTAs that
    // finish the grid are the light ones, so the tail of the last wave is short
    constexpr uint32_t kHeavyFirst[kGroups] = {3, 7, 1, 2, 5, 6, 0, 4};
#pragma unroll
    for (uint32_t i = 0; i < kGroups; ++i) {
        const uint32_t g = a.tune_natural_order ? i : kHeavyFirst[i];
        const uint32_t n = a.counts[g];
        const uint32_t tg = (n + rpc - 1) / rpc;
        if (!t.valid && tile < first + tg) {
            t.valid = true; t.group = g; t.cloud = (int)(g >> 2);
            t.row_base = (tile - first) * rpc;
            t.nrows = min(rpc, n - t.row_base);
        }
        first += tg;
    }
    t.total_tiles = first;
    return t;
}
__device__ __forceinline__ uint32_t tile_row(const SelectArgs& a, const TileInfo& t, uint32_t slot) {
    return a.order[(size_t)t.group * a.P + t.row_base + slot];
}

// Merge the segment result, and let the last CTA of the tile finish the rows (finish_row).
__device__ __forceinline__ void finish_tile(const SelectArgs& a, const TileInfo& t, uint32_t tile, uint32_t S, int* s_last) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        uint32_t ticket = atomicAdd(&a.tile_ctr[tile], 1u);
        *s_last = (ticket == S - 1);
    }
    __syncthreads();
    if (!*s_last) return;
    __threadfence();
    for (uint32_t slot = threadIdx.x; slot < t.nrows; slot += blockDim.x) {
        const uint32_t row = tile_row(a, t, slot);
        finish_row(a, a.view[t.cloud], row, __ldcg(a.pos + row));
    }
    if (a.n_out > 1 && a.self_out < 0) __threadfence_system();  // direct peer stores are performed system-wide before this grid completes
    // The counters clean themselves (no memset launch per call): this CTA is the last one to touch the tile's
    // ticket, and the CTA that finishes the last tile of the grid clears the group counts.  Every CTA of a valid
    // tile read the counts before it took its ticket; CTAs past the last tile that read them late see fewer
    // tiles, never more, and still return.
    if (threadIdx.x == 0) {
        a.tile_ctr[tile] = 0u;
        if (atomicAdd(a.done, 1u) + 1u == t.total_tiles) {
#pragma unroll
            for (uint32_t g = 0; g < kGroups; ++g) a.counts[g] = 0u;
            *a.done = 0u;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// K1 (packed): one u32 per offer.
//   kPos = true  (layout bits <= 18): 2.5 instructions per offer-score -- IMAD.IADD d = o - r (FMA pipe),
//                LOP3 key = (~d & guard) | (d & pos_mask) (ALU), half a VIMNMX3 (ALU).  The surviving key is
//                the lowest feasible position of the segment, or >= 2^kPosBits when nothing is feasible.
//   kPos = false (wider layouts): sub + LOP3-with-predicate + select; positions walked in descending order
//                so that a lower one overwrites.
// ---------------------------------------------------------------------------------------------------------
template <int R, bool kPos>
__global__ void __launch_bounds__(kCtaThreads, 3) k_select_packed(SelectArgs a, uint32_t S, uint32_t seg_len) {
    extern __shared__ __align__(128) uint32_t s_off[];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ int s_last;
    constexpr uint32_t RPC = kWarpsPerCta * R;
    const uint32_t tile = blockIdx.x / S, seg = blockIdx.x - tile * S;
    pdl_wait();     // k_pod_prep (counts, order, rw, pos) has completed
    pdl_trigger();  // a dependent (the peer fence) may be scheduled; it waits for this grid to complete
    const TileInfo t = decode_tile(a, tile, RPC);
    if (!t.valid) return;
    const uint32_t Gc = ((a.G + kChunk - 1) / kChunk) * kChunk;
    const uint32_t g0 = seg * seg_len;
    const uint32_t len = g0 < Gc ? min(seg_len, Gc - g0) : 0;
    if (threadIdx.x == 0) { mbar_init(&s_bar, 1); mbar_fence_init(); }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(&s_bar, len * 4u);
        if (len) bulk_g2s(s_off, a.view[t.cloud].packed + g0, len * 4u, &s_bar);
    }
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t rw[R], best[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const uint32_t slot = warp * R + r;
        rw[r] = slot < t.nrows ? a.rw[tile_row(a, t, slot)] : 0u;
        best[r] = kNone;
    }
    const uint32_t guard = a.pk.guard;
    mbar_wait(&s_bar, 0);
    const uint4* s4 = reinterpret_cast<const uint4*>(s_off);
    if (kPos) {
        constexpr uint32_t kLow = (1u << kPosBits) - 1;
        for (int ch = (int)(len / kChunk) - 1; ch >= 0; --ch) {
            const uint4 o = s4[ch * 32 + lane];
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const uint32_t d0 = o.x - rw[r], d1 = o.y - rw[r], d2 = o.z - rw[r], d3 = o.w - rw[r];
                const uint32_t k0 = (~d0 & guard) | (d0 & kLow), k1 = (~d1 & guard) | (d1 & kLow);
                const uint32_t k2 = (~d2 & guard) | (d2 & kLow), k3 = (~d3 & guard) | (d3 & kLow);
                best[r] = min(min(best[r], k0), k1);
                best[r] = min(min(best[r], k2), k3);
            }
        }
    } else {
        for (int ch = (int)(len / kChunk) - 1; ch >= 0; --ch) {
            const uint4 o = s4[ch * 32 + lane];
            const uint32_t j0 = g0 + (uint32_t)ch * kChunk + lane * 4u;
            // descending positions: a lower position overwrites, so the lowest feasible one survives
#pragma unroll
            for (int r = 0; r < R; ++r) {
                if ((~(o.w - rw[r]) & guard) == 0) best[r] = j0 + 3;
                if ((~(o.z - rw[r]) & guard) == 0) best[r] = j0 + 2;
                if ((~(o.y - rw[r]) & guard) == 0) best[r] = j0 + 1;
                if ((~(o.x - rw[r]) & guard) == 0) best[r] = j0;
            }
        }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
        uint32_t m = __reduce_min_sync(0xFFFFFFFFu, best[r]);
        if (kPos) m = m < (1u << kPosBits) ? g0 + m : kNone;  // segments are 2^kPosBits-aligned
        const uint32_t slot = warp * R + r;
        if (lane == 0 && slot < t.nrows && m != kNone) atomicMin(&a.pos[tile_row(a, t, slot)], m);
    }
    finish_tile(a, t, tile, S, &s_last);
}

// ---------------------------------------------------------------------------------------------------------
// K1 (bit-sliced): the offer side of a 32-offer chunk is three precomputed 32-bit masks (one per column,
// picked by the row's rank thresholds), so ONE LOP3 evaluates the feasibility of 32 (pod, offer) pairs:
//     m = mask_mem[chunk][t_mem] & mask_vcpu[chunk][t_vcpu] & mask_ram[chunk][t_ram]
// Every pair of the grid is still evaluated (bit j of m IS the predicate of runpod_client.go:478 minus the
// price bound for offer j) -- there is no early exit and no deduplication of equal rows.  Each lane owns RPL
// pod rows; all lanes walk the same chunk, reading their own three words of its 128-byte row (distinct words
// = distinct banks, equal words = broadcast).  Chunks are walked in descending price order so the last hit
// is the cheapest; its mask is re-read once at the end for the bit position.
// ---------------------------------------------------------------------------------------------------------
template <int RPL, int STRIDE, bool NEEDV, bool NEEDR>
__device__ __forceinline__ void bitmap_walk(const uint32_t* s_off, int n, const uint32_t (&o1)[RPL], const uint32_t (&o2)[RPL],
                                            const uint32_t (&o3)[RPL], uint32_t (&bc)[RPL]) {
    int ch = n - 1;
    for (; ch >= 3; ch -= 4) {
        const uint32_t* p = s_off + (size_t)(ch - 3) * STRIDE;
#pragma unroll
        for (int u = 3; u >= 0; --u) {
#pragma unroll
            for (int r = 0; r < RPL; ++r) {
                uint32_t m = p[u * STRIDE + o1[r]];
                if (NEEDV) m &= p[u * STRIDE + o2[r]];
                if (NEEDR) m &= p[u * STRIDE + o3[r]];
                if (m) bc[r] = (uint32_t)(ch - 3 + u);
            }
        }
    }
    for (; ch >= 0; --ch) {
        const uint32_t* p = s_off + (size_t)ch * STRIDE;
#pragma unroll
        for (int r = 0; r < RPL; ++r) {
            uint32_t m = p[o1[r]];
            if (NEEDV) m &= p[o2[r]];
            if (NEEDR) m &= p[o3[r]];
            if (m) bc[r] = (uint32_t)ch;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// K1 (bit-sliced, fused, small batches): one launch does what a row sort, a grid kernel and its epilogue would do,
// for batches too small to fill the GPU anyway (micro-batches of the streaming path, BASELINE config 2), and for
// an empty table at any batch size.  One lane per pod row in arrival order, no grouping, no atomics, no counters
// to clear: the CTA walks every segment of the view(s) its rows use, so each row's result is final when its loop ends.
// ---------------------------------------------------------------------------------------------------------
template <int STRIDE>
__global__ void __launch_bounds__(kCtaThreads) k_select_fused(SelectArgs a, uint32_t seg_chunks) {
    extern __shared__ __align__(128) uint32_t s_off[];
    __shared__ __align__(8) uint64_t s_bar;
    const uint32_t p = blockIdx.x * kCtaThreads + threadIdx.x;
    const bool valid = p < a.P;
    uint32_t cls = 2;
    uint32_t o1[1] = {0}, o2[1] = {0}, o3[1] = {0};
    bool needv = false, needr = false;
    if (valid) {
        const uint8_t c = a.cloud ? a.cloud[p] : (uint8_t)RPK_CLOUD_SECURE;
        cls = c <= 1 ? c : 2;
        const uint32_t tm = lower_bound_i32(a.distinct[0], a.D[0], a.req_mem[p]) + 1;
        const uint32_t tv = lower_bound_i32(a.distinct[1], a.D[1], a.req_vcpu ? a.req_vcpu[p] : 0);
        const uint32_t tr = lower_bound_i32(a.distinct[2], a.D[2], a.req_ram ? a.req_ram[p] : 0);
        o1[0] = tm - 1; o2[0] = a.pk.bm_off_vcpu + tv; o3[0] = a.pk.bm_off_ram + tr;
        needv = tv != 0; needr = tr != 0;
        a.rw[p] = o1[0] | (o2[0] << 8) | (o3[0] << 16);  // k_select_top5_bitmap reads it
        if (cls == 2 && a.top5) for (int k = 0; k < RPK_TOPK; ++k) a.top5[(size_t)p * RPK_TOPK + k] = -1;
    }
    const bool wv = __any_sync(0xFFFFFFFFu, needv), wr = __any_sync(0xFFFFFFFFu, needr);  // warp-uniform
    if (threadIdx.x == 0) { mbar_init(&s_bar, 1); mbar_fence_init(); }
    __syncthreads();
    const uint32_t total_chunks = (a.G + 31) / 32;
    const uint32_t S = total_chunks ? (total_chunks + seg_chunks - 1) / seg_chunks : 0;
    uint32_t gpos = kNone, loads = 0;
    for (uint32_t c = 0; c < 2; ++c) {
        if (!__syncthreads_or(cls == c)) continue;  // no row of this CTA uses view c
        for (int seg = (int)S - 1; seg >= 0; --seg) {  // descending price: the last hit is the cheapest
            const uint32_t c0 = (uint32_t)seg * seg_chunks;
            const uint32_t n = min(seg_chunks, total_chunks - c0);
            if (threadIdx.x == 0) {
                mbar_expect_tx(&s_bar, n * STRIDE * 4u);
                bulk_g2s(s_off, a.view[c].bitmap + (size_t)c0 * STRIDE, n * STRIDE * 4u, &s_bar);
            }
            mbar_wait(&s_bar, loads & 1);
            ++loads;
            if (cls == c) {
                uint32_t bc[1] = {kNone};
                switch ((wv ? 2 : 0) | (wr ? 1 : 0)) {
                    case 0: bitmap_walk<1, STRIDE, false, false>(s_off, (int)n, o1, o2, o3, bc); break;
                    case 1: bitmap_walk<1, STRIDE, false, true>(s_off, (int)n, o1, o2, o3, bc); break;
                    case 2: bitmap_walk<1, STRIDE, true, false>(s_off, (int)n, o1, o2, o3, bc); break;
                    default: bitmap_walk<1, STRIDE, true, true>(s_off, (int)n, o1, o2, o3, bc); break;
                }
                if (bc[0] != kNone) {
                    const uint32_t* q = s_off + (size_t)bc[0] * STRIDE;
                    const uint32_t m = q[o1[0]] & q[o2[0]] & q[o3[0]];
                    gpos = (c0 + bc[0]) * 32u + (uint32_t)__ffs(m) - 1u;
                }
            }
            __syncthreads();  // everyone is done with the segment before the next bulk copy overwrites it
        }
    }
    if (valid) finish_row(a, a.view[cls], p, gpos);  // a row of neither cloud walked nothing: gpos = kNone
}

// ---------------------------------------------------------------------------------------------------------
// K1 (generic): full-range int32 columns, one int4 per offer, 4 instructions per offer-score
// ---------------------------------------------------------------------------------------------------------
template <int R>
__global__ void __launch_bounds__(kCtaThreads, 2) k_select_wide(SelectArgs a, uint32_t S, uint32_t seg_len) {
    extern __shared__ __align__(128) uint32_t s_off[];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ int s_last;
    constexpr uint32_t RPC = kWarpsPerCta * R;
    const uint32_t tile = blockIdx.x / S, seg = blockIdx.x - tile * S;
    pdl_wait();     // k_pod_prep (counts, order, rw, pos) has completed
    pdl_trigger();  // a dependent (the peer fence) may be scheduled; it waits for this grid to complete
    const TileInfo t = decode_tile(a, tile, RPC);
    if (!t.valid) return;
    const uint32_t Gc = ((a.G + kChunk - 1) / kChunk) * kChunk;
    const uint32_t g0 = seg * seg_len;
    const uint32_t len = g0 < Gc ? min(seg_len, Gc - g0) : 0;
    if (threadIdx.x == 0) { mbar_init(&s_bar, 1); mbar_fence_init(); }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(&s_bar, len * 16u);
        if (len) bulk_g2s(s_off, a.view[t.cloud].wide + g0, len * 16u, &s_bar);
    }
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int32_t qm[R], qv[R], qr[R];
    uint32_t best[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const uint32_t slot = warp * R + r;
        const uint32_t row = slot < t.nrows ? tile_row(a, t, slot) : 0u;
        const bool ok = slot < t.nrows;
        qm[r] = ok ? a.req_mem[row] : INT32_MAX;
        qv[r] = ok && a.req_vcpu ? a.req_vcpu[row] : 0;
        qr[r] = ok && a.req_ram ? a.req_ram[row] : 0;
        best[r] = kNone;
    }
    mbar_wait(&s_bar, 0);
    const int4* s4 = reinterpret_cast<const int4*>(s_off);
    for (int ch = (int)(len / 32u) - 1; ch >= 0; --ch) {
        const int4 o = s4[ch * 32 + lane];
        const uint32_t j = g0 + (uint32_t)ch * 32u + lane;
#pragma unroll
        for (int r = 0; r < R; ++r)
            if (o.x >= qm[r] && o.y >= qv[r] && o.z >= qr[r]) best[r] = j;  // mem/vcpu/ram >= request (:478, non-strict)
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const uint32_t m = __reduce_min_sync(0xFFFFFFFFu, best[r]);
        const uint32_t slot = warp * R + r;
        if (lane == 0 && slot < t.nrows && m != kNone) atomicMin(&a.pos[tile_row(a, t, slot)], m);
    }
    finish_tile(a, t, tile, S, &s_last);
}

// ---------------------------------------------------------------------------------------------------------
// top-5: "Take up to 5 GPUs" (runpod_client.go:502-509).  The two walks below are the rule, once: the top-5 kernels
// and the pending results' reselect (k_pod_reselect_top5) call them.
// ---------------------------------------------------------------------------------------------------------
// One warp per pod row (every lane passes the same row) walks the wide view of cloud c in ascending price order,
// ballots feasibility over 32 positions at a time and stops after five hits or at the first position whose price is
// not < mx (everything after it is at least as expensive).  Lane 0 writes row p of a.top5, -1 padded.  Gc: G rounded up to
// kChunk; lane: threadIdx.x & 31.
__device__ __forceinline__ void top5_walk_wide(const SelectArgs& a, uint8_t c, uint32_t lane, uint32_t Gc, int32_t qm, int32_t qv,
                                               int32_t qr, double mx, uint32_t p) {
    const int4* __restrict__ wide = a.view[c].wide;
    const double* __restrict__ price = a.view[c].price;
    int cnt = 0;
    for (uint32_t base = 0; base < Gc && cnt < RPK_TOPK; base += 32) {
        const int4 o = wide[base + lane];
        const bool price_ok = price[base + lane] < mx;  // NaN (unavailable / padding) fails
        const bool f = price_ok && o.x >= qm && o.y >= qv && o.z >= qr;
        uint32_t mask = __ballot_sync(0xFFFFFFFFu, f);
        const bool stop = __ballot_sync(0xFFFFFFFFu, !price_ok) != 0;
        while (mask && cnt < RPK_TOPK) {
            const int b = __ffs(mask) - 1;
            const int idx = __shfl_sync(0xFFFFFFFFu, o.w, b);
            if (lane == 0) a.top5[(size_t)p * RPK_TOPK + cnt] = idx;
            ++cnt;
            mask &= mask - 1;
        }
        if (stop) break;
    }
    if (lane == 0) for (int k = cnt; k < RPK_TOPK; ++k) a.top5[(size_t)p * RPK_TOPK + k] = -1;
}

// One lane per pod row on the bit-sliced view (its price, bitmap and perm arrays): o1 / o2 / o3 are the row's three mask
// words (its rank thresholds), mx its price bound.  The bound is a prefix of the sorted view (binary search for its
// length), inside it the row's three masks give 32 positions per step; the walk stops at five hits.  Writes out[0, 5),
// -1 padded.  The views come in as restrict parameters: that keeps the load kinds the top-5 kernel had with its own
// restrict locals (price and perm through the read-only path, the masks not).
template <int STRIDE>
__device__ __forceinline__ void top5_walk_bitmap(const double* __restrict__ price, const uint32_t* __restrict__ bm,
                                                 const int32_t* __restrict__ perm, uint32_t G, uint32_t o1, uint32_t o2,
                                                 uint32_t o3, double mx, int32_t* out) {
    uint32_t lo = 0, hi = G;  // number of positions with price < mx (NaN = unavailable sorts last and fails)
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (price[mid] < mx) lo = mid + 1; else hi = mid; }
    const uint32_t cut = lo;
    int cnt = 0;
    for (uint32_t base = 0; base < cut && cnt < RPK_TOPK; base += 32) {
        const uint32_t* row = bm + (size_t)(base >> 5) * STRIDE;
        uint32_t m = row[o1] & row[o2] & row[o3];
        if (cut - base < 32) m &= (1u << (cut - base)) - 1u;
        while (m && cnt < RPK_TOPK) {
            out[cnt++] = perm[base + (uint32_t)__ffs(m) - 1u];
            m &= m - 1;
        }
    }
    for (; cnt < RPK_TOPK; ++cnt) out[cnt] = -1;
}

__global__ void __launch_bounds__(256) k_select_top5(SelectArgs a) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t Gc = ((a.G + kChunk - 1) / kChunk) * kChunk;
    for (uint32_t p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < a.P; p += nwarps) {
        const uint8_t c = a.cloud ? a.cloud[p] : (uint8_t)RPK_CLOUD_SECURE;
        if (c > 1) continue;  // filled by k_pod_prep
        const int32_t qm = a.req_mem[p], qv = a.req_vcpu ? a.req_vcpu[p] : 0, qr = a.req_ram ? a.req_ram[p] : 0;
        const double mx = a.max_price ? a.max_price[p] : RPK_DEFAULT_MAX_PRICE;
        top5_walk_wide(a, c, lane, Gc, qm, qv, qr, mx, p);
    }
}

template <int STRIDE>
__global__ void __launch_bounds__(256) k_select_top5_bitmap(SelectArgs a) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= a.P) return;
    const uint8_t c = a.cloud ? a.cloud[p] : (uint8_t)RPK_CLOUD_SECURE;
    if (c > 1) return;  // filled by k_pod_prep
    const uint32_t w = a.rw[p];
    const uint32_t o1 = w & 0xFFu, o2 = (w >> 8) & 0xFFu, o3 = (w >> 16) & 0xFFu;
    const double mx = a.max_price ? a.max_price[p] : RPK_DEFAULT_MAX_PRICE;
    top5_walk_bitmap<STRIDE>(a.view[c].price, a.view[c].bitmap, a.view[c].perm, a.G, o1, o2, o3, mx, a.top5 + (size_t)p * RPK_TOPK);
}

// The reselect of rpk_select_pending_changed*: rows [0, n) of r.list, n = r.dn[1] as the stale step left it on the
// device, so the launch may be sized for a worst case and needs no count on the host.  Row i gathers its slot's five
// columns into r.out (the columns the diff stores with the result) and writes its top-5 list to r.s.top5 -- what
// k_pod_gather, a select and its top-5 kernel leave for the same rows, bit for bit; best is not needed (it is top5[0]).
// STRIDE 32 / 64: the bit-sliced view, one lane per row, the rank thresholds computed here as the select kernels compute
// them.  STRIDE 0: the wide view (tables without pk.bm_words), one warp per row, which compares the raw columns.  A row
// whose cloud byte is above 1 gets five -1.  Grid-stride: the grid is a few waves whatever the count.
template <int STRIDE>
__global__ void __launch_bounds__(256) k_pod_reselect_top5(ReselectArgs r) {
    const SelectArgs& a = r.s;
    if (r.counts && blockIdx.x == 0 && threadIdx.x == 0) { r.counts[0] = r.dn[0]; r.counts[1] = r.dn[1]; }
    const uint32_t n = r.dn[1];
    constexpr uint32_t kRowThreads = STRIDE ? 1u : 32u;
    const uint32_t step = gridDim.x * blockDim.x / kRowThreads;
    for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) / kRowThreads; i < n; i += step) {
        const uint32_t s = r.list[i];
        const int32_t mem = r.t.mem[s], vcpu = r.t.vcpu[s], ram = r.t.ram[s];
        const double mx = r.t.max_price[s];
        const uint8_t c = r.t.cloud[s];
        if (STRIDE || (threadIdx.x & 31) == 0) {
            r.out.mem[i] = mem; r.out.vcpu[i] = vcpu; r.out.ram[i] = ram; r.out.max_price[i] = mx; r.out.cloud[i] = c;
            if (c > 1) for (int k = 0; k < RPK_TOPK; ++k) a.top5[(size_t)i * RPK_TOPK + k] = -1;
        }
        if (c > 1) continue;
        if constexpr (STRIDE != 0) {
            const uint32_t o1 = lower_bound_i32(a.distinct[0], a.D[0], mem);
            const uint32_t o2 = a.pk.bm_off_vcpu + lower_bound_i32(a.distinct[1], a.D[1], vcpu);
            const uint32_t o3 = a.pk.bm_off_ram + lower_bound_i32(a.distinct[2], a.D[2], ram);
            top5_walk_bitmap<STRIDE>(a.view[c].price, a.view[c].bitmap, a.view[c].perm, a.G, o1, o2, o3, mx,
                                     a.top5 + (size_t)i * RPK_TOPK);
        } else {
            top5_walk_wide(a, c, threadIdx.x & 31, ((a.G + kChunk - 1) / kChunk) * kChunk, mem, vcpu, ram, mx, i);
        }
    }
}

int launch_pod_reselect(const ReselectArgs& r, uint32_t n_max, int sm_count, cudaStream_t st) {
    const uint32_t rows_per_cta = r.s.pk.bm_words ? 256u : 8u;
    const uint32_t blocks = std::max<uint32_t>(1u, std::min<uint32_t>((n_max + rows_per_cta - 1) / rows_per_cta, (uint32_t)sm_count * 8));
    if (!r.s.pk.bm_words) k_pod_reselect_top5<0><<<blocks, 256, 0, st>>>(r);
    else if (r.s.pk.bm_stride == 64) k_pod_reselect_top5<64><<<blocks, 256, 0, st>>>(r);
    else k_pod_reselect_top5<32><<<blocks, 256, 0, st>>>(r);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

// ---------------------------------------------------------------------------------------------------------
// the all-gather: push this shard's finished slice [row0, row0 + P) of the local vector into every peer's vector
// with 16-byte stores over NVLink (grid = CTAs per peer x peers).  Launched behind the select kernels with PDL.
// ---------------------------------------------------------------------------------------------------------
struct PushArgs { const int32_t* src; int32_t* dst[RPK_MAX_GPUS]; uint32_t count; };

__global__ void __launch_bounds__(256) k_gather_push(PushArgs a) {
    pdl_wait();     // the select kernels have completed: the local slice is final
    pdl_trigger();  // the peer fence may be scheduled behind this grid
    const int32_t* src = a.src;  // read with ld.global.cg: written by the grid this kernel overlaps with (never the .nc path)
    int32_t* dst = a.dst[blockIdx.y];
    const SliceSplit sp = slice_split(src, a.count);  // the host checked that every vector shares the slice's 16-byte phase
    const uint32_t nvec = sp.nvec;
    if (blockIdx.x == 0) copy_slice_edges(src, 0, a.count, sp, threadIdx.x, 1, -1, [&](int) { return dst; });
    const uint4* s4 = reinterpret_cast<const uint4*>(src + sp.head);
    uint4* d4 = reinterpret_cast<uint4*>(dst + sp.head);
    // four 16-byte loads in flight per thread before the first store: the copy is latency-bound, not bandwidth-bound
    constexpr int kU = 4;
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 < nvec; i0 += stride * kU) {
        uint4 v[kU];
#pragma unroll
        for (int u = 0; u < kU; ++u) { const uint32_t i = i0 + (uint32_t)u * stride; if (i < nvec) v[u] = __ldcg(s4 + i); }
#pragma unroll
        for (int u = 0; u < kU; ++u) { const uint32_t i = i0 + (uint32_t)u * stride; if (i < nvec) d4[i] = v[u]; }
    }
    __threadfence_system();  // this thread's peer stores are performed system-wide before the grid completes
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
static Tune parse_tune() {
    Tune t;
    const char* e = getenv("RPK_TUNE");
    if (!e) return t;
    t.pdl = strstr(e, "pdl=off") == nullptr;
    t.natural_order = strstr(e, "order=natural") != nullptr;
    if (const char* p = strstr(e, "stagekb=")) t.stage_kb = atoi(p + 8);
    if (const char* p = strstr(e, "ipw=")) t.items_per_warp = atoi(p + 4);
    if (const char* p = strstr(e, "k0ctas=")) { const int v = atoi(p + 7); if (v > 0) t.k0ctas = v; }
    return t;
}
Tune read_tune() {
    static const bool reload = getenv("RPK_TUNE_RELOAD") != nullptr;
    if (reload) return parse_tune();
    static const Tune cached = parse_tune();
    return cached;
}

uint32_t select_tiles_max(uint32_t P, int rows_per_warp) {
    const uint32_t rpc = (uint32_t)(kWarpsPerCta * rows_per_warp);
    return (P + rpc - 1) / rpc + kGroups;  // every row group can end in one partial tile
}

static void seg_plan(uint32_t G, uint32_t seg_cap, uint32_t* S, uint32_t* seg_len) {
    const uint32_t Gc = ((G + kChunk - 1) / kChunk) * kChunk;
    uint32_t s = (Gc + seg_cap - 1) / seg_cap;
    if (s == 0) s = 1;
    uint32_t len = ((Gc + s - 1) / s + kChunk - 1) / kChunk * kChunk;
    *S = s; *seg_len = len;
}

int pick_rows_per_warp(uint32_t P, int sm_count) {
    // enough CTAs for ~4 waves of 3 CTAs/SM, else fewer rows per warp
    const uint64_t want = (uint64_t)sm_count * 3 * 4;
    for (int r = 16; r > 1; r >>= 1) {
        const uint64_t tiles = (P + (uint64_t)kWarpsPerCta * r - 1) / ((uint64_t)kWarpsPerCta * r);
        if (tiles >= want) return r;
    }
    return 1;
}

template <int R>
static void launch_grid(const SelectArgs& a, cudaStream_t st) {
    static thread_local int dev_pos = -1, dev_packed = -1, dev_wide = -1;
    const bool pdl = read_tune().pdl;
    uint32_t S, seg_len;
    const uint32_t tiles = select_tiles_max(a.P, R);
    if (a.pk.bits && a.pk.pos_bits) {
        // fixed 2^kPosBits-offer segments: the embedded positions are segment-local
        const uint32_t Gc = ((a.G + kChunk - 1) / kChunk) * kChunk;
        S = (Gc + kSegPacked - 1) / kSegPacked; if (S == 0) S = 1;
        seg_len = kSegPacked;
        allow_smem(k_select_packed<R, true>, (int)(kSegPacked * 4), &dev_pos);
        launch_pdl(k_select_packed<R, true>, dim3(tiles * S), dim3(kCtaThreads), (size_t)kSegPacked * 4, st, pdl, a, S, seg_len);
    } else if (a.pk.bits) {
        seg_plan(a.G, kSegPacked, &S, &seg_len);
        const size_t smem = (size_t)seg_len * 4;
        allow_smem(k_select_packed<R, false>, (int)(kSegPacked * 4), &dev_packed);
        launch_pdl(k_select_packed<R, false>, dim3(tiles * S), dim3(kCtaThreads), smem, st, pdl, a, S, seg_len);
    } else {
        seg_plan(a.G, kSegWide, &S, &seg_len);
        const size_t smem = (size_t)seg_len * 16;
        allow_smem(k_select_wide<R>, (int)(kSegWide * 16), &dev_wide);
        launch_pdl(k_select_wide<R>, dim3(tiles * S), dim3(kCtaThreads), smem, st, pdl, a, S, seg_len);
    }
}

template <int STRIDE>
static void launch_fused(const SelectArgs& a, cudaStream_t st) {
    constexpr uint32_t kSegChunks = kBmSegBytes / (STRIDE * 4);
    static thread_local int attr_dev = -1;
    allow_smem(k_select_fused<STRIDE>, (int)kBmSegBytes, &attr_dev);
    // small tables need a small stage: size the dynamic shared memory to the table
    const uint32_t total_chunks = (a.G + 31) / 32;
    const uint32_t chunks = total_chunks < kSegChunks ? (total_chunks ? total_chunks : 1) : kSegChunks;
    k_select_fused<STRIDE><<<(a.P + kCtaThreads - 1) / kCtaThreads, kCtaThreads, (size_t)chunks * STRIDE * 4, st>>>(a, kSegChunks);
}

static int launch_select_kernels(const SelectArgs& a, int R, const PersistPlan* pl, int sm_count, cudaStream_t st, bool* fused_push);

// Forward the finished slice [off, off + count) of outs[self] to every other vector of outs (the all-gather), with PDL
// behind the kernel that finished it.
static int launch_gather_push(int32_t* const* outs, int n_out, int self, size_t off, uint32_t count, int sm_count, cudaStream_t st) {
    PushArgs pa{};
    pa.src = outs[self] + off;
    int np = 0;
    for (int o = 0; o < n_out; ++o) if (o != self) pa.dst[np++] = outs[o] + off;
    pa.count = count;
    const uint32_t nvec = count / 4;
    uint32_t per_peer = (nvec + 1023) / 1024;  // one pass of four 16-byte units per thread, up to two CTAs per SM
    const uint32_t max_per_peer = 2u * (uint32_t)sm_count;
    per_peer = per_peer < 1 ? 1 : per_peer > max_per_peer ? max_per_peer : per_peer;
    launch_pdl(k_gather_push, dim3(per_peer, (unsigned)np), dim3(256), 0, st, read_tune().pdl, pa);
    return 1;
}

int launch_select(const SelectArgs& args, int R, const PersistPlan* pl, int sm_count, cudaStream_t st, const Top5Gather* t5) {
    SelectArgs a = args;
    a.tune_natural_order = read_tune().natural_order ? 1u : 0u;
    if (a.n_out == 1) a.self_out = 0;
    // The signal must follow the last peer store.  With a top-5 gather that is the lists' push behind the top-5 kernel,
    // so the select kernels (the persistent one signals from its last pusher) get no peer group to signal.
    const bool t5_push = t5 && t5->n_out > 1;
    if (t5_push) a.peers.n = 0;
    bool fused_push = false;  // the persistent kernel pushes (and signals) itself
    int launches = launch_select_kernels(a, R, pl, sm_count, st, &fused_push);
    if (!fused_push && a.n_out > 1 && a.self_out >= 0) launches += launch_gather_push(a.best_out, a.n_out, a.self_out, a.row0, a.P, sm_count, st);
    if (t5_push) launches += launch_gather_push(t5->out, t5->n_out, t5->self_out, (size_t)RPK_TOPK * a.row0, RPK_TOPK * a.P, sm_count, st);
    if (args.peers.n > 0 && (!fused_push || t5_push)) launches += launch_peer_signal(args.peers, 0, args.peers.inline_wait != 0, st);
    return launches;
}

static int launch_select_kernels(const SelectArgs& a, int R, const PersistPlan* pl, int sm_count, cudaStream_t st, bool* fused_push) {
    int launches = 0;
    if (a.pk.bm_words) {
        if (pl) {  // persistent kernel on the transposed view: sorts, selects, pushes, signals
            launches += launch_select_persist(a, *pl, st);
            *fused_push = true;
        } else {
            if (a.pk.bm_stride == 64) launch_fused<64>(a, st); else launch_fused<32>(a, st);
            ++launches;
        }
        if (a.top5) {
            if (a.pk.bm_stride == 64) k_select_top5_bitmap<64><<<(a.P + 255) / 256, 256, 0, st>>>(a);
            else k_select_top5_bitmap<32><<<(a.P + 255) / 256, 256, 0, st>>>(a);
            ++launches;
        }
        RPK_CUDA(cudaGetLastError());
        return launches;
    }
    // counts / done / tile tickets are zero here: zeroed when allocated, and every grid kernel leaves them zero
    k_pod_prep<<<(a.P + 1023) / 1024, 1024, 0, st>>>(a); ++launches;
    switch (R) {
        case 16: launch_grid<16>(a, st); break;
        case 8: launch_grid<8>(a, st); break;
        case 4: launch_grid<4>(a, st); break;
        case 2: launch_grid<2>(a, st); break;
        default: launch_grid<1>(a, st); break;
    }
    ++launches;
    if (a.top5) {
        const uint32_t blocks = (uint32_t)min((uint64_t)(a.P + 7) / 8, (uint64_t)sm_count * 32);
        k_select_top5<<<blocks, 256, 0, st>>>(a); ++launches;
    }
    RPK_CUDA(cudaGetLastError());
    return launches;
}

}  // namespace rpk
