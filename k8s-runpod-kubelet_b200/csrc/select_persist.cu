// select_persist.cu -- the P x G grid on the bit-sliced view, second generation (kernel kind 4, batches above the
// fused kernel's size).  Same predicate and tie rule as select.cu (reference runpod_client.go:465-509); what changes
// is how the mask words reach the lanes and who owns a stage of the offer table:
//
//   k_pod_classify   row -> rank thresholds -> class key (cloud, thresholds; see class_key for the order); one wave of
//                    CTAs, each looping over 512-row chunks: shared-memory histogram -> global class counts, one
//                    atomic per non-empty class whose return value is the CTA's first position inside the class
//                    (k0_base); fills pos[] = none when the grid kernel merges through it; block 0 resets the queue
//                    state of the grid kernel.
//   k_pod_scatter    counting-sort scatter, same CTAs and rows: every CTA scans the class counts itself, adds its
//                    class bases from classify and writes ONE {row, thresholds} pair per row in
//                    class order (ord_rw[]); block 0 publishes per-group row / work totals (a group is a cloud, or a
//                    (cloud, mem threshold) pair on the per-mem-threshold view).  Rows of neither cloud are final here
//                    (-1, runpod_client.go:469-475).
//   k_select_persist persistent CTAs (512 threads, one per SM).  A CTA loads ONE stage -- `per`
//                    64-chunk sub-ranges, 8 bulk async copies on 8 mbarriers, so the first items start before the whole
//                    stage has landed -- and keeps it for the whole call.  A stage is, where the table allows it, the
//                    slice of one mem threshold m over the whole price range (bitmapM: rows mem[m] & vcpu[v] and
//                    mem[m] & ram[r]; a row reads ONE word per chunk, two when both its vcpu and ram requests
//                    constrain), else a price range of the per-threshold view (bitmapT: one word for mem plus one per
//                    constraining column).  Its warps pull items (64 consecutive rows of one group x a range of
//                    sub-ranges) from the stage's queue with one atomic each.  A lane owns two rows and reads its rows'
//                    mask words for FOUR chunks with one LDS.128 (the views are [row][chunk]-major); rows of a warp
//                    share their thresholds after the sort, so the 32 lanes read at most a few distinct 16-byte
//                    addresses and the load costs 2 LSU cycles instead of the ~5 that four LDS.32 cost
//                    (tools/microbench/lds_probe.cu on H100: LDS.128 with <= 8 distinct addresses = 2.0 cycles/warp,
//                    LDS.32 = 1.2).  Every (row, chunk) mask is still loaded and ANDed -- bit j of it IS the predicate
//                    of runpod_client.go:478 (minus the price bound) for offer j; eight chunks are OR-folded before the
//                    "any hit" test, the cheapest hit's block is re-read once at the end for the bit position.
//                    An item that spans the whole table is final after its walk: price < maxPrice on the winner (strict,
//                    :478; the bound is a prefix of the price order) and the offer index is stored at once.  Otherwise
//                    segments merge with atomicMin and the warp that takes a row block's last ticket does that.
//   fused all-gather every retired row block adds its rows to one counter; a CTA that has run out of items waits until the
//                    counter reaches the row count (one polling thread per CTA), then EVERY warp of the grid copies an
//                    equal share of the slice to every peer with 16-byte NVLink stores; the CTA that finishes last
//                    signals the peers' flag words (rpk_peer_bind) and, with rpk_peer_inline_wait, waits for theirs.
//                    No drain, no copy kernel, no signal kernel, no wait kernel.
#include <math_constants.h>

#include "rpk_device.cuh"
#include "rpk_internal.cuh"

namespace rpk {
using namespace dev;

constexpr int kPThreads = 512;
constexpr int kPWarps = kPThreads / 32;
constexpr int kCopyGroups = 8;
constexpr int kRpl = 2;  // pod rows per lane
constexpr int kK0Batch = 4;  // K0: rows per thread whose loads are in flight together (one per 512-row chunk of the CTA)
constexpr uint32_t kSubWords = kSubStride;

// ---------------------------------------------------------------------------------------------------------
// row classes
// ---------------------------------------------------------------------------------------------------------
struct ClassDims { uint32_t Dm1, Dv1, Dr1, use_mem, C, slice; };
__host__ __device__ __forceinline__ ClassDims class_dims(const uint32_t (&D)[3], uint32_t slice) {
    ClassDims cd;
    cd.Dm1 = D[0] + 1; cd.Dv1 = D[1] + 1; cd.Dr1 = D[2] + 1;
    // bm_words = Dm1 + Dv1 + Dr1 <= 64, so 2 * Dv1 * Dr1 <= 1922 always fits; the mem threshold joins the key when it fits too
    // (bitmapM is only built, and `slice` only set, when it does)
    cd.use_mem = 2u * cd.Dm1 * cd.Dv1 * cd.Dr1 <= kMaxClasses ? 1u : 0u;
    cd.C = 2u * cd.Dv1 * cd.Dr1 * (cd.use_mem ? cd.Dm1 : 1u);
    cd.slice = slice;
    return cd;
}
// Class order = processing order.  Table staged by price: cloud, then vcpu threshold DEscending, ram threshold
// descending (rows whose requests constrain nothing -- one mask word per chunk -- come last, so the warps that finish
// the grid are the light ones), then the mem threshold.  Table staged per mem threshold (slice): cloud, mem threshold,
// vcpu threshold descending, ram threshold descending -- each (cloud, mem threshold) group is one run of the order.
__device__ __forceinline__ uint32_t class_key(const ClassDims& cd, uint32_t c, uint32_t tm1, uint32_t tv, uint32_t tr) {
    if (cd.slice) return ((c * cd.Dm1 + tm1) * cd.Dv1 + (cd.Dv1 - 1 - tv)) * cd.Dr1 + (cd.Dr1 - 1 - tr);
    uint32_t k = (c * cd.Dv1 + (cd.Dv1 - 1 - tv)) * cd.Dr1 + (cd.Dr1 - 1 - tr);
    return cd.use_mem ? k * cd.Dm1 + tm1 : k;
}
__device__ __forceinline__ uint32_t class_weight(const ClassDims& cd, uint32_t key) {  // mask words per (row, chunk)
    const uint32_t k = cd.use_mem && !cd.slice ? key / cd.Dm1 : key;
    const bool nv = k / cd.Dr1 % cd.Dv1 != cd.Dv1 - 1, nr = k % cd.Dr1 != cd.Dr1 - 1;
    if (cd.slice) return nv && nr ? 2u : 1u;  // mem & vcpu and mem & ram are stored: the one or two that constrain
    return 1u + (nv ? 1u : 0u) + (nr ? 1u : 0u);
}
// row group = K1's unit of queues: the cloud, or (cloud, mem threshold) on the per-mem-threshold view
__device__ __forceinline__ uint32_t class_group(const ClassDims& cd, uint32_t key) {
    return cd.slice ? key / (cd.Dv1 * cd.Dr1) : key / (cd.C / 2);
}

// The grid kernel's threshold word on the per-mem-threshold view: the row's mask rows inside its mem threshold's slice --
// mem & vcpu[tv] or mem & ram[tr] (mem itself when neither constrains) first, then mem & ram[tr] when both constrain,
// else the first again (ANDing it twice changes nothing).  rw: the row's bitmap words.
__device__ __forceinline__ uint32_t slice_rw(const ClassDims& cd, const PackLayout& pk, uint32_t rw) {
    const uint32_t tv = ((rw >> 8) & 0xFFu) - pk.bm_off_vcpu, tr = ((rw >> 16) & 0xFFu) - pk.bm_off_ram;
    const uint32_t i1 = tv ? tv : tr ? cd.Dv1 + tr : 0u, i2 = tv && tr ? cd.Dv1 + tr : i1;
    return i1 | (i2 << 8) | (i1 << 16);
}

// lower_bound_i32 on a shared-memory array (that one loads through __ldg, which is for global memory only)
__device__ __forceinline__ uint32_t lb_smem(const int32_t* a, uint32_t n, int32_t x) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (a[mid] < x) lo = mid + 1; else hi = mid; }
    return lo;
}

// ---------------------------------------------------------------------------------------------------------
// fused all-gather: push-block accounting.  Called by whole warps; `row` / `valid` per lane.
// ---------------------------------------------------------------------------------------------------------
// copy this warp's share of the local slice [row0, row0 + P) into every peer's vector.  The slice's 16-byte body is
// split evenly over ALL warps of the grid (a 125k-row slice is ~7 units per warp: one load, then one store per peer),
// so the copy has no hand-out counter and its latency is one L2 load + one NVLink store per lane.
__device__ __forceinline__ void push_share(const SelectArgs& a) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t wpc = blockDim.x >> 5, gw = blockIdx.x * wpc + (threadIdx.x >> 5), nw = gridDim.x * wpc;
    const int32_t* src = a.best_out[a.self_out];
    const uint32_t g_lo = a.row0, n = a.P;
    const SliceSplit sp = slice_split(src + g_lo, n);  // the host checked that every vector shares the slice's 16-byte phase
    const uint32_t head = sp.head, nvec = sp.nvec;
    if (gw == 0)
        copy_slice_edges(src, g_lo, n, sp, lane, a.n_out, a.self_out, [&](int o) { return a.best_out[o]; });
    const uint32_t per = (nvec + nw - 1) / nw;
    const uint32_t v_lo = min(nvec, gw * per), v_hi = min(nvec, v_lo + per);
    const uint4* s4 = reinterpret_cast<const uint4*>(src + g_lo + head);
    for (uint32_t i0 = v_lo; i0 < v_hi; i0 += 32 * 4) {
        uint4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) { const uint32_t i = i0 + (uint32_t)u * 32 + lane; if (i < v_hi) v[u] = __ldcg(s4 + i); }
        for (int o = 0; o < a.n_out; ++o) {
            if (o == a.self_out) continue;
            uint4* d4 = reinterpret_cast<uint4*>(a.best_out[o] + g_lo + head);
#pragma unroll
            for (int u = 0; u < 4; ++u) { const uint32_t i = i0 + (uint32_t)u * 32 + lane; if (i < v_hi) d4[i] = v[u]; }
        }
    }
}

// Fused all-gather, the way it works: natural-order push blocks only become complete near the END of the grid kernel
// (the rows of any 1024-row block are spread over all classes, and the classes are processed one after the other), so
// pushing "a block as soon as it is complete" degenerates into a serial tail on the few warps that finalise the last
// rows.  Instead every retired row block adds its rows to one counter; warps that run
// out of work wait for the counter to reach P -- the slowest warp is at most one item behind -- and then EVERY warp of
// the grid copies an equal share of the slice to the peers (push_share); the CTA that finishes last signals.
// No copy kernel, no drain, no signal kernel, no hand-out counter; the copy itself is spread over the whole grid.
__device__ __forceinline__ bool fused_gather(const SelectArgs& a) { return a.n_out > 1 && a.self_out >= 0; }

// whole-warp: `n` rows of this warp are final in the local vector
__device__ __forceinline__ void count_rows_done(const SelectArgs& a, uint32_t n) {
    if (!fused_gather(a)) return;
    __threadfence();  // this lane's store into the local vector is visible before the rows count as done
    __syncwarp();
    if ((threadIdx.x & 31) == 0 && n) atomicAdd(&a.hdr[kHdrRowsDone], n);
}

// whole CTA, after its warps have run out of items: one thread waits until every row is final (one poller per CTA, on
// a cache line nothing else touches while the grid runs), then every warp of the grid copies its share of the slice to
// the peers; the CTA that finishes last signals (and, with inline_wait, waits for the peers' signals)
__device__ __forceinline__ void push_tail(const SelectArgs& a) {
    if (!fused_gather(a)) return;
    __syncthreads();
    if (threadIdx.x == 0) {
        const volatile uint32_t* done = a.hdr + kHdrRowsDone;
        while (*done < a.P) __nanosleep(100);
    }
    __syncthreads();
    __threadfence();  // every row counted done is visible here
    push_share(a);
    __threadfence_system();  // this lane's peer stores are performed system-wide before its CTA counts as pushed
    __syncthreads();
    if (threadIdx.x < 32) {
        uint32_t last = 0;
        if (threadIdx.x == 0) last = atomicAdd(&a.hdr[kHdrPushed], 1u) + 1u == gridDim.x ? 1u : 0u;
        last = __shfl_sync(0xFFFFFFFFu, last, 0);
        // every peer store of this grid is performed system-wide (each pusher fenced before its CTA counted itself); with
        // inline_wait this warp, the grid's last worker anyway, also does the other half of the fence
        if (last && a.peers.n > 0) signal_peers(a.peers, kFlagSelect, kFlagSelectCtr, 0, a.peers.inline_wait != 0);
    }
}

// ---------------------------------------------------------------------------------------------------------
// K0a: classify.  No block waits for another one: the class counts are only added to here (the grid kernel of the
// previous call zeroed them once the scatter kernel was done with them); block 0 resets the grid kernel's queue cursors.
// Both K0 kernels run four CTAs per SM in one wave (launch_select_persist), so they are held to 32 registers.
// ---------------------------------------------------------------------------------------------------------
// fill_pos: the grid kernel merges row blocks through pos[] (more than one item per row block); a direct plan never
// reads it, so its 4 bytes per row are not written.
__global__ void __launch_bounds__(kPThreads, 4) k_pod_classify(SelectArgs a, uint32_t n_cursors, uint32_t fill_pos) {
    pdl_trigger();  // k_pod_scatter may be scheduled; it waits before it reads anything written here
    __shared__ int32_t s_dist[3][64];
    __shared__ uint32_t s_hist[kMaxClasses];
    const uint32_t tid = threadIdx.x;
    const ClassDims cd = class_dims(a.D, a.slice);
    uint32_t* hist = a.hist;
    for (uint32_t i = tid; i < 192; i += kPThreads) {
        const uint32_t d = i >> 6, k = i & 63;
        s_dist[d][k] = k < a.D[d] ? __ldg(a.distinct[d] + k) : INT32_MAX;
    }
    for (uint32_t i = tid; i < cd.C; i += kPThreads) s_hist[i] = 0u;
    if (blockIdx.x == 0) {  // the previous call's kernels have completed (this is not a programmatic launch): its queue state is free
        for (uint32_t i = tid; i < n_cursors; i += kPThreads) a.hdr[kHdrCursors + i] = 0u;
        if (tid == 0) { a.hdr[kHdrPushed] = 0u; a.hdr[kHdrRowsDone] = 0u; }
    }
    __syncthreads();
    // a CTA takes 512-row chunks b, b + grid, ...: the 4096-bin histogram (zeroing, flush) is paid once per CTA, not per
    // chunk.  A thread loads the columns of its next kK0Batch rows before it searches any of them, so their DRAM trips
    // overlap instead of one per row.
    const uint32_t stride = gridDim.x * kPThreads;
    for (uint32_t p0 = blockIdx.x * kPThreads + tid; p0 < a.P; p0 += kK0Batch * stride) {
        uint32_t c[kK0Batch];
        int32_t m[kK0Batch], v[kK0Batch], r[kK0Batch];
#pragma unroll
        for (int u = 0; u < kK0Batch; ++u) {
            const uint32_t p = p0 + (uint32_t)u * stride;
            const bool ok = p < a.P;
            c[u] = !ok ? 2u : a.cloud ? a.cloud[p] : (uint32_t)RPK_CLOUD_SECURE;
            m[u] = ok ? a.req_mem[p] : 0;
            v[u] = ok && a.req_vcpu ? a.req_vcpu[p] : 0;
            r[u] = ok && a.req_ram ? a.req_ram[p] : 0;
        }
#pragma unroll
        for (int u = 0; u < kK0Batch; ++u) {
            const uint32_t p = p0 + (uint32_t)u * stride;
            if (p >= a.P) break;
            const uint32_t tm1 = lb_smem(s_dist[0], a.D[0], m[u]);
            const uint32_t tv = lb_smem(s_dist[1], a.D[1], v[u]);
            const uint32_t tr = lb_smem(s_dist[2], a.D[2], r[u]);
            a.rw[p] = tm1 | ((a.pk.bm_off_vcpu + tv) << 8) | ((a.pk.bm_off_ram + tr) << 16);  // bitmap words (the top-5 kernel reads these)
            uint32_t key = 0xFFFFu;  // neither SECURE nor COMMUNITY: nothing is feasible (runpod_client.go:469-475)
            if (c[u] <= 1) { key = class_key(cd, c[u], tm1, tv, tr); atomicAdd(&s_hist[key], 1u); }
            a.key[p] = (uint16_t)key;
            if (fill_pos) a.pos[p] = kNone;  // "no feasible offer yet" for sorted position p (positions [0, valid rows) are used: a coalesced fill)
        }
    }
    __syncthreads();
    // flush: one atomic per non-empty class.  What it returns -- the rows of the class that CTAs before this one flushed --
    // is this CTA's first position inside the class, which the scatter kernel reads back instead of counting its rows
    // and reserving them again.  Class i is flushed by thread i % 512, whose <= 8 atomics go out back to back.
    uint32_t* base = a.k0_base + (size_t)blockIdx.x * kMaxClasses;
    constexpr uint32_t kPer = kMaxClasses / kPThreads;
    uint32_t n[kPer], got[kPer];
#pragma unroll
    for (uint32_t k = 0; k < kPer; ++k) { const uint32_t i = tid + k * kPThreads; n[k] = i < cd.C ? s_hist[i] : 0u; }
#pragma unroll
    for (uint32_t k = 0; k < kPer; ++k) got[k] = n[k] ? atomicAdd(&hist[tid + k * kPThreads], n[k]) : 0u;
#pragma unroll
    for (uint32_t k = 0; k < kPer; ++k) if (n[k]) base[tid + k * kPThreads] = got[k];
}

// Block 0 of the scatter: rows and mask-word work per row group, which the grid kernel shares its CTAs out by.  A group
// is a run of classes, so warp w sums groups w, w + 16, ... over the class totals (L2): a lane per class, the work in
// 64 bits per lane, then a warp reduction -- no shared-memory atomics.
__device__ __forceinline__ void publish_group_totals(const SelectArgs& a, const ClassDims& cd) {
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    const uint32_t n_groups = cd.slice ? 2u * cd.Dm1 : 2u, per_group = cd.C / n_groups;  // class_group
    for (uint32_t g = tid >> 5; g < n_groups; g += kPWarps) {
        uint32_t rows = 0;
        unsigned long long work = 0ull;
        for (uint32_t i = g * per_group + lane; i < (g + 1) * per_group; i += 32) {
            const uint32_t n = __ldcg(a.hist + i);
            rows += n; work += (unsigned long long)n * class_weight(cd, i);
        }
#pragma unroll
        for (int d = 16; d; d >>= 1) { rows += __shfl_xor_sync(0xFFFFFFFFu, rows, d); work += __shfl_xor_sync(0xFFFFFFFFu, work, d); }
        if (lane == 0) {
            a.hdr[kHdrGroupRows + g] = rows;
            a.hdr[kHdrGroupWork + g] = (uint32_t)min(work >> 2, 0xFFFFFFFFull);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// K0b: scatter into class order.  A CTA takes the same 512-row chunks b, b + grid, ... as in k_pod_classify.  Every
// CTA scans the <= 4096 class totals itself (cheaper than a serial "last block" phase in the kernel before) and adds
// its own first position inside each class, which its classify flush returned: that is the shared table "next free
// position per class", with no counting pass and no reservation here.  Pass 2 re-reads the keys (L2 hits) and hands
// every row its position.  The per-CTA cost of the 4096-bin table is paid once per CTA, not once per 512 rows.  Block
// 0 also publishes the per-group row / work totals the grid kernel shares its CTAs out by.
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kPThreads, 4) k_pod_scatter(SelectArgs a) {
    __shared__ uint32_t s_base[kMaxClasses];
    __shared__ uint32_t s_warp[kPWarps];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const ClassDims cd = class_dims(a.D, a.slice);
    pdl_wait();     // k_pod_classify has completed: keys, rw, class counts, per-CTA class bases
    pdl_trigger();  // the grid kernel may be scheduled; it waits before it reads anything written here
    const uint32_t stride = gridDim.x * kPThreads;
    // thread t owns classes [8t, 8t + 8): their totals and this CTA's bases, two 16-byte loads each (both buffers hold
    // kMaxClasses words per row; words at or above the class count are not used)
    constexpr uint32_t kPer = kMaxClasses / kPThreads;
    static_assert(kPer == 8, "two uint4 per thread");
    const uint4* h4 = reinterpret_cast<const uint4*>(a.hist + tid * kPer);
    const uint4* b4 = reinterpret_cast<const uint4*>(a.k0_base + (size_t)blockIdx.x * kMaxClasses + tid * kPer);
    const uint4 h0 = __ldcg(h4), h1 = __ldcg(h4 + 1), b0 = __ldcg(b4), b1 = __ldcg(b4 + 1);
    const uint32_t v[kPer] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w}, b[kPer] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    uint32_t sum = 0;
#pragma unroll
    for (uint32_t k = 0; k < kPer; ++k) sum += tid * kPer + k < cd.C ? v[k] : 0u;
    uint32_t inc = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t n = __shfl_up_sync(0xFFFFFFFFu, inc, d); if ((int)lane >= d) inc += n; }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    uint32_t run = inc - sum;
    for (uint32_t w = 0; w < warp; ++w) run += s_warp[w];
#pragma unroll
    for (uint32_t k = 0; k < kPer; ++k) {  // class start + this CTA's first position inside the class
        const uint32_t i = tid * kPer + k;
        if (i < cd.C) { s_base[i] = run + b[k]; run += v[k]; }
    }
    __syncthreads();
    if (blockIdx.x == 0) publish_group_totals(a, cd);
    // pass 2: positions (the order inside a class is arbitrary -- results go back by row id).  kK0Batch chunks at a
    // time: every key and threshold word is loaded, then every position taken, then every pair stored.
    uint32_t n_neither = 0;
    for (uint32_t c0 = blockIdx.x * kPThreads; c0 < a.P; c0 += kK0Batch * stride) {  // whole warps: the ballot below
        uint32_t key[kK0Batch], w[kK0Batch], dst[kK0Batch];
#pragma unroll
        for (int u = 0; u < kK0Batch; ++u) {
            const uint32_t p = c0 + (uint32_t)u * stride + tid;
            key[u] = p < a.P ? (uint32_t)a.key[p] : kNone;
            w[u] = p < a.P ? a.rw[p] : 0u;
        }
#pragma unroll
        for (int u = 0; u < kK0Batch; ++u) dst[u] = key[u] < 0xFFFFu ? atomicAdd(&s_base[key[u]], 1u) : 0u;
#pragma unroll
        for (int u = 0; u < kK0Batch; ++u) {
            const uint32_t p = c0 + (uint32_t)u * stride + tid;
            const bool neither = key[u] == 0xFFFFu;
            if (key[u] < 0xFFFFu) a.ord_rw[dst[u]] = make_uint2(p, cd.slice ? slice_rw(cd, a.pk, w[u]) : w[u]);  // the one scattered store of the sort
            if (neither) finish_row_no_cloud(a, p);
            n_neither += (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, neither));
        }
    }
    if (n_neither) count_rows_done(a, n_neither);
}

// ---------------------------------------------------------------------------------------------------------
// K1: persistent grid kernel
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 lds4(const uint32_t* p) { return *reinterpret_cast<const uint4*>(p); }

template <int RPL, bool NV, bool NR>
__device__ __forceinline__ void walk(const uint32_t* __restrict__ stage, uint32_t w68, int sub_lo, int sub_hi, const uint32_t (&o1)[RPL],
                                     const uint32_t (&o2)[RPL], const uint32_t (&o3)[RPL], uint32_t (&bb)[RPL]) {
    for (int sub = sub_hi - 1; sub >= sub_lo; --sub) {  // descending price: the last hit is the cheapest
        const uint32_t* sp = stage + (size_t)sub * w68;
#pragma unroll
        for (int b8 = 7; b8 >= 0; --b8) {
#pragma unroll
            for (int r = 0; r < RPL; ++r) {
                const uint4 a0 = lds4(sp + o1[r] + b8 * 8), a1 = lds4(sp + o1[r] + b8 * 8 + 4);
                uint32_t any;
                if (!NV && !NR) {
                    any = (a0.x | a0.y | a0.z) | (a0.w | a1.x | a1.y) | (a1.z | a1.w);
                } else if (NV != NR) {
                    const uint32_t ob = NV ? o2[r] : o3[r];
                    const uint4 b0 = lds4(sp + ob + b8 * 8), b1 = lds4(sp + ob + b8 * 8 + 4);
                    any = (a0.x & b0.x) | (a0.y & b0.y);
                    any |= (a0.z & b0.z); any |= (a0.w & b0.w);
                    any |= (a1.x & b1.x); any |= (a1.y & b1.y);
                    any |= (a1.z & b1.z); any |= (a1.w & b1.w);
                } else {
                    const uint4 b0 = lds4(sp + o2[r] + b8 * 8), b1 = lds4(sp + o2[r] + b8 * 8 + 4);
                    const uint4 c0 = lds4(sp + o3[r] + b8 * 8), c1 = lds4(sp + o3[r] + b8 * 8 + 4);
                    any = (a0.x & b0.x & c0.x) | (a0.y & b0.y & c0.y) | (a0.z & b0.z & c0.z);
                    any |= (a0.w & b0.w & c0.w) | (a1.x & b1.x & c1.x);
                    any |= (a1.y & b1.y & c1.y) | (a1.z & b1.z & c1.z);
                    any |= (a1.w & b1.w & c1.w);
                }
                if (any) bb[r] = (uint32_t)(sub * 8 + b8);
            }
        }
    }
}

struct PersistArgs {
    uint32_t S, per, qspan, n_groups, tickets_per_block;
    uint32_t slice, groups, groups_per_cloud;  // slice: stages are cut from bitmapM; row groups in all / per cloud
};

// The (group, stage) queue CTA `cta` of `grid` serves when every queue has at least one CTA.  Queue q = (non-empty row
// group q / S, stage q % S) holds the group's weighted rows times the sub-ranges of the stage -- the walk covers whole
// sub-ranges, the table's partial last one included, so the last stage can be the lighter one.  A CTA keeps its queue
// for the whole call, so the call ends when the queue with the most work per CTA drains: the split minimises that.
// Bisection finds (to float precision) the least load per CTA T for which max(1, ceil(load / T)) CTAs per queue add
// up to at most `grid`; each queue gets that many, and any CTAs left over join queues 0, 1, ... one each.  Whole warp
// (lane l owns a run of queues: 32 halvings of a few divisions each); every CTA computes the same split from the same
// totals.  work: per non-empty group.
__device__ uint32_t persist_queue_of(uint32_t cta, uint32_t grid, uint32_t npairs, uint32_t S, uint32_t per, uint32_t nsub,
                                     const uint32_t* work) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t k = (npairs + 31) / 32, q0 = min(npairs, lane * k), q1 = min(npairs, q0 + k);
    auto load = [&](uint32_t q) { return (float)max(work[q / S], 1u) * (float)min(per, nsub - q % S * per); };
    auto ctas = [&](uint32_t q, float T) { return (uint32_t)fmaxf(1.f, ceilf(load(q) / T)); };
    auto need = [&](float T) {
        uint32_t n = 0;
        for (uint32_t q = q0; q < q1; ++q) n += ctas(q, T);
#pragma unroll
        for (int d = 16; d; d >>= 1) n += __shfl_xor_sync(0xFFFFFFFFu, n, d);
        return n;
    };
    float tot = 0.f, hi = 0.f;
    for (uint32_t q = q0; q < q1; ++q) { tot += load(q); hi = fmaxf(hi, load(q)); }
#pragma unroll
    for (int d = 16; d; d >>= 1) { tot += __shfl_down_sync(0xFFFFFFFFu, tot, d); hi = fmaxf(hi, __shfl_xor_sync(0xFFFFFFFFu, hi, d)); }
    float lo = __shfl_sync(0xFFFFFFFFu, tot, 0) / (float)grid;  // no split does better; hi (one CTA each) fits: npairs <= grid
    for (int i = 0; i < 32; ++i) {
        const float mid = 0.5f * (lo + hi);
        if (need(mid) <= grid) hi = mid; else lo = mid;
    }
    uint32_t mine = 0;
    for (uint32_t q = q0; q < q1; ++q) mine += ctas(q, hi);
    uint32_t incl = mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t n = __shfl_up_sync(0xFFFFFFFFu, incl, d); if ((int)lane >= d) incl += n; }
    const uint32_t total = __shfl_sync(0xFFFFFFFFu, incl, 31);
    if (cta >= total) return (cta - total) % npairs;
    uint32_t found = kNone;
    if (incl - mine <= cta && cta < incl)
        for (uint32_t q = q0, acc = incl - mine; q < q1 && found == kNone; ++q) { acc += ctas(q, hi); if (cta < acc) found = q; }
    const uint32_t owner = __ffs(__ballot_sync(0xFFFFFFFFu, found != kNone)) - 1;
    return __shfl_sync(0xFFFFFFFFu, found, owner);
}

// 96 registers: the CTA owns the SM's shared memory, and 16K registers stay free -- exactly one 256-thread CTA of the
// status sweep kernel, so a sweep enqueued beside the select (other stream) really runs side by side with it, one kernel
// bound by shared memory, the other by HBM and integer multiplies.  With the whole register file (128 per thread) the
// sweep could not start on the SM until the select is over -- or, if it got there first, would delay it.
__global__ void __maxnreg__(96) k_select_persist(SelectArgs a, PersistArgs pa) {
    constexpr int RPL = kRpl;
    extern __shared__ __align__(128) uint32_t s_stage[];
    __shared__ __align__(8) uint64_t s_bar[kCopyGroups];
    __shared__ uint32_t s_first, s_ng;
    // the non-empty row groups in class order: group id, rows, first row (of the class order), first row block, work
    __shared__ uint32_t s_grp[kMaxGroups], s_rows[kMaxGroups], s_start[kMaxGroups], s_blk0[kMaxGroups], s_work[kMaxGroups];
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    constexpr uint32_t RPI = 32 * RPL;  // rows per item
    if (tid == 0) {
        for (int g = 0; g < kCopyGroups; ++g) mbar_init(&s_bar[g], 1);
        mbar_fence_init();
    }
    pdl_wait();     // k_pod_scatter (and k_pod_classify before it) has completed
    pdl_trigger();  // a dependent (the peer wait) may be scheduled; it waits for this grid to complete
    // the scatter kernel is done with the class counts: zero them for the next call (all kMaxClasses words -- the table,
    // and with it the class count, may change between calls)
    if (blockIdx.x == 0) for (uint32_t i = tid; i < kMaxClasses; i += kPThreads) a.hist[i] = 0u;
    if (tid < 32) {
        uint32_t row_run = 0, blk_run = 0, n_ne = 0;
        for (uint32_t g0 = 0; g0 < pa.groups; g0 += 32) {
            const uint32_t g = g0 + lane;
            const uint32_t r = g < pa.groups ? __ldcg(a.hdr + kHdrGroupRows + g) : 0u, b = (r + RPI - 1) / RPI;
            uint32_t ir = r, ib = b;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t xr = __shfl_up_sync(0xFFFFFFFFu, ir, d), xb = __shfl_up_sync(0xFFFFFFFFu, ib, d);
                if ((int)lane >= d) { ir += xr; ib += xb; }
            }
            const uint32_t ne = __ballot_sync(0xFFFFFFFFu, r != 0);
            if (r) {
                const uint32_t j = n_ne + __popc(ne & ((1u << lane) - 1u));
                s_grp[j] = g; s_rows[j] = r; s_start[j] = row_run + ir - r; s_blk0[j] = blk_run + ib - b;
                s_work[j] = __ldcg(a.hdr + kHdrGroupWork + g);
            }
            row_run += __shfl_sync(0xFFFFFFFFu, ir, 31); blk_run += __shfl_sync(0xFFFFFFFFu, ib, 31); n_ne += __popc(ne);
        }
        if (lane == 0) s_ng = n_ne;
    }
    __syncthreads();
    const uint32_t S = pa.S, w68 = (pa.slice ? a.pk.slice_rows : a.pk.bm_words) * kSubWords;
    const uint32_t npairs = S * s_ng;  // 0: every row was final in the scatter kernel (neither cloud); only the push is left
    // which (group, stage) queues this CTA serves: with at least as many CTAs as queues the CTAs are shared out over
    // the queues in proportion to their work (persist_queue_of) and every CTA keeps one queue for the whole call;
    // otherwise CTA b serves queues b, b + grid, ... one after the other
    uint32_t first, step;
    if (npairs == 0) {
        first = 0; step = 1;
    } else if (npairs <= gridDim.x) {
        if (tid < 32) { const uint32_t q = persist_queue_of(blockIdx.x, gridDim.x, npairs, S, pa.per, a.nsub, s_work); if (lane == 0) s_first = q; }
        __syncthreads();
        first = s_first;
        step = npairs;  // one queue only
    } else {
        first = blockIdx.x; step = gridDim.x;
    }
    const uint32_t w_none = pa.slice ? 0u : (a.pk.bm_off_vcpu << 8) | (a.pk.bm_off_ram << 16);  // padding rows: no constraint
    // an item that covers the whole table (one stage, one item per row block) leaves its rows final: no merge
    const bool direct = pa.tickets_per_block == 1;
    uint32_t it = 0, phase_bits = 0;  // bit g: parity of copy group g's next completion (groups are not all used by every stage)
    uint32_t last_used = 0, last_parity = 0;  // the copy groups of the stage loaded last, and the parity they complete with
    for (uint32_t pair = first; pair < npairs; pair += step, ++it) {
        const uint32_t gi = pair / S, s = pair % S, grp = s_grp[gi];
        const uint32_t c = grp / pa.groups_per_cloud;
        const uint32_t* src = pa.slice ? a.view[c].bitmapM + (size_t)(grp % pa.groups_per_cloud) * a.nsub * w68 : a.view[c].bitmapT;
        const uint32_t sub0 = s * pa.per, nsubs = min(pa.per, a.nsub - sub0);
        const uint32_t gs = (nsubs + pa.n_groups - 1) / pa.n_groups;  // subs per copy group
        if (it) __syncthreads();  // every warp is done with the previous stage
        uint32_t used = 0;
        for (uint32_t g = 0; g * gs < nsubs; ++g) {
            used |= 1u << g;
            if (tid == 0) {
                const uint32_t g0 = g * gs, gn = min(gs, nsubs - g0);
                mbar_expect_tx(&s_bar[g], gn * w68 * 4u);
                bulk_g2s(s_stage + (size_t)g0 * w68, src + ((size_t)sub0 + g0) * w68, gn * w68 * 4u, &s_bar[g]);
            }
        }
        const uint32_t parity = phase_bits;
        phase_bits ^= used;
        last_used = used; last_parity = parity;
        uint32_t ready = 0;  // copy groups this warp has seen complete
        const uint32_t n_c = s_rows[gi], c_start = s_start[gi];
        const uint32_t nblk = (n_c + RPI - 1) / RPI;
        const uint32_t Qi = (nsubs + pa.qspan - 1) / pa.qspan;
        const uint32_t n_items = nblk * Qi;
        uint32_t* cursor = a.hdr + kHdrCursors + grp * S + s;
        uint32_t* tickets = a.tile_ctr + s_blk0[gi];
        uint32_t item = 0;
        if (lane == 0) item = atomicAdd(cursor, 1u);
        item = __shfl_sync(0xFFFFFFFFu, item, 0);
        uint32_t w_cur[RPL];
#pragma unroll
        for (int r = 0; r < RPL; ++r) {
            const uint32_t local = (item / Qi) * RPI + (uint32_t)r * 32 + lane;
            w_cur[r] = item < n_items && local < n_c ? __ldcg(a.ord_rw + c_start + local).y : w_none;
        }
        uint32_t pend1_blk = kNone, pend2_blk = kNone, pend2_ticket = 0;  // merge pipeline (see below)
        // the row block whose ticket was taken one iteration ago: if that was its last ticket, every segment of its rows
        // has been merged -- price < maxPrice on the winner, position -> offer index
        auto retire = [&](uint32_t rblk, uint32_t ticket) {
            if (rblk == kNone) return;
            if (__shfl_sync(0xFFFFFFFFu, ticket, 0) != pa.tickets_per_block - 1) return;
            __threadfence();
            if (lane == 0) tickets[rblk] = 0u;  // self-cleaning
            uint32_t n_final = 0;
#pragma unroll
            for (int r = 0; r < RPL; ++r) {
                const uint32_t local = rblk * RPI + (uint32_t)r * 32 + lane;
                const bool ok = local < n_c;
                n_final += (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, ok));
                if (ok) finish_row(a, a.view[c], a.ord_rw[c_start + local].x, __ldcg(a.pos + c_start + local));
            }
            count_rows_done(a, n_final);
            if (a.n_out > 1 && a.self_out < 0) __threadfence_system();  // direct peer stores: performed before the grid completes
        };
        while (item < n_items) {
            uint32_t next = 0;
            if (lane == 0) next = atomicAdd(cursor, 1u);  // in flight while this item is walked
            const uint32_t blk = item / Qi, qi = item - blk * Qi;
            const int sub_lo = (int)(qi * pa.qspan), sub_hi = (int)min(nsubs, (qi + 1) * pa.qspan);
            uint32_t idx[RPL], o1[RPL], o2[RPL], o3[RPL], bb[RPL];
            bool valid[RPL];
            bool nv = false, nr = false;
#pragma unroll
            for (int r = 0; r < RPL; ++r) {
                const uint32_t local = blk * RPI + (uint32_t)r * 32 + lane;
                valid[r] = local < n_c;
                idx[r] = c_start + local;
                const uint32_t w = w_cur[r];
                const uint32_t i1 = w & 0xFFu, i2 = (w >> 8) & 0xFFu, i3 = (w >> 16) & 0xFFu;
                o1[r] = i1 * kSubWords; o2[r] = i2 * kSubWords; o3[r] = i3 * kSubWords;
                // slice: a second word only when both vcpu and ram constrain (i3 = i1 never adds one)
                if (pa.slice) nv |= i2 != i1;
                else { nv |= i2 != a.pk.bm_off_vcpu; nr |= i3 != a.pk.bm_off_ram; }
                bb[r] = kNone;
            }
            nv = __any_sync(0xFFFFFFFFu, nv); nr = __any_sync(0xFFFFFFFFu, nr);
            for (uint32_t g = (uint32_t)sub_lo / gs; g * gs < (uint32_t)sub_hi; ++g)
                if (!(ready >> g & 1u)) { mbar_wait(&s_bar[g], parity >> g & 1u); ready |= 1u << g; }
            // rows of an item share the "column constrains" flags except at class boundaries; a word a row does not
            // need is all-available for it (price stages: the column's threshold 0; slice: its own first word)
            if (!nv && !nr) walk<RPL, false, false>(s_stage, w68, sub_lo, sub_hi, o1, o2, o3, bb);
            else if (nv && !nr) walk<RPL, true, false>(s_stage, w68, sub_lo, sub_hi, o1, o2, o3, bb);
            else if (!nv && nr) walk<RPL, false, true>(s_stage, w68, sub_lo, sub_hi, o1, o2, o3, bb);
            else walk<RPL, true, true>(s_stage, w68, sub_lo, sub_hi, o1, o2, o3, bb);
            // The merge of an item costs two device-wide round trips (its atomicMin's must be performed before its ticket is
            // taken, and the ticket's return value says whether these rows are final), so it is pipelined over the
            // NEXT items' walks: here the item walked one iteration ago takes its ticket (its atomicMin's were issued a
            // whole walk ago: the fence returns at once), and the item before that reads its ticket and, if it was the
            // last one of its row block, runs the epilogue.  Direct items never enter the pipeline.
            retire(pend2_blk, pend2_ticket);
            pend2_blk = pend1_blk; pend2_ticket = 0;
            if (pend1_blk != kNone) {
                __threadfence();
                if (lane == 0) pend2_ticket = atomicAdd(&tickets[pend1_blk], 1u);  // consumed after the next walk
            }
            // the next item's thresholds are fetched under this item's resolve and the next walk's start
            const uint32_t item_next = __shfl_sync(0xFFFFFFFFu, next, 0);
#pragma unroll
            for (int r = 0; r < RPL; ++r) {
                const uint32_t local = (item_next / Qi) * RPI + (uint32_t)r * 32 + lane;
                w_cur[r] = item_next < n_items && local < n_c ? __ldcg(a.ord_rw + c_start + local).y : w_none;
            }
            uint32_t n_final = 0;
#pragma unroll
            for (int r = 0; r < RPL; ++r) {
                uint32_t p = kNone;
                if (valid[r] && bb[r] != kNone) {  // re-read the cheapest block with a hit: first chunk, first bit
                    const uint32_t sub = bb[r] >> 3, b8 = bb[r] & 7u;
                    const uint32_t* sp = s_stage + (size_t)sub * w68 + b8 * 8;
                    uint32_t j = 0, m = 0;
#pragma unroll
                    for (int k = 7; k >= 0; --k) {
                        const uint32_t mk = sp[o1[r] + k] & sp[o2[r] + k] & sp[o3[r] + k];
                        if (mk) { j = (uint32_t)k; m = mk; }
                    }
                    p = (((sub0 + sub) * kSubChunks + b8 * 8 + j) << 5) + (uint32_t)__ffs(m) - 1u;
                }
                if (direct) {
                    n_final += (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, valid[r]));
                    if (valid[r]) finish_row(a, a.view[c], a.ord_rw[idx[r]].x, p);
                } else if (p != kNone) {
                    atomicMin(&a.pos[idx[r]], p);
                }
            }
            if (direct) {
                count_rows_done(a, n_final);
                if (a.n_out > 1 && a.self_out < 0) __threadfence_system();
            }
            pend1_blk = direct ? kNone : blk;
            item = item_next;
        }
        // drain the pipeline: the last two items of this stage
        retire(pend2_blk, pend2_ticket);
        pend2_blk = pend1_blk; pend2_ticket = 0; pend1_blk = kNone;
        if (pend2_blk != kNone) {
            __threadfence();
            if (lane == 0) pend2_ticket = atomicAdd(&tickets[pend2_blk], 1u);
        }
        retire(pend2_blk, pend2_ticket);
        pend2_blk = kNone;
    }
    // A warp waits only on the copy groups its items cover, so a CTA that found its queue already drained has waited on
    // none of its stage's bulk copies.  Shared memory lives as long as its CTA, and nothing in the PTX ISA makes the
    // CTA's exit wait for asynchronous writes into it: drain the last stage's copies before this CTA can exit (a group
    // some warp already waited on returns at once; earlier stages were drained by their items before the next load).
    if (tid == 0)
        for (uint32_t g = 0; g < (uint32_t)kCopyGroups; ++g)
            if (last_used >> g & 1u) mbar_wait(&s_bar[g], last_parity >> g & 1u);
    push_tail(a);
}

// ---------------------------------------------------------------------------------------------------------
// peer signal / wait.  The persistent kernel signals from its last pusher; the other select paths, a top-5 gather (behind
// the lists' push) and an empty shard launch k_peer_signal behind their kernels, and so does rpk_peer_fence (signal and
// wait in one); k_peer_wait is the wait half for a bound group.
// ---------------------------------------------------------------------------------------------------------
__global__ void k_peer_signal(PeerGroup g, uint32_t epoch, uint32_t wait) {
    pdl_wait();  // everything this stream did before (peer stores included) has completed
    signal_peers(g, kFlagSelect, kFlagSelectCtr, epoch, wait != 0);
}

__global__ void k_peer_wait(PeerGroup g, uint32_t what) {
    pdl_wait();  // the kernels that signalled for this rank have completed: the own epoch counters are final
    const uint32_t lane = threadIdx.x;
    const volatile uint32_t* mine = g.flags[g.my_rank];
    if ((int)lane < g.n) {
        if (what & 1u) { const uint32_t e = mine[kFlagSelectCtr]; while ((int32_t)(mine[kFlagSelect + lane] - e) < 0) __nanosleep(32); }
        if (what & 2u) { const uint32_t e = mine[kFlagStatusCtr]; while ((int32_t)(mine[kFlagStatus + lane] - e) < 0) __nanosleep(32); }
        __threadfence_system();
    }
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
uint32_t persist_hdr_words(const PersistPlan& pl) { return kHdrCursors + pl.n_cursors + 8; }

PersistPlan persist_plan(const SelectArgs& a, int sm_count) {
    const Tune t = read_tune();
    PersistPlan pl;
    uint32_t max_stage = (uint32_t)(t.stage_kb > 0 ? t.stage_kb : 220) * 1024u;
    if (max_stage > 220u * 1024u) max_stage = 220u * 1024u;
    // Stages per mem threshold (bitmapM) when the view exists and one of its sub-ranges fits a stage: a row then reads
    // one mask word per chunk, two when both its vcpu and ram requests constrain, instead of one per constraining
    // column plus mem.  A queue is (cloud, mem threshold, stage), and at the usual table sizes one stage holds the whole
    // slice.  Otherwise a stage is a price range of the per-threshold view bitmapT and a queue is (cloud, stage).
    const uint32_t slice_bytes = a.pk.slice_rows * kSubWords * 4u;
    pl.slice = a.pk.slice_rows && !a.pk.no_slice && slice_bytes <= max_stage ? 1u : 0u;
    const uint32_t sub_bytes = pl.slice ? slice_bytes : a.pk.bm_words * kSubWords * 4u;
    uint32_t cap = max_stage / sub_bytes;
    if (cap == 0) cap = 1;
    const uint32_t S = (a.nsub + cap - 1) / cap;
    const uint32_t per = (a.nsub + S - 1) / S;
    pl.S = (a.nsub + per - 1) / per; pl.per = per;
    pl.smem_bytes = per * sub_bytes;
    pl.grid = (uint32_t)sm_count;  // one CTA per SM: the stage takes the SM's shared memory
    pl.sm_count = sm_count;
    const uint64_t warps = (uint64_t)pl.grid * kPWarps;
    const uint64_t nblk = ((uint64_t)a.P + 32u * kRpl - 1) / (32u * kRpl);
    const uint64_t want = (uint64_t)(t.items_per_warp > 0 ? t.items_per_warp : 4) * warps;  // items per warp: the tail is one item long
    const uint64_t visits = nblk * pl.S > 0 ? nblk * pl.S : 1;  // (row block, stage) visits
    uint64_t Qi = (want + visits - 1) / visits;
    if (Qi < 1) Qi = 1;
    if (Qi > per) Qi = per;
    pl.qspan = (uint32_t)((per + Qi - 1) / Qi);
    pl.n_cursors = (pl.slice ? 2u * (a.D[0] + 1u) : 2u) * pl.S;
    // K0: one wave of CTAs (four per SM), each looping over 512-row chunks.  Four fill an SM's threads, so a status
    // sweep enqueued beside the select waits for K0 and then runs beside K1.  Three per SM would let the sweep in
    // beside K0, but the two then share HBM and K0 is on the select's critical path: with a 1M-slot sweep beside it, a
    // 1M-row select took 383 us that way against 376 us with four (H100 SXM, 400 W, profiles/h100_step_sweep.json).
    const uint32_t chunks = (a.P + kPThreads - 1) / kPThreads;
    const uint32_t k0ctas = t.k0ctas > 0 ? (uint32_t)t.k0ctas : 4u * (uint32_t)sm_count;
    pl.k0_blocks = chunks < k0ctas ? (chunks ? chunks : 1u) : k0ctas;
    return pl;
}

int launch_select_persist(const SelectArgs& args, const PersistPlan& pl, cudaStream_t st) {
    const Tune t = read_tune();
    SelectArgs a = args;
    a.slice = pl.slice;
    PersistArgs pa;
    pa.S = pl.S; pa.per = pl.per; pa.qspan = pl.qspan;
    pa.slice = pl.slice; pa.groups_per_cloud = pl.slice ? a.D[0] + 1u : 1u; pa.groups = 2u * pa.groups_per_cloud;
    pa.n_groups = pl.per < (uint32_t)kCopyGroups ? pl.per : (uint32_t)kCopyGroups;
    uint32_t tickets = 0;
    for (uint32_t s = 0; s < pl.S; ++s) {
        const uint32_t sub0 = s * pl.per, nsubs = a.nsub - sub0 < pl.per ? a.nsub - sub0 : pl.per;
        tickets += (nsubs + pl.qspan - 1) / pl.qspan;
    }
    pa.tickets_per_block = tickets;
    // K0 over pl.k0_blocks CTAs: both kernels must use the same grid (a scatter CTA reads the class bases its classify
    // twin wrote for the same rows)
    const uint32_t blocks = pl.k0_blocks;
    k_pod_classify<<<blocks, kPThreads, 0, st>>>(a, pl.n_cursors, pa.tickets_per_block != 1 ? 1u : 0u);
    launch_pdl(k_pod_scatter, dim3(blocks), dim3(kPThreads), 0, st, t.pdl, a);
    static thread_local int attr_dev = -1;
    allow_smem(k_select_persist, 224 * 1024, &attr_dev);
    launch_pdl(k_select_persist, dim3(pl.grid), dim3(kPThreads), pl.smem_bytes, st, t.pdl, a, pa);
    RPK_CUDA(cudaGetLastError());
    return 3;
}

int launch_peer_signal(const PeerGroup& g, uint32_t epoch, bool wait, cudaStream_t st) {
    launch_pdl(k_peer_signal, dim3(1), dim3(32), 0, st, read_tune().pdl, g, epoch, wait ? 1u : 0u);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

int launch_peer_wait(const PeerGroup& g, uint32_t what, cudaStream_t st) {
    launch_pdl(k_peer_wait, dim3(1), dim3(32), 0, st, read_tune().pdl, g, what);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace rpk
