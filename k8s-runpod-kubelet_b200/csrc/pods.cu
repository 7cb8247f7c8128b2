// pods.cu -- the pod-requirement table: the five pod columns of every tracked pod, kept on each GPU and indexed by
// the slot ids the Provider already gives the status table, so that a pending-pod tick (processPendingPods,
// kubelet.go:747-814) uploads 4 bytes of slot id per pod instead of the 21 bytes of its columns.
//
// Kernels:
//   k_pod_fill      every row := the columns of a pod with no annotations, not pending (rpk_pods_reset)
//   k_pod_seed      row slots[i] := element i of each staged column; a NULL column writes its default (rpk_pods_seed_slots)
//   k_pod_gather    compact columns of one rpk_select_slots sub-batch, or of one rpk_select_slots_device* call: element
//                   i := row slots[i] of the table, written into the lane's pod-column buffers, which the select kernels
//                   then read as rpk_select's uploaded ones
//   k_pod_mark      pending flag of slot slots[i] := pending[i] != 0 (rpk_pods_mark_pending)
//   k_pod_pending   the ascending list of the slots whose flag is set, and their number: what rpk_select_pending selects
//                   over and rpk_pods_pending_list_device returns.  The list is in range by construction, so no host
//                   check and no upload stand before the gather.
//   k_pod_stale     of one GPU's owned slots: the ascending list of the pending slots whose stored result is stale, their
//                   number and the number of pending slots (rpk_select_pending_changed*, before the reselect)
//   k_pod_stale_reach  the same against a non-empty change window of rpk_offers_refresh: a result older than the
//                   current table is stale only below the floor or when a changed offer reaches the row
//   k_pod_result_diff_xchg  over the rows k_pod_reselect_top5 returned, their number read on the device: store each
//                   row's result and write the rows whose list changed, ascending, into one region per output (the
//                   host call: its device copy of the rows; the one-process-per-GPU forms: region my_rank of every
//                   rank's exchange buffer), then a peer signal if a group is bound (rpk_select_pending_changed[_gather],
//                   rpk_select_pending_changed_device_gather)
// The host entry points check every slot against the table's N before its upload.  The device entry points cannot, so
// an entry outside [0, N) is defined here: the seed skips it, and the gather writes a row with cloud byte kCloudNone,
// which every select path finishes as "neither cloud" (runpod_client.go:469-475): -1 and five -1.  No caller input
// can make these kernels touch memory outside the table.
#include <algorithm>

#include "rpk_device.cuh"
#include "rpk_internal.cuh"

namespace rpk {
using namespace dev;

constexpr int kPodThreads = 256;
constexpr int32_t kDefaultMemGb = 16;  // extractGPUMemory("") (runpod_client.go:1182)
constexpr uint8_t kCloudNone = 2;      // neither RPK_CLOUD_SECURE nor RPK_CLOUD_COMMUNITY: no offer is feasible

__global__ void k_pod_fill(PodRows t, uint8_t* __restrict__ pending, uint32_t N) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
        t.mem[i] = kDefaultMemGb; t.vcpu[i] = 0; t.ram[i] = 0; t.max_price[i] = RPK_DEFAULT_MAX_PRICE; t.cloud[i] = RPK_CLOUD_SECURE;
        pending[i] = 0;
    }
}

__global__ void k_pod_seed(PodRows t, uint32_t N, uint32_t n, const uint32_t* __restrict__ slots, PodCols in) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = slots[i];
    if (s >= N) return;
    t.mem[s] = in.req_mem[i];
    t.vcpu[s] = in.req_vcpu ? in.req_vcpu[i] : 0;
    t.ram[s] = in.req_ram ? in.req_ram[i] : 0;
    t.max_price[s] = in.max_price ? in.max_price[i] : RPK_DEFAULT_MAX_PRICE;
    t.cloud[s] = in.cloud ? in.cloud[i] : (uint8_t)RPK_CLOUD_SECURE;
}

__global__ void k_pod_gather(PodRows t, uint32_t N, uint32_t n, const uint32_t* __restrict__ slots, PodRows out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = slots[i];
    if (s >= N) {  // a row nothing matches; the other columns hold a pod with no annotations
        out.mem[i] = kDefaultMemGb; out.vcpu[i] = 0; out.ram[i] = 0; out.max_price[i] = RPK_DEFAULT_MAX_PRICE; out.cloud[i] = kCloudNone;
        return;
    }
    out.mem[i] = __ldg(t.mem + s); out.vcpu[i] = __ldg(t.vcpu + s); out.ram[i] = __ldg(t.ram + s);
    out.max_price[i] = __ldg(t.max_price + s); out.cloud[i] = __ldg(t.cloud + s);
}

// ---- pending set -------------------------------------------------------------------------------------------
__global__ void k_pod_mark(uint8_t* __restrict__ flags, uint32_t N, uint32_t n, const uint32_t* __restrict__ slots,
                           const uint8_t* __restrict__ pending) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = slots[i];
    if (s < N) flags[s] = pending[i] != 0;
}

// Ordered stream compaction of the flag column.  A unit is 16 slots (one 16-byte load), a tile the kPendThreads units a
// CTA turns into list entries per round.  A CTA takes its id from a ticket and owns the id-th contiguous share of the
// units.  Pass 1 counts the CTA's set flags, four independent loads per thread in flight; the count is published and the
// counts of the CTAs before it are summed (sum_before: those CTAs have started, since ids follow scheduling order, so
// the kernel may share the GPU with a select or a sweep).  Pass 2 reads the share again (a CTA's share of a 1M-slot
// table is 8 KB: it hits L1 / L2) tile by tile: a block scan of the per-unit counts places every id in a shared-memory
// tile, which goes out in coalesced stores at the CTA's offset.  The output is ascending whatever the CTA scheduling.
// The last CTA to finish zeroes the look-back state and the tickets, so no memset stands before the next launch and a
// captured launch can be replayed.
constexpr int kPendThreads = 256;
constexpr uint32_t kPendUnit = 16;
constexpr uint32_t kPendTile = (uint32_t)kPendThreads * kPendUnit;

// the 16 flags of unit u as four words (slot 16 u + k in byte k); the last unit of a table whose N is not a multiple of 16
// is read byte by byte, so nothing outside [0, N) is read
__device__ __forceinline__ uint4 load_flags(const uint8_t* __restrict__ flags, uint32_t u, uint32_t N) {
    const uint32_t s0 = u * kPendUnit;
    if (N - s0 >= kPendUnit) return __ldg(reinterpret_cast<const uint4*>(flags) + u);
    uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (uint32_t k = 0; k < kPendUnit; ++k)
        if (k < N - s0) w[k >> 2] |= (uint32_t)__ldg(flags + s0 + k) << ((k & 3u) * 8u);
    return make_uint4(w[0], w[1], w[2], w[3]);
}
__device__ __forceinline__ uint32_t count_flags(const uint4& v) {
    return (uint32_t)(__popc(__vcmpne4(v.x, 0u)) + __popc(__vcmpne4(v.y, 0u)) + __popc(__vcmpne4(v.z, 0u)) + __popc(__vcmpne4(v.w, 0u))) >> 3;
}

// The compaction itself, shared by the kernels that turn 16-item units into an ascending list: k_pod_pending (units of
// the flag column), k_pod_stale[_reach] (units of a GPU's owned slots) and k_pod_result_diff_xchg (units of the reselected
// rows).
// The policy Pol says what a unit holds:
//   prepare(c_lo, c_hi)             every thread, once the CTA's share [c_lo, c_hi) is known, before pass 1
//   V none()                        a unit past the CTA's share
//   V load(u)                       pass 1's view of unit u
//   V reload(u)                     pass 2's view of unit u (the thread that loaded u in pass 1: u - c_lo is the same
//                                   modulo kPendThreads in both passes, so a policy may hand pass 2 what pass 1 wrote)
//   Count count1(V)                 pass 1: the unit's kept items in the low 32 bits (anything else above them)
//   uint32_t count(V), bool keep(V, k), uint32_t id(u, k), emit(i, id)   pass 2: list entry i := id of kept item k of u
//   set_count(n)                    the list's length (the last CTA in unit order)
//   cta_total(Count)                the CTA's pass-1 total, once per CTA
//   fence()                         every thread, after its last emit and before its CTA counts as finished
//   last()                          thread 0 of the CTA that finishes last, after every other CTA is done
//   last_warp()                     warp 0 of that CTA, after last()
template <class Pol>
__device__ __forceinline__ void compact_units(Pol& p, uint32_t n_units, unsigned long long* tile_state, uint32_t* ticket) {
    using V = typename Pol::V;
    using Count = typename Pol::Count;
    constexpr uint32_t kWarps = kPendThreads / 32;
    __shared__ uint32_t s_ids[kPendTile];
    __shared__ Count s_warp[kWarps];
    __shared__ uint32_t s_id, s_excl, s_last;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_id = atomicAdd(ticket, 1u);
    __syncthreads();
    const uint32_t cid = s_id, n_ctas = gridDim.x;
    const uint32_t c_lo = (uint32_t)((unsigned long long)n_units * cid / n_ctas), c_hi = (uint32_t)((unsigned long long)n_units * (cid + 1) / n_ctas);
    p.prepare(c_lo, c_hi);
    // ---- pass 1: the CTA's count -> its offset among the CTAs ----
    Count mine = 0;
    for (uint32_t u0 = c_lo + tid; u0 < c_hi; u0 += 4 * kPendThreads) {
        V v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t u = u0 + (uint32_t)k * kPendThreads;
            v[k] = u < c_hi ? p.load(u) : p.none();
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) mine += p.count1(v[k]);
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) mine += __shfl_xor_sync(0xFFFFFFFFu, mine, d);
    if (lane == 0) s_warp[warp] = mine;
    __syncthreads();
    if (warp == 0) {
        Count total = lane < kWarps ? s_warp[lane] : (Count)0;
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) total += __shfl_xor_sync(0xFFFFFFFFu, total, d);
        const uint32_t excl = sum_before(tile_state, cid, (uint32_t)total, lane);
        if (lane == 0) {
            s_excl = excl;
            if (cid == n_ctas - 1) p.set_count(excl + (uint32_t)total);  // the last CTA in unit order owns the count
            p.cta_total(total);
        }
    }
    __syncthreads();
    // ---- pass 2: one tile per round, thread t the t-th unit of the tile ----
    uint32_t at = s_excl;
    for (uint32_t r0 = c_lo; r0 < c_hi; r0 += kPendThreads) {
        const uint32_t u = r0 + tid;
        const V v = u < c_hi ? p.reload(u) : p.none();
        const uint32_t c = p.count(v);
        uint32_t inc = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t n = __shfl_up_sync(0xFFFFFFFFu, inc, d); if ((int)lane >= d) inc += n; }
        if (lane == 31) s_warp[warp] = inc;
        __syncthreads();
        uint32_t wbase = 0, round = 0;
#pragma unroll
        for (uint32_t w = 0; w < kWarps; ++w) { const uint32_t x = (uint32_t)s_warp[w]; if (w < warp) wbase += x; round += x; }
        uint32_t off = wbase + inc - c;
#pragma unroll
        for (uint32_t k = 0; k < kPendUnit; ++k)
            if (p.keep(v, k)) s_ids[off++] = p.id(u, k);
        __syncthreads();
        for (uint32_t i = tid; i < round; i += kPendThreads) p.emit(at + i, s_ids[i]);
        at += round;
        __syncthreads();  // the tile and the warp sums are rewritten by the next round
    }
    p.fence();
    __syncthreads();
    if (tid == 0) s_last = atomicAdd(ticket + 1, 1u) == n_ctas - 1 ? 1u : 0u;
    __syncthreads();
    if (!s_last) return;
    // last CTA to finish: every look-back is over -- clean the state for the next call
    for (uint32_t i = tid; i < n_ctas; i += kPendThreads) tile_state[i] = 0ull;
    if (tid == 0) { ticket[0] = 0u; ticket[1] = 0u; p.last(); }
    if (warp == 0) p.last_warp();
}

// k_pod_pending's units: 16 flag bytes, slot 16 u + k in byte k
struct FlagUnits {
    using V = uint4;
    using Count = uint32_t;
    const PendingArgs& a;
    __device__ __forceinline__ V none() const { return make_uint4(0u, 0u, 0u, 0u); }
    __device__ __forceinline__ V load(uint32_t u) const { return load_flags(a.flags, u, a.N); }
    __device__ __forceinline__ V reload(uint32_t u) const { return load_flags(a.flags, u, a.N); }
    __device__ __forceinline__ Count count1(const V& v) const { return count_flags(v); }
    __device__ __forceinline__ uint32_t count(const V& v) const { return count_flags(v); }
    __device__ __forceinline__ bool keep(const V& v, uint32_t k) const {
        const uint32_t w = k < 4 ? v.x : k < 8 ? v.y : k < 12 ? v.z : v.w;
        return (w >> ((k & 3u) * 8u)) & 0xFFu;
    }
    __device__ __forceinline__ uint32_t id(uint32_t u, uint32_t k) const { return u * kPendUnit + k; }
    __device__ __forceinline__ void emit(uint32_t i, uint32_t id) const { a.out[i] = id; }
    __device__ __forceinline__ void set_count(uint32_t n) const { *a.n_out = n; }
    __device__ __forceinline__ void cta_total(Count) const {}
    __device__ __forceinline__ void fence() const { __threadfence(); }
    __device__ __forceinline__ void last() const {}
    __device__ __forceinline__ void last_warp() const {}
    __device__ __forceinline__ void prepare(uint32_t, uint32_t) const {}
};

__global__ void __launch_bounds__(kPendThreads, 1024 / kPendThreads) k_pod_pending(PendingArgs a, uint32_t n_units) {
    FlagUnits p{a};
    compact_units(p, n_units, a.tile_state, a.ticket);
}

// ---- pending results (rpk_select_pending_changed) --------------------------------------------------------------
// bit k of the result: byte k of the 16 bytes of v is non-zero
__device__ __forceinline__ uint32_t nonzero_bytes16(const uint4& v) {
    const uint32_t w[4] = {__vcmpne4(v.x, 0u), __vcmpne4(v.y, 0u), __vcmpne4(v.z, 0u), __vcmpne4(v.w, 0u)};
    uint32_t m = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) m |= ((w[q] & 1u) | ((w[q] >> 7) & 2u) | ((w[q] >> 14) & 4u) | ((w[q] >> 21) & 8u)) << (4 * q);
    return m;
}
// bit k: a[k] != b[k], bit for bit, over 16 elements of 4 or 8 bytes (16-byte aligned)
__device__ __forceinline__ uint32_t differ16(const int32_t* a, const int32_t* b) {
    uint32_t m = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int4 x = reinterpret_cast<const int4*>(a)[q], y = reinterpret_cast<const int4*>(b)[q];
        m |= ((uint32_t)(x.x != y.x) | (uint32_t)(x.y != y.y) << 1 | (uint32_t)(x.z != y.z) << 2 | (uint32_t)(x.w != y.w) << 3) << (4 * q);
    }
    return m;
}
__device__ __forceinline__ uint32_t differ16(const double* a, const double* b) {
    uint32_t m = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const longlong2 x = reinterpret_cast<const longlong2*>(a)[q], y = reinterpret_cast<const longlong2*>(b)[q];
        m |= ((uint32_t)(x.x != y.x) | (uint32_t)(x.y != y.y) << 1) << (2 * q);
    }
    return m;
}
__device__ __forceinline__ uint32_t differ16(const uint8_t* a, const uint8_t* b) {
    const uint4 x = *reinterpret_cast<const uint4*>(a), y = *reinterpret_cast<const uint4*>(b);
    return nonzero_bytes16(make_uint4(x.x ^ y.x, x.y ^ y.y, x.z ^ y.z, x.w ^ y.w));
}

// k_pod_stale's units: 16 owned slots.  A slot is kept when it is pending and its stored result is stale: a generation
// other than the offer table's (0: never reported) or columns that differ from the table row.  Pass 1 leaves the kept
// bits in mask[u] for pass 2 and counts the pending slots above the kept ones.
struct StaleUnits {
    struct V { uint32_t keep, pend; };
    using Count = unsigned long long;
    const StaleArgs& a;
    __device__ __forceinline__ V none() const { return V{0u, 0u}; }
    __device__ __forceinline__ V load(uint32_t u) const {
        const uint32_t g = a.u_lo + u, j = u * kPendUnit;  // global unit, first owned index
        const uint32_t pm = nonzero_bytes16(load_flags(a.flags, g, a.N));
        uint32_t keep = 0;
        if (pm) {
            const uint32_t s = g * kPendUnit;
            uint32_t gen = 0;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const uint4 x = reinterpret_cast<const uint4*>(a.r.gen + j)[q];
                gen |= ((uint32_t)(x.x != a.gen) | (uint32_t)(x.y != a.gen) << 1 | (uint32_t)(x.z != a.gen) << 2 | (uint32_t)(x.w != a.gen) << 3) << (4 * q);
            }
            const uint32_t cols = differ16(a.t.mem + s, a.r.mem + j) | differ16(a.t.vcpu + s, a.r.vcpu + j) |
                                  differ16(a.t.ram + s, a.r.ram + j) | differ16(a.t.max_price + s, a.r.max_price + j) |
                                  differ16(a.t.cloud + s, a.r.cloud + j);
            keep = pm & (gen | cols);
        }
        a.mask[u] = (uint16_t)keep;
        return V{keep, (uint32_t)__popc(pm)};
    }
    __device__ __forceinline__ V reload(uint32_t u) const { return V{a.mask[u], 0u}; }
    __device__ __forceinline__ Count count1(const V& v) const { return (Count)v.pend << 32 | (uint32_t)__popc(v.keep); }
    __device__ __forceinline__ uint32_t count(const V& v) const { return (uint32_t)__popc(v.keep); }
    __device__ __forceinline__ bool keep(const V& v, uint32_t k) const { return (v.keep >> k) & 1u; }
    __device__ __forceinline__ uint32_t id(uint32_t u, uint32_t k) const { return (a.u_lo + u) * kPendUnit + k; }
    __device__ __forceinline__ void emit(uint32_t i, uint32_t id) const { a.out[i] = id; }
    __device__ __forceinline__ void set_count(uint32_t n) const { *a.n_out = n; }
    __device__ __forceinline__ void cta_total(Count total) const { atomicAdd(a.ticket + 2, (uint32_t)(total >> 32)); }
    __device__ __forceinline__ void fence() const { __threadfence(); }
    __device__ __forceinline__ void last() const { *a.n_pending = atomicExch(a.ticket + 2, 0u); }
    __device__ __forceinline__ void last_warp() const {}
    __device__ __forceinline__ void prepare(uint32_t, uint32_t) const {}
};

__global__ void __launch_bounds__(kPendThreads, 1024 / kPendThreads) k_pod_stale(StaleArgs a, uint32_t n_units) {
    StaleUnits p{a};
    compact_units(p, n_units, a.tile_state, a.ticket);
}

// The change window of k_pod_stale_reach, staged once per CTA: entry e is offer idx[e], changed at generation gen[e]
// (newest first), with its columns in the current table
struct WindowStage {
    uint32_t idx[RPK_OFFERS_DELTA_MAX], gen[RPK_OFFERS_DELTA_MAX];
    int32_t mem[RPK_OFFERS_DELTA_MAX], vcpu[RPK_OFFERS_DELTA_MAX], ram[RPK_OFFERS_DELTA_MAX];
    double sp[RPK_OFFERS_DELTA_MAX], cp[RPK_OFFERS_DELTA_MAX];
    uint8_t flags[RPK_OFFERS_DELTA_MAX];
};

// k_pod_stale_reach's units: k_pod_stale's, after a pre-pass over the CTA's share (prepare) that marks current every
// pending slot whose stored result is older than the current generation, not below the floor, made from the table
// row's columns, and reached by no window entry newer than it (rpk.h, rpk_select_pending_changed): its list is the
// row's list under the current table.  Pass 1 then keeps exactly the slots k_pod_stale keeps, and later calls skip the
// marked slots.  The pre-pass runs before pass 1's four loads are in flight, so the two never share registers; a thread
// marks the units it loads in pass 1 (u - c_lo the same modulo kPendThreads), so no barrier stands between them.
struct StaleReachUnits : StaleUnits {
    const StaleReachArgs& x;
    const WindowStage& w;
    // some window entry newer than generation rg reaches the row of global slot s, whose stored list sits at owned index j
    __device__ __forceinline__ bool reached(uint32_t s, uint32_t j, uint32_t rg) const {
        uint32_t n = 0;  // the entries newer than rg: a prefix of the window
        while (n < x.n_win && w.gen[n] > rg) ++n;
        const int32_t* l = a.r.top5 + (size_t)j * RPK_TOPK;
        for (int q = 0; q < RPK_TOPK; ++q) {  // rule 1: an entry of the list changed
            const int32_t lq = l[q];
            for (uint32_t e = 0; e < n; ++e)
                if ((int32_t)w.idx[e] == lq) return true;
        }
        const uint8_t cloud = a.t.cloud[s];
        if (cloud > RPK_CLOUD_COMMUNITY) return false;  // nothing is feasible
        const int32_t mem = a.t.mem[s], vcpu = a.t.vcpu[s], ram = a.t.ram[s], l4 = l[4];
        const double mx = a.t.max_price[s];
        const double* price = cloud ? w.cp : w.sp;
        const double p4 = l4 >= 0 ? (cloud ? x.cp : x.sp)[l4] : 0.0;  // L[4] did not change: its price is the one it was listed at
        const uint8_t bit = cloud ? (uint8_t)RPK_FLAG_COMMUNITY_CLOUD : (uint8_t)RPK_FLAG_SECURE_CLOUD;
        for (uint32_t e = 0; e < n; ++e) {  // rule 2: a changed offer is feasible, and L is short or it comes before L[4]
            const double p = price[e];
            const int32_t c = (int32_t)w.idx[e];
            if ((w.flags[e] & bit) && p > 0.0 && p < mx && w.mem[e] >= mem && w.vcpu[e] >= vcpu && w.ram[e] >= ram &&
                (l4 < 0 || p < p4 || (p == p4 && c < l4)))
                return true;
        }
        return false;
    }
    __device__ __forceinline__ void prepare(uint32_t c_lo, uint32_t c_hi) const {
        for (uint32_t u = c_lo + threadIdx.x; u < c_hi; u += kPendThreads) {
            const uint32_t g = a.u_lo + u, j = u * kPendUnit, s = g * kPendUnit;
            const uint32_t pm = nonzero_bytes16(load_flags(a.flags, g, a.N));
            if (!pm) continue;
            uint32_t test = 0;  // pending, older than the current generation, not below the floor
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const uint4 v = reinterpret_cast<const uint4*>(a.r.gen + j)[q];
                test |= ((uint32_t)(v.x != a.gen && v.x >= x.floor) | (uint32_t)(v.y != a.gen && v.y >= x.floor) << 1 |
                         (uint32_t)(v.z != a.gen && v.z >= x.floor) << 2 | (uint32_t)(v.w != a.gen && v.w >= x.floor) << 3) << (4 * q);
            }
            for (test &= pm; test; test &= test - 1) {
                const uint32_t k = (uint32_t)__ffs(test) - 1;
                if (a.t.mem[s + k] != a.r.mem[j + k] || a.t.vcpu[s + k] != a.r.vcpu[j + k] || a.t.ram[s + k] != a.r.ram[j + k] ||
                    __double_as_longlong(a.t.max_price[s + k]) != __double_as_longlong(a.r.max_price[j + k]) ||
                    a.t.cloud[s + k] != a.r.cloud[j + k] || reached(s + k, j + k, a.r.gen[j + k]))
                    continue;
                a.r.gen[j + k] = a.gen;
            }
        }
    }
};

__global__ void __launch_bounds__(kPendThreads, 1024 / kPendThreads) k_pod_stale_reach(StaleReachArgs x, uint32_t n_units) {
    __shared__ WindowStage w;
    for (uint32_t e = threadIdx.x; e < x.n_win; e += kPendThreads) {
        const uint2 en = x.win[e];
        w.idx[e] = en.x; w.gen[e] = en.y;
        w.mem[e] = x.mem[en.x]; w.vcpu[e] = x.vcpu[en.x]; w.ram[e] = x.ram[en.x];
        w.sp[e] = x.sp[en.x]; w.cp[e] = x.cp[en.x]; w.flags[e] = x.flags[en.x];
    }
    __syncthreads();
    StaleReachUnits p{{x.s}, x, w};
    compact_units(p, n_units, x.s.tile_state, x.s.ticket);
}

// k_pod_result_diff_xchg's units: 16 reselected rows of the n the stale step listed.  Pass 1 compares each row's new
// list with the stored one (a slot never reported has none, and differs), stores the row's result -- its list, the
// columns the reselect took it from and the offer-table generation -- and leaves the changed bits in mask[u]; pass 2
// writes each changed row into every output region (peer stores over NVLink for an exchange buffer) and the last CTA in
// unit order writes the count into every count word.  The stores are made visible system-wide before a CTA counts as
// finished, so the CTA that finishes last can signal the results epoch: a peer past its wait reads every region.
struct DiffXchgUnits {
    struct V { uint32_t keep; };
    using Count = uint32_t;
    const ResultDiffArgs& a;
    const ResultXchgArgs& x;
    uint32_t n;
    __device__ __forceinline__ V none() const { return V{0u}; }
    __device__ __forceinline__ V load(uint32_t u) const {
        uint32_t keep = 0;
        for (uint32_t k = 0; k < kPendUnit; ++k) {
            const uint32_t i = u * kPendUnit + k;
            if (i >= n) break;
            const uint32_t j = a.list[i] - a.r_lo;
            const int32_t* nt = a.top5 + (size_t)i * RPK_TOPK;
            int32_t* ot = a.r.top5 + (size_t)j * RPK_TOPK;
            bool ch = a.r.gen[j] == 0u;
#pragma unroll
            for (int q = 0; q < RPK_TOPK; ++q) { const int32_t x = nt[q]; ch |= ot[q] != x; ot[q] = x; }
            a.r.mem[j] = a.cols.mem[i]; a.r.vcpu[j] = a.cols.vcpu[i]; a.r.ram[j] = a.cols.ram[i];
            a.r.max_price[j] = a.cols.max_price[i]; a.r.cloud[j] = a.cols.cloud[i]; a.r.gen[j] = a.gen;
            keep |= (uint32_t)ch << k;
        }
        a.mask[u] = (uint16_t)keep;
        return V{keep};
    }
    __device__ __forceinline__ V reload(uint32_t u) const { return V{a.mask[u]}; }
    __device__ __forceinline__ Count count1(const V& v) const { return (uint32_t)__popc(v.keep); }
    __device__ __forceinline__ uint32_t count(const V& v) const { return (uint32_t)__popc(v.keep); }
    __device__ __forceinline__ bool keep(const V& v, uint32_t k) const { return (v.keep >> k) & 1u; }
    __device__ __forceinline__ uint32_t id(uint32_t u, uint32_t k) const { return u * kPendUnit + k; }
    __device__ __forceinline__ void emit(uint32_t i, uint32_t row) const {  // best is the list's first entry
        const int32_t* t = a.top5 + (size_t)row * RPK_TOPK;
        const uint32_t s = a.list[row];
        int32_t v[RPK_TOPK];
#pragma unroll
        for (int q = 0; q < RPK_TOPK; ++q) v[q] = t[q];
        for (int o = 0; o < x.n_out; ++o) {
            uint32_t* r = x.region[o];
            r[i] = s; r[x.cap + i] = (uint32_t)v[0];
            uint32_t* r5 = r + 2 * (size_t)x.cap + (size_t)i * RPK_TOPK;
#pragma unroll
            for (int q = 0; q < RPK_TOPK; ++q) r5[q] = (uint32_t)v[q];
        }
    }
    __device__ __forceinline__ void set_count(uint32_t n) const { for (int o = 0; o < x.n_out; ++o) *x.count[o] = n; }
    __device__ __forceinline__ void cta_total(Count) const {}
    __device__ __forceinline__ void fence() const { __threadfence_system(); }
    __device__ __forceinline__ void last() const {}
    __device__ __forceinline__ void last_warp() const {
        if (x.peers.n > 0) signal_peers(x.peers, kFlagResults, kFlagResultsCtr, 0, x.peers.inline_wait != 0);
    }
    __device__ __forceinline__ void prepare(uint32_t, uint32_t) const {}
};

// The row count is *d_n, read here, and the grid was sized for the worst case: the units of the count are shared out
// over the whole grid, so a CTA past them publishes a zero count at once and the look-back, the count stores and the
// last CTA's signal complete as for a launch sized for the count
__global__ void __launch_bounds__(kPendThreads, 1024 / kPendThreads) k_pod_result_diff_xchg(ResultXchgArgs x, const uint32_t* __restrict__ d_n) {
    const uint32_t n = *d_n;
    DiffXchgUnits p{x.d, x, n};
    compact_units(p, (n + kPendUnit - 1) / kPendUnit, x.d.tile_state, x.d.ticket);
}

int launch_pod_fill(const PodRows& t, uint8_t* pending, uint32_t N, int sm_count, cudaStream_t st) {
    if (N == 0) return 0;
    const uint32_t blocks = std::min<uint32_t>((N + kPodThreads - 1) / kPodThreads, (uint32_t)sm_count * 8);
    k_pod_fill<<<blocks, kPodThreads, 0, st>>>(t, pending, N);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

int launch_pod_seed(const PodRows& t, uint32_t N, uint32_t n, const uint32_t* d_slots, const PodCols& in, cudaStream_t st) {
    if (n == 0) return 0;
    k_pod_seed<<<(n + kPodThreads - 1) / kPodThreads, kPodThreads, 0, st>>>(t, N, n, d_slots, in);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

int launch_pod_gather(const PodRows& t, uint32_t N, uint32_t n, const uint32_t* d_slots, const PodRows& out, cudaStream_t st) {
    if (n == 0) return 0;
    k_pod_gather<<<(n + kPodThreads - 1) / kPodThreads, kPodThreads, 0, st>>>(t, N, n, d_slots, out);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

int launch_pod_mark(uint8_t* flags, uint32_t N, uint32_t n, const uint32_t* d_slots, const uint8_t* d_pending, cudaStream_t st) {
    if (n == 0) return 0;
    k_pod_mark<<<(n + kPodThreads - 1) / kPodThreads, kPodThreads, 0, st>>>(flags, N, n, d_slots, d_pending);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

// u64 entries of PendingArgs::tile_state: one per CTA, and launch_pod_pending never launches more CTAs than SMs
uint32_t pending_state_words(int sm_count) { return (uint32_t)sm_count + 8; }

// one tile per CTA until every SM has its CTA (at most one per SM: the launch fits beside a running select), then
// longer shares
static uint32_t compact_grid(uint32_t n_units, int sm_count) {
    return std::min<uint32_t>((n_units + kPendThreads - 1) / kPendThreads, (uint32_t)sm_count);
}

int launch_pod_pending(const PendingArgs& a, int sm_count, cudaStream_t st) {
    if (a.N == 0) {
        RPK_CUDA(cudaMemsetAsync(a.n_out, 0, sizeof(uint32_t), st));
        return 0;
    }
    const uint32_t n_units = (a.N + kPendUnit - 1) / kPendUnit;
    k_pod_pending<<<compact_grid(n_units, sm_count), kPendThreads, 0, st>>>(a, n_units);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

int launch_pod_stale(const StaleArgs& a, uint32_t n_units, int sm_count, cudaStream_t st) {
    if (n_units == 0) return 0;
    k_pod_stale<<<compact_grid(n_units, sm_count), kPendThreads, 0, st>>>(a, n_units);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

int launch_pod_stale_reach(const StaleReachArgs& a, uint32_t n_units, int sm_count, cudaStream_t st) {
    if (n_units == 0) return 0;
    k_pod_stale_reach<<<compact_grid(n_units, sm_count), kPendThreads, 0, st>>>(a, n_units);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

int launch_pod_result_xchg(const ResultXchgArgs& x, const uint32_t* d_n, uint32_t n_max, int sm_count, cudaStream_t st) {
    const uint32_t n_units = (n_max + kPendUnit - 1) / kPendUnit;  // no rows: one CTA publishes the count and signals
    k_pod_result_diff_xchg<<<std::max<uint32_t>(compact_grid(n_units, sm_count), 1u), kPendThreads, 0, st>>>(x, d_n);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace rpk
