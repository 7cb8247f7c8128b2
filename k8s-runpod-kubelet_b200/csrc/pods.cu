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

__global__ void __launch_bounds__(kPendThreads, 1024 / kPendThreads) k_pod_pending(PendingArgs a, uint32_t n_units) {
    constexpr uint32_t kWarps = kPendThreads / 32;
    __shared__ uint32_t s_ids[kPendTile];
    __shared__ uint32_t s_warp[kWarps];
    __shared__ uint32_t s_id, s_excl, s_last;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_id = atomicAdd(a.ticket, 1u);
    __syncthreads();
    const uint32_t cid = s_id, n_ctas = gridDim.x;
    const uint32_t c_lo = (uint32_t)((unsigned long long)n_units * cid / n_ctas), c_hi = (uint32_t)((unsigned long long)n_units * (cid + 1) / n_ctas);
    // ---- pass 1: the CTA's count -> its offset among the CTAs ----
    uint32_t mine = 0;
    for (uint32_t u0 = c_lo + tid; u0 < c_hi; u0 += 4 * kPendThreads) {
        uint4 v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t u = u0 + (uint32_t)k * kPendThreads;
            v[k] = u < c_hi ? load_flags(a.flags, u, a.N) : make_uint4(0u, 0u, 0u, 0u);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) mine += count_flags(v[k]);
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) mine += __shfl_xor_sync(0xFFFFFFFFu, mine, d);
    if (lane == 0) s_warp[warp] = mine;
    __syncthreads();
    if (warp == 0) {
        uint32_t total = lane < kWarps ? s_warp[lane] : 0u;
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) total += __shfl_xor_sync(0xFFFFFFFFu, total, d);
        const uint32_t excl = sum_before(a.tile_state, cid, total, lane);
        if (lane == 0) {
            s_excl = excl;
            if (cid == n_ctas - 1) *a.n_out = excl + total;  // the last CTA in slot order owns the count
        }
    }
    __syncthreads();
    // ---- pass 2: one tile per round, thread t the t-th unit of the tile ----
    uint32_t at = s_excl;
    for (uint32_t r0 = c_lo; r0 < c_hi; r0 += kPendThreads) {
        const uint32_t u = r0 + tid;
        const uint4 v = u < c_hi ? load_flags(a.flags, u, a.N) : make_uint4(0u, 0u, 0u, 0u);
        const uint32_t c = count_flags(v);
        uint32_t inc = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t n = __shfl_up_sync(0xFFFFFFFFu, inc, d); if ((int)lane >= d) inc += n; }
        if (lane == 31) s_warp[warp] = inc;
        __syncthreads();
        uint32_t wbase = 0, round = 0;
#pragma unroll
        for (uint32_t w = 0; w < kWarps; ++w) { const uint32_t x = s_warp[w]; if (w < warp) wbase += x; round += x; }
        uint32_t off = wbase + inc - c;
        const uint32_t word[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (uint32_t k = 0; k < kPendUnit; ++k)
            if ((word[k >> 2] >> ((k & 3u) * 8u)) & 0xFFu) s_ids[off++] = u * kPendUnit + k;
        __syncthreads();
        for (uint32_t i = tid; i < round; i += kPendThreads) a.out[at + i] = s_ids[i];
        at += round;
        __syncthreads();  // the tile and the warp sums are rewritten by the next round
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = atomicAdd(a.ticket + 1, 1u) == n_ctas - 1 ? 1u : 0u;
    __syncthreads();
    if (!s_last) return;
    // last CTA to finish: every look-back is over -- clean the state for the next call
    for (uint32_t i = tid; i < n_ctas; i += kPendThreads) a.tile_state[i] = 0ull;
    if (tid == 0) { a.ticket[0] = 0u; a.ticket[1] = 0u; }
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

int launch_pod_pending(const PendingArgs& a, int sm_count, cudaStream_t st) {
    if (a.N == 0) {
        RPK_CUDA(cudaMemsetAsync(a.n_out, 0, sizeof(uint32_t), st));
        return 0;
    }
    const uint32_t n_units = (a.N + kPendUnit - 1) / kPendUnit;
    // one tile per CTA until every SM has its CTA (at most one per SM: the launch fits beside a running select), then
    // longer shares
    const uint32_t grid = std::min<uint32_t>((n_units + kPendThreads - 1) / kPendThreads, (uint32_t)sm_count);
    k_pod_pending<<<grid, kPendThreads, 0, st>>>(a, n_units);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace rpk
