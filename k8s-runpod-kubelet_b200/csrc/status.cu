// status.cu -- batched pod-status diff: the predicate of Provider.updateAllPodStatuses
// (reference kubelet.go:857-880) over N tracked slots in one pass, plus what the reference does next for the
// slots that changed (translateRunPodStatus, kubelet.go:1848-2024) as a 16-bit code.
//
// One record = exactly the two fields the reference compares (InstanceInfo.Status, .PortsExposed:
// runpod_client.go:103,108) in a fixed slot
//     [b0][status ASCII][0x00][ports][zero pad],   b0 = len | flag << 7,   len = strlen(status) + 2
// The previous state lives on the device as one 64-bit XXH64 per slot; "status changed || ports changed"
// (kubelet.go:870-873) becomes hash != previous hash.  The hash covers the slot's zero-padded prefix in whole
// 8-byte lanes -- bytes [0, 8 * ceil((1 + len) / 8)) with the flag bit cleared -- so it is self-delimiting (the
// length byte is inside), independent of the table's stride, and needs none of XXH64's byte-wise tail steps.
// The flag bit (host: "statusMessage contains error/fail", kubelet.go:1907-1908) is NOT a compared field and is
// not hashed; it only selects the EXITED branch of the code.
//
// Kernels:
//   k_status_stream<STRIDE, THREADS>
//                            every stride: HBM-bound scan.  Persistent CTAs; every WARP owns a contiguous run of
//                            slots and streams it with 16-byte global loads, the next unit's loads in flight while
//                            the current one is hashed; changed slots are staged in slot order in the warp's own
//                            part of a staging array -- no CTA barrier in the loop.  At the end each CTA publishes
//                            its count, finds its offset by decoupled look-back over the CTAs before it (ids are
//                            handed out in scheduling order) and copies its staged indices / codes to their final,
//                            ascending position (and, for the sharded sweep, into every peer's exchange buffer).
//                            STRIDE 16 and 32 are compiled for their stride; STRIDE 0 is the wide form (48..256),
//                            which takes the stride from the arguments.
//   k_status_seed_slots      previous state of individual slots (CreatePod writes ONE InstanceInfo, kubelet.go:391-401).
// The first also sweeps a list of slots (template flag SLOTS, rpk_status_diff_slots): the listed slots' packed
// records are a table of their own, streamed the same way; only the hash row (slots[i] - idx_base) and the id
// reported (slots[i]) differ.  updateAllPodStatuses compares only the pods it fetched this cycle (kubelet.go:836-864).
// A sharded list sweep exchanges its changed list with its peers exactly as a whole-table one does
// (rpk_status_diff_slots_device_gather).
#include "rpk_device.cuh"
#include "rpk_internal.cuh"

namespace rpk {
using namespace dev;

using u64 = unsigned long long;

constexpr u64 P1 = 0x9E3779B185EBCA87ull, P2 = 0xC2B2AE3D27D4EB4Full, P3 = 0x165667B19E3779F9ull,
              P4 = 0x85EBCA77C2B2AE63ull, P5 = 0x27D4EB2F165667C5ull;

__device__ __forceinline__ u64 rotl64(u64 x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ u64 xround(u64 acc, u64 in) { return rotl64(acc + in * P2, 31) * P1; }
__device__ __forceinline__ u64 xmerge(u64 h, u64 v) { return (h ^ xround(0, v)) * P1 + P4; }
__device__ __forceinline__ u64 step8(u64 h, u64 lane) { h ^= xround(0, lane); return rotl64(h, 27) * P1 + P4; }
__device__ __forceinline__ u64 avalanche(u64 h) { h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32; return h; }
__device__ __forceinline__ u64 mk64(uint32_t lo, uint32_t hi) { return (u64)lo | ((u64)hi << 32); }

// XXH64, seed 0, over nl 8-byte lanes (public xxHash spec; what github.com/cespare/xxhash/v2 Sum64 computes,
// go.mod:60).  nl <= 3 is the short path (no stripes); nl == 4 is exactly one 32-byte stripe.
__device__ __noinline__ u64 xxh64_stripe32(u64 l0, u64 l1, u64 l2, u64 l3) {  // exactly one 32-byte stripe (nl == 4)
    const u64 v1 = xround(P1 + P2, l0), v2 = xround(P2, l1), v3 = xround(0, l2), v4 = xround(0ull - P1, l3);
    u64 h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
    h = xmerge(h, v1); h = xmerge(h, v2); h = xmerge(h, v3); h = xmerge(h, v4);
    return avalanche(h + 32ull);
}
__device__ __noinline__ u64 xxh64_words(const uint32_t* w, uint32_t nbytes, uint32_t w0);
// WIDE (strides 48..256): a record of nl > 4 lanes goes on past the 32 bytes in l0..l3, so every record of 4 or more
// lanes is hashed in one out-of-line call over `rec`, the record in global memory
template <bool WIDE = false>
__device__ __forceinline__ u64 xxh64_lanes4(u64 l0, u64 l1, u64 l2, u64 l3, uint32_t nl, const uint32_t* rec = nullptr) {
    u64 h = P5 + (u64)(nl * 8u);
    h = step8(h, l0);
    const u64 h2 = step8(h, l1);
    h = nl >= 2 ? h2 : h;
    // no RunPod status needs a third lane (15+ characters) or the stripe form (23+): warp-uniformly skipped in practice,
    // and kept out of line so that the hot path does not carry their registers
    if (__any_sync(0xFFFFFFFFu, nl >= 3)) {
        if (nl == 3) h = step8(h, l2);
        if (__any_sync(0xFFFFFFFFu, nl >= 4)) {
            if constexpr (WIDE) {
                if (nl >= 4) return xxh64_words(rec, nl * 8u, (uint32_t)l0);
            } else {
                const u64 hs = xxh64_stripe32(l0, l1, l2, l3);
                if (nl >= 4) return hs;
            }
        }
    }
    return avalanche(h);
}
__device__ __forceinline__ u64 xxh64_lanes2(u64 l0, u64 l1, uint32_t nl) {  // 16-byte slots: one or two lanes
    u64 h = P5 + (u64)(nl * 8u);
    h = step8(h, l0);
    const u64 h2 = step8(h, l1);
    return avalanche(nl >= 2 ? h2 : h);
}

// General form over 32-bit words in memory, nbytes a multiple of 8 (records of 4+ lanes at wide strides, per-slot seed).
// Out of line, like the stripe: the wide sweep calls it for rare long records and must not carry its registers.
__device__ __noinline__ u64 xxh64_words(const uint32_t* w, uint32_t nbytes, uint32_t w0) {  // w0: word 0 with the flag bit cleared
    uint32_t off = 0;  // in words
    u64 h;
    auto rd = [&](uint32_t q) { return mk64(q == 0 ? w0 : w[q], w[q + 1]); };
    if (nbytes >= 32) {
        u64 v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0ull - P1;
        do {
            v1 = xround(v1, rd(off)); v2 = xround(v2, rd(off + 2)); v3 = xround(v3, rd(off + 4)); v4 = xround(v4, rd(off + 6));
            off += 8;
        } while ((off + 8) * 4 <= nbytes);
        h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
        h = xmerge(h, v1); h = xmerge(h, v2); h = xmerge(h, v3); h = xmerge(h, v4);
    } else {
        h = P5;
    }
    h += (u64)nbytes;
    while ((off + 2) * 4 <= nbytes) { h = step8(h, rd(off)); off += 2; }
    return avalanche(h);
}

// ---- what translateRunPodStatus decides, as a code (kubelet.go:1866-1975) ---------------------------------
// kind: 0 RUNNING 1 STARTING 2 EXITED 3 TERMINATING 4 TERMINATED 5 NOT_FOUND 6 anything else (default:, :1967)
// bits: [2:0] phase  [3] ready  [4] started  [6:5] state  [7] exit code  [10:8] reason  [12:11] message kind (rpk.h)
__device__ __forceinline__ uint32_t status_code(uint32_t kind, bool ports, bool msg_err) {
    switch (kind) {
        case 0: return ports ? 0x003Au : 0x0901u;    // :1867-1891  Running+ready | Pending, ContainerCreating, "ports not yet exposed"
        case 1: return 0x0101u;                      // :1893-1903  Pending, ContainerCreating, statusMessage
        case 2: return msg_err ? 0x03C4u : 0x0243u;  // :1905-1929  Failed, Error, exit 1 | Succeeded, Completed
        case 3: return 0x003Au;                      // :1931-1941  Running+ready
        case 4: return 0x0443u;                      // :1943-1955  Succeeded, Terminated
        case 5: return 0x15C4u;                      // :1957-1969  Failed, PodDeleted, exit 1, "Pod was deleted from RunPod API"
        default: return 0x1E00u;                     // :1971-1979  Unknown, ContainerStatusUnknown, "Unknown RunPod status: %s"
    }
}
// (status, ports) from the first two lanes of a slot.  Every known status has its own length (8..13), so the length
// picks the one candidate and two masked 64-bit compares decide; the ports byte sits at byte `len`.
__device__ __forceinline__ uint32_t classify_status(u64 l0, u64 l1, uint32_t len, bool* ports) {
    // lane images of "<len>RUNNING\0", ... with the ports byte (and everything after it) cleared
    constexpr u64 kL0[6] = {0x474E494E4E555209ull /* \x09RUNNING */, 0x4E4954524154530Aull /* \x0aSTARTIN */, 0x0044455449584508ull /* \x08EXITED\0 */,
                            0x414E494D5245540Dull /* \x0dTERMINA */, 0x414E494D5245540Cull /* \x0cTERMINA */, 0x554F465F544F4E0Bull /* \x0bNOT_FOU */};
    constexpr u64 kL1[6] = {0x0ull, 0x47ull /* G */, 0x0ull, 0x474E4954ull /* TING */, 0x444554ull /* TED */, 0x444Eull /* ND */};
    constexpr int kLen[6] = {9, 10, 8, 13, 12, 11};
    *ports = false;
    if (len < 8 || len > 13) return 6u;
    const uint32_t sh = (len - 8u) * 8u;  // the ports byte is byte (len - 8) of lane 1
    *ports = ((l1 >> sh) & 0xFFull) != 0ull;
    const u64 l1m = l1 & ((1ull << sh) - 1ull);
    uint32_t kind = 6u;
#pragma unroll
    for (int k = 0; k < 6; ++k)
        if ((int)len == kLen[k] && l0 == kL0[k] && l1m == kL1[k]) kind = (uint32_t)k;
    return kind;
}

#define kFlagAgg (1ull << 32)
#define kFlagMask (3ull << 32)

// Decoupled look-back over the CTAs before `id` (one warp): returns the exclusive prefix.  There is at most one CTA
// per SM, and they all finish at about the same time, so walking back window by window would cost one L2 round trip
// per 32 predecessors.  Every CTA publishes its count once (kFlagAgg | count; an entry without a flag bit is not there
// yet) and sums ALL entries before it in one pass of independent loads, retrying only the ones that are not there yet.
__device__ __forceinline__ uint32_t sum_before(volatile u64* st, uint32_t id, uint32_t total, uint32_t lane) {
    if (lane == 0) st[id] = kFlagAgg | total;
    uint32_t acc = 0;
    for (uint32_t base = 0; base < id; base += 128) {  // four independent loads per lane and pass
        u64 v[4];
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

// ---------------------------------------------------------------------------------------------------------
// streamed scan
// ---------------------------------------------------------------------------------------------------------
// One 1024-thread CTA per SM owns a contiguous range of units (64 slots each); its 32 warps take the units of the range
// round-robin, so the CTA reads ONE sequential stream, 32 units (64 KB of 32-byte slots + 16 KB of hashes) per round --
// DRAM sees one long sequential stream per SM instead of thousands of short ones.  A warp keeps the next unit's loads in
// flight while it hashes the current one.  Changed slots are staged at the unit's own position of the staging arrays
// (unit * 64 + rank) with the unit's count beside them, so warps never wait for each other; at the end the CTA sums
// its counts, finds its offset by decoupled look-back over the CTAs before it (ids are handed out in scheduling
// order) and copies its staged indices / codes to their final, ascending position (and, for the sharded sweep, into
// every peer's exchange buffer).
constexpr int kStreamItems = 2;                          // slots per lane per unit
constexpr uint32_t kUnit = 32 * kStreamItems;            // slots per warp per unit
// Two launch shapes of the same kernel.  1024-thread CTAs, one per SM: the CTA's 32 warps read one long sequential
// stream -- the shape for a sweep that has the GPU to itself over a large table (HBM-bound regime).  256-thread CTAs,
// at most one per SM: 16K registers, exactly what the 96-register persistent select kernel leaves free, so the sweep of
// a tick runs next to the selection instead of in front of it; used for tables below kBigTable slots (latency regime).
// A second or third sweep CTA on an SM would keep the select's CTA off that SM until they leave; alone on the GPU, one
// CTA per SM is also faster at 1M slots than four (fewer look-back entries and copy rounds).
constexpr uint32_t kBigTable = 4u << 20;
// control words (StatusArgs::tile_counter): [0] scheduling ticket, [1] finished CTAs
// col (SLOTS only): the entry's row of hash_prev, kNone when the slot lies outside the column
template <int STRIDE> struct SlotData { uint4 lo; uint4 hi; u64 prev; uint32_t col; };

// Bytes per record: STRIDE, or the call's stride in the wide form (STRIDE 0, strides 48..256).  The wide form loads
// the first 32 bytes of a slot as stride 32 does: the status code reads two lanes, and a hash over more than four
// lanes goes back to the record (xxh64_lanes4<true>).
template <int STRIDE> __device__ __forceinline__ uint32_t rec_stride(const StatusArgs& a) { return STRIDE ? (uint32_t)STRIDE : a.stride; }

template <int STRIDE, bool SLOTS>
__device__ __forceinline__ void load_unit(const StatusArgs& a, uint32_t base, uint32_t lane, SlotData<STRIDE> (&d)[kStreamItems]) {
#pragma unroll
    for (int k = 0; k < kStreamItems; ++k) {
        const uint32_t s = base + (uint32_t)k * 32 + lane;
        d[k].lo = make_uint4(0, 0, 0, 0); d[k].hi = d[k].lo; d[k].prev = 0;
        if constexpr (SLOTS) d[k].col = kNone;
        if (s < a.N) {
            const uint4* p = reinterpret_cast<const uint4*>(a.records + (size_t)s * rec_stride<STRIDE>(a));
            d[k].lo = __ldg(p);  // the two halves of a 32-byte slot share a sector: the second load hits L1
            if (STRIDE != 16) d[k].hi = __ldg(p + 1);
            if constexpr (SLOTS) {
                const uint32_t c = __ldg(a.slots + s) - a.idx_base;  // below idx_base wraps around: outside
                if (c < a.col_n) { d[k].col = c; d[k].prev = a.hash_prev[c]; }
            } else {
                d[k].prev = a.hash_prev[s];
            }
        }
    }
}

// SLOTS: the table is a packed slot list (StatusArgs::slots).  The exchange (n_out, flags) is the same for both forms:
// what it publishes is the list of global slot ids the final copy computes
template <int STRIDE, int THREADS, bool SLOTS = false>
__global__ void __launch_bounds__(THREADS, 1024 / THREADS) k_status_stream(StatusArgs a, uint32_t n_units) {
    constexpr int kSThreads = THREADS, kSWarps = THREADS / 32;
    __shared__ uint32_t s_warp[kSWarps];
    __shared__ uint32_t s_id, s_excl, s_last, s_carry;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    pdl_trigger();
    const bool report = a.stage_idx != nullptr;
    // reporting sweeps take their id from a ticket (scheduling order: the look-back below cannot starve); a seed has no
    // look-back and must not touch the ticket (nobody would reset it)
    if (tid == 0) s_id = report ? atomicAdd(a.tile_counter, 1u) : blockIdx.x;
    __syncthreads();
    const uint32_t cid = s_id, n_ctas = gridDim.x;
    const uint32_t c_lo = (uint32_t)((u64)n_units * cid / n_ctas), c_hi = (uint32_t)((u64)n_units * (cid + 1) / n_ctas);
    // one unit: hash, compare, stage the changed slots at the unit's own position, publish the unit's count
    auto process = [&](uint32_t u, SlotData<STRIDE> (&d)[kStreamItems]) {
        uint32_t running = 0;
#pragma unroll
        for (int k = 0; k < kStreamItems; ++k) {
            const uint32_t s = u * kUnit + (uint32_t)k * 32 + lane;
            const uint32_t len = min(d[k].lo.x & 0x7Fu, rec_stride<STRIDE>(a) - 1u);
            const uint32_t nl = (len + 8u) >> 3;  // lanes covering bytes [0, 1 + len)
            const u64 l0 = mk64(d[k].lo.x & ~0x80u, d[k].lo.y), l1 = mk64(d[k].lo.z, d[k].lo.w);
            const u64 l2 = mk64(d[k].hi.x, d[k].hi.y), l3 = mk64(d[k].hi.z, d[k].hi.w);
            u64 h;
            if (STRIDE == 16) h = xxh64_lanes2(l0, l1, nl);
            else if (STRIDE == 32) h = xxh64_lanes4(l0, l1, l2, l3, nl);
            else h = xxh64_lanes4<true>(l0, l1, l2, l3, nl, reinterpret_cast<const uint32_t*>(a.records + (size_t)s * a.stride));
            bool changed = false;
            if constexpr (SLOTS) {
                if (s < a.N && d[k].col != kNone) {
                    changed = (d[k].prev == 0ull) || (h != d[k].prev);
                    if (changed) a.hash_prev[d[k].col] = h;
                }
            } else if (s < a.N) {
                changed = (d[k].prev == 0ull) || (h != d[k].prev);  // 0 = never seen
                if (changed) a.hash_prev[s] = h;                     // kubelet.go:875-880
                if (a.hash_out) a.hash_out[s] = h;
            }
            if (report) {
                const uint32_t bal = __ballot_sync(0xFFFFFFFFu, changed);
                if (changed) a.stage_idx[u * kUnit + running + (uint32_t)__popc(bal & ((1u << lane) - 1u))] = s;
                running += (uint32_t)__popc(bal);
            }
        }
        if (report && lane == 0) a.unit_cnt[u] = running;
    };
    // two register sets, used alternately: the next unit's loads are in flight while the current one is hashed
    SlotData<STRIDE> ra[kStreamItems], rb[kStreamItems];
    uint32_t u = c_lo + warp;
    if (u < c_hi) load_unit<STRIDE, SLOTS>(a, u * kUnit, lane, ra);
    while (u < c_hi) {
        if (u + kSWarps < c_hi) load_unit<STRIDE, SLOTS>(a, (u + kSWarps) * kUnit, lane, rb);
        process(u, ra);
        u += kSWarps;
        if (u >= c_hi) break;
        if (u + kSWarps < c_hi) load_unit<STRIDE, SLOTS>(a, (u + kSWarps) * kUnit, lane, ra);
        process(u, rb);
        u += kSWarps;
    }
    if (!report) return;  // seed: state only
    // ---- CTA count -> offset among the CTAs (look-back) -> final, ascending position ----
    __syncthreads();  // every unit of the range has its count and its staged entries (same CTA: visible after the barrier)
    uint32_t mine = 0;
    for (uint32_t v = c_lo + tid; v < c_hi; v += kSThreads) mine += a.unit_cnt[v];
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) mine += __shfl_xor_sync(0xFFFFFFFFu, mine, d);
    if (lane == 0) s_warp[warp] = mine;
    __syncthreads();
    if (warp == 0) {
        uint32_t total = lane < (uint32_t)kSWarps ? s_warp[lane] : 0u;
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) total += __shfl_xor_sync(0xFFFFFFFFu, total, d);
        const uint32_t excl = sum_before(a.tile_state, cid, total, lane);
        if (lane == 0) {
            s_excl = excl; s_carry = 0;
            if (cid == n_ctas - 1) {  // the last CTA in slot order owns the count
                *a.n_changed = excl + total;
                for (int o = 0; o < a.n_out; ++o) a.out_count[o][a.peers.my_rank] = excl + total;
            }
        }
    }
    __syncthreads();
    const bool want_codes = a.changed_code != nullptr || (a.n_out > 0 && a.out_code[0] != nullptr);
    // exclusive scan of the unit counts in unit order, 1024 units per round; thread t copies unit t's staged entries
    for (uint32_t r0 = c_lo; r0 < c_hi; r0 += kSThreads) {
        const uint32_t v = r0 + tid;
        const uint32_t c = v < c_hi ? a.unit_cnt[v] : 0u;
        uint32_t inc = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t n = __shfl_up_sync(0xFFFFFFFFu, inc, d); if ((int)lane >= d) inc += n; }
        if (lane == 31) s_warp[warp] = inc;
        __syncthreads();
        uint32_t wbase = 0;
        for (uint32_t w = 0; w < warp; ++w) wbase += s_warp[w];
        const uint32_t off = s_excl + s_carry + wbase + inc - c;
        for (uint32_t i = 0; i < c; ++i) {
            const uint32_t slot = a.stage_idx[v * kUnit + i];
            const uint32_t x = SLOTS ? __ldg(a.slots + slot) : a.idx_base + slot;  // SLOTS: slot is the list position
            if (a.changed_idx) a.changed_idx[off + i] = x;
            for (int o = 0; o < a.n_out; ++o) a.out_idx[o][off + i] = x;
            if (want_codes) {  // translateRunPodStatus's decision, for the changed slots only: their records are read once more
                const uint4 r = __ldg(reinterpret_cast<const uint4*>(a.records + (size_t)slot * rec_stride<STRIDE>(a)));
                bool ports;
                const uint32_t len = min(r.x & 0x7Fu, rec_stride<STRIDE>(a) - 1u);
                const uint32_t kind = classify_status(mk64(r.x & ~0x80u, r.y), mk64(r.z, r.w), len, &ports);
                const uint16_t cc = (uint16_t)status_code(kind, ports, (r.x & 0x80u) != 0u);
                if (a.changed_code) a.changed_code[off + i] = cc;
                for (int o = 0; o < a.n_out; ++o) if (a.out_code[o]) a.out_code[o][off + i] = cc;
            }
        }
        __syncthreads();
        if (tid == kSThreads - 1) s_carry += wbase + inc;  // this round's total
        __syncthreads();
    }
    if (a.n_out > 0) __threadfence_system();  // peer stores are performed system-wide before this CTA counts as finished
    else __threadfence();
    __syncthreads();
    if (tid == 0) s_last = atomicAdd(a.tile_counter + 1, 1u) == n_ctas - 1 ? 1u : 0u;
    __syncthreads();
    if (!s_last) return;
    // last CTA to finish: every look-back is over -- clean the state for the next call, then tell the peers
    for (uint32_t i = tid; i < n_ctas; i += kSThreads) a.tile_state[i] = 0ull;
    if (tid == 0) { a.tile_counter[0] = 0u; a.tile_counter[1] = 0u; }
    if (a.peers.n > 0 && warp == 0) signal_peers(a.peers, kFlagStatus, kFlagStatusCtr, 0, a.peers.inline_wait != 0);
}

// previous state of individual slots: hash_prev[slots[i] - idx_base] = hash(records[i]) for the slots of this shard
__global__ void k_status_seed_slots(uint32_t n, const uint32_t* __restrict__ slots, const uint8_t* __restrict__ records, uint32_t stride,
                                    u64* __restrict__ hash_prev, uint32_t lo, uint32_t hi) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = slots[i];
    if (s < lo || s >= hi) return;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(records + (size_t)i * stride);
    const uint32_t len = min(w[0] & 0x7Fu, stride - 1);
    const uint32_t nbytes = min(((len + 8u) >> 3) << 3, stride);
    hash_prev[s - lo] = xxh64_words(w, nbytes, w[0] & ~0x80u);
}

int launch_status_seed_slots(uint32_t n, const uint32_t* d_slots, const uint8_t* d_records, uint32_t stride, uint64_t* hash_prev,
                             uint32_t lo, uint32_t hi, cudaStream_t st) {
    if (n == 0) return 0;
    k_status_seed_slots<<<(n + 127) / 128, 128, 0, st>>>(n, d_slots, d_records, stride, reinterpret_cast<u64*>(hash_prev), lo, hi);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

// u64 entries of StatusArgs::tile_state: one per CTA, and launch_status never launches more CTAs than SMs
uint32_t status_state_words(int sm_count) { return (uint32_t)sm_count + 8; }

// SLOTS: a slot-list sweep, whose launch shape follows from the list length (a.N) exactly as a table's does from N
template <bool SLOTS>
static int launch_status(const StatusArgs& a, int sm_count, cudaStream_t st) {
    if (a.N == 0) {
        if (a.n_changed) RPK_CUDA(cudaMemsetAsync(a.n_changed, 0, sizeof(uint32_t), st));
        // an empty shard of a sharded sweep still has to publish its (zero) count and signal: one tiny CTA does it
        if (a.n_out == 0 && a.peers.n == 0) return 0;
    }
    const uint32_t n_units = (a.N + kUnit - 1) / kUnit;
    const bool big = a.N >= kBigTable;
    const uint32_t warps = big ? 32u : 8u, max_grid = (uint32_t)sm_count;
    // one unit per warp until every SM has its CTA, then longer runs per warp
    uint32_t grid = (n_units + warps - 1) / warps;
    if (grid > max_grid) grid = max_grid;
    if (grid == 0) grid = 1;
    StatusArgs b = a;
    if (a.changed_idx == nullptr && a.n_out == 0) { b.stage_idx = nullptr; b.stage_code = nullptr; }
    // one loop, two launch shapes (see kBigTable).  Other loops -- three or four half-unit register sets, a per-warp
    // shared-memory ring filled by bulk copies -- were within 4 % of it at 16.8M slots on an H100 SXM (700 W) and
    // none was faster at both strides (DESIGN §4, profiles/h100_k2_tune.json)
    if (big) {
        if (a.stride == 16) k_status_stream<16, 1024, SLOTS><<<grid, 1024, 0, st>>>(b, n_units);
        else if (a.stride == 32) k_status_stream<32, 1024, SLOTS><<<grid, 1024, 0, st>>>(b, n_units);
        else k_status_stream<0, 1024, SLOTS><<<grid, 1024, 0, st>>>(b, n_units);
    } else {
        if (a.stride == 16) k_status_stream<16, 256, SLOTS><<<grid, 256, 0, st>>>(b, n_units);
        else if (a.stride == 32) k_status_stream<32, 256, SLOTS><<<grid, 256, 0, st>>>(b, n_units);
        else k_status_stream<0, 256, SLOTS><<<grid, 256, 0, st>>>(b, n_units);
    }
    RPK_CUDA(cudaGetLastError());
    return 1;
}

int launch_status_diff(const StatusArgs& a, int sm_count, cudaStream_t st) {
    return a.slots ? launch_status<true>(a, sm_count, st) : launch_status<false>(a, sm_count, st);
}

}  // namespace rpk
