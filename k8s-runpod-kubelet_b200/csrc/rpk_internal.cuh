// rpk_internal.cuh -- shared declarations of the rpk engine (not part of the C-ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <utility>
#include <vector>

#include "rpk.h"

namespace rpk {

constexpr uint32_t kNone = 0xFFFFFFFFu;      // "no feasible position"
constexpr uint32_t kGroups = 8;              // row groups: cloud view x (vcpu constrains) x (ram constrains)
constexpr int kWarpsPerCta = 8;              // select kernels: 256 threads
constexpr int kCtaThreads = kWarpsPerCta * 32;
constexpr uint32_t kChunk = 128;             // offers per warp-iteration (LDS.128 per lane)
constexpr uint32_t kSegPacked = 16384;       // packed words staged per CTA (64 KB); a power of two (see kPosBits)
constexpr uint32_t kPosBits = 14;            // log2(kSegPacked): position-in-segment bits of a "pos" packed word
constexpr uint32_t kSegWide = 4096;          // wide int4 views staged per CTA (64 KB)

// Layout of the packed offer word (sorted-by-price order, one u32 per offer), from bit `sh_ram` up:
//   [guard1][mem rank' : b1][guard2][vcpu rank : b2][guard3][ram rank : b3][position in segment : pos_bits]
// rank' = rank+1 (0 = offer not available in this cloud).  A pod's word holds its thresholds in the same
// fields with guards 0, so (offer - pod) keeps a field's guard iff offer_field >= pod_field.
// pos_bits = kPosBits when bits <= 32 - kPosBits: the low bits then carry the offer's position inside its
// 16384-offer segment and the kernel reduces key = (~d & guard) | (d & pos_mask) with a plain unsigned min
// (feasible keys are positions, infeasible ones are >= 2^pos_bits).  Otherwise pos_bits = 0 and the kernel
// tracks the position itself with predicated selects.
struct PackLayout {
    uint32_t guard;    // the three guard bits
    uint32_t sh_mem;   // shift of the mem field
    uint32_t sh_vcpu;  // shift of the vcpu field
    uint32_t sh_ram;   // shift of the ram field (= pos_bits)
    uint32_t pos_bits; // kPosBits or 0
    uint32_t bits;     // field + guard bits used (0 = table not packable -> generic kernel)
    // bit-sliced view (kernel kind 4): per 32-offer chunk, kBmStride words; word i < bm_words is the 32-bit
    // mask "offer j of the chunk passes threshold i" -- mem thresholds first (rank' >= t', t' = 1..D_mem+1, so
    // unavailable offers fail all of them), then vcpu thresholds 0..D_vcpu, then ram thresholds 0..D_ram.
    uint32_t bm_words; // D_mem+1 + D_vcpu+1 + D_ram+1 if that fits 64 words, else 0
    uint32_t bm_off_vcpu, bm_off_ram;
    uint32_t bm_stride; // words per chunk row: 32 (conflict-free) or 64 (up to 64 thresholds; words 32 apart share a bank)
    uint32_t no_fused;  // test hook (RPK_FORCE_KERNEL=bitmap_grouped): small batches also take the persistent kernel
    uint32_t slice_rows; // rows per sub-range of the per-mem-threshold view bitmapM (D_vcpu+1 + D_ram+1); 0 = not built
    uint32_t no_slice;   // test hook (RPK_FORCE_KERNEL=bitmap_price): the persistent kernel stages the table by price
};
constexpr uint32_t kBmMaxStride = 64;
constexpr uint32_t kBmSegBytes = 65536;      // bit-sliced rows staged per CTA: 512 chunks (stride 32) or 256 (stride 64)
constexpr uint32_t kFusedRowsMax = 16384;    // up to this many rows one fused launch beats the multi-kernel paths
constexpr uint32_t kSmallBatch = 4096;       // rows: the host entry point's single-copy latency path
// transposed bit-sliced view (persistent kernel): the chunk axis is cut into 64-chunk sub-ranges; sub-range s holds
// bm_words rows of kSubStride words -- word (threshold i, chunk 64 s + k) at bmT[(s * bm_words + i) * kSubStride + k].
// 68 = 64 + 4: consecutive threshold rows start 4 words (one 16-byte bank group) apart, so an LDS.128 whose lanes
// read up to 8 different threshold rows at the same chunk offset is conflict-free.
constexpr uint32_t kSubChunks = 64;
constexpr uint32_t kSubStride = 68;
constexpr uint32_t kMaxClasses = 4096;       // row classes (cloud x thresholds) the pod-side counting sort distinguishes
constexpr uint32_t kMaxGroups = 2 * kBmMaxStride;  // row groups of the persistent select: cloud, or (cloud, mem threshold)
// control words of the persistent select (Lane::hdr)
// (RowsDone is polled while the grid kernel runs and sits on a cache line of its own; Pushed counts CTAs in the push
// tail; the per-group row / work totals are written before the grid kernel starts; the queue cursors follow them)
enum : uint32_t { kHdrRowsDone = 32, kHdrPushed = 64, kHdrGroupRows = 96, kHdrGroupWork = kHdrGroupRows + kMaxGroups,
                  kHdrCursors = kHdrGroupWork + kMaxGroups };

// A peer group's flag arrays (rpk_peer_bind, rpk_peer_fence): flags[r] is rank r's array of >= 64 words; n = 0: none.
// Word layout (rpk.h): a rank's epochs as seen by rank r sit at word kFlagSelect + my_rank / kFlagStatus + my_rank /
// kFlagResults + my_rank of r's array; each rank counts its own epochs in kFlagSelectCtr / kFlagStatusCtr /
// kFlagResultsCtr of its own array.
struct PeerGroup {
    uint32_t* flags[RPK_MAX_GPUS];
    int n, my_rank;
    int inline_wait;  // the signalling warp also waits for every peer's signal (rpk_peer_inline_wait)
};
enum : uint32_t { kFlagSelect = 0, kFlagStatus = 8, kFlagResults = 16, kFlagSelectCtr = 32, kFlagStatusCtr = 33, kFlagResultsCtr = 34 };

// One warp signals the group: epoch 0 bumps the rank's own counter word `ctr` and uses the new value (the launch then
// carries no per-call value and can be replayed from a CUDA graph), any other epoch is used as given and leaves `ctr`
// alone.  After a system-scope fence (everything this grid and its stream did before, peer stores included, is visible
// first) lane r stores the epoch into word `word0 + my_rank` of rank r's array; with `wait` it then spins until word
// `word0 + r` of the own array has reached the same epoch.
__device__ __forceinline__ void signal_peers(const PeerGroup& g, uint32_t word0, uint32_t ctr, uint32_t epoch, bool wait) {
    const uint32_t lane = threadIdx.x & 31;
    uint32_t e = epoch;
    if (epoch == 0) {
        if (lane == 0) { e = g.flags[g.my_rank][ctr] + 1u; g.flags[g.my_rank][ctr] = e; }
        e = __shfl_sync(0xFFFFFFFFu, e, 0);
    }
    __threadfence_system();
    if ((int)lane < g.n) {
        *reinterpret_cast<volatile uint32_t*>(g.flags[lane] + word0 + g.my_rank) = e;
        if (wait) {
            const volatile uint32_t* mine = g.flags[g.my_rank] + word0 + lane;
            while ((int32_t)(*mine - e) < 0) __nanosleep(32);
            __threadfence_system();
        }
    }
}

struct OfferView {       // one per cloud, all arrays in price-sorted order, length Gpad
    uint32_t* packed = nullptr;
    uint32_t* bitmap = nullptr;  // [Gpad/32][bm_stride]
    uint32_t* bitmapT = nullptr; // [nsub][bm_words][kSubStride] (transposed, see kSubChunks)
    uint32_t* bitmapM = nullptr; // [D_mem+1][nsub][slice_rows][kSubStride]: per mem threshold m, rows mem[m] & vcpu[v]
                                 // (v = 0..D_vcpu), then mem[m] & ram[r] (r = 0..D_ram); null when not built
    int4* wide = nullptr;     // (mem_gb, vcpu, ram_gb, offer index)
    double* price = nullptr;  // NaN when the offer is not available in this cloud / padding
    int32_t* perm = nullptr;  // offer index, -1 when unavailable / padding
};

struct SelectArgs {
    // pod columns of this shard (device); nullable ones follow the C-ABI defaults
    const int32_t* req_mem;
    const int32_t* req_vcpu;
    const int32_t* req_ram;
    const double* max_price;
    const uint8_t* cloud;
    uint32_t P;
    // offer views
    OfferView view[2];
    uint32_t G, Gpad;
    const int32_t* distinct[3];
    uint32_t D[3];
    PackLayout pk;
    // per-call scratch
    uint32_t* rw;        // [P] packed thresholds
    uint32_t* order;     // [kGroups][P] row indices per group
    uint32_t* pos;       // [P] best sorted position so far (atomicMin target)
    uint32_t* counts;    // [kGroups] rows per group          } zero between calls: the grid kernel's last CTAs
    uint32_t* done;      // [1] row tiles finished             } clear them again (finish_tile), so no memset is
    uint32_t* tile_ctr;  // [ntiles] CTAs arrived per row tile } launched per call
    // outputs: the shard's slice is written into every peer's full-length vector at row0
    int32_t* best_out[RPK_MAX_GPUS];
    int n_out;
    int self_out;        // which of best_out lives on this GPU: the select kernels store there only and k_gather_push copies
                         // the slice to the peers in 16-byte NVLink stores; -1 = unknown, the kernels store to every vector
    uint32_t row0;
    int32_t* top5;       // [P*5] local, nullable
    // persistent bit-sliced path (kind 4, batches above the fused kernel's size)
    uint32_t nsub;       // 64-chunk sub-ranges of the transposed view
    uint16_t* key;       // [P] row class (0xFFFF: neither cloud)
    uint2* ord_rw;       // [P] {row id, threshold word} in class order (pos[] is indexed the same way): ONE scattered store per row
    uint32_t* hist;      // [kMaxClasses] rows per class: zero between calls (the grid kernel's block 0 clears it)
    uint32_t* k0_base;   // [K0 CTAs][kMaxClasses] first position of each class-sort CTA inside each class it has rows of
    uint32_t* hdr;       // control words, kHdr*
    PeerGroup peers;     // bound with rpk_peer_bind: the gather signals every peer once its slice has landed
    uint32_t tune_natural_order;  // tuning hook (RPK_TUNE=order=natural): row tiles in group order instead of heaviest first
    uint32_t slice;      // persistent select: rows grouped and the table staged per (cloud, mem threshold) on bitmapM
};

// One row's result.  With several output vectors (the all-gather) only the local one is written here -- scattered
// 4-byte stores over NVLink are far slower than 16-byte ones -- and the finished slice is pushed to the peers after.
__device__ __forceinline__ void store_best(const SelectArgs& a, uint32_t row, int32_t b) {
    if (a.self_out >= 0) { a.best_out[a.self_out][a.row0 + row] = b; return; }
    for (int o = 0; o < a.n_out; ++o) a.best_out[o][a.row0 + row] = b;
}

// The result of a row whose cheapest feasible offer sits at sorted position p of its cloud's view v (kNone: none): the
// offer index if its price is under the row's bound (strict, runpod_client.go:478; the bound is a prefix of the price
// order), else -1.
__device__ __forceinline__ void finish_row(const SelectArgs& a, const OfferView& v, uint32_t row, uint32_t p) {
    int32_t b = -1;
    if (p != kNone) {
        const double pr = v.price[p];
        const double mx = a.max_price ? a.max_price[row] : RPK_DEFAULT_MAX_PRICE;
        if (pr < mx) b = v.perm[p];
    }
    store_best(a, row, b);
}

// A row of neither SECURE nor COMMUNITY cloud: nothing is feasible (runpod_client.go:469-475)
__device__ __forceinline__ void finish_row_no_cloud(const SelectArgs& a, uint32_t row) {
    store_best(a, row, -1);
    if (a.top5) for (int k = 0; k < RPK_TOPK; ++k) a.top5[(size_t)row * RPK_TOPK + k] = -1;
}

// first position of the ascending array a[0, n) whose value is >= x (read-only data: the .nc path)
__device__ __forceinline__ uint32_t lower_bound_i32(const int32_t* __restrict__ a, uint32_t n, int32_t x) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(a + mid) < x) lo = mid + 1; else hi = mid; }
    return lo;
}

struct StatusArgs {
    const uint8_t* records;
    uint32_t stride;
    uint32_t N;
    uint64_t* hash_prev;    // updated in place
    uint64_t* hash_out;     // nullable
    uint32_t* changed_idx;  // nullable (seed, or a sharded sweep that only fills the exchange buffers)
    uint16_t* changed_code; // nullable: translateRunPodStatus code per changed slot (rpk.h RPK_CODE_*)
    uint32_t* n_changed;    // nullable (seed)
    uint32_t idx_base;      // added to emitted indices (shard offset)
    unsigned long long* tile_state;  // look-back state: one entry per CTA; zero between calls
    uint32_t* tile_counter;          // [2] scheduling ticket, finished CTAs; zero between calls
    uint32_t* stage_idx;             // [N] per-warp ordered index segments
    uint16_t* stage_code;            // [N] codes staged alongside
    uint32_t* unit_cnt;              // [N / 64 + 1] changed slots per 64-slot unit
    // sharded sweep: the changed list also goes into region `peers.my_rank` of every rank's exchange buffer
    int n_out;
    uint32_t* out_idx[RPK_MAX_GPUS];    // start of this rank's index region in rank o's buffer
    uint16_t* out_code[RPK_MAX_GPUS];   // ... code region (nullable)
    uint32_t* out_count[RPK_MAX_GPUS];  // rank o's count words (one per source rank)
    PeerGroup peers;                    // bound flags (n = 0: none), my_rank from the call: the CTA that finishes last signals
    // slot-list sweep (rpk_status_diff_slots): records[i] is the state of global slot slots[i] (ascending), whose previous
    // hash is hash_prev[slots[i] - idx_base]; entries outside [idx_base, idx_base + col_n) are skipped.  N = list length.
    const uint32_t* slots;  // null: whole-table sweep
    uint32_t col_n;
};

// launchers (each returns the number of kernels it launched, or throws CudaError)
struct CudaError { cudaError_t err; const char* what; const char* file; int line; };
#define RPK_CUDA(x) do { cudaError_t e__ = (x); if (e__ != cudaSuccess) throw ::rpk::CudaError{e__, #x, __FILE__, __LINE__}; } while (0)

// RPK_TUNE="pdl=off,order=natural,stagekb=<KB>,ipw=<n>,k0ctas=<n>" -- measurement hooks for tools/k1_tune.py; unset =
// the defaults chosen from those measurements.  The environment is read ONCE per process (this sits on the
// tens-of-microseconds latency path of production callers); tools that sweep settings inside one process set
// RPK_TUNE_RELOAD=1 before the first call.
struct Tune {
    bool pdl = true;             // pdl=off: launch without programmatic dependent launch
    bool natural_order = false;  // order=natural: row tiles in group order instead of heaviest first (packed / wide kernels)
    int stage_kb = 0;            // stagekb=: persistent select's stage cap (0: 220 KB)
    int items_per_warp = 0;      // ipw=: persistent select's items per warp (0: 4)
    int k0ctas = 0;              // k0ctas=: CTAs of the persistent select's class sort (0: four per SM)
    int grid_tiles = 0;          // gridtiles=: row tiles per launch of the packed / wide grid (0: as many as gridDim.x takes)
};
Tune read_tune();

// Launch with the programmatic-serialization attribute (PDL, rpk_device.cuh): the kernel may start before its stream
// predecessor has finished and synchronises with griddepcontrol.wait itself.
template <typename... KArgs, typename... Args>
void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
    RPK_CUDA(cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...));
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is per (function, device): set it once per (thread, device), so a
// warmed-up launch path issues nothing but launches (stream capture).  attr_dev: the call site's thread_local record.
template <typename K>
void allow_smem(K kernel, int bytes, int* attr_dev) {
    int dev = 0;
    RPK_CUDA(cudaGetDevice(&dev));
    if (*attr_dev == dev) return;
    RPK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    *attr_dev = dev;
}

struct OfferIngest {   // raw device columns in, views out
    uint32_t G;
    const int32_t* mem; const int32_t* vcpu; const int32_t* ram;  // vcpu/ram never null here (zero-filled)
    const double* secure_price; const double* community_price; const uint8_t* flags;
};

struct DeviceState;
int launch_offer_ingest(DeviceState& ds, const OfferIngest& in, cudaStream_t st);
// rpk_offers_refresh: the offers whose six columns differ bit for bit between `was` and `in` (same G).  Their number
// and the first RPK_OFFERS_DELTA_MAX of their indices, in no particular order, land in out[0] and out[1, ...) (mapped
// host memory) once the stream has run the kernel.  state: [2] words, zero between calls (the last CTA clears them).
struct OfferDiffArgs { OfferIngest was, in; uint32_t* state; uint32_t* idx; uint32_t* out; };
int launch_offer_diff(const OfferDiffArgs& a, cudaStream_t st);
struct PersistPlan;
// The top-5 lists' all-gather (rpk_select_device_gather_top5): the top-5 kernel writes out[self_out] (SelectArgs::top5
// points into it at 5 * row0), and the finished slice [5 * row0, 5 * (row0 + P)) is pushed into the other vectors.
struct Top5Gather { int32_t* out[RPK_MAX_GPUS]; int n_out; int self_out; };
int launch_select(const SelectArgs& a, int rows_per_warp, const PersistPlan* pl, int sm_count, cudaStream_t st,
                  const Top5Gather* t5 = nullptr);
uint32_t select_tiles_max(uint32_t P, int rows_per_warp);
int pick_rows_per_warp(uint32_t P, int sm_count);
int launch_status_diff(const StatusArgs& a, int sm_count, cudaStream_t st);
// one warp behind the stream's earlier work: signal the group's select words (epoch 0: self-counting), with `wait` also
// wait for every rank's signal; what: bit 0 = wait for the select epoch, bit 1 = the status epoch, bit 2 = the pending
// results epoch
int launch_peer_signal(const PeerGroup& g, uint32_t epoch, bool wait, cudaStream_t st);
int launch_peer_wait(const PeerGroup& g, uint32_t what, cudaStream_t st);
// persistent bit-sliced select (select_persist.cu)
struct PersistPlan { uint32_t S, per, qspan, grid, smem_bytes, slice, n_cursors, k0_blocks; int sm_count; };
PersistPlan persist_plan(const SelectArgs& a, int sm_count);  // a.pk.bm_words and a.nsub non-zero
uint32_t persist_hdr_words(const PersistPlan& pl);
int launch_select_persist(const SelectArgs& a, const PersistPlan& pl, cudaStream_t st);
uint32_t status_state_words(int sm_count);
// The five pod columns of a select: the caller's host columns (rpk_select, rpk_tick; the optional ones null when not
// passed), or staged device columns of a pod-table seed (same nullability).
struct PodCols { const int32_t* req_mem; const int32_t* req_vcpu; const int32_t* req_ram; const double* max_price; const uint8_t* cloud; };
// Five device columns, none null: the pod-requirement table (rows = slots) or a lane's compact pod columns
struct PodRows { int32_t* mem; int32_t* vcpu; int32_t* ram; double* max_price; uint8_t* cloud; };
// pod-requirement table (pods.cu): N = the table's rows; an entry of d_slots outside [0, N) is skipped by the seed and
// gathered as a row nothing matches (cloud byte 2)
// pending is the table's flag column (one byte per slot), cleared with the rows
int launch_pod_fill(const PodRows& t, uint8_t* pending, uint32_t N, int sm_count, cudaStream_t st);
int launch_pod_seed(const PodRows& t, uint32_t N, uint32_t n, const uint32_t* d_slots, const PodCols& in, cudaStream_t st);
int launch_pod_gather(const PodRows& t, uint32_t N, uint32_t n, const uint32_t* d_slots, const PodRows& out, cudaStream_t st);
// pending set of the pod table (pods.cu): flags[s] != 0 marks slot s pending
int launch_pod_mark(uint8_t* flags, uint32_t N, uint32_t n, const uint32_t* d_slots, const uint8_t* d_pending, cudaStream_t st);
struct PendingArgs {
    const uint8_t* flags;            // [N], 16-byte aligned
    uint32_t N;
    uint32_t* out;                   // [N] the pending slot ids, ascending
    uint32_t* n_out;                 // their number (device or mapped host memory)
    unsigned long long* tile_state;  // look-back state: pending_state_words entries; zero between calls
    uint32_t* ticket;                // [2] scheduling ticket, finished CTAs; zero between calls
};
uint32_t pending_state_words(int sm_count);
int launch_pod_pending(const PendingArgs& a, int sm_count, cudaStream_t st);
// pending results (rpk_select_pending_changed): per owned slot j (global slot r_lo + j), the last reported result -- its
// top-5 list, the five columns it was selected from and the offer-table generation it was selected against (0: none)
struct StoredResults { int32_t* mem; int32_t* vcpu; int32_t* ram; double* max_price; uint8_t* cloud; uint32_t* gen; int32_t* top5; };
struct StaleArgs {
    const uint8_t* flags; PodRows t; uint32_t N;  // the pending flags and the pod table (N slots)
    uint32_t u_lo;                   // first owned 16-slot unit; the owned slots start at 16 u_lo
    StoredResults r; uint32_t gen;   // stored results of the owned slots, the ctx's offer-table generation
    uint16_t* mask;                  // [units] scratch: the kept slots of each unit, from pass 1 to pass 2
    uint32_t* out;                   // the stale slot ids, ascending
    uint32_t* n_out;                 // their number (device memory)
    uint32_t* n_pending;             // the owned pending slots (device memory)
    unsigned long long* tile_state;  // look-back state: pending_state_words entries; zero between calls
    uint32_t* ticket;                // [3] scheduling ticket, finished CTAs, pending count; zero between calls
};
struct ResultDiffArgs {
    const uint32_t* list;              // the reselected slots, ascending
    PodRows cols; const int32_t* top5; // row i: the columns the reselect took and its top-5 list
    StoredResults r; uint32_t r_lo, gen;
    uint16_t* mask;                    // [units] scratch, as StaleArgs::mask
    unsigned long long* tile_state; uint32_t* ticket;  // as StaleArgs
};
// Where the diff writes: the changed rows, ascending, into each of n_out regions, their count into each count word,
// and the CTA that finishes last signals the results epoch when peers are bound.  The host call has one region, its
// device copy of the rows, and one count word in mapped memory; the one-process-per-GPU forms write region my_rank and
// word my_rank of every rank's exchange buffer.  Region of capacity cap: [slot : cap][best : cap][top5 : 5 cap] words.
struct ResultXchgArgs {
    ResultDiffArgs d;
    int n_out; uint32_t cap;
    uint32_t* region[RPK_MAX_GPUS];  // region my_rank of buffer o
    uint32_t* count[RPK_MAX_GPUS];   // word my_rank of buffer o
    PeerGroup peers;                 // bound flags (n = 0: none), my_rank from the call
};
// The stale step against a change window (rpk_offers_refresh): a result is also stale below the floor generation, or
// when a window entry newer than it reaches its row (rpk.h); one that nothing reaches gets generation s.gen.  win holds
// n_win (offer index, generation) pairs, newest first; the six raw columns are the current table's.
struct StaleReachArgs {
    StaleArgs s;
    uint32_t floor;
    const uint2* win; uint32_t n_win;
    const int32_t* mem; const int32_t* vcpu; const int32_t* ram; const double* sp; const double* cp; const uint8_t* flags;
};
// The reselect of the pending results (rpk_select_pending_changed*, select.cu): rows [0, dn[1]) of list, the count the
// stale step left on the device.  Row i's five columns go to out, its top-5 list to s.top5 (s: the offer views,
// G, the rank thresholds' distinct values and pk, as enqueue_select fills them).  counts (nullable) := dn[0, 2).
struct ReselectArgs {
    SelectArgs s;
    PodRows t;              // the pod table
    PodRows out;            // row i: the columns the list entry's row holds
    const uint32_t* list;   // the reselected slots
    const uint32_t* dn;     // [n_pending, n_reselected], written by the stale step
    uint32_t* counts;       // nullable: the caller's copy of dn
};
// a few waves sized for the worst case of n_max rows, the count read on the device; launches for n_max = 0 too
int launch_pod_reselect(const ReselectArgs& r, uint32_t n_max, int sm_count, cudaStream_t st);
int launch_pod_stale(const StaleArgs& a, uint32_t n_units, int sm_count, cudaStream_t st);
int launch_pod_stale_reach(const StaleReachArgs& a, uint32_t n_units, int sm_count, cudaStream_t st);
// the diff of the *d_n reselected rows, the count read on the device: the grid is sized for n_max rows, the worst case,
// and the CTAs past the count publish a zero count at once.  Launches for n_max = 0 too: the count 0 still goes out and
// the peers are still signalled
int launch_pod_result_xchg(const ResultXchgArgs& x, const uint32_t* d_n, uint32_t n_max, int sm_count, cudaStream_t st);
int launch_status_seed_slots(uint32_t n, const uint32_t* d_slots, const uint8_t* d_records, uint32_t stride, uint64_t* hash_prev,
                             uint32_t lo, uint32_t hi, cudaStream_t st);
// rpk_explain (explain.cu): out[i] for pod row i of the columns (req_mem required, the others nullable with rpk_select's
// defaults) against the two cloud views wide / price of a G-offer table
struct ExplainArgs {
    PodCols rows; uint32_t P;
    const int4* wide[2]; const double* price[2]; uint32_t G;
    rpk_explanation* out;
};
int launch_explain(const ExplainArgs& a, cudaStream_t st);

template <typename T>
struct DevBuf {  // grow-only device buffer, freed by its destructor
    T* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
    void reserve(size_t n) {
        if (n <= cap) return;
        if (p) RPK_CUDA(cudaFree(p));
        p = nullptr; cap = 0;
        size_t want = n + n / 4 + 256;
        RPK_CUDA(cudaMalloc(&p, want * sizeof(T)));
        cap = want;
    }
    void swap(DevBuf& o) { std::swap(p, o.p); std::swap(cap, o.cap); }
    template <typename S, typename F, typename... O> static void each(S& s, F&& f, O&... o) { f(s, o...); }  // a set of one (Grow)
};

// The five pod columns of a lane, of the pod table or of the stored results, each an allocation of its own: a column that
// grows moves alone (rpk.h, "Graph capture").  each: f(s.c, o.c...) for each column c in order; o...: PodBufs or PodRows.
struct PodBufs {
    DevBuf<int32_t> mem, vcpu, ram; DevBuf<double> max_price; DevBuf<uint8_t> cloud;
    template <typename S, typename F, typename... O> static void each(S& s, F&& f, O&... o) {
        f(s.mem, o.mem...); f(s.vcpu, o.vcpu...); f(s.ram, o.ram...); f(s.max_price, o.max_price...); f(s.cloud, o.cloud...);
    }
    PodRows rows() const { return PodRows{mem.p, vcpu.p, ram.p, max_price.p, cloud.p}; }
    PodCols cols() const { return PodCols{mem.p, vcpu.p, ram.p, max_price.p, cloud.p}; }
    void reserve(size_t n, const PodCols* only = nullptr) {  // n rows; with `only` (host columns): in the passed ones only
        mem.reserve(n);
        if (!only || only->req_vcpu) vcpu.reserve(n);
        if (!only || only->req_ram) ram.reserve(n);
        if (!only || only->max_price) max_price.reserve(n);
        if (!only || only->cloud) cloud.reserve(n);
    }
};

// The six columns of an offer table as uploaded, each its own allocation.  each: f(s.c, o.c...) for each column c in order.
struct OfferBufs {
    DevBuf<int32_t> mem, vcpu, ram; DevBuf<double> secure_price, community_price; DevBuf<uint8_t> flags;
    template <typename S, typename F, typename... O> static void each(S& s, F&& f, O&... o) {
        f(s.mem, o.mem...); f(s.vcpu, o.vcpu...); f(s.ram, o.ram...); f(s.secure_price, o.secure_price...);
        f(s.community_price, o.community_price...); f(s.flags, o.flags...);
    }
    void swap(OfferBufs& o) { each(*this, [](auto& a, auto& b) { a.swap(b); }, o); }
    OfferIngest view(uint32_t G) const { return OfferIngest{G, mem.p, vcpu.p, ram.p, secure_price.p, community_price.p, flags.p}; }
};

// One buffer, or one PodBufs, of a grow (rpk_pods_grow, rpk_status_grow).  The replacement of a column whose capacity is
// short (with `always`: of every column whatever its capacity) is allocated for every GPU before anything is copied or
// resized, so a refused allocation frees what was allocated and leaves the ctx as it was.  commit() puts the
// replacements in place once every copy is done; the old columns are freed with the Grow.
template <typename S>
struct Grow {
    S* b = nullptr;
    S fresh;
    void alloc(S& set, size_t n, bool always = false) { b = &set; S::each(set, [&](auto& old, auto& f) { if (always || n > old.cap) f.reserve(n); }, fresh); }
    template <typename F, typename... O> void each(F&& f, O&... o) const {  // f(old, dst, o.c...): column c now, after commit()
        S::each(*b, [&](auto& old, const auto& fr, auto&... x) { f(old, fr.p ? fr.p : old.p, x...); }, fresh, o...);
    }
    auto dst() const { return fresh.p ? fresh.p : b->p; }  // a buffer's address and capacity after commit()
    size_t dst_cap() const { return fresh.p ? fresh.cap : b->cap; }
    void keep(size_t n, cudaStream_t st) const {  // the first n rows stay as they are
        each([&](auto& old, auto* dst) { if (dst != old.p && n) RPK_CUDA(cudaMemcpyAsync(dst, old.p, n * sizeof(*dst), cudaMemcpyDeviceToDevice, st)); });
    }
    void commit() { S::each(*b, [](auto& old, auto& f) { if (f.p) old.swap(f); }, fresh); }
};

struct PinnedBuf {  // grow-only pinned host block, mapped: the device reaches it at d
    unsigned char* h = nullptr;
    unsigned char* d = nullptr;
    size_t cap = 0;
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf&) = delete;
    PinnedBuf& operator=(const PinnedBuf&) = delete;
    ~PinnedBuf() { if (h) cudaFreeHost(h); }
    void reserve(size_t n) {
        if (n <= cap) return;
        if (h) RPK_CUDA(cudaFreeHost(h));
        h = d = nullptr; cap = 0;
        const size_t want = n + n / 4;
        RPK_CUDA(cudaHostAlloc((void**)&h, want, cudaHostAllocMapped | cudaHostAllocPortable));
        RPK_CUDA(cudaHostGetDevicePointer((void**)&d, h, 0));
        cap = want;
    }
    void swap(PinnedBuf& o) { std::swap(h, o.h); std::swap(d, o.d); std::swap(cap, o.cap); }
};

// One ordering scope of a shard (rpk.h, "Ordering"): the buffers its device entry points share -- the device select
// scratch with the offer and pod tables, which host calls also write, or the device sweep scratch -- and the last device
// call that used them.  Host calls wait for that call before they start.  Inside a stream capture a device call neither waits nor records (an event recorded outside a capture cannot
// be waited on inside it), so a captured step keeps each entry point on one stream, as bench.py does.
struct ScratchScope {
    cudaStream_t last = nullptr;  // the stream of the last device call outside a capture
    cudaEvent_t ev = nullptr;     // recorded behind it
    // a device entry point, before its launches on st: false inside a capture, and then device_end records nothing
    bool device_begin(cudaStream_t st) {
        cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
        if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) { cudaGetLastError(); cs = cudaStreamCaptureStatusNone; }
        if (cs != cudaStreamCaptureStatusNone) return false;
        if (last != nullptr && last != st) RPK_CUDA(cudaStreamWaitEvent(st, ev, 0));
        return true;
    }
    void device_end(cudaStream_t st, bool tracked) {
        if (!tracked) return;
        RPK_CUDA(cudaEventRecord(ev, st));
        last = st;
    }
    void host_wait() { if (last) RPK_CUDA(cudaEventSynchronize(ev)); }
};

// One GPU of a ctx.  Built once at its final place (never copied or moved); the destructor synchronises the streams
// and destroys them and the events, then the members free the buffers with this device still current.
struct DeviceState {
    int dev = -1;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    // offer table
    uint32_t G = 0, Gpad = 0;
    bool offers_ready = false;
    // raw: the table's columns.  rpk_offers_refresh: the new columns land in raw_next next to them and take their place
    // after the diff; the diff's state words and index list, its mapped output, and the change window's device copy
    OfferBufs raw, raw_next;
    DevBuf<uint32_t> delta_state, delta_idx; PinnedBuf h_delta; DevBuf<uint2> win;
    DevBuf<unsigned long long> sort_keys; DevBuf<uint32_t> sort_vals;
    DevBuf<uint32_t> v_packed[2]; DevBuf<uint32_t> v_bitmap[2]; DevBuf<uint32_t> v_bitmapT[2]; DevBuf<uint32_t> v_bitmapM[2]; uint32_t nsub = 0; DevBuf<int4> v_wide[2]; DevBuf<double> v_price[2]; DevBuf<int32_t> v_perm[2];
    DevBuf<int32_t> distinct[3]; DevBuf<uint32_t> dcount;
    uint32_t D[3] = {0, 0, 0};
    PackLayout pk = {};
    int force_kind = 0;  // RPK_FORCE_KERNEL (tests): 0 auto, 1 generic, 2 packed+select, 3 packed+pos, 4 bit-sliced,
                         // 5 / 6 every batch of a non-empty table through the persistent / price-staged persistent kernel
    // select scratch.  The host entry points pipeline row sub-batches over four lanes (stream + staging +
    // scratch each) so that the H2D of one sub-batch, the kernels of another and the D2H of a third overlap;
    // the device entry points use dev_lane's scratch on the caller's stream.
    struct Lane {
        cudaStream_t stream = nullptr;
        cudaEvent_t done = nullptr;
        PodBufs cols; DevBuf<uint32_t> p_slots;  // rpk_select_slots: the sub-batch's slot ids, gathered into cols
        DevBuf<int32_t> top5;
        DevBuf<uint32_t> rw, order, pos, ctrs;
        DevBuf<uint16_t> key; DevBuf<uint2> ord_rw; DevBuf<uint32_t> hist, k0_base, hdr;  // persistent path
        bool ctrs_dirty = false;  // a select on this lane failed between its launches: re-zero the counters before the next one
        bool persist_dirty = false;
    };
    static constexpr int kLanes = 4;  // one per sub-batch of a 1M-row call: no upload ever waits for a kernel to free its buffers
    Lane lane[kLanes];
    // the rpk_select*_device* calls' scratch (no stream of its own): only device calls size it, so no host call of any
    // size frees what a captured device call points at (rpk.h, "Graph capture")
    Lane dev_lane;
    DevBuf<int32_t> best_full;
    // small-batch (latency) path: one pinned staging block in, one out
    PinnedBuf h_small; DevBuf<unsigned char> d_small_in; DevBuf<int32_t> d_small_out;
    // status
    DevBuf<uint8_t> s_records; DevBuf<uint64_t> s_hash_prev, s_hash_out;
    // a sweep's scratch: the look-back state and the ticket words (zero between calls by construction), the per-warp index
    // and code stages and the per-unit counts.  The host sweeps and rpk_tick use `sweep`; the rpk_status_diff*_device*
    // calls use `dev_sweep`, which only they size, as dev_lane above
    struct SweepScratch {
        DevBuf<unsigned long long> tile_state; DevBuf<uint32_t> misc;
        DevBuf<uint32_t> stage_idx; DevBuf<uint16_t> stage_code; DevBuf<uint32_t> unit_cnt;
        bool dirty = false;  // a launch failed midway: re-zero the look-back state before the next one
    };
    SweepScratch sweep, dev_sweep;
    DevBuf<uint32_t> s_seed_slots; DevBuf<uint8_t> s_seed_recs;  // slot lists of rpk_status_seed_slots and rpk_status_diff_slots
    PinnedBuf h_changed;                   // the host sweep's changed list: count, indices, codes
    DevBuf<rpk_explanation> explain_out;   // rpk_explain*: the shard's rows, copied to the caller (host-call scratch)
    cudaStream_t status_stream = nullptr;  // rpk_tick: the sweep next to the selection
    ScratchScope sel_scope, status_scope;  // the offer views, the pod table and dev_lane; dev_sweep
    uint32_t statusN = 0; bool status_sized = false;
    // pod-requirement table (rpk_pods_reset): the five columns of podsN slots, the whole table on every GPU of the ctx
    PodBufs pt_cols;
    DevBuf<unsigned char> pt_seed;         // rpk_pods_seed_slots: the slot ids and the columns of one seed
    // pending set: one flag byte per slot, the list k_pod_pending makes of it, and that kernel's look-back state and
    // tickets (zero between calls by construction, zeroed when allocated)
    DevBuf<uint8_t> pt_pending; DevBuf<uint32_t> pt_list; DevBuf<unsigned long long> pt_state; DevBuf<uint32_t> pt_ticket;
    PinnedBuf h_pending;                   // rpk_select_pending: the list's length, written by the kernel
    cudaStream_t pending_stream = nullptr; // rpk_select_pending: the list's copy to the caller, beside the select
    uint32_t podsN = 0; bool pods_sized = false;
    // pending results (rpk_select_pending_changed*), allocated on the first call after a reset: the stored results of the
    // owned slots, the stale list, the per-unit masks, [n_pending, n_reselected] of the stale step (r_dn), the reselected
    // rows' columns and top-5 lists (r_lane: sized once for the owned range, so a captured device-form call keeps
    // pointing at them), the host call's changed rows (r_out: [slots : cap][best : cap][top5 : 5 cap]) and their host
    // copy behind the counts (h_res: [r_dn's copy, the changed count : 64 bytes][the r_out layout]).  res_ready:
    // allocated for this table and not cleared since (rpk_pods_reset, a failed call)
    PodBufs r_cols; DevBuf<uint32_t> r_gen, r_list; DevBuf<int32_t> r_top5, r_out; DevBuf<uint16_t> r_mask;
    DevBuf<uint32_t> r_dn; Lane r_lane;
    PinnedBuf h_res;
    bool res_ready = false;
    // the owned range [res_lo, res_hi) the stored results were made for, set by the first call after rpk_pods_reset
    // (res_bound), and the (n_ranks, my_rank) it was computed from (rpk_select_pending_changed: the ctx's GPUs and the
    // shard); a call over another range is refused
    bool res_bound = false; uint32_t res_lo = 0, res_hi = 0; int res_ranks = 0, res_rank = 0;
    StoredResults results() const { const PodRows c = r_cols.rows(); return StoredResults{c.mem, c.vcpu, c.ram, c.max_price, c.cloud, r_gen.p, r_top5.p}; }
    PodRows pods_table() const { return pt_cols.rows(); }
    ~DeviceState();
};

}  // namespace rpk
