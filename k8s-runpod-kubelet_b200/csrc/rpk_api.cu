// rpk_api.cu -- the C-ABI of include/rpk.h: argument checks, device buffers, H2D/D2H, shard fan-out.
// No CPU implementation of any kernel lives here (or anywhere in the product): if CUDA is unusable every
// entry point returns an error.
#include <algorithm>
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <condition_variable>
#include <exception>
#include <functional>
#include <memory>
#include <mutex>
#include <new>
#include <thread>

#include "rpk_internal.cuh"

using namespace rpk;

// One host thread per extra GPU of a multi-GPU ctx: the per-shard halves of rpk_select / rpk_status_diff / rpk_tick
// (a dozen cudaMemcpyAsync + launches each) are issued in parallel instead of one shard after the other -- with 8
// GPUs behind one caller thread the serial issue, not PCIe, was the end-to-end bound.
struct ShardWorkers {
    struct W {
        std::thread th; std::mutex m; std::condition_variable cv;
        std::function<void()> job; bool has = false, quit = false;
    };
    std::vector<std::unique_ptr<W>> w;
    std::mutex dm; std::condition_variable dcv; int pending = 0;
    std::vector<std::exception_ptr> err;

    void start(int n) {
        err.resize((size_t)n);
        for (int i = 1; i < n; ++i) {
            w.emplace_back(new W());
            W* x = w.back().get();
            x->th = std::thread([this, x]() {
                for (;;) {
                    std::function<void()> job;
                    {
                        std::unique_lock<std::mutex> lk(x->m);
                        x->cv.wait(lk, [x] { return x->has || x->quit; });
                        if (x->quit) return;
                        job = std::move(x->job); x->has = false;
                    }
                    job();
                    { std::lock_guard<std::mutex> g(dm); --pending; }
                    dcv.notify_one();
                }
            });
        }
    }
    void stop() {
        for (auto& x : w) { { std::lock_guard<std::mutex> g(x->m); x->quit = true; } x->cv.notify_one(); x->th.join(); }
        w.clear();
    }
    // fn(s) for every shard s in [0, n): shard 0 on the calling thread, the others on their workers; rethrows the first failure
    template <typename F>
    void run(int n, F&& fn) {
        for (auto& e : err) e = nullptr;
        if (n > 1) {
            { std::lock_guard<std::mutex> g(dm); pending = n - 1; }
            for (int s = 1; s < n; ++s) {
                W* x = w[(size_t)s - 1].get();
                { std::lock_guard<std::mutex> g(x->m); x->job = [this, s, &fn]() { try { fn(s); } catch (...) { err[(size_t)s] = std::current_exception(); } }; x->has = true; }
                x->cv.notify_one();
            }
        }
        try { fn(0); } catch (...) { err[0] = std::current_exception(); }
        if (n > 1) { std::unique_lock<std::mutex> lk(dm); dcv.wait(lk, [this] { return pending == 0; }); }
        for (auto& e : err) if (e) std::rethrow_exception(e);
    }
};

struct rpk_ctx {
    std::vector<DeviceState> devs;  // one per shard, never resized: a DeviceState is neither copied nor moved
    std::vector<PeerGroup> bind;    // per shard: flag arrays bound with rpk_peer_bind (value-initialised: none)
    ShardWorkers workers;           // stopped (rpk_destroy) before devs is destroyed
    std::vector<std::pair<int, void*>> ipc_owned, ipc_mapped;  // (shard, ptr)
    std::string err;
    rpk_stats stats;
    uint64_t launches = 0;
    // the offer-table generation stored with a pending result: bumped by every upload and by every refresh that changes
    // an offer, skipping 0.  Results below offer_floor are stale; window (offer index, generation of its latest change;
    // newest first) lists the offers changed since offer_floor.  Empty window: offer_floor == offer_gen.
    uint32_t offer_gen = 0, offer_floor = 0;
    std::vector<uint2> window;
    explicit rpk_ctx(int n_gpus) : devs((size_t)n_gpus), bind((size_t)n_gpus) {}
};

rpk::DeviceState::~DeviceState() {
    if (dev < 0 || cudaSetDevice(dev) != cudaSuccess) { cudaGetLastError(); return; }  // creation failed before this GPU
    if (stream) cudaStreamSynchronize(stream);
    if (status_stream) cudaStreamSynchronize(status_stream);
    if (pending_stream) cudaStreamSynchronize(pending_stream);
    for (auto& ln : lane) if (ln.stream) cudaStreamSynchronize(ln.stream);
    for (auto& ln : lane) {
        if (ln.done) cudaEventDestroy(ln.done);
        if (ln.stream) cudaStreamDestroy(ln.stream);
    }
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    if (sel_scope.ev) cudaEventDestroy(sel_scope.ev);
    if (status_scope.ev) cudaEventDestroy(status_scope.ev);
    if (status_stream) cudaStreamDestroy(status_stream);
    if (pending_stream) cudaStreamDestroy(pending_stream);
    if (stream) cudaStreamDestroy(stream);
    cudaGetLastError();
}

static thread_local std::string g_create_err;

namespace {

int fail(rpk_ctx* ctx, int code, const std::string& msg) {
    if (ctx) ctx->err = msg; else g_create_err = msg;
    return code;
}

template <typename F>
int guarded(rpk_ctx* ctx, F&& f) {
    try {
        return f();
    } catch (const CudaError& e) {
        char buf[512];
        snprintf(buf, sizeof(buf), "CUDA error %d (%s) at %s:%d: %s", (int)e.err, cudaGetErrorString(e.err), e.file, e.line, e.what);
        cudaGetLastError();  // clear the sticky-free error state
        return fail(ctx, e.err == cudaErrorMemoryAllocation ? RPK_ENOMEM : RPK_ECUDA, buf);
    } catch (const std::bad_alloc&) {
        return fail(ctx, RPK_ENOMEM, "host allocation failed");
    } catch (...) {
        return fail(ctx, RPK_ECUDA, "unexpected exception");
    }
}

inline void shard_range(uint32_t total, int n, int s, uint32_t* lo, uint32_t* hi) {
    *lo = (uint32_t)((uint64_t)total * (uint64_t)s / (uint64_t)n);
    *hi = (uint32_t)((uint64_t)total * (uint64_t)(s + 1) / (uint64_t)n);
}

bool bad_shard(const rpk_ctx* ctx, int shard) { return shard < 0 || (size_t)shard >= ctx->devs.size(); }

// A device entry point on GPU `shard` (in range, its arguments checked), by the ordering rule of rpk.h: under guarded,
// with the device set, prep(ds) sizes buffers and makes the refusals that need the device (nonzero: its code, and nothing
// is enqueued); then run(ds, st) enqueues the call on st, the caller's stream or, when NULL, the shard's own, after the
// last device call of `scope` and recorded as its last one (no scope: neither).
template <typename Prep, typename Run>
int device_call(rpk_ctx* ctx, int shard, void* stream, ScratchScope DeviceState::*scope, Prep&& prep, Run&& run) {
    DeviceState& ds = ctx->devs[(size_t)shard];
    return guarded(ctx, [&]() -> int {
        RPK_CUDA(cudaSetDevice(ds.dev));
        if (int rc = prep(ds)) return rc;
        const cudaStream_t st = stream ? (cudaStream_t)stream : ds.stream;
        const bool tracked = scope && (ds.*scope).device_begin(st);
        run(ds, st);
        if (scope) (ds.*scope).device_end(st, tracked);
        return RPK_OK;
    });
}
template <typename Run>
int device_call(rpk_ctx* ctx, int shard, void* stream, ScratchScope DeviceState::*scope, Run&& run) {
    return device_call(ctx, shard, stream, scope, [](DeviceState&) { return RPK_OK; }, run);
}

// Where the rows of a select come from.  Host sources (rpk_select, rpk_tick: columns; rpk_select_slots: a list) become
// device sources by their upload.  Device sources are on the selecting GPU (rpk_select_device*: columns;
// rpk_select_slots_device*: a list; rpk_select_pending*: the list k_pod_pending or k_pod_stale left there).
struct RowSource {
    enum Kind { HostCols, HostList, DevCols, DevList };
    Kind kind;
    PodCols cols;           // HostCols, DevCols: row i of the call is row i of the columns (the optional ones nullable)
    const uint32_t* slots;  // HostList, DevList: row i of the call is pod-table row slots[i]
};

// every entry of slots[0, n) is a row of a pod table of N rows.  The pipelined select runs this per sub-batch on the
// thread that enqueues the next sub-batch, so its cost lands on the call in full: the CPU reads the list, measured at
// 0.3-0.65 ns per id on an H100 host (0.35-0.56 ms per 1M ids, DESIGN section 4 "Pod table").
// RPK_MEASURE_UNCHECKED_SLOTS: only for the copy of the library tools/select_slots_probe.py builds to time the check; it
// accepts every list (k_pod_gather gathers an entry outside the table as a row nothing matches and reads nothing there).
bool slots_below(const uint32_t* slots, uint32_t n, uint32_t N) {
#ifdef RPK_MEASURE_UNCHECKED_SLOTS
    return true;
#endif
    uint32_t bad = 0;
    for (uint32_t i = 0; i < n; ++i) bad |= (uint32_t)(slots[i] >= N);
    return bad == 0;
}

// The buffers of lane ln that a select of `rows` rows from src writes: the pod columns it uploads or gathers, a host list's
// slot ids, the top-5 lists.  Allocates only when one grows, so a device call stays capturable after a call of its size.
void reserve_lane(DeviceState::Lane& ln, size_t rows, const RowSource& src, bool top5) {
    // a list's gather writes all five columns, host columns only the ones passed
    if (src.kind != RowSource::DevCols) ln.cols.reserve(rows, src.kind == RowSource::HostCols ? &src.cols : nullptr);
    if (src.kind == RowSource::HostList) ln.p_slots.reserve(rows);
    if (top5) ln.top5.reserve(rows * RPK_TOPK);
}

// SelectArgs keeps its pod columns flat for the kernels: set them to c from row b0 on (null stays null), and read them back
void set_pod_cols(SelectArgs& a, const PodCols& c, uint32_t b0 = 0) {
    const auto at = [b0](auto* col) { return col ? col + b0 : nullptr; };
    a.req_mem = at(c.req_mem); a.req_vcpu = at(c.req_vcpu); a.req_ram = at(c.req_ram); a.max_price = at(c.max_price); a.cloud = at(c.cloud);
}
PodCols pod_cols(const SelectArgs& a) { return PodCols{a.req_mem, a.req_vcpu, a.req_ram, a.max_price, a.cloud}; }

// Host columns c on the device: put(col, to.x) copies each passed column col to to.x (a lane's buffer, a staging offset)
template <typename To, typename Put> PodCols to_device(const PodCols& c, To& to, Put&& put) {
    const auto at = [&](const auto* col, auto& dst) -> decltype(col) { return col ? (decltype(col))put(col, dst) : nullptr; };
    return PodCols{at(c.req_mem, to.mem), at(c.req_vcpu, to.vcpu), at(c.req_ram, to.ram), at(c.max_price, to.max_price), at(c.cloud, to.cloud)};
}

// a's pod columns: rows [b0, b0 + n) of the device source src.  Columns go in as pointers; a list is gathered from the
// pod table into lane ln's columns on st.  Returns the kernels launched.
int pod_columns(DeviceState& ds, DeviceState::Lane& ln, const RowSource& src, uint32_t b0, uint32_t n, SelectArgs& a, cudaStream_t st) {
    if (src.kind == RowSource::DevCols) {
        set_pod_cols(a, src.cols, b0);
        return 0;
    }
    set_pod_cols(a, ln.cols.cols());
    return launch_pod_gather(ds.pods_table(), ds.podsN, n, src.slots + b0, ln.cols.rows(), st);
}

// One select on ds in lane ln's scratch: `a` holds the pod columns, P and the outputs; this adds the offer views and the
// scratch and launches on st.  A bit-sliced table takes the persistent kernel above the fused kernel's batch size and
// the fused kernel otherwise (which also serves an empty table at any batch size).  t5: the top-5 lists' gather, if
// any.  Returns the kernels launched.
// a's offer side: ds's views, G, the distinct values of the rank thresholds and the pack layout
void offer_args(const DeviceState& ds, SelectArgs& a) {
    for (int c = 0; c < 2; ++c) {
        a.view[c].packed = ds.v_packed[c].p; a.view[c].bitmap = ds.v_bitmap[c].p; a.view[c].bitmapT = ds.v_bitmapT[c].p;
        a.view[c].bitmapM = ds.pk.slice_rows ? ds.v_bitmapM[c].p : nullptr; a.view[c].wide = ds.v_wide[c].p;
        a.view[c].price = ds.v_price[c].p; a.view[c].perm = ds.v_perm[c].p;
    }
    a.G = ds.G; a.Gpad = ds.Gpad; a.pk = ds.pk; a.nsub = ds.nsub;
    for (int d = 0; d < 3; ++d) { a.distinct[d] = ds.distinct[d].p; a.D[d] = ds.D[d]; }
}

int enqueue_select(DeviceState& ds, DeviceState::Lane& ln, SelectArgs& a, cudaStream_t st, const Top5Gather* t5 = nullptr) {
    offer_args(ds, a);
    const uint32_t P = a.P;
    const int R = ds.pk.bm_words ? 0 : pick_rows_per_warp(P, ds.sm_count);  // rows per warp of the packed / wide kernels
    const uint32_t tiles = R ? select_tiles_max(P, R) : 0u;
    ln.rw.reserve(P); ln.order.reserve((size_t)kGroups * P); ln.pos.reserve(P);
    // worst case (1 row per warp; the persistent kernel's row blocks: one partial block per row group): never regrown mid-pipeline
    const size_t need = std::max<size_t>((size_t)2 * kGroups + tiles, (size_t)P / 8 + 3 * kGroups + kMaxGroups);
    if (need > ln.ctrs.cap || ln.ctrs_dirty) {
        // the counters are zero between calls by construction (finish_tile); a fresh or suspect buffer is zeroed here
        ln.ctrs.reserve(need);
        RPK_CUDA(cudaMemset(ln.ctrs.p, 0, ln.ctrs.cap * sizeof(uint32_t)));
        RPK_CUDA(cudaDeviceSynchronize());
        ln.ctrs_dirty = false;
    }
    a.rw = ln.rw.p; a.order = ln.order.p; a.pos = ln.pos.p;
    a.counts = ln.ctrs.p; a.done = ln.ctrs.p + kGroups; a.tile_ctr = ln.ctrs.p + 2 * kGroups;
    const bool persist = ds.pk.bm_words && ds.nsub && (P > kFusedRowsMax || ds.pk.no_fused);
    PersistPlan pl;
    if (persist) {
        pl = persist_plan(a, ds.sm_count);
        ln.key.reserve(P); ln.ord_rw.reserve(P);
        const size_t hdr_words = persist_hdr_words(pl);
        const bool fresh = !ln.hist.p || hdr_words > ln.hdr.cap;
        ln.hist.reserve(2 * kMaxClasses); ln.hdr.reserve(hdr_words);
        ln.k0_base.reserve((size_t)pl.k0_blocks * kMaxClasses);  // written by k_pod_classify before k_pod_scatter reads it: never zeroed
        if (fresh || ln.persist_dirty) {  // zero between calls by construction (k_pod_classify's last block, the pushers)
            RPK_CUDA(cudaMemset(ln.hist.p, 0, ln.hist.cap * sizeof(uint32_t)));
            RPK_CUDA(cudaMemset(ln.hdr.p, 0, ln.hdr.cap * sizeof(uint32_t)));
            RPK_CUDA(cudaDeviceSynchronize());
            ln.persist_dirty = false;
        }
        a.key = ln.key.p; a.ord_rw = ln.ord_rw.p; a.hist = ln.hist.p; a.k0_base = ln.k0_base.p; a.hdr = ln.hdr.p;
    }
    // the lane's counters are suspect until every launch of the call was accepted
    ln.ctrs_dirty = true; ln.persist_dirty = true;
    const int n = launch_select(a, R, persist ? &pl : nullptr, ds.sm_count, st, t5);
    ln.ctrs_dirty = false; ln.persist_dirty = false;
    return n;
}

void count_select(rpk_ctx* ctx, uint32_t P, uint32_t G) {
    ctx->stats.select_calls += 1;
    ctx->stats.offer_scores += (uint64_t)P * G;
}

// The push kernel moves 16-byte units: every vector must share the slice's alignment.
bool same_phase(int n_out, int32_t* const* ptrs) {
    for (int o = 1; o < n_out; ++o)
        if (((uintptr_t)ptrs[o] & 15u) != ((uintptr_t)ptrs[0] & 15u)) return false;
    return true;
}

// Which of the vectors lives on GPU `shard` (the others are peers' memory); -1 if none does.  Vectors this ctx
// allocated (rpk_ipc_alloc) or mapped from a peer (rpk_ipc_open) are known exactly; anything else is asked of the driver.
int local_vector(const rpk_ctx* ctx, int shard, int dev, int n_out, int32_t* const* ptrs) {
    for (int o = 0; o < n_out; ++o)
        for (const auto& m : ctx->ipc_owned) if (m.first == shard && m.second == (void*)ptrs[o]) return o;
    for (int o = 0; o < n_out; ++o) {
        bool mapped = false;
        for (const auto& m : ctx->ipc_mapped) if (m.second == (void*)ptrs[o]) { mapped = true; break; }
        if (mapped) continue;  // a peer's vector, whatever the driver reports for IPC mappings
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, ptrs[o]) != cudaSuccess) { cudaGetLastError(); continue; }
        if (at.type == cudaMemoryTypeDevice && at.device == dev) return o;
    }
    return -1;
}

// The output vector of an assignment gather the select kernels write (-1: they store into every vector directly).  A
// single vector is written whatever memory it is.
int find_local_vector(const rpk_ctx* ctx, int shard, int dev, int n_out, int32_t* const* ptrs) {
    if (n_out == 1) return 0;
    return same_phase(n_out, ptrs) ? local_vector(ctx, shard, dev, n_out, ptrs) : -1;
}

// Row sub-batches of the host entry point.  The first one is small, so that the first kernel starts after ~3 MB of
// H2D; the following ones grow (128k, 256k, 384k, 512k, 512k ... rows), because every select call pays a fixed cost
// (class sort, stage load, queue tail) that eight equal sub-batches paid eight times: with growing sizes each kernel
// is about as long as the upload of the next, larger sub-batch.
constexpr uint32_t kSubBatchRows = 131072;
constexpr uint32_t kSubBatchMaxMul = 4;
// The pending list (a device list in a host call) needs no upload for the sub-batches to hide, but they still overlap
// the copies of best and top5 back to the host: measured at 1M rows on an H100 (700 W), the sub-batches take 0.97 ms
// against 1.02 ms for one select over the whole list with top-5, which the Provider's tick asks for, and 0.55 against
// 0.52 ms without, each inside the other's spread (DESIGN section 4, "Pending set"): the list keeps the pipeline's shape.
// RPK_MEASURE_PENDING_ONE_SELECT: only for the copy of the library tools/select_pending_probe.py builds to time the other
// shape.
inline uint32_t sub_batch_rows(RowSource::Kind kind, int j, uint32_t remaining) {
#ifdef RPK_MEASURE_PENDING_ONE_SELECT
    if (kind == RowSource::DevList) return remaining;
#endif
    (void)kind;
    const uint32_t want = kSubBatchRows * (uint32_t)((j + 1) < (int)kSubBatchMaxMul ? (j + 1) : (int)kSubBatchMaxMul);
    return remaining < want + kSubBatchRows / 2 ? remaining : want;  // do not leave a sliver behind
}
inline uint32_t sub_batch_cap(RowSource::Kind kind, uint32_t Ps) {  // largest sub-batch a shard of Ps rows produces
    uint32_t cap = 0, left = Ps;
    for (int j = 0; left; ++j) { const uint32_t nb = sub_batch_rows(kind, j, left); cap = nb > cap ? nb : cap; left -= nb; }
    return cap ? cap : 1;
}

// Where n pod rows go in a staging block from byte `base` on: [mem][vcpu][ram][max_price, 8-byte aligned][cloud], then its end
struct PodBlock { size_t mem, vcpu, ram, max_price, cloud, end; };
PodBlock pod_block(size_t n, size_t base) {
    const size_t price = (base + 12 * n + 7) & ~(size_t)7;
    return PodBlock{base, base + 4 * n, base + 8 * n, price, price + 8 * n, price + 9 * n};
}

// Latency path of the host entry point (micro-batches, one GPU): the five pod columns -- or, from the pod table, the
// slot ids -- are packed into one pinned block -> ONE H2D (then the gather, for slots); best and top5 come back in ONE
// D2H; one stream synchronise.  Same kernels.  Slot ids are in range here.  Returns the kernels launched.
int select_small(DeviceState& ds, uint32_t P, const RowSource& src, int32_t* best, int32_t* top5) {
    RPK_CUDA(cudaSetDevice(ds.dev));
    ds.sel_scope.host_wait();
    const size_t in_cap = (size_t)kSmallBatch * 24, out_cap = (size_t)kSmallBatch * 6 * 4;
    ds.h_small.reserve(in_cap + out_cap);
    ds.d_small_in.reserve(in_cap); ds.d_small_out.reserve((size_t)kSmallBatch * 6);
    unsigned char* h = ds.h_small.h;
    DeviceState::Lane& ln = ds.lane[0];
    cudaStream_t st = ln.stream;
    unsigned char* d = ds.d_small_in.p;
    RowSource dev = src;  // the rows' device source: the block's columns or slot ids in d_small_in, or the pending list
    size_t bytes = 0;
    if (src.kind == RowSource::HostList) {
        bytes = (size_t)P * 4;
        memcpy(h, src.slots, bytes);
        dev = RowSource{RowSource::DevList, PodCols{}, (const uint32_t*)d};
    } else if (src.kind == RowSource::HostCols) {
        const PodBlock blk = pod_block(P, 0);
        bytes = blk.end;
        const auto pack = [&](const auto* col, size_t o) { memcpy(h + o, col, (size_t)P * sizeof(*col)); return d + o; };
        dev = RowSource{RowSource::DevCols, to_device(src.cols, blk, pack), nullptr};
    }
    reserve_lane(ln, kSmallBatch, dev, false);
    if (bytes) RPK_CUDA(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, st));
    SelectArgs a{};
    int launches = pod_columns(ds, ln, dev, 0, P, a, st);
    a.P = P;
    a.best_out[0] = ds.d_small_out.p; a.n_out = 1; a.self_out = 0; a.row0 = 0; a.top5 = top5 ? ds.d_small_out.p + P : nullptr;
    launches += enqueue_select(ds, ln, a, st);
    int32_t* hout = (int32_t*)(h + in_cap);
    RPK_CUDA(cudaMemcpyAsync(hout, ds.d_small_out.p, (size_t)P * 4 * (top5 ? 6 : 1), cudaMemcpyDeviceToHost, st));
    RPK_CUDA(cudaStreamSynchronize(st));
    memcpy(best, hout, (size_t)P * 4);
    if (top5) memcpy(top5, hout + P, (size_t)P * 4 * RPK_TOPK);
    return launches;
}

bool has_int32_max(const int32_t* col, uint32_t n) {
    if (!col) return false;
    for (uint32_t i = 0; i < n; ++i) if (col[i] == INT32_MAX) return true;
    return false;
}


// The pipelined host select of a run_host call: P rows from src[s] on GPU s into the caller's best and top5 (nullable)
struct HostSelect { uint32_t P; std::vector<RowSource> src; int32_t* best; int32_t* top5; };

// Buffers of the pipelined host select, sized from the calling thread (peers write into each other's best_full, so
// every GPU's vector must exist before any shard is enqueued).  After the first call of a size this allocates nothing.
void reserve_select(rpk_ctx* ctx, const HostSelect& sel) {
    const int n = (int)ctx->devs.size();
    for (int s = 0; s < n; ++s) {
        DeviceState& ds = ctx->devs[(size_t)s];
        uint32_t lo, hi; shard_range(sel.P, n, s, &lo, &hi);
        const uint32_t Ps = hi - lo;
        const uint32_t cap = sub_batch_cap(sel.src[(size_t)s].kind, Ps);
        RPK_CUDA(cudaSetDevice(ds.dev));
        ds.best_full.reserve(sel.P);
        for (auto& ln : ds.lane) {
            reserve_lane(ln, cap, sel.src[(size_t)s], sel.top5 != nullptr);
            if (cap == Ps) break;  // a single sub-batch uses lane 0 only
        }
    }
}

// Rows [b0, b0 + nb) of src as a device source for pod_columns, from row *at on: a host source's rows are uploaded into
// lane ln's buffers on st (*at = 0; a host list's slot ids must already be checked), a device source is src itself
// (*at = b0).
RowSource upload_rows(DeviceState::Lane& ln, const RowSource& src, uint32_t b0, uint32_t nb, cudaStream_t st, uint32_t* at) {
    *at = 0;
    if (src.kind == RowSource::HostList) {
        RPK_CUDA(cudaMemcpyAsync(ln.p_slots.p, src.slots + b0, (size_t)nb * 4, cudaMemcpyHostToDevice, st));
        return RowSource{RowSource::DevList, PodCols{}, ln.p_slots.p};
    }
    if (src.kind == RowSource::HostCols) {
        const auto upload = [&](const auto* col, auto& buf) {  // rows [b0, b0 + nb) into the lane's buffer
            RPK_CUDA(cudaMemcpyAsync(buf.p, col + b0, (size_t)nb * sizeof(*col), cudaMemcpyHostToDevice, st));
            return buf.p;
        };
        return RowSource{RowSource::DevCols, to_device(src.cols, ln.cols, upload), nullptr};
    }
    *at = b0;
    return src;
}

// One shard's half of the host select: row sub-batches rotate over the lanes; within a lane everything is stream
// ordered (H2D -> kernels -> D2H), across lanes copies and kernels overlap.  ds.ev[0] / ds.ev[3] bracket it on ds.stream;
// the caller synchronises ds.stream.  Slot ids are checked per sub-batch just before their upload: false = an entry
// outside the pod table, and nothing from that sub-batch on was enqueued (the lanes still drain into ds.stream).
bool enqueue_select_shard(rpk_ctx* ctx, int s, const HostSelect& sel, uint64_t* launches) {
    const int n = (int)ctx->devs.size();
    DeviceState& ds = ctx->devs[(size_t)s];
    const RowSource& src = sel.src[(size_t)s];
    uint32_t lo, hi; shard_range(sel.P, n, s, &lo, &hi);
    RPK_CUDA(cudaSetDevice(ds.dev));
    RPK_CUDA(cudaEventRecord(ds.ev[0], ds.stream));
    for (auto& ln : ds.lane) RPK_CUDA(cudaStreamWaitEvent(ln.stream, ds.ev[0], 0));
    bool ok = true;
    int j = 0;
    for (uint32_t b0 = lo, nb = 0; b0 < hi; b0 += nb, ++j) {
        nb = sub_batch_rows(src.kind, j, hi - b0);
        DeviceState::Lane& ln = ds.lane[j % DeviceState::kLanes];
        cudaStream_t st = ln.stream;
        if (src.kind == RowSource::HostList && !slots_below(src.slots + b0, nb, ds.podsN)) { ok = false; break; }
        uint32_t at;
        const RowSource dev = upload_rows(ln, src, b0, nb, st, &at);
        SelectArgs a{};
        *launches += (uint64_t)pod_columns(ds, ln, dev, at, nb, a, st);
        a.P = nb;
        for (int o = 0; o < n; ++o) a.best_out[o] = ctx->devs[(size_t)o].best_full.p;
        a.n_out = n; a.row0 = b0; a.top5 = sel.top5 ? ln.top5.p : nullptr;
        a.self_out = s;  // own vector; finished push blocks / sub-batches are forwarded to the peers
        *launches += (uint64_t)enqueue_select(ds, ln, a, st);
        RPK_CUDA(cudaMemcpyAsync(sel.best + b0, ds.best_full.p + b0, (size_t)nb * 4, cudaMemcpyDeviceToHost, st));
        if (sel.top5) RPK_CUDA(cudaMemcpyAsync(sel.top5 + (size_t)b0 * RPK_TOPK, ln.top5.p, (size_t)nb * RPK_TOPK * 4, cudaMemcpyDeviceToHost, st));
    }
    for (auto& ln : ds.lane) {
        RPK_CUDA(cudaEventRecord(ln.done, ln.stream));
        RPK_CUDA(cudaStreamWaitEvent(ds.stream, ln.done, 0));
    }
    RPK_CUDA(cudaEventRecord(ds.ev[3], ds.stream));
    return ok;
}

// Scratch w of a sweep over N records (or list entries) on a GPU of sm_count SMs: the look-back state and tickets --
// zero between calls by construction, zeroed here when (re)allocated -- and the per-warp index stage, its code stage
// (`codes`) and the per-unit counts.
void reserve_sweep_scratch(DeviceState::SweepScratch& w, int sm_count, uint32_t N, bool codes) {
    const uint32_t cap = N ? N : 1;
    const size_t need = status_state_words(sm_count);
    if (need > w.tile_state.cap || !w.misc.p || w.dirty) {
        w.tile_state.reserve(need);
        w.misc.reserve(64);
        RPK_CUDA(cudaMemset(w.tile_state.p, 0, w.tile_state.cap * sizeof(unsigned long long)));
        RPK_CUDA(cudaMemset(w.misc.p, 0, w.misc.cap * sizeof(uint32_t)));
        RPK_CUDA(cudaDeviceSynchronize());
        w.dirty = false;
    }
    w.stage_idx.reserve(cap + 64); w.unit_cnt.reserve(cap / 32 + 2);
    if (codes) w.stage_code.reserve(cap + 64);
}

// the StatusArgs fields of the scratch reserve_sweep_scratch sized
void sweep_scratch_args(const DeviceState::SweepScratch& w, bool codes, StatusArgs& a) {
    a.tile_state = w.tile_state.p; a.tile_counter = w.misc.p;
    a.stage_idx = w.stage_idx.p; a.stage_code = codes ? w.stage_code.p : nullptr; a.unit_cnt = w.unit_cnt.p;
}

struct StatusHostArgs {
    uint32_t N; const uint8_t* records; uint32_t stride;
    uint32_t* changed_idx; uint16_t* changed_code; uint32_t* n_changed; uint64_t* hashes_out; bool report;
    const uint32_t* slots; uint32_t n_slots;  // rpk_status_diff_slots: records holds the n_slots listed slots (ascending)
};

// Shard s of a host sweep: its hash column holds global slots [lo, hi); its records are [p0, p1) of the caller's table
// (the same range) or, for a slot list, the entries whose slot lies in [lo, hi) -- two binary searches, since the list
// is ascending.
struct ShardPart { uint32_t lo, hi, p0, p1; };
ShardPart shard_part(const rpk_ctx* ctx, int s, const StatusHostArgs& h) {
    ShardPart p;
    shard_range(h.N, (int)ctx->devs.size(), s, &p.lo, &p.hi);
    p.p0 = p.lo; p.p1 = p.hi;
    if (h.slots) {
        p.p0 = (uint32_t)(std::lower_bound(h.slots, h.slots + h.n_slots, p.lo) - h.slots);
        p.p1 = (uint32_t)(std::lower_bound(h.slots, h.slots + h.n_slots, p.hi) - h.slots);
    }
    return p;
}

// Sizes one shard's buffers (calling thread).  The changed list comes back through mapped pinned memory -- the kernel's
// final copy writes indices, codes and the count straight into it, so the host needs ONE stream synchronise and no
// device-to-host copy whose size it would first have to learn.
void reserve_status_shard(rpk_ctx* ctx, int s, const StatusHostArgs& h) {
    DeviceState& ds = ctx->devs[(size_t)s];
    const ShardPart sp = shard_part(ctx, s, h);
    const uint32_t Ns = sp.p1 - sp.p0, cap = Ns ? Ns : 1;
    RPK_CUDA(cudaSetDevice(ds.dev));
    ds.s_records.reserve((size_t)cap * h.stride);
    if (h.slots) ds.s_seed_slots.reserve(cap);
    if (h.hashes_out) ds.s_hash_out.reserve(cap);
    reserve_sweep_scratch(ds.sweep, ds.sm_count, Ns, h.changed_code != nullptr);
    ds.h_changed.reserve(h.report ? (size_t)cap * (h.changed_code ? 6 : 4) + 64 : 64);
}

// One shard's half of a host sweep, enqueued on st (ds.ev[0..2] bracket copy and kernel, ds.ev[3] follows the hash
// copy); the caller synchronises.
void enqueue_status_shard(rpk_ctx* ctx, int s, const StatusHostArgs& h, cudaStream_t st, uint64_t* launches) {
    DeviceState& ds = ctx->devs[(size_t)s];
    const ShardPart sp = shard_part(ctx, s, h);
    const uint32_t lo = sp.lo, Ns = sp.p1 - sp.p0, cap = Ns ? Ns : 1;
    RPK_CUDA(cudaSetDevice(ds.dev));
    RPK_CUDA(cudaEventRecord(ds.ev[0], st));
    if (Ns) RPK_CUDA(cudaMemcpyAsync(ds.s_records.p, h.records + (size_t)sp.p0 * h.stride, (size_t)Ns * h.stride, cudaMemcpyHostToDevice, st));
    if (Ns && h.slots) RPK_CUDA(cudaMemcpyAsync(ds.s_seed_slots.p, h.slots + sp.p0, (size_t)Ns * 4, cudaMemcpyHostToDevice, st));
    RPK_CUDA(cudaEventRecord(ds.ev[1], st));
    // mapped block: [count : 64 bytes][indices : cap u32][codes : cap u16]
    uint32_t* m_count = reinterpret_cast<uint32_t*>(ds.h_changed.d);
    uint32_t* m_idx = reinterpret_cast<uint32_t*>(ds.h_changed.d + 64);
    uint16_t* m_code = reinterpret_cast<uint16_t*>(ds.h_changed.d + 64 + (size_t)cap * 4);
    *reinterpret_cast<volatile uint32_t*>(ds.h_changed.h) = 0u;
    StatusArgs a{};
    a.records = ds.s_records.p; a.stride = h.stride; a.N = Ns; a.hash_prev = ds.s_hash_prev.p;
    a.hash_out = h.hashes_out ? ds.s_hash_out.p : nullptr;
    a.changed_idx = h.report ? m_idx : nullptr; a.n_changed = h.report ? m_count : nullptr;
    a.changed_code = h.report && h.changed_code ? m_code : nullptr;
    a.idx_base = lo;
    sweep_scratch_args(ds.sweep, h.changed_code != nullptr, a);
    if (h.slots) { a.slots = ds.s_seed_slots.p; a.col_n = sp.hi - sp.lo; }
    ds.sweep.dirty = true;
    if (Ns) *launches += (uint64_t)launch_status_diff(a, ds.sm_count, st);
    ds.sweep.dirty = false;
    RPK_CUDA(cudaEventRecord(ds.ev[2], st));
    if (h.hashes_out && Ns) RPK_CUDA(cudaMemcpyAsync(h.hashes_out + lo, ds.s_hash_out.p, (size_t)Ns * 8, cudaMemcpyDeviceToHost, st));
    RPK_CUDA(cudaEventRecord(ds.ev[3], st));
}

// after the shard's stream has been synchronised: this shard's part of the caller's arrays (ascending over shards)
uint32_t collect_status_shard(rpk_ctx* ctx, int s, const StatusHostArgs& h, uint32_t out_at) {
    DeviceState& ds = ctx->devs[(size_t)s];
    const ShardPart sp = shard_part(ctx, s, h);
    const uint32_t Ns = sp.p1 - sp.p0, cap = Ns ? Ns : 1;
    if (!h.report || !Ns) return 0;
    const uint32_t cnt = *reinterpret_cast<volatile uint32_t*>(ds.h_changed.h);
    memcpy(h.changed_idx + out_at, ds.h_changed.h + 64, (size_t)cnt * 4);
    if (h.changed_code) memcpy(h.changed_code + out_at, ds.h_changed.h + 64 + (size_t)cap * 4, (size_t)cnt * 2);
    return cnt;
}

// The host calls' shard loop, once their arguments are checked: the pipelined host select (sel), a host sweep (h), or
// both in a tick (tick: the sweep runs on status_stream beside the select, and no timing is reported, since both halves
// record ds.ev).  Every shard first waits for the last device call in the scopes it uses; then the calling thread sizes
// the buffers, every shard enqueues and synchronises on its worker, and the outputs, launches and stats are collected.
// false: a slot id outside the pod table (best and top5 unspecified, stats untouched).
bool run_host(rpk_ctx* ctx, const HostSelect* sel, const StatusHostArgs* h, bool tick) {
    const int n = (int)ctx->devs.size();
    for (auto& ds : ctx->devs) {
        if (sel) ds.sel_scope.host_wait();
        if (h) ds.status_scope.host_wait();
    }
    if (sel) reserve_select(ctx, *sel);
    if (h) for (int s = 0; s < n; ++s) reserve_status_shard(ctx, s, *h);
    std::vector<uint64_t> launches((size_t)n, 0);
    std::vector<float> km((size_t)n, 0.f), tm((size_t)n, 0.f);
    std::vector<char> shard_ok((size_t)n, 1);
    ctx->workers.run(n, [&](int s) {
        DeviceState& ds = ctx->devs[(size_t)s];
        const cudaStream_t sweep = tick ? ds.status_stream : ds.stream;
        // the selection goes first: its kernels are the long pole and start after the first 128k-row sub-batch has
        // landed; in a tick the sweep's records follow on the status stream, concurrent with the lanes, and its kernel
        // runs under the selection's tail
        if (sel) shard_ok[(size_t)s] = enqueue_select_shard(ctx, s, *sel, &launches[(size_t)s]);
        if (h) enqueue_status_shard(ctx, s, *h, sweep, &launches[(size_t)s]);
        if (h) RPK_CUDA(cudaStreamSynchronize(sweep));
        if (sel) RPK_CUDA(cudaStreamSynchronize(ds.stream));
        if (tick) return;
        if (h) RPK_CUDA(cudaEventElapsedTime(&km[(size_t)s], ds.ev[1], ds.ev[2]));
        RPK_CUDA(cudaEventElapsedTime(&tm[(size_t)s], ds.ev[0], ds.ev[3]));
    });
    uint32_t total = 0;
    float kmax = 0.f, tmax = 0.f;
    bool ok = true;
    for (int s = 0; s < n; ++s) {
        if (h) total += collect_status_shard(ctx, s, *h, total);
        ctx->launches += launches[(size_t)s];
        kmax = km[(size_t)s] > kmax ? km[(size_t)s] : kmax; tmax = tm[(size_t)s] > tmax ? tm[(size_t)s] : tmax;
        ok = ok && shard_ok[(size_t)s];
    }
    if (!ok) return false;
    if (sel && !tick) {  // copies and kernels overlap in the pipelined host path: only the total is meaningful
        ctx->stats.last_select_kernel_ms = 0.f; ctx->stats.last_select_total_ms = tmax;
    }
    if (sel) count_select(ctx, sel->P, ctx->devs[0].G);
    if (h) {
        if (h->report) *h->n_changed = total;
        if (!tick) { ctx->stats.last_status_kernel_ms = kmax; ctx->stats.last_status_total_ms = tmax; }
        ctx->stats.status_calls += 1; ctx->stats.status_records += h->slots ? h->n_slots : h->N;
    }
    return true;
}

// rpk_select and rpk_select_slots once their arguments are checked: one GPU and up to kSmallBatch rows take the latency
// path, everything else the sub-batch pipeline on every GPU.  A slot id outside the pod table: RPK_EINVAL (best and
// top5 unspecified, stats untouched).
int select_host(rpk_ctx* ctx, const HostSelect& sel, const char* who) {
    return guarded(ctx, [&]() -> int {
        bool ok;
        if (ctx->devs.size() == 1 && sel.P <= kSmallBatch) {
            ok = sel.src[0].kind != RowSource::HostList || slots_below(sel.src[0].slots, sel.P, ctx->devs[0].podsN);
            if (ok) {
                ctx->launches += (uint64_t)select_small(ctx->devs[0], sel.P, sel.src[0], sel.best, sel.top5);
                ctx->stats.last_select_kernel_ms = 0.f; ctx->stats.last_select_total_ms = 0.f;  // single copy: not timed
                count_select(ctx, sel.P, ctx->devs[0].G);
            }
        } else {
            ok = run_host(ctx, &sel, nullptr, false);
        }
        return ok ? RPK_OK : fail(ctx, RPK_EINVAL, std::string(who) + ": slot index outside the pod table");
    });
}

// RPK_ESTATE unless the tables a select reads exist: the pod table, for rows taken from it, and (needs_offers) the offer
// table, on GPU `shard` or, with -1, on every GPU of the ctx.  The calls that write the pod table check it alone.
int check_select_ready(rpk_ctx* ctx, const char* who, bool needs_pod_table, int shard = -1, bool needs_offers = true) {
    for (size_t s = shard < 0 ? 0 : (size_t)shard, end = shard < 0 ? ctx->devs.size() : s + 1; s < end; ++s) {
        if (needs_pod_table && !ctx->devs[s].pods_sized)
            return fail(ctx, RPK_ESTATE, std::string(who) + (shard < 0 ? ": no pod table" : ": no pod table on this shard") + " (call rpk_pods_reset first)");
        if (needs_offers && !ctx->devs[s].offers_ready) return fail(ctx, RPK_ESTATE, std::string(who) + ": no offer table uploaded (call rpk_offers_upload first)");
    }
    return RPK_OK;
}

// The six rpk_select*_device* calls (`who` names the one called; src is a device list for the rpk_select_slots_device*
// calls): the select of P rows into d_best_full[0, n_out) from row row0 on and into d_top5, or, with gather_top5 (the
// _top5 calls), the select whose top-5 lists are gathered into d_top5_full[0, n_out).  The top-5 call finds its local
// top-5 vector before the other refusals, and an empty one still looks it up.
int select_device(rpk_ctx* ctx, const char* who, int shard, uint32_t P, const RowSource& src, int n_out, int32_t* const* d_best_full,
                  uint32_t row0, int32_t* d_top5, bool gather_top5, int32_t* const* d_top5_full, void* stream) {
    if (!ctx) return RPK_EINVAL;
    const std::string w(who);
    const bool list = src.kind == RowSource::DevList;
    if (bad_shard(ctx, shard)) return fail(ctx, RPK_EINVAL, w + ": shard out of range");
    if (list && P > 0 && !src.slots) return fail(ctx, RPK_EINVAL, w + ": d_slots is required");
    Top5Gather t5{};
    if (gather_top5) {
        if (!d_best_full || !d_top5_full || n_out < 1 || n_out > RPK_MAX_GPUS) return fail(ctx, RPK_EINVAL, w + ": 1..8 best and top-5 vectors are required");
        for (int o = 0; o < n_out; ++o) if (!d_best_full[o] || !d_top5_full[o]) return fail(ctx, RPK_EINVAL, w + ": NULL output vector");
        if ((uint64_t)P * RPK_TOPK > UINT32_MAX) return fail(ctx, RPK_EINVAL, w + ": 5*P does not fit in uint32_t");
        if (!same_phase(n_out, d_top5_full)) return fail(ctx, RPK_EINVAL, w + ": the top-5 vectors differ in 16-byte phase");
        for (int o = 0; o < n_out; ++o) t5.out[o] = d_top5_full[o];
        t5.n_out = n_out;
    }
    const PeerGroup& peers = ctx->bind[(size_t)shard];
    // P = 0: nothing to select, but a bound gather still tells its peers that this (empty) shard is done, after the
    // last gather's epoch counter
    const bool signal = P == 0 && n_out > 1 && peers.n > 0;
    if (P == 0 && !signal && !gather_top5) return RPK_OK;
    return device_call(ctx, shard, stream, P > 0 || signal ? &DeviceState::sel_scope : nullptr,
        [&](DeviceState& ds) -> int {
            if (gather_top5 && (t5.self_out = local_vector(ctx, shard, ds.dev, n_out, d_top5_full)) < 0)
                return fail(ctx, RPK_EINVAL, w + ": no top-5 vector lives on GPU `shard`");
            if (P == 0) return RPK_OK;
            if ((!list && !src.cols.req_mem) || !d_best_full || n_out < 1 || n_out > RPK_MAX_GPUS)
                return fail(ctx, RPK_EINVAL, w + (list ? ": " : ": req_mem_gb and ") + "1..8 output vectors are required");
            for (int o = 0; o < n_out; ++o) if (!d_best_full[o]) return fail(ctx, RPK_EINVAL, w + ": NULL output vector");
            if (int rc = check_select_ready(ctx, who, list, shard)) return rc;
            reserve_lane(ds.dev_lane, P, src, false);
            return RPK_OK;
        },
        [&](DeviceState& ds, cudaStream_t st) {
            if (P == 0) {
                if (signal) ctx->launches += (uint64_t)launch_peer_signal(peers, 0, peers.inline_wait != 0, st);
                return;
            }
            DeviceState::Lane& ln = ds.dev_lane;  // the gather writes the lane's columns: after the last device select
            SelectArgs a{};
            ctx->launches += (uint64_t)pod_columns(ds, ln, src, 0, P, a, st);
            a.P = P;
            for (int o = 0; o < n_out; ++o) a.best_out[o] = d_best_full[o];
            a.n_out = n_out; a.row0 = row0;
            a.top5 = gather_top5 ? t5.out[t5.self_out] + (size_t)RPK_TOPK * row0 : d_top5;
            a.self_out = find_local_vector(ctx, shard, ds.dev, n_out, d_best_full);
            if (n_out > 1) a.peers = peers;
            ctx->launches += (uint64_t)enqueue_select(ds, ln, a, st, gather_top5 ? &t5 : nullptr);
            count_select(ctx, P, ds.G);
        });
}

// rpk_explain and rpk_explain_slots once their arguments are checked (`who` names the one called): every GPU explains
// its contiguous share of the P rows, rpk_select's split, staged in its host lane 0 as a select's rows are, and copies
// the results into out.  A slot list is checked whole before anything is enqueued.  Counts nothing in rpk_stats.
int explain_host(rpk_ctx* ctx, uint32_t P, const RowSource& src, rpk_explanation* out, const char* who) {
    if (src.kind == RowSource::HostList && !slots_below(src.slots, P, ctx->devs[0].podsN))
        return fail(ctx, RPK_EINVAL, std::string(who) + ": slot index outside the pod table");
    return guarded(ctx, [&]() -> int {
        const int n = (int)ctx->devs.size();
        for (int s = 0; s < n; ++s) {  // sized from the calling thread, behind the scope's last device call
            DeviceState& ds = ctx->devs[(size_t)s];
            uint32_t lo, hi; shard_range(P, n, s, &lo, &hi);
            RPK_CUDA(cudaSetDevice(ds.dev));
            ds.sel_scope.host_wait();
            reserve_lane(ds.lane[0], std::max<uint32_t>(hi - lo, 1u), src, false);
            ds.explain_out.reserve(std::max<uint32_t>(hi - lo, 1u));
        }
        std::vector<uint64_t> launches((size_t)n, 0);
        ctx->workers.run(n, [&](int s) {
            DeviceState& ds = ctx->devs[(size_t)s];
            uint32_t lo, hi; shard_range(P, n, s, &lo, &hi);
            if (lo == hi) return;
            RPK_CUDA(cudaSetDevice(ds.dev));
            DeviceState::Lane& ln = ds.lane[0];
            uint32_t at;
            const RowSource dev = upload_rows(ln, src, lo, hi - lo, ln.stream, &at);
            SelectArgs a{};
            launches[(size_t)s] += (uint64_t)pod_columns(ds, ln, dev, at, hi - lo, a, ln.stream);
            ExplainArgs e{};
            e.rows = pod_cols(a); e.P = hi - lo;
            for (int c = 0; c < 2; ++c) { e.wide[c] = ds.v_wide[c].p; e.price[c] = ds.v_price[c].p; }
            e.G = ds.G; e.out = ds.explain_out.p;
            launches[(size_t)s] += (uint64_t)launch_explain(e, ln.stream);
            RPK_CUDA(cudaMemcpyAsync(out + lo, ds.explain_out.p, (size_t)(hi - lo) * sizeof(rpk_explanation), cudaMemcpyDeviceToHost, ln.stream));
            RPK_CUDA(cudaStreamSynchronize(ln.stream));
        });
        for (uint64_t l : launches) ctx->launches += l;
        return RPK_OK;
    });
}

struct SlotRange { uint32_t lo, hi; };

// Columns sharded by slot range move from the old ranges `was` to the new ones `now`.  grow(s) is GPU s's Grow of them (a
// buffer or a PodBufs; a slot is per_slot elements of each column): every slot of was[s] is copied from s's old column
// into the new one of the shard d whose new range holds it, on d's stream (a peer copy between GPUs).  A shard whose
// column is the one it had (same buffer, same first slot) keeps its slots in place; its new range then holds all of
// them, as a range with the same first slot only grows.
template <typename GrowOf>
void move_slots(rpk_ctx* ctx, const std::vector<SlotRange>& was, const std::vector<SlotRange>& now, GrowOf&& grow, size_t per_slot) {
    const size_t n = ctx->devs.size();
    for (size_t d = 0; d < n; ++d) {
        DeviceState& dd = ctx->devs[d];
        RPK_CUDA(cudaSetDevice(dd.dev));
        for (size_t s = 0; s < n; ++s) {
            const uint32_t lo = std::max(was[s].lo, now[d].lo), hi = std::min(was[s].hi, now[d].hi);
            grow(s).each([&](auto& src, auto*, auto& to, auto& to_fresh) {
                auto* dst = to_fresh.p ? to_fresh.p : to.p;
                const size_t bytes = per_slot * sizeof(*dst);
                if (lo >= hi || src.p == dst) return;
                RPK_CUDA(cudaMemcpyPeerAsync(reinterpret_cast<char*>(dst) + (size_t)(lo - now[d].lo) * bytes, dd.dev,
                                             reinterpret_cast<const char*>(src.p) + (size_t)(lo - was[s].lo) * bytes, ctx->devs[s].dev,
                                             (size_t)(hi - lo) * bytes, dd.stream));
            }, *grow(d).b, grow(d).fresh);
        }
    }
}

void sync_all(rpk_ctx* ctx) {
    for (auto& ds : ctx->devs) {
        RPK_CUDA(cudaSetDevice(ds.dev));
        RPK_CUDA(cudaStreamSynchronize(ds.stream));
    }
}

}  // namespace

extern "C" {

int rpk_abi_version(void) { return RPK_ABI_VERSION; }

const char* rpk_last_error(const rpk_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_err.c_str(); }

void* rpk_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
void rpk_host_free(void* p) { if (p) cudaFreeHost(p); }

int rpk_create(int n_gpus, const int* device_ids, rpk_ctx** out) {
    if (!out) return fail(nullptr, RPK_EINVAL, "rpk_create: out is NULL");
    *out = nullptr;
    if (n_gpus < 1 || n_gpus > RPK_MAX_GPUS) return fail(nullptr, RPK_EINVAL, "rpk_create: n_gpus must be in [1, 8]");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        cudaGetLastError();
        return fail(nullptr, RPK_ENODEV, std::string("rpk_create: no CUDA device (") + cudaGetErrorString(e) + "); there is no CPU fallback");
    }
    rpk_ctx* ctx = nullptr;
    try { ctx = new rpk_ctx(n_gpus); } catch (const std::bad_alloc&) { return fail(nullptr, RPK_ENOMEM, "rpk_create: host allocation failed"); }
    memset(&ctx->stats, 0, sizeof(ctx->stats));
    // test hook (several shards of one ctx on one GPU, so that a one-GPU machine runs the sharded host paths): consulted
    // once per ctx, here, and never on a select or sweep path.  Shards that share a device already address each other's
    // memory, so they are neither refused as duplicates nor enabled as peers.
    const char* shared_env = getenv("RPK_TEST_SHARED_DEVICE");
    const bool shared_device = shared_env && !strcmp(shared_env, "1");
    int rc = guarded(nullptr, [&]() -> int {
        for (int i = 0; i < n_gpus; ++i) {
            const int dev = device_ids ? device_ids[i] : i;
            if (dev < 0 || dev >= count) return fail(nullptr, RPK_EINVAL, "rpk_create: device id out of range");
            for (int j = 0; j < i && !shared_device; ++j) if (ctx->devs[(size_t)j].dev == dev) return fail(nullptr, RPK_EINVAL, "rpk_create: duplicate device id");
            cudaDeviceProp prop;
            RPK_CUDA(cudaGetDeviceProperties(&prop, dev));
            if (prop.major != 9 || prop.minor != 0) {
                char buf[160];
                snprintf(buf, sizeof(buf), "rpk_create: device %d is sm_%d%d; this library holds sm_90a code only and has no fallback", dev, prop.major, prop.minor);
                return fail(nullptr, RPK_ENODEV, buf);
            }
            DeviceState& ds = ctx->devs[(size_t)i];
            ds.dev = dev; ds.sm_count = prop.multiProcessorCount;
            RPK_CUDA(cudaSetDevice(dev));
            // the selection is the latency-critical half of a tick, the sweep is background work: when both have CTAs
            // pending, the block scheduler places the selection's first
            int prio_lo = 0, prio_hi = 0;
            RPK_CUDA(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
            RPK_CUDA(cudaStreamCreateWithPriority(&ds.stream, cudaStreamNonBlocking, prio_hi));
            RPK_CUDA(cudaStreamCreateWithPriority(&ds.status_stream, cudaStreamNonBlocking, prio_lo));
            RPK_CUDA(cudaStreamCreateWithPriority(&ds.pending_stream, cudaStreamNonBlocking, prio_lo));
            for (auto& ev : ds.ev) RPK_CUDA(cudaEventCreate(&ev));
            RPK_CUDA(cudaEventCreateWithFlags(&ds.sel_scope.ev, cudaEventDisableTiming));
            RPK_CUDA(cudaEventCreateWithFlags(&ds.status_scope.ev, cudaEventDisableTiming));
            for (auto& ln : ds.lane) {
                RPK_CUDA(cudaStreamCreateWithPriority(&ln.stream, cudaStreamNonBlocking, prio_hi));
                RPK_CUDA(cudaEventCreateWithFlags(&ln.done, cudaEventDisableTiming));
            }
        }
        for (int i = 0; i < n_gpus && n_gpus > 1; ++i) {
            RPK_CUDA(cudaSetDevice(ctx->devs[(size_t)i].dev));
            for (int j = 0; j < n_gpus; ++j) {
                if (ctx->devs[(size_t)i].dev == ctx->devs[(size_t)j].dev) continue;  // itself, or a shard on the same GPU
                int can = 0;
                RPK_CUDA(cudaDeviceCanAccessPeer(&can, ctx->devs[(size_t)i].dev, ctx->devs[(size_t)j].dev));
                if (!can) return fail(nullptr, RPK_ENODEV, "rpk_create: GPUs of the ctx cannot access each other (NVLink/P2P required for n_gpus > 1)");
                cudaError_t pe = cudaDeviceEnablePeerAccess(ctx->devs[(size_t)j].dev, 0);
                if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) RPK_CUDA(pe);
                cudaGetLastError();
            }
        }
        ctx->stats.n_gpus = (uint32_t)n_gpus;
        ctx->workers.start(n_gpus);
        return RPK_OK;
    });
    if (rc != RPK_OK) { rpk_destroy(ctx); return rc; }
    *out = ctx;
    return RPK_OK;
}

void rpk_destroy(rpk_ctx* ctx) {
    if (!ctx) return;
    ctx->workers.stop();
    for (auto& m : ctx->ipc_mapped) if (cudaSetDevice(ctx->devs[(size_t)m.first].dev) == cudaSuccess) cudaIpcCloseMemHandle(m.second);
    for (auto& m : ctx->ipc_owned) if (cudaSetDevice(ctx->devs[(size_t)m.first].dev) == cudaSuccess) { cudaDeviceSynchronize(); cudaFree(m.second); }
    delete ctx;  // every DeviceState synchronises its streams and frees what it holds
    cudaGetLastError();
}

namespace {
// Every stored pending result is stale from here on: a new generation becomes the floor and the window is cleared.
// After 2^32 generations they start over, and so do the stored results.
void invalidate_results(rpk_ctx* ctx) {
    if (++ctx->offer_gen == 0) {
        ctx->offer_gen = 1;
        for (auto& ds : ctx->devs) ds.res_ready = false;
    }
    ctx->offer_floor = ctx->offer_gen;
    ctx->window.clear();
}

// The changed offers the refresh's diffs listed (each GPU diffed its own replica) join the window at a new generation,
// newest first, and the window goes to every GPU.  Returns the number of changed offers, or UINT32_MAX after a wholesale
// invalidation: too many changes for the window.
uint32_t merge_window(rpk_ctx* ctx) {
    std::vector<uint32_t> changed;
    for (auto& ds : ctx->devs) {
        const volatile uint32_t* o = reinterpret_cast<const volatile uint32_t*>(ds.h_delta.h);
        const uint32_t n = o[0];
        if (n > RPK_OFFERS_DELTA_MAX) { invalidate_results(ctx); return UINT32_MAX; }
        for (uint32_t k = 0; k < n; ++k) changed.push_back((uint32_t)o[1 + k]);
    }
    std::sort(changed.begin(), changed.end());
    changed.erase(std::unique(changed.begin(), changed.end()), changed.end());
    if (changed.empty()) return 0;
    const uint32_t gen = ctx->offer_gen + 1;
    if (gen == 0) { invalidate_results(ctx); return UINT32_MAX; }
    std::vector<uint2> w;
    for (uint32_t c : changed) w.push_back(make_uint2(c, gen));
    for (const uint2& e : ctx->window)
        if (!std::binary_search(changed.begin(), changed.end(), e.x)) w.push_back(e);
    if (w.size() > RPK_OFFERS_DELTA_MAX) { invalidate_results(ctx); return UINT32_MAX; }
    ctx->offer_gen = gen;
    ctx->window.swap(w);
    for (auto& ds : ctx->devs) {  // on the GPU's stream, finished before the call returns: every reader comes later
        RPK_CUDA(cudaSetDevice(ds.dev));
        ds.win.reserve(RPK_OFFERS_DELTA_MAX);
        RPK_CUDA(cudaMemcpyAsync(ds.win.p, ctx->window.data(), ctx->window.size() * sizeof(uint2), cudaMemcpyHostToDevice, ds.stream));
        RPK_CUDA(cudaStreamSynchronize(ds.stream));
    }
    return (uint32_t)changed.size();
}

// rpk_offers_upload (refresh false) and rpk_offers_refresh: one ingest.  A refresh of a table with the resident G
// uploads the new columns next to the resident ones, diffs the two and installs the new ones; everything else is the
// upload, which invalidates the stored results wholesale.
int install_offers(rpk_ctx* ctx, const char* who, bool refresh, uint32_t G, const int32_t* mem_gb, const int32_t* vcpu,
                   const int32_t* ram_gb, const double* secure_price, const double* community_price, const uint8_t* flags,
                   uint32_t* n_offers_changed) {
    if (!ctx) return RPK_EINVAL;
    if (G > 0 && (!mem_gb || !secure_price || !community_price || !flags))
        return fail(ctx, RPK_EINVAL, std::string(who) + ": mem_gb, secure_price, community_price and flags are required");
    if (G > (1u << 26)) return fail(ctx, RPK_EINVAL, std::string(who) + ": G above 2^26 offers is not supported");
    if (has_int32_max(mem_gb, G) || has_int32_max(vcpu, G) || has_int32_max(ram_gb, G))
        return fail(ctx, RPK_EINVAL, std::string(who) + ": offer columns must be < INT32_MAX (requests saturate there)");
    const OfferIngest host{G, mem_gb, vcpu, ram_gb, secure_price, community_price, flags};
    bool diff = refresh;
    for (const auto& ds : ctx->devs) diff = diff && ds.offers_ready && ds.G == G;
    if (!diff) invalidate_results(ctx);
    uint32_t changed = UINT32_MAX;
    const int rc = guarded(ctx, [&]() -> int {
        for (auto& ds : ctx->devs) {
            RPK_CUDA(cudaSetDevice(ds.dev));
            ds.sel_scope.host_wait();  // a device select may still read the views rewritten below
            ds.offers_ready = false;
            ds.force_kind = 0;
            // test hook (exercise every kernel on any table): consulted once per table upload, never on the select path
            if (const char* fk = getenv("RPK_FORCE_KERNEL")) {
                if (!strcmp(fk, "generic")) ds.force_kind = 1; else if (!strcmp(fk, "packed")) ds.force_kind = 2;
                else if (!strcmp(fk, "packed_pos")) ds.force_kind = 3; else if (!strcmp(fk, "bitmap")) ds.force_kind = 4;
                else if (!strcmp(fk, "bitmap_grouped")) ds.force_kind = 5;  // every batch size through the persistent kernel
                else if (!strcmp(fk, "bitmap_price")) ds.force_kind = 6;    // ... through the persistent kernel, table staged by price
            }
            OfferBufs& c = diff ? ds.raw_next : ds.raw;  // after the diff, raw_next becomes raw
            OfferBufs::each(c, [G](auto& b) { b.reserve(G ? G : 1); });
            if (G) OfferBufs::each(c, [&](auto& b, const auto* col) {  // the caller's columns; vcpu and ram: zeros when not passed
                if (col) RPK_CUDA(cudaMemcpyAsync(b.p, col, (size_t)G * sizeof(*col), cudaMemcpyHostToDevice, ds.stream));
                else RPK_CUDA(cudaMemsetAsync(b.p, 0, (size_t)G * sizeof(*col), ds.stream));
            }, host);
            if (diff) {
                if (!ds.delta_state.p) {  // zero between calls: the diff's last CTA clears it again
                    ds.delta_state.reserve(2); ds.delta_idx.reserve(RPK_OFFERS_DELTA_MAX);
                    RPK_CUDA(cudaMemsetAsync(ds.delta_state.p, 0, ds.delta_state.cap * sizeof(uint32_t), ds.stream));
                }
                ds.h_delta.reserve(4 * (1 + RPK_OFFERS_DELTA_MAX));
                *reinterpret_cast<volatile uint32_t*>(ds.h_delta.h) = 0u;
                const OfferDiffArgs da{ds.raw.view(G), c.view(G), ds.delta_state.p, ds.delta_idx.p, reinterpret_cast<uint32_t*>(ds.h_delta.d)};
                ctx->launches += (uint64_t)launch_offer_diff(da, ds.stream);
                ds.raw.swap(ds.raw_next);
            }
            ctx->launches += (uint64_t)launch_offer_ingest(ds, ds.raw.view(G), ds.stream);
            RPK_CUDA(cudaStreamSynchronize(ds.stream));
        }
        if (diff) changed = merge_window(ctx);
        const DeviceState& d0 = ctx->devs[0];
        ctx->stats.select_kernel_kind = d0.pk.bm_words ? 4u : d0.pk.bits ? (d0.pk.pos_bits ? 3u : 2u) : 1u;
        ctx->stats.distinct_mem = d0.D[0]; ctx->stats.distinct_vcpu = d0.D[1]; ctx->stats.distinct_ram = d0.D[2];
        ctx->stats.packed_bits = d0.pk.bits;
        return RPK_OK;
    });
    if (rc != RPK_OK && diff) invalidate_results(ctx);  // the table may be half new
    if (rc == RPK_OK && n_offers_changed) *n_offers_changed = changed;
    return rc;
}
}  // namespace

int rpk_offers_upload(rpk_ctx* ctx, uint32_t G, const int32_t* mem_gb, const int32_t* vcpu, const int32_t* ram_gb,
                      const double* secure_price, const double* community_price, const uint8_t* flags) {
    return install_offers(ctx, "rpk_offers_upload", false, G, mem_gb, vcpu, ram_gb, secure_price, community_price, flags, nullptr);
}

int rpk_offers_refresh(rpk_ctx* ctx, uint32_t G, const int32_t* mem_gb, const int32_t* vcpu, const int32_t* ram_gb,
                       const double* secure_price, const double* community_price, const uint8_t* flags,
                       uint32_t* n_offers_changed) {
    return install_offers(ctx, "rpk_offers_refresh", true, G, mem_gb, vcpu, ram_gb, secure_price, community_price, flags,
                          n_offers_changed);
}

int rpk_select_device_gather(rpk_ctx* ctx, int shard, uint32_t P, const int32_t* d_req_mem_gb, const int32_t* d_req_vcpu,
                             const int32_t* d_req_ram_gb, const double* d_max_price, const uint8_t* d_cloud,
                             int n_out, int32_t* const* d_best_full, uint32_t row0, int32_t* d_top5, void* stream) {
    const RowSource src{RowSource::DevCols, PodCols{d_req_mem_gb, d_req_vcpu, d_req_ram_gb, d_max_price, d_cloud}, nullptr};
    return select_device(ctx, "rpk_select_device_gather", shard, P, src, n_out, d_best_full, row0, d_top5, false, nullptr, stream);
}

int rpk_select_device_gather_top5(rpk_ctx* ctx, int shard, uint32_t P, const int32_t* d_req_mem_gb, const int32_t* d_req_vcpu,
                                  const int32_t* d_req_ram_gb, const double* d_max_price, const uint8_t* d_cloud, int n_out,
                                  int32_t* const* d_best_full, int32_t* const* d_top5_full, uint32_t row0, void* stream) {
    const RowSource src{RowSource::DevCols, PodCols{d_req_mem_gb, d_req_vcpu, d_req_ram_gb, d_max_price, d_cloud}, nullptr};
    return select_device(ctx, "rpk_select_device_gather_top5", shard, P, src, n_out, d_best_full, row0, nullptr, true, d_top5_full, stream);
}

int rpk_select_device(rpk_ctx* ctx, int shard, uint32_t P, const int32_t* d_req_mem_gb, const int32_t* d_req_vcpu,
                      const int32_t* d_req_ram_gb, const double* d_max_price, const uint8_t* d_cloud, int32_t* d_best,
                      int32_t* d_top5, void* stream) {
    int32_t* outs[1] = {d_best};
    const RowSource src{RowSource::DevCols, PodCols{d_req_mem_gb, d_req_vcpu, d_req_ram_gb, d_max_price, d_cloud}, nullptr};
    return select_device(ctx, "rpk_select_device", shard, P, src, 1, outs, 0, d_top5, false, nullptr, stream);
}

int rpk_select(rpk_ctx* ctx, uint32_t P, const int32_t* req_mem_gb, const int32_t* req_vcpu, const int32_t* req_ram_gb,
               const double* max_price, const uint8_t* cloud, int32_t* best, int32_t* top5) {
    if (!ctx) return RPK_EINVAL;
    if (P == 0) return RPK_OK;
    if (!req_mem_gb || !best) return fail(ctx, RPK_EINVAL, "rpk_select: req_mem_gb and best are required");
    if (int rc = check_select_ready(ctx, "rpk_select", false)) return rc;
    const RowSource rows{RowSource::HostCols, PodCols{req_mem_gb, req_vcpu, req_ram_gb, max_price, cloud}, nullptr};
    return select_host(ctx, HostSelect{P, std::vector<RowSource>(ctx->devs.size(), rows), best, top5}, "rpk_select");
}

// ---- pod-requirement table -------------------------------------------------------------------------------

int rpk_pods_reset(rpk_ctx* ctx, uint32_t N) {
    if (!ctx) return RPK_EINVAL;
    for (auto& ds : ctx->devs) ds.pods_sized = ds.res_ready = ds.res_bound = false;  // a failure below leaves no table rather than a mix of sizes
    return guarded(ctx, [&]() -> int {
        for (auto& ds : ctx->devs) {
            RPK_CUDA(cudaSetDevice(ds.dev));
            ds.sel_scope.host_wait();  // a device select may still gather from the table
            const size_t cap = N ? N : 1;
            ds.pt_cols.reserve(cap);
            ds.pt_pending.reserve(cap);
            ctx->launches += (uint64_t)launch_pod_fill(ds.pods_table(), ds.pt_pending.p, N, ds.sm_count, ds.stream);
            RPK_CUDA(cudaStreamSynchronize(ds.stream));
            ds.podsN = N;
        }
        for (auto& ds : ctx->devs) ds.pods_sized = true;
        return RPK_OK;
    });
}

// slots[0, n) inside `table` (of N rows; "pod table" or "tracked table" in the message) and, with `ascending`, strictly
// ascending: what the calls that write a table require
static int check_slots(rpk_ctx* ctx, uint32_t n, const uint32_t* slots, uint32_t N, bool ascending, const char* who, const char* table) {
    for (uint32_t i = 0; i < n; ++i) {
        if (slots[i] >= N) return fail(ctx, RPK_EINVAL, std::string(who) + ": slot index outside the " + table);
        if (ascending && i > 0 && slots[i] <= slots[i - 1]) return fail(ctx, RPK_EINVAL, std::string(who) + ": slots must be strictly ascending");
    }
    return RPK_OK;
}

int rpk_pods_seed_slots(rpk_ctx* ctx, uint32_t n_slots, const uint32_t* slots, const int32_t* req_mem_gb, const int32_t* req_vcpu,
                        const int32_t* req_ram_gb, const double* max_price, const uint8_t* cloud) {
    if (!ctx) return RPK_EINVAL;
    if (n_slots == 0) return RPK_OK;
    if (!slots || !req_mem_gb) return fail(ctx, RPK_EINVAL, "rpk_pods_seed_slots: slots and req_mem_gb are required");
    if (int rc = check_select_ready(ctx, "rpk_pods_seed_slots", true, -1, false)) return rc;
    if (int rc = check_slots(ctx, n_slots, slots, ctx->devs[0].podsN, true, "rpk_pods_seed_slots", "pod table")) return rc;
    return guarded(ctx, [&]() -> int {
        // staging block: [slots : 4n], then the rows
        const size_t n = n_slots;
        const PodBlock blk = pod_block(n, 4 * n);
        for (auto& ds : ctx->devs) {  // the table is replicated: every GPU gets every row
            RPK_CUDA(cudaSetDevice(ds.dev));
            ds.sel_scope.host_wait();  // after a device select's gather
            ds.pt_seed.reserve(blk.end);
            unsigned char* d = ds.pt_seed.p;
            const auto up = [&](const auto* col, size_t o) { RPK_CUDA(cudaMemcpyAsync(d + o, col, n * sizeof(*col), cudaMemcpyHostToDevice, ds.stream)); return d + o; };
            const uint32_t* d_slots = (const uint32_t*)up(slots, 0);
            const PodCols in = to_device(PodCols{req_mem_gb, req_vcpu, req_ram_gb, max_price, cloud}, blk, up);
            ctx->launches += (uint64_t)launch_pod_seed(ds.pods_table(), ds.podsN, n_slots, d_slots, in, ds.stream);
            RPK_CUDA(cudaStreamSynchronize(ds.stream));
        }
        return RPK_OK;
    });
}

int rpk_select_slots(rpk_ctx* ctx, uint32_t n_slots, const uint32_t* slots, int32_t* best, int32_t* top5) {
    if (!ctx) return RPK_EINVAL;
    if (n_slots == 0) return RPK_OK;
    if (!slots || !best) return fail(ctx, RPK_EINVAL, "rpk_select_slots: slots and best are required");
    if (int rc = check_select_ready(ctx, "rpk_select_slots", true)) return rc;
    const std::vector<RowSource> rows(ctx->devs.size(), RowSource{RowSource::HostList, PodCols{}, slots});
    return select_host(ctx, HostSelect{n_slots, rows, best, top5}, "rpk_select_slots");
}

int rpk_explain(rpk_ctx* ctx, uint32_t P, const int32_t* req_mem_gb, const int32_t* req_vcpu, const int32_t* req_ram_gb,
                const double* max_price, const uint8_t* cloud, rpk_explanation* out) {
    if (!ctx) return RPK_EINVAL;
    if (P == 0) return RPK_OK;
    if (!req_mem_gb || !out) return fail(ctx, RPK_EINVAL, "rpk_explain: req_mem_gb and out are required");
    if (int rc = check_select_ready(ctx, "rpk_explain", false)) return rc;
    const RowSource rows{RowSource::HostCols, PodCols{req_mem_gb, req_vcpu, req_ram_gb, max_price, cloud}, nullptr};
    return explain_host(ctx, P, rows, out, "rpk_explain");
}

int rpk_explain_slots(rpk_ctx* ctx, uint32_t n_slots, const uint32_t* slots, rpk_explanation* out) {
    if (!ctx) return RPK_EINVAL;
    if (n_slots == 0) return RPK_OK;
    if (!slots || !out) return fail(ctx, RPK_EINVAL, "rpk_explain_slots: slots and out are required");
    if (int rc = check_select_ready(ctx, "rpk_explain_slots", true)) return rc;
    return explain_host(ctx, n_slots, RowSource{RowSource::HostList, PodCols{}, slots}, out, "rpk_explain_slots");
}

int rpk_select_slots_device_gather(rpk_ctx* ctx, int shard, uint32_t n_slots, const uint32_t* d_slots, int n_out,
                                   int32_t* const* d_best_full, uint32_t row0, int32_t* d_top5, void* stream) {
    const RowSource src{RowSource::DevList, PodCols{}, d_slots};
    return select_device(ctx, "rpk_select_slots_device_gather", shard, n_slots, src, n_out, d_best_full, row0, d_top5, false, nullptr, stream);
}

int rpk_select_slots_device_gather_top5(rpk_ctx* ctx, int shard, uint32_t n_slots, const uint32_t* d_slots, int n_out,
                                        int32_t* const* d_best_full, int32_t* const* d_top5_full, uint32_t row0, void* stream) {
    const RowSource src{RowSource::DevList, PodCols{}, d_slots};
    return select_device(ctx, "rpk_select_slots_device_gather_top5", shard, n_slots, src, n_out, d_best_full, row0, nullptr, true, d_top5_full, stream);
}

int rpk_select_slots_device(rpk_ctx* ctx, int shard, uint32_t n_slots, const uint32_t* d_slots, int32_t* d_best, int32_t* d_top5,
                            void* stream) {
    int32_t* outs[1] = {d_best};
    const RowSource src{RowSource::DevList, PodCols{}, d_slots};
    return select_device(ctx, "rpk_select_slots_device", shard, n_slots, src, 1, outs, 0, d_top5, false, nullptr, stream);
}

// ---- pending set of the pod table ---------------------------------------------------------------------------

int rpk_pods_mark_pending(rpk_ctx* ctx, uint32_t n_slots, const uint32_t* slots, const uint8_t* pending) {
    if (!ctx) return RPK_EINVAL;
    if (n_slots == 0) return RPK_OK;
    if (!slots || !pending) return fail(ctx, RPK_EINVAL, "rpk_pods_mark_pending: slots and pending are required");
    if (int rc = check_select_ready(ctx, "rpk_pods_mark_pending", true, -1, false)) return rc;
    if (int rc = check_slots(ctx, n_slots, slots, ctx->devs[0].podsN, true, "rpk_pods_mark_pending", "pod table")) return rc;
    return guarded(ctx, [&]() -> int {
        const size_t n = n_slots;  // staging block: [slots : 4n][pending : n]
        for (auto& ds : ctx->devs) {  // the table is replicated: every GPU gets every flag
            RPK_CUDA(cudaSetDevice(ds.dev));
            ds.sel_scope.host_wait();  // after a device call's pending list
            ds.pt_seed.reserve(5 * n);
            RPK_CUDA(cudaMemcpyAsync(ds.pt_seed.p, slots, 4 * n, cudaMemcpyHostToDevice, ds.stream));
            RPK_CUDA(cudaMemcpyAsync(ds.pt_seed.p + 4 * n, pending, n, cudaMemcpyHostToDevice, ds.stream));
            ctx->launches += (uint64_t)launch_pod_mark(ds.pt_pending.p, ds.podsN, n_slots, (const uint32_t*)ds.pt_seed.p, ds.pt_seed.p + 4 * n, ds.stream);
            RPK_CUDA(cudaStreamSynchronize(ds.stream));
        }
        return RPK_OK;
    });
}

namespace {
// The look-back state and tickets of the pod table's compactions (k_pod_pending, k_pod_stale, k_pod_result_diff: select
// scope, so never two at once): zero between calls by construction (each kernel's last CTA), zeroed when allocated
void reserve_compaction_state(DeviceState& ds) {
    const size_t need = pending_state_words(ds.sm_count);
    if (need > ds.pt_state.cap || !ds.pt_ticket.p) {
        ds.pt_state.reserve(need); ds.pt_ticket.reserve(3);
        RPK_CUDA(cudaMemset(ds.pt_state.p, 0, ds.pt_state.cap * sizeof(unsigned long long)));
        RPK_CUDA(cudaMemset(ds.pt_ticket.p, 0, ds.pt_ticket.cap * sizeof(uint32_t)));
        RPK_CUDA(cudaDeviceSynchronize());
    }
}

// k_pod_pending on ds over its replica of the flags: the list into d_out (capacity podsN), its length into d_n
int enqueue_pending_list(DeviceState& ds, uint32_t* d_out, uint32_t* d_n, cudaStream_t st) {
    reserve_compaction_state(ds);
    const PendingArgs a{ds.pt_pending.p, ds.podsN, d_out, d_n, ds.pt_state.p, ds.pt_ticket.p};
    return launch_pod_pending(a, ds.sm_count, st);
}
}  // namespace

int rpk_pods_pending_list_device(rpk_ctx* ctx, int shard, uint32_t* d_slots_out, uint32_t* d_n, void* stream) {
    if (!ctx) return RPK_EINVAL;
    if (bad_shard(ctx, shard)) return fail(ctx, RPK_EINVAL, "rpk_pods_pending_list_device: shard out of range");
    if (int rc = check_select_ready(ctx, "rpk_pods_pending_list_device", true, shard, false)) return rc;
    DeviceState& ds = ctx->devs[(size_t)shard];
    if (!d_n || (ds.podsN > 0 && !d_slots_out)) return fail(ctx, RPK_EINVAL, "rpk_pods_pending_list_device: d_slots_out and d_n are required");
    // the look-back state is the shard's: after the last list
    return device_call(ctx, shard, stream, &DeviceState::sel_scope, [&](DeviceState&, cudaStream_t st) {
        ctx->launches += (uint64_t)enqueue_pending_list(ds, d_slots_out, d_n, st);
    });
}

int rpk_select_pending(rpk_ctx* ctx, uint32_t cap, uint32_t* slots_out, uint32_t* n_pending, int32_t* best, int32_t* top5) {
    if (!ctx) return RPK_EINVAL;
    if (!n_pending || (cap > 0 && !best)) return fail(ctx, RPK_EINVAL, "rpk_select_pending: n_pending and best are required");
    if (int rc = check_select_ready(ctx, "rpk_select_pending", true)) return rc;
    // every GPU compacts its own replica of the flags: the table is replicated and the order ascending, so the lists are
    // identical, and each GPU then gathers its shard of the rows from its own copy.  The count lands in mapped pinned
    // memory, so the one synchronise that the list's length costs needs no copy behind it.
    uint32_t n = 0;
    int rc = guarded(ctx, [&]() -> int {
        for (auto& ds : ctx->devs) {
            RPK_CUDA(cudaSetDevice(ds.dev));
            ds.sel_scope.host_wait();
            ds.pt_list.reserve(ds.podsN ? ds.podsN : 1);
            ds.h_pending.reserve(64);
            ctx->launches += (uint64_t)enqueue_pending_list(ds, ds.pt_list.p, reinterpret_cast<uint32_t*>(ds.h_pending.d), ds.stream);
        }
        for (auto& ds : ctx->devs) {
            RPK_CUDA(cudaSetDevice(ds.dev));
            RPK_CUDA(cudaStreamSynchronize(ds.stream));
        }
        n = *reinterpret_cast<volatile uint32_t*>(ctx->devs[0].h_pending.h);
        return RPK_OK;
    });
    if (rc != RPK_OK) return rc;
    *n_pending = n;
    if (n > cap) return fail(ctx, RPK_EINVAL, "rpk_select_pending: more slots pending than cap");
    if (n == 0) return RPK_OK;
    DeviceState& d0 = ctx->devs[0];
    if (slots_out) {  // the list goes back on a stream of its own while the select runs
        rc = guarded(ctx, [&]() -> int {
            RPK_CUDA(cudaSetDevice(d0.dev));
            RPK_CUDA(cudaMemcpyAsync(slots_out, d0.pt_list.p, (size_t)n * 4, cudaMemcpyDeviceToHost, d0.pending_stream));
            return RPK_OK;
        });
        if (rc != RPK_OK) return rc;
    }
    HostSelect sel{n, {}, best, top5};
    for (auto& ds : ctx->devs) sel.src.push_back(RowSource{RowSource::DevList, PodCols{}, ds.pt_list.p});
    rc = select_host(ctx, sel, "rpk_select_pending");
    if (slots_out) {
        const int rc2 = guarded(ctx, [&]() -> int {
            RPK_CUDA(cudaSetDevice(d0.dev));
            RPK_CUDA(cudaStreamSynchronize(d0.pending_stream));
            return RPK_OK;
        });
        if (rc == RPK_OK) rc = rc2;
    }
    return rc;
}

// ---- pending results ----------------------------------------------------------------------------------------

namespace {
// The slots GPU s of n owns in the stored results: its share of the table's 16-slot units (k_pod_stale's unit)
void result_range(uint32_t N, int n, int s, uint32_t* lo, uint32_t* hi) {
    const uint32_t units = (uint32_t)(((uint64_t)N + 15) / 16);
    uint32_t ulo, uhi;
    shard_range(units, n, s, &ulo, &uhi);
    *lo = (uint32_t)std::min<uint64_t>((uint64_t)ulo * 16, N);
    *hi = (uint32_t)std::min<uint64_t>((uint64_t)uhi * 16, N);
}

// The stored results of ds's owned slots [lo, hi), allocated on the first call after a reset with every generation 0
// (nothing reported), and the scratch and mapped output of a call that reselects all of them.  The owned range is fixed
// until the next reset (check_results_range) or grow, so no other call grows r_lane.  [lo, hi) is range my_rank of
// n_ranks (result_range).  The caller has waited.
void reserve_results(DeviceState& ds, uint32_t lo, uint32_t hi, int n_ranks, int my_rank) {
    if (ds.res_ready) return;
    const size_t n = ((size_t)(hi - lo) + 15) / 16 * 16 + 16;  // whole units: k_pod_stale loads 16 slots at a time
    ds.r_cols.reserve(n);
    ds.r_gen.reserve(n); ds.r_top5.reserve(n * RPK_TOPK); ds.r_list.reserve(n); ds.r_mask.reserve(n / 16 + 1); ds.r_dn.reserve(2);
    reserve_lane(ds.r_lane, std::max<uint32_t>(hi - lo, 1u), RowSource{RowSource::DevList, PodCols{}, ds.r_list.p}, true);
    ds.r_out.reserve(n * (2 + RPK_TOPK)); ds.h_res.reserve(64 + ds.r_out.cap * 4);  // result_rows: the same layout
    RPK_CUDA(cudaMemset(ds.r_gen.p, 0, ds.r_gen.cap * sizeof(uint32_t)));
    RPK_CUDA(cudaDeviceSynchronize());
    ds.res_ready = true;
    ds.res_bound = true; ds.res_lo = lo; ds.res_hi = hi; ds.res_ranks = n_ranks; ds.res_rank = my_rank;
}

// RPK_ESTATE when ds's stored results were made for another owned range than [lo, hi) since the last rpk_pods_reset:
// their offsets, and possibly their size, belong to that range
int check_results_range(rpk_ctx* ctx, const DeviceState& ds, uint32_t lo, uint32_t hi, const char* who) {
    if (!ds.res_bound || (ds.res_lo == lo && ds.res_hi == hi)) return RPK_OK;
    return fail(ctx, RPK_ESTATE, std::string(who) + ": the stored results of this GPU were made for another slot range (call rpk_pods_reset first)");
}

// The counts in mapped memory (the device's view with d = true): [n_pending, n_reselected] as the stale step left them
// in r_dn, then the diff's count of changed rows.  The changed rows: in r_out (d = true), or their host copy in h_res
// (false).  The rows go back in three copies of the length the count says: written to mapped memory straight from the
// kernel, row by row, they cost 9 ms at 1M changed rows on an H100 (4- and 20-byte PCIe writes).
struct ResultRows { uint32_t* counts; uint32_t* slot; int32_t* best; int32_t* top5; };
ResultRows result_rows(DeviceState& ds, bool d) {
    const size_t cap = ds.r_out.cap / (2 + RPK_TOPK);
    uint32_t* counts = reinterpret_cast<uint32_t*>(d ? ds.h_res.d : ds.h_res.h);
    int32_t* b = d ? ds.r_out.p : reinterpret_cast<int32_t*>(ds.h_res.h + 64);
    return ResultRows{counts, reinterpret_cast<uint32_t*>(b), b + cap, b + 2 * cap};
}

// The stale step of ds over its owned slots [lo, hi): k_pod_stale lists the stale pending slots in r_list and writes
// [n_pending, n_reselected] to r_dn (zeroed here for an empty range, where nothing is launched).  While the ctx's change
// window is not empty, k_pod_stale_reach takes k_pod_stale's place.  The caller has reserved the results and waited for
// the select scope.  Returns the kernels launched.
int enqueue_stale(const rpk_ctx* ctx, DeviceState& ds, uint32_t lo, uint32_t hi, cudaStream_t st) {
    if (hi == lo) {
        RPK_CUDA(cudaMemsetAsync(ds.r_dn.p, 0, 2 * sizeof(uint32_t), st));
        return 0;
    }
    StaleArgs a{};
    a.flags = ds.pt_pending.p; a.t = ds.pods_table(); a.N = ds.podsN; a.u_lo = lo / 16; a.r = ds.results(); a.gen = ctx->offer_gen;
    a.mask = ds.r_mask.p; a.out = ds.r_list.p; a.n_out = ds.r_dn.p + 1; a.n_pending = ds.r_dn.p;
    a.tile_state = ds.pt_state.p; a.ticket = ds.pt_ticket.p;
    if (ctx->window.empty()) return launch_pod_stale(a, (hi - lo + 15) / 16, ds.sm_count, st);
    const OfferIngest o = ds.raw.view(ds.G);
    const StaleReachArgs x{a, ctx->offer_floor, ds.win.p, (uint32_t)ctx->window.size(),
                           o.mem, o.vcpu, o.ram, o.secure_price, o.community_price, o.flags};
    return launch_pod_stale_reach(x, (hi - lo + 15) / 16, ds.sm_count, st);
}

// The host-sync forms' read of the stale step's counts: r_dn is copied into the mapped block behind it, and read there
// once st has been synchronised
void copy_stale_counts(DeviceState& ds, cudaStream_t st) {
    RPK_CUDA(cudaMemcpyAsync(result_rows(ds, false).counts, ds.r_dn.p, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
}

// The reselect of the rows enqueue_stale listed, whose number the kernels read from r_dn on the device, sized for n_max
// rows: the count the host read (host_count), or the owned range's worst case.  k_pod_reselect_top5 writes their
// columns and top-5 lists to r_lane (and r_dn to d_counts, if not null); the diff stores each row's result and writes
// the changed rows where x says (x.d is filled here).  With a host count of 0 only the diff runs, which still publishes
// the count 0 and signals.  Returns the kernels launched.
int enqueue_reselect(DeviceState& ds, uint32_t n_max, bool host_count, uint32_t lo, uint32_t gen, ResultXchgArgs& x,
                     uint32_t* d_counts, cudaStream_t st) {
    const DeviceState::Lane& ln = ds.r_lane;
    const PodRows cols = ln.cols.rows();
    int launches = 0;
    if (n_max || !host_count) {
        ReselectArgs r{};
        offer_args(ds, r.s);
        r.s.top5 = ln.top5.p;
        r.t = ds.pods_table(); r.out = cols;
        r.list = ds.r_list.p; r.dn = ds.r_dn.p; r.counts = d_counts;
        launches += launch_pod_reselect(r, n_max, ds.sm_count, st);
    }
    ResultDiffArgs& d = x.d;
    d.list = ds.r_list.p; d.cols = cols; d.top5 = ln.top5.p;
    d.r = ds.results(); d.r_lo = lo; d.gen = gen; d.mask = ds.r_mask.p;
    d.tile_state = ds.pt_state.p; d.ticket = ds.pt_ticket.p;
    return launches + launch_pod_result_xchg(x, ds.r_dn.p + 1, n_max, ds.sm_count, st);
}
}  // namespace

int rpk_select_pending_changed(rpk_ctx* ctx, uint32_t cap, uint32_t* n_pending, uint32_t* n_reselected, uint32_t* slots_out,
                               int32_t* best, int32_t* top5, uint32_t* n_changed) {
    if (!ctx) return RPK_EINVAL;
    if (!n_pending || !n_reselected || !n_changed || (cap > 0 && (!slots_out || !best || !top5)))
        return fail(ctx, RPK_EINVAL, "rpk_select_pending_changed: n_pending, n_reselected, n_changed and, with cap > 0, slots_out, best and top5 are required");
    if (int rc = check_select_ready(ctx, "rpk_select_pending_changed", true)) return rc;
    const int n = (int)ctx->devs.size();
    const uint32_t N = ctx->devs[0].podsN, gen = ctx->offer_gen;
    for (int s = 0; s < n; ++s) {
        uint32_t lo, hi; result_range(N, n, s, &lo, &hi);
        if (int rc = check_results_range(ctx, ctx->devs[(size_t)s], lo, hi, "rpk_select_pending_changed")) return rc;
    }
    std::vector<uint32_t> pend((size_t)n, 0), stale((size_t)n, 0);
    std::vector<uint64_t> launches((size_t)n, 0);
    // 1. every GPU lists the stale pending slots of its own range (the flags and the table are replicated); both counts
    //    are copied into mapped memory ahead of the one synchronise
    int rc = guarded(ctx, [&]() -> int {
        for (int s = 0; s < n; ++s) {
            DeviceState& ds = ctx->devs[(size_t)s];
            uint32_t lo, hi; result_range(N, n, s, &lo, &hi);
            RPK_CUDA(cudaSetDevice(ds.dev));
            ds.sel_scope.host_wait();
            reserve_results(ds, lo, hi, n, s);
            reserve_compaction_state(ds);
            launches[(size_t)s] += (uint64_t)enqueue_stale(ctx, ds, lo, hi, ds.stream);
            copy_stale_counts(ds, ds.stream);
        }
        for (int s = 0; s < n; ++s) {
            DeviceState& ds = ctx->devs[(size_t)s];
            RPK_CUDA(cudaSetDevice(ds.dev));
            RPK_CUDA(cudaStreamSynchronize(ds.stream));
            const volatile uint32_t* c = result_rows(ds, false).counts;
            pend[(size_t)s] = c[0]; stale[(size_t)s] = c[1];
        }
        return RPK_OK;
    });
    if (rc != RPK_OK) return rc;
    uint32_t P = 0, R = 0;
    for (int s = 0; s < n; ++s) { P += pend[(size_t)s]; R += stale[(size_t)s]; }
    *n_pending = P; *n_reselected = R;
    // 2. the refusal and the call with nothing to reselect: no stored result changed and nothing is counted but the
    //    launches of a call that succeeds
    if (R > cap) return fail(ctx, RPK_EINVAL, "rpk_select_pending_changed: more slots to reselect than cap");
    if (R == 0) {
        *n_changed = 0;
        for (int s = 0; s < n; ++s) ctx->launches += launches[(size_t)s];
        return RPK_OK;
    }
    // 3. every GPU reselects and diffs its stale rows on its own thread; the diff writes the changed rows to r_out, as one
    //    region without peers, and their count to mapped memory; the rows themselves come back in copies of that
    //    length, and they are copied out in GPU order, which is ascending
    return guarded(ctx, [&]() -> int {
        ctx->workers.run(n, [&](int s) {
            DeviceState& ds = ctx->devs[(size_t)s];
            const uint32_t k = stale[(size_t)s];
            if (!k) return;
            uint32_t lo, hi; result_range(N, n, s, &lo, &hi);
            RPK_CUDA(cudaSetDevice(ds.dev));
            const ResultRows m = result_rows(ds, true);
            const ResultRows h = result_rows(ds, false);
            ResultXchgArgs x{};
            x.n_out = 1; x.cap = (uint32_t)(ds.r_out.cap / (2 + RPK_TOPK)); x.region[0] = m.slot; x.count[0] = m.counts + 2;
            ds.res_ready = false;  // until the diff has stored every reselected row
            launches[(size_t)s] += (uint64_t)enqueue_reselect(ds, k, true, lo, gen, x, nullptr, ds.stream);
            RPK_CUDA(cudaStreamSynchronize(ds.stream));
            ds.res_ready = true;
            const uint32_t c = reinterpret_cast<volatile uint32_t*>(h.counts)[2];
            if (c) {
                RPK_CUDA(cudaMemcpyAsync(h.slot, m.slot, (size_t)c * 4, cudaMemcpyDeviceToHost, ds.stream));
                RPK_CUDA(cudaMemcpyAsync(h.best, m.best, (size_t)c * 4, cudaMemcpyDeviceToHost, ds.stream));
                RPK_CUDA(cudaMemcpyAsync(h.top5, m.top5, (size_t)c * 4 * RPK_TOPK, cudaMemcpyDeviceToHost, ds.stream));
                RPK_CUDA(cudaStreamSynchronize(ds.stream));
            }
        });
        uint32_t at = 0;
        for (int s = 0; s < n; ++s) {
            DeviceState& ds = ctx->devs[(size_t)s];
            ctx->launches += launches[(size_t)s];
            if (!stale[(size_t)s]) continue;
            const ResultRows h = result_rows(ds, false);
            const uint32_t c = reinterpret_cast<volatile uint32_t*>(h.counts)[2];
            memcpy(slots_out + at, h.slot, (size_t)c * 4);
            memcpy(best + at, h.best, (size_t)c * 4);
            memcpy(top5 + (size_t)at * RPK_TOPK, h.top5, (size_t)c * 4 * RPK_TOPK);
            at += c;
        }
        *n_changed = at;
        count_select(ctx, R, ctx->devs[0].G);
        return RPK_OK;
    });
}

size_t rpk_results_xchg_bytes(int n_ranks, uint32_t cap) {
    if (n_ranks < 1 || n_ranks > RPK_MAX_GPUS) return 0;
    return (8 + (size_t)n_ranks * cap * (2 + RPK_TOPK)) * 4 + 16;
}

namespace {
// The refusals of rpk_select_pending_changed_gather and its device form, in order (`who` names the call; args_ok: its
// own pointer arguments, refused with the n_ranks / my_rank message `required`).  On RPK_OK [*lo, *hi) is the rank's
// owned range.  Every refusal comes before the first launch, and cap >= hi - lo bounds what the diff can write: once the
// stale step has run, the call always finishes with its count and its signal, so no peer is left waiting.
int check_results_gather(rpk_ctx* ctx, const char* who, int shard, int n_ranks, int my_rank, uint32_t* const* d_xchg, uint32_t cap,
                         bool args_ok, const char* required, uint32_t* lo, uint32_t* hi) {
    if (bad_shard(ctx, shard)) return fail(ctx, RPK_EINVAL, std::string(who) + ": shard out of range");
    if (n_ranks < 1 || n_ranks > RPK_MAX_GPUS || my_rank < 0 || my_rank >= n_ranks || !d_xchg || !args_ok)
        return fail(ctx, RPK_EINVAL, std::string(who) + ": " + required);
    for (int o = 0; o < n_ranks; ++o)
        if (!d_xchg[o] || ((uintptr_t)d_xchg[o] & 15)) return fail(ctx, RPK_EINVAL, std::string(who) + ": NULL or not 16-byte aligned exchange buffer");
    if (int rc = check_select_ready(ctx, who, true, shard)) return rc;
    const DeviceState& ds = ctx->devs[(size_t)shard];
    result_range(ds.podsN, n_ranks, my_rank, lo, hi);
    if (cap < *hi - *lo) return fail(ctx, RPK_EINVAL, std::string(who) + ": cap is below the number of slots the rank owns");
    return check_results_range(ctx, ds, *lo, *hi, who);
}

// The exchange of rank my_rank: buffer o is [counts : 8 words][region r: slot[cap], best[cap], top5[5 cap]]...; the diff
// fills and signals under the rank the call names (x.d is the caller's)
ResultXchgArgs results_xchg(const rpk_ctx* ctx, int shard, int n_ranks, int my_rank, uint32_t* const* d_xchg, uint32_t cap) {
    ResultXchgArgs x{};
    x.n_out = n_ranks; x.cap = cap;
    for (int o = 0; o < n_ranks; ++o) {
        x.region[o] = d_xchg[o] + 8 + (size_t)my_rank * (2 + RPK_TOPK) * cap;
        x.count[o] = d_xchg[o] + my_rank;
    }
    x.peers = ctx->bind[(size_t)shard];
    x.peers.my_rank = my_rank;
    return x;
}
}  // namespace

int rpk_select_pending_changed_gather(rpk_ctx* ctx, int shard, int n_ranks, int my_rank, uint32_t* const* d_xchg, uint32_t cap,
                                      uint32_t* n_pending, uint32_t* n_reselected, void* stream) {
    static const char* who = "rpk_select_pending_changed_gather";
    if (!ctx) return RPK_EINVAL;
    uint32_t lo, hi;
    if (int rc = check_results_gather(ctx, who, shard, n_ranks, my_rank, d_xchg, cap, n_pending && n_reselected,
                                      "n_ranks in 1..8, my_rank in [0, n_ranks), d_xchg, n_pending and n_reselected are required", &lo, &hi))
        return rc;
    DeviceState& ds = ctx->devs[(size_t)shard];
    const uint32_t gen = ctx->offer_gen;
    return device_call(ctx, shard, stream, nullptr, [&](DeviceState&, cudaStream_t st) {
        ds.sel_scope.host_wait();
        reserve_results(ds, lo, hi, n_ranks, my_rank);
        reserve_compaction_state(ds);
        uint64_t launches = (uint64_t)enqueue_stale(ctx, ds, lo, hi, st);
        copy_stale_counts(ds, st);
        RPK_CUDA(cudaStreamSynchronize(st));  // the reselect is sized for the row count the host reads
        const volatile uint32_t* c = result_rows(ds, false).counts;
        const uint32_t k = c[1];
        *n_pending = c[0]; *n_reselected = k;
        ResultXchgArgs x = results_xchg(ctx, shard, n_ranks, my_rank, d_xchg, cap);
        ds.res_ready = false;       // until the diff is enqueued behind the reselect
        launches += (uint64_t)enqueue_reselect(ds, k, true, lo, gen, x, nullptr, st);
        ds.res_ready = true;
        ds.sel_scope.device_end(st, true);
        ctx->launches += launches;
        if (k) count_select(ctx, k, ds.G);
    });
}

// The same tick with the row count kept on the device: the reselect and the diff are sized for the rank's worst case,
// hi - lo rows, so nothing waits for the host.  Every buffer is sized in prep for that worst case: after one call the
// call only enqueues.  The reselected rows' columns and lists go to r_lane, which no select grows, so a select of any
// size on the ctx cannot free what a captured graph writes.
int rpk_select_pending_changed_device_gather(rpk_ctx* ctx, int shard, int n_ranks, int my_rank, uint32_t* const* d_xchg,
                                             uint32_t cap, uint32_t* d_counts, void* stream) {
    static const char* who = "rpk_select_pending_changed_device_gather";
    if (!ctx) return RPK_EINVAL;
    uint32_t lo, hi;
    if (int rc = check_results_gather(ctx, who, shard, n_ranks, my_rank, d_xchg, cap, ((uintptr_t)d_counts & 3) == 0,
                                      "n_ranks in 1..8, my_rank in [0, n_ranks) and d_xchg are required, d_counts 4-byte aligned", &lo, &hi))
        return rc;
    DeviceState& ds = ctx->devs[(size_t)shard];
    const uint32_t gen = ctx->offer_gen;
    const auto prep = [&](DeviceState&) {
        reserve_results(ds, lo, hi, n_ranks, my_rank);
        reserve_compaction_state(ds);
        return RPK_OK;
    };
    return device_call(ctx, shard, stream, &DeviceState::sel_scope, prep, [&](DeviceState&, cudaStream_t st) {
        ds.res_ready = false;  // until every launch is enqueued
        uint64_t launches = (uint64_t)enqueue_stale(ctx, ds, lo, hi, st);
        ResultXchgArgs x = results_xchg(ctx, shard, n_ranks, my_rank, d_xchg, cap);
        launches += (uint64_t)enqueue_reselect(ds, hi - lo, false, lo, gen, x, d_counts, st);
        ds.res_ready = true;
        ctx->launches += launches;
    });
}

// ---- growing the tables ---------------------------------------------------------------------------------------

int rpk_pods_grow(rpk_ctx* ctx, uint32_t N) {
    static const char* who = "rpk_pods_grow";
    if (!ctx) return RPK_EINVAL;
    if (int rc = check_select_ready(ctx, who, true, -1, false)) return rc;
    const uint32_t N0 = ctx->devs[0].podsN;
    if (N < N0) return fail(ctx, RPK_EINVAL, std::string(who) + ": N is below the pod table's size (a table only grows)");
    if (N == N0) return RPK_OK;
    const int n = (int)ctx->devs.size();
    // The stored results move with their slots when every GPU holds the range rpk_select_pending_changed gives it.  Any
    // other results were made for the range of a one-process-per-GPU rank, whose peers' results live in other processes:
    // they are cleared, as rpk_pods_reset clears them.
    bool move_results = true;
    for (int s = 0; s < n; ++s) {
        const DeviceState& ds = ctx->devs[(size_t)s];
        move_results = move_results && ds.res_ready && ds.res_bound && ds.res_ranks == n && ds.res_rank == s;
    }
    std::vector<SlotRange> was((size_t)n), now((size_t)n);
    for (int s = 0; s < n; ++s) {
        result_range(N0, n, s, &was[(size_t)s].lo, &was[(size_t)s].hi);
        result_range(N, n, s, &now[(size_t)s].lo, &now[(size_t)s].hi);
    }
    struct Bufs {
        Grow<PodBufs> rows, r_cols, l_cols; Grow<DevBuf<uint8_t>> pending; Grow<DevBuf<uint32_t>> list, r_gen, r_list;
        Grow<DevBuf<int32_t>> r_top5, r_out, l_top5; Grow<DevBuf<uint16_t>> r_mask;
        PinnedBuf h_res;
    };
    std::vector<std::unique_ptr<Bufs>> g;
    const int rc = guarded(ctx, [&]() -> int {
        // 1. every GPU's new buffers, before anything changes
        for (int s = 0; s < n; ++s) {
            DeviceState& ds = ctx->devs[(size_t)s];
            RPK_CUDA(cudaSetDevice(ds.dev));
            ds.sel_scope.host_wait();  // a device select may still gather from the table
            g.emplace_back(new Bufs());
            Bufs& b = *g.back();
            b.rows.alloc(ds.pt_cols, N); b.pending.alloc(ds.pt_pending, N);
            b.list.alloc(ds.pt_list, ds.pt_list.p ? N : 0);
            if (!move_results) continue;
            // the sizes reserve_results gives a range; a range whose first slot moves gets new columns
            const SlotRange r = now[(size_t)s];
            const bool moved = r.lo != was[(size_t)s].lo;
            const size_t m = ((size_t)(r.hi - r.lo) + 15) / 16 * 16 + 16, rows = std::max<uint32_t>(r.hi - r.lo, 1u);
            b.r_cols.alloc(ds.r_cols, m, moved); b.r_gen.alloc(ds.r_gen, m, moved); b.r_top5.alloc(ds.r_top5, m * RPK_TOPK, moved);
            b.r_list.alloc(ds.r_list, m); b.r_mask.alloc(ds.r_mask, m / 16 + 1);
            b.l_cols.alloc(ds.r_lane.cols, rows); b.l_top5.alloc(ds.r_lane.top5, rows * RPK_TOPK);
            b.r_out.alloc(ds.r_out, m * (2 + RPK_TOPK));
            if (64 + b.r_out.dst_cap() * 4 > ds.h_res.cap) b.h_res.reserve(64 + b.r_out.dst_cap() * 4);
        }
        // 2. the rows and flags of [0, N0) stay, [N0, N) become reset rows (k_pod_fill on the new part alone); the stored
        //    results go to their new owners, and every owned slot without one has generation 0
        for (int s = 0; s < n; ++s) {
            DeviceState& ds = ctx->devs[(size_t)s];
            Bufs& b = *g[(size_t)s];
            RPK_CUDA(cudaSetDevice(ds.dev));
            b.rows.keep(N0, ds.stream); b.pending.keep(N0, ds.stream);
            PodRows fresh_rows{};
            b.rows.each([N0](auto&, auto* dst, auto*& row) { row = dst + N0; }, fresh_rows);
            ctx->launches += (uint64_t)launch_pod_fill(fresh_rows, b.pending.dst() + N0, N - N0, ds.sm_count, ds.stream);
            if (!move_results) continue;
            const size_t kept = b.r_gen.dst() == ds.r_gen.p ? was[(size_t)s].hi - was[(size_t)s].lo : 0;
            RPK_CUDA(cudaMemsetAsync(b.r_gen.dst() + kept, 0, (b.r_gen.dst_cap() - kept) * sizeof(uint32_t), ds.stream));
        }
        if (move_results) {
            const auto of = [&g](auto Bufs::*m) { return [&g, m](size_t s) -> auto& { return (*g[s]).*m; }; };
            move_slots(ctx, was, now, of(&Bufs::r_cols), 1); move_slots(ctx, was, now, of(&Bufs::r_gen), 1);
            move_slots(ctx, was, now, of(&Bufs::r_top5), RPK_TOPK);
        }
        sync_all(ctx);
        // 3. the new buffers and sizes take effect together
        for (int s = 0; s < n; ++s) {
            DeviceState& ds = ctx->devs[(size_t)s];
            Bufs& b = *g[(size_t)s];
            b.rows.commit(); b.pending.commit(); b.list.commit();
            ds.podsN = N;
            if (!move_results) { ds.res_ready = ds.res_bound = false; continue; }
            b.r_cols.commit(); b.r_gen.commit(); b.r_top5.commit(); b.r_list.commit(); b.r_mask.commit(); b.r_out.commit();
            b.l_cols.commit(); b.l_top5.commit();
            if (b.h_res.h) ds.h_res.swap(b.h_res);
            ds.res_lo = now[(size_t)s].lo; ds.res_hi = now[(size_t)s].hi;
        }
        return RPK_OK;
    });
    if (rc != RPK_OK) ctx->err = std::string(who) + ": " + ctx->err;
    return rc;
}

// ---- cross-process peer vectors (CUDA IPC) ---------------------------------------------------------------

int rpk_ipc_alloc(rpk_ctx* ctx, int shard, size_t bytes, void** d_ptr, unsigned char handle_out[64]) {
    if (!ctx) return RPK_EINVAL;
    if (bad_shard(ctx, shard) || !d_ptr || !handle_out || bytes == 0) return fail(ctx, RPK_EINVAL, "rpk_ipc_alloc: bad argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle is 64 bytes");
    return device_call(ctx, shard, nullptr, nullptr, [&](DeviceState&, cudaStream_t) {
        void* p = nullptr;
        RPK_CUDA(cudaMalloc(&p, bytes));
        RPK_CUDA(cudaMemset(p, 0, bytes));
        cudaIpcMemHandle_t h;
        cudaError_t e = cudaIpcGetMemHandle(&h, p);
        if (e != cudaSuccess) { cudaFree(p); RPK_CUDA(e); }
        memcpy(handle_out, &h, 64);
        ctx->ipc_owned.emplace_back(shard, p);
        *d_ptr = p;
    });
}

int rpk_ipc_open(rpk_ctx* ctx, int shard, const unsigned char handle[64], void** d_peer_ptr) {
    if (!ctx) return RPK_EINVAL;
    if (bad_shard(ctx, shard) || !handle || !d_peer_ptr) return fail(ctx, RPK_EINVAL, "rpk_ipc_open: bad argument");
    return device_call(ctx, shard, nullptr, nullptr, [&](DeviceState&, cudaStream_t) {
        cudaIpcMemHandle_t h;
        memcpy(&h, handle, 64);
        void* p = nullptr;
        RPK_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
        ctx->ipc_mapped.emplace_back(shard, p);
        *d_peer_ptr = p;
    });
}

static int drop_entry(std::vector<std::pair<int, void*>>& v, int shard, void* p) {
    for (size_t i = 0; i < v.size(); ++i)
        if (v[i].first == shard && v[i].second == p) { v.erase(v.begin() + (long)i); return 1; }
    return 0;
}

int rpk_ipc_close(rpk_ctx* ctx, int shard, void* d_peer_ptr) {
    if (!ctx) return RPK_EINVAL;
    if (!drop_entry(ctx->ipc_mapped, shard, d_peer_ptr)) return fail(ctx, RPK_EINVAL, "rpk_ipc_close: pointer was not opened by this ctx");
    return device_call(ctx, shard, nullptr, nullptr, [&](DeviceState&, cudaStream_t) { RPK_CUDA(cudaIpcCloseMemHandle(d_peer_ptr)); });
}

int rpk_ipc_free(rpk_ctx* ctx, int shard, void* d_ptr) {
    if (!ctx) return RPK_EINVAL;
    if (!drop_entry(ctx->ipc_owned, shard, d_ptr)) return fail(ctx, RPK_EINVAL, "rpk_ipc_free: pointer was not allocated by this ctx");
    return device_call(ctx, shard, nullptr, nullptr, [&](DeviceState&, cudaStream_t) { RPK_CUDA(cudaFree(d_ptr)); });
}

int rpk_peer_fence(rpk_ctx* ctx, int shard, int n, uint32_t* const* d_flags, int my_rank, uint32_t epoch, void* stream) {
    if (!ctx) return RPK_EINVAL;
    if (bad_shard(ctx, shard) || n < 1 || n > RPK_MAX_GPUS || !d_flags || my_rank < 0 || my_rank >= n)
        return fail(ctx, RPK_EINVAL, "rpk_peer_fence: bad argument");
    for (int r = 0; r < n; ++r) if (!d_flags[r]) return fail(ctx, RPK_EINVAL, "rpk_peer_fence: NULL flag array");
    return device_call(ctx, shard, stream, nullptr, [&](DeviceState&, cudaStream_t st) {
        PeerGroup g{};
        for (int r = 0; r < n; ++r) g.flags[r] = d_flags[r];
        g.n = n; g.my_rank = my_rank;
        ctx->launches += (uint64_t)launch_peer_signal(g, epoch, true, st);
    });
}

int rpk_peer_bind(rpk_ctx* ctx, int shard, int n, uint32_t* const* d_flags, int my_rank) {
    if (!ctx) return RPK_EINVAL;
    if (bad_shard(ctx, shard) || n < 0 || n > RPK_MAX_GPUS || (n > 0 && (!d_flags || my_rank < 0 || my_rank >= n)))
        return fail(ctx, RPK_EINVAL, "rpk_peer_bind: bad argument");
    for (int r = 0; r < n; ++r) if (!d_flags[r]) return fail(ctx, RPK_EINVAL, "rpk_peer_bind: NULL flag array");
    PeerGroup& b = ctx->bind[(size_t)shard];
    const int keep = b.inline_wait;
    b = PeerGroup{};
    for (int r = 0; r < n; ++r) b.flags[r] = d_flags[r];
    b.n = n; b.my_rank = my_rank; b.inline_wait = keep;
    return RPK_OK;
}

int rpk_peer_inline_wait(rpk_ctx* ctx, int shard, int on) {
    if (!ctx) return RPK_EINVAL;
    if (bad_shard(ctx, shard)) return fail(ctx, RPK_EINVAL, "rpk_peer_inline_wait: shard out of range");
    ctx->bind[(size_t)shard].inline_wait = on ? 1 : 0;
    return RPK_OK;
}

int rpk_peer_wait(rpk_ctx* ctx, int shard, unsigned what, void* stream) {
    if (!ctx) return RPK_EINVAL;
    if (bad_shard(ctx, shard) || (what & ~7u) || !what) return fail(ctx, RPK_EINVAL, "rpk_peer_wait: bad argument");
    if (ctx->bind[(size_t)shard].n == 0) return fail(ctx, RPK_ESTATE, "rpk_peer_wait: no flags bound (rpk_peer_bind)");
    return device_call(ctx, shard, stream, nullptr, [&](DeviceState&, cudaStream_t st) {
        ctx->launches += (uint64_t)launch_peer_wait(ctx->bind[(size_t)shard], what, st);
    });
}

/* test / integration hook: device pointer of GPU `shard`'s copy of the last full assignment vector */
const int32_t* rpk_best_device_ptr(const rpk_ctx* ctx, int shard) {
    if (!ctx || bad_shard(ctx, shard)) return nullptr;
    return ctx->devs[(size_t)shard].best_full.p;
}

/* test hook: the ctx-owned device buffers a _device call on `shard` hands its kernels, in a fixed order */
int rpk_test_capture_buffers(const rpk_ctx* ctx, int shard, const void** ptrs, size_t cap, size_t* n) {
    if (!ctx || bad_shard(ctx, shard) || !n || (cap > 0 && !ptrs)) return RPK_EINVAL;
    const DeviceState& ds = ctx->devs[(size_t)shard];
    std::vector<const void*> v;
    const auto add = [&v](const auto& b) { v.push_back(b.p); };
    const auto lane = [&](const DeviceState::Lane& ln) {
        PodBufs::each(ln.cols, add);
        v.insert(v.end(), {ln.p_slots.p, ln.top5.p, ln.rw.p, ln.order.p, ln.pos.p, ln.ctrs.p, ln.key.p, ln.ord_rw.p, ln.hist.p,
                           ln.k0_base.p, ln.hdr.p});
    };
    lane(ds.dev_lane);
    const DeviceState::SweepScratch& w = ds.dev_sweep;
    v.insert(v.end(), {w.tile_state.p, w.misc.p, w.stage_idx.p, w.stage_code.p, w.unit_cnt.p});
    for (int c = 0; c < 2; ++c)
        v.insert(v.end(), {ds.v_packed[c].p, ds.v_bitmap[c].p, ds.v_bitmapT[c].p, ds.v_bitmapM[c].p, ds.v_wide[c].p, ds.v_price[c].p,
                           ds.v_perm[c].p});
    for (const auto& d : ds.distinct) add(d);
    OfferBufs::each(ds.raw, add); add(ds.win);
    PodBufs::each(ds.pt_cols, add); v.insert(v.end(), {ds.pt_pending.p, ds.pt_state.p, ds.pt_ticket.p});
    PodBufs::each(ds.r_cols, add); v.insert(v.end(), {ds.r_gen.p, ds.r_top5.p, ds.r_list.p, ds.r_mask.p, ds.r_dn.p});

    lane(ds.r_lane);
    *n = v.size();
    for (size_t i = 0; i < v.size() && i < cap; ++i) ptrs[i] = v[i];
    return RPK_OK;
}

// ---- status --------------------------------------------------------------------------------------------

static int check_stride(rpk_ctx* ctx, uint32_t stride, const char* who) {
    if (stride < 16 || stride > 256 || (stride & 15)) return fail(ctx, RPK_EINVAL, std::string(who) + ": status stride must be a multiple of 16 in [16, 256]");
    return RPK_OK;
}

int rpk_status_reset(rpk_ctx* ctx, uint32_t N) {
    if (!ctx) return RPK_EINVAL;
    return guarded(ctx, [&]() -> int {
        const int n = (int)ctx->devs.size();
        for (int s = 0; s < n; ++s) {
            DeviceState& ds = ctx->devs[(size_t)s];
            uint32_t lo, hi; shard_range(N, n, s, &lo, &hi);
            RPK_CUDA(cudaSetDevice(ds.dev));
            ds.s_hash_prev.reserve((hi - lo) ? (hi - lo) : 1);
            RPK_CUDA(cudaMemsetAsync(ds.s_hash_prev.p, 0, (size_t)((hi - lo) ? (hi - lo) : 1) * 8, ds.stream));
            RPK_CUDA(cudaStreamSynchronize(ds.stream));
            ds.statusN = N; ds.status_sized = true;
        }
        return RPK_OK;
    });
}

int rpk_status_grow(rpk_ctx* ctx, uint32_t N) {
    static const char* who = "rpk_status_grow";
    if (!ctx) return RPK_EINVAL;
    if (!ctx->devs[0].status_sized) return fail(ctx, RPK_ESTATE, std::string(who) + ": no tracked table (call rpk_status_reset first)");
    const uint32_t N0 = ctx->devs[0].statusN;
    if (N < N0) return fail(ctx, RPK_EINVAL, std::string(who) + ": N is below the tracked table's size (a table only grows)");
    if (N == N0) return RPK_OK;
    const int n = (int)ctx->devs.size();
    std::vector<SlotRange> was((size_t)n), now((size_t)n);
    for (int s = 0; s < n; ++s) {
        shard_range(N0, n, s, &was[(size_t)s].lo, &was[(size_t)s].hi);
        shard_range(N, n, s, &now[(size_t)s].lo, &now[(size_t)s].hi);
    }
    std::vector<std::unique_ptr<Grow<DevBuf<uint64_t>>>> g;
    const int rc = guarded(ctx, [&]() -> int {
        // 1. every GPU's new column, before anything changes; a shard whose first slot moves gets a new one
        for (int s = 0; s < n; ++s) {
            DeviceState& ds = ctx->devs[(size_t)s];
            RPK_CUDA(cudaSetDevice(ds.dev));
            g.emplace_back(new Grow<DevBuf<uint64_t>>());
            g.back()->alloc(ds.s_hash_prev, std::max<uint32_t>(now[(size_t)s].hi - now[(size_t)s].lo, 1u), now[(size_t)s].lo != was[(size_t)s].lo);
        }
        // 2. every new slot is never seen (hash 0), the hashes of [0, N0) go to their new shards
        for (int s = 0; s < n; ++s) {
            DeviceState& ds = ctx->devs[(size_t)s];
            const Grow<DevBuf<uint64_t>>& b = *g[(size_t)s];
            RPK_CUDA(cudaSetDevice(ds.dev));
            const size_t kept = b.dst() == ds.s_hash_prev.p ? was[(size_t)s].hi - was[(size_t)s].lo : 0;
            const size_t m = std::max<uint32_t>(now[(size_t)s].hi - now[(size_t)s].lo, 1u);
            RPK_CUDA(cudaMemsetAsync(b.dst() + kept, 0, (m - kept) * sizeof(uint64_t), ds.stream));
        }
        move_slots(ctx, was, now, [&g](size_t s) -> auto& { return *g[s]; }, 1);
        sync_all(ctx);
        // 3. the new columns and the size take effect together
        for (int s = 0; s < n; ++s) { g[(size_t)s]->commit(); ctx->devs[(size_t)s].statusN = N; }
        return RPK_OK;
    });
    if (rc != RPK_OK) ctx->err = std::string(who) + ": " + ctx->err;
    return rc;
}

namespace {

// The argument checks of a whole-table host sweep (rpk_status_diff*, rpk_status_seed, rpk_tick; `who` names the entry
// point in the messages).  The first sweep of a ctx sizes the tracked table to its N.
int check_sweep(rpk_ctx* ctx, const StatusHostArgs& h, const char* who) {
    const std::string w(who);
    if (int rc = check_stride(ctx, h.stride, who)) return rc;
    if (h.N > 0 && !h.records) return fail(ctx, RPK_EINVAL, w + ": records is NULL");
    if (h.report && (!h.n_changed || (h.N > 0 && !h.changed_idx))) return fail(ctx, RPK_EINVAL, w + ": changed_idx and n_changed are required");
    if (!ctx->devs[0].status_sized) { if (int rc = rpk_status_reset(ctx, h.N)) return rc; }
    if (ctx->devs[0].statusN != h.N) return fail(ctx, RPK_ESTATE, w + ": N differs from the tracked table (call rpk_status_reset to resize)");
    return RPK_OK;
}

int status_host(rpk_ctx* ctx, const StatusHostArgs& h, const char* who) {
    if (!ctx) return RPK_EINVAL;
    if (int rc = check_sweep(ctx, h, who)) return rc;
    return guarded(ctx, [&]() -> int { run_host(ctx, nullptr, &h, false); return RPK_OK; });
}

}  // namespace

int rpk_status_diff(rpk_ctx* ctx, uint32_t N, const uint8_t* records, uint32_t stride, uint32_t* changed_idx,
                    uint32_t* n_changed, uint64_t* hashes_out) {
    return status_host(ctx, StatusHostArgs{N, records, stride, changed_idx, nullptr, n_changed, hashes_out, true}, "rpk_status_diff");
}

int rpk_status_diff_codes(rpk_ctx* ctx, uint32_t N, const uint8_t* records, uint32_t stride, uint32_t* changed_idx,
                          uint16_t* changed_code, uint32_t* n_changed, uint64_t* hashes_out) {
    return status_host(ctx, StatusHostArgs{N, records, stride, changed_idx, changed_code, n_changed, hashes_out, true}, "rpk_status_diff_codes");
}

int rpk_status_seed(rpk_ctx* ctx, uint32_t N, const uint8_t* records, uint32_t stride) {
    return status_host(ctx, StatusHostArgs{N, records, stride, nullptr, nullptr, nullptr, nullptr, false}, "rpk_status_seed");
}

int rpk_status_seed_slots(rpk_ctx* ctx, uint32_t n_slots, const uint32_t* slots, const uint8_t* records, uint32_t stride) {
    if (!ctx) return RPK_EINVAL;
    if (int rc = check_stride(ctx, stride, "rpk_status_seed_slots")) return rc;
    if (n_slots == 0) return RPK_OK;
    if (!slots || !records) return fail(ctx, RPK_EINVAL, "rpk_status_seed_slots: slots and records are required");
    if (!ctx->devs[0].status_sized) return fail(ctx, RPK_ESTATE, "rpk_status_seed_slots: no tracked table (call rpk_status_reset first)");
    const uint32_t N = ctx->devs[0].statusN;
    if (int rc = check_slots(ctx, n_slots, slots, N, false, "rpk_status_seed_slots", "tracked table")) return rc;
    return guarded(ctx, [&]() -> int {
        const int n = (int)ctx->devs.size();
        for (int s = 0; s < n; ++s) {  // a handful of slots: every GPU gets the list and keeps the ones of its shard
            DeviceState& ds = ctx->devs[(size_t)s];
            uint32_t lo, hi; shard_range(N, n, s, &lo, &hi);
            bool any = false;
            for (uint32_t i = 0; i < n_slots && !any; ++i) any = slots[i] >= lo && slots[i] < hi;
            if (!any) continue;
            RPK_CUDA(cudaSetDevice(ds.dev));
            ds.s_seed_slots.reserve(n_slots); ds.s_seed_recs.reserve((size_t)n_slots * stride);
            RPK_CUDA(cudaMemcpyAsync(ds.s_seed_slots.p, slots, (size_t)n_slots * 4, cudaMemcpyHostToDevice, ds.stream));
            RPK_CUDA(cudaMemcpyAsync(ds.s_seed_recs.p, records, (size_t)n_slots * stride, cudaMemcpyHostToDevice, ds.stream));
            ctx->launches += (uint64_t)launch_status_seed_slots(n_slots, ds.s_seed_slots.p, ds.s_seed_recs.p, stride, ds.s_hash_prev.p, lo, hi, ds.stream);
            RPK_CUDA(cudaStreamSynchronize(ds.stream));
        }
        return RPK_OK;
    });
}

int rpk_status_diff_slots(rpk_ctx* ctx, uint32_t n_slots, const uint32_t* slots, const uint8_t* records, uint32_t stride,
                          uint32_t* changed_idx, uint16_t* changed_code, uint32_t* n_changed) {
    if (!ctx) return RPK_EINVAL;
    if (int rc = check_stride(ctx, stride, "rpk_status_diff_slots")) return rc;
    if (!n_changed) return fail(ctx, RPK_EINVAL, "rpk_status_diff_slots: n_changed is required");
    if (n_slots == 0) { *n_changed = 0; return RPK_OK; }
    if (!slots || !records || !changed_idx) return fail(ctx, RPK_EINVAL, "rpk_status_diff_slots: slots, records and changed_idx are required");
    if (!ctx->devs[0].status_sized) return fail(ctx, RPK_ESTATE, "rpk_status_diff_slots: no tracked table (call rpk_status_reset first)");
    const uint32_t N = ctx->devs[0].statusN;
    if (int rc = check_slots(ctx, n_slots, slots, N, true, "rpk_status_diff_slots", "tracked table")) return rc;
    StatusHostArgs h{N, records, stride, changed_idx, changed_code, n_changed, nullptr, true};
    h.slots = slots; h.n_slots = n_slots;
    return guarded(ctx, [&]() -> int { run_host(ctx, nullptr, &h, false); return RPK_OK; });
}

// One tick of the kubelet: the pending-pod selection (processPendingPods, kubelet.go:747-814) and the status sweep
// (updateAllPodStatuses, kubelet.go:816-974) are independent, so their copies and kernels are enqueued together --
// the sweep's upload runs behind the selection's, the kernels of one under the copies of the other -- and the
// call synchronises once.
int rpk_tick(rpk_ctx* ctx, uint32_t P, const int32_t* req_mem_gb, const int32_t* req_vcpu, const int32_t* req_ram_gb,
             const double* max_price, const uint8_t* cloud, int32_t* best, int32_t* top5, uint32_t N, const uint8_t* records,
             uint32_t stride, uint32_t* changed_idx, uint16_t* changed_code, uint32_t* n_changed) {
    if (!ctx) return RPK_EINVAL;
    if (P > 0 && (!req_mem_gb || !best)) return fail(ctx, RPK_EINVAL, "rpk_tick: req_mem_gb and best are required");
    if (P > 0) { if (int rc = check_select_ready(ctx, "rpk_tick", false)) return rc; }
    const StatusHostArgs h{N, records, stride, changed_idx, changed_code, n_changed, nullptr, true};
    if (int rc = check_sweep(ctx, h, "rpk_tick")) return rc;
    const RowSource rows{RowSource::HostCols, PodCols{req_mem_gb, req_vcpu, req_ram_gb, max_price, cloud}, nullptr};
    const HostSelect sel{P, std::vector<RowSource>(ctx->devs.size(), rows), best, top5};
    return guarded(ctx, [&]() -> int { run_host(ctx, P > 0 ? &sel : nullptr, &h, true); return RPK_OK; });
}

namespace {
// The arguments of a device sweep, the device counterpart of StatusHostArgs.  list (the rpk_status_diff_slots_device*
// calls): slots[0, N) lists global slot ids, and the hash column (col_n rows) holds global slots [idx_base, idx_base +
// col_n).  gather (the _gather calls): the changed list goes into region my_rank of the n_out exchange buffers, of cap
// entries per rank; with n_out = 0 the call sweeps as the calls without an exchange do.
struct StatusDeviceArgs {
    uint32_t N; const uint8_t* records; uint32_t stride; uint64_t* hash_prev; uint32_t idx_base;
    uint32_t* changed_idx; uint16_t* changed_code; uint32_t* n_changed;
    bool list; const uint32_t* slots; uint32_t col_n;
    bool gather; int n_out; uint32_t* const* xchg; uint32_t cap; int my_rank;
};

// The five rpk_status_diff*_device* calls (`who` names the one called)
int status_device(rpk_ctx* ctx, const char* who, int shard, const StatusDeviceArgs& d, void* stream) {
    if (!ctx) return RPK_EINVAL;
    const std::string w(who);
    if (d.list && d.N > 0 && !d.slots) return fail(ctx, RPK_EINVAL, w + ": d_slots is NULL");
    if (d.list && d.gather && d.n_out < 1) return fail(ctx, RPK_EINVAL, w + ": n_ranks must be 1..8");
    if (bad_shard(ctx, shard)) return fail(ctx, RPK_EINVAL, w + ": shard out of range");
    if (int rc = check_stride(ctx, d.stride, who)) return rc;
    if (d.N > 0 && (!d.records || !d.hash_prev)) return fail(ctx, RPK_EINVAL, w + ": NULL column");
    if (d.n_out == 0 && d.N > 0 && !d.changed_idx) return fail(ctx, RPK_EINVAL, w + ": d_changed_idx is NULL");
    if (!d.n_changed) return fail(ctx, RPK_EINVAL, w + ": d_n_changed is NULL");
    if (((uintptr_t)d.records | (uintptr_t)d.hash_prev) & 15) return fail(ctx, RPK_EINVAL, w + ": d_records and d_hash_prev must be 16-byte aligned");
    if (d.n_out < 0 || d.n_out > RPK_MAX_GPUS || (d.n_out > 0 && (!d.xchg || d.my_rank < 0 || d.my_rank >= d.n_out || d.N > d.cap)))
        return fail(ctx, RPK_EINVAL, w + ": bad exchange arguments (N must fit the per-rank capacity)");
    for (int o = 0; o < d.n_out; ++o) if (!d.xchg[o]) return fail(ctx, RPK_EINVAL, w + ": NULL exchange buffer");
    const uint32_t col_n = d.N > 0 ? d.col_n : 0;  // an empty list sweeps as an empty table does
    if ((uint64_t)d.idx_base + col_n > (1ull << 32)) return fail(ctx, RPK_EINVAL, w + ": idx_base + N exceeds the slot range");
    const bool codes = d.changed_code || d.n_out > 0;
    return device_call(ctx, shard, stream, &DeviceState::status_scope,
        [&](DeviceState& ds) { reserve_sweep_scratch(ds.dev_sweep, ds.sm_count, d.N, codes); return RPK_OK; },
        [&](DeviceState& ds, cudaStream_t st) {
            StatusArgs a{};
            a.records = d.records; a.stride = d.stride; a.N = d.N; a.hash_prev = d.hash_prev; a.hash_out = nullptr;
            a.changed_idx = d.changed_idx; a.changed_code = d.changed_code; a.n_changed = d.n_changed; a.idx_base = d.idx_base;
            sweep_scratch_args(ds.dev_sweep, codes, a);
            a.n_out = d.n_out;
            a.slots = d.N > 0 ? d.slots : nullptr; a.col_n = col_n;
            for (int o = 0; o < d.n_out; ++o) {  // rank o's buffer: [counts : 8 words][n_out index regions of cap][n_out code regions of cap u16]
                uint32_t* base = d.xchg[o];
                a.out_count[o] = base;
                a.out_idx[o] = base + 8 + (size_t)d.my_rank * d.cap;
                a.out_code[o] = reinterpret_cast<uint16_t*>(base + 8 + (size_t)d.n_out * d.cap) + (size_t)d.my_rank * d.cap;
            }
            if (d.n_out > 0) a.peers = ctx->bind[(size_t)shard];
            a.peers.my_rank = d.my_rank;  // the sweep fills and signals under the rank its call names
            ds.dev_sweep.dirty = true;
            ctx->launches += (uint64_t)launch_status_diff(a, ds.sm_count, st);
            ds.dev_sweep.dirty = false;
            ctx->stats.status_calls += 1; ctx->stats.status_records += d.N;
        });
}
}  // namespace

int rpk_status_diff_device(rpk_ctx* ctx, int shard, uint32_t N, const uint8_t* d_records, uint32_t stride,
                           uint64_t* d_hash_prev, uint32_t* d_changed_idx, uint32_t* d_n_changed, void* stream) {
    return status_device(ctx, "rpk_status_diff_device", shard,
                         StatusDeviceArgs{N, d_records, stride, d_hash_prev, 0, d_changed_idx, nullptr, d_n_changed}, stream);
}

int rpk_status_diff_device_codes(rpk_ctx* ctx, int shard, uint32_t N, const uint8_t* d_records, uint32_t stride,
                                 uint64_t* d_hash_prev, uint32_t* d_changed_idx, uint16_t* d_changed_code, uint32_t* d_n_changed, void* stream) {
    return status_device(ctx, "rpk_status_diff_device_codes", shard,
                         StatusDeviceArgs{N, d_records, stride, d_hash_prev, 0, d_changed_idx, d_changed_code, d_n_changed}, stream);
}

int rpk_status_diff_slots_device(rpk_ctx* ctx, int shard, uint32_t N, uint32_t idx_base, uint32_t n_slots,
                                 const uint32_t* d_slots, const uint8_t* d_records, uint32_t stride, uint64_t* d_hash_prev,
                                 uint32_t* d_changed_idx, uint16_t* d_changed_code, uint32_t* d_n_changed, void* stream) {
    return status_device(ctx, "rpk_status_diff_slots_device", shard,
                         StatusDeviceArgs{n_slots, d_records, stride, d_hash_prev, idx_base, d_changed_idx, d_changed_code, d_n_changed,
                                          true, d_slots, N}, stream);
}

size_t rpk_xchg_bytes(int n_ranks, uint32_t cap) { return (size_t)(8 + (size_t)n_ranks * cap) * 4 + (size_t)n_ranks * cap * 2 + 16; }

int rpk_status_diff_device_gather(rpk_ctx* ctx, int shard, uint32_t N, const uint8_t* d_records, uint32_t stride,
                                  uint64_t* d_hash_prev, uint32_t idx_base, int n_ranks, uint32_t* const* d_xchg, uint32_t cap,
                                  int my_rank, uint32_t* d_n_changed, void* stream) {
    return status_device(ctx, "rpk_status_diff_device_gather", shard,
                         StatusDeviceArgs{N, d_records, stride, d_hash_prev, idx_base, nullptr, nullptr, d_n_changed,
                                          false, nullptr, 0, true, n_ranks, d_xchg, cap, my_rank}, stream);
}

// n_slots bounds what a region receives (list order is not checked on the device), so it is what must fit the capacity
int rpk_status_diff_slots_device_gather(rpk_ctx* ctx, int shard, uint32_t N, uint32_t idx_base, uint32_t n_slots,
                                        const uint32_t* d_slots, const uint8_t* d_records, uint32_t stride,
                                        uint64_t* d_hash_prev, int n_ranks, uint32_t* const* d_xchg, uint32_t cap,
                                        int my_rank, uint32_t* d_n_changed, void* stream) {
    return status_device(ctx, "rpk_status_diff_slots_device_gather", shard,
                         StatusDeviceArgs{n_slots, d_records, stride, d_hash_prev, idx_base, nullptr, nullptr, d_n_changed,
                                          true, d_slots, N, true, n_ranks, d_xchg, cap, my_rank}, stream);
}

int rpk_stats_get(const rpk_ctx* ctx, rpk_stats* out) {
    if (!ctx || !out) return RPK_EINVAL;
    *out = ctx->stats;
    return RPK_OK;
}

uint64_t rpk_launch_count(const rpk_ctx* ctx) { return ctx ? ctx->launches : 0; }

}  // extern "C"
