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
    explicit rpk_ctx(int n_gpus) : devs((size_t)n_gpus), bind((size_t)n_gpus) {}
};

rpk::DeviceState::~DeviceState() {
    if (dev < 0 || cudaSetDevice(dev) != cudaSuccess) { cudaGetLastError(); return; }  // creation failed before this GPU
    if (stream) cudaStreamSynchronize(stream);
    if (status_stream) cudaStreamSynchronize(status_stream);
    for (auto& ln : lane) if (ln.stream) cudaStreamSynchronize(ln.stream);
    for (auto& ln : lane) {
        if (ln.done) cudaEventDestroy(ln.done);
        if (ln.stream) cudaStreamDestroy(ln.stream);
    }
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    if (sel_scope.ev) cudaEventDestroy(sel_scope.ev);
    if (status_scope.ev) cudaEventDestroy(status_scope.ev);
    if (status_stream) cudaStreamDestroy(status_stream);
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

// Where the rows of a select come from: the caller's columns (rpk_select, rpk_tick: host memory; rpk_select_device*:
// device memory), or rows of the pod table (rpk_select_slots: a host list, each sub-batch uploads its slot ids and
// gathers the five columns on the device; rpk_select_slots_device*: a device list, gathered in one pass).
struct PodSource {
    PodCols cols;
    const uint32_t* slots;  // non-null: row i of the call is pod-table row slots[i]; cols is unused
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

// The gather of n pod-table rows whose slot ids are at d_slots (device) into lane ln's pod columns, on st; a's pod columns
// then point at them.  Returns the kernels launched.
int gather_pod_rows(DeviceState& ds, DeviceState::Lane& ln, uint32_t n, const uint32_t* d_slots, SelectArgs& a, cudaStream_t st) {
    const PodRows out{ln.p_req_mem.p, ln.p_req_vcpu.p, ln.p_req_ram.p, ln.p_max_price.p, ln.p_cloud.p};
    a.req_mem = out.mem; a.req_vcpu = out.vcpu; a.req_ram = out.ram; a.max_price = out.max_price; a.cloud = out.cloud;
    return launch_pod_gather(ds.pods_table(), ds.podsN, n, d_slots, out, st);
}

// One select on ds in lane ln's scratch: `a` holds the pod columns, P and the outputs; this adds the offer views and the
// scratch and launches on st.  A bit-sliced table takes the persistent kernel above the fused kernel's batch size and
// the fused kernel otherwise (which also serves an empty table at any batch size).  t5: the top-5 lists' gather, if
// any.  Returns the kernels launched.
int enqueue_select(DeviceState& ds, DeviceState::Lane& ln, SelectArgs& a, cudaStream_t st, const Top5Gather* t5 = nullptr) {
    for (int c = 0; c < 2; ++c) {
        a.view[c].packed = ds.v_packed[c].p; a.view[c].bitmap = ds.v_bitmap[c].p; a.view[c].bitmapT = ds.v_bitmapT[c].p;
        a.view[c].bitmapM = ds.pk.slice_rows ? ds.v_bitmapM[c].p : nullptr; a.view[c].wide = ds.v_wide[c].p;
        a.view[c].price = ds.v_price[c].p; a.view[c].perm = ds.v_perm[c].p;
    }
    a.G = ds.G; a.Gpad = ds.Gpad; a.pk = ds.pk; a.nsub = ds.nsub;
    for (int d = 0; d < 3; ++d) { a.distinct[d] = ds.distinct[d].p; a.D[d] = ds.D[d]; }
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
inline uint32_t sub_batch_rows(int j, uint32_t remaining) {
    const uint32_t want = kSubBatchRows * (uint32_t)((j + 1) < (int)kSubBatchMaxMul ? (j + 1) : (int)kSubBatchMaxMul);
    return remaining < want + kSubBatchRows / 2 ? remaining : want;  // do not leave a sliver behind
}
inline uint32_t sub_batch_cap(uint32_t Ps) {  // largest sub-batch a shard of Ps rows produces
    uint32_t cap = 0, left = Ps;
    for (int j = 0; left; ++j) { const uint32_t nb = sub_batch_rows(j, left); cap = nb > cap ? nb : cap; left -= nb; }
    return cap ? cap : 1;
}

// Latency path of the host entry point (micro-batches, one GPU): the five pod columns -- or, from the pod table, the
// slot ids -- are packed into one pinned block -> ONE H2D (then the gather, for slots); best and top5 come back in ONE
// D2H; one stream synchronise.  Same kernels.  Slot ids are in range here.  Returns the kernels launched.
int select_small(DeviceState& ds, uint32_t P, const PodSource& src, int32_t* best, int32_t* top5) {
    RPK_CUDA(cudaSetDevice(ds.dev));
    ds.sel_scope.host_wait();
    const size_t in_cap = (size_t)kSmallBatch * 24, out_cap = (size_t)kSmallBatch * 6 * 4;
    ds.h_small.reserve(in_cap + out_cap);
    ds.d_small_in.reserve(in_cap); ds.d_small_out.reserve((size_t)kSmallBatch * 6);
    unsigned char* h = ds.h_small.h;
    DeviceState::Lane& ln = ds.lane[0];
    cudaStream_t st = ln.stream;
    unsigned char* d = ds.d_small_in.p;
    SelectArgs a{};
    int launches = 0;
    if (src.slots) {
        ln.p_req_mem.reserve(kSmallBatch); ln.p_req_vcpu.reserve(kSmallBatch); ln.p_req_ram.reserve(kSmallBatch);
        ln.p_max_price.reserve(kSmallBatch); ln.p_cloud.reserve(kSmallBatch);
        memcpy(h, src.slots, (size_t)P * 4);
        RPK_CUDA(cudaMemcpyAsync(d, h, (size_t)P * 4, cudaMemcpyHostToDevice, st));
        launches += gather_pod_rows(ds, ln, P, (const uint32_t*)d, a, st);
    } else {
        const PodCols& pods = src.cols;
        const size_t o_mem = 0, o_vcpu = (size_t)P * 4, o_ram = (size_t)P * 8, o_price = ((size_t)P * 12 + 7) & ~(size_t)7,
                     o_cloud = o_price + (size_t)P * 8, total = o_cloud + P;
        memcpy(h + o_mem, pods.req_mem, (size_t)P * 4);
        if (pods.req_vcpu) memcpy(h + o_vcpu, pods.req_vcpu, (size_t)P * 4);
        if (pods.req_ram) memcpy(h + o_ram, pods.req_ram, (size_t)P * 4);
        if (pods.max_price) memcpy(h + o_price, pods.max_price, (size_t)P * 8);
        if (pods.cloud) memcpy(h + o_cloud, pods.cloud, P);
        RPK_CUDA(cudaMemcpyAsync(d, h, total, cudaMemcpyHostToDevice, st));
        a.req_mem = (const int32_t*)(d + o_mem); a.req_vcpu = pods.req_vcpu ? (const int32_t*)(d + o_vcpu) : nullptr;
        a.req_ram = pods.req_ram ? (const int32_t*)(d + o_ram) : nullptr; a.max_price = pods.max_price ? (const double*)(d + o_price) : nullptr;
        a.cloud = pods.cloud ? (const uint8_t*)(d + o_cloud) : nullptr;
    }
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


// Buffers of the pipelined host select, sized from the calling thread (peers write into each other's best_full, so
// every GPU's vector must exist before any shard is enqueued).  After the first call of a size this only compares
// capacities.
void reserve_select(rpk_ctx* ctx, uint32_t P, const PodSource& src, bool top5) {
    const int n = (int)ctx->devs.size();
    const PodCols& pods = src.cols;
    const bool all = src.slots != nullptr;  // the gather writes all five columns
    const bool vcpu = all || pods.req_vcpu, ram = all || pods.req_ram, price = all || pods.max_price, cloud = all || pods.cloud;
    for (int s = 0; s < n; ++s) {
        DeviceState& ds = ctx->devs[(size_t)s];
        uint32_t lo, hi; shard_range(P, n, s, &lo, &hi);
        const uint32_t Ps = hi - lo;
        const uint32_t cap = sub_batch_cap(Ps);
        bool grow = P > ds.best_full.cap;
        for (auto& ln : ds.lane) {
            grow = grow || cap > ln.p_req_mem.cap || (vcpu && cap > ln.p_req_vcpu.cap) || (ram && cap > ln.p_req_ram.cap) ||
                   (price && cap > ln.p_max_price.cap) || (cloud && cap > ln.p_cloud.cap) || (all && cap > ln.p_slots.cap) ||
                   (top5 && (size_t)cap * RPK_TOPK > ln.top5.cap);
            if (cap == Ps) break;  // a single sub-batch uses lane 0 only
        }
        if (!grow) continue;
        RPK_CUDA(cudaSetDevice(ds.dev));
        ds.best_full.reserve(P);
        for (auto& ln : ds.lane) {
            ln.p_req_mem.reserve(cap);
            if (vcpu) ln.p_req_vcpu.reserve(cap);
            if (ram) ln.p_req_ram.reserve(cap);
            if (price) ln.p_max_price.reserve(cap);
            if (cloud) ln.p_cloud.reserve(cap);
            if (all) ln.p_slots.reserve(cap);
            if (top5) ln.top5.reserve((size_t)cap * RPK_TOPK);
            if (cap == Ps) break;
        }
    }
}

// One shard's half of the host select: row sub-batches rotate over the lanes; within a lane everything is stream
// ordered (H2D -> kernels -> D2H), across lanes copies and kernels overlap.  ds.ev[0] / ds.ev[3] bracket it on ds.stream;
// the caller synchronises ds.stream.  Slot ids are checked per sub-batch just before their upload: false = an entry
// outside the pod table, and nothing from that sub-batch on was enqueued (the lanes still drain into ds.stream).
bool enqueue_select_shard(rpk_ctx* ctx, int s, uint32_t P, const PodSource& src, int32_t* best, int32_t* top5, uint64_t* launches) {
    const int n = (int)ctx->devs.size();
    DeviceState& ds = ctx->devs[(size_t)s];
    uint32_t lo, hi; shard_range(P, n, s, &lo, &hi);
    RPK_CUDA(cudaSetDevice(ds.dev));
    RPK_CUDA(cudaEventRecord(ds.ev[0], ds.stream));
    for (auto& ln : ds.lane) RPK_CUDA(cudaStreamWaitEvent(ln.stream, ds.ev[0], 0));
    bool ok = true;
    int j = 0;
    for (uint32_t b0 = lo, nb = 0; b0 < hi; b0 += nb, ++j) {
        nb = sub_batch_rows(j, hi - b0);
        DeviceState::Lane& ln = ds.lane[j % DeviceState::kLanes];
        cudaStream_t st = ln.stream;
        SelectArgs a{};
        if (src.slots) {
            if (!slots_below(src.slots + b0, nb, ds.podsN)) { ok = false; break; }
            RPK_CUDA(cudaMemcpyAsync(ln.p_slots.p, src.slots + b0, (size_t)nb * 4, cudaMemcpyHostToDevice, st));
            *launches += (uint64_t)gather_pod_rows(ds, ln, nb, ln.p_slots.p, a, st);
        } else {
            const PodCols& pods = src.cols;
            // rows [b0, b0 + nb) of a column into the lane's buffer; null stays null
            auto upload = [&](auto& buf, const auto* col) -> decltype(buf.p) {
                if (!col) return nullptr;
                RPK_CUDA(cudaMemcpyAsync(buf.p, col + b0, (size_t)nb * sizeof(*col), cudaMemcpyHostToDevice, st));
                return buf.p;
            };
            a.req_mem = upload(ln.p_req_mem, pods.req_mem); a.req_vcpu = upload(ln.p_req_vcpu, pods.req_vcpu);
            a.req_ram = upload(ln.p_req_ram, pods.req_ram); a.max_price = upload(ln.p_max_price, pods.max_price);
            a.cloud = upload(ln.p_cloud, pods.cloud);
        }
        a.P = nb;
        for (int o = 0; o < n; ++o) a.best_out[o] = ctx->devs[(size_t)o].best_full.p;
        a.n_out = n; a.row0 = b0; a.top5 = top5 ? ln.top5.p : nullptr;
        a.self_out = s;  // own vector; finished push blocks / sub-batches are forwarded to the peers
        *launches += (uint64_t)enqueue_select(ds, ln, a, st);
        RPK_CUDA(cudaMemcpyAsync(best + b0, ds.best_full.p + b0, (size_t)nb * 4, cudaMemcpyDeviceToHost, st));
        if (top5) RPK_CUDA(cudaMemcpyAsync(top5 + (size_t)b0 * RPK_TOPK, ln.top5.p, (size_t)nb * RPK_TOPK * 4, cudaMemcpyDeviceToHost, st));
    }
    for (auto& ln : ds.lane) {
        RPK_CUDA(cudaEventRecord(ln.done, ln.stream));
        RPK_CUDA(cudaStreamWaitEvent(ds.stream, ln.done, 0));
    }
    RPK_CUDA(cudaEventRecord(ds.ev[3], ds.stream));
    return ok;
}

// Scratch of a sweep over N records (or list entries) on ds: the look-back state and tickets -- zero between calls by
// construction, zeroed here when (re)allocated -- and the per-warp index stage, its code stage (`codes`) and the
// per-unit counts.
void reserve_sweep_scratch(DeviceState& ds, uint32_t N, bool codes) {
    const uint32_t cap = N ? N : 1;
    const size_t need = status_state_words(ds.sm_count);
    if (need > ds.s_tile_state.cap || !ds.s_misc.p || ds.status_dirty) {
        ds.s_tile_state.reserve(need);
        ds.s_misc.reserve(64);
        RPK_CUDA(cudaMemset(ds.s_tile_state.p, 0, ds.s_tile_state.cap * sizeof(unsigned long long)));
        RPK_CUDA(cudaMemset(ds.s_misc.p, 0, ds.s_misc.cap * sizeof(uint32_t)));
        RPK_CUDA(cudaDeviceSynchronize());
        ds.status_dirty = false;
    }
    ds.s_stage_idx.reserve(cap + 64); ds.s_unit_cnt.reserve(cap / 32 + 2);
    if (codes) ds.s_stage_code.reserve(cap + 64);
}

// the StatusArgs fields of the scratch reserve_sweep_scratch sized
void sweep_scratch_args(const DeviceState& ds, bool codes, StatusArgs& a) {
    a.tile_state = ds.s_tile_state.p; a.tile_counter = ds.s_misc.p;
    a.stage_idx = ds.s_stage_idx.p; a.stage_code = codes ? ds.s_stage_code.p : nullptr; a.unit_cnt = ds.s_unit_cnt.p;
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
    reserve_sweep_scratch(ds, Ns, h.changed_code != nullptr);
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
    sweep_scratch_args(ds, h.changed_code != nullptr, a);
    if (h.slots) { a.slots = ds.s_seed_slots.p; a.col_n = sp.hi - sp.lo; }
    ds.status_dirty = true;
    if (Ns) *launches += (uint64_t)launch_status_diff(a, ds.sm_count, st);
    ds.status_dirty = false;
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

// The pipelined host select of a run_host call: P rows from src into the caller's best and top5 (nullable)
struct HostSelect { uint32_t P; PodSource src; int32_t* best; int32_t* top5; };

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
    if (sel) reserve_select(ctx, sel->P, sel->src, sel->top5 != nullptr);
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
        if (sel) shard_ok[(size_t)s] = enqueue_select_shard(ctx, s, sel->P, sel->src, sel->best, sel->top5, &launches[(size_t)s]);
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
int select_host(rpk_ctx* ctx, uint32_t P, const PodSource& src, int32_t* best, int32_t* top5, const char* who) {
    return guarded(ctx, [&]() -> int {
        bool ok;
        if (ctx->devs.size() == 1 && P <= kSmallBatch) {
            ok = !src.slots || slots_below(src.slots, P, ctx->devs[0].podsN);
            if (ok) {
                ctx->launches += (uint64_t)select_small(ctx->devs[0], P, src, best, top5);
                ctx->stats.last_select_kernel_ms = 0.f; ctx->stats.last_select_total_ms = 0.f;  // single copy: not timed
                count_select(ctx, P, ctx->devs[0].G);
            }
        } else {
            const HostSelect sel{P, src, best, top5};
            ok = run_host(ctx, &sel, nullptr, false);
        }
        return ok ? RPK_OK : fail(ctx, RPK_EINVAL, std::string(who) + ": slot index outside the pod table");
    });
}

// rpk_select_device_gather, and rpk_select_device_gather_top5 with t5 (its own arguments checked, a.top5 then points
// into the local top-5 vector); with src.slots, the rpk_select_slots_device* calls of the same name (a NULL list with
// P > 0 already refused).  The shard is in range.
int select_device_gather(rpk_ctx* ctx, int shard, uint32_t P, const PodSource& src, int n_out, int32_t* const* d_best_full,
                         uint32_t row0, int32_t* d_top5, const Top5Gather* t5, void* stream) {
    DeviceState& ds = ctx->devs[(size_t)shard];
    const PeerGroup& peers = ctx->bind[(size_t)shard];
    cudaStream_t st = stream ? (cudaStream_t)stream : ds.stream;
    if (P == 0) {  // nothing to select, but a bound gather still tells its peers that this (empty) shard is done
        if (n_out <= 1 || peers.n == 0) return RPK_OK;
        return guarded(ctx, [&]() -> int {
            RPK_CUDA(cudaSetDevice(ds.dev));
            const bool tracked = ds.sel_scope.device_begin(st);  // orders the epoch counter after the last gather's
            ctx->launches += (uint64_t)launch_peer_signal(peers, 0, peers.inline_wait != 0, st);
            ds.sel_scope.device_end(st, tracked);
            return RPK_OK;
        });
    }
    if ((!src.slots && !src.cols.req_mem) || !d_best_full || n_out < 1 || n_out > RPK_MAX_GPUS) return fail(ctx, RPK_EINVAL, "rpk_select_device: req_mem_gb and 1..8 output vectors are required");
    for (int o = 0; o < n_out; ++o) if (!d_best_full[o]) return fail(ctx, RPK_EINVAL, "rpk_select_device: NULL output vector");
    if (src.slots && !ds.pods_sized) return fail(ctx, RPK_ESTATE, "rpk_select_slots_device: no pod table on this shard (call rpk_pods_reset first)");
    if (!ds.offers_ready) return fail(ctx, RPK_ESTATE, "rpk_select: no offer table uploaded (call rpk_offers_upload first)");
    return guarded(ctx, [&]() -> int {
        RPK_CUDA(cudaSetDevice(ds.dev));
        DeviceState::Lane& ln = ds.lane[0];
        if (src.slots) {  // the gather's compact columns: allocated on the first call of a size only
            ln.p_req_mem.reserve(P); ln.p_req_vcpu.reserve(P); ln.p_req_ram.reserve(P); ln.p_max_price.reserve(P); ln.p_cloud.reserve(P);
        }
        SelectArgs a{};
        const bool tracked = ds.sel_scope.device_begin(st);  // the gather writes lane 0's columns: after the last select
        if (src.slots) {
            ctx->launches += (uint64_t)gather_pod_rows(ds, ln, P, src.slots, a, st);
        } else {
            const PodCols& c = src.cols;
            a.req_mem = c.req_mem; a.req_vcpu = c.req_vcpu; a.req_ram = c.req_ram; a.max_price = c.max_price; a.cloud = c.cloud;
        }
        a.P = P;
        for (int o = 0; o < n_out; ++o) a.best_out[o] = d_best_full[o];
        a.n_out = n_out; a.row0 = row0;
        a.top5 = t5 ? t5->out[t5->self_out] + (size_t)RPK_TOPK * row0 : d_top5;
        a.self_out = find_local_vector(ctx, shard, ds.dev, n_out, d_best_full);
        if (n_out > 1) a.peers = peers;
        ctx->launches += (uint64_t)enqueue_select(ds, ln, a, st, t5);
        ds.sel_scope.device_end(st, tracked);
        count_select(ctx, P, ds.G);
        return RPK_OK;
    });
}

// rpk_select_device_gather_top5 and rpk_select_slots_device_gather_top5: the top-5 vectors' checks, then the gather.
// The shard is in range.
int select_device_gather_top5(rpk_ctx* ctx, int shard, uint32_t P, const PodSource& src, int n_out, int32_t* const* d_best_full,
                              int32_t* const* d_top5_full, uint32_t row0, void* stream) {
    if (!d_best_full || !d_top5_full || n_out < 1 || n_out > RPK_MAX_GPUS)
        return fail(ctx, RPK_EINVAL, "rpk_select_device_gather_top5: 1..8 best and top-5 vectors are required");
    for (int o = 0; o < n_out; ++o)
        if (!d_best_full[o] || !d_top5_full[o]) return fail(ctx, RPK_EINVAL, "rpk_select_device_gather_top5: NULL output vector");
    if ((uint64_t)P * RPK_TOPK > UINT32_MAX) return fail(ctx, RPK_EINVAL, "rpk_select_device_gather_top5: 5*P does not fit in uint32_t");
    if (!same_phase(n_out, d_top5_full))
        return fail(ctx, RPK_EINVAL, "rpk_select_device_gather_top5: the top-5 vectors differ in 16-byte phase");
    DeviceState& ds = ctx->devs[(size_t)shard];
    Top5Gather t5{};
    const int rc = guarded(ctx, [&]() -> int {
        RPK_CUDA(cudaSetDevice(ds.dev));
        t5.self_out = local_vector(ctx, shard, ds.dev, n_out, d_top5_full);
        return RPK_OK;
    });
    if (rc != RPK_OK) return rc;
    if (t5.self_out < 0) return fail(ctx, RPK_EINVAL, "rpk_select_device_gather_top5: no top-5 vector lives on GPU `shard`");
    for (int o = 0; o < n_out; ++o) t5.out[o] = d_top5_full[o];
    t5.n_out = n_out;
    return select_device_gather(ctx, shard, P, src, n_out, d_best_full, row0, nullptr, &t5, stream);
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
    int rc = guarded(nullptr, [&]() -> int {
        for (int i = 0; i < n_gpus; ++i) {
            const int dev = device_ids ? device_ids[i] : i;
            if (dev < 0 || dev >= count) return fail(nullptr, RPK_EINVAL, "rpk_create: device id out of range");
            for (int j = 0; j < i; ++j) if (ctx->devs[(size_t)j].dev == dev) return fail(nullptr, RPK_EINVAL, "rpk_create: duplicate device id");
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
                if (i == j) continue;
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

int rpk_offers_upload(rpk_ctx* ctx, uint32_t G, const int32_t* mem_gb, const int32_t* vcpu, const int32_t* ram_gb,
                      const double* secure_price, const double* community_price, const uint8_t* flags) {
    if (!ctx) return RPK_EINVAL;
    if (G > 0 && (!mem_gb || !secure_price || !community_price || !flags))
        return fail(ctx, RPK_EINVAL, "rpk_offers_upload: mem_gb, secure_price, community_price and flags are required");
    if (G > (1u << 26)) return fail(ctx, RPK_EINVAL, "rpk_offers_upload: G above 2^26 offers is not supported");
    if (has_int32_max(mem_gb, G) || has_int32_max(vcpu, G) || has_int32_max(ram_gb, G))
        return fail(ctx, RPK_EINVAL, "rpk_offers_upload: offer columns must be < INT32_MAX (requests saturate there)");
    return guarded(ctx, [&]() -> int {
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
            const size_t n = G ? G : 1;
            ds.raw_mem.reserve(n); ds.raw_vcpu.reserve(n); ds.raw_ram.reserve(n); ds.raw_sp.reserve(n); ds.raw_cp.reserve(n); ds.raw_flags.reserve(n);
            if (G) {
                RPK_CUDA(cudaMemcpyAsync(ds.raw_mem.p, mem_gb, (size_t)G * 4, cudaMemcpyHostToDevice, ds.stream));
                if (vcpu) RPK_CUDA(cudaMemcpyAsync(ds.raw_vcpu.p, vcpu, (size_t)G * 4, cudaMemcpyHostToDevice, ds.stream));
                else RPK_CUDA(cudaMemsetAsync(ds.raw_vcpu.p, 0, (size_t)G * 4, ds.stream));
                if (ram_gb) RPK_CUDA(cudaMemcpyAsync(ds.raw_ram.p, ram_gb, (size_t)G * 4, cudaMemcpyHostToDevice, ds.stream));
                else RPK_CUDA(cudaMemsetAsync(ds.raw_ram.p, 0, (size_t)G * 4, ds.stream));
                RPK_CUDA(cudaMemcpyAsync(ds.raw_sp.p, secure_price, (size_t)G * 8, cudaMemcpyHostToDevice, ds.stream));
                RPK_CUDA(cudaMemcpyAsync(ds.raw_cp.p, community_price, (size_t)G * 8, cudaMemcpyHostToDevice, ds.stream));
                RPK_CUDA(cudaMemcpyAsync(ds.raw_flags.p, flags, (size_t)G, cudaMemcpyHostToDevice, ds.stream));
            }
            OfferIngest in{G, ds.raw_mem.p, ds.raw_vcpu.p, ds.raw_ram.p, ds.raw_sp.p, ds.raw_cp.p, ds.raw_flags.p};
            ctx->launches += (uint64_t)launch_offer_ingest(ds, in, ds.stream);
            RPK_CUDA(cudaStreamSynchronize(ds.stream));
        }
        const DeviceState& d0 = ctx->devs[0];
        ctx->stats.select_kernel_kind = d0.pk.bm_words ? 4u : d0.pk.bits ? (d0.pk.pos_bits ? 3u : 2u) : 1u;
        ctx->stats.distinct_mem = d0.D[0]; ctx->stats.distinct_vcpu = d0.D[1]; ctx->stats.distinct_ram = d0.D[2];
        ctx->stats.packed_bits = d0.pk.bits;
        return RPK_OK;
    });
}

int rpk_select_device_gather(rpk_ctx* ctx, int shard, uint32_t P, const int32_t* d_req_mem_gb, const int32_t* d_req_vcpu,
                             const int32_t* d_req_ram_gb, const double* d_max_price, const uint8_t* d_cloud,
                             int n_out, int32_t* const* d_best_full, uint32_t row0, int32_t* d_top5, void* stream) {
    if (!ctx) return RPK_EINVAL;
    if (shard < 0 || (size_t)shard >= ctx->devs.size()) return fail(ctx, RPK_EINVAL, "rpk_select_device: shard out of range");
    const PodSource src{PodCols{d_req_mem_gb, d_req_vcpu, d_req_ram_gb, d_max_price, d_cloud}, nullptr};
    return select_device_gather(ctx, shard, P, src, n_out, d_best_full, row0, d_top5, nullptr, stream);
}

int rpk_select_device_gather_top5(rpk_ctx* ctx, int shard, uint32_t P, const int32_t* d_req_mem_gb, const int32_t* d_req_vcpu,
                                  const int32_t* d_req_ram_gb, const double* d_max_price, const uint8_t* d_cloud, int n_out,
                                  int32_t* const* d_best_full, int32_t* const* d_top5_full, uint32_t row0, void* stream) {
    if (!ctx) return RPK_EINVAL;
    if (shard < 0 || (size_t)shard >= ctx->devs.size()) return fail(ctx, RPK_EINVAL, "rpk_select_device_gather_top5: shard out of range");
    const PodSource src{PodCols{d_req_mem_gb, d_req_vcpu, d_req_ram_gb, d_max_price, d_cloud}, nullptr};
    return select_device_gather_top5(ctx, shard, P, src, n_out, d_best_full, d_top5_full, row0, stream);
}

int rpk_select_device(rpk_ctx* ctx, int shard, uint32_t P, const int32_t* d_req_mem_gb, const int32_t* d_req_vcpu,
                      const int32_t* d_req_ram_gb, const double* d_max_price, const uint8_t* d_cloud, int32_t* d_best,
                      int32_t* d_top5, void* stream) {
    int32_t* outs[1] = {d_best};
    return rpk_select_device_gather(ctx, shard, P, d_req_mem_gb, d_req_vcpu, d_req_ram_gb, d_max_price, d_cloud, 1, outs, 0, d_top5, stream);
}

int rpk_select(rpk_ctx* ctx, uint32_t P, const int32_t* req_mem_gb, const int32_t* req_vcpu, const int32_t* req_ram_gb,
               const double* max_price, const uint8_t* cloud, int32_t* best, int32_t* top5) {
    if (!ctx) return RPK_EINVAL;
    if (P == 0) return RPK_OK;
    if (!req_mem_gb || !best) return fail(ctx, RPK_EINVAL, "rpk_select: req_mem_gb and best are required");
    for (auto& ds : ctx->devs) if (!ds.offers_ready) return fail(ctx, RPK_ESTATE, "rpk_select: no offer table uploaded (call rpk_offers_upload first)");
    return select_host(ctx, P, PodSource{PodCols{req_mem_gb, req_vcpu, req_ram_gb, max_price, cloud}, nullptr}, best, top5, "rpk_select");
}

// ---- pod-requirement table -------------------------------------------------------------------------------

int rpk_pods_reset(rpk_ctx* ctx, uint32_t N) {
    if (!ctx) return RPK_EINVAL;
    for (auto& ds : ctx->devs) ds.pods_sized = false;  // a failure below leaves no table rather than a mix of sizes
    return guarded(ctx, [&]() -> int {
        for (auto& ds : ctx->devs) {
            RPK_CUDA(cudaSetDevice(ds.dev));
            ds.sel_scope.host_wait();  // a device select may still gather from the table
            const size_t cap = N ? N : 1;
            ds.pt_mem.reserve(cap); ds.pt_vcpu.reserve(cap); ds.pt_ram.reserve(cap); ds.pt_max_price.reserve(cap); ds.pt_cloud.reserve(cap);
            ctx->launches += (uint64_t)launch_pod_fill(ds.pods_table(), N, ds.sm_count, ds.stream);
            RPK_CUDA(cudaStreamSynchronize(ds.stream));
            ds.podsN = N;
        }
        for (auto& ds : ctx->devs) ds.pods_sized = true;
        return RPK_OK;
    });
}

int rpk_pods_seed_slots(rpk_ctx* ctx, uint32_t n_slots, const uint32_t* slots, const int32_t* req_mem_gb, const int32_t* req_vcpu,
                        const int32_t* req_ram_gb, const double* max_price, const uint8_t* cloud) {
    if (!ctx) return RPK_EINVAL;
    if (n_slots == 0) return RPK_OK;
    if (!slots || !req_mem_gb) return fail(ctx, RPK_EINVAL, "rpk_pods_seed_slots: slots and req_mem_gb are required");
    if (!ctx->devs[0].pods_sized) return fail(ctx, RPK_ESTATE, "rpk_pods_seed_slots: no pod table (call rpk_pods_reset first)");
    const uint32_t N = ctx->devs[0].podsN;
    for (uint32_t i = 0; i < n_slots; ++i) {
        if (slots[i] >= N) return fail(ctx, RPK_EINVAL, "rpk_pods_seed_slots: slot index outside the pod table");
        if (i > 0 && slots[i] <= slots[i - 1]) return fail(ctx, RPK_EINVAL, "rpk_pods_seed_slots: slots must be strictly ascending");
    }
    return guarded(ctx, [&]() -> int {
        // staging block: [slots : 4n][mem : 4n][vcpu : 4n][ram : 4n][max_price : 8n, 8-byte aligned][cloud : n]
        const size_t n = n_slots, o_mem = 4 * n, o_vcpu = 8 * n, o_ram = 12 * n, o_price = (16 * n + 7) & ~(size_t)7,
                     o_cloud = o_price + 8 * n;
        for (auto& ds : ctx->devs) {  // the table is replicated: every GPU gets every row
            RPK_CUDA(cudaSetDevice(ds.dev));
            ds.sel_scope.host_wait();  // after a device select's gather
            ds.pt_seed.reserve(o_cloud + n);
            unsigned char* d = ds.pt_seed.p;
            auto up = [&](size_t off, const void* col, size_t bytes) -> const unsigned char* {
                if (!col) return nullptr;
                RPK_CUDA(cudaMemcpyAsync(d + off, col, bytes, cudaMemcpyHostToDevice, ds.stream));
                return d + off;
            };
            const uint32_t* d_slots = (const uint32_t*)up(0, slots, 4 * n);
            const PodCols in{(const int32_t*)up(o_mem, req_mem_gb, 4 * n), (const int32_t*)up(o_vcpu, req_vcpu, 4 * n),
                             (const int32_t*)up(o_ram, req_ram_gb, 4 * n), (const double*)up(o_price, max_price, 8 * n),
                             (const uint8_t*)up(o_cloud, cloud, n)};
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
    if (!ctx->devs[0].pods_sized) return fail(ctx, RPK_ESTATE, "rpk_select_slots: no pod table (call rpk_pods_reset first)");
    for (auto& ds : ctx->devs) if (!ds.offers_ready) return fail(ctx, RPK_ESTATE, "rpk_select_slots: no offer table uploaded (call rpk_offers_upload first)");
    return select_host(ctx, n_slots, PodSource{PodCols{}, slots}, best, top5, "rpk_select_slots");
}

int rpk_select_slots_device_gather(rpk_ctx* ctx, int shard, uint32_t n_slots, const uint32_t* d_slots, int n_out,
                                   int32_t* const* d_best_full, uint32_t row0, int32_t* d_top5, void* stream) {
    if (!ctx) return RPK_EINVAL;
    if (shard < 0 || (size_t)shard >= ctx->devs.size()) return fail(ctx, RPK_EINVAL, "rpk_select_slots_device: shard out of range");
    if (n_slots > 0 && !d_slots) return fail(ctx, RPK_EINVAL, "rpk_select_slots_device: d_slots is required");
    return select_device_gather(ctx, shard, n_slots, PodSource{PodCols{}, d_slots}, n_out, d_best_full, row0, d_top5, nullptr, stream);
}

int rpk_select_slots_device_gather_top5(rpk_ctx* ctx, int shard, uint32_t n_slots, const uint32_t* d_slots, int n_out,
                                        int32_t* const* d_best_full, int32_t* const* d_top5_full, uint32_t row0, void* stream) {
    if (!ctx) return RPK_EINVAL;
    if (shard < 0 || (size_t)shard >= ctx->devs.size()) return fail(ctx, RPK_EINVAL, "rpk_select_slots_device_gather_top5: shard out of range");
    if (n_slots > 0 && !d_slots) return fail(ctx, RPK_EINVAL, "rpk_select_slots_device_gather_top5: d_slots is required");
    return select_device_gather_top5(ctx, shard, n_slots, PodSource{PodCols{}, d_slots}, n_out, d_best_full, d_top5_full, row0, stream);
}

int rpk_select_slots_device(rpk_ctx* ctx, int shard, uint32_t n_slots, const uint32_t* d_slots, int32_t* d_best, int32_t* d_top5,
                            void* stream) {
    int32_t* outs[1] = {d_best};
    return rpk_select_slots_device_gather(ctx, shard, n_slots, d_slots, 1, outs, 0, d_top5, stream);
}

// ---- cross-process peer vectors (CUDA IPC) ---------------------------------------------------------------

int rpk_ipc_alloc(rpk_ctx* ctx, int shard, size_t bytes, void** d_ptr, unsigned char handle_out[64]) {
    if (!ctx) return RPK_EINVAL;
    if (shard < 0 || (size_t)shard >= ctx->devs.size() || !d_ptr || !handle_out || bytes == 0) return fail(ctx, RPK_EINVAL, "rpk_ipc_alloc: bad argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle is 64 bytes");
    return guarded(ctx, [&]() -> int {
        RPK_CUDA(cudaSetDevice(ctx->devs[(size_t)shard].dev));
        void* p = nullptr;
        RPK_CUDA(cudaMalloc(&p, bytes));
        RPK_CUDA(cudaMemset(p, 0, bytes));
        cudaIpcMemHandle_t h;
        cudaError_t e = cudaIpcGetMemHandle(&h, p);
        if (e != cudaSuccess) { cudaFree(p); RPK_CUDA(e); }
        memcpy(handle_out, &h, 64);
        ctx->ipc_owned.emplace_back(shard, p);
        *d_ptr = p;
        return RPK_OK;
    });
}

int rpk_ipc_open(rpk_ctx* ctx, int shard, const unsigned char handle[64], void** d_peer_ptr) {
    if (!ctx) return RPK_EINVAL;
    if (shard < 0 || (size_t)shard >= ctx->devs.size() || !handle || !d_peer_ptr) return fail(ctx, RPK_EINVAL, "rpk_ipc_open: bad argument");
    return guarded(ctx, [&]() -> int {
        RPK_CUDA(cudaSetDevice(ctx->devs[(size_t)shard].dev));
        cudaIpcMemHandle_t h;
        memcpy(&h, handle, 64);
        void* p = nullptr;
        RPK_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
        ctx->ipc_mapped.emplace_back(shard, p);
        *d_peer_ptr = p;
        return RPK_OK;
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
    return guarded(ctx, [&]() -> int {
        RPK_CUDA(cudaSetDevice(ctx->devs[(size_t)shard].dev));
        RPK_CUDA(cudaIpcCloseMemHandle(d_peer_ptr));
        return RPK_OK;
    });
}

int rpk_ipc_free(rpk_ctx* ctx, int shard, void* d_ptr) {
    if (!ctx) return RPK_EINVAL;
    if (!drop_entry(ctx->ipc_owned, shard, d_ptr)) return fail(ctx, RPK_EINVAL, "rpk_ipc_free: pointer was not allocated by this ctx");
    return guarded(ctx, [&]() -> int {
        RPK_CUDA(cudaSetDevice(ctx->devs[(size_t)shard].dev));
        RPK_CUDA(cudaFree(d_ptr));
        return RPK_OK;
    });
}

int rpk_peer_fence(rpk_ctx* ctx, int shard, int n, uint32_t* const* d_flags, int my_rank, uint32_t epoch, void* stream) {
    if (!ctx) return RPK_EINVAL;
    if (shard < 0 || (size_t)shard >= ctx->devs.size() || n < 1 || n > RPK_MAX_GPUS || !d_flags || my_rank < 0 || my_rank >= n)
        return fail(ctx, RPK_EINVAL, "rpk_peer_fence: bad argument");
    for (int r = 0; r < n; ++r) if (!d_flags[r]) return fail(ctx, RPK_EINVAL, "rpk_peer_fence: NULL flag array");
    DeviceState& ds = ctx->devs[(size_t)shard];
    return guarded(ctx, [&]() -> int {
        RPK_CUDA(cudaSetDevice(ds.dev));
        PeerGroup g{};
        for (int r = 0; r < n; ++r) g.flags[r] = d_flags[r];
        g.n = n; g.my_rank = my_rank;
        ctx->launches += (uint64_t)launch_peer_signal(g, epoch, true, stream ? (cudaStream_t)stream : ds.stream);
        return RPK_OK;
    });
}

int rpk_peer_bind(rpk_ctx* ctx, int shard, int n, uint32_t* const* d_flags, int my_rank) {
    if (!ctx) return RPK_EINVAL;
    if (shard < 0 || (size_t)shard >= ctx->devs.size() || n < 0 || n > RPK_MAX_GPUS || (n > 0 && (!d_flags || my_rank < 0 || my_rank >= n)))
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
    if (shard < 0 || (size_t)shard >= ctx->devs.size()) return fail(ctx, RPK_EINVAL, "rpk_peer_inline_wait: shard out of range");
    ctx->bind[(size_t)shard].inline_wait = on ? 1 : 0;
    return RPK_OK;
}

int rpk_peer_wait(rpk_ctx* ctx, int shard, unsigned what, void* stream) {
    if (!ctx) return RPK_EINVAL;
    if (shard < 0 || (size_t)shard >= ctx->devs.size() || (what & ~3u) || !what) return fail(ctx, RPK_EINVAL, "rpk_peer_wait: bad argument");
    if (ctx->bind[(size_t)shard].n == 0) return fail(ctx, RPK_ESTATE, "rpk_peer_wait: no flags bound (rpk_peer_bind)");
    DeviceState& ds = ctx->devs[(size_t)shard];
    return guarded(ctx, [&]() -> int {
        RPK_CUDA(cudaSetDevice(ds.dev));
        ctx->launches += (uint64_t)launch_peer_wait(ctx->bind[(size_t)shard], what, stream ? (cudaStream_t)stream : ds.stream);
        return RPK_OK;
    });
}

/* test / integration hook: device pointer of GPU `shard`'s copy of the last full assignment vector */
const int32_t* rpk_best_device_ptr(const rpk_ctx* ctx, int shard) {
    if (!ctx || shard < 0 || (size_t)shard >= ctx->devs.size()) return nullptr;
    return ctx->devs[(size_t)shard].best_full.p;
}

// ---- status --------------------------------------------------------------------------------------------

static int check_stride(rpk_ctx* ctx, uint32_t stride) {
    if (stride < 16 || stride > 256 || (stride & 15)) return fail(ctx, RPK_EINVAL, "status stride must be a multiple of 16 in [16, 256]");
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

namespace {

// The argument checks of a whole-table host sweep (rpk_status_diff*, rpk_status_seed, rpk_tick; `who` names the entry
// point in the messages).  The first sweep of a ctx sizes the tracked table to its N.
int check_sweep(rpk_ctx* ctx, const StatusHostArgs& h, const char* who) {
    const std::string w(who);
    if (int rc = check_stride(ctx, h.stride)) return rc;
    if (h.N > 0 && !h.records) return fail(ctx, RPK_EINVAL, w + ": records is NULL");
    if (h.report && (!h.n_changed || (h.N > 0 && !h.changed_idx))) return fail(ctx, RPK_EINVAL, w + ": changed_idx and n_changed are required");
    if (!ctx->devs[0].status_sized) { if (int rc = rpk_status_reset(ctx, h.N)) return rc; }
    if (ctx->devs[0].statusN != h.N) return fail(ctx, RPK_ESTATE, w + ": N differs from the tracked table (call rpk_status_reset to resize)");
    return RPK_OK;
}

int status_host(rpk_ctx* ctx, const StatusHostArgs& h) {
    if (!ctx) return RPK_EINVAL;
    if (int rc = check_sweep(ctx, h, "rpk_status_diff")) return rc;
    return guarded(ctx, [&]() -> int { run_host(ctx, nullptr, &h, false); return RPK_OK; });
}

}  // namespace

int rpk_status_diff(rpk_ctx* ctx, uint32_t N, const uint8_t* records, uint32_t stride, uint32_t* changed_idx,
                    uint32_t* n_changed, uint64_t* hashes_out) {
    return status_host(ctx, StatusHostArgs{N, records, stride, changed_idx, nullptr, n_changed, hashes_out, true});
}

int rpk_status_diff_codes(rpk_ctx* ctx, uint32_t N, const uint8_t* records, uint32_t stride, uint32_t* changed_idx,
                          uint16_t* changed_code, uint32_t* n_changed, uint64_t* hashes_out) {
    return status_host(ctx, StatusHostArgs{N, records, stride, changed_idx, changed_code, n_changed, hashes_out, true});
}

int rpk_status_seed(rpk_ctx* ctx, uint32_t N, const uint8_t* records, uint32_t stride) {
    return status_host(ctx, StatusHostArgs{N, records, stride, nullptr, nullptr, nullptr, nullptr, false});
}

int rpk_status_seed_slots(rpk_ctx* ctx, uint32_t n_slots, const uint32_t* slots, const uint8_t* records, uint32_t stride) {
    if (!ctx) return RPK_EINVAL;
    if (int rc = check_stride(ctx, stride)) return rc;
    if (n_slots == 0) return RPK_OK;
    if (!slots || !records) return fail(ctx, RPK_EINVAL, "rpk_status_seed_slots: slots and records are required");
    if (!ctx->devs[0].status_sized) return fail(ctx, RPK_ESTATE, "rpk_status_seed_slots: no tracked table (call rpk_status_reset first)");
    const uint32_t N = ctx->devs[0].statusN;
    for (uint32_t i = 0; i < n_slots; ++i) if (slots[i] >= N) return fail(ctx, RPK_EINVAL, "rpk_status_seed_slots: slot index outside the tracked table");
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
    if (int rc = check_stride(ctx, stride)) return rc;
    if (!n_changed) return fail(ctx, RPK_EINVAL, "rpk_status_diff_slots: n_changed is required");
    if (n_slots == 0) { *n_changed = 0; return RPK_OK; }
    if (!slots || !records || !changed_idx) return fail(ctx, RPK_EINVAL, "rpk_status_diff_slots: slots, records and changed_idx are required");
    if (!ctx->devs[0].status_sized) return fail(ctx, RPK_ESTATE, "rpk_status_diff_slots: no tracked table (call rpk_status_reset first)");
    const uint32_t N = ctx->devs[0].statusN;
    for (uint32_t i = 0; i < n_slots; ++i) {
        if (slots[i] >= N) return fail(ctx, RPK_EINVAL, "rpk_status_diff_slots: slot index outside the tracked table");
        if (i > 0 && slots[i] <= slots[i - 1]) return fail(ctx, RPK_EINVAL, "rpk_status_diff_slots: slots must be strictly ascending");
    }
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
    if (P > 0) for (auto& ds : ctx->devs) if (!ds.offers_ready) return fail(ctx, RPK_ESTATE, "rpk_tick: no offer table uploaded (call rpk_offers_upload first)");
    const StatusHostArgs h{N, records, stride, changed_idx, changed_code, n_changed, nullptr, true};
    if (int rc = check_sweep(ctx, h, "rpk_tick")) return rc;
    const HostSelect sel{P, PodSource{PodCols{req_mem_gb, req_vcpu, req_ram_gb, max_price, cloud}, nullptr}, best, top5};
    return guarded(ctx, [&]() -> int { run_host(ctx, P > 0 ? &sel : nullptr, &h, true); return RPK_OK; });
}

namespace {
int status_device(rpk_ctx* ctx, int shard, uint32_t N, const uint8_t* d_records, uint32_t stride, uint64_t* d_hash_prev,
                  uint32_t idx_base, uint32_t* d_changed_idx, uint16_t* d_changed_code, uint32_t* d_n_changed, int n_out,
                  uint32_t* const* d_xchg, uint32_t cap, int my_rank, void* stream, const uint32_t* d_slots = nullptr, uint32_t col_n = 0) {
    // d_slots: N is the list's length, and the column (col_n rows) holds global slots [idx_base, idx_base + col_n)
    if (!ctx) return RPK_EINVAL;
    if (shard < 0 || (size_t)shard >= ctx->devs.size()) return fail(ctx, RPK_EINVAL, "rpk_status_diff_device: shard out of range");
    if (int rc = check_stride(ctx, stride)) return rc;
    if (N > 0 && (!d_records || !d_hash_prev)) return fail(ctx, RPK_EINVAL, "rpk_status_diff_device: NULL column");
    if (n_out == 0 && N > 0 && !d_changed_idx) return fail(ctx, RPK_EINVAL, "rpk_status_diff_device: d_changed_idx is NULL");
    if (!d_n_changed) return fail(ctx, RPK_EINVAL, "rpk_status_diff_device: d_n_changed is NULL");
    if (((uintptr_t)d_records | (uintptr_t)d_hash_prev) & 15) return fail(ctx, RPK_EINVAL, "rpk_status_diff_device: d_records and d_hash_prev must be 16-byte aligned");
    if (n_out < 0 || n_out > RPK_MAX_GPUS || (n_out > 0 && (!d_xchg || my_rank < 0 || my_rank >= n_out || N > cap)))
        return fail(ctx, RPK_EINVAL, "rpk_status_diff_device_gather: bad exchange arguments (N must fit the per-rank capacity)");
    for (int o = 0; o < n_out; ++o) if (!d_xchg[o]) return fail(ctx, RPK_EINVAL, "rpk_status_diff_device_gather: NULL exchange buffer");
    if (d_slots == nullptr && col_n != 0) return fail(ctx, RPK_EINVAL, "rpk_status_diff_slots_device: d_slots is NULL");
    if ((uint64_t)idx_base + col_n > (1ull << 32)) return fail(ctx, RPK_EINVAL, "rpk_status_diff_slots_device: idx_base + N exceeds the slot range");
    DeviceState& ds = ctx->devs[(size_t)shard];
    return guarded(ctx, [&]() -> int {
        RPK_CUDA(cudaSetDevice(ds.dev));
        const bool codes = d_changed_code || n_out > 0;
        reserve_sweep_scratch(ds, N, codes);
        StatusArgs a{};
        a.records = d_records; a.stride = stride; a.N = N; a.hash_prev = d_hash_prev; a.hash_out = nullptr;
        a.changed_idx = d_changed_idx; a.changed_code = d_changed_code; a.n_changed = d_n_changed; a.idx_base = idx_base;
        sweep_scratch_args(ds, codes, a);
        a.n_out = n_out;
        a.slots = d_slots; a.col_n = col_n;
        for (int o = 0; o < n_out; ++o) {  // rank o's buffer: [counts : 8 words][n_out index regions of cap][n_out code regions of cap u16]
            uint32_t* base = d_xchg[o];
            a.out_count[o] = base;
            a.out_idx[o] = base + 8 + (size_t)my_rank * cap;
            a.out_code[o] = reinterpret_cast<uint16_t*>(base + 8 + (size_t)n_out * cap) + (size_t)my_rank * cap;
        }
        if (n_out > 0) a.peers = ctx->bind[(size_t)shard];
        a.peers.my_rank = my_rank;  // the sweep fills and signals under the rank its call names
        cudaStream_t st = stream ? (cudaStream_t)stream : ds.stream;
        const bool tracked = ds.status_scope.device_begin(st);
        ds.status_dirty = true;
        ctx->launches += (uint64_t)launch_status_diff(a, ds.sm_count, st);
        ds.status_dirty = false;
        ds.status_scope.device_end(st, tracked);
        ctx->stats.status_calls += 1; ctx->stats.status_records += N;
        return RPK_OK;
    });
}
}  // namespace

int rpk_status_diff_device(rpk_ctx* ctx, int shard, uint32_t N, const uint8_t* d_records, uint32_t stride,
                           uint64_t* d_hash_prev, uint32_t* d_changed_idx, uint32_t* d_n_changed, void* stream) {
    return status_device(ctx, shard, N, d_records, stride, d_hash_prev, 0, d_changed_idx, nullptr, d_n_changed, 0, nullptr, 0, 0, stream);
}

int rpk_status_diff_device_codes(rpk_ctx* ctx, int shard, uint32_t N, const uint8_t* d_records, uint32_t stride,
                                 uint64_t* d_hash_prev, uint32_t* d_changed_idx, uint16_t* d_changed_code, uint32_t* d_n_changed, void* stream) {
    return status_device(ctx, shard, N, d_records, stride, d_hash_prev, 0, d_changed_idx, d_changed_code, d_n_changed, 0, nullptr, 0, 0, stream);
}

int rpk_status_diff_slots_device(rpk_ctx* ctx, int shard, uint32_t N, uint32_t idx_base, uint32_t n_slots,
                                 const uint32_t* d_slots, const uint8_t* d_records, uint32_t stride, uint64_t* d_hash_prev,
                                 uint32_t* d_changed_idx, uint16_t* d_changed_code, uint32_t* d_n_changed, void* stream) {
    if (ctx && n_slots > 0 && !d_slots) return fail(ctx, RPK_EINVAL, "rpk_status_diff_slots_device: d_slots is NULL");
    return status_device(ctx, shard, n_slots, d_records, stride, d_hash_prev, idx_base, d_changed_idx, d_changed_code, d_n_changed,
                         0, nullptr, 0, 0, stream, n_slots > 0 ? d_slots : nullptr, n_slots > 0 ? N : 0);
}

size_t rpk_xchg_bytes(int n_ranks, uint32_t cap) { return (size_t)(8 + (size_t)n_ranks * cap) * 4 + (size_t)n_ranks * cap * 2 + 16; }

int rpk_status_diff_device_gather(rpk_ctx* ctx, int shard, uint32_t N, const uint8_t* d_records, uint32_t stride,
                                  uint64_t* d_hash_prev, uint32_t idx_base, int n_ranks, uint32_t* const* d_xchg, uint32_t cap,
                                  int my_rank, uint32_t* d_n_changed, void* stream) {
    return status_device(ctx, shard, N, d_records, stride, d_hash_prev, idx_base, nullptr, nullptr, d_n_changed, n_ranks, d_xchg, cap, my_rank, stream);
}

// n_slots bounds what a region receives (list order is not checked on the device), so it is what must fit the capacity
int rpk_status_diff_slots_device_gather(rpk_ctx* ctx, int shard, uint32_t N, uint32_t idx_base, uint32_t n_slots,
                                        const uint32_t* d_slots, const uint8_t* d_records, uint32_t stride,
                                        uint64_t* d_hash_prev, int n_ranks, uint32_t* const* d_xchg, uint32_t cap,
                                        int my_rank, uint32_t* d_n_changed, void* stream) {
    if (ctx && n_slots > 0 && !d_slots) return fail(ctx, RPK_EINVAL, "rpk_status_diff_slots_device_gather: d_slots is NULL");
    if (ctx && n_ranks < 1) return fail(ctx, RPK_EINVAL, "rpk_status_diff_slots_device_gather: n_ranks must be 1..8");
    return status_device(ctx, shard, n_slots, d_records, stride, d_hash_prev, idx_base, nullptr, nullptr, d_n_changed, n_ranks,
                         d_xchg, cap, my_rank, stream, n_slots > 0 ? d_slots : nullptr, n_slots > 0 ? N : 0);
}

int rpk_stats_get(const rpk_ctx* ctx, rpk_stats* out) {
    if (!ctx || !out) return RPK_EINVAL;
    *out = ctx->stats;
    return RPK_OK;
}

uint64_t rpk_launch_count(const rpk_ctx* ctx) { return ctx ? ctx->launches : 0; }

}  // extern "C"
