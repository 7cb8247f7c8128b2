/*
 * rpk.h -- C-ABI of the H100 batch scheduling engine ("rpk") for the RunPod virtual kubelet.
 *
 * This is the whole drop-in boundary: what a cgo binding under pkg/virtual_kubelet calls in place of
 * the two Go loop bodies on the hot path (INTEGRATION.md shows the binding):
 *
 *   reference (paths relative to pkg/virtual_kubelet/ of the reference) replaced by
 *   ------------------------------------------------------------------------  ---------------------
 *   Client.GetGPUTypes filter loop          runpod_client.go:465-495          rpk_offers_upload +
 *   sort.Slice by price + take <=5          runpod_client.go:497-509          rpk_select
 *   per-pod call site                        runpod_client.go:1281             (one call per batch of pods)
 *   updateAllPodStatuses diff predicate      kubelet.go:857-880                rpk_status_diff
 *   previous-state table (InstanceInfo)      runpod_client.go:98-109,          device-resident hash column,
 *                                            kubelet.go:41-45                  rpk_status_seed / _reset
 *
 * Conventions
 *   - plain C, no torch / C++ types; every pointer is CALLER-OWNED memory borrowed for the duration of
 *     the call only (cgo pointer rule: C must not retain Go pointers).  Device memory is ctx-owned.
 *   - return value 0 = ok, <0 = error code below; never aborts, never throws across the boundary; the
 *     message is available from rpk_last_error().
 *   - a ctx is NOT re-entrant: serialise calls on one ctx (the Go wrapper holds a mutex -- at least four
 *     goroutines can reach it: kubelet.go:384, 718, 292, 734).  Every call binds its CUDA device itself
 *     (goroutines migrate between OS threads).
 *   - there is NO CPU fallback: without a usable sm_90 device rpk_create fails and the provider must
 *     refuse to start.
 *   - "host" entry points take host pointers (pageable or pinned; pinned from rpk_host_alloc is faster);
 *     "_device" entry points take device pointers on the shard's GPU and enqueue on the given stream
 *     without synchronising it.
 *   - Ordering.  The calls on one shard share ctx-owned buffers in two scopes: the select scope (the offer table, the
 *     pod table and the select scratch) and the status scope (the sweep scratch).  A _device call issued on another
 *     stream than the last _device call of its scope first waits for that call, so any streams may be used.  A host
 *     call waits for the last _device call of its scopes before it touches anything, and returns after its own work is
 *     done; the caller needs no synchronise between the two.  Select scope: rpk_offers_upload, rpk_pods_reset,
 *     rpk_pods_seed_slots, rpk_select, rpk_select_slots, and rpk_tick with P > 0.  Status scope: rpk_status_diff,
 *     rpk_status_diff_codes, rpk_status_seed, rpk_status_diff_slots and rpk_tick.  rpk_status_reset and
 *     rpk_status_seed_slots touch only buffers no _device call uses and do not wait.  A _device call inside a stream
 *     capture neither waits nor is waited for (keep each captured entry point on one stream), and the library does
 *     not see replays of a captured graph: a caller that replays a captured device step orders its host calls after
 *     the replay itself.
 */
#ifndef RPK_H_
#define RPK_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RPK_ABI_VERSION 2

#define RPK_OK 0
#define RPK_EINVAL (-1)  /* bad argument (NULL, size, INT32_MAX in an offer column, ...) */
#define RPK_ECUDA (-2)   /* a CUDA call failed; message has the CUDA error string */
#define RPK_ENOMEM (-3)  /* host or device allocation failed */
#define RPK_ESTATE (-4)  /* call order: select before offers_upload, diff with other N than reset, ... */
#define RPK_ENODEV (-5)  /* no usable sm_90 device */

/* cloud column values: validateCloudType's result (runpod_client.go:1115-1134).  Any other byte behaves
 * like a cloudType string that is neither (runpod_client.go:469-475): nothing is feasible. */
#define RPK_CLOUD_SECURE 0
#define RPK_CLOUD_COMMUNITY 1

/* flags column bits: GPUType.SecureCloud / GPUType.CommunityCloud (runpod_client.go:87,89) */
#define RPK_FLAG_SECURE_CLOUD 1u
#define RPK_FLAG_COMMUNITY_CLOUD 2u

#define RPK_TOPK 5              /* "Take up to 5 GPUs", runpod_client.go:502-509 */
#define RPK_DEFAULT_MAX_PRICE 0.5 /* DefaultMaxPrice, runpod_client.go:48 */
#define RPK_MAX_GPUS 8

typedef struct rpk_ctx rpk_ctx;

typedef struct rpk_stats {
    uint64_t select_calls;        /* rpk_select + rpk_select_slots + rpk_select_device + rpk_select_slots_device */
    uint64_t offer_scores;        /* sum of P*G over those calls */
    uint64_t status_calls;
    uint64_t status_records;      /* sum of N */
    float last_select_kernel_ms;  /* 0: rpk_select overlaps copies and kernels (sub-batch pipeline), only the total is meaningful */
    float last_select_total_ms;   /* rpk_select: H2D + kernels + D2H of the last call (0 on the micro-batch latency path) */
    float last_status_kernel_ms;
    float last_status_total_ms;
    uint32_t select_kernel_kind;  /* 0 none, 1 generic int32 compare, 2 packed rank fields + select,
                                     3 packed + embedded position (min), 4 bit-sliced threshold masks */
    uint32_t n_gpus;
    uint32_t distinct_mem, distinct_vcpu, distinct_ram; /* distinct offer values found at upload */
    uint32_t packed_bits;         /* bits used by the packed offer word incl. guards (<=32), 0 if generic */
} rpk_stats;

/* ---- lifecycle ------------------------------------------------------------------------------------ */

/* n_gpus in [1, RPK_MAX_GPUS]; device_ids == NULL means 0..n_gpus-1.  With n_gpus > 1 (one host process
 * driving a whole box, the shape a Go kubelet has) pod rows / status slots are split into contiguous
 * shards, one per GPU, and every GPU writes its shard of the assignment vector straight into all peers'
 * copies over NVLink (peer access is enabled here). */
int rpk_create(int n_gpus, const int* device_ids, rpk_ctx** out);
void rpk_destroy(rpk_ctx* ctx);
/* ctx-owned string, valid until the next call on that ctx; ctx == NULL returns the last rpk_create error
 * of the calling thread. */
const char* rpk_last_error(const rpk_ctx* ctx);
int rpk_abi_version(void);

/* pinned host memory for callers that want full-speed H2D/D2H (Go: C.rpk_host_alloc-backed slices) */
void* rpk_host_alloc(size_t bytes);
void rpk_host_free(void* p);

/* ---- offer table: []GPUType as struct-of-arrays (runpod_client.go:83-95) ------------------------- */

/* Copies the G-row table to every GPU of the ctx and prepares the two per-cloud views (sorted by price,
 * ties by offer index) the select kernels consume.  vcpu / ram_gb may be NULL (= all 0: the reference has
 * no such fields).  Prices are the Go float64 values, compared with IEEE semantics on the device
 * (price > 0 && price < maxPrice, runpod_client.go:478).  mem_gb/vcpu/ram_gb must be < INT32_MAX.
 * Replaces the per-pod GraphQL decode of the same table (runpod_client.go:447-455). */
int rpk_offers_upload(rpk_ctx* ctx, uint32_t G, const int32_t* mem_gb, const int32_t* vcpu, const int32_t* ram_gb,
                      const double* secure_price, const double* community_price, const uint8_t* flags);

/* ---- selection: P pods x G offers ----------------------------------------------------------------- */

/* For pod row p: feasible(g) = cloud ok && price > 0 && price < max_price[p] && mem_gb[g] >= req_mem_gb[p]
 * && vcpu[g] >= req_vcpu[p] && ram_gb[g] >= req_ram_gb[p]; best[p] = the feasible offer with the lowest
 * price, ties to the lowest offer index, or -1 (an empty gpuTypeIds is not an error,
 * runpod_client.go:511-517).  top5 (nullable, P*5, -1 padded) is the whole gpuTypeIds list in order.
 * NULL req_vcpu / req_ram_gb = 0; NULL max_price = 0.5 for every pod (the reference's only behaviour,
 * runpod_client.go:1281); NULL cloud = SECURE.  P == 0 is a no-op. */
int rpk_select(rpk_ctx* ctx, uint32_t P, const int32_t* req_mem_gb, const int32_t* req_vcpu,
               const int32_t* req_ram_gb, const double* max_price, const uint8_t* cloud, int32_t* best,
               int32_t* top5);

/* ---- pod-requirement table: the selection over a list of pending slots ---------------------------------- */

/* processPendingPods (kubelet.go:747-814) retries every tracked pod that is still Pending without a RunPod id, every
 * 30 s, and its columns are usually the same as on the last tick.  The pod table keeps the five columns of every
 * tracked slot on the device (the slot ids the caller gives the status table), so a tick seeds the rows that changed
 * and selects by slot id: 4 bytes up per pending pod instead of 21.
 *
 * (Re)size the pod table to N slots on every GPU of the ctx and set every row to the columns of a pod with no
 * annotations: req_mem_gb 16 (extractGPUMemory(""), runpod_client.go:1182), vcpu 0, ram 0, max_price 0.5, SECURE.
 * Independent of rpk_status_reset.  The table is replicated: 21 bytes x N on each GPU. */
int rpk_pods_reset(rpk_ctx* ctx, uint32_t N);
/* Row slots[i] := element i of each column.  Columns may be NULL exactly where rpk_select's may, with the same defaults
 * (req_mem_gb is required).  slots must be strictly ascending and < N of the pod table (else RPK_EINVAL, nothing
 * written; no pod table: RPK_ESTATE).  Rows not listed are not touched.  Every GPU of the ctx gets the rows.
 * n_slots == 0 is a no-op. */
int rpk_pods_seed_slots(rpk_ctx* ctx, uint32_t n_slots, const uint32_t* slots, const int32_t* req_mem_gb,
                        const int32_t* req_vcpu, const int32_t* req_ram_gb, const double* max_price, const uint8_t* cloud);
/* rpk_select over rows of the pod table: best[i] / top5[5i, 5i+5) (top5 nullable) are what rpk_select returns for the
 * row held at slot slots[i], bit for bit.  The list may be in any order and may repeat a slot.  An entry >= N of the
 * pod table: RPK_EINVAL, best and top5 unspecified, no table or offer state changed (each sub-batch's part of the list
 * is checked just before its upload).  No pod table or no offer table: RPK_ESTATE.  Counts as one select in rpk_stats
 * (select_calls, offer_scores += n_slots * G).  n_slots == 0 is a no-op. */
int rpk_select_slots(rpk_ctx* ctx, uint32_t n_slots, const uint32_t* slots, int32_t* best, int32_t* top5);

/* Same on device-resident columns of GPU `shard` (index into the ctx's device list), enqueued on `stream`
 * (a cudaStream_t; NULL = the ctx's own stream for that shard; pass cudaStreamLegacy (0x1) for the legacy
 * default stream).  Does not synchronise.  d_best must hold
 * P int32; d_top5 is nullable.  Used by one-process-per-GPU callers that shard pod rows themselves. */
int rpk_select_device(rpk_ctx* ctx, int shard, uint32_t P, const int32_t* d_req_mem_gb, const int32_t* d_req_vcpu,
                      const int32_t* d_req_ram_gb, const double* d_max_price, const uint8_t* d_cloud,
                      int32_t* d_best, int32_t* d_top5, void* stream);

/* Shard + all-gather: the shard's P results end up at [row0, row0+P) of EVERY vector in d_best_full[0..n_out)
 * -- the caller's own full-length vector and its peers' (peer-mapped device pointers: cudaDeviceEnablePeerAccess
 * in one process, cudaIpcOpenMemHandle across processes).  The select kernels write the vector that lives on
 * GPU `shard`; a copy kernel launched behind them pushes the finished slice into the other vectors with 16-byte
 * stores over NVLink, so no collective follows; the caller only needs a barrier (rpk_peer_fence) before reading
 * a peer-written vector.  All vectors must share the slice's 16-byte alignment (same offset from cudaMalloc'ed
 * bases); if none of them lives on GPU `shard`, or the alignments differ, every result is stored into all
 * vectors directly from the select epilogue instead (slower, same result).  After one call of a given size the
 * function only enqueues launches, so it can be captured in a CUDA graph. */
int rpk_select_device_gather(rpk_ctx* ctx, int shard, uint32_t P, const int32_t* d_req_mem_gb,
                             const int32_t* d_req_vcpu, const int32_t* d_req_ram_gb, const double* d_max_price,
                             const uint8_t* d_cloud, int n_out, int32_t* const* d_best_full, uint32_t row0,
                             int32_t* d_top5, void* stream);

/* The same gather carrying the whole gpuTypeIds lists: one-process-per-GPU callers that deploy with the list (as
 * GetGPUTypes + PrepareRunPodParameters do, runpod_client.go:497-509, :1339) get every pod's list without a second
 * collective.
 *   - Outputs: the shard's results land at [row0, row0+P) of every d_best_full[o], exactly as rpk_select_device_gather
 *     puts them (same rules, direct-store fallback included); its lists land at elements [5*row0, 5*(row0+P)) of every
 *     d_top5_full[o], in rpk_select's top5 order and -1 padding.  n_out counts both arrays.
 *   - Placement: one of the d_top5_full vectors must live on GPU `shard` and all of them must share its 16-byte phase;
 *     the top-5 kernel writes that one, and the 16-byte push kernel copies the finished lists to the others.
 *   - One signal: with flags bound (rpk_peer_bind) and n_out > 1 the call signals the select epoch ONCE, behind the
 *     lists' push -- after both slices have reached every vector -- so a peer past rpk_peer_wait(what = 1) or the inline
 *     wait can read both.  The flag words move exactly as for rpk_select_device_gather (+1 on word my_rank of every
 *     peer and on word 32).  P == 0 signals and writes nothing.
 *   - RPK_EINVAL, before anything is enqueued and without signalling: no top-5 vector on GPU `shard`, top-5 vectors of
 *     different 16-byte phase, a NULL vector pointer, n_out outside 1..8, or 5*P beyond uint32_t.
 *   - After one call of a given size the function only enqueues launches (CUDA-graph capturable). */
int rpk_select_device_gather_top5(rpk_ctx* ctx, int shard, uint32_t P, const int32_t* d_req_mem_gb,
                                  const int32_t* d_req_vcpu, const int32_t* d_req_ram_gb, const double* d_max_price,
                                  const uint8_t* d_cloud, int n_out, int32_t* const* d_best_full,
                                  int32_t* const* d_top5_full, uint32_t row0, void* stream);

/* The three calls above over rows of the pod table, for one-process-per-GPU callers: the pending pods are a device list
 * of slot ids instead of five device columns (4 bytes per pod instead of 21; the table is seeded from the host with
 * rpk_pods_seed_slots as the rows change).
 *   - Rows: output row i is what rpk_select_slots returns for list entry i, bit for bit.  The row is read from GPU
 *     `shard`'s copy of the ctx's pod table; the table is replicated, so every shard of a multi-GPU ctx has it.
 *   - List: d_slots[0, n_slots) is device memory on GPU `shard`, in any order, and may repeat a slot.
 *   - Entries outside the table: nothing checks the list on the host.  An entry >= N of the pod table gives -1 and a
 *     list of five -1, the result of a pod with nothing feasible.  No kernel reads outside the table.
 *   - Outputs, placement, alignment, direct-store fallback, signal, inline wait and refusals: exactly as the column call
 *     of the same name, with n_slots in place of P.  n_slots == 0 behaves like P == 0 there: a bound gather signals, and
 *     nothing else happens.
 *   - No pod table or no offer table on GPU `shard`: RPK_ESTATE.  d_slots NULL with n_slots > 0: RPK_EINVAL.  Both
 *     before anything is enqueued.
 *   - Counts as one select in rpk_stats (offer_scores += n_slots * G).  One gather kernel runs ahead of the select.
 *   - After one call of a given size the call only enqueues launches, so it can be captured in a CUDA graph.  A replay
 *     reads the table as it is at replay time, so seeds between replays are picked up (the caller orders a seed after
 *     a replay still in flight; the library does not see replays).  rpk_pods_reset invalidates a captured graph: the
 *     graph keeps the old N and possibly buffers the reset freed. */
int rpk_select_slots_device(rpk_ctx* ctx, int shard, uint32_t n_slots, const uint32_t* d_slots, int32_t* d_best,
                            int32_t* d_top5, void* stream);
int rpk_select_slots_device_gather(rpk_ctx* ctx, int shard, uint32_t n_slots, const uint32_t* d_slots, int n_out,
                                   int32_t* const* d_best_full, uint32_t row0, int32_t* d_top5, void* stream);
int rpk_select_slots_device_gather_top5(rpk_ctx* ctx, int shard, uint32_t n_slots, const uint32_t* d_slots, int n_out,
                                        int32_t* const* d_best_full, int32_t* const* d_top5_full, uint32_t row0,
                                        void* stream);

/* Cross-process peer vectors for one-process-per-GPU callers (torchrun-style): allocate a plain cudaMalloc
 * buffer on GPU `shard` and export its 64-byte CUDA IPC handle; another process opens the handle and gets a
 * device pointer it can pass in d_best_full[] of rpk_select_device_gather (peer access over NVLink is
 * enabled by the open).  Buffers/mappings are released by rpk_ipc_free / rpk_ipc_close or rpk_destroy. */
int rpk_ipc_alloc(rpk_ctx* ctx, int shard, size_t bytes, void** d_ptr, unsigned char handle_out[64]);
int rpk_ipc_open(rpk_ctx* ctx, int shard, const unsigned char handle[64], void** d_peer_ptr);
int rpk_ipc_close(rpk_ctx* ctx, int shard, void* d_peer_ptr);
int rpk_ipc_free(rpk_ctx* ctx, int shard, void* d_ptr);

/* Cross-GPU fence for the fused gather (one tiny kernel, no NCCL): lane r stores `epoch` into rank r's flag
 * array at index my_rank (system-scope fence first, so every peer store issued by earlier work of this stream
 * -- the gather's NVLink stores -- is visible before the flag), then spins until its own flag array
 * shows `epoch` from every rank.  d_flags[r] is rank r's array of >= n uint32 (zero-initialised,
 * rpk_ipc_alloc'ed and rpk_ipc_open'ed like the vectors); epochs must increase by one per fence.
 * epoch = 0 selects the self-counting mode: the kernel keeps the count in word 32 of the rank's own array
 * (arrays of >= 33 words), so the launch has no per-call argument and can be captured in a CUDA graph and
 * replayed; all ranks of a group must use the same mode for the life of the arrays. */
int rpk_peer_fence(rpk_ctx* ctx, int shard, int n, uint32_t* const* d_flags, int my_rank, uint32_t epoch, void* stream);

/* Split fence for the fused gather.  rpk_peer_bind registers the N flag arrays of a peer group with GPU `shard` of
 * this ctx (d_flags[r] = rank r's array of >= 64 uint32, zero-initialised, rpk_ipc_alloc'ed / rpk_ipc_open'ed like the
 * vectors; n = 0 unbinds).  While bound, every rpk_select_device_gather on that shard with n_out > 1 SIGNALS by itself:
 * the warp that pushes the last block of the slice (or a one-warp kernel behind the copy kernel on the small-batch
 * paths, or behind nothing for an empty shard) bumps the rank's select epoch (word 32 of its own array) and stores it
 * into word `my_rank` of every peer's array, after a system-scope fence.  rpk_status_diff_device_gather does the same
 * with the status epoch (word 33, flag words 8 + my_rank).  rpk_peer_wait enqueues the other half: one warp that
 * spins until every rank's flag shows this rank's own current epoch (what: bit 0 = select, bit 1 = status sweep;
 * all ranks of a group must issue the same sequence of gathers).  Launches carry no per-call value, so a step can be
 * captured in a CUDA graph and replayed.  Do not mix rpk_peer_fence and the bound mode on the same arrays (both use
 * words 0..7 and 32).
 * Ordering given: a peer's results are visible after the wait.  NOT given: once rank A has passed the wait of step e it
 * may run step e+1 and overwrite its slice of rank B's vector while B still reads step e -- consumers that read the
 * vector every step alternate between two sets of vectors (even / odd steps), as bench.py does. */
int rpk_peer_bind(rpk_ctx* ctx, int shard, int n, uint32_t* const* d_flags, int my_rank);
int rpk_peer_wait(rpk_ctx* ctx, int shard, unsigned what, void* stream);
/* on != 0: the warp that signals also WAITS (spins on its own flag words) until every rank of the group has signalled
 * the same epoch, so a bound gather only completes once all peers' results have landed and no rpk_peer_wait launch is
 * needed (one kernel boundary less per step).  All ranks of a group must use the same setting.  A host thread that
 * drives SEVERAL shards of a group must enable it only after one call of each size has sized the scratch: a call that
 * allocates synchronises its device, which would wait for a kernel that waits for a peer not launched yet. */
int rpk_peer_inline_wait(rpk_ctx* ctx, int shard, int on);

/* Device pointer of GPU `shard`'s copy of the full assignment vector written by the last rpk_select or rpk_select_slots
 * (ctx-owned; every GPU of the ctx holds the whole vector after the call). */
const int32_t* rpk_best_device_ptr(const rpk_ctx* ctx, int shard);

/* ---- status sweep diff ------------------------------------------------------------------------------ */

/* records: N slots of `stride` bytes (stride a multiple of 16, 16..256):
 *   [b0][status ASCII][0x00][ports_exposed:u8][zero pad],  b0 = len | flag << 7,  len = strlen(status)+2 <= min(stride-1, 127)
 * i.e. exactly the two fields compared at kubelet.go:870-871.  A slot's 64-bit XXH64 (seed 0) over its zero-padded
 * prefix in whole 8-byte lanes -- bytes [0, 8*ceil((1+len)/8)), flag bit cleared: the length byte is inside, so the
 * value is self-delimiting and does not depend on the stride -- is compared with the hash kept on the device from the
 * previous call; slots that differ (or have never been seen) are returned ascending in changed_idx[0..*n_changed)
 * (capacity N) and their stored hash is replaced (kubelet.go:875-880).  hashes_out (nullable, N) receives the new hash
 * column.  The flag bit is the host's "statusMessage contains error/fail" (kubelet.go:1907-1908): not a compared field,
 * not hashed, only used by the codes below.  Strides 16 (status <= 13 chars: every RunPod status) and 32 take the
 * streaming kernel; wider strides exist for longer strings. */
int rpk_status_diff(rpk_ctx* ctx, uint32_t N, const uint8_t* records, uint32_t stride, uint32_t* changed_idx,
                    uint32_t* n_changed, uint64_t* hashes_out);

/* What translateRunPodStatus (kubelet.go:1848-2024) decides for a slot, as a 16-bit code -- emitted per CHANGED slot
 * next to its index, so the caller builds v1.PodStatus for the changed subset without touching the strings again:
 *   bits 2:0  phase      0 Unknown 1 Pending 2 Running 3 Succeeded 4 Failed
 *   bit  3    ready      containerStatus.Ready and the Ready / ContainersReady conditions (kubelet.go:1972-1975)
 *   bit  4    started    containerStatus.Started
 *   bits 6:5  state      0 Waiting 1 Running 2 Terminated
 *   bit  7    exit code  (0 / 1)
 *   bits 10:8 reason     0 none 1 ContainerCreating 2 Completed 3 Error 4 Terminated 5 PodDeleted 6 ContainerStatusUnknown
 *   bits 12:11 message   0 statusMessage  1 "Container reported as running but ports not yet exposed" (:1885)
 *                        2 "Pod was deleted from RunPod API" (:1963)  3 "Unknown RunPod status: <status>" (:1975) */
#define RPK_CODE_PHASE(c) ((c) & 7u)
#define RPK_CODE_READY(c) (((c) >> 3) & 1u)
#define RPK_CODE_STARTED(c) (((c) >> 4) & 1u)
#define RPK_CODE_STATE(c) (((c) >> 5) & 3u)
#define RPK_CODE_EXIT(c) (((c) >> 7) & 1u)
#define RPK_CODE_REASON(c) (((c) >> 8) & 7u)
#define RPK_CODE_MESSAGE(c) (((c) >> 11) & 3u)
/* rpk_status_diff + changed_code[0..*n_changed) (nullable = rpk_status_diff) */
int rpk_status_diff_codes(rpk_ctx* ctx, uint32_t N, const uint8_t* records, uint32_t stride, uint32_t* changed_idx,
                          uint16_t* changed_code, uint32_t* n_changed, uint64_t* hashes_out);

/* Load previous state without reporting (CreatePod / LoadRunning fill InstanceInfo the same way,
 * kubelet.go:393-400, 1380-1535). */
int rpk_status_seed(rpk_ctx* ctx, uint32_t N, const uint8_t* records, uint32_t stride);
/* ... of individual slots: records holds n_slots packed slots of `stride` bytes, records[i] becomes the previous state
 * of slot slots[i] (CreatePod writes ONE InstanceInfo, kubelet.go:391-401; handleMissingRunPodInstance rewrites one,
 * :976-1040).  Nothing else is touched, so a sweep whose records are already staged loses nothing. */
int rpk_status_seed_slots(rpk_ctx* ctx, uint32_t n_slots, const uint32_t* slots, const uint8_t* records, uint32_t stride);
/* Diff of individual slots of the tracked table: records holds n_slots packed slots of `stride` bytes, records[i]
 * is this sweep's state of slot slots[i] (updateAllPodStatuses compares only the pods it fetched this cycle,
 * kubelet.go:836-864).  slots must be strictly ascending and < N of the tracked table (else RPK_EINVAL, nothing
 * changed; no tracked table: RPK_ESTATE).  Same predicate, state update and codes as rpk_status_diff_codes restricted
 * to the listed slots: changed_idx (capacity n_slots) receives the changed SLOT ids ascending, changed_code
 * (nullable) their codes.  Slots not listed are neither compared nor touched.  n_slots == 0: *n_changed = 0.
 * Counts n_slots records in rpk_stats.status_records. */
int rpk_status_diff_slots(rpk_ctx* ctx, uint32_t n_slots, const uint32_t* slots, const uint8_t* records,
                          uint32_t stride, uint32_t* changed_idx, uint16_t* changed_code, uint32_t* n_changed);
/* Device variant on a caller-owned column: d_hash_prev holds global slots [idx_base, idx_base + N).  An entry whose
 * slot lies outside that range is skipped (never read, written or reported), so the ranks of a sharded table can
 * all be handed the same global list.  Enqueued on `stream`, no synchronisation, graph-capturable after one call
 * of the size.  d_records and d_hash_prev 16-byte aligned (else RPK_EINVAL); d_changed_idx capacity n_slots.  Order
 * is a precondition here (not checked): with a list that is not strictly ascending the changed list is unspecified,
 * but no memory outside d_hash_prev[0, N) and the outputs is touched. */
int rpk_status_diff_slots_device(rpk_ctx* ctx, int shard, uint32_t N, uint32_t idx_base, uint32_t n_slots,
                                 const uint32_t* d_slots, const uint8_t* d_records, uint32_t stride,
                                 uint64_t* d_hash_prev, uint32_t* d_changed_idx, uint16_t* d_changed_code,
                                 uint32_t* d_n_changed, void* stream);
/* Forget all previous hashes and (re)size the table to N slots: every slot reports changed next time. */
int rpk_status_reset(rpk_ctx* ctx, uint32_t N);

/* One tick: rpk_select (P rows; P = 0 skips it) and rpk_status_diff_codes (N slots) enqueued together -- the two are
 * independent (processPendingPods kubelet.go:747-814, updateAllPodStatuses :816-974), so the sweep's upload follows the
 * selection's on the PCIe link while the selection's kernels run, every shard of a multi-GPU ctx is driven by its own
 * host thread, and the call synchronises once.  Argument meaning as in the two calls. */
int rpk_tick(rpk_ctx* ctx, uint32_t P, const int32_t* req_mem_gb, const int32_t* req_vcpu, const int32_t* req_ram_gb,
             const double* max_price, const uint8_t* cloud, int32_t* best, int32_t* top5, uint32_t N, const uint8_t* records,
             uint32_t stride, uint32_t* changed_idx, uint16_t* changed_code, uint32_t* n_changed);

/* Device-resident variant on GPU `shard`: d_records N*stride bytes, d_hash_prev N uint64 updated in place
 * (caller-owned column; 0 = never seen; both 16-byte aligned, else RPK_EINVAL), d_changed_idx capacity N, d_n_changed
 * one uint32.  Enqueued on
 * `stream`, no synchronisation.  Ordering against the shard's other calls: see "Ordering" at the top. */
int rpk_status_diff_device(rpk_ctx* ctx, int shard, uint32_t N, const uint8_t* d_records, uint32_t stride,
                           uint64_t* d_hash_prev, uint32_t* d_changed_idx, uint32_t* d_n_changed, void* stream);
int rpk_status_diff_device_codes(rpk_ctx* ctx, int shard, uint32_t N, const uint8_t* d_records, uint32_t stride,
                                 uint64_t* d_hash_prev, uint32_t* d_changed_idx, uint16_t* d_changed_code,
                                 uint32_t* d_n_changed, void* stream);

/* Sharded sweep with exchange (one process per GPU): rank `my_rank` sweeps its N slots (global ids idx_base + i) and
 * writes its changed list -- count, ascending global ids, codes -- into region `my_rank` of EVERY rank's exchange buffer
 * d_xchg[0..n_ranks) (peer-mapped like the assignment vectors; each rpk_xchg_bytes(n_ranks, cap) bytes, cap >= any
 * rank's N), straight from the kernel's final copy over NVLink.  Layout of a buffer, in uint32 words:
 *   [0, 8) count per source rank | [8 + r*cap, ...) ids of rank r | then uint16 codes: region r at
 *   ((uint16*)(words + 8 + n_ranks*cap)) + r*cap.
 * With flags bound (rpk_peer_bind) the CTA that finishes last signals the status epoch; rpk_peer_wait(what = 2) on
 * every rank makes all regions readable.  Every stride of rpk_status_diff (16..256), so a table that
 * Provider::WidenRecords has widened for a long status string keeps the exchange.  A rank with N = 0 still publishes
 * its zero count and signals.  Graph-capturable after one call of the size. */
size_t rpk_xchg_bytes(int n_ranks, uint32_t cap);
int rpk_status_diff_device_gather(rpk_ctx* ctx, int shard, uint32_t N, const uint8_t* d_records, uint32_t stride,
                                  uint64_t* d_hash_prev, uint32_t idx_base, int n_ranks, uint32_t* const* d_xchg, uint32_t cap,
                                  int my_rank, uint32_t* d_n_changed, void* stream);
/* The slot-list sweep (rpk_status_diff_slots_device) with the same exchange: the sweep one process per GPU runs when it
 * compares only the pods it fetched.  d_slots[0..n_slots) lists global slot ids, d_records holds their n_slots packed
 * records, and rank `my_rank`'s column d_hash_prev holds global slots [idx_base, idx_base + N) (entries outside it are
 * skipped: never read, written or reported).  Region `my_rank` of every buffer d_xchg[0..n_ranks) receives the count,
 * the global slot ids of the listed entries that changed in list order, and their codes, in the rpk_xchg_bytes layout
 * above; *d_n_changed gets the count.  Buffers, bound signal (an empty list publishes 0 and signals too), inline wait
 * and graph capture as for rpk_status_diff_device_gather.  List order is a precondition, not checked, so n_slots is
 * what must fit: n_slots > cap, d_slots NULL with n_slots > 0, n_ranks outside 1..8, my_rank outside [0, n_ranks), a
 * NULL buffer, d_records or d_hash_prev not 16-byte aligned, or a bad stride: RPK_EINVAL before anything is enqueued.
 * When rank r's column precedes rank r+1's and every list is ascending, the regions concatenated in rank order are the
 * ascending global changed list.  Hand each rank only its own part of the global list (one searchsorted of the column
 * boundaries on the host): a rank handed the whole list is still correct, but reads every listed record. */
int rpk_status_diff_slots_device_gather(rpk_ctx* ctx, int shard, uint32_t N, uint32_t idx_base, uint32_t n_slots,
                                        const uint32_t* d_slots, const uint8_t* d_records, uint32_t stride,
                                        uint64_t* d_hash_prev, int n_ranks, uint32_t* const* d_xchg, uint32_t cap,
                                        int my_rank, uint32_t* d_n_changed, void* stream);

int rpk_stats_get(const rpk_ctx* ctx, rpk_stats* out);

/* number of kernel launches issued by this ctx since creation (bench.py's gpu_launches) */
uint64_t rpk_launch_count(const rpk_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* RPK_H_ */
