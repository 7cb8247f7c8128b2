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
 *   - Ordering.  The calls on one shard are ordered in two scopes: the select scope (the offer table and the pod table,
 *     which host and _device calls share, and the _device selects' scratch) and the status scope (the _device sweeps'
 *     scratch).  Host calls have select and sweep scratch of their own ("Graph capture" below).  A _device call issued
 *     on another stream than the last _device call of its scope first waits for that call, so any streams may be used.
 *     A host call waits for the last _device call of its scopes before it touches anything, so host and _device calls
 *     of one scope never overlap, and returns after its own work is done; the caller needs no synchronise between the
 *     two.  Select scope: rpk_offers_upload, rpk_offers_refresh, rpk_pods_reset, rpk_pods_grow,
 *     rpk_pods_seed_slots, rpk_pods_mark_pending, rpk_select, rpk_select_slots, rpk_select_pending,
 *     rpk_select_pending_changed, rpk_explain, rpk_explain_slots, the _device call
 *     rpk_pods_pending_list_device, rpk_select_pending_changed_gather (which also waits on the host),
 *     rpk_select_pending_changed_device_gather, and rpk_tick
 *     with P > 0.  Status scope: rpk_status_diff,
 *     rpk_status_diff_codes, rpk_status_seed, rpk_status_diff_slots and rpk_tick.  rpk_status_reset, rpk_status_grow
 *     and rpk_status_seed_slots touch only buffers no _device call uses and do not wait.  A _device call inside a stream
 *     capture neither waits nor is waited for (keep each captured entry point on one stream), and the library does
 *     not see replays of a captured graph: a caller that replays a captured device step orders its host calls after
 *     the replay itself.
 *   - Graph capture.  After one call of a given size a _device call only enqueues launches, so it can be captured in a
 *     CUDA graph and replayed.  The graph keeps every ctx-owned device buffer the call handed its kernels
 *     (rpk_test_capture_buffers lists them) and the values the call read at capture.  Host calls have scratch of their
 *     own, and the _device calls of a shard share one select scratch and one sweep scratch that only _device calls size.
 *     A capture of a _device call on shard s stays valid across:
 *       - every host call, of any size, on any shard (rpk_select, rpk_select_slots, rpk_select_pending*, rpk_explain,
 *         rpk_explain_slots, the host sweeps, rpk_tick, rpk_status_reset, rpk_status_grow, ...);
 *       - the seeds and marks: rpk_pods_seed_slots, rpk_pods_mark_pending, rpk_status_seed, rpk_status_seed_slots (a
 *         replay reads the rows, flags and hashes as they are at replay time);
 *       - _device calls on s that need no more scratch than the calls made on s before the capture.
 *     It is invalidated by (capture again after them, after one call outside the capture):
 *       - a _device call on s that needs more scratch: a select of more rows, or a sweep of more records or list
 *         entries, than any before (the scratch grows and frees the buffers the graph points at);
 *       - rpk_offers_upload and rpk_offers_refresh (new views and columns; G, the layout and the change window are
 *         copied at capture);
 *       - rpk_pods_reset and rpk_pods_grow, for the calls that read the pod table or the flags
 *         (rpk_select_slots_device*, rpk_pods_pending_list_device, rpk_select_pending_changed_device_gather): N is an
 *         argument of their kernels, so a grow invalidates them even when no buffer moves;
 *       - rpk_peer_bind and rpk_peer_inline_wait, for the bound gathers (the group is copied at capture).
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
    uint64_t select_calls;        /* rpk_select + rpk_select_slots + rpk_select_pending + rpk_select_pending_changed + rpk_select_device + rpk_select_slots_device */
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
 * copies over NVLink (peer access is enabled here).  A device id may appear once.
 * Test only: with RPK_TEST_SHARED_DEVICE=1 in the environment (read here, once per ctx, and nowhere else) a repeated
 * device id is accepted and shards on the same GPU are not enabled as each other's peers, so a one-GPU machine can run
 * an n-shard ctx.  Do not queue rpk_peer_fence, or a bound gather that waits, between shards that share a GPU. */
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

/* Offers a refresh remembers as changed between two wholesale invalidations of the pending results (below). */
#define RPK_OFFERS_DELTA_MAX 16

/* rpk_offers_upload for a table that is mostly the one already resident: the same arguments, argument rules, refusals,
 * installed table and views.  The one difference is what happens to the results rpk_select_pending_changed[_gather]
 * stored.  When a table with the same G is resident, every GPU compares the new columns with it, offer by offer and bit
 * for bit (-0.0 and 0.0 differ), and the changed offers join the ctx's change window: one entry per offer, at the
 * generation of its latest change.  A stored result then stays valid unless a changed offer can reach its row (the rule
 * under rpk_select_pending_changed).  *n_offers_changed (nullable) receives the number of offers that differ, or
 * UINT32_MAX when the stored results are invalidated wholesale instead, as after rpk_offers_upload: no table resident,
 * another G, or a window that would hold more than RPK_OFFERS_DELTA_MAX offers.  The window is cleared then, and by
 * every rpk_offers_upload.  An identical table changes nothing (*n_offers_changed = 0).  Select scope, host call. */
int rpk_offers_refresh(rpk_ctx* ctx, uint32_t G, const int32_t* mem_gb, const int32_t* vcpu, const int32_t* ram_gb,
                       const double* secure_price, const double* community_price, const uint8_t* flags,
                       uint32_t* n_offers_changed);

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
 * No slot is pending afterwards (rpk_pods_mark_pending), and every result rpk_select_pending_changed stored is cleared.
 * Independent of rpk_status_reset.  The table is replicated: 22 bytes x N on each GPU (the five columns and the pending
 * flag).  rpk_select_pending_changed adds, per slot a GPU owns, 45 bytes of stored results (the columns a result came
 * from, an offer-table generation and the five list entries), about 36 bytes of device scratch and 28 bytes of pinned
 * host memory for the rows it returns, all allocated by its first call, so callers that never use it pay nothing. */
int rpk_pods_reset(rpk_ctx* ctx, uint32_t N);
/* Grow the pod table from its N0 slots to N >= N0 on every GPU of the ctx, keeping what it holds, so a caller whose
 * pods outgrow the table need not reset it (and reselect and report every pending slot on the next tick).
 *   - Slots [0, N0) keep their rows and pending flags bit for bit; slots [N0, N) get what rpk_pods_reset(N) gives them
 *     (the columns of a pod with no annotations, not pending).
 *   - The results rpk_select_pending_changed stored are kept.  On a multi-GPU ctx each GPU's owned range moves with N,
 *     and each stored result moves to its slot's new owner (a peer copy).  A ctx grown from N0 to N therefore returns from
 *     every later call what a ctx reset at N with the same history returns: growing reselects and reports nothing.
 *   - Results made by rpk_select_pending_changed_gather or its device form for another range than
 *     rpk_select_pending_changed's (n_ranks above the ctx's GPUs) are cleared, as rpk_pods_reset clears them: the other
 *     ranks' results live in other processes.  Each rank's next call binds its new range and reports every pending slot
 *     of it once.  With n_ranks = the ctx's GPUs (a one-GPU ctx with n_ranks = 1) the results are kept.
 *   - N < N0: RPK_EINVAL; no pod table: RPK_ESTATE; N == N0: RPK_OK and nothing is touched.  A failed allocation:
 *     RPK_ENOMEM and the ctx as it was (every GPU's buffers are allocated before anything is copied).
 *   - Select scope, host call: waits for the scope's last _device call first.  Invalidates captured graphs as
 *     rpk_pods_reset does ("Graph capture" at the top).  A grow within the 25 % of spare capacity the table keeps
 *     allocates nothing. */
int rpk_pods_grow(rpk_ctx* ctx, uint32_t N);
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

/* ---- explaining an empty gpuTypeIds list ------------------------------------------------------------------- */

/* Why a pod gets no GPU type: for one row, what rules out each offer of the resident table.  An offer is OFFERED to
 * the row when it passes the cloud check and price > 0 in the row's cloud (a cloud byte other than SECURE or COMMUNITY
 * offers nothing).  Four requirements are then checked on every offered offer: RPK_REQ_PRICE price < max_price (IEEE:
 * a NaN bound fails every offer), RPK_REQ_MEM mem_gb >= req_mem_gb, RPK_REQ_VCPU vcpu >= req_vcpu and RPK_REQ_RAM
 * ram_gb >= req_ram_gb -- rpk_select's predicate, split into its parts.  Invariants: n_unoffered + n_feasible + (the
 * offered offers failing at least one requirement) == G; n_feasible > 0 exactly when rpk_select's best != -1, and
 * min(n_feasible, 5) is the length of its top-5 list. */
#define RPK_REQ_PRICE 0
#define RPK_REQ_MEM 1
#define RPK_REQ_VCPU 2
#define RPK_REQ_RAM 3
typedef struct rpk_explanation {
    uint32_t n_feasible;   /* offered offers passing all four: what rpk_select's predicate keeps */
    uint32_t n_unoffered;  /* G - offered */
    uint32_t n_fail[4];    /* offered offers failing requirement r (an offer may count under several r) */
    uint32_t n_only[4];    /* offered offers failing requirement r and no other */
    int32_t nearest[4];    /* among the n_only[r] offers, the lowest (price in the row's cloud, offer index); -1 if
                              n_only[r] == 0.  The offer the pod would get if only r were relaxed, whenever n_feasible == 0 */
} rpk_explanation;
/* out[i] for pod row i (out: P entries).  Columns, their NULL rules and defaults as rpk_select's.  P == 0 is a no-op.
 * No offer table: RPK_ESTATE.  On a multi-GPU ctx the rows are split over the GPUs as rpk_select splits them; the result
 * does not depend on the number of GPUs.  Select scope, host call: it waits for the scope's last _device call, and reads
 * no stored pending result and writes no pending flag, pod row, change window or rpk_stats counter; its scratch is the
 * host calls' own, so a captured _device graph stays valid across it. */
int rpk_explain(rpk_ctx* ctx, uint32_t P, const int32_t* req_mem_gb, const int32_t* req_vcpu, const int32_t* req_ram_gb,
                const double* max_price, const uint8_t* cloud, rpk_explanation* out);
/* rpk_explain over rows of the pod table: out[i] is what rpk_explain returns for the row held at slot slots[i].  The
 * list may be in any order and may repeat a slot.  An entry >= N of the pod table: RPK_EINVAL, before anything is
 * enqueued.  No pod table or no offer table: RPK_ESTATE.  n_slots == 0 is a no-op.  Otherwise as rpk_explain. */
int rpk_explain_slots(rpk_ctx* ctx, uint32_t n_slots, const uint32_t* slots, rpk_explanation* out);

/* The pending set: which slots processPendingPods would retry, kept in the table next to the columns, so that a tick
 * sends no list at all.  The set changes as slowly as the columns do: a pod enters it in CreatePod and leaves it when a
 * deploy succeeds, the pod is deleted, or it is failed after 15 minutes.
 *
 * pending[i] != 0 marks slot slots[i] pending, 0 clears it: processPendingPods' predicate (Phase == Pending and no
 * runpod.io/pod-id, kubelet.go:752, :768), kept per slot.  slots strictly ascending and < N of the pod table (else
 * RPK_EINVAL, nothing written; no pod table: RPK_ESTATE), as rpk_pods_seed_slots.  Every GPU of the ctx gets the
 * flags.  Slots not listed are not touched.  rpk_pods_seed_slots changes no flag and this call no column.
 * n_slots == 0 is a no-op.  Select scope, host call. */
int rpk_pods_mark_pending(rpk_ctx* ctx, uint32_t n_slots, const uint32_t* slots, const uint8_t* pending);
/* rpk_select_slots over every pending slot of the pod table, ascending, with no list from the caller: the device builds
 * the list from the flags (in range by construction: nothing to check, nothing to upload).
 *   *n_pending   the number of pending slots (always written on RPK_OK and on the cap refusal below)
 *   slots_out    nullable, capacity cap: the pending slot ids, ascending (a caller that mirrors the flags knows them)
 *   best, top5   capacity cap and 5*cap (top5 nullable): row i is what rpk_select_slots returns for slot slots_out[i],
 *                bit for bit
 * More than cap slots pending: RPK_EINVAL, *n_pending set, no other output written, nothing counted.  No pod table or
 * no offer table: RPK_ESTATE.  Zero pending: RPK_OK, *n_pending = 0, and what rpk_select_slots does for n_slots == 0.
 * Counts as one select in rpk_stats (offer_scores += n_pending * G).  Select scope, host call. */
int rpk_select_pending(rpk_ctx* ctx, uint32_t cap, uint32_t* slots_out, uint32_t* n_pending, int32_t* best, int32_t* top5);
/* The pending tick without the rows that did not change.  A row's result depends only on its five columns and the offer
 * table, and both change rarely, so the library keeps, per slot, the last result this call REPORTED for it, and
 * reselects and reports only what may have changed.
 *   - Result of a slot s: R(s) is what rpk_select_slots returns for s now, bit for bit, with its top-5 list (the deploy
 *     sends the whole list); best is top5[0].
 *   - Reselected: a pending slot with no reported result, whose five columns differ bit for bit from the ones its
 *     reported result came from, or whose result predates the last rpk_offers_upload (an upload of an identical table
 *     included) or the last wholesale invalidation of rpk_offers_refresh.  After that, a result that predates a refresh
 *     is reselected only when an offer c the window says changed since the result was made reaches the row: c is in the
 *     reported list L, or c is feasible for the row under the current table (rpk_select's predicate) and L has fewer
 *     than five entries or (price(c), c) < (price(L[4]), L[4]) in the row's cloud.  Otherwise the list under the current
 *     table is L, exactly.  No other pending slot is recomputed.  *n_reselected counts them.
 *   - A pending slot whose result predates a refresh and that no changed offer reaches has its result marked current,
 *     so later calls do not test it again; this happens on the cap refusal below too, and is not observable: the
 *     stored list is R(s).
 *   - Reported, ascending by slot: every reselected slot whose R(s) differs from its reported result, or that has none.
 *     Row i is slots_out[i], best[i], top5[5i, 5i+5); *n_changed <= *n_reselected rows.  Each reported R(s) becomes the
 *     slot's reported result.  A caller that applies every report to a mirror kept per SLOT holds R(s) for every pending
 *     slot afterwards.
 *   - Stored results outlive the pending flag: a slot that leaves the set and comes back with the same columns and offer
 *     table is not reported again, and a slot reused by another pod needs nothing special (the result depends on the
 *     columns only).  rpk_pods_reset clears them all and rpk_pods_grow moves them with their slots; no other call reads
 *     or writes them.
 *   - *n_pending, *n_reselected and *n_changed are always required; with cap > 0 so are slots_out, best and top5
 *     (capacities cap, cap and 5*cap); else RPK_EINVAL.  No pod table or no offer table: RPK_ESTATE.  Both before
 *     anything is enqueued.
 *   - More than cap slots to reselect: RPK_EINVAL with *n_pending and *n_reselected written, nothing else written, no
 *     stored list changed (only the marking above), nothing counted; retry with cap = *n_reselected.
 *   - Counts as one select in rpk_stats (offer_scores += n_reselected * G) when it reselects anything; a call that
 *     reselects nothing counts no select.  Select scope, host call.
 *   - Multi-GPU ctx: the stored results are sharded by slot range (GPU k owns a contiguous range, its boundaries on
 *     16-slot units); each GPU reselects and diffs its own slots, and the rows come back in GPU order, ascending. */
int rpk_select_pending_changed(rpk_ctx* ctx, uint32_t cap, uint32_t* n_pending, uint32_t* n_reselected, uint32_t* slots_out,
                               int32_t* best, int32_t* top5, uint32_t* n_changed);

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
 * function only enqueues launches, so it can be captured in a CUDA graph ("Graph capture" at the top). */
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
 *   - After one call of a given size the function only enqueues launches (CUDA-graph capturable: "Graph capture" at the
 *     top). */
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
 *   - After one call of a given size the call only enqueues launches, so it can be captured in a CUDA graph ("Graph
 *     capture" at the top).  A replay reads the table as it is at replay time, so seeds between replays are picked up
 *     (the caller orders a seed after a replay still in flight; the library does not see replays).  rpk_pods_reset
 *     invalidates a captured graph: the graph keeps the old N and possibly buffers the reset freed. */
int rpk_select_slots_device(rpk_ctx* ctx, int shard, uint32_t n_slots, const uint32_t* d_slots, int32_t* d_best,
                            int32_t* d_top5, void* stream);
int rpk_select_slots_device_gather(rpk_ctx* ctx, int shard, uint32_t n_slots, const uint32_t* d_slots, int n_out,
                                   int32_t* const* d_best_full, uint32_t row0, int32_t* d_top5, void* stream);
int rpk_select_slots_device_gather_top5(rpk_ctx* ctx, int shard, uint32_t n_slots, const uint32_t* d_slots, int n_out,
                                        int32_t* const* d_best_full, int32_t* const* d_top5_full, uint32_t row0,
                                        void* stream);

/* The pending list only, for one-process-per-GPU callers: d_slots_out (capacity N of the pod table, on GPU `shard`)
 * receives the pending slot ids ascending, *d_n (device memory on GPU `shard`) their number; entries of d_slots_out
 * beyond *d_n are not written.  It is the launch rpk_select_pending makes, exposed: one kernel, no memset before it.
 * Enqueued on `stream`, no synchronisation; select scope, device call (ordered like rpk_select_slots_device).  The
 * select kernels take no device-side row count: the caller reads *d_n (or knows it from its own mirror of the flags)
 * and passes it as n_slots, with the list, to rpk_select_slots_device[_gather[_top5]].  No pod table: RPK_ESTATE; NULL
 * output: RPK_EINVAL; both before anything is enqueued.  Graph-capturable after one call ("Graph capture" at the top); a
 * replay reads the flags as they are at replay time. */
int rpk_pods_pending_list_device(rpk_ctx* ctx, int shard, uint32_t* d_slots_out, uint32_t* d_n, void* stream);

/* rpk_select_pending_changed for one-process-per-GPU callers: each rank reselects the pending slots of its own range and
 * sends only its changed rows to every rank, over the exchange buffers and the bound flags.
 *   - Owned range: rank my_rank of n_ranks owns slots [lo, hi) of the pod table, the range GPU my_rank of an n_ranks-GPU
 *     ctx owns in rpk_select_pending_changed (boundaries on 16-slot units), so the ranks' ranges tile the table in rank
 *     order; a range may be empty.  Every rank keeps the whole pod table and the flags (every rank seeds and marks the
 *     same rows, as for rpk_select_slots_device_gather); a rank's stored results cover its own range only.
 *   - Semantics: exactly rpk_select_pending_changed restricted to [lo, hi): the same stale rule (with the reach rule of
 *     rpk_offers_refresh against this ctx's change window, and the same marking of unreached results), one select with top-5,
 *     the same diff, and each reported result becomes the slot's stored result.  *n_pending and *n_reselected count the
 *     rank's own slots.  Counts as one select in rpk_stats when it reselects anything.
 *   - Exchange: the rank's changed rows, ascending by slot, land in region my_rank of every buffer d_xchg[0..n_ranks)
 *     (peer-mapped like the assignment vectors; each rpk_results_xchg_bytes(n_ranks, cap) bytes, 16-byte aligned).  A
 *     buffer in uint32 words: [0, 8) the count per source rank; from word 8, region r = r * 7 * cap words on: slot[cap],
 *     best[cap], top5[5 * cap] (best is top5[0]).  Entries past a region's count are not written.  The regions of all
 *     ranks concatenated in rank order are rpk_select_pending_changed's slots_out / best / top5, bit for bit.
 *   - Signal: with flags bound (rpk_peer_bind) the CTA that finishes last signals the pending results epoch (word 34 of
 *     the rank's own array, flag words 16 + my_rank) after a system-scope fence; rpk_peer_wait(what = 4) or the inline
 *     wait makes every region readable.  A rank with nothing to reselect, or an empty range, still writes its count 0
 *     into every buffer and signals.
 *   - RPK_EINVAL, before anything is enqueued and without signalling: n_ranks outside 1..8, my_rank outside [0, n_ranks),
 *     a NULL or misaligned buffer, a NULL count pointer, or cap < hi - lo (every rank must hold its worst case, so no
 *     refusal can come after the stale step while peers wait).  RPK_ESTATE, the same way: no pod table or no offer table
 *     on GPU `shard`, or stored results made for another range since the last rpk_pods_reset or rpk_pods_grow (another
 *     my_rank or n_ranks, or rpk_select_pending_changed on the same ctx with another range).
 *   - Ordering: select scope.  The call waits on the host for the scope's last device call, synchronises `stream` once
 *     after the stale step (the select needs the row count on the host), and returns with the gather, select, diff,
 *     push and signal enqueued on `stream`.  NOT graph-capturable.  A rank's first call after rpk_pods_reset (and a call
 *     that grows the select scratch) synchronises the device, so a host thread that drives several ranks turns the
 *     inline wait on only after each rank has made one call, as rpk_peer_inline_wait says. */
size_t rpk_results_xchg_bytes(int n_ranks, uint32_t cap);
int rpk_select_pending_changed_gather(rpk_ctx* ctx, int shard, int n_ranks, int my_rank, uint32_t* const* d_xchg, uint32_t cap,
                                      uint32_t* n_pending, uint32_t* n_reselected, void* stream);
/* rpk_select_pending_changed_gather with the row count kept on the device, so the tick never waits for the host and can
 * be captured in a CUDA graph.  Everything not listed here is as there.
 *   - Semantics: identical.  The owned range, the stale rule (the reach rule against the ctx's change window and the
 *     marking of unreached results included), one select with top-5, the diff, each reported result becoming the slot's
 *     stored result, the exchange layout (rpk_results_xchg_bytes), the bound signal on the pending results epoch (word
 *     34, flag words 16 + my_rank) and the inline wait.  The regions are bit for bit what the host-sync form writes after
 *     the same history; the two forms may be mixed on one ctx.
 *   - Counts: d_counts (nullable; device memory on GPU `shard`, 4-byte aligned) receives [n_pending, n_reselected] of
 *     the rank's range.  Nothing is read back to the host.
 *   - Refusals: every refusal of rpk_select_pending_changed_gather except the NULL count pointers, plus a d_counts that is
 *     not 4-byte aligned (RPK_EINVAL); all before anything is enqueued and without signalling.
 *   - Ordering: a _device call of the select scope, ordered like rpk_select_slots_device: no host wait; host calls wait for
 *     it as for any other device call.  The kernels are sized for the rank's worst case, hi - lo rows, and read the row
 *     count the stale step left on the device.
 *   - Graph capture: the first call after rpk_pods_reset sizes every buffer for hi - lo rows and synchronises the device
 *     (make it outside a capture, and before the inline wait is turned on, as for the host-sync form).  After one call
 *     with the same (n_ranks, my_rank, cap) on a pod table of the same N, the call only enqueues launches.  A replay reads
 *     the flags, the pod rows and the stored results as they are at replay time, so seeds and marks between replays are
 *     picked up.  The reselected rows go to scratch of this call's own (41 bytes per owned slot, allocated by its first
 *     call), so selects of any size on the ctx between replays leave a captured graph valid ("Graph capture" at the
 *     top).  The offer-table generation
 *     and change window are taken at capture: rpk_offers_upload, rpk_offers_refresh and rpk_pods_reset each invalidate a
 *     captured graph (re-capture after them), as does a call with another range, which is refused at call time but not
 *     at replay.
 *   - Stats: not counted in rpk_stats (the host never learns n_reselected); rpk_launch_count counts what was enqueued. */
int rpk_select_pending_changed_device_gather(rpk_ctx* ctx, int shard, int n_ranks, int my_rank, uint32_t* const* d_xchg,
                                             uint32_t cap, uint32_t* d_counts, void* stream);

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
 * with the status epoch (word 33, flag words 8 + my_rank), and rpk_select_pending_changed_gather with the pending
 * results epoch (word 34, flag words 16 + my_rank).  rpk_peer_wait enqueues the other half: one warp that
 * spins until every rank's flag shows this rank's own current epoch (what: bit 0 = select, bit 1 = status sweep,
 * bit 2 = pending results; all ranks of a group must issue the same sequence of gathers).  Launches carry no per-call value, so a step can be
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

/* Test hook: the ctx-owned device buffers a _device call on GPU `shard` passes to its kernels, as pointers (NULL: not
 * allocated), in a fixed order: the device select lane (16), the device sweep scratch (5), the two offer views (7
 * each), the distinct values (3), the raw offer columns (6) and the change window, the pod table and its flags (6), the
 * compaction state (2), the stored pending results (10) and their reselect lane (16).  *n receives the count; the first
 * min(cap, *n) go to ptrs.  A call that leaves every one of them in place leaves a captured graph valid ("Graph
 * capture" at the top).  RPK_EINVAL for a NULL ctx or n, a bad shard, or cap > 0 with NULL ptrs. */
int rpk_test_capture_buffers(const rpk_ctx* ctx, int shard, const void** ptrs, size_t cap, size_t* n);

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
 * but no memory outside d_hash_prev[0, N) and the outputs is touched.  "Graph capture" at the top says which calls keep
 * a capture valid. */
int rpk_status_diff_slots_device(rpk_ctx* ctx, int shard, uint32_t N, uint32_t idx_base, uint32_t n_slots,
                                 const uint32_t* d_slots, const uint8_t* d_records, uint32_t stride,
                                 uint64_t* d_hash_prev, uint32_t* d_changed_idx, uint16_t* d_changed_code,
                                 uint32_t* d_n_changed, void* stream);
/* Forget all previous hashes and (re)size the table to N slots: every slot reports changed next time. */
int rpk_status_reset(rpk_ctx* ctx, uint32_t N);
/* Grow the tracked table from its N0 slots to N >= N0, keeping every hash: slots [0, N0) report only real changes on the
 * next sweep, slots [N0, N) are never seen (hash 0), as after rpk_status_reset(N).  On a multi-GPU ctx the hashes move
 * with the shard boundaries.  The whole-table host sweeps and rpk_tick then take N.  N < N0: RPK_EINVAL; no tracked
 * table: RPK_ESTATE; N == N0: RPK_OK, nothing touched; a failed allocation: RPK_ENOMEM, the table as it was.  Like
 * rpk_status_reset it touches no buffer a _device call uses and does not wait. */
int rpk_status_grow(rpk_ctx* ctx, uint32_t N);

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
 * its zero count and signals.  Graph-capturable after one call of the size ("Graph capture" at the top). */
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
