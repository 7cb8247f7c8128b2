"""Restatement of the persistent select's launch plan: ``class_dims`` and ``persist_plan`` in
k8s-runpod-kubelet_b200/csrc/select_persist.cu, with the constants of rpk_internal.cuh, the view layout
``launch_offer_ingest`` (offers.cu) picks from the distinct counts (``layout``, which includes the bitmapM condition)
the host entry point's row sub-batches (``sub_batch_rows``, rpk_api.cu), and the grid of the packed and wide kernels
that tables without a bit-sliced view take (``pick_rows_per_warp``, ``select_tiles_max``, ``seg_plan`` and
``launch_grid`` in select.cu).

The GPU tests assert through it which regime each case reaches, so a change to a constant that moves a case off its
regime fails the case instead of quietly testing something else."""
from types import SimpleNamespace

import numpy as np

SUB_CHUNKS, SUB_STRIDE = 64, 68       # kSubChunks, kSubStride: 64 chunks of 32 offers per sub-range, 68-word rows
MAX_CLASSES, BM_MAX_STRIDE = 4096, 64  # kMaxClasses, kBmMaxStride
PWARPS, RPI = 16, 64                   # warps per 512-thread CTA; rows per item (32 lanes x kRpl)
STAGE_MAX = 220 * 1024                 # persist_plan's stage cap
FUSED_ROWS_MAX, SMALL_BATCH = 16384, 4096  # kFusedRowsMax, kSmallBatch
SUB_BATCH_ROWS = 131072                # kSubBatchRows (x1, x2, x3, then x4)
POS_BITS = 14                          # kPosBits: position-in-segment bits of a packed_pos word (kSegPacked = 2^14)
WARPS_PER_CTA, GROUPS, CHUNK = 8, 8, 128  # kWarpsPerCta, kGroups (cloud x vcpu constrains x ram constrains), kChunk
SEG_PACKED, SEG_WIDE = 1 << POS_BITS, 4096  # kSegPacked, kSegWide: offers staged per CTA of the packed / wide kernels
GRID_X_MAX = 2**31 - 1                 # gridDim.x limit: launch_grid cuts larger grids into launches of whole row tiles
# RPK_FORCE_KERNEL values as install_offers (rpk_api.cu) reads them; any other string is the automatic choice
FORCE_KINDS = {"generic": 1, "packed": 2, "packed_pos": 3, "bitmap": 4, "bitmap_grouped": 5, "bitmap_price": 6}
KIND_NAMES = {1: "generic", 2: "packed", 3: "packed_pos", 4: "bitmap"}  # rpk_stats.select_kernel_kind


def cdiv(a, b):
    return -(-a // b)


def bitlen(x):
    """offers.cu's bitlen: the bits of x, at least 1"""
    return max(int(x).bit_length(), 1)


def layout(D, force=None):
    """the offer views launch_offer_ingest builds for distinct counts D = [mem, vcpu, ram] under RPK_FORCE_KERNEL
    `force` (None: the automatic choice).  The packed word holds mem rank' + 1 in [0, D0] against thresholds up to
    D0 + 1, and vcpu / ram ranks against thresholds up to D, each field with a guard bit; it exists when the fields
    total 32 bits or less, and carries the 14-bit position in its segment when they total 18 or less.  The bit-sliced
    view has one mask word per threshold, (D0 + 1) + (D1 + 1) + (D2 + 1) of them, in rows of 32 or 64 words, and
    per-mem-threshold slices when the class key keeps the mem threshold (and the table is not empty).
    kind is rpk_stats.select_kernel_kind: 4 bitmap, 3 packed_pos, 2 packed, 1 generic."""
    k = FORCE_KINDS.get(force, 0)
    b1, b2, b3 = bitlen(D[0] + 1), bitlen(D[1]), bitlen(D[2])
    bits = b1 + b2 + b3 + 3
    if bits > 32:
        bits = 0
    pos_bits = POS_BITS if bits and bits + POS_BITS <= 32 else 0
    bm_words = (D[0] + 1) + (D[1] + 1) + (D[2] + 1)
    if bm_words > BM_MAX_STRIDE:
        bm_words = 0
    if k == 1:
        bits = pos_bits = bm_words = 0
    elif k == 2:
        pos_bits = bm_words = 0
    elif k == 3:
        bm_words = 0
    kind = 4 if bm_words else 3 if pos_bits else 2 if bits else 1
    return SimpleNamespace(kind=kind, name=KIND_NAMES[kind], packed_bits=bits, pos_bits=pos_bits, bm_words=bm_words,
                           bm_stride=(32 if bm_words <= 32 else 64) if bm_words else 0,
                           slice=bool(bm_words) and D[0] > 0 and class_dims(D)[3],
                           no_fused=k >= 5, no_slice=k == 6)


def distinct(offers):
    """the sorted distinct values of mem / vcpu / ram (a missing column is all zero)"""
    G = len(offers["mem_gb"])
    return [np.unique(offers[k]) if offers.get(k) is not None else np.zeros(min(G, 1), np.int32)
            for k in ("mem_gb", "vcpu", "ram_gb")]


def class_dims(D):
    """-> (Dm1, Dv1, Dr1, use_mem, C): the mem threshold joins the class key (and bitmapM exists) when it fits"""
    Dm1, Dv1, Dr1 = D[0] + 1, D[1] + 1, D[2] + 1
    use_mem = 2 * Dm1 * Dv1 * Dr1 <= MAX_CLASSES
    return Dm1, Dv1, Dr1, use_mem, 2 * Dv1 * Dr1 * (Dm1 if use_mem else 1)


def plan(G, P, D, sm_count, stage_kb=0, items_per_warp=0, no_slice=False, k0ctas=0):
    """persist_plan for a table of G offers with distinct counts D and a batch of P rows (RPK_TUNE stagekb / ipw /
    k0ctas when non-zero; no_slice: RPK_FORCE_KERNEL=bitmap_price)"""
    Dm1, Dv1, Dr1, use_mem, C = class_dims(D)
    bm_words = Dm1 + Dv1 + Dr1
    assert bm_words <= BM_MAX_STRIDE, "no bit-sliced view: the table takes the packed or generic kernels"
    nsub = cdiv(cdiv(G, 32), SUB_CHUNKS)
    slice_rows = Dv1 + Dr1 if nsub and use_mem else 0
    max_stage = min(stage_kb if stage_kb > 0 else 220, 220) * 1024
    slice_bytes = slice_rows * SUB_STRIDE * 4
    sl = bool(slice_rows) and not no_slice and slice_bytes <= max_stage
    sub_bytes = slice_bytes if sl else bm_words * SUB_STRIDE * 4
    cap = max(max_stage // sub_bytes, 1)
    per = cdiv(nsub, cdiv(nsub, cap))
    S = cdiv(nsub, per)
    visits = max(cdiv(P, RPI) * S, 1)
    Qi = min(max(cdiv((items_per_warp if items_per_warp > 0 else 4) * sm_count * PWARPS, visits), 1), per)
    qspan = cdiv(per, Qi)
    tickets = sum(cdiv(min(per, nsub - s * per), qspan) for s in range(S))
    k0 = k0ctas if k0ctas > 0 else 4 * sm_count
    return SimpleNamespace(slice=sl, nsub=nsub, S=S, per=per, qspan=qspan, tickets_per_block=tickets,
                           direct=tickets == 1, classes=C, smem_bytes=per * sub_bytes, grid=sm_count,
                           k0_blocks=max(min(cdiv(P, 512), k0), 1), groups_per_cloud=Dm1 if sl else 1)


def queues(pl, dist, pods):
    """non-empty (row group, stage) queues of one call: a row group is the cloud, or (cloud, mem threshold) when the
    stages are slices of bitmapM; rows of neither cloud have no group"""
    P = len(pods["req_mem_gb"])
    cloud = pods.get("cloud")
    cloud = np.zeros(P, np.int64) if cloud is None else cloud.astype(np.int64)
    keep = cloud <= 1
    grp = cloud[keep]
    if pl.slice:
        grp = grp * pl.groups_per_cloud + np.searchsorted(dist[0], pods["req_mem_gb"][keep], side="left")
    return len(np.unique(grp)) * pl.S


def iterations_per_cta(pl, n_queues):
    """stages the busiest CTA loads in one call: with more queues than CTAs, CTA b serves queues b, b + grid, ...;
    otherwise every CTA keeps one queue"""
    return cdiv(n_queues, pl.grid) if n_queues > pl.grid else min(n_queues, 1)


def copy_groups(pl, s):
    """copy groups (bulk copies on their own mbarrier, at most kCopyGroups = 8) that load stage s"""
    nsubs = min(pl.per, pl.nsub - s * pl.per)
    gs = cdiv(nsubs, min(pl.per, 8))
    return cdiv(nsubs, gs)


def host_sub_batches(P):
    """row counts of the host entry point's sub-batches on one GPU (sub_batch_rows); P <= SMALL_BATCH is one call"""
    out, j = [], 0
    while P > 0:
        want = SUB_BATCH_ROWS * min(j + 1, 4)
        nb = P if P < want + SUB_BATCH_ROWS // 2 else want
        out.append(nb)
        P -= nb
        j += 1
    return out


def persistent(P, no_fused=False):
    """a bit-sliced, non-empty table takes the persistent kernel above the fused kernel's size (or when forced)"""
    return P > FUSED_ROWS_MAX or no_fused


def tune_value(env, key):
    """the number after `key` in an RPK_TUNE string, parsed like parse_tune (select.cu); 0 when absent"""
    i = env.find(key)
    if i < 0:
        return 0
    digits = ""
    for ch in env[i + len(key):]:
        if not ch.isdigit():
            break
        digits += ch
    return int(digits or 0)


def tune_from_env(env):
    """(stage_kb, items_per_warp, k0ctas) of an RPK_TUNE string"""
    return tune_value(env, "stagekb="), tune_value(env, "ipw="), tune_value(env, "k0ctas=")


# ---- the packed and wide kernels (kinds 3 / 2 / 1) -------------------------------------------------------------------
def rows_per_warp(P, sm):
    """pick_rows_per_warp: the most rows per warp (16, 8, 4, 2) that still give ~4 waves of 3 CTAs per SM, else 1"""
    for r in (16, 8, 4, 2):
        if cdiv(P, WARPS_PER_CTA * r) >= sm * 12:
            return r
    return 1


def rows_per_warp_bounds(sm):
    """the smallest P at which rows_per_warp reaches 2, 4, 8 and 16"""
    return [(sm * 12 - 1) * WARPS_PER_CTA * r + 1 for r in (2, 4, 8, 16)]


def tiles_max(P, R):
    """select_tiles_max: row tiles of R rows per warp, every row group ending in at most one partial tile"""
    return cdiv(P, WARPS_PER_CTA * R) + GROUPS


def grid_segments(kind, G):
    """(S, segment length) of the offer segments: packed_pos (3) takes fixed 2^14-offer segments, since its words carry
    the position inside the segment; packed (2) and wide (1) split the table evenly (seg_plan) into segments of at
    most 16 384 and 4 096 offers, each a multiple of 128"""
    Gc = cdiv(G, CHUNK) * CHUNK
    if kind == 3:
        return max(cdiv(Gc, SEG_PACKED), 1), SEG_PACKED
    assert kind in (1, 2), kind
    S = max(cdiv(Gc, SEG_PACKED if kind == 2 else SEG_WIDE), 1)
    return S, cdiv(cdiv(Gc, S), CHUNK) * CHUNK


def grid_launches(P, R, S, grid_tiles=0):
    """[(first tile, CTAs)] of launch_grid: tiles_max x S CTAs in launches of at most GRID_X_MAX // S whole tiles
    (RPK_TUNE gridtiles=N: at most N)"""
    tiles = tiles_max(P, R)
    per = min(tiles, GRID_X_MAX // S)
    if grid_tiles > 0:
        per = min(per, grid_tiles)
    return [(t0, min(per, tiles - t0) * S) for t0 in range(0, tiles, per)]


def row_groups(kind, dist, pods):
    """rows per k_pod_prep row group, cloud * 4 + (vcpu threshold > 0) * 2 + (ram threshold > 0); the generic kernel
    (kind 1) has no rank thresholds and puts every row in group 3 or 7; rows of neither cloud join no group"""
    P = len(pods["req_mem_gb"])
    cloud = pods.get("cloud")
    cloud = np.zeros(P, np.int64) if cloud is None else np.asarray(cloud).astype(np.int64)
    if kind == 1:
        need = np.full(P, 3, np.int64)
    else:
        th = [np.searchsorted(d, np.zeros(P, np.int32) if pods.get(k) is None else pods[k], side="left") > 0
              for d, k in zip(dist[1:], ("req_vcpu", "req_ram_gb"))]
        need = th[0] * 2 + th[1]
    keep = cloud <= 1
    return np.bincount(cloud[keep] * 4 + need[keep], minlength=GROUPS)


def valid_tiles(counts, R):
    """row tiles holding rows (decode_tile's total_tiles): tiles [0, valid_tiles) are walked, later ones return"""
    return int(sum(cdiv(int(n), WARPS_PER_CTA * R) for n in counts))


def top5_rows_per_pass(P, sm):
    """rows (one warp each) of one grid-stride pass of k_select_top5: min(ceil(P / 8), 32 x sm) blocks of 8 warps"""
    return min(cdiv(P, 8), 32 * sm) * 8
