"""The reach rule of rpk_offers_refresh (include/rpk.h, rpk_select_pending_changed) in numpy.

A row's stored list L was selected against an earlier table; the current table differs from it only at the offer
indices in `changed`.  The row's list under the current table is L unless a changed offer reaches the row: it is in L,
or it is feasible for the row now and L has fewer than five entries or (price(c), c) < (price(L[4]), L[4])."""
import numpy as np

COLS = ("mem_gb", "vcpu", "ram_gb", "secure_price", "community_price", "flags")


def column(offers, name):
    G = len(offers["mem_gb"])
    v = offers.get(name)
    return np.zeros(G, np.int32) if v is None else np.asarray(v)


def changed_offers(old, new):
    """ascending indices of the offers whose six columns differ bit for bit (same G)"""
    diff = np.zeros(len(old["mem_gb"]), bool)
    for k in COLS:
        a, b = column(old, k), column(new, k)
        diff |= (a.view(np.uint8).reshape(len(a), -1) != b.view(np.uint8).reshape(len(b), -1)).any(axis=1)
    return np.flatnonzero(diff)


def reached(offers, pods, top5, changed):
    """bool[P]: some offer of `changed` reaches row p, whose stored list is top5[p], under the current table `offers`"""
    P = len(pods["req_mem_gb"])
    changed = np.asarray(changed, np.int64)
    if not len(changed) or not P:
        return np.zeros(P, bool)
    mem, vcpu, ram = (column(offers, k)[changed][None, :] for k in ("mem_gb", "vcpu", "ram_gb"))
    sp, cp = column(offers, "secure_price"), column(offers, "community_price")
    flags = column(offers, "flags")[changed][None, :]
    req_vcpu = pods.get("req_vcpu") if pods.get("req_vcpu") is not None else np.zeros(P, np.int32)
    req_ram = pods.get("req_ram_gb") if pods.get("req_ram_gb") is not None else np.zeros(P, np.int32)
    mx = pods.get("max_price") if pods.get("max_price") is not None else np.full(P, 0.5)
    cloud = pods.get("cloud") if pods.get("cloud") is not None else np.zeros(P, np.uint8)
    cloud = cloud.astype(np.int64)[:, None]
    in_list = (top5[:, :, None] == changed[None, None, :]).any(axis=1)
    price = np.where(cloud == 1, cp[changed][None, :], sp[changed][None, :])
    bit = np.where(cloud == 1, 2, 1)
    with np.errstate(invalid="ignore"):
        feasible = ((cloud <= 1) & ((flags & bit) != 0) & (price > 0) & (price < mx[:, None]) &
                    (mem >= pods["req_mem_gb"][:, None]) & (vcpu >= req_vcpu[:, None]) & (ram >= req_ram[:, None]))
        l4 = top5[:, 4].astype(np.int64)[:, None]
        p4 = np.where(cloud == 1, cp[np.maximum(l4, 0)], sp[np.maximum(l4, 0)])
        before = (l4 < 0) | (price < p4) | ((price == p4) & (changed[None, :] < l4))
    return in_list.any(axis=1) | (feasible & before).any(axis=1)
