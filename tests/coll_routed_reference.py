"""Reference of the device-routed expert dispatch (b200collExpertDispatch), in numpy: from every rank's expert ids, the route of every
slot, the rows stored per local expert, the dropped rows, and which (source rank, token) every row of every recv holds."""
import numpy as np


class Layout:
    """route[s]: int32 [tokens, top_k] (peer * recv_rows + row, or -1); counts[d]: int32 [E / N]; dropped[d]: int; source[d]: int64
    [recv_rows, 2] (source rank, token) of each stored row of d's recv, (-1, -1) for a row nothing lands in."""

    def __init__(self, route, counts, dropped, source):
        self.route, self.counts, self.dropped, self.source = route, counts, dropped, source


def layout(topk, num_experts, recv_rows):
    """topk: one [tokens, top_k] integer array per rank (tokens may differ between ranks). Expert e lives on rank e // (E / N); an id
    outside [0, E) drops its slot. Rank d's recv holds its experts ascending, each expert's rows by source rank, then in row-major
    (token, slot) order; rows at or past recv_rows are dropped."""
    n, E = len(topk), num_experts
    epr = E // n
    flats = [np.asarray(t, dtype=np.int64).reshape(-1) for t in topk]
    cnt = np.zeros((n, E), dtype=np.int64)
    for s, f in enumerate(flats):
        ok = (f >= 0) & (f < E)
        cnt[s] = np.bincount(f[ok], minlength=E)
    total = cnt.sum(axis=0)
    below = np.concatenate([[0], np.cumsum(total)[:-1]])             # rows of all experts below e
    owner = np.arange(E) // epr
    base = below - below[owner * epr]                                # rows of the owner's experts below e
    routes = []
    source = [np.full((recv_rows, 2), -1, dtype=np.int64) for _ in range(n)]
    for s, f in enumerate(flats):
        ok = (f >= 0) & (f < E)
        rank = np.zeros(f.size, dtype=np.int64)
        slots = np.nonzero(ok)[0]
        order = np.argsort(f[slots], kind="stable")                  # slots grouped by expert, slot order kept within a group
        keys = f[slots][order]
        first = np.searchsorted(keys, keys, side="left")
        rank[slots[order]] = np.arange(keys.size) - first
        route = np.full(f.size, -1, dtype=np.int64)
        e = f[slots]
        row = base[e] + cnt[:s, e].sum(axis=0) + rank[slots]
        keep = row < recv_rows
        route[slots[keep]] = owner[e[keep]] * recv_rows + row[keep]
        routes.append(route.reshape(np.shape(topk[s])).astype(np.int32))
        tok = slots[keep] // np.shape(topk[s])[1]
        for d, r, t in zip(owner[e[keep]], row[keep], tok):
            source[d][r] = (s, t)
    counts, dropped = [], []
    for d in range(n):
        mine = slice(d * epr, (d + 1) * epr)
        stored = np.clip(recv_rows - base[mine], 0, total[mine])
        counts.append(stored.astype(np.int32))
        dropped.append(int(total[mine].sum() - stored.sum()))
    return Layout(routes, counts, dropped, source)


def brute_force(topk, num_experts, recv_rows):
    """The same layout, placed one slot at a time: for every receiver, its experts in order, the sources in order, the slots in order."""
    n, E = len(topk), num_experts
    epr = E // n
    routes = [np.full(np.shape(t), -1, dtype=np.int64) for t in topk]
    source = [np.full((recv_rows, 2), -1, dtype=np.int64) for _ in range(n)]
    counts, dropped = [], []
    for d in range(n):
        row, cnt, drop = 0, [], 0
        for e in range(d * epr, (d + 1) * epr):
            stored = 0
            for s in range(n):
                ids = np.asarray(topk[s]).reshape(np.shape(topk[s]))
                for t in range(ids.shape[0]):
                    for j in range(ids.shape[1]):
                        if ids[t, j] != e:
                            continue
                        if row < recv_rows:
                            routes[s][t, j] = d * recv_rows + row
                            source[d][row] = (s, t)
                            stored += 1
                        else:
                            drop += 1
                        row += 1
            cnt.append(stored)
        counts.append(np.asarray(cnt, dtype=np.int32))
        dropped.append(drop)
    return Layout([r.astype(np.int32) for r in routes], counts, dropped, source)


def recv_rows_of(lay, xs, d, poison):
    """Rank d's expected recv as bytes: row r holds x[s][t] for source[d][r] = (s, t), the poison row elsewhere. xs: one [tokens, row_bytes]
    uint8 array per rank; poison: [recv_rows, row_bytes] uint8."""
    want = poison.copy()
    for r, (s, t) in enumerate(lay.source[d]):
        if s >= 0:
            want[r] = xs[s][t]
    return want
