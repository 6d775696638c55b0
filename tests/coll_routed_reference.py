"""Reference of the device-routed expert dispatch (b200collExpertDispatch), in numpy: from every rank's expert ids, the route of every
slot, the rows stored per local expert, the dropped rows, and which (source rank, token) every row of every recv holds; the seeded
routings the routed tests draw, and the combine's lookup of a route."""
import numpy as np

INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1


def routing(kind, n, E, k, seed, tokens=None, skew=1.2):
    """One [tokens, top_k] int32 array per rank. uniform; zipf (expert_dispatch_plan's skewed draw, popularity 1 / rank^skew); one
    (every slot to one expert); mixed: uniform with every kind of invalid id, a token naming one expert twice, and (n > 1) a last rank
    with no tokens."""
    rng = np.random.default_rng(seed)
    tokens = tokens or [17 + 5 * s for s in range(n)]
    if kind == "zipf":
        from container_engine_accelerators_b200.models.workloads import expert_dispatch_plan
        p = expert_dispatch_plan(n, max(tokens), 16, experts_per_rank=E // n, top_k=k, skew=skew, seed=seed)
        return [p.experts[s][:tokens[s]] for s in range(n)]
    if kind == "one":
        return [np.full((tokens[s], k), (seed * 7) % E, dtype=np.int32) for s in range(n)]
    out = [rng.integers(0, E, size=(tokens[s], k)).astype(np.int64) for s in range(n)]
    if kind == "mixed":
        bad = [-1, -2, E, E + 3, INT32_MIN, INT32_MAX]
        for s in range(n):
            ids = out[s]
            pos = rng.choice(ids.size, size=min(ids.size, len(bad)), replace=False)
            for i, p in enumerate(pos):
                ids.flat[p] = bad[i]
            if k >= 2 and ids.shape[0] >= 2:
                ids[1, 0] = ids[1, 1] = s % E                           # the same expert twice
        if n > 1:
            out[-1] = np.zeros((0, k), dtype=np.int64)
    return [o.astype(np.int32) for o in out]


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
        tok, dest, rows = slots[keep] // np.shape(topk[s])[1], owner[e[keep]], row[keep]
        for d in range(n):
            at = dest == d
            source[d][rows[at], 0] = s
            source[d][rows[at], 1] = tok[at]
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
    src = lay.source[d]
    for s in range(len(xs)):
        at = src[:, 0] == s
        want[at] = xs[s][src[at, 1]]
    return want


def route_lookup(eo, recv_rows):
    """coll_combine_reference.combine's lookup for routes: route in [0, nranks * recv_rows) names row route % recv_rows of rank
    route // recv_rows."""
    n = len(eo)

    def f(col):
        col = np.asarray(col, dtype=np.int64)
        valid = (col >= 0) & (col < n * recv_rows)
        y = np.zeros((col.size, eo[0].shape[1]), dtype=np.float32)
        i = np.nonzero(valid)[0]
        for p in range(n):
            at = i[col[i] // recv_rows == p]
            y[at] = eo[p][col[at] % recv_rows]
        return valid, y
    return f
