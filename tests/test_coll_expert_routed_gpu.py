"""Device-routed expert dispatch and combine on an H100 (`pytest -m gpu`), virtual ranks sharing cuda:0 unless said otherwise.

Every recv starts poisoned with 0x5A; stored rows are compared byte for byte with tests/coll_routed_reference.layout (NaN payloads and
-0 included), every other row must keep the poison, and expert_counts, route and dropped must match exactly. Combine outputs are
compared bit for bit with tests/coll_combine_reference.combine through a route lookup."""
import ctypes as C

import numpy as np
import pytest

from container_engine_accelerators_b200.ops.coll import INVALID_ARGUMENT, INVALID_USAGE
from tests import coll_combine_reference as cr
from tests import coll_quant_reference as qr
from tests import coll_routed_reference as rr
from tests.coll_fp_reference import assert_same
from tests.coll_gpu_harness import DTYPES, Group, assert_nothing_launched, coll_mod, expect_refused, run_perf, torch_cuda  # noqa: F401
from tests.coll_routed_reference import INT32_MAX, INT32_MIN, route_lookup, routing

pytestmark = pytest.mark.gpu
ROW = 48
POISON = 0x5A


def _x_bytes(rng, tokens, row_bytes, esize):
    """Random bits, with -0 and a NaN payload in every row (raw bits: the dispatch must move them unchanged)."""
    x = rng.integers(0, 256, size=(tokens, row_bytes), dtype=np.uint8)
    if tokens:
        neg0 = {2: [0x00, 0x80], 4: [0, 0, 0, 0x80]}[esize]
        nan = {2: [0x35, 0x7F], 4: [0x35, 0x12, 0xC1, 0x7F]}[esize]
        x[:, :esize] = neg0
        x[:, esize:2 * esize] = nan
    return x


def dev_rows(g, c, a, dt):
    """[tokens, row bytes] uint8 rows on c's device, viewed as dt (also for tokens == 0)."""
    t = g.torch.empty(a.shape, dtype=g.torch.uint8, device=f"cuda:{c.device}")
    if a.size:
        t.copy_(g.torch.from_numpy(np.ascontiguousarray(a)))
    return t.view(dt)


def recv_bufs(g, recv_rows, dt):
    bufs = [c.empty(recv_rows * ROW, dt) for c in g.comms]
    for b in bufs:
        b.view(g.torch.uint8).fill_(POISON)
    return bufs


def small_outputs(g, topk, E):
    """Every rank's (expert_counts, route, dropped), allocated up front like every other buffer here, so the loop over ranks only
    enqueues."""
    torch = g.torch
    return [(torch.empty(E // g.n, dtype=torch.int32, device=f"cuda:{c.device}"), torch.empty(topk[r].shape, dtype=torch.int32, device=f"cuda:{c.device}"),
             torch.empty(1, dtype=torch.int32, device=f"cuda:{c.device}")) for r, c in enumerate(g.comms)]


def run_dispatch(g, xs_np, topk, E, recv, dt):
    """Dispatch on every rank's stream; returns the CPU copies of (recv bytes, counts, route, dropped) per rank."""
    torch = g.torch
    xd = [dev_rows(g, c, xs_np[r], dt) for r, c in enumerate(g.comms)]
    idx = [g.dev(c, topk[r]) for r, c in enumerate(g.comms)]
    small = small_outputs(g, topk, E)
    g.sync()
    res = []
    for r, c in enumerate(g.comms):
        res.append(c.expert_dispatch(xd[r], idx[r], E, recv[r], *small[r], stream=g.streams[r]))
    g.sync()
    g.check_async()
    return [(o[0].view(torch.uint8).cpu().numpy().reshape(-1, ROW * xd[0].element_size()), o[1].cpu().numpy(), o[2].cpu().numpy(), int(o[3].item()))
            for o in res]


def check_dispatch(lay, xs_np, got, what):
    for d, (rb, counts, route, dropped) in enumerate(got):
        poison = np.full(rb.shape, POISON, dtype=np.uint8)
        want = rr.recv_rows_of(lay, xs_np, d, poison)
        bad = np.nonzero((rb != want).any(axis=1))[0]
        assert bad.size == 0, f"{what}: rank {d} recv rows {bad[:8].tolist()} differ"
        assert (counts == lay.counts[d]).all(), f"{what}: rank {d} counts {counts.tolist()} want {lay.counts[d].tolist()}"
        assert (route == lay.route[d]).all(), f"{what}: rank {d} route differs"
        assert dropped == lay.dropped[d], f"{what}: rank {d} dropped {dropped} want {lay.dropped[d]}"


def _configs(n):
    cfg = [(n, 1), (4 * n, 2), (8 * n, 8)]
    if n == 8:
        cfg.append((256, 8))
    return cfg


@pytest.mark.parametrize("dt_name", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_dispatch_bit_exact(torch_cuda, coll_mod, n, dt_name):
    """(E, top_k) in (N, 1), (4N, 2), (8N, 8) (and 256 experts top-8 at 8 ranks) x uniform, Zipf, one-expert and mixed routings x ample
    and tight capacity; two launches per call and the stats under alltoall."""
    torch, coll = torch_cuda, coll_mod
    dt = DTYPES[dt_name]
    es = dt.itemsize
    with Group(torch, coll, n) as g:
        rng = np.random.default_rng(n * 100 + es)
        clipped_inside = 0
        for E, k in _configs(n):
            for kind in ("uniform", "zipf", "one", "mixed"):
                topk = routing(kind, n, E, k, seed=E + k + n)
                ample = rr.layout(topk, E, 1 << 20)
                load = max(int(c.sum()) for c in ample.counts)
                for cap_name, recv_rows in (("ample", load + 3), ("tight", max(1, load * 3 // 5))):
                    lay = rr.layout(topk, E, recv_rows)
                    totals = rr.layout(topk, E, 1 << 20).counts
                    clipped_inside += sum(int(((lay.counts[d] > 0) & (lay.counts[d] < totals[d])).sum()) for d in range(n))
                    xs = [_x_bytes(rng, t.shape[0], ROW * es, es) for t in topk]
                    recv = recv_bufs(g, recv_rows, dt)
                    before = [c.stats() for c in g.comms]
                    got = run_dispatch(g, xs, topk, E, recv, dt)
                    what = f"n={n} {dt_name} E={E} top_k={k} {kind} {cap_name}"
                    check_dispatch(lay, xs, got, what)
                    for r, c in enumerate(g.comms):
                        st, b = c.stats(), before[r]
                        assert st["kernel_launches"] == b["kernel_launches"] + 2, what
                        algo = "copy" if n == 1 else "twoshot"
                        assert st["algo_calls"][algo] == b["algo_calls"][algo] + 1, what
                        assert st["calls"][coll.OP_ALLTOALL] == b["calls"][coll.OP_ALLTOALL] + 1, what
                        assert st["bytes"][coll.OP_ALLTOALL] == b["bytes"][coll.OP_ALLTOALL] + topk[r].size * ROW * es, what
                    for c, b in zip(g.comms, recv):
                        c.release(b)
        assert clipped_inside > 0                                      # some receiver stored part of an expert


def _spoil(route, n, recv_rows, rng):
    r = route.astype(np.int64).copy()
    if r.size:
        bad = [-1, INT32_MIN, INT32_MAX, n * recv_rows]
        for i, p in enumerate(rng.choice(r.size, size=min(r.size, 8), replace=False)):
            r.flat[p] = bad[i % len(bad)]
    return r.astype(np.int32)


@pytest.mark.parametrize("n", [1, 2, 4])
def test_combine_bit_exact(torch_cuda, coll_mod, n):
    """Every type pair, with weights and without, on routes from a dispatch and on spoiled routes (-1, INT32_MIN, INT32_MAX,
    nranks * recv_rows); one launch per call, the stats under alltoall."""
    torch, coll = torch_cuda, coll_mod
    with Group(torch, coll, n) as g:
        rng = np.random.default_rng(n)
        E, k = 4 * n, 3
        topk = routing("mixed", n, E, k, seed=5)
        recv_rows = max(1, max(int(c.sum()) for c in rr.layout(topk, E, 1 << 20).counts) * 4 // 5)
        recv = recv_bufs(g, recv_rows, torch.bfloat16)
        xs = [_x_bytes(rng, t.shape[0], ROW * 2, 2) for t in topk]
        got = run_dispatch(g, xs, topk, E, recv, torch.bfloat16)
        routes = [o[2] for o in got]
        for r in range(n):
            assert (routes[r] == rr.layout(topk, E, recv_rows).route[r]).all()
        for c, b in zip(g.comms, recv):
            c.release(b)
        for in_name in ("bf16", "f16", "f32"):
            in_dt = DTYPES[in_name]
            xs_eo = [qr.gen(recv_rows * ROW, in_dt, 16, 31 * r + 7) for r in range(n)]
            eo = []
            for c, x in zip(g.comms, xs_eo):
                d = c.empty(x.numel(), in_dt)
                d.copy_(x)
                eo.append(d)
            eo_np = [x.float().numpy().reshape(-1, ROW) for x in xs_eo]
            for out_name in ("bf16", "f16", "f32"):
                out_dt = DTYPES[out_name]
                for spoiled in (False, True):
                    rts = [_spoil(rt, n, recv_rows, rng) if spoiled else rt for rt in routes]
                    for weights, scale in ((True, 1.0), (False, 0.75)):
                        w = [rng.uniform(-1.5, 1.5, size=rt.shape).astype(np.float32) for rt in rts]
                        outs = [torch.full((rt.shape[0], ROW), float("nan"), dtype=out_dt, device="cuda") for rt in rts]
                        rd = [g.dev(c, rts[r]) for r, c in enumerate(g.comms)]
                        wd = [g.dev(c, w[r]) if weights else None for r, c in enumerate(g.comms)]
                        g.sync()
                        before = [c.stats() for c in g.comms]
                        for r, c in enumerate(g.comms):
                            c.expert_combine(eo[r], rd[r], wd[r], outs[r], scale=scale, stream=g.streams[r])
                        g.sync()
                        g.check_async()
                        what = f"n={n} {in_name}->{out_name} spoiled={spoiled} weights={weights}"
                        for r, c in enumerate(g.comms):
                            want = cr.combine(route_lookup(eo_np, recv_rows), rts[r], w[r] if weights else None, scale, out_dt)
                            assert_same(outs[r].cpu(), want, f"{what}: rank {r}")
                            st, b = c.stats(), before[r]
                            assert st["kernel_launches"] == b["kernel_launches"] + 1, what
                            algo = "copy" if n == 1 else "oneshot"
                            assert st["algo_calls"][algo] == b["algo_calls"][algo] + 1, what
                            assert st["bytes"][coll.OP_ALLTOALL] == b["bytes"][coll.OP_ALLTOALL] + rts[r].size * ROW * in_dt.itemsize, what
            for c, d in zip(g.comms, eo):
                c.release(d)


@pytest.mark.parametrize("n", [2, 3])
def test_cuda_graph_without_host_sync(torch_cuda, coll_mod, n):
    """Each rank captures dispatch then combine (recv as the expert output) in one CUDA graph; topk_idx is rewritten in place between
    replays so counts, clipping and routes change, and every replay is checked."""
    torch, coll = torch_cuda, coll_mod
    with Group(torch, coll, n) as g:
        rng = np.random.default_rng(40 + n)
        E, k, tokens = 4 * n, 2, 24
        recv_rows = tokens * k * 3 // 4
        recv = recv_bufs(g, recv_rows, torch.bfloat16)
        xs = [_x_bytes(rng, tokens, ROW * 2, 2) for _ in range(n)]
        xs[0][:, :] = (np.arange(ROW * 2) % 7).astype(np.uint8)          # finite values too, so the sums are not all NaN
        xd = [dev_rows(g, c, xs[r], torch.bfloat16) for r, c in enumerate(g.comms)]
        idx = [torch.zeros(tokens, k, dtype=torch.int32, device="cuda") for _ in range(n)]
        w = [rng.uniform(0.1, 1.0, size=(tokens, k)).astype(np.float32) for _ in range(n)]
        wd = [g.dev(c, w[r]) for r, c in enumerate(g.comms)]
        counts = [torch.empty(E // n, dtype=torch.int32, device="cuda") for _ in range(n)]
        route = [torch.empty(tokens, k, dtype=torch.int32, device="cuda") for _ in range(n)]
        dropped = [torch.empty(1, dtype=torch.int32, device="cuda") for _ in range(n)]
        outs = [torch.empty(tokens, ROW, dtype=torch.float32, device="cuda") for _ in range(n)]
        g.sync()
        graphs = []
        for r, c in enumerate(g.comms):
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=g.streams[r]):
                c.expert_dispatch(xd[r], idx[r], E, recv[r], counts[r], route[r], dropped[r])
                c.expert_combine(recv[r].view(-1, ROW), route[r], wd[r], outs[r])
            graphs.append(gr)
        for rep, kind in enumerate(("uniform", "one", "mixed", "zipf")):
            topk = routing(kind, n, E, k, seed=rep, tokens=[tokens] * n)
            topk = [t if t.shape[0] == tokens else np.full((tokens, k), -1, dtype=np.int32) for t in topk]
            for r in range(n):
                idx[r].copy_(torch.from_numpy(topk[r]))
            for b in recv:
                b.view(torch.uint8).fill_(POISON)
            g.sync()
            for r, gr in enumerate(graphs):
                with torch.cuda.stream(g.streams[r]):
                    gr.replay()
            g.sync()
            g.check_async()
            lay = rr.layout(topk, E, recv_rows)
            got = [(recv[r].view(torch.uint8).cpu().numpy().reshape(-1, ROW * 2), counts[r].cpu().numpy(), route[r].cpu().numpy(), int(dropped[r].item()))
                   for r in range(n)]
            check_dispatch(lay, xs, got, f"replay {rep} ({kind})")
            eo = [recv[r].float().cpu().numpy().reshape(-1, ROW) for r in range(n)]
            for r in range(n):
                want = cr.combine(route_lookup(eo, recv_rows), lay.route[r], w[r], 1.0, torch.float32)
                assert_same(outs[r].cpu(), want, f"replay {rep} ({kind}): combine rank {r}")
        del graphs


def test_interleaved_with_other_collectives(torch_cuda, coll_mod):
    """dispatch, all_reduce, combine, all_to_all_v, dispatch on every rank's stream, then every result checked: the epochs and the
    count mailbox stay in step with the other collectives."""
    torch, coll = torch_cuda, coll_mod
    n, E, k, tokens = 4, 16, 2, 40
    with Group(torch, coll, n) as g:
        rng = np.random.default_rng(3)
        t1, t2 = routing("zipf", n, E, k, seed=1, tokens=[tokens] * n), routing("uniform", n, E, k, seed=2, tokens=[tokens] * n)
        recv_rows = tokens * k
        r1, r2 = recv_bufs(g, recv_rows, torch.float32), recv_bufs(g, recv_rows, torch.float32)
        xs = [_x_bytes(rng, tokens, ROW * 4, 4) for _ in range(n)]
        xs[0][:, 8:] = 0
        xd = [dev_rows(g, c, xs[r], torch.float32) for r, c in enumerate(g.comms)]
        i1 = [g.dev(c, t1[r]) for r, c in enumerate(g.comms)]
        i2 = [g.dev(c, t2[r]) for r, c in enumerate(g.comms)]
        ar = [c.empty(4096, torch.float32) for c in g.comms]
        for r, a in enumerate(ar):
            a.fill_(float(r + 1))
        from container_engine_accelerators_b200.models.workloads import expert_dispatch_plan
        p = expert_dispatch_plan(n, 20, ROW, top_k=1, seed=9)
        sends = [torch.randn(20 * ROW, device="cuda").to(torch.bfloat16) for _ in range(n)]
        a2a = [c.empty(p.max_rows * ROW, torch.bfloat16) for c in g.comms]
        outs = [torch.empty(tokens, ROW, dtype=torch.bfloat16, device="cuda") for _ in range(n)]
        s1, s2 = small_outputs(g, t1, E), small_outputs(g, t2, E)
        g.sync()
        # each operation enqueued for every rank before the next one, no host sync in between: every stream runs the five in order
        res1 = [c.expert_dispatch(xd[r], i1[r], E, r1[r], *s1[r], stream=g.streams[r]) for r, c in enumerate(g.comms)]
        for r, c in enumerate(g.comms):
            c.all_reduce(ar[r], stream=g.streams[r])
        for r, c in enumerate(g.comms):
            c.expert_combine(r1[r].view(-1, ROW), res1[r][2], None, outs[r], stream=g.streams[r])
        for r, c in enumerate(g.comms):
            c.all_to_all_v(sends[r], a2a[r], ROW, p.rows[r].tolist(), p.send_off[r].tolist(), [int(p.recv_off[d, r]) for d in range(n)], stream=g.streams[r])
        res2 = [c.expert_dispatch(xd[r], i2[r], E, r2[r], *s2[r], stream=g.streams[r]) for r, c in enumerate(g.comms)]
        g.sync()
        g.check_async()
        for t, res in ((t1, res1), (t2, res2)):
            lay = rr.layout(t, E, recv_rows)
            got = [(o[0].view(torch.uint8).cpu().numpy().reshape(-1, ROW * 4), o[1].cpu().numpy(), o[2].cpu().numpy(), int(o[3].item())) for o in res]
            check_dispatch(lay, xs, got, "interleaved dispatch")
        lay = rr.layout(t1, E, recv_rows)
        eo = [r1[r].cpu().numpy().reshape(-1, ROW) for r in range(n)]
        for r in range(n):
            assert_same(outs[r].cpu(), cr.combine(route_lookup(eo, recv_rows), lay.route[r], None, 1.0, torch.bfloat16), f"interleaved combine rank {r}")
            assert bool((ar[r] == float(n * (n + 1) // 2)).all())
            for s in range(n):
                lo, cnt = int(p.recv_off[r, s]), int(p.rows[s, r])
                want = sends[s][int(p.send_off[s, r]) * ROW:(int(p.send_off[s, r]) + cnt) * ROW]
                assert torch.equal(a2a[r][lo * ROW:(lo + cnt) * ROW], want)


def _raw_dispatch(coll, comm, **a):
    i32 = lambda p: C.cast(C.c_void_p(p), C.POINTER(C.c_int32))
    return coll.load().b200collExpertDispatch(C.c_void_p(a["x"]), C.c_void_p(a["recv"]), a["row_elems"], a["recv_rows"], i32(a["topk"]), a["tokens"],
                                              a["top_k"], a["E"], i32(a["counts"]), i32(a["route"]), i32(a["dropped"]), a["dt"], comm._h, None)


def _raw_combine(coll, comm, **a):
    ep = coll.Epilogue(a["in_dt"], a["out_dt"], 1.0)
    return coll.load().b200collExpertCombine(C.c_void_p(a["eo"]), C.c_void_p(a["out"]), a["row_elems"], a["recv_rows"],
                                             C.cast(C.c_void_p(a["route"]), C.POINTER(C.c_int32)), C.cast(C.c_void_p(a["weights"]), C.POINTER(C.c_float)),
                                             a["tokens"], a["top_k"], C.byref(ep), comm._h, None)


def test_refusals_launch_nothing(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    with Group(torch, coll, 2) as g:
        c = g.comms[0]
        row, rows_n, tokens, k = 64, 16, 4, 2
        recv = c.empty(rows_n * row, torch.bfloat16)
        plain = torch.empty(rows_n * row, dtype=torch.bfloat16, device="cuda")
        x = torch.empty(tokens, row, dtype=torch.bfloat16, device="cuda")
        small = torch.zeros(256, dtype=torch.int32, device="cuda")
        TK, CN, RT, DR = small.data_ptr(), small.data_ptr() + 64, small.data_ptr() + 128, small.data_ptr() + 192
        R, X = recv.data_ptr(), x.data_ptr()
        BF, E4 = coll.BF16, coll.FP8_E4M3
        ok = dict(x=X, recv=R, row_elems=row, recv_rows=rows_n, topk=TK, tokens=tokens, top_k=k, E=4, counts=CN, route=RT, dropped=DR, dt=BF)
        # (what, code, arguments that break only that rule, the words of the rule in the error text)
        cases = [("recv outside the arena", INVALID_USAGE, dict(recv=plain.data_ptr()), "symmetric arena")] + [(what, INVALID_ARGUMENT, kw, msg) for what, kw, msg in [
            ("null x", dict(x=0), "null argument"), ("null recv", dict(recv=0), "null argument"), ("null topk_idx", dict(topk=0), "null argument"),
            ("null expert_counts", dict(counts=0), "null argument"), ("null route", dict(route=0), "null argument"),
            ("null dropped", dict(dropped=0), "null argument"), ("FP8 rows", dict(dt=E4), "dtype must be"), ("int32 rows", dict(dt=coll.I32), "dtype must be"),
            ("row_elems 0", dict(row_elems=0), "row_elems"), ("row_elems 40", dict(row_elems=40), "row_elems"), ("top_k 0", dict(top_k=0), "top_k must be"),
            ("0 experts", dict(E=0), "num_experts"), ("1025 experts", dict(E=1025), "num_experts"), ("3 experts for 2 ranks", dict(E=3), "num_experts"),
            ("misaligned x", dict(x=X + 8), "16-byte aligned"), ("misaligned recv", dict(recv=R + 8), "16-byte aligned"),
            ("misaligned topk_idx", dict(topk=TK + 2), "4-byte aligned"), ("misaligned expert_counts", dict(counts=CN + 1), "4-byte aligned"),
            ("misaligned route", dict(route=RT + 2), "4-byte aligned"), ("misaligned dropped", dict(dropped=DR + 3), "4-byte aligned"),
            ("recv overlaps x", dict(x=R), "recv must not overlap x"), ("route overlaps expert_counts", dict(route=CN), "each other"),
            ("dropped overlaps route", dict(dropped=RT + 4), "each other"), ("route overlaps topk_idx", dict(route=TK + 4), "topk_idx, x or recv"),
            ("expert_counts in recv", dict(counts=R + 64), "topk_idx, x or recv"), ("dropped in x", dict(dropped=X), "topk_idx, x or recv"),
            ("tokens * top_k > 2^31 - 1", dict(tokens=1 << 30, top_k=2, row_elems=16), "tokens * top_k"),
            ("nranks * recv_rows > 2^31 - 1", dict(recv_rows=1 << 30), "nranks * recv_rows"),
            ("more than 2^31 - 1 vectors", dict(tokens=1 << 24, top_k=8, row_elems=512), "16-byte vectors"),  # 2^27 slots x 64 vectors
        ]]
        for what, want, kw, msg in cases:
            expect_refused(_raw_dispatch(coll, c, **dict(ok, **kw)), want, msg, what=what)
        eo = c.empty(rows_n * row, torch.bfloat16)
        out = torch.empty(tokens, row, dtype=torch.bfloat16, device="cuda")
        wts = torch.ones(tokens, k, device="cuda")
        EO, O, W = eo.data_ptr(), out.data_ptr(), wts.data_ptr()
        okc = dict(eo=EO, out=O, row_elems=row, recv_rows=rows_n, route=RT, weights=W, tokens=tokens, top_k=k, in_dt=BF, out_dt=BF)
        ccases = [("expert_out outside the arena", INVALID_USAGE, dict(eo=plain.data_ptr()), "symmetric arena")] + [(what, INVALID_ARGUMENT, kw, msg) for what, kw, msg in [
            ("null expert_out", dict(eo=0), "null argument"), ("null out", dict(out=0), "null argument"), ("null route", dict(route=0), "null argument"),
            ("FP8 in", dict(in_dt=E4), "in_dtype and out_dtype"), ("FP8 out", dict(out_dt=E4), "in_dtype and out_dtype"),
            ("row_elems 40", dict(row_elems=40), "row_elems"), ("top_k 0", dict(top_k=0), "top_k must be"),
            ("misaligned expert_out", dict(eo=EO + 8), "16-byte aligned"), ("misaligned out", dict(out=O + 4), "16-byte aligned"),
            ("misaligned route", dict(route=RT + 2), "4-byte aligned"), ("misaligned weights", dict(weights=W + 1), "4-byte aligned"),
            ("out overlaps expert_out", dict(out=EO), "out must not overlap"), ("out overlaps route", dict(route=O + 16), "out must not overlap"),
            ("out overlaps weights", dict(weights=O + 64), "out must not overlap"), ("nranks * recv_rows > 2^31 - 1", dict(recv_rows=1 << 30), "nranks * recv_rows"),
            ("more than 2^31 - 1 vectors of out", dict(tokens=1 << 28, row_elems=128), "vectors of out"),
            ("tokens * top_k > 2^31 - 1", dict(tokens=1 << 30, top_k=4, row_elems=16), "tokens * top_k"),
        ]]
        for what, want, kw, msg in ccases:
            expect_refused(_raw_combine(coll, c, **dict(okc, **kw)), want, msg, what=what)
        with pytest.raises(ValueError):
            c.expert_dispatch(x, torch.zeros(tokens, k, dtype=torch.int32, device="cuda"), 3, recv)       # 3 experts for 2 ranks
        with pytest.raises(ValueError):
            c.expert_combine(eo, torch.zeros(tokens, k, dtype=torch.int64, device="cuda"), None, out)
        assert_nothing_launched(c)
        g.check_async()


def _perf_route(devs, procs, extra):
    out = run_perf(["--op", "alltoall", *extra, "-w", "1", "-n", "2", "-c", "1"], devs, procs, env={"B200COLL_TIMEOUT_MS": "20000"})
    assert [l for l in out.splitlines() if l.strip() and not l.startswith("#")], out


def test_two_processes_on_two_gpus(torch_cuda, coll_lib):
    """One process per rank, one GPU per process: the perf tool's --procs mode forks the ranks, which rendezvous over the bootstrap
    and check every received byte, count, route and combine output against the host layout."""
    if torch_cuda.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    _perf_route("0,1", True, ["-d", "bfloat16", "--route", "16:4", "--row-len", "7168", "-b", "1M", "-e", "16M", "-f", "4"])
    _perf_route("0,1", True, ["-d", "float", "--out-dtype", "bfloat16", "--route", "256:8", "-b", "256K", "-e", "256K"])


def test_two_processes_on_one_gpu(torch_cuda, coll_lib):
    """The same two-process protocol with both ranks on cuda:0, so it also runs on a one-GPU machine."""
    _perf_route("0,0", True, ["-d", "bfloat16", "--route", "16:4", "-b", "64K", "-e", "1M", "-f", "4"])


def test_multi_gpu(torch_cuda, coll_mod):
    """One process driving two GPUs: the library makes each communicator's device current for its calls."""
    torch, coll = torch_cuda, coll_mod
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    n = 2
    with Group(torch, coll, n, devices=[0, 1]) as g:
        rng = np.random.default_rng(11)
        E, k = 8, 4
        topk = routing("zipf", n, E, k, seed=3, tokens=[300, 200])
        recv_rows = max(int(c.sum()) for c in rr.layout(topk, E, 1 << 20).counts) * 4 // 5
        lay = rr.layout(topk, E, recv_rows)
        xs = [_x_bytes(rng, t.shape[0], ROW * 2, 2) for t in topk]
        recv = recv_bufs(g, recv_rows, torch.bfloat16)
        got = run_dispatch(g, xs, topk, E, recv, torch.bfloat16)
        check_dispatch(lay, xs, got, "two GPUs")
        outs = [torch.empty(t.shape[0], ROW, dtype=torch.float32, device=f"cuda:{c.device}") for t, c in zip(topk, g.comms)]
        routes = [g.dev(c, lay.route[r]) for r, c in enumerate(g.comms)]
        g.sync()
        for r, c in enumerate(g.comms):
            c.expert_combine(recv[r].view(-1, ROW), routes[r], None, outs[r], stream=g.streams[r])
        g.sync()
        g.check_async()
        eo = [recv[r].float().cpu().numpy().reshape(-1, ROW) for r in range(n)]
        for r in range(n):
            assert_same(outs[r].cpu(), cr.combine(route_lookup(eo, recv_rows), lay.route[r], None, 1.0, torch.float32), f"two GPUs combine rank {r}")


def test_perf_tool_route_mode(torch_cuda, coll_lib):
    for devs, extra in (("0", ["-d", "bfloat16", "--route", "16:4", "-b", "64K", "-e", "1M", "-f", "4"]),
                        ("0,0", ["-d", "float", "--route", "8:2", "--row-len", "96", "-b", "256K", "-e", "256K"]),
                        ("0,0", ["-d", "half", "--route", "256:8", "-b", "1M", "-e", "1M"])):
        out = run_perf(["--op", "alltoall", *extra, "-w", "1", "-n", "2", "-c", "1"], devs)
        rows = [l for l in out.splitlines() if l.strip() and not l.startswith("#")]
        assert rows, out
