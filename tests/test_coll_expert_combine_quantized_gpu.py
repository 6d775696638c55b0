"""The quantising expert combine on an H100 (`pytest -m gpu`), virtual ranks sharing cuda:0 unless said otherwise.

Bit-exact means equal (NaN matching NaN at the same position) to tests/coll_combine_reference.combine over the dequantised rows
tests/coll_quant_reference.quantize(row)[2] of every rank's expert_out: each rank quantises its whole expert_out by the per-block rule, and
each slot's row is summed in slot order exactly as the wide combine of the same map sums it."""
import ctypes as C
import numpy as np
import pytest

from container_engine_accelerators_b200.ops.coll import INVALID_ARGUMENT, OUT_OF_MEMORY
from tests import coll_combine_reference as cr
from tests import coll_quant_reference as qr
from tests import coll_routed_reference as rr
from tests.coll_fp_reference import assert_same
from tests.coll_gpu_harness import (DTYPES, Group, Plan, assert_nothing_launched, coll_mod, expect_refused, run_perf, run_python,  # noqa: F401
                                    torch_cuda)
from tests.coll_routed_reference import route_lookup, routing

pytestmark = pytest.mark.gpu

ROW = 512                                                               # whole blocks of every size tested
PAIRS = [(i, o) for i in ("bf16", "f16", "f32") for o in ("bf16", "f16", "f32")]


def segment_plan(topk, E, tight, seed):
    """The all-to-all-v combine of a routing: rank s's send buffer holds its valid slots grouped by destination rank, in slot order, each
    group starting where the previous one ends. With `tight` only the first 3/5 of a group are sent; the others fall in the gap before
    the next group (a dropped slot), as do invalid ids (-1). Destination ranges are packed by source rank."""
    n = len(topk)
    epr = E // n
    rows = np.zeros((n, n), dtype=np.int64)
    send_off = np.zeros((n, n), dtype=np.int64)
    index, weights = [], []
    rng = np.random.default_rng(seed)
    for s, ids in enumerate(topk):
        flat = ids.astype(np.int64).reshape(-1)
        valid = (flat >= 0) & (flat < E)
        dest = np.where(valid, flat // epr, -1)
        idx = np.full(flat.size, -1, dtype=np.int64)
        at = 0
        for d in range(n):
            slots = np.nonzero(dest == d)[0]
            send_off[s, d] = at
            rows[s, d] = slots.size * 3 // 5 if tight else slots.size
            idx[slots] = at + np.arange(slots.size)
            at += slots.size
        index.append(idx.reshape(ids.shape).astype(np.int32))
        weights.append(rng.uniform(-1.5, 1.5, size=ids.shape).astype(np.float32))
    recv_off = np.zeros((n, n), dtype=np.int64)
    for d in range(n):
        recv_off[d] = np.concatenate([[0], np.cumsum(rows[:, d])[:-1]])
    return Plan(rows, send_off, recv_off, index, weights)


def dequantised(torch, eo, block, wire):
    """Per rank: the [recv_rows, ROW] float32 values every row of its expert_out becomes on the wire."""
    return [qr.quantize(e.reshape(-1), block, wire)[2].numpy().reshape(-1, ROW) for e in eo]


def expert_outs(torch, n, recv_rows, in_dt, block, seed, used=None):
    """Per rank a [recv_rows, ROW] CPU tensor from qr.gen (zeros, +-0, +-inf, NaN and a tiny amax in the first blocks); rows at or past
    used[r] hold NaN and inf (no slot reads them)."""
    eo = [qr.gen(recv_rows * ROW, in_dt, block, seed + 13 * r).view(recv_rows, ROW) for r in range(n)]
    for r, e in enumerate(eo):
        if used is not None and used[r] < recv_rows:
            e[used[r]:, ::7] = float("nan")
            e[used[r]:, 3::11] = float("inf")
    return eo


def run(g, kind, plan_or_routes, eo, recv_rows, in_dt, out_dt, wire, block, weights, scale, tokens):
    """One quantising combine on every rank's stream: expert_out a plain tensor (n > 1: outside the arena), out poisoned with NaN.
    Returns (outs, stats before, stats after)."""
    torch = g.torch
    eod = [eo[r].to(in_dt).to(f"cuda:{c.device}") for r, c in enumerate(g.comms)]
    outs = [torch.full((tokens[r], ROW), float("nan"), dtype=out_dt, device=f"cuda:{c.device}") for r, c in enumerate(g.comms)]
    wd = [g.dev(c, weights[r]) if weights is not None else None for r, c in enumerate(g.comms)]
    if kind == "segment":
        idx = [g.dev(c, plan_or_routes.index[r]) for r, c in enumerate(g.comms)]
    else:
        idx = [g.dev(c, plan_or_routes[r]) for r, c in enumerate(g.comms)]
    if g.n > 1:
        assert not any(c.is_symmetric(e) for c, e in zip(g.comms, eod))
    g.sync()
    before = [c.stats() for c in g.comms]
    for r, c in enumerate(g.comms):
        if kind == "segment":
            c.all_to_all_v_combine_quantized(eod[r], outs[r].view(-1), ROW, *plan_or_routes.args(r), idx[r], wd[r], block=block, wire=wire, scale=scale,
                                             stream=g.streams[r])
        else:
            c.expert_combine_quantized(eod[r].view(-1, ROW), idx[r], wd[r], outs[r], block=block, wire=wire, scale=scale, stream=g.streams[r])
    g.sync()
    g.check_async()
    return [o.cpu() for o in outs], before, [c.stats() for c in g.comms]


# block -> (experts per rank, top_k)
CONFIGS = {16: (4, 2), 128: (8, 8), 512: (1, 1)}


@pytest.mark.parametrize("kind", ["segment", "route"])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_combine_bit_exact(torch_cuda, coll_mod, n, kind):
    """Both maps x both wire types x blocks 16, 128, 512 x uniform, Zipf, one-expert and mixed routings (invalid ids, a token naming one
    expert twice, an empty rank) x ample and tight capacity, weights given and None, scale != 1, the 9 (in, out) pairs in turn; inputs
    with specials; rows no slot reads hold NaN and inf; two launches, the algorithm and the bytes of the wide combine."""
    torch, coll = torch_cuda, coll_mod
    with Group(torch, coll, n) as g:
        case = 0
        for block, (epr, k) in CONFIGS.items():
            E = epr * n
            for rkind in ("uniform", "zipf", "one", "mixed"):
                topk = routing(rkind, n, E, k, seed=E + k + n + block)
                tokens = [t.shape[0] for t in topk]
                for cap in ("ample", "tight"):
                    if kind == "segment":
                        plan = segment_plan(topk, E, cap == "tight", seed=case)
                        used = [int(plan.rows[:, d].sum()) for d in range(n)]
                        recv_rows = max(used) + (3 if cap == "ample" else 0)
                        recv_rows = max(recv_rows, 1)
                        maps, wts = plan, plan.weights
                    else:
                        load = max(int(c.sum()) for c in rr.layout(topk, E, 1 << 20).counts)
                        recv_rows = load + 3 if cap == "ample" else max(1, load * 3 // 5)
                        lay = rr.layout(topk, E, recv_rows)
                        used = [int(c.sum()) for c in lay.counts]
                        rng = np.random.default_rng(case)
                        maps, wts = lay.route, [rng.uniform(-1.5, 1.5, size=t.shape).astype(np.float32) for t in topk]
                    for wire_name in ("e4m3", "e5m2"):
                        in_name, out_name = PAIRS[case % len(PAIRS)]
                        with_w = case % 2 == 0
                        scale = 1.0 if with_w else 0.75
                        case += 1
                        in_dt, out_dt, wire = DTYPES[in_name], DTYPES[out_name], DTYPES[wire_name]
                        eo = expert_outs(torch, n, recv_rows, in_dt, block, seed=case, used=used)
                        deq = dequantised(torch, eo, block, wire)
                        w = wts if with_w else None
                        outs, before, after = run(g, kind, maps, eo, recv_rows, in_dt, out_dt, wire, block, w, scale, tokens)
                        what = f"{kind} n={n} {in_name}->{wire_name}->{out_name} block={block} {rkind} {cap} weights={with_w}"
                        for r in range(n):
                            if kind == "segment":
                                rows_r, so, ro = maps.args(r)
                                look, ix = cr.plan_lookup(deq, rows_r, so, ro), maps.index[r]
                            else:
                                look, ix = route_lookup(deq, recv_rows), maps[r]
                            want = cr.combine(look, ix, w[r] if w is not None else None, scale, out_dt)
                            assert_same(outs[r], want, f"{what}: rank {r}")
                            st, b = after[r], before[r]
                            assert st["kernel_launches"] == b["kernel_launches"] + 2, what
                            algo = "copy" if n == 1 else "oneshot"
                            assert st["algo_calls"][algo] == b["algo_calls"][algo] + 1, what
                            assert st["calls"][coll.OP_ALLTOALL] == b["calls"][coll.OP_ALLTOALL] + 1, what
                            nbytes = (int(maps.rows[r].sum()) if kind == "segment" else ix.size) * ROW * in_dt.itemsize
                            assert st["bytes"][coll.OP_ALLTOALL] == b["bytes"][coll.OP_ALLTOALL] + nbytes, what


def test_rank_count_makes_no_difference(torch_cuda, coll_mod):
    """The same global rows, routes and weights give identical bits on one rank and on four: rank 0's tokens at n = 4 read rows spread
    over all four ranks' expert_out; at n = 1 the same rows sit in one expert_out."""
    torch, coll = torch_cuda, coll_mod
    R, tokens, k, block = 24, 40, 6, 64
    wire = torch.float8_e4m3fn
    rng = np.random.default_rng(11)
    rows_g = qr.gen(4 * R * ROW, torch.bfloat16, block, 77).view(4 * R, ROW)
    gidx = rng.integers(-1, 4 * R, size=(tokens, k)).astype(np.int32)              # global rows, -1 dropped
    w = rng.uniform(-2, 2, size=(tokens, k)).astype(np.float32)
    results = {}
    for n in (1, 4):
        with Group(torch, coll, n) as g:
            recv_rows = 4 * R // n
            eo = [rows_g[r * recv_rows:(r + 1) * recv_rows].cuda() for r in range(n)]
            route = np.where(gidx >= 0, (gidx // recv_rows) * recv_rows + gidx % recv_rows, -1).astype(np.int32)
            routes = [g.dev(c, route) for c in g.comms]
            wd = [g.dev(c, w) for c in g.comms]
            outs = [torch.empty(tokens, ROW, dtype=torch.float32, device="cuda") for _ in g.comms]
            g.sync()
            for r, c in enumerate(g.comms):
                c.expert_combine_quantized(eo[r], routes[r], wd[r], outs[r], block=block, wire=wire, scale=0.5, stream=g.streams[r])
            g.sync()
            g.check_async()
            results[n] = outs[0].cpu()
    assert torch.equal(results[1].view(torch.int32), results[4].view(torch.int32))
    deq = dequantised(torch, [rows_g], block, wire)
    assert_same(results[1], cr.combine(route_lookup(deq, 4 * R), gidx, w, 0.5, torch.float32), "one rank vs the reference")


@pytest.mark.parametrize("n", [2, 3])
def test_cuda_graph_dispatch_expert_combine(torch_cuda, coll_mod, n):
    """Each rank captures the FP8 routed dispatch, an expert stand-in that writes a plain (non-arena) bf16 tensor, and
    expert_combine_quantized over the dispatch's route in one CUDA graph, at a size the scratch already holds; topk_idx is rewritten in
    place between replays and every replay is checked."""
    torch, coll = torch_cuda, coll_mod
    with Group(torch, coll, n) as g:
        rng = np.random.default_rng(60 + n)
        block, wire = 128, torch.float8_e4m3fn
        nb = ROW // block
        E, k, tokens = 4 * n, 2, 24
        recv_rows = tokens * k * 3 // 4
        xs = [qr.gen(tokens * ROW, torch.bfloat16, block, 9 + s, specials=False).view(tokens, ROW) for s in range(n)]
        xd = [x.cuda() for x in xs]
        idx = [torch.zeros(tokens, k, dtype=torch.int32, device="cuda") for _ in range(n)]
        w = [rng.uniform(0.1, 1.0, size=(tokens, k)).astype(np.float32) for _ in range(n)]
        wd = [g.dev(c, w[r]) for r, c in enumerate(g.comms)]
        small = [(torch.empty(E // n, dtype=torch.int32, device="cuda"), torch.empty(tokens, k, dtype=torch.int32, device="cuda"),
                  torch.empty(1, dtype=torch.int32, device="cuda")) for _ in range(n)]
        recv = [c.empty(recv_rows * ROW, wire) for c in g.comms]
        sc = [c.empty(recv_rows * ROW // block, torch.float32) for c in g.comms]
        eo = [torch.empty(recv_rows, ROW, dtype=torch.bfloat16, device="cuda") for _ in range(n)]
        outs = [torch.empty(tokens, ROW, dtype=torch.float32, device="cuda") for _ in range(n)]
        for t in recv + sc:
            t.view(torch.uint8).zero_()
        for r in range(n):
            eo[r].zero_()
            small[r][1].fill_(-1)
        g.sync()
        for r, c in enumerate(g.comms):                                # the scratch grows here, outside the capture
            c.expert_combine_quantized(eo[r], small[r][1], wd[r], outs[r], block=block, stream=g.streams[r])
        g.sync()
        graphs = []
        for r, c in enumerate(g.comms):
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=g.streams[r]):
                c.expert_dispatch_quantized(xd[r], idx[r], E, recv[r], sc[r], block, *small[r])
                eo[r].view(-1, nb, block).copy_((recv[r].view(-1, nb, block).float() * sc[r].view(-1, nb, 1) * 0.5).to(torch.bfloat16))
                c.expert_combine_quantized(eo[r], small[r][1], wd[r], outs[r], block=block)
            graphs.append(gr)
        for rep, rkind in enumerate(("uniform", "one", "mixed", "zipf")):
            topk = routing(rkind, n, E, k, seed=rep, tokens=[tokens] * n)
            topk = [t if t.shape[0] == tokens else np.full((tokens, k), -1, dtype=np.int32) for t in topk]
            for r in range(n):
                idx[r].copy_(torch.from_numpy(topk[r]))
            g.sync()
            for r, gr in enumerate(graphs):
                with torch.cuda.stream(g.streams[r]):
                    gr.replay()
            g.sync()
            g.check_async()
            lay = rr.layout(topk, E, recv_rows)
            for r in range(n):
                assert (small[r][1].cpu().numpy() == lay.route[r]).all(), f"replay {rep} ({rkind}): route rank {r}"
            deq = dequantised(torch, [e.cpu() for e in eo], block, wire)
            for r in range(n):
                want = cr.combine(route_lookup(deq, recv_rows), lay.route[r], w[r], 1.0, torch.float32)
                assert_same(outs[r].cpu(), want, f"replay {rep} ({rkind}): combine rank {r}")
        del graphs


def test_shared_scratch_with_quantised_all_reduce(torch_cuda, coll_mod):
    """On every rank's stream, with no host sync: the quantising combine and all_reduce_quantized in turn, at sizes that make the shared
    scratch grow between calls; every result is exact. A graph of a combine captured before the growth still replays exactly."""
    torch, coll = torch_cuda, coll_mod
    n, block, wire = 2, 32, torch.float8_e5m2
    with Group(torch, coll, n) as g:
        rng = np.random.default_rng(3)
        def combine_case(recv_rows, tokens, k, seed):
            eo = [qr.gen(recv_rows * ROW, torch.float16, block, seed + r).view(recv_rows, ROW) for r in range(n)]
            routes = [rng.integers(-2, n * recv_rows + 2, size=(tokens, k)).astype(np.int32) for _ in range(n)]
            w = [rng.uniform(-1, 1, size=(tokens, k)).astype(np.float32) for _ in range(n)]
            dev = ([e.cuda() for e in eo], [g.dev(c, routes[r]) for r, c in enumerate(g.comms)], [g.dev(c, w[r]) for r, c in enumerate(g.comms)],
                   [torch.empty(tokens, ROW, dtype=torch.bfloat16, device="cuda") for _ in range(n)])
            deq = dequantised(torch, eo, block, wire)
            want = [cr.combine(route_lookup(deq, recv_rows), routes[r], w[r], 1.0, torch.bfloat16) for r in range(n)]
            return dev, want

        def ar_case(count, seed):
            xs = [qr.gen(count, torch.float32, block, seed + r) for r in range(n)]
            return [x.cuda() for x in xs], [torch.empty(count, dtype=torch.float32, device="cuda") for _ in range(n)], qr.all_reduce(xs, block, wire, 1.0, torch.float32)

        def enqueue_combine(dev, r, c):
            eo, rt, w, out = dev
            c.expert_combine_quantized(eo[r], rt[r], w[r], out[r], block=block, wire=wire, stream=g.streams[r])

        small, small_want = combine_case(8, 20, 3, 1)
        warm = ar_case(2 * block, 9)
        g.sync()
        for r, c in enumerate(g.comms):
            enqueue_combine(small, r, c)
        g.sync()
        # the all-reduce's kernel launched once before the interleaving: its first launch under lazy module loading would otherwise wait
        # behind this rank's combine, which waits for the next rank's call
        for r, c in enumerate(g.comms):
            c.all_reduce_quantized(warm[0][r], warm[1][r], block=block, wire=wire, stream=g.streams[r])
        g.sync()
        graphs = []
        for r, c in enumerate(g.comms):
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=g.streams[r]):
                c.expert_combine_quantized(small[0][r], small[1][r], small[2][r], small[3][r], block=block, wire=wire)
            graphs.append(gr)
        mid, mid_want = combine_case(64, 30, 4, 2)
        a1 = ar_case(96 * ROW, 3)                                   # larger than the mid combine's scratch
        big, big_want = combine_case(256, 50, 2, 4)
        a2 = ar_case(16 * ROW, 5)
        g.sync()
        for r, c in enumerate(g.comms):
            enqueue_combine(mid, r, c)
            c.all_reduce_quantized(a1[0][r], a1[1][r], block=block, wire=wire, stream=g.streams[r])
            enqueue_combine(big, r, c)
            c.all_reduce_quantized(a2[0][r], a2[1][r], block=block, wire=wire, stream=g.streams[r])
        g.sync()
        g.check_async()
        for r in range(n):
            assert_same(mid[3][r].cpu(), mid_want[r], f"mid combine rank {r}")
            assert_same(big[3][r].cpu(), big_want[r], f"big combine rank {r}")
            assert_same(a1[1][r].cpu(), a1[2], f"all_reduce 1 rank {r}")
            assert_same(a2[1][r].cpu(), a2[2], f"all_reduce 2 rank {r}")
        for o in small[3]:
            o.fill_(float("nan"))
        g.sync()
        for r, gr in enumerate(graphs):
            with torch.cuda.stream(g.streams[r]):
                gr.replay()
        g.sync()
        g.check_async()
        for r in range(n):
            assert_same(small[3][r].cpu(), small_want[r], f"graph captured before the growth, rank {r}")
        del graphs


def _raw_a2av(coll, comm, a):
    arr = lambda xs: (C.c_int64 * len(xs))(*xs)
    ep = coll.Epilogue(a["in_dt"], a["out_dt"], 1.0)
    return coll.load().b200collAllToAllvCombineQuantized(C.c_void_p(a["eo"]), C.c_void_p(a["out"]), a["row_elems"], a["recv_rows"], arr(a["rows"]),
                                                         arr(a["soff"]), arr(a["roff"]), C.cast(C.c_void_p(a["idx"]), C.POINTER(C.c_int32)),
                                                         C.cast(C.c_void_p(a["w"]), C.POINTER(C.c_float)), a["tokens"], a["top_k"], a["wire"], a["block"],
                                                         C.byref(ep) if a["ep"] else None, comm._h, None)


def _raw_expert(coll, comm, a):
    ep = coll.Epilogue(a["in_dt"], a["out_dt"], 1.0)
    return coll.load().b200collExpertCombineQuantized(C.c_void_p(a["eo"]), C.c_void_p(a["out"]), a["row_elems"], a["recv_rows"],
                                                      C.cast(C.c_void_p(a["idx"]), C.POINTER(C.c_int32)), C.cast(C.c_void_p(a["w"]), C.POINTER(C.c_float)),
                                                      a["tokens"], a["top_k"], a["wire"], a["block"], C.byref(ep) if a["ep"] else None, comm._h, None)


def test_refusals_launch_nothing(torch_cuda, coll_mod):
    """Every refusal of both calls, each breaking one rule, returns its code and message and launches nothing: the stats stay at zero.
    OutOfMemory comes from a scratch the arena cannot hold."""
    torch, coll = torch_cuda, coll_mod
    with Group(torch, coll, 2, arena_mb=8) as g:
        c = g.comms[0]
        row, block, rows_n, tokens, k = 128, 32, 16, 4, 2
        eo = torch.empty(rows_n * row, dtype=torch.bfloat16, device="cuda")
        out = torch.empty(tokens * 512, dtype=torch.float32, device="cuda")            # room for the 512-element rows of the OutOfMemory cases
        small = torch.zeros(64, dtype=torch.int32, device="cuda")
        big = torch.empty(65536 * 512, dtype=torch.bfloat16, device="cuda")          # its 32 MiB FP8 copy does not fit an 8 MiB arena
        EO, OUT, IDX, W = eo.data_ptr(), out.data_ptr(), small.data_ptr(), small.data_ptr() + 64
        BF, F32, E4, E5 = coll.BF16, coll.F32, coll.FP8_E4M3, coll.FP8_E5M2
        base = dict(eo=EO, out=OUT, row_elems=row, recv_rows=rows_n, idx=IDX, w=W, tokens=tokens, top_k=k, wire=E4, block=block, in_dt=BF, out_dt=F32, ep=True)
        a2av = dict(base, rows=[2, 3], soff=[0, 2], roff=[0, 4])
        common = [
            ("null expert_out", dict(eo=0), "null argument"), ("null out", dict(out=0), "null argument"), ("null index", dict(idx=0), "null argument"),
            ("null epilogue", dict(ep=False), "null argument"),
            ("FP8 in", dict(in_dt=E4), "in_dtype and out_dtype"), ("FP8 out", dict(out_dt=E5), "in_dtype and out_dtype"),
            ("int32 in", dict(in_dt=coll.I32), "in_dtype and out_dtype"),
            ("bf16 wire", dict(wire=BF), "wire_dtype must be"), ("block 24", dict(block=24), "block must be"), ("block 1024", dict(block=1024), "block must be"),
            ("row_elems % block", dict(block=256), "row_elems must be a positive multiple of block"), ("row_elems 0", dict(row_elems=0), "row_elems"),
            ("top_k 0", dict(top_k=0), "top_k must be"), ("misaligned expert_out", dict(eo=EO + 8), "16-byte aligned"),
            ("misaligned out", dict(out=OUT + 8), "16-byte aligned"), ("misaligned weights", dict(w=W + 2), "4-byte aligned"),
            ("out overlaps expert_out", dict(out=EO), "must not overlap"), ("out overlaps index", dict(out=IDX), "must not overlap"),
            ("more than 2^31 - 1 vectors of out", dict(tokens=1 << 26, row_elems=512, block=512, recv_rows=2), "vectors of out"),
            ("tokens * top_k > 2^31 - 1", dict(tokens=1 << 30, top_k=4, row_elems=16, block=16), "tokens * top_k"),
            ("more than 2^31 - 1 vectors of expert_out", dict(recv_rows=1 << 26, row_elems=512, block=512, eo=big.data_ptr()), "vectors of expert_out"),
        ]
        cases = [("a2av " + what, _raw_a2av, dict(a2av, **kw), INVALID_ARGUMENT, msg) for what, kw, msg in common] + [
            ("a2av negative send_rows", _raw_a2av, dict(a2av, rows=[-1, 3]), INVALID_ARGUMENT, "negative"),
            ("a2av destination past recv_rows", _raw_a2av, dict(a2av, roff=[0, 14]), INVALID_ARGUMENT, "past recv_rows"),
            ("a2av overlapping send ranges", _raw_a2av, dict(a2av, soff=[0, 1]), INVALID_ARGUMENT, "two send ranges overlap"),
            ("a2av scratch larger than the arena", _raw_a2av, dict(a2av, eo=big.data_ptr(), row_elems=512, recv_rows=65536, rows=[0, 0]), OUT_OF_MEMORY,
             "cannot hold"),
        ] + [("expert " + what, _raw_expert, dict(base, **kw), INVALID_ARGUMENT, msg) for what, kw, msg in common] + [
            ("expert nranks * recv_rows > 2^31 - 1", _raw_expert, dict(base, recv_rows=1 << 30, row_elems=16, block=16), INVALID_ARGUMENT,
             "nranks * recv_rows"),
            ("expert scratch larger than the arena", _raw_expert, dict(base, eo=big.data_ptr(), row_elems=512, recv_rows=65536), OUT_OF_MEMORY, "cannot hold"),
        ]
        for what, fn, args, want, msg in cases:
            expect_refused(fn(coll, c, args), want, msg, "quantised expert combine: " if fn is _raw_expert else "quantised all-to-all-v combine: ", what)
        with pytest.raises(ValueError):
            c.expert_combine_quantized(eo.view(-1, row), torch.zeros(tokens, k, dtype=torch.int32, device="cuda"), None,
                                       out[:tokens * row].view(tokens, row), block=256)
        assert_nothing_launched(c)
        g.check_async()


_LAZY = r'''
import numpy as np
import torch
from container_engine_accelerators_b200.ops import coll
from tests import coll_combine_reference as cr
from tests import coll_quant_reference as qr
from tests import coll_routed_reference as rr
from tests.coll_fp_reference import assert_same
n, E, k, tokens, row, block = 2, 8, 2, 32, 256, 64
comms = coll.Comm.init_all([0, 0], arena_mb=32)
streams = [torch.cuda.Stream() for _ in comms]
rng = np.random.default_rng(5)
topk = [rng.integers(0, E, size=(tokens, k)).astype(np.int32) for _ in range(n)]
recv_rows = tokens * k * 3 // 4
lay = rr.layout(topk, E, recv_rows)
xs = [qr.gen(tokens * row, torch.bfloat16, block, 11 + s).view(tokens, row) for s in range(n)]
eo = [qr.gen(recv_rows * row, torch.bfloat16, block, 21 + s).view(recv_rows, row) for s in range(n)]
xd, eod = [x.cuda() for x in xs], [e.cuda() for e in eo]
idx = [torch.from_numpy(t).cuda() for t in topk]
w = [rng.uniform(-1, 1, size=(tokens, k)).astype(np.float32) for _ in range(n)]
wd = [torch.from_numpy(v).cuda() for v in w]
small = [(torch.empty(E // n, dtype=torch.int32, device="cuda"), torch.empty(tokens, k, dtype=torch.int32, device="cuda"),
          torch.empty(1, dtype=torch.int32, device="cuda")) for _ in range(n)]
q = [c.empty(recv_rows * row, torch.float8_e4m3fn) for c in comms]
sc = [c.empty(recv_rows * row // block, torch.float32) for c in comms]
outs = [torch.empty(tokens, row, dtype=torch.float32, device="cuda") for _ in comms]
torch.cuda.synchronize()
for r, c in enumerate(comms):                 # per rank, back to back: the FP8 dispatch, then the quantising combine over its route
    c.expert_dispatch_quantized(xd[r], idx[r], E, q[r], sc[r], block, *small[r], stream=streams[r])
    c.expert_combine_quantized(eod[r], small[r][1], wd[r], outs[r], block=block, stream=streams[r])
torch.cuda.synchronize()
for c in comms:
    c.check_async_error()
ref_x = [qr.quantize(x.reshape(-1), block, torch.float8_e4m3fn) for x in xs]
deq = [qr.quantize(e.reshape(-1), block, torch.float8_e4m3fn)[2].numpy().reshape(-1, row) for e in eo]
for d in range(n):
    gq = q[d].cpu().view(-1, row)
    for r, (s, t) in enumerate(lay.source[d]):
        if s >= 0:
            assert_same(gq[r], ref_x[s][0].view(-1, row)[t], f"fp8 rank {d} row {r}")
    assert (small[d][1].cpu().numpy() == lay.route[d]).all()
    def look(col):
        col = np.asarray(col, dtype=np.int64)
        valid = (col >= 0) & (col < n * recv_rows)
        y = np.zeros((col.size, row), dtype=np.float32)
        for i in np.nonzero(valid)[0]:
            y[i] = deq[col[i] // recv_rows][col[i] % recv_rows]
        return valid, y
    assert_same(outs[d].cpu(), cr.combine(look, lay.route[d], w[d], 1.0, torch.float32), f"combine rank {d}")
for c in comms:
    c.destroy()
print("lazy ok")
'''


def test_lazy_module_loading_dispatch_then_combine(torch_cuda, coll_lib):
    """A fresh process with lazy module loading and a short watchdog drives two virtual ranks from one thread, enqueueing per rank the
    FP8 routed dispatch and the quantising combine back to back: the first launch of the combine's kernels must not wait behind the
    rank's own layout kernel, which waits for the other rank's call. Both results must be exact."""
    run_python(_LAZY, {"CUDA_MODULE_LOADING": "LAZY", "B200COLL_TIMEOUT_MS": "10000"}, "lazy ok")


def _perf(devs, procs, extra, header):
    out = run_perf(["--op", "alltoall", *extra, "-w", "1", "-n", "2", "-c", "1"], devs, procs, env={"B200COLL_TIMEOUT_MS": "20000"})
    assert header in out, out
    assert [l for l in out.splitlines() if l.strip() and not l.startswith("#")], out


def test_perf_tool_quantising_combine_modes(torch_cuda, coll_lib):
    _perf("0", False, ["-d", "bfloat16", "--combine", "4", "--combine-quantize", "e4m3:128", "--row-len", "256", "-b", "64K", "-e", "1M", "-f", "4"],
          "quantising combine")
    _perf("0,0", False, ["-d", "half", "--out-dtype", "float", "--combine", "3", "--combine-quantize", "e5m2:16", "--row-len", "96", "-b", "256K",
                         "-e", "256K"], "quantising combine")
    _perf("0,0", False, ["-d", "float", "--out-dtype", "bfloat16", "--route", "8:2", "--combine-quantize", "e4m3:32", "--row-len", "96", "-b", "256K",
                         "-e", "256K"], "routed dispatch + quantising combine")
    _perf("0,0", True, ["-d", "bfloat16", "--route", "64:8", "--combine-quantize", "e4m3:512", "--row-len", "1024", "-b", "1M", "-e", "1M"],
          "routed dispatch + quantising combine")


def test_two_processes_on_two_gpus(torch_cuda, coll_lib):
    if torch_cuda.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    _perf("0,1", True, ["-d", "bfloat16", "--route", "16:4", "--combine-quantize", "e4m3:128", "--row-len", "7168", "-b", "1M", "-e", "16M", "-f", "4"],
          "routed dispatch + quantising combine")
    _perf("0,1", True, ["-d", "bfloat16", "--combine", "8", "--combine-quantize", "e4m3:128", "--row-len", "7168", "-b", "4M", "-e", "16M", "-f", "4"],
          "quantising combine")


def test_one_process_on_two_gpus(torch_cuda, coll_mod):
    """One process driving two GPUs: the library makes each communicator's device current for its calls."""
    torch, coll = torch_cuda, coll_mod
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    n, E, k, block = 2, 8, 4, 128
    with Group(torch, coll, n, devices=[0, 1]) as g:
        topk = routing("zipf", n, E, k, seed=3, tokens=[300, 200])
        recv_rows = max(int(c.sum()) for c in rr.layout(topk, E, 1 << 20).counts) * 4 // 5
        lay = rr.layout(topk, E, recv_rows)
        eo = expert_outs(torch, n, recv_rows, torch.bfloat16, block, seed=5)
        rng = np.random.default_rng(2)
        w = [rng.uniform(-1, 1, size=t.shape).astype(np.float32) for t in topk]
        outs, _, _ = run(g, "route", lay.route, eo, recv_rows, torch.bfloat16, torch.bfloat16, torch.float8_e4m3fn, block, w, 1.0, [t.shape[0] for t in topk])
        deq = dequantised(torch, eo, block, torch.float8_e4m3fn)
        for r in range(n):
            assert_same(outs[r], cr.combine(route_lookup(deq, recv_rows), lay.route[r], w[r], 1.0, torch.bfloat16), f"two GPUs rank {r}")
