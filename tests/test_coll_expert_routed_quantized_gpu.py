"""Device-routed FP8 expert dispatch on an H100 (`pytest -m gpu`), virtual ranks sharing cuda:0 unless said otherwise.

Every recv and recv_scales starts poisoned with 0x5A bytes. Every stored row must hold, bit for bit (NaN matches NaN at the same position,
as in the other quantised tests), tests/coll_quant_reference.quantize of its source token's row (the source from
tests/coll_routed_reference.layout), and its scales that block's scales; every other row must keep the poison in both buffers.
expert_counts, route and dropped must equal the layout reference and the bf16 routed dispatch's."""
import ctypes as C
import numpy as np
import pytest

from container_engine_accelerators_b200.ops.coll import INVALID_ARGUMENT, INVALID_USAGE
from tests import coll_combine_reference as cr
from tests import coll_quant_reference as qr
from tests import coll_routed_reference as rr
from tests.coll_fp_reference import assert_same
from tests.coll_gpu_harness import (DTYPES, Group, assert_nothing_launched, coll_mod, expect_refused, release, run_perf, run_python,  # noqa: F401
                                    torch_cuda)
from tests.coll_routed_reference import route_lookup, routing

pytestmark = pytest.mark.gpu

ROW = 512                                                               # whole blocks of every size tested, 32 vectors per row
POISON = 0x5A


def small_outputs(g, topk, E):
    """Every rank's (expert_counts, route, dropped), allocated before any rank enqueues."""
    torch = g.torch
    return [(torch.empty(E // g.n, dtype=torch.int32, device=f"cuda:{c.device}"), torch.empty(topk[r].shape, dtype=torch.int32, device=f"cuda:{c.device}"),
             torch.empty(1, dtype=torch.int32, device=f"cuda:{c.device}")) for r, c in enumerate(g.comms)]


def q_bufs(g, recv_rows, wire, block):
    """Poisoned arena recv ([recv_rows * ROW] of wire) and recv_scales ([recv_rows * ROW / block] float32) on every rank."""
    torch = g.torch
    recv = [c.empty(recv_rows * ROW, wire) for c in g.comms]
    sc = [c.empty(recv_rows * ROW // block, torch.float32) for c in g.comms]
    for t in recv + sc:
        t.view(torch.uint8).fill_(POISON)
    return recv, sc


def inputs(torch, topk, in_dt, block, seed, specials=True):
    """One [tokens, ROW] CPU tensor of in_dt per rank, from qr.gen: blocks in their own binades, with zeros, +-0, +-inf, NaN and a tiny
    amax in the first blocks."""
    return [qr.gen(t.shape[0] * ROW, in_dt, block, seed + 17 * s, specials=specials).view(t.shape[0], ROW) for s, t in enumerate(topk)]


def quant_ref(torch, xs, block, wire):
    """Per rank: (FP8 bytes [tokens, ROW] uint8, scale bits [tokens, ROW / block] int32, dequantised values [tokens, ROW] float32)."""
    out = []
    for x in xs:
        q, s, v = qr.quantize(x.reshape(-1), block, wire)
        out.append((q.view(torch.uint8).numpy().reshape(-1, ROW), s.view(torch.int32).numpy().reshape(-1, ROW // block), v.numpy().reshape(-1, ROW)))
    return out


def read_back(torch, recv, sc, small, block):
    return [(recv[r].view(torch.uint8).cpu().numpy().reshape(-1, ROW), sc[r].view(torch.int32).cpu().numpy().reshape(-1, ROW // block),
             small[r][0].cpu().numpy(), small[r][1].cpu().numpy(), int(small[r][2].item())) for r in range(len(recv))]


def check_q(torch, lay, ref, got, wire, what):
    for d, (qb, sb, counts, route, dropped) in enumerate(got):
        want_q = np.full(qb.shape, POISON, dtype=np.uint8)
        want_s = np.full(sb.shape, int.from_bytes(bytes([POISON] * 4), "little"), dtype=np.int32)
        for r, (s, t) in enumerate(lay.source[d]):
            if s >= 0:
                want_q[r], want_s[r] = ref[s][0][t], ref[s][1][t]
        assert_same(torch.from_numpy(qb).view(wire), torch.from_numpy(want_q).view(wire), f"{what}: rank {d} FP8 rows")
        assert_same(torch.from_numpy(sb).view(torch.float32), torch.from_numpy(want_s).view(torch.float32), f"{what}: rank {d} scales")
        assert (counts == lay.counts[d]).all(), f"{what}: rank {d} counts {counts.tolist()} want {lay.counts[d].tolist()}"
        assert (route == lay.route[d]).all(), f"{what}: rank {d} route differs"
        assert dropped == lay.dropped[d], f"{what}: rank {d} dropped {dropped} want {lay.dropped[d]}"


def run_q(g, xd, idx, E, recv_rows, wire, block):
    """The FP8 dispatch on every rank's stream into fresh poisoned buffers; returns (CPU results, buffers)."""
    torch = g.torch
    topk_shapes = [i.shape for i in idx]
    small = small_outputs(g, [np.empty(s) for s in topk_shapes], E)
    recv, sc = q_bufs(g, recv_rows, wire, block)
    g.sync()
    for r, c in enumerate(g.comms):
        c.expert_dispatch_quantized(xd[r], idx[r], E, recv[r], sc[r], block, *small[r], stream=g.streams[r])
    g.sync()
    g.check_async()
    return read_back(torch, recv, sc, small, block), (recv, sc)


def run_bf16_small(g, xd, idx, E, recv_rows):
    """The bf16 (raw rows) routed dispatch of the same ids: its (counts, route, dropped) per rank."""
    torch = g.torch
    small = small_outputs(g, [np.empty(i.shape) for i in idx], E)
    recv = [c.empty(max(1, recv_rows) * ROW, xd[0].dtype) for c in g.comms]
    g.sync()
    for r, c in enumerate(g.comms):
        c.expert_dispatch(xd[r], idx[r], E, recv[r][:recv_rows * ROW], *small[r], stream=g.streams[r])
    g.sync()
    g.check_async()
    release(g.comms, recv)
    return [(s[0].cpu().numpy(), s[1].cpu().numpy(), int(s[2].item())) for s in small]


# block -> (experts per rank, top_k): the three routing shapes of the bf16 test, one per block size
CONFIGS = {16: (4, 2), 128: (8, 8), 512: (1, 1)}


@pytest.mark.parametrize("in_name", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_dispatch_bit_exact(torch_cuda, coll_mod, n, in_name):
    """Both wire types x blocks 16, 128, 512 x uniform, Zipf, one-expert and mixed routings (invalid ids, a token naming one expert twice,
    an empty rank) x ample and tight capacity; small outputs equal to the layout and to the bf16 dispatch's; two launches and the stats."""
    torch, coll = torch_cuda, coll_mod
    in_dt = DTYPES[in_name]
    with Group(torch, coll, n) as g:
        clipped_inside = twice = 0
        for block, (epr, k) in CONFIGS.items():
            E = epr * n
            for kind in ("uniform", "zipf", "one", "mixed"):
                topk = routing(kind, n, E, k, seed=E + k + n + block)
                load = max(int(c.sum()) for c in rr.layout(topk, E, 1 << 20).counts)
                xs = inputs(torch, topk, in_dt, block, seed=block + n)
                xd = [xs[r].to(f"cuda:{c.device}") for r, c in enumerate(g.comms)]
                idx = [g.dev(c, topk[r]) for r, c in enumerate(g.comms)]
                for cap_name, recv_rows in (("ample", load + 3), ("tight", max(1, load * 3 // 5))):
                    lay = rr.layout(topk, E, recv_rows)
                    totals = rr.layout(topk, E, 1 << 20).counts
                    clipped_inside += sum(int(((lay.counts[d] > 0) & (lay.counts[d] < totals[d])).sum()) for d in range(n))
                    wide = run_bf16_small(g, xd, idx, E, recv_rows)
                    for wire_name in ("e4m3", "e5m2"):
                        wire = DTYPES[wire_name]
                        ref = quant_ref(torch, xs, block, wire)
                        before = [c.stats() for c in g.comms]
                        got, bufs = run_q(g, xd, idx, E, recv_rows, wire, block)
                        what = f"n={n} {in_name}->{wire_name} block={block} E={E} top_k={k} {kind} {cap_name}"
                        check_q(torch, lay, ref, got, wire, what)
                        for r in range(n):
                            assert (got[r][2] == wide[r][0]).all() and (got[r][3] == wide[r][1]).all() and got[r][4] == wide[r][2], f"{what}: rank {r} vs bf16"
                        if kind == "mixed" and k >= 2 and topk[0].shape[0] > 1:          # token 1 of rank 0 names one expert twice
                            rt = lay.route[0][1]
                            if rt[0] >= 0 and rt[1] >= 0:
                                d, r0, r1 = rt[0] // recv_rows, rt[0] % recv_rows, rt[1] % recv_rows
                                assert (got[d][0][r0] == got[d][0][r1]).all() and (got[d][1][r0] == got[d][1][r1]).all(), what
                                twice += 1
                        for r, c in enumerate(g.comms):
                            st, b = c.stats(), before[r]
                            assert st["kernel_launches"] == b["kernel_launches"] + 2, what
                            algo = "copy" if n == 1 else "twoshot"
                            assert st["algo_calls"][algo] == b["algo_calls"][algo] + 1, what
                            assert st["calls"][coll.OP_ALLTOALL] == b["calls"][coll.OP_ALLTOALL] + 1, what
                            assert st["bytes"][coll.OP_ALLTOALL] == b["bytes"][coll.OP_ALLTOALL] + topk[r].size * ROW * in_dt.itemsize, what
                        release(g.comms, *bufs)
        assert clipped_inside > 0                                      # some receiver stored part of an expert
        assert twice > 0


@pytest.mark.parametrize("n", [2, 3])
def test_cuda_graph_dispatch_dequantise_combine(torch_cuda, coll_mod, n):
    """Each rank captures the FP8 dispatch, a PyTorch dequantise standing in for the expert (float(q) * s into an fp32 arena buffer), and
    expert_combine over the dispatch's route in one CUDA graph; topk_idx is rewritten in place between replays, and every replay's
    dispatch and combine are checked."""
    torch, coll = torch_cuda, coll_mod
    with Group(torch, coll, n) as g:
        rng = np.random.default_rng(40 + n)
        block, wire = 128, torch.float8_e4m3fn
        nb = ROW // block
        E, k, tokens = 4 * n, 2, 24
        recv_rows = tokens * k * 3 // 4
        xs = [qr.gen(tokens * ROW, torch.bfloat16, block, 7 + s, specials=False).view(tokens, ROW) for s in range(n)]
        ref = quant_ref(torch, xs, block, wire)
        xd = [x.cuda() for x in xs]
        idx = [torch.zeros(tokens, k, dtype=torch.int32, device="cuda") for _ in range(n)]
        w = [rng.uniform(0.1, 1.0, size=(tokens, k)).astype(np.float32) for _ in range(n)]
        wd = [g.dev(c, w[r]) for r, c in enumerate(g.comms)]
        small = small_outputs(g, [np.empty((tokens, k))] * n, E)
        recv, sc = q_bufs(g, recv_rows, wire, block)
        eo = [c.empty(recv_rows * ROW, torch.float32) for c in g.comms]
        outs = [torch.empty(tokens, ROW, dtype=torch.float32, device="cuda") for _ in range(n)]
        g.sync()
        graphs = []
        for r, c in enumerate(g.comms):
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=g.streams[r]):
                c.expert_dispatch_quantized(xd[r], idx[r], E, recv[r], sc[r], block, *small[r])
                eo[r].view(-1, nb, block).copy_(recv[r].view(-1, nb, block).float() * sc[r].view(-1, nb, 1))
                c.expert_combine(eo[r].view(-1, ROW), small[r][1], wd[r], outs[r])
            graphs.append(gr)
        for rep, kind in enumerate(("uniform", "one", "mixed", "zipf")):
            topk = routing(kind, n, E, k, seed=rep, tokens=[tokens] * n)
            topk = [t if t.shape[0] == tokens else np.full((tokens, k), -1, dtype=np.int32) for t in topk]
            for r in range(n):
                idx[r].copy_(torch.from_numpy(topk[r]))
            for t in recv + sc:
                t.view(torch.uint8).fill_(POISON)
            g.sync()
            for r, gr in enumerate(graphs):
                with torch.cuda.stream(g.streams[r]):
                    gr.replay()
            g.sync()
            g.check_async()
            lay = rr.layout(topk, E, recv_rows)
            check_q(torch, lay, ref, read_back(torch, recv, sc, small, block), wire, f"replay {rep} ({kind})")
            # every stored row dequantised is its source token's dequantised row; the combine sums those in slot order
            deq = [np.zeros((recv_rows, ROW), dtype=np.float32) for _ in range(n)]
            for d in range(n):
                for r, (s, t) in enumerate(lay.source[d]):
                    if s >= 0:
                        deq[d][r] = ref[s][2][t]
            for r in range(n):
                want = cr.combine(route_lookup(deq, recv_rows), lay.route[r], w[r], 1.0, torch.float32)
                assert_same(outs[r].cpu(), want, f"replay {rep} ({kind}): combine rank {r}")
        del graphs


def test_interleaved_with_other_collectives(torch_cuda, coll_mod):
    """FP8 dispatch, bf16 routed dispatch, all_reduce, all_to_all_v and FP8 dispatch again (other wire and block) on every rank's stream
    with no host sync in between, then every result checked: the epochs and the count mailbox stay in step."""
    torch, coll = torch_cuda, coll_mod
    n, E, k, tokens = 4, 16, 2, 40
    with Group(torch, coll, n) as g:
        t1, t2 = routing("zipf", n, E, k, seed=1, tokens=[tokens] * n), routing("uniform", n, E, k, seed=2, tokens=[tokens] * n)
        recv_rows = tokens * k * 3 // 4
        xs = [qr.gen(tokens * ROW, torch.float32, 16, 3 + s).view(tokens, ROW) for s in range(n)]
        xd = [x.cuda() for x in xs]
        i1 = [g.dev(c, t1[r]) for r, c in enumerate(g.comms)]
        i2 = [g.dev(c, t2[r]) for r, c in enumerate(g.comms)]
        q1, s1 = q_bufs(g, recv_rows, torch.float8_e4m3fn, 128)
        q2, s2 = q_bufs(g, recv_rows, torch.float8_e5m2, 16)
        wide = [c.empty(recv_rows * ROW, torch.float32) for c in g.comms]
        ar = [c.empty(4096, torch.float32) for c in g.comms]
        for r, a in enumerate(ar):
            a.fill_(float(r + 1))
        from container_engine_accelerators_b200.models.workloads import expert_dispatch_plan
        p = expert_dispatch_plan(n, 20, 64, top_k=1, seed=9)
        sends = [torch.randn(20 * 64, device="cuda").to(torch.bfloat16) for _ in range(n)]
        a2a = [c.empty(p.max_rows * 64, torch.bfloat16) for c in g.comms]
        sm1, smw, sm2 = small_outputs(g, t1, E), small_outputs(g, t2, E), small_outputs(g, t2, E)
        g.sync()
        for r, c in enumerate(g.comms):
            c.expert_dispatch_quantized(xd[r], i1[r], E, q1[r], s1[r], 128, *sm1[r], stream=g.streams[r])
        for r, c in enumerate(g.comms):
            c.expert_dispatch(xd[r], i2[r], E, wide[r], *smw[r], stream=g.streams[r])
        for r, c in enumerate(g.comms):
            c.all_reduce(ar[r], stream=g.streams[r])
        for r, c in enumerate(g.comms):
            c.all_to_all_v(sends[r], a2a[r], 64, p.rows[r].tolist(), p.send_off[r].tolist(), [int(p.recv_off[d, r]) for d in range(n)], stream=g.streams[r])
        for r, c in enumerate(g.comms):
            c.expert_dispatch_quantized(xd[r], i2[r], E, q2[r], s2[r], 16, *sm2[r], stream=g.streams[r])
        g.sync()
        g.check_async()
        check_q(torch, rr.layout(t1, E, recv_rows), quant_ref(torch, xs, 128, torch.float8_e4m3fn), read_back(torch, q1, s1, sm1, 128),
                torch.float8_e4m3fn, "interleaved FP8 dispatch 1")
        lay2 = rr.layout(t2, E, recv_rows)
        check_q(torch, lay2, quant_ref(torch, xs, 16, torch.float8_e5m2), read_back(torch, q2, s2, sm2, 16), torch.float8_e5m2, "interleaved FP8 dispatch 2")
        for r in range(n):
            got = wide[r].cpu().view(-1, ROW)
            for row, (s, t) in enumerate(lay2.source[r]):
                if s >= 0:
                    assert torch.equal(got[row].view(torch.int32), xs[s][t].view(torch.int32)), f"interleaved bf16 dispatch rank {r} row {row}"
            assert (smw[r][1].cpu().numpy() == lay2.route[r]).all()
            assert bool((ar[r] == float(n * (n + 1) // 2)).all())
            for s in range(n):
                lo, cnt = int(p.recv_off[r, s]), int(p.rows[s, r])
                want = sends[s][int(p.send_off[s, r]) * 64:(int(p.send_off[s, r]) + cnt) * 64]
                assert torch.equal(a2a[r][lo * 64:(lo + cnt) * 64], want)


def _raw(coll, comm, **a):
    i32 = lambda p: C.cast(C.c_void_p(p), C.POINTER(C.c_int32))
    return coll.load().b200collExpertDispatchQuantized(C.c_void_p(a["x"]), C.c_void_p(a["recv"]), C.cast(C.c_void_p(a["scales"]), C.POINTER(C.c_float)),
                                                       a["row_elems"], a["recv_rows"], i32(a["topk"]), a["tokens"], a["top_k"], a["E"], i32(a["counts"]),
                                                       i32(a["route"]), i32(a["dropped"]), a["in_dt"], a["wire"], a["block"], comm._h, None)


def test_refusals_launch_nothing(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    with Group(torch, coll, 2) as g:
        c = g.comms[0]
        row, block, rows_n, tokens, k = 128, 32, 16, 4, 2
        recv = c.empty(rows_n * row, torch.float8_e4m3fn)
        scales = c.empty(rows_n * row // block, torch.float32)
        plain = torch.empty(rows_n * row * 4, dtype=torch.uint8, device="cuda")
        x = torch.empty(tokens, row, dtype=torch.bfloat16, device="cuda")
        small = torch.zeros(256, dtype=torch.int32, device="cuda")
        TK, CN, RT, DR = small.data_ptr(), small.data_ptr() + 64, small.data_ptr() + 128, small.data_ptr() + 192
        R, S, X = recv.data_ptr(), scales.data_ptr(), x.data_ptr()
        BF, E4, E5 = coll.BF16, coll.FP8_E4M3, coll.FP8_E5M2
        ok = dict(x=X, recv=R, scales=S, row_elems=row, recv_rows=rows_n, topk=TK, tokens=tokens, top_k=k, E=4, counts=CN, route=RT, dropped=DR,
                  in_dt=BF, wire=E4, block=block)
        # (what, code, arguments that break only that rule, the words of the rule in the error text)
        cases = [("recv outside the arena", INVALID_USAGE, dict(recv=plain.data_ptr()), "symmetric arena"),
                 ("recv_scales outside the arena", INVALID_USAGE, dict(scales=plain.data_ptr()), "symmetric arena")] + [
            (what, INVALID_ARGUMENT, kw, msg) for what, kw, msg in [
                ("null x", dict(x=0), "null argument"), ("null recv", dict(recv=0), "null argument"), ("null recv_scales", dict(scales=0), "null argument"),
                ("null topk_idx", dict(topk=0), "null argument"), ("null route", dict(route=0), "null argument"),
                ("null expert_counts", dict(counts=0), "null argument"), ("null dropped", dict(dropped=0), "null argument"),
                ("FP8 in", dict(in_dt=E4), "in_dtype must be"), ("int32 in", dict(in_dt=coll.I32), "in_dtype must be"),
                ("bf16 wire", dict(wire=BF), "wire_dtype must be"), ("block 24", dict(block=24), "block must be"), ("block 1024", dict(block=1024), "block must be"),
                ("block 8", dict(block=8), "block must be"), ("row_elems % block", dict(block=256), "row_elems must be a positive multiple of block"),
                ("row_elems 0", dict(row_elems=0), "row_elems"), ("top_k 0", dict(top_k=0), "top_k must be"), ("3 experts for 2 ranks", dict(E=3), "num_experts"),
                ("misaligned x", dict(x=X + 8), "16-byte aligned"), ("misaligned recv", dict(recv=R + 8), "16-byte aligned"),
                ("misaligned recv_scales", dict(scales=S + 2), "recv_scales must be 4-byte aligned"),
                ("misaligned route", dict(route=RT + 2), "4-byte aligned"),
                ("recv overlaps x", dict(x=R), "recv must not overlap x"), ("recv_scales overlaps x", dict(scales=X + 64), "recv_scales must not overlap x"),
                ("recv overlaps recv_scales", dict(scales=R + 64), "recv and recv_scales must not overlap"),
                ("route overlaps expert_counts", dict(route=CN), "each other"),
                ("dropped in recv_scales", dict(dropped=S + 8), "topk_idx, x, recv or recv_scales"),
                ("expert_counts in recv", dict(counts=R + 64), "topk_idx, x, recv or recv_scales"),
                ("tokens * top_k > 2^31 - 1", dict(tokens=1 << 30, top_k=2), "tokens * top_k"),
                ("nranks * recv_rows > 2^31 - 1", dict(recv_rows=1 << 30), "nranks * recv_rows"),
                ("more than 2^31 - 1 vectors of x", dict(tokens=1 << 24, top_k=1, row_elems=2048), "vectors of x"),
                ("more than 2^31 - 1 vectors offered", dict(tokens=1 << 22, top_k=32, row_elems=512), "16-byte vectors offered"),
            ]]
        for what, want, kw, msg in cases:
            expect_refused(_raw(coll, c, **dict(ok, **kw)), want, msg, what=what)
        with pytest.raises(ValueError):
            c.expert_dispatch_quantized(x, torch.zeros(tokens, k, dtype=torch.int32, device="cuda"), 3, recv, scales, block)    # 3 experts, 2 ranks
        with pytest.raises(ValueError):
            c.expert_dispatch_quantized(x, torch.zeros(tokens, k, dtype=torch.int32, device="cuda"), 4, recv, scales, 64)       # scales hold block 32
        assert_nothing_launched(c)
        g.check_async()


_LAZY = r'''
import numpy as np
import torch
from container_engine_accelerators_b200.ops import coll
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
xd = [x.cuda() for x in xs]
idx = [torch.from_numpy(t).cuda() for t in topk]
small = [(torch.empty(E // n, dtype=torch.int32, device="cuda"), torch.empty(tokens, k, dtype=torch.int32, device="cuda"),
          torch.empty(1, dtype=torch.int32, device="cuda")) for _ in range(2 * n)]
wide = [c.empty(recv_rows * row, torch.bfloat16) for c in comms]
q = [c.empty(recv_rows * row, torch.float8_e4m3fn) for c in comms]
sc = [c.empty(recv_rows * row // block, torch.float32) for c in comms]
torch.cuda.synchronize()
for r, c in enumerate(comms):                 # the bf16 dispatch first: it loads the push kernels of both dispatches
    c.expert_dispatch(xd[r], idx[r], E, wide[r], *small[r], stream=streams[r])
torch.cuda.synchronize()
for r, c in enumerate(comms):                 # then the FP8 one, whose push kernel this process has never launched
    c.expert_dispatch_quantized(xd[r], idx[r], E, q[r], sc[r], block, *small[n + r], stream=streams[r])
torch.cuda.synchronize()
for c in comms:
    c.check_async_error()
for d in range(n):
    ref_q = [qr.quantize(x.reshape(-1), block, torch.float8_e4m3fn) for x in xs]
    gw, gq, gs = wide[d].cpu().view(-1, row), q[d].cpu().view(-1, row), sc[d].cpu().view(-1, row // block)
    for r, (s, t) in enumerate(lay.source[d]):
        if s < 0:
            continue
        assert torch.equal(gw[r].view(torch.int16), xs[s][t].view(torch.int16)), ("bf16", d, r)
        assert_same(gq[r], ref_q[s][0].view(-1, row)[t], f"fp8 rank {d} row {r}")          # NaN matches NaN at the same position
        assert_same(gs[r], ref_q[s][1].view(-1, row // block)[t], f"scales rank {d} row {r}")
    for j in range(2):
        assert (small[j * n + d][1].cpu().numpy() == lay.route[d]).all() and (small[j * n + d][0].cpu().numpy() == lay.counts[d]).all()
for c in comms:
    c.destroy()
print("lazy ok")
'''


def test_lazy_module_loading_bf16_dispatch_first(torch_cuda, coll_lib):
    """A fresh process with lazy module loading and a short watchdog runs the bf16 routed dispatch, then the FP8 one, on two virtual ranks
    driven by one thread: the first dispatch on the device loads every push kernel that can follow a layout kernel, so the FP8 push's
    first launch does not wait behind a layout kernel that waits for the next rank's launch. Both results must be exact."""
    run_python(_LAZY, {"CUDA_MODULE_LOADING": "LAZY", "B200COLL_TIMEOUT_MS": "10000"}, "lazy ok")


def _perf(devs, procs, extra):
    out = run_perf(["--op", "alltoall", *extra, "-w", "1", "-n", "2", "-c", "1"], devs, procs, env={"B200COLL_TIMEOUT_MS": "20000"})
    assert "routed FP8 dispatch" in out, out
    assert [l for l in out.splitlines() if l.strip() and not l.startswith("#")], out


def test_perf_tool_routed_fp8_mode(torch_cuda, coll_lib):
    _perf("0", False, ["-d", "bfloat16", "--route", "16:4", "--quantize", "e4m3:128", "-b", "64K", "-e", "1M", "-f", "4"])
    _perf("0,0", False, ["-d", "float", "--route", "8:2", "--quantize", "e5m2:16", "--row-len", "96", "-b", "256K", "-e", "256K"])
    _perf("0,0", True, ["-d", "half", "--route", "256:8", "--quantize", "e4m3:512", "--row-len", "1024", "-b", "1M", "-e", "1M"])


def test_two_processes_on_two_gpus(torch_cuda, coll_lib):
    if torch_cuda.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    _perf("0,1", True, ["-d", "bfloat16", "--route", "16:4", "--quantize", "e4m3:128", "--row-len", "7168", "-b", "1M", "-e", "16M", "-f", "4"])


def test_one_process_on_two_gpus(torch_cuda, coll_mod):
    """One process driving two GPUs: the library makes each communicator's device current for its calls."""
    torch, coll = torch_cuda, coll_mod
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    n, E, k, block = 2, 8, 4, 128
    with Group(torch, coll, n, devices=[0, 1]) as g:
        topk = routing("zipf", n, E, k, seed=3, tokens=[300, 200])
        recv_rows = max(int(c.sum()) for c in rr.layout(topk, E, 1 << 20).counts) * 4 // 5
        xs = inputs(torch, topk, torch.bfloat16, block, seed=21)
        xd = [xs[r].to(f"cuda:{c.device}") for r, c in enumerate(g.comms)]
        idx = [g.dev(c, topk[r]) for r, c in enumerate(g.comms)]
        got, bufs = run_q(g, xd, idx, E, recv_rows, torch.float8_e4m3fn, block)
        check_q(torch, rr.layout(topk, E, recv_rows), quant_ref(torch, xs, block, torch.float8_e4m3fn), got, torch.float8_e4m3fn, "two GPUs")
        release(g.comms, *bufs)
