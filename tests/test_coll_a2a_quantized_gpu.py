"""Quantising all-to-all-v on an H100 (`pytest -m gpu`), virtual ranks sharing cuda:0 unless said otherwise.

Every received FP8 byte and scale is checked bit for bit against tests/coll_quant_reference.quantize applied to the rows that were sent
(NaN matches NaN at the same position); recv and recv_scales start poisoned with 0x5A, and every byte outside the received ranges must
still hold it."""
import ctypes as C

import numpy as np
import pytest

from container_engine_accelerators_b200.ops.coll import INVALID_ARGUMENT, INVALID_USAGE
from tests import coll_quant_reference as qr
from tests.coll_fp_reference import assert_same
from tests.coll_gpu_harness import DTYPES, Group, Plan, assert_nothing_launched, coll_mod, expect_refused, run_perf, torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu
ROW = {16: 80, 128: 384, 512: 1024}                                     # row_elems per block: several blocks per row, or one


def dispatch_plan(n, seed, skew=1.2, tokens=48):
    from container_engine_accelerators_b200.models.workloads import expert_dispatch_plan
    p = expert_dispatch_plan(n, tokens, 1, skew=skew, seed=seed)
    return Plan(p.rows, p.send_off, p.recv_off)


def hand_plan(n):
    """The last rank sends nothing, rank 0 receives nothing (n >= 2), ranks in between send rows to themselves; send ranges are laid out in
    reverse peer order with one-row gaps, destination ranges in rank order with two-row gaps."""
    rows = np.zeros((n, n), dtype=np.int64)
    for s in range(n):
        for d in range(n):
            if n == 1 or (s != n - 1 and d != 0):
                rows[s, d] = (s + 2 * d) % 3 + 1 + (5 if n == 1 else 0)
    send_off, recv_off = np.zeros_like(rows), np.zeros_like(rows)
    for s in range(n):
        at = 1
        for d in reversed(range(n)):
            send_off[s, d] = at
            at += rows[s, d] + 1
    for d in range(n):
        at = 2
        for s in range(n):
            recv_off[d, s] = at
            at += rows[s, d] + 2
    return Plan(rows, send_off, recv_off)


def expected(torch, xs, plan, d, row_elems, block, wire, recv_rows, start=None):
    """(q, s) rank d must hold: `start` (default all 0x5A) with every received range replaced by the quantised rows."""
    spr = row_elems // block
    if start is None:
        q = torch.full((recv_rows * row_elems,), 0x5A, dtype=torch.uint8)
        s = torch.full((recv_rows * spr * 4,), 0x5A, dtype=torch.uint8).view(torch.float32)
    else:
        q, s = start[0].view(torch.uint8).clone(), start[1].clone()
    for src in range(len(xs)):
        r, so, ro = int(plan.rows[src, d]), int(plan.send_off[src, d]), int(plan.recv_off[d, src])
        if r == 0:
            continue
        wq, ws, _ = qr.quantize(xs[src][so * row_elems:(so + r) * row_elems], block, wire)
        q[ro * row_elems:(ro + r) * row_elems] = wq.view(torch.uint8)
        s[ro * spr:(ro + r) * spr] = ws
    return q.view(wire), s


def inputs(g, rows, row_elems, in_dt, block, seed, arena=False):
    torch = g.torch
    xs = [qr.gen(rows * row_elems, in_dt, block, seed + 17 * r) for r in range(g.n)]
    ds = []
    for c, x in zip(g.comms, xs):
        with torch.cuda.device(c.device):
            d = c.empty(x.numel(), in_dt) if arena else torch.empty(x.numel(), dtype=in_dt, device=f"cuda:{c.device}")
            d.copy_(x)
        ds.append(d)
    g.sync()
    return xs, ds


def outputs(g, recv_rows, row_elems, block, wire):
    torch = g.torch
    outs = []
    for c in g.comms:
        with torch.cuda.device(c.device):
            q, s = c.empty(recv_rows * row_elems, wire), c.empty(recv_rows * row_elems // block, torch.float32)
            q.view(torch.uint8).fill_(0x5A)
            s.view(torch.uint8).fill_(0x5A)
        outs.append((q, s))
    g.sync()
    return outs


def call(g, ds, outs, plan, row_elems, block):
    g.run(lambda r, c, st: c.all_to_all_v_quantized(ds[r], outs[r][0], outs[r][1], row_elems, *plan.args(r), block=block, stream=st))


def fetch(outs):
    """CPU copies of every rank's (q, s): the checks take these, so a failing assert never holds device tensors whose arena memory the
    clean-up unmaps before the report is written."""
    return [(q.cpu(), s.cpu()) for q, s in outs]


def check(g, xs, got, plan, row_elems, block, wire, what, starts=None):
    for d in range(g.n):
        q, s = got[d]
        wq, ws = expected(g.torch, xs, plan, d, row_elems, block, wire, q.numel() // row_elems, None if starts is None else starts[d])
        assert_same(q, wq, f"{what}: rank {d} FP8 rows")
        assert_same(s, ws, f"{what}: rank {d} scales")


@pytest.mark.parametrize("in_name", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_grid_bit_exact(torch_cuda, coll_mod, n, in_name):
    """Every wire type and block size, on a skewed expert-dispatch plan and on the hand plan (a rank that sends nothing, one that
    receives nothing, rows to self); one launch per call and rank, stats under alltoall."""
    torch, coll = torch_cuda, coll_mod
    in_dt = DTYPES[in_name]
    with Group(torch, coll, n) as g:
        for wire_name in ("e4m3", "e5m2"):
            wire = DTYPES[wire_name]
            for block in (16, 128, 512):
                row_elems = ROW[block]
                plans = [dispatch_plan(n, seed=n + block), hand_plan(n)]
                src_rows = max(p.src_rows for p in plans)
                recv_rows = max(p.recv_rows for p in plans) + 3
                xs, ds = inputs(g, src_rows, row_elems, in_dt, block, seed=block + n)
                for k, plan in enumerate(plans):
                    outs = outputs(g, recv_rows, row_elems, block, wire)
                    before = [c.stats() for c in g.comms]
                    call(g, ds, outs, plan, row_elems, block)
                    what = f"n={n} {in_name}->{wire_name} block {block} plan {k}"
                    check(g, xs, fetch(outs), plan, row_elems, block, wire, what)
                    for r, c in enumerate(g.comms):
                        st, b = c.stats(), before[r]
                        assert st["kernel_launches"] == b["kernel_launches"] + 1, what
                        algo = "copy" if n == 1 else "twoshot"
                        assert st["algo_calls"][algo] == b["algo_calls"][algo] + 1, (what, st["algo_calls"])
                        assert st["calls"][coll.OP_ALLTOALL] == b["calls"][coll.OP_ALLTOALL] + 1, what
                        sent = int(plan.rows[r].sum()) * row_elems * in_dt.itemsize
                        assert st["bytes"][coll.OP_ALLTOALL] == b["bytes"][coll.OP_ALLTOALL] + sent, what
                    for c, (q, s) in zip(g.comms, outs):
                        c.release(q)
                        c.release(s)


def test_arena_send_repeated_calls_and_few_ctas(torch_cuda, coll_mod):
    """send in the arena; two back-to-back calls with different plans into the same buffers, with few CTAs so each walks many warps."""
    torch, coll = torch_cuda, coll_mod
    n, block, row_elems, wire = 4, 64, 256, torch.float8_e4m3fn
    with Group(torch, coll, n) as g:
        for c in g.comms:
            c.set_max_ctas(3)
        a, b = hand_plan(n), dispatch_plan(n, seed=5, tokens=200)
        xs, ds = inputs(g, max(a.src_rows, b.src_rows), row_elems, torch.bfloat16, block, seed=31, arena=True)
        recv_rows = max(a.recv_rows, b.recv_rows)
        outs = outputs(g, recv_rows, row_elems, block, wire)
        for r, c in enumerate(g.comms):
            for plan in (a, b):
                c.all_to_all_v_quantized(ds[r], outs[r][0], outs[r][1], row_elems, *plan.args(r), block=block, stream=g.streams[r])
        g.sync()
        g.check_async()
        starts = [expected(torch, xs, a, d, row_elems, block, wire, recv_rows) for d in range(n)]
        check(g, xs, fetch(outs), b, row_elems, block, wire, "second of two back-to-back calls", starts=starts)
        for c in g.comms:
            assert c.stats()["kernel_launches"] == 2


def test_cuda_graph_replays_the_same_bits(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    n, block, row_elems, wire = 3, 128, 512, torch.float8_e5m2
    with Group(torch, coll, n) as g:
        plan = dispatch_plan(n, seed=9)
        xs, ds = inputs(g, plan.src_rows, row_elems, torch.float32, block, seed=44)
        outs = outputs(g, plan.recv_rows + 1, row_elems, block, wire)
        graphs = []
        for r, c in enumerate(g.comms):
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=g.streams[r]):
                c.all_to_all_v_quantized(ds[r], outs[r][0], outs[r][1], row_elems, *plan.args(r), block=block)
            graphs.append(gr)
        for rep in range(2):
            for q, s in outs:
                q.view(torch.uint8).fill_(0x5A)
                s.view(torch.uint8).fill_(0x5A)
            g.sync()
            for r, gr in enumerate(graphs):
                with torch.cuda.stream(g.streams[r]):
                    gr.replay()
            g.sync()
            g.check_async()
            check(g, xs, fetch(outs), plan, row_elems, block, wire, f"graph replay {rep}")
        del graphs


def test_received_blocks_feed_the_block_scaled_all_gather(torch_cuda, coll_mod):
    """(q, s) as received is a valid block-scaled input with block (1, block): a one-rank all-gather of it gives round(float(q) * s)."""
    torch, coll = torch_cuda, coll_mod
    n, block, row_elems, wire = 2, 32, 128, torch.float8_e4m3fn
    with Group(torch, coll, n) as g:
        plan = dispatch_plan(n, seed=3)
        xs, ds = inputs(g, plan.src_rows, row_elems, torch.bfloat16, block, seed=8)
        outs = outputs(g, plan.recv_rows, row_elems, block, wire)
        call(g, ds, outs, plan, row_elems, block)
        got = fetch(outs)
    with Group(torch, coll, 1, arena_mb=16) as g1:
        c1 = g1.comms[0]
        for d, (q, s) in enumerate(got):
            rows = q.numel() // row_elems
            bq, bs = c1.empty(q.numel(), wire), c1.empty(s.numel(), torch.float32)        # arena tensors, released below
            aq, as_ = bq.view(rows, row_elems), bs.view(rows, row_elems // block)
            aq.copy_(q.view(rows, row_elems).cuda())
            as_.copy_(s.view(rows, row_elems // block).cuda())
            out = torch.empty(rows, row_elems, dtype=torch.float32, device="cuda")
            c1.all_gather_block_scaled(aq, as_, out, block=(1, block))
            torch.cuda.synchronize()
            with np.errstate(invalid="ignore", over="ignore"):
                v = (q.float().numpy().reshape(rows, -1, block) * s.numpy().reshape(rows, -1, 1)).astype(np.float32)
            want = qr.reduce([torch.from_numpy(v.reshape(-1))], 1.0, torch.float32)
            assert_same(out.cpu().reshape(-1), want, f"rank {d}: block-scaled all-gather of the received blocks")
            del aq, as_
            c1.release(bq)
            c1.release(bs)
        c1.check_async_error()


def _raw(coll, comm, send, recv, scales, row_elems, recv_rows, rows, soff, roff, in_dt, wire, block):
    n = comm.nranks
    arr = lambda xs: (C.c_int64 * n)(*xs)
    return coll.load().b200collAllToAllvQuantized(C.c_void_p(send), C.c_void_p(recv), C.cast(C.c_void_p(scales), C.POINTER(C.c_float)), row_elems, recv_rows,
                                                  arr(rows), arr(soff), arr(roff), in_dt, wire, block, comm._h, None)


def test_placement_and_argument_errors(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    with Group(torch, coll, 2) as g:
        c = g.comms[0]
        row, blk, rows = 256, 128, 8
        send = torch.empty(rows * row, dtype=torch.bfloat16, device="cuda")
        q, s = c.empty(rows * row, torch.float8_e4m3fn), c.empty(rows * row // blk, torch.float32)
        plain_q = torch.empty(rows * row, dtype=torch.uint8, device="cuda")
        plain_s = torch.empty(rows * row // blk, dtype=torch.float32, device="cuda")
        S, Q, SC = send.data_ptr(), q.data_ptr(), s.data_ptr()
        BF, E4 = coll.BF16, coll.FP8_E4M3
        ok = dict(send=S, recv=Q, scales=SC, row_elems=row, recv_rows=rows, rows=[2, 3], soff=[0, 2], roff=[0, 4], in_dt=BF, wire=E4, block=blk)
        cases = [
            ("recv outside the arena", INVALID_USAGE, dict(recv=plain_q.data_ptr())),
            ("recv_scales outside the arena", INVALID_USAGE, dict(scales=plain_s.data_ptr())),
        ] + [(what, INVALID_ARGUMENT, kw) for what, kw in [
            ("destination past recv_rows", dict(roff=[0, 6])),
            ("destination offset past recv_rows, no rows", dict(rows=[2, 0], roff=[0, 9])),
            ("send overlaps recv", dict(send=Q)),
            ("send overlaps recv_scales", dict(send=SC - 256)),
            ("recv overlaps recv_scales", dict(scales=Q + 64)),
            ("FP8 input", dict(in_dt=E4)),
            ("bf16 wire", dict(wire=BF)),
            ("block 24", dict(block=24, row_elems=240)),
            ("row_elems % block", dict(row_elems=192)),
            ("negative rows", dict(rows=[2, -3])),
            ("negative send offset", dict(soff=[-1, 2])),
            ("negative destination", dict(roff=[0, -4])),
            ("misaligned send", dict(send=S + 8)),
            ("misaligned recv", dict(recv=Q + 4)),
            ("null recv_scales", dict(scales=0)),
            ("more than 2^31 - 1 vectors", dict(row_elems=1 << 30, recv_rows=64, block=512, rows=[17, 16], soff=[0, 17], roff=[0, 17])),
        ]]
        for what, want, kw in cases:
            a = dict(ok, **kw)
            rc = _raw(coll, c, a["send"], a["recv"], a["scales"], a["row_elems"], a["recv_rows"], a["rows"], a["soff"], a["roff"], a["in_dt"], a["wire"], a["block"])
            expect_refused(rc, want, what=what)
        with pytest.raises(ValueError):
            c.all_to_all_v_quantized(send, q, s, row, [2, 3], [0, 2], [0, 6])                   # Python refuses it before the library call
        assert_nothing_launched(c)                                                              # nothing was launched or counted
        g.check_async()
    # one rank: recv and recv_scales may be any device buffers
    with Group(torch, coll, 1) as g:
        block, row_elems, wire = 16, 64, torch.float8_e5m2
        plan = hand_plan(1)
        xs, ds = inputs(g, plan.src_rows, row_elems, torch.float16, block, seed=2)
        q = torch.full((plan.recv_rows * row_elems,), 0x5A, dtype=torch.uint8, device="cuda").view(wire)
        s = torch.full((plan.recv_rows * row_elems // block * 4,), 0x5A, dtype=torch.uint8, device="cuda").view(torch.float32)
        assert not g.comms[0].is_symmetric(q) and not g.comms[0].is_symmetric(s)
        call(g, ds, [(q, s)], plan, row_elems, block)
        check(g, xs, fetch([(q, s)]), plan, row_elems, block, wire, "one rank outside the arena")
        assert g.comms[0].stats()["algo_calls"]["copy"] == 1 and g.comms[0].stats()["kernel_launches"] == 1


def test_multi_gpu(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    n, block, row_elems, wire = torch.cuda.device_count(), 128, 1024, torch.float8_e4m3fn
    with Group(torch, coll, n, arena_mb=256, devices=list(range(n))) as g:
        for plan in (dispatch_plan(n, seed=1, tokens=512), hand_plan(n)):
            xs, ds = inputs(g, plan.src_rows, row_elems, torch.bfloat16, block, seed=90)
            outs = outputs(g, plan.recv_rows, row_elems, block, wire)
            call(g, ds, outs, plan, row_elems, block)
            check(g, xs, fetch(outs), plan, row_elems, block, wire, "multi-GPU")


def test_perf_tool_alltoall_quantize_bit_exact(torch_cuda, coll_lib):
    out = run_perf(["--op", "alltoall", "-d", "bfloat16", "--out-dtype", "e4m3", "--quantize", "e4m3:128", "-b", "64K", "-e", "4M", "-f", "8",
                    "-w", "1", "-n", "2", "-c", "1"], "0,0")
    assert "quantised: wire=e4m3 block=128" in out, out[-2000:]
    rows = [l for l in out.splitlines() if l.strip() and not l.startswith("#")]
    assert len(rows) == 3, out                                           # 64 KiB, 512 KiB and 4 MiB
    for devs, extra in (("0,0,0", ["-d", "half", "--quantize", "e5m2:32", "--row-len", "96"]), ("0", ["-d", "float", "--quantize", "e4m3:512"])):
        run_perf(["--op", "alltoall", *extra, "-b", "1M", "-e", "1M", "-w", "1", "-n", "2", "-c", "1"], devs)
