"""Expert combine on an H100 (`pytest -m gpu`), virtual ranks sharing cuda:0 unless said otherwise.

Every out starts poisoned with 0x5A, and every element is compared bit for bit with tests/coll_combine_reference.combine applied to
the expert_out rows each slot names (NaN matches NaN at the same position)."""
import ctypes as C

import numpy as np
import pytest

from container_engine_accelerators_b200.ops.coll import INVALID_ARGUMENT, INVALID_USAGE
from tests import coll_combine_reference as cr
from tests import coll_quant_reference as qr
from tests.coll_fp_reference import assert_same
from tests.coll_gpu_harness import DTYPES, Group, Plan, assert_nothing_launched, coll_mod, expect_refused, run_perf, torch_cuda  # noqa: F401
from tests.coll_routed_reference import INT32_MAX, INT32_MIN

pytestmark = pytest.mark.gpu
ROW = 48


def _spoil(index, rng):
    """Dropped slots of every kind: -1, INT32_MIN, INT32_MAX, past every range, and a token with every slot dropped."""
    idx = index.astype(np.int64).copy()
    t, k = idx.shape
    if t == 0:
        return idx.astype(np.int32)
    end = int(idx.max()) + 1 if idx.size else 0
    bad = [-1, INT32_MIN, INT32_MAX, end, end + 5]
    pos = rng.choice(t * k, size=min(t * k, 6), replace=False)
    for i, p in enumerate(pos):
        idx.flat[p] = bad[i % len(bad)]
    idx[t // 2, :] = -1
    return idx.astype(np.int32)


def dispatch_plan(n, top_k, seed, tokens=24):
    from container_engine_accelerators_b200.models.workloads import expert_dispatch_plan
    p = expert_dispatch_plan(n, tokens, ROW, top_k=top_k, skew=1.2, seed=seed)
    rng = np.random.default_rng(seed)
    return Plan(p.rows, p.send_off, p.recv_off, [_spoil(i, rng) for i in p.index], p.weights)


def hand_plan(n, top_k, seed):
    """Send ranges in reverse peer order with one-row gaps, destination ranges with two-row gaps; the last rank sends nothing and has no
    tokens, rank 0 receives nothing (n >= 2). Indices are drawn over every row up to past the last range, so gap rows, -1 and the
    rows past the end all occur, plus INT32_MIN and INT32_MAX."""
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
    rng = np.random.default_rng(seed)
    index, weights = [], []
    for s in range(n):
        tokens = 0 if (n > 1 and s == n - 1) else 9
        end = int((send_off[s] + rows[s]).max()) + 2
        idx = rng.integers(-1, end, size=(tokens, top_k)).astype(np.int64)
        if tokens:
            idx.flat[0] = INT32_MIN
            idx.flat[-1] = INT32_MAX
            idx[tokens // 2, :] = -1
        index.append(idx.astype(np.int32))
        weights.append(rng.uniform(-1.5, 1.5, size=(tokens, top_k)).astype(np.float32))
    return Plan(rows, send_off, recv_off, index, weights)


def expert_outs(g, recv_rows, in_dt, seed, specials=True):
    """(CPU copies, arena tensors) of every rank's [recv_rows, ROW] expert_out."""
    torch = g.torch
    xs = [qr.gen(recv_rows * ROW, in_dt, 16, seed + 17 * r, specials=specials) for r in range(g.n)]
    ds = []
    for c, x in zip(g.comms, xs):
        with torch.cuda.device(c.device):
            d = c.empty(x.numel(), in_dt)
            d.copy_(x)
        ds.append(d)
    g.sync()
    return xs, ds


def poisoned_outs(g, plan, out_dt):
    """Every rank's out, all bytes 0x5A."""
    torch = g.torch
    res = []
    for r, c in enumerate(g.comms):
        t = torch.full((plan.index[r].shape[0] * ROW * torch.empty((), dtype=out_dt).element_size(),), 0x5A, dtype=torch.uint8, device=f"cuda:{c.device}")
        res.append(t.view(out_dt))
    return res


def call(g, eo, outs, plan, weights, scale, idx_dev=None, w_dev=None):
    idx_dev = idx_dev or [g.dev(c, plan.index[r]) for r, c in enumerate(g.comms)]
    w_dev = w_dev or [g.dev(c, plan.weights[r]) if weights else None for r, c in enumerate(g.comms)]
    g.sync()                                                         # index and weights were copied on the default stream
    g.run(lambda r, c, st: c.all_to_all_v_combine(eo[r], outs[r], ROW, *plan.args(r), idx_dev[r], w_dev[r], scale=scale, stream=st))


def check(g, xs, outs, plan, weights, scale, what):
    got = [o.cpu() for o in outs]
    eo = [x.float().numpy().reshape(-1, ROW) for x in xs]
    for r in range(g.n):
        rows, so, ro = plan.args(r)
        look = cr.plan_lookup(eo, rows, so, ro)
        want = cr.combine(look, plan.index[r], plan.weights[r] if weights else None, scale, got[r].dtype)
        assert_same(got[r], want.reshape(-1), f"{what}: rank {r}")


@pytest.mark.parametrize("out_name", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("in_name", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_grid_bit_exact(torch_cuda, coll_mod, n, in_name, out_name):
    """top_k 1, 2 and 8, with weights and without, scale 1 and not; a skewed dispatch plan and the hand plan; dropped slots of every
    kind; one launch per call and rank, the stats under alltoall."""
    torch, coll = torch_cuda, coll_mod
    in_dt, out_dt = DTYPES[in_name], DTYPES[out_name]
    with Group(torch, coll, n) as g:
        for top_k in (1, 2, 8):
            plans = [dispatch_plan(n, top_k, seed=n * 10 + top_k), hand_plan(n, top_k, seed=n + top_k)]
            recv_rows = max(p.recv_rows for p in plans) + 3
            xs, eo = expert_outs(g, recv_rows, in_dt, seed=top_k + n)
            for k, plan in enumerate(plans):
                for weights, scale in ((True, 1.0), (True, 0.375), (False, 1.0), (False, -3.0)):
                    outs = poisoned_outs(g, plan, out_dt)
                    before = [c.stats() for c in g.comms]
                    call(g, eo, outs, plan, weights, scale)
                    what = f"n={n} {in_name}->{out_name} top_k {top_k} plan {k} weights {weights} scale {scale}"
                    check(g, xs, outs, plan, weights, scale, what)
                    for r, c in enumerate(g.comms):
                        st, b = c.stats(), before[r]
                        assert st["kernel_launches"] == b["kernel_launches"] + 1, what
                        algo = "copy" if n == 1 else "oneshot"
                        assert st["algo_calls"][algo] == b["algo_calls"][algo] + 1, (what, st["algo_calls"])
                        assert st["calls"][coll.OP_ALLTOALL] == b["calls"][coll.OP_ALLTOALL] + 1, what
                        pulled = int(plan.rows[r].sum()) * ROW * in_dt.itemsize
                        assert st["bytes"][coll.OP_ALLTOALL] == b["bytes"][coll.OP_ALLTOALL] + pulled, what
            for c, d in zip(g.comms, eo):
                c.release(d)


def _dispatch_send(torch, x, index):
    """The dispatch send buffer of one rank: row index[t, j] holds token t's row."""
    send = torch.empty((int(index.max()) + 1 if index.size else 0, x.shape[1]), dtype=x.dtype)
    for j in range(index.shape[1]):
        send[torch.from_numpy(index[:, j].astype(np.int64))] = x
    return send


@pytest.mark.parametrize("n", [2, 3])
def test_inverse_of_all_to_all_v(torch_cuda, coll_mod, n):
    """top_k 1, no weights, scale 1, bf16: all_to_all_v then the combine gives the tokens back bit for bit."""
    torch, coll = torch_cuda, coll_mod
    from container_engine_accelerators_b200.models.workloads import expert_dispatch_plan
    p = expert_dispatch_plan(n, 40, ROW, top_k=1, skew=1.3, seed=4)
    with Group(torch, coll, n) as g:
        gen = torch.Generator().manual_seed(7)
        xs = [(torch.randn(40, ROW, generator=gen) * 3 + 0.5).to(torch.bfloat16) for _ in range(n)]
        sends = [_dispatch_send(torch, xs[r], p.index[r]).cuda() for r in range(n)]
        plan = Plan(p.rows, p.send_off, p.recv_off, p.index, p.weights)
        eo = [c.empty(plan.recv_rows * ROW, torch.bfloat16) for c in g.comms]
        g.sync()
        for r, c in enumerate(g.comms):
            c.all_to_all_v(sends[r].view(-1), eo[r], ROW, *plan.args(r), stream=g.streams[r])
        outs = poisoned_outs(g, plan, torch.bfloat16)
        g.sync()
        call(g, eo, outs, plan, False, 1.0)
        for r in range(n):
            assert_same(outs[r].cpu().view(40, ROW), xs[r], f"rank {r}: combine after all_to_all_v", nan_payloads=True)
        for c, d in zip(g.comms, eo):
            c.release(d)


def test_moe_round_trip(torch_cuda, coll_mod):
    """FP8 dispatch, a stand-in expert per rank (dequantise, scale by an expert factor, write the arena expert_out on the rank's stream),
    then the combine with the plan's weights: bit-exact against the reference from expert_out, within FP8 tolerance of fp32."""
    torch, coll = torch_cuda, coll_mod
    from container_engine_accelerators_b200.models.workloads import expert_dispatch_plan
    n, tokens, top_k, block, row = 4, 64, 2, 128, 256
    p = expert_dispatch_plan(n, tokens, row, top_k=top_k, skew=1.0, seed=12)
    plan = Plan(p.rows, p.send_off, p.recv_off, p.index, p.weights)
    with Group(torch, coll, n) as g:
        gen = torch.Generator().manual_seed(3)
        xs = [torch.randn(tokens, row, generator=gen).to(torch.bfloat16) for _ in range(n)]
        sends = [_dispatch_send(torch, xs[r], p.index[r]).cuda().view(-1) for r in range(n)]
        q = [c.empty(plan.recv_rows * row, torch.float8_e4m3fn) for c in g.comms]
        sc = [c.empty(plan.recv_rows * row // block, torch.float32) for c in g.comms]
        eo = [c.empty(plan.recv_rows * row, torch.bfloat16) for c in g.comms]
        outs = [torch.full((tokens * row,), float("nan"), dtype=torch.float32, device="cuda") for _ in range(n)]
        factor = [1.0 + 0.25 * d for d in range(n)]
        idx = [torch.from_numpy(p.index[r]).cuda() for r in range(n)]
        gate = [torch.from_numpy(p.weights[r]).cuda() for r in range(n)]
        g.sync()
        for r, c in enumerate(g.comms):
            c.all_to_all_v_quantized(sends[r], q[r], sc[r], row, *plan.args(r), block=block, stream=g.streams[r])
        for r, c in enumerate(g.comms):
            with torch.cuda.stream(g.streams[r]):
                y = q[r].float().view(-1, block) * sc[r].view(-1, 1) * factor[r]
                eo[r].copy_(y.view(-1).to(torch.bfloat16))
        for r, c in enumerate(g.comms):
            c.all_to_all_v_combine(eo[r], outs[r], row, *plan.args(r), idx[r], gate[r], stream=g.streams[r])
        g.sync()
        g.check_async()
        eo_cpu = [e.float().cpu().numpy().reshape(-1, row) for e in eo]
        for r in range(n):
            rows, so, ro = plan.args(r)
            want = cr.combine(cr.plan_lookup(eo_cpu, rows, so, ro), p.index[r], p.weights[r], 1.0, torch.float32)
            got = outs[r].cpu().view(tokens, row)
            assert_same(got, want, f"rank {r}: combine of the expert outputs")
            dest = np.searchsorted(p.send_off[r], p.index[r], side="right") - 1                    # the rank each slot went to
            wf = torch.from_numpy((p.weights[r] * np.asarray(factor, dtype=np.float32)[dest]).sum(axis=1).astype(np.float32))
            exact = xs[r].float() * wf[:, None]
            tol = 0.08 * exact.abs() + 1e-3 * wf[:, None] * xs[r].float().abs().amax(dim=1, keepdim=True)
            assert ((got - exact).abs() <= tol).all(), f"rank {r}: {float((got - exact).abs().max())}"


def test_back_to_back_calls_with_few_ctas(torch_cuda, coll_mod):
    """Two calls with expert_out rewritten between them on every rank's own stream, and 3 CTAs so each walks many warps: the closing
    barrier must keep every peer's first pull ahead of the rewrite."""
    torch, coll = torch_cuda, coll_mod
    n, top_k = 4, 8
    with Group(torch, coll, n) as g:
        for c in g.comms:
            c.set_max_ctas(3)
        plan = dispatch_plan(n, top_k, seed=21, tokens=160)
        xs, eo = expert_outs(g, plan.recv_rows, torch.bfloat16, seed=5)
        xs2 = [qr.gen(plan.recv_rows * ROW, torch.bfloat16, 16, 900 + r) for r in range(n)]
        new = [x.cuda() for x in xs2]
        idx = [g.dev(c, plan.index[r]) for r, c in enumerate(g.comms)]
        w = [g.dev(c, plan.weights[r]) for r, c in enumerate(g.comms)]
        o1, o2 = poisoned_outs(g, plan, torch.float32), poisoned_outs(g, plan, torch.float32)
        g.sync()
        for r, c in enumerate(g.comms):
            c.all_to_all_v_combine(eo[r], o1[r], ROW, *plan.args(r), idx[r], w[r], stream=g.streams[r])
            with torch.cuda.stream(g.streams[r]):
                eo[r].copy_(new[r])
            c.all_to_all_v_combine(eo[r], o2[r], ROW, *plan.args(r), idx[r], w[r], stream=g.streams[r])
        g.sync()
        g.check_async()
        check(g, xs, o1, plan, True, 1.0, "first of two calls")
        check(g, xs2, o2, plan, True, 1.0, "second of two calls")
        for c in g.comms:
            assert c.stats()["kernel_launches"] == 2


def test_cuda_graph_replays_the_same_bits(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    n, top_k = 3, 2
    with Group(torch, coll, n) as g:
        plan = dispatch_plan(n, top_k, seed=9)
        xs, eo = expert_outs(g, plan.recv_rows, torch.float16, seed=44)
        idx = [g.dev(c, plan.index[r]) for r, c in enumerate(g.comms)]
        w = [g.dev(c, plan.weights[r]) for r, c in enumerate(g.comms)]
        outs = poisoned_outs(g, plan, torch.bfloat16)
        g.sync()
        graphs = []
        for r, c in enumerate(g.comms):
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=g.streams[r]):
                c.all_to_all_v_combine(eo[r], outs[r], ROW, *plan.args(r), idx[r], w[r], scale=0.5)
            graphs.append(gr)
        for rep in range(2):
            for o in outs:
                o.view(torch.uint8).fill_(0x5A)
            g.sync()
            for r, gr in enumerate(graphs):
                with torch.cuda.stream(g.streams[r]):
                    gr.replay()
            g.sync()
            g.check_async()
            check(g, xs, outs, plan, True, 0.5, f"graph replay {rep}")
        del graphs


def _raw(coll, comm, eo, out, row_elems, recv_rows, rows, soff, roff, index, weights, tokens, top_k, in_dt, out_dt):
    n = comm.nranks
    arr = lambda xs: (C.c_int64 * n)(*xs)
    ep = coll.Epilogue(in_dt, out_dt, 1.0)
    return coll.load().b200collAllToAllvCombine(C.c_void_p(eo), C.c_void_p(out), row_elems, recv_rows, arr(rows), arr(soff), arr(roff),
                                                C.cast(C.c_void_p(index), C.POINTER(C.c_int32)), C.cast(C.c_void_p(weights), C.POINTER(C.c_float)),
                                                tokens, top_k, C.byref(ep), comm._h, None)


def test_placement_and_argument_errors(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    with Group(torch, coll, 2) as g:
        c = g.comms[0]
        row, rows_n = 64, 8
        eo = c.empty(rows_n * row, torch.bfloat16)
        plain_eo = torch.empty(rows_n * row, dtype=torch.bfloat16, device="cuda")
        out = torch.empty(4 * row, dtype=torch.bfloat16, device="cuda")
        idx = torch.zeros(4, 2, dtype=torch.int32, device="cuda")
        w = torch.ones(4, 2, device="cuda")
        EO, O, I, W = eo.data_ptr(), out.data_ptr(), idx.data_ptr(), w.data_ptr()
        BF, E4 = coll.BF16, coll.FP8_E4M3
        ok = dict(eo=EO, out=O, row_elems=row, recv_rows=rows_n, rows=[2, 3], soff=[0, 2], roff=[0, 4], index=I, weights=W, tokens=4,
                  top_k=2, in_dt=BF, out_dt=BF)
        cases = [("expert_out outside the arena", INVALID_USAGE, dict(eo=plain_eo.data_ptr()))] + [(what, INVALID_ARGUMENT, kw) for what, kw in [
            ("null expert_out", dict(eo=0)),
            ("null out", dict(out=0)),
            ("null index with tokens", dict(index=0)),
            ("FP8 input", dict(in_dt=E4)),
            ("FP8 output", dict(out_dt=E4)),
            ("row_elems 0", dict(row_elems=0)),
            ("row_elems 40", dict(row_elems=40)),
            ("top_k 0", dict(top_k=0)),
            ("negative rows", dict(rows=[2, -3])),
            ("negative send offset", dict(soff=[-1, 2])),
            ("negative destination", dict(roff=[0, -4])),
            ("destination past recv_rows", dict(roff=[0, 6])),
            ("destination offset past recv_rows, no rows", dict(rows=[2, 0], roff=[0, 9])),
            ("overlapping send ranges", dict(soff=[0, 1])),
            ("misaligned expert_out", dict(eo=EO + 8)),
            ("misaligned out", dict(out=O + 4)),
            ("misaligned index", dict(index=I + 2)),
            ("misaligned weights", dict(weights=W + 1)),
            ("out overlaps expert_out", dict(out=EO)),
            ("out overlaps index", dict(index=O + 16)),
            ("out overlaps weights", dict(weights=O + 64)),
            ("more than 2^31 - 1 vectors of out", dict(tokens=(1 << 31) // 4)),
            ("tokens * top_k > 2^31 - 1", dict(tokens=1 << 30, top_k=4, row_elems=16)),
        ]]
        for what, want, kw in cases:
            a = dict(ok, **kw)
            rc = _raw(coll, c, a["eo"], a["out"], a["row_elems"], a["recv_rows"], a["rows"], a["soff"], a["roff"], a["index"], a["weights"],
                      a["tokens"], a["top_k"], a["in_dt"], a["out_dt"])
            expect_refused(rc, want, what=what)
        with pytest.raises(ValueError):
            c.all_to_all_v_combine(eo, out, row, [2, 3], [0, 1], [0, 4], idx, w)          # Python refuses it before the library call
        assert_nothing_launched(c)                                                      # nothing was launched or counted
        g.check_async()
        del eo
    # one rank: expert_out may be any device buffer
    with Group(torch, coll, 1) as g:
        plan = hand_plan(1, 3, seed=2)
        xs = [qr.gen(plan.recv_rows * ROW, torch.float32, 16, 8)]
        eo = [xs[0].cuda()]
        assert not g.comms[0].is_symmetric(eo[0])
        outs = poisoned_outs(g, plan, torch.float16)
        call(g, eo, outs, plan, True, 2.0)
        check(g, xs, outs, plan, True, 2.0, "one rank outside the arena")
        assert g.comms[0].stats()["algo_calls"]["copy"] == 1 and g.comms[0].stats()["kernel_launches"] == 1


def test_multi_gpu(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    n = torch.cuda.device_count()
    with Group(torch, coll, n, arena_mb=256, devices=list(range(n))) as g:
        for plan in (dispatch_plan(n, 8, seed=1, tokens=512), hand_plan(n, 2, seed=3)):
            xs, eo = expert_outs(g, plan.recv_rows, torch.bfloat16, seed=90)
            outs = poisoned_outs(g, plan, torch.bfloat16)
            call(g, eo, outs, plan, True, 1.0)
            check(g, xs, outs, plan, True, 1.0, "multi-GPU")
            for c, d in zip(g.comms, eo):
                c.release(d)


def test_perf_tool_combine_bit_exact(torch_cuda, coll_lib):
    for devs, extra in (("0,0", ["-d", "bfloat16", "--out-dtype", "float", "--combine", "4", "-b", "64K", "-e", "4M", "-f", "8"]),
                        ("0,0,0", ["-d", "half", "--out-dtype", "bfloat16", "--combine", "2", "--row-len", "96", "-b", "1M", "-e", "1M"]),
                        ("0", ["-d", "float", "--out-dtype", "half", "--combine", "8", "--row-len", "512", "-b", "1M", "-e", "1M"])):
        out = run_perf(["--op", "alltoall", *extra, "-w", "1", "-n", "2", "-c", "1"], devs)
        rows = [l for l in out.splitlines() if l.strip() and not l.startswith("#")]
        assert rows, out
