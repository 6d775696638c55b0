"""The fused reduce-scatter, residual add and RMSNorm for sequence-parallel layers, wide and FP8, on an H100 (`pytest -m gpu`), virtual
ranks sharing cuda:0 unless a test says otherwise.

Bit-exact means equal (NaN matching NaN at the same position) to tests/coll_rs_rmsnorm_reference, on every rank. Every rank holds a
different residual shard, so a row read or stored at the wrong index shows."""
import pytest

from container_engine_accelerators_b200.ops.coll import INVALID_ARGUMENT, INVALID_USAGE
from tests import coll_quant_reference as Q
from tests import coll_rs_rmsnorm_reference as ref
from tests.coll_fp_reference import assert_same
from tests.coll_gpu_harness import (DTYPES, Group, assert_nothing_launched, coll_mod, expect_refused, poison, run_perf,  # noqa: F401
                                    run_python, torch_cuda)

pytestmark = pytest.mark.gpu

DT_NAMES = ("bf16", "f16", "f32")
_groups = {}


@pytest.fixture(scope="module")
def groups(torch_cuda, coll_mod):
    def get(n):
        if n not in _groups:
            _groups[n] = Group(torch_cuda, coll_mod, n)
        return _groups[n]
    yield get
    for g in _groups.values():
        g.destroy()
    _groups.clear()


def data(torch, n, s, row_len, dt, seed):
    """Per rank x [n*s, row_len], per rank residual shard [s, row_len] (each at its own scale), gamma."""
    g = torch.Generator().manual_seed(seed)
    xs = [(torch.randn(n * s, row_len, generator=g) * (0.5 + r)).to(dt) for r in range(n)]
    shards = [(torch.randn(s, row_len, generator=g) * (1 + r)).to(dt) for r in range(n)]
    gamma = ((torch.rand(row_len, generator=g) * 2 - 0.5) * torch.exp2(torch.randint(-3, 4, (row_len,), generator=g).float())).to(dt)
    return xs, shards, gamma


def run(g, xs, shards, gamma, eps, gather, quant=None):
    """One call on every rank: x in the arena, the residual shard a plain tensor, out (q, scales) in the arena when gathering, else plain
    tensors; outputs poisoned first. quant: None (the wide call) or (block, wire). Returns [(shard, out) or (shard, q, scales)] per rank on
    the CPU, and the stats before and after."""
    torch = g.torch
    n = g.n
    s, row_len = shards[0].shape
    rows, dt = n * s, shards[0].dtype
    o_rows = rows if gather else s
    bases, bufs = [], []

    def arena(c, k, t):
        base = c.empty(max(k, 1), t)
        bases.append((c, base))
        return base[:k]

    def out_buf(c, k, t):
        return arena(c, k, t) if gather else torch.empty(k, dtype=t, device="cuda")

    for r, c in enumerate(g.comms):
        x = arena(c, rows * row_len, dt).view(rows, row_len)
        x.copy_(xs[r].cuda())
        rd = shards[r].clone().cuda()
        if quant is None:
            outs = (out_buf(c, o_rows * row_len, dt).view(o_rows, row_len),)
        else:
            block, wire = quant
            outs = (out_buf(c, o_rows * row_len, wire).view(o_rows, row_len),
                    out_buf(c, o_rows * (row_len // block), torch.float32).view(o_rows, row_len // block))
        poison(outs)
        bufs.append((x, rd) + outs)
    gd = gamma.cuda()
    torch.cuda.synchronize()
    before = [c.stats() for c in g.comms]
    if quant is None:
        g.run(lambda r, c, st: c.reduce_scatter_rms_norm(bufs[r][0], bufs[r][1], gd, bufs[r][2], eps=eps, gather=gather, stream=st))
    else:
        g.run(lambda r, c, st: c.reduce_scatter_rms_norm_quantized(bufs[r][0], bufs[r][1], gd, bufs[r][2], bufs[r][3], block=quant[0], wire=quant[1],
                                                                   eps=eps, gather=gather, stream=st))
    after = [c.stats() for c in g.comms]
    got = [tuple(t.cpu() for t in b[1:]) for b in bufs]
    for c, base in bases:
        c.release(base)
    return got, before, after


def check(got, want, what):
    for r, (gs, ws) in enumerate(zip(got, want)):
        assert len(gs) == len(ws)
        for i, (a, b) in enumerate(zip(gs, ws)):
            assert_same(a.reshape(-1), b.reshape(-1), f"{what} output {i} rank {r}")


def check_stats(before, after, n, s, row_len, es, what):
    algo = "copy" if n == 1 else "twoshot"
    for b, a in zip(before, after):
        assert a["algo_calls"][algo] == b["algo_calls"][algo] + 1, what
        assert sum(a["algo_calls"].values()) == sum(b["algo_calls"].values()) + 1, what
        assert a["calls"][2] == b["calls"][2] + 1 and sum(a["calls"]) == sum(b["calls"]) + 1, what      # reducescatter
        assert a["bytes"][2] - b["bytes"][2] == s * row_len * es, what
        assert a["kernel_launches"] == b["kernel_launches"] + 1, what


SWEEP = [(1, [0, 1, 5]), (2, [0, 1, 4]), (3, [0, 1, 3]), (4, [0, 1, 3]), (8, [0, 1, 2])]


@pytest.mark.parametrize("dtn", DT_NAMES)
@pytest.mark.parametrize("n,s_list", SWEEP, ids=[f"n{n}" for n, _ in SWEEP])
def test_bit_exact_sweep(torch_cuda, groups, n, s_list, dtn):
    torch = torch_cuda
    dt = DTYPES[dtn]
    g = groups(n)
    es = torch.empty((), dtype=dt).element_size()
    for row_len in (16, 4096, 7168, 16384):
        for s in s_list:
            xs, shards, gamma = data(torch, n, s, row_len, dt, seed=s * 31 + row_len + n)
            for gather in (False, True):
                want = ref.rs_rms_norm(xs, shards, gamma, 1e-6, dt, gather)
                got, before, after = run(g, xs, shards, gamma, 1e-6, gather)
                what = f"n={n} {dtn} s={s} row_len={row_len} gather={gather}"
                check(got, want, what)
                check_stats(before, after, n, s, row_len, es, what)


QSWEEP = [(1, 3), (2, 2), (3, 1), (4, 3), (8, 1)]


@pytest.mark.parametrize("n,s", QSWEEP, ids=[f"n{n}" for n, _ in QSWEEP])
def test_quantised_bit_exact_sweep(torch_cuda, groups, n, s):
    torch = torch_cuda
    g = groups(n)
    for dtn in DT_NAMES:
        dt = DTYPES[dtn]
        es = torch.empty((), dtype=dt).element_size()
        for row_len, block in ((512, 16), (4096, 128), (7168, 128), (16384, 512)):
            for wn in ("e4m3", "e5m2"):
                xs, shards, gamma = data(torch, n, s, row_len, dt, seed=row_len + n + block)
                for gather in (False, True):
                    want = ref.rs_rms_norm_quantized(xs, shards, gamma, 1e-6, dt, block, DTYPES[wn], gather)
                    got, before, after = run(g, xs, shards, gamma, 1e-6, gather, (block, DTYPES[wn]))
                    what = f"n={n} {dtn}->{wn} block={block} s={s} row_len={row_len} gather={gather}"
                    check(got, want, what)
                    check_stats(before, after, n, s, row_len, es, what)


@pytest.mark.parametrize("n", [2, 3, 4])
def test_equals_the_all_reduce_form_on_the_stacked_residual(torch_cuda, groups, n):
    """The header's equivalence, against the library itself: all_reduce_rms_norm (and its quantised form) on the stacked residual leaves
    the new shards slice by slice, and its out (q, scales) is every rank's gathered out and, slice by slice, the scattered one."""
    torch = torch_cuda
    g = groups(n)
    s, row_len = 5, 7168
    for dtn in DT_NAMES:
        dt = DTYPES[dtn]
        xs, shards, gamma = data(torch, n, s, row_len, dt, seed=70 + n)
        full = torch.cat(shards)
        for quant in (None, (128, torch.float8_e4m3fn)):
            xb = [c.empty(n * s * row_len, dt) for c in g.comms]
            xa = [t.view(n * s, row_len) for t in xb]
            for r in range(n):
                xa[r].copy_(xs[r].cuda())
            res = [full.clone().cuda() for _ in g.comms]
            gd = gamma.cuda()
            if quant is None:
                outs = [(torch.empty(n * s, row_len, dtype=dt, device="cuda"),) for _ in g.comms]
                g.run(lambda r, c, st: c.all_reduce_rms_norm(xa[r], res[r], gd, outs[r][0], eps=1e-6, stream=st))
            else:
                outs = [(torch.empty(n * s, row_len, dtype=quant[1], device="cuda"), torch.empty(n * s, row_len // quant[0], device="cuda"))
                        for _ in g.comms]
                g.run(lambda r, c, st: c.all_reduce_rms_norm_quantized(xa[r], res[r], gd, *outs[r], block=quant[0], wire=quant[1], eps=1e-6, stream=st))
            for c, t in zip(g.comms, xb):
                c.release(t)
            wide_h, wide_o = res[0].cpu(), [t.cpu() for t in outs[0]]
            for gather in (False, True):
                got, _, _ = run(g, xs, shards, gamma, 1e-6, gather, quant)
                for r in range(n):
                    what = f"n={n} {dtn} quant={quant} gather={gather} rank {r}"
                    assert_same(got[r][0], wide_h[r * s:(r + 1) * s], what + " residual")
                    for i, w in enumerate(wide_o):
                        assert_same(got[r][1 + i], w if gather else w[r * s:(r + 1) * s], f"{what} output {i}")


def _ulps(torch, a, b, dt):
    """|a - b| in units of the last place of dt at the larger magnitude (normal range; subnormals share the smallest normal's ulp)."""
    mant = {torch.bfloat16: 7, torch.float16: 10}[dt]
    emin = {torch.bfloat16: -126, torch.float16: -14}[dt]
    a, b = a.double(), b.double()
    m = torch.maximum(a.abs(), b.abs())
    e = torch.floor(torch.log2(torch.where(m > 0, m, torch.ones_like(m)))).clamp(min=emin)
    return ((a - b).abs() / torch.exp2(e - mant)).max().item()


@pytest.mark.parametrize("n", [2, 4])
def test_agrees_with_the_unfused_composition(torch_cuda, groups, n):
    """reduce_scatter + add_ + F.rms_norm + all_gather, the four calls the fused one replaces, agree within 2 ulp of bf16 or fp16. x holds
    small multiples of 1/4, so the reduce-scatter's sum is exact and the residual gets the same bits; out differs only by how PyTorch
    rounds the norm and the gamma product."""
    import torch.nn.functional as F
    torch = torch_cuda
    g = groups(n)
    s, row_len = 6, 4096
    for dtn in ("bf16", "f16"):
        dt = DTYPES[dtn]
        gen = torch.Generator().manual_seed(n)
        xs = [(torch.randint(-8, 9, (n * s, row_len), generator=gen).float() / 4).to(dt) for _ in range(n)]
        shards = [(torch.randn(s, row_len, generator=gen) * 2).to(dt) for _ in range(n)]
        gamma = (torch.rand(row_len, generator=gen) + 0.5).to(dt)
        fused, _, _ = run(g, xs, shards, gamma, 1e-6, True)
        xa = [c.empty(n * s * row_len, dt) for c in g.comms]
        part = [c.empty(s * row_len, dt) for c in g.comms]
        normed = [c.empty(s * row_len, dt) for c in g.comms]
        outs = [c.empty(n * s * row_len, dt) for c in g.comms]
        for r in range(n):
            xa[r].copy_(xs[r].reshape(-1).cuda())
        res = [sh.clone().cuda() for sh in shards]
        gd = gamma.cuda()

        # in phases: a PyTorch kernel's first launch loads its module, which waits for the kernels already running, so it must not be
        # enqueued while a rank's collective waits for a peer this thread has not launched yet
        g.run(lambda r, c, st: c.reduce_scatter(xa[r], part[r], stream=st))
        for r in range(n):
            res[r].add_(part[r].view(s, row_len))
            normed[r].copy_(F.rms_norm(res[r], (row_len,), gd, 1e-6).reshape(-1))
        g.run(lambda r, c, st: c.all_gather(normed[r], outs[r], stream=st))
        for r in range(n):
            what = f"n={n} {dtn} rank {r}"
            assert_same(res[r].cpu(), fused[r][0], what + " residual")
            assert _ulps(torch, outs[r].cpu().view(n * s, row_len), fused[r][1], dt) <= 2, what
        for c, lst in zip(g.comms, zip(xa, part, normed, outs)):
            for t in lst:
                c.release(t)


@pytest.mark.parametrize("n", [1, 2])
def test_special_values(torch_cuda, groups, n):
    torch = torch_cuda
    g = groups(n)
    s, row_len = 5, 512
    for dtn in DT_NAMES:
        dt = DTYPES[dtn]
        xs, shards, gamma = data(torch, n, s, row_len, dt, seed=3)
        xs[0][0, 3] = float("nan")                                   # row 0: rank 0's slice
        xs[-1][n * s - 1, 300] = float("inf")                        # the last row: the last rank's slice
        shards[-1][1, 40] = float("-inf")
        for x in xs:
            x[2].zero_()
        shards[0][2].zero_()                                         # row 2: all zero
        for eps in (0.0, 1e-6):
            for gather in (False, True):
                want = ref.rs_rms_norm(xs, shards, gamma, eps, dt, gather)
                got, _, _ = run(g, xs, shards, gamma, eps, gather)
                check(got, want, f"{dtn} eps={eps} gather={gather}")
                out0 = got[0][1]
                assert torch.isnan(out0[0]).all(), "a NaN in h makes the whole row NaN"
                assert torch.isnan(out0[2]).all() == (eps == 0.0), "0 / sqrt(0) is NaN, eps > 0 gives zeros"
                if eps:
                    assert (out0[2] == 0).all()
                for block, wn in ((128, "e4m3"),):
                    qwant = ref.rs_rms_norm_quantized(xs, shards, gamma, eps, dt, block, DTYPES[wn], gather)
                    qgot, _, _ = run(g, xs, shards, gamma, eps, gather, (block, DTYPES[wn]))
                    check(qgot, qwant, f"{dtn}->{wn} eps={eps} gather={gather}")


def test_forced_algorithms_change_nothing(torch_cuda, groups):
    torch = torch_cuda
    n, s, row_len, dt = 4, 3, 4096, torch.bfloat16
    g = groups(n)
    xs, shards, gamma = data(torch, n, s, row_len, dt, seed=11)
    want = ref.rs_rms_norm(xs, shards, gamma, 1e-6, dt, True)
    try:
        for algo in ("oneshot", "ll", "ll2", "twoshot", "nvls", "auto"):
            for c in g.comms:
                c.set_algo(algo)
            got, before, after = run(g, xs, shards, gamma, 1e-6, True)
            check(got, want, algo)
            check_stats(before, after, n, s, row_len, 2, algo)
    finally:
        for c in g.comms:
            c.set_algo("auto")


def test_x_overwritten_right_after_the_call(torch_cuda, groups):
    """The closing barrier frees x: each rank's stream overwrites its x right after the call, and every rank still gets the values of
    the x it passed."""
    torch = torch_cuda
    n, s, row_len, dt = 4, 8, 16384, torch.bfloat16
    g = groups(n)
    xs, shards, gamma = data(torch, n, s, row_len, dt, seed=21)
    xb = [c.empty(n * s * row_len, dt) for c in g.comms]
    ob = [c.empty(n * s * row_len, dt) for c in g.comms]
    xa, outs = [t.view(n * s, row_len) for t in xb], [t.view(n * s, row_len) for t in ob]
    res = [sh.clone().cuda() for sh in shards]
    for r in range(n):
        xa[r].copy_(xs[r].cuda())
    gd = gamma.cuda()
    torch.cuda.synchronize()
    for r, c in enumerate(g.comms):
        c.reduce_scatter_rms_norm(xa[r], res[r], gd, outs[r], gather=True, stream=g.streams[r])
    for r in range(n):                                               # enqueued once every rank's call is (see the unfused test)
        with torch.cuda.stream(g.streams[r]):
            xa[r].fill_(float("nan"))
    g.sync()
    g.check_async()
    check([(res[r].cpu(), outs[r].cpu()) for r in range(n)], ref.rs_rms_norm(xs, shards, gamma, 1e-6, dt, True), "x overwritten")
    for c, a, b in zip(g.comms, xb, ob):
        c.release(a)
        c.release(b)


@pytest.mark.parametrize("n", [2, 4])
def test_scattered_q_feeds_the_block_scaled_all_gather(torch_cuda, groups, n):
    """Each rank's scattered q and scales [S, row_len] are a valid input of all_gather_block_scaled(block=(1, block)); what it gathers is
    the gathered call's q dequantised."""
    torch = torch_cuda
    g = groups(n)
    s, row_len, dt = 3, 4096, torch.bfloat16
    for wn in ("e4m3", "e5m2"):
        for block in (32, 128):
            wire = DTYPES[wn]
            xs, shards, gamma = data(torch, n, s, row_len, dt, seed=block + n)
            bases = [(c.empty(n * s * row_len, dt), c.empty(s * row_len, wire), c.empty(s * row_len // block, torch.float32)) for c in g.comms]
            xa = [b[0].view(n * s, row_len) for b in bases]
            qs, ss = [b[1].view(s, row_len) for b in bases], [b[2].view(s, row_len // block) for b in bases]
            res = [sh.clone().cuda() for sh in shards]
            outs = [torch.full((n * s, row_len), float("nan"), device="cuda") for _ in g.comms]
            for r in range(n):
                xa[r].copy_(xs[r].cuda())
            gd = gamma.cuda()
            g.run(lambda r, c, st: c.reduce_scatter_rms_norm_quantized(xa[r], res[r], gd, qs[r], ss[r], block=block, wire=wire, stream=st))
            g.run(lambda r, c, st: c.all_gather_block_scaled(qs[r], ss[r], outs[r], block=(1, block), stream=st))
            gathered, _, _ = run(g, xs, shards, gamma, 1e-6, True, (block, wire))
            _, wq, wsc = gathered[0]
            deq = (wq.float().view(n * s, -1, block) * wsc.view(n * s, -1, 1)).reshape(-1)
            want = Q.reduce([deq], 1.0, torch.float32).view(n * s, row_len)     # the all-gather's (+0 + v) * scale: -0 comes out as +0
            for r in range(n):
                assert_same(outs[r].cpu(), want, f"{wn} block={block} rank {r}")
                assert_same(gathered[r][1].view(torch.uint8), wq.view(torch.uint8), f"{wn} block={block} gathered q rank {r}")
            for c, b in zip(g.comms, bases):
                for t in b:
                    c.release(t)


def test_cuda_graph_interleaved(torch_cuda, groups):
    """Capture the reduce-scatter form (wide, gathered; quantised, scattered) between all-reduce rms-norm calls on the same comms, replay
    twice with new inputs, and check every result."""
    torch = torch_cuda
    n = 2
    g = groups(n)
    dt, s, row_len, block, wire = torch.bfloat16, 6, 4096, 128, torch.float8_e4m3fn
    rows = n * s
    bases = [[c.empty(rows * row_len, dt) for _ in range(4)] + [c.empty(s * row_len, wire), c.empty(s * row_len // block, torch.float32)]
             for c in g.comms]
    xs, ars, aos, rso = ([b[i].view(rows, row_len) for b in bases] for i in range(4))
    qs, ss = [b[4].view(s, row_len) for b in bases], [b[5].view(s, row_len // block) for b in bases]
    shw = [torch.empty(s, row_len, dtype=dt, device="cuda") for _ in range(n)]
    shq = [torch.empty(s, row_len, dtype=dt, device="cuda") for _ in range(n)]
    gamma = (torch.rand(row_len) + 0.5).to(dt)
    gd = gamma.cuda()
    graphs = [torch.cuda.CUDAGraph() for _ in g.comms]
    torch.cuda.synchronize()
    for r, c in enumerate(g.comms):
        with torch.cuda.graph(graphs[r], stream=g.streams[r]):
            c.all_reduce_rms_norm(xs[r], ars[r], gd, aos[r], stream=g.streams[r])
            c.reduce_scatter_rms_norm(xs[r], shw[r], gd, rso[r], gather=True, stream=g.streams[r])
            c.reduce_scatter_rms_norm_quantized(xs[r], shq[r], gd, qs[r], ss[r], block=block, wire=wire, stream=g.streams[r])
    torch.cuda.synchronize()
    from tests import coll_rmsnorm_reference as R
    for it in range(2):
        gen = torch.Generator().manual_seed(200 + it)
        hx = [torch.randn(rows, row_len, generator=gen).to(dt) for _ in range(n)]
        hres = torch.randn(rows, row_len, generator=gen).to(dt)
        hsh = [torch.randn(s, row_len, generator=gen).to(dt) for _ in range(n)]
        for r in range(n):
            xs[r].copy_(hx[r].cuda())
            ars[r].copy_(hres.cuda())
            shw[r].copy_(hsh[r].cuda())
            shq[r].copy_(hsh[r].cuda())
        torch.cuda.synchronize()
        for r in range(n):
            with torch.cuda.stream(g.streams[r]):
                graphs[r].replay()
        torch.cuda.synchronize()
        g.check_async()
        wh, wo = R.rms_norm(hx, hres, gamma, 1e-6, dt)
        wide = ref.rs_rms_norm(hx, hsh, gamma, 1e-6, dt, True)
        quant = ref.rs_rms_norm_quantized(hx, hsh, gamma, 1e-6, dt, block, wire, False)
        for r in range(n):
            assert_same(ars[r].cpu(), wh, f"all-reduce residual replay {it} rank {r}")
            assert_same(aos[r].cpu(), wo, f"all-reduce out replay {it} rank {r}")
        check([(shw[r].cpu(), rso[r].cpu()) for r in range(n)], wide, f"wide replay {it}")
        check([(shq[r].cpu(), qs[r].cpu(), ss[r].cpu()) for r in range(n)], quant, f"quantised replay {it}")
    del graphs
    torch.cuda.synchronize()
    for c, b in zip(g.comms, bases):
        for t in b:
            c.release(t)


def test_refusals_launch_nothing(torch_cuda, coll_mod):
    import ctypes as C
    torch, coll = torch_cuda, coll_mod
    L = coll.load()
    with Group(torch, coll, 2) as g:
        c = g.comms[0]
        dt = torch.bfloat16
        xb = c.empty(8 * 256, dt)
        x = xb.view(8, 256)
        res = torch.zeros(4, 256, dtype=dt, device="cuda")
        gam = torch.ones(256, dtype=dt, device="cuda")
        out = torch.zeros(8, 256, dtype=dt, device="cuda")
        q = torch.zeros(8, 256, dtype=torch.float8_e4m3fn, device="cuda")
        sc = torch.zeros(8, 2, dtype=torch.float32, device="cuda")
        plain_x = torch.zeros(8, 256, dtype=dt, device="cuda")
        BF16, E4M3 = (coll.torch_dtype_code(t) for t in (dt, torch.float8_e4m3fn))
        p = lambda t, off=0: C.c_void_p(t.data_ptr() + off)
        f = lambda t, off=0: C.cast(C.c_void_p(t.data_ptr() + off), C.POINTER(C.c_float))
        ok = dict(x=p(x), res=p(res), gam=p(gam), out=p(out), q=p(q), s=f(sc), rows=8, row_len=256, eps=1e-6, gather=0, dt=BF16, wire=E4M3,
                  block=128)

        def wide(**kw):
            a = {**ok, **kw}
            return L.b200collReduceScatterRmsNorm(a["x"], a["res"], a["gam"], a["out"], a["rows"], a["row_len"], a["eps"], a["gather"], a["dt"],
                                                  c._h, C.c_void_p(0))

        def quant(**kw):
            a = {**ok, **kw}
            return L.b200collReduceScatterRmsNormQuantized(a["x"], a["res"], a["gam"], a["q"], a["s"], a["rows"], a["row_len"], a["eps"], a["gather"],
                                                           a["dt"], a["wire"], a["block"], c._h, C.c_void_p(0))

        cases = [
            (wide, dict(rows=7), INVALID_ARGUMENT, "rows must be a multiple of nranks"),
            (wide, dict(gather=2), INVALID_ARGUMENT, "gather must be 0 or 1"),
            (wide, dict(gather=-1), INVALID_ARGUMENT, "gather must be 0 or 1"),
            (wide, dict(dt=E4M3), INVALID_ARGUMENT, "dtype"),
            (wide, dict(row_len=24), INVALID_ARGUMENT, "row_len"),
            (wide, dict(eps=-1.0), INVALID_ARGUMENT, "eps"),
            (wide, dict(rows=1 << 31), INVALID_ARGUMENT, "2^31"),
            (wide, dict(out=C.c_void_p(0)), INVALID_ARGUMENT, "null"),
            (wide, dict(res=p(res, 2)), INVALID_ARGUMENT, "16-byte"),
            (wide, dict(out=p(res)), INVALID_ARGUMENT, "out must not overlap"),
            (wide, dict(out=p(res, -2048), gather=1), INVALID_ARGUMENT, "out must not overlap"),     # sized by the gathered shape
            (wide, dict(res=p(x, 2048)), INVALID_ARGUMENT, "residual must not overlap"),
            (wide, dict(x=p(plain_x)), INVALID_USAGE, "symmetric arena"),
            (wide, dict(gather=1), INVALID_USAGE, "out (gather) must lie in the symmetric arena"),
            (quant, dict(rows=5), INVALID_ARGUMENT, "rows must be a multiple of nranks"),
            (quant, dict(gather=3), INVALID_ARGUMENT, "gather must be 0 or 1"),
            (quant, dict(block=100), INVALID_ARGUMENT, "block must be"),
            (quant, dict(wire=BF16), INVALID_ARGUMENT, "wire_dtype"),
            (quant, dict(s=f(q, 64)), INVALID_ARGUMENT, "q must not overlap"),
            (quant, dict(s=f(res)), INVALID_ARGUMENT, "scales must not overlap"),
            (quant, dict(x=p(plain_x)), INVALID_USAGE, "symmetric arena"),
            (quant, dict(gather=1), INVALID_USAGE, "q and scales (gather) must lie in the symmetric arena"),
        ]
        torch.cuda.synchronize()
        for fn, kw, code, msg in cases:
            prefix = "reduce-scatter rms-norm: " if fn is wide else "quantised reduce-scatter rms-norm: "
            expect_refused(fn(**kw), code, msg, prefix=prefix, what=(msg, kw))
        assert_nothing_launched(c)
        c.release(xb)


_LAZY = r'''
import torch
from container_engine_accelerators_b200.ops import coll
from tests import coll_rs_rmsnorm_reference as ref
from tests.coll_fp_reference import assert_same
n, s, row_len = 2, 5, 7168
comms = coll.Comm.init_all([0, 0], arena_mb=32)
streams = [torch.cuda.Stream() for _ in comms]
g = torch.Generator().manual_seed(4)
# k_rs_norm<bf16, gather>, k_rs_normq<half, e5m2, scattered>, k_rs_norm<float, scattered>, k_rs_normq<bf16, e4m3, gather>: four different
# kernels of the family, back to back on each rank
plan = [(torch.bfloat16, None, True), (torch.float16, torch.float8_e5m2, False), (torch.float32, None, False), (torch.bfloat16, torch.float8_e4m3fn, True)]
calls = []
for dt, wire, gather in plan:
    xs = [torch.randn(n * s, row_len, generator=g).to(dt) for _ in range(n)]
    shards = [torch.randn(s, row_len, generator=g).to(dt) for _ in range(n)]
    gamma = torch.rand(row_len, generator=g).to(dt)
    o = n * s if gather else s
    new = (lambda c, k, t: c.empty(k, t)) if gather else (lambda c, k, t: torch.empty(k, dtype=t, device="cuda"))
    bufs = []
    for r, c in enumerate(comms):
        x = c.empty(n * s * row_len, dt).view(n * s, row_len)
        x.copy_(xs[r].cuda())
        outs = (new(c, o * row_len, dt).view(o, row_len),) if wire is None else (new(c, o * row_len, wire).view(o, row_len),
                                                                                 new(c, o * row_len // 128, torch.float32).view(o, -1))
        bufs.append((x, shards[r].clone().cuda(), gamma.cuda()) + outs)
    calls.append((xs, shards, gamma, dt, wire, gather, bufs))
torch.cuda.synchronize()
for r, c in enumerate(comms):
    for _, _, _, _, wire, gather, bufs in calls:
        if wire is None:
            c.reduce_scatter_rms_norm(*bufs[r], gather=gather, stream=streams[r])
        else:
            c.reduce_scatter_rms_norm_quantized(*bufs[r], block=128, wire=wire, gather=gather, stream=streams[r])
torch.cuda.synchronize()
for c in comms:
    c.check_async_error()
for xs, shards, gamma, dt, wire, gather, bufs in calls:
    if wire is None:
        want = ref.rs_rms_norm(xs, shards, gamma, 1e-6, dt, gather)
    else:
        want = ref.rs_rms_norm_quantized(xs, shards, gamma, 1e-6, dt, 128, wire, gather)
    for r in range(n):
        for i, (t, w) in enumerate(zip((bufs[r][1],) + tuple(bufs[r][3:]), want[r])):
            assert_same(t.cpu().reshape(-1), w.reshape(-1), f"output {i} rank {r}")
print("lazy ok")
'''


def test_lazy_module_loading_mixed_calls(torch_cuda, coll_lib):
    """A fresh process with lazy module loading and a short watchdog drives two virtual ranks from one thread, each rank enqueueing four
    calls that run four different kernels: the first launch of each must not wait behind the rank's own earlier kernel, which waits at
    its barrier for the other rank's call. The results must be exact."""
    run_python(_LAZY, {"CUDA_MODULE_LOADING": "LAZY", "B200COLL_TIMEOUT_MS": "10000"}, "lazy ok")


@pytest.mark.parametrize("devs,dtype,row_len,extra", [("0", "bfloat16", 7168, []), ("0,0", "half", 4096, ["--rms-norm-gather"]),
                                                      ("0,0", "bfloat16", 4096, ["--rms-norm-quantize", "e5m2:16"]),
                                                      ("0,0,0,0", "float", 8192, ["--rms-norm-gather", "--algo", "oneshot"]),
                                                      ("0,0,0,0", "bfloat16", 16384, ["--rms-norm-gather", "--rms-norm-quantize", "e4m3:128"])])
def test_perf_tool_checks_every_value(torch_cuda, coll_lib, devs, dtype, row_len, extra):
    out = run_perf(["--op", "reduce_scatter", "-d", dtype, "--rms-norm", str(row_len), *extra, "-b", "64K", "-e", "4M", "-f", "4", "-w", "1", "-n", "2",
                    "-c", "1"], devs, env={"B200COLL_TIMEOUT_MS": "20000"})
    assert "op=reduce_scatter + rms-norm" in out, out
    n = len(devs.split(","))
    rows = [l for l in out.splitlines() if l and not l.startswith("#")]
    assert rows and all(l.split()[3] == ("copy" if n == 1 else "twoshot") and int(l.split()[1]) % n == 0 for l in rows), out


def test_multi_gpu_perf_tool_processes_cross_checked(torch_cuda, coll_lib):
    """One process per GPU with B200COLL_CHECK=1: the ranks exchange (rows, row_len, gather), the offsets and (block, wire) before
    every launch, and every value is checked."""
    torch = torch_cuda
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    devs = ",".join(str(i) for i in range(n))
    for extra in ([], ["--rms-norm-gather"], ["--rms-norm-gather", "--rms-norm-quantize", "e4m3:128"]):
        run_perf(["--op", "reduce_scatter", "-d", "bfloat16", "--rms-norm", "8192", *extra, "-b", "1M", "-e", "16M", "-f", "4", "-w", "1", "-n", "3",
                  "-c", "1"], devs, procs=True, env={"B200COLL_CHECK": "1", "B200COLL_TIMEOUT_MS": "20000"}, timeout=300)
