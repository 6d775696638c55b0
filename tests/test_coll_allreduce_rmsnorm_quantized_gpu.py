"""The fused all-reduce, residual add, RMSNorm and FP8 block quantisation on an H100 (`pytest -m gpu`), virtual ranks sharing cuda:0.

Bit-exact means equal (NaN matching NaN at the same position) to tests/coll_rmsnorm_quant_reference.rms_norm_quantized, for the new
residual, q and the scales, on every rank."""
import pytest

from container_engine_accelerators_b200.ops.coll import INVALID_ARGUMENT, INVALID_USAGE
from tests import coll_quant_reference as Q
from tests import coll_rmsnorm_quant_reference as ref
from tests import coll_rmsnorm_reference as R
from tests.coll_fp_reference import assert_same
from tests.coll_gpu_harness import (DTYPES, Group, assert_nothing_launched, coll_mod, expect_refused, poison, run_perf,  # noqa: F401
                                    run_python, torch_cuda)

pytestmark = pytest.mark.gpu

DT_NAMES = ("bf16", "f16", "f32")
WIRES = ("e4m3", "e5m2")


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


def data(torch, n, rows, row_len, dt, seed):
    """Per rank x, one residual, gamma: normal values at a few scales, so sums round and the blocks' amax values differ."""
    g = torch.Generator().manual_seed(seed)
    xs = [(torch.randn(rows, row_len, generator=g) * (0.5 + r)).to(dt) for r in range(n)]
    res = (torch.randn(rows, row_len, generator=g) * 2).to(dt)
    gamma = ((torch.rand(row_len, generator=g) * 2 - 0.5) * torch.exp2(torch.randint(-3, 4, (row_len,), generator=g).float())).to(dt)
    return xs, res, gamma


def run(g, xs, res, gamma, eps, algo, placed, block, wire):
    """One quantised call on every rank. x always in the arena; residual, q and scales in the arena when `placed`, else plain tensors (the
    two-shot fallback). q and scales are poisoned first. Returns [(residual, q, scales)] per rank on the CPU, and the stats before and
    after."""
    torch = g.torch
    rows, row_len = res.shape
    dt = res.dtype
    bases, bufs = [], []

    def arena(c, n, t):
        base = c.empty(max(n, 1), t)
        bases.append((c, base))
        return base[:n]

    for r, c in enumerate(g.comms):
        c.set_algo(algo)
        x = arena(c, rows * row_len, dt).view(rows, row_len)
        x.copy_(xs[r].cuda())
        if placed:
            rd = arena(c, rows * row_len, dt).view(rows, row_len)
            rd.copy_(res.cuda())
            q = arena(c, rows * row_len, wire).view(rows, row_len)
            s = arena(c, rows * (row_len // block), torch.float32).view(rows, row_len // block)
        else:
            rd = res.clone().cuda()
            q = torch.empty(rows, row_len, dtype=wire, device="cuda")
            s = torch.empty(rows, row_len // block, dtype=torch.float32, device="cuda")
        poison([q, s])
        bufs.append((x, rd, q, s))
    gd = gamma.cuda()
    torch.cuda.synchronize()
    before = [c.stats() for c in g.comms]
    g.run(lambda r, c, st: c.all_reduce_rms_norm_quantized(bufs[r][0], bufs[r][1], gd, bufs[r][2], bufs[r][3], block=block, wire=wire, eps=eps,
                                                           stream=st))
    after = [c.stats() for c in g.comms]
    outs = [(rd.cpu(), q.cpu(), s.cpu()) for _, rd, q, s in bufs]
    for c in g.comms:
        c.set_algo("auto")
    for c, base in bases:
        c.release(base)
    return outs, before, after


def check(outs, want, what):
    want_h, want_q, want_s = want
    for r, (h, q, s) in enumerate(outs):
        assert_same(h, want_h, f"{what} residual rank {r}")
        assert_same(q.reshape(-1), want_q.reshape(-1), f"{what} q rank {r}")
        assert_same(s.reshape(-1), want_s.reshape(-1), f"{what} scales rank {r}")


SWEEP = [(1, [0, 1, 5]), (2, [0, 1, 7]), (3, [0, 1, 8]), (4, [0, 1, 10]), (8, [0, 1, 13])]


@pytest.mark.parametrize("dtn", DT_NAMES)
@pytest.mark.parametrize("n,rows_list", SWEEP, ids=[f"n{n}" for n, _ in SWEEP])
def test_bit_exact_sweep(torch_cuda, groups, n, rows_list, dtn):
    torch = torch_cuda
    dt = DTYPES[dtn]
    g = groups(n)
    algos = ("oneshot", "twoshot") if n > 1 else ("auto",)
    es = torch.empty((), dtype=dt).element_size()
    for row_len in (512, 4096, 7168, 16384):
        for rows in rows_list:
            xs, res, gamma = data(torch, n, rows, row_len, dt, seed=rows * 31 + row_len + n)
            for wn in WIRES:
                for block in (16, 128, 512):
                    want = ref.rms_norm_quantized(xs, res, gamma, 1e-6, dt, block, DTYPES[wn])
                    for algo in algos:
                        for placed in ((True, False) if algo == "twoshot" else (True,)):
                            outs, before, after = run(g, xs, res, gamma, 1e-6, algo, placed, block, DTYPES[wn])
                            what = f"n={n} {dtn}->{wn} block={block} rows={rows} row_len={row_len} {algo} placed={placed}"
                            check(outs, want, what)
                            algo_want = "copy" if n == 1 else ("twoshot" if algo == "twoshot" and placed and rows else "oneshot")
                            for b, a in zip(before, after):
                                assert a["algo_calls"][algo_want] == b["algo_calls"][algo_want] + 1, what
                                assert sum(a["algo_calls"].values()) == sum(b["algo_calls"].values()) + 1, what
                                assert a["calls"][0] == b["calls"][0] + 1 and a["bytes"][0] - b["bytes"][0] == rows * row_len * es, what
                                assert a["kernel_launches"] == b["kernel_launches"] + 1, what


@pytest.mark.parametrize("n", [1, 2, 4])
def test_equals_the_wide_call_then_the_quantiser(torch_cuda, groups, n):
    """The header's equivalence: all_reduce_rms_norm, then its out quantised per row by the quantising collectives' rule, gives the fused
    call's bits, and both calls leave the same residual."""
    torch = torch_cuda
    g = groups(n)
    rows, row_len = 9, 7168
    for dtn in DT_NAMES:
        dt = DTYPES[dtn]
        xs, res, gamma = data(torch, n, rows, row_len, dt, seed=40 + n)
        xa = [c.empty(rows * row_len, dt) for c in g.comms]
        wide = []
        for r, c in enumerate(g.comms):
            xa[r].view(rows, row_len).copy_(xs[r].cuda())
            wide.append((res.clone().cuda(), torch.empty(rows, row_len, dtype=dt, device="cuda")))
        gd = gamma.cuda()
        g.run(lambda r, c, st: c.all_reduce_rms_norm(xa[r].view(rows, row_len), wide[r][0], gd, wide[r][1], eps=1e-6, stream=st))
        for c, t in zip(g.comms, xa):
            c.release(t)
        for wn in WIRES:
            for block in (16, 128):
                for algo in (("oneshot", "twoshot") if n > 1 else ("auto",)):
                    outs, _, _ = run(g, xs, res, gamma, 1e-6, algo, True, block, DTYPES[wn])
                    for r, (h, q, s) in enumerate(outs):
                        wh, wo = wide[r][0].cpu(), wide[r][1].cpu()
                        what = f"n={n} {dtn}->{wn} block={block} {algo} rank {r}"
                        assert_same(h, wh, what + " residual")
                        for i in range(rows):
                            cq, cs, _ = Q.quantize(wo[i], block, DTYPES[wn])
                            assert_same(q[i], cq, f"{what} q row {i}")
                            assert_same(s[i], cs, f"{what} scales row {i}")


@pytest.mark.parametrize("n", [1, 2])
def test_special_values(torch_cuda, groups, n):
    torch = torch_cuda
    g = groups(n)
    rows, row_len, block = 6, 512, 128
    for dtn in DT_NAMES:
        dt = DTYPES[dtn]
        xs, res, gamma = data(torch, n, rows, row_len, dt, seed=3)
        xs[0][0, 3] = float("nan")
        xs[-1][1, 300] = float("inf")
        res[2, 40] = float("-inf")
        for t in xs + [res]:
            t[4].zero_()                                              # an all-zero row
        for wn in WIRES:
            for eps in (0.0, 1e-6):
                want = ref.rms_norm_quantized(xs, res, gamma, eps, dt, block, DTYPES[wn])
                for algo in (("oneshot", "twoshot") if n > 1 else ("auto",)):
                    outs, _, _ = run(g, xs, res, gamma, eps, algo, True, block, DTYPES[wn])
                    check(outs, want, f"{dtn}->{wn} eps={eps} {algo}")
                    _, q, s = outs[-1]
                    qf = q.float().view(rows, -1, block)
                    what = (dtn, wn, eps, algo)
                    assert torch.isnan(qf[0]).all() and torch.isnan(s[0]).all(), ("a NaN in h makes the whole row NaN", what)
                    for i, b in ((1, 300 // block), (2, 40 // block)):   # an inf in h: inv = 0, its block NaN, the others +-0 with s = 1
                        nan = torch.zeros(row_len // block, dtype=torch.bool)
                        nan[b] = True
                        assert torch.equal(torch.isnan(qf[i]).all(dim=1), nan) and torch.equal(torch.isnan(s[i]), nan), (i, what)
                        assert (qf[i][~nan] == 0).all() and (s[i][~nan] == 1).all(), (i, what)
                    if eps == 0.0:
                        assert torch.isnan(qf[4]).all() and torch.isnan(s[4]).all(), ("0 / sqrt(0) is NaN", what)
                    else:
                        assert (qf[4] == 0).all() and (s[4] == 1).all(), ("an all-zero row with eps > 0 gives q = 0, s = 1", what)
                    assert not torch.isnan(qf[3]).any() and not torch.isnan(qf[5]).any(), what


@pytest.mark.parametrize("n", [2, 4])
def test_layout_feeds_the_block_scaled_all_gather(torch_cuda, groups, n):
    """q and scales in the arena are a valid input of all_gather_block_scaled(block=(1, block)): every rank receives every rank's
    dequantised rows, float(q) * s (each rank holds the same rows)."""
    torch = torch_cuda
    g = groups(n)
    rows, row_len, dt = 5, 4096, torch.bfloat16
    for wn in WIRES:
        for block in (32, 128):
            xs, res, gamma = data(torch, n, rows, row_len, dt, seed=block + n)
            bases = [(c.empty(rows * row_len, dt), c.empty(rows * row_len, dt), c.empty(rows * row_len, DTYPES[wn]),
                      c.empty(rows * row_len // block, torch.float32)) for c in g.comms]
            xa, rd, qs = ([b[i].view(rows, row_len) for b in bases] for i in range(3))
            ss = [b[3].view(rows, row_len // block) for b in bases]
            outs = [torch.full((n * rows, row_len), float("nan"), device="cuda") for _ in g.comms]
            for r in range(n):
                xa[r].copy_(xs[r].cuda())
                rd[r].copy_(res.cuda())
            gd = gamma.cuda()
            g.run(lambda r, c, st: c.all_reduce_rms_norm_quantized(xa[r], rd[r], gd, qs[r], ss[r], block=block, wire=DTYPES[wn], stream=st))
            g.run(lambda r, c, st: c.all_gather_block_scaled(qs[r], ss[r], outs[r], block=(1, block), stream=st))
            _, wq, wsc = ref.rms_norm_quantized(xs, res, gamma, 1e-6, dt, block, DTYPES[wn])
            deq = (wq.float().view(rows, -1, block) * wsc.view(rows, -1, 1)).reshape(-1)
            want = Q.reduce([deq], 1.0, torch.float32).view(rows, row_len)   # the all-gather's (+0 + v) * scale: -0 comes out as +0
            for r in range(n):
                assert_same(outs[r].cpu(), want.repeat(n, 1), f"{wn} block={block} rank {r}")
            for c, b in zip(g.comms, bases):
                for t in b:
                    c.release(t)


def test_cuda_graph_interleaved(torch_cuda, groups):
    """Capture the quantised call between an all-reduce, the wide call and a quantising all-reduce on the same comms, replay it twice
    with new inputs, and check every result."""
    torch = torch_cuda
    n = 2
    g = groups(n)
    dt, rows, row_len, block, wire = torch.bfloat16, 12, 4096, 128, torch.float8_e4m3fn
    bases = [[c.empty(rows * row_len, dt) for _ in range(4)] + [c.empty(rows * row_len, wire), c.empty(rows * row_len // block, torch.float32),
                                                               c.empty(4096, torch.float32), c.empty(4096, torch.float32)] for c in g.comms]
    xs, rqs, rws, ods = ([b[i].view(rows, row_len) for b in bases] for i in range(4))
    qs, ss = [b[4].view(rows, row_len) for b in bases], [b[5].view(rows, row_len // block) for b in bases]
    ars, aqs = [b[6] for b in bases], [b[7] for b in bases]
    gamma = (torch.rand(row_len) + 0.5).to(dt)
    gd = gamma.cuda()
    for t in aqs:
        t.fill_(0.5)
    graphs = [torch.cuda.CUDAGraph() for _ in g.comms]
    for c in g.comms:
        c.set_algo("auto")
    torch.cuda.synchronize()
    for r, c in enumerate(g.comms):
        with torch.cuda.graph(graphs[r], stream=g.streams[r]):
            c.all_reduce(ars[r], stream=g.streams[r])
            c.all_reduce_rms_norm_quantized(xs[r], rqs[r], gd, qs[r], ss[r], block=block, wire=wire, stream=g.streams[r])
            c.all_reduce_rms_norm(xs[r], rws[r], gd, ods[r], eps=1e-6, stream=g.streams[r])
            c.all_reduce_quantized(aqs[r], stream=g.streams[r])
    torch.cuda.synchronize()
    for it in range(2):
        gen = torch.Generator().manual_seed(100 + it)
        hx = [torch.randn(rows, row_len, generator=gen).to(dt) for _ in range(n)]
        hres = torch.randn(rows, row_len, generator=gen).to(dt)
        har = [torch.randn(4096, generator=gen) for _ in range(n)]
        for r in range(n):
            xs[r].copy_(hx[r].cuda())
            rqs[r].copy_(hres.cuda())
            rws[r].copy_(hres.cuda())
            ars[r].copy_(har[r].cuda())
        torch.cuda.synchronize()
        for r in range(n):
            with torch.cuda.stream(g.streams[r]):                  # each rank's graph on its own stream: the ranks meet inside kernels
                graphs[r].replay()
        torch.cuda.synchronize()
        g.check_async()
        check([(rqs[r].cpu(), qs[r].cpu(), ss[r].cpu()) for r in range(n)], ref.rms_norm_quantized(hx, hres, gamma, 1e-6, dt, block, wire),
              f"replay {it}")
        wh, wo = R.rms_norm(hx, hres, gamma, 1e-6, dt)
        want_ar = (torch.zeros(4096) + har[0]) + har[1]
        for r in range(n):
            assert_same(rws[r].cpu(), wh, f"wide residual replay {it} rank {r}")
            assert_same(ods[r].cpu(), wo, f"wide out replay {it} rank {r}")
            assert torch.equal(ars[r].cpu(), want_ar), f"all_reduce replay {it} rank {r}"
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
        xb = c.empty(4 * 256, dt)
        x = xb.view(4, 256)
        res = torch.zeros(4, 256, dtype=dt, device="cuda")
        gam = torch.ones(256, dtype=dt, device="cuda")
        q = torch.zeros(4, 256, dtype=torch.float8_e4m3fn, device="cuda")
        sc = torch.zeros(4, 2, dtype=torch.float32, device="cuda")
        plain_x = torch.zeros(4, 256, dtype=dt, device="cuda")
        BF16, E4M3, E5M2 = (coll.torch_dtype_code(t) for t in (dt, torch.float8_e4m3fn, torch.float8_e5m2))
        p = lambda t, off=0: C.c_void_p(t.data_ptr() + off)
        f = lambda t, off=0: C.cast(C.c_void_p(t.data_ptr() + off), C.POINTER(C.c_float))
        nul = C.cast(C.c_void_p(0), C.POINTER(C.c_float))
        ok = dict(x=p(x), res=p(res), gam=p(gam), q=p(q), s=f(sc), rows=4, row_len=256, eps=1e-6, dt=BF16, wire=E4M3, block=128)

        def args(**kw):
            a = {**ok, **kw}
            return (a["x"], a["res"], a["gam"], a["q"], a["s"], a["rows"], a["row_len"], a["eps"], a["dt"], a["wire"], a["block"])

        cases = [
            (args(wire=BF16), INVALID_ARGUMENT, "wire_dtype"),
            (args(wire=coll.torch_dtype_code(torch.int8)), INVALID_ARGUMENT, "wire_dtype"),
            (args(block=100), INVALID_ARGUMENT, "block must be"),
            (args(block=8), INVALID_ARGUMENT, "block must be"),
            (args(block=1024), INVALID_ARGUMENT, "block must be"),
            (args(rows=2, row_len=384, block=256), INVALID_ARGUMENT, "multiple of block"),
            (args(dt=E4M3), INVALID_ARGUMENT, "dtype"),
            (args(row_len=0), INVALID_ARGUMENT, "row_len"),
            (args(rows=1, row_len=16384 + 128), INVALID_ARGUMENT, "row_len"),
            (args(eps=-1.0), INVALID_ARGUMENT, "eps"),
            (args(eps=float("nan")), INVALID_ARGUMENT, "eps"),
            (args(rows=1 << 31, row_len=128), INVALID_ARGUMENT, "2^31"),
            (args(q=C.c_void_p(0)), INVALID_ARGUMENT, "null"),
            (args(s=nul), INVALID_ARGUMENT, "null"),
            (args(x=C.c_void_p(0)), INVALID_ARGUMENT, "null"),
            (args(q=p(q, 8)), INVALID_ARGUMENT, "16-byte"),
            (args(res=p(res, 2), rows=3), INVALID_ARGUMENT, "16-byte"),
            (args(s=f(sc, 2)), INVALID_ARGUMENT, "4-byte"),
            (args(q=p(x)), INVALID_ARGUMENT, "q must not overlap"),
            (args(q=p(res, 512), rows=2), INVALID_ARGUMENT, "q must not overlap"),
            (args(q=p(gam), rows=1), INVALID_ARGUMENT, "q must not overlap"),
            (args(s=f(q, 64)), INVALID_ARGUMENT, "q must not overlap"),
            (args(s=f(x, 16)), INVALID_ARGUMENT, "scales must not overlap"),
            (args(s=f(res)), INVALID_ARGUMENT, "scales must not overlap"),
            (args(s=f(gam)), INVALID_ARGUMENT, "scales must not overlap"),
            (args(res=p(x, 256), rows=2), INVALID_ARGUMENT, "residual must not overlap"),
            (args(x=p(plain_x)), INVALID_USAGE, "symmetric arena"),
            (args(x=p(plain_x), wire=E5M2, block=16), INVALID_USAGE, "symmetric arena"),
        ]
        torch.cuda.synchronize()
        for a, code, msg in cases:
            expect_refused(L.b200collAllReduceRmsNormQuantized(*a, c._h, C.c_void_p(0)), code, msg, prefix="quantised all-reduce rms-norm: ",
                           what=(msg, a))
        assert_nothing_launched(c)
        c.release(xb)


_LAZY = r'''
import torch
from container_engine_accelerators_b200.ops import coll
from tests import coll_rmsnorm_quant_reference as ref
from tests import coll_rmsnorm_reference as R
from tests.coll_fp_reference import assert_same
n, rows, row_len = 2, 9, 7168
comms = coll.Comm.init_all([0, 0], arena_mb=32)
streams = [torch.cuda.Stream() for _ in comms]
g = torch.Generator().manual_seed(4)
# twoshot<bf16, e4m3> quantised, twoshot<bf16> wide, oneshot<half, e5m2> quantised (unplaced), oneshot<float> wide (unplaced),
# twoshot<float, e4m3> quantised: five different kernels of the family, back to back on each rank
plan = [(torch.bfloat16, torch.float8_e4m3fn, True), (torch.bfloat16, None, True), (torch.float16, torch.float8_e5m2, False), (torch.float32, None, False),
        (torch.float32, torch.float8_e4m3fn, True)]
calls = []
for dt, wire, placed in plan:
    xs = [torch.randn(rows, row_len, generator=g).to(dt) for _ in range(n)]
    res = torch.randn(rows, row_len, generator=g).to(dt)
    gamma = torch.rand(row_len, generator=g).to(dt)
    new = (lambda c, k, t: c.empty(k, t)) if placed else (lambda c, k, t: torch.empty(k, dtype=t, device="cuda"))
    bufs = []
    for r, c in enumerate(comms):
        x = c.empty(rows * row_len, dt).view(rows, row_len)
        x.copy_(xs[r].cuda())
        rd = new(c, rows * row_len, dt).view(rows, row_len)
        rd.copy_(res.cuda())
        if wire is None:
            bufs.append((x, rd, gamma.cuda(), new(c, rows * row_len, dt).view(rows, row_len)))
        else:
            bufs.append((x, rd, gamma.cuda(), new(c, rows * row_len, wire).view(rows, row_len), new(c, rows * row_len // 128, torch.float32).view(rows, -1)))
    calls.append((xs, res, gamma, dt, wire, bufs))
for c in comms:
    c.set_algo("twoshot")
torch.cuda.synchronize()
for r, c in enumerate(comms):
    for _, _, _, _, wire, bufs in calls:
        if wire is None:
            c.all_reduce_rms_norm(*bufs[r], stream=streams[r])
        else:
            c.all_reduce_rms_norm_quantized(*bufs[r], block=128, wire=wire, stream=streams[r])
torch.cuda.synchronize()
for c in comms:
    c.check_async_error()
for xs, res, gamma, dt, wire, bufs in calls:
    if wire is None:
        want = R.rms_norm(xs, res, gamma, 1e-6, dt)
    else:
        want = ref.rms_norm_quantized(xs, res, gamma, 1e-6, dt, 128, wire)
    for r in range(n):
        got = (bufs[r][1],) + tuple(bufs[r][3:])                   # residual, then out or (q, scales)
        for i, (t, w) in enumerate(zip(got, want)):
            assert_same(t.cpu().reshape(-1), w.reshape(-1), f"output {i} rank {r}")
print("lazy ok")
'''


def test_lazy_module_loading_mixed_calls(torch_cuda, coll_lib):
    """A fresh process with lazy module loading and a short watchdog drives two virtual ranks from one thread, each rank enqueueing five
    calls, wide and quantised, that run five different kernels: the first launch of each must not wait behind the rank's own earlier
    kernel, which waits at its barrier for the other rank's call. The results must be exact."""
    run_python(_LAZY, {"CUDA_MODULE_LOADING": "LAZY", "B200COLL_TIMEOUT_MS": "10000"}, "lazy ok")


@pytest.mark.parametrize("devs,dtype,row_len,wq,algo", [("0", "bfloat16", 7168, "e4m3:128", "auto"), ("0,0", "half", 4096, "e5m2:16", "auto"),
                                                        ("0,0,0", "float", 8192, "e4m3:512", "oneshot"),
                                                        ("0,0,0,0", "bfloat16", 16384, "e4m3:128", "twoshot")])
def test_perf_tool_checks_every_value(torch_cuda, coll_lib, devs, dtype, row_len, wq, algo):
    out = run_perf(["--op", "all_reduce", "-d", dtype, "--rms-norm", str(row_len), "--rms-norm-quantize", wq, "--algo", algo, "-b", "64K", "-e", "4M",
                    "-f", "4", "-w", "1", "-n", "2", "-c", "1"], devs, env={"B200COLL_TIMEOUT_MS": "20000"})
    assert "op=all_reduce + rms-norm + quantize" in out, out
    if algo != "auto":
        rows = [l for l in out.splitlines() if l and not l.startswith("#")]
        assert rows and all(l.split()[3] == algo for l in rows), out
