"""The fused all-reduce, residual add and RMSNorm on an H100 (`pytest -m gpu`), virtual ranks sharing cuda:0.

Bit-exact means equal (NaN matching NaN at the same position) to tests/coll_rmsnorm_reference.rms_norm, for both the new residual and
out, on every rank."""
import pytest

from container_engine_accelerators_b200.ops.coll import INVALID_ARGUMENT, INVALID_USAGE
from tests import coll_rmsnorm_reference as ref
from tests.coll_fp_reference import assert_same
from tests.coll_gpu_harness import DTYPES, Group, coll_mod, expect_refused, run_perf, run_python, torch_cuda  # noqa: F401

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


def data(torch, n, rows, row_len, dt, seed):
    """Per rank x, one residual, gamma: normal values at a few scales, so sums round and the fold sees a spread of magnitudes."""
    g = torch.Generator().manual_seed(seed)
    xs = [(torch.randn(rows, row_len, generator=g) * (0.5 + r)).to(dt) for r in range(n)]
    res = (torch.randn(rows, row_len, generator=g) * 2).to(dt)
    gamma = (torch.rand(row_len, generator=g) * 2 - 0.5).to(dt)
    return xs, res, gamma


def run(g, xs, res, gamma, eps, algo, placed):
    """One call on every rank. x always in the arena; residual and out in the arena when `placed`, else plain tensors (the two-shot
    fallback). out is poisoned with NaN. Returns [(residual, out)] per rank on the CPU, and the stats before and after."""
    torch = g.torch
    rows, row_len = res.shape
    dt = res.dtype
    bufs, bases = [], []
    numel = max(rows * row_len, 1)

    def arena(c):
        base = c.empty(numel, dt)
        bases.append((c, base))
        return base[:rows * row_len].view(rows, row_len)

    for r, c in enumerate(g.comms):
        c.set_algo(algo)
        x = arena(c)
        x.copy_(xs[r].cuda())
        if placed:
            rd, od = arena(c), arena(c)
            rd.copy_(res.cuda())
            od.fill_(float("nan"))
        else:
            rd = res.clone().cuda()
            od = torch.full((rows, row_len), float("nan"), dtype=dt, device="cuda")
        bufs.append((x, rd, od, gamma.cuda()))
    torch.cuda.synchronize()
    before = [c.stats() for c in g.comms]
    for r, c in enumerate(g.comms):
        x, rd, od, gd = bufs[r]
        c.all_reduce_rms_norm(x, rd, gd, od, eps=eps, stream=g.streams[r])
    torch.cuda.synchronize()
    for c in g.comms:
        c.check_async_error()
    after = [c.stats() for c in g.comms]
    outs = [(rd.cpu(), od.cpu()) for _, rd, od, _ in bufs]
    for c in g.comms:
        c.set_algo("auto")
    for c, base in bases:
        c.release(base)
    return outs, before, after


def check(outs, xs, res, gamma, eps, what):
    want_h, want_o = ref.rms_norm(xs, res, gamma, eps, res.dtype)
    for r, (h, o) in enumerate(outs):
        assert_same(h, want_h, f"{what} residual rank {r}")
        assert_same(o, want_o, f"{what} out rank {r}")


SWEEP = [(1, [0, 1, 5]), (2, [0, 1, 7]), (3, [0, 1, 8]), (4, [0, 1, 10]), (8, [0, 1, 13])]


@pytest.mark.parametrize("dtn", DT_NAMES)
@pytest.mark.parametrize("n,rows_list", SWEEP, ids=[f"n{n}" for n, _ in SWEEP])
def test_bit_exact_sweep(torch_cuda, groups, n, rows_list, dtn):
    torch = torch_cuda
    dt = DTYPES[dtn]
    g = groups(n)
    algos = ("oneshot", "twoshot") if n > 1 else ("auto",)
    for row_len in (16, 4096, 7168, 16384):
        for rows in rows_list:
            xs, res, gamma = data(torch, n, rows, row_len, dt, seed=rows * 31 + row_len + n)
            for algo in algos:
                for placed in ((True, False) if algo == "twoshot" else (True,)):
                    outs, before, after = run(g, xs, res, gamma, 1e-6, algo, placed)
                    what = f"n={n} {dtn} rows={rows} row_len={row_len} {algo} placed={placed}"
                    check(outs, xs, res, gamma, 1e-6, what)
                    want = "copy" if n == 1 else ("twoshot" if algo == "twoshot" and placed and rows else "oneshot")
                    es = torch.empty((), dtype=dt).element_size()
                    for b, a in zip(before, after):
                        assert a["algo_calls"][want] == b["algo_calls"][want] + 1, what
                        assert a["calls"][0] == b["calls"][0] + 1 and a["bytes"][0] - b["bytes"][0] == rows * row_len * es, what
                        assert a["kernel_launches"] == b["kernel_launches"] + 1, what


@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_algorithm_independence(torch_cuda, groups, n):
    torch = torch_cuda
    g = groups(n)
    for dtn in DT_NAMES:
        xs, res, gamma = data(torch, n, 37, 7168, DTYPES[dtn], seed=n)
        one, _, _ = run(g, xs, res, gamma, 1e-5, "oneshot", True)
        two, _, _ = run(g, xs, res, gamma, 1e-5, "twoshot", True)
        for r in range(n):
            assert_same(one[r][0], two[r][0], f"{dtn} residual rank {r}")
            assert_same(one[r][1], two[r][1], f"{dtn} out rank {r}")


@pytest.mark.parametrize("n", [1, 2, 4])
def test_agrees_with_pytorch(torch_cuda, groups, n):
    """Within 2 ulp of dtype (bf16, fp16) of an fp32 PyTorch computation: catches a reference that is wrong the same way as the kernel.
    fp32 out: within 8 ulp, because there both the contract's arithmetic (inv rounded, then two rounded products) and PyTorch's fp32
    rms_norm lie about 3 fp32 ulp from the exact value, in different directions."""
    import torch.nn.functional as F
    torch = torch_cuda
    g = groups(n)
    for dtn in DT_NAMES:
        dt = DTYPES[dtn]
        for row_len in (4096, 7168):
            xs, res, gamma = data(torch, n, 64, row_len, dt, seed=7 + n)
            outs, _, _ = run(g, xs, res, gamma, 1e-6, "auto", True)
            h = (sum(x.float() for x in xs) + res.float()).to(dt)
            y = F.rms_norm(h.float(), (row_len,), gamma.float(), 1e-6).to(dt)
            bits, tiny, k = {torch.bfloat16: (8, 2.0 ** -133, 2), torch.float16: (11, 2.0 ** -24, 2), torch.float32: (24, 2.0 ** -149, 8)}[dt]
            _, e = torch.frexp(y.float())
            tol = torch.clamp(k * torch.ldexp(torch.ones_like(y, dtype=torch.float32), e - bits), min=k * tiny)   # k ulp of y in dtype
            for r, (hr, o) in enumerate(outs):
                assert torch.equal(hr, h), f"{dtn} residual rank {r}"
                assert ((o.float() - y.float()).abs() <= tol).all(), f"{dtn} out rank {r} {row_len}"


@pytest.mark.parametrize("n", [1, 2])
def test_special_values(torch_cuda, groups, n):
    torch = torch_cuda
    g = groups(n)
    for dtn in DT_NAMES:
        dt = DTYPES[dtn]
        xs, res, gamma = data(torch, n, 6, 64, dt, seed=3)
        xs[0][0, 3] = float("nan")
        xs[-1][1, 17] = float("inf")
        res[2, 40] = float("-inf")
        res[3, 0] = float("nan")
        for t in xs + [res]:
            t[4].zero_()                                              # an all-zero row
        for eps in (0.0, 1e-6):
            for algo in (("oneshot", "twoshot") if n > 1 else ("auto",)):
                outs, _, _ = run(g, xs, res, gamma, eps, algo, True)
                check(outs, xs, res, gamma, eps, f"{dtn} eps={eps} {algo}")
                o = outs[0][1].float()
                assert torch.isnan(o[0]).all() and torch.isnan(o[3]).all(), "a NaN in a row makes the whole row NaN"
                if eps == 0.0:
                    assert torch.isnan(o[4]).all(), "0 / sqrt(0) is NaN"
                else:
                    assert (o[4] == 0).all(), "an all-zero row with eps > 0 gives zeros"


@pytest.mark.parametrize("n", [2])
def test_cuda_graph_interleaved(torch_cuda, coll_mod, groups, n):
    """Capture the fused call between an all-reduce, a quantising all-reduce and an expert dispatch on the same comms, replay it twice
    with new inputs, and check every result."""
    torch, coll = torch_cuda, coll_mod
    g = groups(n)
    dt, rows, row_len, E, tokens, k = torch.bfloat16, 12, 4096, 4, 8, 2
    bases = [[c.empty(rows * row_len, dt) for _ in range(3)] + [c.empty(4096, torch.float32), c.empty(4096, torch.float32),
                                                               c.empty(tokens * k * n * 256, dt)] for c in g.comms]
    xs, rds, ods = ([b[i].view(rows, row_len) for b in bases] for i in range(3))
    ars, qs = [b[3] for b in bases], [b[4] for b in bases]
    recv = [b[5].view(-1, 256) for b in bases]
    dx = [torch.randn(tokens, 256, device="cuda").to(dt) for _ in g.comms]
    ids = [torch.randint(0, E, (tokens, k), dtype=torch.int32, device="cuda") for _ in g.comms]
    small = [(torch.empty(E // n, dtype=torch.int32, device="cuda"), torch.empty(tokens, k, dtype=torch.int32, device="cuda"),
              torch.empty(1, dtype=torch.int32, device="cuda")) for _ in g.comms]
    gamma = (torch.rand(row_len) + 0.5).to(dt)
    gd = gamma.cuda()
    graphs = [torch.cuda.CUDAGraph() for _ in g.comms]
    for c in g.comms:
        c.set_algo("auto")
    torch.cuda.synchronize()
    for r, c in enumerate(g.comms):
        with torch.cuda.graph(graphs[r], stream=g.streams[r]):
            c.all_reduce(ars[r], stream=g.streams[r])
            c.all_reduce_rms_norm(xs[r], rds[r], gd, ods[r], eps=1e-6, stream=g.streams[r])
            c.all_reduce_quantized(qs[r], stream=g.streams[r])
            c.expert_dispatch(dx[r], ids[r], E, recv[r], *small[r], stream=g.streams[r])
    torch.cuda.synchronize()
    for it in range(2):
        gen = torch.Generator().manual_seed(100 + it)
        hx = [(torch.randn(rows, row_len, generator=gen)).to(dt) for _ in range(n)]
        hres = torch.randn(rows, row_len, generator=gen).to(dt)
        har = [torch.randn(4096, generator=gen) for _ in range(n)]
        for r in range(n):
            xs[r].copy_(hx[r].cuda())
            rds[r].copy_(hres.cuda())
            ars[r].copy_(har[r].cuda())
        torch.cuda.synchronize()
        for r in range(n):
            with torch.cuda.stream(g.streams[r]):                  # each rank's graph on its own stream: the ranks meet inside kernels
                graphs[r].replay()
        torch.cuda.synchronize()
        for c in g.comms:
            c.check_async_error()
        check([(rds[r].cpu(), ods[r].cpu()) for r in range(n)], hx, hres, gamma, 1e-6, f"replay {it}")
        want = (((torch.zeros(4096) + har[0]) + har[1]))
        for r in range(n):
            assert torch.equal(ars[r].cpu(), want), f"all_reduce replay {it} rank {r}"
    del graphs
    torch.cuda.synchronize()
    for c, b in zip(g.comms, bases):
        for t in b:
            c.release(t)


def test_refusals_launch_nothing(torch_cuda, coll_mod, groups):
    torch, coll = torch_cuda, coll_mod
    L = coll.load()
    import ctypes as C
    g = groups(2)
    c = g.comms[0]
    dt = torch.bfloat16
    xb = c.empty(4 * 64, dt)
    x = xb.view(4, 64)
    res = torch.zeros(4, 64, dtype=dt, device="cuda")
    out = torch.zeros(4, 64, dtype=dt, device="cuda")
    gam = torch.ones(64, dtype=dt, device="cuda")
    plain_x = torch.zeros(4, 64, dtype=dt, device="cuda")
    BF16 = coll.torch_dtype_code(dt)
    p = lambda t, off=0: C.c_void_p(t.data_ptr() + off)
    cases = [
        ((p(x), p(res), p(gam), p(out), 4, 64, 1e-6, coll.torch_dtype_code(torch.float8_e4m3fn)), INVALID_ARGUMENT),
        ((p(x), p(res), p(gam), p(out), 4, 72, 1e-6, BF16), INVALID_ARGUMENT),
        ((p(x), p(res), p(gam), p(out), 4, 0, 1e-6, BF16), INVALID_ARGUMENT),
        ((p(x), p(res), p(gam), p(out), 1, 16384 + 16, 1e-6, BF16), INVALID_ARGUMENT),
        ((p(x), p(res), p(gam), p(out), 4, 64, -1.0, BF16), INVALID_ARGUMENT),
        ((p(x), p(res), p(gam), p(out), 4, 64, float("nan"), BF16), INVALID_ARGUMENT),
        ((p(x), p(res), p(gam), p(out), 4, 64, float("inf"), BF16), INVALID_ARGUMENT),
        ((C.c_void_p(0), p(res), p(gam), p(out), 4, 64, 1e-6, BF16), INVALID_ARGUMENT),
        ((p(x), p(res, 2), p(gam), p(out), 3, 64, 1e-6, BF16), INVALID_ARGUMENT),
        ((p(x), p(res), p(gam), p(res, 128), 2, 64, 1e-6, BF16), INVALID_ARGUMENT),
        ((p(x), p(res), p(res), p(out), 4, 64, 1e-6, BF16), INVALID_ARGUMENT),
        ((p(x), p(x, 128), p(gam), p(out), 2, 64, 1e-6, BF16), INVALID_ARGUMENT),
        ((p(x), p(res), p(gam), p(out), 1 << 31, 16, 1e-6, BF16), INVALID_ARGUMENT),
        ((p(plain_x), p(res), p(gam), p(out), 4, 64, 1e-6, BF16), INVALID_USAGE),
    ]
    torch.cuda.synchronize()
    for args, code in cases:
        before = c.stats()
        expect_refused(L.b200collAllReduceRmsNorm(*args, c._h, C.c_void_p(0)), code, what=args)
        after = c.stats()
        assert after["kernel_launches"] == before["kernel_launches"] and after["calls"] == before["calls"], args
    c.release(xb)


_LAZY = r'''
import torch
from container_engine_accelerators_b200.ops import coll
from tests import coll_rmsnorm_reference as ref
from tests.coll_fp_reference import assert_same
n, rows, row_len = 2, 9, 7168
comms = coll.Comm.init_all([0, 0], arena_mb=32)
streams = [torch.cuda.Stream() for _ in comms]
g = torch.Generator().manual_seed(4)
calls = []
for dt, placed in ((torch.bfloat16, False), (torch.float32, True), (torch.float16, False)):     # oneshot<bf16>, twoshot<float>, oneshot<half>
    xs = [torch.randn(rows, row_len, generator=g).to(dt) for _ in range(n)]
    res = torch.randn(rows, row_len, generator=g).to(dt)
    gamma = torch.rand(row_len, generator=g).to(dt)
    bufs = []
    for r, c in enumerate(comms):
        x = c.empty(rows * row_len, dt).view(rows, row_len)
        x.copy_(xs[r].cuda())
        rd = c.empty(rows * row_len, dt).view(rows, row_len) if placed else torch.empty(rows, row_len, dtype=dt, device="cuda")
        od = c.empty(rows * row_len, dt).view(rows, row_len) if placed else torch.empty(rows, row_len, dtype=dt, device="cuda")
        rd.copy_(res.cuda())
        bufs.append((x, rd, gamma.cuda(), od))                   # all_reduce_rms_norm's argument order
    calls.append((xs, res, gamma, dt, bufs))
for c in comms:
    c.set_algo("twoshot")
torch.cuda.synchronize()
for r, c in enumerate(comms):                     # per rank, back to back: three calls, three different kernels of this family
    for _, _, _, _, bufs in calls:
        c.all_reduce_rms_norm(*bufs[r], stream=streams[r])
torch.cuda.synchronize()
for c in comms:
    c.check_async_error()
for xs, res, gamma, dt, bufs in calls:
    h, o = ref.rms_norm(xs, res, gamma, 1e-6, dt)
    for r in range(n):
        assert_same(bufs[r][1].cpu(), h, f"residual {r}")
        assert_same(bufs[r][3].cpu(), o, f"out {r}")
print("lazy ok")
'''


def test_lazy_module_loading_rms_norm(torch_cuda, coll_lib):
    """A fresh process with lazy module loading and a short watchdog drives two virtual ranks from one thread, each rank enqueueing three
    fused calls that run three different kernels: the first launch of the second and third must not wait behind the rank's own first
    kernel, which waits at its barrier for the other rank's call. The results must be exact."""
    run_python(_LAZY, {"CUDA_MODULE_LOADING": "LAZY", "B200COLL_TIMEOUT_MS": "10000"}, "lazy ok")


@pytest.mark.parametrize("devs,dtype,row_len", [("0", "bfloat16", 8192), ("0,0", "half", 7168), ("0,0,0", "float", 4096)])
def test_perf_tool_checks_every_value(torch_cuda, coll_lib, devs, dtype, row_len):
    out = run_perf(["--op", "all_reduce", "-d", dtype, "--rms-norm", str(row_len), "-b", "64K", "-e", "4M", "-f", "4", "-w", "1", "-n", "2", "-c", "1"],
                   devs, env={"B200COLL_TIMEOUT_MS": "20000"})
    assert "op=all_reduce + rms-norm" in out, out
