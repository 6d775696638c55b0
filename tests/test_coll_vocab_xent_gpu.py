"""The vocab-parallel cross-entropy (b200collVocabParallelCrossEntropy / ...Backward) on an H100 (`pytest -m gpu`), virtual ranks
sharing cuda:0 unless a test says otherwise. Every result is compared bit for bit with tests/coll_xent_reference.py (NaN by position):
loss and lse on every rank, and every rank's grad."""
import ctypes as C

import numpy as np
import pytest

from container_engine_accelerators_b200.ops.coll import INVALID_ARGUMENT
from tests import coll_xent_reference as ref
from tests.coll_gpu_harness import Group, assert_nothing_launched, coll_mod, expect_refused, poison, torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu

DTS = ["bf16", "f16", "f32"]
_groups = {}


@pytest.fixture(scope="module")
def groups(torch_cuda, coll_mod):
    def get(n):
        if n not in _groups:
            _groups[n] = Group(torch_cuda, coll_mod, n, arena_mb=128)
        return _groups[n]
    yield get
    for g in _groups.values():
        g.destroy()
    _groups.clear()


def tdt(torch, name):
    return {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}[name]


def same_f32(got, want, what):
    got = np.asarray(got, dtype=np.float32)
    want = np.asarray(want, dtype=np.float32)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), f"{what}: NaN positions differ"
    bad = np.nonzero(got.view(np.int32)[~nan] != want.view(np.int32)[~nan])[0]
    assert bad.size == 0, f"{what}: {bad.size} differ, first at {bad[0]}: {got[~nan][bad[0]]!r} vs {want[~nan][bad[0]]!r}"


def same_t(torch, got, want, what):
    iv = {2: torch.int16, 4: torch.int32}[got.element_size()]
    gn, wn = torch.isnan(got.float()), torch.isnan(want.float())
    assert torch.equal(gn, wn), f"{what}: NaN positions differ"
    eq = (got.view(iv) == want.view(iv)) | wn
    assert bool(eq.all()), f"{what}: {int((~eq).sum())} elements differ"


def make_logits(torch, n, rows, vl, dt, seed, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(rows, vl, generator=g) * scale).to(dt) for _ in range(n)]


def run(g, host, target, ignore_index=-100, dloss=None, inplace=False):
    """Forward and backward on every rank from CPU logits `host`; checks loss, lse and grad against the reference. Returns the device
    (loss, lse, grads) per rank."""
    torch, n = g.torch, g.n
    rows, vl = host[0].shape
    xs = [h.cuda() for h in host]
    tg = torch.as_tensor(np.asarray(target, dtype=np.int64)).cuda()
    dl = torch.linspace(0.25, 2.0, rows, device="cuda") if dloss is None else dloss.cuda()
    outs = [None] * n
    torch.cuda.synchronize()
    g.run(lambda r, c, st: outs.__setitem__(r, c.vocab_parallel_cross_entropy(xs[r], tg, ignore_index, stream=st)))
    want_loss, want_lse = ref.forward(host, np.asarray(target), ignore_index)
    for r in range(n):
        same_f32(outs[r][0].cpu().numpy(), want_loss, f"n={n} loss rank {r}")
        same_f32(outs[r][1].cpu().numpy(), want_lse, f"n={n} lse rank {r}")
    grads = [None] * n
    src = [x.clone() for x in xs] if inplace else xs
    g.run(lambda r, c, st: grads.__setitem__(r, c.vocab_parallel_cross_entropy_backward(src[r], tg, outs[r][1], dl, src[r] if inplace else None,
                                                                                        ignore_index, stream=st)))
    for r in range(n):
        want = ref.backward(host[r], r, n, np.asarray(target), want_lse, dl.cpu().numpy(), ignore_index)
        same_t(torch, grads[r].cpu(), want, f"n={n} grad rank {r}")
    return outs, grads


def targets(rng, rows, n, vl, ignore_index=-100):
    t = rng.integers(0, n * vl, rows)
    if rows > 3:
        t[1] = ignore_index
        t[2] = n * vl                    # out of range
        t[3] = -7
    return t


# ------------------------------------------------------------------------------------------------- bit-exact sweeps
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("n", [1, 2, 3, 4, 6, 8])
def test_bit_exact_sweep(groups, n, dt):
    g = groups(n)
    torch = g.torch
    rng = np.random.default_rng(10 * n + DTS.index(dt))
    step = 4 if dt == "f32" else 8
    for vl in sorted({step, 24, 40, 16 * 33 + step, 8008 - 8008 % step, 16040}):   # partial chunks, < and > 512 chunks
        rows = 37
        host = make_logits(torch, n, rows, vl, tdt(torch, dt), seed=vl + n)
        run(g, host, targets(rng, rows, n, vl))


@pytest.mark.parametrize("dt", DTS)
def test_one_rank_large_vocabularies(groups, dt):
    """One rank, Vl from 8 to 151936: rows staged in shared memory and rows read twice from global memory."""
    g = groups(1)
    torch = g.torch
    rng = np.random.default_rng(5)
    for vl in (8, 32000, 100000, 128256, 151936):
        host = make_logits(torch, 1, 9, vl, tdt(torch, dt), seed=vl, scale=6.0)
        run(g, host, targets(rng, 9, 1, vl))


@pytest.mark.parametrize("dt", DTS)
def test_special_values(groups, dt):
    torch = groups(1).torch
    inf, nan = float("inf"), float("nan")
    for n in (1, 2, 4):
        g = groups(n)
        vl, rows = 40, 8
        host = make_logits(torch, n, rows, vl, tdt(torch, dt), seed=n)
        for x in host:
            x[0, 3] = -inf                     # one -inf column
        host[0][1, :] = -inf                   # a whole -inf slice on rank 0
        for x in host:
            x[2, :] = -inf                     # the whole row -inf everywhere
        host[-1][3, 5] = inf                   # +inf
        host[n // 2][4, 7] = nan               # NaN in one slice
        host[0][5, :] = -inf
        host[0][5, 9] = nan                    # NaN in a slice that is otherwise -inf
        host[-1][6, 0] = -0.0
        t = np.arange(rows) * 3 % (n * vl)
        run(g, host, t)
        run(g, host, t, inplace=True)


def test_ignore_index_and_rows_zero(groups):
    torch = groups(1).torch
    for n in (1, 3):
        g = groups(n)
        vl = 64
        host = make_logits(torch, n, 6, vl, torch.bfloat16, seed=9)
        run(g, host, np.array([5, 0, 7, 5, n * vl - 1, 1 << 40]), ignore_index=5)        # an ignore_index inside the vocabulary
        run(g, host, np.array([-1, -1, 3, -1, 2, -1]), ignore_index=-1)
        empty = [torch.zeros(0, vl, dtype=torch.bfloat16) for _ in range(n)]
        before = [c.stats()["kernel_launches"] for c in g.comms]
        run(g, empty, np.zeros(0, dtype=np.int64))
        assert [c.stats()["kernel_launches"] - b for c, b in zip(g.comms, before)] == [1] * n    # the forward launches, the backward not


def test_same_bits_under_launch_shapes_and_repeats(torch_cuda, coll_mod):
    """The result does not depend on the grid: 1, 2, 3 and 7 CTAs per rank, and repeated calls give the same bits."""
    torch = torch_cuda
    rng = np.random.default_rng(3)
    for n in (1, 4):
        host = make_logits(torch, n, 29, 1032, torch.bfloat16, seed=4)
        t = targets(rng, 29, n, 1032)
        first = None
        for ctas in (1, 2, 3, 7, 0):
            with Group(torch, coll_mod, n, arena_mb=32) as g:
                if ctas:
                    for c in g.comms:
                        c.set_launch_shape("p2p", max_ctas=ctas)
                        c.set_max_ctas(ctas)
                for _ in range(2):
                    outs, grads = run(g, host, t)
                    got = [o[0].cpu() for o in outs] + [gr.cpu() for gr in grads]
                    if first is None:
                        first = got
                    for a, b in zip(got, first):
                        assert torch.equal(a.view(torch.int16 if a.element_size() == 2 else torch.int32),
                                           b.view(torch.int16 if b.element_size() == 2 else torch.int32))


# ------------------------------------------------------------------------------------------------- accuracy and training
def test_accuracy_against_torch_cross_entropy(groups):
    """N = 1, fp32 logits: loss within 2e-6 relative and grad within 1e-6 absolute of F.cross_entropy's (the library's exp and log are
    within 1 ulp; the sums are taken in another order)."""
    g = groups(1)
    torch = g.torch
    rows, V = 256, 32000
    gen = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(rows, V, device="cuda", generator=gen) * 4
    t = torch.randint(0, V, (rows,), device="cuda", generator=gen)
    loss, lse = g.comms[0].vocab_parallel_cross_entropy(x, t)
    want = torch.nn.functional.cross_entropy(x.double(), t, reduction="none")
    assert torch.allclose(loss.double(), want, rtol=2e-6, atol=2e-6), (loss.double() - want).abs().max()
    xr = x.clone().requires_grad_()
    torch.nn.functional.cross_entropy(xr, t, reduction="sum").backward()
    grad = g.comms[0].vocab_parallel_cross_entropy_backward(x, t, lse, torch.ones(rows, device="cuda"))
    assert torch.allclose(grad, xr.grad, atol=1e-6), (grad - xr.grad).abs().max()


@pytest.mark.parametrize("n", [2, 4])
def test_tp_training_step(groups, n):
    """A toy LM head [V, H] split by rows over N ranks (column-parallel output layer), trained through the autograd wrapper: the mean
    loss and the head's and the hidden states' gradients match the unsplit torch model."""
    g = groups(n)
    torch = g.torch
    T, H, V = 64, 32, 512
    gen = torch.Generator().manual_seed(n)
    h0 = torch.randn(T, H, generator=gen)
    w0 = torch.randn(V, H, generator=gen) * 0.2
    t = torch.randint(0, V, (T,), generator=gen)
    t[5] = -100
    # the unsplit model in float64
    hr, wr = h0.double().requires_grad_(), w0.double().requires_grad_()
    ref_loss = torch.nn.functional.cross_entropy(hr @ wr.t(), t, ignore_index=-100)
    ref_loss.backward()
    vl = V // n
    hs = [h0.cuda().requires_grad_() for _ in range(n)]
    ws = [w0[r * vl:(r + 1) * vl].cuda().requires_grad_() for r in range(n)]
    tc = t.cuda()
    losses, per_tok, counts, logits = [None] * n, [None] * n, [None] * n, [None] * n

    # Three phases, each over every rank: the local GEMM; the loss, whose kernel waits for every rank; the backward. No kernel a rank
    # enqueues behind its own waiting loss kernel is loaded for the first time before every rank's loss kernel is enqueued (with lazy
    # module loading a first load waits for the kernels already running, which wait for the other ranks).
    def gemm(r, c, st):
        with torch.cuda.stream(st):
            logits[r] = hs[r] @ ws[r].t()                               # [T, V/N], this rank's vocabulary slice
            counts[r] = (tc != -100).sum()

    def loss_fn(r, c, st):
        with torch.cuda.stream(st):
            per_tok[r] = c.vocab_parallel_cross_entropy_loss(logits[r], tc, inplace_backward=r % 2 == 1, stream=st)

    def backward(r, c, st):
        with torch.cuda.stream(st):
            loss = per_tok[r].sum() / counts[r]
            loss.backward()
            losses[r] = loss.detach()
    for phase in (gemm, loss_fn, backward):
        for r, c in enumerate(g.comms):
            with torch.cuda.device(c.device):
                g.streams[r].wait_stream(torch.cuda.current_stream())
                phase(r, c, g.streams[r])
    g.sync()
    g.check_async()
    for r in range(n):
        assert abs(losses[r].item() - ref_loss.item()) < 1e-5, (r, losses[r].item(), ref_loss.item())
        assert torch.allclose(ws[r].grad.cpu().double(), wr.grad[r * vl:(r + 1) * vl], atol=1e-5)
    # the hidden states' gradient is the sum over the ranks' slices (the all-reduce a column-parallel layer's backward makes)
    dh = sum(h.grad.cpu().double() for h in hs)
    assert torch.allclose(dh, hr.grad, atol=1e-5)


def test_past_4_gib(torch_cuda, coll_mod):
    """One bf16 call of 16384 x 151936 (4.6 GiB) at one rank and two: row offsets past 2^32 bytes. Rows at both ends are checked
    against the reference; the backward runs in place."""
    torch = torch_cuda
    rows, vl = 16384, 151936
    need = 2 * rows * vl * 2 + (3 << 30)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB free, {free / 2**30:.1f} GiB free")
    for n in (1, 2):
        with Group(torch, coll_mod, n, arena_mb=64) as g:
            v = vl // n
            gen = torch.Generator(device="cuda").manual_seed(n)
            big = torch.empty(rows, vl, dtype=torch.bfloat16, device="cuda")
            big.normal_(generator=gen).mul_(3)
            xs = [big[:, r * v:(r + 1) * v].contiguous() for r in range(n)] if n > 1 else [big]
            if n > 1:
                del big
            t = torch.randint(0, vl, (rows,), device="cuda", generator=gen)
            outs = [None] * n
            g.run(lambda r, c, st: outs.__setitem__(r, c.vocab_parallel_cross_entropy(xs[r], t, stream=st)))
            pick = list(range(4)) + list(range(rows - 4, rows))
            host = [x[pick].cpu() for x in xs]
            tp = t[pick].cpu().numpy()
            wl, ws = ref.forward(host, tp)
            for r in range(n):
                same_f32(outs[r][0][pick].cpu().numpy(), wl, f"past 4 GiB n={n} loss rank {r}")
                same_f32(outs[r][1][pick].cpu().numpy(), ws, f"past 4 GiB n={n} lse rank {r}")
            dl = torch.ones(rows, device="cuda")
            g.run(lambda r, c, st: c.vocab_parallel_cross_entropy_backward(xs[r], t, outs[r][1], dl, xs[r], stream=st))
            for r in range(n):
                want = ref.backward(host[r], r, n, tp, ws, np.ones(len(pick), np.float32))
                same_t(torch, xs[r][pick].cpu(), want, f"past 4 GiB n={n} grad rank {r}")
            del xs
            torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------- stats, refusals, graphs, mixing
def test_stats(groups):
    torch = groups(1).torch
    for n in (1, 3):
        g = groups(n)
        host = make_logits(torch, n, 10, 64, torch.bfloat16, seed=2)
        before = [c.stats() for c in g.comms]
        run(g, host, np.arange(10))
        algo = "copy" if n == 1 else "twoshot"
        for b, c in zip(before, g.comms):
            a = c.stats()
            assert a["kernel_launches"] - b["kernel_launches"] == 2
            assert a["calls"][0] - b["calls"][0] == 1 and sum(a["calls"]) - sum(b["calls"]) == 1
            assert a["bytes"][0] - b["bytes"][0] == 10 * 16
            assert a["algo_calls"][algo] - b["algo_calls"][algo] == 1


def test_refusals_launch_nothing(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    L = coll.load()
    with Group(torch, coll, 2) as g:
        c = g.comms[0]
        BF16, F32 = coll.torch_dtype_code(torch.bfloat16), coll.torch_dtype_code(torch.float32)
        buf = torch.zeros(1 << 16, dtype=torch.float32, device="cuda")
        p = buf.data_ptr()
        x, t, lo, ls = p, p + 65536, p + 131072, p + 196608

        def fwd(x=x, t=t, lo=lo, ls=ls, rows=4, vl=64, dt=BF16):
            return L.b200collVocabParallelCrossEntropy(x, t, lo, ls, rows, vl, -100, dt, c._h, C.c_void_p(0))

        def bwd(x=x, t=t, ls=ls, dl=lo, gr=p + 131072 + 4096, rows=4, vl=64, dt=BF16):
            return L.b200collVocabParallelCrossEntropyBackward(x, t, ls, dl, gr, rows, vl, -100, dt, c._h, C.c_void_p(0))

        cases = [
            (dict(dt=coll.I32), "dtype must be"), (dict(vl=0), "vocab_local must be positive"), (dict(vl=12), "multiple of 16"),
            (dict(vl=1 << 30), "below 2^31"), (dict(rows=1 << 31), "rows must be below"), (dict(x=0), "null argument"),
            (dict(lo=0), "null argument"), (dict(x=x + 8), "16-byte aligned"), (dict(t=t + 4), "8-byte aligned"),
            (dict(lo=lo + 2), "4-byte aligned"), (dict(lo=x + 64), "must not overlap the inputs"), (dict(ls=lo + 8), "overlap each other"),
            (dict(dt=F32, vl=6), "multiple of 16"),
        ]
        for kw, msg in cases:                                   # one call at a time: each leaves its own last-error message
            expect_refused(fwd(**kw), INVALID_ARGUMENT, msg, prefix="vocab-parallel cross-entropy: ", what=msg)
        bcases = [(dict(gr=x + 16), "must not overlap the inputs"), (dict(gr=ls), "must not overlap the inputs"),
                  (dict(gr=x + 8), "16-byte aligned"), (dict(dl=0), "null argument"), (dict(dt=coll.I32), "dtype must be")]
        for kw, msg in bcases:
            expect_refused(bwd(**kw), INVALID_ARGUMENT, msg, prefix="vocab-parallel cross-entropy backward: ", what=msg)
        assert_nothing_launched(c)


def test_cuda_graph_replay(groups):
    g = groups(3)
    torch, n = g.torch, 3
    rows, vl = 20, 136
    xs = [torch.empty(rows, vl, dtype=torch.bfloat16, device="cuda") for _ in range(n)]
    tg = torch.empty(rows, dtype=torch.int64, device="cuda")
    dl = torch.ones(rows, device="cuda")
    outs = [(torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")) for _ in range(n)]
    grads = [torch.empty_like(x) for x in xs]
    graphs = [torch.cuda.CUDAGraph() for _ in range(n)]
    torch.cuda.synchronize()
    for r, c in enumerate(g.comms):
        with torch.cuda.graph(graphs[r], stream=g.streams[r]):
            c.vocab_parallel_cross_entropy(xs[r], tg, loss=outs[r][0], lse=outs[r][1], stream=g.streams[r])
            c.vocab_parallel_cross_entropy_backward(xs[r], tg, outs[r][1], dl, grads[r], stream=g.streams[r])
    torch.cuda.synchronize()
    rng = np.random.default_rng(0)
    for it in range(3):
        host = make_logits(torch, n, rows, vl, torch.bfloat16, seed=100 + it)
        t = targets(rng, rows, n, vl)
        for x, h in zip(xs, host):
            x.copy_(h)
        tg.copy_(torch.as_tensor(t))
        poison([o for pair in outs for o in pair] + grads)
        torch.cuda.synchronize()
        for r in range(n):
            with torch.cuda.stream(g.streams[r]):
                graphs[r].replay()
        torch.cuda.synchronize()
        g.check_async()
        wl, ws = ref.forward(host, t)
        for r in range(n):
            same_f32(outs[r][0].cpu().numpy(), wl, f"replay {it} loss rank {r}")
            same_f32(outs[r][1].cpu().numpy(), ws, f"replay {it} lse rank {r}")
            same_t(torch, grads[r].cpu(), ref.backward(host[r], r, n, t, ws, np.ones(rows, np.float32)), f"replay {it} grad rank {r}")
    del graphs


def test_back_to_back_without_host_sync(torch_cuda, coll_mod):
    """Three steps on one communicator with no host sync: all_reduce_rms_norm, an FSDP shard gather, a context-parallel gather and the
    cross-entropy forward and backward, ranks launched in a different order every phase."""
    torch, n = torch_cuda, 4
    with Group(torch, coll_mod, n, arena_mb=64, timeout_ms=30000) as g:
        rng = np.random.default_rng(1)
        rows, vl, steps = 24, 200, 3
        hosts = [make_logits(torch, n, rows, vl, torch.bfloat16, seed=50 + s) for s in range(steps)]
        tgs = [targets(rng, rows, n, vl) for _ in range(steps)]
        xs = [[h.cuda() for h in host] for host in hosts]
        tcs = [torch.as_tensor(t).cuda() for t in tgs]
        res = [[None] * n for _ in range(steps)]
        grads = [[None] * n for _ in range(steps)]
        rx = [c.empty(16 * 256, torch.bfloat16).view(16, 256).fill_(0.5) for c in g.comms]
        resid = [torch.zeros(16, 256, dtype=torch.bfloat16, device="cuda") for _ in g.comms]
        gam = torch.ones(256, dtype=torch.bfloat16, device="cuda")
        shards = [torch.full((4, 16), float(r)).cuda() for r in range(n)]
        fulls = [c.empty(16 * 16, torch.bfloat16).view(16, 16) for c in g.comms]
        kv = [torch.full((1, 8, 64), float(r), dtype=torch.bfloat16, device="cuda") for r in range(n)]
        kvf = [c.empty(n * 8 * 64, torch.bfloat16).view(1, n * 8, 64) for c in g.comms]
        dl = torch.ones(rows, device="cuda")
        torch.cuda.synchronize()
        phases = [
            lambda s, r, c, st: c.all_reduce_rms_norm(rx[r], resid[r], gam, stream=st),
            lambda s, r, c, st: res[s].__setitem__(r, c.vocab_parallel_cross_entropy(xs[s][r], tcs[s], stream=st)),
            lambda s, r, c, st: c.all_gather_shards([shards[r]], [fulls[r]], stream=st),
            lambda s, r, c, st: grads[s].__setitem__(r, c.vocab_parallel_cross_entropy_backward(xs[s][r], tcs[s], res[s][r][1], dl, xs[s][r], stream=st)),
            lambda s, r, c, st: c.all_gather_context([kv[r]], [kvf[r]], chunks=1, stream=st),
        ]
        orders = [list(range(n)), list(reversed(range(n))), [2, 0, 3, 1], [1, 3, 0, 2]]
        for s in range(steps):
            for k, ph in enumerate(phases):
                for r in orders[(s + k) % len(orders)]:
                    with torch.cuda.stream(g.streams[r]):
                        ph(s, r, g.comms[r], g.streams[r])
        g.sync()
        g.check_async()
        for s in range(steps):
            wl, ws = ref.forward(hosts[s], tgs[s])
            for r in range(n):
                same_f32(res[s][r][0].cpu().numpy(), wl, f"step {s} loss rank {r}")
                same_t(torch, grads[s][r].cpu(), ref.backward(hosts[s][r], r, n, tgs[s], ws, np.ones(rows, np.float32)),
                       f"step {s} grad rank {r}")
        for r in range(n):
            assert torch.equal(fulls[r].float().cpu(), torch.cat([torch.full((4, 16), float(s)) for s in range(n)]))
            assert torch.equal(kvf[r].float().cpu().view(n, 8, 64)[:, 0, 0], torch.arange(n).float())


def test_multi_gpu(torch_cuda, coll_mod):
    """One rank per visible GPU (two or more): the same bits as the reference."""
    torch = torch_cuda
    n = min(torch.cuda.device_count(), 8)
    if n < 2:
        pytest.skip("needs two or more GPUs")
    with Group(torch, coll_mod, n, devices=list(range(n))) as g:
        rows, vl = 64, 4008
        host = make_logits(torch, n, rows, vl, torch.bfloat16, seed=77)
        t = targets(np.random.default_rng(2), rows, n, vl)
        outs = [None] * n
        xs = [h.to(f"cuda:{c.device}") for h, c in zip(host, g.comms)]
        tg = [torch.as_tensor(t).to(f"cuda:{c.device}") for c in g.comms]
        g.run(lambda r, c, st: outs.__setitem__(r, c.vocab_parallel_cross_entropy(xs[r], tg[r], stream=st)))
        wl, ws = ref.forward(host, t)
        for r in range(n):
            same_f32(outs[r][0].cpu().numpy(), wl, f"multi-GPU loss rank {r}")
            same_f32(outs[r][1].cpu().numpy(), ws, f"multi-GPU lse rank {r}")
