"""The vocab-parallel embedding (b200collVocabParallelEmbedding / ...Backward) on an H100 (`pytest -m gpu`), virtual ranks sharing
cuda:0. Every forward is compared bit for bit with tests/coll_embedding_reference.py and every backward bit for bit as well (NaN by
position), at 1 to 8 ranks, tensor- and sequence-parallel."""
import numpy as np
import pytest

from tests import coll_embedding_reference as ref
from tests import coll_xent_reference as xref
from tests.coll_gpu_harness import Group, coll_mod, poison, torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu

DTS = ["bf16", "f16", "f32"]
_groups = {}


@pytest.fixture(scope="module")
def groups(torch_cuda, coll_mod):
    def get(n):
        if n not in _groups:
            _groups[n] = Group(torch_cuda, coll_mod, n, arena_mb=512)
        return _groups[n]
    yield get
    for g in _groups.values():
        g.destroy()
    _groups.clear()


def tdt(torch, name):
    return {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}[name]


def arena(c, shape, dtype):
    """An arena tensor of `shape` that Comm.release accepts (a view of Comm.empty's tensor, its allocation carried over)."""
    base = c.empty(int(np.prod(shape)), dtype)
    v = base.view(shape)
    v._b200coll_buf = base._b200coll_buf
    return v


def ivt(torch, name):
    return torch.int16 if name != "f32" else torch.int32


def to_dev(g, c, bits, dt, in_arena):
    """Raw bits (numpy) as a device tensor of dtype dt, in c's arena when `in_arena`."""
    torch = g.torch
    t = torch.from_numpy(bits.view(np.int16 if dt != "f32" else np.int32).copy()).view(tdt(torch, dt))
    if not in_arena or t.numel() == 0:           # an empty sequence-parallel shard is never read
        return t.cuda()
    a = arena(c, t.shape, t.dtype)
    a.copy_(t)
    return a


def bits_of(t, dt):
    return t.cpu().view(ivt(__import__("torch"), dt)).numpy().view(np.uint16 if dt != "f32" else np.uint32)


def same_bits(got, want, dt, what):
    gn, wn = np.isnan(ref.widen(got, dt)), np.isnan(ref.widen(want, dt))
    assert np.array_equal(gn, wn), f"{what}: NaN positions differ"
    bad = np.nonzero((got != want) & ~wn)
    assert bad[0].size == 0, f"{what}: {bad[0].size} differ, first at {tuple(b[0] for b in bad)}"


def rand_bits(rng, shape, dt, scale=2.0):
    return ref.narrow((rng.standard_normal(shape) * scale).astype(np.float32), dt)


def run(g, dt, ids, vl, h, sp=False, wdt=None, accumulate=False, seed=0, tables=None, dout=None):
    """Forward and backward on every rank; both checked bit for bit against the reference."""
    torch, n = g.torch, g.n
    wdt = wdt or dt
    rng = np.random.default_rng(seed)
    ids = np.asarray(ids, dtype=np.int64)
    T = ids.shape[0]
    on_arena = n > 1
    tables = tables if tables is not None else [rand_bits(rng, (vl, h), dt) for _ in range(n)]
    ws = [to_dev(g, c, tables[r], dt, on_arena) for r, c in enumerate(g.comms)]
    idd = torch.from_numpy(ids).cuda()
    nr = T // n if sp else T
    outs = [torch.empty((nr, h), dtype=tdt(torch, dt), device="cuda") for _ in range(n)]
    poison(outs)
    torch.cuda.synchronize()
    g.run(lambda r, c, st: c.vocab_parallel_embedding(idd, ws[r], sequence_parallel=sp, out=outs[r], stream=st))
    for r in range(n):
        got, want = bits_of(outs[r], dt), ref.forward(tables, ids, sp, r)
        assert np.array_equal(got, want), f"n={n} forward rank {r}: {int((got != want).sum())} bit patterns differ"   # NaN payloads too
    dout = dout if dout is not None else rand_bits(rng, (T, h), dt)
    if sp:
        gos = [to_dev(g, c, dout[r * nr:(r + 1) * nr], dt, on_arena) for r, c in enumerate(g.comms)]
    else:
        d = to_dev(g, None, dout, dt, False)
        gos = [d] * n
    olds = [rand_bits(rng, (vl, h), wdt) for _ in range(n)]
    dws = [to_dev(g, None, olds[r], wdt, False) for r in range(n)]
    if not accumulate:
        poison(dws)
    torch.cuda.synchronize()
    g.run(lambda r, c, st: c.vocab_parallel_embedding_backward(idd, gos[r], dws[r], sequence_parallel=sp, accumulate=accumulate, stream=st))
    for r in range(n):
        want = ref.backward(ids, dout, dt, r, n, vl, wdt, olds[r] if accumulate else None)
        same_bits(bits_of(dws[r], wdt), want, wdt, f"n={n} backward rank {r} sp={sp} acc={accumulate}")
    if on_arena:
        for r, c in enumerate(g.comms):
            c.release(ws[r])
            if sp and getattr(gos[r], "_b200coll_buf", None) is not None:
                c.release(gos[r])
    return outs, dws


def id_sets(rng, T, n, vl):
    nv = n * vl
    zipf = np.minimum(rng.zipf(1.3, T) - 1, nv - 1)
    sets = {
        "uniform": rng.integers(0, nv, T),
        "zipf": zipf,
        "same": np.full(T, min(3, nv - 1)),
        "out_of_range": rng.integers(nv, nv + 100, T),
        "negative": -rng.integers(1, 50, T),
        "mixed_edges": rng.choice(np.array([-1, 0, nv - 1, nv, vl, vl - 1]), T),
    }
    return sets


# ------------------------------------------------------------------------------------------------- bit-exact sweeps
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("n", [1, 2, 3, 4, 6, 8])
def test_bit_exact_sweep(groups, n, dt):
    g = groups(n)
    rng = np.random.default_rng(10 * n + DTS.index(dt))
    es = 2 if dt != "f32" else 4
    shapes = [(37 * n, 5, 16 // es), (2049 * n, 300, 64), (6000 // n * n, 1, 8 * (8 // es)), (n, 7, 256 // es)]
    for k, (T, vl, h) in enumerate(shapes):
        sets = list(id_sets(rng, T, n, vl).items())
        for name, ids in sets[k % 2::2] if T > n else sets:            # every distribution at two shapes, all at T == N
            sp = bool(rng.integers(0, 2))
            wdt = "f32" if rng.integers(0, 2) else dt
            run(g, dt, ids, vl, h, sp=sp, wdt=wdt, accumulate=bool(rng.integers(0, 2)), seed=T + vl)


@pytest.mark.parametrize("n", [1, 2, 4, 8])
def test_every_mode(groups, n):
    """TP and SP, dweight fp32 and in dout's dtype, accumulate on and off, at one shape with repeated ids."""
    g = groups(n)
    rng = np.random.default_rng(n)
    for dt in DTS:
        T, vl, h = 4104 // n * n, 97, 96
        ids = rng.integers(-5, n * vl + 5, T)
        for sp in (False, True):
            for wdt in sorted({dt, "f32"}):
                for acc in (False, True):
                    run(g, dt, ids, vl, h, sp=sp, wdt=wdt, accumulate=acc, seed=int(rng.integers(1 << 30)))


def test_empty_and_one_token(groups):
    for n in (1, 2, 4):
        g = groups(n)
        for sp in (False, True):
            run(g, "bf16", np.zeros(0, dtype=np.int64), 4, 8, sp=sp, wdt="f32")
            run(g, "bf16", np.zeros(0, dtype=np.int64), 4, 8, sp=sp, wdt="f32", accumulate=True)
        run(g, "f32", np.array([n * 4 - 1]), 4, 4, wdt="f32")
        run(g, "bf16", np.arange(n) * 4 + 3, 4, 8, sp=True)


@pytest.mark.parametrize("dt", DTS)
def test_large_vocabularies_and_hidden(groups, dt):
    """One rank up to Vl = 151936 (three sort passes), H up to 8192, T not a multiple of the 2048-token tile; two ranks at Vl = 75968."""
    rng = np.random.default_rng(3)
    es = 2 if dt != "f32" else 4
    for n, vl, h, T in ((1, 151936, 64, 5000), (1, 128256, 32 // es * 8, 700), (1, 2048, 8192, 700), (2, 75968, 128, 4099), (1, 256, 16 // es * 4, 70001)):
        g = groups(n)
        ids = rng.integers(-10, n * vl + 10, T)
        ids[: T // 3] = rng.integers(0, 40, T // 3)          # repeated rows
        run(g, dt, ids, vl, h, sp=False, wdt="f32", seed=vl)


def test_special_values(groups):
    inf, nan = np.float32("inf"), np.float32("nan")
    for dt in DTS:
        for n in (1, 2, 4):
            g = groups(n)
            rng = np.random.default_rng(4)
            vl, h = 6, 64
            vals = np.array([0.0, -0.0, inf, -inf, nan, 1.0, -1.0, 65504.0], dtype=np.float32)
            tables = [ref.narrow(rng.choice(vals, (vl, h)), dt) for _ in range(n)]
            if dt == "f32":
                tables[0][0, 0] = 0x7FC12345                     # a NaN payload survives the forward bit copy
            else:
                tables[0][0, 0] = 0x7F95 if dt == "bf16" else 0x7E55           # non-canonical NaNs (exponent all ones, payload set)
            T = 40 * n
            ids = rng.integers(0, n * vl, T)
            ids[0] = 0
            dout = ref.narrow(rng.choice(vals, (T, h)), dt)
            for sp in (False, True):
                for wdt in sorted({dt, "f32"}):
                    run(g, dt, ids, vl, h, sp=sp, wdt=wdt, tables=tables, dout=dout)


# ------------------------------------------------------------------------------------------------- agreement with torch
def test_agrees_with_torch_and_megatron(groups):
    torch = groups(1).torch
    F = torch.nn.functional
    for n in (1, 2, 4):
        g = groups(n)
        vl, h, T = 50, 128, 512
        full = torch.randn(n * vl, h).to(torch.bfloat16)
        ids = torch.randint(0, n * vl, (T,))
        ids[:100] = 7
        idd = ids.cuda()
        ws = [arena(g.comms[r], (vl, h), torch.bfloat16) if n > 1 else torch.empty(vl, h, dtype=torch.bfloat16, device="cuda")
              for r in range(n)]
        for r in range(n):
            ws[r].copy_(full[r * vl:(r + 1) * vl])
        outs = [None] * n
        torch.cuda.synchronize()
        g.run(lambda r, c, st: outs.__setitem__(r, c.vocab_parallel_embedding(idd, ws[r], stream=st)))
        want = F.embedding(idd, full.cuda())
        # Megatron's composition: masked local lookups summed over the ranks (exact: one non-zero term per row)
        meg = sum(F.embedding((idd - r * vl).clamp(0, vl - 1), ws[r]) * ((idd >= r * vl) & (idd < (r + 1) * vl))[:, None] for r in range(n))
        for r in range(n):
            assert torch.equal(outs[r].view(torch.int16), want.view(torch.int16))
            assert torch.equal(outs[r].float(), meg.float())
        dout = torch.randn(T, h, device="cuda").to(torch.bfloat16)
        dws = [None] * n
        g.run(lambda r, c, st: dws.__setitem__(r, c.vocab_parallel_embedding_backward(idd, dout, vocab_local=vl, stream=st)))
        wfull = full.cuda().float().requires_grad_()
        F.embedding(idd, wfull).backward(dout.float())
        for r in range(n):
            torch.testing.assert_close(dws[r], wfull.grad[r * vl:(r + 1) * vl], rtol=1e-5, atol=1e-4)
        if n > 1:
            for r, c in enumerate(g.comms):
                c.release(ws[r])


# ------------------------------------------------------------------------------------------------- launch shapes and replay
def test_forced_launch_shapes_give_identical_bits(groups):
    for n in (1, 3):
        g = groups(n)
        rng = np.random.default_rng(9)
        ids = rng.integers(0, 12, 3001 // n * n)
        ids[:500] = 2
        base = run(g, "bf16", ids, 4 if n == 3 else 12, 1024, sp=n > 1, wdt="f32", seed=5)
        for ctas, threads in ((1, 32), (3, 96), (7, 512)):
            for c in g.comms:
                c.set_launch_shape("p2p", ctas, threads)
            try:
                again = run(g, "bf16", ids, 4 if n == 3 else 12, 1024, sp=n > 1, wdt="f32", seed=5)
            finally:
                for c in g.comms:
                    c.set_launch_shape("p2p", 0, 0)
            for a, b in zip(base[1], again[1]):
                assert g.torch.equal(a.view(g.torch.int32), b.view(g.torch.int32))


def test_cuda_graph_capture_and_replay(groups):
    n = 2
    g = groups(n)
    torch = g.torch
    vl, h, T = 33, 64, 1000
    rng = np.random.default_rng(11)
    ws = [arena(c, (vl, h), torch.bfloat16) for c in g.comms]
    gos = [arena(c, (T // n, h), torch.bfloat16) for c in g.comms]
    idd = torch.zeros(T, dtype=torch.int64, device="cuda")
    outs = [torch.empty(T // n, h, dtype=torch.bfloat16, device="cuda") for _ in range(n)]
    dws = [torch.empty(vl, h, dtype=torch.float32, device="cuda") for _ in range(n)]
    # warm up (scratch taken, kernels loaded) before the capture
    torch.cuda.synchronize()
    g.run(lambda r, c, st: (c.vocab_parallel_embedding(idd, ws[r], sequence_parallel=True, out=outs[r], stream=st),
                            c.vocab_parallel_embedding_backward(idd, gos[r], dws[r], sequence_parallel=True, stream=st)))
    graphs = [torch.cuda.CUDAGraph() for _ in range(n)]
    for r, c in enumerate(g.comms):
        with torch.cuda.graph(graphs[r], stream=g.streams[r]):
            c.vocab_parallel_embedding(idd, ws[r], sequence_parallel=True, out=outs[r], stream=g.streams[r])
            c.vocab_parallel_embedding_backward(idd, gos[r], dws[r], sequence_parallel=True, stream=g.streams[r])
    for it in range(3):
        tables = [rand_bits(rng, (vl, h), "bf16") for _ in range(n)]
        ids = rng.integers(-3, n * vl + 3, T)
        ids[: 200] = 5
        dout = rand_bits(rng, (T, h), "bf16")
        for r in range(n):
            ws[r].copy_(torch.from_numpy(tables[r].view(np.int16)).view(torch.bfloat16))
            gos[r].copy_(torch.from_numpy(dout[r * T // n:(r + 1) * T // n].view(np.int16)).view(torch.bfloat16))
        idd.copy_(torch.from_numpy(ids))
        torch.cuda.synchronize()
        for r in range(n):
            with torch.cuda.stream(g.streams[r]):
                graphs[r].replay()
        torch.cuda.synchronize()
        g.check_async()
        for r in range(n):
            same_bits(bits_of(outs[r], "bf16"), ref.forward(tables, ids, True, r), "bf16", f"replay {it} forward {r}")
            same_bits(bits_of(dws[r], "f32"), ref.backward(ids, dout, "bf16", r, n, vl, "f32"), "f32", f"replay {it} backward {r}")
    for r, c in enumerate(g.comms):
        c.release(ws[r])
        c.release(gos[r])


# ------------------------------------------------------------------------------------------------- scale and training
def test_out_past_4_gib(groups):
    g = groups(1)
    torch = g.torch
    h, vl = 8192, 1024
    T = (4 << 30) // (h * 2) + 4099
    need = T * h * 2 + T * 8 + (64 << 20)
    free = torch.cuda.mem_get_info()[0]
    if free < need + (1 << 30):
        pytest.skip(f"needs {need / 2**30:.1f} GiB free")
    w = torch.randn(vl, h, device="cuda").to(torch.bfloat16)
    ids = torch.randint(-2, vl + 2, (T,), device="cuda")
    ids[-1] = vl - 1
    out = g.comms[0].vocab_parallel_embedding(ids, w)
    torch.cuda.synchronize()
    ok = (ids >= 0) & (ids < vl)
    tail = slice(T - 70000, T)
    zero = torch.zeros((), dtype=w.dtype, device="cuda")
    want = torch.where(ok[tail, None], torch.nn.functional.embedding(ids[tail].clamp(0, vl - 1), w), zero)
    assert torch.equal(out[tail].view(torch.int16), want.view(torch.int16))
    head = slice(0, 70000)
    want = torch.where(ok[head, None], torch.nn.functional.embedding(ids[head].clamp(0, vl - 1), w), zero)
    assert torch.equal(out[head].view(torch.int16), want.view(torch.int16))
    del out


def test_weight_and_dweight_past_4_gib(groups):
    """One rank: a bf16 weight of 4.2 GiB read at its head and tail rows, and an fp32 dweight of 4.1 GiB written there. Each hit row has
    one token, so its gradient is that token's row widened; every other row is +0."""
    g = groups(1)
    torch = g.torch
    h = 8192
    vlw, vld = (4 << 30) // (h * 2) + 3001, (4 << 30) // (h * 4) + 1501
    free = torch.cuda.mem_get_info()[0]
    if free < (vlw * h * 2 + vld * h * 4) + (2 << 30):
        pytest.skip(f"needs {(vlw * h * 2 + vld * h * 4) / 2**30:.1f} GiB free")
    c = g.comms[0]
    w = torch.empty(vlw, h, dtype=torch.bfloat16, device="cuda")
    rows = torch.cat([torch.arange(0, 64), torch.arange(vlw - 2000, vlw, 7)]).cuda()
    w[rows] = torch.randn(rows.numel(), h, device="cuda").to(torch.bfloat16)
    ids = rows[torch.randperm(rows.numel(), device="cuda")]
    out = c.vocab_parallel_embedding(ids, w)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), w[ids].view(torch.int16))
    del w, out
    torch.cuda.empty_cache()
    drows = torch.cat([torch.arange(0, 64), torch.arange(vld - 2000, vld, 7)]).cuda()
    ids = drows[torch.randperm(drows.numel(), device="cuda")]
    dout = torch.randn(ids.numel(), h, device="cuda").to(torch.bfloat16)
    dw = torch.empty(vld, h, dtype=torch.float32, device="cuda")
    c.vocab_parallel_embedding_backward(ids, dout, dw)
    torch.cuda.synchronize()
    assert torch.equal(dw[ids].view(torch.int32), dout.float().view(torch.int32))
    untouched = torch.ones(vld, dtype=torch.bool, device="cuda")
    untouched[ids] = False
    nonzero = (dw.view(torch.int32) != 0).any(1)
    assert not bool(nonzero[untouched].any())                               # +0 bits exactly, head, middle and tail
    del dw


@pytest.mark.parametrize("sp", [False, True])
@pytest.mark.parametrize("n", [2, 4])
def test_training_step_through_autograd(groups, n, sp):
    """Embedding, a column-parallel LM head, vocab_parallel_cross_entropy_loss; loss and every gradient against the unsplit torch model."""
    g = groups(n)
    torch = g.torch
    vl, h, T, vh = 24, 32, 64, 16                # vocabulary slice of the table and of the head
    gen = torch.Generator().manual_seed(20 + n)
    emb = torch.randn(n * vl, h, generator=gen)
    head = torch.randn(n * vh, h, generator=gen) * 0.2
    ids = torch.randint(0, n * vl, (T,), generator=gen)
    tgt = torch.randint(0, n * vh, (T,), generator=gen)
    idd, tgd = ids.cuda(), tgt.cuda()
    ws = [arena(g.comms[r], (vl, h), torch.float32) for r in range(n)]
    for r in range(n):
        ws[r].copy_(emb[r * vl:(r + 1) * vl])
    params = [torch.nn.Parameter(ws[r]) for r in range(n)]
    heads = [torch.nn.Parameter(head[r * vh:(r + 1) * vh].cuda()) for r in range(n)]
    torch.cuda.synchronize()
    outs = [None] * n
    for r, c in enumerate(g.comms):
        with torch.cuda.stream(g.streams[r]):
            g.streams[r].wait_stream(torch.cuda.default_stream())
            outs[r] = c.vocab_parallel_embedding_lookup(idd, params[r], sequence_parallel=sp)
    for st in g.streams:
        torch.cuda.default_stream().wait_stream(st)
    class Replicated(torch.autograd.Function):
        """The tensor-parallel head's input: every rank's (equal) embedding output forward, the summed gradient back to every rank
        (Megatron's copy-to-tensor-parallel-region, whose backward is an all-reduce)."""
        @staticmethod
        def forward(ctx, *xs):
            return xs[0].clone()

        @staticmethod
        def backward(ctx, grad):
            return tuple(grad for _ in range(n))

    hfull = torch.cat(outs) if sp else Replicated.apply(*outs)      # SP: the all-gather before the column-parallel head
    losses = [None] * n
    for r, c in enumerate(g.comms):
        h_r = hfull
        with torch.cuda.stream(g.streams[r]):
            g.streams[r].wait_stream(torch.cuda.default_stream())
            losses[r] = c.vocab_parallel_cross_entropy_loss((h_r @ heads[r].t()).contiguous(), tgd)
    for st in g.streams:
        torch.cuda.default_stream().wait_stream(st)
    # every rank holds the whole loss; each backpropagates its own (its xent backward covers its vocabulary slice of the logits)
    sum(l.mean() for l in losses).backward()
    torch.cuda.synchronize()
    g.check_async()
    # the unsplit model in float64
    E = emb.double().requires_grad_()
    Hd = head.double().requires_grad_()
    want = torch.nn.functional.cross_entropy(torch.nn.functional.embedding(ids, E) @ Hd.t(), tgt)
    want.backward()
    for l in losses:
        torch.testing.assert_close(l.mean().double().cpu(), want.detach(), rtol=1e-4, atol=1e-4)
    for r in range(n):
        torch.testing.assert_close(params[r].grad.double().cpu(), E.grad[r * vl:(r + 1) * vl], rtol=1e-3, atol=1e-5)
        torch.testing.assert_close(heads[r].grad.double().cpu(), Hd.grad[r * vh:(r + 1) * vh], rtol=1e-3, atol=1e-5)
    for r, c in enumerate(g.comms):
        c.release(ws[r])


def test_tied_weights_accumulate_into_one_main_grad(groups):
    """A tied LM head: its gradient lands in the fp32 main_grad first, the embedding's is added with accumulate=1."""
    n = 2
    g = groups(n)
    torch = g.torch
    vl, h, T = 16, 64, 300
    rng = np.random.default_rng(13)
    ids = rng.integers(0, n * vl, T)
    dout = rand_bits(rng, (T, h), "bf16")
    head_grads = [rng.standard_normal((vl, h)).astype(np.float32) for _ in range(n)]
    main = [torch.from_numpy(hg.copy()).cuda() for hg in head_grads]
    idd = torch.from_numpy(ids).cuda()
    d = to_dev(g, None, dout, "bf16", False)
    torch.cuda.synchronize()
    g.run(lambda r, c, st: c.vocab_parallel_embedding_backward(idd, d, main[r], accumulate=True, stream=st))
    for r in range(n):
        want = ref.backward(ids, dout, "bf16", r, n, vl, "f32", head_grads[r].view(np.uint32))
        same_bits(bits_of(main[r], "f32"), want, "f32", f"tied rank {r}")


# ------------------------------------------------------------------------------------------------- back to back with the other families
CHAIN_A = ["emb_fwd_tp", "emb_fwd_sp", "xent_fwd", "xent_bwd", "rmsnorm", "ag_shards", "rs_shards", "ag_ctx", "rs_ctx", "emb_bwd_tp",
           "emb_bwd_sp"]
CHAIN_BEFORE = ["emb_fwd_tp", "emb_fwd_sp", "rmsnorm", "ag_shards", "emb_bwd_sp", "emb_bwd_tp", "xent_fwd", "rs_shards", "ag_ctx",
                "xent_bwd", "rs_ctx"]
CHAIN_AFTER = ["emb_fwd_sp", "ag_ctx", "emb_fwd_tp", "xent_fwd", "emb_bwd_tp", "emb_bwd_sp", "xent_bwd", "rs_ctx", "rmsnorm",
               "rs_shards", "ag_shards"]


class _Chain:
    """Inputs and output buffers of every call of the chain on every rank, fresh for each run (the RMSNorm updates its residual in
    place). Arena tensors are allocated in the same order on every rank."""

    def __init__(self, g, seed):
        torch, n = g.torch, g.n
        self.g = g
        rng = np.random.default_rng(seed)
        gen = torch.Generator().manual_seed(seed)
        self.vl, self.h, self.T = 40, 64, 96 * n
        self.tables = [rand_bits(rng, (self.vl, self.h), "bf16") for _ in range(n)]
        self.ids = rng.integers(-3, n * self.vl + 3, self.T)
        self.ids[: self.T // 4] = 5                                    # one row hit by a quarter of the tokens
        self.dout = rand_bits(rng, (self.T, self.h), "bf16")
        self.idd = torch.from_numpy(self.ids).cuda()
        nr = self.T // n
        self.ws = [to_dev(g, c, self.tables[r], "bf16", True) for r, c in enumerate(g.comms)]
        self.gsp = [to_dev(g, c, self.dout[r * nr:(r + 1) * nr], "bf16", True) for r, c in enumerate(g.comms)]
        self.gtp = to_dev(g, None, self.dout, "bf16", False)
        self.out_tp = [torch.empty(self.T, self.h, dtype=torch.bfloat16, device="cuda") for _ in range(n)]
        self.out_sp = [torch.empty(nr, self.h, dtype=torch.bfloat16, device="cuda") for _ in range(n)]
        self.dw_tp = [torch.empty(self.vl, self.h, dtype=torch.float32, device="cuda") for _ in range(n)]
        self.dw_sp = [torch.empty(self.vl, self.h, dtype=torch.float32, device="cuda") for _ in range(n)]
        # cross-entropy: [rows, 32] bf16 logits per rank
        self.xrows, self.xvl = 80, 32
        self.logits_host = [(torch.randn(self.xrows, self.xvl, generator=gen) * 3).to(torch.bfloat16) for _ in range(n)]
        self.target = rng.integers(0, n * self.xvl, self.xrows)
        self.target[1] = -100
        self.logits = [x.cuda() for x in self.logits_host]
        self.tgd = torch.from_numpy(self.target).cuda()
        self.dloss = torch.linspace(0.5, 1.5, self.xrows, device="cuda")
        self.loss = [torch.empty(self.xrows, device="cuda") for _ in range(n)]
        self.lse = [torch.empty(self.xrows, device="cuda") for _ in range(n)]
        self.xgrad = [torch.empty_like(x) for x in self.logits]
        # RMSNorm all-reduce
        self.x = [arena(c, (16, 256), torch.bfloat16) for c in g.comms]
        for t in self.x:
            t.copy_(torch.randn(16, 256, generator=gen).to(torch.bfloat16))
        self.res = [torch.randn(16, 256, generator=gen).to(torch.bfloat16).cuda() for _ in range(n)]
        self.gamma = torch.randn(256, generator=gen).to(torch.bfloat16).cuda()
        self.norm = [torch.empty(16, 256, dtype=torch.bfloat16, device="cuda") for _ in range(n)]
        # FSDP: one [8n, 64] parameter, fp32 shards -> bf16 full, and bf16 full gradients -> fp32 shards (scale 1/N)
        self.shards = [torch.randn(8, 64, generator=gen).cuda() for _ in range(n)]
        self.pfull = [arena(c, (8 * n, 64), torch.bfloat16) for c in g.comms]
        self.gfull = [arena(c, (8 * n, 64), torch.bfloat16) for c in g.comms]
        for t in self.gfull:
            t.copy_(torch.randn(8 * n, 64, generator=gen).to(torch.bfloat16))
        self.gshard = [torch.empty(8, 64, device="cuda") for _ in range(n)]
        # context parallelism: K [1, 6, 2, 64] bf16 shards, load-balanced chunks
        self.kv = [torch.randn(1, 6, 2, 64, generator=gen).to(torch.bfloat16).cuda() for _ in range(n)]
        self.kfull = [arena(c, (1, 6 * n, 2, 64), torch.bfloat16) for c in g.comms]
        self.dkfull = [arena(c, (1, 6 * n, 2, 64), torch.bfloat16) for c in g.comms]
        for t in self.dkfull:
            t.copy_(torch.randn(1, 6 * n, 2, 64, generator=gen).to(torch.bfloat16))
        self.dk = [torch.empty(1, 6, 2, 64, dtype=torch.bfloat16, device="cuda") for _ in range(n)]
        for t in self.out_tp + self.out_sp + self.dw_tp + self.dw_sp + self.loss + self.lse + self.xgrad + self.norm + self.gshard + \
                self.pfull + self.kfull + self.dk:
            poison([t])
        torch.cuda.synchronize()

    def call(self, op, r, c, st):
        if op == "emb_fwd_tp":
            c.vocab_parallel_embedding(self.idd, self.ws[r], out=self.out_tp[r], stream=st)
        elif op == "emb_fwd_sp":
            c.vocab_parallel_embedding(self.idd, self.ws[r], sequence_parallel=True, out=self.out_sp[r], stream=st)
        elif op == "emb_bwd_tp":                                        # no barrier: nothing crosses ranks
            c.vocab_parallel_embedding_backward(self.idd, self.gtp, self.dw_tp[r], stream=st)
        elif op == "emb_bwd_sp":
            c.vocab_parallel_embedding_backward(self.idd, self.gsp[r], self.dw_sp[r], sequence_parallel=True, stream=st)
        elif op == "xent_fwd":
            c.vocab_parallel_cross_entropy(self.logits[r], self.tgd, loss=self.loss[r], lse=self.lse[r], stream=st)
        elif op == "xent_bwd":
            c.vocab_parallel_cross_entropy_backward(self.logits[r], self.tgd, self.lse[r], self.dloss, self.xgrad[r], stream=st)
        elif op == "rmsnorm":
            c.all_reduce_rms_norm(self.x[r], self.res[r], self.gamma, out=self.norm[r], stream=st)
        elif op == "ag_shards":
            c.all_gather_shards([self.shards[r]], [self.pfull[r]], stream=st)
        elif op == "rs_shards":
            c.reduce_scatter_shards([self.gfull[r]], [self.gshard[r]], scale=1.0 / self.g.n, stream=st)
        elif op == "ag_ctx":
            c.all_gather_context([self.kv[r]], [self.kfull[r]], chunks=2, stream=st)
        elif op == "rs_ctx":
            c.reduce_scatter_context([self.dkfull[r]], [self.dk[r]], chunks=2, stream=st)

    def results(self):
        return {k: [t.clone() for t in getattr(self, k)] for k in ("out_tp", "out_sp", "dw_tp", "dw_sp", "loss", "lse", "xgrad", "norm",
                                                                    "res", "pfull", "gshard", "kfull", "dk")}

    def release(self):
        for r, c in enumerate(self.g.comms):
            for lst in (self.ws, self.gsp, self.x, self.pfull, self.gfull, self.kfull, self.dkfull):
                c.release(lst[r])


def _run_chain(g, order, seed, alone):
    """Every call of `order` on every rank. alone: each call on its own, a sync after it (the reference run); otherwise op-major (call i
    on every rank before call i + 1 on any rank), no host sync until the end."""
    ch = _Chain(g, seed)
    for op in order:
        for r, c in enumerate(g.comms):
            with g.torch.cuda.device(c.device):
                g.streams[r].wait_stream(g.torch.cuda.current_stream())
                ch.call(op, r, c, g.streams[r])
        if alone:
            g.sync()
            g.check_async()
    g.sync()
    g.check_async()
    return ch, ch.results()


@pytest.mark.parametrize("order", ["end", "before_xent", "after_xent"])
@pytest.mark.parametrize("n", [2, 4])
def test_back_to_back_with_other_families(groups, n, order):
    """The embedding calls (TP and SP, forward and backward) chained with the cross-entropy, the RMSNorm all-reduce, the FSDP and the
    context-parallel calls on one communicator, with no host sync between calls: the TP backward (no barrier) and the SP backward sort in
    the quantising scratch that the cross-entropy's mailbox shares. The embedding and cross-entropy results are checked bit for bit
    against their references, every result bit for bit against the same calls run one at a time."""
    g = groups(n)
    torch = g.torch
    chain = {"end": CHAIN_A, "before_xent": CHAIN_BEFORE, "after_xent": CHAIN_AFTER}[order]
    seed = 100 * n + len(order)
    ch, solo = _run_chain(g, chain, seed, alone=True)
    ch.release()
    for rep in range(2):
        ch, got = _run_chain(g, chain, seed, alone=False)
        for k in solo:
            for r in range(n):
                a, b = got[k][r], solo[k][r]
                iv = torch.int32 if a.element_size() == 4 else torch.int16
                assert torch.equal(a.view(iv), b.view(iv)), f"{order} rep {rep}: {k} rank {r} differs from the call run alone"
        for r in range(n):
            assert np.array_equal(bits_of(got["out_tp"][r], "bf16"), ref.forward(ch.tables, ch.ids, False, r)), f"emb forward TP rank {r}"
            assert np.array_equal(bits_of(got["out_sp"][r], "bf16"), ref.forward(ch.tables, ch.ids, True, r)), f"emb forward SP rank {r}"
            want = ref.backward(ch.ids, ch.dout, "bf16", r, n, ch.vl, "f32")
            same_bits(bits_of(got["dw_tp"][r], "f32"), want, "f32", f"{order}: emb backward TP rank {r}")
            same_bits(bits_of(got["dw_sp"][r], "f32"), want, "f32", f"{order}: emb backward SP rank {r}")
        wl, wlse = xref.forward(ch.logits_host, ch.target, -100)
        for r in range(n):
            assert np.array_equal(got["loss"][r].cpu().numpy().view(np.int32), np.asarray(wl, np.float32).view(np.int32)), f"xent loss {r}"
            assert np.array_equal(got["lse"][r].cpu().numpy().view(np.int32), np.asarray(wlse, np.float32).view(np.int32)), f"xent lse {r}"
            wg = xref.backward(ch.logits_host[r], r, n, ch.target, wlse, ch.dloss.cpu().numpy(), -100)
            assert torch.equal(got["xgrad"][r].cpu().view(torch.int16), wg.view(torch.int16)), f"xent grad rank {r}"
        ch.release()
