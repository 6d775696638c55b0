"""The context-parallel all-gather and reduce-scatter (b200collAllGatherContext / ReduceScatterContext) on an H100 (`pytest -m gpu`),
virtual ranks sharing cuda:0 unless a test says otherwise.

Gather sources are random bytes, so NaN payloads, -0 and inf occur in every float type, and every rank's bytes differ: a byte read or
stored at the wrong place shows. Reduce-scatter inputs come from coll_fp_reference.gen_inputs, which tells summation orders apart.
Outputs are poisoned first and compared with tests/coll_context_reference."""
import ctypes as C

import pytest

from container_engine_accelerators_b200.ops.coll import INVALID_ARGUMENT, INVALID_USAGE
from tests import coll_context_reference as ref
from tests import coll_fp_reference as R
from tests.coll_gpu_harness import (DTYPES, Group, assert_nothing_launched, coll_mod, expect_refused, poison, run_perf,  # noqa: F401
                                    torch_cuda)

pytestmark = pytest.mark.gpu

DT_NAMES = ("bf16", "f16", "f32", "e4m3", "e5m2")
_groups = {}


@pytest.fixture(scope="module")
def groups(torch_cuda, coll_mod):
    def get(n):
        if n not in _groups:
            _groups[n] = Group(torch_cuda, coll_mod, n, arena_mb=256)
        return _groups[n]
    yield get
    for g in _groups.values():
        g.destroy()
    _groups.clear()


def random_bytes(torch, shape, dt, gen):
    es = torch.empty((), dtype=dt).element_size()
    n = 1
    for d in shape:
        n *= d
    return torch.randint(0, 256, (n * es,), dtype=torch.uint8, generator=gen).view(dt).view(shape)


def arena_like(c, shape, dt):
    n = 1
    for d in shape:
        n *= d
    base = c.empty(max(n, 1), dt)
    return base, base[:n].view(shape)


def check_bytes(got, want, what):
    g, w = got.contiguous().view(-1), want.contiguous().view(-1)
    assert g.numel() == w.numel(), what
    bad = (g != w).nonzero()
    assert bad.numel() == 0, f"{what}: {bad.numel()} bytes differ, first at byte {int(bad[0])}"


def packed_views(buf, B, S_l, q_cols, widths):
    """Column slices [B, S_l, W_i] of a packed [B * S_l, q_cols + sum(widths)] buffer, after its first q_cols (Q) columns."""
    cols = [q_cols]
    for w in widths:
        cols.append(cols[-1] + w)
    return [buf[:, cols[i]:cols[i + 1]].view(B, S_l, w) for i, w in enumerate(widths)]


def run_gather(g, B, S_l, widths, dt, chunks, packed, seed):
    """One all_gather_context of len(widths) tensors, checked on every rank against the reference. widths in elements; packed: the
    shards are column slices of one [B * S_l, 64 bytes of Q + sum(widths)] buffer per rank. Returns the stats before and after."""
    torch, n = g.torch, g.n
    es = torch.empty((), dtype=dt).element_size()
    gen = torch.Generator().manual_seed(seed)
    host, dev, bases = [], [], []
    for _ in range(n):
        if packed:
            buf = random_bytes(torch, (B * S_l, 64 // es + sum(widths)), dt, gen)
            xs = packed_views(buf, B, S_l, 64 // es, widths)
            d = packed_views(buf.cuda(), B, S_l, 64 // es, widths)
        else:
            xs = [random_bytes(torch, (B, S_l, w), dt, gen) for w in widths]
            d = [x.cuda() for x in xs]
        host.append(xs)
        dev.append(d)
    fulls = []
    for c in g.comms:
        row = []
        for w in widths:
            b, f = arena_like(c, (B, n * S_l, w), dt)
            bases.append((c, b))
            row.append(f)
        poison(row)
        fulls.append(row)
    torch.cuda.synchronize()
    before = [c.stats() for c in g.comms]
    g.run(lambda r, c, st: c.all_gather_context(dev[r], fulls[r], chunks=chunks, stream=st))
    after = [c.stats() for c in g.comms]
    what = f"n={n} {dt} B={B} S_l={S_l} widths={widths} chunks={chunks} packed={packed}"
    for i in range(len(widths)):
        want = ref.all_gather([host[s][i] for s in range(n)], chunks)
        for r in range(n):
            check_bytes(fulls[r][i].cpu().view(torch.uint8), want.reshape(-1), f"{what} tensor {i} rank {r}")
    for c, b in bases:
        c.release(b)
    return before, after


# (B, S_l, widths in bytes, packed); S_l odd only with chunks = 1
GATHER_CASES = [(1, 6, (256, 256), True), (3, 5, (512, 16, 64), False), (3, 4, (48,), False), (1, 2, (16, 2048), True),
                (2, 8, (1024, 128), False), (3, 3, (32, 32, 32), True)]


@pytest.mark.parametrize("dtn", DT_NAMES)
@pytest.mark.parametrize("n", [1, 2, 3, 4, 6, 8])
def test_gather_bit_exact_sweep(torch_cuda, groups, n, dtn):
    dt = DTYPES[dtn]
    es = torch_cuda.empty((), dtype=dt).element_size()
    g = groups(n)
    for k, (B, S_l, wb, packed) in enumerate(GATHER_CASES):
        for chunks in (1, 2):
            if chunks == 2 and S_l % 2:
                continue
            run_gather(g, B, S_l, tuple(w // es for w in wb), dt, chunks, packed, seed=1000 * n + 10 * k + chunks)


def run_reduce_scatter(g, B, S_l, widths, dt, chunks, seed, inputs=None):
    """One reduce_scatter_context of len(widths) tensors into the column slices of a packed dQKV [B * S_l, 64 + sum(widths)] per rank
    whose 64 Q columns are poisoned and must stay so; checked against the reference (NaN by position). inputs: per rank, per tensor,
    the [B, N * S_l, W] fulls on the host (default: gen_inputs)."""
    torch, n = g.torch, g.n
    S = n * S_l
    if inputs is None:
        per = [R.gen_inputs(n, B * S * w, dt, seed + i, device="cpu") for i, w in enumerate(widths)]
        inputs = [[per[i][r].view(B, S, w) for i, w in enumerate(widths)] for r in range(n)]
    fulls, dq, bases = [], [], []
    for r, c in enumerate(g.comms):
        row = []
        for i, w in enumerate(widths):
            b, f = arena_like(c, (B, S, w), dt)
            bases.append((c, b))
            f.copy_(inputs[r][i])
            row.append(f)
        fulls.append(row)
        buf = torch.empty(B * S_l, 64 + sum(widths), dtype=dt, device="cuda")
        poison([buf])
        dq.append(buf)
    shards = [packed_views(buf, B, S_l, 64, widths) for buf in dq]
    torch.cuda.synchronize()
    before = [c.stats() for c in g.comms]
    g.run(lambda r, c, st: c.reduce_scatter_context(fulls[r], shards[r], chunks=chunks, stream=st))
    after = [c.stats() for c in g.comms]
    what = f"n={n} {dt} B={B} S_l={S_l} widths={widths} chunks={chunks}"
    for i in range(len(widths)):
        want = ref.reduce_scatter([inputs[s][i] for s in range(n)], chunks)
        for r in range(n):
            R.assert_same(shards[r][i].cpu().contiguous(), want[r], f"{what} tensor {i} rank {r}", nan_payloads=n == 1)
    for r in range(n):
        assert bool((dq[r][:, :64].cpu().view(-1).view(torch.uint8) == 0x7B).all()), f"{what}: rank {r}'s Q columns were written"
    for c, b in bases:
        c.release(b)
    return before, after


@pytest.mark.parametrize("dtn", ("bf16", "f16", "f32"))
@pytest.mark.parametrize("n", [1, 2, 3, 4, 6, 8])
def test_reduce_scatter_bit_exact_sweep(torch_cuda, groups, n, dtn):
    dt = DTYPES[dtn]
    es = torch_cuda.empty((), dtype=dt).element_size()
    g = groups(n)
    for k, (B, S_l, wb) in enumerate([(1, 6, (256, 256)), (3, 5, (512, 16)), (2, 4, (1024,)), (1, 8, (16, 64, 32))]):
        for chunks in (1, 2):
            if chunks == 2 and S_l % 2:
                continue
            run_reduce_scatter(g, B, S_l, tuple(w // es for w in wb), dt, chunks, seed=2000 * n + 10 * k + chunks)


@pytest.mark.parametrize("dtn", ("bf16", "f16", "f32"))
def test_reduce_scatter_special_values(torch_cuda, groups, dtn):
    """+-inf, NaN, inf - inf, and sums of -0 on every rank (+0 with N > 1: the sum starts from +0; -0 with one rank: a bit copy)."""
    torch = torch_cuda
    dt = DTYPES[dtn]
    W = 64 // torch.empty((), dtype=dt).element_size()
    for n in (1, 2, 4):
        g = groups(n)
        S_l, S = 4, 4 * n
        inputs = []
        for r in range(n):
            f = torch.full((1, S, W), -0.0, dtype=torch.float32)
            f[0, :, 1] = float("inf")
            f[0, :, 2] = float("inf") if r % 2 == 0 else float("-inf")
            f[0, :, 3] = float("nan") if r == n - 1 else 1.0
            f[0, :, 4] = 1.5 * (r + 1)
            inputs.append([f.to(dt)])
        run_reduce_scatter(g, 1, S_l, (W,), dt, 2, seed=0, inputs=inputs)
        shard = ref.reduce_scatter([x[0] for x in inputs], 2)[0]
        zbits = shard[0, :, 0].view(R.INT_VIEW[R.esize(dt)])
        assert bool((zbits == (0 if n > 1 else torch.tensor(-0.0, dtype=dt).view(R.INT_VIEW[R.esize(dt)]))).all()), (n, zbits)


def test_gather_equals_the_unfused_composition(torch_cuda, groups):
    """The gather equals what a layer writes without the fused call, byte for byte: a dense copy of the K slice, comm.all_gather, and an
    index_select from rank-chunk order into token order."""
    torch = torch_cuda
    n, B, S_l, W, dt, chunks = 4, 2, 10, 256, torch.bfloat16, 2
    g = groups(n)
    gen = torch.Generator().manual_seed(5)
    qkv = [random_bytes(torch, (B * S_l, 1024 + 2 * W), dt, gen).cuda() for _ in range(n)]
    ks = [packed_views(b, B, S_l, 1024, (W,))[0] for b in qkv]
    bases, fused, sends, recvs = [], [], [], []
    for c in g.comms:
        b, f = arena_like(c, (B, n * S_l, W), dt)
        bases.append((c, b))
        fused.append(f)
        b, s = arena_like(c, (B, S_l, W), dt)
        bases.append((c, b))
        sends.append(s)
        b, rv = arena_like(c, (n, B, S_l, W), dt)
        bases.append((c, b))
        recvs.append(rv)
    poison(fused + recvs)
    torch.cuda.synchronize()
    g.run(lambda r, c, st: c.all_gather_context([ks[r]], [fused[r]], chunks=chunks, stream=st))
    for r in range(n):
        sends[r].copy_(ks[r])
    torch.cuda.synchronize()
    g.run(lambda r, c, st: c.all_gather(sends[r].view(-1), recvs[r].view(-1), stream=st))
    idx = ref.token_index(n, chunks, S_l).cuda()
    for r in range(n):
        composed = recvs[r].permute(1, 0, 2, 3).reshape(B, n * S_l, W).index_select(1, idx)
        assert torch.equal(composed.view(torch.int16), fused[r].view(torch.int16)), r
    for c, b in bases:
        c.release(b)


def test_reduce_scatter_of_the_gather(torch_cuda, groups):
    """Every rank feeds the gathered K back as its gradient: the reduce-scatter sums N equal contributions, against the reference."""
    torch = torch_cuda
    for n, dt in ((2, torch.bfloat16), (4, torch.float16), (8, torch.float32)):
        g = groups(n)
        B, S_l, W, chunks = 1, 6, 128, 2
        xs = [R.gen_inputs(n, B * S_l * W, dt, seed=40 + n, device="cpu")[r].view(B, S_l, W) for r in range(n)]
        fulls, bases = [], []
        for c in g.comms:
            b, f = arena_like(c, (B, n * S_l, W), dt)
            bases.append((c, b))
            fulls.append(f)
        torch.cuda.synchronize()
        dev = [x.cuda() for x in xs]
        g.run(lambda r, c, st: c.all_gather_context([dev[r]], [fulls[r]], chunks=chunks, stream=st))
        outs = [torch.empty(B, S_l, W, dtype=dt, device="cuda") for _ in range(n)]
        g.run(lambda r, c, st: c.reduce_scatter_context([fulls[r]], [outs[r]], chunks=chunks, stream=st))
        full = ref.all_gather(xs, chunks).view(dt).view(B, n * S_l, W)
        want = ref.reduce_scatter([full] * n, chunks)
        for r in range(n):
            R.assert_same(outs[r].cpu(), want[r], f"n={n} {dt} rank {r}")
        for c, b in bases:
            c.release(b)


def test_stats_one_launch(torch_cuda, groups):
    torch = torch_cuda
    for n in (1, 4):
        g = groups(n)
        B, S_l, widths = 2, 6, (128, 64)
        algo = "copy" if n == 1 else "twoshot"
        for op, (before, after) in ((1, run_gather(g, B, S_l, widths, torch.bfloat16, 2, True, seed=11)),
                                    (2, run_reduce_scatter(g, B, S_l, widths, torch.bfloat16, 2, seed=12))):
            for b, a in zip(before, after):
                assert a["kernel_launches"] == b["kernel_launches"] + 1
                assert a["calls"][op] == b["calls"][op] + 1 and sum(a["calls"]) == sum(b["calls"]) + 1
                assert a["bytes"][op] - b["bytes"][op] == B * S_l * sum(widths) * 2
                assert a["algo_calls"][algo] == b["algo_calls"][algo] + 1 and sum(a["algo_calls"].values()) == sum(b["algo_calls"].values()) + 1


def test_back_to_back_without_host_sync(torch_cuda, coll_mod):
    """Three layers on one communicator with no host sync: the K and V gather, a torch op reading the full tensors and writing their
    gradient, the gradient's reduce-scatter into a packed dQKV, with an all_to_all_seq_to_heads, a reduce_scatter_rms_norm and an
    all_gather between them, ranks launched in a different order every phase, and the K and V sources overwritten on their rank's stream
    right after the gather that read them."""
    with Group(torch_cuda, coll_mod, 4, arena_mb=64, timeout_ms=30000) as g:       # a hang fails in 30 s
        _back_to_back(torch_cuda, g)


def _back_to_back(torch, g):
    n, B, S_l, W, dt, chunks = 4, 2, 8, 128, torch.bfloat16, 2
    layers = 3
    gen = torch.Generator().manual_seed(31)
    # small finite values (a doubling and a sum of four stay exact)
    srcs = [[[((random_bytes(torch, (B, S_l, W), dt, gen).view(torch.int16) % 64).to(torch.float32) / 8).to(dt) for _ in range(2)]
             for _ in range(n)] for _ in range(layers)]
    qkv = [torch.empty(B * S_l, 256 + 2 * W, dtype=dt, device="cuda") for _ in range(n)]
    kv = [packed_views(b, B, S_l, 256, (W, W)) for b in qkv]
    fulls, grads, dqkv, saved = [], [], [], []
    uly_x, uly_y, rms, ag_in, ag_out = [], [], [], [], []
    for r, c in enumerate(g.comms):
        fulls.append([arena_like(c, (B, n * S_l, W), dt)[1] for _ in range(2)])
        grads.append([arena_like(c, (B, n * S_l, W), dt)[1] for _ in range(2)])
        dqkv.append([torch.full((B * S_l, 256 + 2 * W), 3.0, dtype=dt, device="cuda") for _ in range(layers)])
        saved.append([[torch.empty(B, n * S_l, W, dtype=dt, device="cuda") for _ in range(2)] for _ in range(layers)])
        uly_x.append(torch.arange(B * S_l * n * 64, device="cuda").to(dt).view(B, S_l, n, 64) + r)
        uly_y.append(arena_like(c, (B, n * S_l, 1, 64), dt)[1])
        x = arena_like(c, (8 * n, 256), dt)[1]
        x.fill_(0.5)
        rms.append((x, torch.zeros(8, 256, dtype=dt, device="cuda"), torch.ones(256, dtype=dt, device="cuda"),
                    torch.empty(8, 256, dtype=dt, device="cuda")))
        t = arena_like(c, (1024,), dt)[1]
        t.copy_(torch.arange(1024, device="cuda").to(dt) + r)
        ag_in.append(t)
        ag_out.append(arena_like(c, (n * 1024,), dt)[1])
    nxt = [[[x.cuda() for x in row] for row in layer] for layer in srcs]
    torch.cuda.synchronize()
    # Each phase is enqueued for every rank before the next, in a rank order that changes from phase to phase (see the Ulysses test:
    # a PyTorch kernel's first launch must not queue behind a collective that waits for a rank this thread has not launched yet).
    def copy_in(r, c, st, L):
        for x, s in zip(kv[r], nxt[L][r]):
            x.copy_(s)

    def gather(r, c, st, L):
        c.all_gather_context(kv[r], fulls[r], chunks=chunks, stream=st)

    def overwrite_and_read(r, c, st, L):
        qkv[r].fill_(-7.0)                                                  # the sources overwritten right after the call
        for f, s, d in zip(fulls[r], saved[r][L], grads[r]):
            s.copy_(f)
            torch.mul(f, 2, out=d)                                          # the attention backward stand-in reads the full K and V

    def ulysses(r, c, st, L):
        c.all_to_all_seq_to_heads([uly_x[r]], [uly_y[r]], stream=st)

    def rs(r, c, st, L):
        c.reduce_scatter_context(grads[r], packed_views(dqkv[r][L], B, S_l, 256, (W, W)), chunks=chunks, stream=st)

    def rms_norm(r, c, st, L):
        c.reduce_scatter_rms_norm(*rms[r], stream=st)

    def ag(r, c, st, L):
        c.all_gather(ag_in[r], ag_out[r], stream=st)

    phases = [copy_in, gather, overwrite_and_read, ulysses, rs, rms_norm, ag]
    orders = [list(range(n)), list(reversed(range(n))), [2, 0, 3, 1], [1, 3, 0, 2]]
    for L in range(layers):
        for k, phase in enumerate(phases):
            for r in orders[(L + k) % len(orders)]:
                with torch.cuda.stream(g.streams[r]):
                    phase(r, g.comms[r], g.streams[r], L)
    g.sync()
    g.check_async()
    for L in range(layers):
        for i in range(2):
            want = ref.all_gather([srcs[L][s][i] for s in range(n)], chunks).view(dt).view(B, n * S_l, W)
            for r in range(n):
                assert torch.equal(saved[r][L][i].cpu().view(torch.int16), want.view(torch.int16)), f"layer {L} gather {i} rank {r}"
            back = ref.reduce_scatter([want * 2] * n, chunks)
            for r in range(n):
                got = packed_views(dqkv[r][L].cpu(), B, S_l, 256, (W, W))[i]
                assert torch.equal(got.contiguous().view(torch.int16), back[r].view(torch.int16)), f"layer {L} reduce-scatter {i} rank {r}"
        for r in range(n):
            assert bool((dqkv[r][L][:, :256] == 3.0).all()), f"layer {L} rank {r}: Q columns of dQKV written"
    for r in range(n):
        assert torch.equal(ag_out[r], torch.cat([ag_in[q] for q in range(n)])), r
        want = torch.cat([uly_x[s][:, :, r:r + 1] for s in range(n)], dim=1)
        assert torch.equal(uly_y[r], want), r


def test_cuda_graph_replay(torch_cuda, groups):
    """A graph per rank capturing the gather of K and V from a packed QKV and the reduce-scatter of their gradient into a packed dQKV,
    replayed several times with new inputs."""
    torch = torch_cuda
    n, B, S_l, W, dt, chunks = 4, 1, 12, 256, torch.bfloat16, 2
    g = groups(n)
    qkv, fulls, grads, dqkv, bases = [], [], [], [], []
    for c in g.comms:
        qkv.append(torch.empty(B * S_l, 512 + 2 * W, dtype=dt, device="cuda"))
        row, grow = [], []
        for _ in range(2):
            b, f = arena_like(c, (B, n * S_l, W), dt)
            bases.append((c, b))
            row.append(f)
            b, f = arena_like(c, (B, n * S_l, W), dt)
            bases.append((c, b))
            grow.append(f)
        fulls.append(row)
        grads.append(grow)
        dqkv.append(torch.empty(B * S_l, 512 + 2 * W, dtype=dt, device="cuda"))
    graphs = [torch.cuda.CUDAGraph() for _ in g.comms]
    torch.cuda.synchronize()
    for r, c in enumerate(g.comms):
        with torch.cuda.graph(graphs[r], stream=g.streams[r]):
            c.all_gather_context(packed_views(qkv[r], B, S_l, 512, (W, W)), fulls[r], chunks=chunks, stream=g.streams[r])
            c.reduce_scatter_context(grads[r], packed_views(dqkv[r], B, S_l, 512, (W, W)), chunks=chunks, stream=g.streams[r])
    torch.cuda.synchronize()
    for it in range(3):
        gen = torch.Generator().manual_seed(300 + it)
        host_kv, host_g = [], []
        for r in range(n):
            hq = random_bytes(torch, (B * S_l, 512 + 2 * W), dt, gen)
            qkv[r].copy_(hq.cuda())
            host_kv.append(packed_views(hq, B, S_l, 512, (W, W)))
            gs = [x.view(B, n * S_l, W) for x in R.gen_inputs(1, B * n * S_l * W, dt, seed=500 + 10 * it + r, device="cpu") * 2]
            for d, s in zip(grads[r], gs):
                d.copy_(s)
            host_g.append(gs)
        poison([f for row in fulls for f in row] + dqkv)
        torch.cuda.synchronize()
        for r in range(n):
            with torch.cuda.stream(g.streams[r]):
                graphs[r].replay()
        torch.cuda.synchronize()
        g.check_async()
        for i in range(2):
            want = ref.all_gather([host_kv[s][i] for s in range(n)], chunks)
            back = ref.reduce_scatter([host_g[s][i] for s in range(n)], chunks)
            for r in range(n):
                check_bytes(fulls[r][i].cpu().view(torch.uint8), want.reshape(-1), f"replay {it} gather {i} rank {r}")
                got = packed_views(dqkv[r].cpu(), B, S_l, 512, (W, W))[i].contiguous()
                R.assert_same(got, back[r], f"replay {it} reduce-scatter {i} rank {r}")
    del graphs
    torch.cuda.synchronize()
    for c, b in bases:
        c.release(b)


def test_refusals_launch_nothing(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    L = coll.load()
    with Group(torch, coll, 2) as g:
        c = g.comms[0]
        dt = torch.bfloat16
        BF16 = coll.torch_dtype_code(dt)
        B, S_l, W = 1, 4, 256
        qkv = torch.zeros(B * S_l, 6 * W, dtype=dt, device="cuda")
        fb = c.empty(1 << 16, dt)
        plain = torch.zeros(1 << 16, dtype=dt, device="cuda")
        full = fb.data_ptr()
        T = coll.ContextTensor
        AG, RS = L.b200collAllGatherContext, L.b200collReduceScatterContext

        def call(fn=AG, tensors=None, nt=None, batch=B, seq_local=S_l, chunks=2, dtype=BF16):
            ts = tensors if tensors is not None else [T(qkv.data_ptr(), 6 * W, full, W)]
            arr = (T * max(len(ts), 1))(*ts)
            return fn(arr, len(ts) if nt is None else nt, batch, seq_local, chunks, dtype, c._h, C.c_void_p(0))

        k, v = qkv.data_ptr() + 4 * W * 2, qkv.data_ptr() + 5 * W * 2
        cases = [
            (dict(nt=0), INVALID_ARGUMENT, "ntensors must be 1, 2 or 3"),
            (dict(nt=4), INVALID_ARGUMENT, "ntensors must be 1, 2 or 3"),
            (dict(dtype=coll.I32), INVALID_ARGUMENT, "dtype must be"),
            (dict(fn=RS, dtype=coll.torch_dtype_code(torch.float8_e4m3fn)), INVALID_ARGUMENT, "dtype must be bf16, fp16 or fp32"),
            (dict(chunks=3), INVALID_ARGUMENT, "chunks must be 1 or 2"),
            (dict(chunks=2, seq_local=3), INVALID_ARGUMENT, "even seq_local"),
            (dict(tensors=[T(k, 6 * W, full, 4)]), INVALID_ARGUMENT, "width * sizeof(dtype)"),
            (dict(tensors=[T(k, 6 * W, full, 0)]), INVALID_ARGUMENT, "width * sizeof(dtype)"),
            (dict(tensors=[T(k, W - 8, full, W)]), INVALID_ARGUMENT, "row_stride must be at least width"),
            (dict(tensors=[T(k, 6 * W + 4, full, W)]), INVALID_ARGUMENT, "multiple of 16 bytes"),
            (dict(tensors=[T(k + 2, 6 * W, full, W)]), INVALID_ARGUMENT, "16-byte aligned"),
            (dict(tensors=[T(0, 6 * W, full, W)]), INVALID_ARGUMENT, "null pointer"),
            (dict(batch=1 << 31), INVALID_ARGUMENT, "below 2^31"),
            (dict(seq_local=1 << 30, batch=1), INVALID_ARGUMENT, "2^31 - 1"),
            (dict(tensors=[T(k, 1 << 40, full, W)]), INVALID_ARGUMENT, "2^31 - 1"),
            (dict(tensors=[T(k, 6 * W, k - 64, W)]), INVALID_ARGUMENT, "output 0 overlaps source 0"),
            (dict(tensors=[T(k, 6 * W, full, W), T(v, 6 * W, full + 64, W)]), INVALID_ARGUMENT, "outputs 0 and 1 overlap"),
            (dict(fn=RS, tensors=[T(k, 6 * W, full, W), T(k + 64, 6 * W, full + 4096, W)]), INVALID_ARGUMENT, "outputs 0 and 1 overlap"),
            (dict(tensors=[T(k, 6 * W, plain.data_ptr(), W)]), INVALID_USAGE, "symmetric arena"),
            (dict(fn=RS, tensors=[T(k, 6 * W, plain.data_ptr(), W)]), INVALID_USAGE, "symmetric arena"),
        ]
        torch.cuda.synchronize()
        for kw, code, msg in cases:
            prefix = "reduce-scatter context: " if kw.get("fn") is RS else "all-gather context: "
            expect_refused(call(**kw), code, msg, prefix=prefix, what=(msg, kw))
        # B * S_l == 0 returns at once, with nothing launched
        assert call(batch=0) == 0 and call(fn=RS, seq_local=0) == 0
        assert_nothing_launched(c)
        c.release(fb)


@pytest.mark.parametrize("devs,dtype,op,spec", [("0", "bfloat16", "all_gather", "32:8:128:2"), ("0", "e4m3", "all_gather", "512:1"),
                                                ("0", "float", "reduce_scatter", "32:8:128:2"), ("0,0", "half", "all_gather", "64:8:128:2"),
                                                ("0,0", "bfloat16", "reduce_scatter", "512:2"),
                                                ("0,0,0,0", "bfloat16", "all_gather", "32:8:128:2"),
                                                ("0,0,0,0", "e5m2", "all_gather", "64:1"),
                                                ("0,0,0,0", "bfloat16", "reduce_scatter", "32:8:128:2"),
                                                ("0,0,0", "float", "reduce_scatter", "64:1")])
def test_perf_tool_checks_every_byte(torch_cuda, coll_lib, devs, dtype, op, spec):
    out = run_perf(["--op", op, "-d", dtype, "--context", spec, "-b", "64K", "-e", "4M", "-f", "4", "-w", "1", "-n", "2", "-c", "1"],
                   devs, env={"B200COLL_TIMEOUT_MS": "20000"})
    assert "context" in out, out
    n = len(devs.split(","))
    rows = [l for l in out.splitlines() if l and not l.startswith("#")]
    assert rows and all(l.split()[3] == ("copy" if n == 1 else "twoshot") for l in rows), out


def test_multi_gpu_perf_tool_processes_cross_checked(torch_cuda, coll_lib):
    """One process per GPU with B200COLL_CHECK=1: the ranks exchange the direction, shapes, chunks, widths, row strides and full offsets
    before every launch, and every byte is checked."""
    torch = torch_cuda
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    devs = ",".join(str(i) for i in range(n))
    for op, spec in (("all_gather", "32:8:128:2"), ("reduce_scatter", "32:8:128:2"), ("all_gather", "576:1")):
        run_perf(["--op", op, "-d", "bfloat16", "--context", spec, "-b", "1M", "-e", "16M", "-f", "4", "-w", "1", "-n", "3", "-c", "1"],
                 devs, procs=True, env={"B200COLL_CHECK": "1", "B200COLL_TIMEOUT_MS": "20000"}, timeout=300)
