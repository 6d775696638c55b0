"""The Ulysses all-to-all (b200collAllToAllSeqToHeads / HeadsToSeq) on an H100 (`pytest -m gpu`), virtual ranks sharing cuda:0 unless a
test says otherwise.

Sources are random bytes, so NaN payloads, -0 and inf occur in every float type, and every rank's bytes differ: a byte read or stored at
the wrong place shows. Outputs are poisoned first and compared byte for byte with tests/coll_ulysses_reference."""
import ctypes as C

import pytest

from container_engine_accelerators_b200.ops.coll import INVALID_ARGUMENT, INVALID_USAGE
from tests import coll_ulysses_reference as ref
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


def head_configs(n):
    """(name, Hq, Hkv): MHA, GQA with Hkv >= N, GQA with Hkv < N (K and V replicated) and MQA, where the rank count allows them."""
    cfgs = [("mha", 2 * n, 2 * n), ("gqa", 4 * n, n)]
    small = [h for h in range(2, n) if n % h == 0]
    if small:
        cfgs.append(("gqa-replicated", 4 * n, small[-1]))
    if n > 1:
        cfgs.append(("mqa", 2 * n, 1))
    return cfgs


def random_bytes(torch, shape, dt, gen):
    es = torch.empty((), dtype=dt).element_size()
    n = 1
    for d in shape:
        n *= d
    return torch.randint(0, 256, (n * es,), dtype=torch.uint8, generator=gen).view(dt).view(shape)


def sources(torch, n, B, S_l, heads, D, dt, packed, seed):
    """Per rank, the [B, S_l, H_i, D] sources on the device: column slices of one packed QKV tensor, or separate dense tensors; and their
    host copies."""
    gen = torch.Generator().manual_seed(seed)
    host, dev = [], []
    for _ in range(n):
        if packed:
            qkv = random_bytes(torch, (B * S_l, sum(heads) * D), dt, gen).cuda()
            cols = [0] + [sum(heads[:i + 1]) for i in range(len(heads))]
            xs = [qkv[:, cols[i] * D:cols[i + 1] * D].view(B, S_l, h, D) for i, h in enumerate(heads)]
        else:
            xs = [random_bytes(torch, (B, S_l, h, D), dt, gen).cuda() for h in heads]
        dev.append(xs)
        host.append([x.cpu() for x in xs])
    return host, dev


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


def run_round_trip(g, B, S_l, heads, D, dt, packed, seed):
    """seq -> heads for every tensor, checked; then heads -> seq of every non-replicated output, into column slices of one packed buffer
    (packed) or dense tensors, checked against the original sources. Returns the stats before and after the first call."""
    torch, n = g.torch, g.n
    host, dev = sources(torch, n, B, S_l, heads, D, dt, packed, seed)
    bases, ys = [], []
    for c in g.comms:
        outs = []
        for h in heads:
            b, y = arena_like(c, (B, n * S_l, ref.local_heads(n, h), D), dt)
            bases.append((c, b))
            outs.append(y)
        poison(outs)
        ys.append(outs)
    torch.cuda.synchronize()
    before = [c.stats() for c in g.comms]
    g.run(lambda r, c, st: c.all_to_all_seq_to_heads(dev[r], ys[r], stream=st))
    after = [c.stats() for c in g.comms]
    what = f"n={n} {dt} B={B} S_l={S_l} heads={heads} D={D} packed={packed}"
    for i in range(len(heads)):
        want = ref.seq_to_heads([host[s][i] for s in range(n)])
        for r in range(n):
            check_bytes(ys[r][i].cpu().view(torch.uint8), want[r].reshape(-1), f"{what} seq->heads tensor {i} rank {r}")
    back_ids = [i for i, h in enumerate(heads) if h % n == 0]
    backs = []
    for c in g.comms:
        if packed:
            width = sum(heads[i] for i in back_ids)
            b, buf = arena_like(c, (B * S_l, width * D), dt)
            bases.append((c, b))
            cols = [0] + [sum(heads[j] for j in back_ids[:k + 1]) for k in range(len(back_ids))]
            outs = [buf[:, cols[k] * D:cols[k + 1] * D].view(B, S_l, heads[i], D) for k, i in enumerate(back_ids)]
            poison([buf])
        else:
            outs = []
            for i in back_ids:
                b, x = arena_like(c, (B, S_l, heads[i], D), dt)
                bases.append((c, b))
                outs.append(x)
            poison(outs)
        backs.append(outs)
    torch.cuda.synchronize()
    g.run(lambda r, c, st: c.all_to_all_heads_to_seq([ys[r][i] for i in back_ids], backs[r], stream=st))
    for k, i in enumerate(back_ids):
        for r in range(n):
            check_bytes(backs[r][k].cpu().contiguous().view(torch.uint8), host[r][i].contiguous().view(torch.uint8).reshape(-1),
                        f"{what} heads->seq(seq->heads) tensor {i} rank {r}")
    for c, b in bases:
        c.release(b)
    return before, after


SHAPES = [(1, 1, 0), (3, 7, 256), (1, 512, 64), (3, 7, 0), (3, 512, 128), (1, 7, 128)]     # (B, S_l, D), D 0: 16 bytes per head


@pytest.mark.parametrize("dtn", DT_NAMES)
@pytest.mark.parametrize("n", [1, 2, 3, 4, 6, 8])
def test_bit_exact_sweep(torch_cuda, groups, n, dtn):
    torch = torch_cuda
    dt = DTYPES[dtn]
    es = torch.empty((), dtype=dt).element_size()
    g = groups(n)
    k = 0
    for name, hq, hkv in head_configs(n):
        for packed in (False, True):
            B, S_l, D = SHAPES[(k + n) % len(SHAPES)]
            D = D or 16 // es
            k += 1
            run_round_trip(g, B, S_l, (hq, hkv, hkv), D, dt, packed, seed=1000 * n + k)
    # one and two tensors in a call
    run_round_trip(g, 3, 7, (2 * n,), 16 // es, dt, False, seed=7)
    run_round_trip(g, 1, 7, (n, n), 128, dt, True, seed=8)


def test_equals_the_unfused_composition(torch_cuda, groups):
    """The outputs equal the composition an attention layer writes without the fused call, byte for byte: permute + contiguous,
    repeat_interleave of K and V up to N heads, one comm.all_to_all per tensor, permute back."""
    torch = torch_cuda
    n, B, S_l, D, dt = 4, 2, 33, 128, torch.bfloat16
    heads = (8, 2, 2)
    g = groups(n)
    _, dev = sources(torch, n, B, S_l, heads, D, dt, True, seed=3)
    fused, bases = [], []
    for c in g.comms:
        row = []
        for h in heads:
            b, y = arena_like(c, (B, n * S_l, ref.local_heads(n, h), D), dt)
            bases.append((c, b))
            row.append(y)
        poison(row)
        fused.append(row)
    torch.cuda.synchronize()
    g.run(lambda r, c, st: c.all_to_all_seq_to_heads(dev[r], fused[r], stream=st))
    for i, h in enumerate(heads):
        hl = ref.local_heads(n, h)
        sends, recvs = [], []
        for r, c in enumerate(g.comms):
            x = dev[r][i]
            if h % n:
                x = x.repeat_interleave(n // h, dim=2)
            s = c.empty(x.numel(), dt)
            s.copy_(x.reshape(B, S_l, n, hl, D).permute(2, 0, 1, 3, 4).reshape(-1))
            rv = c.empty(x.numel(), dt)
            sends.append(s)
            recvs.append(rv)
        torch.cuda.synchronize()
        g.run(lambda r, c, st: c.all_to_all(sends[r], recvs[r], stream=st))
        for r in range(n):
            y = recvs[r].view(n, B, S_l, hl, D).permute(1, 0, 2, 3, 4).reshape(B, n * S_l, hl, D)
            assert torch.equal(y.view(torch.int16), fused[r][i].view(torch.int16)), (i, r)
        for c, s, rv in zip(g.comms, sends, recvs):
            c.release(s)
            c.release(rv)
    for c, b in bases:
        c.release(b)


@pytest.mark.parametrize("dtn,codes", [("bf16", (0x7FC1, 0xFFA5, 0x8000, 0x7F80, 0xFF80, 0x0001)), ("e4m3", (0x7F, 0xFF, 0x80, 0x01, 0x7E))])
def test_special_values(torch_cuda, groups, dtn, codes):
    """NaN payloads, -0, +-inf and denormals come through both directions unchanged."""
    torch = torch_cuda
    n, B, S_l, D = 2, 2, 5, 64
    dt = DTYPES[dtn]
    it = torch.int16 if dt.itemsize == 2 else torch.uint8
    g = groups(n)
    heads = (4, 2)
    xs, ys, backs, bases = [], [], [], []
    for r, c in enumerate(g.comms):
        row = []
        for h in heads:
            bits = torch.tensor(codes, dtype=torch.int32).repeat(B * S_l * h * D // len(codes) + 1)[:B * S_l * h * D]
            row.append(bits.to(it).view(dt).view(B, S_l, h, D).roll(r, dims=3).cuda())
        xs.append(row)
        outs, bk = [], []
        for h in heads:
            b, y = arena_like(c, (B, n * S_l, h // n, D), dt)
            bases.append((c, b))
            outs.append(y)
            b, x = arena_like(c, (B, S_l, h, D), dt)
            bases.append((c, b))
            bk.append(x)
        poison(outs + bk)
        ys.append(outs)
        backs.append(bk)
    torch.cuda.synchronize()
    g.run(lambda r, c, st: c.all_to_all_seq_to_heads(xs[r], ys[r], stream=st))
    g.run(lambda r, c, st: c.all_to_all_heads_to_seq(ys[r], backs[r], stream=st))
    for i in range(len(heads)):
        want = ref.seq_to_heads([xs[s][i].cpu() for s in range(n)])
        for r in range(n):
            check_bytes(ys[r][i].cpu().view(torch.uint8), want[r].reshape(-1), f"{dtn} specials seq->heads {i} rank {r}")
            assert torch.equal(backs[r][i].view(it), xs[r][i].view(it)), (dtn, i, r)
    for c, b in bases:
        c.release(b)


def test_stats_one_launch(torch_cuda, groups):
    torch = torch_cuda
    for n in (1, 4):
        g = groups(n)
        B, S_l, D = 2, 9, 64
        heads = (4 * n, 2, 2) if n == 4 else (4, 2, 2)
        before, after = run_round_trip(g, B, S_l, heads, D, torch.bfloat16, True, seed=11)
        algo = "copy" if n == 1 else "twoshot"
        for b, a in zip(before, after):
            assert a["kernel_launches"] == b["kernel_launches"] + 1
            assert a["calls"][3] == b["calls"][3] + 1 and sum(a["calls"]) == sum(b["calls"]) + 1      # alltoall
            assert a["bytes"][3] - b["bytes"][3] == B * S_l * sum(heads) * D * 2
            assert a["algo_calls"][algo] == b["algo_calls"][algo] + 1 and sum(a["algo_calls"].values()) == sum(b["algo_calls"].values()) + 1


def test_forced_algorithm_changes_nothing(torch_cuda, groups):
    torch = torch_cuda
    g = groups(2)
    for c in g.comms:
        c.set_algo("ll")
    try:
        before, after = run_round_trip(g, 1, 5, (4, 2), 64, torch.float16, False, seed=12)
        assert all(a["algo_calls"]["twoshot"] == b["algo_calls"]["twoshot"] + 1 for b, a in zip(before, after))
    finally:
        for c in g.comms:
            c.set_algo("auto")


def test_back_to_back_without_host_sync(torch_cuda, coll_mod):
    """Three layers on one communicator with no host sync: seq -> heads, a torch op reading the head shards, heads -> seq, the next
    layer's seq -> heads into the same outputs, with an all_to_all, an all_reduce_rms_norm and an expert_dispatch between them, ranks
    launched in a different order every layer, and every source overwritten on its rank's stream right after the call that read it."""
    with Group(torch_cuda, coll_mod, 4, arena_mb=64, timeout_ms=30000) as g:       # a hang fails in 30 s
        _back_to_back(torch_cuda, g)


def _back_to_back(torch, g):
    n, B, S_l, D, dt = 4, 2, 16, 64, torch.bfloat16
    heads = (8, 2, 2)
    layers = 3
    gen = torch.Generator().manual_seed(21)
    srcs = [[[random_bytes(torch, (B, S_l, h, D), dt, gen) for h in heads] for _ in range(n)] for _ in range(layers)]
    # small finite values for the attention stand-in (a doubling stays exact)
    srcs = [[[((x.view(torch.int16) % 64).to(torch.float32) / 8).to(dt) for x in row] for row in layer] for layer in srcs]
    dev = [[x.cuda() for x in row] for row in srcs[0]]
    ys, attn, backs, saved = [], [], [], []
    a2a_in, a2a_out, rms = [], [], []
    for r, c in enumerate(g.comms):
        row = []
        for h in heads:
            _, y = arena_like(c, (B, n * S_l, ref.local_heads(n, h), D), dt)
            row.append(y)
        ys.append(row)
        attn.append(torch.empty(B, n * S_l, heads[0] // n, D, dtype=dt, device="cuda"))
        lb = []
        for _ in range(layers):
            _, x = arena_like(c, (B, S_l, heads[0], D), dt)
            lb.append(x)
        backs.append(lb)
        saved.append([[torch.empty_like(y) for y in row] for _ in range(layers)])
        _, t = arena_like(c, (n * 1024,), dt)
        t.copy_(torch.arange(n * 1024, device="cuda").to(dt) + r)
        a2a_in.append(t)
        _, t = arena_like(c, (n * 1024,), dt)
        a2a_out.append(t)
        _, x = arena_like(c, (8, 256), dt)
        x.fill_(0.5)
        rms.append((x, torch.zeros(8, 256, dtype=dt, device="cuda"), torch.ones(256, dtype=dt, device="cuda"), torch.empty(8, 256, dtype=dt, device="cuda")))
    ex = []
    for r, c in enumerate(g.comms):
        x = torch.full((6, 64), float(r), dtype=dt, device="cuda")
        idx = (torch.arange(12, dtype=torch.int32, device="cuda").view(6, 2) + r) % 8
        _, recv = arena_like(c, (64, 64), dt)
        outs = (torch.empty(8 // n, dtype=torch.int32, device="cuda"), torch.empty(6, 2, dtype=torch.int32, device="cuda"),
                torch.empty(1, dtype=torch.int32, device="cuda"))
        ex.append((x, idx, recv, outs))
    nxt = [[[x.cuda() for x in row] for row in layer] for layer in srcs]
    torch.cuda.synchronize()
    # Each phase is enqueued for every rank before the next, in a rank order that changes from phase to phase: with virtual ranks driven
    # from one thread, a PyTorch kernel's first launch loads its module, which waits for the kernels already running, so it must not be
    # enqueued behind a rank's collective that waits for a peer this thread has not launched yet.
    def copy_in(r, c, st, L):
        for x, s in zip(dev[r], nxt[L][r]):
            x.copy_(s)

    def s2h(r, c, st, L):
        c.all_to_all_seq_to_heads(dev[r], ys[r], stream=st)

    def overwrite_and_read(r, c, st, L):
        for x in dev[r]:
            x.fill_(-7.0)                                                    # the source overwritten right after the call
        for y, s in zip(ys[r], saved[r][L]):
            s.copy_(y)
        torch.mul(ys[r][0], 2, out=attn[r])                                  # the attention stand-in reads the head shards

    def a2a(r, c, st, L):
        c.all_to_all(a2a_in[r], a2a_out[r], stream=st)

    def h2s(r, c, st, L):
        c.all_to_all_heads_to_seq([attn[r]], [backs[r][L]], stream=st)

    def rms_norm(r, c, st, L):
        c.all_reduce_rms_norm(*rms[r], stream=st)

    def dispatch(r, c, st, L):
        xe, idx, recv, (cnt, route, dropped) = ex[r]
        c.expert_dispatch(xe, idx, 8, recv, cnt, route, dropped, stream=st)

    phases = [copy_in, s2h, overwrite_and_read, a2a, h2s, rms_norm, dispatch]
    orders = [list(range(n)), list(reversed(range(n))), [2, 0, 3, 1], [1, 3, 0, 2]]
    for L in range(layers):
        for k, phase in enumerate(phases):
            for r in orders[(L + k) % len(orders)]:
                with torch.cuda.stream(g.streams[r]):
                    phase(r, g.comms[r], g.streams[r], L)
    g.sync()
    g.check_async()
    for L in range(layers):
        for i in range(len(heads)):
            want = ref.seq_to_heads([srcs[L][s][i] for s in range(n)])
            for r in range(n):
                check_bytes(saved[r][L][i].cpu().view(torch.uint8), want[r].reshape(-1), f"layer {L} seq->heads tensor {i} rank {r}")
        for r in range(n):
            assert torch.equal(backs[r][L].cpu(), srcs[L][r][0] * 2), f"layer {L} heads->seq rank {r}"
    for r in range(n):
        want = torch.cat([a2a_in[q][r * 1024:(r + 1) * 1024] for q in range(n)])
        assert torch.equal(a2a_out[r], want), r


def test_cuda_graph_replay(torch_cuda, groups):
    """A graph per rank capturing seq -> heads and heads -> seq, replayed several times with new inputs."""
    torch = torch_cuda
    n, B, S_l, D, dt = 4, 1, 24, 128, torch.bfloat16
    heads = (8, 2, 2)
    g = groups(n)
    dev, ys, backs, bases = [], [], [], []
    for c in g.comms:
        qkv = torch.empty(B * S_l, sum(heads) * D, dtype=dt, device="cuda")
        dev.append((qkv, [qkv[:, a * D:(a + h) * D].view(B, S_l, h, D) for a, h in ((0, 8), (8, 2), (10, 2))]))
        row = []
        for h in heads:
            b, y = arena_like(c, (B, n * S_l, ref.local_heads(n, h), D), dt)
            bases.append((c, b))
            row.append(y)
        ys.append(row)
        b, x = arena_like(c, (B, S_l, heads[0], D), dt)
        bases.append((c, b))
        backs.append(x)
    graphs = [torch.cuda.CUDAGraph() for _ in g.comms]
    torch.cuda.synchronize()
    for r, c in enumerate(g.comms):
        with torch.cuda.graph(graphs[r], stream=g.streams[r]):
            c.all_to_all_seq_to_heads(dev[r][1], ys[r], stream=g.streams[r])
            c.all_to_all_heads_to_seq(ys[r][:1], [backs[r]], stream=g.streams[r])
    torch.cuda.synchronize()
    for it in range(3):
        gen = torch.Generator().manual_seed(300 + it)
        host = []
        for r in range(n):
            hq = random_bytes(torch, (B * S_l, sum(heads) * D), dt, gen)
            dev[r][0].copy_(hq.cuda())
            host.append([hq[:, a * D:(a + h) * D].reshape(B, S_l, h, D) for a, h in ((0, 8), (8, 2), (10, 2))])
        poison([y for row in ys for y in row] + backs)
        torch.cuda.synchronize()
        for r in range(n):
            with torch.cuda.stream(g.streams[r]):
                graphs[r].replay()
        torch.cuda.synchronize()
        g.check_async()
        for i in range(3):
            want = ref.seq_to_heads([host[s][i] for s in range(n)])
            for r in range(n):
                check_bytes(ys[r][i].cpu().view(torch.uint8), want[r].reshape(-1), f"replay {it} tensor {i} rank {r}")
        for r in range(n):
            assert torch.equal(backs[r].cpu().view(torch.int16), host[r][0].view(torch.int16)), (it, r)
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
        B, S_l, D = 2, 4, 64
        qkv = torch.zeros(B * S_l, 12 * D, dtype=dt, device="cuda")
        yb = c.empty(1 << 16, dt)
        plain = torch.zeros(1 << 16, dtype=dt, device="cuda")
        q_out = yb.data_ptr()
        T = coll.UlyssesTensor

        def call(fn=L.b200collAllToAllSeqToHeads, tensors=None, nt=None, batch=B, seq_local=S_l, head_dim=D, dtype=BF16):
            ts = tensors if tensors is not None else [T(qkv.data_ptr(), 12 * D, q_out, 8)]
            arr = (T * max(len(ts), 1))(*ts)
            return fn(arr, len(ts) if nt is None else nt, batch, seq_local, head_dim, dtype, c._h, C.c_void_p(0))

        q, k = qkv.data_ptr(), qkv.data_ptr() + 8 * D * 2
        cases = [
            (dict(nt=0), INVALID_ARGUMENT, "ntensors must be 1, 2 or 3"),
            (dict(nt=4), INVALID_ARGUMENT, "ntensors must be 1, 2 or 3"),
            (dict(dtype=coll.I32), INVALID_ARGUMENT, "dtype must be"),
            (dict(head_dim=4), INVALID_ARGUMENT, "head_dim * sizeof(dtype)"),
            (dict(tensors=[T(q, 12 * D, q_out, 0)]), INVALID_ARGUMENT, "heads must be positive"),
            (dict(tensors=[T(q, 12 * D, q_out, 3)]), INVALID_ARGUMENT, "multiple or a divisor of nranks"),
            (dict(tensors=[T(q, 4 * D, q_out, 8)]), INVALID_ARGUMENT, "row_stride must be at least"),
            (dict(tensors=[T(q, 12 * D + 4, q_out, 8)]), INVALID_ARGUMENT, "multiple of 16 bytes"),
            (dict(tensors=[T(q + 2, 12 * D, q_out, 8)]), INVALID_ARGUMENT, "16-byte aligned"),
            (dict(tensors=[T(0, 12 * D, q_out, 8)]), INVALID_ARGUMENT, "null pointer"),
            (dict(batch=1 << 31), INVALID_ARGUMENT, "below 2^31"),
            (dict(seq_local=1 << 30, batch=1), INVALID_ARGUMENT, "2^31 - 1"),
            (dict(tensors=[T(q, 1 << 40, q_out, 8)]), INVALID_ARGUMENT, "2^31 - 1"),
            (dict(tensors=[T(q, 12 * D, q + 64, 8)]), INVALID_ARGUMENT, "output 0 overlaps source 0"),
            (dict(tensors=[T(q, 12 * D, q_out, 8), T(k, 12 * D, q_out + 64, 2)]), INVALID_ARGUMENT, "outputs 0 and 1 overlap"),
            (dict(fn=L.b200collAllToAllHeadsToSeq, tensors=[T(q_out, 12 * D, k, 1)]), INVALID_ARGUMENT, "the replicated layout has no inverse"),
            (dict(tensors=[T(q, 12 * D, plain.data_ptr(), 8)]), INVALID_USAGE, "symmetric arena"),
            (dict(fn=L.b200collAllToAllHeadsToSeq, tensors=[T(q, 12 * D, q_out, 8)]), INVALID_USAGE, "symmetric arena"),
        ]
        torch.cuda.synchronize()
        for kw, code, msg in cases:
            prefix = "all-to-all heads->seq: " if kw.get("fn") is L.b200collAllToAllHeadsToSeq else "all-to-all seq->heads: "
            expect_refused(call(**kw), code, msg, prefix=prefix, what=(msg, kw))
        # B * S_l == 0 returns at once, with nothing launched
        assert call(batch=0) == 0 and call(seq_local=0) == 0
        assert_nothing_launched(c)
        c.release(yb)


@pytest.mark.parametrize("devs,dtype,spec,extra", [("0", "bfloat16", "64:8:128", []), ("0", "e4m3", "32:8:128", ["--ulysses-back"]),
                                                   ("0,0", "half", "32:8:128", []), ("0,0,0,0", "bfloat16", "32:2:128", []),
                                                   ("0,0,0,0", "float", "64:1:64", []), ("0,0,0,0", "bfloat16", "64:8:128", ["--ulysses-back"])])
def test_perf_tool_checks_every_byte(torch_cuda, coll_lib, devs, dtype, spec, extra):
    out = run_perf(["--op", "alltoall", "-d", dtype, "--ulysses", spec, *extra, "-b", "64K", "-e", "4M", "-f", "4", "-w", "1", "-n", "2", "-c", "1"],
                   devs, env={"B200COLL_TIMEOUT_MS": "20000"})
    assert "ulysses" in out, out
    n = len(devs.split(","))
    rows = [l for l in out.splitlines() if l and not l.startswith("#")]
    assert rows and all(l.split()[3] == ("copy" if n == 1 else "twoshot") for l in rows), out


def test_multi_gpu_perf_tool_processes_cross_checked(torch_cuda, coll_lib):
    """One process per GPU with B200COLL_CHECK=1: the ranks exchange the direction, shapes, heads, row strides and output offsets before
    every launch, and every byte is checked."""
    torch = torch_cuda
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    devs = ",".join(str(i) for i in range(n))
    for spec, extra in (("32:8:128", []), ("32:1:128", []), ("32:8:128", ["--ulysses-back"])):
        run_perf(["--op", "alltoall", "-d", "bfloat16", "--ulysses", spec, *extra, "-b", "1M", "-e", "16M", "-f", "4", "-w", "1", "-n", "3", "-c", "1"],
                 devs, procs=True, env={"B200COLL_CHECK": "1", "B200COLL_TIMEOUT_MS": "20000"}, timeout=300)
