"""The FSDP shard all-gather and reduce-scatter (b200collAllGatherShards / ReduceScatterShards) on an H100 (`pytest -m gpu`), virtual
ranks sharing cuda:0 unless a test says otherwise.

Bit-copy gather sources are random bytes, so NaN payloads, -0 and inf occur in every float type and every rank's bytes differ; cast
sources are random fp32 bits (subnormals, overflow to inf and NaN included). Reduce-scatter gradients come from
coll_fp_reference.gen_inputs, which tells summation orders apart, and old shards from a seeded normal. Outputs are poisoned first,
padding rows of a shard must stay poisoned, and everything is compared with tests/coll_shards_reference."""
import ctypes as C

import pytest

from container_engine_accelerators_b200.ops.coll import INVALID_ARGUMENT, INVALID_USAGE
from tests import coll_context_reference as cref
from tests import coll_fp_reference as R
from tests import coll_shards_reference as ref
from tests.coll_gpu_harness import (DTYPES, Group, assert_nothing_launched, coll_mod, expect_refused, poison, run_perf,  # noqa: F401
                                    torch_cuda)

pytestmark = pytest.mark.gpu

GATHER_PAIRS = [("f32", "bf16"), ("f32", "f16"), ("bf16", "bf16"), ("f16", "f16"), ("f32", "f32"), ("e4m3", "e4m3"), ("e5m2", "e5m2")]
RS_PAIRS = [("bf16", "bf16"), ("f16", "f16"), ("f32", "f32"), ("bf16", "f32"), ("f16", "f32")]
# d not divisible by N, a 1-D tensor, a 3-D one, a 1-row one and a 3-row one (ranks with no rows from N = 4 on); d * W a multiple of 16
UNIT = [(24, 16), (7, 16), (48,), (5, 4, 8), (1, 32), (3, 16)]
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


def numel(shape):
    n = 1
    for d in shape:
        n *= d
    return n


def rows_per_rank(shape, n, es_min):
    """FSDP2's ceil(d / N), rounded up until p * W is a whole number of 16-byte vectors in the narrower dtype."""
    d, W = shape[0], numel(shape[1:])
    p = ref.default_rows(d, n)
    while (p * W * es_min) % 16:
        p += 1
    return p


def random_bytes(torch, shape, dt, gen):
    es = torch.empty((), dtype=dt).element_size()
    return torch.randint(0, 256, (numel(shape) * es,), dtype=torch.uint8, generator=gen).view(dt).view(shape)


def arena(c, shape, dt):
    """An arena tensor of `shape` and the base to release."""
    base = c.empty(max(numel(shape), 1), dt)
    return base, base[:numel(shape)].view(shape)


def release(bases):
    for c, b in bases:
        c.release(b)


def make_shards(torch, n, shapes, ps, host_rows, sdt, device="cuda"):
    """Per rank, per tensor: a [p, ...] shard whose first n_r rows are host_rows[r][i] and whose padding is poisoned."""
    out = []
    for r in range(n):
        row = []
        for i, (sh, p) in enumerate(zip(shapes, ps)):
            x = torch.empty((p, *sh[1:]), dtype=sdt, device=device)
            poison([x])
            k = ref.shard_range(sh[0], p, r)[1]
            if k:
                x[:k].copy_(host_rows[r][i])
            row.append(x)
        out.append(row)
    return out


def run_gather(g, shapes, sdt, fdt, seed, ps=None, host=None):
    """One all_gather_shards of `shapes` on every rank, checked against the reference. host: per rank, per tensor, the n_r source rows
    (default: random bytes, or random fp32 bits for a cast). Returns (stats before, stats after)."""
    torch, n = g.torch, g.n
    es_min = min(R.esize(sdt), R.esize(fdt))
    ps = ps or [rows_per_rank(sh, n, es_min) for sh in shapes]
    gen = torch.Generator().manual_seed(seed)
    if host is None:
        host = [[random_bytes(torch, (ref.shard_range(sh[0], p, r)[1], *sh[1:]), sdt, gen) for sh, p in zip(shapes, ps)] for r in range(n)]
    shards = make_shards(torch, n, shapes, ps, host, sdt)
    bases, fulls = [], []
    for c in g.comms:
        row = []
        for sh in shapes:
            b, f = arena(c, sh, fdt)
            bases.append((c, b))
            row.append(f)
        poison(row)
        fulls.append(row)
    torch.cuda.synchronize()
    before = [c.stats() for c in g.comms]
    g.run(lambda r, c, st: c.all_gather_shards(shards[r], fulls[r], shard_rows=ps, stream=st))
    after = [c.stats() for c in g.comms]
    what = f"n={n} {sdt}->{fdt}"
    for i, sh in enumerate(shapes):
        want = ref.all_gather([host[s][i] for s in range(n)], sh[0], fdt, ps[i])
        for r in range(n):
            R.assert_same(fulls[r][i].cpu(), want, f"{what} tensor {i} {sh} rank {r}", nan_payloads=sdt == fdt)
    release(bases)
    return before, after


def run_rs(g, shapes, fdt, sdt, scale, accumulate, seed, ps=None, inputs=None, olds=None):
    """One reduce_scatter_shards of `shapes` on every rank into [p, ...] shards with poisoned padding (which must stay so), checked
    against the reference. inputs: per rank, per tensor, the [d, ...] gradients on the host (default gen_inputs); olds: per rank, per
    tensor, the n_r old shard rows (default a seeded normal). Returns (stats before, stats after)."""
    torch, n = g.torch, g.n
    es_min = min(R.esize(sdt), R.esize(fdt))
    ps = ps or [rows_per_rank(sh, n, es_min) for sh in shapes]
    gen = torch.Generator().manual_seed(seed)
    if inputs is None:
        per = [R.gen_inputs(n, numel(sh), fdt, seed + i, device="cpu") for i, sh in enumerate(shapes)]
        inputs = [[per[i][r].view(sh) for i, sh in enumerate(shapes)] for r in range(n)]
    if olds is None:
        olds = [[(torch.randn((ref.shard_range(sh[0], p, r)[1], *sh[1:]), generator=gen) * 4).to(sdt) for sh, p in zip(shapes, ps)]
                for r in range(n)]
    shards = make_shards(torch, n, shapes, ps, olds, sdt)
    bases, fulls = [], []
    for r, c in enumerate(g.comms):
        row = []
        for i, sh in enumerate(shapes):
            b, f = arena(c, sh, fdt)
            bases.append((c, b))
            f.copy_(inputs[r][i])
            row.append(f)
        fulls.append(row)
    torch.cuda.synchronize()
    before = [c.stats() for c in g.comms]
    g.run(lambda r, c, st: c.reduce_scatter_shards(fulls[r], shards[r], scale=scale, accumulate=accumulate, shard_rows=ps, stream=st))
    after = [c.stats() for c in g.comms]
    what = f"n={n} {fdt}->{sdt} scale={scale} accumulate={accumulate}"
    bit_copy = n == 1 and fdt == sdt and scale == 1.0 and not accumulate
    for i, sh in enumerate(shapes):
        want = ref.reduce_scatter([inputs[s][i] for s in range(n)], sdt, scale, [o[i] for o in olds] if accumulate else None, ps[i])
        for r in range(n):
            k = want[r].shape[0]
            got = shards[r][i].cpu()
            R.assert_same(got[:k], want[r], f"{what} tensor {i} {sh} rank {r}", nan_payloads=bit_copy)
            assert bool((got[k:].contiguous().view(-1).view(torch.uint8) == 0x7B).all()), f"{what} tensor {i} rank {r}: padding written"
    release(bases)
    return before, after


# ------------------------------------------------------------------------------------------------- bit-exact sweeps
@pytest.mark.parametrize("pair", GATHER_PAIRS, ids=lambda p: "->".join(p))
@pytest.mark.parametrize("n", [1, 2, 3, 4, 6, 8])
def test_gather_bit_exact_sweep(groups, n, pair):
    run_gather(groups(n), UNIT, DTYPES[pair[0]], DTYPES[pair[1]], seed=100 * n + GATHER_PAIRS.index(pair))


@pytest.mark.parametrize("pair", RS_PAIRS, ids=lambda p: "->".join(p))
@pytest.mark.parametrize("n", [1, 2, 3, 4, 6, 8])
def test_reduce_scatter_bit_exact_sweep(groups, n, pair):
    g = groups(n)
    for k, (accumulate, scale) in enumerate(((False, 1.0), (False, 1.0 / n), (True, 1.0), (True, 1.0 / n))):
        run_rs(g, UNIT, DTYPES[pair[0]], DTYPES[pair[1]], scale, accumulate, seed=1000 * n + 10 * RS_PAIRS.index(pair) + k)


# ------------------------------------------------------------------------------------------------- special values
def test_gather_cast_special_values(torch_cuda, groups):
    """NaN, +-inf, -0, subnormals and fp16 overflow through the fp32 -> bf16 / fp16 cast: exactly what Tensor.to gives (NaN by
    position)."""
    torch = torch_cuda
    vals = torch.tensor([float("nan"), float("inf"), float("-inf"), -0.0, 0.0, 65504.0, 65519.0, 65520.0, 70000.0, -1e9, 1e-40, -3e-39,
                         5.96e-8, 2.9e-8, 3.3895e38, 3.4e38], dtype=torch.float32)
    for n in (1, 2, 3):
        g = groups(n)
        shapes = [(4 * n, 16)]
        for fdt in (torch.bfloat16, torch.float16):
            host = [[vals.repeat(4, 1)[:ref.shard_range(4 * n, 4, r)[1]] * (1 + r)] for r in range(n)]
            run_gather(g, shapes, torch.float32, fdt, seed=0, ps=[4], host=host)
    assert torch.tensor([70000.0]).to(torch.float16).isinf().all() and torch.tensor([65519.0]).to(torch.float16).item() == 65504.0


@pytest.mark.parametrize("pair", RS_PAIRS, ids=lambda p: "->".join(p))
def test_reduce_scatter_special_values(torch_cuda, groups, pair):
    """+-inf, NaN, inf - inf, -0 on every rank (+0 from a sum that starts at +0; -0 kept by the one-rank bit copy), fp16 overflow of
    the sum, and accumulation into -0 and inf."""
    torch = torch_cuda
    fdt, sdt = DTYPES[pair[0]], DTYPES[pair[1]]
    for n in (1, 2, 4):
        g = groups(n)
        d, W = 2 * n, 16
        inputs = []
        for r in range(n):
            f = torch.full((d, W), -0.0)
            f[:, 1] = float("inf")
            f[:, 2] = float("inf") if r % 2 == 0 else float("-inf")
            f[:, 3] = float("nan") if r == n - 1 else 1.0
            f[:, 4] = 1.5 * (r + 1)
            f[:, 5] = 60000.0
            inputs.append([f.to(fdt)])
        olds = [[torch.tensor([-0.0, 1.0, 2.0, 3.0, float("inf"), -1.0] + [0.25] * 10).repeat(2, 1).to(sdt)] for _ in range(n)]
        for scale, acc in ((1.0, False), (0.5, False), (1.0, True)):
            run_rs(g, [(d, W)], fdt, sdt, scale, acc, seed=0, ps=[2], inputs=inputs, olds=olds)


# ------------------------------------------------------------------------------------------------- FSDP2's own composition
def _fsdp2_gather(torch, g, shards32, d_list, p_list, W_list, fdt):
    """FSDP2's all-gather: the per-parameter cast, all_gather_copy_in into the flat input, comm.all_gather, and split_with_sizes_copy
    into the padded unsharded parameters, narrowed to d rows."""
    import torch.distributed.fsdp._fully_shard._fsdp_collectives  # noqa: F401  (registers torch.ops.fsdp)
    n = g.n
    sizes = [p * W for p, W in zip(p_list, W_list)]
    numel_in = sum(sizes)
    bases, ins, outs = [], [], []
    for c in g.comms:
        b, x = arena(c, (numel_in,), fdt)
        bases.append((c, b))
        ins.append(x)
        b, y = arena(c, (n * numel_in,), fdt)
        bases.append((c, b))
        outs.append(y)
    params = [[torch.empty((n * p, W), dtype=fdt, device="cuda") for p, W in zip(p_list, W_list)] for _ in range(n)]
    for r in range(n):
        cast = [x.to(fdt).reshape(-1) for x in shards32[r]]
        torch.ops.fsdp.all_gather_copy_in(cast, ins[r], sizes, numel_in, 0)
    torch.cuda.synchronize()
    g.run(lambda r, c, st: c.all_gather(ins[r], outs[r], stream=st))
    for r in range(n):
        torch.ops.fsdp.split_with_sizes_copy(outs[r].view(n, -1), sizes, dim=1, out=[q.view(n, -1) for q in params[r]])
    torch.cuda.synchronize()
    release(bases)
    return [[q[:d] for q, d in zip(row, d_list)] for row in params]


def test_equals_the_fsdp2_composition(torch_cuda, groups):
    """The gather equals FSDP2's cast, copy-in, all-gather and copy-out byte for byte; the reduce-scatter with accumulation equals its
    chunk_cat (with the fp32 cast of reduce_dtype), reduce-scatter, divide and _foreach_add_, on gradients whose sums are exact."""
    import torch.distributed.fsdp._fully_shard._fsdp_collectives  # noqa: F401
    torch = torch_cuda
    n = 4
    g = groups(n)
    shapes = [(40, 32), (10, 32), (10, 32), (40, 32), (96, 32), (96, 32), (32, 96), (32,), (32,)]
    d_list = [s[0] for s in shapes]
    W_list = [numel(s[1:]) for s in shapes]
    p_list = [ref.default_rows(d, n) for d in d_list]
    gen = torch.Generator().manual_seed(7)
    shards32 = [[torch.randn((p, W), generator=gen).cuda() for p, W in zip(p_list, W_list)] for _ in range(n)]
    for r in range(n):                                   # FSDP2 pads with zeros; the fused call never reads the padding
        for x, d, p in zip(shards32[r], d_list, p_list):
            x[max(0, min(p, d - r * p)):] = 0
    composed = _fsdp2_gather(torch, g, shards32, d_list, p_list, W_list, torch.bfloat16)
    bases, fused = [], []
    for c in g.comms:
        row = []
        for sh in shapes:
            b, f = arena(c, sh, torch.bfloat16)
            bases.append((c, b))
            row.append(f)
        fused.append(row)
    shards_view = [[x.view((x.shape[0], *sh[1:])) for x, sh in zip(row, shapes)] for row in shards32]
    g.run(lambda r, c, st: c.all_gather_shards(shards_view[r], fused[r], stream=st))
    for r in range(n):
        for i in range(len(shapes)):
            assert torch.equal(fused[r][i].reshape(d_list[i], -1).view(torch.int16), composed[r][i].view(torch.int16)), (r, i)
    # reduce-scatter: bf16 gradients that are multiples of 1/8 below 16, so every fp32 sum and the 1/N are exact
    grads = [[((torch.randint(-128, 128, sh, generator=gen).float() / 8).to(torch.bfloat16)).cuda() for sh in shapes] for _ in range(n)]
    old = [[torch.randint(-64, 64, (p, W), generator=gen).float().cuda() / 4 for p, W in zip(p_list, W_list)] for _ in range(n)]
    chunk = sum(p * W for p, W in zip(p_list, W_list))
    rs_bases, rs_in, rs_out = [], [], []
    for c in g.comms:
        b, x = arena(c, (n * chunk,), torch.float32)
        rs_bases.append((c, b))
        rs_in.append(x)
        b, y = arena(c, (chunk,), torch.float32)
        rs_bases.append((c, b))
        rs_out.append(y)
    for r in range(n):
        torch.ops.fsdp.chunk_cat([x.float().reshape(x.shape[0], -1) for x in grads[r]], 0, n, out=rs_in[r].view(n, -1))
    torch.cuda.synchronize()
    g.run(lambda r, c, st: c.reduce_scatter(rs_in[r], rs_out[r], stream=st))
    composed = []
    for r in range(n):
        rs_out[r].div_(n)
        parts = torch.split(rs_out[r], [p * W for p, W in zip(p_list, W_list)])
        acc = [o.clone() for o in old[r]]
        torch._foreach_add_(acc, [q.view(p, W) for q, p, W in zip(parts, p_list, W_list)])
        composed.append(acc)
    torch.cuda.synchronize()
    gfull = []                                          # the fused call pulls the gradients from the arena
    for r, c in enumerate(g.comms):
        row = []
        for x in grads[r]:
            b, f = arena(c, tuple(x.shape), torch.bfloat16)
            bases.append((c, b))
            f.copy_(x)
            row.append(f)
        gfull.append(row)
    outs = [[o.clone().view((o.shape[0], *sh[1:])) for o, sh in zip(old[r], shapes)] for r in range(n)]
    torch.cuda.synchronize()
    g.run(lambda r, c, st: c.reduce_scatter_shards(gfull[r], outs[r], scale=1.0 / n, accumulate=True, stream=st))
    for r in range(n):
        for i, (d, p) in enumerate(zip(d_list, p_list)):
            k = ref.shard_range(d, p, r)[1]
            assert torch.equal(outs[r][i].reshape(p, -1)[:k], composed[r][i][:k]), (r, i)
    release(bases + rs_bases)


def test_reduce_scatter_of_the_gather(torch_cuda, groups):
    """Every rank feeds the gathered parameters back as its gradient: the reduce-scatter gives each rank N times its own shard (exact
    for these values), and the reference agrees."""
    torch = torch_cuda
    for n, dt in ((2, torch.bfloat16), (3, torch.float16), (8, torch.float32)):
        g = groups(n)
        shapes = [(37, 16), (64,), (6, 2, 8)]
        ps = [rows_per_rank(sh, n, R.esize(dt)) for sh in shapes]
        gen = torch.Generator().manual_seed(n)
        host = [[(torch.randint(-64, 64, (ref.shard_range(sh[0], p, r)[1], *sh[1:]), generator=gen).float() / 4).to(dt)
                 for sh, p in zip(shapes, ps)] for r in range(n)]
        shards = make_shards(torch, n, shapes, ps, host, dt)
        bases, fulls = [], []
        for c in g.comms:
            row = []
            for sh in shapes:
                b, f = arena(c, sh, dt)
                bases.append((c, b))
                row.append(f)
            fulls.append(row)
        torch.cuda.synchronize()
        g.run(lambda r, c, st: c.all_gather_shards(shards[r], fulls[r], shard_rows=ps, stream=st))
        outs = make_shards(torch, n, shapes, ps, host, dt)
        g.run(lambda r, c, st: c.reduce_scatter_shards(fulls[r], outs[r], shard_rows=ps, stream=st))
        for r in range(n):
            for i in range(len(shapes)):
                k = host[r][i].shape[0]
                assert torch.equal(outs[r][i][:k].cpu(), (host[r][i].float() * n).to(dt)), (n, r, i)
        release(bases)


# ------------------------------------------------------------------------------------------------- stats, refusals, graphs
def test_stats_one_launch(torch_cuda, groups):
    torch = torch_cuda
    for n in (1, 4):
        g = groups(n)
        shapes = [(10, 16), (3, 16)]
        algo = "copy" if n == 1 else "twoshot"
        for op, fdt, (before, after) in ((1, torch.bfloat16, run_gather(g, shapes, torch.float32, torch.bfloat16, seed=3)),
                                         (2, torch.bfloat16, run_rs(g, shapes, torch.bfloat16, torch.float32, 0.5, True, seed=4))):
            for r, (b, a) in enumerate(zip(before, after)):
                mine = sum(ref.shard_range(sh[0], rows_per_rank(sh, n, 2), r)[1] * numel(sh[1:]) for sh in shapes) * 2
                assert a["kernel_launches"] == b["kernel_launches"] + 1
                assert a["calls"][op] == b["calls"][op] + 1 and sum(a["calls"]) == sum(b["calls"]) + 1
                assert a["bytes"][op] - b["bytes"][op] == mine, (n, r, op)
                assert a["algo_calls"][algo] == b["algo_calls"][algo] + 1 and sum(a["algo_calls"].values()) == sum(b["algo_calls"].values()) + 1


def test_refusals_launch_nothing(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    L = coll.load()
    with Group(torch, coll, 2) as g:
        c = g.comms[0]
        F32, BF16, F16 = (coll.torch_dtype_code(t) for t in (torch.float32, torch.bfloat16, torch.float16))
        E4M3 = coll.torch_dtype_code(torch.float8_e4m3fn)
        fb = c.empty(1 << 16, torch.bfloat16)
        plain = torch.zeros(1 << 16, dtype=torch.bfloat16, device="cuda")
        sb = torch.zeros(1 << 16, dtype=torch.float32, device="cuda")
        full, shard = fb.data_ptr(), sb.data_ptr()
        T = coll.ShardTensor
        AG, RS = L.b200collAllGatherShards, L.b200collReduceScatterShards

        def call(fn=AG, tensors=None, nt=None, a=F32, b=BF16, scale=1.0, acc=0):
            ts = tensors if tensors is not None else [T(shard, full, 64, 16, 32)]
            arr = (T * max(len(ts), 1))(*ts)
            nt = len(ts) if nt is None else nt
            if fn is AG:
                return fn(arr, nt, a, b, c._h, C.c_void_p(0))
            return fn(arr, nt, a, b, C.c_float(scale), acc, c._h, C.c_void_p(0))

        cases = [
            (dict(nt=0), INVALID_ARGUMENT, "ntensors must be 1 to 64"),
            (dict(nt=65), INVALID_ARGUMENT, "ntensors must be 1 to 64"),
            (dict(a=BF16, b=F32), INVALID_ARGUMENT, "dtype pair"),
            (dict(a=F16, b=BF16), INVALID_ARGUMENT, "dtype pair"),
            (dict(a=coll.I32, b=coll.I32), INVALID_ARGUMENT, "dtype pair"),
            (dict(fn=RS, a=F32, b=BF16), INVALID_ARGUMENT, "dtype pair"),
            (dict(fn=RS, a=E4M3, b=E4M3), INVALID_ARGUMENT, "dtype pair"),
            (dict(tensors=[T(shard, full, 0, 16, 32)]), INVALID_ARGUMENT, "must be positive"),
            (dict(tensors=[T(shard, full, 64, 0, 32)]), INVALID_ARGUMENT, "must be positive"),
            (dict(tensors=[T(shard, full, 64, 16, 0)]), INVALID_ARGUMENT, "must be positive"),
            (dict(tensors=[T(shard, full, 64, 16, 31)]), INVALID_ARGUMENT, "nranks * shard_rows must be at least rows"),
            (dict(tensors=[T(shard, full, 64, 1, 33)]), INVALID_ARGUMENT, "multiples of 16 bytes"),
            (dict(tensors=[T(shard, full, 63, 1, 32)]), INVALID_ARGUMENT, "multiples of 16 bytes"),
            (dict(tensors=[T(shard + 4, full, 64, 16, 32)]), INVALID_ARGUMENT, "16-byte aligned"),
            (dict(tensors=[T(shard, full + 2, 64, 16, 32)]), INVALID_ARGUMENT, "16-byte aligned"),
            (dict(tensors=[T(0, full, 64, 16, 32)]), INVALID_ARGUMENT, "null pointer"),
            (dict(tensors=[T(shard, 0, 64, 16, 32)]), INVALID_ARGUMENT, "null pointer"),
            (dict(tensors=[T(shard, full, 1 << 31, 16, 1 << 30)]), INVALID_ARGUMENT, "2^31 - 1"),
            (dict(tensors=[T(shard, full, (1 << 29) - 8, 16, (1 << 28) - 4)] * 5), INVALID_ARGUMENT, "2^31 - 1 16-byte vectors in the call"),
            (dict(tensors=[T(full + 1024, full, 64, 16, 32)], a=BF16, b=BF16), INVALID_ARGUMENT, "output 0 overlaps source 0"),
            (dict(tensors=[T(shard, full, 64, 16, 32), T(shard + 8192, full + 64, 64, 16, 32)]), INVALID_ARGUMENT, "outputs 0 and 1 overlap"),
            (dict(fn=RS, a=BF16, b=F32, tensors=[T(shard, full, 64, 16, 32), T(shard + 64, full + 4096, 64, 16, 32)]), INVALID_ARGUMENT,
             "outputs 0 and 1 overlap"),
            (dict(tensors=[T(shard, plain.data_ptr(), 64, 16, 32)]), INVALID_USAGE, "symmetric arena"),
            (dict(fn=RS, a=BF16, b=F32, tensors=[T(shard, plain.data_ptr(), 64, 16, 32)]), INVALID_USAGE, "symmetric arena"),
        ]
        torch.cuda.synchronize()
        for kw, code, msg in cases:
            prefix = "reduce-scatter shards: " if kw.get("fn") is RS else "all-gather shards: "
            expect_refused(call(**kw), code, msg, prefix=prefix, what=(msg, kw))
        assert_nothing_launched(c)
        c.release(fb)


def test_cuda_graph_replay(torch_cuda, groups):
    """A graph per rank capturing the gather of a unit's parameters (fp32 -> bf16) and the accumulating reduce-scatter of its
    gradients (bf16 -> fp32, scale 1/N), replayed several times with new inputs."""
    torch = torch_cuda
    n = 4
    g = groups(n)
    shapes = [(24, 16), (48,), (3, 16)]
    ps = [rows_per_rank(sh, n, 2) for sh in shapes]
    bases, fulls, grads, shards, gshards = [], [], [], [], []
    for r, c in enumerate(g.comms):
        fr, gr = [], []
        for sh in shapes:
            b, f = arena(c, sh, torch.bfloat16)
            bases.append((c, b))
            fr.append(f)
            b, f = arena(c, sh, torch.bfloat16)
            bases.append((c, b))
            gr.append(f)
        fulls.append(fr)
        grads.append(gr)
        shards.append([torch.zeros((p, *sh[1:]), device="cuda") for sh, p in zip(shapes, ps)])
        gshards.append([torch.zeros((p, *sh[1:]), device="cuda") for sh, p in zip(shapes, ps)])
    graphs = [torch.cuda.CUDAGraph() for _ in g.comms]
    torch.cuda.synchronize()
    for r, c in enumerate(g.comms):
        with torch.cuda.graph(graphs[r], stream=g.streams[r]):
            c.all_gather_shards(shards[r], fulls[r], shard_rows=ps, stream=g.streams[r])
            c.reduce_scatter_shards(grads[r], gshards[r], scale=1.0 / n, accumulate=True, shard_rows=ps, stream=g.streams[r])
    torch.cuda.synchronize()
    for it in range(3):
        gen = torch.Generator().manual_seed(300 + it)
        hs, hg, olds = [], [], []
        for r in range(n):
            hs.append([torch.randn((p, *sh[1:]), generator=gen) for sh, p in zip(shapes, ps)])
            hg.append([x.view(sh) for x, sh in zip((R.gen_inputs(1, numel(sh), torch.bfloat16, seed=500 + 10 * it + r + j, device="cpu")[0]
                                                    for j, sh in enumerate(shapes)), shapes)])
            olds.append([x.cpu() for x in gshards[r]])
            for d, s in zip(shards[r], hs[r]):
                d.copy_(s)
            for d, s in zip(grads[r], hg[r]):
                d.copy_(s)
        poison([f for row in fulls for f in row])
        torch.cuda.synchronize()
        for r in range(n):
            with torch.cuda.stream(g.streams[r]):
                graphs[r].replay()
        torch.cuda.synchronize()
        g.check_async()
        for i, sh in enumerate(shapes):
            want = ref.all_gather([hs[s][i] for s in range(n)], sh[0], torch.bfloat16, ps[i])
            back = ref.reduce_scatter([hg[s][i] for s in range(n)], torch.float32, 1.0 / n, [o[i] for o in olds], ps[i])
            for r in range(n):
                R.assert_same(fulls[r][i].cpu(), want, f"replay {it} gather {i} rank {r}")
                R.assert_same(gshards[r][i][:back[r].shape[0]].cpu(), back[r], f"replay {it} reduce-scatter {i} rank {r}")
    del graphs
    torch.cuda.synchronize()
    release(bases)


# ------------------------------------------------------------------------------------------------- back to back with every family
def test_back_to_back_without_host_sync(torch_cuda, coll_mod):
    """Three layers on one communicator with no host sync: the unit's parameter gather, a torch op reading the parameters and writing
    their gradient, the gradient's accumulating reduce-scatter, with a context-parallel gather, a Ulysses all-to-all, a
    reduce_scatter_rms_norm and an expert dispatch and combine between them, ranks launched in a different order every phase, and the
    shards overwritten on their rank's stream right after the gather that read them."""
    with Group(torch_cuda, coll_mod, 4, arena_mb=64, timeout_ms=30000) as g:       # a hang fails in 30 s
        _back_to_back(torch_cuda, g)


def _back_to_back(torch, g):
    n, layers = 4, 3
    shapes = [(24, 16), (48,), (3, 16)]
    ps = [rows_per_rank(sh, n, 2) for sh in shapes]
    gen = torch.Generator().manual_seed(31)
    # multiples of 1/8 below 8: bf16 exact, and every doubled sum over 4 ranks exact in fp32
    srcs = [[[(torch.randint(-64, 64, (p, *sh[1:]), generator=gen).float() / 8) for sh, p in zip(shapes, ps)] for _ in range(n)]
            for _ in range(layers)]
    shards = [[torch.empty((p, *sh[1:]), device="cuda") for sh, p in zip(shapes, ps)] for _ in range(n)]
    gshards = [[[torch.full((p, *sh[1:]), 0.5, device="cuda") for sh, p in zip(shapes, ps)] for _ in range(layers)] for _ in range(n)]
    fulls, grads, saved = [], [], []
    cp_kv, cp_full, uly_x, uly_y, rms, ex = [], [], [], [], [], []
    for r, c in enumerate(g.comms):
        fulls.append([arena(c, sh, torch.bfloat16)[1] for sh in shapes])
        grads.append([arena(c, sh, torch.bfloat16)[1] for sh in shapes])
        saved.append([[torch.empty(sh, dtype=torch.bfloat16, device="cuda") for sh in shapes] for _ in range(layers)])
        cp_kv.append(torch.arange(8 * 64, device="cuda").to(torch.bfloat16).view(1, 8, 64) + r)
        cp_full.append(arena(c, (1, n * 8, 64), torch.bfloat16)[1])
        uly_x.append(torch.arange(2 * 8 * n * 64, device="cuda").to(torch.bfloat16).view(2, 8, n, 64) + r)
        uly_y.append(arena(c, (2, n * 8, 1, 64), torch.bfloat16)[1])
        x = arena(c, (8 * n, 256), torch.bfloat16)[1]
        x.fill_(0.5)
        rms.append((x, torch.zeros(8, 256, dtype=torch.bfloat16, device="cuda"), torch.ones(256, dtype=torch.bfloat16, device="cuda"),
                    torch.empty(8, 256, dtype=torch.bfloat16, device="cuda")))
        E, tokens, row = 8, 16, 64
        ids = (torch.arange(tokens * 2, device="cuda", dtype=torch.int32).view(tokens, 2) * 3 + r) % E
        recv = arena(c, (n * tokens * 2, row), torch.bfloat16)[1]
        small = (torch.zeros(E // n, dtype=torch.int32, device="cuda"), torch.zeros(tokens, 2, dtype=torch.int32, device="cuda"),
                 torch.zeros(1, dtype=torch.int32, device="cuda"))
        ex.append(dict(x=torch.ones(tokens, row, dtype=torch.bfloat16, device="cuda") * (r + 1), ids=ids, recv=recv, small=small,
                       w=torch.full((tokens, 2), 0.5, device="cuda"), out=torch.empty(tokens, row, dtype=torch.bfloat16, device="cuda")))
    nxt = [[[x.cuda() for x in row] for row in layer] for layer in srcs]
    torch.cuda.synchronize()

    def copy_in(r, c, st, L):
        for x, s in zip(shards[r], nxt[L][r]):
            x.copy_(s)

    def gather(r, c, st, L):
        c.all_gather_shards(shards[r], fulls[r], shard_rows=ps, stream=st)

    def overwrite_and_read(r, c, st, L):
        for x in shards[r]:
            x.fill_(-7.0)                                                   # the sources overwritten right after the call
        for f, s, d in zip(fulls[r], saved[r][L], grads[r]):
            s.copy_(f)
            torch.mul(f, 2, out=d)                                          # the backward stand-in reads the parameters

    def context(r, c, st, L):
        c.all_gather_context([cp_kv[r]], [cp_full[r]], chunks=2, stream=st)

    def ulysses(r, c, st, L):
        c.all_to_all_seq_to_heads([uly_x[r]], [uly_y[r]], stream=st)

    def rs(r, c, st, L):
        c.reduce_scatter_shards(grads[r], gshards[r][L], scale=1.0 / n, accumulate=True, shard_rows=ps, stream=st)

    def rms_norm(r, c, st, L):
        c.reduce_scatter_rms_norm(*rms[r], stream=st)

    def expert(r, c, st, L):
        e = ex[r]
        c.expert_dispatch(e["x"], e["ids"], 8, e["recv"], *e["small"], stream=st)
        c.expert_combine(e["recv"], e["small"][1], e["w"], e["out"], stream=st)

    phases = [copy_in, gather, overwrite_and_read, context, ulysses, rs, rms_norm, expert]
    orders = [list(range(n)), list(reversed(range(n))), [2, 0, 3, 1], [1, 3, 0, 2]]
    for L in range(layers):
        for k, phase in enumerate(phases):
            for r in orders[(L + k) % len(orders)]:
                with torch.cuda.stream(g.streams[r]):
                    phase(r, g.comms[r], g.streams[r], L)
    g.sync()
    g.check_async()
    for L in range(layers):
        for i, sh in enumerate(shapes):
            want = ref.all_gather([srcs[L][s][i] for s in range(n)], sh[0], torch.bfloat16, ps[i])
            for r in range(n):
                assert torch.equal(saved[r][L][i].cpu().view(torch.int16), want.view(torch.int16)), f"layer {L} gather {i} rank {r}"
            olds = [torch.full((ps[i], *sh[1:]), 0.5)] * n
            back = ref.reduce_scatter([want * 2] * n, torch.float32, 1.0 / n, olds, ps[i])
            for r in range(n):
                got = gshards[r][L][i][:back[r].shape[0]].cpu()
                assert torch.equal(got, back[r]), f"layer {L} reduce-scatter {i} rank {r}"
    for r in range(n):
        want = cref.all_gather([cp_kv[s].cpu() for s in range(n)], 2).view(torch.bfloat16).view(1, n * 8, 64)
        assert torch.equal(cp_full[r].cpu(), want), r
        assert torch.equal(uly_y[r], torch.cat([uly_x[s][:, :, r:r + 1] for s in range(n)], dim=1)), r
        assert bool(torch.isfinite(rms[r][3].float()).all()), r
        assert torch.equal(ex[r]["out"], ex[r]["x"]), r                     # two slots of weight 0.5 bring the row back


# ------------------------------------------------------------------------------------------------- model shapes
def llama_block(H, F, KV):
    return [(H, H), (KV, H), (KV, H), (H, H), (F, H), (F, H), (H, F), (H,), (H,)]


def run_on_device(g, shapes, ps, gen_seed):
    """The fp32 -> bf16 gather and the bf16 -> fp32 accumulating reduce-scatter (scale 1/N) of `shapes` on device, the gradients being
    the gathered parameters times (rank + 1); checked on the device against the reference. Returns nothing; raises on a difference."""
    torch, n = g.torch, g.n
    gen = torch.Generator(device="cuda").manual_seed(gen_seed)
    shards = [[torch.randn((p, *sh[1:]), device="cuda", generator=gen) for sh, p in zip(shapes, ps)] for _ in range(n)]
    bases, fulls = [], []
    for c in g.comms:
        row = []
        for sh in shapes:
            b, f = arena(c, sh, torch.bfloat16)
            bases.append((c, b))
            row.append(f)
        fulls.append(row)
    torch.cuda.synchronize()
    g.run(lambda r, c, st: c.all_gather_shards(shards[r], fulls[r], shard_rows=ps, stream=st))
    for i, sh in enumerate(shapes):
        want = ref.all_gather([s[i] for s in shards], sh[0], torch.bfloat16, ps[i])
        for r in range(n):
            assert torch.equal(fulls[r][i].view(torch.int16), want.view(torch.int16)), (sh, r)
        del want
    for r in range(n):
        for f in fulls[r]:
            f.mul_(r + 1)
    olds = [[torch.randn((p, *sh[1:]), device="cuda", generator=gen) for sh, p in zip(shapes, ps)] for _ in range(n)]
    outs = [[o.clone() for o in row] for row in olds]
    torch.cuda.synchronize()
    g.run(lambda r, c, st: c.reduce_scatter_shards(fulls[r], outs[r], scale=1.0 / n, accumulate=True, shard_rows=ps, stream=st))
    for i, sh in enumerate(shapes):
        want = ref.reduce_scatter([f[i] for f in fulls], torch.float32, 1.0 / n, [o[i] for o in olds], ps[i])
        for r in range(n):
            assert torch.equal(outs[r][i][:want[r].shape[0]].view(torch.int32), want[r].view(torch.int32)), (sh, r)
        del want
    del shards, olds, outs
    release(bases)


@pytest.mark.parametrize("name,H,F,KV", [("llama3-8b", 4096, 14336, 1024), ("llama3-70b", 8192, 28672, 1024)])
def test_llama_blocks_at_8_ranks(torch_cuda, coll_mod, name, H, F, KV):
    torch = torch_cuda
    shapes = llama_block(H, F, KV)
    full_bytes = sum(numel(sh) for sh in shapes) * 2
    need = 16 * full_bytes + (2 << 30)            # arenas (bf16 fulls), fp32 shards, olds and outputs, the reference's temporaries
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB free, {free / 2**30:.1f} GiB free")
    with Group(torch, coll_mod, 8, arena_mb=full_bytes // 2**20 + 64) as g:
        run_on_device(g, shapes, [ref.default_rows(sh[0], 8) for sh in shapes], 1)


def test_awkward_shapes(torch_cuda, groups):
    """A stacked-expert 3-D weight [E, F, H], 1-D norm weights at N = 3 and 6 with p rounded up past ceil(d / N), and 64 tensors in one
    call (the largest unit the call takes)."""
    torch = torch_cuda
    for n in (3, 6, 8):
        g = groups(n)
        experts = [(16, 96, 64)]
        run_on_device(g, experts, [ref.default_rows(16, n)], 10 + n)
        norms = [(4096,), (4096,), (1000,)]
        ps = [rows_per_rank(sh, n, 2) for sh in norms]
        assert n == 8 or any(p != ref.default_rows(sh[0], n) for sh, p in zip(norms, ps))
        run_on_device(g, norms, ps, 20 + n)
    g = groups(4)
    many = [(8 + (k % 7) * 3, 16 * (1 + k % 5)) for k in range(64)]
    run_on_device(g, many, [ref.default_rows(sh[0], 4) for sh in many], 5)
    run_gather(g, many, torch.float32, torch.float32, seed=6)
    with pytest.raises(ValueError, match="1 to 64"):
        g.coll.check_all_gather_shards(4, 0, [torch.zeros(16)] * 65, [torch.zeros(16)] * 65)


def test_full_tensor_past_4_gib(torch_cuda, coll_mod):
    """One bf16 full of 4.5 GiB at two ranks: byte offsets past 2^32 in the gather's pushes and the reduce-scatter's pulls."""
    torch = torch_cuda
    d, W = 9 * (1 << 18), 1024                    # 2359296 rows of 1024 bf16: 4.5 GiB
    full_bytes = d * W * 2
    need = 4 * full_bytes + (4 << 30)             # two arenas, the shards and outputs, the reference's chunks
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB free, {free / 2**30:.1f} GiB free")
    with Group(torch, coll_mod, 2, arena_mb=full_bytes // 2**20 + 64) as g:
        p = d // 2
        gen = torch.Generator(device="cuda").manual_seed(3)
        shards = [torch.randint(-2**15, 2**15, (p, W), dtype=torch.int16, device="cuda", generator=gen).view(torch.bfloat16) for _ in range(2)]
        bases = [c.empty(d * W, torch.bfloat16) for c in g.comms]
        fulls = [b.view(d, W) for b in bases]
        torch.cuda.synchronize()
        g.run(lambda r, c, st: c.all_gather_shards([shards[r]], [fulls[r]], stream=st))
        for r in range(2):
            for s in range(2):
                assert torch.equal(fulls[r][s * p:(s + 1) * p].view(torch.int16), shards[s].view(torch.int16)), (r, s)
        del shards
        outs = [torch.empty(p, W, dtype=torch.bfloat16, device="cuda") for _ in range(2)]
        for f in fulls:                                                     # finite values below 2
            f.view(torch.int16).bitwise_and_(0x3FFF)
        torch.cuda.synchronize()
        g.run(lambda r, c, st: c.reduce_scatter_shards([fulls[r]], [outs[r]], stream=st))
        step = p // 8
        for r in range(2):
            for a in range(0, p, step):                                     # (+0 + rank 0) + rank 1 in fp32, rounded once
                rows = slice(r * p + a, r * p + a + step)
                want = (fulls[0][rows].float() + fulls[1][rows].float()).to(torch.bfloat16)
                assert torch.equal(outs[r][a:a + step].view(torch.int16), want.view(torch.int16)), (r, a)
            del want
        del fulls
        for c, b in zip(g.comms, bases):
            c.release(b)


# ------------------------------------------------------------------------------------------------- a small FSDP training step
def test_fsdp_training_step(torch_cuda, groups):
    """A sharded MLP with RMSNorm weights on 4 virtual ranks: fp32 master shards gathered to bf16 parameters, two micro-batches of
    forward and backward per rank in bf16, the bf16 gradients reduce-scattered into fp32 sharded gradients with scale 1/N, the second
    micro-batch accumulating. The sharded gradients equal the order-exact reference bit for bit and a single-device fp64 mean of the
    same bf16 gradients within fp32 tolerance."""
    torch = torch_cuda
    n, H, F, B = 4, 64, 160, 8
    g = groups(n)
    shapes = [(H,), (F, H), (H, F), (H,)]                   # norm1, w_in, w_out, norm2
    ps = [rows_per_rank(sh, n, 2) for sh in shapes]
    gen = torch.Generator().manual_seed(11)
    master = [torch.randn(sh, generator=gen) * (0.1 if len(sh) > 1 else 1.0) + (1.0 if len(sh) == 1 else 0.0) for sh in shapes]
    shards = [[torch.zeros((p, *sh[1:]), device="cuda") for sh, p in zip(shapes, ps)] for _ in range(n)]
    for r in range(n):
        for i, (sh, p) in enumerate(zip(shapes, ps)):
            f, k = ref.shard_range(sh[0], p, r)
            shards[r][i][:k] = master[i][f:f + k].cuda()
    data = [[torch.randn(B, H, generator=gen).cuda().to(torch.bfloat16) for _ in range(2)] for _ in range(n)]
    bases, params, gfull = [], [], []
    for c in g.comms:
        prow, grow = [], []
        for sh in shapes:
            b, t = arena(c, sh, torch.bfloat16)
            bases.append((c, b))
            prow.append(t)
            b, t = arena(c, sh, torch.bfloat16)
            bases.append((c, b))
            grow.append(t)
        params.append(prow)
        gfull.append(grow)
    grad_shards = [[torch.zeros((p, *sh[1:]), device="cuda") for sh, p in zip(shapes, ps)] for _ in range(n)]

    def loss_fn(ws, x):
        n1, w_in, w_out, n2 = ws
        h = torch.nn.functional.rms_norm(x, (H,), n1, 1e-6)
        h = torch.nn.functional.gelu(h @ w_in.t()) @ w_out.t()
        return torch.nn.functional.rms_norm(h, (H,), n2, 1e-6).float().pow(2).mean()

    torch.cuda.synchronize()
    g.run(lambda r, c, st: c.all_gather_shards(shards[r], params[r], shard_rows=ps, stream=st))
    all_grads = []
    for mb in range(2):
        per_rank = []
        for r in range(n):
            ws = [p.detach().clone().requires_grad_(True) for p in params[r]]
            gs = torch.autograd.grad(loss_fn(ws, data[r][mb]), ws)
            for dst, gr in zip(gfull[r], gs):
                dst.copy_(gr)
            per_rank.append([gr.detach().clone() for gr in gs])
        all_grads.append(per_rank)
        torch.cuda.synchronize()
        g.run(lambda r, c, st: c.reduce_scatter_shards(gfull[r], grad_shards[r], scale=1.0 / n, accumulate=mb > 0, shard_rows=ps,
                                                      stream=st))
    # the order-exact reference: micro-batch 0 overwrites, micro-batch 1 accumulates
    for i, sh in enumerate(shapes):
        first = ref.reduce_scatter([all_grads[0][r][i] for r in range(n)], torch.float32, 1.0 / n, None, ps[i])
        second = ref.reduce_scatter([all_grads[1][r][i] for r in range(n)], torch.float32, 1.0 / n, first, ps[i])
        single = sum(all_grads[mb][r][i].double() for mb in range(2) for r in range(n)) / n        # one device, fp64
        for r in range(n):
            f, k = ref.shard_range(sh[0], ps[i], r)
            got = grad_shards[r][i][:k]
            assert torch.equal(got.view(torch.int32), second[r].view(torch.int32)), (i, r)
            torch.testing.assert_close(got.double(), single[f:f + k], rtol=1e-6, atol=1e-7)
    # and the parameters every rank used are the bf16 cast of the fp32 master
    for r in range(n):
        for i in range(len(shapes)):
            assert torch.equal(params[r][i].cpu(), master[i].to(torch.bfloat16))
    release(bases)


# ------------------------------------------------------------------------------------------------- the perf tool
@pytest.mark.parametrize("devs,op,dt,out,extra", [
    ("0", "all_gather", "float", "bfloat16", []), ("0", "all_gather", "e4m3", "e4m3", []),
    ("0", "reduce_scatter", "bfloat16", "float", ["--accumulate", "--scale", "0.5"]), ("0", "reduce_scatter", "half", "half", []),
    ("0,0", "all_gather", "float", "half", []), ("0,0,0", "reduce_scatter", "bfloat16", "float", ["--accumulate", "--scale", "0.25"]),
    ("0,0,0,0", "all_gather", "bfloat16", "bfloat16", []), ("0,0,0,0", "reduce_scatter", "float", "float", ["--scale", "0.25"]),
])
def test_perf_tool_checks_every_element(torch_cuda, coll_lib, devs, op, dt, out, extra):
    out_s = run_perf(["--op", op, "-d", dt, "--out-dtype", out, "--fsdp", "256:704:64", *extra, "-w", "1", "-n", "2", "-c", "1"], devs,
                     env={"B200COLL_TIMEOUT_MS": "20000"})
    assert "fsdp" in out_s, out_s
    n = len(devs.split(","))
    rows = [line for line in out_s.splitlines() if line and not line.startswith("#")]
    assert len(rows) == 1 and rows[0].split()[2] == ("copy" if n == 1 else "twoshot"), out_s


def test_multi_gpu_perf_tool_processes_cross_checked(torch_cuda, coll_lib):
    """One process per GPU with B200COLL_CHECK=1: the ranks exchange the direction, dtypes, scale, accumulate, and every tensor's rows,
    width, shard rows and full offset before every launch, and every element is checked."""
    torch = torch_cuda
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    devs = ",".join(str(i) for i in range(n))
    for op, dt, out, extra in (("all_gather", "float", "bfloat16", []), ("reduce_scatter", "bfloat16", "float", ["--accumulate", "--scale", "0.125"])):
        run_perf(["--op", op, "-d", dt, "--out-dtype", out, "--fsdp", "1024:3584:256", *extra, "-w", "1", "-n", "3", "-c", "1"], devs, procs=True,
                 env={"B200COLL_CHECK": "1", "B200COLL_TIMEOUT_MS": "20000"}, timeout=300)
