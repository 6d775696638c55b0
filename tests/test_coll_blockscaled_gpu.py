"""Block-scaled FP8 all-gather, reduce-scatter and all-reduce on an H100 (`pytest -m gpu`), virtual ranks sharing cuda:0.

Every numeric check is bit for bit against a torch fp32 reference that applies the semantics literally: each rank's scales expanded to
one per element, v = float(q) * s (one fp32 multiply), a rank-order sum starting from zeros, times the fp32 scale (avg: times the fp32
value 1/N), one cast to the output type. NaN is compared as NaN (the NaN bit pattern a cast produces is not part of the semantics)."""
import ctypes as C

import numpy as np
import pytest

from container_engine_accelerators_b200.ops.coll import INVALID_ARGUMENT, INVALID_USAGE
from tests.coll_fp_reference import random_fp8
from tests.coll_gpu_harness import Group, assert_nothing_launched, coll_mod, expect_refused, group_fixture, run_perf, torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu

# (rows, row_len, block): rows are multiples of 24 so that every N in {2, 3, 4, 8} can reduce-scatter them; the last three leave a
# partial last block column, the last two a partial last block row as well
CASES = [(48, 64, (1, 16)), (48, 400, (1, 128)), (264, 320, (128, 128)), (120, 208, (32, 64))]


group = group_fixture(2, arena_mb=192)          # the heap starts 77 MiB into the arena; the grid test keeps its outputs


def f32(x):
    return float(np.float32(x))


def avg_scale(scale, n):
    return float(np.float32(scale) * (np.float32(1.0) / np.float32(n)))


def scale_grid(torch, rows, row_len, block):
    return (-(-rows // block[0]), -(-row_len // block[1]))


def random_scales(torch, shape, seed, specials=False):
    """fp32 scales 2^-20 .. 2^20 with random 23-bit mantissas and random signs; with specials some blocks are 0, -0, inf, -inf or NaN."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    m = 1.0 + torch.randint(0, 1 << 23, shape, generator=g).double() / (1 << 23)
    e = torch.randint(-20, 21, shape, generator=g)
    sign = torch.where(torch.randint(0, 4, shape, generator=g) == 0, -1.0, 1.0).double()
    s = (sign * torch.ldexp(m, e)).float()
    if specials:
        flat = s.view(-1)
        pick = torch.randperm(flat.numel(), generator=g)[:10]
        for k, v in zip(pick.tolist(), [0.0, -0.0, float("inf"), float("-inf"), float("nan")] * 2):
            flat[k] = v
    return s.cuda()


def fp8_with_specials(torch, n, dt, seed):
    """random_fp8 plus NaN bytes (and inf for e5m2) at a few places."""
    q = random_fp8(torch, n, dt, seed).view(torch.uint8).clone()
    specials = [0x7F, 0xFF] if dt == torch.float8_e4m3fn else [0x7C, 0xFC, 0x7E]
    for i, b in enumerate(specials):
        q[97 * i + 5] = b
    return q.view(dt)


def make_inputs(torch, comms, rows, row_len, block, dt, seed, specials=False):
    qs, ss = [], []
    for r, c in enumerate(comms):
        q = c.empty(rows * row_len, dt).view(rows, row_len)
        q.copy_((fp8_with_specials if specials else random_fp8)(torch, rows * row_len, dt, seed + 31 * r).view(rows, row_len))
        shape = scale_grid(torch, rows, row_len, block)
        s = c.empty(shape[0] * shape[1], torch.float32).view(shape)
        s.copy_(random_scales(torch, shape, seed + 31 * r + 7, specials))
        qs.append(q); ss.append(s)
    torch.cuda.synchronize()
    return qs, ss


def dequant(torch, q, s, block):
    rows, row_len = q.shape
    e = s.repeat_interleave(block[0], dim=0)[:rows].repeat_interleave(block[1], dim=1)[:, :row_len]
    return q.float() * e


def ref_reduce(torch, qs, ss, block, scale, out_dt):
    acc = torch.zeros(qs[0].shape, dtype=torch.float32, device="cuda")
    for q, s in zip(qs, ss):                                            # rank order
        acc = acc + dequant(torch, q, s, block)
    return (acc * torch.tensor(scale, dtype=torch.float32, device="cuda")).to(out_dt)


def ref_gather(torch, qs, ss, block, scale, out_dt):
    return torch.cat([ref_reduce(torch, [q], [s], block, scale, out_dt) for q, s in zip(qs, ss)])


def assert_same(torch, got, want, what):
    """bit for bit, except that any NaN matches any NaN"""
    gn, wn = torch.isnan(got.float()), torch.isnan(want.float())
    if not torch.equal(gn, wn):
        i = int((gn != wn).view(-1).nonzero()[0])
        raise AssertionError(f"{what}: NaN mismatch at element {i}: got {got.view(-1)[i].item()} want {want.view(-1)[i].item()}")
    ib = {1: torch.uint8, 2: torch.int16, 4: torch.int32}[got.element_size()]
    g, w = got.contiguous().view(ib)[~gn], want.contiguous().view(ib)[~wn]
    if not torch.equal(g, w):
        i = int((g != w).nonzero()[0])
        raise AssertionError(f"{what}: first difference at non-NaN element {i}: got {got[~gn][i].item()} want {want[~wn][i].item()}")


def out_dtypes(torch):
    return (torch.bfloat16, torch.float16, torch.float32)


def fp8_dtypes(torch):
    return (torch.float8_e4m3fn, torch.float8_e5m2)


@pytest.mark.parametrize("group", [2, 3, 4, 8], indirect=True)
def test_grid_bit_exact(torch_cuda, coll_mod, group):
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    for ci, (rows, row_len, block) in enumerate(CASES):
        for di, dt in enumerate(fp8_dtypes(torch)):
            qs, ss = make_inputs(torch, comms, rows, row_len, block, dt, seed=1000 * n + 10 * ci + di)
            for oi, out_dt in enumerate(out_dtypes(torch)):
                what = f"n={n} {rows}x{row_len} block={block} {dt}->{out_dt}"
                scale = (1.0, 0.375, 3.0)[oi]
                ag = [c.empty(n * rows * row_len, out_dt).view(n * rows, row_len) for c in comms]
                group.run(lambda r, c, st: c.all_gather_block_scaled(qs[r], ss[r], ag[r], block=block, scale=scale, stream=st))
                want = ref_gather(torch, qs, ss, block, f32(scale), out_dt)
                for r in range(n):
                    assert_same(torch, ag[r], want, f"all_gather {what} rank {r}")
                for op, s_eff in ((coll.SUM, f32(scale)), (coll.AVG, avg_scale(scale, n))):
                    rs = [c.empty(rows // n * row_len, out_dt).view(rows // n, row_len) for c in comms]
                    group.run(lambda r, c, st: c.reduce_scatter_block_scaled(qs[r], ss[r], rs[r], block=block, scale=scale, op=op, stream=st))
                    want = ref_reduce(torch, qs, ss, block, s_eff, out_dt)
                    for r in range(n):
                        assert_same(torch, rs[r], want[r * rows // n:(r + 1) * rows // n], f"reduce_scatter op={op} {what} rank {r}")
                    for algo in ("oneshot", "twoshot"):
                        ar = [c.empty(rows * row_len, out_dt).view(rows, row_len) for c in comms]
                        before = [c.stats()["algo_calls"][algo] for c in comms]
                        group.run(lambda r, c, st: (c.set_algo(algo), c.all_reduce_block_scaled(qs[r], ss[r], ar[r], block=block, scale=scale, op=op, stream=st)))
                        for r in range(n):
                            assert_same(torch, ar[r], want, f"all_reduce {algo} op={op} {what} rank {r}")
                        assert [c.stats()["algo_calls"][algo] for c in comms] == [b + 1 for b in before]
                    for c in comms:
                        c.set_algo("auto")
    assert all(c.stats()["algo_calls"]["nvls"] == 0 for c in comms)


@pytest.mark.parametrize("group", [2, 4], indirect=True)
def test_special_scales_and_values_propagate(torch_cuda, coll_mod, group):
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    rows, row_len, block = 96, 256, (16, 32)
    for dt in fp8_dtypes(torch):
        qs, ss = make_inputs(torch, comms, rows, row_len, block, dt, seed=77, specials=True)
        for out_dt in out_dtypes(torch):
            ag = [c.empty(n * rows * row_len, out_dt).view(n * rows, row_len) for c in comms]
            group.run(lambda r, c, st: c.all_gather_block_scaled(qs[r], ss[r], ag[r], block=block, scale=0.5, stream=st))
            want = ref_gather(torch, qs, ss, block, 0.5, out_dt)
            assert bool(torch.isnan(want.float()).any()) and bool(torch.isinf(want.float()).any())
            for r in range(n):
                assert_same(torch, ag[r], want, f"all_gather specials {dt}->{out_dt} rank {r}")
            want = ref_reduce(torch, qs, ss, block, 2.0, out_dt)
            for algo in ("oneshot", "twoshot"):
                ar = [c.empty(rows * row_len, out_dt).view(rows, row_len) for c in comms]
                group.run(lambda r, c, st: (c.set_algo(algo), c.all_reduce_block_scaled(qs[r], ss[r], ar[r], block=block, scale=2.0, stream=st)))
                for r in range(n):
                    assert_same(torch, ar[r], want, f"all_reduce {algo} specials {dt}->{out_dt} rank {r}")
            rs = [c.empty(rows // n * row_len, out_dt).view(rows // n, row_len) for c in comms]
            group.run(lambda r, c, st: c.reduce_scatter_block_scaled(qs[r], ss[r], rs[r], block=block, scale=2.0, stream=st))
            for r in range(n):
                assert_same(torch, rs[r], want[r * rows // n:(r + 1) * rows // n], f"reduce_scatter specials {dt}->{out_dt} rank {r}")
    for c in comms:
        c.set_algo("auto")


@pytest.mark.parametrize("group", [2], indirect=True)
def test_negative_zero_becomes_positive_zero(torch_cuda, group):
    torch = torch_cuda
    comms = group.comms
    rows, row_len, block = 4, 64, (1, 64)
    qs, ss = [], []
    for c in comms:
        q = c.empty(rows * row_len, torch.float8_e4m3fn).view(rows, row_len)
        q.copy_(torch.full((rows, row_len), -0.0, device="cuda").to(torch.float8_e4m3fn))
        s = c.empty(rows, torch.float32).view(rows, 1); s.fill_(1.0)
        qs.append(q); ss.append(s)
    torch.cuda.synchronize()
    out = [c.empty(2 * rows * row_len, torch.bfloat16).view(2 * rows, row_len) for c in comms]
    group.run(lambda r, c, st: c.all_gather_block_scaled(qs[r], ss[r], out[r], block=block, stream=st))
    for o in out:
        assert int(o.view(torch.int16).abs().max()) == 0        # +0 only: 0 + (-0) is +0


@pytest.mark.parametrize("group", [2, 3], indirect=True)
def test_algorithm_mapping_and_fallback(torch_cuda, coll_mod, group):
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    rows, row_len, block = 48, 256, (1, 128)
    qs, ss = make_inputs(torch, comms, rows, row_len, block, torch.float8_e4m3fn, seed=5)
    want = ref_reduce(torch, qs, ss, block, 1.0, torch.bfloat16)
    # forced: the Lamport ids and oneshot -> one-shot pull; twoshot and nvls -> two-shot pull + push
    for forced, ran in (("ll", "oneshot"), ("ll2", "oneshot"), ("oneshot", "oneshot"), ("twoshot", "twoshot"), ("nvls", "twoshot")):
        ar = [c.empty(rows * row_len, torch.bfloat16).view(rows, row_len) for c in comms]
        before = [c.stats() for c in comms]
        group.run(lambda r, c, st: (c.set_algo(forced), c.all_reduce_block_scaled(qs[r], ss[r], ar[r], block=block, stream=st)))
        for r, c in enumerate(comms):
            assert_same(torch, ar[r], want, f"forced {forced} rank {r}")
            s = c.stats()
            assert s["algo_calls"][ran] == before[r]["algo_calls"][ran] + 1, (forced, s["algo_calls"])
            assert s["calls"][coll.OP_ALLREDUCE] == before[r]["calls"][coll.OP_ALLREDUCE] + 1
            assert s["bytes"][coll.OP_ALLREDUCE] == before[r]["bytes"][coll.OP_ALLREDUCE] + rows * row_len
            assert s["staged_calls"] == before[r]["staged_calls"]
    # two-shot writes into every rank's recv: with recv outside the arena it runs as one-shot
    outside = [torch.empty(rows, row_len, dtype=torch.bfloat16, device="cuda") for _ in comms]
    before = [c.stats()["algo_calls"] for c in comms]
    group.run(lambda r, c, st: (c.set_algo("twoshot"), c.all_reduce_block_scaled(qs[r], ss[r], outside[r], block=block, stream=st)))
    for r, c in enumerate(comms):
        assert_same(torch, outside[r], want, f"two-shot outside the arena rank {r}")
        a = c.stats()["algo_calls"]
        assert a["oneshot"] == before[r]["oneshot"] + 1 and a["twoshot"] == before[r]["twoshot"]
    # all-gather and reduce-scatter count as oneshot, under their own op, with the FP8 input bytes
    before = [c.stats() for c in comms]
    ag = [c.empty(n * rows * row_len, torch.float32).view(n * rows, row_len) for c in comms]
    rs = [torch.empty(rows // n, row_len, dtype=torch.float16, device="cuda") for _ in comms]      # recv of a reduce-scatter may be anywhere
    group.run(lambda r, c, st: (c.set_algo("auto"), c.all_gather_block_scaled(qs[r], ss[r], ag[r], block=block, stream=st)))
    group.run(lambda r, c, st: c.reduce_scatter_block_scaled(qs[r], ss[r], rs[r], block=block, op=coll.AVG, stream=st))
    want_rs = ref_reduce(torch, qs, ss, block, avg_scale(1.0, n), torch.float16)
    for r, c in enumerate(comms):
        assert_same(torch, ag[r], ref_gather(torch, qs, ss, block, 1.0, torch.float32), f"all_gather fp32 rank {r}")
        assert_same(torch, rs[r], want_rs[r * rows // n:(r + 1) * rows // n], f"reduce_scatter outside the arena rank {r}")
        s = c.stats()
        assert s["calls"][coll.OP_ALLGATHER] == before[r]["calls"][coll.OP_ALLGATHER] + 1
        assert s["calls"][coll.OP_REDUCESCATTER] == before[r]["calls"][coll.OP_REDUCESCATTER] + 1
        assert s["bytes"][coll.OP_ALLGATHER] == before[r]["bytes"][coll.OP_ALLGATHER] + rows * row_len
        assert s["bytes"][coll.OP_REDUCESCATTER] == before[r]["bytes"][coll.OP_REDUCESCATTER] + rows * row_len // n
        assert s["algo_calls"]["oneshot"] == before[r]["algo_calls"]["oneshot"] + 2
    # the tuner's pick (no forcing): one-shot or two-shot, never anything else, and the result does not depend on it
    for nbytes_rows in (8, 4096):
        q2, s2 = make_inputs(torch, comms, nbytes_rows, 256, block, torch.float8_e5m2, seed=9)
        ar = [c.empty(nbytes_rows * 256, torch.bfloat16).view(nbytes_rows, 256) for c in comms]
        before = [c.stats()["algo_calls"] for c in comms]
        group.run(lambda r, c, st: c.all_reduce_block_scaled(q2[r], s2[r], ar[r], block=block, stream=st))
        w2 = ref_reduce(torch, q2, s2, block, 1.0, torch.bfloat16)
        for r, c in enumerate(comms):
            assert_same(torch, ar[r], w2, f"auto rows={nbytes_rows} rank {r}")
            a = c.stats()["algo_calls"]
            assert (a["oneshot"] - before[r]["oneshot"]) + (a["twoshot"] - before[r]["twoshot"]) == 1
            assert sum(a.values()) == sum(before[r].values()) + 1


def test_one_rank_is_a_dequantising_copy(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    with Group(torch, coll, 1, arena_mb=96) as g:
        c = g.comms[0]
        for rows, row_len, block in CASES:
            for dt in fp8_dtypes(torch):
                qs, ss = make_inputs(torch, [c], rows, row_len, block, dt, seed=rows + row_len)
                for out_dt in out_dtypes(torch):
                    before = c.stats()
                    a = torch.empty(rows, row_len, dtype=out_dt, device="cuda")
                    b = c.empty(rows * row_len, out_dt).view(rows, row_len)
                    d = torch.empty(rows, row_len, dtype=out_dt, device="cuda")
                    c.all_gather_block_scaled(qs[0], ss[0], a, block=block, scale=0.25)
                    c.reduce_scatter_block_scaled(qs[0], ss[0], b, block=block, scale=0.25, op=coll.AVG)
                    c.set_algo("twoshot")
                    c.all_reduce_block_scaled(qs[0], ss[0], d, block=block, scale=0.25)
                    c.set_algo("auto")
                    torch.cuda.synchronize()
                    want = ref_reduce(torch, qs, ss, block, 0.25, out_dt)
                    for got, what in ((a, "all_gather"), (b, "reduce_scatter"), (d, "all_reduce")):
                        assert_same(torch, got, want, f"one rank {what} {rows}x{row_len} {block} {dt}->{out_dt}")
                    s = c.stats()
                    assert s["algo_calls"]["copy"] == before["algo_calls"]["copy"] + 3
                    assert s["kernel_launches"] == before["kernel_launches"] + 3
                    for op in (coll.OP_ALLREDUCE, coll.OP_ALLGATHER, coll.OP_REDUCESCATTER):
                        assert s["calls"][op] == before["calls"][op] + 1
        c.check_async_error()


@pytest.mark.parametrize("group", [2, 3], indirect=True)
def test_cuda_graph_capture_and_replay(torch_cuda, coll_mod, group):
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    rows, row_len, block = 72, 384, (128, 128)
    qs, ss = make_inputs(torch, comms, rows, row_len, block, torch.float8_e4m3fn, seed=3)
    ag = [c.empty(n * rows * row_len, torch.bfloat16).view(n * rows, row_len) for c in comms]
    rs = [c.empty(rows // n * row_len, torch.float32).view(rows // n, row_len) for c in comms]
    ar1 = [c.empty(rows * row_len, torch.float16).view(rows, row_len) for c in comms]
    ar2 = [c.empty(rows * row_len, torch.bfloat16).view(rows, row_len) for c in comms]
    graphs = []
    for r, c in enumerate(comms):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=group.streams[r]):
            c.all_gather_block_scaled(qs[r], ss[r], ag[r], block=block, scale=0.5, stream=group.streams[r])
            c.reduce_scatter_block_scaled(qs[r], ss[r], rs[r], block=block, op=coll.AVG, stream=group.streams[r])
            c.set_algo("oneshot")
            c.all_reduce_block_scaled(qs[r], ss[r], ar1[r], block=block, stream=group.streams[r])
            c.set_algo("twoshot")
            c.all_reduce_block_scaled(qs[r], ss[r], ar2[r], block=block, scale=4.0, stream=group.streams[r])
            c.set_algo("auto")
        graphs.append(g)
    for it in range(3):
        for r in range(n):
            qs[r].copy_(random_fp8(torch, rows * row_len, torch.float8_e4m3fn, seed=100 * it + r).view(rows, row_len))
            ss[r].mul_(2.0 if it % 2 else 0.5)
        torch.cuda.synchronize()
        for r, g in enumerate(graphs):
            with torch.cuda.stream(group.streams[r]):
                g.replay()
        torch.cuda.synchronize()
        for c in comms:
            c.check_async_error()
        w_ag = ref_gather(torch, qs, ss, block, 0.5, torch.bfloat16)
        w_rs = ref_reduce(torch, qs, ss, block, avg_scale(1.0, n), torch.float32)
        w_1 = ref_reduce(torch, qs, ss, block, 1.0, torch.float16)
        w_2 = ref_reduce(torch, qs, ss, block, 4.0, torch.bfloat16)
        for r in range(n):
            assert_same(torch, ag[r], w_ag, f"graph replay {it} all_gather rank {r}")
            assert_same(torch, rs[r], w_rs[r * rows // n:(r + 1) * rows // n], f"graph replay {it} reduce_scatter rank {r}")
            assert_same(torch, ar1[r], w_1, f"graph replay {it} all_reduce oneshot rank {r}")
            assert_same(torch, ar2[r], w_2, f"graph replay {it} all_reduce twoshot rank {r}")


def _raw(coll, c, fn, q, s, out, count, row_len, br, bc, in_dt, out_dt, *extra):
    """Call the C entry point directly (no Python checks): returns the library's result code."""
    bs = coll.BlockScale(s.data_ptr() if s is not None else None, row_len, br, bc)
    ep = coll.Epilogue(in_dt, out_dt, 1.0)
    return fn(C.c_void_p(q.data_ptr()), C.c_void_p(out.data_ptr()), count, C.byref(bs), C.byref(ep), *extra, c._h, C.c_void_p(0))


@pytest.mark.parametrize("group", [2], indirect=True)
def test_error_codes(torch_cuda, coll_mod, group):
    torch, coll = torch_cuda, coll_mod
    c = group.comms[0]
    L = coll.load()
    rows, row_len = 32, 128
    q = c.empty(rows * row_len, torch.float8_e4m3fn)
    s = c.empty(rows, torch.float32)
    out = c.empty(2 * rows * row_len, torch.bfloat16)
    q_out = torch.empty(rows * row_len, dtype=torch.float8_e4m3fn, device="cuda")
    s_out = torch.empty(rows, dtype=torch.float32, device="cuda")
    E4, E5, BF, F32 = coll.FP8_E4M3, coll.FP8_E5M2, coll.BF16, coll.F32
    AG, RS, AR = L.b200collAllGatherBlockScaled, L.b200collReduceScatterBlockScaled, L.b200collAllReduceBlockScaled
    n_ = rows * row_len
    cases = [
        # (what, fn, q, s, count, row_len, br, bc, in, out, extra, expected code)
        ("send outside the arena", AG, q_out, s, n_, row_len, 1, 128, E4, BF, (), INVALID_USAGE),
        ("scales outside the arena", AG, q, s_out, n_, row_len, 1, 128, E4, BF, (), INVALID_USAGE),
        ("send outside the arena (all-reduce)", AR, q_out, s, n_, row_len, 1, 128, E4, BF, (coll.SUM,), INVALID_USAGE),
        ("scales outside the arena (reduce-scatter)", RS, q, s_out, n_ // 2, row_len, 1, 128, E4, BF, (coll.SUM,), INVALID_USAGE),
        ("row_len % 16", AG, q, s, n_, 24, 1, 128, E4, BF, (), INVALID_ARGUMENT),
        ("block_cols % 16", AG, q, s, n_, row_len, 1, 24, E4, BF, (), INVALID_ARGUMENT),
        ("block_rows 0", AG, q, s, n_, row_len, 0, 128, E4, BF, (), INVALID_ARGUMENT),
        ("count % row_len", AR, q, s, n_ - 16, row_len, 1, 128, E4, BF, (coll.SUM,), INVALID_ARGUMENT),
        ("rows % nranks", RS, q, s, (rows - 1) * row_len // 2, row_len, 1, 128, E4, BF, (coll.SUM,), INVALID_ARGUMENT),
        ("min", AR, q, s, n_, row_len, 1, 128, E4, BF, (coll.MIN,), INVALID_ARGUMENT),
        ("max", RS, q, s, n_ // 2, row_len, 1, 128, E4, BF, (coll.MAX,), INVALID_ARGUMENT),
        ("prod", AR, q, s, n_, row_len, 1, 128, E5, BF, (coll.PROD,), INVALID_ARGUMENT),
        ("bf16 input", AG, q, s, n_, row_len, 1, 128, BF, BF, (), INVALID_ARGUMENT),
        ("fp32 input", AR, q, s, n_, row_len, 1, 128, F32, F32, (coll.SUM,), INVALID_ARGUMENT),
        ("FP8 output", AG, q, s, n_, row_len, 1, 128, E4, E5, (), INVALID_ARGUMENT),
    ]
    for what, fn, qq, ss, count, rl, br, bc, i, o, extra, code in cases:
        expect_refused(_raw(coll, c, fn, qq, ss, out, count, rl, br, bc, i, o, *extra), code, what=what)
    # recv overlapping send
    expect_refused(_raw(coll, c, AR, q, s, q, n_ // 2, row_len, 1, 128, E4, BF, coll.SUM), INVALID_ARGUMENT, "overlap")
    # Python-level mistakes raise ValueError before the library is called; library refusals raise B200CollError
    with pytest.raises(ValueError):
        c.all_gather_block_scaled(q.view(rows, row_len), s.view(rows // 2, 2), out.view(2 * rows, row_len))     # scales of the wrong shape
    with pytest.raises(coll.B200CollError) as e:
        c.all_gather_block_scaled(q_out.view(rows, row_len), s.view(rows, 1), out.view(2 * rows, row_len), block=(1, 128))
    assert e.value.code == INVALID_USAGE
    with pytest.raises(coll.B200CollError) as e:
        c.all_reduce_block_scaled(q.view(rows, row_len), s.view(rows, 1), out[:n_].view(rows, row_len), block=(1, 128), op=coll.MAX)
    assert e.value.code == INVALID_ARGUMENT
    # nothing was launched, nothing was counted, and the communicator still works
    assert_nothing_launched(c)
    group.check_async()


@pytest.mark.parametrize("op", ["all_gather", "reduce_scatter", "all_reduce"])
@pytest.mark.parametrize("dtypes", [("e4m3", "bfloat16", "1x128"), ("e5m2", "float", "128x128"), ("e4m3", "half", "32x64")])
def test_perf_tool_block_scaled_bit_exact(torch_cuda, coll_lib, op, dtypes):
    dt, out, block = dtypes
    stdout = run_perf(["--op", op, "-d", dt, "--out-dtype", out, "--block-scale", block, "--row-len", "1024", "-b", "64K", "-e", "1M", "-f", "16",
                       "-w", "1", "-n", "2", "-c", "1"], "0,0")
    assert "block-scaled: row_len=1024" in stdout, stdout[-2000:]
    rows = [l for l in stdout.splitlines() if l.strip() and not l.startswith("#")]
    assert len(rows) == 2, stdout                                         # 64 KiB and 1 MiB


def test_multi_gpu_block_scaled(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    n = torch.cuda.device_count()
    with Group(torch, coll, n, devices=list(range(n)), arena_mb=256) as g:
        comms = g.comms
        rows, row_len, block = 24 * 64, 2048, (1, 128)
        qs, ss, ag, ar = [], [], [], []
        for r, c in enumerate(comms):
            with torch.cuda.device(r):
                q = c.empty(rows * row_len, torch.float8_e4m3fn).view(rows, row_len)
                q.copy_(random_fp8(torch, rows * row_len, torch.float8_e4m3fn, seed=r).view(rows, row_len).to(f"cuda:{r}"))
                s = c.empty(rows * 16, torch.float32).view(rows, 16)
                s.copy_(random_scales(torch, (rows, 16), seed=50 + r).to(f"cuda:{r}"))
                qs.append(q); ss.append(s)
                ag.append(c.empty(n * rows * row_len, torch.bfloat16).view(n * rows, row_len))
                ar.append(c.empty(rows * row_len, torch.bfloat16).view(rows, row_len))
        for r in range(n):
            torch.cuda.synchronize(r)
        for algo in ("oneshot", "twoshot"):
            for r, c in enumerate(comms):
                with torch.cuda.device(r):
                    c.set_algo(algo)
                    c.all_gather_block_scaled(qs[r], ss[r], ag[r], block=block)
                    c.all_reduce_block_scaled(qs[r], ss[r], ar[r], block=block, op=coll.AVG)
            for r in range(n):
                torch.cuda.synchronize(r)
            q0, s0 = [q.to("cuda:0") for q in qs], [s.to("cuda:0") for s in ss]
            w_ag = ref_gather(torch, q0, s0, block, 1.0, torch.bfloat16)
            w_ar = ref_reduce(torch, q0, s0, block, avg_scale(1.0, n), torch.bfloat16)
            for r, c in enumerate(comms):
                c.check_async_error()
                assert_same(torch, ag[r].to("cuda:0"), w_ag, f"multi-GPU all_gather rank {r}")
                assert_same(torch, ar[r].to("cuda:0"), w_ar, f"multi-GPU all_reduce {algo} rank {r}")
