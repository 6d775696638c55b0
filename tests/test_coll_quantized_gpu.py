"""Quantising all-gather, reduce-scatter and all-reduce on an H100 (`pytest -m gpu`), virtual ranks sharing cuda:0.

Every numeric check is bit for bit against tests/coll_quant_reference.py (per-block amax, IEEE divisions, RNE saturating FP8 pack, one
multiply to dequantise, rank-order fp32 sum, one rounding); NaN matches NaN at the same position."""
import ctypes as C

import pytest

from container_engine_accelerators_b200.ops.coll import INVALID_ARGUMENT, OUT_OF_MEMORY
from tests import coll_quant_reference as qr
from tests.coll_fp_reference import assert_same, avg_scale
from tests.coll_gpu_harness import DTYPES, Group, assert_nothing_launched, coll_mod, expect_refused, run_perf, torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu


def inputs(torch, comms, count, in_dt, block, seed, arena=True):
    """Per-rank CPU reference inputs and their device copies (arena tensors, or plain torch.empty with arena=False)."""
    xs = [qr.gen(count, in_dt, block, seed + 17 * r) for r in range(len(comms))]
    ds = []
    for c, x in zip(comms, xs):
        d = c.empty(count, in_dt) if arena else torch.empty(count, dtype=in_dt, device="cuda")
        d.copy_(x)
        ds.append(d)
    torch.cuda.synchronize()
    return xs, ds


def outputs(torch, comms, numel, dt, arena=True):
    outs = [c.empty(numel, dt) if arena else torch.empty(numel, dtype=dt, device="cuda") for c in comms]
    for o in outs:
        o.view(torch.uint8).fill_(0x5A)                                  # poisoned: every element must be written
    torch.cuda.synchronize()
    return outs


def call(g, op, ds, outs, block, wire, scale=1.0, red=None, algo=None):
    red = g.coll.SUM if red is None else red

    def fn(r, c, st):
        if algo:
            c.set_algo(algo)
        if op == "all_gather":
            c.all_gather_quantized(ds[r], outs[r], block=block, wire=wire, scale=scale, stream=st)
        elif op == "reduce_scatter":
            c.reduce_scatter_quantized(ds[r], outs[r], block=block, wire=wire, scale=scale, op=red, stream=st)
        else:
            c.all_reduce_quantized(ds[r], outs[r], block=block, wire=wire, scale=scale, op=red, stream=st)
    g.run(fn)


def reference(coll, op, xs, block, wire, scale, red, out_dt, rank):
    n = len(xs)
    s = avg_scale(scale, n) if (red == coll.AVG and op != "all_gather") else scale
    if op == "all_gather":
        return qr.all_gather(xs, block, wire, s, out_dt)
    if op == "reduce_scatter":
        return qr.reduce_scatter(xs, block, wire, s, out_dt, rank)
    return qr.all_reduce(xs, block, wire, s, out_dt)


# (nranks, op, algo, in, wire, out, block, blocks per rank): every value of every axis appears; the block counts leave the two-shot
# slices uneven (cut at whole blocks) and give several CTAs and grid-stride iterations
GRID = [
    (1, "all_reduce", None, "bf16", "e4m3", "bf16", 128, 24),
    (1, "all_gather", None, "f32", "e5m2", "f16", 16, 40),
    (1, "reduce_scatter", None, "f16", "e4m3", "f32", 512, 6),
    (2, "all_reduce", "oneshot", "bf16", "e4m3", "bf16", 128, 40),
    (2, "all_reduce", "twoshot", "f32", "e5m2", "f32", 16, 301),
    (2, "all_gather", None, "f16", "e4m3", "bf16", 512, 9),
    (2, "reduce_scatter", None, "bf16", "e5m2", "f16", 128, 24),
    (3, "all_reduce", "twoshot", "bf16", "e4m3", "f32", 512, 13),
    (3, "all_reduce", "oneshot", "f16", "e5m2", "bf16", 16, 200),
    (3, "reduce_scatter", None, "f32", "e4m3", "bf16", 16, 96),
    (3, "all_gather", None, "bf16", "e5m2", "f32", 128, 17),
    (4, "all_reduce", "twoshot", "f16", "e4m3", "f16", 128, 43),
    (4, "reduce_scatter", None, "f16", "e5m2", "f32", 512, 8),
    (4, "all_gather", None, "f32", "e4m3", "f16", 16, 64),
    (8, "all_reduce", "oneshot", "f32", "e4m3", "bf16", 512, 11),
    (8, "all_reduce", "twoshot", "bf16", "e5m2", "f16", 16, 123),
    (8, "reduce_scatter", None, "bf16", "e4m3", "bf16", 128, 16),
    (8, "all_gather", None, "f16", "e5m2", "bf16", 128, 7),
]


@pytest.mark.parametrize("case", GRID, ids=lambda c: "-".join(str(x) for x in c if x is not None))
def test_grid_bit_exact(torch_cuda, coll_mod, case):
    torch, coll = torch_cuda, coll_mod
    n, op, algo, in_name, wire_name, out_name, block, nblk = case
    in_dt, wire, out_dt = DTYPES[in_name], DTYPES[wire_name], DTYPES[out_name]
    count = nblk * block * (n if op == "reduce_scatter" else 1)
    with Group(torch, coll, n, arena_mb=192) as g:
        xs, ds = inputs(torch, g.comms, count, in_dt, block, seed=nblk + block)
        numel = {"all_gather": count * n, "reduce_scatter": count // n, "all_reduce": count}[op]
        for red, scale in ((coll.SUM, 1.0), (coll.AVG, 0.7)):
            if op == "all_gather" and red == coll.AVG:
                red = coll.SUM
            outs = outputs(torch, g.comms, numel, out_dt)
            before = [c.stats() for c in g.comms]
            call(g, op, ds, outs, block, wire, scale, red, algo)
            for r, c in enumerate(g.comms):
                want = reference(coll, op, xs, block, wire, scale, red, out_dt, r)
                assert_same(outs[r].cpu(), want, f"{case} rank {r} op {red} scale {scale}")
                st = c.stats()
                assert st["kernel_launches"] == before[r]["kernel_launches"] + 1
                used = "copy" if n == 1 else (algo or "oneshot")
                assert st["algo_calls"][used] == before[r]["algo_calls"][used] + 1, (used, st["algo_calls"])


def test_algorithms_and_reduce_scatter_agree_and_one_rank_is_the_round_trip(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    n, block, count = 3, 64, 64 * 31 * 3
    with Group(torch, coll, n, arena_mb=192) as g:
        xs, ds = inputs(torch, g.comms, count, torch.bfloat16, block, seed=3)
        one, two = outputs(torch, g.comms, count, torch.float32), outputs(torch, g.comms, count, torch.float32)
        rs = outputs(torch, g.comms, count // n, torch.float32)
        call(g, "all_reduce", ds, one, block, torch.float8_e4m3fn, algo="oneshot")
        call(g, "all_reduce", ds, two, block, torch.float8_e4m3fn, algo="twoshot")
        call(g, "reduce_scatter", ds, rs, block, torch.float8_e4m3fn)
        m = count // n
        for r in range(n):
            assert_same(one[r].cpu(), one[0].cpu(), f"one-shot rank {r} vs rank 0", nan_payloads=True)
            assert_same(two[r].cpu(), one[0].cpu(), f"two-shot rank {r} vs one-shot", nan_payloads=True)
            assert_same(rs[r].cpu(), one[0][r * m:(r + 1) * m].cpu(), f"reduce-scatter rank {r} vs all-reduce slice", nan_payloads=True)
    with Group(torch, coll, 1, arena_mb=192) as g:
        xs, ds = inputs(torch, g.comms, 128 * 8, torch.float32, 128, seed=9, arena=False)
        out = outputs(torch, g.comms, 128 * 8, torch.float32, arena=False)
        call(g, "all_reduce", ds, out, 128, torch.float8_e4m3fn)
        want = qr.quantize(xs[0], 128, torch.float8_e4m3fn)[2]
        assert_same(out[0].cpu(), qr.reduce([want], 1.0, torch.float32), "one rank")
        fin = torch.isfinite(xs[0])
        assert not torch.equal(out[0].cpu()[fin], xs[0][fin]), "one rank must be the round trip, not a copy"


def test_send_outside_the_arena_and_two_shot_fallback(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    n, block, count, wire = 2, 128, 128 * 20 * 2, torch.float8_e5m2
    with Group(torch, coll, n, arena_mb=192) as g:
        xs, ds = inputs(torch, g.comms, count, torch.float16, block, seed=11, arena=False)
        assert not any(c.is_symmetric(d) for c, d in zip(g.comms, ds))
        for op, numel in (("all_gather", count * n), ("reduce_scatter", count // n), ("all_reduce", count)):
            outs = outputs(torch, g.comms, numel, torch.bfloat16)
            call(g, op, ds, outs, block, wire, algo="twoshot")
            for r in range(n):
                assert_same(outs[r].cpu(), reference(coll, op, xs, block, wire, 1.0, coll.SUM, torch.bfloat16, r), f"{op} send outside the arena")
        # two-shot pushes into every recv: with recv outside the arena the call runs one-shot
        outs = outputs(torch, g.comms, count, torch.bfloat16, arena=False)
        before = [c.stats()["algo_calls"] for c in g.comms]
        call(g, "all_reduce", ds, outs, block, wire, algo="twoshot")
        for r, c in enumerate(g.comms):
            after = c.stats()["algo_calls"]
            assert after["oneshot"] == before[r]["oneshot"] + 1 and after["twoshot"] == before[r]["twoshot"], after
            assert_same(outs[r].cpu(), reference(coll, "all_reduce", xs, block, wire, 1.0, coll.SUM, torch.bfloat16, r), "fallback")


@pytest.mark.parametrize("algo", ["oneshot", "twoshot"])
@pytest.mark.parametrize("dts", [("bf16", "bf16"), ("f32", "f32"), ("f16", "bf16")])
def test_in_place_all_reduce(torch_cuda, coll_mod, algo, dts):
    torch, coll = torch_cuda, coll_mod
    n, block = 4, 32
    in_dt, out_dt = DTYPES[dts[0]], DTYPES[dts[1]]
    count = block * 157
    with Group(torch, coll, n, arena_mb=192) as g:
        for c in g.comms:
            c.set_max_ctas(3)                                            # few CTAs: many grid-stride iterations per CTA
        xs, ds = inputs(torch, g.comms, count, in_dt, block, seed=21)
        want = qr.all_reduce(xs, block, torch.float8_e4m3fn, 1.0, out_dt)

        def fn(r, c, st):
            c.set_algo(algo)
            buf = ds[r] if in_dt == out_dt else ds[r].view(out_dt)
            if in_dt == out_dt:
                c.all_reduce_quantized(ds[r], block=block, stream=st)
            else:
                c.all_reduce_quantized(ds[r], buf, block=block, stream=st)
        g.run(fn)
        for r, c in enumerate(g.comms):
            got = ds[r] if in_dt == out_dt else ds[r].view(out_dt)
            assert_same(got.cpu(), want, f"in-place {algo} {dts} rank {r}")
            assert c.stats()["algo_calls"][algo] == 1


def _raw(coll, comm, fn, send, recv, count, wire, block, in_dt, out_dt, *extra):
    ep = coll.Epilogue(in_dt, out_dt, 1.0)
    return fn(C.c_void_p(send), C.c_void_p(recv), count, wire, block, C.byref(ep), *extra, comm._h, None)


def test_argument_errors(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    L = coll.load()
    with Group(torch, coll, 2, arena_mb=192) as g:
        c = g.comms[0]
        send = c.empty(4096, torch.bfloat16)
        recv = c.empty(8192, torch.float32)
        s, r = send.data_ptr(), recv.data_ptr()
        AG, RS, AR = L.b200collAllGatherQuantized, L.b200collReduceScatterQuantized, L.b200collAllReduceQuantized
        E4, E5, BF, F16, F32 = coll.FP8_E4M3, coll.FP8_E5M2, coll.BF16, coll.F16, coll.F32
        cases = [
            # (what, fn, send, recv, count, wire, block, in, out, extra)
            ("FP8 input", AR, s, r, 4096, E4, 128, E4, BF, (coll.SUM,)),
            ("int input", AG, s, r, 4096, E4, 128, coll.I32, BF, ()),
            ("FP8 output", AR, s, r, 4096, E4, 128, BF, E5, (coll.SUM,)),
            ("bf16 wire", AG, s, r, 4096, BF, 128, BF, BF, ()),
            ("fp32 wire", RS, s, r, 2048, F32, 128, BF, F32, (coll.SUM,)),
            ("block 24", AR, s, r, 4080, E4, 24, BF, BF, (coll.SUM,)),
            ("block 8", AR, s, r, 4096, E4, 8, BF, BF, (coll.SUM,)),
            ("block 1024", AR, s, r, 4096, E4, 1024, BF, BF, (coll.SUM,)),
            ("block 0", AG, s, r, 4096, E4, 0, BF, BF, ()),
            ("count % block", AR, s, r, 4096 - 16, E4, 128, BF, BF, (coll.SUM,)),
            ("all-gather count % block", AG, s, r, 4096 - 64, E5, 128, F16, F16, ()),
            ("recvcount % block", RS, s, r, 1024 + 64, E4, 128, BF, BF, (coll.SUM,)),
            ("max", AR, s, r, 4096, E4, 128, BF, BF, (coll.MAX,)),
            ("min", RS, s, r, 2048, E4, 128, BF, BF, (coll.MIN,)),
            ("prod", AR, s, r, 4096, E5, 128, BF, BF, (coll.PROD,)),
            ("misaligned send", AR, s + 2, r, 2048, E4, 128, BF, BF, (coll.SUM,)),
            ("misaligned recv", AG, s, r + 4, 2048, E4, 128, BF, BF, ()),
            ("null send", AR, None, r, 4096, E4, 128, BF, BF, (coll.SUM,)),
            ("all-gather overlap", AG, s, s + 1024, 1024, E4, 128, BF, BF, ()),
            ("all-gather in place", AG, s, s, 1024, E4, 128, BF, BF, ()),
            ("reduce-scatter overlap", RS, s, s + 2048, 1024, E4, 128, BF, BF, (coll.SUM,)),
            ("reduce-scatter in place", RS, s, s, 1024, E4, 128, BF, BF, (coll.SUM,)),
            ("all-reduce partial overlap", AR, s, s + 256, 2048, E4, 128, BF, BF, (coll.SUM,)),
            ("all-reduce in place, other size", AR, s, s, 2048, E4, 128, BF, F32, (coll.SUM,)),
        ]
        for what, fn, snd, rcv, count, wire, block, i, o, extra in cases:
            expect_refused(_raw(coll, c, fn, snd, rcv, count, wire, block, i, o, *extra), INVALID_ARGUMENT, what=what)
        with pytest.raises(ValueError):
            c.all_gather_quantized(send, send[:2048])                    # Python refuses overlap before the library call
        with pytest.raises(ValueError):
            c.reduce_scatter_quantized(send, send[:2048])
        assert_nothing_launched(c)                                       # nothing was counted
        g.check_async()
    # the arena cannot hold the scratch: OutOfMemory with a message, nothing counted
    with Group(torch, coll, 2, arena_mb=4) as g:                # a 4 MiB heap; the scratch needs 8.25 MiB
        big = torch.zeros(8 << 20, dtype=torch.bfloat16, device="cuda")
        out = torch.empty(8 << 20, dtype=torch.bfloat16, device="cuda")
        rc = _raw(coll, g.comms[0], L.b200collAllReduceQuantized, big.data_ptr(), out.data_ptr(), big.numel(), coll.FP8_E4M3, 128, coll.BF16, coll.BF16, coll.SUM)
        expect_refused(rc, OUT_OF_MEMORY, "scratch")
        with pytest.raises(coll.B200CollError) as e:
            g.comms[1].all_gather_quantized(big, torch.empty(2 * big.numel(), dtype=torch.bfloat16, device="cuda"))
        assert e.value.code == OUT_OF_MEMORY
        assert_nothing_launched(g.comms[0])


def test_scratch_growth_keeps_a_captured_graph_valid(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    n, block, wire = 2, 128, torch.float8_e4m3fn
    with Group(torch, coll, n, arena_mb=192) as g:
        # eager calls that grow and shrink the scratch
        for k, count in enumerate((128 * 64, 128 * 256, 128 * 32, 128 * 512, 128 * 16)):
            xs, ds = inputs(torch, g.comms, count, torch.float32, block, seed=40 + k)
            outs = outputs(torch, g.comms, count, torch.bfloat16)
            call(g, "all_reduce", ds, outs, block, wire, algo="twoshot" if k % 2 else "oneshot")
            want = qr.all_reduce(xs, block, wire, 1.0, torch.bfloat16)
            for r in range(n):
                assert_same(outs[r].cpu(), want, f"eager size {count} rank {r}")
        # a graph per rank, captured at a size the current scratch holds
        count = 128 * 600
        xs, ds = inputs(torch, g.comms, count, torch.bfloat16, block, seed=77)
        outs = outputs(torch, g.comms, count, torch.float32)
        graphs = []
        for r, c in enumerate(g.comms):
            c.set_algo("twoshot")
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=g.streams[r]):
                c.all_reduce_quantized(ds[r], outs[r], block=block, wire=wire)
            graphs.append(gr)
        # an eager call four times larger moves the scratch; an arena tensor allocated afterwards must never be written by the replay
        xs4, ds4 = inputs(torch, g.comms, 4 * count, torch.bfloat16, block, seed=78)
        outs4 = outputs(torch, g.comms, 4 * count, torch.bfloat16)
        call(g, "all_reduce", ds4, outs4, block, wire, algo="oneshot")
        want4 = qr.all_reduce(xs4, block, wire, 1.0, torch.bfloat16)
        for r in range(n):
            assert_same(outs4[r].cpu(), want4, f"grown rank {r}")
        guards = [c.empty(count * 2, torch.float32) for c in g.comms]
        for gd in guards:
            gd.fill_(3.25)
        for o in outs:
            o.view(torch.uint8).fill_(0x5A)
        torch.cuda.synchronize()
        for r, gr in enumerate(graphs):
            with torch.cuda.stream(g.streams[r]):
                gr.replay()
        torch.cuda.synchronize()
        for c in g.comms:
            c.check_async_error()
        want = qr.all_reduce(xs, block, wire, 1.0, torch.float32)
        for r in range(n):
            assert_same(outs[r].cpu(), want, f"graph replay rank {r}")
            assert bool((guards[r] == 3.25).all()), f"rank {r}: the replay wrote into memory allocated after the scratch grew"
        del graphs


@pytest.mark.parametrize("op", ["all_gather", "reduce_scatter", "all_reduce"])
def test_perf_tool_quantize_bit_exact(torch_cuda, coll_lib, op):
    out = run_perf(["--op", op, "-d", "bfloat16", "--out-dtype", "float", "--quantize", "e4m3:128", "-b", "64K", "-e", "4M", "-f", "8", "-w", "1",
                    "-n", "2", "-c", "1"], "0,0")
    assert "quantised: wire=e4m3 block=128" in out, out[-2000:]
    rows = [l for l in out.splitlines() if l.strip() and not l.startswith("#")]
    assert len(rows) == 3, out                                           # 64 KiB, 512 KiB and 4 MiB
    run_perf(["--op", op, "-d", "half", "--out-dtype", "bfloat16", "--quantize", "e5m2:32", "--algo", "twoshot", "-b", "1M", "-e", "1M", "-w", "1",
              "-n", "2", "-c", "1"], "0,0,0")


def test_multi_gpu_quantized(torch_cuda, coll_mod):
    torch, coll = torch_cuda, coll_mod
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    n, block, wire = torch.cuda.device_count(), 128, torch.float8_e4m3fn
    count = block * 96 * n
    with Group(torch, coll, n, devices=list(range(n)), arena_mb=256) as g:
        comms = g.comms
        xs = [qr.gen(count, torch.bfloat16, block, 90 + r) for r in range(n)]
        ds, ag, rs, ar = [], [], [], []
        for r, c in enumerate(comms):
            with torch.cuda.device(r):
                ds.append(torch.empty(count, dtype=torch.bfloat16, device=f"cuda:{r}").copy_(xs[r]))
                ag.append(c.empty(count * n, torch.bfloat16))
                rs.append(c.empty(count // n, torch.float32))
                ar.append(c.empty(count, torch.bfloat16))
        for r in range(n):
            torch.cuda.synchronize(r)
        for algo in ("oneshot", "twoshot"):
            for r, c in enumerate(comms):
                with torch.cuda.device(r):
                    c.set_algo(algo)
                    c.all_gather_quantized(ds[r], ag[r], block=block, wire=wire)
                    c.reduce_scatter_quantized(ds[r], rs[r], block=block, wire=wire, op=coll.AVG)
                    c.all_reduce_quantized(ds[r], ar[r], block=block, wire=wire)
            for r in range(n):
                torch.cuda.synchronize(r)
            for r, c in enumerate(comms):
                c.check_async_error()
                assert_same(ag[r].cpu(), qr.all_gather(xs, block, wire, 1.0, torch.bfloat16), f"multi-GPU all_gather rank {r}")
                assert_same(rs[r].cpu(), qr.reduce_scatter(xs, block, wire, avg_scale(1.0, n), torch.float32, r), f"multi-GPU reduce_scatter rank {r}")
                assert_same(ar[r].cpu(), qr.all_reduce(xs, block, wire, 1.0, torch.bfloat16), f"multi-GPU all_reduce {algo} rank {r}")
