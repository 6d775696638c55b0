"""FP8 (e4m3 / e5m2) collectives on an H100 (`pytest -m gpu`), with virtual ranks sharing cuda:0 like the rest of the GPU suite.

The FP8 semantics are exact, so every check is bit for bit: inputs are widened to fp32 and summed in rank order, multiplied by the fp32
scale (avg: 1/N), then rounded once to the output type with saturation to the finite range. The reference does the same in torch; it
clamps before casting because torch's float -> FP8 conversion does not saturate (500 -> e4m3 is NaN there, 448 on the GPU)."""
import ctypes as C
import os

import pytest

from tests.coll_fp_reference import random_fp8
from tests.coll_gpu_harness import ROOT, Group, coll_mod, group_fixture, run_perf, torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu

group = group_fixture(2, arena_mb=96)


def fp8_types(torch):
    return (torch.float8_e4m3fn, torch.float8_e5m2)


def finite_max(torch, dt):
    return {torch.float8_e4m3fn: 448.0, torch.float8_e5m2: 57344.0}.get(dt)


def cast_ref(torch, f32, dt):
    """fp32 -> dt the way the library rounds: RNE, FP8 saturating to the finite range (NaN stays NaN)."""
    m = finite_max(torch, dt)
    if m is not None:
        f32 = f32.clamp(-m, m)
    return f32.to(dt)


def reduce_ref(torch, xs, scale, out_dt):
    acc = torch.zeros(xs[0].numel(), dtype=torch.float32, device=xs[0].device)
    for x in xs:                                                     # rank order
        acc = acc + x.float()
    return cast_ref(torch, acc * torch.tensor(scale, dtype=torch.float32), out_dt)


def bits(torch, t):
    return t.contiguous().view(torch.uint8)


def assert_bits(torch, got, want, what):
    g, w = bits(torch, got), bits(torch, want)
    if not torch.equal(g, w):
        i = int((g != w).nonzero()[0])
        e = got.element_size()
        raise AssertionError(f"{what}: first difference at element {i // e}: got {got.view(-1)[i // e].item()} want {want.view(-1)[i // e].item()}")


STAGED = 600 << 10          # FP8 elements: 600 KiB per rank, beyond the one-shot Lamport path, buffers outside the arena


@pytest.mark.parametrize("group", [2, 4], indirect=True)
def test_all_reduce_grid_bit_exact(torch_cuda, group):
    torch = torch_cuda
    comms, n = group.comms, group.n
    outs = lambda dt: [dt, *[o for o in fp8_types(torch) if o != dt], torch.bfloat16, torch.float16]
    for count in (16, 1003, 1 << 15, STAGED):
        staged = count == STAGED
        ins = [c.empty(count, torch.uint8) if not staged else torch.empty(count, dtype=torch.uint8, device="cuda") for c in comms]
        dsts = [c.empty(2 * count, torch.uint8) if not staged else torch.empty(2 * count, dtype=torch.uint8, device="cuda") for c in comms]
        for in_dt in fp8_types(torch):
            xs = []
            for r in range(n):
                ins[r].view(in_dt).copy_(random_fp8(torch, count, in_dt, seed=1000 * n + 10 * r + count % 7 + (in_dt == torch.float8_e5m2)))
                xs.append(ins[r].view(in_dt))
            torch.cuda.synchronize()
            for algo in ("ll", "ll2", "oneshot", "twoshot"):
                for out_dt in outs(in_dt):
                    for scale, op in ((1.0, 0), (0.125, 0), (1.0, 1)):       # sum, sum x0.125, avg
                        os_ = torch.empty((), dtype=out_dt).element_size()
                        ys = [d[:count * os_].view(out_dt) for d in dsts]

                        def body(r, c, st):
                            c.set_algo(algo)
                            c.all_reduce(xs[r], ys[r], scale=scale, op=op, stream=st)
                        group.run(body)
                        s = scale if op == 0 else scale * (1.0 / n)
                        want = reduce_ref(torch, xs, s, out_dt)
                        for r in range(n):
                            assert_bits(torch, ys[r], want, f"n={n} count={count} {algo} {in_dt}->{out_dt} scale={scale} op={op} rank {r}")
        for c in comms:
            c.set_algo("auto")
    # the NVLS reduction is never recorded for an FP8 input, whatever was forced
    assert all(c.stats()["algo_calls"]["nvls"] == 0 for c in comms)


@pytest.mark.parametrize("group", [2, 4], indirect=True)
def test_in_place_fp8_all_reduce(torch_cuda, group):
    torch = torch_cuda
    comms, n = group.comms, group.n
    for dt in fp8_types(torch):
        for algo in ("ll", "ll2", "twoshot"):
            bufs = [c.empty(4099, dt) for c in comms]
            xs = []
            for r, b in enumerate(bufs):
                b.copy_(random_fp8(torch, 4099, dt, seed=7 * r + 1))
                xs.append(b.clone())
            torch.cuda.synchronize()
            group.run(lambda r, c, st: (c.set_algo(algo), c.all_reduce(bufs[r], op=1, stream=st)))
            want = reduce_ref(torch, xs, 1.0 / n, dt)
            for r in range(n):
                assert_bits(torch, bufs[r], want, f"in-place {algo} {dt} rank {r}")
            for c, b in zip(comms, bufs):
                c.release(b)


@pytest.mark.parametrize("group", [2], indirect=True)
def test_edge_values_saturate_and_nan_propagates(torch_cuda, coll_mod, group):
    torch = torch_cuda
    comms = group.comms
    count = 64
    for algo in ("ll", "twoshot"):
        # 448 on every rank: 896 saturates to 448, not NaN
        xs = [c.empty(count, torch.float8_e4m3fn) for c in comms]
        ys = [c.empty(count, torch.float8_e4m3fn) for c in comms]
        v = torch.full((count,), 448.0); v[1] = -448.0
        for x in xs:
            x.copy_(v.to(torch.float8_e4m3fn))
        torch.cuda.synchronize()
        group.run(lambda r, c, st: (c.set_algo(algo), c.all_reduce(xs[r], ys[r], stream=st)))
        for y in ys:
            assert y[0].float().item() == 448.0 and y[1].float().item() == -448.0 and not torch.isnan(y.float()).any()
        # e5m2 +-inf saturates to +-57344; a NaN on one rank is NaN on every rank
        a = [c.empty(count, torch.float8_e5m2) for c in comms]
        b = [c.empty(count, torch.float8_e5m2) for c in comms]
        v0 = torch.ones(count); v0[0] = float("inf"); v0[1] = float("-inf")
        v1 = torch.ones(count); v1[0] = float("inf"); v1[1] = 2.0; v1[2] = float("nan")
        a[0].copy_(v0.to(torch.float8_e5m2)); a[1].copy_(v1.to(torch.float8_e5m2))
        torch.cuda.synchronize()
        group.run(lambda r, c, st: (c.set_algo(algo), c.all_reduce(a[r], b[r], stream=st)))
        for y in b:
            f = y.float()
            assert f[0].item() == 57344.0 and f[1].item() == -57344.0 and torch.isnan(f[2]).item() and f[3].item() == 2.0
        for c in comms:
            c.set_algo("auto")


@pytest.mark.parametrize("group", [2, 4], indirect=True)
def test_reduce_scatter_and_rooted_reduce(torch_cuda, group):
    torch = torch_cuda
    comms, n = group.comms, group.n
    per = 1 << 12
    for in_dt in fp8_types(torch):
        xs = [c.empty(per * n, in_dt) for c in comms]
        for r, x in enumerate(xs):
            x.copy_(random_fp8(torch, per * n, in_dt, seed=50 + r))
        torch.cuda.synchronize()
        for out_dt in (torch.bfloat16, in_dt):
            for algo in ("ll", "twoshot", "nvls"):
                ys = [c.empty(per, out_dt) for c in comms]
                group.run(lambda r, c, st: (c.set_algo(algo), c.reduce_scatter(xs[r], ys[r], op=1, stream=st)))
                for r in range(n):
                    want = reduce_ref(torch, [x[r * per:(r + 1) * per] for x in xs], 1.0 / n, out_dt)
                    assert_bits(torch, ys[r], want, f"reduce_scatter {algo} {in_dt}->{out_dt} rank {r}")
                for c, y in zip(comms, ys):
                    c.release(y)
            for root in range(n):
                ys = [c.empty(per * n, out_dt) for c in comms]
                group.run(lambda r, c, st: (c.set_algo("nvls"), c.reduce(xs[r], ys[r], root=root, scale=0.5, stream=st)))
                assert_bits(torch, ys[root], reduce_ref(torch, xs, 0.5, out_dt), f"reduce root {root} {in_dt}->{out_dt}")
                for c, y in zip(comms, ys):
                    c.release(y)
    for c in comms:
        c.set_algo("auto")
        assert c.stats()["algo_calls"]["nvls"] == 0


@pytest.mark.parametrize("group", [2], indirect=True)
def test_dequantising_all_gather_broadcast_all_to_all(torch_cuda, group):
    torch = torch_cuda
    comms, n = group.comms, group.n
    inv = 0.0078125
    for count, arena in ((1 << 20, True), (1 << 20, False), (4096, True)):
        mk = (lambda c, k, dt: c.empty(k, dt)) if arena else (lambda c, k, dt: torch.empty(k, dtype=dt, device="cuda"))
        xs = [mk(c, count * n, torch.float8_e4m3fn) for c in comms]
        for r, x in enumerate(xs):
            x.copy_(random_fp8(torch, count * n, torch.float8_e4m3fn, seed=300 + r))
        torch.cuda.synchronize()
        bulk0 = [c.stats()["bulk_launches"] for c in comms]
        deq = lambda x: reduce_ref(torch, [x], inv, torch.bfloat16)     # widened into a zeroed fp32 accumulator (-0 becomes +0), scaled, rounded
        ag = [mk(c, count * n, torch.bfloat16) for c in comms]
        group.run(lambda r, c, st: c.all_gather(xs[r][:count], ag[r], scale=inv, stream=st))
        want = torch.cat([deq(x[:count]) for x in xs])
        for r in range(n):
            assert_bits(torch, ag[r], want, f"all_gather arena={arena} rank {r}")
        bc = [mk(c, count, torch.bfloat16) for c in comms]
        group.run(lambda r, c, st: c.broadcast(xs[r][:count], bc[r], root=1, scale=inv, stream=st))
        for r in range(n):
            assert_bits(torch, bc[r], deq(xs[1][:count]), f"broadcast arena={arena} rank {r}")
        a2a = [mk(c, count * n, torch.bfloat16) for c in comms]
        group.run(lambda r, c, st: c.all_to_all(xs[r], a2a[r], scale=inv, stream=st))
        for r in range(n):
            want = torch.cat([deq(xs[q][r * count:(r + 1) * count]) for q in range(n)])
            assert_bits(torch, a2a[r], want, f"all_to_all arena={arena} rank {r}")
        assert [c.stats()["bulk_launches"] for c in comms] == bulk0      # a scaled cast is never an identity copy


@pytest.mark.parametrize("group", [2, 4], indirect=True)
def test_generic_min_max_prod(torch_cuda, coll_mod, group):
    torch = torch_cuda
    coll = coll_mod
    comms, n = group.comms, group.n
    count = 5003
    for dt in fp8_types(torch):
        for arena in (True, False):
            mk = (lambda c, k: c.empty(k, dt)) if arena else (lambda c, k: torch.empty(k, dtype=dt, device="cuda"))
            xs = [mk(c, count) for c in comms]
            for r, x in enumerate(xs):
                x.copy_(random_fp8(torch, count, dt, seed=900 + r))
            torch.cuda.synchronize()
            for op in (coll.MIN, coll.MAX, coll.PROD):
                ys = [mk(c, count) for c in comms]
                gen0 = [c.stats()["generic_launches"] for c in comms]
                group.run(lambda r, c, st: c.all_reduce(xs[r], ys[r], op=op, stream=st))
                acc = xs[0].float()
                for x in xs[1:]:
                    b = x.float()
                    acc = acc * b if op == coll.PROD else torch.where(b < acc, b, acc) if op == coll.MIN else torch.where(b > acc, b, acc)
                want = cast_ref(torch, acc, dt)
                for r in range(n):
                    assert_bits(torch, ys[r], want, f"generic op={op} {dt} arena={arena} rank {r}")
                assert all(c.stats()["generic_launches"] > g for c, g in zip(comms, gen0))
    c = comms[0]
    x8 = c.empty(64, torch.float8_e4m3fn)
    refused = [
        lambda: c.all_reduce(x8, c.empty(64, torch.float8_e4m3fn), scale=0.5, op=coll.MAX),           # scale on the generic path
        lambda: c.all_reduce(x8, c.empty(64, torch.float8_e5m2), op=coll.MIN),                       # cast on the generic path
        lambda: c.all_reduce(x8, c.empty(64, torch.float32)),                                         # FP8 -> f32
        lambda: c.all_reduce(c.empty(64, torch.int32), c.empty(64, torch.int32), op=coll.AVG),       # avg on the generic path
    ]
    for call in refused:
        with pytest.raises(coll.B200CollError) as e:
            call()
        assert e.value.code == coll.INVALID_ARGUMENT


@pytest.mark.parametrize("group", [2], indirect=True)
def test_all_reduce_host_fp8(torch_cuda, group):
    torch = torch_cuda
    comms, n = group.comms, group.n
    for count, key in ((4096, "host_zero_copy"), (9 << 20, "host_pipelined")):
        ins = [c.host_empty(count, torch.float8_e5m2) for c in comms]
        outs = [c.host_empty(count, torch.float8_e4m3fn) for c in comms]
        for r, h in enumerate(ins):
            h.copy_(random_fp8(torch, count, torch.float8_e5m2, seed=77 + r).cpu())
        before = [c.stats()[key] for c in comms]
        group.run(lambda r, c, st: c.all_reduce_host(ins[r], outs[r], scale=0.25, stream=st))
        want = reduce_ref(torch, [h.cuda() for h in ins], 0.25, torch.float8_e4m3fn).cpu()
        for r in range(n):
            assert_bits(torch, outs[r], want, f"all_reduce_host {count} rank {r}")
        assert all(c.stats()[key] == b + 1 for c, b in zip(comms, before))
        for c, a, b in zip(comms, ins, outs):
            c.host_release(a); c.host_release(b)


# ------------------------------------------------------------------------------------------------- NCCL-API shim
def test_nccl_shim_fp8(torch_cuda, coll_lib):
    torch = torch_cuda
    L = C.CDLL(os.path.join(ROOT, "coll", "lib", "libb200coll_nccl.so"))
    vp, sz, ci = C.c_void_p, C.c_size_t, C.c_int
    L.ncclGetErrorString.restype = C.c_char_p
    L.ncclCommInitAll.argtypes = [C.POINTER(vp), ci, C.POINTER(ci)]
    L.ncclCommDestroy.argtypes = [vp]
    L.ncclAllReduce.argtypes = [vp, vp, sz, ci, ci, vp, vp]
    L.ncclAllGather.argtypes = [vp, vp, sz, ci, vp, vp]
    L.ncclReduceScatter.argtypes = [vp, vp, sz, ci, ci, vp, vp]
    L.ncclBroadcast.argtypes = [vp, vp, sz, ci, ci, vp, vp]
    L.ncclReduce.argtypes = [vp, vp, sz, ci, ci, ci, vp, vp]
    L.ncclSend.argtypes = [vp, sz, ci, ci, vp, vp]
    L.ncclRecv.argtypes = [vp, sz, ci, ci, vp, vp]
    L.ncclAlltoAll.argtypes = [vp, vp, sz, ci, vp, vp]
    L.ncclRedOpCreatePreMulSum.argtypes = [C.POINTER(ci), vp, ci, ci, vp]
    L.ncclRedOpDestroy.argtypes = [ci, vp]
    L.ncclCommGetAsyncError.argtypes = [vp, C.POINTER(ci)]

    def ck(rc):
        assert rc == 0, L.ncclGetErrorString(rc).decode()
    SUM, MAX, AVG = 0, 2, 4
    n = 2
    comms = (C.c_void_p * n)()
    ck(L.ncclCommInitAll(comms, n, (C.c_int * n)(0, 0)))
    try:
        streams = [torch.cuda.Stream() for _ in range(n)]
        st = [C.c_void_p(x.cuda_stream) for x in streams]
        p = lambda t: C.c_void_p(t.data_ptr())

        def every(fn):
            for r in range(n):
                ck(fn(r))
            torch.cuda.synchronize()
            for r in range(n):
                err = C.c_int(-1)
                ck(L.ncclCommGetAsyncError(comms[r], C.byref(err)))
                assert err.value == 0

        for code, dt in ((10, torch.float8_e4m3fn), (11, torch.float8_e5m2)):
            count = 4096
            src = [random_fp8(torch, count * n, dt, seed=5 * r + code) for r in range(n)]
            dst = [torch.empty(count * n, dtype=dt, device="cuda") for _ in range(n)]
            half = torch.tensor([0.5], dtype=torch.float32).to(dt).view(torch.uint8)
            scalar = C.c_uint8(int(half.item()))
            op = C.c_int(-1)
            ck(L.ncclRedOpCreatePreMulSum(C.byref(op), C.byref(scalar), code, 1, comms[0]))
            for nop, scale in ((SUM, 1.0), (AVG, 1.0 / n), (op.value, 0.5)):
                every(lambda r: L.ncclAllReduce(p(src[r]), p(dst[r]), count * n, code, nop, comms[r], st[r]))
                for r in range(n):
                    assert_bits(torch, dst[r], reduce_ref(torch, src, scale, dt), f"ncclAllReduce type {code} op {nop}")
                rs = [torch.empty(count, dtype=dt, device="cuda") for _ in range(n)]
                every(lambda r: L.ncclReduceScatter(p(src[r]), p(rs[r]), count, code, nop, comms[r], st[r]))
                for r in range(n):
                    assert_bits(torch, rs[r], reduce_ref(torch, [s[r * count:(r + 1) * count] for s in src], scale, dt), f"ncclReduceScatter type {code} op {nop}")
                rd = [torch.empty(count * n, dtype=dt, device="cuda") for _ in range(n)]
                every(lambda r: L.ncclReduce(p(src[r]), p(rd[r]), count * n, code, nop, 1, comms[r], st[r]))
                assert_bits(torch, rd[1], reduce_ref(torch, src, scale, dt), f"ncclReduce type {code} op {nop}")
            ck(L.ncclRedOpDestroy(op.value, comms[0]))
            every(lambda r: L.ncclAllReduce(p(src[r]), p(dst[r]), count * n, code, MAX, comms[r], st[r]))
            acc = src[0].float()
            for s in src[1:]:
                acc = torch.where(s.float() > acc, s.float(), acc)
            for r in range(n):
                assert_bits(torch, dst[r], acc.to(dt), f"ncclAllReduce max type {code}")
            # data movement: arbitrary bytes, 0xFF and 0x7F (NaN patterns) included, delivered untouched
            raw = [torch.randint(0, 256, (count,), dtype=torch.int32, device="cuda").to(torch.uint8) for _ in range(n)]
            for r in range(n):
                raw[r][:8] = torch.tensor([0xFF, 0xFF, 0xFF, 0xFF, 0x7F, 0xFF, 0x7F, 0xFF], dtype=torch.uint8)
            gat = [torch.empty(count * n, dtype=torch.uint8, device="cuda") for _ in range(n)]
            every(lambda r: L.ncclAllGather(p(raw[r]), p(gat[r]), count, code, comms[r], st[r]))
            for r in range(n):
                assert torch.equal(gat[r], torch.cat(raw)), f"ncclAllGather type {code}"
            bc = [raw[r].clone() for r in range(n)]
            every(lambda r: L.ncclBroadcast(p(bc[r]), p(bc[r]), count, code, 0, comms[r], st[r]))
            for r in range(n):
                assert torch.equal(bc[r], raw[0]), f"ncclBroadcast type {code}"
            a2a = [torch.empty(count, dtype=torch.uint8, device="cuda") for _ in range(n)]
            every(lambda r: L.ncclAlltoAll(p(raw[r]), p(a2a[r]), count // n, code, comms[r], st[r]))
            h = count // n
            for r in range(n):
                assert torch.equal(a2a[r], torch.cat([raw[q][r * h:(r + 1) * h] for q in range(n)])), f"ncclAlltoAll type {code}"
            box = [torch.empty(count, dtype=torch.uint8, device="cuda") for _ in range(n)]
            for r in range(n):
                ck(L.ncclGroupStart())
                ck(L.ncclSend(p(raw[r]), count, code, 1 - r, comms[r], st[r]))
                ck(L.ncclRecv(p(box[r]), count, code, 1 - r, comms[r], st[r]))
                ck(L.ncclGroupEnd())
            torch.cuda.synchronize()
            for r in range(n):
                assert torch.equal(box[r], raw[1 - r]), f"ncclSend/ncclRecv type {code}"
    finally:
        torch.cuda.synchronize()
        for r in range(n):
            L.ncclCommDestroy(comms[r])


# ------------------------------------------------------------------------------------------------- perf tool, several GPUs
@pytest.mark.parametrize("args", [["--op", "all_reduce", "-d", "e4m3", "--out-dtype", "bf16"], ["--op", "all_reduce", "-d", "e5m2", "--out-dtype", "bf16"],
                                  ["--op", "reduce_scatter", "-d", "e4m3"]])
def test_perf_tool_fp8_zero_errors(torch_cuda, coll_lib, args):
    run_perf([*args, "-b", "1K", "-e", "64M", "-w", "1", "-n", "2"], "0,0,0,0")


def test_multi_gpu_fp8_all_reduce_never_records_nvls(torch_cuda, coll_mod):
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    n = torch.cuda.device_count()
    with Group(torch, coll_mod, n, devices=list(range(n)), arena_mb=256) as g:
        comms = g.comms
        count = 32 << 20
        xs, ys = [], []
        for r, c in enumerate(comms):
            with torch.cuda.device(r):
                x = c.empty(count, torch.float8_e4m3fn); x.copy_(random_fp8(torch, count, torch.float8_e4m3fn, seed=r).to(f"cuda:{r}"))
                xs.append(x); ys.append(c.empty(count, torch.bfloat16))
        for r in range(n):
            torch.cuda.synchronize(r)
        for r, c in enumerate(comms):
            with torch.cuda.device(r):
                c.set_algo("nvls")
                c.all_reduce(xs[r], ys[r])
        for r in range(n):
            torch.cuda.synchronize(r)
        want = reduce_ref(torch, [x.to("cuda:0") for x in xs], 1.0, torch.bfloat16)
        for r, c in enumerate(comms):
            c.check_async_error()
            assert c.stats()["algo_calls"]["nvls"] == 0
            assert_bits(torch, ys[r].to("cuda:0"), want, f"multi-GPU rank {r}")


# ------------------------------------------------------------------------------------------------- process group, two processes
def _fp8_pair(rank, world):
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(0)                                                # two ranks share cuda:0 on a one-GPU box
    pg = dist.group.WORLD
    fb = pg.fallback_calls
    for dt in (torch.float8_e4m3fn, torch.float8_e5m2):
        xs = [random_fp8(torch, 4096, dt, seed=40 + r) for r in range(world)]   # every rank can build every rank's input
        for op, ref in ((dist.ReduceOp.SUM, lambda: reduce_ref(torch, xs, 1.0, dt)), (dist.ReduceOp.AVG, lambda: reduce_ref(torch, xs, 1.0 / world, dt)),
                        (dist.ReduceOp.MAX, lambda: torch.where(xs[1].float() > xs[0].float(), xs[1].float(), xs[0].float()).to(dt))):
            t = xs[rank].clone()
            dist.all_reduce(t, op=op)
            assert_bits(torch, t, ref(), f"all_reduce {dt} {op}")
        out = torch.empty(2048, dtype=dt, device="cuda")
        dist.reduce_scatter_tensor(out, xs[rank].clone())
        assert_bits(torch, out, reduce_ref(torch, [x[rank * 2048:(rank + 1) * 2048] for x in xs], 1.0, dt), f"reduce_scatter_tensor {dt}")
        raws = [torch.randint(0, 256, (4096,), dtype=torch.int32, generator=torch.Generator().manual_seed(60 + r)).to(torch.uint8).cuda() for r in range(world)]
        for raw in raws:
            raw[:4] = 0xFF; raw[4:8] = 0x7F                                  # NaN bytes travel untouched
        g = torch.empty(world * 4096, dtype=dt, device="cuda")
        dist.all_gather_into_tensor(g, raws[rank].view(dt))
        assert torch.equal(g.view(torch.uint8), torch.cat(raws)), f"all_gather_into_tensor {dt}"
    torch.cuda.synchronize()
    assert pg.fallback_calls == fb, (pg.fallback_calls, fb)
    return pg.fast_calls


def test_process_group_fp8_two_ranks(torch_cuda):
    from tests.test_process_group import _run
    _run(_fp8_pair, 2)
