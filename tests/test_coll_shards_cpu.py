"""The FSDP shard all-gather and reduce-scatter (b200collAllGatherShards / ReduceScatterShards) in libb200coll, checked without a GPU:
the reference against a per-element loop rendering of the header's formulas, the C prototypes and struct layout against the ctypes
argtypes, every Python refusal, the kernels' instantiations, ptxas's stack and spill report, and the perf tool's help and refusals."""
import ctypes as C
import os
import subprocess

import pytest
import torch

from container_engine_accelerators_b200.ops import coll
from tests import coll_fp_reference as R
from tests import coll_shards_reference as ref
from tests.coll_binary_facts import kernels, ptxas, template_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PERF = os.path.join(ROOT, "build", "b200coll_perf")


# ------------------------------------------------------------------------------------------------- the reference
def test_shard_ranges():
    """FSDP2's ceil(d / N) rows per rank, the last ranks short or empty: 3 rows on 8 ranks leave ranks 3 .. 7 with none."""
    assert [ref.shard_range(3, 1, r) for r in range(8)] == [(0, 1), (1, 1), (2, 1)] + [(3, 0)] * 5
    assert [ref.shard_range(10, 4, r) for r in range(3)] == [(0, 4), (4, 4), (8, 2)]
    assert [ref.shard_range(10, 8, r) for r in range(3)] == [(0, 8), (8, 2), (10, 0)]      # p rounded up past ceil(d / N)
    assert [coll.shard_range(d, p, r) for d, p, r in ((3, 1, 5), (10, 4, 2), (7, 7, 0))] == [(3, 0), (8, 2), (0, 7)]


@pytest.mark.parametrize("n,d,shape,p", [(1, 5, (3,), None), (2, 5, (4,), None), (3, 7, (2, 2), None), (4, 3, (8,), None),
                                         (6, 11, (), None), (8, 3, (2,), None), (3, 10, (4,), 8), (4, 9, (2,), 4)])
def test_reference_agrees_with_the_loop_rendering(n, d, shape, p):
    g = torch.Generator().manual_seed(n * 100 + d)
    full32 = torch.randn(d, *shape, generator=g)
    pp = ref.default_rows(d, n) if p is None else p
    for sdt, fdt in ((torch.float32, torch.bfloat16), (torch.float32, torch.float16), (torch.bfloat16, torch.bfloat16),
                     (torch.float32, torch.float32)):
        shards = ref.split(full32.to(sdt), n, pp)
        shards = [torch.cat([x, torch.full((pp - x.shape[0], *shape), 7.0, dtype=sdt)]) for x in shards]     # padding is never read
        got, want = ref.all_gather(shards, d, fdt, pp), ref.all_gather_loop(shards, d, fdt, pp)
        assert torch.equal(got.view(R.INT_VIEW[R.esize(fdt)]), want.view(R.INT_VIEW[R.esize(fdt)])), (sdt, fdt)
    for fdt, sdt in ((torch.bfloat16, torch.bfloat16), (torch.float16, torch.float16), (torch.float32, torch.float32),
                     (torch.bfloat16, torch.float32), (torch.float16, torch.float32)):
        fulls = [x.view(d, *shape) for x in R.gen_inputs(n, d * max(1, _numel(shape)), fdt, seed=n + d, device="cpu")]
        olds = [torch.randn(pp, *shape, generator=g).to(sdt) for _ in range(n)]
        for scale, acc in ((1.0, False), (1.0 / n, False), (1.0, True), (0.125, True)):
            o = olds if acc else None
            got, want = ref.reduce_scatter(fulls, sdt, scale, o, pp), ref.reduce_scatter_loop(fulls, sdt, scale, o, pp)
            for r, (a, b) in enumerate(zip(got, want)):
                assert a.shape[0] == ref.shard_range(d, pp, r)[1]
                R.assert_same(a, b, f"n={n} {fdt}->{sdt} scale={scale} acc={acc} rank {r}",
                              nan_payloads=n == 1 and fdt == sdt and scale == 1.0 and not acc)      # bit copies keep NaN payloads


def _numel(shape):
    n = 1
    for e in shape:
        n *= e
    return n


def test_order_scale_and_accumulate_are_separate_roundings():
    """The sum is taken in rank order from +0, then scaled, then added to the old value: three fp32 roundings, not a fused one."""
    big, tiny = 2.0 ** 24, 1.0
    fulls = [torch.tensor([[big]]), torch.tensor([[tiny]]), torch.tensor([[tiny]]), torch.tensor([[-big]])]
    # ((0 + 2^24) + 1) = 2^24 (tie to even), + 1 = 2^24, - 2^24 = 0: rank order loses both ones
    assert ref.reduce_scatter(fulls, torch.float32, p=1)[0].item() == 0.0
    # -0 on every rank sums to +0 from +0; with one rank, scale 1 and no accumulation the bit copy keeps -0
    z = [torch.tensor([[-0.0]])] * 2
    assert ref.reduce_scatter(z, torch.float32, p=1)[0].view(torch.int32).item() == 0
    assert ref.reduce_scatter(z[:1], torch.float32)[0].view(torch.int32).item() == torch.tensor(-0.0).view(torch.int32).item()
    assert ref.reduce_scatter(z[:1], torch.float32, scale=0.5)[0].view(torch.int32).item() == 0
    # accumulate: old + t, then one rounding to bf16
    old = [torch.tensor([[1.0]], dtype=torch.float32)]
    assert ref.reduce_scatter([torch.tensor([[3.0]], dtype=torch.bfloat16)], torch.float32, 0.5, old)[0].item() == 2.5


def test_reduce_scatter_of_the_gather_is_n_times_the_shard():
    n, d, W = 4, 10, 8
    full = torch.arange(d * W, dtype=torch.float32).view(d, W) * 0.25
    shards = ref.split(full, n)
    gathered = ref.all_gather(shards, d, torch.float32)
    assert torch.equal(gathered, full)
    back = ref.reduce_scatter([gathered] * n, torch.float32)
    assert all(torch.equal(b, n * x) for b, x in zip(back, shards))


# ------------------------------------------------------------------------------------------------- C prototypes
def test_header_prototypes_match_the_ctypes_argtypes(tmp_path, coll_lib):
    src = tmp_path / "probe.c"
    src.write_text(r'''
#include <stddef.h>
#include <stdio.h>
#include "b200coll.h"
int main(void) {
  b200collResult_t (*f)(const b200collShardTensor*, int, b200collDataType_t, b200collDataType_t, b200collComm_t, b200collStream_t) =
      b200collAllGatherShards;
  b200collResult_t (*g)(const b200collShardTensor*, int, b200collDataType_t, b200collDataType_t, float, int, b200collComm_t,
                        b200collStream_t) = b200collReduceScatterShards;
  printf("%d %d %zu %zu %zu %zu %zu %zu\n", f != 0, g != 0, sizeof(b200collShardTensor), offsetof(b200collShardTensor, shard),
         offsetof(b200collShardTensor, full), offsetof(b200collShardTensor, rows), offsetof(b200collShardTensor, width),
         offsetof(b200collShardTensor, shard_rows));
  return 0;
}''')
    exe = tmp_path / "probe"
    libdir = os.path.dirname(coll_lib)
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "coll", "include"), str(src), "-o", str(exe),
                    "-L", libdir, "-lb200coll", "-Wl,-rpath," + libdir], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    T = coll.ShardTensor
    assert out == ["1", "1", str(C.sizeof(T)), str(T.shard.offset), str(T.full.offset), str(T.rows.offset), str(T.width.offset),
                   str(T.shard_rows.offset)]
    L = coll.load()
    assert L.b200collAllGatherShards.argtypes == [C.POINTER(T), C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    assert L.b200collReduceScatterShards.argtypes == [C.POINTER(T), C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_void_p]


# ------------------------------------------------------------------------------------------------- Python argument checks
_pool = torch.empty(1 << 18, dtype=torch.float32)


def _v(off, shape, dt=torch.bfloat16):
    """A contiguous tensor of `shape` at byte offset `off` of one pool (alignment and overlaps under the test's control)."""
    es = torch.empty((), dtype=dt).element_size()
    return _pool.view(torch.uint8)[off:off + _numel(shape) * es].view(dt).view(shape)


def _off(t):
    return t.data_ptr() - _pool.data_ptr()


def _unit(n=4, rank=0, sdt=torch.float32, fdt=torch.bfloat16):
    """A small unit: a [32, 16] weight, a 1-D [128] norm weight and a 3-D [8, 4, 8] stacked weight, its fulls and rank's shards."""
    shapes = [(32, 16), (128,), (8, 4, 8)]
    at, fulls, shards = 0, [], []
    for sh in shapes:
        f = _v(at, sh, fdt)
        fulls.append(f)
        at += f.numel() * f.element_size() + 64
    for sh in shapes:
        p = ref.default_rows(sh[0], n)
        x = _v(at, (p, *sh[1:]), sdt)
        shards.append(x)
        at += x.numel() * x.element_size() + 64
    return shards, fulls


def test_checks_accept_valid_calls():
    for n in (1, 2, 4, 8):
        for sdt, fdt in ((torch.float32, torch.bfloat16), (torch.float32, torch.float16), (torch.bfloat16, torch.bfloat16),
                         (torch.float32, torch.float32), (torch.float8_e4m3fn, torch.float8_e4m3fn), (torch.float8_e5m2, torch.float8_e5m2)):
            shards, fulls = _unit(n, n - 1, sdt, fdt)
            want = [(32, 16, -(-32 // n)), (128, 1, -(-128 // n)), (8, 32, -(-8 // n))]
            assert coll.check_all_gather_shards(n, n - 1, shards, fulls) == want, (n, sdt, fdt)
            if fdt.itemsize > 1:
                assert coll.check_reduce_scatter_shards(n, n - 1, fulls, shards) == want
    # the reduce-scatter's widening pairs, and float32 -> float32
    for fdt in (torch.bfloat16, torch.float16, torch.float32):
        shards, fulls = _unit(4, 1, torch.float32, fdt)
        assert len(coll.check_reduce_scatter_shards(4, 1, fulls, shards)) == 3
    # 1-D norm weights at N = 3 with p rounded up to a multiple of 8 (16 bytes of bf16); a rank with no rows
    f = _v(0, (4096,))
    assert coll.check_all_gather_shards(3, 2, [_v(16384, (1368,), torch.float32)], [f], shard_rows=1368) == [(4096, 1, 1368)]
    with pytest.raises(ValueError, match="multiples of 16 bytes"):
        coll.check_all_gather_shards(3, 0, [_v(16384, (1366,), torch.float32)], [f])                   # ceil(4096 / 3) = 1366
    tiny = _v(0, (3, 8))
    empty = _v(4096, (0, 8), torch.float32)
    assert coll.check_all_gather_shards(8, 5, [empty], [tiny]) == [(3, 8, 1)]
    # one shard_rows per tensor
    shards, fulls = _unit(4)
    assert [p for _, _, p in coll.check_all_gather_shards(4, 0, shards, fulls, shard_rows=[8, 32, 2])] == [8, 32, 2]


def _refused(match, n, rank, shards, fulls, gather=True, **kw):
    with pytest.raises(ValueError, match=match):
        if gather:
            coll.check_all_gather_shards(n, rank, shards, fulls, **kw)
        else:
            coll.check_reduce_scatter_shards(n, rank, fulls, shards, **kw)


def test_refusals():
    shards, fulls = _unit(4)
    _refused("1 to 64 tensors", 4, 0, [], [])
    _refused("1 to 64 tensors", 4, 0, shards * 22, fulls * 22)
    _refused("one shard per full", 4, 0, shards, fulls[:2])
    # dtype pairs
    _refused("dtype pair", 4, 0, [s.to(torch.int32) for s in shards], fulls)
    _refused("dtype pair", 4, 0, [s.to(torch.bfloat16) for s in shards], [f.to(torch.float32) for f in fulls])      # widening gather
    _refused("dtype pair", 4, 0, [s.to(torch.float16) for s in shards], fulls)                                        # fp16 -> bf16
    _refused("dtype pair", 4, 0, [s.to(torch.bfloat16) for s in shards], [f.to(torch.float32) for f in fulls], gather=False)   # narrowing
    s8, f8 = _unit(4, 0, torch.float8_e4m3fn, torch.float8_e4m3fn)
    _refused("dtype pair", 4, 0, s8, f8, gather=False)
    _refused("every shard must be", 4, 0, [shards[0], shards[1].to(torch.bfloat16)], fulls[:2])
    _refused("every shard must be", 4, 0, shards[:2], [fulls[0], fulls[1].to(torch.float16)])
    # shapes and shard_rows
    _refused("contiguous tensor of at least one dim", 4, 0, [shards[0]], [fulls[0].t()])
    _refused("rows and width must be positive", 4, 0, [shards[0]], [_v(0, (0, 16))])
    _refused("shard_rows must be positive", 4, 0, shards[:1], fulls[:1], shard_rows=0)
    _refused("at least rows", 4, 0, shards[:1], fulls[:1], shard_rows=7)
    _refused("one int or one per tensor", 4, 0, shards, fulls, shard_rows=[8, 16])
    _refused(r"must be a contiguous \[>= 8, 16\]", 4, 0, [shards[0][:7]], fulls[:1])
    _refused(r"must be a contiguous \[>= 8, 16\]", 4, 0, [_v(_off(shards[0]), (8, 8), torch.float32)], fulls[:1])
    _refused("must be a contiguous", 4, 0, [_v(_off(shards[0]), (16, 8), torch.float32).t()], fulls[:1])
    _refused("must be a contiguous", 4, 0, [_v(_off(shards[0]), (128,), torch.float32)], fulls[:1])
    # alignment: p * W and d * W in 16 bytes of both dtypes, and the pointers
    _refused("multiples of 16 bytes", 4, 0, [_v(8192, (3, 2), torch.float32)], [_v(0, (10, 2))])        # ceil(10 / 4) = 3
    _refused("multiples of 16 bytes", 2, 0, [_v(8192, (4, 2), torch.float32)], [_v(0, (6, 2))], shard_rows=4)   # d * W = 12 bf16
    _refused("16-byte aligned", 4, 0, shards[:1], [_v(_off(fulls[0]) + 8, (32, 16))])
    _refused("16-byte aligned", 4, 0, [_v(_off(shards[0]) + 4, (8, 16), torch.float32)], fulls[:1])
    # a rank with no rows needs no shard rows and no aligned shard
    assert coll.check_all_gather_shards(8, 7, [_v(4, (0, 8), torch.float32)], [_v(0, (3, 8))]) == [(3, 8, 1)]
    # overlaps: an output on a source, two outputs, and the reduce-scatter's shard rows on a gradient
    _refused("output 0 overlaps source 0", 4, 0, shards[:1], [_v(_off(shards[0]) + 256, (32, 16))])
    _refused("outputs 0 and 1 overlap", 4, 0, shards[:2], [fulls[0], _v(_off(fulls[0]) + 512, (64,))])
    _refused("output 1 overlaps source 0", 4, 0, [shards[0], _v(_off(fulls[0]), (32,), torch.float32)], fulls[:2], gather=False)
    _refused("outputs 0 and 1 overlap", 4, 0, [shards[0], _v(_off(shards[0]) + 16, (32,), torch.float32)], fulls[:2], gather=False)
    # padding rows past n_r are never written, so another tensor may live there
    pad = _v(0, (8, 16), torch.float32)
    assert coll.check_reduce_scatter_shards(4, 3, [_v(8192, (30, 16)), _v(16384, (64,))],
                                            [pad, _v(384, (16,), torch.float32)])[0] == (30, 16, 8)     # rank 3: 6 of 8 rows


def test_check_refuses_2_31_vectors():
    huge = torch.empty((1 << 24, 4096), dtype=torch.bfloat16, device="meta")     # 2^37 bytes of fp32: 2^33 vectors in the shard's dtype
    with pytest.raises(ValueError, match="2\\^31 - 1"):
        coll.check_all_gather_shards(8, 0, [torch.empty((1 << 21, 4096), dtype=torch.float32, device="meta")], [huge])
    many = [torch.empty((1 << 16, 4096), dtype=torch.bfloat16, device="meta")] * 64                      # 64 x 2^25 = 2^31 vectors
    with pytest.raises(ValueError, match="in the call"):
        coll.check_all_gather_shards(1, 0, many, many)


def test_comm_methods_refuse_missing_outputs():
    """More than one rank needs the gather's fulls and the reduce-scatter's shards passed, and accumulation needs the old shards. The
    refusal comes before anything reaches the library, so a communicator stand-in is enough."""
    class Fake:
        nranks, rank = 2, 0
    shards, fulls = _unit(2)
    with pytest.raises(ValueError, match="needs fulls"):
        coll.Comm.all_gather_shards(Fake(), shards)
    with pytest.raises(ValueError, match="needs shards"):
        coll.Comm.reduce_scatter_shards(Fake(), fulls)
    Fake.nranks = 1
    with pytest.raises(ValueError, match="needs shards"):
        coll.Comm.reduce_scatter_shards(Fake(), fulls, accumulate=True)
    with pytest.raises(TypeError):
        coll.Comm.reduce_scatter_shards(Fake(), fulls, shards, 0.5)                    # scale is keyword-only


# ------------------------------------------------------------------------------------------------- what the compiler made
def test_one_instantiation_per_dtype_pair_and_locality(coll_lib):
    g = kernels(coll_lib, "b200coll::k_shard_gather<")
    # a bit copy is one kernel whatever the dtype; the casts are fp32 -> bf16 and fp32 -> fp16
    assert sorted(template_args(nm) for nm in g) == sorted((s, f, loc) for s, f in (("float", "float"), ("float", "__nv_bfloat16"),
                                                                                      ("float", "__half")) for loc in ("false", "true")), g
    rs = kernels(coll_lib, "b200coll::k_shard_rs<")
    pairs = [("__nv_bfloat16", "__nv_bfloat16"), ("__half", "__half"), ("float", "float"), ("__nv_bfloat16", "float"), ("__half", "float")]
    assert sorted(template_args(nm) for nm in rs) == sorted((f, s, loc) for f, s in pairs for loc in ("false", "true")), rs


def test_ptxas_new_kernels_no_stack_no_spills():
    report, regs = ptxas("shards.cu")
    mine = {k: v for k, v in report.items() if "k_shard_" in k}
    assert len(mine) == 16, sorted(report)
    for k, (stack, st, ld) in mine.items():
        assert (stack, st, ld) == (0, 0, 0), (k, stack, st, ld)
        assert regs[k] <= 64, (k, regs[k])                     # two 512-thread CTAs per SM


# ------------------------------------------------------------------------------------------------- perf tool
def test_perf_tool_help_and_refusals(coll_lib):
    h = subprocess.run([PERF, "--help"], capture_output=True, text=True)
    assert h.returncode == 0 and "--fsdp H:F[:KV]" in h.stdout and "--accumulate" in h.stdout
    cases = [
        (["--fsdp", "4096"], "positive integers"),
        (["--fsdp", "4096:0"], "positive integers"),
        (["--fsdp", "4096:14336:1024:8"], "positive integers"),
        (["--fsdp", "a:b"], "positive integers"),
        (["--op", "all_reduce", "--fsdp", "256:512"], "takes --op all_gather or reduce_scatter"),
        (["--op", "all_gather", "--fsdp", "256:512", "--ulysses", "32:8:128"], "takes --op all_gather or reduce_scatter"),
        (["--op", "all_gather", "--fsdp", "256:512", "--context", "512:2"], "takes --op all_gather or reduce_scatter"),
        (["--op", "all_gather", "--fsdp", "256:512", "--accumulate"], "--accumulate and --scale take --op reduce_scatter"),
        (["--op", "all_gather", "--fsdp", "256:512", "--scale", "0.5"], "--accumulate and --scale take --op reduce_scatter"),
        (["--op", "all_gather", "-d", "bfloat16", "--out-dtype", "float", "--fsdp", "256:512"], "dtype pair"),
        (["--op", "reduce_scatter", "-d", "float", "--out-dtype", "bfloat16", "--fsdp", "256:512"], "dtype pair"),
        (["--op", "reduce_scatter", "-d", "e4m3", "--fsdp", "256:512"], "dtype pair"),
        (["--accumulate"], "--accumulate takes --fsdp"),
    ]
    for args, msg in cases:
        r = subprocess.run([PERF, *args], capture_output=True, text=True)
        assert r.returncode == 1 and msg in r.stderr, (args, r.stderr)
