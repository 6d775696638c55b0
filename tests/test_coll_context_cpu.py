"""The context-parallel all-gather and reduce-scatter (b200collAllGatherContext / ReduceScatterContext) in libb200coll, checked without a
GPU: the reference against a per-element loop rendering of the header's gtok formula, the C prototypes and struct layout against the
ctypes argtypes, every Python refusal, the kernels' instantiations, ptxas's stack and spill report, and the perf tool's help and
refusals."""
import ctypes as C
import os
import subprocess

import pytest
import torch

from container_engine_accelerators_b200.ops import coll
from tests import coll_context_reference as ref
from tests import coll_fp_reference as R
from tests.coll_binary_facts import kernels, ptxas, template_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PERF = os.path.join(ROOT, "build", "b200coll_perf")


# ------------------------------------------------------------------------------------------------- the reference
@pytest.mark.parametrize("n,B,S_l,chunks", [(1, 2, 3, 1), (1, 1, 4, 2), (2, 1, 3, 1), (2, 2, 4, 2), (3, 2, 2, 2), (4, 1, 6, 2), (4, 3, 5, 1),
                                            (6, 1, 2, 2), (8, 2, 4, 2)])
def test_reference_agrees_with_the_loop_rendering(n, B, S_l, chunks):
    g = torch.Generator().manual_seed(n * 100 + S_l)
    shards = [torch.randn(B, S_l, 2, 4, generator=g).to(torch.bfloat16) for _ in range(n)]
    full = ref.all_gather(shards, chunks)
    assert full.shape == (B, n * S_l, 16)
    assert torch.equal(full, ref.all_gather_loop(shards, chunks))
    for dt in (torch.bfloat16, torch.float16, torch.float32):
        fulls = [x.view(B, n * S_l, 8) for x in R.gen_inputs(n, B * n * S_l * 8, dt, seed=n + S_l, device="cpu")]
        got, want = ref.reduce_scatter(fulls, chunks), ref.reduce_scatter_loop(fulls, chunks)
        for a, b in zip(got, want):
            assert torch.equal(a.view(R.INT_VIEW[R.esize(dt)]), b.view(R.INT_VIEW[R.esize(dt)])), (dt, n)


def test_load_balanced_layout():
    """C = 2 on 4 ranks: rank r holds chunks r and 7 - r of the 8, so every rank holds one early and one late chunk of a causal mask."""
    n, S_l = 4, 4
    holders = [[ref.gtok(n, 2, S_l, r, t) // 2 for t in range(S_l)] for r in range(n)]
    assert holders == [[0, 0, 7, 7], [1, 1, 6, 6], [2, 2, 5, 5], [3, 3, 4, 4]]
    assert [ref.gtok(n, 1, S_l, 2, t) for t in range(S_l)] == [8, 9, 10, 11]
    assert sorted(int(i) for i in ref.token_index(n, 2, S_l)) == list(range(n * S_l))


def test_reduce_scatter_of_the_gather_is_n_times_the_shard():
    """Every rank contributing the gathered tensor unchanged: the reduce-scatter gives each rank N times its own shard (exact here)."""
    n, B, S_l = 4, 2, 6
    shards = [torch.arange(B * S_l * 8, dtype=torch.float32).view(B, S_l, 8) * 0.25 + 100 * r for r in range(n)]
    full = ref.all_gather(shards, 2).view(torch.float32).view(B, n * S_l, 8)
    back = ref.reduce_scatter([full] * n, 2)
    assert all(torch.equal(b, n * x) for b, x in zip(back, shards))


# ------------------------------------------------------------------------------------------------- C prototypes
def test_header_prototypes_match_the_ctypes_argtypes(tmp_path, coll_lib):
    src = tmp_path / "probe.c"
    src.write_text(r'''
#include <stddef.h>
#include <stdio.h>
#include "b200coll.h"
int main(void) {
  b200collResult_t (*f)(const b200collContextTensor*, int, size_t, size_t, int, b200collDataType_t, b200collComm_t, b200collStream_t) =
      b200collAllGatherContext;
  b200collResult_t (*g)(const b200collContextTensor*, int, size_t, size_t, int, b200collDataType_t, b200collComm_t, b200collStream_t) =
      b200collReduceScatterContext;
  printf("%d %d %zu %zu %zu %zu %zu\n", f != 0, g != 0, sizeof(b200collContextTensor), offsetof(b200collContextTensor, shard),
         offsetof(b200collContextTensor, row_stride), offsetof(b200collContextTensor, full), offsetof(b200collContextTensor, width));
  return 0;
}''')
    exe = tmp_path / "probe"
    libdir = os.path.dirname(coll_lib)
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "coll", "include"), str(src), "-o", str(exe),
                    "-L", libdir, "-lb200coll", "-Wl,-rpath," + libdir], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    T = coll.ContextTensor
    assert out == ["1", "1", str(C.sizeof(T)), str(T.shard.offset), str(T.row_stride.offset), str(T.full.offset), str(T.width.offset)]
    L = coll.load()
    want = [C.POINTER(T), C.c_int, C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    assert L.b200collAllGatherContext.argtypes == want
    assert L.b200collReduceScatterContext.argtypes == want


# ------------------------------------------------------------------------------------------------- Python argument checks
_pool = torch.empty(1 << 18, dtype=torch.float32)


def _v(off, shape, dt=torch.bfloat16):
    """A contiguous tensor of `shape` at byte offset `off` of one pool (alignment and overlaps under the test's control)."""
    es = torch.empty((), dtype=dt).element_size()
    n = 1
    for d in shape:
        n *= d
    return _pool.view(torch.uint8)[off:off + n * es].view(dt).view(shape)


def _off(t):
    return t.data_ptr() - _pool.data_ptr()


def _packed(n=2, B=1, S_l=4, hq=8, hkv=2, D=64, dt=torch.bfloat16, off=0):
    """K and V as column slices of one packed [B * S_l, (hq + 2 hkv) * D] QKV, and dense full tensors behind it."""
    es = torch.empty((), dtype=dt).element_size()
    W = (hq + 2 * hkv) * D
    qkv = _v(off, (B * S_l, W), dt)
    shards = [qkv[:, a * D:(a + hkv) * D].view(B, S_l, hkv, D) for a in (hq, hq + hkv)]
    at = off + B * S_l * W * es + 64
    fulls = []
    for _ in range(2):
        f = _v(at, (B, n * S_l, hkv, D), dt)
        fulls.append(f)
        at += f.numel() * es + 64
    return shards, fulls


def test_checks_accept_valid_calls():
    for n in (1, 2, 4, 8):
        for dt in (torch.bfloat16, torch.float16, torch.float32, torch.float8_e4m3fn, torch.float8_e5m2):
            for chunks in (1, 2):
                shards, fulls = _packed(n=n, B=2, dt=dt)
                assert coll.check_all_gather_context(n, shards, fulls, chunks) == (2, 4, [(12 * 64, 128), (12 * 64, 128)])
                if dt.itemsize > 1:
                    assert coll.check_reduce_scatter_context(n, fulls, shards, chunks) == (2, 4, [(12 * 64, 128), (12 * 64, 128)])
    # MLA: c_kv (512) and k_pe (64) of different widths, dense [B, S_l, W] shards; the 16-byte minimum; odd S_l with C = 1
    a, b = _v(0, (1, 3, 512)), _v(4096, (1, 3, 64))
    fa, fb = _v(8192, (1, 6, 512)), _v(16384, (1, 6, 64))
    assert coll.check_all_gather_context(2, [a, b], [fa, fb], 1) == (1, 3, [(512, 512), (64, 64)])
    assert coll.check_reduce_scatter_context(2, [fa, fb], [a, b], 1)[2] == [(512, 512), (64, 64)]
    assert coll.check_all_gather_context(2, [_v(0, (1, 2, 8))], [_v(1024, (1, 4, 8))], 2) == (1, 2, [(8, 8)])
    # one token: the row stride is never used, and the check passes the width
    shards, fulls = _packed(n=2, S_l=1)
    assert coll.check_all_gather_context(2, shards, fulls, 1)[2] == [(128, 128), (128, 128)]
    shards, fulls = _packed(n=2, B=0)
    assert coll.check_all_gather_context(2, shards, fulls, 2)[:2] == (0, 4)


def _refused(match, n, shards, fulls, chunks=2, gather=True):
    with pytest.raises(ValueError, match=match):
        if gather:
            coll.check_all_gather_context(n, shards, fulls, chunks)
        else:
            coll.check_reduce_scatter_context(n, fulls, shards, chunks)


def test_refusals():
    shards, fulls = _packed(n=2)
    _refused("1 to 3 tensors", 2, [], [])
    _refused("1 to 3 tensors", 2, shards * 2, fulls * 2)
    _refused("one full tensor per shard", 2, shards, fulls[:1])
    _refused("dtype must be", 2, [s.to(torch.int16) for s in shards], fulls)
    for dt in (torch.float8_e4m3fn, torch.float8_e5m2):
        s8, f8 = _packed(n=2, dt=dt)
        _refused("dtype must be", 2, s8, f8, gather=False)
    _refused("every tensor must have dtype", 2, shards, [fulls[0], fulls[1].to(torch.float16)])
    _refused("chunks must be 1 or 2", 2, shards, fulls, chunks=3)
    _refused("chunks must be 1 or 2", 2, shards, fulls, chunks=0)
    s3, f3 = _packed(n=2, S_l=3)
    _refused("even seq_local", 2, s3, f3, chunks=2)
    assert coll.check_all_gather_context(2, s3, f3, 1)[1] == 3
    _refused("at least 3-D", 2, [shards[0].reshape(4, 128)], fulls[:1])
    # width * sizeof(dtype) a multiple of 16 bytes
    _refused("multiple of 16 bytes", 2, [_v(0, (1, 4, 4))], [_v(1024, (1, 8, 4))])
    # shapes: the shards' [B, S_l] and the full's shape
    _refused("like the first", 2, [shards[0], shards[1][:, :2]], fulls)
    _refused("must be a contiguous \\[1, 8, 2, 64\\]", 2, shards[:1], [_v(_off(fulls[0]), (1, 6, 2, 64))])
    _refused("must be a contiguous", 2, shards[:1], [fulls[0].transpose(2, 3)])
    # row layout: non-contiguous rows, non-uniform rows, a row stride below the width or not 16-byte aligned
    base = _v(0, (8192,))
    _refused("contiguously", 2, [base.as_strided((1, 4, 2, 64), (4 * 512, 512, 128, 1))], fulls[:1])
    _refused("uniformly strided", 2, [base.as_strided((2, 4, 128), (4 * 512 + 64, 512, 1))], [_v(1 << 19, (2, 8, 128))])
    _refused("row stride .* multiple of 16 bytes", 2, [base.as_strided((1, 4, 128), (4 * 132, 132, 1))], [_v(1 << 19, (1, 8, 128))])
    _refused("row stride", 2, [base.as_strided((1, 4, 128), (4 * 64, 64, 1))], [_v(1 << 19, (1, 8, 128))])
    # alignment
    mis = _v(_off(fulls[0]) + 8, tuple(fulls[0].shape))
    _refused("16-byte aligned", 2, shards[:1], [mis])
    # overlaps: an output on a source, on another output, or two shards in the same columns of the packed buffer
    _refused("output 0 overlaps source 0", 2, shards[:1], [_v(_off(shards[0]) + 256, tuple(fulls[0].shape))])
    _refused("outputs 0 and 1 overlap", 2, shards, [fulls[0], _v(_off(fulls[0]) + 32, tuple(fulls[1].shape))])
    wide = _v(0, (4, 12 * 64))                                              # the packed buffer _packed slices K and V from
    a = wide[:, 8 * 64:10 * 64].view(1, 4, 2, 64)
    b = wide[:, 9 * 64:11 * 64].view(1, 4, 2, 64)
    _refused("outputs 0 and 1 overlap", 2, [a, b], fulls, gather=False)
    _refused("output 0 overlaps source 0", 2, [a], [_v(_off(wide) + 512, (1, 8, 2, 64))], gather=False)
    # the disjoint K and V slices of one packed dQKV are fine
    assert coll.check_reduce_scatter_context(2, fulls, shards, 2)[0] == 1


def test_check_refuses_2_31_vectors():
    big = torch.empty((1, 1 << 22, 1024), dtype=torch.bfloat16, device="meta")     # 2^22 tokens of 1024 bf16: 2^29 vectors per shard
    full = torch.empty((1, 1 << 25, 1024), dtype=torch.bfloat16, device="meta")    # 8 ranks: 2^32 vectors in the full tensor
    with pytest.raises(ValueError, match="2\\^31 - 1"):
        coll.check_all_gather_context(8, [big], [full], 2)
    with pytest.raises(ValueError, match="below 2\\^31"):
        coll.check_all_gather_context(1, [torch.empty((2, 1 << 30, 8), dtype=torch.bfloat16, device="meta")],
                                      [torch.empty((2, 1 << 30, 8), dtype=torch.bfloat16, device="meta")], 2)


def test_comm_methods_refuse_missing_outputs():
    """More than one rank needs the gather's fulls passed: a fresh tensor cannot be arena memory. The refusal comes before anything
    reaches the library, so a communicator stand-in with nranks is enough. chunks has no default."""
    class Fake:
        nranks = 2
    shards, fulls = _packed(n=2)
    with pytest.raises(ValueError, match="needs fulls"):
        coll.Comm.all_gather_context(Fake(), shards, chunks=2)
    with pytest.raises(TypeError):
        coll.Comm.all_gather_context(Fake(), shards, fulls)


# ------------------------------------------------------------------------------------------------- what the compiler made
def test_one_instantiation_per_direction_type_and_locality(coll_lib):
    g = kernels(coll_lib, "b200coll::k_cp_gather<")
    assert sorted(template_args(nm) for nm in g) == [("false",), ("true",)], g
    rs = kernels(coll_lib, "b200coll::k_cp_rs<")
    # one rank is a bit copy whatever the dtype: one local kernel
    assert sorted(template_args(nm) for nm in rs) == sorted([("__half", "false"), ("__nv_bfloat16", "false"), ("float", "false"),
                                                             ("float", "true")]), rs


def test_ptxas_new_kernels_no_stack_no_spills():
    report, regs = ptxas("context.cu")
    mine = {k: v for k, v in report.items() if "k_cp_" in k}
    assert len(mine) == 6, sorted(report)
    for k, (stack, st, ld) in mine.items():
        assert (stack, st, ld) == (0, 0, 0), (k, stack, st, ld)
        assert regs[k] <= 64, (k, regs[k])                     # two 512-thread CTAs per SM


# ------------------------------------------------------------------------------------------------- perf tool
def test_perf_tool_help_and_refusals(coll_lib):
    h = subprocess.run([PERF, "--help"], capture_output=True, text=True)
    assert h.returncode == 0 and "--context W:C | HQ:HKV:D:C" in h.stdout
    cases = [
        (["--context", "512"], "positive integers, C 1 or 2"),
        (["--context", "512:3"], "positive integers, C 1 or 2"),
        (["--context", "0:2"], "positive integers, C 1 or 2"),
        (["--context", "32:8:128"], "positive integers, C 1 or 2"),
        (["--context", "32:8:128:2:1"], "positive integers, C 1 or 2"),
        (["--context", "a:b"], "positive integers, C 1 or 2"),
        (["--op", "all_reduce", "--context", "512:2"], "takes --op all_gather or reduce_scatter"),
        (["--op", "all_gather", "--context", "512:2", "--scale", "2"], "takes --op all_gather or reduce_scatter"),
        (["--op", "all_gather", "--context", "512:2", "--ulysses", "32:8:128"], "takes --op all_gather or reduce_scatter"),
        (["--op", "reduce_scatter", "-d", "e4m3", "--context", "512:2"], "takes -d bfloat16|half|float"),
        (["--op", "all_gather", "--context", "4:2"], "multiple of 16 bytes"),
        (["--op", "all_gather", "--context", "3:1:4:2"], "multiple of 16 bytes"),
    ]
    for args, msg in cases:
        r = subprocess.run([PERF, *args], capture_output=True, text=True)
        assert r.returncode == 1 and msg in r.stderr, (args, r.stderr)
