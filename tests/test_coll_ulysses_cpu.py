"""The Ulysses all-to-all (sequence -> heads and heads -> sequence) in libb200coll, checked without a GPU: the reference against a
per-element loop rendering of the header's formulas, the C prototypes against the ctypes argtypes, every Python refusal, the kernels'
instantiations, ptxas's stack and spill report, and the perf tool's help and refusals."""
import ctypes as C
import os
import subprocess

import pytest
import torch

from container_engine_accelerators_b200.ops import coll
from tests import coll_ulysses_reference as ref
from tests.coll_binary_facts import kernels, ptxas, template_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PERF = os.path.join(ROOT, "build", "b200coll_perf")


# ------------------------------------------------------------------------------------------------- the reference
@pytest.mark.parametrize("n,B,S_l,H,D", [(1, 2, 3, 4, 8), (2, 1, 3, 4, 8), (3, 2, 2, 6, 4), (4, 2, 3, 8, 8), (4, 1, 2, 2, 8), (4, 2, 2, 1, 4),
                                         (8, 1, 2, 2, 4), (6, 2, 1, 3, 4)])
def test_reference_agrees_with_the_loop_rendering(n, B, S_l, H, D):
    g = torch.Generator().manual_seed(n * 100 + H)
    xs = [torch.randn(B, S_l, H, D, generator=g).to(torch.bfloat16) for _ in range(n)]
    ys = ref.seq_to_heads(xs)
    want = ref.seq_to_heads_loop(xs)
    assert all(torch.equal(a, b) for a, b in zip(ys, want))
    assert ys[0].shape == (B, n * S_l, ref.local_heads(n, H), D * 2)
    if H % n == 0:
        back = ref.heads_to_seq([y.view(torch.bfloat16) for y in ys])
        assert all(torch.equal(a, b) for a, b in zip(back, ref.heads_to_seq_loop([y.view(torch.bfloat16) for y in ys])))
        assert all(torch.equal(a, x.view(torch.uint8)) for a, x in zip(back, xs))      # heads -> seq of seq -> heads is the identity


def test_replicated_heads_go_to_the_ranks_that_share_them():
    n, H = 8, 2                                    # GQA with 2 KV heads on 8 ranks: ranks 0-3 get head 0, ranks 4-7 head 1
    xs = [torch.arange(H, dtype=torch.float32).view(1, 1, H, 1).expand(1, 1, H, 4).contiguous() + 10 * s for s in range(n)]
    ys = ref.seq_to_heads(xs)
    for r in range(n):
        got = ys[r].view(torch.float32)[0, :, 0, 0]
        assert got.tolist() == [10 * s + r * H // n for s in range(n)], (r, got)


# ------------------------------------------------------------------------------------------------- C prototypes
def test_header_prototypes_match_the_ctypes_argtypes(tmp_path, coll_lib):
    src = tmp_path / "probe.c"
    src.write_text(r'''
#include <stddef.h>
#include <stdio.h>
#include "b200coll.h"
int main(void) {
  b200collResult_t (*f)(const b200collUlyssesTensor*, int, size_t, size_t, size_t, b200collDataType_t, b200collComm_t, b200collStream_t) =
      b200collAllToAllSeqToHeads;
  b200collResult_t (*g)(const b200collUlyssesTensor*, int, size_t, size_t, size_t, b200collDataType_t, b200collComm_t, b200collStream_t) =
      b200collAllToAllHeadsToSeq;
  printf("%d %d %zu %zu %zu %zu %zu\n", f != 0, g != 0, sizeof(b200collUlyssesTensor), offsetof(b200collUlyssesTensor, seq),
         offsetof(b200collUlyssesTensor, row_stride), offsetof(b200collUlyssesTensor, head), offsetof(b200collUlyssesTensor, heads));
  return 0;
}''')
    exe = tmp_path / "probe"
    libdir = os.path.dirname(coll_lib)
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "coll", "include"), str(src), "-o", str(exe),
                    "-L", libdir, "-lb200coll", "-Wl,-rpath," + libdir], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    T = coll.UlyssesTensor
    assert out == ["1", "1", str(C.sizeof(T)), str(T.seq.offset), str(T.row_stride.offset), str(T.head.offset), str(T.heads.offset)]
    L = coll.load()
    want = [C.POINTER(T), C.c_int, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
    assert L.b200collAllToAllSeqToHeads.argtypes == want
    assert L.b200collAllToAllHeadsToSeq.argtypes == want


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


def _packed(n=2, B=2, S_l=4, hq=8, hkv=2, D=64, dt=torch.bfloat16, off=0):
    """q, k and v as column slices of one packed [B * S_l, (hq + 2 hkv) * D] QKV, and dense head-side outputs behind it."""
    es = torch.empty((), dtype=dt).element_size()
    W = (hq + 2 * hkv) * D
    qkv = _v(off, (B * S_l, W), dt)
    xs = [qkv[:, a * D:(a + h) * D].view(B, S_l, h, D) for a, h in ((0, hq), (hq, hkv), (hq + hkv, hkv))]
    at = off + B * S_l * W * es + 64
    outs = []
    for h in (hq, hkv, hkv):
        o = _v(at, (B, n * S_l, coll.ulysses_local_heads(n, h), D), dt)
        outs.append(o)
        at += o.numel() * es + 64
    return xs, outs


def test_checks_accept_valid_calls():
    for n in (1, 2, 4, 8):
        for dt in (torch.bfloat16, torch.float16, torch.float32, torch.float8_e4m3fn, torch.float8_e5m2):
            xs, outs = _packed(n=n, dt=dt)
            B, S_l, D, per = coll.check_all_to_all_seq_to_heads(n, xs, outs)
            assert (B, S_l, D) == (2, 4, 64) and per == [(12 * 64, 8), (12 * 64, 2), (12 * 64, 2)]
            assert coll.check_all_to_all_seq_to_heads(n, xs[:1], outs[:1])[3] == [(12 * 64, 8)]
    # heads -> seq into the column slices of a packed buffer (an attention output written straight into a wider row)
    xs, outs = _packed(n=2)
    assert coll.check_all_to_all_heads_to_seq(2, outs[:1], xs[:1]) == (2, 4, 64, [(12 * 64, 8)])
    ys = [_v(1 << 19, (2, 8, 2, 64)), _v((1 << 19) + 4096, (2, 8, 2, 64))]
    assert coll.check_all_to_all_heads_to_seq(2, ys, [xs[0][:, :, :4], xs[0][:, :, 4:]])[3] == [(768, 4), (768, 4)]
    # MQA on 8 ranks, fp8 with 16-byte heads; with one token the row stride is never used, and the check passes heads * head_dim
    xs, outs = _packed(n=8, B=1, S_l=1, hq=8, hkv=1, D=16, dt=torch.float8_e4m3fn)
    assert coll.check_all_to_all_seq_to_heads(8, xs, outs)[3] == [(128, 8), (16, 1), (16, 1)]
    xs, outs = _packed(n=8, B=1, S_l=3, hq=8, hkv=1, D=16, dt=torch.float8_e4m3fn)
    assert coll.check_all_to_all_seq_to_heads(8, xs, outs)[3] == [(160, 8), (160, 1), (160, 1)]
    xs, outs = _packed(n=2, B=0)
    assert coll.check_all_to_all_seq_to_heads(2, xs, outs)[:2] == (0, 4)


def _refused(match, n, xs, outs, s2h=True):
    with pytest.raises(ValueError, match=match):
        (coll.check_all_to_all_seq_to_heads if s2h else coll.check_all_to_all_heads_to_seq)(n, xs, outs)


def test_refusals():
    xs, outs = _packed(n=2)
    _refused("1 to 3 tensors", 2, [], [])
    _refused("1 to 3 tensors", 2, xs + xs[:1], outs + outs[:1])
    _refused("one output per tensor", 2, xs, outs[:2])
    _refused("dtype must be", 2, [x.to(torch.int16) for x in xs], outs)
    _refused("every tensor must have dtype", 2, xs, [outs[0], outs[1].to(torch.float16), outs[2]])
    _refused("4-D", 2, [xs[0].reshape(8, 8, 64)], outs[:1])
    # head_dim * sizeof(dtype) a multiple of 16 bytes
    q, o = _packed(n=2, D=4)
    _refused("multiple of 16 bytes", 2, q, o)
    # shapes: heads neither a multiple nor a divisor of nranks, or the output's shape
    q, o = _packed(n=2, hq=6, hkv=2)
    _refused("multiple or a divisor of nranks", 3, q[1:], o[1:])                            # 2 KV heads on 3 ranks
    _refused("must be a contiguous \\[2, 8, 4, 64\\]", 2, xs[:1], [outs[1]])
    _refused("like the first", 2, [xs[0], xs[1][:, :2]], outs[:2])
    # row layout: strided heads, non-uniform rows, a row stride below heads * head_dim or not 16-byte aligned
    base = _v(0, (8 * 8 * 64 + 8,))
    _refused("contiguously", 2, [_v(0, (8192,)).as_strided((2, 4, 8, 64), (4 * 1024, 1024, 128, 1))], outs[:1])     # heads 128 apart
    _refused("uniformly strided", 2, [base.as_strided((2, 4, 8, 64), (4 * 512 + 64, 512, 64, 1))], outs[:1])
    _refused("row stride .* multiple of 16 bytes", 2, [base.as_strided((2, 4, 8, 64), (4 * 516, 516, 64, 1))], outs[:1])
    _refused("row stride", 2, [base.as_strided((2, 4, 8, 64), (4 * 256, 256, 64, 1))], outs[:1])
    # alignment
    mis = _v(_off(outs[0]) + 8, tuple(outs[0].shape))
    _refused("16-byte aligned", 2, xs[:1], [mis])
    # overlaps: an output on a source, on another output, or on a column of the packed buffer
    _refused("output 0 overlaps source 0", 2, xs[:1], [_v(_off(xs[0]) + 256, tuple(outs[0].shape))])
    _refused("outputs 0 and 1 overlap", 2, xs[1:], [outs[1], _v(_off(outs[1]) + 32, tuple(outs[2].shape))])
    ys = [_v(1 << 19, (2, 8, 2, 64)), _v((1 << 19) + 4096, (2, 8, 2, 64))]
    _refused("outputs 0 and 1 overlap", 2, ys, [xs[0][:, :, :4], xs[0][:, :, 3:7]], s2h=False)
    _refused("output 0 overlaps source 1", 2, [ys[0], _v(_off(xs[0]), (2, 8, 2, 64))], [xs[0][:, :, :4], xs[0][:, :, 4:]], s2h=False)


def test_heads_to_seq_refuses_the_replicated_layout():
    xs, outs = _packed(n=4, hq=8, hkv=2)
    _refused("the replicated layout has no inverse", 4, outs[1:2], xs[1:2], s2h=False)
    assert coll.check_all_to_all_heads_to_seq(4, outs[:1], xs[:1])[3] == [(12 * 64, 8)]


def test_check_refuses_2_31_vectors():
    big = torch.empty((1, 1 << 22, 32, 128), dtype=torch.bfloat16, device="meta")     # 2^22 tokens of 32 heads: 2^31 vectors
    out = torch.empty((1, 1 << 23, 16, 128), dtype=torch.bfloat16, device="meta")
    with pytest.raises(ValueError, match="2\\^31 - 1"):
        coll.check_all_to_all_seq_to_heads(2, [big], [out])


def test_comm_methods_refuse_missing_outputs():
    """More than one rank needs the outputs passed: a fresh tensor cannot be arena memory. The refusal comes before anything reaches
    the library, so a communicator stand-in with nranks is enough."""
    class Fake:
        nranks = 2
    xs, outs = _packed(n=2)
    with pytest.raises(ValueError, match="needs outs"):
        coll.Comm.all_to_all_seq_to_heads(Fake(), xs)
    with pytest.raises(ValueError, match="needs outs"):
        coll.Comm.all_to_all_heads_to_seq(Fake(), outs[:1])


# ------------------------------------------------------------------------------------------------- what the compiler made
def test_one_instantiation_per_direction_and_locality(coll_lib):
    names = kernels(coll_lib, "b200coll::k_ulysses<")
    assert sorted(template_args(nm) for nm in names) == sorted((d, l) for d in ("false", "true") for l in ("false", "true")), names


def test_ptxas_new_kernels_no_stack_no_spills():
    report, regs = ptxas("ulysses.cu")
    mine = {k: v for k, v in report.items() if "k_ulysses" in k}
    assert len(mine) == 4, sorted(report)
    for k, (stack, st, ld) in mine.items():
        assert (stack, st, ld) == (0, 0, 0), (k, stack, st, ld)
        assert regs[k] <= 64, (k, regs[k])                     # two 512-thread CTAs per SM


# ------------------------------------------------------------------------------------------------- perf tool
def test_perf_tool_help_and_refusals(coll_lib):
    h = subprocess.run([PERF, "--help"], capture_output=True, text=True)
    assert h.returncode == 0 and "--ulysses HQ:HKV:D" in h.stdout and "--ulysses-back" in h.stdout
    cases = [
        (["--ulysses", "32:8"], "three positive integers"),
        (["--ulysses", "32:0:128"], "three positive integers"),
        (["--ulysses", "a:b:c"], "three positive integers"),
        (["--op", "all_reduce", "--ulysses", "32:8:128"], "takes --op alltoall"),
        (["--op", "alltoall", "--ulysses", "32:8:128", "--scale", "2"], "takes --op alltoall"),
        (["--op", "alltoall", "--ulysses", "32:8:4"], "multiple of 16 bytes"),
        (["--op", "alltoall", "--ranks", "4", "--ulysses", "6:2:128"], "multiple or a divisor"),
        (["--op", "alltoall", "--ranks", "4", "--ulysses", "2:2:128", "--ulysses-back"], "HQ must be a multiple"),
        (["--op", "alltoall", "--ulysses-back"], "--ulysses-back takes --ulysses"),
    ]
    for args, msg in cases:
        r = subprocess.run([PERF, *args], capture_output=True, text=True)
        assert r.returncode == 1 and msg in r.stderr, (args, r.stderr)
