"""The fused all-reduce, residual add, RMSNorm and FP8 block quantisation in libb200coll, checked without a GPU: the C prototype against
the ctypes argtypes, every Python refusal, the kernels' instantiations, ptxas's register, stack and spill report (the new kernels and the
wide ones beside them), the perf tool's help and refusals, and the reference against a plain loop rendering of the same rules."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from container_engine_accelerators_b200.ops import coll
from tests import coll_rmsnorm_quant_reference as ref
from tests.coll_binary_facts import kernels, ptxas, template_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PERF = os.path.join(ROOT, "build", "b200coll_perf")
WIDE = ("__nv_bfloat16", "__half", "float")
WIRES = ("__nv_fp8_e4m3", "__nv_fp8_e5m2")
FAMILIES = ("k_rmsq_local", "k_rmsq_oneshot", "k_rmsq_twoshot")


def test_header_prototype_matches_the_ctypes_argtypes(tmp_path, coll_lib):
    src = tmp_path / "probe.c"
    src.write_text(r'''
#include <stdio.h>
#include "b200coll.h"
int main(void) {
  b200collResult_t (*f)(const void*, void*, const void*, void*, float*, size_t, size_t, float, b200collDataType_t, b200collDataType_t, int,
                        b200collComm_t, b200collStream_t) = b200collAllReduceRmsNormQuantized;
  printf("%d\n", f != 0);
  return 0;
}''')
    exe = tmp_path / "probe"
    libdir = os.path.dirname(coll_lib)
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "coll", "include"), str(src), "-o", str(exe),
                    "-L", libdir, "-lb200coll", "-Wl,-rpath," + libdir], check=True)
    assert subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split() == ["1"]
    L = coll.load()
    vp, sz, ci = C.c_void_p, C.c_size_t, C.c_int
    assert L.b200collAllReduceRmsNormQuantized.argtypes == [vp, vp, vp, vp, C.POINTER(C.c_float), sz, sz, C.c_float, ci, ci, ci, vp, vp]


# ------------------------------------------------------------------------------------------------- Python argument checks
_pool = torch.empty(1 << 16, dtype=torch.float32)


def _v(off, n, dt):
    """n elements of dt at byte offset `off` of one pool (so alignment and overlaps are under the test's control)."""
    es = torch.empty((), dtype=dt).element_size()
    return _pool.view(torch.uint8)[off:off + n * es].view(dt)


def _args(rows=4, row_len=256, dt=torch.bfloat16, block=128, wire=torch.float8_e4m3fn, **kw):
    es = torch.empty((), dtype=dt).element_size()
    mat, ns = rows * row_len * es, max(row_len // block, 1) if type(block) is int else 1
    a = {"x": _v(0, rows * row_len, dt).view(rows, row_len), "residual": _v(mat + 64, rows * row_len, dt).view(rows, row_len),
         "weight": _v(2 * mat + 128, row_len, dt), "q": _v(3 * mat + 192, rows * row_len, wire).view(rows, row_len),
         "scales": _v(4 * mat + 256, rows * ns, torch.float32).view(rows, ns), "block": block, "wire": wire, "eps": 1e-6}
    a.update(kw)
    return a


def _off(t):
    return t.data_ptr() - _pool.data_ptr()


def test_check_accepts_a_valid_call():
    for dt in (torch.bfloat16, torch.float16, torch.float32):
        for wire, code in ((torch.float8_e4m3fn, coll.FP8_E4M3), (torch.float8_e5m2, coll.FP8_E5M2)):
            assert coll.check_all_reduce_rms_norm_quantized(**_args(dt=dt, wire=wire)) == (4, 256, code)
    for block in coll.QUANT_BLOCKS:
        assert coll.check_all_reduce_rms_norm_quantized(**_args(row_len=512, block=block)) == (4, 512, coll.FP8_E4M3)
    a = _args()
    a.pop("wire")                                                     # the default wire is e4m3
    assert coll.check_all_reduce_rms_norm_quantized(**a) == (4, 256, coll.FP8_E4M3)
    a = _args()
    assert coll.check_all_reduce_rms_norm_quantized(a["x"].view(2, 2, 256), a["residual"].view(2, 2, 256), a["weight"], a["q"].view(2, 2, 256),
                                                    a["scales"].view(2, 2, 2), block=128) == (4, 256, coll.FP8_E4M3)
    assert coll.check_all_reduce_rms_norm_quantized(**_args(rows=0)) == (0, 256, coll.FP8_E4M3)


def _refused(match, **kw):
    with pytest.raises(ValueError, match=match):
        coll.check_all_reduce_rms_norm_quantized(**_args(**kw))


def test_check_refusals_shared_with_the_wide_call():
    a = _args()
    _refused("x must be a contiguous bfloat16", x=torch.zeros(4, 256, dtype=torch.float8_e4m3fn))
    _refused("x must be a contiguous", x=torch.zeros(256, 4, dtype=torch.bfloat16).t())
    _refused("weight must have x's dtype", weight=torch.zeros(256, dtype=torch.float16))
    _refused("residual must have x's dtype", residual=torch.zeros(4, 256, dtype=torch.float32))
    _refused("residual must have x's shape", residual=a["residual"].view(-1)[:512].view(2, 256))
    _refused("row_len", rows=2, row_len=24, block=16, scales=torch.zeros(2, 1))
    _refused("row_len", rows=1, row_len=16400, block=16, scales=torch.zeros(1, 1025))
    _refused("weight must have shape", weight=a["weight"][:128])
    for eps in (-1e-6, float("nan"), float("inf"), "1e-6", True):
        _refused("eps", eps=eps)
    _refused("residual must be 16-byte aligned", residual=_v(4096 + 2, 1024, torch.bfloat16).view(4, 256))
    _refused("residual must not overlap", residual=_v(128, 1024, torch.bfloat16).view(4, 256))
    _refused("residual must not overlap", residual=_v(_off(a["weight"]), 1024, torch.bfloat16).view(4, 256))


def test_check_refusals_of_the_quantised_call():
    a = _args()
    _refused("wire must be", wire=torch.bfloat16)
    _refused("wire must be", wire=torch.float8_e4m3fnuz)
    for block in (8, 48, 100, 1024, 128.0, True, "128"):
        _refused("block must be one of", block=block, scales=a["scales"])
    _refused("must be a multiple of block", row_len=256 + 128, block=256, scales=torch.zeros(4, 1))
    _refused("q must be a contiguous", q=torch.zeros(4, 256, dtype=torch.float8_e5m2))              # not the wire dtype
    _refused("q must be a contiguous", q=torch.zeros(4, 256, dtype=torch.bfloat16))
    _refused("q must be a contiguous", q=a["q"].view(8, 128))
    _refused("q must be a contiguous", q=torch.zeros(256, 4, dtype=torch.float8_e4m3fn).t())
    _refused("scales must be a contiguous float32", scales=torch.zeros(4, 2, dtype=torch.float16))
    _refused("scales must be a contiguous float32", scales=a["scales"].view(8))
    _refused("scales must be a contiguous float32", scales=torch.zeros(4, 4))
    _refused("scales must be a contiguous float32", scales=torch.zeros(2, 4).t())
    _refused("q must be 16-byte aligned", q=_v(_off(a["q"]) + 8, 1024, torch.float8_e4m3fn).view(4, 256))
    for t in ("x", "residual", "weight"):
        _refused("q must not overlap", q=_v(_off(a[t]), 1024, torch.float8_e4m3fn).view(4, 256))
        _refused("scales must not overlap", scales=_v(_off(a[t]), 8, torch.float32).view(4, 2))
    _refused("q must not overlap", scales=_v(_off(a["q"]) + 16, 8, torch.float32).view(4, 2))


def test_check_refuses_2_31_rows():
    big = torch.empty((1 << 31, 128), dtype=torch.bfloat16, device="meta")
    w = torch.empty(128, dtype=torch.bfloat16, device="meta")
    with pytest.raises(ValueError, match="2\\^31"):
        coll.check_all_reduce_rms_norm_quantized(big, big, w, big.to(torch.float8_e4m3fn), torch.empty((1 << 31, 1), device="meta"))


# ------------------------------------------------------------------------------------------------- what the compiler made
def test_one_instantiation_per_dtype_wire_and_algorithm(coll_lib):
    want = sorted((t, w) for t in WIDE for w in WIRES)
    for fam in FAMILIES:
        names = kernels(coll_lib, f"b200coll::{fam}<")
        assert sorted(template_args(nm) for nm in names) == want, (fam, names)


def test_ptxas_new_kernels_no_stack_no_spills():
    report, regs = ptxas("rmsnorm.cu")
    mine = {k: v for k, v in report.items() if "k_rmsq_" in k}
    assert len(mine) == 18, sorted(report)
    for k, (stack, st, ld) in mine.items():
        assert (stack, st, ld) == (0, 0, 0), (k, stack, st, ld)
        assert regs[k] <= 128, (k, regs[k])                    # one 512-thread CTA per SM


def test_ptxas_one_rank_16_bit_kernels_fit_two_ctas_per_sm():
    """The one-rank kernel runs 2 CTAs of 512 threads per SM where the registers allow, as the 16-bit wide one does: 64 at most."""
    _, regs = ptxas("rmsnorm.cu")
    mine = {k: n for k, n in regs.items() if "k_rmsq_local" in k and "k_rmsq_localIf" not in k}
    assert len(mine) == 4 and all(n <= 64 for n in mine.values()), mine


def test_ptxas_wide_kernels_keep_their_registers():
    """The wide kernels share their sum, fold and normalisation with the quantising ones; sharing must not cost them registers or stack."""
    report, regs = ptxas("rmsnorm.cu")
    want = {("f", "twoshot"): 108, ("f", "oneshot"): 96, ("f", "local"): 80, ("6__half", "twoshot"): 101, ("6__half", "oneshot"): 90,
            ("6__half", "local"): 63, ("13__nv_bfloat16", "twoshot"): 101, ("13__nv_bfloat16", "oneshot"): 92, ("13__nv_bfloat16", "local"): 63}
    got = {}
    for k, n in regs.items():
        for (t, alg) in want:
            if f"k_rms_{alg}I{t}E" in k:
                got[(t, alg)] = n
                assert report[k] == (0, 0, 0), (k, report[k])
    assert got == want


# ------------------------------------------------------------------------------------------------- perf tool
def test_perf_tool_help_and_refusals(coll_lib):
    h = subprocess.run([PERF, "--help"], capture_output=True, text=True)
    assert h.returncode == 0 and "--rms-norm-quantize WIRE:BLOCK" in h.stdout
    for extra in (["--rms-norm-quantize", "e4m3:128"], ["--op", "all_reduce", "--rms-norm-quantize", "e5m2:16"]):
        r = subprocess.run([PERF, *extra], capture_output=True, text=True)
        assert r.returncode == 1 and "--rms-norm-quantize WIRE:BLOCK takes --rms-norm ROW_LEN" in r.stderr, (extra, r.stderr)
    for rl, blk in (("64", "128"), ("4160", "128"), ("4112", "32")):
        r = subprocess.run([PERF, "--rms-norm", rl, "--rms-norm-quantize", f"e4m3:{blk}"], capture_output=True, text=True)
        assert r.returncode == 1 and "a multiple of BLOCK" in r.stderr, (rl, blk, r.stderr)
    for bad in ("e4m3:100", "bf16:128", "e4m3", "e5m2:1024"):
        r = subprocess.run([PERF, "--rms-norm", "4096", "--rms-norm-quantize", bad], capture_output=True, text=True)
        assert r.returncode == 1 and "--rms-norm-quantize WIRE:BLOCK: WIRE e4m3 or e5m2" in r.stderr, (bad, r.stderr)
    r = subprocess.run([PERF, "--rms-norm", "64", "--quantize", "e4m3:128"], capture_output=True, text=True)
    assert r.returncode == 1 and "--rms-norm ROW_LEN takes --op all_reduce" in r.stderr, r.stderr


# ------------------------------------------------------------------------------------------------- the reference
def _loop(xs, res, gamma, eps, dt, block, wire):
    """Step 6 one block at a time over the loop rendering of steps 1-5, in plain np.float32 scalars."""
    from tests import coll_rmsnorm_reference as R
    from tests.coll_fp_reference import FP8_MAX, cast
    h, out = R.rms_norm_loop(xs, res, gamma, eps, dt)
    o = out.float().numpy()
    rows, row_len = o.shape
    f, fmax = np.float32, np.float32(FP8_MAX[wire])
    q = np.zeros((rows, row_len), dtype=np.float32)
    s = np.zeros((rows, row_len // block), dtype=np.float32)
    with np.errstate(all="ignore"):
        for i in range(rows):
            for b in range(row_len // block):
                blk = o[i, b * block:(b + 1) * block]
                bits = 0
                for v in blk:                                         # the largest bit pattern of |o|: NaN above inf above every number
                    bits = max(bits, int(np.float32(v).view(np.uint32)) & 0x7FFFFFFF)
                amax = np.uint32(bits).view(np.float32)
                inv, sc = f(fmax / amax), f(amax / fmax)
                if amax == 0 or inv == np.inf:
                    inv = sc = f(1.0)
                s[i, b] = sc
                for k, v in enumerate(blk):
                    q[i, b * block + k] = f(v * inv)
    return h, cast(torch.from_numpy(q), wire), torch.from_numpy(s)


@pytest.mark.parametrize("wire", [torch.float8_e4m3fn, torch.float8_e5m2])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16, torch.float32])
def test_reference_agrees_with_the_loop_rendering(dt, wire):
    from tests.coll_fp_reference import assert_same
    for n, rows, row_len, block in ((1, 2, 32, 16), (3, 2, 48, 16), (2, 1, 128, 32), (4, 2, 256, 128)):
        g = torch.Generator().manual_seed(n * 7 + row_len)
        xs = [(torch.randn(rows, row_len, generator=g) * (1 + r)).to(dt) for r in range(n)]
        res = (torch.randn(rows, row_len, generator=g) * 3).to(dt)
        gamma = (torch.rand(row_len, generator=g) * 2 - 0.5).to(dt)
        if rows > 1:
            res[1, 5] = float("inf")
        for eps in (0.0, 1e-6):
            h, q, s = ref.rms_norm_quantized(xs, res, gamma, eps, dt, block, wire)
            lh, lq, ls = _loop(xs, res, gamma, eps, dt, block, wire)
            what = f"n={n} rows={rows} row_len={row_len} block={block} eps={eps}"
            assert_same(h, lh, what + " residual")
            assert_same(q.reshape(-1), lq.reshape(-1), what + " q")
            assert_same(s.reshape(-1), ls.reshape(-1), what + " scales")
            if rows > 1:                                              # inv = 1 / sqrt(inf) = 0: the inf's block is NaN, the others 0
                assert torch.isnan(q[1, :block].float()).all() and torch.isnan(s[1, 0])
                assert (q[1, block:].float() == 0).all() and (s[1, 1:] == 1).all()


def test_reference_is_the_wide_out_quantised():
    """Step 6 quantises out as the wide call stores it (rounded to dt), not the fp32 product: on bf16 the two differ for some block."""
    from tests import coll_quant_reference as Q
    from tests import coll_rmsnorm_reference as R
    g = torch.Generator().manual_seed(5)
    xs = [torch.randn(8, 512, generator=g).to(torch.bfloat16)]
    res = torch.randn(8, 512, generator=g).to(torch.bfloat16)
    gamma = (torch.rand(512, generator=g) + 0.5).to(torch.bfloat16)
    _, q, s = ref.rms_norm_quantized(xs, res, gamma, 1e-6, torch.bfloat16, 128, torch.float8_e4m3fn)
    _, out = R.rms_norm(xs, res, gamma, 1e-6, torch.bfloat16)
    wq, ws, _ = Q.quantize(out.reshape(-1), 128, torch.float8_e4m3fn)
    assert torch.equal(q.view(torch.uint8).reshape(-1), wq.view(torch.uint8)) and torch.equal(s.reshape(-1), ws)
    h = (xs[0].float() + res.float()).to(torch.bfloat16)             # the new residual; in fp32 the same norm gives the unrounded product
    _, o_fp32 = R.rms_norm([h.float()], torch.zeros(8, 512), gamma.float(), 1e-6, torch.float32)
    fq, fs, _ = Q.quantize(o_fp32.reshape(-1), 128, torch.float8_e4m3fn)
    assert not (torch.equal(fq.view(torch.uint8), wq.view(torch.uint8)) and torch.equal(fs, ws))
