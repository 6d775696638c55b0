"""The fused reduce-scatter, residual add and RMSNorm (wide and FP8) for sequence-parallel layers in libb200coll, checked without a GPU:
the C prototypes against the ctypes argtypes, every Python refusal, the kernels' instantiations, ptxas's register, stack and spill report
(the new kernels, and the all-reduce kernels beside them), the perf tool's help and refusals, and the shard reference against a plain
loop rendering of the same rules."""
import ctypes as C
import os
import subprocess

import pytest
import torch

from container_engine_accelerators_b200.ops import coll
from tests import coll_rs_rmsnorm_reference as ref
from tests.coll_binary_facts import kernels, ptxas, template_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PERF = os.path.join(ROOT, "build", "b200coll_perf")
WIDE = ("__nv_bfloat16", "__half", "float")
WIRES = ("__nv_fp8_e4m3", "__nv_fp8_e5m2")


def test_header_prototypes_match_the_ctypes_argtypes(tmp_path, coll_lib):
    src = tmp_path / "probe.c"
    src.write_text(r'''
#include <stdio.h>
#include "b200coll.h"
int main(void) {
  b200collResult_t (*f)(const void*, void*, const void*, void*, size_t, size_t, float, int, b200collDataType_t, b200collComm_t,
                        b200collStream_t) = b200collReduceScatterRmsNorm;
  b200collResult_t (*g)(const void*, void*, const void*, void*, float*, size_t, size_t, float, int, b200collDataType_t, b200collDataType_t,
                        int, b200collComm_t, b200collStream_t) = b200collReduceScatterRmsNormQuantized;
  printf("%d %d\n", f != 0, g != 0);
  return 0;
}''')
    exe = tmp_path / "probe"
    libdir = os.path.dirname(coll_lib)
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "coll", "include"), str(src), "-o", str(exe),
                    "-L", libdir, "-lb200coll", "-Wl,-rpath," + libdir], check=True)
    assert subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split() == ["1", "1"]
    L = coll.load()
    vp, sz, ci = C.c_void_p, C.c_size_t, C.c_int
    assert L.b200collReduceScatterRmsNorm.argtypes == [vp, vp, vp, vp, sz, sz, C.c_float, ci, ci, vp, vp]
    assert L.b200collReduceScatterRmsNormQuantized.argtypes == [vp, vp, vp, vp, C.POINTER(C.c_float), sz, sz, C.c_float, ci, ci, ci, ci, vp, vp]


# ------------------------------------------------------------------------------------------------- Python argument checks
_pool = torch.empty(1 << 16, dtype=torch.float32)


def _v(off, n, dt):
    """n elements of dt at byte offset `off` of one pool (so alignment and overlaps are under the test's control)."""
    es = torch.empty((), dtype=dt).element_size()
    return _pool.view(torch.uint8)[off:off + n * es].view(dt)


def _off(t):
    return t.data_ptr() - _pool.data_ptr()


def _wide(nranks=2, rows=8, row_len=256, dt=torch.bfloat16, gather=False, **kw):
    es = torch.empty((), dtype=dt).element_size()
    s, mat = rows // max(nranks, 1), rows * row_len * es
    o = rows if gather else s
    a = {"nranks": nranks, "x": _v(0, rows * row_len, dt).view(rows, row_len), "residual": _v(mat + 64, s * row_len, dt).view(s, row_len),
         "weight": _v(2 * mat + 128, row_len, dt), "out": _v(3 * mat + 192, o * row_len, dt).view(o, row_len), "eps": 1e-6,
         "gather": gather}
    a.update(kw)
    return a


def _quant(nranks=2, rows=8, row_len=256, dt=torch.bfloat16, block=128, wire=torch.float8_e4m3fn, gather=False, **kw):
    es = torch.empty((), dtype=dt).element_size()
    s, mat = rows // nranks, rows * row_len * es
    o = rows if gather else s
    a = {"nranks": nranks, "x": _v(0, rows * row_len, dt).view(rows, row_len), "residual": _v(mat + 64, s * row_len, dt).view(s, row_len),
         "weight": _v(2 * mat + 128, row_len, dt), "q": _v(3 * mat + 192, o * row_len, wire).view(o, row_len),
         "scales": _v(4 * mat + 256, o * (row_len // block), torch.float32).view(o, row_len // block), "block": block, "wire": wire, "eps": 1e-6,
         "gather": gather}
    a.update(kw)
    return a


def test_checks_accept_valid_calls():
    for n in (1, 2, 4, 8):
        for gather in (False, True):
            for dt in (torch.bfloat16, torch.float16, torch.float32):
                assert coll.check_reduce_scatter_rms_norm(**_wide(nranks=n, dt=dt, gather=gather)) == (8, 256)
                for wire, code in ((torch.float8_e4m3fn, coll.FP8_E4M3), (torch.float8_e5m2, coll.FP8_E5M2)):
                    assert coll.check_reduce_scatter_rms_norm_quantized(**_quant(nranks=n, dt=dt, wire=wire, gather=gather)) == (8, 256, code)
    # a Megatron [s, b, h] layout shards by sequence: dim 0
    a = _wide(nranks=2, rows=8)
    assert coll.check_reduce_scatter_rms_norm(2, a["x"].view(4, 2, 256), a["residual"].view(2, 2, 256), a["weight"], a["out"].view(2, 2, 256)) == (8, 256)
    a = _quant(nranks=2, rows=8, gather=True)
    assert coll.check_reduce_scatter_rms_norm_quantized(2, a["x"].view(4, 2, 256), a["residual"].view(2, 2, 256), a["weight"], a["q"].view(4, 2, 256),
                                                        a["scales"].view(4, 2, 2), gather=True) == (8, 256, coll.FP8_E4M3)
    assert coll.check_reduce_scatter_rms_norm(**_wide(nranks=2, rows=0)) == (0, 256)


def _refused(match, **kw):
    with pytest.raises(ValueError, match=match):
        coll.check_reduce_scatter_rms_norm(**_wide(**kw))


def _refused_q(match, **kw):
    with pytest.raises(ValueError, match=match):
        coll.check_reduce_scatter_rms_norm_quantized(**_quant(**kw))


def test_shape_refusals():
    a = _wide()
    _refused("at least two dimensions", x=a["x"].reshape(-1), residual=a["residual"].reshape(-1), out=a["out"].reshape(-1))
    _refused("multiple of nranks", nranks=3)                                                  # 8 rows over 3 ranks
    _refused_q("multiple of nranks", nranks=3)
    _refused("residual must have the shard's shape", residual=_v(_off(a["residual"]), 2048, torch.bfloat16).view(8, 256))   # the full stream
    _refused("residual must have the shard's shape", residual=a["residual"].view(8, 128), row_len=256)
    _refused("out must have the shard's shape", out=_v(_off(a["out"]), 2048, torch.bfloat16).view(8, 256))
    _refused("out must have x's shape", gather=True, out=a["out"])                            # the slice, but gathering
    with pytest.raises(ValueError, match="residual must have the shard's shape"):            # [s, b, h]: dim 0 is sharded, not dim 1
        coll.check_reduce_scatter_rms_norm(2, a["x"].view(4, 2, 256), a["residual"].view(4, 1, 256), a["weight"], a["out"].view(2, 2, 256))
    q = _quant()
    _refused_q("q must be a contiguous", q=_v(_off(q["q"]), 2048, torch.float8_e4m3fn).view(8, 256))
    _refused_q("q must be a contiguous .* of x's shape", gather=True, q=q["q"], scales=_v(_off(q["scales"]), 16, torch.float32).view(8, 2))
    _refused_q("scales must be a contiguous float32 tensor of shape \\[4, 2\\]", scales=_v(_off(q["scales"]), 16, torch.float32).view(8, 2))
    _refused_q("scales must be a contiguous float32 tensor of shape \\[8, 2\\]", gather=True,         # scales sized for the slice
               scales=_v(_off(q["scales"]), 8, torch.float32).view(4, 2))


def test_refusals_shared_with_the_all_reduce_form():
    a = _wide()
    _refused("x must be a contiguous bfloat16", x=torch.zeros(8, 256, dtype=torch.float8_e4m3fn))
    _refused("weight must have x's dtype", weight=torch.zeros(256, dtype=torch.float16))
    _refused("out must have x's dtype", out=torch.zeros(4, 256, dtype=torch.float32))
    _refused("row_len", rows=8, row_len=24)
    _refused("weight must have shape", weight=a["weight"][:128])
    for eps in (-1e-6, float("nan"), float("inf"), "1e-6", True):
        _refused("eps", eps=eps)
    _refused("residual must be 16-byte aligned", residual=_v(_off(a["residual"]) + 2, 1024, torch.bfloat16).view(4, 256))
    _refused("out must be 16-byte aligned", out=_v(_off(a["out"]) + 8, 1024, torch.bfloat16).view(4, 256))
    _refused("residual must not overlap", residual=_v(128, 1024, torch.bfloat16).view(4, 256))
    _refused("residual must not overlap", residual=_v(_off(a["weight"]), 1024, torch.bfloat16).view(4, 256))
    for t in ("x", "residual", "weight"):
        _refused("out must not overlap", out=_v(_off(a[t]), 1024, torch.bfloat16).view(4, 256))
    # overlaps are sized by the gathered shape: a gathered out reaching into the residual shard
    _refused("out must not overlap", gather=True, out=_v(_off(a["residual"]) - 2048, 2048, torch.bfloat16).view(8, 256))
    q = _quant()
    _refused_q("wire must be", wire=torch.bfloat16)
    _refused_q("block must be one of", block=100, scales=q["scales"])
    _refused_q("q must be 16-byte aligned", q=_v(_off(q["q"]) + 8, 1024, torch.float8_e4m3fn).view(4, 256))
    for t in ("x", "residual", "weight"):
        _refused_q("q must not overlap", q=_v(_off(q[t]), 1024, torch.float8_e4m3fn).view(4, 256))
        _refused_q("scales must not overlap", scales=_v(_off(q[t]), 8, torch.float32).view(4, 2))


def test_comm_methods_refuse_gather_without_outputs():
    """gather=True with more than one rank needs out (q and scales): a fresh tensor cannot be arena memory. The refusal comes before
    anything reaches the library, so a communicator stand-in with nranks is enough."""
    class Fake:
        nranks = 2
    a = _wide(gather=True)
    with pytest.raises(ValueError, match="gather=True needs out"):
        coll.Comm.reduce_scatter_rms_norm(Fake(), a["x"], a["residual"], a["weight"], gather=True)
    q = _quant(gather=True)
    for kw in ({}, {"q": q["q"]}, {"scales": q["scales"]}):
        with pytest.raises(ValueError, match="gather=True needs q and scales"):
            coll.Comm.reduce_scatter_rms_norm_quantized(Fake(), q["x"], q["residual"], q["weight"], gather=True, **kw)
    with pytest.raises(ValueError, match="multiple of nranks"):
        coll.Comm.reduce_scatter_rms_norm(Fake(), a["x"][:7], a["residual"], a["weight"])


def test_check_refuses_2_31_rows():
    big = torch.empty((1 << 31, 128), dtype=torch.bfloat16, device="meta")
    half = torch.empty((1 << 30, 128), dtype=torch.bfloat16, device="meta")
    w = torch.empty(128, dtype=torch.bfloat16, device="meta")
    with pytest.raises(ValueError, match="2\\^31"):
        coll.check_reduce_scatter_rms_norm(2, big, half, w, half)


# ------------------------------------------------------------------------------------------------- what the compiler made
def test_one_instantiation_per_dtype_wire_and_gather(coll_lib):
    names = kernels(coll_lib, "b200coll::k_rs_norm<")
    assert sorted(template_args(nm) for nm in names) == sorted((t, g) for t in WIDE for g in ("false", "true")), names
    names = kernels(coll_lib, "b200coll::k_rs_normq<")
    assert sorted(template_args(nm) for nm in names) == sorted((t, w, g) for t in WIDE for w in WIRES for g in ("false", "true")), names


def test_ptxas_new_kernels_no_stack_no_spills():
    report, regs = ptxas("rmsnorm.cu")
    mine = {k: v for k, v in report.items() if "k_rs_norm" in k}
    assert len(mine) == 18, sorted(report)
    for k, (stack, st, ld) in mine.items():
        assert (stack, st, ld) == (0, 0, 0), (k, stack, st, ld)
        assert regs[k] <= 128, (k, regs[k])                    # one 512-thread CTA per SM


def test_ptxas_all_reduce_kernels_keep_their_registers():
    """The reduce-scatter kernels share rms_row with the 27 all-reduce kernels; sharing must not cost those registers or stack."""
    report, regs = ptxas("rmsnorm.cu")
    wide = {k: n for k, n in regs.items() if "k_rms_" in k}
    quant = {k: n for k, n in regs.items() if "k_rmsq_" in k}
    assert len(wide) == 9 and len(quant) == 18
    assert all(report[k] == (0, 0, 0) for k in list(wide) + list(quant))
    assert sorted(wide.values()) == [63, 63, 80, 90, 92, 96, 101, 101, 108], wide
    assert all(n <= 64 for k, n in quant.items() if "k_rmsq_local" in k and "k_rmsq_localIf" not in k), quant


# ------------------------------------------------------------------------------------------------- perf tool
def test_perf_tool_help_and_refusals(coll_lib):
    h = subprocess.run([PERF, "--help"], capture_output=True, text=True)
    assert h.returncode == 0 and "--op reduce_scatter --rms-norm ROW_LEN" in h.stdout and "--rms-norm-gather" in h.stdout
    for extra in (["--rms-norm-gather"], ["--op", "reduce_scatter", "--rms-norm-gather"], ["--op", "all_reduce", "--rms-norm", "64", "--rms-norm-gather"]):
        r = subprocess.run([PERF, *extra], capture_output=True, text=True)
        assert r.returncode == 1 and "--rms-norm-gather takes --rms-norm ROW_LEN and --op reduce_scatter" in r.stderr, (extra, r.stderr)
    for op in ("all_gather", "alltoall", "broadcast"):
        r = subprocess.run([PERF, "--op", op, "--rms-norm", "64"], capture_output=True, text=True)
        assert r.returncode == 1 and "--rms-norm ROW_LEN takes --op all_reduce or reduce_scatter" in r.stderr, (op, r.stderr)
    r = subprocess.run([PERF, "--op", "reduce_scatter", "--rms-norm", "64", "--rms-norm-quantize", "e4m3:128"], capture_output=True, text=True)
    assert r.returncode == 1 and "a multiple of BLOCK" in r.stderr, r.stderr


# ------------------------------------------------------------------------------------------------- the reference
def _loop(xs, shards, gamma, eps, dt, gather):
    """Each rank's rows one at a time through the loop rendering of steps 1-5, on that rank's own shard."""
    from tests import coll_rmsnorm_reference as R
    n, s = len(xs), shards[0].shape[0]
    per = [R.rms_norm_loop([x[r * s:(r + 1) * s] for x in xs], shards[r], gamma, eps, dt) for r in range(n)]
    full = torch.cat([o for _, o in per]) if gather else None
    return [(h, full if gather else o) for h, o in per]


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16, torch.float32])
def test_reference_agrees_with_the_loop_rendering(dt):
    from tests.coll_fp_reference import assert_same
    for n, s, row_len in ((1, 2, 32), (2, 1, 48), (3, 2, 16), (4, 1, 64)):
        g = torch.Generator().manual_seed(n * 11 + row_len)
        xs = [(torch.randn(n * s, row_len, generator=g) * (1 + r)).to(dt) for r in range(n)]
        shards = [(torch.randn(s, row_len, generator=g) * (2 + r)).to(dt) for r in range(n)]       # a different shard on every rank
        gamma = (torch.rand(row_len, generator=g) * 2 - 0.5).to(dt)
        shards[-1][0, 3] = float("inf")
        for eps in (0.0, 1e-6):
            for gather in (False, True):
                want = _loop(xs, shards, gamma, eps, dt, gather)
                got = ref.rs_rms_norm(xs, shards, gamma, eps, dt, gather)
                for r in range(n):
                    what = f"n={n} s={s} row_len={row_len} eps={eps} gather={gather} rank {r}"
                    assert_same(got[r][0], want[r][0], what + " residual")
                    assert_same(got[r][1], want[r][1], what + " out")
                    assert got[r][1].shape[0] == (n * s if gather else s), what


def test_quantised_reference_is_the_wide_slice_quantised():
    from tests import coll_quant_reference as Q
    n, s, row_len, block, dt, wire = 3, 2, 256, 128, torch.bfloat16, torch.float8_e5m2
    g = torch.Generator().manual_seed(9)
    xs = [torch.randn(n * s, row_len, generator=g).to(dt) for _ in range(n)]
    shards = [torch.randn(s, row_len, generator=g).to(dt) for _ in range(n)]
    gamma = (torch.rand(row_len, generator=g) + 0.5).to(dt)
    for gather in (False, True):
        wide = ref.rs_rms_norm(xs, shards, gamma, 1e-6, dt, gather)
        got = ref.rs_rms_norm_quantized(xs, shards, gamma, 1e-6, dt, block, wire, gather)
        for r in range(n):
            assert torch.equal(got[r][0], wide[r][0])
            out = wide[r][1]
            assert got[r][1].shape == out.shape and got[r][2].shape == (out.shape[0], row_len // block)
            for i in range(out.shape[0]):
                wq, ws, _ = Q.quantize(out[i], block, wire)
                assert torch.equal(got[r][1][i].view(torch.uint8), wq.view(torch.uint8)) and torch.equal(got[r][2][i], ws)
