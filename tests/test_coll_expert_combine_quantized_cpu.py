"""The quantising expert combine in libb200coll, checked without a GPU: both C prototypes against the ctypes argtypes, the Python argument
checks, the pull kernels' instantiations (and the quantise pass they reuse), their SASS (FP8 unpack, separate multiply and add, no fused
multiply-add, no multimem loads) and ptxas's register, stack and spill report, and the perf tool's mode."""
import ctypes as C
import os
import re
import subprocess

import pytest
import torch

from container_engine_accelerators_b200.ops import coll
from tests.coll_binary_facts import kernels, ptxas, sass, template_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E4, E5 = torch.float8_e4m3fn, torch.float8_e5m2
WIDE = ("__nv_bfloat16", "__half", "float")
WIRES = ("__nv_fp8_e4m3", "__nv_fp8_e5m2")
MAPS = ("b200coll::SegmentMap", "b200coll::RouteMap")
FAMILIES = ("k_fp8_combine_pull", "k_fp8_combine_local")
# name patterns other test files count or filter kernels by
FOREIGN = ("k_combine_", "k_routed_", "k_quant_", "k_bsq_", "k_a2av_quant_", "k_expert_quant_push")


def test_header_prototypes_match_the_ctypes_argtypes(tmp_path, coll_lib):
    src = tmp_path / "probe.c"
    src.write_text(r'''
#include <stdio.h>
#include "b200coll.h"
int main(void) {
  b200collResult_t (*a)(const void*, void*, size_t, size_t, const int64_t*, const int64_t*, const int64_t*, const int32_t*, const float*, size_t, int,
                        b200collDataType_t, int, const b200collEpilogue*, b200collComm_t, b200collStream_t) = b200collAllToAllvCombineQuantized;
  b200collResult_t (*e)(const void*, void*, size_t, size_t, const int32_t*, const float*, size_t, int, b200collDataType_t, int, const b200collEpilogue*,
                        b200collComm_t, b200collStream_t) = b200collExpertCombineQuantized;
  printf("%d %d\n", a != 0, e != 0);
  return 0;
}''')
    exe = tmp_path / "probe"
    libdir = os.path.dirname(coll_lib)
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "coll", "include"), str(src), "-o", str(exe),
                    "-L", libdir, "-lb200coll", "-Wl,-rpath," + libdir], check=True)
    assert subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split() == ["1", "1"]
    L = coll.load()
    vp, sz, ci, i32, i64, f32 = C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_float)
    ep = C.POINTER(coll.Epilogue)
    assert L.b200collAllToAllvCombineQuantized.argtypes == [vp, vp, sz, sz, i64, i64, i64, i32, f32, sz, ci, ci, ci, ep, vp, vp]
    assert L.b200collExpertCombineQuantized.argtypes == [vp, vp, sz, sz, i32, f32, sz, ci, ci, ci, ep, vp, vp]


# ------------------------------------------------------------------------------------------------- Python argument checks
def _t(n, dt):
    return torch.empty(n, dtype=dt)


_base = torch.empty(1 << 14, dtype=torch.int32)


def _a(**kw):
    """A valid all-to-all-v combine for 2 ranks: 5 tokens, top-2, rows of 64 bf16 elements, block 32, 10 expert_out rows; rank 0 sent rows
    [0, 3) to itself (landing at row 0) and [3, 7) to rank 1 (landing at row 2). Keyword arguments override."""
    a = dict(nranks=2, expert_out=_t(10 * 64, torch.bfloat16), out=_t(5 * 64, torch.float32), row_elems=64, send_rows=[3, 4], send_row_off=[0, 3],
             recv_row_off_at_peer=[0, 2], index=torch.zeros(5, 2, dtype=torch.int32), weights=torch.ones(5, 2), block=32, wire=None)
    a.update(kw)
    return a


def _e(**kw):
    """A valid expert combine for 2 ranks: 5 tokens, top-3, rows of 64 fp16 elements, block 64, 12 expert_out rows."""
    a = dict(nranks=2, expert_out=_t(12 * 64, torch.float16), route=torch.zeros(5, 3, dtype=torch.int32), weights=None,
             out=torch.empty(5, 64, dtype=torch.bfloat16), block=64, wire=E5)
    a.update(kw)
    return a


def test_checks_accept_the_documented_shapes():
    assert coll.check_all_to_all_v_combine_quantized(**_a()) == (coll.BF16, coll.F32, coll.FP8_E4M3)
    assert coll.check_all_to_all_v_combine_quantized(**_a(wire=E5, block=64, weights=None)) == (coll.BF16, coll.F32, coll.FP8_E5M2)
    assert coll.check_expert_combine_quantized(**_e()) == (coll.F16, coll.BF16, coll.FP8_E5M2)
    assert coll.check_expert_combine_quantized(**_e(wire=E4, block=16, weights=torch.ones(5, 3))) == (coll.F16, coll.BF16, coll.FP8_E4M3)
    # one rank, no tokens, fp32 in 512-element blocks
    assert coll.check_expert_combine_quantized(1, _t(3 * 512, torch.float32), torch.zeros(0, 8, dtype=torch.int32), None,
                                               torch.empty(0, 512), block=512) == (coll.F32, coll.F32, coll.FP8_E4M3)
    # the wide checks are unchanged
    assert coll.check_all_to_all_v_combine(**{k: v for k, v in _a(row_elems=48, expert_out=_t(10 * 48, torch.bfloat16), out=_t(5 * 48, torch.float32)).items()
                                              if k not in ("block", "wire")}) == (coll.BF16, coll.F32)
    assert coll.check_expert_combine(2, _t(12 * 48, torch.float16), torch.zeros(5, 3, dtype=torch.int32), None, torch.empty(5, 48)) == (coll.F16, coll.F32)


@pytest.mark.parametrize("what, kw", [
    ("FP8 expert_out", dict(expert_out=_t(10 * 64, E4))),
    ("FP8 out", dict(out=_t(5 * 64, E4))),
    ("int32 out", dict(out=_t(5 * 64, torch.int32))),
    ("bf16 wire", dict(wire=torch.bfloat16)),
    ("uint8 wire", dict(wire=torch.uint8)),
    ("block 24", dict(block=24)),
    ("block 1024", dict(block=1024)),
    ("block True", dict(block=True)),
    ("row_elems % block", dict(block=128)),
    ("row_elems 0", dict(row_elems=0)),
    ("row_elems not an int", dict(row_elems=64.0)),
    ("expert_out of part of a row", dict(expert_out=_t(10 * 64 - 32, torch.bfloat16))),
    ("int64 index", dict(index=torch.zeros(5, 2, dtype=torch.int64))),
    ("top_k 0", dict(index=torch.zeros(5, 0, dtype=torch.int32), weights=None)),
    ("weights of another shape", dict(weights=torch.ones(5, 3))),
    ("fp16 weights", dict(weights=torch.ones(5, 2, dtype=torch.float16))),
    ("out of other tokens", dict(out=_t(4 * 64, torch.float32))),
    ("send_rows of one rank", dict(send_rows=[3])),
    ("negative send_row_off", dict(send_row_off=[0, -3])),
    ("destination past expert_out", dict(recv_row_off_at_peer=[0, 7])),
    ("overlapping send ranges", dict(send_row_off=[0, 2])),
    ("out overlaps expert_out", dict(expert_out=_base[:320].view(torch.bfloat16), out=_base[300:620].view(torch.float32))),
    ("out overlaps index", dict(index=_base[:10].view(5, 2), out=_base[5:325].view(torch.float32))),
    ("out overlaps weights", dict(weights=_base[:10].view(torch.float32).view(5, 2), out=_base[9:329].view(torch.float32))),
])
def test_all_to_all_v_check_raises_value_error(what, kw):
    with pytest.raises((ValueError, RuntimeError, TypeError)) as e:
        coll.check_all_to_all_v_combine_quantized(**_a(**kw))
    assert e.type is ValueError, (what, e.value)


@pytest.mark.parametrize("what, kw", [
    ("FP8 expert_out", dict(expert_out=_t(12 * 64, E4))),
    ("1-D out", dict(out=_t(5 * 64, torch.bfloat16))),
    ("FP8 out", dict(out=torch.empty(5, 64, dtype=E4))),
    ("non-contiguous out", dict(out=torch.empty(64, 5, dtype=torch.bfloat16).t())),
    ("int8 wire", dict(wire=torch.int8)),
    ("block 8", dict(block=8)),
    ("block 96", dict(block=96)),
    ("row_elems % block", dict(block=128)),
    ("expert_out of part of a row", dict(expert_out=_t(12 * 64 + 16, torch.float16))),
    ("int64 route", dict(route=torch.zeros(5, 3, dtype=torch.int64))),
    ("route of other tokens", dict(route=torch.zeros(4, 3, dtype=torch.int32))),
    ("weights of another shape", dict(weights=torch.ones(5, 2))),
    ("out overlaps expert_out", dict(expert_out=_base[:384].view(torch.float16), out=_base[380:540].view(torch.bfloat16).view(5, 64))),
    ("out overlaps route", dict(route=_base[:15].view(5, 3), out=_base[14:174].view(torch.bfloat16).view(5, 64))),
])
def test_expert_check_raises_value_error(what, kw):
    with pytest.raises((ValueError, RuntimeError, TypeError)) as e:
        coll.check_expert_combine_quantized(**_e(**kw))
    assert e.type is ValueError, (what, e.value)


@pytest.mark.parametrize("what, kw, rule", [
    ("tokens * top_k > 2^31 - 1", dict(index=torch.empty(2 ** 30, 4, dtype=torch.int32, device="meta"), weights=None,
                                       out=torch.empty(2 ** 30 * 16, dtype=torch.float32, device="meta"), row_elems=16, block=16,
                                       expert_out=_t(10 * 16, torch.bfloat16)), "tokens \\* top_k"),
    ("more than 2^31 - 1 vectors of out", dict(index=torch.empty(2 ** 26, 1, dtype=torch.int32, device="meta"), weights=None,
                                              out=torch.empty(2 ** 26 * 512, dtype=torch.bfloat16, device="meta"), row_elems=512, block=512,
                                              expert_out=_t(10 * 512, torch.bfloat16)), "vectors of out"),
    ("more than 2^31 - 1 vectors of expert_out", dict(expert_out=torch.empty(2 ** 26 * 512, dtype=torch.bfloat16, device="meta"), row_elems=512, block=512,
                                                      out=_t(5 * 512, torch.float32)), "vectors of expert_out"),
])
def test_all_to_all_v_size_limits_name_their_rule(what, kw, rule):
    """Each size limit is refused by its own rule, with every other argument valid (meta tensors: no memory behind them)."""
    with pytest.raises(ValueError, match=rule):
        coll.check_all_to_all_v_combine_quantized(**_a(**kw))


@pytest.mark.parametrize("what, kw, rule", [
    ("nranks * expert_out rows > 2^31 - 1", dict(nranks=8, expert_out=torch.empty(2 ** 28 * 64, dtype=torch.float16, device="meta")), "nranks \\* expert_out rows"),
    ("more than 2^31 - 1 vectors of out", dict(route=torch.empty(2 ** 26, 1, dtype=torch.int32, device="meta"),
                                              out=torch.empty(2 ** 26, 512, dtype=torch.bfloat16, device="meta"), block=512,
                                              expert_out=_t(12 * 512, torch.float16)), "vectors of out"),
    ("more than 2^31 - 1 vectors of expert_out", dict(nranks=1, expert_out=torch.empty(2 ** 26 * 512, dtype=torch.float16, device="meta"),
                                                      out=torch.empty(5, 512, dtype=torch.bfloat16), block=512), "vectors of expert_out"),
])
def test_expert_size_limits_name_their_rule(what, kw, rule):
    with pytest.raises(ValueError, match=rule):
        coll.check_expert_combine_quantized(**_e(**kw))


def test_comm_methods_check_before_calling_the_library():
    """A stand-in communicator with no library handle: the methods must raise ValueError before they reach a C call."""
    class _Comm(coll.Comm):
        def __init__(self):
            self.nranks, self._h = 2, None
    c = _Comm()
    eo, route, out = _t(8 * 128, torch.bfloat16), torch.zeros(4, 2, dtype=torch.int32), torch.empty(4, 128)
    with pytest.raises(ValueError):
        c.expert_combine_quantized(eo, route, None, out, block=256)                          # 128-element rows are not whole blocks
    with pytest.raises(ValueError):
        c.expert_combine_quantized(eo, route, None, out, wire=torch.bfloat16)
    with pytest.raises(ValueError):
        c.expert_combine_quantized(eo.view(torch.int16), route, None, out)
    with pytest.raises(ValueError):
        c.all_to_all_v_combine_quantized(eo, out.view(-1), 128, [4, 4], [0, 4], [0, 0], route, block=48)
    with pytest.raises(ValueError):
        c.all_to_all_v_combine_quantized(eo, out.view(-1), 128, [4, 4], [0, 2], [0, 0], route)   # send ranges overlap


# ------------------------------------------------------------------------------------------------- kernels


def test_every_wire_out_and_map_is_instantiated_once(coll_lib):
    ks = kernels(coll_lib, "b200coll::k_fp8_combine_")
    for fam in FAMILIES:
        have = [template_args(k) for k in ks if f"::{fam}<" in k]
        assert sorted(have) == sorted((w, o, m) for w in WIRES for o in WIDE for m in MAPS), (fam, have)
    assert len(ks) == 24, ks
    assert not any(f in k for k in ks for f in FOREIGN), ks
    # the quantise pass is the dispatch's local quantising copy, with its instantiations unchanged
    copies = kernels(coll_lib, "b200coll::k_a2av_quant_copy<")
    assert sorted(template_args(k) for k in copies) == sorted((i, w) for i in WIDE for w in WIRES), copies


def test_sass_unpacks_fp8_and_never_fuses_multiply_and_add(coll_lib):
    funcs = {k: v for k, v in sass(coll_lib).items() if "k_fp8_combine_" in k}
    assert len(funcs) == 24, sorted(funcs)
    for name, body in funcs.items():
        assert not any(f in name for f in FOREIGN), name
        wire = "E4M3" if "e4m3" in name else "E5M2"
        assert f"F2FP.F16.{wire}.UNPACK_B" in body, name                 # the hardware FP8 unpack
        assert re.search(r"\bFMUL\b", body) and re.search(r"\bFADD\b", body), name
        assert "FFMA" not in body, name
        assert "LDGMC" not in body, name
        assert len(re.findall(r"\bLDG\.E\.NA\.128", body)) >= 8, name        # eight slots' FP8 vectors in flight


def test_ptxas_reports_no_stack_no_spills_and_at_most_128_registers():
    """The compiler's own account, with the library's flags: the new kernels have no stack frame and no spill stores or loads, and keep
    combine.cu's 128-register rule for every kernel with combine_ in its name; the 36 wide combine kernels are still there."""
    report, regs = ptxas("combine.cu")
    mine = {k: v for k, v in report.items() if "k_fp8_combine_" in k}
    assert len(mine) == 24, sorted(mine)
    assert all(v == (0, 0, 0) for v in mine.values()), mine
    assert all(r <= 128 for k, r in regs.items() if "combine_" in k), regs
    assert len([k for k in report if "k_combine_" in k]) == 36


def _perf_bin():
    perf = os.path.join(ROOT, "build", "b200coll_perf")
    if not os.path.exists(perf):
        subprocess.run(["make", "-C", os.path.join(ROOT, "coll"), "../build/b200coll_perf"], check=True, capture_output=True)
    return perf


def test_perf_tool_documents_the_quantising_combine(coll_lib):
    out = subprocess.run([_perf_bin(), "--help"], capture_output=True, text=True, check=True).stdout
    assert "--combine-quantize WIRE:BLOCK" in out and "quantising combine" in out


@pytest.mark.parametrize("extra", [
    ["--combine", "4", "--quantize", "e4m3:128"],
    ["--route", "16:4", "--quantize", "e4m3:128"],
    ["--combine", "4", "--block-scale", "1x128"],
    ["--route", "16:4"] + ["--block-scale", "1x128"],
    [],                                                                   # neither --combine nor --route
    ["--combine", "4", "--row-len", "192"],                              # not whole 128-element blocks
])
def test_perf_tool_refuses_the_mode_with_other_fp8_modes(coll_lib, extra):
    r = subprocess.run([_perf_bin(), "--op", "alltoall", "--combine-quantize", "e4m3:128", *extra], capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and "--combine-quantize WIRE:BLOCK takes" in r.stderr, (r.returncode, r.stdout, r.stderr)


@pytest.mark.parametrize("bad", ["e4m3", "e4m3:24", "bf16:128", "e5m2:1024"])
def test_perf_tool_refuses_a_bad_wire_or_block(coll_lib, bad):
    r = subprocess.run([_perf_bin(), "--op", "alltoall", "--combine", "4", "--combine-quantize", bad], capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and "WIRE e4m3 or e5m2" in r.stderr, (r.returncode, r.stderr)
