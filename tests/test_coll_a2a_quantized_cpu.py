"""Quantising all-to-all-v in libb200coll, checked without a GPU: the C prototype against the ctypes argtypes, the Python argument checks,
the kernel instantiations and their SASS (amax across lanes, saturating FP8 pack, no multimem loads, no spills), and the perf tool's mode."""
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
FAMILIES = ("k_a2av_quant_push", "k_a2av_quant_copy")


def test_header_prototype_matches_the_ctypes_argtypes(tmp_path, coll_lib):
    src = tmp_path / "probe.c"
    src.write_text(r'''
#include <stdio.h>
#include "b200coll.h"
int main(void) {
  b200collResult_t (*a2a)(const void*, void*, float*, size_t, size_t, const int64_t*, const int64_t*, const int64_t*, b200collDataType_t,
                          b200collDataType_t, int, b200collComm_t, b200collStream_t) = b200collAllToAllvQuantized;
  printf("%d %zu\n", a2a != 0, sizeof(b200collDataType_t));
  return 0;
}''')
    exe = tmp_path / "probe"
    libdir = os.path.dirname(coll_lib)
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "coll", "include"), str(src), "-o", str(exe),
                    "-L", libdir, "-lb200coll", "-Wl,-rpath," + libdir], check=True)
    linked, enum_size = map(int, subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split())
    assert linked == 1 and enum_size == C.sizeof(C.c_int)
    L = coll.load()
    vp, sz, ci, i64 = C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_int64)
    assert L.b200collAllToAllvQuantized.argtypes == [vp, vp, C.POINTER(C.c_float), sz, sz, i64, i64, i64, ci, ci, ci, vp, vp]


# ------------------------------------------------------------------------------------------------- Python argument checks
def _t(n, dt):
    return torch.empty(n, dtype=dt)


def _args(**kw):
    """A valid call for 3 ranks, 64-element rows, block 32: src holds 10 rows, out 8 rows; keyword arguments override."""
    a = dict(nranks=3, src=_t(640, torch.bfloat16), out=_t(512, E4), out_scales=_t(16, torch.float32), row_elems=64, block=32,
             send_rows=[2, 0, 3], send_row_off=[0, 2, 7], recv_row_off_at_peer=[6, 0, 3])
    a.update(kw)
    return a


def test_check_accepts_the_documented_shapes():
    assert coll.check_all_to_all_v_quantized(**_args()) == (coll.BF16, coll.FP8_E4M3)
    assert coll.check_all_to_all_v_quantized(**_args(src=_t(640, torch.float32), out=_t(512, E5))) == (coll.F32, coll.FP8_E5M2)
    # fp16 rows of 512 elements in one 512-element block each; numpy integers are accepted, ranges may end exactly at the last row
    import numpy as np
    assert coll.check_all_to_all_v_quantized(2, _t(512 * 4, torch.float16), _t(512 * 3, E4), _t(3, torch.float32), 512, 512,
                                             np.array([1, 2]), np.array([0, 2]), np.array([2, 0])) == (coll.F16, coll.FP8_E4M3)
    # nothing sent at all
    assert coll.check_all_to_all_v_quantized(**_args(send_rows=[0, 0, 0])) == (coll.BF16, coll.FP8_E4M3)


_base = torch.empty(4096, dtype=torch.float32)


@pytest.mark.parametrize("what, kw", [
    ("FP8 src", dict(src=_t(640, E4))),
    ("int src", dict(src=_t(640, torch.int32))),
    ("bf16 out", dict(out=_t(512, torch.bfloat16))),
    ("fp16 scales", dict(out_scales=_t(16, torch.float16))),
    ("non-contiguous src", dict(src=_t(1280, torch.bfloat16)[::2])),
    ("non-contiguous out", dict(out=_t(1024, torch.uint8)[::2].view(E4))),
    ("block 24", dict(block=24, row_elems=48)),
    ("block 1024", dict(block=1024, row_elems=1024)),
    ("block True", dict(block=True)),
    ("row_elems % block", dict(row_elems=48)),
    ("row_elems 0", dict(row_elems=0)),
    ("out.numel() % row_elems", dict(out=_t(500, E4), out_scales=_t(15, torch.float32))),
    ("scales too few", dict(out_scales=_t(15, torch.float32))),
    ("scales too many", dict(out_scales=_t(17, torch.float32))),
    ("destination past out", dict(recv_row_off_at_peer=[7, 0, 3])),
    ("destination offset past out, no rows", dict(send_rows=[0, 0, 3], recv_row_off_at_peer=[9, 0, 3])),
    ("send range past src", dict(send_row_off=[0, 2, 8])),
    ("send_rows too short", dict(send_rows=[2, 0])),
    ("send_row_off too long", dict(send_row_off=[0, 2, 7, 9])),
    ("recv_row_off_at_peer too short", dict(recv_row_off_at_peer=[6, 0])),
    ("negative rows", dict(send_rows=[2, -1, 3])),
    ("negative send offset", dict(send_row_off=[0, -2, 7])),
    ("negative destination", dict(recv_row_off_at_peer=[6, 0, -3])),
    ("float entry", dict(send_rows=[2, 0.0, 3])),
    ("src overlaps out", dict(src=_base[:320].view(torch.bfloat16), out=_base[64:192].view(E4))),
    ("src overlaps out_scales", dict(src=_base[:320].view(torch.bfloat16), out_scales=_base[100:116])),
])
def test_check_raises_value_error(what, kw):
    with pytest.raises(ValueError):
        coll.check_all_to_all_v_quantized(**_args(**kw))


def test_comm_method_checks_before_calling_the_library():
    """A stand-in communicator with no library handle: the method must raise ValueError before it reaches a C call."""
    class _Comm(coll.Comm):
        def __init__(self):
            self.nranks, self._h = 2, None
    c = _Comm()
    src, out, sc = _t(256, torch.bfloat16), _t(256, E4), _t(2, torch.float32)
    with pytest.raises(ValueError):
        c.all_to_all_v_quantized(src, out, sc, 128, [1, 1], [0, 1], [0, 2])                      # destination past out
    with pytest.raises(ValueError):
        c.all_to_all_v_quantized(src, out, sc, 128, [1, 1, 0], [0, 1, 0], [0, 1, 0])             # three entries for two ranks
    with pytest.raises(ValueError):
        c.all_to_all_v_quantized(src, out.view(torch.uint8), sc, 128, [1, 1], [0, 1], [0, 1])    # out is not FP8
    with pytest.raises(ValueError):
        c.all_to_all_v_quantized(src, out, sc, 96, [1, 1], [0, 1], [0, 1], block=32)             # out.numel() % row_elems
    with pytest.raises(ValueError):
        c.all_to_all_v_quantized(src, out, sc, 128, [1, 1], [0, 1], [0, 1], block=64)            # out_scales holds 4 floats at block 64


# ------------------------------------------------------------------------------------------------- kernels


def test_every_input_and_wire_pair_is_instantiated_once(coll_lib):
    ks = kernels(coll_lib, "b200coll::k_a2av_quant_")
    for fam in FAMILIES:
        have = [template_args(k) for k in ks if f"::{fam}<" in k]
        assert sorted(have) == sorted((i, w) for i in WIDE for w in WIRES), (fam, have)
    assert len(ks) == 12, ks
    # outside the name patterns other tests count or filter on
    assert not any("k_quant_" in k or "k_bsq_" in k or "k_a2av_push<" in k for k in ks)


def test_sass_reduces_amax_across_lanes_and_packs_saturating(coll_lib):
    funcs = {k: v for k, v in sass(coll_lib).items() if "k_a2av_quant_" in k}
    assert len(funcs) == 12, sorted(funcs)
    for name, body in funcs.items():
        wire = "E4M3" if "e4m3" in name else "E5M2"                      # the input type is never FP8, so the name's FP8 type is the wire's
        assert re.search(r"\b(REDUX|SHFL\.BFLY)\b", body), name         # the block's amax, across its lanes
        assert f"F2FP.SATFINITE.{wire}" in body, name                    # cvt.rn.satfinite pack
        assert "LDGMC" not in body, name


def test_ptxas_reports_no_stack_and_no_spills():
    """The compiler's own account, with the library's flags: no stack frame and no spill stores or loads for the new kernels."""
    report = {k: v for k, v in ptxas("dispatch.cu")[0].items() if "k_a2av_quant_" in k}
    assert len(report) == 12, sorted(report)
    assert all(v == (0, 0, 0) for v in report.values()), report


def test_perf_tool_documents_the_alltoall_mode(coll_lib):
    perf = os.path.join(ROOT, "build", "b200coll_perf")
    if not os.path.exists(perf):
        subprocess.run(["make", "-C", os.path.join(ROOT, "coll"), "../build/b200coll_perf"], check=True, capture_output=True)
    out = subprocess.run([perf, "--help"], capture_output=True, text=True, check=True).stdout
    assert "--quantize WIRE:BLOCK" in out and "--op alltoall" in out and "all-to-all-v" in out
