"""Device-routed FP8 expert dispatch in libb200coll, checked without a GPU: the C prototype against the ctypes argtypes, the Python
argument checks, the push kernel's instantiations, its SASS (amax across lanes, saturating FP8 pack, no multimem loads) and ptxas's stack
and spill report, and the perf tool's mode."""
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
# name patterns other test files count or filter kernels by
FOREIGN = ("k_routed_", "k_quant_", "k_a2av_quant_", "k_bsq_", "combine_")


def test_header_prototype_matches_the_ctypes_argtypes(tmp_path, coll_lib):
    src = tmp_path / "probe.c"
    src.write_text(r'''
#include <stdio.h>
#include "b200coll.h"
int main(void) {
  b200collResult_t (*d)(const void*, void*, float*, size_t, size_t, const int32_t*, size_t, int, int, int32_t*, int32_t*, int32_t*,
                        b200collDataType_t, b200collDataType_t, int, b200collComm_t, b200collStream_t) = b200collExpertDispatchQuantized;
  printf("%d\n", d != 0);
  return 0;
}''')
    exe = tmp_path / "probe"
    libdir = os.path.dirname(coll_lib)
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "coll", "include"), str(src), "-o", str(exe),
                    "-L", libdir, "-lb200coll", "-Wl,-rpath," + libdir], check=True)
    assert subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split() == ["1"]
    L = coll.load()
    vp, sz, ci, i32 = C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_int32)
    assert L.b200collExpertDispatchQuantized.argtypes == [vp, vp, C.POINTER(C.c_float), sz, sz, i32, sz, ci, ci, i32, i32, i32, ci, ci, ci, vp, vp]


# ------------------------------------------------------------------------------------------------- Python argument checks
def _t(n, dt):
    return torch.empty(n, dtype=dt)


def _d(**kw):
    """A valid FP8 dispatch for 2 ranks: 5 tokens of 64 bf16 elements, block 32, top-3 over 8 experts, 12 recv rows; keyword arguments
    override."""
    a = dict(nranks=2, x=torch.empty(5, 64, dtype=torch.bfloat16), topk_idx=torch.zeros(5, 3, dtype=torch.int32), num_experts=8,
             recv=_t(12 * 64, E4), recv_scales=_t(12 * 2, torch.float32), block=32, expert_counts=_t(4, torch.int32),
             route=torch.empty(5, 3, dtype=torch.int32), dropped=_t(1, torch.int32))
    a.update(kw)
    return a


def test_check_accepts_the_documented_shapes():
    assert coll.check_expert_dispatch_quantized(**_d()) == (coll.BF16, coll.FP8_E4M3)
    assert coll.check_expert_dispatch_quantized(**_d(expert_counts=None, route=None, dropped=None)) == (coll.BF16, coll.FP8_E4M3)
    assert coll.check_expert_dispatch_quantized(**_d(x=torch.empty(5, 512), recv=_t(512 * 3, E5), recv_scales=_t(3, torch.float32), block=512,
                                                     num_experts=1024, expert_counts=None)) == (coll.F32, coll.FP8_E5M2)
    # no tokens at all, one rank with one expert, fp16 rows in 16-element blocks, a 2-D recv
    assert coll.check_expert_dispatch_quantized(1, torch.empty(0, 16, dtype=torch.float16), torch.zeros(0, 8, dtype=torch.int32), 1,
                                                torch.empty(3, 16, dtype=E4), _t(3, torch.float32), 16) == (coll.F16, coll.FP8_E4M3)


_base = torch.empty(4096, dtype=torch.int32)


@pytest.mark.parametrize("what, kw", [
    ("FP8 x", dict(x=torch.empty(5, 64, dtype=E4))),
    ("int32 x", dict(x=torch.empty(5, 64, dtype=torch.int32))),
    ("1-D x", dict(x=_t(320, torch.bfloat16))),
    ("non-contiguous x", dict(x=torch.empty(64, 5, dtype=torch.bfloat16).t())),
    ("block 24", dict(block=24)),
    ("block 1024", dict(block=1024)),
    ("block True", dict(block=True)),
    ("row_elems % block", dict(block=128, recv_scales=_t(6, torch.float32))),
    ("int64 topk_idx", dict(topk_idx=torch.zeros(5, 3, dtype=torch.int64))),
    ("top_k 0", dict(topk_idx=torch.zeros(5, 0, dtype=torch.int32), route=None)),
    ("topk_idx of other tokens", dict(topk_idx=torch.zeros(4, 3, dtype=torch.int32), route=None)),
    ("0 experts", dict(num_experts=0)),
    ("1025 experts", dict(num_experts=1025)),
    ("experts not a multiple of nranks", dict(num_experts=7)),
    ("bf16 recv", dict(recv=_t(12 * 64, torch.bfloat16))),
    ("uint8 recv", dict(recv=_t(12 * 64, torch.uint8))),
    ("non-contiguous recv", dict(recv=_t(24 * 64, torch.uint8)[::2].view(E4))),
    ("recv of part of a row", dict(recv=_t(12 * 64 - 32, E4), recv_scales=_t(23, torch.float32))),
    ("fp16 recv_scales", dict(recv_scales=_t(24, torch.float16))),
    ("recv_scales too few", dict(recv_scales=_t(23, torch.float32))),
    ("recv_scales too many", dict(recv_scales=_t(25, torch.float32))),
    ("expert_counts of the wrong size", dict(expert_counts=_t(8, torch.int32))),
    ("int64 route", dict(route=torch.empty(5, 3, dtype=torch.int64))),
    ("dropped of two", dict(dropped=_t(2, torch.int32))),
    ("recv overlaps x", dict(x=_base[:160].view(torch.bfloat16).view(5, 64), recv=_base[100:292].view(E4))),
    ("recv_scales overlaps x", dict(x=_base[:160].view(torch.bfloat16).view(5, 64), recv_scales=_base[150:174].view(torch.float32))),
    ("recv overlaps recv_scales", dict(recv=_base[:192].view(E4), recv_scales=_base[180:204].view(torch.float32))),
    ("route overlaps expert_counts", dict(expert_counts=_base[:4], route=_base[2:17].view(5, 3))),
    ("dropped overlaps route", dict(route=_base[:15].view(5, 3), dropped=_base[14:15])),
    ("route overlaps topk_idx", dict(topk_idx=_base[:15].view(5, 3), route=_base[10:25].view(5, 3))),
    ("expert_counts in recv", dict(recv=_base[:192].view(E4), expert_counts=_base[100:104])),
    ("dropped in recv_scales", dict(recv_scales=_base[:24].view(torch.float32), dropped=_base[20:21])),
])
def test_check_raises_value_error(what, kw):
    with pytest.raises((ValueError, RuntimeError)) as e:
        coll.check_expert_dispatch_quantized(**_d(**kw))
    assert e.type is ValueError, (what, e.value)


@pytest.mark.parametrize("what, kw, rule", [
    ("tokens * top_k > 2^31 - 1", dict(x=torch.empty(2 ** 30, 32, dtype=torch.bfloat16, device="meta"), block=32,
                                       topk_idx=torch.empty(2 ** 30, 2, dtype=torch.int32, device="meta"), route=None), "tokens \\* top_k"),
    ("nranks * recv rows > 2^31 - 1", dict(nranks=8, num_experts=8, expert_counts=_t(1, torch.int32),
                                           recv=torch.empty(2 ** 28 * 64, dtype=E4, device="meta"),
                                           recv_scales=torch.empty(2 ** 28 * 2, dtype=torch.float32, device="meta")), "nranks \\* recv rows"),
    ("more than 2^31 - 1 vectors of x", dict(x=torch.empty(2 ** 24, 2048, dtype=torch.bfloat16, device="meta"), recv=_t(2048 * 2, E4),
                                             recv_scales=_t(2 * 64, torch.float32), topk_idx=torch.empty(2 ** 24, 1, dtype=torch.int32, device="meta"),
                                             route=None), "vectors of x"),
    ("more than 2^31 - 1 vectors offered", dict(x=torch.empty(2 ** 22, 512, dtype=torch.bfloat16, device="meta"), recv=_t(512 * 2, E4),
                                                recv_scales=_t(2 * 16, torch.float32), topk_idx=torch.empty(2 ** 22, 32, dtype=torch.int32, device="meta"),
                                                route=None), "16-byte vectors may be offered"),
])
def test_check_size_limits_name_their_rule(what, kw, rule):
    """Each size limit is refused by its own rule, with every other argument valid (meta tensors: no memory behind them)."""
    with pytest.raises(ValueError, match=rule):
        coll.check_expert_dispatch_quantized(**_d(**kw))


def test_comm_method_checks_before_calling_the_library():
    """A stand-in communicator with no library handle: the method must raise ValueError before it reaches a C call or allocates."""
    class _Comm(coll.Comm):
        def __init__(self):
            self.nranks, self._h = 2, None
    c = _Comm()
    x, idx, recv, sc = torch.empty(4, 128, dtype=torch.bfloat16), torch.zeros(4, 2, dtype=torch.int32), _t(8 * 128, E4), _t(8, torch.float32)
    with pytest.raises(ValueError):
        c.expert_dispatch_quantized(x, idx, 3, recv, sc)                                     # 3 experts for 2 ranks
    with pytest.raises(ValueError):
        c.expert_dispatch_quantized(x, idx.long(), 4, recv, sc)
    with pytest.raises(ValueError):
        c.expert_dispatch_quantized(x, idx, 4, recv.view(torch.uint8), sc)                   # recv is not FP8
    with pytest.raises(ValueError):
        c.expert_dispatch_quantized(x, idx, 4, recv, sc, block=64)                           # recv_scales holds 8 floats at block 128
    with pytest.raises(ValueError):
        c.expert_dispatch_quantized(x, idx, 4, recv, sc, block=256)                          # row_elems 128 is not whole blocks


# ------------------------------------------------------------------------------------------------- kernels


def test_every_input_wire_and_placement_is_instantiated_once(coll_lib):
    ks = kernels(coll_lib, "b200coll::k_expert_quant_push<")
    assert sorted(template_args(k) for k in ks) == sorted((i, w, p) for i in WIDE for w in WIRES for p in ("false", "true")), ks
    assert len(ks) == 12
    assert not any(f in k for k in ks for f in FOREIGN), ks


def test_sass_reduces_amax_across_lanes_and_packs_saturating(coll_lib):
    funcs = {k: v for k, v in sass(coll_lib).items() if "k_expert_quant_push" in k}
    assert len(funcs) == 12, sorted(funcs)
    for name, body in funcs.items():
        assert not any(f in name for f in FOREIGN), name
        wire = "E4M3" if "e4m3" in name else "E5M2"                      # the input type is never FP8, so the name's FP8 type is the wire's
        assert re.search(r"\b(REDUX|SHFL\.BFLY)\b", body), name         # the block's amax, across its lanes
        assert f"F2FP.SATFINITE.{wire}" in body, name                    # cvt.rn.satfinite pack
        assert "LDGMC" not in body, name


def test_ptxas_reports_no_stack_and_no_spills():
    """The compiler's own account, with the library's flags: no stack frame and no spill stores or loads for the new kernels."""
    report = {k: v for k, v in ptxas("dispatch.cu")[0].items() if "k_expert_quant_push" in k}
    assert len(report) == 12, sorted(report)
    assert all(v == (0, 0, 0) for v in report.values()), report


def test_perf_tool_documents_the_routed_fp8_mode(coll_lib):
    perf = os.path.join(ROOT, "build", "b200coll_perf")
    if not os.path.exists(perf):
        subprocess.run(["make", "-C", os.path.join(ROOT, "coll"), "../build/b200coll_perf"], check=True, capture_output=True)
    out = subprocess.run([perf, "--help"], capture_output=True, text=True, check=True).stdout
    assert "--route E:K --quantize WIRE:BLOCK" in out and "device-routed FP8 expert dispatch" in out
