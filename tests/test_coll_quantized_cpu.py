"""Quantising collectives in libb200coll, checked without a GPU: the reference quantiser against hand-worked blocks, the Python argument
checks, the ctypes prototypes against the header, the kernel instantiations and their SASS (amax reduction across lanes, saturating FP8
pack, hardware unpack, no spills), and the perf tool's flag."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from container_engine_accelerators_b200.ops import coll
from tests import coll_quant_reference as qr
from tests.coll_binary_facts import kernels, ptxas, sass, template_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E4, E5 = torch.float8_e4m3fn, torch.float8_e5m2
WIDE = ("__nv_bfloat16", "__half", "float")
WIRES = ("__nv_fp8_e4m3", "__nv_fp8_e5m2")


def _block(vals, dt=torch.float32, n=16):
    x = torch.zeros(n, dtype=dt)
    x[:len(vals)] = torch.tensor(vals, dtype=torch.float32).to(dt)
    return x


def _u8(q):
    return q.view(torch.uint8).tolist()


def _f32(x):
    return np.float32(x)


# ------------------------------------------------------------------------------------------------- the reference, by hand
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16, torch.float16])
def test_all_zero_block_has_unit_scale(dt):
    q, s, v = qr.quantize(torch.zeros(32, dtype=dt), 16, E4)
    assert _u8(q) == [0] * 32 and s.tolist() == [1.0, 1.0] and v.tolist() == [0.0] * 32


def test_negative_zero_comes_out_as_positive_zero():
    x = torch.full((16,), -0.0)
    q, s, v = qr.quantize(x, 16, E4)
    assert _u8(q) == [0x80] * 16 and s.item() == 1.0                   # q keeps the sign, v is -0
    assert torch.signbit(v).all()
    out = qr.reduce([v], 1.0, torch.bfloat16)                           # (0 + -0) is +0
    assert out.view(torch.int16).tolist() == [0] * 16


def test_amax_maps_exactly_to_fmax():
    q, s, v = qr.quantize(_block([1.0, 0.5, -0.25]), 16, E4)
    assert _u8(q)[:4] == [0x7E, 0x76, 0xEE, 0x00]                        # 448, 224, -112, 0
    assert s.item() == float(_f32(1.0) / _f32(448.0))
    assert v[0].item() == float(_f32(448.0) * (_f32(1.0) / _f32(448.0)))
    q5, s5, _ = qr.quantize(_block([2.0]), 16, E5)
    assert _u8(q5)[0] == 0x7B and s5.item() == float(_f32(2.0) / _f32(57344.0))   # 57344


def test_ties_round_to_nearest_even():
    # amax 448 gives inv = s = 1; e4m3 has three mantissa bits, so 1.0625 lies halfway between 1 and 1.125, 1.1875 between 1.125 and 1.25
    q, s, v = qr.quantize(_block([448.0, 1.0625, 1.1875, -1.0625, 0.015625 + 0.0009765625]), 16, E4)
    assert s.item() == 1.0
    assert q.float()[:5].tolist() == [448.0, 1.0, 1.25, -1.0, 0.015625]
    assert v[:5].tolist() == [448.0, 1.0, 1.25, -1.0, 0.015625]


def _amax_over_fmax(fmax):
    """The first fp32 amax >= 1 whose product amax * fl(fmax / amax) rounds above fmax."""
    a = np.arange(1 << 16, dtype=np.uint32) + np.float32(1.0).view(np.uint32)
    a = a.view(np.float32)
    y = (a * (np.float32(fmax) / a).astype(np.float32)).astype(np.float32)
    return float(a[np.argmax(y > np.float32(fmax))]), y


@pytest.mark.parametrize("wire", [E4, E5])
def test_product_just_above_fmax_saturates(wire):
    fmax = qr.FP8_MAX[wire]
    amax, y = _amax_over_fmax(fmax)
    assert (y > np.float32(fmax)).any()
    x = _block([amax, -amax, 1.0])
    inv = _f32(fmax) / _f32(amax)
    assert _f32(amax) * inv > _f32(fmax)                                 # the rounded product is past the largest finite FP8
    q, s, v = qr.quantize(x, 16, wire)
    assert q.float()[:2].tolist() == [fmax, -fmax]                      # saturated, not inf / NaN
    assert v[0].item() == float(_f32(fmax) * (_f32(amax) / _f32(fmax)))


@pytest.mark.parametrize("special", [float("inf"), float("-inf"), float("nan")])
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16, torch.float16])
def test_inf_or_nan_makes_the_whole_block_nan(special, dt):
    x = torch.cat([_block([special, 1.0, -2.0, 0.0], dt), _block([3.0, 5.0], dt)])
    q, s, v = qr.quantize(x, 16, E4)
    assert torch.isnan(v[:16]).all() and not torch.isnan(v[16:]).any()
    for out_dt in (torch.bfloat16, torch.float16, torch.float32):
        assert torch.isnan(qr.reduce([v], 1.0, out_dt).float()[:16]).all()


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16])
def test_tiny_block_takes_unit_scale(dt):
    tiny = 1e-37                                                         # below 448 / FLT_MAX: fmax / amax overflows to inf
    x = _block([tiny, -tiny / 2], dt)
    amax = _f32(x[0].float().item())
    with np.errstate(over="ignore"):
        assert np.isinf(_f32(448.0) / amax)
    q, s, v = qr.quantize(x, 16, E4)
    assert s.item() == 1.0 and v.abs().max().item() == 0.0              # x * 1 rounds to (signed) zero in e4m3


def test_generator_spans_binades_and_places_specials():
    for dt in (torch.float32, torch.bfloat16, torch.float16):
        x = qr.gen(128 * 64, dt, 128, 5)
        _, s, v = qr.quantize(x, 128, E4)
        fin = s[torch.isfinite(s) & (s != 1.0)]
        assert float(fin.max() / fin.min()) > 2 ** 20, dt
        assert torch.isnan(v[2 * 128:5 * 128]).all() and not torch.isnan(v[5 * 128:]).any()
        assert s[0].item() == 1.0


# ------------------------------------------------------------------------------------------------- Python argument checks
def _t(n, dt):
    return torch.empty(n, dtype=dt)


def test_check_quantized_accepts_the_documented_shapes():
    assert coll.check_quantized("all_gather", 4, _t(512, torch.bfloat16), _t(2048, torch.float32), 128) == coll.FP8_E4M3
    assert coll.check_quantized("reduce_scatter", 3, _t(3 * 64, torch.float32), _t(64, torch.float16), 64, E5) == coll.FP8_E5M2
    x = _t(1024, torch.float16)
    assert coll.check_quantized("all_reduce", 2, x, x, 512) == coll.FP8_E4M3                          # in place
    assert coll.check_quantized("all_reduce", 2, x, x.view(torch.bfloat16), 16) == coll.FP8_E4M3      # in place, same element size


_base = torch.empty(8192, dtype=torch.float32)


@pytest.mark.parametrize("what, args", [
    ("unknown op", ("all_to_all", 2, _t(256, torch.bfloat16), _t(256, torch.bfloat16), 128, None)),
    ("FP8 input", ("all_reduce", 2, _t(256, E4), _t(256, torch.bfloat16), 128, None)),
    ("int input", ("all_reduce", 2, _t(256, torch.int32), _t(256, torch.bfloat16), 128, None)),
    ("FP8 output", ("all_reduce", 2, _t(256, torch.bfloat16), _t(256, E5), 128, None)),
    ("bf16 wire", ("all_reduce", 2, _t(256, torch.bfloat16), _t(256, torch.bfloat16), 128, torch.bfloat16)),
    ("block 24", ("all_reduce", 2, _t(384, torch.bfloat16), _t(384, torch.bfloat16), 24, None)),
    ("block 8", ("all_reduce", 2, _t(256, torch.bfloat16), _t(256, torch.bfloat16), 8, None)),
    ("block 1024", ("all_reduce", 2, _t(2048, torch.bfloat16), _t(2048, torch.bfloat16), 1024, None)),
    ("block True", ("all_reduce", 2, _t(256, torch.bfloat16), _t(256, torch.bfloat16), True, None)),
    ("count % block", ("all_reduce", 2, _t(200, torch.bfloat16), _t(200, torch.bfloat16), 128, None)),
    ("all-gather out size", ("all_gather", 2, _t(256, torch.bfloat16), _t(256, torch.bfloat16), 128, None)),
    ("all-gather count % block", ("all_gather", 2, _t(48, torch.bfloat16), _t(96, torch.bfloat16), 32, None)),
    ("reduce-scatter numel % N", ("reduce_scatter", 3, _t(256, torch.bfloat16), _t(85, torch.bfloat16), 16, None)),
    ("reduce-scatter slice % block", ("reduce_scatter", 2, _t(256, torch.bfloat16), _t(128, torch.bfloat16), 256, None)),
    ("reduce-scatter out size", ("reduce_scatter", 2, _t(256, torch.bfloat16), _t(256, torch.bfloat16), 128, None)),
    ("all-reduce out size", ("all_reduce", 2, _t(256, torch.bfloat16), _t(512, torch.bfloat16), 128, None)),
    ("non-contiguous src", ("all_reduce", 2, _t(512, torch.bfloat16)[::2], _t(256, torch.bfloat16), 128, None)),
    ("all-gather overlap", ("all_gather", 2, _base[:1024], _base[512:2560], 128, None)),
    ("reduce-scatter overlap", ("reduce_scatter", 2, _base[:2048], _base[1024:2048], 128, None)),
    ("reduce-scatter in place", ("reduce_scatter", 2, _base[:2048], _base[:1024], 128, None)),
    ("all-reduce partial overlap", ("all_reduce", 2, _base[:1024], _base[128:1152], 128, None)),
    ("all-reduce in place, other size", ("all_reduce", 2, _base[:1024], _base[:1024].view(torch.bfloat16)[:1024], 128, None)),
])
def test_check_quantized_raises_value_error(what, args):
    with pytest.raises(ValueError):
        coll.check_quantized(*args)


def test_comm_methods_check_before_calling_the_library():
    """A stand-in communicator with no library handle: every method must raise ValueError before it reaches a C call."""
    class _Comm(coll.Comm):
        def __init__(self):
            self.nranks, self._h = 2, None
    c = _Comm()
    with pytest.raises(ValueError):
        c.all_gather_quantized(_t(256, torch.bfloat16), _t(256, torch.bfloat16))
    with pytest.raises(ValueError):
        c.reduce_scatter_quantized(_t(256, torch.float32), _t(128, torch.float32), block=256)
    with pytest.raises(ValueError):
        c.all_reduce_quantized(_t(256, torch.float16), wire=torch.float16)
    with pytest.raises(ValueError):
        c.all_reduce_quantized(_t(200, torch.float16))
    with pytest.raises(ValueError):
        c.all_reduce_quantized(_t(256, E4), _t(256, torch.bfloat16))


# ------------------------------------------------------------------------------------------------- C API and binding
def test_header_prototypes_match_the_ctypes_argtypes(tmp_path, coll_lib):
    src = tmp_path / "probe.c"
    src.write_text(r'''
#include <stdio.h>
#include "b200coll.h"
int main(void) {
  b200collResult_t (*ag)(const void*, void*, size_t, b200collDataType_t, int, const b200collEpilogue*, b200collComm_t, b200collStream_t) = b200collAllGatherQuantized;
  b200collResult_t (*rs)(const void*, void*, size_t, b200collDataType_t, int, const b200collEpilogue*, b200collRedOp_t, b200collComm_t, b200collStream_t) = b200collReduceScatterQuantized;
  b200collResult_t (*ar)(const void*, void*, size_t, b200collDataType_t, int, const b200collEpilogue*, b200collRedOp_t, b200collComm_t, b200collStream_t) = b200collAllReduceQuantized;
  printf("%d %zu %zu\n", ag != 0 && rs != 0 && ar != 0, sizeof(b200collDataType_t), sizeof(b200collRedOp_t));
  return 0;
}''')
    exe = tmp_path / "probe"
    libdir = os.path.dirname(coll_lib)
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "coll", "include"), str(src), "-o", str(exe),
                    "-L", libdir, "-lb200coll", "-Wl,-rpath," + libdir], check=True)
    linked, enum_size, op_size = map(int, subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split())
    assert linked == 1 and enum_size == C.sizeof(C.c_int) and op_size == C.sizeof(C.c_int)
    L = coll.load()
    vp, sz, ci, ep = C.c_void_p, C.c_size_t, C.c_int, C.POINTER(coll.Epilogue)
    assert L.b200collAllGatherQuantized.argtypes == [vp, vp, sz, ci, ci, ep, vp, vp]
    assert L.b200collReduceScatterQuantized.argtypes == [vp, vp, sz, ci, ci, ep, ci, vp, vp]
    assert L.b200collAllReduceQuantized.argtypes == [vp, vp, sz, ci, ci, ep, ci, vp, vp]


def test_every_input_wire_and_output_triple_is_instantiated(coll_lib):
    ks = kernels(coll_lib, "b200coll::k_quant_")
    want = set()
    for fam, extra in (("k_quant_ag", [()]), ("k_quant_pull_reduce", [("false",), ("true",)]), ("k_quant_copy", [()])):
        have = {template_args(k) for k in ks if f"::{fam}<" in k}
        fam_want = {(i, w, o, *e) for i in WIDE for w in WIRES for o in WIDE for e in extra}
        assert have == fam_want, (fam, sorted(fam_want ^ have))
        want |= {(fam, t) for t in fam_want}
    assert len(ks) == len(want) == 72
    assert not any("k_bsq_" in k for k in ks)                          # the block-scaled family keeps its own 24 kernels


def test_sass_reduces_amax_across_lanes_packs_saturating_and_unpacks_in_hardware(coll_lib):
    funcs = {k: v for k, v in sass(coll_lib).items() if "k_quant_" in k}
    assert len(funcs) == 72, sorted(funcs)
    for name, body in funcs.items():
        wire = "E4M3" if "e4m3" in name else "E5M2"                      # the input type is never FP8, so the name's FP8 type is the wire's
        assert re.search(r"\b(REDUX|SHFL\.BFLY)\b", body), name         # the block's amax, across its lanes
        assert f"F2FP.SATFINITE.{wire}" in body, name                    # cvt.rn.satfinite pack
        assert f"F2FP.F16.{wire}.UNPACK_B" in body, name                  # hardware FP8 -> f16 unpack
        assert "LDGMC" not in body, name
        if "k_quant_copy" not in name:
            assert "MATCH.ANY" in body, name                              # pulled scales shared by the lanes that need them


def test_ptxas_reports_no_spill_bytes_in_the_shared_fp8_unit():
    """The compiler's own account, with the library's flags: no stack frame and no spill stores or loads for any k_quant_ kernel of
    blockscaled.cu, the translation unit the quantising kernels share with the block-scaled ones."""
    report = {k: v for k, v in ptxas("blockscaled.cu")[0].items() if "k_quant_" in k}
    assert len(report) == 72, sorted(report)
    spilled = {k: v for k, v in report.items() if v != (0, 0, 0)}
    assert not spilled, spilled


def test_perf_tool_documents_quantize(coll_lib):
    perf = os.path.join(ROOT, "build", "b200coll_perf")
    if not os.path.exists(perf):
        subprocess.run(["make", "-C", os.path.join(ROOT, "coll"), "../build/b200coll_perf"], check=True, capture_output=True)
    out = subprocess.run([perf, "--help"], capture_output=True, text=True, check=True).stdout
    assert "--quantize WIRE:BLOCK" in out
    for bad in ("e4m3:24", "bf16:128", "e5m2:1024", "e4m3"):
        r = subprocess.run([perf, "--quantize", bad], capture_output=True, text=True)
        assert r.returncode != 0 and "--quantize" in r.stderr, bad
