"""Block-scaled FP8 collectives in libb200coll, checked without a GPU: the public struct and symbols as a C compiler sees them and as the
ctypes mirror lays them out, the kernel instantiations and their SASS (hardware FP8 unpack, no multimem, no spills), and the Python
shape and dtype checks."""
import ctypes as C
import os
import re
import subprocess

import pytest
import torch

from container_engine_accelerators_b200.ops import coll
from tests.coll_binary_facts import kernels, ptxas, sass, template_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP8 = ("__nv_fp8_e4m3", "__nv_fp8_e5m2")
OUTS = ("__nv_bfloat16", "__half", "float")


def test_header_struct_layout_and_symbols(tmp_path, coll_lib):
    src = tmp_path / "probe.c"
    src.write_text(r'''
#include <stddef.h>
#include <stdio.h>
#include "b200coll.h"
int main(void) {
  b200collResult_t (*ag)(const void*, void*, size_t, const b200collBlockScale*, const b200collEpilogue*, b200collComm_t, b200collStream_t) = b200collAllGatherBlockScaled;
  b200collResult_t (*rs)(const void*, void*, size_t, const b200collBlockScale*, const b200collEpilogue*, b200collRedOp_t, b200collComm_t, b200collStream_t) = b200collReduceScatterBlockScaled;
  b200collResult_t (*ar)(const void*, void*, size_t, const b200collBlockScale*, const b200collEpilogue*, b200collRedOp_t, b200collComm_t, b200collStream_t) = b200collAllReduceBlockScaled;
  printf("%zu %zu %zu %zu %zu %d\n", sizeof(b200collBlockScale), offsetof(b200collBlockScale, scales), offsetof(b200collBlockScale, row_len),
         offsetof(b200collBlockScale, block_rows), offsetof(b200collBlockScale, block_cols), ag != 0 && rs != 0 && ar != 0);
  return 0;
}''')
    exe = tmp_path / "probe"
    libdir = os.path.dirname(coll_lib)
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "coll", "include"), str(src), "-o", str(exe),
                    "-L", libdir, "-lb200coll", "-Wl,-rpath," + libdir], check=True)
    size, o_sc, o_rl, o_br, o_bc, linked = map(int, subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split())
    assert linked == 1
    m = coll.BlockScale
    assert (size, o_sc, o_rl, o_br, o_bc) == (C.sizeof(m), m.scales.offset, m.row_len.offset, m.block_rows.offset, m.block_cols.offset)
    L = coll.load()
    for name in ("b200collAllGatherBlockScaled", "b200collReduceScatterBlockScaled", "b200collAllReduceBlockScaled"):
        assert getattr(L, name).argtypes[3] is C.POINTER(coll.BlockScale)


def test_every_fp8_input_and_output_pair_is_instantiated(coll_lib):
    ks = kernels(coll_lib, "b200coll::k_bsq_")
    for fam, extra in (("k_bsq_ag_pull<", [[]]), ("k_bsq_pull_reduce<", [["false"], ["true"]]), ("k_bsq_copy<", [[]])):
        have = {template_args(k) for k in ks if fam in k}
        want = {(i, o, *e) for i in FP8 for o in OUTS for e in extra}
        assert want <= have, (fam, sorted(want - have))
    # FP8 -> fp32 exists only in the k_bsq_ family: the existing families' instantiation rules are unchanged
    assert all(re.search(r"k_bsq_[a-z_]+<", k) for k in ks)


def test_sass_unpacks_in_hardware_uses_no_multimem_and_no_64bit_division(coll_lib):
    funcs = {k: v for k, v in sass(coll_lib).items() if "k_bsq_" in k}
    assert len(funcs) >= 24, sorted(funcs)
    for name, body in funcs.items():
        unpack = "F2FP.F16.E4M3.UNPACK_B" if "e4m3" in name else "F2FP.F16.E5M2.UNPACK_B"
        assert unpack in body, name
        assert "LDGMC" not in body, name                          # no multimem.ld_reduce (sm_90a has none for FP8)
        assert "MATCH.ANY" in body, name                          # scales are shared between the lanes that need the same one
        assert "IMAD.HI" in body, name                            # row / block from multiply-high division
        assert "FFMA" not in body, name                           # float(q) * s and the sum round separately
        for call in re.findall(r"CALL\.[A-Z.]+\s+(\S+)", body):  # the only calls are the watchdog's fault recorder
            assert "div" not in call.lower(), (name, call)


def test_source_moves_data_without_multimem():
    """The data path is plain loads and stores over NVLink; the only multicast operation is the shared epoch barrier's counter."""
    quant = open(os.path.join(ROOT, "coll", "src", "quant.cuh")).read()            # the quantise helpers blockscaled.cu includes
    src = open(os.path.join(ROOT, "coll", "src", "blockscaled.cu")).read() + quant
    device = src.split("// ---", 1)[0].split("#include", 1)[1] + quant
    for loop in ("warp_walk", "dequant_range", "pull_reduce_range", "quant_range", "k_bsq_pull_reduce", "k_quant_pull_reduce"):
        assert f" {loop}(" in device, loop                        # the device section the check covers holds every loop
    assert "multimem" not in device
    for helper in ("mc_ld_reduce", "mc_st_words", "c.mc"):
        assert helper not in src, helper


def test_no_spills_in_block_scaled_kernels(coll_lib):
    """cuobjdump reports spill slots as stack frame (STACK:), local arrays as LOCAL:; every k_bsq_ kernel of the built library has neither."""
    out = subprocess.run(["cuobjdump", "-res-usage", coll_lib], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    seen = 0
    for i, line in enumerate(lines):
        if "Function" in line and "k_bsq_" in line:
            usage = lines[i + 1]
            assert re.search(r"STACK:0\b", usage) and re.search(r"LOCAL:0\b", usage), (line, usage)
            seen += 1
    assert seen >= 24


def test_ptxas_reports_no_spill_bytes():
    """The compiler's own account, with the library's flags: 0 bytes spill stores and loads for every k_bsq_ kernel."""
    report = {k: v for k, v in ptxas("blockscaled.cu")[0].items() if "k_bsq_" in k}
    assert len(report) == 24, sorted(report)
    spilled = {k: v for k, v in report.items() if v != (0, 0, 0)}
    assert not spilled, spilled


def _t(shape, dtype):
    return torch.empty(shape, dtype=dtype)


E4, E5 = torch.float8_e4m3fn, torch.float8_e5m2


def test_python_shape_checks_accept_the_documented_shapes():
    q = _t((48, 400), E4)
    assert coll.check_block_scaled("all_gather", 4, q, _t((48, 4), torch.float32), _t((192, 400), torch.bfloat16)) == (1, 128)
    assert coll.check_block_scaled("reduce_scatter", 4, _t((264, 320), E5), _t((3, 3), torch.float32), _t((66, 320), torch.float32),
                                   block=(128, 128)) == (128, 128)
    assert coll.check_block_scaled("all_reduce", 3, _t((120, 208), E5), _t((4, 4), torch.float32), _t((120, 208), torch.float16),
                                   block=(32, 64)) == (32, 64)


@pytest.mark.parametrize("what, args", [
    ("scales shape", ("all_gather", 2, _t((48, 256), E4), _t((48, 1), torch.float32), _t((96, 256), torch.bfloat16), (1, 128))),
    ("scales dtype", ("all_gather", 2, _t((48, 256), E4), _t((48, 2), torch.float16), _t((96, 256), torch.bfloat16), (1, 128))),
    ("block_cols % 16", ("all_reduce", 2, _t((48, 256), E4), _t((48, 11), torch.float32), _t((48, 256), torch.bfloat16), (1, 24))),
    ("block_cols 0", ("all_reduce", 2, _t((48, 256), E4), _t((48, 1), torch.float32), _t((48, 256), torch.bfloat16), (1, 0))),
    ("block_rows 0", ("all_reduce", 2, _t((48, 256), E4), _t((48, 2), torch.float32), _t((48, 256), torch.bfloat16), (0, 128))),
    ("row_len % 16", ("all_reduce", 2, _t((48, 72), E4), _t((48, 1), torch.float32), _t((48, 72), torch.bfloat16), (1, 128))),
    ("rows % N", ("reduce_scatter", 3, _t((16, 256), E4), _t((16, 2), torch.float32), _t((5, 256), torch.bfloat16), (1, 128))),
    ("bf16 input", ("all_reduce", 2, _t((48, 256), torch.bfloat16), _t((48, 2), torch.float32), _t((48, 256), torch.bfloat16), (1, 128))),
    ("uint8 input", ("all_gather", 2, _t((48, 256), torch.uint8), _t((48, 2), torch.float32), _t((96, 256), torch.bfloat16), (1, 128))),
    ("1-D input", ("all_reduce", 2, _t((48 * 256,), E4), _t((48, 2), torch.float32), _t((48, 256), torch.bfloat16), (1, 128))),
    ("FP8 output", ("all_reduce", 2, _t((48, 256), E4), _t((48, 2), torch.float32), _t((48, 256), E5), (1, 128))),
    ("all-gather out shape", ("all_gather", 2, _t((48, 256), E4), _t((48, 2), torch.float32), _t((48, 256), torch.bfloat16), (1, 128))),
    ("reduce-scatter out shape", ("reduce_scatter", 2, _t((48, 256), E4), _t((48, 2), torch.float32), _t((48, 256), torch.bfloat16), (1, 128))),
    ("unknown op", ("all_to_all", 2, _t((48, 256), E4), _t((48, 2), torch.float32), _t((48, 256), torch.bfloat16), (1, 128))),
])
def test_python_shape_checks_raise_value_error(what, args):
    with pytest.raises(ValueError):
        coll.check_block_scaled(*args[:5], block=args[5])


def test_comm_methods_check_before_calling_the_library():
    """The Comm methods run the same checks first: a stand-in communicator with no library handle never reaches the C call."""
    class _Comm(coll.Comm):
        def __init__(self):
            self.nranks, self._h = 2, None
    c = _Comm()
    q, s = _t((48, 256), E4), _t((48, 2), torch.float32)
    with pytest.raises(ValueError):
        c.all_gather_block_scaled(q, s, _t((48, 256), torch.bfloat16))
    with pytest.raises(ValueError):
        c.reduce_scatter_block_scaled(_t((47, 256), E4), _t((47, 2), torch.float32), _t((23, 256), torch.bfloat16))
    with pytest.raises(ValueError):
        c.all_reduce_block_scaled(q, s, _t((48, 256), torch.bfloat16), block=(1, 100))


def test_perf_tool_documents_block_scale_flags(coll_lib):
    perf = os.path.join(ROOT, "build", "b200coll_perf")
    if not os.path.exists(perf):
        subprocess.run(["make", "-C", os.path.join(ROOT, "coll"), "../build/b200coll_perf"], check=True, capture_output=True)
    out = subprocess.run([perf, "--help"], capture_output=True, text=True, check=True).stdout
    assert "--block-scale RxC" in out and "--row-len N" in out
    r = subprocess.run([perf, "--block-scale", "1x24"], capture_output=True, text=True)
    assert r.returncode != 0 and "--block-scale" in r.stderr
