"""FP8 (e4m3 / e5m2) in libb200coll, checked without a GPU: the public enums and sizes, the SASS of the fused unpack, the absence of
NVLS-reduce instantiations for FP8 inputs, and the process group's routing of FP8 reductions to the library instead of Gloo."""
import ctypes as C
import os
import re
import subprocess

import pytest
import torch
import torch.distributed as dist

from container_engine_accelerators_b200.ops import coll
from container_engine_accelerators_b200.parallel import process_group as pgmod

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib(coll_lib):
    return coll.load()


def test_header_enums_and_type_sizes(tmp_path, lib):
    src = tmp_path / "probe.c"
    src.write_text(r'''
#include <stdio.h>
#include "b200coll.h"
int main(void) {
  printf("%d %d %d %zu %zu\n", b200collFloat8e4m3, b200collFloat8e5m2, b200collNumTypes, b200collTypeSize(b200collFloat8e4m3), b200collTypeSize(b200collFloat8e5m2));
  return 0;
}''')
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "coll", "include"), str(src), "-o", str(exe),
                    "-L", os.path.dirname(coll.lib_path()), "-lb200coll", "-Wl,-rpath," + os.path.dirname(coll.lib_path())], check=True)
    out = list(map(int, subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()))
    assert out == [coll.FP8_E4M3, coll.FP8_E5M2, 12, 1, 1]
    assert coll.FP8_E5M2 == 11 and coll.DTYPE_SIZE[coll.FP8_E5M2] == 1 and coll.DTYPE_SIZE[coll.FP8_E4M3] == 1
    assert lib.b200collTypeSize(coll.FP8_E5M2) == 1 and lib.b200collTypeSize(coll.FP8_E4M3) == 1
    assert coll.torch_dtype_code(torch.float8_e5m2) == coll.FP8_E5M2 and coll.torch_dtype_code(torch.float8_e4m3fn) == coll.FP8_E4M3


def test_sass_uses_the_hardware_fp8_unpack(coll_lib):
    sass = subprocess.run(["cuobjdump", "-sass", coll_lib], capture_output=True, text=True, check=True).stdout
    assert "F2FP.F16.E4M3.UNPACK_B" in sass
    assert "F2FP.F16.E5M2.UNPACK_B" in sass


def _kernels(coll_lib):
    names = subprocess.run(["nm", "-C", coll_lib], capture_output=True, text=True, check=True).stdout
    return [l.split(" ", 2)[-1] for l in names.splitlines() if "b200coll::k_" in l]


def test_no_nvls_reduction_is_instantiated_for_fp8_inputs(coll_lib):
    ks = _kernels(coll_lib)
    fp8 = ("__nv_fp8_e4m3", "__nv_fp8_e5m2")
    first_arg = lambda k: k.split("<", 1)[1].split(",", 1)[0].strip()
    nvls_ar = [k for k in ks if "k_ar_nvls<" in k]
    pull_mc = [k for k in ks if re.search(r"k_pull_reduce<[^>]*, (true|false), true>", k)]
    root_mc = [k for k in ks if re.search(r"k_reduce_root<[^>]*, true>", k)]
    assert nvls_ar and pull_mc and root_mc                     # the 16- and 32-bit NVLS reductions are still there
    for k in nvls_ar + pull_mc + root_mc:
        assert first_arg(k) not in fp8, k
    # while the P2P families, the data-movement kernels and the generic kernel do have FP8 inputs
    for fam in ("k_ll<", "k_ll_twoshot<", "k_ar_twoshot<", "k_pull_reduce<", "k_reduce_root<", "k_ag_push<", "k_bcast<", "k_a2av_push<", "k_copy_scale<", "k_generic_reduce<"):
        for t in fp8:
            assert any(fam in k and first_arg(k) == t for k in ks), (fam, t)


def test_fp8_to_f32_is_not_instantiated(coll_lib):
    for k in _kernels(coll_lib):
        m = re.search(r"k_(?:copy_scale|ll|pull_reduce|ar_twoshot|ag_push|a2av_push|bcast|reduce_root)<([^,]+), ([^,>]+)", k)
        if m and m.group(1).strip() in ("__nv_fp8_e4m3", "__nv_fp8_e5m2"):
            assert m.group(2).strip() != "float", k


def test_nccl_shim_knows_both_fp8_types():
    src = open(os.path.join(ROOT, "coll", "src", "nccl_shim.cc")).read()
    assert "ncclFloat8e4m3 = 10" in src and "ncclFloat8e5m2 = 11" in src
    body = src[src.index("bool map_dt(ncclDataType_t"):src.index("bool map_dt_reduce")]
    assert "Float8" not in body                                 # FP8 data movement never goes to the Lamport path


# ------------------------------------------------------------------------------------------------- process group routing (no GPU)
class _DeviceLike(torch.Tensor):
    """A CPU tensor that answers is_cuda=True, so the process group takes its CUDA branch while the test stays on CPU."""
    is_cuda = property(lambda self: True)

    @staticmethod
    def of(t):
        return torch.Tensor._make_subclass(_DeviceLike, t)


def _stub_pg(monkeypatch):
    class _Stream:
        def wait_event(self, e): pass
    class _Event:
        def record(self, s): pass
    stream = _Stream()
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: stream)
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    log = []

    class _Comm:
        nranks = 2
        _algo = "auto"
        def set_algo(self, name): log.append(("algo", name)); self._algo = name
        def bit_exact(self): return pgmod.coll.Comm._BitExact(self)
        def all_reduce(self, t, op=coll.SUM): log.append(("all_reduce", t.dtype, op))
        def reduce(self, t, root=0, op=coll.SUM): log.append(("reduce", t.dtype, op))
        def reduce_scatter(self, src, dst, op=coll.SUM): log.append(("reduce_scatter", src.dtype, dst.dtype, op))
        def all_gather(self, src, dst): log.append(("all_gather", src.dtype, src.numel(), dst.numel()))

    pg = pgmod.B200CollProcessGroup(store=None, rank=0, size=2)
    pg._comm = _Comm()
    pg._via_gloo = lambda *a, **k: pytest.fail("an FP8 collective fell back to Gloo")
    return pg, log


@pytest.mark.parametrize("dtype", [torch.float8_e4m3fn, torch.float8_e5m2])
def test_fp8_reductions_reach_the_library_not_gloo(monkeypatch, dtype):
    pg, log = _stub_pg(monkeypatch)
    t = _DeviceLike.of(torch.zeros(64, dtype=torch.uint8).view(dtype))
    ours = {dist.ReduceOp.SUM: coll.SUM, dist.ReduceOp.AVG: coll.AVG, dist.ReduceOp.MIN: coll.MIN, dist.ReduceOp.MAX: coll.MAX, dist.ReduceOp.PRODUCT: coll.PROD}
    for theirs, op in ours.items():
        o = dist.AllreduceOptions(); o.reduceOp = theirs
        pg.allreduce([t], o)
        assert log[-1] == ("all_reduce", dtype, op)
    assert pg.fast_calls == 5 and pg.fallback_calls == 0
    for theirs, op in ((dist.ReduceOp.SUM, coll.SUM), (dist.ReduceOp.AVG, coll.AVG)):
        o = dist.ReduceScatterOptions(); o.reduceOp = theirs
        pg._reduce_scatter_base(_DeviceLike.of(torch.zeros(32, dtype=torch.uint8).view(dtype)), _DeviceLike.of(torch.zeros(64, dtype=torch.uint8).view(dtype)), o)
        assert log[-1] == ("reduce_scatter", dtype, dtype, op)
    ro = dist.ReduceOptions(); ro.reduceOp = dist.ReduceOp.MAX; ro.rootRank = 1
    pg.reduce([t], ro)
    assert log[-1] == ("reduce", dtype, coll.MAX)
    assert pg.fast_calls == 8 and pg.fallback_calls == 0


def test_fp8_all_gather_stays_on_the_bit_exact_word_path(monkeypatch):
    pg, log = _stub_pg(monkeypatch)
    src = _DeviceLike.of(torch.zeros(64, dtype=torch.uint8).view(torch.float8_e4m3fn))
    out = _DeviceLike.of(torch.zeros(128, dtype=torch.uint8).view(torch.float8_e4m3fn))
    pg._allgather_base(out, src)
    assert log == [("algo", "twoshot"), ("all_gather", torch.float32, 16, 32), ("algo", "auto")]
    assert pg.fast_calls == 1 and pg.fallback_calls == 0
