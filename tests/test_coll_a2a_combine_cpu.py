"""Expert combine in libb200coll, checked without a GPU: the C prototype against the ctypes argtypes, the Python argument checks, the
kernel instantiations and their SASS (no FFMA, no multimem loads), ptxas's stack and spill report, the perf tool's mode, the dispatch
plan's index and weights, and the slot order of the reference the GPU tests use."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from container_engine_accelerators_b200.ops import coll
from tests import coll_combine_reference as cr
from tests.coll_binary_facts import kernels, ptxas, sass, template_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIDE = ("__nv_bfloat16", "__half", "float")
FAMILIES = ("k_combine_pull", "k_combine_local")


def test_header_prototype_matches_the_ctypes_argtypes(tmp_path, coll_lib):
    src = tmp_path / "probe.c"
    src.write_text(r'''
#include <stdio.h>
#include "b200coll.h"
int main(void) {
  b200collResult_t (*f)(const void*, void*, size_t, size_t, const int64_t*, const int64_t*, const int64_t*, const int32_t*, const float*,
                        size_t, int, const b200collEpilogue*, b200collComm_t, b200collStream_t) = b200collAllToAllvCombine;
  printf("%d\n", f != 0);
  return 0;
}''')
    exe = tmp_path / "probe"
    libdir = os.path.dirname(coll_lib)
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "coll", "include"), str(src), "-o", str(exe),
                    "-L", libdir, "-lb200coll", "-Wl,-rpath," + libdir], check=True)
    assert subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split() == ["1"]
    L = coll.load()
    vp, sz, ci, i64 = C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_int64)
    assert L.b200collAllToAllvCombine.argtypes == [vp, vp, sz, sz, i64, i64, i64, C.POINTER(C.c_int32), C.POINTER(C.c_float), sz, ci,
                                                   C.POINTER(coll.Epilogue), vp, vp]


# ------------------------------------------------------------------------------------------------- Python argument checks
def _t(n, dt):
    return torch.empty(n, dtype=dt)


def _args(**kw):
    """A valid call for 3 ranks, 32-element rows: expert_out holds 10 rows, 4 tokens of top_k 2; keyword arguments override."""
    a = dict(nranks=3, expert_out=_t(320, torch.bfloat16), out=_t(128, torch.bfloat16), row_elems=32, send_rows=[2, 0, 3],
             send_row_off=[0, 9, 4], recv_row_off_at_peer=[6, 0, 3], index=torch.zeros(4, 2, dtype=torch.int32),
             weights=torch.ones(4, 2))
    a.update(kw)
    return a


def test_check_accepts_the_documented_shapes():
    assert coll.check_all_to_all_v_combine(**_args()) == (coll.BF16, coll.BF16)
    assert coll.check_all_to_all_v_combine(**_args(expert_out=_t(320, torch.float32), out=_t(128, torch.float16), weights=None)) == (coll.F32, coll.F16)
    # numpy integers, ranges that touch, a destination range ending at the last row, no tokens at all
    assert coll.check_all_to_all_v_combine(2, _t(64, torch.float16), _t(0, torch.float32), 16, np.array([1, 3]), np.array([3, 0]),
                                           np.array([3, 0]), torch.zeros(0, 8, dtype=torch.int32), None) == (coll.F16, coll.F32)


_base = torch.empty(4096, dtype=torch.float32)


@pytest.mark.parametrize("what, kw", [
    ("FP8 expert_out", dict(expert_out=_t(320, torch.float8_e4m3fn))),
    ("FP8 out", dict(out=_t(128, torch.float8_e5m2))),
    ("int out", dict(out=_t(128, torch.int16))),
    ("non-contiguous expert_out", dict(expert_out=_t(640, torch.bfloat16)[::2])),
    ("non-contiguous out", dict(out=_t(256, torch.bfloat16)[::2])),
    ("row_elems 24", dict(row_elems=24, expert_out=_t(240, torch.bfloat16), out=_t(96, torch.bfloat16))),
    ("row_elems 0", dict(row_elems=0)),
    ("row_elems True", dict(row_elems=True)),
    ("expert_out.numel() % row_elems", dict(expert_out=_t(330, torch.bfloat16))),
    ("int64 index", dict(index=torch.zeros(4, 2, dtype=torch.int64))),
    ("1-D index", dict(index=torch.zeros(8, dtype=torch.int32))),
    ("top_k 0", dict(index=torch.zeros(4, 0, dtype=torch.int32), weights=torch.ones(4, 0), out=_t(128, torch.bfloat16))),
    ("non-contiguous index", dict(index=torch.zeros(2, 4, dtype=torch.int32).t())),
    ("fp16 weights", dict(weights=torch.ones(4, 2, dtype=torch.float16))),
    ("weights of another shape", dict(weights=torch.ones(2, 4))),
    ("out too small", dict(out=_t(96, torch.bfloat16))),
    ("out too large", dict(out=_t(160, torch.bfloat16))),
    ("destination past expert_out", dict(recv_row_off_at_peer=[9, 0, 3])),
    ("destination offset past expert_out, no rows", dict(send_rows=[0, 0, 3], recv_row_off_at_peer=[11, 0, 3])),
    ("overlapping send ranges", dict(send_row_off=[0, 9, 1])),
    ("send_rows too short", dict(send_rows=[2, 0])),
    ("send_row_off too long", dict(send_row_off=[0, 9, 4, 5])),
    ("recv_row_off_at_peer too short", dict(recv_row_off_at_peer=[6, 0])),
    ("negative rows", dict(send_rows=[2, -1, 3])),
    ("negative send offset", dict(send_row_off=[0, -2, 4])),
    ("negative destination", dict(recv_row_off_at_peer=[6, 0, -3])),
    ("float entry", dict(send_rows=[2, 0.0, 3])),
    ("out overlaps expert_out", dict(expert_out=_base[:160].view(torch.bfloat16), out=_base[100:164].view(torch.bfloat16))),
    ("out overlaps index", dict(out=_base[:64].view(torch.bfloat16), index=_base[60:68].view(torch.int32).view(4, 2))),
    ("out overlaps weights", dict(out=_base[:64].view(torch.bfloat16), weights=_base[56:64].view(4, 2))),
])
def test_check_raises_value_error(what, kw):
    with pytest.raises(ValueError):
        coll.check_all_to_all_v_combine(**_args(**kw))


def test_comm_method_checks_before_calling_the_library():
    """A stand-in communicator with no library handle: the method must raise ValueError before it reaches a C call."""
    class _Comm(coll.Comm):
        def __init__(self):
            self.nranks, self._h = 2, None
    c = _Comm()
    eo, out, idx = _t(256, torch.bfloat16), _t(64, torch.bfloat16), torch.zeros(2, 2, dtype=torch.int32)
    with pytest.raises(ValueError):
        c.all_to_all_v_combine(eo, out, 32, [4, 4], [0, 4], [0, 5], idx)                    # destination past expert_out
    with pytest.raises(ValueError):
        c.all_to_all_v_combine(eo, out, 32, [4, 4, 0], [0, 4, 0], [0, 4, 0], idx)           # three entries for two ranks
    with pytest.raises(ValueError):
        c.all_to_all_v_combine(eo, out, 32, [4, 4], [0, 2], [0, 4], idx)                    # send ranges overlap
    with pytest.raises(ValueError):
        c.all_to_all_v_combine(eo, out, 32, [4, 4], [0, 4], [0, 4], idx, weights=torch.ones(2, 3))


# ------------------------------------------------------------------------------------------------- kernels


def test_every_input_and_output_pair_is_instantiated_once(coll_lib):
    ks = [k for k in kernels(coll_lib, "b200coll::k_combine_") if "b200coll::SegmentMap>" in k]
    for fam in FAMILIES:
        have = [template_args(k) for k in ks if f"::{fam}<" in k]
        assert sorted(have) == sorted((i, o, "b200coll::SegmentMap") for i in WIDE for o in WIDE), (fam, have)
    assert len(ks) == 18, ks
    # outside the name patterns other tests count or filter on
    assert not any("k_a2av_quant_" in k or "k_quant_" in k or "k_bsq_" in k or "k_a2av_push<" in k for k in ks)


def test_sass_has_no_ffma_and_no_multimem_loads(coll_lib):
    funcs = {k: v for k, v in sass(coll_lib).items() if "k_combine_" in k and "SegmentMap" in k}
    assert len(funcs) == 18, sorted(funcs)
    for name, body in funcs.items():
        assert re.search(r"\bFMUL\b", body) and re.search(r"\bFADD\b", body), name       # the products and sums, each rounded
        assert "FFMA" not in body, name
        assert "LDGMC" not in body, name


def test_ptxas_reports_no_stack_and_no_spills():
    """The compiler's own account, with the library's flags: no stack frame and no spill stores or loads for the combine kernels."""
    report = {k: v for k, v in ptxas("combine.cu")[0].items() if "k_combine_" in k and "SegmentMap" in k}
    assert len(report) == 18, sorted(report)
    assert all(v == (0, 0, 0) for v in report.values()), report


def test_perf_tool_documents_the_combine_mode(coll_lib):
    perf = os.path.join(ROOT, "build", "b200coll_perf")
    if not os.path.exists(perf):
        subprocess.run(["make", "-C", os.path.join(ROOT, "coll"), "../build/b200coll_perf"], check=True, capture_output=True)
    out = subprocess.run([perf, "--help"], capture_output=True, text=True, check=True).stdout
    assert "--combine K" in out and "expert combine" in out and "expert_out bytes read per rank" in out


# ------------------------------------------------------------------------------------------------- dispatch plan
# (rows, send_off, recv_off, max_rows) of expert_dispatch_plan before it gained index and weights
PINNED = {
    (2, 48, 1, 4, 2, 1.2, 3): ([[33, 63], [32, 64]],
          [[0, 33], [0, 32]],
          [[0, 33], [0, 63]], 127),
    (4, 200, 1, 4, 2, 1.2, 5): ([[121, 61, 179, 39], [114, 62, 191, 33], [127, 48, 178, 47], [93, 68, 196, 43]],
          [[0, 121, 182, 361], [0, 114, 176, 367], [0, 127, 175, 353], [0, 93, 161, 357]],
          [[0, 121, 235, 362], [0, 61, 123, 171], [0, 179, 370, 548], [0, 39, 72, 119]], 744),
    (3, 17, 16, 2, 3, 0.0, 11): ([[19, 16, 16], [23, 11, 17], [22, 16, 13]],
          [[0, 19, 35], [0, 23, 34], [0, 22, 38]],
          [[0, 19, 42], [0, 16, 27], [0, 16, 33]], 64),
}


@pytest.mark.parametrize("seed", [0, 1, 7, 23])
@pytest.mark.parametrize("n, top_k", [(1, 1), (2, 2), (4, 3), (8, 8)])
def test_plan_index_fills_every_destination_range_once(n, top_k, seed):
    from container_engine_accelerators_b200.models.workloads import expert_dispatch_plan
    p = expert_dispatch_plan(n, 37, 16, top_k=top_k, skew=1.1, seed=seed)
    assert len(p.index) == n and len(p.weights) == n
    for s in range(n):
        idx = p.index[s]
        assert idx.dtype == np.int32 and idx.shape == (37, top_k)
        assert sorted(idx.ravel().tolist()) == list(range(int(p.rows[s].sum())))           # every dispatch row exactly once
        for d in range(n):
            lo, hi = int(p.send_off[s, d]), int(p.send_off[s, d] + p.rows[s, d])
            flat = idx.ravel()
            mine = flat[(flat >= lo) & (flat < hi)]
            assert mine.tolist() == list(range(lo, hi))                                     # row-major (token, slot) order
        w = p.weights[s]
        assert w.dtype == np.float32 and w.shape == (37, top_k) and (w > 0).all()
        assert np.allclose(w.astype(np.float64).sum(axis=1), 1.0, atol=1e-6)


def test_plan_counts_are_unchanged():
    from container_engine_accelerators_b200.models.workloads import expert_dispatch_plan
    for args, (rows, send_off, recv_off, max_rows) in PINNED.items():
        p = expert_dispatch_plan(*args)
        assert p.rows.tolist() == rows and p.send_off.tolist() == send_off and p.recv_off.tolist() == recv_off and p.max_rows == max_rows, args


# ------------------------------------------------------------------------------------------------- reference
def test_reference_sums_in_slot_order():
    """fp32: (2^24 + 1) + 1 rounds to 2^24 twice, 2^24 + (1 + 1) does not; the reference must give the slot-order bits."""
    big, one = np.float32(2.0 ** 24), np.float32(1.0)
    eo = [np.array([[big] * 16, [one] * 16, [one] * 16], dtype=np.float32)]
    look = cr.plan_lookup(eo, [3], [0], [0])
    index = np.array([[0, 1, 2], [1, 2, 0], [2, -1, 0]])
    got = cr.combine(look, index, None, 1.0, torch.float32)
    assert got[0, 0].item() == 2.0 ** 24                    # ((0 + 2^24) + 1) + 1
    assert got[1, 0].item() == 2.0 ** 24 + 2                # ((0 + 1) + 1) + 2^24
    assert got[2, 0].item() == 2.0 ** 24                    # ((0 + 1) + 2^24), slot 1 dropped
    w = np.array([[1.0, 1.0, 1.0], [0.5, 0.5, 1.0], [1.0, 1.0, 1.0]], dtype=np.float32)
    got = cr.combine(look, index, w, 2.0, torch.bfloat16)
    assert got[1, 0].item() == float(torch.tensor(2.0 * (2.0 ** 24 + 1), dtype=torch.float32).to(torch.bfloat16))
    # all slots dropped, and -0 in: +0 out
    eo = [np.array([[-0.0] * 16], dtype=np.float32)]
    got = cr.combine(cr.plan_lookup(eo, [1], [0], [0]), np.array([[-1, 5], [0, 0]]), None, 1.0, torch.float32)
    assert (got.view(torch.int32) == 0).all()
