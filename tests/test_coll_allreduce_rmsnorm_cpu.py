"""The fused all-reduce, residual add and RMSNorm in libb200coll, checked without a GPU: the C prototype against the ctypes argtypes,
every Python refusal, the kernels' instantiations, ptxas's stack and spill report, the perf tool's help and refusals, and the numpy
reference against a plain loop rendering of the same rules."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from container_engine_accelerators_b200.ops import coll
from tests import coll_rmsnorm_reference as ref
from tests.coll_binary_facts import kernels, ptxas, template_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PERF = os.path.join(ROOT, "build", "b200coll_perf")
WIDE = ("__nv_bfloat16", "__half", "float")
FAMILIES = ("k_rms_local", "k_rms_oneshot", "k_rms_twoshot")


def test_header_prototype_matches_the_ctypes_argtypes(tmp_path, coll_lib):
    src = tmp_path / "probe.c"
    src.write_text(r'''
#include <stdio.h>
#include "b200coll.h"
int main(void) {
  b200collResult_t (*f)(const void*, void*, const void*, void*, size_t, size_t, float, b200collDataType_t, b200collComm_t, b200collStream_t) =
      b200collAllReduceRmsNorm;
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
    assert L.b200collAllReduceRmsNorm.argtypes == [vp, vp, vp, vp, sz, sz, C.c_float, ci, vp, vp]


# ------------------------------------------------------------------------------------------------- Python argument checks
_pool = torch.empty(1 << 16, dtype=torch.float32)


def _v(off, n, dt):
    """n elements of dt at byte offset `off` of one pool (so alignment and overlaps are under the test's control)."""
    es = torch.empty((), dtype=dt).element_size()
    return _pool.view(torch.uint8)[off:off + n * es].view(dt)


def _args(rows=4, row_len=64, dt=torch.bfloat16, **kw):
    es = torch.empty((), dtype=dt).element_size()
    mat = rows * row_len * es
    a = {"x": _v(0, rows * row_len, dt).view(rows, row_len), "residual": _v(mat + 64, rows * row_len, dt).view(rows, row_len),
         "weight": _v(2 * mat + 128, row_len, dt), "out": _v(3 * mat + 192, rows * row_len, dt).view(rows, row_len), "eps": 1e-6}
    a.update(kw)
    return a


def test_check_accepts_a_valid_call():
    for dt in (torch.bfloat16, torch.float16, torch.float32):
        assert coll.check_all_reduce_rms_norm(**_args(dt=dt)) == (4, 64)
    a = _args()
    assert coll.check_all_reduce_rms_norm(a["x"].view(2, 2, 64), a["residual"].view(2, 2, 64), a["weight"], a["out"].view(2, 2, 64)) == (4, 64)
    z = _args(rows=0)
    assert coll.check_all_reduce_rms_norm(**z) == (0, 64)


def _refused(match, **kw):
    with pytest.raises(ValueError, match=match):
        coll.check_all_reduce_rms_norm(**_args(**kw))


def test_check_refusals():
    a = _args()
    _refused("x must be a contiguous bfloat16", x=torch.zeros(4, 64, dtype=torch.float8_e4m3fn))
    _refused("x must be a contiguous", x=torch.zeros(64, 4, dtype=torch.bfloat16).t())
    _refused("weight must have x's dtype", weight=torch.zeros(64, dtype=torch.float16))
    _refused("out must have x's dtype", out=torch.zeros(4, 64, dtype=torch.float32))
    _refused("residual must have x's shape", residual=a["residual"].view(-1)[:128].view(2, 64))
    _refused("out must have x's shape", out=a["out"].view(8, 32))
    _refused("row_len", rows=2, row_len=24)
    _refused("row_len", rows=1, row_len=16400)
    _refused("row_len", x=torch.zeros(4, 8, dtype=torch.bfloat16), residual=torch.zeros(4, 8, dtype=torch.bfloat16),
             out=torch.zeros(4, 8, dtype=torch.bfloat16), weight=torch.zeros(8, dtype=torch.bfloat16))
    _refused("weight must have shape", weight=a["weight"][:32])
    for eps in (-1e-6, float("nan"), float("inf"), "1e-6", True):
        _refused("eps", eps=eps)
    _refused("16-byte aligned", residual=_v(4096 + 2, 256, torch.bfloat16).view(4, 64))
    _refused("out must not overlap", out=a["x"])
    _refused("out must not overlap", out=_v(a["weight"].data_ptr() - _pool.data_ptr(), 256, torch.bfloat16).view(4, 64))
    _refused("residual must not overlap", residual=_v(0 + 128, 256, torch.bfloat16).view(4, 64))
    _refused("residual must not overlap", residual=_v(a["weight"].data_ptr() - _pool.data_ptr(), 256, torch.bfloat16).view(4, 64))


def test_check_refuses_2_31_rows():
    big = torch.empty((1 << 31, 16), dtype=torch.bfloat16, device="meta")
    w = torch.empty(16, dtype=torch.bfloat16, device="meta")
    with pytest.raises(ValueError, match="2\\^31"):
        coll.check_all_reduce_rms_norm(big, big, w, big)


# ------------------------------------------------------------------------------------------------- what the compiler made
def test_one_instantiation_per_dtype_and_algorithm(coll_lib):
    for fam in FAMILIES:
        names = kernels(coll_lib, f"b200coll::{fam}<")
        assert sorted(template_args(nm)[0] for nm in names) == sorted(WIDE), (fam, names)


def test_ptxas_no_stack_no_spills():
    report, regs = ptxas("rmsnorm.cu")
    mine = {k: v for k, v in report.items() if "k_rms_" in k}
    assert len(mine) == 9, sorted(report)
    for k, (stack, st, ld) in mine.items():
        assert (stack, st, ld) == (0, 0, 0), (k, stack, st, ld)
        assert regs[k] <= 128, (k, regs[k])                    # one 512-thread CTA per SM


# ------------------------------------------------------------------------------------------------- perf tool
def test_perf_tool_help_and_refusals(coll_lib):
    h = subprocess.run([PERF, "--help"], capture_output=True, text=True)
    assert h.returncode == 0 and "--rms-norm ROW_LEN" in h.stdout
    for extra in (["--rms-norm", "24"], ["--rms-norm", "0"], ["--rms-norm", "16400"]):
        r = subprocess.run([PERF, *extra], capture_output=True, text=True)
        assert r.returncode == 1 and "a multiple of 16 in [16, 16384]" in r.stderr, (extra, r.stderr)
    for extra in (["--op", "alltoall"], ["-d", "fp8"], ["--out-dtype", "float"], ["--scale", "2"], ["--quantize", "e4m3:128"],
                  ["--block-scale", "1x128"], ["--combine", "2"], ["--route", "8:2"]):
        r = subprocess.run([PERF, "--rms-norm", "64", *extra], capture_output=True, text=True)
        assert r.returncode == 1 and "--rms-norm ROW_LEN takes --op all_reduce" in r.stderr, (extra, r.stderr)


# ------------------------------------------------------------------------------------------------- the reference
def _case(n, rows, row_len, dt, seed):
    g = torch.Generator().manual_seed(seed)
    xs = [(torch.randn(rows, row_len, generator=g) * (1 + r)).to(dt) for r in range(n)]
    res = (torch.randn(rows, row_len, generator=g) * 3).to(dt)
    gamma = (torch.rand(row_len, generator=g) * 2 - 0.5).to(dt)
    return xs, res, gamma


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16, torch.float32])
def test_reference_agrees_with_the_loop_rendering(dt):
    for n, rows, row_len in ((1, 2, 16), (3, 2, 48), (2, 1, 112), (4, 2, 256)):        # 1, 3 (padded), 7 (padded) and 16 chunks
        xs, res, gamma = _case(n, rows, row_len, dt, seed=n * 7 + row_len)
        res[0, 5] = float("inf") if rows > 1 else res[0, 5]
        for eps in (0.0, 1e-6):
            fh, fo = ref.rms_norm(xs, res, gamma, eps, dt)
            lh, lo = ref.rms_norm_loop(xs, res, gamma, eps, dt)
            assert torch.equal(fh.view(-1).float().nan_to_num(7.0), lh.view(-1).float().nan_to_num(7.0))
            assert torch.equal(fo.float().isnan(), lo.float().isnan())
            assert torch.equal(fo.float().nan_to_num(7.0), lo.float().nan_to_num(7.0)), (n, rows, row_len, eps)


def test_reference_special_rows():
    dt = torch.float32
    z = torch.zeros(1, 32, dtype=dt)
    _, o = ref.rms_norm([z], z, torch.ones(32, dtype=dt), 0.0, dt)
    assert o.isnan().all()                                            # 0 * (1 / sqrt(0))
    _, o = ref.rms_norm([z], z, torch.ones(32, dtype=dt), 1e-6, dt)
    assert (o == 0).all()
    x = torch.ones(1, 32, dtype=dt)
    _, o = ref.rms_norm([x], z, torch.ones(32, dtype=dt), 0.0, dt)
    assert (o == 1).all()


def test_reference_fold_order_is_not_a_plain_sum():
    """The fold's order is part of the contract: find a row where it differs from a left-to-right sum of the squares, so a kernel or
    reference that summed in element order would be caught."""
    dt = torch.float32
    rng = np.random.default_rng(1)
    for _ in range(50):
        h = torch.from_numpy((rng.standard_normal((1, 1024)) * np.exp(rng.standard_normal((1, 1024)) * 4)).astype(np.float32))
        _, o = ref.rms_norm([h], torch.zeros_like(h), torch.ones(1024, dtype=dt), 0.0, dt)
        s = np.float32(0)
        for v in h.numpy().reshape(-1):
            s = np.float32(s + np.float32(v * v))
        plain = h.numpy() * (np.float32(1) / np.sqrt(s / np.float32(1024)))
        if not np.array_equal(o.numpy(), plain.astype(np.float32)):
            return
    pytest.fail("the fold agreed with the sequential sum on every row tried")
