"""The vocab-parallel cross-entropy (b200collVocabParallelCrossEntropy / ...Backward) in libb200coll, checked without a GPU: the library's
exp and log against float64 (exp exhaustively on [-87, 0], log on [1, 4) and at random points up to 2^31), the reference against a
per-element loop rendering of the header's formulas, the C prototypes against the ctypes argtypes, every Python refusal, the kernels'
instantiations, and ptxas's register, stack and spill report."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from container_engine_accelerators_b200.ops import coll
from tests import coll_xent_reference as ref
from tests.coll_binary_facts import NVCC_FLAGS, kernels, ptxas, template_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


def _ulps(got, x, fn):
    """|got - fn(x)| in units of the float32 spacing at the float64 value."""
    want = fn(x.astype(np.float64))
    sp = np.spacing(np.abs(want.astype(F))).astype(np.float64)
    with np.errstate(invalid="ignore"):
        return np.abs(got.astype(np.float64) - want) / sp


# ------------------------------------------------------------------------------------------------- exp and log
def test_exp_within_2_ulp_on_every_float_in_minus_87_0():
    lo, hi = int(F(-87.0).view(np.uint32)), 0x80000000           # -87 .. -0 as bit patterns, descending magnitudes
    worst = 0.0
    for a in range(hi, lo + 1, 1 << 25):
        x = np.arange(a, min(a + (1 << 25), lo + 1), dtype=np.uint32).view(F)
        worst = max(worst, float(_ulps(ref.xexp(x), x, np.exp).max()))
    assert worst <= 2.0, worst
    x = np.arange(0, int(F(88.7228317).view(np.uint32)) + 1, 997, dtype=np.uint32).view(F)      # the positive side, sampled
    assert float(_ulps(ref.xexp(x), x, np.exp).max()) <= 2.0


def test_exp_special_points():
    e = ref.xexp(np.array([0.0, -0.0, -87.0, -87.00001, -1e30, -np.inf, 88.7228317, 88.72284, np.inf, np.nan], dtype=F))
    assert e[0] == 1.0 and e[1] == 1.0                            # exp(0) is exactly 1
    assert e[2] > 0 and e[3] == 0 and e[4] == 0 and e[5] == 0     # +0 below -87
    assert np.isfinite(e[6]) and e[7] == np.inf and e[8] == np.inf and np.isnan(e[9])
    assert not np.signbit(e[3:6]).any()


def test_log_within_2_ulp_on_1_4_and_random_points():
    x = np.arange(int(F(1.0).view(np.uint32)), int(F(4.0).view(np.uint32)), dtype=np.uint32).view(F)
    assert float(_ulps(ref.xlog(x), x, np.log).max()) <= 2.0
    rng = np.random.default_rng(7)
    x = np.concatenate([rng.uniform(1, 2.0 ** 31, 1 << 22), np.exp2(rng.uniform(-126, 31, 1 << 22))]).astype(F)
    assert float(_ulps(ref.xlog(x), x, np.log).max()) <= 2.0
    s = ref.xlog(np.array([1.0, 0.0, np.inf, -1.0, np.nan], dtype=F))
    assert s[0] == 0.0 and not np.signbit(s[0]) and s[1] == -np.inf and s[2] == np.inf and np.isnan(s[3]) and np.isnan(s[4])


# ------------------------------------------------------------------------------------------------- the reference
def _logits(n, rows, vl, dt, seed, scale=4.0):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(rows, vl, generator=g) * scale).to(dt) for _ in range(n)]


@pytest.mark.parametrize("n,rows,vl", [(1, 5, 8), (1, 3, 40), (2, 4, 24), (3, 6, 16), (4, 3, 72), (2, 2, 520)])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "f16", "f32"])
def test_reference_agrees_with_the_loop_rendering(n, rows, vl, dt):
    if dt == torch.float32 and vl % 4 or dt != torch.float32 and vl % 8:
        pytest.skip("not a whole 16-byte row")
    xs = _logits(n, rows, vl, dt, seed=n * 31 + vl)
    t = np.random.default_rng(vl).integers(0, n * vl, rows)
    t[0] = -100                                                                   # ignored
    if rows > 2:
        t[1] = n * vl                                                             # out of range: NaN
        xs[0][2, :] = float("-inf")                                               # a whole -inf slice on rank 0
        xs[-1][2, 1] = float("inf") if n > 1 else 0.0
    got, want = ref.forward(xs, t), ref.forward_loop(xs, t)
    for a, b in zip(got, want):
        assert np.array_equal(a, b, equal_nan=True), (a, b)


def test_reference_matches_float64_cross_entropy():
    n, rows, vl = 4, 16, 256
    xs = _logits(n, rows, vl, torch.float32, seed=3)
    t = np.random.default_rng(1).integers(0, n * vl, rows)
    loss, lse = ref.forward(xs, t)
    full = torch.cat(xs, dim=1).double()
    want = torch.nn.functional.cross_entropy(full, torch.from_numpy(t), reduction="none").numpy()
    assert np.allclose(loss, want, rtol=1e-5, atol=1e-5)
    assert np.allclose(lse, torch.logsumexp(full, 1).numpy(), rtol=1e-6)
    # the gradient: softmax minus the one-hot, times dloss
    dl = np.linspace(0.5, 1.5, rows).astype(F)
    grads = torch.cat([ref.backward(xs[r], r, n, t, lse, dl) for r in range(n)], dim=1).double()
    sm = torch.softmax(full, 1) - torch.nn.functional.one_hot(torch.from_numpy(t), n * vl)
    assert torch.allclose(grads, sm * torch.from_numpy(dl).double()[:, None], atol=1e-6)


def test_rank_order_and_special_rows():
    """S sums e_0 .. e_{N-1} from +0 in rank order; NaN anywhere in a slice makes the row NaN even when every other column is -inf."""
    inf = float("inf")
    x = [torch.tensor([[-inf] * 4]), torch.tensor([[-inf, float("nan"), -inf, -inf]])]
    loss, lse = ref.forward(x, np.array([0]))
    assert np.isnan(loss[0]) and np.isnan(lse[0])
    loss, lse = ref.forward([torch.tensor([[-inf] * 4])] * 2, np.array([1]))      # everything -inf: S = +0, lse = -inf, loss NaN
    assert lse[0] == -inf and np.isnan(loss[0])
    loss, _ = ref.forward([torch.tensor([[1.0, 2.0, 3.0, 4.0]])] * 3, np.array([-100]), ignore_index=-100)
    assert loss[0] == 0.0 and not np.signbit(loss[0])
    g = ref.backward(torch.tensor([[1.0, 2.0, 3.0, 4.0]]), 0, 2, np.array([9]), np.array([5.0], F), np.array([1.0], F))
    assert torch.isnan(g).all()                                                   # target 9 outside [0, 8)


# ------------------------------------------------------------------------------------------------- C prototypes
def test_header_prototypes_match_the_ctypes_argtypes(tmp_path, coll_lib):
    src = tmp_path / "probe.c"
    src.write_text(r'''
#include <stdio.h>
#include "b200coll.h"
int main(void) {
  b200collResult_t (*f)(const void*, const int64_t*, float*, float*, size_t, size_t, int64_t, b200collDataType_t, b200collComm_t,
                        b200collStream_t) = b200collVocabParallelCrossEntropy;
  b200collResult_t (*g)(const void*, const int64_t*, const float*, const float*, void*, size_t, size_t, int64_t, b200collDataType_t,
                        b200collComm_t, b200collStream_t) = b200collVocabParallelCrossEntropyBackward;
  printf("%d %d\n", f != 0, g != 0);
  return 0;
}''')
    exe = tmp_path / "probe"
    libdir = os.path.dirname(coll_lib)
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "coll", "include"), str(src), "-o", str(exe),
                    "-L", libdir, "-lb200coll", "-Wl,-rpath," + libdir], check=True)
    assert subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split() == ["1", "1"]
    L = coll.load()
    vp, sz = C.c_void_p, C.c_size_t
    assert L.b200collVocabParallelCrossEntropy.argtypes == [vp, vp, vp, vp, sz, sz, C.c_int64, C.c_int, vp, vp]
    assert L.b200collVocabParallelCrossEntropyBackward.argtypes == [vp, vp, vp, vp, vp, sz, sz, C.c_int64, C.c_int, vp, vp]


# ------------------------------------------------------------------------------------------------- Python argument checks
_pool = torch.empty(1 << 16, dtype=torch.float64)


def _v(off, shape, dt):
    es = torch.empty((), dtype=dt).element_size()
    n = 1
    for d in shape:
        n *= d
    return _pool.view(torch.uint8)[off:off + n * es].view(dt).view(shape)


class _Shifted:
    """A tensor's metadata with its address moved by `by` bytes: misaligned pointers torch views cannot make."""

    def __init__(self, t, by):
        self.t, self.by, self.dtype, self.shape = t, by, t.dtype, t.shape

    def __getattr__(self, name):
        return getattr(self.t, name)

    def data_ptr(self):
        return self.t.data_ptr() + self.by


def _call(n=2, **kw):
    a = dict(logits=_v(0, (4, 64), torch.bfloat16), target=_v(1024, (4,), torch.int64), loss=_v(2048, (4,), torch.float32),
             lse=_v(3072, (4,), torch.float32))
    a.update(kw)
    return coll.check_vocab_parallel_cross_entropy(n, **a)


def _bwd(n=2, **kw):
    a = dict(logits=_v(0, (4, 64), torch.bfloat16), target=_v(1024, (4,), torch.int64), lse=_v(2048, (4,), torch.float32),
             dloss=_v(3072, (4,), torch.float32), grad=_v(4096, (4, 64), torch.bfloat16))
    a.update(kw)
    return coll.check_vocab_parallel_cross_entropy(n, **a)


def test_checks_accept_valid_calls():
    assert _call() == (4, 64)
    assert _bwd() == (4, 64)
    assert _bwd(grad=_v(0, (4, 64), torch.bfloat16)) == (4, 64)                    # in place
    assert _call(8, logits=_v(0, (4, 4), torch.float32)) == (4, 4)
    assert _call(logits=_v(0, (0, 8), torch.float16), target=_v(1024, (0,), torch.int64), loss=_v(2048, (0,), torch.float32),
                 lse=_v(3072, (0,), torch.float32)) == (0, 8)


def test_refusals():
    cases = [
        (dict(logits=_v(0, (4, 64), torch.float64)), "bfloat16, float16 or float32"),
        (dict(logits=_v(0, (4, 8), torch.int32)), "bfloat16, float16 or float32"),
        (dict(logits=_v(0, (256,), torch.bfloat16)), "contiguous \\[rows, vocab_local\\]"),
        (dict(logits=_v(0, (64, 4), torch.bfloat16).t()), "contiguous \\[rows, vocab_local\\]"),
        (dict(logits=_v(0, (4, 0), torch.bfloat16)), "multiple of 16 bytes"),
        (dict(logits=_v(0, (4, 12), torch.bfloat16)), "multiple of 16 bytes"),
        (dict(logits=_v(0, (4, 6), torch.float32)), "multiple of 16 bytes"),
        (dict(target=_v(1024, (4,), torch.int32)), "int64"),
        (dict(target=_v(1024, (5,), torch.int64)), "int64"),
        (dict(loss=_v(2048, (4,), torch.float16)), "loss must be"),
        (dict(lse=_v(3072, (3,), torch.float32)), "lse must be"),
        (dict(logits=_v(8, (4, 64), torch.bfloat16)), "16-byte aligned"),
        (dict(target=_Shifted(_v(1024, (4,), torch.int64), 4)), "8-byte aligned"),
        (dict(loss=_Shifted(_v(2048, (4,), torch.float32), 2)), "4-byte aligned"),
        (dict(loss=_v(64, (4,), torch.float32)), "must not overlap the inputs"),
        (dict(lse=_v(1024, (4,), torch.float32)), "must not overlap the inputs"),
        (dict(lse=_v(2056, (4,), torch.float32)), "must not overlap each other"),
    ]
    for kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            _call(**kw)
    bcases = [
        (dict(grad=_v(4096, (4, 64), torch.float16)), "grad must be"),
        (dict(grad=_v(16, (4, 64), torch.bfloat16)), "must not overlap the inputs"),        # partly over the logits
        (dict(grad=_v(768, (4, 64), torch.bfloat16)), "must not overlap the inputs"),       # over the target
        (dict(grad=_v(2048, (4, 64), torch.bfloat16)), "must not overlap the inputs"),      # over lse and dloss
        (dict(dloss=_Shifted(_v(3072, (4,), torch.float32), 2)), "4-byte aligned"),
        (dict(grad=_v(4104, (4, 64), torch.bfloat16)), "16-byte aligned"),
    ]
    for kw, msg in bcases:
        with pytest.raises(ValueError, match=msg):
            _bwd(**kw)
    with pytest.raises(ValueError, match="below 2\\^31"):
        coll.check_vocab_parallel_cross_entropy(8, torch.empty((2, 1 << 28), dtype=torch.bfloat16, device="meta"),
                                                torch.empty(2, dtype=torch.int64, device="meta"))
    with pytest.raises(ValueError, match="rows must be below"):
        coll.check_vocab_parallel_cross_entropy(1, torch.empty((1 << 31, 8), dtype=torch.bfloat16, device="meta"),
                                                torch.empty(1 << 31, dtype=torch.int64, device="meta"))


# ------------------------------------------------------------------------------------------------- what the compiler made
def test_one_forward_per_dtype_and_locality_one_backward_per_dtype(coll_lib):
    dts = ("__nv_bfloat16", "__half", "float")
    fwd = kernels(coll_lib, "b200coll::k_xent<")
    assert sorted(template_args(k) for k in fwd) == sorted((d, loc) for d in dts for loc in ("false", "true")), fwd
    bwd = kernels(coll_lib, "b200coll::k_xent_bwd<")
    assert sorted(template_args(k) for k in bwd) == sorted((d,) for d in dts), bwd


def test_ptxas_no_stack_no_spills_registers_reported():
    report, regs = ptxas("xent.cu")
    mine = {k: v for k, v in report.items() if "k_xent" in k}
    assert len(mine) == 9, sorted(report)
    for k, (stack, st, ld) in mine.items():
        assert (stack, st, ld) == (0, 0, 0), (k, stack, st, ld)
        assert k in regs and 0 < regs[k] <= 64, (k, regs.get(k))


def test_compiles_without_warnings(tmp_path):
    r = subprocess.run([os.environ.get("NVCC", "nvcc"), *NVCC_FLAGS, "-c", os.path.join(ROOT, "coll", "src", "xent.cu"), "-o",
                        str(tmp_path / "xent.o")], capture_output=True, text=True)
    assert r.returncode == 0 and "warning" not in r.stderr.lower(), r.stderr
