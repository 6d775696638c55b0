"""The vocab-parallel embedding (b200collVocabParallelEmbedding / ...Backward) in libb200coll, checked without a GPU: the reference
against a per-element loop rendering of the header's formulas, the C prototypes against the ctypes argtypes, every Python refusal, the
kernels' instantiations, and ptxas's register, stack and spill report."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from container_engine_accelerators_b200.ops import coll
from tests import coll_embedding_reference as ref
from tests.coll_binary_facts import NVCC_FLAGS, kernels, ptxas, template_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


def _bits(rng, shape, dt):
    x = (rng.standard_normal(shape) * 2).astype(F)
    return ref.narrow(x, dt)


# ------------------------------------------------------------------------------------------------- the reference
@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
def test_forward_matches_per_element_loop(dt):
    rng = np.random.default_rng(1)
    n, vl, h, T = 3, 5, 8, 23
    tables = [_bits(rng, (vl, h), dt) for _ in range(n)]
    ids = rng.integers(-3, n * vl + 3, T)
    ids[0], ids[1] = n * vl, -1
    for sp in (False, True):
        T2 = 21 if sp else T
        for r in range(n):
            got = ref.forward(tables, ids[:T2], sp, r)
            lo = r * T2 // n if sp else 0
            for i in range(got.shape[0]):
                t = lo + i
                for k in range(h):
                    g = int(ids[t])
                    want = tables[g // vl][g % vl, k] if 0 <= g < n * vl else 0
                    assert got[i, k] == want


@pytest.mark.parametrize("dt,wdt", [("bf16", "f32"), ("bf16", "bf16"), ("f16", "f32"), ("f16", "f16"), ("f32", "f32")])
def test_backward_matches_per_element_loop(dt, wdt):
    rng = np.random.default_rng(2)
    n, vl, h, T = 2, 4, 8, 31
    ids = rng.integers(-2, n * vl + 2, T)
    dout = _bits(rng, (T, h), dt)
    old = _bits(rng, (vl, h), wdt)
    for r in range(n):
        for acc in (None, old):
            got = ref.backward(ids, dout, dt, r, n, vl, wdt, acc)
            for j in range(vl):
                for k in range(h):
                    s = ref.widen(acc[j, k:k + 1], wdt)[0] if acc is not None else F(0.0)
                    for t in range(T):
                        if ids[t] == r * vl + j:
                            s = F(s + ref.widen(dout[t, k:k + 1], dt)[0])
                    want = ref.narrow(np.array([s], dtype=F), wdt)[0]
                    assert got[j, k] == want, (r, j, k)


def test_backward_order_is_token_order():
    """Three values whose fp32 sum depends on the order: the fold must be left to right in token order."""
    dout = ref.narrow(np.array([[1e8], [1.0], [-1e8], [1.0]], dtype=F).repeat(4, 1), "f32")
    got = ref.backward([0, 0, 0, 0], dout, "f32", 0, 1, 1, "f32")
    assert ref.widen(got, "f32")[0, 0] == F(F(F(F(1e8) + F(1.0)) + F(-1e8)) + F(1.0))


def test_narrow_is_round_to_nearest_even():
    x = np.array([1.0, 1.00390625, 1.01171875, -0.0, np.inf, 3.4e38], dtype=F)
    got = ref.narrow(x, "bf16")
    assert np.array_equal(got, torch.from_numpy(x).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16))
    assert np.isnan(ref.widen(ref.narrow(np.array([np.nan], dtype=F), "bf16"), "bf16")).all()


# ------------------------------------------------------------------------------------------------- the C API
def test_prototypes_match_ctypes():
    hdr = open(os.path.join(ROOT, "coll", "include", "b200coll.h")).read()
    for name, nargs in (("b200collVocabParallelEmbedding", 10), ("b200collVocabParallelEmbeddingBackward", 12)):
        m = re.search(r"b200collResult_t " + name + r"\(([^)]*)\);", hdr)
        assert m, name
        assert len([a for a in m.group(1).split(",") if a.strip()]) == nargs
    src = open(os.path.join(ROOT, "container_engine_accelerators_b200", "ops", "coll.py")).read()
    assert "L.b200collVocabParallelEmbedding.argtypes = [vp, vp, vp, sz, sz, sz, ci, ci, vp, vp]" in src
    assert "L.b200collVocabParallelEmbeddingBackward.argtypes = [vp, vp, vp, sz, sz, sz, ci, ci, ci, ci, vp, vp]" in src


def test_symbols_exported(coll_lib):
    lib = C.CDLL(coll_lib)
    assert lib.b200collVocabParallelEmbedding and lib.b200collVocabParallelEmbeddingBackward


# ------------------------------------------------------------------------------------------------- the Python refusals
def _v(off, shape, dt):
    """A metadata-only tensor at byte offset `off` of one 64 KiB meta storage."""
    base = torch.empty(1 << 16, dtype=torch.uint8, device="meta")
    return base[off:].view(dt)[:int(np.prod(shape))].view(shape) if shape else base[off:].view(dt)[:0]


class _Shifted:
    def __init__(self, t, by):
        self.t, self.by, self.dtype, self.shape = t, by, t.dtype, t.shape

    def __getattr__(self, name):
        return getattr(self.t, name)

    def data_ptr(self):
        return self.t.data_ptr() + self.by


def _fwd(n=2, sp=False, sym=None, **kw):
    a = dict(ids=_v(0, (8,), torch.int64), table=_v(1024, (16, 64), torch.bfloat16), rows=_v(8192, (8 // n if sp else 8, 64), torch.bfloat16))
    a.update(kw)
    return coll.check_vocab_parallel_embedding(n, a["ids"], a["table"], a["rows"], sequence_parallel=sp, symmetric=sym)


def _bwd(n=2, sp=False, sym=None, **kw):
    a = dict(ids=_v(0, (8,), torch.int64), table=_v(1024, (16, 64), torch.float32), rows=_v(8192, (8 // n if sp else 8, 64), torch.bfloat16))
    a.update(kw)
    return coll.check_vocab_parallel_embedding(n, a["ids"], a["table"], a["rows"], sequence_parallel=sp, backward=True, symmetric=sym)


def test_checks_accept_valid_calls():
    assert _fwd() == (8, 64, 16)
    assert _fwd(sp=True) == (8, 64, 16)
    assert _bwd() == (8, 64, 16)
    assert _bwd(table=_v(1024, (16, 64), torch.bfloat16)) == (8, 64, 16)
    assert _bwd(n=4, sp=True, sym=lambda t: True) == (8, 64, 16)
    assert _fwd(ids=_v(0, (0,), torch.int64), rows=_v(8192, (0, 64), torch.bfloat16)) == (0, 64, 16)
    assert _fwd(n=8, table=_v(1024, (1, 4), torch.float32), rows=_v(8192, (8, 4), torch.float32)) == (8, 4, 1)


def test_refusals():
    cases = [
        (_fwd, dict(table=_v(1024, (16, 64), torch.float64), rows=_v(8192, (8, 64), torch.float64)), "bfloat16, float16 or float32"),
        (_fwd, dict(rows=_v(8192, (8, 64), torch.float16)), "out must have weight's dtype"),
        (_bwd, dict(rows=_v(8192, (8, 64), torch.float64)), "bfloat16, float16 or float32"),
        (_bwd, dict(table=_v(1024, (16, 64), torch.float16)), "dweight must be float32 or grad_out's dtype"),
        (_fwd, dict(ids=_v(0, (8,), torch.int32)), "int64"),
        (_fwd, dict(table=_v(1024, (16, 4), torch.bfloat16), rows=_v(8192, (8, 4), torch.bfloat16)), "multiple of 16 bytes"),
        (_bwd, dict(table=_v(1024, (16, 6), torch.float32), rows=_v(8192, (8, 6), torch.float32)), "multiple of 16 bytes"),
        (_bwd, dict(table=_v(1024, (16, 4), torch.float32), rows=_v(8192, (8, 4), torch.bfloat16)), "multiple of 16 bytes"),   # bf16 dout
        (_fwd, dict(table=_v(1024, (16, 0), torch.bfloat16), rows=_v(8192, (8, 0), torch.bfloat16)), "multiple of 16 bytes"),
        (_fwd, dict(table=_v(1024, (0, 64), torch.bfloat16)), "vocab_local must be positive"),
        (_fwd, dict(ids=_v(0, (6,), torch.int64), rows=_v(8192, (1, 64), torch.bfloat16), n=4, sp=True), "multiple of nranks"),
        (_fwd, dict(rows=_v(8192, (7, 64), torch.bfloat16)), "out must be a contiguous"),
        (_fwd, dict(table=_v(1032, (16, 64), torch.bfloat16)), "16-byte aligned"),
        (_bwd, dict(rows=_v(8200, (8, 64), torch.bfloat16)), "16-byte aligned"),
        (_fwd, dict(ids=_Shifted(_v(0, (8,), torch.int64), 4)), "8-byte aligned"),
        (_fwd, dict(rows=_v(1024, (8, 64), torch.bfloat16)), "out must not overlap weight or ids"),
        (_fwd, dict(rows=_v(0, (8, 64), torch.bfloat16), table=_v(2048, (16, 64), torch.bfloat16)), "out must not overlap weight or ids"),
        (_bwd, dict(rows=_v(2048, (8, 64), torch.bfloat16)), "dweight must not overlap dout or ids"),
        (_bwd, dict(table=_v(0, (16, 64), torch.float32), rows=_v(8192, (8, 64), torch.bfloat16)), "dweight must not overlap dout or ids"),
        (_fwd, dict(sym=lambda t: False), "symmetric arena"),
        (_bwd, dict(sp=True, sym=lambda t: False), "symmetric arena"),
    ]
    for fn, kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            fn(**kw)
    _bwd(sym=lambda t: False)                 # the tensor-parallel dout may be any memory
    _fwd(n=1, sym=lambda t: False)            # and one rank's weight
    meta = lambda shape, dt: torch.empty(shape, dtype=dt, device="meta")      # noqa: E731
    with pytest.raises(ValueError, match="below 2\\^31"):
        coll.check_vocab_parallel_embedding(8, meta(4, torch.int64), meta((1 << 28, 8), torch.bfloat16), meta((4, 8), torch.bfloat16))
    with pytest.raises(ValueError, match="tokens must be below"):
        coll.check_vocab_parallel_embedding(1, meta(1 << 31, torch.int64), meta((4, 8), torch.bfloat16))
    with pytest.raises(ValueError, match="2\\^31 - 1 16-byte vectors"):
        coll.check_vocab_parallel_embedding(1, meta(1 << 20, torch.int64), meta((4, 1 << 15), torch.float32),
                                            meta((1 << 20, 1 << 15), torch.float32))


# ------------------------------------------------------------------------------------------------- what the compiler made
def test_instantiations(coll_lib):
    dts = ("__nv_bfloat16", "__half", "float")
    fwd = kernels(coll_lib, "b200coll::k_emb_fwd<")
    assert sorted(template_args(k) for k in fwd) == [("false",), ("true",)], fwd
    bwd = kernels(coll_lib, "b200coll::k_emb_bwd<")
    want = sorted({(d, w, p) for d in dts for w in (d, "float") for p in ("false", "true")})
    assert sorted(template_args(k) for k in bwd) == want, bwd
    for k in ("k_emb_hist<", "k_emb_scatter<"):
        assert sorted(template_args(x) for x in kernels(coll_lib, "b200coll::" + k)) == [("false",), ("true",)]
    assert kernels(coll_lib, "b200coll::k_emb_scan(") and kernels(coll_lib, "b200coll::k_emb_bounds(")


def test_ptxas_no_stack_no_spills_registers_reported():
    report, regs = ptxas("embedding.cu")
    mine = {k: v for k, v in report.items() if "k_emb_" in k}
    assert len(mine) == 18, sorted(report)          # 10 folds, 2 forwards, 6 sort kernels
    for k, (stack, st, ld) in mine.items():
        assert (stack, st, ld) == (0, 0, 0), (k, stack, st, ld)
        assert k in regs and 0 < regs[k] <= 64, (k, regs.get(k))


def test_compiles_without_warnings(tmp_path):
    r = subprocess.run([os.environ.get("NVCC", "nvcc"), *NVCC_FLAGS, "-c", os.path.join(ROOT, "coll", "src", "embedding.cu"), "-o",
                        str(tmp_path / "embedding.o")], capture_output=True, text=True)
    assert r.returncode == 0 and "warning" not in r.stderr.lower(), r.stderr
