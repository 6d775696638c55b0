"""Device-routed expert dispatch and combine in libb200coll, checked without a GPU: the C prototypes against the ctypes argtypes, the
Python argument checks, the numpy layout reference against slot-by-slot placement, the kernels' instantiations, SASS (no FFMA in any
combine kernel) and ptxas's stack and spill report, the perf tool's mode, and the dispatch plan's expert ids."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from container_engine_accelerators_b200.ops import coll
from tests import coll_routed_reference as rr
from tests.coll_binary_facts import kernels, ptxas, sass, template_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIDE = ("__nv_bfloat16", "__half", "float")


def test_header_prototypes_match_the_ctypes_argtypes(tmp_path, coll_lib):
    src = tmp_path / "probe.c"
    src.write_text(r'''
#include <stdio.h>
#include "b200coll.h"
int main(void) {
  b200collResult_t (*d)(const void*, void*, size_t, size_t, const int32_t*, size_t, int, int, int32_t*, int32_t*, int32_t*, b200collDataType_t,
                        b200collComm_t, b200collStream_t) = b200collExpertDispatch;
  b200collResult_t (*c)(const void*, void*, size_t, size_t, const int32_t*, const float*, size_t, int, const b200collEpilogue*, b200collComm_t,
                        b200collStream_t) = b200collExpertCombine;
  printf("%d %d\n", d != 0, c != 0);
  return 0;
}''')
    exe = tmp_path / "probe"
    libdir = os.path.dirname(coll_lib)
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "coll", "include"), str(src), "-o", str(exe),
                    "-L", libdir, "-lb200coll", "-Wl,-rpath," + libdir], check=True)
    assert subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split() == ["1", "1"]
    L = coll.load()
    vp, sz, ci, i32 = C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_int32)
    assert L.b200collExpertDispatch.argtypes == [vp, vp, sz, sz, i32, sz, ci, ci, i32, i32, i32, ci, vp, vp]
    assert L.b200collExpertCombine.argtypes == [vp, vp, sz, sz, i32, C.POINTER(C.c_float), sz, ci, C.POINTER(coll.Epilogue), vp, vp]


# ------------------------------------------------------------------------------------------------- Python argument checks
def _t(n, dt):
    return torch.empty(n, dtype=dt)


def _d(**kw):
    """A valid dispatch for 2 ranks: 5 tokens of 32 bf16 elements, top-3 over 8 experts, 12 recv rows; keyword arguments override."""
    a = dict(nranks=2, x=torch.empty(5, 32, dtype=torch.bfloat16), topk_idx=torch.zeros(5, 3, dtype=torch.int32), num_experts=8,
             recv=_t(12 * 32, torch.bfloat16), expert_counts=_t(4, torch.int32), route=torch.empty(5, 3, dtype=torch.int32), dropped=_t(1, torch.int32))
    a.update(kw)
    return a


def test_dispatch_check_accepts_the_documented_shapes():
    assert coll.check_expert_dispatch(**_d()) == coll.BF16
    assert coll.check_expert_dispatch(**_d(expert_counts=None, route=None, dropped=None)) == coll.BF16
    assert coll.check_expert_dispatch(**_d(x=torch.empty(5, 16), recv=_t(16 * 40, torch.float32), num_experts=1024, expert_counts=None)) == coll.F32
    # no tokens at all, one rank with one expert, a 2-D recv
    assert coll.check_expert_dispatch(1, torch.empty(0, 16, dtype=torch.float16), torch.zeros(0, 8, dtype=torch.int32), 1,
                                      torch.empty(3, 16, dtype=torch.float16)) == coll.F16


_base = torch.empty(4096, dtype=torch.int32)


@pytest.mark.parametrize("what, kw", [
    ("FP8 x", dict(x=torch.empty(5, 32, dtype=torch.float8_e4m3fn), recv=_t(384, torch.float8_e4m3fn))),
    ("1-D x", dict(x=_t(160, torch.bfloat16))),
    ("non-contiguous x", dict(x=torch.empty(32, 5, dtype=torch.bfloat16).t())),
    ("row_elems 24", dict(x=torch.empty(5, 24, dtype=torch.bfloat16), recv=_t(24 * 12, torch.bfloat16))),
    ("int64 topk_idx", dict(topk_idx=torch.zeros(5, 3, dtype=torch.int64))),
    ("top_k 0", dict(topk_idx=torch.zeros(5, 0, dtype=torch.int32), route=None)),
    ("topk_idx of other tokens", dict(topk_idx=torch.zeros(4, 3, dtype=torch.int32), route=None)),
    ("0 experts", dict(num_experts=0)),
    ("1025 experts", dict(num_experts=1025)),
    ("experts not a multiple of nranks", dict(num_experts=7)),
    ("experts True", dict(nranks=1, num_experts=True)),
    ("recv of another dtype", dict(recv=_t(384, torch.float16))),
    ("recv of part of a row", dict(recv=_t(380, torch.bfloat16))),
    ("expert_counts of the wrong size", dict(expert_counts=_t(8, torch.int32))),
    ("int64 route", dict(route=torch.empty(5, 3, dtype=torch.int64))),
    ("dropped of two", dict(dropped=_t(2, torch.int32))),
    ("nranks * recv rows > 2^31 - 1", dict(nranks=8, num_experts=8, expert_counts=_t(1, torch.int32),
                                           recv=torch.empty(2 ** 28 * 32, dtype=torch.bfloat16, device="meta"))),
    ("recv overlaps x", dict(x=_base[:80].view(torch.bfloat16).view(5, 32), recv=_base[64:256].view(torch.bfloat16))),
    ("route overlaps expert_counts", dict(expert_counts=_base[:4], route=_base[2:17].view(5, 3))),
    ("dropped overlaps route", dict(route=_base[:15].view(5, 3), dropped=_base[14:15])),
    ("route overlaps topk_idx", dict(topk_idx=_base[:15].view(5, 3), route=_base[10:25].view(5, 3))),
    ("expert_counts in recv", dict(recv=_base[:192].view(torch.bfloat16), expert_counts=_base[100:104])),
])
def test_dispatch_check_raises_value_error(what, kw):
    with pytest.raises((ValueError, RuntimeError)) as e:
        coll.check_expert_dispatch(**_d(**kw))
    assert e.type is ValueError, (what, e.value)


@pytest.mark.parametrize("what, kw, rule", [
    ("tokens * top_k > 2^31 - 1", dict(x=torch.empty(2 ** 30, 16, dtype=torch.bfloat16, device="meta"),
                                       topk_idx=torch.empty(2 ** 30, 2, dtype=torch.int32, device="meta"), route=None), "tokens \\* top_k"),
    ("more than 2^31 - 1 vectors", dict(x=torch.empty(2 ** 24, 512, dtype=torch.bfloat16, device="meta"), recv=_t(512 * 12, torch.bfloat16),
                                        topk_idx=torch.empty(2 ** 24, 8, dtype=torch.int32, device="meta"), route=None), "16-byte vectors"),
    ("nranks * recv rows > 2^31 - 1", dict(nranks=8, num_experts=8, expert_counts=_t(1, torch.int32),
                                           recv=torch.empty(2 ** 28 * 32, dtype=torch.bfloat16, device="meta")), "nranks \\* recv rows"),
])
def test_dispatch_check_size_limits_name_their_rule(what, kw, rule):
    """Each size limit is refused by its own rule, with every other argument valid (meta tensors: no memory behind them)."""
    with pytest.raises(ValueError, match=rule):
        coll.check_expert_dispatch(**_d(**kw))


def _c(**kw):
    """A valid combine for 2 ranks: expert_out of 12 rows of 32 elements, 5 tokens of top-3."""
    a = dict(nranks=2, expert_out=_t(12 * 32, torch.bfloat16), route=torch.zeros(5, 3, dtype=torch.int32), weights=torch.ones(5, 3),
             out=torch.empty(5, 32, dtype=torch.float32))
    a.update(kw)
    return a


def test_combine_check_accepts_the_documented_shapes():
    assert coll.check_expert_combine(**_c()) == (coll.BF16, coll.F32)
    assert coll.check_expert_combine(**_c(weights=None, expert_out=_t(64, torch.float16), out=torch.empty(5, 32, dtype=torch.bfloat16))) == (coll.F16, coll.BF16)
    assert coll.check_expert_combine(1, _t(32, torch.float32), torch.zeros(0, 2, dtype=torch.int32), None, torch.empty(0, 16)) == (coll.F32, coll.F32)


@pytest.mark.parametrize("what, kw", [
    ("FP8 expert_out", dict(expert_out=_t(384, torch.float8_e5m2))),
    ("FP8 out", dict(out=torch.empty(5, 32, dtype=torch.float8_e4m3fn))),
    ("1-D out", dict(out=_t(160, torch.float32))),
    ("row_elems 40", dict(out=torch.empty(5, 40), expert_out=_t(400, torch.bfloat16))),
    ("expert_out of part of a row", dict(expert_out=_t(380, torch.bfloat16))),
    ("int64 route", dict(route=torch.zeros(5, 3, dtype=torch.int64))),
    ("route of other tokens", dict(route=torch.zeros(4, 3, dtype=torch.int32), weights=None)),
    ("top_k 0", dict(route=torch.zeros(5, 0, dtype=torch.int32), weights=None)),
    ("fp16 weights", dict(weights=torch.ones(5, 3, dtype=torch.float16))),
    ("weights of another shape", dict(weights=torch.ones(3, 5))),
    ("nranks * expert_out rows > 2^31 - 1", dict(nranks=8, expert_out=torch.empty(2 ** 28 * 32, dtype=torch.bfloat16, device="meta"))),
    ("out overlaps expert_out", dict(expert_out=_base[:192].view(torch.bfloat16), out=_base[100:260].view(torch.float32).view(5, 32))),
    ("out overlaps route", dict(out=_base[:160].view(torch.float32).view(5, 32), route=_base[150:165].view(5, 3))),
    ("out overlaps weights", dict(out=_base[:160].view(torch.float32).view(5, 32), weights=_base[145:160].view(torch.float32).view(5, 3))),
])
def test_combine_check_raises_value_error(what, kw):
    with pytest.raises((ValueError, RuntimeError)) as e:
        coll.check_expert_combine(**_c(**kw))
    assert e.type is ValueError, (what, e.value)


def test_comm_methods_check_before_calling_the_library():
    """A stand-in communicator with no library handle: the methods must raise ValueError before they reach a C call or allocate."""
    class _Comm(coll.Comm):
        def __init__(self):
            self.nranks, self._h = 2, None
    c = _Comm()
    x, idx, recv = torch.empty(4, 32, dtype=torch.bfloat16), torch.zeros(4, 2, dtype=torch.int32), _t(256, torch.bfloat16)
    with pytest.raises(ValueError):
        c.expert_dispatch(x, idx, 3, recv)                                                   # 3 experts for 2 ranks
    with pytest.raises(ValueError):
        c.expert_dispatch(x, idx.long(), 4, recv)
    with pytest.raises(ValueError):
        c.expert_dispatch(x, idx, 4, _t(256, torch.float16))
    with pytest.raises(ValueError):
        c.expert_combine(recv, idx, torch.ones(4, 3), torch.empty(4, 32))
    with pytest.raises(ValueError):
        c.expert_combine(recv, idx, None, torch.empty(4, 24))


# ------------------------------------------------------------------------------------------------- layout reference
@pytest.mark.parametrize("seed", range(12))
def test_layout_reference_matches_slot_by_slot_placement(seed):
    rng = np.random.default_rng(seed)
    for _ in range(25):
        n = int(rng.choice([1, 2, 3, 4, 8]))
        E, k = n * int(rng.integers(1, 6)), int(rng.integers(1, 6))
        topk = [rng.integers(-2, E + 2, size=(int(rng.integers(0, 12)), k)) for _ in range(n)]
        if rng.random() < 0.3:
            topk[0][:] = E - 1                                                              # every slot of a rank to one expert
        valid = sum(int(((t >= 0) & (t < E)).sum()) for t in topk)
        recv_rows = int(rng.integers(0, valid + 3))                                        # from nothing stored to everything
        a, b = rr.layout(topk, E, recv_rows), rr.brute_force(topk, E, recv_rows)
        for s in range(n):
            assert a.route[s].dtype == np.int32 and a.route[s].shape == np.shape(topk[s])
            assert (a.route[s] == b.route[s]).all() and (a.counts[s] == b.counts[s]).all() and a.dropped[s] == b.dropped[s]
            assert (a.source[s] == b.source[s]).all()
        assert sum(a.dropped) + sum(int(c.sum()) for c in a.counts) == valid


@pytest.mark.parametrize("n, E", [(1, 1024), (2, 1024), (3, 1023), (8, 1024)])
def test_layout_reference_matches_slot_by_slot_placement_at_1024_experts_top_10(n, E):
    """The most experts the dispatch takes and a top_k past the combine's slot batch, at small token counts: a hot expert, the last
    expert, invalid ids, and capacities from nothing to everything."""
    rng = np.random.default_rng(n)
    k = 10
    topk = [rng.integers(-2, E + 2, size=(int(rng.integers(0, 6)), k)) for _ in range(n)]
    topk[0] = np.vstack([topk[0], np.full((2, k), E - 1), rng.integers(0, 3, size=(2, k))])
    valid = sum(int(((t >= 0) & (t < E)).sum()) for t in topk)
    for recv_rows in (0, 1, valid // 2, valid - 1, valid, valid + 3):
        a, b = rr.layout(topk, E, recv_rows), rr.brute_force(topk, E, recv_rows)
        for s in range(n):
            assert (a.route[s] == b.route[s]).all() and (a.counts[s] == b.counts[s]).all() and a.dropped[s] == b.dropped[s]
            assert (a.source[s] == b.source[s]).all()
        assert sum(a.dropped) + sum(int(c.sum()) for c in a.counts) == valid


def _recv_rows_by_row(lay, xs, d, poison):
    want = poison.copy()
    for r, (s, t) in enumerate(lay.source[d]):
        if s >= 0:
            want[r] = xs[s][t]
    return want


def _route_lookup_by_slot(eo, recv_rows):
    n = len(eo)

    def f(col):
        col = np.asarray(col, dtype=np.int64)
        valid = (col >= 0) & (col < n * recv_rows)
        y = np.zeros((col.size, eo[0].shape[1]), dtype=np.float32)
        for i in np.nonzero(valid)[0]:
            y[i] = eo[col[i] // recv_rows][col[i] % recv_rows]
        return valid, y
    return f


@pytest.mark.parametrize("seed", range(6))
def test_recv_rows_and_route_lookup_match_row_by_row(seed):
    """recv_rows_of and route_lookup (numpy fancy indexing) against a row-by-row and a slot-by-slot rendering, on brute-force layouts;
    the lookup also sees every kind of value outside the routes."""
    rng = np.random.default_rng(50 + seed)
    for _ in range(10):
        n = int(rng.choice([1, 2, 3, 4, 8]))
        E, k = n * int(rng.integers(1, 6)), int(rng.integers(1, 11))
        topk = [rng.integers(-2, E + 2, size=(int(rng.integers(0, 12)), k)) for _ in range(n)]
        valid = sum(int(((t >= 0) & (t < E)).sum()) for t in topk)
        recv_rows = int(rng.integers(0, valid + 3))
        lay = rr.brute_force(topk, E, recv_rows)
        xs = [rng.integers(0, 256, size=(t.shape[0], 32), dtype=np.uint8) for t in topk]
        poison = np.full((recv_rows, 32), 0x5A, dtype=np.uint8)
        for d in range(n):
            assert (rr.recv_rows_of(lay, xs, d, poison) == _recv_rows_by_row(lay, xs, d, poison)).all()
        eo = [rng.standard_normal((recv_rows, 16)).astype(np.float32) for _ in range(n)]
        for s in range(n):
            cols = np.concatenate([lay.route[s].reshape(-1), [-1, rr.INT32_MIN, rr.INT32_MAX, n * recv_rows, n * recv_rows - 1, 0]])
            (va, ya), (vb, yb) = rr.route_lookup(eo, recv_rows)(cols), _route_lookup_by_slot(eo, recv_rows)(cols)
            assert (va == vb).all() and (ya.view(np.int32) == yb.view(np.int32)).all()


def test_reference_keeps_up_with_model_shapes():
    """8 ranks x 4096 tokens x top-8 (262,144 slots): the layout, one rank's expected recv and one slot column's lookup each take well
    under a second, so the GPU tests at model shapes spend their time on the GPU."""
    import time
    n, E, k, T = 8, 256, 8, 4096
    topk = rr.routing("zipf", n, E, k, seed=1, tokens=[T] * n, skew=2.0)
    t0 = time.perf_counter()
    lay = rr.layout(topk, E, 40000)
    assert time.perf_counter() - t0 < 1.0
    xs = [np.zeros((T, 64), dtype=np.uint8) for _ in range(n)]
    eo = [np.zeros((40000, 32), dtype=np.float32) for _ in range(n)]
    t0 = time.perf_counter()
    rr.recv_rows_of(lay, xs, 0, np.zeros((40000, 64), dtype=np.uint8))
    rr.route_lookup(eo, 40000)(lay.route[0][:, 0])
    assert time.perf_counter() - t0 < 1.0


def test_layout_reference_by_hand():
    """2 ranks, 4 experts (rank 0 owns 0 and 1): rank 1's rows for expert 1 follow rank 0's; expert 0's rows come first."""
    topk = [np.array([[1, 0], [1, 9]]), np.array([[1, 1], [-1, 2]])]
    lay = rr.layout(topk, 4, 4)
    # rank 0 recv: expert 0 (r0 t0), expert 1 (r0 t0, r0 t1, r1 t0, r1 t0 twice) -> 5 rows, 4 fit
    assert lay.route[0].tolist() == [[1, 0], [2, -1]]
    assert lay.route[1].tolist() == [[3, -1], [-1, 4]]                                     # 4 = rank 1, row 0
    assert lay.counts[0].tolist() == [1, 3] and lay.dropped[0] == 1
    assert lay.counts[1].tolist() == [1, 0] and lay.dropped[1] == 0
    assert lay.source[0].tolist() == [[0, 0], [0, 0], [0, 1], [1, 0]]


# ------------------------------------------------------------------------------------------------- kernels


def test_kernels_are_instantiated_once(coll_lib):
    ks = kernels(coll_lib, "b200coll::k_routed_")
    comb = [k for k in kernels(coll_lib, "b200coll::k_combine_") if "b200coll::RouteMap>" in k]
    for fam in ("k_combine_pull", "k_combine_local"):
        have = [template_args(k) for k in comb if f"::{fam}<" in k]
        assert sorted(have) == sorted((i, o, "b200coll::RouteMap") for i in WIDE for o in WIDE), (fam, have)
    assert sum("::k_routed_push<" in k for k in ks) == 2 and sum("::k_routed_layout(" in k for k in ks) == 1
    assert len(ks) + len(comb) == 21, (ks, comb)


def test_sass_of_every_combine_kernel_has_no_ffma(coll_lib):
    funcs = sass(coll_lib)
    combine = {k: v for k, v in funcs.items() if "k_combine_" in k}
    assert len(combine) == 36, sorted(combine)
    for name, body in combine.items():
        assert re.search(r"\bFMUL\b", body) and re.search(r"\bFADD\b", body), name
        assert "FFMA" not in body, name
        assert "LDGMC" not in body, name
    layout = [v for k, v in funcs.items() if "k_routed_layout" in k]
    assert len(layout) == 1 and "MATCH.ANY" in layout[0]                                  # the warp groups lanes by expert id


def test_ptxas_reports_no_stack_and_no_spills():
    """The compiler's own account, with the library's flags: the new kernels and the combine kernels, old and new, have no stack frame
    and no spill stores or loads, and the combine kernels stay within 128 registers."""
    report, _ = ptxas("dispatch.cu")
    mine = {k: v for k, v in report.items() if "k_routed_" in k}
    assert len(mine) == 3, sorted(mine)
    assert all(v == (0, 0, 0) for v in mine.values()), mine
    report, regs = ptxas("combine.cu")
    comb = {k: v for k, v in report.items() if "k_combine_" in k}
    assert len(comb) == 36, sorted(comb)
    assert all(v == (0, 0, 0) for v in comb.values()), comb
    assert all(r <= 128 for k, r in regs.items() if "combine_" in k), regs


def test_perf_tool_documents_the_route_mode(coll_lib):
    perf = os.path.join(ROOT, "build", "b200coll_perf")
    if not os.path.exists(perf):
        subprocess.run(["make", "-C", os.path.join(ROOT, "coll"), "../build/b200coll_perf"], check=True, capture_output=True)
    out = subprocess.run([perf, "--help"], capture_output=True, text=True, check=True).stdout
    assert "--route E:K" in out and "device-routed expert dispatch" in out


# ------------------------------------------------------------------------------------------------- dispatch plan
@pytest.mark.parametrize("n, top_k, epr", [(1, 1, 4), (2, 2, 4), (4, 3, 2), (8, 8, 32)])
def test_plan_experts_are_the_drawn_routing(n, top_k, epr):
    from container_engine_accelerators_b200.models.workloads import expert_dispatch_plan
    p = expert_dispatch_plan(n, 41, 16, experts_per_rank=epr, top_k=top_k, skew=1.1, seed=n)
    assert len(p.experts) == n
    for s in range(n):
        ids = p.experts[s]
        assert ids.dtype == np.int32 and ids.shape == (41, top_k) and ids.min() >= 0 and ids.max() < n * epr
        assert np.bincount((ids // epr).ravel(), minlength=n).tolist() == p.rows[s].tolist()
        dest = ids.astype(np.int64) // epr                                                 # index puts each slot in its destination's range
        assert ((p.index[s] >= p.send_off[s][dest]) & (p.index[s] < p.send_off[s][dest] + p.rows[s][dest])).all()


def test_plan_is_unchanged_by_the_experts_field():
    """rows, offsets, index and weights are what the plan gave before it kept the expert ids (pinned from the parent revision)."""
    from container_engine_accelerators_b200.models.workloads import expert_dispatch_plan
    p = expert_dispatch_plan(2, 48, 1, 4, 2, 1.2, 3)
    assert p.rows.tolist() == [[33, 63], [32, 64]] and p.send_off.tolist() == [[0, 33], [0, 32]]
    assert p.recv_off.tolist() == [[0, 33], [0, 63]] and p.max_rows == 127
    p = expert_dispatch_plan(3, 17, 16, 2, 3, 0.0, 11)
    assert p.rows.tolist() == [[19, 16, 16], [23, 11, 17], [22, 16, 13]] and p.max_rows == 64
    # order-sensitive checksums of index and of the weights' bits
    assert [int((i.ravel().astype(np.int64) * np.arange(i.size)).sum()) for i in p.index] == [35454, 38613, 37104]
    assert [int((w.view(np.int32).ravel().astype(np.int64) % 100003 * np.arange(w.size)).sum()) for w in p.weights] == [66247686, 68854273, 60004812]
