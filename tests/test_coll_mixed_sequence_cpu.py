"""The schedules and size lists of tests/test_coll_mixed_sequence_gpu.py, and the unsigned dtype codes of the generic kernel, without a GPU."""
import numpy as np
import pytest
import torch

from container_engine_accelerators_b200.ops import coll
from tests import coll_fp_reference as R
from tests import test_coll_mixed_sequence_gpu as M


def test_random_schedule_is_deterministic_per_seed():
    for n in (2, 3, 4, 8):
        a, b = M.random_schedule(M.KIND_NAMES, n, 11), M.random_schedule(M.KIND_NAMES, n, 11)
        assert a == b
        assert a != M.random_schedule(M.KIND_NAMES, n, 12)
        steps = [s for w in a for s in w]
        assert len(steps) == 120 and {k for k, _ in steps} <= set(M.KIND_NAMES)
        assert sum(("grow",) in ev for _, ev in steps) == 1
        kinds = {e[0] for _, ev in steps for e in ev}
        assert {"delay", "rewrite"} <= kinds and kinds & {"max_ctas", "shape"}
        assert all(0 <= e[1] < n for _, ev in steps for e in ev if e[0] in ("delay", "rewrite"))
    assert M.pair_schedule(M.KIND_NAMES) == M.pair_schedule(M.KIND_NAMES)


@pytest.mark.parametrize("k", [1, 2, 5, 30, len(M.KIND_NAMES)])
def test_pair_schedule_is_an_eulerian_circuit(k):
    walk = M.eulerian_circuit(k)
    pairs = list(zip(walk, walk[1:]))
    assert len(walk) == k * k + 1 and walk[0] == walk[-1]
    assert sorted(pairs) == [(a, b) for a in range(k) for b in range(k)]


def test_windows_keep_every_pair_adjacent():
    kinds = M.KIND_NAMES
    wins = M.pair_schedule(kinds)
    seq = [kinds[i] for i in M.eulerian_circuit(len(kinds))]
    assert all(len(w) <= M.WINDOW for w in wins)
    assert [k for w in wins for k in w[1:]] == seq[1:] and wins[0][0] == seq[0]
    assert all(a[-1] == b[0] for a, b in zip(wins, wins[1:]))
    inside = {(x, y) for w in wins for x, y in zip(w, w[1:])}
    assert inside == {(a, b) for a in kinds for b in kinds}


@pytest.mark.parametrize("name", list(M.SIZE_CLAIMS))
@pytest.mark.parametrize("n", [2, 3, 4, 8])
@pytest.mark.parametrize("es", [1, 2, 4])
def test_size_lists_straddle_their_thresholds(name, n, es):
    counts_of, claims = M.SIZE_CLAIMS[name]
    nbytes = [c * es for c in counts_of(es, n)]
    for what, bound in claims.items():
        t = bound(n)
        assert min(nbytes) <= t < max(nbytes), (name, what, t, nbytes)
    assert any(c % (16 // es) for c in counts_of(es, n)) == (name == "ll_counts"), "only the all-reduce list has non-vector tails"


@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_special_sizes(n):
    for es in (2, 4):
        big = M.staged_big_count(es, n) * es
        assert big > R.STAGE_HALF_BYTES
        counts = M.host_counts(es, n)
        regimes = [R.host_chunks(c, es, 2, n) for c in counts]
        assert [r for r, _ in regimes] == ["zero_copy", "zero_copy", "pipelined"]
        assert len(set(regimes[-1][1])) == 1, "the pipelined host call cuts into equal chunks"
        assert counts[1] * es == R.LL_ONESHOT_MAX_BYTES


def test_torch_dtype_code_maps_every_generic_type():
    assert coll.torch_dtype_code(torch.uint32) == coll.U32 and coll.torch_dtype_code(torch.uint64) == coll.U64
    for name in M.GENERIC_INT:
        code = coll.torch_dtype_code(getattr(torch, name))
        assert coll.DTYPE_SIZE[code] == torch.empty((), dtype=getattr(torch, name)).element_size()


@pytest.mark.parametrize("dt", [torch.uint32, torch.int64, torch.uint64, torch.int8, torch.int32])
def test_generic_reference_against_python_integers(dt):
    """R.generic_ref on integers is rank 0's value, then ranks 1 .. N-1 in order, wrapped to the type; min / max compare as the type is
    signed or not. Checked against Python's unbounded integers."""
    n, count = 3, 64
    xs = R.int_inputs(n, count, dt, seed=5)
    bits = 8 * np.dtype(R.NP_INT[dt]).itemsize
    signed = np.iinfo(R.NP_INT[dt]).min < 0
    assert signed or any(int(x) >= 2 ** (bits - 1) for a in xs for x in a), "unsigned values with the top bit set"
    for op in (coll.SUM, coll.PROD, coll.MIN, coll.MAX):
        got = R.int_numpy(R.generic_ref([R.int_tensor(x, dt, "cpu") for x in xs], op))
        for i in range(count):
            acc = int(xs[0][i])
            for a in xs[1:]:
                v = int(a[i])
                acc = {coll.SUM: acc + v, coll.PROD: acc * v, coll.MIN: min(acc, v), coll.MAX: max(acc, v)}[op]
            acc &= (1 << bits) - 1
            if signed and acc >= 1 << (bits - 1):
                acc -= 1 << bits
            assert int(got[i]) == acc, (dt, op, i)
