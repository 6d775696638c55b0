"""The fp32 / fp16 / bf16 numerics reference (tests/coll_fp_reference.py), checked without a GPU: its index formulas agree with a
line-by-line copy of the kernel and host formulas, and its seeded data tells the documented model apart from plausible wrong ones.
Without the second part a passing GPU test would say nothing."""
import pytest
import torch

from tests import coll_fp_reference as R

IN_TYPES = [torch.float32, torch.bfloat16, torch.float16]
NARROW_OUT = [torch.bfloat16, torch.float16, torch.float8_e4m3fn, torch.float8_e5m2]


# ------------------------------------------------------------------------------------------------- index formulas
def _owner_by_kernel(count, n, e):
    """k_ar_twoshot + ar_tail_rank0, one thread per vector: rank r reduces v0 <= v < v1 starting at itself; rank 0 sums the tail."""
    out = [None] * count
    nvec = count // e
    for rank in range(n):
        v0, v1 = nvec * rank // n, nvec * (rank + 1) // n
        for v in range(v0, v1):
            for i in range(e):
                out[v * e + i] = rank
    for el in range(nvec * e, count):
        out[el] = 0
    return out


@pytest.mark.parametrize("n", [2, 3, 5, 6, 7, 8])
def test_owner_map_matches_the_kernel_slices(n):
    for e in (4, 8):
        for count in [1, e - 1, e, e + 1, n * e - 1, n * e, n * e + 3, (n - 1) * e + 2, 1003, e * (37 * n + 1) + 3, 4099]:
            want = _owner_by_kernel(count, n, e)
            assert R.owner_map(count, n, e).tolist() == want, (count, n, e)
            nvec = count // e
            assert sum(R.slice_bounds(nvec, n, o)[1] - R.slice_bounds(nvec, n, o)[0] for o in range(n)) == nvec


def test_staged_chunk_formulas():
    h = 32 << 20
    for n in (2, 3, 5, 8):
        for is_, os_ in ((4, 4), (4, 2), (2, 2), (2, 4), (2, 1), (4, 1)):
            assert R.staged_chunk(is_, os_, n, "all_reduce") == min(h // is_, h // os_) // 64 * 64
            assert R.staged_chunk(is_, os_, n, "broadcast") == R.staged_chunk(is_, os_, n, "reduce") == min(h // is_, h // os_) // 64 * 64
            assert R.staged_chunk(is_, os_, n, "reduce_scatter") == (h // is_ // n) // 64 * 64
            assert R.staged_chunk(is_, os_, n, "all_gather") == R.staged_chunk(is_, os_, n, "all_to_all") == (h // os_ // n) // 64 * 64
    assert R.staged_chunk(2, 2, 2, "all_reduce") == 16 << 20 and R.staged_chunk(4, 2, 2, "all_reduce") == 8 << 20
    # the staged all-reduce slices each chunk on its own: chunk + 1003 ends with a short chunk whose slices are short too
    chunk, e, n = 1024, 8, 3
    m = R.staged_owner_map(chunk + 1003, n, e, chunk)
    assert m[:chunk].tolist() == _owner_by_kernel(chunk, n, e) and m[chunk:].tolist() == _owner_by_kernel(1003, n, e)


def test_orders_and_avg_scale():
    xs = [torch.tensor([2.0 ** 24]), torch.tensor([1.0]), torch.tensor([1.0])]
    assert R.ref_sum(xs, [0, 1, 2]).item() == 2.0 ** 24               # each 1 is lost against 2^24
    assert R.ref_sum(xs, ("rotate", 1)).item() == 2.0 ** 24 + 2          # 1 + 1 first, then 2^24
    assert R.ref_sum(xs, ("owner", 3, 1, 1)).item() == 2.0 ** 24         # one element: the tail, rank order
    assert R.ref_sum([torch.tensor([-0.0])], [0]).item() == 0.0 and not torch.signbit(R.ref_sum([torch.tensor([-0.0])], [0])).item()
    assert R.avg_scale(1.0, 3) == float(torch.tensor(1.0) / torch.tensor(3.0))
    assert R.avg_scale(0.1, 5) == float(torch.tensor(0.1) * (torch.tensor(1.0) / torch.tensor(5.0)))
    assert R.cast(torch.tensor([500.0, float("inf"), float("nan")]), torch.float8_e4m3fn).float()[:2].tolist() == [448.0, 448.0]
    assert R.cast_rtz(torch.tensor([1.0 + 2.0 ** -8 + 2.0 ** -20, -(1.0 + 2.0 ** -8 + 2.0 ** -20)]), torch.bfloat16).float().tolist() == [1.0, -1.0]


# ------------------------------------------------------------------------------------------------- the data has teeth
def _share(a, b):
    diff = (R._bits(a) != R._bits(b)) & ~(torch.isnan(a.float()) & torch.isnan(b.float()))
    return float(diff.sum()) / a.numel()


def _hop(xs, in_dt, s, out_dt):
    acc = torch.zeros(xs[0].numel())
    for x in xs:
        acc = (acc + x.float()).to(in_dt).float()                          # the running sum rounded to the input type each hop
    return R.cast(acc * R.f32(s), out_dt)


@pytest.fixture(scope="module")
def data():
    return {(n, dt): R.gen_inputs(n, 40000, dt, seed=11 * n + R.esize(dt), device="cpu") for n in (3, 5) for dt in IN_TYPES}


@pytest.mark.parametrize("n", [3, 5])
@pytest.mark.parametrize("in_dt", IN_TYPES)
def test_wrong_models_disagree_with_the_documented_one(data, n, in_dt):
    xs = data[(n, in_dt)]
    count, e = xs[0].numel(), R.vec_elems(in_dt)
    rank = list(range(n))
    for out_dt in [in_dt, torch.float32, *[t for t in NARROW_OUT if t != in_dt]]:
        for s in (1.0, 0.1):
            doc = R.ref_reduce(xs, rank, s, out_dt)
            what = f"n={n} {in_dt}->{out_dt} s={s}"
            # owner-first where rank order is documented, and the other way round; the P2P reduce-scatter rotation
            assert _share(doc, R.ref_reduce(xs, ("owner", n, e, count), s, out_dt)) > 0.02, what
            assert _share(doc, R.ref_reduce(xs, ("rotate", 1), s, out_dt)) > 0.03, what
            if out_dt != torch.float32:                                     # rounding toward zero instead of to nearest even
                assert _share(doc, R.cast_rtz(R.ref_sum(xs, rank) * R.f32(s), out_dt)) > 0.2, what
            if s != 1.0:                                                    # the scale applied to each input before the sum
                pre = R.cast(R.ref_sum([x.float() * R.f32(s) for x in xs], rank), out_dt)
                assert _share(doc, pre) > (0.3 if out_dt == torch.float32 else 0.002), what
            if in_dt != torch.float32:
                # accumulating in the input type (fp32 inputs: the accumulator is the input type, there is nothing to tell apart)
                assert _share(doc, _hop(xs, in_dt, s, out_dt)) > (0.5 if out_dt == torch.float32 else 0.005), what
                if out_dt != in_dt or s != 1.0:                             # rounding twice: to the input type, then to the output type
                    twice = R.cast(R.cast(R.ref_sum(xs, rank), in_dt).float() * R.f32(s), out_dt)
                    assert _share(doc, twice) > (0.5 if out_dt == torch.float32 else 0.001), what


def _is_tie(x32, dt):
    """x is exactly halfway between two neighbours of dt (normal range)."""
    m, ex = torch.frexp(x32)
    p = R.MANT[dt]
    scaled = torch.ldexp(m, torch.full_like(ex, p + 1))
    fin = torch.isfinite(x32) & (x32 != 0) & (ex - 1 >= R.EMIN[dt])
    if dt in R.FP8_MAX:
        fin = fin & (x32.abs() < R.FP8_MAX[dt])
    elif dt == torch.float16:
        fin = fin & (x32.abs() < 65504)
    return fin & (scaled == scaled.round()) & (scaled.remainder(2) == 1)


@pytest.mark.parametrize("in_dt", IN_TYPES)
def test_exact_ties_occur_for_every_narrow_output(data, in_dt):
    for n in (3, 5):
        acc = R.ref_sum(data[(n, in_dt)], list(range(n)))
        for out_dt in NARROW_OUT:
            ties = int(_is_tie(acc, out_dt).sum())
            assert ties >= 100, (n, in_dt, out_dt, ties)
            assert _is_tie(torch.tensor([1.0 + 2.0 ** -R.MANT[out_dt]]), out_dt).item()


def test_special_values_are_where_the_tests_expect_them():
    for dt in IN_TYPES:
        xs = R.gen_inputs(3, 200, dt, seed=5, device="cpu")
        assert torch.isnan(xs[1][3].float()) and xs[0][11].float().item() == float("inf") and xs[2][19].float().item() == float("-inf")
        assert all(torch.signbit(x[7]).item() and x[7].float().item() == 0.0 for x in xs)           # -0 on every rank
        want = R.ref_reduce(xs, [0, 1, 2], 1.0, dt)
        assert not torch.signbit(want[7]).item() and torch.isnan(want[27].float())                  # +0 from the accumulator; inf - inf
        sub = torch.cat(xs).float().abs()
        assert bool(((sub > 0) & (sub < 2.0 ** R.EMIN[dt])).any())                                  # input-type subnormals
    h = R.gen_inputs(3, 4000, torch.float16, seed=5, device="cpu")
    assert bool(torch.isinf(R.ref_reduce(h, [0, 1, 2], 1.0, torch.float16).float()).sum() > 20)       # fp16 sums that overflow
