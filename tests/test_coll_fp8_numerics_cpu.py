"""The FP8-input part of the numerics reference (tests/coll_fp_reference.py), checked without a GPU: the seeded e4m3 / e5m2 data tells
the documented model apart from plausible wrong ones, and the host-path chunk formula gives the chunks the GPU test relies on.

The documented model for FP8 inputs: widen to fp32 (exact: every FP8 value is exact in fp16), sum from +0 in rank order on every
kernel, multiply once by the fp32 scale, round once to nearest even, saturating to the finite range for FP8 outputs."""
import pytest
import torch

from tests import coll_fp_reference as R

E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
FP8 = [E4M3, E5M2]
OUTS = {E4M3: [E4M3, E5M2, torch.bfloat16, torch.float16], E5M2: [E5M2, E4M3, torch.bfloat16, torch.float16]}
COUNT = 40000


def _share(a, b):
    diff = (R._bits(a) != R._bits(b)) & ~(torch.isnan(a.float()) & torch.isnan(b.float()))
    return float(diff.sum()) / a.numel()


@pytest.fixture(scope="module")
def data():
    return {(n, dt): R.gen_inputs(n, COUNT, dt, seed=17 * n + (dt == E5M2), device="cpu") for n in (3, 5, 8) for dt in FP8}


# ------------------------------------------------------------------------------------------------- orders
@pytest.mark.parametrize("n", [3, 5, 8])
def test_e4m3_sums_are_exact_in_any_order(data, n):
    """Every e4m3 value is k * 2^-9 with |k| <= 229376, so a sum of up to 8 of them is exact in fp32 in any order: rank order, the
    reduce-scatter rotation and the two-shot owner order give the same bits. An order mutation on an FP8 kernel can only show with e5m2."""
    xs = data[(n, E4M3)]
    k = torch.stack([x.float() for x in xs]) * 2.0 ** 9
    fin = torch.isfinite(k)
    assert bool((k[fin] == k[fin].round()).all()) and float(k[fin].abs().max()) <= 229376
    rank = list(range(n))
    for out_dt in OUTS[E4M3]:
        for s in (1.0, 0.1):
            doc = R.ref_reduce(xs, rank, s, out_dt)
            for order in [("rotate", r) for r in range(1, n)] + [("owner", n, 16, COUNT)]:
                assert _share(doc, R.ref_reduce(xs, order, s, out_dt)) == 0.0, (n, out_dt, s, order)


@pytest.mark.parametrize("n", [3, 5])
def test_e5m2_orders_disagree(data, n):
    """e5m2 values span about 32 bits, so cancellations against B = 2^12 .. 2^15 and pairs of tiny values make the fp32 sum depend
    on the order: the rotation of a P2P reduce-scatter and the two-shot owner order each differ from rank order on a measured share."""
    xs = data[(n, E5M2)]
    rank = list(range(n))
    for out_dt in OUTS[E5M2]:
        doc = R.ref_reduce(xs, rank, 1.0, out_dt)
        rot = min(_share(doc, R.ref_reduce(xs, ("rotate", r), 1.0, out_dt)) for r in range(1, n))
        own = _share(doc, R.ref_reduce(xs, ("owner", n, 16, COUNT), 1.0, out_dt))
        # measured at n = 3 / 5: rotation 0.038 .. 0.14, owner order 0.026 .. 0.12 (e4m3 outputs lowest: 3 fewer bits to land in)
        assert rot > 0.015 and own > 0.01, (n, out_dt, rot, own)


# ------------------------------------------------------------------------------------------------- wrong models
def _hop16(xs, s, out_dt):
    """Accumulating in fp16: the running sum rounded to fp16 after every rank (what adding in __half2 before widening computes)."""
    acc = torch.zeros(xs[0].numel())
    for x in xs:
        acc = (acc + x.float()).to(torch.float16).float()
    return R.cast(acc * R.f32(s), out_dt)


@pytest.mark.parametrize("n", [3, 5])
@pytest.mark.parametrize("in_dt", FP8)
def test_wrong_models_disagree_with_the_documented_one(data, n, in_dt):
    xs = data[(n, in_dt)]
    rank = list(range(n))
    for out_dt in OUTS[in_dt]:
        fp8_out = out_dt in R.FP8_MAX
        for s in (1.0, 0.1):
            what = f"n={n} {in_dt}->{out_dt} s={s}"
            acc = R.ref_sum(xs, rank) * R.f32(s)
            doc = R.cast(acc, out_dt)
            # measured shares (n = 3 / 5, 40000 elements): fp16 accumulation >= 0.019, rounding toward zero >= 0.11, rounding through
            # fp16 >= 0.0068 (s = 1), no saturation >= 0.066 (s = 1), scale before the sum >= 0.0014
            assert _share(doc, _hop16(xs, s, out_dt)) > 0.01, what
            assert _share(doc, R.cast_rtz(acc, out_dt)) > 0.05, what
            if fp8_out and s == 1.0:
                # rounding through fp16 first: the near-ties lose their nudge and round to even (the ties are placed for scale 1)
                assert _share(doc, R.cast(R.cast(acc, torch.float16).float(), out_dt)) > 0.003, what
                # no saturation: torch's conversion gives NaN (e4m3) or inf (e5m2) past the finite range; e4m3 sums never leave the
                # e5m2 range
                if not (in_dt == E4M3 and out_dt == E5M2):
                    assert _share(doc, acc.to(out_dt)) > 0.02, what
            if s != 1.0:
                pre = R.cast(R.ref_sum([x.float() * R.f32(s) for x in xs], rank), out_dt)
                assert _share(doc, pre) > 0.0005, what


# ------------------------------------------------------------------------------------------------- coverage of the data
def _is_tie(x32, dt):
    m, ex = torch.frexp(x32)
    p = R.MANT[dt]
    scaled = torch.ldexp(m, torch.full_like(ex, p + 1))
    fin = torch.isfinite(x32) & (x32 != 0) & (ex - 1 >= R.EMIN[dt])
    fin = fin & (x32.abs() < (R.FP8_MAX[dt] if dt in R.FP8_MAX else 65504 if dt == torch.float16 else 3e38))
    return fin & (scaled == scaled.round()) & (scaled.remainder(2) == 1)


@pytest.mark.parametrize("in_dt", FP8)
def test_exact_ties_saturation_and_overflow_occur(data, in_dt):
    for n in (3, 5):
        acc = R.ref_sum(data[(n, in_dt)], list(range(n)))
        for out_dt in OUTS[in_dt]:
            ties = int(_is_tie(acc, out_dt).sum())
            assert ties >= 100, (n, in_dt, out_dt, ties)
        fin = torch.isfinite(acc)
        assert int((acc[fin].abs() > R.FP8_MAX[in_dt]).sum()) >= 100, (n, in_dt)          # FP8 outputs saturate
        if in_dt == E5M2:
            assert int((acc[fin].abs() > 65504).sum()) >= 100, n                            # fp16 outputs overflow
            assert int(torch.isinf(R.cast(acc, torch.float16).float()).sum()) >= 100, n
        sub = torch.cat(data[(n, in_dt)]).float().abs()
        assert bool(((sub > 0) & (sub < 2.0 ** R.EMIN[in_dt])).any())                       # input-type subnormals


@pytest.mark.parametrize("in_dt", FP8)
def test_special_bytes_are_where_the_tests_expect_them(in_dt):
    n = 3
    xs = R.gen_inputs(n, 435, in_dt, seed=5, device="cpu")
    b = [x.view(torch.uint8) for x in xs]
    for pos, r, v in R.FP8_SPECIAL[in_dt]:
        assert int(b[r % n][pos]) == v
    for pos, v in zip((41, 43), R.NAN_PAYLOADS[in_dt]):
        assert all(int(t[pos]) == v for t in b) and all(torch.isnan(x[pos].float()).item() for x in xs)
    assert b[1][48:56].tolist() == [0xFF, 0xFF, 0xFF, 0xFF, 0xFF, 0x7F, 0xFF, 0x7F]
    for pos in (7, 434):                                                                    # -0 on every rank, the last one in a scalar tail
        assert all(int(t[pos]) == 0x80 for t in b)
    want = R.ref_reduce(xs, [0, 1, 2], 1.0, in_dt)
    assert int(want.view(torch.uint8)[7]) == 0 and torch.isnan(want[3].float())            # +0 from the accumulator; NaN from one rank
    if in_dt == E5M2:
        assert want[11].float().item() == 57344.0 and want[19].float().item() == -57344.0   # +-inf saturate
        assert torch.isnan(want[27].float())                                                # inf - inf
        assert torch.isinf(R.ref_reduce(xs, [0, 1, 2], 1.0, torch.bfloat16)[11].float())
    # the Lamport identity model changes the sentinel word only
    moved = R.ll_move(xs[1]).view(torch.uint8)
    assert moved[48:52].tolist() == [0xFF, 0x7F, 0xFF, 0x7F] and torch.equal(moved[:48], b[1][:48]) and torch.equal(moved[52:], b[1][52:])


# ------------------------------------------------------------------------------------------------- host path
def test_host_chunks_match_the_regimes():
    """The host path's plan at the counts the GPU test uses (3 ranks): zero-copy while a Lamport kernel reaches the message and it
    is at most 4 MiB, one chunk below 8 MiB, then chunks of total/6 clamped to [4, 16] MiB, rounded up to 1 KiB."""
    n = 3
    bf, f32, f8 = 2, 4, 1
    assert R.host_chunks(100003, bf, bf, n) == ("zero_copy", [100003])                       # 195 KiB: LL
    assert R.host_chunks(600001, bf, bf, n) == ("zero_copy", [600001])                       # 1.14 MiB: LL2 reach (1.5 MiB)
    assert R.host_chunks(100003, f32, bf, n) == ("zero_copy", [100003])
    assert R.host_chunks(300001, f32, bf, n) == ("single", [300001])                         # past LL, and LL2 needs equal sizes
    assert R.host_chunks((3 << 19) + 5, bf, bf, n) == ("single", [(3 << 19) + 5])            # 3 MiB
    assert R.host_chunks((1 << 20) + 3, f8, f8, n) == ("zero_copy", [(1 << 20) + 3])
    assert R.host_chunks((1 << 20) + 3, f8, bf, n) == ("single", [(1 << 20) + 3])
    c, chunks = R.host_chunks((9 << 19) + 13, bf, bf, n)                                      # 9 MiB: 4 + 4 + 1 MiB (+ 26 bytes)
    assert c == "pipelined" and chunks == [2 << 20, 2 << 20, (1 << 19) + 13]
    c, chunks = R.host_chunks((9 << 18) + 13, f32, bf, n)
    assert c == "pipelined" and chunks == [1 << 20, 1 << 20, (1 << 18) + 13]
    c, chunks = R.host_chunks((9 << 20) + 13, f8, f8, n)
    assert c == "pipelined" and chunks == [4 << 20, 4 << 20, (1 << 20) + 13]
    # large messages: total/6 up to the 16 MiB cap, rounded up to whole KiB
    c, chunks = R.host_chunks(30000000, bf, bf, n)
    assert c == "pipelined" and chunks[0] == (60000000 // 6 + 1023) // 1024 * 1024 // 2 and sum(chunks) == 30000000
    assert R.host_chunks(200 << 20, f8, f8, n)[1][0] == 16 << 20
    assert R.host_chunks(4 << 20, f8, f8, 8) == ("zero_copy", [4 << 20])                     # 4 MiB at 8 ranks: LL2 reach and the zero-copy bound
    assert R.host_chunks((4 << 20) + 16, f8, f8, 8)[0] == "single"
