"""fp32 / fp16 / bf16 collectives on an H100 (`pytest -m gpu`), bit for bit against the order-exact fp32 reference of
tests/coll_fp_reference.py. Virtual ranks share cuda:0 like the rest of the GPU suite.

The inputs are seeded and inexact in every order and precision (cancellations, rounding ties of every output type, subnormals, -0,
NaN and inf), so a kernel that sums in another order, accumulates in the input type, rounds twice, scales before the sum or rounds
toward zero fails here. The order model of each check comes from the algorithm the library recorded for the call (the `algo_calls`
delta), not from the one that was requested."""
import warnings

import pytest

from tests import coll_fp_reference as R
from tests.coll_gpu_harness import DTYPES, Group, algo_snapshot, arena_inputs, coll_mod, group_fixture, poison, ran, release, torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu

PAIRS = [("float32", "float32"), ("float32", "bfloat16"), ("float32", "float16"), ("float32", "float8_e4m3fn"), ("float32", "float8_e5m2"),
         ("bfloat16", "bfloat16"), ("bfloat16", "float32"), ("bfloat16", "float8_e4m3fn"), ("bfloat16", "float8_e5m2"),
         ("float16", "float16"), ("float16", "float32"), ("float16", "float8_e4m3fn"), ("float16", "float8_e5m2")]
SUBSET = [("bfloat16", "bfloat16"), ("float32", "bfloat16"), ("float16", "float16"), ("bfloat16", "float32"), ("float32", "float32"),
          ("float16", "float8_e4m3fn")]


group = group_fixture(3, arena_mb=160, timeout_ms=60000)


def ar_expected(coll, comms, algo, count, is_, os_):
    """The algorithm b200collAllReduce runs on arena buffers (not in place): the forced one, or for auto the tuner's pick, where it is
    feasible; otherwise the first feasible fallback."""
    n, nvls = len(comms), comms[0].nvls
    if algo == "auto":
        algo = coll.tuner_pick(coll.OP_ALLREDUCE, count * is_, n, nvls)
    feasible = {"ll": count * is_ <= R.LL_ONESHOT_MAX_BYTES, "ll2": is_ == os_ and count * is_ <= R.LL_ONESHOT_MAX_BYTES * n,
                "oneshot": True, "twoshot": True, "nvls": nvls}[algo]
    return algo if feasible else ("nvls" if nvls and n > 2 else "twoshot")


def check_all_reduce(torch, coll, g, ins, count, in_name, out_name, algo, op, scale, what, outs=None, xs=None):
    """One all-reduce; returns the algorithm that ran. ins are the send buffers, xs their contents (default: ins)."""
    comms, n = g.comms, g.n
    in_dt, out_dt = DTYPES[in_name], DTYPES[out_name]
    is_, os_ = R.esize(in_dt), R.esize(out_dt)
    xs = ins if xs is None else xs
    own_outs = outs is None
    outs = [c.empty(count, out_dt) for c in comms] if own_outs else outs
    if outs[0].data_ptr() != ins[0].data_ptr():
        poison(outs)
    before = algo_snapshot(comms)
    g.run(lambda r, c, st: (c.set_algo(algo), c.all_reduce(ins[r], outs[r], scale=scale, op=op, stream=st)))
    got = ran(comms, before)
    assert len(got) == 1 and sum(got.values()) == 1, f"{what}: {got}"
    a = next(iter(got))
    want_algo = ar_expected(coll, comms, algo, count, is_, os_)
    assert a == want_algo, f"{what}: asked for {algo}, expected {want_algo}, ran {a}"
    want = R.ref_reduce(xs, R.order_for(a, n, in_dt, count), R.scale_of(coll, op, scale, n), out_dt)
    for r in range(n):
        R.assert_same(outs[r], want, f"{what} rank {r} ran {a}")
    if own_outs:
        release(comms, outs)
    return a


# ------------------------------------------------------------------------------------------------- all-reduce
def ar_counts(e, n):
    return [1, e - 1, e + 1, 1003, e * (37 * n + 1) + 3]


def bound_counts(in_dt, n):
    ll = R.LL_ONESHOT_MAX_BYTES // R.esize(in_dt)
    e = R.vec_elems(in_dt)
    return [ll, ll + e, ll * n, ll * n + e]


@pytest.mark.parametrize("group", [2, 3, 5, 8], indirect=True)
def test_all_reduce_grid(torch_cuda, coll_mod, group):
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    pairs = PAIRS if n <= 3 else SUBSET
    reds = [(coll.SUM, 1.0), (coll.SUM, 0.1), (coll.AVG, 1.0)]
    seen = set()
    auto = {}                                                   # (in, out, count) -> what auto ran
    for in_name in ("float32", "bfloat16", "float16"):
        outs_for = [o for i, o in pairs if i == in_name]
        if not outs_for:
            continue
        in_dt = DTYPES[in_name]
        e = R.vec_elems(in_dt)
        counts = ar_counts(e, n) + (bound_counts(in_dt, n) if n <= 3 or in_name == "bfloat16" else [])
        for count in counts:
            ins = arena_inputs(comms, count, in_dt, seed=100 * n + count % 97)
            for out_name in outs_for:
                for algo in ("ll", "ll2", "oneshot", "twoshot", "auto"):
                    for op, scale in (reds if count < 100000 else reds[:2]):
                        a = check_all_reduce(torch, coll, group, ins, count, in_name, out_name, algo, op, scale,
                                             f"all_reduce n={n} count={count} {in_name}->{out_name} {algo} op={op} scale={scale}")
                        seen.add(a)
                        if algo == "auto":
                            auto[(in_name, out_name, count)] = a
            release(comms, ins)
    assert {"ll", "ll2", "oneshot", "twoshot"} <= seen, seen
    if n <= 3:
        # the auto choice changes at the size bounds: LL up to 512 KiB per rank, then LL2 up to 512 KiB * N (same types), then two-shot
        for in_name, out_name in pairs:
            ll = R.LL_ONESHOT_MAX_BYTES // R.esize(DTYPES[in_name])
            e = R.vec_elems(DTYPES[in_name])
            got = [auto[(in_name, out_name, k)] for k in bound_counts(DTYPES[in_name], n)]
            want = ["ll", "ll2", "ll2", "twoshot"] if in_name == out_name else ["ll", "twoshot", "twoshot", "twoshot"]
            assert got == want, (n, in_name, out_name, ll, e, got)


@pytest.mark.parametrize("group", [6, 7], indirect=True)
def test_all_reduce_odd_rank_counts(torch_cuda, coll_mod, group):
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    for in_name, out_name in SUBSET[:3]:
        in_dt = DTYPES[in_name]
        e = R.vec_elems(in_dt)
        for count in (e + 1, 1003, e * (37 * n + 1) + 3):
            ins = arena_inputs(comms, count, in_dt, seed=7 * n + count)
            for algo in ("ll", "ll2", "twoshot"):
                for op, scale in ((coll.SUM, 0.1), (coll.AVG, 1.0)):
                    check_all_reduce(torch, coll, group, ins, count, in_name, out_name, algo, op, scale,
                                     f"all_reduce n={n} count={count} {in_name}->{out_name} {algo} op={op}")
            release(comms, ins)


@pytest.mark.parametrize("group", [3, 5], indirect=True)
def test_all_reduce_in_place_mixed_sizes(torch_cuda, coll_mod, group):
    """In place, one-shot and two-shot Lamport and two-shot alternating with growing and shrinking ragged counts: the stale-slot
    clearing must follow, and every result is still bit-exact."""
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    seq = [("ll", 4099, "bfloat16"), ("ll2", 1003, "bfloat16"), ("twoshot", 8 * (37 * n + 1) + 3, "bfloat16"), ("ll", 9, "float32"),
           ("ll2", 70001, "float16"), ("twoshot", 1003, "float32"), ("ll2", 17, "bfloat16"), ("ll", 1003, "float16"), ("ll2", 4099, "float32")]
    for it, (algo, count, name) in enumerate(seq):
        bufs = arena_inputs(comms, count, DTYPES[name], seed=it)
        xs = [b.clone() for b in bufs]
        check_all_reduce(torch, coll, group, bufs, count, name, name, algo, coll.AVG, 1.0, f"in place #{it} n={n} {algo} {name} count={count}",
                         outs=bufs, xs=xs)
        release(comms, bufs)


@pytest.mark.parametrize("group", [3], indirect=True)
def test_all_reduce_staged_chunks(torch_cuda, coll_mod, group):
    """Buffers outside the arena: the two-shot runs once per staging chunk, the last one ragged, and slices come from each chunk."""
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    for in_name, out_name, nchunks in (("bfloat16", "bfloat16", 1), ("float32", "bfloat16", 2)):
        in_dt, out_dt = DTYPES[in_name], DTYPES[out_name]
        chunk = R.staged_chunk(R.esize(in_dt), R.esize(out_dt), n, "all_reduce")
        assert chunk == (16 << 20 if in_name == "bfloat16" else 8 << 20)
        count = nchunks * chunk + 1003
        xs = R.gen_inputs(n, count, in_dt, seed=5)
        outs = [torch.empty(count, dtype=out_dt, device="cuda") for _ in comms]
        for op, scale in ((coll.SUM, 0.1), (coll.AVG, 1.0)):
            poison(outs)
            before = algo_snapshot(comms)
            st0 = [c.stats()["staged_calls"] for c in comms]
            group.run(lambda r, c, st: (c.set_algo("auto"), c.all_reduce(xs[r], outs[r], scale=scale, op=op, stream=st)))
            assert ran(comms, before) == {"twoshot": nchunks + 1}
            assert [c.stats()["staged_calls"] - s for c, s in zip(comms, st0)] == [1] * n
            want = R.ref_reduce(xs, ("staged", n, R.vec_elems(in_dt), count, chunk), R.scale_of(coll, op, scale, n), out_dt)
            for r in range(n):
                R.assert_same(outs[r], want, f"staged all_reduce {in_name}->{out_name} count={count} op={op} rank {r}")


# ------------------------------------------------------------------------------------------------- reduce-scatter
@pytest.mark.parametrize("group", [2, 3, 5], indirect=True)
def test_reduce_scatter_grid(torch_cuda, coll_mod, group):
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    pairs = PAIRS if n <= 3 else SUBSET
    for in_name in ("float32", "bfloat16", "float16"):
        in_dt = DTYPES[in_name]
        e = R.vec_elems(in_dt)
        ll = R.LL_ONESHOT_MAX_BYTES // R.esize(in_dt)
        for count in (e, 37 * e, ll, ll + e):
            ins = arena_inputs(comms, count * n, in_dt, seed=count + n)
            for i_, out_name in pairs:
                if i_ != in_name:
                    continue
                out_dt = DTYPES[out_name]
                outs = [c.empty(count, out_dt) for c in comms]
                for algo in ("ll", "twoshot"):
                    for op, scale in ((coll.SUM, 1.0), (coll.SUM, 0.1), (coll.AVG, 1.0)):
                        poison(outs)
                        before = algo_snapshot(comms)
                        group.run(lambda r, c, st: (c.set_algo(algo), c.reduce_scatter(ins[r], outs[r], scale=scale, op=op, stream=st)))
                        a = next(iter(ran(comms, before)))
                        assert a == ("ll" if algo == "ll" and count * R.esize(in_dt) <= R.LL_ONESHOT_MAX_BYTES else "twoshot"), (algo, count, a)
                        for r in range(n):
                            xs = [x[r * count:(r + 1) * count] for x in ins]
                            order = list(range(n)) if a == "ll" else ("rotate", r)
                            R.assert_same(outs[r], R.ref_reduce(xs, order, R.scale_of(coll, op, scale, n), out_dt),
                                          f"reduce_scatter n={n} count={count} {in_name}->{out_name} {algo} ran {a} op={op} scale={scale} rank {r}")
                release(comms, outs)
            release(comms, ins)


@pytest.mark.parametrize("group", [3], indirect=True)
def test_reduce_scatter_staged_two_chunks(torch_cuda, coll_mod, group):
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    for in_name, out_name in (("bfloat16", "bfloat16"), ("float32", "float16")):
        in_dt, out_dt = DTYPES[in_name], DTYPES[out_name]
        chunk = R.staged_chunk(R.esize(in_dt), R.esize(out_dt), n, "reduce_scatter")
        count = chunk + 37 * R.vec_elems(in_dt)
        xs = R.gen_inputs(n, count * n, in_dt, seed=9)
        outs = [torch.empty(count, dtype=out_dt, device="cuda") for _ in comms]
        poison(outs)
        before = algo_snapshot(comms)
        group.run(lambda r, c, st: (c.set_algo("auto"), c.reduce_scatter(xs[r], outs[r], scale=0.1, op=coll.AVG, stream=st)))
        assert ran(comms, before) == {"twoshot": 2}
        for r in range(n):
            R.assert_same(outs[r], R.ref_reduce([x[r * count:(r + 1) * count] for x in xs], ("rotate", r), R.avg_scale(0.1, n), out_dt),
                          f"staged reduce_scatter {in_name}->{out_name} rank {r}")


# ------------------------------------------------------------------------------------------------- reduce
@pytest.mark.parametrize("group", [3, 5], indirect=True)
def test_reduce_every_root(torch_cuda, coll_mod, group):
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    pairs = PAIRS if n <= 3 else SUBSET
    for in_name, out_name in pairs:
        in_dt, out_dt = DTYPES[in_name], DTYPES[out_name]
        e = R.vec_elems(in_dt)
        for count in (1003, e * (37 * n + 1) + 3):
            ins = arena_inputs(comms, count, in_dt, seed=count * 3 + n)
            outs = [c.empty(count, out_dt) for c in comms]
            for root in range(n):
                for op, scale in ((coll.SUM, 0.1), (coll.AVG, 1.0)):
                    poison(outs)
                    untouched = outs[0].view(torch.uint8).clone()
                    group.run(lambda r, c, st: c.reduce(ins[r], outs[r], root=root, scale=scale, op=op, stream=st))
                    what = f"reduce n={n} root={root} count={count} {in_name}->{out_name} op={op}"
                    R.assert_same(outs[root], R.ref_reduce(ins, list(range(n)), R.scale_of(coll, op, scale, n), out_dt), what)
                    for r in range(n):
                        if r != root:
                            assert torch.equal(outs[r].view(torch.uint8), untouched), f"{what}: rank {r}'s recv was written"
            release(comms, outs, ins)
    if n == 3:                                                       # staged: two chunks, the second ragged
        count = R.staged_chunk(2, 2, n, "reduce") + 1003
        xs = R.gen_inputs(n, count, torch.bfloat16, seed=4)
        outs = [torch.empty(count, dtype=torch.bfloat16, device="cuda") for _ in comms]
        poison(outs)
        untouched = outs[0].view(torch.uint8).clone()
        group.run(lambda r, c, st: c.reduce(xs[r], outs[r], root=2, scale=0.1, stream=st))
        R.assert_same(outs[2], R.ref_reduce(xs, [0, 1, 2], 0.1, torch.bfloat16), "staged reduce root 2")
        assert torch.equal(outs[0].view(torch.uint8), untouched) and torch.equal(outs[1].view(torch.uint8), untouched)


# ------------------------------------------------------------------------------------------------- data movement
MOVES = [("float32", "bfloat16", 0.1), ("bfloat16", "float32", 0.1), ("float16", "float8_e4m3fn", 0.1),
         ("bfloat16", "bfloat16", 1.0), ("float32", "float32", 1.0), ("float16", "float16", 1.0)]


@pytest.mark.parametrize("group", [3, 5], indirect=True)
def test_data_movement(torch_cuda, coll_mod, group):
    """All-gather, broadcast, all-to-all and all-to-all-v: round((0 + x) * scale) with a cast or a scale, a bit copy (-0 and NaN
    payloads included) with the identity epilogue. The Lamport path rewrites a word equal to its empty-slot marker, so identity copies
    force the barrier-based kernels, as Comm.bit_exact does (test_coll_fp8_numerics_gpu.py checks the Lamport identity model)."""
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    for in_name, out_name, scale in MOVES:
        in_dt, out_dt = DTYPES[in_name], DTYPES[out_name]
        ident = in_name == out_name and scale == 1.0
        e = R.vec_elems(in_dt)
        mv = lambda x: R.ref_move(x, scale, out_dt, ident)
        tag = f"n={n} {in_name}->{out_name} scale={scale}"
        big = ((1 << 20) // R.esize(in_dt)) + 5 * e                       # >= 1 MiB per rank: the copy-engine ring for the identity
        for count in (37 * e, big):
            src = arena_inputs(comms, count * n, in_dt, seed=count + 31 * n)
            for algo in (("twoshot",) if ident else ("auto", "ll", "twoshot")):
                bulk0 = [c.stats()["bulk_launches"] for c in comms]
                ag = [c.empty(count * n, out_dt) for c in comms]
                poison(ag)
                group.run(lambda r, c, st: (c.set_algo(algo), c.all_gather(src[r][:count], ag[r], scale=scale, stream=st)))
                want = torch.cat([mv(x[:count]) for x in src])
                for r in range(n):
                    R.assert_same(ag[r], want, f"all_gather {tag} count={count} {algo} rank {r}", nan_payloads=ident)
                a2a = [c.empty(count * n, out_dt) for c in comms]
                poison(a2a)
                group.run(lambda r, c, st: (c.set_algo(algo), c.all_to_all(src[r], a2a[r], scale=scale, stream=st)))
                for r in range(n):
                    want = torch.cat([mv(src[q][r * count:(r + 1) * count]) for q in range(n)])
                    R.assert_same(a2a[r], want, f"all_to_all {tag} count={count} {algo} rank {r}", nan_payloads=ident)
                moved = [c.stats()["bulk_launches"] - b for c, b in zip(comms, bulk0)]
                assert moved == ([2] * n if ident and count == big else [0] * n), (tag, count, moved)
                release(comms, a2a, ag)
            for c in comms:
                c.set_algo("auto")
            for bcount in ((435, 37 * e + 3) if count != big else (count,)):        # 435: the scalar tail holds element 434, a -0
                for root in range(n):
                    bc = [c.empty(bcount, out_dt) for c in comms]
                    poison(bc)
                    bulk0 = [c.stats()["bulk_launches"] for c in comms]
                    group.run(lambda r, c, st: c.broadcast(src[r][:bcount], bc[r], root=root, scale=scale, stream=st))
                    for r in range(n):
                        R.assert_same(bc[r], mv(src[root][:bcount]), f"broadcast {tag} count={bcount} root={root} rank {r}", nan_payloads=ident)
                    if ident and bcount == big:
                        assert all(c.stats()["bulk_launches"] == b + 1 for c, b in zip(comms, bulk0))
                    release(comms, bc)
            release(comms, src)
        # all-to-all-v: skewed rows of `hidden` elements
        hidden = 8 * e
        rows = [[(3 * s + 5 * d) % 7 for d in range(n)] for s in range(n)]
        cap = max(max(sum(rows[s]) for s in range(n)), max(sum(rows[s][d] for s in range(n)) for d in range(n))) + 1
        send = arena_inputs(comms, cap * hidden, in_dt, seed=77 + n)
        recv = [c.empty(cap * hidden, out_dt) for c in comms]
        poison(recv)
        send_off = [[sum(rows[s][:d]) for d in range(n)] for s in range(n)]
        recv_off = [[sum(rows[x][d] for x in range(s)) for s in range(n)] for d in range(n)]
        group.run(lambda r, c, st: c.all_to_all_v(send[r], recv[r], hidden, rows[r], send_off[r], [recv_off[d][r] for d in range(n)],
                                                                       scale=scale, stream=st))
        for d in range(n):
            for s in range(n):
                got = recv[d][recv_off[d][s] * hidden:(recv_off[d][s] + rows[s][d]) * hidden]
                want = mv(send[s][send_off[s][d] * hidden:(send_off[s][d] + rows[s][d]) * hidden])
                R.assert_same(got, want, f"all_to_all_v {tag} {s}->{d}", nan_payloads=ident)
        release(comms, recv, send)


@pytest.mark.parametrize("group", [3], indirect=True)
def test_data_movement_staged(torch_cuda, coll_mod, group):
    torch = torch_cuda
    comms, n = group.comms, group.n
    for in_name, out_name, scale in (MOVES[0], MOVES[3]):
        in_dt, out_dt = DTYPES[in_name], DTYPES[out_name]
        ident = scale == 1.0
        mv = lambda x: R.ref_move(x, scale, out_dt, ident)
        e = R.vec_elems(in_dt)
        count = R.staged_chunk(R.esize(in_dt), R.esize(out_dt), n, "all_gather") + 5 * e
        xs = R.gen_inputs(n, count * n, in_dt, seed=21)
        st0 = [c.stats()["staged_calls"] for c in comms]
        ag = [torch.empty(count * n, dtype=out_dt, device="cuda") for _ in comms]
        group.run(lambda r, c, st: (c.set_algo("twoshot"), c.all_gather(xs[r][:count], ag[r], scale=scale, stream=st)))
        for r in range(n):
            R.assert_same(ag[r], torch.cat([mv(x[:count]) for x in xs]), f"staged all_gather {in_name}->{out_name} rank {r}", nan_payloads=ident)
        del ag
        a2a = [torch.empty(count * n, dtype=out_dt, device="cuda") for _ in comms]
        group.run(lambda r, c, st: c.all_to_all(xs[r], a2a[r], scale=scale, stream=st))
        for r in range(n):
            R.assert_same(a2a[r], torch.cat([mv(xs[q][r * count:(r + 1) * count]) for q in range(n)]), f"staged all_to_all {in_name}->{out_name} rank {r}",
                          nan_payloads=ident)
        del a2a
        bcount = R.staged_chunk(R.esize(in_dt), R.esize(out_dt), n, "broadcast") + 1003
        bc = [torch.empty(bcount, dtype=out_dt, device="cuda") for _ in comms]
        src = [x.repeat(2)[:bcount] if x.numel() < bcount else x[:bcount] for x in xs]
        group.run(lambda r, c, st: c.broadcast(src[r], bc[r], root=1, scale=scale, stream=st))
        for r in range(n):
            R.assert_same(bc[r], mv(src[1]), f"staged broadcast {in_name}->{out_name} rank {r}", nan_payloads=ident)
        del bc
        assert [c.stats()["staged_calls"] - s for c, s in zip(comms, st0)] == [3] * n
        for c in comms:
            c.set_algo("auto")


# ------------------------------------------------------------------------------------------------- grid-stride loops
@pytest.mark.parametrize("group", [3], indirect=True)
@pytest.mark.parametrize("shape", ["one_cta", "two_ctas"])
def test_grid_stride_many_passes(torch_cuda, coll_mod, group, shape):
    """One CTA of 128 threads (or a cap of two CTAs): every grid-stride loop runs many passes and ends on a partial unroll. The
    communicators are destroyed afterwards, so the launch shapes do not leak into other tests."""
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    for c in comms:
        if shape == "one_cta":
            c.set_launch_shape("p2p", max_ctas=1, threads=128)
            c.set_launch_shape("ll", 1, 128)
        else:
            c.set_max_ctas(2)
    for in_name, out_name in (("bfloat16", "bfloat16"), ("float32", "bfloat16"), ("float16", "float32")):
        in_dt, out_dt = DTYPES[in_name], DTYPES[out_name]
        e = R.vec_elems(in_dt)
        for count in (1003, e * (37 * n + 1) + 3, 100003):
            ins = arena_inputs(comms, count, in_dt, seed=count)
            for algo in ("ll", "ll2", "oneshot", "twoshot"):
                check_all_reduce(torch, coll, group, ins, count, in_name, out_name, algo, coll.SUM, 0.1, f"{shape} all_reduce {in_name}->{out_name} {count} {algo}")
            red = [c.empty(count, out_dt) for c in comms]
            group.run(lambda r, c, st: c.reduce(ins[r], red[r], root=1, scale=0.1, stream=st))
            R.assert_same(red[1], R.ref_reduce(ins, list(range(n)), 0.1, out_dt), f"{shape} reduce {in_name}->{out_name} {count}")
            bc = [c.empty(count, out_dt) for c in comms]
            group.run(lambda r, c, st: c.broadcast(ins[r], bc[r], root=2, scale=0.1, stream=st))
            for r in range(n):
                R.assert_same(bc[r], R.ref_move(ins[2], 0.1, out_dt, False), f"{shape} broadcast {in_name}->{out_name} {count} rank {r}")
            release(comms, bc, red, ins)
        rcount = 3001 * e
        ins = arena_inputs(comms, rcount * n, in_dt, seed=3)
        outs = [c.empty(rcount, out_dt) for c in comms]
        for algo in ("ll", "twoshot"):
            before = algo_snapshot(comms)
            group.run(lambda r, c, st: (c.set_algo(algo), c.reduce_scatter(ins[r], outs[r], scale=0.1, stream=st)))
            a = next(iter(ran(comms, before)))
            for r in range(n):
                xs = [x[r * rcount:(r + 1) * rcount] for x in ins]
                R.assert_same(outs[r], R.ref_reduce(xs, list(range(n)) if a == "ll" else ("rotate", r), 0.1, out_dt), f"{shape} reduce_scatter {algo} rank {r}")
            ag = [c.empty(rcount * n, out_dt) for c in comms]
            group.run(lambda r, c, st: (c.set_algo(algo), c.all_gather(ins[r][:rcount], ag[r], scale=0.1, stream=st)))
            for r in range(n):
                R.assert_same(ag[r], torch.cat([R.ref_move(x[:rcount], 0.1, out_dt, False) for x in ins]), f"{shape} all_gather {algo} rank {r}")
            release(comms, ag)
        release(comms, outs, ins)


# ------------------------------------------------------------------------------------------------- one rank
def test_one_rank_all_ops(torch_cuda, coll_mod):
    """nranks == 1: every op is the copy epilogue. The identity is a bit copy at every size (-0 and NaN payloads kept; in place it is
    a no-op; from 1 MiB the copy engine moves it); a cast or a scale is round((0 + x) * scale) in the vector body and the tail alike."""
    torch, coll = torch_cuda, coll_mod
    with Group(torch, coll, 1, arena_mb=96, timeout_ms=60000) as g:
        c = g.comms[0]
        cases = [("bfloat16", "bfloat16", 1.0), ("float32", "float32", 1.0), ("float16", "float16", 1.0), ("bfloat16", "float32", 1.0),
                 ("float32", "bfloat16", 1.0), ("float16", "float16", 0.1), ("float32", "float8_e4m3fn", 0.1)]
        for in_name, out_name, scale in cases:
            in_dt, out_dt = DTYPES[in_name], DTYPES[out_name]
            ident = in_name == out_name and scale == 1.0
            e = R.vec_elems(in_dt)
            for count in (1, e + 3, (1 << 20) + 3, (1 << 20) + e):
                (x,) = R.gen_inputs(1, count, in_dt, seed=count)
                want = R.ref_move(x, scale, out_dt, ident)
                for where in ("arena", "plain"):
                    src = c.empty(count, in_dt) if where == "arena" else torch.empty(count, dtype=in_dt, device="cuda")
                    src.copy_(x)
                    calls = {
                        "all_reduce": lambda o: c.all_reduce(src, o, scale=scale),
                        "all_gather": lambda o: c.all_gather(src, o, scale=scale),
                        "reduce_scatter": lambda o: c.reduce_scatter(src, o, scale=scale),
                        "all_to_all": lambda o: c.all_to_all(src, o, scale=scale),
                        "broadcast": lambda o: c.broadcast(src, o, scale=scale),
                        "reduce": lambda o: c.reduce(src, o, scale=scale),
                    }
                    for name, call in calls.items():
                        out = c.empty(count, out_dt) if where == "arena" else torch.empty(count, dtype=out_dt, device="cuda")
                        poison([out])
                        bulk0 = c.stats()["bulk_launches"]
                        call(out)
                        torch.cuda.synchronize()
                        R.assert_same(out, want, f"one rank {name} {where} {in_name}->{out_name} scale={scale} count={count}", nan_payloads=ident)
                        big = ident and count * R.esize(in_dt) >= (1 << 20) and count * R.esize(in_dt) % 16 == 0
                        assert c.stats()["bulk_launches"] - bulk0 == (1 if big else 0), (name, count)
                        if where == "arena":
                            c.release(out)
                    if ident:                                             # in place: returns without touching the buffer
                        k0 = c.stats()["kernel_launches"]
                        c.all_reduce(src)
                        torch.cuda.synchronize()
                        R.assert_same(src, x, f"one rank in-place {in_name} count={count}", nan_payloads=True)
                        assert c.stats()["kernel_launches"] == k0
                    if where == "arena":
                        c.release(src)
        c.check_async_error()


# ------------------------------------------------------------------------------------------------- generic kernel
@pytest.mark.parametrize("group", [3, 5], indirect=True)
def test_generic_kernel(torch_cuda, coll_mod, group):
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    g = torch.Generator(device="cuda").manual_seed(n)
    cases = [(name, op) for name in ("float32", "float16", "bfloat16") for op in (coll.MIN, coll.MAX, coll.PROD)]
    cases += [("int8", coll.SUM), ("uint8", coll.SUM), ("int32", coll.SUM), ("float64", coll.SUM), ("int32", coll.MIN)]
    # unsigned against signed compares (values >= 2^31 and >= 2^63, INT64_MIN and INT64_MAX) and wrapping sums and products
    cases += [(name, op) for name in ("uint32", "int64", "uint64") for op in (coll.SUM, coll.PROD, coll.MIN, coll.MAX)]
    cases += [("int8", coll.PROD), ("int32", coll.PROD)]
    for name, op in cases:
        t = DTYPES[name]
        e = 16 // R.esize(t)
        for count in (1003, e * (37 * n + 1) + 3):
            if t.is_floating_point and t != torch.float64:
                xs = R.gen_inputs(n, count, t, seed=count + op)
                if op == coll.PROD:                                       # keep products finite and inexact
                    xs = [(x.float().abs().clamp(0.5, 2.0) * torch.where(x.float() < 0, -1.0, 1.0)).to(t) for x in xs]
                    for x in xs[1:]:
                        x[3] = float("nan")
            elif t == torch.float64:
                xs = [torch.randn(count, generator=g, device="cuda", dtype=torch.float64) * 2.0 ** torch.randint(-30, 30, (count,), generator=g, device="cuda")
                      for _ in range(n)]
            else:
                xs = [R.int_tensor(x, t) for x in R.int_inputs(n, count, t, seed=count + 10 * op + n)]
            ins = [c.empty(count, t) for c in comms]
            for b, x in zip(ins, xs):
                b.copy_(x)
            want = R.generic_ref(ins, op)
            what = f"generic n={n} {name} op={op} count={count}"
            outs = [c.empty(count, t) for c in comms]
            gen0 = [c.stats()["generic_launches"] for c in comms]
            group.run(lambda r, c, st: c.all_reduce(ins[r], outs[r], op=op, stream=st))
            for r in range(n):
                R.assert_same(outs[r], want, f"{what} all_reduce rank {r}")
            assert all(c.stats()["generic_launches"] == g0 + 1 for c, g0 in zip(comms, gen0))
            for root in (0, n - 1):
                poison(outs)
                untouched = outs[0].view(torch.uint8).clone()
                group.run(lambda r, c, st: c.reduce(ins[r], outs[r], root=root, op=op, stream=st))
                R.assert_same(outs[root], want, f"{what} reduce root {root}")
                assert all(torch.equal(outs[r].view(torch.uint8), untouched) for r in range(n) if r != root)
            release(comms, outs)
            rc = (count // n) // e * e
            rs = [c.empty(rc, t) for c in comms]
            group.run(lambda r, c, st: c.reduce_scatter(ins[r][:rc * n], rs[r], op=op, stream=st))
            for r in range(n):
                R.assert_same(rs[r], want[r * rc:(r + 1) * rc], f"{what} reduce_scatter rank {r}")
            # a reduce-scatter block must be whole 16-byte vectors (the generic kernel has no per-block tail): refused before anything
            # is launched or counted, so one rank may try it alone
            st0 = comms[0].stats()
            with pytest.raises(coll.B200CollError) as err:
                comms[0].reduce_scatter(ins[0], ins[0][:rc + 1], op=op)
            assert err.value.code == coll.INVALID_ARGUMENT and comms[0].stats() == st0
            release(comms, rs, ins)


# ------------------------------------------------------------------------------------------------- several GPUs
def test_multi_gpu_two_shot_and_nvls(torch_cuda, coll_mod):
    """Real peers: two-shot bit for bit; NVLS (the switch adds, in its own order) within one output ulp around an fp64 reference plus
    N * max|x| * 2^-22, except the scalar tail, which rank 0 sums in rank order and is bit for bit."""
    torch, coll = torch_cuda, coll_mod
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    with Group(torch, coll, n, devices=list(range(n)), arena_mb=256, timeout_ms=60000) as g:
        comms = g.comms
        for name in ("bfloat16", "float32"):
            t = DTYPES[name]
            e = R.vec_elems(t)
            count = e * (4099 * n + 1) + 3
            xs = R.gen_inputs(n, count, t, seed=n)
            ins, outs = [], []
            for r, c in enumerate(comms):
                with torch.cuda.device(r):
                    x = c.empty(count, t); x.copy_(xs[r].to(f"cuda:{r}"))
                    ins.append(x); outs.append(c.empty(count, t))
            for r in range(n):
                torch.cuda.synchronize(r)
            for algo in ("twoshot", "nvls"):
                for r, o in enumerate(outs):
                    with torch.cuda.device(r):
                        poison([o])
                for r in range(n):
                    torch.cuda.synchronize(r)
                before = algo_snapshot(comms)
                for r, c in enumerate(comms):
                    with torch.cuda.device(r):
                        c.set_algo(algo)
                        c.all_reduce(ins[r], outs[r])
                for r in range(n):
                    torch.cuda.synchronize(r)
                for c in comms:
                    c.check_async_error()
                a = next(iter(ran(comms, before)))
                assert a == ("nvls" if algo == "nvls" and comms[0].nvls else "twoshot"), (algo, a, comms[0].nvls)
                if algo == "nvls" and not comms[0].nvls:
                    warnings.warn(f"{n} GPUs without multicast: forced NVLS ran two-shot, the NVLS tolerance check did not run")
                tail = count // e * e
                for r in range(n):
                    got = outs[r].to("cuda:0")
                    what = f"multi-GPU {name} {algo} ran {a} rank {r}"
                    if a == "twoshot":
                        R.assert_same(got, R.ref_reduce(xs, ("owner", n, e, count), 1.0, t), what)
                        continue
                    R.assert_same(got[tail:], R.ref_reduce([x[tail:] for x in xs], list(range(n)), 1.0, t), what + " tail")
                    x64 = torch.stack([x[:tail].double() for x in xs])
                    ref = x64.sum(0)
                    fin = torch.isfinite(ref)
                    ulp = (ref.abs().clamp_min(2.0 ** -126) * 2.0 ** (1 - R.MANT[t]))
                    tol = ulp + n * x64.abs().max(0).values * 2.0 ** -22
                    err = (got[:tail].double() - ref).abs()
                    assert bool((err[fin] <= tol[fin]).all()), f"{what}: max error {float((err[fin] - tol[fin]).max())} over tolerance"
