"""FP8-input (e4m3 / e5m2) collectives and the host all-reduce on an H100 (`pytest -m gpu`), bit for bit against the order-exact fp32
reference of tests/coll_fp_reference.py. Virtual ranks share cuda:0 like the rest of the GPU suite.

FP8 inputs are summed in rank order on every P2P kernel, so every reduction here has one order model, [0, 1, ..., N-1]; what each
check asserts about the algorithm is taken from the `algo_calls` delta. The seeded data (cancellations, rounding ties of every output
type, near-ties that rounding through fp16 breaks, saturating sums, fp16 overflow, subnormals, -0, NaN and inf bytes, the Lamport
sentinel word) makes a kernel that sums e5m2 in another order, accumulates in fp16, rounds twice, does not saturate or scales before
the sum fail here. The host all-reduce runs one b200collAllReduce per chunk; its reference is built per chunk with that chunk's
algorithm and order model."""
import pytest
import torch

from tests import coll_fp_reference as R
from tests.coll_gpu_harness import DTYPES, Group, algo_snapshot, arena_inputs, coll_mod, group_fixture, poison, ran, release, torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu

E4, E5 = "float8_e4m3fn", "float8_e5m2"
PAIRS = [(E4, E4), (E4, E5), (E4, "bfloat16"), (E4, "float16"), (E5, E5), (E5, E4), (E5, "bfloat16"), (E5, "float16")]
SUBSET = [(E5, "bfloat16"), (E5, E5), (E4, E5), (E5, E4)]
E = 16                                                          # FP8 elements per 16-byte vector

group = group_fixture(3, arena_mb=160, timeout_ms=60000)


def is_fp8(name):
    return name in (E4, E5)


def ar_pick(coll, n, nvls, algo, nbytes, is_, os_, fp8_in, sym=True, inplace=False):
    """The algorithm b200collAllReduce records: the forced one (or for auto the tuner's pick) when it is feasible, else the first
    feasible of nvls, two-shot, one-shot, LL, LL2; None: staged."""
    if algo == "auto":
        algo = coll.tuner_pick(coll.OP_ALLREDUCE, nbytes, n, nvls)
    feasible = lambda a: {"ll": nbytes <= R.LL_ONESHOT_MAX_BYTES, "ll2": is_ == os_ and nbytes <= R.LL_ONESHOT_MAX_BYTES * n,
                          "oneshot": sym and not inplace, "twoshot": sym, "nvls": nvls and sym and not fp8_in}[a]
    if feasible(algo):
        return algo
    return next((a for a in ("nvls", "twoshot", "oneshot", "ll", "ll2") if feasible(a) and not (a == "nvls" and n == 2)), None)


def check_ar(torch, coll, g, ins, count, in_name, out_name, algo, op, scale, what, outs=None, xs=None):
    """One all-reduce on arena buffers, checked against the rank-order reference; returns the algorithm that ran."""
    comms, n = g.comms, g.n
    in_dt, out_dt = DTYPES[in_name], DTYPES[out_name]
    is_, os_ = R.esize(in_dt), R.esize(out_dt)
    xs = ins if xs is None else xs
    own_outs = outs is None
    outs = [c.empty(count, out_dt) for c in comms] if own_outs else outs
    inplace = outs[0].data_ptr() == ins[0].data_ptr()
    if not inplace:
        poison(outs)
    before = algo_snapshot(comms)
    g.run(lambda r, c, st: (c.set_algo(algo), c.all_reduce(ins[r], outs[r], scale=scale, op=op, stream=st)))
    got = ran(comms, before)
    assert len(got) == 1 and sum(got.values()) == 1, f"{what}: {got}"
    a = next(iter(got))
    want_algo = ar_pick(coll, n, comms[0].nvls, algo, count * is_, is_, os_, True, inplace=inplace)
    assert a == want_algo, f"{what}: asked for {algo}, expected {want_algo}, ran {a}"
    assert a != "nvls" and (a != "ll2" or is_ == os_), f"{what}: ran {a}"
    want = R.ref_reduce(xs, list(range(n)), R.scale_of(coll, op, scale, n), out_dt)
    for r in range(n):
        R.assert_same(outs[r], want, f"{what} rank {r} ran {a}")
    if own_outs:
        release(comms, outs)
    return a


# ------------------------------------------------------------------------------------------------- all-reduce
def bound_counts(n):
    ll = R.LL_ONESHOT_MAX_BYTES
    return [ll, ll + E, ll * n, ll * n + E]


@pytest.mark.parametrize("group", [2, 3, 5, 6, 7, 8], indirect=True)
def test_all_reduce_grid(torch_cuda, coll_mod, group):
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    pairs = PAIRS if n <= 3 else SUBSET
    reds = [(coll.SUM, 1.0), (coll.SUM, 0.1), (coll.AVG, 1.0)]
    algos = ("ll", "ll2", "oneshot", "twoshot", "nvls", "auto")
    seen, auto = set(), {}
    for in_name in (E4, E5):
        outs_for = [o for i, o in pairs if i == in_name]
        if not outs_for:
            continue
        in_dt = DTYPES[in_name]
        counts = [1, 15, 17, 1003, E * (37 * n + 1) + 3] + (bound_counts(n) if n <= 3 or in_name == E5 else [])
        for count in counts:
            ins = arena_inputs(comms, count, in_dt, seed=100 * n + count % 97 + (in_name == E5))
            for out_name in outs_for:
                for algo in algos:
                    for op, scale in (reds if count < 100000 else reds[:2]):
                        a = check_ar(torch, coll, group, ins, count, in_name, out_name, algo, op, scale,
                                     f"all_reduce n={n} count={count} {in_name}->{out_name} {algo} op={op} scale={scale}")
                        seen.add(a)
                        if algo == "auto":
                            auto[(in_name, out_name, count)] = a
            release(comms, ins)
    assert {"ll", "ll2", "oneshot", "twoshot"} <= seen and "nvls" not in seen, seen
    if n <= 3:
        # LL up to 512 KiB per rank, then LL2 up to 512 KiB * N for two FP8 types, then two-shot; FP8 -> 16-bit has no LL2
        for in_name, out_name in pairs:
            got = [auto[(in_name, out_name, k)] for k in bound_counts(n)]
            want = ["ll", "ll2", "ll2", "twoshot"] if is_fp8(out_name) else ["ll", "twoshot", "twoshot", "twoshot"]
            assert got == want, (n, in_name, out_name, got)


@pytest.mark.parametrize("group", [3, 5], indirect=True)
def test_all_reduce_in_place_mixed_sizes(torch_cuda, coll_mod, group):
    """In place, one-shot and two-shot Lamport and two-shot alternating with growing and shrinking ragged counts."""
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    seq = [("ll", 4099, E5), ("ll2", 1003, E4), ("twoshot", E * (37 * n + 1) + 3, E5), ("ll", 9, E4), ("ll2", 70001, E5),
           ("twoshot", 1003, E4), ("ll2", 17, E5), ("ll", 1003, E5), ("ll2", 4099, E4), ("twoshot", 70001, E5)]
    for it, (algo, count, name) in enumerate(seq):
        bufs = arena_inputs(comms, count, DTYPES[name], seed=it)
        xs = [b.clone() for b in bufs]
        check_ar(torch, coll, group, bufs, count, name, name, algo, coll.AVG, 1.0, f"in place #{it} n={n} {algo} {name} count={count}",
                 outs=bufs, xs=xs)
        release(comms, bufs)


@pytest.mark.parametrize("group", [3], indirect=True)
def test_all_reduce_staged_chunks(torch_cuda, coll_mod, group):
    """Buffers outside the arena: one two-shot per staging chunk (16 Mi elements for e5m2 -> bf16, 32 Mi for e4m3 -> e4m3)."""
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    for in_name, out_name, nchunks in ((E5, "bfloat16", 2), (E4, E4, 1)):
        in_dt, out_dt = DTYPES[in_name], DTYPES[out_name]
        chunk = R.staged_chunk(1, R.esize(out_dt), n, "all_reduce")
        assert chunk == (16 << 20 if out_name == "bfloat16" else 32 << 20)
        count = nchunks * chunk + 1003
        xs = R.gen_inputs(n, count, in_dt, seed=5)
        outs = [torch.empty(count, dtype=out_dt, device="cuda") for _ in comms]
        for op, scale in ((coll.SUM, 0.1), (coll.AVG, 1.0)):
            poison(outs)
            before = algo_snapshot(comms)
            group.run(lambda r, c, st: (c.set_algo("auto"), c.all_reduce(xs[r], outs[r], scale=scale, op=op, stream=st)))
            assert ran(comms, before) == {"twoshot": nchunks + 1}
            want = R.ref_reduce(xs, list(range(n)), R.scale_of(coll, op, scale, n), out_dt)
            for r in range(n):
                R.assert_same(outs[r], want, f"staged all_reduce {in_name}->{out_name} count={count} op={op} rank {r}")
        del outs, xs


# ------------------------------------------------------------------------------------------------- reduce-scatter
@pytest.mark.parametrize("group", [2, 3, 5, 7], indirect=True)
def test_reduce_scatter_grid(torch_cuda, coll_mod, group):
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    pairs = PAIRS if n <= 3 else SUBSET
    ll = R.LL_ONESHOT_MAX_BYTES
    for in_name in (E4, E5):
        in_dt = DTYPES[in_name]
        for count in (E, 37 * E, ll, ll + E):
            ins = arena_inputs(comms, count * n, in_dt, seed=count + n + (in_name == E5))
            for i_, out_name in pairs:
                if i_ != in_name:
                    continue
                out_dt = DTYPES[out_name]
                outs = [c.empty(count, out_dt) for c in comms]
                for algo in ("ll", "twoshot", "nvls"):
                    for op, scale in ((coll.SUM, 1.0), (coll.SUM, 0.1), (coll.AVG, 1.0)):
                        poison(outs)
                        before = algo_snapshot(comms)
                        group.run(lambda r, c, st: (c.set_algo(algo), c.reduce_scatter(ins[r], outs[r], scale=scale, op=op, stream=st)))
                        a = next(iter(ran(comms, before)))
                        assert a == ("ll" if algo == "ll" and count <= ll else "twoshot"), (algo, count, a)
                        for r in range(n):
                            xs = [x[r * count:(r + 1) * count] for x in ins]
                            R.assert_same(outs[r], R.ref_reduce(xs, list(range(n)), R.scale_of(coll, op, scale, n), out_dt),
                                          f"reduce_scatter n={n} count={count} {in_name}->{out_name} {algo} ran {a} op={op} scale={scale} rank {r}")
                release(comms, outs)
            release(comms, ins)
    for c in comms:
        c.set_algo("auto")


@pytest.mark.parametrize("group", [3], indirect=True)
def test_reduce_scatter_staged_two_chunks(torch_cuda, coll_mod, group):
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    in_dt, out_dt = DTYPES[E5], torch.bfloat16
    chunk = R.staged_chunk(1, 2, n, "reduce_scatter")
    count = chunk + 37 * E
    xs = R.gen_inputs(n, count * n, in_dt, seed=9)
    outs = [torch.empty(count, dtype=out_dt, device="cuda") for _ in comms]
    poison(outs)
    before = algo_snapshot(comms)
    group.run(lambda r, c, st: (c.set_algo("auto"), c.reduce_scatter(xs[r], outs[r], scale=0.1, op=coll.AVG, stream=st)))
    assert ran(comms, before) == {"twoshot": 2}
    for r in range(n):
        R.assert_same(outs[r], R.ref_reduce([x[r * count:(r + 1) * count] for x in xs], list(range(n)), R.avg_scale(0.1, n), out_dt),
                      f"staged reduce_scatter e5m2->bf16 rank {r}")


# ------------------------------------------------------------------------------------------------- reduce
@pytest.mark.parametrize("group", [3, 5], indirect=True)
def test_reduce_every_root(torch_cuda, coll_mod, group):
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    pairs = PAIRS if n <= 3 else SUBSET
    for in_name, out_name in pairs:
        in_dt, out_dt = DTYPES[in_name], DTYPES[out_name]
        for count in (1003, E * (37 * n + 1) + 3):
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


# ------------------------------------------------------------------------------------------------- data movement
MOVES = [(E4, "bfloat16", 2.0 ** -7), (E4, "bfloat16", 0.1), (E5, "float16", 1.0), (E4, E5, 1.0), (E4, E4, 1.0), (E5, E5, 1.0)]


@pytest.mark.parametrize("group", [3, 5], indirect=True)
def test_data_movement(torch_cuda, coll_mod, group):
    """All-gather, broadcast, all-to-all and all-to-all-v: round((0 + x) * scale) with a cast or a scale; with the identity epilogue a
    bit copy (NaN payloads, -0 and the sentinel words kept) on the barrier kernels, and from 1 MiB on the copy engine."""
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    for in_name, out_name, scale in MOVES:
        in_dt, out_dt = DTYPES[in_name], DTYPES[out_name]
        ident = in_name == out_name and scale == 1.0
        mv = lambda x: R.ref_move(x, scale, out_dt, ident)
        tag = f"n={n} {in_name}->{out_name} scale={scale}"
        big = (1 << 20) + 5 * E                                          # >= 1 MiB per rank: the copy-engine ring for the identity
        for count in (37 * E, big):
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
            for bcount in ((435, 37 * E + 3) if count != big else (count,)):        # 435: the scalar tail holds element 434, a -0
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
        hidden = 8 * E
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
def test_lamport_identity_movement(torch_cuda, coll_mod, group):
    """All-gather and all-to-all forced onto the Lamport path with the identity epilogue store the words as received: every byte
    arrives unchanged (e5m2 +-inf, -0 and NaN payloads included) except a 4-byte word equal to the empty-slot sentinel FF FF FF FF,
    which arrives as FF 7F FF 7F. The same holds for 16- and 32-bit payloads."""
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    for name in (E5, E4, "bfloat16", "float16", "float32"):
        t = DTYPES[name]
        e = R.vec_elems(t)
        for count in (37 * e, 4096 * e):
            src = arena_inputs(comms, count * n, t, seed=count + 3 * n)
            ag = [c.empty(count * n, t) for c in comms]
            a2a = [c.empty(count * n, t) for c in comms]
            poison(ag + a2a)
            before = algo_snapshot(comms)
            # one collective per group.run: with virtual ranks, a second kernel queued behind a spinning one on a rank's stream can hold
            # up another rank's first kernel in the device's shared work queues
            group.run(lambda r, c, st: (c.set_algo("ll"), c.all_gather(src[r][:count], ag[r], stream=st)))
            group.run(lambda r, c, st: c.all_to_all(src[r], a2a[r], stream=st))
            assert ran(comms, before) == {"ll": 2}
            if t == torch.float8_e5m2:                                      # +inf from rank 0 and -inf from rank N-1 stay infinite
                got = [ag[0][p].float().item() for p in (11, count * (n - 1) + 19)]
                assert got == [float("inf"), float("-inf")], f"ll all_gather identity e5m2: +-inf arrived as {got}"
            want_ag = torch.cat([R.ll_move(x[:count]) for x in src])
            for r in range(n):
                R.assert_same(ag[r], want_ag, f"ll all_gather identity {name} count={count} rank {r}", nan_payloads=True)
                want = torch.cat([R.ll_move(src[q][r * count:(r + 1) * count]) for q in range(n)])
                R.assert_same(a2a[r], want, f"ll all_to_all identity {name} count={count} rank {r}", nan_payloads=True)
            if t in R.FP8_MAX:                                               # the model is not vacuous: the sentinel word is in the data
                assert ag[0].view(torch.uint8)[count + 48:count + 56].tolist() == [0xFF, 0x7F, 0xFF, 0x7F] * 2
            release(comms, a2a, ag, src)
    for c in comms:
        c.set_algo("auto")


# ------------------------------------------------------------------------------------------------- generic kernel
@pytest.mark.parametrize("group", [3, 5], indirect=True)
def test_generic_kernel(torch_cuda, coll_mod, group):
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    for name in (E4, E5):
        t = DTYPES[name]
        for op in (coll.MIN, coll.MAX, coll.PROD):
            for count in (1003, E * (37 * n + 1) + 3):
                xs = R.gen_inputs(n, count, t, seed=count + op + n)
                zb = [x.view(torch.uint8) for x in xs]
                for r in range(n):                                                            # +0 against -0 and -0 against +0
                    zb[r][60], zb[r][62] = (0x00, 0x80) if r == 0 else (0x80, 0x00)
                zb[n - 1][64] = 0x7F                                                          # a NaN on the last rank only
                ins = [c.empty(count, t) for c in comms]
                for b, x in zip(ins, xs):
                    b.copy_(x)
                want = R.generic_ref(xs, op)
                if op != coll.PROD:
                    assert int(want.view(torch.uint8)[60]) == 0x00 and int(want.view(torch.uint8)[62]) == 0x80
                what = f"generic n={n} {name} op={op} count={count}"
                outs = [c.empty(count, t) for c in comms]
                poison(outs)
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
                rc = (count // n) // E * E
                rs = [c.empty(rc, t) for c in comms]
                group.run(lambda r, c, st: c.reduce_scatter(ins[r][:rc * n], rs[r], op=op, stream=st))
                for r in range(n):
                    R.assert_same(rs[r], R.generic_ref([x[r * rc:(r + 1) * rc] for x in xs], op), f"{what} reduce_scatter rank {r}")
                release(comms, rs, ins)
            if n == 3:                                                       # staged: buffers outside the arena
                count = 4099
                xs = R.gen_inputs(n, count, t, seed=op)
                outs = [torch.empty(count, dtype=t, device="cuda") for _ in comms]
                poison(outs)
                st0 = [c.stats()["staged_calls"] for c in comms]
                group.run(lambda r, c, st: c.all_reduce(xs[r], outs[r], op=op, stream=st))
                assert [c.stats()["staged_calls"] - s for c, s in zip(comms, st0)] == [1] * n
                for r in range(n):
                    R.assert_same(outs[r], R.generic_ref(xs, op), f"generic staged {name} op={op} rank {r}")


# ------------------------------------------------------------------------------------------------- one rank
def test_one_rank(torch_cuda, coll_mod):
    """nranks == 1: the FP8 identity is a bit copy at every size (the copy engine from 1 MiB when the size is whole 16-byte vectors;
    in place nothing is launched), and e4m3 -> bf16 at scale 0.1 is round((0 + x) * 0.1) in the vector body and the tail alike."""
    torch, coll = torch_cuda, coll_mod
    with Group(torch, coll, 1, arena_mb=96, timeout_ms=60000) as g:
        c = g.comms[0]
        for in_name, out_name, scale in ((E4, E4, 1.0), (E5, E5, 1.0), (E4, "bfloat16", 0.1)):
            in_dt, out_dt = DTYPES[in_name], DTYPES[out_name]
            ident = in_name == out_name
            for count in (1, 17, (1 << 20) + 3, (1 << 20) + 16):
                (x,) = R.gen_inputs(1, count, in_dt, seed=count)
                want = R.ref_move(x, scale, out_dt, ident)
                src = c.empty(count, in_dt)
                src.copy_(x)
                for name, call in (("all_reduce", lambda o: c.all_reduce(src, o, scale=scale)), ("all_gather", lambda o: c.all_gather(src, o, scale=scale)),
                                   ("all_to_all", lambda o: c.all_to_all(src, o, scale=scale)), ("broadcast", lambda o: c.broadcast(src, o, scale=scale)),
                                   ("reduce_scatter", lambda o: c.reduce_scatter(src, o, scale=scale)), ("reduce", lambda o: c.reduce(src, o, scale=scale))):
                    out = c.empty(count, out_dt)
                    poison([out])
                    bulk0 = c.stats()["bulk_launches"]
                    call(out)
                    torch.cuda.synchronize()
                    R.assert_same(out, want, f"one rank {name} {in_name}->{out_name} count={count}", nan_payloads=ident)
                    assert c.stats()["bulk_launches"] - bulk0 == (1 if ident and count == (1 << 20) + 16 else 0), (name, count)
                    c.release(out)
                if ident:
                    k0 = c.stats()["kernel_launches"]
                    c.all_reduce(src)
                    torch.cuda.synchronize()
                    R.assert_same(src, x, f"one rank in-place {in_name} count={count}", nan_payloads=True)
                    assert c.stats()["kernel_launches"] == k0
                c.release(src)
        c.check_async_error()


# ------------------------------------------------------------------------------------------------- grid-stride loops
@pytest.mark.parametrize("group", [3], indirect=True)
def test_one_cta_launch_shape(torch_cuda, coll_mod, group):
    """One CTA of 128 threads: every grid-stride loop runs many passes. The communicators are destroyed afterwards."""
    torch, coll = torch_cuda, coll_mod
    comms, n = group.comms, group.n
    for c in comms:
        c.set_launch_shape("p2p", max_ctas=1, threads=128)
        c.set_launch_shape("ll", 1, 128)
    for out_name in ("bfloat16", E5):
        out_dt = DTYPES[out_name]
        for count in (1003, E * (37 * n + 1) + 3, 100003):
            ins = arena_inputs(comms, count, DTYPES[E5], seed=count)
            for algo in ("ll", "ll2", "oneshot", "twoshot"):
                check_ar(torch, coll, group, ins, count, E5, out_name, algo, coll.SUM, 0.1, f"one CTA all_reduce e5m2->{out_name} {count} {algo}")
            release(comms, ins)
        rcount = 3001 * E
        ins = arena_inputs(comms, rcount * n, DTYPES[E5], seed=3)
        outs = [c.empty(rcount, out_dt) for c in comms]
        for algo in ("ll", "twoshot"):
            poison(outs)
            before = algo_snapshot(comms)
            group.run(lambda r, c, st: (c.set_algo(algo), c.reduce_scatter(ins[r], outs[r], scale=0.1, stream=st)))
            assert ran(comms, before) == {algo: 1}
            for r in range(n):
                R.assert_same(outs[r], R.ref_reduce([x[r * rcount:(r + 1) * rcount] for x in ins], list(range(n)), 0.1, out_dt),
                              f"one CTA reduce_scatter e5m2->{out_name} {algo} rank {r}")
        release(comms, outs, ins)


# ------------------------------------------------------------------------------------------------- host path
HOST_CASES = [("bfloat16", "bfloat16", [100003, 600001, (3 << 19) + 5, (9 << 19) + 13]),
              ("float32", "bfloat16", [100003, 300001, (9 << 18) + 13]),
              (E5, E4, [300001, (1 << 20) + 3, (3 << 20) + 5, (9 << 20) + 13]),
              (E4, "bfloat16", [300001, (1 << 20) + 3, (9 << 20) + 13])]


@pytest.mark.parametrize("group", [3], indirect=True)
def test_all_reduce_host_per_chunk(torch_cuda, coll_mod, group):
    """b200collAllReduceHost at every regime: zero-copy on LL and LL2, one chunk, and the pipeline with a ragged last chunk. Each chunk
    is an all-reduce of its own on arena staging buffers, so each has its own algorithm (predicted here with the tuner and the feasibility
    rules) and, on two-shot with 16- or 32-bit inputs, its own slices: the reference is built chunk by chunk."""
    torch, coll = torch_cuda, coll_mod
    comms = group.comms
    n, nvls = len(comms), comms[0].nvls
    regimes = set()
    for in_name, out_name, counts in HOST_CASES:
        in_dt, out_dt = DTYPES[in_name], DTYPES[out_name]
        is_, os_ = R.esize(in_dt), R.esize(out_dt)
        for count in counts:
            inplace = in_name == out_name == "bfloat16" and count == counts[-1]
            regime, chunks = R.host_chunks(count, is_, os_, n)
            regimes.add(regime)
            xs = R.gen_inputs(n, count, in_dt, seed=count % 1009 + n)
            h_in = [c.host_empty(count, in_dt) for c in comms]
            h_out = h_in if inplace else [c.host_empty(count, out_dt) for c in comms]
            for h, x in zip(h_in, xs):
                h.copy_(x.cpu())
            if not inplace:
                for h in h_out:
                    h.view(torch.uint8).fill_(0x7B)
            sym = regime != "zero_copy"
            algos = [ar_pick(coll, n, nvls, "auto", m * is_, is_, os_, is_fp8(in_name), sym=sym, inplace=inplace and not sym) for m in chunks]
            want_calls = {}
            for a in algos:
                want_calls[a] = want_calls.get(a, 0) + 1
            before = algo_snapshot(comms)
            st0 = [(c.stats()["host_zero_copy"], c.stats()["host_pipelined"]) for c in comms]
            for c in comms:
                c.set_algo("auto")
            group.run(lambda r, c, st: c.all_reduce_host(h_in[r], h_out[r], scale=0.1, stream=st))
            what = f"all_reduce_host n={n} {in_name}->{out_name} count={count} {regime} in_place={inplace}"
            assert ran(comms, before) == want_calls, (what, algos)
            assert [(c.stats()["host_zero_copy"] - z, c.stats()["host_pipelined"] - p) for c, (z, p) in zip(comms, st0)] == \
                [(int(regime == "zero_copy"), int(regime == "pipelined"))] * n, what
            parts, d = [], 0
            for m, a in zip(chunks, algos):
                parts.append(R.ref_reduce([x[d:d + m] for x in xs], R.order_for(a, n, in_dt, m), 0.1, out_dt))
                d += m
            want = torch.cat(parts)
            for r in range(n):
                R.assert_same(h_out[r].cuda(), want, f"{what} chunks={list(zip(chunks, algos))} rank {r}")
            for c, a in zip(comms, h_in):
                c.host_release(a)
            if not inplace:
                for c, b in zip(comms, h_out):
                    c.host_release(b)
    assert regimes == {"zero_copy", "single", "pipelined"}


# ------------------------------------------------------------------------------------------------- several GPUs
def test_multi_gpu_e5m2(torch_cuda, coll_mod):
    """Real peers: e5m2 -> bf16 on two-shot and LL, bit for bit in rank order."""
    torch, coll = torch_cuda, coll_mod
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    with Group(torch, coll, n, devices=list(range(n)), arena_mb=256, timeout_ms=60000) as g:
        comms = g.comms
        t = DTYPES[E5]
        for algo, count in (("twoshot", E * (4099 * n + 1) + 3), ("ll", 100003)):
            xs = R.gen_inputs(n, count, t, seed=n + count % 7)
            ins, outs = [], []
            for r, c in enumerate(comms):
                with torch.cuda.device(r):
                    x = c.empty(count, t); x.copy_(xs[r].to(f"cuda:{r}"))
                    o = c.empty(count, torch.bfloat16); poison([o])
                    ins.append(x); outs.append(o)
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
            assert ran(comms, before) == {algo: 1}
            want = R.ref_reduce(xs, list(range(n)), 1.0, torch.bfloat16)
            for r in range(n):
                R.assert_same(outs[r].to("cuda:0"), want, f"multi-GPU e5m2->bf16 {algo} rank {r}")
            for r, c in enumerate(comms):
                c.release(outs[r]); c.release(ins[r])
