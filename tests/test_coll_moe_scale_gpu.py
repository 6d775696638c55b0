"""Expert dispatch and combine at the shapes MoE models route (`pytest -m gpu`), virtual ranks sharing cuda:0 unless said otherwise.

The other MoE modules check every entry point bit for bit at small shapes. These tests reach the code paths that only run at model
sizes:
- the layout kernel's per-warp carry (a warp walks its 1/32 of the slots 32 at a time; 4096 tokens x top-8 is 32 passes per warp);
- more than 256 experts, up to the 1024 limit, where every thread of the layout CTA owns an expert;
- top_k past the combine's slot batch (8 slots for 2-byte and FP8 inputs, 4 for fp32), with dropped slots in every batch;
- capacity cut exactly at the load, one row below it, and inside a hot expert;
- rows of 7168 bf16 elements, and a recv past 4 GiB, where byte offsets need 64 bits.

References: tests/coll_routed_reference.layout for the layout, tests/coll_combine_reference.combine for the combines and
tests/coll_quant_reference.quantize for the FP8 rows. Past 4 GiB the expected values are built on the device with torch, in the same
order of operations."""
import numpy as np
import pytest

from tests import coll_combine_reference as cr
from tests import coll_quant_reference as qr
from tests import coll_routed_reference as rr
from tests import test_coll_expert_combine_quantized_gpu as cq
from tests import test_coll_expert_routed_gpu as eg
from tests.coll_fp_reference import assert_same
from tests.coll_gpu_harness import DTYPES, Group, coll_mod, release, torch_cuda  # noqa: F401
from tests.coll_routed_reference import INT32_MIN, route_lookup, routing

pytestmark = pytest.mark.gpu
POISON = 0x5A

# (model, experts, top_k, tokens per rank, row dtype, row elements, the FP8 dispatch's wire and block)
SHAPES = [("DeepSeek-V3", 256, 8, 4096, "bf16", 32, "e4m3", 32),
          ("Kimi K2", 384, 8, 2048, "f16", 64, "e5m2", 64),
          ("Qwen3-Next", 512, 10, 2048, "f32", 16, "e4m3", 16),
          ("the limit", 1024, 8, 1024, "bf16", 32, "e5m2", 16)]
ROUTINGS = [("uniform", 1.2), ("zipf", 1.2), ("zipf", 2.0), ("one", 1.2), ("mixed", 1.2)]


def ragged(tokens, n):
    """Tokens per rank: the model's count on rank 0, then a few short of it, one token, none, and more."""
    return [tokens, tokens - 3, 1, 0, tokens // 2, tokens - 1, 7, tokens - 5][:n]


def load_of(topk, E, n):
    """The most rows any rank receives with unlimited capacity."""
    ids = np.concatenate([t.reshape(-1) for t in topk]).astype(np.int64)
    ids = ids[(ids >= 0) & (ids < E)]
    return int(np.bincount(ids // (E // n), minlength=n).max())


def read_small(small):
    return [(s[0].cpu().numpy(), s[1].cpu().numpy(), int(s[2].item())) for s in small]


def wide_dispatch(g, xd, idx, topk, E, recv_rows, row, dt):
    """The wide dispatch on every rank into poisoned arena buffers; returns (recv buffers, [(counts, route, dropped)] per rank)."""
    torch = g.torch
    recv = [c.empty(recv_rows * row, dt) for c in g.comms]
    for b in recv:
        b.view(torch.uint8).fill_(POISON)
    small = eg.small_outputs(g, topk, E)
    g.sync()
    for r, c in enumerate(g.comms):
        c.expert_dispatch(xd[r], idx[r], E, recv[r], *small[r], stream=g.streams[r])
    g.sync()
    g.check_async()
    return recv, read_small(small)


def fp8_dispatch(g, xd, idx, topk, E, recv_rows, row, wire, block):
    """The FP8 dispatch on every rank into poisoned arena buffers; returns (recv, recv_scales, [(counts, route, dropped)] per rank)."""
    torch = g.torch
    recv = [c.empty(recv_rows * row, wire) for c in g.comms]
    sc = [c.empty(recv_rows * row // block, torch.float32) for c in g.comms]
    for b in recv + sc:
        b.view(torch.uint8).fill_(POISON)
    small = eg.small_outputs(g, topk, E)
    g.sync()
    for r, c in enumerate(g.comms):
        c.expert_dispatch_quantized(xd[r], idx[r], E, recv[r], sc[r], block, *small[r], stream=g.streams[r])
    g.sync()
    g.check_async()
    return recv, sc, read_small(small)


def check_rank(lay, xs, d, recv_bytes, small, what):
    """Rank d's recv bytes, expert_counts, route and dropped against the layout reference, as check_dispatch does."""
    counts, route, dropped = small
    want = rr.recv_rows_of(lay, xs, d, np.full(recv_bytes.shape, POISON, dtype=np.uint8))
    bad = np.nonzero((recv_bytes != want).any(axis=1))[0]
    assert bad.size == 0, f"{what}: rank {d} recv rows {bad[:8].tolist()} ({bad.size} rows) differ"
    assert (counts == lay.counts[d]).all(), f"{what}: rank {d} expert_counts differ at experts {np.nonzero(counts != lay.counts[d])[0][:8].tolist()}"
    assert (route == lay.route[d]).all(), f"{what}: rank {d} route differs at {np.argwhere(route != lay.route[d])[:4].tolist()}"
    assert dropped == lay.dropped[d], f"{what}: rank {d} dropped {dropped} want {lay.dropped[d]}"


def layout_sweep(g, shapes, rng):
    """Every shape x routing x capacity (ample, exactly the load, one row less, 3/5 of it) through the wide dispatch, checked against the
    layout reference; per shape and routing, the FP8 dispatch of the same ids at one row less than the load gives the same small outputs."""
    n = g.n
    for name, E, k, T, dt_name, row, wire_name, block in shapes:
        E -= E % n
        dt, wire = DTYPES[dt_name], DTYPES[wire_name]
        es = dt.itemsize
        for kind, skew in ROUTINGS:
            topk = routing(kind, n, E, k, seed=E + k + n + int(10 * skew), tokens=ragged(T, n), skew=skew)
            xs = [eg._x_bytes(rng, t.shape[0], row * es, es) for t in topk]
            xd = [eg.dev_rows(g, c, xs[r], dt) for r, c in enumerate(g.comms)]
            idx = [g.dev(c, topk[r]) for r, c in enumerate(g.comms)]
            load = load_of(topk, E, n)
            for cap, recv_rows in (("ample", load + 5), ("exactly the load", load), ("load - 1", load - 1), ("3/5 of the load", load * 3 // 5)):
                recv_rows = max(1, recv_rows)
                lay = rr.layout(topk, E, recv_rows)
                if cap in ("ample", "exactly the load"):
                    assert sum(lay.dropped) == 0
                elif cap == "load - 1":
                    assert sum(lay.dropped) >= 1
                what = f"n={n} {name} E={E} top_k={k} {dt_name} {kind} skew={skew} {cap} (recv_rows {recv_rows})"
                recv, small = wide_dispatch(g, xd, idx, topk, E, recv_rows, row, dt)
                for d in range(n):
                    check_rank(lay, xs, d, recv[d].view(g.torch.uint8).cpu().numpy().reshape(recv_rows, -1), small[d], what)
                release(g.comms, recv)
                if cap == "load - 1":
                    q, sc, qsmall = fp8_dispatch(g, xd, idx, topk, E, recv_rows, row, wire, block)
                    release(g.comms, q, sc)
                    for d in range(n):
                        (c1, r1, d1), (c2, r2, d2) = small[d], qsmall[d]
                        assert (c1 == c2).all() and (r1 == r2).all() and d1 == d2, f"{what}: rank {d} FP8 dispatch ({wire_name}, block {block}) vs wide"


@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_routed_layout_at_model_shapes(torch_cuda, coll_mod, n):
    """DeepSeek-V3 (256 experts, top-8, 4096 tokens per rank), Kimi K2 (384, top-8, 2048), Qwen3-Next (512, top-10, 2048) and the
    1024-expert limit (top-8, 1024); experts rounded down to a multiple of 3 at n = 3. Ragged token counts, uniform, Zipf 1.2, Zipf 2.0
    (a hot expert), one-expert and mixed routings."""
    with Group(torch_cuda, coll_mod, n) as g:
        layout_sweep(g, SHAPES, np.random.default_rng(n))


# ------------------------------------------------------------------------------------------------- combine past the slot batch
CROW, CBLOCK = 128, 128
PAIRS = [(i, o) for i in ("bf16", "f16", "f32") for o in ("bf16", "f16", "f32")]


def batch_routing(n, k, seed):
    """Uniform ids over 8n experts with dropped slots in the first slot batch (slot 2), at the first slot of the second (slot 8) and at
    the last slot, and one token with every slot dropped."""
    topk = routing("uniform", n, 8 * n, k, seed=seed, tokens=[37, 29, 45, 21, 33, 40, 26, 31][:n])
    for ids in topk:
        ids[0::3, 2] = -1
        ids[1::3, 8] = 8 * n
        ids[2::3, k - 1] = INT32_MIN
        ids[4, :] = -1
    return topk


def combine_sweep(g, k, rng):
    """For one top_k past the slot batch: the wide route and segment combines for all 9 (in, out) pairs, and both FP8 combines at block
    128 for both wire types, each with weights and without (scale 0.75); dropped slots by id, by capacity and by the segment plan."""
    torch, n = g.torch, g.n
    E = 8 * n
    topk = batch_routing(n, k, seed=100 * k + n)
    tokens = [t.shape[0] for t in topk]
    route_rows = max(1, load_of(topk, E, n) * 4 // 5)
    plan = cq.segment_plan(topk, E, True, seed=k)
    maps = {"route": (rr.layout(topk, E, route_rows).route, route_rows), "segment": (plan.index, max(1, plan.recv_rows))}
    for kind, (index, recv_rows) in maps.items():
        for r in range(n):                                          # a dropped slot in each batch
            dropped = (index[r] < 0) | (index[r] >= n * recv_rows)
            assert dropped[:, :8].any() and dropped[:, 8:].any(), (kind, k, r)
    w = [rng.uniform(-1.5, 1.5, size=t.shape).astype(np.float32) for t in topk]
    idx = {kind: [g.dev(c, m[0][r]) for r, c in enumerate(g.comms)] for kind, m in maps.items()}
    wd = [g.dev(c, w[r]) for r, c in enumerate(g.comms)]
    cases = [(kind, in_name, out_name, None) for kind in maps for in_name, out_name in PAIRS]
    cases += [(kind, *PAIRS[(4 * i + 2 * j + k) % 9], wire) for i, kind in enumerate(maps) for j, wire in enumerate(("e4m3", "e5m2"))]
    for case, (kind, in_name, out_name, wire_name) in enumerate(cases):
        index, recv_rows = maps[kind]
        in_dt, out_dt = DTYPES[in_name], DTYPES[out_name]
        xs = [qr.gen(recv_rows * CROW, in_dt, CBLOCK, seed=case + 7 * r).view(recv_rows, CROW) for r in range(n)]
        eo = [c.empty(recv_rows * CROW, in_dt) for c in g.comms]
        for e, x in zip(eo, xs):
            e.copy_(x.reshape(-1))
        if wire_name is None:
            rows = [x.float().numpy() for x in xs]
        else:
            rows = [qr.quantize(x.reshape(-1), CBLOCK, DTYPES[wire_name])[2].numpy().reshape(-1, CROW) for x in xs]
        for weights, scale in ((True, 1.0), (False, 0.75)):
            outs = [torch.full((tokens[r], CROW), float("nan"), dtype=out_dt, device=f"cuda:{c.device}") for r, c in enumerate(g.comms)]
            g.sync()
            for r, c in enumerate(g.comms):
                wr, st = wd[r] if weights else None, g.streams[r]
                if kind == "route" and wire_name is None:
                    c.expert_combine(eo[r], idx[kind][r], wr, outs[r], scale=scale, stream=st)
                elif kind == "route":
                    c.expert_combine_quantized(eo[r].view(-1, CROW), idx[kind][r], wr, outs[r], block=CBLOCK, wire=DTYPES[wire_name], scale=scale, stream=st)
                elif wire_name is None:
                    c.all_to_all_v_combine(eo[r], outs[r].view(-1), CROW, *plan.args(r), idx[kind][r], wr, scale=scale, stream=st)
                else:
                    c.all_to_all_v_combine_quantized(eo[r].view(-1, CROW), outs[r].view(-1), CROW, *plan.args(r), idx[kind][r], wr, block=CBLOCK,
                                                     wire=DTYPES[wire_name], scale=scale, stream=st)
            g.sync()
            g.check_async()
            for r in range(n):
                look = route_lookup(rows, recv_rows) if kind == "route" else cr.plan_lookup(rows, *plan.args(r))
                want = cr.combine(look, index[r], w[r] if weights else None, scale, out_dt)
                assert_same(outs[r].cpu(), want, f"n={n} top_k={k} {kind} {in_name}->{wire_name or 'wide'}->{out_name} weights={weights}: rank {r}")
        release(g.comms, eo)


@pytest.mark.parametrize("k", [9, 10, 16])
@pytest.mark.parametrize("n", [1, 3])
def test_combine_past_the_slot_batch(torch_cuda, coll_mod, n, k):
    with Group(torch_cuda, coll_mod, n) as g:
        combine_sweep(g, k, np.random.default_rng(k))


# ------------------------------------------------------------------------------------------------- one real-width round trip
HIDDEN = 7168


def test_round_trip_at_deepseek_width(torch_cuda, coll_mod):
    """8 ranks, 256 experts, top-8, 512 tokens per rank, rows of 7168 bf16 (Zipf routing, capacity 4/5 of the load): the wide dispatch
    byte for byte; expert_combine with the router's weights over recv as the expert output ("identity expert") bit for bit; the FP8
    dispatch at block 128 against the host quantiser, rows and scales."""
    torch = torch_cuda
    n, E, k, T, block = 8, 256, 8, 512, 128
    topk = routing("zipf", n, E, k, seed=7, tokens=[T] * n)
    recv_rows = load_of(topk, E, n) * 4 // 5
    lay = rr.layout(topk, E, recv_rows)
    assert sum(lay.dropped) > 0
    xs = [qr.gen(T * HIDDEN, torch.bfloat16, block, seed=30 + s).view(T, HIDDEN) for s in range(n)]
    xb = [x.view(torch.uint8).numpy() for x in xs]
    rng = np.random.default_rng(8)
    w = [rng.uniform(0.0, 1.0, size=(T, k)).astype(np.float32) for _ in range(n)]
    arena_mb = (recv_rows * (HIDDEN * 3 + HIDDEN // block * 4)) // (1 << 20) + 32
    with Group(torch, coll_mod, n, arena_mb=arena_mb) as g:
        xd = [x.to(f"cuda:{c.device}") for x, c in zip(xs, g.comms)]
        idx = [g.dev(c, topk[r]) for r, c in enumerate(g.comms)]
        recv, small = wide_dispatch(g, xd, idx, topk, E, recv_rows, HIDDEN, torch.bfloat16)
        for d in range(n):
            check_rank(lay, xb, d, recv[d].view(torch.uint8).cpu().numpy().reshape(recv_rows, -1), small[d], f"width {HIDDEN}")
        route = [g.dev(c, small[r][1]) for r, c in enumerate(g.comms)]
        wd = [g.dev(c, w[r]) for r, c in enumerate(g.comms)]
        outs = [torch.full((T, HIDDEN), float("nan"), dtype=torch.bfloat16, device=f"cuda:{c.device}") for c in g.comms]
        g.sync()
        for r, c in enumerate(g.comms):
            c.expert_combine(recv[r], route[r], wd[r], outs[r], stream=g.streams[r])
        g.sync()
        g.check_async()
        # row r of rank d's recv holds x[s][t] for source[d][r] = (s, t): the identity expert's output, read from the inputs
        src = np.stack(lay.source)
        xf = np.stack([x.float().numpy() for x in xs])

        def look(col):
            col = np.asarray(col, dtype=np.int64)
            valid = (col >= 0) & (col < n * recv_rows)
            y = np.zeros((col.size, HIDDEN), dtype=np.float32)
            i = np.nonzero(valid)[0]
            s, t = src[col[i] // recv_rows, col[i] % recv_rows].T
            y[i] = xf[s, t]
            return valid, y
        for r in range(n):
            assert_same(outs[r].cpu(), cr.combine(look, lay.route[r], w[r], 1.0, torch.bfloat16), f"identity-expert combine rank {r}")
        release(g.comms, recv)
        wire = torch.float8_e4m3fn
        q, sc, qsmall = fp8_dispatch(g, xd, idx, topk, E, recv_rows, HIDDEN, wire, block)
        ref = [qr.quantize(x.reshape(-1), block, wire) for x in xs]
        qb = [a[0].view(torch.uint8).numpy().reshape(T, HIDDEN) for a in ref]
        sb = [a[1].view(torch.uint8).numpy().reshape(T, -1) for a in ref]
        for d in range(n):
            got_q, got_s = q[d].cpu().view(torch.uint8).numpy().reshape(recv_rows, -1), sc[d].cpu().view(torch.uint8).numpy().reshape(recv_rows, -1)
            want_q = rr.recv_rows_of(lay, qb, d, np.full(got_q.shape, POISON, dtype=np.uint8))
            want_s = rr.recv_rows_of(lay, sb, d, np.full(got_s.shape, POISON, dtype=np.uint8))
            assert_same(torch.from_numpy(got_q).view(wire), torch.from_numpy(want_q).view(wire), f"FP8 rows rank {d}")
            assert_same(torch.from_numpy(got_s).view(torch.float32), torch.from_numpy(want_s).view(torch.float32), f"scales rank {d}")
            assert all((a == b).all() for a, b in zip(qsmall[d][:2], small[d][:2])) and qsmall[d][2] == small[d][2], f"FP8 vs wide rank {d}"
        release(g.comms, q, sc)


# ------------------------------------------------------------------------------------------------- past 4 GiB
BIG_SLOTS = 320_000                                        # rows of rank 0's recv: 320,000 x 14,336 B = 4.59 GB
FIRST_PAST_4GIB = (1 << 32) // (HIDDEN * 2)                # row 299,593 starts below 2^32 and ends past it


@pytest.mark.parametrize("n", [1, 2])
def test_recv_past_4_gib(torch_cuda, coll_mod, n):
    """Every slot to rank 0's experts, so rank 0's recv (320,000 rows of 7168 bf16) is larger than 2^32 bytes: n = 1 runs the local
    kernels, n = 2 the peer kernels at arena offsets (rank 1's recv is the same size and must stay untouched). Every row of rank 0's recv
    is compared with x gathered by the layout's source, and the wide combine that reads the rows back with a device sum in fp32 of
    separate multiplies and adds in slot order, the order of coll_combine_reference.combine."""
    torch = torch_cuda
    k, E = 8, 8 * n
    T = BIG_SLOTS // k // n
    row_bytes = HIDDEN * 2
    recv_bytes = BIG_SLOTS * row_bytes
    assert (BIG_SLOTS - 1) * row_bytes >= 1 << 32 and FIRST_PAST_4GIB < BIG_SLOTS
    chunk = 8192
    # both ranks' recv (symmetric arenas), x and out per rank, and the reference's temporaries, plus a margin for other users
    need = n * (recv_bytes + (256 << 20)) + 2 * n * T * row_bytes + 4 * chunk * HIDDEN * 4 + (4 << 30)
    free, total = torch.cuda.mem_get_info(0)
    print(f"n={n}: {free / 2**30:.1f} GiB free of {total / 2**30:.1f} GiB, {need / 2**30:.1f} GiB needed")
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of device memory, {free / 2**30:.1f} GiB free")
    rng = np.random.default_rng(n)
    topk = [rng.integers(0, E // n, size=(T, k)).astype(np.int32) for _ in range(n)]       # rank 0's experts only
    lay = rr.layout(topk, E, BIG_SLOTS)
    assert int(lay.counts[0].sum()) == BIG_SLOTS and sum(lay.dropped) == 0
    with Group(torch, coll_mod, n, arena_mb=recv_bytes // (1 << 20) + 64) as g:
        gen = torch.Generator(device="cuda:0").manual_seed(n)
        xd = [torch.randn(T, HIDDEN, generator=gen, device="cuda:0").to(torch.bfloat16) for _ in range(n)]
        idx = [g.dev(c, topk[r]) for r, c in enumerate(g.comms)]
        w = [torch.rand(T, k, generator=gen, device="cuda:0") for _ in range(n)]
        recv, small = wide_dispatch(g, xd, idx, topk, E, BIG_SLOTS, HIDDEN, torch.bfloat16)
        for d in range(n):
            counts, route, dropped = small[d]
            assert (counts == lay.counts[d]).all() and (route == lay.route[d]).all() and dropped == lay.dropped[d], f"n={n} rank {d}"
        if n == 2:
            assert bool((recv[1].view(torch.uint8) == POISON).all()), "rank 1's recv was written"
        # rank 0's recv, row r = x[s][t] for source[0][r] = (s, t)
        src = torch.from_numpy(lay.source[0]).to("cuda:0")
        xcat = torch.cat(xd)
        at = src[:, 0] * T + src[:, 1]
        r0 = recv[0].view(BIG_SLOTS, HIDDEN)
        for lo in range(0, BIG_SLOTS, chunk):
            hi = min(BIG_SLOTS, lo + chunk)
            same = (r0[lo:hi].view(torch.int16) == xcat[at[lo:hi]].view(torch.int16)).all(dim=1)
            if not bool(same.all()):
                bad = lo + int((~same).nonzero()[0])
                pytest.fail(f"n={n}: recv row {bad} differs ({'at or past' if bad >= FIRST_PAST_4GIB else 'below'} the 2^32-byte boundary, row {FIRST_PAST_4GIB})")
        del xcat, at, src
        outs = [torch.full((T, HIDDEN), float("nan"), dtype=torch.bfloat16, device="cuda:0") for _ in range(n)]
        route = [g.dev(c, lay.route[r]) for r, c in enumerate(g.comms)]
        g.sync()
        for r, c in enumerate(g.comms):
            c.expert_combine(recv[r], route[r], w[r], outs[r], stream=g.streams[r])
        g.sync()
        g.check_async()
        for r in range(n):
            rows = route[r].long()                                  # every route names a row of rank 0's recv
            assert bool((rows >= 0).all()) and bool((rows < BIG_SLOTS).all())
            for lo in range(0, T, chunk):
                hi = min(T, lo + chunk)
                acc = torch.zeros(hi - lo, HIDDEN, dtype=torch.float32, device="cuda:0")
                for j in range(k):
                    prod = torch.mul(w[r][lo:hi, j:j + 1], r0[rows[lo:hi, j]].float())
                    acc = torch.add(acc, prod)
                want = torch.mul(acc, 1.0).to(torch.bfloat16)
                got = outs[r][lo:hi]
                if not torch.equal(got.view(torch.int16), want.view(torch.int16)):
                    bad = lo + int((got.view(torch.int16) != want.view(torch.int16)).any(dim=1).nonzero()[0])
                    pytest.fail(f"n={n}: combine rank {r} token {bad} differs (its rows {rows[bad].tolist()}, row {FIRST_PAST_4GIB} is the first past 2^32 bytes)")
        release(g.comms, recv)


# ------------------------------------------------------------------------------------------------- real devices
def test_on_real_devices(torch_cuda, coll_mod):
    """With one rank per GPU the grid is the full 2 x SM count on every rank, not SM count / N, so the grid-stride loops take other
    strides: the DeepSeek-V3 layout sweep and the top-10 combine sweep on every GPU present."""
    n = torch_cuda.cuda.device_count()
    if n < 2:
        pytest.skip(f"needs >= 2 GPUs, {n} present")
    n = min(n, 8)
    with Group(torch_cuda, coll_mod, n, devices=list(range(n))) as g:
        layout_sweep(g, SHAPES[:1], np.random.default_rng(90))
        combine_sweep(g, 10, np.random.default_rng(91))
