"""Every libb200coll family back to back on one communicator (`pytest -m gpu`): calls of different families follow each other on each
rank's stream with no host sync in between, ranks out of step, launch shapes changing between calls, inputs rewritten on the stream
right after a call, and eager windows between replays of a captured mixed graph. Virtual ranks share cuda:0 like the rest of the GPU
suite.

Every family keeps state on the communicator that the next call of any family inherits: the barrier epoch and flag rows (grids differ
by family and size, so rows one call leaves unused keep older epochs), the Lamport sequence and the spans the next Lamport call clears,
the two staging halves, the FP8 quantisation scratch (grown mid-stream), and the route-count and send/recv mailboxes. Each call here is
a *kind*: one public `Comm` call with its inputs, its own output buffers and its check against the order-exact reference of its family.
The sequence-parallel kinds (the Ulysses all-to-all both ways, the context-parallel gather and reduce-scatter) share the barrier epoch
with every two-shot, block-scaled, RMSNorm, dispatch and combine kernel; each draws its head config (replicated K and V included),
packed or dense layout, chunks, B and S_l from the schedule's rng. The three schedules:

  a. every ordered pair of kinds adjacent once (an Eulerian circuit of the complete directed graph with loops), at n = 3 and 4;
  b. seeded random schedules at n = 2, 3, 4 and 8 with launch-shape changes, one rank held back by a delay kernel, and inputs rewritten
     on the stream after the call that read them;
  c. a mixed window captured in a CUDA graph per rank, replayed with new inputs, with eager windows in between.

Calls are enqueued op-major: call i on every rank before call i + 1 on any rank. The ranks share one GPU, and with more streams than
hardware connections (CUDA_DEVICE_MAX_CONNECTIONS defaults to 8; 8 ranks plus the default stream are 9 streams) a rank-major order can
queue a spinning kernel ahead of the peer kernel it waits for on the same connection. For the same reason, where ranks must share
connections (8 virtual ranks) the schedule leaves out the calls that run several dependent operations on a rank's stream (staged
buffers, the pipelined host all-reduce). A window ends with one sync, the watchdog check, and then every check of the window.

A failure names the schedule, seed and step, the call's kind and parameters and those of the call before it, the rank and the first
differing element. ONLY (below) restricts a run to one schedule label, seed or window."""
import numpy as np
import pytest
import torch

from container_engine_accelerators_b200.ops.coll import AVG, MAX, MIN, PROD, QUANT_BLOCKS, SUM, B200CollError
from tests import coll_combine_reference as CR
from tests import coll_context_reference as cref
from tests import coll_fp_reference as R
from tests import coll_quant_reference as QR
from tests import coll_rmsnorm_quant_reference as RNQ
from tests import coll_rmsnorm_reference as RN
from tests import coll_routed_reference as RR
from tests import coll_rs_rmsnorm_reference as RS
from tests import coll_ulysses_reference as uref
from tests.coll_gpu_harness import DTYPES, Group, Plan, coll_mod, poison, torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu

# Restrict a run, e.g. ONLY = {"label": "random n=3", "seed": 11, "window": 4}; None runs everything.
ONLY = None

WINDOW = 16                     # calls per window of the pair schedule
TIMEOUT_MS = 30000              # the watchdog turns a protocol bug into a RemoteError with a fault record instead of a hung GPU
ARENA_MB = 512
SLEEP_CYCLES = 2_000_000        # about 1 ms at H100 clocks: the held-back rank's peers enter the next call first
WIDE = ("bfloat16", "float16", "float32")
FP8 = ("float8_e4m3fn", "float8_e5m2")
POISON_BYTE = 0x5A
# the epilogue's (in_dtype, out_dtype) pairs: every type to itself and fp32, fp32 to every type, FP8 to FP8, bf16 and fp16
OUTS = {"float32": WIDE + FP8, "bfloat16": ("bfloat16", "float32") + FP8, "float16": ("float16", "float32") + FP8,
        **{f: FP8 + ("bfloat16", "float16") for f in FP8}}


def esize(name):
    return R.esize(DTYPES[name])


# ------------------------------------------------------------------------------------------------- sizes
# Element counts per source that straddle each path's thresholds. `claims` names the thresholds (bytes per source, as a function of
# the rank count) that every list must have a size at or below and a size above; test_coll_mixed_sequence_cpu.py checks them.
def ll_counts(es, n):
    """Around the LL limit per source and the LL2 limit (n x that), plus a short odd count (scalar tail) and a ragged one."""
    ll, e = R.LL_ONESHOT_MAX_BYTES // es, 16 // es
    return [1003, e * 37 + 3, ll, ll + e + 3, ll * n, ll * n + e + 3]


def vec_counts(es, n):
    """Whole 16-byte vectors per rank (reduce-scatter, all-gather, all-to-all): around the LL limit and the copy-engine threshold."""
    ll, e = R.LL_ONESHOT_MAX_BYTES // es, 16 // es
    return [37 * e, ll, ll + e, R.BULK_MIN_BYTES // es + 5 * e]


SIZE_CLAIMS = {
    "ll_counts": (ll_counts, {"LL": lambda n: R.LL_ONESHOT_MAX_BYTES, "LL2": lambda n: R.LL_ONESHOT_MAX_BYTES * n}),
    "vec_counts": (vec_counts, {"LL": lambda n: R.LL_ONESHOT_MAX_BYTES, "copy engine": lambda n: R.BULK_MIN_BYTES - 1}),
}


def staged_big_count(es, n):
    """One all-reduce on buffers outside the arena larger than a staging half: two staging rounds, the second ragged."""
    return R.staged_chunk(es, es, n, "all_reduce") + 1003


def host_counts(es, n):
    """all_reduce_host: zero-copy up to the LL limit, and three equal pipelined chunks (each its own all-reduce) above the pipeline bound."""
    return [1003, R.LL_ONESHOT_MAX_BYTES // es, 3 * R.HOST_PIPELINE_BYTES // 2 // es]


# ------------------------------------------------------------------------------------------------- helpers
def same(got, want, what, nan_payloads=False):
    R.assert_same(got.reshape(-1).to(want.device), want.reshape(-1), what, nan_payloads=nan_payloads)


def check_reduction(got, xs, ran, staged, n, in_dt, count, s, out_dt, what):
    """An all-reduce (or a chunk of one) against the order model of the algorithm it recorded; NVLS (real peers) within one output ulp
    around an fp64 sum plus N * max|x| * 2^-22, its scalar tail bit for bit."""
    assert sum(ran.values()) >= 1 and len(ran) == 1, f"{what}: recorded {ran}"
    a = next(iter(ran))
    if a == "nvls":
        e = R.vec_elems(in_dt)
        tail = count // e * e
        same(got[tail:], R.ref_reduce([x[tail:] for x in xs], list(range(n)), s, out_dt), what + " tail")
        x64 = torch.stack([x[:tail].double() for x in xs])
        ref = x64.sum(0) * float(np.float32(s))
        fin = torch.isfinite(ref)
        tol = ref.abs().clamp_min(2.0 ** -126) * 2.0 ** (1 - R.MANT[out_dt]) + n * x64.abs().max(0).values * abs(s) * 2.0 ** -22
        err = (got[:tail].to(ref.device).double() - ref).abs()
        assert bool((err[fin] <= tol[fin]).all()), f"{what}: NVLS error over tolerance"
        return
    if staged and a == "twoshot" and in_dt not in R.FP8_MAX:
        order = ("staged", n, R.vec_elems(in_dt), count, R.staged_chunk(R.esize(in_dt), R.esize(out_dt), n, "all_reduce"))
    else:
        assert sum(ran.values()) == 1, f"{what}: recorded {ran}"
        order = R.order_for(a, n, in_dt, count)
    same(got, R.ref_reduce(xs, order, s, out_dt), f"{what} ran {a}")


def eff_scale(op, scale, n):
    """The scale a sum (scale) or an avg (scale * 1/N, in fp32) multiplies by."""
    return scale if op == SUM else R.avg_scale(scale, n)


MAX_CONNECTIONS = 8             # CUDA_DEVICE_MAX_CONNECTIONS's default


def one_queue_each(g):
    """Whether every rank's stream (and the default stream) can have a hardware queue of its own. Where two virtual ranks' streams
    share one, a call that runs several dependent operations on a rank's stream (a staged call, the pipelined host all-reduce) can
    hold the queue while the peer operation it waits for sits behind it; one kernel per rank per call, enqueued op-major, cannot."""
    return sum(c.device == g.comms[0].device for c in g.comms) + 1 <= MAX_CONNECTIONS


def pick(rng, seq):
    return seq[int(rng.integers(len(seq)))]


# ------------------------------------------------------------------------------------------------- kinds
class Call:
    """One call of one kind: __init__ draws the parameters and allocates every buffer (nothing is allocated once calls are enqueued: an
    allocation can wait for the device while an earlier rank's kernel waits for this rank); fill(seed) writes fresh inputs and poisons
    the outputs on the current stream; enqueue(r, c, st) makes rank r's call; check() compares every rank with the reference of the
    inputs fill wrote. `inputs[r]` are rank r's read-only inputs: the schedule may overwrite them on the rank's stream after the call."""
    kind = "?"
    graph_ok = True

    def __init__(self, g, rng):
        self.g, self.n, self.rng = g, g.n, rng
        self.p = {}
        self._arena = []
        self.inputs = [[] for _ in range(g.n)]
        self.ran, self.staged = {}, 0

    def place(self, rng, choices):
        """A placement from choices; "plain" (staged through the staging halves: several dependent operations per rank) only where
        every rank's stream has a hardware connection of its own."""
        return pick(rng, [w for w in choices if w != "plain" or one_queue_each(self.g)])

    def desc(self):
        return f"{self.kind}(" + ", ".join(f"{k}={v}" for k, v in self.p.items()) + ")"

    def arena(self, numel, dt):
        ts = []
        for c in self.g.comms:
            with torch.cuda.device(c.device):
                t = c.empty(numel, dt)
            ts.append(t)
        self._arena.append(ts)
        return ts

    def plain(self, numel, dt):
        return [torch.empty(numel, dtype=dt, device=f"cuda:{c.device}") for c in self.g.comms]

    def bufs(self, where, numel, dt):
        return self.arena(numel, dt) if where == "arena" else self.plain(numel, dt)

    def release(self):
        for ts in self._arena:
            for c, t in zip(self.g.comms, ts):
                c.release(t)
        self._arena = []

    def load(self, bufs, xs):
        for b, x in zip(bufs, xs):
            b.view(-1).copy_(x.reshape(-1).to(b.device))


def _order_flag(rng):
    return pick(rng, ["auto", "ll", "ll2", "oneshot", "twoshot"])


class AllReduce(Call):
    """all_reduce on bf16 / fp16 / fp32 (with or without a cast, a scale or avg) or e4m3 / e5m2 inputs; auto or a forced algorithm; arena
    buffers, plain (staged) buffers or in place."""
    kind = "all_reduce"
    IN = WIDE

    def __init__(self, g, rng):
        super().__init__(g, rng)
        i = pick(rng, self.IN)
        o = i if rng.random() < 0.5 else pick(rng, OUTS[i])
        where = self.place(rng, ["arena", "arena", "plain", "in_place"] if esize(i) == esize(o) else ["arena", "arena", "plain"])
        op, scale = pick(rng, [(SUM, 1.0), (SUM, 0.1), (AVG, 1.0), (AVG, 0.375)])
        self.p = dict(dt=f"{i}->{o}", count=pick(rng, ll_counts(esize(i), self.n)), algo=_order_flag(rng), where=where, op=op, scale=scale)
        self.in_dt, self.out_dt = DTYPES[i], DTYPES[o]
        cnt = self.p["count"]
        self.ins = self.bufs("plain" if where == "plain" else "arena", cnt, self.in_dt)
        self.outs = [x.view(self.out_dt) for x in self.ins] if where == "in_place" else self.bufs(where, cnt, self.out_dt)
        if where != "in_place":
            self.inputs = [[x] for x in self.ins]

    def fill(self, seed):
        self.xs = R.gen_inputs(self.n, self.p["count"], self.in_dt, seed)
        self.load(self.ins, self.xs)
        if self.p["where"] != "in_place":
            poison(self.outs)

    def enqueue(self, r, c, st):
        c.set_algo(self.p["algo"])
        c.all_reduce(self.ins[r], self.outs[r], scale=self.p["scale"], op=self.p["op"], stream=st)

    def check(self):
        s = eff_scale(self.p["op"], self.p["scale"], self.n)
        for r in range(self.n):
            check_reduction(self.outs[r], self.xs, self.ran, self.staged, self.n, self.in_dt, self.p["count"], s, self.out_dt, f"rank {r}")


class AllReduceFp8(AllReduce):
    kind = "all_reduce_fp8"
    IN = FP8


class AllReduceStagedBig(AllReduce):
    """bf16 all-reduce on plain buffers larger than one staging half (two staging rounds)."""
    kind = "all_reduce_staged_big"
    graph_ok = False

    def __init__(self, g, rng):
        Call.__init__(self, g, rng)
        self.p = dict(dt="bfloat16->bfloat16", count=staged_big_count(2, self.n), algo="auto", where="plain", op=SUM, scale=0.1)
        self.in_dt = self.out_dt = torch.bfloat16
        self.ins, self.outs = self.plain(self.p["count"], self.in_dt), self.plain(self.p["count"], self.out_dt)
        self.inputs = [[x] for x in self.ins]


class Move(Call):
    """reduce_scatter, all_gather or all_to_all on LL, two-shot or the copy-engine path (identity, >= 1 MiB per rank)."""
    kind = "move"

    def __init__(self, g, rng, op):
        super().__init__(g, rng)
        self.kind, self.op = op, op
        i = pick(rng, WIDE + ("float8_e5m2",))
        ident = op != "reduce_scatter" and rng.random() < 0.5
        o = i if ident else pick(rng, [t for t in OUTS[i] if t in WIDE])
        scale = 1.0 if ident else pick(rng, [1.0, 0.1])
        rop = pick(rng, [SUM, AVG]) if op == "reduce_scatter" else SUM
        where = self.place(rng, ["arena", "arena", "arena", "plain"])
        self.p = dict(dt=f"{i}->{o}", count=pick(rng, vec_counts(esize(i), self.n)), algo=pick(rng, ["auto", "ll", "twoshot"]), where=where,
                      scale=scale, op=rop)
        self.in_dt, self.out_dt, self.ident = DTYPES[i], DTYPES[o], i == o and scale == 1.0       # the library's identity test
        cnt, n = self.p["count"], self.n
        self.ins = self.arena(cnt if op == "all_gather" else cnt * n, self.in_dt)
        self.outs = self.bufs(where, cnt if op == "reduce_scatter" else cnt * n, self.out_dt)
        self.inputs = [[x] for x in self.ins]

    def fill(self, seed):
        self.xs = R.gen_inputs(self.n, self.ins[0].numel(), self.in_dt, seed)
        self.load(self.ins, self.xs)
        poison(self.outs)

    def enqueue(self, r, c, st):
        c.set_algo(self.p["algo"])
        if self.op == "reduce_scatter":
            c.reduce_scatter(self.ins[r], self.outs[r], scale=self.p["scale"], op=self.p["op"], stream=st)
        elif self.op == "all_gather":
            c.all_gather(self.ins[r], self.outs[r], scale=self.p["scale"], stream=st)
        else:
            c.all_to_all(self.ins[r], self.outs[r], scale=self.p["scale"], stream=st)

    def mv(self, x):
        if self.ident and "ll" in self.ran:
            return R.ll_move(x)
        return R.ref_move(x, self.p["scale"], self.out_dt, self.ident)

    def check(self):
        n, m, xs = self.n, self.p["count"], self.xs
        assert len(self.ran) == 1, f"recorded {self.ran}"
        a = next(iter(self.ran))
        for r in range(n):
            what = f"rank {r} ran {a}"
            if self.op == "reduce_scatter":
                order = list(range(n)) if a == "ll" or self.in_dt in R.FP8_MAX else ("rotate", r)
                s = eff_scale(self.p["op"], self.p["scale"], n)
                same(self.outs[r], R.ref_reduce([x[r * m:(r + 1) * m] for x in xs], order, s, self.out_dt), what)
            elif self.op == "all_gather":
                same(self.outs[r], torch.cat([self.mv(x) for x in xs]), what, nan_payloads=self.ident)
            else:
                same(self.outs[r], torch.cat([self.mv(xs[q][r * m:(r + 1) * m]) for q in range(n)]), what, nan_payloads=self.ident)


class Rooted(Call):
    """broadcast or reduce with a varying root."""

    def __init__(self, g, rng, op):
        super().__init__(g, rng)
        self.kind, self.op = op, op
        i = pick(rng, WIDE + (FP8 if op == "reduce" else ()))
        ident = op == "broadcast" and rng.random() < 0.5
        o = i if ident else pick(rng, [t for t in OUTS[i] if t in WIDE])
        scale = 1.0 if ident else pick(rng, [1.0, 0.1])
        es = esize(i)
        counts = [435, 37 * (16 // es) + 3] + ([R.BULK_MIN_BYTES // es + 5 * (16 // es)] if op == "broadcast" else ll_counts(es, self.n)[2:4])
        self.p = dict(dt=f"{i}->{o}", count=pick(rng, counts), root=int(rng.integers(self.n)), where=self.place(rng, ["arena", "arena", "plain"]),
                      scale=scale, op=pick(rng, [SUM, AVG]) if op == "reduce" else SUM)
        self.in_dt, self.out_dt, self.ident = DTYPES[i], DTYPES[o], i == o and scale == 1.0
        self.ins = self.bufs(self.p["where"], self.p["count"], self.in_dt)
        self.outs = self.bufs(self.p["where"], self.p["count"], self.out_dt)
        self.inputs = [[x] for x in self.ins]

    def fill(self, seed):
        self.xs = R.gen_inputs(self.n, self.p["count"], self.in_dt, seed)
        self.load(self.ins, self.xs)
        poison(self.outs)
        self.untouched = self.outs[0].view(torch.uint8).clone()

    def enqueue(self, r, c, st):
        c.set_algo("auto")
        fn = c.broadcast if self.op == "broadcast" else c.reduce
        kw = {} if self.op == "broadcast" else {"op": self.p["op"]}
        fn(self.ins[r], self.outs[r], root=self.p["root"], scale=self.p["scale"], stream=st, **kw)

    def check(self):
        root, n = self.p["root"], self.n
        if self.op == "broadcast":
            x = self.xs[root]
            want = R.ll_move(x) if self.ident and "ll" in self.ran else R.ref_move(x, self.p["scale"], self.out_dt, self.ident)
            for r in range(n):
                same(self.outs[r], want, f"rank {r}", nan_payloads=self.ident)
            return
        s = eff_scale(self.p["op"], self.p["scale"], n)
        same(self.outs[root], R.ref_reduce(self.xs, list(range(n)), s, self.out_dt), f"root {root}")
        for r in range(n):
            if r != root:
                assert torch.equal(self.outs[r].view(torch.uint8).to(self.untouched.device), self.untouched), f"rank {r}'s recv was written"


GENERIC_INT = ("int8", "uint8", "int32", "uint32", "int64", "uint64", "float64")


class Generic(Call):
    """The generic reduction kernel: every operator on the integer types and fp64, min / max / prod on the floating-point types; through
    all_reduce, reduce_scatter or reduce, on arena or plain buffers."""
    kind = "generic"

    def __init__(self, g, rng):
        super().__init__(g, rng)
        name = pick(rng, GENERIC_INT + WIDE + FP8)
        op = pick(rng, [SUM, PROD, MIN, MAX] if name in GENERIC_INT else [PROD, MIN, MAX])
        e = 16 // esize(name)
        via = pick(rng, ["all_reduce", "reduce_scatter", "reduce"])
        self.p = dict(dt=name, op=op, via=via, count=pick(rng, [1003, e * (37 * self.n + 1) + 3]), root=int(rng.integers(self.n)),
                      where=self.place(rng, ["arena", "arena", "plain"]))
        self.dt = DTYPES[name]
        cnt = self.p["count"]
        self.rc = cnt // self.n // e * e
        self.ins = self.bufs(self.p["where"], cnt if via != "reduce_scatter" else self.rc * self.n, self.dt)
        self.outs = self.bufs(self.p["where"], self.rc if via == "reduce_scatter" else cnt, self.dt)
        self.inputs = [[x] for x in self.ins]

    def fill(self, seed):
        n, t, m = self.n, self.dt, self.ins[0].numel()
        if t in R.NP_INT:
            self.xs = [R.int_tensor(x, t) for x in R.int_inputs(n, m, t, seed)]
        elif t == torch.float64:
            g = torch.Generator(device="cuda").manual_seed(seed)
            self.xs = [torch.randn(m, generator=g, device="cuda", dtype=t) * 2.0 ** torch.randint(-30, 30, (m,), generator=g, device="cuda")
                       for _ in range(n)]
        else:
            self.xs = R.gen_inputs(n, m, t, seed)
            if self.p["op"] == PROD:                              # finite, inexact products
                self.xs = [R.cast(x.float().abs().clamp(0.5, 2.0) * torch.where(x.float() < 0, -1.0, 1.0), t) for x in self.xs]
        self.load(self.ins, self.xs)
        poison(self.outs)
        self.untouched = self.outs[0].view(torch.uint8).clone()

    def enqueue(self, r, c, st):
        op, via = self.p["op"], self.p["via"]
        if via == "all_reduce":
            c.all_reduce(self.ins[r], self.outs[r], op=op, stream=st)
        elif via == "reduce_scatter":
            c.reduce_scatter(self.ins[r], self.outs[r], op=op, stream=st)
        else:
            c.reduce(self.ins[r], self.outs[r], root=self.p["root"], op=op, stream=st)

    def check(self):
        n, via, rc = self.n, self.p["via"], self.rc
        want = R.generic_ref(self.xs, self.p["op"])
        for r in range(n):
            if via == "all_reduce":
                same(self.outs[r], want, f"rank {r}")
            elif via == "reduce_scatter":
                same(self.outs[r], want[r * rc:(r + 1) * rc], f"rank {r}")
            elif r == self.p["root"]:
                same(self.outs[r], want, f"root {r}")
            else:
                assert torch.equal(self.outs[r].view(torch.uint8).to(self.untouched.device), self.untouched), f"rank {r}'s recv was written"


class Host(Call):
    """all_reduce_host on pinned host buffers: the zero-copy (Lamport) route or the pipelined route (equal chunks, each an all-reduce)."""
    kind = "all_reduce_host"
    graph_ok = False

    def __init__(self, g, rng):
        super().__init__(g, rng)
        i = pick(rng, ["bfloat16", "float32"])
        self.p = dict(dt=f"{i}->bfloat16", count=pick(rng, host_counts(esize(i), self.n)), scale=pick(rng, [1.0, 0.1]))
        self.in_dt, self.out_dt = DTYPES[i], torch.bfloat16
        cnt = self.p["count"]
        self.h_in = [c.host_empty(cnt, self.in_dt) for c in g.comms]
        self.h_out = [c.host_empty(cnt, self.out_dt) for c in g.comms]

    def release(self):
        for c, a, b in zip(self.g.comms, self.h_in, self.h_out):
            c.host_release(a)
            c.host_release(b)

    def fill(self, seed):
        self.xs = R.gen_inputs(self.n, self.p["count"], self.in_dt, seed)
        for h, x in zip(self.h_in, self.xs):
            h.copy_(x.cpu())
        for h in self.h_out:
            h.view(torch.uint8).fill_(0x7B)

    def enqueue(self, r, c, st):
        c.set_algo("auto")
        c.all_reduce_host(self.h_in[r], self.h_out[r], scale=self.p["scale"], stream=st)

    def check(self):
        n, cnt = self.n, self.p["count"]
        regime, chunks = R.host_chunks(cnt, R.esize(self.in_dt), R.esize(self.out_dt), n)
        assert len(set(chunks)) == 1 and len(self.ran) == 1 and sum(self.ran.values()) == len(chunks), (regime, chunks, self.ran)
        a = next(iter(self.ran))
        parts, d = [], 0
        for m in chunks:
            parts.append(R.ref_reduce([x[d:d + m] for x in self.xs], R.order_for(a, n, self.in_dt, m), self.p["scale"], self.out_dt))
            d += m
        want = torch.cat(parts)
        for r in range(n):
            same(self.h_out[r], want, f"rank {r} {regime} chunks={chunks} ran {a}")


class BlockScaled(Call):
    """all_gather / reduce_scatter / all_reduce_block_scaled: FP8 rows with fp32 block scales in, dequantised and summed in rank order."""

    def __init__(self, g, rng, op):
        super().__init__(g, rng)
        self.kind, self.op = f"{op}_block_scaled", op
        rows, row_len, block = pick(rng, [(48, 64, (1, 16)), (48, 400, (1, 128)), (120, 208, (32, 64))])
        self.p = dict(wire=pick(rng, FP8), out=pick(rng, WIDE), shape=(rows, row_len), block=block, scale=pick(rng, [1.0, 0.375]),
                      op=pick(rng, [SUM, AVG]), algo=pick(rng, ["oneshot", "twoshot", "auto"]))
        self.wire, self.out_dt = DTYPES[self.p["wire"]], DTYPES[self.p["out"]]
        self.grid = (-(-rows // block[0]), -(-row_len // block[1]))
        self.q = [t.view(rows, row_len) for t in self.arena(rows * row_len, self.wire)]
        self.s = [t.view(self.grid) for t in self.arena(self.grid[0] * self.grid[1], torch.float32)]
        out_rows = {"all_gather": self.n * rows, "reduce_scatter": rows // self.n, "all_reduce": rows}[op]
        self.outs = [t.view(out_rows, row_len) for t in self.arena(out_rows * row_len, self.out_dt)]
        self.inputs = [[a, b] for a, b in zip(self.q, self.s)]

    def fill(self, seed):
        rows, row_len = self.p["shape"]
        g = torch.Generator(device="cpu").manual_seed(seed)
        self.qs = [R.random_fp8(torch, rows * row_len, self.wire, seed + 31 * r).view(rows, row_len) for r in range(self.n)]
        self.ss = [(torch.exp2(torch.randint(-12, 13, self.grid, generator=g).float()) * (1 + torch.rand(self.grid, generator=g))).cuda()
                   for _ in range(self.n)]
        self.load(self.q, self.qs)
        self.load(self.s, self.ss)
        poison(self.outs)

    def dequant(self, q, s):
        rows, row_len = self.p["shape"]
        b = self.p["block"]
        return q.float() * s.repeat_interleave(b[0], dim=0)[:rows].repeat_interleave(b[1], dim=1)[:, :row_len]

    def enqueue(self, r, c, st):
        kw = dict(block=self.p["block"], scale=self.p["scale"], stream=st)
        if self.op == "all_gather":
            c.all_gather_block_scaled(self.q[r], self.s[r], self.outs[r], **kw)
        elif self.op == "reduce_scatter":
            c.reduce_scatter_block_scaled(self.q[r], self.s[r], self.outs[r], op=self.p["op"], **kw)
        else:
            c.set_algo(self.p["algo"])
            c.all_reduce_block_scaled(self.q[r], self.s[r], self.outs[r], op=self.p["op"], **kw)

    def check(self):
        n = self.n
        vs = [self.dequant(q, s) for q, s in zip(self.qs, self.ss)]
        if self.op == "all_gather":
            want = torch.cat([R.cast((torch.zeros_like(v) + v) * R.f32(self.p["scale"]).cuda(), self.out_dt) for v in vs])
        else:
            acc = torch.zeros_like(vs[0])
            for v in vs:
                acc = acc + v
            want = R.cast(acc * R.f32(eff_scale(self.p["op"], self.p["scale"], n)).cuda(), self.out_dt)
        m = want.shape[0] // n
        for r in range(n):
            same(self.outs[r], want[r * m:(r + 1) * m] if self.op == "reduce_scatter" else want, f"rank {r}")


class Quantized(Call):
    """all_gather / reduce_scatter / all_reduce_quantized: wide inputs quantised on their rank, FP8 and block scales over NVLink. `grow`
    makes the call large enough to grow the shared quantisation scratch."""

    def __init__(self, g, rng, op, grow=False):
        super().__init__(g, rng)
        self.kind, self.op = f"{op}_quantized", op
        block = pick(rng, (16, 128, 512))
        assert block in QUANT_BLOCKS
        per = block * self.n * (pick(rng, [1, 3, 37]) if not grow else max(1, grow // (block * self.n)))
        self.p = dict(src=pick(rng, WIDE), out=pick(rng, WIDE), block=block, wire=pick(rng, FP8), count=per, scale=pick(rng, [1.0, 0.1]),
                      op=pick(rng, [SUM, AVG]) if op != "all_gather" else SUM, where=pick(rng, ["arena", "plain"]), algo=pick(rng, ["auto", "oneshot", "twoshot"]))
        self.in_dt, self.out_dt, self.wire = DTYPES[self.p["src"]], DTYPES[self.p["out"]], DTYPES[self.p["wire"]]
        cnt = self.p["count"]
        self.ins = self.bufs(self.p["where"], cnt, self.in_dt)
        self.outs = self.arena({"all_gather": cnt * self.n, "reduce_scatter": cnt // self.n, "all_reduce": cnt}[op], self.out_dt)
        self.inputs = [[x] for x in self.ins]

    def fill(self, seed):
        self.xs = [QR.gen(self.p["count"], self.in_dt, self.p["block"], seed + 17 * r) for r in range(self.n)]
        self.load(self.ins, self.xs)
        poison(self.outs)

    def enqueue(self, r, c, st):
        kw = dict(block=self.p["block"], wire=self.wire, scale=self.p["scale"], stream=st)
        if self.op == "all_gather":
            c.all_gather_quantized(self.ins[r], self.outs[r], **kw)
        elif self.op == "reduce_scatter":
            c.reduce_scatter_quantized(self.ins[r], self.outs[r], op=self.p["op"], **kw)
        else:
            c.set_algo(self.p["algo"])
            c.all_reduce_quantized(self.ins[r], self.outs[r], op=self.p["op"], **kw)

    def check(self):
        b, w, n = self.p["block"], self.wire, self.n
        s = eff_scale(self.p["op"], self.p["scale"], n)
        if self.op == "all_gather":
            want = [QR.all_gather(self.xs, b, w, s, self.out_dt)] * n
        elif self.op == "reduce_scatter":
            want = [QR.reduce_scatter(self.xs, b, w, s, self.out_dt, r) for r in range(n)]
        else:
            want = [QR.all_reduce(self.xs, b, w, s, self.out_dt)] * n
        for r in range(n):
            same(self.outs[r].cpu(), want[r], f"rank {r}")


class RmsNorm(Call):
    """all_reduce_rms_norm(_quantized) and reduce_scatter_rms_norm(_quantized) (gather on and off)."""

    def __init__(self, g, rng, rs, quant):
        super().__init__(g, rng)
        self.rs, self.quant = rs, quant
        self.kind = ("reduce_scatter" if rs else "all_reduce") + "_rms_norm" + ("_quantized" if quant else "")
        n = self.n
        rows = n * pick(rng, [1, 3]) if rs else pick(rng, [1, 5, 16])
        self.p = dict(dt=pick(rng, WIDE), rows=rows, row_len=pick(rng, [512, 1024, 4096]), algo=pick(rng, ["auto", "oneshot", "twoshot"]),
                      where=pick(rng, ["arena", "plain"]), gather=bool(rs and rng.random() < 0.5), block=pick(rng, (16, 128)), wire=pick(rng, FP8))
        self.dt, self.wire = DTYPES[self.p["dt"]], DTYPES[self.p["wire"]]
        rows, rl, gather, where = rows, self.p["row_len"], self.p["gather"], self.p["where"]
        s_rows = rows // n if rs else rows
        o_rows = rows if (not rs or gather) else s_rows
        owhere = "arena" if gather else where
        self.x = [t.view(rows, rl) for t in self.arena(rows * rl, self.dt)]
        self.res = [t.view(s_rows, rl) for t in self.bufs(where, s_rows * rl, self.dt)]
        self.gamma = [t for t in self.plain(rl, self.dt)]
        if quant:
            self.q = [t.view(o_rows, rl) for t in self.bufs(owhere, o_rows * rl, self.wire)]
            self.sc = [t.view(o_rows, rl // self.p["block"]) for t in self.bufs(owhere, o_rows * rl // self.p["block"], torch.float32)]
        else:
            self.out = [t.view(o_rows, rl) for t in self.bufs(owhere, o_rows * rl, self.dt)]
        self.inputs = [[a, b] for a, b in zip(self.x, self.gamma)]

    def fill(self, seed):
        g = torch.Generator().manual_seed(seed)
        rows, rl, n = self.p["rows"], self.p["row_len"], self.n
        self.hx = [(torch.randn(rows, rl, generator=g) * 2.0 ** torch.randint(-3, 4, (rows, 1), generator=g)).to(self.dt) for _ in range(n)]
        s_rows = self.res[0].shape[0]
        self.hres = [torch.randn(s_rows, rl, generator=g).to(self.dt) for _ in range(n if self.rs else 1)]
        self.hgamma = (torch.rand(rl, generator=g) + 0.5).to(self.dt)
        self.load(self.x, self.hx)
        self.load(self.res, self.hres * (1 if self.rs else n))
        self.load(self.gamma, [self.hgamma] * n)
        poison(self.q + self.sc if self.quant else self.out)

    def enqueue(self, r, c, st):
        c.set_algo(self.p["algo"])
        x, res, gm = self.x[r], self.res[r], self.gamma[r]
        if not self.rs and not self.quant:
            c.all_reduce_rms_norm(x, res, gm, self.out[r], eps=1e-6, stream=st)
        elif not self.rs:
            c.all_reduce_rms_norm_quantized(x, res, gm, self.q[r], self.sc[r], block=self.p["block"], wire=self.wire, eps=1e-6, stream=st)
        elif not self.quant:
            c.reduce_scatter_rms_norm(x, res, gm, self.out[r], eps=1e-6, gather=self.p["gather"], stream=st)
        else:
            c.reduce_scatter_rms_norm_quantized(x, res, gm, self.q[r], self.sc[r], block=self.p["block"], wire=self.wire, eps=1e-6,
                                                gather=self.p["gather"], stream=st)

    def check(self):
        n, b = self.n, self.p["block"]
        if self.rs:
            per = (RS.rs_rms_norm_quantized(self.hx, self.hres, self.hgamma, 1e-6, self.dt, b, self.wire, self.p["gather"]) if self.quant else
                   RS.rs_rms_norm(self.hx, self.hres, self.hgamma, 1e-6, self.dt, self.p["gather"]))
        else:
            one = (RNQ.rms_norm_quantized(self.hx, self.hres[0], self.hgamma, 1e-6, self.dt, b, self.wire) if self.quant else
                   RN.rms_norm(self.hx, self.hres[0], self.hgamma, 1e-6, self.dt))
            per = [one] * n
        for r in range(n):
            same(self.res[r].cpu(), per[r][0], f"rank {r} residual")
            if self.quant:
                same(self.q[r].cpu(), per[r][1], f"rank {r} q")
                same(self.sc[r].cpu(), per[r][2], f"rank {r} scales")
            else:
                same(self.out[r].cpu(), per[r][1], f"rank {r} out")


def a2a_plan(n, rng):
    """rows[s, d] (some zero), send ranges laid out in a shuffled peer order with gaps, receive ranges by source with gaps."""
    rows = rng.integers(0, 6, size=(n, n))
    rows[rng.random((n, n)) < 0.2] = 0
    send_off, recv_off = np.zeros_like(rows), np.zeros_like(rows)
    for s in range(n):
        at = int(rng.integers(0, 3))
        for d in rng.permutation(n):
            send_off[s, d] = at
            at += rows[s, d] + int(rng.integers(0, 2))
    for d in range(n):
        at = int(rng.integers(0, 3))
        for s in range(n):
            recv_off[d, s] = at
            at += rows[s, d] + int(rng.integers(0, 3))
    return Plan(rows, send_off, recv_off)


class AllToAllV(Call):
    """all_to_all_v (a bit copy or a cast) and all_to_all_v_quantized."""

    def __init__(self, g, rng, quant):
        super().__init__(g, rng)
        self.quant, self.kind = quant, "all_to_all_v" + ("_quantized" if quant else "")
        self.plan = a2a_plan(self.n, rng)
        block = pick(rng, (16, 128))
        i = pick(rng, WIDE)
        o = pick(rng, FP8) if quant else pick(rng, (i, i) + OUTS[i][:2])
        scale = pick(rng, [1.0, 0.1]) if not quant and o != i else 1.0
        self.p = dict(dt=f"{i}->{o}", row=pick(rng, [block, 3 * block]), block=block, scale=scale, rows=self.plan.rows.tolist())
        self.in_dt, self.out_dt, self.ident = DTYPES[i], DTYPES[o], i == o and scale == 1.0
        row, P = self.p["row"], self.plan
        self.ins = self.arena(max(1, P.src_rows) * row, self.in_dt)
        self.recv_rows = max(1, P.recv_rows) + 2
        self.outs = self.arena(self.recv_rows * row, self.out_dt)
        if quant:
            self.scales = self.arena(self.recv_rows * row // block, torch.float32)
        self.inputs = [[x] for x in self.ins]

    def fill(self, seed):
        row, m = self.p["row"], self.ins[0].numel()
        self.xs = ([QR.gen(m, self.in_dt, self.p["block"], seed + 17 * r).cuda() for r in range(self.n)] if self.quant else
                   R.gen_inputs(self.n, m, self.in_dt, seed))
        self.load(self.ins, self.xs)
        for t in self.outs + (self.scales if self.quant else []):
            t.view(torch.uint8).fill_(POISON_BYTE)

    def enqueue(self, r, c, st):
        args = (self.p["row"], *self.plan.args(r))
        if self.quant:
            c.all_to_all_v_quantized(self.ins[r], self.outs[r], self.scales[r], *args, block=self.p["block"], stream=st)
        else:
            c.all_to_all_v(self.ins[r], self.outs[r], *args, scale=self.p["scale"], stream=st)

    def check(self):
        P, row, n, b = self.plan, self.p["row"], self.n, self.p["block"]
        for d in range(n):
            q = self.outs[d].view(torch.uint8).cpu().clone()
            want = torch.full_like(q, POISON_BYTE)
            if self.quant:
                sg = self.scales[d].cpu()
                ws = torch.full((sg.numel() * 4,), POISON_BYTE, dtype=torch.uint8).view(torch.float32)
            for s in range(n):
                cnt, so, ro = int(P.rows[s, d]), int(P.send_off[s, d]), int(P.recv_off[d, s])
                if cnt == 0:
                    continue
                x = self.xs[s][so * row:(so + cnt) * row]
                if self.quant:
                    wq, wsc, _ = QR.quantize(x.cpu(), b, self.out_dt)
                    want[ro * row:(ro + cnt) * row] = wq.view(torch.uint8)
                    ws[ro * row // b:(ro + cnt) * row // b] = wsc
                else:
                    es = R.esize(self.out_dt)
                    want[ro * row * es:(ro + cnt) * row * es] = R.ref_move(x, self.p["scale"], self.out_dt, self.ident).cpu().view(torch.uint8)
            same(q.view(self.out_dt), want.view(self.out_dt), f"rank {d} rows", nan_payloads=self.ident)
            if self.quant:
                same(sg, ws, f"rank {d} scales")


class A2AVCombine(Call):
    """all_to_all_v_combine and all_to_all_v_combine_quantized: the top-k weighted sum of expert rows pulled back along a plan."""

    def __init__(self, g, rng, quant):
        super().__init__(g, rng)
        self.quant, self.kind = quant, "all_to_all_v_combine" + ("_quantized" if quant else "")
        n = self.n
        self.plan = a2a_plan(n, rng)
        block = pick(rng, (16, 128))
        self.p = dict(dt=f"{pick(rng, WIDE)}->{pick(rng, WIDE)}", row=pick(rng, [block, 2 * block]), block=block, wire=pick(rng, FP8),
                      top_k=pick(rng, [1, 2, 5]), tokens=pick(rng, [1, 7, 24]), scale=pick(rng, [1.0, 0.5]), weights=bool(rng.random() < 0.7))
        i, o = self.p["dt"].split("->")
        self.in_dt, self.out_dt, self.wire = DTYPES[i], DTYPES[o], DTYPES[self.p["wire"]]
        self.recv_rows = max(1, self.plan.recv_rows)
        self.eo = self.arena(self.recv_rows * self.p["row"], self.in_dt)
        T, k = self.p["tokens"], self.p["top_k"]
        self.idx = [torch.empty(T, k, dtype=torch.int32, device=f"cuda:{c.device}") for c in g.comms]
        self.w = [torch.empty(T, k, dtype=torch.float32, device=f"cuda:{c.device}") for c in g.comms]
        self.outs = self.plain(T * self.p["row"], self.out_dt)
        self.inputs = [[a, b, c] for a, b, c in zip(self.eo, self.idx, self.w)]

    def fill(self, seed):
        rng = np.random.default_rng(seed)
        n, row, T, k = self.n, self.p["row"], self.p["tokens"], self.p["top_k"]
        self.heo = [QR.gen(self.recv_rows * row, self.in_dt, self.p["block"], seed + 13 * r).view(self.recv_rows, row) for r in range(n)]
        self.hidx = [rng.integers(-1, max(1, self.plan.src_rows) + 1, size=(T, k)).astype(np.int32) for _ in range(n)]
        self.hw = [rng.standard_normal((T, k)).astype(np.float32) for _ in range(n)]
        self.load(self.eo, self.heo)
        self.load(self.idx, [torch.from_numpy(a) for a in self.hidx])
        self.load(self.w, [torch.from_numpy(a) for a in self.hw])
        poison(self.outs)

    def enqueue(self, r, c, st):
        args = (self.outs[r].view(self.p["tokens"], self.p["row"]), self.p["row"], *self.plan.args(r), self.idx[r])
        w = self.w[r] if self.p["weights"] else None
        if self.quant:
            c.all_to_all_v_combine_quantized(self.eo[r].view(-1, self.p["row"]), *args, weights=w, block=self.p["block"], wire=self.wire,
                                             scale=self.p["scale"], stream=st)
        else:
            c.all_to_all_v_combine(self.eo[r].view(-1, self.p["row"]), *args, weights=w, scale=self.p["scale"], stream=st)

    def check(self):
        P, n, row = self.plan, self.n, self.p["row"]
        if self.quant:
            vals = [QR.quantize(e.reshape(-1), self.p["block"], self.wire)[2].numpy().reshape(-1, row) for e in self.heo]
        else:
            vals = [e.float().numpy() for e in self.heo]
        for r in range(n):
            look = CR.plan_lookup(vals, P.rows[r].tolist(), P.send_off[r].tolist(), [int(P.recv_off[d, r]) for d in range(n)])
            want = CR.combine(look, self.hidx[r], self.hw[r] if self.p["weights"] else None, self.p["scale"], self.out_dt)
            same(self.outs[r].cpu(), want, f"rank {r}")


class Expert(Call):
    """expert_dispatch(_quantized) from device top-k ids, and expert_combine(_quantized) along a device route."""

    def __init__(self, g, rng, combine, quant):
        super().__init__(g, rng)
        self.combine, self.quant = combine, quant
        self.kind = "expert_" + ("combine" if combine else "dispatch") + ("_quantized" if quant else "")
        n = self.n
        block = pick(rng, (16, 128))
        self.p = dict(dt=pick(rng, WIDE), out=pick(rng, WIDE), E=n * pick(rng, [1, 4]), top_k=pick(rng, [1, 2, 4]), route=pick(rng, ["uniform", "zipf", "mixed"]),
                      row=pick(rng, [block, 4 * block]), block=block, wire=pick(rng, FP8), tight=bool(rng.random() < 0.3), scale=pick(rng, [1.0, 0.25]),
                      weights=bool(rng.random() < 0.7), seed=int(rng.integers(1 << 20)))
        p = self.p
        self.topk = RR.routing(p["route"], n, p["E"], p["top_k"], seed=p["seed"])
        slots = sum(t.size for t in self.topk)
        self.recv_rows = max(1, slots // 2 if p["tight"] else slots)
        self.lay = RR.layout(self.topk, p["E"], self.recv_rows)
        self.in_dt, self.out_dt, self.wire = DTYPES[p["dt"]], DTYPES[p["out"]], DTYPES[p["wire"]]
        row, dev = p["row"], lambda c: f"cuda:{c.device}"
        if combine:
            self.eo = self.arena(self.recv_rows * row, self.in_dt)
            self.route = [torch.from_numpy(np.ascontiguousarray(rt)).to(dev(c)) for rt, c in zip(self.lay.route, g.comms)]
            self.w = [torch.empty(t.shape, dtype=torch.float32, device=dev(c)) for t, c in zip(self.topk, g.comms)]
            self.outs = [torch.empty(t.shape[0], row, dtype=self.out_dt, device=dev(c)) for t, c in zip(self.topk, g.comms)]
            self.inputs = [[a, b] for a, b in zip(self.eo, self.w)]
        else:
            self.x = [torch.empty(t.shape[0], row, dtype=self.in_dt, device=dev(c)) for t, c in zip(self.topk, g.comms)]
            self.ids = [torch.from_numpy(np.ascontiguousarray(t)).to(dev(c)) for t, c in zip(self.topk, g.comms)]
            self.recv = self.arena(self.recv_rows * row, self.wire if quant else self.in_dt)
            if quant:
                self.rsc = self.arena(self.recv_rows * row // block, torch.float32)
            self.small = [(torch.empty(p["E"] // n, dtype=torch.int32, device=dev(c)), torch.empty(t.shape, dtype=torch.int32, device=dev(c)),
                           torch.empty(1, dtype=torch.int32, device=dev(c))) for t, c in zip(self.topk, g.comms)]
            self.inputs = [[a, b] for a, b in zip(self.x, self.ids)]

    def fill(self, seed):
        row, n = self.p["row"], self.n
        if self.combine:
            rng = np.random.default_rng(seed)
            self.heo = [QR.gen(self.recv_rows * row, self.in_dt, self.p["block"], seed + 13 * r).view(self.recv_rows, row) for r in range(n)]
            self.hw = [rng.standard_normal(t.shape).astype(np.float32) for t in self.topk]
            self.load(self.eo, self.heo)
            self.load(self.w, [torch.from_numpy(a) for a in self.hw])
            poison(self.outs)
        else:
            self.hx = [QR.gen(t.shape[0] * row, self.in_dt, self.p["block"], seed + 17 * s).view(t.shape[0], row) for s, t in enumerate(self.topk)]
            self.load(self.x, self.hx)
            for t in self.recv + (self.rsc if self.quant else []):
                t.view(torch.uint8).fill_(POISON_BYTE)
            for sm in self.small:
                for t in sm:
                    t.fill_(-7)

    def enqueue(self, r, c, st):
        p = self.p
        if self.combine:
            w = self.w[r] if p["weights"] else None
            eo = self.eo[r].view(-1, p["row"])
            if self.quant:
                c.expert_combine_quantized(eo, self.route[r], w, self.outs[r], block=p["block"], wire=self.wire, scale=p["scale"], stream=st)
            else:
                c.expert_combine(eo, self.route[r], w, self.outs[r], scale=p["scale"], stream=st)
        elif self.quant:
            c.expert_dispatch_quantized(self.x[r], self.ids[r], p["E"], self.recv[r], self.rsc[r], p["block"], *self.small[r], stream=st)
        else:
            c.expert_dispatch(self.x[r], self.ids[r], p["E"], self.recv[r], *self.small[r], stream=st)

    def check(self):
        n, row, b, lay = self.n, self.p["row"], self.p["block"], self.lay
        if self.combine:
            if self.quant:
                vals = [QR.quantize(e.reshape(-1), b, self.wire)[2].numpy().reshape(-1, row) for e in self.heo]
            else:
                vals = [e.float().numpy() for e in self.heo]
            for r in range(n):
                want = CR.combine(RR.route_lookup(vals, self.recv_rows), lay.route[r], self.hw[r] if self.p["weights"] else None, self.p["scale"], self.out_dt)
                same(self.outs[r].cpu(), want, f"rank {r}")
            return
        if self.quant:
            ref = [QR.quantize(x.reshape(-1), b, self.wire) for x in self.hx]
            rows_of = [(q.view(torch.uint8).numpy().reshape(-1, row), s.view(torch.int32).numpy().reshape(-1, row // b)) for q, s, _ in ref]
        for d in range(n):
            counts, route, dropped = (t.cpu().numpy() for t in self.small[d])
            assert (counts == lay.counts[d]).all(), f"rank {d} expert_counts {counts.tolist()} want {lay.counts[d].tolist()}"
            assert (route == lay.route[d]).all(), f"rank {d} route differs at {np.argwhere(route != lay.route[d])[:1].tolist()}"
            assert int(dropped[0]) == lay.dropped[d], f"rank {d} dropped {int(dropped[0])} want {lay.dropped[d]}"
            got = self.recv[d].view(torch.uint8).cpu().numpy()
            if self.quant:
                wq = np.full((self.recv_rows, row), POISON_BYTE, dtype=np.uint8)
                wsc = np.full((self.recv_rows, row // b), int.from_bytes(bytes([POISON_BYTE] * 4), "little"), dtype=np.int32)
                for k, (s, t) in enumerate(lay.source[d]):
                    if s >= 0:
                        wq[k], wsc[k] = rows_of[s][0][t], rows_of[s][1][t]
                same(torch.from_numpy(got.copy()).view(self.wire), torch.from_numpy(wq).view(self.wire), f"rank {d} FP8 rows")
                same(self.rsc[d].cpu(), torch.from_numpy(wsc).view(torch.float32), f"rank {d} scales")
            else:
                es = R.esize(self.in_dt)
                xs = [x.contiguous().view(torch.uint8).numpy().reshape(x.shape[0], row * es) for x in self.hx]
                want = RR.recv_rows_of(lay, xs, d, np.full((self.recv_rows, row * es), POISON_BYTE, dtype=np.uint8))
                i = np.argwhere(got.reshape(self.recv_rows, -1) != want)
                assert i.size == 0, f"rank {d} recv row {i[0][0]} byte {i[0][1]} differs (source {lay.source[d][i[0][0]].tolist()})"


class SendRecv(Call):
    """One grouped send/recv ring step: every rank sends to rank + 1 and receives from rank - 1."""
    kind = "send_recv_ring"

    def __init__(self, g, rng):
        super().__init__(g, rng)
        self.p = dict(bytes=pick(rng, [16, 4096 + 16, 300000, (1 << 20) + 48]), src=pick(rng, ["arena", "plain"]), dst=self.place(rng, ["arena", "plain"]))
        nb = self.p["bytes"]
        self.ins = self.bufs(self.p["src"], nb, torch.uint8)
        self.outs = self.bufs(self.p["dst"], nb, torch.uint8)
        self.inputs = [[x] for x in self.ins]

    def fill(self, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.xs = [torch.randint(0, 256, (self.p["bytes"],), generator=g, device="cuda", dtype=torch.uint8) for _ in range(self.n)]
        self.load(self.ins, self.xs)
        poison(self.outs)

    def enqueue(self, r, c, st):
        from container_engine_accelerators_b200.ops import coll
        with coll.group():
            c.send(self.ins[r], (r + 1) % self.n, stream=st)
            c.recv(self.outs[r], (r - 1) % self.n, stream=st)

    def check(self):
        for r in range(self.n):
            same(self.outs[r], self.xs[(r - 1) % self.n], f"rank {r}", nan_payloads=True)


def random_bytes(shape, dt, seed):
    """Host random bytes (NaN payloads, -0 and inf in every float type) viewed as a dt tensor of `shape`."""
    nb = int(np.prod(shape)) * R.esize(dt)
    return torch.randint(0, 256, (nb,), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed)).view(dt).view(shape)


def load_views(bufs, xs):
    """Host tensors into device views of the same shape (column slices of a packed buffer included)."""
    for b, x in zip(bufs, xs):
        b.copy_(x.to(b.device))


def same_bytes(got, want, what):
    g, w = got.contiguous().view(torch.uint8).reshape(-1).cpu(), want.contiguous().view(torch.uint8).reshape(-1).cpu()
    assert g.numel() == w.numel(), f"{what}: {g.numel()} bytes vs {w.numel()}"
    bad = (g != w).nonzero()
    assert bad.numel() == 0, f"{what}: {bad.numel()} bytes differ, first at byte {int(bad[0])}"


def head_choices(n):
    """(name, Hq, Hkv) that n ranks allow: MHA, GQA, GQA with K and V replicated (Hkv a divisor of n below it) and MQA."""
    cfgs = [("mha", 2 * n, 2 * n), ("gqa", 4 * n, n)]
    small = [h for h in range(2, n) if n % h == 0]
    if small:
        cfgs.append(("gqa-replicated", 4 * n, small[-1]))
    cfgs.append(("mqa", 2 * n, 1))
    return cfgs


class Ulysses(Call):
    """all_to_all_seq_to_heads of q, k and v (column slices of one packed QKV or dense tensors; K and V replicated where the head config
    has fewer KV heads than ranks), or all_to_all_heads_to_seq of q alone or of q, k and v (dense head shards into column slices of a
    packed buffer or dense tensors). Head-side outputs and sequence-side outputs live in the arena."""

    def __init__(self, g, rng, s2h):
        super().__init__(g, rng)
        n, self.s2h = self.n, s2h
        self.kind = "all_to_all_seq_to_heads" if s2h else "all_to_all_heads_to_seq"
        name, hq, hkv = pick(rng, head_choices(n) if s2h else [h for h in head_choices(n) if h[2] % n == 0])
        heads = (hq, hkv, hkv) if s2h or rng.random() < 0.5 else (hq,)
        self.p = dict(dt=pick(rng, WIDE + ("float8_e4m3fn",)), heads=f"{name}{heads}", D=pick(rng, [16, 64, 80]), B=pick(rng, [1, 2, 3]),
                      S_l=pick(rng, [1, 5, 8, 33]), layout=pick(rng, ["packed", "dense"]))
        self.heads, self.dt = heads, DTYPES[self.p["dt"]]
        B, S_l, D, dt = self.p["B"], self.p["S_l"], self.p["D"], self.dt
        self.cols = np.cumsum([0] + [h * D for h in heads]).tolist()
        seq_bufs = self.bufs("plain" if s2h else "arena", B * S_l * self.cols[-1], dt) if self.p["layout"] == "packed" else None
        self.seq_whole = [] if seq_bufs is None else [b.view(B * S_l, self.cols[-1]) for b in seq_bufs]
        self.seq = []
        for r in range(n):
            if seq_bufs is not None:
                self.seq.append([self.seq_whole[r][:, self.cols[i]:self.cols[i + 1]].view(B, S_l, h, D) for i, h in enumerate(heads)])
            else:
                self.seq.append([])
        if seq_bufs is None:
            for h in heads:
                for r, t in enumerate(self.bufs("plain" if s2h else "arena", B * S_l * h * D, dt)):
                    self.seq[r].append(t.view(B, S_l, h, D))
        self.head = [[] for _ in range(n)]
        for h in heads:
            hl = h // n if h % n == 0 else 1
            for r, t in enumerate(self.bufs("arena" if s2h else "plain", B * n * S_l * hl * D, dt)):
                self.head[r].append(t.view(B, n * S_l, hl, D))
        src = self.seq if s2h else self.head
        self.inputs = [self.seq_whole[r:r + 1] if s2h and self.seq_whole else list(src[r]) for r in range(n)]

    def fill(self, seed):
        n, B, S_l, D = self.n, self.p["B"], self.p["S_l"], self.p["D"]
        if self.s2h:
            self.hx = [[random_bytes((B, S_l, h, D), self.dt, seed + 31 * r + i) for i, h in enumerate(self.heads)] for r in range(n)]
            load_views([t for row in self.seq for t in row], [t for row in self.hx for t in row])
            poison([t for row in self.head for t in row])
        else:
            self.hy = [[random_bytes(tuple(t.shape), self.dt, seed + 31 * r + i) for i, t in enumerate(self.head[r])] for r in range(n)]
            load_views([t for row in self.head for t in row], [t for row in self.hy for t in row])
            poison(self.seq_whole if self.seq_whole else [t for row in self.seq for t in row])

    def enqueue(self, r, c, st):
        if self.s2h:
            c.all_to_all_seq_to_heads(self.seq[r], self.head[r], stream=st)
        else:
            c.all_to_all_heads_to_seq(self.head[r], self.seq[r], stream=st)

    def check(self):
        n = self.n
        for i in range(len(self.heads)):
            if self.s2h:
                want = uref.seq_to_heads([self.hx[s][i] for s in range(n)])
                for r in range(n):
                    same_bytes(self.head[r][i], want[r], f"tensor {i} rank {r}")
            else:
                want = uref.heads_to_seq([self.hy[s][i] for s in range(n)])
                for r in range(n):
                    same_bytes(self.seq[r][i], want[r], f"tensor {i} rank {r}")


class Context(Call):
    """all_gather_context (bf16, fp16, fp32, e4m3 or e5m2) or reduce_scatter_context (bf16, fp16 or fp32) of one tensor, K and V as column
    slices of a packed QKV (dQKV, whose Q columns must stay poisoned), or an MLA-like pair of dense tensors; contiguous or load-balanced
    chunks. Full tensors live in the arena, and so do the reduce-scatter's shards."""

    def __init__(self, g, rng, gather):
        super().__init__(g, rng)
        n, self.gather = self.n, gather
        self.kind = "all_gather_context" if gather else "reduce_scatter_context"
        dt = pick(rng, WIDE + FP8 if gather else WIDE)
        e = 16 // esize(dt)
        chunks = pick(rng, [1, 2])
        layout = pick(rng, ["kv-packed", "mla-dense", "one"])
        widths = {"kv-packed": (pick(rng, [2, 4]) * e,) * 2, "mla-dense": (8 * e, e), "one": (pick(rng, [1, 3, 5]) * e,)}[layout]
        self.p = dict(dt=dt, layout=layout, widths=widths, chunks=chunks, B=pick(rng, [1, 2, 3]), S_l=pick(rng, [2, 6, 12] if chunks == 2 else [1, 5, 7, 12]))
        self.dt, self.widths = DTYPES[dt], widths
        B, S_l, S = self.p["B"], self.p["S_l"], n * self.p["S_l"]
        self.q_cols = 2 * widths[0] if layout == "kv-packed" else None
        self.full = [[] for _ in range(n)]
        for w in widths:
            for r, t in enumerate(self.arena(B * S * w, self.dt)):
                self.full[r].append(t.view(B, S, w))
        where = "plain" if gather else "arena"
        self.whole, self.shard = [], [[] for _ in range(n)]
        if self.q_cols is not None:
            row = self.q_cols + sum(widths)
            self.whole = [b.view(B * S_l, row) for b in self.bufs(where, B * S_l * row, self.dt)]
            for r, b in enumerate(self.whole):
                c0 = self.q_cols
                for w in widths:
                    self.shard[r].append(b[:, c0:c0 + w].view(B, S_l, w))
                    c0 += w
        else:
            for w in widths:
                for r, t in enumerate(self.bufs(where, B * S_l * w, self.dt)):
                    self.shard[r].append(t.view(B, S_l, w))
        self.inputs = [(self.whole[r:r + 1] if self.whole else list(self.shard[r])) if gather else list(self.full[r]) for r in range(n)]

    def fill(self, seed):
        n, B, S_l = self.n, self.p["B"], self.p["S_l"]
        if self.gather:
            self.hx = [[random_bytes((B, S_l, w), self.dt, seed + 31 * r + i) for i, w in enumerate(self.widths)] for r in range(n)]
            load_views([t for row in self.shard for t in row], [t for row in self.hx for t in row])
            poison([t for row in self.full for t in row])
        else:
            per = [R.gen_inputs(n, B * n * S_l * w, self.dt, seed + i, device="cpu") for i, w in enumerate(self.widths)]
            self.hf = [[per[i][r].view(B, n * S_l, w) for i, w in enumerate(self.widths)] for r in range(n)]
            load_views([t for row in self.full for t in row], [t for row in self.hf for t in row])
            poison(self.whole if self.whole else [t for row in self.shard for t in row])

    def enqueue(self, r, c, st):
        if self.gather:
            c.all_gather_context(self.shard[r], self.full[r], chunks=self.p["chunks"], stream=st)
        else:
            c.reduce_scatter_context(self.full[r], self.shard[r], chunks=self.p["chunks"], stream=st)

    def check(self):
        n, chunks = self.n, self.p["chunks"]
        for i in range(len(self.widths)):
            if self.gather:
                want = cref.all_gather([self.hx[s][i] for s in range(n)], chunks)
                for r in range(n):
                    same_bytes(self.full[r][i], want, f"tensor {i} rank {r}")
            else:
                want = cref.reduce_scatter([self.hf[s][i] for s in range(n)], chunks)
                for r in range(n):
                    same(self.shard[r][i].contiguous(), want[r], f"tensor {i} rank {r}")
        if not self.gather and self.whole:
            for r in range(n):
                assert bool((self.whole[r][:, :self.q_cols].view(torch.uint8) == 0x7B).all()), f"rank {r}'s Q columns of dQKV were written"


class Barrier(Call):
    kind = "barrier"

    def fill(self, seed):
        pass

    def enqueue(self, r, c, st):
        c.barrier(stream=st)

    def check(self):
        pass


KINDS = {
    "all_reduce": AllReduce,
    "all_reduce_fp8": AllReduceFp8,
    "all_reduce_staged_big": AllReduceStagedBig,
    "reduce_scatter": lambda g, rng: Move(g, rng, "reduce_scatter"),
    "all_gather": lambda g, rng: Move(g, rng, "all_gather"),
    "all_to_all": lambda g, rng: Move(g, rng, "all_to_all"),
    "broadcast": lambda g, rng: Rooted(g, rng, "broadcast"),
    "reduce": lambda g, rng: Rooted(g, rng, "reduce"),
    "generic": Generic,
    "all_reduce_host": Host,
    "all_gather_block_scaled": lambda g, rng: BlockScaled(g, rng, "all_gather"),
    "reduce_scatter_block_scaled": lambda g, rng: BlockScaled(g, rng, "reduce_scatter"),
    "all_reduce_block_scaled": lambda g, rng: BlockScaled(g, rng, "all_reduce"),
    "all_gather_quantized": lambda g, rng: Quantized(g, rng, "all_gather"),
    "reduce_scatter_quantized": lambda g, rng: Quantized(g, rng, "reduce_scatter"),
    "all_reduce_quantized": lambda g, rng: Quantized(g, rng, "all_reduce"),
    "all_reduce_rms_norm": lambda g, rng: RmsNorm(g, rng, False, False),
    "all_reduce_rms_norm_quantized": lambda g, rng: RmsNorm(g, rng, False, True),
    "reduce_scatter_rms_norm": lambda g, rng: RmsNorm(g, rng, True, False),
    "reduce_scatter_rms_norm_quantized": lambda g, rng: RmsNorm(g, rng, True, True),
    "all_to_all_v": lambda g, rng: AllToAllV(g, rng, False),
    "all_to_all_v_quantized": lambda g, rng: AllToAllV(g, rng, True),
    "all_to_all_v_combine": lambda g, rng: A2AVCombine(g, rng, False),
    "all_to_all_v_combine_quantized": lambda g, rng: A2AVCombine(g, rng, True),
    "expert_dispatch": lambda g, rng: Expert(g, rng, False, False),
    "expert_dispatch_quantized": lambda g, rng: Expert(g, rng, False, True),
    "expert_combine": lambda g, rng: Expert(g, rng, True, False),
    "expert_combine_quantized": lambda g, rng: Expert(g, rng, True, True),
    "send_recv_ring": SendRecv,
    "barrier": Barrier,
    "all_to_all_seq_to_heads": lambda g, rng: Ulysses(g, rng, True),
    "all_to_all_heads_to_seq": lambda g, rng: Ulysses(g, rng, False),
    "all_gather_context": lambda g, rng: Context(g, rng, True),
    "reduce_scatter_context": lambda g, rng: Context(g, rng, False),
}
KIND_NAMES = list(KINDS)
MULTI_OP = ("all_reduce_host", "all_reduce_staged_big")           # several dependent operations per rank in one call
NOT_IN_GRAPHS = ("all_reduce_host", "all_reduce_staged_big")        # host buffers and a 32 MiB staging round stay out of the captured window
SCRATCH_GROW = 1 << 21          # elements of the large quantised all-reduce of each random schedule (grows the FP8 scratch)


# ------------------------------------------------------------------------------------------------- schedules (no GPU needed)
def eulerian_circuit(k):
    """A closed walk over 0 .. k-1 (K^2 + 1 vertices) in which every ordered pair (a, b), a == b included, is adjacent exactly once:
    Hierholzer's algorithm on the complete directed graph with loops (every vertex has in- and out-degree k)."""
    nxt = [list(range(k - 1, -1, -1)) for _ in range(k)]          # unused out-edges, popped from the end: lowest first
    stack, walk = [0], []
    while stack:
        v = stack[-1]
        if nxt[v]:
            stack.append(nxt[v].pop())
        else:
            walk.append(stack.pop())
    return walk[::-1]


def windows_of(seq, size):
    """seq cut into windows of `size` calls; each window starts with the previous window's last element, so every adjacent pair of seq
    is adjacent inside one window."""
    return [seq[i:i + size] for i in range(0, max(1, len(seq) - 1), size - 1)]


def pair_schedule(kinds, size=WINDOW):
    return windows_of([kinds[i] for i in eulerian_circuit(len(kinds))], size)


def random_schedule(kinds, n, seed, calls=120):
    """Windows of steps: (kind, events before the call). Events: ("shape", kind, max_ctas, threads) or ("max_ctas", m) on every rank,
    ("delay", rank), and after the call ("rewrite", rank). One all_reduce_quantized step carries ("grow",): large enough to grow the
    quantisation scratch."""
    rng = np.random.default_rng(seed)
    steps = []
    grow_at = int(rng.integers(calls))
    for i in range(calls):
        kind = "all_reduce_quantized" if i == grow_at else kinds[int(rng.integers(len(kinds)))]
        ev = []
        u = rng.random()
        if u < 0.12:
            ev.append(("max_ctas", pick(rng, [1, 2, 3, 8, "default"])))
        elif u < 0.24:
            ev.append(("shape", pick(rng, ["p2p", "ll", "rooted"]), int(pick(rng, [0, 1, 2, 5])), int(pick(rng, [0, 128, 256, 512]))))
        if rng.random() < 0.3:
            ev.append(("delay", int(rng.integers(n))))
        if rng.random() < 0.3:
            ev.append(("rewrite", int(rng.integers(n))))
        if i == grow_at:
            ev.append(("grow",))
        steps.append((kind, tuple(ev)))
    out, i = [], 0
    while i < calls:
        w = int(rng.integers(8, 17))
        out.append(steps[i:i + w])
        i += w
    return out


# ------------------------------------------------------------------------------------------------- runner
def _skip(label, seed, w):
    if ONLY is None:
        return False
    return any(ONLY.get(k) not in (None, v) for k, v in (("label", label), ("seed", seed), ("window", w)))


def _stats(c):
    s = c.stats()
    return s["algo_calls"], s["staged_calls"]


def _enqueue(g, call, r):
    """Rank r's call on its stream; records the algorithms and staging rounds it counted."""
    c, st = g.comms[r], g.streams[r]
    a0, s0 = _stats(c)
    with torch.cuda.device(c.device):
        c.set_algo("auto")                                        # a kind that forces an algorithm sets it in enqueue
        call.enqueue(r, c, st)
    a1, s1 = _stats(c)
    return {k: a1[k] - a0[k] for k in a1 if a1[k] != a0[k]}, s1 - s0


def _record(call, per_rank):
    assert all(p == per_rank[0] for p in per_rank), f"ranks recorded different algorithms: {per_rank}"
    call.ran, call.staged = per_rank[0]


def default_ctas(g):
    """The grid cap a communicator starts with: the SMs divided among the ranks that share its GPU. Every rank's blocks of a barrier
    kernel must be resident at once, so a larger cap can leave a virtual rank's blocks waiting for SMs its peers spin on."""
    c = g.comms[0]
    return max(1, c.sm_count // sum(d.device == c.device for d in g.comms))


def _events(g, events, when, call):
    for ev in events:
        if ev[0] == "max_ctas" and when == "before":
            for c in g.comms:
                c.set_max_ctas(default_ctas(g) if ev[1] == "default" else ev[1])
        elif ev[0] == "shape" and when == "before":
            for c in g.comms:
                c.set_launch_shape(ev[1], ev[2], ev[3])
        elif ev[0] == "delay" and when == "before":
            with torch.cuda.device(g.comms[ev[1]].device), torch.cuda.stream(g.streams[ev[1]]):
                torch.cuda._sleep(SLEEP_CYCLES)
        elif ev[0] == "rewrite" and when == "after":
            r = ev[1]
            with torch.cuda.device(g.comms[r].device), torch.cuda.stream(g.streams[r]):
                for t in call.inputs[r]:
                    t.view(-1).view(torch.uint8).fill_(0xA5)             # after the call on this stream: its peers must be done reading


def _check_all(calls, label, steps0):
    for i, call in enumerate(calls):
        prev = calls[i - 1].desc() if i else "(start of window)"
        try:
            call.check()
        except AssertionError as e:
            raise AssertionError(f"{label}: step {steps0 + i}: {call.desc()} after {prev}: ran {call.ran} staged {call.staged}: {e}") from None


def run_window(g, rng, steps, label, step0, seed0, grow=SCRATCH_GROW):
    """One eager window: build every call, fill, sync; then op-major enqueue with the step events; one sync; then every check."""
    calls = []
    for kind, ev in steps:
        call = KINDS[kind](g, rng) if ("grow",) not in ev else Quantized(g, rng, "all_reduce", grow=grow)
        calls.append(call)
    try:
        for i, call in enumerate(calls):
            call.fill(seed0 + i)
        g.sync()
        window = lambda: "; ".join(f"{step0 + i}: {call.desc()} {ev}" for i, (call, (_, ev)) in enumerate(zip(calls, steps)))
        for i, ((kind, ev), call) in enumerate(zip(steps, calls)):
            try:
                _events(g, ev, "before", call)
                _record(call, [_enqueue(g, call, r) for r in range(g.n)])
                _events(g, ev, "after", call)
            except B200CollError as e:
                raise AssertionError(f"{label}: step {step0 + i} ({call.desc()}) refused: {e}; the window: {window()}") from None
        g.sync()
        try:
            g.check_async()
        except B200CollError as e:
            raise AssertionError(f"{label}: steps {step0} .. {step0 + len(calls) - 1}: {e}; the window: {window()}") from None
        _check_all(calls, label, step0)
    finally:
        g.sync()
        for call in calls:
            call.release()
        for c in g.comms:
            c.set_algo("auto")


def _group(torch_cuda, coll_mod, n, devices=None):
    return Group(torch_cuda, coll_mod, n, devices=devices, arena_mb=ARENA_MB, timeout_ms=TIMEOUT_MS)


def _reset_shapes(g):
    for c in g.comms:
        c.set_max_ctas(default_ctas(g))
        for k in ("p2p", "ll", "rooted"):
            c.set_launch_shape(k, 0, 0)


@pytest.mark.parametrize("n", [3, 4])
def test_every_ordered_pair(torch_cuda, coll_mod, n):
    """Schedule a: K^2 + 1 calls in which every ordered pair of kinds runs back to back once, in windows with no reset between them."""
    label = f"pairs n={n}"
    wins = pair_schedule(KIND_NAMES)
    with _group(torch_cuda, coll_mod, n) as g:
        step = 0
        for w, win in enumerate(wins):
            if not _skip(label, 0, w):
                run_window(g, np.random.default_rng([n, w]), [(k, ()) for k in win], f"{label} window {w}", step, 1000 * w)
            step += len(win) - 1


@pytest.mark.parametrize("seed", [11, 12])
@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_random_schedule(torch_cuda, coll_mod, n, seed):
    """Schedule b: seeded random calls with random parameters, launch shapes that grow and shrink, one rank held back by a delay
    kernel, and inputs overwritten on a rank's stream right after the call that read them."""
    label = f"random n={n}"
    with _group(torch_cuda, coll_mod, n) as g:
        kinds = KIND_NAMES if one_queue_each(g) else [k for k in KIND_NAMES if k not in MULTI_OP]
        step = 0
        try:
            for w, win in enumerate(random_schedule(kinds, n, seed)):
                if not _skip(label, seed, w):
                    run_window(g, np.random.default_rng([seed, n, w]), win, f"{label} seed {seed} window {w}", step, 7000 * w + seed)
                step += len(win)
        finally:
            _reset_shapes(g)


def test_random_schedule_real_devices(torch_cuda, coll_mod):
    """Schedule b on one rank per GPU: real peers reach the multicast barrier's per-block call counters and the NVLS paths."""
    nd = torch_cuda.cuda.device_count()
    if nd < 2:
        pytest.skip("needs >= 2 GPUs")
    label, seed = f"real devices n={nd}", 21
    with _group(torch_cuda, coll_mod, nd, devices=list(range(nd))) as g:
        step = 0
        for w, win in enumerate(random_schedule([k for k in KIND_NAMES if k != "all_reduce_host"], nd, seed, calls=60)):
            if not _skip(label, seed, w):
                run_window(g, np.random.default_rng([seed, w]), win, f"{label} window {w}", step, 5000 * w)
            step += len(win)


@pytest.mark.parametrize("n", [2, 4])
def test_graph_replay_between_eager_windows(torch_cuda, coll_mod, n):
    """Schedule c: a mixed window of 12 calls captured on each rank's stream, replayed 3 times with new inputs written on the stream
    first, with an eager mixed window between replays (sequence numbers, Lamport buffer and epochs differ at every replay) whose quantised
    all-reduce grows the scratch the captured quantised calls used."""
    label = f"graph n={n}"
    rng = np.random.default_rng(100 + n)
    kinds = [k for k in KIND_NAMES if k not in NOT_IN_GRAPHS]
    picked = ["all_reduce", "all_reduce_quantized", "expert_dispatch", "all_reduce_rms_norm"]
    picked += [kinds[int(i)] for i in rng.choice(len(kinds), size=8, replace=False)]
    with _group(torch_cuda, coll_mod, n) as g:
        calls = [KINDS[k](g, rng) for k in picked]
        try:
            for i, call in enumerate(calls):
                call.fill(i)
            g.sync()
            graphs = [torch.cuda.CUDAGraph() for _ in g.comms]
            per_rank = [[] for _ in calls]
            for r, c in enumerate(g.comms):                       # capture launches nothing, so rank-major order is safe here
                with torch.cuda.graph(graphs[r], stream=g.streams[r]):
                    for i, call in enumerate(calls):
                        per_rank[i].append(_enqueue(g, call, r))
            for call, pr in zip(calls, per_rank):
                _record(call, pr)
            for c in g.comms:
                c.set_algo("auto")
            for rep in range(3):
                for i, call in enumerate(calls):
                    call.fill(10000 * (rep + 1) + i)
                for r in range(n):
                    g.streams[r].wait_stream(torch.cuda.current_stream())
                for r in range(n):
                    with torch.cuda.stream(g.streams[r]):
                        graphs[r].replay()
                eager = [(str(k), ()) for k in rng.choice(KIND_NAMES, size=8)]
                eager.insert(int(rng.integers(len(eager) + 1)), ("all_reduce_quantized", (("grow",),)))
                if not _skip(label, 0, rep):
                    run_window(g, rng, eager, f"{label} eager window {rep}", 100 * rep, 50000 + rep, grow=(1 << 19) * (rep + 2))
                g.sync()
                g.check_async()
                _check_all(calls, f"{label} replay {rep}", 0)
        finally:
            g.sync()
            for call in calls:
                call.release()

