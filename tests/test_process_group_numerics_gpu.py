"""The `torch.distributed` backend "b200coll" on an H100 (`pytest -m gpu`): every route of parallel/process_group.py at 2, 3 and 4 ranks
(spawned processes sharing cuda:0), bit for bit against the order-exact reference of tests/coll_fp_reference.py and plain PyTorch on
the CPU.

Every rank builds all ranks' inputs from the seed and computes the reference itself. Outputs are filled with a byte pattern first and
sit between guard bytes that must keep it. Every check also reads the route the call took (the group's fast / fallback counters and
the communicator's algorithm, staging, generic-kernel and send counters), so a call that quietly went through the host fails although
its values are right; the summation order of a reduction comes from the algorithm the library recorded. A failed comparison is noted
and the rank carries on, so that the ranks stay in step and one run reports every failure."""
import os
import socket
import sys
import time
import traceback

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import coll_fp_reference as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
POISON = 0x7B
PAD = 64                                                 # guard elements on each side of an output (a multiple of 16 bytes for every type)
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
SUM, AVG, MIN, MAX, PRODUCT = dist.ReduceOp.SUM, dist.ReduceOp.AVG, dist.ReduceOp.MIN, dist.ReduceOp.MAX, dist.ReduceOp.PRODUCT


# ------------------------------------------------------------------------------------------------- processes
def _free_port() -> int:
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _run(fn, world, timeout=600):
    """Spawn `world` ranks, collect one result each, and leave no process behind whatever happened."""
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_entry, args=(fn, r, world, port, q)) for r in range(world)]
    results = []
    try:
        for p in procs:
            p.start()
        deadline = time.monotonic() + timeout
        while len(results) < world and time.monotonic() < deadline:
            try:
                results.append(q.get(timeout=1.0))
            except Exception:                          # queue.Empty: keep waiting while somebody may still report
                if all(not p.is_alive() for p in procs) and q.empty():
                    break
            if any(r[1] != "ok" for r in results):     # a rank failed: its peers may be waiting for it
                break
        for p in procs:
            p.join(10 if len(results) == world and all(r[1] == "ok" for r in results) else 0.1)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
            p.join()
    results.sort()
    bad = "\n".join(f"rank {r[0]}: {r[2]}" for r in results if r[1] != "ok")
    assert len(results) == world and not bad, f"{len(results)} of {world} ranks reported, exit codes {[p.exitcode for p in procs]}\n{bad}"
    return results


def _entry(fn, rank, world, port, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), B200COLL_TIMEOUT_MS="20000", B200COLL_ARENA_MB="512")
        from container_engine_accelerators_b200.parallel import process_group  # noqa: F401  (registers the backend)
        dist.init_process_group("b200coll", rank=rank, world_size=world)
        out = fn(rank, world)
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok", out))
    except Exception as e:
        q.put((rank, "error", traceback.format_exc() + repr(e)))
        sys.exit(1)


# ------------------------------------------------------------------------------------------------- one rank's tools
class Ctx:
    def __init__(self, rank, world, pg=None, members=None):
        self.rank, self.world = rank, world
        self.pg = pg if pg is not None else dist.group.WORLD
        self.group = pg                                  # what dist.* calls take as group=
        self.members = members or list(range(world))     # global ranks of the group, for point to point
        self.errors = []

    # --- routes
    def snap(self):
        s = self.pg.comm.stats()
        return {"fast": self.pg.fast_calls, "fallback": self.pg.fallback_calls, "staged": s["staged_calls"], "generic": s["generic_launches"],
                "sends": s["p2p_sends"], "algo": dict(s["algo_calls"])}

    def delta(self, before):
        """What the calls since `before` did, after they have finished and the watchdog has been asked."""
        if DEV == "cuda":
            torch.cuda.synchronize()
            self.pg.comm.check_async_error()
        now = self.snap()
        d = {k: now[k] - before[k] for k in before if k != "algo"}
        d["algo"] = {k: v - before["algo"][k] for k, v in now["algo"].items() if v != before["algo"][k]}
        return d

    def expect(self, d, what, **want):
        for k, v in want.items():
            if d[k] != v:
                self.errors.append(f"{what} rank {self.rank}: route: {k} is {d[k]}, expected {v} (all: {d})")

    def same(self, got, want, what, nan_payloads=False):
        try:
            R.assert_same(got.detach().cpu(), want, f"{what} rank {self.rank}", nan_payloads=nan_payloads)
        except AssertionError as e:
            self.errors.append(str(e))

    def check(self, ok, what):
        if not ok:
            self.errors.append(f"{what} rank {self.rank}")

    # --- buffers
    def plain(self, numel, dt):
        return torch.empty(numel, dtype=dt, device=DEV)

    def arena(self, numel, dt):
        return self.pg.empty(numel, dt)

    def release(self, t):
        if getattr(t, "_b200coll_buf", None) is not None:
            self.pg.comm.release(t)

    def guarded(self, numel, dt, alloc=None):
        """A poisoned output of `numel` elements between PAD poisoned guard elements: (output, whole buffer)."""
        buf = (alloc or self.plain)(numel + 2 * PAD, dt)
        poison(buf)
        return buf[PAD:PAD + numel], buf

    def guards_kept(self, buf, what):
        b = buf.view(torch.uint8).cpu()
        g = PAD * buf.element_size()
        self.check(bool((b[:g] == POISON).all()) and bool((b[-g:] == POISON).all()), f"{what}: bytes outside the output were written")

    def put(self, x, alloc=None):
        t = (alloc or self.plain)(x.numel(), x.dtype)
        t.view(torch.uint8).copy_(x.contiguous().view(torch.uint8))      # bytes: no conversion can touch a NaN payload
        return t


def poison(t):
    t.view(torch.uint8).fill_(POISON)


def bits(t):
    return t.contiguous().view(torch.uint8)


def one_algo(c, d, what):
    c.check(len(d["algo"]) == 1, f"{what}: algorithms recorded {d['algo']}")
    return next(iter(d["algo"]), "twoshot")


def sum_order(c, d, dt, count, what):
    """The order model of an all-reduce from what the library recorded."""
    n = c.pg.size()
    a = one_algo(c, d, what)
    if dt in R.FP8_MAX or a in ("ll", "ll2", "oneshot"):
        return list(range(n))
    c.check(a == "twoshot", f"{what}: no order model for {a}")
    if d["staged"]:
        return ("staged", n, R.vec_elems(dt), count, R.staged_chunk(R.esize(dt), R.esize(dt), n, "all_reduce"))
    return ("owner", n, R.vec_elems(dt), count)


def scale_of(op, n):
    return R.avg_scale(1.0, n) if op == AVG else 1.0


def counts_for(dt, n):
    e, ll = R.vec_elems(dt), R.LL_ONESHOT_MAX_BYTES // R.esize(dt)
    return [1, e - 1, e + 1, 1003, ll + e]


def int_inputs(n, count, dt, seed, small=False):
    g = torch.Generator().manual_seed(seed)
    if dt == torch.float64:
        return [torch.randn(count, generator=g, dtype=torch.float64) * 2.0 ** torch.randint(-30, 30, (count,), generator=g) for _ in range(n)]
    if dt == torch.bool:
        return [torch.randint(0, 2, (count,), generator=g).bool() for _ in range(n)]
    if small:
        lo, hi = (0 if dt == torch.uint8 else -3), 4
    elif dt == torch.int64:
        lo, hi = -(1 << 62), 1 << 62                                       # far past 2^32
    else:
        lo, hi = torch.iinfo(dt).min, torch.iinfo(dt).max + 1
    xs = [torch.randint(lo, hi, (count,), generator=g, dtype=torch.int64).to(dt) for _ in range(n)]
    if dt == torch.int64 and not small:
        for r, x in enumerate(xs):
            x[r::7] = -1                                                   # all ones: the word the Lamport path would rewrite
    return xs


def generic_ref(xs, op):
    """Rank order from rank 0's value, in the accumulator type (fp32 for bf16); min / max propagate NaN and keep the lower rank on a tie."""
    wide = xs[0].dtype in (BF16, F16)
    acc = xs[0].float() if wide else xs[0].clone()
    for x in xs[1:]:
        b = x.float() if wide else x
        if op == SUM:
            acc = acc + b
        elif op == PRODUCT:
            acc = acc * b
        elif op == MIN:
            acc = torch.where((b < acc) | (b != b), b, acc)
        else:
            acc = torch.where((b > acc) | (b != b), b, acc)
    return acc.to(xs[0].dtype)


# ------------------------------------------------------------------------------------------------- reductions
def check_all_reduce(c):
    n, r = c.world, c.rank
    for dt in (F32, BF16, F16):
        for count in counts_for(dt, n) + ([R.LL_ONESHOT_MAX_BYTES * n // R.esize(dt) + 1003] if dt == BF16 else []):
            xs = R.gen_inputs(n, count, dt, seed=11 * n + count % 89, device="cpu")
            for op in (SUM, AVG):
                for where in ("plain", "arena"):
                    what = f"all_reduce n={n} {dt} count={count} op={op} {where}"
                    t = c.put(xs[r], c.arena if where == "arena" else None)
                    b = c.snap()
                    dist.all_reduce(t, op=op)
                    d = c.delta(b)
                    c.expect(d, what, fast=1, fallback=0, generic=0)
                    if where == "arena":
                        c.expect(d, what, staged=0)
                    elif count * R.esize(dt) > R.LL_ONESHOT_MAX_BYTES * n:
                        c.expect(d, what, staged=1)                          # a plain tensor too big for the Lamport paths is staged
                    c.same(t, R.ref_reduce(xs, sum_order(c, d, dt, count, what), scale_of(op, n), dt), what)
                    c.release(t)
    for dt in (E4M3, E5M2):
        for count in (1, 15, 17, 1003):
            xs = R.gen_inputs(n, count, dt, seed=5 * n + count, device="cpu")
            what = f"all_reduce n={n} {dt} count={count}"
            t = c.put(xs[r])
            b = c.snap()
            dist.all_reduce(t)
            d = c.delta(b)
            c.expect(d, what, fast=1, fallback=0, generic=0)
            c.same(t, R.ref_reduce(xs, sum_order(c, d, dt, count, what), 1.0, dt), what)
    # tensors created under the group's memory pool are arena tensors: not staged even when far past the Lamport sizes
    count = R.LL_ONESHOT_MAX_BYTES * n // 2 + 1003
    xs = R.gen_inputs(n, count, BF16, seed=3, device="cpu")
    with torch.cuda.use_mem_pool(c.pg.mem_pool()):
        t = torch.empty(count, dtype=BF16, device=DEV)
    t.copy_(xs[r])
    c.check(c.pg.comm.is_symmetric(t), "a tensor from the memory pool is not in the arena")
    b = c.snap()
    dist.all_reduce(t, op=AVG)
    d = c.delta(b)
    c.expect(d, "all_reduce pooled", fast=1, fallback=0, staged=0)
    c.same(t, R.ref_reduce(xs, sum_order(c, d, BF16, count, "all_reduce pooled"), scale_of(AVG, n), BF16), "all_reduce pooled")
    del t


def check_generic_reductions(c):
    n, r = c.world, c.rank
    for dt in (BF16, torch.int8, torch.uint8, torch.int32, torch.int64, torch.float64):
        e = 16 // R.esize(dt)
        for op in (MIN, MAX, PRODUCT):
            for count in (1, e - 1, e + 1, 1003):
                if dt == BF16:
                    xs = R.gen_inputs(n, count, dt, seed=count + n, device="cpu")
                    if op == PRODUCT:                                          # keep products finite and inexact
                        xs = [(x.float().abs().clamp(0.5, 2.0) * torch.where(x.float() < 0, -1.0, 1.0)).to(dt) for x in xs]
                else:
                    xs = int_inputs(n, count, dt, seed=count + n, small=op == PRODUCT)
                what = f"all_reduce n={n} {dt} op={op} count={count}"
                t = c.put(xs[r])
                b = c.snap()
                dist.all_reduce(t, op=op)
                d = c.delta(b)
                c.expect(d, what, fast=1, fallback=0, generic=1, algo={"twoshot": 1})      # int64 max through Gloo would be right, and wrong
                c.same(t, generic_ref(xs, op), what)
    # avg of integers is not a library reduction: Gloo on every rank, the quotient toward zero
    xs = [x // 4 for x in int_inputs(n, 1003, torch.int32, seed=n)]
    t = c.put(xs[r])
    b = c.snap()
    dist.all_reduce(t, op=AVG)
    d = c.delta(b)
    c.expect(d, "all_reduce int32 avg", fast=0, fallback=1, algo={})
    c.same(t, torch.div(sum(x.long() for x in xs), n, rounding_mode="trunc").to(torch.int32), "all_reduce int32 avg")
    # a list of two tensors, and the coalesced entry point: one library all-reduce per tensor
    for entry in ("allreduce", "allreduce_coalesced"):
        xa, xb = R.gen_inputs(n, 1003, F32, seed=21, device="cpu"), R.gen_inputs(n, 77, BF16, seed=22, device="cpu")
        ta, tb = c.put(xa[r]), c.put(xb[r])
        opts = dist.AllreduceOptions() if entry == "allreduce" else dist.AllreduceCoalescedOptions()
        opts.reduceOp = AVG
        b = c.snap()
        getattr(c.pg, entry)([ta, tb], opts).wait()
        d = c.delta(b)
        c.expect(d, entry, fast=1, fallback=0)
        c.check(sum(d["algo"].values()) == 2, f"{entry}: {d['algo']}")
        a = set(d["algo"])
        c.check(a <= {"ll", "ll2", "oneshot"}, f"{entry}: small tensors ran {a}")
        c.same(ta, R.ref_reduce(xa, list(range(n)), scale_of(AVG, n), F32), f"{entry} first")
        c.same(tb, R.ref_reduce(xb, list(range(n)), scale_of(AVG, n), BF16), f"{entry} second")


def check_reduce(c):
    n, r = c.world, c.rank
    for dt, count, op in ((F32, 1003, SUM), (BF16, 9, AVG), (E5M2, 1003, SUM)):
        xs = R.gen_inputs(n, count, dt, seed=count + 7 * n, device="cpu")
        for root in range(n):
            what = f"reduce n={n} {dt} count={count} op={op} root={root}"
            t = c.put(xs[r])
            b = c.snap()
            dist.reduce(t, dst=root, op=op)
            d = c.delta(b)
            c.expect(d, what, fast=1, fallback=0, generic=0, algo={"twoshot": 1})
            if r == root:
                c.same(t, R.ref_reduce(xs, list(range(n)), scale_of(op, n), dt), what)
            else:
                c.same(t, xs[r], what + " (not the root: its tensor must be untouched)", nan_payloads=True)
    xs = int_inputs(n, 1003, torch.int64, seed=n)
    for root in range(n):
        t = c.put(xs[r])
        b = c.snap()
        dist.reduce(t, dst=root, op=MAX)
        d = c.delta(b)
        c.expect(d, f"reduce int64 max root={root}", fast=1, fallback=0, generic=1)
        c.same(t, generic_ref(xs, MAX) if r == root else xs[r], f"reduce int64 max root={root}")


def check_reduce_scatter(c):
    n, r = c.world, c.rank
    for dt in (F32, BF16, E4M3):
        e, ll = R.vec_elems(dt), R.LL_ONESHOT_MAX_BYTES // R.esize(dt)
        for count in (e, 37 * e, ll + e):
            xs = R.gen_inputs(n, count * n, dt, seed=count % 97 + n, device="cpu")
            for op in (SUM, AVG):
                for form in ("tensor", "list"):
                    if form == "list" and count > 37 * e:
                        continue
                    what = f"reduce_scatter {form} n={n} {dt} count={count} op={op}"
                    out, buf = c.guarded(count, dt)
                    src = c.put(xs[r])
                    b = c.snap()
                    if form == "tensor":
                        dist.reduce_scatter_tensor(out, src, op=op)
                    else:
                        dist.reduce_scatter(out, list(src.chunk(n)), op=op)
                    d = c.delta(b)
                    c.expect(d, what, fast=1, fallback=0, generic=0)
                    a = one_algo(c, d, what)
                    order = list(range(n)) if a == "ll" or dt in R.FP8_MAX else ("rotate", r)
                    c.check(a in ("ll", "twoshot"), f"{what}: ran {a}")
                    c.same(out, R.ref_reduce([x[r * count:(r + 1) * count] for x in xs], order, scale_of(op, n), dt), what)
                    c.guards_kept(buf, what)
    # max, and integers: the all-reduce-and-slice path on the generic kernel; a slice that is not whole vectors goes the same way
    for dt, op, count in ((F32, MAX, 64), (torch.int32, SUM, 64), (torch.int32, SUM, 3), (BF16, SUM, 5)):
        xs = R.gen_inputs(n, count * n, dt, seed=count, device="cpu") if dt.is_floating_point else [x // 8 for x in int_inputs(n, count * n, dt, seed=count)]
        what = f"reduce_scatter_tensor n={n} {dt} count={count} op={op}"
        out, buf = c.guarded(count, dt)
        b = c.snap()
        dist.reduce_scatter_tensor(out, c.put(xs[r]), op=op)
        d = c.delta(b)
        fused = dt == BF16
        c.expect(d, what, fast=1, fallback=0, generic=0 if fused else 1)
        want = R.ref_reduce(xs, sum_order(c, d, dt, count * n, what), 1.0, dt) if fused else generic_ref(xs, op)
        c.same(out, want[r * count:(r + 1) * count], what)
        c.guards_kept(buf, what)


# ------------------------------------------------------------------------------------------------- data movement
def word_payloads(n, dt, count, seed):
    if dt.is_floating_point:
        xs = R.gen_inputs(n, count, dt, seed, device="cpu")
        if dt == F32:
            for pos, word in R.LL_WORDS:                                    # the Lamport marker and its sanitized form, on every rank
                if pos < count:
                    for x in xs:
                        x.view(torch.int32)[pos] = word - (1 << 32) if word >= 1 << 31 else word
        return xs
    return int_inputs(n, count, dt, seed)


def check_broadcast(c):
    n, r = c.world, c.rank
    cases = [(F32, k, True) for k in (1, 3, 5, 1003)] + [(torch.int64, 1, True), (torch.int64, 1003, True), (torch.bool, 1004, True), (torch.bool, 1002, True),
                                                         (torch.uint8, 1003, False), (BF16, 1003, True), (E4M3, 64, True)]
    for dt, count, lib in cases:
        xs = word_payloads(n, dt, count, seed=count + n)
        for root in range(n):
            what = f"broadcast n={n} {dt} count={count} root={root}"
            out, buf = c.guarded(count, dt)
            if r == root:
                bits(out).copy_(bits(xs[r]))
            b = c.snap()
            dist.broadcast(out, src=root)
            d = c.delta(b)
            c.expect(d, what, fast=1 if lib else 0, fallback=0 if lib else 1, **({"algo": {"twoshot": 1}} if lib else {"algo": {}}))
            c.same(bits(out), bits(xs[root]), what)
            c.guards_kept(buf, what)


def check_all_gather(c):
    n, r = c.world, c.rank
    ll = R.LL_ONESHOT_MAX_BYTES
    cases = [(F32, 4, "float"), (F32, 37 * 4, "float"), (BF16, 37 * 8, "float"), (F32, ll // 4 + 4, "float"),
             (torch.int64, 1002, "words"), (torch.bool, 1008, "words"), (E4M3, 1008, "words"), (E5M2, 16, "words"), (F32, 3, "gloo"), (torch.int64, 1001, "gloo")]
    for dt, count, route in cases:
        xs = word_payloads(n, dt, count, seed=count + 3 * n)
        what = f"all_gather_into_tensor n={n} {dt} count={count}"
        out, buf = c.guarded(count * n, dt)
        b = c.snap()
        dist.all_gather_into_tensor(out, c.put(xs[r]))
        d = c.delta(b)
        if route == "gloo":
            c.expect(d, what, fast=0, fallback=1, algo={})
        else:
            c.expect(d, what, fast=1, fallback=0)
            if route == "words":
                c.expect(d, what, algo={"twoshot": 1})                       # the barrier-based kernel: the Lamport one rewrites marker words
        exact = route != "float" or one_algo(c, d, what) == "twoshot"
        want = torch.cat(xs) if exact else torch.cat([R.ll_move(x) for x in xs])
        c.same(bits(out), bits(want), what)
        c.guards_kept(buf, what)
    # list form: outputs of a 2-D shape on the library; integers through the host
    for dt, shape, lib in ((F32, (5, 8), True), (BF16, (3, 8), True), (torch.int64, (5, 8), False), (F32, (3, 3), False)):
        count = shape[0] * shape[1]
        xs = word_payloads(n, dt, count, seed=count + n)
        what = f"all_gather list n={n} {dt} {shape}"
        outs = [c.guarded(count, dt) for _ in range(n)]
        b = c.snap()
        dist.all_gather([o.view(shape) for o, _ in outs], c.put(xs[r]).view(shape))
        d = c.delta(b)
        c.expect(d, what, fast=1 if lib else 0, fallback=0 if lib else 1)
        for s, (o, buf) in enumerate(outs):
            want = R.ll_move(xs[s]) if lib and one_algo(c, d, what) != "twoshot" else xs[s]
            c.same(bits(o), bits(want), f"{what} from {s}")
            c.guards_kept(buf, what)


def a2a_want(xs, n, r, count):
    return torch.cat([xs[s][r * count:(r + 1) * count] for s in range(n)])


def check_all_to_all(c):
    n, r = c.world, c.rank
    for dt, count, route in ((F32, 37 * 4, "float"), (BF16, 8, "float"), (F32, R.LL_ONESHOT_MAX_BYTES // 4 + 4, "float"), (torch.int64, 1002, "words"),
                             (E5M2, 32, "words"), (F32, 3, "gloo")):
        xs = word_payloads(n, dt, count * n, seed=count + 5 * n)
        what = f"all_to_all_single n={n} {dt} count={count}"
        out, buf = c.guarded(count * n, dt)
        b = c.snap()
        dist.all_to_all_single(out, c.put(xs[r]))
        d = c.delta(b)
        if route == "gloo":
            c.expect(d, what, fast=0, fallback=1, algo={})
        else:
            c.expect(d, what, fast=1, fallback=0)
            if route == "words":
                c.expect(d, what, algo={"twoshot": 1})
        exact = route != "float" or one_algo(c, d, what) == "twoshot"
        want = a2a_want(xs, n, r, count)
        c.same(bits(out), bits(want if exact else R.ll_move(want)), what)
        c.guards_kept(buf, what)
    # in place: the library refuses it, so every rank takes the host route
    xs = word_payloads(n, F32, 16 * n, seed=n)
    t = c.put(xs[r])
    b = c.snap()
    dist.all_to_all_single(t, t)
    d = c.delta(b)
    c.expect(d, "all_to_all_single in place", fast=0, fallback=1, algo={})
    c.same(bits(t), bits(a2a_want(xs, n, r, 16)), "all_to_all_single in place")
    # list form
    xs = word_payloads(n, F32, 64 * n, seed=2 * n)
    outs = [c.guarded(64, F32) for _ in range(n)]
    src = c.put(xs[r])
    b = c.snap()
    dist.all_to_all([o for o, _ in outs], list(src.chunk(n)))
    d = c.delta(b)
    c.expect(d, "all_to_all list", fast=1, fallback=0)
    for s, (o, buf) in enumerate(outs):
        want = xs[s][r * 64:(r + 1) * 64]
        c.same(bits(o), bits(want if one_algo(c, d, "all_to_all list") == "twoshot" else R.ll_move(want)), f"all_to_all list from {s}")
        c.guards_kept(buf, "all_to_all list")


def uneven(c, matrix, cols, dt, what, lib=True, spare=0, layout=None, give=("in", "out")):
    """all_to_all_single with matrix[src][dst] rows of `cols` elements. layout: (rank, "misaligned" | "strided") for that rank's tensors."""
    n, r = c.world, c.rank
    what = f"all_to_all_single uneven n={n} {what} {dt} cols={cols}"
    rows = [sum(m) for m in matrix]
    data = [x.view(-1, cols)[:rows[s]] for s, x in enumerate(R.gen_inputs(n, max(1, max(rows)) * cols, dt, seed=cols + n + sum(rows), device="cpu"))]
    got = sum(matrix[s][r] for s in range(n))
    odd = layout is not None and layout[0] == r
    if odd and layout[1] == "strided":
        src = torch.empty(rows[r], cols, 2, dtype=dt, device=DEV)[..., 0]
        base = torch.empty(got + spare + 2, cols, 2, dtype=dt, device=DEV)
        poison(base)
        out = base[1:1 + got + spare, :, 0]
    else:
        shift = 1 if odd else 0                                             # one element past an aligned start
        src = torch.empty(rows[r] * cols + shift, dtype=dt, device=DEV)[shift:].view(rows[r], cols)
        base = torch.empty((got + spare + 2) * cols + shift, dtype=dt, device=DEV)
        poison(base)
        out = base[shift + cols:shift + (1 + got + spare) * cols].view(got + spare, cols)
    src.copy_(data[r])
    off = [sum(matrix[s][:r]) for s in range(n)]
    want = torch.cat([data[s][off[s]:off[s] + matrix[s][r]] for s in range(n)] + [torch.empty(0, cols, dtype=dt)])
    b = c.snap()
    dist.all_to_all_single(out, src, [matrix[s][r] for s in range(n)] if "out" in give else None, list(matrix[r]) if "in" in give else None)
    d = c.delta(b)
    if lib:
        c.expect(d, what, fast=1, fallback=0, algo={"twoshot": 1})
    else:
        c.expect(d, what, fast=0, fallback=1, algo={})
    c.same(bits(out[:got]), bits(want), what, nan_payloads=True)
    mask = torch.ones(base.shape, dtype=torch.bool)
    if odd and layout[1] == "strided":
        mask[1:1 + got, :, 0] = False
        kept = bits(base.cpu()).view(*base.shape, -1)[mask]
    else:
        mask[shift + cols:shift + (1 + got) * cols] = False
        kept = bits(base.cpu()).view(base.numel(), -1)[mask]
    c.check(bool((kept == POISON).all()), f"{what}: rows past the received ones, or bytes around the output, were written")


def skewed(n):
    """A few hot experts: most rows go to rank 0, some pairs exchange nothing."""
    return [[(5 * s + 3 * d) % 4 * (6 if d == 0 else 1) for d in range(n)] for s in range(n)]


def check_all_to_all_uneven(c):
    n = c.world
    silent = [[0] * n if s == 1 else [s + d + 1 for d in range(n)] for s in range(n)]
    deaf = [[0 if d == n - 1 else 2 * s + d + 1 for d in range(n)] for s in range(n)]
    self_only = [[3 + s if s == d else 0 for d in range(n)] for s in range(n)]
    uneven(c, skewed(n), 16, F32, "skewed")
    uneven(c, skewed(n), 8, BF16, "skewed", spare=3)
    uneven(c, skewed(n), 24, BF16, "skewed")
    uneven(c, silent, 8, F32, "a rank that sends nothing", spare=1)
    uneven(c, deaf, 8, F16, "a rank that receives nothing")
    uneven(c, self_only, 4, F32, "rows to self only")
    uneven(c, skewed(n), 3, F32, "rows that are not whole vectors", lib=False)
    uneven(c, silent, 3, F32, "rows that are not whole vectors, a silent rank", lib=False)
    # receive scratch of two size classes, and the first again
    small, large = [[1] * n for _ in range(n)], [[300 + s] * n for s in range(n)]
    for m, name in ((small, "small"), (large, "large"), (small, "small again")):
        uneven(c, m, 64, F32, f"scratch {name}")
    even = [[2] * n for _ in range(n)]
    uneven(c, even, 8, F32, "only the input splits given", give=("in",))
    uneven(c, even, 8, F32, "only the output splits given", give=("out",))


# ------------------------------------------------------------------------------------------------- point to point
def check_point_to_point(c):
    n, r = c.world, c.rank
    g = lambda k: c.members[k]                                              # group rank -> global rank (dist.send / recv take global ranks)
    xs = word_payloads(n, F32, 1003, seed=n)
    # gather / scatter at every root
    for root in range(n):
        what = f"gather n={n} root={root}"
        outs = [c.guarded(1003, F32) for _ in range(n)] if r == root else None
        b = c.snap()
        dist.gather(c.put(xs[r]), [o for o, _ in outs] if outs else None, dst=g(root), group=c.group)
        d = c.delta(b)
        c.expect(d, what, fast=1, fallback=0, sends=0 if r == root else 1)    # the root's own block is a local copy
        for s, (o, buf) in enumerate(outs or []):
            c.same(bits(o), bits(xs[s]), f"{what} from {s}")
            c.guards_kept(buf, what)
        what = f"scatter n={n} root={root}"
        out, buf = c.guarded(1003, F32)
        b = c.snap()
        dist.scatter(out, [c.put(torch.roll(xs[s], root + 1)) for s in range(n)] if r == root else None, src=g(root), group=c.group)
        d = c.delta(b)
        c.expect(d, what, fast=1, fallback=0, sends=n - 1 if r == root else 0)
        c.same(bits(out), bits(torch.roll(xs[r], root + 1)), what)
        c.guards_kept(buf, what)
    # blocking send / recv around the ring, one pair at a time; the receiver's tensor is strided, then the sender's misaligned
    for s in range(n):
        dst = (s + 1) % n
        for count, side in ((1003, "recv strided"), (1002, "send misaligned")):
            what = f"send {s} -> {dst} {side}"
            b = c.snap()
            if r == s:
                t = torch.empty(count + 1, dtype=F32, device=DEV)[1:] if side == "send misaligned" else torch.empty(count, dtype=F32, device=DEV)
                t.copy_(xs[s][:count])
                dist.send(t, g(dst), group=c.group)
            if r == dst:
                base = torch.empty(count, 2, dtype=F32, device=DEV)
                poison(base)
                out = base[:, 0] if side == "recv strided" else base.view(-1)[:count]
                dist.recv(out, g(s), group=c.group)
            d = c.delta(b)
            c.expect(d, what, fast=int(r == s) + int(r == dst), fallback=0, sends=int(r == s))
            if r == dst:
                c.same(bits(out), bits(xs[s][:count]), what)
                rest = base[:, 1] if side == "recv strided" else base.view(-1)[count:]
                c.check(bool((bits(rest.cpu()) == POISON).all()), f"{what}: bytes outside the received tensor were written")
    # isend + irecv ring: one grouped kernel per rank, no deadlock; then batch_isend_irecv the other way round
    right, left = (r + 1) % n, (r - 1) % n
    out, buf = c.guarded(1003, F32)
    b = c.snap()
    reqs = [dist.isend(c.put(xs[r]), g(right), group=c.group), dist.irecv(out, g(left), group=c.group)]
    for q in reqs:
        q.wait()
    d = c.delta(b)
    c.expect(d, "isend / irecv ring", fast=2, fallback=0, sends=1)
    c.same(bits(out), bits(xs[left]), "isend / irecv ring")
    c.guards_kept(buf, "isend / irecv ring")
    big = R.gen_inputs(n, (1 << 20) + 3, BF16, seed=n, device="cpu")
    out, buf = c.guarded((1 << 20) + 3, BF16)
    b = c.snap()
    for q in dist.batch_isend_irecv([dist.P2POp(dist.isend, c.put(big[r]), g(left), group=c.group), dist.P2POp(dist.irecv, out, g(right), group=c.group)]):
        q.wait()
    d = c.delta(b)
    c.expect(d, "batch_isend_irecv", fast=2, fallback=0, sends=1)
    c.same(bits(out), bits(big[right]), "batch_isend_irecv")
    c.guards_kept(buf, "batch_isend_irecv")
    # a queued isend keeps its place before the next collective
    out, buf = c.guarded(1003, F32)
    ar = R.gen_inputs(n, 1003, F32, seed=9, device="cpu")
    t = c.put(ar[r])
    b = c.snap()
    reqs = [dist.isend(c.put(xs[r]), g(right), group=c.group), dist.irecv(out, g(left), group=c.group)]
    dist.all_reduce(t, group=c.group)
    for q in reqs:
        q.wait()
    d = c.delta(b)
    c.expect(d, "isend, then a collective", fast=3, fallback=0, sends=1)
    c.same(bits(out), bits(xs[left]), "isend, then a collective: the message")
    c.same(t, R.ref_reduce(ar, sum_order(c, d, F32, 1003, "isend, then a collective"), 1.0, F32), "isend, then a collective: the sum")


# ------------------------------------------------------------------------------------------------- ordering, layout, sub-groups
def check_two_streams(c):
    """Collectives issued from two streams back to back: the group orders them, one at a time per communicator. Every rank holds the
    same value after the first round, so each later round is that value added N times in fp32, whatever the order."""
    n, r = c.world, c.rank
    side = torch.cuda.Stream()
    a = torch.full((1 << 18,), float(r + 1), device=DEV)
    bb = torch.full((1 << 18,), 10.0 * (r + 1), device=DEV)
    torch.cuda.synchronize()
    b = c.snap()
    for _ in range(20):
        dist.all_reduce(a)
        with torch.cuda.stream(side):
            dist.all_reduce(bb)
    d = c.delta(b)
    c.expect(d, "two streams", fast=40, fallback=0)
    for t, first in ((a, 1.0), (bb, 10.0)):
        want = torch.tensor(first * n * (n + 1) / 2, dtype=F32)
        for _ in range(19):
            acc = torch.zeros((), dtype=F32)
            for _ in range(n):
                acc = acc + want
            want = acc
        c.same(t, want.expand(1 << 18).contiguous(), f"two streams n={n} (starting at {first})")


def check_layout_differs_by_rank(c):
    """Only rank 1's tensors are misaligned or strided. Every rank still runs the library route, and the results are the reference."""
    n, r = c.world, c.rank

    def laid(x, layout, fill=True):
        """x's values in a tensor that, on rank 1, starts one element past an aligned address or is a column of a wider tensor."""
        if r != 1:
            t = torch.empty(x.numel(), dtype=x.dtype, device=DEV)
        elif layout == "misaligned":
            t = torch.empty(x.numel() + 1, dtype=x.dtype, device=DEV)[1:]
        else:
            t = torch.empty(x.numel(), 2, dtype=x.dtype, device=DEV)[:, 0]
        if fill:
            t.copy_(x)
        else:
            t.fill_(0)
        return t

    for layout in ("misaligned", "strided"):
        for dt, op in ((F32, SUM), (BF16, AVG)):
            xs = R.gen_inputs(n, 1003, dt, seed=n, device="cpu")
            what = f"{layout} on rank 1: all_reduce {dt}"
            t = laid(xs[r], layout)
            b = c.snap()
            dist.all_reduce(t, op=op)
            d = c.delta(b)
            c.expect(d, what, fast=1, fallback=0)
            c.same(t, R.ref_reduce(xs, sum_order(c, d, dt, 1003, what), scale_of(op, n), dt), what)
        xs = int_inputs(n, 1003, torch.int64, seed=n)
        t = laid(xs[r], layout)
        b = c.snap()
        dist.all_reduce(t, op=MAX)
        d = c.delta(b)
        c.expect(d, f"{layout} on rank 1: all_reduce int64 max", fast=1, fallback=0, generic=1)
        c.same(t, generic_ref(xs, MAX), f"{layout} on rank 1: all_reduce int64 max")
        for root in (0, 1):
            t = laid(xs[r], layout)
            b = c.snap()
            dist.broadcast(t, src=root)
            d = c.delta(b)
            c.expect(d, f"{layout} on rank 1: broadcast from {root}", fast=1, fallback=0, algo={"twoshot": 1})
            c.same(t, xs[root], f"{layout} on rank 1: broadcast from {root}")
            fx = R.gen_inputs(n, 1003, F32, seed=root, device="cpu")
            t = laid(fx[r], layout)
            b = c.snap()
            dist.reduce(t, dst=root)
            d = c.delta(b)
            c.expect(d, f"{layout} on rank 1: reduce to {root}", fast=1, fallback=0)
            c.same(t, R.ref_reduce(fx, list(range(n)), 1.0, F32) if r == root else fx[r], f"{layout} on rank 1: reduce to {root}")
        for dt, route in ((F32, "float"), (torch.int64, "words")):
            count = 64
            xs = word_payloads(n, dt, count * n, seed=n + 1)
            what = f"{layout} on rank 1: all_gather_into_tensor {dt}"
            out = laid(torch.zeros(count * n, dtype=dt), layout, fill=False)
            b = c.snap()
            dist.all_gather_into_tensor(out, laid(xs[r][:count], layout))
            d = c.delta(b)
            c.expect(d, what, fast=1, fallback=0)
            want = torch.cat([x[:count] for x in xs])
            c.same(bits(out), bits(want if one_algo(c, d, what) == "twoshot" else R.ll_move(want)), what)
            what = f"{layout} on rank 1: all_to_all_single {dt}"
            out = laid(torch.zeros(count * n, dtype=dt), layout, fill=False)
            b = c.snap()
            dist.all_to_all_single(out, laid(xs[r], layout))
            d = c.delta(b)
            c.expect(d, what, fast=1, fallback=0)
            want = a2a_want(xs, n, r, count)
            c.same(bits(out), bits(want if one_algo(c, d, what) == "twoshot" else R.ll_move(want)), what)
        xs = R.gen_inputs(n, 64 * n, BF16, seed=n + 2, device="cpu")
        what = f"{layout} on rank 1: reduce_scatter_tensor"
        out = laid(torch.zeros(64, dtype=BF16), layout, fill=False)
        b = c.snap()
        dist.reduce_scatter_tensor(out, laid(xs[r], layout), op=AVG)
        d = c.delta(b)
        c.expect(d, what, fast=1, fallback=0)
        order = list(range(n)) if one_algo(c, d, what) == "ll" else ("rotate", r)
        c.same(out, R.ref_reduce([x[r * 64:(r + 1) * 64] for x in xs], order, scale_of(AVG, n), BF16), what)
        uneven(c, skewed(n), 8, F32, f"{layout} on rank 1", spare=2, layout=(1, layout))
        # max through the all-reduce-and-slice path: a strided input used to be refused there
        xs = R.gen_inputs(n, 64 * n, F32, seed=n + 3, device="cpu")
        out = laid(torch.zeros(64, dtype=F32), layout, fill=False)
        b = c.snap()
        dist.reduce_scatter_tensor(out, laid(xs[r], layout), op=MAX)
        d = c.delta(b)
        c.expect(d, f"{layout} on rank 1: reduce_scatter_tensor max", fast=1, fallback=0, generic=1)
        c.same(out, generic_ref(xs, MAX)[r * 64:(r + 1) * 64], f"{layout} on rank 1: reduce_scatter_tensor max")


def check_sub_groups(c):
    """Two disjoint pairs and a cross group at four ranks, each a process group with its own communicator, on seeded data."""
    if c.world != 4:
        return
    groups = [([0, 1], dist.new_group([0, 1])), ([2, 3], dist.new_group([2, 3])), ([0, 2], dist.new_group([0, 2]))]
    for members, pg in groups:
        if c.rank not in members:
            continue
        sub = Ctx(members.index(c.rank), len(members), pg=pg, members=members)
        xs = R.gen_inputs(2, 1003, BF16, seed=sum(members), device="cpu")
        what = f"sub-group {members}"
        t = sub.put(xs[sub.rank])
        b = sub.snap()
        dist.all_reduce(t, op=AVG, group=pg)
        d = sub.delta(b)
        sub.expect(d, what, fast=1, fallback=0)
        sub.same(t, R.ref_reduce(xs, sum_order(sub, d, BF16, 1003, what), scale_of(AVG, 2), BF16), what)
        ids = int_inputs(2, 1002, torch.int64, seed=sum(members))
        out, buf = sub.guarded(2 * 1002, torch.int64)
        b = sub.snap()
        dist.all_gather_into_tensor(out, sub.put(ids[sub.rank]), group=pg)
        d = sub.delta(b)
        sub.expect(d, what + " all_gather", fast=1, fallback=0, algo={"twoshot": 1})
        sub.same(out, torch.cat(ids), what + " all_gather")
        sub.guards_kept(buf, what)
        check_point_to_point(sub)
        c.errors += sub.errors
    dist.all_reduce(torch.zeros(1))            # a CPU tensor: the ranks meet on the host, so nobody waits inside a kernel for the busier ones
    # the world group still works after its members were busy elsewhere
    xs = R.gen_inputs(4, 1003, F32, seed=4, device="cpu")
    t = c.put(xs[c.rank])
    b = c.snap()
    dist.all_reduce(t)
    d = c.delta(b)
    c.expect(d, "world after the sub-groups", fast=1, fallback=0)
    c.same(t, R.ref_reduce(xs, sum_order(c, d, F32, 1003, "world after the sub-groups"), 1.0, F32), "world after the sub-groups")


CHECKS = [check_all_reduce, check_generic_reductions, check_reduce, check_reduce_scatter, check_broadcast, check_all_gather, check_all_to_all,
          check_all_to_all_uneven, check_point_to_point, check_two_streams, check_layout_differs_by_rank, check_sub_groups]


def _all_checks(rank, world):
    if DEV == "cuda":
        torch.cuda.set_device(0)                                            # the ranks share cuda:0
    c = Ctx(rank, world)
    took = {}
    for check in CHECKS:
        t0 = time.monotonic()
        check(c)
        took[check.__name__] = round(time.monotonic() - t0, 1)
    assert not c.errors, f"{len(c.errors)} failures:\n" + "\n".join(c.errors[:30])
    return took


@pytest.mark.parametrize("world", [2, 3, 4])
def test_every_route_bit_for_bit(world):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    _run(_all_checks, world)
