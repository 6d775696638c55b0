"""`torch.distributed` backend "b200coll" (parallel/process_group.py). On CPU every collective takes the Gloo fallback, which
still exercises what is specific to a Python process group: registration, c10d -> trampoline dispatch, the option objects,
Work / Future hand-back to c10d's C++ callers (DDP's reducer), and the all-to-all-v layout maths."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from container_engine_accelerators_b200.parallel import process_group as pgmod


def _free_port() -> int:
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _run(fn, world, *args):
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.SimpleQueue()
    procs = [ctx.Process(target=_entry, args=(fn, r, world, port, q, args)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
    results = sorted(q.get() for _ in range(world))
    assert all(p.exitcode == 0 for p in procs), results
    assert all(r[1] == "ok" for r in results), results
    return results


def _entry(fn, rank, world, port, q, args):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        from container_engine_accelerators_b200.parallel import process_group  # noqa: F401  (registers the backend)
        dist.init_process_group("b200coll", rank=rank, world_size=world)
        out = fn(rank, world, *args)
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok", out))
    except Exception as e:      # surface the failure in the parent
        import traceback
        q.put((rank, "error", traceback.format_exc() + repr(e)))
        sys.exit(1)


def _collectives(rank, world):
    pg = dist.group.WORLD
    assert dist.get_backend() == "b200coll" and isinstance(pg, pgmod.B200CollProcessGroup)
    t = torch.full((5,), float(rank + 1))
    dist.all_reduce(t)
    assert torch.equal(t, torch.full((5,), float(sum(range(1, world + 1)))))
    t = torch.full((4,), float(rank + 1)); dist.all_reduce(t, op=dist.ReduceOp.AVG)
    assert torch.allclose(t, torch.full((4,), (world + 1) / 2))
    t = torch.tensor([rank, 10 - rank]); dist.all_reduce(t, op=dist.ReduceOp.MAX)
    assert t.tolist() == [world - 1, 10]
    b = torch.arange(6, dtype=torch.int64) * (rank + 1); dist.broadcast(b, src=world - 1)
    assert torch.equal(b, torch.arange(6) * world)
    r = torch.ones(3) * (rank + 1); dist.reduce(r, dst=0)
    assert rank != 0 or torch.equal(r, torch.full((3,), float(sum(range(1, world + 1)))))
    outs = [torch.empty(2) for _ in range(world)]; dist.all_gather(outs, torch.tensor([rank, rank + 0.5]))
    assert [o.tolist() for o in outs] == [[float(s), s + 0.5] for s in range(world)]
    big = torch.empty(3 * world); dist.all_gather_into_tensor(big, torch.full((3,), float(rank)))
    assert big.tolist() == [float(s) for s in range(world) for _ in range(3)]
    rs = torch.empty(2); dist.reduce_scatter_tensor(rs, torch.arange(2 * world, dtype=torch.float32) + rank)
    assert rs.tolist() == [world * (2 * rank + k) + sum(range(world)) for k in range(2)]
    a2a = torch.empty(world * 2); dist.all_to_all_single(a2a, torch.arange(world * 2, dtype=torch.float32) + 100 * rank)
    assert a2a.tolist() == [100 * s + 2 * rank + k for s in range(world) for k in range(2)]
    # uneven all_to_all_single: rank r sends (d + 1) rows of width 4 to rank d
    in_splits = [d + 1 for d in range(world)]; out_splits = [rank + 1] * world
    src = torch.arange(sum(in_splits) * 4, dtype=torch.float32).view(-1, 4) + 1000 * rank
    dst = torch.empty(sum(out_splits), 4)
    dist.all_to_all_single(dst, src, out_splits, in_splits)
    off = sum(in_splits[:rank])
    want = torch.cat([(torch.arange(sum(in_splits) * 4, dtype=torch.float32).view(-1, 4) + 1000 * s)[off:off + rank + 1] for s in range(world)])
    assert torch.equal(dst, want)
    g = [torch.empty(1) for _ in range(world)] if rank == 0 else None
    dist.gather(torch.tensor([float(rank)]), g, dst=0)
    assert rank != 0 or [x.item() for x in g] == [float(s) for s in range(world)]
    sc = torch.empty(1); dist.scatter(sc, [torch.tensor([float(10 + s)]) for s in range(world)] if rank == 0 else None, src=0)
    assert sc.item() == 10 + rank
    if rank == 0:
        dist.send(torch.tensor([42.0]), dst=1)
    elif rank == 1:
        m = torch.empty(1); dist.recv(m, src=0); assert m.item() == 42.0
    objs = [{"cfg": rank}] if rank == 0 else [None]
    dist.broadcast_object_list(objs, src=0)
    assert objs == [{"cfg": 0}]
    dist.barrier()
    assert pg.fast_calls == 0 and pg.fallback_calls >= 12          # no GPU here: everything went through Gloo
    return pg.fallback_calls


def test_every_collective_through_the_registered_backend():
    _run(_collectives, 2)


def _ddp(rank, world):
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.ReLU(), torch.nn.Linear(16, 2))
    ddp = torch.nn.parallel.DistributedDataParallel(model)                  # C++ reducer calling into the Python process group
    opt = torch.optim.SGD(ddp.parameters(), lr=0.1)
    torch.manual_seed(100 + rank)
    for _ in range(3):
        x, y = torch.randn(4, 8), torch.randn(4, 2)
        opt.zero_grad()
        torch.nn.functional.mse_loss(ddp(x), y).backward()
        opt.step()
    flat = torch.cat([p.detach().reshape(-1) for p in model.parameters()])
    gathered = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    assert all(torch.allclose(g, gathered[0]) for g in gathered)            # replicas stayed in lock-step: gradients were averaged
    return float(flat.abs().sum())


def test_ddp_trains_in_lock_step_over_the_backend():
    res = _run(_ddp, 2)
    assert res[0][2] == pytest.approx(res[1][2])


def _subgroups(rank, world):
    """TP x DP style: two disjoint pairs plus a cross group, each its own process group (and, on GPUs, its own communicator)."""
    pairs = [dist.new_group([0, 1]), dist.new_group([2, 3])]
    cross = dist.new_group([0, 2])
    mine = pairs[rank // 2]
    assert isinstance(mine, pgmod.B200CollProcessGroup) and mine.size() == 2 and mine.rank() == rank % 2
    t = torch.tensor([float(rank)])
    dist.all_reduce(t, group=mine)
    assert t.item() == (1.0 if rank < 2 else 5.0)
    if rank in (0, 2):
        u = torch.tensor([10.0 + rank]); dist.all_reduce(u, group=cross)
        assert u.item() == 22.0
    w = torch.tensor([1.0]); dist.all_reduce(w)
    assert w.item() == 4.0
    return 0


def test_sub_groups_are_independent_process_groups():
    _run(_subgroups, 4)


def test_reduce_ops_of_option_structs_map_to_library_operators():
    """The ReduceOp inside an options struct equals the ReduceOp.SUM constants but does not hash like them: the mapping must use ==
    (a dict lookup silently sent every all-reduce to the Gloo fallback)."""
    o = dist.AllreduceOptions()
    want = {"SUM": pgmod.coll.SUM, "AVG": pgmod.coll.AVG, "MIN": pgmod.coll.MIN, "MAX": pgmod.coll.MAX, "PRODUCT": pgmod.coll.PROD, "BAND": None}
    for name, ours in want.items():
        o.reduceOp = getattr(dist.ReduceOp, name)
        assert pgmod._red_op(o.reduceOp) == ours, name
        assert pgmod._red_op(getattr(dist.ReduceOp, name)) == ours, name


def test_alltoallv_layout():
    m = [[1, 2, 0], [0, 3, 4], [5, 0, 6]]                                   # m[src][dst]
    assert pgmod.alltoallv_layout(m, 0) == ([1, 2, 0], [0, 1, 3], [0, 0, 0], 10)
    assert pgmod.alltoallv_layout(m, 1) == ([0, 3, 4], [0, 0, 3], [1, 2, 0], 10)
    assert pgmod.alltoallv_layout(m, 2) == ([5, 0, 6], [0, 5, 5], [1, 5, 4], 10)


def test_word_views_for_bit_exact_broadcast():
    f = pgmod.B200CollProcessGroup._as_words
    assert f(torch.zeros(4)) is None                                        # CPU tensors never take the device path


def _gpu_pair(rank, world):
    torch.cuda.set_device(0)                                                # two ranks share cuda:0 on a one-GPU box
    pg = dist.group.WORLD
    x = torch.full((1 << 16,), float(rank + 1), device="cuda", dtype=torch.bfloat16)
    dist.all_reduce(x)
    assert torch.equal(x.float(), torch.full_like(x, 3.0).float())
    sym = pg.empty(1 << 20, torch.float32); sym.fill_(rank + 1.0)
    dist.all_reduce(sym, op=dist.ReduceOp.AVG)
    assert torch.equal(sym, torch.full_like(sym, 1.5))
    ids = torch.arange(1001, device="cuda", dtype=torch.int64) * (rank + 1); dist.broadcast(ids, src=1)
    assert torch.equal(ids, torch.arange(1001, device="cuda") * 2)
    out = torch.empty(2 * 4096, device="cuda"); dist.all_gather_into_tensor(out, torch.full((4096,), float(rank), device="cuda"))
    assert out[:4096].eq(0).all() and out[4096:].eq(1).all()
    rs = torch.empty(4096, device="cuda"); dist.reduce_scatter_tensor(rs, torch.ones(2 * 4096, device="cuda") * (rank + 1))
    assert rs.eq(3).all()
    in_splits = [1, 3] if rank == 0 else [2, 2]; out_splits = [1, 2] if rank == 0 else [3, 2]
    src = (torch.arange(4 * 64, device="cuda", dtype=torch.float32).view(4, 64) + 1000 * rank)
    dst = torch.empty(sum(out_splits), 64, device="cuda")
    dist.all_to_all_single(dst, src, out_splits, in_splits)
    base = torch.arange(4 * 64, device="cuda", dtype=torch.float32).view(4, 64)
    want = torch.cat([base[0:1], base[0:2] + 1000]) if rank == 0 else torch.cat([base[1:4], base[2:4] + 1000])
    assert torch.equal(dst, want)
    fb = pg.fallback_calls
    cnt = torch.tensor([rank], device="cuda"); dist.all_reduce(cnt, op=dist.ReduceOp.MAX)      # integer max: the library's generic reduction kernel, not Gloo
    assert cnt.item() == 1 and pg.fallback_calls == fb
    steps = torch.tensor([3 + rank, 10 - rank, 7], device="cuda", dtype=torch.int32); dist.all_reduce(steps, op=dist.ReduceOp.MIN)
    assert steps.tolist() == [3, 9, 7] and pg.fallback_calls == fb
    prod = torch.full((1000,), 1.5 + rank, device="cuda", dtype=torch.float64); dist.all_reduce(prod, op=dist.ReduceOp.PRODUCT)
    assert torch.equal(prod, torch.full_like(prod, 1.5 * 2.5)) and pg.fallback_calls == fb
    model = torch.nn.Linear(32, 32).cuda()
    ddp = torch.nn.parallel.DistributedDataParallel(model, device_ids=[0])
    torch.manual_seed(rank); ddp(torch.randn(8, 32, device="cuda")).sum().backward()
    g = model.weight.grad.clone(); gs = [torch.empty_like(g) for _ in range(world)]; dist.all_gather(gs, g)
    assert torch.allclose(gs[0], gs[1])
    # collectives issued from two different streams back to back: the group orders them (one collective at a time per communicator)
    side = torch.cuda.Stream()
    a = torch.full((1 << 18,), float(rank + 1), device="cuda"); b = torch.full((1 << 18,), 10.0 * (rank + 1), device="cuda")
    torch.cuda.synchronize()
    for _ in range(20):
        dist.all_reduce(a)
        with torch.cuda.stream(side):
            dist.all_reduce(b)
    torch.cuda.synchronize()
    assert a.eq(3.0 * 2 ** 19).all() and b.eq(30.0 * 2 ** 19).all()              # 1 + 2, then doubled by each of the 19 later rounds
    # point to point: blocking pair, then a ring step as isend + irecv (queued, one grouped kernel at the first wait), a strided tensor,
    # and batch_isend_irecv
    other = 1 - rank
    msg = torch.arange(1 << 12, device="cuda", dtype=torch.float32) + 100 * rank
    got = torch.empty_like(msg)
    if rank == 0:
        dist.send(msg, dst=1); dist.recv(got, src=1)
    else:
        dist.recv(got, src=0); dist.send(msg, dst=0)
    assert torch.equal(got, torch.arange(1 << 12, device="cuda", dtype=torch.float32) + 100 * other)
    before = pg.fallback_calls
    strided = torch.zeros(64, 2, device="cuda")[:, 0]
    reqs = [dist.isend(msg[:64], other), dist.irecv(strided, other)]
    for r in reqs:
        r.wait()
    assert torch.equal(strided, (torch.arange(64, device="cuda", dtype=torch.float32) + 100 * other))
    big = torch.empty(1 << 20, device="cuda", dtype=torch.bfloat16)
    ops = [dist.P2POp(dist.isend, torch.full((1 << 20,), float(rank + 1), device="cuda", dtype=torch.bfloat16), other), dist.P2POp(dist.irecv, big, other)]
    for r in dist.batch_isend_irecv(ops):
        r.wait()
    assert big.eq(float(other + 1)).all() and pg.fallback_calls == before
    # gather / scatter: one grouped kernel around the root
    before = pg.fallback_calls
    mine = torch.full((2048,), float(rank + 1), device="cuda")
    parts = [torch.empty(2048, device="cuda") for _ in range(world)] if rank == 1 else None
    dist.gather(mine, parts, dst=1)
    if rank == 1:
        assert parts[0].eq(1).all() and parts[1].eq(2).all()
    piece = torch.empty(2048, device="cuda")
    dist.scatter(piece, [torch.full((2048,), 10.0 + r, device="cuda") for r in range(world)] if rank == 0 else None, src=0)
    assert piece.eq(10.0 + rank).all() and pg.fallback_calls == before
    # integer payloads ride the same kernels as raw words, bit for bit (an int64 -1 is all ones: the Lamport path would rewrite it)
    before = pg.fallback_calls
    ids = torch.full((4096,), -1, device="cuda", dtype=torch.int64); ids[::7] = rank
    gathered = torch.empty(2 * 4096, device="cuda", dtype=torch.int64)
    dist.all_gather_into_tensor(gathered, ids)
    want0 = torch.full((4096,), -1, device="cuda", dtype=torch.int64); want1 = want0.clone(); want0[::7] = 0; want1[::7] = 1
    assert torch.equal(gathered, torch.cat([want0, want1])) and pg.fallback_calls == before
    # tensors created under the group's memory pool live in the symmetric arena: collectives on them are not staged
    staged_before = pg.comm.stats()["staged_calls"]
    with torch.cuda.use_mem_pool(pg.mem_pool()):
        pooled = torch.full((8 << 20,), float(rank + 1), device="cuda")                   # 32 MiB: far beyond the Lamport path
    assert pg.comm.is_symmetric(pooled)
    dist.all_reduce(pooled)
    torch.cuda.synchronize()
    assert pooled.eq(3.0).all() and pg.comm.stats()["staged_calls"] == staged_before
    del pooled
    assert pg.fast_calls >= 13
    return pg.fast_calls


@pytest.mark.gpu

def test_cuda_fast_paths_two_ranks():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    _run(_gpu_pair, 2)


# ------------------------------------------------------------------------------------------------- point-to-point queueing (no GPU)
class _DeviceLike(torch.Tensor):
    """A CPU tensor that answers is_cuda=True, so the process group takes its CUDA branch while the test stays on CPU."""
    is_cuda = property(lambda self: True)

    @staticmethod
    def of(t):
        return torch.Tensor._make_subclass(_DeviceLike, t)


class _RecordingComm:
    def __init__(self):
        self.calls, self.in_group = [], 0

    def check_async_error(self):
        pass

    def send(self, t, peer):
        self.calls.append(("send", peer, t.numel() * t.element_size(), t.is_contiguous() and t.data_ptr() % 16 == 0, self.in_group))

    def recv(self, t, peer):
        self.calls.append(("recv", peer, t.numel() * t.element_size(), t.is_contiguous() and t.data_ptr() % 16 == 0, self.in_group))
        t.fill_(7.0)                                  # "data from the peer"
        return t

    def barrier(self):
        self.calls.append(("barrier",))


def test_point_to_point_calls_are_queued_and_launched_as_one_group(monkeypatch):
    """isend / irecv on device tensors are queued; the first wait() (or the next collective) launches everything queued inside ONE
    library group, in call order; tensors the kernel cannot take as they are travel through an aligned contiguous temporary."""
    class _Stream:
        def wait_event(self, e): pass
        def synchronize(self): pass
    class _Event:
        def record(self, s): pass
    stream = _Stream()
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: stream)
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    comm = _RecordingComm()
    groups = []

    class _Group:                                      # stands in for ops.coll.group: counts how often a library group is opened
        def __enter__(self): comm.in_group += 1; groups.append(len(comm.calls)); return self
        def __exit__(self, *exc): comm.in_group -= 1; return False
    monkeypatch.setattr(pgmod.coll, "group", _Group)
    pg = pgmod.B200CollProcessGroup(store=None, rank=0, size=2)
    pg._comm = comm
    out = _DeviceLike.of(torch.arange(64, dtype=torch.float32))
    strided = _DeviceLike.of(torch.zeros(32, 2))[:, 0]                   # not contiguous
    inn = _DeviceLike.of(torch.zeros(64))
    w1 = pg.send([out], 1)
    w2 = pg.recv([strided], 1)
    w3 = pg.recv([inn], 1)
    assert comm.calls == [] and len(pg._pending) == 3                     # nothing launched yet
    assert w2.wait() and comm.calls == [("send", 1, 256, True, 1), ("recv", 1, 128, True, 1), ("recv", 1, 256, True, 1)]
    assert groups == [0] and pg._pending == []                            # one group for all three, in call order
    assert strided.eq(7.0).all() and inn.eq(7.0).all()                    # the strided tensor was filled through its temporary
    assert w1.wait() and w3.wait() and len(comm.calls) == 3               # later waits have nothing left to launch
    # a collective issued while sends are queued launches them first (they keep their place in the order of calls)
    pg.send([out], 1)
    pg.barrier().wait()
    assert [c[0] for c in comm.calls[3:]] == ["send", "barrier"] and pg.fast_calls == 5 and pg.fallback_calls == 0
    # empty tensors never reach the library
    pg.send([_DeviceLike.of(torch.zeros(0))], 1).wait()
    assert len(comm.calls) == 5
    # gather / scatter: one group around the root (this rank is rank 0 of 2)
    go = dist.GatherOptions(); go.rootRank = 0
    outs = [_DeviceLike.of(torch.zeros(8)), _DeviceLike.of(torch.zeros(8))]
    pg.gather([outs], [_DeviceLike.of(torch.ones(8))], go).wait()
    assert [(c[0], c[1]) for c in comm.calls[5:]] == [("send", 0), ("recv", 0), ("recv", 1)] and groups[-1] == 5
    so = dist.ScatterOptions(); so.rootRank = 1
    pg.scatter([_DeviceLike.of(torch.zeros(8))], [[]], so).wait()                               # not the root: just one receive from it
    assert [(c[0], c[1]) for c in comm.calls[8:]] == [("recv", 1)] and pg.fallback_calls == 0


def test_ddp_demo_trains_on_the_backend():
    """demo/gpu-training/ddp_b200coll.py under torchrun with two ranks (CPU here: the process group's Gloo fallback carries DDP's bucket
    all-reduces): the loss moves and both replicas end with identical weights."""
    import json
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
                        os.path.join(root, "demo", "gpu-training", "ddp_b200coll.py"), "--steps", "6", "--batch", "2", "--seq", "32", "--dim", "64", "--layers", "2", "--vocab", "256"],
                       capture_output=True, text=True, timeout=300, env={**os.environ, "CUDA_VISIBLE_DEVICES": ""})
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    out = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    assert out["backend"] == "b200coll" and out["world"] == 2 and out["replicas_in_sync"] is True
    assert out["last_loss"] < out["first_loss"] and out["fallback_calls"] > 0


def test_integer_payloads_move_as_words_and_never_take_the_lamport_path(monkeypatch):
    """all_gather_into_tensor / all_to_all_single of int64 token ids on device tensors: viewed as fp32 words, with the communicator switched
    to the bit-exact (barrier-based, identity epilogue) kernels for the duration of the call — the Lamport path rewrites words that look
    like its empty-slot marker, which an int64 -1 does."""
    class _Stream:
        def wait_event(self, e): pass
    class _Event:
        def record(self, s): pass
    stream = _Stream()
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: stream)
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    log = []

    class _Comm:
        nranks = 2
        _algo = "auto"
        def set_algo(self, name): log.append(("algo", name)); self._algo = name
        def bit_exact(self): return pgmod.coll.Comm._BitExact(self)
        def all_gather(self, src, dst): log.append(("all_gather", src.dtype, src.numel(), dst.numel()))
        def all_to_all(self, src, dst): log.append(("all_to_all", src.dtype, src.numel(), dst.numel()))
    pg = pgmod.B200CollProcessGroup(store=None, rank=0, size=2)
    pg._comm = _Comm()
    ids = _DeviceLike.of(torch.full((64,), -1, dtype=torch.int64))
    out = _DeviceLike.of(torch.zeros(128, dtype=torch.int64))
    pg._allgather_base(out, ids)
    assert log == [("algo", "twoshot"), ("all_gather", torch.float32, 128, 256), ("algo", "auto")]
    del log[:]
    pg.alltoall_base(_DeviceLike.of(torch.zeros(64, dtype=torch.int64)), ids, [], [])
    assert log == [("algo", "twoshot"), ("all_to_all", torch.float32, 128, 128), ("algo", "auto")]
    del log[:]
    flt = _DeviceLike.of(torch.zeros(64)); pg._allgather_base(_DeviceLike.of(torch.zeros(128)), flt)      # real floats keep the tuner's choice
    assert log == [("all_gather", torch.float32, 64, 128)] and pg.fast_calls == 3 and pg.fallback_calls == 0


# ------------------------------------------------------------------------------------------------- the route is the same on every rank (no GPU)
class _RouteComm:
    """Stands in for the communicator: logs which library call was made, refuses a buffer the kernels could not take, and writes 7s
    where the kernel would write."""
    nranks = 2
    _algo = "auto"

    def __init__(self, log):
        self.log = log

    def _call(self, name, *bufs, out=None):
        assert all(b.is_contiguous() and b.data_ptr() % 16 == 0 and b.data_ptr() != 0 for b in bufs), f"{name}: a buffer the kernel cannot take"
        self.log.append("lib." + name)
        if out is not None:
            out.fill_(7)

    def check_async_error(self): pass
    def set_algo(self, name): self._algo = name
    def bit_exact(self): self.log.append("bit_exact"); return pgmod.coll.Comm._BitExact(self)
    def empty(self, numel, dtype): return torch.zeros(numel, dtype=dtype)
    def all_reduce(self, t, op=None): self._call("all_reduce", t, out=t)
    def reduce(self, t, root=0, op=None): self._call("reduce", t, out=t)
    def broadcast(self, t, root=0): self._call("broadcast", t, out=t)
    def all_gather(self, src, dst): self._call("all_gather", src, dst, out=dst)
    def reduce_scatter(self, src, dst, op=None): self._call("reduce_scatter", src, dst, out=dst)
    def all_to_all(self, src, dst): self._call("all_to_all", src, dst, out=dst)
    def all_to_all_v(self, src, dst, row_elems, send_rows, send_off, recv_off): self._call("all_to_all_v", src, dst, out=dst)


class _RouteGloo:
    """Stands in for the Gloo group: logs the call; its all-gather hands back the split matrix of the uneven all-to-all."""
    class _Done:
        def wait(self): return True

    def __init__(self, log, matrix):
        self.log, self.matrix = log, matrix

    def allgather(self, outs, ins, *a):
        self.log.append("gloo.allgather")
        for o, row in zip(outs[0], self.matrix):
            if o.numel() == len(row):
                o.copy_(torch.tensor(row))
        return self._Done()

    def __getattr__(self, name):
        def call(*a, **k):
            self.log.append("gloo." + name)
            return self._Done()
        return call


def _route_group(monkeypatch, rank, matrix=((0, 0), (0, 0))):
    class _Stream:
        def wait_event(self, e): pass
        def synchronize(self): pass
    class _Event:
        def record(self, s): pass
    stream = _Stream()
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: stream)
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    log = []
    pg = pgmod.B200CollProcessGroup(store=None, rank=rank, size=2)
    pg._comm, pg._gloo = _RouteComm(log), _RouteGloo(log, [list(r) for r in matrix])
    return pg, log


def _laid_out(layout, numel, dtype=torch.float32, cols=None):
    """A device-like tensor of `numel` elements (rows of `cols`): as the allocator gives it, starting 4 or 8 bytes past a 16-byte
    boundary, or a column slice of a wider tensor."""
    shape = (numel,) if cols is None else (numel // cols, cols)
    if layout == "misaligned":
        return _DeviceLike.of(torch.zeros(numel + 1, dtype=dtype))[1:].view(shape)
    if layout == "strided":
        return _DeviceLike.of(torch.zeros(*shape, 2, dtype=dtype))[..., 0]
    return _DeviceLike.of(torch.zeros(shape, dtype=dtype))


def _ar_opts(op):
    o = dist.AllreduceOptions(); o.reduceOp = op
    return o


def _rs_opts(op):
    o = dist.ReduceScatterOptions(); o.reduceOp = op
    return o


# name -> (call(pg, make) -> the tensor that must have been written, or None; the route every rank must take)
_ROUTE_CASES = {
    "all_reduce fp32 sum": (lambda pg, mk: (lambda t: (pg.allreduce([t], _ar_opts(dist.ReduceOp.SUM)), t)[1])(mk(64)), ["lib.all_reduce"]),
    "all_reduce int64 max": (lambda pg, mk: (lambda t: (pg.allreduce([t], _ar_opts(dist.ReduceOp.MAX)), t)[1])(mk(64, torch.int64)), ["lib.all_reduce"]),
    "all_reduce int32 avg": (lambda pg, mk: (pg.allreduce([mk(64, torch.int32)], _ar_opts(dist.ReduceOp.AVG)), None)[1], ["gloo.allreduce"]),
    "reduce bf16 (root)": (lambda pg, mk: (lambda t: (pg.reduce([t]), t)[1])(mk(64, torch.bfloat16)), ["lib.reduce"]),
    "broadcast int64": (lambda pg, mk: (lambda t: (pg.broadcast([t]), t)[1])(mk(33, torch.int64)), ["lib.broadcast"]),
    "broadcast uint8, odd bytes": (lambda pg, mk: (pg.broadcast([mk(33, torch.uint8)]), None)[1], ["gloo.broadcast"]),
    "all_gather_into_tensor fp32": (lambda pg, mk: (lambda o: (pg._allgather_base(o, mk(64)), o)[1])(mk(128)), ["lib.all_gather"]),
    "all_gather_into_tensor int64": (lambda pg, mk: (lambda o: (pg._allgather_base(o, mk(64, torch.int64)), o)[1])(mk(128, torch.int64)),
                                     ["bit_exact", "lib.all_gather"]),
    "all_gather list fp32": (lambda pg, mk: (lambda outs: (pg.allgather([outs], [mk(64)]), outs[1])[1])([mk(64), mk(64)]), ["lib.all_gather"]),
    "reduce_scatter_tensor bf16 avg": (lambda pg, mk: (lambda o: (pg._reduce_scatter_base(o, mk(128, torch.bfloat16), _rs_opts(dist.ReduceOp.AVG)), o)[1])(mk(64, torch.bfloat16)),
                                       ["lib.reduce_scatter"]),
    "reduce_scatter_tensor fp32 max": (lambda pg, mk: (lambda o: (pg._reduce_scatter_base(o, mk(128), _rs_opts(dist.ReduceOp.MAX)), o)[1])(mk(64)),
                                       ["lib.all_reduce"]),
    "all_to_all_single even fp32": (lambda pg, mk: (lambda o: (pg.alltoall_base(o, mk(128), [], []), o)[1])(mk(128)), ["lib.all_to_all"]),
    "all_to_all_single even int64": (lambda pg, mk: (lambda o: (pg.alltoall_base(o, mk(128, torch.int64), [], []), o)[1])(mk(128, torch.int64)),
                                     ["bit_exact", "lib.all_to_all"]),
}


@pytest.mark.parametrize("case", sorted(_ROUTE_CASES))
def test_the_route_does_not_depend_on_this_ranks_layout(monkeypatch, case):
    """Every rank must take the same route, so the route may depend only on what the ranks share (device type, dtype, counts, operator).
    The same call with this rank's tensors misaligned or strided takes the route the plain call takes, the kernel still only sees
    aligned contiguous buffers (_RouteComm checks), and the result reaches the caller's tensor."""
    call, want = _ROUTE_CASES[case]
    for layout in ("plain", "misaligned", "strided"):
        pg, log = _route_group(monkeypatch, rank=0)
        written = call(pg, lambda numel, dtype=torch.float32: _laid_out(layout, numel, dtype))
        assert log == want, (case, layout, log)
        assert (pg.fast_calls, pg.fallback_calls) == ((1, 0) if want[-1].startswith("lib.") else (0, 1)), (case, layout)
        if written is not None and want[-1].startswith("lib."):
            assert bool((written != 0).all()), (case, layout, "the result never reached the caller's tensor")


def _uneven(pg, rows_in, rows_out, in_splits, out_splits, layout="plain", cols=8, dtype=torch.float32):
    src = _laid_out(layout, rows_in * cols, dtype, cols) if rows_in else _DeviceLike.of(torch.zeros(0, cols, dtype=dtype))
    dst = _laid_out(layout, rows_out * cols, dtype, cols) if rows_out else _DeviceLike.of(torch.zeros(0, cols, dtype=dtype))
    pg.alltoall_base(dst, src, out_splits, in_splits)
    return dst


def test_uneven_all_to_all_route_is_the_same_on_a_rank_without_rows(monkeypatch):
    """Expert dispatch: rank 0 sends 2 + 3 rows, rank 1 sends nothing (a silent sender) and rank 0 receives nothing from it. Both must
    enter the all-to-all-v (the split matrix over Gloo, then the library call); the silent rank hands the library a real send pointer."""
    matrix = ((2, 3), (0, 0))
    want = ["gloo.allgather", "lib.all_to_all_v"]
    pg0, log0 = _route_group(monkeypatch, 0, matrix)
    out0 = _uneven(pg0, 5, 2, [2, 3], [2, 0])
    pg1, log1 = _route_group(monkeypatch, 1, matrix)
    out1 = _uneven(pg1, 0, 3, [0, 0], [3, 0])
    assert log0 == want and log1 == want, (log0, log1)
    assert out0.eq(7).all() and out1.eq(7).all() and pg1.fallback_calls == 0
    # nothing to receive either: still the same route
    pg1, log1 = _route_group(monkeypatch, 1, ((2, 0), (0, 0)))
    _uneven(pg1, 0, 0, [0, 0], [0, 0])
    assert log1 == want
    # layout of this rank's rows does not matter, and spare output rows are left alone
    for layout in ("misaligned", "strided"):
        pg0, log0 = _route_group(monkeypatch, 0, matrix)
        out = _uneven(pg0, 5, 4, [2, 3], [2, 0], layout)
        assert log0 == want and out[:2].eq(7).all() and out[2:].eq(0).all(), layout
    # rows that are not whole 16-byte vectors, or an integer payload: Gloo, on the silent rank too
    for cols, dtype in ((3, torch.float32), (8, torch.int64)):
        for rank, rows_in, splits in ((0, 5, [2, 3]), (1, 0, [0, 0])):
            pg, log = _route_group(monkeypatch, rank, matrix)
            _uneven(pg, rows_in, 2, splits, [2, 0], cols=cols, dtype=dtype)
            assert log == ["gloo.alltoall_base"], (cols, dtype, rank, log)


def test_uneven_all_to_all_with_one_split_list_left_out(monkeypatch):
    """c10d: a split list left out means equal blocks. The rank's row of the split matrix is then the even split, not an empty list."""
    sent = []
    pg, log = _route_group(monkeypatch, 0, ((2, 2), (1, 3)))
    pg._gloo.allgather = lambda outs, ins, *a: (sent.append(ins[0].tolist()), _RouteGloo.allgather(pg._gloo, outs, ins))[1]
    out = _uneven(pg, 4, 3, [], [2, 1])
    assert sent == [[2, 2]] and log == ["gloo.allgather", "lib.all_to_all_v"] and out.eq(7).all()
