"""The harness every libb200coll GPU test module shares: the torch and library fixtures, dtype names, N virtual ranks as one Group, the
all-to-all-v Plan, and runners for the perf tool, fresh interpreters and refused raw calls.

Not collected by pytest (no test_ prefix). A test module imports the fixtures it uses by name (`# noqa: F401`)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import coll_fp_reference as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PERF = os.path.join(ROOT, "build", "b200coll_perf")

DTYPES = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32, "e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2,
          **{name: getattr(torch, name) for name in ("bfloat16", "float16", "float32", "float64", "float8_e4m3fn", "float8_e5m2", "int8",
                                                      "uint8", "int32", "uint32", "int64", "uint64")}}


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


@pytest.fixture(scope="module")
def coll_mod(coll_lib):
    from container_engine_accelerators_b200.ops import coll
    coll.load()          # raises if the .so is missing: GPU tests must never pass on a fallback
    return coll


class Group:
    """N virtual ranks: one communicator per device in `devices` (default: n ranks on cuda:0), one stream per rank on its device."""

    def __init__(self, torch, coll, n, devices=None, arena_mb=64, timeout_ms=None):
        self.torch, self.coll, self.n = torch, coll, n
        kw = {} if timeout_ms is None else {"timeout_ms": timeout_ms}
        self.comms = coll.Comm.init_all(devices if devices is not None else [0] * n, arena_mb=arena_mb, **kw)
        self.streams = []
        for c in self.comms:
            with torch.cuda.device(c.device):
                self.streams.append(torch.cuda.Stream())

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.destroy()

    def sync(self):
        for d in {c.device for c in self.comms}:
            self.torch.cuda.synchronize(d)

    def check_async(self):
        for c in self.comms:
            c.check_async_error()

    def run(self, fn):
        """fn(r, comm, stream) for every rank, on the rank's device, its stream first waiting for the device's current stream (where the
        inputs were filled); then sync and every communicator's async error check."""
        for r, c in enumerate(self.comms):
            with self.torch.cuda.device(c.device):
                self.streams[r].wait_stream(self.torch.cuda.current_stream())
                fn(r, c, self.streams[r])
        self.sync()
        self.check_async()

    def dev(self, c, a):
        """A numpy array copied to c's device."""
        return self.torch.from_numpy(np.ascontiguousarray(a)).to(f"cuda:{c.device}")

    def destroy(self):
        self.sync()
        for c in self.comms:
            c.destroy()


def group_fixture(n, **kw):
    """A `group` fixture: a Group of request.param ranks (default n) made with **kw, destroyed after the test."""
    @pytest.fixture
    def group(torch_cuda, coll_mod, request):
        with Group(torch_cuda, coll_mod, getattr(request, "param", n), **kw) as g:
            yield g
    return group


def release(comms, *per_rank_lists):
    """Hand every rank's arena tensor in each list back to its communicator."""
    for lst in per_rank_lists:
        for c, t in zip(comms, lst):
            c.release(t)


def algo_snapshot(comms):
    return [c.stats()["algo_calls"] for c in comms]


def ran(comms, before):
    """The algorithms the last call(s) recorded: {name: calls}, the same on every rank."""
    after = algo_snapshot(comms)
    deltas = [{k: a[k] - b[k] for k in a if a[k] != b[k]} for a, b in zip(after, before)]
    assert all(d == deltas[0] for d in deltas), deltas
    return deltas[0]


def poison(ts):
    """Fill receive buffers with a byte pattern first, so that an element a kernel never wrote cannot pass as a stale right answer."""
    for t in ts:
        t.view(-1).view(torch.uint8).fill_(0x7B)


def arena_inputs(comms, count, in_dt, seed):
    """coll_fp_reference.gen_inputs in arena buffers (one per rank)."""
    xs = R.gen_inputs(len(comms), count, in_dt, seed)
    bufs = [c.empty(count, in_dt) for c in comms]
    for b, x in zip(bufs, xs):
        b.copy_(x)
    torch.cuda.synchronize()
    return bufs


class Plan:
    """An all-to-all-v plan: rows[s, d] rows go from rank s (starting at its row send_off[s, d]) to rank d (landing at its row
    recv_off[d, s]). For a combine, index[s] and weights[s] are rank s's [tokens, top_k] arguments."""

    def __init__(self, rows, send_off, recv_off, index=None, weights=None):
        self.rows, self.send_off, self.recv_off = (np.asarray(a, dtype=np.int64) for a in (rows, send_off, recv_off))
        self.index, self.weights = index, weights
        n = len(self.rows)
        self.src_rows = int(max((self.send_off[s] + self.rows[s]).max() for s in range(n)))
        self.recv_rows = int(max((self.recv_off[d] + self.rows[:, d]).max() for d in range(n)))

    def args(self, r):
        """Rank r's (send_rows, send_offsets, recv_offsets) lists."""
        n = len(self.rows)
        return self.rows[r].tolist(), self.send_off[r].tolist(), [int(self.recv_off[d, r]) for d in range(n)]


def run_perf(args, devs, procs=False, env=None, timeout=600):
    """Run build/b200coll_perf on `devs` (one process per rank with `procs`), `env` added to the environment; assert it exits 0 with
    errors=0 and return its stdout."""
    r = subprocess.run([PERF, "--devs", devs, *(["--procs"] if procs else []), *args], capture_output=True, text=True, timeout=timeout,
                       env=None if env is None else {**os.environ, **env})
    assert r.returncode == 0 and "errors=0" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


def run_python(script, env, marker, timeout=300):
    """Run `script` in a fresh interpreter with the repository root on sys.path and `env` added to the environment; assert it exits 0
    and prints `marker`."""
    code = f"import sys\nsys.path.insert(0, {ROOT!r})\n{script}"
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env={**os.environ, **env}, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0 and marker in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


def expect_refused(rc, code, msg="", prefix=None, what=None):
    """A raw library call returned `code` and left a last-error message that contains `msg` and starts with `prefix`."""
    from container_engine_accelerators_b200.ops import coll
    err = coll.load().b200collGetLastError().decode()
    assert rc == code, (what, rc, err)
    assert err and msg in err, (what, err)
    assert prefix is None or err.startswith(prefix), (what, err)


def assert_nothing_launched(comm):
    st = comm.stats()
    assert st["kernel_launches"] == 0 and all(v == 0 for v in st["calls"]) and all(v == 0 for v in st["bytes"]), st
