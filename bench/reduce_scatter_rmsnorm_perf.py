#!/usr/bin/env python
"""reduce_scatter_rmsnorm_perf — the sequence-parallel pre-norm step, fused, against the two-shot all-reduce form and the four calls it
replaces.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 bench/reduce_scatter_rmsnorm_perf.py   # one GPU per rank
    python bench/reduce_scatter_rmsnorm_perf.py --virtual 4      # 4 virtual ranks sharing cuda:0 in one process (Comm.init_all)

For each (tokens, hidden) of allreduce_rmsnorm_perf.py's shapes with tokens a multiple of the rank count N, bf16, S = tokens / N, it
times device-side calls of
(a) comm.reduce_scatter_rms_norm(x, shard, gamma, out, gather=True): one kernel; the residual is this rank's [S, hidden] shard;
(b) comm.all_reduce_rms_norm(x, residual, gamma, out) forced to two-shot, with the full [tokens, hidden] residual on every rank;
(c) comm.reduce_scatter(x, part), shard.add_(part), F.rms_norm(shard, (hidden,), gamma, eps) copied into an arena buffer,
    comm.all_gather(normed, out): the four calls a caller writes today, plus the copy that lets the all-gather read from the arena.
The three are timed alternately in rounds within one process (median per call reported); x, out and (b)'s residual are in the arena.
With --virtual every call enqueues each rank's work on its own stream, and NVLink traffic is HBM traffic of the one GPU.

matches says that on fresh data (a)'s out and new shards equal (b)'s out and new residual slices bit for bit, and (c)'s new shard
equals (a)'s and its out lies within 2 bf16 ulp of (a)'s (x holds multiples of 1/4, so the reduce-scatter's sum is exact). bytes gives, per rank and per call, computed from the shapes (E = S * hidden * 2 bytes, one slice), what
each variant reads from and writes to the rank's own HBM, what crosses to or from its peers, and the residual elements it keeps. (a)
pushes (N-1) * E of out against (b)'s 2 * (N-1) * E of residual and out, and keeps S * hidden residual elements against N * S * hidden.
Rank 0 prints one JSON line."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TOKENS = (16, 128, 1024, 4096, 16384)
HIDDEN = (4096, 7168, 8192)
EPS = 1e-6
ROUNDS = 5


def _card(dev: int) -> dict:
    """The card name, power limit and SM clock maximum, read now (they are part of any number printed)."""
    import torch
    info = {"gpu": torch.cuda.get_device_name(dev)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"], info["sm_clock_max_mhz"] = float(q[0]), float(q[1])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        info["power_limit_w"] = info["sm_clock_max_mhz"] = None
    return info


def _bytes(n: int, s: int, hidden: int) -> dict:
    """Per rank and call, from the shapes: the rank's HBM read and written (by any rank's kernels), the bytes that cross between it and
    its peers (pulled and pushed), the bytes it pushes, and the residual elements it keeps. E is one slice of bf16 rows. Gamma
    (hidden * 2 bytes) is left out: every variant reads it once."""
    e = s * hidden * 2
    return {
        # every rank pulls its slice of my x (N * E read); my shard read and written; every rank's slice of out lands in mine
        "fused_rs": {"read": n * e + e, "written": e + n * e, "nvlink": 2 * (n - 1) * e, "pushed": (n - 1) * e, "residual_elems": s * hidden},
        # the same pull, my slice of the residual read; every rank's residual and out slices land in mine
        "twoshot_ar": {"read": n * e + e, "written": 2 * n * e, "nvlink": 3 * (n - 1) * e, "pushed": 2 * (n - 1) * e, "residual_elems": n * s * hidden},
        # reduce_scatter (x read, part written), add_ (shard and part read, shard written), rms_norm (shard read, normed written),
        # all_gather (normed read, out written); its pushes depend on the algorithms the two collectives pick
        "four_call": {"read": n * e + 2 * e + e + e, "written": e + e + e + n * e, "nvlink": 2 * (n - 1) * e, "pushed": None,
                      "residual_elems": s * hidden},
    }


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--virtual", type=int, default=0, metavar="N", help="N virtual ranks on cuda:0 in this process instead of torchrun's ranks")
    args = ap.parse_args()
    import torch
    import torch.nn.functional as F
    from container_engine_accelerators_b200.ops import coll
    dt = torch.bfloat16
    max_elems = max(TOKENS) * max(HIDDEN)
    arena_mb = (5 * max_elems * 2 >> 20) + 256
    if args.virtual:
        rank, world, dev = 0, args.virtual, 0
        torch.cuda.set_device(0)
        comms = coll.Comm.init_all([0] * world, arena_mb=arena_mb)
        streams = [torch.cuda.Stream() for _ in comms]
    else:
        rank, world, dev = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
        torch.cuda.set_device(dev)
        comms = [coll.Comm.from_env(arena_mb=arena_mb, tag="rs_rmsnorm_perf")]
        streams = [torch.cuda.current_stream()]
    ranks = [rank + i for i in range(len(comms))]          # the global rank of each local communicator
    bufs = [{k: c.empty(max_elems, dt) for k in ("x", "res", "out", "part", "normed")} for c in comms]
    shards = [torch.empty(max_elems // world, dtype=dt, device="cuda") for _ in comms]
    cur = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    shapes, matches = [], True
    for hidden in HIDDEN:
        gamma = (torch.rand(hidden, device="cuda", generator=torch.Generator("cuda").manual_seed(hidden)) + 0.5).to(dt)
        for tokens in TOKENS:
            if tokens % world:
                continue
            s, n = tokens // world, tokens * hidden
            # x: multiples of 1/4 in [-2, 2], so the ranks' sum is exact in bf16 and (c)'s two roundings (reduce-scatter, then add_) give
            # the residual (a) and (b) give; out then differs only by how PyTorch rounds the norm
            x0 = [(torch.randint(-8, 9, (tokens, hidden), device="cuda", generator=torch.Generator("cuda").manual_seed(tokens * 131 + hidden + r)) / 4)
                  .to(dt) for r in ranks]
            res0 = (torch.randn(tokens, hidden, device="cuda", generator=torch.Generator("cuda").manual_seed(tokens + hidden)) * 2).to(dt)
            v = [{k: t[:n].view(tokens, hidden) for k, t in b.items()} for b in bufs]     # part and normed use their first S rows
            sh = [t[:s * hidden].view(s, hidden) for t in shards]

            def reset():
                for i, r in enumerate(ranks):
                    v[i]["x"].copy_(x0[i]); v[i]["res"].copy_(res0); sh[i].copy_(res0[r * s:(r + 1) * s])

            def fused(i, c, st):
                c.reduce_scatter_rms_norm(v[i]["x"], sh[i], gamma, v[i]["out"], eps=EPS, gather=True, stream=st)

            def twoshot(i, c, st):
                c.set_algo("twoshot")                     # for this call only: (c)'s collectives keep the tuner's picks
                c.all_reduce_rms_norm(v[i]["x"], v[i]["res"], gamma, v[i]["out"], eps=EPS, stream=st)
                c.set_algo("auto")

            def rs(i, c, st):
                c.reduce_scatter(v[i]["x"], v[i]["part"].view(-1)[:s * hidden], stream=st)

            def add_norm(i, c, st):
                with torch.cuda.stream(st):
                    sh[i].add_(v[i]["part"].view(-1)[:s * hidden].view(s, hidden))
                    v[i]["normed"].view(-1)[:s * hidden].copy_(F.rms_norm(sh[i], (hidden,), gamma, EPS).view(-1))

            def ag(i, c, st):
                c.all_gather(v[i]["normed"].view(-1)[:s * hidden], v[i]["out"], stream=st)

            # a variant is a list of phases, each enqueued for every local rank before the next: with virtual ranks a PyTorch kernel's
            # first launch loads its module, which waits for the kernels already running, so it must not be enqueued while a rank's
            # collective waits for a peer this thread has not launched yet
            def run(phases, iters=1):
                for st in streams:
                    st.wait_stream(cur)
                for _ in range(iters):
                    for f in phases:
                        for i, (c, st) in enumerate(zip(comms, streams)):
                            f(i, c, st)
                for st in streams:
                    cur.wait_stream(st)

            # matches, on fresh data: rank r's slice of (b) against (a), and (c) within 2 bf16 ulp of (a)
            got = {}
            for name, f in (("fused", [fused]), ("twoshot", [twoshot]), ("four_call", [rs, add_norm, ag])):
                reset()
                run(f)
                torch.cuda.synchronize()
                got[name] = [(sh[i].clone(), v[i]["res"].clone(), v[i]["out"].clone()) for i in range(len(comms))]
            near = lambda a, b: bool(((a.float() - b.float()).abs() <= 2 * 2.0 ** -7 * b.float().abs() + 1e-30).all())
            same, close = True, True
            for i, r in enumerate(ranks):
                fs, _, fo = got["fused"][i]
                _, tr, to = got["twoshot"][i]
                cs, _, co = got["four_call"][i]
                same = same and torch.equal(fs.view(torch.int16), tr[r * s:(r + 1) * s].view(torch.int16)) and torch.equal(fo.view(torch.int16), to.view(torch.int16))
                close = close and torch.equal(cs.view(torch.int16), fs.view(torch.int16)) and near(co, fo)
            ok = same and close
            matches = matches and ok
            iters = max(10, min(300, (1 << 30) // (n * 2 * world)))
            per = {"fused_rs": [], "twoshot_ar": [], "four_call": []}
            variants = (("fused_rs", [fused]), ("twoshot_ar", [twoshot]), ("four_call", [rs, add_norm, ag]))
            for _, f in variants:
                run(f, 3)
            for _ in range(ROUNDS):
                for name, f in variants:
                    reset()
                    torch.cuda.synchronize()
                    e0.record(cur)
                    run(f, iters)
                    e1.record(cur)
                    e1.synchronize()
                    per[name].append(e0.elapsed_time(e1) * 1e3 / iters)
            med = {k: round(sorted(t)[len(t) // 2], 2) for k, t in per.items()}
            shapes.append({"tokens": tokens, "hidden": hidden, **{k + "_us": t for k, t in med.items()}, "matches": ok, "equals_twoshot": same,
                           "four_call_within_2ulp": close, "bytes": _bytes(world, s, hidden)})
    for c in comms:
        c.check_async_error()
    if rank == 0:
        print(json.dumps({"metric": "reduce_scatter_rmsnorm", "ranks": world, "virtual": bool(args.virtual), "dtype": "bf16", **_card(dev), "eps": EPS,
                          "shapes": shapes, "matches": matches}), flush=True)
    torch.cuda.synchronize()
    for c, b in zip(comms, bufs):
        for t in b.values():
            c.release(t)
        c.destroy()
    return 0 if matches else 1


if __name__ == "__main__":
    sys.exit(main())
