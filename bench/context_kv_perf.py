#!/usr/bin/env python
"""context_kv_perf — the context-parallel K and V all-gather and its gradient reduce-scatter, fused, against the composition a layer
writes with plain all_gather and reduce_scatter.

    python bench/context_kv_perf.py                                                          # one rank on cuda:0
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 bench/context_kv_perf.py   # one GPU per rank

B = 1, bf16, C = 2 (the load-balanced causal layout), for Llama-3-8B (Hq 32, Hkv 8, D 128: K and V column slices of a packed QKV), and
Llama-3-70B (Hq 64, Hkv 8, D 128), and an MLA-like pair of dense tensors of widths 512 (c_kv) and 64 (k_pe), at full sequences S of
32k and 128k tokens (S_l = S / N per rank), it times device-side calls of
  gather  (a) comm.all_gather_context over the K and V slices (or the two MLA tensors) into dense [S, W] arena tensors: one kernel;
          (b) per tensor: a dense copy of the slice into an arena send buffer, comm.all_gather, and an index_select from rank-chunk
              order into token order;
  reduce-scatter, the gradient: each rank's [S, W] full-sequence dK and dV
          (a) comm.reduce_scatter_context straight into the K and V slices of a packed dQKV: one kernel;
          (b) per tensor: an index_select from token order into rank-chunk order (into an arena buffer), comm.reduce_scatter, and a copy
              into the dQKV slice.
The two are alternated in five rounds within one process and the median per call is reported. matches says whether (a) and (b)
produced the same output: the gather bit for bit; the reduce-scatter either bit for bit (max_ulp 0) or within max_ulp bf16 ulps, since
reduce_scatter sums receiving-rank-first and the fused call in rank order (at one rank both are copies). bytes gives, per rank and
call, computed from the shapes, what each variant reads from and writes to the rank's HBM (the pushes and pulls of peers touch it too),
and ops how many kernels or collective calls each enqueues. At one rank nothing crosses NVLink: the difference is the copies and
launches (b) makes. Rank 0 prints one JSON line with the card name and power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# (name, Hq, Hkv, D) packed K and V slices, or (name, None, (W0, W1), None) two dense tensors
MODELS = (("llama3-8b", 32, 8, 128), ("llama3-70b", 64, 8, 128), ("mla", None, (512, 64), None))
SEQ = (32768, 131072)
CHUNKS = 2
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


def _model(n: int, sl: int, widths, es: int) -> dict:
    """Per rank and call, from the shapes: HBM bytes read + written on this rank, and the kernels or collective calls enqueued. x is a
    shard (S_l * W), f a full tensor (N * S_l * W). Gather: (a) reads x, and every rank's pushes write f here; (b) densifies x (2x),
    all_gather reads x and writes f, index_select reads and writes f (2f). Reduce-scatter: (a) reads f (pulled by every rank) and writes
    x; (b) index_select (2f), reduce_scatter reads f and writes x, copy into the slice (2x)."""
    xs = sum(sl * w * es for w in widths)
    fs = n * xs
    return {"gather": {"fused": {"hbm": xs + fs, "ops": 1}, "unfused": {"hbm": 2 * xs + (xs + fs) + 2 * fs, "ops": 3 * len(widths)}},
            "reduce_scatter": {"fused": {"hbm": fs + xs, "ops": 1}, "unfused": {"hbm": 2 * fs + (fs + xs) + 2 * xs, "ops": 3 * len(widths)}}}


def _max_ulp(a, b) -> int:
    """The largest difference in bf16 ulps between two bf16 tensors of finite values (ordered as sign-magnitude integers)."""
    import torch
    def key(t):
        i = t.view(torch.int16).to(torch.int32)
        return torch.where(i < 0, -(i & 0x7FFF), i)
    return int((key(a) - key(b)).abs().max()) if a.numel() else 0


def main() -> int:
    argparse.ArgumentParser(description=__doc__.split("\n")[0]).parse_args()
    import torch
    from container_engine_accelerators_b200.ops import coll
    dt, es, B = torch.bfloat16, 2, 1
    if "WORLD_SIZE" in os.environ:
        rank, world, dev = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", 0))
    else:
        rank, world, dev = 0, 1, 0
    torch.cuda.set_device(dev)
    # the arena holds, for the largest shape, the fused fulls, the unfused send and receive buffers, and the gradient fulls
    sl_max = max(SEQ) // world
    wmax = max(2 * m[2] * m[3] if m[1] else sum(m[2]) for m in MODELS)
    arena_mb = (sl_max * wmax * es * (4 * world + 2) >> 20) + 256
    if world > 1:
        comm = coll.Comm.from_env(arena_mb=arena_mb, tag="context_kv_perf")
    else:
        (comm,) = coll.Comm.init_all([dev], arena_mb=arena_mb)
    st = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    shapes, matches = [], True
    for name, hq, kv, D in MODELS:
        for S in SEQ:
            sl = S // world
            gen = torch.Generator("cuda").manual_seed(S + rank + len(name))
            if hq is not None:
                widths = (kv * D, kv * D)
                row = (hq + 2 * kv) * D
                cols = (hq * D, (hq + kv) * D)
            else:
                widths = kv
                row = None
            arena = []

            def empty(shape):
                n = 1
                for d in shape:
                    n *= d
                t = comm.empty(n, dt)
                arena.append(t)
                return t.view(shape)

            if row is not None:
                qkv = torch.randn(B * sl, row, device="cuda", generator=gen).to(dt)
                xs = [qkv[:, c:c + w].view(B, sl, w) for c, w in zip(cols, widths)]
                dqkv_a = torch.zeros(B * sl, row, dtype=dt, device="cuda")
                dqkv_b = torch.zeros(B * sl, row, dtype=dt, device="cuda")
                dxa = [dqkv_a[:, c:c + w].view(B, sl, w) for c, w in zip(cols, widths)]
                dxb = [dqkv_b[:, c:c + w].view(B, sl, w) for c, w in zip(cols, widths)]
            else:
                xs = [torch.randn(B, sl, w, device="cuda", generator=gen).to(dt) for w in widths]
                dxa = [torch.zeros(B, sl, w, dtype=dt, device="cuda") for w in widths]
                dxb = [torch.zeros(B, sl, w, dtype=dt, device="cuda") for w in widths]
            fa = [empty((B, S, w)) for w in widths]                          # fused gather outputs
            send = [empty((B, sl, w)) for w in widths]                       # unfused gather: dense shard, then all_gather
            recv = [empty((world, B, sl, w)) for w in widths]
            fb = [torch.empty(B, S, w, dtype=dt, device="cuda") for w in widths]
            grads = [empty((B, S, w)) for w in widths]                       # dK / dV over the whole sequence (arena: the fused call pulls)
            for gr in grads:
                gr.copy_(torch.randn(gr.shape, device="cuda", generator=gen).to(dt))
            rs_in = [empty((world, B, sl, w)) for w in widths]               # unfused reduce-scatter: chunk order, then reduce_scatter
            rs_out = [empty((B, sl, w)) for w in widths]
            c = sl // CHUNKS
            idx = torch.empty(world * sl, dtype=torch.int64)                 # token g is at chunk-order position idx[g] = s * S_l + t
            for s in range(world):
                for k in range(CHUNKS):
                    g0 = (s if k == 0 else 2 * world - 1 - s) * c
                    idx[g0:g0 + c] = s * sl + k * c + torch.arange(c)
            idx = idx.cuda()
            inv = torch.empty_like(idx)
            inv[idx] = torch.arange(world * sl, device="cuda")                  # chunk-order position p holds token inv[p]

            def fused_ag():
                comm.all_gather_context(xs, fa, chunks=CHUNKS, stream=st)

            def unfused_ag():
                for x, s_, r_, f in zip(xs, send, recv, fb):
                    s_.copy_(x)
                    comm.all_gather(s_.view(-1), r_.view(-1), stream=st)
                    torch.index_select(r_.permute(1, 0, 2, 3).reshape(B, world * sl, -1), 1, idx, out=f)

            def fused_rs():
                comm.reduce_scatter_context(grads, dxa, chunks=CHUNKS, stream=st)

            def unfused_rs():
                for gr, ri, ro, d in zip(grads, rs_in, rs_out, dxb):
                    torch.index_select(gr, 1, inv, out=ri.view(B, world * sl, -1))      # B = 1: [S, W] is [N, 1, S_l, W]
                    comm.reduce_scatter(ri.view(-1), ro.view(-1), stream=st)
                    d.copy_(ro)

            for kind, fused, unfused in (("gather", fused_ag, unfused_ag), ("reduce_scatter", fused_rs, unfused_rs)):
                for t in (fa + fb) if kind == "gather" else (dxa + dxb):       # poisoned, so an unwritten byte cannot match
                    t.view(torch.int16).fill_(0x7B7B)
                fused()
                unfused()
                torch.cuda.synchronize()
                got, want = (fa, fb) if kind == "gather" else (dxa, dxb)
                ulp = 0
                ok = all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(got, want))
                if kind == "reduce_scatter" and not ok:
                    ulp = max(_max_ulp(a.contiguous(), b.contiguous()) for a, b in zip(got, want))
                    ok = ulp <= 2
                matches = matches and ok
                moved = sum(x.numel() for x in xs) * es
                iters = max(5, min(200, (2 << 30) // (moved * max(world, 1))))
                for f in (fused, unfused):
                    for _ in range(3):
                        f()
                per = {"fused": [], "unfused": []}
                for _ in range(ROUNDS):
                    for which, f in (("fused", fused), ("unfused", unfused)):
                        torch.cuda.synchronize()
                        e0.record(st)
                        for _ in range(iters):
                            f()
                        e1.record(st)
                        e1.synchronize()
                        per[which].append(e0.elapsed_time(e1) * 1e3 / iters)
                med = {k: round(sorted(t)[len(t) // 2], 2) for k, t in per.items()}
                shapes.append({"op": kind, "model": name, "widths": list(widths), "seq": S, "seq_local": sl, "shard_bytes": moved,
                               "fused_us": med["fused"], "unfused_us": med["unfused"], "matches": ok, "max_ulp": ulp,
                               "per_rank": _model(world, sl, widths, es)[kind]})
            torch.cuda.synchronize()
            for t in arena:
                comm.release(t)
    comm.check_async_error()
    if rank == 0:
        print(json.dumps({"metric": "context_kv", "ranks": world, "dtype": "bf16", "batch": B, "chunks": CHUNKS, **_card(dev), "shapes": shapes,
                          "matches": matches}), flush=True)
    torch.cuda.synchronize()
    comm.destroy()
    return 0 if matches else 1


if __name__ == "__main__":
    sys.exit(main())
