#!/usr/bin/env python
"""fsdp_shards_perf — the FSDP parameter all-gather and gradient reduce-scatter of one transformer block, fused, against the composition
FSDP2 (torch.distributed.fsdp.fully_shard) builds around plain all_gather and reduce_scatter.

    python bench/fsdp_shards_perf.py                                                          # one rank on cuda:0
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 bench/fsdp_shards_perf.py   # one GPU per rank

For a Llama-3-8B block (H 4096, MLP 14336, K/V 1024) and a Llama-3-70B block (H 8192, MLP 28672, K/V 1024) — q, k, v, o, gate, up,
down and two RMSNorm weights, sharded along dim 0 with ceil(d / N) rows per rank — it times device-side calls of
  gather  fp32 shards to bf16 parameters
          (a) comm.all_gather_shards: one kernel, the cast on the owning rank;
          (b) FSDP2's: a cast per parameter, torch.ops.fsdp.all_gather_copy_in into the flat input, comm.all_gather, and
              torch.ops.fsdp.split_with_sizes_copy into the padded unsharded parameters;
  reduce-scatter  bf16 gradients to fp32 sharded gradients, scaled by 1 / N and accumulated (the second micro-batch)
          (a) comm.reduce_scatter_shards(scale=1/N, accumulate=True): one kernel;
          (b) FSDP2's with reduce_dtype=float32: torch.ops.fsdp.chunk_cat (casting to fp32) into the flat input, comm.reduce_scatter,
              the divide, and _foreach_add_ into the sharded gradients.
The two are alternated in five rounds within one process and the median per call is reported. matches says whether (a) and (b)
produced the same output: the gather bit for bit; the reduce-scatter bit for bit on gradients whose fp32 sums are exact (the two sum in
different rank orders). bytes gives, per rank and call, computed from the shapes, what each variant reads from and writes to the rank's
HBM (the pushes and pulls of peers touch it too), and ops how many kernels or collective calls each enqueues. At one rank nothing
crosses NVLink: the difference is the copies and launches (b) makes. Rank 0 prints one JSON line with the card name and power limit
read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MODELS = (("llama3-8b", 4096, 14336, 1024), ("llama3-70b", 8192, 28672, 1024))
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


def block(H: int, F: int, KV: int):
    return [(H, H), (KV, H), (KV, H), (H, H), (F, H), (F, H), (H, F), (H,), (H,)]


def _model(n: int, shapes, rank: int) -> dict:
    """Per rank and call, from the shapes: HBM bytes read + written on this rank, and the kernels or collective calls enqueued. s is
    this rank's rows (fp32 shard bytes s4, bf16 s2), u the block (bf16 bytes u2, fp32 u4), P the padded flat buffers (N * p rows).
    Gather: (a) reads s4, every rank's pushes write u2 here; (b) casts (s4 + s2), copies in (2 s2), all_gather reads s2 and writes P2,
    copies out (2 P2). Reduce-scatter: (a) reads u2 (pulled by every rank), reads and writes s4; (b) chunk_cat reads u2 and writes P4,
    reduce_scatter reads P4 and writes s4, the divide (2 s4), the add (3 s4)."""
    s = u = P = 0
    for sh in shapes:
        d, W = sh[0], 1
        for e in sh[1:]:
            W *= e
        p = -(-d // n)
        s += max(0, min(d - rank * p, p)) * W
        u += d * W
        P += n * p * W
    k = len(shapes)
    return {"gather": {"fused": {"hbm": 4 * s + 2 * u, "ops": 1}, "unfused": {"hbm": 6 * s + 4 * s + 2 * s + 2 * P + 4 * P, "ops": k + 3}},
            "reduce_scatter": {"fused": {"hbm": 2 * u + 8 * s, "ops": 1},
                               "unfused": {"hbm": 2 * u + 4 * P + 4 * P + 4 * s + 8 * s + 12 * s, "ops": 3 + 1}}}


def main() -> int:
    argparse.ArgumentParser(description=__doc__.split("\n")[0]).parse_args()
    import torch
    import torch.distributed.fsdp._fully_shard._fsdp_collectives  # noqa: F401  (registers torch.ops.fsdp)
    from container_engine_accelerators_b200.ops import coll
    if "WORLD_SIZE" in os.environ:
        rank, world, dev = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", 0))
    else:
        rank, world, dev = 0, 1, 0
    torch.cuda.set_device(dev)
    # the arena holds, for the largest block: the fused bf16 fulls and bf16 gradients, the unfused bf16 input and output, and the
    # unfused fp32 reduce-scatter input and output
    big = max(sum(_numel(sh) for sh in block(*m[1:])) for m in MODELS)
    arena_mb = ((big * 2 * 2 + big * 2 * (1 + 1 / world) + big * 4 * (1 + 1 / world)) * 1.02 / 2**20).__ceil__() + 256
    if world > 1:
        comm = coll.Comm.from_env(arena_mb=arena_mb, tag="fsdp_shards_perf")
    else:
        (comm,) = coll.Comm.init_all([dev], arena_mb=arena_mb)
    st = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    results, matches = [], True
    for name, H, F, KV in MODELS:
        shapes = block(H, F, KV)
        ds = [sh[0] for sh in shapes]
        Ws = [_numel(sh[1:]) for sh in shapes]
        ps = [-(-d // world) for d in ds]
        ks = [max(0, min(d - rank * p, p)) for d, p in zip(ds, ps)]
        sizes = [p * W for p, W in zip(ps, Ws)]
        numel = sum(sizes)
        gen = torch.Generator("cuda").manual_seed(17 + rank)
        arena = []

        def empty(shape, dt):
            t = comm.empty(_numel(shape), dt)
            arena.append(t)
            return t.view(shape)

        # FSDP2's sharded parameters are padded to p rows; the padding is zero
        shards = []
        for p, k, sh in zip(ps, ks, shapes):
            x = torch.zeros((p, *sh[1:]), device="cuda")
            x[:k] = torch.randn((k, *sh[1:]), device="cuda", generator=gen)
            shards.append(x)
        fulls = [empty(sh, torch.bfloat16) for sh in shapes]                     # (a): the unsharded parameters
        ag_in = empty((numel,), torch.bfloat16)                                  # (b): the flat input and output, and the padded params
        ag_out = empty((world * numel,), torch.bfloat16)
        padded = [torch.empty((world * p, *sh[1:]), dtype=torch.bfloat16, device="cuda") for p, sh in zip(ps, shapes)]
        # gradients: multiples of 1/8 below 16, so every fp32 sum is exact and the two rank orders agree
        grads = [empty(sh, torch.bfloat16) for sh in shapes]
        for gr in grads:
            gr.copy_((torch.randint(-128, 128, gr.shape, device="cuda", generator=gen).float() / 8).to(torch.bfloat16))
        old = [torch.randint(-64, 64, (p, *sh[1:]), device="cuda", generator=gen).float() / 4 for p, sh in zip(ps, shapes)]
        acc_a = [o.clone() for o in old]
        acc_b = [o.clone() for o in old]
        rs_in = empty((world * numel,), torch.float32)
        rs_out = empty((numel,), torch.float32)

        def fused_ag():
            comm.all_gather_shards(shards, fulls, stream=st)

        def unfused_ag():
            cast = [x.to(torch.bfloat16).view(-1) for x in shards]
            torch.ops.fsdp.all_gather_copy_in(cast, ag_in, sizes, numel, 0)
            comm.all_gather(ag_in, ag_out, stream=st)
            torch.ops.fsdp.split_with_sizes_copy(ag_out.view(world, -1), sizes, dim=1, out=[q.view(world, -1) for q in padded])

        def fused_rs():
            comm.reduce_scatter_shards(grads, acc_a, scale=1.0 / world, accumulate=True, stream=st)

        def unfused_rs():
            torch.ops.fsdp.chunk_cat(grads, 0, world, out=rs_in.view(world, -1))
            comm.reduce_scatter(rs_in, rs_out, stream=st)
            rs_out.div_(world)
            torch._foreach_add_(acc_b, [q.view(a.shape) for q, a in zip(torch.split(rs_out, sizes), acc_b)])

        for kind, fused, unfused in (("gather", fused_ag, unfused_ag), ("reduce_scatter", fused_rs, unfused_rs)):
            if kind == "gather":
                for t in fulls + padded:                                        # poisoned, so an unwritten byte cannot match
                    t.view(torch.int16).fill_(0x7B7B)
            fused()
            unfused()
            torch.cuda.synchronize()
            if kind == "gather":
                ok = all(torch.equal(f.view(torch.int16), q[:d].view(torch.int16)) for f, q, d in zip(fulls, padded, ds))
            else:
                ok = all(torch.equal(a[:k], b[:k]) for a, b, k in zip(acc_a, acc_b, ks))
            matches = matches and ok
            iters = max(5, min(100, (4 << 30) // (sum(d * W for d, W in zip(ds, Ws)) * 2 * max(world, 1))))
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
            results.append({"op": kind, "model": name, "hidden": H, "mlp": F, "kv": KV, "tensors": len(shapes),
                            "dtypes": "f32->bf16" if kind == "gather" else "bf16->f32, scale 1/N, accumulate",
                            "fused_us": med["fused"], "unfused_us": med["unfused"], "speedup": round(med["unfused"] / med["fused"], 2),
                            "matches": ok, "per_rank": _model(world, shapes, rank)[kind]})
        torch.cuda.synchronize()
        for t in arena:
            comm.release(t)
    comm.check_async_error()
    if rank == 0:
        print(json.dumps({"metric": "fsdp_shards", "ranks": world, **_card(dev), "shapes": results, "matches": matches}), flush=True)
    torch.cuda.synchronize()
    comm.destroy()
    return 0 if matches else 1


def _numel(shape) -> int:
    n = 1
    for d in shape:
        n *= d
    return n


if __name__ == "__main__":
    sys.exit(main())
