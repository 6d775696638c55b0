#!/usr/bin/env python
"""ulysses_a2a_perf — the Ulysses all-to-all of sequence-parallel attention, fused, against the composition an attention layer writes
with plain all_to_all.

    python bench/ulysses_a2a_perf.py                                                          # one rank on cuda:0
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 bench/ulysses_a2a_perf.py   # one GPU per rank

B = 1, bf16, for Hq / Hkv / D of 32/8/128 (Llama-3-8B), 64/8/128 (Llama-3-70B), 32/32/128 (MHA) and 64/1/128 (MQA), and full
sequences S of 8k, 32k and 128k tokens (S_l = S / N per rank), it times device-side calls of
  seq->heads  (a) comm.all_to_all_seq_to_heads over q, k and v, the column slices of one packed [S_l, (Hq + 2 Hkv) * D] QKV projection
                  output: one kernel;
              (b) per tensor: repeat_interleave of K and V up to N heads when Hkv < N, permute + contiguous into [N, B, S_l, Hl, D],
                  comm.all_to_all, and (B > 1 only) permute back to [B, S, Hl, D];
  heads->seq  (a) comm.all_to_all_heads_to_seq of the [B, S, Hq / N, D] attention output: one kernel;
              (b) (B > 1 only) permute + contiguous, comm.all_to_all, and (N > 1 only) permute back into [B, S_l, Hq, D].
The two are alternated in five rounds within one process and the median per call is reported. Outputs are arena memory. matches says
that (a) and (b) produced the same bytes. bytes gives, per rank and call, computed from the shapes, what each variant reads from and
writes to the rank's HBM (the pushes of peers land there too), and ops how many kernels or collective calls each enqueues. At one rank
nothing crosses NVLink: the difference is the copies and launches (b) makes. Rank 0 prints one JSON line with the card name and power
limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HEADS = ((32, 8, 128), (64, 8, 128), (32, 32, 128), (64, 1, 128))
SEQ = (8192, 32768, 131072)
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


def _local(n: int, h: int) -> int:
    return h // n if h % n == 0 else 1


def _model(n: int, B: int, sl: int, heads, D: int, back: bool) -> dict:
    """Per rank and call, from the shapes: HBM bytes read + written on this rank (bf16), and the kernels or collective calls enqueued."""
    if back:
        t = B * n * sl * _local(n, heads[0]) * D * 2
        return {"fused": {"hbm": 2 * t, "ops": 1},
                "unfused": {"hbm": 2 * t * (1 + (B > 1) + (n > 1)), "ops": 1 + (B > 1) + (n > 1)}}
    fused = unfused = ops = 0
    for h in heads:
        x, t = B * sl * h * D * 2, B * n * sl * _local(n, h) * D * 2
        rep = h % n != 0
        fused += x + t
        unfused += (x + t if rep else 0) + (t if rep else x) + t + 2 * t + (2 * t if B > 1 else 0)
        ops += 1 + rep + 1 + (B > 1)
    return {"fused": {"hbm": fused, "ops": 1}, "unfused": {"hbm": unfused, "ops": ops}}


def main() -> int:
    argparse.ArgumentParser(description=__doc__.split("\n")[0]).parse_args()
    import torch
    from container_engine_accelerators_b200.ops import coll
    dt, B = torch.bfloat16, 1
    if "WORLD_SIZE" in os.environ:
        rank, world, dev = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", 0))
    else:
        rank, world, dev = 0, 1, 0
    torch.cuda.set_device(dev)
    # the arena holds the fused outputs, the unfused receive buffers and the heads->seq output of the largest shape
    sl_max = max(SEQ) // world
    tot = max(sum(B * world * sl_max * _local(world, h) * D for h in (hq, hkv, hkv)) for hq, hkv, D in HEADS)
    q_max = max(B * sl_max * hq * D for hq, _, D in HEADS)
    arena_mb = ((2 * tot + 2 * q_max) * 2 >> 20) + 256
    if world > 1:
        comm = coll.Comm.from_env(arena_mb=arena_mb, tag="ulysses_a2a_perf")
    else:
        (comm,) = coll.Comm.init_all([dev], arena_mb=arena_mb)
    st = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    shapes, matches = [], True
    for hq, hkv, D in HEADS:
        heads = (hq, hkv, hkv)
        if any(h % world and world % h for h in heads) or hq % world:
            continue
        for S in SEQ:
            sl = S // world
            hl = [_local(world, h) for h in heads]
            gen = torch.Generator("cuda").manual_seed(S + hq * 7 + hkv + rank)
            qkv = torch.randn(B * sl, sum(heads) * D, device="cuda", generator=gen).to(dt)
            cols = (0, hq, hq + hkv, hq + 2 * hkv)
            xs = [qkv[:, cols[i] * D:cols[i + 1] * D].view(B, sl, h, D) for i, h in enumerate(heads)]
            arena = []

            def empty(shape):
                n = 1
                for d in shape:
                    n *= d
                t = comm.empty(n, dt)
                arena.append(t)
                return t.view(shape)

            ys = [empty((B, S, hl[i], D)) for i in range(3)]                       # fused seq->heads outputs
            rv = [empty((world, B, sl, hl[i], D)) for i in range(3)]                # unfused receive buffers
            sd = [torch.empty(world, B, sl, hl[i], D, dtype=dt, device="cuda") for i in range(3)]
            uys = [r.permute(1, 0, 2, 3, 4).reshape(B, S, hl[i], D) if B == 1 else torch.empty(B, S, hl[i], D, dtype=dt, device="cuda")
                   for i, r in enumerate(rv)]
            xb = empty((B, sl, hq, D))                                             # fused heads->seq output
            ub = torch.empty(B, sl, hq, D, dtype=dt, device="cuda") if world > 1 else rv[0].view(B, sl, hq, D)

            def fused_s2h():
                comm.all_to_all_seq_to_heads(xs, ys, stream=st)

            def unfused_s2h():
                for i, h in enumerate(heads):
                    x = xs[i] if h % world == 0 else xs[i].repeat_interleave(world // h, dim=2)
                    sd[i].copy_(x.view(B, sl, world, hl[i], D).permute(2, 0, 1, 3, 4))
                    comm.all_to_all(sd[i].view(-1), rv[i].view(-1), stream=st)
                    if B > 1:
                        uys[i].copy_(rv[i].permute(1, 0, 2, 3, 4).reshape(B, S, hl[i], D))

            def fused_h2s():
                comm.all_to_all_heads_to_seq([ys[0]], [xb], stream=st)

            def unfused_h2s():
                y = ys[0].view(B, world, sl, hl[0], D).permute(1, 0, 2, 3, 4)
                src = y.reshape(-1) if B == 1 else sd[0].copy_(y).view(-1)
                comm.all_to_all(src, rv[0].view(-1), stream=st)
                if world > 1:
                    ub.copy_(rv[0].permute(1, 2, 0, 3, 4).reshape(B, sl, hq, D))

            for back, fused, unfused in ((False, fused_s2h, unfused_s2h), (True, fused_h2s, unfused_h2s)):
                for t in [xb, rv[0]] if back else ys + rv:                            # poisoned, so an unwritten byte cannot match
                    t.view(torch.int16).fill_(0x7B7B)
                fused()
                got = [xb.clone()] if back else [y.clone() for y in ys]
                unfused()
                torch.cuda.synchronize()
                want = [ub] if back else uys
                ok = all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(got, want))
                matches = matches and ok
                moved = sum(x.numel() for x in xs) * 2 if not back else ys[0].numel() * 2
                iters = max(5, min(200, (4 << 30) // moved))
                for f in (fused, unfused):
                    for _ in range(3):
                        f()
                per = {"fused": [], "unfused": []}
                for _ in range(ROUNDS):
                    for name, f in (("fused", fused), ("unfused", unfused)):
                        torch.cuda.synchronize()
                        e0.record(st)
                        for _ in range(iters):
                            f()
                        e1.record(st)
                        e1.synchronize()
                        per[name].append(e0.elapsed_time(e1) * 1e3 / iters)
                med = {k: round(sorted(t)[len(t) // 2], 2) for k, t in per.items()}
                shapes.append({"direction": "heads_to_seq" if back else "seq_to_heads", "hq": hq, "hkv": hkv, "d": D, "seq": S, "seq_local": sl,
                               "source_bytes": moved, "fused_us": med["fused"], "unfused_us": med["unfused"], "matches": ok,
                               "per_rank": _model(world, B, sl, heads, D, back)})
            torch.cuda.synchronize()
            for t in arena:
                comm.release(t)
    comm.check_async_error()
    if rank == 0:
        print(json.dumps({"metric": "ulysses_a2a", "ranks": world, "dtype": "bf16", "batch": B, **_card(dev), "shapes": shapes, "matches": matches}),
              flush=True)
    torch.cuda.synchronize()
    comm.destroy()
    return 0 if matches else 1


if __name__ == "__main__":
    sys.exit(main())
