#!/usr/bin/env python
"""allreduce_rmsnorm_perf — the pre-norm step of a tensor-parallel block, fused against the three calls it replaces.

    python bench/allreduce_rmsnorm_perf.py                     # one rank, cuda:0
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 bench/allreduce_rmsnorm_perf.py
    python bench/allreduce_rmsnorm_perf.py --quantize e4m3:128  # the FP8 output for an FP8 GEMM (see below)

For each (tokens, hidden) of the decode and prefill shapes below, bf16: device-timed calls of
(a) comm.all_reduce_rms_norm(x, residual, gamma, out): one kernel, residual += all_reduce(x) in place and out = rms_norm(residual);
(b) comm.all_reduce(x) in place, residual.add_(x), F.rms_norm(residual, (hidden,), gamma, eps): what a caller writes today.
The two are timed alternately in rounds within one process (median per call reported), with x, residual and out in the arena.
At one rank nothing crosses NVLink (and the in-place identity all-reduce launches nothing), so the difference is the saved HBM passes
and launches. matches says that on fresh data (a) left the residual bit for bit as (b) did, and that its out lies within 2 bf16 ulp of
(b)'s F.rms_norm (more ranks: the residual within 2 ulp too). Rank 0 prints one JSON line.

With --quantize WIRE:BLOCK (WIRE e4m3 or e5m2, BLOCK 16 .. 512) the same shapes, rounds and medians time instead
(a) comm.all_reduce_rms_norm_quantized(x, residual, gamma, q, scales): one kernel, out quantised to WIRE with one fp32 scale per 1 x BLOCK;
(b) comm.all_reduce_rms_norm(x, residual, gamma, out), then the cheapest PyTorch quantise a caller would write: amax per block, two true
    divisions, the saturating cast. It leaves out the amax == 0 guard, which no block of these inputs needs.
matches then says that on fresh data (a) and (b) agree bit for bit on q, the scales and the residual (at rank 0)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TOKENS = (1, 16, 128, 1024, 4096, 16384)
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


def _wire_block(v: str):
    import torch
    wire, _, block = v.partition(":")
    wires = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}
    if wire not in wires or not block.isdigit() or int(block) not in (16, 32, 64, 128, 256, 512):
        raise argparse.ArgumentTypeError("WIRE:BLOCK: WIRE e4m3 or e5m2, BLOCK 16, 32, 64, 128, 256 or 512")
    return wire, wires[wire], int(block)


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--quantize", type=_wire_block, metavar="WIRE:BLOCK", help="time the FP8 output instead (see the module docstring)")
    args = ap.parse_args()
    import torch
    import torch.nn.functional as F
    from container_engine_accelerators_b200.ops import coll
    if args.quantize:
        return _quantized(*args.quantize)
    rank, world, lr = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(lr)
    dt = torch.bfloat16
    max_bytes = max(TOKENS) * max(HIDDEN) * 2
    comm = coll.Comm.from_env(arena_mb=(4 * max_bytes >> 20) + 256, tag="rmsnorm_perf")
    st = torch.cuda.current_stream()
    xa, ra, oa = (comm.empty(max(TOKENS) * max(HIDDEN), dt) for _ in range(3))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    shapes, matches = [], True
    for hidden in HIDDEN:
        gamma = (torch.rand(hidden, device="cuda", generator=torch.Generator("cuda").manual_seed(hidden)) + 0.5).to(dt)
        for tokens in TOKENS:
            n = tokens * hidden
            x, res, out = xa[:n].view(tokens, hidden), ra[:n].view(tokens, hidden), oa[:n].view(tokens, hidden)
            g = torch.Generator("cuda").manual_seed(tokens * 131 + hidden + rank)
            x0 = torch.randn(tokens, hidden, device="cuda", generator=g).to(dt)
            res0 = (torch.randn(tokens, hidden, device="cuda", generator=torch.Generator("cuda").manual_seed(tokens + hidden)) * 2).to(dt)

            def fused():
                comm.all_reduce_rms_norm(x, res, gamma, out, eps=EPS, stream=st)

            def three_calls():
                comm.all_reduce(x, stream=st)
                res.add_(x)
                return F.rms_norm(res, (hidden,), gamma, EPS)

            # matches, on fresh data
            x.copy_(x0); res.copy_(res0)
            fused()
            h_f, o_f = res.clone(), out.clone()
            x.copy_(x0); res.copy_(res0)
            y = three_calls()
            torch.cuda.synchronize()
            near = lambda a, b: bool(((a.float() - b.float()).abs() <= 2 * 2.0 ** -7 * b.float().abs() + 1e-30).all())   # 2 bf16 ulp
            # more ranks: (b) rounds the all-reduce to bf16 before the add, so its residual may differ in the last place
            ok = (torch.equal(h_f.view(torch.int16), res.view(torch.int16)) if world == 1 else near(h_f, res)) and near(o_f, y)
            matches = matches and ok
            iters = max(10, min(300, (1 << 30) // (n * 2)))
            per = {"fused": [], "three_call": []}
            for f in (fused, three_calls):
                for _ in range(3):
                    f()
            for _ in range(ROUNDS):
                for name, f in (("fused", fused), ("three_call", three_calls)):
                    x.copy_(x0); res.copy_(res0)
                    torch.cuda.synchronize()
                    e0.record(st)
                    for _ in range(iters):
                        f()
                    e1.record(st)
                    e1.synchronize()
                    per[name].append(e0.elapsed_time(e1) * 1e3 / iters)
            med = {k: sorted(v)[len(v) // 2] for k, v in per.items()}
            shapes.append({"tokens": tokens, "hidden": hidden, "fused_us": round(med["fused"], 2), "three_call_us": round(med["three_call"], 2),
                           "speedup": round(med["three_call"] / med["fused"], 3), "matches": ok})
    comm.check_async_error()
    if rank == 0:
        print(json.dumps({"metric": "allreduce_rmsnorm", "ranks": world, "dtype": "bf16", **_card(lr), "eps": EPS, "shapes": shapes,
                          "matches": matches}), flush=True)
    torch.cuda.synchronize()
    for t in (xa, ra, oa):
        comm.release(t)
    comm.destroy()
    return 0 if matches else 1


def _quantized(wire_name: str, wire, block: int) -> int:
    import torch
    from container_engine_accelerators_b200.ops import coll
    rank, world, lr = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(lr)
    dt = torch.bfloat16
    max_elems = max(TOKENS) * max(HIDDEN)
    comm = coll.Comm.from_env(arena_mb=(4 * max_elems * 2 >> 20) + 256, tag="rmsnorm_quant_perf")
    st = torch.cuda.current_stream()
    xa, ra, oa = (comm.empty(max_elems, dt) for _ in range(3))
    qa, sa = comm.empty(max_elems, wire), comm.empty(max_elems // block, torch.float32)
    fmax = torch.tensor(torch.finfo(wire).max, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    shapes, matches = [], True
    for hidden in HIDDEN:
        gamma = (torch.rand(hidden, device="cuda", generator=torch.Generator("cuda").manual_seed(hidden)) + 0.5).to(dt)
        for tokens in TOKENS:
            n = tokens * hidden
            x, res, out = xa[:n].view(tokens, hidden), ra[:n].view(tokens, hidden), oa[:n].view(tokens, hidden)
            q, s = qa[:n].view(tokens, hidden), sa[:n // block].view(tokens, hidden // block)
            g = torch.Generator("cuda").manual_seed(tokens * 131 + hidden + rank)
            x0 = torch.randn(tokens, hidden, device="cuda", generator=g).to(dt)
            res0 = (torch.randn(tokens, hidden, device="cuda", generator=torch.Generator("cuda").manual_seed(tokens + hidden)) * 2).to(dt)

            def fused():
                comm.all_reduce_rms_norm_quantized(x, res, gamma, q, s, block=block, wire=wire, eps=EPS, stream=st)
                return q, s

            def two_step():
                comm.all_reduce_rms_norm(x, res, gamma, out, eps=EPS, stream=st)
                v = out.view(tokens, -1, block).float()
                amax = v.abs().amax(dim=-1, keepdim=True)
                yq = (v * (fmax / amax)).clamp(-fmax, fmax).to(wire)     # fmax a tensor: true divisions, not reciprocal multiplies
                return yq.view(tokens, hidden), (amax / fmax).view(tokens, -1)

            # matches, on fresh data
            x.copy_(x0); res.copy_(res0)
            q_f, s_f = (t.clone() for t in fused())
            h_f = res.clone()
            x.copy_(x0); res.copy_(res0)
            q_b, s_b = two_step()
            torch.cuda.synchronize()
            ok = (torch.equal(h_f.view(torch.int16), res.view(torch.int16)) and torch.equal(q_f.view(torch.uint8), q_b.view(torch.uint8)) and
                  torch.equal(s_f.view(torch.int32), s_b.view(torch.int32)))
            matches = matches and ok
            iters = max(10, min(300, (1 << 30) // (n * 2)))
            per = {"fused": [], "two_step": []}
            for f in (fused, two_step):
                for _ in range(3):
                    f()
            for _ in range(ROUNDS):
                for name, f in (("fused", fused), ("two_step", two_step)):
                    x.copy_(x0); res.copy_(res0)
                    torch.cuda.synchronize()
                    e0.record(st)
                    for _ in range(iters):
                        f()
                    e1.record(st)
                    e1.synchronize()
                    per[name].append(e0.elapsed_time(e1) * 1e3 / iters)
            med = {k: sorted(v)[len(v) // 2] for k, v in per.items()}
            shapes.append({"tokens": tokens, "hidden": hidden, "fused_us": round(med["fused"], 2), "two_step_us": round(med["two_step"], 2),
                           "speedup": round(med["two_step"] / med["fused"], 3), "matches": ok})
    comm.check_async_error()
    if rank == 0:
        print(json.dumps({"metric": "allreduce_rmsnorm_quantized", "ranks": world, "dtype": "bf16", "wire": wire_name, "block": block, **_card(lr),
                          "eps": EPS, "shapes": shapes, "matches": matches}), flush=True)
    torch.cuda.synchronize()
    for t in (xa, ra, oa, qa, sa):
        comm.release(t)
    comm.destroy()
    return 0 if matches else 1


if __name__ == "__main__":
    sys.exit(main())
