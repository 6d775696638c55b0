#!/usr/bin/env python
"""vocab_xent_perf — the vocab-parallel cross-entropy of a tensor-parallel LM head, fused, against Megatron's composition on the same
communicator.

    python bench/vocab_xent_perf.py                                                          # one rank on cuda:0
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 bench/vocab_xent_perf.py   # one GPU per rank

For tokens in {1024, 4096, 16384} and V in {32000, 128256, 151936}, bf16 logits [tokens, V / N] per rank, it times device-side
forward + backward of
  (a) comm.vocab_parallel_cross_entropy and comm.vocab_parallel_cross_entropy_backward: one kernel each;
  (b) Megatron's vocab_parallel_cross_entropy on the same Comm: logits.float(), the row max, all_reduce(MAX) (the generic kernel), the
      subtract, exp and sum, all_reduce(SUM), the masked gather of the target logit, a third all_reduce(SUM), the divide that keeps the
      fp32 softmax, and for the backward the one-hot subtract, the multiply by dloss and the cast to bf16;
  (c) at one rank, also F.cross_entropy(logits.float(), target) with its backward.
The variants alternate in five rounds within one process and the median per call is reported. matches: the loss of (a) within 1e-5
relative of (b)'s and every gradient element within one bf16 ulp of (b)'s (b's fp32 softmax is rounded once to bf16 as well). The
forward's bytes/s is the logits' bytes over (a)'s forward time alone, against the H100 SXM's 3.35 TB/s. Rank 0 prints one JSON line with
the card name, power limit and SM clock read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TOKENS = (1024, 4096, 16384)
VOCABS = (32000, 128256, 151936)
ROUNDS = 5
HBM_TBS = 3.35


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


def main() -> int:
    p = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    p.add_argument("--tokens", type=int, nargs="*", default=list(TOKENS))
    p.add_argument("--vocab", type=int, nargs="*", default=list(VOCABS))
    args = p.parse_args()
    import torch
    import torch.nn.functional as Fn
    from container_engine_accelerators_b200.ops import coll
    if "WORLD_SIZE" in os.environ:
        rank, world, dev = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", 0))
    else:
        rank, world, dev = 0, 1, 0
    torch.cuda.set_device(dev)
    if world > 1:
        comm = coll.Comm.from_env(arena_mb=256, tag="vocab_xent_perf")
    else:
        (comm,) = coll.Comm.init_all([dev], arena_mb=256)
    st = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    results, matches = [], True
    for V in args.vocab:
        vl = V // world
        for T in args.tokens:
            gen = torch.Generator("cuda").manual_seed(5)
            full = torch.randn(T, vl * world, device="cuda", generator=gen).mul_(4).to(torch.bfloat16)
            x = full[:, rank * vl:(rank + 1) * vl].contiguous()
            del full
            target = torch.randint(0, vl * world, (T,), device="cuda", generator=gen)
            dloss = torch.full((T,), 1.0 / T, device="cuda")
            lo, hi = rank * vl, (rank + 1) * vl
            red = comm.empty(T, torch.float32)

            def fused():
                loss, lse = comm.vocab_parallel_cross_entropy(x, target, stream=st)
                return loss, comm.vocab_parallel_cross_entropy_backward(x, target, lse, dloss, stream=st)

            def megatron():
                lf = x.float()
                m = lf.max(dim=-1)[0]
                red.copy_(m)
                comm.all_reduce(red, red, op=coll.MAX, stream=st)
                lf = lf - red.unsqueeze(1)
                mask = (target < lo) | (target >= hi)
                mt = (target - lo).masked_fill(mask, 0)
                pred = lf.gather(1, mt.unsqueeze(1)).squeeze(1).masked_fill(mask, 0.0)
                red.copy_(pred)
                comm.all_reduce(red, red, stream=st)
                pred = red.clone()
                e = lf.exp_()
                red.copy_(e.sum(dim=-1))
                comm.all_reduce(red, red, stream=st)
                loss = torch.log(red) - pred
                sm = e.div_(red.unsqueeze(1))                                  # kept for the backward
                g = sm.clone()
                rows = torch.arange(T, device="cuda")
                g[rows, mt] -= (~mask).float()
                g.mul_(dloss.unsqueeze(1))
                return loss, g.to(torch.bfloat16)

            def torch_ce():
                xr = x.float().requires_grad_()
                loss = Fn.cross_entropy(xr, target, reduction="none")
                (loss * dloss).sum().backward()
                return loss, xr.grad.to(torch.bfloat16)

            la, ga = fused()
            lb, gb = megatron()
            torch.cuda.synchronize()
            ok_loss = bool(torch.allclose(la, lb, rtol=1e-5, atol=1e-5))
            ulp = (ga.view(torch.int16).int() - gb.view(torch.int16).int()).abs()
            ok_grad = bool((ulp <= 1).all() | torch.equal(ga.float(), gb.float()))
            ok = ok_loss and ok_grad
            matches = matches and ok
            del la, lb, ga, gb
            variants = [("fused", fused), ("megatron", megatron)] + ([("torch", torch_ce)] if world == 1 else [])
            iters = max(3, min(50, (2 << 30) // (T * vl * 2)))
            for _, f in variants:
                for _ in range(2):
                    f()

            def fwd_only():
                comm.vocab_parallel_cross_entropy(x, target, stream=st)
            per = {k: [] for k, _ in variants}
            per["fused_forward"] = []
            for _ in range(ROUNDS):
                for which, f in variants + [("fused_forward", fwd_only)]:
                    torch.cuda.synchronize()
                    e0.record(st)
                    for _ in range(iters):
                        f()
                    e1.record(st)
                    e1.synchronize()
                    per[which].append(e0.elapsed_time(e1) * 1e3 / iters)
            med = {k: round(sorted(t)[len(t) // 2], 2) for k, t in per.items()}
            fwd_bytes = T * vl * 2
            results.append({"tokens": T, "vocab": V, "vocab_local": vl, "fused_us": med["fused"], "megatron_us": med["megatron"],
                            **({"torch_ce_us": med["torch"]} if world == 1 else {}), "fused_forward_us": med["fused_forward"],
                            "forward_tb_s": round(fwd_bytes / (med["fused_forward"] * 1e-6) / 1e12, 3),
                            "forward_share_of_hbm": round(fwd_bytes / (med["fused_forward"] * 1e-6) / (HBM_TBS * 1e12), 3),
                            "speedup_vs_megatron": round(med["megatron"] / med["fused"], 2), "matches": ok,
                            "max_grad_ulp": int(ulp.max().item())})
            print(f"tokens {T} V {V}: {results[-1]}", file=sys.stderr, flush=True)
            comm.release(red)
            del x
            torch.cuda.empty_cache()
    comm.check_async_error()
    if rank == 0:
        print(json.dumps({"metric": "vocab_xent", "ranks": world, "dtype": "bf16", **_card(dev), "shapes": results,
                          "matches": matches, "loss_rtol": 1e-5, "grad_ulp": 1}), flush=True)
    torch.cuda.synchronize()
    comm.destroy()
    return 0 if matches else 1


if __name__ == "__main__":
    sys.exit(main())
