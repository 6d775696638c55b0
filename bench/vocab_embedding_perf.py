#!/usr/bin/env python
"""vocab_embedding_perf — the vocab-parallel embedding of a tensor-parallel input layer, fused, against Megatron's composition on the
same communicator.

    python bench/vocab_embedding_perf.py                                                          # one rank on cuda:0
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 bench/vocab_embedding_perf.py   # one GPU per rank

For (V, H) in {(128256, 4096) Llama-3-8B, (128256, 8192) Llama-3-70B, (152064, 3584) Qwen2-7B}, T in {4096, 8192, 16384, 32768}
and two id distributions (uniform, and every token the same id, a padding id: the skewed case whose one row folds all T tokens), a
bf16 table [V / N, H] per rank and an fp32 main_grad, it times device-side
  (a) comm.vocab_parallel_embedding and comm.vocab_parallel_embedding_backward (accumulate=0);
  (b) Megatron's composition on the same Comm: the mask, the shift, the masked_fill, F.embedding of the local shard, the zeroing of the
      masked rows and an all_reduce of [T, H] (sequence parallel: a reduce_scatter); backward a local embedding_dense_backward over the
      masked ids into fp32 (sequence parallel: an all_gather of the [T / N, H] gradient first). At one rank (b) is F.embedding and its
      backward.
TP and SP are both timed with more than one rank. The variants alternate in five rounds within one process and the median per call is
reported. bytes: what each arm must move, from shapes: (a) forward T·H·2 read + written (T / N rows with SP), backward T·H·2 read plus
V/N·H·4 written; the bandwidth is those bytes over the time, against the H100 SXM's 3.35 TB/s. Rank 0 prints one JSON line per shape
with the card name, power limit and SM clock read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MODELS = ((128256, 4096), (128256, 8192), (152064, 3584))
TOKENS = (4096, 8192, 16384, 32768)
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
    p.add_argument("--models", type=str, nargs="*", default=[f"{v}:{h}" for v, h in MODELS], help="V:H pairs")
    p.add_argument("--ids", type=str, nargs="*", default=["uniform", "same"], choices=["uniform", "same"])
    args = p.parse_args()
    import torch
    import torch.nn.functional as Fn
    from container_engine_accelerators_b200.ops import coll
    if "WORLD_SIZE" in os.environ:
        rank, world, dev = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", 0))
    else:
        rank, world, dev = 0, 1, 0
    torch.cuda.set_device(dev)
    card = _card(dev)
    comm = coll.Comm.init_all([dev], arena_mb=8192)[0] if world == 1 else coll.Comm.from_env(arena_mb=8192)
    st = torch.cuda.current_stream()

    def timed(fn, reps):
        fn()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(reps):
            fn()
        e.record()
        e.synchronize()
        return s.elapsed_time(e) * 1e3 / reps          # µs

    for mh in args.models:
        V, H = (int(x) for x in mh.split(":"))
        vl = V // world
        wb = comm.empty(vl * H, torch.bfloat16)
        w = wb.view(vl, H)
        w.normal_()
        for T, dist in [(t, d) for t in args.tokens for d in args.ids]:
            ids = torch.randint(0, vl * world, (T,), device="cuda", generator=torch.Generator("cuda").manual_seed(T))
            if dist == "same":
                ids.fill_(3)
            lo, hi = rank * vl, (rank + 1) * vl
            for sp in ([False] if world == 1 else [False, True]):
                nr = T // world if sp else T
                db = comm.empty(nr * H, torch.bfloat16)
                dout = db.view(nr, H)
                dout.normal_()
                dw = torch.empty(vl, H, dtype=torch.float32, device="cuda")
                full_grad = torch.empty(T, H, dtype=torch.bfloat16, device="cuda")

                def fused_f():
                    return comm.vocab_parallel_embedding(ids, w, sequence_parallel=sp, stream=st)

                def fused_b():
                    comm.vocab_parallel_embedding_backward(ids, dout, dw, sequence_parallel=sp, stream=st)

                def comp_f():
                    if world == 1:
                        return Fn.embedding(ids, w)
                    mask = (ids < lo) | (ids >= hi)
                    m = (ids - lo).masked_fill(mask, 0)
                    out = Fn.embedding(m, w)
                    out[mask] = 0
                    if sp:
                        o = torch.empty(nr, H, dtype=out.dtype, device="cuda")
                        comm.reduce_scatter(out, o)
                        return o
                    comm.all_reduce(out)
                    return out

                def comp_b():
                    g = dout
                    if world > 1 and sp:
                        comm.all_gather(dout, full_grad)
                        g = full_grad
                    m = ids if world == 1 else (ids - lo).masked_fill((ids < lo) | (ids >= hi), 0)
                    torch.ops.aten.embedding_dense_backward(g.float(), m, vl, -1, False)

                reps = 20
                res = {k: [] for k in ("fused_fwd", "fused_bwd", "comp_fwd", "comp_bwd")}
                for _ in range(ROUNDS):
                    res["fused_fwd"].append(timed(fused_f, reps))
                    res["comp_fwd"].append(timed(comp_f, reps))
                    res["fused_bwd"].append(timed(fused_b, reps))
                    res["comp_bwd"].append(timed(comp_b, reps))
                med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
                same = bool(torch.equal(fused_f().view(torch.int16), comp_f().view(torch.int16)))
                fwd_bytes = 2 * nr * H * 2                                   # the rows read and written
                bwd_bytes = T * H * 2 // (world if sp else 1) + vl * H * 4   # dout read (this rank's share), dweight written
                if rank == 0:
                    print(json.dumps({**card, "ranks": world, "V": V, "H": H, "T": T, "ids": dist, "sequence_parallel": sp,
                                      **{k + "_us": round(v, 1) for k, v in med.items()},
                                      "fwd_bytes": fwd_bytes, "bwd_bytes": bwd_bytes,
                                      "fused_fwd_tbs": round(fwd_bytes / med["fused_fwd"] / 1e6, 3),
                                      "fused_bwd_tbs": round(bwd_bytes / med["fused_bwd"] / 1e6, 3), "hbm_tbs": HBM_TBS,
                                      "forward_equal": same}), flush=True)
                comm.release(db)
        comm.release(wb)
    comm.destroy()
    return 0


if __name__ == "__main__":
    sys.exit(main())
