#!/usr/bin/env python
"""Per-call cost of the one-rank copy: a bf16 identity all-reduce on a one-rank communicator, which is a device-to-device copy (the
copy-engine kernel from 1 MiB up). It is what every call of `bench.py --gpus 1` runs, so its fixed per-call cost F and its streaming
rate BW set the headline.

    python bench/one_rank_copy.py                                        # the library the package loads
    python bench/one_rank_copy.py --lib a/libb200coll.so --lib b/libb200coll.so --rounds 3

Each (round, library) runs in a child process with B200COLL_LIB pointing at that library, so two builds alternate in one process
tree. Per size: `--warmup` untimed calls, then `--steps` back-to-back calls through the public API timed with CUDA events, buffers
rotating through a 192 MiB window (larger than the 50 MB L2), as bench.py's harness does. Then a least-squares fit of
t = F + bytes / BW on relative error, over sizes >= --fit-min (below that the Python launch loop, not the GPU, sets the pace).
In the first round two yardsticks run as well, with the first library: the same call with B200COLL_BULK=0 (k_copy_scale, LDG/STG)
and torch's copy_ (a device-to-device memcpy). The card's name, power limit and max SM clock come from nvidia-smi, read only.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def sizes(lo: int, hi: int) -> list[int]:
    out, b = [], lo
    while b <= hi:
        out.append(b)
        b *= 2
    return out


def fit(rows: dict[int, float], fit_min: int) -> tuple[float, float]:
    """(F in us, BW in GB/s) minimising the relative error of t = F + bytes / BW over the sizes >= fit_min."""
    import numpy as np
    pts = [(b, t) for b, t in rows.items() if b >= fit_min]
    a = np.array([[1.0 / t, b / t] for b, t in pts])
    (f, k), *_ = np.linalg.lstsq(a, np.ones(len(pts)), rcond=None)
    return float(f), float(1e-3 / k)


def child(args) -> int:
    import torch
    from container_engine_accelerators_b200.parallel import harness
    torch.cuda.set_device(0)
    dist = harness.Dist()
    dtype = torch.bfloat16
    backend = harness.OursBackend(dist, max(args.max, harness.WINDOW) // 2 + 4096, dtype, tag="one_rank_copy")
    harness.seed_inputs(backend, dist, dtype)
    stream = torch.cuda.current_stream()
    st = stream.cuda_stream
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    arms = {"lib": {}, "torch": {}} if args.torch else {"lib": {}}
    launches0 = backend.launches()
    for nbytes in sizes(args.min, args.max):
        count = nbytes // 2
        slot = (nbytes + 4095) // 4096 * 4096
        slots = max(1, min(64, harness.WINDOW // slot))
        sb, rb = backend.send.data_ptr(), backend.recv.data_ptr()
        views = [(backend.send[i * slot // 2:i * slot // 2 + count], backend.recv[i * slot // 2:i * slot // 2 + count]) for i in range(slots)]
        calls = {"lib": lambda i: backend.launch("all_reduce", sb + (i % slots) * slot, rb + (i % slots) * slot, count, st),
                 "torch": lambda i: views[i % slots][1].copy_(views[i % slots][0])}
        for arm in arms:
            call = calls[arm]
            for i in range(args.warmup):
                call(i)
            torch.cuda.synchronize()
            e0.record(stream)
            for i in range(args.steps):
                call(i)
            e1.record(stream)
            torch.cuda.synchronize()
            arms[arm][nbytes] = e0.elapsed_time(e1) * 1e3 / args.steps
            last = views[(args.steps - 1) % slots]
            if arm == "lib" and not torch.equal(last[1].view(torch.int16), last[0].view(torch.int16)):
                raise SystemExit(f"one_rank_copy: the copy of {nbytes} bytes is not bit-exact")
    stats = backend.comm.stats()
    print(json.dumps({"us": arms, "launches": backend.launches() - launches0, "bulk_launches": stats["bulk_launches"],
                      "version": backend.version, "lib": backend.L._name}), flush=True)
    backend.close()
    return 0


def run_child(args, lib: str | None, env_extra: dict, torch_arm: bool) -> dict:
    env = dict(os.environ, **env_extra)
    if lib:
        env["B200COLL_LIB"] = os.path.abspath(lib)
    cmd = [sys.executable, os.path.abspath(__file__), "--child", "--min", str(args.min), "--max", str(args.max), "--steps", str(args.steps),
           "--warmup", str(args.warmup)] + (["--torch"] if torch_arm else [])
    out = subprocess.run(cmd, env=env, capture_output=True, text=True)
    if out.returncode != 0:
        raise SystemExit(f"one_rank_copy: child failed ({lib or 'default'} {env_extra}):\n{out.stderr[-3000:]}")
    res = json.loads(out.stdout.strip().splitlines()[-1])
    res["us"] = {arm: {int(b): t for b, t in rows.items()} for arm, rows in res["us"].items()}
    return res


def card() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or f"nvidia-smi printed nothing ({q.stderr.strip()[:200]})"
    except (OSError, subprocess.TimeoutExpired) as e:
        return f"nvidia-smi unavailable: {e}"


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="libb200coll.so to measure; repeat to alternate builds (default: the one the package loads)")
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--min", type=int, default=1 << 20)
    ap.add_argument("--max", type=int, default=1 << 30)
    ap.add_argument("--fit-min", type=int, default=8 << 20)
    ap.add_argument("--no-yardsticks", action="store_true")
    ap.add_argument("--json", help="also write every measurement to this file")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--torch", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)
    libs = args.lib or [None]
    gpu = card()
    print(f"# card: {gpu}", flush=True)
    runs = []      # (label, round, us rows)
    for rnd in range(args.rounds):
        for i, lib in enumerate(libs):
            yard = rnd == 0 and i == 0 and not args.no_yardsticks
            res = run_child(args, lib, {}, torch_arm=yard)
            label = lib or "default"
            runs.append((label, rnd, res["us"]["lib"]))
            if yard:
                runs.append(("torch copy_", rnd, res["us"]["torch"]))
                runs.append(("B200COLL_BULK=0", rnd, run_child(args, lib, {"B200COLL_BULK": "0"}, torch_arm=False)["us"]["lib"]))
            print(f"# round {rnd} {label}: {res['version']} ({res['lib']}), {res['launches']} launches", flush=True)
    labels = list(dict.fromkeys(r[0] for r in runs))
    size_list = sizes(args.min, args.max)
    print("\n# us per call: min-max over rounds")
    for i, lb in enumerate(labels):
        print(f"# [{i}] {lb}")
    print(f"{'bytes':>12} " + " ".join(f"{'[' + str(i) + ']':>20}" for i in range(len(labels))))
    for b in size_list:
        cells = []
        for lb in labels:
            ts = [r[2][b] for r in runs if r[0] == lb]
            cells.append(f"{min(ts):.2f}-{max(ts):.2f}")
        print(f"{b:>12} " + " ".join(f"{c:>20}" for c in cells))
    print(f"\n# fit t = F + bytes/BW over sizes >= {args.fit_min} bytes, one fit per run")
    fits = {}
    for lb in labels:
        fs = [fit(r[2], args.fit_min) for r in runs if r[0] == lb]
        fits[lb] = fs
        print(f"{lb}: F = " + ", ".join(f"{f:.2f}" for f, _ in fs) + " us; BW = " + ", ".join(f"{bw / 1e3:.3f}" for _, bw in fs) + " TB/s copied (twice that in HBM read + write)")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"card": gpu, "runs": [{"label": lb, "round": rnd, "us": {str(b): t for b, t in rows.items()}} for lb, rnd, rows in runs],
                       "fits": {lb: [{"F_us": f_, "BW_GBs": bw} for f_, bw in fs] for lb, fs in fits.items()}}, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
