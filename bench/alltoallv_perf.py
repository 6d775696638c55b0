#!/usr/bin/env python
"""alltoallv_perf — expert-dispatch shaped all-to-all (BASELINE config 4), libb200coll vs NCCL on the same box.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29500 bench/alltoallv_perf.py

For each (tokens per rank, hidden, skew): device-timed dispatch of bf16 token rows to the ranks that own their experts, with
(a) libb200coll all_to_all_v, bf16 on the wire; (b) the same with the fp8-e4m3 quantise fused into the dispatch kernel (half the
bytes on NVLink, no separate cast kernel); (c) NCCL all_to_all_single with split sizes (torch.distributed, the way MoE stacks call it);
(d) all_to_all_v_quantized, the block-scaled dispatch FP8 recipes use: e4m3 rows with one fp32 scale per 1x128 block, one kernel.
Then the combine back, with the dispatched rows standing in for the expert outputs: (e) all_to_all_v_combine, each rank pulling its
tokens' top-k rows and summing them with the gate weights in one kernel, against (f) NCCL all_to_all_single back plus the PyTorch
gather and weighted sum a MoE stack runs; combine_matches says ours equals an explicit slot-order fp32 sum bit for bit.
Then the same routing from the router's device-side expert ids: (g) expert_dispatch, layout, count exchange and push with no host sync,
and (h) expert_combine over its route, against (i) what a caller writes today to reach all_to_all_v from device ids: a device bincount,
a .cpu(), an all-gather of the counts, the offsets on the host, an argsort permute of the rows, then all_to_all_v. routed_matches says
nothing was dropped, the counts add up to the plan's rows, and the routed combine equals the slot-order fp32 sum bit for bit.
Then (j) expert_dispatch_quantized, the same routing with e4m3 rows and 1x128 block scales on the wire, into recv8 / recv_scales;
routed_fp8_matches says its counts, route and dropped equal the bf16 routed dispatch's and every stored row, dequantised, lies within
amax * 2^-4 of its source token's row (amax of the element's block: half an e4m3 ulp at the block's largest value).
Then the quantising combines, e4m3 with 1x128 block scales on the wire: (k) all_to_all_v_combine_quantized over (e)'s expert outputs and
(l) expert_combine_quantized over (h)'s; q_combine_matches says both equal, bit for bit, the slot-order fp32 sum of the rows quantised
and dequantised (amax, two fp32 divisions, e4m3 cast, one multiply). At one rank nothing crosses NVLink, so their time over the wide
combines' is the HBM cost of the quantise pass.
Bus bandwidth = (bytes a rank sends off-chip, max over ranks) / time. Rank 0 prints one JSON line per shape."""
from __future__ import annotations

import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main() -> int:
    import torch
    import torch.distributed as dist
    from container_engine_accelerators_b200.models.workloads import expert_dispatch_plan
    from container_engine_accelerators_b200.ops import coll
    rank, world, lr = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(lr)
    dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
    iters, warm = int(os.environ.get("ITERS", 20)), 5
    shapes = [(4096, 4096, 0.0), (4096, 7168, 1.0), (16384, 7168, 1.0), (65536, 7168, 1.2)]
    cap_rows = max(expert_dispatch_plan(world, t, h, skew=s).max_rows for t, h, s in shapes)
    cap_hidden = max(h for _, h, _ in shapes)
    # send, recv, recv8 and recv_scales, plus the quantising combines' scratch (1.03 bytes per expert_out element, every size's kept)
    comm = coll.Comm.from_env(arena_mb=int(cap_rows * cap_hidden * 2 * 3.4 / (1 << 20)) + 256, tag="a2av")
    send = comm.empty(cap_rows * cap_hidden, torch.bfloat16)
    recv = comm.empty(cap_rows * cap_hidden, torch.bfloat16)
    recv8 = comm.empty(cap_rows * cap_hidden, torch.float8_e4m3fn)
    recv_scales = comm.empty(cap_rows * cap_hidden // 128, torch.float32)
    send.copy_((torch.arange(send.numel(), device="cuda") % 251).to(torch.bfloat16) * 0.01)
    nccl_recv = torch.empty(cap_rows * cap_hidden, dtype=torch.bfloat16, device="cuda")
    nccl_back = torch.empty(cap_rows * cap_hidden, dtype=torch.bfloat16, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn) -> float:
        for _ in range(warm):
            fn()
        torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
        e0.record()
        for _ in range(iters):
            fn()
        e1.record(); torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1) / iters], device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return t.item() * 1e3

    def roundtrip(rows):
        """bf16 rows quantised to e4m3 in 128-element blocks and dequantised, in fp32: amax, two divisions, the cast, one multiply."""
        v = rows.float().view(rows.shape[0], -1, 128)
        amax = v.abs().amax(dim=-1, keepdim=True)
        fmax = torch.full_like(amax, 448.0)                                  # tensor operands: true divisions, not products with 1 / 448
        inv, s = fmax / amax, amax / fmax
        one = (amax == 0) | torch.isinf(inv)
        inv, s = torch.where(one, torch.ones_like(inv), inv), torch.where(one, torch.ones_like(s), s)
        q = (v * inv).clamp(-448.0, 448.0).to(torch.float8_e4m3fn)
        return (q.float() * s).view(rows.shape[0], -1)
    for tokens, hidden, skew in shapes:
        plan = expert_dispatch_plan(world, tokens, hidden, skew=skew, seed=1)
        rows, so, ro = plan.rows[rank].tolist(), plan.send_off[rank].tolist(), [int(plan.recv_off[d, rank]) for d in range(world)]
        n_send = int(plan.rows[rank].sum()) * hidden
        n_recv = int(plan.rows[:, rank].sum()) * hidden
        us_ours = timed(lambda: comm.all_to_all_v(send, recv, hidden, rows, so, ro))
        comm.check_async_error()
        # correctness of the bf16 path against NCCL's result
        in_split = [r * hidden for r in rows]
        out_split = [int(plan.rows[s, rank]) * hidden for s in range(world)]
        dist.all_to_all_single(nccl_recv[:n_recv], send[:n_send], out_split, in_split)
        torch.cuda.synchronize()
        ok = bool(torch.equal(recv[:n_recv], nccl_recv[:n_recv]))
        us_fp8 = timed(lambda: comm.all_to_all_v(send, recv8, hidden, rows, so, ro, scale=1.0))
        q_rows = plan.max_rows                                   # the same on every rank, as the symmetric recv needs
        us_bsq = timed(lambda: comm.all_to_all_v_quantized(send, recv8[:q_rows * hidden], recv_scales[:q_rows * hidden // 128], hidden, rows, so, ro, block=128))
        us_nccl = timed(lambda: dist.all_to_all_single(nccl_recv[:n_recv], send[:n_send], out_split, in_split))
        # combine: recv holds the bf16 dispatch result (the expert outputs' stand-in), so dispatch row i's expert row is send row i
        comm.all_to_all_v(send, recv, hidden, rows, so, ro)
        idx = torch.from_numpy(plan.index[rank]).cuda()
        gate = torch.from_numpy(plan.weights[rank]).cuda()
        out = torch.empty(tokens, hidden, dtype=torch.bfloat16, device="cuda")
        eo = recv[:q_rows * hidden]
        us_comb = timed(lambda: comm.all_to_all_v_combine(eo, out, hidden, rows, so, ro, idx, gate))
        comm.check_async_error()
        y = send[:n_send].view(-1, hidden)
        acc = torch.zeros(tokens, hidden, device="cuda")
        for j in range(idx.shape[1]):
            acc = acc + gate[:, j:j + 1] * y[idx[:, j].long()].float()
        comb_ok = bool(torch.equal(out.view(torch.int16), acc.to(torch.bfloat16).view(torch.int16)))
        qout = torch.empty(tokens, hidden, dtype=torch.bfloat16, device="cuda")
        us_q_comb = timed(lambda: comm.all_to_all_v_combine_quantized(eo, qout, hidden, rows, so, ro, idx, gate, block=128))
        comm.check_async_error()
        yq = roundtrip(y)
        acc = torch.zeros(tokens, hidden, device="cuda")
        for j in range(idx.shape[1]):
            acc = acc + gate[:, j:j + 1] * yq[idx[:, j].long()]
        q_comb_ok = bool(torch.equal(qout.view(torch.int16), acc.to(torch.bfloat16).view(torch.int16)))
        idx_l = idx.long()

        def nccl_combine():
            dist.all_to_all_single(nccl_back[:n_send], nccl_recv[:n_recv], in_split, out_split)
            return (nccl_back[:n_send].view(-1, hidden)[idx_l].float() * gate.unsqueeze(-1)).sum(dim=1).to(torch.bfloat16)
        us_nccl_comb = timed(nccl_combine)
        # device-routed dispatch and combine from the plan's expert ids (4 experts per rank), into the same symmetric recv
        n_exp, x = world * 4, send[:tokens * hidden].view(tokens, hidden)
        topk = torch.from_numpy(plan.experts[rank]).cuda()
        rrecv = recv[:q_rows * hidden]
        _, counts, route, dropped = comm.expert_dispatch(x, topk, n_exp, rrecv)
        us_routed = timed(lambda: comm.expert_dispatch(x, topk, n_exp, rrecv, counts, route, dropped))
        us_routed_comb = timed(lambda: comm.expert_combine(rrecv.view(-1, hidden), route, gate, out))
        comm.check_async_error()
        us_routed_q_comb = timed(lambda: comm.expert_combine_quantized(rrecv.view(-1, hidden), route, gate, qout, block=128))
        comm.check_async_error()
        xq = roundtrip(x)
        acc = torch.zeros(tokens, hidden, device="cuda")
        for j in range(topk.shape[1]):
            acc = acc + gate[:, j:j + 1] * xq
        q_comb_ok = q_comb_ok and bool(torch.equal(qout.view(torch.int16), acc.to(torch.bfloat16).view(torch.int16)))
        # the same routing with FP8 on the wire; x is the same on every rank (send is filled the same way everywhere), so a stored row
        # only needs its source token, which the gathered routes give
        q8, s8 = recv8[:q_rows * hidden], recv_scales[:q_rows * hidden // 128]
        c8, r8, d8 = torch.empty_like(counts), torch.empty_like(route), torch.empty_like(dropped)
        us_routed_fp8 = timed(lambda: comm.expert_dispatch_quantized(x, topk, n_exp, q8, s8, 128, c8, r8, d8))
        comm.check_async_error()
        routes = torch.empty(world, *route.shape, dtype=route.dtype, device="cuda")
        dist.all_gather_into_tensor(routes, r8)
        mine = (routes >= rank * q_rows) & (routes < (rank + 1) * q_rows)
        rows_at = (routes[mine] - rank * q_rows).long()
        src_tok = torch.nonzero(mine)[:, 1]                                # slot (s, t, j) -> token t
        deq = q8.view(q_rows, -1, 128).float() * s8.view(q_rows, -1, 1)
        ref = x[src_tok].float().view(len(src_tok), -1, 128)
        amax = ref.abs().amax(dim=-1, keepdim=True)
        # e4m3 keeps 3 mantissa bits: half an ulp is at most 2^-4 of the value; the slack covers the fp32 roundings of x * inv and q * s
        fp8_ok = (torch.equal(c8, counts) and torch.equal(r8, route) and torch.equal(d8, dropped)
                  and bool(((deq[rows_at] - ref).abs() <= amax * (2.0 ** -4 + 2.0 ** -20)).all()))
        # recv holds every rank's rows (plan.max_rows >= any rank's load): nothing dropped, this rank's counts add up to the rows the
        # plan sends it, every slot routed, and the combine of the returned rows is the slot-order sum of each token's own row
        xr = x.float()
        acc = torch.zeros(tokens, hidden, device="cuda")
        for j in range(topk.shape[1]):
            acc = acc + gate[:, j:j + 1] * xr
        routed_ok = (int(dropped.item()) == 0 and int(counts.sum().item()) == int(plan.rows[:, rank].sum()) and bool((route >= 0).all())
                     and bool(torch.equal(out.view(torch.int16), acc.to(torch.bfloat16).view(torch.int16))))
        all_counts = torch.empty(world * world, dtype=torch.int64, device="cuda")

        def host_plan():
            dest = (topk // 4).view(-1).long()
            mine = torch.bincount(dest, minlength=world)
            dist.all_gather_into_tensor(all_counts, mine)
            m = all_counts.cpu().view(world, world).tolist()             # m[s][d]: rows s sends to d
            h_rows = m[rank]
            h_so = [sum(h_rows[:d]) for d in range(world)]
            h_ro = [sum(m[s][d] for s in range(rank)) for d in range(world)]
            order = torch.argsort(dest, stable=True)
            permuted = x[order // topk.shape[1]]
            comm.all_to_all_v(permuted, recv, hidden, h_rows, h_so, h_ro)
        us_host_plan = timed(host_plan)
        offchip = max(int(plan.rows[s].sum() - plan.rows[s, s]) for s in range(world)) * hidden * 2
        oks = torch.tensor([1.0 if ok else 0.0, 1.0 if comb_ok else 0.0, 1.0 if routed_ok else 0.0, 1.0 if fp8_ok else 0.0, 1.0 if q_comb_ok else 0.0],
                           device="cuda")
        dist.all_reduce(oks, op=dist.ReduceOp.MIN)
        if rank == 0:
            print(json.dumps({"bench": "alltoallv_perf", "n_gpus": world, "tokens_per_rank": tokens, "hidden": hidden, "skew": skew, "top_k": 2,
                              "max_offchip_bytes_per_rank": offchip, "imbalance_max_over_mean": round(float(plan.rows.sum(axis=0).max() / plan.rows.sum(axis=0).mean()), 3),
                              "ours_us": round(us_ours, 2), "ours_busbw": round(offchip / us_ours / 1e3, 2), "ours_fused_fp8_us": round(us_fp8, 2),
                              "nccl_us": round(us_nccl, 2), "nccl_busbw": round(offchip / us_nccl / 1e3, 2), "speedup": round(us_nccl / us_ours, 2),
                              "fp8_speedup_vs_nccl_bf16": round(us_nccl / us_fp8, 2), "matches_nccl": bool(oks[0].item() == 1.0),
                              "ours_block_fp8_us": round(us_bsq, 2), "ours_combine_us": round(us_comb, 2), "nccl_combine_us": round(us_nccl_comb, 2),
                              "combine_matches": bool(oks[1].item() == 1.0), "ours_routed_us": round(us_routed, 2),
                              "ours_routed_combine_us": round(us_routed_comb, 2), "host_plan_us": round(us_host_plan, 2),
                              "routed_matches": bool(oks[2].item() == 1.0), "ours_routed_fp8_us": round(us_routed_fp8, 2),
                              "routed_fp8_matches": bool(oks[3].item() == 1.0), "ours_q_combine_us": round(us_q_comb, 2),
                              "ours_routed_q_combine_us": round(us_routed_q_comb, 2), "q_combine_matches": bool(oks[4].item() == 1.0)}), flush=True)
    comm.destroy()
    dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
