"""Synthetic workload shapes for the collective benchmarks (BASELINE config 4: "alltoall_perf 8xH100, expert-dispatch shape").

expert_dispatch_plan(): tokens routed top-k to experts that are sharded across ranks (expert parallelism). Returns, per
source rank, how many token rows go to each destination rank plus the row offsets both sides need — exactly the arguments of
Comm.all_to_all_v(). Routing is drawn from a Zipf-like popularity so some experts are hot (the load-imbalance case SURVEY
§7.3-7 warns about)."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np


@dataclass
class DispatchPlan:
    nranks: int
    hidden: int
    rows: np.ndarray            # rows[s, d]: token rows rank s sends to rank d
    send_off: np.ndarray        # send_off[s, d]: first row of that block in s's send buffer
    recv_off: np.ndarray        # recv_off[d, s]: first row of s's block in d's recv buffer
    max_rows: int               # buffer capacity (rows) that fits every rank's send and recv side
    # index[s]: [tokens, top_k] int32, the row of rank s's send buffer each (token, slot) is dispatched as (within a destination's
    # range, rows in row-major (token, slot) order); weights[s]: [tokens, top_k] float32 gate weights summing to 1 per token. Together
    # with rows / send_off / recv_off they are the arguments of Comm.all_to_all_v_combine().
    index: list = field(default_factory=list)
    weights: list = field(default_factory=list)
    # experts[s]: [tokens, top_k] int32, the expert each (token, slot) of rank s is routed to (experts [d * experts_per_rank, + experts_per_rank)
    # live on rank d): the topk_idx argument of Comm.expert_dispatch(), from the same draw as rows and index.
    experts: list = field(default_factory=list)

    def bytes_sent(self, rank: int, itemsize: int = 2) -> int:
        return int(self.rows[rank].sum()) * self.hidden * itemsize


def expert_dispatch_plan(nranks: int, tokens_per_rank: int, hidden: int, experts_per_rank: int = 4, top_k: int = 2, skew: float = 1.0, seed: int = 0) -> DispatchPlan:
    rng = np.random.default_rng(seed)
    n_experts = nranks * experts_per_rank
    pop = 1.0 / np.arange(1, n_experts + 1) ** skew if skew > 0 else np.ones(n_experts)
    pop = rng.permutation(pop / pop.sum())
    rows = np.zeros((nranks, nranks), dtype=np.int64)
    dests, experts = [], []
    for s in range(nranks):
        choice = rng.choice(n_experts, size=(tokens_per_rank, top_k), p=pop)
        experts.append(choice.astype(np.int32))
        dest = choice // experts_per_rank
        dests.append(dest)
        rows[s] = np.bincount(dest.ravel(), minlength=nranks)
    send_off = np.zeros_like(rows)
    send_off[:, 1:] = np.cumsum(rows, axis=1)[:, :-1]
    index = []
    for s, dest in enumerate(dests):
        flat = dest.ravel()
        order = np.argsort(flat, kind="stable")                  # row-major (token, slot) order within each destination
        idx = np.empty(flat.size, dtype=np.int64)
        idx[order] = np.arange(flat.size)                        # rank among all slots sorted by destination = row in s's send buffer
        index.append(idx.reshape(tokens_per_rank, top_k).astype(np.int32))
    wrng = np.random.default_rng([seed, 0x6A7E])                 # its own generator: the routing above stays what it was
    weights = []
    for s in range(nranks):
        w = wrng.random((tokens_per_rank, top_k)) + 0.05
        weights.append((w / w.sum(axis=1, keepdims=True)).astype(np.float32))
    recv_off = np.zeros_like(rows)                       # recv_off[d, s]
    recv_off[:, 1:] = np.cumsum(rows.T, axis=1)[:, :-1]
    max_rows = int(max(rows.sum(axis=1).max(), rows.sum(axis=0).max()))
    return DispatchPlan(nranks, hidden, rows, send_off, recv_off, max_rows, index, weights, experts)


def uniform_plan(nranks: int, rows_per_peer: int, hidden: int) -> DispatchPlan:
    rows = np.full((nranks, nranks), rows_per_peer, dtype=np.int64)
    off = np.tile(np.arange(nranks) * rows_per_peer, (nranks, 1))
    return DispatchPlan(nranks, hidden, rows, off.copy(), off.copy(), rows_per_peer * nranks)
