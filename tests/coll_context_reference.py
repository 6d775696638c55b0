"""Reference for the context-parallel all-gather and reduce-scatter (b200collAllGatherContext / ReduceScatterContext): the gather built
from stacking and index_select on byte views, so every dtype (FP8 included) moves bit for bit; the reduce-scatter from
coll_fp_reference.ref_sum in rank order plus cast. One tensor at a time; a rank's shard is [B, S_l, ...] and a full tensor
[B, N * S_l, ...]. all_gather and reduce_scatter run on the device their inputs are on."""
import numpy as np
import torch

from tests import coll_fp_reference as R


def gtok(n, chunks, S_l, r, t):
    """The header's global token of rank r's local token t: G(r, k) * c + u, c = S_l / chunks, k = t // c, u = t % c, G(r, 0) = r and
    G(r, 1) = 2N - 1 - r."""
    c = S_l // chunks
    k, u = divmod(t, c)
    return (r if k == 0 else 2 * n - 1 - r) * c + u


def token_index(n, chunks, S_l, device="cpu"):
    """idx[g] = s * S_l + t for the (rank s, local token t) that holds global token g: the gather's index over the stacked shards."""
    c = S_l // chunks
    idx = torch.empty(n * S_l, dtype=torch.int64, device=device)
    for s in range(n):
        for k in range(chunks):
            g0 = (s if k == 0 else 2 * n - 1 - s) * c
            idx[g0:g0 + c] = s * S_l + k * c + torch.arange(c, device=device)
    return idx


def local_index(n, chunks, S_l, r, device="cpu"):
    """g[t] = gtok(r, t) for every local token t of rank r: the reduce-scatter's index into the full tensors."""
    c = S_l // chunks
    t = torch.arange(S_l, device=device)
    return torch.where(t < c, r * c + t, (2 * n - 1 - r) * c + t - c)


def _bytes(t):
    """t as a contiguous [B, S_l, row bytes] uint8 tensor."""
    t = t.contiguous()
    return t.view(torch.uint8).reshape(t.shape[0], t.shape[1], -1)


def all_gather(shards, chunks):
    """shards[s]: rank s's [B, S_l, ...] shard. Returns the full [B, N * S_l, row bytes] uint8 tensor every rank holds."""
    n = len(shards)
    x = torch.stack([_bytes(t) for t in shards], dim=1)                     # [B, N(s), S_l, Wb]
    B, _, S_l, Wb = x.shape
    return x.reshape(B, n * S_l, Wb).index_select(1, token_index(n, chunks, S_l, x.device))


def reduce_scatter(fulls, chunks):
    """fulls[s]: rank s's [B, N * S_l, ...] full tensor (bf16, fp16 or fp32). Returns shards[r]: rank r's [B, S_l, ...] sum over the ranks
    in rank order, in fp32, rounded once to the dtype. One rank: a bit copy."""
    n = len(fulls)
    B, S = fulls[0].shape[:2]
    S_l = S // n
    if n == 1:
        return [fulls[0].clone()]
    out = []
    for r in range(n):
        g = local_index(n, chunks, S_l, r, fulls[0].device)
        xs = [f.index_select(1, g).reshape(-1) for f in fulls]
        out.append(R.cast(R.ref_sum(xs, list(range(n))), fulls[0].dtype).view(B, S_l, *fulls[0].shape[2:]))
    return out


def all_gather_loop(shards, chunks):
    """all_gather by the header's formula, one (rank s, b, t) at a time: full[b, gtok(s, t)] = shard_s[b, t]."""
    n = len(shards)
    xb = [_bytes(t) for t in shards]
    B, S_l, Wb = xb[0].shape
    full = torch.zeros(B, n * S_l, Wb, dtype=torch.uint8)
    for s in range(n):
        for b in range(B):
            for t in range(S_l):
                full[b, gtok(n, chunks, S_l, s, t)] = xb[s][b, t]
    return full


def reduce_scatter_loop(fulls, chunks):
    """reduce_scatter by the header's formula, one element at a time in numpy fp32: shard_r[b, t, e] = round_once(((+0 + full_0[b, g, e])
    + full_1[b, g, e]) + ...), g = gtok(r, t)."""
    n = len(fulls)
    B, S = fulls[0].shape[:2]
    S_l = S // n
    if n == 1:
        return [fulls[0].clone()]
    fs = [f.float().reshape(B, S, -1).numpy() for f in fulls]
    out = []
    for r in range(n):
        acc = np.zeros((B, S_l, fs[0].shape[2]), dtype=np.float32)
        for b in range(B):
            for t in range(S_l):
                g = gtok(n, chunks, S_l, r, t)
                for e in range(acc.shape[2]):
                    a = np.float32(0.0)
                    with np.errstate(invalid="ignore", over="ignore"):      # inf - inf and overflow are part of the data
                        for s in range(n):
                            a = np.float32(a + fs[s][b, g, e])
                    acc[b, t, e] = a
        out.append(R.cast(torch.from_numpy(acc), fulls[0].dtype).view(B, S_l, *fulls[0].shape[2:]))
    return out
