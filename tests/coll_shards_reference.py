"""Reference for the FSDP shard all-gather and reduce-scatter (b200collAllGatherShards / ReduceScatterShards): the gather built from
byte views (a bit copy) or Tensor.to (the fp32 -> bf16 / fp16 cast); the reduce-scatter in fp32 in rank order, then the scale, then the
old shard, each a separate fp32 op, rounded once. Tensor i's full is [d, ...]; rank s's shard holds its n_s rows first. The functions
run on the device their inputs are on; the *_loop renderings take one element at a time in numpy fp32."""
import numpy as np
import torch

from tests import coll_fp_reference as R


def default_rows(d, n):
    """FSDP2's rows per rank: ceil(d / N)."""
    return -(-d // n)


def shard_range(d, p, r):
    """The header's rows of rank r: [first, first + n_r), first = r * p, n_r = clamp(d - r * p, 0, p)."""
    first = min(d, r * p)
    return first, max(0, min(d - first, p))


def split(full, n, p=None):
    """The N shards of an unsharded tensor: rank r's n_r rows (a copy), padded with nothing."""
    d = full.shape[0]
    p = default_rows(d, n) if p is None else p
    return [full[f:f + k].clone() for f, k in (shard_range(d, p, r) for r in range(n))]


def all_gather(shards, d, full_dtype, p=None):
    """shards[s]: rank s's shard ([>= n_s, ...]). Returns the [d, ...] full tensor every rank holds: rank s's rows cast to full_dtype
    (a bit copy when the dtypes agree)."""
    n = len(shards)
    p = default_rows(d, n) if p is None else p
    out = torch.empty((d, *shards[0].shape[1:]), dtype=full_dtype, device=shards[0].device)
    for s, x in enumerate(shards):
        f, k = shard_range(d, p, s)
        if k:
            src = x[:k]
            out[f:f + k] = src.view(full_dtype) if src.dtype == full_dtype else src.to(full_dtype)
    return out


def reduce_scatter(fulls, shard_dtype, scale=1.0, olds=None, p=None):
    """fulls[s]: rank s's [d, ...] gradient. Returns shards[r]: rank r's [n_r, ...] rows of round_once((sum over s in rank order of
    fulls[s], from +0) * scale [+ old]) in shard_dtype; olds[r] (or None) is rank r's shard before the call. One rank, one dtype,
    scale 1 and no olds: a bit copy."""
    n = len(fulls)
    d = fulls[0].shape[0]
    p = default_rows(d, n) if p is None else p
    s32 = R.f32(scale).to(fulls[0].device)
    out = []
    for r in range(n):
        f, k = shard_range(d, p, r)
        rows = [x[f:f + k] for x in fulls]
        if n == 1 and shard_dtype == fulls[0].dtype and scale == 1.0 and olds is None:
            out.append(rows[0].clone())
            continue
        t = R.ref_sum([x.reshape(-1) for x in rows], list(range(n))) * s32
        if olds is not None:
            t = olds[r][:k].reshape(-1).float() + t
        out.append(R.cast(t, shard_dtype).view(k, *fulls[0].shape[1:]))
    return out


def all_gather_loop(shards, d, full_dtype, p=None):
    """all_gather by the header's formula, one row at a time: full[s * p + j] = cast(shard_s[j]) for j < n_s."""
    n = len(shards)
    p = default_rows(d, n) if p is None else p
    out = torch.zeros((d, *shards[0].shape[1:]), dtype=full_dtype)
    for s in range(n):
        for j in range(shard_range(d, p, s)[1]):
            row = shards[s][j]
            out[s * p + j] = row.view(full_dtype) if row.dtype == full_dtype else row.to(full_dtype)
    return out


def reduce_scatter_loop(fulls, shard_dtype, scale=1.0, olds=None, p=None):
    """reduce_scatter by the header's formula, one element at a time in numpy fp32: t = ((+0 + full_0[e]) + ...) ; t = t * scale;
    t = old + t; round once."""
    n = len(fulls)
    d = fulls[0].shape[0]
    p = default_rows(d, n) if p is None else p
    fs = [x.float().reshape(d, -1).numpy() for x in fulls]
    W = fs[0].shape[1]
    sc = np.float32(scale)
    out = []
    for r in range(n):
        f, k = shard_range(d, p, r)
        if n == 1 and shard_dtype == fulls[0].dtype and scale == 1.0 and olds is None:
            out.append(fulls[0][f:f + k].clone())
            continue
        old = None if olds is None else olds[r].float().reshape(-1, W).numpy()
        acc = np.zeros((k, W), dtype=np.float32)
        with np.errstate(invalid="ignore", over="ignore"):          # inf - inf and overflow are part of the data
            for j in range(k):
                for e in range(W):
                    t = np.float32(0.0)
                    for s in range(n):
                        t = np.float32(t + fs[s][f + j, e])
                    t = np.float32(t * sc)
                    if old is not None:
                        t = np.float32(old[j, e] + t)
                    acc[j, e] = t
        out.append(R.cast(torch.from_numpy(acc), shard_dtype).view(k, *fulls[0].shape[1:]))
    return out
