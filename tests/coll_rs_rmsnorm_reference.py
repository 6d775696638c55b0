"""Order-exact reference of b200collReduceScatterRmsNorm and b200collReduceScatterRmsNormQuantized (coll/include/b200coll.h): the
header's equivalence, rendered directly. The N ranks' residual shards are stacked into the full residual stream, the all-reduce form's
reference (coll_rmsnorm_reference.rms_norm, coll_rmsnorm_quant_reference.rms_norm_quantized) runs on it, and its results are cut back
into slices: rank r's new shard and out rows are rows [r*S, (r+1)*S), or every row of out when gathering.

Not collected by pytest (no test_ prefix)."""
import torch

from tests import coll_rmsnorm_quant_reference as RQ
from tests import coll_rmsnorm_reference as R


def shards(t, n):
    """t cut along dim 0 into n equal slices (copies)."""
    s = t.shape[0] // n
    return [t[r * s:(r + 1) * s].clone() for r in range(n)]


def rs_rms_norm(xs, res_shards, gamma, eps, dt, gather):
    """xs: the N ranks' [rows, row_len] tensors; res_shards: the N ranks' [rows / N, row_len] residual shards; gamma [row_len]; all of
    dt (CPU). Returns [(new shard, out)] per rank: out is the rank's [S, row_len] slice, or all [rows, row_len] when gathering."""
    n = len(xs)
    h, out = R.rms_norm(xs, torch.cat(res_shards), gamma, eps, dt)
    return [(hs, out if gather else os_) for hs, os_ in zip(shards(h, n), shards(out, n))]


def rs_rms_norm_quantized(xs, res_shards, gamma, eps, dt, block, wire, gather):
    """As rs_rms_norm, with (new shard, q, scales) per rank: q and scales the rank's slice, or all rows when gathering."""
    n = len(xs)
    h, q, s = RQ.rms_norm_quantized(xs, torch.cat(res_shards), gamma, eps, dt, block, wire)
    return [(hs, q if gather else qs, s if gather else ss) for hs, qs, ss in zip(shards(h, n), shards(q, n), shards(s, n))]
