"""The vocab-parallel embedding (b200collVocabParallelEmbedding / ...Backward) in numpy, as coll/include/b200coll.h states it: the
forward a row gather from the stacked tables with +0 rows for out-of-range ids, the backward each owned row's token-order fp32 fold, one
np.float32 add at a time. Tables and gradients are handled as raw bits (uint16 for bf16 and fp16, uint32 for fp32)."""
import numpy as np

_BITS = {"bf16": np.uint16, "f16": np.uint16, "f32": np.uint32}


def widen(bits, dt):
    """Raw bits of dtype `dt` ("bf16", "f16", "f32") to float32, bit for bit (-0 and NaN payloads kept)."""
    bits = np.asarray(bits)
    if dt == "bf16":
        return (bits.astype(np.uint32) << 16).view(np.float32)
    if dt == "f16":
        return bits.view(np.float16).astype(np.float32)
    return bits.view(np.float32)


def narrow(x, dt):
    """float32 to the raw bits of `dt`, round to nearest even (fp16 overflows to inf; NaN stays NaN)."""
    x = np.asarray(x, dtype=np.float32)
    if dt == "f32":
        return x.view(np.uint32).copy()
    if dt == "f16":
        return x.astype(np.float16).view(np.uint16)
    u = x.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    nan = np.isnan(x)
    r[nan] = ((u[nan] >> 16) | 0x40).astype(np.uint16)
    return r


def forward(tables, ids, sequence_parallel=False, rank=0):
    """out bits of `rank`: tables[r] is rank r's [Vl, H] bits; ids [T] int64."""
    n = len(tables)
    vl, h = tables[0].shape
    ids = np.asarray(ids, dtype=np.int64)
    T = ids.shape[0]
    lo, hi = (rank * T // n, (rank + 1) * T // n) if sequence_parallel else (0, T)
    full = np.concatenate(tables, axis=0)
    out = np.zeros((hi - lo, h), dtype=tables[0].dtype)
    sel = ids[lo:hi]
    ok = (sel >= 0) & (sel < n * vl)
    out[ok] = full[sel[ok]]
    return out


def backward(ids, dout_bits, dout_dt, rank, n, vl, dweight_dt, old_bits=None):
    """dweight bits of `rank` ([Vl, H]): dout_bits is the whole [T, H] output gradient (every rank's shard stacked under sequence
    parallelism); old_bits the dweight to accumulate into, or None."""
    ids = np.asarray(ids, dtype=np.int64)
    h = dout_bits.shape[1]
    acc = widen(old_bits, dweight_dt).copy() if old_bits is not None else np.zeros((vl, h), dtype=np.float32)
    j = ids - rank * vl
    own = (j >= 0) & (j < vl)
    # ufunc.at applies acc[j[i]] = acc[j[i]] + x[i] one i at a time, in index order: one IEEE fp32 add per element, token order
    np.add.at(acc, j[own], widen(dout_bits, dout_dt)[own])
    return narrow(acc, dweight_dt)
