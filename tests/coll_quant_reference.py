"""Reference for the quantising collectives of libb200coll (b200collAllGatherQuantized, ...ReduceScatterQuantized, ...AllReduceQuantized),
and seeded inputs whose blocks span many binades.

Per block of `block` consecutive elements of one rank's input x (bf16, fp16 or fp32, widened exactly to fp32), FMAX = 448 (e4m3) or
57344 (e5m2):
    amax = max |x|                 the largest bit pattern of |x|, so a NaN anywhere makes amax NaN
    inv = FMAX / amax, s = amax / FMAX     fp32 divisions rounded to nearest; inv = s = 1 when amax == 0 or inv is +inf
    q = cast(x * inv, wire)        the product rounded to fp32, then RNE to FP8 with saturation (coll_fp_reference.cast)
    v = float(q) * s               one fp32 multiply
All-reduce and reduce-scatter give cast(((0 + v_0) + v_1 + ...) * scale, out) in rank order; all-gather shard r is cast((0 + v_r) * scale).

Not collected by pytest (no test_ prefix); imported by the test_coll_quantized_* files."""
import numpy as np
import torch

from tests.coll_fp_reference import FP8_MAX, cast

BLOCKS = (16, 32, 64, 128, 256, 512)


def quantize(x, block, wire):
    """(q, s, v) for a 1-D CPU tensor x: q the FP8 tensor, s the fp32 scale of every block, v the dequantised fp32 values."""
    x32 = x.reshape(-1, block).float().numpy()
    amax = (x32.view(np.uint32) & np.uint32(0x7FFFFFFF)).max(axis=1).view(np.float32)
    fmax = np.float32(FP8_MAX[wire])
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        inv = fmax / amax
        s = amax / fmax
    one = (amax == 0) | (inv == np.float32(np.inf))
    inv = np.where(one, np.float32(1), inv).astype(np.float32)
    s = np.where(one, np.float32(1), s).astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        y = (x32 * inv[:, None]).astype(np.float32)
    q = cast(torch.from_numpy(y.reshape(-1).copy()), wire)
    with np.errstate(invalid="ignore", over="ignore"):
        v = (q.float().numpy().reshape(-1, block) * s[:, None]).astype(np.float32)
    return q, torch.from_numpy(s.copy()), torch.from_numpy(v.reshape(-1).copy())


def reduce(vs, scale, out_dt):
    """cast(((0 + v_0) + v_1 + ...) * scale, out_dt), the sum in fp32 in the order given."""
    acc = np.zeros(vs[0].numel(), dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for v in vs:
            acc = (acc + v.numpy()).astype(np.float32)
        acc = (acc * np.float32(scale)).astype(np.float32)
    return cast(torch.from_numpy(acc), out_dt)


def all_reduce(xs, block, wire, scale, out_dt):
    return reduce([quantize(x, block, wire)[2] for x in xs], scale, out_dt)


def all_gather(xs, block, wire, scale, out_dt):
    return torch.cat([reduce([quantize(x, block, wire)[2]], scale, out_dt) for x in xs])


def reduce_scatter(xs, block, wire, scale, out_dt, rank):
    m = xs[0].numel() // len(xs)
    return all_reduce([x[rank * m:(rank + 1) * m] for x in xs], block, wire, scale, out_dt)


def gen(count, in_dt, block, seed, specials=True):
    """count elements of in_dt: every block gets its own binade (fp32 2^-60 .. 2^60, bf16 2^-40 .. 2^40, fp16 2^-12 .. 2^12) and random
    signs and mantissas, so products round and ties occur. With specials the first blocks are, in this order: all zeros; -0 and +0
    mixed with small values; one +inf; one NaN; -inf; and (bf16 and fp32) a tiny block whose amax is below FMAX / FLT_MAX."""
    g = torch.Generator().manual_seed(seed)
    nblk = count // block
    span = {torch.float32: 60, torch.bfloat16: 40, torch.float16: 12}[in_dt]
    e = torch.randint(-span, span + 1, (nblk, 1), generator=g).float()
    m = torch.rand(nblk, block, generator=g) * 2 - 1
    x = (m * torch.exp2(e)).reshape(-1)
    # mantissas coarse enough to tie in FP8 after scaling: an eighth of the blocks hold small integers only
    ints = torch.randint(-16, 17, (nblk, block), generator=g).float().reshape(-1)
    coarse = (torch.arange(nblk) % 8 == 5).repeat_interleave(block)
    x = torch.where(coarse, ints, x).to(in_dt)
    if specials and nblk >= 6:
        x[0:block] = 0
        x[block:2 * block:3] = -0.0
        x[2 * block + 1] = float("inf")
        x[3 * block + 2] = float("nan")
        x[4 * block + 3] = float("-inf")
        if in_dt != torch.float16:
            x[5 * block:6 * block] = (torch.rand(block, generator=g) * 2 - 1).mul(1e-37).to(in_dt)
    return x
