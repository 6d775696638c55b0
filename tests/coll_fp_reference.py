"""Order-exact fp32 reference for the fp32 / fp16 / bf16 collectives of libb200coll, and seeded data that can tell orders apart.

Every fused sum / avg path widens each input to fp32, accumulates from +0 in a fixed order, multiplies once by the fp32 scale (avg: the
fp32 product scale * (1/N)) and rounds once, to nearest even, to the output type (FP8 saturates, fp16 overflows to inf). The order is
a property of the kernel that ran, so the reference takes it as an argument:

    [r0, r1, ...]                 that rank order for every element (LL, LL2, one-shot, rooted reduce, the generic kernel)
    ("rotate", r)                 r, r+1, ..., r-1 (P2P reduce-scatter at receiving rank r)
    ("owner", N, E, count)        two-shot all-reduce: vector v belongs to slice o with nvec*o//N <= v < nvec*(o+1)//N and is summed
                                  o, o+1, ..., o-1; elements past the last whole vector are summed in rank order (ar_tail_rank0)
    ("staged", N, E, count, chunk)  the staged all-reduce: two-shot on each chunk of `chunk` elements, slices from the chunk's nvec

Not collected by pytest (no test_ prefix); imported by test_coll_fp_numerics_cpu.py and test_coll_fp_numerics_gpu.py."""
import torch

STAGE_HALF_BYTES = 32 << 20          # coll/src/layout.h kStageHalfBytes
LL_ONESHOT_MAX_BYTES = 512 << 10     # kLLOneShotMaxBytes: per source

FP8_MAX = {torch.float8_e4m3fn: 448.0, torch.float8_e5m2: 57344.0}
# significand bits (implicit bit included) and exponent of the smallest normal
MANT = {torch.float32: 24, torch.bfloat16: 8, torch.float16: 11, torch.float8_e4m3fn: 4, torch.float8_e5m2: 3}
EMIN = {torch.float32: -126, torch.bfloat16: -126, torch.float16: -14, torch.float8_e4m3fn: -6, torch.float8_e5m2: -14}
INT_VIEW = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def esize(dt):
    return torch.empty((), dtype=dt).element_size()


def vec_elems(dt):
    """Elements of one 16-byte vector (E)."""
    return 16 // esize(dt)


def f32(x):
    return torch.tensor(x, dtype=torch.float32)


def avg_scale(scale, n):
    """What the host multiplies by for avg: fp32(scale) * fp32(1 / N), both rounded in fp32."""
    return float(f32(scale) * (f32(1.0) / f32(float(n))))


def cast(x32, dt):
    """fp32 -> dt with RNE; FP8 saturates to the finite range (NaN stays NaN), which torch's own conversion does not do."""
    m = FP8_MAX.get(dt)
    if m is not None:
        x32 = x32.clamp(-m, m)
    return x32.to(dt)


def cast_rtz(x32, dt):
    """fp32 -> dt rounding toward zero: one step toward zero wherever RNE moved away from it (a wrong model for the tests)."""
    y = cast(x32, dt)
    if dt == torch.float32:
        return y
    nb = 8 * esize(dt)
    bits = y.view(INT_VIEW[esize(dt)])
    away = (y.float().abs() > x32.abs()) & ~torch.isnan(x32)
    sbit = (1 << 7) if nb == 8 else -(1 << (nb - 1))                        # the sign bit in the signed (or uint8) view
    stepped = ((bits & ((1 << (nb - 1)) - 1)) - 1) | (bits & sbit)            # sign-magnitude: one less magnitude is one ulp closer to 0
    return torch.where(away, stepped, bits).view(dt)


# ------------------------------------------------------------------------------------------------- index formulas
def slice_bounds(nvec, n, o):
    """k_ar_twoshot: vectors [nvec*o/N, nvec*(o+1)/N) are rank o's slice (size_t arithmetic)."""
    return nvec * o // n, nvec * (o + 1) // n


def owner_map(count, n, e, device="cpu"):
    """Per element: the rank whose order sums it on the two-shot all-reduce. Tail elements (ar_tail_rank0) are summed in rank order,
    which is rank 0's rotation, so they map to 0."""
    nvec = count // e
    own = torch.zeros(count, dtype=torch.int64, device=device)
    for o in range(n):
        lo, hi = slice_bounds(nvec, n, o)
        own[lo * e:hi * e] = o
    return own


def staged_chunk(in_size, out_size, nranks, op):
    """Elements per staging round of the staged (buffers outside the arena) path of `op`, as collectives.cu computes it."""
    h = STAGE_HALF_BYTES
    if op in ("all_reduce", "broadcast", "reduce"):
        return min(h // in_size, h // out_size) // 64 * 64
    if op == "reduce_scatter":
        return (h // in_size // nranks) // 64 * 64
    if op in ("all_gather", "all_to_all"):
        return (h // out_size // nranks) // 64 * 64
    raise ValueError(op)


def staged_owner_map(count, n, e, chunk, device="cpu"):
    parts = [owner_map(min(chunk, count - d), n, e, device) for d in range(0, count, chunk)]
    return torch.cat(parts)


def rotation(r, n):
    return [(r + j) % n for j in range(n)]


# ------------------------------------------------------------------------------------------------- reference ops
def _sum(xs, order):
    acc = torch.zeros(xs[0].numel(), dtype=torch.float32, device=xs[0].device)
    for r in order:
        acc = acc + xs[r].float()
    return acc


def ref_sum(xs, order):
    """The fp32 accumulator (before the scale) for an order model (see the module docstring)."""
    n = len(xs)
    if isinstance(order, tuple) and order[0] == "rotate":
        return _sum(xs, rotation(order[1], n))
    if isinstance(order, tuple) and order[0] in ("owner", "staged"):
        _, nn, e, count = order[:4]
        assert nn == n and count == xs[0].numel()
        own = owner_map(count, n, e, xs[0].device) if order[0] == "owner" else staged_owner_map(count, n, e, order[4], xs[0].device)
        acc = torch.empty(count, dtype=torch.float32, device=xs[0].device)
        for o in range(n):
            sel = own == o
            if bool(sel.any()):
                acc[sel] = _sum(xs, rotation(o, n))[sel]
        return acc
    return _sum(xs, list(order))


def ref_reduce(xs, order, s, out_dtype):
    """round_once(sum_in_order(xs) * fp32(s)) in out_dtype."""
    return cast(ref_sum(xs, order) * f32(s).to(xs[0].device), out_dtype)


def ref_move(x, s, out_dtype, identity):
    """All-gather / broadcast / all-to-all element: a bit copy with the identity epilogue, else round_once((0 + x) * s)."""
    if identity:
        return x.clone()
    return ref_reduce([x], [0], s, out_dtype)


# ------------------------------------------------------------------------------------------------- data
def _exp2(e):
    return torch.exp2(e.float())


def gen_inputs(n, count, in_dt, seed, device="cuda"):
    """Seeded per-rank inputs of in_dt (generated on `device`) built so that the order, the accumulator type, the number of roundings,
    where the scale is applied and the rounding mode all show in the result:
      * random signs and exponents 2^-20 .. 2^12 (fp32 sums of bf16 / fp16 inputs are inexact),
      * cancellation: +B and -B on two ranks and small values elsewhere (the small ones survive only in some orders),
      * rounding ties of bf16, fp16, e4m3 and e5m2: B on one rank and half an output ulp of B on another, plus nothing (an exact tie),
        one small value (just above or below the tie) or two tiny values that tip it only when they meet before B,
      * input-type subnormals, -0 on every rank at some positions and at the last one, values near 65504 for fp16 (sums overflow),
      * NaN and +-inf at fixed positions."""
    g = torch.Generator(device=device).manual_seed(seed)
    dev = device
    rnd = lambda *shape: torch.rand(shape, generator=g, device=dev)
    rint = lambda lo, hi, *shape: torch.randint(lo, hi, shape, generator=g, device=dev)
    sign = torch.where(rnd(n, count) < 0.5, -1.0, 1.0)
    x = sign * _exp2(rint(-20, 13, n, count)) * (1 + rnd(n, count))
    cls = rint(0, 100, count)
    ranks = torch.arange(n, device=dev).unsqueeze(1)
    a = rint(0, n, count)
    b = (a + 1 + (rint(0, max(1, n - 1), count) if n > 1 else 0)) % n
    is_a, is_b = ranks == a, ranks == b
    rest = ~(is_a | is_b)
    psign = torch.where(rnd(count) < 0.5, -1.0, 1.0)

    # cancellation: +B / -B, the others small enough to vanish when added to B
    big = _exp2(rint(12, 15, count)) * psign
    small = sign * _exp2(rint(-16, -11, n, count)) * (1 + rnd(n, count))
    canc = torch.where(is_a, big, torch.where(is_b, -big, small))
    x = torch.where((cls >= 50) & (cls < 65), canc, x)

    # ties of an output type (chosen per position); B with min(p_in, p_out) significant bits so that it is exact in both
    pin = MANT[in_dt]
    tie_types = [torch.bfloat16, torch.float16, torch.float8_e4m3fn, torch.float8_e5m2]
    pout = torch.tensor([MANT[t] for t in tie_types], device=dev)[cls % 4]
    q = torch.minimum(pout, torch.tensor(pin, device=dev))
    eb = rint(2, 8, count)
    k = (rnd(count) * _exp2(q - 1)).floor()
    bval = psign * _exp2(eb) * (1 + k / _exp2(q - 1))
    half = psign * _exp2(eb - pout)                                            # half an output ulp at B
    variant = rint(0, 4, count)
    first_rest = (ranks == (b + 1) % n) & rest
    tiny = psign * 1.5 * _exp2(eb - 25)                                        # 0.75 fp32 ulp of B: lost alone, not in pairs
    nudge = torch.where(rnd(count) < 0.5, -1.0, 1.0) * psign * _exp2(eb - pout - 6)
    eps = torch.where(variant == 0, torch.zeros_like(tiny),                    # exact tie
                      torch.where(variant == 1, nudge,                          # just above / below the tie
                                  tiny))                                        # tiny: sums matter
    eps_r = torch.where(variant == 1, first_rest, rest)                        # one nudge; tiny on every other rank
    negz = torch.where(rnd(n, count) < 0.5, -0.0, 0.0)
    tie = torch.where(is_a, bval, torch.where(is_b, half, torch.where(eps_r, eps, negz)))
    x = torch.where((cls >= 65) & (cls < 85), tie, x)

    # input-type subnormals
    emin = EMIN[in_dt]
    sub = sign * _exp2(rint(emin - MANT[in_dt] + 1, emin, n, count)) * (1 + rnd(n, count))
    x = torch.where((cls >= 85) & (cls < 92), sub, x)
    if in_dt == torch.float16:                                                 # near 65504: the sum overflows in fp16
        x = torch.where((cls >= 92) & (cls < 96), psign * (32768.0 + rnd(n, count) * 32000.0), x)

    idx = torch.arange(count, device=dev)
    x = torch.where((idx % 61 == 7) | (idx == count - 1), torch.full_like(x, -0.0), x)   # -0 on every rank (the last element: in a scalar tail)
    out = x.to(in_dt)
    special = [(3, 1 % n, float("nan")), (11, 0, float("inf")), (19, n - 1, float("-inf")), (27, 0, float("inf")), (27, 1 % n, float("-inf")),
               (35, n - 1, float("nan"))]
    for pos, r, v in special:
        if pos < count:
            out[r, pos] = v
    iv = INT_VIEW[esize(in_dt)]
    for pos, bits in zip((41, 43), NAN_PAYLOADS[in_dt]):                      # NaNs with payloads on every rank: bit copies keep them
        if pos < count:
            out[:, pos] = torch.tensor(bits, dtype=torch.int64).to(iv).view(in_dt)
    return [out[r].clone() for r in range(n)]                                 # own allocations: 16-byte aligned like any buffer


NAN_PAYLOADS = {torch.float32: (0x7F800001, -0x3FFEDD), torch.bfloat16: (0x7F81, -0x3D), torch.float16: (0x7C01, -0x1C9)}


# ------------------------------------------------------------------------------------------------- comparison
def _bits(t):
    return t.contiguous().view(INT_VIEW[esize(t.dtype)])


def first_difference(got, want):
    """Index of the first element whose bits differ (NaN matches NaN of any payload at the same position), or None."""
    g, w = got.reshape(-1), want.reshape(-1)
    same = _bits(g) == _bits(w)
    if g.dtype.is_floating_point:
        same = same | (torch.isnan(g.float()) & torch.isnan(w.float()))
    bad = (~same).nonzero()
    return None if bad.numel() == 0 else int(bad[0])


def assert_same(got, want, what, nan_payloads=False):
    """Bit-for-bit equality except NaN, which is compared by position (nan_payloads=True: NaN bits too, for bit copies). `what` names
    the rank, algorithm, type pair and count."""
    assert got.dtype == want.dtype and got.numel() == want.numel(), f"{what}: {got.dtype}[{got.numel()}] vs {want.dtype}[{want.numel()}]"
    if nan_payloads:
        bad = (_bits(got.reshape(-1)) != _bits(want.reshape(-1))).nonzero()
        i = None if bad.numel() == 0 else int(bad[0])
    else:
        i = first_difference(got, want)
    if i is not None:
        g, w = got.reshape(-1), want.reshape(-1)
        nbad = int((_bits(g) != _bits(w)).sum())
        raise AssertionError(f"{what}: element {i} of {got.numel()} differs (about {nbad} elements): got {g[i].item()!r} "
                             f"(bits {int(_bits(g)[i]):#x}) want {w[i].item()!r} (bits {int(_bits(w)[i]):#x})")
