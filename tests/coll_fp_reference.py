"""Order-exact fp32 reference for the fp32 / fp16 / bf16 / e4m3 / e5m2 collectives of libb200coll, and seeded data that can tell
orders apart.

Every fused sum / avg path widens each input to fp32, accumulates from +0 in a fixed order, multiplies once by the fp32 scale (avg: the
fp32 product scale * (1/N)) and rounds once, to nearest even, to the output type (FP8 saturates, fp16 overflows to inf). The order is
a property of the kernel that ran, so the reference takes it as an argument:

    [r0, r1, ...]                 that rank order for every element (LL, LL2, one-shot, rooted reduce, the generic kernel)
    ("rotate", r)                 r, r+1, ..., r-1 (P2P reduce-scatter at receiving rank r)
    ("owner", N, E, count)        two-shot all-reduce: vector v belongs to slice o with nvec*o//N <= v < nvec*(o+1)//N and is summed
                                  o, o+1, ..., o-1; elements past the last whole vector are summed in rank order (ar_tail_rank0)
    ("staged", N, E, count, chunk)  the staged all-reduce: two-shot on each chunk of `chunk` elements, slices from the chunk's nvec

FP8 inputs are summed in rank order on every P2P kernel (the two-shot all-reduce and the P2P reduce-scatter included), so their
order model is always [0, 1, ..., N-1].

Not collected by pytest (no test_ prefix); imported by the test_coll_fp_numerics_* and test_coll_fp8_numerics_* files and the other
GPU tests."""
import numpy as np
import torch

from container_engine_accelerators_b200.ops.coll import MAX, MIN, PROD, SUM

STAGE_HALF_BYTES = 32 << 20          # coll/src/layout.h kStageHalfBytes
LL_ONESHOT_MAX_BYTES = 512 << 10     # kLLOneShotMaxBytes: per source
HOST_ZEROCOPY_BYTES = 4096 << 10     # hostpath.cu defaults: B200COLL_HOST_ZEROCOPY_KB
HOST_PIPELINE_BYTES = 8192 << 10     # B200COLL_HOST_PIPELINE_KB
BULK_MIN_BYTES = 1 << 20             # collectives.cu bulk_min_bytes default (B200COLL_BULK_MIN_KB): identity moves from here on the copy engine
LL_SENTINEL, LL_SANITIZED = 0xFFFFFFFF, 0x7FFF7FFF    # layout.h kLLSentinel / kLLSanitized

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


def scale_of(coll, op, scale, n):
    """The scale a sum (scale) or an avg (avg_scale) multiplies by."""
    return scale if op == coll.SUM else avg_scale(scale, n)


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


def host_chunks(count, in_size, out_size, nranks):
    """b200collAllReduceHost with its default knobs (they are read once per process): the regime and the element count of each
    b200collAllReduce it makes, in order. "zero_copy" is one call on the mapped host pointers; "single" and "pipelined" run on arena
    staging buffers, so each chunk is an all-reduce of its own, with its own algorithm choice and (two-shot) its own slices."""
    nbytes = count * in_size
    zc_feasible = nranks == 1 or nbytes <= LL_ONESHOT_MAX_BYTES or (in_size == out_size and nbytes <= LL_ONESHOT_MAX_BYTES * nranks)
    if nbytes <= HOST_ZEROCOPY_BYTES and zc_feasible:
        return "zero_copy", [count]
    chunk = min(16 << 20, max(4 << 20, nbytes // 6))
    if nbytes < HOST_PIPELINE_BYTES:
        chunk = nbytes
    chunk = (chunk + 1023) // 1024 * 1024
    if chunk >= nbytes:
        return "single", [count]
    ce = chunk // in_size
    return "pipelined", [min(ce, count - d) for d in range(0, count, ce)]


def staged_owner_map(count, n, e, chunk, device="cpu"):
    parts = [owner_map(min(chunk, count - d), n, e, device) for d in range(0, count, chunk)]
    return torch.cat(parts)


def rotation(r, n):
    return [(r + j) % n for j in range(n)]


RANK_ORDER_ALGOS = ("ll", "ll2", "oneshot")


def order_for(algo, n, in_dt, count):
    """The order model of an all-reduce that recorded `algo`: FP8 inputs are summed in rank order on every kernel; 16- and 32-bit inputs
    in rank order except on two-shot (slice owner first)."""
    if in_dt in FP8_MAX or algo in RANK_ORDER_ALGOS:
        return list(range(n))
    assert algo == "twoshot", f"no bit-exact order model for {algo}"
    return ("owner", n, vec_elems(in_dt), count)


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


def ll_move(x):
    """The identity epilogue on the Lamport (ll) path: a bit copy except that every 4-byte word equal to the empty-slot sentinel
    (0xFFFFFFFF, NaN in every type) arrives as its sanitized form 0x7FFF7FFF (bytes FF 7F FF 7F, still NaN in every type). Words are
    counted from the start of the buffer, which is 16-byte aligned."""
    u = x.contiguous().view(torch.uint8).clone()
    w = u[:u.numel() // 4 * 4].view(torch.int32)                              # a partial last word is padded with zeros: never the sentinel
    w[w == -1] = LL_SANITIZED
    return u.view(x.dtype)


# the generic kernel (coll/src/generic.cu): every type, sum / prod / min / max
NP_INT = {torch.int8: np.int8, torch.uint8: np.uint8, torch.int32: np.int32, torch.uint32: np.uint32, torch.int64: np.int64,
          torch.uint64: np.uint64}


def int_numpy(t):
    """An integer tensor's values as a numpy array of its own type (through its bytes: torch has few kernels for uint32 / uint64)."""
    return t.contiguous().view(torch.uint8).cpu().numpy().view(NP_INT[t.dtype])


def int_tensor(a, dtype, device="cuda"):
    """A numpy integer array as a tensor of dtype (same width) on `device`, bit for bit."""
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).to(device).view(dtype)


def generic_ref(xs, op):
    """The generic kernel's result: rank 0's value, then ranks 1 .. N-1 in order. Integers wrap (numpy arithmetic in the type's own
    width; min and max compare as the type is signed or not). Floating point accumulates in fp32 for fp16, bf16 and FP8 and in its own
    type otherwise, and is rounded once at the end (FP8 saturates); min / max propagate a NaN from any rank and keep the lower rank's
    value on a tie."""
    dt = xs[0].dtype
    if dt in NP_INT:
        a = [int_numpy(x) for x in xs]
        acc = a[0].copy()
        with np.errstate(over="ignore"):
            for b in a[1:]:
                acc = {SUM: np.add, PROD: np.multiply, MIN: np.minimum, MAX: np.maximum}[op](acc, b).astype(a[0].dtype)
        return int_tensor(acc, dt, xs[0].device)
    wide = dt in (torch.float16, torch.bfloat16) or dt in FP8_MAX
    acc = xs[0].float() if wide else xs[0].clone()
    for x in xs[1:]:
        b = x.float() if wide else x
        if op == SUM:
            acc = acc + b
        elif op == PROD:
            acc = acc * b
        elif op == MIN:
            acc = torch.where((b < acc) | (b != b), b, acc)
        else:
            assert op == MAX, op
            acc = torch.where((b > acc) | (b != b), b, acc)
    return cast(acc, dt)


def int_inputs(n, count, dtype, seed):
    """Seeded per-rank integers over the type's whole range (so half are >= 2^31 or 2^63 as unsigned, negative as signed, and sums and
    products wrap), with the type's extremes at fixed positions: at element 5 + k, rank k % N holds the k-th of min, max, 0, all ones,
    the top bit alone and the top bit's complement, and element 17 holds max on rank 0 and min on the other ranks (13: the reverse)."""
    nt = NP_INT[dtype]
    info = np.iinfo(nt)
    rng = np.random.default_rng(seed)
    bits = 8 * np.dtype(nt).itemsize
    u = np.dtype(f"u{bits // 8}")
    xs = [rng.integers(0, 1 << bits, size=count, dtype=np.uint64).astype(u).view(nt) for _ in range(n)]
    as_t = lambda v: np.array([v], dtype=u).view(nt)[0]
    extremes = [info.min, info.max, 0, as_t((1 << bits) - 1), as_t(1 << (bits - 1)), as_t((1 << (bits - 1)) - 1)]
    for k, v in enumerate(extremes):
        if 5 + k < count:
            xs[k % n][5 + k] = v
    for pos, first, rest in ((17, info.max, info.min), (13, info.min, info.max)):
        if pos < count:
            for r in range(n):
                xs[r][pos] = first if r == 0 else rest
    return xs


# ------------------------------------------------------------------------------------------------- data
def random_fp8(torch, n, dt, seed):
    """Seeded random bytes reinterpreted as FP8, NaN and inf patterns replaced: every exponent occurs, subnormals and values near the
    maximum included, so sums round and saturate."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    b = torch.randint(0, 256, (n,), generator=g, dtype=torch.int32)
    if dt == torch.float8_e4m3fn:
        b = torch.where((b & 0x7F) == 0x7F, b - 1, b)                # S.1111.111 is NaN
    else:
        b = torch.where((b & 0x7C) == 0x7C, b & 0x83 | 0x78, b)      # exponent 11111 is inf / NaN
    return b.to(torch.uint8).view(dt).cuda()


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
    if in_dt in FP8_MAX:
        return _gen_fp8(n, count, in_dt, seed, device)
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


NAN_PAYLOADS = {torch.float32: (0x7F800001, -0x3FFEDD), torch.bfloat16: (0x7F81, -0x3D), torch.float16: (0x7C01, -0x1C9),
                torch.float8_e4m3fn: (0x7F, 0xFF), torch.float8_e5m2: (0x7D, 0xFE)}
# FP8 bytes at fixed positions (position, rank or None for every rank, byte). e4m3 has no inf: 0x7F and 0xFF are its only NaNs.
FP8_SPECIAL = {
    torch.float8_e4m3fn: [(3, 1, 0x7F), (35, -1, 0xFF)],
    torch.float8_e5m2: [(3, 1, 0x7E), (11, 0, 0x7C), (19, -1, 0xFC), (27, 0, 0x7C), (27, 1, 0xFC), (35, -1, 0xFF)],
}
LL_WORDS = ((48, LL_SENTINEL), (52, LL_SANITIZED))     # element (byte) offset of a 4-byte word on rank 1 % N


def _gen_fp8(n, count, in_dt, seed, device):
    """gen_inputs for e4m3 / e5m2 inputs; every value is built exactly in the input type (no rounding on the way in):
      * random signs, 4 (e4m3) or 3 (e5m2) significant bits and a spread of exponents,
      * cancellation: +B and -B on two ranks (B in 2^12 .. 2^15 for e5m2, 2^6 .. 2^8 for e4m3) and small values down to 2^-16 (e5m2) or
        2^-9 (e4m3) elsewhere; for e5m2 the small ones survive only in some orders, for e4m3 every sum is exact in fp32 in any order,
      * rounding ties of bf16, fp16, e4m3 and e5m2 outputs: B (with as many significant bits as the input type has) on one rank and half
        an output ulp of B on another, plus nothing (an exact tie), a nudge just above or below it by less than half an fp16 ulp (rounding
        through fp16 removes it), or, for e5m2 with B >= 2^8, a tiny value of half an fp32 ulp of B on every other rank: lost one by one,
        a whole ulp when two meet before B,
      * same-sign values near the maximum: sums past 448 (e4m3) and past 57344 and 65504 (e5m2), so FP8 outputs saturate and fp16
        outputs overflow to inf,
      * input-type subnormals, -0 on every rank at positions 7 mod 61 and at the last one (a scalar tail),
      * FP8_SPECIAL bytes (NaN, and for e5m2 +-inf, with payloads), NAN_PAYLOADS at positions 41 and 43 on every rank, and on rank 1 % N
        the words LL_WORDS: the Lamport sentinel FF FF FF FF at byte 48 and its sanitized form FF 7F FF 7F at byte 52."""
    g = torch.Generator(device=device).manual_seed(seed)
    dev = device
    e5 = in_dt == torch.float8_e5m2
    p = MANT[in_dt]
    rnd = lambda *shape: torch.rand(shape, generator=g, device=dev)
    rint = lambda lo, hi, *shape: torch.randint(lo, hi, shape, generator=g, device=dev)
    frac = lambda k: 1 + k.float() / (1 << (p - 1))                               # 1.m with p - 1 fraction bits
    sign = torch.where(rnd(n, count) < 0.5, -1.0, 1.0)
    x = sign * _exp2(rint(-12, 13, n, count) if e5 else rint(-6, 8, n, count)) * frac(rint(0, 1 << (p - 1), n, count))
    cls = rint(0, 100, count)
    ranks = torch.arange(n, device=dev).unsqueeze(1)
    a = rint(0, n, count)
    b = (a + 1 + (rint(0, max(1, n - 1), count) if n > 1 else 0)) % n
    is_a, is_b = ranks == a, ranks == b
    rest = ~(is_a | is_b)
    psign = torch.where(rnd(count) < 0.5, -1.0, 1.0)

    # cancellation
    big = psign * (_exp2(rint(12, 16, count)) * frac(rint(0, 3, count)) if e5 else _exp2(rint(6, 9, count)) * frac(rint(0, 7, count)))
    se = rint(-16, -8, n, count) if e5 else rint(-9, -3, n, count)
    small = sign * _exp2(se) * torch.where(se >= EMIN[in_dt], frac(rint(0, 1 << (p - 1), n, count)), torch.ones_like(sign))
    x = torch.where((cls >= 50) & (cls < 65), torch.where(is_a, big, torch.where(is_b, -big, small)), x)

    # ties of an output type (chosen per position)
    tie_types = [torch.bfloat16, torch.float16, torch.float8_e4m3fn, torch.float8_e5m2]
    tsel = cls % 4
    pout = torch.tensor([MANT[t] for t in tie_types], device=dev)[tsel]
    q = torch.minimum(pout, torch.tensor(p, device=dev))                         # significant bits of B: exact in input and output
    if e5:
        # e4m3 output: B + half must stay below 448, so B is 256, 320 or 384 (half = 16); otherwise B in 2^8 .. 2^13
        eb = torch.where(tsel == 2, torch.full_like(cls, 8), rint(8, 14, count))
        kmax = torch.where(tsel == 2, torch.full_like(cls, 3), _exp2(q - 1).long())
    else:
        eb = rint(3, 8, count)                                                    # half an fp16 ulp of B (2^(eb-11)) is still >= 2^-9
        kmax = _exp2(q - 1).long()
    k = (rnd(count) * kmax).floor()
    bval = psign * _exp2(eb) * (1 + k / _exp2(q - 1))
    half = psign * _exp2(eb - pout)
    variant = rint(0, 4, count)
    if not e5:
        variant = torch.where(variant >= 2, variant - 2, variant)                 # no tiny pairs for e4m3: exact ties and nudges
    first_rest = (ranks == (b + 1) % n) & rest
    tiny = psign * _exp2(eb - 24)                                                 # half an fp32 ulp of B: lost alone (B is even), not in pairs
    nudge = torch.where(rnd(count) < 0.5, -1.0, 1.0) * psign * _exp2(eb - (13 if e5 else 12))   # < half an fp16 ulp of B
    eps = torch.where(variant == 0, torch.zeros_like(tiny), torch.where(variant == 1, nudge, tiny))
    eps_r = torch.where(variant == 1, first_rest, rest)
    negz = torch.where(rnd(n, count) < 0.5, -0.0, 0.0)
    tie = torch.where(is_a, bval, torch.where(is_b, half, torch.where(eps_r, eps, negz)))
    x = torch.where((cls >= 65) & (cls < 85), tie, x)

    # saturation: one sign per position, magnitudes near the maximum on every rank
    top = _exp2(rint(14, 16, n, count)) * frac(rint(0, 4, n, count)) if e5 else _exp2(rint(7, 9, n, count)) * frac(rint(0, 7, n, count))
    x = torch.where((cls >= 85) & (cls < 92), psign * top.clamp(max=FP8_MAX[in_dt]), x)

    # input-type subnormals: k * 2^(emin - p + 1)
    sub = sign * rint(1, 1 << (p - 1), n, count).float() * _exp2(torch.tensor(EMIN[in_dt] - p + 1, device=dev))
    x = torch.where((cls >= 92) & (cls < 99), sub, x)

    idx = torch.arange(count, device=dev)
    x = torch.where((idx % 61 == 7) | (idx == count - 1), torch.full_like(x, -0.0), x)
    out = x.to(in_dt)
    bits = out.view(torch.uint8)
    for pos, r, v in FP8_SPECIAL[in_dt]:
        if pos < count:
            bits[r % n, pos] = v
    for pos, v in zip((41, 43), NAN_PAYLOADS[in_dt]):
        if pos < count:
            bits[:, pos] = v
    for pos, word in LL_WORDS:
        if pos + 4 <= count:
            bits[1 % n, pos:pos + 4] = torch.tensor(list(word.to_bytes(4, "little")), dtype=torch.uint8, device=dev)
    return [out[r].clone() for r in range(n)]


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
