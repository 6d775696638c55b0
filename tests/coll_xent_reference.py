"""Reference for the vocab-parallel cross-entropy (b200collVocabParallelCrossEntropy / ...Backward): the header's formulas in numpy
float32, one IEEE operation at a time, in the kernels' order. exp and log are the library's own (coll/src/xent.cu's xent_exp and
xent_log), mirrored here operation for operation, so the reference and the kernels agree bit for bit; the *_loop renderings take one
element at a time and use the same two functions.

Logits are given per rank as [rows, Vl] arrays of bf16, fp16 or fp32 (torch tensors on the CPU); results are numpy float32 arrays
(grad: a torch tensor of the logits' dtype)."""
import numpy as np
import torch

F = np.float32
LOG2E = F(1.44269504088896341)
LN2_HI, LN2_LO = F(0.693359375), F(-2.12194440e-4)
EXP_P = [F(c) for c in (1.9875691500e-4, 1.3981999507e-3, 8.3334519073e-3, 4.1665795894e-2, 1.6666665459e-1, 5.0000001201e-1)]
EXP_LO, EXP_HI = F(-87.0), F(88.7228317)
LOG_P = [F(c) for c in (7.0376836292e-2, -1.1514610310e-1, 1.1676998740e-1, -1.2420140846e-1, 1.4249322787e-1, -1.6668057665e-1,
                        2.0000714765e-1, -2.4999993993e-1, 3.3333331174e-1)]
SQRTH_BITS = 0x3F3504F3          # sqrt(0.5) rounded to fp32


def xexp(x):
    """xent_exp, elementwise on a float32 array: k = rint(x * log2(e)); r = (x - k * LN2_HI) - k * LN2_LO; y = ((p(r) * r^2) + r) + 1
    with p a degree-5 Horner polynomial; the result y * 2^k by adding k to y's exponent bits. x < -87 gives +0, x > 88.7228317 gives
    +inf, NaN stays NaN."""
    x = np.asarray(x, dtype=F)
    with np.errstate(invalid="ignore", over="ignore"):
        kf = np.rint(x * LOG2E).astype(F)
        r = ((x - kf * LN2_HI) - kf * LN2_LO).astype(F)
        z = (r * r).astype(F)
        p = np.full_like(r, EXP_P[0])
        for c in EXP_P[1:]:
            p = (p * r + c).astype(F)                    # two roundings: numpy float32 has no fused multiply-add
        y = ((p * z + r) + F(1.0)).astype(F)
        ok = (x >= EXP_LO) & (x <= EXP_HI)
        k = np.where(ok, kf, 0).astype(np.int32)
        res = (y.view(np.int32) + (k << 23)).view(F)
    res = np.where(x < EXP_LO, F(0.0), res)
    res = np.where(x > EXP_HI, F(np.inf), res)
    return np.where(np.isnan(x), x, res).astype(F)


def xlog(x):
    """xent_log, elementwise on a float32 array: x = 2^e * m with m in [sqrt(1/2), sqrt(2)) by exponent-bit arithmetic, f = m - 1,
    log = (((f + ((f^3 * q(f)) + e * LN2_LO)) + -0.5 * f^2) + e * LN2_HI) in that order (q degree 8). Defined on +0, the positive
    normal numbers and +inf (+0 gives -inf, +inf gives +inf, negative or NaN gives NaN); the library calls it only on S >= 1, +0, +inf
    and NaN."""
    x = np.asarray(x, dtype=F)
    bits = x.view(np.int32)
    e = ((bits - np.int32(SQRTH_BITS)) >> 23).astype(np.int32)
    m = (bits - (e << 23)).view(F)
    with np.errstate(invalid="ignore", over="ignore"):
        f = (m - F(1.0)).astype(F)
        z = (f * f).astype(F)
        q = np.full_like(f, LOG_P[0])
        for c in LOG_P[1:]:
            q = (q * f + c).astype(F)
        ef = e.astype(F)
        y = ((q * f) * z).astype(F)
        y = (y + ef * LN2_LO).astype(F)
        y = (y + F(-0.5) * z).astype(F)
        res = ((f + y) + ef * LN2_HI).astype(F)
    res = np.where(x == 0, F(-np.inf), res)
    res = np.where(x == np.inf, F(np.inf), res)
    return np.where(np.isnan(x) | (x < 0), F(np.nan), res).astype(F)


def widen(t):
    """A bf16 / fp16 / fp32 torch tensor as a numpy float32 array, exactly."""
    return t.float().numpy().astype(F)


def chunk_fold(v):
    """The header's sum of one row's exp values v (float32): 16-element chunk sums in element order from +0, padded with +0 to a power
    of two P, folded p[:P/2] + p[P/2:] until one value is left. v is [..., L]; returns [...]."""
    v = np.asarray(v, dtype=F)
    L = v.shape[-1]
    C = -(-L // 16)
    pad = np.zeros(v.shape[:-1] + (C * 16 - L,), dtype=F)
    ch = np.concatenate([v, pad], axis=-1).reshape(v.shape[:-1] + (C, 16))
    p = np.zeros(v.shape[:-1] + (C,), dtype=F)
    for i in range(16):
        p = (p + ch[..., i]).astype(F)
    P = 1
    while P < C:
        P *= 2
    p = np.concatenate([p, np.zeros(v.shape[:-1] + (P - C,), dtype=F)], axis=-1)
    while P > 1:
        P //= 2
        p = (p[..., :P] + p[..., P:]).astype(F)
    return p[..., 0]


def partials(x, r, vl, target):
    """Rank r's records for every row: (m, s, z, owns) as float32 / bool arrays. x: [rows, Vl] float32."""
    rows = x.shape[0]
    if vl:
        with np.errstate(invalid="ignore"):
            m = np.max(x, axis=1).astype(F) if rows else np.zeros(0, F)        # np.max propagates NaN
    else:
        m = np.full(rows, -np.inf, F)
    with np.errstate(invalid="ignore"):
        s = chunk_fold(xexp(x - m[:, None])) if rows else np.zeros(0, F)
    s = np.where(m == -np.inf, F(0.0), s).astype(F)
    col = target - r * vl
    owns = (col >= 0) & (col < vl)
    z = np.zeros(rows, F)
    if owns.any():
        idx = np.nonzero(owns)[0]
        z[idx] = x[idx, col[idx]]
    return m, s, z, owns


def combine(recs, target, ignore_index, n, vl):
    """The records of ranks 0 .. N-1 (a list of partials()) combined in rank order: (loss, lse)."""
    rows = len(target)
    M = recs[0][0].copy()
    for m, _, _, _ in recs[1:]:
        M = np.where(np.isnan(M) | (M >= m), M, m).astype(F)
        M = np.where(np.isnan(m), m, M).astype(F)
    S = np.zeros(rows, F)
    z = np.zeros(rows, F)
    with np.errstate(invalid="ignore", over="ignore"):
        for m, s, zr, owns in recs:
            e = (s * xexp(m - M)).astype(F)
            e = np.where(m == -np.inf, F(0.0), e)
            S = (S + e).astype(F)
            z = np.where(owns, zr, z)
        lse = (M + xlog(S)).astype(F)
        loss = (lse - z).astype(F)
    loss = np.where((target < 0) | (target >= n * vl), F(np.nan), loss)
    loss = np.where(target == ignore_index, F(0.0), loss)
    return loss.astype(F), lse


def forward(logits, target, ignore_index=-100):
    """logits: per rank [rows, Vl] torch tensors (bf16, fp16 or fp32); target: [rows] int64 global ids. Returns (loss, lse), the same on
    every rank."""
    n = len(logits)
    vl = logits[0].shape[1]
    t = np.asarray(target, dtype=np.int64)
    recs = [partials(widen(x), r, vl, t) for r, x in enumerate(logits)]
    return combine(recs, t, ignore_index, n, vl)


def backward(logits_r, r, n, target, lse, dloss, ignore_index=-100):
    """Rank r's grad, [rows, Vl] of the logits' dtype: round((exp(x - lse) - [col == target]) * dloss), +0 on ignored rows, NaN on
    rows whose target is out of range."""
    x = widen(logits_r)
    rows, vl = x.shape
    t = np.asarray(target, dtype=np.int64)
    lse = np.asarray(lse, dtype=F)
    dl = np.asarray(dloss, dtype=F)
    with np.errstate(invalid="ignore", over="ignore"):
        e = xexp((x - lse[:, None]).astype(F))
        hit = (np.arange(vl)[None, :] + r * vl) == t[:, None]
        d = np.where(hit, (e - F(1.0)).astype(F), e)
        g = (d * dl[:, None]).astype(F)
    bad = (t < 0) | (t >= n * vl)
    g = np.where(bad[:, None] & (t != ignore_index)[:, None], F(np.nan), g)
    g = np.where((t == ignore_index)[:, None], F(0.0), g)
    return torch.from_numpy(np.ascontiguousarray(g)).to(logits_r.dtype)


def forward_loop(logits, target, ignore_index=-100):
    """forward() one element at a time: the max, the chunk sums and their fold written out as loops over Python floats held in
    np.float32."""
    n = len(logits)
    vl = logits[0].shape[1]
    rows = len(target)
    xs = [widen(x) for x in logits]
    loss, lse = np.zeros(rows, F), np.zeros(rows, F)
    for t in range(rows):
        recs = []
        for r in range(n):
            m = F(-np.inf)
            for j in range(vl):
                v = xs[r][t, j]
                if np.isnan(v) or np.isnan(m):
                    m = v if np.isnan(v) else m
                elif v > m:
                    m = v
            if m == -np.inf:
                s = F(0.0)
            else:
                chunks = []
                for c in range(-(-vl // 16)):
                    p = F(0.0)
                    for j in range(16 * c, min(vl, 16 * c + 16)):
                        p = F(p + xexp(F(xs[r][t, j] - m)))
                    chunks.append(p)
                P = 1
                while P < len(chunks):
                    P *= 2
                chunks += [F(0.0)] * (P - len(chunks))
                while len(chunks) > 1:
                    h = len(chunks) // 2
                    chunks = [F(chunks[i] + chunks[i + h]) for i in range(h)]
                s = chunks[0]
            col = int(target[t]) - r * vl
            owns = 0 <= col < vl
            recs.append((m, s, xs[r][t, col] if owns else F(0.0), owns))
        M = recs[0][0]
        for m, _, _, _ in recs[1:]:
            if np.isnan(m) or np.isnan(M):
                M = m if np.isnan(m) else M
            elif m > M:
                M = m
        S, z = F(0.0), F(0.0)
        for m, s, zr, owns in recs:
            e = F(0.0) if m == -np.inf else F(s * xexp(F(m - M)))
            S = F(S + e)
            if owns:
                z = zr
        lse[t] = F(M + xlog(S))
        tt = int(target[t])
        if tt == ignore_index:
            loss[t] = F(0.0)
        elif tt < 0 or tt >= n * vl:
            loss[t] = F(np.nan)
        else:
            loss[t] = F(lse[t] - z)
    return loss, lse
