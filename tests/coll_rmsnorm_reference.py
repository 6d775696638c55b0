"""Order-exact reference of b200collAllReduceRmsNorm (coll/include/b200coll.h), steps 1-5 in fp32 with every product and sum rounded
on its own:

    h[e]   = round_dtype(((+0 + x_0[e]) + ... + x_{N-1}[e]) + residual[e])
    sq[e]  = h[e] * h[e]
    p[c]   = ((+0 + sq[16c]) + sq[16c+1]) + ... + sq[16c+15]; p padded with +0 to the next power of two P and folded
             p = p[:P/2] + p[P/2:] until one value is left
    inv    = 1 / sqrt(fold / row_len + eps)              (IEEE, rounded to nearest)
    out[e] = round_dtype((h[e] * inv) * gamma[e])

numpy's float32 arithmetic rounds every operation (no fused multiply-add), and its sqrt and division are correctly rounded, so the
vectorised `rms_norm` is the contract itself. `rms_norm_loop` renders the same rules one element at a time, as a cross-check of the
vectorised fold. Not collected by pytest (no test_ prefix)."""
import numpy as np
import torch


def _round(a32, dt):
    """fp32 numpy array -> torch tensor of dt, rounded to nearest even."""
    return torch.from_numpy(np.ascontiguousarray(a32, dtype=np.float32)).to(dt)


def _f32(t):
    return t.float().numpy()


def rms_norm(xs, residual, gamma, eps, dt):
    """xs: the N ranks' [rows, row_len] tensors; residual [rows, row_len]; gamma [row_len]; all of dt (CPU). Returns (new residual, out),
    tensors of dt."""
    rows, row_len = residual.shape
    with np.errstate(all="ignore"):
        acc = np.zeros((rows, row_len), dtype=np.float32)
        for x in xs:
            acc = acc + _f32(x)
        h = _round(acc + _f32(residual), dt)
        hf = _f32(h)
        sq = hf * hf
        nch = row_len // 16
        by_chunk = sq.reshape(rows, nch, 16)
        p = np.zeros((rows, nch), dtype=np.float32)
        for i in range(16):
            p = p + by_chunk[:, :, i]
        P = 1
        while P < nch:
            P *= 2
        p = np.concatenate([p, np.zeros((rows, P - nch), dtype=np.float32)], axis=1)
        while P > 1:
            P //= 2
            p = p[:, :P] + p[:, P:]
        ms = p[:, 0] / np.float32(row_len)
        inv = np.float32(1.0) / np.sqrt(ms + np.float32(eps))
        out = (hf * inv[:, None]) * _f32(gamma)[None, :]
    return h, _round(out, dt)


def rms_norm_loop(xs, residual, gamma, eps, dt):
    """The same rules as plain sequential loops over np.float32 scalars (tiny shapes only)."""
    rows, row_len = residual.shape
    f = np.float32
    xs32 = [_f32(x) for x in xs]
    r32, g32 = _f32(residual), _f32(gamma)
    h = np.zeros((rows, row_len), dtype=np.float32)
    out = np.zeros((rows, row_len), dtype=np.float32)
    with np.errstate(all="ignore"):
        for i in range(rows):
            for e in range(row_len):
                a = f(0.0)
                for x in xs32:
                    a = f(a + x[i, e])
                h[i, e] = a + r32[i, e]
            hr = _f32(_round(h[i], dt))
            p = []
            for c in range(row_len // 16):
                s = f(0.0)
                for e in range(16 * c, 16 * c + 16):
                    s = f(s + f(hr[e] * hr[e]))
                p.append(s)
            while len(p) & (len(p) - 1):
                p.append(f(0.0))
            while len(p) > 1:
                half = len(p) // 2
                p = [f(p[k] + p[k + half]) for k in range(half)]
            inv = f(f(1.0) / np.sqrt(f(f(p[0] / f(row_len)) + f(eps))))
            for e in range(row_len):
                out[i, e] = f(f(hr[e] * inv) * g32[e])
    return _round(h, dt), _round(out, dt)
