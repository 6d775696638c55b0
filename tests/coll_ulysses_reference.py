"""Reference for the Ulysses all-to-all (b200collAllToAllSeqToHeads / HeadsToSeq), built from plain torch permutes on byte views, so
every dtype (FP8 included) moves bit for bit. One tensor at a time; a rank's tensor is a [B, S_l, H, D] sequence shard or a
[B, S, Hl, D] head shard."""
import torch


def _bytes(t):
    """t as a contiguous uint8 tensor with the head dim widened to D * sizeof(dtype) bytes."""
    return t.contiguous().view(torch.uint8)


def local_heads(nranks, heads):
    """Hl: heads // nranks, or 1 when heads divides nranks (each head replicated to nranks // heads ranks)."""
    if heads % nranks == 0:
        return heads // nranks
    assert nranks % heads == 0, (nranks, heads)
    return 1


def seq_to_heads(xs):
    """xs[s]: rank s's [B, S_l, H, D] shard. Returns ys[r]: rank r's [B, N * S_l, Hl, D], as uint8 (widened head dim)."""
    n = len(xs)
    x = torch.stack([_bytes(t) for t in xs])                        # [N(s), B, S_l, H, Db]
    N, B, S_l, H, Db = x.shape
    if H % n:                                                        # replicated: head r * H // N of every rank r
        x = x.repeat_interleave(n // H, dim=3)
        H = n
    hl = H // n
    y = x.view(N, B, S_l, n, hl, Db).permute(3, 1, 0, 2, 4, 5)       # [N(r), B, N(s), S_l, Hl, Db]
    return list(y.reshape(n, B, N * S_l, hl, Db).unbind(0))


def heads_to_seq(ys):
    """ys[s]: rank s's [B, N * S_l, H / N, D] head shard. Returns xs[r]: rank r's [B, S_l, H, D] sequence shard, as uint8."""
    n = len(ys)
    y = torch.stack([_bytes(t) for t in ys])                        # [N(s), B, S, Hl, Db]
    N, B, S, hl, Db = y.shape
    x = y.view(N, B, n, S // n, hl, Db).permute(2, 1, 3, 0, 4, 5)    # [N(r), B, S_l, N(s), Hl, Db]
    return list(x.reshape(n, B, S // n, N * hl, Db).unbind(0))


def seq_to_heads_loop(xs):
    """seq_to_heads by the header's formula, one (rank, b, s, t, j) at a time: y_r[b, s * S_l + t, j] = x_s[b, t, head(r, j)]."""
    n = len(xs)
    xb = [_bytes(t) for t in xs]
    B, S_l, H, Db = xb[0].shape
    hl = local_heads(n, H)
    ys = [torch.zeros(B, n * S_l, hl, Db, dtype=torch.uint8) for _ in range(n)]
    for r in range(n):
        for j in range(hl):
            h = r * H // n + j if H % n == 0 else r * H // n
            for s in range(n):
                for b in range(B):
                    for t in range(S_l):
                        ys[r][b, s * S_l + t, j] = xb[s][b, t, h]
    return ys


def heads_to_seq_loop(ys):
    """heads_to_seq by the header's formula: x_r[b, t, h] = y_{h // Hl}[b, r * S_l + t, h % Hl]."""
    n = len(ys)
    yb = [_bytes(t) for t in ys]
    B, S, hl, Db = yb[0].shape
    S_l, H = S // n, hl * n
    xs = [torch.zeros(B, S_l, H, Db, dtype=torch.uint8) for _ in range(n)]
    for r in range(n):
        for h in range(H):
            for b in range(B):
                for t in range(S_l):
                    xs[r][b, t, h] = yb[h // hl][b, r * S_l + t, h % hl]
    return xs
