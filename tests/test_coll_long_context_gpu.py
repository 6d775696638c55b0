"""The Ulysses all-to-all and the context-parallel all-gather and reduce-scatter at long-context shapes (`pytest -m gpu`), virtual ranks
sharing cuda:0 unless a test says otherwise.

tests/test_coll_ulysses_gpu.py and tests/test_coll_context_gpu.py check both families at toy shapes, where a call is one pass of the
kernels' grid-stride loop and every byte offset fits 32 bits. These tests reach what only long sequences reach:
  a. model shapes: Llama-3-8B and -70B, MHA, MQA and replicated GQA through Ulysses; Llama K and V and the MLA pair (c_kv 512 + k_pe 64)
     through context parallelism; at 32k and 128k tokens on 2, 4 and 8 ranks; the fused calls against the unfused composition at
     Llama-3-70B, 128k tokens, 8 ranks;
  b. awkward geometry: segments of 8 to 32 vectors, odd and non-power-of-two shards, B = 3 with load-balanced chunks, 3 and 6 ranks,
     three tensors whose prefix boundaries fall inside an unroll group;
  c. launch shapes: one to three CTAs and pinned thread counts, with totals that leave the last unroll group partial;
  d. past 4 GiB: a context-parallel full tensor and a Ulysses call whose both sides are larger than 2^32 bytes;
  e. one rank per GPU, when more than one is visible.

References: tests/coll_ulysses_reference and tests/coll_context_reference run on device tensors (checked against their CPU run and the
per-element formula loops at a small shape first), with coll_fp_reference.ref_sum and cast for the reduce-scatter; past 4 GiB the
expected bytes are built slice by slice. Gather and Ulysses sources are random bytes (NaN payloads, -0, inf), reduce-scatter inputs come
from coll_fp_reference.gen_inputs, and outputs are poisoned first. A mismatch names the tensor, rank, batch row, token and byte (or
element) of the first difference, and how many differ."""
import contextlib

import pytest
import torch

from tests import coll_context_reference as cref
from tests import coll_fp_reference as R
from tests import coll_ulysses_reference as uref
from tests.coll_gpu_harness import Group, coll_mod, poison, torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu

TIMEOUT_MS = 60000              # the watchdog turns a protocol bug into a RemoteError instead of a hung GPU
POISON = 0x7B                   # the byte harness.poison writes
BF16 = torch.bfloat16
GEN_BLOCK = 1 << 21             # elements per gen_inputs call when filling large reduce-scatter inputs
SEQ = (32768, 131072)           # full sequence lengths of the model shapes (S_l = S / N)
D_MODEL = 128


def prod(shape):
    n = 1
    for d in shape:
        n *= d
    return n


@contextlib.contextmanager
def make_group(coll, n, arena_bytes, devices=None):
    """A Group with room for arena_bytes per rank. A failure inside is reported by its message alone: a traceback shows each frame's
    arguments, and rendering an arena tensor once the group is destroyed would read unmapped device memory."""
    with Group(torch, coll, n, devices=devices, arena_mb=arena_bytes // (1 << 20) + 64, timeout_ms=TIMEOUT_MS) as g:
        try:
            yield g
            return
        except Exception as e:
            msg = f"{type(e).__name__}: {e}"
    pytest.fail(msg, pytrace=False)


class Arena:
    """Arena tensors of a group, released together."""

    def __init__(self, g):
        self.g, self.held = g, []

    def __call__(self, r, shape, dt):
        c = self.g.comms[r]
        with torch.cuda.device(c.device):
            t = c.empty(prod(shape), dt)
        self.held.append((c, t))
        return t.view(shape)

    def free(self, views):
        self.g.sync()
        ptrs = {v.data_ptr() for v in views}
        for c, t in self.held:
            if t.data_ptr() in ptrs:
                c.release(t)
        self.held = [(c, t) for c, t in self.held if t.data_ptr() not in ptrs]

    def release(self):
        self.g.sync()
        for c, t in self.held:
            c.release(t)
        self.held = []


def dev_of(g, r):
    return f"cuda:{g.comms[r].device}"


def random_bytes(shape, dt, seed, device):
    gen = torch.Generator(device=device).manual_seed(seed)
    nb = prod(shape) * R.esize(dt)
    return torch.randint(0, 256, (nb,), dtype=torch.uint8, generator=gen, device=device).view(dt).view(shape)


def packed_views(buf, B, S_l, cols, widths):
    """Column slices [B, S_l, W_i] of a packed [B * S_l, ...] buffer, starting at column cols."""
    out = []
    for w in widths:
        out.append(buf[:, cols:cols + w].view(B, S_l, w))
        cols += w
    return out


def row_bytes(t):
    """t [B, T, ...] as a [B, T, row bytes] uint8 tensor (a copy only where t is a strided view)."""
    t = t.contiguous()
    return t.view(torch.uint8).reshape(t.shape[0], t.shape[1], -1)


def first_of(bad):
    """(b, token, column) of the first True of a [B, T, X] mask, and how many are True."""
    _, T, X = bad.shape
    i = int(torch.argmax(bad.reshape(-1).to(torch.uint8)))
    return (i // (T * X), i // X % T, i % X), int(bad.sum())


def check_bytes(got, want, what):
    """got and want [B, T, ...] of any dtype hold the same bytes; else the count and the first differing (b, token, byte)."""
    g, w = row_bytes(got), row_bytes(want).to(got.device)
    assert g.shape == w.shape, f"{what}: shape {tuple(g.shape)} vs {tuple(w.shape)}"
    if torch.equal(g, w):
        return
    (b, t, x), nbad = first_of(g != w)
    raise AssertionError(f"{what}: {nbad} bytes differ, the first at b {b} token {t} byte {x}: got {int(g[b, t, x]):#04x}, "
                         f"want {int(w[b, t, x]):#04x}")


def check_values(got, want, what):
    """A reduce-scatter output [B, T, ...]: the bits of want, NaN compared by position; else the count and the first (b, token, element)."""
    iv = R.INT_VIEW[R.esize(got.dtype)]
    g = got.contiguous().reshape(got.shape[0], got.shape[1], -1)
    w = want.to(got.device).contiguous().reshape(g.shape)
    ok = (g.view(iv) == w.view(iv)) | (torch.isnan(g) & torch.isnan(w))
    if bool(ok.all()):
        return
    (b, t, x), nbad = first_of(~ok)
    raise AssertionError(f"{what}: {nbad} elements differ, the first at b {b} token {t} element {x}: got {g[b, t, x].item()!r} "
                         f"(bits {int(g[b, t, x].view(iv)):#x}), want {w[b, t, x].item()!r} (bits {int(w[b, t, x].view(iv)):#x})")


def check_poisoned(t, what):
    bad = t.view(torch.uint8) != POISON
    if bool(bad.any()):
        raise AssertionError(f"{what}: {int(bad.sum())} bytes written that must stay poisoned")


# ------------------------------------------------------------------------------------------------- one call of each family, checked
def ulysses_case(g, B, S_l, heads, D, dt, seed, what, packed=True, back=None):
    """seq -> heads of up to three tensors (column slices of one packed QKV per rank, or dense), against the reference on the device;
    then heads -> seq of the tensors in `back` (default: q, and every non-replicated one when not packed) into column slices of a packed
    buffer laid out as the source, whose other columns must stay poisoned."""
    n = g.n
    es = R.esize(dt)
    cols = [0]
    for h in heads:
        cols.append(cols[-1] + h * D)
    arena = Arena(g)
    try:
        xs = []
        for r in range(n):
            if packed:
                qkv = random_bytes((B * S_l, cols[-1]), dt, seed + r, dev_of(g, r))
                xs.append([qkv[:, cols[i]:cols[i + 1]].view(B, S_l, h, D) for i, h in enumerate(heads)])
            else:
                xs.append([random_bytes((B, S_l, h, D), dt, seed + 7 * r + i, dev_of(g, r)) for i, h in enumerate(heads)])
        ys = [[arena(r, (B, n * S_l, uref.local_heads(n, h), D), dt) for h in heads] for r in range(n)]
        poison([y for row in ys for y in row])
        g.run(lambda r, c, st: c.all_to_all_seq_to_heads(xs[r], ys[r], stream=st))
        what = f"{what} n={n} B={B} S_l={S_l} heads={heads} D={D} {dt} packed={packed}"
        for i in range(len(heads)):
            want = uref.seq_to_heads([xs[s][i].to(dev_of(g, 0)) for s in range(n)])
            for r in range(n):
                check_bytes(ys[r][i], want[r], f"{what}: seq->heads tensor {i} rank {r}")
            del want
        if back is None:
            back = [0] if packed else [i for i, h in enumerate(heads) if h % n == 0]
        assert all(heads[i] % n == 0 for i in back)
        bufs = [arena(r, (B * S_l, cols[-1]), dt) for r in range(n)]
        poison(bufs)
        outs = [[bufs[r][:, cols[i]:cols[i + 1]].view(B, S_l, heads[i], D) for i in back] for r in range(n)]
        g.run(lambda r, c, st: c.all_to_all_heads_to_seq([ys[r][i] for i in back], outs[r], stream=st))
        for r in range(n):
            for k, i in enumerate(back):
                check_bytes(outs[r][k], xs[r][i], f"{what}: heads->seq tensor {i} rank {r}")
            for i in range(len(heads)):
                if i not in back:
                    check_poisoned(bufs[r][:, cols[i]:cols[i + 1]], f"{what}: heads->seq rank {r}, columns of tensor {i}")
        return B * S_l * sum(heads) * D * es // 16
    finally:
        arena.release()


def fill_sum_inputs(fulls, dt, seed):
    """fulls[r][i]: rank r's tensor i, filled with coll_fp_reference.gen_inputs data GEN_BLOCK elements at a time."""
    n = len(fulls)
    for i in range(len(fulls[0])):
        flat = [f[i].view(-1) for f in fulls]
        for k, lo in enumerate(range(0, flat[0].numel(), GEN_BLOCK)):
            hi = min(flat[0].numel(), lo + GEN_BLOCK)
            xs = R.gen_inputs(n, hi - lo, dt, seed + 1009 * i + k, device=flat[0].device)
            for r in range(n):
                flat[r][lo:hi].copy_(xs[r])


def cp_case(g, B, S_l, widths, q_cols, chunks, seed, what, gather_dt=BF16, rs_dt=BF16):
    """all_gather_context of the tensors (column slices after q_cols Q columns of one packed QKV per rank, or dense when q_cols is None)
    against the reference on every rank; then reduce_scatter_context of gen_inputs fulls into a packed dQKV laid out the same way, whose
    Q columns must stay poisoned (or into dense shards). A dtype of None leaves that direction out."""
    n, S = g.n, g.n * S_l
    what = f"{what} n={n} B={B} S_l={S_l} widths={widths} q_cols={q_cols} chunks={chunks}"
    arena = Arena(g)

    def shards_of(r, dt, gen_seed):
        """Rank r's shards and the packed buffer they are slices of (none when dense); random bytes, or uninitialised (gen_seed None)."""
        if q_cols is None:
            if gen_seed is None:
                return [torch.empty(B, S_l, w, dtype=dt, device=dev_of(g, r)) for w in widths], []
            return [random_bytes((B, S_l, w), dt, gen_seed + 7 * r + i, dev_of(g, r)) for i, w in enumerate(widths)], []
        if gen_seed is None:
            buf = torch.empty(B * S_l, q_cols + sum(widths), dtype=dt, device=dev_of(g, r))
        else:
            buf = random_bytes((B * S_l, q_cols + sum(widths)), dt, gen_seed + r, dev_of(g, r))
        return packed_views(buf, B, S_l, q_cols, widths), [buf]

    try:
        if gather_dt is not None:
            shards = [shards_of(r, gather_dt, seed)[0] for r in range(n)]
            fulls = [[arena(r, (B, S, w), gather_dt) for w in widths] for r in range(n)]
            poison([f for row in fulls for f in row])
            g.run(lambda r, c, st: c.all_gather_context(shards[r], fulls[r], chunks=chunks, stream=st))
            for i in range(len(widths)):
                want = cref.all_gather([shards[s][i].to(dev_of(g, 0)) for s in range(n)], chunks)
                for r in range(n):
                    check_bytes(fulls[r][i], want, f"{what} {gather_dt}: gather tensor {i} rank {r}")
                del want
            del shards, fulls
            arena.release()
        if rs_dt is not None:
            fulls = [[arena(r, (B, S, w), rs_dt) for w in widths] for r in range(n)]
            fill_sum_inputs(fulls, rs_dt, seed)
            outs, whole = zip(*[shards_of(r, rs_dt, None) for r in range(n)])
            poison([t for row in (whole if q_cols is not None else outs) for t in row])
            g.run(lambda r, c, st: c.reduce_scatter_context(fulls[r], outs[r], chunks=chunks, stream=st))
            for i in range(len(widths)):
                want = cref.reduce_scatter([fulls[s][i].to(dev_of(g, 0)) for s in range(n)], chunks)
                for r in range(n):
                    check_values(outs[r][i], want[r], f"{what} {rs_dt}: reduce-scatter tensor {i} rank {r}")
                del want
            if q_cols is not None:
                for r in range(n):
                    check_poisoned(whole[r][0][:, :q_cols], f"{what}: rank {r}'s Q columns of dQKV")
        return B * S_l * sum(widths)
    finally:
        arena.release()


# ------------------------------------------------------------------------------------------------- the device references
def test_device_references_match_cpu_and_formula_loops(torch_cuda):
    """The references below run on device tensors; at a small shape their device run equals their CPU run and the per-element loops
    that render the header's formulas."""
    n, B, S_l, D = 4, 2, 6, 16
    for heads in ((8, 4, 2), (4, 1)):
        xs = [random_bytes((B, S_l, h, D), BF16, 10 * r + h, "cpu") for r in range(n) for h in heads]
        for i, h in enumerate(heads):
            per = [xs[r * len(heads) + i] for r in range(n)]
            cpu = uref.seq_to_heads(per)
            dev = uref.seq_to_heads([x.cuda() for x in per])
            loop = uref.seq_to_heads_loop(per)
            for r in range(n):
                assert torch.equal(dev[r].cpu(), cpu[r]) and torch.equal(cpu[r], loop[r]), (heads, i, r)
            if h % n == 0:
                ys = [y.view(BF16).view(B, n * S_l, h // n, D) for y in cpu]
                back_dev = uref.heads_to_seq([y.cuda() for y in ys])
                back_loop = uref.heads_to_seq_loop(ys)
                for r in range(n):
                    assert torch.equal(back_dev[r].cpu(), back_loop[r]), (heads, i, r)
    for chunks in (1, 2):
        shards = [random_bytes((B, S_l, 24), BF16, 50 + r, "cpu") for r in range(n)]
        cpu = cref.all_gather(shards, chunks)
        assert torch.equal(cref.all_gather([x.cuda() for x in shards], chunks).cpu(), cpu)
        assert torch.equal(cpu, cref.all_gather_loop(shards, chunks))
        for dt in (BF16, torch.float16, torch.float32):
            fulls = [x.view(B, n * S_l, 8) for x in R.gen_inputs(n, B * n * S_l * 8, dt, seed=60 + chunks, device="cpu")]
            cpu = cref.reduce_scatter(fulls, chunks)
            dev = cref.reduce_scatter([f.cuda() for f in fulls], chunks)
            loop = cref.reduce_scatter_loop(fulls, chunks)
            for r in range(n):
                R.assert_same(dev[r].cpu(), cpu[r], f"device vs CPU {dt} chunks={chunks} rank {r}")
                R.assert_same(cpu[r], loop[r], f"CPU vs loop {dt} chunks={chunks} rank {r}")


# ------------------------------------------------------------------------------------------------- a. model shapes
# (name, Hq, Hkv, the rank counts it runs at); D = 128
ULYSSES_MODELS = [("llama3-8b", 32, 8, (2, 4, 8)), ("llama3-70b", 64, 8, (2, 4, 8)), ("mha", 32, 32, (2, 4, 8)), ("mqa", 64, 1, (2, 4, 8)),
                  ("gqa-replicated", 64, 4, (8,))]
# (name, Q columns of the packed QKV or None for dense tensors, widths)
CP_MODELS = [("llama3-8b", 32 * D_MODEL, (8 * D_MODEL, 8 * D_MODEL)), ("llama3-70b", 64 * D_MODEL, (8 * D_MODEL, 8 * D_MODEL)),
             ("mla", None, (512, 64))]


def ulysses_arena_bytes(n, S, heads, D, es):
    """The seq -> heads outputs and the packed heads -> seq buffer of one rank."""
    return sum(S * uref.local_heads(n, h) * D * es for h in heads) + S // n * sum(heads) * D * es + 4096


@pytest.mark.parametrize("n", [2, 4, 8])
def test_ulysses_at_model_shapes(torch_cuda, coll_mod, n):
    """q, k and v as column slices of one packed QKV, seq -> heads, then q back into a packed buffer, at 32k and 128k tokens."""
    models = [m for m in ULYSSES_MODELS if n in m[3]]
    need = max(ulysses_arena_bytes(n, S, (hq, hkv, hkv), D_MODEL, 2) for _, hq, hkv, _ in models for S in SEQ)
    with make_group(coll_mod, n, need) as g:
        for name, hq, hkv, _ in models:
            for S in SEQ:
                ulysses_case(g, 1, S // n, (hq, hkv, hkv), D_MODEL, BF16, seed=S + hq + hkv + n, what=f"{name} S={S}")


@pytest.mark.parametrize("n", [2, 4, 8])
def test_context_at_model_shapes(torch_cuda, coll_mod, n):
    """K and V of Llama-3-8B and -70B as slices of a packed QKV and the MLA pair as dense tensors: the load-balanced gather, then the
    reduce-scatter into a packed dQKV, at 32k and 128k tokens; at n = 4 also an e4m3 gather and an fp32 reduce-scatter at 128k."""
    need = 131072 * 2 * D_MODEL * 8 * 4 + 4096
    with make_group(coll_mod, n, need) as g:
        for name, q_cols, widths in CP_MODELS:
            for S in SEQ:
                cp_case(g, 1, S // n, widths, q_cols, 2, seed=S + n + len(name), what=f"{name} S={S}")
        if n == 4:
            cp_case(g, 1, 131072 // n, CP_MODELS[0][2], CP_MODELS[0][1], 2, seed=77, what="llama3-8b S=131072",
                    gather_dt=torch.float8_e4m3fn, rs_dt=torch.float32)


def test_fused_equals_the_unfused_composition_at_llama3_70b(torch_cuda, coll_mod):
    """Llama-3-70B (Hq 64, Hkv 8, D 128), 128k tokens, 8 ranks: each fused call equals, byte for byte, the composition that
    bench/ulysses_a2a_perf.py and bench/context_kv_perf.py time it against. Ulysses: a permute copy and comm.all_to_all per tensor, a
    permute back; for heads -> seq, comm.all_to_all of the head shard and a permute into the packed buffer. Context: a dense copy of
    the K or V slice, comm.all_gather and an index_select into token order; for the gradient, an index_select into rank-chunk order and
    comm.reduce_scatter. That reduce-scatter sums in another rank order, so its gradients are multiples of 1/8 below 8 in magnitude:
    every fp32 sum of 8 of them is exact, and both round the same sum once."""
    n, S, hq, hkv, D, dt = 8, 131072, 64, 8, D_MODEL, BF16
    S_l, B = S // n, 1
    heads, W = (hq, hkv, hkv), hkv * D
    cols = [0, hq * D, (hq + hkv) * D, (hq + 2 * hkv) * D]
    per_rank = ulysses_arena_bytes(n, S, heads, D, 2) + 2 * S_l * hq * D * 2
    with make_group(coll_mod, n, max(per_rank, 3 * S * W * 2 + S_l * W * 2) + (64 << 20)) as g:
        arena = Arena(g)
        qkv = [random_bytes((B * S_l, cols[-1]), dt, 900 + r, dev_of(g, r)) for r in range(n)]
        xs = [[q[:, cols[i]:cols[i + 1]].view(B, S_l, h, D) for i, h in enumerate(heads)] for q in qkv]
        try:
            ys = [[arena(r, (B, S, 1 if i else hq // n, D), dt) for i in range(3)] for r in range(n)]
            poison([y for row in ys for y in row])
            g.run(lambda r, c, st: c.all_to_all_seq_to_heads(xs[r], ys[r], stream=st))
            for i, h in enumerate(heads):
                hl = h // n
                send = [arena(r, (n, B, S_l, hl, D), dt) for r in range(n)]
                recv = [arena(r, (n, B, S_l, hl, D), dt) for r in range(n)]
                for r in range(n):
                    send[r].copy_(xs[r][i].reshape(B, S_l, n, hl, D).permute(2, 0, 1, 3, 4))
                g.run(lambda r, c, st: c.all_to_all(send[r].view(-1), recv[r].view(-1), stream=st))
                for r in range(n):
                    check_bytes(ys[r][i], recv[r].permute(1, 0, 2, 3, 4).reshape(B, S, hl, D), f"seq->heads tensor {i} rank {r} vs the composition")
                arena.free(send + recv)
            back = [arena(r, (B * S_l, cols[-1]), dt) for r in range(n)]
            poison(back)
            outs = [[b[:, :hq * D].view(B, S_l, hq, D)] for b in back]
            g.run(lambda r, c, st: c.all_to_all_heads_to_seq([ys[r][0]], outs[r], stream=st))
            recv = [arena(r, (n, B, S_l, hq // n, D), dt) for r in range(n)]
            g.run(lambda r, c, st: c.all_to_all(ys[r][0].view(-1), recv[r].view(-1), stream=st))
            for r in range(n):
                check_bytes(outs[r][0], recv[r].permute(1, 2, 0, 3, 4).reshape(B, S_l, hq, D), f"heads->seq rank {r} vs the composition")
                check_poisoned(back[r][:, hq * D:], f"heads->seq rank {r}, K and V columns")
        finally:
            arena.release()
        del ys, back, outs, recv
        kv = [[q[:, cols[1 + i]:cols[2 + i]].view(B, S_l, W) for i in range(2)] for q in qkv]
        idx = cref.token_index(n, 2, S_l, dev_of(g, 0))
        try:
            fulls = [[arena(r, (B, S, W), dt) for _ in range(2)] for r in range(n)]
            poison([f for row in fulls for f in row])
            g.run(lambda r, c, st: c.all_gather_context(kv[r], fulls[r], chunks=2, stream=st))
            for i in range(2):
                send = [arena(r, (B, S_l, W), dt) for r in range(n)]
                recv = [arena(r, (n, B, S_l, W), dt) for r in range(n)]
                for r in range(n):
                    send[r].copy_(kv[r][i])
                g.run(lambda r, c, st: c.all_gather(send[r].view(-1), recv[r].view(-1), stream=st))
                for r in range(n):
                    composed = recv[r].permute(1, 0, 2, 3).reshape(B, S, W).index_select(1, idx)
                    check_bytes(fulls[r][i], composed, f"gather tensor {i} rank {r} vs the composition")
                del composed
                arena.free(send + recv)
        finally:
            arena.release()
        del fulls
        inv = torch.empty_like(idx)
        inv[idx] = torch.arange(S, device=idx.device)
        try:
            grads = [[arena(r, (B, S, W), dt) for _ in range(2)] for r in range(n)]
            gen = torch.Generator(device=dev_of(g, 0)).manual_seed(901)
            for row in grads:
                for t in row:
                    t.copy_(torch.randint(-63, 64, t.shape, generator=gen, device=t.device).to(torch.float32).div_(8))
            dq = [torch.empty(B * S_l, cols[-1], dtype=dt, device=dev_of(g, r)) for r in range(n)]
            poison(dq)
            dkv = [[b[:, cols[1 + i]:cols[2 + i]].view(B, S_l, W) for i in range(2)] for b in dq]
            g.run(lambda r, c, st: c.reduce_scatter_context(grads[r], dkv[r], chunks=2, stream=st))
            for i in range(2):
                rs_in = [arena(r, (n, B, S_l, W), dt) for r in range(n)]
                rs_out = [arena(r, (B, S_l, W), dt) for r in range(n)]
                for r in range(n):
                    torch.index_select(grads[r][i], 1, inv, out=rs_in[r].view(B, S, W))
                g.run(lambda r, c, st: c.reduce_scatter(rs_in[r].view(-1), rs_out[r].view(-1), stream=st))
                for r in range(n):
                    check_bytes(dkv[r][i], rs_out[r], f"reduce-scatter tensor {i} rank {r} vs the composition")
                arena.free(rs_in + rs_out)
            for r in range(n):
                check_poisoned(dq[r][:, :hq * D], f"rank {r}'s Q columns of dQKV")
        finally:
            arena.release()


# ------------------------------------------------------------------------------------------------- b. awkward geometry
@pytest.mark.parametrize("D", [64, 80, 96, 112, 192, 256])
def test_ulysses_awkward_geometry(torch_cuda, coll_mod, D):
    """bf16 head sizes whose one-head segments are 8 to 32 vectors (FastDiv by 10, 12 and 14 among them), at an odd, non-power-of-two
    shard of 12289 tokens, at B = 3 with 4099 tokens, and at 3 and 6 ranks; MHA, GQA, replicated GQA and MQA; packed and dense."""
    cases = [(4, 1, 12289, (4, 2, 1), True), (3, 3, 4099, (6, 3, 1), False), (6, 2, 1031, (12, 6, 2), True), (4, 3, 2 * 4099, (8, 4, 4), False)]
    need = max(ulysses_arena_bytes(n, n * B * S_l, heads, D, 2) for n, B, S_l, heads, _ in cases)
    for n, B, S_l, heads, packed in cases:
        with make_group(coll_mod, n, need) as g:
            ulysses_case(g, B, S_l, heads, D, BF16, seed=D + n, what="awkward", packed=packed)


# (n, B, S_l, widths in bf16 elements, Q columns or None, chunks)
CP_AWKWARD = [(3, 1, 12289, (512, 64), None, 1),
              (6, 3, 2 * 4099, (512, 64), None, 2),
              (3, 3, 2 * 4099, (56, 24, 40), 128, 2),
              (6, 1, 12289, (80, 96, 112), 256, 1),
              (3, 1, 12289, (1024, 1024), 4096, 1)]


@pytest.mark.parametrize("case", range(len(CP_AWKWARD)))
def test_context_awkward_geometry(torch_cuda, coll_mod, case):
    """3 and 6 ranks, an odd 12289-token shard with chunks = 1, B = 3 with chunks = 2 and S_l = 2 * 4099 (the second chunk far from the
    first: tok1 - tok0 = (2N - 2 - 2 me) * 4099), the MLA widths 64 and 8 vectors in one call, and three tensors of 7, 3 and 5 (10, 12
    and 14) vectors whose prefix boundaries fall inside an unroll group; gather in bf16, reduce-scatter in bf16, fp16 and fp32."""
    n, B, S_l, widths, q_cols, chunks = CP_AWKWARD[case]
    for k in range(1, len(widths)):
        pre = B * S_l * sum(widths[:k]) * 2 // 16
        assert pre % 512, f"the prefix boundary {pre} starts a thread's part of an unroll group"
    with make_group(coll_mod, n, B * n * S_l * sum(widths) * 4 + 4096) as g:
        cp_case(g, B, S_l, widths, q_cols, chunks, seed=300 + case, what="awkward")
        cp_case(g, B, S_l, widths, q_cols, chunks, seed=310 + case, what="awkward", gather_dt=None, rs_dt=(torch.float16, torch.float32)[case % 2])


# ------------------------------------------------------------------------------------------------- c. launch shapes
# ("max_ctas", m) on every rank, or ("p2p", max_ctas, threads) pinned; threads 512 where not pinned (a few MiB per rank never fits fewer)
LAUNCH = [("default",), ("max_ctas", 1), ("max_ctas", 3)] + [("p2p", m, t) for m in (1, 2) for t in (128, 256, 512)]


def rows_for(target, wsum, modulus, residue):
    """The smallest row count >= target with rows * wsum = residue (mod modulus); wsum odd, modulus a power of two."""
    want = residue * pow(wsum, -1, modulus) % modulus
    return target + (want - target) % modulus


def default_ctas(g):
    c = g.comms[0]
    return max(1, c.sm_count // sum(d.device == c.device for d in g.comms))


@pytest.mark.parametrize("shape", LAUNCH, ids=lambda s: "-".join(map(str, s)))
def test_launch_shapes(torch_cuda, coll_mod, shape):
    """Both families under one to three CTAs and pinned thread counts, set the same on every rank: totals (16-byte vectors per rank) of
    1, threads and 4 * threads - 1 modulo 4 * threads, so the last pass of the grid-stride loop ends with a partial unroll group (or one
    lone vector). Ulysses: 3 ranks, heads (9, 3, 3) of D = 40 (5 vectors); context: 3 ranks, widths of 7, 3 and 1 vectors, load-balanced
    chunks where the row count is even."""
    n = 3
    threads = shape[2] if shape[0] == "p2p" else 512
    M = 4 * threads
    uly_heads, D, cp_widths = (9, 3, 3), 40, (56, 24, 8)
    uly_w, cp_w = sum(uly_heads) * D * 2 // 16, sum(cp_widths) * 2 // 16
    with make_group(coll_mod, n, 64 << 20) as g:
        try:
            for c in g.comms:
                if shape[0] == "max_ctas":
                    c.set_max_ctas(shape[1])
                elif shape[0] == "p2p":
                    c.set_launch_shape("p2p", shape[1], shape[2])
            for k, residue in enumerate((1, threads, M - 1)):
                rows = rows_for((1 << 18) // uly_w, uly_w, M, residue)
                assert ulysses_case(g, 1, rows, uly_heads, D, BF16, seed=40 + k, what=f"launch {shape}", packed=k != 1, back=[0, 1, 2]) % M == residue
                rows = rows_for((1 << 18) // cp_w, cp_w, M, residue)
                chunks = 2 if rows % 2 == 0 else 1
                got = cp_case(g, 1, rows, cp_widths, 64 if k != 1 else None, chunks, seed=50 + k, what=f"launch {shape}")
                assert got * 2 // 16 % M == residue
        finally:
            for c in g.comms:
                c.set_max_ctas(default_ctas(g))
                c.set_launch_shape("p2p", 0, 0)


# ------------------------------------------------------------------------------------------------- d. past 4 GiB
GIB = 1 << 30
SLICE = 1 << 16                 # tokens per slice of the comparisons (and per generated source block)


def skip_unless_free(need, what):
    free, total = torch.cuda.mem_get_info(0)
    print(f"{what}: {need / GIB:.2f} GiB needed, {free / GIB:.1f} GiB free of {total / GIB:.1f} GiB")
    if free < need:
        pytest.skip(f"{what}: needs {need / GIB:.2f} GiB of device memory, {free / GIB:.1f} GiB free")
    torch.cuda.reset_peak_memory_stats(0)


def report_peak(what, n, arena_bytes):
    """The device memory the test used: every rank's arena (as make_group sizes it), and torch's peak (sources, shards and comparison
    temporaries)."""
    arenas = n * (arena_bytes // (1 << 20) + 64) / 1024
    peak = torch.cuda.max_memory_allocated(0) / GIB
    print(f"{what}: peak {arenas + peak:.2f} GiB of device memory: arenas {arenas:.2f} GiB + torch {peak:.2f} GiB")


def test_context_full_past_4_gib(torch_cuda, coll_mod):
    """2 ranks, one bf16 tensor of width 1024 (128 vectors), S_l = 1 179 648, chunks = 2: each shard is 2.25 GiB and each full 4.5 GiB,
    so the arena offset of the upper half of the full (16 * full_v) is past 2^32. The gather is checked slice by slice against the
    shards; then the reduce-scatter of the gathered fulls into the shards, against ref_sum of the fulls' slices."""
    n, B, S_l, W, chunks = 2, 1, 1179648, 1024, 2
    S, c_tok = n * S_l, S_l // chunks
    full_bytes, shard_bytes = B * S * W * 2, B * S_l * W * 2
    assert full_bytes > (4 << 30) and c_tok % SLICE == 0
    need = n * (full_bytes + (64 << 20)) + n * shard_bytes + 8 * SLICE * W * 4
    skip_unless_free(need, "context past 4 GiB")
    with make_group(coll_mod, n, full_bytes) as g:
        arena = Arena(g)
        try:
            fulls = [arena(r, (B, S, W), BF16) for r in range(n)]
            poison(fulls)
            shards = [torch.empty(B, S_l, W, dtype=BF16, device="cuda:0") for _ in range(n)]
            for r in range(n):
                for k, lo in enumerate(range(0, S_l, SLICE)):
                    shards[r][:, lo:lo + SLICE].copy_(random_bytes((B, SLICE, W), BF16, 1000 * r + k, "cuda:0"))
            g.run(lambda r, c, st: c.all_gather_context([shards[r]], [fulls[r]], chunks=chunks, stream=st))
            for j in range(2 * n):                                  # global chunk j is chunk k of rank s
                s, k = (j, 0) if j < n else (2 * n - 1 - j, 1)
                for u in range(0, c_tok, SLICE):
                    want = shards[s][:, k * c_tok + u:k * c_tok + u + SLICE]
                    for r in range(n):
                        check_bytes(fulls[r][:, j * c_tok + u:j * c_tok + u + SLICE], want,
                                    f"gather rank {r} tokens from {j * c_tok + u} (byte offset {(j * c_tok + u) * W * 2:#x})")
            poison(shards)
            g.run(lambda r, c, st: c.reduce_scatter_context([fulls[r]], [shards[r]], chunks=chunks, stream=st))
            for r in range(n):
                for t in range(0, S_l, SLICE):
                    gt = cref.gtok(n, chunks, S_l, r, t)
                    xs = [f[:, gt:gt + SLICE].reshape(-1) for f in fulls]
                    want = R.cast(R.ref_sum(xs, list(range(n))), BF16).view(B, SLICE, W)
                    check_values(shards[r][:, t:t + SLICE], want, f"reduce-scatter rank {r} tokens from {t} (full token {gt})")
            report_peak("context past 4 GiB", n, full_bytes)
        finally:
            arena.release()


def test_ulysses_both_sides_past_4_gib(torch_cuda, coll_mod):
    """2 ranks, one bf16 tensor of 16 heads of 128, S_l = 2^20 + 2^16: the sequence side and the head side of each rank are 4.25 GiB.
    seq -> heads, then heads -> seq back into the (poisoned) sources. Sources are generated per block of tokens from a seeded generator
    and generated again for each comparison, so only the call's own buffers are kept."""
    n, B, S_l, H, D = 2, 1, (1 << 20) + (1 << 16), 16, 128
    hl, row = H // n, H * D * 2
    side = B * S_l * row
    assert side > (4 << 30) and S_l % SLICE == 0
    need = n * (2 * side + (64 << 20)) + 6 * SLICE * row
    skip_unless_free(need, "Ulysses past 4 GiB")

    def block(r, k):
        return random_bytes((B, SLICE, H, D), BF16, 5000 + 100 * r + k, "cuda:0")

    with make_group(coll_mod, n, 2 * side) as g:
        arena = Arena(g)
        try:
            xs = [arena(r, (B, S_l, H, D), BF16) for r in range(n)]
            ys = [arena(r, (B, n * S_l, hl, D), BF16) for r in range(n)]
            for r in range(n):
                for k in range(S_l // SLICE):
                    xs[r][:, k * SLICE:(k + 1) * SLICE].copy_(block(r, k))
            poison(ys)
            g.run(lambda r, c, st: c.all_to_all_seq_to_heads([xs[r]], [ys[r]], stream=st))
            for s in range(n):
                for k in range(S_l // SLICE):
                    x = block(s, k)
                    for r in range(n):
                        tok = s * S_l + k * SLICE
                        check_bytes(ys[r][:, tok:tok + SLICE], x[:, :, r * hl:(r + 1) * hl],
                                    f"seq->heads rank {r} tokens from {tok} (byte offset {tok * hl * D * 2:#x})")
            poison(xs)
            g.run(lambda r, c, st: c.all_to_all_heads_to_seq([ys[r]], [xs[r]], stream=st))
            for r in range(n):
                for k in range(S_l // SLICE):
                    check_bytes(xs[r][:, k * SLICE:(k + 1) * SLICE], block(r, k),
                                f"heads->seq rank {r} tokens from {k * SLICE} (byte offset {k * SLICE * row:#x})")
            report_peak("Ulysses past 4 GiB", n, 2 * side)
        finally:
            arena.release()


# ------------------------------------------------------------------------------------------------- e. real devices
def test_on_real_devices(torch_cuda, coll_mod):
    """One rank per GPU: the grid is the communicator's full CTA count instead of SMs / N, so the grid-stride loops take other strides,
    and stores and loads cross NVLink. Llama-3-8B through Ulysses and context parallelism at 32k tokens."""
    n = min(torch_cuda.cuda.device_count(), 8)
    if n < 2:
        pytest.skip(f"needs >= 2 GPUs, {n} present")
    S = 32768
    with make_group(coll_mod, n, ulysses_arena_bytes(n, S, (32, 8, 8), D_MODEL, 2) + S * 2048 * 2, devices=list(range(n))) as g:
        ulysses_case(g, 1, S // n, (32, 8, 8), D_MODEL, BF16, seed=70, what="real devices llama3-8b")
        cp_case(g, 1, S // n, CP_MODELS[0][2], CP_MODELS[0][1], 2, seed=71, what="real devices llama3-8b")
