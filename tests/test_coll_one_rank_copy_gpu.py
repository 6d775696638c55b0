"""The one-rank copy-engine copy (k_copy_bulk) on an H100: bit-exact at the boundaries of its launch plan, into arena and plain
destinations, one launch per call; and ordered like any stream operation although it is launched with programmatic dependent launch —
a chain of copies each reading the previous output, a copy overwriting an earlier copy's source, and torch kernels in between."""
import ctypes as C

import pytest

pytestmark = pytest.mark.gpu

KIB, MIB = 1 << 10, 1 << 20


@pytest.fixture(scope="module")
def one_rank(coll_lib):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from container_engine_accelerators_b200.ops import coll
    coll.load()
    (c,) = coll.Comm.init_all([0], arena_mb=512, timeout_ms=60000)
    yield torch, coll, c
    torch.cuda.synchronize()
    c.destroy()


def random_bits(torch, nbytes, seed):
    """bf16 words with every bit pattern possible: NaN payloads, infinities, -0 and denormals included."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(-32768, 32768, (nbytes // 2,), generator=g, device="cuda", dtype=torch.int32).to(torch.int16).view(torch.bfloat16)


def same_bits(torch, a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def plan_sizes(coll_lib, sm_count):
    """Sizes at which the plan changes for this GPU: the threshold and one vector past it, where the grid stops growing, where a second
    round begins, and sizes whose last chunk is short."""
    L = C.CDLL(coll_lib)
    cap = 2 * sm_count
    sizes = {MIB, MIB + 16, cap * 4 * KIB - 16, cap * 4 * KIB + 16, cap * 16 * KIB, cap * 16 * KIB + 16, 12 * MIB + 592, 64 * MIB + 48}
    for s in sizes:
        blocks, chunk, rounds, resident = C.c_int(), C.c_uint(), C.c_uint(), C.c_int()
        assert L.b200collDebugPlanCopy(C.c_size_t(s), sm_count, C.byref(blocks), C.byref(chunk), C.byref(rounds), C.byref(resident)) == 0
        assert blocks.value <= resident.value
    return sorted(sizes)


def test_bit_exact_at_plan_boundaries_arena_and_plain(one_rank, coll_lib):
    torch, coll, c = one_rank
    for i, nbytes in enumerate(plan_sizes(coll_lib, c.sm_count)):
        src = c.empty(nbytes // 2, torch.bfloat16)
        src.copy_(random_bits(torch, nbytes, i))
        for where in ("arena", "plain"):
            dst = c.empty(nbytes // 2, torch.bfloat16) if where == "arena" else torch.empty(nbytes // 2, dtype=torch.bfloat16, device="cuda")
            dst.view(torch.int16).fill_(0x7FC1)
            s0 = c.stats()
            c.all_reduce(src, dst)
            torch.cuda.synchronize()
            s1 = c.stats()
            assert same_bits(torch, dst, src), (nbytes, where)
            assert (s1["bulk_launches"] - s0["bulk_launches"], s1["kernel_launches"] - s0["kernel_launches"]) == (1, 1), (nbytes, where)
            if where == "arena":
                c.release(dst)
        c.release(src)
    c.check_async_error()


def test_chain_of_copies_each_reading_the_previous_output(one_rank):
    torch, coll, c = one_rank
    nbytes = 24 * MIB + 16
    bufs = [c.empty(nbytes // 2, torch.bfloat16) for _ in range(6)]
    want = random_bits(torch, nbytes, 7)
    bufs[0].copy_(want)
    for b in bufs[1:]:
        b.zero_()
    torch.cuda.synchronize()
    for rep in range(3):               # back to back, no host synchronisation: every copy depends on the one before it
        for a, b in zip(bufs, bufs[1:]):
            c.all_reduce(a, b)
        c.all_reduce(bufs[-1], bufs[0])
    torch.cuda.synchronize()
    for b in bufs:
        assert same_bits(torch, b, want)
    # write after read: the second copy overwrites the first copy's source, which must already have been read in full
    other = random_bits(torch, nbytes, 8)
    bufs[2].copy_(other)
    torch.cuda.synchronize()
    c.all_reduce(bufs[0], bufs[1])
    c.all_reduce(bufs[2], bufs[0])
    torch.cuda.synchronize()
    assert same_bits(torch, bufs[1], want) and same_bits(torch, bufs[0], other)
    c.check_async_error()
    for b in bufs:
        c.release(b)


def test_torch_kernels_between_copies(one_rank):
    torch, coll, c = one_rank
    nbytes = 8 * MIB
    src = c.empty(nbytes // 2, torch.bfloat16)
    first, second = c.empty(nbytes // 2, torch.bfloat16), torch.empty(nbytes // 2, dtype=torch.bfloat16, device="cuda")
    orig = random_bits(torch, nbytes, 9)
    src.copy_(orig)
    torch.cuda.synchronize()
    for rep in range(4):
        c.all_reduce(src, first)
        src.view(torch.int16).bitwise_not_()          # a torch kernel rewrites the source between two copies
        c.all_reduce(src, second)
        checksum = first.view(torch.int16).to(torch.int64).sum()   # and one reads the first copy's output after the second copy
        torch.cuda.synchronize()
        assert same_bits(torch, first, orig) and same_bits(torch, second, src), rep
        assert checksum.item() == orig.view(torch.int16).to(torch.int64).sum().item(), rep
        orig = src.clone()
    c.check_async_error()
