"""The launch plan of the one-rank copy-engine copy (collectives.cu plan_copy, through the b200collDebugPlanCopy hook; no GPU needed):
chunks in whole 128-byte lines that fit a ring slot, dealt round-robin in whole rounds so that every CTA moves the same number of chunks
give or take one, and a grid that never exceeds what is resident at once, which is what makes launching it with programmatic dependent
launch safe."""
import ctypes as C

import pytest

KIB, MIB = 1 << 10, 1 << 20


def plan(lib_path, nbytes, sm_count):
    L = C.CDLL(lib_path)
    blocks, chunk, rounds, resident = C.c_int(), C.c_uint(), C.c_uint(), C.c_int()
    rc = L.b200collDebugPlanCopy(C.c_size_t(nbytes), sm_count, C.byref(blocks), C.byref(chunk), C.byref(rounds), C.byref(resident))
    return rc, blocks.value, chunk.value, rounds.value, resident.value


def boundary_sizes(sm_count):
    cap = 2 * sm_count
    return sorted({MIB, MIB + 16, 12 * MIB + 592,                              # the threshold, one vector past it, a short last chunk
                   cap * 4 * KIB - 16, cap * 4 * KIB, cap * 4 * KIB + 16,      # the grid stops growing
                   cap * 16 * KIB - 16, cap * 16 * KIB, cap * 16 * KIB + 16,   # a second round begins
                   64 * MIB, 64 * MIB + 48, 256 * MIB, 1 << 30, (1 << 34) + 16, 16, 4 * KIB + 16})


@pytest.mark.parametrize("sm_count", [132, 114, 8, 1])
def test_plan_deals_line_aligned_chunks_in_whole_rounds_within_resident_capacity(coll_lib, sm_count):
    for nbytes in boundary_sizes(sm_count):
        rc, blocks, chunk, rounds, resident = plan(coll_lib, nbytes, sm_count)
        assert rc == 0 and resident == 2 * sm_count
        assert 1 <= blocks <= resident, (nbytes, blocks)
        assert chunk % 128 == 0 and 128 <= chunk <= 16 * KIB, (nbytes, chunk)     # every chunk but the last starts and ends on a line
        nchunks = -(-nbytes // chunk)                   # chunk i covers [i * chunk, min(bytes, (i + 1) * chunk)): every byte once
        assert (nchunks - 1) * chunk < nbytes <= nchunks * chunk
        # CTA b takes chunks b, b + blocks, ...: no CTA is idle, none moves more than `rounds`, and the last round is (nearly) full
        assert blocks <= nchunks <= blocks * rounds, (nbytes, blocks, rounds, nchunks)
        assert blocks * rounds - nchunks <= blocks * rounds // 32 + 1, (nbytes, blocks, rounds, nchunks)
        if nbytes >= resident * 16 * KIB:
            assert blocks == resident, (nbytes, blocks)                                # enough work: every resident slot is used


def test_plan_on_an_h100(coll_lib):
    # 132 SMs. 16 MiB: 264 CTAs, 4 rounds of 16000-byte chunks, 1049 of them (7 CTAs move 3). 16 KiB chunks dealt to 264 CTAs
    # would give 232 CTAs 4 chunks and 32 CTAs 3. From 256 MiB up the chunk is the ring slot again.
    assert plan(coll_lib, 16 * MIB, 132)[:4] == (0, 264, 16000, 4)
    assert -(-16 * MIB // 16000) == 1049
    assert plan(coll_lib, 1 << 30, 132)[:4] == (0, 264, 16 * KIB, 249)


def test_plan_rejects_bad_arguments(coll_lib):
    assert plan(coll_lib, MIB, 0)[0] != 0
    L = C.CDLL(coll_lib)
    assert L.b200collDebugPlanCopy(C.c_size_t(MIB), 132, None, None, None, None) != 0
