"""ctypes binding for libb200coll (coll/lib/libb200coll.so) — the only thing PyTorch is used for here is
launching ranks and holding the synthetic buffers (BASELINE.json north-star: "PyTorch is only the harness").

The library is the transport-installer payload (reference role: gpudirect-rdma/nccl-rdma-installer.yaml:70-77);
this module is what a pod's Python code imports once the device plugin's Allocate has mounted it.
Fails loudly when the shared object is missing on a GPU box — there is no eager/PyTorch fallback.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from pathlib import Path
from typing import Optional

REPO_ROOT = Path(__file__).resolve().parents[2]
_LIB_CANDIDATES = [
    os.environ.get("B200COLL_LIB", ""),
    str(REPO_ROOT / "coll" / "lib" / "libb200coll.so"),
    "/usr/local/nvidia/lib64/libb200coll.so",   # where Allocate mounts the installer's drop
    "libb200coll.so",
]

# b200collResult_t
(SUCCESS, UNHANDLED_CUDA_ERROR, SYSTEM_ERROR, INTERNAL_ERROR, INVALID_ARGUMENT, INVALID_USAGE, REMOTE_ERROR, IN_PROGRESS, OUT_OF_MEMORY,
 NO_DRIVER) = range(10)
MAX_RANKS = 8

F32, F16, BF16, FP8_E4M3, I8, U8, I32, U32, I64, U64, F64, FP8_E5M2 = range(12)
SUM, AVG, PROD, MIN, MAX = range(5)
OP_ALLREDUCE, OP_ALLGATHER, OP_REDUCESCATTER, OP_ALLTOALL = 0, 1, 2, 3
ALGO_AUTO, ALGO_LL, ALGO_ONESHOT, ALGO_TWOSHOT, ALGO_NVLS, ALGO_COPY, ALGO_LL2 = range(7)
ALGO_NAMES = ["auto", "ll", "oneshot", "twoshot", "nvls", "copy", "ll2"]
DTYPE_SIZE = {F32: 4, F16: 2, BF16: 2, FP8_E4M3: 1, I8: 1, U8: 1, I32: 4, U32: 4, I64: 8, U64: 8, F64: 8, FP8_E5M2: 1}


class UniqueId(C.Structure):
    _fields_ = [("internal", C.c_char * 128)]


class Epilogue(C.Structure):
    _fields_ = [("in_dtype", C.c_int), ("out_dtype", C.c_int), ("scale", C.c_float)]


class BlockScale(C.Structure):
    _fields_ = [("scales", C.c_void_p), ("row_len", C.c_size_t), ("block_rows", C.c_int), ("block_cols", C.c_int)]


class UlyssesTensor(C.Structure):
    _fields_ = [("seq", C.c_void_p), ("row_stride", C.c_size_t), ("head", C.c_void_p), ("heads", C.c_int)]


class ContextTensor(C.Structure):
    _fields_ = [("shard", C.c_void_p), ("row_stride", C.c_size_t), ("full", C.c_void_p), ("width", C.c_size_t)]


class ShardTensor(C.Structure):
    _fields_ = [("shard", C.c_void_p), ("full", C.c_void_p), ("rows", C.c_size_t), ("width", C.c_size_t), ("shard_rows", C.c_size_t)]


class Config(C.Structure):
    _fields_ = [("arena_bytes", C.c_size_t), ("enable_nvls", C.c_int), ("max_ctas", C.c_int), ("timeout_ms", C.c_int), ("debug", C.c_int)]


class CommInfo(C.Structure):
    _fields_ = [("rank", C.c_int), ("nranks", C.c_int), ("device", C.c_int), ("nvls", C.c_int), ("p2p_ok", C.c_int),
                ("same_device_loopback", C.c_int), ("arena_bytes", C.c_size_t), ("arena_used", C.c_size_t), ("sm_count", C.c_int),
                ("driver_version", C.c_int)]


class Stats(C.Structure):
    _fields_ = [("calls", C.c_uint64 * 6), ("bytes", C.c_uint64 * 6), ("algo_calls", C.c_uint64 * 7), ("kernel_launches", C.c_uint64),
                ("staged_calls", C.c_uint64), ("p2p_sends", C.c_uint64), ("p2p_recvs", C.c_uint64), ("p2p_bytes", C.c_uint64),
                ("host_calls", C.c_uint64), ("host_bytes", C.c_uint64), ("host_zero_copy", C.c_uint64), ("host_pipelined", C.c_uint64), ("bulk_launches", C.c_uint64), ("generic_launches", C.c_uint64)]


class Fault(C.Structure):
    _fields_ = [("code", C.c_uint32), ("rank", C.c_uint32), ("peer", C.c_uint32), ("block", C.c_uint32), ("expected", C.c_uint32),
                ("observed", C.c_uint32), ("op", C.c_uint32), ("reserved", C.c_uint32)]


class B200CollError(RuntimeError):
    def __init__(self, code: int, what: str, detail: str):
        super().__init__(f"{what}: {detail}" if detail else what)
        self.code = code


_lib: Optional[C.CDLL] = None


def lib_path() -> Optional[str]:
    for cand in _LIB_CANDIDATES[:-1]:
        if cand and os.path.exists(cand):
            return cand
    return None


def load() -> C.CDLL:
    """dlopen the library once and declare prototypes."""
    global _lib
    if _lib is not None:
        return _lib
    last = None
    for cand in _LIB_CANDIDATES:
        if not cand:
            continue
        try:
            _lib = C.CDLL(cand, mode=C.RTLD_GLOBAL)
            break
        except OSError as e:   # keep looking
            last = e
    if _lib is None:
        raise ImportError(f"libb200coll.so not found (run `python -c 'import __graft_entry__ as g; g.build()'` or `make -C coll`): {last}")
    L = _lib
    vp, sz, ci = C.c_void_p, C.c_size_t, C.c_int
    L.b200collGetErrorString.restype = C.c_char_p; L.b200collGetErrorString.argtypes = [ci]
    L.b200collGetLastError.restype = C.c_char_p
    L.b200collGetVersion.restype = ci
    L.b200collConfigDefault.argtypes = [C.POINTER(Config)]
    L.b200collGetUniqueId.argtypes = [C.POINTER(UniqueId)]
    L.b200collUniqueIdFromString.argtypes = [C.c_char_p, C.POINTER(UniqueId)]
    L.b200collCommInitRank.argtypes = [C.POINTER(vp), ci, C.POINTER(UniqueId), ci, C.POINTER(Config)]
    L.b200collCommInitAll.argtypes = [C.POINTER(vp), ci, C.POINTER(ci), C.POINTER(Config)]
    L.b200collCommDestroy.argtypes = [vp]
    L.b200collCommSplit.argtypes = [vp, ci, ci, C.POINTER(vp), C.POINTER(Config)]
    L.b200collDebugSplitPlan.argtypes = [ci, ci, C.POINTER(ci), C.POINTER(ci), C.POINTER(ci), C.POINTER(ci)]
    L.b200collCommInfoGet.argtypes = [vp, C.POINTER(CommInfo)]
    L.b200collCommStatsGet.argtypes = [vp, C.POINTER(Stats)]
    L.b200collCommGetAsyncError.argtypes = [vp, C.POINTER(Fault)]
    L.b200collHostBarrier.argtypes = [vp]
    L.b200collMemAlloc.argtypes = [vp, C.POINTER(vp), sz]
    L.b200collMemFree.argtypes = [vp, vp]
    L.b200collIsSymmetric.argtypes = [vp, vp, sz]
    L.b200collSetAllocatorComm.argtypes = [vp]
    L.b200collTorchAlloc.argtypes = [sz, ci, vp]; L.b200collTorchAlloc.restype = vp
    L.b200collTorchFree.argtypes = [vp, sz, ci, vp]; L.b200collTorchFree.restype = None
    L.b200collAllReduce.argtypes = [vp, vp, sz, C.POINTER(Epilogue), ci, vp, vp]
    L.b200collAllGather.argtypes = [vp, vp, sz, C.POINTER(Epilogue), vp, vp]
    L.b200collReduceScatter.argtypes = [vp, vp, sz, C.POINTER(Epilogue), ci, vp, vp]
    L.b200collAllToAll.argtypes = [vp, vp, sz, C.POINTER(Epilogue), vp, vp]
    L.b200collAllToAllv.argtypes = [vp, vp, sz, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(Epilogue), vp, vp]
    L.b200collBroadcast.argtypes = [vp, vp, sz, C.POINTER(Epilogue), ci, vp, vp]
    L.b200collReduce.argtypes = [vp, vp, sz, C.POINTER(Epilogue), ci, ci, vp, vp]
    L.b200collBarrier.argtypes = [vp, vp]
    L.b200collAllGatherBlockScaled.argtypes = [vp, vp, sz, C.POINTER(BlockScale), C.POINTER(Epilogue), vp, vp]
    L.b200collReduceScatterBlockScaled.argtypes = [vp, vp, sz, C.POINTER(BlockScale), C.POINTER(Epilogue), ci, vp, vp]
    L.b200collAllReduceBlockScaled.argtypes = [vp, vp, sz, C.POINTER(BlockScale), C.POINTER(Epilogue), ci, vp, vp]
    L.b200collAllGatherQuantized.argtypes = [vp, vp, sz, ci, ci, C.POINTER(Epilogue), vp, vp]
    L.b200collReduceScatterQuantized.argtypes = [vp, vp, sz, ci, ci, C.POINTER(Epilogue), ci, vp, vp]
    L.b200collAllReduceQuantized.argtypes = [vp, vp, sz, ci, ci, C.POINTER(Epilogue), ci, vp, vp]
    i64p = C.POINTER(C.c_int64)
    L.b200collAllToAllvQuantized.argtypes = [vp, vp, C.POINTER(C.c_float), sz, sz, i64p, i64p, i64p, ci, ci, ci, vp, vp]
    L.b200collAllToAllvCombine.argtypes = [vp, vp, sz, sz, i64p, i64p, i64p, C.POINTER(C.c_int32), C.POINTER(C.c_float), sz, ci,
                                           C.POINTER(Epilogue), vp, vp]
    i32p = C.POINTER(C.c_int32)
    L.b200collExpertDispatch.argtypes = [vp, vp, sz, sz, i32p, sz, ci, ci, i32p, i32p, i32p, ci, vp, vp]
    L.b200collExpertDispatchQuantized.argtypes = [vp, vp, C.POINTER(C.c_float), sz, sz, i32p, sz, ci, ci, i32p, i32p, i32p, ci, ci, ci, vp, vp]
    L.b200collExpertCombine.argtypes = [vp, vp, sz, sz, i32p, C.POINTER(C.c_float), sz, ci, C.POINTER(Epilogue), vp, vp]
    L.b200collAllToAllvCombineQuantized.argtypes = [vp, vp, sz, sz, i64p, i64p, i64p, i32p, C.POINTER(C.c_float), sz, ci, ci, ci, C.POINTER(Epilogue),
                                                    vp, vp]
    L.b200collExpertCombineQuantized.argtypes = [vp, vp, sz, sz, i32p, C.POINTER(C.c_float), sz, ci, ci, ci, C.POINTER(Epilogue), vp, vp]
    L.b200collAllReduceRmsNorm.argtypes = [vp, vp, vp, vp, sz, sz, C.c_float, ci, vp, vp]
    L.b200collAllReduceRmsNormQuantized.argtypes = [vp, vp, vp, vp, C.POINTER(C.c_float), sz, sz, C.c_float, ci, ci, ci, vp, vp]
    L.b200collReduceScatterRmsNorm.argtypes = [vp, vp, vp, vp, sz, sz, C.c_float, ci, ci, vp, vp]
    L.b200collReduceScatterRmsNormQuantized.argtypes = [vp, vp, vp, vp, C.POINTER(C.c_float), sz, sz, C.c_float, ci, ci, ci, ci, vp, vp]
    L.b200collAllToAllSeqToHeads.argtypes = [C.POINTER(UlyssesTensor), ci, sz, sz, sz, ci, vp, vp]
    L.b200collAllToAllHeadsToSeq.argtypes = [C.POINTER(UlyssesTensor), ci, sz, sz, sz, ci, vp, vp]
    L.b200collAllGatherContext.argtypes = [C.POINTER(ContextTensor), ci, sz, sz, ci, ci, vp, vp]
    L.b200collReduceScatterContext.argtypes = [C.POINTER(ContextTensor), ci, sz, sz, ci, ci, vp, vp]
    L.b200collAllGatherShards.argtypes = [C.POINTER(ShardTensor), ci, ci, ci, vp, vp]
    L.b200collReduceScatterShards.argtypes = [C.POINTER(ShardTensor), ci, ci, ci, C.c_float, ci, vp, vp]
    L.b200collVocabParallelCrossEntropy.argtypes = [vp, vp, vp, vp, sz, sz, C.c_int64, ci, vp, vp]
    L.b200collVocabParallelCrossEntropyBackward.argtypes = [vp, vp, vp, vp, vp, sz, sz, C.c_int64, ci, vp, vp]
    L.b200collVocabParallelEmbedding.argtypes = [vp, vp, vp, sz, sz, sz, ci, ci, vp, vp]
    L.b200collVocabParallelEmbeddingBackward.argtypes = [vp, vp, vp, sz, sz, sz, ci, ci, ci, ci, vp, vp]
    L.b200collHostAlloc.argtypes = [vp, C.POINTER(vp), sz]
    L.b200collHostFree.argtypes = [vp, vp]
    L.b200collAllReduceHost.argtypes = [vp, vp, sz, C.POINTER(Epilogue), ci, vp, vp]
    L.b200collCommNumaGet.argtypes = [vp, C.POINTER(ci), C.c_char_p, sz]
    L.b200collDebugParseCpuList.argtypes = [C.c_char_p, C.POINTER(ci), ci]
    L.b200collGroupStart.argtypes = []; L.b200collGroupEnd.argtypes = []
    L.b200collSend.argtypes = [vp, sz, ci, vp, vp]
    L.b200collRecv.argtypes = [vp, sz, ci, vp, vp]
    L.b200collTunerPick.argtypes = [ci, sz, ci, ci]; L.b200collTunerPick.restype = ci
    L.b200collCommSetAlgo.argtypes = [vp, ci]
    L.b200collCommGetAlgo.argtypes = [vp]; L.b200collCommGetAlgo.restype = ci
    L.b200collCommSetMaxCtas.argtypes = [vp, ci]
    L.b200collCommSetLaunchShape.argtypes = [vp, ci, ci, ci]
    L.b200collCommSetP2pWindow.argtypes = [vp, sz]
    L.b200collAlgoName.argtypes = [ci]; L.b200collAlgoName.restype = C.c_char_p
    L.b200collTypeSize.argtypes = [ci]; L.b200collTypeSize.restype = sz
    L.b200collSelfCheck.argtypes = [C.c_char_p, sz]
    return L


def _check(rc: int, what: str) -> None:
    if rc != SUCCESS:
        L = load()
        raise B200CollError(rc, f"{what}: {L.b200collGetErrorString(rc).decode()}", L.b200collGetLastError().decode())


class group:
    """`with coll.group(): comm.send(...); comm.recv(...)`: every send / recv issued inside (by this thread, on any communicator)
    becomes one kernel per communicator at exit (ncclGroupStart / ncclGroupEnd). Needed whenever a rank both sends and receives in
    one step: outside a group each call waits for its peer before the next one is launched."""

    def __enter__(self):
        _check(load().b200collGroupStart(), "GroupStart")
        return self

    def __exit__(self, exc_type, exc, tb):
        rc = load().b200collGroupEnd()
        if exc_type is None:
            _check(rc, "GroupEnd")
        return False


def tuner_pick(op: int, nbytes: int, nranks: int, nvls: bool) -> str:
    return ALGO_NAMES[load().b200collTunerPick(op, nbytes, nranks, 1 if nvls else 0)]


def self_check() -> tuple[bool, str]:
    buf = C.create_string_buffer(8192)
    rc = load().b200collSelfCheck(buf, len(buf))
    return rc == SUCCESS, buf.value.decode()


def torch_dtype_code(dtype) -> int:
    import torch
    return {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16, torch.float8_e4m3fn: FP8_E4M3, torch.float8_e5m2: FP8_E5M2, torch.int8: I8, torch.uint8: U8, torch.int32: I32,
            torch.uint32: U32, torch.int64: I64, torch.uint64: U64, torch.float64: F64, torch.bool: U8}[dtype]


def check_block_scaled(op: str, nranks: int, q, scales, out, block=(1, 128)) -> tuple[int, int]:
    """Shape and dtype rules of the block-scaled collectives ("all_gather", "reduce_scatter", "all_reduce"), checked on the tensors'
    metadata only (no device, no communicator): raises ValueError, returns (block_rows, block_cols).
    q: 2-D contiguous float8_e4m3fn / float8_e5m2 [rows, row_len]; scales: contiguous float32 (ceil(rows/br), ceil(row_len/bc));
    out: bfloat16 / float16 / float32 of shape (nranks*rows, row_len) for all-gather, (rows/nranks, row_len) for reduce-scatter,
    (rows, row_len) for all-reduce."""
    import torch
    if op not in ("all_gather", "reduce_scatter", "all_reduce"):
        raise ValueError(f"unknown block-scaled op {op!r}")
    if q.dtype not in (torch.float8_e4m3fn, torch.float8_e5m2):
        raise ValueError(f"q must be float8_e4m3fn or float8_e5m2, not {q.dtype}")
    if q.dim() != 2 or not q.is_contiguous():
        raise ValueError(f"q must be a contiguous 2-D [rows, row_len] tensor, got shape {tuple(q.shape)}")
    try:
        br, bc = (int(b) for b in block)
    except (TypeError, ValueError):
        raise ValueError(f"block must be (block_rows, block_cols), got {block!r}") from None
    if br < 1 or bc < 16 or bc % 16:
        raise ValueError(f"block {block!r}: block_rows must be >= 1 and block_cols a positive multiple of 16")
    rows, row_len = q.shape
    if row_len % 16:
        raise ValueError(f"row_len {row_len} must be a multiple of 16")
    want = (-(-rows // br), -(-row_len // bc))
    if scales.dtype != torch.float32 or tuple(scales.shape) != want or not scales.is_contiguous():
        raise ValueError(f"scales must be a contiguous float32 tensor of shape {want}, got {scales.dtype} {tuple(scales.shape)}")
    if out.dtype not in (torch.bfloat16, torch.float16, torch.float32) or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous bfloat16, float16 or float32 tensor, got {out.dtype}")
    if op == "reduce_scatter" and rows % nranks:
        raise ValueError(f"reduce_scatter: rows ({rows}) must be a multiple of nranks ({nranks})")
    out_shape = {"all_gather": (nranks * rows, row_len), "reduce_scatter": (rows // nranks, row_len), "all_reduce": (rows, row_len)}[op]
    if tuple(out.shape) != out_shape:
        raise ValueError(f"{op}: out must have shape {out_shape}, got {tuple(out.shape)}")
    return br, bc


QUANT_BLOCKS = (16, 32, 64, 128, 256, 512)


def _check_wide(name: str, t, rows: bool = False) -> None:
    """t must be a contiguous bfloat16, float16 or float32 tensor; rows: also 2-D, [tokens, row_elems]."""
    import torch
    if t.dtype not in (torch.bfloat16, torch.float16, torch.float32) or not t.is_contiguous() or (rows and t.dim() != 2):
        raise ValueError(f"{name} must be a contiguous bfloat16, float16 or float32 [tokens, row_elems] tensor, got {t.dtype}{list(t.shape)}" if rows
                         else f"{name} must be a contiguous bfloat16, float16 or float32 tensor, got {t.dtype}")


def _check_block(block) -> None:
    if isinstance(block, bool) or not isinstance(block, int) or block not in QUANT_BLOCKS:
        raise ValueError(f"block must be one of {QUANT_BLOCKS}, got {block!r}")


def _check_topk(name: str, t) -> None:
    """t must be a contiguous int32 [tokens, top_k] tensor with top_k >= 1."""
    import torch
    if t.dtype != torch.int32 or t.dim() != 2 or not t.is_contiguous() or t.shape[1] < 1:
        raise ValueError(f"{name} must be a contiguous int32 [tokens, top_k] tensor with top_k >= 1, got {t.dtype}{list(t.shape)}")


def _host_rows(nranks: int, send_rows, send_row_off, recv_row_off_at_peer) -> list[tuple[int, int, int]]:
    """The three host lists of an all-to-all-v call, checked (nranks non-negative integers each): [(rows, send_off, recv_off)] by peer."""
    import operator
    vals = []
    for name, xs in (("send_rows", send_rows), ("send_row_off", send_row_off), ("recv_row_off_at_peer", recv_row_off_at_peer)):
        try:
            v = [operator.index(x) for x in xs]
        except TypeError:
            raise ValueError(f"{name} must be a sequence of integers") from None
        if len(v) != nranks:
            raise ValueError(f"{name} must have nranks = {nranks} entries, got {len(v)}")
        if any(x < 0 for x in v):
            raise ValueError(f"{name} must not hold negative entries: {v}")
        vals.append(v)
    return list(zip(*vals))


def check_quantized(op: str, nranks: int, src, out, block: int = 128, wire=None) -> int:
    """Rules of the quantising collectives ("all_gather", "reduce_scatter", "all_reduce"), checked on the tensors' metadata only (no
    communicator, no library call): raises ValueError, returns the wire type's library code. src and out: contiguous bfloat16, float16
    or float32; wire: torch.float8_e4m3fn (default) or torch.float8_e5m2; block one of QUANT_BLOCKS. out has nranks * src.numel()
    elements for all-gather, src.numel() / nranks for reduce-scatter and src.numel() for all-reduce, and every rank's share is whole
    blocks. Only the all-reduce may run in place (out is src, or a tensor with the same data pointer and element size)."""
    import torch
    wire = torch.float8_e4m3fn if wire is None else wire
    if op not in ("all_gather", "reduce_scatter", "all_reduce"):
        raise ValueError(f"unknown quantised op {op!r}")
    _check_wide("src", src)
    _check_wide("out", out)
    if wire not in (torch.float8_e4m3fn, torch.float8_e5m2):
        raise ValueError(f"wire must be torch.float8_e4m3fn or torch.float8_e5m2, not {wire}")
    _check_block(block)
    n = src.numel()
    if op == "reduce_scatter" and n % nranks:
        raise ValueError(f"reduce_scatter: src.numel() ({n}) must be a multiple of nranks ({nranks})")
    want = {"all_gather": nranks * n, "reduce_scatter": n // nranks, "all_reduce": n}[op]
    if out.numel() != want:
        raise ValueError(f"{op}: out must have {want} elements, got {out.numel()}")
    share = n // nranks if op == "reduce_scatter" else n
    if share % block:
        raise ValueError(f"{op}: {'the per-rank slice' if op == 'reduce_scatter' else 'src.numel()'} ({share}) must be a multiple of block ({block})")
    a, na = src.data_ptr(), n * src.element_size()
    b, nb = out.data_ptr(), out.numel() * out.element_size()
    in_place = op == "all_reduce" and a == b and src.element_size() == out.element_size()
    if n and not in_place and a < b + nb and b < a + na:
        raise ValueError(f"{op}: out must not overlap src" + (" (in place needs out to be src, with a dtype of the same size)" if op == "all_reduce" else ""))
    return torch_dtype_code(wire)


def check_all_to_all_v_quantized(nranks: int, src, out, out_scales, row_elems: int, block: int, send_rows, send_row_off,
                                 recv_row_off_at_peer) -> tuple[int, int]:
    """Rules of the quantising all-to-all-v, checked on the tensors' metadata and the host lists only (no communicator, no library call):
    raises ValueError, returns the library codes of (src's type, the wire type). src: contiguous bfloat16, float16 or float32; out:
    contiguous float8_e4m3fn or float8_e5m2 (the wire type), out.numel() a multiple of row_elems; out_scales: contiguous float32 with
    out.numel() // block elements; block one of QUANT_BLOCKS and row_elems a positive multiple of it. The three lists have nranks
    non-negative entries; every send range [send_row_off[p], + send_rows[p]) lies inside src and every destination range
    [recv_row_off_at_peer[p], + send_rows[p]) inside out, in rows of row_elems elements. src must not overlap out or out_scales."""
    import torch
    _check_wide("src", src)
    if out.dtype not in (torch.float8_e4m3fn, torch.float8_e5m2) or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous float8_e4m3fn or float8_e5m2 tensor (the wire type), got {out.dtype}")
    if out_scales.dtype != torch.float32 or not out_scales.is_contiguous():
        raise ValueError(f"out_scales must be a contiguous float32 tensor, got {out_scales.dtype}")
    _check_block(block)
    if isinstance(row_elems, bool) or not isinstance(row_elems, int) or row_elems <= 0 or row_elems % block:
        raise ValueError(f"row_elems must be a positive multiple of block ({block}), got {row_elems!r}")
    if out.numel() % row_elems:
        raise ValueError(f"out.numel() ({out.numel()}) must be a multiple of row_elems ({row_elems})")
    if out_scales.numel() != out.numel() // block:
        raise ValueError(f"out_scales must hold out.numel() // block = {out.numel() // block} floats, got {out_scales.numel()}")
    src_rows, out_rows = src.numel() // row_elems, out.numel() // row_elems
    for p, (rows, so, ro) in enumerate(_host_rows(nranks, send_rows, send_row_off, recv_row_off_at_peer)):
        if so + rows > src_rows:
            raise ValueError(f"peer {p}: send rows [{so}, {so + rows}) lie past the {src_rows} whole rows of src")
        if ro + rows > out_rows:
            raise ValueError(f"peer {p}: destination rows [{ro}, {ro + rows}) lie past the {out_rows} rows of out")
    if _overlap(src, out) or _overlap(src, out_scales):
        raise ValueError("src must not overlap out or out_scales")
    return torch_dtype_code(src.dtype), torch_dtype_code(out.dtype)


def _check_combine_quant(fp8, row_elems: int) -> int:
    """The quantising combine's own rules, fp8 = (block, wire): wire torch.float8_e4m3fn (None) or torch.float8_e5m2, block one of
    QUANT_BLOCKS and row_elems a positive multiple of it. Returns the wire type's library code."""
    import torch
    block, wire = fp8
    wire = torch.float8_e4m3fn if wire is None else wire
    if wire not in (torch.float8_e4m3fn, torch.float8_e5m2):
        raise ValueError(f"wire must be torch.float8_e4m3fn or torch.float8_e5m2, not {wire}")
    _check_block(block)
    if isinstance(row_elems, bool) or not isinstance(row_elems, int) or row_elems <= 0 or row_elems % block:
        raise ValueError(f"row_elems must be a positive multiple of block ({block}), got {row_elems!r}")
    return torch_dtype_code(wire)


def _check_combine_sizes(tokens: int, top_k: int, row_elems: int, eo_rows: int) -> None:
    """The quantising combine's 32-bit limits: tokens * top_k slots, the 16-element vectors of out and of expert_out."""
    if tokens * top_k > _I31:
        raise ValueError("tokens * top_k must be at most 2^31 - 1")
    if tokens * (row_elems // 16) > _I31:
        raise ValueError("at most 2^31 - 1 16-element vectors of out (tokens * row_elems / 16)")
    if eo_rows * (row_elems // 16) > _I31:
        raise ValueError("at most 2^31 - 1 16-element vectors of expert_out (expert_out.numel() / 16)")


def _check_a2av_combine(nranks: int, expert_out, out, row_elems: int, send_rows, send_row_off, recv_row_off_at_peer, index, weights,
                        fp8=None) -> tuple:
    """The rules of both all-to-all-v combines; fp8 is None (check_all_to_all_v_combine) or (block, wire), which adds the quantising
    call's rules, as combine_prepare in coll/src/combine.cu takes a CombineQuant."""
    import torch
    _check_wide("expert_out", expert_out)
    _check_wide("out", out)
    if fp8 is not None:
        wc = _check_combine_quant(fp8, row_elems)
    elif isinstance(row_elems, bool) or not isinstance(row_elems, int) or row_elems <= 0 or row_elems % 16:
        raise ValueError(f"row_elems must be a positive multiple of 16, got {row_elems!r}")
    if expert_out.numel() % row_elems:
        raise ValueError(f"expert_out.numel() ({expert_out.numel()}) must be a multiple of row_elems ({row_elems})")
    _check_topk("index", index)
    tokens, top_k = index.shape
    if weights is not None and (weights.dtype != torch.float32 or tuple(weights.shape) != (tokens, top_k) or not weights.is_contiguous()):
        raise ValueError(f"weights must be None or a contiguous float32 [{tokens}, {top_k}] tensor, got {weights.dtype}{list(weights.shape)}")
    if out.numel() != tokens * row_elems:
        raise ValueError(f"out must hold tokens * row_elems = {tokens * row_elems} elements, got {out.numel()}")
    eo_rows = expert_out.numel() // row_elems
    if fp8 is not None:
        _check_combine_sizes(tokens, top_k, row_elems, eo_rows)
    ranges = []
    for p, (rows, so, ro) in enumerate(_host_rows(nranks, send_rows, send_row_off, recv_row_off_at_peer)):
        if ro + rows > eo_rows:
            raise ValueError(f"peer {p}: destination rows [{ro}, {ro + rows}) lie past the {eo_rows} rows of expert_out")
        if rows:
            ranges.append((so, so + rows, p))
    ranges.sort()
    for (lo0, hi0, p0), (lo1, hi1, p1) in zip(ranges, ranges[1:]):
        if lo1 < hi0:
            raise ValueError(f"the send ranges of peers {p0} [{lo0}, {hi0}) and {p1} [{lo1}, {hi1}) overlap: a dispatch row must belong to one peer")
    for name, t in (("expert_out", expert_out), ("index", index), ("weights", weights)):
        if t is not None and _overlap(out, t):
            raise ValueError(f"out must not overlap {name}")
    codes = (torch_dtype_code(expert_out.dtype), torch_dtype_code(out.dtype))
    return codes if fp8 is None else codes + (wc,)


def check_all_to_all_v_combine(nranks: int, expert_out, out, row_elems: int, send_rows, send_row_off, recv_row_off_at_peer, index,
                               weights) -> tuple[int, int]:
    """Rules of the expert combine, checked on the tensors' metadata and the host lists only (no communicator, no library call): raises
    ValueError, returns the library codes of (expert_out's type, out's type). expert_out and out: contiguous bfloat16, float16 or float32;
    row_elems a positive multiple of 16 dividing expert_out.numel(); index: contiguous int32 [tokens, top_k] with top_k >= 1; weights:
    None or contiguous float32 of index's shape; out.numel() == tokens * row_elems. The three lists have nranks non-negative entries,
    the non-empty send ranges [send_row_off[p], + send_rows[p]) are disjoint, and every destination range [recv_row_off_at_peer[p],
    + send_rows[p]) lies inside expert_out, in rows of row_elems elements. out must not overlap expert_out, index or weights."""
    return _check_a2av_combine(nranks, expert_out, out, row_elems, send_rows, send_row_off, recv_row_off_at_peer, index, weights)


def check_all_to_all_v_combine_quantized(nranks: int, expert_out, out, row_elems: int, send_rows, send_row_off, recv_row_off_at_peer, index,
                                         weights, block: int = 128, wire=None) -> tuple[int, int, int]:
    """Rules of the quantising all-to-all-v combine, checked on the tensors' metadata and the host lists only: raises ValueError, returns
    the library codes of (expert_out's type, out's type, the wire type). Everything check_all_to_all_v_combine checks, and: wire
    torch.float8_e4m3fn (None, the default) or torch.float8_e5m2; block one of QUANT_BLOCKS and row_elems a positive multiple of it;
    tokens * top_k, tokens * row_elems / 16 and expert_out.numel() / 16 at most 2^31 - 1."""
    return _check_a2av_combine(nranks, expert_out, out, row_elems, send_rows, send_row_off, recv_row_off_at_peer, index, weights, fp8=(block, wire))


MAX_EXPERTS = 1024
_I31 = 2 ** 31 - 1


def _numel(shape) -> int:
    n = 1
    for d in shape:
        n *= d
    return n


def _overlap(t, u) -> bool:
    a, na = t.data_ptr(), t.numel() * t.element_size()
    b, nb = u.data_ptr(), u.numel() * u.element_size()
    return bool(na and nb and a < b + nb and b < a + na)


RMS_NORM_MAX_ROW = 16384


def _rs_shapes(x, nranks: int, gather: bool) -> tuple[tuple, tuple]:
    """The reduce-scatter form's (residual shape, out shape): x's shape with dim 0 divided by nranks, and x's own when gathering."""
    if x.dim() < 2:
        raise ValueError("x must have at least two dimensions (the sequence, sharded along dim 0, then the rows' elements)")
    shape = tuple(x.shape)
    if shape[0] % nranks:
        raise ValueError(f"x.shape[0] ({shape[0]}) must be a multiple of nranks ({nranks})")
    shard = (shape[0] // nranks,) + shape[1:]
    return shard, (shape if gather else shard)


def _check_rms_norm(x, residual, weight, eps, out=None, sp=None) -> tuple[int, int]:
    """The rules the all-reduce and reduce-scatter + RMSNorm calls share, and out's when it is given (the wide calls): returns (rows,
    row_len), rows counting every row of x. sp: None (the all-reduce form: residual and out of x's shape) or (nranks, gather), the
    reduce-scatter form's shapes."""
    import math
    wides = (("x", x), ("residual", residual), ("weight", weight)) + ((("out", out),) if out is not None else ())
    for name, t in wides:
        _check_wide(name, t)
        if t.dtype != x.dtype:
            raise ValueError(f"{name} must have x's dtype {x.dtype}, got {t.dtype}")
    if x.dim() < 1:
        raise ValueError("x must have at least one dimension")
    shape = tuple(x.shape)
    want = {"residual": shape, "out": shape}
    if sp is not None:
        want["residual"], want["out"] = _rs_shapes(x, *sp)
    for name, t in wides[1:]:
        if name != "weight" and tuple(t.shape) != want[name]:
            whose = "x's shape" if want[name] == shape else "the shard's shape"
            raise ValueError(f"{name} must have {whose} {list(want[name])}, got {list(t.shape)}")
    row_len = shape[-1]
    if row_len < 16 or row_len > RMS_NORM_MAX_ROW or row_len % 16:
        raise ValueError(f"row_len (the last dimension) must be a multiple of 16 in [16, {RMS_NORM_MAX_ROW}], got {row_len}")
    if tuple(weight.shape) != (row_len,):
        raise ValueError(f"weight must have shape [{row_len}], got {list(weight.shape)}")
    if isinstance(eps, bool) or not isinstance(eps, (int, float)) or not math.isfinite(eps) or eps < 0:
        raise ValueError(f"eps must be a finite number >= 0, got {eps!r}")
    rows = _numel(shape[:-1])
    if rows > _I31:
        raise ValueError(f"at most 2^31 - 1 rows, got {rows}")
    if rows:
        for name, t in wides:
            if t.data_ptr() % 16:
                raise ValueError(f"{name} must be 16-byte aligned")
        if out is not None and any(_overlap(out, t) for t in (x, residual, weight)):
            raise ValueError("out must not overlap x, residual or weight")
        if _overlap(residual, x) or _overlap(residual, weight):
            raise ValueError("residual must not overlap x or weight")
    return rows, row_len


def check_all_reduce_rms_norm(x, residual, weight, out, eps: float = 1e-6) -> tuple[int, int]:
    """The rules of Comm.all_reduce_rms_norm, checked on the tensors' metadata (no device, no communicator): raises ValueError, returns
    (rows, row_len). x, residual and out are contiguous [..., row_len] tensors of one shape, weight a contiguous [row_len] tensor, all four of
    one dtype (bfloat16, float16 or float32); row_len a multiple of 16 in [16, 16384]; eps finite and >= 0; fewer than 2^31 rows; every
    pointer 16-byte aligned; out must not overlap x, residual or weight, residual must not overlap x or weight."""
    return _check_rms_norm(x, residual, weight, eps, out)


def check_all_reduce_rms_norm_quantized(x, residual, weight, q, scales, block: int = 128, wire=None, eps: float = 1e-6) -> tuple[int, int, int]:
    """The rules of Comm.all_reduce_rms_norm_quantized, checked on the tensors' metadata (no device, no communicator): raises ValueError,
    returns (rows, row_len, the wire type's library code). x, residual and weight as in check_all_reduce_rms_norm; wire
    torch.float8_e4m3fn (None, the default) or torch.float8_e5m2; block one of QUANT_BLOCKS and row_len a multiple of it; q a contiguous
    tensor of x's shape and the wire dtype, 16-byte aligned; scales a contiguous float32 [..., row_len // block] tensor (x's leading
    dimensions); x, residual, weight, q and scales must not overlap."""
    return _check_rms_norm_quantized(x, residual, weight, q, scales, block, wire, eps)


def _check_rms_norm_quantized(x, residual, weight, q, scales, block, wire, eps, sp=None) -> tuple[int, int, int]:
    """The rules of both quantising + RMSNorm calls; sp as in _check_rms_norm (q and scales take out's rows)."""
    import torch
    rows, row_len = _check_rms_norm(x, residual, weight, eps, sp=sp)
    oshape = tuple(x.shape) if sp is None else _rs_shapes(x, *sp)[1]
    wire = torch.float8_e4m3fn if wire is None else wire
    if wire not in (torch.float8_e4m3fn, torch.float8_e5m2):
        raise ValueError(f"wire must be torch.float8_e4m3fn or torch.float8_e5m2, not {wire}")
    _check_block(block)
    if row_len % block:
        raise ValueError(f"row_len ({row_len}) must be a multiple of block ({block})")
    if q.dtype != wire or tuple(q.shape) != oshape or not q.is_contiguous():
        whose = "x's shape" if oshape == tuple(x.shape) else "the shard's shape"
        raise ValueError(f"q must be a contiguous {wire} tensor of {whose} {list(oshape)}, got {q.dtype}{list(q.shape)}")
    want = oshape[:-1] + (row_len // block,)
    if scales.dtype != torch.float32 or tuple(scales.shape) != want or not scales.is_contiguous():
        raise ValueError(f"scales must be a contiguous float32 tensor of shape {list(want)}, got {scales.dtype}{list(scales.shape)}")
    if rows:
        if q.data_ptr() % 16:
            raise ValueError("q must be 16-byte aligned")
        if any(_overlap(q, t) for t in (x, residual, weight, scales)):
            raise ValueError("q must not overlap x, residual, weight or scales")
        if any(_overlap(scales, t) for t in (x, residual, weight)):
            raise ValueError("scales must not overlap x, residual or weight")
    return rows, row_len, torch_dtype_code(wire)


def check_reduce_scatter_rms_norm(nranks: int, x, residual, weight, out, eps: float = 1e-6, gather: bool = False) -> tuple[int, int]:
    """The rules of Comm.reduce_scatter_rms_norm, checked on the tensors' metadata (no device, no communicator): raises ValueError, returns
    (rows, row_len), rows counting every row of x. As check_all_reduce_rms_norm, except for the shapes: x has at least two dimensions
    and x.shape[0] is a multiple of nranks (the sequence is sharded along dim 0); residual has x's shape with dim 0 divided by nranks;
    out has residual's shape, or x's when gathering."""
    return _check_rms_norm(x, residual, weight, eps, out, sp=(nranks, bool(gather)))


def check_reduce_scatter_rms_norm_quantized(nranks: int, x, residual, weight, q, scales, block: int = 128, wire=None, eps: float = 1e-6,
                                            gather: bool = False) -> tuple[int, int, int]:
    """The rules of Comm.reduce_scatter_rms_norm_quantized, checked on the tensors' metadata: raises ValueError, returns (rows, row_len,
    the wire type's library code). Shapes as in check_reduce_scatter_rms_norm, with q of out's shape and scales [..., row_len // block]
    of out's leading dimensions; everything else as in check_all_reduce_rms_norm_quantized."""
    return _check_rms_norm_quantized(x, residual, weight, q, scales, block, wire, eps, sp=(nranks, bool(gather)))


def ulysses_local_heads(nranks: int, heads: int, replicate: bool = True) -> int:
    """Heads per rank on the head-sharded side of the Ulysses all-to-all: heads // nranks when nranks divides heads, else 1 when heads
    divides nranks (each head replicated to nranks // heads ranks; replicate=False, heads -> sequence, refuses it); ValueError otherwise."""
    if heads % nranks == 0:
        return heads // nranks
    if not replicate:
        raise ValueError(f"heads ({heads}) must be a multiple of nranks ({nranks}): the replicated layout has no inverse move")
    if nranks % heads:
        raise ValueError(f"heads ({heads}) must be a multiple or a divisor of nranks ({nranks})")
    return 1


def _seq_row_stride(name: str, t) -> int:
    """The row stride (elements) of a sequence-side [B, S_l, H, D] view whose token rows are uniformly strided."""
    B, S_l, H, D = t.shape
    if (D > 1 and t.stride(3) != 1) or (H > 1 and t.stride(2) != D):
        raise ValueError(f"{name}: each token row must hold its heads * head_dim elements contiguously (stride(3) == 1, stride(2) == head_dim), "
                         f"got strides {t.stride()}")
    rs = t.stride(1) if S_l > 1 or B == 1 else t.stride(0)
    if S_l > 1 and B > 1 and t.stride(0) != S_l * rs:
        raise ValueError(f"{name}: token rows must be uniformly strided (stride(0) == seq_local * stride(1)), got strides {t.stride()}")
    return rs if B * S_l > 1 else H * D          # one token row: its stride is never used


def _spans_overlap(a, b) -> bool:
    """Whether two row-strided byte regions (ptr, rows, stride, width) share a byte; as the library decides it."""
    ext = [0 if r == 0 else (r - 1) * s + w for _, r, s, w in (a, b)]
    if not ext[0] or not ext[1] or not (a[0] < b[0] + ext[1] and b[0] < a[0] + ext[0]):
        return False
    if a[1] < 2 or b[1] < 2 or a[2] != b[2] or a[3] > a[2] or b[3] > b[2]:
        return True
    dd = (b[0] - a[0]) % a[2]
    return dd < a[3] or dd + b[3] > a[2]


def _check_ulysses(nranks: int, seqs, heads, s2h: bool) -> tuple[int, int, int, list[tuple[int, int]]]:
    import torch
    what = "seq_to_heads" if s2h else "heads_to_seq"
    seqs, heads = list(seqs), list(heads)
    if not 1 <= len(seqs) <= 3 or len(heads) != len(seqs):
        raise ValueError(f"{what}: 1 to 3 tensors and one output per tensor, got {len(seqs)} and {len(heads)}")
    sname, hname = ("xs", "outs") if s2h else ("outs", "ys")
    dt = seqs[0].dtype
    if dt not in (torch.bfloat16, torch.float16, torch.float32, torch.float8_e4m3fn, torch.float8_e5m2):
        raise ValueError(f"{what}: dtype must be bfloat16, float16, float32, float8_e4m3fn or float8_e5m2, got {dt}")
    if any(t.dim() != 4 for t in seqs + heads):
        raise ValueError(f"{what}: every tensor must be 4-D: [B, S_l, H, D] on the sequence side, [B, S, H / N, D] on the head side")
    B, S_l, _, D = seqs[0].shape
    es = seqs[0].element_size()
    if (D * es) % 16 or D == 0:
        raise ValueError(f"{what}: head_dim * sizeof(dtype) must be a positive multiple of 16 bytes, got {D} x {es}")
    rows = B * S_l
    if rows > _I31:
        raise ValueError(f"{what}: batch * seq_local must be below 2^31, got {rows}")
    per, srcs, dsts, moved = [], [], [], 0
    for i, (x, y) in enumerate(zip(seqs, heads)):
        if x.dtype != dt or y.dtype != dt:
            raise ValueError(f"{what}: tensor {i}: every tensor must have dtype {dt}, got {x.dtype} and {y.dtype}")
        if (x.shape[0], x.shape[1], x.shape[3]) != (B, S_l, D):
            raise ValueError(f"{what}: {sname}[{i}] must be [{B}, {S_l}, H, {D}] like the first, got {list(x.shape)}")
        H = x.shape[2]
        if H < 1:
            raise ValueError(f"{what}: {sname}[{i}] has no heads")
        hl = ulysses_local_heads(nranks, H, s2h)
        want = (B, nranks * S_l, hl, D)
        if tuple(y.shape) != want or not y.is_contiguous():
            raise ValueError(f"{what}: {hname}[{i}] must be a contiguous {list(want)} tensor, got {list(y.shape)}")
        rs = _seq_row_stride(f"{sname}[{i}]", x)
        if rs < H * D or (rs * es) % 16:
            raise ValueError(f"{what}: {sname}[{i}]: the row stride ({rs}) must be at least heads * head_dim ({H * D}) and a multiple of 16 bytes")
        if rows and (x.data_ptr() % 16 or y.data_ptr() % 16):
            raise ValueError(f"{what}: tensor {i}: every pointer must be 16-byte aligned")
        dv = D * es // 16
        if (rows - 1) * rs * es // 16 + H * dv > _I31 or y.numel() * es // 16 > _I31:
            raise ValueError(f"{what}: tensor {i}: more than 2^31 - 1 16-byte vectors per rank")
        moved += rows * H * dv
        seq_span = (x.data_ptr(), rows, rs * es, H * D * es)          # (address, rows, stride, width) in bytes
        head_span = (y.data_ptr(), 1, y.numel() * es, y.numel() * es)
        srcs.append(seq_span if s2h else head_span)
        dsts.append(head_span if s2h else seq_span)
        per.append((rs, H))
    if moved > _I31:
        raise ValueError(f"{what}: more than 2^31 - 1 16-byte vectors moved per rank")
    for i, d in enumerate(dsts):
        for j, s in enumerate(srcs):
            if _spans_overlap(d, s):
                raise ValueError(f"{what}: output {i} overlaps source {j}")
        for j in range(i + 1, len(dsts)):
            if _spans_overlap(d, dsts[j]):
                raise ValueError(f"{what}: outputs {i} and {j} overlap")
    return B, S_l, D, per


def check_all_to_all_seq_to_heads(nranks: int, xs, outs) -> tuple[int, int, int, list[tuple[int, int]]]:
    """The rules of Comm.all_to_all_seq_to_heads, checked on the tensors' metadata (no device, no communicator): raises ValueError, returns
    (batch, seq_local, head_dim, [(row_stride, heads)] per tensor). xs: 1 to 3 [B, S_l, H_i, D] views of one dtype (bfloat16, float16,
    float32, float8_e4m3fn or float8_e5m2) whose token rows are uniformly strided (stride(3) == 1, stride(2) == D, stride(0) == S_l *
    stride(1)), such as column slices of a packed QKV tensor; outs: contiguous [B, N * S_l, Hl_i, D], Hl_i = H_i / N, or 1 when H_i divides
    N (ulysses_local_heads). D * sizeof(dtype) and every row stride a multiple of 16 bytes, every pointer 16-byte aligned, B * S_l below
    2^31, at most 2^31 - 1 16-byte vectors per rank; no output may overlap a source or another output."""
    return _check_ulysses(nranks, xs, outs, True)


def check_all_to_all_heads_to_seq(nranks: int, ys, outs) -> tuple[int, int, int, list[tuple[int, int]]]:
    """The rules of Comm.all_to_all_heads_to_seq, checked on the tensors' metadata: raises ValueError, returns as
    check_all_to_all_seq_to_heads. ys: 1 to 3 contiguous [B, N * S_l, H_i / N, D] tensors; outs: the [B, S_l, H_i, D] sequence-side views
    (row-strided as xs there). H_i must be a multiple of N: the replicated layout has no inverse. Everything else as seq-to-heads."""
    return _check_ulysses(nranks, outs, ys, False)


def _shard_row_stride(name: str, t) -> int:
    """The row stride (elements) of a [B, S_l, ...] view whose token rows are uniformly strided and hold their elements contiguously."""
    B, S_l = t.shape[:2]
    want = 1
    for size, st in reversed(list(zip(t.shape[2:], t.stride()[2:]))):
        if size > 1 and st != want:
            raise ValueError(f"{name}: each token row must hold its elements contiguously, got shape {list(t.shape)} and strides {t.stride()}")
        want *= size
    rs = t.stride(1) if S_l > 1 or B == 1 else t.stride(0)
    if S_l > 1 and B > 1 and t.stride(0) != S_l * rs:
        raise ValueError(f"{name}: token rows must be uniformly strided (stride(0) == seq_local * stride(1)), got strides {t.stride()}")
    return rs if B * S_l > 1 else want          # one token row: its stride is never used


def _check_context(nranks: int, shards, fulls, chunks: int, gather: bool) -> tuple[int, int, list[tuple[int, int]]]:
    import torch
    what = "all_gather_context" if gather else "reduce_scatter_context"
    shards, fulls = list(shards), list(fulls)
    if not 1 <= len(shards) <= 3 or len(fulls) != len(shards):
        raise ValueError(f"{what}: 1 to 3 tensors and one full tensor per shard, got {len(shards)} shards and {len(fulls)} fulls")
    dt = shards[0].dtype
    allowed = (torch.bfloat16, torch.float16, torch.float32) + ((torch.float8_e4m3fn, torch.float8_e5m2) if gather else ())
    if dt not in allowed:
        raise ValueError(f"{what}: dtype must be one of {', '.join(str(d).split('.')[-1] for d in allowed)}, got {dt}")
    if chunks not in (1, 2):
        raise ValueError(f"{what}: chunks must be 1 or 2, got {chunks}")
    if any(t.dim() < 3 for t in shards + fulls):
        raise ValueError(f"{what}: every tensor must be [B, S_l, ...] (shards) or [B, N * S_l, ...] (fulls), at least 3-D")
    B, S_l = shards[0].shape[:2]
    if chunks == 2 and S_l % 2:
        raise ValueError(f"{what}: chunks = 2 needs an even seq_local, got {S_l}")
    rows = B * S_l
    if rows > _I31:
        raise ValueError(f"{what}: batch * seq_local must be below 2^31, got {rows}")
    es = shards[0].element_size()
    per, srcs, dsts, moved = [], [], [], 0
    for i, (x, f) in enumerate(zip(shards, fulls)):
        if x.dtype != dt or f.dtype != dt:
            raise ValueError(f"{what}: tensor {i}: every tensor must have dtype {dt}, got {x.dtype} and {f.dtype}")
        if tuple(x.shape[:2]) != (B, S_l):
            raise ValueError(f"{what}: shards[{i}] must be [{B}, {S_l}, ...] like the first, got {list(x.shape)}")
        want = (B, nranks * S_l, *x.shape[2:])
        if tuple(f.shape) != want or not f.is_contiguous():
            raise ValueError(f"{what}: fulls[{i}] must be a contiguous {list(want)} tensor, got {list(f.shape)}")
        W = _prod(x.shape[2:])
        if W == 0 or (W * es) % 16:
            raise ValueError(f"{what}: tensor {i}: width * sizeof(dtype) must be a positive multiple of 16 bytes, got {W} x {es}")
        rs = _shard_row_stride(f"shards[{i}]", x)
        if rs < W or (rs * es) % 16:
            raise ValueError(f"{what}: shards[{i}]: the row stride ({rs}) must be at least the width ({W}) and a multiple of 16 bytes")
        if rows and (x.data_ptr() % 16 or f.data_ptr() % 16):
            raise ValueError(f"{what}: tensor {i}: every pointer must be 16-byte aligned")
        wv = W * es // 16
        if rows and ((rows - 1) * rs * es // 16 + wv > _I31 or nranks * rows * wv > _I31):
            raise ValueError(f"{what}: tensor {i}: more than 2^31 - 1 16-byte vectors per rank")
        moved += rows * wv
        shard_span = (x.data_ptr(), rows, rs * es, W * es)           # (address, rows, stride, width) in bytes
        full_span = (f.data_ptr(), 1, f.numel() * es, f.numel() * es)
        srcs.append(shard_span if gather else full_span)
        dsts.append(full_span if gather else shard_span)
        per.append((rs, W))
    if moved > _I31:
        raise ValueError(f"{what}: more than 2^31 - 1 16-byte vectors moved per rank")
    for i, d in enumerate(dsts):
        for j, s in enumerate(srcs):
            if _spans_overlap(d, s):
                raise ValueError(f"{what}: output {i} overlaps source {j}")
        for j in range(i + 1, len(dsts)):
            if _spans_overlap(d, dsts[j]):
                raise ValueError(f"{what}: outputs {i} and {j} overlap")
    return B, S_l, per


def _prod(shape) -> int:
    n = 1
    for d in shape:
        n *= d
    return n


def check_all_gather_context(nranks: int, shards, fulls, chunks: int) -> tuple[int, int, list[tuple[int, int]]]:
    """The rules of Comm.all_gather_context, checked on the tensors' metadata (no device, no communicator): raises ValueError, returns
    (batch, seq_local, [(row_stride, width)] per tensor). shards: 1 to 3 [B, S_l, ...] views of one dtype (bfloat16, float16, float32,
    float8_e4m3fn or float8_e5m2) whose token rows are uniformly strided and hold their W elements contiguously, such as the K and V
    column slices of a packed QKV tensor; fulls: contiguous [B, N * S_l, ...] with the shards' trailing shape. chunks 1 or 2 (2 needs an
    even S_l); W * sizeof(dtype) and every row stride a multiple of 16 bytes, every pointer 16-byte aligned, B * S_l below 2^31, at most
    2^31 - 1 16-byte vectors per rank; no output may overlap a source or another output."""
    return _check_context(nranks, shards, fulls, chunks, True)


def check_reduce_scatter_context(nranks: int, fulls, shards, chunks: int) -> tuple[int, int, list[tuple[int, int]]]:
    """The rules of Comm.reduce_scatter_context, checked on the tensors' metadata: raises ValueError, returns as
    check_all_gather_context. fulls: 1 to 3 contiguous [B, N * S_l, ...] tensors of bfloat16, float16 or float32; shards: the [B, S_l,
    ...] outputs, row-strided views allowed (the K and V column slices of a packed dQKV tensor). Everything else as the gather."""
    return _check_context(nranks, shards, fulls, chunks, False)


MAX_SHARD_TENSORS = 64


def shard_range(rows: int, shard_rows: int, rank: int) -> tuple[int, int]:
    """The rows [first, first + n) that rank owns of a tensor of `rows` rows sharded `shard_rows` per rank along dim 0, as the header
    states it: first = rank * shard_rows, n = clamp(rows - first, 0, shard_rows) (first clamped to rows when n is 0)."""
    first = min(rows, rank * shard_rows)
    return first, max(0, min(rows - first, shard_rows))


def _check_shards(nranks: int, rank: int, shards, fulls, shard_rows, gather: bool) -> list[tuple[int, int, int]]:
    import torch
    what = "all_gather_shards" if gather else "reduce_scatter_shards"
    shards, fulls = list(shards), list(fulls)
    if not 1 <= len(fulls) <= MAX_SHARD_TENSORS or len(shards) != len(fulls):
        raise ValueError(f"{what}: 1 to {MAX_SHARD_TENSORS} tensors and one shard per full, got {len(shards)} shards and {len(fulls)} fulls")
    sdt, fdt = shards[0].dtype, fulls[0].dtype
    if gather:
        ok = (sdt == fdt and sdt in (torch.bfloat16, torch.float16, torch.float32, torch.float8_e4m3fn, torch.float8_e5m2)) or \
             (sdt == torch.float32 and fdt in (torch.bfloat16, torch.float16))
        pairs = "one dtype in and out (bfloat16, float16, float32, float8_e4m3fn or float8_e5m2), or float32 -> bfloat16 or float16"
    else:
        ok = (sdt == fdt and sdt in (torch.bfloat16, torch.float16, torch.float32)) or \
             (sdt == torch.float32 and fdt in (torch.bfloat16, torch.float16))
        pairs = "bfloat16, float16 or float32 -> the same, or bfloat16 or float16 -> float32"
    if not ok:
        src, dst = (sdt, fdt) if gather else (fdt, sdt)
        raise ValueError(f"{what}: the dtype pair must be {pairs}, got {src} -> {dst}")
    if shard_rows is None or isinstance(shard_rows, int):
        rows_per = [shard_rows] * len(fulls)
    else:
        rows_per = list(shard_rows)
        if len(rows_per) != len(fulls):
            raise ValueError(f"{what}: shard_rows must be one int or one per tensor, got {len(rows_per)} for {len(fulls)} tensors")
    ess, esf = shards[0].element_size(), fulls[0].element_size()
    per, srcs, dsts, total = [], [], [], 0
    for i, (x, f, p) in enumerate(zip(shards, fulls, rows_per)):
        if x.dtype != sdt or f.dtype != fdt:
            raise ValueError(f"{what}: tensor {i}: every shard must be {sdt} and every full {fdt}, got {x.dtype} and {f.dtype}")
        if f.dim() < 1 or not f.is_contiguous():
            raise ValueError(f"{what}: fulls[{i}] must be a contiguous tensor of at least one dim, got shape {list(f.shape)}")
        d, W = f.shape[0], _prod(f.shape[1:])
        if d == 0 or W == 0:
            raise ValueError(f"{what}: tensor {i}: rows and width must be positive, got shape {list(f.shape)}")
        p = -(-d // nranks) if p is None else p
        if p < 1:
            raise ValueError(f"{what}: tensor {i}: shard_rows must be positive, got {p}")
        if nranks * p < d:
            raise ValueError(f"{what}: tensor {i}: nranks * shard_rows must be at least rows, got {nranks} x {p} < {d}")
        _, n_r = shard_range(d, p, rank)
        if x.dim() != f.dim() or tuple(x.shape[1:]) != tuple(f.shape[1:]) or x.shape[0] < n_r or not x.is_contiguous():
            raise ValueError(f"{what}: shards[{i}] must be a contiguous [>= {n_r}, {', '.join(str(e) for e in f.shape[1:])}] tensor "
                             f"(rank {rank}'s rows of fulls[{i}]), got {list(x.shape)}")
        if any((p * W * es) % 16 or (d * W * es) % 16 for es in (ess, esf)):
            raise ValueError(f"{what}: tensor {i}: shard_rows * width and rows * width must be multiples of 16 bytes in both dtypes, "
                             f"got {p} x {W} and {d} x {W}")
        if max(d, p) * W * max(ess, esf) // 16 > _I31:
            raise ValueError(f"{what}: tensor {i}: more than 2^31 - 1 16-byte vectors in one side")
        if f.data_ptr() % 16 or (n_r and x.data_ptr() % 16):
            raise ValueError(f"{what}: tensor {i}: every pointer must be 16-byte aligned")
        total += p * W * esf // 16
        shard_span = (x.data_ptr(), 1, n_r * W * ess, n_r * W * ess)
        full_span = (f.data_ptr(), 1, d * W * esf, d * W * esf)
        srcs.append(shard_span if gather else full_span)
        dsts.append(full_span if gather else shard_span)
        per.append((d, W, p))
    if total > _I31:
        raise ValueError(f"{what}: more than 2^31 - 1 16-byte vectors in the call")
    for i, dd in enumerate(dsts):
        for j, sp in enumerate(srcs):
            if _spans_overlap(dd, sp):
                raise ValueError(f"{what}: output {i} overlaps source {j}")
        for j in range(i + 1, len(dsts)):
            if _spans_overlap(dd, dsts[j]):
                raise ValueError(f"{what}: outputs {i} and {j} overlap")
    return per


def check_all_gather_shards(nranks: int, rank: int, shards, fulls, shard_rows=None) -> list[tuple[int, int, int]]:
    """The rules of Comm.all_gather_shards, checked on the tensors' metadata (no device, no communicator): raises ValueError, returns
    [(rows, width, shard_rows)] per tensor. fulls: 1 to 64 contiguous tensors; rows d is dim 0 and width W the product of the other
    dims. shard_rows p: None (FSDP2's ceil(d / nranks)), one int, or one per tensor, with nranks * p >= d. shards: contiguous, with the
    full's trailing shape and at least n_r = clamp(d - rank * p, 0, p) rows. Dtypes (shard -> full): one dtype in and out (bfloat16,
    float16, float32, float8_e4m3fn or float8_e5m2), or float32 -> bfloat16 or float16. p * W and d * W whole multiples of 16 bytes in
    both dtypes, pointers 16-byte aligned, at most 2^31 - 1 16-byte vectors per side and in sum p * W; no output may overlap a source
    or another output."""
    return _check_shards(nranks, rank, shards, fulls, shard_rows, True)


def check_reduce_scatter_shards(nranks: int, rank: int, fulls, shards, shard_rows=None) -> list[tuple[int, int, int]]:
    """The rules of Comm.reduce_scatter_shards, checked on the tensors' metadata: raises ValueError, returns as check_all_gather_shards.
    Dtypes (full -> shard): bfloat16, float16 or float32 to the same, or bfloat16 or float16 to float32. Everything else as the
    gather."""
    return _check_shards(nranks, rank, shards, fulls, shard_rows, False)


def _xent_overlap(a, b) -> bool:
    return a[1] > 0 and b[1] > 0 and a[0] < b[0] + b[1] and b[0] < a[0] + a[1]


def check_vocab_parallel_cross_entropy(nranks: int, logits, target, loss=None, lse=None, dloss=None, grad=None) -> tuple[int, int]:
    """The rules of Comm.vocab_parallel_cross_entropy (and, with dloss given, of its backward), checked on the tensors' metadata (no
    device, no communicator), as xent_check in coll/src/xent.cu: raises ValueError, returns (rows, vocab_local). logits: a contiguous
    [rows, Vl] bfloat16, float16 or float32 tensor, Vl > 0 and Vl * itemsize a multiple of 16 bytes, nranks * Vl < 2^31, rows < 2^31;
    target: contiguous [rows] int64; loss, lse, dloss: contiguous [rows] float32; grad: logits' dtype and shape. Alignment: logits and
    grad 16 bytes, target 8, the float32 arrays 4. No output (loss and lse; grad) may overlap an input or another output, except
    grad is logits (the in-place backward)."""
    import torch
    what = "vocab_parallel_cross_entropy" + ("_backward" if dloss is not None else "")
    if logits.dtype not in (torch.bfloat16, torch.float16, torch.float32):
        raise ValueError(f"{what}: logits must be bfloat16, float16 or float32, got {logits.dtype}")
    if logits.dim() != 2 or not logits.is_contiguous():
        raise ValueError(f"{what}: logits must be a contiguous [rows, vocab_local] tensor, got shape {list(logits.shape)}")
    rows, vl = logits.shape
    es = logits.element_size()
    if vl == 0 or (vl * es) % 16:
        raise ValueError(f"{what}: vocab_local must be positive and vocab_local * itemsize a multiple of 16 bytes, got {vl} x {es}")
    if nranks * vl >= 2 ** 31:
        raise ValueError(f"{what}: nranks * vocab_local must be below 2^31, got {nranks} x {vl}")
    if rows >= 2 ** 31:
        raise ValueError(f"{what}: rows must be below 2^31, got {rows}")
    if target.dtype != torch.int64 or tuple(target.shape) != (rows,) or not target.is_contiguous():
        raise ValueError(f"{what}: target must be a contiguous [{rows}] int64 tensor, got {target.dtype} {list(target.shape)}")
    f32 = {"loss": loss, "lse": lse, "dloss": dloss}
    for name, t in f32.items():
        if t is not None and (t.dtype != torch.float32 or tuple(t.shape) != (rows,) or not t.is_contiguous()):
            raise ValueError(f"{what}: {name} must be a contiguous [{rows}] float32 tensor, got {t.dtype} {list(t.shape)}")
    if grad is not None and (grad.dtype != logits.dtype or tuple(grad.shape) != (rows, vl) or not grad.is_contiguous()):
        raise ValueError(f"{what}: grad must be a contiguous {logits.dtype} [{rows}, {vl}] tensor, got {grad.dtype} {list(grad.shape)}")
    if logits.data_ptr() % 16 or (grad is not None and grad.data_ptr() % 16):
        raise ValueError(f"{what}: logits and grad must be 16-byte aligned")
    if target.data_ptr() % 8:
        raise ValueError(f"{what}: target must be 8-byte aligned")
    if any(t is not None and t.data_ptr() % 4 for t in f32.values()):
        raise ValueError(f"{what}: loss, lse and dloss must be 4-byte aligned")
    if rows:
        span = lambda t: (t.data_ptr(), t.numel() * t.element_size())     # noqa: E731
        ins = [span(logits), span(target)]
        if dloss is not None:
            outs, ins = [span(grad)] if grad is not None else [], ins + [span(lse), span(dloss)]
        else:
            outs = [span(t) for t in (loss, lse) if t is not None]
        for i, o in enumerate(outs):
            for j, x in enumerate(ins):
                if _xent_overlap(o, x) and not (dloss is not None and j == 0 and o == x):
                    raise ValueError(f"{what}: outputs must not overlap the inputs (grad is logits is the one overlap allowed)")
            for o2 in outs[i + 1:]:
                if _xent_overlap(o, o2):
                    raise ValueError(f"{what}: outputs must not overlap each other")
    return rows, vl


def check_vocab_parallel_embedding(nranks: int, ids, table, rows=None, *, sequence_parallel: bool = False, backward: bool = False,
                                   symmetric=None) -> tuple[int, int, int]:
    """The rules of Comm.vocab_parallel_embedding (table = weight, rows = out) and, with backward=True, of its backward (table =
    dweight, rows = grad_out), checked on the tensors' metadata as emb_check in coll/src/embedding.cu: raises ValueError, returns (T, H,
    Vl). ids: contiguous [T] int64, T < 2^31 and, under sequence parallelism, a multiple of nranks. table: contiguous [Vl, H], Vl > 0,
    nranks * Vl < 2^31; weight bfloat16, float16 or float32; dweight float32 or grad_out's dtype. rows: contiguous [T / nranks or T, H]
    (bfloat16, float16 or float32, weight's dtype in the forward). H > 0 and H * itemsize a multiple of 16 bytes for every dtype; at most
    2^31 - 1 16-byte vectors in each tensor. Alignment: ids 8 bytes, the others 16. out must not overlap weight or ids, dweight not
    grad_out or ids. symmetric(tensor) -> bool, given with nranks > 1: weight (forward) or the sequence-parallel grad_out (backward) must
    be arena memory when T > 0."""
    import torch
    what = "vocab_parallel_embedding" + ("_backward" if backward else "")
    wide = (torch.bfloat16, torch.float16, torch.float32)
    if ids.dtype != torch.int64 or ids.dim() != 1 or not ids.is_contiguous():
        raise ValueError(f"{what}: ids must be a contiguous [tokens] int64 tensor, got {ids.dtype} {list(ids.shape)}")
    T = ids.shape[0]
    if table.dim() != 2 or not table.is_contiguous():
        raise ValueError(f"{what}: {'dweight' if backward else 'weight'} must be a contiguous [vocab_local, hidden] tensor, got shape {list(table.shape)}")
    vl, h = table.shape
    rdt = rows.dtype if rows is not None else table.dtype
    if rdt not in wide or (not backward and table.dtype not in wide):
        raise ValueError(f"{what}: {'grad_out' if backward else 'weight'} must be bfloat16, float16 or float32, got {rdt if backward else table.dtype}")
    if backward and table.dtype not in (torch.float32, rdt):
        raise ValueError(f"{what}: dweight must be float32 or grad_out's dtype {rdt}, got {table.dtype}")
    if not backward and rows is not None and rows.dtype != table.dtype:
        raise ValueError(f"{what}: out must have weight's dtype {table.dtype}, got {rows.dtype}")
    ers, ets = torch.empty((), dtype=rdt).element_size(), table.element_size()
    if h == 0 or (h * ers) % 16 or (h * ets) % 16:
        raise ValueError(f"{what}: hidden must be positive and hidden * itemsize a multiple of 16 bytes for every dtype, got {h}")
    if vl == 0:
        raise ValueError(f"{what}: vocab_local must be positive")
    if nranks * vl >= 2 ** 31:
        raise ValueError(f"{what}: nranks * vocab_local must be below 2^31, got {nranks} x {vl}")
    if T >= 2 ** 31:
        raise ValueError(f"{what}: tokens must be below 2^31, got {T}")
    if sequence_parallel and T % nranks:
        raise ValueError(f"{what}: tokens must be a multiple of nranks under sequence parallelism, got {T} and {nranks}")
    nr = T // nranks if sequence_parallel else T
    if max(nr * h * ers, vl * h * ers, vl * h * ets) // 16 > 2 ** 31 - 1:
        raise ValueError(f"{what}: more than 2^31 - 1 16-byte vectors in one tensor")
    if rows is not None and (tuple(rows.shape) != (nr, h) or not rows.is_contiguous()):
        raise ValueError(f"{what}: {'grad_out' if backward else 'out'} must be a contiguous [{nr}, {h}] tensor, got {list(rows.shape)}")
    if ids.data_ptr() % 8:
        raise ValueError(f"{what}: ids must be 8-byte aligned")
    if table.data_ptr() % 16 or (rows is not None and rows.data_ptr() % 16):
        raise ValueError(f"{what}: {'dout and dweight' if backward else 'weight and out'} must be 16-byte aligned")
    if T and rows is not None:
        span = lambda t: (t.data_ptr(), t.numel() * t.element_size())     # noqa: E731
        o, ins = (span(table), [span(rows), span(ids)]) if backward else (span(rows), [span(table), span(ids)])
        if any(_xent_overlap(o, x) for x in ins):
            raise ValueError(f"{what}: " + ("dweight must not overlap dout or ids" if backward else "out must not overlap weight or ids"))
    if nranks > 1 and T and symmetric is not None and (not backward or sequence_parallel):
        t = rows if backward else table
        if t is not None and not symmetric(t):
            raise ValueError(f"{what}: {'grad_out' if backward else 'weight'} must lie in the symmetric arena (Comm.empty), at the same offset on every rank")
    return T, h, vl


def _check_routed(nranks: int, x, topk_idx, num_experts: int, recv, expert_counts, route, dropped, fp8=None) -> None:
    """The rules of both device-routed dispatches; fp8 is None (check_expert_dispatch) or (recv_scales, block), which adds the FP8
    call's rules, as routed_prepare in coll/src/dispatch.cu takes a RoutedQuant."""
    import torch
    _check_wide("x", x, rows=True)
    tokens, row_elems = x.shape
    if fp8 is None:
        if row_elems <= 0 or row_elems % 16:
            raise ValueError(f"row_elems (x.shape[1] = {row_elems}) must be a positive multiple of 16")
    else:
        recv_scales, block = fp8
        _check_block(block)
        if row_elems <= 0 or row_elems % block:
            raise ValueError(f"row_elems (x.shape[1] = {row_elems}) must be a positive multiple of block ({block})")
    _check_topk("topk_idx", topk_idx)
    if topk_idx.shape[0] != tokens:
        raise ValueError(f"topk_idx has {topk_idx.shape[0]} tokens, x has {tokens}")
    top_k = topk_idx.shape[1]
    if isinstance(num_experts, bool) or not isinstance(num_experts, int) or not 1 <= num_experts <= MAX_EXPERTS or num_experts % nranks:
        raise ValueError(f"num_experts must be an int in [1, {MAX_EXPERTS}] and a multiple of nranks ({nranks}), got {num_experts!r}")
    inputs = [("topk_idx", topk_idx), ("x", x), ("recv", recv)]
    if fp8 is None:
        if recv.dtype != x.dtype or not recv.is_contiguous() or recv.numel() % row_elems:
            raise ValueError(f"recv must be a contiguous {x.dtype} tensor of whole {row_elems}-element rows, got {recv.dtype} with {recv.numel()} elements")
    else:
        if recv.dtype not in (torch.float8_e4m3fn, torch.float8_e5m2) or not recv.is_contiguous() or recv.numel() % row_elems:
            raise ValueError(f"recv must be a contiguous float8_e4m3fn or float8_e5m2 tensor (the wire type) of whole {row_elems}-element rows, "
                             f"got {recv.dtype} with {recv.numel()} elements")
        if recv_scales.dtype != torch.float32 or not recv_scales.is_contiguous() or recv_scales.numel() != recv.numel() // block:
            raise ValueError(f"recv_scales must be a contiguous float32 tensor of recv.numel() // block = {recv.numel() // block} elements, "
                             f"got {recv_scales.dtype} with {recv_scales.numel()}")
        inputs.append(("recv_scales", recv_scales))
    if tokens * top_k > _I31:
        raise ValueError(f"tokens * top_k ({tokens * top_k}) must be at most 2^31 - 1")
    if nranks * (recv.numel() // row_elems) > _I31:
        raise ValueError("nranks * recv rows must be at most 2^31 - 1 (a route is an int32)")
    if fp8 is not None and tokens * (row_elems // 16) > _I31:
        raise ValueError("at most 2^31 - 1 16-element vectors of x (tokens * row_elems / 16)")
    if tokens * top_k * (row_elems * x.element_size() // 16) > _I31:
        raise ValueError("at most 2^31 - 1 16-byte vectors may be offered (tokens * top_k * row bytes / 16)")
    for an, bn in [("recv", "x")] + ([("recv_scales", "x"), ("recv", "recv_scales")] if fp8 is not None else []):
        if _overlap(dict(inputs)[an], dict(inputs)[bn]):
            raise ValueError(f"{an} must not overlap {bn}")
    outs = [(n, t, shape) for n, t, shape in (("expert_counts", expert_counts, (num_experts // nranks,)), ("route", route, (tokens, top_k)),
                                              ("dropped", dropped, (1,))) if t is not None]
    for name, t, shape in outs:
        if t.dtype != torch.int32 or not t.is_contiguous() or t.numel() != _numel(shape):
            raise ValueError(f"{name} must be a contiguous int32 tensor of shape {shape}, got {t.dtype}{list(t.shape)}")
    for k, (name, t, _) in enumerate(outs):
        for other, u in [(n, o) for n, o, _ in outs[k + 1:]] + inputs:
            if _overlap(t, u):
                raise ValueError(f"{name} must not overlap {other}")


def check_expert_dispatch(nranks: int, x, topk_idx, num_experts: int, recv, expert_counts=None, route=None, dropped=None) -> int:
    """Rules of the device-routed expert dispatch, checked on the tensors' metadata only (no communicator, no library call, no device
    read): raises ValueError, returns the library code of x's type. x: contiguous bfloat16, float16 or float32 [tokens, row_elems] with
    row_elems a positive multiple of 16; topk_idx: contiguous int32 [tokens, top_k], top_k >= 1; num_experts in [1, MAX_EXPERTS] and a
    multiple of nranks; recv: contiguous, x's dtype, a whole number of rows; expert_counts (num_experts // nranks), route (tokens, top_k)
    and dropped (1 element): contiguous int32 when given. tokens * top_k, nranks * recv rows and tokens * top_k * row bytes / 16 are at
    most 2^31 - 1. recv must not overlap x, and no output may overlap another output, topk_idx, x or recv."""
    _check_routed(nranks, x, topk_idx, num_experts, recv, expert_counts, route, dropped)
    return torch_dtype_code(x.dtype)


def check_expert_dispatch_quantized(nranks: int, x, topk_idx, num_experts: int, recv, recv_scales, block: int, expert_counts=None, route=None,
                                    dropped=None) -> tuple[int, int]:
    """Rules of the device-routed expert dispatch with FP8 on the wire, checked on the tensors' metadata only (no communicator, no
    library call, no device read): raises ValueError, returns the library codes of (x's type, the wire type). x, topk_idx, num_experts,
    expert_counts, route and dropped as in check_expert_dispatch; block one of QUANT_BLOCKS and row_elems (x.shape[1]) a positive multiple
    of it; recv: contiguous float8_e4m3fn or float8_e5m2 (the wire type) of whole rows; recv_scales: contiguous float32 with
    recv.numel() // block elements. tokens * top_k, nranks * recv rows, tokens * row_elems / 16 (the 16-element vectors of x) and
    tokens * top_k * row bytes / 16 are at most 2^31 - 1. x, recv and recv_scales must not overlap, and no output may overlap another
    output, topk_idx, x, recv or recv_scales."""
    _check_routed(nranks, x, topk_idx, num_experts, recv, expert_counts, route, dropped, fp8=(recv_scales, block))
    return torch_dtype_code(x.dtype), torch_dtype_code(recv.dtype)


def _check_expert_combine(nranks: int, expert_out, route, weights, out, fp8=None) -> tuple:
    """The rules of both expert combines; fp8 is None (check_expert_combine) or (block, wire), which adds the quantising call's rules."""
    import torch
    _check_wide("out", out, rows=True)
    tokens, row_elems = out.shape
    if fp8 is not None:
        wc = _check_combine_quant(fp8, row_elems)
    elif row_elems <= 0 or row_elems % 16:
        raise ValueError(f"row_elems (out.shape[1] = {row_elems}) must be a positive multiple of 16")
    if expert_out.dtype not in (torch.bfloat16, torch.float16, torch.float32) or not expert_out.is_contiguous() or expert_out.numel() % row_elems:
        raise ValueError(f"expert_out must be a contiguous bfloat16, float16 or float32 tensor of whole {row_elems}-element rows, got {expert_out.dtype}")
    if route.dtype != torch.int32 or route.dim() != 2 or not route.is_contiguous() or route.shape[1] < 1 or route.shape[0] != tokens:
        raise ValueError(f"route must be a contiguous int32 [{tokens}, top_k] tensor with top_k >= 1, got {route.dtype}{list(route.shape)}")
    if weights is not None and (weights.dtype != torch.float32 or weights.shape != route.shape or not weights.is_contiguous()):
        raise ValueError(f"weights must be None or a contiguous float32 {list(route.shape)} tensor, got {weights.dtype}{list(weights.shape)}")
    if tokens * route.shape[1] > _I31:
        raise ValueError("tokens * top_k must be at most 2^31 - 1")
    if nranks * (expert_out.numel() // row_elems) > _I31:
        raise ValueError("nranks * expert_out rows must be at most 2^31 - 1 (a route is an int32)")
    if fp8 is not None:
        _check_combine_sizes(tokens, route.shape[1], row_elems, expert_out.numel() // row_elems)
    for name, t in (("expert_out", expert_out), ("route", route), ("weights", weights)):
        if t is not None and _overlap(out, t):
            raise ValueError(f"out must not overlap {name}")
    codes = (torch_dtype_code(expert_out.dtype), torch_dtype_code(out.dtype))
    return codes if fp8 is None else codes + (wc,)


def check_expert_combine(nranks: int, expert_out, route, weights, out) -> tuple[int, int]:
    """Rules of the expert combine from a device route, checked on the tensors' metadata only: raises ValueError, returns the library
    codes of (expert_out's type, out's type). out: contiguous bfloat16, float16 or float32 [tokens, row_elems], row_elems a positive
    multiple of 16; expert_out: contiguous bfloat16, float16 or float32 of whole rows; route: contiguous int32 [tokens, top_k], top_k >= 1;
    weights: None or contiguous float32 of route's shape. nranks * expert_out rows is at most 2^31 - 1. out must not overlap expert_out,
    route or weights."""
    return _check_expert_combine(nranks, expert_out, route, weights, out)


def check_expert_combine_quantized(nranks: int, expert_out, route, weights, out, block: int = 128, wire=None) -> tuple[int, int, int]:
    """Rules of the quantising expert combine from a device route, checked on the tensors' metadata only: raises ValueError, returns the
    library codes of (expert_out's type, out's type, the wire type). Everything check_expert_combine checks, and: wire
    torch.float8_e4m3fn (None, the default) or torch.float8_e5m2; block one of QUANT_BLOCKS and row_elems (out.shape[1]) a positive
    multiple of it; tokens * row_elems / 16 and expert_out.numel() / 16 at most 2^31 - 1."""
    return _check_expert_combine(nranks, expert_out, route, weights, out, fp8=(block, wire))


class _CudaArray:
    """Minimal __cuda_array_interface__ carrier so torch can alias arena memory without a copy."""

    def __init__(self, ptr: int, nbytes: int, owner):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}
        self._owner = owner


@dataclass
class SymBuffer:
    ptr: int
    nbytes: int


class Comm:
    """One communicator rank. `Comm.from_env()` under torchrun; `Comm.init_all()` for in-process groups."""

    def __init__(self, handle: int, owner_group=None):
        self._h = C.c_void_p(handle)
        self._group = owner_group
        self._allocs: dict[int, int] = {}
        info = CommInfo()
        _check(load().b200collCommInfoGet(self._h, C.byref(info)), "CommInfoGet")
        self.rank, self.nranks, self.device, self.nvls = info.rank, info.nranks, info.device, bool(info.nvls)
        self.loopback = bool(info.same_device_loopback)
        self.sm_count = info.sm_count

    # ---------------------------------------------------------------- construction
    @staticmethod
    def make_config(arena_mb: Optional[int] = None, nvls: Optional[int] = None, timeout_ms: Optional[int] = None) -> Config:
        cfg = Config()
        load().b200collConfigDefault(C.byref(cfg))
        if arena_mb is not None:
            cfg.arena_bytes = int(arena_mb) << 20
        if nvls is not None:
            cfg.enable_nvls = nvls
        if timeout_ms is not None:
            cfg.timeout_ms = timeout_ms
        return cfg

    @classmethod
    def from_env(cls, arena_mb: Optional[int] = None, tag: str = "0", **kw) -> "Comm":
        """torchrun-style: RANK / WORLD_SIZE / LOCAL_RANK / MASTER_ADDR / MASTER_PORT. The caller has already
        selected its GPU (torch.cuda.set_device(LOCAL_RANK))."""
        rank = int(os.environ.get("RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1"))
        key = f"{os.environ.get('MASTER_ADDR', '127.0.0.1')}:{os.environ.get('MASTER_PORT', '0')}/{os.environ.get('TORCHELASTIC_RUN_ID', '')}/{tag}"
        return cls.init_rank(rank, world, key, arena_mb=arena_mb, **kw)

    @classmethod
    def init_rank(cls, rank: int, nranks: int, key: str, arena_mb: Optional[int] = None, **kw) -> "Comm":
        L = load()
        uid = UniqueId()
        _check(L.b200collUniqueIdFromString(key.encode(), C.byref(uid)), "UniqueIdFromString")
        cfg = cls.make_config(arena_mb, **kw)
        h = C.c_void_p()
        _check(L.b200collCommInitRank(C.byref(h), nranks, C.byref(uid), rank, C.byref(cfg)), "CommInitRank")
        return cls(h.value)

    @classmethod
    def init_all(cls, devices: list[int], arena_mb: Optional[int] = None, **kw) -> list["Comm"]:
        L = load()
        n = len(devices)
        hs = (C.c_void_p * n)()
        devs = (C.c_int * n)(*devices)
        cfg = cls.make_config(arena_mb, **kw)
        _check(L.b200collCommInitAll(hs, n, devs, C.byref(cfg)), "CommInitAll")
        return [cls(hs[i]) for i in range(n)]

    def mem_pool(self):
        """A `torch.cuda.MemPool` whose memory is this communicator's symmetric arena (PyTorch's pluggable-allocator hook calling
        b200collMemAlloc). Tensors created under `torch.cuda.use_mem_pool(pool)` — a model's parameters, DDP's gradient buckets with
        `gradient_as_bucket_view=True` — are then arena tensors: collectives on them skip staging and may use NVLS. Every rank must
        allocate the same sizes in the same order inside the pool (SPMD code does). One pool-backed communicator per process."""
        import torch
        from torch.cuda.memory import CUDAPluggableAllocator
        if getattr(self, "_pool", None) is None:
            _check(load().b200collSetAllocatorComm(self._h), "SetAllocatorComm")
            self._pool_allocator = CUDAPluggableAllocator(lib_path(), "b200collTorchAlloc", "b200collTorchFree")
            self._pool = torch.cuda.MemPool(self._pool_allocator.allocator())
        return self._pool

    def split(self, color: int, key: int = 0, arena_mb: Optional[int] = None, **kw) -> Optional["Comm"]:
        """ncclCommSplit: every rank of this (multi-process) communicator calls it; ranks with the same color >= 0 get a new communicator
        with its own arena, ordered by (key, rank here). A negative color takes part and returns None. Tensor-parallel and data-parallel
        groups of one job are two splits of the world communicator."""
        cfg = self.make_config(arena_mb, **kw) if (arena_mb is not None or kw) else None
        h = C.c_void_p()
        _check(load().b200collCommSplit(self._h, color, key, C.byref(h), C.byref(cfg) if cfg is not None else None), "CommSplit")
        return type(self)(h.value) if h.value else None

    def destroy(self) -> None:
        if self._h:
            load().b200collCommDestroy(self._h)
            self._h = None

    # ---------------------------------------------------------------- memory
    def alloc(self, nbytes: int) -> SymBuffer:
        p = C.c_void_p()
        _check(load().b200collMemAlloc(self._h, C.byref(p), nbytes), "MemAlloc")
        self._allocs[p.value] = nbytes
        return SymBuffer(p.value, nbytes)

    def free(self, buf: SymBuffer) -> None:
        _check(load().b200collMemFree(self._h, C.c_void_p(buf.ptr)), "MemFree")
        self._allocs.pop(buf.ptr, None)

    def empty(self, numel: int, dtype):
        """A torch tensor living in the symmetric arena (zero-copy fast paths, NVLS capable)."""
        import torch
        itemsize = torch.empty((), dtype=dtype).element_size()
        buf = self.alloc(numel * itemsize)
        raw = torch.as_tensor(_CudaArray(buf.ptr, buf.nbytes, self), device=torch.device("cuda", self.device))
        t = raw.view(dtype)[:numel]
        t._b200coll_buf = buf   # keep the allocation discoverable
        return t

    def release(self, tensor) -> None:
        """Give a tensor from `empty()` back to the arena. Explicit on purpose: allocation is a collective contract (same order and
        sizes on every rank keep the offsets identical), so it must not depend on when each rank's garbage collector runs.
        The caller guarantees no collective is still using the tensor."""
        buf = getattr(tensor, "_b200coll_buf", None)
        if buf is None:
            raise ValueError("tensor was not allocated with Comm.empty()")
        self.free(buf)
        tensor._b200coll_buf = None

    def is_symmetric(self, tensor) -> bool:
        return bool(load().b200collIsSymmetric(self._h, C.c_void_p(tensor.data_ptr()), tensor.numel() * tensor.element_size()))

    # ---------------------------------------------------------------- collectives (tensors)
    @staticmethod
    def _stream(stream) -> C.c_void_p:
        import torch
        s = stream if stream is not None else torch.cuda.current_stream()
        return C.c_void_p(s.cuda_stream)

    def _ep(self, src, dst, scale: float) -> Epilogue:
        return Epilogue(torch_dtype_code(src.dtype), torch_dtype_code(dst.dtype), float(scale))

    def all_reduce(self, src, dst=None, scale: float = 1.0, op: int = SUM, stream=None):
        dst = src if dst is None else dst
        ep = self._ep(src, dst, scale)
        _check(load().b200collAllReduce(C.c_void_p(src.data_ptr()), C.c_void_p(dst.data_ptr()), src.numel(), C.byref(ep), op, self._h, self._stream(stream)), "AllReduce")
        return dst

    def all_reduce_from_host(self, host_in, out, chunk_bytes: int = 32 << 20, scale: float = 1.0, op: int = SUM, stream=None):
        """End-to-end step: `out` (device, ideally from `empty()`) = all-reduce of every rank's pinned host tensor `host_in`.
        The host→device copy is pipelined with the collective: chunk i+1 crosses PCIe on a copy stream while chunk i is reduced out
        of one of two arena staging buffers, so the step costs about the copy time instead of copy + collective. Same call (sizes,
        chunking) on every rank. EXPERIMENTAL: composed from validated pieces (copies, events, `all_reduce`) but not yet timed on hardware."""
        import torch
        assert host_in.device.type == "cpu" and out.is_cuda and host_in.numel() == out.numel() and host_in.is_contiguous() and out.is_contiguous()
        main = stream if stream is not None else torch.cuda.current_stream()
        itemsize = host_in.element_size()
        chunk = max(1, chunk_bytes // itemsize // 64 * 64)
        if not hasattr(self, "_h2d"):
            self._h2d = {"stream": torch.cuda.Stream(), "bufs": {}, "ready": [torch.cuda.Event(), torch.cuda.Event()], "free": [torch.cuda.Event(), torch.cuda.Event()]}
        st = self._h2d
        key = (chunk, host_in.dtype)
        if key not in st["bufs"]:
            st["bufs"][key] = [self.empty(chunk, host_in.dtype), self.empty(chunk, host_in.dtype)]
        bufs, ready, free, copy_stream = st["bufs"][key], st["ready"], st["free"], st["stream"]
        copy_stream.wait_stream(main)                       # staging buffers may still be in use by earlier work on the caller's stream
        n_total, flat_in, flat_out = host_in.numel(), host_in.view(-1), out.view(-1)
        for i, off in enumerate(range(0, n_total, chunk)):
            k, n = i & 1, min(chunk, n_total - off)
            with torch.cuda.stream(copy_stream):
                if i >= 2:
                    copy_stream.wait_event(free[k])         # the collective that read this staging buffer two chunks ago is done
                bufs[k][:n].copy_(flat_in[off:off + n], non_blocking=True)
                ready[k].record(copy_stream)
            main.wait_event(ready[k])
            self.all_reduce(bufs[k][:n], flat_out[off:off + n], scale=scale, op=op, stream=main)
            free[k].record(main)
        return out

    def host_empty(self, numel: int, dtype):
        """A pinned, device-mapped CPU tensor on the NUMA node of this rank's GPU (b200collHostAlloc): the buffer to hand to
        `all_reduce_host`. On a two-socket 8-GPU box this placement is what keeps eight concurrent host<->device copies at link rate."""
        import torch
        itemsize = torch.empty((), dtype=dtype).element_size()
        nbytes = max(1, numel * itemsize)
        p = C.c_void_p()
        _check(load().b200collHostAlloc(self._h, C.byref(p), nbytes), "HostAlloc")
        raw = (C.c_uint8 * nbytes).from_address(p.value)
        t = torch.frombuffer(raw, dtype=torch.uint8).view(dtype)[:numel]
        t._b200coll_host = p.value
        self._host_allocs = getattr(self, "_host_allocs", {})
        self._host_allocs[p.value] = raw
        return t

    def host_release(self, tensor) -> None:
        p = getattr(tensor, "_b200coll_host", None)
        if p is None:
            raise ValueError("tensor was not allocated with Comm.host_empty()")
        _check(load().b200collHostFree(self._h, C.c_void_p(p)), "HostFree")
        self._host_allocs.pop(p, None)
        tensor._b200coll_host = None

    def numa(self) -> tuple[int, str]:
        """(NUMA node of this rank's GPU or -1, its local CPU list as sysfs prints it)."""
        node = C.c_int(-1)
        buf = C.create_string_buffer(256)
        _check(load().b200collCommNumaGet(self._h, C.byref(node), buf, len(buf)), "CommNumaGet")
        return node.value, buf.value.decode()

    def all_reduce_host(self, host_in, host_out=None, scale: float = 1.0, op: int = SUM, stream=None):
        """The end-to-end step as one library call: `host_out` (pinned CPU tensor, default in place) = cast(scale * sum over ranks
        of `host_in`). Asynchronous on `stream`; tiny messages run as one zero-copy kernel over PCIe, large ones are chunked so that
        the copy in, the all-reduce and the copy back overlap (b200collAllReduceHost, coll/src/hostpath.cu). Same call on every rank."""
        host_out = host_in if host_out is None else host_out
        assert host_in.device.type == "cpu" and host_out.device.type == "cpu" and host_in.is_contiguous() and host_out.is_contiguous()
        assert host_in.numel() == host_out.numel()
        ep = self._ep(host_in, host_out, scale)
        _check(load().b200collAllReduceHost(C.c_void_p(host_in.data_ptr()), C.c_void_p(host_out.data_ptr()), host_in.numel(), C.byref(ep), op, self._h,
                                            self._stream(stream)), "AllReduceHost")
        return host_out

    def all_gather(self, src, dst, scale: float = 1.0, stream=None):
        ep = self._ep(src, dst, scale)
        _check(load().b200collAllGather(C.c_void_p(src.data_ptr()), C.c_void_p(dst.data_ptr()), src.numel(), C.byref(ep), self._h, self._stream(stream)), "AllGather")
        return dst

    def reduce_scatter(self, src, dst, scale: float = 1.0, op: int = SUM, stream=None):
        ep = self._ep(src, dst, scale)
        _check(load().b200collReduceScatter(C.c_void_p(src.data_ptr()), C.c_void_p(dst.data_ptr()), dst.numel(), C.byref(ep), op, self._h, self._stream(stream)), "ReduceScatter")
        return dst

    def _block_scaled(self, what, fn, op_name, q, scales, out, block, scale, extra, count, stream):
        br, bc = check_block_scaled(op_name, self.nranks, q, scales, out, block)
        bs = BlockScale(scales.data_ptr(), q.shape[1], br, bc)
        ep = self._ep(q, out, scale)
        _check(fn(C.c_void_p(q.data_ptr()), C.c_void_p(out.data_ptr()), count, C.byref(bs), C.byref(ep), *extra, self._h, self._stream(stream)), what)
        return out

    def all_gather_block_scaled(self, q, scales, out, block=(1, 128), scale: float = 1.0, stream=None):
        """out[r-th shard] = round(scale * dequant(q of rank r)), dequant = float(q) times the fp32 scale of its block_rows x block_cols
        block. q [rows, row_len] FP8 and scales (ceil(rows/br), ceil(row_len/bc)) fp32 must be arena tensors (`empty()`); out is bf16,
        fp16 or fp32 of shape (nranks*rows, row_len). FP8 and scales cross NVLink; the receiver dequantises (b200collAllGatherBlockScaled)."""
        return self._block_scaled("AllGatherBlockScaled", load().b200collAllGatherBlockScaled, "all_gather", q, scales, out, block, scale, (), q.numel(), stream)

    def reduce_scatter_block_scaled(self, q, scales, out, block=(1, 128), scale: float = 1.0, op: int = SUM, stream=None):
        """out = round(scale * sum over ranks, in rank order, of dequant(row slice `rank` of q)); op SUM or AVG; out (rows/nranks, row_len)."""
        return self._block_scaled("ReduceScatterBlockScaled", load().b200collReduceScatterBlockScaled, "reduce_scatter", q, scales, out, block, scale, (op,),
                                  q.numel() // self.nranks, stream)

    def all_reduce_block_scaled(self, q, scales, out, block=(1, 128), scale: float = 1.0, op: int = SUM, stream=None):
        """out = round(scale * sum over ranks, in rank order, of dequant(q)); op SUM or AVG; out (rows, row_len). Two-shot needs out in the arena."""
        return self._block_scaled("AllReduceBlockScaled", load().b200collAllReduceBlockScaled, "all_reduce", q, scales, out, block, scale, (op,), q.numel(), stream)

    def all_gather_quantized(self, src, out, block: int = 128, wire=None, scale: float = 1.0, stream=None):
        """out[r-th shard] = round(scale * dequant(quant(src of rank r))): src (bf16, fp16 or fp32, any device tensor) is quantised on
        this rank to `wire` FP8 with one fp32 scale per `block` elements, and FP8 and scales cross NVLink (b200collAllGatherQuantized).
        out: bf16, fp16 or fp32 with nranks * src.numel() elements. The scratch comes from the arena: the same calls on every rank."""
        w = check_quantized("all_gather", self.nranks, src, out, block, wire)
        ep = self._ep(src, out, scale)
        _check(load().b200collAllGatherQuantized(C.c_void_p(src.data_ptr()), C.c_void_p(out.data_ptr()), src.numel(), w, block, C.byref(ep), self._h,
                                                 self._stream(stream)), "AllGatherQuantized")
        return out

    def reduce_scatter_quantized(self, src, out, block: int = 128, wire=None, scale: float = 1.0, op: int = SUM, stream=None):
        """out = round(scale * sum over ranks, in rank order, of dequant(quant(slice `rank` of src))); op SUM or AVG; out has
        src.numel() / nranks elements, a multiple of block."""
        w = check_quantized("reduce_scatter", self.nranks, src, out, block, wire)
        ep = self._ep(src, out, scale)
        _check(load().b200collReduceScatterQuantized(C.c_void_p(src.data_ptr()), C.c_void_p(out.data_ptr()), out.numel(), w, block, C.byref(ep), op, self._h,
                                                     self._stream(stream)), "ReduceScatterQuantized")
        return out

    def all_reduce_quantized(self, src, out=None, block: int = 128, wire=None, scale: float = 1.0, op: int = SUM, stream=None):
        """out = round(scale * sum over ranks, in rank order, of dequant(quant(src))); op SUM or AVG; out=None runs in place. Two-shot
        needs out in the arena (`empty()`), else the call runs one-shot."""
        out = src if out is None else out
        w = check_quantized("all_reduce", self.nranks, src, out, block, wire)
        ep = self._ep(src, out, scale)
        _check(load().b200collAllReduceQuantized(C.c_void_p(src.data_ptr()), C.c_void_p(out.data_ptr()), src.numel(), w, block, C.byref(ep), op, self._h,
                                                 self._stream(stream)), "AllReduceQuantized")
        return out

    def all_reduce_rms_norm(self, x, residual, weight, out=None, eps: float = 1e-6, stream=None):
        """The pre-norm step of a tensor-parallel block in one kernel: residual += all_reduce(x) in place (ranks summed in rank order,
        one rounding), then out = rms_norm(residual, weight, eps), bit for bit as coll/include/b200coll.h's b200collAllReduceRmsNorm
        states. Returns out (a new tensor when None). With more than one rank x must be arena memory (`empty()`); two-shot also needs
        residual and out there, else the call runs one-shot."""
        out = x.new_empty(x.shape) if out is None else out
        rows, row_len = check_all_reduce_rms_norm(x, residual, weight, out, eps)
        _check(load().b200collAllReduceRmsNorm(C.c_void_p(x.data_ptr()), C.c_void_p(residual.data_ptr()), C.c_void_p(weight.data_ptr()),
                                               C.c_void_p(out.data_ptr()), rows, row_len, float(eps), torch_dtype_code(x.dtype), self._h,
                                               self._stream(stream)), "AllReduceRmsNorm")
        return out

    def all_reduce_rms_norm_quantized(self, x, residual, weight, q=None, scales=None, block: int = 128, wire=None, eps: float = 1e-6,
                                      stream=None):
        """all_reduce_rms_norm with its out quantised for an FP8 GEMM, in one kernel: residual += all_reduce(x) in place, then
        o = rms_norm(residual, weight, eps) as all_reduce_rms_norm would store it, quantised per 1 x `block` group of each row to `wire`
        (torch.float8_e4m3fn by default, or torch.float8_e5m2) with one fp32 scale per group, bit for bit as coll/include/b200coll.h's
        b200collAllReduceRmsNormQuantized states. Returns (q, scales): q of x's shape and the wire dtype, scales float32
        [..., row_len // block] (new tensors when None). With more than one rank x must be arena memory (`empty()`); two-shot also needs
        residual, q and scales there, else the call runs one-shot."""
        import torch
        w = torch.float8_e4m3fn if wire is None else wire
        q = x.new_empty(x.shape, dtype=w) if q is None else q
        if scales is None:
            _check_block(block)
            scales = x.new_empty(tuple(x.shape[:-1]) + ((x.shape[-1] if x.dim() else 0) // block,), dtype=torch.float32)
        rows, row_len, wc = check_all_reduce_rms_norm_quantized(x, residual, weight, q, scales, block, wire, eps)
        _check(load().b200collAllReduceRmsNormQuantized(C.c_void_p(x.data_ptr()), C.c_void_p(residual.data_ptr()), C.c_void_p(weight.data_ptr()),
                                                        C.c_void_p(q.data_ptr()), C.cast(C.c_void_p(scales.data_ptr()), C.POINTER(C.c_float)), rows,
                                                        row_len, float(eps), torch_dtype_code(x.dtype), wc, block, self._h, self._stream(stream)),
               "AllReduceRmsNormQuantized")
        return q, scales

    def reduce_scatter_rms_norm(self, x, residual, weight, out=None, eps: float = 1e-6, gather: bool = False, stream=None):
        """The sequence-parallel pre-norm step in one kernel: x's rows are summed over the ranks, and this rank keeps its slice of dim 0
        (rows [rank * S, (rank + 1) * S), S = x.shape[0] // nranks). residual, this rank's [S, ...] shard of the residual stream, gets
        that slice added in place, then out = rms_norm(residual, weight, eps), bit for bit as coll/include/b200coll.h's
        b200collReduceScatterRmsNorm states. gather=True also all-gathers out: every rank receives every slice, out of x's shape.
        Returns out (a new tensor when None and not gathering). With more than one rank x must be arena memory (`empty()`), and when
        gathering so must out: it has to be passed then."""
        sp = _rs_shapes(x, self.nranks, bool(gather))
        if out is None:
            if gather and self.nranks > 1:
                raise ValueError("gather=True needs out: an arena tensor (Comm.empty) of x's shape, the same on every rank")
            out = x.new_empty(sp[1])
        rows, row_len = check_reduce_scatter_rms_norm(self.nranks, x, residual, weight, out, eps, gather)
        _check(load().b200collReduceScatterRmsNorm(C.c_void_p(x.data_ptr()), C.c_void_p(residual.data_ptr()), C.c_void_p(weight.data_ptr()),
                                                   C.c_void_p(out.data_ptr()), rows, row_len, float(eps), int(bool(gather)),
                                                   torch_dtype_code(x.dtype), self._h, self._stream(stream)), "ReduceScatterRmsNorm")
        return out

    def reduce_scatter_rms_norm_quantized(self, x, residual, weight, q=None, scales=None, block: int = 128, wire=None, eps: float = 1e-6,
                                          gather: bool = False, stream=None):
        """reduce_scatter_rms_norm with its out quantised for an FP8 GEMM, in one kernel, as all_reduce_rms_norm_quantized quantises:
        `wire` torch.float8_e4m3fn (the default) or torch.float8_e5m2, one fp32 scale per 1 x `block` group, bit for bit as
        b200collReduceScatterRmsNormQuantized states. Returns (q, scales): q of residual's shape (x's when gathering) and the wire dtype,
        scales float32 [..., row_len // block] (new tensors when None and not gathering). gather=True with more than one rank needs q
        and scales passed, as arena tensors."""
        import torch
        sp = _rs_shapes(x, self.nranks, bool(gather))
        if (q is None or scales is None) and gather and self.nranks > 1:
            raise ValueError("gather=True needs q and scales: arena tensors (Comm.empty) of the gathered shapes, the same on every rank")
        w = torch.float8_e4m3fn if wire is None else wire
        q = x.new_empty(sp[1], dtype=w) if q is None else q
        if scales is None:
            _check_block(block)
            scales = x.new_empty(sp[1][:-1] + (sp[1][-1] // block,), dtype=torch.float32)
        rows, row_len, wc = check_reduce_scatter_rms_norm_quantized(self.nranks, x, residual, weight, q, scales, block, wire, eps, gather)
        _check(load().b200collReduceScatterRmsNormQuantized(C.c_void_p(x.data_ptr()), C.c_void_p(residual.data_ptr()),
                                                            C.c_void_p(weight.data_ptr()), C.c_void_p(q.data_ptr()),
                                                            C.cast(C.c_void_p(scales.data_ptr()), C.POINTER(C.c_float)), rows, row_len, float(eps),
                                                            int(bool(gather)), torch_dtype_code(x.dtype), wc, block, self._h, self._stream(stream)),
               "ReduceScatterRmsNormQuantized")
        return q, scales

    def all_to_all(self, src, dst, scale: float = 1.0, stream=None):
        ep = self._ep(src, dst, scale)
        _check(load().b200collAllToAll(C.c_void_p(src.data_ptr()), C.c_void_p(dst.data_ptr()), src.numel() // self.nranks, C.byref(ep), self._h, self._stream(stream)), "AllToAll")
        return dst

    def _ulysses(self, fn, name, seqs, heads, per, B, S_l, D, stream):
        arr = (UlyssesTensor * len(seqs))(*[UlyssesTensor(x.data_ptr(), rs, y.data_ptr(), h) for x, y, (rs, h) in zip(seqs, heads, per)])
        _check(fn(arr, len(seqs), B, S_l, D, torch_dtype_code(seqs[0].dtype), self._h, self._stream(stream)), name)

    def all_to_all_seq_to_heads(self, xs, outs=None, stream=None):
        """Ulysses all-to-all before attention, one kernel for up to three tensors (q, k, v): each [B, S_l, H_i, D] sequence shard in xs
        (views with uniformly strided token rows, e.g. column slices of a packed QKV projection output) becomes a dense [B, N * S_l, Hl_i, D]
        head shard, Hl_i = H_i / N; with fewer heads than ranks (GQA or MQA K and V, H_i dividing N) Hl_i = 1 and rank r gets head
        r * H_i // N. Bit for bit as coll/include/b200coll.h's b200collAllToAllSeqToHeads states. Returns outs. With more than one rank outs
        must be given, as arena tensors (`empty()`) at the same offsets on every rank; with one rank None allocates them."""
        xs = list(xs)
        if outs is None:
            if self.nranks > 1:
                raise ValueError("seq_to_heads with more than one rank needs outs: arena tensors (Comm.empty) of [B, S, H / N, D], the same on every rank")
            outs = [x.new_empty(x.shape) for x in xs]
        outs = list(outs)
        B, S_l, D, per = check_all_to_all_seq_to_heads(self.nranks, xs, outs)
        self._ulysses(load().b200collAllToAllSeqToHeads, "AllToAllSeqToHeads", xs, outs, per, B, S_l, D, stream)
        return outs

    def all_to_all_heads_to_seq(self, ys, outs=None, stream=None):
        """The inverse of all_to_all_seq_to_heads, after attention: each dense [B, N * S_l, H_i / N, D] head shard in ys becomes the
        [B, S_l, H_i, D] sequence shard in outs, which may be row-strided views; H_i must be a multiple of N. Bit for bit as
        b200collAllToAllHeadsToSeq states. Returns outs. With more than one rank outs must be given, as arena tensors; with one rank None
        allocates them."""
        ys = list(ys)
        if outs is None:
            if self.nranks > 1:
                raise ValueError("heads_to_seq with more than one rank needs outs: arena tensors (Comm.empty) of [B, S_l, H, D], the same on every rank")
            outs = [y.new_empty(y.shape) for y in ys]
        outs = list(outs)
        B, S_l, D, per = check_all_to_all_heads_to_seq(self.nranks, ys, outs)
        self._ulysses(load().b200collAllToAllHeadsToSeq, "AllToAllHeadsToSeq", outs, ys, per, B, S_l, D, stream)
        return outs

    def _context(self, fn, name, shards, fulls, per, B, S_l, chunks, stream):
        arr = (ContextTensor * len(shards))(*[ContextTensor(x.data_ptr(), rs, f.data_ptr(), w) for x, f, (rs, w) in zip(shards, fulls, per)])
        _check(fn(arr, len(shards), B, S_l, chunks, torch_dtype_code(shards[0].dtype), self._h, self._stream(stream)), name)

    def all_gather_context(self, shards, fulls=None, *, chunks: int, stream=None):
        """Context-parallel all-gather before attention, one kernel for up to three tensors (K and V): each [B, S_l, ...] sequence shard
        in shards (views with uniformly strided token rows, e.g. the K and V column slices of a packed QKV projection output) is gathered
        from every rank into the dense [B, N * S_l, ...] full tensor in fulls, in token order. chunks is the sharding: 1 contiguous (rank
        r holds tokens [r * S_l, (r + 1) * S_l)), 2 load-balanced for causal attention (the sequence cut into 2N chunks, rank r holding
        chunks r and 2N - 1 - r). A bit copy, as coll/include/b200coll.h's b200collAllGatherContext states. Returns fulls. With more than
        one rank fulls must be given, as arena tensors (`empty()`) at the same offsets on every rank; with one rank None allocates them."""
        shards = list(shards)
        if fulls is None:
            if self.nranks > 1:
                raise ValueError("all_gather_context with more than one rank needs fulls: arena tensors (Comm.empty) of [B, N * S_l, ...], "
                                 "the same on every rank")
            fulls = [x.new_empty(x.shape) for x in shards]
        fulls = list(fulls)
        B, S_l, per = check_all_gather_context(self.nranks, shards, fulls, chunks)
        self._context(load().b200collAllGatherContext, "AllGatherContext", shards, fulls, per, B, S_l, chunks, stream)
        return fulls

    def reduce_scatter_context(self, fulls, shards=None, *, chunks: int, stream=None):
        """The gradient of all_gather_context, after attention's backward: every rank's [B, N * S_l, ...] full tensors in fulls (dK and
        dV over the whole sequence, partial sums over the rank's own queries) are summed in fp32 in rank order, rounded once, and this
        rank's tokens (the layout chunks names) stored into the [B, S_l, ...] shards, which may be row-strided views such as the K and V
        column slices of a packed dQKV tensor. bfloat16, float16 or float32; bit for bit as b200collReduceScatterContext states. Returns
        shards. With more than one rank fulls must be arena tensors at the same offsets on every rank; shards may be any device tensors,
        and None allocates them."""
        fulls = list(fulls)
        if shards is None:
            shards = [f.new_empty((f.shape[0], f.shape[1] // self.nranks, *f.shape[2:])) for f in fulls]
        shards = list(shards)
        B, S_l, per = check_reduce_scatter_context(self.nranks, fulls, shards, chunks)
        self._context(load().b200collReduceScatterContext, "ReduceScatterContext", shards, fulls, per, B, S_l, chunks, stream)
        return shards

    def _shard_tensors(self, shards, fulls, per):
        return (ShardTensor * len(fulls))(*[ShardTensor(x.data_ptr(), f.data_ptr(), d, w, p) for x, f, (d, w, p) in zip(shards, fulls, per)])

    def all_gather_shards(self, shards, fulls=None, *, shard_rows=None, stream=None):
        """FSDP's parameter all-gather before forward, one kernel for up to 64 tensors (one unit): this rank's dim-0 shard of each
        parameter (rows [rank * p, rank * p + n_r) of the unsharded tensor, p = shard_rows, by default ceil(rows / N)) is cast on this
        rank (float32 -> bfloat16 or float16, or kept as it is) and stored into its rows of the unsharded tensor in fulls on every rank.
        Bit for bit as coll/include/b200coll.h's b200collAllGatherShards states. Returns fulls. With more than one rank fulls must be
        given, as arena tensors (`empty()` or the communicator's `mem_pool()`) at the same offsets on every rank; with one rank None
        allocates them in the shards' dtype."""
        shards = list(shards)
        if fulls is None:
            if self.nranks > 1:
                raise ValueError("all_gather_shards with more than one rank needs fulls: arena tensors (Comm.empty or Comm.mem_pool) of the "
                                 "unsharded shapes, the same on every rank")
            fulls = [x.new_empty(x.shape) for x in shards]
        fulls = list(fulls)
        per = check_all_gather_shards(self.nranks, self.rank, shards, fulls, shard_rows)
        arr = self._shard_tensors(shards, fulls, per)
        _check(load().b200collAllGatherShards(arr, len(fulls), torch_dtype_code(shards[0].dtype), torch_dtype_code(fulls[0].dtype), self._h,
                                              self._stream(stream)), "AllGatherShards")
        return fulls

    def reduce_scatter_shards(self, fulls, shards=None, *, scale: float = 1.0, accumulate: bool = False, shard_rows=None, stream=None):
        """FSDP's gradient reduce-scatter after backward, one kernel for up to 64 tensors: every rank's unsharded gradients in fulls
        are summed in fp32 in rank order, multiplied by scale (1 / N for a mean), added to the gradient already in shards if
        accumulate, rounded once and stored into this rank's rows of each shard (bfloat16 or float16 gradients may go to float32
        shards). Bit for bit as b200collReduceScatterShards states. Returns shards. With more than one rank fulls must be arena tensors
        at the same offsets on every rank and shards must be given (any device tensors); with one rank None allocates them in the
        fulls' dtype, unless accumulate asks for the old values."""
        fulls = list(fulls)
        if shards is None:
            if self.nranks > 1 or accumulate:
                raise ValueError("reduce_scatter_shards needs shards with more than one rank or with accumulate: this rank's sharded "
                                 "gradients, one per full")
            shards = [f.new_empty(f.shape) for f in fulls]
        shards = list(shards)
        per = check_reduce_scatter_shards(self.nranks, self.rank, fulls, shards, shard_rows)
        arr = self._shard_tensors(shards, fulls, per)
        _check(load().b200collReduceScatterShards(arr, len(fulls), torch_dtype_code(fulls[0].dtype), torch_dtype_code(shards[0].dtype),
                                                  float(scale), int(bool(accumulate)), self._h, self._stream(stream)), "ReduceScatterShards")
        return shards

    def vocab_parallel_cross_entropy(self, logits, target, ignore_index: int = -100, *, loss=None, lse=None, stream=None):
        """The tensor-parallel LM head's cross-entropy, one kernel: logits is this rank's [rows, Vl] slice of the vocabulary (global
        columns [rank * Vl, (rank + 1) * Vl)), target the [rows] int64 global labels, the same on every rank. Returns (loss, lse), [rows]
        float32 each, the same on every rank, bit for bit as coll/include/b200coll.h's b200collVocabParallelCrossEntropy states: loss =
        logsumexp over the whole vocabulary minus the target logit, +0 where target == ignore_index, NaN where the target is out of
        range. Any device tensors; only a 16-byte record per row and rank crosses NVLink."""
        import torch
        rows = logits.shape[0] if logits.dim() else 0
        loss = logits.new_empty(rows, dtype=torch.float32) if loss is None else loss
        lse = logits.new_empty(rows, dtype=torch.float32) if lse is None else lse
        rows, vl = check_vocab_parallel_cross_entropy(self.nranks, logits, target, loss, lse)
        _check(load().b200collVocabParallelCrossEntropy(logits.data_ptr(), target.data_ptr(), loss.data_ptr(), lse.data_ptr(), rows, vl,
                                                        int(ignore_index), torch_dtype_code(logits.dtype), self._h, self._stream(stream)),
               "VocabParallelCrossEntropy")
        return loss, lse

    def vocab_parallel_cross_entropy_backward(self, logits, target, lse, dloss, grad=None, ignore_index: int = -100, *, stream=None):
        """The gradient of vocab_parallel_cross_entropy's loss with respect to this rank's logits, one elementwise kernel, no
        communication: grad = round((exp(logits - lse) - onehot(target)) * dloss), +0 on ignored rows. grad=logits runs in place
        (Megatron's way of not keeping a second [rows, Vl] buffer); grad=None allocates it. Returns grad."""
        grad = logits.new_empty(logits.shape) if grad is None else grad
        rows, vl = check_vocab_parallel_cross_entropy(self.nranks, logits, target, lse=lse, dloss=dloss, grad=grad)
        _check(load().b200collVocabParallelCrossEntropyBackward(logits.data_ptr(), target.data_ptr(), lse.data_ptr(), dloss.data_ptr(),
                                                                grad.data_ptr(), rows, vl, int(ignore_index), torch_dtype_code(logits.dtype),
                                                                self._h, self._stream(stream)), "VocabParallelCrossEntropyBackward")
        return grad

    def vocab_parallel_cross_entropy_loss(self, logits, target, ignore_index: int = -100, *, inplace_backward: bool = False, stream=None):
        """vocab_parallel_cross_entropy as an autograd function: returns the [rows] float32 loss; .backward() runs
        vocab_parallel_cross_entropy_backward on this communicator. Only the logits, target and lse are saved. inplace_backward writes
        the gradient over the logits (they must not be needed afterwards)."""
        return _vocab_xent_fn().apply(logits, target, self, int(ignore_index), bool(inplace_backward), stream)

    def vocab_parallel_embedding(self, ids, weight, *, sequence_parallel: bool = False, out=None, stream=None):
        """The tensor-parallel input embedding, one kernel: weight is this rank's [Vl, H] rows of the table (global ids
        [rank * Vl, (rank + 1) * Vl)), ids the [T] int64 global ids, the same on every rank. Returns out = the unsplit table's rows of ids
        (+0 rows for ids outside [0, nranks * Vl)), bit for bit: [T, H] on every rank, or with sequence_parallel this rank's rows
        [rank * T / N, (rank + 1) * T / N). With more than one rank weight must be arena memory (Comm.empty); each rank pulls its rows
        from their owners over NVLink."""
        T = ids.shape[0] if ids.dim() == 1 else 0
        nr = T // self.nranks if sequence_parallel else T
        if out is None:
            out = weight.new_empty((nr, weight.shape[1] if weight.dim() == 2 else 0))
        T, h, vl = check_vocab_parallel_embedding(self.nranks, ids, weight, out, sequence_parallel=sequence_parallel,
                                                  symmetric=self.is_symmetric)
        _check(load().b200collVocabParallelEmbedding(ids.data_ptr(), weight.data_ptr(), out.data_ptr(), T, h, vl, int(bool(sequence_parallel)),
                                                     torch_dtype_code(weight.dtype), self._h, self._stream(stream)), "VocabParallelEmbedding")
        return out

    def vocab_parallel_embedding_backward(self, ids, grad_out, grad_weight=None, *, vocab_local: Optional[int] = None,
                                          sequence_parallel: bool = False, accumulate: bool = False, stream=None):
        """The gradient of vocab_parallel_embedding with respect to this rank's weight: grad_weight[j] = the sum, in fp32 and in token
        order, of grad_out's rows of the tokens whose id is rank * Vl + j, rounded once (added to grad_weight's old value with
        accumulate). grad_out is [T, H] (the same on every rank), or with sequence_parallel this rank's [T / N, H] shard, which must then
        be arena memory with more than one rank. grad_weight: a [Vl, H] float32 (a main_grad) or grad_out-dtype tensor, or None to
        allocate a float32 one (vocab_local required then). Returns grad_weight."""
        import torch
        if grad_weight is None:
            if vocab_local is None:
                raise ValueError("vocab_parallel_embedding_backward: give grad_weight or vocab_local")
            grad_weight = grad_out.new_empty((int(vocab_local), grad_out.shape[-1]), dtype=torch.float32)
        T, h, vl = check_vocab_parallel_embedding(self.nranks, ids, grad_weight, grad_out, sequence_parallel=sequence_parallel, backward=True,
                                                  symmetric=self.is_symmetric)
        _check(load().b200collVocabParallelEmbeddingBackward(ids.data_ptr(), grad_out.data_ptr(), grad_weight.data_ptr(), T, h, vl,
                                                             int(bool(sequence_parallel)), torch_dtype_code(grad_out.dtype),
                                                             torch_dtype_code(grad_weight.dtype), int(bool(accumulate)), self._h,
                                                             self._stream(stream)), "VocabParallelEmbeddingBackward")
        return grad_weight

    def vocab_parallel_embedding_lookup(self, ids, weight, *, sequence_parallel: bool = False, stream=None):
        """vocab_parallel_embedding as an autograd function: returns out; .backward() runs vocab_parallel_embedding_backward on this
        communicator into a fresh grad_weight of weight's dtype. Under sequence parallelism the backward needs its incoming gradient
        in arena memory, so with more than one rank it is always copied into the communicator's arena staging buffer first (one
        [T / N, H] copy on the call's stream; the same decision on every rank keeps the arena allocations in step)."""
        return _vocab_embedding_fn().apply(ids, weight, self, bool(sequence_parallel), stream)

    def _embedding_stage(self, g, stream=None):
        """g copied into this communicator's arena staging buffer for the sequence-parallel embedding gradient (one [T / N, H] copy on
        the call's stream), returned as a view of the buffer. One buffer per communicator, grown to at least twice its size when a
        call needs more; a superseded buffer is kept until the communicator is destroyed (a kernel already queued, or a peer's pull of
        it, may still read it), so all of them together stay below twice the largest. Every rank stages the same sizes in the same
        order, which keeps the arena allocations, a collective contract, the same on every rank. Reusing the buffer on one stream is
        safe: the backward's closing barrier ends every peer's reads before the stream moves on."""
        import torch
        need = g.numel() * g.element_size()
        buf = self.__dict__.get("_emb_stage")
        if buf is None or buf.numel() < need:
            if buf is not None:
                self.__dict__.setdefault("_emb_stage_retired", []).append(buf)
            buf = self.empty(max(need, 2 * (buf.numel() if buf is not None else 0)), torch.uint8)
            self._emb_stage = buf
        staged = buf[:need].view(g.dtype).view(g.shape)
        s = stream if stream is not None else torch.cuda.current_stream(g.device)
        s.wait_stream(torch.cuda.current_stream(g.device))
        with torch.cuda.stream(s):
            staged.copy_(g)
        g.record_stream(s)
        return staged

    def _rows(self, xs):
        """A host list of nranks row counts or offsets, as the library's int64[nranks]."""
        return (C.c_int64 * self.nranks)(*[int(x) for x in xs])

    def _routed_outputs(self, x, num_experts: int, top_k: int, expert_counts, route, dropped, stream):
        """The routed dispatch's small int32 outputs, each one not given allocated on x's device and the call's stream."""
        import torch
        with torch.cuda.device(x.device), torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream(x.device)):
            expert_counts = torch.empty(num_experts // self.nranks, dtype=torch.int32, device=x.device) if expert_counts is None else expert_counts
            route = torch.empty(x.shape[0], top_k, dtype=torch.int32, device=x.device) if route is None else route
            dropped = torch.empty(1, dtype=torch.int32, device=x.device) if dropped is None else dropped
        return expert_counts, route, dropped

    def all_to_all_v(self, src, dst, row_elems: int, send_rows, send_row_off, recv_row_off_at_peer, scale: float = 1.0, stream=None):
        ep = self._ep(src, dst, scale)
        arr = self._rows
        _check(load().b200collAllToAllv(C.c_void_p(src.data_ptr()), C.c_void_p(dst.data_ptr()), row_elems, arr(send_rows), arr(send_row_off), arr(recv_row_off_at_peer),
                                        C.byref(ep), self._h, self._stream(stream)), "AllToAllv")
        return dst

    def all_to_all_v_quantized(self, src, out, out_scales, row_elems: int, send_rows, send_row_off, recv_row_off_at_peer, block: int = 128,
                               stream=None):
        """Expert dispatch with FP8 on the wire (b200collAllToAllvQuantized): send_rows[p] rows of row_elems elements of src (bf16, fp16
        or fp32, any device tensor), starting at row send_row_off[p], are quantised on this rank in blocks of `block` elements with one
        fp32 scale per block, and land at row recv_row_off_at_peer[p] of peer p's out (FP8: its dtype is the wire type) and out_scales
        ([rows, row_elems // block] fp32). Returns (out, out_scales). With more than one rank, out and out_scales must be arena tensors
        (`empty()`) of the same size on every rank; every rank calls, a rank that sends nothing included."""
        ic, wc = check_all_to_all_v_quantized(self.nranks, src, out, out_scales, row_elems, block, send_rows, send_row_off, recv_row_off_at_peer)
        arr = self._rows
        _check(load().b200collAllToAllvQuantized(C.c_void_p(src.data_ptr()), C.c_void_p(out.data_ptr()), C.cast(C.c_void_p(out_scales.data_ptr()), C.POINTER(C.c_float)),
                                                 row_elems, out.numel() // row_elems, arr(send_rows), arr(send_row_off), arr(recv_row_off_at_peer), ic, wc, block,
                                                 self._h, self._stream(stream)), "AllToAllvQuantized")
        return out, out_scales

    def all_to_all_v_combine(self, expert_out, out, row_elems: int, send_rows, send_row_off, recv_row_off_at_peer, index, weights=None,
                             scale: float = 1.0, stream=None):
        """Expert combine (b200collAllToAllvCombine), the reverse of all_to_all_v with the top-k weighted sum fused: the three lists are
        the ones this rank passed to its dispatch call; index [tokens, top_k] int32 names, per token and slot, a row of that dispatch's
        send buffer (-1: dropped); weights [tokens, top_k] float32 or None (all ones). out[t] = round(scale * sum over slots in slot
        order of weights[t, j] * (expert output of row index[t, j])), pulled from the expert_out of the peer that row went to. Returns
        out. With more than one rank, expert_out must be an arena tensor (`empty()`) of the same size on every rank; every rank calls,
        a rank with no tokens included."""
        ic, oc = check_all_to_all_v_combine(self.nranks, expert_out, out, row_elems, send_rows, send_row_off, recv_row_off_at_peer, index, weights)
        arr = self._rows
        tokens, top_k = index.shape
        ep = Epilogue(ic, oc, float(scale))
        w = C.cast(C.c_void_p(weights.data_ptr() if weights is not None else None), C.POINTER(C.c_float))
        _check(load().b200collAllToAllvCombine(C.c_void_p(expert_out.data_ptr()), C.c_void_p(out.data_ptr()), row_elems, expert_out.numel() // row_elems,
                                               arr(send_rows), arr(send_row_off), arr(recv_row_off_at_peer),
                                               C.cast(C.c_void_p(index.data_ptr()), C.POINTER(C.c_int32)), w, tokens, top_k, C.byref(ep),
                                               self._h, self._stream(stream)), "AllToAllvCombine")
        return out

    def expert_dispatch(self, x, topk_idx, num_experts: int, recv, expert_counts=None, route=None, dropped=None, stream=None):
        """Device-routed expert dispatch (b200collExpertDispatch): slot (t, j) sends row t of x ([tokens, row_elems] bf16, fp16 or fp32)
        to expert topk_idx[t, j] (int32 on the device; an id outside [0, num_experts) drops the slot). Rank d owns experts
        [d * E / N, (d + 1) * E / N); its recv holds them in ascending order, each expert's rows by source rank, then in (token, slot)
        order, and rows past recv's end are dropped. Returns (recv, expert_counts [E / N] int32: rows stored per local expert,
        route [tokens, top_k] int32: peer * recv_rows + row or -1, dropped [1] int32: rows for this rank that did not fit). The small
        outputs are allocated on the call's stream when not given. Nothing is read back to the host. A program that drives several ranks
        from one thread (virtual ranks sharing a GPU) passes them, allocated before the first rank's call: an allocation between two
        ranks' calls can wait for the device (a cache flush frees memory, and freeing synchronises), while the earlier rank's layout
        kernel waits at its barrier for the next rank's call. With more than one rank, recv
        must be an arena tensor (`empty()`) of the same size on every rank; every rank calls, a rank with no tokens included."""
        code = check_expert_dispatch(self.nranks, x, topk_idx, num_experts, recv, expert_counts, route, dropped)
        tokens, row_elems = x.shape
        top_k = topk_idx.shape[1]
        if expert_counts is None or route is None or dropped is None:
            expert_counts, route, dropped = self._routed_outputs(x, num_experts, top_k, expert_counts, route, dropped, stream)
            check_expert_dispatch(self.nranks, x, topk_idx, num_experts, recv, expert_counts, route, dropped)
        i32 = lambda t: C.cast(C.c_void_p(t.data_ptr()), C.POINTER(C.c_int32))
        _check(load().b200collExpertDispatch(C.c_void_p(x.data_ptr()), C.c_void_p(recv.data_ptr()), row_elems, recv.numel() // row_elems, i32(topk_idx),
                                             tokens, top_k, num_experts, i32(expert_counts), i32(route), i32(dropped), code, self._h,
                                             self._stream(stream)), "ExpertDispatch")
        return recv, expert_counts, route, dropped

    def expert_dispatch_quantized(self, x, topk_idx, num_experts: int, recv, recv_scales, block: int = 128, expert_counts=None, route=None,
                                  dropped=None, stream=None):
        """Device-routed expert dispatch with FP8 on the wire (b200collExpertDispatchQuantized): expert_dispatch's layout (the same rows,
        expert_counts, route and dropped for the same ids), with each token's row quantised once on its own rank in blocks of `block`
        elements and one fp32 scale per block: recv ([recv_rows * row_elems] FP8, its dtype is the wire type) gets the FP8 rows and
        recv_scales ([recv_rows * row_elems // block] float32) their scales, row for row; rows not stored keep their bytes in both.
        Returns (recv, recv_scales, expert_counts, route, dropped). The small outputs are allocated on the call's stream when not given.
        Nothing is read back to the host. A program that drives several ranks from one thread (virtual ranks sharing a GPU) passes them,
        allocated before the first rank's call: an allocation between two ranks' calls can wait for the device (a cache flush frees
        memory, and freeing synchronises), while the earlier rank's layout kernel waits at its barrier for the next rank's call. With more
        than one rank, recv and recv_scales must be arena tensors (`empty()`) of the same sizes on every rank; every rank calls, a rank
        with no tokens included."""
        ic, wc = check_expert_dispatch_quantized(self.nranks, x, topk_idx, num_experts, recv, recv_scales, block, expert_counts, route, dropped)
        tokens, row_elems = x.shape
        top_k = topk_idx.shape[1]
        if expert_counts is None or route is None or dropped is None:
            expert_counts, route, dropped = self._routed_outputs(x, num_experts, top_k, expert_counts, route, dropped, stream)
            check_expert_dispatch_quantized(self.nranks, x, topk_idx, num_experts, recv, recv_scales, block, expert_counts, route, dropped)
        i32 = lambda t: C.cast(C.c_void_p(t.data_ptr()), C.POINTER(C.c_int32))
        _check(load().b200collExpertDispatchQuantized(C.c_void_p(x.data_ptr()), C.c_void_p(recv.data_ptr()),
                                                      C.cast(C.c_void_p(recv_scales.data_ptr()), C.POINTER(C.c_float)), row_elems,
                                                      recv.numel() // row_elems, i32(topk_idx), tokens, top_k, num_experts, i32(expert_counts),
                                                      i32(route), i32(dropped), ic, wc, block, self._h, self._stream(stream)),
               "ExpertDispatchQuantized")
        return recv, recv_scales, expert_counts, route, dropped

    def expert_combine(self, expert_out, route, weights, out, scale: float = 1.0, stream=None):
        """Expert combine from the dispatch's device route (b200collExpertCombine): out[t] ([tokens, row_elems]) = round(scale * sum
        over slots in slot order of weights[t, j] * row route[t, j] % recv_rows of peer route[t, j] // recv_rows's expert_out); a route
        outside [0, nranks * recv_rows) is a dropped slot, weights None means all ones. Returns out. With more than one rank, expert_out
        must be an arena tensor (`empty()`) of the same size on every rank; every rank calls."""
        ic, oc = check_expert_combine(self.nranks, expert_out, route, weights, out)
        tokens, row_elems = out.shape
        ep = Epilogue(ic, oc, float(scale))
        w = C.cast(C.c_void_p(weights.data_ptr() if weights is not None else None), C.POINTER(C.c_float))
        _check(load().b200collExpertCombine(C.c_void_p(expert_out.data_ptr()), C.c_void_p(out.data_ptr()), row_elems, expert_out.numel() // row_elems,
                                            C.cast(C.c_void_p(route.data_ptr()), C.POINTER(C.c_int32)), w, tokens, route.shape[1], C.byref(ep),
                                            self._h, self._stream(stream)), "ExpertCombine")
        return out

    def all_to_all_v_combine_quantized(self, expert_out, out, row_elems: int, send_rows, send_row_off, recv_row_off_at_peer, index, weights=None,
                                       block: int = 128, wire=None, scale: float = 1.0, stream=None):
        """all_to_all_v_combine with FP8 on the wire (b200collAllToAllvCombineQuantized): every row of this rank's expert_out (bf16, fp16 or
        fp32, any device tensor) is quantised on this rank to `wire` (torch.float8_e4m3fn, the default, or torch.float8_e5m2) with one
        fp32 scale per `block` elements, and the slots pull FP8 rows and scales: out[t] = round(scale * sum over slots in slot order of
        weights[t, j] * float(q) * s). Returns out. The scratch comes from the arena: the same calls in the same order on every rank."""
        ic, oc, wc = check_all_to_all_v_combine_quantized(self.nranks, expert_out, out, row_elems, send_rows, send_row_off, recv_row_off_at_peer, index,
                                                          weights, block, wire)
        arr = self._rows
        tokens, top_k = index.shape
        ep = Epilogue(ic, oc, float(scale))
        w = C.cast(C.c_void_p(weights.data_ptr() if weights is not None else None), C.POINTER(C.c_float))
        _check(load().b200collAllToAllvCombineQuantized(C.c_void_p(expert_out.data_ptr()), C.c_void_p(out.data_ptr()), row_elems,
                                                        expert_out.numel() // row_elems, arr(send_rows), arr(send_row_off), arr(recv_row_off_at_peer),
                                                        C.cast(C.c_void_p(index.data_ptr()), C.POINTER(C.c_int32)), w, tokens, top_k, wc, block,
                                                        C.byref(ep), self._h, self._stream(stream)), "AllToAllvCombineQuantized")
        return out

    def expert_combine_quantized(self, expert_out, route, weights, out, block: int = 128, wire=None, scale: float = 1.0, stream=None):
        """expert_combine with FP8 on the wire (b200collExpertCombineQuantized): every row of this rank's expert_out (bf16, fp16 or fp32,
        any device tensor, for example a grouped GEMM's output) is quantised on this rank to `wire` (torch.float8_e4m3fn, the default, or
        torch.float8_e5m2) with one fp32 scale per `block` elements; each slot pulls its FP8 row and scales from the peer the route names,
        and out[t] = round(scale * sum over slots in slot order of weights[t, j] * float(q) * s). Returns out. The scratch comes from the
        arena: the same calls in the same order on every rank."""
        ic, oc, wc = check_expert_combine_quantized(self.nranks, expert_out, route, weights, out, block, wire)
        tokens, row_elems = out.shape
        ep = Epilogue(ic, oc, float(scale))
        w = C.cast(C.c_void_p(weights.data_ptr() if weights is not None else None), C.POINTER(C.c_float))
        _check(load().b200collExpertCombineQuantized(C.c_void_p(expert_out.data_ptr()), C.c_void_p(out.data_ptr()), row_elems,
                                                     expert_out.numel() // row_elems, C.cast(C.c_void_p(route.data_ptr()), C.POINTER(C.c_int32)), w,
                                                     tokens, route.shape[1], wc, block, C.byref(ep), self._h, self._stream(stream)),
               "ExpertCombineQuantized")
        return out

    def broadcast(self, src, dst=None, root: int = 0, scale: float = 1.0, stream=None):
        """dst on every rank = cast(scale * src of `root`). src is read on the root only (ncclBroadcast)."""
        dst = src if dst is None else dst
        ep = self._ep(src, dst, scale)
        _check(load().b200collBroadcast(C.c_void_p(src.data_ptr()), C.c_void_p(dst.data_ptr()), dst.numel(), C.byref(ep), root, self._h, self._stream(stream)), "Broadcast")
        return dst

    def reduce(self, src, dst=None, root: int = 0, scale: float = 1.0, op: int = SUM, stream=None):
        """dst on `root` = cast(scale * sum over ranks of src); dst is untouched elsewhere (ncclReduce)."""
        dst = src if dst is None else dst
        ep = self._ep(src, dst, scale)
        _check(load().b200collReduce(C.c_void_p(src.data_ptr()), C.c_void_p(dst.data_ptr()), src.numel(), C.byref(ep), op, root, self._h, self._stream(stream)), "Reduce")
        return dst

    def send(self, src, peer: int, stream=None) -> None:
        """Send the bytes of (contiguous) `src` to rank `peer` (ncclSend). Pairs with the peer's recv of the same size, in call order.
        Outside `group()` the call blocks the stream until the peer's recv runs."""
        _check(load().b200collSend(C.c_void_p(src.data_ptr()), src.numel() * src.element_size(), peer, self._h, self._stream(stream)), "Send")

    def recv(self, dst, peer: int, stream=None):
        """Receive into (contiguous) `dst` from rank `peer` (ncclRecv): written over NVLink in place when dst is an arena tensor, else staged."""
        _check(load().b200collRecv(C.c_void_p(dst.data_ptr()), dst.numel() * dst.element_size(), peer, self._h, self._stream(stream)), "Recv")
        return dst

    def barrier(self, stream=None) -> None:
        _check(load().b200collBarrier(self._h, self._stream(stream)), "Barrier")

    def host_barrier(self) -> None:
        _check(load().b200collHostBarrier(self._h), "HostBarrier")

    # ---------------------------------------------------------------- control / introspection
    def set_algo(self, name: str) -> None:
        _check(load().b200collCommSetAlgo(self._h, ALGO_NAMES.index(name)), "CommSetAlgo")
        self._algo = name

    class _BitExact:
        """Payloads that are not floating point (token ids, masks) must not take the Lamport path: it recognises empty slots by a NaN bit
        pattern and rewrites payload words that collide with it (0xFFFFFFFF becomes 0x7FFF7FFF: harmless for floats, which stay NaN,
        fatal for an int64 -1). The barrier-based push kernels forward 16-byte vectors untouched when the epilogue is the identity."""

        def __init__(self, comm):
            self.comm = comm
            self.prev = getattr(comm, "_algo", None) or ALGO_NAMES[load().b200collCommGetAlgo(comm._h)]      # B200COLL_ALGO may have forced one at init

        def __enter__(self):
            self.comm.set_algo("twoshot")
            return self.comm

        def __exit__(self, *exc):
            self.comm.set_algo(self.prev)
            return False

    def bit_exact(self) -> "Comm._BitExact":
        """`with comm.bit_exact(): comm.all_gather(words, out)` — moves arbitrary bits (viewed as fp16 / fp32 words) unchanged."""
        return Comm._BitExact(self)

    def set_max_ctas(self, n: int) -> None:
        _check(load().b200collCommSetMaxCtas(self._h, n), "CommSetMaxCtas")

    def set_p2p_window(self, nbytes: int) -> None:
        """Staging-window size for receives into tensors outside the arena (0 = automatic)."""
        _check(load().b200collCommSetP2pWindow(self._h, nbytes), "CommSetP2pWindow")

    def set_launch_shape(self, kind: str, max_ctas: int = 0, threads: int = 0) -> None:
        _check(load().b200collCommSetLaunchShape(self._h, {"nvls": 0, "p2p": 1, "ll": 2, "nvls_rs": 3, "rooted": 4}[kind], max_ctas, threads), "CommSetLaunchShape")

    def stats(self) -> dict:
        s = Stats()
        _check(load().b200collCommStatsGet(self._h, C.byref(s)), "CommStatsGet")
        return {"calls": list(s.calls), "bytes": list(s.bytes), "algo_calls": dict(zip(ALGO_NAMES, s.algo_calls)),
                "kernel_launches": s.kernel_launches, "staged_calls": s.staged_calls,
                "p2p_sends": s.p2p_sends, "p2p_recvs": s.p2p_recvs, "p2p_bytes": s.p2p_bytes,
                "host_calls": s.host_calls, "host_bytes": s.host_bytes, "host_zero_copy": s.host_zero_copy, "host_pipelined": s.host_pipelined, "bulk_launches": s.bulk_launches, "generic_launches": s.generic_launches}

    def check_async_error(self) -> None:
        f = Fault()
        rc = load().b200collCommGetAsyncError(self._h, C.byref(f))
        if rc != SUCCESS:
            raise B200CollError(rc, "watchdog", f"code={f.code} rank={f.rank} peer={f.peer} block={f.block} expected={f.expected} observed={f.observed} op={f.op}")


_VOCAB_XENT_FN = None


def _vocab_xent_fn():
    """The torch.autograd.Function behind Comm.vocab_parallel_cross_entropy_loss, built on first use (torch is imported lazily here)."""
    global _VOCAB_XENT_FN
    if _VOCAB_XENT_FN is None:
        import torch

        class VocabParallelCrossEntropy(torch.autograd.Function):
            @staticmethod
            def forward(ctx, logits, target, comm, ignore_index, inplace, stream):
                logits = logits.contiguous()
                loss, lse = comm.vocab_parallel_cross_entropy(logits, target, ignore_index, stream=stream)
                ctx.save_for_backward(logits, target, lse)
                ctx.comm, ctx.ignore_index, ctx.inplace, ctx.stream = comm, ignore_index, inplace, stream
                return loss

            @staticmethod
            def backward(ctx, dloss):
                logits, target, lse = ctx.saved_tensors
                grad = logits if ctx.inplace else None
                grad = ctx.comm.vocab_parallel_cross_entropy_backward(logits, target, lse, dloss.float().contiguous(), grad,
                                                                      ctx.ignore_index, stream=ctx.stream)
                return grad, None, None, None, None, None

        _VOCAB_XENT_FN = VocabParallelCrossEntropy
    return _VOCAB_XENT_FN


_VOCAB_EMBEDDING_FN = None


def _vocab_embedding_fn():
    """The torch.autograd.Function behind Comm.vocab_parallel_embedding_lookup, built on first use (torch is imported lazily here)."""
    global _VOCAB_EMBEDDING_FN
    if _VOCAB_EMBEDDING_FN is None:
        import torch

        class VocabParallelEmbedding(torch.autograd.Function):
            @staticmethod
            def forward(ctx, ids, weight, comm, sequence_parallel, stream):
                out = comm.vocab_parallel_embedding(ids, weight, sequence_parallel=sequence_parallel, stream=stream)
                ctx.save_for_backward(ids)
                ctx.comm, ctx.sp, ctx.stream = comm, sequence_parallel, stream
                ctx.vl, ctx.wdtype = weight.shape[0], weight.dtype
                return out

            @staticmethod
            def backward(ctx, grad_out):
                (ids,) = ctx.saved_tensors
                comm = ctx.comm
                g = grad_out.to(ctx.wdtype).contiguous()
                if ctx.sp and comm.nranks > 1 and ids.shape[0]:
                    # always staged (never decided per rank from where g happens to lie): the staging buffer is an arena allocation
                    g = comm._embedding_stage(g, ctx.stream)
                gw = torch.empty((ctx.vl, g.shape[1]), dtype=ctx.wdtype, device=g.device)
                comm.vocab_parallel_embedding_backward(ids, g, gw, sequence_parallel=ctx.sp, stream=ctx.stream)
                return None, gw, None, None, None

        _VOCAB_EMBEDDING_FN = VocabParallelEmbedding
    return _VOCAB_EMBEDDING_FN
