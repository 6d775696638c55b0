/*
 * libb200coll — intra-node collective library for up to 8×H100 (sm_90a) over NVLink 4 / NVSwitch.
 *
 * Role parity: this is the payload the transport-installer DaemonSet drops into
 * /home/kubernetes/bin/nvidia/lib64 and the device plugin's Allocate mounts into the pod —
 * the slot the reference fills with pre-built NCCL net plugins
 * (reference: fast-socket-installer/fast-socket-installer.yaml:41-45,
 *  gpudirect-rdma/nccl-rdma-installer.yaml:70-77, gpudirect-tcpxo/nccl-tcpxo-installer.yaml:83-91).
 * On a single NVSwitch box a *net* plugin is never on the data path, so the product here is the
 * collective itself: one-shot (Lamport/LL), two-shot P2P and NVLS-multimem kernels with the
 * cast/scale epilogue fused, chosen per (op, bytes, nranks) by a measured table (the
 * libnccl-tuner.so analogue, reference: gpudirect-tcpxo/README.md:80-81).
 *
 * C ABI, no C++ types cross the boundary. All collectives are asynchronous on `stream`
 * and never block the host on a peer.
 */
#ifndef B200COLL_H_
#define B200COLL_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200COLL_VERSION_MAJOR 0
#define B200COLL_VERSION_MINOR 1
#define B200COLL_MAX_RANKS 8
#define B200COLL_UNIQUE_ID_BYTES 128

typedef struct b200collComm* b200collComm_t;
typedef struct { char internal[B200COLL_UNIQUE_ID_BYTES]; } b200collUniqueId;
typedef void* b200collStream_t; /* cudaStream_t */

typedef enum {
  b200collSuccess = 0,
  b200collUnhandledCudaError = 1,
  b200collSystemError = 2,
  b200collInternalError = 3,
  b200collInvalidArgument = 4,
  b200collInvalidUsage = 5,
  b200collRemoteError = 6,   /* a peer timed out or aborted (watchdog) */
  b200collInProgress = 7,
  b200collOutOfMemory = 8,
  b200collNoDriver = 9       /* libcuda / GPU not present (CPU-only box) */
} b200collResult_t;

typedef enum {
  b200collFloat32 = 0,
  b200collFloat16 = 1,
  b200collBfloat16 = 2,
  b200collFloat8e4m3 = 3,   /* OCP FP8 E4M3 (finite max 448) */
  /* the types below take the generic reduction path (src/generic.cu): same type in and out, no scale, any operator but avg */
  b200collInt8 = 4,
  b200collUint8 = 5,
  b200collInt32 = 6,
  b200collUint32 = 7,
  b200collInt64 = 8,
  b200collUint64 = 9,
  b200collFloat64 = 10,
  b200collFloat8e5m2 = 11,  /* OCP FP8 E5M2 (finite max 57344) */
  b200collNumTypes = 12
} b200collDataType_t;

/* Fused-epilogue types are fp32, fp16, bf16, e4m3 and e5m2. Supported (in_dtype, out_dtype) pairs:
 *   f32 -> f32, f16, bf16, e4m3, e5m2      f16 -> f16, f32, e4m3, e5m2      bf16 -> bf16, f32, e4m3, e5m2
 *   e4m3 / e5m2 -> e4m3, e5m2, f16, bf16   (FP8 -> f32 is refused with InvalidArgument)
 * Sum and avg: every input element is widened to fp32, accumulated from +0 (so -0 inputs give +0) in a fixed order, multiplied once
 * by scale (avg: the fp32 product scale * (1/nranks)) and rounded ONCE, to nearest even, to the output type, so every rank holds
 * bit-identical results. The order depends on the kernel:
 *   FP8 inputs, every P2P kernel                            ranks 0 .. N-1
 *   LL and LL2 all-reduce, LL reduce-scatter                ranks 0 .. N-1
 *   one-shot all-reduce, P2P rooted reduce                  ranks 0 .. N-1
 *   two-shot all-reduce (16- and 32-bit inputs)             vector v lies in slice o where nvec*o/N <= v < nvec*(o+1)/N (nvec = count /
 *                                                           (16 / sizeof(in))); it is summed o, o+1, .., N-1, 0, .., o-1. Elements past
 *                                                           the last whole vector are summed in rank order. A staged all-reduce (buffers
 *                                                           outside the arena) runs this per staging chunk, slices taken from the chunk.
 *   P2P reduce-scatter (16- and 32-bit inputs)              receiving rank r sums r, r+1, .., N-1, 0, .., r-1
 *   context-parallel reduce-scatter                         ranks 0 .. N-1
 *   FSDP shard reduce-scatter (ReduceScatterShards)         ranks 0 .. N-1, then * scale, then + the old shard
 *   vocab-parallel cross-entropy (VocabParallelCrossEntropy) ranks 0 .. N-1 for S = sum_r s_r * exp(m_r - M); in a rank's slice, its
 *                                                           16-element chunk sums folded as RMSNorm's (see the entry below)
 *   NVLS (multimem.ld_reduce)                               the switch's order: within an ulp of the exact sum, not bit-reproducible
 * Rounding to FP8 saturates to the finite range (+-inf becomes +-max, NaN stays NaN); fp16 overflows to inf.
 * All-gather, broadcast and all-to-all(v) apply the same epilogue per element: round((0 + x) * scale) (e4m3 in, bf16 out, scale =
 * inverse quantisation scale is a dequantising all-gather). With the identity epilogue (same type, scale 1) they are bit copies, -0,
 * +-inf and NaN payloads included, on the barrier-based and copy-engine kernels. The Lamport (ll) path stores the received words too,
 * with one exception: a 4-byte word equal to its empty-slot marker 0xFFFFFFFF (bytes FF FF FF FF) arrives as 0x7FFF7FFF (FF 7F FF 7F),
 * which is still NaN in every type; payloads that are not floating point must therefore force the two-shot family. With one rank every
 * op is a copy with this epilogue, and the identity is a bit copy at every size (in place: nothing is launched).
 * The NVLS switch of an H100 cannot reduce FP8 (sm_90a has no FP8 multimem.ld_reduce), so FP8 reductions run on the P2P algorithms;
 * FP8 data movement may still use multimem.st. */

/* sum and avg of fp16 / bf16 / fp32 / e4m3 / e5m2 run on the fused fast paths (Lamport, two-shot, NVLS for the 16- and 32-bit types);
 * prod, min, max — and every operator on the integer types and fp64 — run on one barrier-based P2P kernel that accumulates in the
 * element type (fp16 / bf16 / FP8 in fp32), starting from rank 0's value (not +0) and going through ranks 1 .. N-1; integer sums wrap.
 * min / max propagate a NaN from any rank (as torch.minimum / maximum do) and keep the lower rank's value on a tie (-0 against +0). */
typedef enum { b200collSum = 0, b200collAvg = 1, b200collProd = 2, b200collMin = 3, b200collMax = 4 } b200collRedOp_t;

typedef enum {
  b200collOpAllReduce = 0,
  b200collOpAllGather = 1,
  b200collOpReduceScatter = 2,
  b200collOpAllToAll = 3,
  b200collOpBroadcast = 4,
  b200collOpReduce = 5,
  b200collNumOps = 6
} b200collOp_t;

/* Algorithm ids (tuner output; B200COLL_ALGO overrides). */
typedef enum {
  b200collAlgoAuto = 0,
  b200collAlgoLL = 1,        /* Lamport flag-in-payload push, zero barriers  (tiny)  */
  b200collAlgoOneShot = 2,   /* barrier + pull all peers + reduce in regs    (small) */
  b200collAlgoTwoShot = 3,   /* P2P pull-reduce own slice + push to peers    (mid/large, no multicast needed) */
  b200collAlgoNvls = 4,      /* multimem.ld_reduce / multimem.st through the switch (large) */
  b200collAlgoCopy = 5,      /* nranks == 1: fused scale/cast copy */
  b200collAlgoLL2 = 6,       /* two-shot Lamport all-reduce: zero barriers, 2S bytes received instead of N*S (mid) */
  b200collNumAlgos = 7
} b200collAlgo_t;

/* Fused epilogue: out = cast<out_dtype>(reduce(in) * scale). scale==1.0f and equal dtypes is the plain collective. */
typedef struct {
  b200collDataType_t in_dtype;
  b200collDataType_t out_dtype;
  float scale;
} b200collEpilogue;

typedef struct {
  size_t arena_bytes;        /* symmetric user heap per rank (default: env B200COLL_ARENA_MB or 2560 MiB) */
  int enable_nvls;           /* -1 auto (probe), 0 off, 1 require */
  int max_ctas;              /* 0 = auto */
  int timeout_ms;            /* device-side watchdog for every cross-GPU spin and the rendezvous: default 600000 (env B200COLL_TIMEOUT_MS), 0 = none, < 0 = default */
  int debug;                 /* 0 quiet, 1 info, 2 trace (env B200COLL_DEBUG) */
} b200collConfig;

typedef struct {
  int rank, nranks, device;
  int nvls;                  /* multicast window mapped */
  int p2p_ok;                /* full P2P matrix */
  int same_device_loopback;  /* virtual ranks share one GPU (test mode) */
  size_t arena_bytes;
  size_t arena_used;
  int sm_count;
  int driver_version;
} b200collCommInfo;

typedef struct {
  uint64_t calls[b200collNumOps];
  uint64_t bytes[b200collNumOps];
  uint64_t algo_calls[b200collNumAlgos];
  uint64_t kernel_launches;
  uint64_t staged_calls;     /* calls that went through the staging copy (unregistered buffers) */
  uint64_t p2p_sends, p2p_recvs, p2p_bytes;   /* point-to-point operations and the bytes they moved (sent + received) */
  uint64_t host_calls, host_bytes;            /* b200collAllReduceHost calls and the input bytes they carried */
  uint64_t host_zero_copy, host_pipelined;    /* ... of which: one-kernel zero-copy calls / chunked three-leg pipelines */
  uint64_t bulk_launches;                     /* kernels that moved their payload with the copy engine (cp.async.bulk ring) */
  uint64_t generic_launches;                  /* min / max / prod / integer / fp64 reduction kernels */
} b200collStats;

/* Device-written watchdog record (host-pinned). code != 0 means the comm is poisoned. */
typedef struct {
  uint32_t code;             /* 0 ok, 1 barrier timeout, 2 LL data timeout, 3 send/recv peer never showed up, 4 send/recv sizes differ, 5 bulk copy never completed (bulk variant) */
  uint32_t rank, peer, block;
  uint32_t expected, observed;
  uint32_t op, reserved;
} b200collFault;

const char* b200collGetErrorString(b200collResult_t r);
const char* b200collGetLastError(void);
int b200collGetVersion(void);

void b200collConfigDefault(b200collConfig* cfg);

/* --- multi-process: one rank per process, rendezvous over an abstract Unix socket (SCM_RIGHTS fd passing). */
b200collResult_t b200collGetUniqueId(b200collUniqueId* id);
/* Deterministic id from a string (e.g. "$MASTER_ADDR:$MASTER_PORT/0") so torchrun ranks need no side channel. */
b200collResult_t b200collUniqueIdFromString(const char* s, b200collUniqueId* id);
b200collResult_t b200collCommInitRank(b200collComm_t* comm, int nranks, const b200collUniqueId* id, int rank,
                                      const b200collConfig* cfg);
/* --- single process: n ranks, one per entry of devs (entries may repeat: virtual ranks on one GPU for tests). */
b200collResult_t b200collCommInitAll(b200collComm_t* comms, int n, const int* devs, const b200collConfig* cfg);
/* ncclCommSplit: a collective call on a multi-process communicator. Ranks that pass the same color >= 0 form a new communicator
 * (its own arena: cfg, or the parent's settings when NULL), ordered by (key, rank in the parent); color < 0 takes part and gets none. */
b200collResult_t b200collCommSplit(b200collComm_t comm, int color, int key, b200collComm_t* newcomm, const b200collConfig* cfg);
/* Test hook: the (rank, size) a split would give `rank`, from everybody's colors and keys. */
b200collResult_t b200collDebugSplitPlan(int nranks, int rank, const int* colors, const int* keys, int* new_rank, int* new_size);
b200collResult_t b200collCommDestroy(b200collComm_t comm);
b200collResult_t b200collCommInfoGet(b200collComm_t comm, b200collCommInfo* info);
b200collResult_t b200collCommStatsGet(b200collComm_t comm, b200collStats* stats);
b200collResult_t b200collCommGetAsyncError(b200collComm_t comm, b200collFault* fault);
/* Host-level barrier over the bootstrap channel (multi-process comms only; no-op for InitAll comms). */
b200collResult_t b200collHostBarrier(b200collComm_t comm);

/* --- symmetric memory: collective calls, same order and size on every rank (ncclMemAlloc analogue). */
b200collResult_t b200collMemAlloc(b200collComm_t comm, void** ptr, size_t bytes);
b200collResult_t b200collMemFree(b200collComm_t comm, void* ptr);
/* PyTorch glue: `torch.cuda.memory.CUDAPluggableAllocator(lib, "b200collTorchAlloc", "b200collTorchFree")` + `torch.cuda.MemPool` put
 * tensors into the arena of the communicator named by SetAllocatorComm (same allocation sequence on every rank, as for MemAlloc). */
b200collResult_t b200collSetAllocatorComm(b200collComm_t comm);
void* b200collTorchAlloc(size_t size, int device, void* stream);
void b200collTorchFree(void* ptr, size_t size, int device, void* stream);
/* 1 if [ptr, ptr+bytes) lies in this rank's symmetric arena. */
int b200collIsSymmetric(b200collComm_t comm, const void* ptr, size_t bytes);

/* --- collectives. count is in elements of ep->in_dtype.
 * Buffers inside the symmetric arena take the zero-copy paths; any other device pointer is staged. */
b200collResult_t b200collAllReduce(const void* send, void* recv, size_t count, const b200collEpilogue* ep,
                                   b200collRedOp_t op, b200collComm_t comm, b200collStream_t stream);
/* recv holds nranks*sendcount elements; rank r's contribution lands at r*sendcount. */
b200collResult_t b200collAllGather(const void* send, void* recv, size_t sendcount, const b200collEpilogue* ep,
                                   b200collComm_t comm, b200collStream_t stream);
/* send holds nranks*recvcount elements; rank r receives the reduction of slice r. */
b200collResult_t b200collReduceScatter(const void* send, void* recv, size_t recvcount, const b200collEpilogue* ep,
                                       b200collRedOp_t op, b200collComm_t comm, b200collStream_t stream);
/* send/recv hold nranks*count elements; block p of send goes to block `rank` of peer p's recv. */
b200collResult_t b200collAllToAll(const void* send, void* recv, size_t count, const b200collEpilogue* ep,
                                  b200collComm_t comm, b200collStream_t stream);
/* Expert-dispatch shape: rows of `row_elems` elements; send_rows[p] rows go to peer p starting at row
 * send_row_off[p] of send; they land at row recv_row_off[src] of the destination (all four arrays are
 * host arrays of length nranks; recv_row_off[src] = where rank `src`'s rows start in MY recv). */
b200collResult_t b200collAllToAllv(const void* send, void* recv, size_t row_elems, const int64_t* send_rows,
                                   const int64_t* send_row_off, const int64_t* recv_row_off_at_peer,
                                   const b200collEpilogue* ep, b200collComm_t comm, b200collStream_t stream);
/* Rooted collectives (ncclBroadcast / ncclReduce). Broadcast: root's send -> every rank's recv (cast/scale fused);
 * send is read on the root only. Reduce: root's recv = scale * sum over ranks of send; recv is written on the root only.
 * Ranks that do not use a buffer may pass any 16-byte aligned device pointer for it. */
b200collResult_t b200collBroadcast(const void* send, void* recv, size_t count, const b200collEpilogue* ep, int root,
                                   b200collComm_t comm, b200collStream_t stream);
b200collResult_t b200collReduce(const void* send, void* recv, size_t count, const b200collEpilogue* ep,
                                b200collRedOp_t op, int root, b200collComm_t comm, b200collStream_t stream);
b200collResult_t b200collBarrier(b200collComm_t comm, b200collStream_t stream);

/* --- block-scaled FP8 (src/blockscaled.cu, with the quantising collectives below): per-block dequantisation fused into all-gather, reduce-scatter and all-reduce.
 * Each rank's send buffer is a row-major matrix [rows, row_len] of e4m3 or e5m2 (rows = count / row_len) with one fp32 scale per
 * block_rows x block_cols block of THAT rank's matrix: ceil(rows / block_rows) x ceil(row_len / block_cols) scales, row-major, the last
 * block row and column may be partial. Element (i, j) of rank r has the value v = float(q) * s[i / block_rows][j / block_cols] (one fp32
 * multiply, round to nearest even).
 *   all-reduce, reduce-scatter:  out = round_once(((0 + v_0) + v_1 + ... + v_{N-1}) * scale), summed in fp32 in rank order; avg multiplies
 *                                scale by the fp32 value 1/N; other operators are refused (InvalidArgument)
 *   all-gather:                  out[shard r] = round_once((0 + v_r) * scale)   (so -0 comes out as +0)
 * ep->in_dtype is e4m3 or e5m2, ep->out_dtype bf16, fp16 or fp32 (FP8 -> fp32 is allowed here), ep->scale the global multiplier.
 * Rounding is RNE; NaN and inf in q or in a scale propagate as the fp32 arithmetic produces them.
 * Constraints (InvalidArgument unless noted, message in b200collGetLastError): row_len % 16 == 0; block_cols % 16 == 0 and block_rows >= 1
 * (so each 16-byte FP8 vector lies in one block); count % row_len == 0; reduce-scatter: rows % nranks == 0 (every slice is whole rows);
 * send and scales in the symmetric arena at the same offsets on every rank, else InvalidUsage (there is no staging path); recv any
 * 16-byte aligned device buffer that does not overlap send.
 * FP8 crosses NVLink (receivers pull FP8 and scales and dequantise in registers). All-gather and reduce-scatter count as oneshot in
 * b200collStats; all-reduce maps the tuner's pick (or the forced algorithm): ll / ll2 / oneshot -> oneshot (pull the whole matrix),
 * twoshot / nvls -> twoshot (pull my slice, push the result into every recv), and twoshot falls back to oneshot when recv is outside the
 * arena. Each rank makes that choice from its own recv, so all-reduce recv must be placed alike on every rank: in the arena at the same
 * offset everywhere, or outside it everywhere (ranks that disagree run different kernels and end in a watchdog fault; B200COLL_CHECK=1
 * turns the disagreement into InvalidUsage before the launch on multi-process communicators). One rank: a local dequantising copy, counted as copy.
 * bytes = FP8 input bytes (per rank; reduce-scatter: recvcount). At most 2^35 - 16 elements per rank. */
typedef struct {
  const float* scales;   /* ceil(rows/block_rows) x ceil(row_len/block_cols) fp32, row-major, in the symmetric arena */
  size_t row_len;        /* elements per row of the send matrix */
  int block_rows, block_cols;
} b200collBlockScale;
/* recv holds nranks*sendcount elements of out_dtype; shard r is rank r's matrix dequantised with rank r's scales. */
b200collResult_t b200collAllGatherBlockScaled(const void* send, void* recv, size_t sendcount, const b200collBlockScale* bs,
                                              const b200collEpilogue* ep, b200collComm_t comm, b200collStream_t stream);
/* send holds nranks*recvcount elements (rows whole rows); rank r receives the reduction of row slice r. */
b200collResult_t b200collReduceScatterBlockScaled(const void* send, void* recv, size_t recvcount, const b200collBlockScale* bs,
                                                  const b200collEpilogue* ep, b200collRedOp_t op, b200collComm_t comm, b200collStream_t stream);
b200collResult_t b200collAllReduceBlockScaled(const void* send, void* recv, size_t count, const b200collBlockScale* bs,
                                              const b200collEpilogue* ep, b200collRedOp_t op, b200collComm_t comm, b200collStream_t stream);

/* --- quantising collectives (src/blockscaled.cu, sharing the block-scaled pull): bf16, fp16 or fp32 in, block-scaled FP8 over NVLink, one kernel per call.
 * Each rank quantises its own send buffer, cut into blocks of `block` consecutive elements, to wire_dtype (e4m3 or e5m2) with one fp32
 * scale per block; peers pull the FP8 data and scales, dequantise in registers, sum in fp32 in rank order and store out_dtype.
 * Per block, with x widened exactly to fp32 and FMAX = 448 (e4m3) or 57344 (e5m2):
 *   amax = max |x| over the block (a NaN anywhere makes amax NaN)
 *   inv = FMAX / amax, s = amax / FMAX     IEEE fp32 divisions rounded to nearest; inv = s = 1 if amax == 0 or inv is +inf
 *   q = fp8_rne_satfinite(x * inv)         the product rounded to fp32 first; NaN stays NaN
 *   v = float(q) * s                       one fp32 multiply, rounded to nearest even
 * From there the block-scaled rules above apply, v_r being rank r's v:
 *   all-reduce, reduce-scatter:  out = round_once(((0 + v_0) + v_1 + ... + v_{N-1}) * scale); sum or avg only (avg multiplies scale by
 *                                the fp32 value 1/N)
 *   all-gather:                  out[shard r] = round_once((0 + v_r) * scale)
 * So a block holding +-inf or NaN comes out NaN in every element (q = 0 and s = inf, or NaN throughout), -0 comes out as +0, every rank
 * holds bit-identical results (a rank's own all-gather shard is the round trip of its input, not a copy of it), one-shot and two-shot
 * give the same bits, and one rank computes the same formula with N = 1 (a local round trip, counted as copy).
 * Arguments (InvalidArgument unless noted, message in b200collGetLastError): ep->in_dtype and ep->out_dtype bf16, fp16 or fp32;
 * wire_dtype e4m3 or e5m2; block 16, 32, 64, 128, 256 or 512; the per-rank count (reduce-scatter: recvcount) a multiple of block;
 * send and recv 16-byte aligned. send may be any device buffer (only the local rank reads it). recv may be any device buffer; the
 * two-shot all-reduce needs it in the arena (peers write into it) and falls back to one-shot otherwise, with the algorithm chosen as in
 * b200collAllReduceBlockScaled (the tuner's pick for an FP8 all-reduce of count bytes), so recv must be placed alike on every rank.
 * The all-reduce may run in place (send == recv, with in_dtype and out_dtype of one size); any other overlap of send and recv is refused.
 * A poisoned communicator gives RemoteError.
 * Scratch: the FP8 copy and its scales (count + 4 * count / block bytes per rank) live in a library-owned buffer taken from the symmetric
 * heap with b200collMemAlloc on first use and grown on demand, so these calls are a collective contract like MemAlloc (same calls in the
 * same order on every rank); OutOfMemory when the arena cannot hold it. A superseded scratch is kept until CommDestroy, so a CUDA graph
 * captured before a later call grew the scratch stays valid.
 * b200collStats count the input bytes (reduce-scatter: recvcount elements) under oneshot, twoshot or copy. At most 2^35 - 16 elements per rank. */
/* recv holds nranks*sendcount elements of out_dtype; shard r is rank r's send buffer quantised and dequantised. */
b200collResult_t b200collAllGatherQuantized(const void* send, void* recv, size_t sendcount, b200collDataType_t wire_dtype, int block,
                                            const b200collEpilogue* ep, b200collComm_t comm, b200collStream_t stream);
/* send holds nranks*recvcount elements; rank r receives the reduction of slice r. */
b200collResult_t b200collReduceScatterQuantized(const void* send, void* recv, size_t recvcount, b200collDataType_t wire_dtype, int block,
                                                const b200collEpilogue* ep, b200collRedOp_t op, b200collComm_t comm, b200collStream_t stream);
b200collResult_t b200collAllReduceQuantized(const void* send, void* recv, size_t count, b200collDataType_t wire_dtype, int block,
                                            const b200collEpilogue* ep, b200collRedOp_t op, b200collComm_t comm, b200collStream_t stream);
/* --- MoE expert dispatch (src/dispatch.cu) and combine (src/combine.cu). */

/* Quantising all-to-all-v (expert dispatch): bf16, fp16 or fp32 rows in, FP8 rows and their block scales out, one kernel per call. The
 * row geometry is b200collAllToAllv's: send_rows[p] rows of row_elems elements, starting at row send_row_off[p] of send, go to peer p and
 * land at row recv_row_off_at_peer[p] of that peer's recv and recv_scales (host arrays of length nranks). The sender quantises in
 * registers and pushes FP8 and scales straight into each receiver's buffers: row_elems * (1 + 4 / block) bytes per row cross NVLink.
 *   Per-row blocks: every row is cut into blocks of `block` consecutive elements (row_elems % block == 0), each quantised by the rule
 *   above (amax the largest bit pattern of |x|; inv and s IEEE divisions, inv = s = 1 when amax == 0 or inv is +inf; q = satfinite
 *   RNE(x * inv)), so a row's q and s are the bits b200collAllGatherQuantized writes into its scratch for the same block.
 *   recv: [recv_rows, row_elems] of wire_dtype. recv_scales: [recv_rows, row_elems / block] fp32, row-major: the block_rows = 1,
 *   block_cols = block layout of b200collBlockScale, so the result is also an input of the block-scaled collectives. Rows outside the
 *   received ranges are not written.
 *   in_dtype bf16, fp16 or fp32; wire_dtype e4m3 or e5m2; block 16, 32, 64, 128, 256 or 512.
 *   recv_rows: the rows recv and recv_scales hold, the same on every rank (they are symmetric allocations). Every destination range
 *   [recv_row_off_at_peer[p], + send_rows[p]) must lie inside it, else InvalidArgument before anything is launched.
 * Placement: send any 16-byte aligned device buffer (only its own rank reads it). With more than one rank, recv and recv_scales must be
 * arena memory at the same offsets on every rank, else InvalidUsage; with B200COLL_CHECK=1 on multi-process communicators, ranks that
 * disagree on (recv_rows, recv, recv_scales) get InvalidUsage instead of a watchdog fault. send overlapping recv or recv_scales, or recv
 * overlapping recv_scales, is InvalidArgument.
 * Other arguments (InvalidArgument, message in b200collGetLastError): null pointers, negative counts or offsets, send or recv not 16-byte
 * aligned or recv_scales not 4-byte aligned, more than 2^31 - 1 16-element vectors sent per rank. A poisoned communicator gives RemoteError.
 * Every rank launches on every call, a rank that sends nothing included (its peers' barriers wait for it), as with b200collAllToAllv.
 * One rank: a local quantising copy with no barrier, recv and recv_scales any device buffers, counted as copy.
 * b200collStats count the input bytes sent under alltoall, algorithm twoshot (or copy). */
b200collResult_t b200collAllToAllvQuantized(const void* send, void* recv, float* recv_scales, size_t row_elems, size_t recv_rows,
                                            const int64_t* send_rows, const int64_t* send_row_off, const int64_t* recv_row_off_at_peer,
                                            b200collDataType_t in_dtype, b200collDataType_t wire_dtype, int block,
                                            b200collComm_t comm, b200collStream_t stream);
/* Expert combine: the reverse of b200collAllToAllv / b200collAllToAllvQuantized with the top-k weighted sum fused, one kernel per call.
 * Each rank pulls the expert output rows its tokens need straight from the peers' expert_out, sums them in registers in slot order and
 * writes [tokens, row_elems] once: no landing buffer, no second kernel, no atomics, the same bits on every run.
 *   send_rows, send_row_off, recv_row_off_at_peer: the host arrays (length nranks) this rank passed to its dispatch call, same meaning.
 *   Dispatch row i belongs to peer p when send_row_off[p] <= i < send_row_off[p] + send_rows[p]; its expert output is row
 *   recv_row_off_at_peer[p] + (i - send_row_off[p]) of peer p's expert_out.
 *   expert_out: [recv_rows, row_elems] of ep->in_dtype on every rank, written by the experts before the call.
 *   index: device [tokens, top_k] int32 dispatch rows, -1 for a dropped slot. weights: device [tokens, top_k] fp32, or NULL for all ones.
 *   out: [tokens, row_elems] of ep->out_dtype.
 * Result, per token t and element e: out[t, e] = round_once(scale * acc), acc = ((+0 + w[t,0]*y(index[t,0])[e]) + w[t,1]*y(index[t,1])[e])
 * + ... for j = 0 .. top_k-1, every product and every sum rounded to fp32 on its own (no fused multiply-add), slots in slot order. A
 * slot whose index names no dispatch row (negative, in a gap between ranges, or past every range) is skipped; weights == NULL gives the
 * bits of all-ones weights. scale = ep->scale; rounding RNE, fp16 overflows to inf; NaN and inf propagate as the fp32 arithmetic makes
 * them; -0 comes out as +0; a token whose slots are all dropped gets +0 (times scale). The result depends only on the expert_out values
 * and the weights, not on the number of ranks or on which rank held a row.
 *   in_dtype and out_dtype: each bf16, fp16 or fp32 (9 pairs); FP8 on either side is InvalidArgument.
 * Refused with InvalidArgument before anything is launched (message in b200collGetLastError): null pointers (index and out may be NULL
 * only when tokens == 0), row_elems == 0 or row_elems % 16 != 0, top_k < 1, negative counts or offsets, a destination range
 * [recv_row_off_at_peer[p], + send_rows[p]) past recv_rows, two non-empty send ranges that overlap (the row -> peer map must be unique),
 * expert_out or out not 16-byte aligned, index or weights not 4-byte aligned, out overlapping expert_out, index or weights, more than
 * 2^31 - 1 16-element vectors of out, tokens * top_k > 2^31 - 1.
 * Placement: with more than one rank, expert_out must be arena memory at the same offset on every rank (else InvalidUsage) and recv_rows
 * the same on every rank; with B200COLL_CHECK=1 on multi-process communicators, (recv_rows, arena offset of expert_out) is compared across
 * ranks. out, index and weights may be any device buffers. A poisoned communicator gives RemoteError.
 * The kernel never reads outside a destination range of a peer, whatever index holds (index is device data the host cannot check).
 * Every rank launches on every call, a rank with tokens == 0 or no rows included (its peers' barriers wait for it). The call returns
 * (on its stream) only after every peer has finished reading this rank's expert_out, so the caller may overwrite it right after.
 * One rank: a local gather and sum with no barrier, expert_out any device buffer.
 * b200collStats count the call under alltoall, algorithm oneshot (copy with one rank), sum_p send_rows[p] * row_elems * sizeof(in) bytes,
 * and one kernel launch. */
b200collResult_t b200collAllToAllvCombine(const void* expert_out, void* out, size_t row_elems, size_t recv_rows,
                                          const int64_t* send_rows, const int64_t* send_row_off, const int64_t* recv_row_off_at_peer,
                                          const int32_t* index, const float* weights, size_t tokens, int top_k,
                                          const b200collEpilogue* ep, b200collComm_t comm, b200collStream_t stream);
/* Device-routed expert dispatch: the router's top-k expert ids in (device), rows grouped by expert out, with no host sync. Two kernels
 * per call: a one-CTA layout kernel (per-expert counts, exchanged between ranks through a mailbox in the arena, and each slot's row),
 * then a push of the rows over NVLink. Nothing the host must know depends on device data, so the call can be captured in a CUDA graph.
 *   Experts: num_experts (E) experts, 1 <= E <= 1024, E a multiple of nranks; rank d owns experts [d*E/N, (d+1)*E/N).
 *   topk_idx: device [tokens, top_k] int32. Slot (t, j) sends row t of x to expert topk_idx[t, j]; an id outside [0, E) drops the slot.
 *   A token may name one expert twice: it is then sent twice.
 *   x: [tokens, row_elems] of dtype (bf16, fp16 or fp32), any 16-byte aligned device buffer (only its own rank reads it). Rows move as
 *   raw bits: NaN payloads and -0 survive.
 *   recv: [recv_rows, row_elems] of dtype. On rank d it holds d's experts in ascending order; within an expert, rows by source rank
 *   ascending; within a source, in row-major (token, slot) order. The row of slot (t, j) of rank s sent to expert e is
 *   base_d(e) + sum_{s' < s} cnt[s'][e] + #{(t', j') < (t, j) on rank s with topk_idx = e}, base_d(e) the total rows of d's experts
 *   below e over all sources. A row at or past recv_rows is dropped; rows not stored keep their previous bytes.
 *   expert_counts: device [E/N] int32, rows stored per local expert: clamp(recv_rows - base_d(e), 0, total[e]).
 *   route: device [tokens, top_k] int32, peer * recv_rows + row for a stored slot, -1 for a dropped one (what b200collExpertCombine reads).
 *   dropped: device [1] int32, rows addressed to this rank that did not fit (saturating at 2^31 - 1).
 * Refused with InvalidArgument before anything is launched: null pointers (x, topk_idx and route may be NULL only when tokens == 0),
 * a dtype other than bf16, fp16 or fp32, row_elems == 0 or row_elems % 16 != 0, top_k < 1, E outside [1, 1024] or not a multiple of
 * nranks, x or recv not 16-byte aligned, topk_idx, expert_counts, route or dropped not 4-byte aligned, recv overlapping x, an output
 * array overlapping another, topk_idx, x or recv, tokens * top_k > 2^31 - 1, nranks * recv_rows > 2^31 - 1, more than 2^31 - 1 16-byte
 * vectors offered (tokens * top_k * row_bytes / 16).
 * Placement: with more than one rank, recv must be arena memory at the same offset on every rank (else InvalidUsage), and recv_rows the
 * same on every rank; with B200COLL_CHECK=1 on multi-process communicators (E, row_elems, recv_rows, arena offset of recv) is compared
 * across ranks. A poisoned communicator gives RemoteError.
 * Every rank launches on every call, a rank with tokens == 0 included (its peers' barriers wait for it). One rank: no barriers, recv any
 * device buffer, counted as copy. b200collStats count the call under alltoall, algorithm twoshot (copy with one rank), two kernel
 * launches, and tokens * top_k * row_elems * sizeof(dtype) bytes: the slots offered, which the host knows, not the rows stored. */
b200collResult_t b200collExpertDispatch(const void* x, void* recv, size_t row_elems, size_t recv_rows, const int32_t* topk_idx, size_t tokens,
                                        int top_k, int num_experts, int32_t* expert_counts, int32_t* route, int32_t* dropped,
                                        b200collDataType_t dtype, b200collComm_t comm, b200collStream_t stream);
/* Device-routed expert dispatch with FP8 on the wire: b200collExpertDispatch's layout, b200collAllToAllvQuantized's rows. Two kernels per
 * call, the same layout kernel, then a push that quantises every token's row once and stores the FP8 row and its block scales to every
 * stored slot of the token: row_elems * (1 + 4 / block) bytes per row cross NVLink instead of row_elems * sizeof(in_dtype). No host sync,
 * so the call can be captured in a CUDA graph.
 *   Layout: exactly b200collExpertDispatch's for the same arguments: expert ownership, the row of every slot, expert_counts, route,
 *   dropped and the capacity rule (rows at or past recv_rows are dropped) are the same, bit for bit.
 *   x: [tokens, row_elems] of in_dtype (bf16, fp16 or fp32), any 16-byte aligned device buffer.
 *   recv: [recv_rows, row_elems] of wire_dtype (e4m3 or e5m2). Row r holds the quantisation of its source token's row, by the rule of
 *   b200collAllToAllvQuantized (amax the largest bit pattern of |x| per block of `block` elements; inv and s IEEE divisions, inv = s = 1
 *   when amax == 0 or inv is +inf; q = satfinite RNE(x * inv)). recv_scales: [recv_rows, row_elems / block] fp32, row r's scales (the
 *   block_rows = 1, block_cols = block layout of b200collBlockScale). Every stored slot of one token gets the same bytes and scales; rows
 *   not stored keep their previous bytes in both buffers. block: 16, 32, 64, 128, 256 or 512, dividing row_elems.
 * Refused with InvalidArgument before anything is launched: everything b200collExpertDispatch refuses, and in_dtype other than bf16,
 * fp16 or fp32, wire_dtype other than e4m3 or e5m2, a block not in the list, row_elems % block != 0, recv_scales NULL or not 4-byte
 * aligned, any overlap among x, recv and recv_scales, an output array overlapping recv_scales, more than 2^31 - 1 16-element vectors
 * of x (tokens * row_elems / 16).
 * Placement: with more than one rank, recv and recv_scales must be arena memory at the same offsets on every rank (else InvalidUsage), and
 * recv_rows the same on every rank; with B200COLL_CHECK=1 on multi-process communicators, recv_rows, both arena offsets and (E, row_elems,
 * block, wire_dtype) are compared across ranks. A poisoned communicator gives RemoteError.
 * Every rank launches on every call, a rank with tokens == 0 included. One rank: no barriers, recv and recv_scales any device buffers,
 * counted as copy. b200collStats count the call under alltoall, algorithm twoshot (copy with one rank), two kernel launches, and
 * tokens * top_k * row_elems * sizeof(in_dtype) bytes. */
b200collResult_t b200collExpertDispatchQuantized(const void* x, void* recv, float* recv_scales, size_t row_elems, size_t recv_rows,
                                                 const int32_t* topk_idx, size_t tokens, int top_k, int num_experts,
                                                 int32_t* expert_counts, int32_t* route, int32_t* dropped,
                                                 b200collDataType_t in_dtype, b200collDataType_t wire_dtype, int block,
                                                 b200collComm_t comm, b200collStream_t stream);
/* Expert combine from a device route: b200collAllToAllvCombine's result and rules, with each slot's (peer, row) read from the route
 * b200collExpertDispatch wrote instead of the dispatch's host arrays. Slot j of token t reads row route % recv_rows of peer
 * route / recv_rows's expert_out ([recv_rows, row_elems] of ep->in_dtype); a route outside [0, nranks * recv_rows) is a dropped slot, and
 * the kernel reads nothing else whatever the device array holds. out[t] = round_once(scale * ((+0 + w0*y0) + w1*y1 + ...)) in slot order,
 * no fused multiply-add, 9 type pairs; weights NULL gives all ones.
 * Refused with InvalidArgument before anything is launched: null pointers (route and out may be NULL only when tokens == 0), in or out
 * type not bf16, fp16 or fp32, row_elems == 0 or row_elems % 16 != 0, top_k < 1, expert_out or out not 16-byte aligned, route or weights
 * not 4-byte aligned, out overlapping expert_out, route or weights, more than 2^31 - 1 16-element vectors of out, tokens * top_k > 2^31 - 1,
 * nranks * recv_rows > 2^31 - 1. Placement, the closing barrier (the caller may overwrite expert_out right after the call), the one-rank
 * path and RemoteError are those of b200collAllToAllvCombine. b200collStats count the call under alltoall, algorithm oneshot (copy with
 * one rank), one kernel launch, and tokens * top_k * row_elems * sizeof(in) bytes (the slots offered). */
b200collResult_t b200collExpertCombine(const void* expert_out, void* out, size_t row_elems, size_t recv_rows, const int32_t* route,
                                       const float* weights, size_t tokens, int top_k, const b200collEpilogue* ep, b200collComm_t comm,
                                       b200collStream_t stream);
/* Quantising expert combine: b200collAllToAllvCombine (segment table) and b200collExpertCombine (device route) with FP8 on the wire:
 * row_elems * (1 + 4 / block) bytes per pulled row cross NVLink instead of row_elems * sizeof(in). Two kernels per call: each rank
 * quantises every row of its expert_out ([recv_rows, row_elems] of ep->in_dtype, bf16, fp16 or fp32) into a library-owned scratch, by
 * the rule of the quantising collectives: blocks of `block` elements along the row, wire_dtype e4m3 or e5m2, one fp32 scale per block,
 * the bytes and scales b200collAllToAllvQuantized stores for that row. Then it pulls its slots' FP8 rows and scales from the peers'
 * scratch and sums them.
 * Result, per token t and element e, with v = float(q) * s (one fp32 multiply):
 *   out[t, e] = round_once(scale * ((+0 + w0*v0[e]) + w1*v1[e] + ...)), slots in slot order, every product and every sum rounded to
 *   fp32 on its own (no fused multiply-add). A slot maps to a row, or is dropped, exactly as in the wide combine of the same map. A block
 *   holding NaN or +-inf dequantises to NaN throughout (its amax is NaN or inf). The result depends only on the values and the weights:
 *   the rank count and which rank held a row make no difference, and one rank gives the same bits as eight.
 *   ep->out_dtype bf16, fp16 or fp32; weights NULL gives all ones; scale = ep->scale.
 * Refused with InvalidArgument before anything is launched: everything the matching wide combine refuses, except that expert_out need
 * not be arena memory; and in or out type not bf16, fp16 or fp32, wire_dtype not e4m3 or e5m2, block not 16, 32, 64, 128, 256 or 512,
 * row_elems % block != 0, more than 2^31 - 1 16-element vectors of expert_out (recv_rows * row_elems / 16).
 * Placement: expert_out, out, index / route and weights may be any device buffers (peers read only the scratch). recv_rows must be the
 * same on every rank; with B200COLL_CHECK=1 on multi-process communicators, (recv_rows, scratch offsets) and (row_elems, block,
 * wire_dtype) are compared across ranks. A poisoned communicator gives RemoteError.
 * Scratch: recv_rows * row_elems * (1 + 4 / block) bytes, in the scratch of the quantising collectives (a collective contract: the same
 * calls in the same order on every rank); OutOfMemory, before anything is launched, when the arena cannot hold it. A superseded scratch
 * is kept until CommDestroy, so a CUDA graph captured earlier stays valid. The quantise pass covers all recv_rows rows, read or not.
 * Every rank launches on every call. The call returns (on its stream) only after every peer has finished reading this rank's scratch;
 * expert_out is read only by this rank's quantise pass, so the caller may overwrite it right after the call. One rank: the same two
 * kernels with no barrier. b200collStats count the call under alltoall, algorithm oneshot (copy with one rank), two kernel launches, and
 * the bytes the matching wide combine counts. */
b200collResult_t b200collAllToAllvCombineQuantized(const void* expert_out, void* out, size_t row_elems, size_t recv_rows,
                                                   const int64_t* send_rows, const int64_t* send_row_off, const int64_t* recv_row_off_at_peer,
                                                   const int32_t* index, const float* weights, size_t tokens, int top_k,
                                                   b200collDataType_t wire_dtype, int block, const b200collEpilogue* ep, b200collComm_t comm,
                                                   b200collStream_t stream);
b200collResult_t b200collExpertCombineQuantized(const void* expert_out, void* out, size_t row_elems, size_t recv_rows, const int32_t* route,
                                                const float* weights, size_t tokens, int top_k, b200collDataType_t wire_dtype, int block,
                                                const b200collEpilogue* ep, b200collComm_t comm, b200collStream_t stream);

/* --- fused all-reduce, residual add and RMSNorm (src/rmsnorm.cu): the step after the attention output projection and the MLP down
 * projection of a pre-norm tensor-parallel block, one kernel per call. x is this rank's [rows, row_len] partial sums, residual
 * [rows, row_len] (the same on every rank in tensor parallelism), gamma [row_len], all of `dtype` (bf16, fp16 or fp32), as is out. Per row
 * and element e, in fp32, every product and sum rounded on its own (no fused multiply-add):
 *   1. h[e] = round_dtype(((+0 + x_0[e]) + x_1[e] + ... + x_{N-1}[e]) + residual[e]): ranks summed in rank order, one rounding at the
 *      end. h is written back into residual, in place (the new residual stream).
 *   2. sq[e] = h[e] * h[e], with h as stored (the norm sees exactly the residual the next layer reads).
 *   3. p[c] = the sum of the 16 sq of chunk c (elements 16c .. 16c+15) in element order from +0; p padded with +0 to the next power of
 *      two P, then folded p = p[:P/2] + p[P/2:] until one value is left.
 *   4. ms = fold / row_len, inv = 1 / sqrt(ms + eps): IEEE division and square root, rounded to nearest (no rsqrt approximation).
 *   5. out[e] = round_dtype((h[e] * inv) * gamma[e]).
 * Rounding is RNE; NaN and inf propagate as the arithmetic makes them (an all-zero row with eps = 0 gives NaN). The result depends only on
 * the values and the rank count, not on the algorithm or the launch shape. Every rank holds the same out and new residual provided the
 * ranks passed the same residual (the caller's condition); on two-shot a row comes from the residual of the rank that owns it.
 * Algorithms (the tuner's all-reduce pick for rows * row_len * sizeof(dtype) bytes, or the forced algorithm): ll, ll2 and oneshot ->
 * oneshot (every rank pulls every row of every peer's x and stores residual and out locally); twoshot and nvls -> twoshot (rank r pulls
 * rows [rows*r/N, rows*(r+1)/N), pushes their residual and out rows into every rank), which needs residual and out in the arena and falls
 * back to oneshot otherwise. Each rank decides from its own buffers, so residual and out must be placed alike on every rank: in the arena
 * at the same offsets everywhere, or outside it everywhere (B200COLL_CHECK=1 cross-checks rows, row_len, the offsets and the algorithm
 * and turns a disagreement into InvalidUsage on multi-process communicators). The kernel ends with a releasing barrier, so the caller
 * may overwrite x right after the call.
 * Arguments (InvalidArgument, message in b200collGetLastError, nothing launched): dtype bf16, fp16 or fp32; row_len a multiple of 16 in
 * [16, 16384]; eps finite and >= 0; rows < 2^31; no null pointer when rows > 0; x, residual, gamma and out 16-byte aligned; out must not
 * overlap x, residual or gamma, residual must not overlap x or gamma. More than one rank: x in the symmetric arena at the same offset on
 * every rank, else InvalidUsage. A poisoned communicator gives RemoteError. rows == 0 still launches on every rank (peers' barriers wait
 * for it), one-shot, and reads and writes nothing, so its pointers may lie anywhere or be null. One rank: a local kernel, no barrier, any device buffers. b200collStats count an allreduce of rows * row_len * sizeof(dtype)
 * bytes under oneshot, twoshot or copy, one kernel launch. */
b200collResult_t b200collAllReduceRmsNorm(const void* x, void* residual, const void* gamma, void* out, size_t rows, size_t row_len,
                                          float eps, b200collDataType_t dtype, b200collComm_t comm, b200collStream_t stream);
/* Fused all-reduce, residual add, RMSNorm and FP8 block quantisation: the normed rows go straight to an FP8 GEMM (the QKV projection after
 * the attention norm, the gate/up projection after the MLP norm) as e4m3 or e5m2 rows with one fp32 scale per 1 x block group, in one
 * kernel per call. Steps 1-4 are b200collAllReduceRmsNorm's, unchanged, and residual receives the same bits in place. Then, per row:
 *   5. o[e] = round_dtype((h[e] * inv) * gamma[e]): the value b200collAllReduceRmsNorm stores in out.
 *   6. The row is cut into blocks of `block` consecutive elements, and each block of o, widened exactly to fp32, is quantised by the rule
 *      of the quantising collectives: amax the largest bit pattern of |o| (a NaN anywhere makes amax NaN); inv = FMAX / amax and
 *      s = amax / FMAX, IEEE divisions rounded to nearest, inv = s = 1 when amax == 0 or inv is +inf; q = satfinite RNE(o * inv). FMAX is
 *      448 (e4m3) or 57344 (e5m2).
 * q: [rows, row_len] of wire_dtype. scales: [rows, row_len / block] fp32, row-major: the block_rows = 1, block_cols = block layout of
 * b200collBlockScale, so q and scales are also an input of b200collAllGatherBlockScaled.
 * Equivalence: the result is b200collAllReduceRmsNorm's out quantised by b200collAllToAllvQuantized's rule, bit for bit. Step 6 quantises
 * the rounded o, not the fp32 product, which is what makes this hold (for fp32 the two are the same). A block whose o holds a NaN comes
 * out as NaN codes throughout with a NaN scale: a NaN in h makes the whole row's o NaN, as does an all-zero row with eps = 0, and an inf
 * in h makes that element's o NaN and the rest of the row +-0 (inv = 0), so its block is NaN and the others are zeros with s = 1. An
 * all-zero row with eps > 0 gives q = 0 and s = 1.
 * Arguments: everything b200collAllReduceRmsNorm refuses is refused the same way (with q in place of out). Also InvalidArgument, before
 * anything is launched: wire_dtype not e4m3 or e5m2; block not 16, 32, 64, 128, 256 or 512; row_len % block != 0; q not 16-byte aligned
 * or scales not 4-byte aligned; q or scales null when rows > 0; any overlap among x, residual, gamma, q and scales. rows == 0 behaves as
 * in b200collAllReduceRmsNorm.
 * Algorithms and placement as in b200collAllReduceRmsNorm, with q and scales in place of out: the tuner's all-reduce pick for
 * rows * row_len * sizeof(dtype) bytes, or the forced algorithm; ll, ll2 and oneshot -> oneshot; twoshot and nvls -> twoshot, which
 * needs residual, q and scales in the arena and falls back to oneshot otherwise. Two-shot pushes FP8 rows and scales to the peers,
 * row_len * (1 + 4 / block) bytes per row instead of row_len * sizeof(dtype). B200COLL_CHECK=1 cross-checks rows, row_len, the x offset,
 * the algorithm, the two-shot offsets of residual, q and scales, and (block, wire_dtype). The kernel ends with a releasing barrier, so the
 * caller may overwrite x right after the call. b200collStats count an allreduce of rows * row_len * sizeof(dtype) bytes under oneshot,
 * twoshot or copy, one kernel launch. */
b200collResult_t b200collAllReduceRmsNormQuantized(const void* x, void* residual, const void* gamma, void* q, float* scales, size_t rows,
                                                   size_t row_len, float eps, b200collDataType_t dtype, b200collDataType_t wire_dtype,
                                                   int block, b200collComm_t comm, b200collStream_t stream);
/* Fused reduce-scatter, residual add and RMSNorm for sequence-parallel layers (Megatron-style sequence parallelism: the residual stream
 * and the norms are sharded along the sequence), one kernel per call, with the all-gather for the next column-parallel GEMM fused in
 * when `gather` is 1.
 * Shapes: x is this rank's [rows, row_len] partial sums; rows % nranks == 0 and S = rows / nranks. residual is this rank's shard
 * [S, row_len], rows [rank * S, (rank + 1) * S) of the residual stream, updated in place. gamma is [row_len]. All of `dtype`.
 * Result: steps 1-5 are exactly b200collAllReduceRmsNorm's, applied to the rows of slice `rank` (6 for the quantised call, exactly
 * b200collAllReduceRmsNormQuantized's). Equivalence, bit for bit: stack the N ranks' shards into a full residual R; then the new shards
 * are b200collAllReduceRmsNorm(x, R, ...)'s new residual slice by slice, out (q, scales) is that call's output rows of slice `rank`, and
 * with gather every rank's full out (q, scales) is that call's out.
 * gather == 0: out [S, row_len] (q [S, row_len], scales [S, row_len / block]), any device buffer, written by the local rank only.
 * gather == 1: out [rows, row_len] (q [rows, row_len], scales [rows, row_len / block]); rank r pushes slice r into every rank, so every
 * rank ends with all rows. These must be arena memory at the same offsets on every rank, else InvalidUsage: there is no fallback, as no
 * rank holds another rank's residual.
 * Placement: with more than one rank, x in the arena at the same offset on every rank, else InvalidUsage. residual and gamma may be any
 * device buffers; only the local rank reads or writes residual. gather must be the same on every rank. B200COLL_CHECK=1 cross-checks
 * (rows, row_len, gather), the x offset, the out (q, scales) offsets when gathering, and (block, wire_dtype) on multi-process
 * communicators.
 * Algorithm: one with more than one rank (rank r pulls rows [r*S, (r+1)*S) of every rank's x, as two-shot does); the tuner and
 * b200collCommSetAlgo do not apply, and forcing oneshot or ll changes nothing. One rank: S == rows, gather is irrelevant, and the call
 * runs b200collAllReduceRmsNorm's (...Quantized's) local kernel. b200collStats count a reducescatter of S * row_len * sizeof(dtype) bytes
 * under twoshot (copy with one rank), one kernel launch.
 * Arguments (InvalidArgument, nothing launched): everything the all-reduce form refuses, with residual sized [S, row_len] and out (q,
 * scales) sized by S or, gathering, by rows in the alignment and overlap checks; rows % nranks != 0; gather not 0 or 1. rows == 0 still
 * launches on every rank and touches nothing. The kernel ends with a releasing barrier, so the caller may overwrite x right after the
 * call. */
b200collResult_t b200collReduceScatterRmsNorm(const void* x, void* residual, const void* gamma, void* out, size_t rows, size_t row_len,
                                              float eps, int gather, b200collDataType_t dtype, b200collComm_t comm, b200collStream_t stream);
b200collResult_t b200collReduceScatterRmsNormQuantized(const void* x, void* residual, const void* gamma, void* q, float* scales, size_t rows,
                                                       size_t row_len, float eps, int gather, b200collDataType_t dtype,
                                                       b200collDataType_t wire_dtype, int block, b200collComm_t comm, b200collStream_t stream);

/* Ulysses all-to-all for sequence-parallel attention (DeepSpeed-Ulysses), one kernel per call for 1 to 3 tensors (q, k and v, or one
 * attention output) of one element type and one batch, seq_local and head_dim. N ranks, B = batch, S_l = seq_local, S = N * S_l,
 * D = head_dim. Tensor i has heads H_i, counted in the full (unsharded) layout, and two sides:
 *   seq:  the sequence-sharded side [B, S_l, H_i, D], row-strided: token row (b, t) starts row_stride elements after row (b, t - 1) (and
 *         row (b, 0) after (b - 1, S_l - 1)), and holds H_i * D contiguous elements. A column slice of a packed [B * S_l, (Hq + 2 Hkv) * D]
 *         QKV projection output has this shape.
 *   head: the head-sharded side, dense [B, S, Hl_i, D].
 * SeqToHeads (before attention): on rank r, head[b, s * S_l + t, j, :] = seq of rank s [b, t, head_i(r, j), :], where
 *   H_i % N == 0:  Hl_i = H_i / N and head_i(r, j) = r * H_i / N + j;
 *   else N % H_i == 0 (fewer KV heads than ranks, MQA included):  Hl_i = 1 and head_i(r, 0) = floor(r * H_i / N), the KV head of rank r's
 *   query heads whenever Hq % N == 0; each source head goes to N / H_i ranks;
 *   anything else is InvalidArgument.
 * HeadsToSeq (after attention), the inverse layout move: on rank r, seq[b, t, h, :] = head of rank h / (H_i / N) [b, r * S_l + t,
 * h % (H_i / N), :]. It needs H_i % N == 0 (the replicated layout is refused: its inverse is a sum over the replicas). HeadsToSeq of
 * SeqToHeads is the identity for every tensor that is not replicated.
 * Values: a bit copy (NaN payloads, -0 and inf survive), no cast and no scale. dtype bf16, fp16, fp32, e4m3 or e5m2.
 * Arguments (InvalidArgument, message in b200collGetLastError, nothing launched): ntensors not in [1, 3]; head_dim * sizeof(dtype) not a
 * positive multiple of 16; heads <= 0; a pointer not 16-byte aligned, or null when B * S_l > 0; row_stride < heads * head_dim, or
 * row_stride * sizeof(dtype) not a multiple of 16; B * S_l >= 2^31; more than 2^31 - 1 16-byte vectors per rank in one side of a tensor or
 * moved by the call; an output (head for SeqToHeads, seq for HeadsToSeq) overlapping any source or another output (column slices of one
 * buffer with one row stride overlap only where their columns meet).
 * Placement, as b200collAllToAllv (the kernel pushes): with more than one rank every output must be arena memory at the same offset on
 * every rank, else InvalidUsage (there is no staging path); sources may be any device buffer, as only their own rank reads them. Shapes
 * must be equal on every rank; B200COLL_CHECK=1 cross-checks the direction, ntensors, B, S_l, D, dtype, every heads, row_stride and output
 * offset on multi-process communicators and turns a disagreement into InvalidUsage. B * S_l == 0 (then the same on every rank) returns
 * without a launch. A poisoned communicator gives RemoteError. The kernel ends with a releasing barrier, so the outputs may be read and the
 * sources overwritten by the next operation on the stream. The host reads no device data, so the call can be captured in a CUDA graph.
 * One rank: a local strided copy, no barrier, any device buffers (splitting a packed QKV into dense q, k and v).
 * b200collStats count an alltoall of the source bytes (B * S_l * H_i * D * sizeof(dtype) summed over the tensors) under twoshot (copy with
 * one rank), one kernel launch. The tuner and b200collCommSetAlgo do not apply. */
typedef struct {
  void* seq;            /* the sequence-sharded side: source of SeqToHeads, destination of HeadsToSeq */
  size_t row_stride;    /* elements between consecutive token rows of seq (>= heads * head_dim) */
  void* head;           /* the head-sharded side, dense: destination of SeqToHeads, source of HeadsToSeq */
  int heads;            /* H_i, in the full layout */
} b200collUlyssesTensor;
b200collResult_t b200collAllToAllSeqToHeads(const b200collUlyssesTensor* tensors, int ntensors, size_t batch, size_t seq_local,
                                            size_t head_dim, b200collDataType_t dtype, b200collComm_t comm, b200collStream_t stream);
b200collResult_t b200collAllToAllHeadsToSeq(const b200collUlyssesTensor* tensors, int ntensors, size_t batch, size_t seq_local,
                                            size_t head_dim, b200collDataType_t dtype, b200collComm_t comm, b200collStream_t stream);

/* Context parallelism, all-gather form (Llama 3's long-context training, cp_comm_type "all_gather" in Megatron / TransformerEngine):
 * each rank keeps its query shard and gathers K and V over the whole sequence before attention (AllGatherContext); after it, the
 * full-sequence dK and dV, partial sums over the rank's own queries, are reduce-scattered back to the sequence shards
 * (ReduceScatterContext). One kernel per call for 1 to 3 tensors (K and V, or MLA's c_kv and k_pe) of one element type and one batch,
 * seq_local and chunks. N ranks, B = batch, S_l = seq_local, S = N * S_l, C = chunks. Tensor i has width W_i elements per token and
 * two sides:
 *   shard: this rank's [B, S_l, W_i], row-strided: token row (b, t) starts row_stride elements after row (b, t - 1) (and row (b, 0)
 *          after (b - 1, S_l - 1)), and holds W_i contiguous elements. A column slice of a packed QKV (or dQKV) tensor has this shape.
 *   full:  dense [B, S, W_i], tokens in sequence order.
 * Layout. C is 1 or 2; c = S_l / C. Local token t of rank r has k = t / c, u = t % c and global token gtok(r, t) = G(r, k) * c + u with
 *   G(r, 0) = r,  G(r, 1) = 2N - 1 - r.
 * C = 1 is contiguous sharding; C = 2 is the load-balanced causal layout (the sequence cut into 2N chunks, rank r holding chunks r
 * and 2N - 1 - r), and needs S_l even.
 * AllGatherContext: on every rank, full[b, gtok(s, t), :] = shard of rank s [b, t, :] for every rank s. A bit copy (NaN payloads, -0 and
 * inf survive); dtype bf16, fp16, fp32, e4m3 or e5m2.
 * ReduceScatterContext: on rank r, shard[b, t, :] = round_once(((+0 + full_0[b, g, :]) + full_1[b, g, :]) + .. + full_{N-1}[b, g, :])
 * with g = gtok(r, t) and full_s rank s's full: summed in fp32 in rank order (the order table above) and rounded once to nearest even;
 * dtype bf16, fp16 or fp32. With one rank it is a bit copy, as b200collReduceScatter is.
 * Arguments (InvalidArgument, message in b200collGetLastError, nothing launched): ntensors not in [1, 3]; chunks not 1 or 2, or 2 with
 * S_l odd; W_i * sizeof(dtype) not a positive multiple of 16; row_stride < W_i, or row_stride * sizeof(dtype) not a multiple of 16; a
 * pointer not 16-byte aligned, or null when B * S_l > 0; B * S_l >= 2^31; more than 2^31 - 1 16-byte vectors in one side of a tensor
 * or moved by the call; a dtype outside the lists above; an output (full for the gather, shard for the reduce-scatter) overlapping any
 * source or another output (column slices of one buffer with one row stride overlap only where their columns meet).
 * Placement: with more than one rank every full must be arena memory at the same offset on every rank, else InvalidUsage (the gather
 * pushes into it, the reduce-scatter pulls from it; there is no staging path); shard may be any device buffer, as only its own rank
 * touches it. With one rank any device buffers. Shapes must be equal on every rank; B200COLL_CHECK=1 cross-checks the direction,
 * ntensors, dtype, B, S_l, C, and every W_i, row_stride and full offset on multi-process communicators and turns a disagreement into
 * InvalidUsage. B * S_l == 0 (then the same on every rank) returns without a launch. A poisoned communicator gives RemoteError. The
 * kernel starts with a barrier (no rank stores into or reads a full that an earlier operation on a peer's stream still uses) and ends
 * with a releasing one, so the outputs may be read and the sources overwritten by the next operation on the stream. The host reads no
 * device data, so both calls can be captured in a CUDA graph. One rank: a local strided copy, no barrier.
 * b200collStats count an allgather (AllGatherContext) or a reducescatter (ReduceScatterContext) of the shard bytes (B * S_l * W_i *
 * sizeof(dtype) summed over the tensors) under twoshot (copy with one rank), one kernel launch. The tuner and b200collCommSetAlgo do
 * not apply. */
typedef struct {
  void* shard;          /* this rank's [B, S_l, W] rows, row-strided: source of the gather, destination of the reduce-scatter */
  size_t row_stride;    /* elements between consecutive token rows of shard (>= width) */
  void* full;           /* dense [B, S, W] in token order: destination of the gather, source of the reduce-scatter */
  size_t width;         /* W, elements per token row (Hkv * D for K or V) */
} b200collContextTensor;
b200collResult_t b200collAllGatherContext(const b200collContextTensor* tensors, int ntensors, size_t batch, size_t seq_local, int chunks,
                                          b200collDataType_t dtype, b200collComm_t comm, b200collStream_t stream);
b200collResult_t b200collReduceScatterContext(const b200collContextTensor* tensors, int ntensors, size_t batch, size_t seq_local, int chunks,
                                              b200collDataType_t dtype, b200collComm_t comm, b200collStream_t stream);

/* FSDP / ZeRO-3, dim-0 sharding (torch.distributed.fsdp.fully_shard's Shard(0)): before forward each rank gathers a unit's parameters
 * from their shards, casting them on the owning rank (AllGatherShards); after backward the unit's gradients are reduce-scattered back
 * to the shards, summed in fp32, scaled and optionally added to the gradient already there (ReduceScatterShards). One kernel per call
 * for 1 to 64 tensors (one unit: a Llama block has 9) sharing one pair of dtypes. N ranks, this rank r. Tensor i has rows d_i (its
 * unsharded dim 0), width W_i (the product of its other dims) and shard_rows p_i, the rows per rank, with N * p_i >= d_i (FSDP2 uses
 * p_i = ceil(d_i / N); a caller may round it up to meet the alignment rule below). Rank s owns rows [s * p_i, s * p_i + n_s) with
 *   n_s = clamp(d_i - s * p_i, 0, p_i)
 * (a 3-row tensor on 8 ranks leaves ranks 3 .. 7 with none). Two sides:
 *   shard: this rank's rows, dense [>= n_r, W_i]; rows n_r .. p_i - 1 (padding) are never read or written.
 *   full:  the unsharded tensor, dense [d_i, W_i], no padding.
 * AllGatherShards: on every rank, full[s * p_i + j, :] = cast(shard of rank s [j, :]) for every rank s and j < n_s. Pairs (shard ->
 * full): one dtype in and out (bf16, fp16, fp32, e4m3 or e5m2), a bit copy (NaN payloads, -0 and inf survive); or fp32 -> bf16 or
 * fp16, IEEE round to nearest even with overflow to inf, as Tensor.to (NaN stays NaN, its payload not kept). The cast runs on the
 * owning rank, before the push, so the narrow type is what crosses NVLink.
 * ReduceScatterShards: on rank r, for j < n_r and e = (r * p_i + j, :), every step in fp32 with no FMA contraction:
 *   t = ((+0 + full_0[e]) + full_1[e]) + .. + full_{N-1}[e]     (full_s rank s's full; rank order, the order table above)
 *   t = t * scale
 *   t = (float)shard[j, :] + t                                 if accumulate
 *   shard[j, :] = round_once(t)                                 to nearest even; fp16 overflows to inf
 * Pairs (full -> shard): bf16 -> bf16, fp16 -> fp16, fp32 -> fp32, bf16 -> fp32, fp16 -> fp32. With one rank, one dtype, scale == 1
 * and accumulate == 0 it is a bit copy, as b200collReduceScatter is; in every other case the formula holds with N = 1.
 * Arguments (InvalidArgument, message in b200collGetLastError, nothing launched): ntensors not in [1, 64]; a dtype pair outside the
 * lists above; d_i, W_i or p_i zero; N * p_i < d_i; p_i * W_i or d_i * W_i not a multiple of 16 bytes in either dtype; a pointer not
 * 16-byte aligned, full null, or shard null when n_r > 0; more than 2^31 - 1 16-byte vectors in a side of a tensor or in sum p_i * W_i;
 * an output (full for the gather, this rank's n_r rows of shard for the reduce-scatter) overlapping any source or another output.
 * Placement: with more than one rank every full must be arena memory at the same offset on every rank, else InvalidUsage (the gather
 * pushes into it, the reduce-scatter pulls from it; there is no staging path: gradients reach the arena through the communicator's
 * memory pool); shard may be any device buffer, as only its own rank touches it. With one rank any device buffers. Shapes, dtypes,
 * scale and accumulate must be equal on every rank; B200COLL_CHECK=1 cross-checks the direction, ntensors, both dtypes, the bits of
 * scale, accumulate, and every d_i, W_i, p_i and full offset on multi-process communicators and turns a disagreement into InvalidUsage.
 * A poisoned communicator gives RemoteError. The kernel starts with a barrier (no rank stores into or reads a full that an earlier
 * operation on a peer's stream still uses) and ends with a releasing one, so the outputs may be read and the sources overwritten by the
 * next operation on the stream. Every rank launches the same grid, sized from sum p_i * W_i, so a rank with no rows still takes part.
 * The host reads no device data, so both calls can be captured in a CUDA graph. One rank: a local copy or reduction, no barrier.
 * b200collStats count an allgather (AllGatherShards) or a reducescatter (ReduceScatterShards) of this rank's rows in the full dtype
 * (n_r * W_i * sizeof(full dtype) summed over the tensors) under twoshot (copy with one rank), one kernel launch. The tuner and
 * b200collCommSetAlgo do not apply. */
typedef struct {
  void* shard;          /* this rank's rows, dense [>= n_r, W]: source of the gather, destination of the reduce-scatter */
  void* full;           /* dense [rows, W]: destination of the gather, source of the reduce-scatter */
  size_t rows;          /* d, the unsharded dim 0 */
  size_t width;         /* W, the product of the other dims */
  size_t shard_rows;    /* p, rows per rank (N * p >= d) */
} b200collShardTensor;
b200collResult_t b200collAllGatherShards(const b200collShardTensor* tensors, int ntensors, b200collDataType_t shard_dtype,
                                         b200collDataType_t full_dtype, b200collComm_t comm, b200collStream_t stream);
b200collResult_t b200collReduceScatterShards(const b200collShardTensor* tensors, int ntensors, b200collDataType_t full_dtype,
                                             b200collDataType_t shard_dtype, float scale, int accumulate, b200collComm_t comm,
                                             b200collStream_t stream);

/* Vocab-parallel cross-entropy for a tensor-parallel LM head (Megatron's vocab_parallel_cross_entropy), one kernel per direction
 * (src/xent.cu). N ranks, this rank r, Vl = vocab_local. logits: this rank's dense [rows, Vl] of `dtype` (bf16, fp16 or fp32), its
 * columns being the global vocabulary ids [r * Vl, (r + 1) * Vl) (Megatron's uniform split). target: [rows] int64 global ids, THE SAME
 * ON EVERY RANK (the caller's condition; nothing checks it). loss, lse, dloss: [rows] fp32. Every product and sum is an IEEE fp32 op
 * rounded on its own (no fused multiply-add); exp and log are the library's own fixed sequences of fp32 multiplies, adds, rint and
 * exponent-bit arithmetic (no hardware approximation), within 1 ulp of the exact value, exp(0) == 1, exp(x) == +0 for x < -87,
 * exp(x) == +inf for x > 88.7228317, log(1) == 0, log(+0) == -inf; tests/coll_xent_reference.py mirrors both in numpy. Per row t:
 *   1. On rank r, with x the widened logits of the row:
 *        m_r = max_j x_j, NaN if any x_j is NaN (+inf if any is +inf and none is NaN);
 *        s_r = sum_j exp(x_j - m_r): the sums of the 16-element chunks (columns 16c .. 16c+15, the last one short) in column order from
 *              +0, padded with +0 to a power of two P and folded p = p[:P/2] + p[P/2:] until one value is left; s_r = +0 if m_r = -inf;
 *        z_r = x_{target - r * Vl} if 0 <= target - r * Vl < Vl (this rank owns the target).
 *      (m_r, s_r, z_r, owns) is pushed as one 16-byte record into row t of every rank's mailbox.
 *   2. Every rank combines the N records in rank order: M = max_r m_r (NaN-aware), S = ((+0 + e_0) + e_1) + .. + e_{N-1} with
 *      e_r = s_r * exp(m_r - M) (e_r = +0 if m_r = -inf), lse = M + log(S), loss = lse - z with z from the owning rank. If
 *      target == ignore_index, loss = +0; else if target is outside [0, N * Vl), loss = NaN, and nothing outside the row is read. lse is
 *      stored for every row.
 *   Backward (no communication): grad[t, j] = round_dtype((exp(x_j - lse[t]) - [r * Vl + j == target]) * dloss[t]), RNE; +0 on rows with
 *   target == ignore_index, NaN on rows whose target is out of range. grad == logits (the whole buffer) runs in place.
 * Every rank holds the same loss and lse. The result depends only on the values and N, not on the launch shape.
 * Arguments (InvalidArgument, message in b200collGetLastError, nothing launched): dtype not bf16, fp16 or fp32; Vl == 0 or Vl * sizeof(dtype)
 * not a multiple of 16; N * Vl >= 2^31; rows >= 2^31; a null pointer when rows > 0; logits or grad not 16-byte aligned, target not
 * 8-byte aligned, loss, lse or dloss not 4-byte aligned; any overlap among the outputs (loss and lse; grad) and the inputs other than
 * grad == logits. A poisoned communicator gives RemoteError.
 * Placement: every buffer may be any device memory, as only its own rank reads or writes it. The only cross-rank memory is the mailbox,
 * rows * N * 16 bytes of the quantising collectives' scratch (a collective contract like b200collMemAlloc: every rank makes the same
 * calls in the same order; OutOfMemory, before anything is launched, when the arena cannot hold it; a superseded scratch is kept until
 * CommDestroy, so a captured CUDA graph stays valid). rows, Vl, ignore_index and dtype must be equal on every rank; B200COLL_CHECK=1
 * cross-checks them and the mailbox offset on multi-process communicators. The forward starts with a relaxed barrier (every rank has
 * finished the previous user of its mailbox) and publishes the records with a releasing one; rows == 0 still launches on every rank.
 * The host reads no device data, so both calls can be captured in a CUDA graph. One rank: a local kernel, no barrier, no mailbox.
 * b200collStats count the forward as an allreduce of rows * 16 bytes under twoshot (copy with one rank), one kernel launch; the
 * backward as one kernel launch and no operation (rows == 0: nothing). The tuner and b200collCommSetAlgo do not apply. */
b200collResult_t b200collVocabParallelCrossEntropy(const void* logits, const int64_t* target, float* loss, float* lse, size_t rows,
                                                   size_t vocab_local, int64_t ignore_index, b200collDataType_t dtype, b200collComm_t comm,
                                                   b200collStream_t stream);
b200collResult_t b200collVocabParallelCrossEntropyBackward(const void* logits, const int64_t* target, const float* lse, const float* dloss,
                                                           void* grad, size_t rows, size_t vocab_local, int64_t ignore_index,
                                                           b200collDataType_t dtype, b200collComm_t comm, b200collStream_t stream);

/* --- host path (src/hostpath.cu). CommInitRank binds the calling thread to the CPUs of the GPU's NUMA node (B200COLL_AFFINITY=0:
 * leave it alone, 2: restore the previous mask after init). HostAlloc returns pinned, device-mapped host memory on that node.
 * AllReduceHost is the end-to-end step "pinned host -> GPU -> all-reduce -> pinned host" as one asynchronous call on `stream`:
 * tiny messages run as ONE kernel that reads and writes host memory over PCIe, large ones are chunked so that the host-to-device
 * copy of chunk i+1, the all-reduce of chunk i and the copy-back of chunk i-1 overlap. Same call on every rank; staging comes from
 * the symmetric heap on first use (a collective contract, like MemAlloc). */
b200collResult_t b200collHostAlloc(b200collComm_t comm, void** ptr, size_t bytes);
b200collResult_t b200collHostFree(b200collComm_t comm, void* ptr);
b200collResult_t b200collAllReduceHost(const void* host_send, void* host_recv, size_t count, const b200collEpilogue* ep,
                                       b200collRedOp_t op, b200collComm_t comm, b200collStream_t stream);
/* NUMA node of this rank's GPU (-1 unknown) and its local CPU list as sysfs prints it. */
b200collResult_t b200collCommNumaGet(b200collComm_t comm, int* numa_node, char* cpulist, size_t len);
/* Test hook (no GPU needed): what CommInitRank does with the GPU's sysfs directory (files numa_node, local_cpulist): returns the NUMA node
 * read (-1 if absent); with mode != 0 the calling thread's affinity is narrowed to the listed CPUs it is allowed to use (*changed = 1 if so). */
int b200collDebugApplyLocality(const char* sysfs_dir, int mode, int* changed);
/* Test hook: parse a sysfs cpulist ("0-31,64-95") into at most `max` CPU numbers; returns how many. */
int b200collDebugParseCpuList(const char* s, int* cpus, int max);

/* --- point to point (ncclSend / ncclRecv / ncclGroupStart / ncclGroupEnd). `bytes` of opaque data; buffers 16-byte aligned.
 * A send pairs with the peer's recv of the same size, in call order per pair. Everything between GroupStart and GroupEnd
 * (a ring step, a pipeline hand-over, any mix of peers) becomes ONE kernel per communicator, launched at GroupEnd on the
 * stream of the group's first operation; outside a group each call is a group of its own and blocks the stream until the
 * peer arrives (so "send then recv" on both sides of a pair deadlocks exactly as it does with NCCL: group them).
 * The receiver's buffer is written directly over NVLink when it lies in the symmetric arena; otherwise through staging. */
b200collResult_t b200collGroupStart(void);
b200collResult_t b200collGroupEnd(void);
b200collResult_t b200collSend(const void* buf, size_t bytes, int peer, b200collComm_t comm, b200collStream_t stream);
b200collResult_t b200collRecv(void* buf, size_t bytes, int peer, b200collComm_t comm, b200collStream_t stream);
/* Test hook (no GPU needed): plans one group of point-to-point operations for `rank` on a stand-in communicator and writes the
 * launches it would make as text: CTA ranges per operation, direct or staged receive, window layout, follow-up kernels. */
b200collResult_t b200collDebugPlanP2p(int rank, int nranks, int loopback, size_t window, int nops, const int* is_send, const int* peer,
                                      const size_t* bytes, const int* in_arena, char* out, size_t outlen);
/* Test hook (no GPU needed): the launch plan of the one-rank copy-engine copy of `bytes` (a multiple of 16) on a GPU with `sm_count`
 * SMs. [0, bytes) is cut into chunks of `chunk` bytes (the last one shorter) and CTA b of `blocks` copies chunks b, b + blocks, ...:
 * `rounds` of them, or one fewer. `max_resident` is how many of its CTAs fit on the GPU at once, which `blocks` never exceeds. */
b200collResult_t b200collDebugPlanCopy(size_t bytes, int sm_count, int* blocks, unsigned* chunk, unsigned* rounds, int* max_resident);

/* --- tuner (libnccl-tuner.so analogue). */
b200collAlgo_t b200collTunerPick(b200collOp_t op, size_t bytes, int nranks, int nvls_available);
/* Force an algorithm for subsequent calls on this comm (b200collAlgoAuto restores the table). */
b200collResult_t b200collCommSetAlgo(b200collComm_t comm, b200collAlgo_t algo);
b200collAlgo_t b200collCommGetAlgo(b200collComm_t comm);   /* what SetAlgo (or B200COLL_ALGO) last forced; Auto = the tuner decides */
b200collResult_t b200collCommSetMaxCtas(b200collComm_t comm, int max_ctas);
/* Receives into buffers outside the arena go through two staging windows per operation; this caps the window size (a multiple of
 * 512 bytes; 0 = an equal share of the 64 MiB staging area). A private choice of the receiver: the sender follows what is posted. */
b200collResult_t b200collCommSetP2pWindow(b200collComm_t comm, size_t bytes);
/* Launch shape per kernel family: kind 0 = NVLS all-reduce/all-gather, 1 = P2P pull/push kernels, 2 = LL, 3 = NVLS reduce-scatter, 4 = NVLS broadcast / reduce (root only).
 * max_ctas <= 0 keeps the current cap; threads == 0 lets the library pick {128,256,512} by work size.
 * Defaults: NVLS wants few CTAs (32 x 256 threads); LL and rooted NVLS ops run one CTA per SM. */
b200collResult_t b200collCommSetLaunchShape(b200collComm_t comm, int kind, int max_ctas, int threads);
const char* b200collAlgoName(b200collAlgo_t a);
size_t b200collTypeSize(b200collDataType_t t);

/* --- start-up self check (guest-config-checker analogue, reference: gpudirect-tcpxo/README.md:84,239).
 * Writes a human-readable report into buf; returns b200collSuccess iff the box can run the fast paths. */
b200collResult_t b200collSelfCheck(char* buf, size_t buflen);

#ifdef __cplusplus
}
#endif
#endif /* B200COLL_H_ */
