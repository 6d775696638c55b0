// libb200coll Ulysses all-to-all for sequence-parallel attention (DeepSpeed-Ulysses): q, k and v move from sequence shards to head
// shards before attention (b200collAllToAllSeqToHeads), and the attention output moves back (b200collAllToAllHeadsToSeq), one kernel
// per call for up to three tensors:
//
//   k_ulysses<S2H, LOCAL>   S2H: sequence -> heads, else heads -> sequence. LOCAL: one rank, a strided copy with no barrier. Otherwise
//                           relaxed barrier, push every segment straight into its final place in the peer's output, releasing barrier
//
// Geometry (the header states it as formulas). Rows are the B * S_l token rows (b, t) of this rank's sequence shard. Tensor i has H_i
// heads of D elements; Hl_i = H_i / N heads per rank, or 1 when N % H_i == 0 (fewer KV heads than ranks: head h is replicated to the
// ranks h * N / H_i .. (h + 1) * N / H_i - 1). A *segment* is the Hl_i * D elements of one row that are contiguous both on the sequence
// side (row-strided, row_stride_i elements apart) and on the head side (dense [B, S, Hl_i, D]). Segment g of a row is heads
// [g * Hl_i, (g + 1) * Hl_i): it goes to (sequence -> heads) or comes from (heads -> sequence) rank g, or in the replicated case the N / H_i
// ranks that share KV head g. In 16-byte vectors, with seg = Hl_i * D * sizeof(dtype) / 16 and row = b * S_l + t:
//   sequence side of rank X:  seq  + row * row_stride_v + g * seg + v
//   head side of rank Y:      head + (row + b * (N - 1) * S_l + Y * S_l) * seg + v     (= token b * S + Y * S_l + t)
// Sequence -> heads reads the sequence side at g and writes the head side of rank g at Y = me; heads -> sequence reads the head side at
// Y = g and writes the sequence side of rank g at X = me.
//
// Work. The (tensor, segment g, row, vector) space is flattened with a prefix over the tensors, as A2AvArgs does over the peers, so one
// tensor or a skewed mix of q, k and v still spreads over every CTA; within a tensor, segments run in the staggered order g0, g0 + 1, ...
// (g0 = the segment of rank me + 1), so that the ranks do not all start on the same peer. Each thread keeps U 16-byte loads in flight,
// as k_a2av_push does, and stores each vector once, or once per replica. Indices are 32-bit (the host caps every vector count at
// 2^31 - 1) and divided by precomputed multipliers (FastDiv) instead of integer division.
//
// Ordering. The argument of the two-shot kernels. The entry barrier is relaxed: a rank arrives only once its stream has reached this
// call, so everything earlier on its stream (an attention kernel still reading last layer's output) is done before any peer stores into
// its outputs, and every source was written by an earlier kernel on its own rank's stream. Sources are read by their own rank only. The
// closing barrier is releasing: when a rank leaves it, every peer's pushes into its outputs are visible, so the next kernel on its stream
// may read them, and its sources may be overwritten. Both barriers pair CTA b with CTA b; every rank launches the same grid, because the
// shapes (and so the work) are equal on every rank.
#include <stdint.h>

#include <atomic>
#include <mutex>
#include <string>

#include "comm.h"
#include "index.cuh"
#include "launch.cuh"

namespace b200coll {

constexpr int kUlyThreads = 512;
constexpr int kUlyUnroll = 4;
constexpr int kUlyMaxTensors = 3;
constexpr size_t kI31 = ((size_t)1 << 31) - 1;

struct UlyTensor {
  const char* src;                 // this rank's source
  unsigned long long dst;          // the output: its arena offset (every rank's is the same), or with LOCAL its address
  unsigned long long row_stride;   // vectors between the sequence side's rows
  FastDiv seg;                     // vectors per segment
  uint32_t groups;                 // segments per row: N, or H_i when replicated
  uint32_t g0;                     // the first segment in the staggered order
  uint32_t rep;                    // destination ranks per segment: 1, or N / H_i
};

struct UlyArgs {
  UlyTensor t[kUlyMaxTensors];
  uint32_t prefix[kUlyMaxTensors + 1];   // vectors before tensor i
  FastDiv rows;                          // B * S_l
  FastDiv seq_local;                     // S_l
  uint32_t ntensors;
};

template <bool S2H, bool LOCAL>
__global__ void __launch_bounds__(kUlyThreads) k_ulysses(COMM_PARAM, const __grid_constant__ UlyArgs a, uint32_t op) {
  pdl_prologue();
  constexpr int U = kUlyUnroll;
  uint32_t s = 0;
  if (!LOCAL) {
    s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;        // every rank is done with the previous contents of its outputs
  }
  const uint32_t total = a.prefix[a.ntensors];
  const uint32_t me = LOCAL ? 0u : (uint32_t)c.rank, nr = LOCAL ? 1u : (uint32_t)c.nranks;
  const uint32_t sl = a.seq_local.d;
  const uint32_t stride = gridDim.x * blockDim.x * U;
  for (uint32_t base = blockIdx.x * blockDim.x * U + threadIdx.x; base < total; base += stride) {
    uint4 d[U];
    unsigned long long off[U];    // the destination: its address (LOCAL) or its arena offset on every destination rank
    uint32_t first[U], rep[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const uint32_t g = base + (uint32_t)u * blockDim.x;
      rep[u] = 0; first[u] = 0; off[u] = 0;
      if (g < total) {
        uint32_t i = 0;
#pragma unroll
        for (int q = 1; q < kUlyMaxTensors; q++) if ((uint32_t)q < a.ntensors && g >= a.prefix[q]) i = q;
        const UlyTensor& t = a.t[i];
        const uint32_t l = g - a.prefix[i];
        const uint32_t jrow = div_by(l, t.seg), v = l - jrow * t.seg.d;
        const uint32_t j = div_by(jrow, a.rows), row = jrow - j * a.rows.d;
        uint32_t grp = t.g0 + j; if (grp >= t.groups) grp -= t.groups;
        const uint32_t b = div_by(row, a.seq_local);
        const unsigned long long seq_v = (unsigned long long)row * t.row_stride + v;              // + X * seg
        const unsigned long long head_v = ((unsigned long long)row + (unsigned long long)b * (nr - 1) * sl) * t.seg.d + v;   // + Y * S_l * seg
        const unsigned long long src_v = S2H ? seq_v + (unsigned long long)grp * t.seg.d : head_v + (unsigned long long)grp * sl * t.seg.d;
        off[u] = t.dst + 16ull * (S2H ? head_v + (unsigned long long)me * sl * t.seg.d : seq_v + (unsigned long long)me * t.seg.d);
        first[u] = grp * t.rep; rep[u] = t.rep;
        d[u] = ld_vec(t.src + 16ull * src_v);
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (LOCAL) {
        if (rep[u]) st_vec(reinterpret_cast<char*>(off[u]), d[u]);
      } else {
        for (uint32_t k = 0; k < rep[u]; k++) st_vec(c.peer[first[u] + k] + off[u], d[u]);
      }
    }
  }
  if (!LOCAL) {
    if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;          // publishes the pushes; nobody reads my sources any more
    if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
  }
}

// Once per device, before the first kernel of this family launches: load all four. With lazy module loading a kernel's first launch
// loads it, and the load waits for kernels already running; with virtual ranks, a rank whose first Ulysses launch came behind its own
// barrier kernel, which waits for another rank's launch on the same thread, would never get there.
static void ulysses_preload(const b200collComm* c) {
  static std::atomic<unsigned long long> done{0};
  static std::mutex mu;
  const unsigned long long bit = 1ull << (c->device & 63);
  if (done.load(std::memory_order_acquire) & bit) return;
  const std::lock_guard<std::mutex> lk(mu);
  if (done.load(std::memory_order_acquire) & bit) return;
  cudaFuncAttributes fa;
  cudaFuncGetAttributes(&fa, k_ulysses<true, false>);
  cudaFuncGetAttributes(&fa, k_ulysses<true, true>);
  cudaFuncGetAttributes(&fa, k_ulysses<false, false>);
  cudaFuncGetAttributes(&fa, k_ulysses<false, true>);
  done.fetch_or(bit, std::memory_order_acq_rel);
}

static b200collResult_t ulysses(b200collComm* c, bool s2h, const b200collUlyssesTensor* ts, int ntensors, size_t batch, size_t seq_local,
                                size_t head_dim, b200collDataType_t dtype, b200collStream_t stream) {
  const std::string who = s2h ? "all-to-all seq->heads: " : "all-to-all heads->seq: ";
  auto refuse = [&](const std::string& msg) { set_last_error(who + msg); return b200collInvalidArgument; };
  if (!c) return refuse("null communicator");
  if (ntensors < 1 || ntensors > kUlyMaxTensors) return refuse("ntensors must be 1, 2 or 3");
  if (!ts) return refuse("null tensor array");
  const size_t es = b200collTypeSize(dtype);
  if (dtype != b200collBfloat16 && dtype != b200collFloat16 && dtype != b200collFloat32 && !is_fp8(dtype))
    return refuse("dtype must be bf16, fp16, fp32, e4m3 or e5m2");
  if (head_dim == 0 || head_dim >= ((size_t)1 << 31) || (head_dim * es) % 16 != 0) return refuse("head_dim * sizeof(dtype) must be a positive multiple of 16 bytes");
  const size_t N = (size_t)c->nranks, rows = batch * seq_local;
  if (seq_local >= ((size_t)1 << 31) || batch >= ((size_t)1 << 31) || rows >= ((size_t)1 << 31)) return refuse("batch * seq_local must be below 2^31");
  const size_t dv = head_dim * es / 16;           // vectors per head
  UlyArgs a = {};
  Span src[kUlyMaxTensors], dst[kUlyMaxTensors];
  size_t total = 0, src_bytes = 0;
  for (int i = 0; i < ntensors; i++) {
    const b200collUlyssesTensor& t = ts[i];
    const std::string ti = "tensor " + std::to_string(i) + ": ";
    if (t.heads <= 0) return refuse(ti + "heads must be positive");
    const size_t H = (size_t)t.heads;
    const bool replicated = H % N != 0;
    if (replicated && N % H != 0) return refuse(ti + "heads (" + std::to_string(H) + ") must be a multiple or a divisor of nranks (" + std::to_string(N) + ")");
    if (replicated && !s2h) return refuse(ti + "heads (" + std::to_string(H) + ") must be a multiple of nranks (" + std::to_string(N) + "): the replicated layout has no inverse move");
    const size_t hl = replicated ? 1 : H / N;
    if (H > ((size_t)1 << 31) / head_dim) return refuse(ti + "heads * head_dim must be below 2^31");
    if (t.row_stride < H * head_dim) return refuse(ti + "row_stride must be at least heads * head_dim");
    if (t.row_stride > kI31 * 16) return refuse(ti + "more than 2^31 - 1 16-byte vectors per rank");   // keeps the extent below in 64 bits
    if ((t.row_stride * es) % 16 != 0) return refuse(ti + "row_stride * sizeof(dtype) must be a multiple of 16 bytes");
    if (rows > 0 && (!t.seq || !t.head)) return refuse(ti + "null pointer");
    if (!aligned(t.seq, 16) || !aligned(t.head, 16)) return refuse(ti + "seq and head must be 16-byte aligned");
    const size_t seg = hl * dv, groups = replicated ? H : N;
    const size_t seq_vecs = rows == 0 ? 0 : (rows - 1) * (t.row_stride * es / 16) + H * dv;   // the sequence side's extent
    const size_t head_vecs = rows * N * seg;                                                  // B * S * Hl * D
    const size_t moved = rows * H * dv;                                                       // source vectors
    if (seq_vecs > (size_t)kI31 || head_vecs > (size_t)kI31 || moved > (size_t)kI31 - total)
      return refuse(ti + "more than 2^31 - 1 16-byte vectors per rank");
    const Span seq_span = {(uintptr_t)t.seq, rows, t.row_stride * es, H * head_dim * es};
    const Span head_span = {(uintptr_t)t.head, 1, head_vecs * 16, head_vecs * 16};
    src[i] = s2h ? seq_span : head_span;
    dst[i] = s2h ? head_span : seq_span;
    UlyTensor& u = a.t[i];
    u.src = static_cast<const char*>(s2h ? t.seq : t.head);
    u.row_stride = t.row_stride * es / 16;
    u.seg = fast_div((uint32_t)seg);
    u.groups = (uint32_t)groups;
    u.rep = replicated ? (uint32_t)(N / H) : 1u;
    u.g0 = (uint32_t)(((size_t)(c->rank + 1) % N) / u.rep);
    a.prefix[i] = (uint32_t)total;
    total += moved;
    src_bytes += moved * 16;
  }
  for (int i = ntensors; i <= kUlyMaxTensors; i++) a.prefix[i] = (uint32_t)total;
  a.ntensors = (uint32_t)ntensors;
  for (int i = 0; i < ntensors; i++)
    for (int j = 0; j < ntensors; j++) {
      if (spans_overlap(dst[i], src[j])) return refuse("output " + std::to_string(i) + " overlaps source " + std::to_string(j));
      if (j > i && spans_overlap(dst[i], dst[j])) return refuse("outputs " + std::to_string(i) + " and " + std::to_string(j) + " overlap");
    }
  if (comm_poisoned(c)) return b200collRemoteError;
  const bool local = c->nranks == 1;
  if (!local && rows > 0) {
    for (int i = 0; i < ntensors; i++) {
      const b200collResult_t rc = in_arena(c, who, s2h ? "every output (head)" : "every output (seq)", {{reinterpret_cast<const void*>(dst[i].p), dst[i].extent()}});
      if (rc != b200collSuccess) return rc;
    }
  }
  // B200COLL_CHECK=1: (direction, ntensors, dtype, B, S_l, D) in one exchange, then each tensor's heads, output offset and row stride
  const b200collAlgo_t algo = local ? b200collAlgoCopy : b200collAlgoTwoShot;
  if (!local) {
    const size_t fmt = ((size_t)dtype << 8) | ((size_t)ntensors << 1) | (s2h ? 1 : 0);
    b200collResult_t rc = cross_check(c, b200collOpAllToAll, algo, fmt, batch, (seq_local << 32) | head_dim);
    for (int i = 0; i < ntensors && rc == b200collSuccess; i++)
      rc = cross_check(c, b200collOpAllToAll, algo, (size_t)ts[i].heads, rows > 0 ? arena_off(c, reinterpret_cast<const void*>(dst[i].p)) : 0,
                       ts[i].row_stride);
    if (rc != b200collSuccess) return rc;
  }
  if (rows == 0) return b200collSuccess;
  for (int i = 0; i < ntensors; i++)
    a.t[i].dst = local ? (unsigned long long)dst[i].p : (unsigned long long)arena_off(c, reinterpret_cast<const void*>(dst[i].p));
  a.rows = fast_div((uint32_t)rows);
  a.seq_local = fast_div((uint32_t)seq_local);
  const DeviceScope on_device(c->device);
  ulysses_preload(c);
  account(c, b200collOpAllToAll, src_bytes, algo);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const Grid g = pick_grid(c, kShapeP2p, total, kUlyUnroll);
  const uint32_t op = (uint32_t)b200collOpAllToAll;
  if (s2h) {
    if (local) launch_k(k_ulysses<true, true>, g.blocks, g.threads, st, c->dev, a, op);
    else launch_k(k_ulysses<true, false>, g.blocks, g.threads, st, c->dev, a, op);
  } else {
    if (local) launch_k(k_ulysses<false, true>, g.blocks, g.threads, st, c->dev, a, op);
    else launch_k(k_ulysses<false, false>, g.blocks, g.threads, st, c->dev, a, op);
  }
  LAUNCH_CHECK(c);
  return b200collSuccess;
}

}  // namespace b200coll

using namespace b200coll;

extern "C" {

b200collResult_t b200collAllToAllSeqToHeads(const b200collUlyssesTensor* tensors, int ntensors, size_t batch, size_t seq_local, size_t head_dim,
                                            b200collDataType_t dtype, b200collComm_t comm, b200collStream_t stream) {
  return ulysses(comm, true, tensors, ntensors, batch, seq_local, head_dim, dtype, stream);
}

b200collResult_t b200collAllToAllHeadsToSeq(const b200collUlyssesTensor* tensors, int ntensors, size_t batch, size_t seq_local, size_t head_dim,
                                            b200collDataType_t dtype, b200collComm_t comm, b200collStream_t stream) {
  return ulysses(comm, false, tensors, ntensors, batch, seq_local, head_dim, dtype, stream);
}

}  // extern "C"
