// libb200coll context parallelism, all-gather form: K and V gathered over the whole sequence before attention
// (b200collAllGatherContext), and dK and dV reduce-scattered back to the sequence shards after it (b200collReduceScatterContext), one
// kernel per call for up to three tensors:
//
//   k_cp_gather<LOCAL>   relaxed barrier, push every vector of this rank's shard straight into its token's place in every rank's full,
//                        releasing barrier. LOCAL: one rank, a strided copy with no barrier
//   k_cp_rs<T, LOCAL>    relaxed barrier, pull the vector of this rank's token from every rank's full, sum in fp32 in rank order, round
//                        once, store into the shard, releasing barrier. LOCAL: one rank, a strided bit copy with no barrier (one
//                        instantiation serves every dtype)
//
// Geometry (the header states it as formulas). Rows are the B * S_l token rows (b, t) of this rank's shard; tensor i has W_i elements,
// wv_i 16-byte vectors, per row. With c = S_l / C, local token t < c is global token G(me, 0) * c + t, and t >= c is G(me, 1) * c + t - c,
// so the host passes tok0 = me * c and tok1 = (2N - 1 - me) * c - c and the kernel needs no division for it. In vectors:
//   shard:  shard + row * row_stride_v + v
//   full:   full + (b * S + gtok) * wv + v       (the same offset on every rank: each rank's full holds the same tokens)
//
// Work. The (tensor, row, vector) space of this rank's shard is flattened with a prefix over the tensors, as in k_ulysses, so K and V of
// different widths still spread over every CTA. The gather keeps U 16-byte loads in flight per thread and stores each vector to every
// rank, staggered from rank me + 1 so that the ranks do not all start on the same peer; the reduce-scatter issues all N loads of a vector
// before it sums them (the order of the sum is fixed, not the order of the loads). Indices are 32-bit (the host caps every vector count
// at 2^31 - 1) and divided by precomputed multipliers (FastDiv).
//
// Ordering. The argument of the two-shot kernels and k_ulysses. The entry barrier is relaxed: a rank arrives only once its stream has
// reached this call, so a peer's full written by an earlier kernel on the peer's stream is complete before anyone pulls it, and a full
// still read by an earlier kernel (last layer's attention) is not pushed into. The closing barrier is releasing: when a rank leaves it,
// every push into its full is visible, so the next kernel on its stream may read it, and no peer reads its full any more, so it may be
// overwritten. Shards are touched by their own rank only. Both barriers pair CTA b with CTA b; every rank launches the same grid, because
// the shapes (and so the work) are equal on every rank.
#include <stdint.h>

#include <atomic>
#include <mutex>
#include <string>

#include "comm.h"
#include "index.cuh"
#include "launch.cuh"

namespace b200coll {

constexpr int kCpThreads = 512;
constexpr int kCpUnroll = 4;
constexpr int kCpMaxTensors = 3;
constexpr size_t kCpI31 = ((size_t)1 << 31) - 1;

struct CpTensor {
  char* shard;                     // this rank's shard
  unsigned long long full;         // the full tensor: its arena offset (every rank's is the same), or with LOCAL its address
  unsigned long long row_stride;   // vectors between the shard's rows
  FastDiv width;                   // vectors per token row
};

struct CpArgs {
  CpTensor t[kCpMaxTensors];
  uint32_t prefix[kCpMaxTensors + 1];   // vectors before tensor i
  FastDiv seq_local;                    // S_l
  uint32_t chunk;                       // c = S_l / C
  uint32_t tok0, tok1;                  // gtok(me, t) = tok0 + t for t < c, tok1 + t otherwise
  uint32_t seq;                         // S = N * S_l
  uint32_t ntensors;
};

// Where flattened vector g of this rank's shard lives: its tensor, its vector index in the shard and in the full tensor.
struct CpPlace {
  uint32_t i;
  unsigned long long shard_v, full_v;
};
__device__ __forceinline__ CpPlace cp_place(const CpArgs& a, uint32_t g) {
  uint32_t i = 0;
#pragma unroll
  for (int q = 1; q < kCpMaxTensors; q++) if ((uint32_t)q < a.ntensors && g >= a.prefix[q]) i = q;
  const CpTensor& t = a.t[i];
  const uint32_t l = g - a.prefix[i];
  const uint32_t row = div_by(l, t.width), v = l - row * t.width.d;
  const uint32_t b = div_by(row, a.seq_local), tk = row - b * a.seq_local.d;
  const uint32_t gtok = (tk < a.chunk ? a.tok0 : a.tok1) + tk;
  return CpPlace{i, (unsigned long long)row * t.row_stride + v, ((unsigned long long)b * a.seq + gtok) * t.width.d + v};
}

template <bool LOCAL>
__global__ void __launch_bounds__(kCpThreads) k_cp_gather(COMM_PARAM, const __grid_constant__ CpArgs a, uint32_t op) {
  pdl_prologue();
  constexpr int U = kCpUnroll;
  uint32_t s = 0;
  if (!LOCAL) {
    s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;        // every rank is done with the previous contents of its full
  }
  const uint32_t total = a.prefix[a.ntensors];
  const uint32_t me = LOCAL ? 0u : (uint32_t)c.rank, nr = LOCAL ? 1u : (uint32_t)c.nranks;
  const uint32_t stride = gridDim.x * blockDim.x * U;
  for (uint32_t base = blockIdx.x * blockDim.x * U + threadIdx.x; base < total; base += stride) {
    uint4 d[U];
    unsigned long long off[U];    // the destination: its address (LOCAL) or its arena offset on every rank
    bool act[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const uint32_t g = base + (uint32_t)u * blockDim.x;
      act[u] = g < total; off[u] = 0;
      if (act[u]) {
        const CpPlace p = cp_place(a, g);
        off[u] = a.t[p.i].full + 16ull * p.full_v;
        d[u] = ld_vec(a.t[p.i].shard + 16ull * p.shard_v);
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (!act[u]) continue;
      if (LOCAL) {
        st_vec(reinterpret_cast<char*>(off[u]), d[u]);
      } else {
        for (uint32_t k = 1; k <= nr; k++) {
          uint32_t p = me + k; if (p >= nr) p -= nr;
          st_vec(c.peer[p] + off[u], d[u]);
        }
      }
    }
  }
  if (!LOCAL) {
    if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;          // publishes the pushes; nobody reads my shard any more
    if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
  }
}

template <typename T, bool LOCAL>
__global__ void __launch_bounds__(kCpThreads) k_cp_rs(COMM_PARAM, const __grid_constant__ CpArgs a, uint32_t op) {
  pdl_prologue();
  constexpr int E = Epv<T>::value;
  constexpr int U = LOCAL ? kCpUnroll : 1;       // the peer form has N loads in flight per vector already
  constexpr int R = LOCAL ? 1 : kMaxRanks;
  uint32_t s = 0;
  if (!LOCAL) {
    s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;        // every rank's full is written
  }
  const uint32_t total = a.prefix[a.ntensors];
  const uint32_t nr = LOCAL ? 1u : (uint32_t)c.nranks;
  const uint32_t stride = gridDim.x * blockDim.x * U;
  for (uint32_t base = blockIdx.x * blockDim.x * U + threadIdx.x; base < total; base += stride) {
    uint4 d[U][R];
    char* dst[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const uint32_t g = base + (uint32_t)u * blockDim.x;
      dst[u] = nullptr;
      if (g < total) {
        const CpPlace p = cp_place(a, g);
        dst[u] = a.t[p.i].shard + 16ull * p.shard_v;
        const unsigned long long off = a.t[p.i].full + 16ull * p.full_v;
        if (LOCAL) {
          d[u][0] = ld_vec(reinterpret_cast<const char*>(off));
        } else {
#pragma unroll
          for (int j = 0; j < R; j++) if ((uint32_t)j < nr) d[u][j] = ld_vec(c.peer[j] + off);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (!dst[u]) continue;
      if (LOCAL) {
        st_vec(dst[u], d[u][0]);
      } else {
        float acc[E] = {};
#pragma unroll
        for (int j = 0; j < R; j++) if ((uint32_t)j < nr) unpack_add<T>(acc, d[u][j]);     // rank order: the same sum on every rank
        uint32_t w[Pack<T, E>::W];
        Pack<T, E>::run(acc, w);
        st_words<Pack<T, E>::W>(dst[u], w);
      }
    }
  }
  if (!LOCAL) {
    if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;          // nobody reads my full any more; my shard is stored
    if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
  }
}

// Once per device, before the first kernel of this family launches: load all six (see ulysses_preload: with lazy module loading and
// virtual ranks, a first launch queued behind a peer-waiting barrier kernel would never load).
static void context_preload(const b200collComm* c) {
  static std::atomic<unsigned long long> done{0};
  static std::mutex mu;
  const unsigned long long bit = 1ull << (c->device & 63);
  if (done.load(std::memory_order_acquire) & bit) return;
  const std::lock_guard<std::mutex> lk(mu);
  if (done.load(std::memory_order_acquire) & bit) return;
  cudaFuncAttributes fa;
  cudaFuncGetAttributes(&fa, k_cp_gather<false>);
  cudaFuncGetAttributes(&fa, k_cp_gather<true>);
  cudaFuncGetAttributes(&fa, k_cp_rs<__nv_bfloat16, false>);
  cudaFuncGetAttributes(&fa, k_cp_rs<__half, false>);
  cudaFuncGetAttributes(&fa, k_cp_rs<float, false>);
  cudaFuncGetAttributes(&fa, k_cp_rs<float, true>);
  done.fetch_or(bit, std::memory_order_acq_rel);
}

static b200collResult_t context(b200collComm* c, bool gather, const b200collContextTensor* ts, int ntensors, size_t batch, size_t seq_local,
                                int chunks, b200collDataType_t dtype, b200collStream_t stream) {
  const std::string who = gather ? "all-gather context: " : "reduce-scatter context: ";
  auto refuse = [&](const std::string& msg) { set_last_error(who + msg); return b200collInvalidArgument; };
  if (!c) return refuse("null communicator");
  if (ntensors < 1 || ntensors > kCpMaxTensors) return refuse("ntensors must be 1, 2 or 3");
  if (!ts) return refuse("null tensor array");
  const bool wide = dtype == b200collBfloat16 || dtype == b200collFloat16 || dtype == b200collFloat32;
  if (gather && !wide && !is_fp8(dtype)) return refuse("dtype must be bf16, fp16, fp32, e4m3 or e5m2");
  if (!gather && !wide) return refuse("dtype must be bf16, fp16 or fp32");
  if (chunks != 1 && chunks != 2) return refuse("chunks must be 1 or 2");
  if (chunks == 2 && seq_local % 2) return refuse("chunks = 2 needs an even seq_local");
  const size_t es = b200collTypeSize(dtype);
  const size_t N = (size_t)c->nranks, rows = batch * seq_local;
  if (seq_local >= ((size_t)1 << 31) || batch >= ((size_t)1 << 31) || rows >= ((size_t)1 << 31)) return refuse("batch * seq_local must be below 2^31");
  CpArgs a = {};
  Span src[kCpMaxTensors], dst[kCpMaxTensors];
  size_t total = 0;
  for (int i = 0; i < ntensors; i++) {
    const b200collContextTensor& t = ts[i];
    const std::string ti = "tensor " + std::to_string(i) + ": ";
    if (t.width == 0 || t.width >= ((size_t)1 << 31) || (t.width * es) % 16 != 0) return refuse(ti + "width * sizeof(dtype) must be a positive multiple of 16 bytes");
    if (t.row_stride < t.width) return refuse(ti + "row_stride must be at least width");
    if (t.row_stride > kCpI31 * 16) return refuse(ti + "more than 2^31 - 1 16-byte vectors per rank");   // keeps the extent below in 64 bits
    if ((t.row_stride * es) % 16 != 0) return refuse(ti + "row_stride * sizeof(dtype) must be a multiple of 16 bytes");
    if (rows > 0 && (!t.shard || !t.full)) return refuse(ti + "null pointer");
    if (!aligned(t.shard, 16) || !aligned(t.full, 16)) return refuse(ti + "shard and full must be 16-byte aligned");
    const size_t wv = t.width * es / 16;
    const size_t shard_vecs = rows == 0 ? 0 : (rows - 1) * (t.row_stride * es / 16) + wv;   // the shard's extent
    const size_t full_vecs = N * rows * wv;                                                  // B * S * W
    const size_t moved = rows * wv;
    if (shard_vecs > kCpI31 || full_vecs > kCpI31 || moved > kCpI31 - total) return refuse(ti + "more than 2^31 - 1 16-byte vectors per rank");
    const Span shard_span = {(uintptr_t)t.shard, rows, t.row_stride * es, t.width * es};
    const Span full_span = {(uintptr_t)t.full, 1, full_vecs * 16, full_vecs * 16};
    src[i] = gather ? shard_span : full_span;
    dst[i] = gather ? full_span : shard_span;
    CpTensor& u = a.t[i];
    u.shard = static_cast<char*>(t.shard);
    u.row_stride = t.row_stride * es / 16;
    u.width = fast_div((uint32_t)wv);
    a.prefix[i] = (uint32_t)total;
    total += moved;
  }
  for (int i = ntensors; i <= kCpMaxTensors; i++) a.prefix[i] = (uint32_t)total;
  a.ntensors = (uint32_t)ntensors;
  for (int i = 0; i < ntensors; i++)
    for (int j = 0; j < ntensors; j++) {
      if (spans_overlap(dst[i], src[j])) return refuse("output " + std::to_string(i) + " overlaps source " + std::to_string(j));
      if (j > i && spans_overlap(dst[i], dst[j])) return refuse("outputs " + std::to_string(i) + " and " + std::to_string(j) + " overlap");
    }
  if (comm_poisoned(c)) return b200collRemoteError;
  const bool local = c->nranks == 1;
  const Span* full = gather ? dst : src;
  if (!local && rows > 0) {
    for (int i = 0; i < ntensors; i++) {
      const b200collResult_t rc = in_arena(c, who, "every full", {{reinterpret_cast<const void*>(full[i].p), full[i].extent()}});
      if (rc != b200collSuccess) return rc;
    }
  }
  // B200COLL_CHECK=1: (direction, ntensors, dtype, C, B, S_l) in one exchange, then each tensor's width, full offset and row stride
  const b200collOp_t stats_op = gather ? b200collOpAllGather : b200collOpReduceScatter;
  const b200collAlgo_t algo = local ? b200collAlgoCopy : b200collAlgoTwoShot;
  if (!local) {
    const size_t fmt = ((size_t)dtype << 8) | ((size_t)ntensors << 2) | ((size_t)(chunks - 1) << 1) | (gather ? 1 : 0);
    b200collResult_t rc = cross_check(c, stats_op, algo, fmt, batch, seq_local);
    for (int i = 0; i < ntensors && rc == b200collSuccess; i++)
      rc = cross_check(c, stats_op, algo, ts[i].width, rows > 0 ? arena_off(c, reinterpret_cast<const void*>(full[i].p)) : 0, ts[i].row_stride);
    if (rc != b200collSuccess) return rc;
  }
  if (rows == 0) return b200collSuccess;
  for (int i = 0; i < ntensors; i++)
    a.t[i].full = local ? (unsigned long long)full[i].p : (unsigned long long)arena_off(c, reinterpret_cast<const void*>(full[i].p));
  const size_t chunk = seq_local / (size_t)chunks, me = (size_t)c->rank;
  a.seq_local = fast_div((uint32_t)seq_local);
  a.chunk = (uint32_t)chunk;
  a.tok0 = (uint32_t)(me * chunk);
  a.tok1 = (uint32_t)((2 * N - 2 - me) * chunk);          // G(me, 1) * c - c
  a.seq = (uint32_t)(N * seq_local);
  const DeviceScope on_device(c->device);
  context_preload(c);
  account(c, stats_op, total * 16, algo);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint32_t op = (uint32_t)stats_op;
  if (gather) {
    const Grid g = pick_grid(c, kShapeP2p, total, kCpUnroll);
    if (local) launch_k(k_cp_gather<true>, g.blocks, g.threads, st, c->dev, a, op);
    else launch_k(k_cp_gather<false>, g.blocks, g.threads, st, c->dev, a, op);
  } else if (local) {
    const Grid g = pick_grid(c, kShapeP2p, total, kCpUnroll);
    launch_k(k_cp_rs<float, true>, g.blocks, g.threads, st, c->dev, a, op);     // a bit copy: the element type does not matter
  } else {
    const Grid g = pick_grid(c, kShapeP2p, total, 1);
    if (dtype == b200collBfloat16) launch_k(k_cp_rs<__nv_bfloat16, false>, g.blocks, g.threads, st, c->dev, a, op);
    else if (dtype == b200collFloat16) launch_k(k_cp_rs<__half, false>, g.blocks, g.threads, st, c->dev, a, op);
    else launch_k(k_cp_rs<float, false>, g.blocks, g.threads, st, c->dev, a, op);
  }
  LAUNCH_CHECK(c);
  return b200collSuccess;
}

}  // namespace b200coll

using namespace b200coll;

extern "C" {

b200collResult_t b200collAllGatherContext(const b200collContextTensor* tensors, int ntensors, size_t batch, size_t seq_local, int chunks,
                                          b200collDataType_t dtype, b200collComm_t comm, b200collStream_t stream) {
  return context(comm, true, tensors, ntensors, batch, seq_local, chunks, dtype, stream);
}

b200collResult_t b200collReduceScatterContext(const b200collContextTensor* tensors, int ntensors, size_t batch, size_t seq_local, int chunks,
                                              b200collDataType_t dtype, b200collComm_t comm, b200collStream_t stream) {
  return context(comm, false, tensors, ntensors, batch, seq_local, chunks, dtype, stream);
}

}  // extern "C"
