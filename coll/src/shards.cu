// libb200coll FSDP / ZeRO-3 layout collectives: a unit's parameters all-gathered from their dim-0 shards before forward
// (b200collAllGatherShards), and its gradients reduce-scattered back to the shards after backward (b200collReduceScatterShards), one
// kernel per call for up to 64 tensors:
//
//   k_shard_gather<TS, TF, LOCAL>   relaxed barrier, read this rank's rows of every shard, cast them from TS to TF in registers, push
//                                   them into their place in every rank's full, releasing barrier. LOCAL: one rank, a copy with no
//                                   barrier. TS == TF is a bit copy, and one instantiation (float, float) serves every such dtype.
//   k_shard_rs<TF, TS, LOCAL>       relaxed barrier, pull this rank's rows from every rank's full, sum in fp32 in rank order, scale, add
//                                   the old shard if accumulating, round once to TS, store into the shard, releasing barrier. LOCAL: one
//                                   rank, the same arithmetic with no barrier. One rank with TF == TS, scale 1 and no accumulation is a
//                                   bit copy, run by k_shard_gather<float, float, true> from full to shard.
//
// Geometry (the header states it as formulas). Tensor i has d_i rows of W_i elements and p_i rows per rank; rank r owns rows
// [r p_i, r p_i + n_r), n_r = clamp(d_i - r p_i, 0, p_i). Both sides of those rows are dense, so rank r's part of tensor i is one
// contiguous run of n_r W_i elements in the shard (from its start) and in the full (from element r p_i W_i). The host checks that
// p_i W_i and d_i W_i are whole 16-byte vectors in both dtypes, so the run is whole vectors too, and the kernels count in vectors of the
// full's dtype: vector v is 16 bytes of the full and 16 sizeof(TS) / sizeof(TF) bytes of the shard (16, or 32 for fp32 shards of a
// bf16 / fp16 full, or for fp32 shards of a bf16 / fp16 gradient). Rows themselves need not be whole vectors (a 1-D norm weight).
//
// Work. The (tensor, vector) space of this rank's rows is flattened with a prefix over the tensors, and a vector finds its tensor by a
// binary search over the prefix, so a block of 9 (or 64) tensors of very different sizes spreads over every CTA. The gather keeps U
// vectors of loads in flight per thread and stores each cast vector to every rank, staggered from rank me + 1; the reduce-scatter issues
// all N loads of a vector before it sums them (the order of the sum is fixed, not the order of the loads). Indices are 32-bit (the host
// caps every vector count at 2^31 - 1).
//
// Ordering. The argument of k_cp_gather / k_cp_rs. The entry barrier is relaxed: a rank arrives only once its stream has reached this
// call, so a peer's full written by an earlier kernel on the peer's stream (the backward that produced the gradient) is complete before
// anyone pulls it, and a full still read by an earlier kernel (the last forward through this unit) is not pushed into. The closing
// barrier is releasing: when a rank leaves it, every push into its full is visible, and no peer reads its full any more. Shards are
// touched by their own rank only. Both barriers pair CTA b with CTA b, so every rank must launch the same grid; n_r differs between
// ranks, so the grid is sized from sum p_i W_i, which is the same on every rank, and CTAs with no rows here take part in both barriers.
#include <stdint.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <string>
#include <type_traits>

#include "comm.h"
#include "index.cuh"
#include "launch.cuh"

namespace b200coll {

constexpr int kShThreads = 512;
constexpr int kShUnroll = 4;
constexpr int kShMaxTensors = 64;
constexpr size_t kShI31 = ((size_t)1 << 31) - 1;

struct ShTensor {
  char* shard;                     // this rank's rows
  unsigned long long full;         // row r p_i of the full tensor: its arena offset (every rank's is the same), or with LOCAL its address
};

struct ShArgs {
  ShTensor t[kShMaxTensors];
  uint32_t prefix[kShMaxTensors + 1];   // vectors of this rank's rows before tensor i
  uint32_t ntensors;
  float scale;                          // reduce-scatter: t = sum * scale
  uint32_t accumulate;                  // reduce-scatter: t = (float)shard + t
};
// The descriptors travel in the kernel parameters: keep the whole parameter block within the classic 4 KB limit.
static_assert(sizeof(ShArgs) + sizeof(CommDev) + sizeof(uint32_t) <= 4096, "kernel parameters above 4 KB");

// The tensor flattened vector g (< prefix[ntensors]) belongs to: the last i < ntensors with prefix[i] <= g (tensors with no rows here
// are skipped, as their prefix equals the next one's). A binary search of six fixed steps over the nondecreasing prefix.
__device__ __forceinline__ uint32_t sh_tensor(const ShArgs& a, uint32_t g) {
  uint32_t i = 0;
#pragma unroll
  for (uint32_t step = kShMaxTensors / 2; step >= 1; step >>= 1)
    if (i + step < a.ntensors && a.prefix[i + step] <= g) i += step;
  return i;
}

// One full vector from its KS shard vectors: the bit pattern (TS == TF), or 8 fp32 values rounded to nearest even (bf16 / fp16).
template <typename TS, typename TF> __device__ __forceinline__ uint4 sh_cast(const uint4* raw) {
  if constexpr (std::is_same<TS, TF>::value) {
    return raw[0];
  } else {
    static_assert(std::is_same<TS, float>::value, "the gather casts fp32 shards only");
    const float f[8] = {__uint_as_float(raw[0].x), __uint_as_float(raw[0].y), __uint_as_float(raw[0].z), __uint_as_float(raw[0].w),
                        __uint_as_float(raw[1].x), __uint_as_float(raw[1].y), __uint_as_float(raw[1].z), __uint_as_float(raw[1].w)};
    uint32_t w[4];
    Pack<TF, 8>::run(f, w);
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
}

// E elements of TS held in 16-byte words, widened to fp32 exactly (-0 stays -0).
template <typename TS, int E> __device__ __forceinline__ void sh_widen(const uint4* raw, float* x) {
  constexpr int KS = E * (int)sizeof(TS) / 16;
#pragma unroll
  for (int k = 0; k < KS; k++) {
    const uint32_t w[4] = {raw[k].x, raw[k].y, raw[k].z, raw[k].w};
#pragma unroll
    for (int i = 0; i < 4; i++) {
      if constexpr (std::is_same<TS, float>::value) {
        x[4 * k + i] = __uint_as_float(w[i]);
      } else if constexpr (std::is_same<TS, __nv_bfloat16>::value) {
        x[8 * k + 2 * i] = __uint_as_float(w[i] << 16); x[8 * k + 2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
      } else {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
        x[8 * k + 2 * i] = f.x; x[8 * k + 2 * i + 1] = f.y;
      }
    }
  }
}

template <typename TS, typename TF, bool LOCAL>
__global__ void __launch_bounds__(kShThreads) k_shard_gather(COMM_PARAM, const __grid_constant__ ShArgs a, uint32_t op) {
  pdl_prologue();
  constexpr int U = kShUnroll;
  constexpr int KS = sizeof(TS) / sizeof(TF);      // 16-byte shard loads per full vector
  uint32_t s = 0;
  if (!LOCAL) {
    s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;        // every rank is done with the previous contents of its full
  }
  const uint32_t total = a.prefix[a.ntensors];
  const uint32_t me = LOCAL ? 0u : (uint32_t)c.rank, nr = LOCAL ? 1u : (uint32_t)c.nranks;
  const uint32_t stride = gridDim.x * blockDim.x * U;
  for (uint32_t base = blockIdx.x * blockDim.x * U + threadIdx.x; base < total; base += stride) {
    uint4 raw[U][KS];
    unsigned long long off[U];    // the destination: its address (LOCAL) or its arena offset on every rank
    bool act[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const uint32_t g = base + (uint32_t)u * blockDim.x;
      act[u] = g < total; off[u] = 0;
      if (act[u]) {
        const uint32_t i = sh_tensor(a, g), l = g - a.prefix[i];
        off[u] = a.t[i].full + 16ull * l;
#pragma unroll
        for (int k = 0; k < KS; k++) raw[u][k] = ld_vec(a.t[i].shard + 16ull * (KS * (unsigned long long)l + k));
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (!act[u]) continue;
      const uint4 d = sh_cast<TS, TF>(raw[u]);                   // on the owning rank: the narrow type is what crosses NVLink
      if (LOCAL) {
        st_vec(reinterpret_cast<char*>(off[u]), d);
      } else {
#pragma unroll 1
        for (uint32_t k = 1; k <= nr; k++) {
          uint32_t p = me + k; if (p >= nr) p -= nr;
          st_vec(c.peer[p] + off[u], d);
        }
      }
    }
  }
  if (!LOCAL) {
    if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;          // publishes the pushes; nobody reads my shards any more
    if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
  }
}

template <typename TF, typename TS, bool LOCAL>
__global__ void __launch_bounds__(kShThreads) k_shard_rs(COMM_PARAM, const __grid_constant__ ShArgs a, uint32_t op) {
  pdl_prologue();
  constexpr int E = Epv<TF>::value;                 // elements per full vector
  constexpr int KS = sizeof(TS) / sizeof(TF);       // 16-byte shard vectors per full vector
  constexpr int U = LOCAL ? kShUnroll / KS : 1;     // the peer form has N loads in flight per vector already; a widening one 2 each
  constexpr int R = LOCAL ? 1 : kMaxRanks;
  uint32_t s = 0;
  if (!LOCAL) {
    s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;        // every rank's full is written
  }
  const uint32_t total = a.prefix[a.ntensors];
  const uint32_t nr = LOCAL ? 1u : (uint32_t)c.nranks;
  const float scale = a.scale;
  const bool accumulate = a.accumulate != 0;
  const uint32_t stride = gridDim.x * blockDim.x * U;
  for (uint32_t base = blockIdx.x * blockDim.x * U + threadIdx.x; base < total; base += stride) {
    uint4 d[U][R];
    uint4 old[U][KS];
    char* dst[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const uint32_t g = base + (uint32_t)u * blockDim.x;
      dst[u] = nullptr;
      if (g < total) {
        const uint32_t i = sh_tensor(a, g), l = g - a.prefix[i];
        dst[u] = a.t[i].shard + 16ull * KS * l;
        const unsigned long long off = a.t[i].full + 16ull * l;
        if (LOCAL) {
          d[u][0] = ld_vec(reinterpret_cast<const char*>(off));
        } else {
#pragma unroll
          for (int j = 0; j < R; j++) if ((uint32_t)j < nr) d[u][j] = ld_vec(c.peer[j] + off);
        }
        if (accumulate) {
#pragma unroll
          for (int k = 0; k < KS; k++) old[u][k] = ld_vec(dst[u] + 16 * k);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (!dst[u]) continue;
      float acc[E] = {};                                          // +0
#pragma unroll
      for (int j = 0; j < R; j++) if ((uint32_t)j < nr) unpack_add<TF>(acc, d[u][j]);     // rank order: the same sum on every rank
#pragma unroll
      for (int e = 0; e < E; e++) acc[e] = __fmul_rn(acc[e], scale);
      if (accumulate) {
        float o[E];
        sh_widen<TS, E>(old[u], o);
#pragma unroll
        for (int e = 0; e < E; e++) acc[e] = __fadd_rn(o[e], acc[e]);
      }
      uint32_t w[Pack<TS, E>::W];
      Pack<TS, E>::run(acc, w);
      st_words<Pack<TS, E>::W>(dst[u], w);
    }
  }
  if (!LOCAL) {
    if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;          // nobody reads my full any more; my shards are stored
    if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
  }
}

// Once per device, before the first kernel of this family launches: load all sixteen (see ulysses_preload: with lazy module loading and
// virtual ranks, a first launch queued behind a peer-waiting barrier kernel would never load).
static void shards_preload(const b200collComm* c) {
  static std::atomic<unsigned long long> done{0};
  static std::mutex mu;
  const unsigned long long bit = 1ull << (c->device & 63);
  if (done.load(std::memory_order_acquire) & bit) return;
  const std::lock_guard<std::mutex> lk(mu);
  if (done.load(std::memory_order_acquire) & bit) return;
  cudaFuncAttributes fa;
  cudaFuncGetAttributes(&fa, k_shard_gather<float, float, false>);
  cudaFuncGetAttributes(&fa, k_shard_gather<float, float, true>);
  cudaFuncGetAttributes(&fa, k_shard_gather<float, __nv_bfloat16, false>);
  cudaFuncGetAttributes(&fa, k_shard_gather<float, __nv_bfloat16, true>);
  cudaFuncGetAttributes(&fa, k_shard_gather<float, __half, false>);
  cudaFuncGetAttributes(&fa, k_shard_gather<float, __half, true>);
  cudaFuncGetAttributes(&fa, k_shard_rs<__nv_bfloat16, __nv_bfloat16, false>);
  cudaFuncGetAttributes(&fa, k_shard_rs<__nv_bfloat16, __nv_bfloat16, true>);
  cudaFuncGetAttributes(&fa, k_shard_rs<__half, __half, false>);
  cudaFuncGetAttributes(&fa, k_shard_rs<__half, __half, true>);
  cudaFuncGetAttributes(&fa, k_shard_rs<float, float, false>);
  cudaFuncGetAttributes(&fa, k_shard_rs<float, float, true>);
  cudaFuncGetAttributes(&fa, k_shard_rs<__nv_bfloat16, float, false>);
  cudaFuncGetAttributes(&fa, k_shard_rs<__nv_bfloat16, float, true>);
  cudaFuncGetAttributes(&fa, k_shard_rs<__half, float, false>);
  cudaFuncGetAttributes(&fa, k_shard_rs<__half, float, true>);
  done.fetch_or(bit, std::memory_order_acq_rel);
}

template <typename TF, typename TS>
static void launch_rs(bool local, const Grid& g, cudaStream_t st, b200collComm* c, const ShArgs& a, uint32_t op) {
  if (local) launch_k(k_shard_rs<TF, TS, true>, g.blocks, g.threads, st, c->dev, a, op);
  else launch_k(k_shard_rs<TF, TS, false>, g.blocks, g.threads, st, c->dev, a, op);
}

static bool wide(b200collDataType_t t) { return t == b200collBfloat16 || t == b200collFloat16 || t == b200collFloat32; }

// gather: src_dt is the shards' dtype, dst_dt the fulls'; reduce-scatter: src_dt is the fulls', dst_dt the shards'.
static b200collResult_t shards(b200collComm* c, bool gather, const b200collShardTensor* ts, int ntensors, b200collDataType_t src_dt,
                               b200collDataType_t dst_dt, float scale, int accumulate, b200collStream_t stream) {
  const std::string who = gather ? "all-gather shards: " : "reduce-scatter shards: ";
  auto refuse = [&](const std::string& msg) { set_last_error(who + msg); return b200collInvalidArgument; };
  if (!c) return refuse("null communicator");
  if (ntensors < 1 || ntensors > kShMaxTensors) return refuse("ntensors must be 1 to 64");
  if (!ts) return refuse("null tensor array");
  const b200collDataType_t sdt = gather ? src_dt : dst_dt, fdt = gather ? dst_dt : src_dt;
  if (gather) {
    const bool same = src_dt == dst_dt && (wide(src_dt) || is_fp8(src_dt));
    const bool cast = src_dt == b200collFloat32 && (dst_dt == b200collBfloat16 || dst_dt == b200collFloat16);
    if (!same && !cast) return refuse("dtype pair must be one dtype in and out (bf16, fp16, fp32, e4m3 or e5m2), or fp32 -> bf16 or fp16");
  } else {
    const bool same = src_dt == dst_dt && wide(src_dt);
    const bool widen = dst_dt == b200collFloat32 && (src_dt == b200collBfloat16 || src_dt == b200collFloat16);
    if (!same && !widen) return refuse("dtype pair must be bf16 -> bf16, fp16 -> fp16, fp32 -> fp32, bf16 -> fp32 or fp16 -> fp32");
  }
  const size_t ess = b200collTypeSize(sdt), esf = b200collTypeSize(fdt), esmax = std::max(ess, esf);
  const size_t N = (size_t)c->nranks, me = (size_t)c->rank;
  ShArgs a = {};
  Span src[kShMaxTensors], dst[kShMaxTensors];
  size_t total = 0, grid_vecs = 0;
  for (int i = 0; i < ntensors; i++) {
    const b200collShardTensor& t = ts[i];
    const std::string ti = "tensor " + std::to_string(i) + ": ";
    const size_t d = t.rows, W = t.width, p = t.shard_rows;
    if (d == 0 || W == 0 || p == 0) return refuse(ti + "rows, width and shard_rows must be positive");
    const size_t lim = kShI31 * 16;                                              // elements; keeps every product below in 64 bits
    if (W > lim || d > lim / W || p > lim / W) return refuse(ti + "more than 2^31 - 1 16-byte vectors in one side");
    if (p * N < d) return refuse(ti + "nranks * shard_rows must be at least rows");
    if ((p * W * ess) % 16 || (p * W * esf) % 16 || (d * W * ess) % 16 || (d * W * esf) % 16)
      return refuse(ti + "shard_rows * width and rows * width must be multiples of 16 bytes in both dtypes");
    if (d * W * esmax / 16 > kShI31 || p * W * esmax / 16 > kShI31) return refuse(ti + "more than 2^31 - 1 16-byte vectors in one side");
    const size_t first = std::min(d, me * p), n_r = std::min(d - first, p);     // this rank's rows [first, first + n_r)
    if (!t.full || (n_r > 0 && !t.shard)) return refuse(ti + "null pointer");
    if (!aligned(t.full, 16) || !aligned(t.shard, 16)) return refuse(ti + "shard and full must be 16-byte aligned");
    const size_t vecs = n_r * W * esf / 16, gv = p * W * esf / 16;
    if (gv > kShI31 - grid_vecs) return refuse("more than 2^31 - 1 16-byte vectors in the call");
    grid_vecs += gv;
    const Span shard_span = {(uintptr_t)t.shard, 1, n_r * W * ess, n_r * W * ess};
    const Span full_span = {(uintptr_t)t.full, 1, d * W * esf, d * W * esf};
    src[i] = gather ? shard_span : full_span;
    dst[i] = gather ? full_span : shard_span;
    a.t[i].shard = static_cast<char*>(t.shard);
    a.prefix[i] = (uint32_t)total;
    total += vecs;
  }
  for (int i = ntensors; i <= kShMaxTensors; i++) a.prefix[i] = (uint32_t)total;
  a.ntensors = (uint32_t)ntensors;
  a.scale = scale;
  a.accumulate = accumulate ? 1u : 0u;
  for (int i = 0; i < ntensors; i++)
    for (int j = 0; j < ntensors; j++) {
      if (spans_overlap(dst[i], src[j])) return refuse("output " + std::to_string(i) + " overlaps source " + std::to_string(j));
      if (j > i && spans_overlap(dst[i], dst[j])) return refuse("outputs " + std::to_string(i) + " and " + std::to_string(j) + " overlap");
    }
  if (comm_poisoned(c)) return b200collRemoteError;
  const bool local = c->nranks == 1;
  const Span* full = gather ? dst : src;
  if (!local) {
    for (int i = 0; i < ntensors; i++) {
      const b200collResult_t rc = in_arena(c, who, "every full", {{reinterpret_cast<const void*>(full[i].p), full[i].extent()}});
      if (rc != b200collSuccess) return rc;
    }
  }
  // B200COLL_CHECK=1: (direction, ntensors, both dtypes, accumulate) and the bits of scale in one exchange, then each tensor's d, W, p
  // and full offset
  const b200collOp_t stats_op = gather ? b200collOpAllGather : b200collOpReduceScatter;
  const b200collAlgo_t algo = local ? b200collAlgoCopy : b200collAlgoTwoShot;
  if (!local) {
    uint32_t sbits;
    memcpy(&sbits, &scale, sizeof sbits);
    const size_t fmt = ((size_t)sdt << 24) | ((size_t)fdt << 16) | ((size_t)ntensors << 2) | ((size_t)(accumulate ? 1 : 0) << 1) | (gather ? 1 : 0);
    b200collResult_t rc = cross_check(c, stats_op, algo, fmt, sbits, 0);
    for (int i = 0; i < ntensors && rc == b200collSuccess; i++) {
      rc = cross_check(c, stats_op, algo, ts[i].rows, ts[i].width, ts[i].shard_rows);
      if (rc == b200collSuccess) rc = cross_check(c, stats_op, algo, arena_off(c, ts[i].full), 0, 0);
    }
    if (rc != b200collSuccess) return rc;
  }
  const bool bit_copy = !gather && local && sdt == fdt && scale == 1.0f && !accumulate;
  for (int i = 0; i < ntensors; i++) {
    const size_t row0 = std::min(ts[i].rows, me * ts[i].shard_rows) * ts[i].width * esf;      // bytes before this rank's rows
    if (bit_copy) {                                   // the local gather copy, run from full to shard
      a.t[i].shard = static_cast<char*>(ts[i].full);
      a.t[i].full = (unsigned long long)ts[i].shard;
    } else if (local) {
      a.t[i].full = (unsigned long long)(full[i].p + row0);
    } else {
      a.t[i].full = (unsigned long long)(arena_off(c, ts[i].full) + row0);
    }
  }
  const DeviceScope on_device(c->device);
  shards_preload(c);
  account(c, stats_op, total * 16, algo);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint32_t op = (uint32_t)stats_op;
  // Sized from sum p_i W_i, the same on every rank, so that the barriers pair every CTA; one rank sizes it from its own rows.
  const size_t sized = local ? total : grid_vecs;
  if (gather || bit_copy) {
    const Grid g = pick_grid(c, kShapeP2p, sized, kShUnroll);
    if (sdt == fdt || bit_copy) {
      if (local) launch_k(k_shard_gather<float, float, true>, g.blocks, g.threads, st, c->dev, a, op);
      else launch_k(k_shard_gather<float, float, false>, g.blocks, g.threads, st, c->dev, a, op);
    } else if (fdt == b200collBfloat16) {
      if (local) launch_k(k_shard_gather<float, __nv_bfloat16, true>, g.blocks, g.threads, st, c->dev, a, op);
      else launch_k(k_shard_gather<float, __nv_bfloat16, false>, g.blocks, g.threads, st, c->dev, a, op);
    } else {
      if (local) launch_k(k_shard_gather<float, __half, true>, g.blocks, g.threads, st, c->dev, a, op);
      else launch_k(k_shard_gather<float, __half, false>, g.blocks, g.threads, st, c->dev, a, op);
    }
  } else {
    const Grid g = pick_grid(c, kShapeP2p, sized, local ? kShUnroll * (int)esf / (int)ess : 1);
    if (fdt == b200collBfloat16 && sdt == b200collBfloat16) launch_rs<__nv_bfloat16, __nv_bfloat16>(local, g, st, c, a, op);
    else if (fdt == b200collFloat16 && sdt == b200collFloat16) launch_rs<__half, __half>(local, g, st, c, a, op);
    else if (fdt == b200collFloat32) launch_rs<float, float>(local, g, st, c, a, op);
    else if (fdt == b200collBfloat16) launch_rs<__nv_bfloat16, float>(local, g, st, c, a, op);
    else launch_rs<__half, float>(local, g, st, c, a, op);
  }
  LAUNCH_CHECK(c);
  return b200collSuccess;
}

}  // namespace b200coll

using namespace b200coll;

extern "C" {

b200collResult_t b200collAllGatherShards(const b200collShardTensor* tensors, int ntensors, b200collDataType_t shard_dtype,
                                         b200collDataType_t full_dtype, b200collComm_t comm, b200collStream_t stream) {
  return shards(comm, true, tensors, ntensors, shard_dtype, full_dtype, 1.0f, 0, stream);
}

b200collResult_t b200collReduceScatterShards(const b200collShardTensor* tensors, int ntensors, b200collDataType_t full_dtype,
                                             b200collDataType_t shard_dtype, float scale, int accumulate, b200collComm_t comm,
                                             b200collStream_t stream) {
  return shards(comm, false, tensors, ntensors, full_dtype, shard_dtype, scale, accumulate, stream);
}

}  // extern "C"
