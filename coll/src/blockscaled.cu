// libb200coll block-scaled FP8 collectives: e4m3 / e5m2 matrices with one fp32 scale per block_rows x block_cols block (1x128 activation
// and gradient blocks, 128x128 weight blocks), dequantised in registers and delivered as bf16, fp16 or fp32. FP8 crosses NVLink, the
// wider type is only ever written locally (or, in the two-shot all-reduce, pushed once as the finished result):
//
//   k_bsq_ag_pull<InT, OutT>              all-gather: barrier, pull every rank's FP8 shard and scales, dequantise, store locally, barrier
//   k_bsq_pull_reduce<InT, OutT, false>   reduce-scatter (my row slice) / one-shot all-reduce (whole matrix): pull from every rank in
//                                         rank order, dequantise with that rank's scales, sum in fp32, scale, round once, store locally
//   k_bsq_pull_reduce<InT, OutT, true>    two-shot all-reduce: the same over my vector slice, the result pushed into every rank's recv
//   k_bsq_copy<InT, OutT>                 one rank: local dequantising copy, no barrier
//
// Scales: a 16-byte FP8 vector lies in exactly one block (row_len and block_cols are multiples of 16), so a vector needs one scale per
// rank. Lanes of a warp hold consecutive vectors and usually share scales (8 lanes per 1x128 block, whole warps per 128x128 block):
// __match_any_sync groups the lanes by scale index, the lowest lane of each group loads the scale and __shfl_sync hands it to the rest,
// so each distinct scale is read once per warp and rank. The vector -> (row, column) -> block arithmetic is 32-bit multiply-high
// division by host-computed constants: no integer division in the loops.
#include <limits.h>
#include <stdint.h>

#include "blockscale.cuh"
#include "comm.h"
#include "launch.cuh"

namespace b200coll {

using bf16 = __nv_bfloat16;
using f8 = __nv_fp8_e4m3;
using e5m2 = __nv_fp8_e5m2;

constexpr int kBsqThreads = 512;

// What every kernel needs to find vector v of a rank's send matrix and its scale. Vector indices are 32-bit (the host refuses larger).
struct BsqGeom {
  size_t send_off, scale_off;     // arena offsets of the FP8 matrix and of its scales (the same on every rank)
  uint32_t nvec;                  // 16-element vectors in one rank's matrix
  uint32_t ncb;                   // block columns (scales per block row)
  FastDiv vpr, br, vpb;           // vectors per row, rows per block, vectors per block column
};

__device__ __forceinline__ uint32_t bsq_scale_index(const BsqGeom& g, uint32_t v) {
  const uint32_t row = g.vpr.div(v), cv = v - row * g.vpr.d;
  return g.br.div(row) * g.ncb + g.vpb.div(cv);
}

// Dequantise vectors [0, nvec) of one rank's matrix into dst. Loops run on the warp's first vector so that whole warps stay together
// for the scale exchange.
template <typename InT, typename OutT>
__device__ __forceinline__ void bsq_dequant_range(const BsqGeom& g, const char* src, const char* scales, OutT* dst, float scale) {
  const uint32_t lane = threadIdx.x & 31;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t b = (size_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); b < g.nvec; b += stride) {
    const size_t v = b + lane;
    const bool act = v < g.nvec;
    uint4 q = make_uint4(0, 0, 0, 0);
    if (act) q = ld_vec(src + v * 16);
    const uint32_t idx = act ? bsq_scale_index(g, (uint32_t)v) : 0u;
    const WarpScale ws(idx, act);
    const float s = ws.get(scales, idx);
    if (act) {
      float acc[16] = {};
      bsq_dequant_add<InT>(acc, q, s);
      bsq_store<OutT>(dst + v * 16, acc, scale);
    }
  }
}

template <typename InT, typename OutT>
__global__ void __launch_bounds__(kBsqThreads) k_bsq_copy(const __grid_constant__ BsqGeom g, const char* __restrict__ in, const char* __restrict__ scales,
                                                       OutT* __restrict__ out, float scale) {
  pdl_prologue();
  bsq_dequant_range<InT, OutT>(g, in, scales, out, scale);
}

// out holds nranks shards of nvec*16 elements; shard r is rank r's matrix dequantised with rank r's scales
template <typename InT, typename OutT>
__global__ void __launch_bounds__(kBsqThreads) k_bsq_ag_pull(COMM_PARAM, const __grid_constant__ BsqGeom g, OutT* __restrict__ out, float scale, uint32_t op) {
  pdl_prologue();
  const uint32_t s = load_seq(c, kSeqBarrier);
  if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;          // every rank's shard and scales are written
  for (int j = 0; j < c.nranks; j++) {                          // peers visited starting with myself: spreads the pulls over the links
    int r = c.rank + j; if (r >= c.nranks) r -= c.nranks;
    bsq_dequant_range<InT, OutT>(g, c.peer[r] + g.send_off, c.peer[r] + g.scale_off, out + (size_t)r * g.nvec * 16, scale);
  }
  if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;           // nobody reads my shard any more: I may overwrite it
  if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
}

// Vectors [v0, v1) summed over ranks in rank order: acc = ((0 + v_0) + v_1 + ...), then round_once(acc * scale).
// PUSH=false: stored at out_local[(v - v0) * 16] (reduce-scatter: my slice; one-shot all-reduce: v0 = 0, v1 = nvec).
// PUSH=true: stored at arena offset out_off + v * 16 * sizeof(OutT) of every rank (two-shot all-reduce, my vector slice).
// One 512-thread CTA per SM, like the other P2P reduction kernels (k_pull_reduce, k_ar_twoshot: about 100 registers): with eight pulled
// vectors and 16 accumulators live, squeezing the kernel into the 64 registers of two CTAs per SM made ptxas spill the loop state.
template <typename InT, typename OutT, bool PUSH>
__global__ void __launch_bounds__(kBsqThreads, 1) k_bsq_pull_reduce(COMM_PARAM, const __grid_constant__ BsqGeom g, OutT* __restrict__ out_local, size_t out_off,
                                                              uint32_t v0, uint32_t v1, float scale, uint32_t op) {
  pdl_prologue();
  {
    const uint32_t s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;
  }
  // 32-bit vector indices: the host keeps nvec below 2^31, so b + stride cannot wrap
  const uint32_t lane = threadIdx.x & 31;
  for (uint32_t b = v0 + blockIdx.x * blockDim.x + (threadIdx.x & ~31u); b < v1; b += gridDim.x * blockDim.x) {
    const uint32_t v = b + lane;
    const bool act = v < v1;
    uint4 d[kMaxRanks];
#pragma unroll
    for (int r = 0; r < kMaxRanks; r++) if (r < c.nranks) d[r] = act ? ld_vec(c.peer[r] + g.send_off + (size_t)v * 16) : make_uint4(0, 0, 0, 0);
    const uint32_t idx = act ? bsq_scale_index(g, v) : 0u;
    const WarpScale ws(idx, act);
    float acc[16] = {};
#pragma unroll
    for (int r = 0; r < kMaxRanks; r++) if (r < c.nranks) {
      const float sr = ws.get(c.peer[r] + g.scale_off, idx);
      bsq_dequant_add<InT>(acc, d[r], sr);
    }
    if (act) {
      if (PUSH) {
#pragma unroll
        for (int j = 0; j < kMaxRanks; j++) if (j < c.nranks) {
          int r = c.rank + j; if (r >= c.nranks) r -= c.nranks;
          bsq_store<OutT>(c.peer[r] + out_off + (size_t)v * (16 * sizeof(OutT)), acc, scale);
        }
      } else {
        bsq_store<OutT>(out_local + (size_t)(v - v0) * 16, acc, scale);
      }
    }
  }
  // the sequence number is read again rather than kept live across the loop: only the last block, after the barrier below, bumps it
  const uint32_t s = load_seq(c, kSeqBarrier);
  if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;
  if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
}

// ------------------------------------------------------------------------------------------------ host side
template <typename T> struct Tag { using type = T; };

template <typename F>
static b200collResult_t dispatch_bsq(b200collDataType_t in, b200collDataType_t out, F&& f) {
  auto outs = [&](auto ti) -> b200collResult_t {
    switch (out) {
      case b200collBfloat16: return f(ti, Tag<bf16>{});
      case b200collFloat16: return f(ti, Tag<__half>{});
      case b200collFloat32: return f(ti, Tag<float>{});
      default: set_last_error("block-scaled collectives: out_dtype must be bf16, fp16 or fp32"); return b200collInvalidArgument;
    }
  };
  if (in == b200collFloat8e4m3) return outs(Tag<f8>{});
  if (in == b200collFloat8e5m2) return outs(Tag<e5m2>{});
  set_last_error("block-scaled collectives: in_dtype must be e4m3 or e5m2");
  return b200collInvalidArgument;
}

static bool overlaps(const void* a, size_t na, const void* b, size_t nb) {
  const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
  return x < y + nb && y < x + na;
}

struct BsqCall {
  b200collComm* c;
  size_t count;                   // elements of one rank's send matrix
  size_t out_bytes;               // bytes of my recv
  size_t nscales;
  float scale;                    // ep->scale, times 1/nranks for avg
  BsqGeom g;
};

// Everything the three entry points check before they launch. On success `call` is filled in; count == 0 is left to the caller.
static b200collResult_t bsq_prepare(b200collComm* c, b200collOp_t which, const void* send, void* recv, size_t count, const b200collBlockScale* bs,
                                    const b200collEpilogue* ep, b200collRedOp_t rop, BsqCall* call) {
  if (!c || !send || !recv || !bs || !ep || !bs->scales) { set_last_error("null argument"); return b200collInvalidArgument; }
  if (ep->in_dtype != b200collFloat8e4m3 && ep->in_dtype != b200collFloat8e5m2) { set_last_error("block-scaled collectives: in_dtype must be e4m3 or e5m2"); return b200collInvalidArgument; }
  if (ep->out_dtype != b200collBfloat16 && ep->out_dtype != b200collFloat16 && ep->out_dtype != b200collFloat32) { set_last_error("block-scaled collectives: out_dtype must be bf16, fp16 or fp32"); return b200collInvalidArgument; }
  if (which != b200collOpAllGather && rop != b200collSum && rop != b200collAvg) { set_last_error("block-scaled reductions take sum or avg only"); return b200collInvalidArgument; }
  if (bs->row_len == 0 || bs->row_len % 16 != 0) { set_last_error("block-scaled collectives: row_len must be a positive multiple of 16"); return b200collInvalidArgument; }
  if (bs->block_rows < 1 || bs->block_cols < 16 || bs->block_cols % 16 != 0) { set_last_error("block-scaled collectives: block_rows must be >= 1 and block_cols a positive multiple of 16"); return b200collInvalidArgument; }
  if (count % bs->row_len != 0) { set_last_error("block-scaled collectives: the send count must be a multiple of row_len"); return b200collInvalidArgument; }
  if (count / 16 >= ((size_t)1 << 31)) { set_last_error("block-scaled collectives: fewer than 2^35 elements per rank"); return b200collInvalidArgument; }
  const size_t rows = count / bs->row_len;
  if (which == b200collOpReduceScatter && rows % (size_t)c->nranks != 0) { set_last_error("block-scaled reduce-scatter: the number of rows must be a multiple of nranks"); return b200collInvalidArgument; }
  if (!aligned(send, 16) || !aligned(recv, 16) || !aligned(bs->scales, 4)) { set_last_error("send and recv must be 16-byte aligned, scales 4-byte aligned"); return b200collInvalidArgument; }
  if (c->fault_host && *const_cast<volatile uint32_t*>(&c->fault_host->code) != 0) { set_last_error("communicator is poisoned by an earlier watchdog fault"); return b200collRemoteError; }
  const size_t os = b200collTypeSize(ep->out_dtype);
  const size_t vpr = bs->row_len / 16, vpb = (size_t)bs->block_cols / 16;
  const size_t nbr = (rows + bs->block_rows - 1) / bs->block_rows, ncb = (vpr + vpb - 1) / vpb;
  call->c = c;
  call->count = count;
  call->out_bytes = (which == b200collOpAllGather ? count * c->nranks : which == b200collOpReduceScatter ? count / c->nranks : count) * os;
  call->nscales = nbr * ncb;
  call->scale = ep->scale * (rop == b200collAvg && which != b200collOpAllGather ? 1.0f / (float)c->nranks : 1.0f);
  if (count == 0) return b200collSuccess;
  if (overlaps(send, count, recv, call->out_bytes)) { set_last_error("block-scaled collectives: recv must not overlap send"); return b200collInvalidArgument; }
  // peers read my matrix and scales at MY arena offsets: both must be arena memory (there is no staging path for these ops)
  if (!b200collIsSymmetric(c, send, count) || !b200collIsSymmetric(c, bs->scales, call->nscales * 4)) {
    set_last_error("block-scaled collectives: send and scales must lie in the symmetric arena (b200collMemAlloc), at the same offsets on every rank");
    return b200collInvalidUsage;
  }
  BsqGeom& g = call->g;
  g.send_off = arena_off(c, send); g.scale_off = arena_off(c, bs->scales);
  g.nvec = (uint32_t)(count / 16); g.ncb = (uint32_t)ncb;
  g.vpr = make_fastdiv((uint32_t)vpr); g.br = make_fastdiv((uint32_t)bs->block_rows); g.vpb = make_fastdiv((uint32_t)vpb);
  return b200collSuccess;
}

// nranks == 1: no peers, no barrier; grid as for the fused copy (streaming, 8 CTAs of 256 threads per SM at most)
static b200collResult_t bsq_copy(const BsqCall& k, const void* send, const b200collBlockScale* bs, void* recv, const b200collEpilogue* ep, cudaStream_t st) {
  b200collComm* c = k.c;
  return dispatch_bsq(ep->in_dtype, ep->out_dtype, [&](auto ti, auto to) -> b200collResult_t {
    using InT = typename decltype(ti)::type; using OutT = typename decltype(to)::type;
    const int blocks = (int)std::max<size_t>(1, std::min<size_t>(((size_t)k.g.nvec + 255) / 256, (size_t)std::max(1, c->sm_count) * 8));
    launch_k(k_bsq_copy<InT, OutT>, blocks, 256, st, k.g, static_cast<const char*>(send), reinterpret_cast<const char*>(bs->scales), static_cast<OutT*>(recv), k.scale);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  });
}

static b200collResult_t bsq_reduce(const BsqCall& k, b200collOp_t which, b200collAlgo_t algo, void* recv, const b200collEpilogue* ep, cudaStream_t st) {
  b200collComm* c = k.c;
  const uint32_t n = (uint32_t)c->nranks, me = (uint32_t)c->rank;
  uint32_t v0 = 0, v1 = k.g.nvec;
  if (which == b200collOpReduceScatter || algo == b200collAlgoTwoShot) {
    v0 = (uint32_t)((unsigned long long)k.g.nvec * me / n); v1 = (uint32_t)((unsigned long long)k.g.nvec * (me + 1) / n);
  }
  return dispatch_bsq(ep->in_dtype, ep->out_dtype, [&](auto ti, auto to) -> b200collResult_t {
    using InT = typename decltype(ti)::type; using OutT = typename decltype(to)::type;
    if (algo == b200collAlgoTwoShot) {
      const Grid gr = pick_grid(c, kShapeP2p, k.g.nvec / n + 1, 1);
      launch_k(k_bsq_pull_reduce<InT, OutT, true>, gr.blocks, gr.threads, st, c->dev, k.g, static_cast<OutT*>(nullptr), arena_off(c, recv), v0, v1, k.scale, (uint32_t)which);
    } else {
      const Grid gr = pick_grid(c, kShapeP2p, which == b200collOpReduceScatter ? k.g.nvec / n : k.g.nvec, 1);
      launch_k(k_bsq_pull_reduce<InT, OutT, false>, gr.blocks, gr.threads, st, c->dev, k.g, static_cast<OutT*>(recv), (size_t)0, v0, v1, k.scale, (uint32_t)which);
    }
    LAUNCH_CHECK(c);
    return b200collSuccess;
  });
}

}  // namespace b200coll

using namespace b200coll;

extern "C" {

b200collResult_t b200collAllGatherBlockScaled(const void* send, void* recv, size_t sendcount, const b200collBlockScale* bs, const b200collEpilogue* ep,
                                              b200collComm_t c, b200collStream_t stream) {
  BsqCall k;
  b200collResult_t rc = bsq_prepare(c, b200collOpAllGather, send, recv, sendcount, bs, ep, b200collSum, &k);
  if (rc != b200collSuccess || sendcount == 0) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (c->nranks == 1) { account(c, b200collOpAllGather, sendcount, b200collAlgoCopy); return bsq_copy(k, send, bs, recv, ep, st); }
  rc = cross_check(c, b200collOpAllGather, b200collAlgoOneShot, sendcount, k.g.send_off, k.g.scale_off);
  if (rc != b200collSuccess) return rc;
  account(c, b200collOpAllGather, sendcount, b200collAlgoOneShot);
  return dispatch_bsq(ep->in_dtype, ep->out_dtype, [&](auto ti, auto to) -> b200collResult_t {
    using InT = typename decltype(ti)::type; using OutT = typename decltype(to)::type;
    const Grid gr = pick_grid(c, kShapeP2p, k.g.nvec, 1);
    launch_k(k_bsq_ag_pull<InT, OutT>, gr.blocks, gr.threads, st, c->dev, k.g, static_cast<OutT*>(recv), k.scale, (uint32_t)b200collOpAllGather);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  });
}

b200collResult_t b200collReduceScatterBlockScaled(const void* send, void* recv, size_t recvcount, const b200collBlockScale* bs, const b200collEpilogue* ep,
                                                  b200collRedOp_t op, b200collComm_t c, b200collStream_t stream) {
  if (c && recvcount > SIZE_MAX / B200COLL_MAX_RANKS) { set_last_error("recvcount too large"); return b200collInvalidArgument; }
  BsqCall k;
  b200collResult_t rc = bsq_prepare(c, b200collOpReduceScatter, send, recv, c ? recvcount * c->nranks : 0, bs, ep, op, &k);
  if (rc != b200collSuccess || recvcount == 0) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (c->nranks == 1) { account(c, b200collOpReduceScatter, recvcount, b200collAlgoCopy); return bsq_copy(k, send, bs, recv, ep, st); }
  rc = cross_check(c, b200collOpReduceScatter, b200collAlgoOneShot, recvcount, k.g.send_off, k.g.scale_off);
  if (rc != b200collSuccess) return rc;
  account(c, b200collOpReduceScatter, recvcount, b200collAlgoOneShot);
  return bsq_reduce(k, b200collOpReduceScatter, b200collAlgoOneShot, recv, ep, st);
}

b200collResult_t b200collAllReduceBlockScaled(const void* send, void* recv, size_t count, const b200collBlockScale* bs, const b200collEpilogue* ep,
                                              b200collRedOp_t op, b200collComm_t c, b200collStream_t stream) {
  BsqCall k;
  b200collResult_t rc = bsq_prepare(c, b200collOpAllReduce, send, recv, count, bs, ep, op, &k);
  if (rc != b200collSuccess || count == 0) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (c->nranks == 1) { account(c, b200collOpAllReduce, count, b200collAlgoCopy); return bsq_copy(k, send, bs, recv, ep, st); }
  // the table's pick for an FP8 all-reduce of this many bytes (or the forced algorithm): the Lamport paths and one-shot become the
  // one-shot pull, two-shot and NVLS the two-shot pull + push, which needs recv in the arena (peers write into it)
  const b200collAlgo_t want = c->forced_algo != b200collAlgoAuto ? c->forced_algo : b200collTunerPick(b200collOpAllReduce, count, c->nranks, c->nvls);
  b200collAlgo_t algo = (want == b200collAlgoTwoShot || want == b200collAlgoNvls) ? b200collAlgoTwoShot : b200collAlgoOneShot;
  if (algo == b200collAlgoTwoShot && !b200collIsSymmetric(c, recv, k.out_bytes)) algo = b200collAlgoOneShot;
  rc = cross_check(c, b200collOpAllReduce, algo, count, k.g.send_off, algo == b200collAlgoTwoShot ? arena_off(c, recv) : k.g.scale_off);
  if (rc != b200collSuccess) return rc;
  account(c, b200collOpAllReduce, count, algo);
  return bsq_reduce(k, b200collOpAllReduce, algo, recv, ep, st);
}

}  // extern "C"
