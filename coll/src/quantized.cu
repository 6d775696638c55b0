// libb200coll quantising collectives: bf16, fp16 or fp32 in, block-scaled FP8 over NVLink, bf16, fp16 or fp32 out, one kernel per call.
// Each rank quantises its own send buffer to e4m3 / e5m2 with one fp32 scale per `block` consecutive elements, into a library-owned
// symmetric scratch; peers pull the FP8 copy and its scales, dequantise in registers and sum in fp32 in rank order (blockscale.cuh):
//
//   k_quant_ag<InT, WireT, OutT>                  all-gather: quantise my shard, barrier, pull and dequantise every rank's shard, barrier
//   k_quant_pull_reduce<InT, WireT, OutT, false>  reduce-scatter (my slice) / one-shot all-reduce (whole buffer): quantise, barrier,
//                                                 pull from every rank in rank order, sum in fp32, scale, round once, store locally
//   k_quant_pull_reduce<InT, WireT, OutT, true>   two-shot all-reduce: the same over my block slice, the result pushed into every recv
//   k_quant_copy<InT, WireT, OutT>                one rank: the quantise / dequantise round trip in registers, no scratch, no barrier
//
// Per block: amax = max |x| (the largest unsigned bit pattern of |x|, so a NaN anywhere makes amax NaN); inv = FMAX / amax and
// s = amax / FMAX, both IEEE divisions rounded to nearest, inv = s = 1 when amax == 0 or inv overflows; q = fp8_satfinite(x * inv);
// the dequantised value is float(q) * s. FMAX is 448 (e4m3) or 57344 (e5m2).
//
// Fusing the quantise phase into the pull kernel is sound because of three properties, which the code below keeps:
//   * Same-index CTAs only. The epoch barrier orders CTA b of this rank against CTA b of every peer, nothing else. So the quantise
//     loop walks each rank-slice exactly as the pull loop walks it (same grid, same start per slice, same stride): every vector CTA b
//     pulls from a peer after the barrier was quantised by CTA b on that peer before it. All-gather walks the whole shard; reduce-scatter
//     and two-shot walk each of the N slices in turn; one-shot walks the whole buffer once.
//   * Blocks stay inside one warp iteration. block is a power of two from 16 to 512 elements (1 to 32 vectors), a warp's first vector
//     is the slice start plus a multiple of 32, and slice starts and ends fall on whole blocks (the two-shot slices are cut at
//     nblk*r/N blocks, not nvec*r/N vectors). So the lanes of one block are consecutive lanes of one warp, all active or all idle, and
//     the amax is a butterfly over those lanes: no shared memory, no cross-warp step.
//   * The first barrier releases. The block-scaled kernels take it relaxed because their inputs were written by earlier kernels; here
//     this CTA's own scratch stores must be visible to the peers that pull them, so it is barrier_blocks<true>.
// The same argument makes the in-place all-reduce safe on both algorithms: vector v of send is read only by the CTA that walks it, and
// is overwritten (by that CTA locally in one-shot, by CTA b of the slice owner in two-shot) only after that CTA has passed the first
// barrier, which follows the read.
//
// The final barrier keeps the scratch safe to reuse: no rank's kernel ends before every peer's CTAs have finished pulling from it.
#include <math.h>
#include <stdint.h>

#include <type_traits>

#include "blockscale.cuh"
#include "comm.h"
#include "launch.cuh"

namespace b200coll {

constexpr int kQuantThreads = 512;

template <typename WireT> constexpr float kWireMax = 448.0f;
template <> constexpr float kWireMax<__nv_fp8_e5m2> = 57344.0f;

struct QuantGeom {
  size_t q_off, s_off;   // arena offsets of the scratch FP8 copy and of its scales (the same on every rank)
  uint32_t nvec;         // 16-element vectors in one rank's send buffer
  uint32_t nblk;         // blocks in one rank's send buffer
  uint32_t lvpb;         // log2(vectors per block)
};

// the first vector of slice s of n: slices are cut at whole blocks
__device__ __forceinline__ uint32_t quant_slice_start(const QuantGeom& g, uint32_t s, uint32_t n) {
  return (uint32_t)((unsigned long long)g.nblk * s / n) << g.lvpb;
}

// 16 elements of InT at p, widened (exactly) to fp32
template <typename InT> __device__ __forceinline__ void quant_load16(const char* p, float* x) {
  if constexpr (std::is_same<InT, float>::value) {
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const uint4 v = ld_vec(p + 16 * k);
      x[4 * k] = __uint_as_float(v.x); x[4 * k + 1] = __uint_as_float(v.y); x[4 * k + 2] = __uint_as_float(v.z); x[4 * k + 3] = __uint_as_float(v.w);
    }
  } else {
#pragma unroll
    for (int k = 0; k < 2; k++) {
      const uint4 v = ld_vec(p + 16 * k);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int i = 0; i < 4; i++) {
        if constexpr (std::is_same<InT, __nv_bfloat16>::value) {
          x[8 * k + 2 * i] = __uint_as_float(w[i] << 16); x[8 * k + 2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
        } else {
          const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
          x[8 * k + 2 * i] = f.x; x[8 * k + 2 * i + 1] = f.y;
        }
      }
    }
  }
}

// Quantise this lane's 16 elements with the amax of its block, whose vectors are held by the aligned group of `gl` lanes (a power of
// two up to 32) this lane belongs to. All 32 lanes call it; idle lanes pass zeros, and their groups are wholly idle. Returns the FP8
// vector; *scale receives s.
template <typename WireT> __device__ __forceinline__ uint4 quant_vec(const float* x, uint32_t gl, float* scale) {
  uint32_t m = 0;
#pragma unroll
  for (int i = 0; i < 16; i++) m = max(m, __float_as_uint(x[i]) & 0x7FFFFFFFu);
  for (uint32_t o = 1; o < gl; o <<= 1) m = max(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
  const float amax = __uint_as_float(m);
  float inv = __fdiv_rn(kWireMax<WireT>, amax), s = __fdiv_rn(amax, kWireMax<WireT>);
  if (amax == 0.0f || inv == INFINITY) { inv = 1.0f; s = 1.0f; }
  float y[16];
#pragma unroll
  for (int i = 0; i < 16; i++) y[i] = __fmul_rn(x[i], inv);
  uint32_t w[4];
  Pack<WireT, 16>::run(y, w);                                     // cvt.rn.satfinite: F2FP.SATFINITE.E4M3 / .E5M2
  *scale = s;
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// Quantise vectors [v0, v1) of my send buffer into my scratch, walked exactly as the pull loops below walk a slice.
template <typename InT, typename WireT>
__device__ __forceinline__ void quant_range(const QuantGeom& g, const char* in, char* q, char* scales, uint32_t v0, uint32_t v1) {
  const uint32_t lane = threadIdx.x & 31, gl = 1u << g.lvpb;
  for (uint32_t b = v0 + blockIdx.x * blockDim.x + (threadIdx.x & ~31u); b < v1; b += gridDim.x * blockDim.x) {
    const uint32_t v = b + lane;
    const bool act = v < v1;
    float x[16] = {};
    if (act) quant_load16<InT>(in + (size_t)v * (16 * sizeof(InT)), x);
    float s;
    const uint4 w = quant_vec<WireT>(x, gl, &s);
    if (act) {
      st_vec(q + (size_t)v * 16, w);
      if ((lane & (gl - 1)) == 0) *reinterpret_cast<float*>(scales + (size_t)(v >> g.lvpb) * 4) = s;
    }
  }
}

template <typename InT, typename WireT, typename OutT>
__global__ void __launch_bounds__(kQuantThreads) k_quant_copy(const char* in, OutT* out, uint32_t nvec, uint32_t lvpb, float scale) {
  pdl_prologue();
  const uint32_t lane = threadIdx.x & 31, gl = 1u << lvpb;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t b = (size_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); b < nvec; b += stride) {
    const size_t v = b + lane;
    const bool act = v < nvec;
    float x[16] = {};
    if (act) quant_load16<InT>(in + v * (16 * sizeof(InT)), x);
    float s;
    const uint4 w = quant_vec<WireT>(x, gl, &s);
    if (act) {
      float acc[16] = {};
      bsq_dequant_add<WireT>(acc, w, s);
      bsq_store<OutT>(out + v * 16, acc, scale);
    }
  }
}

// out holds nranks shards of nvec*16 elements; shard r is rank r's send buffer quantised and dequantised with rank r's scales
template <typename InT, typename WireT, typename OutT>
__global__ void __launch_bounds__(kQuantThreads) k_quant_ag(COMM_PARAM, const __grid_constant__ QuantGeom g, const char* __restrict__ in, OutT* __restrict__ out,
                                                            float scale, uint32_t op) {
  pdl_prologue();
  quant_range<InT, WireT>(g, in, c.peer[c.rank] + g.q_off, c.peer[c.rank] + g.s_off, 0, g.nvec);
  const uint32_t s = load_seq(c, kSeqBarrier);
  if (!barrier_blocks<true>(c, 2 * s + 1, op)) return;           // every rank's CTA b has quantised the vectors CTA b pulls below
  const uint32_t lane = threadIdx.x & 31;
  for (int j = 0; j < c.nranks; j++) {                          // peers visited starting with myself: spreads the pulls over the links
    int r = c.rank + j; if (r >= c.nranks) r -= c.nranks;
    const char* q = c.peer[r] + g.q_off;
    const char* sc = c.peer[r] + g.s_off;
    OutT* dst = out + (size_t)r * g.nvec * 16;
    for (uint32_t b = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); b < g.nvec; b += gridDim.x * blockDim.x) {
      const uint32_t v = b + lane;
      const bool act = v < g.nvec;
      uint4 d = make_uint4(0, 0, 0, 0);
      if (act) d = ld_vec(q + (size_t)v * 16);
      const uint32_t idx = v >> g.lvpb;
      const WarpScale ws(idx, act);
      const float sr = ws.get(sc, idx);
      if (act) {
        float acc[16] = {};
        bsq_dequant_add<WireT>(acc, d, sr);
        bsq_store<OutT>(dst + (size_t)v * 16, acc, scale);
      }
    }
  }
  if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;           // nobody reads my scratch any more: the next call may overwrite it
  if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
}

// nslices == 1: one-shot all-reduce, the whole buffer is quantised and reduced (stored at out_local[v * 16]).
// nslices == N: reduce-scatter (PUSH=false, my slice stored at out_local[(v - v0) * 16]) or two-shot all-reduce (PUSH=true, my slice
// stored at arena offset out_off + v * 16 * sizeof(OutT) of every rank). in and out_local may be the same buffer (in-place all-reduce).
template <typename InT, typename WireT, typename OutT, bool PUSH>
__global__ void __launch_bounds__(kQuantThreads, 1) k_quant_pull_reduce(COMM_PARAM, const __grid_constant__ QuantGeom g, const char* in, OutT* out_local, size_t out_off,
                                                                        uint32_t nslices, float scale, uint32_t op) {
  pdl_prologue();
  for (uint32_t sl = 0; sl < nslices; sl++)
    quant_range<InT, WireT>(g, in, c.peer[c.rank] + g.q_off, c.peer[c.rank] + g.s_off, quant_slice_start(g, sl, nslices), quant_slice_start(g, sl + 1, nslices));
  {
    const uint32_t s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<true>(c, 2 * s + 1, op)) return;
  }
  const uint32_t me = nslices == 1 ? 0u : (uint32_t)c.rank;
  const uint32_t v0 = quant_slice_start(g, me, nslices), v1 = quant_slice_start(g, me + 1, nslices);
  const uint32_t lane = threadIdx.x & 31;
  for (uint32_t b = v0 + blockIdx.x * blockDim.x + (threadIdx.x & ~31u); b < v1; b += gridDim.x * blockDim.x) {
    const uint32_t v = b + lane;
    const bool act = v < v1;
    uint4 d[kMaxRanks];
#pragma unroll
    for (int r = 0; r < kMaxRanks; r++) if (r < c.nranks) d[r] = act ? ld_vec(c.peer[r] + g.q_off + (size_t)v * 16) : make_uint4(0, 0, 0, 0);
    const uint32_t idx = v >> g.lvpb;
    const WarpScale ws(idx, act);
    float acc[16] = {};
#pragma unroll
    for (int r = 0; r < kMaxRanks; r++) if (r < c.nranks) {
      const float sr = ws.get(c.peer[r] + g.s_off, idx);
      bsq_dequant_add<WireT>(acc, d[r], sr);
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
  const uint32_t s = load_seq(c, kSeqBarrier);
  if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;
  if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
}

// ------------------------------------------------------------------------------------------------ host side
template <typename T> struct QTag { using type = T; };

template <typename F>
static b200collResult_t dispatch_quant(b200collDataType_t in, b200collDataType_t wire, b200collDataType_t out, F&& f) {
  auto outs = [&](auto ti, auto tw) -> b200collResult_t {
    switch (out) {
      case b200collBfloat16: return f(ti, tw, QTag<__nv_bfloat16>{});
      case b200collFloat16: return f(ti, tw, QTag<__half>{});
      default: return f(ti, tw, QTag<float>{});
    }
  };
  auto wires = [&](auto ti) -> b200collResult_t {
    return wire == b200collFloat8e4m3 ? outs(ti, QTag<__nv_fp8_e4m3>{}) : outs(ti, QTag<__nv_fp8_e5m2>{});
  };
  switch (in) {
    case b200collBfloat16: return wires(QTag<__nv_bfloat16>{});
    case b200collFloat16: return wires(QTag<__half>{});
    default: return wires(QTag<float>{});
  }
}

static bool wide_type(b200collDataType_t t) { return t == b200collBfloat16 || t == b200collFloat16 || t == b200collFloat32; }

static bool ranges_overlap(const void* a, size_t na, const void* b, size_t nb) {
  const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
  return x < y + nb && y < x + na;
}

struct QuantCall {
  b200collComm* c;
  size_t count;        // elements of one rank's send buffer
  size_t in_bytes;     // bytes of my send
  size_t out_bytes;    // bytes of my recv
  float scale;         // ep->scale, times 1/nranks for avg
  QuantGeom g;
};

// Everything the three entry points check before they touch the scratch or launch; count == 0 is left to the caller.
static b200collResult_t quant_prepare(b200collComm* c, b200collOp_t which, const void* send, void* recv, size_t count, b200collDataType_t wire, int block,
                                      const b200collEpilogue* ep, b200collRedOp_t rop, QuantCall* call) {
  if (!c || !send || !recv || !ep) { set_last_error("null argument"); return b200collInvalidArgument; }
  if (!wide_type(ep->in_dtype)) { set_last_error("quantised collectives: in_dtype must be bf16, fp16 or fp32"); return b200collInvalidArgument; }
  if (!wide_type(ep->out_dtype)) { set_last_error("quantised collectives: out_dtype must be bf16, fp16 or fp32"); return b200collInvalidArgument; }
  if (wire != b200collFloat8e4m3 && wire != b200collFloat8e5m2) { set_last_error("quantised collectives: wire_dtype must be e4m3 or e5m2"); return b200collInvalidArgument; }
  if (block < 16 || block > 512 || (block & (block - 1)) != 0) { set_last_error("quantised collectives: block must be 16, 32, 64, 128, 256 or 512"); return b200collInvalidArgument; }
  if (which != b200collOpAllGather && rop != b200collSum && rop != b200collAvg) { set_last_error("quantised reductions take sum or avg only"); return b200collInvalidArgument; }
  const size_t per_rank_check = which == b200collOpReduceScatter ? count / (size_t)c->nranks : count;
  if (per_rank_check % (size_t)block != 0) {
    set_last_error(which == b200collOpReduceScatter ? "quantised reduce-scatter: recvcount must be a multiple of block" : "quantised collectives: the count must be a multiple of block");
    return b200collInvalidArgument;
  }
  if (count / 16 >= ((size_t)1 << 31)) { set_last_error("quantised collectives: fewer than 2^35 elements per rank"); return b200collInvalidArgument; }
  if (!aligned(send, 16) || !aligned(recv, 16)) { set_last_error("send and recv must be 16-byte aligned"); return b200collInvalidArgument; }
  if (c->fault_host && *const_cast<volatile uint32_t*>(&c->fault_host->code) != 0) { set_last_error("communicator is poisoned by an earlier watchdog fault"); return b200collRemoteError; }
  const size_t is = b200collTypeSize(ep->in_dtype), os = b200collTypeSize(ep->out_dtype);
  call->c = c;
  call->count = count;
  call->in_bytes = count * is;
  call->out_bytes = (which == b200collOpAllGather ? count * c->nranks : which == b200collOpReduceScatter ? count / c->nranks : count) * os;
  call->scale = ep->scale * (rop == b200collAvg && which != b200collOpAllGather ? 1.0f / (float)c->nranks : 1.0f);
  if (count == 0) return b200collSuccess;
  // in place (all-reduce only): every vector is read and rewritten at the same position, so the element sizes must agree
  const bool in_place = which == b200collOpAllReduce && send == recv && is == os;
  if (!in_place && ranges_overlap(send, call->in_bytes, recv, call->out_bytes)) {
    set_last_error(which == b200collOpAllReduce ? "quantised all-reduce: recv must be send (with in_dtype and out_dtype of one size) or not overlap it"
                                                : "quantised collectives: recv must not overlap send");
    return b200collInvalidArgument;
  }
  QuantGeom& g = call->g;
  g.nvec = (uint32_t)(count / 16);
  g.nblk = (uint32_t)(count / (size_t)block);
  g.lvpb = 0;
  while ((16u << g.lvpb) < (uint32_t)block) g.lvpb++;
  return b200collSuccess;
}

// The FP8 copy (count bytes) and its scales (count / block fp32) of one call, in the symmetric heap. Taken with b200collMemAlloc on first
// use and grown on demand: a collective contract like MemAlloc (every rank makes the same quantised calls in the same order, so every
// rank gets the same offsets). A superseded scratch is never given back before CommDestroy: a CUDA graph captured earlier still
// addresses it, and must stay valid when a later, larger call moves the scratch.
static b200collResult_t quant_scratch(b200collComm* c, QuantCall* k) {
  const size_t qbytes = k->count, need = qbytes + (size_t)k->g.nblk * 4;
  if (c->quant_scratch_bytes < need) {
    void* p = nullptr;
    size_t bytes = std::max(need, 2 * c->quant_scratch_bytes);
    b200collResult_t rc = b200collMemAlloc(c, &p, bytes);
    if (rc != b200collSuccess && bytes != need) rc = b200collMemAlloc(c, &p, bytes = need);
    if (rc != b200collSuccess) {
      set_last_error("quantised collectives: the symmetric arena cannot hold the " + std::to_string(need) + "-byte FP8 scratch (raise B200COLL_ARENA_MB)");
      return rc;
    }
    if (c->quant_scratch) c->quant_scratch_retired.push_back(c->quant_scratch);
    c->quant_scratch = p;
    c->quant_scratch_bytes = bytes;
  }
  k->g.q_off = arena_off(c, c->quant_scratch);
  k->g.s_off = k->g.q_off + qbytes;                               // count is a multiple of 16: the scales are 16-byte aligned
  return b200collSuccess;
}

// nranks == 1: the round trip in registers; grid as for the fused copy (streaming, 8 CTAs of 256 threads per SM at most)
static b200collResult_t quant_copy(const QuantCall& k, const void* send, void* recv, b200collDataType_t wire, const b200collEpilogue* ep, cudaStream_t st) {
  b200collComm* c = k.c;
  return dispatch_quant(ep->in_dtype, wire, ep->out_dtype, [&](auto ti, auto tw, auto to) -> b200collResult_t {
    using InT = typename decltype(ti)::type; using WireT = typename decltype(tw)::type; using OutT = typename decltype(to)::type;
    const int blocks = (int)std::max<size_t>(1, std::min<size_t>(((size_t)k.g.nvec + 255) / 256, (size_t)std::max(1, c->sm_count) * 8));
    launch_k(k_quant_copy<InT, WireT, OutT>, blocks, 256, st, static_cast<const char*>(send), static_cast<OutT*>(recv), k.g.nvec, k.g.lvpb, k.scale);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  });
}

// whole warps: a block's lanes must never straddle a partial warp
static Grid quant_grid(const b200collComm* c, size_t vecs) {
  Grid gr = pick_grid(c, kShapeP2p, vecs, 1);
  gr.threads = std::max(32, gr.threads & ~31);
  return gr;
}

static b200collResult_t quant_reduce(const QuantCall& k, b200collOp_t which, b200collAlgo_t algo, const void* send, void* recv, b200collDataType_t wire,
                                     const b200collEpilogue* ep, cudaStream_t st) {
  b200collComm* c = k.c;
  const uint32_t n = (uint32_t)c->nranks;
  const uint32_t nslices = (which == b200collOpReduceScatter || algo == b200collAlgoTwoShot) ? n : 1u;
  return dispatch_quant(ep->in_dtype, wire, ep->out_dtype, [&](auto ti, auto tw, auto to) -> b200collResult_t {
    using InT = typename decltype(ti)::type; using WireT = typename decltype(tw)::type; using OutT = typename decltype(to)::type;
    const char* in = static_cast<const char*>(send);
    if (algo == b200collAlgoTwoShot) {
      const Grid gr = quant_grid(c, k.g.nvec / n + 1);
      launch_k(k_quant_pull_reduce<InT, WireT, OutT, true>, gr.blocks, gr.threads, st, c->dev, k.g, in, static_cast<OutT*>(nullptr), arena_off(c, recv), nslices, k.scale,
               (uint32_t)which);
    } else {
      const Grid gr = quant_grid(c, which == b200collOpReduceScatter ? k.g.nvec / n : k.g.nvec);
      launch_k(k_quant_pull_reduce<InT, WireT, OutT, false>, gr.blocks, gr.threads, st, c->dev, k.g, in, static_cast<OutT*>(recv), (size_t)0, nslices, k.scale,
               (uint32_t)which);
    }
    LAUNCH_CHECK(c);
    return b200collSuccess;
  });
}

}  // namespace b200coll

using namespace b200coll;

extern "C" {

b200collResult_t b200collAllGatherQuantized(const void* send, void* recv, size_t sendcount, b200collDataType_t wire_dtype, int block,
                                            const b200collEpilogue* ep, b200collComm_t c, b200collStream_t stream) {
  QuantCall k;
  b200collResult_t rc = quant_prepare(c, b200collOpAllGather, send, recv, sendcount, wire_dtype, block, ep, b200collSum, &k);
  if (rc != b200collSuccess || sendcount == 0) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (c->nranks == 1) { account(c, b200collOpAllGather, k.in_bytes, b200collAlgoCopy); return quant_copy(k, send, recv, wire_dtype, ep, st); }
  if ((rc = quant_scratch(c, &k)) != b200collSuccess) return rc;
  rc = cross_check(c, b200collOpAllGather, b200collAlgoOneShot, sendcount, k.g.q_off, k.g.s_off);
  if (rc != b200collSuccess) return rc;
  account(c, b200collOpAllGather, k.in_bytes, b200collAlgoOneShot);
  return dispatch_quant(ep->in_dtype, wire_dtype, ep->out_dtype, [&](auto ti, auto tw, auto to) -> b200collResult_t {
    using InT = typename decltype(ti)::type; using WireT = typename decltype(tw)::type; using OutT = typename decltype(to)::type;
    const Grid gr = quant_grid(c, k.g.nvec);
    launch_k(k_quant_ag<InT, WireT, OutT>, gr.blocks, gr.threads, st, c->dev, k.g, static_cast<const char*>(send), static_cast<OutT*>(recv), k.scale,
             (uint32_t)b200collOpAllGather);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  });
}

b200collResult_t b200collReduceScatterQuantized(const void* send, void* recv, size_t recvcount, b200collDataType_t wire_dtype, int block,
                                                const b200collEpilogue* ep, b200collRedOp_t op, b200collComm_t c, b200collStream_t stream) {
  if (c && recvcount > SIZE_MAX / B200COLL_MAX_RANKS) { set_last_error("recvcount too large"); return b200collInvalidArgument; }
  QuantCall k;
  b200collResult_t rc = quant_prepare(c, b200collOpReduceScatter, send, recv, c ? recvcount * c->nranks : 0, wire_dtype, block, ep, op, &k);
  if (rc != b200collSuccess || recvcount == 0) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t bytes = recvcount * b200collTypeSize(ep->in_dtype);
  if (c->nranks == 1) { account(c, b200collOpReduceScatter, bytes, b200collAlgoCopy); return quant_copy(k, send, recv, wire_dtype, ep, st); }
  if ((rc = quant_scratch(c, &k)) != b200collSuccess) return rc;
  rc = cross_check(c, b200collOpReduceScatter, b200collAlgoOneShot, recvcount, k.g.q_off, k.g.s_off);
  if (rc != b200collSuccess) return rc;
  account(c, b200collOpReduceScatter, bytes, b200collAlgoOneShot);
  return quant_reduce(k, b200collOpReduceScatter, b200collAlgoOneShot, send, recv, wire_dtype, ep, st);
}

b200collResult_t b200collAllReduceQuantized(const void* send, void* recv, size_t count, b200collDataType_t wire_dtype, int block,
                                            const b200collEpilogue* ep, b200collRedOp_t op, b200collComm_t c, b200collStream_t stream) {
  QuantCall k;
  b200collResult_t rc = quant_prepare(c, b200collOpAllReduce, send, recv, count, wire_dtype, block, ep, op, &k);
  if (rc != b200collSuccess || count == 0) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (c->nranks == 1) { account(c, b200collOpAllReduce, k.in_bytes, b200collAlgoCopy); return quant_copy(k, send, recv, wire_dtype, ep, st); }
  // the same mapping as b200collAllReduceBlockScaled: the table's pick for an FP8 all-reduce of `count` bytes (or the forced algorithm);
  // two-shot pushes into every rank's recv, so it needs recv in the arena and falls back to one-shot otherwise
  const b200collAlgo_t want = c->forced_algo != b200collAlgoAuto ? c->forced_algo : b200collTunerPick(b200collOpAllReduce, count, c->nranks, c->nvls);
  b200collAlgo_t algo = (want == b200collAlgoTwoShot || want == b200collAlgoNvls) ? b200collAlgoTwoShot : b200collAlgoOneShot;
  if (algo == b200collAlgoTwoShot && !b200collIsSymmetric(c, recv, k.out_bytes)) algo = b200collAlgoOneShot;
  if ((rc = quant_scratch(c, &k)) != b200collSuccess) return rc;
  rc = cross_check(c, b200collOpAllReduce, algo, count, k.g.q_off, algo == b200collAlgoTwoShot ? arena_off(c, recv) : k.g.s_off);
  if (rc != b200collSuccess) return rc;
  account(c, b200collOpAllReduce, k.in_bytes, algo);
  return quant_reduce(k, b200collOpAllReduce, algo, send, recv, wire_dtype, ep, st);
}

}  // extern "C"
