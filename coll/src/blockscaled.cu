// libb200coll block-scaled FP8 collectives, in two families that share one pull-and-dequantise core. FP8 and fp32 block scales cross
// NVLink; receivers pull them from every peer, dequantise in registers, sum in fp32 in rank order, round once and store bf16, fp16 or
// fp32 locally (or, in the two-shot all-reduce, push the finished result once).
//
// Block-scaled: e4m3 / e5m2 matrices with one fp32 scale per block_rows x block_cols block (1x128 activation and gradient blocks,
// 128x128 weight blocks), written by the caller into the arena:
//
//   k_bsq_ag_pull<InT, OutT>              all-gather: barrier, pull every rank's FP8 shard and scales, dequantise, store locally, barrier
//   k_bsq_pull_reduce<InT, OutT, false>   reduce-scatter (my row slice) / one-shot all-reduce (whole matrix): pull from every rank in
//                                         rank order, dequantise with that rank's scales, sum in fp32, scale, round once, store locally
//   k_bsq_pull_reduce<InT, OutT, true>    two-shot all-reduce: the same over my vector slice, the result pushed into every rank's recv
//   k_bsq_copy<InT, OutT>                 one rank: local dequantising copy, no barrier
//
// Quantising: bf16, fp16 or fp32 in, one kernel per call. Each rank quantises its own send buffer to e4m3 / e5m2 with one fp32 scale
// per `block` consecutive elements, into a library-owned symmetric scratch; from there the block-scaled pull applies:
//
//   k_quant_ag<InT, WireT, OutT>                  all-gather: quantise my shard, barrier, pull and dequantise every rank's shard, barrier
//   k_quant_pull_reduce<InT, WireT, OutT, false>  reduce-scatter (my slice) / one-shot all-reduce (whole buffer): quantise, barrier,
//                                                 pull from every rank in rank order, sum in fp32, scale, round once, store locally
//   k_quant_pull_reduce<InT, WireT, OutT, true>   two-shot all-reduce: the same over my block slice, the result pushed into every recv
//   k_quant_copy<InT, WireT, OutT>                one rank: the quantise / dequantise round trip in registers, no scratch, no barrier
//
// Scales: a 16-byte FP8 vector lies in exactly one block (row_len and block_cols are multiples of 16; a quantising block is a whole
// number of vectors), so a vector needs one scale per rank. Lanes of a warp hold consecutive vectors and usually share scales (8 lanes
// per 1x128 block, whole warps per 128x128 block): __match_any_sync groups the lanes by scale index, the lowest lane of each group loads
// the scale and __shfl_sync hands it to the rest, so each distinct scale is read once per warp and rank. Each family's geometry maps a
// vector to its scale: the block-scaled vector -> (row, column) -> block arithmetic is 32-bit multiply-high division by host-computed
// constants (no integer division in the loops), a quantising block is a shift.
//
// Quantising, per block: the rule in quant.cuh, which also holds the quantise and dequantise helpers this file shares with dispatch.cu
// and combine.cu. The quantising combine (combine.cu) shares this file's scratch (quant_scratch_take).
//
// Fusing the quantise phase into the pull kernel is sound because of three properties, which the code below keeps:
//   * Same-index CTAs only. The epoch barrier orders CTA b of this rank against CTA b of every peer, nothing else. Every vector loop in
//     this file is warp_walk, so the quantise loop walks each rank-slice exactly as the pull loop walks it (same grid, same start per slice,
//     same stride): every vector CTA b pulls from a peer after the barrier was quantised by CTA b on that peer before it. All-gather
//     walks the whole shard; reduce-scatter and two-shot walk each of the N slices in turn; one-shot walks the whole buffer once.
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
#include <limits.h>
#include <math.h>
#include <stdint.h>

#include <type_traits>

#include "comm.h"
#include "launch.cuh"
#include "quant.cuh"

namespace b200coll {

// q = floor(n / d) for every 32-bit n as (umulhi(n, m) + n) >> l, l = ceil(log2 d), m = floor(2^32 (2^l - d) / d) + 1 (Granlund and
// Montgomery, "Division by invariant integers using multiplication", 1994). The sum needs 33 bits, so it is formed in 64.
struct FastDiv {
  uint32_t d, m, l;
  __device__ __forceinline__ uint32_t div(uint32_t n) const { return (uint32_t)(((unsigned long long)__umulhi(n, m) + n) >> l); }
};
inline FastDiv make_fastdiv(uint32_t d) {
  uint32_t l = 0;
  while (l < 32 && (1ull << l) < d) l++;
  return FastDiv{d, (uint32_t)(((1ull << 32) * ((1ull << l) - d)) / d + 1), l};
}

// What every kernel needs to find vector v of a rank's FP8 data and its scale. Vector indices are 32-bit (the host refuses larger).
struct BsqGeom {
  size_t data_off, scale_off;     // arena offsets of the caller's FP8 matrix and of its scales (the same on every rank)
  uint32_t nvec;                  // 16-element vectors in one rank's matrix
  uint32_t ncb;                   // block columns (scales per block row)
  FastDiv vpr, br, vpb;           // vectors per row, rows per block, vectors per block column
  __device__ __forceinline__ uint32_t scale_index(uint32_t v) const {
    const uint32_t row = vpr.div(v), cv = v - row * vpr.d;
    return br.div(row) * ncb + vpb.div(cv);
  }
};

// The scale of every lane's vector, one load per distinct index in the warp. All 32 lanes call it; `active` lanes have a vector.
struct WarpScale {
  unsigned leader;
  bool loads;
  __device__ __forceinline__ WarpScale(uint32_t idx, bool active) {
    const unsigned same = __match_any_sync(0xFFFFFFFFu, active ? idx : 0xFFFFFFFFu);
    leader = __ffs(same) - 1;
    loads = active && (threadIdx.x & 31) == leader;
  }
  __device__ __forceinline__ float get(const char* scales, uint32_t idx) const {
    float s = 0.f;
    if (loads) s = *reinterpret_cast<const float*>(scales + (size_t)idx * 4);
    return __shfl_sync(0xFFFFFFFFu, s, leader);
  }
};

// Dequantise vectors [0, nvec) of one rank's FP8 data into dst.
template <typename WireT, typename OutT, typename Geom>
__device__ __forceinline__ void dequant_range(const Geom& g, const char* src, const char* scales, OutT* dst, float scale) {
  warp_walk(0, g.nvec, [&](uint32_t v, bool act) {
    uint4 q = make_uint4(0, 0, 0, 0);
    if (act) q = ld_vec(src + (size_t)v * 16);
    const uint32_t idx = act ? g.scale_index(v) : 0u;
    const WarpScale ws(idx, act);
    const float s = ws.get(scales, idx);
    if (act) {
      float acc[16] = {};
      bsq_dequant_add<WireT>(acc, q, s);
      store16_scaled<OutT>(dst + (size_t)v * 16, acc, scale);
    }
  });
}

// All-gather: out holds nranks shards of nvec*16 elements; shard r is rank r's FP8 data dequantised with rank r's scales
template <typename WireT, typename OutT, typename Geom>
__device__ __forceinline__ void ag_pull(const CommDev& c, const Geom& g, OutT* out, float scale) {
  for (int j = 0; j < c.nranks; j++) {                          // peers visited starting with myself: spreads the pulls over the links
    int r = c.rank + j; if (r >= c.nranks) r -= c.nranks;
    dequant_range<WireT, OutT>(g, c.peer[r] + g.data_off, c.peer[r] + g.scale_off, out + (size_t)r * g.nvec * 16, scale);
  }
}

// Vectors [v0, v1) summed over ranks in rank order: acc = ((0 + v_0) + v_1 + ...), then round_once(acc * scale).
// PUSH=false: stored at out_local[(v - v0) * 16] (reduce-scatter: my slice; one-shot all-reduce: v0 = 0, v1 = nvec).
// PUSH=true: stored at arena offset out_off + v * 16 * sizeof(OutT) of every rank (two-shot all-reduce, my vector slice).
template <typename WireT, typename OutT, bool PUSH, typename Geom>
__device__ __forceinline__ void pull_reduce_range(const CommDev& c, const Geom& g, OutT* out_local, size_t out_off, uint32_t v0, uint32_t v1, float scale) {
  warp_walk(v0, v1, [&](uint32_t v, bool act) {
    uint4 d[kMaxRanks];
#pragma unroll
    for (int r = 0; r < kMaxRanks; r++) if (r < c.nranks) d[r] = act ? ld_vec(c.peer[r] + g.data_off + (size_t)v * 16) : make_uint4(0, 0, 0, 0);
    const uint32_t idx = act ? g.scale_index(v) : 0u;
    const WarpScale ws(idx, act);
    float acc[16] = {};
#pragma unroll
    for (int r = 0; r < kMaxRanks; r++) if (r < c.nranks) {
      const float sr = ws.get(c.peer[r] + g.scale_off, idx);
      bsq_dequant_add<WireT>(acc, d[r], sr);
    }
    if (act) {
      if (PUSH) {
#pragma unroll
        for (int j = 0; j < kMaxRanks; j++) if (j < c.nranks) {
          int r = c.rank + j; if (r >= c.nranks) r -= c.nranks;
          store16_scaled<OutT>(c.peer[r] + out_off + (size_t)v * (16 * sizeof(OutT)), acc, scale);
        }
      } else {
        store16_scaled<OutT>(out_local + (size_t)(v - v0) * 16, acc, scale);
      }
    }
  });
}

// Block-scaled kernels.
template <typename InT, typename OutT>
__global__ void __launch_bounds__(kBsqThreads) k_bsq_copy(const __grid_constant__ BsqGeom g, const char* __restrict__ in, const char* __restrict__ scales,
                                                       OutT* __restrict__ out, float scale) {
  pdl_prologue();
  dequant_range<InT, OutT>(g, in, scales, out, scale);
}

template <typename InT, typename OutT>
__global__ void __launch_bounds__(kBsqThreads) k_bsq_ag_pull(COMM_PARAM, const __grid_constant__ BsqGeom g, OutT* __restrict__ out, float scale, uint32_t op) {
  pdl_prologue();
  const uint32_t s = load_seq(c, kSeqBarrier);
  if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;          // every rank's shard and scales are written
  ag_pull<InT, OutT>(c, g, out, scale);
  if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;           // nobody reads my shard any more: I may overwrite it
  if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
}

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
  pull_reduce_range<InT, OutT, PUSH>(c, g, out_local, out_off, v0, v1, scale);
  // the sequence number is read again rather than kept live across the loop: only the last block, after the barrier below, bumps it
  const uint32_t s = load_seq(c, kSeqBarrier);
  if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;
  if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
}

// Quantising kernels.
// the first vector of slice s of n: slices are cut at whole blocks
__device__ __forceinline__ uint32_t quant_slice_start(const QuantGeom& g, uint32_t s, uint32_t n) {
  return (uint32_t)((unsigned long long)g.nblk * s / n) << g.lvpb;
}

template <typename InT, typename WireT, typename OutT>
__global__ void __launch_bounds__(kBsqThreads) k_quant_copy(const char* in, OutT* out, uint32_t nvec, uint32_t lvpb, float scale) {
  pdl_prologue();
  const uint32_t gl = 1u << lvpb;
  warp_walk(0, nvec, [&](uint32_t v, bool act) {
    float x[16] = {};
    if (act) quant_load16<InT>(in + (size_t)v * (16 * sizeof(InT)), x);
    float s;
    const uint4 w = quant_vec<WireT>(x, gl, &s);
    if (act) {
      float acc[16] = {};
      bsq_dequant_add<WireT>(acc, w, s);
      store16_scaled<OutT>(out + (size_t)v * 16, acc, scale);
    }
  });
}

template <typename InT, typename WireT, typename OutT>
__global__ void __launch_bounds__(kBsqThreads) k_quant_ag(COMM_PARAM, const __grid_constant__ QuantGeom g, const char* __restrict__ in, OutT* __restrict__ out,
                                                          float scale, uint32_t op) {
  pdl_prologue();
  quant_range<InT, WireT>(g, in, c.peer[c.rank] + g.data_off, c.peer[c.rank] + g.scale_off, 0, g.nvec);
  const uint32_t s = load_seq(c, kSeqBarrier);
  if (!barrier_blocks<true>(c, 2 * s + 1, op)) return;           // every rank's CTA b has quantised the vectors CTA b pulls below
  ag_pull<WireT, OutT>(c, g, out, scale);
  if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;           // nobody reads my scratch any more: the next call may overwrite it
  if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
}

// nslices == 1: one-shot all-reduce, the whole buffer is quantised and reduced. nslices == N: reduce-scatter (PUSH=false) or two-shot
// all-reduce (PUSH=true) of my block slice. in and out_local may be the same buffer (in-place all-reduce).
template <typename InT, typename WireT, typename OutT, bool PUSH>
__global__ void __launch_bounds__(kBsqThreads, 1) k_quant_pull_reduce(COMM_PARAM, const __grid_constant__ QuantGeom g, const char* in, OutT* out_local, size_t out_off,
                                                                      uint32_t nslices, float scale, uint32_t op) {
  pdl_prologue();
  for (uint32_t sl = 0; sl < nslices; sl++)
    quant_range<InT, WireT>(g, in, c.peer[c.rank] + g.data_off, c.peer[c.rank] + g.scale_off, quant_slice_start(g, sl, nslices), quant_slice_start(g, sl + 1, nslices));
  {
    const uint32_t s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<true>(c, 2 * s + 1, op)) return;
  }
  const uint32_t me = nslices == 1 ? 0u : (uint32_t)c.rank;
  pull_reduce_range<WireT, OutT, PUSH>(c, g, out_local, out_off, quant_slice_start(g, me, nslices), quant_slice_start(g, me + 1, nslices), scale);
  const uint32_t s = load_seq(c, kSeqBarrier);
  if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;
  if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
}

// ------------------------------------------------------------------------------------------------ host side
template <typename Geom> struct Fp8Call {
  b200collComm* c;
  size_t count;                   // elements of one rank's send buffer
  size_t in_bytes;                // bytes of my send
  size_t out_bytes;               // bytes of my recv
  float scale;                    // ep->scale, times 1/nranks for avg
  Geom g;
};

// The argument rules both families share; `family_check` returns the message of the first family rule the call breaks, or "".
// Every refusal comes before the poisoned-communicator check. On success `call` is filled in except for its geometry.
template <typename Check, typename Geom>
static b200collResult_t fp8_prepare(b200collComm* c, b200collOp_t which, const void* send, const void* recv, size_t count, const b200collEpilogue* ep,
                                    b200collRedOp_t rop, const char* family, Check&& family_check, Fp8Call<Geom>* call) {
  auto refuse = [](const std::string& msg) { set_last_error(msg); return b200collInvalidArgument; };
  if (!c || !send || !recv || !ep) return refuse("null argument");
  if (const std::string e = family_check(); !e.empty()) return refuse(e);
  if (!wide_type(ep->out_dtype)) return refuse(std::string(family) + " collectives: out_dtype must be bf16, fp16 or fp32");
  if (which != b200collOpAllGather && rop != b200collSum && rop != b200collAvg) return refuse(std::string(family) + " reductions take sum or avg only");
  if (count / 16 >= ((size_t)1 << 31)) return refuse(std::string(family) + " collectives: fewer than 2^35 elements per rank");
  if (!aligned(send, 16) || !aligned(recv, 16)) return refuse("send and recv must be 16-byte aligned");
  if (comm_poisoned(c)) return b200collRemoteError;
  call->c = c;
  call->count = count;
  call->in_bytes = count * b200collTypeSize(ep->in_dtype);
  call->out_bytes = (which == b200collOpAllGather ? count * c->nranks : which == b200collOpReduceScatter ? count / c->nranks : count) * b200collTypeSize(ep->out_dtype);
  call->scale = ep->scale * (rop == b200collAvg && which != b200collOpAllGather ? 1.0f / (float)c->nranks : 1.0f);
  return b200collSuccess;
}

// The all-reduce algorithm of both families: the table's pick for an FP8 all-reduce of `count` bytes, or the forced algorithm. The
// Lamport paths and one-shot become the one-shot pull, two-shot and NVLS the two-shot pull + push, which needs recv in the arena (peers
// write into it) and falls back to one-shot otherwise.
static b200collAlgo_t fp8_all_reduce_algo(b200collComm* c, size_t count, const void* recv, size_t out_bytes) {
  const b200collAlgo_t want = c->forced_algo != b200collAlgoAuto ? c->forced_algo : b200collTunerPick(b200collOpAllReduce, count, c->nranks, c->nvls);
  const bool two = (want == b200collAlgoTwoShot || want == b200collAlgoNvls) && b200collIsSymmetric(c, recv, out_bytes);
  return two ? b200collAlgoTwoShot : b200collAlgoOneShot;
}

// the pull-reduce grid: sized to my slice (reduce-scatter, two-shot) or to the whole buffer (one-shot)
static Grid reduce_grid(const b200collComm* c, b200collOp_t which, b200collAlgo_t algo, uint32_t nvec) {
  const uint32_t n = (uint32_t)c->nranks;
  return warp_grid(c, algo == b200collAlgoTwoShot ? nvec / n + 1 : which == b200collOpReduceScatter ? nvec / n : nvec);
}

// ---- block-scaled
using BsqCall = Fp8Call<BsqGeom>;

// Everything the three entry points check before they launch. On success `call` is filled in; count == 0 is left to the caller.
static b200collResult_t bsq_prepare(b200collComm* c, b200collOp_t which, const void* send, void* recv, size_t count, const b200collBlockScale* bs,
                                    const b200collEpilogue* ep, b200collRedOp_t rop, BsqCall* call) {
  b200collResult_t rc = fp8_prepare(c, which, send, recv, count, ep, rop, "block-scaled", [&]() -> std::string {
    if (!bs || !bs->scales) return "null argument";
    if (!is_fp8(ep->in_dtype)) return "block-scaled collectives: in_dtype must be e4m3 or e5m2";
    if (bs->row_len == 0 || bs->row_len % 16 != 0) return "block-scaled collectives: row_len must be a positive multiple of 16";
    if (bs->block_rows < 1 || bs->block_cols < 16 || bs->block_cols % 16 != 0) return "block-scaled collectives: block_rows must be >= 1 and block_cols a positive multiple of 16";
    if (count % bs->row_len != 0) return "block-scaled collectives: the send count must be a multiple of row_len";
    if (which == b200collOpReduceScatter && (count / bs->row_len) % (size_t)c->nranks != 0) return "block-scaled reduce-scatter: the number of rows must be a multiple of nranks";
    if (!aligned(bs->scales, 4)) return "block-scaled collectives: scales must be 4-byte aligned";
    return "";
  }, call);
  if (rc != b200collSuccess || count == 0) return rc;
  const size_t rows = count / bs->row_len, vpr = bs->row_len / 16, vpb = (size_t)bs->block_cols / 16;
  const size_t nbr = (rows + bs->block_rows - 1) / bs->block_rows, ncb = (vpr + vpb - 1) / vpb;
  if (overlaps(send, call->in_bytes, recv, call->out_bytes)) { set_last_error("block-scaled collectives: recv must not overlap send"); return b200collInvalidArgument; }
  // peers read my matrix and scales (there is no staging path for these ops)
  if ((rc = in_arena(c, "block-scaled collectives: ", "send and scales", {{send, count}, {bs->scales, nbr * ncb * 4}})) != b200collSuccess) return rc;
  BsqGeom& g = call->g;
  g.data_off = arena_off(c, send); g.scale_off = arena_off(c, bs->scales);
  g.nvec = (uint32_t)(count / 16); g.ncb = (uint32_t)ncb;
  g.vpr = make_fastdiv((uint32_t)vpr); g.br = make_fastdiv((uint32_t)bs->block_rows); g.vpb = make_fastdiv((uint32_t)vpb);
  return b200collSuccess;
}

static b200collResult_t bsq_copy(const BsqCall& k, const void* send, const b200collBlockScale* bs, void* recv, const b200collEpilogue* ep, cudaStream_t st) {
  b200collComm* c = k.c;
  return with_fp8(ep->in_dtype, [&](auto ti) { return with_wide(ep->out_dtype, [&](auto to) -> b200collResult_t {
    using InT = typename decltype(ti)::type; using OutT = typename decltype(to)::type;
    launch_k(k_bsq_copy<InT, OutT>, copy_blocks(c, k.g.nvec), 256, st, k.g, static_cast<const char*>(send), reinterpret_cast<const char*>(bs->scales),
             static_cast<OutT*>(recv), k.scale);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  }); });
}

static b200collResult_t bsq_reduce(const BsqCall& k, b200collOp_t which, b200collAlgo_t algo, void* recv, const b200collEpilogue* ep, cudaStream_t st) {
  b200collComm* c = k.c;
  const uint32_t n = (uint32_t)c->nranks, me = (uint32_t)c->rank;
  uint32_t v0 = 0, v1 = k.g.nvec;
  if (which == b200collOpReduceScatter || algo == b200collAlgoTwoShot) {
    v0 = (uint32_t)((unsigned long long)k.g.nvec * me / n); v1 = (uint32_t)((unsigned long long)k.g.nvec * (me + 1) / n);
  }
  const Grid gr = reduce_grid(c, which, algo, k.g.nvec);
  return with_fp8(ep->in_dtype, [&](auto ti) { return with_wide(ep->out_dtype, [&](auto to) -> b200collResult_t {
    using InT = typename decltype(ti)::type; using OutT = typename decltype(to)::type;
    if (algo == b200collAlgoTwoShot)
      launch_k(k_bsq_pull_reduce<InT, OutT, true>, gr.blocks, gr.threads, st, c->dev, k.g, static_cast<OutT*>(nullptr), arena_off(c, recv), v0, v1, k.scale, (uint32_t)which);
    else
      launch_k(k_bsq_pull_reduce<InT, OutT, false>, gr.blocks, gr.threads, st, c->dev, k.g, static_cast<OutT*>(recv), (size_t)0, v0, v1, k.scale, (uint32_t)which);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  }); });
}

// ---- quantising
using QuantCall = Fp8Call<QuantGeom>;

// Everything the three entry points check before they touch the scratch or launch; count == 0 is left to the caller.
static b200collResult_t quant_prepare(b200collComm* c, b200collOp_t which, const void* send, void* recv, size_t count, b200collDataType_t wire, int block,
                                      const b200collEpilogue* ep, b200collRedOp_t rop, QuantCall* call) {
  b200collResult_t rc = fp8_prepare(c, which, send, recv, count, ep, rop, "quantised", [&]() -> std::string {
    if (!wide_type(ep->in_dtype)) return "quantised collectives: in_dtype must be bf16, fp16 or fp32";
    if (!is_fp8(wire)) return "quantised collectives: wire_dtype must be e4m3 or e5m2";
    if (quant_lvpb(block) < 0) return std::string("quantised collectives: ") + kBlockRule;
    const bool rs = which == b200collOpReduceScatter;
    if ((rs ? count / (size_t)c->nranks : count) % (size_t)block != 0)
      return rs ? "quantised reduce-scatter: recvcount must be a multiple of block" : "quantised collectives: the count must be a multiple of block";
    return "";
  }, call);
  if (rc != b200collSuccess || count == 0) return rc;
  // in place (all-reduce only): every vector is read and rewritten at the same position, so the element sizes must agree
  const bool in_place = which == b200collOpAllReduce && send == recv && call->in_bytes == call->out_bytes;
  if (!in_place && overlaps(send, call->in_bytes, recv, call->out_bytes)) {
    set_last_error(which == b200collOpAllReduce ? "quantised all-reduce: recv must be send (with in_dtype and out_dtype of one size) or not overlap it"
                                                : "quantised collectives: recv must not overlap send");
    return b200collInvalidArgument;
  }
  QuantGeom& g = call->g;
  g.nvec = (uint32_t)(count / 16);
  g.nblk = (uint32_t)(count / (size_t)block);
  g.lvpb = (uint32_t)quant_lvpb(block);
  return b200collSuccess;
}

// The FP8 copy and its scales of one call, in the symmetric heap. Taken with b200collMemAlloc on first use and grown on demand: a
// collective contract like MemAlloc (every rank makes the same quantised calls in the same order, so every rank gets the same offsets).
// A superseded scratch is never given back before CommDestroy: a CUDA graph captured earlier still addresses it, and must stay valid
// when a later, larger call moves the scratch.
b200collResult_t quant_scratch_take(b200collComm* c, size_t need, const char* who, size_t* off) {
  if (c->quant_scratch_bytes < need) {
    void* p = nullptr;
    size_t bytes = std::max(need, 2 * c->quant_scratch_bytes);
    b200collResult_t rc = b200collMemAlloc(c, &p, bytes);
    if (rc != b200collSuccess && bytes != need) rc = b200collMemAlloc(c, &p, bytes = need);
    if (rc != b200collSuccess) {
      set_last_error(std::string(who) + ": the symmetric arena cannot hold the " + std::to_string(need) + "-byte FP8 scratch (raise B200COLL_ARENA_MB)");
      return rc;
    }
    if (c->quant_scratch) c->quant_scratch_retired.push_back(c->quant_scratch);
    c->quant_scratch = p;
    c->quant_scratch_bytes = bytes;
  }
  *off = arena_off(c, c->quant_scratch);
  return b200collSuccess;
}

// The FP8 copy (count bytes) and its scales (count / block fp32) of one call
static b200collResult_t quant_scratch(b200collComm* c, QuantCall* k) {
  const size_t qbytes = k->count;
  const b200collResult_t rc = quant_scratch_take(c, qbytes + (size_t)k->g.nblk * 4, "quantised collectives", &k->g.data_off);
  k->g.scale_off = k->g.data_off + qbytes;                        // count is a multiple of 16: the scales are 16-byte aligned
  return rc;
}

// nranks == 1: the round trip in registers
static b200collResult_t quant_copy(const QuantCall& k, const void* send, void* recv, b200collDataType_t wire, const b200collEpilogue* ep, cudaStream_t st) {
  b200collComm* c = k.c;
  return with_wide(ep->in_dtype, [&](auto ti) { return with_fp8(wire, [&](auto tw) { return with_wide(ep->out_dtype, [&](auto to) -> b200collResult_t {
    using InT = typename decltype(ti)::type; using WireT = typename decltype(tw)::type; using OutT = typename decltype(to)::type;
    launch_k(k_quant_copy<InT, WireT, OutT>, copy_blocks(c, k.g.nvec), 256, st, static_cast<const char*>(send), static_cast<OutT*>(recv), k.g.nvec, k.g.lvpb, k.scale);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  }); }); });
}

static b200collResult_t quant_reduce(const QuantCall& k, b200collOp_t which, b200collAlgo_t algo, const void* send, void* recv, b200collDataType_t wire,
                                     const b200collEpilogue* ep, cudaStream_t st) {
  b200collComm* c = k.c;
  const uint32_t nslices = (which == b200collOpReduceScatter || algo == b200collAlgoTwoShot) ? (uint32_t)c->nranks : 1u;
  const Grid gr = reduce_grid(c, which, algo, k.g.nvec);
  return with_wide(ep->in_dtype, [&](auto ti) { return with_fp8(wire, [&](auto tw) { return with_wide(ep->out_dtype, [&](auto to) -> b200collResult_t {
    using InT = typename decltype(ti)::type; using WireT = typename decltype(tw)::type; using OutT = typename decltype(to)::type;
    const char* in = static_cast<const char*>(send);
    if (algo == b200collAlgoTwoShot)
      launch_k(k_quant_pull_reduce<InT, WireT, OutT, true>, gr.blocks, gr.threads, st, c->dev, k.g, in, static_cast<OutT*>(nullptr), arena_off(c, recv), nslices, k.scale,
               (uint32_t)which);
    else
      launch_k(k_quant_pull_reduce<InT, WireT, OutT, false>, gr.blocks, gr.threads, st, c->dev, k.g, in, static_cast<OutT*>(recv), (size_t)0, nslices, k.scale,
               (uint32_t)which);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  }); }); });
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
  rc = cross_check(c, b200collOpAllGather, b200collAlgoOneShot, sendcount, k.g.data_off, k.g.scale_off);
  if (rc != b200collSuccess) return rc;
  account(c, b200collOpAllGather, sendcount, b200collAlgoOneShot);
  return with_fp8(ep->in_dtype, [&](auto ti) { return with_wide(ep->out_dtype, [&](auto to) -> b200collResult_t {
    using InT = typename decltype(ti)::type; using OutT = typename decltype(to)::type;
    const Grid gr = warp_grid(c, k.g.nvec);
    launch_k(k_bsq_ag_pull<InT, OutT>, gr.blocks, gr.threads, st, c->dev, k.g, static_cast<OutT*>(recv), k.scale, (uint32_t)b200collOpAllGather);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  }); });
}

b200collResult_t b200collReduceScatterBlockScaled(const void* send, void* recv, size_t recvcount, const b200collBlockScale* bs, const b200collEpilogue* ep,
                                                  b200collRedOp_t op, b200collComm_t c, b200collStream_t stream) {
  if (c && recvcount > SIZE_MAX / B200COLL_MAX_RANKS) { set_last_error("recvcount too large"); return b200collInvalidArgument; }
  BsqCall k;
  b200collResult_t rc = bsq_prepare(c, b200collOpReduceScatter, send, recv, c ? recvcount * c->nranks : 0, bs, ep, op, &k);
  if (rc != b200collSuccess || recvcount == 0) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (c->nranks == 1) { account(c, b200collOpReduceScatter, recvcount, b200collAlgoCopy); return bsq_copy(k, send, bs, recv, ep, st); }
  rc = cross_check(c, b200collOpReduceScatter, b200collAlgoOneShot, recvcount, k.g.data_off, k.g.scale_off);
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
  const b200collAlgo_t algo = fp8_all_reduce_algo(c, count, recv, k.out_bytes);
  rc = cross_check(c, b200collOpAllReduce, algo, count, k.g.data_off, algo == b200collAlgoTwoShot ? arena_off(c, recv) : k.g.scale_off);
  if (rc != b200collSuccess) return rc;
  account(c, b200collOpAllReduce, count, algo);
  return bsq_reduce(k, b200collOpAllReduce, algo, recv, ep, st);
}

b200collResult_t b200collAllGatherQuantized(const void* send, void* recv, size_t sendcount, b200collDataType_t wire_dtype, int block,
                                            const b200collEpilogue* ep, b200collComm_t c, b200collStream_t stream) {
  QuantCall k;
  b200collResult_t rc = quant_prepare(c, b200collOpAllGather, send, recv, sendcount, wire_dtype, block, ep, b200collSum, &k);
  if (rc != b200collSuccess || sendcount == 0) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (c->nranks == 1) { account(c, b200collOpAllGather, k.in_bytes, b200collAlgoCopy); return quant_copy(k, send, recv, wire_dtype, ep, st); }
  if ((rc = quant_scratch(c, &k)) != b200collSuccess) return rc;
  rc = cross_check(c, b200collOpAllGather, b200collAlgoOneShot, sendcount, k.g.data_off, k.g.scale_off);
  if (rc != b200collSuccess) return rc;
  account(c, b200collOpAllGather, k.in_bytes, b200collAlgoOneShot);
  return with_wide(ep->in_dtype, [&](auto ti) { return with_fp8(wire_dtype, [&](auto tw) { return with_wide(ep->out_dtype, [&](auto to) -> b200collResult_t {
    using InT = typename decltype(ti)::type; using WireT = typename decltype(tw)::type; using OutT = typename decltype(to)::type;
    const Grid gr = warp_grid(c, k.g.nvec);
    launch_k(k_quant_ag<InT, WireT, OutT>, gr.blocks, gr.threads, st, c->dev, k.g, static_cast<const char*>(send), static_cast<OutT*>(recv), k.scale,
             (uint32_t)b200collOpAllGather);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  }); }); });
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
  rc = cross_check(c, b200collOpReduceScatter, b200collAlgoOneShot, recvcount, k.g.data_off, k.g.scale_off);
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
  const b200collAlgo_t algo = fp8_all_reduce_algo(c, count, recv, k.out_bytes);
  if ((rc = quant_scratch(c, &k)) != b200collSuccess) return rc;
  rc = cross_check(c, b200collOpAllReduce, algo, count, k.g.data_off, algo == b200collAlgoTwoShot ? arena_off(c, recv) : k.g.scale_off);
  if (rc != b200collSuccess) return rc;
  account(c, b200collOpAllReduce, k.in_bytes, algo);
  return quant_reduce(k, b200collOpAllReduce, algo, send, recv, wire_dtype, ep, st);
}

}  // extern "C"
