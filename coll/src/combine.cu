// libb200coll expert combine: the reverse of the all-to-all-v dispatch with the top-k weighted sum fused, one kernel per call.
//
//   k_combine_pull<InT, OutT, Map>    barrier, pull each token's top_k expert rows from the peers' expert_out, sum in slot order in
//                                     fp32, round once, store locally, barrier
//   k_combine_local<InT, OutT, Map>   one rank: the same gather and sum from a local expert_out, no barrier
//
// Map names the expert_out row of a slot: SegmentMap for b200collAllToAllvCombine, RouteMap for b200collExpertCombine.
//
// The quantising combine (b200collAllToAllvCombineQuantized, b200collExpertCombineQuantized): bf16, fp16 or fp32 expert_out in, FP8 on
// the wire, two kernels per call:
//
//   k_a2av_quant_copy<InT, WireT>            (dispatch.cu) every row of my expert_out quantised by quant.cuh's rule into the quantising
//                                            scratch (blockscaled.cu's quant_scratch_take): FP8 rows, then one fp32 scale per block
//   k_fp8_combine_pull<WireT, OutT, Map>     barrier, pull each slot's FP8 vector and its block's scale from the peer's scratch,
//                                            dequantise (float(q) * s), sum in slot order as above, round once, store locally, barrier
//   k_fp8_combine_local<WireT, OutT, Map>    one rank: the same from the local scratch, no barrier
//
// The quantise pass covers all recv_rows rows, whatever the load: a rank does not know which of its rows its peers will read.
//
// Each rank walks (token, 16-element vector) pairs of its own out. For slot j of token t, index[t, j] is a row of the dispatch send
// buffer; the segment table (A2AvRows, the rows of the dispatch call) maps it to (peer p, row of p's expert_out). A row in no segment
// is a dropped slot. So every load lies inside a destination range [dst_row[p], + rows[p]) of a peer, which the host has checked against
// recv_rows: whatever the device-side index holds, the kernel reads nothing else. b200collExpertCombine reads each slot's (peer, row)
// from the device route that b200collExpertDispatch wrote instead, and any route outside [0, nranks * recv_rows) is a dropped slot.
//
// Per thread, up to kSlots slots are loaded before the first of them is added, so several NVLink (or HBM) reads are in flight; the adds
// then run in slot order, acc = (acc + w_j * y_j) with both roundings kept, so the batching does not change the result.
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "a2av.h"
#include "comm.h"
#include "launch.cuh"
#include "quant.cuh"

namespace b200coll {

constexpr int kCombineThreads = 512;

// The (peer, expert_out row) of dispatch row i, or false when i names no dispatch row. The host refuses overlapping send ranges, so at
// most one segment matches. The one-rank kernel passes nranks = 1, so the loop folds to one compare.
struct SegmentMap {
  A2AvRows g;
  __device__ __forceinline__ bool operator()(int32_t i, int nranks, int* peer, unsigned long long* row) const {
    bool hit = false;
#pragma unroll
    for (int q = 0; q < kMaxRanks; q++) {
      const unsigned long long d = (unsigned long long)((long long)i - (long long)g.src_row[q]);     // negative -> huge -> no match
      if (q < nranks && d < g.rows[q]) { *peer = q; *row = g.dst_row[q] + d; hit = true; }
    }
    return hit;
  }
};

// The (peer, expert_out row) of a route written by b200collExpertDispatch (peer * recv_rows + row), or false for any value outside
// [0, limit), limit = nranks * recv_rows <= 2^31 - 1 (the host checks it): negative values are >= 2^31 as unsigned.
struct RouteMap {
  uint32_t limit, recv_rows;
  __device__ __forceinline__ bool operator()(int32_t i, int, int* peer, unsigned long long* row) const {
    if ((uint32_t)i >= limit) return false;
    const uint32_t p = (uint32_t)i / recv_rows;
    *peer = (int)p;
    *row = (uint32_t)i - p * recv_rows;
    return true;
  }
};

// How a (slot, vector) becomes 16 fp32 values. `vec` is the vector's index in the peer's [recv_rows, vpr] grid of 16-element vectors;
// load() issues the loads of one slot, widen() turns what they returned into fp32.
// Wide: the raw bf16 / fp16 / fp32 words of the peer's expert_out (base(p)), widened exactly: 8 (2-byte types) or 4 (fp32) slots in
// flight per thread, 64 registers of raw data.
template <typename InT, typename Base>
struct WideSlots {
  static constexpr int kSlots = 16 / (int)sizeof(InT);
  struct Raw { uint4 w[sizeof(InT)]; };
  Base base;
  __device__ __forceinline__ void load(Raw& r, int p, unsigned long long vec) const {
    const char* src = base(p) + vec * (16 * sizeof(InT));
#pragma unroll
    for (int k = 0; k < (int)sizeof(InT); k++) r.w[k] = ld_vec(src + 16 * k);
  }
  __device__ __forceinline__ void widen(const Raw& r, float* x) const { widen16<InT>(r.w, x); }
};

// FP8: one 16-byte vector of the peer's FP8 copy (q(p)) and its block's fp32 scale (s(p), one per 2^lvpb vectors; a row is whole
// blocks, so the scale index of row r's vector c is (r * vpr + c) >> lvpb), dequantised by quant.cuh's dequant16: 8 slots in flight,
// 40 registers.
template <typename WireT, typename QBase, typename SBase>
struct Fp8Slots {
  static constexpr int kSlots = 8;
  struct Raw { uint4 q; float s; };
  QBase q;
  SBase s;
  uint32_t lvpb;
  __device__ __forceinline__ void load(Raw& r, int p, unsigned long long vec) const {
    r.q = ld_vec(q(p) + vec * 16);
    r.s = *reinterpret_cast<const float*>(s(p) + (vec >> lvpb) * 4);
  }
  __device__ __forceinline__ void widen(const Raw& r, float* x) const { dequant16<WireT>(r.q, r.s, x); }
};

// Vectors [0, tokens * vpr) of out, vpr = row_elems / 16. map(index value, &peer, &row) names the expert_out row of a slot (false: a
// dropped slot) and src loads and widens a slot's vector. Consecutive threads take consecutive vectors of a row, so the loads of a warp
// are coalesced; lanes of one token read index and weights at one address (a broadcast). 32-bit indices: the host keeps tokens * vpr
// below 2^31, so v + stride cannot wrap.
template <typename OutT, typename Map, typename Src>
__device__ __forceinline__ void combine_range(Map&& map, const Src& src, const int32_t* __restrict__ index, const float* __restrict__ weights,
                                              OutT* __restrict__ out, uint32_t tokens, uint32_t top_k, uint32_t vpr, float scale) {
  constexpr int kSlots = Src::kSlots;
  const uint32_t nvec = tokens * vpr;
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += gridDim.x * blockDim.x) {
    const uint32_t t = v / vpr, col = v - t * vpr;
    const int32_t* it = index + (size_t)t * top_k;
    const float* wt = weights + (size_t)t * top_k;
    float acc[16];
#pragma unroll
    for (int e = 0; e < 16; e++) acc[e] = 0.0f;
    for (uint32_t j0 = 0; j0 < top_k; j0 += kSlots) {
      typename Src::Raw raw[kSlots];
      float w[kSlots];
      bool hit[kSlots];
#pragma unroll
      for (int b = 0; b < kSlots; b++) {
        hit[b] = false;
        w[b] = 1.0f;
        int p = 0;
        unsigned long long row = 0;
        if (j0 + b < top_k && map(it[j0 + b], &p, &row)) {
          hit[b] = true;
          if (weights) w[b] = wt[j0 + b];
          src.load(raw[b], p, row * vpr + col);
        }
      }
#pragma unroll
      for (int b = 0; b < kSlots; b++) {
        if (!hit[b]) continue;
        float x[16];
        src.widen(raw[b], x);
#pragma unroll
        for (int e = 0; e < 16; e++) acc[e] = __fadd_rn(acc[e], __fmul_rn(w[b], x[e]));
      }
    }
    store16_scaled<OutT>(out + (size_t)v * 16, acc, scale);
  }
}

template <typename InT, typename Base> __device__ __forceinline__ WideSlots<InT, Base> wide_slots(Base b) { return {b}; }
template <typename WireT, typename QBase, typename SBase> __device__ __forceinline__ Fp8Slots<WireT, QBase, SBase> fp8_slots(QBase q, SBase s, uint32_t lvpb) {
  return {q, s, lvpb};
}

// Launched on full_grid. The first barrier (relaxed: expert_out was written by earlier kernels on each peer's stream) means every
// peer's expert_out is complete before any CTA pulls, and the closing barrier means no rank's kernel ends before every CTA of every
// peer has finished its pulls, so the caller may overwrite expert_out right after the call on its own stream.
template <typename InT, typename OutT, typename Map>
__global__ void __launch_bounds__(kCombineThreads, 1) k_combine_pull(COMM_PARAM, size_t eo_off, const __grid_constant__ Map m,
                                                                     const int32_t* __restrict__ index, const float* __restrict__ weights,
                                                                     OutT* __restrict__ out, uint32_t tokens, uint32_t top_k, uint32_t vpr,
                                                                     float scale, uint32_t op) {
  pdl_prologue();
  {
    const uint32_t s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;        // every peer's expert_out is written
  }
  combine_range<OutT>([&](int32_t i, int* p, unsigned long long* row) { return m(i, c.nranks, p, row); },
                      wide_slots<InT>([&](int p) -> const char* { return c.peer[p] + eo_off; }), index, weights, out, tokens, top_k, vpr, scale);
  // the sequence number is read again rather than kept live across the loop: only the last block, after the barrier below, bumps it
  const uint32_t s = load_seq(c, kSeqBarrier);
  if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;           // nobody reads my expert_out any more: the caller may overwrite it
  if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
}

// m is a plain parameter here, not __grid_constant__: the compiler then keeps a RouteMap's two fields in registers across the loop.
template <typename InT, typename OutT, typename Map>
__global__ void __launch_bounds__(kCombineThreads, 1) k_combine_local(const Map m, const char* __restrict__ expert_out,
                                                                      const int32_t* __restrict__ index, const float* __restrict__ weights,
                                                                      OutT* __restrict__ out, uint32_t tokens, uint32_t top_k, uint32_t vpr,
                                                                      float scale) {
  pdl_prologue();
  combine_range<OutT>([&](int32_t i, int* p, unsigned long long* row) { return m(i, 1, p, row); },
                      wide_slots<InT>([&](int) { return expert_out; }), index, weights, out, tokens, top_k, vpr, scale);
}

// The quantising combine's pull. Ordering, for rank s and its call k (the scratch is the one quant_scratch_take hands out, shared with
// the quantising collectives):
// - Entry barrier, relaxed. Every peer's scratch holds the FP8 copy of its expert_out once the peer arrives: its quantise pass ran as
//   the previous kernel on the peer's stream and was complete before the peer's pull began, the same argument as for the wide combine's
//   expert_out.
// - My quantise pass may overwrite my scratch: the previous user of the scratch on my stream (a quantising collective or combine) ended
//   with a releasing closing barrier that every peer passes only after its last pull from my scratch, and my quantise pass starts after
//   that kernel has ended. That closing barrier is what makes one scratch safe to share between stream-ordered calls.
// - Closing barrier, releasing: no rank's pull ends before every CTA of every peer has finished pulling from its scratch, so the next
//   call on its stream may overwrite the scratch, and the caller may overwrite expert_out right after the call (only the quantise pass,
//   on its own rank, ever reads expert_out).
// Launched on full_grid, like k_combine_pull: the barriers pair CTA b of every rank.
template <typename WireT, typename OutT, typename Map>
__global__ void __launch_bounds__(kCombineThreads, 1) k_fp8_combine_pull(COMM_PARAM, size_t q_off, size_t s_off, const __grid_constant__ Map m,
                                                                         const int32_t* __restrict__ index, const float* __restrict__ weights,
                                                                         OutT* __restrict__ out, uint32_t tokens, uint32_t top_k, uint32_t vpr,
                                                                         uint32_t lvpb, float scale, uint32_t op) {
  pdl_prologue();
  {
    const uint32_t s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;        // every peer's quantise pass is complete
  }
  combine_range<OutT>([&](int32_t i, int* p, unsigned long long* row) { return m(i, c.nranks, p, row); },
                      fp8_slots<WireT>([&](int p) -> const char* { return c.peer[p] + q_off; }, [&](int p) -> const char* { return c.peer[p] + s_off; }, lvpb),
                      index, weights, out, tokens, top_k, vpr, scale);
  const uint32_t s = load_seq(c, kSeqBarrier);
  if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;           // nobody reads my scratch any more: the next call may overwrite it
  if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
}

// One rank: the same sum from the local scratch (q, scales), no barrier
template <typename WireT, typename OutT, typename Map>
__global__ void __launch_bounds__(kCombineThreads, 1) k_fp8_combine_local(const Map m, const char* __restrict__ q, const char* __restrict__ scales,
                                                                          const int32_t* __restrict__ index, const float* __restrict__ weights,
                                                                          OutT* __restrict__ out, uint32_t tokens, uint32_t top_k, uint32_t vpr,
                                                                          uint32_t lvpb, float scale) {
  pdl_prologue();
  combine_range<OutT>([&](int32_t i, int* p, unsigned long long* row) { return m(i, 1, p, row); },
                      fp8_slots<WireT>([&](int) { return q; }, [&](int) { return scales; }, lvpb), index, weights, out, tokens, top_k, vpr, scale);
}

// ------------------------------------------------------------------------------------------------ host side
// What the quantising combine adds to the wide one: the wire type and the quantising block.
struct CombineQuant {
  b200collDataType_t wire;
  int block;
};

// The argument rules all four combines share, after their null checks ("" or why the call is refused); max_rows bounds recv_rows so
// that every byte offset fits in size_t with room to spare. `index` is the index (the all-to-all-v combines) or the route (the expert
// combines). q == nullptr: a wide combine, whose messages these are; otherwise the quantising combine's rules are added.
static std::string combine_shape(const void* expert_out, const void* out, size_t row_elems, size_t recv_rows, const int32_t* index, const float* weights,
                                 size_t tokens, int top_k, const b200collEpilogue* ep, const char* index_name, const CombineQuant* q, size_t* max_rows) {
  if (!wide_type(ep->in_dtype) || !wide_type(ep->out_dtype)) return "in_dtype and out_dtype must be bf16, fp16 or fp32";
  if (q && !is_fp8(q->wire)) return "wire_dtype must be e4m3 or e5m2";
  if (q && quant_lvpb(q->block) < 0) return kBlockRule;
  if (q ? row_elems == 0 || row_elems % (size_t)q->block != 0 : row_elems == 0 || row_elems % 16 != 0)
    return q ? "row_elems must be a positive multiple of block" : "row_elems must be a positive multiple of 16";
  if (top_k < 1) return "top_k must be at least 1";
  if (!aligned(expert_out, 16) || !aligned(out, 16)) return "expert_out and out must be 16-byte aligned";
  if (!aligned(index, 4) || !aligned(weights, 4)) return std::string(index_name) + " and weights must be 4-byte aligned";
  const size_t max_vecs = ((size_t)1 << 31) - 1;
  if (tokens > max_vecs / (row_elems / 16)) return "at most 2^31 - 1 16-element vectors of out";
  if (tokens > max_vecs / (size_t)top_k) return "tokens * top_k must be at most 2^31 - 1";
  *max_rows = (SIZE_MAX >> 4) / (row_elems * b200collTypeSize(ep->in_dtype));
  if (recv_rows > *max_rows) return "recv_rows * row_elems is too large";
  // the quantise pass walks the 16-element vectors of expert_out with 32-bit indices
  if (q && recv_rows > max_vecs / (row_elems / 16)) return "at most 2^31 - 1 16-element vectors of expert_out (recv_rows * row_elems / 16)";
  return "";
}

// The placement rules all four combines share: out overlapping expert_out, index or weights (InvalidArgument), a poisoned communicator
// (RemoteError), a multi-rank wide expert_out outside the arena (InvalidUsage). The quantising combine's peers read only its scratch,
// so its expert_out may be any device buffer.
static b200collResult_t combine_place(b200collComm* c, const void* expert_out, void* out, size_t row_elems, size_t recv_rows, const int32_t* index,
                                      const float* weights, size_t tokens, int top_k, const b200collEpilogue* ep, const char* what, const char* index_name,
                                      const CombineQuant* q) {
  const size_t is = b200collTypeSize(ep->in_dtype), os = b200collTypeSize(ep->out_dtype);
  const size_t eo_bytes = recv_rows * row_elems * is, out_bytes = tokens * row_elems * os, idx_bytes = tokens * (size_t)top_k * 4;
  if (overlaps(out, out_bytes, expert_out, eo_bytes) || (index && overlaps(out, out_bytes, index, idx_bytes)) ||
      (weights && overlaps(out, out_bytes, weights, idx_bytes))) {
    set_last_error(std::string(what) + ": out must not overlap expert_out, " + index_name + " or weights");
    return b200collInvalidArgument;
  }
  if (comm_poisoned(c)) return b200collRemoteError;
  // peers pull from my expert_out
  if (c->nranks == 1 || q) return b200collSuccess;
  return in_arena(c, std::string(what) + ": ", "expert_out", {{expert_out, eo_bytes}});
}

// The stats of both wide combines, as copy with one rank; with more, oneshot after the B200COLL_CHECK=1 cross-check of recv_rows and the
// expert_out offset.
static b200collResult_t combine_account(b200collComm* c, size_t recv_rows, const void* expert_out, size_t bytes) {
  if (c->nranks == 1) {
    account(c, b200collOpAllToAll, bytes, b200collAlgoCopy);
    return b200collSuccess;
  }
  const b200collResult_t rc = cross_check(c, b200collOpAllToAll, b200collAlgoOneShot, recv_rows, arena_off(c, expert_out), 0);
  if (rc == b200collSuccess) account(c, b200collOpAllToAll, bytes, b200collAlgoOneShot);
  return rc;
}

// Everything the all-to-all-v combines check before they launch (q == nullptr: b200collAllToAllvCombine); on success `g` holds the
// segment table and `in_bytes` the bytes of expert_out the dispatch rows cover.
static b200collResult_t combine_prepare(b200collComm* c, const void* expert_out, void* out, size_t row_elems, size_t recv_rows, const int64_t* send_rows,
                                        const int64_t* send_row_off, const int64_t* recv_row_off_at_peer, const int32_t* index, const float* weights,
                                        size_t tokens, int top_k, const b200collEpilogue* ep, const CombineQuant* q, A2AvRows* g, size_t* in_bytes) {
  const char* what = q ? "quantised all-to-all-v combine" : "all-to-all-v combine";
  auto refuse = [&](const std::string& msg) { set_last_error(std::string(what) + ": " + msg); return b200collInvalidArgument; };
  if (!c || !expert_out || !ep || !send_rows || !send_row_off || !recv_row_off_at_peer || ((!index || !out) && tokens > 0)) return refuse("null argument");
  size_t max_rows = 0;
  const std::string shape = combine_shape(expert_out, out, row_elems, recv_rows, index, weights, tokens, top_k, ep, "index", q, &max_rows);
  if (!shape.empty()) return refuse(shape);
  const size_t is = b200collTypeSize(ep->in_dtype);
  const std::string bad = a2av_rows(c->nranks, send_rows, send_row_off, recv_row_off_at_peer, recv_rows, max_rows, g);
  if (!bad.empty()) return refuse(bad);
  std::vector<std::pair<unsigned long long, unsigned long long>> ranges;     // non-empty send ranges [lo, hi)
  *in_bytes = 0;
  for (int p = 0; p < c->nranks; p++) {
    if (g->rows[p]) ranges.emplace_back(g->src_row[p], g->src_row[p] + g->rows[p]);
    *in_bytes += g->rows[p] * row_elems * is;
  }
  std::sort(ranges.begin(), ranges.end());
  for (size_t k = 1; k < ranges.size(); k++)
    if (ranges[k].first < ranges[k - 1].second) return refuse("two send ranges overlap: a dispatch row must belong to one peer");
  return combine_place(c, expert_out, out, row_elems, recv_rows, index, weights, tokens, top_k, ep, what, "index", q);
}

// Everything the expert combines check before they launch (q == nullptr: b200collExpertCombine).
static b200collResult_t expert_combine_prepare(b200collComm* c, const void* expert_out, void* out, size_t row_elems, size_t recv_rows, const int32_t* route,
                                               const float* weights, size_t tokens, int top_k, const b200collEpilogue* ep, const CombineQuant* q) {
  const char* what = q ? "quantised expert combine" : "expert combine";
  auto refuse = [&](const std::string& msg) { set_last_error(std::string(what) + ": " + msg); return b200collInvalidArgument; };
  if (!c || !expert_out || !ep || ((!route || !out) && tokens > 0)) return refuse("null argument");
  size_t max_rows = 0;
  const std::string shape = combine_shape(expert_out, out, row_elems, recv_rows, route, weights, tokens, top_k, ep, "route", q, &max_rows);
  if (!shape.empty()) return refuse(shape);
  if (recv_rows > (((size_t)1 << 31) - 1) / (size_t)c->nranks) return refuse("nranks * recv_rows must be at most 2^31 - 1 (a route is an int32)");
  return combine_place(c, expert_out, out, row_elems, recv_rows, route, weights, tokens, top_k, ep, what, "route", q);
}

// (in, out) -> one launch of k_combine_pull (more than one rank) or k_combine_local
template <typename Map>
static b200collResult_t combine_launch(b200collComm* c, const Map& m, const void* expert_out, void* out, size_t row_elems, const int32_t* index,
                                       const float* weights, size_t tokens, int top_k, const b200collEpilogue* ep, cudaStream_t st) {
  const uint32_t vpr = (uint32_t)(row_elems / 16), nvec = (uint32_t)(tokens * vpr);
  const bool peers = c->nranks > 1;
  const Grid gr = peers ? full_grid(c, 1)
                        : Grid{(int)std::max<size_t>(1, std::min<size_t>(((size_t)nvec + kCombineThreads - 1) / kCombineThreads, (size_t)std::max(1, c->sm_count))),
                               kCombineThreads};
  return with_wide(ep->in_dtype, [&](auto ti) { return with_wide(ep->out_dtype, [&](auto to) -> b200collResult_t {
    using InT = typename decltype(ti)::type; using OutT = typename decltype(to)::type;
    if (peers)
      launch_k(k_combine_pull<InT, OutT, Map>, gr.blocks, gr.threads, st, c->dev, arena_off(c, expert_out), m, index, weights, static_cast<OutT*>(out),
               (uint32_t)tokens, (uint32_t)top_k, vpr, ep->scale, (uint32_t)b200collOpAllToAll);
    else
      launch_k(k_combine_local<InT, OutT, Map>, gr.blocks, gr.threads, st, m, static_cast<const char*>(expert_out), index, weights, static_cast<OutT*>(out),
               (uint32_t)tokens, (uint32_t)top_k, vpr, ep->scale);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  }); });
}

// Both quantising combines after their checks: the scratch (OutOfMemory before any launch), the B200COLL_CHECK=1 cross-checks, the stats
// (`bytes`, as the matching wide combine counts them), then the quantise pass over all recv_rows rows of expert_out and one launch of
// k_fp8_combine_pull (more than one rank) or k_fp8_combine_local.
template <typename Map>
static b200collResult_t quant_combine_launch(b200collComm* c, const Map& m, const void* expert_out, void* out, size_t row_elems, size_t recv_rows,
                                             const int32_t* index, const float* weights, size_t tokens, int top_k, const b200collEpilogue* ep,
                                             const CombineQuant& q, size_t bytes, const char* what, cudaStream_t st) {
  const DeviceScope on_device(c->device);
  routed_preload(c);
  const size_t qbytes = recv_rows * row_elems;                    // a multiple of 16: the scales are 16-byte aligned
  size_t q_off = 0;
  b200collResult_t rc = recv_rows ? quant_scratch_take(c, qbytes + qbytes / (size_t)q.block * 4, what, &q_off) : b200collSuccess;
  if (rc != b200collSuccess) return rc;
  const size_t s_off = q_off + qbytes;
  const bool peers = c->nranks > 1;
  if (peers) {
    // two exchanges: (recv_rows, both scratch offsets), then (row_elems, block and wire)
    if ((rc = cross_check(c, b200collOpAllToAll, b200collAlgoOneShot, recv_rows, q_off, s_off)) != b200collSuccess) return rc;
    rc = cross_check(c, b200collOpAllToAll, b200collAlgoOneShot, row_elems, (size_t)q.block, (size_t)q.wire);
    if (rc != b200collSuccess) return rc;
  }
  account(c, b200collOpAllToAll, bytes, peers ? b200collAlgoOneShot : b200collAlgoCopy);
  char* scratch = reinterpret_cast<char*>(c->peer_va[c->rank]);
  const uint32_t lvpb = (uint32_t)quant_lvpb(q.block), vpr = (uint32_t)(row_elems / 16), nvec = (uint32_t)(tokens * vpr);
  if ((rc = launch_quant_copy(c, ep->in_dtype, q.wire, expert_out, scratch + q_off, scratch + s_off, (uint32_t)(qbytes / 16), lvpb, st)) != b200collSuccess)
    return rc;
  const Grid gr = peers ? full_grid(c, 1)
                        : Grid{(int)std::max<size_t>(1, std::min<size_t>(((size_t)nvec + kCombineThreads - 1) / kCombineThreads, (size_t)std::max(1, c->sm_count))),
                               kCombineThreads};
  return with_fp8(q.wire, [&](auto tw) { return with_wide(ep->out_dtype, [&](auto to) -> b200collResult_t {
    using WireT = typename decltype(tw)::type; using OutT = typename decltype(to)::type;
    if (peers)
      launch_k(k_fp8_combine_pull<WireT, OutT, Map>, gr.blocks, gr.threads, st, c->dev, q_off, s_off, m, index, weights, static_cast<OutT*>(out),
               (uint32_t)tokens, (uint32_t)top_k, vpr, lvpb, ep->scale, (uint32_t)b200collOpAllToAll);
    else
      launch_k(k_fp8_combine_local<WireT, OutT, Map>, gr.blocks, gr.threads, st, m, static_cast<const char*>(scratch + q_off),
               static_cast<const char*>(scratch + s_off), index, weights, static_cast<OutT*>(out), (uint32_t)tokens, (uint32_t)top_k, vpr, lvpb, ep->scale);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  }); });
}

template <typename Map> static void preload_map() {
  cudaFuncAttributes fa;
  for (b200collDataType_t out : {b200collBfloat16, b200collFloat16, b200collFloat32})
    with_wide(out, [&](auto to) {
      using OutT = typename decltype(to)::type;
      for (b200collDataType_t in : {b200collBfloat16, b200collFloat16, b200collFloat32})
        with_wide(in, [&](auto ti) {
          using InT = typename decltype(ti)::type;
          cudaFuncGetAttributes(&fa, k_combine_pull<InT, OutT, Map>);
          cudaFuncGetAttributes(&fa, k_combine_local<InT, OutT, Map>);
        });
      for (b200collDataType_t wire : {b200collFloat8e4m3, b200collFloat8e5m2})
        with_fp8(wire, [&](auto tw) {
          using WireT = typename decltype(tw)::type;
          cudaFuncGetAttributes(&fa, k_fp8_combine_pull<WireT, OutT, Map>);
          cudaFuncGetAttributes(&fa, k_fp8_combine_local<WireT, OutT, Map>);
        });
    });
}

void combine_preload() {
  preload_map<SegmentMap>();
  preload_map<RouteMap>();
}

}  // namespace b200coll

using namespace b200coll;

extern "C" {

b200collResult_t b200collAllToAllvCombine(const void* expert_out, void* out, size_t row_elems, size_t recv_rows,
                                          const int64_t* send_rows, const int64_t* send_row_off, const int64_t* recv_row_off_at_peer,
                                          const int32_t* index, const float* weights, size_t tokens, int top_k,
                                          const b200collEpilogue* ep, b200collComm_t c, b200collStream_t stream) {
  A2AvRows g;
  size_t in_bytes = 0;
  b200collResult_t rc = combine_prepare(c, expert_out, out, row_elems, recv_rows, send_rows, send_row_off, recv_row_off_at_peer, index, weights, tokens,
                                        top_k, ep, nullptr, &g, &in_bytes);
  if (rc != b200collSuccess) return rc;
  if ((rc = combine_account(c, recv_rows, expert_out, in_bytes)) != b200collSuccess) return rc;
  return combine_launch(c, SegmentMap{g}, expert_out, out, row_elems, index, weights, tokens, top_k, ep, static_cast<cudaStream_t>(stream));
}

b200collResult_t b200collExpertCombine(const void* expert_out, void* out, size_t row_elems, size_t recv_rows, const int32_t* route,
                                       const float* weights, size_t tokens, int top_k, const b200collEpilogue* ep, b200collComm_t c,
                                       b200collStream_t stream) {
  b200collResult_t rc = expert_combine_prepare(c, expert_out, out, row_elems, recv_rows, route, weights, tokens, top_k, ep, nullptr);
  if (rc != b200collSuccess) return rc;
  if ((rc = combine_account(c, recv_rows, expert_out, tokens * (size_t)top_k * row_elems * b200collTypeSize(ep->in_dtype))) != b200collSuccess) return rc;
  const DeviceScope on_device(c->device);
  const RouteMap m{(uint32_t)(c->nranks * recv_rows), (uint32_t)recv_rows};
  return combine_launch(c, m, expert_out, out, row_elems, route, weights, tokens, top_k, ep, static_cast<cudaStream_t>(stream));
}

b200collResult_t b200collAllToAllvCombineQuantized(const void* expert_out, void* out, size_t row_elems, size_t recv_rows,
                                                   const int64_t* send_rows, const int64_t* send_row_off, const int64_t* recv_row_off_at_peer,
                                                   const int32_t* index, const float* weights, size_t tokens, int top_k,
                                                   b200collDataType_t wire_dtype, int block, const b200collEpilogue* ep, b200collComm_t c,
                                                   b200collStream_t stream) {
  const CombineQuant q{wire_dtype, block};
  A2AvRows g;
  size_t in_bytes = 0;
  const b200collResult_t rc = combine_prepare(c, expert_out, out, row_elems, recv_rows, send_rows, send_row_off, recv_row_off_at_peer, index, weights,
                                              tokens, top_k, ep, &q, &g, &in_bytes);
  if (rc != b200collSuccess) return rc;
  return quant_combine_launch(c, SegmentMap{g}, expert_out, out, row_elems, recv_rows, index, weights, tokens, top_k, ep, q, in_bytes,
                              "quantised all-to-all-v combine", static_cast<cudaStream_t>(stream));
}

b200collResult_t b200collExpertCombineQuantized(const void* expert_out, void* out, size_t row_elems, size_t recv_rows, const int32_t* route,
                                                const float* weights, size_t tokens, int top_k, b200collDataType_t wire_dtype, int block,
                                                const b200collEpilogue* ep, b200collComm_t c, b200collStream_t stream) {
  const CombineQuant q{wire_dtype, block};
  const b200collResult_t rc = expert_combine_prepare(c, expert_out, out, row_elems, recv_rows, route, weights, tokens, top_k, ep, &q);
  if (rc != b200collSuccess) return rc;
  const RouteMap m{(uint32_t)(c->nranks * recv_rows), (uint32_t)recv_rows};
  return quant_combine_launch(c, m, expert_out, out, row_elems, recv_rows, route, weights, tokens, top_k, ep, q,
                              tokens * (size_t)top_k * row_elems * b200collTypeSize(ep->in_dtype), "quantised expert combine",
                              static_cast<cudaStream_t>(stream));
}

}  // extern "C"
