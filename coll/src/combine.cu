// libb200coll expert combine: the reverse of the all-to-all-v dispatch with the top-k weighted sum fused, one kernel per call.
//
//   k_combine_pull<InT, OutT, Map>    barrier, pull each token's top_k expert rows from the peers' expert_out, sum in slot order in
//                                     fp32, round once, store locally, barrier
//   k_combine_local<InT, OutT, Map>   one rank: the same gather and sum from a local expert_out, no barrier
//
// Map names the expert_out row of a slot: SegmentMap for b200collAllToAllvCombine, RouteMap for b200collExpertCombine.
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

// Vectors [0, tokens * vpr) of out, vpr = row_elems / 16. map(index value, &peer, &row) names the expert_out row of a slot (false: a
// dropped slot) and base(p) is the address of peer p's expert_out. Consecutive threads take consecutive vectors of a row, so the loads
// of a warp are coalesced; lanes of one token read index and weights at one address (a broadcast). 32-bit indices: the host keeps
// tokens * vpr below 2^31, so v + stride cannot wrap.
template <typename InT, typename OutT, typename Map, typename Base>
__device__ __forceinline__ void combine_range(Map&& map, Base&& base, const int32_t* __restrict__ index,
                                              const float* __restrict__ weights, OutT* __restrict__ out, uint32_t tokens, uint32_t top_k,
                                              uint32_t vpr, float scale) {
  constexpr int NW = (int)sizeof(InT);                           // 16-byte words per 16 elements: 2 (bf16, fp16) or 4 (fp32)
  constexpr int kSlots = 16 / (int)sizeof(InT);                  // slots in flight per thread: 8 or 4, 64 registers of raw data
  const uint32_t nvec = tokens * vpr;
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += gridDim.x * blockDim.x) {
    const uint32_t t = v / vpr, col = v - t * vpr;
    const int32_t* it = index + (size_t)t * top_k;
    const float* wt = weights + (size_t)t * top_k;
    float acc[16];
#pragma unroll
    for (int e = 0; e < 16; e++) acc[e] = 0.0f;
    for (uint32_t j0 = 0; j0 < top_k; j0 += kSlots) {
      uint4 raw[kSlots][NW];
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
          const char* src = base(p) + (row * vpr + col) * (16 * sizeof(InT));
#pragma unroll
          for (int k = 0; k < NW; k++) raw[b][k] = ld_vec(src + 16 * k);
        }
      }
#pragma unroll
      for (int b = 0; b < kSlots; b++) {
        if (!hit[b]) continue;
        float x[16];
        widen16<InT>(raw[b], x);
#pragma unroll
        for (int e = 0; e < 16; e++) acc[e] = __fadd_rn(acc[e], __fmul_rn(w[b], x[e]));
      }
    }
    store16_scaled<OutT>(out + (size_t)v * 16, acc, scale);
  }
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
  combine_range<InT, OutT>([&](int32_t i, int* p, unsigned long long* row) { return m(i, c.nranks, p, row); },
                           [&](int p) -> const char* { return c.peer[p] + eo_off; }, index, weights, out, tokens, top_k, vpr, scale);
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
  combine_range<InT, OutT>([&](int32_t i, int* p, unsigned long long* row) { return m(i, 1, p, row); },
                           [&](int) { return expert_out; }, index, weights, out, tokens, top_k, vpr, scale);
}

// ------------------------------------------------------------------------------------------------ host side
// The argument rules both combines share, after their null checks ("" or why the call is refused); max_rows bounds recv_rows so that
// every byte offset fits in size_t with room to spare. `index` is the index (b200collAllToAllvCombine) or the route (b200collExpertCombine).
static std::string combine_shape(const void* expert_out, const void* out, size_t row_elems, size_t recv_rows, const int32_t* index, const float* weights,
                                 size_t tokens, int top_k, const b200collEpilogue* ep, const char* index_name, size_t* max_rows) {
  if (!wide_type(ep->in_dtype) || !wide_type(ep->out_dtype)) return "in_dtype and out_dtype must be bf16, fp16 or fp32";
  if (row_elems == 0 || row_elems % 16 != 0) return "row_elems must be a positive multiple of 16";
  if (top_k < 1) return "top_k must be at least 1";
  if (!aligned(expert_out, 16) || !aligned(out, 16)) return "expert_out and out must be 16-byte aligned";
  if (!aligned(index, 4) || !aligned(weights, 4)) return std::string(index_name) + " and weights must be 4-byte aligned";
  const size_t max_vecs = ((size_t)1 << 31) - 1;
  if (tokens > max_vecs / (row_elems / 16)) return "at most 2^31 - 1 16-element vectors of out";
  if (tokens > max_vecs / (size_t)top_k) return "tokens * top_k must be at most 2^31 - 1";
  *max_rows = (SIZE_MAX >> 4) / (row_elems * b200collTypeSize(ep->in_dtype));
  if (recv_rows > *max_rows) return "recv_rows * row_elems is too large";
  return "";
}

// The placement rules both combines share: out overlapping expert_out, index or weights (InvalidArgument), a poisoned communicator
// (RemoteError), a multi-rank expert_out outside the arena (InvalidUsage).
static b200collResult_t combine_place(b200collComm* c, const void* expert_out, void* out, size_t row_elems, size_t recv_rows, const int32_t* index,
                                      const float* weights, size_t tokens, int top_k, const b200collEpilogue* ep, const char* what, const char* index_name) {
  const size_t is = b200collTypeSize(ep->in_dtype), os = b200collTypeSize(ep->out_dtype);
  const size_t eo_bytes = recv_rows * row_elems * is, out_bytes = tokens * row_elems * os, idx_bytes = tokens * (size_t)top_k * 4;
  if (overlaps(out, out_bytes, expert_out, eo_bytes) || (index && overlaps(out, out_bytes, index, idx_bytes)) ||
      (weights && overlaps(out, out_bytes, weights, idx_bytes))) {
    set_last_error(std::string(what) + ": out must not overlap expert_out, " + index_name + " or weights");
    return b200collInvalidArgument;
  }
  if (comm_poisoned(c)) return b200collRemoteError;
  // peers pull from my expert_out
  if (c->nranks == 1) return b200collSuccess;
  return in_arena(c, std::string(what) + ": ", "expert_out", {{expert_out, eo_bytes}});
}

// The stats of both combines, as copy with one rank; with more, oneshot after the B200COLL_CHECK=1 cross-check of recv_rows and the
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

// Everything b200collAllToAllvCombine checks before it launches; on success `g` holds the segment table and `in_bytes` the bytes of
// expert_out the dispatch rows cover.
static b200collResult_t combine_prepare(b200collComm* c, const void* expert_out, void* out, size_t row_elems, size_t recv_rows, const int64_t* send_rows,
                                        const int64_t* send_row_off, const int64_t* recv_row_off_at_peer, const int32_t* index, const float* weights,
                                        size_t tokens, int top_k, const b200collEpilogue* ep, A2AvRows* g, size_t* in_bytes) {
  auto refuse = [](const std::string& msg) { set_last_error("all-to-all-v combine: " + msg); return b200collInvalidArgument; };
  if (!c || !expert_out || !ep || !send_rows || !send_row_off || !recv_row_off_at_peer || ((!index || !out) && tokens > 0)) return refuse("null argument");
  size_t max_rows = 0;
  const std::string shape = combine_shape(expert_out, out, row_elems, recv_rows, index, weights, tokens, top_k, ep, "index", &max_rows);
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
  return combine_place(c, expert_out, out, row_elems, recv_rows, index, weights, tokens, top_k, ep, "all-to-all-v combine", "index");
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
                                        top_k, ep, &g, &in_bytes);
  if (rc != b200collSuccess) return rc;
  if ((rc = combine_account(c, recv_rows, expert_out, in_bytes)) != b200collSuccess) return rc;
  return combine_launch(c, SegmentMap{g}, expert_out, out, row_elems, index, weights, tokens, top_k, ep, static_cast<cudaStream_t>(stream));
}

b200collResult_t b200collExpertCombine(const void* expert_out, void* out, size_t row_elems, size_t recv_rows, const int32_t* route,
                                       const float* weights, size_t tokens, int top_k, const b200collEpilogue* ep, b200collComm_t c,
                                       b200collStream_t stream) {
  auto refuse = [](const std::string& msg) { set_last_error("expert combine: " + msg); return b200collInvalidArgument; };
  if (!c || !expert_out || !ep || ((!route || !out) && tokens > 0)) return refuse("null argument");
  size_t max_rows = 0;
  const std::string shape = combine_shape(expert_out, out, row_elems, recv_rows, route, weights, tokens, top_k, ep, "route", &max_rows);
  if (!shape.empty()) return refuse(shape);
  if (recv_rows > (((size_t)1 << 31) - 1) / (size_t)c->nranks) return refuse("nranks * recv_rows must be at most 2^31 - 1 (a route is an int32)");
  b200collResult_t rc = combine_place(c, expert_out, out, row_elems, recv_rows, route, weights, tokens, top_k, ep, "expert combine", "route");
  if (rc != b200collSuccess) return rc;
  if ((rc = combine_account(c, recv_rows, expert_out, tokens * (size_t)top_k * row_elems * b200collTypeSize(ep->in_dtype))) != b200collSuccess) return rc;
  const DeviceScope on_device(c->device);
  const RouteMap m{(uint32_t)(c->nranks * recv_rows), (uint32_t)recv_rows};
  return combine_launch(c, m, expert_out, out, row_elems, route, weights, tokens, top_k, ep, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
