// libb200coll expert dispatch: the three calls that move each token's rows to the ranks that own its experts.
//
// Quantising all-to-all-v (b200collAllToAllvQuantized): bf16, fp16 or fp32 rows in, FP8 rows and their per-row block scales out, host
// row counts, one kernel:
//
//   k_a2av_quant_push<InT, WireT>   barrier, quantise my rows for every peer and push FP8 and scales into its recv, barrier (releases)
//   k_a2av_quant_copy<InT, WireT>   one rank: a local quantising copy, no barrier; also the quantising combine's quantise pass
//
// Device-routed (b200collExpertDispatch, b200collExpertDispatchQuantized): the router's top-k expert ids in, rows grouped by expert out,
// no host sync. Two kernels per call:
//
//   k_routed_layout                      one CTA: each slot's rank among this rank's slots to the same expert, the per-expert counts,
//                                        the count exchange through the mailbox (layout.h, kOffRouteCounts) and one releasing barrier,
//                                        then every slot's route
//   k_routed_push<P>                     every (slot, 16-byte vector) pair with a route is copied to its row of the owner's recv; P: over
//                                        NVLink into the peers' arenas, closing releasing barrier; !P (one rank): into a local buffer,
//                                        no barrier
//   k_expert_quant_push<InT, WireT, P>   the FP8 call's push, in place of k_routed_push: quantise each token's row once, store FP8 and
//                                        scales to every routed row of the owners' recv and recv_scales, with the same barriers
//
// The quantisers are quant.cuh's, as in the quantising collectives. The ordering argument below covers k_expert_quant_push word for
// word, with "recv" read as "recv and recv_scales".
//
// Layout. The slots [0, tokens * top_k) are cut into 32 contiguous segments, one per warp of the layout CTA. A warp walks its segment
// 32 slots at a time: __match_any_sync groups the lanes that name one expert, a lane's rank in the group is the popcount of the lower
// lanes in it, and the group's lowest lane adds the group's size to the warp's running count of that expert in shared memory. So a slot's
// rank is the number of earlier slots of its segment with the same expert; a prefix over the warps' counts (segment order is slot order)
// makes it the rank among all of this rank's slots. No atomic hands out a position: the layout is the same on every run.
//
// Ordering argument (rank s, call k; "A" is the layout kernel's barrier, "B" the push kernel's closing barrier; both release, and CTA b
// of every rank meets CTA b of every other rank in them):
// - A peer's mailbox row [s] is free when s writes it in call k: the peer read its mailbox in its layout kernel of call k - 1, which
//   ended before its push kernel of call k - 1 began, and s only starts call k after passing B of call k - 1, which waits for every peer
//   to arrive there. Collectives between the two calls only add barriers (or none: LL takes no barrier and uses no mailbox).
// - A peer's recv is free when s pushes into it in call k: s passed A of call k first, and a peer arrives at A only once its own stream
//   has reached call k, so everything the peer's stream did before (an expert GEMM reading recv) is complete. That is why the push kernel
//   takes no entry barrier: A, one kernel earlier on the same stream, already orders it. Receivers see the rows after their push kernel
//   ends because of B (released by every sender after its stores).
// - Sender and receiver agree on every row: both compute it from the same [nranks][E] count matrix, read after A, and the same rule.
// - The grids cannot differ between ranks: the layout kernel is one CTA everywhere, and the push kernel is launched on full_grid.
// - Graph replay: both kernels read the epoch from the communicator's state word (load_seq) and bump it once, the counts travel in
//   device memory, and the host passes only shapes and pointers: nothing about the epoch or the routing lives in kernel arguments.
#include <stdint.h>

#include <algorithm>
#include <atomic>
#include <mutex>
#include <string>

#include "a2av.h"
#include "comm.h"
#include "launch.cuh"
#include "quant.cuh"

namespace b200coll {

constexpr int kLayoutThreads = 1024, kLayoutWarps = kLayoutThreads / 32;
constexpr int kRoutedPushThreads = 512, kRoutedPushUnroll = 4;

// Shared memory of k_routed_layout: int32 counts [warp][E], int64 bases [E], int64 warp sums [kLayoutWarps + 1].
constexpr size_t layout_smem(int E) { return (size_t)kLayoutWarps * E * 4 + (size_t)E * 8 + (kLayoutWarps + 1) * 8; }

__global__ void __launch_bounds__(kLayoutThreads, 1) k_routed_layout(COMM_PARAM, const int32_t* __restrict__ topk_idx, uint32_t slots, int E,
                                                                     uint32_t recv_rows, int32_t* __restrict__ route, int32_t* __restrict__ expert_counts,
                                                                     int32_t* __restrict__ dropped, uint32_t op) {
  pdl_prologue();
  extern __shared__ __align__(16) unsigned char smem[];
  int* cnt = reinterpret_cast<int*>(smem);
  long long* base = reinterpret_cast<long long*>(smem + (size_t)kLayoutWarps * E * 4);
  long long* wsum = base + E;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const uint32_t per = (slots + kLayoutWarps - 1) / kLayoutWarps;
  const uint32_t lo = min(slots, (uint32_t)w * per), hi = min(slots, lo + per);
  for (int i = threadIdx.x; i < kLayoutWarps * E; i += blockDim.x) cnt[i] = 0;
  __syncthreads();

  // 1. each slot's rank within its warp's segment, kept in route until step 4
  int* mine = cnt + w * E;
  for (uint32_t b = lo; b < hi; b += 32) {
    const uint32_t i = b + lane;
    int e = -1;
    if (i < hi) { const int32_t id = topk_idx[i]; if ((uint32_t)id < (uint32_t)E) e = id; }
    const unsigned same = __match_any_sync(0xFFFFFFFFu, e);
    const int lower = __popc(same & ((1u << lane) - 1u));
    const int r = e >= 0 ? mine[e] + lower : 0;
    __syncwarp();
    if (e >= 0 && lower == 0) mine[e] += __popc(same);
    __syncwarp();
    if (i < hi) route[i] = r;
  }
  __syncthreads();

  // 2. per expert: the exclusive prefix of the warps' counts, and this rank's count of it
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    int run = 0;
    for (int v = 0; v < kLayoutWarps; v++) { const int x = cnt[v * E + e]; cnt[v * E + e] = run; run += x; }
    base[e] = run;
  }
  __syncthreads();

  // 3. the exchange: my counts into row [my rank] of every rank's mailbox, one releasing barrier, then the whole matrix. E <= blockDim:
  // thread e owns expert e from here on.
  const int e = threadIdx.x;
  const bool exchange = c.nranks > 1;
  const uint32_t s = load_seq(c, kSeqBarrier);
  if (exchange) {
    if (e < E)
      for (int p = 0; p < c.nranks; p++) reinterpret_cast<int*>(c.peer[p] + kOffRouteCounts)[c.rank * kRouteMaxExperts + e] = (int)base[e];
    if (!barrier_blocks<true>(c, 2 * s + 1, op)) {               // watchdog: route no row, so the push kernel moves nothing
      for (uint32_t i = threadIdx.x; i < slots; i += blockDim.x) route[i] = -1;
      return;
    }
  }
  long long total = 0, before_me = 0;                            // rows of expert e over all ranks, and from ranks below mine
  if (e < E) {
    if (exchange) {
      const uint32_t* box = reinterpret_cast<const uint32_t*>(c.peer[c.rank] + kOffRouteCounts) + e;
      for (int q = 0; q < c.nranks; q++) {
        const long long m = (int)ld_relaxed_sys(box + (size_t)q * kRouteMaxExperts);
        total += m;
        if (q < c.rank) before_me += m;
      }
    } else {
      total = base[e];
    }
  }
  // exclusive prefix of total over the experts: a warp scan, then the warps' sums
  long long x = total;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const long long y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= d) x += y; }
  if (lane == 31) wsum[w] = x;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long run = 0;
    for (int v = 0; v < kLayoutWarps; v++) { const long long t = wsum[v]; wsum[v] = run; run += t; }
    wsum[kLayoutWarps] = 0;                                      // the dropped rows, summed below
  }
  __syncthreads();
  const long long below = x - total + wsum[w];                   // rows of all experts below e
  if (e < E) base[e] = below;
  __syncthreads();
  const int epr = E / c.nranks;
  long long first = 0;                                           // base_d(e): rows of the owner's experts below e
  if (e < E) first = below - base[e / epr * epr];
  __syncthreads();
  if (e < E) {
    base[e] = first + before_me;                                 // my first row for expert e in its owner's recv
    if (e / epr == c.rank) {
      const long long stored = min(max((long long)recv_rows - first, 0ll), total);
      expert_counts[e - c.rank * epr] = (int32_t)stored;
      if (total > stored) atomicAdd(reinterpret_cast<unsigned long long*>(&wsum[kLayoutWarps]), (unsigned long long)(total - stored));
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) *dropped = (int32_t)min(wsum[kLayoutWarps], (long long)INT32_MAX);

  // 4. every slot's route: its owner and row, or -1 when the id is invalid or the row falls at or past recv_rows
  for (uint32_t i = lo + lane; i < hi; i += 32) {
    const int32_t id = topk_idx[i];
    int32_t r = -1;
    if ((uint32_t)id < (uint32_t)E) {
      const long long row = base[id] + mine[id] + route[i];
      if (row < (long long)recv_rows) r = (int32_t)((long long)(id / epr) * recv_rows + row);
    }
    route[i] = r;
  }
  if (exchange && threadIdx.x == 0) c.state[kSeqBarrier] = s + 1;   // one CTA: every thread read s before the barrier
}

// Vectors [0, nvec) = (slot, 16-byte vector of its row), vpr vectors per row. A slot's route names (peer, row) or is outside
// [0, nranks * recv_rows) and moves nothing. The host keeps nvec and nranks * recv_rows below 2^31, so 32-bit indices cannot wrap.
template <bool kPeers>
__global__ void __launch_bounds__(kRoutedPushThreads) k_routed_push(COMM_PARAM, const char* __restrict__ x, char* __restrict__ recv, size_t recv_off,
                                                                    const int32_t* __restrict__ route, uint32_t top_k, uint32_t vpr, uint32_t nvec,
                                                                    uint32_t recv_rows, uint32_t op) {
  pdl_prologue();
  constexpr int U = kRoutedPushUnroll;
  const uint32_t limit = (uint32_t)c.nranks * recv_rows;
  for (uint32_t b = blockIdx.x * blockDim.x * U + threadIdx.x; b < nvec; b += gridDim.x * blockDim.x * U) {
    uint4 d[U];
    char* dst[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const uint32_t v = b + u * blockDim.x;
      dst[u] = nullptr;
      if (v < nvec) {
        const uint32_t slot = v / vpr, col = v - slot * vpr;
        const uint32_t r = (uint32_t)route[slot];
        if (r < limit) {
          const uint32_t p = r / recv_rows, row = r - p * recv_rows;
          dst[u] = (kPeers ? c.peer[p] + recv_off : recv) + ((size_t)row * vpr + col) * 16;
          d[u] = ld_vec(x + ((size_t)(slot / top_k) * vpr + col) * 16);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++)
      if (dst[u]) st_vec(dst[u], d[u]);
  }
  if constexpr (kPeers) {
    const uint32_t s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<true>(c, 2 * s + 1, op)) return;         // my rows are in every receiver's recv before its kernel ends
    if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
  }
}

// Quantising all-to-all-v. A2AvArgs counts 16-element vectors here: src_vec[p] of my send, dst_vec[p] of peer p's recv (FP8, 16 bytes
// per vector), and the prefix over the staggered peer order. The scale of destination vector d is fp32 element d >> lvpb of the peer's
// recv_scales. Blocks never straddle a warp or a peer's segment: every prefix entry and every destination offset is whole rows, a row is
// whole blocks, and a block is a power of two of at most 32 vectors. So warp_walk's 32-aligned warps hold whole blocks of one segment
// (a block's lanes are one aligned lane group, all active or all idle), and quant_vec's butterfly sees exactly the block's lanes.
template <typename InT, typename WireT>
__global__ void __launch_bounds__(kBsqThreads) k_a2av_quant_push(COMM_PARAM, const char* __restrict__ in, size_t q_off, size_t s_off,
                                                                 const __grid_constant__ A2AvArgs a, uint32_t lvpb, uint32_t op) {
  pdl_prologue();
  const uint32_t s = load_seq(c, kSeqBarrier);
  if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;          // every peer has entered the call: its recv is free to overwrite
  const uint32_t lane = threadIdx.x & 31, gl = 1u << lvpb;
  warp_walk(0, (uint32_t)a.prefix[c.nranks], [&](uint32_t v, bool act) {
    int p = 0;
    uint32_t lv = 0;
    float x[16] = {};
    if (act) {
      int j = 0;
#pragma unroll
      for (int q = 1; q < kMaxRanks; q++) if (q < c.nranks && v >= a.prefix[q]) j = q;
      p = c.rank + 1 + j; if (p >= c.nranks) p -= c.nranks;
      lv = v - (uint32_t)a.prefix[j];
      quant_load16<InT>(in + (a.src_vec[p] + lv) * (16 * sizeof(InT)), x);
    }
    float sc;
    const uint4 w = quant_vec<WireT>(x, gl, &sc);
    if (act) {
      const unsigned long long d = a.dst_vec[p] + lv;
      st_vec(c.peer[p] + q_off + d * 16, w);
      if ((lane & (gl - 1)) == 0) *reinterpret_cast<float*>(c.peer[p] + s_off + (d >> lvpb) * 4) = sc;
    }
  });
  if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;           // releases my stores to their receivers
  if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
}

// One rank: vectors [0, g.nvec) of in quantised into q and scales (all three already offset to the first row), no barrier
template <typename InT, typename WireT>
__global__ void __launch_bounds__(kBsqThreads) k_a2av_quant_copy(const __grid_constant__ QuantGeom g, const char* __restrict__ in, char* __restrict__ q,
                                                                 char* __restrict__ scales) {
  pdl_prologue();
  quant_range<InT, WireT>(g, in, q, scales, 0, g.nvec);
}

// Routed FP8 dispatch (b200collExpertDispatchQuantized launches k_routed_layout before it on the same stream). Vectors
// [0, nvec) of x are (token, 16-element vector of its row), vpr vectors per row. Each is loaded, widened and quantised once, then stored
// to every stored slot of its token: the FP8 vector to row `row` of the owner's recv, and the block's scale, by the block's lowest lane,
// to the same row of the owner's recv_scales. A route outside [0, nranks * recv_rows) stores nothing, so a token's slots all get the
// same bytes and scales. quant_vec's butterfly sees exactly one block's lanes: a row is whole blocks, a token's first vector t * vpr is a
// multiple of the vectors per block, and a block is a power of two of at most 32 vectors; so with warp_walk's 32-aligned warps a block's
// lanes are one aligned lane group of one warp, all active or all idle (and, being one token's, they read the same routes).
// kPeers: stores into the owners' arenas at q_off / s_off. No entry barrier: layout barrier A, one kernel earlier on this stream, already
// freed every peer's recv and recv_scales (the ordering argument above, as for k_routed_push); one closing releasing barrier.
// !kPeers (one rank): stores into recv and scales, no barrier.
template <typename InT, typename WireT, bool kPeers>
__global__ void __launch_bounds__(kBsqThreads) k_expert_quant_push(COMM_PARAM, const char* __restrict__ x, char* __restrict__ recv, char* __restrict__ scales,
                                                                   size_t q_off, size_t s_off, const int32_t* __restrict__ route, uint32_t top_k,
                                                                   uint32_t vpr, uint32_t nvec, uint32_t recv_rows, uint32_t lvpb, uint32_t op) {
  pdl_prologue();
  const uint32_t lane = threadIdx.x & 31, gl = 1u << lvpb, limit = (uint32_t)c.nranks * recv_rows;
  warp_walk(0, nvec, [&](uint32_t v, bool act) {
    float xv[16] = {};
    if (act) quant_load16<InT>(x + (size_t)v * (16 * sizeof(InT)), xv);
    float sc;
    const uint4 w = quant_vec<WireT>(xv, gl, &sc);
    if (act) {
      const uint32_t t = v / vpr, col = v - t * vpr;
      for (uint32_t j = 0; j < top_k; j++) {
        const uint32_t r = (uint32_t)route[(size_t)t * top_k + j];
        if (r >= limit) continue;
        const uint32_t p = r / recv_rows, row = r - p * recv_rows;
        const size_t d = (size_t)row * vpr + col;                   // FP8 vector d of the owner's recv; its scale is element d >> lvpb
        st_vec((kPeers ? c.peer[p] + q_off : recv) + d * 16, w);
        if ((lane & (gl - 1)) == 0) *reinterpret_cast<float*>((kPeers ? c.peer[p] + s_off : scales) + (d >> lvpb) * 4) = sc;
      }
    }
  });
  if constexpr (kPeers) {
    const uint32_t s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<true>(c, 2 * s + 1, op)) return;         // my rows and scales are in every owner's buffers before its kernel ends
    if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
  }
}

// What the FP8 dispatch adds to the bf16 one: the scales buffer, the wire type and the quantising block.
struct RoutedQuant {
  float* recv_scales;
  b200collDataType_t wire;
  int block;
};

// The argument and placement rules of both routed dispatches (q == nullptr: b200collExpertDispatch, whose messages and codes these are).
// InvalidArgument before anything else, then RemoteError for a poisoned communicator, then InvalidUsage for buffers outside the arena
// and the B200COLL_CHECK=1 cross-check. Host only: nothing is launched.
static b200collResult_t routed_prepare(b200collComm* c, const void* x, const void* recv, size_t row_elems, size_t recv_rows, const int32_t* topk_idx,
                                       size_t tokens, int top_k, int num_experts, const int32_t* expert_counts, const int32_t* route,
                                       const int32_t* dropped, b200collDataType_t dtype, const RoutedQuant* q) {
  const std::string who = q ? "quantised expert dispatch: " : "expert dispatch: ";
  auto refuse = [&](const std::string& msg) { set_last_error(who + msg); return b200collInvalidArgument; };
  if (!c || !recv || !expert_counts || !dropped || (q && !q->recv_scales) || ((!x || !topk_idx || !route) && tokens > 0)) return refuse("null argument");
  if (!wide_type(dtype)) return refuse(q ? "in_dtype must be bf16, fp16 or fp32" : "dtype must be bf16, fp16 or fp32");
  if (q && !is_fp8(q->wire)) return refuse("wire_dtype must be e4m3 or e5m2");
  if (q && quant_lvpb(q->block) < 0) return refuse(kBlockRule);
  if (q ? row_elems == 0 || row_elems % (size_t)q->block != 0 : row_elems == 0 || row_elems % 16 != 0)
    return refuse(q ? "row_elems must be a positive multiple of block" : "row_elems must be a positive multiple of 16");
  if (top_k < 1) return refuse("top_k must be at least 1");
  if (num_experts < 1 || num_experts > kRouteMaxExperts || num_experts % c->nranks != 0)
    return refuse("num_experts must be in [1, 1024] and a multiple of nranks");
  const size_t max31 = ((size_t)1 << 31) - 1;
  if (tokens > max31 / (size_t)top_k) return refuse("tokens * top_k must be at most 2^31 - 1");
  if (recv_rows > max31 / (size_t)c->nranks) return refuse("nranks * recv_rows must be at most 2^31 - 1 (a route is an int32)");
  // the FP8 push walks (token, 16-element vector) pairs of x with 32-bit indices
  if (q && tokens > max31 / (row_elems / 16)) return refuse("at most 2^31 - 1 16-element vectors of x (tokens * row_elems / 16)");
  const size_t row_bytes = row_elems * b200collTypeSize(dtype), vpr = row_bytes / 16, slots = tokens * (size_t)top_k;
  if (slots > max31 / vpr) return refuse("at most 2^31 - 1 16-byte vectors offered (tokens * top_k * row_bytes / 16)");
  if (!aligned(x, 16) || !aligned(recv, 16)) return refuse("x and recv must be 16-byte aligned");
  if (q && !aligned(q->recv_scales, 4)) return refuse("recv_scales must be 4-byte aligned");
  if (!aligned(topk_idx, 4) || !aligned(expert_counts, 4) || !aligned(route, 4) || !aligned(dropped, 4))
    return refuse("topk_idx, expert_counts, route and dropped must be 4-byte aligned");
  // recv holds FP8 rows in the quantised call
  const size_t x_bytes = tokens * row_bytes, recv_bytes = recv_rows * (q ? row_elems : row_bytes), idx_bytes = slots * 4,
               counts_bytes = (size_t)(num_experts / c->nranks) * 4, scale_bytes = q ? recv_rows * (row_elems / (size_t)q->block) * 4 : 0;
  if (x && overlaps(recv, recv_bytes, x, x_bytes)) return refuse("recv must not overlap x");
  if (q && x && overlaps(q->recv_scales, scale_bytes, x, x_bytes)) return refuse("recv_scales must not overlap x");
  if (q && overlaps(q->recv_scales, scale_bytes, recv, recv_bytes)) return refuse("recv and recv_scales must not overlap");
  const struct { const void* p; size_t n; } outs[] = {{expert_counts, counts_bytes}, {route, idx_bytes}, {dropped, 4}},
                                         others[] = {{topk_idx, idx_bytes}, {x, x_bytes}, {recv, recv_bytes}, {q ? q->recv_scales : nullptr, scale_bytes}};
  for (size_t i = 0; i < 3; i++) {
    if (!outs[i].p) continue;
    for (size_t j = i + 1; j < 3; j++)
      if (outs[j].p && overlaps(outs[i].p, outs[i].n, outs[j].p, outs[j].n)) return refuse("expert_counts, route and dropped must not overlap each other");
    for (const auto& o : others)
      if (o.p && overlaps(outs[i].p, outs[i].n, o.p, o.n))
        return refuse(q ? "expert_counts, route and dropped must not overlap topk_idx, x, recv or recv_scales"
                        : "expert_counts, route and dropped must not overlap topk_idx, x or recv");
  }
  if (comm_poisoned(c)) return b200collRemoteError;
  if (c->nranks == 1) return b200collSuccess;
  // peers push into my recv (and recv_scales)
  b200collResult_t rc = q ? in_arena(c, who, "recv and recv_scales", {{recv, recv_bytes}, {q->recv_scales, scale_bytes}}) : in_arena(c, who, "recv", {{recv, recv_bytes}});
  if (rc != b200collSuccess) return rc;
  // (E, row_elems) travel as one number: E < 2048
  if (!q) return cross_check(c, b200collOpAllToAll, b200collAlgoTwoShot, recv_rows, arena_off(c, recv), row_elems * 2048 + (size_t)num_experts);
  // the FP8 call has one more offset, so two exchanges: (recv_rows, both offsets), then (row_elems, E, block and wire)
  rc = cross_check(c, b200collOpAllToAll, b200collAlgoTwoShot, recv_rows, arena_off(c, recv), arena_off(c, q->recv_scales));
  if (rc != b200collSuccess) return rc;
  return cross_check(c, b200collOpAllToAll, b200collAlgoTwoShot, row_elems, (size_t)num_experts, (size_t)q->block * 2 + (q->wire == b200collFloat8e5m2));
}

// Once per device, before the first layout kernel of either dispatch and before the first quantising combine launches anything: the
// layout kernel's shared-memory limit, and every kernel that can follow it loaded: both dispatches' push kernels, the quantise pass
// k_a2av_quant_copy, and every combine kernel, wide and quantising. With lazy module loading the first launch of a kernel loads it, and
// the load waits for kernels already running: a kernel launched for the first time behind a layout (or pull) kernel that waits at its
// barrier for another rank's launch would hold that launch up, whether the other rank is driven by the same host thread or by another
// thread waiting for the load. Whichever call runs first on a device loads the others' kernels too.
// One thread loads at a time, and the others wait on the host: a thread that finds the work done makes no CUDA call here, so no load
// can start after another rank's layout kernel is already running.
void routed_preload(const b200collComm* c) {
  static std::atomic<unsigned long long> attr_done{0};          // per device, as in launch_bulk
  static std::mutex mu;
  const unsigned long long bit = 1ull << (c->device & 63);
  if (attr_done.load(std::memory_order_acquire) & bit) return;
  const std::lock_guard<std::mutex> lk(mu);
  if (attr_done.load(std::memory_order_acquire) & bit) return;
  cudaFuncSetAttribute(k_routed_layout, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)layout_smem(kRouteMaxExperts));
  cudaFuncAttributes fa;
  cudaFuncGetAttributes(&fa, k_routed_push<true>);
  cudaFuncGetAttributes(&fa, k_routed_push<false>);
  for (b200collDataType_t in : {b200collBfloat16, b200collFloat16, b200collFloat32})
    for (b200collDataType_t wire : {b200collFloat8e4m3, b200collFloat8e5m2})
      with_wide(in, [&](auto ti) { with_fp8(wire, [&](auto tw) {
        using InT = typename decltype(ti)::type; using WireT = typename decltype(tw)::type;
        cudaFuncGetAttributes(&fa, k_expert_quant_push<InT, WireT, true>);
        cudaFuncGetAttributes(&fa, k_expert_quant_push<InT, WireT, false>);
        cudaFuncGetAttributes(&fa, k_a2av_quant_copy<InT, WireT>);
      }); });
  combine_preload();
  attr_done.fetch_or(bit, std::memory_order_acq_rel);
}

b200collResult_t launch_quant_copy(b200collComm* c, b200collDataType_t in_dtype, b200collDataType_t wire, const void* in, char* q, char* scales,
                                   uint32_t nvec, uint32_t lvpb, cudaStream_t st) {
  QuantGeom g = {};
  g.nvec = nvec;
  g.lvpb = lvpb;
  return with_wide(in_dtype, [&](auto ti) { return with_fp8(wire, [&](auto tw) -> b200collResult_t {
    using InT = typename decltype(ti)::type; using WireT = typename decltype(tw)::type;
    launch_k(k_a2av_quant_copy<InT, WireT>, copy_blocks(c, g.nvec), 256, st, g, static_cast<const char*>(in), q, scales);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  }); });
}

static b200collResult_t launch_layout(b200collComm* c, const int32_t* topk_idx, size_t slots, int num_experts, size_t recv_rows, int32_t* route,
                                      int32_t* expert_counts, int32_t* dropped, cudaStream_t st) {
  routed_preload(c);
  launch_k_smem(k_routed_layout, 1, kLayoutThreads, layout_smem(num_experts), st, c->dev, topk_idx, (uint32_t)slots, num_experts, (uint32_t)recv_rows,
                route, expert_counts, dropped, (uint32_t)b200collOpAllToAll);
  LAUNCH_CHECK(c);
  return b200collSuccess;
}

// Everything b200collAllToAllvQuantized checks before it launches; on success `a` holds the vector geometry (prefix not yet filled),
// `nv` the vectors per peer and `in_bytes` the input bytes sent.
static b200collResult_t a2aq_prepare(b200collComm* c, const void* send, void* recv, float* recv_scales, size_t row_elems, size_t recv_rows,
                                     const int64_t* send_rows, const int64_t* send_row_off, const int64_t* recv_row_off_at_peer,
                                     b200collDataType_t in_dtype, b200collDataType_t wire, int block, A2AvArgs* a, unsigned long long* nv,
                                     size_t* in_bytes) {
  auto refuse = [](const std::string& msg) { set_last_error("quantised all-to-all-v: " + msg); return b200collInvalidArgument; };
  if (!c || !send || !recv || !recv_scales || !send_rows || !send_row_off || !recv_row_off_at_peer) return refuse("null argument");
  if (!wide_type(in_dtype)) return refuse("in_dtype must be bf16, fp16 or fp32");
  if (!is_fp8(wire)) return refuse("wire_dtype must be e4m3 or e5m2");
  if (quant_lvpb(block) < 0) return refuse(kBlockRule);
  if (row_elems == 0 || row_elems % (size_t)block != 0) return refuse("row_elems must be a positive multiple of block");
  if (!aligned(send, 16) || !aligned(recv, 16) || !aligned(recv_scales, 4)) return refuse("send and recv must be 16-byte aligned, recv_scales 4-byte aligned");
  const size_t is = b200collTypeSize(in_dtype);
  const size_t max_rows = (SIZE_MAX >> 4) / (row_elems * is);     // every byte offset below then fits in size_t with room to spare
  if (recv_rows > max_rows) return refuse("recv_rows * row_elems is too large");
  const unsigned long long row_vecs = row_elems / 16, max_vecs = (1ull << 31) - 1;
  unsigned long long total = 0;
  size_t send_end = 0;                                            // the bytes of send that are read
  *in_bytes = 0;
  A2AvRows rg;
  const std::string bad = a2av_rows(c->nranks, send_rows, send_row_off, recv_row_off_at_peer, recv_rows, max_rows, &rg);
  if (!bad.empty()) return refuse(bad);
  for (int p = 0; p < c->nranks; p++) {
    const size_t rows = rg.rows[p], src = rg.src_row[p], dst = rg.dst_row[p];
    if (rows > (max_vecs - total) / row_vecs) return refuse("at most 2^31 - 1 16-element vectors may be sent per rank");
    total += rows * row_vecs;
    a->src_vec[p] = src * row_vecs;
    a->dst_vec[p] = dst * row_vecs;
    nv[p] = rows * row_vecs;
    *in_bytes += rows * row_elems * is;
    if (rows) send_end = std::max(send_end, (src + rows) * row_elems * is);
  }
  if (comm_poisoned(c)) return b200collRemoteError;
  const size_t q_bytes = recv_rows * row_elems, s_bytes = recv_rows * (row_elems / (size_t)block) * 4;
  if (overlaps(send, send_end, recv, q_bytes) || overlaps(send, send_end, recv_scales, s_bytes)) return refuse("send must not overlap recv or recv_scales");
  if (overlaps(recv, q_bytes, recv_scales, s_bytes)) return refuse("recv and recv_scales must not overlap");
  // peers store into my recv and recv_scales
  if (c->nranks == 1) return b200collSuccess;
  return in_arena(c, "quantised all-to-all-v: ", "recv and recv_scales", {{recv, q_bytes}, {recv_scales, s_bytes}});
}

}  // namespace b200coll

using namespace b200coll;

extern "C" {

b200collResult_t b200collAllToAllvQuantized(const void* send, void* recv, float* recv_scales, size_t row_elems, size_t recv_rows,
                                            const int64_t* send_rows, const int64_t* send_row_off, const int64_t* recv_row_off_at_peer,
                                            b200collDataType_t in_dtype, b200collDataType_t wire_dtype, int block,
                                            b200collComm_t c, b200collStream_t stream) {
  A2AvArgs a = {};
  unsigned long long nv[kMaxRanks] = {};
  size_t in_bytes = 0;
  b200collResult_t rc = a2aq_prepare(c, send, recv, recv_scales, row_elems, recv_rows, send_rows, send_row_off, recv_row_off_at_peer, in_dtype, wire_dtype,
                                     block, &a, nv, &in_bytes);
  if (rc != b200collSuccess) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint32_t lvpb = (uint32_t)quant_lvpb(block);
  if (c->nranks == 1) {
    account(c, b200collOpAllToAll, in_bytes, b200collAlgoCopy);
    if (nv[0] == 0) return b200collSuccess;
    const char* in = static_cast<const char*>(send) + a.src_vec[0] * 16 * b200collTypeSize(in_dtype);
    char* q = static_cast<char*>(recv) + a.dst_vec[0] * 16;
    char* s = reinterpret_cast<char*>(recv_scales) + (a.dst_vec[0] >> lvpb) * 4;
    return launch_quant_copy(c, in_dtype, wire_dtype, in, q, s, (uint32_t)nv[0], lvpb, st);
  }
  rc = cross_check(c, b200collOpAllToAll, b200collAlgoTwoShot, recv_rows, arena_off(c, recv), arena_off(c, recv_scales));
  if (rc != b200collSuccess) return rc;
  a2av_prefix(c->rank, c->nranks, nv, &a);
  account(c, b200collOpAllToAll, in_bytes, b200collAlgoTwoShot);
  const Grid gr = full_grid(c, 1, true);
  return with_wide(in_dtype, [&](auto ti) { return with_fp8(wire_dtype, [&](auto tw) -> b200collResult_t {
    using InT = typename decltype(ti)::type; using WireT = typename decltype(tw)::type;
    launch_k(k_a2av_quant_push<InT, WireT>, gr.blocks, gr.threads, st, c->dev, static_cast<const char*>(send), arena_off(c, recv), arena_off(c, recv_scales), a,
             lvpb, (uint32_t)b200collOpAllToAll);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  }); });
}

b200collResult_t b200collExpertDispatch(const void* x, void* recv, size_t row_elems, size_t recv_rows, const int32_t* topk_idx, size_t tokens,
                                        int top_k, int num_experts, int32_t* expert_counts, int32_t* route, int32_t* dropped,
                                        b200collDataType_t dtype, b200collComm_t c, b200collStream_t stream) {
  b200collResult_t rc = routed_prepare(c, x, recv, row_elems, recv_rows, topk_idx, tokens, top_k, num_experts, expert_counts, route, dropped, dtype, nullptr);
  if (rc != b200collSuccess) return rc;
  const DeviceScope on_device(c->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool peers = c->nranks > 1;
  const size_t row_bytes = row_elems * b200collTypeSize(dtype), vpr = row_bytes / 16, slots = tokens * (size_t)top_k;
  account(c, b200collOpAllToAll, slots * row_bytes, peers ? b200collAlgoTwoShot : b200collAlgoCopy);
  if ((rc = launch_layout(c, topk_idx, slots, num_experts, recv_rows, route, expert_counts, dropped, st)) != b200collSuccess) return rc;
  const uint32_t nvec = (uint32_t)(slots * vpr);
  if (peers) {
    const Grid gr = full_grid(c, kRoutedPushUnroll);
    launch_k(k_routed_push<true>, gr.blocks, gr.threads, st, c->dev, static_cast<const char*>(x), static_cast<char*>(nullptr), arena_off(c, recv), route,
             (uint32_t)top_k, (uint32_t)vpr, nvec, (uint32_t)recv_rows, (uint32_t)b200collOpAllToAll);
  } else {
    const size_t per_cta = (size_t)kRoutedPushThreads * kRoutedPushUnroll;
    const int blocks = (int)std::max<size_t>(1, std::min<size_t>((nvec + per_cta - 1) / per_cta, (size_t)4 * std::max(1, c->sm_count)));
    launch_k(k_routed_push<false>, blocks, kRoutedPushThreads, st, c->dev, static_cast<const char*>(x), static_cast<char*>(recv), (size_t)0, route,
             (uint32_t)top_k, (uint32_t)vpr, nvec, (uint32_t)recv_rows, (uint32_t)b200collOpAllToAll);
  }
  LAUNCH_CHECK(c);
  return b200collSuccess;
}

b200collResult_t b200collExpertDispatchQuantized(const void* x, void* recv, float* recv_scales, size_t row_elems, size_t recv_rows,
                                                 const int32_t* topk_idx, size_t tokens, int top_k, int num_experts,
                                                 int32_t* expert_counts, int32_t* route, int32_t* dropped,
                                                 b200collDataType_t in_dtype, b200collDataType_t wire_dtype, int block,
                                                 b200collComm_t c, b200collStream_t stream) {
  const RoutedQuant q{recv_scales, wire_dtype, block};
  b200collResult_t rc = routed_prepare(c, x, recv, row_elems, recv_rows, topk_idx, tokens, top_k, num_experts, expert_counts, route, dropped, in_dtype, &q);
  if (rc != b200collSuccess) return rc;
  const DeviceScope on_device(c->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t slots = tokens * (size_t)top_k;
  account(c, b200collOpAllToAll, slots * row_elems * b200collTypeSize(in_dtype), c->nranks > 1 ? b200collAlgoTwoShot : b200collAlgoCopy);
  if ((rc = launch_layout(c, topk_idx, slots, num_experts, recv_rows, route, expert_counts, dropped, st)) != b200collSuccess) return rc;
  const uint32_t lvpb = (uint32_t)quant_lvpb(block);
  const uint32_t vpr = (uint32_t)(row_elems / 16), nvec = (uint32_t)(tokens * vpr);
  const char* in = static_cast<const char*>(x);
  return with_wide(in_dtype, [&](auto ti) { return with_fp8(wire_dtype, [&](auto tw) -> b200collResult_t {
    using InT = typename decltype(ti)::type; using WireT = typename decltype(tw)::type;
    if (c->nranks > 1) {
      const Grid gr = full_grid(c, 1, true);
      launch_k(k_expert_quant_push<InT, WireT, true>, gr.blocks, gr.threads, st, c->dev, in, static_cast<char*>(nullptr), static_cast<char*>(nullptr),
               arena_off(c, recv), arena_off(c, recv_scales), route, (uint32_t)top_k, vpr, nvec, (uint32_t)recv_rows, lvpb, (uint32_t)b200collOpAllToAll);
    } else {
      launch_k(k_expert_quant_push<InT, WireT, false>, copy_blocks(c, nvec), 256, st, c->dev, in, static_cast<char*>(recv), reinterpret_cast<char*>(recv_scales),
               (size_t)0, (size_t)0, route, (uint32_t)top_k, vpr, nvec, (uint32_t)recv_rows, lvpb, (uint32_t)b200collOpAllToAll);
    }
    LAUNCH_CHECK(c);
    return b200collSuccess;
  }); });
}

}  // extern "C"
