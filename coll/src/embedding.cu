// libb200coll vocab-parallel embedding for tensor-parallel input layers (b200collVocabParallelEmbedding / ...Backward): the table is split
// by vocabulary, rank r owning the rows of the global ids [r * Vl, (r + 1) * Vl), and every output row has exactly one source, so the
// forward fetches it instead of summing N mostly-zero tensors, and the backward sums each owned row's gradient in token order:
//
//   k_emb_fwd<LOCAL>             relaxed barrier, pull every 16-byte vector of this rank's output rows from the owner's weight (the same
//                                arena offset on every rank), +0 for an id outside [0, N * Vl), releasing barrier. LOCAL: one rank, a
//                                gather from any device memory, no barrier
//   k_emb_hist<FIRST>            one CTA per tile of kEmbTile tokens: the tile's count of each 8-bit digit of the key
//   k_emb_scan                   one CTA: the exclusive prefix of the counts in (digit, tile) order
//   k_emb_scatter<FIRST>         one CTA per tile: each key's stable rank among the tile's keys with its digit, and the key and its token
//                                stored at their place in the next order
//   k_emb_bounds                 bounds[j] = the first place of local row j in the sorted keys (binary search), j = 0 .. Vl
//   k_emb_bwd<TD, TW, PEER>      per (local row, 16-byte vector of dout): fold the row's tokens in token order in fp32, round once into
//                                dweight. PEER (sequence parallel, N > 1): dout row t pulled from rank t / (T / N) between a relaxed
//                                entry barrier and a releasing closing barrier; otherwise dout is local and there is no barrier
//
// Grouping. The backward needs this rank's tokens grouped by local row in token order. The key of token t is ids[t] - r * Vl when that
// lies in [0, Vl), else Vl (not owned: sorted past every row and never read). An LSD radix sort over the key's 8-bit digits, lowest first,
// one hist / scan / scatter triple per digit (ceil(bits(Vl) / 8) triples: 3 for a 152K vocabulary at one rank), orders the tokens by key
// and, because every pass is stable, by token within a key: the order of numpy's stable argsort. Stability inside a pass: a tile is 16
// warps, warp w walking its 128 consecutive keys 32 at a time; __match_any_sync groups the lanes with one digit, a lane's rank in the
// group is the popcount of the lower lanes in it, and the group's lowest lane adds the group's size to the warp's count of that digit in
// shared memory. A key's place is then the scanned count of (digit, tile), plus the counts of the lower warps of its tile, plus its rank in
// its warp. No atomic hands out a place, so the order, and with it every sum below, is the same on every run. (k_routed_layout in
// dispatch.cu ranks the same way inside one CTA for up to 1024 experts; Vl is too wide for one CTA's counters, hence the tiles and the
// scan. The two share no helper: the layout keeps its counts per expert across the whole call, the sort per digit and tile.)
//
// Sum. k_emb_bwd walks (row, vector) items a warp at a time: a warp owns 32 consecutive vectors (512 bytes of dout columns) of one row,
// and consecutive warp items go to consecutive CTAs, so one row hit by every token (a padding id) is spread over H * sizeof(dout) / 512
// warps on as many SMs rather than serialised on one. Each lane folds its E columns over the row's tokens in sorted (token) order, from
// +0 or from dweight when accumulating, every add an IEEE fp32 add rounded on its own (__fadd_rn), with the next kEmbBwdUnroll tokens'
// vectors loaded ahead; then rounds once (RNE) to dweight's type. The fold of one column is sequential by definition, so its length, the
// row's token count, bounds the time of a skewed call; the work of distinct rows and columns runs in parallel. Nothing depends on the
// launch shape. The scratch (keys and tokens twice, the tile counts and the bounds: 16 T + 1024 * tiles + 4 (Vl + 1) bytes, each part
// 16-byte aligned) is this rank's own: it lies in the quantising collectives' scratch, taken like the cross-entropy's mailbox.
//
// Ordering (rank s, call k). The forward: the entry barrier is relaxed; a peer arrives only once its stream has reached this call, so its
// weight (last written by its optimizer step, an earlier kernel on its stream) is complete before any rank pulls it. The closing barrier
// is releasing: no rank leaves before every peer has pulled its rows, so the next kernel on a peer's stream may change its weight, and out
// is this rank's own. The SP backward has the same two barriers around the pulls of dout. Its sort kernels come before the entry barrier
// on the same stream and touch only this rank's scratch: a peer writes into this rank's scratch only inside a later call, after an entry
// barrier that this rank reaches when this call's kernels have ended (the cross-entropy's mailbox), and reads it only before a closing
// barrier this rank has already passed (the quantising collectives). Both barriers pair CTA b with CTA b; every rank launches the same
// grid, as T, H and Vl are equal on every rank. Graph replay: the kernels read the epoch from the communicator's state word (load_seq)
// and bump it once; no epoch and no device data travel through the host.
#include <stdint.h>

#include <atomic>
#include <mutex>
#include <string>

#include "comm.h"
#include "index.cuh"
#include "launch.cuh"

namespace b200coll {

constexpr int kEmbThreads = 512, kEmbUnroll = 4;                 // the forward
constexpr int kEmbSortThreads = 512, kEmbSortWarps = kEmbSortThreads / 32, kEmbSortItems = 4;
constexpr uint32_t kEmbTile = kEmbSortThreads * kEmbSortItems;    // 2048 keys per tile
constexpr int kEmbDigits = 256, kEmbScanThreads = 1024;
constexpr int kEmbBwdUnroll = 8;
constexpr size_t kEmbI31 = ((size_t)1 << 31) - 1;

struct EmbFwdArgs {
  const int64_t* ids;
  unsigned long long weight;       // this rank's weight: its arena offset (every rank's is the same), or with LOCAL its address
  char* out;
  uint32_t tok0;                   // the token of out's first row
  uint32_t total;                  // out rows * vectors per row
  uint32_t nvocab;                 // N * Vl
  FastDiv nvec;                    // 16-byte vectors per row
  FastDiv vl;
};

template <bool LOCAL>
__global__ void __launch_bounds__(kEmbThreads) k_emb_fwd(COMM_PARAM, const __grid_constant__ EmbFwdArgs a, uint32_t op) {
  pdl_prologue();
  constexpr int U = kEmbUnroll;
  uint32_t s = 0;
  if (!LOCAL) {
    s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;        // every rank's weight is written
  }
  const uint32_t stride = gridDim.x * blockDim.x * U;
  for (uint32_t base = blockIdx.x * blockDim.x * U + threadIdx.x; base < a.total; base += stride) {
    uint4 d[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const uint32_t g = base + (uint32_t)u * blockDim.x;
      d[u] = make_uint4(0u, 0u, 0u, 0u);
      if (g < a.total) {
        const uint32_t row = div_by(g, a.nvec), v = g - row * a.nvec.d;
        const int64_t id = __ldg(a.ids + a.tok0 + row);
        if (id >= 0 && id < (int64_t)a.nvocab) {
          const uint32_t p = div_by((uint32_t)id, a.vl), lr = (uint32_t)id - p * a.vl.d;
          const unsigned long long off = a.weight + 16ull * ((unsigned long long)lr * a.nvec.d + v);
          d[u] = ld_vec(LOCAL ? reinterpret_cast<const char*>(off) : c.peer[p] + off);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const uint32_t g = base + (uint32_t)u * blockDim.x;
      if (g < a.total) st_vec(a.out + 16ull * g, d[u]);
    }
  }
  if (!LOCAL) {
    if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;          // every rank has pulled its rows: weights may change again
    if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
  }
}

// ---------------------------------------------------------------- the stable grouping by local row
struct EmbSortArgs {
  const int64_t* ids;
  const uint32_t* keys_in;         // !FIRST: the previous pass's order
  const uint32_t* toks_in;
  uint32_t* keys_out;
  uint32_t* toks_out;
  uint32_t* hist;                  // [256][tiles]
  int64_t start;                   // r * Vl
  uint32_t tokens, vl, tiles, shift;
};

template <bool FIRST>
__device__ __forceinline__ void emb_key(const EmbSortArgs& a, uint32_t i, uint32_t* key, uint32_t* tok) {
  if (FIRST) {
    const int64_t k = a.ids[i] - a.start;
    *key = k >= 0 && k < (int64_t)a.vl ? (uint32_t)k : a.vl;
    *tok = i;
  } else {
    *key = a.keys_in[i];
    *tok = a.toks_in[i];
  }
}

template <bool FIRST>
__global__ void __launch_bounds__(kEmbSortThreads) k_emb_hist(const __grid_constant__ EmbSortArgs a) {
  pdl_prologue();
  __shared__ uint32_t cnt[kEmbDigits];
  if (threadIdx.x < kEmbDigits) cnt[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t t0 = blockIdx.x * kEmbTile;
#pragma unroll
  for (int k = 0; k < kEmbSortItems; k++) {
    const uint32_t i = t0 + (uint32_t)k * kEmbSortThreads + threadIdx.x;
    if (i < a.tokens) {
      uint32_t key, tok;
      emb_key<FIRST>(a, i, &key, &tok);
      atomicAdd(&cnt[(key >> a.shift) & 255u], 1u);             // an integer count: the same whatever the order of the adds
    }
  }
  __syncthreads();
  if (threadIdx.x < kEmbDigits) a.hist[(size_t)threadIdx.x * a.tiles + blockIdx.x] = cnt[threadIdx.x];
}

// the exclusive prefix of hist[0 .. n) in place, one CTA: each thread a contiguous chunk
__global__ void __launch_bounds__(kEmbScanThreads) k_emb_scan(uint32_t* hist, uint32_t n) {
  pdl_prologue();
  __shared__ uint32_t wsum[kEmbScanThreads / 32];
  const uint32_t t = threadIdx.x, lane = t & 31, w = t >> 5;
  const uint32_t per = (n + kEmbScanThreads - 1) / kEmbScanThreads;
  const uint32_t lo = min(n, t * per), hi = min(n, lo + per);
  uint32_t sum = 0;
  for (uint32_t i = lo; i < hi; i++) sum += hist[i];
  uint32_t x = sum;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= (uint32_t)d) x += y; }
  if (lane == 31) wsum[w] = x;
  __syncthreads();
  if (t == 0) {
    uint32_t run = 0;
    for (int v = 0; v < kEmbScanThreads / 32; v++) { const uint32_t q = wsum[v]; wsum[v] = run; run += q; }
  }
  __syncthreads();
  uint32_t run = x - sum + wsum[w];
  for (uint32_t i = lo; i < hi; i++) { const uint32_t q = hist[i]; hist[i] = run; run += q; }
}

template <bool FIRST>
__global__ void __launch_bounds__(kEmbSortThreads) k_emb_scatter(const __grid_constant__ EmbSortArgs a) {
  pdl_prologue();
  __shared__ uint32_t cnt[kEmbSortWarps][kEmbDigits];
  const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (uint32_t i = threadIdx.x; i < kEmbSortWarps * kEmbDigits; i += blockDim.x) (&cnt[0][0])[i] = 0;
  __syncthreads();
  // 1. each key's rank among the keys of its warp's segment with the same digit (segment order is token order within the tile)
  const uint32_t seg = blockIdx.x * kEmbTile + w * (32u * kEmbSortItems);
  uint32_t key[kEmbSortItems], tok[kEmbSortItems], rank[kEmbSortItems];
#pragma unroll
  for (int k = 0; k < kEmbSortItems; k++) {
    const uint32_t i = seg + (uint32_t)k * 32 + lane;
    uint32_t dg = kEmbDigits;                                    // past the end: a group of its own that takes no place
    key[k] = 0; tok[k] = 0; rank[k] = 0;
    if (i < a.tokens) { emb_key<FIRST>(a, i, &key[k], &tok[k]); dg = (key[k] >> a.shift) & 255u; }
    const unsigned same = __match_any_sync(0xFFFFFFFFu, dg);
    const uint32_t lower = __popc(same & ((1u << lane) - 1u));
    if (dg < kEmbDigits) rank[k] = cnt[w][dg] + lower;
    __syncwarp();
    if (dg < kEmbDigits && lower == 0) cnt[w][dg] += __popc(same);
    __syncwarp();
  }
  __syncthreads();
  // 2. per digit: the tile's scanned base plus the exclusive prefix over the warps
  for (uint32_t dg = threadIdx.x; dg < kEmbDigits; dg += blockDim.x) {
    uint32_t run = a.hist[(size_t)dg * a.tiles + blockIdx.x];
    for (int v = 0; v < kEmbSortWarps; v++) { const uint32_t x = cnt[v][dg]; cnt[v][dg] = run; run += x; }
  }
  __syncthreads();
  // 3. the stores
#pragma unroll
  for (int k = 0; k < kEmbSortItems; k++) {
    const uint32_t i = seg + (uint32_t)k * 32 + lane;
    if (i < a.tokens) {
      const uint32_t pos = cnt[w][(key[k] >> a.shift) & 255u] + rank[k];
      a.keys_out[pos] = key[k];
      a.toks_out[pos] = tok[k];
    }
  }
}

// bounds[j] = the number of sorted keys below j, j = 0 .. vl: row j's tokens are toks[bounds[j] .. bounds[j + 1])
__global__ void __launch_bounds__(256) k_emb_bounds(const uint32_t* __restrict__ keys, uint32_t tokens, uint32_t vl, uint32_t* __restrict__ bounds) {
  pdl_prologue();
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j <= vl; j += gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = tokens;
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      if (keys[mid] < j) lo = mid + 1; else hi = mid;
    }
    bounds[j] = lo;
  }
}

// ---------------------------------------------------------------- the fold
struct EmbBwdArgs {
  unsigned long long dout;         // PEER: dout's arena offset (every rank's is the same); otherwise its address
  char* dweight;
  const uint32_t* toks;            // the sorted tokens, nullptr when T == 0
  const uint32_t* bounds;
  uint32_t total;                  // Vl * vectors of dout per row
  uint32_t accumulate;
  FastDiv nvd;                     // 16-byte vectors of dout per row
  FastDiv shard;                   // PEER: T / N, the rows of each rank's dout
};

// one 16-byte vector of T widened to fp32 bit for bit (-0 and NaN payloads kept)
template <typename T> __device__ __forceinline__ void emb_widen(const uint4& v, float* x) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; i++) {
    if constexpr (std::is_same<T, float>::value) {
      x[i] = __uint_as_float(w[i]);
    } else if constexpr (std::is_same<T, __nv_bfloat16>::value) {
      x[2 * i] = __uint_as_float(w[i] << 16); x[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
    } else {
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
      x[2 * i] = f.x; x[2 * i + 1] = f.y;
    }
  }
}

template <typename TD, typename TW, bool PEER>
__global__ void __launch_bounds__(kEmbThreads, 2) k_emb_bwd(COMM_PARAM, const __grid_constant__ EmbBwdArgs a, uint32_t op) {
  pdl_prologue();
  constexpr int E = Epv<TD>::value, U = kEmbBwdUnroll;
  constexpr int WV = E * (int)sizeof(TW) / 16;                   // 16-byte vectors of dweight per vector of dout: 1, or 2 (fp32 from 16-bit)
  uint32_t s = 0;
  if (PEER) {
    s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;        // every rank's dout is written
  }
  const uint32_t lane = threadIdx.x & 31, wpc = blockDim.x >> 5;
  const uint32_t items = (a.total + 31) / 32;                    // warp items: 32 consecutive (row, vector) pairs
  for (uint32_t wi = blockIdx.x + gridDim.x * (threadIdx.x >> 5); wi < items; wi += gridDim.x * wpc) {
    const uint32_t g = wi * 32 + lane;
    if (g >= a.total) continue;
    const uint32_t row = div_by(g, a.nvd), v = g - row * a.nvd.d;
    char* dw = a.dweight + 16ull * WV * g;                        // row * nvd + v == g
    float acc[E];
    if (a.accumulate) {
#pragma unroll
      for (int q = 0; q < WV; q++) emb_widen<TW>(ld_vec(dw + 16 * q), acc + q * (E / WV));
    } else {
#pragma unroll
      for (int i = 0; i < E; i++) acc[i] = 0.0f;
    }
    const uint32_t lo = a.toks ? a.bounds[row] : 0u, hi = a.toks ? a.bounds[row + 1] : 0u;
    for (uint32_t i = lo; i < hi; i += U) {
      uint4 d[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        if (i + u < hi) {
          const uint32_t t = a.toks[i + u];
          if (PEER) {
            const uint32_t p = div_by(t, a.shard);
            d[u] = ld_vec(c.peer[p] + a.dout + 16ull * ((unsigned long long)(t - p * a.shard.d) * a.nvd.d + v));
          } else {
            d[u] = ld_vec(reinterpret_cast<const char*>(a.dout) + 16ull * ((unsigned long long)t * a.nvd.d + v));
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        if (i + u < hi) {                                        // token order: the sorted order
          float x[E];
          emb_widen<TD>(d[u], x);
#pragma unroll
          for (int k = 0; k < E; k++) acc[k] = __fadd_rn(acc[k], x[k]);
        }
      }
    }
    uint32_t o[Pack<TW, E>::W];
    Pack<TW, E>::run(acc, o);
    st_words<Pack<TW, E>::W>(dw, o);
  }
  if (PEER) {
    if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;          // every rank has pulled its rows: dout may change again
    if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
  }
}

// Once per device, before the first kernel of this family launches: load all of them (see ulysses_preload: with lazy module loading and
// virtual ranks, a first launch queued behind a peer-waiting barrier kernel would never load).
static void embedding_preload(const b200collComm* c) {
  static std::atomic<unsigned long long> done{0};
  static std::mutex mu;
  const unsigned long long bit = 1ull << (c->device & 63);
  if (done.load(std::memory_order_acquire) & bit) return;
  const std::lock_guard<std::mutex> lk(mu);
  if (done.load(std::memory_order_acquire) & bit) return;
  cudaFuncAttributes fa;
  cudaFuncGetAttributes(&fa, k_emb_fwd<true>);
  cudaFuncGetAttributes(&fa, k_emb_fwd<false>);
  cudaFuncGetAttributes(&fa, k_emb_hist<true>);
  cudaFuncGetAttributes(&fa, k_emb_hist<false>);
  cudaFuncGetAttributes(&fa, k_emb_scan);
  cudaFuncGetAttributes(&fa, k_emb_scatter<true>);
  cudaFuncGetAttributes(&fa, k_emb_scatter<false>);
  cudaFuncGetAttributes(&fa, k_emb_bounds);
  for (b200collDataType_t td : {b200collBfloat16, b200collFloat16, b200collFloat32})
    with_wide(td, [&](auto t) {
      using TD = typename decltype(t)::type;
      cudaFuncGetAttributes(&fa, k_emb_bwd<TD, TD, false>);
      cudaFuncGetAttributes(&fa, k_emb_bwd<TD, TD, true>);
      cudaFuncGetAttributes(&fa, k_emb_bwd<TD, float, false>);
      cudaFuncGetAttributes(&fa, k_emb_bwd<TD, float, true>);
    });
  done.fetch_or(bit, std::memory_order_acq_rel);
}

// The rules both calls share. InvalidArgument (nothing launched) for every one of them, then RemoteError for a poisoned communicator.
// `table` is weight (forward) or dweight (backward), `rows` the forward's out or the backward's dout. Returns the rows of out (forward) or
// dout (backward) on this rank.
static b200collResult_t emb_check(b200collComm* c, const std::string& who, bool forward, const int64_t* ids, const void* table, const void* rows,
                                  size_t tokens, size_t hidden, size_t vl, int sp, b200collDataType_t dt_rows, b200collDataType_t dt_table,
                                  size_t* out_rows) {
  auto refuse = [&](const std::string& msg) { set_last_error(who + msg); return b200collInvalidArgument; };
  if (!c) return refuse("null communicator");
  if (!wide_type(dt_rows)) return refuse(forward ? "dtype must be bf16, fp16 or fp32" : "dout_dtype must be bf16, fp16 or fp32");
  if (!forward && dt_table != b200collFloat32 && dt_table != dt_rows) return refuse("dweight_dtype must be fp32 or dout_dtype");
  const size_t er = b200collTypeSize(dt_rows), et = b200collTypeSize(dt_table), N = (size_t)c->nranks;
  if (hidden == 0 || (hidden * er) % 16 != 0 || (hidden * et) % 16 != 0)
    return refuse("hidden must be positive and hidden * sizeof(dtype) a multiple of 16 bytes for every dtype");
  if (vl == 0) return refuse("vocab_local must be positive");
  if (vl >= ((size_t)1 << 31) || N * vl >= ((size_t)1 << 31)) return refuse("nranks * vocab_local must be below 2^31");
  if (tokens >= ((size_t)1 << 31)) return refuse("tokens must be below 2^31");
  if (sp && tokens % N != 0) return refuse("tokens must be a multiple of nranks under sequence parallelism");
  const size_t nr = (sp ? tokens / N : tokens);
  const size_t vr = hidden * er / 16, vt = hidden * et / 16;
  if (nr * vr > kEmbI31 || vl * vr > kEmbI31 || vl * vt > kEmbI31) return refuse("more than 2^31 - 1 16-byte vectors in one tensor");
  if (!table) return refuse(forward ? "null weight" : "null dweight");
  if (tokens > 0 && (!ids || !rows)) return refuse("null argument");
  if (!aligned(ids, 8)) return refuse("ids must be 8-byte aligned");
  if (!aligned(table, 16) || !aligned(rows, 16)) return refuse(forward ? "weight and out must be 16-byte aligned" : "dout and dweight must be 16-byte aligned");
  const size_t table_bytes = vl * hidden * et, rows_bytes = nr * hidden * er;
  if (forward) {
    if (tokens > 0 && (overlaps(rows, rows_bytes, table, table_bytes) || overlaps(rows, rows_bytes, ids, tokens * 8)))
      return refuse("out must not overlap weight or ids");
  } else {
    if (tokens > 0 && (overlaps(table, table_bytes, rows, rows_bytes) || overlaps(table, table_bytes, ids, tokens * 8)))
      return refuse("dweight must not overlap dout or ids");
  }
  if (comm_poisoned(c)) return b200collRemoteError;
  // peers pull from this rank's weight (forward) or sequence-parallel dout (backward) at this rank's arena offset
  const bool peers_read = N > 1 && tokens > 0 && (forward || sp);
  if (peers_read) {
    const void* p = forward ? table : rows;
    const size_t n = forward ? table_bytes : rows_bytes;
    if (!b200collIsSymmetric(c, p, std::max<size_t>(n, 1)))
      return refuse(std::string(forward ? "weight" : "dout") + " must lie in the symmetric arena (b200collMemAlloc), at the same offset on every rank");
  }
  *out_rows = nr;
  return b200collSuccess;
}

static b200collResult_t emb_forward(b200collComm* c, const int64_t* ids, const void* weight, void* out, size_t tokens, size_t hidden, size_t vl,
                                    int sp, b200collDataType_t dtype, b200collStream_t stream) {
  const std::string who = "vocab-parallel embedding: ";
  size_t nr = 0;
  b200collResult_t rc = emb_check(c, who, true, ids, weight, out, tokens, hidden, vl, sp, dtype, dtype, &nr);
  if (rc != b200collSuccess) return rc;
  const bool local = c->nranks == 1;
  const b200collAlgo_t algo = local ? b200collAlgoCopy : b200collAlgoTwoShot;
  if (!local) {
    // B200COLL_CHECK=1: (T, H, Vl), then (dtype and SP flag, the weight's arena offset)
    if ((rc = cross_check(c, b200collOpAllGather, algo, tokens, hidden, vl)) != b200collSuccess) return rc;
    const size_t woff = tokens > 0 ? arena_off(c, weight) : 0;
    if ((rc = cross_check(c, b200collOpAllGather, algo, ((size_t)dtype << 1) | (sp ? 1 : 0), woff, 0)) != b200collSuccess) return rc;
  }
  const size_t es = b200collTypeSize(dtype);
  account(c, b200collOpAllGather, nr * hidden * es, algo);
  if (tokens == 0) return b200collSuccess;                          // the same on every rank: nothing to read or write, no peer waits
  EmbFwdArgs a = {};
  a.ids = ids;
  a.weight = local ? (unsigned long long)reinterpret_cast<uintptr_t>(weight) : (unsigned long long)arena_off(c, weight);
  a.out = static_cast<char*>(out);
  a.tok0 = (uint32_t)(sp ? (size_t)c->rank * nr : 0);
  a.nvec = fast_div((uint32_t)(hidden * es / 16));
  a.total = (uint32_t)(nr * a.nvec.d);
  a.nvocab = (uint32_t)((size_t)c->nranks * vl);
  a.vl = fast_div((uint32_t)vl);
  const DeviceScope on_device(c->device);
  embedding_preload(c);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint32_t op = (uint32_t)b200collOpAllGather;
  // the grid follows the shapes only (equal on every rank), as the barriers pair CTA b with CTA b
  const Grid g = pick_grid(c, kShapeP2p, a.total, kEmbUnroll);
  if (local) launch_k(k_emb_fwd<true>, g.blocks, g.threads, st, c->dev, a, op);
  else launch_k(k_emb_fwd<false>, g.blocks, g.threads, st, c->dev, a, op);
  LAUNCH_CHECK(c);
  return b200collSuccess;
}

static size_t emb_align16(size_t n) { return (n + 15) / 16 * 16; }

static b200collResult_t emb_backward(b200collComm* c, const int64_t* ids, const void* dout, void* dweight, size_t tokens, size_t hidden, size_t vl,
                                     int sp, b200collDataType_t dt_out, b200collDataType_t dt_w, int accumulate, b200collStream_t stream) {
  const std::string who = "vocab-parallel embedding backward: ";
  size_t nr = 0;
  b200collResult_t rc = emb_check(c, who, false, ids, dweight, dout, tokens, hidden, vl, sp, dt_out, dt_w, &nr);
  if (rc != b200collSuccess) return rc;
  const bool local = c->nranks == 1, peer = !local && sp && tokens > 0;
  const size_t tiles = (tokens + kEmbTile - 1) / kEmbTile;
  const size_t o_keys1 = emb_align16(tokens * 4), o_toks0 = 2 * o_keys1, o_toks1 = 3 * o_keys1, o_hist = 4 * o_keys1;
  const size_t o_bounds = o_hist + emb_align16(tiles * kEmbDigits * 4), need = o_bounds + emb_align16((vl + 1) * 4);
  size_t soff = 0;
  if (tokens > 0 && (rc = quant_scratch_take(c, need, "vocab-parallel embedding backward", &soff)) != b200collSuccess) return rc;
  const b200collAlgo_t algo = local ? b200collAlgoCopy : b200collAlgoTwoShot;
  if (!local) {
    // B200COLL_CHECK=1: (T, H, Vl), then (dtypes, SP flag, accumulate; dout's arena offset under SP; the scratch offset)
    if ((rc = cross_check(c, b200collOpAllGather, algo, tokens, hidden, vl)) != b200collSuccess) return rc;
    const size_t fmt = ((size_t)dt_w << 16) | ((size_t)dt_out << 8) | ((size_t)(accumulate ? 1 : 0) << 1) | (sp ? 1 : 0);
    if ((rc = cross_check(c, b200collOpAllGather, algo, fmt, peer ? arena_off(c, dout) : 0, soff)) != b200collSuccess) return rc;
  }
  if (peer) account(c, b200collOpAllGather, nr * hidden * b200collTypeSize(dt_out), algo);
  const size_t er = b200collTypeSize(dt_out);
  EmbBwdArgs a = {};
  a.dout = peer ? (unsigned long long)arena_off(c, dout) : (unsigned long long)reinterpret_cast<uintptr_t>(dout);
  a.dweight = static_cast<char*>(dweight);
  a.nvd = fast_div((uint32_t)(hidden * er / 16));
  a.total = (uint32_t)(vl * a.nvd.d);
  a.accumulate = accumulate ? 1u : 0u;
  a.shard = fast_div((uint32_t)std::max<size_t>(nr, 1));
  const DeviceScope on_device(c->device);
  embedding_preload(c);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (tokens > 0) {
    char* base = static_cast<char*>(c->quant_scratch);            // this rank's view of the scratch (soff is its arena offset)
    uint32_t* keys[2] = {reinterpret_cast<uint32_t*>(base), reinterpret_cast<uint32_t*>(base + o_keys1)};
    uint32_t* toks[2] = {reinterpret_cast<uint32_t*>(base + o_toks0), reinterpret_cast<uint32_t*>(base + o_toks1)};
    uint32_t* hist = reinterpret_cast<uint32_t*>(base + o_hist);
    uint32_t* bounds = reinterpret_cast<uint32_t*>(base + o_bounds);
    int bits = 0;
    while (bits < 32 && (vl >> bits) != 0) bits++;                  // keys run to vl (not owned)
    const int passes = (bits + 7) / 8;
    EmbSortArgs s = {};
    s.ids = ids;
    s.start = (int64_t)c->rank * (int64_t)vl;
    s.tokens = (uint32_t)tokens;
    s.vl = (uint32_t)vl;
    s.tiles = (uint32_t)tiles;
    s.hist = hist;
    for (int p = 0; p < passes; p++) {
      s.shift = (uint32_t)(8 * p);
      s.keys_in = keys[(p + 1) & 1];
      s.toks_in = toks[(p + 1) & 1];
      s.keys_out = keys[p & 1];
      s.toks_out = toks[p & 1];
      if (p == 0) launch_k(k_emb_hist<true>, (int)tiles, kEmbSortThreads, st, s);
      else launch_k(k_emb_hist<false>, (int)tiles, kEmbSortThreads, st, s);
      LAUNCH_CHECK(c);
      launch_k(k_emb_scan, 1, kEmbScanThreads, st, hist, (uint32_t)(tiles * kEmbDigits));
      LAUNCH_CHECK(c);
      if (p == 0) launch_k(k_emb_scatter<true>, (int)tiles, kEmbSortThreads, st, s);
      else launch_k(k_emb_scatter<false>, (int)tiles, kEmbSortThreads, st, s);
      LAUNCH_CHECK(c);
    }
    const int last = (passes - 1) & 1;
    const int bb = (int)std::max<size_t>(1, std::min<size_t>((vl + 1 + 255) / 256, (size_t)std::max(1, c->sm_count) * 8));
    launch_k(k_emb_bounds, bb, 256, st, static_cast<const uint32_t*>(keys[last]), (uint32_t)tokens, (uint32_t)vl, bounds);
    LAUNCH_CHECK(c);
    a.toks = toks[last];
    a.bounds = bounds;
  }
  // warp items of 32 vectors; the grid follows the shapes only (equal on every rank), as the barriers pair CTA b with CTA b
  Grid g = warp_grid(c, ((size_t)a.total + 31) / 32 * 32);
  const uint32_t op = (uint32_t)b200collOpAllGather;
  return with_wide(dt_out, [&](auto td) -> b200collResult_t {
    using TD = typename decltype(td)::type;
    if (dt_w == b200collFloat32) {
      if (peer) launch_k(k_emb_bwd<TD, float, true>, g.blocks, g.threads, st, c->dev, a, op);
      else launch_k(k_emb_bwd<TD, float, false>, g.blocks, g.threads, st, c->dev, a, op);
    } else {
      if (peer) launch_k(k_emb_bwd<TD, TD, true>, g.blocks, g.threads, st, c->dev, a, op);
      else launch_k(k_emb_bwd<TD, TD, false>, g.blocks, g.threads, st, c->dev, a, op);
    }
    LAUNCH_CHECK(c);
    return b200collSuccess;
  });
}

}  // namespace b200coll

using namespace b200coll;

extern "C" {

b200collResult_t b200collVocabParallelEmbedding(const int64_t* ids, const void* weight, void* out, size_t tokens, size_t hidden, size_t vocab_local,
                                                int sequence_parallel, b200collDataType_t dtype, b200collComm_t comm, b200collStream_t stream) {
  return emb_forward(comm, ids, weight, out, tokens, hidden, vocab_local, sequence_parallel, dtype, stream);
}

b200collResult_t b200collVocabParallelEmbeddingBackward(const int64_t* ids, const void* dout, void* dweight, size_t tokens, size_t hidden,
                                                        size_t vocab_local, int sequence_parallel, b200collDataType_t dout_dtype,
                                                        b200collDataType_t dweight_dtype, int accumulate, b200collComm_t comm,
                                                        b200collStream_t stream) {
  return emb_backward(comm, ids, dout, dweight, tokens, hidden, vocab_local, sequence_parallel, dout_dtype, dweight_dtype, accumulate, stream);
}

}  // extern "C"
