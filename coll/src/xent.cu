// libb200coll vocab-parallel cross-entropy for tensor-parallel LM heads (b200collVocabParallelCrossEntropy / ...Backward): each rank
// holds the logits of a slice of the vocabulary, and one kernel per direction turns them into the loss, its log-sum-exp and the
// gradient:
//
//   k_xent<T, LOCAL>    relaxed barrier, per row: the NaN-aware max m_r of this rank's slice, s_r = sum exp(x - m_r) in the header's
//                       chunk-and-fold order, the target logit z_r if this rank owns the target; (m_r, s_r, z_r, owns) pushed as one
//                       16-byte record into the row's slot of every rank's mailbox; releasing barrier; then every rank combines the N
//                       records of each row in rank order into lse and loss. LOCAL: one rank, the one record combined at once, no
//                       barrier and no mailbox.
//   k_xent_bwd<T>       grad = round_T((exp(x - lse) - [col == target]) * dloss), one elementwise pass, no communication; grad may be
//                       the logits themselves (each element is read and then written by the same thread).
//
// exp and log. xent_exp and xent_log below are part of the result: fixed sequences of IEEE fp32 multiplies and adds (every one
// __fmul_rn / __fadd_rn, so nothing is contracted into an FMA), rint and exponent-bit arithmetic, no MUFU approximation, so that the
// numpy reference (tests/coll_xent_reference.py) computes the same bits on the CPU. exp is a Cody-Waite reduction by ln 2 (the high part
// of ln 2 has 9 significant bits, so k * ln2_hi is exact for every k that reaches it and x - k * ln2_hi is exact by Sterbenz) and a
// degree-5 Horner polynomial (Cephes' expf coefficients); log splits off the exponent around sqrt(1/2) and evaluates Cephes' logf
// polynomial. Both are within 1 ulp of the float64 value on [-87, 88.72] and on the positive normal numbers (the CPU tests check exp
// exhaustively on [-87, 0] and log on [1, 4)); exp(0) == 1 and log(1) == 0 exactly.
//
// One CTA owns one row at a time (rows b, b + grid, ... on every rank: the mailbox slot of a row is filled by CTA b of every rank, and
// the releasing barrier pairs exactly those CTAs). Pass 1 reads the row once from HBM with four 16-byte loads in flight per thread,
// keeps the max, and, when the row fits (at most kXeStageMax bytes of shared memory with the fold's stack: 100 K bf16 columns, so every
// Megatron TP slice of Llama-3's or Qwen's vocabulary from TP = 2 on), copies it into shared memory; pass 2 reads it back from there. A
// row that does not fit (one rank with a 128K or 152K bf16 vocabulary) is read from global memory again: the second read of a row comes
// a few microseconds after the first, and whether it still hits L2 depends on how many rows are in flight (bench/vocab_xent_perf.py
// measures it).
//
// The order of the sum does not depend on the launch shape. The header pads the C chunk sums p[c] with +0 to a power of two P and folds
// p[:P/2] + p[P/2:] until one value is left, i.e. index bits from the highest down. Thread t takes the chunks c = t + 512 j, so the bits
// of j are the high bits: a thread folds its own J = P / 512 chunk sums first, visiting j in bit-reversed order with a binary counter
// (stack level l of thread t in shared memory), which is exactly the MSB-first fold of its J values; then bits 8..5 across the 16 warps
// through shared memory and bits 4..0 in the lane butterfly, as rmsnorm.cu's fold. When P < 512, the extra levels add +0 to chunk sums
// that are never -0, which changes nothing. A chunk past the row's end is padded with -inf columns, whose exp is +0.
//
// Ordering. The entry barrier is relaxed: a rank arrives once its stream has reached this call, so every earlier reader of its mailbox
// (the previous call's combine, or a quantising collective that shares the scratch) is done before a peer pushes into it. The releasing
// barrier publishes the records. Nothing else crosses ranks: the logits, target, loss and lse are read and written by their own rank
// only, so no closing barrier is needed, and the next call's entry barrier frees the mailbox again.
#include <stdint.h>

#include <atomic>
#include <cmath>
#include <mutex>
#include <string>

#include "comm.h"
#include "launch.cuh"

namespace b200coll {

constexpr int kXeThreads = 512, kXeWarps = kXeThreads / 32;   // the fold below is written for 16 warps
constexpr int kXeUnroll = 4;
constexpr size_t kXeStageMax = 200 << 10;                      // dynamic shared memory: the fold's stack and the staged row

// ---------------------------------------------------------------- exp and log (mirrored by tests/coll_xent_reference.py)
__device__ __forceinline__ float xent_exp(float x) {
  const float kf = rintf(__fmul_rn(x, 1.44269504088896341f));
  const float r = __fsub_rn(__fsub_rn(x, __fmul_rn(kf, 0.693359375f)), __fmul_rn(kf, -2.12194440e-4f));
  const float z = __fmul_rn(r, r);
  float p = 1.9875691500e-4f;
  p = __fadd_rn(__fmul_rn(p, r), 1.3981999507e-3f);
  p = __fadd_rn(__fmul_rn(p, r), 8.3334519073e-3f);
  p = __fadd_rn(__fmul_rn(p, r), 4.1665795894e-2f);
  p = __fadd_rn(__fmul_rn(p, r), 1.6666665459e-1f);
  p = __fadd_rn(__fmul_rn(p, r), 5.0000001201e-1f);
  const float y = __fadd_rn(__fadd_rn(__fmul_rn(p, z), r), 1.0f);
  // y * 2^k through the exponent field; NaN converts to k = 0 and stays NaN; the selects take the range ends (and +-inf)
  const float v = __int_as_float(__float_as_int(y) + (__float2int_rn(kf) << 23));
  return x < -87.0f ? 0.0f : (x > 88.7228317f ? __int_as_float(0x7F800000) : v);
}

__device__ __forceinline__ float xent_log(float x) {
  const int bits = __float_as_int(x);
  const int e = (bits - 0x3F3504F3) >> 23;                     // x = 2^e * m, m in [sqrt(1/2), sqrt(2))
  const float f = __fsub_rn(__int_as_float(bits - (e << 23)), 1.0f);
  const float z = __fmul_rn(f, f);
  float q = 7.0376836292e-2f;
  q = __fadd_rn(__fmul_rn(q, f), -1.1514610310e-1f);
  q = __fadd_rn(__fmul_rn(q, f), 1.1676998740e-1f);
  q = __fadd_rn(__fmul_rn(q, f), -1.2420140846e-1f);
  q = __fadd_rn(__fmul_rn(q, f), 1.4249322787e-1f);
  q = __fadd_rn(__fmul_rn(q, f), -1.6668057665e-1f);
  q = __fadd_rn(__fmul_rn(q, f), 2.0000714765e-1f);
  q = __fadd_rn(__fmul_rn(q, f), -2.4999993993e-1f);
  q = __fadd_rn(__fmul_rn(q, f), 3.3333331174e-1f);
  const float ef = (float)e;
  float y = __fmul_rn(__fmul_rn(q, f), z);
  y = __fadd_rn(y, __fmul_rn(ef, -2.12194440e-4f));
  y = __fadd_rn(y, __fmul_rn(-0.5f, z));
  const float v = __fadd_rn(__fadd_rn(f, y), __fmul_rn(ef, 0.693359375f));
  if (x != x || x < 0.0f) return __int_as_float(0x7FFFFFFF);
  if (x == 0.0f) return __int_as_float(0xFF800000);
  return x == __int_as_float(0x7F800000) ? x : v;
}

// max that returns NaN when either input is NaN (fmaxf would drop it)
__device__ __forceinline__ float xent_max(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

// The 16-byte word of -inf columns in T: pads the last chunk of a row
template <typename T> __device__ __forceinline__ uint32_t xent_neg_inf_word() {
  if constexpr (std::is_same<T, float>::value) return 0xFF800000u;
  else if constexpr (std::is_same<T, __half>::value) return 0xFC00FC00u;
  else return 0xFF80FF80u;
}

// one 16-byte vector of T widened to fp32 bit for bit
template <typename T> __device__ __forceinline__ void xent_widen(const uint4& v, float* x) {
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

struct XeRec { float m, s, z; uint32_t owns; };               // one rank's record of one row: 16 bytes
static_assert(sizeof(XeRec) == 16, "one 16-byte store per record");

struct XeArgs {
  const char* logits;                 // [rows, vl] of T
  const int64_t* target;
  float* loss;
  float* lse;
  const float* dloss;                 // backward
  char* grad;                         // backward
  unsigned long long mbox_off;        // the mailbox [rows][nranks] records: its arena offset
  int64_t ignore_index;
  uint32_t rows, vl, nvec, nchunks;   // nvec 16-byte vectors and nchunks 16-element chunks per row
  uint32_t lj;                        // log2(chunks per thread), 0 when the row has at most 512 chunks
  uint32_t stage;                     // 1: the row is staged in shared memory between the passes
};

// loss and lse of one row from its N records, in rank order (the header's step 2). get(r) returns rank r's record; the loops are unrolled
// over kMaxRanks so that nothing is indexed at run time (no stack).
template <int R, typename Get>
__device__ __forceinline__ void xent_combine(Get get, uint32_t n, int64_t tgt, const XeArgs& a, uint32_t row) {
  float M = get(0).m;
#pragma unroll
  for (int r = 1; r < R; r++) if ((uint32_t)r < n) M = xent_max(M, get(r).m);
  float S = 0.0f, z = 0.0f;
#pragma unroll
  for (int r = 0; r < R; r++) {
    if ((uint32_t)r < n) {
      const XeRec q = get(r);
      const float e = q.m == __int_as_float(0xFF800000) ? 0.0f : __fmul_rn(q.s, xent_exp(__fsub_rn(q.m, M)));
      S = __fadd_rn(S, e);
      if (q.owns) z = q.z;
    }
  }
  const float lse = __fadd_rn(M, xent_log(S));
  float loss = __fsub_rn(lse, z);
  if (tgt == a.ignore_index) loss = 0.0f;
  else if (tgt < 0 || tgt >= (int64_t)n * a.vl) loss = __int_as_float(0x7FFFFFFF);
  a.loss[row] = loss;
  a.lse[row] = lse;
}

// This rank's record of one row, valid in thread 0. stack: (lj + 1) * 512 floats; stage: the row's bytes (when a.stage).
template <typename T>
__device__ __forceinline__ XeRec xent_partial(const XeArgs& a, uint32_t me, uint32_t row, float* stack, char* stage, float* red, float* fold) {
  constexpr int E = Epv<T>::value, K = (int)sizeof(T);       // elements per vector, vectors per 16-element chunk
  const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const char* x = a.logits + (size_t)row * a.nvec * 16;        // 64-bit: rows * row bytes passes 2^32
  // pass 1: the max, the row staged on the way
  float mx = __int_as_float(0xFF800000);
  for (uint32_t base = t; base < a.nvec; base += kXeThreads * kXeUnroll) {
    uint4 w[kXeUnroll];
#pragma unroll
    for (int u = 0; u < kXeUnroll; u++) {
      const uint32_t v = base + (uint32_t)u * kXeThreads;
      if (v < a.nvec) w[u] = ld_vec(x + 16ull * v);
    }
#pragma unroll
    for (int u = 0; u < kXeUnroll; u++) {
      const uint32_t v = base + (uint32_t)u * kXeThreads;
      if (v < a.nvec) {
        if (a.stage) *reinterpret_cast<uint4*>(stage + 16ull * v) = w[u];
        float f[E];
        xent_widen<T>(w[u], f);
#pragma unroll
        for (int i = 0; i < E; i++) mx = xent_max(mx, f[i]);
      }
    }
  }
#pragma unroll
  for (int l = 16; l >= 1; l >>= 1) mx = xent_max(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, l));
  if (lane == 0) red[warp] = mx;
  __syncthreads();                                             // also: the staged row is complete
  float m = red[0];
#pragma unroll
  for (int i = 1; i < kXeWarps; i++) m = xent_max(m, red[i]);
  // pass 2: chunk sums of exp(x - m), folded MSB first; m == -inf (the whole slice -inf) gives s = +0
  float p = 0.0f;
  if (m != __int_as_float(0xFF800000)) {
    const uint32_t J = 1u << a.lj;
    for (uint32_t k = 0; k < J; k++) {
      const uint32_t j = a.lj ? __brev(k) >> (32 - a.lj) : 0u;
      const uint32_t c = t + (uint32_t)kXeThreads * j;
      p = 0.0f;
      if (c < a.nchunks) {
        float f[16];
#pragma unroll
        for (int q = 0; q < K; q++) {
          const uint32_t v = c * (uint32_t)K + (uint32_t)q;
          uint4 w;
          if (v >= a.nvec) {
            const uint32_t ni = xent_neg_inf_word<T>();
            w = make_uint4(ni, ni, ni, ni);
          } else if (a.stage) {
            w = *reinterpret_cast<const uint4*>(stage + 16ull * v);
          } else {
            w = ld_vec(x + 16ull * v);
          }
          xent_widen<T>(w, f + q * E);
        }
#pragma unroll
        for (int i = 0; i < 16; i++) p = __fadd_rn(p, xent_exp(__fsub_rn(f[i], m)));
      }
      uint32_t l = 0;
      for (; (k >> l) & 1u; l++) p = __fadd_rn(stack[l * kXeThreads + t], p);     // the binary counter over bit-reversed j
      stack[l * kXeThreads + t] = p;
    }
  }
  // bits 8..5 across warps, 4..0 in the butterfly (rmsnorm.cu's fold)
  fold[t] = p;
  __syncthreads();
  float w[kXeWarps];
#pragma unroll
  for (int i = 0; i < kXeWarps; i++) w[i] = fold[32 * i + lane];
#pragma unroll
  for (int i = 0; i < 8; i++) w[i] = __fadd_rn(w[i], w[i + 8]);
#pragma unroll
  for (int i = 0; i < 4; i++) w[i] = __fadd_rn(w[i], w[i + 4]);
  w[0] = __fadd_rn(w[0], w[2]); w[1] = __fadd_rn(w[1], w[3]);
  float s = __fadd_rn(w[0], w[1]);
#pragma unroll
  for (int l = 4; l >= 0; l--) s = __fadd_rn(s, __shfl_xor_sync(0xFFFFFFFFu, s, 1 << l));
  XeRec rec = {m, s, 0.0f, 0u};
  if (t == 0) {
    const int64_t col = a.target[row] - (int64_t)me * a.vl;
    if (col >= 0 && col < (int64_t)a.vl) {
      rec.z = to_float<T>(*reinterpret_cast<const T*>(x + (size_t)col * sizeof(T)));   // exact: -0 and NaN payloads survive
      rec.owns = 1u;
    }
  }
  return rec;
}

template <typename T, bool LOCAL>
__global__ void __launch_bounds__(kXeThreads, 1) k_xent(COMM_PARAM, const __grid_constant__ XeArgs a, uint32_t op) {
  pdl_prologue();
  extern __shared__ float4 xe_dyn[];
  __shared__ float red[kXeWarps];
  __shared__ float fold[kXeThreads];
  float* stack = reinterpret_cast<float*>(xe_dyn);
  char* stage = reinterpret_cast<char*>(stack + (a.lj + 1) * kXeThreads);
  uint32_t s = 0;
  if (!LOCAL) {
    s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;      // every rank is done with the previous contents of its mailbox
  }
  const uint32_t me = LOCAL ? 0u : (uint32_t)c.rank, nr = LOCAL ? 1u : (uint32_t)c.nranks;
  for (uint32_t row = blockIdx.x; row < a.rows; row += gridDim.x) {
    const XeRec rec = xent_partial<T>(a, me, row, stack, stage, red, fold);
    if (threadIdx.x == 0) {
      if (LOCAL) {
        xent_combine<1>([&](int) { return rec; }, 1, a.target[row], a, row);
      } else {
        const uint4 w = make_uint4(__float_as_uint(rec.m), __float_as_uint(rec.s), __float_as_uint(rec.z), rec.owns);
        const unsigned long long off = a.mbox_off + 16ull * ((unsigned long long)row * nr + me);
#pragma unroll 1
        for (uint32_t k = 1; k <= nr; k++) {
          uint32_t p = me + k; if (p >= nr) p -= nr;
          st_vec(c.peer[p] + off, w);
        }
      }
    }
  }
  if (!LOCAL) {
    if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;        // every rank's records of my rows are in my mailbox
    const char* mbox = c.peer[me] + a.mbox_off;
    for (uint32_t row = blockIdx.x + gridDim.x * threadIdx.x; row < a.rows; row += gridDim.x * blockDim.x) {
      const char* slot = mbox + 16ull * ((unsigned long long)row * nr);
      auto get = [&](int r) {
        const uint4 w = ld_vec(slot + 16 * r);
        return XeRec{__uint_as_float(w.x), __uint_as_float(w.y), __uint_as_float(w.z), w.w};
      };
      xent_combine<kMaxRanks>(get, nr, a.target[row], a, row);
    }
    if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
  }
}

template <typename T>
__global__ void __launch_bounds__(kXeThreads) k_xent_bwd(COMM_PARAM, const __grid_constant__ XeArgs a) {
  pdl_prologue();
  constexpr int E = Epv<T>::value;
  const int64_t nvocab = (int64_t)c.nranks * a.vl;
  for (uint32_t row = blockIdx.x; row < a.rows; row += gridDim.x) {
    const int64_t tgt = a.target[row];
    const bool ignored = tgt == a.ignore_index, bad = !ignored && (tgt < 0 || tgt >= nvocab);
    const int64_t col = tgt - (int64_t)c.rank * a.vl;          // this rank's column of the target (outside [0, vl): none)
    const float lse = a.lse[row], dl = a.dloss[row];
    const char* x = a.logits + (size_t)row * a.nvec * 16;
    char* g = a.grad + (size_t)row * a.nvec * 16;
    for (uint32_t base = threadIdx.x; base < a.nvec; base += blockDim.x * kXeUnroll) {
      uint4 w[kXeUnroll];
      if (!ignored && !bad) {
#pragma unroll
        for (int u = 0; u < kXeUnroll; u++) {
          const uint32_t v = base + (uint32_t)u * blockDim.x;
          if (v < a.nvec) w[u] = ld_vec(x + 16ull * v);
        }
      }
#pragma unroll
      for (int u = 0; u < kXeUnroll; u++) {
        const uint32_t v = base + (uint32_t)u * blockDim.x;
        if (v >= a.nvec) continue;
        float f[E];
        if (ignored || bad) {
#pragma unroll
          for (int i = 0; i < E; i++) f[i] = ignored ? 0.0f : __int_as_float(0x7FFFFFFF);
        } else {
          xent_widen<T>(w[u], f);
#pragma unroll
          for (int i = 0; i < E; i++) {
            float d = xent_exp(__fsub_rn(f[i], lse));
            if ((int64_t)v * E + i == col) d = __fsub_rn(d, 1.0f);
            f[i] = __fmul_rn(d, dl);
          }
        }
        uint32_t o[Pack<T, E>::W];
        Pack<T, E>::run(f, o);
        st_words<Pack<T, E>::W>(g + 16ull * v, o);
      }
    }
  }
}

// Once per device: load the nine kernels (see shards_preload: a first launch queued behind a peer-waiting barrier kernel would never
// load with lazy module loading and virtual ranks) and allow the forward kernels kXeStageMax bytes of dynamic shared memory.
static void xent_preload(const b200collComm* c) {
  static std::atomic<unsigned long long> done{0};
  static std::mutex mu;
  const unsigned long long bit = 1ull << (c->device & 63);
  if (done.load(std::memory_order_acquire) & bit) return;
  const std::lock_guard<std::mutex> lk(mu);
  if (done.load(std::memory_order_acquire) & bit) return;
  cudaFuncAttributes fa;
  for (b200collDataType_t t : {b200collBfloat16, b200collFloat16, b200collFloat32})
    with_wide(t, [&](auto tt) {
      using T = typename decltype(tt)::type;
      cudaFuncGetAttributes(&fa, k_xent<T, true>);
      cudaFuncGetAttributes(&fa, k_xent<T, false>);
      cudaFuncGetAttributes(&fa, k_xent_bwd<T>);
      cudaFuncSetAttribute(k_xent<T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kXeStageMax);
      cudaFuncSetAttribute(k_xent<T, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kXeStageMax);
    });
  done.fetch_or(bit, std::memory_order_acq_rel);
}

// The argument rules of both calls, before the poisoned-communicator check; nothing is launched on a refusal.
static b200collResult_t xent_check(b200collComm* c, const char* who, const void* logits, const int64_t* target, size_t rows, size_t vl,
                                   b200collDataType_t dtype, std::initializer_list<std::pair<const void*, size_t>> outs,
                                   std::initializer_list<std::pair<const void*, size_t>> ins, const void* grad) {
  auto refuse = [&](const std::string& msg) { set_last_error(std::string(who) + msg); return b200collInvalidArgument; };
  if (!c) return refuse("null communicator");
  if (!wide_type(dtype)) return refuse("dtype must be bf16, fp16 or fp32");
  const size_t es = b200collTypeSize(dtype);
  if (vl == 0 || (vl * es) % 16 != 0) return refuse("vocab_local must be positive and vocab_local * sizeof(dtype) a multiple of 16 bytes");
  if (vl >= ((size_t)1 << 31) / (size_t)c->nranks || (size_t)c->nranks * vl >= ((size_t)1 << 31)) return refuse("nranks * vocab_local must be below 2^31");
  if (rows >= ((size_t)1 << 31)) return refuse("rows must be below 2^31");
  if (rows > 0) {
    if (!logits || !target) return refuse("null argument");
    for (const auto& b : outs) if (!b.first) return refuse("null argument");
    for (const auto& b : ins) if (!b.first) return refuse("null argument");
  }
  if (!aligned(logits, 16) || (grad && !aligned(grad, 16))) return refuse("logits and grad must be 16-byte aligned");
  if (!aligned(target, 8)) return refuse("target must be 8-byte aligned");
  for (const auto& b : outs) if (b.first != grad && !aligned(b.first, 4)) return refuse("loss, lse and dloss must be 4-byte aligned");
  for (const auto& b : ins) if (!aligned(b.first, 4)) return refuse("loss, lse and dloss must be 4-byte aligned");
  if (rows > 0) {
    const size_t mat = rows * vl * es;
    const std::pair<const void*, size_t> all_in[] = {{logits, mat}, {target, rows * 8}};
    for (auto o = outs.begin(); o != outs.end(); ++o) {
      for (const auto& i : all_in)
        if (overlaps(o->first, o->second, i.first, i.second) && !(o->first == grad && grad == logits && i.first == logits))
          return refuse("outputs must not overlap the inputs (grad == logits is the one overlap allowed)");
      for (const auto& i : ins)
        if (overlaps(o->first, o->second, i.first, i.second)) return refuse("outputs must not overlap the inputs (grad == logits is the one overlap allowed)");
      for (auto p = o + 1; p != outs.end(); ++p)
        if (overlaps(o->first, o->second, p->first, p->second)) return refuse("outputs must not overlap each other");
    }
  }
  if (comm_poisoned(c)) return b200collRemoteError;
  return b200collSuccess;
}

static b200collResult_t xent_forward(b200collComm* c, const void* logits, const int64_t* target, float* loss, float* lse, size_t rows,
                                     size_t vl, int64_t ignore_index, b200collDataType_t dtype, b200collStream_t stream) {
  const char* who = "vocab-parallel cross-entropy: ";
  b200collResult_t rc = xent_check(c, who, logits, target, rows, vl, dtype, {{loss, rows * 4}, {lse, rows * 4}}, {}, nullptr);
  if (rc != b200collSuccess) return rc;
  const bool local = c->nranks == 1;
  const size_t N = (size_t)c->nranks;
  size_t mbox_off = 0;
  if (!local && rows > 0 && (rc = quant_scratch_take(c, rows * N * sizeof(XeRec), "vocab-parallel cross-entropy", &mbox_off)) != b200collSuccess)
    return rc;
  const b200collAlgo_t algo = local ? b200collAlgoCopy : b200collAlgoTwoShot;
  if (!local) {
    // B200COLL_CHECK=1: (rows, vocab_local, mailbox offset), then (dtype, ignore_index)
    if ((rc = cross_check(c, b200collOpAllReduce, algo, rows, vl, mbox_off)) != b200collSuccess) return rc;
    if ((rc = cross_check(c, b200collOpAllReduce, algo, (size_t)dtype, (size_t)ignore_index, 0)) != b200collSuccess) return rc;
  }
  XeArgs a = {};
  a.logits = static_cast<const char*>(logits);
  a.target = target;
  a.loss = loss;
  a.lse = lse;
  a.mbox_off = mbox_off;
  a.ignore_index = ignore_index;
  a.rows = (uint32_t)rows;
  a.vl = (uint32_t)vl;
  a.nvec = (uint32_t)(vl * b200collTypeSize(dtype) / 16);
  a.nchunks = (uint32_t)((vl + 15) / 16);
  uint32_t P = 1;
  while (P < a.nchunks) P <<= 1;
  while (P > (uint32_t)kXeThreads << a.lj) a.lj++;
  const size_t stack_bytes = (size_t)(a.lj + 1) * kXeThreads * 4, row_bytes = (size_t)a.nvec * 16;
  a.stage = stack_bytes + row_bytes <= kXeStageMax ? 1u : 0u;
  const size_t smem = stack_bytes + (a.stage ? row_bytes : 0);
  // one CTA per row at a time: as many as fit on the device (one rank; at most twice the communicator's CTA cap), or the P2P shape, the same on every rank (the barrier pairs CTA b
  // of every rank); never more than the rows, at least one (rows == 0 still takes part in the barriers)
  int blocks;
  if (local) {
    const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(2048 / kXeThreads, (227u << 10) / (smem + (3u << 10))));
    const size_t cap = std::min<size_t>((size_t)std::max(1, c->sm_count) * per_sm, 2 * (size_t)std::max(1, c->max_ctas));
    blocks = (int)std::max<size_t>(1, std::min<size_t>(rows, cap));
  } else {
    blocks = (int)std::max<size_t>(1, std::min<size_t>(rows, (size_t)full_grid(c, 1).blocks));
  }
  const DeviceScope on_device(c->device);
  xent_preload(c);
  account(c, b200collOpAllReduce, rows * sizeof(XeRec), algo);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint32_t op = (uint32_t)b200collOpAllReduce;
  return with_wide(dtype, [&](auto tt) -> b200collResult_t {
    using T = typename decltype(tt)::type;
    if (local) launch_k_smem(k_xent<T, true>, blocks, kXeThreads, smem, st, c->dev, a, op);
    else launch_k_smem(k_xent<T, false>, blocks, kXeThreads, smem, st, c->dev, a, op);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  });
}

static b200collResult_t xent_backward(b200collComm* c, const void* logits, const int64_t* target, const float* lse, const float* dloss, void* grad,
                                      size_t rows, size_t vl, int64_t ignore_index, b200collDataType_t dtype, b200collStream_t stream) {
  const char* who = "vocab-parallel cross-entropy backward: ";
  const size_t es = (c && wide_type(dtype)) ? b200collTypeSize(dtype) : 1;
  const b200collResult_t rc = xent_check(c, who, logits, target, rows, vl, dtype, {{grad, rows * vl * es}}, {{lse, rows * 4}, {dloss, rows * 4}}, grad);
  if (rc != b200collSuccess) return rc;
  XeArgs a = {};
  a.logits = static_cast<const char*>(logits);
  a.target = target;
  a.lse = const_cast<float*>(lse);
  a.dloss = dloss;
  a.grad = static_cast<char*>(grad);
  a.ignore_index = ignore_index;
  a.rows = (uint32_t)rows;
  a.vl = (uint32_t)vl;
  a.nvec = (uint32_t)(vl * es / 16);
  if (rows == 0) return b200collSuccess;                         // nothing to read or write, no peer waits
  const int threads = (int)std::min<size_t>(kXeThreads, std::max<size_t>(32, ((size_t)a.nvec + 31) / 32 * 32));
  const int blocks = (int)std::max<size_t>(1, std::min<size_t>(rows, (size_t)std::max(1, c->sm_count) * (2048 / threads)));
  const DeviceScope on_device(c->device);
  xent_preload(c);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return with_wide(dtype, [&](auto tt) -> b200collResult_t {
    using T = typename decltype(tt)::type;
    launch_k(k_xent_bwd<T>, blocks, threads, st, c->dev, a);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  });
}

}  // namespace b200coll

using namespace b200coll;

extern "C" {

b200collResult_t b200collVocabParallelCrossEntropy(const void* logits, const int64_t* target, float* loss, float* lse, size_t rows,
                                                   size_t vocab_local, int64_t ignore_index, b200collDataType_t dtype, b200collComm_t comm,
                                                   b200collStream_t stream) {
  return xent_forward(comm, logits, target, loss, lse, rows, vocab_local, ignore_index, dtype, stream);
}

b200collResult_t b200collVocabParallelCrossEntropyBackward(const void* logits, const int64_t* target, const float* lse, const float* dloss,
                                                           void* grad, size_t rows, size_t vocab_local, int64_t ignore_index,
                                                           b200collDataType_t dtype, b200collComm_t comm, b200collStream_t stream) {
  return xent_backward(comm, logits, target, lse, dloss, grad, rows, vocab_local, ignore_index, dtype, stream);
}

}  // extern "C"
