// libb200coll fused all-reduce, residual add and RMSNorm (b200collAllReduceRmsNorm): the step that follows the attention output projection
// and the MLP down projection of every pre-norm tensor-parallel block, one kernel per call:
//
//   k_rms_local<T>       one rank: residual = h, out = norm(h) for every row, no barrier
//   k_rms_oneshot<T>     relaxed barrier, pull every row of every rank's x in rank order, store residual and out locally, releasing barrier
//   k_rms_twoshot<T>     relaxed barrier, pull my row slice, push its residual and out rows into every rank's residual and out, releasing
//                        barrier
//
// and the quantising call (b200collAllReduceRmsNormQuantized), the same three kernels with step 6 in place of the out store:
//
//   k_rmsq_local<T, WireT>, k_rmsq_oneshot<T, WireT>, k_rmsq_twoshot<T, WireT>
//                        o = round_T((h * inv) * gamma) quantised per block of the row with quant.cuh's quant_vec: q and the block scales
//                        stored locally, or (two-shot) pushed into every rank's q and scales
//
// and the reduce-scatter form for sequence parallelism (b200collReduceScatterRmsNorm, ...Quantized), where each rank holds only its
// shard of the residual stream, rows [rows*r/N, rows*(r+1)/N) (one rank: the local kernels above):
//
//   k_rs_norm<T, GATHER>, k_rs_normq<T, WireT, GATHER>
//                        two-shot's body: relaxed barrier, pull my row slice, read and write my residual shard locally at row - r0, store
//                        out (q, scales) locally at row - r0, or (GATHER) push it into every rank's out at row, releasing barrier
//
// One CTA (kRmsThreads threads) owns one row at a time, walking rows b, b + gridDim.x, ... of its range. Thread t holds the 16-element
// chunks t and t + kRmsThreads (row_len <= 16384 is at most 1024 chunks), so the new residual h of a whole row stays in registers
// between the sum and the normalisation.
//
// Order, and why the result does not depend on the launch shape. h[e] is (+0 + x_0[e]) + ... + x_{N-1}[e] + residual[e] in fp32, in that
// order, rounded once. The chunk sums p[c] add their 16 squares of the rounded h in element order from +0. The header's fold pads p with
// +0 to the next power of two P and halves it, p[i] + p[i + P/2]; this kernel pads to 1024 instead. Every p[c] is +0, positive, +inf or
// NaN (squares and their sums are never -0), and x + (+0) is exactly x for all of them, so the levels above P only add +0 to the values
// the header's fold starts from: the same bits. The levels then run in the same index order: chunk t + 512 onto chunk t in registers;
// bits 8..5 of the chunk index across the CTA's warps through shared memory, every warp folding all 512 values itself (so no second
// block barrier); bits 4..0 in the lane butterfly xor 16, 8, 4, 2, 1. Lane i of a butterfly step adds its partner's value to its own,
// so lanes above the partner add in the opposite order. IEEE addition is commutative and a NaN sum is the canonical NaN either way, so
// every lane ends with lane 0's bits. Every product and sum is __fmul_rn / __fadd_rn (no FFMA contraction), and ms, sqrt and 1 / sqrt
// are the correctly rounded __fdiv_rn and __fsqrt_rn.
//
// Ordering. The entry barrier is relaxed, as in the pull-reduce all-reduce: every x was written by an earlier kernel on its rank's stream,
// and a peer arrives only once its stream has reached this call. One-shot writes only its own residual and out. Two-shot writes rows of
// slice r only from rank r, into every rank's residual and out; rank p reads only the rows of slice p from its own residual, and a rank
// reaches the entry barrier only after everything earlier on its stream (a GEMM reading out) is done, so no store lands on a row that is
// still read. The closing barrier releases the two-shot stores to every rank and tells each rank that nobody pulls its x any more, so the
// caller may overwrite x right after the call. Both barriers pair CTA b with CTA b, and every rank launches full_grid's CTAs whatever its
// row count.
// The reduce-scatter kernels: rank r reads and writes only its own residual rows, so no other rank's store can meet them. With GATHER,
// rank r stores rows of slice r into every rank's out, and rank p reaches the entry barrier only after everything earlier on its stream
// (a GEMM reading out) is done: the same argument as two-shot's, so a peer's out rows are free. Without GATHER nothing is stored outside
// the rank. The closing barrier both publishes the pushed out rows and tells each rank that nobody pulls its x any more.
//
// Step 6. A quantising block is 1 to 32 chunks (16 to 512 elements, a power of two) and row_len is a multiple of it, so the chunks of
// one block are consecutive lanes of one warp (chunk t or t + 512 of thread t), starting on an aligned group of lanes: the contract of
// quant_vec. Lanes past the row pass zeros, and they make up whole groups; a warp wholly past the row skips the step. The lowest lane of
// each group stores the block's scale.
#include <stdint.h>

#include <atomic>
#include <mutex>
#include <string>

#include "comm.h"
#include "launch.cuh"
#include "quant.cuh"

namespace b200coll {

constexpr int kRmsThreads = 512, kRmsWarps = kRmsThreads / 32;       // the fold below is written for 16 warps
constexpr int kRmsMaxChunks = 2 * kRmsThreads;               // 16384 elements
constexpr size_t kRmsMaxRowLen = 16 * (size_t)kRmsMaxChunks;

// 16 elements of T at p, widened to fp32 bit for bit
template <typename T> __device__ __forceinline__ void rms_load16(const char* p, float* x) {
  uint4 raw[sizeof(T)];
#pragma unroll
  for (int k = 0; k < (int)sizeof(T); k++) raw[k] = ld_vec(p + 16 * k);
  widen16<T>(raw, x);
}

template <typename T> __device__ __forceinline__ float round_to(float v) {
  if constexpr (std::is_same<T, float>::value) return v;
  else return to_float<T>(from_float<T>(v));
}

// Where a kernel finds x, residual and out of row `row`. x_off: arena offset of x (every rank), read from peer 0 .. nranks-1 (one rank:
// x_local). res / out: local pointers, or (PUSH) arena offsets res_off / out_off stored into every rank.
struct RmsArgs {
  const char* x_local;
  const char* res_in;           // my residual, the rows I read
  char* res_out;                // my residual (local kernels) or nullptr (PUSH)
  char* out;                    // my out (local kernels) or nullptr (PUSH)
  const char* gamma;
  size_t x_off, res_off, out_off;
  uint32_t row_len, nchunks;
  float eps;
};

// What the quantising kernels add: where q and the scales of row `row` go, and the block. q: [rows, row_len] FP8, scales:
// [rows, row_len / block] fp32. Local pointers, or (PUSH) arena offsets q_off / s_off stored into every rank.
struct RmsQuant {
  char* q;
  char* scales;
  size_t q_off, s_off;
  uint32_t lvpb;                // log2(chunks per block)
};

// One row: h = round((+0 + x_0 + .. + x_{N-1}) + residual), residual = h, out = round((h * inv) * gamma), inv = 1 / sqrt(fold / row_len + eps).
// LOCAL: one rank, x is a.x_local; else rank r's x is at a.x_off of its arena. sbuf: this row's 512 floats of shared memory.
// WireT void: out is stored (qa unused); else out is quantised to WireT per block into qa's q and scales.
// x is read at row `row`. RES_PUSH: the residual is read locally and pushed into every rank at `row`; else read and written locally at
// `lrow`. OUT_PUSH: out (q, scales) pushed into every rank at `row`; else stored locally at `lrow`. The all-reduce kernels pass
// lrow == row; the reduce-scatter kernels pass the row's index in this rank's shard.
template <typename T, typename WireT, bool LOCAL, bool RES_PUSH, bool OUT_PUSH>
__device__ __forceinline__ void rms_row(const CommDev& c, const RmsArgs& a, const RmsQuant& qa, size_t row, size_t lrow, float* sbuf) {
  const int t = threadIdx.x, lane = t & 31;
  const size_t row_bytes = (size_t)a.row_len * sizeof(T);
  const size_t res_row = RES_PUSH ? row : lrow, out_row = OUT_PUSH ? row : lrow;
  float h[2][16];
  float p[2];
#pragma unroll
  for (int k = 0; k < 2; k++) {
    const uint32_t ch = (uint32_t)t + (uint32_t)k * kRmsThreads;
    p[k] = 0.f;
    if (ch < a.nchunks) {
      const size_t off = row * row_bytes + (size_t)ch * 16 * sizeof(T);
      float acc[16];
#pragma unroll
      for (int i = 0; i < 16; i++) acc[i] = 0.f;
#pragma unroll
      for (int r = 0; r < (LOCAL ? 1 : kMaxRanks); r++) {
        if (LOCAL || r < c.nranks) {
          float v[16];
          rms_load16<T>((LOCAL ? a.x_local : c.peer[r] + a.x_off) + off, v);
#pragma unroll
          for (int i = 0; i < 16; i++) acc[i] = __fadd_rn(acc[i], v[i]);
        }
      }
      const size_t roff = res_row * row_bytes + (size_t)ch * 16 * sizeof(T);
      float res[16];
      rms_load16<T>(a.res_in + roff, res);
#pragma unroll
      for (int i = 0; i < 16; i++) {
        h[k][i] = round_to<T>(__fadd_rn(acc[i], res[i]));
        p[k] = __fadd_rn(p[k], __fmul_rn(h[k][i], h[k][i]));
      }
      if (RES_PUSH) {
#pragma unroll
        for (int j = 0; j < kMaxRanks; j++) if (j < c.nranks) {
          int q = c.rank + j; if (q >= c.nranks) q -= c.nranks;
          store16_scaled<T>(c.peer[q] + a.res_off + roff, h[k], 1.0f);
        }
      } else {
        store16_scaled<T>(a.res_out + roff, h[k], 1.0f);
      }
    }
  }
  // the fold: bit 9 in registers, bits 8..5 across warps, bits 4..0 in the butterfly
  sbuf[t] = __fadd_rn(p[0], p[1]);
  __syncthreads();
  float w[kRmsWarps];
#pragma unroll
  for (int i = 0; i < kRmsWarps; i++) w[i] = sbuf[32 * i + lane];
#pragma unroll
  for (int i = 0; i < 8; i++) w[i] = __fadd_rn(w[i], w[i + 8]);
#pragma unroll
  for (int i = 0; i < 4; i++) w[i] = __fadd_rn(w[i], w[i + 4]);
  w[0] = __fadd_rn(w[0], w[2]); w[1] = __fadd_rn(w[1], w[3]);
  float f = __fadd_rn(w[0], w[1]);
#pragma unroll
  for (int l = 4; l >= 0; l--) f = __fadd_rn(f, __shfl_xor_sync(0xFFFFFFFFu, f, 1 << l));
  const float inv = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(__fdiv_rn(f, (float)a.row_len), a.eps)));
  if constexpr (std::is_void<WireT>::value) {
#pragma unroll
    for (int k = 0; k < 2; k++) {
      const uint32_t ch = (uint32_t)t + (uint32_t)k * kRmsThreads;
      if (ch < a.nchunks) {
        const size_t off = out_row * row_bytes + (size_t)ch * 16 * sizeof(T);
        float g[16], o[16];
        rms_load16<T>(a.gamma + (size_t)ch * 16 * sizeof(T), g);
#pragma unroll
        for (int i = 0; i < 16; i++) o[i] = __fmul_rn(__fmul_rn(h[k][i], inv), g[i]);
        if (OUT_PUSH) {
#pragma unroll
          for (int j = 0; j < kMaxRanks; j++) if (j < c.nranks) {
            int q = c.rank + j; if (q >= c.nranks) q -= c.nranks;
            store16_scaled<T>(c.peer[q] + a.out_off + off, o, 1.0f);
          }
        } else {
          store16_scaled<T>(a.out + off, o, 1.0f);
        }
      }
    }
  } else {
    // step 6, one chunk at a time: o as the wide call would store it, widened back, then quantised with its block's amax
    const uint32_t gl = 1u << qa.lvpb;
    const size_t q_row = out_row * a.row_len, s_row = out_row * (a.nchunks >> qa.lvpb);
#pragma unroll
    for (int k = 0; k < 2; k++) {
      const uint32_t ch = (uint32_t)t + (uint32_t)k * kRmsThreads;
      if ((ch & ~31u) >= a.nchunks) continue;                        // the whole warp is past the row
      const bool act = ch < a.nchunks;
      float o[16];
      if (act) {
        float g[16];
        rms_load16<T>(a.gamma + (size_t)ch * 16 * sizeof(T), g);
#pragma unroll
        for (int i = 0; i < 16; i++) o[i] = round_to<T>(__fmul_rn(__fmul_rn(h[k][i], inv), g[i]));
      } else {
#pragma unroll
        for (int i = 0; i < 16; i++) o[i] = 0.f;
      }
      float s;
      const uint4 w = quant_vec<WireT>(o, gl, &s);
      if (act) {
        const size_t q_off = q_row + (size_t)ch * 16, s_off = (s_row + (ch >> qa.lvpb)) * 4;
        const bool lead = (lane & (gl - 1)) == 0;
        if (OUT_PUSH) {
#pragma unroll
          for (int j = 0; j < kMaxRanks; j++) if (j < c.nranks) {
            int q = c.rank + j; if (q >= c.nranks) q -= c.nranks;
            st_vec(c.peer[q] + qa.q_off + q_off, w);
            if (lead) *reinterpret_cast<float*>(c.peer[q] + qa.s_off + s_off) = s;
          }
        } else {
          st_vec(qa.q + q_off, w);
          if (lead) *reinterpret_cast<float*>(qa.scales + s_off) = s;
        }
      }
    }
  }
}

// Rows [r0, r1), CTA b taking r0 + b, r0 + b + gridDim.x, ...; the shared buffer alternates by row so that one block barrier per row
// suffices (a warp that writes row i + 2's buffer has passed row i + 1's barrier, which every warp reaches only after reading row i's).
// Local buffers are indexed from `base`: row - base is the row's index in them.
template <typename T, typename WireT, bool LOCAL, bool RES_PUSH, bool OUT_PUSH>
__device__ __forceinline__ void rms_rows(const CommDev& c, const RmsArgs& a, const RmsQuant& qa, uint32_t r0, uint32_t r1, uint32_t base) {
  __shared__ float sbuf[2][kRmsThreads];
  uint32_t i = 0;
  for (uint32_t row = r0 + blockIdx.x; row < r1; row += gridDim.x, i ^= 1)
    rms_row<T, WireT, LOCAL, RES_PUSH, OUT_PUSH>(c, a, qa, row, row - base, sbuf[i]);
}

// The kernel bodies, shared by the wide kernels (WireT void) and the quantising ones.
template <typename T, typename WireT>
__device__ __forceinline__ void rms_local(const CommDev& c, const RmsArgs& a, const RmsQuant& qa, uint32_t rows) {
  pdl_prologue();
  rms_rows<T, WireT, true, false, false>(c, a, qa, 0, rows, 0);
}

template <typename T, typename WireT>
__device__ __forceinline__ void rms_oneshot(const CommDev& c, const RmsArgs& a, const RmsQuant& qa, uint32_t rows, uint32_t op) {
  pdl_prologue();
  {
    const uint32_t s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;        // every rank's x is written
  }
  rms_rows<T, WireT, false, false, false>(c, a, qa, 0, rows, 0);
  const uint32_t s = load_seq(c, kSeqBarrier);
  if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;           // nobody reads my x any more
  if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
}

template <typename T, typename WireT>
__device__ __forceinline__ void rms_twoshot(const CommDev& c, const RmsArgs& a, const RmsQuant& qa, uint32_t rows, uint32_t op) {
  pdl_prologue();
  {
    const uint32_t s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;        // every rank's x is written, and its residual and out (q, scales) are free
  }
  const uint32_t r0 = (uint32_t)((unsigned long long)rows * c.rank / c.nranks), r1 = (uint32_t)((unsigned long long)rows * (c.rank + 1) / c.nranks);
  rms_rows<T, WireT, false, true, true>(c, a, qa, r0, r1, 0);
  const uint32_t s = load_seq(c, kSeqBarrier);
  if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;           // my rows are in every rank's residual and out; nobody reads my x
  if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
}

// The reduce-scatter form: two-shot's slice, with my residual shard read and written locally at row - r0, and out (q, scales) stored
// locally at row - r0 or (GATHER) pushed into every rank at row.
template <typename T, typename WireT, bool GATHER>
__device__ __forceinline__ void rs_norm(const CommDev& c, const RmsArgs& a, const RmsQuant& qa, uint32_t rows, uint32_t op) {
  pdl_prologue();
  {
    const uint32_t s = load_seq(c, kSeqBarrier);
    if (!barrier_blocks<false>(c, 2 * s + 1, op)) return;        // every rank's x is written, and (GATHER) its out (q, scales) is free
  }
  const uint32_t r0 = (uint32_t)((unsigned long long)rows * c.rank / c.nranks), r1 = (uint32_t)((unsigned long long)rows * (c.rank + 1) / c.nranks);
  rms_rows<T, WireT, false, false, GATHER>(c, a, qa, r0, r1, r0);
  const uint32_t s = load_seq(c, kSeqBarrier);
  if (!barrier_blocks<true>(c, 2 * s + 2, op)) return;           // (GATHER) my rows are in every rank's out; nobody reads my x
  if (threadIdx.x == 0 && last_block_ticket(c)) c.state[kSeqBarrier] = s + 1;
}

template <typename T>
__global__ void __launch_bounds__(kRmsThreads, 1) k_rms_local(COMM_PARAM, const __grid_constant__ RmsArgs a, uint32_t rows) {
  rms_local<T, void>(c, a, RmsQuant{}, rows);
}

template <typename T>
__global__ void __launch_bounds__(kRmsThreads, 1) k_rms_oneshot(COMM_PARAM, const __grid_constant__ RmsArgs a, uint32_t rows, uint32_t op) {
  rms_oneshot<T, void>(c, a, RmsQuant{}, rows, op);
}

template <typename T>
__global__ void __launch_bounds__(kRmsThreads, 1) k_rms_twoshot(COMM_PARAM, const __grid_constant__ RmsArgs a, uint32_t rows, uint32_t op) {
  rms_twoshot<T, void>(c, a, RmsQuant{}, rows, op);
}

// 16-bit T: 2 CTAs per SM (at most 64 registers), as the 16-bit wide local kernels fit; fp32 would spill there
template <typename T, typename WireT>
__global__ void __launch_bounds__(kRmsThreads, sizeof(T) == 2 ? 2 : 1) k_rmsq_local(COMM_PARAM, const __grid_constant__ RmsArgs a, const __grid_constant__ RmsQuant qa,
                                                                uint32_t rows) {
  rms_local<T, WireT>(c, a, qa, rows);
}

template <typename T, typename WireT>
__global__ void __launch_bounds__(kRmsThreads, 1) k_rmsq_oneshot(COMM_PARAM, const __grid_constant__ RmsArgs a, const __grid_constant__ RmsQuant qa,
                                                                  uint32_t rows, uint32_t op) {
  rms_oneshot<T, WireT>(c, a, qa, rows, op);
}

template <typename T, typename WireT>
__global__ void __launch_bounds__(kRmsThreads, 1) k_rmsq_twoshot(COMM_PARAM, const __grid_constant__ RmsArgs a, const __grid_constant__ RmsQuant qa,
                                                                  uint32_t rows, uint32_t op) {
  rms_twoshot<T, WireT>(c, a, qa, rows, op);
}

template <typename T, bool GATHER>
__global__ void __launch_bounds__(kRmsThreads, 1) k_rs_norm(COMM_PARAM, const __grid_constant__ RmsArgs a, uint32_t rows, uint32_t op) {
  rs_norm<T, void, GATHER>(c, a, RmsQuant{}, rows, op);
}

template <typename T, typename WireT, bool GATHER>
__global__ void __launch_bounds__(kRmsThreads, 1) k_rs_normq(COMM_PARAM, const __grid_constant__ RmsArgs a, const __grid_constant__ RmsQuant qa,
                                                              uint32_t rows, uint32_t op) {
  rs_norm<T, WireT, GATHER>(c, a, qa, rows, op);
}

// Once per device, before the first kernel of this family launches: load all 45 kernels, all-reduce and reduce-scatter, wide and
// quantising. With lazy module loading a kernel's first launch loads it, and the load waits for kernels already running; a rank whose
// first launch of one of these kernels came behind its own barrier kernel, which waits for another rank's launch on the same thread,
// would never get there. One thread loads at a time.
static void rmsnorm_preload(const b200collComm* c) {
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
      cudaFuncGetAttributes(&fa, k_rms_local<T>);
      cudaFuncGetAttributes(&fa, k_rms_oneshot<T>);
      cudaFuncGetAttributes(&fa, k_rms_twoshot<T>);
      cudaFuncGetAttributes(&fa, k_rs_norm<T, false>);
      cudaFuncGetAttributes(&fa, k_rs_norm<T, true>);
      for (b200collDataType_t w : {b200collFloat8e4m3, b200collFloat8e5m2})
        with_fp8(w, [&](auto tw) {
          using WireT = typename decltype(tw)::type;
          cudaFuncGetAttributes(&fa, k_rmsq_local<T, WireT>);
          cudaFuncGetAttributes(&fa, k_rmsq_oneshot<T, WireT>);
          cudaFuncGetAttributes(&fa, k_rmsq_twoshot<T, WireT>);
          cudaFuncGetAttributes(&fa, k_rs_normq<T, WireT, false>);
          cudaFuncGetAttributes(&fa, k_rs_normq<T, WireT, true>);
        });
    });
  done.fetch_or(bit, std::memory_order_acq_rel);
}

// What the quantising call passes instead of out.
struct RmsQuantCall {
  void* q;
  float* scales;
  b200collDataType_t wire;
  int block;
};

// The reduce-scatter form's extra argument (nullptr: the all-reduce form).
struct RsCall {
  int gather;
};

static const char* rms_who(const RmsQuantCall* qz, const RsCall* rs) {
  if (rs) return qz ? "quantised reduce-scatter rms-norm: " : "reduce-scatter rms-norm: ";
  return qz ? "quantised all-reduce rms-norm: " : "all-reduce rms-norm: ";
}

// The argument rules of all four calls (qz == nullptr: the wide call; rs == nullptr: the all-reduce form, whose messages these are), all
// before the poisoned-communicator check; nothing is launched on a refusal. The reduce-scatter form's residual is [rows / nranks, row_len],
// and its out (q, scales) has rows / nranks rows, or rows when gathering.
static b200collResult_t rms_prepare(b200collComm* c, const void* x, const void* residual, const void* gamma, const void* out, size_t rows, size_t row_len,
                                    float eps, b200collDataType_t dtype, const RmsQuantCall* qz, const RsCall* rs = nullptr) {
  const std::string who = rms_who(qz, rs);
  auto refuse = [&](const std::string& msg) { set_last_error(who + msg); return b200collInvalidArgument; };
  if (!c) return refuse("null communicator");
  if (!wide_type(dtype)) return refuse("dtype must be bf16, fp16 or fp32");
  if (qz && !is_fp8(qz->wire)) return refuse("wire_dtype must be e4m3 or e5m2");
  if (qz && quant_lvpb(qz->block) < 0) return refuse(kBlockRule);
  if (row_len < 16 || row_len > kRmsMaxRowLen || row_len % 16 != 0) return refuse("row_len must be a multiple of 16 in [16, 16384]");
  if (qz && row_len % (size_t)qz->block != 0) return refuse("row_len must be a multiple of block");
  if (!(eps >= 0.0f) || !isfinite(eps)) return refuse("eps must be finite and non-negative");
  if (rows >= ((size_t)1 << 31)) return refuse("rows must be below 2^31");
  if (rs && rs->gather != 0 && rs->gather != 1) return refuse("gather must be 0 or 1");
  if (rs && rows % (size_t)c->nranks != 0) return refuse("rows must be a multiple of nranks");
  const size_t shard = rs ? rows / (size_t)c->nranks : rows, out_rows = rs && !rs->gather ? shard : rows;
  const size_t es = b200collTypeSize(dtype), mat = rows * row_len * es, g = row_len * es, res = shard * row_len * es, om = out_rows * row_len * es;
  if (!qz) {
    if (rows > 0 && (!x || !residual || !gamma || !out)) return refuse("null argument");
    if (!aligned(x, 16) || !aligned(residual, 16) || !aligned(gamma, 16) || !aligned(out, 16)) return refuse("x, residual, gamma and out must be 16-byte aligned");
    if (rows > 0 && (overlaps(out, om, x, mat) || overlaps(out, om, residual, res) || overlaps(out, om, gamma, g)))
      return refuse("out must not overlap x, residual or gamma");
  } else {
    if (rows > 0 && (!x || !residual || !gamma || !qz->q || !qz->scales)) return refuse("null argument");
    if (!aligned(x, 16) || !aligned(residual, 16) || !aligned(gamma, 16) || !aligned(qz->q, 16)) return refuse("x, residual, gamma and q must be 16-byte aligned");
    if (!aligned(qz->scales, 4)) return refuse("scales must be 4-byte aligned");
    const size_t qb = out_rows * row_len, sb = out_rows * (row_len / (size_t)qz->block) * 4;
    if (rows > 0 && (overlaps(qz->q, qb, x, mat) || overlaps(qz->q, qb, residual, res) || overlaps(qz->q, qb, gamma, g) || overlaps(qz->q, qb, qz->scales, sb)))
      return refuse("q must not overlap x, residual, gamma or scales");
    if (rows > 0 && (overlaps(qz->scales, sb, x, mat) || overlaps(qz->scales, sb, residual, res) || overlaps(qz->scales, sb, gamma, g)))
      return refuse("scales must not overlap x, residual or gamma");
  }
  if (rows > 0 && (overlaps(residual, res, x, mat) || overlaps(residual, res, gamma, g))) return refuse("residual must not overlap x or gamma");
  if (comm_poisoned(c)) return b200collRemoteError;
  return b200collSuccess;
}

// Both all-reduce calls after their arguments passed: the algorithm, the B200COLL_CHECK=1 cross-check, one launch. qz == nullptr: the
// wide call. The reduce-scatter form with one rank is this call's local kernel, counted under `stats_op`.
static b200collResult_t rms_run(b200collComm* c, const void* x, void* residual, const void* gamma, void* out, size_t rows, size_t row_len, float eps,
                                b200collDataType_t dtype, const RmsQuantCall* qz, b200collStream_t stream,
                                b200collOp_t stats_op = b200collOpAllReduce) {
  const char* who = rms_who(qz, nullptr);
  b200collResult_t rc = b200collSuccess;
  const size_t mat = rows * row_len * b200collTypeSize(dtype);
  const size_t qb = qz ? rows * row_len : 0, sb = qz ? rows * (row_len / (size_t)qz->block) * 4 : 0;
  b200collAlgo_t algo = b200collAlgoCopy;
  if (c->nranks > 1) {
    // peers pull my x at my arena offset. rows == 0 reads nothing (any pointer, even null, will do) and runs one-shot: only the barriers
    if (rows > 0 && (rc = in_arena(c, who, "x", {{x, mat}})) != b200collSuccess) return rc;
    // the tuner's pick for an all-reduce of these bytes, or the forced algorithm: ll, ll2 and oneshot pull every row; twoshot and nvls
    // push my rows into the peers' residual and out (or q and scales), so these must be arena memory, else one-shot
    const b200collAlgo_t want = c->forced_algo != b200collAlgoAuto ? c->forced_algo : b200collTunerPick(b200collOpAllReduce, mat, c->nranks, c->nvls);
    const bool two = rows > 0 && (want == b200collAlgoTwoShot || want == b200collAlgoNvls) && b200collIsSymmetric(c, residual, mat) &&
                     (qz ? b200collIsSymmetric(c, qz->q, qb) && b200collIsSymmetric(c, qz->scales, sb) : b200collIsSymmetric(c, out, mat));
    algo = two ? b200collAlgoTwoShot : b200collAlgoOneShot;
    // (rows, row_len) travel as one number (row_len < 2^15), and with them the x offset and, quantising, (block, wire); two-shot adds a
    // second exchange for the residual and out (q) offsets, and quantising a third for the scales offset
    const size_t shape = (rows << 15) | row_len, fmt = qz ? (size_t)qz->block * 2 + (qz->wire == b200collFloat8e5m2) : 0;
    if ((rc = cross_check(c, b200collOpAllReduce, algo, shape, rows > 0 ? arena_off(c, x) : 0, fmt)) != b200collSuccess) return rc;
    if (two && (rc = cross_check(c, b200collOpAllReduce, algo, shape, arena_off(c, residual), arena_off(c, qz ? qz->q : out))) != b200collSuccess) return rc;
    if (two && qz && (rc = cross_check(c, b200collOpAllReduce, algo, shape, arena_off(c, qz->scales), 0)) != b200collSuccess) return rc;
  }
  const DeviceScope on_device(c->device);
  rmsnorm_preload(c);
  account(c, stats_op, mat, algo);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RmsArgs a = {};
  a.x_local = static_cast<const char*>(x);
  a.res_in = static_cast<const char*>(residual);
  a.gamma = static_cast<const char*>(gamma);
  a.row_len = (uint32_t)row_len;
  a.nchunks = (uint32_t)(row_len / 16);
  a.eps = eps;
  RmsQuant qa = {};
  if (qz) qa.lvpb = (uint32_t)quant_lvpb(qz->block);
  // one launch of the local, one-shot or two-shot kernel: the wide one (WireT void) or the quantising one
  auto launch = [&](auto tt, auto tw) -> b200collResult_t {
    using T = typename decltype(tt)::type; using WireT = typename decltype(tw)::type;
    constexpr bool kQuant = !std::is_void<WireT>::value;
    const uint32_t op = (uint32_t)b200collOpAllReduce;
    if (algo == b200collAlgoTwoShot) {
      a.x_off = arena_off(c, x);
      a.res_off = arena_off(c, residual);
      if (qz) { qa.q_off = arena_off(c, qz->q); qa.s_off = arena_off(c, qz->scales); }
      else a.out_off = arena_off(c, out);
      const Grid gr = full_grid(c, 1);
      if constexpr (kQuant) launch_k(k_rmsq_twoshot<T, WireT>, gr.blocks, kRmsThreads, st, c->dev, a, qa, (uint32_t)rows, op);
      else launch_k(k_rms_twoshot<T>, gr.blocks, kRmsThreads, st, c->dev, a, (uint32_t)rows, op);
    } else {
      a.res_out = static_cast<char*>(residual);
      a.out = static_cast<char*>(out);
      if (qz) { qa.q = static_cast<char*>(qz->q); qa.scales = reinterpret_cast<char*>(qz->scales); }
      if (algo == b200collAlgoCopy) {
        const int blocks = (int)std::max<size_t>(1, std::min<size_t>(rows, (size_t)2 * std::max(1, c->sm_count)));   // 2 per SM where the registers allow
        if constexpr (kQuant) launch_k(k_rmsq_local<T, WireT>, blocks, kRmsThreads, st, c->dev, a, qa, (uint32_t)rows);
        else launch_k(k_rms_local<T>, blocks, kRmsThreads, st, c->dev, a, (uint32_t)rows);
      } else {
        a.x_off = arena_off(c, x);
        const Grid gr = full_grid(c, 1);
        if constexpr (kQuant) launch_k(k_rmsq_oneshot<T, WireT>, gr.blocks, kRmsThreads, st, c->dev, a, qa, (uint32_t)rows, op);
        else launch_k(k_rms_oneshot<T>, gr.blocks, kRmsThreads, st, c->dev, a, (uint32_t)rows, op);
      }
    }
    LAUNCH_CHECK(c);
    return b200collSuccess;
  };
  return with_wide(dtype, [&](auto tt) -> b200collResult_t {
    if (!qz) return launch(tt, Tag<void>{});
    return with_fp8(qz->wire, [&](auto tw) { return launch(tt, tw); });
  });
}

// Both reduce-scatter calls after their arguments passed. One rank: the all-reduce form's local kernel (the shard is every row). More:
// one algorithm, k_rs_norm / k_rs_normq, whatever the tuner or b200collCommSetAlgo says.
static b200collResult_t rs_run(b200collComm* c, const void* x, void* residual, const void* gamma, void* out, size_t rows, size_t row_len, float eps,
                               b200collDataType_t dtype, const RmsQuantCall* qz, const RsCall& rs, b200collStream_t stream) {
  if (c->nranks == 1) return rms_run(c, x, residual, gamma, out, rows, row_len, eps, dtype, qz, stream, b200collOpReduceScatter);
  const char* who = rms_who(qz, &rs);
  b200collResult_t rc = b200collSuccess;
  const size_t es = b200collTypeSize(dtype), mat = rows * row_len * es, shard = rows / (size_t)c->nranks;
  const size_t qb = rows * row_len, sb = qz ? rows * (row_len / (size_t)qz->block) * 4 : 0;
  // peers pull my x at my arena offset, and with gather push their rows into my out (q, scales) at my offsets. rows == 0 touches
  // nothing, so any pointer will do.
  if (rows > 0 && (rc = in_arena(c, who, "x", {{x, mat}})) != b200collSuccess) return rc;
  if (rows > 0 && rs.gather) {
    if (qz) rc = in_arena(c, who, "q and scales (gather)", {{qz->q, qb}, {qz->scales, sb}});
    else rc = in_arena(c, who, "out (gather)", {{out, mat}});
    if (rc != b200collSuccess) return rc;
  }
  // (rows, row_len, gather) travel as one number (row_len < 2^15), with the x offset and, quantising, (block, wire); gathering adds a
  // second exchange for the out (q) and scales offsets
  const size_t shape = (rows << 16) | (row_len << 1) | (size_t)rs.gather, fmt = qz ? (size_t)qz->block * 2 + (qz->wire == b200collFloat8e5m2) : 0;
  const b200collAlgo_t algo = b200collAlgoTwoShot;
  if ((rc = cross_check(c, b200collOpReduceScatter, algo, shape, rows > 0 ? arena_off(c, x) : 0, fmt)) != b200collSuccess) return rc;
  if (rs.gather && (rc = cross_check(c, b200collOpReduceScatter, algo, shape, rows > 0 ? arena_off(c, qz ? qz->q : out) : 0,
                                     rows > 0 && qz ? arena_off(c, qz->scales) : 0)) != b200collSuccess)
    return rc;
  const DeviceScope on_device(c->device);
  rmsnorm_preload(c);
  account(c, b200collOpReduceScatter, shard * row_len * es, algo);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RmsArgs a = {};
  a.res_in = static_cast<const char*>(residual);
  a.res_out = static_cast<char*>(residual);
  a.gamma = static_cast<const char*>(gamma);
  a.row_len = (uint32_t)row_len;
  a.nchunks = (uint32_t)(row_len / 16);
  a.eps = eps;
  if (rows > 0) a.x_off = arena_off(c, x);
  RmsQuant qa = {};
  if (qz) qa.lvpb = (uint32_t)quant_lvpb(qz->block);
  if (rs.gather && rows > 0) {
    if (qz) { qa.q_off = arena_off(c, qz->q); qa.s_off = arena_off(c, qz->scales); }
    else a.out_off = arena_off(c, out);
  } else {
    a.out = static_cast<char*>(out);
    if (qz) { qa.q = static_cast<char*>(qz->q); qa.scales = reinterpret_cast<char*>(qz->scales); }
  }
  const Grid gr = full_grid(c, 1);
  const uint32_t op = (uint32_t)b200collOpReduceScatter;
  auto launch = [&](auto tt, auto tw, auto tg) -> b200collResult_t {
    using T = typename decltype(tt)::type; using WireT = typename decltype(tw)::type;
    constexpr bool kGather = decltype(tg)::value;
    if constexpr (std::is_void<WireT>::value) launch_k(k_rs_norm<T, kGather>, gr.blocks, kRmsThreads, st, c->dev, a, (uint32_t)rows, op);
    else launch_k(k_rs_normq<T, WireT, kGather>, gr.blocks, kRmsThreads, st, c->dev, a, qa, (uint32_t)rows, op);
    LAUNCH_CHECK(c);
    return b200collSuccess;
  };
  return with_wide(dtype, [&](auto tt) -> b200collResult_t {
    auto with_gather = [&](auto tw) {
      return rs.gather ? launch(tt, tw, std::true_type{}) : launch(tt, tw, std::false_type{});
    };
    if (!qz) return with_gather(Tag<void>{});
    return with_fp8(qz->wire, [&](auto tw) { return with_gather(tw); });
  });
}

}  // namespace b200coll

using namespace b200coll;

extern "C" {

b200collResult_t b200collAllReduceRmsNorm(const void* x, void* residual, const void* gamma, void* out, size_t rows, size_t row_len, float eps,
                                          b200collDataType_t dtype, b200collComm_t c, b200collStream_t stream) {
  const b200collResult_t rc = rms_prepare(c, x, residual, gamma, out, rows, row_len, eps, dtype, nullptr);
  if (rc != b200collSuccess) return rc;
  return rms_run(c, x, residual, gamma, out, rows, row_len, eps, dtype, nullptr, stream);
}

b200collResult_t b200collAllReduceRmsNormQuantized(const void* x, void* residual, const void* gamma, void* q, float* scales, size_t rows, size_t row_len,
                                                   float eps, b200collDataType_t dtype, b200collDataType_t wire_dtype, int block, b200collComm_t c,
                                                   b200collStream_t stream) {
  const RmsQuantCall qz = {q, scales, wire_dtype, block};
  const b200collResult_t rc = rms_prepare(c, x, residual, gamma, nullptr, rows, row_len, eps, dtype, &qz);
  if (rc != b200collSuccess) return rc;
  return rms_run(c, x, residual, gamma, nullptr, rows, row_len, eps, dtype, &qz, stream);
}

b200collResult_t b200collReduceScatterRmsNorm(const void* x, void* residual, const void* gamma, void* out, size_t rows, size_t row_len, float eps,
                                              int gather, b200collDataType_t dtype, b200collComm_t c, b200collStream_t stream) {
  const RsCall rs = {gather};
  const b200collResult_t rc = rms_prepare(c, x, residual, gamma, out, rows, row_len, eps, dtype, nullptr, &rs);
  if (rc != b200collSuccess) return rc;
  return rs_run(c, x, residual, gamma, out, rows, row_len, eps, dtype, nullptr, rs, stream);
}

b200collResult_t b200collReduceScatterRmsNormQuantized(const void* x, void* residual, const void* gamma, void* q, float* scales, size_t rows,
                                                       size_t row_len, float eps, int gather, b200collDataType_t dtype, b200collDataType_t wire_dtype,
                                                       int block, b200collComm_t c, b200collStream_t stream) {
  const RmsQuantCall qz = {q, scales, wire_dtype, block};
  const RsCall rs = {gather};
  const b200collResult_t rc = rms_prepare(c, x, residual, gamma, nullptr, rows, row_len, eps, dtype, &qz, &rs);
  if (rc != b200collSuccess) return rc;
  return rs_run(c, x, residual, gamma, nullptr, rows, row_len, eps, dtype, &qz, rs, stream);
}

}  // extern "C"
