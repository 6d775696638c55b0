// b200coll_perf — nccl-tests-style benchmark + correctness checker for libb200coll.
// The reference's benchmark protocol (reference: gpudirect-tcpx/nccl-config.yaml:61-62,
// gpudirect-rdma/nccl-test-a4x-max-jobset.yaml:141-153): `-b <min> -e <max> -f 2 -g 1 -w 5 --iters 100 -c 1`,
// one rank per GPU, out-of-place and in-place, time = avg over iters, algbw = bytes/time,
// busbw = algbw * {AR: 2(N-1)/N; AG/RS/A2A: (N-1)/N}.
//
// Modes:  default      one process, one host thread per rank, ranks from --devs (repeat a device id for
//                      virtual ranks on one GPU: protocol tests on a single-GPU box)
//         --procs      fork one process per rank and rendezvous over the Unix-socket bootstrap
// Timing: CUDA events on each rank's stream around `iters` back-to-back launches, max over ranks.
// Buffers rotate through a >L2 window so every timed launch sees cold lines.
// Exit status: 0 every check passed; 1 a bad argument; 2 a CUDA error; 3 a library error; 4 a -c 1 check found a wrong value (in every
// mode); 5 the library's watchdog recorded a fault; 6 a host barrier timed out.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <fcntl.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/wait.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <string>
#include <thread>
#include <vector>

#include "../include/b200coll.h"

#define RT(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "CUDA %s:%d %s -> %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); exit(2); } } while (0)
#define CC(x) do { b200collResult_t r_ = (x); if (r_ != b200collSuccess) { fprintf(stderr, "b200coll %s:%d %s -> %s (%s)\n", __FILE__, __LINE__, #x, b200collGetErrorString(r_), b200collGetLastError()); exit(3); } } while (0)

struct Opts {
  std::string op = "all_reduce";
  std::vector<int> devs;
  int nranks = 0;
  bool procs = false;
  size_t min_bytes = 1024, max_bytes = 1ull << 30;
  int factor = 2;
  b200collDataType_t in_dt = b200collBfloat16, out_dt = b200collBfloat16;
  float scale = 1.0f;
  std::string algo = "auto";
  int iters = 20, warmup = 5, check = 1;
  int inplace = 2;   // 0 out-of-place only, 1 in-place only, 2 both
  int max_ctas = 0;
  size_t window = 192ull << 20;
  std::string json;
  int skew_us = 0;   // delay rank 0's launches (race hunting)
  struct Shape { int kind, ctas, threads; };
  std::vector<Shape> shapes;   // --sweep kind:ctas:threads,... (launch-shape tuning inside one process)
  int bs_rows = 0, bs_cols = 0;   // --block-scale RxC: block-scaled FP8 collectives (0 = off)
  size_t row_len = 2048;          // --row-len N: columns of the block-scaled matrix
  int q_block = 0;                // --quantize WIRE:BLOCK: quantising collectives (0 = off)
  b200collDataType_t q_wire = b200collFloat8e4m3;
  int combine_k = 0;              // --combine K: the expert combine with top_k = K (0 = off)
  int route_e = 0, route_k = 0;   // --route E:K: the device-routed dispatch and combine, E experts, top-K (0 = off)
  int cq_block = 0;               // --combine-quantize WIRE:BLOCK: the quantising combine in --combine / --route (0 = off)
  b200collDataType_t cq_wire = b200collFloat8e4m3;
  size_t rms_row = 0;             // --rms-norm ROW_LEN: the fused all-reduce, residual add and RMSNorm (0 = off)
  int rq_block = 0;               // --rms-norm-quantize WIRE:BLOCK: its FP8 out, one fp32 scale per 1 x BLOCK (0 = off)
  bool rms_gather = false;        // --rms-norm-gather: with --op reduce_scatter, the normed rows all-gathered in the same kernel
  b200collDataType_t rq_wire = b200collFloat8e4m3;
  int uly_hq = 0, uly_hkv = 0, uly_d = 0;   // --ulysses HQ:HKV:D: the Ulysses all-to-all of a packed QKV (0 = off)
  bool uly_back = false;                    // --ulysses-back: heads -> sequence, the attention output
  int cp_c = 0;                             // --context W:C or HQ:HKV:D:C: the context-parallel gather / reduce-scatter, C chunks per rank (0 = off)
  int cp_hq = 0, cp_hkv = 0, cp_d = 0;      // packed QKV (K and V column slices), or 0 with cp_w
  size_t cp_w = 0;                          // one dense tensor of cp_w elements per token
  int fs_h = 0, fs_f = 0, fs_kv = 0;        // --fsdp H:F[:KV]: the FSDP shard gather / reduce-scatter of one Llama block (0 = off)
  bool accumulate = false;                  // --accumulate: the reduce-scatter adds into the old shard
};

// Block-scaled mode: each rank's send buffer is a [rows, row_len] FP8 matrix with one fp32 scale per bs_rows x bs_cols block. Scales are
// seeded (hash of rank and block index): mantissas use all 23 bits, exponents span 2^-8..2^8, so products round and the check below,
// which repeats the library's arithmetic on the host, is bit for bit.
static size_t bs_max_scales(const Opts& o) {
  const size_t rows = o.max_bytes / o.row_len + 1;
  return (rows / o.bs_rows + 1) * (o.row_len / o.bs_cols + 1);
}
static float bs_scale(int rank, size_t idx) {
  uint32_t h = (uint32_t)(idx * 2654435761u) ^ (uint32_t)(rank * 40503u + 0x9E3779B9u);
  h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 12;
  return ldexpf(1.0f + (float)(h & 0x7FFFFF) * 0x1p-23f, (int)((h >> 23) % 17) - 8);
}
static uint32_t out_bits(float v, b200collDataType_t dt) {
  if (dt == b200collFloat32) { uint32_t u; memcpy(&u, &v, 4); return u; }
  if (dt == b200collFloat16) { __half h = __float2half_rn(v); uint16_t u; memcpy(&u, &h, 2); return u; }
  __nv_bfloat16 b = __float2bfloat16_rn(v); uint16_t u; memcpy(&u, &b, 2); return u;
}
static uint32_t got_bits(const void* p, size_t i, b200collDataType_t dt) {
  if (dt == b200collFloat32) { uint32_t u; memcpy(&u, (const char*)p + 4 * i, 4); return u; }
  uint16_t u; memcpy(&u, (const char*)p + 2 * i, 2); return u;
}

// The quantising all-to-all-v receives one fp32 scale per block of its FP8 rows, into an arena buffer that holds the scales of a whole
// window or of the largest message.
static size_t q_a2a_scale_bytes(const Opts& o) {
  return (std::max(o.window, o.max_bytes) + 4096) / b200collTypeSize(o.in_dt) / o.q_block * 4 + 4096;
}
// The library's quantisation scratch (FP8 copy plus scales per rank) grows with the sweep and keeps every superseded buffer: reserve
// twice the largest one. The all-to-all-v takes no scratch, only its scale buffer.
static size_t q_scratch_bytes(const Opts& o) {
  if (!o.q_block) return 0;
  if (o.op == "alltoall") return q_a2a_scale_bytes(o);
  const size_t elems = o.max_bytes / b200collTypeSize(o.in_dt);
  return 2 * (elems + elems / o.q_block * 4) + (4u << 20);
}

static size_t parse_size(const char* s) {
  char* end; double v = strtod(s, &end);
  if (*end == 'K' || *end == 'k') v *= 1024; else if (*end == 'M' || *end == 'm') v *= 1 << 20; else if (*end == 'G' || *end == 'g') v *= 1 << 30;
  return (size_t)v;
}
static b200collDataType_t parse_dt(const char* s) {
  if (!strcmp(s, "f32") || !strcmp(s, "float")) return b200collFloat32;
  if (!strcmp(s, "f16") || !strcmp(s, "half")) return b200collFloat16;
  if (!strcmp(s, "bf16") || !strcmp(s, "bfloat16")) return b200collBfloat16;
  if (!strcmp(s, "fp8") || !strcmp(s, "e4m3")) return b200collFloat8e4m3;
  if (!strcmp(s, "e5m2")) return b200collFloat8e5m2;
  fprintf(stderr, "bad dtype %s\n", s); exit(1);
}
// --quantize, --combine-quantize and --rms-norm-quantize WIRE:BLOCK
static void parse_wire_block(const std::string& flag, const char* s, b200collDataType_t* wire, int* block) {
  char w[16] = {};
  if (sscanf(s, "%15[a-z0-9]:%d", w, block) != 2 || (strcmp(w, "e4m3") && strcmp(w, "e5m2")) || *block < 16 || *block > 512 || (*block & (*block - 1))) {
    fprintf(stderr, "%s WIRE:BLOCK: WIRE e4m3 or e5m2, BLOCK 16, 32, 64, 128, 256 or 512\n", flag.c_str()); exit(1);
  }
  *wire = parse_dt(w);
}
static const char* dt_name(b200collDataType_t t) { return t == b200collFloat32 ? "f32" : t == b200collFloat16 ? "f16" : t == b200collBfloat16 ? "bf16" : t == b200collFloat8e5m2 ? "e5m2" : "e4m3"; }
static bool wide(b200collDataType_t t) { return t == b200collBfloat16 || t == b200collFloat16 || t == b200collFloat32; }

// Deterministic input: multiples of 0.25 in [-2, 2] (exact in e4m3 and e5m2 too) so sums over <= 8 ranks are exact in bf16/f16/f32.
// With block > 0 (the quantising modes) each value is also multiplied by a power of two that changes from block to block (2^-6 .. 2^6,
// exact in bf16, fp16 and fp32), so blocks have different amax values.
__host__ __device__ inline float gen(int rank, size_t i, int block = 0) {
  const float v = (float)((int)((i * 7 + (size_t)rank * 13 + (i >> 9)) % 17) - 8) * 0.25f;
  return block ? v * ldexpf(1.0f, (int)(((i / block) * 5 + (size_t)rank * 3) % 13) - 6) : v;
}
template <typename T> __global__ void k_fill(T* p, size_t n, int rank, int block) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = T(gen(rank, i, block));
}
static void fill(void* p, size_t n, b200collDataType_t dt, int rank, cudaStream_t st, int block = 0) {
  if (dt == b200collFloat32) k_fill<float><<<256, 256, 0, st>>>((float*)p, n, rank, block);
  else if (dt == b200collFloat16) k_fill<__half><<<256, 256, 0, st>>>((__half*)p, n, rank, block);
  else if (dt == b200collFloat8e4m3) k_fill<__nv_fp8_e4m3><<<256, 256, 0, st>>>((__nv_fp8_e4m3*)p, n, rank, block);
  else if (dt == b200collFloat8e5m2) k_fill<__nv_fp8_e5m2><<<256, 256, 0, st>>>((__nv_fp8_e5m2*)p, n, rank, block);
  else k_fill<__nv_bfloat16><<<256, 256, 0, st>>>((__nv_bfloat16*)p, n, rank, block);
  RT(cudaGetLastError());
}

// The library's per-block quantisation rule on the host: amax, two IEEE divisions, the RNE saturating pack of each value times inv into
// q. Returns the block's scale; dequant() turns a code back into a value with one multiply. The checks repeat it bit for bit.
static __nv_fp8_interpretation_t fp8_kind(b200collDataType_t wire) { return wire == b200collFloat8e4m3 ? __NV_E4M3 : __NV_E5M2; }
static float quantise_block(const float* x, int n, b200collDataType_t wire, __nv_fp8_storage_t* q) {
  const float fmax = wire == b200collFloat8e4m3 ? 448.0f : 57344.0f;
  float amax = 0.0f;
  for (int k = 0; k < n; k++) amax = std::max(amax, fabsf(x[k]));
  volatile float a = amax;                                     // keep both divisions as written: IEEE, rounded to nearest
  float inv = fmax / a, s = a / fmax;
  if (amax == 0.0f || isinf(inv)) inv = s = 1.0f;
  for (int k = 0; k < n; k++) q[k] = __nv_cvt_float_to_fp8(x[k] * inv, __NV_SATFINITE, fp8_kind(wire));
  return s;
}
static float dequant(__nv_fp8_storage_t q, float s, b200collDataType_t wire) {
  volatile float v = __half2float(__half(__nv_cvt_fp8_to_halfraw(q, fp8_kind(wire)))) * s;
  return v;
}
// Quantising mode: the FP8 code of rank r's element gen(r, i, q_block); `memo` keeps the last block's codes and scale, as the checks
// walk elements in order.
struct QMemo { size_t blk = SIZE_MAX; float s = 1.0f; __nv_fp8_storage_t q[512]; };
static __nv_fp8_storage_t q_code(const Opts& o, int rank, size_t i, QMemo* memo) {
  const size_t blk = i / o.q_block;
  if (memo->blk != blk) {
    float x[512];
    for (int k = 0; k < o.q_block; k++) x[k] = gen(rank, blk * o.q_block + k, o.q_block);
    memo->s = quantise_block(x, o.q_block, o.q_wire, memo->q);
    memo->blk = blk;
  }
  return memo->q[i % o.q_block];
}
// ... and its dequantised value
static float q_val(const Opts& o, int rank, size_t i, QMemo* memo) {
  const __nv_fp8_storage_t q = q_code(o, rank, i, memo);
  return dequant(q, memo->s, o.q_wire);
}
// The quantising combine's host reference: n values quantised block by block and dequantised, in place.
static void q_roundtrip(float* x, size_t n, int block, b200collDataType_t wire) {
  __nv_fp8_storage_t q[512];
  for (size_t b0 = 0; b0 < n; b0 += block) {
    const float s = quantise_block(x + b0, block, wire, q);
    for (int k = 0; k < block; k++) x[b0 + k] = dequant(q[k], s, wire);
  }
}
// The quantising combine's scratch (FP8 copy plus scales of every expert_out row) grows with the sweep and keeps every superseded
// buffer: reserve twice the largest one.
static size_t cq_scratch_bytes(const Opts& o) {
  if (!o.cq_block) return 0;
  const size_t elems = o.max_bytes / b200collTypeSize(o.in_dt) * (o.route_e ? o.route_k : 1);
  return 2 * (elems + elems / o.cq_block * 4) + (4u << 20);
}

static float to_f(const void* p, size_t i, b200collDataType_t dt) {
  switch (dt) {
    case b200collFloat32: return ((const float*)p)[i];
    case b200collFloat16: return __half2float(((const __half*)p)[i]);
    case b200collBfloat16: return __bfloat162float(((const __nv_bfloat16*)p)[i]);
    case b200collFloat8e5m2: return (float)(((const __nv_fp8_e5m2*)p)[i]);
    default: return (float)(((const __nv_fp8_e4m3*)p)[i]);
  }
}

struct Shared {   // cross-process (mmap MAP_SHARED) or cross-thread rendezvous for timing
  std::atomic<int> arrive[4];
  float ms[B200COLL_MAX_RANKS];
  long errors[B200COLL_MAX_RANKS];
};

static void spin_barrier(Shared* sh, int which, int n, int* gen) {
  (*gen)++;
  sh->arrive[which].fetch_add(1);
  const time_t t0 = time(nullptr);
  while (sh->arrive[which].load() < (*gen) * n) {
    sched_yield();
    if (time(nullptr) - t0 > 90) { fprintf(stderr, "host barrier %d timed out (a rank died?)\n", which); _exit(6); }
  }
}

constexpr int kRoot = 0;   // rooted ops (broadcast, reduce) are driven from rank 0, like nccl-tests' default

struct RankCtx {
  int rank, nranks; b200collComm_t comm; int dev;
  Shared* sh;
  cudaStream_t st = nullptr; cudaEvent_t e0 = nullptr, e1 = nullptr;   // made by run_rank
  int barrier_gen[4] = {0, 0, 0, 0};
  void barrier(int which) { spin_barrier(sh, which, nranks, &barrier_gen[which]); }
};

// A fault the library's watchdog recorded ends the rank.
static void watchdog(const RankCtx& c, const char* when) {
  b200collFault f;
  if (b200collCommGetAsyncError(c.comm, &f) != b200collSuccess) {
    fprintf(stderr, "rank %d WATCHDOG (%s) code=%u peer=%u block=%u expected=%u observed=%u op=%u\n", c.rank, when, f.code, f.peer, f.block, f.expected,
            f.observed, f.op);
    _exit(5);
  }
}
// The -c 1 launch: inputs ready on every rank (barrier 0), rank 0 late by --skew-us, launch(0), every rank done (barrier 1).
template <typename F> static void check_launch(const Opts& o, RankCtx& c, F&& launch) {
  RT(cudaStreamSynchronize(c.st));
  c.barrier(0);
  if (o.skew_us && c.rank == 0) usleep(o.skew_us);
  launch(0);
  RT(cudaStreamSynchronize(c.st));
  c.barrier(1);
  watchdog(c, "check");
}
// The timing protocol: launch(i) for `warmup` untimed iterations, all ranks lined up (barrier 2), then CUDA events on this rank's stream
// around `iters` back-to-back launches. Every rank posts its per-launch ms and error count `errs` (barrier 3) and reads all of them;
// barrier 0 keeps the page stable until everyone has. Returns the worst ms over ranks and the sum of their errors.
struct Timing { float ms; long errors; };
template <typename F> static Timing timed(const Opts& o, RankCtx& c, long errs, F&& launch) {
  for (int i = 0; i < o.warmup; i++) launch(i);
  RT(cudaStreamSynchronize(c.st));
  c.barrier(2);
  RT(cudaEventRecord(c.e0, c.st));
  for (int i = 0; i < o.iters; i++) launch(i);
  RT(cudaEventRecord(c.e1, c.st));
  RT(cudaEventSynchronize(c.e1));
  float ms = 0; RT(cudaEventElapsedTime(&ms, c.e0, c.e1));
  c.sh->ms[c.rank] = ms / o.iters; c.sh->errors[c.rank] = errs;
  c.barrier(3);
  Timing t{0, 0};
  for (int r = 0; r < c.nranks; r++) { t.ms = std::max(t.ms, c.sh->ms[r]); t.errors += c.sh->errors[r]; }
  c.barrier(0);
  watchdog(c, "timing");
  return t;
}

// The end of a mode runner (--combine, --rms-norm, --route): rank 0 reports the launches and the errors of every size.
static int mode_result(const RankCtx& c, long total_errors) {
  b200collStats s; CC(b200collCommStatsGet(c.comm, &s));
  if (c.rank == 0) {
    printf("# launches=%llu errors=%ld\n", (unsigned long long)s.kernel_launches, total_errors);
    fflush(stdout);
  }
  return total_errors ? 4 : 0;
}

// Expert-combine mode (--combine K). Per size, every rank's expert_out holds `bytes` of whole --row-len rows, an even split: rpp rows
// came from every rank. So rank r's dispatch rows for peer p are rows [p * rpp, + rpp) of its (notional) send buffer and their expert
// outputs are rows [r * rpp, + rpp) of p's expert_out. tokens = n * rpp / K, and token t's slot j goes to range (t + j + h(t)) % n
// (K different ranges where n >= K), to the next unused row of that range, or is dropped (-1) when the range is used up. Weights are
// seeded in [0.25, 1.25). Expert-out values are exact in every input type and the weights have full mantissas, so products and sums
// round; -c 1 repeats the slot-order fp32 arithmetic on the host and compares every output element bit for bit.
static uint32_t co_hash(uint32_t x) { x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16; return x; }
static int run_combine(const Opts& o, RankCtx& ctx, void* expert_out, void* out) {
  const int n = ctx.nranks, rank = ctx.rank, K = o.combine_k;
  const size_t is = b200collTypeSize(o.in_dt), os = b200collTypeSize(o.out_dt), row = o.row_len;
  const b200collEpilogue ep{o.in_dt, o.out_dt, o.scale};
  const cudaStream_t st = ctx.st;
  long total_errors = 0;
  if (rank == 0 && o.cq_block) {
    printf("# b200coll_perf op=alltoall quantising combine top_k=%d nranks=%d in=%s wire=%s block=%d out=%s scale=%g row_len=%zu: size = expert_out bytes per rank\n",
           K, n, dt_name(o.in_dt), dt_name(o.cq_wire), o.cq_block, dt_name(o.out_dt), o.scale, row);
  } else if (rank == 0) {
    printf("# b200coll_perf op=alltoall combine top_k=%d nranks=%d in=%s out=%s scale=%g row_len=%zu: size = expert_out bytes read per rank\n", K, n, dt_name(o.in_dt),
           dt_name(o.out_dt), o.scale, row);
  }
  if (rank == 0) {
    printf("#%13s %12s %6s %8s | %10s %8s %6s\n", "size(B)", "tokens", "type", "algo", "us", "algbw", "#wrong");
    fflush(stdout);
  }
  for (size_t bytes = o.min_bytes; bytes <= o.max_bytes; bytes *= o.factor) {
    const size_t rpp = bytes / is / row / n, recv_rows = rpp * n, tokens = recv_rows / K;
    if (tokens == 0) continue;
    std::vector<int64_t> rows(n, (int64_t)rpp), soff(n), roff(n, (int64_t)(rank * rpp));
    for (int p = 0; p < n; p++) soff[p] = (int64_t)(p * rpp);
    std::vector<int32_t> idx(tokens * K);
    std::vector<float> w(tokens * K);
    std::vector<size_t> used(n, 0);
    for (size_t t = 0; t < tokens; t++) {
      const uint32_t h = co_hash((uint32_t)t * 2654435761u ^ (uint32_t)rank * 97u);
      for (int j = 0; j < K; j++) {
        const int p = (int)((t + j + h) % n);
        idx[t * K + j] = used[p] < rpp ? (int32_t)(soff[p] + used[p]++) : -1;
        w[t * K + j] = 0.25f + (float)(co_hash(h + 31u * j) & 0xFFFFFF) * 0x1p-24f;
      }
    }
    int32_t* d_idx = nullptr; float* d_w = nullptr;
    RT(cudaMalloc(&d_idx, idx.size() * 4)); RT(cudaMalloc(&d_w, w.size() * 4));
    RT(cudaMemcpy(d_idx, idx.data(), idx.size() * 4, cudaMemcpyHostToDevice));
    RT(cudaMemcpy(d_w, w.data(), w.size() * 4, cudaMemcpyHostToDevice));
    const size_t eo_elems = recv_rows * row, out_elems = tokens * row;
    fill(expert_out, eo_elems, o.in_dt, rank, st, 16);
    RT(cudaMemsetAsync(out, 0x5A, out_elems * os, st));
    auto launch = [&](int) {
      if (o.cq_block)
        CC(b200collAllToAllvCombineQuantized(expert_out, out, row, recv_rows, rows.data(), soff.data(), roff.data(), d_idx, d_w, tokens, K, o.cq_wire,
                                             o.cq_block, &ep, ctx.comm, st));
      else
        CC(b200collAllToAllvCombine(expert_out, out, row, recv_rows, rows.data(), soff.data(), roff.data(), d_idx, d_w, tokens, K, &ep, ctx.comm, st));
    };
    long errs = 0;
    if (o.check) {
      check_launch(o, ctx, launch);
      std::vector<char> host(out_elems * os);
      RT(cudaMemcpy(host.data(), out, host.size(), cudaMemcpyDeviceToHost));
      // --combine-quantize: the rows this rank reads (rows [rank * rpp, + rpp) of every peer's expert_out), quantised and dequantised
      std::vector<float> deq(o.cq_block ? (size_t)n * rpp * row : 0);
      for (size_t i = 0; i < deq.size(); i++) deq[i] = gen((int)(i / (rpp * row)), (size_t)rank * rpp * row + i % (rpp * row), 16);
      for (size_t r = 0; r < deq.size() / row; r++) q_roundtrip(deq.data() + r * row, row, o.cq_block, o.cq_wire);
      for (size_t t = 0; t < tokens; t++) {
        for (size_t e = 0; e < row; e++) {
          float acc = 0.0f;
          for (int j = 0; j < K; j++) {
            const int32_t i = idx[t * K + j];
            if (i < 0) continue;
            const int p = (int)(i / (int64_t)rpp);                      // the range row i lies in, and its row of p's expert_out
            const size_t r = (size_t)rank * rpp + (size_t)(i - soff[p]);
            volatile float prod = w[t * K + j] * (o.cq_block ? deq[((size_t)p * rpp + (size_t)(i - soff[p])) * row + e] : gen(p, r * row + e, 16));
            acc = acc + prod;
          }
          const uint32_t want = out_bits(acc * o.scale, o.out_dt), got = got_bits(host.data(), t * row + e, o.out_dt);
          if (got != want) { if (errs < 4) fprintf(stderr, "rank %d combine size %zu token %zu elem %zu: got bits 0x%x want 0x%x\n", rank, bytes, t, e, got, want); errs++; }
        }
      }
    }
    const Timing tm = timed(o, ctx, errs, launch);
    total_errors += tm.errors;
    if (rank == 0) {
      const size_t eo_bytes = recv_rows * row * is;
      printf("%14zu %12zu %6s %8s | %10.2f %8.2f %6ld\n", eo_bytes, tokens, dt_name(o.in_dt), n > 1 ? "oneshot" : "copy", tm.ms * 1e3, eo_bytes / (tm.ms * 1e3) / 1e3,
             tm.errors);
      fflush(stdout);
    }
    RT(cudaFree(d_idx)); RT(cudaFree(d_w));
  }
  return mode_result(ctx, total_errors);
}

// All-reduce + RMSNorm mode (--rms-norm ROW_LEN). Per size, every rank's x holds `bytes` of whole rows (k_fill values of its rank), the
// residual the same k_fill rows on every rank, gamma one k_fill row; x, residual and out are arena memory. -c 1 runs one call and
// repeats steps 1-5 of b200collAllReduceRmsNorm on the host (every sum and product rounded on its own, IEEE sqrt and division), then
// compares every residual and out element bit for bit. The timed calls keep updating the residual in place. "rw GB/s" counts the bytes
// one rank's HBM moves at one rank: x, residual and gamma read, residual and out written.
// With --rms-norm-quantize WIRE:BLOCK it runs b200collAllReduceRmsNormQuantized: out holds the FP8 rows q and an arena buffer their
// scales; -c 1 adds step 6 on the host (each row's out values, rounded to the dtype, quantised per BLOCK by quantise_block) and compares
// every residual element, FP8 byte and scale bit for bit. "rw GB/s" then counts q and the scales written instead of out.
// With --op reduce_scatter it runs b200collReduceScatterRmsNorm (...Quantized): rows are rounded down to a multiple of nranks, and rank r
// passes rows [r*S, (r+1)*S) of the residual buffer as its shard. -c 1 checks the shard's rows and that no other residual row changed,
// and out (q, scales) for the slice, stored from row 0, or with --rms-norm-gather for every row. "rw GB/s" counts x, the shard read and
// written, gamma, and the out rows this rank stores.
static size_t rms_scale_bytes(const Opts& o) {
  return o.rq_block ? o.max_bytes / b200collTypeSize(o.in_dt) / o.rq_block * 4 + 4096 : 0;
}
static float round_dt(float v, b200collDataType_t dt) {
  if (dt == b200collFloat32) return v;
  if (dt == b200collFloat16) return __half2float(__float2half_rn(v));
  return __bfloat162float(__float2bfloat16_rn(v));
}
static int run_rms(const Opts& o, RankCtx& ctx, void* x, void* out, void* residual) {
  const int n = ctx.nranks, rank = ctx.rank;
  const b200collDataType_t dt = o.in_dt;
  const size_t es = b200collTypeSize(dt), row = o.rms_row;
  const float eps = 1e-6f;
  const cudaStream_t st = ctx.st;
  const int blk = o.rq_block;
  const bool sp = o.op == "reduce_scatter", gather = sp && o.rms_gather;
  long total_errors = 0;
  if (rank == 0 && sp) {
    printf("# b200coll_perf op=reduce_scatter + rms-norm%s%s nranks=%d dtype=%s wire=%s block=%d row_len=%zu eps=%g: size = x bytes per rank; rw GB/s = "
           "(x + residual shard + gamma read, residual shard + %s written) / time\n", gather ? " + gather" : "", blk ? " + quantize" : "", n, dt_name(dt),
           blk ? dt_name(o.rq_wire) : "-", blk, row, eps, blk ? "q + scales" : "out");
  } else if (rank == 0 && blk) {
    printf("# b200coll_perf op=all_reduce + rms-norm + quantize nranks=%d dtype=%s wire=%s block=%d row_len=%zu eps=%g: size = x bytes per rank; rw GB/s = "
           "(x + residual + gamma read, residual + q + scales written) / time\n", n, dt_name(dt), dt_name(o.rq_wire), blk, row, eps);
  } else if (rank == 0) {
    printf("# b200coll_perf op=all_reduce + rms-norm nranks=%d dtype=%s row_len=%zu eps=%g: size = x bytes per rank; rw GB/s = (x + residual + gamma read, "
           "residual + out written) / time\n", n, dt_name(dt), row, eps);
  }
  if (rank == 0) {
    printf("#%13s %10s %6s %8s | %10s %8s %8s %6s\n", "size(B)", "rows", "type", "algo", "us", "algbw", "rw_GB/s", "#wrong");
    fflush(stdout);
  }
  void* gamma = nullptr;
  RT(cudaMalloc(&gamma, row * es));
  fill(gamma, row, dt, 7, st);
  float* scales = nullptr;                                         // --rms-norm-quantize: the scales of q, in the arena like q
  if (blk) CC(b200collMemAlloc(ctx.comm, (void**)&scales, rms_scale_bytes(o)));
  for (size_t bytes = o.min_bytes; bytes <= o.max_bytes; bytes *= o.factor) {
    const size_t rows = sp ? bytes / es / row / n * n : bytes / es / row, elems = rows * row;
    if (rows == 0) continue;
    // the reduce-scatter form: my shard of the residual, and the rows of out (q, scales) I store, from row o_row0 of mine
    const size_t shard = sp ? rows / n : rows, r0 = sp ? shard * rank : 0, o_rows = sp && !gather ? shard : rows, o_row0 = gather || !sp ? 0 : r0;
    char* res = static_cast<char*>(residual) + r0 * row * es;
    fill(x, elems, dt, rank, st);
    fill(residual, elems, dt, 99, st);
    const size_t nblk = blk ? elems / blk : 0, out_bytes = (blk ? elems + nblk * 4 : elems * es) / rows * o_rows;    // q and scales, or out
    RT(cudaMemsetAsync(out, 0x5A, blk ? elems : elems * es, st));
    if (blk) RT(cudaMemsetAsync(scales, 0x5A, nblk * 4, st));
    auto launch = [&](int) {
      if (sp && blk) CC(b200collReduceScatterRmsNormQuantized(x, res, gamma, out, scales, rows, row, eps, gather, dt, o.rq_wire, blk, ctx.comm, st));
      else if (sp) CC(b200collReduceScatterRmsNorm(x, res, gamma, out, rows, row, eps, gather, dt, ctx.comm, st));
      else if (blk) CC(b200collAllReduceRmsNormQuantized(x, residual, gamma, out, scales, rows, row, eps, dt, o.rq_wire, blk, ctx.comm, st));
      else CC(b200collAllReduceRmsNorm(x, residual, gamma, out, rows, row, eps, dt, ctx.comm, st));
    };
    long errs = 0;
    if (o.check) {
      check_launch(o, ctx, launch);
      std::vector<char> gres(elems * es), gout(blk ? elems : elems * es);
      std::vector<float> gsc(nblk);
      RT(cudaMemcpy(gres.data(), residual, gres.size(), cudaMemcpyDeviceToHost));
      RT(cudaMemcpy(gout.data(), out, gout.size(), cudaMemcpyDeviceToHost));
      if (blk) RT(cudaMemcpy(gsc.data(), scales, nblk * 4, cudaMemcpyDeviceToHost));
      const size_t nch = row / 16;
      size_t P = 1;
      while (P < nch) P *= 2;
      std::vector<float> h(row), p(P), y(row);
      std::vector<__nv_fp8_storage_t> qw(row);
      for (size_t i = 0; i < rows; i++) {
        for (size_t e = 0; e < row; e++) {
          volatile float acc = 0.0f;
          for (int r = 0; r < n; r++) acc = acc + gen(r, i * row + e);     // the fill values, exact in every dtype
          h[e] = round_dt(acc + gen(99, i * row + e), dt);
        }
        for (size_t c = 0; c < P; c++) {
          volatile float s = 0.0f;
          for (size_t e = 16 * c; c < nch && e < 16 * c + 16; e++) { volatile float sq = h[e] * h[e]; s = s + sq; }
          p[c] = s;
        }
        for (size_t w = P / 2; w >= 1; w /= 2)
          for (size_t c = 0; c < w; c++) { volatile float v = p[c] + p[c + w]; p[c] = v; }
        volatile float ms = p[0] / (float)row;
        volatile float den = sqrtf(ms + eps);
        const float inv = 1.0f / den;
        for (size_t e = 0; e < row; e++) {
          volatile float hi = h[e] * inv;
          volatile float ye = hi * gen(7, e);
          y[e] = blk ? round_dt(ye, dt) : ye;                            // step 6 quantises out as stored
        }
        const bool mine = i >= r0 && i < r0 + shard, stored = mine || gather;    // residual row i changes, out row i is stored here
        const size_t oi = i - o_row0;                                    // (stored) out row i's index in out
        for (size_t b = 0; blk && stored && b < row / blk; b++) {
          const float sw = quantise_block(y.data() + b * blk, blk, o.rq_wire, qw.data() + b * blk), sg = gsc[oi * (row / blk) + b];
          uint32_t want_s, got_s; memcpy(&want_s, &sw, 4); memcpy(&got_s, &sg, 4);
          if (got_s != want_s) {
            if (errs < 4) fprintf(stderr, "rank %d rms-norm size %zu row %zu block %zu: scale 0x%x want 0x%x\n", rank, bytes, i, b, got_s, want_s);
            errs++;
          }
        }
        for (size_t e = 0; e < row; e++) {
          const uint32_t want_h = out_bits(mine ? h[e] : gen(99, i * row + e), dt), got_h = got_bits(gres.data(), i * row + e, dt);
          uint32_t want_o = 0, got_o = 0;
          if (stored) {
            want_o = blk ? qw[e] : out_bits(y[e], dt);
            got_o = blk ? (uint8_t)gout[oi * row + e] : got_bits(gout.data(), oi * row + e, dt);
          }
          if (got_h != want_h || got_o != want_o) {
            if (errs < 4) fprintf(stderr, "rank %d rms-norm size %zu row %zu elem %zu: residual 0x%x want 0x%x, %s 0x%x want 0x%x\n", rank, bytes, i, e, got_h,
                                  want_h, blk ? "q" : "out", got_o, want_o);
            errs++;
          }
        }
      }
    }
    b200collStats s0; CC(b200collCommStatsGet(ctx.comm, &s0));
    const Timing tm = timed(o, ctx, errs, launch);
    b200collStats s1; CC(b200collCommStatsGet(ctx.comm, &s1));
    total_errors += tm.errors;
    if (rank == 0) {
      const char* algo = "?";
      for (int a = 0; a < b200collNumAlgos; a++) if (s1.algo_calls[a] != s0.algo_calls[a]) algo = b200collAlgoName((b200collAlgo_t)a);
      const size_t mat = elems * es, rw = mat + 2 * shard * row * es + row * es + out_bytes;
      printf("%14zu %10zu %6s %8s | %10.2f %8.2f %8.1f %6ld\n", mat, rows, dt_name(dt), algo, tm.ms * 1e3, mat / (tm.ms * 1e3) / 1e3, rw / (tm.ms * 1e3) / 1e3,
             tm.errors);
      fflush(stdout);
    }
  }
  RT(cudaFree(gamma));
  if (scales) CC(b200collMemFree(ctx.comm, scales));
  return mode_result(ctx, total_errors);
}

// Routed mode (--route E:K). Per size, every rank holds tokens = size / row bytes tokens of x (k_fill values) and routes slot (t, j) to
// expert h(rank, t, j) % E, or drops it (id -1) every 61st slot; the hash is seeded, so every rank can draw every rank's ids on the host.
// recv holds tokens * K rows on every rank, the mean load, so some receivers clip and some do not. -c 1 repeats the layout on the host
// (per-expert counts, then each slot's row) and checks every byte of recv (stored rows, and the 0x5A poison elsewhere), every count,
// every route and dropped; then the combine (recv as the expert output, seeded weights) bit for bit against the slot-order reference.
// With --quantize WIRE:BLOCK it runs the FP8 routed dispatch instead: x holds the quantising mode's values (gen with BLOCK), recv FP8 rows
// and recv_scales one fp32 scale per block; -c 1 checks every FP8 byte and scale against the host quantiser (q_code) and the 0x5A
// poison of rows not stored in both, besides counts, routes and dropped. The combine needs a wide expert_out, so only the dispatch is timed.
static size_t route_scale_bytes(const Opts& o) {
  return o.route_e && o.q_block ? o.max_bytes / b200collTypeSize(o.in_dt) * o.route_k / o.q_block * 4 + 4096 : 0;
}
static int32_t ro_id(int rank, size_t t, int j, int E) {
  const uint32_t h = co_hash((uint32_t)(t * 0x9E3779B1u) ^ (uint32_t)(rank * 0x85EBCA77u) ^ (uint32_t)(j * 0xC2B2AE3Du));
  return h % 61 == 7 ? -1 : (int32_t)(h % (uint32_t)E);
}
static int run_route(const Opts& o, RankCtx& ctx, void* x) {
  const int n = ctx.nranks, rank = ctx.rank, E = o.route_e, K = o.route_k, epr = E / n;
  const bool quant = o.q_block > 0;
  const size_t is = b200collTypeSize(o.in_dt), os = b200collTypeSize(o.out_dt), row = o.row_len, rs = quant ? 1 : is;   // rs: bytes of a recv element
  const b200collEpilogue ep{o.in_dt, o.out_dt, o.scale};
  const cudaStream_t st = ctx.st;
  void* recv = nullptr;
  CC(b200collMemAlloc(ctx.comm, &recv, o.max_bytes * K + 4096));     // tokens * K rows at the largest size, the same on every rank
  float* recv_scales = nullptr;
  if (quant) CC(b200collMemAlloc(ctx.comm, (void**)&recv_scales, route_scale_bytes(o)));
  int32_t* small = nullptr;
  RT(cudaMalloc(&small, (size_t)(epr + 1) * 4));
  int32_t *d_counts = small, *d_dropped = small + epr;
  long total_errors = 0;
  if (rank == 0 && quant) {
    printf("# b200coll_perf op=alltoall routed FP8 dispatch experts=%d top_k=%d nranks=%d in=%s wire=%s block=%d row_len=%zu: size = x bytes per rank; combine not run\n",
           E, K, n, dt_name(o.in_dt), dt_name(o.q_wire), o.q_block, row);
  } else if (rank == 0 && o.cq_block) {
    printf("# b200coll_perf op=alltoall routed dispatch + quantising combine experts=%d top_k=%d nranks=%d in=%s wire=%s block=%d out=%s scale=%g row_len=%zu: "
           "size = x bytes per rank\n", E, K, n, dt_name(o.in_dt), dt_name(o.cq_wire), o.cq_block, dt_name(o.out_dt), o.scale, row);
  } else if (rank == 0) {
    printf("# b200coll_perf op=alltoall routed dispatch + combine experts=%d top_k=%d nranks=%d in=%s out=%s scale=%g row_len=%zu: size = x bytes per rank\n", E, K,
           n, dt_name(o.in_dt), dt_name(o.out_dt), o.scale, row);
  }
  if (rank == 0) {
    printf("#%13s %12s %6s %8s | %12s %12s %6s\n", "size(B)", "tokens", "type", "algo", "dispatch us", "combine us", "#wrong");
    fflush(stdout);
  }
  for (size_t bytes = o.min_bytes; bytes <= o.max_bytes; bytes *= o.factor) {
    const size_t tokens = bytes / is / row, slots = tokens * K, recv_rows = slots;
    if (tokens == 0) continue;
    // every rank's ids, counts and layout on the host
    std::vector<std::vector<int32_t>> ids(n, std::vector<int32_t>(slots));
    std::vector<std::vector<long long>> cnt(n, std::vector<long long>(E, 0));
    for (int s = 0; s < n; s++)
      for (size_t i = 0; i < slots; i++) { const int32_t e = ro_id(s, i / K, (int)(i % K), E); ids[s][i] = e; if (e >= 0) cnt[s][e]++; }
    std::vector<long long> total(E, 0), below(E, 0), base(E, 0);
    for (int e = 0; e < E; e++) for (int s = 0; s < n; s++) total[e] += cnt[s][e];
    for (int e = 1; e < E; e++) below[e] = below[e - 1] + total[e - 1];
    for (int e = 0; e < E; e++) base[e] = below[e] - below[e / epr * epr];
    // the row of every slot of every rank (-1: invalid id or past recv_rows)
    std::vector<std::vector<long long>> rowof(n, std::vector<long long>(slots, -1));
    for (int s = 0; s < n; s++) {
      std::vector<long long> seen(E, 0);
      for (size_t i = 0; i < slots; i++) {
        const int32_t e = ids[s][i];
        if (e < 0) continue;
        long long r = base[e] + seen[e]++;
        for (int q = 0; q < s; q++) r += cnt[q][e];
        if (r < (long long)recv_rows) rowof[s][i] = r;
      }
    }
    std::vector<float> w(slots);
    for (size_t i = 0; i < slots; i++) w[i] = 0.25f + (float)(co_hash((uint32_t)i * 31u + (uint32_t)rank) & 0xFFFFFF) * 0x1p-24f;
    int32_t *d_idx = nullptr, *d_route = nullptr; float* d_w = nullptr; void* out = nullptr;
    RT(cudaMalloc(&d_idx, slots * 4)); RT(cudaMalloc(&d_route, slots * 4)); RT(cudaMalloc(&d_w, slots * 4)); RT(cudaMalloc(&out, tokens * row * os));
    RT(cudaMemcpy(d_idx, ids[rank].data(), slots * 4, cudaMemcpyHostToDevice));
    RT(cudaMemcpy(d_w, w.data(), slots * 4, cudaMemcpyHostToDevice));
    const size_t nsc = quant ? recv_rows * row / o.q_block : 0;     // scales in recv_scales
    fill(x, tokens * row, o.in_dt, rank, st, o.q_block);
    RT(cudaMemsetAsync(recv, 0x5A, recv_rows * row * rs, st));
    if (quant) RT(cudaMemsetAsync(recv_scales, 0x5A, nsc * 4, st));
    auto dispatch = [&](int) {
      if (quant)
        CC(b200collExpertDispatchQuantized(x, recv, recv_scales, row, recv_rows, d_idx, tokens, K, E, d_counts, d_route, d_dropped, o.in_dt, o.q_wire, o.q_block,
                                           ctx.comm, st));
      else
        CC(b200collExpertDispatch(x, recv, row, recv_rows, d_idx, tokens, K, E, d_counts, d_route, d_dropped, o.in_dt, ctx.comm, st));
    };
    auto combine = [&](int) {
      if (o.cq_block) CC(b200collExpertCombineQuantized(recv, out, row, recv_rows, d_route, d_w, tokens, K, o.cq_wire, o.cq_block, &ep, ctx.comm, st));
      else CC(b200collExpertCombine(recv, out, row, recv_rows, d_route, d_w, tokens, K, &ep, ctx.comm, st));
    };
    long errs = 0;
    auto bad = [&](const char* what, size_t a, long long got, long long want) {
      if (errs < 4) fprintf(stderr, "rank %d route size %zu %s %zu: got %lld want %lld\n", rank, bytes, what, a, got, want);
      errs++;
    };
    if (o.check) {
      check_launch(o, ctx, [&](int) { dispatch(0); if (!quant) combine(0); });
      std::vector<unsigned char> h_recv(recv_rows * row * rs);
      std::vector<int32_t> h_route(slots), h_small(epr + 1);
      std::vector<char> h_out(tokens * row * os);
      RT(cudaMemcpy(h_recv.data(), recv, h_recv.size(), cudaMemcpyDeviceToHost));
      RT(cudaMemcpy(h_route.data(), d_route, slots * 4, cudaMemcpyDeviceToHost));
      RT(cudaMemcpy(h_small.data(), small, h_small.size() * 4, cudaMemcpyDeviceToHost));
      RT(cudaMemcpy(h_out.data(), out, h_out.size(), cudaMemcpyDeviceToHost));
      std::vector<float> h_scales(nsc);
      if (quant) RT(cudaMemcpy(h_scales.data(), recv_scales, nsc * 4, cudaMemcpyDeviceToHost));
      // recv: which (source, token) each of my rows holds
      std::vector<long long> src(recv_rows, -1);
      for (int s = 0; s < n; s++)
        for (size_t i = 0; i < slots; i++)
          if (rowof[s][i] >= 0 && ids[s][i] / epr == rank) src[rowof[s][i]] = (long long)s * tokens + (long long)(i / K);
      for (size_t r = 0; r < recv_rows && quant; r++) {      // FP8 bytes and scales from the host quantiser, or the poison
        QMemo memo;
        const int s = src[r] < 0 ? -1 : (int)(src[r] / (long long)tokens);
        const size_t t = src[r] < 0 ? 0 : (size_t)(src[r] % (long long)tokens);
        for (size_t e = 0; e < row; e++) {
          const size_t at = r * row + e;
          const long long got = h_recv[at], want = s < 0 ? 0x5A : (long long)q_code(o, s, t * row + e, &memo);
          if (got != want) bad("recv FP8 byte", at, got, want);
          if (e % o.q_block == 0) {
            const size_t j = at / o.q_block;
            const long long gs = out_bits(h_scales[j], b200collFloat32), ws = s < 0 ? 0x5A5A5A5All : (long long)out_bits(memo.s, b200collFloat32);
            if (gs != ws) bad("recv scale bits", j, gs, ws);
          }
        }
      }
      for (size_t r = 0; r < recv_rows && !quant; r++) {
        for (size_t e = 0; e < row; e++) {
          const size_t at = r * row + e;
          long long got = 0, want = 0;
          memcpy(&got, h_recv.data() + at * is, is);
          if (src[r] < 0) { want = is == 4 ? 0x5A5A5A5All : 0x5A5All; }
          else want = out_bits(gen((int)(src[r] / (long long)tokens), (size_t)(src[r] % (long long)tokens) * row + e), o.in_dt);
          if (got != want) bad("recv element", at, got, want);
        }
      }
      long long dropped = 0;
      for (int e = rank * epr; e < (rank + 1) * epr; e++) {
        const long long stored = std::min(std::max((long long)recv_rows - base[e], 0ll), total[e]);
        dropped += total[e] - stored;
        if (h_small[e - rank * epr] != stored) bad("expert_counts", (size_t)e, h_small[e - rank * epr], stored);
      }
      if (h_small[epr] != dropped) bad("dropped", 0, h_small[epr], dropped);
      for (size_t i = 0; i < slots; i++) {
        const long long want = rowof[rank][i] < 0 ? -1 : (long long)(ids[rank][i] / epr) * (long long)recv_rows + rowof[rank][i];
        if (h_route[i] != want) bad("route", i, h_route[i], want);
      }
      // the combine of identity experts: every stored slot of token t brings back t's own row (--combine-quantize: quantised and
      // dequantised, blocks along the row)
      std::vector<float> xrow(row);
      for (size_t t = 0; t < tokens && !quant; t++) {
        for (size_t e = 0; e < row; e++) xrow[e] = gen(rank, t * row + e);
        if (o.cq_block) q_roundtrip(xrow.data(), row, o.cq_block, o.cq_wire);
        for (size_t e = 0; e < row; e++) {
          float acc = 0.0f;
          for (int j = 0; j < K; j++) {
            if (rowof[rank][t * K + j] < 0) continue;
            volatile float prod = w[t * K + j] * xrow[e];
            acc = acc + prod;
          }
          const uint32_t want = out_bits(acc * o.scale, o.out_dt), got = got_bits(h_out.data(), t * row + e, o.out_dt);
          if (got != want) bad("combine element", t * row + e, got, want);
        }
      }
    }
    const Timing td = timed(o, ctx, errs, dispatch);                          // errors are counted with the dispatch only
    const Timing tc = quant ? Timing{0, 0} : timed(o, ctx, 0, combine);
    total_errors += td.errors;
    if (rank == 0 && quant) {
      printf("%14zu %12zu %6s %8s | %12.2f %12s %6ld\n", tokens * row * is, tokens, dt_name(o.in_dt), n > 1 ? "twoshot" : "copy", td.ms * 1e3, "-", td.errors);
      fflush(stdout);
    } else if (rank == 0) {
      printf("%14zu %12zu %6s %8s | %12.2f %12.2f %6ld\n", tokens * row * is, tokens, dt_name(o.in_dt), n > 1 ? "twoshot" : "copy", td.ms * 1e3, tc.ms * 1e3,
             td.errors);
      fflush(stdout);
    }
    RT(cudaFree(d_idx)); RT(cudaFree(d_route)); RT(cudaFree(d_w)); RT(cudaFree(out));
  }
  RT(cudaFree(small));
  return mode_result(ctx, total_errors);
}

// expected value of output element e (element index in the op's output) for this rank
static float expected(const Opts& o, int rank, int n, size_t e, size_t count) {
  if (o.op == "all_reduce" || o.op == "reduce") { float s = 0; for (int r = 0; r < n; r++) s += gen(r, e); return s * o.scale; }
  if (o.op == "broadcast") return gen(kRoot, e) * o.scale;
  if (o.op == "sendrecv") return gen((rank + n - 1) % n, e);      // ring step: my output is my left neighbour's input, untouched
  if (o.op == "all_gather" || o.op == "gather" || o.op == "hypercube") { int src = (int)(e / count); return gen(src, e % count) * o.scale; }
  if (o.op == "scatter") return gen(kRoot, (size_t)rank * count + e);
  if (o.op == "reduce_scatter") { float s = 0; for (int r = 0; r < n; r++) s += gen(r, (size_t)rank * count + e); return s * o.scale; }
  /* alltoall */ { int src = (int)(e / count); return gen(src, (size_t)rank * count + e % count) * o.scale; }
}

// Ulysses mode (--ulysses HQ:HKV:D). B = 1. Sequence -> heads: every rank's source is a packed QKV projection output [S_l, (HQ + 2 HKV) * D]
// whose q, k and v are column slices (row stride (HQ + 2 HKV) * D), moved by one b200collAllToAllSeqToHeads into three dense head shards
// [S, Hl, D]. --ulysses-back: the attention output, a dense [S, HQ / N, D] head shard, back to a dense [S_l, HQ, D] sequence shard. S_l is
// the largest token count whose source fits in `bytes`. Sources hold a hash of (rank, 32-bit word), so every misplaced byte shows; -c 1
// computes every output byte's source on the host. "rw GB/s" counts the source bytes read and the output bytes written.
static uint32_t uly_word(int rank, size_t w) { return co_hash((uint32_t)w * 2654435761u ^ (uint32_t)(w >> 32) ^ (uint32_t)rank * 0x9E3779B9u); }
static uint8_t uly_byte(int rank, size_t b) { return (uint8_t)(uly_word(rank, b / 4) >> (8 * (b % 4))); }
__global__ void k_uly_fill(uint32_t* p, size_t n, int rank) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t x = (uint32_t)i * 2654435761u ^ (uint32_t)(i >> 32) ^ (uint32_t)rank * 0x9E3779B9u;
    x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;     // co_hash
    p[i] = x;
  }
}
static size_t uly_local_heads(int n, int h) { return h % n == 0 ? (size_t)(h / n) : 1; }
// Output bytes per source byte, at most: the replicated heads are stored N / H times.
static size_t uly_out_bytes(const Opts& o, int n, size_t src_bytes) {
  if (o.uly_back) return src_bytes;
  const size_t in = (size_t)o.uly_hq + 2 * (size_t)o.uly_hkv, out = (size_t)n * (uly_local_heads(n, o.uly_hq) + 2 * uly_local_heads(n, o.uly_hkv));
  return src_bytes / in * out + 4096;
}
static int run_ulysses(const Opts& o, RankCtx& ctx) {
  const int n = ctx.nranks, rank = ctx.rank;
  const size_t es = b200collTypeSize(o.in_dt), D = (size_t)o.uly_d, hb = D * es;   // head bytes
  const int nt = o.uly_back ? 1 : 3;
  const int H[3] = {o.uly_hq, o.uly_hkv, o.uly_hkv};
  const size_t col[3] = {0, (size_t)o.uly_hq, (size_t)o.uly_hq + o.uly_hkv};     // the first head of q, k and v in the packed row
  const size_t src_row = o.uly_back ? (size_t)o.uly_hq / n * hb : ((size_t)o.uly_hq + 2 * (size_t)o.uly_hkv) * hb;   // source bytes per token row
  void *src = nullptr, *dst = nullptr;
  CC(b200collMemAlloc(ctx.comm, &src, o.max_bytes + 4096));
  CC(b200collMemAlloc(ctx.comm, &dst, uly_out_bytes(o, n, o.max_bytes + 4096)));
  const cudaStream_t st = ctx.st;
  long total_errors = 0;
  if (rank == 0) {
    printf("# b200coll_perf op=alltoall ulysses %s nranks=%d dtype=%s HQ=%d HKV=%d D=%zu B=1: size = source bytes per rank (%s); rw GB/s = "
           "(source read + output written) / time\n", o.uly_back ? "heads->seq" : "seq->heads", n, dt_name(o.in_dt), o.uly_hq, o.uly_hkv, D,
           o.uly_back ? "the attention output" : "q + k + v, packed");
    printf("#%13s %10s %6s %8s | %10s %8s %6s\n", "size(B)", "seq_local", "type", "algo", "us", "rwGB/s", "#wrong");
    fflush(stdout);
  }
  for (size_t bytes = o.min_bytes; bytes <= o.max_bytes; bytes *= o.factor) {
    const size_t sl = o.uly_back ? bytes / (src_row * n) : bytes / src_row;           // back: the source is [S = N * S_l, HQ / N, D]
    if (sl == 0) continue;
    const size_t S = sl * n, src_bytes = o.uly_back ? S * src_row : sl * src_row;
    b200collUlyssesTensor t[3];
    size_t out_off[3], out_bytes = 0;
    for (int i = 0; i < nt; i++) {
      out_off[i] = out_bytes;
      const size_t hl = uly_local_heads(n, H[i]);
      if (o.uly_back) t[i] = {dst, (size_t)o.uly_hq * D, src, o.uly_hq};
      else t[i] = {static_cast<char*>(src) + col[i] * hb, ((size_t)o.uly_hq + 2 * (size_t)o.uly_hkv) * D, static_cast<char*>(dst) + out_bytes, H[i]};
      out_bytes += o.uly_back ? sl * o.uly_hq * hb : S * hl * hb;
    }
    k_uly_fill<<<256, 256, 0, st>>>(static_cast<uint32_t*>(src), src_bytes / 4, rank);
    RT(cudaGetLastError());
    RT(cudaMemsetAsync(dst, 0x7B, out_bytes, st));
    auto launch = [&](int) {
      if (o.uly_back) CC(b200collAllToAllHeadsToSeq(t, nt, 1, sl, D, o.in_dt, ctx.comm, st));
      else CC(b200collAllToAllSeqToHeads(t, nt, 1, sl, D, o.in_dt, ctx.comm, st));
    };
    long errs = 0;
    if (o.check) {
      check_launch(o, ctx, launch);
      std::vector<uint8_t> host(out_bytes);
      RT(cudaMemcpy(host.data(), dst, out_bytes, cudaMemcpyDeviceToHost));
      for (int i = 0; i < nt; i++) {
        const size_t hl = uly_local_heads(n, H[i]);
        const uint8_t* got = host.data() + out_off[i];
        if (o.uly_back) {                     // x_r[t, h] = y_{h / Hl}[r * S_l + t, h % Hl]
          const size_t hlq = (size_t)o.uly_hq / n;
          for (size_t tk = 0; tk < sl; tk++)
            for (size_t h = 0; h < (size_t)o.uly_hq; h++)
              for (size_t e = 0; e < hb; e++) {
                const uint8_t want = uly_byte((int)(h / hlq), (((size_t)rank * sl + tk) * hlq + h % hlq) * hb + e), g = got[(tk * o.uly_hq + h) * hb + e];
                if (g != want) { if (errs < 4) fprintf(stderr, "rank %d ulysses back size %zu token %zu head %zu byte %zu: got 0x%02x want 0x%02x\n", rank, bytes, tk, h, e, g, want); errs++; }
              }
        } else {                              // y_r[s * S_l + t, j] = x_s[t, head(r, j)], x_s a column slice of the packed row
          for (size_t T = 0; T < S; T++)
            for (size_t j = 0; j < hl; j++) {
              const size_t s = T / sl, tk = T % sl, h = H[i] % n == 0 ? (size_t)rank * hl + j : (size_t)rank * H[i] / n;
              for (size_t e = 0; e < hb; e++) {
                const uint8_t want = uly_byte((int)s, tk * src_row + (col[i] + h) * hb + e), g = got[(T * hl + j) * hb + e];
                if (g != want) { if (errs < 4) fprintf(stderr, "rank %d ulysses tensor %d size %zu token %zu head %zu byte %zu: got 0x%02x want 0x%02x\n", rank, i, bytes, T, j, e, g, want); errs++; }
              }
            }
        }
      }
    }
    const Timing tm = timed(o, ctx, errs, launch);
    total_errors += tm.errors;
    if (rank == 0) {
      printf("%14zu %10zu %6s %8s | %10.2f %8.2f %6ld\n", src_bytes, sl, dt_name(o.in_dt), n > 1 ? "twoshot" : "copy", tm.ms * 1e3,
             (src_bytes + out_bytes) / (tm.ms * 1e3) / 1e3, tm.errors);
      fflush(stdout);
    }
  }
  CC(b200collMemFree(ctx.comm, dst));
  CC(b200collMemFree(ctx.comm, src));
  return mode_result(ctx, total_errors);
}

// Context-parallel mode (--context W:C or HQ:HKV:D:C). B = 1. --op all_gather: b200collAllGatherContext from each rank's shard, either K
// and V as column slices of a packed QKV projection output [S_l, (HQ + 2 HKV) * D] or one dense [S_l, W] tensor, into dense [S, W]
// full tensors (W = HKV * D) in token order. --op reduce_scatter: b200collReduceScatterContext from the full tensors back into the K and
// V column slices of a packed dQKV [S_l, (HQ + 2 HKV) * D] (its Q columns poisoned, and checked untouched) or into a dense [S_l, W].
// C = 1 contiguous sharding, 2 the load-balanced causal layout. The size is the shard bytes per rank (K + V, or the one tensor), rounded
// down to whole tokens (an even count with C = 2). Gather sources hold a hash of (rank, 32-bit word); reduce-scatter fulls hold seeded
// values with full mantissas, so the sums round. -c 1 checks every output byte on the host: the gather against the source byte the
// header's gtok places there, the reduce-scatter against the fp32 sum in rank order rounded once. "rw GB/s" counts the shard bytes and
// the full bytes this rank reads or writes.
__host__ __device__ inline float cp_val(int rank, size_t i) {
  uint32_t h = (uint32_t)(i * 2654435761u) ^ (uint32_t)(rank * 40503u + 0x9E3779B9u) ^ (uint32_t)(i >> 32);
  h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 12;
  return ((h >> 31) ? -1.0f : 1.0f) * ldexpf(1.0f + (float)(h & 0x7FFFFF) * 0x1p-23f, (int)((h >> 23) % 17) - 8);
}
template <typename T> __global__ void k_cp_fill(T* p, size_t n, int rank) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = T(cp_val(rank, i));
}
static bool cp_packed(const Opts& o) { return o.cp_d > 0; }
static size_t cp_width(const Opts& o) { return cp_packed(o) ? (size_t)o.cp_hkv * o.cp_d : o.cp_w; }          // elements per token of one tensor
static size_t cp_row(const Opts& o) { return cp_packed(o) ? ((size_t)o.cp_hq + 2 * (size_t)o.cp_hkv) * o.cp_d : o.cp_w; }   // shard row stride
static int cp_tensors(const Opts& o) { return cp_packed(o) ? 2 : 1; }
// The shard buffer (packed QKV / dQKV, or the dense tensor) and the full tensors, in bytes, for shards of at most max_bytes.
static size_t cp_shard_bytes(const Opts& o) { return o.max_bytes / (cp_tensors(o) * cp_width(o)) * cp_row(o) + 4096; }
static size_t cp_full_bytes(const Opts& o, int n) { return (size_t)n * o.max_bytes + 4096; }
static int run_context(const Opts& o, RankCtx& ctx) {
  const int n = ctx.nranks, rank = ctx.rank, C = o.cp_c, nt = cp_tensors(o);
  const bool gather = o.op == "all_gather";
  const b200collDataType_t dt = o.in_dt;
  const size_t es = b200collTypeSize(dt), W = cp_width(o), rowe = cp_row(o);
  const size_t col[2] = {cp_packed(o) ? (size_t)o.cp_hq * o.cp_d : 0, cp_packed(o) ? ((size_t)o.cp_hq + o.cp_hkv) * o.cp_d : 0};   // K and V columns
  void *shard = nullptr, *full = nullptr;
  CC(b200collMemAlloc(ctx.comm, &shard, cp_shard_bytes(o)));
  CC(b200collMemAlloc(ctx.comm, &full, cp_full_bytes(o, n)));
  const cudaStream_t st = ctx.st;
  long total_errors = 0;
  if (rank == 0) {
    printf("# b200coll_perf op=%s context nranks=%d dtype=%s chunks=%d B=1 %s: size = shard bytes per rank; rw GB/s = (shard + full bytes "
           "this rank reads or writes) / time\n", o.op.c_str(), n, dt_name(dt), C, cp_packed(o) ? "K and V column slices of a packed QKV" : "one dense tensor");
    if (cp_packed(o)) printf("# HQ=%d HKV=%d D=%d W=%zu\n", o.cp_hq, o.cp_hkv, o.cp_d, W);
    else printf("# W=%zu\n", W);
    printf("#%13s %10s %6s %8s | %10s %8s %6s\n", "size(B)", "seq_local", "type", "algo", "us", "rwGB/s", "#wrong");
    fflush(stdout);
  }
  for (size_t bytes = o.min_bytes; bytes <= o.max_bytes; bytes *= o.factor) {
    const size_t sl = bytes / (nt * W * es) / C * C;
    if (sl == 0) continue;
    const size_t S = sl * n, c = sl / C, shard_bytes = sl * nt * W * es, full_one = S * W * es;
    b200collContextTensor t[2];
    for (int i = 0; i < nt; i++) t[i] = {static_cast<char*>(shard) + col[i] * es, rowe, static_cast<char*>(full) + i * full_one, W};
    auto gtok = [&](int r, size_t tk) { const size_t k = tk / c; return (k == 0 ? (size_t)r : (size_t)(2 * n - 1 - r)) * c + tk % c; };
    if (gather) {
      k_uly_fill<<<256, 256, 0, st>>>(static_cast<uint32_t*>(shard), sl * rowe * es / 4, rank);
      RT(cudaGetLastError());
      RT(cudaMemsetAsync(full, 0x7B, nt * full_one, st));
    } else {
      if (dt == b200collFloat32) k_cp_fill<float><<<256, 256, 0, st>>>(static_cast<float*>(full), nt * S * W, rank);
      else if (dt == b200collFloat16) k_cp_fill<__half><<<256, 256, 0, st>>>(static_cast<__half*>(full), nt * S * W, rank);
      else k_cp_fill<__nv_bfloat16><<<256, 256, 0, st>>>(static_cast<__nv_bfloat16*>(full), nt * S * W, rank);
      RT(cudaGetLastError());
      RT(cudaMemsetAsync(shard, 0x7B, sl * rowe * es, st));
    }
    auto launch = [&](int) {
      if (gather) CC(b200collAllGatherContext(t, nt, 1, sl, C, dt, ctx.comm, st));
      else CC(b200collReduceScatterContext(t, nt, 1, sl, C, dt, ctx.comm, st));
    };
    long errs = 0;
    if (o.check) {
      check_launch(o, ctx, launch);
      if (gather) {                       // full[gtok(s, t)] = shard_s[t], a column slice of rank s's packed row
        std::vector<uint8_t> host(nt * full_one);
        RT(cudaMemcpy(host.data(), full, host.size(), cudaMemcpyDeviceToHost));
        for (int i = 0; i < nt; i++)
          for (int s = 0; s < n; s++)
            for (size_t tk = 0; tk < sl; tk++) {
              const uint8_t* got = host.data() + i * full_one + gtok(s, tk) * W * es;
              for (size_t e = 0; e < W * es; e++) {
                const uint8_t want = uly_byte(s, tk * rowe * es + col[i] * es + e);
                if (got[e] != want) {
                  if (errs < 4) fprintf(stderr, "rank %d context gather size %zu tensor %d from rank %d token %zu byte %zu: got 0x%02x want 0x%02x\n", rank, bytes, i, s, tk, e, got[e], want);
                  errs++;
                }
              }
            }
      } else {                            // shard[t] = round_once(sum over s in rank order of full_s[gtok(rank, t)]); other columns untouched
        std::vector<uint8_t> host(sl * rowe * es);
        RT(cudaMemcpy(host.data(), shard, host.size(), cudaMemcpyDeviceToHost));
        std::vector<bool> mine(rowe, false);
        for (int i = 0; i < nt; i++) for (size_t e = 0; e < W; e++) mine[col[i] + e] = true;
        for (size_t tk = 0; tk < sl; tk++) {
          const size_t g = gtok(rank, tk);
          for (size_t e = 0; e < rowe; e++) {
            const void* row = host.data() + tk * rowe * es;
            if (!mine[e]) {
              bool ok = true;
              for (size_t b = 0; b < es; b++) ok = ok && ((const uint8_t*)row)[e * es + b] == 0x7B;
              if (!ok) { if (errs < 4) fprintf(stderr, "rank %d context reduce-scatter size %zu token %zu column %zu: written, not one of ours\n", rank, bytes, tk, e); errs++; }
              continue;
            }
            const int i = (nt == 2 && e >= col[1]) ? 1 : 0;
            float acc = 0.0f;
            for (int s = 0; s < n; s++) acc += round_dt(cp_val(s, i * S * W + g * W + (e - col[i])), dt);
            const uint32_t want = out_bits(acc, dt), got = got_bits(row, e, dt);
            if (got != want) {
              if (errs < 4) fprintf(stderr, "rank %d context reduce-scatter size %zu token %zu column %zu: got 0x%x want 0x%x\n", rank, bytes, tk, e, got, want);
              errs++;
            }
          }
        }
      }
    }
    const Timing tm = timed(o, ctx, errs, launch);
    total_errors += tm.errors;
    if (rank == 0) {
      printf("%14zu %10zu %6s %8s | %10.2f %8.2f %6ld\n", shard_bytes, sl, dt_name(dt), n > 1 ? "twoshot" : "copy", tm.ms * 1e3,
             (shard_bytes + nt * full_one) / (tm.ms * 1e3) / 1e3, tm.errors);
      fflush(stdout);
    }
  }
  CC(b200collMemFree(ctx.comm, full));
  CC(b200collMemFree(ctx.comm, shard));
  return mode_result(ctx, total_errors);
}

// FSDP mode (--fsdp H:F[:KV]). One Llama block's nine tensors, in this order: q [H, H], k [KV, H], v [KV, H], o [H, H], gate [F, H],
// up [F, H], down [H, F], and the attention and MLP norm weights [H] (KV = H by default). Tensor i is sharded along dim 0 with p_i =
// ceil(d_i / N) rows per rank, rounded up until p_i * W_i is a whole number of 16-byte vectors. --op all_gather: b200collAllGatherShards
// from -d shards (float with --out-dtype bfloat16|half: the cast) into --out-dtype fulls. --op reduce_scatter: b200collReduceScatterShards
// from -d gradients into --out-dtype shards (bfloat16|half -> float), times --scale, added to the old shard with --accumulate. Every
// tensor lives in the arena, the fulls back to back at 256-byte offsets in one buffer and the shards in another. Bit-copy gather sources
// hold a hash of (rank, 32-bit word); cast sources, gradients and old shards hold seeded values with full mantissas (cp_val), so casts
// and sums round. -c 1 checks every output element on the host: the gather against the source bits or their cast, the reduce-scatter
// against t = sum over ranks in rank order from +0, t * scale, old + t, rounded once. The size is the block's bytes in the full dtype;
// "rw GB/s" counts the shard and full bytes this rank reads or writes.
struct FsTensor { size_t d, W, p, foff, soff; };      // rows, width, rows per rank, byte offsets in the full and shard buffers
static std::vector<FsTensor> fs_tensors(const Opts& o, int n, size_t* full_bytes, size_t* shard_bytes) {
  const size_t H = o.fs_h, F = o.fs_f, KV = o.fs_kv ? o.fs_kv : o.fs_h;
  const size_t ess = b200collTypeSize(o.op == "all_gather" ? o.in_dt : o.out_dt), esf = b200collTypeSize(o.op == "all_gather" ? o.out_dt : o.in_dt);
  const size_t es = std::min(ess, esf);
  const size_t shapes[9][2] = {{H, H}, {KV, H}, {KV, H}, {H, H}, {F, H}, {F, H}, {H, F}, {H, 1}, {H, 1}};
  std::vector<FsTensor> ts;
  size_t fo = 0, so = 0;
  for (const auto& sh : shapes) {
    FsTensor t{sh[0], sh[1], (sh[0] + n - 1) / n, fo, so};
    while ((t.p * t.W * es) % 16) t.p++;
    fo += (t.d * t.W * esf + 255) / 256 * 256;
    so += (t.p * t.W * ess + 255) / 256 * 256;
    ts.push_back(t);
  }
  *full_bytes = fo; *shard_bytes = so;
  return ts;
}
static size_t fs_arena_bytes(const Opts& o) {
  size_t fb = 0, sb = 0;
  fs_tensors(o, o.nranks, &fb, &sb);
  return fb + sb + 8192;
}
static int run_fsdp(const Opts& o, RankCtx& ctx) {
  const int n = ctx.nranks, rank = ctx.rank;
  const bool gather = o.op == "all_gather";
  const b200collDataType_t sdt = gather ? o.in_dt : o.out_dt, fdt = gather ? o.out_dt : o.in_dt;
  const size_t ess = b200collTypeSize(sdt), esf = b200collTypeSize(fdt);
  size_t full_bytes = 0, shard_bytes = 0;
  const std::vector<FsTensor> ts = fs_tensors(o, n, &full_bytes, &shard_bytes);
  void *full = nullptr, *shard = nullptr;
  CC(b200collMemAlloc(ctx.comm, &full, full_bytes));
  CC(b200collMemAlloc(ctx.comm, &shard, shard_bytes));
  std::vector<b200collShardTensor> desc;
  size_t unit = 0, mine = 0;                         // the block's bytes in the full dtype; this rank's rows of it
  auto own = [&](const FsTensor& t, int r) { const size_t f = std::min(t.d, (size_t)r * t.p); return std::min(t.d - f, t.p); };
  for (const FsTensor& t : ts) {
    desc.push_back({static_cast<char*>(shard) + t.soff, static_cast<char*>(full) + t.foff, t.d, t.W, t.p});
    unit += t.d * t.W * esf;
    mine += own(t, rank) * t.W * esf;
  }
  const bool cast_in = gather && sdt != fdt;
  const cudaStream_t st = ctx.st;
  if (gather) {
    if (cast_in) k_cp_fill<float><<<256, 256, 0, st>>>(static_cast<float*>(shard), shard_bytes / 4, rank);
    else k_uly_fill<<<256, 256, 0, st>>>(static_cast<uint32_t*>(shard), shard_bytes / 4, rank);
    RT(cudaGetLastError());
    RT(cudaMemsetAsync(full, 0x7B, full_bytes, st));
  } else {
    if (fdt == b200collFloat32) k_cp_fill<float><<<256, 256, 0, st>>>(static_cast<float*>(full), full_bytes / 4, rank);
    else if (fdt == b200collFloat16) k_cp_fill<__half><<<256, 256, 0, st>>>(static_cast<__half*>(full), full_bytes / 2, rank);
    else k_cp_fill<__nv_bfloat16><<<256, 256, 0, st>>>(static_cast<__nv_bfloat16*>(full), full_bytes / 2, rank);
    if (sdt == b200collFloat32) k_cp_fill<float><<<256, 256, 0, st>>>(static_cast<float*>(shard), shard_bytes / 4, 1000 + rank);
    else if (sdt == b200collFloat16) k_cp_fill<__half><<<256, 256, 0, st>>>(static_cast<__half*>(shard), shard_bytes / 2, 1000 + rank);
    else k_cp_fill<__nv_bfloat16><<<256, 256, 0, st>>>(static_cast<__nv_bfloat16*>(shard), shard_bytes / 2, 1000 + rank);
    RT(cudaGetLastError());
  }
  if (rank == 0) {
    printf("# b200coll_perf op=%s fsdp nranks=%d %s -> %s H=%d F=%d KV=%d tensors=9%s%s: size = the block's bytes in the full dtype; rw GB/s = "
           "(shard + full bytes this rank reads or writes) / time\n", o.op.c_str(), n, dt_name(gather ? sdt : fdt), dt_name(gather ? fdt : sdt),
           o.fs_h, o.fs_f, o.fs_kv ? o.fs_kv : o.fs_h, gather ? "" : (o.accumulate ? " accumulate" : " overwrite"), gather ? "" : (" scale=" + std::to_string(o.scale)).c_str());
    printf("#%13s %6s %8s | %10s %8s %6s\n", "size(B)", "type", "algo", "us", "rwGB/s", "#wrong");
    fflush(stdout);
  }
  auto launch = [&](int) {
    if (gather) CC(b200collAllGatherShards(desc.data(), (int)desc.size(), sdt, fdt, ctx.comm, st));
    else CC(b200collReduceScatterShards(desc.data(), (int)desc.size(), fdt, sdt, o.scale, o.accumulate ? 1 : 0, ctx.comm, st));
  };
  long errs = 0;
  if (o.check) {
    check_launch(o, ctx, launch);
    if (gather) {                        // full[s * p + j] = cast(shard_s[j]) for every rank s
      std::vector<uint8_t> host(full_bytes);
      RT(cudaMemcpy(host.data(), full, full_bytes, cudaMemcpyDeviceToHost));
      for (size_t i = 0; i < ts.size(); i++) {
        const FsTensor& t = ts[i];
        for (int s = 0; s < n; s++)
          for (size_t e = 0; e < own(t, s) * t.W; e++) {
            const size_t fe = s * t.p * t.W + e;                                 // element of the full tensor
            uint32_t want = 0, got = 0;
            if (cast_in) {
              want = out_bits(cp_val(s, t.soff / 4 + e), fdt);
              got = got_bits(host.data() + t.foff, fe, fdt);
            } else {
              for (size_t b = 0; b < esf; b++) {
                want |= (uint32_t)uly_byte(s, t.soff + e * esf + b) << (8 * b);
                got |= (uint32_t)host[t.foff + fe * esf + b] << (8 * b);
              }
            }
            if (got != want) {
              if (errs < 4) fprintf(stderr, "rank %d fsdp gather tensor %zu from rank %d element %zu: got 0x%x want 0x%x\n", rank, i, s, e, got, want);
              errs++;
            }
          }
      }
    } else {                             // shard[j] = round_once(old + (sum over s in rank order of full_s[r p + j]) * scale)
      std::vector<uint8_t> host(shard_bytes);
      RT(cudaMemcpy(host.data(), shard, shard_bytes, cudaMemcpyDeviceToHost));
      const bool bit_copy = n == 1 && sdt == fdt && o.scale == 1.0f && !o.accumulate;
      for (size_t i = 0; i < ts.size(); i++) {
        const FsTensor& t = ts[i];
        for (size_t e = 0; e < own(t, rank) * t.W; e++) {
          const size_t fe = t.foff / esf + rank * t.p * t.W + e;              // element of the full buffer
          float acc = 0.0f;
          for (int s = 0; s < n; s++) acc = acc + round_dt(cp_val(s, fe), fdt);
          acc = acc * o.scale;
          if (o.accumulate) acc = round_dt(cp_val(1000 + rank, t.soff / ess + e), sdt) + acc;
          const uint32_t want = bit_copy ? out_bits(round_dt(cp_val(0, fe), fdt), fdt) : out_bits(acc, sdt);
          const uint32_t got = got_bits(host.data() + t.soff, e, sdt);
          if (got != want) {
            if (errs < 4) fprintf(stderr, "rank %d fsdp reduce-scatter tensor %zu element %zu: got 0x%x want 0x%x\n", rank, i, e, got, want);
            errs++;
          }
        }
      }
    }
  }
  const Timing tm = timed(o, ctx, errs, launch);
  if (rank == 0) {
    const size_t rw = gather ? mine / esf * ess + (size_t)n * mine : mine * n + mine / esf * ess * (o.accumulate ? 2 : 1);
    printf("%14zu %6s %8s | %10.2f %8.2f %6ld\n", unit, dt_name(fdt), n > 1 ? "twoshot" : "copy", tm.ms * 1e3, rw / (tm.ms * 1e3) / 1e3, tm.errors);
    fflush(stdout);
  }
  CC(b200collMemFree(ctx.comm, shard));
  CC(b200collMemFree(ctx.comm, full));
  return mode_result(ctx, tm.errors);
}

static int run_rank(const Opts& o, RankCtx ctx) {
  const int n = ctx.nranks, rank = ctx.rank;
  RT(cudaSetDevice(ctx.dev));
  RT(cudaStreamCreateWithFlags(&ctx.st, cudaStreamNonBlocking));
  RT(cudaEventCreate(&ctx.e0)); RT(cudaEventCreate(&ctx.e1));
  const cudaStream_t st = ctx.st;
  if (o.algo != "auto") {
    for (int a = 0; a < b200collNumAlgos; a++) if (o.algo == b200collAlgoName((b200collAlgo_t)a)) CC(b200collCommSetAlgo(ctx.comm, (b200collAlgo_t)a));
  }
  if (o.max_ctas > 0) CC(b200collCommSetMaxCtas(ctx.comm, o.max_ctas));
  if (o.uly_d) return run_ulysses(o, ctx);
  if (o.cp_c) return run_context(o, ctx);
  if (o.fs_h) return run_fsdp(o, ctx);
  const size_t is = b200collTypeSize(o.in_dt), os = b200collTypeSize(o.out_dt);
  const bool is_bc = o.op == "broadcast", is_rd = o.op == "reduce", is_sr = o.op == "sendrecv";
  const bool is_ar = o.op == "all_reduce" || is_bc || is_rd || is_sr;      // "whole message" geometry: count elements in, count out
  const bool is_hc = o.op == "hypercube";          // nccl-tests hypercube_perf: an all-gather made of log2(n) pairwise exchanges of doubling size
  const bool is_ga = o.op == "gather" || is_hc, is_sc = o.op == "scatter";                 // nccl-tests gather_perf / scatter_perf: one send/recv group around the root
  const bool is_ag = o.op == "all_gather" || is_ga, is_rs = o.op == "reduce_scatter" || is_sc;      // same buffer geometry
  // nccl-tests convention: "size" is the larger of the two buffers in bytes of the input type
  const size_t max_in_bytes = o.max_bytes, max_out_bytes = o.max_bytes / is * os;
  const size_t send_cap = std::max(o.window, max_in_bytes), recv_cap = std::max(o.window / is * os, max_out_bytes);
  void *send = nullptr, *recv = nullptr;
  CC(b200collMemAlloc(ctx.comm, &send, send_cap + 4096));
  CC(b200collMemAlloc(ctx.comm, &recv, recv_cap + 4096));
  if (o.rms_row) {
    void* residual = nullptr;
    CC(b200collMemAlloc(ctx.comm, &residual, max_in_bytes + 4096));
    return run_rms(o, ctx, send, recv, residual);
  }
  if (o.combine_k) return run_combine(o, ctx, send, recv);
  if (o.route_e) return run_route(o, ctx, send);
  const bool bs_mode = o.bs_rows > 0, q_mode = o.q_block > 0, is_a2a = o.op == "alltoall";
  float* q_scales = nullptr;                                     // quantising alltoall: the received scales, one window of them
  if (q_mode && is_a2a) CC(b200collMemAlloc(ctx.comm, (void**)&q_scales, q_a2a_scale_bytes(o)));
  float* scales = nullptr;
  std::vector<float> host_scales;
  if (bs_mode) CC(b200collMemAlloc(ctx.comm, (void**)&scales, bs_max_scales(o) * 4));
  b200collEpilogue ep{o.in_dt, o.out_dt, o.scale};
  std::vector<char> host;
  b200collCommInfo info; CC(b200collCommInfoGet(ctx.comm, &info));
  if (rank == 0) {
    printf("# b200coll_perf op=%s nranks=%d in=%s out=%s scale=%g algo=%s nvls=%d loopback=%d mode=%s\n", o.op.c_str(), n, dt_name(o.in_dt), dt_name(o.out_dt), o.scale, o.algo.c_str(),
           info.nvls, info.same_device_loopback, o.procs ? "procs" : "threads");
    if (bs_mode) printf("# block-scaled: row_len=%zu block=%dx%d (one fp32 scale per block, seeded)\n", o.row_len, o.bs_rows, o.bs_cols);
    if (q_mode) printf("# quantised: wire=%s block=%d (each rank quantises its input, one fp32 scale per block)\n", dt_name(o.q_wire), o.q_block);
    if (q_mode && is_a2a) printf("# all-to-all-v: an even split of whole %zu-element rows to every peer; FP8 rows and scales are checked\n", o.row_len);
    printf("#%13s %12s %6s %8s | %10s %8s %8s %6s | %10s %8s %8s %6s\n", "size(B)", "count", "type", "algo", "oop us", "algbw", "busbw", "#wrong", "ip us", "algbw", "busbw", "#wrong");
    fflush(stdout);
  }
  FILE* jf = (rank == 0 && !o.json.empty()) ? fopen(o.json.c_str(), "a") : nullptr;
  long total_errors = 0;
  double busbw_sum = 0; int busbw_n = 0;   // nccl-tests' "Avg bus bandwidth": mean over every (size, placement) measured
  for (size_t bytes = o.min_bytes; bytes <= o.max_bytes; bytes *= o.factor) {
    // element counts per the op
    size_t count;          // the `count` argument of the API
    size_t in_elems, out_elems;
    if (is_ar) { count = bytes / is; in_elems = out_elems = count; }
    else if (is_ag) { count = bytes / is / n; in_elems = count; out_elems = count * n; }
    else if (is_rs) { count = bytes / is / n; in_elems = count * n; out_elems = count; }
    else { count = bytes / is / n; in_elems = out_elems = count * n; }
    const size_t E = 16 / is;
    if (!is_ar) count = count / E * E;
    if (bs_mode) count = count / o.row_len * o.row_len;      // whole rows on every rank (reduce-scatter: rows = n * count / row_len)
    if (q_mode) count = count / o.q_block * o.q_block;       // whole blocks on every rank (reduce-scatter: every slice)
    if (q_mode && is_a2a) count = count / o.row_len * o.row_len;      // whole rows to every peer
    if (count == 0) continue;
    // quantising alltoall: rpp rows to every peer; rank r's rows for p start at row p * rpp and land at row r * rpp of p's recv
    const size_t rpp = count / o.row_len;
    std::vector<int64_t> a2a_rows(n, (int64_t)rpp), a2a_soff(n), a2a_roff(n, (int64_t)(rank * rpp));
    for (int p = 0; p < n; p++) a2a_soff[p] = (int64_t)(p * rpp);
    const size_t bs_rows_total = bs_mode ? (is_rs ? count * n : count) / o.row_len : 0;
    const size_t bs_ncb = bs_mode ? (o.row_len + o.bs_cols - 1) / o.bs_cols : 0;
    const size_t bs_nscales = bs_mode ? (bs_rows_total + o.bs_rows - 1) / o.bs_rows * bs_ncb : 0;
    if (bs_mode) {
      host_scales.resize(bs_nscales);
      for (size_t k = 0; k < bs_nscales; k++) host_scales[k] = bs_scale(rank, k);
      RT(cudaMemcpy(scales, host_scales.data(), bs_nscales * 4, cudaMemcpyHostToDevice));
    }
    const b200collBlockScale bsd{scales, o.row_len, o.bs_rows, o.bs_cols};
    // value of element i of rank r's send matrix, dequantised (one fp32 multiply)
    auto bs_val = [&](int r, size_t i) { return gen(r, i) * bs_scale(r, (i / o.row_len / o.bs_rows) * bs_ncb + (i % o.row_len) / o.bs_cols); };
    if (!is_ar) { in_elems = is_ag ? count : count * n; out_elems = is_rs ? count : count * n; }
    const size_t in_b = in_elems * is, out_b = out_elems * os;
    const size_t slot_b = (std::max(in_b, out_b / os * is) + 4095) / 4096 * 4096;
    int slots = (int)std::min<size_t>(64, std::max<size_t>(1, o.window / slot_b));
    const size_t nshapes = o.shapes.empty() ? 1 : o.shapes.size();
    for (size_t si = 0; si < nshapes; si++) {
    if (!o.shapes.empty()) CC(b200collCommSetLaunchShape(ctx.comm, o.shapes[si].kind, o.shapes[si].ctas, o.shapes[si].threads));
    double res_us[2] = {-1, -1}; long res_err[2] = {0, 0};
    const char* algo_used = "?";
    for (int ip = 0; ip < 2; ip++) {
      if ((ip == 0 && o.inplace == 1) || (ip == 1 && o.inplace == 0)) continue;
      if (ip == 1 && (o.op == "alltoall" || is_sr || is_ga || is_sc || is != os)) continue;
      if (ip == 1 && q_mode && !is_ar) continue;              // the quantising all-gather and reduce-scatter refuse overlapping buffers
      auto sbuf = [&](int slot) -> char* {
        char* base = ip ? (char*)recv : (char*)send;
        size_t off = (size_t)slot * slot_b;
        if (ip && is_ag) off += (size_t)rank * count * os;     // in-place all-gather: send = recv + rank*count
        return base + off;
      };
      auto rbuf = [&](int slot) -> char* {
        size_t off = (size_t)slot * (ip ? slot_b : slot_b / is * os);
        if (ip && is_rs) off += (size_t)rank * count * is;     // in-place reduce-scatter: recv = send + rank*count
        return (char*)recv + off;
      };
      auto qsbuf = [&](int slot) -> float* { return q_scales + (size_t)slot * (slot_b / is / o.q_block); };   // the scales of rbuf(slot)
      auto launch = [&](int slot) {
        if (is_hc) {
          RT(cudaMemcpyAsync(rbuf(slot) + (size_t)rank * count * is, sbuf(slot), count * is, cudaMemcpyDeviceToDevice, st));
          for (int mask = 1; mask < n; mask <<= 1) {      // after the step with this mask every rank holds the 2*mask blocks of its sub-cube
            const int peer = rank ^ mask, mine0 = rank & ~(mask - 1), theirs0 = peer & ~(mask - 1);
            CC(b200collGroupStart());
            CC(b200collSend(rbuf(slot) + (size_t)mine0 * count * is, (size_t)mask * count * is, peer, ctx.comm, st));
            CC(b200collRecv(rbuf(slot) + (size_t)theirs0 * count * is, (size_t)mask * count * is, peer, ctx.comm, st));
            CC(b200collGroupEnd());
          }
        } else if (is_ga) {
          CC(b200collGroupStart());
          CC(b200collSend(sbuf(slot), count * is, kRoot, ctx.comm, st));
          if (rank == kRoot) for (int p = 0; p < n; p++) CC(b200collRecv(rbuf(slot) + (size_t)p * count * is, count * is, p, ctx.comm, st));
          CC(b200collGroupEnd());
        } else if (is_sc) {
          CC(b200collGroupStart());
          if (rank == kRoot) for (int p = 0; p < n; p++) CC(b200collSend(sbuf(slot) + (size_t)p * count * is, count * is, p, ctx.comm, st));
          CC(b200collRecv(rbuf(slot), count * is, kRoot, ctx.comm, st));
          CC(b200collGroupEnd());
        }
        else if (is_sr) {      // nccl-tests sendrecv_perf: one grouped send to the right neighbour and recv from the left one
          CC(b200collGroupStart());
          CC(b200collSend(sbuf(slot), count * is, (rank + 1) % n, ctx.comm, st));
          CC(b200collRecv(rbuf(slot), count * is, (rank + n - 1) % n, ctx.comm, st));
          CC(b200collGroupEnd());
        }
        else if (q_mode && is_ar) CC(b200collAllReduceQuantized(sbuf(slot), rbuf(slot), count, o.q_wire, o.q_block, &ep, b200collSum, ctx.comm, st));
        else if (q_mode && is_ag) CC(b200collAllGatherQuantized(sbuf(slot), rbuf(slot), count, o.q_wire, o.q_block, &ep, ctx.comm, st));
        else if (q_mode && is_rs) CC(b200collReduceScatterQuantized(sbuf(slot), rbuf(slot), count, o.q_wire, o.q_block, &ep, b200collSum, ctx.comm, st));
        else if (q_mode && is_a2a)
          CC(b200collAllToAllvQuantized(sbuf(slot), rbuf(slot), qsbuf(slot), o.row_len, rpp * n, a2a_rows.data(), a2a_soff.data(), a2a_roff.data(), o.in_dt, o.q_wire,
                                        o.q_block, ctx.comm, st));
        else if (bs_mode && is_ar) CC(b200collAllReduceBlockScaled(sbuf(slot), rbuf(slot), count, &bsd, &ep, b200collSum, ctx.comm, st));
        else if (bs_mode && is_ag) CC(b200collAllGatherBlockScaled(sbuf(slot), rbuf(slot), count, &bsd, &ep, ctx.comm, st));
        else if (bs_mode && is_rs) CC(b200collReduceScatterBlockScaled(sbuf(slot), rbuf(slot), count, &bsd, &ep, b200collSum, ctx.comm, st));
        else if (is_bc) CC(b200collBroadcast(sbuf(slot), rbuf(slot), count, &ep, kRoot, ctx.comm, st));
        else if (is_rd) CC(b200collReduce(sbuf(slot), rbuf(slot), count, &ep, b200collSum, kRoot, ctx.comm, st));
        else if (is_ar) CC(b200collAllReduce(sbuf(slot), rbuf(slot), count, &ep, b200collSum, ctx.comm, st));
        else if (is_ag) CC(b200collAllGather(sbuf(slot), rbuf(slot), count, &ep, ctx.comm, st));
        else if (is_rs) CC(b200collReduceScatter(sbuf(slot), rbuf(slot), count, &ep, b200collSum, ctx.comm, st));
        else CC(b200collAllToAll(sbuf(slot), rbuf(slot), count, &ep, ctx.comm, st));
      };
      // ---- correctness on slot 0 (fresh data, poisoned output)
      long errs = 0;
      if (o.check) {
        if (!ip) RT(cudaMemsetAsync(rbuf(0), 0x5A, out_b, st));
        if (q_mode && is_a2a) RT(cudaMemsetAsync(qsbuf(0), 0x5A, out_elems / o.q_block * 4, st));
        fill(sbuf(0), in_elems, o.in_dt, rank, st, o.q_block);       // in-place reduce-scatter: sbuf(0) is recv
        check_launch(o, ctx, launch);
        const char* outp = (ip && is_rs) ? rbuf(0) : (ip ? (char*)recv : rbuf(0));
        const size_t check_elems = ((is_rd || (is_ga && !is_hc)) && rank != kRoot) ? 0 : out_elems;   // a rooted reduce defines the root's output only
        host.resize(check_elems * os);
        RT(cudaMemcpy(host.data(), outp, check_elems * os, cudaMemcpyDeviceToHost));
        const size_t stride = check_elems > (1u << 22) ? 61 : 1;   // sample large buffers
        for (size_t e = 0; e < check_elems && bs_mode; e += stride) {      // bit for bit: ((0 + v_0) + v_1 + ...) * scale, rounded once
          float acc = 0.0f;
          if (is_ag) acc += bs_val((int)(e / count), e % count);
          else for (int r = 0; r < n; r++) acc += bs_val(r, is_rs ? (size_t)rank * count + e : e);
          const uint32_t want = out_bits(acc * o.scale, o.out_dt), got = got_bits(host.data(), e, o.out_dt);
          if (got != want) { if (errs < 4) fprintf(stderr, "rank %d %s block-scaled size %zu elem %zu: got bits 0x%x want 0x%x\n", rank, o.op.c_str(), bytes, e, got, want); errs++; }
        }
        std::vector<QMemo> memo(n);
        if (q_mode && is_a2a) {      // bit for bit: my recv element e is rank e / count's element rank * count + e % count, quantised
          for (size_t e = 0; e < check_elems; e += stride) {
            const int src = (int)(e / count);
            const uint32_t want = q_code(o, src, (size_t)rank * count + e % count, &memo[src]), got = (unsigned char)host[e];
            if (got != want) { if (errs < 4) fprintf(stderr, "rank %d alltoall quantised size %zu elem %zu: got FP8 0x%x want 0x%x\n", rank, bytes, e, got, want); errs++; }
          }
          const size_t nsc = out_elems / o.q_block, sstride = nsc > (1u << 18) ? 61 : 1;
          std::vector<float> got_s(nsc);
          RT(cudaMemcpy(got_s.data(), qsbuf(0), nsc * 4, cudaMemcpyDeviceToHost));
          std::vector<QMemo> smemo(n);
          for (size_t j = 0; j < nsc; j += sstride) {
            const size_t e = j * o.q_block;
            const int src = (int)(e / count);
            q_code(o, src, (size_t)rank * count + e % count, &smemo[src]);
            const uint32_t want = out_bits(smemo[src].s, b200collFloat32), got = out_bits(got_s[j], b200collFloat32);
            if (got != want) { if (errs < 4) fprintf(stderr, "rank %d alltoall quantised size %zu scale %zu: got bits 0x%x want 0x%x\n", rank, bytes, j, got, want); errs++; }
          }
        }
        for (size_t e = 0; e < check_elems && q_mode && !is_a2a; e += stride) {      // bit for bit: ((0 + v_0) + v_1 + ...) * scale, rounded once
          float acc = 0.0f;
          if (is_ag) acc += q_val(o, (int)(e / count), e % count, &memo[e / count]);
          else for (int r = 0; r < n; r++) acc += q_val(o, r, is_rs ? (size_t)rank * count + e : e, &memo[r]);
          const uint32_t want = out_bits(acc * o.scale, o.out_dt), got = got_bits(host.data(), e, o.out_dt);
          if (got != want) { if (errs < 4) fprintf(stderr, "rank %d %s quantised size %zu %s elem %zu: got bits 0x%x want 0x%x\n", rank, o.op.c_str(), bytes, ip ? "ip" : "oop", e, got, want); errs++; }
        }
        for (size_t e = 0; e < check_elems && !bs_mode && !q_mode; e += stride) {
          const float want = expected(o, rank, n, e, count), got = to_f(host.data(), e, o.out_dt);
          // FP8 outputs round once: half an ulp is 2^-4 (e4m3) or 2^-3 (e5m2) of the value
          const float tol = o.out_dt == b200collFloat8e4m3 ? fabsf(want) * 0.0725f + 0.002f : o.out_dt == b200collFloat8e5m2 ? fabsf(want) * 0.135f + 0.002f : 0.0f;
          if (!(fabsf(got - want) <= tol)) { if (errs < 4) fprintf(stderr, "rank %d %s size %zu %s elem %zu: got %g want %g\n", rank, o.op.c_str(), bytes, ip ? "ip" : "oop", e, got, want); errs++; }
        }
      }
      const Timing tm = timed(o, ctx, errs, [&](int i) { launch(i % slots); });
      res_us[ip] = tm.ms * 1e3; res_err[ip] = tm.errors; total_errors += tm.errors;
    }
    if (rank == 0) {
      size_t tb = is_ar ? count * is : count * is * n;   // nccl-tests "size"
      b200collOp_t opid = is_bc ? b200collOpBroadcast : is_rd ? b200collOpReduce : is_ar ? b200collOpAllReduce : is_ag ? b200collOpAllGather : is_rs ? b200collOpReduceScatter : b200collOpAllToAll;
      if (is_sr || is_ga || is_sc) algo_used = "p2p";
      else if (q_mode && is_a2a) algo_used = n > 1 ? "twoshot" : "copy";
      else if (o.algo == "auto") algo_used = b200collAlgoName(b200collTunerPick(opid, is_ar ? count * is : count * is, n, info.nvls)); else algo_used = o.algo.c_str();
      const double factor = (is_bc || is_rd || is_sr) ? 1.0 : is_ar ? 2.0 * (n - 1) / n : (double)(n - 1) / n;
      double ab[2], bb[2];
      for (int ip = 0; ip < 2; ip++) { ab[ip] = res_us[ip] > 0 ? tb / res_us[ip] / 1e3 : 0; bb[ip] = n > 1 ? ab[ip] * factor : ab[ip]; if (res_us[ip] > 0) { busbw_sum += bb[ip]; busbw_n++; } }
      if (!o.shapes.empty()) printf("[k%d c%d t%d] ", o.shapes[si].kind, o.shapes[si].ctas, o.shapes[si].threads);
      printf("%14zu %12zu %6s %8s | %10.2f %8.2f %8.2f %6ld | %10.2f %8.2f %8.2f %6ld\n", tb, count, dt_name(o.in_dt), algo_used, res_us[0], ab[0], bb[0], res_err[0], res_us[1], ab[1], bb[1], res_err[1]);
      fflush(stdout);
      if (jf) {
        fprintf(jf, "{\"op\":\"%s\",\"nranks\":%d,\"bytes\":%zu,\"in\":\"%s\",\"out\":\"%s\",\"scale\":%g,\"algo\":\"%s\",\"oop_us\":%.3f,\"ip_us\":%.3f,\"oop_busbw\":%.3f,\"ip_busbw\":%.3f,\"errors\":%ld,\"mode\":\"%s\",\"shape\":\"%d:%d:%d\"}\n",
                o.op.c_str(), n, tb, dt_name(o.in_dt), dt_name(o.out_dt), o.scale, algo_used, res_us[0], res_us[1], bb[0], bb[1], res_err[0] + res_err[1], o.procs ? "procs" : "threads", o.shapes.empty() ? -1 : o.shapes[si].kind, o.shapes.empty() ? 0 : o.shapes[si].ctas, o.shapes.empty() ? 0 : o.shapes[si].threads);
        fflush(jf);
      }
    }
    }   // shapes
  }
  if (jf) fclose(jf);
  b200collStats s; CC(b200collCommStatsGet(ctx.comm, &s));
  if (rank == 0) {
    printf("# Out of bounds values : %ld %s\n", total_errors, total_errors ? "FAILED" : "OK");
    printf("# Avg bus bandwidth    : %g\n", busbw_n ? busbw_sum / busbw_n : 0.0);
    printf("# launches=%llu staged_calls=%llu errors=%ld\n", (unsigned long long)s.kernel_launches, (unsigned long long)s.staged_calls, total_errors);
    fflush(stdout);      // --procs children leave through _exit(): nothing buffered survives it
  }
  if (scales) CC(b200collMemFree(ctx.comm, scales));
  if (q_scales) CC(b200collMemFree(ctx.comm, q_scales));
  CC(b200collMemFree(ctx.comm, recv));
  CC(b200collMemFree(ctx.comm, send));
  RT(cudaStreamDestroy(st));
  return total_errors ? 4 : 0;
}

// nccl-tests compatibility (the reference's pods run `<op>_perf -b .. -e .. -f 2 -g 1 -w 5 --iters 100 -c 0` under mpirun,
// gpudirect-tcpx/nccl-config.yaml:61-62, gpudirect-rdma/nccl-test-a4x-max-jobset.yaml:153): the binary answers to those
// names through symlinks, takes the same flags, and when a launcher exported a rank (OpenMPI, PMI, torchrun) it is ONE rank
// of the job instead of forking its own.
static const struct { const char* name; const char* op; } kOps[] = {{"all_reduce_perf", "all_reduce"}, {"all_gather_perf", "all_gather"}, {"reduce_scatter_perf", "reduce_scatter"},
                                                                    {"alltoall_perf", "alltoall"}, {"broadcast_perf", "broadcast"}, {"reduce_perf", "reduce"}, {"sendrecv_perf", "sendrecv"}, {"gather_perf", "gather"}, {"scatter_perf", "scatter"}, {"hypercube_perf", "hypercube"}};
static const char* op_from_argv0(const char* argv0) {
  const char* base = strrchr(argv0, '/'); base = base ? base + 1 : argv0;
  for (auto& k : kOps) if (!strcmp(base, k.name)) return k.op;
  return nullptr;
}
struct LauncherRank { int rank = -1, size = 0, local_rank = 0; std::string job; };
static LauncherRank launcher_rank() {
  LauncherRank l;
  static const char* kRank[] = {"OMPI_COMM_WORLD_RANK", "PMI_RANK", "PMIX_RANK", "RANK"};
  static const char* kSize[] = {"OMPI_COMM_WORLD_SIZE", "PMI_SIZE", "", "WORLD_SIZE"};
  static const char* kLocal[] = {"OMPI_COMM_WORLD_LOCAL_RANK", "MPI_LOCALRANKID", "", "LOCAL_RANK"};
  for (int i = 0; i < 4; i++) {
    const char* r = getenv(kRank[i]); const char* s = *kSize[i] ? getenv(kSize[i]) : nullptr;
    if (!r || !s) continue;
    l.rank = atoi(r); l.size = atoi(s);
    const char* lr = *kLocal[i] ? getenv(kLocal[i]) : nullptr;
    l.local_rank = lr ? atoi(lr) : l.rank;
    break;
  }
  // every rank must derive the same id: an explicit job id, else the launcher's, else the rendezvous address
  for (const char* k : {"B200COLL_JOB_ID", "OMPI_MCA_ess_base_jobid", "PMIX_NAMESPACE", "PMI_JOBID", "TORCHELASTIC_RUN_ID"}) if (const char* v = getenv(k)) { l.job = std::string(k) + "=" + v; break; }
  if (l.job.empty()) { const char* a = getenv("MASTER_ADDR"); const char* p = getenv("MASTER_PORT"); l.job = std::string(a ? a : "local") + ":" + (p ? p : "0"); }
  return l;
}

// Every conflict between flags and with the number of ranks (o.nranks), refused before any communicator or buffer exists.
static bool flags_ok(const Opts& o) {
  const int n = o.nranks;
  if (o.uly_back && !o.uly_d) { fprintf(stderr, "--ulysses-back takes --ulysses HQ:HKV:D\n"); return false; }
  if (o.accumulate && !o.fs_h) { fprintf(stderr, "--accumulate takes --fsdp H:F[:KV]\n"); return false; }
  if (o.fs_h) {
    const bool gather = o.op == "all_gather";
    if ((!gather && o.op != "reduce_scatter") || o.q_block || o.bs_rows || o.combine_k || o.route_e || o.cq_block || o.rms_row || o.uly_d || o.cp_c) {
      fprintf(stderr, "--fsdp H:F[:KV] takes --op all_gather or reduce_scatter, and no --quantize, --block-scale, --combine, --route, --rms-norm,\n"
                      "--ulysses or --context\n");
      return false;
    }
    if (gather && (o.accumulate || o.scale != 1.0f)) { fprintf(stderr, "--fsdp: --accumulate and --scale take --op reduce_scatter\n"); return false; }
    const b200collDataType_t a = o.in_dt, b = o.out_dt;
    const bool ok = gather ? ((a == b) || (a == b200collFloat32 && (b == b200collBfloat16 || b == b200collFloat16)))
                           : ((a == b && wide(a)) || (b == b200collFloat32 && (a == b200collBfloat16 || a == b200collFloat16)));
    if (!ok) {
      fprintf(stderr, "--fsdp: dtype pair (-d -> --out-dtype) must be, for all_gather, one dtype or float -> bfloat16|half; for reduce_scatter,\n"
                      "bfloat16|half|float -> the same or bfloat16|half -> float\n");
      return false;
    }
    return true;
  }
  if (o.cp_c) {
    if ((o.op != "all_gather" && o.op != "reduce_scatter") || o.out_dt != o.in_dt || o.scale != 1.0f || o.q_block || o.bs_rows || o.combine_k ||
        o.route_e || o.cq_block || o.rms_row || o.uly_d) {
      fprintf(stderr, "--context W:C takes --op all_gather or reduce_scatter, and no --out-dtype, --scale, --quantize, --block-scale, --combine, --route,\n"
                      "--rms-norm or --ulysses\n");
      return false;
    }
    if (o.op == "reduce_scatter" && !wide(o.in_dt)) { fprintf(stderr, "--context W:C with --op reduce_scatter takes -d bfloat16|half|float\n"); return false; }
    const size_t es = b200collTypeSize(o.in_dt);
    if ((cp_width(o) * es) % 16 || (cp_row(o) * es) % 16) { fprintf(stderr, "--context W:C: W * sizeof(dtype) (HKV * D * sizeof(dtype)) must be a multiple of 16 bytes\n"); return false; }
    return true;
  }
  if (o.uly_d) {
    if (o.op != "alltoall" || o.out_dt != o.in_dt || o.scale != 1.0f || o.q_block || o.bs_rows || o.combine_k || o.route_e || o.cq_block || o.rms_row) {
      fprintf(stderr, "--ulysses HQ:HKV:D takes --op alltoall, and no --out-dtype, --scale, --quantize, --block-scale, --combine, --route or --rms-norm\n");
      return false;
    }
    if (((size_t)o.uly_d * b200collTypeSize(o.in_dt)) % 16) { fprintf(stderr, "--ulysses HQ:HKV:D: D * sizeof(dtype) must be a multiple of 16 bytes\n"); return false; }
    for (int h : {o.uly_hq, o.uly_hkv})
      if (h % n && n % h) { fprintf(stderr, "--ulysses HQ:HKV:D: HQ and HKV must each be a multiple or a divisor of the %d ranks\n", n); return false; }
    if (o.uly_back && o.uly_hq % n) { fprintf(stderr, "--ulysses-back: HQ must be a multiple of the %d ranks\n", n); return false; }
    return true;
  }
  if (o.rms_row && ((o.op != "all_reduce" && o.op != "reduce_scatter") || o.out_dt != o.in_dt || o.scale != 1.0f || o.q_block || o.bs_rows || o.combine_k || o.route_e || o.cq_block ||
                    !wide(o.in_dt))) {
    fprintf(stderr, "--rms-norm ROW_LEN takes --op all_reduce or reduce_scatter and -d bfloat16|half|float, and no --out-dtype, --scale, --quantize,\n"
                    "--block-scale, --combine or --route\n");
    return false;
  }
  if (o.rms_gather && (!o.rms_row || o.op != "reduce_scatter")) {
    fprintf(stderr, "--rms-norm-gather takes --rms-norm ROW_LEN and --op reduce_scatter\n");
    return false;
  }
  if (o.rq_block && (!o.rms_row || o.rms_row % o.rq_block != 0)) {
    fprintf(stderr, "--rms-norm-quantize WIRE:BLOCK takes --rms-norm ROW_LEN, with ROW_LEN a multiple of BLOCK\n");
    return false;
  }
  if (o.cq_block && ((!o.combine_k && !o.route_e) || o.q_block || o.bs_rows || o.row_len % o.cq_block != 0)) {
    fprintf(stderr, "--combine-quantize WIRE:BLOCK takes --combine K or --route E:K, a --row-len that is a multiple of BLOCK, and no --quantize or\n"
                    "--block-scale\n");
    return false;
  }
  if (o.bs_rows && (o.row_len == 0 || o.row_len % 16)) { fprintf(stderr, "--row-len must be a positive multiple of 16\n"); return false; }
  if (o.op == "hypercube" && (n & (n - 1))) { fprintf(stderr, "hypercube needs a power-of-two number of ranks\n"); return false; }
  if ((o.op == "sendrecv" || o.op == "gather" || o.op == "hypercube" || o.op == "scatter") && (o.in_dt != o.out_dt || o.scale != 1.0f)) {
    fprintf(stderr, "%s moves opaque bytes: --in and --out must match and --scale must be 1\n", o.op.c_str());
    return false;
  }
  if (std::none_of(std::begin(kOps), std::end(kOps), [&](const auto& k) { return o.op == k.op; })) { fprintf(stderr, "unknown --op %s\n", o.op.c_str()); return false; }
  if (o.combine_k && (o.op != "alltoall" || o.q_block || o.bs_rows || o.row_len == 0 || o.row_len % 16 || !wide(o.in_dt) || !wide(o.out_dt))) {
    fprintf(stderr, "--combine K takes --op alltoall, -d and --out-dtype bfloat16|half|float, a --row-len that is a multiple of 16, and no --quantize or --block-scale\n");
    return false;
  }
  if (o.combine_k) return true;           // --combine runs the combine mode, whatever --route says
  // with --quantize there is no combine, so no out type: the quantising alltoall defaults --out-dtype to the wire type
  if (o.route_e && (o.op != "alltoall" || o.bs_rows || o.row_len == 0 || o.row_len % 16 || !wide(o.in_dt) || (!o.q_block && !wide(o.out_dt)) ||
                    o.route_e % n != 0 || (o.q_block && o.row_len % o.q_block != 0))) {
    fprintf(stderr, "--route E:K takes --op alltoall, -d and --out-dtype bfloat16|half|float, a --row-len that is a multiple of 16, E a multiple of the\n"
                    "number of ranks, and no --block-scale or --combine; with --quantize WIRE:BLOCK (the FP8 dispatch) a --row-len that is a\n"
                    "multiple of BLOCK\n");
    return false;
  }
  if (o.route_e) return true;             // --quantize with --route is the FP8 dispatch, checked above
  const bool is_a2a = o.op == "alltoall";
  if (o.q_block && ((o.op != "all_gather" && o.op != "reduce_scatter" && o.op != "all_reduce" && !is_a2a) || o.bs_rows || !wide(o.in_dt) ||
                    (is_a2a ? o.out_dt != o.q_wire || o.row_len % o.q_block != 0 : !wide(o.out_dt)))) {
    fprintf(stderr, "--quantize takes --op all_gather, reduce_scatter or all_reduce with -d and --out-dtype bfloat16|half|float, or --op alltoall with\n"
                    "-d bfloat16|half|float, --out-dtype WIRE (or none) and a --row-len that is a multiple of BLOCK; and no --block-scale\n");
    return false;
  }
  if (o.bs_rows && o.op != "all_gather" && o.op != "reduce_scatter" && o.op != "all_reduce") {
    fprintf(stderr, "--block-scale takes --op all_gather, reduce_scatter or all_reduce\n");
    return false;
  }
  return true;
}

// The arena every rank needs: the send and receive windows (or the largest buffers), 64 MiB of slack, and what each mode adds.
static size_t arena_bytes(const Opts& o) {
  const size_t is = b200collTypeSize(o.in_dt), os = b200collTypeSize(o.out_dt);
  return std::max(o.window, o.max_bytes) + std::max(o.window / is * os, o.max_bytes / is * os) + (64u << 20) + (o.bs_rows ? bs_max_scales(o) * 4 : 0) +
         q_scratch_bytes(o) + (o.route_e ? o.max_bytes * o.route_k + 4096 : 0) + route_scale_bytes(o) + cq_scratch_bytes(o) +     // --route: recv holds K rows per token
         (o.rms_row ? o.max_bytes + 4096 : 0) + rms_scale_bytes(o) +                                  // --rms-norm: the residual (and the scales of q)
         (o.uly_d ? uly_out_bytes(o, o.nranks, o.max_bytes + 4096) : 0) +                            // --ulysses: the head shards
         (o.cp_c ? cp_shard_bytes(o) + cp_full_bytes(o, o.nranks) : 0) +                              // --context: the shards and full tensors
         (o.fs_h ? fs_arena_bytes(o) : 0);                                                          // --fsdp: the block's fulls and shards
}

int main(int argc, char** argv) {
  Opts o;
  int gpus_per_proc = 0;
  bool out_given = false;
  if (const char* op = op_from_argv0(argv[0])) o.op = op;
  for (int i = 1; i < argc; i++) {
    std::string a = argv[i];
    auto next = [&]() -> const char* { if (i + 1 >= argc) { fprintf(stderr, "missing value for %s\n", a.c_str()); exit(1); } return argv[++i]; };
    if (a == "--op") o.op = next();
    else if (a == "--ranks") o.nranks = atoi(next());
    else if (a == "--devs") { std::string s = next(); size_t p = 0; while (p < s.size()) { o.devs.push_back(atoi(s.c_str() + p)); p = s.find(',', p); if (p == std::string::npos) break; p++; } }
    else if (a == "--procs") o.procs = true;
    else if (a == "-b" || a == "--min") o.min_bytes = parse_size(next());
    else if (a == "-e" || a == "--max") o.max_bytes = parse_size(next());
    else if (a == "-f" || a == "--factor") o.factor = atoi(next());
    else if (a == "--dtype" || a == "-d" || a == "--datatype") { o.in_dt = o.out_dt = parse_dt(next()); out_given = false; }
    else if (a == "-g" || a == "--ngpus") gpus_per_proc = atoi(next());
    else if (a == "-o" || a == "--redop") { std::string v = next(); if (v != "sum") { fprintf(stderr, "only -o sum is benchmarked (avg is a fused scale: use --scale)\n"); return 1; } }
    else if (a == "-t" || a == "--nthreads" || a == "-m" || a == "--agg_iters" || a == "-p" || a == "--parallel_init" || a == "-z" || a == "--blocking" || a == "-a" || a == "--average" ||
             a == "-G" || a == "--cudagraph" || a == "-C" || a == "--report_cputime" || a == "-R" || a == "--local_register" || a == "-T" || a == "--timeout" || a == "-r" || a == "--root") (void)next();   // accepted, no effect here
    else if (a == "--out-dtype") { o.out_dt = parse_dt(next()); out_given = true; }
    else if (a == "--block-scale") { if (sscanf(next(), "%dx%d", &o.bs_rows, &o.bs_cols) != 2 || o.bs_rows < 1 || o.bs_cols < 16 || o.bs_cols % 16) { fprintf(stderr, "--block-scale RxC: R >= 1, C a multiple of 16\n"); return 1; } }
    else if (a == "--row-len") o.row_len = (size_t)atoll(next());
    else if (a == "--quantize") parse_wire_block(a, next(), &o.q_wire, &o.q_block);
    else if (a == "--combine-quantize") parse_wire_block(a, next(), &o.cq_wire, &o.cq_block);
    else if (a == "--rms-norm-quantize") parse_wire_block(a, next(), &o.rq_wire, &o.rq_block);
    else if (a == "--rms-norm-gather") o.rms_gather = true;
    else if (a == "--rms-norm") {
      const long long v = atoll(next());
      if (v < 16 || v > 16384 || v % 16) { fprintf(stderr, "--rms-norm ROW_LEN: a multiple of 16 in [16, 16384]\n"); return 1; }
      o.rms_row = (size_t)v;
    }
    else if (a == "--ulysses") {
      if (sscanf(next(), "%d:%d:%d", &o.uly_hq, &o.uly_hkv, &o.uly_d) != 3 || o.uly_hq < 1 || o.uly_hkv < 1 || o.uly_d < 1) {
        fprintf(stderr, "--ulysses HQ:HKV:D: three positive integers\n"); return 1;
      }
    }
    else if (a == "--ulysses-back") o.uly_back = true;
    else if (a == "--fsdp") {
      const char* v = next();
      int h = 0, f = 0, kv = 0, used = 0;
      const int got = sscanf(v, "%d:%d%n:%d%n", &h, &f, &used, &kv, &used);
      if (!((got == 2 || got == 3) && !v[used] && h > 0 && f > 0 && (got == 2 || kv > 0) && h % 16 == 0 && f % 16 == 0 && kv % 16 == 0)) {
        fprintf(stderr, "--fsdp H:F[:KV]: positive integers, each a multiple of 16\n"); return 1;
      }
      o.fs_h = h; o.fs_f = f; o.fs_kv = got == 3 ? kv : 0;
    }
    else if (a == "--accumulate") o.accumulate = true;
    else if (a == "--context") {
      const char* v = next();
      long long w = 0;
      int c = 0, hq = 0, hkv = 0, d = 0, used = 0;
      if (sscanf(v, "%d:%d:%d:%d%n", &hq, &hkv, &d, &c, &used) == 4 && !v[used] && hq > 0 && hkv > 0 && d > 0 && (c == 1 || c == 2)) {
        o.cp_hq = hq; o.cp_hkv = hkv; o.cp_d = d; o.cp_c = c;
      } else if (sscanf(v, "%lld:%d%n", &w, &c, &used) == 2 && !v[used] && w > 0 && (c == 1 || c == 2)) {
        o.cp_w = (size_t)w; o.cp_c = c;
      } else {
        fprintf(stderr, "--context W:C or HQ:HKV:D:C: positive integers, C 1 or 2\n"); return 1;
      }
    }
    else if (a == "--combine") { o.combine_k = atoi(next()); if (o.combine_k < 1) { fprintf(stderr, "--combine K: K >= 1\n"); return 1; } }
    else if (a == "--route") {
      if (sscanf(next(), "%d:%d", &o.route_e, &o.route_k) != 2 || o.route_e < 1 || o.route_e > 1024 || o.route_k < 1) { fprintf(stderr, "--route E:K: 1 <= E <= 1024, K >= 1\n"); return 1; }
    }
    else if (a == "--scale") o.scale = (float)atof(next());
    else if (a == "--algo") o.algo = next();
    else if (a == "--iters" || a == "-n") o.iters = atoi(next());
    else if (a == "--warmup" || a == "-w") o.warmup = atoi(next());
    else if (a == "--check" || a == "-c") o.check = atoi(next());
    else if (a == "--inplace") o.inplace = atoi(next());
    else if (a == "--max-ctas") o.max_ctas = atoi(next());
    else if (a == "--window") o.window = parse_size(next());
    else if (a == "--json") o.json = next();
    else if (a == "--skew-us") o.skew_us = atoi(next());
    else if (a == "--sweep") {
      std::string v = next(); size_t p = 0;
      while (p < v.size()) {
        Opts::Shape sh{0, 0, 0};
        if (sscanf(v.c_str() + p, "%d:%d:%d", &sh.kind, &sh.ctas, &sh.threads) == 3) o.shapes.push_back(sh);
        p = v.find(',', p); if (p == std::string::npos) break; p++;
      }
    }
    else if (a == "--selfcheck") { char buf[4096]; b200collResult_t r = b200collSelfCheck(buf, sizeof(buf)); fputs(buf, stdout); return r == b200collSuccess ? 0 : 1; }
    else if (a == "-h" || a == "--help") {
      puts("b200coll_perf (also all_reduce_perf, all_gather_perf, reduce_scatter_perf, alltoall_perf, broadcast_perf, reduce_perf, sendrecv_perf, gather_perf, scatter_perf, hypercube_perf): nccl-tests style sweep on libb200coll\n"
           "  --op NAME                 collective (implied by the name the binary is called by)\n"
           "  -b/-e SIZE -f N           sweep from -b to -e bytes multiplying by -f (1K, 64M, 1G ...)\n"
           "  -g N | --ranks N | --devs a,b,..   ranks in this process (threads); --procs forks one process per rank instead\n"
           "  under mpirun / torchrun (OMPI_COMM_WORLD_*, PMI_*, RANK/WORLD_SIZE/LOCAL_RANK) each process is one rank; B200COLL_JOB_ID names the job\n"
           "  -w N -n/--iters N -c 0|1  warm-up, timed iterations, check results against the host reference\n"
           "  -d float|half|bfloat16|e4m3|e5m2 (fp8 = e4m3)   input type; --out-dtype T and --scale X fuse a cast / scale into the collective\n"
           "  --block-scale RxC         block-scaled FP8 (all_gather, reduce_scatter, all_reduce): -d e4m3|e5m2 [R x C]-blocked matrices, one seeded\n"
           "                            fp32 scale per block, --out-dtype bfloat16|half|float; -c 1 checks bit for bit against the host\n"
           "  --row-len N               columns of the block-scaled matrix, or row length of the quantising alltoall (default 2048; N and C\n"
           "                            multiples of 16, N a multiple of BLOCK)\n"
           "  --quantize WIRE:BLOCK     quantising collectives (all_gather, reduce_scatter, all_reduce, alltoall): -d bfloat16|half|float in, each rank\n"
           "                            quantises to WIRE (e4m3|e5m2) with one fp32 scale per BLOCK (16..512) elements, --out-dtype bfloat16|half|float;\n"
           "                            seeded inputs whose blocks differ in amax; -c 1 checks bit for bit against the host\n"
           "                            --op alltoall: the quantising all-to-all-v, -d bfloat16|half|float in, --out-dtype WIRE (the default); each rank\n"
           "                            sends an even split of whole --row-len rows to every peer and receives FP8 rows plus one fp32 scale per\n"
           "                            BLOCK; -c 1 checks every FP8 byte and scale bit for bit against the host quantiser\n"
           "  --combine K               --op alltoall: the expert combine (all-to-all-v back, top-K weighted sum fused), -d bfloat16|half|float the\n"
           "                            expert_out type, --out-dtype bfloat16|half|float the out type, --row-len a multiple of 16; every rank returns\n"
           "                            an even split of whole rows, each token takes K slots from K different ranges where there are enough (seeded\n"
           "                            routing and weights); size = expert_out bytes read per rank; -c 1 checks every output element bit for bit\n"
           "                            against the slot-order host reference\n"
           "  --route E:K               --op alltoall: the device-routed expert dispatch and its combine, E experts (a multiple of the ranks, at most\n"
           "                            1024) sharded over the ranks, seeded top-K expert ids per token on the device, -d bfloat16|half|float rows,\n"
           "                            --out-dtype the combine's out type, recv sized to the mean load (tokens * K rows); size = x bytes per rank;\n"
           "                            reports the dispatch (layout, count exchange and push) and the combine; -c 1 checks every received byte,\n"
           "                            count, route and dropped, and the combine bit for bit, against the host layout\n"
           "  --route E:K --quantize WIRE:BLOCK   the device-routed FP8 expert dispatch: the same layout, each token's row quantised once to\n"
           "                            WIRE with one fp32 scale per BLOCK elements (--row-len a multiple of BLOCK); reports the dispatch only (the\n"
           "                            combine needs a wide expert_out); -c 1 checks every FP8 byte, scale, count, route and dropped against the\n"
           "                            host layout and the host quantiser\n"
           "  --combine-quantize WIRE:BLOCK   with --combine K or --route E:K (no --quantize): the quantising combine in place of the wide one;\n"
           "                            each rank quantises its whole expert_out to WIRE (e4m3|e5m2) with one fp32 scale per BLOCK elements\n"
           "                            (--row-len a multiple of BLOCK) and the slots pull FP8 rows and scales; -c 1 checks every output element bit\n"
           "                            for bit against the host quantiser and the slot-order reference\n"
           "  --algo auto|ll|ll2|oneshot|twoshot|nvls   --inplace 0|1|2   --max-ctas N   --sweep kind:ctas:threads,...   --json FILE   --window SIZE\n"
           "  --rms-norm ROW_LEN        --op all_reduce, -d bfloat16|half|float: the fused all-reduce, residual add and RMSNorm over rows of ROW_LEN\n"
           "                            elements (a multiple of 16 in [16, 16384]); -c 1 checks every residual and out element bit for bit\n"
           "  --rms-norm-quantize WIRE:BLOCK   with --rms-norm ROW_LEN (a multiple of BLOCK): out quantised in the same kernel to WIRE (e4m3|e5m2)\n"
           "                            rows with one fp32 scale per 1 x BLOCK (16..512) group; rw GB/s counts q and scales written instead of out;\n"
           "                            -c 1 checks every residual element, FP8 byte and scale bit for bit against the host quantiser\n"
           "  --op reduce_scatter --rms-norm ROW_LEN   the sequence-parallel form: the fused reduce-scatter, residual add and RMSNorm; rows\n"
           "                            are rounded down to a multiple of the ranks, each rank keeps a residual shard of rows / nranks rows and\n"
           "                            stores the out rows of its slice; -c 1 checks the shard, every other residual row unchanged, and out\n"
           "  --rms-norm-gather         with --op reduce_scatter --rms-norm ROW_LEN: the normed rows all-gathered in the same kernel\n"
           "  --ulysses HQ:HKV:D        --op alltoall, -d bfloat16|half|float|e4m3|e5m2: the Ulysses all-to-all of sequence-parallel attention, B = 1;\n"
           "                            every rank's packed QKV [S_l, (HQ + 2 HKV) * D] (q, k and v column slices) to dense head shards in one\n"
           "                            call; size = source bytes per rank, rounded down to whole tokens; -c 1 checks every output byte\n"
           "  --ulysses-back            with --ulysses HQ:HKV:D: heads -> sequence, the [S, HQ / N, D] attention output back to [S_l, HQ, D]\n"
           "  --context W:C | HQ:HKV:D:C   --op all_gather or reduce_scatter (bfloat16|half|float; the gather also e4m3|e5m2): context parallelism,\n"
           "                            B = 1, C = 1 contiguous or 2 load-balanced (causal) sharding. all_gather: K and V, the column slices of a\n"
           "                            packed QKV [S_l, (HQ + 2 HKV) * D] (or one dense [S_l, W]), gathered into dense [S, HKV * D] in token\n"
           "                            order in one call; reduce_scatter: the gradient, [S, HKV * D] summed over the ranks into the K and V\n"
           "                            slices of a packed dQKV; size = shard bytes per rank, rounded down to whole tokens; -c 1 checks every\n"
           "                            output byte (the reduce-scatter against the fp32 sum in rank order)\n"
           "  --fsdp H:F[:KV]           --op all_gather or reduce_scatter: FSDP's dim-0 shards of one Llama block (q, k, v, o, gate, up, down and two\n"
           "                            norm weights; hidden H, MLP F, K/V width KV, default H), one call for the nine tensors, p = ceil(d / N)\n"
           "                            rows per rank. all_gather: -d shards -> --out-dtype fulls (float -> bfloat16|half casts, else one dtype);\n"
           "                            reduce_scatter: -d gradients -> --out-dtype shards (bfloat16|half -> float widens), times --scale X,\n"
           "                            --accumulate adds into the old shard; -c 1 checks every output element against the header's formulas\n"
           "  --accumulate              with --fsdp and --op reduce_scatter: shard = round_once(old + sum * scale)\n"
           "  --selfcheck              report whether this node can run the NVLink fast paths (exit 1 if not)");
      return 0;
    }
    else { fprintf(stderr, "unknown flag %s\n", a.c_str()); return 1; }
  }
  if (o.factor < 2) o.factor = 2;
  if (o.q_block && o.op == "alltoall" && !out_given) o.out_dt = o.q_wire;     // the quantising alltoall receives the wire type
  const LauncherRank lr = launcher_rank();
  const bool launched = lr.size > 1 && o.devs.empty() && !o.procs;         // one rank of an mpirun / torchrun job (nccl-tests' -g 1 layout)
  if (launched) {
    if (gpus_per_proc > 1) { fprintf(stderr, "-g %d under a launcher is not supported: run one rank per GPU (-g 1)\n", gpus_per_proc); return 1; }
    if (lr.size > B200COLL_MAX_RANKS) { fprintf(stderr, "libb200coll is an intra-node transport: %d ranks > %d GPUs of one NVSwitch domain\n", lr.size, B200COLL_MAX_RANKS); return 1; }
    o.nranks = lr.size; o.procs = true;
  } else {
    if (gpus_per_proc > 0 && o.nranks == 0) o.nranks = gpus_per_proc;     // nccl-tests -g N without a launcher: N ranks in this process
    if (!o.devs.empty()) o.nranks = (int)o.devs.size();
    if (o.nranks == 0) { int nd = 0; cudaGetDeviceCount(&nd); o.nranks = nd > 0 ? nd : 1; }     // no rank count given: one rank per GPU
  }
  if (!flags_ok(o)) return 1;
  b200collConfig cfg; b200collConfigDefault(&cfg);
  if (!getenv("B200COLL_ARENA_MB")) cfg.arena_bytes = arena_bytes(o);
  if (launched) {
    // rendezvous on the job id, timing page in /dev/shm
    int nd = 0; RT(cudaGetDeviceCount(&nd));
    const int dev = nd > 0 ? lr.local_rank % nd : 0;
    unsigned h = 2166136261u; for (char ch : lr.job) h = (h ^ (unsigned char)ch) * 16777619u;
    char shm_name[64]; snprintf(shm_name, sizeof shm_name, "/b200coll_perf.%08x", h);
    int fd = shm_open(shm_name, O_CREAT | O_RDWR, 0600);
    if (fd < 0 || ftruncate(fd, sizeof(Shared)) != 0) { perror("shm_open"); return 1; }
    Shared* sh = (Shared*)mmap(nullptr, sizeof(Shared), PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    close(fd);
    if (sh == MAP_FAILED) { perror("mmap"); return 1; }
    b200collUniqueId id; CC(b200collUniqueIdFromString(("perf/" + lr.job).c_str(), &id));
    RT(cudaSetDevice(dev));
    b200collComm_t comm;
    CC(b200collCommInitRank(&comm, lr.size, &id, lr.rank, &cfg));
    // a crashed earlier job with the same id may have left counters behind: wipe the page between two host barriers,
    // i.e. after everybody mapped it and before anybody counts on it
    CC(b200collHostBarrier(comm));
    if (lr.rank == 0) memset((void*)sh, 0, sizeof(Shared));
    CC(b200collHostBarrier(comm));
    int rc = run_rank(o, RankCtx{lr.rank, lr.size, comm, dev, sh});
    CC(b200collCommDestroy(comm));          // ends with a host barrier: every rank is past its last use of the page
    if (lr.rank == 0) shm_unlink(shm_name);
    return rc;
  }
  if (o.devs.empty()) {                     // the ranks take the visible GPUs in turn
    int nd = 0; cudaGetDeviceCount(&nd);
    for (int i = 0; i < o.nranks; i++) o.devs.push_back(nd > 0 ? i % nd : 0);
  }
  const int n = o.nranks;
  Shared* sh = (Shared*)mmap(nullptr, sizeof(Shared), PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
  memset(sh, 0, sizeof(Shared));
  if (o.procs) {
    b200collUniqueId id; CC(b200collGetUniqueId(&id));
    std::vector<pid_t> kids;
    for (int r = 0; r < n; r++) {
      pid_t p = fork();
      if (p == 0) {
        RT(cudaSetDevice(o.devs[r]));
        b200collComm_t comm;
        CC(b200collCommInitRank(&comm, n, &id, r, &cfg));
        int rc = run_rank(o, RankCtx{r, n, comm, o.devs[r], sh});
        CC(b200collCommDestroy(comm));
        _exit(rc);
      }
      kids.push_back(p);
    }
    int worst = 0;
    for (pid_t p : kids) { int stt = 0; waitpid(p, &stt, 0); int rc = WIFEXITED(stt) ? WEXITSTATUS(stt) : 128; worst = std::max(worst, rc); }
    return worst;
  }
  std::vector<b200collComm_t> comms(n);
  CC(b200collCommInitAll(comms.data(), n, o.devs.data(), &cfg));
  std::vector<std::thread> th;
  std::vector<int> rcs(n, 0);
  for (int r = 0; r < n; r++) th.emplace_back([&, r] { rcs[r] = run_rank(o, RankCtx{r, n, comms[r], o.devs[r], sh}); });
  for (auto& t : th) t.join();
  for (int r = 0; r < n; r++) CC(b200collCommDestroy(comms[r]));
  int worst = 0; for (int rc : rcs) worst = std::max(worst, rc);
  return worst;
}
