// Host-side launch helpers shared by the collective entry points (collectives.cu, generic.cu, blockscaled.cu, combine.cu and
// dispatch.cu): kernel launch through cudaLaunchKernelEx with optional programmatic dependent launch, the launch-shape pickers,
// argument, placement and communicator checks, the type dispatch, and call accounting.
#pragma once
#include <stdlib.h>

#include <algorithm>
#include <initializer_list>
#include <string>
#include <utility>

#include "comm.h"

namespace b200coll {

#define LAUNCH_CHECK(c)                                                                                  \
  do {                                                                                                   \
    cudaError_t e__ = cudaGetLastError();                                                                \
    if (e__ != cudaSuccess) { set_last_error(std::string("kernel launch failed: ") + cudaGetErrorString(e__)); return b200collUnhandledCudaError; } \
    (c)->stats.kernel_launches++;                                                                        \
  } while (0)

struct Grid { int blocks, threads; };

// Every kernel goes through cudaLaunchKernelEx so that back-to-back collectives can use programmatic dependent launch
// (on by default, B200COLL_PDL=0 disables): the next kernel's launch latency overlaps the current kernel's execution; each kernel starts with
// griddepcontrol.launch_dependents + griddepcontrol.wait, so it still observes its predecessor's completed memory.
// Never with virtual ranks (several communicators on one GPU): a pre-launched dependent grid parks its CTAs on SMs
// that another rank's current kernel still needs, and ranks that spin on each other then deadlock (seen at 1 MiB with
// 4 ranks on one GPU). With one rank per GPU every CTA of kernel i is resident before kernel i+1 may start.
// The overlap pays for tiny messages and costs time for larger ones (the early-launched grid sits on the SMs while its predecessor
// still needs them, and its griddepcontrol.wait returns only after the predecessor's memory flush). So only launches whose message is
// at most B200COLL_PDL_MAX_KB (default 8) carry the attribute; the cut-off has not been re-measured on multi-GPU H100 systems. launch_ll sets the flag for the launch it is about to make.
// One exception, at every size: the one-rank copy-engine copy (k_copy_bulk). Its grid never exceeds what is resident at once (2 CTAs of
// 96 KiB per SM), so every one of its CTAs already holds its slot when a dependent grid is released, and a dependent can only take
// slots the copy does not need; what PDL saves there is the launch gap between back-to-back copies.
inline thread_local bool t_pdl = false;
struct PdlScope {           // the launches made while it lives carry the attribute (if pdl_enabled() allows it)
  explicit PdlScope(bool v) { t_pdl = v; }
  ~PdlScope() { t_pdl = false; }
};
inline size_t pdl_max_bytes() {
  static const size_t v = [] { const char* e = getenv("B200COLL_PDL_MAX_KB"); return (size_t)(e && *e ? atol(e) : 8) << 10; }();
  return v;
}
inline bool pdl_enabled() {
  static const bool on = [] { const char* e = getenv("B200COLL_PDL"); return !(e && *e == '0'); }();      // on unless B200COLL_PDL=0
  return on && t_pdl && g_loopback_comms.load(std::memory_order_relaxed) == 0;
}
template <typename... KArgs, typename... Args>
static void launch_k_smem(void (*kernel)(KArgs...), int blocks, int threads, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)blocks); cfg.blockDim = dim3((unsigned)threads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr;
  if (pdl_enabled()) {
    attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr.val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = &attr; cfg.numAttrs = 1;
  }
  (void)cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
template <typename... KArgs, typename... Args>
static void launch_k(void (*kernel)(KArgs...), int blocks, int threads, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)blocks); cfg.blockDim = dim3((unsigned)threads); cfg.dynamicSmemBytes = 0; cfg.stream = st;
  cudaLaunchAttribute attr;
  if (pdl_enabled()) {
    attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr.val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = &attr; cfg.numAttrs = 1;
  }
  (void)cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);   // the error is picked up by LAUNCH_CHECK's cudaGetLastError
}

// Pick the smallest block size that still covers `vecs` with <= max_ctas blocks (small work spreads over more SMs),
// unless the family's shape pins the thread count.
enum { kShapeNvls = 0, kShapeP2p = 1, kShapeLL = 2, kShapeNvlsRs = 3, kShapeRooted = 4 };
inline Grid pick_grid(const b200collComm* c, int kind, size_t vecs, int unroll) {
  static const int forced = [] { const char* e = getenv("B200COLL_FORCE_THREADS"); return e ? atoi(e) : 0; }();
  const int max_ctas = std::max(1, std::min(c->shape[kind].max_ctas > 0 ? c->shape[kind].max_ctas : c->max_ctas, c->max_ctas));
  int pinned = c->shape[kind].threads;
  if (forced >= 32 && forced <= 512) pinned = forced;
  if (pinned) {
    size_t b = (vecs + (size_t)pinned * unroll - 1) / ((size_t)pinned * unroll);
    return Grid{(int)std::max<size_t>(1, std::min<size_t>(b, (size_t)max_ctas)), pinned};
  }
  for (int t : {128, 256, 512}) {
    size_t b = (vecs + (size_t)t * unroll - 1) / ((size_t)t * unroll);
    if (b <= (size_t)max_ctas || t == 512) return Grid{(int)std::max<size_t>(1, std::min<size_t>(b, (size_t)max_ctas)), t};
  }
  return Grid{1, 128};
}

// Whole warps: WarpScale and the amax butterfly are full-mask warp intrinsics, and pick_grid takes a forced thread count as given.
inline Grid warp_grid(const b200collComm* c, size_t vecs) {
  Grid gr = pick_grid(c, kShapeP2p, vecs, 1);
  gr.threads = std::max(32, gr.threads & ~31);
  return gr;
}

// The grid of every all-to-all kernel with a closing barrier: the full P2P shape of the communicator, whatever this rank's work. The
// epoch barrier pairs CTA b of this rank with CTA b of every peer and nothing else, and each rank knows only its own rows or tokens, so
// a grid sized to them would differ from rank to rank, and a CTA missing on one rank would leave CTA b of its peers waiting. CTAs
// without work take only the barriers. `warps`: whole warps, for the kernels that walk with warp_walk.
inline Grid full_grid(const b200collComm* c, int unroll, bool warps = false) {
  return warps ? warp_grid(c, ~(size_t)0 >> 8) : pick_grid(c, kShapeP2p, ~(size_t)0 >> 8, unroll);
}

// nranks == 1: no peers, no barrier; grid as for the fused copy (streaming, 8 CTAs of 256 threads per SM at most)
inline int copy_blocks(const b200collComm* c, uint32_t nvec) {
  return (int)std::max<size_t>(1, std::min<size_t>(((size_t)nvec + 255) / 256, (size_t)std::max(1, c->sm_count) * 8));
}

// The quantising block: a power of two from 16 to 512 elements, so 1 to 32 16-element vectors. Returns log2(vectors per block), or
// -1 (and the caller refuses with kBlockRule) for any other block.
constexpr const char* kBlockRule = "block must be 16, 32, 64, 128, 256 or 512";
inline int quant_lvpb(int block) {
  if (block < 16 || block > 512 || (block & (block - 1)) != 0) return -1;
  int l = 0;
  while ((16 << l) < block) l++;
  return l;
}

// Makes the communicator's GPU current while it lives and restores the caller's: a process may drive communicators on several GPUs,
// and a launch onto a stream of another device than the current one fails (after the peers' kernels are already waiting for it).
struct DeviceScope {
  int prev = -1;
  bool switched = false;
  explicit DeviceScope(int want) { if (cudaGetDevice(&prev) == cudaSuccess && prev != want) switched = cudaSetDevice(want) == cudaSuccess; }
  ~DeviceScope() { if (switched) cudaSetDevice(prev); }
};

inline size_t arena_off(b200collComm* c, const void* p) { return reinterpret_cast<CUdeviceptr>(p) - c->peer_va[c->rank]; }
inline bool aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) % a) == 0; }
inline bool overlaps(const void* a, size_t na, const void* b, size_t nb) {
  const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
  return x < y + nb && y < x + na;
}

// A kernel that hit its watchdog deadline poisons the communicator: every later call is refused (the caller returns RemoteError).
inline bool comm_poisoned(const b200collComm* c) {
  if (!c->fault_host || *const_cast<volatile uint32_t*>(&c->fault_host->code) == 0) return false;
  set_last_error("communicator is poisoned by an earlier watchdog fault");
  return true;
}

// Peers read or write these buffers at MY arena offsets, so each must be arena memory: InvalidUsage (with `who`, the entry point's
// message prefix) when one is not. A zero-length buffer is checked as one byte.
inline b200collResult_t in_arena(b200collComm* c, const std::string& who, const char* names, std::initializer_list<std::pair<const void*, size_t>> bufs) {
  for (const auto& b : bufs) {
    if (b200collIsSymmetric(c, b.first, std::max<size_t>(b.second, 1))) continue;
    set_last_error(who + names + " must lie in the symmetric arena (b200collMemAlloc), at the same offset" + (bufs.size() > 1 ? "s" : "") + " on every rank");
    return b200collInvalidUsage;
  }
  return b200collSuccess;
}

// type dispatch: f(Tag<T>{}) instantiates a launch for an element type; nest one per template parameter. The argument checks have
// refused every other type, so the last case takes what is left.
template <typename T> struct Tag { using type = T; };
inline bool wide_type(b200collDataType_t t) { return t == b200collBfloat16 || t == b200collFloat16 || t == b200collFloat32; }
inline bool is_fp8(b200collDataType_t t) { return t == b200collFloat8e4m3 || t == b200collFloat8e5m2; }
template <typename F> auto with_wide(b200collDataType_t t, F&& f) {      // bf16, fp16, fp32
  switch (t) {
    case b200collBfloat16: return f(Tag<__nv_bfloat16>{});
    case b200collFloat16: return f(Tag<__half>{});
    default: return f(Tag<float>{});
  }
}
template <typename F> auto with_fp8(b200collDataType_t t, F&& f) {       // e4m3, e5m2
  return t == b200collFloat8e4m3 ? f(Tag<__nv_fp8_e4m3>{}) : f(Tag<__nv_fp8_e5m2>{});
}

// collectives.cu: count a call in the stats (and mark it for NVTX / debug traces); B200COLL_CHECK=1 cross-check of a symmetric launch
void account(b200collComm* c, b200collOp_t op, size_t bytes, b200collAlgo_t algo);
b200collResult_t cross_check(b200collComm* c, b200collOp_t op, b200collAlgo_t algo, size_t count, size_t off_a, size_t off_b);

}  // namespace b200coll
