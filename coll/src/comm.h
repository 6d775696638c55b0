// Host-side communicator state for libb200coll.
#pragma once
#include <cuda.h>
#include <sched.h>
#include <cuda_runtime.h>

#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../include/b200coll.h"
#include "bootstrap.h"
#include "device.cuh"

namespace b200coll {

// Driver entry points resolved at run time (cudaGetDriverEntryPoint) so the library loads — and its
// CPU-side logic is testable — on a box without libcuda.
#define B200COLL_DRV_FUNCS(X)                                                                                          \
  X(cuMemCreate) X(cuMemRelease) X(cuMemMap) X(cuMemUnmap) X(cuMemAddressReserve) X(cuMemAddressFree)                   \
  X(cuMemSetAccess) X(cuMemExportToShareableHandle) X(cuMemImportFromShareableHandle)                                  \
  X(cuMemGetAllocationGranularity) X(cuMulticastCreate) X(cuMulticastAddDevice) X(cuMulticastBindMem)                  \
  X(cuMulticastUnbind) X(cuMulticastGetGranularity) X(cuDeviceGet) X(cuDeviceGetAttribute) X(cuGetErrorString)         \
  X(cuDriverGetVersion) X(cuDeviceGetUuid)

struct Drv {
#define X(n) decltype(&::n) n = nullptr;
  B200COLL_DRV_FUNCS(X)
#undef X
  bool ok = false;
  std::string why;
};
const Drv& drv();

void set_last_error(const std::string& s);
void dbg(int level, const char* fmt, ...);
int debug_level();

struct FreeBlock { size_t off, len; };

struct Arena {
  CUmemGenericAllocationHandle handle = 0;
  size_t total = 0;               // bytes, granularity-rounded (control + heap)
  int device = -1;
};

// Host path (hostpath.cu): copy streams, events and the two staging pairs of b200collAllReduceHost.
struct HostPath {
  cudaStream_t h2d = nullptr, d2h = nullptr;
  cudaEvent_t ev_start = nullptr, ev_in_ready[2] = {}, ev_in_free[2] = {}, ev_out_free[2] = {};
  void* in[2] = {};
  void* out[2] = {};
  size_t chunk_bytes = 0;
};

extern std::atomic<int> g_loopback_comms;   // live communicators whose ranks share a GPU (virtual ranks): PDL stays off

struct SharedGroup;   // in-process groups (InitAll) share ownership bookkeeping

}  // namespace b200coll

struct b200collComm {
  int rank = 0, nranks = 1, device = 0;
  b200collConfig cfg{};
  b200coll::Arena arena;
  CUdeviceptr peer_va[B200COLL_MAX_RANKS] = {};
  CUmemGenericAllocationHandle peer_handle[B200COLL_MAX_RANKS] = {};   // imported (multi-process) or borrowed (in-process)
  bool peer_handle_owned[B200COLL_MAX_RANKS] = {};
  CUdeviceptr mc_va = 0;
  CUmemGenericAllocationHandle mc_handle = 0;
  bool mc_owned = false, mc_bound = false;
  bool nvls = false, loopback = false, loopback_counted = false;
  int sm_count = 0, driver_version = 0;
  uint32_t* state_dev = nullptr;
  b200collFault* fault_host = nullptr;
  b200collFault* fault_dev = nullptr;
  b200coll::CommDev dev{};
  std::unique_ptr<b200coll::Bootstrap> boot;
  // symmetric heap allocator (offsets relative to arena base)
  std::vector<b200coll::FreeBlock> free_list;
  std::map<size_t, size_t> live;   // off -> len
  std::mutex mu;
  b200collAlgo_t forced_algo = b200collAlgoAuto;
  int max_ctas = 0;
  // NVLS all-reduce/all-gather, P2P, LL, NVLS reduce-scatter, rooted NVLS ops. The multimem all-reduce wants few CTAs (32 x 256
  // threads); the ld_reduce-only reduce-scatter kernel (2 loads in flight per thread) needs 64 x 512. LL and the rooted NVLS ops run
  // one CTA per SM (max_ctas 0 here: finalize_comm sets it from the device's SM count); in a rooted op only the root moves data, so ONE
  // rank must keep the link busy: an SM's worth of CTAs x 512 threads x 2-4 vectors in flight.
  struct Shape { int max_ctas; int threads; } shape[5] = {{32, 256}, {0, 0}, {0, 0}, {64, 512}, {0, 512}};
  b200collStats stats{};
  std::shared_ptr<b200coll::SharedGroup> group;
  void* stats_shm = nullptr;       // exported stats page (metrics exporter reads it)
  std::string stats_shm_name;
  std::string boot_name;                // rendezvous name this communicator was created under (multi-process only); splits derive theirs from it
  uint32_t split_seq = 0;               // CommSplit calls so far (a collective call, so the same on every rank)
  size_t p2p_window = 0;                // staged receives: bytes per staging window; 0 = an equal share of the staging area
  uint32_t stats_tick = 0;              // collective calls since init; the counters page is refreshed every 256
  unsigned long long bulk_grid_hint = 0; // chunks the largest rank of a rooted / personalised bulk launch has (set by the caller, consumed by launch_bulk)
  int numa_node = -1;                   // of this rank's GPU (sysfs), -1 unknown
  std::string local_cpulist;            // GPU-local CPUs as sysfs prints them
  cpu_set_t affinity_saved;             // the calling thread's mask before CommInitRank narrowed it
  bool affinity_changed = false;
  b200coll::HostPath host;
  std::map<void*, size_t> host_allocs;  // HostAlloc: base -> mapped length
  // quantising collectives (blockscaled.cu): the symmetric scratch for the FP8 copy and its scales, grown on demand. Superseded scratch
  // buffers stay allocated until CommDestroy (a captured CUDA graph may still address them).
  void* quant_scratch = nullptr;
  size_t quant_scratch_bytes = 0;
  std::vector<void*> quant_scratch_retired;
};

namespace b200coll {

struct LaunchPlan {
  b200collAlgo_t algo;
  int blocks;
  int threads;
};

// tuner.cc
void stats_page_publish(b200collComm* c);   // comm.cu
int tuner_blocks(b200collOp_t op, b200collAlgo_t algo, size_t work_vecs, int max_ctas, int unroll);

// generic.cu
bool needs_generic(const b200collEpilogue* ep, b200collRedOp_t rop);
b200collResult_t generic_reduce(b200collComm* c, b200collOp_t which, const void* send, void* recv, size_t count, const b200collEpilogue* ep, b200collRedOp_t rop, int root, cudaStream_t st);

// hostpath.cu
void bind_to_gpu_numa(b200collComm* c, bool allow_bind);   // allow_bind=false: only record the node (in-process groups spanning GPUs)
void restore_affinity_after_init(b200collComm* c);
void hostpath_destroy(b200collComm* c);

// collectives.cu
b200collResult_t launch_fill_sentinel(b200collComm* c, cudaStream_t s);

// blockscaled.cu: `need` bytes of the quantising scratch that the quantising collectives and the quantising combine share, at arena offset
// *off (the same on every rank); OutOfMemory, the message led by `who`, when the arena cannot hold it
b200collResult_t quant_scratch_take(b200collComm* c, size_t need, const char* who, size_t* off);

// dispatch.cu: one launch of k_a2av_quant_copy<in, wire> (no barrier): nvec 16-element vectors of `in` quantised into q and scales,
// 2^lvpb vectors per block
b200collResult_t launch_quant_copy(b200collComm* c, b200collDataType_t in_dtype, b200collDataType_t wire, const void* in, char* q, char* scales,
                                   uint32_t nvec, uint32_t lvpb, cudaStream_t st);
// dispatch.cu: once per device, load every kernel that can run behind a layout kernel or inside a quantising combine (lazy module loading)
void routed_preload(const b200collComm* c);

// combine.cu: load every combine kernel, wide and quantising (routed_preload calls it)
void combine_preload();

}  // namespace b200coll
