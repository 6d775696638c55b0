// Arena layout, per-communicator device state and the communicator descriptor kernels receive. Plain C++ (no CUDA headers): shared by
// the device code (device.cuh) and by the host-side protocol emulator (coll/tests/p2p_emu.cc).
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "../include/b200coll.h"

namespace b200coll {

// ---- arena layout (identical on every rank; offsets in bytes from the arena base) ----
constexpr int kMaxRanks = B200COLL_MAX_RANKS;
constexpr int kMaxBlocks = 1024;                        // flag rows
constexpr size_t kOffFlags = 0;                         // u32 [kMaxBlocks][kMaxRanks]
constexpr size_t kFlagsBytes = (size_t)kMaxBlocks * kMaxRanks * 4;
constexpr size_t kOffLL = 1 << 20;                      // Lamport scratch: [3][kMaxRanks][kLLMaxVecs] x 16 B
constexpr size_t kLLMaxBytes = 1 << 20;                 // per-source slot: lo half = one-shot / phase 1, hi half = two-shot phase 2
constexpr size_t kLLMaxVecs = kLLMaxBytes / 16;
constexpr size_t kLLHalfVecs = kLLMaxVecs / 2;
constexpr size_t kLLOneShotMaxBytes = kLLHalfVecs * 16; // 512 KiB per source
constexpr size_t kLLBytes = 3 * (size_t)kMaxRanks * kLLMaxBytes;
constexpr size_t kOffStage = kOffLL + kLLBytes;         // staging for buffers outside the arena (2 halves)
constexpr size_t kStageHalfBytes = 32u << 20;
constexpr size_t kOffHeap = kOffStage + 2 * kStageHalfBytes;   // user heap starts here (77 MiB)
constexpr uint32_t kLLSentinel = 0xFFFFFFFFu;           // a NaN pattern in f32/f16x2/bf16x2 (four NaNs in e4m3x4 and e5m2x4); payload words equal to it are rewritten
constexpr uint32_t kLLSanitized = 0x7FFF7FFFu;          // still NaN in every supported type (e4m3 / e5m2: 0x7F and 0xFF bytes are NaN), so
                                                        // bit-exact movement of arbitrary bytes uses the barrier-based kernels instead

// Point-to-point mailboxes, in the zero-initialised part of the first megabyte that the flag matrix does not use.
//   post: u64 [receiver rank][CTA][2 slots][2 words], written by the RECEIVER into the SENDER's arena ("write n bytes at this offset of mine")
//   done: u32 [sender rank][CTA],                      written by the SENDER into the RECEIVER's arena ("chunk number seq has landed")
constexpr int kP2pMaxBlocks = 32;                       // CTAs per send or recv operation: mailbox capacity (the default cap is lower, see p2p_blocks)
constexpr size_t kOffP2pPost = 256 << 10;
constexpr size_t kP2pPostBytes = (size_t)kMaxRanks * kP2pMaxBlocks * 2 * 2 * 8;
constexpr size_t kOffP2pDone = kOffP2pPost + kP2pPostBytes;
constexpr size_t kP2pDoneBytes = (size_t)kMaxRanks * kP2pMaxBlocks * 4;
static_assert(kOffP2pDone + kP2pDoneBytes <= kOffLL, "p2p mailboxes must fit below the Lamport scratch");
constexpr int kP2pTagBits = 24, kP2pValueBits = 40;     // each post word = (chunk sequence number mod 2^24) << 40 | value

// Routed expert dispatch (dispatch.cu): the count mailbox, int32 [source rank][kRouteMaxExperts]. Before the dispatch's exchange barrier
// every rank writes its per-expert slot counts into row [its rank] of every rank's mailbox; after it each rank reads the whole matrix.
constexpr int kRouteMaxExperts = 1024;
constexpr size_t kOffRouteCounts = 512 << 10;
constexpr size_t kRouteCountsBytes = (size_t)kMaxRanks * kRouteMaxExperts * 4;
static_assert(kOffRouteCounts >= kOffP2pDone + kP2pDoneBytes, "the route count mailbox must lie clear of the p2p mailboxes");
static_assert(kOffRouteCounts + kRouteCountsBytes <= kOffLL, "the route count mailbox must fit below the Lamport scratch");

// local (non-symmetric) per-comm state words
enum { kSeqBarrier = 0, kSeqLL = 1, kTicket = 2, kLLUsedLo0 = 3 /* 3,4,5 */, kLLUsedHi0 = 6 /* 6,7,8 */,
       kP2pSendSeq0 = 16 /* [peer][CTA]: chunks sent so far */, kP2pRecvSeq0 = kP2pSendSeq0 + kMaxRanks * kP2pMaxBlocks /* chunks received so far */,
       kStateWords = kP2pRecvSeq0 + kMaxRanks * kP2pMaxBlocks };

struct CommDev {
  int rank, nranks;
  char* peer[kMaxRanks];      // this process's mapping of every rank's arena (peer[rank] is mine)
  char* mc;                   // multicast alias of the arena, or nullptr
  uint32_t* state;            // local words, see enum above
  b200collFault* fault;       // host-pinned
  unsigned long long timeout_ns;
  int mcbar;                  // 1: cross-rank barriers are one multimem.red on a multicast counter + one polled local word (needs mc); 0: flag exchange
};

}  // namespace b200coll
