// The per-peer argument blocks of the all-to-all(v) kernels (k_a2av_push in kernels.cuh, k_a2av_quant_push in dispatch.cu,
// k_combine_pull<…, SegmentMap> in combine.cu) and the host code that fills and checks them. Plain C++: the kernels take them by value, the host
// entry points build them.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <string>

#include "layout.h"

namespace b200coll {

// Per destination p: nvec[p] input vectors starting at vector src_vec[p] of my send buffer go to output-vector offset dst_vec[p] of peer
// p's recv buffer (the kernel defines the units). The (peer, vector) space is flattened with a prefix table so skewed expert loads still
// spread over all CTAs.
struct A2AvArgs {
  unsigned long long src_vec[kMaxRanks];
  unsigned long long dst_vec[kMaxRanks];
  unsigned long long prefix[kMaxRanks + 1];   // prefix over the staggered order j = 0..nranks-1 (peer = rank+1+j)
};

// Fill the flattened prefix in the kernels' staggered order (j -> peer rank+1+j).
inline void a2av_prefix(int rank, int nranks, const unsigned long long* nvec_by_peer, A2AvArgs* a) {
  a->prefix[0] = 0;
  for (int j = 0; j < nranks; j++) {
    int p = rank + 1 + j; if (p >= nranks) p -= nranks;
    a->prefix[j + 1] = a->prefix[j] + nvec_by_peer[p];
  }
  for (int j = nranks + 1; j <= kMaxRanks; j++) a->prefix[j] = a->prefix[nranks];
}

// The row geometry of one all-to-all-v call, in rows: rows[p] rows starting at row src_row[p] of the dispatch send buffer go to row
// dst_row[p] of peer p's symmetric receive buffer. Entries past nranks are zero.
struct A2AvRows {
  unsigned long long src_row[kMaxRanks];
  unsigned long long dst_row[kMaxRanks];
  unsigned long long rows[kMaxRanks];
};

// The host arrays of an all-to-all-v call (length nranks), checked and converted: no negative entry, every destination range inside
// the recv_rows rows of the receive buffers, and every send row below max_rows (the caller's bound that keeps byte offsets in size_t).
// Returns "" or why the arrays are refused.
inline std::string a2av_rows(int nranks, const int64_t* send_rows, const int64_t* send_row_off, const int64_t* recv_row_off_at_peer, size_t recv_rows,
                             size_t max_rows, A2AvRows* g) {
  *g = A2AvRows{};
  for (int p = 0; p < nranks; p++) {
    if (send_rows[p] < 0 || send_row_off[p] < 0 || recv_row_off_at_peer[p] < 0) return "negative row count or offset";
    const size_t rows = (size_t)send_rows[p], src = (size_t)send_row_off[p], dst = (size_t)recv_row_off_at_peer[p];
    if (rows > recv_rows || dst > recv_rows - rows)
      return "rows for peer " + std::to_string(p) + " land at [" + std::to_string(dst) + ", +" + std::to_string(rows) + "), past recv_rows = " + std::to_string(recv_rows);
    if (src > max_rows || rows > max_rows - src) return "the send range of peer " + std::to_string(p) + " is too large";
    g->src_row[p] = src;
    g->dst_row[p] = dst;
    g->rows[p] = rows;
  }
  return "";
}

}  // namespace b200coll
