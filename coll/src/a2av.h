// The per-peer argument block of the all-to-all(v) push kernels (k_a2av_push in kernels.cuh, k_a2av_quant_push in blockscaled.cu) and
// the host code that fills its prefix. Plain C++: the kernels take it by value, the host entry points build it.
#pragma once
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

}  // namespace b200coll
