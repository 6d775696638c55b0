// Index helpers shared by the layout-move kernels (ulysses.cu, context.cu): 32-bit division by a host-computed multiplier, and the
// row-strided byte regions whose overlap the host checks before a launch.
#pragma once
#include <stddef.h>
#include <stdint.h>

namespace b200coll {

// n / d for n < 2^31 and 1 <= d < 2^31: q = (umulhi(n, m) + n) >> l with l = ceil(log2 d) and m = floor(2^32 * (2^l - d) / d) + 1.
struct FastDiv {
  uint32_t d, m, l;
};
inline FastDiv fast_div(uint32_t d) {
  uint32_t l = 0;
  while (l < 32 && (1ull << l) < d) l++;
  return FastDiv{d, (uint32_t)((((1ull << l) - d) << 32) / d + 1), l};
}
__device__ __forceinline__ uint32_t div_by(uint32_t n, const FastDiv& f) { return (__umulhi(n, f.m) + n) >> f.l; }

// A row-strided byte region: rows rows of width bytes, stride bytes apart (a dense buffer is one row).
struct Span {
  uintptr_t p;
  size_t rows, stride, width;
  size_t extent() const { return rows == 0 ? 0 : (rows - 1) * stride + width; }
};

// Whether two regions share a byte. Disjoint extents never do. Two views with one row stride (column slices of one packed buffer) share
// a byte only if their columns meet, modulo the stride; anything else with overlapping extents counts as overlapping.
static bool spans_overlap(const Span& a, const Span& b) {
  const size_t ea = a.extent(), eb = b.extent();
  if (ea == 0 || eb == 0 || !(a.p < b.p + eb && b.p < a.p + ea)) return false;
  if (a.rows < 2 || b.rows < 2 || a.stride != b.stride || a.width > a.stride || b.width > b.stride) return true;
  const size_t dd = (b.p >= a.p ? b.p - a.p : a.stride - (a.p - b.p) % a.stride) % a.stride;   // b's columns start at dd, modulo the stride
  return dd < a.width || dd + b.width > a.stride;
}

}  // namespace b200coll
