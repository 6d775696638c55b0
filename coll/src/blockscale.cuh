// Device helpers shared by the block-scaled FP8 collectives (blockscaled.cu) and the quantising collectives (quantized.cu): invariant
// integer division, the per-warp scale exchange, the dequantising accumulate and the rounding store.
#pragma once
#include <stdint.h>

#include <type_traits>

#include "device.cuh"

namespace b200coll {

// q = floor(n / d) for every 32-bit n as (umulhi(n, m) + n) >> l, l = ceil(log2 d), m = floor(2^32 (2^l - d) / d) + 1 (Granlund and
// Montgomery, "Division by invariant integers using multiplication", 1994). The sum needs 33 bits, so it is formed in 64.
struct FastDiv {
  uint32_t d, m, l;
  __device__ __forceinline__ uint32_t div(uint32_t n) const { return (uint32_t)(((unsigned long long)__umulhi(n, m) + n) >> l); }
};
inline FastDiv make_fastdiv(uint32_t d) {
  uint32_t l = 0;
  while (l < 32 && (1ull << l) < d) l++;
  return FastDiv{d, (uint32_t)(((1ull << 32) * ((1ull << l) - d)) / d + 1), l};
}

// The scale of every lane's vector, one load per distinct index in the warp. All 32 lanes call it; `active` lanes have a vector.
struct WarpScale {
  unsigned leader;
  bool loads;
  __device__ __forceinline__ WarpScale(uint32_t idx, bool active) {
    const unsigned same = __match_any_sync(0xFFFFFFFFu, active ? idx : 0xFFFFFFFFu);
    leader = __ffs(same) - 1;
    loads = active && (threadIdx.x & 31) == leader;
  }
  __device__ __forceinline__ float get(const char* scales, uint32_t idx) const {
    float s = 0.f;
    if (loads) s = *reinterpret_cast<const float*>(scales + (size_t)idx * 4);
    return __shfl_sync(0xFFFFFFFFu, s, leader);
  }
};

// acc[i] += float(q[i]) * s, both roundings kept (no fused multiply-add): the value of an element is the rounded product.
template <typename InT> __device__ __forceinline__ void bsq_dequant_add(float* acc, const uint4& v, float s) {
  constexpr __nv_fp8_interpretation_t I = std::is_same<InT, __nv_fp8_e4m3>::value ? __NV_E4M3 : __NV_E5M2;
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; i++) {
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const __half2_raw r = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w[i] >> (16 * h)), I);   // F2FP.F16.E4M3 / E5M2.UNPACK_B
      const float2 f = __half22float2(__half2(r));
      acc[4 * i + 2 * h] = __fadd_rn(acc[4 * i + 2 * h], __fmul_rn(f.x, s));
      acc[4 * i + 2 * h + 1] = __fadd_rn(acc[4 * i + 2 * h + 1], __fmul_rn(f.y, s));
    }
  }
}

// out = round_once(acc * scale): 16 elements, 32 (bf16 / fp16) or 64 (fp32) bytes
template <typename OutT> __device__ __forceinline__ void bsq_store(void* dst, const float* acc, float scale) {
  constexpr int W = Pack<OutT, 16>::W;
  float f[16];
#pragma unroll
  for (int i = 0; i < 16; i++) f[i] = __fmul_rn(acc[i], scale);
  uint32_t w[W];
  Pack<OutT, 16>::run(f, w);
  if constexpr (W == 16) {
#pragma unroll
    for (int k = 0; k < 4; k++) st_vec(reinterpret_cast<char*>(dst) + 16 * k, make_uint4(w[4 * k], w[4 * k + 1], w[4 * k + 2], w[4 * k + 3]));
  } else {
    st_words<W>(dst, w);
  }
}

}  // namespace b200coll
