// The quantise side of the FP8 kernels, shared by the quantising collectives (blockscaled.cu), the quantising dispatches (dispatch.cu)
// and the quantising combine (combine.cu): the one walk over 16-element vectors, the load-and-widen of a vector, the per-block
// quantiser, and the dequantiser.
//
// Quantising, per block: amax = max |x| (the largest unsigned bit pattern of |x|, so a NaN anywhere makes amax NaN); inv = FMAX / amax
// and s = amax / FMAX, both IEEE divisions rounded to nearest, inv = s = 1 when amax == 0 or inv overflows; q = fp8_satfinite(x * inv);
// the dequantised value is float(q) * s. FMAX is 448 (e4m3) or 57344 (e5m2).
//
// Blocks stay inside one warp iteration. block is a power of two from 16 to 512 elements (1 to 32 vectors), and every caller starts a
// warp's vectors on a whole block: so the lanes of one block are consecutive lanes of one warp, all active or all idle, and the amax is
// a butterfly over those lanes: no shared memory, no cross-warp step.
#pragma once
#include <math.h>
#include <stdint.h>

#include <type_traits>

#include "device.cuh"

namespace b200coll {

constexpr int kBsqThreads = 512;

template <typename WireT> constexpr float kWireMax = 448.0f;
template <> constexpr float kWireMax<__nv_fp8_e5m2> = 57344.0f;

struct QuantGeom {
  size_t data_off, scale_off;     // arena offsets of the scratch FP8 copy and of its scales (the same on every rank)
  uint32_t nvec;                  // 16-element vectors in one rank's send buffer
  uint32_t nblk;                  // blocks in one rank's send buffer
  uint32_t lvpb;                  // log2(vectors per block)
  __device__ __forceinline__ uint32_t scale_index(uint32_t v) const { return v >> lvpb; }
};

// The one walk over vectors [v0, v1): a warp takes 32 consecutive vectors starting at v0 plus a multiple of 32, the grid strides
// over the range, and all 32 lanes run every iteration (f(v, active), active = v < v1), so the full-mask warp intrinsics below always
// see whole warps. 32-bit indices: the host keeps nvec below 2^31, so b + stride cannot wrap.
template <typename F>
__device__ __forceinline__ void warp_walk(uint32_t v0, uint32_t v1, F&& f) {
  const uint32_t lane = threadIdx.x & 31;
  for (uint32_t b = v0 + blockIdx.x * blockDim.x + (threadIdx.x & ~31u); b < v1; b += gridDim.x * blockDim.x) f(b + lane, b + lane < v1);
}

// 16 elements of InT at p, widened (exactly) to fp32
template <typename InT> __device__ __forceinline__ void quant_load16(const char* p, float* x) {
  uint4 raw[sizeof(InT)];
#pragma unroll
  for (int k = 0; k < (int)sizeof(InT); k++) raw[k] = ld_vec(p + 16 * k);
  widen16<InT>(raw, x);
}

// Quantise this lane's 16 elements with the amax of its block, whose vectors are held by the aligned group of `gl` lanes (a power of
// two up to 32) this lane belongs to. All 32 lanes call it; idle lanes pass zeros, and their groups are wholly idle. Returns the FP8
// vector; *scale receives s.
template <typename WireT> __device__ __forceinline__ uint4 quant_vec(const float* x, uint32_t gl, float* scale) {
  uint32_t m = 0;
#pragma unroll
  for (int i = 0; i < 16; i++) m = max(m, __float_as_uint(x[i]) & 0x7FFFFFFFu);
  for (uint32_t o = 1; o < gl; o <<= 1) m = max(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
  const float amax = __uint_as_float(m);
  float inv = __fdiv_rn(kWireMax<WireT>, amax), s = __fdiv_rn(amax, kWireMax<WireT>);
  if (amax == 0.0f || inv == INFINITY) { inv = 1.0f; s = 1.0f; }
  float y[16];
#pragma unroll
  for (int i = 0; i < 16; i++) y[i] = __fmul_rn(x[i], inv);
  uint32_t w[4];
  Pack<WireT, 16>::run(y, w);                                     // cvt.rn.satfinite: F2FP.SATFINITE.E4M3 / .E5M2
  *scale = s;
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// x[i] = float(q[i]) * s for the 16 FP8 elements of v: the dequantised value of an element is the rounded product.
template <typename WireT> __device__ __forceinline__ void dequant16(const uint4& v, float s, float* x) {
  constexpr __nv_fp8_interpretation_t I = std::is_same<WireT, __nv_fp8_e4m3>::value ? __NV_E4M3 : __NV_E5M2;
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; i++) {
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const __half2_raw r = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w[i] >> (16 * h)), I);   // F2FP.F16.E4M3 / E5M2.UNPACK_B
      const float2 f = __half22float2(__half2(r));
      x[4 * i + 2 * h] = __fmul_rn(f.x, s);
      x[4 * i + 2 * h + 1] = __fmul_rn(f.y, s);
    }
  }
}

// acc[i] += float(q[i]) * s, both roundings kept (no fused multiply-add)
template <typename WireT> __device__ __forceinline__ void bsq_dequant_add(float* acc, const uint4& v, float s) {
  float x[16];
  dequant16<WireT>(v, s, x);
#pragma unroll
  for (int i = 0; i < 16; i++) acc[i] = __fadd_rn(acc[i], x[i]);
}

// Quantise vectors [v0, v1) of in into q and its scales, walked as the pull loops walk a slice.
template <typename InT, typename WireT>
__device__ __forceinline__ void quant_range(const QuantGeom& g, const char* in, char* q, char* scales, uint32_t v0, uint32_t v1) {
  const uint32_t lane = threadIdx.x & 31, gl = 1u << g.lvpb;
  warp_walk(v0, v1, [&](uint32_t v, bool act) {
    float x[16] = {};
    if (act) quant_load16<InT>(in + (size_t)v * (16 * sizeof(InT)), x);
    float s;
    const uint4 w = quant_vec<WireT>(x, gl, &s);
    if (act) {
      st_vec(q + (size_t)v * 16, w);
      if ((lane & (gl - 1)) == 0) *reinterpret_cast<float*>(scales + (size_t)g.scale_index(v) * 4) = s;
    }
  });
}

}  // namespace b200coll
