// The exact per-row score of sgpt_rerank (include/sgpt_b200.h), shared by ivfpq.cu's rerank_kernel and graph.cu's
// beam search so that both return the same bits for the same (query, row).
#pragma once
#include "common.cuh"

namespace sgpt {

// One warp: the unscaled score of the 16-byte-aligned rows qp and cp of row_bytes bytes (int8: D bytes, bf16: 2 D), the
// same value in every lane.  The caller applies q_scale, c_scale and the NaN mapping.
template <bool kS8>
__device__ __forceinline__ float rerank_dot(const uint4* __restrict__ qp, const uint4* __restrict__ cp, int units,
                                            int lane) {
  if constexpr (kS8) {
    int acc = 0;  // exact: |sum| <= 65536 x 128 x 128
    for (int u = lane; u < units; u += 32) {
      const uint4 a = __ldg(qp + u), b = __ldg(cp + u);
      acc = __dp4a(static_cast<int>(a.x), static_cast<int>(b.x), acc);
      acc = __dp4a(static_cast<int>(a.y), static_cast<int>(b.y), acc);
      acc = __dp4a(static_cast<int>(a.z), static_cast<int>(b.z), acc);
      acc = __dp4a(static_cast<int>(a.w), static_cast<int>(b.w), acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    return __int2float_rn(acc);
  } else {
    // lane l: 16-byte units l, l + 32, ... in order, the 8 elements of a unit in order; every bf16 x bf16 product is exact
    // in fp32, so fmaf adds it with one rounding.  Then the xor butterfly over the lanes (offsets 16, 8, 4, 2, 1): lanes
    // i and i ^ o add the same two values, so every lane ends with the same sum
    float acc = 0.f;
    auto dot2 = [](uint32_t a, uint32_t b, float s) {
      return fmaf(bf16_hi(a), bf16_hi(b), fmaf(bf16_lo(a), bf16_lo(b), s));
    };
#pragma unroll 2
    for (int u = lane; u < units; u += 32) {
      const uint4 a = __ldg(qp + u), b = __ldg(cp + u);
      acc = dot2(a.w, b.w, dot2(a.z, b.z, dot2(a.y, b.y, dot2(a.x, b.x, acc))));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    return acc;
  }
}

}  // namespace sgpt
