// Row quantization for int8 corpus shards and their queries (include/sgpt_b200.h sgpt_quantize_rows_i8): one warp per
// row, two passes over the row (absolute maximum, then quantize and sum the squares; the second pass hits L1/L2).
// Sign bits for binary corpus shards (sgpt_quantize_rows_b1): one warp per row, one ballot per 32 dimensions.
// e4m3 rows for the fp8 linear layers (sgpt_quantize_rows_fp8): one warp per row, two passes as for int8.
#include <cuda_fp8.h>

#include "../../include/sgpt_b200.h"
#include "common.cuh"
#include "gemm_api.h"
#include "host_utils.h"

using namespace sgpt;

namespace {

constexpr int kQuantThreads = 256;
constexpr int kQuantRows = kQuantThreads / 32;  // rows per CTA

// elements [off, off + 4) of the input, widened to fp32
__device__ __forceinline__ void load4(const void* __restrict__ x, int x_bf16, long long off, float (&v)[4]) {
  if (x_bf16) {
    const uint2 u = __ldg(reinterpret_cast<const uint2*>(static_cast<const uint16_t*>(x) + off));
    v[0] = bf16_lo(u.x);
    v[1] = bf16_hi(u.x);
    v[2] = bf16_lo(u.y);
    v[3] = bf16_hi(u.y);
  } else {
    const float4 f = __ldg(reinterpret_cast<const float4*>(static_cast<const float*>(x) + off));
    v[0] = f.x;
    v[1] = f.y;
    v[2] = f.z;
    v[3] = f.w;
  }
}

__global__ void __launch_bounds__(kQuantThreads) quantize_rows_i8_kernel(const void* __restrict__ x, int x_bf16,
                                                                          int8_t* __restrict__ q, float* __restrict__ scale,
                                                                          float* __restrict__ cos_scale, long long n,
                                                                          int D) {
  pdl_sync();
  const long long row = static_cast<long long>(blockIdx.x) * kQuantRows + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= n) return;  // warp-uniform
  const long long base = row * D;
  float amax = 0.f;
  bool finite = true;
  for (int i = 4 * lane; i < D; i += 128) {
    float v[4];
    load4(x, x_bf16, base + i, v);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      finite = finite && isfinite(v[u]);
      amax = fmaxf(amax, fabsf(v[u]));
    }
  }
  amax = warp_max(amax);
  finite = __all_sync(0xffffffffu, finite);
  char4* qr = reinterpret_cast<char4*>(q + base);
  if (!finite || amax == 0.f) {  // NaN / inf anywhere: every score against the row is NaN (-> -1); zero row: scores 0
    for (int i = 4 * lane; i < D; i += 128) qr[i >> 2] = make_char4(0, 0, 0, 0);
    if (lane == 0) scale[row] = cos_scale[row] = finite ? 0.f : __int_as_float(0x7fc00000);
    return;
  }
  const float m = __fdiv_rn(127.0f, amax);
  int ss = 0;  // <= 127^2 x 65536 < 2^31
  for (int i = 4 * lane; i < D; i += 128) {
    float v[4];
    load4(x, x_bf16, base + i, v);
    int c[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float t = fminf(fmaxf(rintf(__fmul_rn(v[u], m)), -127.f), 127.f);  // rint: round half to even
      c[u] = static_cast<int>(t);
      ss += c[u] * c[u];
    }
    qr[i >> 2] = make_char4(static_cast<signed char>(c[0]), static_cast<signed char>(c[1]),
                            static_cast<signed char>(c[2]), static_cast<signed char>(c[3]));
  }
  ss = __reduce_add_sync(0xffffffffu, ss);
  if (lane == 0) {
    const float s = __fdiv_rn(amax, 127.0f);
    scale[row] = s;
    cos_scale[row] = __fdiv_rn(s, fmaxf(__fmul_rn(s, __fsqrt_rn(__int2float_rn(ss))), 1e-12f));
  }
}

// Ballot word -> the np.packbits layout of its 32 dimensions.  The ballot has dimension j0 + l at bit l (lane order);
// np.packbits puts dimension j at bit 7 - (j & 7) of byte j / 8, i.e. byte i of the word holds dimensions j0 + 8 i ..
// j0 + 8 i + 7 with the first one at its MOST significant bit.  __brev reverses all 32 bits (bit l -> 31 - l), which
// reverses the bits inside every byte but also the byte order; the byte permutation 0x0123 restores the byte order.
__device__ __forceinline__ uint32_t packbits_order(uint32_t ballot) { return __byte_perm(__brev(ballot), 0, 0x0123); }

// Row `row`: lane c of the warp holds the word of dimensions base + 32 c .. + 31 for every 1024-dimension step; the word
// store is then one coalesced 128-byte row segment per step.  popc = the row's number of set bits.
__global__ void __launch_bounds__(kQuantThreads) quantize_rows_b1_kernel(const void* __restrict__ x, int x_bf16,
                                                                          const float* __restrict__ thresholds,
                                                                          uint32_t* __restrict__ bits,
                                                                          int32_t* __restrict__ popc, long long n, int D) {
  pdl_sync();
  const long long row = static_cast<long long>(blockIdx.x) * kQuantRows + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= n) return;  // warp-uniform
  const long long base = row * D;
  uint32_t* out = bits + row * (D / 32);
  int count = 0;
  for (int j0 = 0; j0 < D; j0 += 1024) {
    uint32_t mine = 0;
#pragma unroll 4
    for (int c = 0; c < 32; ++c) {
      const int j = j0 + 32 * c + lane;
      if (j0 + 32 * c >= D) break;  // warp-uniform (D % 128 == 0)
      const float v = x_bf16 ? bf16_lo(static_cast<uint32_t>(__ldg(static_cast<const uint16_t*>(x) + base + j)))
                             : __ldg(static_cast<const float*>(x) + base + j);
      const float t = thresholds != nullptr ? __ldg(thresholds + j) : 0.f;
      const uint32_t w = __ballot_sync(0xffffffffu, v > t);  // strict; a NaN on either side gives 0
      if (lane == c) mine = packbits_order(w);
    }
    if (j0 + 32 * lane < D) {
      out[(j0 >> 5) + lane] = mine;
      count += __popc(mine);
    }
  }
  count = __reduce_add_sync(0xffffffffu, count);
  if (lane == 0) popc[row] = count;
}

// Row of K bf16 -> K e4m3 + one fp32 scale (include/sgpt_b200.h fp8 linear layers).  Lane l handles 4 consecutive
// elements (one 8-byte load, one 4-byte store) of every 128-element step; the second pass hits L1/L2.
__global__ void __launch_bounds__(kQuantThreads) quantize_rows_fp8_kernel(const uint16_t* __restrict__ x,
                                                                           uint8_t* __restrict__ q,
                                                                           float* __restrict__ scale, long long n,
                                                                           int K) {
  pdl_sync();
  const long long row = static_cast<long long>(blockIdx.x) * kQuantRows + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= n) return;  // warp-uniform
  const long long base = row * K;
  float amax = 0.f;
  bool finite = true;
  for (int i = 4 * lane; i < K; i += 128) {
    float v[4];
    load4(x, 1, base + i, v);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      finite = finite && isfinite(v[u]);
      amax = fmaxf(amax, fabsf(v[u]));
    }
  }
  amax = warp_max(amax);
  finite = __all_sync(0xffffffffu, finite);
  uint32_t* qr = reinterpret_cast<uint32_t*>(q + base);
  if (!finite) {  // NaN / inf anywhere: q = 0 and scale = NaN, so every output of the row is NaN
    for (int i = 4 * lane; i < K; i += 128) qr[i >> 2] = 0u;
    if (lane == 0) scale[row] = __int_as_float(0x7fc00000);
    return;
  }
  // zero row: inv = 0, q = +-0, scale = 0; inv stays finite even for the tiniest bf16 amax
  const float inv = amax > 0.f ? fminf(__fdiv_rn(448.0f, amax), 3.40282347e38f) : 0.f;
  for (int i = 4 * lane; i < K; i += 128) {
    float v[4];
    load4(x, 1, base + i, v);
    const __nv_fp8x2_storage_t lo = __nv_cvt_float2_to_fp8x2(make_float2(__fmul_rn(v[0], inv), __fmul_rn(v[1], inv)),
                                                             __NV_SATFINITE, __NV_E4M3);
    const __nv_fp8x2_storage_t hi = __nv_cvt_float2_to_fp8x2(make_float2(__fmul_rn(v[2], inv), __fmul_rn(v[3], inv)),
                                                             __NV_SATFINITE, __NV_E4M3);
    qr[i >> 2] = static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
  }
  if (lane == 0) scale[row] = __fdiv_rn(amax, 448.0f);
}

}  // namespace

extern "C" int sgpt_quantize_rows_fp8(const void* x, void* q_out, float* scale_out, int64_t n, int K,
                                      sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(n >= 0, "sgpt_quantize_rows_fp8: bad row count n=%lld", (long long)n);
  SGPT_REQUIRE(K > 0 && K % 16 == 0, "sgpt_quantize_rows_fp8: K=%d must be a positive multiple of 16", K);
  if (n == 0) return SGPT_OK;
  SGPT_REQUIRE(x != nullptr && q_out != nullptr && scale_out != nullptr, "sgpt_quantize_rows_fp8: null argument");
  SGPT_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(q_out) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(scale_out) & 3) == 0,
               "sgpt_quantize_rows_fp8: x and q_out must be 16-byte aligned, scale_out 4-byte aligned");
  const long long blocks = (n + kQuantRows - 1) / kQuantRows;
  SGPT_REQUIRE(blocks < (1ll << 31), "sgpt_quantize_rows_fp8: too many rows");
  LaunchScope _ls(kCatMisc, stream);
  SGPT_CHECK_CUDA(launch_kernel(quantize_rows_fp8_kernel, dim3(static_cast<unsigned>(blocks)), dim3(kQuantThreads), 0,
                                stream, static_cast<const uint16_t*>(x), static_cast<uint8_t*>(q_out), scale_out,
                                static_cast<long long>(n), K));
  return SGPT_OK;
}

extern "C" int sgpt_quantize_rows_b1(const void* x, int x_bf16, const float* thresholds, void* bits_out,
                                     int32_t* popc_out, int64_t n, int D, sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(n >= 0, "sgpt_quantize_rows_b1: bad row count n=%lld", (long long)n);
  SGPT_REQUIRE(D > 0 && D % 128 == 0 && D <= kMaxDimB1,
               "sgpt_quantize_rows_b1: D=%d must be a positive multiple of 128, at most %d", D, kMaxDimB1);
  if (n == 0) return SGPT_OK;
  SGPT_REQUIRE(x != nullptr && bits_out != nullptr && popc_out != nullptr, "sgpt_quantize_rows_b1: null argument");
  SGPT_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(bits_out) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(popc_out) & 3) == 0 && (reinterpret_cast<uintptr_t>(thresholds) & 3) == 0,
               "sgpt_quantize_rows_b1: x and bits_out must be 16-byte aligned, popc_out and thresholds 4-byte aligned");
  const long long blocks = (n + kQuantRows - 1) / kQuantRows;
  SGPT_REQUIRE(blocks < (1ll << 31), "sgpt_quantize_rows_b1: too many rows");
  LaunchScope _ls(kCatMisc, stream);
  SGPT_CHECK_CUDA(launch_kernel(quantize_rows_b1_kernel, dim3(static_cast<unsigned>(blocks)), dim3(kQuantThreads), 0,
                                stream, x, x_bf16, thresholds, static_cast<uint32_t*>(bits_out), popc_out,
                                static_cast<long long>(n), D));
  return SGPT_OK;
}

extern "C" int sgpt_quantize_rows_i8(const void* x, int x_bf16, void* q_out, float* scale_out, float* cos_scale_out,
                                     int64_t n, int D, sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(n >= 0, "sgpt_quantize_rows_i8: bad row count n=%lld", (long long)n);
  SGPT_REQUIRE(D > 0 && D % 16 == 0 && D <= kMaxDimI8,
               "sgpt_quantize_rows_i8: D=%d must be a positive multiple of 16, at most %d", D, kMaxDimI8);
  if (n == 0) return SGPT_OK;
  SGPT_REQUIRE(x != nullptr && q_out != nullptr && scale_out != nullptr && cos_scale_out != nullptr,
               "sgpt_quantize_rows_i8: null argument");
  SGPT_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(q_out) & 15) == 0,
               "sgpt_quantize_rows_i8: x and q_out must be 16-byte aligned");
  const long long blocks = (n + kQuantRows - 1) / kQuantRows;
  SGPT_REQUIRE(blocks < (1ll << 31), "sgpt_quantize_rows_i8: too many rows");
  LaunchScope _ls(kCatMisc, stream);
  SGPT_CHECK_CUDA(launch_kernel(quantize_rows_i8_kernel, dim3(static_cast<unsigned>(blocks)), dim3(kQuantThreads), 0,
                                stream, x, x_bf16, static_cast<int8_t*>(q_out), scale_out, cos_scale_out,
                                static_cast<long long>(n), D));
  return SGPT_OK;
}
