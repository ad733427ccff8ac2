// Row quantization for int8 corpus shards and their queries (include/sgpt_b200.h sgpt_quantize_rows_i8): one warp per
// row, two passes over the row (absolute maximum, then quantize and sum the squares; the second pass hits L1/L2).
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

}  // namespace

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
