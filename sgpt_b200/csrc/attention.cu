// F4: causal (optionally sliding-window) self-attention over a ragged batch, HF:gpt_neo/modeling_gpt_neo.py:105-130.
//
// Tensor-core kernel (impl 0): FlashAttention-2 style with mma.sync.m16n8k16 (bf16 operands, fp32 accumulate).  One CTA =
// one (head, sequence, 64-query tile), 4 warps; warp w owns query rows 16 w .. 16 w + 15, and each thread holds two rows
// (g, g + 8 of its warp's 16) of the score and output fragments, so a row reduction is two shuffles inside a quad.
//   smem : Q [64 x hd] | two stages of { K_j [KT x hd], V_j [KT x hd] } (KT = 64 keys, 32 at hd = 256), rows padded by
//          16 bytes so that every ldmatrix phase hits 8 distinct bank groups; filled by cp.async, positions beyond the
//          sequence zero-filled
//   loop over the key tiles j the causal / window mask can reach (K_{j+1}, V_{j+1} load while tile j computes):
//       S  = Q K_j^T                    mma.sync, A = Q (ldmatrix), B = K_j (ldmatrix: [key, hd] rows are K-major)
//       online softmax in fp32 in the exp2 domain (running max m and per-thread partial sum l per row)
//       O  = alpha * O + P V_j          P re-packed from the S accumulators into bf16 A fragments (no smem round trip),
//                                       B = V_j (ldmatrix.trans: V is [key, hd] row-major)
//   epilogue: O / l -> bf16 -> out[token, head*hd : (head+1)*hd]
//
// SIMT kernel (impl 1): one warp per (token, head), fp32 everywhere — test cross-check only.
#include <math.h>
#include <stdlib.h>

#include "../../include/sgpt_b200.h"
#include "common.cuh"
#include "host_utils.h"

namespace sgpt {

constexpr int kAttnQ = 64;  // query rows per CTA (4 warps x 16)
constexpr int kAttnThreads = 128;

template <int HD>
struct AttnCfg {
  static constexpr int KT = HD == 256 ? 32 : 64;  // keys per tile (hd 256: the 128 output accumulators need the registers)
  static constexpr int kPitch = HD + 8;            // bf16 per smem row
  static constexpr int kQElems = kAttnQ * kPitch;
  static constexpr int kKVElems = KT * kPitch;
  static constexpr int kSmemBytes = (kQElems + 4 * kKVElems) * 2;
};

__device__ __forceinline__ void cp_async_16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}
// c[16 x 8] += a[16 x 16] * b[16 x 8]   (bf16 operands, fp32 accumulators)
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// `rows` rows of HD bf16 (sequence positions p0 .. p0 + rows - 1, columns col .. col + HD - 1 of the qkv matrix) ->
// smem rows of kPitch; positions at or beyond the sequence length are zero-filled
template <int HD>
__device__ __forceinline__ void attn_load_rows(uint32_t sdst, const __nv_bfloat16* __restrict__ qkv, size_t ld, int seq0,
                                               int p0, int rows, int len, int col, int tid) {
  constexpr int C = HD / 8;  // 16-byte chunks per row
  for (int i = tid; i < rows * C; i += kAttnThreads) {
    const int r = i / C, c = i - r * C;
    const int p = p0 + r;
    const bool ok = p < len;
    cp_async_16(sdst + (r * AttnCfg<HD>::kPitch + c * 8) * 2, qkv + static_cast<size_t>(seq0 + (ok ? p : 0)) * ld + col + c * 8,
                ok);
  }
}

template <int HD>
__global__ void __launch_bounds__(kAttnThreads) attention_mma_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                                     __nv_bfloat16* __restrict__ out,
                                                                     const int32_t* __restrict__ cu, int H, float sl2,
                                                                     int window, const float* __restrict__ alibi) {
  using Cfg = AttnCfg<HD>;
  constexpr int KT = Cfg::KT, P = Cfg::kPitch;
  // heads vary fastest over the grid: the CTAs resident at the same time read all heads' q / k / v pieces of the same
  // token rows, i.e. whole rows of the qkv matrix
  const int h = blockIdx.x, b = blockIdx.y, qt = blockIdx.z;
  pdl_sync();  // programmatic dependent launch: see common.cuh
  const int seq0 = __ldg(cu + b);
  const int len = __ldg(cu + b + 1) - seq0;
  const int qp0 = qt * kAttnQ;
  if (qp0 >= len) return;

  extern __shared__ __align__(16) uint8_t attn_smem[];
  const uint32_t sQ = smem_u32(attn_smem);
  const uint32_t sKV = sQ + Cfg::kQElems * 2;  // stage s: K at sKV + 2 s kKVElems * 2, V right behind it
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int d = H * HD;
  const size_t ld = 3 * static_cast<size_t>(d);

  const int lo_pos = (window > 0) ? max(0, qp0 - window + 1) : 0;
  const int j_lo = lo_pos / KT;
  const int j_hi = min(qp0 + kAttnQ - 1, len - 1) / KT;

  attn_load_rows<HD>(sQ, qkv, ld, seq0, qp0, kAttnQ, len, h * HD, tid);
  attn_load_rows<HD>(sKV, qkv, ld, seq0, j_lo * KT, KT, len, d + h * HD, tid);
  attn_load_rows<HD>(sKV + Cfg::kKVElems * 2, qkv, ld, seq0, j_lo * KT, KT, len, 2 * d + h * HD, tid);
  cp_async_commit();

  // BLOOM ALiBi (HF:bloom/modeling_bloom.py:84-86): + slope_h * (key position) before the softmax, here pre-multiplied
  // by log2(e) because the softmax runs in the exp2 domain
  const float slope2 = (alibi != nullptr) ? __ldg(alibi + h) * 1.4426950408889634f : 0.f;
  const int g = lane >> 2, t4 = lane & 3;
  int vis_hi[2], vis_lo[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qpos = qp0 + warp * 16 + g + 8 * r;
    vis_hi[r] = min(qpos, len - 1);
    vis_lo[r] = (window > 0) ? (qpos - window + 1) : 0;
  }
  float o[HD / 8][4];
#pragma unroll
  for (int n = 0; n < HD / 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  for (int j = j_lo; j <= j_hi; ++j) {
    const int s = (j - j_lo) & 1;
    if (j < j_hi) {  // the other stage was released by the __syncthreads at the end of the previous tile
      const uint32_t nk = sKV + (s ^ 1) * 2 * Cfg::kKVElems * 2;
      attn_load_rows<HD>(nk, qkv, ld, seq0, (j + 1) * KT, KT, len, d + h * HD, tid);
      attn_load_rows<HD>(nk + Cfg::kKVElems * 2, qkv, ld, seq0, (j + 1) * KT, KT, len, 2 * d + h * HD, tid);
    }
    cp_async_commit();
    cp_async_wait<1>();  // everything but the prefetch just issued has landed
    __syncthreads();
    const uint32_t sK = sKV + s * 2 * Cfg::kKVElems * 2, sV = sK + Cfg::kKVElems * 2;

    // ---- S = Q K_j^T ----
    float sc[KT / 8][4];
#pragma unroll
    for (int n = 0; n < KT / 8; ++n) sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {
      uint32_t a[4];
      ldmatrix_x4(sQ + ((warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * P + kk * 16 + (lane >> 4) * 8) * 2, a);
#pragma unroll
      for (int nb = 0; nb < KT / 16; ++nb) {
        uint32_t kb[4];
        ldmatrix_x4(sK + ((nb * 16 + (lane & 7) + (lane >> 4) * 8) * P + kk * 16 + ((lane >> 3) & 1) * 8) * 2, kb);
        mma_bf16_16816(sc[2 * nb], a, kb[0], kb[1]);
        mma_bf16_16816(sc[2 * nb + 1], a, kb[2], kb[3]);
      }
    }

    // ---- online softmax (exp2 domain); element e of sc[n] is row g + 8 (e / 2), key kv0 + 8 n + 2 t4 + e % 2 ----
    const int kv0 = j * KT;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int n = 0; n < KT / 8; ++n) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = e >> 1;
        const int kp = kv0 + 8 * n + 2 * t4 + (e & 1);
        const float x = fmaf(sc[n][e], sl2, slope2 * static_cast<float>(kp));
        sc[n][e] = (kp <= vis_hi[r] && kp >= vis_lo[r]) ? x : -INFINITY;
        mx[r] = fmaxf(mx[r], sc[n][e]);
      }
    }
    float alpha[2], m_use[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m_run[r], mx[r]);
      m_use[r] = (m_new == -INFINITY) ? 0.f : m_new;
      alpha[r] = exp2f(m_run[r] - m_use[r]);
      m_run[r] = m_new;
    }
    float lsum[2] = {0.f, 0.f};
#pragma unroll
    for (int n = 0; n < KT / 8; ++n) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        sc[n][e] = exp2f(sc[n][e] - m_use[e >> 1]);
        lsum[e >> 1] += sc[n][e];
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) l_run[r] = l_run[r] * alpha[r] + lsum[r];
#pragma unroll
    for (int n = 0; n < HD / 8; ++n) {
      o[n][0] *= alpha[0];
      o[n][1] *= alpha[0];
      o[n][2] *= alpha[1];
      o[n][3] *= alpha[1];
    }

    // ---- O += P V_j ----
#pragma unroll
    for (int kk = 0; kk < KT / 16; ++kk) {
      uint32_t a[4];
      a[0] = pack_bf16(sc[2 * kk][0], sc[2 * kk][1]);
      a[1] = pack_bf16(sc[2 * kk][2], sc[2 * kk][3]);
      a[2] = pack_bf16(sc[2 * kk + 1][0], sc[2 * kk + 1][1]);
      a[3] = pack_bf16(sc[2 * kk + 1][2], sc[2 * kk + 1][3]);
#pragma unroll
      for (int nd = 0; nd < HD / 16; ++nd) {
        uint32_t vb[4];
        ldmatrix_x4_trans(sV + ((kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * P + nd * 16 + (lane >> 4) * 8) * 2, vb);
        mma_bf16_16816(o[2 * nd], a, vb[0], vb[1]);
        mma_bf16_16816(o[2 * nd + 1], a, vb[2], vb[3]);
      }
    }
    __syncthreads();  // stage s may be refilled by the next iteration's prefetch
  }

  // ---- epilogue: O / l -> bf16 ----
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = l_run[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv_l = (l > 0.f) ? 1.0f / l : 0.f;
    const int qpos = qp0 + warp * 16 + g + 8 * r;
    if (qpos < len) {
      __nv_bfloat16* dst = out + static_cast<size_t>(seq0 + qpos) * d + h * HD + 2 * t4;
#pragma unroll
      for (int n = 0; n < HD / 8; ++n)
        *reinterpret_cast<uint32_t*>(dst + 8 * n) = pack_bf16(o[n][2 * r] * inv_l, o[n][2 * r + 1] * inv_l);
    }
  }
}

template <int HD>
static int launch_attention_mma(const void* qkv, void* out, const int32_t* cu, int B, int H, float scale, int window,
                                int max_seqlen, const float* alibi, cudaStream_t stream) {
  using Cfg = AttnCfg<HD>;
  auto kern = attention_mma_kernel<HD>;
  static PerDeviceOnce attr_once;
  if (attr_once.first())
    SGPT_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
  const int QT = (max_seqlen + kAttnQ - 1) / kAttnQ;
  const float sl2 = scale * 1.4426950408889634f;
  LaunchScope _ls(kCatAttention, stream);
  SGPT_CHECK_CUDA(launch_kernel(kern, dim3(H, B, QT), dim3(kAttnThreads), Cfg::kSmemBytes, stream,
                                static_cast<const __nv_bfloat16*>(qkv), static_cast<__nv_bfloat16*>(out), cu, H, sl2, window,
                                alibi));
  return SGPT_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// SIMT cross-check: one warp per (token, head); lanes split the head dimension; fp32 online softmax.
// ---------------------------------------------------------------------------------------------------------------
template <int HD>
__global__ void __launch_bounds__(256) attention_simt_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                             __nv_bfloat16* __restrict__ out,
                                                             const int32_t* __restrict__ cu, int B, int T, int H,
                                                             float scale, int window, const float* __restrict__ alibi) {
  pdl_sync();  // programmatic dependent launch: see common.cuh
  constexpr int E = HD / 32;
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int h = blockIdx.y;
  const int lane = threadIdx.x & 31;
  if (t >= T) return;
  // sequence containing token t: largest b with cu[b] <= t
  int lo = 0, hi = B;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(cu + mid) <= t) lo = mid; else hi = mid;
  }
  const int seq0 = __ldg(cu + lo);
  const int d = H * HD;
  const size_t ld = 3 * static_cast<size_t>(d);
  float q[E], o[E];
#pragma unroll
  for (int e = 0; e < E; ++e) {
    q[e] = __bfloat162float(qkv[t * ld + h * HD + lane * E + e]);
    o[e] = 0.f;
  }
  int k_lo = seq0;
  if (window > 0) k_lo = max(seq0, t - window + 1);
  float m = -INFINITY, l = 0.f;
  for (int kt = k_lo; kt <= t; ++kt) {
    float s = 0.f;
#pragma unroll
    for (int e = 0; e < E; ++e) s += q[e] * __bfloat162float(qkv[kt * ld + d + h * HD + lane * E + e]);
    s = warp_sum(s) * scale;
    if (alibi != nullptr) s += __ldg(alibi + h) * static_cast<float>(kt - seq0);
    const float mn = fmaxf(m, s);
    const float a = expf(m - mn), p = expf(s - mn);
    l = l * a + p;
#pragma unroll
    for (int e = 0; e < E; ++e)
      o[e] = o[e] * a + p * __bfloat162float(qkv[kt * ld + 2 * d + h * HD + lane * E + e]);
    m = mn;
  }
#pragma unroll
  for (int e = 0; e < E; ++e)
    out[static_cast<size_t>(t) * d + h * HD + lane * E + e] = __float2bfloat16_rn(o[e] / l);
}

template <int HD>
static int launch_attention_simt(const void* qkv, void* out, const int32_t* cu, int B, int T, int H, float scale,
                                 int window, const float* alibi, cudaStream_t stream) {
  dim3 grid((T + 7) / 8, H);
  LaunchScope _ls(kCatAttention, stream);
  SGPT_CHECK_CUDA(launch_kernel(attention_simt_kernel<HD>, grid, dim3(256), 0, stream,
                                static_cast<const __nv_bfloat16*>(qkv), static_cast<__nv_bfloat16*>(out), cu, B, T, H,
                                scale, window, alibi));
  return SGPT_OK;
}
}  // namespace sgpt

using namespace sgpt;

extern "C" int sgpt_attention(const void* qkv, void* out, const int32_t* cu_seqlens, int B, int T, int H, int hd,
                              float scale, int window, int max_seqlen, const float* alibi_slopes, int impl,
                              sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(B >= 0 && T >= 0 && H > 0, "sgpt_attention: bad sizes B=%d T=%d H=%d", B, T, H);
  SGPT_REQUIRE(hd == 64 || hd == 128 || hd == 256, "sgpt_attention: head_dim %d not in {64,128,256}", hd);
  SGPT_REQUIRE(scale > 0.f, "sgpt_attention: scale must be positive");
  SGPT_REQUIRE(window >= 0, "sgpt_attention: window must be >= 0");
  SGPT_REQUIRE(max_seqlen > 0 || T == 0, "sgpt_attention: max_seqlen must be positive");
  if (B == 0 || T == 0) return SGPT_OK;
  if (impl == 0 || impl == 2) {
    SGPT_REQUIRE(H <= 65535 && B <= 65535 && (max_seqlen + kAttnQ - 1) / kAttnQ <= 65535,
                 "sgpt_attention: grid limits exceeded (B=%d H=%d max_seqlen=%d)", B, H, max_seqlen);
    switch (hd) {
      case 64: return launch_attention_mma<64>(qkv, out, cu_seqlens, B, H, scale, window, max_seqlen, alibi_slopes, stream);
      case 128: return launch_attention_mma<128>(qkv, out, cu_seqlens, B, H, scale, window, max_seqlen, alibi_slopes, stream);
      default: return launch_attention_mma<256>(qkv, out, cu_seqlens, B, H, scale, window, max_seqlen, alibi_slopes, stream);
    }
  } else if (impl == 1) {
    switch (hd) {
      case 64: return launch_attention_simt<64>(qkv, out, cu_seqlens, B, T, H, scale, window, alibi_slopes, stream);
      case 128: return launch_attention_simt<128>(qkv, out, cu_seqlens, B, T, H, scale, window, alibi_slopes, stream);
      default: return launch_attention_simt<256>(qkv, out, cu_seqlens, B, T, H, scale, window, alibi_slopes, stream);
    }
  }
  set_error("sgpt_attention: unknown impl %d", impl);
  return SGPT_ERR_INVALID;
}
