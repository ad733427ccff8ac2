// Continuation log-likelihood scoring on top of the encoder (SURVEY.md §8f row 4: the SGPT cross-encoder,
// crossencoder/beir/sgptce.py:150-262).  After the GPT forward pass, only the rows whose next-token distribution is
// needed (the positions that predict a continuation token) go through ln_f and the LM head:
//     logits[m, :] = LN_f(resid[rows[m], :]) @ W_lm^T (+ b_lm)          wgmma GEMM (gemm.cu: sgpt_scores)
//     logprob[m]   = logits[m, target[m]] - logsumexp(logits[m, :])     == F.log_softmax(...).gather(...)  (:221, :247)
// The [rows, vocab] fp32 logits live only in the caller's workspace, a chunk of rows at a time; the full
// [batch, seq, vocab] tensor of the reference (:221) is never formed.
#include <float.h>

#include "../../include/sgpt_b200.h"
#include "common.cuh"
#include "host_utils.h"

namespace sgpt {

// One CTA (256 threads) per row: pass 1 max (+ argmax, lowest index wins ties like torch.argmax), pass 2 sum of exp.
__global__ void __launch_bounds__(256) token_logprob_kernel(const float* __restrict__ logits, long long lds, int vocab,
                                                            const float* __restrict__ bias,
                                                            const int32_t* __restrict__ targets,
                                                            float* __restrict__ logprob, int32_t* __restrict__ greedy) {
  pdl_sync();  // programmatic dependent launch: see common.cuh
  __shared__ float s_val[8];
  __shared__ int s_idx[8];
  __shared__ float s_bcast;
  const int row = blockIdx.x;
  const float* z = logits + static_cast<size_t>(row) * lds;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float m = -FLT_MAX;
  int mi = 0x7fffffff;
  for (int v = threadIdx.x; v < vocab; v += 256) {
    const float x = z[v] + (bias != nullptr ? __ldg(bias + v) : 0.f);
    if (x > m) { m = x; mi = v; }  // strided ascending visit: the first maximum a thread meets has its lowest index
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o);
    const int oi = __shfl_xor_sync(0xffffffffu, mi, o);
    if (om > m || (om == m && oi < mi)) { m = om; mi = oi; }
  }
  if (lane == 0) { s_val[warp] = m; s_idx[warp] = mi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float bm = s_val[0];
    int bi = s_idx[0];
    for (int w = 1; w < 8; ++w)
      if (s_val[w] > bm || (s_val[w] == bm && s_idx[w] < bi)) { bm = s_val[w]; bi = s_idx[w]; }
    s_bcast = bm;
    if (greedy != nullptr) greedy[row] = bi;
  }
  __syncthreads();
  const float mx = s_bcast;
  float sum = 0.f;
  for (int v = threadIdx.x; v < vocab; v += 256) {
    const float x = z[v] + (bias != nullptr ? __ldg(bias + v) : 0.f);
    sum += expf(x - mx);
  }
  sum = warp_sum(sum);
  __syncthreads();  // s_val is reused
  if (lane == 0) s_val[warp] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += s_val[w];
    const int tgt = __ldg(targets + row);
    const float zt = z[tgt] + (bias != nullptr ? __ldg(bias + tgt) : 0.f);
    logprob[row] = (zt - mx) - logf(t);
  }
}

// out[r] = sum of x[offsets[r] .. offsets[r+1]) in index order (deterministic): float(logits.sum()), sgptce.py:250
__global__ void __launch_bounds__(128) segment_sum_kernel(const float* __restrict__ x, const int32_t* __restrict__ offsets,
                                                          int R, float* __restrict__ out) {
  pdl_sync();  // programmatic dependent launch: see common.cuh
  const int r = blockIdx.x * 128 + threadIdx.x;
  if (r >= R) return;
  float s = 0.f;
  for (int i = __ldg(offsets + r); i < __ldg(offsets + r + 1); ++i) s += x[i];
  out[r] = s;
}

}  // namespace sgpt

using namespace sgpt;

extern "C" int sgpt_token_logprobs(const float* logits, int64_t lds, int M, int vocab, const float* bias,
                                   const int32_t* targets, float* logprob, int32_t* greedy, sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(M >= 0 && vocab > 0 && lds >= vocab, "sgpt_token_logprobs: bad sizes M=%d vocab=%d lds=%lld", M, vocab,
               (long long)lds);
  SGPT_REQUIRE(logits != nullptr && targets != nullptr && logprob != nullptr, "sgpt_token_logprobs: null argument");
  if (M == 0) return SGPT_OK;
  LaunchScope _ls(kCatMisc, stream);
  SGPT_CHECK_CUDA(launch_kernel(token_logprob_kernel, dim3(M), dim3(256), 0, stream, logits,
                                static_cast<long long>(lds), vocab, bias, targets, logprob, greedy));
  return SGPT_OK;
}

extern "C" int sgpt_segment_sum(const float* x, const int32_t* offsets, int R, float* out, sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(R >= 0, "sgpt_segment_sum: negative size");
  SGPT_REQUIRE(R == 0 || (x != nullptr && offsets != nullptr && out != nullptr), "sgpt_segment_sum: null argument");
  if (R == 0) return SGPT_OK;
  LaunchScope _ls(kCatMisc, stream);
  SGPT_CHECK_CUDA(launch_kernel(segment_sum_kernel, dim3((R + 127) / 128), dim3(128), 0, stream, x, offsets, R, out));
  return SGPT_OK;
}
