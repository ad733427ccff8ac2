// Host launchers for the wgmma GEMM (gemm.cuh): nn.Linear with fused epilogues (F3/F5/F6), the query x corpus
// similarity (S1) and its threshold-filter variant used by the fused search (search.cu).
#include "gemm.cuh"

#include <stdlib.h>


#include "../../include/sgpt_b200.h"
#include "gemm_api.h"
#include "host_utils.h"

namespace sgpt {

template <int BN, class Epi, int CL = 1>
static int launch_gemm(const void* a, int64_t lda, const void* b, int64_t ldb, int M, int N, int K,
                       const typename Epi::Params& ep, cudaStream_t stream, int cat = kCatGemm,
                       TileMap tmap = TileMap()) {
  using Cfg = GemmCfg<BN, EpiStaging<Epi>::value>;
  CUtensorMap ta, tb;
  int rc = make_tma_2d_bf16(&ta, a, static_cast<uint64_t>(M), static_cast<uint64_t>(K), static_cast<uint64_t>(lda),
                            kGemmBM, kGemmBK);
  if (rc != SGPT_OK) return rc;
  rc = make_tma_2d_bf16(&tb, b, static_cast<uint64_t>(N), static_cast<uint64_t>(K), static_cast<uint64_t>(ldb), BN,
                        kGemmBK);
  if (rc != SGPT_OK) return rc;
  auto kern = gemm_bf16_tn_kernel<BN, Epi, CL>;
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    SGPT_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
  }
  const int m_tiles = ((M + kGemmBM - 1) / kGemmBM + CL - 1) / CL;
  const int n_tiles = tmap.count((N + BN - 1) / BN);
  // work units (CL CTAs each): tile groups x K slices
  const long long tiles = static_cast<long long>(m_tiles) * n_tiles * tmap.ksplit;
  if (tiles == 0) return SGPT_OK;
  long long units = sm_count() / CL;
  if (tiles < units) units = tiles;
  LaunchScope _ls(cat, stream);
  SGPT_CHECK_CUDA(launch_kernel(kern, dim3(static_cast<unsigned>(units * CL)), dim3(kGemmThreads), Cfg::kSmemBytes, stream,
                                ta, tb, M, N, K, ep, tmap));
  return SGPT_OK;
}

// nn.Linear dispatch: 128 x 128 tiles (the 128 x 128 fp32 accumulator the epilogue reads back from shared memory leaves room
// for four operand stages; 256-wide tiles would leave one).  Tile rasterisation (gemm.cuh TileMap::band): banded M-fastest
// order once the weight matrix no longer fits in the H100's 50 MB L2 next to the activations.  SGPT_GEMM_BAND=<g> forces a
// band height (0 = N fastest) for A/B measurements; read per call.
static int pick_band(int M, int N, int K) {
  if (const char* e = getenv("SGPT_GEMM_BAND")) return atoi(e);
  const long long w_bytes = 2ll * N * K;
  const int m_tiles = (M + kGemmBM - 1) / kGemmBM;
  return (w_bytes >= (32ll << 20) && m_tiles >= 16) ? 8 : 0;
}

template <class Epi>
static int launch_linear(const void* x, int64_t ldx, const void* w, int64_t ldw, int M, int N, int K,
                         const typename Epi::Params& p, cudaStream_t stream, int ksplit = 1) {
  TileMap tm;
  tm.ksplit = ksplit;
  tm.band = pick_band(M, N, K);
  return launch_gemm<128, Epi, 1>(x, ldx, w, ldw, M, N, K, p, stream, kCatGemm, tm);
}

// Split-K for the reduce-add (residual) epilogues: OFF unless SGPT_GEMM_SPLITK=2/3/4 asks for it (experiments, tests).
// S K-slices per tile give S x as many work units of 1/S the length, so the tail of the last wave shrinks, at the price
// of a second reduce-add per output element.  It is not free semantically: with S > 1 the order in which the slices'
// partial sums reach the bf16 residual stream varies from run to run, so the encoder is no longer bit-reproducible
// (tests/test_gpu_full_depth.py).  A slice is at least 16 k-blocks (1024 of K).
static int pick_ksplit(int K) {
  const char* env = getenv("SGPT_GEMM_SPLITK");  // read per call: the GPU tests flip it in-process
  const int forced = env != nullptr ? atoi(env) : -1;
  const int num_kb = (K + kGemmBK - 1) / kGemmBK;
  if (forced >= 2) return (forced <= 4 && num_kb / forced >= 16) ? forced : 1;
  return 1;
}

FilterGeometry filter_geometry(long long tiles, int nq) {
  // queries above one M-tile are scanned by two CTAs per work unit (256 rows): one group per (unit slot, column half)
  const long long units = nq > kGemmBM ? sm_count() / 2 : sm_count();
  const long long ctas = tiles < units ? (tiles > 0 ? tiles : 1) : units;
  const long long per_cta = (tiles + ctas - 1) / ctas;
  FilterGeometry g;
  g.groups = static_cast<int>(2 * ctas);
  g.L = static_cast<int>(per_cta * (kSimBN / 2));
  return g;
}

// nq <= 128: one CTA per work unit (M = 128).  128 < nq <= 256: two CTAs per work unit, each with 128 of the queries and
// the same corpus tile — the second read of the tile is an L2 hit, so one pass over the shard from HBM serves 256 queries.
template <class P>
static int launch_filter_gemm(const void* Q, const void* C, int nq, int n, int D, const P& p, cudaStream_t stream, TileMap tm) {
  if (nq > kGemmBM) return launch_gemm<kSimBN, EpiFilterRows, 2>(Q, D, C, D, nq, n, D, p, stream, kCatScores, tm);
  return launch_gemm<kSimBN, EpiFilterRows, 1>(Q, D, C, D, nq, n, D, p, stream, kCatScores, tm);
}

int launch_filter_candidates(const void* Q, const void* C, const float* q_scale, const float* c_scale,
                             const float* tau, const float* tau_hi, uint2* cand, int* counts, int* counts_back,
                             long long stride_q, int L, int group0, int nq, int n, int D, int tile_mode, int tile_stride,
                             cudaStream_t stream) {
  SGPT_REQUIRE(nq <= 2 * kGemmBM, "filter GEMM: at most %d queries per launch (got %d)", 2 * kGemmBM, nq);
  TileMap tm;
  tm.mode = tile_mode;
  tm.stride = tile_stride;
  const FilterGeometry g = filter_geometry(tm.count((n + kSimBN - 1) / kSimBN), nq);
  SGPT_REQUIRE(L >= g.L && (L % 2) == 0 && (stride_q % 2) == 0, "filter GEMM: candidate lists too small (L=%d < %d)", L,
               g.L);
  EpiFilterRows::Params p{q_scale, c_scale, tau, tau_hi, cand, counts, counts_back, stride_q, L, group0, nq, nullptr, 0, 0,
                          nq > kGemmBM ? 1 : 0};
  return launch_filter_gemm(Q, C, nq, n, D, p, stream, tm);
}

int launch_sample_maxima(const void* Q, const void* C, const float* q_scale, const float* c_scale, float* pool,
                         long long stride_p, int Lp, int nq, int n, int D, int tile_stride, cudaStream_t stream) {
  SGPT_REQUIRE(nq <= 2 * kGemmBM, "sample GEMM: at most %d queries per launch (got %d)", 2 * kGemmBM, nq);
  TileMap tm;
  tm.mode = 1;
  tm.stride = tile_stride;
  const FilterGeometry g = filter_geometry(tm.count((n + kSimBN - 1) / kSimBN), nq);
  SGPT_REQUIRE(Lp >= g.L / 4 && (Lp % 8) == 0 && (stride_p % 8) == 0 && stride_p >= static_cast<long long>(g.groups) * Lp,
               "sample GEMM: maxima lists too small (Lp=%d < %d)", Lp, g.L / 4);
  EpiFilterRows::Params p{q_scale, c_scale, nullptr, nullptr, nullptr, nullptr, nullptr, 0, 0, 0, nq, pool, stride_p, Lp,
                          nq > kGemmBM ? 1 : 0};
  return launch_filter_gemm(Q, C, nq, n, D, p, stream, tm);
}

}  // namespace sgpt

using namespace sgpt;

extern "C" int sgpt_profile_gemm_clock(double* sm_cycles, double* nanoseconds) {
  SGPT_REQUIRE(sm_cycles != nullptr && nanoseconds != nullptr, "sgpt_profile_gemm_clock: null output");
  unsigned long long h[2] = {0, 0}, zero[2] = {0, 0};
  SGPT_CHECK_CUDA(cudaDeviceSynchronize());
  SGPT_CHECK_CUDA(cudaMemcpyFromSymbol(h, g_gemm_clock, sizeof(h)));
  SGPT_CHECK_CUDA(cudaMemcpyToSymbol(g_gemm_clock, zero, sizeof(zero)));
  *sm_cycles = static_cast<double>(h[0]);
  *nanoseconds = static_cast<double>(h[1]);
  return SGPT_OK;
}

extern "C" int sgpt_linear(const void* x, int64_t ldx, const void* w, int64_t ldw, const float* bias, void* out,
                           int64_t ldo, const float* resid, int M, int N, int K, int epilogue,
                           sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(M >= 0 && N > 0 && K > 0, "sgpt_linear: bad sizes M=%d N=%d K=%d", M, N, K);
  SGPT_REQUIRE(K % 8 == 0 && ldx % 8 == 0 && ldw % 8 == 0, "sgpt_linear: K, ldx, ldw must be multiples of 8");
  SGPT_REQUIRE(ldx >= K && ldw >= K && ldo >= N, "sgpt_linear: row pitch smaller than the row");
  if (M == 0) return SGPT_OK;
  switch (epilogue) {
    case SGPT_EPI_BF16:
    case SGPT_EPI_GELU_BF16: {
      SGPT_REQUIRE(ldo % 8 == 0, "sgpt_linear: ldo must be a multiple of 8 for bf16 output");
      // output boxes of 32 rows x 64 bf16 (one 128-byte row segment per row), written by the epilogue through TMA
      CUtensorMap om;
      int rc = make_tma_2d_bf16(&om, out, static_cast<uint64_t>(M), static_cast<uint64_t>(N),
                                static_cast<uint64_t>(ldo), 32, 64);
      if (rc != SGPT_OK) return rc;
      if (epilogue == SGPT_EPI_BF16) {
        EpiBiasActBF16<false>::Params p{om, bias, out, static_cast<int>(ldo)};
        return launch_linear<EpiBiasActBF16<false>>(x, ldx, w, ldw, M, N, K, p, stream);
      }
      EpiBiasActBF16<true>::Params p{om, bias, out, static_cast<int>(ldo)};
      return launch_linear<EpiBiasActBF16<true>>(x, ldx, w, ldw, M, N, K, p, stream);
    }
    case SGPT_EPI_RESID_F32: {
      SGPT_REQUIRE(resid != nullptr, "sgpt_linear: SGPT_EPI_RESID_F32 needs resid");
      SGPT_REQUIRE(ldo % 4 == 0, "sgpt_linear: ldo must be a multiple of 4 for fp32 output");
      if (resid != static_cast<const float*>(out)) {
        // not in place: seed the output with the residual, the epilogue then adds acc + bias into it
        SGPT_CHECK_CUDA(cudaMemcpy2DAsync(out, static_cast<size_t>(ldo) * 4, resid, static_cast<size_t>(ldo) * 4,
                                          static_cast<size_t>(N) * 4, static_cast<size_t>(M),
                                          cudaMemcpyDeviceToDevice, stream));
      }
      CUtensorMap om;
      int rc = make_tma_2d_f32(&om, out, static_cast<uint64_t>(M), static_cast<uint64_t>(N),
                               static_cast<uint64_t>(ldo), 32, 32);
      if (rc != SGPT_OK) return rc;
      EpiResidualF32::Params p{om, bias, out, static_cast<int>(ldo)};
      return launch_linear<EpiResidualF32>(x, ldx, w, ldw, M, N, K, p, stream, pick_ksplit(K));
    }
    case SGPT_EPI_RESID_BF16: {
      SGPT_REQUIRE(resid != nullptr && static_cast<const void*>(resid) == out,
                   "sgpt_linear: SGPT_EPI_RESID_BF16 updates the bf16 residual stream in place (resid must alias out)");
      SGPT_REQUIRE(ldo % 8 == 0, "sgpt_linear: ldo must be a multiple of 8 for bf16 output");
      CUtensorMap om;
      int rc = make_tma_2d_bf16(&om, out, static_cast<uint64_t>(M), static_cast<uint64_t>(N),
                                static_cast<uint64_t>(ldo), 32, 64);
      if (rc != SGPT_OK) return rc;
      EpiResidualBF16::Params p{om, bias, out, static_cast<int>(ldo)};
      return launch_linear<EpiResidualBF16>(x, ldx, w, ldw, M, N, K, p, stream, pick_ksplit(K));
    }
    case 102:
    case 103:
    case 104:
    case 105: {  // profiling aids: bf16 epilogue without the TMA store (102) / without the smem-reuse wait (103)
      CUtensorMap om;
      int rc = make_tma_2d_bf16(&om, out, static_cast<uint64_t>(M), static_cast<uint64_t>(N),
                                static_cast<uint64_t>(ldo), 32, 64);
      if (rc != SGPT_OK) return rc;
      OpTmaBiasActBF16<false>::Params p{om, bias, out, static_cast<int>(ldo)};
      if (epilogue == 102) return launch_linear<EpiTma<OpTmaBiasActBF16<false>, 1>>(x, ldx, w, ldw, M, N, K, p, stream);
      if (epilogue == 105) return launch_linear<EpiTma<OpTmaBiasActBF16<false>, 4>>(x, ldx, w, ldw, M, N, K, p, stream);
      if (epilogue == 104) return launch_linear<EpiTma<OpTmaBiasActBF16<false>, 3>>(x, ldx, w, ldw, M, N, K, p, stream);
      return launch_linear<EpiTma<OpTmaBiasActBF16<false>, 2>>(x, ldx, w, ldw, M, N, K, p, stream);
    }
    case 100: {  // profiling aid: mainloop only
      EpiDebugNull<false>::Params p{0};
      return launch_linear<EpiDebugNull<false>>(x, ldx, w, ldw, M, N, K, p, stream);
    }
    case 101: {  // profiling aid: mainloop + accumulator loads
      EpiDebugNull<true>::Params p{0};
      return launch_linear<EpiDebugNull<true>>(x, ldx, w, ldw, M, N, K, p, stream);
    }
    default:
      set_error("sgpt_linear: unknown epilogue %d", epilogue);
      return SGPT_ERR_INVALID;
  }
}

extern "C" int sgpt_linear_qkv_rotary(const void* x, int64_t ldx, const void* w_qkv, void* qkv, const int32_t* pos,
                                      const float* cos_sin, int M, int d_model, int head_dim, int rotary_dim,
                                      int max_pos, sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(M >= 0 && d_model > 0 && d_model % 8 == 0 && ldx % 8 == 0 && ldx >= d_model,
               "sgpt_linear_qkv_rotary: bad sizes M=%d d=%d ldx=%lld", M, d_model, (long long)ldx);
  SGPT_REQUIRE(head_dim > 0 && d_model % head_dim == 0 && head_dim % 8 == 0, "sgpt_linear_qkv_rotary: bad head_dim %d",
               head_dim);
  SGPT_REQUIRE(rotary_dim >= 0 && rotary_dim <= head_dim && rotary_dim % 8 == 0,
               "sgpt_linear_qkv_rotary: rotary_dim %d must be a multiple of 8 and <= head_dim", rotary_dim);
  SGPT_REQUIRE(pos != nullptr && cos_sin != nullptr && max_pos > 0, "sgpt_linear_qkv_rotary: pos / cos_sin missing");
  if (M == 0) return SGPT_OK;
  const int N = 3 * d_model;
  CUtensorMap om;
  int rc = make_tma_2d_bf16(&om, qkv, static_cast<uint64_t>(M), static_cast<uint64_t>(N), static_cast<uint64_t>(N), 32,
                            64);
  if (rc != SGPT_OK) return rc;
  EpiRotaryBF16::Params p{om, pos, reinterpret_cast<const float2*>(cos_sin), M, d_model, head_dim, rotary_dim, max_pos,
                          qkv, N};
  return launch_linear<EpiRotaryBF16>(x, ldx, w_qkv, d_model, M, N, d_model, p, stream);
}

// F2+F3 / F2+F6 with the LayerNorm folded into the GEMM (gemm.cuh OpTmaLnBiasActBF16): x_bf16 is the bf16 copy of the
// residual stream, w the gamma-folded weight, bias / colsum the folded vectors, row_stats the partial sums.
extern "C" int sgpt_linear_lnfold(const void* x_bf16, int64_t ldx, const void* w_folded, int64_t ldw,
                                  const float* bias_folded, const float* colsum, const float* row_stats, int n_groups,
                                  float eps, void* out, int64_t ldo, int M, int N, int K, int gelu,
                                  sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(M >= 0 && N > 0 && K > 0, "sgpt_linear_lnfold: bad sizes M=%d N=%d K=%d", M, N, K);
  SGPT_REQUIRE(K % 8 == 0 && ldx % 8 == 0 && ldw % 8 == 0 && ldo % 8 == 0, "sgpt_linear_lnfold: K, ldx, ldw, ldo must be multiples of 8");
  SGPT_REQUIRE(ldx >= K && ldw >= K && ldo >= N, "sgpt_linear_lnfold: row pitch smaller than the row");
  SGPT_REQUIRE(bias_folded != nullptr && colsum != nullptr && row_stats != nullptr && n_groups > 0,
               "sgpt_linear_lnfold: folded bias / column sums / row statistics are required");
  SGPT_REQUIRE(N % 4 == 0, "sgpt_linear_lnfold: N must be a multiple of 4");
  if (M == 0) return SGPT_OK;
  CUtensorMap om;
  int rc = make_tma_2d_bf16(&om, out, static_cast<uint64_t>(M), static_cast<uint64_t>(N), static_cast<uint64_t>(ldo), 32, 64);
  if (rc != SGPT_OK) return rc;
  const float inv_d = 1.0f / static_cast<float>(K);
  if (gelu) {
    EpiLnBiasActBF16<true>::Params p{om, bias_folded, colsum, reinterpret_cast<const float2*>(row_stats), n_groups, inv_d, eps,
                                     out, static_cast<int>(ldo)};
    return launch_linear<EpiLnBiasActBF16<true>>(x_bf16, ldx, w_folded, ldw, M, N, K, p, stream);
  }
  EpiLnBiasActBF16<false>::Params p{om, bias_folded, colsum, reinterpret_cast<const float2*>(row_stats), n_groups, inv_d, eps,
                                    out, static_cast<int>(ldo)};
  return launch_linear<EpiLnBiasActBF16<false>>(x_bf16, ldx, w_folded, ldw, M, N, K, p, stream);
}

extern "C" int sgpt_linear_qkv_rotary_lnfold(const void* x_bf16, int64_t ldx, const void* w_folded,
                                             const float* bias_folded, const float* colsum, const float* row_stats,
                                             int n_groups, float eps, void* qkv, const int32_t* pos,
                                             const float* cos_sin, int M, int d_model, int head_dim, int rotary_dim,
                                             int max_pos, sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(M >= 0 && d_model > 0 && d_model % 8 == 0 && ldx % 8 == 0 && ldx >= d_model,
               "sgpt_linear_qkv_rotary_lnfold: bad sizes M=%d d=%d ldx=%lld", M, d_model, (long long)ldx);
  SGPT_REQUIRE(head_dim > 0 && d_model % head_dim == 0 && head_dim % 8 == 0, "sgpt_linear_qkv_rotary_lnfold: bad head_dim %d",
               head_dim);
  SGPT_REQUIRE(rotary_dim >= 0 && rotary_dim <= head_dim && rotary_dim % 8 == 0,
               "sgpt_linear_qkv_rotary_lnfold: rotary_dim %d must be a multiple of 8 and <= head_dim", rotary_dim);
  SGPT_REQUIRE(pos != nullptr && cos_sin != nullptr && max_pos > 0, "sgpt_linear_qkv_rotary_lnfold: pos / cos_sin missing");
  SGPT_REQUIRE(bias_folded != nullptr && colsum != nullptr && row_stats != nullptr && n_groups > 0,
               "sgpt_linear_qkv_rotary_lnfold: folded bias / column sums / row statistics are required");
  if (M == 0) return SGPT_OK;
  const int N = 3 * d_model;
  CUtensorMap om;
  int rc = make_tma_2d_bf16(&om, qkv, static_cast<uint64_t>(M), static_cast<uint64_t>(N), static_cast<uint64_t>(N), 32, 64);
  if (rc != SGPT_OK) return rc;
  EpiLnRotaryBF16::Params p{{om, pos, reinterpret_cast<const float2*>(cos_sin), M, d_model, head_dim, rotary_dim, max_pos, qkv, N},
                            bias_folded, colsum, reinterpret_cast<const float2*>(row_stats), n_groups,
                            1.0f / static_cast<float>(d_model), eps, qkv, N};
  return launch_linear<EpiLnRotaryBF16>(x_bf16, ldx, w_folded, d_model, M, N, d_model, p, stream);
}

// F5 / F6b with the statistics of the NEXT LayerNorm (gemm.cuh EpiResidLn): resid += x w^T + bias in place, plus the
// bf16 copy and the per-(row, 128-column group) partial sums of the new residual.
extern "C" int sgpt_linear_resid_ln(const void* x, int64_t ldx, const void* w, int64_t ldw, const float* bias,
                                    float* resid, void* xb_out, float* stats_out, int M, int N, int K,
                                    sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(M >= 0 && N > 0 && K > 0, "sgpt_linear_resid_ln: bad sizes M=%d N=%d K=%d", M, N, K);
  SGPT_REQUIRE(K % 8 == 0 && ldx % 8 == 0 && ldw % 8 == 0 && ldx >= K && ldw >= K, "sgpt_linear_resid_ln: bad pitches");
  SGPT_REQUIRE(N % 64 == 0, "sgpt_linear_resid_ln: N=%d must be a multiple of 64", N);
  SGPT_REQUIRE(resid != nullptr && xb_out != nullptr && stats_out != nullptr, "sgpt_linear_resid_ln: null output");
  if (M == 0) return SGPT_OK;
  EpiResidLn::Params p;
  int rc = make_tma_2d_f32(&p.resid_map, resid, static_cast<uint64_t>(M), static_cast<uint64_t>(N), static_cast<uint64_t>(N), 32, 32);
  if (rc != SGPT_OK) return rc;
  rc = make_tma_2d_bf16(&p.xb_map, xb_out, static_cast<uint64_t>(M), static_cast<uint64_t>(N), static_cast<uint64_t>(N), 32, 64);
  if (rc != SGPT_OK) return rc;
  p.bias = bias;
  p.stats = reinterpret_cast<float2*>(stats_out);
  p.P = (N + 127) / 128;
  {
    static const int l2pf = [] { const char* e = getenv("SGPT_RESID_L2_PREFETCH"); return (e != nullptr && e[0] == '0') ? 0 : 1; }();
    p.l2_prefetch = l2pf;
  }
  // 128-wide tiles and four epilogue warps: each warp owns exactly one 128-column statistics group
  return launch_gemm<128, EpiResidLn, 1>(x, ldx, w, ldw, M, N, K, p, stream);
}

extern "C" int sgpt_scores(const void* Q, const void* C, const float* q_scale, const float* c_scale, float* scores,
                           int64_t lds, int nq, int64_t n, int D, sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(nq >= 0 && n >= 0 && D > 0 && D % 8 == 0, "sgpt_scores: bad sizes nq=%d n=%lld D=%d", nq,
               (long long)n, D);
  SGPT_REQUIRE(n < (1ll << 31), "sgpt_scores: shard too large for one launch (n=%lld)", (long long)n);
  SGPT_REQUIRE(lds >= n, "sgpt_scores: lds < n");
  if (nq == 0 || n == 0) return SGPT_OK;
  EpiScoresF32::Params p{scores, q_scale, c_scale, static_cast<long long>(lds)};
  // lanes = queries (A operand), columns = corpus rows (B operand, streamed once from HBM)
  return launch_gemm<128, EpiScoresF32>(Q, D, C, D, nq, static_cast<int>(n), D, p, stream, kCatScores);
}
