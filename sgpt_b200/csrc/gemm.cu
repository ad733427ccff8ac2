// Host launchers for the wgmma GEMM (gemm.cuh): nn.Linear with fused epilogues (F3/F5/F6), the query x corpus
// similarity (S1) and its threshold-filter variant used by the fused search (search.cu).
#include "gemm.cuh"

#include <stdlib.h>


#include "../../include/sgpt_b200.h"
#include "gemm_api.h"
#include "host_utils.h"

namespace sgpt {

// a, b, lda, ldb and K in TMA elements: bf16, int8, or bytes of packed bits (kB1)
template <int BN, class Epi, int CL = 1, Operand kOp = Operand::kBF16>
static int launch_gemm(const void* a, int64_t lda, const void* b, int64_t ldb, int M, int N, int K,
                       const typename Epi::Params& ep, cudaStream_t stream, int cat = kCatGemm,
                       TileMap tmap = TileMap()) {
  using Cfg = GemmCfg<BN, Epi::kStagingBytes>;
  // one 128-byte row segment per box row: 64 bf16, 128 int8 or 1024 bits
  constexpr bool kS8 = kOp != Operand::kBF16;
  auto make_map = kS8 ? make_tma_2d_u8 : make_tma_2d_bf16;
  const uint32_t box_k = kS8 ? 2 * kGemmBK : kGemmBK;
  CUtensorMap ta, tb;
  int rc = make_map(&ta, a, static_cast<uint64_t>(M), static_cast<uint64_t>(K), static_cast<uint64_t>(lda), kGemmBM,
                    box_k);
  if (rc != SGPT_OK) return rc;
  rc = make_map(&tb, b, static_cast<uint64_t>(N), static_cast<uint64_t>(K), static_cast<uint64_t>(ldb), BN, box_k);
  if (rc != SGPT_OK) return rc;
  auto kern = gemm_bf16_tn_kernel<BN, Epi, CL, kOp>;
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

// nn.Linear dispatch: gemm_linear_kernel, 128 x 128 tiles.  Tile rasterisation (gemm.cuh TileMap::band): banded
// M-fastest order once the weight matrix no longer fits in the H100's 50 MB L2 next to the activations.
// SGPT_GEMM_BAND=<g> forces a band height (0 = N fastest) for A/B measurements; read per call.
static int pick_band(int M, int N, int K, int w_elem_bytes = 2) {
  if (const char* e = getenv("SGPT_GEMM_BAND")) return atoi(e);
  const long long w_bytes = static_cast<long long>(w_elem_bytes) * N * K;
  const int m_tiles = (M + kGemmBM - 1) / kGemmBM;
  return (w_bytes >= (32ll << 20) && m_tiles >= 16) ? 8 : 0;
}

// kOp = kE4M3: x, w, ldx, ldw and K in bytes (e4m3 elements), UINT8 tensor maps with 128-element K boxes
template <class Op, Operand kOp = Operand::kBF16>
static int launch_linear(const void* x, int64_t ldx, const void* w, int64_t ldw, int M, int N, int K,
                         const typename Op::Params& p, cudaStream_t stream, int ksplit = 1) {
  constexpr bool kF8 = kOp == Operand::kE4M3;
  TileMap tm;
  tm.ksplit = ksplit;
  tm.band = pick_band(M, N, K, kF8 ? 1 : 2);
  auto make_map = kF8 ? make_tma_2d_u8 : make_tma_2d_bf16;
  const uint32_t box_k = kF8 ? 2 * kGemmBK : kGemmBK;  // one 128-byte row segment per box row
  CUtensorMap ta, tb;
  int rc = make_map(&ta, x, static_cast<uint64_t>(M), static_cast<uint64_t>(K), static_cast<uint64_t>(ldx), kGemmBM,
                    box_k);
  if (rc != SGPT_OK) return rc;
  // each CTA of a cluster loads one half of the weight tile's rows and multicasts it to both
  rc = make_map(&tb, w, static_cast<uint64_t>(N), static_cast<uint64_t>(K), static_cast<uint64_t>(ldw), LinearCfg::kBRows,
                box_k);
  if (rc != SGPT_OK) return rc;
  auto kern = gemm_linear_kernel<Op, kOp>;
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    SGPT_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, LinearCfg::kSmemBytes));
  }
  // The persistent grid is as many clusters as can be resident at once: GPC sizes can leave fewer than sm_count() / 2
  // pairs of SMs for two-CTA clusters.  Cached per device.
  static int max_clusters[64] = {};
  int dev = 0;
  SGPT_CHECK_CUDA(cudaGetDevice(&dev));
  SGPT_REQUIRE(dev >= 0 && dev < 64, "launch_linear: device %d out of range", dev);
  if (max_clusters[dev] == 0) {
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = kLinCluster;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(static_cast<unsigned>(kLinCluster * sm_count()));
    cfg.blockDim = dim3(kLinThreads);
    cfg.dynamicSmemBytes = LinearCfg::kSmemBytes;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    int n = 0;
    SGPT_CHECK_CUDA(cudaOccupancyMaxActiveClusters(&n, kern, &cfg));
    SGPT_REQUIRE(n > 0, "launch_linear: no %d-CTA cluster of the linear-layer GEMM fits on device %d", kLinCluster, dev);
    max_clusters[dev] = n;  // benign race: every thread writes the same value
  }
  const int m_pairs = ((M + kGemmBM - 1) / kGemmBM + kLinCluster - 1) / kLinCluster;
  const long long units = static_cast<long long>(m_pairs) * ((N + kLinBN - 1) / kLinBN) * ksplit;  // pair units
  if (units == 0) return SGPT_OK;
  const long long clusters = units < max_clusters[dev] ? units : max_clusters[dev];
  LaunchScope _ls(kCatGemm, stream);
  SGPT_CHECK_CUDA(launch_kernel_cluster(kern, dim3(static_cast<unsigned>(kLinCluster * clusters)), dim3(kLinThreads),
                                        LinearCfg::kSmemBytes, stream, kLinCluster, ta, tb, M, N, K, p, tm));
  return SGPT_OK;
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
template <class Epi, Operand kOp = Operand::kBF16>
static int launch_filter_gemm(const void* Q, const void* C, int nq, int n, int D, const typename Epi::Params& p,
                              cudaStream_t stream, TileMap tm) {
  const int K = kOp == Operand::kB1 ? D / 8 : D;  // TMA elements per row
  if (nq > kGemmBM) return launch_gemm<kSimBN, Epi, 2, kOp>(Q, K, C, K, nq, n, K, p, stream, kCatScores, tm);
  return launch_gemm<kSimBN, Epi, 1, kOp>(Q, K, C, K, nq, n, K, p, stream, kCatScores, tm);
}

int check_doc_mask(const char* fn, long long n, DocMask mask) {
  const long long words = (n + 31) / 32;
  SGPT_REQUIRE(mask.pitch >= 0, "%s: negative mask pitch %lld", fn, mask.pitch);
  SGPT_REQUIRE(mask.pitch == 0 || mask.bits != nullptr, "%s: mask pitch %lld without a mask", fn, mask.pitch);
  SGPT_REQUIRE(mask.pitch == 0 || mask.pitch >= words, "%s: mask pitch %lld words is below ceil(n / 32) = %lld", fn,
               mask.pitch, words);
  return SGPT_OK;
}

int shard_operand(const char* fn, int dtype, Operand* op) {
  SGPT_REQUIRE(dtype == SGPT_DTYPE_BF16 || dtype == SGPT_DTYPE_I8 || dtype == SGPT_DTYPE_B1, "%s: unknown shard dtype %d",
               fn, dtype);
  *op = dtype == SGPT_DTYPE_I8 ? Operand::kS8 : dtype == SGPT_DTYPE_B1 ? Operand::kB1 : Operand::kBF16;
  return SGPT_OK;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int check_operands(const char* fn, Operand op, const void* Q, const void* C, const float* q_scale, const float* c_scale,
                   int nq, int D) {
  switch (op) {
    case Operand::kS8:
      SGPT_REQUIRE(D > 0 && D % 16 == 0 && D <= kMaxDimI8, "%s: int8 D=%d must be a positive multiple of 16, at most %d",
                   fn, D, kMaxDimI8);
      return SGPT_OK;
    case Operand::kB1:
      SGPT_REQUIRE(D > 0 && D % 128 == 0 && D <= kMaxDimB1,
                   "%s: binary D=%d must be a positive multiple of 128, at most %d", fn, D, kMaxDimB1);
      if (nq == 0) return SGPT_OK;
      SGPT_REQUIRE(q_scale != nullptr && c_scale != nullptr, "%s: binary rows need their popcounts (q_scale, c_scale)", fn);
      SGPT_REQUIRE(aligned16(Q) && aligned16(C) && aligned16(c_scale),
                   "%s: binary Q, C and the document popcounts must be 16-byte aligned", fn);
      return SGPT_OK;
    default:
      SGPT_REQUIRE(D > 0 && D % 8 == 0, "%s: D=%d must be a positive multiple of 8", fn, D);
      return SGPT_OK;
  }
}

size_t operand_row_bytes(Operand op, int D) {
  return op == Operand::kS8 ? static_cast<size_t>(D) : op == Operand::kB1 ? static_cast<size_t>(D) / 8 : 2 * static_cast<size_t>(D);
}

// the masked epilogue only when a mask is given: unmasked searches run the unmasked instantiations
static int launch_filter_any(const void* Q, const void* C, int nq, int n, int D, const EpiFilterRows::Params& p,
                             DocMask mask, cudaStream_t stream, TileMap tm, Operand op) {
  FilterRowsParams pm = p;
  pm.mask = mask.bits;
  pm.mask_pitch = mask.pitch;
  const bool masked = mask.bits != nullptr;
  switch (op) {
    case Operand::kS8:
      if (!masked) return launch_filter_gemm<EpiFilterRows, Operand::kS8>(Q, C, nq, n, D, p, stream, tm);
      return launch_filter_gemm<EpiFilterRowsMasked, Operand::kS8>(Q, C, nq, n, D, pm, stream, tm);
    case Operand::kB1:
      if (!masked) return launch_filter_gemm<EpiFilterRowsB1, Operand::kB1>(Q, C, nq, n, D, p, stream, tm);
      return launch_filter_gemm<EpiFilterRowsB1Masked, Operand::kB1>(Q, C, nq, n, D, pm, stream, tm);
    default:
      if (!masked) return launch_filter_gemm<EpiFilterRows>(Q, C, nq, n, D, p, stream, tm);
      return launch_filter_gemm<EpiFilterRowsMasked>(Q, C, nq, n, D, pm, stream, tm);
  }
}

int launch_filter_candidates(const void* Q, const void* C, const float* q_scale, const float* c_scale,
                             const float* tau, const float* tau_hi, uint2* cand, int* counts, int* counts_back,
                             long long stride_q, int L, int group0, int nq, int n, int D, int tile_mode, int tile_stride,
                             DocMask mask, Operand op, cudaStream_t stream) {
  SGPT_REQUIRE(nq <= 2 * kGemmBM, "filter GEMM: at most %d queries per launch (got %d)", 2 * kGemmBM, nq);
  TileMap tm;
  tm.mode = tile_mode;
  tm.stride = tile_stride;
  const FilterGeometry g = filter_geometry(tm.count((n + kSimBN - 1) / kSimBN), nq);
  SGPT_REQUIRE(L >= g.L && (L % 2) == 0 && (stride_q % 2) == 0, "filter GEMM: candidate lists too small (L=%d < %d)", L,
               g.L);
  FilterRowsParams p{q_scale, c_scale, tau, tau_hi, cand, counts, counts_back, stride_q, L, group0, nq, nullptr, 0, 0,
                     nq > kGemmBM ? 1 : 0};
  return launch_filter_any(Q, C, nq, n, D, p, mask, stream, tm, op);
}

int launch_sample_maxima(const void* Q, const void* C, const float* q_scale, const float* c_scale, float* pool,
                         long long stride_p, int Lp, int nq, int n, int D, int tile_stride, DocMask mask, Operand op,
                         cudaStream_t stream) {
  SGPT_REQUIRE(nq <= 2 * kGemmBM, "sample GEMM: at most %d queries per launch (got %d)", 2 * kGemmBM, nq);
  TileMap tm;
  tm.mode = 1;
  tm.stride = tile_stride;
  const FilterGeometry g = filter_geometry(tm.count((n + kSimBN - 1) / kSimBN), nq);
  SGPT_REQUIRE(Lp >= g.L / 4 && (Lp % 8) == 0 && (stride_p % 8) == 0 && stride_p >= static_cast<long long>(g.groups) * Lp,
               "sample GEMM: maxima lists too small (Lp=%d < %d)", Lp, g.L / 4);
  FilterRowsParams p{q_scale, c_scale, nullptr, nullptr, nullptr, nullptr, nullptr, 0, 0, 0, nq, pool, stride_p, Lp,
                     nq > kGemmBM ? 1 : 0};
  return launch_filter_any(Q, C, nq, n, D, p, mask, stream, tm, op);
}

template <class Epi>
static int launch_ivf_units(const CUtensorMap& ta, const CUtensorMap& tb, int rows, int n, int D,
                            const typename Epi::Params& p, bool s8, cudaStream_t stream) {
  using Cfg = GemmCfg<kSimBN, Epi::kStagingBytes>;
  auto kern = s8 ? gemm_bf16_tn_kernel<kSimBN, Epi, 1, Operand::kS8, true>
                 : gemm_bf16_tn_kernel<kSimBN, Epi, 1, Operand::kBF16, true>;
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    SGPT_CHECK_CUDA(cudaFuncSetAttribute(gemm_bf16_tn_kernel<kSimBN, Epi, 1, Operand::kS8, true>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    SGPT_CHECK_CUDA(cudaFuncSetAttribute(gemm_bf16_tn_kernel<kSimBN, Epi, 1, Operand::kBF16, true>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
  }
  // the unit count is only known on the device: one persistent CTA per SM, at most one per possible unit
  const int ctas = p.max_units < sm_count() ? p.max_units : sm_count();
  LaunchScope _ls(kCatScores, stream);
  SGPT_CHECK_CUDA(launch_kernel(kern, dim3(static_cast<unsigned>(ctas)), dim3(kGemmThreads), Cfg::kSmemBytes, stream, ta,
                                tb, rows, n, D, p, TileMap()));
  return SGPT_OK;
}

int launch_ivf_scan(const void* A, int rows, const void* C, int n, int D, const IvfRowsParams& p, long long mask_pitch,
                    int nprobe, bool s8, cudaStream_t stream) {
  SGPT_REQUIRE(rows > 0 && n > 0 && p.max_units > 0, "IVF scan: empty launch (rows=%d n=%d units=%d)", rows, n,
               p.max_units);
  SGPT_REQUIRE(mask_pitch == 0 || (p.mask != nullptr && nprobe > 0), "IVF scan: per-query masks need a bitmap");
  auto make_map = s8 ? make_tma_2d_u8 : make_tma_2d_bf16;
  const uint32_t box_k = s8 ? 2 * kGemmBK : kGemmBK;
  CUtensorMap ta, tb;
  int rc = make_map(&ta, A, static_cast<uint64_t>(rows), static_cast<uint64_t>(D), static_cast<uint64_t>(D), kGemmBM,
                    box_k);
  if (rc != SGPT_OK) return rc;
  rc = make_map(&tb, C, static_cast<uint64_t>(n), static_cast<uint64_t>(D), static_cast<uint64_t>(D), kSimBN, box_k);
  if (rc != SGPT_OK) return rc;
  if (mask_pitch == 0) return launch_ivf_units<EpiIvfRows>(ta, tb, rows, n, D, p, s8, stream);
  IvfRowsMaskedParams pm;
  static_cast<IvfRowsParams&>(pm) = p;
  pm.mask_pitch = mask_pitch;
  pm.nprobe = nprobe;
  return launch_ivf_units<EpiIvfRowsMasked>(ta, tb, rows, n, D, pm, s8, stream);
}

int launch_scores(const void* Q, const void* C, const float* q_scale, const float* c_scale, float* scores, long long lds,
                  int nq, int n, int D, DocMask mask, Operand op, cudaStream_t stream) {
  if (nq == 0 || n == 0) return SGPT_OK;
  constexpr Operand kS8 = Operand::kS8, kB1 = Operand::kB1;
  if (op == kB1) {  // K in bytes of packed bits
    const int K = D / 8;
    if (mask.bits == nullptr) {
      EpiScoresB1::Params p{scores, q_scale, c_scale, lds, nullptr, 0};
      return launch_gemm<128, EpiScoresB1, 1, kB1>(Q, K, C, K, nq, n, K, p, stream, kCatScores);
    }
    EpiScoresB1Masked::Params p{scores, q_scale, c_scale, lds, mask.bits, mask.pitch};
    return launch_gemm<128, EpiScoresB1Masked, 1, kB1>(Q, K, C, K, nq, n, K, p, stream, kCatScores);
  }
  if (mask.bits == nullptr) {
    EpiScoresF32::Params p{scores, q_scale, c_scale, lds, nullptr, 0};
    // lanes = queries (A operand), columns = corpus rows (B operand, streamed once from HBM)
    if (op == kS8) return launch_gemm<128, EpiScoresF32, 1, kS8>(Q, D, C, D, nq, n, D, p, stream, kCatScores);
    return launch_gemm<128, EpiScoresF32>(Q, D, C, D, nq, n, D, p, stream, kCatScores);
  }
  EpiScoresF32Masked::Params p{scores, q_scale, c_scale, lds, mask.bits, mask.pitch};
  if (op == kS8) return launch_gemm<128, EpiScoresF32Masked, 1, kS8>(Q, D, C, D, nq, n, D, p, stream, kCatScores);
  return launch_gemm<128, EpiScoresF32Masked>(Q, D, C, D, nq, n, D, p, stream, kCatScores);
}

int launch_lm_logits(const void* X, const void* W, float* logits, long long lds, int M, int vocab, int d,
                     cudaStream_t stream) {
  if (M == 0) return SGPT_OK;
  EpiLogitsF32::Params p{logits, nullptr, nullptr, lds, nullptr, 0};
  return launch_gemm<128, EpiLogitsF32>(X, d, W, d, M, vocab, d, p, stream, kCatScores);
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
                           int64_t ldo, const void* resid, int M, int N, int K, int epilogue,
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
        OpTmaBiasActBF16<false>::Params p{om, bias};
        return launch_linear<OpTmaBiasActBF16<false>>(x, ldx, w, ldw, M, N, K, p, stream);
      }
      OpTmaBiasActBF16<true>::Params p{om, bias};
      return launch_linear<OpTmaBiasActBF16<true>>(x, ldx, w, ldw, M, N, K, p, stream);
    }
    case SGPT_EPI_RESID_BF16: {
      SGPT_REQUIRE(resid != nullptr && resid == out,
                   "sgpt_linear: SGPT_EPI_RESID_BF16 updates the bf16 residual stream in place (resid must alias out)");
      SGPT_REQUIRE(ldo % 8 == 0, "sgpt_linear: ldo must be a multiple of 8 for bf16 output");
      CUtensorMap om;
      int rc = make_tma_2d_bf16(&om, out, static_cast<uint64_t>(M), static_cast<uint64_t>(N),
                                static_cast<uint64_t>(ldo), 32, 64);
      if (rc != SGPT_OK) return rc;
      OpTmaResidAddBF16::Params p{om, bias};
      return launch_linear<OpTmaResidAddBF16>(x, ldx, w, ldw, M, N, K, p, stream, pick_ksplit(K));
    }
    case 100:  // profiling aid: gemm_linear_kernel without its global stores (the product kernel's mainloop and epilogue)
      return launch_linear<OpNoStoreBF16>(x, ldx, w, ldw, M, N, K, {0}, stream);
    case 101: {  // profiling aid: gemm_bf16_tn_kernel's mainloop, fp32 accumulator hand-over and read-back
      TileMap tm;
      tm.band = pick_band(M, N, K);
      return launch_gemm<128, EpiDebugNull<true>>(x, ldx, w, ldw, M, N, K, {0}, stream, kCatGemm, tm);
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
  OpTmaRotaryBF16::Params p{om, pos, reinterpret_cast<const float2*>(cos_sin), M, d_model, head_dim, rotary_dim, max_pos};
  return launch_linear<OpTmaRotaryBF16>(x, ldx, w_qkv, d_model, M, N, d_model, p, stream);
}

extern "C" int sgpt_scores(const void* Q, const void* C, const float* q_scale, const float* c_scale, float* scores,
                           int64_t lds, int nq, int64_t n, int D, sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(nq >= 0 && n >= 0 && D > 0 && D % 8 == 0, "sgpt_scores: bad sizes nq=%d n=%lld D=%d", nq,
               (long long)n, D);
  SGPT_REQUIRE(n < (1ll << 31), "sgpt_scores: shard too large for one launch (n=%lld)", (long long)n);
  SGPT_REQUIRE(lds >= n, "sgpt_scores: lds < n");
  return launch_scores(Q, C, q_scale, c_scale, scores, lds, nq, static_cast<int>(n), D, DocMask(), Operand::kBF16, stream);
}

extern "C" int sgpt_scores_i8(const void* Q, const void* C, const float* q_scale, const float* c_scale, float* scores,
                              int64_t lds, int nq, int64_t n, int D, sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(nq >= 0 && n >= 0, "sgpt_scores_i8: bad sizes nq=%d n=%lld", nq, (long long)n);
  SGPT_REQUIRE(D > 0 && D % 16 == 0 && D <= kMaxDimI8, "sgpt_scores_i8: D=%d must be a positive multiple of 16, at most %d",
               D, kMaxDimI8);
  SGPT_REQUIRE(n < (1ll << 31), "sgpt_scores_i8: shard too large for one launch (n=%lld)", (long long)n);
  SGPT_REQUIRE(lds >= n, "sgpt_scores_i8: lds < n");
  SGPT_REQUIRE(nq == 0 || n == 0 || scores != nullptr, "sgpt_scores_i8: null output");
  return launch_scores(Q, C, q_scale, c_scale, scores, lds, nq, static_cast<int>(n), D, DocMask(), Operand::kS8, stream);
}

// ---------------------------------------------------------------------------------------------------------------
// fp8 linear layers (include/sgpt_b200.h): e4m3 x e4m3 with fp32 accumulation, the bf16 epilogues behind
// OpDequantE4M3.  No split-K.
// ---------------------------------------------------------------------------------------------------------------
static int check_fp8_operands(const char* fn, const void* xq, int64_t ldx, const float* x_scale, const void* wq,
                              int64_t ldw, const float* w_scale, int M, int N, int K) {
  SGPT_REQUIRE(M >= 0 && N > 0 && K > 0, "%s: bad sizes M=%d N=%d K=%d", fn, M, N, K);
  SGPT_REQUIRE(K % 16 == 0 && ldx % 16 == 0 && ldw % 16 == 0,
               "%s: K, ldx and ldw must be multiples of 16 (e4m3 rows of 16-byte multiples)", fn);
  SGPT_REQUIRE(ldx >= K && ldw >= K, "%s: row pitch smaller than the row", fn);
  SGPT_REQUIRE(M == 0 || (xq != nullptr && wq != nullptr && x_scale != nullptr && w_scale != nullptr),
               "%s: null operand or scale", fn);
  return SGPT_OK;
}

extern "C" int sgpt_linear_fp8(const void* xq, int64_t ldx, const float* x_scale, const void* wq, int64_t ldw,
                               const float* w_scale, const float* bias, void* out, int64_t ldo, const void* resid, int M,
                               int N, int K, int epilogue, sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int rc0 = check_fp8_operands("sgpt_linear_fp8", xq, ldx, x_scale, wq, ldw, w_scale, M, N, K);
  if (rc0 != SGPT_OK) return rc0;
  SGPT_REQUIRE(ldo >= N && ldo % 8 == 0, "sgpt_linear_fp8: ldo must be >= N and a multiple of 8");
  SGPT_REQUIRE(epilogue == SGPT_EPI_BF16 || epilogue == SGPT_EPI_GELU_BF16 || epilogue == SGPT_EPI_RESID_BF16,
               "sgpt_linear_fp8: unknown epilogue %d", epilogue);
  SGPT_REQUIRE(epilogue != SGPT_EPI_RESID_BF16 || (resid != nullptr && resid == out),
               "sgpt_linear_fp8: SGPT_EPI_RESID_BF16 updates the bf16 residual stream in place (resid must alias out)");
  if (const char* e = getenv("SGPT_GEMM_SPLITK"))
    SGPT_REQUIRE(atoi(e) <= 1, "sgpt_linear_fp8: split-K is not supported for fp8 operands (SGPT_GEMM_SPLITK=%s)", e);
  if (M == 0) return SGPT_OK;
  CUtensorMap om;
  int rc = make_tma_2d_bf16(&om, out, static_cast<uint64_t>(M), static_cast<uint64_t>(N), static_cast<uint64_t>(ldo), 32,
                            64);
  if (rc != SGPT_OK) return rc;
  constexpr Operand kF8 = Operand::kE4M3;
  if (epilogue == SGPT_EPI_RESID_BF16) {
    using Op = OpDequantE4M3<OpTmaResidAddBF16>;
    Op::Params p{{om, bias}, x_scale, w_scale};
    return launch_linear<Op, kF8>(xq, ldx, wq, ldw, M, N, K, p, stream);
  }
  if (epilogue == SGPT_EPI_BF16) {
    using Op = OpDequantE4M3<OpTmaBiasActBF16<false>>;
    Op::Params p{{om, bias}, x_scale, w_scale};
    return launch_linear<Op, kF8>(xq, ldx, wq, ldw, M, N, K, p, stream);
  }
  using Op = OpDequantE4M3<OpTmaBiasActBF16<true>>;
  Op::Params p{{om, bias}, x_scale, w_scale};
  return launch_linear<Op, kF8>(xq, ldx, wq, ldw, M, N, K, p, stream);
}

extern "C" int sgpt_linear_qkv_rotary_fp8(const void* xq, int64_t ldx, const float* x_scale, const void* wq_qkv,
                                          const float* w_scale, void* qkv, const int32_t* pos, const float* cos_sin, int M,
                                          int d_model, int head_dim, int rotary_dim, int max_pos,
                                          sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int rc0 = check_fp8_operands("sgpt_linear_qkv_rotary_fp8", xq, ldx, x_scale, wq_qkv, d_model, w_scale, M,
                                     3 * d_model, d_model);
  if (rc0 != SGPT_OK) return rc0;
  SGPT_REQUIRE(head_dim > 0 && d_model % head_dim == 0 && head_dim % 8 == 0,
               "sgpt_linear_qkv_rotary_fp8: bad head_dim %d", head_dim);
  SGPT_REQUIRE(rotary_dim >= 0 && rotary_dim <= head_dim && rotary_dim % 8 == 0,
               "sgpt_linear_qkv_rotary_fp8: rotary_dim %d must be a multiple of 8 and <= head_dim", rotary_dim);
  SGPT_REQUIRE(pos != nullptr && cos_sin != nullptr && max_pos > 0, "sgpt_linear_qkv_rotary_fp8: pos / cos_sin missing");
  if (M == 0) return SGPT_OK;
  const int N = 3 * d_model;
  CUtensorMap om;
  int rc = make_tma_2d_bf16(&om, qkv, static_cast<uint64_t>(M), static_cast<uint64_t>(N), static_cast<uint64_t>(N), 32,
                            64);
  if (rc != SGPT_OK) return rc;
  using Op = OpDequantE4M3<OpTmaRotaryBF16>;
  Op::Params p{{om, pos, reinterpret_cast<const float2*>(cos_sin), M, d_model, head_dim, rotary_dim, max_pos}, x_scale,
               w_scale};
  return launch_linear<Op, Operand::kE4M3>(xq, ldx, wq_qkv, d_model, M, N, d_model, p, stream);
}
