// IVF-PQ search (include/sgpt_b200.h sgpt_pq_tables, sgpt_ivfpq_search, sgpt_rerank): product-quantized lists scanned
// from per-query lookup tables in shared memory, and the exact re-rank of a short candidate list against a stored shard.
//
// Per block of up to kPqBlock queries of sgpt_ivfpq_search, without a host synchronisation:
//   count    ivf.cu's count kernel (launch_ivf_counts): every pair's candidate count is its clamped list length.
//   scan     one CTA per work unit (query, slice of its probes, and with few pairs a group of each list's tiles): the
//            query's table is staged into shared memory once per
//            unit (m <= kWholeMaxM) or kChunkM subspaces at a time together with the codes (larger m), the codes of one
//            list tile (kTile documents) per step with cp.async.bulk on an mbarrier, double-buffered so that the next
//            step's copies overlap this step's lookups.  Thread = document: it sums its m table entries in subspace order
//            (its partial sum carries across the chunks of a tile) and writes (score bits, global id) of its position to
//            the pair's candidate list, the layout of ivf.cu, two slots per 16-byte store.
//   select   launch_ivf_select: launch_topk_select over G = nprobe packed lists per query (global ids).
// The list offsets and probes are device data: offsets are clamped (list_range) and skipped probes never read, so
// inconsistent inputs give wrong results, never an out-of-bounds access.
#include "../../include/sgpt_b200.h"
#include "common.cuh"
#include "host_utils.h"
#include "ivf.cuh"
#include "topk.cuh"

using namespace sgpt;

namespace {

constexpr int kPqBlock = 256;     // queries per block of sgpt_ivfpq_search (blocks reuse the workspace)
constexpr int kTile = 256;        // documents per staged code tile = threads of the scan CTA
constexpr int kWholeMaxM = 128;   // m up to this: the query's whole table (m KB) stays in shared memory for the unit
constexpr int kChunkM = 64;       // larger m: table and codes staged kChunkM subspaces per step, two buffers of each
constexpr int kThreads = 256;
constexpr int kBarBytes = 128;    // the three mbarriers, padded
constexpr int kMaxM = 4096;
constexpr int kMaxCandidates = 1 << 24;

inline int64_t align256(int64_t x) { return (x + 255) & ~int64_t(255); }

// Shared-memory pitch of a staged code row of `bytes` (a multiple of 16): an odd number of 16-byte units, so that the
// 16-byte code reads of 8 consecutive threads (one shared-memory wavefront) hit 8 distinct bank groups.
__host__ __device__ constexpr int code_pitch(int bytes) { return ((bytes / 16) & 1) ? bytes : bytes + 16; }

template <bool kWhole>
size_t scan_smem_bytes(int m) {
  const int mc = kWhole ? m : kChunkM;
  const size_t table = kWhole ? static_cast<size_t>(m) * 1024 : 2 * static_cast<size_t>(kChunkM) * 1024;
  return kBarBytes + 2 * static_cast<size_t>(kTile) * code_pitch(mc) + table;
}

// ---- tables ---------------------------------------------------------------------------------------------------------
// lut[q][j][c] = sum_t Q[q][j dsub + t] B[j][c][t], one thread per (q, j, c): an fp32 FMA chain from 0 in ascending t
__global__ void __launch_bounds__(kThreads) pq_lut_kernel(const float* __restrict__ Q, const float* __restrict__ cb,
                                                          int nq, int D, int m, float* __restrict__ lut) {
  pdl_sync();
  const long long i = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x;
  if (i >= static_cast<long long>(nq) * m * 256) return;
  const int c = static_cast<int>(i & 255);
  const long long qj = i >> 8;
  const int j = static_cast<int>(qj % m);
  const long long q = qj / m;
  const int dsub = D / m;
  const float* x = Q + q * D + static_cast<long long>(j) * dsub;
  const float* b = cb + (static_cast<long long>(j) * 256 + c) * dsub;
  float acc = 0.f;
  for (int t = 0; t < dsub; ++t) acc = fmaf(__ldg(x + t), __ldg(b + t), acc);
  lut[i] = acc;
}

// base[q][p] = sum_t Q[q][t] centroids[probes[q][p]][t], one thread per pair (FMA chain from 0 in ascending t); a skipped
// probe reads no centroid and gets 0.  Neighbouring threads read rows D * 4 bytes apart (uncoalesced, served by L1); a
// warp per 32 pairs staging 32-dimension chunks of the rows in shared memory keeps the chain but measured slower at the
// benchmark's sizes (DESIGN.md §4).
__global__ void __launch_bounds__(kThreads) pq_base_kernel(const float* __restrict__ Q, const float* __restrict__ cent,
                                                           const int32_t* __restrict__ probes, int nq, int D, int nlist,
                                                           int nprobe, float* __restrict__ base) {
  pdl_sync();
  const long long i = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x;
  if (i >= static_cast<long long>(nq) * nprobe) return;
  const int l = __ldg(probes + i);
  float acc = 0.f;
  if (l >= 0 && l < nlist) {
    const float* x = Q + (i / nprobe) * D;
    const float* c = cent + static_cast<long long>(l) * D;
    for (int t = 0; t < D; ++t) acc = fmaf(__ldg(x + t), __ldg(c + t), acc);
  }
  base[i] = acc;
}

// ---- scan -----------------------------------------------------------------------------------------------------------
struct ScanArgs {
  const float* lut;         // [nb][m][256] of the block's queries
  const float* base;        // [nb][nprobe]
  const uint8_t* codes;     // [n][m] in list order
  int n, m;
  const int64_t* offsets;   // [nlist + 1]
  int nlist;
  long long max_len;
  const int32_t* doc_ids;   // [n]
  const int32_t* probes;    // [nb][nprobe]
  int nprobe;
  const uint32_t* mask;     // shared bitmap of allowed positions or null
  uint2* cand;              // [nb * nprobe][Ls]
  long long Ls;
  int slice;                // probes per work unit
  int groups;               // tile groups per (query, probe slice): > 1 only with slice = 1 (few pairs, long lists)
  int group_tiles;          // tiles of a list per group: group g scans tiles [g group_tiles, (g + 1) group_tiles)
};

// one step of a unit: chunk c of tile t of the list [b, e) of probe p (p >= the unit's end: no step)
struct Step {
  int p, b, e, t, c;
};

template <bool kWhole>
__global__ void __launch_bounds__(kThreads, 1) ivfpq_scan_kernel(const ScanArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int units_per_q = (a.nprobe + a.slice - 1) / a.slice;
  const int u = static_cast<int>(blockIdx.x) / a.groups, grp = static_cast<int>(blockIdx.x) - u * a.groups;
  const int ql = u / units_per_q;
  const int p_lo = (u - ql * units_per_q) * a.slice;
  const int p_hi = min(a.nprobe, p_lo + a.slice);
  const int t_lo = grp * a.group_tiles, t_hi = t_lo + a.group_tiles;  // this unit's tiles of each list
  const int m = a.m;
  const int mc = kWhole ? m : kChunkM;  // subspaces per step (the last chunk may hold fewer)
  const int nc = kWhole ? 1 : (m + kChunkM - 1) / kChunkM;
  const int pitch = code_pitch(mc);
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem);  // [0], [1]: the two step buffers; [2]: the whole table
  uint8_t* codes_s = smem + kBarBytes;
  float* lut_s = reinterpret_cast<float*>(codes_s + 2 * kTile * pitch);
  if (tid == 0) {
    mbar_init(bar + 0, 1);
    mbar_init(bar + 1, 1);
    mbar_init(bar + 2, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();
  const float* lut_q = a.lut + static_cast<long long>(ql) * m * 256;
  const int32_t* probes_q = a.probes + static_cast<long long>(ql) * a.nprobe;

  auto seek = [&](Step& s) {  // first probed list at or after probe s.p that has a tile in [t_lo, t_hi)
    for (; s.p < p_hi; ++s.p) {
      const int l = __ldg(probes_q + s.p);
      if (l < 0 || l >= a.nlist) continue;
      list_range(a.offsets, l, a.n, a.max_len, s.b, s.e);
      if (static_cast<long long>(s.b) + static_cast<long long>(kTile) * t_lo < s.e) {
        s.t = t_lo;
        s.c = 0;
        return;
      }
    }
  };
  auto advance = [&](Step& s) {
    if (++s.c < nc) return;
    s.c = 0;
    ++s.t;
    if (s.t < t_hi && static_cast<long long>(s.b) + static_cast<long long>(kTile) * s.t < s.e) return;
    ++s.p;
    seek(s);
  };
  // warp 0 stages a step into buffer `buf`: one bulk copy per code row (rows of the chunk are not contiguous in global
  // memory, and the padded pitch needs a copy per row anyway) plus, chunked, the step's table chunk
  auto issue = [&](const Step& s, int buf) {
    if (warp != 0) return;
    const int pos0 = s.b + kTile * s.t;
    const int cnt = min(kTile, s.e - pos0);
    const int c0 = s.c * kChunkM;
    const int bytes = kWhole ? m : min(kChunkM, m - c0);
    if (lane == 0) mbar_expect_tx(bar + buf, static_cast<uint32_t>(cnt * bytes + (kWhole ? 0 : bytes * 1024)));
    __syncwarp();
    if (!kWhole && lane == 0)
      bulk_load_1d(lut_s + buf * kChunkM * 256, lut_q + static_cast<long long>(c0) * 256,
                   static_cast<uint32_t>(bytes * 1024), bar + buf);
    const uint8_t* src = a.codes + static_cast<long long>(pos0) * m + c0;
    uint8_t* dst = codes_s + buf * kTile * pitch;
    for (int r = lane; r < cnt; r += 32)
      bulk_load_1d(dst + r * pitch, src + static_cast<long long>(r) * m, static_cast<uint32_t>(bytes), bar + buf);
  };

  Step cur{p_lo, 0, 0, 0, 0};
  seek(cur);
  if (cur.p >= p_hi) return;  // nothing probed (no copy in flight)
  if (kWhole && tid == 0) {
    mbar_expect_tx(bar + 2, static_cast<uint32_t>(m * 1024));
    bulk_load_1d(lut_s, lut_q, static_cast<uint32_t>(m * 1024), bar + 2);
  }
  issue(cur, 0);
  uint32_t phase = 0;  // bit b: parity of buffer b's next completion
  float acc = 0.f;
  for (int s = 0; cur.p < p_hi; ++s) {
    Step nxt = cur;
    advance(nxt);
    const int buf = s & 1;
    if (nxt.p < p_hi) issue(nxt, buf ^ 1);  // buffer buf ^ 1 was released by the barrier that ended step s - 1
    if (kWhole && s == 0) mbar_wait(bar + 2, 0);
    mbar_wait(bar + buf, (phase >> buf) & 1u);
    phase ^= 1u << buf;
    const int pos0 = cur.b + kTile * cur.t;
    const int cnt = min(kTile, cur.e - pos0);
    const int c0 = cur.c * kChunkM;
    const int bytes = kWhole ? m : min(kChunkM, m - c0);
    if (cur.c == 0) acc = 0.f;
    if (tid < cnt) {
      const uint8_t* row = codes_s + buf * kTile * pitch + tid * pitch;
      const float* tab = kWhole ? lut_s : lut_s + buf * kChunkM * 256;
      // acc += lut[j][code[j]] for j ascending: plain fp32 adds in this order (no reassociation without fast-math)
#pragma unroll 1
      for (int u = 0; u < bytes; u += 16) {
        const uint4 v = *reinterpret_cast<const uint4*>(row + u);
        const float* tj = tab + u * 256;
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 16; ++i) acc += tj[i * 256 + ((w[i >> 2] >> (8 * (i & 3))) & 255u)];
      }
    }
    if (cur.c == nc - 1) {  // block-uniform: the tile's scores are complete
      const int pos = pos0 + tid;
      uint32_t sb = 0u, gid = 0xffffffffu;
      if (tid < cnt) {
        float x = acc + __ldg(a.base + static_cast<long long>(ql) * a.nprobe + cur.p);
        x = (x != x) ? -1.f : x;
        int g = __ldg(a.doc_ids + pos);
        if (a.mask != nullptr && !((__ldg(a.mask + (pos >> 5)) >> (pos & 31)) & 1u)) g = -1;
        sb = __float_as_uint(x);
        gid = static_cast<uint32_t>(g);
      }
      const uint32_t sb1 = __shfl_down_sync(0xffffffffu, sb, 1), gid1 = __shfl_down_sync(0xffffffffu, gid, 1);
      // slot of position pos = pos - b; the tile starts at an even slot and Ls is even, so even threads store 16 bytes
      uint2* dst = a.cand + (static_cast<long long>(ql) * a.nprobe + cur.p) * a.Ls + (pos0 - cur.b);
      if ((tid & 1) == 0 && tid < cnt) {
        if (tid + 1 < cnt) *reinterpret_cast<uint4*>(dst + tid) = make_uint4(sb, gid, sb1, gid1);
        else dst[tid] = make_uint2(sb, gid);
      }
    }
    __syncthreads();
    cur = nxt;
  }
}

// ---- re-rank --------------------------------------------------------------------------------------------------------
// one warp per (query, candidate): the exact score of the candidate's stored row, (score bits, id) or an empty slot
template <bool kS8>
__global__ void __launch_bounds__(kThreads) rerank_kernel(const uint8_t* __restrict__ Q, const uint8_t* __restrict__ C,
                                                          const float* __restrict__ q_scale,
                                                          const float* __restrict__ c_scale, int nq, int n, int D,
                                                          long long id_base, const int64_t* __restrict__ cand, int kc,
                                                          uint2* __restrict__ out) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const long long w = (static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x) >> 5;  // warp-uniform
  if (w >= static_cast<long long>(nq) * kc) return;
  const long long q = w / kc;
  const long long id = __ldg(reinterpret_cast<const long long*>(cand) + w);
  if (id < 0 || id < id_base || id >= id_base + n) {
    if (lane == 0) out[w] = make_uint2(__float_as_uint(-INFINITY), 0xffffffffu);
    return;
  }
  const long long row = id - id_base;
  const long long row_bytes = kS8 ? D : 2ll * D;
  const uint4* qp = reinterpret_cast<const uint4*>(Q + q * row_bytes);
  const uint4* cp = reinterpret_cast<const uint4*>(C + row * row_bytes);
  const int units = static_cast<int>(row_bytes / 16);
  float x;
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
    x = __int2float_rn(acc);
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
    x = acc;
  }
  // the filter epilogue's order: (acc * q_scale) * c_scale, NaN -> -1
  x = x * (q_scale != nullptr ? __ldg(q_scale + q) : 1.f) * (c_scale != nullptr ? __ldg(c_scale + row) : 1.f);
  x = (x != x) ? -1.f : x;
  if (lane == 0) out[w] = make_uint2(__float_as_uint(x), static_cast<uint32_t>(static_cast<int32_t>(id)));
}

// ---- argument checks (no CUDA call) ---------------------------------------------------------------------------------
bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// the size checks shared by the workspace query and the search; the wording of ivf.cu's
int check_pq_sizes(const char* fn, int nq, int nlist, int nprobe, int64_t max_list_len, int m) {
  SGPT_REQUIRE(nq >= 0, "%s: bad query count nq=%d", fn, nq);
  SGPT_REQUIRE(m >= 16 && m % 16 == 0 && m <= kMaxM, "%s: m=%d must be a positive multiple of 16, at most %d", fn, m,
               kMaxM);
  SGPT_REQUIRE(nlist >= 1, "%s: nlist=%d must be positive", fn, nlist);
  SGPT_REQUIRE(nprobe >= 1 && nprobe <= nlist, "%s: nprobe=%d outside [1, nlist=%d]", fn, nprobe, nlist);
  SGPT_REQUIRE(max_list_len >= 0 && max_list_len < (1ll << 31), "%s: max_list_len=%lld outside [0, 2^31)", fn,
               (long long)max_list_len);
  const int64_t Ls = ivf_list_stride(max_list_len);
  SGPT_REQUIRE(static_cast<int64_t>(nprobe) * ((Ls + 31) & ~int64_t(31)) < (1ll << 32),
               "%s: nprobe=%d lists of max_list_len=%lld entries exceed the 2^32-entry selection space", fn, nprobe,
               (long long)max_list_len);
  const int64_t nb = nq < kPqBlock ? (nq > 0 ? nq : 1) : kPqBlock;
  SGPT_REQUIRE(nb * nprobe < (1ll << 31), "%s: %lld (query, probe) pairs per block of %lld queries, more than 2^31", fn,
               (long long)(nb * nprobe), (long long)nb);
  return SGPT_OK;
}

// Workspace of one query block of sgpt_ivfpq_search (the same for every block of a call)
struct PqLayout {
  int nb;
  int64_t pairs, Ls;
  int64_t cand, counts, total;
};

PqLayout make_pq_layout(int nq, int nlist, int nprobe, int64_t max_list_len) {
  PqLayout w{};
  w.nb = nq < kPqBlock ? (nq > 0 ? nq : 1) : kPqBlock;
  w.pairs = static_cast<int64_t>(w.nb) * nprobe;
  w.Ls = ivf_list_stride(max_list_len);
  w.cand = 0;
  w.counts = align256(w.pairs * w.Ls * 8);
  w.total = w.counts + align256(w.pairs * 4);
  return w;
}

bool dtype_known(int dtype) { return dtype == SGPT_DTYPE_BF16 || dtype == SGPT_DTYPE_I8; }

int check_rerank_sizes(const char* fn, int nq, int64_t kc) {
  SGPT_REQUIRE(nq >= 0, "%s: bad query count nq=%d", fn, nq);
  SGPT_REQUIRE(kc >= 1 && kc <= kMaxCandidates, "%s: kc=%lld outside [1, %d]", fn, (long long)kc, kMaxCandidates);
  return SGPT_OK;
}

}  // namespace

extern "C" int sgpt_pq_tables(const float* Q, const float* codebooks, const float* centroids, const int32_t* probes,
                              int nq, int D, int m, int nlist, int nprobe, float* lut_out, float* base_out,
                              sgpt_stream_t stream_) {
  const char* fn = "sgpt_pq_tables";
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(nq >= 0, "%s: bad query count nq=%d", fn, nq);
  SGPT_REQUIRE(D > 0 && D % 8 == 0, "%s: D=%d must be a positive multiple of 8", fn, D);
  SGPT_REQUIRE(m >= 16 && m % 16 == 0 && m <= kMaxM, "%s: m=%d must be a positive multiple of 16, at most %d", fn, m,
               kMaxM);
  SGPT_REQUIRE(D % m == 0, "%s: D=%d is not a multiple of m=%d", fn, D, m);
  SGPT_REQUIRE(nlist >= 1, "%s: nlist=%d must be positive", fn, nlist);
  SGPT_REQUIRE(nprobe >= 1 && nprobe <= nlist, "%s: nprobe=%d outside [1, nlist=%d]", fn, nprobe, nlist);
  SGPT_REQUIRE(Q != nullptr && codebooks != nullptr && centroids != nullptr && probes != nullptr,
               "%s: null input (Q, codebooks, centroids and probes are required)", fn);
  SGPT_REQUIRE(lut_out != nullptr && base_out != nullptr, "%s: null output", fn);
  if (nq == 0) return SGPT_OK;
  const long long entries = static_cast<long long>(nq) * m * 256, pairs = static_cast<long long>(nq) * nprobe;
  LaunchScope _ls(kCatMisc, stream);
  SGPT_CHECK_CUDA(launch_kernel(pq_lut_kernel, dim3(static_cast<unsigned>((entries + kThreads - 1) / kThreads)),
                                dim3(kThreads), 0, stream, Q, codebooks, nq, D, m, lut_out));
  SGPT_CHECK_CUDA(launch_kernel(pq_base_kernel, dim3(static_cast<unsigned>((pairs + kThreads - 1) / kThreads)),
                                dim3(kThreads), 0, stream, Q, centroids, probes, nq, D, nlist, nprobe, base_out));
  return SGPT_OK;
}

extern "C" int64_t sgpt_ivfpq_search_workspace_bytes(int nq, int nlist, int nprobe, int64_t max_list_len, int m) {
  if (check_pq_sizes("sgpt_ivfpq_search_workspace_bytes", nq, nlist, nprobe, max_list_len, m) != SGPT_OK) return -1;
  return make_pq_layout(nq, nlist, nprobe, max_list_len).total;
}

extern "C" int sgpt_ivfpq_search(const float* lut, const float* base, const uint8_t* codes, int nq, int64_t n, int m,
                                 const int64_t* list_offsets, int nlist, int64_t max_list_len, const int32_t* doc_ids,
                                 const int32_t* probes, int nprobe, int k, const uint32_t* mask, float* out_scores,
                                 int64_t* out_ids, void* ws, int64_t ws_bytes, sgpt_stream_t stream_) {
  const char* fn = "sgpt_ivfpq_search";
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (check_pq_sizes(fn, nq, nlist, nprobe, max_list_len, m) != SGPT_OK) return SGPT_ERR_INVALID;
  SGPT_REQUIRE(n >= 0 && n < (1ll << 31), "%s: corpus size n=%lld outside [0, 2^31)", fn, (long long)n);
  SGPT_REQUIRE(max_list_len <= n, "%s: max_list_len=%lld exceeds n=%lld", fn, (long long)max_list_len, (long long)n);
  SGPT_REQUIRE(lut != nullptr && base != nullptr && codes != nullptr && list_offsets != nullptr && doc_ids != nullptr &&
                   probes != nullptr,
               "%s: null input (lut, base, codes, list_offsets, doc_ids and probes are required)", fn);
  SGPT_REQUIRE(aligned16(lut) && aligned16(codes), "%s: lut and codes must be 16-byte aligned", fn);
  SGPT_REQUIRE(k >= 1 && k <= 4096, "%s: k=%d outside [1, 4096]", fn, k);
  SGPT_REQUIRE(out_scores != nullptr && out_ids != nullptr, "%s: null output", fn);
  const PqLayout w = make_pq_layout(nq, nlist, nprobe, max_list_len);
  SGPT_REQUIRE(ws != nullptr && ws_bytes >= w.total, "%s: workspace too small (%lld < %lld bytes)", fn,
               (long long)ws_bytes, (long long)w.total);
  if (nq == 0) return SGPT_OK;
  const bool whole = m <= kWholeMaxM;
  const size_t smem = whole ? scan_smem_bytes<true>(m) : scan_smem_bytes<false>(m);
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    SGPT_CHECK_CUDA(cudaFuncSetAttribute(ivfpq_scan_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(scan_smem_bytes<true>(kWholeMaxM))));
    SGPT_CHECK_CUDA(cudaFuncSetAttribute(ivfpq_scan_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(scan_smem_bytes<false>(kWholeMaxM + 16))));
  }
  uint8_t* wsb = static_cast<uint8_t*>(ws);
  uint2* cand = reinterpret_cast<uint2*>(wsb + w.cand);
  int* counts = reinterpret_cast<int*>(wsb + w.counts);
  const int target_units = 2 * sm_count();
  for (int q0 = 0; q0 < nq; q0 += kPqBlock) {
    const int nb = nq - q0 < kPqBlock ? nq - q0 : kPqBlock;
    const int32_t* pr = probes + static_cast<long long>(q0) * nprobe;
    int rc = launch_ivf_counts(pr, list_offsets, nlist, static_cast<int>(n), max_list_len, nb, nprobe, counts, nullptr,
                               stream);
    if (rc != SGPT_OK) return rc;
    // Work units: enough to fill the GPU twice over, with as few table stagings as that allows.  Many pairs: several
    // probes per unit.  Fewer pairs than that target: one probe per unit, and each list's tiles split into groups
    // (sized by the longest list, as the lengths are device data), so a long list does not run on a single SM.
    const long long pairs = static_cast<long long>(nb) * nprobe;
    long long slice = (pairs + target_units - 1) / target_units;
    slice = slice < 1 ? 1 : (slice > nprobe ? nprobe : slice);
    const long long tiles_max = max_list_len > 0 ? (max_list_len + kTile - 1) / kTile : 1;
    long long groups = 1;
    if (slice == 1) {
      groups = (target_units + pairs - 1) / pairs;
      groups = groups > tiles_max ? tiles_max : groups;
    }
    const long long group_tiles = (tiles_max + groups - 1) / groups;
    groups = (tiles_max + group_tiles - 1) / group_tiles;
    const long long units = static_cast<long long>(nb) * ((nprobe + slice - 1) / slice) * groups;
    ScanArgs a{lut + static_cast<long long>(q0) * m * 256, base + static_cast<long long>(q0) * nprobe, codes,
               static_cast<int>(n), m, list_offsets, nlist, static_cast<long long>(max_list_len), doc_ids, pr, nprobe,
               mask, cand, static_cast<long long>(w.Ls), static_cast<int>(slice), static_cast<int>(groups),
               static_cast<int>(group_tiles)};
    {
      LaunchScope _ls(kCatScores, stream);
      if (whole)
        SGPT_CHECK_CUDA(launch_kernel(ivfpq_scan_kernel<true>, dim3(static_cast<unsigned>(units)), dim3(kThreads), smem,
                                      stream, a));
      else
        SGPT_CHECK_CUDA(launch_kernel(ivfpq_scan_kernel<false>, dim3(static_cast<unsigned>(units)), dim3(kThreads), smem,
                                      stream, a));
    }
    rc = launch_ivf_select(cand, counts, nb, nprobe, w.Ls, k, out_scores + static_cast<long long>(q0) * k,
                           out_ids + static_cast<long long>(q0) * k, stream);
    if (rc != SGPT_OK) return rc;
  }
  return SGPT_OK;
}

extern "C" int64_t sgpt_rerank_workspace_bytes(int nq, int64_t kc) {
  if (check_rerank_sizes("sgpt_rerank_workspace_bytes", nq, kc) != SGPT_OK) return -1;
  return align256(static_cast<int64_t>(nq > 0 ? nq : 1) * kc * 8);
}

extern "C" int sgpt_rerank(int dtype, const void* Q, const void* C, const float* q_scale, const float* c_scale, int nq,
                           int64_t n, int D, int64_t id_base, const int64_t* cand_ids, int64_t kc, int k,
                           float* out_scores, int64_t* out_ids, void* ws, int64_t ws_bytes, sgpt_stream_t stream_) {
  const char* fn = "sgpt_rerank";
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(dtype_known(dtype), "%s: unknown shard dtype %d", fn, dtype);
  if (check_rerank_sizes(fn, nq, kc) != SGPT_OK) return SGPT_ERR_INVALID;
  const bool s8 = dtype == SGPT_DTYPE_I8;
  if (s8)
    SGPT_REQUIRE(D > 0 && D % 16 == 0 && D <= 65536, "%s: int8 D=%d must be a positive multiple of 16, at most %d", fn,
                 D, 65536);
  else
    SGPT_REQUIRE(D > 0 && D % 8 == 0, "%s: D=%d must be a positive multiple of 8", fn, D);
  SGPT_REQUIRE(n >= 0 && n < (1ll << 31), "%s: corpus size n=%lld outside [0, 2^31)", fn, (long long)n);
  SGPT_REQUIRE(id_base >= 0 && id_base + n <= (1ll << 31), "%s: global ids id_base=%lld + n=%lld must fit in int32", fn,
               (long long)id_base, (long long)n);
  SGPT_REQUIRE(k >= 1 && k <= 4096, "%s: k=%d outside [1, 4096]", fn, k);
  SGPT_REQUIRE(Q != nullptr && C != nullptr && cand_ids != nullptr, "%s: null input (Q, C and cand_ids are required)",
               fn);
  SGPT_REQUIRE(aligned16(Q) && aligned16(C), "%s: Q and C must be 16-byte aligned", fn);
  SGPT_REQUIRE(out_scores != nullptr && out_ids != nullptr, "%s: null output", fn);
  const int64_t need = align256(static_cast<int64_t>(nq > 0 ? nq : 1) * kc * 8);
  SGPT_REQUIRE(ws != nullptr && ws_bytes >= need, "%s: workspace too small (%lld < %lld bytes)", fn, (long long)ws_bytes,
               (long long)need);
  if (nq == 0) return SGPT_OK;
  uint2* packed = static_cast<uint2*>(ws);
  const long long warps = static_cast<long long>(nq) * kc;
  const dim3 grid(static_cast<unsigned>((warps * 32 + kThreads - 1) / kThreads));
  {
    LaunchScope _ls(kCatScores, stream);
    if (s8)
      SGPT_CHECK_CUDA(launch_kernel(rerank_kernel<true>, grid, dim3(kThreads), 0, stream,
                                    static_cast<const uint8_t*>(Q), static_cast<const uint8_t*>(C), q_scale, c_scale, nq,
                                    static_cast<int>(n), D, static_cast<long long>(id_base), cand_ids,
                                    static_cast<int>(kc), packed));
    else
      SGPT_CHECK_CUDA(launch_kernel(rerank_kernel<false>, grid, dim3(kThreads), 0, stream,
                                    static_cast<const uint8_t*>(Q), static_cast<const uint8_t*>(C), q_scale, c_scale, nq,
                                    static_cast<int>(n), D, static_cast<long long>(id_base), cand_ids,
                                    static_cast<int>(kc), packed));
  }
  TopkSrc src{};
  src.packed = packed;
  src.packed_global = 1;
  src.G = 1;
  src.nq = nq;
  src.L = kc;
  src.stride_g = kc;
  src.stride_q = kc;
  return launch_topk_select(src, nq, k, out_scores, out_ids, stream);
}
