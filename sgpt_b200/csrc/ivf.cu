// IVF search over a list-ordered corpus (include/sgpt_b200.h sgpt_ivf_search): per query, the exact top-k of the documents
// in its probed lists, with the scores and tie rule of the exact search.
//
// Per block of up to kIvfBlock queries, without a host synchronisation:
//   count    one thread per (query, probe) pair: the pair's candidate count is the clamped length of its list (0 for a
//            skipped probe or an empty list); pairs with a non-empty list are counted per list (histogram).
//   offsets  one CTA: exclusive scans over the lists give every list its first pair row and its first work unit; the
//            unit total stays in device memory.
//   gather   one warp per pair: a row of its list's pair segment (the slot inside the segment comes from an atomic
//            counter; which pairs share a tile changes no score), the query row and scale copied there and the pair's
//            (candidate list, list start) recorded — A of the scan is then contiguous rows that TMA loads as it is.
//   units    one warp per list: (block of <= 128 pair rows) x (256-document tile) work units, tile-major, so that the pair
//            blocks of one tile run back to back on neighbouring CTAs and share the tile in L2.
//   scan     the filter GEMM's mainloop over the unit table (gemm.cuh kUnits + EpiIvfRows): (score, global id) of every
//            probed document into its pair's candidate list, positions the shared or the query's own bitmap excludes
//            as empty slots (sgpt_ivf_search_masked; sgpt_ivf_search is its pitch-0 case).
//   select   launch_topk_select over G = nprobe packed lists per query (global ids) with per-pair counts.
// The range search (sgpt_ivf_range_search) runs the same front half (ivf_scan_block) and replaces the selection with the
// threshold compaction below.
// The list offsets and probes are device data: every read and write above is bounded by the clamped list ranges and
// the workspace layout, so inconsistent inputs give wrong results, never an out-of-bounds access.
#include "../../include/sgpt_b200.h"
#include "common.cuh"
#include "gemm_api.h"
#include "host_utils.h"
#include "topk.cuh"

using namespace sgpt;

namespace {

constexpr int kIvfBlock = 256;        // queries per block (blocks reuse the workspace)
constexpr int kPairRows = 128;        // pair rows per work unit (one M-tile)
constexpr int kThreads = 256;
constexpr int kScanThreads = 1024;

inline int64_t align256(int64_t x) { return (x + 255) & ~int64_t(255); }

// positions [b, e) of list l: the offsets clamped to [0, n] and the length to max_len
__device__ __forceinline__ void list_range(const int64_t* __restrict__ offsets, int l, int n, long long max_len, int& b,
                                           int& e) {
  long long lo = __ldg(reinterpret_cast<const long long*>(offsets) + l);
  long long hi = __ldg(reinterpret_cast<const long long*>(offsets) + l + 1);
  lo = lo < 0 ? 0 : (lo > n ? n : lo);
  hi = hi < lo ? lo : (hi > n ? n : hi);
  if (hi - lo > max_len) hi = lo + max_len;
  b = static_cast<int>(lo);
  e = static_cast<int>(hi);
}

__global__ void __launch_bounds__(kThreads) ivf_count_kernel(const int32_t* __restrict__ probes,
                                                             const int64_t* __restrict__ offsets, int nlist, int n,
                                                             long long max_len, int nb, int nprobe,
                                                             int* __restrict__ counts, int* __restrict__ hist) {
  pdl_sync();
  const long long i = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x;  // pair = q * nprobe + p
  if (i >= static_cast<long long>(nb) * nprobe) return;
  const int q = static_cast<int>(i / nprobe), p = static_cast<int>(i - static_cast<long long>(q) * nprobe);
  const int l = __ldg(probes + i);
  int len = 0;
  if (l >= 0 && l < nlist) {
    int b, e;
    list_range(offsets, l, n, max_len, b, e);
    len = e - b;
  }
  counts[static_cast<long long>(p) * nb + q] = len;  // the selection's counts[g * nq + q]
  if (len > 0) atomicAdd(hist + l, 1);
}

// exclusive scan of two values per thread over the CTA (kScanThreads); *tot = the CTA's sums
__device__ __forceinline__ int2 block_exclusive_scan2(int2 v, int2* s_warp, int2* tot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int2 incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int a = __shfl_up_sync(0xffffffffu, incl.x, o), b = __shfl_up_sync(0xffffffffu, incl.y, o);
    if (lane >= o) {
      incl.x += a;
      incl.y += b;
    }
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  int2 before = make_int2(0, 0), sum = make_int2(0, 0);
  for (int w = 0; w < kScanThreads / 32; ++w) {
    const int2 x = s_warp[w];
    if (w < warp) {
      before.x += x.x;
      before.y += x.y;
    }
    sum.x += x.x;
    sum.y += x.y;
  }
  __syncthreads();  // s_warp is reused by the next call
  *tot = sum;
  return make_int2(before.x + incl.x - v.x, before.y + incl.y - v.y);
}

// first pair row and first work unit of every list; *n_units = total units
__global__ void __launch_bounds__(kScanThreads) ivf_offsets_kernel(const int* __restrict__ hist,
                                                                   const int64_t* __restrict__ offsets, int nlist, int n,
                                                                   long long max_len, int* __restrict__ pair_off,
                                                                   int* __restrict__ unit_off, int* __restrict__ n_units) {
  __shared__ int2 s_warp[kScanThreads / 32];
  pdl_sync();
  int2 carry = make_int2(0, 0);
  for (int l0 = 0; l0 < nlist; l0 += kScanThreads) {
    const int l = l0 + static_cast<int>(threadIdx.x);
    int2 v = make_int2(0, 0);  // (pair rows, units) of list l
    if (l < nlist) {
      v.x = hist[l];
      if (v.x > 0) {
        int b, e;
        list_range(offsets, l, n, max_len, b, e);
        v.y = ((v.x + kPairRows - 1) / kPairRows) * ((e - b + kSimBN - 1) / kSimBN);
      }
    }
    int2 tot;
    const int2 ex = block_exclusive_scan2(v, s_warp, &tot);
    if (l < nlist) {
      pair_off[l] = carry.x + ex.x;
      unit_off[l] = carry.y + ex.y;
    }
    carry.x += tot.x;
    carry.y += tot.y;
  }
  if (threadIdx.x == 0) *n_units = carry.y;
}

// one warp per pair: its row of the A operand, the row's query scale and (candidate list, list start)
__global__ void __launch_bounds__(kThreads) ivf_gather_kernel(const int32_t* __restrict__ probes,
                                                              const int64_t* __restrict__ offsets, int nlist, int n,
                                                              long long max_len, int nb, int nprobe,
                                                              const uint8_t* __restrict__ Q, long long row_bytes,
                                                              const float* __restrict__ q_scale,
                                                              const int* __restrict__ pair_off, int* __restrict__ fill,
                                                              uint8_t* __restrict__ A, float* __restrict__ row_scale,
                                                              int2* __restrict__ row_info) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const long long i = (static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x) >> 5;  // warp-uniform
  const long long pairs = static_cast<long long>(nb) * nprobe;
  if (i >= pairs) return;
  const int l = __ldg(probes + i);
  if (l < 0 || l >= nlist) return;
  int b, e;
  list_range(offsets, l, n, max_len, b, e);
  if (e == b) return;
  long long r = 0;
  if (lane == 0) r = static_cast<long long>(pair_off[l]) + atomicAdd(fill + l, 1);
  r = __shfl_sync(0xffffffffu, r, 0);
  if (r < 0 || r >= pairs) return;
  const long long q = i / nprobe;
  const uint4* src = reinterpret_cast<const uint4*>(Q + q * row_bytes);
  uint4* dst = reinterpret_cast<uint4*>(A + r * row_bytes);
  for (long long v = lane; v < row_bytes / 16; v += 32) dst[v] = __ldg(src + v);
  if (lane == 0) {
    row_scale[r] = q_scale != nullptr ? __ldg(q_scale + q) : 1.f;
    row_info[r] = make_int2(static_cast<int>(i), b);
  }
}

// one warp per list: its units (m0, m_end, n0, n_end), tile-major
__global__ void __launch_bounds__(kThreads) ivf_units_kernel(const int* __restrict__ hist,
                                                             const int* __restrict__ pair_off,
                                                             const int* __restrict__ unit_off,
                                                             const int64_t* __restrict__ offsets, int nlist, int n,
                                                             long long max_len, long long rows, int max_units,
                                                             int4* __restrict__ units) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const long long l = (static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x) >> 5;
  if (l >= nlist) return;
  const int P = hist[l];
  if (P <= 0) return;
  int b, e;
  list_range(offsets, static_cast<int>(l), n, max_len, b, e);
  const int blocks = (P + kPairRows - 1) / kPairRows, tiles = (e - b + kSimBN - 1) / kSimBN;
  const long long u0 = unit_off[l], m_lo = pair_off[l];
  const long long m_hi = m_lo + P < rows ? m_lo + P : rows;
  for (long long j = lane; j < static_cast<long long>(blocks) * tiles; j += 32) {
    if (u0 + j < 0 || u0 + j >= max_units) break;
    const long long t = j / blocks, m0 = m_lo + kPairRows * (j - t * blocks);
    if (m0 < 0 || m0 >= m_hi) continue;  // (only with inconsistent counts)
    units[u0 + j] = make_int4(static_cast<int>(m0), static_cast<int>(m0 + kPairRows < m_hi ? m0 + kPairRows : m_hi),
                              static_cast<int>(b + kSimBN * t), e);
  }
}

// ---- range search: threshold compaction of the candidate lists (sgpt_ivf_range_search) ----------------------------
//   count    one warp per pair: its admitted slots among 0 .. len - 1 (len = the pair's clamped list length).
//   scan     one warp per query: exclusive scan of its nprobe pair counts in probe order (in place) and its total.
//   offsets  one CTA: the block's totals scanned onto the running total of earlier blocks -> out_counts, and each query's
//            output offset, or -1 when its entries would pass `cap`.
//   fill     one warp per pair of a fitting query: its admitted slots in slot order (ballot / popc), at the query's offset
//            plus the pair's.
// Slot order is ascending list position and pairs are in probe order, so the output order is fixed by the inputs alone:
// no atomics, and a second launch returns the same bits.

// slot e admitted: a real document (id >= 0) whose score (NaN as -1) is >= threshold
__device__ __forceinline__ bool range_admits(uint2 e, float threshold) {
  float s = __uint_as_float(e.x);
  s = (s != s) ? -1.f : s;
  return static_cast<int>(e.y) >= 0 && s >= threshold;
}

// the pair's candidate count as the count kernel wrote it, clamped to the list's entries
__device__ __forceinline__ int pair_len(const int* __restrict__ counts, long long i, int nb, int nprobe, long long Ls) {
  const int q = static_cast<int>(i / nprobe), p = static_cast<int>(i - static_cast<long long>(q) * nprobe);
  const int len = __ldg(counts + static_cast<long long>(p) * nb + q);
  return len < 0 ? 0 : (len > Ls ? static_cast<int>(Ls) : len);
}

__global__ void __launch_bounds__(kThreads) ivf_range_count_kernel(const uint2* __restrict__ cand,
                                                                   const int* __restrict__ counts, int nb, int nprobe,
                                                                   long long Ls, float threshold,
                                                                   long long* __restrict__ padm) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const long long i = (static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x) >> 5;  // warp-uniform
  if (i >= static_cast<long long>(nb) * nprobe) return;
  const int len = pair_len(counts, i, nb, nprobe, Ls);
  const uint2* list = cand + i * Ls;
  int c = 0;
  for (int s0 = 0; s0 < len; s0 += 32) {
    const bool a = s0 + lane < len && range_admits(__ldg(list + s0 + lane), threshold);
    c += __popc(__ballot_sync(0xffffffffu, a));
  }
  if (lane == 0) padm[i] = c;
}

// warp per query: padm[q * nprobe + p] <- exclusive scan in probe order; qcount[q] = the query's total
__global__ void __launch_bounds__(kThreads) ivf_range_scan_kernel(long long* __restrict__ padm, int nb, int nprobe,
                                                                  long long* __restrict__ qcount) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const long long q = (static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x) >> 5;  // warp-uniform
  if (q >= nb) return;
  long long* row = padm + q * nprobe;
  long long carry = 0;
  for (int p0 = 0; p0 < nprobe; p0 += 32) {
    const long long v = p0 + lane < nprobe ? row[p0 + lane] : 0ll;
    long long incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    if (p0 + lane < nprobe) row[p0 + lane] = carry + incl - v;
    carry += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (lane == 0) qcount[q] = carry;
}

// one CTA: out_counts of the block's queries, their output offsets (-1: past cap) and the running total
__global__ void __launch_bounds__(kIvfBlock) ivf_range_offsets_kernel(const long long* __restrict__ qcount, int nb,
                                                                      int first, long long cap, long long* running,
                                                                      int64_t* __restrict__ out_counts,
                                                                      long long* __restrict__ qoff) {
  __shared__ long long s_warp[kIvfBlock / 32];
  pdl_sync();
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;  // nb <= kIvfBlock
  const long long base = first ? 0ll : *running;
  const long long c = t < nb ? qcount[t] : 0ll;
  long long incl = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  long long before = 0, total = 0;
#pragma unroll
  for (int w = 0; w < kIvfBlock / 32; ++w) {
    before += w < warp ? s_warp[w] : 0ll;
    total += s_warp[w];
  }
  const long long off = base + before + incl - c;
  if (t < nb) {
    out_counts[t] = c;
    qoff[t] = off + c <= cap ? off : -1ll;
  }
  if (t == 0) *running = base + total;  // (every thread read *running before the barrier)
}

__global__ void __launch_bounds__(kThreads) ivf_range_fill_kernel(const uint2* __restrict__ cand,
                                                                  const int* __restrict__ counts, int nb, int nprobe,
                                                                  long long Ls, float threshold,
                                                                  const long long* __restrict__ padm,
                                                                  const long long* __restrict__ qcount,
                                                                  const long long* __restrict__ qoff,
                                                                  float* __restrict__ out_scores,
                                                                  int64_t* __restrict__ out_ids) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const long long i = (static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x) >> 5;  // warp-uniform
  if (i >= static_cast<long long>(nb) * nprobe) return;
  const long long q = i / nprobe;
  const long long base = qoff[q];
  if (base < 0) return;  // the query does not fit: its part of the output keeps its bits
  // the pair's entries: [padm[i], next pair's offset or the query's total) of the query's result
  const long long o = padm[i];
  const long long end = (i - q * nprobe + 1 < nprobe) ? padm[i + 1] : qcount[q];
  const int len = pair_len(counts, i, nb, nprobe, Ls);
  const uint2* list = cand + i * Ls;
  long long w = 0;  // entries written so far
  for (int s0 = 0; s0 < len; s0 += 32) {
    uint2 e = make_uint2(0u, 0xffffffffu);
    if (s0 + lane < len) e = __ldg(list + s0 + lane);
    const bool a = range_admits(e, threshold);
    const uint32_t bal = __ballot_sync(0xffffffffu, a);
    const long long at = o + w + __popc(bal & ((1u << lane) - 1u));
    if (a && at < end) {
      out_scores[base + at] = __uint_as_float(e.x);
      out_ids[base + at] = static_cast<int>(e.y);
    }
    w += __popc(bal);
  }
}

// Workspace of one query block (the same for every block of a call)
struct Layout {
  int nb;             // queries per block
  int64_t pairs;      // pair rows per block: nb x nprobe
  int64_t Ls;         // entries per candidate list: max_list_len rounded up to even, >= 2
  int64_t max_units;  // upper bound of the work units of a block
  int64_t cand, counts, rows, row_scale, row_info, units, hist, fill, pair_off, unit_off, n_units, total;  // offsets
  // the range search's compaction after `total`: per-pair admitted counts / offsets (int64 [pairs]), per-query totals
  // and output offsets (int64 [nb] each) and the running output offset carried across blocks (int64)
  int64_t padm, qcount, qoff, running, range_total;
};

Layout make_layout(int nq, int nlist, int nprobe, int64_t max_list_len, int D, int elem_bytes) {
  Layout w{};
  w.nb = nq < kIvfBlock ? (nq > 0 ? nq : 1) : kIvfBlock;
  w.pairs = static_cast<int64_t>(w.nb) * nprobe;
  w.Ls = max_list_len < 2 ? 2 : (max_list_len + 1) & ~int64_t(1);
  // sum over lists of ceil(P_l / 128) <= (lists with a pair) + pairs / 128, and every list has at most ceil(L / 256) tiles
  const int64_t lists_hit = nlist < w.pairs ? nlist : w.pairs;
  int64_t blocks = lists_hit + w.pairs / kPairRows;
  if (blocks > w.pairs) blocks = w.pairs;
  w.max_units = blocks * ((max_list_len + kSimBN - 1) / kSimBN);
  int64_t o = 0;
  auto take = [&](int64_t bytes) {
    const int64_t at = o;
    o += align256(bytes);
    return at;
  };
  w.cand = take(w.pairs * w.Ls * 8);
  w.counts = take(w.pairs * 4);
  w.rows = take(w.pairs * D * elem_bytes);
  w.row_scale = take(w.pairs * 4);
  w.row_info = take(w.pairs * 8);
  w.units = take(w.max_units * 16);
  w.hist = take(static_cast<int64_t>(nlist) * 4);
  w.fill = take(static_cast<int64_t>(nlist) * 4);
  w.pair_off = take(static_cast<int64_t>(nlist) * 4);
  w.unit_off = take(static_cast<int64_t>(nlist) * 4);
  w.n_units = take(4);
  w.total = o;
  w.padm = take(w.pairs * 8);
  w.qcount = take(static_cast<int64_t>(w.nb) * 8);
  w.qoff = take(static_cast<int64_t>(w.nb) * 8);
  w.running = take(8);
  w.range_total = o;
  return w;
}

bool dtype_known(int dtype) { return dtype == SGPT_DTYPE_BF16 || dtype == SGPT_DTYPE_I8; }

// the size checks shared by the workspace query and the search (no CUDA call)
int check_sizes(const char* fn, int dtype, int nq, int nlist, int nprobe, int64_t max_list_len, int D) {
  SGPT_REQUIRE(dtype_known(dtype), "%s: unknown shard dtype %d", fn, dtype);
  SGPT_REQUIRE(nq >= 0, "%s: bad query count nq=%d", fn, nq);
  if (dtype == SGPT_DTYPE_I8)
    SGPT_REQUIRE(D > 0 && D % 16 == 0 && D <= kMaxDimI8, "%s: int8 D=%d must be a positive multiple of 16, at most %d", fn,
                 D, kMaxDimI8);
  else
    SGPT_REQUIRE(D > 0 && D % 8 == 0, "%s: D=%d must be a positive multiple of 8", fn, D);
  SGPT_REQUIRE(nlist >= 1, "%s: nlist=%d must be positive", fn, nlist);
  SGPT_REQUIRE(nprobe >= 1 && nprobe <= nlist, "%s: nprobe=%d outside [1, nlist=%d]", fn, nprobe, nlist);
  SGPT_REQUIRE(max_list_len >= 0 && max_list_len < (1ll << 31), "%s: max_list_len=%lld outside [0, 2^31)", fn,
               (long long)max_list_len);
  // the selection ranks nprobe lists of max_list_len entries (each padded to 32) in one 2^32-entry space
  const int64_t Ls = max_list_len < 2 ? 2 : (max_list_len + 1) & ~int64_t(1);
  SGPT_REQUIRE(static_cast<int64_t>(nprobe) * ((Ls + 31) & ~int64_t(31)) < (1ll << 32),
               "%s: nprobe=%d lists of max_list_len=%lld entries exceed the 2^32-entry selection space", fn, nprobe,
               (long long)max_list_len);
  const Layout w = make_layout(nq, nlist, nprobe, max_list_len, D, dtype == SGPT_DTYPE_I8 ? 1 : 2);
  SGPT_REQUIRE(w.pairs < (1ll << 31) && w.max_units < (1ll << 31),
               "%s: %lld (query, probe) pairs per block of %d queries need %lld work units, more than 2^31", fn,
               (long long)w.pairs, w.nb, (long long)w.max_units);
  return SGPT_OK;
}

}  // namespace

extern "C" int64_t sgpt_ivf_search_workspace_bytes(int dtype, int nq, int nlist, int nprobe, int64_t max_list_len, int D) {
  if (check_sizes("sgpt_ivf_search_workspace_bytes", dtype, nq, nlist, nprobe, max_list_len, D) != SGPT_OK) return -1;
  return make_layout(nq, nlist, nprobe, max_list_len, D, dtype == SGPT_DTYPE_I8 ? 1 : 2).total;
}

extern "C" int64_t sgpt_ivf_range_search_workspace_bytes(int dtype, int nq, int nlist, int nprobe, int64_t max_list_len,
                                                         int D) {
  if (check_sizes("sgpt_ivf_range_search_workspace_bytes", dtype, nq, nlist, nprobe, max_list_len, D) != SGPT_OK)
    return -1;
  return make_layout(nq, nlist, nprobe, max_list_len, D, dtype == SGPT_DTYPE_I8 ? 1 : 2).range_total;
}

namespace {

// the argument checks both operations make (no CUDA call); `fn` names the entry point called in error messages
int check_search_args(const char* fn, int dtype, const void* Q, const void* C, int nq, int64_t n, int D,
                      const int64_t* list_offsets, int nlist, int64_t max_list_len, const int32_t* doc_ids,
                      const int32_t* probes, int nprobe, const uint32_t* mask, int64_t mask_pitch) {
  if (check_sizes(fn, dtype, nq, nlist, nprobe, max_list_len, D) != SGPT_OK) return SGPT_ERR_INVALID;
  SGPT_REQUIRE(n >= 0 && n < (1ll << 31), "%s: corpus size n=%lld outside [0, 2^31)", fn, (long long)n);
  SGPT_REQUIRE(max_list_len <= n, "%s: max_list_len=%lld exceeds n=%lld", fn, (long long)max_list_len, (long long)n);
  SGPT_REQUIRE(Q != nullptr && C != nullptr && list_offsets != nullptr && doc_ids != nullptr && probes != nullptr,
               "%s: null input (Q, C, list_offsets, doc_ids and probes are required)", fn);
  SGPT_REQUIRE((reinterpret_cast<uintptr_t>(Q) & 15) == 0, "%s: Q must be 16-byte aligned", fn);
  return check_doc_mask(fn, n, DocMask{mask, mask_pitch});
}

// The front half of both operations for the query block q0 .. q0 + nb - 1: the pair counts (`counts` of the layout) and,
// after the scan, every probed document of every pair in the pair's candidate list.
int ivf_scan_block(const Layout& w, uint8_t* base, int s8, const void* Q, const void* C, const float* q_scale,
                   const float* c_scale, int64_t n, int D, const int64_t* list_offsets, int nlist,
                   int64_t max_list_len, const int32_t* doc_ids, const int32_t* probes, int nprobe,
                   const uint32_t* mask, int64_t mask_pitch, int q0, int nb, cudaStream_t stream) {
  const long long row_bytes = static_cast<long long>(D) * (s8 ? 1 : 2);
  uint2* cand = reinterpret_cast<uint2*>(base + w.cand);
  int* counts = reinterpret_cast<int*>(base + w.counts);
  uint8_t* rows = base + w.rows;
  float* row_scale = reinterpret_cast<float*>(base + w.row_scale);
  int2* row_info = reinterpret_cast<int2*>(base + w.row_info);
  int4* units = reinterpret_cast<int4*>(base + w.units);
  int* hist = reinterpret_cast<int*>(base + w.hist);
  int* pair_off = reinterpret_cast<int*>(base + w.pair_off);
  int* unit_off = reinterpret_cast<int*>(base + w.unit_off);
  int* n_units = reinterpret_cast<int*>(base + w.n_units);
  int* fill = reinterpret_cast<int*>(base + w.fill);
  const int N = static_cast<int>(n);
  const long long max_len = max_list_len;
  const long long pairs = static_cast<long long>(nb) * nprobe;
  const int32_t* pr = probes + static_cast<long long>(q0) * nprobe;
  // hist and fill are adjacent
  SGPT_CHECK_CUDA(cudaMemsetAsync(hist, 0, static_cast<size_t>(w.pair_off - w.hist), stream));
  {
    LaunchScope _ls(kCatMisc, stream);
    SGPT_CHECK_CUDA(launch_kernel(ivf_count_kernel, dim3(static_cast<unsigned>((pairs + kThreads - 1) / kThreads)),
                                  dim3(kThreads), 0, stream, pr, list_offsets, nlist, N, max_len, nb, nprobe, counts,
                                  hist));
  }
  if (n > 0 && w.max_units > 0) {
    {
      LaunchScope _ls(kCatMisc, stream);
      SGPT_CHECK_CUDA(launch_kernel(ivf_offsets_kernel, dim3(1), dim3(kScanThreads), 0, stream, hist, list_offsets,
                                    nlist, N, max_len, pair_off, unit_off, n_units));
    }
    {
      LaunchScope _ls(kCatMisc, stream);
      SGPT_CHECK_CUDA(launch_kernel(ivf_gather_kernel, dim3(static_cast<unsigned>((pairs * 32 + kThreads - 1) / kThreads)),
                                    dim3(kThreads), 0, stream, pr, list_offsets, nlist, N, max_len, nb, nprobe,
                                    static_cast<const uint8_t*>(Q) + static_cast<long long>(q0) * row_bytes, row_bytes,
                                    q_scale != nullptr ? q_scale + q0 : nullptr, pair_off, fill, rows, row_scale,
                                    row_info));
    }
    {
      LaunchScope _ls(kCatMisc, stream);
      SGPT_CHECK_CUDA(launch_kernel(ivf_units_kernel,
                                    dim3(static_cast<unsigned>((static_cast<long long>(nlist) * 32 + kThreads - 1) / kThreads)),
                                    dim3(kThreads), 0, stream, hist, pair_off, unit_off, list_offsets, nlist, N, max_len,
                                    pairs, static_cast<int>(w.max_units), units));
    }
    // per-query bitmaps: the block's queries start at query q0
    const uint32_t* block_mask = mask != nullptr ? mask + q0 * mask_pitch : nullptr;
    IvfRowsParams p{units, n_units, static_cast<int>(w.max_units), row_scale, c_scale, row_info, doc_ids, block_mask,
                    cand, static_cast<long long>(w.Ls)};
    const int rc = launch_ivf_scan(rows, static_cast<int>(pairs), C, N, D, p, mask_pitch, nprobe, s8, stream);
    if (rc != SGPT_OK) return rc;
  }
  return SGPT_OK;
}

// both search entry points: `fn` names the one called in error messages
int ivf_search(const char* fn, int dtype, const void* Q, const void* C, const float* q_scale, const float* c_scale, int nq,
               int64_t n, int D, const int64_t* list_offsets, int nlist, int64_t max_list_len, const int32_t* doc_ids,
               const int32_t* probes, int nprobe, int k, const uint32_t* mask, int64_t mask_pitch, float* out_scores,
               int64_t* out_ids, void* ws, int64_t ws_bytes, sgpt_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (check_search_args(fn, dtype, Q, C, nq, n, D, list_offsets, nlist, max_list_len, doc_ids, probes, nprobe, mask,
                        mask_pitch) != SGPT_OK)
    return SGPT_ERR_INVALID;
  SGPT_REQUIRE(k >= 1 && k <= 4096, "%s: k=%d outside [1, 4096]", fn, k);
  SGPT_REQUIRE(out_scores != nullptr && out_ids != nullptr, "%s: null output", fn);
  const bool s8 = dtype == SGPT_DTYPE_I8;
  const Layout w = make_layout(nq, nlist, nprobe, max_list_len, D, s8 ? 1 : 2);
  SGPT_REQUIRE(ws != nullptr && ws_bytes >= w.total, "%s: workspace too small (%lld < %lld bytes)", fn,
               (long long)ws_bytes, (long long)w.total);
  if (nq == 0) return SGPT_OK;
  uint8_t* base = static_cast<uint8_t*>(ws);
  for (int q0 = 0; q0 < nq; q0 += kIvfBlock) {
    const int nb = nq - q0 < kIvfBlock ? nq - q0 : kIvfBlock;
    int rc = ivf_scan_block(w, base, s8, Q, C, q_scale, c_scale, n, D, list_offsets, nlist, max_list_len, doc_ids,
                            probes, nprobe, mask, mask_pitch, q0, nb, stream);
    if (rc != SGPT_OK) return rc;
    TopkSrc src{};
    src.packed = reinterpret_cast<uint2*>(base + w.cand);
    src.packed_global = 1;
    src.counts = reinterpret_cast<int*>(base + w.counts);
    src.G = nprobe;
    src.nq = nb;
    src.L = w.Ls;
    src.stride_g = w.Ls;
    src.stride_q = static_cast<long long>(nprobe) * w.Ls;
    rc = launch_topk_select(src, nb, k, out_scores + static_cast<long long>(q0) * k,
                            out_ids + static_cast<long long>(q0) * k, stream);
    if (rc != SGPT_OK) return rc;
  }
  return SGPT_OK;
}

}  // namespace

extern "C" int sgpt_ivf_search(int dtype, const void* Q, const void* C, const float* q_scale, const float* c_scale, int nq,
                               int64_t n, int D, const int64_t* list_offsets, int nlist, int64_t max_list_len,
                               const int32_t* doc_ids, const int32_t* probes, int nprobe, int k, const uint32_t* mask,
                               float* out_scores, int64_t* out_ids, void* ws, int64_t ws_bytes, sgpt_stream_t stream) {
  return ivf_search("sgpt_ivf_search", dtype, Q, C, q_scale, c_scale, nq, n, D, list_offsets, nlist, max_list_len,
                    doc_ids, probes, nprobe, k, mask, 0, out_scores, out_ids, ws, ws_bytes, stream);
}

extern "C" int sgpt_ivf_search_masked(int dtype, const void* Q, const void* C, const float* q_scale,
                                      const float* c_scale, int nq, int64_t n, int D, const int64_t* list_offsets,
                                      int nlist, int64_t max_list_len, const int32_t* doc_ids, const int32_t* probes,
                                      int nprobe, int k, const uint32_t* mask, int64_t mask_pitch_words,
                                      float* out_scores, int64_t* out_ids, void* ws, int64_t ws_bytes,
                                      sgpt_stream_t stream) {
  return ivf_search("sgpt_ivf_search_masked", dtype, Q, C, q_scale, c_scale, nq, n, D, list_offsets, nlist,
                    max_list_len, doc_ids, probes, nprobe, k, mask, mask_pitch_words, out_scores, out_ids, ws, ws_bytes,
                    stream);
}

extern "C" int sgpt_ivf_range_search(int dtype, const void* Q, const void* C, const float* q_scale, const float* c_scale,
                                     int nq, int64_t n, int D, const int64_t* list_offsets, int nlist,
                                     int64_t max_list_len, const int32_t* doc_ids, const int32_t* probes, int nprobe,
                                     float threshold, const uint32_t* mask, int64_t mask_pitch_words,
                                     int64_t* out_counts, int64_t cap, float* out_scores, int64_t* out_ids, void* ws,
                                     int64_t ws_bytes, sgpt_stream_t stream_) {
  const char* fn = "sgpt_ivf_range_search";
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (check_search_args(fn, dtype, Q, C, nq, n, D, list_offsets, nlist, max_list_len, doc_ids, probes, nprobe, mask,
                        mask_pitch_words) != SGPT_OK)
    return SGPT_ERR_INVALID;
  SGPT_REQUIRE(threshold == threshold, "%s: threshold is NaN", fn);
  SGPT_REQUIRE(cap >= 0, "%s: cap=%lld is negative", fn, (long long)cap);
  SGPT_REQUIRE(out_counts != nullptr, "%s: null out_counts", fn);
  SGPT_REQUIRE(cap == 0 || (out_scores != nullptr && out_ids != nullptr), "%s: null out_scores / out_ids with cap=%lld",
               fn, (long long)cap);
  const bool s8 = dtype == SGPT_DTYPE_I8;
  const Layout w = make_layout(nq, nlist, nprobe, max_list_len, D, s8 ? 1 : 2);
  SGPT_REQUIRE(ws != nullptr && ws_bytes >= w.range_total, "%s: workspace too small (%lld < %lld bytes)", fn,
               (long long)ws_bytes, (long long)w.range_total);
  if (nq == 0) return SGPT_OK;
  uint8_t* base = static_cast<uint8_t*>(ws);
  const uint2* cand = reinterpret_cast<const uint2*>(base + w.cand);
  const int* counts = reinterpret_cast<const int*>(base + w.counts);
  long long* padm = reinterpret_cast<long long*>(base + w.padm);
  long long* qcount = reinterpret_cast<long long*>(base + w.qcount);
  long long* qoff = reinterpret_cast<long long*>(base + w.qoff);
  long long* running = reinterpret_cast<long long*>(base + w.running);
  const long long Ls = w.Ls;
  for (int q0 = 0; q0 < nq; q0 += kIvfBlock) {
    const int nb = nq - q0 < kIvfBlock ? nq - q0 : kIvfBlock;
    const int rc = ivf_scan_block(w, base, s8, Q, C, q_scale, c_scale, n, D, list_offsets, nlist, max_list_len,
                                  doc_ids, probes, nprobe, mask, mask_pitch_words, q0, nb, stream);
    if (rc != SGPT_OK) return rc;
    const long long pairs = static_cast<long long>(nb) * nprobe;
    const dim3 pair_grid(static_cast<unsigned>((pairs * 32 + kThreads - 1) / kThreads));
    LaunchScope _ls(kCatTopk, stream);
    SGPT_CHECK_CUDA(launch_kernel(ivf_range_count_kernel, pair_grid, dim3(kThreads), 0, stream, cand, counts, nb, nprobe,
                                  Ls, threshold, padm));
    SGPT_CHECK_CUDA(launch_kernel(ivf_range_scan_kernel, dim3(static_cast<unsigned>((nb * 32 + kThreads - 1) / kThreads)),
                                  dim3(kThreads), 0, stream, padm, nb, nprobe, qcount));
    SGPT_CHECK_CUDA(launch_kernel(ivf_range_offsets_kernel, dim3(1), dim3(kIvfBlock), 0, stream,
                                  static_cast<const long long*>(qcount), nb, q0 == 0 ? 1 : 0, (long long)cap, running,
                                  out_counts + q0, qoff));
    if (cap > 0)
      SGPT_CHECK_CUDA(launch_kernel(ivf_range_fill_kernel, pair_grid, dim3(kThreads), 0, stream, cand, counts, nb, nprobe,
                                    Ls, threshold, static_cast<const long long*>(padm),
                                    static_cast<const long long*>(qcount), static_cast<const long long*>(qoff),
                                    out_scores, out_ids));
  }
  return SGPT_OK;
}
