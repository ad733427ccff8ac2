// Exact threshold (range) search over one corpus shard: every document whose score against a query is >= threshold, as a
// deterministic CSR result (ST/util.py:385-448 needs exactly this set; include/sgpt_b200.h sgpt_range_search).
//
//   filter   the search's pass-B GEMM (gemm.cuh EpiFilterRows) with tau[q] = threshold and no tau_hi: every admitted score
//            lands at the front of its (query, group) list, and a list can never overflow (sized for every score).
//   runs     one CTA per query.  Every 128-document half tile h belongs to exactly one group (g = 2 (tile % slots) +
//            h % 2, the persistent CTA of slot s visiting tiles s, s + slots, ... in increasing order), so the group's
//            list is ascending in document index and half tile h is one contiguous run of it, found by two binary
//            searches.  A block-wide scan over h gives every run its offset inside the query's result.
//   offsets  one CTA: the counts of the query block, their scan, and the running total of earlier query blocks (kept on
//            the device: no host synchronisation between blocks).  A query whose entries would pass `cap` is marked.
//   fill     one warp per run copies it to its place: output order = half tile order = ascending document index.
// No atomics anywhere, so a second launch returns the same bits.
#include "../../include/sgpt_b200.h"
#include "common.cuh"
#include "gemm_api.h"
#include "host_utils.h"

using namespace sgpt;

namespace {

constexpr int kRangeThreads = 256;
constexpr int kRangeBlock = 256;        // queries per filter launch (CTA pairs above 128, gemm.cu launch_filter_gemm)
constexpr int kHalfTile = kSimBN / 2;   // documents per group run
constexpr int kFillBlocksX = 32;        // CTAs per query of the fill kernel (8 warps each, striding over the half tiles)

inline int64_t align256(int64_t x) { return (x + 255) & ~int64_t(255); }

// Fixed head of the workspace, the same for every query block: the running output offset (int64) and tau[kRangeBlock].
constexpr int64_t kHeadBytes = 256 + kRangeBlock * 4;

struct Layout {
  FilterGeometry g;
  int64_t stride_q;  // list entries per query
  int64_t H;         // half tiles of the shard
  int64_t bytes;     // plan-dependent part (after the head)
};

Layout make_layout(int nb, int64_t n) {
  Layout l{};
  const int64_t tiles = (n + kSimBN - 1) / kSimBN;
  l.g = filter_geometry(tiles, nb);
  l.stride_q = static_cast<int64_t>(l.g.groups) * l.g.L;
  l.H = (n + kHalfTile - 1) / kHalfTile;
  l.bytes = align256(nb * l.stride_q * 8) + align256(static_cast<int64_t>(l.g.groups) * nb * 4) +
            2 * align256(nb * l.H * 4) + align256(nb * 4) + align256(nb * 8);
  return l;
}

// inclusive block-wide scan of one value per thread (kRangeThreads threads); *total = the block's sum
template <class T>
__device__ __forceinline__ T block_inclusive_scan(T v, T* s_warp, T* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  if (lane == 31) s_warp[warp] = v;
  __syncthreads();
  T before = 0, sum = 0;
#pragma unroll
  for (int w = 0; w < kRangeThreads / 32; ++w) {
    const T x = s_warp[w];
    before += (w < warp) ? x : T(0);
    sum += x;
  }
  __syncthreads();  // s_warp is reused by the next call
  *total = sum;
  return v + before;
}

// first position in list[0, cnt) whose document index is >= doc (the list is ascending in document index)
__device__ __forceinline__ int lower_bound_doc(const uint2* __restrict__ list, int cnt, uint32_t doc) {
  int lo = 0, hi = cnt;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(&list[mid].y) < doc) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// runs: per query, the start of every half tile's run in its group list and the run's offset inside the query's result
__global__ void __launch_bounds__(kRangeThreads) range_runs_kernel(const uint2* __restrict__ cand,
                                                                    const int* __restrict__ counts, long long stride_q,
                                                                    int L, int slots, int nq, long long H,
                                                                    int* __restrict__ run_start, int* __restrict__ run_off,
                                                                    int* __restrict__ qcount) {
  __shared__ int s_warp[kRangeThreads / 32];
  const int q = blockIdx.x;
  pdl_sync();
  const uint2* lists = cand + static_cast<long long>(q) * stride_q;
  int carry = 0;
  for (long long h0 = 0; h0 < H; h0 += kRangeThreads) {
    const long long h = h0 + threadIdx.x;
    int start = 0, len = 0;
    if (h < H) {
      const long long tile = h >> 1;
      const int g = 2 * static_cast<int>(tile % slots) + static_cast<int>(h & 1);
      const int cnt = __ldg(counts + static_cast<long long>(g) * nq + q);
      if (cnt > 0) {
        const uint2* list = lists + static_cast<long long>(g) * L;
        const uint32_t lo = static_cast<uint32_t>(h * kHalfTile);
        start = lower_bound_doc(list, cnt, lo);
        len = lower_bound_doc(list + start, cnt - start, lo + kHalfTile);
      }
    }
    int total;
    const int incl = block_inclusive_scan(len, s_warp, &total);
    if (h < H) {
      run_start[static_cast<long long>(q) * H + h] = start;
      run_off[static_cast<long long>(q) * H + h] = carry + incl - len;
    }
    carry += total;
  }
  if (threadIdx.x == 0) qcount[q] = carry;
}

// offsets: counts of the block's queries -> out_counts, their global output offsets (or -1: does not fit), running total
__global__ void __launch_bounds__(kRangeThreads) range_offsets_kernel(const int* __restrict__ qcount, int nb, int first,
                                                                       long long cap, long long* running,
                                                                       int64_t* __restrict__ out_counts,
                                                                       long long* __restrict__ qoff) {
  __shared__ long long s_warp[kRangeThreads / 32];
  pdl_sync();
  const long long base = first ? 0ll : *running;
  const int t = threadIdx.x;  // nb <= kRangeBlock == kRangeThreads
  const long long c = t < nb ? static_cast<long long>(qcount[t]) : 0ll;
  long long total;
  const long long off = base + block_inclusive_scan(c, s_warp, &total) - c;  // (the scan's barriers order the read above)
  if (t < nb) {
    out_counts[t] = c;
    qoff[t] = (off + c <= cap) ? off : -1ll;
  }
  if (t == 0) *running = base + total;
}

// fill: warp per half-tile run; the run's entries go to out[qoff[q] + run_off .. + len) in list (= document) order
__global__ void __launch_bounds__(kRangeThreads) range_fill_kernel(const uint2* __restrict__ cand,
                                                                    long long stride_q, int L, int slots, long long H,
                                                                    const int* __restrict__ run_start,
                                                                    const int* __restrict__ run_off,
                                                                    const int* __restrict__ qcount,
                                                                    const long long* __restrict__ qoff,
                                                                    long long id_base, float* __restrict__ out_scores,
                                                                    int64_t* __restrict__ out_ids) {
  const int q = blockIdx.y;
  const int lane = threadIdx.x & 31;
  pdl_sync();
  const long long base = qoff[q];
  if (base < 0) return;  // the query does not fit: its slots of the output keep their bits
  const uint2* lists = cand + static_cast<long long>(q) * stride_q;
  const int* rs = run_start + static_cast<long long>(q) * H;
  const int* ro = run_off + static_cast<long long>(q) * H;
  const int total = qcount[q];
  const long long warps = static_cast<long long>(gridDim.x) * (kRangeThreads / 32);
  for (long long h = static_cast<long long>(blockIdx.x) * (kRangeThreads / 32) + (threadIdx.x >> 5); h < H; h += warps) {
    const int o = ro[h];
    const int len = (h + 1 < H ? ro[h + 1] : total) - o;
    if (len == 0) continue;  // (warp-uniform)
    const long long tile = h >> 1;
    const int g = 2 * static_cast<int>(tile % slots) + static_cast<int>(h & 1);
    const uint2* src = lists + static_cast<long long>(g) * L + rs[h];
    const long long dst = base + o;
    for (int i = lane; i < len; i += 32) {
      const uint2 e = __ldg(src + i);
      out_scores[dst + i] = __uint_as_float(e.x);
      out_ids[dst + i] = id_base + static_cast<long long>(e.y);
    }
  }
}

__global__ void range_tau_kernel(float* __restrict__ tau, int nb, float threshold) {
  pdl_sync();
  if (static_cast<int>(threadIdx.x) < nb) tau[threadIdx.x] = threshold;
}

int64_t block_bytes(int nb, int64_t n) { return make_layout(nb, n).bytes; }

}  // namespace

extern "C" int64_t sgpt_range_search_workspace_bytes(int nq, int64_t n) {
  if (nq < 0 || n < 0) return 0;
  // blocks of kRangeBlock queries reuse the workspace; the last block may hold <= 128 queries and then takes the
  // single-CTA geometry, whose lists are laid out differently (as sgpt_search_workspace_bytes)
  int64_t b = block_bytes(nq < 128 ? nq : 128, n);
  if (nq > 128) {
    const int64_t a = block_bytes(nq < kRangeBlock ? nq : kRangeBlock, n);
    if (a > b) b = a;
  }
  return kHeadBytes + b;
}

// op: the type of the Q and C rows (gemm_api.h Operand); everything after the filter GEMM is the same.  mask: the filter admits allowed
// documents only, so the lists stay ascending in document index and the run / offset / fill kernels are unchanged.
static int range_search(const void* Q, const void* Cm, const float* q_scale, const float* c_scale, int nq, int64_t n, int D,
                        float threshold, int64_t id_base, int64_t* out_counts, int64_t cap, float* out_scores,
                        int64_t* out_ids, void* ws, int64_t ws_bytes, DocMask mask, Operand op, cudaStream_t stream) {
  SGPT_REQUIRE(threshold == threshold, "sgpt_range_search: threshold is NaN");
  if (check_doc_mask("sgpt_range_search", n, mask) != SGPT_OK) return SGPT_ERR_INVALID;
  if (check_operands("sgpt_range_search", op, Q, Cm, q_scale, c_scale, nq, D) != SGPT_OK) return SGPT_ERR_INVALID;
  const size_t row_bytes = operand_row_bytes(op, D);
  SGPT_REQUIRE(n >= 0 && n < (1ll << 31), "sgpt_range_search: shard size n=%lld outside [0, 2^31)", (long long)n);
  SGPT_REQUIRE(nq >= 0 && cap >= 0, "sgpt_range_search: bad sizes nq=%d cap=%lld", nq, (long long)cap);
  SGPT_REQUIRE(nq == 0 || out_counts != nullptr, "sgpt_range_search: null out_counts");
  SGPT_REQUIRE(nq == 0 || cap == 0 || (out_scores != nullptr && out_ids != nullptr),
               "sgpt_range_search: null out_scores / out_ids with cap=%lld", (long long)cap);
  const int64_t need = sgpt_range_search_workspace_bytes(nq, n);
  SGPT_REQUIRE(ws != nullptr && ws_bytes >= need, "sgpt_range_search: workspace too small (%lld < %lld bytes)",
               (long long)ws_bytes, (long long)need);
  if (nq == 0) return SGPT_OK;

  uint8_t* head = static_cast<uint8_t*>(ws);
  long long* running = reinterpret_cast<long long*>(head);
  float* tau = reinterpret_cast<float*>(head + 256);
  uint8_t* body = head + kHeadBytes;
  {
    LaunchScope _ls(kCatTopk, stream);
    SGPT_CHECK_CUDA(launch_kernel(range_tau_kernel, dim3(1), dim3(kRangeBlock), 0, stream, tau,
                                  nq < kRangeBlock ? nq : kRangeBlock, threshold));
  }
  for (int q0 = 0; q0 < nq; q0 += kRangeBlock) {
    const int nb = (nq - q0 < kRangeBlock) ? nq - q0 : kRangeBlock;
    const Layout l = make_layout(nb, n);
    uint8_t* w = body;
    uint2* cand = reinterpret_cast<uint2*>(w);
    w += align256(nb * l.stride_q * 8);
    int* cnt = reinterpret_cast<int*>(w);
    w += align256(static_cast<int64_t>(l.g.groups) * nb * 4);
    int* run_start = reinterpret_cast<int*>(w);
    w += align256(nb * l.H * 4);
    int* run_off = reinterpret_cast<int*>(w);
    w += align256(nb * l.H * 4);
    int* qcount = reinterpret_cast<int*>(w);
    w += align256(nb * 4);
    long long* qoff = reinterpret_cast<long long*>(w);
    const void* Qb = static_cast<const uint8_t*>(Q) + static_cast<size_t>(q0) * row_bytes;
    const float* qs = q_scale ? q_scale + q0 : nullptr;

    DocMask mb = mask;
    if (mb.bits != nullptr) mb.bits += q0 * mb.pitch;
    if (n > 0) {
      int rc = launch_filter_candidates(Qb, Cm, qs, c_scale, tau, nullptr, cand, cnt, nullptr, l.stride_q, l.g.L, 0, nb,
                                        static_cast<int>(n), D, /*tile_mode=*/0, 1, mb, op, stream);
      if (rc != SGPT_OK) return rc;
    }
    LaunchScope _ls(kCatTopk, stream);
    SGPT_CHECK_CUDA(launch_kernel(range_runs_kernel, dim3(nb), dim3(kRangeThreads), 0, stream,
                                  static_cast<const uint2*>(cand), static_cast<const int*>(cnt), (long long)l.stride_q,
                                  l.g.L, l.g.groups / 2, nb, (long long)l.H, run_start, run_off, qcount));
    SGPT_CHECK_CUDA(launch_kernel(range_offsets_kernel, dim3(1), dim3(kRangeThreads), 0, stream,
                                  static_cast<const int*>(qcount), nb, q0 == 0 ? 1 : 0, (long long)cap, running,
                                  out_counts + q0, qoff));
    if (cap > 0 && l.H > 0) {
      const long long bx = (l.H + kRangeThreads / 32 - 1) / (kRangeThreads / 32);
      SGPT_CHECK_CUDA(launch_kernel(range_fill_kernel, dim3(static_cast<unsigned>(bx < kFillBlocksX ? bx : kFillBlocksX), nb),
                                    dim3(kRangeThreads), 0, stream, static_cast<const uint2*>(cand), (long long)l.stride_q,
                                    l.g.L, l.g.groups / 2, (long long)l.H, static_cast<const int*>(run_start),
                                    static_cast<const int*>(run_off), static_cast<const int*>(qcount),
                                    static_cast<const long long*>(qoff), (long long)id_base, out_scores, out_ids));
    }
  }
  return SGPT_OK;
}

extern "C" int sgpt_range_search(const void* Q, const void* Cm, const float* q_scale, const float* c_scale, int nq,
                                 int64_t n, int D, float threshold, int64_t id_base, int64_t* out_counts, int64_t cap,
                                 float* out_scores, int64_t* out_ids, void* ws, int64_t ws_bytes,
                                 sgpt_stream_t stream_) {
  return range_search(Q, Cm, q_scale, c_scale, nq, n, D, threshold, id_base, out_counts, cap, out_scores, out_ids, ws,
                      ws_bytes, DocMask(), Operand::kBF16, static_cast<cudaStream_t>(stream_));
}

extern "C" int sgpt_range_search_i8(const void* Q, const void* Cm, const float* q_scale, const float* c_scale, int nq,
                                    int64_t n, int D, float threshold, int64_t id_base, int64_t* out_counts, int64_t cap,
                                    float* out_scores, int64_t* out_ids, void* ws, int64_t ws_bytes,
                                    sgpt_stream_t stream_) {
  return range_search(Q, Cm, q_scale, c_scale, nq, n, D, threshold, id_base, out_counts, cap, out_scores, out_ids, ws,
                      ws_bytes, DocMask(), Operand::kS8, static_cast<cudaStream_t>(stream_));
}

extern "C" int sgpt_range_search_masked(int dtype, const void* Q, const void* Cm, const float* q_scale,
                                        const float* c_scale, int nq, int64_t n, int D, float threshold, int64_t id_base,
                                        const uint32_t* mask, int64_t mask_pitch_words, int64_t* out_counts, int64_t cap,
                                        float* out_scores, int64_t* out_ids, void* ws, int64_t ws_bytes,
                                        sgpt_stream_t stream_) {
  Operand op;
  if (shard_operand("sgpt_range_search_masked", dtype, &op) != SGPT_OK) return SGPT_ERR_INVALID;
  return range_search(Q, Cm, q_scale, c_scale, nq, n, D, threshold, id_base, out_counts, cap, out_scores, out_ids, ws,
                      ws_bytes, DocMask{mask, mask_pitch_words}, op, static_cast<cudaStream_t>(stream_));
}
