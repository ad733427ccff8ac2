// Graph index (include/sgpt_b200.h sgpt_graph_prune, sgpt_graph_search): the rank-based detour pruning of k-NN lists
// and the beam search over the pruned graph.
//
//   prune    one CTA per row a: the row's K ids in a shared-memory map id -> rank, then one warp per valid neighbour b
//            walks b's list and counts, for every entry i of a's list that b's list holds before position i, one detour
//            (a per-warp bitmap of the ranks already counted for b keeps repeats in b's list from counting twice).  The
//            counts are integers, so the shared-memory atomics leave the output deterministic.  Each valid entry's
//            place in the output is the number of valid entries with a smaller (count, rank).
//   search   one CTA per query.  B (the itopk best entries so far) and the step's new candidates are 64-bit keys
//            (score key, position, expanded flag) in one shared-memory buffer, sorted by a bitonic sort after every
//            step; the visited set is an open-addressing table in shared memory sized so that it is never more than
//            half full.  One warp scores one candidate with sgpt_rerank's loop (rerank.cuh).
#include "../../include/sgpt_b200.h"
#include "common.cuh"
#include "gemm_api.h"
#include "host_utils.h"
#include "rerank.cuh"
#include "topk.cuh"

using namespace sgpt;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxK = 256;          // prune: entries per k-NN list
constexpr int kMapSize = 512;       // prune: map slots (at most half full)
constexpr int kMaxStep = 512;       // search: seeds, and search_width x degree candidates of one step
constexpr int kMaxWidth = 8;        // search: search_width
constexpr int kMaxTable = 32768;    // search: visited-table slots
constexpr uint64_t kEmpty = ~0ull;  // search: an empty entry of B (sorts last, reads as expanded)

__host__ __device__ constexpr int next_pow2(long long x) {
  int p = 1;
  while (p < x) p <<= 1;
  return p;
}

__device__ __forceinline__ uint32_t slot_of(uint32_t x, int bits) { return (x * 0x9E3779B1u) >> (32 - bits); }

// the seed hash of include/sgpt_b200.h: murmur3's 32-bit finalizer of seed + 0x9E3779B1 q + 0x85EBCA77 j (mod 2^32)
__device__ __forceinline__ uint32_t seed_hash(uint32_t seed, uint32_t q, uint32_t j) {
  uint32_t x = seed + 0x9E3779B1u * q + 0x85EBCA77u * j;
  x ^= x >> 16;
  x *= 0x85EBCA6Bu;
  x ^= x >> 13;
  x *= 0xC2B2AE35u;
  x ^= x >> 16;
  return x;
}

// ---- prune ----------------------------------------------------------------------------------------------------------
// kAppend: the rows n_old .. n - 1 only (one CTA each, block r = row n_old + r, knn row r); the list of a position
// b < n_old is graph[b][0 .. degree-1], of a later one knn[b - n_old]
template <bool kAppend>
__global__ void __launch_bounds__(kThreads) graph_prune_kernel(const int32_t* __restrict__ knn, int n, int K, int degree,
                                                               int32_t* __restrict__ out,
                                                               const int32_t* __restrict__ graph, int n_old) {
  __shared__ int32_t ids[kMaxK];  // row a's entries; -1: empty (outside [0, n), a itself, or a repeat)
  __shared__ int32_t map_id[kMapSize], map_rank[kMapSize];
  __shared__ uint32_t detours[kMaxK];
  __shared__ uint32_t counted[kWarps][kMaxK / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int row = static_cast<int>(blockIdx.x);
  const int a = kAppend ? n_old + row : row;
  for (int s = tid; s < kMapSize; s += kThreads) {
    map_id[s] = -1;
    map_rank[s] = kMaxK;
  }
  pdl_sync();
  int v = -1;
  if (tid < K) {
    v = __ldg(knn + static_cast<long long>(row) * K + tid);
    v = (v >= 0 && v < n && v != a) ? v : -1;
    detours[tid] = 0;
  }
  __syncthreads();
  if (v >= 0) {  // insert; a repeated id keeps its first rank
    for (uint32_t s = slot_of(v, 9);; s = (s + 1) & (kMapSize - 1)) {
      const int prev = atomicCAS(&map_id[s], -1, v);
      if (prev == -1 || prev == v) {
        atomicMin(&map_rank[s], tid);
        break;
      }
    }
  }
  __syncthreads();
  auto rank_of = [&](int x) {  // rank of x in a's list, or -1
    if (x < 0) return -1;
    for (uint32_t s = slot_of(x, 9);; s = (s + 1) & (kMapSize - 1)) {
      const int id = map_id[s];
      if (id == x) return map_rank[s];
      if (id == -1) return -1;
    }
  };
  if (v >= 0 && rank_of(v) != tid) v = -1;
  if (tid < K) ids[tid] = v;
  __syncthreads();
  for (int j = warp; j < K; j += kWarps) {
    const int b = ids[j];
    if (b < 0) continue;  // warp-uniform
    if (lane < kMaxK / 32) counted[warp][lane] = 0u;
    __syncwarp();
    const int32_t* list = knn + static_cast<long long>(b) * K;
    int len = K - 1;  // entries at positions below K - 1 can precede an entry of a's list
    if constexpr (kAppend) {
      if (b < n_old) {
        list = graph + static_cast<long long>(b) * degree;
        len = min(degree, K - 1);
      } else {
        list = knn + static_cast<long long>(b - n_old) * K;
      }
    }
    for (int p = lane; p < len; p += 32) {
      const int i = rank_of(__ldg(list + p));
      if (i > j && i > p) {
        const uint32_t bit = 1u << (i & 31);
        if (!(atomicOr(&counted[warp][i >> 5], bit) & bit)) atomicAdd(&detours[i], 1u);
      }
    }
    __syncwarp();
  }
  __syncthreads();
  // order (detours, rank) as one key: both are below 256
  const uint32_t key = v >= 0 ? (detours[tid] << 8 | static_cast<uint32_t>(tid)) : 0xffffffffu;
  __syncthreads();
  if (tid < K) detours[tid] = key;
  const int valid = __syncthreads_count(v >= 0);
  int32_t* dst = out + static_cast<long long>(row) * degree;
  if (v >= 0) {
    int r = 0;
    for (int i = 0; i < K; ++i) r += detours[i] < key;
    if (r < degree) dst[r] = v;
  }
  for (int r = valid + tid; r < degree; r += kThreads) dst[r] = -1;
}

// ---- search ---------------------------------------------------------------------------------------------------------
struct SearchArgs {
  const uint8_t* Q;
  const uint8_t* C;
  const float* q_scale;
  const float* c_scale;
  int n, D;
  long long id_base;
  const int32_t* graph;
  int degree;
  const int32_t* seeds;
  int num_seeds;
  uint32_t seed;
  int itopk, search_width, max_iterations, k;
  const uint32_t* mask;
  float* out_scores;
  int64_t* out_ids;
  int32_t* out_visited;
  int sort_cap;    // entries of the sort buffer: next_pow2(itopk + max(num_seeds, search_width x degree))
  int table_bits;  // log2 of the visited-table slots
  long long mask_pitch;  // filtered search: words per query's bitmap, 0 = one shared bitmap
};

// (score descending, position ascending) as an ascending 64-bit key; bit 0 is the expanded flag, which never decides the
// order because positions are distinct
__device__ __forceinline__ uint64_t entry_key(float s, int x) {
  return (static_cast<uint64_t>(~score_key(s)) << 32) | (static_cast<uint64_t>(x) << 1);
}

size_t search_smem_bytes(int sort_cap, int table_bits) {
  return static_cast<size_t>(sort_cap) * 8 + kMaxStep * 4 + (static_cast<size_t>(4) << table_bits);
}

// entries of the filtered search's result buffer: R (k keys), then the allowed keys of one step
int result_cap(int k, int step) { return next_pow2(k + step); }

// kFiltered: the walk is the same; R, the best k keys of the positions in V that the mask (shared, or one bitmap per
// query) allows, is kept next to it and is the output
template <bool kS8, bool kFiltered = false>
__global__ void __launch_bounds__(kThreads) graph_search_kernel(const SearchArgs a) {
  extern __shared__ __align__(16) uint8_t smem[];
  uint64_t* buf = reinterpret_cast<uint64_t*>(smem);              // [sort_cap]: B, then the step's candidates
  int32_t* cand = reinterpret_cast<int32_t*>(buf + a.sort_cap);   // [kMaxStep]: positions first visited in this step
  int32_t* table = cand + kMaxStep;                               // [1 << table_bits]: visited positions, -1 = free
  __shared__ int s_count, s_np, s_p[kMaxWidth];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int q = static_cast<int>(blockIdx.x);
  const int tsize = 1 << a.table_bits;
  for (int i = tid; i < tsize; i += kThreads) table[i] = -1;
  for (int i = tid; i < a.itopk; i += kThreads) buf[i] = kEmpty;
  if (tid == 0) s_count = 0;
  uint64_t* res = reinterpret_cast<uint64_t*>(table + tsize);  // filtered: [result_cap]: R, then the step's allowed keys
  const uint32_t* qmask = a.mask != nullptr ? a.mask + q * a.mask_pitch : nullptr;
  __shared__ int s_rcount;  // filtered: allowed keys after R in this step
  if constexpr (kFiltered) {
    for (int i = tid; i < a.k; i += kThreads) res[i] = kEmpty;
    if (tid == 0) s_rcount = 0;
  }
  __syncthreads();
  pdl_sync();
  // V holds at most num_seeds + max_iterations x search_width x degree <= tsize / 2 positions: probing always ends
  auto visit = [&](int x) {
    for (uint32_t s = slot_of(static_cast<uint32_t>(x), a.table_bits);; s = (s + 1) & (tsize - 1)) {
      const int prev = atomicCAS(&table[s], -1, x);
      if (prev == -1) {
        cand[atomicAdd(&s_count, 1)] = x;
        return;
      }
      if (prev == x) return;
    }
  };
  for (int j = tid; j < a.num_seeds; j += kThreads) {
    int x;
    if (a.seeds != nullptr) {
      x = __ldg(a.seeds + static_cast<long long>(q) * a.num_seeds + j);
      if (x < 0 || x >= a.n) continue;
    } else {
      x = static_cast<int>(seed_hash(a.seed, static_cast<uint32_t>(q), static_cast<uint32_t>(j)) %
                           static_cast<uint32_t>(a.n));
    }
    visit(x);
  }
  __syncthreads();
  const long long row_bytes = kS8 ? a.D : 2ll * a.D;
  const int units = static_cast<int>(row_bytes / 16);
  const uint4* qp = reinterpret_cast<const uint4*>(a.Q + q * row_bytes);
  int visited = 0;
  for (int t = 0;; ++t) {
    // score the positions first visited in the last step into buf[itopk ..), then B = the best itopk of both
    const int count = s_count;
    visited += count;
    for (int c = warp; c < count; c += kWarps) {
      const int x = cand[c];
      float s = rerank_dot<kS8>(qp, reinterpret_cast<const uint4*>(a.C + x * row_bytes), units, lane);
      s = s * (a.q_scale != nullptr ? __ldg(a.q_scale + q) : 1.f) * (a.c_scale != nullptr ? __ldg(a.c_scale + x) : 1.f);
      s = (s != s) ? -1.f : s;
      if (lane == 0) buf[a.itopk + c] = entry_key(s, x);
      if constexpr (kFiltered) {
        // only keys that beat R's k-th can enter R (R never gets worse), so steps without one skip R's sort
        const uint64_t key = entry_key(s, x);
        if (lane == 0 && key < res[a.k - 1] && (qmask == nullptr || ((__ldg(qmask + (x >> 5)) >> (x & 31)) & 1u)))
          res[a.k + atomicAdd(&s_rcount, 1)] = key;
      }
    }
    const int total = a.itopk + count;
    const int S = next_pow2(total);
    for (int i = total + tid; i < S; i += kThreads) buf[i] = kEmpty;
    __syncthreads();
    for (int size = 2; size <= S; size <<= 1) {
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        for (int i = tid; i < S / 2; i += kThreads) {
          const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
          const uint64_t x = buf[lo], y = buf[hi];
          if ((x > y) == ((lo & size) == 0)) {
            buf[lo] = y;
            buf[hi] = x;
          }
        }
        __syncthreads();
      }
    }
    if constexpr (kFiltered) {
      // R = the best k of R and the step's allowed keys (s_rcount is read after the barriers of the sort above)
      const int rn = s_rcount;
      if (rn > 0) {
        const int rs = next_pow2(a.k + rn);
        for (int i = a.k + rn + tid; i < rs; i += kThreads) res[i] = kEmpty;
        __syncthreads();
        for (int size = 2; size <= rs; size <<= 1) {
          for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = tid; i < rs / 2; i += kThreads) {
              const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
              const uint64_t x = res[lo], y = res[hi];
              if ((x > y) == ((lo & size) == 0)) {
                res[lo] = y;
                res[hi] = x;
              }
            }
            __syncthreads();
          }
        }
        if (tid == 0) s_rcount = 0;
      }
    }
    if (t == a.max_iterations) break;
    // P = the first search_width unexpanded entries of B, marked expanded
    if (warp == 0) {
      int np = 0;
      for (int b0 = 0; b0 < a.itopk && np < a.search_width; b0 += 32) {
        const uint64_t key = buf[b0 + lane];
        const bool open = (key & 1ull) == 0;
        const uint32_t m = __ballot_sync(0xffffffffu, open);
        const int r = np + __popc(m & ((1u << lane) - 1u));
        if (open && r < a.search_width) {
          s_p[r] = static_cast<int>(static_cast<uint32_t>(key) >> 1);
          buf[b0 + lane] = key | 1ull;
        }
        np += __popc(m);
      }
      if (lane == 0) {
        s_np = min(np, a.search_width);
        s_count = 0;
      }
    }
    __syncthreads();
    const int np = s_np;
    if (np == 0) break;
    for (int e = tid; e < np * a.degree; e += kThreads) {
      const int p = s_p[e / a.degree];
      const int x = __ldg(a.graph + static_cast<long long>(p) * a.degree + e % a.degree);
      if (x >= 0 && x < a.n) visit(x);
    }
    __syncthreads();
  }
  if (warp != 0) return;
  const long long o = static_cast<long long>(q) * a.k;
  if constexpr (kFiltered) {
    for (int r = lane; r < a.k; r += 32) {
      const uint64_t key = res[r];
      const bool ok = (key >> 32) != 0xffffffffull;
      a.out_scores[o + r] = ok ? key_score(~static_cast<uint32_t>(key >> 32)) : -INFINITY;
      a.out_ids[o + r] = ok ? a.id_base + static_cast<int>(static_cast<uint32_t>(key) >> 1) : -1ll;
    }
    if (lane == 0 && a.out_visited != nullptr) a.out_visited[q] = visited;
    return;
  }
  // the first k entries of B that the mask allows
  int got = 0;
  for (int b0 = 0; b0 < a.itopk && got < a.k; b0 += 32) {
    const uint64_t key = buf[b0 + lane];
    const int x = static_cast<int>(static_cast<uint32_t>(key) >> 1);
    const bool ok = (key >> 32) != 0xffffffffull &&
                    (a.mask == nullptr || ((__ldg(a.mask + (x >> 5)) >> (x & 31)) & 1u));
    const uint32_t m = __ballot_sync(0xffffffffu, ok);
    const int r = got + __popc(m & ((1u << lane) - 1u));
    if (ok && r < a.k) {
      a.out_scores[o + r] = key_score(~static_cast<uint32_t>(key >> 32));
      a.out_ids[o + r] = a.id_base + x;
    }
    got += __popc(m);
  }
  for (int r = min(got, a.k) + lane; r < a.k; r += 32) {
    a.out_scores[o + r] = -INFINITY;
    a.out_ids[o + r] = -1;
  }
  if (lane == 0 && a.out_visited != nullptr) a.out_visited[q] = visited;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int graph_prune(const char* fn, const int32_t* knn, int64_t n, int K, int degree, int32_t* out, cudaStream_t stream) {
  SGPT_REQUIRE(n >= 0 && n < (1ll << 31), "%s: n=%lld outside [0, 2^31)", fn, (long long)n);
  SGPT_REQUIRE(degree >= 16 && degree <= 128 && degree % 16 == 0, "%s: degree=%d must be a multiple of 16 in [16, 128]",
               fn, degree);
  SGPT_REQUIRE(K >= degree && K <= kMaxK, "%s: K=%d outside [degree=%d, %d]", fn, K, degree, kMaxK);
  SGPT_REQUIRE(knn != nullptr, "%s: null input knn", fn);
  SGPT_REQUIRE(out != nullptr, "%s: null output", fn);
  if (n == 0) return SGPT_OK;
  LaunchScope _ls(kCatMisc, stream);
  SGPT_CHECK_CUDA(launch_kernel(graph_prune_kernel<false>, dim3(static_cast<unsigned>(n)), dim3(kThreads), 0, stream,
                                knn, static_cast<int>(n), K, degree, out, static_cast<const int32_t*>(nullptr), 0));
  return SGPT_OK;
}

int graph_prune_append(const char* fn, const int32_t* graph, int64_t n_old, int degree, const int32_t* knn, int64_t m,
                       int K, int32_t* out, cudaStream_t stream) {
  SGPT_REQUIRE(n_old >= 0 && m >= 0 && n_old + m < (1ll << 31),
               "%s: n_old=%lld and m=%lld must be non-negative with n_old + m < 2^31", fn, (long long)n_old,
               (long long)m);
  SGPT_REQUIRE(degree >= 16 && degree <= 128 && degree % 16 == 0, "%s: degree=%d must be a multiple of 16 in [16, 128]",
               fn, degree);
  SGPT_REQUIRE(K >= degree && K <= kMaxK, "%s: K=%d outside [degree=%d, %d]", fn, K, degree, kMaxK);
  SGPT_REQUIRE(graph != nullptr || n_old == 0, "%s: null input graph with n_old=%lld", fn, (long long)n_old);
  SGPT_REQUIRE(knn != nullptr, "%s: null input knn", fn);
  SGPT_REQUIRE(out != nullptr, "%s: null output", fn);
  if (m == 0) return SGPT_OK;
  LaunchScope _ls(kCatMisc, stream);
  SGPT_CHECK_CUDA(launch_kernel(graph_prune_kernel<true>, dim3(static_cast<unsigned>(m)), dim3(kThreads), 0, stream,
                                knn, static_cast<int>(n_old + m), K, degree, out, graph, static_cast<int>(n_old)));
  return SGPT_OK;
}

int graph_search(const char* fn, int dtype, const void* Q, const void* C, const float* q_scale, const float* c_scale,
                 int nq, int64_t n, int D, int64_t id_base, const int32_t* graph, int degree, const int32_t* seeds,
                 int num_seeds, uint32_t seed, int itopk, int search_width, int max_iterations, int k,
                 const uint32_t* mask, int64_t mask_pitch, bool filtered, float* out_scores, int64_t* out_ids,
                 int32_t* out_visited, cudaStream_t stream) {
  SGPT_REQUIRE(dtype == SGPT_DTYPE_BF16 || dtype == SGPT_DTYPE_I8, "%s: shard dtype %d must be bf16 (0) or int8 (1)", fn,
               dtype);
  const bool s8 = dtype == SGPT_DTYPE_I8;
  SGPT_REQUIRE(nq >= 0, "%s: bad query count nq=%d", fn, nq);
  if (s8)
    SGPT_REQUIRE(D > 0 && D % 16 == 0 && D <= 65536, "%s: int8 D=%d must be a positive multiple of 16, at most %d", fn,
                 D, 65536);
  else
    SGPT_REQUIRE(D > 0 && D % 8 == 0, "%s: D=%d must be a positive multiple of 8", fn, D);
  SGPT_REQUIRE(n >= 1 && n < (1ll << 31), "%s: corpus size n=%lld outside [1, 2^31)", fn, (long long)n);
  SGPT_REQUIRE(id_base >= 0 && id_base + n <= (1ll << 31), "%s: global ids id_base=%lld + n=%lld must fit in int32", fn,
               (long long)id_base, (long long)n);
  SGPT_REQUIRE(itopk >= 32 && itopk <= 512 && itopk % 32 == 0, "%s: itopk=%d must be a multiple of 32 in [32, 512]", fn,
               itopk);
  SGPT_REQUIRE(k >= 1 && k <= itopk, "%s: k=%d outside [1, itopk=%d]", fn, k, itopk);
  SGPT_REQUIRE(degree >= 1, "%s: degree=%d must be positive", fn, degree);
  SGPT_REQUIRE(search_width >= 1 && search_width <= kMaxWidth, "%s: search_width=%d outside [1, %d]", fn, search_width,
               kMaxWidth);
  SGPT_REQUIRE(static_cast<int64_t>(search_width) * degree <= kMaxStep,
               "%s: search_width=%d x degree=%d exceeds %d candidates per step", fn, search_width, degree, kMaxStep);
  SGPT_REQUIRE(num_seeds >= 1 && num_seeds <= kMaxStep, "%s: num_seeds=%d outside [1, %d]", fn, num_seeds, kMaxStep);
  SGPT_REQUIRE(max_iterations >= 1, "%s: max_iterations=%d must be positive", fn, max_iterations);
  const int64_t most = 2 * (num_seeds + static_cast<int64_t>(max_iterations) * search_width * degree);
  SGPT_REQUIRE(most <= kMaxTable,
               "%s: the visited table of 2 x (num_seeds + max_iterations x search_width x degree) = %lld slots exceeds %d",
               fn, (long long)most, kMaxTable);
  SGPT_REQUIRE(Q != nullptr && C != nullptr && graph != nullptr, "%s: null input (Q, C and graph are required)", fn);
  SGPT_REQUIRE(aligned16(Q) && aligned16(C), "%s: Q and C must be 16-byte aligned", fn);
  SGPT_REQUIRE(out_scores != nullptr && out_ids != nullptr, "%s: null output", fn);
  if (filtered && check_doc_mask(fn, n, DocMask{mask, mask_pitch}) != SGPT_OK) return SGPT_ERR_INVALID;
  if (nq == 0) return SGPT_OK;
  const int step = num_seeds > search_width * degree ? num_seeds : search_width * degree;
  const int table = next_pow2(most);
  int bits = 0;
  while ((1 << bits) < table) ++bits;
  SearchArgs a{static_cast<const uint8_t*>(Q), static_cast<const uint8_t*>(C), q_scale, c_scale, static_cast<int>(n), D,
               static_cast<long long>(id_base), graph, degree, seeds, num_seeds, seed, itopk, search_width,
               max_iterations, k, mask, out_scores, out_ids, out_visited, next_pow2(itopk + step), bits, mask_pitch};
  if (filtered) {
    const size_t smem = search_smem_bytes(a.sort_cap, bits) + static_cast<size_t>(result_cap(k, step)) * 8;
    void (*kern)(const SearchArgs) = s8 ? graph_search_kernel<true, true> : graph_search_kernel<false, true>;
    static PerDeviceOnce attr_once;
    if (attr_once.first()) {
      const int most_smem =
          static_cast<int>(search_smem_bytes(next_pow2(512 + kMaxStep), 15) + result_cap(512, kMaxStep) * 8);
      SGPT_CHECK_CUDA(cudaFuncSetAttribute(graph_search_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           most_smem));
      SGPT_CHECK_CUDA(cudaFuncSetAttribute(graph_search_kernel<false, true>,
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, most_smem));
    }
    LaunchScope _ls(kCatScores, stream);
    SGPT_CHECK_CUDA(launch_kernel(kern, dim3(static_cast<unsigned>(nq)), dim3(kThreads), smem, stream, a));
    return SGPT_OK;
  }
  const size_t smem = search_smem_bytes(a.sort_cap, bits);
  void (*kern)(const SearchArgs) = s8 ? graph_search_kernel<true> : graph_search_kernel<false>;
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    const int most_smem = static_cast<int>(search_smem_bytes(next_pow2(512 + kMaxStep), 15));
    SGPT_CHECK_CUDA(cudaFuncSetAttribute(graph_search_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         most_smem));
    SGPT_CHECK_CUDA(cudaFuncSetAttribute(graph_search_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         most_smem));
  }
  LaunchScope _ls(kCatScores, stream);
  SGPT_CHECK_CUDA(launch_kernel(kern, dim3(static_cast<unsigned>(nq)), dim3(kThreads), smem, stream, a));
  return SGPT_OK;
}

}  // namespace

extern "C" int sgpt_graph_prune(const int32_t* knn, int64_t n, int K, int degree, int32_t* out, sgpt_stream_t stream) {
  return graph_prune("sgpt_graph_prune", knn, n, K, degree, out, static_cast<cudaStream_t>(stream));
}

extern "C" int sgpt_graph_prune_append(const int32_t* graph, int64_t n_old, int degree, const int32_t* knn, int64_t m,
                                       int K, int32_t* out, sgpt_stream_t stream) {
  return graph_prune_append("sgpt_graph_prune_append", graph, n_old, degree, knn, m, K, out,
                            static_cast<cudaStream_t>(stream));
}

extern "C" int sgpt_graph_search(int dtype, const void* Q, const void* C, const float* q_scale, const float* c_scale,
                                 int nq, int64_t n, int D, int64_t id_base, const int32_t* graph, int degree,
                                 const int32_t* seeds, int num_seeds, uint32_t seed, int itopk, int search_width,
                                 int max_iterations, int k, const uint32_t* mask, float* out_scores, int64_t* out_ids,
                                 int32_t* out_visited, sgpt_stream_t stream) {
  return graph_search("sgpt_graph_search", dtype, Q, C, q_scale, c_scale, nq, n, D, id_base, graph, degree, seeds,
                      num_seeds, seed, itopk, search_width, max_iterations, k, mask, 0, false, out_scores, out_ids,
                      out_visited, static_cast<cudaStream_t>(stream));
}

extern "C" int sgpt_graph_search_filtered(int dtype, const void* Q, const void* C, const float* q_scale,
                                          const float* c_scale, int nq, int64_t n, int D, int64_t id_base,
                                          const int32_t* graph, int degree, const int32_t* seeds, int num_seeds,
                                          uint32_t seed, int itopk, int search_width, int max_iterations, int k,
                                          const uint32_t* mask, int64_t mask_pitch_words, float* out_scores,
                                          int64_t* out_ids, int32_t* out_visited, sgpt_stream_t stream) {
  return graph_search("sgpt_graph_search_filtered", dtype, Q, C, q_scale, c_scale, nq, n, D, id_base, graph, degree,
                      seeds, num_seeds, seed, itopk, search_width, max_iterations, k, mask, mask_pitch_words, true,
                      out_scores, out_ids, out_visited, static_cast<cudaStream_t>(stream));
}
