// S2/S3: exact row-wise top-k selection (torch.topk at XS:102-108; heapq.nlargest merge at XS:121-132) and the kernels
// around it.
//
//   topk_select_kernel    one CTA (1024 threads) per query; keys = an order-preserving 32-bit image of the fp32 score, cached
//                         in shared memory.  Fast path: sample pivot -> one compaction pass -> exact k-th key by a radix-4
//                         bitwise search on register-resident keys; fallback: MSD radix select (11 + 11 + 10 bits,
//                         warp-aggregated histograms).  Then the k winners are placed, their ids fetched, and sorted
//                         (score descending, id ascending).  Sources through `TopkSrc`:
//                           - a dense score row           scores[q, 0..n)                    (ids = id_base + column)
//                           - filtered candidate lists    packed (score, local idx) pairs with per-(list, query) counts,
//                                                         optionally two-sided (front / back parts, topk.cuh)
//                           - G gathered lists            [G, nq, L] scores + ids or packed entries (cross-chunk /
//                                                         cross-shard merge; id < 0 = empty slot; optional peer-signal wait)
//   tau_select_kernel     the two admission thresholds of the two-pass search from its sampled block maxima
//   merge_sorted_kernel   S3 for few already-sorted packed lists: positions by binary search, no selection, no sort
//   front_select_kernel   opt-in experiment: sort all entries above the upper threshold instead of selecting (slower)
#include <math.h>
#include <stdlib.h>

#include "../../include/sgpt_b200.h"
#include "common.cuh"
#include "host_utils.h"
#include "topk.cuh"

namespace sgpt {

__device__ __forceinline__ uint32_t score_key(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_score(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

struct Elem {
  uint32_t key;  // 0 = invalid / empty
  long long id;
};

__device__ __forceinline__ long long list_len(const TopkSrc& s, int q, int g) {
  if (g >= s.G) {  // back part of list g - G (two-sided candidate lists, topk.cuh)
    long long c = s.counts_back[(g - s.G) * s.nq + q];
    return c < s.L ? c : s.L;
  }
  if (s.counts != nullptr) {
    long long c = s.counts[g * s.nq + q];
    return c < s.L ? c : s.L;
  }
  return s.L;
}

// offset of entry 0 of list g of query q (`len` = its length, needed for back parts only: they END at the list's end)
__device__ __forceinline__ long long list_base(const TopkSrc& s, int q, int g, long long len) {
  if (g >= s.G) return (g - s.G) * s.stride_g + q * s.stride_q + (s.L - len);
  return g * s.stride_g + q * s.stride_q;
}

__device__ __forceinline__ Elem load_elem_at(const TopkSrc& s, int q, long long off, long long i) {
  Elem e;
  if (s.packed != nullptr) {
    const uint2 p = s.packed[off];
    e.key = score_key(__uint_as_float(p.x));
    if (s.packed_global) {
      e.id = static_cast<long long>(static_cast<int32_t>(p.y));
      if (e.id < 0 || (s.exclude != nullptr && e.id == s.exclude[q])) e.key = 0;
    } else {
      e.id = s.id_base + static_cast<long long>(p.y);
    }
  } else {
    e.key = score_key(s.scores[off]);
    if (s.ids != nullptr) {
      e.id = s.ids[off];
      if (e.id < 0 || (s.exclude != nullptr && e.id == s.exclude[q])) e.key = 0;
    } else {
      e.id = s.id_base + i;
    }
  }
  return e;
}

__device__ __forceinline__ Elem load_elem(const TopkSrc& s, int q, int g, long long i) {
  return load_elem_at(s, q, list_base(s, q, g, g >= s.G ? list_len(s, q, g) : 0) + i, i);
}

constexpr int kTopkThreads = 1024;

// Phase timeline of the selection kernel (sgpt_debug_topk_timeline): thread 0 of CTA 0 stamps %globaltimer at the phase
// boundaries of every launch; the last launch's stamps stay readable.  One store per phase: no measurable cost.
__device__ unsigned long long g_topk_timeline[16];
__device__ __forceinline__ unsigned long long timeline_now() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void timeline_mark(int slot) {
  if (blockIdx.x == 0 && threadIdx.x == 0) g_topk_timeline[slot] = timeline_now();
}
__device__ __forceinline__ void timeline_set(int slot, unsigned long long t) {
  if (blockIdx.x == 0 && threadIdx.x == 0) g_topk_timeline[slot] = t;
}

// Sum of `v` over the 1024 threads of the CTA, returned to every thread; ONE barrier per call (scratch double-buffered by
// call parity: a buffer is rewritten two calls later, i.e. after the barrier of the call in between).
__device__ __forceinline__ uint32_t block_sum(uint32_t v, uint32_t (*buf)[32], uint32_t& parity, int lane, int warp) {
  v = __reduce_add_sync(0xffffffffu, v);
  if (lane == 0) buf[parity][warp] = v;
  __syncthreads();
  const uint32_t t = __reduce_add_sync(0xffffffffu, buf[parity][lane]);
  parity ^= 1u;
  return t;
}
// two sums at once (same single barrier)
__device__ __forceinline__ uint2 block_sum2(uint32_t a, uint32_t b, uint2 (*buf)[32], uint32_t& parity, int lane, int warp) {
  a = __reduce_add_sync(0xffffffffu, a);
  b = __reduce_add_sync(0xffffffffu, b);
  if (lane == 0) buf[parity][warp] = make_uint2(a, b);
  __syncthreads();
  const uint2 t = buf[parity][lane];
  parity ^= 1u;
  return make_uint2(__reduce_add_sync(0xffffffffu, t.x), __reduce_add_sync(0xffffffffu, t.y));
}

// One radix-4 step of the bitwise search for the rank-th largest key: with `pv` fixed above bit b+1, the counts of keys
// >= pv|1<<b, >= pv|2<<b, >= pv|3<<b decide two bits per block-wide reduction (n1 and n2 travel packed in one word: both
// are <= 49152 < 2^16).  NK keys per thread in registers.
template <int NK>
__device__ __forceinline__ uint32_t radix4_step(const uint32_t (&kr)[NK], uint32_t pv, int b, uint32_t rank, uint2 (*buf)[32],
                                                uint32_t& parity, int lane, int warp) {
  const uint32_t c1 = pv | (1u << b), c2 = pv | (2u << b), c3 = pv | (3u << b);
  uint32_t n12 = 0, n3 = 0;
#pragma unroll
  for (int i = 0; i < NK; ++i) {
    n12 += (kr[i] >= c1 ? 1u : 0u) + (kr[i] >= c2 ? 0x10000u : 0u);
    n3 += (kr[i] >= c3 ? 1u : 0u);
  }
  const uint2 t = block_sum2(n12, n3, buf, parity, lane, warp);
  const uint32_t n1 = t.x & 0xffffu, n2 = t.x >> 16;
  if (t.y >= rank) return c3;
  if (n2 >= rank) return c2;
  if (n1 >= rank) return c1;
  return pv;
}

constexpr int kBins = 2048;

constexpr int kMaxFlatLists = 1024;
constexpr int kSubCap = 8192;  // cached mode: keys sharing the k-th key's first radix digit are compacted into smem

// Visit every element of query q's lists: f(g, i, valid).  With at most kMaxFlatLists lists (always, in practice) the
// lists are laid end to end in a flat index space — each padded to a multiple of 32 so that the 32 lanes of a warp are
// always inside the same list — and all 1024 threads stride that space; the list of a flat index is found by binary
// search in the shared prefix array `off`.  This keeps every thread busy for one long list (dense rows), a few
// (cross-shard merges) or hundreds of short ones (the per-(CTA, half) candidate lists of the fused search).
// kPad also visits the padding (valid = false) so that warps stay converged for __match_any_sync.
template <bool kPad, class F>
__device__ __forceinline__ void for_each_elem(const TopkSrc& s, int nl, int q, int tid, const uint32_t* off,
                                              const uint32_t* len, F&& f) {
  if (nl <= kMaxFlatLists) {
    const uint32_t total = off[nl];
    for (uint32_t j = tid; j < total; j += kTopkThreads) {
      int lo = 0, hi = nl;
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (off[mid] <= j) lo = mid; else hi = mid;
      }
      const uint32_t i = j - off[lo];
      const bool valid = i < len[lo];
      if (kPad || valid) f(lo, static_cast<long long>(i), valid);
    }
  } else {
    for (int g = 0; g < nl; ++g) {
      const long long n = list_len(s, q, g);
      const long long end = kPad ? ((n + 31) & ~31ll) : n;
      for (long long i = tid; i < end; i += kTopkThreads) f(g, i, i < n);
    }
  }
}

// Final outputs of a selection: skey[i] / sid[i], i < k, hold the winners in order (key 0 = empty slot).  fp32 scores + int64
// ids and/or the packed 8-byte entries written to this rank's buffer and the peers' gather buffers (16-byte-aligned rows;
// over NVLink for peer-mapped destinations), then one system-scope release per destination.  Called by ALL threads.
__device__ __forceinline__ void write_topk_outputs(int q, int k, const uint32_t* skey, const long long* sid,
                                                   float* __restrict__ out_scores, long long* __restrict__ out_ids,
                                                   const TopkExtra& extra, int tid) {
  if (out_scores != nullptr) {
    for (int i = tid; i < k; i += kTopkThreads) {
      const uint32_t key = skey[i];
      out_scores[static_cast<size_t>(q) * k + i] = key ? key_score(key) : -INFINITY;
      out_ids[static_cast<size_t>(q) * k + i] = key ? sid[i] : -1;
    }
  }
  if (extra.n_dst > 0) {
    for (int p = 0; p < extra.n_dst; ++p) {
      uint2* row = extra.dst[p] + (static_cast<size_t>(extra.dst_slot) * extra.dst_nq + q) * k;
      for (int i = tid; i < k; i += kTopkThreads) {
        const uint32_t key = skey[i];
        row[i] = key ? make_uint2(__float_as_uint(key_score(key)), static_cast<uint32_t>(static_cast<int32_t>(sid[i])))
                     : make_uint2(0xff800000u, 0xffffffffu);  // (-inf, -1)
      }
    }
    __syncthreads();
    if (tid == 0) {
      __threadfence_system();
      for (int p = 0; p < extra.n_dst; ++p)
        if (extra.flag[p] != nullptr)
          asm volatile("red.release.sys.global.add.u32 [%0], 1;" ::"l"(extra.flag[p] + q) : "memory");
    }
  }
}

// sorted[] / sorted_id[]: KP (power of two >= k) slots in dynamic smem
// ckeys[]: when the flat (padded) index space of the query fits `cache_keys` entries of dynamic smem behind the sort
// buffers, every key is fetched from global memory ONCE (one warp per list, several loads in flight) and the three
// histogram passes and the winner scan run out of shared memory; otherwise every pass re-reads global memory.
__global__ void __launch_bounds__(kTopkThreads, 1) topk_select_kernel(TopkSrc src, int k, int KP, uint32_t cache_keys,
                                                                   float* __restrict__ out_scores,
                                                                   long long* __restrict__ out_ids, TopkExtra extra) {
  extern __shared__ uint8_t dsm[];
  uint32_t* skey = reinterpret_cast<uint32_t*>(dsm);
  long long* sid = reinterpret_cast<long long*>(dsm + static_cast<size_t>(KP) * 4);
  uint32_t* sub_key = reinterpret_cast<uint32_t*>(dsm + static_cast<size_t>(KP) * 12);  // survivors of the first digit
  uint32_t* ckeys = sub_key + kSubCap;
  __shared__ uint32_t s_sub_n;
  __shared__ uint32_t hist[kBins];
  __shared__ uint32_t warp_tot[32];
  __shared__ uint32_t s_off[kMaxFlatLists + 1];  // padded list offsets in the flat index space
  __shared__ uint32_t s_len[kMaxFlatLists];
  __shared__ uint32_t s_bin, s_need, s_cnt_gt, s_cnt_eq;
  __shared__ uint32_t s_total;  // < 2^32 (checked by the launcher)
  __shared__ uint32_t s_red[2][32];
  __shared__ uint2 s_red2[2][32];

  const int q = blockIdx.x;
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;

  const unsigned long long t_entry = timeline_now();
  pdl_sync();  // programmatic dependent launch: see common.cuh
  // two-pass search: the front-list kernel (front_select_kernel) has already answered this query
  if (src.run_flag != nullptr && src.run_flag[q] == 0) return;  // (block-uniform)
  timeline_set(0, t_entry);
  timeline_mark(1);
  if (src.wait_flag != nullptr) {
    // cross-GPU gather: the lists of this query are complete once every rank has signalled (topk.cuh TopkExtra::flag)
    if (tid == 0) {
      unsigned int v, polls = 0;
      do {
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(src.wait_flag + q) : "memory");
        if (static_cast<int>(v - src.wait_target) >= 0) break;
        if (++polls > (1u << 26)) {
          printf("sgpt: cross-GPU gather timed out (query %d: flag %u, waiting for %u)\n", q, v, src.wait_target);
          __trap();
        }
        __nanosleep(64);
      } while (true);
    }
    __syncthreads();
  }
  uint32_t red_par = 0;
  // Two-sided candidate lists (topk.cuh TopkSrc::counts_back): the front parts hold the scores above the search's upper
  // threshold; when they alone contain k entries the back parts cannot contribute a winner and are never touched.
  int nl = src.G;  // lists this selection reads
  uint32_t len_pre = 0;  // length of list `tid` (front parts, then back parts), fetched in ONE round of loads
  if (src.counts_back != nullptr) {
    if (tid < 2 * src.G) len_pre = static_cast<uint32_t>(list_len(src, q, tid));
    uint32_t f = (tid < src.G) ? len_pre : 0u;
    for (int g = tid + kTopkThreads; g < src.G; g += kTopkThreads) f += static_cast<uint32_t>(list_len(src, q, g));
    if (block_sum(f, s_red, red_par, lane, warp) < static_cast<uint32_t>(k)) nl = 2 * src.G;
  }
  timeline_mark(2);
  const bool pk_local = (src.packed != nullptr) && !src.packed_global;  // every stored entry is valid
  // flat index space over the lists: s_len[g], s_off[g] = sum of the padded lengths of lists < g (block-wide scan)
  uint32_t sum_len = 0;
  if (nl <= kMaxFlatLists) {
    const uint32_t mylen = (tid >= nl) ? 0u
                           : (src.counts_back != nullptr) ? len_pre : static_cast<uint32_t>(list_len(src, q, tid));
    const uint32_t mypad = (mylen + 31u) & ~31u;
    uint32_t incl = mypad;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) warp_tot[warp] = incl;
    sum_len = __reduce_add_sync(0xffffffffu, mylen);
    if (lane == 0) s_red[red_par][warp] = sum_len;  // (the barrier below serves both reductions)
    __syncthreads();
    sum_len = __reduce_add_sync(0xffffffffu, s_red[red_par][lane]);
    red_par ^= 1u;
    uint32_t base = 0;
    for (int w = 0; w < warp; ++w) base += warp_tot[w];
    if (tid < nl) {
      s_len[tid] = mylen;
      s_off[tid + 1] = base + incl;
    }
    if (tid == 0) s_off[0] = 0;
  }
  // number of valid elements (needed to cap k)
  if (tid == 0) s_total = 0;
  __syncthreads();
  timeline_mark(3);
  const bool cached = (nl <= kMaxFlatLists) && (s_off[nl <= kMaxFlatLists ? nl : 0] <= cache_keys);
  const uint32_t flat_total = cached ? s_off[nl] : 0u;
  if (cached) {
    // One warp per list, THREE lists per warp iteration with all their loads issued before the first store: the phase is
    // a chain of L2 round trips (hundreds of short lists per query), so lists in flight are what shortens it.  Lists of
    // at most 128 packed entries — the normal case of the fused search — are fetched as two 16-byte loads per lane.
    for (int g0 = warp; g0 < nl; g0 += 3 * (kTopkThreads / 32)) {
      uint32_t len[3], base[3];
      long long lb[3];
      bool fast = pk_local;
#pragma unroll
      for (int u = 0; u < 3; ++u) {
        const int g = g0 + u * (kTopkThreads / 32);
        len[u] = (g < nl) ? s_len[g] : 0u;
        base[u] = (g < nl) ? s_off[g] : 0u;
        lb[u] = (g < nl) ? list_base(src, q, g, len[u]) : 0ll;
        fast = fast && len[u] <= 128u && (lb[u] & 1ll) == 0;
      }
      if (fast) {
        uint4 v[3][2];
#pragma unroll
        for (int u = 0; u < 3; ++u)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint32_t idx = 2u * lane + 64u * h;
            v[u][h] = (idx < len[u]) ? *reinterpret_cast<const uint4*>(src.packed + lb[u] + idx) : make_uint4(0u, 0u, 0u, 0u);
          }
#pragma unroll
        for (int u = 0; u < 3; ++u)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint32_t idx = 2u * lane + 64u * h;
            if (idx < ((len[u] + 31u) & ~31u))
              *reinterpret_cast<uint2*>(&ckeys[base[u] + idx]) =
                  make_uint2(idx < len[u] ? score_key(__uint_as_float(v[u][h].x)) : 0u,
                             idx + 1u < len[u] ? score_key(__uint_as_float(v[u][h].z)) : 0u);
          }
      } else {
#pragma unroll
        for (int u = 0; u < 3; ++u) {
          const uint32_t end = (len[u] + 31u) & ~31u;
#pragma unroll 4
          for (uint32_t i = lane; i < end; i += 32)
            ckeys[base[u] + i] = (i < len[u]) ? load_elem_at(src, q, lb[u] + i, i).key : 0u;
        }
      }
    }
    __syncthreads();
  }
  uint32_t total;
  if (pk_local && nl <= kMaxFlatLists) {
    total = sum_len;
  } else {
    uint32_t local = 0;
    if (cached) {
      for (uint32_t j = tid; j < flat_total; j += kTopkThreads) local += (ckeys[j] != 0);
    } else if (src.ids == nullptr && src.packed == nullptr) {
      for (int g = tid; g < nl; g += kTopkThreads) local += static_cast<uint32_t>(list_len(src, q, g));
    } else {
      for_each_elem<false>(src, nl, q, tid, s_off, s_len, [&](int g, long long i, bool) { local += (load_elem(src, q, g, i).key != 0); });
    }
    local = __reduce_add_sync(0xffffffffu, local);  // 64-bit shared atomics are CAS loops: one 32-bit add per warp
    if (lane == 0 && local) atomicAdd(&s_total, local);
    __syncthreads();
    total = s_total;
  }
  timeline_mark(4);
  const uint32_t kk = total < static_cast<uint32_t>(k) ? total : static_cast<uint32_t>(k);

  uint32_t prefix = 0, mask = 0, need = kk;
  uint32_t sub_n = 0;
  bool use_sub = false;  // digits 2 and 3 run over the compacted survivors of digit 1 instead of all keys
  // ---- fast path (all keys cached in shared memory) ------------------------------------------------------------------
  // Histogram passes cost ~3 shared-memory atomics / warp-matches per key.  Instead: (1) a 1024-key strided SAMPLE (one key per thread) gives, by a 32-round bitwise
  // search with block-wide counts, a pivot `lo` that is below the k-th largest key with overwhelming probability but
  // keeps only a few k / n of the keys; (2) ONE pass compacts the keys >= lo (with their flat positions) into a short
  // list and counts them — the count proves the pivot valid, otherwise the histogram path below takes over; (3) the
  // exact k-th key is found by the same bitwise search on the short list (<= 4 keys per thread, in registers).
  uint2* sub_kj = reinterpret_cast<uint2*>(sub_key);  // (key, flat index) pairs, kSubCap / 2 entries
  constexpr uint32_t kSubPairs = kSubCap / 2;
  bool fast_done = false;
  if (cached && kk > 0) {
    uint32_t lo_key = 1u;  // smallest valid key: keeps everything
    if (total > kSubPairs) {
      const uint32_t step = flat_total / kTopkThreads;  // >= 1 here (flat_total >= total > 4096)
      const uint32_t skeyv = ckeys[static_cast<uint32_t>(tid) * step];
      // expected rank of the k-th key inside the sample, plus ~4 sigma of the sampling noise
      const float er = static_cast<float>(kk) * static_cast<float>(kTopkThreads) / static_cast<float>(total);
      const uint32_t rank = static_cast<uint32_t>(er + 4.0f * sqrtf(er) + 4.0f);
      if (rank < static_cast<uint32_t>(kTopkThreads)) {
        // (the low 12 bits stay zero: a pivot up to 2^-11 (relative) lower keeps a handful of extra keys, nothing else)
        uint32_t pv = 0;
        const uint32_t sk1[1] = {skeyv};
#pragma unroll 1
        for (int b = 30; b >= 12; b -= 2) pv = radix4_step<1>(sk1, pv, b, rank, s_red2, red_par, lane, warp);
        lo_key = pv > 0u ? pv : 1u;  // (a lower bound of) the rank-th largest sampled key
      }
    }
    timeline_mark(5);
    // (2) compaction of the keys >= lo_key
    if (tid == 0) s_sub_n = 0;
    __syncthreads();
    for (uint32_t j0 = 0; j0 < flat_total; j0 += kTopkThreads) {  // flat_total is a multiple of 32: warps stay converged
      const uint32_t j = j0 + tid;
      const uint32_t key = (j < flat_total) ? ckeys[j] : 0u;
      const bool keep = key >= lo_key && key != 0u;
      const uint32_t m = __ballot_sync(0xffffffffu, keep);
      if (m != 0u) {
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(&s_sub_n, __popc(m));
        base = __shfl_sync(0xffffffffu, base, 0);
        const uint32_t slot = base + __popc(m & ((1u << lane) - 1u));
        if (keep && slot < kSubPairs) sub_kj[slot] = make_uint2(key, j);
      }
    }
    __syncthreads();
    sub_n = s_sub_n;
    timeline_mark(6);
    if (sub_n >= kk && sub_n <= kSubPairs) {
      // (3) exact kk-th largest key of the short list: <= 4 keys per thread in registers
      uint32_t kr[kSubPairs / kTopkThreads];  // (kSubPairs / kTopkThreads = 4)
#pragma unroll
      for (uint32_t i = 0; i < kSubPairs / kTopkThreads; ++i) {
        const uint32_t e = tid + i * kTopkThreads;
        kr[i] = e < sub_n ? sub_kj[e].x : 0u;
      }
      uint32_t pv = 0;
#pragma unroll 1
      for (int b = 30; b >= 0; b -= 2) pv = radix4_step<kSubPairs / kTopkThreads>(kr, pv, b, kk, s_red2, red_par, lane, warp);
      prefix = pv;
      uint32_t cgt = 0;
#pragma unroll
      for (uint32_t i = 0; i < kSubPairs / kTopkThreads; ++i) cgt += (kr[i] > pv) ? 1u : 0u;
      need = kk - block_sum(cgt, s_red, red_par, lane, warp);  // winners among the keys equal to the kk-th key
      fast_done = true;
    }
  }
  if (kk > 0 && !fast_done) {
    const int shifts[3] = {21, 10, 0};
    const uint32_t widths[3] = {11, 11, 10};
#pragma unroll 1
    for (int pass = 0; pass < 3; ++pass) {
      const int shift = shifts[pass];
      const uint32_t bmask = (1u << widths[pass]) - 1u;
      for (int i = tid; i < kBins; i += kTopkThreads) hist[i] = 0;
      __syncthreads();
      auto tally = [&](uint32_t key) {  // executed by converged warps
        const bool ok = (key != 0) && ((key & mask) == prefix);
        const uint32_t bin = ok ? ((key >> shift) & bmask) : 0xffffffffu;
        const uint32_t peers = __match_any_sync(0xffffffffu, bin);
        if (ok && lane == (__ffs(peers) - 1)) atomicAdd(&hist[bin], __popc(peers));
      };
      if (use_sub) {
        for (uint32_t j = tid; j < ((sub_n + 31u) & ~31u); j += kTopkThreads) tally(j < sub_n ? sub_key[j] : 0u);
      } else if (cached) {
        for (uint32_t j = tid; j < flat_total; j += kTopkThreads) tally(ckeys[j]);
      } else {
        for_each_elem<true>(src, nl, q, tid, s_off, s_len, [&](int g, long long i, bool valid) {
          tally(valid ? load_elem(src, q, g, i).key : 0u);
        });
      }
      __syncthreads();
      // suffix scan over bins: thread t owns bins 2t, 2t+1
      const uint32_t h0 = hist[2 * tid], h1 = hist[2 * tid + 1];
      const uint32_t c = h0 + h1;
      uint32_t incl = c;  // inclusive suffix within the warp (higher lanes = higher bins)
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_down_sync(0xffffffffu, incl, o);
        if (lane + o < 32) incl += v;
      }
      if (lane == 0) warp_tot[warp] = incl;
      __syncthreads();
      uint32_t above = incl - c;  // elements in higher bins of this warp
      for (int w = warp + 1; w < 32; ++w) above += warp_tot[w];
      if (above < need && need <= above + c) {
        if (above + h1 >= need) {
          s_bin = 2 * tid + 1;
          s_need = need - above;
        } else {
          s_bin = 2 * tid;
          s_need = need - above - h1;
        }
      }
      __syncthreads();
      prefix |= s_bin << shift;
      mask |= bmask << shift;
      need = s_need;
      if (pass == 0 && cached) {
        // compact the keys that share the selected first digit (typically a few hundred to a few thousand)
        if (tid == 0) s_sub_n = 0;
        __syncthreads();
        for (uint32_t j = tid; j < flat_total; j += kTopkThreads) {
          const uint32_t key = ckeys[j];
          if (key != 0 && (key & mask) == prefix) {
            const uint32_t slot = atomicAdd(&s_sub_n, 1u);
            if (slot < kSubCap) sub_key[slot] = key;
          }
        }
        __syncthreads();
        sub_n = s_sub_n;
        use_sub = sub_n <= kSubCap;
      }
      __syncthreads();
    }
  }
  timeline_mark(7);
  // prefix == key of the kk-th largest element; `need` of the elements equal to it are winners.
  if (tid == 0) { s_cnt_gt = 0; s_cnt_eq = 0; }
  for (int i = tid; i < KP; i += kTopkThreads) { skey[i] = 0; sid[i] = -1; }
  __syncthreads();
  if (kk > 0) {
    const uint32_t n_gt = kk - need;
    auto place = [&](uint32_t key, int g, long long i) {  // winners only: fetch the id
      if (key > prefix) {
        const uint32_t slot = atomicAdd(&s_cnt_gt, 1u);
        skey[slot] = key;
        sid[slot] = load_elem(src, q, g, i).id;
      } else {
        const uint32_t s = atomicAdd(&s_cnt_eq, 1u);
        if (s < need) {
          skey[n_gt + s] = key;
          sid[n_gt + s] = load_elem(src, q, g, i).id;
        }
      }
    };
    if (fast_done) {
      // winners come from the short list; their ids are fetched afterwards by ONE thread per winner
      for (uint32_t e = tid; e < sub_n; e += kTopkThreads) {
        const uint2 kj = sub_kj[e];
        if (kj.x > prefix) {
          const uint32_t slot = atomicAdd(&s_cnt_gt, 1u);
          skey[slot] = kj.x;
          sid[slot] = static_cast<long long>(kj.y);  // flat position for now
        } else if (kj.x == prefix) {
          const uint32_t e2 = atomicAdd(&s_cnt_eq, 1u);
          if (e2 < need) {
            skey[n_gt + e2] = kj.x;
            sid[n_gt + e2] = static_cast<long long>(kj.y);
          }
        }
      }
      __syncthreads();
      for (uint32_t t = tid; t < kk; t += kTopkThreads) {
        const uint32_t j = static_cast<uint32_t>(sid[t]);
        int lo = 0, hi = nl;
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          if (s_off[mid] <= j) lo = mid; else hi = mid;
        }
        sid[t] = load_elem(src, q, lo, static_cast<long long>(j - s_off[lo])).id;
      }
    } else if (cached) {
      for (uint32_t j = tid; j < flat_total; j += kTopkThreads) {
        const uint32_t key = ckeys[j];
        if (key == 0 || key < prefix) continue;
        int lo = 0, hi = nl;
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          if (s_off[mid] <= j) lo = mid; else hi = mid;
        }
        place(key, lo, static_cast<long long>(j - s_off[lo]));
      }
    } else {
      for_each_elem<false>(src, nl, q, tid, s_off, s_len, [&](int g, long long i, bool) {
        const uint32_t key = load_elem(src, q, g, i).key;
        if (key != 0 && key >= prefix) place(key, g, i);
      });
    }
  }
  __syncthreads();
  timeline_mark(8);
  // bitonic sort, descending by key then ascending by id (skipped when only the threshold / unordered seeds are wanted).
  // KP <= 1024: one element per thread; partners closer than a warp are exchanged with shuffles (40 of the 55 stages at
  // KP = 1024 need no barrier), the others through the sort buffers.
  const bool want_sort = (out_scores != nullptr || extra.n_dst > 0);
  if (want_sort && KP <= kTopkThreads) {
    uint32_t ka = (tid < KP) ? skey[tid] : 0u;
    long long ia = (tid < KP) ? sid[tid] : -1;
    for (int size = 2; size <= KP; size <<= 1) {
      const bool desc = ((tid & size) == 0);
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        uint32_t kb;
        long long ib;
        if (stride >= 32) {
          __syncthreads();  // the previous round's readers are done
          if (tid < KP) { skey[tid] = ka; sid[tid] = ia; }
          __syncthreads();
          const int pt = tid ^ stride;
          kb = (tid < KP) ? skey[pt] : 0u;
          ib = (tid < KP) ? sid[pt] : -1;
        } else {
          kb = __shfl_xor_sync(0xffffffffu, ka, stride);
          const uint32_t lo32 = __shfl_xor_sync(0xffffffffu, static_cast<uint32_t>(ia), stride);
          const uint32_t hi32 = __shfl_xor_sync(0xffffffffu, static_cast<uint32_t>(static_cast<unsigned long long>(ia) >> 32), stride);
          ib = static_cast<long long>((static_cast<unsigned long long>(hi32) << 32) | lo32);
        }
        const bool is_lo = (tid & stride) == 0;
        const bool mine_first = (ka > kb) || (ka == kb && ia <= ib);  // "mine before the partner's" in descending order
        // the lower index keeps the element that comes first in a descending run, the last in an ascending run
        if (mine_first != (is_lo == desc)) { ka = kb; ia = ib; }
      }
    }
    __syncthreads();
    if (tid < KP) { skey[tid] = ka; sid[tid] = ia; }
    __syncthreads();
  }
  for (int size = 2; size <= KP && want_sort && KP > kTopkThreads; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < KP / 2; i += kTopkThreads) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool desc = ((lo & size) == 0);
        const uint32_t ka = skey[lo], kb = skey[hi];
        const long long ia = sid[lo], ib = sid[hi];
        // "a before b" in the desired descending order
        const bool a_first = (ka > kb) || (ka == kb && ia <= ib);
        if (a_first != desc) {
          skey[lo] = kb; skey[hi] = ka;
          sid[lo] = ib; sid[hi] = ia;
        }
      }
      __syncthreads();
    }
  }
  timeline_mark(9);
  write_topk_outputs(q, k, skey, sid, out_scores, out_ids, extra, tid);
  // optional side outputs for the two-pass search: winners re-packed as the head of another candidate list, and the
  // k-th best score as that query's admission threshold
  if (extra.packed != nullptr) {
    for (int i = tid; i < static_cast<int>(kk); i += kTopkThreads)
      extra.packed[static_cast<long long>(q) * extra.cap + i] =
          make_uint2(__float_as_uint(key_score(skey[i])), static_cast<uint32_t>(sid[i] - src.id_base));
    if (tid == 0) extra.count[q] = static_cast<int>(kk);
  }
  if (extra.tau != nullptr && tid == 0)
    extra.tau[q] = (kk >= static_cast<uint32_t>(k)) ? key_score(prefix) : -INFINITY;  // key of the k-th best
  timeline_mark(10);
}

// ---------------------------------------------------------------------------------------------------------------
// Final selection of the two-pass search for the NORMAL case: the front parts of a query's candidate lists (the scores
// above the upper threshold, ~2.5 k per query) hold at least k and at most kFrontCap entries.  Then nothing has to be
// selected at all: the entries are packed end to end into shared memory as 64-bit composites (order key << 32 | ~local
// index: larger = earlier, ties by ascending document id), sorted by one bitonic network over 4096 slots — four per
// thread: strides 1 and 2 stay inside a thread, strides 4..64 are warp shuffles, only strides >= 128 go through shared
// memory — and the first k are the answer, ids included (no histogram, no pivot, no compaction, no second trip to global
// memory for the ids).  Queries outside that case (front parts short: the back parts are needed; or more than kFrontCap
// ties) set need_generic[q] and are answered by topk_select_kernel, which is launched right behind with
// TopkSrc::run_flag = need_generic and returns at once for every other query.
// Loads: 4 lanes per list, 16 bytes (two entries) per lane, 256 lists of the query in flight at a time.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kFrontCap = 4096;

__device__ __forceinline__ void cx_sorted(unsigned long long& lo, unsigned long long& hi, bool desc) {
  const bool swap = desc ? (lo < hi) : (lo > hi);
  if (swap) {
    const unsigned long long t = lo;
    lo = hi;
    hi = t;
  }
}

__global__ void __launch_bounds__(kTopkThreads, 1) front_select_kernel(TopkSrc src, int k, int KP,
                                                                    float* __restrict__ out_scores,
                                                                    long long* __restrict__ out_ids, TopkExtra extra,
                                                                    int* __restrict__ need_generic) {
  extern __shared__ __align__(16) uint8_t dsm_front[];  // KP >= 4 (launcher): every region below is 16-byte aligned
  uint32_t* skey = reinterpret_cast<uint32_t*>(dsm_front);
  long long* sid = reinterpret_cast<long long*>(dsm_front + static_cast<size_t>(KP) * 4);
  unsigned long long* cbuf = reinterpret_cast<unsigned long long*>(dsm_front + static_cast<size_t>(KP) * 12);  // [kFrontCap]
  __shared__ uint32_t s_coff[kMaxFlatLists + 1];  // compact offsets of the lists (exclusive prefix of their lengths)
  __shared__ uint32_t warp_tot[32];

  const int q = blockIdx.x;
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const unsigned long long t_entry = timeline_now();
  pdl_sync();
  const unsigned long long t_dep = timeline_now();
  const int G = src.G;  // <= kMaxFlatLists (launcher)
  const uint32_t mylen = (tid < G) ? static_cast<uint32_t>(list_len(src, q, tid)) : 0u;
  uint32_t incl = mylen;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  uint32_t base = 0, total = 0;
#pragma unroll 8
  for (int w = 0; w < 32; ++w) {
    const uint32_t v = warp_tot[w];
    base += (w < warp) ? v : 0u;
    total += v;
  }
  const bool mine = total >= static_cast<uint32_t>(k) && total <= static_cast<uint32_t>(kFrontCap);  // block-uniform
  if (tid == 0) need_generic[q] = mine ? 0 : 1;
  if (!mine) return;
  timeline_set(0, t_entry);
  timeline_set(1, t_dep);
  timeline_set(2, t_dep);
  if (tid < G) s_coff[tid] = base + incl - mylen;
  if (tid == 0) s_coff[G] = total;
  for (uint32_t i = total + tid; i < static_cast<uint32_t>(kFrontCap); i += kTopkThreads) cbuf[i] = 0ull;  // sorts last
  __syncthreads();
  timeline_mark(3);
  {
    const uint32_t sl = lane & 3u;
    for (int g = warp * 8 + static_cast<int>(lane >> 2); g < G; g += (kTopkThreads / 32) * 8) {
      const uint32_t c0 = s_coff[g], len = s_coff[g + 1] - c0;
      const uint2* lst = src.packed + static_cast<long long>(g) * src.stride_g + static_cast<long long>(q) * src.stride_q;
      for (uint32_t idx = 2u * sl; idx < len; idx += 8u) {  // (the second entry of a pair may lie beyond len: unused slot of the list)
        const uint4 v = *reinterpret_cast<const uint4*>(lst + idx);
        cbuf[c0 + idx] = (static_cast<unsigned long long>(score_key(__uint_as_float(v.x))) << 32) | static_cast<uint32_t>(~v.y);
        if (idx + 1u < len)
          cbuf[c0 + idx + 1u] = (static_cast<unsigned long long>(score_key(__uint_as_float(v.z))) << 32) | static_cast<uint32_t>(~v.w);
      }
    }
  }
  __syncthreads();
  timeline_mark(4);
  timeline_mark(5);
  timeline_mark(6);
  timeline_mark(7);
  timeline_mark(8);
  // ---- bitonic sort of the kFrontCap slots, descending; thread t owns slots 4 t .. 4 t + 3 ----
  unsigned long long e[4];
  {
    const ulonglong2 a = *reinterpret_cast<const ulonglong2*>(cbuf + 4 * tid);
    const ulonglong2 b = *reinterpret_cast<const ulonglong2*>(cbuf + 4 * tid + 2);
    e[0] = a.x; e[1] = a.y; e[2] = b.x; e[3] = b.y;
  }
#pragma unroll 1
  for (int size = 2; size <= kFrontCap; size <<= 1) {
    const bool desc = ((4 * tid) & size) == 0;  // direction of this thread's run (all four slots share it for size >= 4)
#pragma unroll 1
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      if (stride >= 128) {
        __syncthreads();  // the previous exchange's readers are done
        *reinterpret_cast<ulonglong2*>(cbuf + 4 * tid) = make_ulonglong2(e[0], e[1]);
        *reinterpret_cast<ulonglong2*>(cbuf + 4 * tid + 2) = make_ulonglong2(e[2], e[3]);
        __syncthreads();
        const int pt = (4 * tid) ^ stride;
        const ulonglong2 a = *reinterpret_cast<const ulonglong2*>(cbuf + pt);
        const ulonglong2 b = *reinterpret_cast<const ulonglong2*>(cbuf + pt + 2);
        const unsigned long long o[4] = {a.x, a.y, b.x, b.y};
        const bool keep_max = (((4 * tid) & stride) == 0) == desc;
#pragma unroll
        for (int r = 0; r < 4; ++r) e[r] = keep_max ? (e[r] > o[r] ? e[r] : o[r]) : (e[r] < o[r] ? e[r] : o[r]);
      } else if (stride >= 4) {
        const int lm = stride >> 2;  // partner lane = lane ^ lm
        const bool keep_max = ((lane & lm) == 0) == desc;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const uint32_t olo = __shfl_xor_sync(0xffffffffu, static_cast<uint32_t>(e[r]), lm);
          const uint32_t ohi = __shfl_xor_sync(0xffffffffu, static_cast<uint32_t>(e[r] >> 32), lm);
          const unsigned long long o = (static_cast<unsigned long long>(ohi) << 32) | olo;
          e[r] = keep_max ? (e[r] > o ? e[r] : o) : (e[r] < o ? e[r] : o);
        }
      } else if (stride == 2) {  // (size >= 4)
        cx_sorted(e[0], e[2], desc);
        cx_sorted(e[1], e[3], desc);
      } else {  // stride 1
        if (size == 2) {  // slots 4t, 4t+1: descending pair; 4t+2, 4t+3: ascending pair
          cx_sorted(e[0], e[1], true);
          cx_sorted(e[2], e[3], false);
        } else {
          cx_sorted(e[0], e[1], desc);
          cx_sorted(e[2], e[3], desc);
        }
      }
    }
  }
  __syncthreads();  // cbuf readers of the last exchange are done; skey / sid are separate arrays anyway
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int i = 4 * tid + r;
    if (i < KP) {
      const uint32_t key = static_cast<uint32_t>(e[r] >> 32);
      skey[i] = key;
      sid[i] = key ? src.id_base + static_cast<long long>(~static_cast<uint32_t>(e[r])) : -1;
    }
  }
  __syncthreads();
  timeline_mark(9);
  write_topk_outputs(q, k, skey, sid, out_scores, out_ids, extra, tid);
  timeline_mark(10);
}

// Launch of the front-list kernel; *taken = false when the source does not qualify (then only the generic kernel runs).
int launch_front_select(const TopkSrc& src, int nq, int k, float* out_scores, int64_t* out_ids, cudaStream_t stream,
                        const TopkExtra& extra, int* need_generic, bool* taken) {
  *taken = false;
  if (src.packed == nullptr || src.packed_global || src.counts == nullptr || src.counts_back == nullptr ||
      src.G > kMaxFlatLists || (src.stride_g & 1) != 0 || (src.stride_q & 1) != 0 || k <= 0 || k > kFrontCap ||
      need_generic == nullptr)
    return SGPT_OK;
  // OFF by default: sorting all 4096 slots is 78 compare-exchange stages over 4 slots per thread, against compaction + exact
  // k-th key + placing + sorting only the 1024 winners in the generic kernel.  SGPT_FRONT_SELECT=1 (read per call) keeps it
  // testable.
  {
    const char* e = getenv("SGPT_FRONT_SELECT");
    if (!(e != nullptr && e[0] == '1')) return SGPT_OK;
  }
  int KP = 4;
  while (KP < k) KP <<= 1;
  const size_t dsm = static_cast<size_t>(KP) * 12 + static_cast<size_t>(kFrontCap) * 8;
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    SGPT_CHECK_CUDA(cudaFuncSetAttribute(front_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
  }
  LaunchScope _ls(kCatTopk, stream);
  SGPT_CHECK_CUDA(launch_kernel(front_select_kernel, dim3(nq), dim3(kTopkThreads), dsm, stream, src, k, KP, out_scores,
                                reinterpret_cast<long long*>(out_ids), extra, need_generic));
  *taken = true;
  return SGPT_OK;
}

// Admission thresholds of the two-pass search (search.cu) from the sampled block maxima (gemm.cuh EpiFilterRows, sample
// mode): tau_lo[q] = a lower bound, tight to 2^-11 relative, of the k-th largest of the `total` floats at pool + q *
// stride_q (0xffffffff = unused slot), tau_hi[q] the same for rank k_hi <= k; -inf when fewer than k (k_hi) are valid.
// All keys of a query live in registers (<= 12 per thread), so each threshold is ten block-wide radix-4 counting steps
// and nothing else: no histogram, no compaction, no winners, no sort — the sample is only ever used for its thresholds.
constexpr int kTauKeys = 12;
static_assert(kTauKeys * kTopkThreads == kMaxTauSample, "topk.cuh kMaxTauSample");

__global__ void __launch_bounds__(kTopkThreads, 1) tau_select_kernel(const float* __restrict__ pool, long long stride_q,
                                                                  int total, int k, int k_hi, float* __restrict__ tau_lo,
                                                                  float* __restrict__ tau_hi) {
  __shared__ uint32_t s_red[2][32];
  __shared__ uint2 s_red2[2][32];
  const int q = blockIdx.x;
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  pdl_sync();
  const uint4* src = reinterpret_cast<const uint4*>(pool + static_cast<long long>(q) * stride_q);
  const int n4 = total >> 2;
  uint32_t kr[kTauKeys];
  uint32_t valid = 0;
#pragma unroll
  for (int i = 0; i < kTauKeys / 4; ++i) {
    const int j = tid + i * kTopkThreads;
    const uint4 v = (j < n4) ? __ldg(src + j) : make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu);
    kr[4 * i] = score_key(__uint_as_float(v.x));
    kr[4 * i + 1] = score_key(__uint_as_float(v.y));
    kr[4 * i + 2] = score_key(__uint_as_float(v.z));
    kr[4 * i + 3] = score_key(__uint_as_float(v.w));
  }
#pragma unroll
  for (int i = 0; i < kTauKeys; ++i) valid += (kr[i] != 0u) ? 1u : 0u;
  uint32_t red_par = 0;
  const uint32_t n_valid = block_sum(valid, s_red, red_par, lane, warp);
#pragma unroll 1
  for (int t = 0; t < 2; ++t) {
    const uint32_t rank = static_cast<uint32_t>(t == 0 ? k : k_hi);
    float* out = (t == 0) ? tau_lo : tau_hi;
    if (out == nullptr) continue;  // (block-uniform)
    uint32_t pv = 0;
    if (n_valid >= rank) {  // (block-uniform)
#pragma unroll 1
      for (int b = 30; b >= 12; b -= 2) pv = radix4_step<kTauKeys>(kr, pv, b, rank, s_red2, red_par, lane, warp);
    }
    // pv = the largest key with 12 zero low bits that at least `rank` keys reach: <= the rank-th largest key
    if (tid == 0) out[q] = pv != 0u ? key_score(pv) : -INFINITY;
  }
}

int launch_tau_select(const float* pool, long long stride_q, int total, int nq, int k, int k_hi, float* tau_lo,
                      float* tau_hi, cudaStream_t stream) {
  if (total <= 0 || (total & 7) != 0 || total > kMaxTauSample || (stride_q & 3) != 0 || k_hi < 1 || k_hi > k) {
    set_error("tau select: %d sampled maxima per query (must be a multiple of 8, at most %d), ranks %d / %d", total,
              kMaxTauSample, k, k_hi);
    return SGPT_ERR_INVALID;
  }
  LaunchScope _ls(kCatTopk, stream);
  SGPT_CHECK_CUDA(launch_kernel(tau_select_kernel, dim3(nq), dim3(kTopkThreads), 0, stream, pool, stride_q, total, k, k_hi,
                                tau_lo, tau_hi));
  return SGPT_OK;
}

// S3 for lists that are already SORTED (the packed per-shard results of sgpt_search_packed / the peer gather buffers:
// descending score, ascending id on ties, empty slots (-inf, -1) at the tail): no selection and no sort — the final
// position of an entry is the number of entries that precede it, i.e. its index in its own list plus one binary search
// per other list; entries whose position is below k are written straight to that position.  All lists of a query are
// staged in shared memory as 64-bit composites (order key << 32 | ~id: larger = earlier; 0 = empty slot); the self-match
// (exclude[q], XS:118) is found while staging and every entry it precedes moves up by one.  One CTA per query.
__global__ void __launch_bounds__(kTopkThreads, 1) merge_sorted_kernel(TopkSrc src, int k, float* __restrict__ out_scores,
                                                                    long long* __restrict__ out_ids) {
  extern __shared__ uint8_t dsm[];
  unsigned long long* comp = reinterpret_cast<unsigned long long*>(dsm);  // [G][L]
  __shared__ unsigned long long s_excl;  // composite of the excluded entry (0 = none among the lists)
  __shared__ uint32_t s_red[2][32];
  const int q = blockIdx.x;
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int G = src.G, L = static_cast<int>(src.L);
  pdl_sync();
  if (src.wait_flag != nullptr) {  // cross-GPU gather: see topk_select_kernel
    if (tid == 0) {
      unsigned int v, polls = 0;
      do {
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(src.wait_flag + q) : "memory");
        if (static_cast<int>(v - src.wait_target) >= 0) break;
        if (++polls > (1u << 26)) {
          printf("sgpt: cross-GPU gather timed out (query %d: flag %u, waiting for %u)\n", q, v, src.wait_target);
          __trap();
        }
        __nanosleep(64);
      } while (true);
    }
  }
  if (tid == 0) s_excl = 0ull;
  __syncthreads();
  const long long excl = (src.exclude != nullptr) ? src.exclude[q] : -1;
  const int total = G * L;
  uint32_t n_valid = 0;
  for (int j = tid; j < total; j += kTopkThreads) {
    const int g = j / L, i = j - g * L;
    const uint2 p = src.packed[g * src.stride_g + q * src.stride_q + i];
    const int32_t id = static_cast<int32_t>(p.y);
    unsigned long long c = 0ull;
    if (id >= 0) {
      c = (static_cast<unsigned long long>(score_key(__uint_as_float(p.x))) << 32) | static_cast<uint32_t>(~id);
      if (static_cast<long long>(id) == excl) s_excl = c;  // ids are unique across shards: at most one writer
      else ++n_valid;
    }
    comp[j] = c;
  }
  uint32_t red_par = 0;
  n_valid = block_sum(n_valid, s_red, red_par, lane, warp);  // (its barrier also publishes comp[] and s_excl)
  const unsigned long long cx = s_excl;
  for (int j = tid; j < total; j += kTopkThreads) {
    const unsigned long long c = comp[j];
    if (c == 0ull || c == cx) continue;
    const int g = j / L;
    int rank = (j - g * L) - ((cx > c) ? 1 : 0);  // entries ahead of it in its own list; the self-match does not count
    for (int h = 0; h < G && rank < k; ++h) {
      if (h == g) continue;
      // number of entries of list h that precede c: first index whose composite is <= c (descending list)
      const unsigned long long* lst = comp + h * L;
      int lo = 0, hi = L;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (lst[mid] > c) lo = mid + 1; else hi = mid;
      }
      rank += lo;
    }
    if (rank < k) {
      out_scores[static_cast<size_t>(q) * k + rank] = key_score(static_cast<uint32_t>(c >> 32));
      out_ids[static_cast<size_t>(q) * k + rank] = static_cast<long long>(static_cast<int32_t>(~static_cast<uint32_t>(c)));
    }
  }
  for (int r = static_cast<int>(n_valid) + tid; r < k; r += kTopkThreads) {  // fewer than k real entries: empty tail
    out_scores[static_cast<size_t>(q) * k + r] = -INFINITY;
    out_ids[static_cast<size_t>(q) * k + r] = -1;
  }
}

// true when the launch was taken (sorted packed global lists that fit in shared memory)
static bool launch_merge_sorted(const TopkSrc& src, int nq, int k, float* out_scores, int64_t* out_ids, cudaStream_t stream,
                                int* rc) {
  constexpr size_t kDynMax = 200 * 1024;
  const size_t bytes = static_cast<size_t>(src.G) * static_cast<size_t>(src.L) * 8;
  // Every entry pays one binary search per OTHER list, so the rank-merge beats selecting again only for a few lists.
  if (!src.lists_sorted || src.packed == nullptr || !src.packed_global || src.counts != nullptr || out_scores == nullptr ||
      out_ids == nullptr || bytes > kDynMax || src.G < 1 || src.G > 3)
    return false;
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    if (cudaFuncSetAttribute(merge_sorted_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kDynMax)) !=
        cudaSuccess) {
      cudaGetLastError();
      return false;
    }
  }
  LaunchScope _ls(kCatTopk, stream);
  const cudaError_t e = launch_kernel(merge_sorted_kernel, dim3(nq), dim3(kTopkThreads), bytes, stream, src, k, out_scores,
                                      reinterpret_cast<long long*>(out_ids));
  if (e != cudaSuccess) {
    set_error("merge_sorted_kernel: %s", cudaGetErrorString(e));
    *rc = SGPT_ERR_CUDA;
  } else {
    *rc = SGPT_OK;
  }
  return true;
}

int launch_topk_select(const TopkSrc& src, int nq, int k, float* out_scores, int64_t* out_ids, cudaStream_t stream,
                       const TopkExtra& extra) {
  if (k <= 0 || k > 4096) {
    set_error("top-k: k=%d outside [1, 4096]", k);
    return SGPT_ERR_INVALID;
  }
  if (extra.n_dst == 0 && extra.packed == nullptr && extra.tau == nullptr) {
    int rc = SGPT_OK;
    if (launch_merge_sorted(src, nq, k, out_scores, out_ids, stream, &rc)) return rc;
  }
  if (static_cast<long long>(src.G) * ((src.L + 31) & ~31ll) >= (1ll << 32)) {
    set_error("top-k: %d lists of %lld entries exceed the 2^32-entry selection space", src.G, src.L);
    return SGPT_ERR_INVALID;
  }
  if (src.counts_back != nullptr && (src.packed == nullptr || src.packed_global || src.counts == nullptr)) {
    set_error("top-k: two-sided lists need packed local entries with front counts");
    return SGPT_ERR_INVALID;
  }
  int KP = 2;
  while (KP < k) KP <<= 1;
  // dynamic smem: sort buffers (KP x 12 B) + as many cached keys as the rest of the SM's shared memory holds
  constexpr size_t kDynMax = 208 * 1024;  // 227 KB per CTA minus the kernel's static arrays
  size_t cache_keys = 0;
  if (src.G <= kMaxFlatLists) {
    const size_t want = static_cast<size_t>(src.G) * static_cast<size_t>((src.L + 31) & ~31ll);  // padded worst case
    const size_t room = (kDynMax - static_cast<size_t>(KP) * 12 - kSubCap * 4) / 4;
    cache_keys = want < room ? want : room;
  }
  const size_t dsm = static_cast<size_t>(KP) * 12 + kSubCap * 4 + cache_keys * 4;
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    SGPT_CHECK_CUDA(cudaFuncSetAttribute(topk_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(kDynMax)));
  }
  LaunchScope _ls(kCatTopk, stream);
  SGPT_CHECK_CUDA(launch_kernel(topk_select_kernel, dim3(nq), dim3(kTopkThreads), dsm, stream, src, k, KP,
                                static_cast<uint32_t>(cache_keys), out_scores, reinterpret_cast<long long*>(out_ids),
                                extra));
  return SGPT_OK;
}

}  // namespace sgpt

using namespace sgpt;

extern "C" int sgpt_debug_topk_timeline(uint64_t* stamps_ns, int n) {
  SGPT_REQUIRE(stamps_ns != nullptr && n >= 1 && n <= 16, "sgpt_debug_topk_timeline: bad arguments");
  unsigned long long h[16];
  SGPT_CHECK_CUDA(cudaDeviceSynchronize());
  SGPT_CHECK_CUDA(cudaMemcpyFromSymbol(h, g_topk_timeline, sizeof(h)));
  for (int i = 0; i < n; ++i) stamps_ns[i] = h[i];
  return SGPT_OK;
}

extern "C" int64_t sgpt_topk_workspace_bytes(int nq, int64_t n, int k) {
  (void)nq; (void)n; (void)k;
  return 256;  // selection runs entirely in shared memory; a token size keeps callers' allocation path uniform
}

extern "C" int sgpt_topk(const float* scores, int64_t lds, int nq, int64_t n, int k, int64_t id_base,
                         float* out_scores, int64_t* out_ids, void* ws, sgpt_stream_t stream_) {
  (void)ws;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(nq >= 0 && n >= 0 && lds >= n, "sgpt_topk: bad sizes nq=%d n=%lld lds=%lld", nq, (long long)n,
               (long long)lds);
  if (nq == 0) return SGPT_OK;
  TopkSrc src{};
  src.scores = scores;
  src.id_base = id_base;
  src.G = 1;
  src.nq = nq;
  src.L = n;
  src.stride_q = lds;
  return launch_topk_select(src, nq, k, out_scores, out_ids, stream);
}

extern "C" int sgpt_topk_merge(const float* in_scores, const int64_t* in_ids, int G, int nq, int k,
                               float* out_scores, int64_t* out_ids, const int64_t* exclude_ids, void* ws,
                               sgpt_stream_t stream_) {
  (void)ws;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SGPT_REQUIRE(G >= 1 && nq >= 0, "sgpt_topk_merge: bad sizes G=%d nq=%d", G, nq);
  if (nq == 0) return SGPT_OK;
  TopkSrc src{};
  src.scores = in_scores;
  src.ids = reinterpret_cast<const long long*>(in_ids);
  src.exclude = reinterpret_cast<const long long*>(exclude_ids);
  src.G = G;
  src.nq = nq;
  src.L = k;
  src.stride_g = static_cast<long long>(nq) * k;
  src.stride_q = k;
  return launch_topk_select(src, nq, k, out_scores, out_ids, stream);
}
