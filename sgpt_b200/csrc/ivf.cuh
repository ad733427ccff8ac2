// Pieces of the IVF search (ivf.cu) that the IVF-PQ search (ivfpq.cu) shares: the clamped list range, the per-pair
// candidate counts and the selection over the per-pair candidate lists.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sgpt {

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

// Entries per candidate list of a (query, probe) pair: max_list_len rounded up to even, at least 2 (slot 0 of every list
// is then 16-byte aligned, so the scans write two slots per 16-byte store).
inline int64_t ivf_list_stride(int64_t max_list_len) { return max_list_len < 2 ? 2 : (max_list_len + 1) & ~int64_t(1); }

// counts[p * nb + q] = the clamped length of query q's p-th probed list (0 for a skipped probe), for the nb queries whose
// probes start at `probes`; with hist != nullptr also hist[l] += the number of pairs with a non-empty list l (hist zeroed
// by the caller).
int launch_ivf_counts(const int32_t* probes, const int64_t* offsets, int nlist, int n, long long max_len, int nb,
                      int nprobe, int* counts, int* hist, cudaStream_t stream);

// Top-k of nb queries over their nprobe candidate lists cand[(q * nprobe + p) * Ls ...] of (score bits, int32 global id)
// entries, counts as launch_ivf_counts writes them: score descending, ties by ascending global id, tail (-inf, -1).
int launch_ivf_select(const uint2* cand, const int* counts, int nb, int nprobe, long long Ls, int k, float* out_scores,
                      int64_t* out_ids, cudaStream_t stream);

}  // namespace sgpt
