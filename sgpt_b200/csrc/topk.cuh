// Source descriptor for the top-k selection kernel (topk.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sgpt {

// The order-preserving 32-bit image of an fp32 score that every selection sorts by (larger key = better score).
// -0.0 takes the key of +0.0: equal scores, so their order is decided by the ids like any other tie
__device__ __forceinline__ uint32_t score_key(float x) {
  uint32_t u = __float_as_uint(x);
  u = (u == 0x80000000u) ? 0u : u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_score(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

struct TopkSrc {
  const float* scores = nullptr;     // dense scores or gathered list scores
  const long long* ids = nullptr;    // explicit ids (id < 0 = empty slot); null -> id = id_base + position
  const long long* exclude = nullptr;  // per-query id to drop (self match, XS:118); only with explicit ids
  const uint2* packed = nullptr;     // (score bits, local index) pairs; overrides scores/ids when set
  int packed_global = 0;             // packed.y is a signed GLOBAL id (< 0 = empty slot) instead of a local index: the
                                     // gathered per-shard lists of a cross-shard merge (exclude applies)
  int lists_sorted = 0;              // (packed_global) every list is sorted: score descending, id ascending on ties, empty
                                     // slots at the tail — what sgpt_search_packed / the peer push write.  Selects the
                                     // rank-merge kernel (no selection, no sort) when the lists fit in shared memory
  // cross-GPU gather: before touching the lists, wait until wait_flag[q] >= wait_target (system-scope acquire): the
  // producers of the lists are the selection kernels of the OTHER ranks, writing through NVLink peer mappings
  const unsigned int* wait_flag = nullptr;
  unsigned int wait_target = 0;
  const int32_t* counts = nullptr;   // per-(list, query) valid length (clamped to L); null -> L
  // Two-sided lists (packed local entries only): list g additionally holds counts_back[g * nq + q] entries at its END
  // (slots L - count .. L - 1) — the candidates between the search's lower and upper admission thresholds.  The
  // selection reads them (as lists G .. 2G-1) only when the front parts together hold fewer than k entries.
  const int32_t* counts_back = nullptr;
  // per-query switch (two-pass search): the selection kernel returns at once for queries with run_flag[q] == 0 — they were
  // answered by the front-list kernel (launch_front_select) launched just before it
  const int* run_flag = nullptr;
  // dense rows that may hold masked entries (score bits 0xffffffff, the invalid key: the masked search's dense plan):
  // the valid elements must be counted instead of taken to be every column
  int dense_masked = 0;
  long long id_base = 0;
  int G = 1;                         // lists per query
  int nq = 0;
  long long L = 0;                   // capacity / length of each list
  long long stride_g = 0, stride_q = 0;
};

// Optional side outputs of a selection (two-pass search): the winners re-packed as the head of a candidate list
// (local index = id - src.id_base) with its count, and the k-th best score as the query's admission threshold.
constexpr int kMaxPeers = 16;
struct TopkExtra {
  uint2* packed = nullptr;  // [nq, cap]
  int* count = nullptr;     // [nq]
  long long cap = 0;
  float* tau = nullptr;     // [nq]
  // packed final output (score bits, int32 global id; id -1 = empty), written to `n_dst` destinations — this rank's
  // buffer and, for a sharded corpus, the gather buffers of every peer GPU (peer-mapped pointers): row
  // dst[p][(dst_slot * dst_nq + q) * k + i].  After the rows of query q have been written, flag[p][q] is incremented
  // with a system-scope release (flag[p] == nullptr: no signal).
  uint2* dst[kMaxPeers] = {};
  unsigned int* flag[kMaxPeers] = {};
  int n_dst = 0;
  int dst_slot = 0;
  int dst_nq = 0;
};

// out_scores / out_ids may be null when only the side outputs are wanted.
int launch_topk_select(const TopkSrc& src, int nq, int k, float* out_scores, int64_t* out_ids, cudaStream_t stream,
                       const TopkExtra& extra = TopkExtra());

// Final selection of the two-pass search from the FRONT parts of two-sided lists alone (topk.cu front_select_kernel): answers
// every query whose front parts hold between k and 4096 entries and clears need_generic[q] for it; sets need_generic[q] = 1
// for the others, which launch_topk_select (with TopkSrc::run_flag = need_generic) then answers.  *taken = false when the
// source does not qualify (nothing launched, need_generic untouched).
int launch_front_select(const TopkSrc& src, int nq, int k, float* out_scores, int64_t* out_ids, cudaStream_t stream,
                        const TopkExtra& extra, int* need_generic, bool* taken);

// tau_lo[q] / tau_hi[q] = lower bounds (tight to 2^-11 relative) of the k-th / k_hi-th largest of the `total` floats at
// pool + q * stride_q (0xffffffff = unused slot; total % 8 == 0, total <= kMaxTauSample, 1 <= k_hi <= k); -inf when fewer
// than k (k_hi) are valid.
constexpr int kMaxTauSample = 12 * 1024;
int launch_tau_select(const float* pool, long long stride_q, int total, int nq, int k, int k_hi, float* tau_lo,
                      float* tau_hi, cudaStream_t stream);

}  // namespace sgpt
