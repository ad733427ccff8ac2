// Internal (C++) entry points of gemm.cu used by search.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sgpt {

constexpr int kSimBN = 256;  // corpus rows per similarity tile (N-tile width of the query x corpus GEMM)
// int8 operands: at most this many dimensions, so that no s32 dot product can overflow (2^16 x 128 x 128 = 2^30)
constexpr int kMaxDimI8 = 65536;
// packed sign bits: at most this many dimensions (the parked 4 a + D <= 5 D stays an exact fp32 integer)
constexpr int kMaxDimB1 = 65536;

// Operand type of the similarity GEMM (gemm.cuh gemm_bf16_tn_kernel): bf16 rows, int8 rows, or packed sign bits (D / 8
// bytes per row, include/sgpt_b200.h binary corpus shards).  Functions below take D in dimensions for every type.
// kE4M3: fp8 rows of the linear-layer GEMM only (gemm.cuh gemm_linear_kernel, include/sgpt_b200.h fp8 linear layers).
enum class Operand : int { kBF16 = 0, kS8 = 1, kB1 = 2, kE4M3 = 3 };

// Geometry of the candidate lists the filter GEMM writes for a launch over `tiles` corpus tiles: every (CTA, column
// half) is a group with a private list of `L` entries per query (worst case: every score of every visited tile).
struct FilterGeometry {
  int groups;  // 2 x CTAs (nq <= 128) or 2 x CTA pairs (128 < nq <= 256) of the launch
  int L;       // entries per (query, group) list
};
FilterGeometry filter_geometry(long long tiles, int nq);

// Document mask of a launch's queries (include/sgpt_b200.h, masked searches): bits == nullptr = every document allowed;
// otherwise query q of the launch reads the bitmap at bits + q * pitch (pitch 0: one bitmap shared by all queries).
struct DocMask {
  const uint32_t* bits = nullptr;
  long long pitch = 0;
};
// SGPT_OK, or SGPT_ERR_INVALID with the message set for a negative pitch, 0 < pitch < ceil(n / 32) or a pitch without a
// bitmap (no CUDA call)
int check_doc_mask(const char* fn, long long n, DocMask mask);

// The `dtype` argument of the masked entry points -> operand type; SGPT_ERR_INVALID with the message set for an unknown
// dtype (no CUDA call)
int shard_operand(const char* fn, int dtype, Operand* op);
// The D rules of the operand type and, for kB1 with nq > 0, non-null popcounts and 16-byte aligned Q, C and document
// popcounts: SGPT_OK, or SGPT_ERR_INVALID with the message set (no CUDA call)
int check_operands(const char* fn, Operand op, const void* Q, const void* C, const float* q_scale, const float* c_scale,
                   int nq, int D);
// bytes per row of D dimensions
size_t operand_row_bytes(Operand op, int D);

// Similarity GEMM whose epilogue appends every score >= tau[q] (tau == nullptr: every score) as (score bits, local doc
// index) to the list cand[q * stride_q + (group0 + g) * L + ...] — scores >= tau_hi[q] at its front, the others at its
// back (tau_hi == nullptr: all at the front) — and writes counts / counts_back[(group0 + g) * nq + q] for the groups g of
// this launch (filter_geometry of the visited tile count).  tile_mode/tile_stride select the corpus tiles visited
// (gemm.cuh TileMap).  nq <= 256 (above 128: CTA pairs, M = 256).  op: the type of the Q and C rows (gemm.cuh; kB1: the
// scales are the int32 popcounts of the rows).  Documents the mask excludes are never admitted.
int launch_filter_candidates(const void* Q, const void* C, const float* q_scale, const float* c_scale,
                             const float* tau, const float* tau_hi, uint2* cand, int* counts, int* counts_back,
                             long long stride_q, int L, int group0, int nq, int n, int D, int tile_mode, int tile_stride,
                             DocMask mask, Operand op, cudaStream_t stream);

// The same GEMM over every tile_stride-th corpus tile in sample mode: pool[q * stride_p + g * Lp + ...] receives the
// maximum score of every 4 consecutive (allowed) documents the group visited (filter_geometry(sampled tiles).L / 4 floats
// per list, unused slots = 0xffffffff).  Input of launch_tau_select (topk.cuh).
int launch_sample_maxima(const void* Q, const void* C, const float* q_scale, const float* c_scale, float* pool,
                         long long stride_p, int Lp, int nq, int n, int D, int tile_stride, DocMask mask, Operand op,
                         cudaStream_t stream);

// Dense scores [nq, lds] (sgpt_scores / sgpt_scores_i8); with a mask, masked documents get score bits 0xffffffff, which
// the selection kernels treat as absent (topk.cu score_key: invalid key 0).
int launch_scores(const void* Q, const void* C, const float* q_scale, const float* c_scale, float* scores, long long lds,
                  int nq, int n, int D, DocMask mask, Operand op, cudaStream_t stream);

// LM-head logits of sgpt_lm_logprobs (model.cu): logits[m, j] = <X[m,:], W[j,:]> as the fp32 accumulator holds it,
// fp32 [M, lds], with X bf16 [M, d] and W bf16 [vocab, d].  Unlike launch_scores a NaN stays NaN (gemm.cuh
// EpiLogitsF32), so a broken hidden state reaches the log-softmax.  d % 8 == 0, lds >= vocab; X, W and logits 16-byte
// aligned.
int launch_lm_logits(const void* X, const void* W, float* logits, long long lds, int M, int vocab, int d,
                     cudaStream_t stream);

// Grouped scan of the IVF search (ivf.cu; gemm.cuh EpiIvfRows): the filter GEMM's mainloop (BN = kSimBN, bf16 or s8)
// over the work units of p.units, A = rows x D gathered query rows, C = the n x D list-ordered corpus.  Launches
// min(p.max_units, SMs) persistent CTAs; the unit count is read on the device.
struct IvfRowsParams {
  const int4* units;        // (m0, m_end, n0, n_end) per work unit
  const int* n_units;       // [1] number of units (written by the unit-table kernel)
  int max_units;            // capacity of `units`
  const float* row_scale;   // [rows] scale of each pair row's query (1 when the scores take none)
  const float* col_scale;   // [n] or null
  const int2* row_info;     // [rows] (candidate list of the pair, first position of the probed list)
  const int32_t* doc_ids;   // [n] global id of each position
  const uint32_t* mask;     // shared bitmap of allowed positions, or null
  uint2* cand;              // [pairs of the block][Ls]
  long long Ls;             // entries per candidate list (even)
};
// The scan with one bitmap per query (gemm.cuh EpiIvfRowsT<true>): `mask` is the bitmap of the block's first query, and
// pair row r reads the bitmap at mask + (row_info[r].x / nprobe) * mask_pitch.
struct IvfRowsMaskedParams : IvfRowsParams {
  long long mask_pitch;  // words between consecutive queries' bitmaps (> 0)
  int nprobe;            // pairs per query: row_info.x / nprobe is the pair's query inside the block
};
// mask_pitch == 0: p.mask is null or one shared bitmap (EpiIvfRows); mask_pitch > 0: one bitmap per query of the block,
// p.mask + q * mask_pitch for query q of the block (EpiIvfRowsMasked).
int launch_ivf_scan(const void* A, int rows, const void* C, int n, int D, const IvfRowsParams& p, long long mask_pitch,
                    int nprobe, bool s8, cudaStream_t stream);

}  // namespace sgpt
