/*
 * sgpt_b200 — C ABI of the H100-native (sm_90a) SGPT bi-encoder hot path.
 *
 * The reference (Muennighoff/sgpt @ 37c8bf09) is pure Python and has no FFI layer; its plug-in boundary is the pair
 * of duck-typed protocols in biencoder/beir/custommodels/exact_search.py:22-32 (embedder: encode_queries /
 * encode_corpus; retriever: search).  This header is the C boundary that sits *underneath* those protocols: every
 * entry point replaces the PyTorch/HF library call(s) cited next to it.  All pointers are DEVICE pointers owned by
 * the caller unless stated otherwise; no torch types cross this boundary.  Every function returns SGPT_OK (0) or an
 * error code; sgpt_last_error() returns a thread-local message.  Nothing throws.  A handle is bound to the device
 * that was current when it was created, is not thread-safe, and may be used on any stream of that device as long
 * as calls are externally ordered.
 *
 * Abbreviations in citations:  BDR = biencoder/beir/beir_dense_retriever.py, XS = .../custommodels/exact_search.py,
 * ST/ = biencoder/nli_msmarco/sentence-transformers/sentence_transformers/, HF: = transformers/models/ (third-party
 * dependency of the reference, pinned >=4.6,<5 by ST's setup.py:21).
 */
#ifndef SGPT_B200_H_
#define SGPT_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SGPT_ABI_VERSION 4  /* 4: the embed / layernorm / pool entry points changed signature (one per operation) */

#define SGPT_OK 0
#define SGPT_ERR_INVALID 1     /* bad argument / unsupported shape */
#define SGPT_ERR_CUDA 2        /* a CUDA runtime/driver call failed */
#define SGPT_ERR_UNSUPPORTED 3 /* valid request this build does not implement */

typedef void* sgpt_stream_t; /* cudaStream_t */

int sgpt_abi_version(void);
const char* sgpt_last_error(void);

/* ------------------------------------------------------------------------------------------------------------------
 * Encoder building blocks (rows F1–F7 of SURVEY.md §8a).  Token-major, *ragged* layout: the B sequences of a batch
 * are packed back to back into T = sum(len_b) rows ("tokens"); padding never exists on the device.
 * ------------------------------------------------------------------------------------------------------------------ */

/* The residual stream is bf16: HF keeps hidden_states in the model dtype, i.e. bf16 for the reference's bf16 configs
 * (BASELINE configs 3-5).  The embedding writes it, LayerNorm reads it, and sgpt_linear(..., SGPT_EPI_RESID_BF16) adds
 * into it with a bf16 TMA reduce.  Sums and statistics are fp32. */

/* F1. resid[t,:] = bf16(wte[ids[t],:] (+ wpe[pos[t],:] if wpe != NULL))       HF:gpt_neo/modeling_gpt_neo.py:462-463
 *     ids,pos int32[T]; wte bf16[vocab,d]; wpe bf16[max_pos,d] or NULL (GPT-J / BLOOM); resid bf16[T,d].
 *     An id outside [0, vocab) or a position outside [0, max_pos) is clamped to the nearest row of its table. */
int sgpt_embed_tokens(const int32_t* ids, const int32_t* pos, const void* wte, const void* wpe, void* resid, int T,
                      int d, int vocab, int max_pos, sgpt_stream_t stream);

/* F2/F7. y = LayerNorm(x; gamma, beta, eps) row-wise, fp32 statistics, bf16 output.   HF:gpt_neo/...:332,345,492
 *     x bf16[T,d]; gamma,beta fp32[d]; y bf16[T,d]; y may alias x (BLOOM word_embeddings_layernorm runs in place,
 *     HF:bloom/modeling_bloom.py:496). */
int sgpt_layernorm(const void* x, const float* gamma, const float* beta, void* y, int T, int d, float eps,
                   sgpt_stream_t stream);

/* F3/F5/F6. y = epilogue(x @ w^T + bias).   torch.nn.Linear call sites HF:gpt_neo/...:84-87,153,295-309
 *     x bf16[M,K] (row pitch ldx), w bf16[N,K] (nn.Linear weight layout, row pitch ldw), bias fp32[N] or NULL.
 *     epilogue: SGPT_EPI_BF16       out bf16[M,N]  = acc + bias
 *               SGPT_EPI_GELU_BF16  out bf16[M,N]  = gelu_new(acc + bias)       (HF activations.py NewGELUActivation)
 *               SGPT_EPI_RESID_BF16 out bf16[M,N] += acc + bias                 (in place: resid == out, the residual
 *                                                                                stream)
 *     Runs on the wgmma tensor cores (TMA-staged tiles, register accumulators). */
#define SGPT_EPI_BF16 0
#define SGPT_EPI_GELU_BF16 1
#define SGPT_EPI_RESID_BF16 3
int sgpt_linear(const void* x, int64_t ldx, const void* w, int64_t ldw, const float* bias, void* out, int64_t ldo,
                const void* resid, int M, int N, int K, int epilogue, sgpt_stream_t stream);

/* F7'. y[m,:] = LayerNorm(x[rows[m],:]) for a gathered subset of rows (bf16 out): the LM-head input of
 *      sgpt_lm_logprobs.  x bf16[T,d]; rows int32[M] (values in [0,T)); y bf16[M,d]. */
int sgpt_layernorm_gather(const void* x, const int32_t* rows, const float* gamma, const float* beta, void* y, int M,
                          int d, float eps, sgpt_stream_t stream);

/* F3'. GPT-J fused q/k/v projection with rotary position embedding in the epilogue
 *     (HF:gptj/modeling_gptj.py:98-101 bias-free projections, :55-67 + :196-207 rotary on the first rotary_dim dims of
 *     every q and k head, interleaved pairs).  x bf16[M,d] (pitch ldx), w_qkv bf16[3d,d] rows [q|k|v],
 *     qkv bf16[M,3d]; pos int32[M]; cos_sin fp32[max_pos, rotary_dim/2, 2] = (cos, sin) of pos * 10000^(-2i/rotary_dim). */
int sgpt_linear_qkv_rotary(const void* x, int64_t ldx, const void* w_qkv, void* qkv, const int32_t* pos,
                           const float* cos_sin, int M, int d_model, int head_dim, int rotary_dim, int max_pos,
                           sgpt_stream_t stream);

/* F4. Causal self-attention over a ragged batch.    HF:gpt_neo/modeling_gpt_neo.py:105-130 (_attn)
 *     qkv bf16[T, 3*H*hd]: per token [q(H*hd) | k(H*hd) | v(H*hd)];  out bf16[T, H*hd].
 *     cu_seqlens int32[B+1] (row offsets of each sequence; cu[B] == T).
 *     scale: multiplies q.k before softmax (GPT-Neo: 1.0 — unscaled, :110; GPT-J: 1/sqrt(hd)).
 *     window: 0 = plain causal; w > 0 = GPT-Neo local attention (key j visible to query i iff i-w < j <= i, :63-66).
 *     alibi_slopes: fp32[H] or NULL; adds slope_h * (key position in its sequence) to the scaled scores (BLOOM ALiBi,
 *                   HF:bloom/modeling_bloom.py:43-86; the bias depends on the key only).
 *     impl: 0 = tensor-core (mma.sync) kernel, 1 = SIMT cross-check kernel (test infrastructure). */
int sgpt_attention(const void* qkv, void* out, const int32_t* cu_seqlens, int B, int T, int H, int hd, float scale,
                   int window, int max_seqlen, const float* alibi_slopes, int impl, sgpt_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * P1/P2. Pooling over the ragged sequence dimension, fp32 accumulate.
 *     BDR:258-270 == ST/models/Pooling.py:99-125 (weightedmean), BDR:238-242 (mean), BDR:271-282 (lasttoken)
 *     x bf16[T,d] (x_bf16 = 1: the residual stream) or fp32[T,d] (x_bf16 = 0: a hidden state); pos int32[T] = index
 *     of the token in its *padded* row (weight of token t is pos[t]+1 for weightedmean); out fp32[B,d].
 *     If gamma != NULL the final LayerNorm (ln_f, F7) is applied to every row on the fly before it is pooled.
 *     clamp_denominator != 0 reproduces ST's clamp(min=1e-9) (Pooling.py:122); 0 reproduces the script (no clamp).
 *     normalize != 0 additionally L2-normalises each output row (ST/models/Normalize.py:13-14).
 *     row_stats_ws: fp32[2*T + B] scratch, needed with gamma or normalize (else may be NULL).
 *     pos_weights: fp32[n_pos_weights] or NULL.  With a table (mode must be WEIGHTEDMEAN) the weight of token t is
 *     pos_weights[pos[t]] instead of pos[t]+1 — the learnt per-position weights of ST/models/WeightedMeanPooling.py:21-37
 *     (`position_weights[:positions]`, indexed by the position in the padded row; that module always clamps the
 *     denominator, :34).  pos[t] >= n_pos_weights is the caller's error (the reference asserts, :30); the kernel clamps
 *     the index instead of reading out of bounds.
 *     out = (accumulate ? out : 0) + out_scale * pool(x): the building block of the all-hidden-state modes below; mode
 *     is one of MEAN / WEIGHTEDMEAN / LASTTOKEN; normalize (if set) acts on the accumulated rows, so pass it with the
 *     last state.  The result is bit-reproducible: a sequence's row depends neither on the launch nor on the sequence's
 *     position in the batch.
 * ------------------------------------------------------------------------------------------------------------------ */
#define SGPT_POOL_MEAN 0
#define SGPT_POOL_WEIGHTEDMEAN 1
#define SGPT_POOL_LASTTOKEN 2
/* All-hidden-state modes, accepted by sgpt_encode only: the mean over the L+1 hidden states (embedding output, every
 * block output, ln_f of the last) of the per-state mean / last-token embedding — BDR:243-257 (meanmean: the mask sum is
 * the same for every layer, so sum/sum == mean of means) and BDR:284-301 (lasttokenmean).  layer_idx is ignored, as in
 * the reference. */
#define SGPT_POOL_MEANMEAN 3
#define SGPT_POOL_LASTTOKENMEAN 4
int sgpt_pool(const void* x, int x_bf16, const int32_t* pos, const int32_t* cu_seqlens, const float* gamma,
              const float* beta, float eps, const float* pos_weights, int n_pos_weights, float* out, float* row_stats_ws,
              int B, int T, int d, int mode, int clamp_denominator, int normalize, int accumulate, float out_scale,
              sgpt_stream_t stream);

/* Sentence-embedding head applied after pooling: y = act(x @ w^T + bias), all fp32 (ST/models/Dense.py:40-43 with
 * key_name "sentence_embedding"; nn.Linear weight layout).  x fp32[B,in], w fp32[out,in], bias fp32[out] or NULL,
 * y fp32[B,out] (must not alias x). */
#define SGPT_ACT_IDENTITY 0
#define SGPT_ACT_TANH 1
#define SGPT_ACT_RELU 2
#define SGPT_ACT_SIGMOID 3
int sgpt_dense(const float* x, const float* w, const float* bias, float* y, int B, int in_features, int out_features,
               int activation, sgpt_stream_t stream);

/* P2 stand-alone: x[b,:] /= max(||x[b,:]||_2, 1e-12) in place (ST/models/Normalize.py:13-14;
 * SentenceTransformer.py:248-249) for embeddings that passed through a head after pooling.  x fp32[B,d]. */
int sgpt_normalize_rows(float* x, int B, int d, sgpt_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Whole-encoder handle (F1..F7 + P1 in one call).
 * ------------------------------------------------------------------------------------------------------------------ */
#define SGPT_ARCH_GPT_NEO 0
#define SGPT_ARCH_GPTJ 1
#define SGPT_ARCH_BLOOM 2

typedef struct sgpt_model_config {
  int32_t arch;
  int32_t n_layer, d_model, n_head, d_ff, vocab, max_pos;
  int32_t window;     /* GPT-Neo local-attention window (256) */
  int32_t rotary_dim; /* GPT-J */
  float ln_eps;
  int32_t max_tokens; /* workspace capacity: largest T a single sgpt_encode call may carry */
  int32_t max_batch;  /* largest B */
} sgpt_model_config;

/* Per-layer device pointers.  Linear weights are bf16 in nn.Linear layout [out,in]; biases and LayerNorm
 * parameters are fp32.  Unused entries (arch-dependent) are NULL. */
typedef struct sgpt_layer_weights {
  const float *ln1_g, *ln1_b;
  const void* w_qkv;   /* bf16[3d, d]: rows [q | k | v] */
  const float* b_qkv;  /* fp32[3d] or NULL (GPT-Neo / GPT-J have no q,k,v bias) */
  const void* w_o;     /* bf16[d, d] */
  const float* b_o;    /* fp32[d] or NULL */
  const float *ln2_g, *ln2_b;
  const void* w_fc;    /* bf16[ff, d] */
  const float* b_fc;   /* fp32[ff] */
  const void* w_proj;  /* bf16[d, ff] */
  const float* b_proj; /* fp32[d] */
  int32_t local_attention; /* GPT-Neo: 1 for "local" layers */
  int32_t _pad;
} sgpt_layer_weights;

typedef struct sgpt_model_weights {
  const void* wte; /* bf16[vocab, d] */
  const void* wpe; /* bf16[max_pos, d] or NULL */
  const float *lnf_g, *lnf_b;
  const sgpt_layer_weights* layers; /* HOST array of n_layer entries (copied at create) */
  const float *emb_ln_g, *emb_ln_b; /* BLOOM word_embeddings_layernorm, else NULL */
} sgpt_model_weights;

typedef struct sgpt_model* sgpt_model_t;

/* Replaces AutoModel.from_pretrained(...).to(device) at BDR:123 / ST/models/Transformer.py:38 (weights are handed
 * over already on the device).  The handle borrows every weight buffer for its whole lifetime: none of them may be freed
 * or changed before sgpt_model_destroy.  It owns only its activation workspace.  Synchronises the device. */
int sgpt_model_create(const sgpt_model_config* cfg, const sgpt_model_weights* w, sgpt_model_t* out);
void sgpt_model_destroy(sgpt_model_t m);

/* Replaces self.model(**batch_tokens, output_hidden_states=True) + pooling, BDR:205 + BDR:233-304
 * (ST path: ST/models/Transformer.py:72 + ST/models/Pooling.py:85-168).
 *     ids,pos int32[T]; cu_seqlens int32[B+1]; out fp32[B,d].
 *     layer_idx: which entry of HF hidden_states to pool: -1 / n_layer = after ln_f (the reference default, BDR:44);
 *                0..n_layer-1 = input of block i (no final LayerNorm). */
int sgpt_encode(sgpt_model_t m, const int32_t* ids, const int32_t* pos, const int32_t* cu_seqlens, int B, int T,
                int max_seqlen, int layer_idx, int pool_mode, int clamp_denominator, int normalize, float* out,
                sgpt_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Continuation log-likelihoods with the same encoder (SURVEY.md §8f row 4; the SGPT cross-encoder scorer,
 * crossencoder/beir/sgptce.py:150-262 `_loglikelihood_tokens`).
 * ------------------------------------------------------------------------------------------------------------------ */

/* The GPT forward pass alone (F1..F6 of every block): replaces `model(inps)` at sgptce.py:76-83 up to the final
 * LayerNorm.  Leaves the bf16 residual stream [T,d] in the handle for sgpt_lm_logprobs / sgpt_model_read_residual. */
int sgpt_forward(sgpt_model_t m, const int32_t* ids, const int32_t* pos, const int32_t* cu_seqlens, int B, int T,
                 int max_seqlen, sgpt_stream_t stream);

/* token_logprobs[i] = log_softmax(LN_f(resid[rows[i]]) @ lm_head_w^T + lm_head_bias)[targets[i]]
 *     == F.log_softmax(logits, -1) (sgptce.py:221) gathered at the continuation tokens (:247), for the packed token
 *     rows `rows` of the batch the last sgpt_forward ran.  lm_head_w bf16[vocab,d] (the tied wte for GPT-Neo / BLOOM,
 *     lm_head.weight for GPT-J), lm_head_bias fp32[vocab] or NULL (GPT-J has one); rows,targets int32[M];
 *     greedy int32[M] or NULL receives argmax(logits) (:229, lowest index on ties).  The [M,vocab] logits exist only in
 *     `ws`, rows_per_chunk rows at a time (ws >= sgpt_lm_logprobs_workspace_bytes(d_model, vocab, rows_per_chunk));
 *     ws must be 16-byte aligned (checked before any CUDA call, for every M).
 *     The logits are not NaN-fixed like sgpt_scores: a selected row whose hidden state holds a NaN or +-inf gets a NaN
 *     log-prob and greedy 0, the sgpt_token_logprobs rules for a row of NaN (the reference returns NaN too, :221). */
int64_t sgpt_lm_logprobs_workspace_bytes(int d_model, int vocab, int rows_per_chunk);
int sgpt_lm_logprobs(sgpt_model_t m, const void* lm_head_w, const float* lm_head_bias, int vocab, const int32_t* rows,
                     const int32_t* targets, int M, float* token_logprobs, int32_t* greedy, void* ws, int64_t ws_bytes,
                     int rows_per_chunk, sgpt_stream_t stream);

/* Building blocks of the above.  sgpt_token_logprobs: logits fp32[M,lds] (vocab valid columns) -> log-softmax value of
 * the target column per row (+ optional argmax: the lowest index of the largest value that is not NaN, so a row of -inf
 * gives 0; NaN is never chosen, where torch.argmax would return the first NaN, and a row of NaN only gives 0).
 * sgpt_segment_sum: out[r] = sum(x[offsets[r]..offsets[r+1])) in index
 * order — the per-request `float(logits.sum())` of sgptce.py:250; offsets int32[R+1]. */
int sgpt_token_logprobs(const float* logits, int64_t lds, int M, int vocab, const float* bias, const int32_t* targets,
                        float* logprob, int32_t* greedy, sgpt_stream_t stream);
int sgpt_segment_sum(const float* x, const int32_t* offsets, int R, float* out, sgpt_stream_t stream);

/* Installs (w != NULL) or removes (w == NULL) a learnt position-weight table for pool_mode WEIGHTEDMEAN in sgpt_encode
 * (ST/models/WeightedMeanPooling.py).  w is a DEVICE fp32[n] buffer borrowed by the handle; sgpt_encode then fails with
 * SGPT_ERR_INVALID when max_seqlen > n, like the reference's shape assert (:30). */
int sgpt_model_set_position_weights(sgpt_model_t m, const float* w, int n);

/* Debug/parity tap: copies the residual stream (hidden_states[layer] before ln_f) left by the LAST sgpt_encode, widened
 * to fp32, into dst (device, capacity_elems floats) and reports its shape. */
int sgpt_model_read_residual(sgpt_model_t m, float* dst, int64_t capacity_elems, int* T, int* d, sgpt_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * S1–S3. Exact dense retrieval over one corpus shard.
 * ------------------------------------------------------------------------------------------------------------------ */

/* inv_norm[i] = 1 / max(||x_i||_2, 1e-12) for bf16 rows (F.normalize semantics, ST/util.py:41-42).  x bf16[n,D].
 *     fp32: per-lane sums of squares, a warp tree, then IEEE sqrt and divide.  A row holding a NaN gets 1 / 1e-12 like a
 *     zero row (the max takes the non-NaN operand); its dot products are NaN regardless, so its scores are -1. */
int sgpt_row_inv_norms(const void* x, float* inv_norm, int64_t n, int D, sgpt_stream_t stream);

/* fp32 -> bf16 row conversion (round-to-nearest-even) used to store embeddings in a shard. */
int sgpt_f32_to_bf16(const float* x, void* y, int64_t count, sgpt_stream_t stream);

/* S1. scores[q,j] = fixnan( <Q[q,:], C[j,:]> * q_scale[q] * c_scale[j] )      ST/util.py:24-63, XS:96-99
 *     Q bf16[nq,D], C bf16[n,D], q_scale fp32[nq]|NULL, c_scale fp32[n]|NULL (NULL = 1: dot_score),
 *     scores fp32[nq, lds]; NaN -> -1 as XS:99.  wgmma GEMM, corpus streamed once from HBM. */
int sgpt_scores(const void* Q, const void* C, const float* q_scale, const float* c_scale, float* scores, int64_t lds,
                int nq, int64_t n, int D, sgpt_stream_t stream);

/* Order of every top-k result below (sgpt_topk, sgpt_topk_merge, sgpt_search, sgpt_search_packed,
 * sgpt_topk_merge_packed, sgpt_search_gather): the k winners are the first k entries in (score descending, id ascending)
 * order, returned in that order, so equal scores that straddle the cut keep the lowest ids and the result depends only on
 * the input.  -0.0 and +0.0 are the same score.  Scores passed to sgpt_topk / sgpt_topk_merge must not be NaN (the
 * library's own score producers map NaN to -1, XS:99).  1 <= k <= 4096. */

/* S2. Row-wise exact top-k of a score matrix (torch.topk(..., largest=True, sorted=False), XS:102-108), with the
 *     winners returned in DESCENDING score order (ties: ascending id).  ids are offset by id_base (global doc ids of a
 *     shard).  scores fp32[nq, lds] (n valid columns); out_scores fp32[nq,k]; out_ids int64[nq,k].
 *     If n < k the tail is filled with (-inf, -1).  ws: scratch of sgpt_topk_workspace_bytes(nq,n,k) bytes. */
int64_t sgpt_topk_workspace_bytes(int nq, int64_t n, int k);
int sgpt_topk(const float* scores, int64_t lds, int nq, int64_t n, int k, int64_t id_base, float* out_scores,
              int64_t* out_ids, void* ws, sgpt_stream_t stream);

/* S3. Merge G candidate lists per query (cross-chunk heapq.nlargest merge XS:121-132; cross-shard merge after the
 *     all-gather): in_scores fp32[G,nq,k], in_ids int64[G,nq,k] -> out fp32/int64[nq,k], descending; entries with
 *     id < 0 are ignored, and so are entries whose id equals exclude_ids[q] (the `corpus_id != query_id` self-match
 *     rule of XS:118; exclude_ids int64[nq] or NULL). */
int sgpt_topk_merge(const float* in_scores, const int64_t* in_ids, int G, int nq, int k, float* out_scores,
                    int64_t* out_ids, const int64_t* exclude_ids, void* ws, sgpt_stream_t stream);

/* S1+S2 in one call: exact top-k of one corpus shard for a batch of queries (XS:96-108 for one chunk).
 *     Q bf16[nq,D], C bf16[n,D], q_scale/c_scale as sgpt_scores; out_scores fp32[nq,k], out_ids int64[nq,k]
 *     (descending, ids offset by id_base, tail (-inf,-1) when n < k).  ws: sgpt_search_workspace_bytes(nq,n,k). */
int64_t sgpt_search_workspace_bytes(int nq, int64_t n, int k);
int sgpt_search(const void* Q, const void* C, const float* q_scale, const float* c_scale, int nq, int64_t n, int D,
                int k, int64_t id_base, float* out_scores, int64_t* out_ids, void* ws, int64_t ws_bytes,
                sgpt_stream_t stream);

/* Same search, result as ONE packed list: out_packed uint64[nq,k], entry = (int32 global id << 32) | fp32 score bits,
 *     descending, empty slots (-inf, -1); requires id_base + n < 2^31.  This is the 8-byte entry of SURVEY.md §8e: one
 *     all-gather of Q*(k+1)*8 bytes per rank when the exchange goes through NCCL (sgpt_b200/dist.py). */
int sgpt_search_packed(const void* Q, const void* C, const float* q_scale, const float* c_scale, int nq, int64_t n,
                       int D, int k, int64_t id_base, uint64_t* out_packed, void* ws, int64_t ws_bytes,
                       sgpt_stream_t stream);
/* Range search: every document of one shard whose score is >= threshold (the `cos_scores >= threshold` sets of
 *     community_detection, ST/util.py:385-448, without the [nq, n] score matrix).  Q, C, q_scale, c_scale, D and id_base
 *     as sgpt_search (NULL scale = dot product; a NaN score is -1, XS:99); any nq (blocks of 256 queries reuse ws).
 *     out_counts int64[nq] (device) is always written: the number of documents with score >= threshold.  With
 *     off[q] = counts[0] + ... + counts[q-1], query q's entries go to out_scores fp32 / out_ids int64
 *     [off[q], off[q] + counts[q]) if and only if off[q] + counts[q] <= cap, in ascending id order, ids offset by
 *     id_base; entries of queries that do not fit are not written and the rest of both buffers keeps its bits (cap = 0
 *     only counts).  The output depends only on the input (no atomics decide the order).  SGPT_ERR_INVALID for a NaN
 *     threshold, D % 8 != 0, n >= 2^31, nq < 0, cap < 0, null outputs that would be written and a workspace smaller
 *     than sgpt_range_search_workspace_bytes(nq, n). */
int64_t sgpt_range_search_workspace_bytes(int nq, int64_t n);
int sgpt_range_search(const void* Q, const void* C, const float* q_scale, const float* c_scale, int nq, int64_t n,
                      int D, float threshold, int64_t id_base, int64_t* out_counts, int64_t cap, float* out_scores,
                      int64_t* out_ids, void* ws, int64_t ws_bytes, sgpt_stream_t stream);

/* S3 on packed lists: in_packed uint64[G,nq,k] (the all-gathered sgpt_search_packed outputs; chunk = shard in
 *     XS:121-132) -> out_scores fp32[nq,k], out_ids int64[nq,k]; ids < 0 and ids == exclude_ids[q] (XS:118) dropped.
 *     Every input list must be in the order sgpt_search_packed writes (score descending, id ascending on ties, empty
 *     slots last) and ids must be unique across the lists (disjoint shards): the merge ranks entries by binary search
 *     instead of selecting and sorting again. */
int sgpt_topk_merge_packed(const uint64_t* in_packed, int G, int nq, int k, float* out_scores, int64_t* out_ids,
                           const int64_t* exclude_ids, sgpt_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * int8 corpus shards: half the bytes per document of a bf16 shard, read by an int8 wgmma filter GEMM (s32 accumulate).
 *
 * Quantization of a row x (fp32, or bf16 widened to fp32) into q int8[D], scale fp32, cos_scale fp32, all in fp32
 * round-to-nearest arithmetic:
 *   amax = max |x_i|;
 *   a row holding a NaN or +-inf: q = 0, scale = cos_scale = NaN (every score against it is NaN, i.e. -1 as XS:99);
 *   amax == 0: q = 0, scale = cos_scale = 0;
 *   otherwise m = 127.0f / amax, q_i = clamp(rint(x_i * m), -127, 127) (rint: half to even), scale = amax / 127.0f,
 *   ss = sum q_i^2 (exact in integers), cos_scale = scale / fmaxf(scale * sqrtf((float)ss), 1e-12f) — F.normalize of the
 *   dequantized row (ST/util.py:41-42) folded with the dequantization scale.
 * Score: score[q,j] = fixnan(float_rn(sum_d Q[q,d] C[j,d]) * q_scale[q] * c_scale[j]), evaluated in that order; the dot
 *   product is exact in s32 (D % 16 == 0 for the TMA row pitch and D <= 65536, so no int8 input, -128 included, can
 *   overflow).  q_scale / c_scale: `scale` for dot products, `cos_scale` for cos_sim; NULL = 1.
 * The _i8 entry points take the arguments of their bf16 counterparts with Q int8[nq,D] and C int8[n,D], return results
 * in the same order (top-k: score descending, ties by ascending id, as above) and use the same workspace sizes
 * (sgpt_search_workspace_bytes, sgpt_range_search_workspace_bytes).  Arguments are checked as for the bf16 entry points,
 * and D % 16 != 0 or D > 65536 are rejected with SGPT_ERR_INVALID, before any CUDA call.
 * ------------------------------------------------------------------------------------------------------------------ */
/* x fp32[n,D] (x_bf16 = 0) or bf16[n,D] (x_bf16 = 1) -> q_out int8[n,D], scale_out / cos_scale_out fp32[n]; x and q_out
 *     16-byte aligned. */
int sgpt_quantize_rows_i8(const void* x, int x_bf16, void* q_out, float* scale_out, float* cos_scale_out, int64_t n,
                          int D, sgpt_stream_t stream);
int sgpt_scores_i8(const void* Q, const void* C, const float* q_scale, const float* c_scale, float* scores, int64_t lds,
                   int nq, int64_t n, int D, sgpt_stream_t stream);
int sgpt_search_i8(const void* Q, const void* C, const float* q_scale, const float* c_scale, int nq, int64_t n, int D,
                   int k, int64_t id_base, float* out_scores, int64_t* out_ids, void* ws, int64_t ws_bytes,
                   sgpt_stream_t stream);
int sgpt_search_packed_i8(const void* Q, const void* C, const float* q_scale, const float* c_scale, int nq, int64_t n,
                          int D, int k, int64_t id_base, uint64_t* out_packed, void* ws, int64_t ws_bytes,
                          sgpt_stream_t stream);
int sgpt_range_search_i8(const void* Q, const void* C, const float* q_scale, const float* c_scale, int nq, int64_t n,
                         int D, float threshold, int64_t id_base, int64_t* out_counts, int64_t cap, float* out_scores,
                         int64_t* out_ids, void* ws, int64_t ws_bytes, sgpt_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * fp8 linear layers: every nn.Linear of an encoder block as an e4m3 x e4m3 wgmma GEMM with fp32 accumulation (the
 * H100's fp8 tensor-core rate).  Everything else (embedding, LayerNorm, attention, the bf16 residual stream, pooling,
 * ln_f, the LM head) is the bf16 flow unchanged.
 *
 * Row quantization (weights and activations alike), a row x of K bf16 values widened to fp32, fp32 round-to-nearest:
 *   amax = max |x_j|;
 *   a row holding a NaN or +-inf: q = 0, scale = NaN (every output of the row / output channel is NaN, as the bf16
 *     GEMM's would be; it never turns finite);
 *   amax == 0: inv = 0, q = +-0 (the signs of the zeros), scale = 0;
 *   otherwise inv = min(448.0f / amax, FLT_MAX) (the min only acts for amax < 1.3e-36), q_j = cvt.rn.satfinite.e4m3(x_j *
 *     inv) (round to nearest even, e4m3 subnormals kept, |q| <= 448), scale = amax / 448.0f.
 * Weights: one row per output channel of the [out, in] weight, from the bf16 values the bf16 path stores, quantized once.
 * Activations: one row per token of the GEMM's A operand, i.e. the bf16 tensor the bf16 path feeds that GEMM: the
 *   LayerNorm output (quantized once and shared by QKV and fc on GPT-J's parallel branch), the attention output and the
 *   gelu output, each quantized in a pass of its own.
 * GEMM: acc = sum_k q_x[m,k] q_w[n,k] on the tensor cores (fp32 accumulator), then v = (acc * x_scale[m]) * w_scale[n] in
 *   this order, then the bf16 path's epilogue unchanged (bias, gelu_new, GPT-J rotary, bf16 reduce-add).
 * Accumulation precision (measured on an H100 80GB HBM3 at a 700 W power limit, tools/bench_fp8.py): with columns that
 *   cancel exactly, so that the output is the accumulation error alone, the e4m3 accumulator stays within 2.9e-4
 *   (~2^-11.8) of sum_k |x_k w_k| (median 6e-6 to 9e-6) at every K from 768 to 16384, against 7e-7 for the bf16 GEMM:
 *   the hardware keeps far fewer accumulator bits for fp8, but the error does not grow with K.  No split accumulator is
 *   used; the encoders' error against a quantization-aware fp32 reference is dominated by e4m3 codes that flip between
 *   the fp32 reference and the GPU's bf16 intermediates (tests/test_gpu_fp8.py), not by the accumulation.
 *
 * sgpt_quantize_rows_fp8: x bf16[n, K] (16-byte aligned) -> q_out e4m3[n, K] (16-byte aligned), scale_out fp32[n];
 *   K % 16 == 0.
 * sgpt_linear_fp8: sgpt_linear with xq e4m3[M, K] (pitch ldx bytes), x_scale fp32[M], wq e4m3[N, K] (pitch ldw),
 *   w_scale fp32[N]; K, ldx, ldw multiples of 16; the three epilogues of sgpt_linear.  Split-K is not supported
 *   (SGPT_GEMM_SPLITK > 1 is rejected).
 * sgpt_linear_qkv_rotary_fp8: sgpt_linear_qkv_rotary with xq e4m3[M, d] (pitch ldx), x_scale fp32[M], wq_qkv e4m3[3d, d],
 *   w_scale fp32[3d].
 * sgpt_model_create_fp8: sgpt_model_create whose linear layers run in fp8: fp8_layers is a HOST array of n_layer entries
 *   (copied at create) of borrowed device (e4m3 weight, fp32 scale) pairs, the weights quantized by
 *   sgpt_quantize_rows_fp8 in the layouts of sgpt_layer_weights.  The bf16 linear pointers of w->layers are not read
 *   and may be NULL.  The handle additionally owns an e4m3 activation buffer [max_tokens, max(d_model, d_ff)] and
 *   fp32 scales [max_tokens].  sgpt_encode, sgpt_forward, sgpt_lm_logprobs, sgpt_model_read_residual and
 *   sgpt_model_set_position_weights take the handle unchanged.
 * Arguments are checked (sizes, K % 16, null operands or scales, unknown epilogue, split-K) before any CUDA call.
 * ------------------------------------------------------------------------------------------------------------------ */
int sgpt_quantize_rows_fp8(const void* x, void* q_out, float* scale_out, int64_t n, int K, sgpt_stream_t stream);
int sgpt_linear_fp8(const void* xq, int64_t ldx, const float* x_scale, const void* wq, int64_t ldw, const float* w_scale,
                    const float* bias, void* out, int64_t ldo, const void* resid, int M, int N, int K, int epilogue,
                    sgpt_stream_t stream);
int sgpt_linear_qkv_rotary_fp8(const void* xq, int64_t ldx, const float* x_scale, const void* wq_qkv,
                               const float* w_scale, void* qkv, const int32_t* pos, const float* cos_sin, int M,
                               int d_model, int head_dim, int rotary_dim, int max_pos, sgpt_stream_t stream);

typedef struct sgpt_fp8_layer_weights {
  const void* w_qkv;   /* e4m3[3d, d] */
  const float* s_qkv;  /* fp32[3d] */
  const void* w_o;     /* e4m3[d, d] */
  const float* s_o;    /* fp32[d] */
  const void* w_fc;    /* e4m3[ff, d] */
  const float* s_fc;   /* fp32[ff] */
  const void* w_proj;  /* e4m3[d, ff] */
  const float* s_proj; /* fp32[d] */
} sgpt_fp8_layer_weights;

int sgpt_model_create_fp8(const sgpt_model_config* cfg, const sgpt_model_weights* w,
                          const sgpt_fp8_layer_weights* fp8_layers, sgpt_model_t* out);

/* ------------------------------------------------------------------------------------------------------------------
 * §8e without a collective library call: the per-shard top-k lists are PUSHED into every rank's gather buffer by the
 * final selection kernel itself (stores through NVLink peer mappings + a system-scope release per query) and merged by
 * a kernel that acquires those per-query counters — the reference's sequential chunk/heapq merge (XS:80-132) with
 * chunk = GPU.  One context per process (= per GPU):
 *   sgpt_gather_create    allocates this rank's buffer and returns its CUDA IPC handle (SGPT_IPC_HANDLE_BYTES bytes);
 *   sgpt_gather_connect   maps the buffers of all ranks from the concatenated handles [world][SGPT_IPC_HANDLE_BYTES]
 *                         (exchanged by the host, e.g. torch.distributed.all_gather_object);
 *   sgpt_search_gather    = sgpt_search on this rank's shard + push + merge: every rank of the group must call it with
 *                         the same nq and k, in the same order; all ranks receive the identical merged top-k
 *                         (out_scores fp32[nq,k], out_ids int64[nq,k], self matches exclude_ids[q] dropped).
 * ------------------------------------------------------------------------------------------------------------------ */
#define SGPT_IPC_HANDLE_BYTES 64
typedef struct sgpt_gather* sgpt_gather_t;
int sgpt_gather_create(int rank, int world, int nq_cap, int k, sgpt_gather_t* out, void* handle_out);
int sgpt_gather_connect(sgpt_gather_t g, const void* all_handles);
void sgpt_gather_destroy(sgpt_gather_t g);
int sgpt_search_gather(sgpt_gather_t g, const void* Q, const void* C, const float* q_scale, const float* c_scale,
                       int nq, int64_t n, int D, int k, int64_t id_base, const int64_t* exclude_ids, float* out_scores,
                       int64_t* out_ids, void* ws, int64_t ws_bytes, sgpt_stream_t stream);
/* The same on an int8 shard (Q int8[nq,D], C int8[n,D]; see the int8 shard section above). */
int sgpt_search_gather_i8(sgpt_gather_t g, const void* Q, const void* C, const float* q_scale, const float* c_scale,
                          int nq, int64_t n, int D, int k, int64_t id_base, const int64_t* exclude_ids, float* out_scores,
                          int64_t* out_ids, void* ws, int64_t ws_bytes, sgpt_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Filtered (masked) search: the same searches over the ALLOWED documents of a shard only (document deletion, per-tenant
 * or per-query filters).  One entry point per operation; `dtype` selects the shard format (SGPT_DTYPE_BF16: the
 * arguments of the bf16 entry point; SGPT_DTYPE_I8: those of its _i8 twin).  The unmasked entry points are these with a
 * null mask, and the workspace sizes are the same.
 *   Mask: uint32 words (device); bit j % 32 of word j / 32 set = local document j allowed.  mask_pitch_words = 0: one
 *     bitmap [ceil(n/32)] shared by all queries; mask_pitch_words >= ceil(n/32): one bitmap per query, [nq][pitch].
 *     mask == NULL (with pitch 0): every document allowed.  Bits at or past n are ignored.
 *   Results: exactly those of the unmasked call computed over the allowed documents only — top-k in (score descending,
 *     id ascending) order with the same tie rule, tail (-inf, -1) when fewer than k documents are allowed; range search
 *     counts and returns allowed documents only, in ascending id order.  Masked documents never appear, also when every
 *     document is masked.  With a NULL or all-ones mask every output is bit-identical to the unmasked entry point.
 *   SGPT_ERR_INVALID, before any CUDA call, for an unknown dtype, a negative pitch, 0 < pitch < ceil(n/32) and a
 *     non-zero pitch with a NULL mask, besides the rejections of the unmasked entry point.
 * ------------------------------------------------------------------------------------------------------------------ */
#define SGPT_DTYPE_BF16 0
#define SGPT_DTYPE_I8 1
#define SGPT_DTYPE_B1 3 /* binary corpus shards (packed sign bits), see below */
int sgpt_search_masked(int dtype, const void* Q, const void* C, const float* q_scale, const float* c_scale, int nq,
                       int64_t n, int D, int k, int64_t id_base, const uint32_t* mask, int64_t mask_pitch_words,
                       float* out_scores, int64_t* out_ids, void* ws, int64_t ws_bytes, sgpt_stream_t stream);
int sgpt_search_packed_masked(int dtype, const void* Q, const void* C, const float* q_scale, const float* c_scale,
                              int nq, int64_t n, int D, int k, int64_t id_base, const uint32_t* mask,
                              int64_t mask_pitch_words, uint64_t* out_packed, void* ws, int64_t ws_bytes,
                              sgpt_stream_t stream);
int sgpt_range_search_masked(int dtype, const void* Q, const void* C, const float* q_scale, const float* c_scale,
                             int nq, int64_t n, int D, float threshold, int64_t id_base, const uint32_t* mask,
                             int64_t mask_pitch_words, int64_t* out_counts, int64_t cap, float* out_scores,
                             int64_t* out_ids, void* ws, int64_t ws_bytes, sgpt_stream_t stream);
/* The mask applies to this rank's shard only (local document indices); the other ranks pass their own. */
int sgpt_search_gather_masked(int dtype, sgpt_gather_t g, const void* Q, const void* C, const float* q_scale,
                              const float* c_scale, int nq, int64_t n, int D, int k, int64_t id_base,
                              const uint32_t* mask, int64_t mask_pitch_words, const int64_t* exclude_ids,
                              float* out_scores, int64_t* out_ids, void* ws, int64_t ws_bytes, sgpt_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Binary corpus shards: every document stored as D sign bits, D / 8 bytes (8x less than int8), searched exactly by a
 * single-bit wgmma filter GEMM (wgmma .b1.b1.and.popc).  The format of sentence-transformers' quantize_embeddings(...,
 * precision="ubinary").
 *   Bits: a row x (fp32, or bf16 widened) becomes b_j = (x_j > t_j), t the fp32 thresholds [D] (NULL: all 0, which is
 *     ubinary exactly).  The compare is strict (x_j == t_j gives 0) and a NaN gives 0.  Packed in np.packbits order:
 *     dimension j is bit 7 - (j & 7) of byte j / 8; a row is D / 8 bytes.  popc = the row's number of set bits (int32).
 *     D % 128 == 0 (rows a multiple of 16 bytes) and D <= 65536.
 *   Score of query bits q against document bits d: a = popc(q AND d), h = popc(q) + popc(d) - 2 a (the Hamming
 *     distance), s = D - 2 h = 4 a - 2 popc(d) - 2 popc(q) + D: the dot product of the two +-1 vectors, an integer with
 *     |s| <= D, exact in fp32.  The device evaluates it as ((float)(4 a + D) - 2 popc(q)) - 2 popc(d), every step exact.
 *     Every entry point below returns s; cos_sim of the +-1 vectors is s / D (one correctly rounded fp32 division,
 *     monotone in s), which the caller applies to the scores it receives (sgpt_b200.index.CorpusShard does), and a
 *     cos_sim threshold t is the threshold s0 = the smallest integer with fl(s0 / D) >= t on s.
 *   Top-k: the tie rule of every search (score descending, ids ascending); with D + 1 possible scores, ties are common.
 * sgpt_quantize_rows_b1: x fp32 [n, D] (x_bf16 = 0) or bf16 [n, D] (x_bf16 = 1), 16-byte aligned; thresholds fp32 [D] or
 *   NULL; bits_out uint8 [n, D / 8] (16-byte aligned) and popc_out int32 [n].  SGPT_ERR_INVALID, before any CUDA call,
 *   for n < 0, D not a positive multiple of 128 or above 65536, and (n > 0) null or unaligned pointers.
 * SGPT_DTYPE_B1 in sgpt_search_masked, sgpt_search_packed_masked, sgpt_search_gather_masked and
 *   sgpt_range_search_masked: Q uint8 [nq, D / 8] and C uint8 [n, D / 8] are bit rows; q_scale and c_scale point at the
 *   int32 popcounts of the query and document rows (int32 [nq] and int32 [n], passed through the float pointers; NULL is
 *   rejected when nq > 0).  Q, C and c_scale 16-byte aligned.  Masks, workspaces, output order and every other argument
 *   as for the other dtypes; the range search's threshold applies to s (a Hamming radius r is the threshold D - 2 r).
 *   SGPT_ERR_INVALID, before any CUDA call, for D % 128 != 0, D > 65536, null popcounts and unaligned rows, besides the
 *   other rejections.  The IVF and IVF-PQ entry points reject SGPT_DTYPE_B1.
 * SGPT_DTYPE_B1 in sgpt_rerank (rescoring bit candidates with the float query): Q fp32 [nq, D] (for cos_sim the caller
 *   passes F.normalize(q)), C the bit rows [n, D / 8]; c_scale is not read.  The score is the asymmetric
 *   r = sum_j q_j s_j, s_j = +1 where bit j is set and -1 elsewhere, evaluated in this order: lane l (0..31) takes the
 *   16-byte bit units l, l + 32, l + 64, ... (128 dimensions each) in ascending order and the 128 dimensions of a unit in
 *   ascending order, acc_l += (bit ? q_j : -q_j) with one rounding per add; then for o = 16, 8, 4, 2, 1:
 *   acc_l = acc_l + acc_(l xor o); score = fixnan(acc_0 * q_scale[q]) with q_scale = fp32(1 / sqrt(D)) for cos_sim and
 *   NULL (= 1) for dot.  Reproducible in numpy bit for bit.  D % 128 == 0 and D <= 65536.
 *   (sgpt_b200.index.CorpusShard.search(..., rescore=) passes Q = q - t, the query centered on the shard's thresholds
 *   t, normalized for cos_sim: with zero thresholds that is sentence-transformers' rescoring of q itself; with non-zero
 *   thresholds it keeps a common offset of the embeddings, which the bits do not encode, out of the score.)
 * ------------------------------------------------------------------------------------------------------------------ */
int sgpt_quantize_rows_b1(const void* x, int x_bf16, const float* thresholds, void* bits_out, int32_t* popc_out,
                          int64_t n, int D, sgpt_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * IVF (inverted-file) search: a corpus split into nlist lists (k-means cells), of which each query scans only the
 * `nprobe` it probes.  The search is exact relative to its lists: it returns exactly what the exact search returns over
 * the undeleted documents of the probed lists — the same scores (the rows of C as stored: bf16 with c_scale = 1/||row||,
 * or int8 with per-row scales, see the int8 shard section), the same order (score descending, ties by ascending GLOBAL
 * id) and the tail (-inf, -1) when fewer than k documents are probed.  Choosing the probes (e.g. the exact top-nprobe of
 * the centroids) is the caller's part.
 *   dtype       SGPT_DTYPE_BF16: Q bf16[nq,D], C bf16[n,D] (D % 8 == 0); SGPT_DTYPE_I8: Q int8[nq,D], C int8[n,D]
 *               (D % 16 == 0, D <= 65536).  q_scale [nq] / c_scale [n] as in sgpt_search (NULL = 1).  Q 16-byte aligned.
 *   C           the rows in list order: list l is rows [list_offsets[l], list_offsets[l+1]) (int64 [nlist+1], device).
 *               max_list_len >= every list's length (the workspace and the candidate lists are sized by it).
 *   doc_ids     int32 [n] (device): the global id of each row; results carry these ids (< 0 = never returned).
 *   probes      int32 [nq, nprobe] (device): the lists query q scans.  Entries outside [0, nlist) are skipped; the
 *               entries of one query must be distinct.
 *   mask        shared bitmap of the ALLOWED rows (row positions, the format of the masked searches, pitch 0) or NULL.
 *   out_scores  fp32 [nq, k], out_ids int64 [nq, k] (device).
 * Any nq (blocks of 256 queries reuse ws); no host synchronisation.  The device inputs bound every access: offsets are
 * clamped to [0, n] and lengths to max_list_len, so inconsistent offsets or probes give wrong results, never an
 * out-of-bounds access.  SGPT_ERR_INVALID, before any CUDA call, for an unknown dtype, nq < 0, the D rules of the dtype,
 * nlist < 1, nprobe outside [1, nlist], k outside [1, 4096], n outside [0, 2^31), max_list_len outside [0, n],
 * nprobe x max_list_len beyond the selection's 2^32 entries, null inputs or outputs, an unaligned Q and a workspace
 * smaller than sgpt_ivf_search_workspace_bytes (which returns -1 for arguments the search rejects).
 *
 * sgpt_ivf_search_masked: the same search with a filter, shared or per query, in the mask format of the masked searches
 * above, indexed by row position of C (list order): mask_pitch_words = 0: one bitmap [ceil(n/32)] shared by all queries
 * (sgpt_ivf_search's `mask`); mask_pitch_words >= ceil(n/32): one bitmap per query, [nq][pitch]; NULL with pitch 0:
 * every row allowed.  Bits at or past n are ignored.  The result is exactly sgpt_ivf_search's over the allowed rows of
 * each query's probed lists (same scores, order and tie rule, tail (-inf, -1)); a masked row never appears.  The probes
 * are the caller's and do not see the mask.  sgpt_ivf_search(..., mask, ...) is this call with pitch 0, and the workspace
 * is the same.  SGPT_ERR_INVALID, before any CUDA call, for sgpt_ivf_search's rejections and, as in the masked searches,
 * a negative pitch, 0 < pitch < ceil(n/32) and a non-zero pitch with a NULL mask.
 * ------------------------------------------------------------------------------------------------------------------ */
int64_t sgpt_ivf_search_workspace_bytes(int dtype, int nq, int nlist, int nprobe, int64_t max_list_len, int D);
int sgpt_ivf_search(int dtype, const void* Q, const void* C, const float* q_scale, const float* c_scale, int nq,
                    int64_t n, int D, const int64_t* list_offsets, int nlist, int64_t max_list_len,
                    const int32_t* doc_ids, const int32_t* probes, int nprobe, int k, const uint32_t* mask,
                    float* out_scores, int64_t* out_ids, void* ws, int64_t ws_bytes, sgpt_stream_t stream);
int sgpt_ivf_search_masked(int dtype, const void* Q, const void* C, const float* q_scale, const float* c_scale, int nq,
                           int64_t n, int D, const int64_t* list_offsets, int nlist, int64_t max_list_len,
                           const int32_t* doc_ids, const int32_t* probes, int nprobe, int k, const uint32_t* mask,
                           int64_t mask_pitch_words, float* out_scores, int64_t* out_ids, void* ws, int64_t ws_bytes,
                           sgpt_stream_t stream);

/* sgpt_ivf_range_search: threshold (range) search over the same lists.  Every input means what it means in
 * sgpt_ivf_search_masked, with `threshold` in place of k.  Query q's result is every position of its probed lists whose
 * score is >= threshold (a NaN score counts as -1), which the mask allows and whose doc_ids entry is >= 0, with the
 * exact search's score bits: exactly the set sgpt_range_search_masked returns over those positions.
 *   out_counts  int64 [nq] (device), always written.  The entries go to out_scores fp32 / out_ids int64 (global ids)
 *               [cap] in query order, query q's at [off[q], off[q] + counts[q]) with off the exclusive sum of the counts,
 *               if and only if off[q] + counts[q] <= cap; entries that do not fit are not written (those slots keep their
 *               bits), and cap = 0 only counts.  The running offset carries across blocks of 256 queries on the device,
 *               with no host synchronisation.
 *   order       within a query, its probes in the order given, and within each probe ascending list position.  This is
 *               NOT id order: sort by (query, id) for the order of sgpt_range_search.  No atomics decide any order, so a
 *               second launch returns the same bits.
 * The workspace holds sgpt_ivf_search's plus the compaction's per-pair and per-query offsets; the device inputs bound
 * every access as in sgpt_ivf_search.  SGPT_ERR_INVALID, before any CUDA call, for sgpt_ivf_search_masked's rejections
 * other than those about k, a NaN threshold, cap < 0, a null out_counts, null out_scores or out_ids with cap > 0, and a
 * workspace smaller than sgpt_ivf_range_search_workspace_bytes (which returns -1 for arguments the search rejects). */
int64_t sgpt_ivf_range_search_workspace_bytes(int dtype, int nq, int nlist, int nprobe, int64_t max_list_len, int D);
int sgpt_ivf_range_search(int dtype, const void* Q, const void* C, const float* q_scale, const float* c_scale, int nq,
                          int64_t n, int D, const int64_t* list_offsets, int nlist, int64_t max_list_len,
                          const int32_t* doc_ids, const int32_t* probes, int nprobe, float threshold,
                          const uint32_t* mask, int64_t mask_pitch_words, int64_t* out_counts, int64_t cap,
                          float* out_scores, int64_t* out_ids, void* ws, int64_t ws_bytes, sgpt_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * IVF-PQ search: the IVF lists above with every document stored as m product-quantization codes of 8 or 4 bits instead
 * of its row, scanned from per-query lookup tables, plus an exact re-rank of a short candidate list against a stored shard.
 *
 * Definitions.  D, m, dsub = D / m, nbits in {4, 8}: K = 2^nbits codewords per sub-quantizer.  m % 16 == 0, and
 * m % 32 == 0 for nbits = 4 (a document's code row of m nbits / 8 bytes starts 16-byte aligned, so a run of list
 * positions is one aligned byte range), D % m == 0 and D % 8 == 0.  The entry points without _nbits take nbits = 8.
 *   Code row: nbits = 8: code[j] is byte j.  nbits = 4: code[j] is in byte j >> 1, the low nibble for even j and the
 *     high nibble for odd j (byte i = code[2i] | code[2i+1] << 4).
 *   Stored document: x~ = normalize(x) for cos_sim, x for dot, x the stored row of the source (an int8 row dequantized
 *     with its scale).  Residual r = x~ - c[list(x)] (c: the coarse centroids fp32 [nlist, D]).  Code:
 *     code[j] = argmin_c ||r[j dsub .. (j+1) dsub) - B[j][c]||^2 (B: the codebooks fp32 [m, K, dsub]), ties to the
 *     lowest c.  (The library's encoder evaluates it in fp32: d = 0; for t ascending: e = r_t - B_t, d = d + e * e,
 *     each operation rounded on its own.)
 *   Query: q~ = F.normalize(q) for cos_sim, q for dot, in fp32.
 *   Tables: lut[q][j][c] = sum_t q~[j dsub + t] B[j][c][t] and base[q][p] = sum_t q~[t] c[probe[q][p]][t], both fp32 FMA
 *     chains from 0 in ascending t.
 *   ADC score of the document at list position pos for the pair (q, p):
 *     acc = 0; for j = 0 .. m-1: acc += lut[q][j][codes[pos][j]]   (plain fp32 adds, in this order, never reassociated)
 *     score = fixnan(acc + base[q][p])   (NaN counts as -1).
 *   The order holds however the kernel stages the tables: a document's partial sum carries across table chunks, so a
 *   restatement of these two lines reproduces every device score bit for bit from the device's tables.
 *
 * sgpt_pq_tables[_nbits]: lut_out fp32 [nq, m, K] and base_out fp32 [nq, nprobe] of Q fp32 [nq, D] (q~, already
 *   normalized for cos_sim), codebooks fp32 [m, K, dsub], centroids fp32 [nlist, D], probes int32 [nq, nprobe].  A
 *   probe outside [0, nlist) is skipped: no centroid is read and its base is 0.  SGPT_ERR_INVALID, before any CUDA
 *   call, for nq < 0, D not a positive multiple of 8, m not a positive multiple of 16 or above 4096, nbits not 4 or 8,
 *   nbits = 4 with m % 32 != 0, D % m != 0, nlist < 1, nprobe outside [1, nlist] and null pointers.
 *
 * sgpt_ivfpq_search[_nbits]: per query, the top-k by ADC score over its probed positions that the mask allows and whose doc_ids
 *   entry is >= 0: score descending, ties by ascending global id, tail (-inf, -1).  This is sgpt_ivf_search's contract
 *   with the ADC score in place of the dot product.
 *   lut, base   the tables of sgpt_pq_tables for these queries and probes (device; lut 16-byte aligned).
 *   codes       uint8 [n, m nbits / 8] in list order (device, 16-byte aligned); list l is positions
 *               [list_offsets[l], list_offsets[l+1]).  list_offsets, max_list_len, doc_ids, probes and mask (the shared
 *               bitmap of allowed positions, pitch 0, or NULL) as in sgpt_ivf_search.
 *   Any nq (blocks of 256 queries reuse ws); no host synchronisation.  Offsets are clamped and skipped probes never read
 *   as in sgpt_ivf_search, so inconsistent device inputs give wrong results, never an out-of-bounds access.
 *   SGPT_ERR_INVALID, before any CUDA call, for sgpt_ivf_search's rejections with the same wording (nq < 0, nlist < 1,
 *   nprobe outside [1, nlist], k outside [1, 4096], n outside [0, 2^31), max_list_len outside [0, n], nprobe x
 *   max_list_len beyond the selection's 2^32 entries, null inputs or outputs, a workspace smaller than
 *   sgpt_ivfpq_search_workspace_bytes), and m not a positive multiple of 16 or above 4096, nbits not 4 or 8, nbits = 4
 *   with m % 32 != 0, and an unaligned lut or codes.  The workspace query returns -1 for the size arguments the search
 *   rejects.  The workspace does not depend on the code width: sgpt_ivfpq_search_workspace_bytes serves both widths.
 *
 * sgpt_ivfpq_search_masked: sgpt_ivfpq_search_nbits with a filter, shared or per query, in the mask format of
 *   sgpt_ivf_search_masked, indexed by list position (the rows of codes): mask_pitch_words = 0: one bitmap
 *   [ceil(n/32)] shared by all queries; mask_pitch_words >= ceil(n/32): one bitmap per query, [nq][pitch]; NULL with
 *   pitch 0: every position allowed.  Bits at or past n are ignored.  A position the mask does not allow is an empty
 *   slot, as a negative doc_ids entry is, so the result is the top-k by ADC score over the probed positions that query
 *   q's bitmap allows and whose doc_ids entry is >= 0 (same scores, order and tie rule, tail (-inf, -1)); a masked
 *   position never appears.  The probes are the caller's and do not see the mask.  sgpt_ivfpq_search[_nbits](..., mask,
 *   ...) is this call with pitch 0, and the workspace is the same (sgpt_ivfpq_search_workspace_bytes).
 *   SGPT_ERR_INVALID, before any CUDA call, for sgpt_ivfpq_search_nbits's rejections and, as in sgpt_ivf_search_masked,
 *   a negative pitch, 0 < pitch < ceil(n/32) and a non-zero pitch with a NULL mask.
 *
 * sgpt_rerank: the exact score of each candidate against a stored shard, then its top-k.  dtype, Q, C, q_scale,
 *   c_scale, D, n and id_base mean what they mean in sgpt_search_masked (Q and C 16-byte aligned).  cand_ids int64
 *   [nq, kc] (device): global ids; a candidate < 0 or outside [id_base, id_base + n) is an empty slot, and the valid
 *   candidates of one query must be distinct.  out_scores fp32 [nq, k], out_ids int64 [nq, k]: the top-k of the
 *   candidates' scores with the exact search's tie rule (score descending, ids ascending), tail (-inf, -1).
 *   int8:  acc = the exact s32 dot product, score = fixnan(float_rn(acc) * q_scale[q] * c_scale[row]) in the filter
 *          epilogue's order: bit-identical to sgpt_search_masked's score of that document.
 *   bf16:  every product is exact in fp32.  Lane l (0..31) sums the 8-element groups g = l, l + 32, l + 64, ... of the
 *          row in ascending g, and each group's elements in ascending order (acc_l += Q[8g+i] C[8g+i], one rounding per
 *          add); then for o = 16, 8, 4, 2, 1: acc_l = acc_l + acc_(l xor o) for every lane; score =
 *          fixnan(acc_0 * q_scale[q] * c_scale[row]).  Reproducible in numpy bit for bit; within fp32 rounding of the
 *          tensor-core sum of sgpt_search_masked.
 *   SGPT_ERR_INVALID, before any CUDA call, for an unknown dtype, nq < 0, kc outside [1, 2^24], the D rules of the
 *   dtype, n outside [0, 2^31), id_base < 0 or id_base + n > 2^31, k outside [1, 4096], null inputs or outputs, an
 *   unaligned Q or C and a workspace smaller than sgpt_rerank_workspace_bytes (which returns -1 for bad nq / kc).
 * ------------------------------------------------------------------------------------------------------------------ */
int sgpt_pq_tables(const float* Q, const float* codebooks, const float* centroids, const int32_t* probes, int nq, int D,
                   int m, int nlist, int nprobe, float* lut_out, float* base_out, sgpt_stream_t stream);
int64_t sgpt_ivfpq_search_workspace_bytes(int nq, int nlist, int nprobe, int64_t max_list_len, int m);
int sgpt_ivfpq_search(const float* lut, const float* base, const uint8_t* codes, int nq, int64_t n, int m,
                      const int64_t* list_offsets, int nlist, int64_t max_list_len, const int32_t* doc_ids,
                      const int32_t* probes, int nprobe, int k, const uint32_t* mask, float* out_scores,
                      int64_t* out_ids, void* ws, int64_t ws_bytes, sgpt_stream_t stream);
int sgpt_pq_tables_nbits(const float* Q, const float* codebooks, const float* centroids, const int32_t* probes,
                         int nq, int D, int m, int nbits, int nlist, int nprobe, float* lut_out, float* base_out,
                         sgpt_stream_t stream);
int sgpt_ivfpq_search_nbits(const float* lut, const float* base, const uint8_t* codes, int nq, int64_t n, int m,
                            int nbits, const int64_t* list_offsets, int nlist, int64_t max_list_len,
                            const int32_t* doc_ids, const int32_t* probes, int nprobe, int k, const uint32_t* mask,
                            float* out_scores, int64_t* out_ids, void* ws, int64_t ws_bytes, sgpt_stream_t stream);
int sgpt_ivfpq_search_masked(const float* lut, const float* base, const uint8_t* codes, int nq, int64_t n, int m,
                             int nbits, const int64_t* list_offsets, int nlist, int64_t max_list_len,
                             const int32_t* doc_ids, const int32_t* probes, int nprobe, int k, const uint32_t* mask,
                             int64_t mask_pitch_words, float* out_scores, int64_t* out_ids, void* ws, int64_t ws_bytes,
                             sgpt_stream_t stream);
int64_t sgpt_rerank_workspace_bytes(int nq, int64_t kc);
int sgpt_rerank(int dtype, const void* Q, const void* C, const float* q_scale, const float* c_scale, int nq, int64_t n,
                int D, int64_t id_base, const int64_t* cand_ids, int64_t kc, int k, float* out_scores,
                int64_t* out_ids, void* ws, int64_t ws_bytes, sgpt_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Graph index: a fixed-degree, pruned k-NN graph over a stored shard, searched by a beam search (one CTA per query, one
 * launch per batch).  Positions are local rows of the shard (0 .. n-1); results carry global ids id_base + position.
 *
 * sgpt_graph_prune: rank-based detour pruning of k-NN lists, an exact integer contract.
 *   knn      int32 [n, K] (device): row a lists its candidate neighbours, best first.  An entry outside [0, n), equal to
 *            a, or equal to an earlier entry of the same row is empty; the others are the row's valid entries.
 *   detours  for each valid entry i of row a: d_i = #{ j < i : knn[a][j] is valid and knn[a][i] occurs in
 *            knn[knn[a][j]][0 .. i-1] } (raw entries of that row, valid or not).
 *   out      int32 [n, degree] (device): the valid entries of row a ordered by (d_i ascending, i ascending), cut to
 *            degree, padded with -1.
 *   The counts are integers, so the output does not depend on the order of the atomics that count them.
 *   SGPT_ERR_INVALID, before any CUDA call, for n outside [0, 2^31), degree not a multiple of 16 in [16, 128], K outside
 *   [degree, 256] and null pointers.
 *
 * sgpt_graph_search: per query, a beam search over graph int32 [n, degree] (device; entries outside [0, n) are empty).
 *   dtype, Q, C, q_scale, c_scale, D, n and id_base mean what they mean in sgpt_rerank (bf16 and int8 only), and
 *   s(q, x) is sgpt_rerank's score of query q against position x, bit for bit.  Keys order entries by score descending
 *   (-0 = +0) and ties by ascending position; scores are never NaN (NaN counts as -1).
 *   seeds    int32 [nq, num_seeds] (device) of positions, or NULL for hashed seeds.
 *   mask     shared bitmap of the ALLOWED positions (the format of the masked searches, pitch 0), or NULL.
 *   out_scores fp32 [nq, k], out_ids int64 [nq, k], out_visited int32 [nq] or NULL (device).
 *   Per query q (q = its row in this call):
 *     V = {} (visited), B = [] (entries (s, x, expanded), kept in key order)
 *     S = seeds[q][0 .. num_seeds-1] (entries outside [0, n) skipped), or, with seeds == NULL,
 *         S_j = h(seed, q, j) mod n for j < num_seeds, where h is, in uint32 arithmetic (mod 2^32):
 *           x = seed + 0x9E3779B1 q + 0x85EBCA77 j; x ^= x >> 16; x *= 0x85EBCA6B; x ^= x >> 13; x *= 0xC2B2AE35;
 *           x ^= x >> 16; h = x
 *     every x in S not in V: add x to V and score it; B = the best itopk of them, all unexpanded
 *     for t in 0 .. max_iterations-1:
 *       P = the first search_width unexpanded entries of B; stop if P is empty; mark them expanded
 *       every e in graph[p][0 .. degree-1] for p in P with 0 <= e < n and e not in V: add e to V and score it
 *       B = the best itopk entries of B and the newly scored ones (flags carried)
 *     output: the first k entries of B whose position the mask allows, as (s, id_base + x); tail (-inf, -1)
 *     out_visited[q] = |V|
 *   The result does not depend on the order in which threads insert into V.  Disallowed (deleted) positions are still
 *   scored and expanded; they are only never returned.  The visited set is an exact table of
 *   next_pow2(2 (num_seeds + max_iterations search_width degree)) slots in shared memory, never more than half full.
 *   SGPT_ERR_INVALID, before any CUDA call, for a dtype other than bf16 and int8, nq < 0, the D rules of the dtype,
 *   n outside [1, 2^31), id_base < 0 or id_base + n > 2^31, itopk not a multiple of 32 in [32, 512], k outside
 *   [1, itopk], degree < 1, search_width outside [1, 8], search_width x degree > 512, num_seeds outside [1, 512],
 *   max_iterations < 1 or 2 (num_seeds + max_iterations search_width degree) > 32768, null Q, C, graph, out_scores or
 *   out_ids, and an unaligned Q or C.
 *
 * sgpt_graph_search_filtered: sgpt_graph_search with a filter, shared or per query, in the mask format of the masked
 *   searches: mask_pitch_words = 0: one bitmap [ceil(n/32)] of the ALLOWED positions, or NULL (every position allowed);
 *   mask_pitch_words >= ceil(n/32): one bitmap per query, [nq][pitch].  Bits at or past n are ignored.
 *   The walk does not see the mask: V, B, every P, the stopping rule and out_visited are exactly those of
 *   sgpt_graph_search with the same arguments, and disallowed positions are still scored and expanded.
 *     output: the best k entries of {x in V : the mask allows x for query q} in key order (score descending, ties by
 *     ascending position), as (s, id_base + x), s bit for bit sgpt_rerank's score; tail (-inf, -1)
 *   The final B is the top-itopk of V, so with a NULL or all-ones mask the output equals sgpt_graph_search's with
 *   mask = NULL, bit for bit.  A tail (-inf, -1) means V holds fewer than k allowed positions, not that the shard does.
 *   The best k allowed keys are kept in next_pow2(k + max(num_seeds, search_width degree)) further 8-byte slots of shared
 *   memory (at most 8 KB).  SGPT_ERR_INVALID, before any CUDA call, for every rejection of sgpt_graph_search and, as in
 *   the masked searches, a negative pitch, 0 < pitch < ceil(n/32) and a non-zero pitch with a NULL mask.
 *
 * sgpt_graph_prune_append: the detour pruning of m rows appended to a graph over n_old rows, for rows a = n_old + r,
 *   r < m.  Row a's list is L = knn[r] (int32 [m, K], device, local positions); an entry is empty if it lies outside
 *   [0, n_old + m), equals a, or repeats an earlier entry of L.  The list of a position b is graph[b][0 .. degree-1]
 *   (int32 [n_old, degree], device) for b < n_old and knn[b - n_old] for b >= n_old.  d_i = #{ j < i : L[j] is valid and
 *   L[i] occurs in list(L[j])[0 .. i-1] } (raw entries); out[r] (int32 [m, degree], device) holds the valid entries of
 *   L ordered by (d_i ascending, i ascending), cut to degree, padded with -1.  One CTA per new row; the old rows are
 *   never launched over.  With n_old = 0 (graph may then be NULL) this is exactly sgpt_graph_prune of knn.
 *   SGPT_ERR_INVALID, before any CUDA call, for a negative n_old or m, n_old + m >= 2^31, degree not a multiple of 16 in
 *   [16, 128], K outside [degree, 256], a null graph with n_old > 0, and a null knn or out.
 * ------------------------------------------------------------------------------------------------------------------ */
int sgpt_graph_prune(const int32_t* knn, int64_t n, int K, int degree, int32_t* out, sgpt_stream_t stream);
int sgpt_graph_search(int dtype, const void* Q, const void* C, const float* q_scale, const float* c_scale, int nq,
                      int64_t n, int D, int64_t id_base, const int32_t* graph, int degree, const int32_t* seeds,
                      int num_seeds, uint32_t seed, int itopk, int search_width, int max_iterations, int k,
                      const uint32_t* mask, float* out_scores, int64_t* out_ids, int32_t* out_visited,
                      sgpt_stream_t stream);
int sgpt_graph_search_filtered(int dtype, const void* Q, const void* C, const float* q_scale, const float* c_scale,
                               int nq, int64_t n, int D, int64_t id_base, const int32_t* graph, int degree,
                               const int32_t* seeds, int num_seeds, uint32_t seed, int itopk, int search_width,
                               int max_iterations, int k, const uint32_t* mask, int64_t mask_pitch_words,
                               float* out_scores, int64_t* out_ids, int32_t* out_visited, sgpt_stream_t stream);
int sgpt_graph_prune_append(const int32_t* graph, int64_t n_old, int degree, const int32_t* knn, int64_t m, int K,
                            int32_t* out, sgpt_stream_t stream);

/* bf16 -> fp32 conversion of count elements (count % 4 == 0), e.g. of the residual stream. */
int sgpt_bf16_to_f32(const void* x, float* y, int64_t count, sgpt_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Measurement hooks (bench.py): launch counters are always on; with profiling enabled every kernel launch issued
 * through this library is bracketed by CUDA events on its stream.  sgpt_profile_read waits for them, returns the
 * summed device milliseconds and launch counts per category since the previous read, and resets the timed set.
 * Categories: 0 embed, 1 layernorm, 2 linear GEMM, 3 attention, 4 pool, 5 similarity GEMM, 6 top-k, 7 misc.
 * ------------------------------------------------------------------------------------------------------------------ */
#define SGPT_NUM_LAUNCH_CATEGORIES 8
int sgpt_profile_enable(int on);
int sgpt_profile_read(double* ms_by_cat, int64_t* timed_launches_by_cat, int64_t* total_launches_by_cat);
/* SM clock the GEMM kernels actually ran at: every GEMM launch has one thread read %clock64 and %globaltimer
 * at its start and end and accumulate both deltas on the device.  Returns the accumulated SM cycles and nanoseconds
 * since the previous call (cycles / ns = GHz under load, which nvidia-smi sampling cannot resolve) and resets them.
 * Synchronises the device. */
int sgpt_profile_gemm_clock(double* sm_cycles, double* nanoseconds);
/* Phase timeline of the most recent exact-selection launch (topk.cu): %globaltimer nanoseconds stamped by CTA 0 at
 * [0] kernel entry, [1] predecessor complete, [2] front/back decision, [3] list offsets, [4] keys in shared memory,
 * [5] sample pivot, [6] compaction, [7] exact k-th key, [8] winners placed + ids fetched, [9] sorted, [10] outputs
 * written.  n <= 16.  Synchronises the device.  A measurement aid, not part of any reference interface. */
int sgpt_debug_topk_timeline(uint64_t* stamps_ns, int n);

#ifdef __cplusplus
}
#endif
#endif /* SGPT_B200_H_ */
