// Whole-encoder handle: token ids -> GPT forward (F1..F7) -> pooled embeddings (P1/P2) in one C call.
// Replaces `self.model(**batch_tokens, output_hidden_states=True)` + the pooling block of the reference
// (biencoder/beir/beir_dense_retriever.py:205, :233-304).  Three block layouts (SURVEY.md §8 model table):
//   GPT-Neo  HF:gpt_neo/modeling_gpt_neo.py:320-350   ln_1 -> attn (unscaled QK^T, local window on odd layers) -> +res
//                                                       -> ln_2 -> c_fc/gelu_new/c_proj -> +res
//   GPT-J    HF:gptj/modeling_gptj.py:390-415          ln_1 -> {attn (rotary q,k; 1/sqrt(hd)), fc_in/gelu_new/fc_out}
//                                                       in parallel on the SAME ln_1 output -> res + attn + mlp
//   BLOOM    HF:bloom/modeling_bloom.py:340-420        LN(word_emb) -> input_layernorm -> attn (ALiBi, 1/sqrt(hd), qkv
//                                                       bias) -> +res -> post_attention_layernorm -> mlp (tanh gelu) -> +res
// The handle borrows the caller's weight buffers and owns only its activation workspace, laid out for a ragged batch
// of at most cfg.max_tokens rows:
//     resid bf16[T,d] | xb bf16[T,d] | qkv bf16[T,3d] | attn bf16[T,d] | ffn bf16[T,ff] | stats fp32[2T+B]
// and, with fp8 linear layers (sgpt_model_create_fp8), the quantized A operand of the next GEMM:
//     xq e4m3[T, max(d,ff)] | xs fp32[T]
//
// Each block runs LayerNorm as a pass of its own (residual stream -> bf16 xb), then GEMMs with bias / gelu epilogues for
// the layers that read xb and bf16 reduce-add epilogues for the layers that update the bf16 residual stream.
#include <math.h>
#include <string.h>

#include <vector>

#include "../../include/sgpt_b200.h"
#include "gemm_api.h"
#include "host_utils.h"

struct sgpt_model {
  sgpt_model_config cfg;
  sgpt_model_weights w;
  std::vector<sgpt_layer_weights> layers;
  std::vector<sgpt_fp8_layer_weights> fp8_layers;  // non-empty: the linear layers run in fp8
  void* xq = nullptr;     // fp8: e4m3 rows of the GEMM's A operand
  float* xs = nullptr;    // fp8: their scales
  int device = 0;
  void* resid = nullptr;  // the residual stream, bf16
  void* xn = nullptr;     // xb: LayerNorm output, the A operand of the QKV / c_fc GEMMs
  void* qkv = nullptr;
  void* attn = nullptr;
  void* ffn = nullptr;
  float* stats = nullptr;
  float* rotary = nullptr;  // GPT-J: (cos, sin)[max_pos, rotary_dim/2]
  float* alibi = nullptr;   // BLOOM: slopes[n_head]
  const float* pool_w = nullptr;  // learnt position weights (borrowed), see sgpt_model_set_position_weights
  int n_pool_w = 0;
  int last_T = 0;
};

using namespace sgpt;

extern "C" int sgpt_abi_version(void) { return SGPT_ABI_VERSION; }

// build_alibi_tensor slopes, HF:bloom/modeling_bloom.py:62-78
static std::vector<float> alibi_slopes(int n_head) {
  const int cp2 = 1 << static_cast<int>(floor(log2(static_cast<double>(n_head))));
  std::vector<float> s;
  const float base = static_cast<float>(pow(2.0, -pow(2.0, -(log2(static_cast<double>(cp2)) - 3.0))));
  for (int i = 1; i <= cp2; ++i) s.push_back(powf(base, static_cast<float>(i)));
  if (cp2 != n_head) {
    const float extra = static_cast<float>(pow(2.0, -pow(2.0, -(log2(2.0 * cp2) - 3.0))));
    const int rem = n_head - cp2 < cp2 ? n_head - cp2 : cp2;
    for (int i = 0; i < rem; ++i) s.push_back(powf(extra, static_cast<float>(1 + 2 * i)));
  }
  return s;
}

// fp8_layers == nullptr: the bf16 handle (sgpt_model_create)
static int model_create(const sgpt_model_config* cfg, const sgpt_model_weights* w,
                        const sgpt_fp8_layer_weights* fp8_layers, sgpt_model_t* out) {
  SGPT_REQUIRE(cfg != nullptr && w != nullptr && out != nullptr, "sgpt_model_create: null argument");
  *out = nullptr;
  SGPT_REQUIRE(cfg->arch == SGPT_ARCH_GPT_NEO || cfg->arch == SGPT_ARCH_GPTJ || cfg->arch == SGPT_ARCH_BLOOM,
               "sgpt_model_create: unknown arch %d", cfg->arch);
  SGPT_REQUIRE(cfg->n_layer > 0 && cfg->d_model > 0 && cfg->n_head > 0 && cfg->d_ff > 0, "sgpt_model_create: bad dims");
  SGPT_REQUIRE(cfg->d_model % cfg->n_head == 0, "sgpt_model_create: d_model %% n_head != 0");
  const int hd = cfg->d_model / cfg->n_head;
  SGPT_REQUIRE(hd == 64 || hd == 128 || hd == 256, "sgpt_model_create: head_dim %d not in {64,128,256}", hd);
  SGPT_REQUIRE(cfg->d_model % 64 == 0 && cfg->d_ff % 64 == 0, "sgpt_model_create: d_model and d_ff must be multiples of 64");
  SGPT_REQUIRE(cfg->max_tokens > 0 && cfg->max_batch > 0, "sgpt_model_create: max_tokens/max_batch must be positive");
  SGPT_REQUIRE(w->wte != nullptr && w->lnf_g != nullptr && w->lnf_b != nullptr && w->layers != nullptr,
               "sgpt_model_create: missing weights");
  if (cfg->arch == SGPT_ARCH_GPT_NEO) SGPT_REQUIRE(w->wpe != nullptr, "sgpt_model_create: GPT-Neo needs wpe");
  if (cfg->arch == SGPT_ARCH_GPTJ)
    SGPT_REQUIRE(cfg->rotary_dim > 0 && cfg->rotary_dim <= hd && cfg->rotary_dim % 8 == 0 && cfg->max_pos > 0,
                 "sgpt_model_create: GPT-J needs 0 < rotary_dim <= head_dim, multiple of 8");
  if (cfg->arch == SGPT_ARCH_BLOOM)
    SGPT_REQUIRE(w->emb_ln_g != nullptr && w->emb_ln_b != nullptr, "sgpt_model_create: BLOOM needs the embedding LayerNorm");

  sgpt_model* m = new sgpt_model();
  m->cfg = *cfg;
  m->w = *w;
  m->layers.assign(w->layers, w->layers + cfg->n_layer);
  m->w.layers = m->layers.data();
  if (fp8_layers != nullptr) m->fp8_layers.assign(fp8_layers, fp8_layers + cfg->n_layer);
  for (int l = 0; l < cfg->n_layer; ++l) {
    const sgpt_layer_weights& lw = m->layers[l];
    const bool need_ln2 = cfg->arch != SGPT_ARCH_GPTJ;
    const bool linear_ok = fp8_layers != nullptr
                               ? (fp8_layers[l].w_qkv && fp8_layers[l].s_qkv && fp8_layers[l].w_o && fp8_layers[l].s_o &&
                                  fp8_layers[l].w_fc && fp8_layers[l].s_fc && fp8_layers[l].w_proj && fp8_layers[l].s_proj)
                               : (lw.w_qkv && lw.w_o && lw.w_fc && lw.w_proj);
    if (!lw.ln1_g || !lw.ln1_b || !linear_ok || (need_ln2 && (!lw.ln2_g || !lw.ln2_b))) {
      delete m;
      set_error("sgpt_model_create: layer %d has missing weights", l);
      return SGPT_ERR_INVALID;
    }
  }
  cudaError_t e = cudaGetDevice(&m->device);
  const size_t T = static_cast<size_t>(cfg->max_tokens), d = static_cast<size_t>(cfg->d_model);
  if (e == cudaSuccess) e = cudaMalloc(&m->resid, T * d * 2);
  if (e == cudaSuccess) e = cudaMalloc(&m->xn, T * d * 2);
  if (e == cudaSuccess) e = cudaMalloc(&m->qkv, T * d * 3 * 2);
  if (e == cudaSuccess) e = cudaMalloc(&m->attn, T * d * 2);
  if (e == cudaSuccess) e = cudaMalloc(&m->ffn, T * static_cast<size_t>(cfg->d_ff) * 2);
  // (mean, rstd) per row for ln_f, then the per-sequence sums of squares of the normalisation (sgpt_pool)
  if (e == cudaSuccess) e = cudaMalloc(&m->stats, (2 * T + static_cast<size_t>(cfg->max_batch)) * 4);
  if (e == cudaSuccess && fp8_layers != nullptr) {
    e = cudaMalloc(&m->xq, T * static_cast<size_t>(cfg->d_ff > cfg->d_model ? cfg->d_ff : cfg->d_model));
    if (e == cudaSuccess) e = cudaMalloc(&m->xs, T * 4);
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e == cudaSuccess && cfg->arch == SGPT_ARCH_GPTJ) {
    // create_sinusoidal_positions, HF:gptj/modeling_gptj.py:45-48: angle(p, i) = p * 10000^(-2i/rotary_dim), fp32
    const int half = cfg->rotary_dim / 2;
    std::vector<float> tab(static_cast<size_t>(cfg->max_pos) * half * 2);
    for (int p = 0; p < cfg->max_pos; ++p)
      for (int i = 0; i < half; ++i) {
        const float inv_freq = 1.0f / powf(10000.0f, static_cast<float>(2 * i) / static_cast<float>(cfg->rotary_dim));
        const float ang = static_cast<float>(p) * inv_freq;
        tab[(static_cast<size_t>(p) * half + i) * 2 + 0] = static_cast<float>(cos(static_cast<double>(ang)));
        tab[(static_cast<size_t>(p) * half + i) * 2 + 1] = static_cast<float>(sin(static_cast<double>(ang)));
      }
    e = cudaMalloc(&m->rotary, tab.size() * 4);
    if (e == cudaSuccess) e = cudaMemcpy(m->rotary, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice);
  }
  if (e == cudaSuccess && cfg->arch == SGPT_ARCH_BLOOM) {
    const std::vector<float> s = alibi_slopes(cfg->n_head);
    e = cudaMalloc(&m->alibi, s.size() * 4);
    if (e == cudaSuccess) e = cudaMemcpy(m->alibi, s.data(), s.size() * 4, cudaMemcpyHostToDevice);
  }
  if (e != cudaSuccess) {
    set_error("sgpt_model_create: workspace allocation failed: %s", cudaGetErrorString(e));
    sgpt_model_destroy(m);
    return SGPT_ERR_CUDA;
  }
  *out = m;
  return SGPT_OK;
}

extern "C" int sgpt_model_create(const sgpt_model_config* cfg, const sgpt_model_weights* w, sgpt_model_t* out) {
  return model_create(cfg, w, nullptr, out);
}

extern "C" int sgpt_model_create_fp8(const sgpt_model_config* cfg, const sgpt_model_weights* w,
                                     const sgpt_fp8_layer_weights* fp8_layers, sgpt_model_t* out) {
  SGPT_REQUIRE(fp8_layers != nullptr, "sgpt_model_create_fp8: null fp8 layer weights");
  return model_create(cfg, w, fp8_layers, out);
}

extern "C" void sgpt_model_destroy(sgpt_model_t m) {
  if (!m) return;
  cudaFree(m->resid);
  cudaFree(m->xn);
  cudaFree(m->qkv);
  cudaFree(m->attn);
  cudaFree(m->ffn);
  cudaFree(m->stats);
  cudaFree(m->rotary);
  cudaFree(m->alibi);
  cudaFree(m->xq);
  cudaFree(m->xs);
  delete m;
}

#define SGPT_TRY(call)              \
  do {                              \
    int _rc = (call);               \
    if (_rc != SGPT_OK) return _rc; \
  } while (0)

constexpr int kNoPooling = -1;  // internal pool_mode of sgpt_forward: run the blocks, leave the residual stream

extern "C" int sgpt_encode(sgpt_model_t m, const int32_t* ids, const int32_t* pos, const int32_t* cu_seqlens, int B,
                           int T, int max_seqlen, int layer_idx, int pool_mode, int clamp_denominator, int normalize,
                           float* out, sgpt_stream_t stream) {
  SGPT_REQUIRE(m != nullptr, "sgpt_encode: null model");
  SGPT_REQUIRE(pool_mode == kNoPooling || (pool_mode >= SGPT_POOL_MEAN && pool_mode <= SGPT_POOL_LASTTOKENMEAN),
               "sgpt_encode: unknown pooling mode %d", pool_mode);
  SGPT_REQUIRE(pool_mode == kNoPooling || out != nullptr, "sgpt_encode: null output");
  const sgpt_model_config& c = m->cfg;
  SGPT_REQUIRE(B >= 0 && T >= 0, "sgpt_encode: negative sizes");
  SGPT_REQUIRE(T <= c.max_tokens && B <= c.max_batch, "sgpt_encode: batch (B=%d, T=%d) exceeds workspace (B<=%d, T<=%d)",
               B, T, c.max_batch, c.max_tokens);
  SGPT_REQUIRE(c.arch == SGPT_ARCH_BLOOM || max_seqlen <= c.max_pos,
               "sgpt_encode: max_seqlen %d exceeds max_position_embeddings %d", max_seqlen, c.max_pos);
  // meanmean / lasttokenmean (BDR:243-257, 284-301) average the mean / last-token embedding of ALL L+1 hidden states
  const bool all_layers = (pool_mode == SGPT_POOL_MEANMEAN || pool_mode == SGPT_POOL_LASTTOKENMEAN);
  const int base_mode = pool_mode == SGPT_POOL_MEANMEAN ? SGPT_POOL_MEAN
                        : pool_mode == SGPT_POOL_LASTTOKENMEAN ? SGPT_POOL_LASTTOKEN : pool_mode;
  const float layer_scale = all_layers ? 1.0f / static_cast<float>(c.n_layer + 1) : 1.0f;
  if (all_layers) layer_idx = c.n_layer;  // the reference ignores layeridx for these modes
  if (layer_idx < 0) layer_idx += c.n_layer + 1;
  SGPT_REQUIRE(layer_idx >= 0 && layer_idx <= c.n_layer, "sgpt_encode: layer index out of range for %d hidden states",
               c.n_layer + 1);
  const float* pool_w = (pool_mode == SGPT_POOL_WEIGHTEDMEAN) ? m->pool_w : nullptr;
  SGPT_REQUIRE(pool_w == nullptr || max_seqlen <= m->n_pool_w,
               "sgpt_encode: max_seqlen %d exceeds the %d learnt position weights", max_seqlen, m->n_pool_w);
  if (B == 0) return SGPT_OK;
  const int d = c.d_model, H = c.n_head, hd = d / H, ff = c.d_ff;
  const float inv_sqrt_hd = 1.0f / sqrtf(static_cast<float>(hd));
  m->last_T = T;

  SGPT_TRY(sgpt_embed_tokens(ids, pos, m->w.wte, c.arch == SGPT_ARCH_GPT_NEO ? m->w.wpe : nullptr, m->resid, T, d,
                             c.vocab, c.max_pos, stream));
  if (c.arch == SGPT_ARCH_BLOOM)
    SGPT_TRY(sgpt_layernorm(m->resid, m->w.emb_ln_g, m->w.emb_ln_b, m->resid, T, d, c.ln_eps, stream));
  const int n_run = layer_idx;  // hidden_states[i] is the input of block i; hidden_states[L] is ln_f(output of block L-1)
  // fp8 linear layers: `quant` turns the bf16 A operand of the next GEMM(s) into m->xq / m->xs, `lin` runs a GEMM on it
  const bool f8 = !m->fp8_layers.empty();
  auto quant = [&](const void* x, int K) { return f8 ? sgpt_quantize_rows_fp8(x, m->xq, m->xs, T, K, stream) : SGPT_OK; };
  auto lin = [&](const void* x, int K, const void* w, const void* wq, const float* ws, const float* b, void* out, int N,
                 int epi) {
    const void* resid = epi == SGPT_EPI_RESID_BF16 ? out : nullptr;
    if (f8) return sgpt_linear_fp8(m->xq, K, m->xs, wq, K, ws, b, out, N, resid, T, N, K, epi, stream);
    return sgpt_linear(x, K, w, K, b, out, N, resid, T, N, K, epi, stream);
  };
  for (int l = 0; l < n_run && l < c.n_layer; ++l) {
    const sgpt_layer_weights& lw = m->layers[l];
    const sgpt_fp8_layer_weights fw = f8 ? m->fp8_layers[l] : sgpt_fp8_layer_weights{};
    if (all_layers)  // hidden_states[l] = the residual stream entering block l (no ln_f)
      SGPT_TRY(sgpt_pool(m->resid, 1, pos, cu_seqlens, nullptr, nullptr, c.ln_eps, nullptr, 0, out, nullptr, B, T, d,
                         base_mode, clamp_denominator, 0, /*accumulate=*/l > 0, layer_scale, stream));
    SGPT_TRY(sgpt_layernorm(m->resid, lw.ln1_g, lw.ln1_b, m->xn, T, d, c.ln_eps, stream));
    SGPT_TRY(quant(m->xn, d));
    if (c.arch == SGPT_ARCH_GPT_NEO) {
      SGPT_TRY(lin(m->xn, d, lw.w_qkv, fw.w_qkv, fw.s_qkv, lw.b_qkv, m->qkv, 3 * d, SGPT_EPI_BF16));
      const int window = (lw.local_attention && c.window > 0 && max_seqlen > c.window) ? c.window : 0;
      SGPT_TRY(sgpt_attention(m->qkv, m->attn, cu_seqlens, B, T, H, hd, /*scale=*/1.0f, window, max_seqlen, nullptr, 0,
                              stream));
      SGPT_TRY(quant(m->attn, d));
      SGPT_TRY(lin(m->attn, d, lw.w_o, fw.w_o, fw.s_o, lw.b_o, m->resid, d, SGPT_EPI_RESID_BF16));
      SGPT_TRY(sgpt_layernorm(m->resid, lw.ln2_g, lw.ln2_b, m->xn, T, d, c.ln_eps, stream));
      SGPT_TRY(quant(m->xn, d));
      SGPT_TRY(lin(m->xn, d, lw.w_fc, fw.w_fc, fw.s_fc, lw.b_fc, m->ffn, ff, SGPT_EPI_GELU_BF16));
      SGPT_TRY(quant(m->ffn, ff));
      SGPT_TRY(lin(m->ffn, ff, lw.w_proj, fw.w_proj, fw.s_proj, lw.b_proj, m->resid, d, SGPT_EPI_RESID_BF16));
    } else if (c.arch == SGPT_ARCH_GPTJ) {
      if (f8)
        SGPT_TRY(sgpt_linear_qkv_rotary_fp8(m->xq, d, m->xs, fw.w_qkv, fw.s_qkv, m->qkv, pos, m->rotary, T, d, hd,
                                            c.rotary_dim, c.max_pos, stream));
      else
        SGPT_TRY(sgpt_linear_qkv_rotary(m->xn, d, lw.w_qkv, m->qkv, pos, m->rotary, T, d, hd, c.rotary_dim, c.max_pos,
                                        stream));
      SGPT_TRY(sgpt_attention(m->qkv, m->attn, cu_seqlens, B, T, H, hd, inv_sqrt_hd, 0, max_seqlen, nullptr, 0, stream));
      // both branches read the same ln_1 output and are accumulated into the residual stream (attn + mlp + residual);
      // with fp8 the quantized ln_1 output is still in xq here
      SGPT_TRY(lin(m->xn, d, lw.w_fc, fw.w_fc, fw.s_fc, lw.b_fc, m->ffn, ff, SGPT_EPI_GELU_BF16));
      SGPT_TRY(quant(m->attn, d));
      SGPT_TRY(lin(m->attn, d, lw.w_o, fw.w_o, fw.s_o, lw.b_o, m->resid, d, SGPT_EPI_RESID_BF16));
      SGPT_TRY(quant(m->ffn, ff));
      SGPT_TRY(lin(m->ffn, ff, lw.w_proj, fw.w_proj, fw.s_proj, lw.b_proj, m->resid, d, SGPT_EPI_RESID_BF16));
    } else {  // BLOOM
      SGPT_TRY(lin(m->xn, d, lw.w_qkv, fw.w_qkv, fw.s_qkv, lw.b_qkv, m->qkv, 3 * d, SGPT_EPI_BF16));
      SGPT_TRY(sgpt_attention(m->qkv, m->attn, cu_seqlens, B, T, H, hd, inv_sqrt_hd, 0, max_seqlen, m->alibi, 0, stream));
      SGPT_TRY(quant(m->attn, d));
      SGPT_TRY(lin(m->attn, d, lw.w_o, fw.w_o, fw.s_o, lw.b_o, m->resid, d, SGPT_EPI_RESID_BF16));
      SGPT_TRY(sgpt_layernorm(m->resid, lw.ln2_g, lw.ln2_b, m->xn, T, d, c.ln_eps, stream));
      SGPT_TRY(quant(m->xn, d));
      SGPT_TRY(lin(m->xn, d, lw.w_fc, fw.w_fc, fw.s_fc, lw.b_fc, m->ffn, ff, SGPT_EPI_GELU_BF16));
      SGPT_TRY(quant(m->ffn, ff));
      SGPT_TRY(lin(m->ffn, ff, lw.w_proj, fw.w_proj, fw.s_proj, lw.b_proj, m->resid, d, SGPT_EPI_RESID_BF16));
    }
  }
  if (pool_mode == kNoPooling) return SGPT_OK;
  const bool final_ln = (layer_idx == c.n_layer);
  SGPT_TRY(sgpt_pool(m->resid, 1, pos, cu_seqlens, final_ln ? m->w.lnf_g : nullptr, final_ln ? m->w.lnf_b : nullptr, c.ln_eps,
                     pool_w, pool_w ? m->n_pool_w : 0, out, m->stats, B, T, d, base_mode, clamp_denominator, normalize,
                     /*accumulate=*/all_layers && c.n_layer > 0, layer_scale, stream));
  return SGPT_OK;
}

extern "C" int sgpt_forward(sgpt_model_t m, const int32_t* ids, const int32_t* pos, const int32_t* cu_seqlens, int B, int T,
                            int max_seqlen, sgpt_stream_t stream) {
  return sgpt_encode(m, ids, pos, cu_seqlens, B, T, max_seqlen, /*layer_idx=*/-1, kNoPooling, 0, 0, nullptr, stream);
}

static inline int64_t lm_lds(int vocab) { return (static_cast<int64_t>(vocab) + 3) & ~int64_t(3); }
static inline int64_t lm_align(int64_t x) { return (x + 255) & ~int64_t(255); }

extern "C" int64_t sgpt_lm_logprobs_workspace_bytes(int d_model, int vocab, int rows_per_chunk) {
  if (d_model <= 0 || vocab <= 0 || rows_per_chunk <= 0) return 0;
  return lm_align(static_cast<int64_t>(rows_per_chunk) * d_model * 2) +
         lm_align(static_cast<int64_t>(rows_per_chunk) * lm_lds(vocab) * 4) + 256;
}

extern "C" int sgpt_lm_logprobs(sgpt_model_t m, const void* lm_head_w, const float* lm_head_bias, int vocab,
                                const int32_t* rows, const int32_t* targets, int M, float* token_logprobs,
                                int32_t* greedy, void* ws, int64_t ws_bytes, int rows_per_chunk, sgpt_stream_t stream) {
  SGPT_REQUIRE(m != nullptr && lm_head_w != nullptr, "sgpt_lm_logprobs: null model or LM head");
  SGPT_REQUIRE(M >= 0 && vocab > 0 && rows_per_chunk > 0, "sgpt_lm_logprobs: bad sizes");
  SGPT_REQUIRE(M == 0 || (rows != nullptr && targets != nullptr && token_logprobs != nullptr),
               "sgpt_lm_logprobs: null argument");
  const int d = m->cfg.d_model;
  SGPT_REQUIRE(ws != nullptr && ws_bytes >= sgpt_lm_logprobs_workspace_bytes(d, vocab, rows_per_chunk),
               "sgpt_lm_logprobs: workspace too small (%lld < %lld bytes)", (long long)ws_bytes,
               (long long)sgpt_lm_logprobs_workspace_bytes(d, vocab, rows_per_chunk));
  // the gathered rows are read by TMA, which needs 16-byte aligned addresses
  SGPT_REQUIRE(reinterpret_cast<uintptr_t>(ws) % 16 == 0, "sgpt_lm_logprobs: ws must be 16-byte aligned");
  uint8_t* w = static_cast<uint8_t*>(ws);
  void* xsel = w;
  float* logits = reinterpret_cast<float*>(w + lm_align(static_cast<int64_t>(rows_per_chunk) * d * 2));
  const int64_t lds = lm_lds(vocab);
  for (int m0 = 0; m0 < M; m0 += rows_per_chunk) {
    const int mc = (M - m0 < rows_per_chunk) ? M - m0 : rows_per_chunk;
    // hidden_states[-1] of the selected positions: ln_f of the residual stream the last sgpt_forward left behind
    SGPT_TRY(sgpt_layernorm_gather(m->resid, rows + m0, m->w.lnf_g, m->w.lnf_b, xsel, mc, d, m->cfg.ln_eps, stream));
    SGPT_TRY(launch_lm_logits(xsel, lm_head_w, logits, lds, mc, vocab, d, static_cast<cudaStream_t>(stream)));
    SGPT_TRY(sgpt_token_logprobs(logits, lds, mc, vocab, lm_head_bias, targets + m0, token_logprobs + m0,
                                 greedy ? greedy + m0 : nullptr, stream));
  }
  return SGPT_OK;
}

extern "C" int sgpt_model_set_position_weights(sgpt_model_t m, const float* w, int n) {
  SGPT_REQUIRE(m != nullptr, "sgpt_model_set_position_weights: null model");
  SGPT_REQUIRE(w == nullptr || n > 0, "sgpt_model_set_position_weights: n must be positive");
  m->pool_w = w;
  m->n_pool_w = w ? n : 0;
  return SGPT_OK;
}

extern "C" int sgpt_model_read_residual(sgpt_model_t m, float* dst, int64_t capacity_elems, int* T, int* d,
                                        sgpt_stream_t stream) {
  SGPT_REQUIRE(m != nullptr && dst != nullptr && T != nullptr && d != nullptr, "sgpt_model_read_residual: null argument");
  *T = m->last_T;
  *d = m->cfg.d_model;
  const int64_t n = static_cast<int64_t>(m->last_T) * m->cfg.d_model;
  SGPT_REQUIRE(capacity_elems >= n, "sgpt_model_read_residual: destination too small");
  return sgpt_bf16_to_f32(m->resid, dst, n, stream);
}
