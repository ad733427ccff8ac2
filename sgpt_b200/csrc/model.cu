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
//     resid fp32[T,d] | xb bf16[T,d] | qkv bf16[T,3d] | attn bf16[T,d] | ffn bf16[T,ff] | stats fp32[2T*P+B]
//
// Two block flows (chosen when the handle is created):
//   default         LayerNorm as its own HBM pass (fp32 residual -> bf16), GEMMs with bias / gelu / reduce-add epilogues.
//   SGPT_LN_FOLD=1  no LayerNorm pass inside the blocks: the kernels that WRITE the residual stream (token embedding;
//                   out-proj / c_proj epilogues, gemm.cuh EpiResidLn) also leave xb = bf16(resid) and per-row partial sums
//                   (sum x, sum x^2 per 128 columns); the GEMMs that consume LN(resid) (QKV, c_fc) run on xb with gamma folded
//                   into their weight columns and apply  y = r (xb W'^T) - r mu c + b'  per row in the epilogue
//                   (OpTmaLnBiasActBF16); ln_f is folded into the pooling kernel the same way.  Parity-tested like the
//                   default; opt-in (every instruction and byte the GEMM epilogues add can cost as much time as the
//                   LayerNorm pass it replaces).
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../include/sgpt_b200.h"
#include "host_utils.h"

struct sgpt_model {
  sgpt_model_config cfg;
  sgpt_model_weights w;
  std::vector<sgpt_layer_weights> layers;
  int device = 0;
  float* resid = nullptr;
  void* xn = nullptr;  // xb: bf16 copy of the residual stream
  int P = 0;           // statistics groups per row = ceil(d / 128)
  bool ln_fold = false;  // SGPT_LN_FOLD=1 at creation
  bool resid_bf16 = true;   // residual stream stored in bf16 (default; SGPT_RESID_BF16=0 at creation: fp32; default flow only)
  float* sumsq = nullptr;
  // LayerNorm-folded parameters per layer (library-owned)
  std::vector<void*> wq_f, wfc_f;
  std::vector<float*> cq, bq, cfc, bfc;
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

extern "C" int sgpt_model_create(const sgpt_model_config* cfg, const sgpt_model_weights* w, sgpt_model_t* out) {
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
  for (int l = 0; l < cfg->n_layer; ++l) {
    const sgpt_layer_weights& lw = m->layers[l];
    const bool need_ln2 = cfg->arch != SGPT_ARCH_GPTJ;
    if (!lw.ln1_g || !lw.ln1_b || !lw.w_qkv || !lw.w_o || !lw.w_fc || !lw.w_proj ||
        (need_ln2 && (!lw.ln2_g || !lw.ln2_b))) {
      delete m;
      set_error("sgpt_model_create: layer %d has missing weights", l);
      return SGPT_ERR_INVALID;
    }
  }
  cudaError_t e = cudaGetDevice(&m->device);
  const size_t T = static_cast<size_t>(cfg->max_tokens), d = static_cast<size_t>(cfg->d_model);
  if (e == cudaSuccess) e = cudaMalloc(&m->resid, T * d * 4);
  if (e == cudaSuccess) e = cudaMalloc(&m->xn, T * d * 2);
  if (e == cudaSuccess) e = cudaMalloc(&m->qkv, T * d * 3 * 2);
  if (e == cudaSuccess) e = cudaMalloc(&m->attn, T * d * 2);
  if (e == cudaSuccess) e = cudaMalloc(&m->ffn, T * static_cast<size_t>(cfg->d_ff) * 2);
  m->P = (cfg->d_model + 127) / 128;
  {
    const char* lf = getenv("SGPT_LN_FOLD");
    m->ln_fold = (lf != nullptr && lf[0] == '1');
    const char* rb = getenv("SGPT_RESID_BF16");
    m->resid_bf16 = !(rb != nullptr && rb[0] == '0') && !m->ln_fold;  // default ON; SGPT_RESID_BF16=0 keeps the stream in fp32
  }
  if (e == cudaSuccess) e = cudaMalloc(&m->stats, (2 * T * m->P + static_cast<size_t>(cfg->max_batch)) * 4);
  if (e == cudaSuccess) e = cudaMalloc(&m->sumsq, static_cast<size_t>(cfg->max_batch) * 4);
  // fold ln_1 into the QKV projection and ln_2 (GPT-J: ln_1 again) into the MLP's first layer
  for (int l = 0; l < cfg->n_layer && e == cudaSuccess && m->ln_fold; ++l) {
    const sgpt_layer_weights& lw = m->layers[l];
    const size_t ff = static_cast<size_t>(cfg->d_ff);
    void *wq = nullptr, *wf = nullptr;
    float *cq = nullptr, *bq = nullptr, *cf = nullptr, *bf = nullptr;
    e = cudaMalloc(&wq, 3 * d * d * 2);
    if (e == cudaSuccess) e = cudaMalloc(&cq, 3 * d * 4);
    if (e == cudaSuccess) e = cudaMalloc(&bq, 3 * d * 4);
    if (e == cudaSuccess) e = cudaMalloc(&wf, ff * d * 2);
    if (e == cudaSuccess) e = cudaMalloc(&cf, ff * 4);
    if (e == cudaSuccess) e = cudaMalloc(&bf, ff * 4);
    m->wq_f.push_back(wq); m->cq.push_back(cq); m->bq.push_back(bq);
    m->wfc_f.push_back(wf); m->cfc.push_back(cf); m->bfc.push_back(bf);
    if (e != cudaSuccess) break;
    const bool gptj = cfg->arch == SGPT_ARCH_GPTJ;
    int rc = sgpt_fold_layernorm(lw.w_qkv, lw.ln1_g, lw.ln1_b, lw.b_qkv, wq, cq, bq, 3 * cfg->d_model, cfg->d_model, nullptr);
    if (rc == SGPT_OK)
      rc = sgpt_fold_layernorm(lw.w_fc, gptj ? lw.ln1_g : lw.ln2_g, gptj ? lw.ln1_b : lw.ln2_b, lw.b_fc, wf, cf, bf, cfg->d_ff,
                               cfg->d_model, nullptr);
    if (rc != SGPT_OK) e = cudaErrorUnknown;
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

extern "C" void sgpt_model_destroy(sgpt_model_t m) {
  if (!m) return;
  cudaFree(m->resid);
  cudaFree(m->xn);
  cudaFree(m->qkv);
  cudaFree(m->attn);
  cudaFree(m->ffn);
  cudaFree(m->stats);
  cudaFree(m->sumsq);
  for (void* p : m->wq_f) cudaFree(p);
  for (void* p : m->wfc_f) cudaFree(p);
  for (float* p : m->cq) cudaFree(p);
  for (float* p : m->bq) cudaFree(p);
  for (float* p : m->cfc) cudaFree(p);
  for (float* p : m->bfc) cudaFree(p);
  cudaFree(m->rotary);
  cudaFree(m->alibi);
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

  const int rb = m->resid_bf16 ? 1 : 0;  // residual stream dtype: 0 fp32, 1 bf16 (same buffer, half of it used)
  const int epi_resid = rb ? SGPT_EPI_RESID_BF16 : SGPT_EPI_RESID_F32;
  SGPT_TRY(sgpt_embed_tokens_ex(ids, pos, m->w.wte, c.arch == SGPT_ARCH_GPT_NEO ? m->w.wpe : nullptr, m->resid, T, d,
                                c.vocab, c.max_pos, rb, stream));
  if (c.arch == SGPT_ARCH_BLOOM) {
    if (rb) SGPT_TRY(sgpt_layernorm_ex(m->resid, 1, m->w.emb_ln_g, m->w.emb_ln_b, m->resid, T, d, c.ln_eps, stream));
    else SGPT_TRY(sgpt_layernorm_f32_inplace(m->resid, m->w.emb_ln_g, m->w.emb_ln_b, T, d, c.ln_eps, stream));
  }
  const int n_run = layer_idx;  // hidden_states[i] is the input of block i; hidden_states[L] is ln_f(output of block L-1)
  if (m->ln_fold) {
  // bf16 copy + LayerNorm partial sums of the embedded residual stream; inside the blocks the residual epilogues keep
  // both up to date
  SGPT_TRY(sgpt_resid_stats(m->resid, m->xn, m->stats, T, d, stream));
  const int P = m->P;
  for (int l = 0; l < n_run && l < c.n_layer; ++l) {
    const sgpt_layer_weights& lw = m->layers[l];
    if (all_layers)  // hidden_states[l] = the residual stream entering block l (no ln_f)
      SGPT_TRY(sgpt_pool_accumulate(m->resid, pos, cu_seqlens, nullptr, nullptr, c.ln_eps, out, nullptr, B, T, d,
                                    base_mode, clamp_denominator, 0, /*accumulate=*/l > 0, layer_scale, stream));
    if (c.arch == SGPT_ARCH_GPT_NEO || c.arch == SGPT_ARCH_BLOOM) {
      // ln_1 -> q,k,v   (GPT-Neo: no q/k/v bias, un-scaled logits, local window on odd layers; BLOOM: bias, ALiBi, 1/sqrt(hd))
      SGPT_TRY(sgpt_linear_lnfold(m->xn, d, m->wq_f[l], d, m->bq[l], m->cq[l], m->stats, P, c.ln_eps, m->qkv, 3 * d, T, 3 * d,
                                  d, /*gelu=*/0, stream));
      if (c.arch == SGPT_ARCH_GPT_NEO) {
        const int window = (lw.local_attention && c.window > 0 && max_seqlen > c.window) ? c.window : 0;
        SGPT_TRY(sgpt_attention(m->qkv, m->attn, cu_seqlens, B, T, H, hd, /*scale=*/1.0f, window, max_seqlen, nullptr, 0,
                                stream));
      } else {
        SGPT_TRY(sgpt_attention(m->qkv, m->attn, cu_seqlens, B, T, H, hd, inv_sqrt_hd, 0, max_seqlen, m->alibi, 0, stream));
      }
      // out-proj + residual; the epilogue also emits xb / partial sums for ln_2
      SGPT_TRY(sgpt_linear_resid_ln(m->attn, d, lw.w_o, d, lw.b_o, m->resid, m->xn, m->stats, T, d, d, stream));
      // ln_2 -> c_fc -> gelu
      SGPT_TRY(sgpt_linear_lnfold(m->xn, d, m->wfc_f[l], d, m->bfc[l], m->cfc[l], m->stats, P, c.ln_eps, m->ffn, ff, T, ff, d,
                                  /*gelu=*/1, stream));
      // c_proj + residual; xb / partial sums for the next block's ln_1 (or ln_f)
      SGPT_TRY(sgpt_linear_resid_ln(m->ffn, ff, lw.w_proj, ff, lw.b_proj, m->resid, m->xn, m->stats, T, d, ff, stream));
    } else {  // GPT-J: attention and MLP both read ln_1(resid); res + attn + mlp
      SGPT_TRY(sgpt_linear_qkv_rotary_lnfold(m->xn, d, m->wq_f[l], m->bq[l], m->cq[l], m->stats, P, c.ln_eps, m->qkv, pos,
                                             m->rotary, T, d, hd, c.rotary_dim, c.max_pos, stream));
      SGPT_TRY(sgpt_attention(m->qkv, m->attn, cu_seqlens, B, T, H, hd, inv_sqrt_hd, 0, max_seqlen, nullptr, 0, stream));
      SGPT_TRY(sgpt_linear_lnfold(m->xn, d, m->wfc_f[l], d, m->bfc[l], m->cfc[l], m->stats, P, c.ln_eps, m->ffn, ff, T, ff, d,
                                  /*gelu=*/1, stream));
      // the first of the two residual updates is a plain reduce-add; the second one sees the complete sum and emits xb / stats
      SGPT_TRY(sgpt_linear(m->attn, d, lw.w_o, d, lw.b_o, m->resid, d, m->resid, T, d, d, SGPT_EPI_RESID_F32, stream));
      SGPT_TRY(sgpt_linear_resid_ln(m->ffn, ff, lw.w_proj, ff, lw.b_proj, m->resid, m->xn, m->stats, T, d, ff, stream));
    }
  }
  } else {
    for (int l = 0; l < n_run && l < c.n_layer; ++l) {
      const sgpt_layer_weights& lw = m->layers[l];
      if (all_layers)  // hidden_states[l] = the residual stream entering block l (no ln_f)
        SGPT_TRY(sgpt_pool_ex2(m->resid, rb, pos, cu_seqlens, nullptr, nullptr, c.ln_eps, nullptr, 0, out, nullptr, B, T, d,
                               base_mode, clamp_denominator, 0, /*accumulate=*/l > 0, layer_scale, stream));
      SGPT_TRY(sgpt_layernorm_ex(m->resid, rb, lw.ln1_g, lw.ln1_b, m->xn, T, d, c.ln_eps, stream));
      if (c.arch == SGPT_ARCH_GPT_NEO) {
        SGPT_TRY(sgpt_linear(m->xn, d, lw.w_qkv, d, lw.b_qkv, m->qkv, 3 * d, nullptr, T, 3 * d, d, SGPT_EPI_BF16, stream));
        const int window = (lw.local_attention && c.window > 0 && max_seqlen > c.window) ? c.window : 0;
        SGPT_TRY(sgpt_attention(m->qkv, m->attn, cu_seqlens, B, T, H, hd, /*scale=*/1.0f, window, max_seqlen, nullptr, 0,
                                stream));
        SGPT_TRY(sgpt_linear(m->attn, d, lw.w_o, d, lw.b_o, m->resid, d, m->resid, T, d, d, epi_resid, stream));
        SGPT_TRY(sgpt_layernorm_ex(m->resid, rb, lw.ln2_g, lw.ln2_b, m->xn, T, d, c.ln_eps, stream));
        SGPT_TRY(sgpt_linear(m->xn, d, lw.w_fc, d, lw.b_fc, m->ffn, ff, nullptr, T, ff, d, SGPT_EPI_GELU_BF16, stream));
        SGPT_TRY(sgpt_linear(m->ffn, ff, lw.w_proj, ff, lw.b_proj, m->resid, d, m->resid, T, d, ff, epi_resid,
                             stream));
      } else if (c.arch == SGPT_ARCH_GPTJ) {
        SGPT_TRY(sgpt_linear_qkv_rotary(m->xn, d, lw.w_qkv, m->qkv, pos, m->rotary, T, d, hd, c.rotary_dim, c.max_pos,
                                        stream));
        SGPT_TRY(sgpt_attention(m->qkv, m->attn, cu_seqlens, B, T, H, hd, inv_sqrt_hd, 0, max_seqlen, nullptr, 0, stream));
        // both branches read the same ln_1 output and are accumulated into the residual stream (attn + mlp + residual)
        SGPT_TRY(sgpt_linear(m->xn, d, lw.w_fc, d, lw.b_fc, m->ffn, ff, nullptr, T, ff, d, SGPT_EPI_GELU_BF16, stream));
        SGPT_TRY(sgpt_linear(m->attn, d, lw.w_o, d, lw.b_o, m->resid, d, m->resid, T, d, d, epi_resid, stream));
        SGPT_TRY(sgpt_linear(m->ffn, ff, lw.w_proj, ff, lw.b_proj, m->resid, d, m->resid, T, d, ff, epi_resid,
                             stream));
      } else {  // BLOOM
        SGPT_TRY(sgpt_linear(m->xn, d, lw.w_qkv, d, lw.b_qkv, m->qkv, 3 * d, nullptr, T, 3 * d, d, SGPT_EPI_BF16, stream));
        SGPT_TRY(sgpt_attention(m->qkv, m->attn, cu_seqlens, B, T, H, hd, inv_sqrt_hd, 0, max_seqlen, m->alibi, 0, stream));
        SGPT_TRY(sgpt_linear(m->attn, d, lw.w_o, d, lw.b_o, m->resid, d, m->resid, T, d, d, epi_resid, stream));
        SGPT_TRY(sgpt_layernorm_ex(m->resid, rb, lw.ln2_g, lw.ln2_b, m->xn, T, d, c.ln_eps, stream));
        SGPT_TRY(sgpt_linear(m->xn, d, lw.w_fc, d, lw.b_fc, m->ffn, ff, nullptr, T, ff, d, SGPT_EPI_GELU_BF16, stream));
        SGPT_TRY(sgpt_linear(m->ffn, ff, lw.w_proj, ff, lw.b_proj, m->resid, d, m->resid, T, d, ff, epi_resid,
                             stream));
      }
    }
  }
  if (pool_mode == kNoPooling) return SGPT_OK;
  const bool final_ln = (layer_idx == c.n_layer);
  if (final_ln && m->ln_fold) {
    // ln_f folded into the pooling kernel; its row statistics come from the partial sums the last c_proj (or the
    // embedding, for a 0-layer run) left behind: ONE pass over the residual stream
    SGPT_TRY(sgpt_pool_partials(m->resid, pos, cu_seqlens, m->w.lnf_g, m->w.lnf_b, c.ln_eps, pool_w, pool_w ? m->n_pool_w : 0,
                                out, m->stats, m->P, m->sumsq, B, T, d, base_mode, clamp_denominator, normalize,
                                /*accumulate=*/all_layers && c.n_layer > 0, layer_scale, stream));
  } else {
    // (the partial sums are dead after the last block: the scratch only hosts the normalisation's per-row sums here)
    SGPT_TRY(sgpt_pool_ex2(m->resid, rb, pos, cu_seqlens, final_ln ? m->w.lnf_g : nullptr, final_ln ? m->w.lnf_b : nullptr, c.ln_eps,
                          pool_w, pool_w ? m->n_pool_w : 0, out, m->stats, B, T, d, base_mode, clamp_denominator, normalize,
                          /*accumulate=*/all_layers && c.n_layer > 0, layer_scale, stream));
  }
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
  uint8_t* w = static_cast<uint8_t*>(ws);
  void* xsel = w;
  float* logits = reinterpret_cast<float*>(w + lm_align(static_cast<int64_t>(rows_per_chunk) * d * 2));
  const int64_t lds = lm_lds(vocab);
  for (int m0 = 0; m0 < M; m0 += rows_per_chunk) {
    const int mc = (M - m0 < rows_per_chunk) ? M - m0 : rows_per_chunk;
    // hidden_states[-1] of the selected positions: ln_f of the residual stream the last sgpt_forward left behind
    SGPT_TRY(sgpt_layernorm_gather_ex(m->resid, m->resid_bf16 ? 1 : 0, rows + m0, m->w.lnf_g, m->w.lnf_b, xsel, mc, d,
                                      m->cfg.ln_eps, stream));
    SGPT_TRY(sgpt_scores(xsel, lm_head_w, nullptr, nullptr, logits, lds, mc, vocab, d, stream));
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
  if (m->resid_bf16) return sgpt_bf16_to_f32(m->resid, dst, n, stream);
  SGPT_CHECK_CUDA(cudaMemcpyAsync(dst, m->resid, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToDevice,
                                  static_cast<cudaStream_t>(stream)));
  return SGPT_OK;
}
