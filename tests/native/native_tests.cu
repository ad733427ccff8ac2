// Native GPU self-test for libsgpt_b200.so: every kernel against a straightforward host computation on the same
// bf16-rounded inputs.  Runs on the GPU box (gpurun); prints one PASS/FAIL line per case and exits non-zero on any
// failure.  This is kernel bring-up infrastructure; the parity tests proper live in tests/test_*_gpu.py.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <random>
#include <vector>

#include "../../include/sgpt_b200.h"

#define CK(x)                                                                                  \
  do {                                                                                         \
    cudaError_t e_ = (x);                                                                      \
    if (e_ != cudaSuccess) {                                                                   \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__);          \
      exit(2);                                                                                 \
    }                                                                                          \
  } while (0)
#define SG(x)                                                                                  \
  do {                                                                                         \
    int r_ = (x);                                                                              \
    if (r_ != SGPT_OK) {                                                                       \
      printf("sgpt error %d (%s) at %s:%d\n", r_, sgpt_last_error(), __FILE__, __LINE__);      \
      exit(3);                                                                                 \
    }                                                                                          \
  } while (0)

static int g_fail = 0;
static std::mt19937 rng(1234);

static float bf16r(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

template <class T>
static T* dalloc(size_t n) {
  T* p;
  CK(cudaMalloc(&p, n * sizeof(T) + 256));
  return p;
}
template <class T>
static T* to_dev(const std::vector<T>& h) {
  T* p = dalloc<T>(h.size());
  CK(cudaMemcpy(p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
  return p;
}
template <class T>
static std::vector<T> to_host(const T* d, size_t n) {
  std::vector<T> h(n);
  CK(cudaMemcpy(h.data(), d, n * sizeof(T), cudaMemcpyDeviceToHost));
  return h;
}
static std::vector<float> randn(size_t n, float sd) {
  std::normal_distribution<float> nd(0.f, sd);
  std::vector<float> v(n);
  for (auto& x : v) x = nd(rng);
  return v;
}
static std::vector<__nv_bfloat16> to_bf16(std::vector<float>& v) {  // also rounds v in place
  std::vector<__nv_bfloat16> o(v.size());
  for (size_t i = 0; i < v.size(); ++i) {
    o[i] = __float2bfloat16_rn(v[i]);
    v[i] = __bfloat162float(o[i]);
  }
  return o;
}
static void report(const char* name, double err, double tol, double ms = -1) {
  const bool ok = err <= tol && err == err;
  if (!ok) g_fail++;
  if (ms >= 0) printf("%s %-58s err=%.3e tol=%.1e  %.3f ms\n", ok ? "PASS" : "FAIL", name, err, tol, ms);
  else printf("%s %-58s err=%.3e tol=%.1e\n", ok ? "PASS" : "FAIL", name, err, tol);
  fflush(stdout);
}
static float time_ms(cudaEvent_t a, cudaEvent_t b) {
  float ms;
  CK(cudaEventElapsedTime(&ms, a, b));
  return ms;
}
static float gelu_ref(float x) { return 0.5f * x * (1.f + tanhf(0.7978845608028654f * (x + 0.044715f * x * x * x))); }

// ---------------------------------------------------------------------------------------------------------------
static void test_linear(int M, int N, int K, int epi, int check_rows) {
  auto x = randn((size_t)M * K, 1.0f), w = randn((size_t)N * K, 0.05f), bias = randn(N, 0.5f);
  auto resid = randn((size_t)M * N, 1.0f);
  auto xb = to_bf16(x), wb = to_bf16(w);
  auto *dx = to_dev(xb), *dw = to_dev(wb);
  float* dbias = to_dev(bias);
  float* dres = to_dev(resid);
  void* dout = (epi == SGPT_EPI_RESID_F32) ? (void*)dres : (void*)dalloc<__nv_bfloat16>((size_t)M * N);
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  // timing: 1 warm-up + 5 timed launches into a scratch output (the checked launch below runs once, on fresh data)
  float ms = 0.f;
  {
    void* scratch = (epi == SGPT_EPI_RESID_F32) ? (void*)dalloc<float>((size_t)M * N) : dout;
    const float* rsrc = (epi == SGPT_EPI_RESID_F32) ? (const float*)scratch : dres;
    if (epi == SGPT_EPI_RESID_F32) CK(cudaMemset(scratch, 0, (size_t)M * N * 4));
    SG(sgpt_linear(dx, K, dw, K, dbias, scratch, N, rsrc, M, N, K, epi, 0));
    CK(cudaEventRecord(e0));
    for (int it = 0; it < 5; ++it) SG(sgpt_linear(dx, K, dw, K, dbias, scratch, N, rsrc, M, N, K, epi, 0));
    CK(cudaEventRecord(e1));
    CK(cudaDeviceSynchronize());
    ms = time_ms(e0, e1) / 5.f;
    if (epi == SGPT_EPI_RESID_F32) cudaFree(scratch);
  }
  SG(sgpt_linear(dx, K, dw, K, dbias, dout, N, dres, M, N, K, epi, 0));
  CK(cudaDeviceSynchronize());
  std::vector<float> got((size_t)M * N);
  if (epi == SGPT_EPI_RESID_F32) got = to_host((float*)dout, (size_t)M * N);
  else {
    auto gb = to_host((__nv_bfloat16*)dout, (size_t)M * N);
    for (size_t i = 0; i < gb.size(); ++i) got[i] = __bfloat162float(gb[i]);
  }
  double maxerr = 0;
  std::vector<int> rows;
  if (check_rows >= M) for (int i = 0; i < M; ++i) rows.push_back(i);
  else {
    rows.push_back(0); rows.push_back(M - 1); rows.push_back(127 % M); rows.push_back(128 % M);
    for (int i = 0; i < check_rows; ++i) rows.push_back(rng() % M);
  }
  for (int m : rows) {
    for (int n = 0; n < N; ++n) {
      double acc = 0;
      const float* xr = &x[(size_t)m * K];
      const float* wr = &w[(size_t)n * K];
      for (int k = 0; k < K; ++k) acc += (double)xr[k] * wr[k];
      float ref = (float)acc + bias[n];
      float tol_scale = 1.f;
      if (epi == SGPT_EPI_GELU_BF16) ref = gelu_ref(ref);
      if (epi == SGPT_EPI_RESID_F32) ref += resid[(size_t)m * N + n];
      else tol_scale = fmaxf(1.f, fabsf(ref));  // bf16 output rounding is relative
      const double err = fabs((double)got[(size_t)m * N + n] - ref) / tol_scale;
      maxerr = std::max(maxerr, err);
    }
  }
  char name[128];
  const char* en[] = {"bf16", "gelu_bf16", "resid_f32"};
  snprintf(name, sizeof name, "linear M=%d N=%d K=%d epi=%s (%.1f TFLOP/s)", M, N, K, epi < 3 ? en[epi] : "stub",
           2.0 * M * N * K / (ms * 1e9));
  if (epi >= 100) maxerr = 0;  // profiling stubs write nothing meaningful: timing only
  report(name, maxerr, epi == SGPT_EPI_RESID_F32 ? 2e-3 : 1.2e-2, ms);
  cudaFree(dx); cudaFree(dw); cudaFree(dbias); cudaFree(dres);
  if (epi != SGPT_EPI_RESID_F32) cudaFree(dout);
}

// ---------------------------------------------------------------------------------------------------------------
static void attention_ref(const std::vector<float>& qkv, std::vector<float>& out, const std::vector<int>& cu, int H,
                          int hd, float scale, int window, const std::vector<float>* alibi = nullptr) {
  const int B = (int)cu.size() - 1, d = H * hd;
  const size_t ld = 3 * (size_t)d;
  std::vector<double> p;
  for (int b = 0; b < B; ++b) {
    for (int t = cu[b]; t < cu[b + 1]; ++t) {
      for (int h = 0; h < H; ++h) {
        int lo = cu[b];
        if (window > 0) lo = std::max(lo, t - window + 1);
        p.assign(t - lo + 1, 0.0);
        double mx = -1e300;
        for (int kt = lo; kt <= t; ++kt) {
          double s = 0;
          for (int e = 0; e < hd; ++e) s += (double)qkv[t * ld + h * hd + e] * qkv[kt * ld + d + h * hd + e];
          s *= scale;
          if (alibi) s += (*alibi)[h] * (kt - cu[b]);
          p[kt - lo] = s;
          mx = std::max(mx, s);
        }
        double l = 0;
        for (auto& v : p) { v = exp(v - mx); l += v; }
        for (int e = 0; e < hd; ++e) {
          double o = 0;
          for (int kt = lo; kt <= t; ++kt) o += p[kt - lo] * qkv[kt * ld + 2 * d + h * hd + e];
          out[(size_t)t * d + h * hd + e] = (float)(o / l);
        }
      }
    }
  }
}

static void test_attention(const std::vector<int>& lens, int H, int hd, float scale, int window, float qk_sd,
                           bool use_alibi = false) {
  const int B = (int)lens.size();
  std::vector<float> slopes(H);
  for (int h = 0; h < H; ++h) slopes[h] = powf(2.f, -8.f * (h + 1) / H);
  float* dalibi = use_alibi ? to_dev(slopes) : nullptr;
  std::vector<int> cu(B + 1, 0);
  int maxlen = 0;
  for (int b = 0; b < B; ++b) { cu[b + 1] = cu[b] + lens[b]; maxlen = std::max(maxlen, lens[b]); }
  const int T = cu[B], d = H * hd;
  auto qkv = randn((size_t)T * 3 * d, qk_sd);
  auto qkvb = to_bf16(qkv);
  auto* dqkv = to_dev(qkvb);
  int* dcu = to_dev(cu);
  auto* dout = dalloc<__nv_bfloat16>((size_t)T * d);
  auto* dout2 = dalloc<__nv_bfloat16>((size_t)T * d);
  std::vector<float> ref((size_t)T * d);
  attention_ref(qkv, ref, cu, H, hd, scale, window, use_alibi ? &slopes : nullptr);
  for (int impl = 1; impl >= 0; --impl) {
    __nv_bfloat16* o = impl ? dout2 : dout;
    CK(cudaMemset(o, 0xff, (size_t)T * d * 2));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0));
    SG(sgpt_attention(dqkv, o, dcu, B, T, H, hd, scale, window, maxlen, dalibi, impl, 0));
    CK(cudaEventRecord(e1));
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
      printf("FAIL attention impl=%d launch error: %s\n", impl, cudaGetErrorString(e));
      g_fail++;
      exit(4);
    }
    auto got = to_host(o, (size_t)T * d);
    double maxerr = 0;
    for (size_t i = 0; i < got.size(); ++i)
      maxerr = std::max(maxerr, (double)fabsf(__bfloat162float(got[i]) - ref[i]) / std::max(1.0, (double)fabsf(ref[i])));
    char name[160];
    snprintf(name, sizeof name, "attention %s B=%d maxlen=%d T=%d H=%d hd=%d win=%d scale=%.3f", impl ? "simt" : "tc",
             B, maxlen, T, H, hd, window, scale);
    report(name, maxerr, 2e-2, time_ms(e0, e1));
  }
  cudaFree(dqkv); cudaFree(dcu); cudaFree(dout); cudaFree(dout2);
}

// ---------------------------------------------------------------------------------------------------------------
static void test_rows(int T, int d) {
  // embed + layernorm + pool(ln_f fused) on a ragged batch
  const int vocab = 1000, max_pos = 512;
  std::vector<int> lens = {1, 37, 64, 5, 128, 2};
  while ((int)lens.size() < 8) lens.push_back(16);
  std::vector<int> cu(1, 0), ids, pos;
  for (int L : lens) {
    for (int i = 0; i < L; ++i) { ids.push_back(rng() % vocab); pos.push_back(i); }
    cu.push_back(cu.back() + L);
  }
  T = cu.back();
  const int B = (int)lens.size();
  auto wte = randn((size_t)vocab * d, 0.5f), wpe = randn((size_t)max_pos * d, 0.5f);
  auto g = randn(d, 0.3f), bt = randn(d, 0.3f);
  for (auto& v : g) v += 1.f;
  auto wteb = to_bf16(wte), wpeb = to_bf16(wpe);
  auto *dwte = to_dev(wteb), *dwpe = to_dev(wpeb);
  int *dids = to_dev(ids), *dpos = to_dev(pos), *dcu = to_dev(cu);
  float *dg = to_dev(g), *db = to_dev(bt);
  float* dres = dalloc<float>((size_t)T * d);
  auto* dy = dalloc<__nv_bfloat16>((size_t)T * d);
  float* dpool = dalloc<float>((size_t)B * d);
  float* dstats = dalloc<float>(2 * (size_t)T + B);
  SG(sgpt_embed_tokens(dids, dpos, dwte, dwpe, dres, T, d, vocab, max_pos, 0));
  SG(sgpt_layernorm(dres, dg, db, dy, T, d, 1e-5f, 0));
  SG(sgpt_pool(dres, dpos, dcu, dg, db, 1e-5f, dpool, dstats, B, T, d, SGPT_POOL_WEIGHTEDMEAN, 0, 0, 0));
  CK(cudaDeviceSynchronize());
  auto res = to_host(dres, (size_t)T * d);
  auto y = to_host(dy, (size_t)T * d);
  auto pool = to_host(dpool, (size_t)B * d);
  double e_emb = 0, e_ln = 0, e_pool = 0;
  std::vector<double> ln((size_t)T * d);
  for (int t = 0; t < T; ++t) {
    double mean = 0, var = 0;
    for (int c = 0; c < d; ++c) {
      const float r = wte[(size_t)ids[t] * d + c] + wpe[(size_t)pos[t] * d + c];
      e_emb = std::max(e_emb, (double)fabsf(r - res[(size_t)t * d + c]));
      mean += r;
    }
    mean /= d;
    for (int c = 0; c < d; ++c) { double dv = res[(size_t)t * d + c] - mean; var += dv * dv; }
    var /= d;
    const double rstd = 1.0 / sqrt(var + 1e-5);
    for (int c = 0; c < d; ++c) {
      const double v = (res[(size_t)t * d + c] - mean) * rstd * g[c] + bt[c];
      ln[(size_t)t * d + c] = v;
      e_ln = std::max(e_ln, fabs(v - __bfloat162float(y[(size_t)t * d + c])) / std::max(1.0, fabs(v)));
    }
  }
  for (int b = 0; b < B; ++b)
    for (int c = 0; c < d; ++c) {
      double num = 0, den = 0;
      for (int t = cu[b]; t < cu[b + 1]; ++t) { num += ln[(size_t)t * d + c] * (pos[t] + 1); den += pos[t] + 1; }
      e_pool = std::max(e_pool, fabs(num / den - pool[(size_t)b * d + c]));
    }
  char name[96];
  snprintf(name, sizeof name, "embed d=%d", d); report(name, e_emb, 1e-6);
  snprintf(name, sizeof name, "layernorm d=%d", d); report(name, e_ln, 8e-3);
  snprintf(name, sizeof name, "pool weightedmean + ln_f d=%d", d); report(name, e_pool, 2e-5);
  // mean / lasttoken without LN, with normalize
  SG(sgpt_pool(dres, dpos, dcu, nullptr, nullptr, 0.f, dpool, dstats, B, T, d, SGPT_POOL_LASTTOKEN, 1, 1, 0));
  CK(cudaDeviceSynchronize());
  pool = to_host(dpool, (size_t)B * d);
  double e_last = 0;
  for (int b = 0; b < B; ++b) {
    double nn = 0;
    for (int c = 0; c < d; ++c) nn += (double)res[(size_t)(cu[b + 1] - 1) * d + c] * res[(size_t)(cu[b + 1] - 1) * d + c];
    nn = sqrt(nn);
    for (int c = 0; c < d; ++c)
      e_last = std::max(e_last, fabs(res[(size_t)(cu[b + 1] - 1) * d + c] / nn - pool[(size_t)b * d + c]));
  }
  snprintf(name, sizeof name, "pool lasttoken + normalize d=%d", d); report(name, e_last, 2e-6);
  cudaFree(dwte); cudaFree(dwpe); cudaFree(dids); cudaFree(dpos); cudaFree(dcu); cudaFree(dg); cudaFree(db);
  cudaFree(dres); cudaFree(dy); cudaFree(dpool); cudaFree(dstats);
}

// ---------------------------------------------------------------------------------------------------------------
static void test_scores_topk(int nq, int n, int D, int k) {
  auto q = randn((size_t)nq * D, 1.f), c = randn((size_t)n * D, 1.f);
  // plant near-duplicates so the top of the ranking is meaningful
  for (int i = 0; i < n; i += 97) {
    const int qq = (i / 97) % nq;
    for (int e = 0; e < D; ++e) c[(size_t)i * D + e] = q[(size_t)qq * D + e] + 0.5f * c[(size_t)i * D + e];
  }
  auto qb = to_bf16(q), cb = to_bf16(c);
  auto *dq = to_dev(qb), *dc = to_dev(cb);
  float *dqn = dalloc<float>(nq), *dcn = dalloc<float>(n);
  SG(sgpt_row_inv_norms(dq, dqn, nq, D, 0));
  SG(sgpt_row_inv_norms(dc, dcn, n, D, 0));
  const int64_t lds = (n + 3) & ~3;
  float* ds = dalloc<float>((size_t)nq * lds);
  float* dts = dalloc<float>((size_t)nq * k);
  int64_t* dti = dalloc<int64_t>((size_t)nq * k);
  cudaEvent_t e0, e1, e2;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1)); CK(cudaEventCreate(&e2));
  CK(cudaEventRecord(e0));
  SG(sgpt_scores(dq, dc, dqn, dcn, ds, lds, nq, n, D, 0));
  CK(cudaEventRecord(e1));
  SG(sgpt_topk(ds, lds, nq, n, k, 1000, dts, dti, nullptr, 0));
  CK(cudaEventRecord(e2));
  CK(cudaDeviceSynchronize());
  auto s = to_host(ds, (size_t)nq * lds);
  auto ts = to_host(dts, (size_t)nq * k);
  auto ti = to_host(dti, (size_t)nq * k);
  // host scores on a subset of queries
  double e_s = 0;
  int bad_topk = 0;
  std::vector<double> cn(n);
  for (int j = 0; j < n; ++j) {
    double a = 0;
    for (int e = 0; e < D; ++e) a += (double)c[(size_t)j * D + e] * c[(size_t)j * D + e];
    cn[j] = 1.0 / std::max(sqrt(a), 1e-12);
  }
  for (int qi = 0; qi < nq; qi += std::max(1, nq / 4)) {
    double a = 0;
    for (int e = 0; e < D; ++e) a += (double)q[(size_t)qi * D + e] * q[(size_t)qi * D + e];
    const double qn = 1.0 / std::max(sqrt(a), 1e-12);
    for (int j = 0; j < n; ++j) {
      double acc = 0;
      for (int e = 0; e < D; ++e) acc += (double)q[(size_t)qi * D + e] * c[(size_t)j * D + e];
      e_s = std::max(e_s, fabs(acc * qn * cn[j] - s[(size_t)qi * lds + j]));
    }
  }
  // top-k vs std::partial_sort on the DEVICE scores (bit-exact selection check)
  for (int qi = 0; qi < nq; ++qi) {
    std::vector<std::pair<float, int64_t>> v(n);
    for (int j = 0; j < n; ++j) v[j] = {-s[(size_t)qi * lds + j], (int64_t)j + 1000};
    const int kk = std::min(k, n);
    std::partial_sort(v.begin(), v.begin() + kk, v.end());
    for (int i = 0; i < k; ++i) {
      if (i < kk) {
        if (ts[(size_t)qi * k + i] != -v[i].first) bad_topk++;
        // ids may differ only among exactly tied scores
        if (ti[(size_t)qi * k + i] != v[i].second && !(i + 1 < kk && v[i].first == v[i + 1].first) &&
            !(i > 0 && v[i].first == v[i - 1].first) && !(kk < n && v[kk - 1].first == v[kk].first))
          bad_topk++;
      } else if (ti[(size_t)qi * k + i] != -1) bad_topk++;
    }
  }
  char name[128];
  snprintf(name, sizeof name, "scores nq=%d n=%d D=%d (%.0f GB/s corpus)", nq, n, D,
           (double)n * D * 2 / (time_ms(e0, e1) * 1e6));
  report(name, e_s, 2e-5, time_ms(e0, e1));
  snprintf(name, sizeof name, "topk nq=%d n=%d k=%d mismatches", nq, n, k);
  report(name, bad_topk, 0, time_ms(e1, e2));
  // merge: split the result list in 3 shuffled parts + empties and merge back
  {
    const int G = 3;
    std::vector<float> ms((size_t)G * nq * k, 0.f);
    std::vector<int64_t> mi((size_t)G * nq * k, -1);
    for (int qi = 0; qi < nq; ++qi)
      for (int i = 0; i < k; ++i) {
        const int g = (i * 7 + qi) % G;
        ms[((size_t)g * nq + qi) * k + i] = ts[(size_t)qi * k + i];
        mi[((size_t)g * nq + qi) * k + i] = ti[(size_t)qi * k + i];
      }
    float* dms = to_dev(ms);
    int64_t* dmi = to_dev(mi);
    float* dos = dalloc<float>((size_t)nq * k);
    int64_t* doi = dalloc<int64_t>((size_t)nq * k);
    SG(sgpt_topk_merge(dms, dmi, G, nq, k, dos, doi, nullptr, nullptr, 0));
    CK(cudaDeviceSynchronize());
    auto os = to_host(dos, (size_t)nq * k);
    auto oi = to_host(doi, (size_t)nq * k);
    int bad = 0;
    for (size_t i = 0; i < os.size(); ++i)
      if (oi[i] != ti[i] || (ti[i] >= 0 && os[i] != ts[i])) bad++;
    snprintf(name, sizeof name, "topk_merge G=%d nq=%d k=%d mismatches", G, nq, k);
    report(name, bad, 0);
    cudaFree(dms); cudaFree(dmi); cudaFree(dos); cudaFree(doi);
  }
  cudaFree(dq); cudaFree(dc); cudaFree(dqn); cudaFree(dcn); cudaFree(ds); cudaFree(dts); cudaFree(dti);
}

// fused search (two-pass threshold filter for large shards) against host scores on the same bf16 inputs
static void test_search(int nq, int n, int D, int k) {
  auto q = randn((size_t)nq * D, 1.f), c = randn((size_t)n * D, 1.f);
  for (int i = 0; i < n; i += 97) {
    const int qq = (i / 97) % nq;
    for (int e = 0; e < D; ++e) c[(size_t)i * D + e] = q[(size_t)qq * D + e] + 0.5f * c[(size_t)i * D + e];
  }
  auto qb = to_bf16(q), cb = to_bf16(c);
  auto *dq = to_dev(qb), *dc = to_dev(cb);
  float *dqn = dalloc<float>(nq), *dcn = dalloc<float>(n);
  SG(sgpt_row_inv_norms(dq, dqn, nq, D, 0));
  SG(sgpt_row_inv_norms(dc, dcn, n, D, 0));
  const int64_t wsb = sgpt_search_workspace_bytes(nq, n, k);
  uint8_t* ws = dalloc<uint8_t>(wsb);
  float* dts = dalloc<float>((size_t)nq * k);
  int64_t* dti = dalloc<int64_t>((size_t)nq * k);
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  SG(sgpt_search(dq, dc, dqn, dcn, nq, n, D, k, 5000, dts, dti, ws, wsb, 0));
  CK(cudaEventRecord(e0));
  for (int it = 0; it < 3; ++it) SG(sgpt_search(dq, dc, dqn, dcn, nq, n, D, k, 5000, dts, dti, ws, wsb, 0));
  CK(cudaEventRecord(e1));
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("FAIL search launch error: %s\n", cudaGetErrorString(e)); exit(4); }
  auto ts = to_host(dts, (size_t)nq * k);
  auto ti = to_host(dti, (size_t)nq * k);
  auto qn = to_host(dqn, nq);
  auto cn = to_host(dcn, n);
  int bad = 0;
  double maxerr = 0;
  std::vector<float> sc(n);
  for (int qi = 0; qi < nq; ++qi) {
    for (int j = 0; j < n; ++j) {
      double acc = 0;
      for (int d = 0; d < D; ++d) acc += (double)q[(size_t)qi * D + d] * c[(size_t)j * D + d];
      sc[j] = (float)(acc * qn[qi] * cn[j]);
    }
    std::vector<float> sorted(sc);
    const int kk = std::min(k, n);
    std::nth_element(sorted.begin(), sorted.begin() + (kk - 1), sorted.end(), std::greater<float>());
    const float cut = sorted[kk - 1];
    std::vector<char> seen(n, 0);
    for (int i = 0; i < kk; ++i) {
      const int64_t id = ti[(size_t)qi * k + i] - 5000;
      if (id < 0 || id >= n || seen[id]) { bad++; continue; }
      seen[id] = 1;
      if (sc[id] < cut - 2e-6f) bad++;                               // not a member of the true top-k
      maxerr = std::max(maxerr, (double)fabsf(sc[id] - ts[(size_t)qi * k + i]));
      if (i > 0 && ts[(size_t)qi * k + i] > ts[(size_t)qi * k + i - 1]) bad++;  // descending
    }
    int must = 0, have = 0;  // every doc clearly above the cut must be present
    for (int j = 0; j < n; ++j) if (sc[j] > cut + 2e-6f) { must++; have += seen[j]; }
    if (must != have) bad++;
  }
  char name[160];
  const double ms = time_ms(e0, e1) / 3;
  snprintf(name, sizeof name, "search nq=%d n=%d D=%d k=%d (%.0f GB/s corpus, %.0f q/s) wrong", nq, n, D, k,
           (double)n * D * 2 / (ms * 1e6), nq / (ms * 1e-3));
  report(name, bad, 0, ms);
  snprintf(name, sizeof name, "search nq=%d n=%d score error", nq, n);
  report(name, maxerr, 2e-5);
  cudaFree(dq); cudaFree(dc); cudaFree(dqn); cudaFree(dcn); cudaFree(ws); cudaFree(dts); cudaFree(dti);
}

int main(int argc, char** argv) {
  const char* only = argc > 1 ? argv[1] : "all";
  auto want = [&](const char* s) { return !strcmp(only, "all") || !strcmp(only, s); };
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  printf("device: %s, %d SMs, cc %d.%d, abi %d\n", prop.name, prop.multiProcessorCount, prop.major, prop.minor,
         sgpt_abi_version());
  if (want("rows")) { test_rows(0, 768); test_rows(0, 2048); test_rows(0, 4096); }
  if (want("linear")) {
    test_linear(128, 128, 64, SGPT_EPI_BF16, 1 << 30);
    test_linear(128, 256, 128, SGPT_EPI_BF16, 1 << 30);
    test_linear(300, 768, 768, SGPT_EPI_BF16, 1 << 30);
    test_linear(257, 2304, 768, SGPT_EPI_BF16, 1 << 30);
    test_linear(200, 3072, 768, SGPT_EPI_GELU_BF16, 1 << 30);
    test_linear(333, 768, 3072, SGPT_EPI_RESID_F32, 1 << 30);
    test_linear(77, 200, 72, SGPT_EPI_BF16, 1 << 30);   // ragged N and K tails
    test_linear(77, 200, 72, SGPT_EPI_RESID_F32, 1 << 30);
    test_linear(32768, 2304, 768, SGPT_EPI_BF16, 24);
    test_linear(32768, 768, 768, SGPT_EPI_RESID_F32, 24);
    test_linear(32768, 3072, 768, SGPT_EPI_GELU_BF16, 24);
    test_linear(32768, 768, 3072, SGPT_EPI_RESID_F32, 24);
    test_linear(16384, 8192, 2048, SGPT_EPI_GELU_BF16, 16);
  }
  if (!strcmp(only, "linperf")) {  // the four per-layer GEMMs of SGPT-125M at batch 256 x 128 (ncu target)
    test_linear(32768, 2304, 768, SGPT_EPI_BF16, 4);
    test_linear(32768, 768, 768, SGPT_EPI_RESID_F32, 4);
    test_linear(32768, 3072, 768, SGPT_EPI_GELU_BF16, 4);
    test_linear(32768, 768, 3072, SGPT_EPI_RESID_F32, 4);
  }
  if (!strcmp(only, "nullepi")) {  // timing only: mainloop without / with accumulator loads in the epilogue
    for (int epi = 100; epi <= 105; ++epi)
      for (int K : {768, 3072}) {
        const int M = 32768, N = 2304;
        auto x = randn((size_t)M * K, 1.0f), w = randn((size_t)N * K, 0.05f);
        auto xb = to_bf16(x), wb = to_bf16(w);
        auto *dx = to_dev(xb), *dw = to_dev(wb);
        auto* dout = dalloc<__nv_bfloat16>((size_t)M * N);
        cudaEvent_t e0, e1;
        CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
        SG(sgpt_linear(dx, K, dw, K, nullptr, dout, N, nullptr, M, N, K, epi, 0));
        CK(cudaEventRecord(e0));
        for (int it = 0; it < 5; ++it) SG(sgpt_linear(dx, K, dw, K, nullptr, dout, N, nullptr, M, N, K, epi, 0));
        CK(cudaEventRecord(e1));
        CK(cudaDeviceSynchronize());
        const double ms = time_ms(e0, e1) / 5;
        printf("INFO epi=%d M=%d N=%d K=%d: %.3f ms  %.1f TFLOP/s\n", epi, M, N, K, ms, 2.0 * M * N * K / (ms * 1e9));
        cudaFree(dx); cudaFree(dw); cudaFree(dout);
      }
  }
  if (!strcmp(only, "clockprobe")) {  // what SM clock do the GEMM bursts actually run at?
    const int M = 32768, N = 2304;
    for (int launches : {5, 60})
      for (int K : {768, 3072})
        for (int epi : {100, 102, (int)SGPT_EPI_BF16}) {
          auto x = randn((size_t)M * K, 1.0f), w = randn((size_t)N * K, 0.05f);
          auto xb = to_bf16(x), wb = to_bf16(w);
          auto *dx = to_dev(xb), *dw = to_dev(wb);
          auto* dout = dalloc<__nv_bfloat16>((size_t)M * N);
          SG(sgpt_linear(dx, K, dw, K, nullptr, dout, N, nullptr, M, N, K, epi, 0));
          double cyc, ns;
          SG(sgpt_profile_gemm_clock(&cyc, &ns));
          cudaEvent_t e0, e1;
          CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
          CK(cudaEventRecord(e0));
          for (int it = 0; it < launches; ++it) SG(sgpt_linear(dx, K, dw, K, nullptr, dout, N, nullptr, M, N, K, epi, 0));
          CK(cudaEventRecord(e1));
          CK(cudaDeviceSynchronize());
          SG(sgpt_profile_gemm_clock(&cyc, &ns));
          const double ms = time_ms(e0, e1) / launches;
          printf("INFO clockprobe launches=%d K=%d epi=%d: %.3f ms/launch %.1f TFLOP/s | in-kernel %.3f ms, SM clock %.0f MHz\n",
                 launches, K, epi, ms, 2.0 * M * N * K / (ms * 1e9), ns / launches * 1e-6, 1e3 * cyc / ns);
          cudaFree(dx); cudaFree(dw); cudaFree(dout);
        }
  }
  if (!strcmp(only, "resid")) {  // is the fp32 reduce-add epilogue what bounds the d x d out-projection?
    test_linear(32768, 768, 768, SGPT_EPI_BF16, 2);
    test_linear(32768, 768, 768, SGPT_EPI_RESID_F32, 2);
    test_linear(32768, 768, 768, 100, 0);
    test_linear(32768, 768, 3072, SGPT_EPI_BF16, 2);
    test_linear(32768, 768, 3072, SGPT_EPI_RESID_F32, 2);
    test_linear(32768, 768, 3072, 100, 0);
  }
  if (!strcmp(only, "sweep")) {  // which dimension limits the GEMM rate?
    const int shapes[][3] = {{32768, 2304, 768}, {32768, 2304, 2048}, {16384, 8192, 768},  {16384, 2304, 768},
                             {32768, 8192, 768}, {8192, 8192, 2048},  {32768, 2304, 3072}, {65536, 2304, 768},
                             {32768, 2048, 768}, {32768, 2048, 1024}};
    for (auto& sh : shapes) test_linear(sh[0], sh[1], sh[2], SGPT_EPI_BF16, 2);
  }
  if (!strcmp(only, "attnperf")) {  // the bench shape: 256 sequences x 128 tokens, 12 heads x 64 (timing only)
    const int B = 256, S = 128, H = 12, hd = 64, T = B * S, d = H * hd;
    auto qkv = randn((size_t)T * 3 * d, 0.3f);
    auto qb = to_bf16(qkv);
    auto* dq = to_dev(qb);
    auto* dout = dalloc<__nv_bfloat16>((size_t)T * d);
    std::vector<int> cu(B + 1);
    for (int b = 0; b <= B; ++b) cu[b] = b * S;
    int* dcu = to_dev(cu);
    for (int impl : {0, 0}) {
      cudaEvent_t e0, e1;
      CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
      SG(sgpt_attention(dq, dout, dcu, B, T, H, hd, 1.0f, 0, S, nullptr, impl, 0));
      CK(cudaEventRecord(e0));
      for (int it = 0; it < 20; ++it) SG(sgpt_attention(dq, dout, dcu, B, T, H, hd, 1.0f, 0, S, nullptr, impl, 0));
      CK(cudaEventRecord(e1));
      CK(cudaDeviceSynchronize());
      const double ms = time_ms(e0, e1) / 20;
      printf("INFO attention impl=%d: %.1f us, %.0f GB/s of qkv+out\n", impl, ms * 1e3,
             (double)T * d * 2 * 4 / (ms * 1e6));
    }
  }
  if (want("attention")) {
    test_attention({128}, 1, 64, 1.0f, 0, 0.3f);
    test_attention({1, 37, 128, 5, 64, 100}, 3, 64, 1.0f, 0, 0.3f);
    test_attention({300, 129, 256, 17}, 2, 64, 1.0f, 0, 0.3f);
    test_attention({300, 260, 40}, 2, 64, 1.0f, 256, 0.3f);
    test_attention({130, 64, 300}, 2, 128, 0.0883883f, 0, 1.0f);
    test_attention({300, 77}, 2, 256, 0.0625f, 0, 1.0f);
    test_attention({700, 513}, 1, 64, 0.125f, 256, 1.0f);
    test_attention({300, 41, 128}, 4, 128, 0.0883883f, 0, 1.0f, /*alibi=*/true);  // BLOOM-style
  }
  if (want("search")) {
    test_scores_topk(4, 1000, 64, 10);
    test_scores_topk(128, 5000, 768, 1001);
    test_scores_topk(37, 20011, 2048, 1001);
    test_scores_topk(3, 700, 128, 1001);  // n < k
    test_search(16, 400000, 128, 1001);   // two-pass threshold path
    test_search(5, 330001, 64, 10);       // two-pass, ragged last tile, small k
    test_search(130, 3000, 64, 50);       // > 128 queries -> query blocks, dense path
  }
  if (want("searchperf")) {
    // timing only: 128 queries x 1M docs x 768 (correctness of this path is covered above at smaller D)
    const int nq = 128, n = 1000000, D = 768, k = 1001;
    auto q = randn((size_t)nq * D, 1.f);
    auto qb = to_bf16(q);
    auto* dq = to_dev(qb);
    __nv_bfloat16* dc = dalloc<__nv_bfloat16>((size_t)n * D);
    {
      auto chunk = randn((size_t)100000 * D, 1.f);
      auto cb = to_bf16(chunk);
      for (int i = 0; i < 10; ++i)
        CK(cudaMemcpy(dc + (size_t)i * 100000 * D, cb.data(), cb.size() * 2, cudaMemcpyHostToDevice));
    }
    float *dqn = dalloc<float>(nq), *dcn = dalloc<float>(n);
    SG(sgpt_row_inv_norms(dq, dqn, nq, D, 0));
    SG(sgpt_row_inv_norms(dc, dcn, n, D, 0));
    const int64_t wsb = sgpt_search_workspace_bytes(nq, n, k);
    uint8_t* ws = dalloc<uint8_t>(wsb);
    float* dts = dalloc<float>((size_t)nq * k);
    int64_t* dti = dalloc<int64_t>((size_t)nq * k);
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    SG(sgpt_search(dq, dc, dqn, dcn, nq, n, D, k, 0, dts, dti, ws, wsb, 0));
    CK(cudaEventRecord(e0));
    for (int it = 0; it < 5; ++it) SG(sgpt_search(dq, dc, dqn, dcn, nq, n, D, k, 0, dts, dti, ws, wsb, 0));
    CK(cudaEventRecord(e1));
    CK(cudaDeviceSynchronize());
    const double ms = time_ms(e0, e1) / 5;
    printf("INFO search 128 x 1M x 768 top-1001: %.3f ms  (%.0f GB/s of corpus, %.0f q/s)\n", ms,
           (double)n * D * 2 / (ms * 1e6), nq / (ms * 1e-3));
  }
  printf("%s: %d failure(s)\n", g_fail ? "FAILED" : "ALL PASSED", g_fail);
  return g_fail ? 1 : 0;
}
