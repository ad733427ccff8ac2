// Stand-alone microbenchmark of bf16 -> bf16 LayerNorm kernel variants (tools/, not part of the library).
//   build:  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -o tools/ln_bench tools/ln_bench.cu
//   run:    tools/ln_bench T d     (e.g. 32768 768, 16384 2048, 9600 4096)
// Every variant is checked against a double-precision host LayerNorm of sampled rows (1 bf16 ulp), then timed with CUDA
// events over 40 launches, L2-warm (the same 2 buffers) and L2-cold (rotating over buffer pairs > 126 MB in total).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cmath>
#include <vector>

#define CK(x)                                                                                   \
  do {                                                                                          \
    cudaError_t e_ = (x);                                                                       \
    if (e_ != cudaSuccess) {                                                                    \
      fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));        \
      exit(1);                                                                                  \
    }                                                                                           \
  } while (0)

__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ void unpack8(const uint4& u, float (&v)[8]) {
  v[0] = bf16_lo(u.x); v[1] = bf16_hi(u.x); v[2] = bf16_lo(u.y); v[3] = bf16_hi(u.y);
  v[4] = bf16_lo(u.z); v[5] = bf16_hi(u.z); v[6] = bf16_lo(u.w); v[7] = bf16_hi(u.w);
}

template <int TPR>
__device__ __forceinline__ float group_sum(float v, float* scratch, int row_in_cta, int lane_in_row) {
  v = warp_sum(v);
  if (TPR == 32) return v;
  constexpr int W = TPR / 32;
  __syncthreads();
  if ((lane_in_row & 31) == 0) scratch[row_in_cta * W + (lane_in_row >> 5)] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < W; ++i) s += scratch[row_in_cta * W + i];
  return s;
}

// ---- variant B: the library's kernel (one row per TPR threads, one row per thread group per CTA) -------------------
template <int TPR, int V8, int MINB, bool kGB>
__global__ void __launch_bounds__(256, MINB) ln_base(const uint4* x, const float4* __restrict__ g,
                                                     const float4* __restrict__ b, uint4* y, int T, int d8, float eps) {
  constexpr int ROWS = 256 / TPR;
  __shared__ float scratch[ROWS * (TPR / 32) + 1];
  const int row_in_cta = threadIdx.x / TPR;
  const int l = threadIdx.x % TPR;
  const int row = blockIdx.x * ROWS + row_in_cta;
  const bool active = row < T;
  float v[V8][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < V8; ++i) {
    const int c = l + i * TPR;
    uint4 u = make_uint4(0u, 0u, 0u, 0u);
    if (active && c < d8) u = x[static_cast<size_t>(row) * d8 + c];
    unpack8(u, v[i]);
    s += ((v[i][0] + v[i][1]) + (v[i][2] + v[i][3])) + ((v[i][4] + v[i][5]) + (v[i][6] + v[i][7]));
  }
  const float inv_d = 1.0f / static_cast<float>(d8 * 8);
  const float mean = group_sum<TPR>(s, scratch, row_in_cta, l) * inv_d;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < V8; ++i) {
    if (l + i * TPR < d8) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float a = v[i][e] - mean;
        q = fmaf(a, a, q);
      }
    }
  }
  const float var = group_sum<TPR>(q, scratch, row_in_cta, l) * inv_d;
  const float rstd = rsqrtf(var + eps);
  if (!active) return;
#pragma unroll
  for (int i = 0; i < V8; ++i) {
    const int c = l + i * TPR;
    if (c < d8) {
      float gg[8] = {1, 1, 1, 1, 1, 1, 1, 1}, bb[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (kGB) {
        const float4 g0 = __ldg(g + 2 * c), g1 = __ldg(g + 2 * c + 1), b0 = __ldg(b + 2 * c), b1 = __ldg(b + 2 * c + 1);
        gg[0] = g0.x; gg[1] = g0.y; gg[2] = g0.z; gg[3] = g0.w; gg[4] = g1.x; gg[5] = g1.y; gg[6] = g1.z; gg[7] = g1.w;
        bb[0] = b0.x; bb[1] = b0.y; bb[2] = b0.z; bb[3] = b0.w; bb[4] = b1.x; bb[5] = b1.y; bb[6] = b1.z; bb[7] = b1.w;
      }
      float o[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = (v[i][e] - mean) * rstd * gg[e] + bb[e];
      y[static_cast<size_t>(row) * d8 + c] =
          make_uint4(pack_bf16(o[0], o[1]), pack_bf16(o[2], o[3]), pack_bf16(o[4], o[5]), pack_bf16(o[6], o[7]));
    }
  }
}

// ---- variant P: persistent thread groups, gamma / beta held in registers, PF rows of loads in flight per group --------
template <int TPR, int V8>
__device__ __forceinline__ void load_row(uint4 (&buf)[V8], const uint4* x, int row, int T, int d8, int l) {
#pragma unroll
  for (int i = 0; i < V8; ++i) {
    const int c = l + i * TPR;
    buf[i] = make_uint4(0u, 0u, 0u, 0u);
    if (row < T && c < d8) buf[i] = x[static_cast<size_t>(row) * d8 + c];
  }
}

template <int TPR, bool kWholeCta>
__device__ __forceinline__ float group_sum2(float v, float* scratch /* [ROWS][W] of this parity */, int row_in_cta,
                                            int lane_in_row) {
  v = warp_sum(v);
  if (TPR == 32) return v;
  constexpr int W = TPR / 32;
  if ((lane_in_row & 31) == 0) scratch[row_in_cta * W + (lane_in_row >> 5)] = v;
  if (kWholeCta) __syncthreads();
  else asm volatile("bar.sync %0, %1;" ::"r"(row_in_cta + 1), "r"(TPR) : "memory");
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < W; ++i) s += scratch[row_in_cta * W + i];
  return s;
}

template <int TPR, int V8, int PF, int MINB, int NT = 256>
__global__ void __launch_bounds__(NT, MINB) ln_persist(const uint4* x, const float4* __restrict__ g,
                                                        const float4* __restrict__ b, uint4* y, int T, int d8,
                                                        float eps) {
  constexpr int ROWS = NT / TPR;
  constexpr int W = TPR / 32;
  static_assert(NT % TPR == 0 && TPR % 32 == 0, "thread groups");
  __shared__ float scratch[2][ROWS * W + 1];
  const int rg = threadIdx.x / TPR;
  const int l = threadIdx.x % TPR;
  float gg[V8][8], bb[V8][8];
#pragma unroll
  for (int i = 0; i < V8; ++i) {
    const int c = l + i * TPR;
    float4 g0 = make_float4(0, 0, 0, 0), g1 = g0, b0 = g0, b1 = g0;
    if (c < d8) {
      g0 = __ldg(g + 2 * c); g1 = __ldg(g + 2 * c + 1); b0 = __ldg(b + 2 * c); b1 = __ldg(b + 2 * c + 1);
    }
    gg[i][0] = g0.x; gg[i][1] = g0.y; gg[i][2] = g0.z; gg[i][3] = g0.w;
    gg[i][4] = g1.x; gg[i][5] = g1.y; gg[i][6] = g1.z; gg[i][7] = g1.w;
    bb[i][0] = b0.x; bb[i][1] = b0.y; bb[i][2] = b0.z; bb[i][3] = b0.w;
    bb[i][4] = b1.x; bb[i][5] = b1.y; bb[i][6] = b1.z; bb[i][7] = b1.w;
  }
  const int stride = gridDim.x * ROWS;
  const int row0 = blockIdx.x * ROWS + rg;
  const int cta_row0 = blockIdx.x * ROWS;
  const int n_iter = cta_row0 < T ? (T - cta_row0 + stride - 1) / stride : 0;  // CTA-uniform
  const float inv_d = 1.0f / static_cast<float>(d8 * 8);
  uint4 buf[PF][V8];
#pragma unroll
  for (int p = 0; p < PF; ++p) load_row<TPR, V8>(buf[p], x, row0 + p * stride, T, d8, l);
  for (int it = 0; it < n_iter; it += PF) {
#pragma unroll
    for (int p = 0; p < PF; ++p) {
      if (it + p < n_iter) {  // CTA-uniform
        const int row = row0 + (it + p) * stride;
        float v[V8][8];
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < V8; ++i) {
          unpack8(buf[p][i], v[i]);
          s += ((v[i][0] + v[i][1]) + (v[i][2] + v[i][3])) + ((v[i][4] + v[i][5]) + (v[i][6] + v[i][7]));
        }
        // the registers of this row are free: fetch the row PF iterations ahead
        load_row<TPR, V8>(buf[p], x, row0 + (it + p + PF) * stride, T, d8, l);
        const float mean = group_sum2<TPR, TPR == NT>(s, scratch[0], rg, l) * inv_d;
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < V8; ++i) {
          if (l + i * TPR < d8) {
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              const float a = v[i][e] - mean;
              q = fmaf(a, a, q);
            }
          }
        }
        const float var = group_sum2<TPR, TPR == NT>(q, scratch[1], rg, l) * inv_d;
        const float rstd = rsqrtf(var + eps);
        if (row < T) {
#pragma unroll
          for (int i = 0; i < V8; ++i) {
            const int c = l + i * TPR;
            if (c < d8) {
              float o[8];
#pragma unroll
              for (int e = 0; e < 8; ++e) o[e] = (v[i][e] - mean) * rstd * gg[i][e] + bb[i][e];
              y[static_cast<size_t>(row) * d8 + c] =
                  make_uint4(pack_bf16(o[0], o[1]), pack_bf16(o[2], o[3]), pack_bf16(o[4], o[5]), pack_bf16(o[6], o[7]));
            }
          }
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256) copy_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, size_t n) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) y[i] = x[i];
}

// ---------------------------------------------------------------------------------------------------------------------
static float bf2f(uint16_t h) {
  uint32_t u = static_cast<uint32_t>(h) << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
static uint16_t f2bf(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  u += 0x7fffu + ((u >> 16) & 1u);
  return static_cast<uint16_t>(u >> 16);
}

struct Ctx {
  int T, d, d8, nbuf;
  std::vector<uint16_t*> x, y;
  float *g, *b;
  std::vector<uint16_t> hx;
  std::vector<float> hg, hb;
  float eps = 1e-5f;
  int sms;
};

template <class F>
static void run_variant(const char* name, Ctx& c, F launch, bool check = true) {
  // correctness on buffer 0
  CK(cudaMemset(c.y[0], 0, static_cast<size_t>(c.T) * c.d * 2));
  launch(c.x[0], c.y[0]);
  CK(cudaDeviceSynchronize());
  double max_ulp = 0;
  if (check) {
    std::vector<uint16_t> hy(static_cast<size_t>(c.T) * c.d);
    CK(cudaMemcpy(hy.data(), c.y[0], hy.size() * 2, cudaMemcpyDeviceToHost));
    for (int r = 0; r < c.T; r += (c.T / 61 > 0 ? c.T / 61 : 1)) {
      const uint16_t* xr = &c.hx[static_cast<size_t>(r) * c.d];
      double m = 0, q = 0;
      for (int k = 0; k < c.d; ++k) m += bf2f(xr[k]);
      m /= c.d;
      for (int k = 0; k < c.d; ++k) q += (bf2f(xr[k]) - m) * (bf2f(xr[k]) - m);
      const double rstd = 1.0 / sqrt(q / c.d + c.eps);
      for (int k = 0; k < c.d; ++k) {
        const double ref = (bf2f(xr[k]) - m) * rstd * c.hg[k] + c.hb[k];
        const double got = bf2f(hy[static_cast<size_t>(r) * c.d + k]);
        const double ulp = fabs(ref) * (1.0 / 128) + 1e-3;
        const double e = fabs(got - ref) / ulp;
        if (e > max_ulp) max_ulp = e;
      }
    }
    // last row too
  }
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  float ms_warm = 0, ms_cold = 0;
  const int iters = 40;
  for (int i = 0; i < 5; ++i) launch(c.x[0], c.y[0]);
  CK(cudaEventRecord(e0));
  for (int i = 0; i < iters; ++i) launch(c.x[0], c.y[0]);
  CK(cudaEventRecord(e1));
  CK(cudaEventSynchronize(e1));
  CK(cudaEventElapsedTime(&ms_warm, e0, e1));
  for (int i = 0; i < c.nbuf; ++i) launch(c.x[i], c.y[i]);
  CK(cudaEventRecord(e0));
  for (int i = 0; i < iters; ++i) launch(c.x[i % c.nbuf], c.y[i % c.nbuf]);
  CK(cudaEventRecord(e1));
  CK(cudaEventSynchronize(e1));
  CK(cudaEventElapsedTime(&ms_cold, e0, e1));
  const double mb = 2.0 * c.T * c.d * 2 / 1e6;
  printf("{\"variant\": \"%s\", \"T\": %d, \"d\": %d, \"us_l2_warm\": %.2f, \"us_l2_cold\": %.2f, \"tb_s_cold\": %.2f, "
         "\"max_err_ulp\": %.2f}\n",
         name, c.T, c.d, ms_warm * 1e3 / iters, ms_cold * 1e3 / iters, mb / (ms_cold * 1e3 / iters),
         max_ulp);
  fflush(stdout);
}

int main(int argc, char** argv) {
  Ctx c;
  c.T = argc > 1 ? atoi(argv[1]) : 32768;
  c.d = argc > 2 ? atoi(argv[2]) : 768;
  c.d8 = c.d / 8;
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  c.sms = prop.multiProcessorCount;
  const size_t n = static_cast<size_t>(c.T) * c.d;
  c.nbuf = static_cast<int>(900e6 / (4.0 * n)) + 1;  // > 126 MB L2 several times over
  if (c.nbuf > 12) c.nbuf = 12;
  if (c.nbuf < 3) c.nbuf = 3;
  c.hx.resize(n);
  c.hg.resize(c.d);
  c.hb.resize(c.d);
  uint32_t s = 12345u;
  auto rnd = [&]() {
    s = s * 1664525u + 1013904223u;
    return (static_cast<float>(s >> 8) / 16777216.0f) * 2.f - 1.f;
  };
  for (size_t i = 0; i < n; ++i) c.hx[i] = f2bf(rnd() * 3.f + ((i % c.d) == 7 ? 40.f : 0.3f));
  for (int k = 0; k < c.d; ++k) {
    c.hg[k] = 1.f + 0.2f * rnd();
    c.hb[k] = 0.1f * rnd();
  }
  c.x.resize(c.nbuf);
  c.y.resize(c.nbuf);
  for (int i = 0; i < c.nbuf; ++i) {
    CK(cudaMalloc(&c.x[i], n * 2));
    CK(cudaMalloc(&c.y[i], n * 2));
    CK(cudaMemcpy(c.x[i], c.hx.data(), n * 2, cudaMemcpyHostToDevice));
  }
  CK(cudaMalloc(&c.g, c.d * 4));
  CK(cudaMalloc(&c.b, c.d * 4));
  CK(cudaMemcpy(c.g, c.hg.data(), c.d * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(c.b, c.hb.data(), c.d * 4, cudaMemcpyHostToDevice));
  const int T = c.T, d8 = c.d8;
  const float eps = c.eps;
  const float4* g = reinterpret_cast<const float4*>(c.g);
  const float4* b = reinterpret_cast<const float4*>(c.b);
#define XY reinterpret_cast<const uint4*>(x), g, b, reinterpret_cast<uint4*>(y), T, d8, eps
  run_variant("copy", c, [&](uint16_t* x, uint16_t* y) {
    copy_kernel<<<c.sms * 8, 256>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(y), n / 8);
  }, false);
#define P(name, TPR, V8, PF, MINB, NT) \
  run_variant(name, c, [&](uint16_t* x, uint16_t* y) { ln_persist<TPR, V8, PF, MINB, NT><<<c.sms * MINB, NT>>>(XY); })
  if (d8 <= 96) {
    run_variant("base<32,3,6>", c, [&](uint16_t* x, uint16_t* y) { ln_base<32, 3, 6, true><<<(T + 7) / 8, 256>>>(XY); });
    run_variant("base<32,3,6> no gamma/beta loads", c,
                [&](uint16_t* x, uint16_t* y) { ln_base<32, 3, 6, false><<<(T + 7) / 8, 256>>>(XY); }, false);
    P("persist<32,3> PF1 2x256", 32, 3, 1, 2, 256);
    P("persist<32,3> PF2 2x256", 32, 3, 2, 2, 256);
    P("persist<32,3> PF3 2x256", 32, 3, 3, 2, 256);
    P("persist<32,3> PF2 4x128", 32, 3, 2, 4, 128);
    // one 16-byte chunk per thread, 96 threads per row: gamma / beta cost 16 registers
    P("persist<96,1> PF2 5x192", 96, 1, 2, 5, 192);
    P("persist<96,1> PF4 5x192", 96, 1, 4, 5, 192);
    P("persist<96,1> PF2 6x192", 96, 1, 2, 6, 192);
    P("persist<96,1> PF1 8x192", 96, 1, 1, 8, 192);
    P("persist<96,1> PF2 3x384", 96, 1, 2, 3, 384);
    P("persist<96,1> PF4 2x384", 96, 1, 4, 2, 384);
  } else if (d8 <= 256) {
    run_variant("base<128,4>", c, [&](uint16_t* x, uint16_t* y) { ln_base<128, 4, 1, true><<<(T + 1) / 2, 256>>>(XY); });
    run_variant("base<128,2,4>", c, [&](uint16_t* x, uint16_t* y) { ln_base<128, 2, 4, true><<<(T + 1) / 2, 256>>>(XY); });
    run_variant("base<128,2,4> no gamma/beta loads", c,
                [&](uint16_t* x, uint16_t* y) { ln_base<128, 2, 4, false><<<(T + 1) / 2, 256>>>(XY); }, false);
    P("persist<128,2> PF1 3x256", 128, 2, 1, 3, 256);
    P("persist<128,2> PF2 3x256", 128, 2, 2, 3, 256);
    P("persist<128,2> PF4 2x256", 128, 2, 4, 2, 256);
    P("persist<256,1> PF2 4x256", 256, 1, 2, 4, 256);
    P("persist<256,1> PF4 4x256", 256, 1, 4, 4, 256);
    P("persist<256,1> PF4 2x512", 256, 1, 4, 2, 512);
    P("persist<256,1> PF8 2x512", 256, 1, 8, 2, 512);
    P("persist<256,1> PF2 5x256", 256, 1, 2, 5, 256);
  } else {
    run_variant("base<256,4>", c, [&](uint16_t* x, uint16_t* y) { ln_base<256, 4, 1, true><<<T, 256>>>(XY); });
    run_variant("base<256,2,4>", c, [&](uint16_t* x, uint16_t* y) { ln_base<256, 2, 4, true><<<T, 256>>>(XY); });
    run_variant("base<256,2,4> no gamma/beta loads", c,
                [&](uint16_t* x, uint16_t* y) { ln_base<256, 2, 4, false><<<T, 256>>>(XY); }, false);
    P("persist<256,2> PF1 3x256", 256, 2, 1, 3, 256);
    P("persist<256,2> PF2 3x256", 256, 2, 2, 3, 256);
    P("persist<256,2> PF4 2x256", 256, 2, 4, 2, 256);
    P("persist<512,1> PF2 2x512", 512, 1, 2, 2, 512);
    P("persist<512,1> PF4 2x512", 512, 1, 4, 2, 512);
    P("persist<512,1> PF8 2x512", 512, 1, 8, 2, 512);
  }
  CK(cudaDeviceSynchronize());
  return 0;
}
