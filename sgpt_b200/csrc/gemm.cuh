// Persistent, warp-specialised wgmma GEMM for sm_90a:  C[M,N] = A[M,K] * B[N,K]^T  (bf16 in, fp32 accumulate; int8 or
// single-bit in, s32 accumulate for the similarity kernels, see kOp).
//
//   A : activations / queries, row-major [M,K]  -> K-major wgmma operand A
//   B : nn.Linear weight [out,in] / corpus shard [n,D], row-major [N,K] -> K-major wgmma operand B
//
// Two kernels share the operand pipeline (a TMA producer filling a kStages-deep smem ring of {A 128x64, B BNx64} tiles,
// SWIZZLE_128B, handed over with mbarriers only; the producer runs ahead across tiles):
//
// gemm_bf16_tn_kernel (similarity, filter and IVF scans; 9 warps = 288 threads, 1 CTA per SM):
//   warps 0..7   two consumer warpgroups: warpgroup g runs wgmma m64nBNk16 for rows [64 g, 64 g + 64) of the 128 x BN
//                tile with the fp32 accumulator in its registers, then the epilogue
//   warp  8      TMA producer
//   The consumers park the accumulator in shared memory (fp32, 128 rows x BN, each 128-byte row segment XOR-swizzled by
//   (row & 7) so that both the fragment stores and the row reads are free of bank conflicts), and the epilogue warps read
//   it back with thread = row, 32 consecutive columns per read (acc_ld_32): the score epilogues compare, scale and append
//   per query row.  E = 4 or 8 epilogue warps: warp w owns the 32-row slab (w % 4) and, with 8 warps, the column half
//   (w / 4).  EpiStaged<Op> (similarity scores) adds an smem transpose so that lane = column pair and each warp
//   instruction touches one contiguous row segment.
//
// gemm_linear_kernel (nn.Linear outputs, bf16; 3 warpgroups = 384 threads, 1 CTA per SM): ping-pong consumers, see there.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "gemm_api.h"

namespace sgpt {

constexpr int kGemmBM = 128;
constexpr int kGemmBK = 64;
constexpr int kGemmMmaWarps = 8;                        // two consumer warpgroups of 64 rows
constexpr int kGemmThreads = 32 * (kGemmMmaWarps + 1);  // + the TMA producer warp

template <int BN, int kStaging>
struct GemmCfg {
  static constexpr int kABytes = kGemmBM * kGemmBK * 2;
  static constexpr int kBBytes = BN * kGemmBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;  // 32 KB (BN 128) / 48 KB (BN 256)
  static constexpr int kBarrierBytes = 512;
  static constexpr int kAccBytes = kGemmBM * BN * 4;     // the fp32 accumulator handed to the epilogue
  static constexpr int kStagingBytes = kStaging;         // the epilogue's own shared memory (Epi::kStagingBytes)
  static constexpr int kStagesFit = (232448 - 1024 - kAccBytes - kStagingBytes - kBarrierBytes) / kStageBytes;
  static constexpr int kStages = kStagesFit < 4 ? kStagesFit : 4;
  static_assert(kStages >= 2, "not enough shared memory for a double-buffered mainloop");
  // smem: [<=1024 align slack][stages * (A|B)][accumulator][epilogue staging][barriers]
  static constexpr int kSmemBytes = 1024 + kStages * kStageBytes + kAccBytes + kStagingBytes + kBarrierBytes;
  static_assert(kSmemBytes <= 232448, "exceeds the 227 KB per-CTA shared memory limit");
};

// [0] SM cycles, [1] nanoseconds spent inside GEMM kernels (sgpt_profile_gemm_clock); one thread per launch adds to it
__device__ unsigned long long g_gemm_clock[2];
__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// 32 consecutive accumulator columns of this thread's row from the swizzled smem accumulator; `addr` is the row's
// address at a column that is a multiple of 32 (a 128-byte segment), chunk j of the segment sits at j ^ (row & 7)
// (row & 7 == lane & 7: the epilogue warps own 32-row slabs).
__device__ __forceinline__ void acc_ld_32(uint32_t addr, uint32_t (&v)[32]) {
  const uint32_t sw = threadIdx.x & 7u;
#pragma unroll
  for (uint32_t j = 0; j < 8; ++j) {
    const float4 x = lds_v4(addr + ((j ^ sw) << 4));
    v[4 * j] = __float_as_uint(x.x);
    v[4 * j + 1] = __float_as_uint(x.y);
    v[4 * j + 2] = __float_as_uint(x.z);
    v[4 * j + 3] = __float_as_uint(x.w);
  }
}

// Pins the accumulator registers at this point of the instruction stream: the compiler sees each wgmma as a synchronous
// read-modify-write of them, so without this it may copy or reorder accesses to registers an in-flight wgmma still writes.
template <int N>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int N>
__device__ __forceinline__ void wgmma_fence_acc(int32_t (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

template <int BN>
__device__ __forceinline__ void wgmma_mma(float (&d)[BN / 2], uint64_t da, uint64_t db, int scale_d) {
  if constexpr (BN == 128) wgmma_bf16_m64n128(d, da, db, scale_d);
  else wgmma_bf16_m64n256(d, da, db, scale_d);
}
template <int BN>
__device__ __forceinline__ void wgmma_mma(int32_t (&d)[BN / 2], uint64_t da, uint64_t db, int scale_d) {
  if constexpr (BN == 128) wgmma_s8_m64n128(d, da, db, scale_d);
  else wgmma_s8_m64n256(d, da, db, scale_d);
}
template <int BN>
__device__ __forceinline__ void wgmma_mma_b1(int32_t (&d)[BN / 2], uint64_t da, uint64_t db, int scale_d) {
  if constexpr (BN == 128) wgmma_b1_m64n128(d, da, db, scale_d);
  else wgmma_b1_m64n256(d, da, db, scale_d);
}

// accumulator element -> the fp32 bits parked in shared memory (an s32 dot product is rounded to nearest: cvt.rn.f32.s32)
__device__ __forceinline__ uint32_t acc_bits(float x) { return __float_as_uint(x); }
__device__ __forceinline__ uint32_t acc_bits(int32_t x) { return __float_as_uint(__int2float_rn(x)); }
// single-bit operands: a = popc(q AND d) -> 4 a + D, an exact fp32 integer (D <= 65536); the epilogue adds the row terms
__device__ __forceinline__ uint32_t acc_bits_b1(int32_t a, int dims) { return __float_as_uint(__int2float_rn(4 * a + dims)); }

// Optional selection of N-tiles: the similarity search scans a strided sample of corpus tiles first (to establish
// per-query thresholds) and the remaining tiles afterwards.
//   mode 0: all tiles;  mode 1: tiles 0, s, 2s, ...;  mode 2: every tile that is NOT a multiple of s   (s >= 2)
struct TileMap {
  int mode = 0;
  int stride = 1;
  // split-K (reduce-add epilogues only): every output tile is computed as `ksplit` work units over disjoint K ranges,
  // each adding its partial sum into the output; unit index = tile * ksplit + k-slice
  int ksplit = 1;
  // Rasterisation of the output tiles over the persistent CTAs.  band <= 1: N fastest (consecutive work units share the
  // activation rows and sweep the whole weight matrix: right while the weights stay in L2).  band = g: M-tile groups are
  // taken in bands of g, and inside a band the M index runs fastest — the 132 CTAs working at the same time then cover
  // g M-tiles x ~132/g N-tiles and fetch g + 132/g operand tiles instead of 1-2 + 131: for weight matrices larger than the
  // L2 (GPT-J / BLOOM-7B c_fc: 134 MB, streamed once per ~1 M-tile with N fastest) the operand traffic per wave drops
  // several-fold.
  int band = 0;
  __host__ __device__ void coords(int tile, int m_tiles, int n_tiles, int& mg, int& nt) const {
    if (band <= 1) {
      mg = tile / n_tiles;
      nt = tile - mg * n_tiles;
      return;
    }
    const int per_band = band * n_tiles;
    const int b = tile / per_band, r = tile - b * per_band;
    const int rest = m_tiles - b * band;
    const int h = rest < band ? rest : band;  // height of this band (the last one may be lower)
    nt = r / h;
    mg = b * band + (r - nt * h);
  }
  __host__ __device__ int count(int n_tiles) const {
    if (mode == 0) return n_tiles;
    const int sampled = (n_tiles + stride - 1) / stride;
    return mode == 1 ? sampled : n_tiles - sampled;
  }
  __host__ __device__ int map(int j) const {
    if (mode == 0) return j;
    if (mode == 1) return j * stride;
    return j + j / (stride - 1) + 1;
  }
};

// CL = 1: one 128 x BN tile per work unit.
// CL = 2: two CTAs per work unit on the same N-tile and adjacent M-tiles (CTA r of the unit owns rows [128 r, 128 r + 128)
//   of a 256 x BN tile group): the similarity search scans up to 256 queries per pass over the corpus this way, and both
//   CTAs of a unit share the candidate-list group of the unit (EpiFilterRows).
// kOp: the operand type (gemm_api.h Operand).  kS8: int8 operands (int8 corpus shards, similarity epilogues only).  A
//   K-block is then 128 int8 = the same 128 bytes per row as 64 bf16, so the stage layout, TMA boxes, descriptor steps
//   and ring are unchanged; wgmma k32 accumulates in s32, exact for |dot| < 2^31, and the accumulator is converted to
//   fp32 where it is parked in shared memory, so every epilogue runs unchanged.
//   kB1: packed sign bits (binary corpus shards), K counted in bytes (D / 8).  A K-block is again 128 bytes = 1024 bits
//   per row and a wgmma k256 (.and.popc) takes 32 bytes, the s8 geometry exactly; TMA zero fill of a ragged last k-block
//   adds no AND bits.  The s32 a = popc(q AND d) is parked as the fp32 integer 4 a + D, and the b1 epilogues
//   (kB1 of EpiFilterRowsT / OpScoresF32T) add the query and document terms -2 popc(q), -2 popc(d) to it.
// kUnits: the work units are read from a table in device memory instead of being derived from (M, N) and the TileMap:
//   unit u is ep.units[u] = (m0, m_end, n0, n_end), one 128 x BN tile at rows m0 / columns n0 whose epilogue sees only
//   rows < m_end and columns < n_end (passed to it as M and N), and min(*ep.n_units, ep.max_units) units exist.  The
//   count is read on the device, so the grid is fixed at launch and nothing waits for the host (the grouped IVF scan,
//   ivf.cu).  CL = 1 and no split-K; M and N bound the tensor maps only.
template <int BN, class Epi, int CL = 1, Operand kOp = Operand::kBF16, bool kUnits = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_tn_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b, int M,
                    int N, int K, const __grid_constant__ typename Epi::Params ep, TileMap tmap) {
  using Cfg = GemmCfg<BN, Epi::kStagingBytes>;
  constexpr bool kS8 = kOp != Operand::kBF16;      // 1-byte K elements (int8, or 8 packed bits)
  using Acc = typename std::conditional<kS8, int32_t, float>::type;
  constexpr int kBK = kS8 ? 2 * kGemmBK : kGemmBK;  // K elements per k-block (128 bytes per row either way)
  constexpr int kMmaK = kS8 ? 32 : 16;              // K elements per wgmma
  constexpr int kStages = Cfg::kStages;
  static_assert(CL == 1 || CL == 2, "work unit size");
  static_assert(Epi::kEpiWarps == 4 || Epi::kEpiWarps == 8, "4 or 8 epilogue warps");
  static_assert(BN == 128 || BN == 256, "tile width");
  static_assert(!kUnits || CL == 1, "unit tables name single-CTA tiles");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_tiles = smem;
  uint8_t* acc_smem = smem + kStages * Cfg::kStageBytes;
  float* stage_base = reinterpret_cast<float*>(acc_smem + Cfg::kAccBytes);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(acc_smem + Cfg::kAccBytes + Cfg::kStagingBytes);
  uint64_t* empty_bar = full_bar + kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr int kWarpProducer = kGemmMmaWarps;

  const int crank = CL > 1 ? static_cast<int>(blockIdx.x % CL) : 0;  // M-tile of the unit's tile group
  const int cid = blockIdx.x / CL, ncl = gridDim.x / CL;               // unit slot / number of unit slots
  const int m_tiles = ((M + kGemmBM - 1) / kGemmBM + CL - 1) / CL;    // M-tile groups (CL tiles each)
  const int n_tiles = tmap.count((N + BN - 1) / BN);                  // N-tiles this launch visits
  const int ksplit = tmap.ksplit;
  int num_tiles = m_tiles * n_tiles * ksplit;  // work units
  const int num_kb = (K + kBK - 1) / kBK;
  const int kb_per = (num_kb + ksplit - 1) / ksplit;  // k-blocks per slice (the host keeps every slice non-empty)

  if (warp == kWarpProducer && lane == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kGemmMmaWarps);  // one arrive per consumer warp: each warp waits for its own wgmma part
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();  // everything above overlapped the previous kernel's tail; global memory is touched only below
  if constexpr (kUnits) num_tiles = min(__ldg(ep.n_units), ep.max_units);
  const bool clock_probe = (blockIdx.x == 0 && threadIdx.x == 0);
  const long long probe_c0 = clock_probe ? clock64() : 0;
  const uint64_t probe_t0 = clock_probe ? global_timer_ns() : 0;

  if (warp == kWarpProducer) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int unit = cid; unit < num_tiles; unit += ncl) {
        const int tile = unit / ksplit, ks = unit - tile * ksplit;
        int m0, n0;
        if constexpr (kUnits) {
          const int4 u = __ldg(ep.units + unit);
          m0 = u.x;
          n0 = u.z;
        } else {
          int mg, nt;
          tmap.coords(tile, m_tiles, n_tiles, mg, nt);
          m0 = (mg * CL + crank) * kGemmBM;
          n0 = tmap.map(nt) * BN;
        }
        const int kb_end = min(num_kb, (ks + 1) * kb_per);
        for (int kb = ks * kb_per; kb < kb_end; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem_tiles + stage * Cfg::kStageBytes;
          uint8_t* sb = sa + Cfg::kABytes;
          mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          tma_load_2d(sa, &tma_a, &full_bar[stage], kb * kBK, m0);
          tma_load_2d(sb, &tma_b, &full_bar[stage], kb * kBK, n0);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: wgmma mainloop, then the epilogue =====================
    const int wg = warp >> 2;              // consumer warpgroup = 64-row half of the tile
    const int ew = warp & 3;               // 32-row slab of the tile this warp's epilogue owns
    const int half = warp >> 2;            // column half handled by this warp's epilogue (always 0 with 4 epilogue warps)
    const bool epi_warp = warp < Epi::kEpiWarps;
    constexpr int kColsPerWarp = BN / (Epi::kEpiWarps / 4);
    constexpr int kSlabBytes = Cfg::kStagingBytes / Epi::kEpiWarps;
    float* stage_slab = stage_base + (epi_warp ? warp : 0) * (kSlabBytes / 4);
    const uint32_t acc_base = smem_u32(acc_smem);
    typename Epi::State st;
    if (epi_warp) Epi::init(st, ep);
    int stage = 0;
    uint32_t phase = 0;
    for (int unit = cid; unit < num_tiles; unit += ncl) {
      const int tile = unit / ksplit;
      const int ks = unit - tile * ksplit;
      int m0, n0, Me = M, Ne = N;  // this warp's 32-row slab / column half, and the bounds its epilogue sees
      if constexpr (kUnits) {
        const int4 u = __ldg(ep.units + unit);
        m0 = u.x + ew * 32;
        n0 = u.z + half * kColsPerWarp;
        Me = u.y;
        Ne = u.w;
      } else {
        int mg, ntile;
        tmap.coords(tile, m_tiles, n_tiles, mg, ntile);
        m0 = (mg * CL + crank) * kGemmBM + ew * 32;
        n0 = tmap.map(ntile) * BN + half * kColsPerWarp;
      }
      if (epi_warp) {
        // work that does not depend on the accumulator (EpiFilterRows: the document scales and thresholds of the tile)
        // overlaps the mainloop
        Epi::template pre_tile<kColsPerWarp, kSlabBytes>(st, ep, m0, n0, lane, stage_slab, Me, Ne);
      }

      Acc acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = Acc(0);
      const int kb_begin = ks * kb_per, kb_end = min(num_kb, kb_begin + kb_per);
      int prev_stage = -1;
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem_tiles + stage * Cfg::kStageBytes) + wg * (64 * 128);
        const uint32_t sb = smem_u32(smem_tiles + stage * Cfg::kStageBytes) + Cfg::kABytes;
        const uint64_t da = make_wgmma_desc_sw128(sa), db = make_wgmma_desc_sw128(sb);
        wgmma_fence_acc(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / kMmaK; ++k) {
          if constexpr (kOp == Operand::kB1) wgmma_mma_b1<BN>(acc, da + 2 * k, db + 2 * k, (kb > kb_begin || k > 0) ? 1 : 0);
          else wgmma_mma<BN>(acc, da + 2 * k, db + 2 * k, (kb > kb_begin || k > 0) ? 1 : 0);
        }
        wgmma_commit();
        wgmma_fence_acc(acc);
        if constexpr (BN == 128) {
          // one k-block stays in flight: the stage of the PREVIOUS k-block has been read once its group completed
          wgmma_wait<1>();
          if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
          prev_stage = stage;
        } else {
          // 128 accumulators per thread: keeping a group in flight across the next barrier wait spills them (the
          // 288-thread CTA caps a thread at 168 registers), so this k-block completes before the next one is issued
          wgmma_wait<0>();
          if (lane == 0) mbar_arrive(&empty_bar[stage]);
        }
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);

      // accumulator -> smem (the previous tile's epilogue reads must be over), then the epilogue reads it back by rows
      named_bar_sync(1, 32 * kGemmMmaWarps);
      {
        const int t = threadIdx.x & 127;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2) + 8 * h;
          const uint32_t rbase = acc_base + static_cast<uint32_t>(row) * (BN * 4);
          const uint32_t sw = static_cast<uint32_t>(row & 7);
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const uint32_t col = 8 * j + 2 * (t & 3);
            const uint32_t chunk = col >> 2;
            const uint32_t phys = (chunk & ~7u) | ((chunk & 7u) ^ sw);
            if constexpr (kOp == Operand::kB1)
              sts_v2(rbase + phys * 16 + (col & 3u) * 4, acc_bits_b1(acc[4 * j + 2 * h], 8 * K),
                     acc_bits_b1(acc[4 * j + 2 * h + 1], 8 * K));
            else
              sts_v2(rbase + phys * 16 + (col & 3u) * 4, acc_bits(acc[4 * j + 2 * h]), acc_bits(acc[4 * j + 2 * h + 1]));
          }
        }
      }
      named_bar_sync(1, 32 * kGemmMmaWarps);
      if (epi_warp) {
        const uint32_t trow = acc_base + static_cast<uint32_t>(ew * 32 + lane) * (BN * 4) + half * kColsPerWarp * 4;
        Epi::template tile<kColsPerWarp, kSlabBytes>(st, ep, m0, n0, lane, trow, stage_slab, Me, Ne);
      }
    }
    if (epi_warp) {
      Epi::finish(st, ep, crank * kGemmBM + ew * 32 + lane);  // row inside the CL x 128-row tile group
      if (clock_probe) {
        atomicAdd(&g_gemm_clock[0], static_cast<unsigned long long>(clock64() - probe_c0));
        atomicAdd(&g_gemm_clock[1], static_cast<unsigned long long>(global_timer_ns() - probe_t0));
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Linear-layer GEMM: out[M,N] (bf16) = Op(A[M,K] B[N,K]^T), written by TMA as a tensor store or a reduce-add.
//
// Roles (3 warpgroups = 384 threads, 1 CTA per SM, clusters of 2 CTAs):
//   warpgroup 0      TMA producer (one lane), lowered to 40 registers per thread (setmaxnreg.dec)
//   warpgroups 1, 2  consumers, raised to 232 registers per thread (setmaxnreg.inc).  Consumer c takes work units
//                    c, c + 2, c + 4, ... of the CTA's sequence and computes each whole 128 x 128 tile (two m64n128k16
//                    per K step, 128 fp32 accumulators per thread), then runs its epilogue.
// Cluster pairing: a work unit is a pair of vertically adjacent M-tiles on one N-tile (and one K slice with split-K);
// cluster rank r computes M-tile 2 mp + r of pair mp, and both CTAs walk the same unit sequence and k-blocks, which is
// all that keeps their rings in step.  Per k-block each producer loads its own A box (128 x 64) and one 64-row half of
// the shared B tile, multicast into the same stage of both CTAs: 24 KB of L2 reads per CTA instead of 32 KB.  A stage
// therefore holds bytes written by both producers, and it is refilled only once the owning consumer of BOTH CTAs has
// read it: its empty barrier takes 8 arrivals, each consumer warp arriving on its own CTA's barrier and on the
// partner's.  With an odd number of M-tiles, rank 1 of the last pair loads a box wholly past M (TMA zero fill, its full
// byte count) and stores nothing, but takes part in every load, multicast and barrier like any other unit.  No CTA
// leaves before the final cluster barrier: its partner may still multicast into its shared memory or arrive on its
// barriers until then.
// Ping-pong: once a consumer has issued its last k-block it arrives at the other consumer's turn barrier, so one
// consumer's mainloop runs while the other runs its epilogue (kBarTurn + c, 256 threads: every arrive is matched by the
// one wait of the next unit).  The producer walks the same unit sequence (TileMap banding over pair units, split-K).
// Epilogue: Op::pair maps each fp32 accumulator pair to two bf16 in registers; the words go to the consumer's own 32 KB
// output tile (8 SWIZZLE_128B boxes of 32 rows x 64 columns, the box of the output tensor map) and one thread hands the
// boxes to the TMA engine.  The tile is rewritten only once the previous tile's stores have read it (wait_group.read),
// which by then lies a whole mainloop back.  The score epilogues keep gemm_bf16_tn_kernel: they need a thread to own a
// query row (per-row thresholds and candidate lists), i.e. the fp32 hand-over through shared memory.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kLinThreads = 384;
constexpr int kLinBN = 128;
constexpr int kLinCluster = 2;  // CTAs per cluster: two M-tiles sharing each weight tile
struct LinearCfg {
  static constexpr int kABytes = kGemmBM * kGemmBK * 2;
  static constexpr int kBRows = kLinBN / kLinCluster;                 // B rows each CTA loads and multicasts
  static constexpr int kBPartBytes = kBRows * kGemmBK * 2;            // 8 KB
  static constexpr int kStageBytes = kABytes + kLinBN * kGemmBK * 2;  // 32 KB
  static constexpr int kStages = 5;  // 5 x 32 KB: measured faster than 4 with the cluster pairing (DESIGN.md)
  static constexpr int kOutBytes = kGemmBM * kLinBN * 2;              // one consumer's bf16 output tile
  static constexpr int kBarrierBytes = 512;
  // smem: [<=1024 align slack][stages * (A|B)][2 output tiles][barriers]
  static constexpr int kSmemBytes = 1024 + kStages * kStageBytes + 2 * kOutBytes + kBarrierBytes;
  static_assert(kSmemBytes <= 232448, "exceeds the 227 KB per-CTA shared memory limit");
  // the B parts stack into the layout of one 128-row SWIZZLE_128B box (the swizzle repeats every 8 rows = 1 KB)
  static_assert(kBPartBytes % 1024 == 0 && kBPartBytes * kLinCluster == kLinBN * kGemmBK * 2, "B tile split");
};
// named barriers of gemm_linear_kernel (0 is __syncthreads): all consumers; turn of consumer c; epilogue of consumer c
constexpr int kBarConsumers = 1, kBarTurn = 2, kBarEpi = 4;

// kOp: kBF16, or kE4M3 (fp8 linear layers): a K-block is then 128 e4m3 = the same 128 bytes per row as 64 bf16, so the
// stages, TMA boxes, ring and the +32-byte descriptor step per MMA are unchanged; 4 m64n128k32 per k-block and operand
// half instead of 4 m64n128k16, fp32 accumulators either way (Op is the dequantizing OpDequantE4M3<...>).
template <class Op, Operand kOp = Operand::kBF16>
__global__ void __launch_bounds__(kLinThreads, 1)
gemm_linear_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b, int M, int N,
                   int K, const __grid_constant__ typename Op::Params ep, TileMap tmap) {
  using Cfg = LinearCfg;
  constexpr int kStages = Cfg::kStages;
  static_assert(kOp == Operand::kBF16 || kOp == Operand::kE4M3, "linear-layer operand type");
  constexpr bool kF8 = kOp == Operand::kE4M3;
  constexpr int kBK = kF8 ? 2 * kGemmBK : kGemmBK;  // K elements per k-block (128 bytes per row either way)
  constexpr int kMmaK = kF8 ? 32 : 16;              // K elements per wgmma
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_tiles = smem;
  uint8_t* out_smem = smem + kStages * Cfg::kStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(out_smem + 2 * Cfg::kOutBytes);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* probe = empty_bar + kStages;  // clock probe: start cycle and time (kept out of the consumers' registers)

  const int rank = static_cast<int>(cluster_ctarank());  // M-tile of the pair this CTA computes
  const int cid = blockIdx.x / kLinCluster, ncl = gridDim.x / kLinCluster;  // cluster / number of clusters
  const int m_tiles = (M + kGemmBM - 1) / kGemmBM;
  const int m_pairs = (m_tiles + kLinCluster - 1) / kLinCluster;
  const int n_tiles = (N + kLinBN - 1) / kLinBN;
  const int ksplit = tmap.ksplit;
  const int num_units = m_pairs * n_tiles * ksplit;
  const int num_kb = (K + kBK - 1) / kBK;
  const int kb_per = (num_kb + ksplit - 1) / ksplit;  // k-blocks per slice (the host keeps every slice non-empty)

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    // full: the local producer's arrive.expect_tx (the bytes come from both producers)
    // empty: one arrive per warp of the stage's consumer, in this CTA and in the partner
    constexpr uint32_t kFullArrivals = 1, kEmptyArrivals = 4 * kLinCluster;
    static_assert(kEmptyArrivals == 8, "4 local + 4 remote consumer warps release a stage");
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], kFullArrivals);
      mbar_init(&empty_bar[i], kEmptyArrivals);
    }
    fence_mbar_init();
  }
  cluster_sync();  // both CTAs' barriers are initialised before any multicast or remote arrive can reach them
  pdl_sync();  // everything above overlapped the previous kernel's tail; global memory is touched only below

  if (threadIdx.x < 128) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int unit = cid; unit < num_units; unit += ncl) {
        const int tile = unit / ksplit, ks = unit - tile * ksplit;
        int mp, nt;
        tmap.coords(tile, m_pairs, n_tiles, mp, nt);
        const int m0 = (kLinCluster * mp + rank) * kGemmBM, nb = nt * kLinBN + rank * Cfg::kBRows;
        const int kb_end = min(num_kb, (ks + 1) * kb_per);
        for (int kb = ks * kb_per; kb < kb_end; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);  // read by the owning consumer of both CTAs
          uint8_t* sa = smem_tiles + stage * Cfg::kStageBytes;
          mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          tma_load_2d(sa, &tma_a, &full_bar[stage], kb * kBK, m0);
          tma_load_2d_multicast(sa + Cfg::kABytes + rank * Cfg::kBPartBytes, &tma_b, &full_bar[stage], kb * kBK, nb,
                                (1u << kLinCluster) - 1);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    cluster_sync();
    return;
  }

  // ===================== consumers: whole tiles, alternating =====================
  setmaxnreg_inc<232>();
  const int c = (threadIdx.x >> 7) - 1;
  const int t = threadIdx.x & 127;
  const int lane = t & 31;
  const int r0 = 16 * (t >> 5) + (lane >> 2);  // this thread's fragment rows: r0 + {0, 8, 64, 72}
  const int c0 = 2 * (lane & 3);               // this thread's fragment column pairs: c0 + 8 j, j = 0..15
  const uint32_t out_tile = smem_u32(out_smem + c * Cfg::kOutBytes);
  const bool clock_probe = (blockIdx.x == 0 && threadIdx.x == 128);
  if (clock_probe) {
    probe[0] = static_cast<uint64_t>(clock64());
    probe[1] = global_timer_ns();
  }
  // a stage is released on this CTA's empty barrier and on the partner's (its B part came from there)
  auto release = [&](int s) {
    mbar_arrive(&empty_bar[s]);
    mbar_arrive_cluster(mapa_shared(smem_u32(&empty_bar[s]), cluster_ctarank() ^ 1u));
  };
  int stage = 0;
  uint32_t phase = 0;
  int i = 0;  // position of the unit in this cluster's sequence
  for (int unit = cid; unit < num_units; unit += ncl, ++i) {
    const int tile = unit / ksplit, ks = unit - tile * ksplit;
    const int kb_begin = ks * kb_per, kb_end = min(num_kb, kb_begin + kb_per);
    if ((i & 1) != c) {  // the other consumer's unit: step over its k-blocks in the ring
      stage += kb_end - kb_begin;
      phase ^= static_cast<uint32_t>(stage / kStages) & 1u;
      stage %= kStages;
      continue;
    }
    float acc0[64], acc1[64];  // rows [0, 64) and [64, 128) of the tile
#pragma unroll
    for (int j = 0; j < 64; ++j) acc0[j] = acc1[j] = 0.f;
    if (i > 0) named_bar_sync(kBarTurn + c, 256);  // the other consumer has issued its last k-block
    int prev_stage = -1;
    for (int kb = kb_begin; kb < kb_end; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem_tiles + stage * Cfg::kStageBytes);
      const uint64_t da0 = make_wgmma_desc_sw128(sa), da1 = make_wgmma_desc_sw128(sa + 64 * 128);
      const uint64_t db = make_wgmma_desc_sw128(sa + Cfg::kABytes);
      wgmma_fence_acc(acc0);
      wgmma_fence_acc(acc1);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBK / kMmaK; ++k) {
        const int scale_d = (kb > kb_begin || k > 0) ? 1 : 0;
        if constexpr (kF8) {
          wgmma_e4m3_m64n128(acc0, da0 + 2 * k, db + 2 * k, scale_d);
          wgmma_e4m3_m64n128(acc1, da1 + 2 * k, db + 2 * k, scale_d);
        } else {
          wgmma_bf16_m64n128(acc0, da0 + 2 * k, db + 2 * k, scale_d);
          wgmma_bf16_m64n128(acc1, da1 + 2 * k, db + 2 * k, scale_d);
        }
      }
      wgmma_commit();
      wgmma_fence_acc(acc0);
      wgmma_fence_acc(acc1);
      // one k-block stays in flight: the stage of the PREVIOUS k-block has been read once its group completed
      wgmma_wait<1>();
      if (prev_stage >= 0 && lane == 0) release(prev_stage);
      prev_stage = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    if (unit + ncl < num_units) named_bar_arrive(kBarTurn + (c ^ 1), 256);
    wgmma_wait<0>();
    wgmma_fence_acc(acc0);
    wgmma_fence_acc(acc1);
    if (prev_stage >= 0 && lane == 0) release(prev_stage);

    int mp, nt;
    tmap.coords(tile, m_pairs, n_tiles, mp, nt);
    const int m0 = (kLinCluster * mp + rank) * kGemmBM, n0 = nt * kLinBN;
    // epilogue: all results are computed before any is stored, so the loads inside Op::rows / Op::col / Op::pair are
    // ordinary loads the compiler batches up front (the volatile smem stores would otherwise fence them apart)
    typename Op::Rows rw;
    Op::rows(ep, rw, m0 + r0, M);
    uint32_t o[4][16];  // [fragment row][column pair]
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const typename Op::Col cl = Op::col(ep, n0 + c0 + 8 * j, N, ks == 0);
      o[0][j] = Op::pair(ep, rw, cl, 0, acc0[4 * j], acc0[4 * j + 1]);
      o[1][j] = Op::pair(ep, rw, cl, 1, acc0[4 * j + 2], acc0[4 * j + 3]);
      o[2][j] = Op::pair(ep, rw, cl, 2, acc1[4 * j], acc1[4 * j + 1]);
      o[3][j] = Op::pair(ep, rw, cl, 3, acc1[4 * j + 2], acc1[4 * j + 3]);
    }
    if (t == 0) bulk_wait_group_read<0>();  // this consumer's previous stores have read the output tile
    named_bar_sync(kBarEpi + c, 128);
    // box b = (row / 32) * 2 + column / 64; 16-byte chunk q of box row rr sits at q ^ (rr & 7), and rr & 7 = lane / 4
#pragma unroll
    for (int ri = 0; ri < 4; ++ri) {
      const int row = r0 + 8 * (ri & 1) + 64 * (ri >> 1);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const uint32_t box = static_cast<uint32_t>((row >> 5) * 2 + (j >> 3));
        sts_b32(out_tile + box * 4096u + static_cast<uint32_t>(row & 31) * 128u +
                    ((static_cast<uint32_t>(j & 7) ^ static_cast<uint32_t>(lane >> 2)) << 4) + 4u * (lane & 3),
                o[ri][j]);
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(kBarEpi + c, 128);
    if (t == 0) {
#pragma unroll 1
      for (int b = 0; b < 8; ++b) {  // boxes wholly past M or N are skipped; the tensor map clips the others
        const int bm = m0 + 32 * (b >> 1), bn = n0 + 64 * (b & 1);
        if (bm < M && bn < N)
          Op::issue(ep, reinterpret_cast<const void*>(__cvta_shared_to_generic(out_tile + b * 4096u)), bn, bm);
      }
      bulk_commit_group();
    }
  }
  if (t == 0) bulk_wait_group<0>();  // all stores of this consumer have fully completed
  named_bar_sync(kBarConsumers, 256);
  if (clock_probe) {
    atomicAdd(&g_gemm_clock[0], static_cast<unsigned long long>(clock64()) - probe[0]);
    atomicAdd(&g_gemm_clock[1], static_cast<unsigned long long>(global_timer_ns()) - probe[1]);
  }
  cluster_sync();  // the partner's last multicasts into this CTA and arrives on its barriers are over
}

// ---------------------------------------------------------------------------------------------------------------
// Linear-layer epilogue ops, applied in the accumulator fragment, whose rows are r, r + 8, r + 64, r + 72 (ri = 0..3) and
// whose column pairs start at col0 + 8 j (j = 0..15) of the tile: Op::rows fetches what the rows need (r0: global row of
// ri = 0), Op::col what the pair starting at global column `col` needs, and Op::pair maps the fp32 accumulators of the
// pair in row ri to two packed bf16.
// ---------------------------------------------------------------------------------------------------------------
// bias of columns (col, col + 1), 0 without a bias; columns beyond N are clipped by the tensor map, their bias is read
// from the last valid entry
__device__ __forceinline__ float2 bias_pair(const float* bias, int col, int N) {
  if (bias == nullptr) return make_float2(0.f, 0.f);
  if (col + 2 <= N) return __ldg(reinterpret_cast<const float2*>(bias + col));
  return make_float2(__ldg(bias + (col < N ? col : N - 1)), __ldg(bias + (col + 1 < N ? col + 1 : N - 1)));
}
struct NoRows {};

// out_bf16[m, n] = act(acc + bias[n])          act = identity | gelu_new
template <bool kGelu>
struct OpTmaBiasActBF16 {
  struct Params {
    CUtensorMap out_map;  // bf16 [M, N], box 32 rows x 64 cols, SWIZZLE_128B
    const float* bias;    // may be null
  };
  using Rows = NoRows;
  using Col = float2;  // bias
  static __device__ __forceinline__ void rows(const Params&, Rows&, int, int) {}
  static __device__ __forceinline__ Col col(const Params& p, int c, int N, bool) { return bias_pair(p.bias, c, N); }
  static __device__ __forceinline__ uint32_t pair(const Params&, const Rows&, Col b, int, float x0, float x1) {
    x0 = x0 + b.x;
    x1 = x1 + b.y;
    if (kGelu) {
      x0 = gelu_new(x0);
      x1 = gelu_new(x1);
    }
    return pack_bf16(x0, x1);
  }
  static __device__ __forceinline__ void issue(const Params& p, const void* box, int n, int m0) {
    tma_store_2d(&p.out_map, box, n, m0);
  }
};

// Profiling aid (sgpt_linear epilogue 100): the whole kernel, epilogue arithmetic and output-tile writes included, but no
// stores to global memory, so that the product time minus this time is what the stores cost on the same kernel.
struct OpNoStoreBF16 {
  struct Params {
    int unused;
  };
  using Rows = NoRows;
  using Col = float2;
  static __device__ __forceinline__ void rows(const Params&, Rows&, int, int) {}
  static __device__ __forceinline__ Col col(const Params&, int, int, bool) { return make_float2(0.f, 0.f); }
  static __device__ __forceinline__ uint32_t pair(const Params&, const Rows&, Col, int, float x0, float x1) {
    return pack_bf16(x0, x1);
  }
  static __device__ __forceinline__ void issue(const Params&, const void*, int, int) {}
};

// GPT-J fused q/k/v projection: out_bf16[m, n] = rotary(acc) for the first `rotary_dim` dims of every q and k head
// (HF:gptj/modeling_gptj.py:55-67, 196-207: interleaved pairs (x[2i], x[2i+1]) -> (x[2i] c - x[2i+1] s, x[2i+1] c + x[2i] s)
// with angle pos[m] * 10000^(-2i/rotary_dim)); v columns and the non-rotary dims pass through.  No bias (:98-101).  The
// rotated pairs are exactly the accumulator fragment's column pairs.
struct OpTmaRotaryBF16 {
  struct Params {
    CUtensorMap out_map;     // bf16 [M, 3d]
    const int32_t* pos;      // [M] position of each token row
    const float2* table;     // [max_pos, rotary_dim/2] (cos, sin)
    int M, d_model, head_dim, rotary_dim, max_pos;
  };
  struct Rows { const float2* t[4]; };  // the table row of each fragment row's position
  using Col = int;                       // rotated pair: its index in the head's table row; -1: passes through
  static __device__ __forceinline__ void rows(const Params& p, Rows& rw, int r0, int) {
#pragma unroll
    for (int ri = 0; ri < 4; ++ri) {
      const int row = r0 + 8 * (ri & 1) + 64 * (ri >> 1);
      int ps = __ldg(p.pos + (row < p.M ? row : p.M - 1));
      ps = min(max(ps, 0), p.max_pos - 1);
      rw.t[ri] = p.table + static_cast<size_t>(ps) * (p.rotary_dim >> 1);
    }
  }
  static __device__ __forceinline__ Col col(const Params& p, int c, int, bool) {
    const int in_head = c % p.head_dim;
    return (c < 2 * p.d_model && in_head < p.rotary_dim) ? (in_head >> 1) : -1;
  }
  static __device__ __forceinline__ uint32_t pair(const Params&, const Rows& rw, Col k, int ri, float x0, float x1) {
    if (k >= 0) {
      const float2 cs = __ldg(rw.t[ri] + k);
      const float e = x0, od = x1;
      x0 = e * cs.x - od * cs.y;
      x1 = od * cs.x + e * cs.y;
    }
    return pack_bf16(x0, x1);
  }
  static __device__ __forceinline__ void issue(const Params& p, const void* box, int n, int m0) {
    tma_store_2d(&p.out_map, box, n, m0);
  }
};

// resid_bf16[m, n] += acc + bias[n]     (the residual stream updated in place by a bf16 TMA reduce-add performed by
// the L2: no residual load in the SM).  Split-K: every K slice adds its partial sum, only slice 0 adds the bias.
struct OpTmaResidAddBF16 {
  struct Params {
    CUtensorMap out_map;  // bf16 [M, N], box 32 rows x 64 cols, SWIZZLE_128B
    const float* bias;    // may be null
  };
  using Rows = NoRows;
  using Col = float2;  // bias (0 in the K slices after the first)
  static __device__ __forceinline__ void rows(const Params&, Rows&, int, int) {}
  static __device__ __forceinline__ Col col(const Params& p, int c, int N, bool first_slice) {
    return bias_pair(first_slice ? p.bias : nullptr, c, N);
  }
  static __device__ __forceinline__ uint32_t pair(const Params&, const Rows&, Col b, int, float x0, float x1) {
    return pack_bf16(x0 + b.x, x1 + b.y);
  }
  static __device__ __forceinline__ void issue(const Params& p, const void* box, int n, int m0) {
    tma_reduce_add_2d(&p.out_map, box, n, m0);
  }
};

// fp8 linear layers (include/sgpt_b200.h): the e4m3 accumulator is dequantized as v = (acc * x_scale[m]) * w_scale[n],
// in this order, and handed to the bf16 path's Op unchanged.  Scales of rows / columns beyond M / N are read from the
// last valid entry (their outputs are clipped by the tensor map).
template <class Op>
struct OpDequantE4M3 {
  struct Params {
    typename Op::Params op;
    const float* x_scale;  // [M] per token
    const float* w_scale;  // [N] per output channel
  };
  struct Rows {
    typename Op::Rows op;
    float s[4];
  };
  struct Col {
    typename Op::Col op;
    float2 s;
  };
  static __device__ __forceinline__ void rows(const Params& p, Rows& rw, int r0, int M) {
    Op::rows(p.op, rw.op, r0, M);
#pragma unroll
    for (int ri = 0; ri < 4; ++ri) {
      const int row = r0 + 8 * (ri & 1) + 64 * (ri >> 1);
      rw.s[ri] = __ldg(p.x_scale + (row < M ? row : M - 1));
    }
  }
  static __device__ __forceinline__ Col col(const Params& p, int c, int N, bool first_slice) {
    Col cl;
    cl.op = Op::col(p.op, c, N, first_slice);
    cl.s = make_float2(__ldg(p.w_scale + (c < N ? c : N - 1)), __ldg(p.w_scale + (c + 1 < N ? c + 1 : N - 1)));
    return cl;
  }
  static __device__ __forceinline__ uint32_t pair(const Params& p, const Rows& rw, const Col& cl, int ri, float x0,
                                                  float x1) {
    return Op::pair(p.op, rw.op, cl.op, ri, __fmul_rn(__fmul_rn(x0, rw.s[ri]), cl.s.x),
                    __fmul_rn(__fmul_rn(x1, rw.s[ri]), cl.s.y));
  }
  static __device__ __forceinline__ void issue(const Params& p, const void* box, int n, int m0) {
    Op::issue(p.op, box, n, m0);
  }
};

// ---------------------------------------------------------------------------------------------------------------
// Staged epilogue driver: accumulator -> registers (thread = row) -> smem slab -> (lane = column pair) -> Op::rows()
// The slab is [32 rows][32 column pairs] of float2 without padding; pair p of row r is stored at p ^ (r & 15), which
// makes both the row-wise writes and the column-wise reads bank-conflict free for 8-byte accesses.
// ---------------------------------------------------------------------------------------------------------------
struct EpiNoState {};

template <class Op>
struct EpiStaged {
  using Params = typename Op::Params;
  using State = EpiNoState;
  static constexpr int kEpiWarps = 4;
  static constexpr int kStagingBytes = kEpiWarps * 32 * 256;  // one [32 x 32] float2 slab per epilogue warp
  static __device__ __forceinline__ void init(State&, const Params&) {}
  template <int BN, int kSlabBytes>
  static __device__ __forceinline__ void pre_tile(State&, const Params&, int, int, int, float*, int, int) {}
  static __device__ __forceinline__ void finish(State&, const Params&, int) {}

  template <int BN, int kSlabBytes>
  static __device__ __forceinline__ void tile(State&, const Params& p, int m0, int n0, int lane, uint32_t trow,
                                              float* slab_ptr, int M, int N) {
    const int rows = min(32, M - m0);  // warp-uniform; <= 0 when the whole slab is out of range
    const uint32_t slab = smem_u32(slab_ptr);
#pragma unroll 1
    for (int c = 0; c < BN; c += 64) {
      const int n = n0 + c;
      if (n >= N) break;  // warp-uniform
      uint32_t v0[32], v1[32];
      acc_ld_32(trow + 4 * c, v0);
      if (n + 32 < N) {
        acc_ld_32(trow + 4 * (c + 32), v1);
      } else {
#pragma unroll
        for (int i = 0; i < 32; ++i) v1[i] = 0u;
      }
      __syncwarp();  // the previous slab's readers are done
      const uint32_t wrow = slab + lane * 256u;
      const uint32_t sw = lane & 15;
#pragma unroll
      for (int i = 0; i < 16; ++i) sts_v2(wrow + ((i ^ sw) << 3), v0[2 * i], v0[2 * i + 1]);
#pragma unroll
      for (int i = 0; i < 16; ++i) sts_v2(wrow + (((16 + i) ^ sw) << 3), v1[2 * i], v1[2 * i + 1]);
      __syncwarp();
      if (rows > 0) Op::rows(p, slab, m0, rows, n + 2 * lane, N, lane);
    }
  }
};

// columns (2*lane, 2*lane+1) of staged row r
__device__ __forceinline__ float2 slab_read(uint32_t slab, int r, int lane) {
  return lds_v2(slab + r * 256u + ((lane ^ (r & 15)) << 3));
}

// Document mask of the masked searches (include/sgpt_b200.h): bit j % 32 of word j / 32 of a query's bitmap set = local
// document j allowed; pitch 0 = one bitmap for every query, else query q's bitmap starts at word q * pitch.
__device__ __forceinline__ const uint32_t* mask_row(const uint32_t* mask, long long pitch, int q) {
  return mask + static_cast<long long>(q) * pitch;
}

// Bits of a masked score (a NaN with the sign bit): score_key maps them to the invalid key 0, so the selection kernels
// (topk.cu) treat the document as absent, exactly like an empty slot.
constexpr uint32_t kMaskedScoreBits = 0xffffffffu;

// Score of a parked accumulator v with the query term r and the document term c.  bf16 / int8 operands: v * r * c (the
// scales, in this order).  kB1 (binary shards): v = 4 a + D, r = -2 popc(q), c = -2 popc(d) and the score is
// (v + r) + c = D - 2 hamming(q, d), every step an exact fp32 integer.
template <bool kB1>
__device__ __forceinline__ float epi_score(float v, float r, float c) {
  if constexpr (kB1) return (v + r) + c;
  else return v * r * c;
}
// kB1: the int32 popcount p read through a scale pointer -> the term -2 p
__device__ __forceinline__ float b1_term(float bits) { return __int2float_rn(-2 * __float_as_int(bits)); }

// scores_f32[q, doc] = fixnan(acc * row_scale[q] * col_scale[doc])       (cos_sim / dot_score, NaN -> -1)
// kMasked: masked documents get kMaskedScoreBits instead (the dense plan of the masked search).
// kB1: row_scale / col_scale hold int32 popcounts and the score is epi_score<true> (binary shards).
// !kFixNaN: a NaN is stored as it is (the LM-head logits, whose NaN must reach the log-softmax).
template <bool kMasked, bool kB1 = false, bool kFixNaN = true>
struct OpScoresF32T {
  struct Params {
    float* out;
    const float* row_scale;  // per query  (1/||q|| for cos_sim; null = 1)
    const float* col_scale;  // per doc    (1/||d|| for cos_sim; null = 1)
    long long ldc;
    const uint32_t* mask;    // kMasked: document bitmaps
    long long mask_pitch;    // kMasked: words between consecutive queries' bitmaps (0 = shared)
  };
  static __device__ __forceinline__ void rows(const Params& p, uint32_t slab, int m0, int rows, int col, int N,
                                              int lane) {
    const bool ok0 = col < N, ok1 = col + 1 < N;
    float c0 = 1.f, c1 = 1.f;
    if (p.col_scale) {
      if (ok0) c0 = __ldg(p.col_scale + col);
      if (ok1) c1 = __ldg(p.col_scale + col + 1);
    }
    if constexpr (kB1) {
      c0 = b1_term(c0);
      c1 = b1_term(c1);
    }
    const bool vec = ok1 && ((p.ldc & 1) == 0);
    float* dst = p.out + static_cast<size_t>(m0) * p.ldc + col;
    float my_rs = 1.f;  // lane r keeps row m0 + r's scale; broadcast per row with a shuffle
    if (p.row_scale && lane < rows) my_rs = __ldg(p.row_scale + m0 + lane);
    if constexpr (kB1) my_rs = b1_term(my_rs);
    // (col is even: both columns of the lane sit in one mask word)
    const uint32_t shared_word = (kMasked && p.mask_pitch == 0 && ok0) ? __ldg(p.mask + (col >> 5)) : 0u;
    auto masked = [&](int row, float& x, float& y) {
      if constexpr (kMasked) {
        const uint32_t w = p.mask_pitch == 0 ? shared_word
                                             : (ok0 ? __ldg(mask_row(p.mask, p.mask_pitch, row) + (col >> 5)) : 0u);
        if (!((w >> (col & 31)) & 1u)) x = __uint_as_float(kMaskedScoreBits);
        if (!((w >> ((col + 1) & 31)) & 1u)) y = __uint_as_float(kMaskedScoreBits);
      }
    };
    int r = 0;
    for (; r + 8 <= rows; r += 8) {
      float2 a[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) a[u] = slab_read(slab, r + u, lane);
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const float rs = __shfl_sync(0xffffffffu, my_rs, r + u);
        float x = epi_score<kB1>(a[u].x, rs, c0), y = epi_score<kB1>(a[u].y, rs, c1);
        if constexpr (kFixNaN) {
          x = (x != x) ? -1.f : x;
          y = (y != y) ? -1.f : y;
        }
        masked(m0 + r + u, x, y);
        if (vec) *reinterpret_cast<float2*>(dst) = make_float2(x, y);
        else {
          if (ok0) dst[0] = x;
          if (ok1) dst[1] = y;
        }
        dst += p.ldc;
      }
    }
    for (; r < rows; ++r) {
      const float rs = __shfl_sync(0xffffffffu, my_rs, r);
      const float2 a = slab_read(slab, r, lane);
      float x = epi_score<kB1>(a.x, rs, c0), y = epi_score<kB1>(a.y, rs, c1);
      if constexpr (kFixNaN) {
        x = (x != x) ? -1.f : x;
        y = (y != y) ? -1.f : y;
      }
      masked(m0 + r, x, y);
      if (vec) *reinterpret_cast<float2*>(dst) = make_float2(x, y);
      else {
        if (ok0) dst[0] = x;
        if (ok1) dst[1] = y;
      }
      dst += p.ldc;
    }
  }
};

// Threshold filter of the fused search (search.cu): score = fixnan(acc * row_scale[q] * col_scale[doc]); every score
// >= tau[q] is appended as a packed (score bits, local doc index) pair to a candidate list; the score matrix itself is
// never written to HBM.
//
// In the accumulator's native layout thread r of a warp owns query row r, i.e. ONE admission threshold: the compare
// needs no transpose, no shuffles and no ballots.  Each (CTA, column-half) pair is a GROUP with a PRIVATE list per query
// (cand[q][group][L]); the thread keeps its list length in a register across all tiles of the persistent kernel and
// writes it out once at the end, so there are NO atomics at all.  (The first version reserved space in one list per
// query with an atomicAdd per 32-document chunk: ~17 k same-address atomics per counter per search serialised in the
// L2 and, not the HBM stream, set the kernel's duration.)  L is sized for the worst case (every score of every tile the
// CTA visits admitted), so there is no overflow path; only the touched prefix of each list generates memory traffic.
// 8 epilogue warps (two per 32-row slab, half the tile's documents each); no staging memory.
//
// Sample mode (Params::pool != nullptr; pass A of the search): nothing is filtered; the thread writes the MAXIMUM of
// every 4 consecutive documents' scores (32 floats per query and tile half) to pool[q][group][Lp].  Each maximum is the
// score of a distinct real document, so the k-th largest of a query's maxima is a valid lower bound of its final k-th
// best score — at a quarter of the entries (and no document indices) the full sample would need.  Slots this thread never
// fills are written as 0xffffffff (maps to the invalid key 0 of the selection kernels).
//
// kMasked (the masked searches): only documents whose bit is set in the query's bitmap (Params::mask) are admitted, and
// a sample maximum is taken over those documents only; a 4-document block without any is an unused slot (0xffffffff),
// so every valid maximum is still the score of a distinct ALLOWED document and tau stays a lower bound of the k-th best
// allowed score (-inf, i.e. admit every allowed document, when the sample holds fewer than k maxima).  The four mask
// words of the warp's half tile are fetched in pre_tile with the document scales.  The unmasked instantiation compiles
// to the code it had before the mask existed.
//
// kB1 (binary shards): row_scale / col_scale hold int32 popcounts; pre_tile turns them into the terms -2 popc of the
// query and of the tile's documents (b1_term) where it stages the scales, and every score is epi_score<true>.  Masks,
// thresholds, sample maxima and lists act on that score exactly as on a scaled one.
struct FilterRowsParams {
  const float* row_scale;  // [M] or null
  const float* col_scale;  // [N] or null
  const float* tau;        // [M] per-query admission threshold; null -> admit everything
  const float* tau_hi;     // [M] upper threshold (>= tau) or null: scores >= tau_hi are appended at the FRONT of the list,
                           // scores in [tau, tau_hi) at its BACK (filled downwards from slot L - 1); null -> all front
  uint2* cand;             // [M][groups][L]
  int* counts;             // [groups][M] front entries
  int* counts_back;        // [groups][M] back entries (only with tau_hi)
  long long stride_q;      // entries between consecutive queries' list blocks
  int L;                   // entries per (query, group) list
  int group0;              // first group index this launch writes
  int nq;
  float* pool;             // sample mode: [M][groups][Lp] block maxima (cand / counts / tau unused)
  long long stride_p;      // floats between consecutive queries' blocks of `pool`
  int Lp;                  // floats per (query, group): 32 x tiles per CTA
  int pair;                // 1: launched with two CTAs per work unit (CL = 2: 256 queries per scan)
  const uint32_t* mask;    // kMasked: document bitmaps of the launch's queries
  long long mask_pitch;    // kMasked: words between consecutive queries' bitmaps (0 = one bitmap for all)
};

template <bool kMasked, bool kB1 = false>
struct EpiFilterRowsT {
  using Params = FilterRowsParams;
  struct State {
    int cnt;    // front entries (sample mode: maxima written)
    int cnt_b;  // back entries
    // per-tile constants fetched in pre_tile, i.e. BEFORE the wait for the accumulator: lane l holds the inverse norms of
    // documents n0 + 4 l .. + 3 of this warp's 128-document half tile (broadcast by shuffles below), the query's scale and
    // its admission threshold.  (Fetched inside the chunk loop, the norms cost one exposed HBM round trip per 32 documents
    // — 4 B per document that nobody else has touched — while the TMA stream saturates the memory system: ~4 serial
    // misses per tile per warp against a tile time of 9 us.)
    float4 cs;
    float rs, tau, tau_hi;
  };
  // kMasked: this query's mask words of documents n0 .. n0 + 127 (words past the shard's last document are never read:
  // bits at or past N are ignored)
  static __device__ __forceinline__ const uint32_t* mask_words(const Params& p, int q, int n0) {
    return mask_row(p.mask, p.mask_pitch, q) + (n0 >> 5);
  }
  static constexpr int kEpiWarps = 8;
  static constexpr int kStagingBytes = 1024;  // (none used)
  // one group per (work-unit slot, column half): with two CTAs per unit (Params::pair = 1: up to 256 queries per scan, CTA r
  // of the unit owns queries 128 r .. 128 r + 127 and all 256 documents of the tile) both CTAs write the SAME group's lists —
  // of different queries
  static __device__ __forceinline__ int group_of(const Params& p) {
    return p.group0 + static_cast<int>(blockIdx.x >> p.pair) * 2 + static_cast<int>(threadIdx.x >> 7);
  }
  static __device__ __forceinline__ void init(State& st, const Params&) { st.cnt = 0; st.cnt_b = 0; }
  template <int COLS, int kSlabBytes>
  static __device__ __forceinline__ void pre_tile(State& st, const Params& p, int m0, int n0, int lane, float*, int M, int N) {
    static_assert(COLS == 128, "one float4 of document scales per lane covers the warp's half tile");
    const int q = m0 + lane;
    const bool qok = q < M;
    st.rs = (qok && p.row_scale) ? __ldg(p.row_scale + q) : 1.f;
    st.tau = !qok ? INFINITY : (p.tau != nullptr ? __ldg(p.tau + q) : -INFINITY);  // +inf: rows beyond nq admit nothing
    st.tau_hi = (qok && p.tau_hi != nullptr) ? fmaxf(__ldg(p.tau_hi + q), st.tau) : st.tau;
    st.cs = make_float4(1.f, 1.f, 1.f, 1.f);
    if (p.col_scale != nullptr && m0 < M) {
      const int c = n0 + 4 * lane;
      if (c + 4 <= N) {
        st.cs = __ldg(reinterpret_cast<const float4*>(p.col_scale + c));
      } else if (N > 0) {
        st.cs.x = __ldg(p.col_scale + min(c, N - 1));
        st.cs.y = __ldg(p.col_scale + min(c + 1, N - 1));
        st.cs.z = __ldg(p.col_scale + min(c + 2, N - 1));
        st.cs.w = __ldg(p.col_scale + min(c + 3, N - 1));
      }
    }
    if constexpr (kB1) {
      st.rs = b1_term(st.rs);
      st.cs = make_float4(b1_term(st.cs.x), b1_term(st.cs.y), b1_term(st.cs.z), b1_term(st.cs.w));
    }
    if constexpr (kMasked) {
      // Only an L1 prefetch here: four words held in registers across the mainloop would push the 168-register kernel
      // into spills.  tile() loads them from L1 (the 16 bytes may straddle two lines when the pitch is not a multiple of 4)
      if (qok && n0 < N) {
        const uint32_t* w = mask_words(p, q, n0);
        const int last = min(3, (N - 1 - n0) >> 5);
        asm volatile("prefetch.global.L1 [%0];" ::"l"(w));
        asm volatile("prefetch.global.L1 [%0];" ::"l"(w + last));
      }
    }
  }
  static __device__ __forceinline__ void finish(State& st, const Params& p, int lane_row) {
    if (lane_row >= p.nq) return;
    if (p.pool != nullptr) {
      uint32_t* d = reinterpret_cast<uint32_t*>(p.pool + static_cast<long long>(lane_row) * p.stride_p +
                                               static_cast<long long>(group_of(p)) * p.Lp);
      for (int i = st.cnt; i < p.Lp; ++i) d[i] = 0xffffffffu;  // CTAs that visited fewer tiles than the longest
    } else {
      p.counts[static_cast<long long>(group_of(p)) * p.nq + lane_row] = st.cnt;  // cnt + cnt_b <= L by construction
      if (p.counts_back != nullptr) p.counts_back[static_cast<long long>(group_of(p)) * p.nq + lane_row] = st.cnt_b;
    }
  }

  template <int COLS, int kSlabBytes>
  static __device__ __forceinline__ void tile(State& st, const Params& p, int m0, int n0, int lane, uint32_t trow,
                                              float*, int M, int N) {
    if (m0 >= M) return;  // warp-uniform
    const int q = m0 + lane;
    const bool qok = q < M;
    const float rs = st.rs;
    const bool pooled = (p.pool != nullptr);
    const float tau = st.tau, tau_hi = st.tau_hi;
    // warp-uniform; a b1 score is an integer, never NaN
    const bool nan_path = !kB1 && __any_sync(0xffffffffu, !pooled && tau <= -1.0f) != 0;
    const float csv[4] = {st.cs.x, st.cs.y, st.cs.z, st.cs.w};
    uint2* dst = p.cand + static_cast<long long>(qok ? q : 0) * p.stride_q + static_cast<long long>(group_of(p)) * p.L;
    int cnt = st.cnt, cnt_b = st.cnt_b;
    uint32_t mw[4] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};  // bit i of mw[j]: document n0 + 32 j + i allowed
    if constexpr (kMasked) {
      const uint32_t* w = mask_words(p, qok ? q : 0, n0);
#pragma unroll
      for (int j = 0; j < 4; ++j) mw[j] = (qok && n0 + 32 * j < N) ? __ldg(w + j) : 0u;
    }
#pragma unroll 1
    for (int c = 0; c < COLS; c += 32) {
      const int n = n0 + c;
      if (n >= N) break;  // warp-uniform
      uint32_t v[32];
      acc_ld_32(trow + 4 * c, v);
      const bool full = (n + 32 <= N);
      // bit i: document n + i may be admitted (selects instead of mw[c >> 5]: a dynamic index would put mw in local memory)
      const uint32_t allow = c == 0 ? mw[0] : c == 32 ? mw[1] : c == 64 ? mw[2] : mw[3];
      // scale of column c + i: component i % 4 of lane (c + i) / 4 (all lanes take part: the loop is warp-uniform)
      float cs[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) cs[i] = __shfl_sync(0xffffffffu, csv[i & 3], (c >> 2) + (i >> 2));
      // XS:99 maps a NaN score to -1.  While tau > -1 (always, except for degenerate corpora) a NaN fails `x >= tau` exactly
      // as its image -1 would, and in sample mode fmaxf drops it (a smaller maximum keeps tau a valid lower bound): the
      // explicit mapping (two instructions per score) is only executed when some row of the warp could admit a -1.
      float x[32];
      if (nan_path) {
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const float s = epi_score<kB1>(__uint_as_float(v[i]), rs, cs[i]);
          x[i] = (s != s) ? -1.f : s;
        }
      } else {
#pragma unroll
        for (int i = 0; i < 32; ++i) x[i] = epi_score<kB1>(__uint_as_float(v[i]), rs, cs[i]);
      }
      if (pooled) {
        // sample pass: maxima of 4 consecutive documents, two 16-byte stores (cnt is a multiple of 8, the lists 32-byte
        // aligned); documents beyond the shard never win
        float m[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float mx = -INFINITY;
          bool any = false;
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const bool ok = (full || n + 4 * j + u < N) && (!kMasked || ((allow >> (4 * j + u)) & 1u));
            mx = ok ? fmaxf(mx, x[4 * j + u]) : mx;
            any = any || ok;
          }
          if constexpr (kMasked) mx = any ? mx : __uint_as_float(kMaskedScoreBits);  // no allowed document: unused slot
          m[j] = mx;
        }
        if (qok && cnt + 8 <= p.Lp) {
          float4* d4 = reinterpret_cast<float4*>(p.pool + static_cast<long long>(q) * p.stride_p +
                                                 static_cast<long long>(group_of(p)) * p.Lp + cnt);
          d4[0] = make_float4(m[0], m[1], m[2], m[3]);
          d4[1] = make_float4(m[4], m[5], m[6], m[7]);
        }
        cnt += 8;
      } else {
        // Branch-free admission: one predicated 8-byte store per score, the two list lengths advance by predicates.  (With
        // a branch per score — taken by SOME lane for ~60 % of the scores at a 3 % admission rate — the 32 convergence
        // regions per chunk were the longest dependent chain of the epilogue.)  cnt + cnt_b never exceeds L: L is every
        // score of every tile this CTA visits (checked by the launcher).
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          // tau = +inf for rows beyond the query count
          const bool pass = (full || n + i < N) && x[i] >= tau && (!kMasked || ((allow >> i) & 1u));
          const bool hi = x[i] >= tau_hi;
          const uint32_t slot = static_cast<uint32_t>(hi ? cnt : (p.L - 1 - cnt_b));  // unsigned: one IMAD.WIDE.U32 per address
          // (a predicated store in PTX: as plain C++ the compiler wraps the store and its address arithmetic in a branch)
          asm volatile(
              "{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %0, 0;\n\t@p st.global.v2.u32 [%1], {%2, %3};\n\t}\n" ::"r"(
                  static_cast<uint32_t>(pass)),
              "l"(dst + slot), "r"(__float_as_uint(x[i])), "r"(static_cast<uint32_t>(n + i))
              : "memory");
          cnt += (pass && hi) ? 1 : 0;
          cnt_b += (pass && !hi) ? 1 : 0;
        }
      }
    }
    st.cnt = cnt;
    st.cnt_b = cnt_b;
  }
};
using EpiFilterRows = EpiFilterRowsT<false>;
using EpiFilterRowsMasked = EpiFilterRowsT<true>;
using EpiFilterRowsB1 = EpiFilterRowsT<false, true>;
using EpiFilterRowsB1Masked = EpiFilterRowsT<true, true>;

// Grouped scan of the IVF search (ivf.cu), run with kUnits: A row r is one (query, probe) pair of the query block, all
// rows of a unit probe the same list, and the unit's columns are one 256-document tile of that list (the unit's M / N
// bounds are the end of its pair block and of the list).  Thread = pair row, as in EpiFilterRows, with the same score
// arithmetic — fixnan(acc * row_scale * col_scale) on the accumulator of the same mainloop — so every score has the bits
// the exact search computes for that document.  Nothing is filtered: the thread writes (score bits, int32 global id) of
// every document of the tile to its pair's candidate list, slot = position - first position of the list, so after all
// tiles of the list the slots 0 .. len - 1 of the list are filled.  A position the shared bitmap excludes (deletions) is
// written as an empty slot, id -1.  Slots are written two per 16-byte store (slot 0 is 16-byte aligned: Ls is even).
// Params: gemm_api.h IvfRowsParams.
//
// kPerQuery (sgpt_ivf_search_masked with a pitch): every pair row reads its own query's bitmap (query = row_info.x /
// nprobe inside the block) instead of the shared one.  List starts are not multiples of 32, so the row's 32 positions
// n .. n + 31 of a chunk straddle two mask words: both are loaded and the row's 32 bits taken with a funnel shift; a
// position whose bit is 0 becomes an empty slot, as a deletion does.  pre_tile only prefetches the row's words into L1
// (words held in registers across the mainloop would spill it).  The shared instantiation compiles to the code it had
// before the per-query mask existed.
template <bool kPerQuery>
struct EpiIvfRowsT {
  using Params = typename std::conditional<kPerQuery, IvfRowsMaskedParams, IvfRowsParams>::type;
  struct State {
    float4 cs;  // document scales n0 + 4 lane .. + 3 of the warp's half tile (broadcast by shuffles)
    float rs;   // this row's query scale
    int list;   // this row's candidate list
    int begin;  // first position of the probed list
  };
  static constexpr int kEpiWarps = 8;
  static constexpr int kStagingBytes = 1024;  // (none used)
  static __device__ __forceinline__ void init(State&, const Params&) {}
  static __device__ __forceinline__ void finish(State&, const Params&, int) {}
  template <int COLS, int kSlabBytes>
  static __device__ __forceinline__ void pre_tile(State& st, const Params& p, int m0, int n0, int lane, float*, int M, int N) {
    static_assert(COLS == 128, "one float4 of document scales per lane covers the warp's half tile");
    const int r = m0 + lane;
    const bool rok = r < M;
    st.rs = rok ? __ldg(p.row_scale + r) : 1.f;
    const int2 info = rok ? __ldg(p.row_info + r) : make_int2(0, 0);
    st.list = info.x;
    st.begin = info.y;
    st.cs = make_float4(1.f, 1.f, 1.f, 1.f);
    if (m0 >= M || n0 >= N) return;  // warp-uniform: tile() writes nothing
    const int c = n0 + 4 * lane;
    if (p.col_scale != nullptr) {
      st.cs.x = __ldg(p.col_scale + min(c, N - 1));
      st.cs.y = __ldg(p.col_scale + min(c + 1, N - 1));
      st.cs.z = __ldg(p.col_scale + min(c + 2, N - 1));
      st.cs.w = __ldg(p.col_scale + min(c + 3, N - 1));
    }
    // the ids (and mask words) tile() reads once the accumulator is ready
    if (c < N) asm volatile("prefetch.global.L1 [%0];" ::"l"(p.doc_ids + c));
    if constexpr (kPerQuery) {
      if (rok) {  // the row's words of positions n0 .. min(n0 + 128, N) - 1 (at most 5 words, at most two L1 lines)
        const uint32_t* w = p.mask + static_cast<long long>(info.x / p.nprobe) * p.mask_pitch;
        asm volatile("prefetch.global.L1 [%0];" ::"l"(w + (n0 >> 5)));
        asm volatile("prefetch.global.L1 [%0];" ::"l"(w + ((min(n0 + COLS, N) - 1) >> 5)));
      }
    } else if (p.mask != nullptr && lane < 4 && n0 + 32 * lane < N) {
      asm volatile("prefetch.global.L1 [%0];" ::"l"(p.mask + ((n0 + 32 * lane) >> 5)));
    }
  }

  template <int COLS, int kSlabBytes>
  static __device__ __forceinline__ void tile(State& st, const Params& p, int m0, int n0, int lane, uint32_t trow,
                                              float*, int M, int N) {
    if (m0 >= M) return;  // warp-uniform
    const bool rok = m0 + lane < M;
    const float rs = st.rs;
    const float csv[4] = {st.cs.x, st.cs.y, st.cs.z, st.cs.w};
    // dst[pos] = the slot of position pos in this row's list
    uint2* dst = p.cand + static_cast<long long>(rok ? st.list : 0) * p.Ls - st.begin;
    const uint32_t* qmask = nullptr;  // kPerQuery: this row's query's bitmap
    if constexpr (kPerQuery) qmask = p.mask + static_cast<long long>(rok ? st.list / p.nprobe : 0) * p.mask_pitch;
#pragma unroll 1
    for (int c = 0; c < COLS; c += 32) {
      const int n = n0 + c;
      if (n >= N) break;  // warp-uniform
      uint32_t v[32];
      acc_ld_32(trow + 4 * c, v);
      // lane i: global id of position n + i (-1 when excluded or past the list)
      const int pos = n + lane;
      int gid = -1;
      if (pos < N) {
        gid = __ldg(p.doc_ids + pos);
        if (!kPerQuery && p.mask != nullptr && !((__ldg(p.mask + (pos >> 5)) >> (pos & 31)) & 1u)) gid = -1;
      }
      // kPerQuery: bit i = position n + i allowed for this row's query.  n < N <= the corpus size, so word n / 32 exists;
      // the next word is read only when it holds a position below N
      uint32_t allow = 0xffffffffu;
      if constexpr (kPerQuery) {
        const int w = n >> 5, s = n & 31;
        const uint32_t lo = rok ? __ldg(qmask + w) : 0u;
        const uint32_t hi = (rok && s != 0 && (w + 1) * 32 < N) ? __ldg(qmask + w + 1) : 0u;
        allow = __funnelshift_r(lo, hi, s);
      }
      float cs[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) cs[i] = __shfl_sync(0xffffffffu, csv[i & 3], (c >> 2) + (i >> 2));
      const bool full = n + 32 <= N;
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        float x0 = __uint_as_float(v[i]) * rs * cs[i];
        float x1 = __uint_as_float(v[i + 1]) * rs * cs[i + 1];
        x0 = (x0 != x0) ? -1.f : x0;
        x1 = (x1 != x1) ? -1.f : x1;
        int g0 = __shfl_sync(0xffffffffu, gid, i), g1 = __shfl_sync(0xffffffffu, gid, i + 1);
        if constexpr (kPerQuery) {
          g0 = ((allow >> i) & 1u) ? g0 : -1;
          g1 = ((allow >> (i + 1)) & 1u) ? g1 : -1;
        }
        if (!rok) continue;
        if (full || n + i + 1 < N) {
          *reinterpret_cast<uint4*>(dst + n + i) =
              make_uint4(__float_as_uint(x0), static_cast<uint32_t>(g0), __float_as_uint(x1), static_cast<uint32_t>(g1));
        } else if (n + i < N) {
          dst[n + i] = make_uint2(__float_as_uint(x0), static_cast<uint32_t>(g0));
        }
      }
    }
  }
};
using EpiIvfRows = EpiIvfRowsT<false>;
using EpiIvfRowsMasked = EpiIvfRowsT<true>;


// Profiling aid of gemm_bf16_tn_kernel (sgpt_linear epilogue code 101: kLoad): the mainloop and the accumulator hand-over
// with no epilogue work at all, or with the accumulator loads only.
template <bool kLoad>
struct EpiDebugNull {
  struct Params { int dummy; };
  using State = EpiNoState;
  static constexpr int kEpiWarps = 4;
  static constexpr int kStagingBytes = EpiStaged<OpScoresF32T<false>>::kStagingBytes;  // (none used)
  static __device__ __forceinline__ void init(State&, const Params&) {}
  template <int BN, int kSlabBytes>
  static __device__ __forceinline__ void pre_tile(State&, const Params&, int, int, int, float*, int, int) {}
  static __device__ __forceinline__ void finish(State&, const Params&, int) {}
  template <int BN, int kSlabBytes>
  static __device__ __forceinline__ void tile(State&, const Params&, int, int, int, uint32_t trow, float*, int, int) {
    if (kLoad) {
      uint32_t acc = 0;
#pragma unroll 1
      for (int c = 0; c < BN; c += 32) {
        uint32_t v[32];
        acc_ld_32(trow + 4 * c, v);
#pragma unroll
        for (int i = 0; i < 32; ++i) acc ^= v[i];
      }
      asm volatile("" ::"r"(acc));  // keep the loads alive (no call: it would serialise the wgmma pipeline)
    }
  }
};
using EpiScoresF32 = EpiStaged<OpScoresF32T<false>>;
using EpiScoresF32Masked = EpiStaged<OpScoresF32T<true>>;
using EpiScoresB1 = EpiStaged<OpScoresF32T<false, true>>;
using EpiScoresB1Masked = EpiStaged<OpScoresF32T<true, true>>;
using EpiLogitsF32 = EpiStaged<OpScoresF32T<false, false, false>>;  // LM-head logits: acc stored unchanged, NaN kept

}  // namespace sgpt
