// Host-side helpers: error plumbing for the C ABI and TMA tensor-map construction (driver entry point resolved
// at run time through the CUDA runtime, so the library never links libcuda directly).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace sgpt {

// thread-local last-error message, returned by sgpt_last_error()
void set_error(const char* fmt, ...);
const char* get_error();

#define SGPT_CHECK_CUDA(expr)                                                               \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess) {                                                                \
      ::sgpt::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return SGPT_ERR_CUDA;                                                                 \
    }                                                                                       \
  } while (0)

#define SGPT_REQUIRE(cond, ...)        \
  do {                                 \
    if (!(cond)) {                     \
      ::sgpt::set_error(__VA_ARGS__);  \
      return SGPT_ERR_INVALID;         \
    }                                  \
  } while (0)

// 2-D bf16 row-major tensor [rows, cols] with row pitch `ld` elements; box = [box_rows, box_cols] with the
// 128-byte swizzle (box_cols must be 64 bf16 = 128 B).  Returns 0 on success.
int make_tma_2d_bf16(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                     uint32_t box_rows, uint32_t box_cols);
// Same for int8 elements (box_cols = 128 bytes); out-of-bounds elements of a box read as zero, which covers the K tail.
int make_tma_2d_u8(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                   uint32_t box_cols);

int sm_count();  // multiprocessors of the CURRENT device (cached per device)

// "Do this once per device": kernel attributes such as cudaFuncAttributeMaxDynamicSharedMemorySize are per device, so a
// process that drives several GPUs (one Encoder / CorpusShard per device) must opt in on each of them.
//   static PerDeviceOnce once;  if (once.first()) cudaFuncSetAttribute(...);
struct PerDeviceOnce {
  bool first();            // true exactly once per CUDA device (current device), thread-safe
  unsigned char done_[64] = {};
};

// Programmatic dependent launch is on unless SGPT_PDL=0 is set in the environment (A/B measurements).
bool pdl_enabled();

// Launch with the programmatic-stream-serialization attribute (common.cuh: pdl_wait / pdl_launch_dependents) and, for
// cluster > 1, in thread-block clusters of `cluster` CTAs along x.
template <class... KArgs, class... Args>
inline cudaError_t launch_kernel_cluster(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                         cudaStream_t stream, int cluster, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  cfg.attrs = attr;
  cfg.numAttrs = 0;
  if (pdl_enabled()) {
    attr[cfg.numAttrs].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[cfg.numAttrs].val.programmaticStreamSerializationAllowed = 1;
    ++cfg.numAttrs;
  }
  if (cluster > 1) {
    attr[cfg.numAttrs].id = cudaLaunchAttributeClusterDimension;
    attr[cfg.numAttrs].val.clusterDim.x = static_cast<unsigned>(cluster);
    attr[cfg.numAttrs].val.clusterDim.y = 1;
    attr[cfg.numAttrs].val.clusterDim.z = 1;
    ++cfg.numAttrs;
  }
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

template <class... KArgs, class... Args>
inline cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                 Args&&... args) {
  return launch_kernel_cluster(kern, grid, block, smem, stream, 1, static_cast<Args&&>(args)...);
}

}  // namespace sgpt

// ---------------------------------------------------------------------------------------------------------------
// Launch accounting (always on) and optional per-category CUDA-event timing (sgpt_profile_*).
// ---------------------------------------------------------------------------------------------------------------
namespace sgpt {
enum LaunchCat { kCatEmbed = 0, kCatLayerNorm, kCatGemm, kCatAttention, kCatPool, kCatScores, kCatTopk, kCatMisc, kNumCats };

struct LaunchScope {
  LaunchScope(int cat, cudaStream_t stream);
  ~LaunchScope();
  int cat_;
  cudaStream_t stream_;
  int slot_;
};
}  // namespace sgpt
