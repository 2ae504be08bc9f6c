// Host-side helpers shared by the C-ABI entry points: error reporting, launch counting, tensor-map encoding.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <utility>

#include "../../include/b200vit.h"

namespace b200 {

void set_error(const char* fmt, ...);
extern std::atomic<int64_t> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define B200_CHECK_ARG(cond, ...)        \
  do {                                   \
    if (!(cond)) {                       \
      b200::set_error(__VA_ARGS__);      \
      return B200VIT_ERR_INVALID;        \
    }                                    \
  } while (0)

#define B200_CHECK_CUDA(expr)                                                                     \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      b200::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return B200VIT_ERR_CUDA;                                                                    \
    }                                                                                             \
  } while (0)

// cuTensorMapEncodeTiled resolved through the runtime (libcuda is only a stub at build time).
// Encodes a rank-`rank` bf16 tensor map with 128B swizzle.  dims/box innermost first; strides in BYTES for dims 1..
int encode_tmap_bf16(CUtensorMap* tm, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                     const uint32_t* box, bool swizzle128 = true);
// same, with the swizzle width in bytes (0 = none, 32, 64, 128)
int encode_tmap_bf16_sw(CUtensorMap* tm, const void* base, int rank, const uint64_t* dims,
                        const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes);
int encode_tmap_f32(CUtensorMap* tm, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, bool swizzle128 = false);

void tmap_cache_stats(int64_t* hits, int64_t* misses);

// The head widths (dim_head) the attention, head-norm and pooling kernels are built for.
inline bool head_width_ok(int dh) { return dh == 32 || dh == 64 || dh == 80 || dh == 128; }

// The persistent fixed-length attention kernel (attention_short.cu): the lengths and head widths it is built for, and
// its launch.  Same bits as the tiled kernel of attention.cu; b200vit_attention_ex chooses between them.
bool attention_short_ok(int N, int dh);
int attention_short(const void* qkv, void* out, int B, int N, int H, int dh, float scale_log2e, cudaStream_t stream);

// test hooks 12 and 14 (gemm.cu)
void gemm_set_block_n(int v);
void gemm_set_direct_store(int v);

// SM count of the CURRENT device (cached per device).
int num_sms();
// B200VIT_PDL=0 in the environment turns programmatic dependent launch off (A/B measurements); default on.
bool pdl_enabled();
// Launch through cudaLaunchKernelEx; `pdl` adds the programmaticStreamSerialization attribute (only for kernels that
// call pdl_wait() before touching global memory, see common.cuh).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                 bool pdl, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = (pdl && pdl_enabled()) ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device): the attribute is per device, so a flag
// that is static per process would leave the second GPU of a process without it.  Returns 0 / B200VIT_ERR_CUDA.
int ensure_dyn_smem(const void* kernel, size_t bytes);
#define B200_ENSURE_SMEM(kern, bytes)                                                       \
  do {                                                                                      \
    int _rc = b200::ensure_dyn_smem(reinterpret_cast<const void*>(kern), (size_t)(bytes));  \
    if (_rc) return _rc;                                                                    \
  } while (0)

}  // namespace b200
