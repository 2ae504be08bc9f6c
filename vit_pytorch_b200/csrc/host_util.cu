#include "host_util.h"

#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <unordered_map>
#include <utility>

namespace b200 {

static thread_local char g_err[512] = "";
std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// Descriptor cache: a forward re-encodes the same (pointer, shape, box) maps every call -- weights
// never move and the caching allocator hands the same activation buffers back -- so the 128-byte descriptors are
// kept per key.  The descriptor depends on nothing but the key, so a stale entry cannot exist; the table is simply
// emptied when it grows past kTmapCacheMax entries.
struct TmapKey {
  uint64_t base;
  uint64_t dims[5];
  uint64_t strides[4];
  uint32_t box[5];
  int32_t rank, dt, sw;
  bool operator==(const TmapKey& o) const { return memcmp(this, &o, sizeof(TmapKey)) == 0; }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    const uint64_t* w = reinterpret_cast<const uint64_t*>(&k);
    uint64_t h = 1469598103934665603ull;
    for (size_t i = 0; i < sizeof(TmapKey) / 8; ++i) h = (h ^ w[i]) * 1099511628211ull;
    return (size_t)h;
  }
};
static_assert(sizeof(TmapKey) % 8 == 0, "TmapKey is hashed as 64-bit words");
constexpr size_t kTmapCacheMax = 4096;
static std::mutex g_tmap_mu;
static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> g_tmap_cache;
static std::atomic<int64_t> g_tmap_hits{0}, g_tmap_misses{0};

static int encode_uncached(CUtensorMap* tm, CUtensorMapDataType dt, const void* base, int rank, const uint64_t* dims,
                           const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle sw);

static int encode_generic(CUtensorMap* tm, CUtensorMapDataType dt, const void* base, int rank, const uint64_t* dims,
                          const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle sw) {
  TmapKey k;
  memset(&k, 0, sizeof(k));
  k.base = reinterpret_cast<uint64_t>(base);
  k.rank = rank; k.dt = (int32_t)dt; k.sw = (int32_t)sw;
  for (int i = 0; i < rank; ++i) {
    k.dims[i] = dims[i];
    k.box[i] = box[i];
    if (i > 0) k.strides[i - 1] = strides_bytes[i - 1];
  }
  {
    std::lock_guard<std::mutex> lock(g_tmap_mu);
    auto it = g_tmap_cache.find(k);
    if (it != g_tmap_cache.end()) {
      *tm = it->second;
      g_tmap_hits.fetch_add(1, std::memory_order_relaxed);
      return 0;
    }
  }
  int rc = encode_uncached(tm, dt, base, rank, dims, strides_bytes, box, sw);
  if (rc) return rc;
  g_tmap_misses.fetch_add(1, std::memory_order_relaxed);
  std::lock_guard<std::mutex> lock(g_tmap_mu);
  if (g_tmap_cache.size() >= kTmapCacheMax) g_tmap_cache.clear();
  g_tmap_cache.emplace(k, *tm);
  return 0;
}

void tmap_cache_stats(int64_t* hits, int64_t* misses) {
  *hits = g_tmap_hits.load();
  *misses = g_tmap_misses.load();
}

static int encode_uncached(CUtensorMap* tm, CUtensorMapDataType dt, const void* base, int rank, const uint64_t* dims,
                           const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle sw) {
  EncodeTiledFn fn = get_encode();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled could not be resolved (driver too old?)");
    return B200VIT_ERR_CUDA;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i - 1];
  }
  CUresult r = fn(tm, dt, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d, dims %llu,%llu box %u,%u)", (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0], rank > 1 ? box[1] : 0);
    return B200VIT_ERR_CUDA;
  }
  return 0;
}

int encode_tmap_bf16(CUtensorMap* tm, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                     const uint32_t* box, bool swizzle128) {
  return encode_generic(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, rank, dims, strides_bytes, box,
                        swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE);
}
int encode_tmap_bf16_sw(CUtensorMap* tm, const void* base, int rank, const uint64_t* dims,
                        const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes) {
  const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                                      : CU_TENSOR_MAP_SWIZZLE_NONE;
  return encode_generic(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, rank, dims, strides_bytes, box, sw);
}
int encode_tmap_f32(CUtensorMap* tm, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, bool swizzle128) {
  return encode_generic(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, base, rank, dims, strides_bytes, box,
                        swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE);
}

constexpr int kMaxDevices = 64;

int num_sms() {
  static std::atomic<int> n[kMaxDevices];
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDevices) dev = 0;
  int v = n[dev].load(std::memory_order_relaxed);
  if (v == 0) {
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    n[dev].store(v, std::memory_order_relaxed);
  }
  return v;
}

bool pdl_enabled() {
  static const bool on = [] {
    const char* e = getenv("B200VIT_PDL");
    return !(e && e[0] == '0');
  }();
  return on;
}

int ensure_dyn_smem(const void* kernel, size_t bytes) {
  if (bytes <= 48 * 1024) return 0;
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, size_t> done;
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lock(mu);
  size_t& have = done[std::make_pair(kernel, dev)];
  if (have >= bytes) return 0;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) {
    set_error("cudaFuncSetAttribute(MaxDynamicSharedMemorySize=%zu) failed on device %d: %s", bytes, dev,
              cudaGetErrorString(e));
    return B200VIT_ERR_CUDA;
  }
  have = bytes;
  return 0;
}

}  // namespace b200

extern "C" {

const char* b200vit_last_error(void) { return b200::g_err; }
int b200vit_version(void) { return 300; }  /* sm_90a kernels */
int64_t b200vit_launch_count(void) { return b200::g_launches.load(); }
void b200vit_reset_launch_count(void) { b200::g_launches.store(0); }

int b200vit_device_ok(int dev) {
  cudaDeviceProp prop;
  cudaError_t e = cudaGetDeviceProperties(&prop, dev);
  if (e != cudaSuccess) {
    b200::set_error("cudaGetDeviceProperties(%d): %s", dev, cudaGetErrorString(e));
    return B200VIT_ERR_CUDA;
  }
  if (prop.major != 9 || prop.minor != 0) {
    b200::set_error("device %d is sm_%d%d; libb200vit contains sm_90a code only", dev, prop.major, prop.minor);
    return B200VIT_ERR_DEVICE;
  }
  if (!b200::get_encode()) {
    b200::set_error("cuTensorMapEncodeTiled could not be resolved");
    return B200VIT_ERR_CUDA;
  }
  return 0;
}

}  // extern "C"
