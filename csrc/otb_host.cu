// otter_b200 — host-side helpers: error channel, launch counter, TMA descriptor encoding.
#include "otb_host.h"

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <unordered_map>

namespace otb {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// libcuda is not linked: the driver entry point is resolved through the runtime at first use, so
// the library loads (and exports its symbols) on a machine without a GPU driver.
static EncodeTiledFn get_encode_fn() {
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

// ---- descriptor cache --------------------------------------------------------------------------------------
// A CUtensorMap is a pure function of (base, rows, cols, pitch, box, element type): identical keys always encode to
// identical 128 bytes, so a hit can never be stale.  The cache removes the driver call (~1 us each, 2-4 per launch)
// from eager-mode launches (generate(), the tests); it is guarded by a mutex because serving calls generate() from
// worker threads (SURVEY.md 8b threading row) and bounded so that long-running processes cannot grow it.
namespace {
struct TmapKey {
  uintptr_t base; uint64_t rows, cols, ld; uint32_t box_rows, box_cols, elt;
  bool operator==(const TmapKey& o) const {
    return base == o.base && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows &&
           box_cols == o.box_cols && elt == o.elt;
  }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    uint64_t h = k.base * 0x9E3779B97F4A7C15ull;
    h ^= (k.rows + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
    h ^= (k.cols + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
    h ^= (k.ld + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
    h ^= ((uint64_t(k.box_rows) << 34) | (uint64_t(k.box_cols) << 2) | k.elt) + (h << 6) + (h >> 2);
    return static_cast<size_t>(h);
  }
};
std::mutex g_tmap_mu;
std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> g_tmap_cache;
constexpr size_t kTmapCacheMax = 8192;
std::atomic<long long> g_tmap_hits{0}, g_tmap_misses{0};
}  // namespace

static int make_tmap_2d(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                        uint32_t box_rows, uint32_t box_cols, bool f32) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return set_error(OTB_ERR_CUDA, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  const uint32_t esz = f32 ? 4 : 2;
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return set_error(OTB_ERR_INVALID, "TMA base not 16B aligned");
  if ((ld * esz) % 16 != 0)
    return set_error(OTB_ERR_INVALID, "TMA row pitch %llu elements not a multiple of 16 bytes", (unsigned long long)ld);
  if (box_cols * esz != 128 || box_rows > 256) return set_error(OTB_ERR_INVALID, "bad TMA box");
  const TmapKey key{reinterpret_cast<uintptr_t>(base), rows, cols, ld, box_rows, box_cols, esz};
  {
    std::lock_guard<std::mutex> lk(g_tmap_mu);
    auto it = g_tmap_cache.find(key);
    if (it != g_tmap_cache.end()) {
      *map = it->second;
      g_tmap_hits.fetch_add(1, std::memory_order_relaxed);
      return OTB_OK;
    }
  }
  // The driver call needs a current context on this thread.  A thread that has made no runtime call yet (the autograd
  // engine's device thread, when the first backward reaches this library before any torch kernel there) has none:
  // make the device's primary context current through the runtime.
  int dev = 0;
  cudaError_t ce = cudaGetDevice(&dev);
  if (ce == cudaSuccess) ce = cudaSetDevice(dev);
  if (ce != cudaSuccess) return set_error(OTB_ERR_CUDA, "cudaSetDevice before cuTensorMapEncodeTiled: %s", cudaGetErrorString(ce));
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * esz};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                  const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(OTB_ERR_CUDA, "cuTensorMapEncodeTiled(%s) failed (%d) rows=%llu cols=%llu ld=%llu box=%ux%u",
                     f32 ? "f32" : "bf16", (int)r, (unsigned long long)rows, (unsigned long long)cols,
                     (unsigned long long)ld, box_rows, box_cols);
  g_tmap_misses.fetch_add(1, std::memory_order_relaxed);
  std::lock_guard<std::mutex> lk(g_tmap_mu);
  if (g_tmap_cache.size() >= kTmapCacheMax) g_tmap_cache.clear();
  g_tmap_cache.emplace(key, *map);
  return OTB_OK;
}

int make_tmap_bf16_2d(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                      uint32_t box_rows, uint32_t box_cols) {
  return make_tmap_2d(map, base, rows, cols, ld, box_rows, box_cols, false);
}

int make_tmap_f32_2d(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                     uint32_t box_cols) {
  return make_tmap_2d(map, base, rows, cols, ld, box_rows, box_cols, true);
}

bool pdl_enabled() {
  static const bool on = [] { const char* e = getenv("OTB_PDL"); return (e && e[0] == '1'); }();
  return on;
}

// Per-device state.  Function attributes and the SM count belong to a DEVICE, not to the process: the reference's
// demos place the model with device_map="auto" (pipeline/demos/demo_models.py:37), so one process may launch on several
// GPUs, and from several threads.
constexpr int kMaxDevices = 64;

int sm_count() {
  static std::atomic<int> cache[kMaxDevices];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return 132;
  int n = cache[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cache[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

cudaError_t ensure_dyn_smem(const void* func, int bytes) {
  static std::mutex mu;
  static std::unordered_map<const void*, uint64_t> done;     // func -> bit mask of devices already configured
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= kMaxDevices) return cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  std::lock_guard<std::mutex> lk(mu);
  uint64_t& mask = done[func];
  if (mask & (1ull << dev)) return cudaSuccess;
  e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) mask |= (1ull << dev);
  return e;
}

}  // namespace otb

extern "C" {
const char* otb_last_error(void) { return otb::g_err; }
int otb_version(void) { return 1; }
int otb_compiled_arch(void) { return 90; }
long long otb_launch_count(void) { return otb::g_launches.load(); }
long long otb_tmap_cache_stat(int which) { return which ? otb::g_tmap_misses.load() : otb::g_tmap_hits.load(); }
int otb_abi_sizeof(int which) {
  switch (which) {
    case 0: return (int)sizeof(otb_gemm_epilogue);
    case 1: return (int)sizeof(otb_attn_desc);
    case 2: return (int)sizeof(otb_attn_grads);
    case 3: return (int)sizeof(otb_lm_attn_desc);
    case 4: return (int)sizeof(otb_lm_attn_grads);
    case 5: return (int)sizeof(otb_lm_attn_decode_desc);
    default: return -1;
  }
}
}
