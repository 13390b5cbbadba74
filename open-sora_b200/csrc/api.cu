// osb200 library management: init, thread-local error string, launch accounting, TMA descriptor
// encoding through the driver entry point (no link-time dependency on libcuda).
#include <cudaTypedefs.h>
#include <stdarg.h>

#include <stdlib.h>

#include <atomic>
#include <mutex>
#include <unordered_map>

#include "common.cuh"

namespace osb {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};
static bool g_init = false;
static int g_sms = 0;
static PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
bool initialised() { return g_init; }
bool pdl_enabled() {
  static const bool on = [] { const char* e = getenv("OSB_PDL"); return !(e && e[0] == '0'); }();
  return on;
}
int sm_count() { return g_sms; }

// Descriptor cache (SURVEY.md §8b: "process-global state limited to per-device immutable caches (TMA descriptors keyed
// by pointer/shape)").  A tensor map is a pure function of (base, rows, cols, ld, box), so an entry can never go stale;
// the block loop of a denoise step re-uses ~40 distinct operand views 346 times, and a CUDA-graph capture or a
// sequence-parallel rank with 2 048 tokens is host-bound on cuTensorMapEncodeTiled otherwise.
struct TmapKey {
  uint64_t base, rows, cols, ld, box;
  uint32_t elem_bytes;
  bool operator==(const TmapKey& o) const {
    return base == o.base && rows == o.rows && cols == o.cols && ld == o.ld && box == o.box && elem_bytes == o.elem_bytes;
  }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    uint64_t h = k.base * 0x9E3779B97F4A7C15ull;
    h ^= (k.rows + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
    h ^= (k.cols + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
    h ^= (k.ld + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
    h ^= (k.box + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
    return (size_t)h;
  }
};
static std::mutex g_tmap_mu;
static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> g_tmap_cache;
static std::atomic<int64_t> g_tmap_hits{0}, g_tmap_misses{0};

// elem_bytes 2: bf16, 1: e4m3 (ld and cols in elements; the swizzle row is 128 bytes either way)
static int make_tmap_2d(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                        uint32_t box_cols, uint32_t elem_bytes) {
  if (!g_encode) {
    set_error("osb_init() has not been called");
    return OSB_ERR_NOT_INIT;
  }
  const TmapKey key{reinterpret_cast<uint64_t>(base), rows, cols, ld, ((uint64_t)box_rows << 32) | box_cols, elem_bytes};
  {
    std::lock_guard<std::mutex> lk(g_tmap_mu);
    auto it = g_tmap_cache.find(key);
    if (it != g_tmap_cache.end()) {
      *map = it->second;
      g_tmap_hits.fetch_add(1, std::memory_order_relaxed);
      return OSB_OK;
    }
  }
  g_tmap_misses.fetch_add(1, std::memory_order_relaxed);
  if ((reinterpret_cast<uintptr_t>(base) & 15) || ((ld * elem_bytes) & 15)) {
    set_error("TMA operand must be 16-byte aligned (base %p, ld %llu elements)", base,
              (unsigned long long)ld);
    return OSB_ERR_INVALID;
  }
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld * elem_bytes};  // bytes, dims 1..rank-1
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estride[2] = {1, 1};
  CUresult r = g_encode(map, elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                        const_cast<void*>(base), gdim,
                        gstride, box, estride, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rows %llu cols %llu ld %llu box %ux%u)",
              (int)r, (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld,
              box_rows, box_cols);
    return OSB_ERR_CUDA;
  }
  {
    std::lock_guard<std::mutex> lk(g_tmap_mu);
    if (g_tmap_cache.size() >= 8192) g_tmap_cache.clear();   // bounded: a long-lived process with many shapes starts over
    g_tmap_cache.emplace(key, *map);
  }
  return OSB_OK;
}

int make_tmap_2d_bf16(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols,
                      uint64_t ld, uint32_t box_rows, uint32_t box_cols) {
  return make_tmap_2d(map, base, rows, cols, ld, box_rows, box_cols, 2);
}

int make_tmap_2d_e4m3(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols,
                      uint64_t ld, uint32_t box_rows, uint32_t box_cols) {
  return make_tmap_2d(map, base, rows, cols, ld, box_rows, box_cols, 1);
}

int make_tmap_5d_bf16(CUtensorMap* map, const void* base, const uint64_t dims[5], const uint64_t strides_bytes[4],
                      const uint32_t box[5], const uint32_t elem_strides[5]) {
  if (!g_encode) {
    set_error("osb_init() has not been called");
    return OSB_ERR_NOT_INIT;
  }
  if (reinterpret_cast<uintptr_t>(base) & 15) {
    set_error("TMA operand must be 16-byte aligned (base %p)", base);
    return OSB_ERR_INVALID;
  }
  cuuint64_t gdim[5], gstride[4];
  cuuint32_t b[5], es[5];
  for (int i = 0; i < 5; ++i) { gdim[i] = dims[i]; b[i] = box[i]; es[i] = elem_strides[i]; }
  for (int i = 0; i < 4; ++i) {
    if (strides_bytes[i] & 15) {
      set_error("TMA stride %d (%llu bytes) is not a multiple of 16", i, (unsigned long long)strides_bytes[i]);
      return OSB_ERR_INVALID;
    }
    gstride[i] = strides_bytes[i];
  }
  CUresult r = g_encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(base), gdim, gstride, b, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(5D) failed with CUresult %d (dims %llu %llu %llu %llu %llu box %u %u %u %u %u)", (int)r,
              (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2],
              (unsigned long long)dims[3], (unsigned long long)dims[4], box[0], box[1], box[2], box[3], box[4]);
    return OSB_ERR_CUDA;
  }
  return OSB_OK;
}

int make_row_scatter(RowScatter* dst, const osb_scatter* src, int64_t rows, const char* who) {
  *dst = RowScatter();
  if (src == nullptr || src->mode == 0) return OSB_OK;
  if (src->mode < 1 || src->mode > 4) { set_error("%s: unknown scatter mode %d", who, src->mode); return OSB_ERR_INVALID; }
  if (src->P < 1 || src->P > OSB_MAX_PEERS || src->rank < 0 || src->rank >= src->P || src->I <= 0 || src->J <= 0) {
    set_error("%s: bad scatter (P %d rank %d I %d J %d)", who, src->P, src->rank, src->I, src->J);
    return OSB_ERR_INVALID;
  }
  const int split = src->mode == 2 ? src->I : (src->mode == 3 ? src->P : src->J);
  if (split % src->P != 0 || rows % ((int64_t)src->I * src->J) != 0 || rows >= (1ll << 31)) {
    set_error("%s: scatter of [*, %d, %d] rows over %d ranks does not divide (%lld rows)", who, src->I, src->J, src->P, (long long)rows);
    return OSB_ERR_INVALID;
  }
  dst->mode = src->mode; dst->P = src->P; dst->rank = src->rank; dst->I = src->I; dst->J = src->J;
  for (int p = 0; p < src->P; ++p) {
    if (src->peer[p] == nullptr || (reinterpret_cast<uintptr_t>(src->peer[p]) & 15)) {
      set_error("%s: peer buffer %d is null or not 16-byte aligned", who, p);
      return OSB_ERR_INVALID;
    }
    dst->peer[p] = src->peer[p];
  }
  return OSB_OK;
}

int gemm_init();   // gemm_sm90.cu
int attn_init();   // attn_sm90.cu
int attn_fp8_init();   // attn_fp8_sm90.cu

}  // namespace osb

extern "C" {

int osb_version(void) { return 200; }
const char* osb_last_error(void) { return osb::g_err; }
int64_t osb_launch_count(void) { return osb::g_launches.load(); }

void osb_tmap_cache_stats(int64_t* hits, int64_t* misses) {
  if (hits) *hits = osb::g_tmap_hits.load();
  if (misses) *misses = osb::g_tmap_misses.load();
}

int osb_init(int device) {
  using namespace osb;
  // bind for the duration of the call only: the caller's current device is restored (kernels launch on the device
  // that owns the stream they are given)
  int prev_device = -1;
  OSB_CHECK_CUDA(cudaGetDevice(&prev_device));
  struct Restore { int d; ~Restore() { if (d >= 0) cudaSetDevice(d); } } restore{prev_device == device ? -1 : prev_device};
  OSB_CHECK_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  OSB_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("osb200 is built for sm_90a only; device %d is sm_%d%d", device, prop.major,
              prop.minor);
    return OSB_ERR_UNSUPPORTED;
  }
  g_sms = prop.multiProcessorCount;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  OSB_CHECK_CUDA(cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &fn, 12000,
                                                  cudaEnableDefault, &qres));
  if (qres != cudaDriverEntryPointSuccess || fn == nullptr) {
    set_error("cuTensorMapEncodeTiled not available from the driver");
    return OSB_ERR_CUDA;
  }
  g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  int rc = gemm_init();
  if (rc) return rc;
  rc = attn_init();
  if (rc) return rc;
  rc = attn_fp8_init();
  if (rc) return rc;
  g_init = true;
  return OSB_OK;
}

}  // extern "C"
