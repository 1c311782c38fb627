// mqdet_b200 — error plumbing shared by all C-ABI entry points.
#include "common.cuh"
#include "../../include/mqdet_b200.h"
#include <stdarg.h>
#include <atomic>
#include <mutex>
#include <unordered_map>

namespace mqdet {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return MQDET_ERR_CUDA;
  }
  return MQDET_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Host helpers shared by the TMA / wgmma kernels: TMA tensor maps (cached per thread: encoding one costs a driver call, and the
// same (pointer, shape) tuples recur every step because the caller's allocator recycles its blocks), the SM count and the
// dynamic shared-memory opt-in, both per device.
// ---------------------------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static std::atomic<PFN_encodeTiled> fn{nullptr};  // process-wide driver entry point (not per-device state)
  PFN_encodeTiled f = fn.load(std::memory_order_acquire);
  if (!f) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !ptr) {
      set_error("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: %s", cudaGetErrorString(e));
      return nullptr;
    }
    f = reinterpret_cast<PFN_encodeTiled>(ptr);
    fn.store(f, std::memory_order_release);
  }
  return f;
}

namespace {
struct MapKey {
  uint64_t v[10];
  bool operator==(const MapKey& o) const { return memcmp(v, o.v, sizeof(v)) == 0; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    uint64_t h = 1469598103934665603ull;
    for (uint64_t x : k.v) h = (h ^ x) * 1099511628211ull;
    return (size_t)h;
  }
};
struct MapCache {
  std::unordered_map<MapKey, CUtensorMap, MapKeyHash> m;
  const CUtensorMap* find(const MapKey& k) {
    auto it = m.find(k);
    return it == m.end() ? nullptr : &it->second;
  }
  void put(const MapKey& k, const CUtensorMap& v) {
    if (m.size() > 8192) m.clear();
    m.emplace(k, v);
  }
};
thread_local MapCache g_maps;
}  // namespace

// 4-D map over an fp16 operand viewed as [b2][b1][rows][K]; box = [1][1][box_rows][64], 128B swizzle.
int make_operand_map(CUtensorMap* map, const void* ptr, long rows, long K, long ld, int nb1, long s1, int nb2, long s2,
                     int box_rows, int* bcast1, int* bcast2) {
  *bcast1 = (s1 == 0 || nb1 == 1);
  *bcast2 = (s2 == 0 || nb2 == 1);
  const MapKey key = {{(uint64_t)(uintptr_t)ptr, (uint64_t)rows, (uint64_t)K, (uint64_t)ld, (uint64_t)nb1, (uint64_t)s1,
                       (uint64_t)nb2, (uint64_t)s2, (uint64_t)box_rows, 0x100u}};
  if (const CUtensorMap* hit = g_maps.find(key)) {
    *map = *hit;
    return MQDET_OK;
  }
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return MQDET_ERR_CUDA;
  cuuint64_t dims[4] = {(cuuint64_t)K, (cuuint64_t)rows, (cuuint64_t)(*bcast1 ? 1 : nb1),
                        (cuuint64_t)(*bcast2 ? 1 : nb2)};
  // strides (bytes) of dims 1..3; unused batch dims get a harmless non-zero stride
  cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)((*bcast1 ? ld * rows : s1) * 2),
                           (cuuint64_t)((*bcast2 ? ld * rows : s2) * 2)};
  if (strides[1] == 0) strides[1] = 16;
  if (strides[2] == 0) strides[2] = 16;
  cuuint32_t box[4] = {64u, (cuuint32_t)box_rows, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): rows=%ld K=%ld ld=%ld nb1=%d s1=%ld nb2=%d s2=%ld ptr=%p", (int)r,
              rows, K, ld, nb1, s1, nb2, s2, ptr);
    return MQDET_ERR_CUDA;
  }
  g_maps.put(key, *map);
  return MQDET_OK;
}

// 4-D map over an OUTPUT viewed as [b2][b1][M][N] (c_dtype MQDET_F16 / MQDET_F32); box = [1][1][box_rows][128 bytes],
// 128B swizzle (the TMA-store epilogues of the GEMM (128 rows) and swin_mlp (64 rows); the unit clips the M / N edges).  The
// caller guarantees a 16-byte aligned base, ldc and the batch strides of batch dims > 1 multiples of 16 bytes; a batch dim of
// size 1 gets a harmless stride.
int make_store_map(CUtensorMap* map, void* C, int c_dtype, long M, long N, long ldc, int nb1, long c_b1, int nb2, long c_b2,
                   int box_rows) {
  const MapKey key = {{(uint64_t)(uintptr_t)C, (uint64_t)M, (uint64_t)N, (uint64_t)ldc, (uint64_t)nb1, (uint64_t)c_b1,
                       (uint64_t)nb2, (uint64_t)c_b2, (uint64_t)c_dtype, 0x200u | ((uint64_t)box_rows << 12)}};
  if (const CUtensorMap* hit = g_maps.find(key)) {
    *map = *hit;
    return MQDET_OK;
  }
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return MQDET_ERR_CUDA;
  const int es = (c_dtype == MQDET_F16) ? 2 : 4;
  cuuint64_t dims[4] = {(cuuint64_t)N, (cuuint64_t)M, (cuuint64_t)nb1, (cuuint64_t)nb2};
  cuuint64_t strides[3] = {(cuuint64_t)ldc * es, (cuuint64_t)(nb1 > 1 ? c_b1 : ldc * M) * es,
                           (cuuint64_t)(nb2 > 1 ? c_b2 : ldc * M) * es};
  cuuint32_t box[4] = {(cuuint32_t)(128 / es), (cuuint32_t)box_rows, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(map, c_dtype == MQDET_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, C, dims,
                   strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(C) failed (%d): M=%ld N=%ld ldc=%ld", (int)r, M, N, ldc);
    return MQDET_ERR_CUDA;
  }
  g_maps.put(key, *map);
  return MQDET_OK;
}

static const int kMaxDev = 64;

// SMs the persistent one-CTA-per-SM kernels leave free (process-wide, set once before the first launch / graph capture):
// a collective that runs next to the forward (one NCCL CTA spinning on a peer) otherwise takes the SM of one persistent CTA, whose
// tiles then wait behind it in every kernel of the step.
static std::atomic<int> g_reserved_sms{0};

extern "C" int mqdet_reserve_sms(int n) {
  if (n < 0 || n > 64) {
    mqdet::set_error("mqdet_reserve_sms: 0 <= n <= 64 (got %d)", n);
    return MQDET_ERR_ARG;
  }
  g_reserved_sms.store(n, std::memory_order_relaxed);
  return MQDET_OK;
}

int num_sms() {
  static std::atomic<int> n[kMaxDev];
  int dev = 0;
  cudaGetDevice(&dev);
  const int slot = dev >= 0 && dev < kMaxDev ? dev : 0;
  int v = n[slot].load(std::memory_order_relaxed);
  if (!v) {
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    if (v <= 0) v = 132;
    n[slot].store(v, std::memory_order_relaxed);
  }
  const int r = g_reserved_sms.load(std::memory_order_relaxed);
  return v - r > 8 ? v - r : v;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is per (function, device): remember which pairs have been set.
int ensure_dyn_smem(const void* func, int bytes) {
  static std::mutex mu;
  static std::unordered_map<uint64_t, int> done;
  int dev = 0;
  cudaGetDevice(&dev);
  const uint64_t key = ((uint64_t)(uintptr_t)func) * 64u + (uint64_t)(dev & 63);
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = done.find(key);
    if (it != done.end() && it->second >= bytes) return MQDET_OK;
  }
  cudaError_t e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) {
    set_error("cudaFuncSetAttribute(smem=%d) failed: %s", bytes, cudaGetErrorString(e));
    (void)cudaGetLastError();  // the failure is reported here; do not leave it for the caller's next CUDA call
    return MQDET_ERR_CUDA;
  }
  std::lock_guard<std::mutex> g(mu);
  done[key] = bytes;
  return MQDET_OK;
}

}  // namespace mqdet

extern "C" const char* mqdet_last_error(void) { return mqdet::g_err; }
extern "C" int mqdet_version(void) { return 100; }
