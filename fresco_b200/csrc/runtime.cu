// Error state, launch accounting, TMA tensor maps and per-device launch set-up.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <utility>

#include "fresco_internal.h"

namespace fresco {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};
static thread_local char g_last_kernel[128] = "";

int set_error(int code, const char* msg) {
  snprintf(g_err, sizeof(g_err), "%s", msg);
  return code;
}

int set_cuda_error(cudaError_t e, const char* where) {
  snprintf(g_err, sizeof(g_err), "%s: %s", where, cudaGetErrorString(e));
  return FRESCO_ERR_CUDA;
}

int check_launch(const char* kernel) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  snprintf(g_last_kernel, sizeof(g_last_kernel), "%s", kernel);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error(e, kernel);
  return FRESCO_OK;
}

int check_launchf(const char* fmt, ...) {
  char name[sizeof(g_last_kernel)];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(name, sizeof(name), fmt, ap);
  va_end(ap);
  return check_launch(name);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int encode_tiled_map(CUtensorMap* map, CUtensorMapDataType dtype, int rank, void* base, const cuuint64_t* dims,
                     const cuuint64_t* strides_bytes, const cuuint32_t* box, const cuuint32_t* elem_strides,
                     CUtensorMapSwizzle swizzle) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return set_error(FRESCO_ERR_TENSORMAP, "cuTensorMapEncodeTiled entry point not available (no driver?)");
  CUresult r = fn(map, dtype, (cuuint32_t)rank, base, dims, strides_bytes, box, elem_strides,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof(buf),
             "cuTensorMapEncodeTiled failed (CUresult %d): rank %d dims {%llu,%llu,%llu,%llu} box {%u,%u,%u,%u}",
             (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
             (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0],
             rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
    return set_error(FRESCO_ERR_TENSORMAP, buf);
  }
  return FRESCO_OK;
}

int make_kmajor_map(CUtensorMap* map, const void* base, int rows, int K, int batch, int box_rows) {
  const cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)rows, (cuuint64_t)batch};
  const cuuint64_t strides[2] = {(cuuint64_t)K * 2, (cuuint64_t)rows * K * 2};
  const cuuint32_t box[3] = {64, (cuuint32_t)box_rows, 1};
  const cuuint32_t es[3] = {1, 1, 1};
  return encode_tiled_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, es,
                          CU_TENSOR_MAP_SWIZZLE_128B);
}

int make_mnmajor_map(CUtensorMap* map, const void* base, int K, int N, int batch) {
  const cuuint64_t dims[3] = {(cuuint64_t)N, (cuuint64_t)K, (cuuint64_t)batch};
  const cuuint64_t strides[2] = {(cuuint64_t)N * 2, (cuuint64_t)K * N * 2};
  const cuuint32_t box[3] = {64, 64, 1};
  const cuuint32_t es[3] = {1, 1, 1};
  return encode_tiled_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, es,
                          CU_TENSOR_MAP_SWIZZLE_128B);
}

// per-device state: the dynamic shared memory each kernel may use, and the SM count
static std::mutex g_device_mu;
static std::map<std::pair<const void*, int>, size_t> g_smem_allowed;
static std::map<int, int> g_sm_count;

int allow_dynamic_smem(const void* kernel, size_t bytes, const char* what) {
  if (bytes <= 48 * 1024) return FRESCO_OK;
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lock(g_device_mu);
  size_t& allowed = g_smem_allowed[{kernel, dev}];
  if (bytes <= allowed) return FRESCO_OK;
  const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) {
    char where[128];
    snprintf(where, sizeof(where), "cudaFuncSetAttribute(%s)", what);
    return set_cuda_error(e, where);
  }
  allowed = bytes;
  return FRESCO_OK;
}

static const char* const kOptionNames[OPT_COUNT] = {"FRESCO_ATTN_WIDE", "FRESCO_ATTN_POLY", "FRESCO_ATTN_ROWSUM",
                                                    "FRESCO_TEMPORAL_V", "FRESCO_GRAM_V"};
static std::atomic<int> g_opt_state[OPT_COUNT];      // 0 = not looked at, 1 = unset (use the default), 2 = set
static std::atomic<int> g_opt_value[OPT_COUNT];

int option(Option which, int dflt) {
  int st = g_opt_state[which].load(std::memory_order_acquire);
  if (st == 0) {
    const char* v = getenv(kOptionNames[which]);
    if (v) g_opt_value[which].store(atoi(v), std::memory_order_relaxed);
    st = v ? 2 : 1;
    g_opt_state[which].store(st, std::memory_order_release);
  }
  return st == 2 ? g_opt_value[which].load(std::memory_order_relaxed) : dflt;
}

int sm_count() {
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lock(g_device_mu);
  int& n = g_sm_count[dev];
  if (n == 0) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 148;
  }
  return n;
}

}  // namespace fresco

extern "C" int fresco_abi_version(void) { return FRESCO_ABI_VERSION; }
extern "C" const char* fresco_last_error(void) { return fresco::g_err; }
extern "C" long long fresco_launch_count(void) { return fresco::g_launches.load(); }
extern "C" const char* fresco_last_kernel(void) { return fresco::g_last_kernel; }
extern "C" int fresco_set_option(const char* name, int value) {
  using namespace fresco;
  if (!name) return set_error(FRESCO_ERR_ARG, "fresco_set_option: null name");
  for (int i = 0; i < OPT_COUNT; ++i)
    if (strcmp(name, kOptionNames[i]) == 0) {
      if (value < 0) {                       // negative: back to the built-in default
        g_opt_state[i].store(1, std::memory_order_release);
      } else {
        g_opt_value[i].store(value, std::memory_order_relaxed);
        g_opt_state[i].store(2, std::memory_order_release);
      }
      return FRESCO_OK;
    }
  return set_error(FRESCO_ERR_ARG, "fresco_set_option: unknown option");
}
