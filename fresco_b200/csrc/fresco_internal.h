// Internal helpers shared by the .cu translation units of libfresco_b200.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/fresco_b200.h"

namespace fresco {

int set_error(int code, const char* msg);
int set_cuda_error(cudaError_t e, const char* where);
// records `kernel` as the calling thread's last launch (fresco_last_kernel) and checks the launch for errors;
// check_launchf formats the name, so a templated launch site can name its instantiation
int check_launch(const char* kernel);
int check_launchf(const char* fmt, ...) __attribute__((format(printf, 1, 2)));

// cuTensorMapEncodeTiled resolved at run time through cudaGetDriverEntryPoint, so the library
// has no link-time dependency on libcuda.so (it must load on a driver-less build box).
int encode_tiled_map(CUtensorMap* map, CUtensorMapDataType dtype, int rank, void* base, const cuuint64_t* dims,
                     const cuuint64_t* strides_bytes, const cuuint32_t* box, const cuuint32_t* elem_strides,
                     CUtensorMapSwizzle swizzle);
// fp16 GEMM operands, 128-byte swizzle.  K-major [batch, rows, K] -> {K, rows, batch}, box {64, box_rows, 1};
// MN-major [batch, K rows, N cols] -> {N, K, batch}, box {64, 64, 1}
int make_kmajor_map(CUtensorMap* map, const void* base, int rows, int K, int batch, int box_rows);
int make_mnmajor_map(CUtensorMap* map, const void* base, int K, int N, int batch);

// Lets `kernel` launch with up to `bytes` of dynamic shared memory on the current device.  The attribute is set once
// per (kernel, device), raised only when a larger amount is asked for, and never needed at or below the 48 KB
// default; thread-safe.  Failure is reported through set_cuda_error, naming `what`.
int allow_dynamic_smem(const void* kernel, size_t bytes, const char* what);

// multiprocessor count of the current device, looked up once per device
int sm_count();

// Tuning options: each has the name of an environment variable, which is read ONCE (first use); fresco_set_option()
// overrides it afterwards (tests, tools).  Nothing on a launch path calls getenv.
enum Option { OPT_ATTN_WIDE = 0, OPT_ATTN_POLY, OPT_ATTN_ROWSUM, OPT_TEMPORAL_V, OPT_GRAM_V, OPT_COUNT };
int option(Option which, int dflt);

}  // namespace fresco
