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

int sm_count();

// Tuning options: each has the name of an environment variable, which is read ONCE (first use); fresco_set_option()
// overrides it afterwards (tests, tools).  Nothing on a launch path calls getenv.
enum Option { OPT_ATTN_WIDE = 0, OPT_ATTN_POLY, OPT_ATTN_ROWSUM, OPT_TEMPORAL_V, OPT_GRAM_V, OPT_COUNT };
int option(Option which, int dflt);

}  // namespace fresco
