// Error plumbing and small arithmetic helpers shared by every translation unit of lib3dhg_sm90a.so.
#pragma once
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

namespace hg {

constexpr int kNumSMsH100 = 132;

void set_error(const char* fmt, ...);  // defined in abi.cu (thread-local message)

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return 2;
  }
  return 0;
}

#define HG_REQUIRE(cond, ...)        \
  do {                               \
    if (!(cond)) {                   \
      hg::set_error(__VA_ARGS__);    \
      return 1;                      \
    }                                \
  } while (0)

// fp32 pairs: one rounding per lane, never contracted (the Cody-Waite reductions depend on the separate roundings)
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }

inline int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = kNumSMsH100;
  }
  return n;
}

}  // namespace hg
