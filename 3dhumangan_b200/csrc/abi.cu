// Error state + version of the C ABI (include/hg3d.h).
#include <string.h>

#include "common.cuh"

namespace hg {
static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace hg

extern "C" {

const char* hg_last_error(void) { return hg::g_err; }

int hg_abi_version(void) { return 1; }

// Returns 0 when the current device is an sm_90 part (H100 / H200) this library was compiled for.
int hg_check_device(void) {
  int dev = 0;
  cudaDeviceProp p;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&p, dev) != cudaSuccess) {
    hg::set_error("hg_check_device: no CUDA device");
    return 2;
  }
  if (p.major != 9 || p.minor != 0) {
    hg::set_error("hg_check_device: device '%s' is sm_%d%d; this library contains sm_90a code only", p.name, p.major,
                  p.minor);
    return 1;
  }
  return 0;
}

}  // extern "C"
