// Error reporting + library identification for the C-ABI (include/b200rl.h).
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

static thread_local char g_err[512] = "";

extern "C" void b200rl_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" const char* b200rl_last_error(void) { return g_err; }

extern "C" int b200rl_abi_version(void) { return 1; }

// Compiled-for architecture, so the loader can refuse anything but sm_90a.
extern "C" const char* b200rl_build_arch(void) { return "sm_90a"; }

extern "C" int b200rl_device_check(void) {
  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
    b200rl_set_error("no CUDA device");
    return B200RL_ERR_CUDA;
  }
  if (prop.major != 9 || prop.minor != 0) {
    b200rl_set_error("b200rl is built for sm_90a only; found sm_%d%d", prop.major, prop.minor);
    return B200RL_ERR_CUDA;
  }
  return B200RL_OK;
}
