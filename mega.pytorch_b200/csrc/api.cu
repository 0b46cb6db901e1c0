// Library-level entry points of libmega_b200.so (error string, version, device probe).
#include <stdarg.h>
#include "common.cuh"
#include "mega_b200.h"

static thread_local char g_err[1024] = "";

void mega_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" const char* mega_last_error(void) { return g_err; }
extern "C" int mega_abi_version(void) { return 7; }
extern "C" int mega_device_ok(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return -1;
  return (prop.major == 9 && prop.minor == 0) ? 1 : 0;
}
