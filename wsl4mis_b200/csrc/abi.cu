// Error plumbing + library info for the C ABI (see include/wsl4mis_b200.h).
#include "common.cuh"
#include <stdarg.h>
#include <string.h>

static thread_local char g_err[512] = "";

void wsl_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int wsl_check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    wsl_set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return -2;
  }
  return 0;
}

WSL_API const char* wsl_last_error(void) { return g_err; }
WSL_API int wsl_abi_version(void) { return 2; }
WSL_API int wsl_workspace_floats(void) { return WSL_WS_FLOATS; }
