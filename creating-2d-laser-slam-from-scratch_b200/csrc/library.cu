// Library-wide entry points of libb200slam: the ABI version, the device count, and the thread-local text of the last
// failure that every translation unit records through set_last_error (B2S_FAIL, B2S_CUDA_CHECK).
#include "common.cuh"

namespace b2s {

static thread_local std::string g_last_error;
void set_last_error(const std::string &s) { g_last_error = s; }
std::string &last_error_ref() { return g_last_error; }

}  // namespace b2s

extern "C" {

int b2s_abi_version(void) { return B2S_ABI_VERSION; }
const char *b2s_last_error(void) { return b2s::last_error_ref().c_str(); }
int b2s_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

}  // extern "C"
