#include "cc_common.h"
#include <stdarg.h>
#include <string.h>

namespace cc {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }

PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

int Arena::reserve(size_t bytes) {
  if (bytes <= cap) return CC_OK;
  CC_REQUIRE(owned, "workspace too small: the plan needs %zu bytes, the caller-owned workspace holds %zu", bytes, cap);
  if (base) { cudaFree(base); base = nullptr; cap = 0; }     // cudaFree synchronises: nothing in flight still reads it
  bytes = (bytes + (size_t(1) << 21) - 1) & ~((size_t(1) << 21) - 1);
  if (cudaMalloc(&base, bytes) != cudaSuccess) {
    base = nullptr;
    set_error("workspace: cudaMalloc(%zu) failed", bytes);
    return CC_ERR_CUDA;
  }
  cap = bytes;
  ++gen;
  return CC_OK;
}
int Arena::adopt(void* d_ws, size_t bytes) {
  if (owned && base) cudaFree(base);
  base = d_ws; cap = d_ws ? bytes : 0; owned = d_ws == nullptr;
  ++gen;
  return CC_OK;
}

int device_sm_count() {
  static int n = -2;
  if (n == -2) {
    int dev = 0;
    cudaDeviceProp prop;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
      n = -1;
    } else if (prop.major != 9) {
      n = -1;
    } else {
      n = prop.multiProcessorCount;
    }
  }
  return n;
}

}  // namespace cc
