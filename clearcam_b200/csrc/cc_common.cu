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

int check_workspace(const char* who, const void* handle, const void* d_ws) {
  CC_REQUIRE(handle, "%s: null handle", who);
  CC_REQUIRE(d_ws == nullptr || (reinterpret_cast<uintptr_t>(d_ws) & 255) == 0, "%s: the workspace must be 256-byte aligned", who);
  return CC_OK;
}

int HostTensors::fill(const char* w, int n, const char* const* names, const float* const* data, const int64_t* numels) {
  who = w;
  CC_REQUIRE(n >= 0 && (n == 0 || (names && data && numels)), "%s: null argument", who);
  for (int i = 0; i < n; ++i) {
    CC_REQUIRE(names[i] && data[i], "%s: tensor %d is NULL", who, i);
    map[names[i]] = {data[i], static_cast<long long>(numels[i])};
  }
  return CC_OK;
}
int HostTensors::get(const std::string& name, long long n, const float** out) const {
  auto it = map.find(name);
  CC_REQUIRE(it != map.end(), "%s: missing tensor '%s'", who, name.c_str());
  CC_REQUIRE(it->second.second == n, "%s: '%s' has %lld elements, expected %lld", who, name.c_str(), it->second.second, n);
  *out = it->second.first;
  return CC_OK;
}

int DeviceWeights::upload(const void* h, size_t bytes, void** d) {
  CC_CHECK_CUDA(cudaMalloc(d, bytes));
  allocs.push_back(*d);
  CC_CHECK_CUDA(cudaMemcpy(*d, h, bytes, cudaMemcpyHostToDevice));
  return CC_OK;
}
int DeviceWeights::up_f32(const std::string& name, long long n, float** d) {
  const float* h;
  if (int rc = host.get(name, n, &h)) return rc;
  return upload(h, n * 4, reinterpret_cast<void**>(d));
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
