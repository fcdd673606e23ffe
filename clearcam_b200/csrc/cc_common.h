// clearcam_b200 — shared host-side helpers: error reporting (never abort: the reference's caller
// supervises failures itself, clearcam.py:543-546), CUDA checks, driver entry points.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <map>
#include <memory>
#include <string>
#include <utility>
#include <vector>

namespace cc {

enum : int {
  CC_OK = 0,
  CC_ERR_INVALID = -1,   // bad argument / unsupported shape
  CC_ERR_CUDA = -2,      // CUDA runtime / driver error
  CC_ERR_NOGPU = -3,     // no sm_90 device
  CC_ERR_STATE = -4,     // handle used in the wrong state
};

void set_error(const char* fmt, ...);
const char* last_error();

#define CC_CHECK_CUDA(expr)                                                                  \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      ::cc::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return ::cc::CC_ERR_CUDA;                                                              \
    }                                                                                        \
  } while (0)

#define CC_REQUIRE(cond, ...)          \
  do {                                 \
    if (!(cond)) {                     \
      ::cc::set_error(__VA_ARGS__);    \
      return ::cc::CC_ERR_INVALID;     \
    }                                  \
  } while (0)

// cuTensorMapEncodeTiled resolved through the runtime (no link-time libcuda dependency, so the
// library loads on a box without a driver and fails only when a GPU op is actually requested).
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_tiled();

int device_sm_count();  // cached; <=0 if no usable device

// One device workspace shared by every cached plan of a handle.  A plan is a list of launches whose pointers / TMA
// descriptors are baked against `base`; plans never own device memory, so any number of input shapes costs the memory of
// the LARGEST one (the reference's TinyJit keeps one buffer set per captured shape, utils/helpers.py:214-221).  Growing
// or replacing the workspace bumps `gen`; a cached plan built against an older generation is rebuilt on its next use.
// Consequence: the plans of one handle must run in stream order (one stream per handle, as the reference's single
// inference thread does, clearcam.py:247-279).
struct Arena {
  void* base = nullptr;
  size_t cap = 0;
  bool owned = true;          // false: caller-owned (cc_*_set_workspace), never grown
  uint64_t gen = 1;
  ~Arena() { if (owned && base) cudaFree(base); }
  int reserve(size_t bytes);  // CC_OK when cap >= bytes afterwards
  int adopt(void* d_ws, size_t bytes);   // caller-owned workspace; nullptr returns to the internal allocation
};
// Bump allocation inside an arena; `dry` only measures (pointers are fake but aligned, nothing may dereference them).
struct Bump {
  uint8_t* base = nullptr;
  size_t off = 0;
  bool dry = false;
  void* take(size_t bytes) {
    off = (off + 1023) & ~size_t(1023);
    void* p = (dry ? reinterpret_cast<uint8_t*>(uintptr_t(1) << 30) : base) + off;
    off += bytes;
    return p;
  }
};


// The plans of one handle, keyed by input shape, all addressing one Arena.  At most kMaxPlans are kept (host metadata only:
// plans own no device memory); the least recently used goes first.  A plan built against an older workspace generation is
// stale: it is dropped when the next plan is built and rebuilt on its next use.
template <class Key, class Plan>
struct PlanCache {
  static constexpr size_t kMaxPlans = 16;
  struct Entry { std::unique_ptr<Plan> plan; uint64_t gen = 0, last_use = 0; };
  const char* who;             // names the network in refusals ("yolo" -> "yolo plan: ...")
  Arena arena;                 // declared before `plans`, so the plans (and the CUDA graphs they hold) go first
  std::map<Key, Entry> plans;
  uint64_t tick = 0;
  explicit PlanCache(const char* w) : who(w) {}

  // The plan of `key`.  On a miss, measure(size_t* bytes) sizes the workspace with a dry pass, then build(Plan&, uint8_t*
  // base, size_t* used) builds the plan against the reserved workspace and reports the bytes it addresses.
  template <class Measure, class Build>
  int get(const Key& key, Measure&& measure, Build&& build, Plan** out) {
    auto it = plans.find(key);
    if (it != plans.end() && it->second.gen == arena.gen) {
      it->second.last_use = ++tick;
      *out = it->second.plan.get();
      return CC_OK;
    }
    size_t bytes = 0, used = 0;
    if (int rc = measure(&bytes)) return rc;
    if (int rc = arena.reserve(bytes)) return rc;
    for (auto p = plans.begin(); p != plans.end();)
      p = p->second.gen != arena.gen ? plans.erase(p) : std::next(p);
    std::unique_ptr<Plan> P(new Plan());
    if (int rc = build(*P, static_cast<uint8_t*>(arena.base), &used)) return rc;
    CC_REQUIRE(used <= arena.cap, "%s plan: workspace overrun (%zu > %zu)", who, used, arena.cap);
    if (plans.size() >= kMaxPlans) {
      auto lru = plans.begin();
      for (auto p = plans.begin(); p != plans.end(); ++p)
        if (p->second.last_use < lru->second.last_use) lru = p;
      plans.erase(lru);
    }
    Entry& e = plans[key];
    e.plan = std::move(P);
    e.gen = arena.gen;
    e.last_use = ++tick;
    *out = e.plan.get();
    return CC_OK;
  }
  // cc_*_set_workspace after check_workspace: every plan is rebuilt against the new workspace
  int adopt(void* d_ws, size_t bytes) {
    plans.clear();
    return arena.adopt(d_ws, bytes);
  }
};

// The checks every cc_*_set_workspace makes: a handle, and a workspace that is NULL or 256-byte aligned.
int check_workspace(const char* who, const void* handle, const void* d_ws);

// The host tensors a cc_*_create call receives, by name.  The pointers are borrowed: valid only during that call.
struct HostTensors {
  int fill(const char* who, int n, const char* const* names, const float* const* data, const int64_t* numels);
  int get(const std::string& name, long long n, const float** out) const;   // tensor `name`, which must have n elements
  void clear() { map.clear(); }  // before the create call returns: the pointers are the caller's
 private:
  const char* who = "";        // the entry point, named in refusals
  std::map<std::string, std::pair<const float*, long long>> map;
};

// A model's weights on the device: one allocation per upload, all freed with the model.
struct DeviceWeights {
  HostTensors host;            // the create call's tensors; emptied before it returns
  std::vector<void*> allocs;
  ~DeviceWeights() { for (void* p : allocs) cudaFree(p); }
  int upload(const void* h, size_t bytes, void** d);
  template <class E>
  int upload(const std::vector<E>& v, E** d) { return upload(v.data(), v.size() * sizeof(E), reinterpret_cast<void**>(d)); }
  int up_f32(const std::string& name, long long n, float** d);   // host tensor `name` of n elements, as it is
};

}  // namespace cc
