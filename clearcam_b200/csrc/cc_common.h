// clearcam_b200 — shared host-side helpers: error reporting (never abort: the reference's caller
// supervises failures itself, clearcam.py:543-546), CUDA checks, driver entry points.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

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

}  // namespace cc
