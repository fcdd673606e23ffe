// The op list of the network plans: run, profile, conv taps and the layer tap kernel (plan.h).
#include "plan.h"
#include <mutex>
#include <unordered_set>

namespace cc {

const char* intern(const std::string& s) {
  static std::mutex mu;
  static std::unordered_set<std::string> pool;   // node-based: an element's c_str() never moves
  std::lock_guard<std::mutex> lock(mu);
  return pool.insert(s).first->c_str();
}

PlanOp plan_op(const std::string& name, const char* kind, PlanOp::Launch launch, double flops, double bytes) {
  PlanOp op;
  op.name = intern(name); op.kind = kind; op.flops = flops; op.bytes = bytes; op.launch = std::move(launch);
  return op;
}

PlanOp gemm_op(const std::string& name, const ConvDesc& d, const ChainDesc& c, const GemmLaunch& L) {
  PlanOp op = plan_op(name, "conv_gemm", [L](const PlanIO& io, cudaStream_t st) {
    if (!io.trace) return conv_gemm_launch(L, st);
    GemmLaunch g = L;
    g.p.trace = io.trace;
    return conv_gemm_launch(g, st);
  }, L.flops, L.bytes);
  op.conv = conv_op_of(d, c, L);
  return op;
}

int run_ops(const std::vector<PlanOp>& ops, const PlanIO& io, cudaStream_t st, size_t first, size_t last, std::vector<cudaEvent_t>* ev) {
  if (last > ops.size()) last = ops.size();
  PlanIO o = io;
  size_t e = 0;
  for (size_t k = first; k < last; ++k) {
    if (ev) cudaEventRecord((*ev)[e++], st);
    if (io.trace) o.trace = io.trace + 12 * k;
    if (int rc = ops[k].launch(o, st)) return rc;
  }
  if (ev) cudaEventRecord((*ev)[e], st);
  return CC_OK;
}

int profile_ops(const std::vector<PlanOp>& ops, const PlanIO& io, cudaStream_t st, int cap, float* ms, double* flops, double* bytes,
                const char** kinds, const char** names) {
  const size_t n = ops.size();
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& e : ev) CC_CHECK_CUDA(cudaEventCreate(&e));
  int rc = run_ops(ops, io, st, 0, n, &ev);
  if (!rc) {
    CC_CHECK_CUDA(cudaStreamSynchronize(st));
    for (size_t i = 0; i < n && static_cast<int>(i) < cap; ++i) {
      float t = 0.f;
      cudaEventElapsedTime(&t, ev[i], ev[i + 1]);
      if (ms) ms[i] = t;
      if (flops) flops[i] = ops[i].flops;
      if (bytes) bytes[i] = ops[i].bytes;
      if (kinds) kinds[i] = ops[i].kind;
      if (names) names[i] = ops[i].name;
    }
  }
  for (auto& e : ev) cudaEventDestroy(e);
  return rc;
}

int op_conv_tap(const char* who, const std::vector<PlanOp>& ops, int i, cc_conv_op* out) {
  const int n = static_cast<int>(ops.size());
  if (!out) return n;
  CC_REQUIRE(i >= 0 && i < n, "%s: op %d of a plan of %d ops", who, i, n);
  *out = ops[i].conv;
  snprintf(out->name, sizeof(out->name), "%s", ops[i].name);
  return n;
}

int check_range(const char* who, int first, int last, int n) {
  CC_REQUIRE(0 <= first && first <= last && last <= n, "%s: ops [%d, %d) of a plan of %d ops", who, first, last, n);
  return CC_OK;
}

__global__ void slice_to_f32_kernel(const __nv_bfloat16* src, int f32, int cs, int co, int C, long long npix, float* dst) {
  const long long total = npix * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long pix = i / C;
    const int c = static_cast<int>(i % C);
    dst[i] = f32 ? reinterpret_cast<const float*>(src)[pix * cs + co + c] : __bfloat162float(src[pix * cs + co + c]);
  }
}

int slice_to_f32_launch(const TSlice& s, float* dst, cudaStream_t st) {
  slice_to_f32_kernel<<<132 * 8, 256, 0, st>>>(s.p, s.f32 ? 1 : 0, s.cs, s.co, s.C, static_cast<long long>(s.N) * s.H * s.W, dst);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

}  // namespace cc
