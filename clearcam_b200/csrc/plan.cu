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

cc_operand operand(const TSlice& s, int N, int H, int W, int ns) {
  cc_operand o{};
  o.s = cc_slice{s.p, s.cs, s.co, s.C, N, H, W, s.f32 ? 1 : 0};
  o.type = s.f32 ? CC_OP_F32 : CC_OP_BF16;
  o.ns = ns;
  return o;
}

cc_operand operand(const void* p, int type, int N, int H, int W, int C, int cs, int co, int ns) {
  cc_operand o{};
  o.s = cc_slice{const_cast<void*>(p), cs ? cs : C, co, C, N, H, W, type == CC_OP_F32 ? 1 : 0};
  o.type = type;
  o.ns = ns;
  return o;
}

cc_op_io op_io(std::initializer_list<cc_operand> in, std::initializer_list<cc_operand> out) {
  cc_op_io io{};
  for (const cc_operand& o : in) if (io.n_in < CC_OP_IO_MAX) io.in[io.n_in++] = o;
  for (const cc_operand& o : out) if (io.n_out < CC_OP_IO_MAX) io.out[io.n_out++] = o;
  return io;
}

cc_op_io conv_io(const cc_conv_op& c) {
  auto op = [](const cc_slice& s, int ns) {
    cc_operand o{};
    o.s = s; o.type = s.f32 ? CC_OP_F32 : CC_OP_BF16; o.ns = ns;
    return o;
  };
  cc_op_io io{};
  io.in[io.n_in++] = op(c.in, 0);
  if (c.res.p) io.in[io.n_in++] = op(c.res, c.out_ns);
  if (c.pre) io.in[io.n_in++] = op(cc_slice{const_cast<float*>(c.pre), c.out.C, 0, c.out.C, c.out.N, c.pre_h, c.pre_w, 1}, 0);
  if (c.part.p) io.in[io.n_in++] = op(c.part, 0);
  if (c.out.p && (c.kind != CC_CONV_OP_CHAIN || c.store1)) io.out[io.n_out++] = op(c.out, c.out_ns);
  if (c.kind == CC_CONV_OP_CHAIN) io.out[io.n_out++] = op(c.out2, 0);
  return io;
}

PlanOp plan_op(const std::string& name, const char* kind, const cc_op_io& io, PlanOp::Launch launch, double flops, double bytes) {
  PlanOp op;
  op.name = intern(name); op.kind = kind; op.io = io; op.flops = flops; op.bytes = bytes; op.launch = std::move(launch);
  return op;
}

PlanOp gemm_op(const std::string& name, const ConvDesc& d, const ChainDesc& c, const GemmLaunch& L) {
  const cc_conv_op conv = conv_op_of(d, c, L);
  PlanOp op = plan_op(name, "conv_gemm", conv_io(conv), [L](const PlanIO& io, cudaStream_t st) {
    if (!io.trace) return conv_gemm_launch(L, st);
    GemmLaunch g = L;
    g.p.trace = io.trace;
    return conv_gemm_launch(g, st);
  }, L.flops, L.bytes);
  op.conv = conv;
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

int op_io_tap(const char* who, const std::vector<PlanOp>& ops, int i, cc_op_io* out) {
  const int n = static_cast<int>(ops.size());
  if (!out) return n;
  CC_REQUIRE(i >= 0 && i < n, "%s: op %d of a plan of %d ops", who, i, n);
  *out = ops[i].io;
  snprintf(out->kind, sizeof(out->kind), "%s", ops[i].kind);
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
