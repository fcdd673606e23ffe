// The op list every network plan (YOLOv9, CLIP, AdaFace) is made of, and the functions that run, time and report it.
#pragma once
#include "cc_common.h"
#include "conv_gemm.cuh"
#include <functional>
#include <initializer_list>

namespace cc {

// What one call of a plan supplies at run time; everything else a launch reads is baked in when the plan is built.
struct PlanIO {
  const void* in = nullptr;              // the frames, images, token ids or faces of the call
  float* out = nullptr;                  // the call's output, rows of out_stride floats
  long long out_stride = 0;
  float* raw = nullptr;                  // the detector's optional [B,84,A] tap
  unsigned long long* trace = nullptr;   // run_ops: this op's 12 trace slots (nullptr: not tracing)
};

// One launch of a plan.
struct PlanOp {
  using Launch = std::function<int(const PlanIO&, cudaStream_t)>;
  const char* name = "";                 // interned: valid for the life of the process
  const char* kind = "";                 // the kernel, as the profile and trace report it ("conv_gemm", "avgpool2_pad", ...)
  double flops = 0, bytes = 0;           // algorithmic FLOPs and HBM bytes the profile reports
  cc_conv_op conv{};                     // what the cc_*_op_conv taps report (name left empty); CC_CONV_OP_NONE: not a conv
  cc_op_io io{};                         // what the cc_*_op_io taps report (kind and name left empty); the launch never reads it
  Launch launch;
};

// Operands of a cc_op_io: a slice with its extent (bf16 or f32 as s.f32 says), or a buffer of `type` elements.  ns: elements
// from one image to the next (0: dense).
cc_operand operand(const TSlice& s, int N, int H, int W, int ns = 0);
inline cc_operand operand(const TSlice& s) { return operand(s, s.N, s.H, s.W); }
cc_operand operand(const void* p, int type, int N, int H, int W, int C, int cs = 0, int co = 0, int ns = 0);
cc_op_io op_io(std::initializer_list<cc_operand> in, std::initializer_list<cc_operand> out);

const char* intern(const std::string& s);   // a copy of s that lives as long as the process
PlanOp plan_op(const std::string& name, const char* kind, const cc_op_io& io, PlanOp::Launch launch, double flops = 0,
               double bytes = 0);
// The operands of a conv op (the cc_op_io of cc_conv_op c)
cc_op_io conv_io(const cc_conv_op& c);
// A conv GEMM launch L built from d (and the chained 1x1 c, if c.out.p): FLOPs and bytes are L's.
PlanOp gemm_op(const std::string& name, const ConvDesc& d, const ChainDesc& c, const GemmLaunch& L);

// Launches ops [first, last) of `ops` (clamped to its size) on st.  ev: one event recorded before each op and one after the
// last.  When io.trace is set, op k gets the slots io.trace + 12 k.
int run_ops(const std::vector<PlanOp>& ops, const PlanIO& io, cudaStream_t st, size_t first = 0, size_t last = SIZE_MAX,
            std::vector<cudaEvent_t>* ev = nullptr);
// Runs every op with an event between launches, synchronises, and fills up to cap entries of each non-NULL array.
int profile_ops(const std::vector<PlanOp>& ops, const PlanIO& io, cudaStream_t st, int cap, float* ms, double* flops, double* bytes,
                const char** kinds, const char** names);
// The cc_*_op_conv taps: op i's conv with its name; returns the op count (out == NULL only counts).
int op_conv_tap(const char* who, const std::vector<PlanOp>& ops, int i, cc_conv_op* out);
// The cc_*_op_io taps: op i's operands with its kind and name; returns the op count (out == NULL only counts).
int op_io_tap(const char* who, const std::vector<PlanOp>& ops, int i, cc_op_io* out);
// The cc_*_run_ops range check.
int check_range(const char* who, int first, int last, int n);
// The layer taps: slice s (N x H x W pixels) -> dense fp32 [N*H*W][C].
int slice_to_f32_launch(const TSlice& s, float* dst, cudaStream_t st);

}  // namespace cc
