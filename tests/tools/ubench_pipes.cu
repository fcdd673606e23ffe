// Throughput of the epilogue's candidate instructions on one SM sub-partition mix: cycles per warp-instruction with
// 1, 2, 4, 8 warps per scheduler.  build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ubench_pipes ubench_pipes.cu
#include <cstdio>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

template <int OP>
__global__ void k(float* out, int iters, unsigned long long* cyc) {
  float a[8];
  for (int i = 0; i < 8; ++i) a[i] = threadIdx.x * 0.001f + i * 0.37f - 1.0f;
  uint32_t acc = 0;
  __syncthreads();
  const long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (OP == 0) asm volatile("tanh.approx.f32 %0, %0;" : "+f"(a[i]));
      if (OP == 1) asm volatile("ex2.approx.ftz.f32 %0, %0;" : "+f"(a[i]));
      if (OP == 2) asm volatile("rcp.approx.ftz.f32 %0, %0;" : "+f"(a[i]));
      if (OP == 3) a[i] = fmaf(a[i], 1.0001f, 0.5f);
    }
    if (OP == 4) {   // 4 cvt.rn.bf16x2.f32 packs
#pragma unroll
      for (int i = 0; i < 8; i += 2) {
        uint32_t r;
        asm volatile("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(a[i]), "f"(a[i + 1]));
        acc ^= r;
        a[i] += 1.0f;
      }
    }
    if (OP == 5) {   // integer half-up packs: 2 IADD + PRMT per pair
#pragma unroll
      for (int i = 0; i < 8; i += 2) {
        const uint32_t x = __float_as_uint(a[i]) + 0x8000u, y = __float_as_uint(a[i + 1]) + 0x8000u;
        acc ^= __byte_perm(x, y, 0x7632);
        a[i] += 1.0f;
      }
    }
    if (OP == 6) {   // tanh.approx.bf16x2 on 4 packed pairs
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        uint32_t r = __float_as_uint(a[i]);
        asm volatile("tanh.approx.bf16x2 %0, %0;" : "+r"(r));
        a[i] = __uint_as_float(r);
      }
    }
    if (OP == 7) {   // tanh.approx.f16x2
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        uint32_t r = __float_as_uint(a[i]);
        asm volatile("tanh.approx.f16x2 %0, %0;" : "+r"(r));
        a[i] = __uint_as_float(r);
      }
    }
  }
  const long long t1 = clock64();
  float s = 0;
  for (int i = 0; i < 8; ++i) s += a[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s + acc;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}

template <int OP>
void run(const char* name, int per_iter) {
  float* out; unsigned long long* cyc;
  cudaMalloc(&out, 1024 * 4 * 148); cudaMalloc(&cyc, 8);
  const int iters = 2000;
  printf("%-28s", name);
  for (int warps : {4, 8, 16, 32}) {      // per block = per SM (1 block per SM): 1, 2, 4, 8 warps per scheduler
    k<OP><<<148, warps * 32>>>(out, iters, cyc);
    cudaDeviceSynchronize();
    k<OP><<<148, warps * 32>>>(out, iters, cyc);
    cudaDeviceSynchronize();
    unsigned long long c; cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
    // cycles per warp-instruction per scheduler = cycles / (iters * per_iter * warps_per_scheduler)
    printf("  %2d w/sched: %6.2f cyc/inst", warps / 4, double(c) / (double(iters) * per_iter * (warps / 4)));
  }
  printf("\n");
  cudaFree(out); cudaFree(cyc);
}

int main() {
  run<0>("tanh.approx.f32", 8);
  run<1>("ex2.approx.ftz.f32", 8);
  run<2>("rcp.approx.ftz.f32", 8);
  run<3>("fma.f32", 8);
  run<4>("cvt.rn.bf16x2.f32 (+xor,add)", 4);
  run<5>("2 iadd + prmt (+xor,add)", 4);
  run<6>("tanh.approx.bf16x2", 4);
  run<7>("tanh.approx.f16x2", 4);
  return 0;
}
