// Dev tool (no GPU needed): run conv_gemm_build's host-side tiling / shared-memory budget over the conv shapes of the
// detector and the CLIP linears with a stub tensor-map encoder, and print the configuration each one gets.
//   nvcc -gencode arch=compute_90a,code=sm_90a -std=c++17 --expt-relaxed-constexpr -I clearcam_b200/csrc -I include \
//        -o /tmp/hbc tests/tools/host_budget_check.cu && /tmp/hbc
#include "../../clearcam_b200/csrc/conv_gemm.cu"
#include <stdarg.h>
namespace cc {
static char g_err[1024];
void set_error(const char* fmt, ...) { va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap); }
const char* last_error() { return g_err; }
static CUresult fake_enc(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                         const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill) {
  return CUDA_SUCCESS;
}
PFN_encodeTiled get_encode_tiled() { return fake_enc; }
int device_sm_count() { return 132; }   // H100 SXM
}
using namespace cc;
int main() {
  struct S { int N, H, W, Cin, Cout, k, s, f32, res; };
  const S shapes[] = {
      {1, 1, 32 * 320 * 320, 32, 64, 1, 1, 0, 0}, {32, 320, 320, 64, 128, 3, 2, 0, 0}, {32, 160, 160, 128, 128, 1, 1, 0, 0},
      {32, 160, 160, 64, 64, 1, 1, 0, 0},  {32, 160, 160, 32, 32, 3, 1, 0, 0},  {32, 160, 160, 32, 32, 3, 1, 0, 1},
      {32, 160, 160, 64, 64, 3, 1, 0, 0},  {32, 160, 160, 256, 256, 1, 1, 0, 0}, {32, 160, 160, 128, 128, 3, 2, 0, 0},
      {32, 80, 80, 128, 128, 1, 1, 0, 0},  {32, 80, 80, 64, 64, 3, 1, 0, 1},    {32, 80, 80, 128, 128, 3, 1, 0, 0},
      {32, 80, 80, 512, 512, 1, 1, 0, 0},  {32, 80, 80, 256, 256, 3, 2, 0, 0},  {32, 40, 40, 256, 256, 1, 1, 0, 0},
      {32, 40, 40, 128, 128, 3, 1, 0, 1},  {32, 40, 40, 256, 256, 3, 1, 0, 0},  {32, 40, 40, 1024, 512, 1, 1, 0, 0},
      {32, 20, 20, 256, 256, 3, 1, 0, 0},  {32, 20, 20, 128, 128, 3, 1, 0, 1},  {32, 20, 20, 1024, 512, 1, 1, 0, 0},
      {32, 80, 80, 256, 320, 3, 1, 0, 0},  {32, 80, 80, 64, 64, 3, 1, 0, 0},    {32, 80, 80, 64, 64, 1, 1, 1, 0},
      {32, 80, 80, 256, 80, 1, 1, 1, 0},   {32, 40, 40, 512, 320, 3, 1, 0, 0},  {32, 20, 20, 512, 320, 3, 1, 0, 0},
      {8, 20, 20, 512, 256, 3, 1, 0, 0},   {1, 40, 40, 256, 256, 3, 1, 0, 0},   {2, 20, 20, 64, 96, 3, 1, 0, 0},
      {3, 33, 21, 48, 16, 3, 1, 0, 0},     {2, 20, 20, 64, 16, 1, 1, 1, 0},
      // CLIP linears (rows = B*L)
      {1, 1, 256 * 50, 768, 2304, 1, 1, 0, 0}, {1, 1, 256 * 50, 768, 768, 1, 1, 1, 1}, {1, 1, 256 * 50, 768, 3072, 1, 1, 0, 0},
      {1, 1, 256 * 50, 3072, 768, 1, 1, 1, 1}, {1, 1, 64 * 257, 1024, 3072, 1, 1, 0, 0}, {1, 1, 64 * 257, 4096, 1024, 1, 1, 1, 1},
      // precise mode: 6 planes
      {32, 160, 160, 192, 32, 3, 1, 1, 0}, {32, 160, 160, 384, 64, 3, 1, 1, 0}, {32, 40, 40, 1536, 256, 3, 1, 1, 0},
      {32, 40, 40, 6144, 512, 1, 1, 1, 0}, {32, 160, 160, 768, 128, 3, 2, 1, 0}};
  static float dummy[64];
  int bad = 0;
  printf("%-34s %4s %3s %2s %4s %7s %6s %6s\n", "shape", "BN", "BK", "S", "bres", "smem", "tiles", "grid");
  for (const S& q : shapes) {
    const TSlice out = nhwc_slice(dummy, q.Cout, 0, q.Cout, q.f32);
    const ConvDesc d = conv_desc(nhwc_slice(dummy, q.Cin, 0, q.Cin, 0, q.N, q.H, q.W), dummy, dummy, q.k, q.s, out, 1, q.res ? &out : nullptr);
    GemmLaunch L;
    char name[96];
    snprintf(name, sizeof(name), "%dx%dx%d %d->%d k%d s%d %s%s", q.N, q.H, q.W, q.Cin, q.Cout, q.k, q.s, q.f32 ? "f32" : "bf16", q.res ? "+res" : "");
    int rc = conv_gemm_build(d, device_sm_count(), &L);
    if (rc) { printf("%-34s FAILED: %s\n", name, last_error()); ++bad; continue; }
    const GemmParams& p = L.p;
    printf("%-34s %4d %3d %2d %4d %7d %6d %6d\n", name, p.BN, p.BK, p.stages, p.b_res, L.smem_bytes, p.num_tiles, L.grid);
    if (L.smem_bytes > kMaxSmem) { printf("   ^^^ exceeds shared memory\n"); ++bad; }
  }
  return bad ? 1 : 0;
}
