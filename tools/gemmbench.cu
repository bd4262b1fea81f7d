// gemmbench.cu -- per-layer time of the wgmma GroupNorm-prologue 1x1-convolution GEMM (kernels_gemm.cu) on every fused
// ResNetV2-50 shape at 224 px: norm1 -> conv1 (blocks without a downsample branch) and norm3 -> conv3 (+ shortcut).
// Prints ms, algorithmic GB/s (x read once + out written (+ shortcut read) + weights) and TFLOP/s per shape, plus the
// statistics pass in front of it.  Buffers rotate over > 300 MB so that no launch finds its operands in L2.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o gemmbench tools/gemmbench.cu \
//        -Ldorpatch_b200/lib -ldorpatch -Xlinker -rpath,$PWD/dorpatch_b200/lib
//   ./gemmbench [N]
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../dorpatch_b200/csrc/kernels.h"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA %s at %d: %s\n", #x, __LINE__, cudaGetErrorString(e_)); exit(1); } } while (0)

struct Shape { int P, K, Nout; bool shortcut; int count; const char* name; };

int main(int argc, char** argv) {
  const int N = argc > 1 ? atoi(argv[1]) : 256;
  const Shape shapes[] = {
      {3136, 64, 256, true, 3, "s1 conv3"}, {3136, 256, 64, false, 2, "s1 conv1"},
      {784, 128, 512, true, 4, "s2 conv3"}, {784, 512, 128, false, 3, "s2 conv1"},
      {196, 256, 1024, true, 6, "s3 conv3"}, {196, 1024, 256, false, 5, "s3 conv1"},
      {49, 512, 2048, true, 3, "s4 conv3"}, {49, 2048, 512, false, 2, "s4 conv1"},
  };
  cudaStream_t st; CK(cudaStreamCreate(&st));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  double tot_ms = 0, tot_stats = 0, tot_bytes = 0;
  for (const Shape& s : shapes) {
    if (!dp::gn_gemm_supported(s.P, s.K, s.Nout)) { printf("%-9s unsupported\n", s.name); continue; }
    const size_t M = (size_t)N * s.P;
    const size_t xb = M * s.K * 2, ob = M * s.Nout * 2;
    int R = (int)((320ull << 20) / (xb + ob)) + 1;
    if (R > 16) R = 16;
    if (R < 2) R = 2;
    __nv_bfloat16 *x, *out, *res, *w, *wp;
    float *stats, *gamma, *beta, *partial;
    CK(cudaMalloc(&x, xb * R)); CK(cudaMalloc(&out, ob * R)); CK(cudaMalloc(&res, ob * R));
    CK(cudaMalloc(&w, (size_t)s.Nout * s.K * 2)); CK(cudaMalloc(&wp, (size_t)s.Nout * s.K * 2));
    CK(cudaMalloc(&stats, (size_t)N * 64 * 4)); CK(cudaMalloc(&gamma, s.K * 4)); CK(cudaMalloc(&beta, s.K * 4));
    CK(cudaMalloc(&partial, ((size_t)N * dp::GN_WS_FLOATS_PER_SAMPLE + dp::GN_WS_FLOATS_EXTRA) * 4));
    CK(cudaMemset(x, 0x3c, xb * R)); CK(cudaMemset(res, 0x3c, ob * R)); CK(cudaMemset(w, 0x3c, (size_t)s.Nout * s.K * 2));
    std::vector<float> ones(s.K, 1.0f), zeros(s.K, 0.0f);
    CK(cudaMemcpy(gamma, ones.data(), s.K * 4, cudaMemcpyHostToDevice)); CK(cudaMemcpy(beta, zeros.data(), s.K * 4, cudaMemcpyHostToDevice));
    dp::launch_gn_gemm_pack(w, wp, s.Nout, s.K, st);
    dp::launch_gn_stats(x, partial, stats, N, s.P, s.K, true, st);
    CK(cudaStreamSynchronize(st));
    auto gemm = [&](int r) {
      dp::launch_gn_gemm_forward((char*)x + xb * r, wp, stats, gamma, beta, s.shortcut ? (char*)res + ob * r : nullptr, (char*)out + ob * r, N, s.P, s.K, s.Nout, st);
    };
    auto statsf = [&](int r) { dp::launch_gn_stats((char*)x + xb * r, partial, stats, N, s.P, s.K, true, st); };
    auto time_it = [&](auto&& f) {
      for (int r = 0; r < R; ++r) f(r);
      CK(cudaStreamSynchronize(st));
      const int reps = 3 * R;
      CK(cudaEventRecord(e0, st));
      for (int i = 0; i < reps; ++i) f(i % R);
      CK(cudaEventRecord(e1, st));
      CK(cudaEventSynchronize(e1));
      float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
      return ms / reps;
    };
    const float tg = time_it(gemm), ts = time_it(statsf);
    CK(cudaGetLastError());
    const double bytes = (double)xb + ob * (s.shortcut ? 2.0 : 1.0) + (double)s.Nout * s.K * 2;
    const double flops = 2.0 * M * s.K * s.Nout;
    printf("%-9s P=%4d K=%4d Nout=%4d x%d | gemm %7.3f ms %5.0f GB/s %6.1f TF/s | stats %7.3f ms %5.0f GB/s | per step (x%d): %.3f + %.3f ms\n", s.name, s.P, s.K,
           s.Nout, s.count, tg, bytes / tg / 1e6, flops / tg / 1e9, ts, (double)xb / ts / 1e6, s.count, tg * s.count, ts * s.count);
    fflush(stdout);
    tot_ms += tg * s.count; tot_stats += ts * s.count; tot_bytes += bytes * s.count;
    cudaFree(x); cudaFree(out); cudaFree(res); cudaFree(w); cudaFree(wp); cudaFree(stats); cudaFree(gamma); cudaFree(beta); cudaFree(partial);
  }
  printf("all fused layers, N=%d: gemm %.3f ms (%.0f GB/s algorithmic), statistics passes %.3f ms\n", N, tot_ms, tot_bytes / tot_ms / 1e6, tot_stats);
  return 0;
}
