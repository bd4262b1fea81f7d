// l2bench.cu -- ceiling of an "L2-windowed two-kernel" GroupNorm: the statistics pass and the apply pass run as two
// plain streaming kernels over a WINDOW of samples small enough that the apply pass re-reads x from L2 (50 MB on the H100) instead of
// HBM.  HBM traffic is then the cluster kernels' (1 read + 1 write forward; x, dy read + dx written backward) but no CTA holds a
// slab, no cluster barrier, every SM streams.  Prints effective GB/s = algorithmic bytes / time for window sizes 8..96 MB and
// for the unwindowed two-pass baseline (window = whole buffer: the second read comes from HBM).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o build/l2bench tools/l2bench.cu && build/l2bench
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

__device__ __forceinline__ float f4sum(const uint4& v) {
  return __uint_as_float(v.x) + __uint_as_float(v.y) + __uint_as_float(v.z) + __uint_as_float(v.w);
}
// statistics-like pass: read NS streams, reduce, one partial per CTA
template <int NS, int U>
__global__ void __launch_bounds__(256) pass_stats(const uint4* __restrict__ a, const uint4* __restrict__ b, size_t n, float* __restrict__ partial) {
  float acc = 0.f;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + (U - 1) * stride < n; i += U * stride) {
    uint4 va[U], vb[U];
#pragma unroll
    for (int u = 0; u < U; ++u) { va[u] = __ldcg(a + i + u * stride); if (NS > 1) vb[u] = __ldcg(b + i + u * stride); }
#pragma unroll
    for (int u = 0; u < U; ++u) { acc += f4sum(va[u]); if (NS > 1) acc = fmaf(f4sum(vb[u]), 0.5f, acc); }
  }
  for (; i < n; i += stride) { acc += f4sum(__ldcg(a + i)); if (NS > 1) acc += f4sum(__ldcg(b + i)); }
  for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ float s[8];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) { float t = 0.f; for (int w = 0; w < 8; ++w) t += s[w]; partial[blockIdx.x] = t; }
}
// apply-like pass: re-read NS streams (L2 hits when the window fits), a few FMAs, write one stream
template <int NS, int U>
__global__ void __launch_bounds__(256) pass_apply(const uint4* __restrict__ a, const uint4* __restrict__ b, uint4* __restrict__ out, size_t n,
                                                  const float* __restrict__ partial) {
  const float k = partial[0] * 1e-30f + 1.0f;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  auto f = [&](const uint4& x, const uint4& y) {
    uint4 o;
    o.x = __float_as_uint(fmaxf(fmaf(__uint_as_float(x.x), k, NS > 1 ? __uint_as_float(y.x) : 0.1f), 0.f));
    o.y = __float_as_uint(fmaxf(fmaf(__uint_as_float(x.y), k, NS > 1 ? __uint_as_float(y.y) : 0.1f), 0.f));
    o.z = __float_as_uint(fmaxf(fmaf(__uint_as_float(x.z), k, NS > 1 ? __uint_as_float(y.z) : 0.1f), 0.f));
    o.w = __float_as_uint(fmaxf(fmaf(__uint_as_float(x.w), k, NS > 1 ? __uint_as_float(y.w) : 0.1f), 0.f));
    return o;
  };
  for (; i + (U - 1) * stride < n; i += U * stride) {
    uint4 va[U], vb[U];
#pragma unroll
    for (int u = 0; u < U; ++u) { va[u] = __ldcg(a + i + u * stride); if (NS > 1) vb[u] = __ldcg(b + i + u * stride); }
#pragma unroll
    for (int u = 0; u < U; ++u) __stcs(out + i + u * stride, f(va[u], NS > 1 ? vb[u] : va[u]));
  }
  for (; i < n; i += stride) __stcs(out + i, f(__ldcg(a + i), NS > 1 ? __ldcg(b + i) : __ldcg(a + i)));
}

template <int NS>
static void run(const char* name, const unsigned char* a, const unsigned char* b, unsigned char* out, size_t bytes, size_t window, int ctas_per_sm, int sms,
                float* partial, bool streaming_store) {
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  const int grid = sms * ctas_per_sm;
  auto once = [&] {
    for (size_t off = 0; off < bytes; off += window) {
      const size_t w = bytes - off < window ? bytes - off : window;
      pass_stats<NS, 4><<<grid, 256>>>((const uint4*)(a + off), (const uint4*)(b + off), w / 16, partial);
      pass_apply<NS, 4><<<grid, 256>>>((const uint4*)(a + off), (const uint4*)(b + off), (uint4*)(out + off), w / 16, partial);
    }
  };
  once(); CK(cudaDeviceSynchronize());
  float best = 1e30f;
  for (int r = 0; r < 3; ++r) {
    CK(cudaEventRecord(e0)); once(); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); best = ms < best ? ms : best;
  }
  CK(cudaGetLastError());
  const double alg = (double)bytes * (NS + 1);
  printf("%-10s window %6.1f MB  %2d CTA/SM : %7.3f ms  %6.0f GB/s algorithmic (%d read + 1 write)  [%zu launches]\n", name, window / 1048576.0, ctas_per_sm,
         best, alg / best / 1e6, NS, 2 * ((bytes + window - 1) / window));
  cudaEventDestroy(e0); cudaEventDestroy(e1);
}

int main() {
  int dev = 0, sms = 0; CK(cudaGetDevice(&dev)); CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const size_t bytes = (size_t)1 << 30;
  unsigned char *a, *b, *o; float* partial;
  CK(cudaMalloc(&a, bytes)); CK(cudaMalloc(&b, bytes)); CK(cudaMalloc(&o, bytes)); CK(cudaMalloc(&partial, 1 << 20));
  CK(cudaMemset(a, 0, bytes)); CK(cudaMemset(b, 0, bytes)); CK(cudaMemset(o, 0, bytes));
  printf("SMs %d; 1 GiB per stream\n", sms);
  const double mb = 1048576.0;
  for (int ctas : {4, 8}) {
    for (double w : {8.0, 16.0, 24.0, 32.0, 48.0, 64.0, 96.0, 1024.0})
      run<1>("fwd-like", a, b, o, bytes, (size_t)(w * mb), ctas, sms, partial, true);
    for (double w : {4.0, 8.0, 12.0, 16.0, 24.0, 32.0, 48.0, 1024.0})
      run<2>("bwd-like", a, b, o, bytes, (size_t)(w * mb), ctas, sms, partial, true);
  }
  return 0;
}
