// membench.cu -- what does an SM-side access pattern cost?  Diagnostic for the GroupNorm kernels, which sit
// at a fraction of the copy peak whatever the CTA shape, while K1's bulk stores come much closer to it.
// Each pattern moves the same buffers; prints GB/s (bytes read + written).  Standalone:
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o build/membench tools/membench.cu && build/membench
#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(n)); }
__device__ __forceinline__ void mbar_expect(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done)
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- A: LDG read, U independent 16-byte loads in flight per thread ---------------------------------------
template <int U>
__global__ void read_ldg(const uint4* __restrict__ src, size_t n, uint4* sink) {
  uint4 acc = make_uint4(0, 0, 0, 0);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + (U - 1) * stride < n; i += U * stride) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) v[u] = __ldg(src + i + u * stride);
#pragma unroll
    for (int u = 0; u < U; ++u) { acc.x ^= v[u].x; acc.y ^= v[u].y; acc.z ^= v[u].z; acc.w ^= v[u].w; }
  }
  if ((acc.x ^ acc.y ^ acc.z ^ acc.w) == 0x12345678u) *sink = acc;
}
// ---- B: classic copy, U loads in flight ------------------------------------------------------------------
template <int U>
__global__ void copy_ldg(const uint4* __restrict__ src, uint4* __restrict__ dst, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + (U - 1) * stride < n; i += U * stride) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) v[u] = __ldg(src + i + u * stride);
#pragma unroll
    for (int u = 0; u < U; ++u) dst[i + u * stride] = v[u];
  }
}
// ---- C: slab pattern of the cluster GroupNorm kernels: a CTA bulk-loads ONE contiguous slab, waits for all of
//         it, then writes it back (mode 0: 16-byte st.global from ld.shared, mode 1: bulk stores), one slab per CTA
__global__ void slab_copy(const unsigned char* __restrict__ src, unsigned char* __restrict__ dst, uint32_t slab, int mode) {
  extern __shared__ __align__(128) unsigned char sm[];
  const uint32_t bar = smem_u32(sm), buf = smem_u32(sm + 128);
  const size_t off = (size_t)blockIdx.x * slab;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    fence_async();
    mbar_expect(bar, slab);
    for (uint32_t o = 0; o < slab; o += 32768) bulk_g2s(buf + o, src + off + o, slab - o < 32768 ? slab - o : 32768, bar);
  }
  __syncthreads();
  mbar_wait(bar, 0);
  if (mode == 0) {
    const uint4* s = reinterpret_cast<const uint4*>(sm + 128);
    uint4* d = reinterpret_cast<uint4*>(dst + off);
    for (uint32_t i = threadIdx.x; i < slab / 16; i += blockDim.x) d[i] = s[i];
  } else if (threadIdx.x == 0) {
    for (uint32_t o = 0; o < slab; o += 32768) bulk_s2g(dst + off + o, buf + o, slab - o < 32768 ? slab - o : 32768);
    bulk_commit();
    bulk_wait_read0();
  }
}
// ---- D: persistent ring: each CTA walks its slabs with a STAGES-deep ring of `chunk`-byte bulk loads and writes
//         each chunk back as soon as it lands (mode 0 st.global / mode 1 bulk store / mode 2 read only)
template <int STAGES>
__global__ void ring_copy(const unsigned char* __restrict__ src, unsigned char* __restrict__ dst, size_t total, uint32_t chunk, int mode) {
  extern __shared__ __align__(128) unsigned char sm[];
  const uint32_t bars = smem_u32(sm), buf = smem_u32(sm + 128);
  const size_t nchunks = total / chunk;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) mbar_init(bars + 8 * s, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    fence_async();
  }
  __syncthreads();
  size_t issued = blockIdx.x, done = blockIdx.x;
  int is = 0, ds = 0;
  uint32_t dphase = 0;
  if (threadIdx.x == 0)
    for (; is < STAGES && issued < nchunks; ++is, issued += gridDim.x) {
      mbar_expect(bars + 8 * is, chunk);
      bulk_g2s(buf + is * chunk, src + issued * chunk, chunk, bars + 8 * is);
    }
  for (; done < nchunks; done += gridDim.x) {
    mbar_wait(bars + 8 * ds, dphase);
    if (mode == 0) {
      const uint4* s = reinterpret_cast<const uint4*>(sm + 128 + (size_t)ds * chunk);
      uint4* d = reinterpret_cast<uint4*>(dst + done * chunk);
      for (uint32_t i = threadIdx.x; i < chunk / 16; i += blockDim.x) d[i] = s[i];
    } else if (mode == 1 && threadIdx.x == 0) {
      bulk_s2g(dst + done * chunk, buf + ds * chunk, chunk);
      bulk_commit();
      bulk_wait_read0();
    }
    __syncthreads();                       // everyone is done with this stage
    if (threadIdx.x == 0) {
      const size_t nxt = done + (size_t)STAGES * gridDim.x;
      if (nxt < nchunks) {
        fence_async();
        mbar_expect(bars + 8 * ds, chunk);
        bulk_g2s(buf + ds * chunk, src + nxt * chunk, chunk, bars + 8 * ds);
      }
    }
    if (++ds == STAGES) { ds = 0; dphase ^= 1u; }
  }
}

template <typename F>
static float time_ms(F&& launch, int reps = 5) {
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  launch(); CK(cudaDeviceSynchronize());
  CK(cudaEventRecord(a));
  for (int i = 0; i < reps; ++i) launch();
  CK(cudaEventRecord(b));
  CK(cudaEventSynchronize(b));
  CK(cudaGetLastError());
  float ms = 0; CK(cudaEventElapsedTime(&ms, a, b));
  return ms / reps;
}

// ---- E: gn_fwd_cluster_kernel rebuilt step by step on the slab pattern (bf16, [N][P][C], one cluster of CL CTAs
//         per sample, CTA slab = P/CL rows).  STEP 0: cluster launch, slab copy only.  1: + the apply math
//         (unpack, fma, relu, pack).  2: + the statistics pass over the slab in shared memory and a CTA reduction.
//         3: + cluster.sync, DSMEM reduce of the partials, split cluster barrier at the end (= the product kernel).
namespace cg = cooperative_groups;
__device__ __forceinline__ void unpack8(uint4 v, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) { float2 t = __bfloat1622float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 v; __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return v;
}
template <int STEP, int VAR>   // VAR 0: as the product; 1: 4 independent rows per loop trip (ILP); 2: 1 + packed fma.rn.relu.bf16x2 apply
__global__ void __launch_bounds__(512) slab_gn(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int P, int C) {
  extern __shared__ __align__(128) unsigned char sm[];
  cg::cluster_group cluster = cg::this_cluster();
  const int CL = (int)cluster.num_blocks(), rank = (int)cluster.block_rank(), n = blockIdx.x / CL;
  const uint32_t bar = smem_u32(sm);
  float* part = reinterpret_cast<float*>(sm + 64);            // [32][2]
  float* s_stat = reinterpret_cast<float*>(sm + 64 + 256);    // [32][2]
  float* tp = reinterpret_cast<float*>(sm + 1024);            // [threads][2]
  unsigned char* slab = sm + 1024 + 512 * 8;
  const int p0 = (int)(((long long)P * rank) / CL), p1 = (int)(((long long)P * (rank + 1)) / CL), rows = p1 - p0;
  const uint32_t bytes = (uint32_t)rows * C * 2;
  const size_t base = ((size_t)n * P + p0) * C;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    fence_async();
    mbar_expect(bar, bytes);
    for (uint32_t o = 0; o < bytes; o += 32768) bulk_g2s(smem_u32(slab) + o, (const unsigned char*)(x + base) + o, bytes - o < 32768 ? bytes - o : 32768, bar);
  }
  __syncthreads();
  mbar_wait(bar, 0);
  const int cols = C / 8, rpi = (int)blockDim.x / cols, tcol = threadIdx.x % cols, trow = threadIdx.x / cols;
  const uint4* srow = reinterpret_cast<const uint4*>(slab);
  float sa[8], sb[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { sa[i] = 1.0f + 0.001f * i; sb[i] = 0.01f * i; }
  if (STEP >= 2) {
    float a[8], q[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { a[i] = 0.f; q[i] = 0.f; }
    if (VAR == 0) {
      for (int r = trow; r < rows; r += rpi) {
        float f[8]; unpack8(srow[(size_t)r * cols + tcol], f);
#pragma unroll
        for (int i = 0; i < 8; ++i) { a[i] += f[i]; q[i] = fmaf(f[i], f[i], q[i]); }
      }
    } else {
      for (int r0 = trow; r0 < rows; r0 += 4 * rpi) {
        uint4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = r0 + u * rpi < rows ? srow[(size_t)(r0 + u * rpi) * cols + tcol] : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          float f[8]; unpack8(v[u], f);
#pragma unroll
          for (int i = 0; i < 8; ++i) { a[i] += f[i]; q[i] = fmaf(f[i], f[i], q[i]); }
        }
      }
    }
    float ta = 0.f, tq = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { ta += a[i]; tq += q[i]; }
    tp[threadIdx.x * 2] = ta; tp[threadIdx.x * 2 + 1] = tq;
    __syncthreads();
    if (threadIdx.x < 32) {
      float s = 0.f, t = 0.f;
      for (int j = threadIdx.x; j < (int)blockDim.x; j += 32) { s += tp[j * 2]; t += tp[j * 2 + 1]; }
      part[threadIdx.x * 2] = s; part[threadIdx.x * 2 + 1] = t;
    }
    if (STEP >= 3) {
      cluster.sync();
      if (threadIdx.x < 32) {
        float s = 0.f, t = 0.f;
        for (int r = 0; r < CL; ++r) { const float* rp = cluster.map_shared_rank(part, r); s += rp[threadIdx.x * 2]; t += rp[threadIdx.x * 2 + 1]; }
        s_stat[threadIdx.x * 2] = s; s_stat[threadIdx.x * 2 + 1] = t;
      }
      __syncthreads();
      cluster.barrier_arrive();
    } else {
      __syncthreads();
      if (threadIdx.x < 32) { s_stat[threadIdx.x * 2] = part[threadIdx.x * 2]; s_stat[threadIdx.x * 2 + 1] = part[threadIdx.x * 2 + 1]; }
      __syncthreads();
    }
    const float m = s_stat[(tcol & 31) * 2] * 1e-30f, v = s_stat[(tcol & 31) * 2 + 1] * 1e-30f;   // keep the result live, ~0
#pragma unroll
    for (int i = 0; i < 8; ++i) { sa[i] += v; sb[i] -= m; }
  }
  uint4* drow = reinterpret_cast<uint4*>(y + base);
  if (VAR == 0) {
    for (int r = trow; r < rows; r += rpi) {
      uint4 v = srow[(size_t)r * cols + tcol];
      if (STEP >= 1) {
        float f[8]; unpack8(v, f);
#pragma unroll
        for (int i = 0; i < 8; ++i) f[i] = fmaxf(fmaf(sa[i], f[i], sb[i]), 0.f);
        v = pack8(f);
      }
      drow[(size_t)r * cols + tcol] = v;
    }
  } else {
    uint32_t pa[4], pb[4];                                   // scale / shift as bf16x2 (VAR 2)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 ha = __floats2bfloat162_rn(sa[2 * i], sa[2 * i + 1]), hb = __floats2bfloat162_rn(sb[2 * i], sb[2 * i + 1]);
      pa[i] = *reinterpret_cast<uint32_t*>(&ha); pb[i] = *reinterpret_cast<uint32_t*>(&hb);
    }
    for (int r0 = trow; r0 < rows; r0 += 4 * rpi) {
      uint4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = r0 + u * rpi < rows ? srow[(size_t)(r0 + u * rpi) * cols + tcol] : make_uint4(0, 0, 0, 0);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (STEP >= 1) {
          if (VAR == 2) {
            uint32_t* w = reinterpret_cast<uint32_t*>(&v[u]);
#pragma unroll
            for (int i = 0; i < 4; ++i) asm("fma.rn.relu.bf16x2 %0, %1, %2, %3;" : "=r"(w[i]) : "r"(pa[i]), "r"(w[i]), "r"(pb[i]));
          } else {
            float f[8]; unpack8(v[u], f);
#pragma unroll
            for (int i = 0; i < 8; ++i) f[i] = fmaxf(fmaf(sa[i], f[i], sb[i]), 0.f);
            v[u] = pack8(f);
          }
        }
        if (r0 + u * rpi < rows) drow[(size_t)(r0 + u * rpi) * cols + tcol] = v[u];
      }
    }
  }
  if (STEP >= 3) { __syncthreads(); cluster.barrier_wait(); }
}
template <int STEP, int VAR>
static float run_slab_gn(const void* src, void* dst, int N, int P, int C, int CL, int threads, size_t* moved) {
  const size_t slab = (((size_t)((P + CL - 1) / CL)) * C * 2 + 127) / 128 * 128, smem = 1024 + 512 * 8 + slab;
  CK(cudaFuncSetAttribute(slab_gn<STEP, VAR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  if (CL > 8) CK(cudaFuncSetAttribute(slab_gn<STEP, VAR>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(N * CL); cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = smem; cfg.stream = 0;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  *moved = (size_t)2 * N * P * C * 2;
  return time_ms([&] { CK(cudaLaunchKernelEx(&cfg, slab_gn<STEP, VAR>, (const __nv_bfloat16*)src, (__nv_bfloat16*)dst, P, C)); });
}

// ---- F: gn_bwd_cluster_kernel step by step (x slab by TMA into shared memory, dy streamed from global twice with 4
//         loads in flight, dx written).  STEP 0: dx = dy copy with the x slab loaded.  1: + the dx math of pass 2.
//         2: + pass 1 (sum dg, sum dg*xhat) and the CTA reduction.  3: + cluster.sync / DSMEM reduce (= the product).
//         VAR 1: algebraically leaner passes (sum dg*x instead of dg*xhat; dx = fma(dg, rs, fma(x, c1, c0))).
template <int STEP, int VAR>
__global__ void __launch_bounds__(512, 1) slab_gn_bwd(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                                                       __nv_bfloat16* __restrict__ dx, int P, int C) {
  extern __shared__ __align__(128) unsigned char sm[];
  cg::cluster_group cluster = cg::this_cluster();
  const int CL = (int)cluster.num_blocks(), rank = (int)cluster.block_rank(), n = blockIdx.x / CL;
  const uint32_t bar = smem_u32(sm);
  float* part = reinterpret_cast<float*>(sm + 64);
  float* s_stat = reinterpret_cast<float*>(sm + 64 + 256);
  float* tp = reinterpret_cast<float*>(sm + 1024);
  unsigned char* slab = sm + 1024 + 512 * 8;
  const int p0 = (int)(((long long)P * rank) / CL), p1 = (int)(((long long)P * (rank + 1)) / CL), rows = p1 - p0;
  const uint32_t bytes = (uint32_t)rows * C * 2;
  const size_t base = ((size_t)n * P + p0) * C;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    fence_async();
    mbar_expect(bar, bytes);
    for (uint32_t o = 0; o < bytes; o += 32768) bulk_g2s(smem_u32(slab) + o, (const unsigned char*)(x + base) + o, bytes - o < 32768 ? bytes - o : 32768, bar);
  }
  __syncthreads();
  const int cols = C / 8, rpi = (int)blockDim.x / cols, tcol = threadIdx.x % cols, trow = threadIdx.x / cols;
  const uint4* srow = reinterpret_cast<const uint4*>(slab);
  const uint4* gdy = reinterpret_cast<const uint4*>(dy + base);
  uint4* gdx = reinterpret_cast<uint4*>(dx + base);
  float ga[8], sa[8], sb[8];
  const float mu = 0.01f, rs = 1.3f;
#pragma unroll
  for (int i = 0; i < 8; ++i) { ga[i] = 1.0f + 0.01f * i; sa[i] = rs * ga[i]; sb[i] = 0.02f * i - mu * sa[i]; }
  mbar_wait(bar, 0);
  float m1 = 0.001f, m2 = 0.002f;
  if (STEP >= 2) {
    float a[8], q[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { a[i] = 0.f; q[i] = 0.f; }
    for (int r0 = trow; r0 < rows; r0 += 4 * rpi) {
      uint4 vd[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) vd[u] = r0 + u * rpi < rows ? __ldg(gdy + (size_t)(r0 + u * rpi) * cols + tcol) : make_uint4(0, 0, 0, 0);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (r0 + u * rpi < rows) {
          float fx[8], fd[8]; unpack8(srow[(size_t)(r0 + u * rpi) * cols + tcol], fx); unpack8(vd[u], fd);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float pre = fmaf(sa[i], fx[i], sb[i]);
            const float dg = pre > 0.f ? fd[i] * ga[i] : 0.f;
            if (VAR == 0) { const float xh = (fx[i] - mu) * rs; a[i] += dg; q[i] = fmaf(dg, xh, q[i]); }
            else { a[i] += dg; q[i] = fmaf(dg, fx[i], q[i]); }
          }
        }
      }
    }
    float ta = 0.f, tq = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { ta += a[i]; tq += q[i]; }
    tp[threadIdx.x * 2] = ta; tp[threadIdx.x * 2 + 1] = tq;
    __syncthreads();
    if (threadIdx.x < 32) {
      float s = 0.f, t = 0.f;
      for (int j = threadIdx.x; j < (int)blockDim.x; j += 32) { s += tp[j * 2]; t += tp[j * 2 + 1]; }
      part[threadIdx.x * 2] = s; part[threadIdx.x * 2 + 1] = t;
    }
    if (STEP >= 3) {
      cluster.sync();
      if (threadIdx.x < 32) {
        float s = 0.f, t = 0.f;
        for (int r = 0; r < CL; ++r) { const float* rp = cluster.map_shared_rank(part, r); s += rp[threadIdx.x * 2]; t += rp[threadIdx.x * 2 + 1]; }
        s_stat[threadIdx.x * 2] = s; s_stat[threadIdx.x * 2 + 1] = t;
      }
      __syncthreads();
      cluster.barrier_arrive();
    } else {
      __syncthreads();
      if (threadIdx.x < 32) { s_stat[threadIdx.x * 2] = part[threadIdx.x * 2]; s_stat[threadIdx.x * 2 + 1] = part[threadIdx.x * 2 + 1]; }
      __syncthreads();
    }
    m1 += s_stat[(tcol & 31) * 2] * 1e-30f; m2 += s_stat[(tcol & 31) * 2 + 1] * 1e-30f;
  }
  const float c1 = -rs * rs * m2, c0 = -rs * m1 - c1 * mu;      // VAR 1: dx = rs*dg + c1*x + c0
  for (int r0 = trow; r0 < rows; r0 += 4 * rpi) {
    uint4 vd[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) vd[u] = r0 + u * rpi < rows ? __ldg(gdy + (size_t)(r0 + u * rpi) * cols + tcol) : make_uint4(0, 0, 0, 0);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (r0 + u * rpi < rows) {
        uint4 out = vd[u];
        if (STEP >= 1) {
          float fx[8], fd[8], fo[8]; unpack8(srow[(size_t)(r0 + u * rpi) * cols + tcol], fx); unpack8(vd[u], fd);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float pre = fmaf(sa[i], fx[i], sb[i]);
            const float dg = pre > 0.f ? fd[i] * ga[i] : 0.f;
            if (VAR == 0) { const float xh = (fx[i] - mu) * rs; fo[i] = rs * (dg - m1 - xh * m2); }
            else fo[i] = fmaf(dg, rs, fmaf(fx[i], c1, c0));
          }
          out = pack8(fo);
        }
        gdx[(size_t)(r0 + u * rpi) * cols + tcol] = out;
      }
    }
  }
  if (STEP >= 3) { __syncthreads(); cluster.barrier_wait(); }
}
template <int STEP, int VAR>
static float run_slab_gn_bwd(const void* x, const void* dy, void* dx, int N, int P, int C, int CL, int threads, size_t* moved) {
  const size_t slab = (((size_t)((P + CL - 1) / CL)) * C * 2 + 127) / 128 * 128, smem = 1024 + 512 * 8 + slab;
  CK(cudaFuncSetAttribute(slab_gn_bwd<STEP, VAR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  if (CL > 8) CK(cudaFuncSetAttribute(slab_gn_bwd<STEP, VAR>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(N * CL); cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = smem; cfg.stream = 0;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  *moved = (size_t)3 * N * P * C * 2;                            // x + dy + dx (the second dy read is expected from L2)
  return time_ms([&] { CK(cudaLaunchKernelEx(&cfg, slab_gn_bwd<STEP, VAR>, (const __nv_bfloat16*)x, (const __nv_bfloat16*)dy, (__nv_bfloat16*)dx, P, C)); });
}

int main() {
  const size_t bytes = (size_t)1 << 30;                 // 1 GiB in, 1 GiB out (>> L2)
  unsigned char *src, *dst; uint4* sink;
  CK(cudaMalloc(&src, bytes)); CK(cudaMalloc(&dst, bytes)); CK(cudaMalloc(&sink, 16));
  CK(cudaMemset(src, 1, bytes)); CK(cudaMemset(dst, 0, bytes));
  int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  const size_t n16 = bytes / 16;
  auto gbs = [&](double moved, float ms) { return moved / ms / 1e6; };
  printf("SMs %d, buffer %zu MiB\n", sms, bytes >> 20);
  { float ms = time_ms([&] { CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice)); }); printf("cudaMemcpy D2D                         %8.0f GB/s\n", gbs(2.0 * bytes, ms)); }
  { float ms = time_ms([&] { CK(cudaMemsetAsync(dst, 0, bytes)); }); printf("cudaMemset                             %8.0f GB/s (write only)\n", gbs(1.0 * bytes, ms)); }
#define RD(U, CTAS) { float ms = time_ms([&] { read_ldg<U><<<sms * CTAS, 256>>>((const uint4*)src, n16, sink); }); printf("read  ldg  U=%d  %2d CTA/SM x256          %8.0f GB/s (read only)\n", U, CTAS, gbs(1.0 * bytes, ms)); }
  RD(1, 8) RD(4, 8) RD(8, 8) RD(8, 4) RD(8, 2)
#define CP(U, CTAS) { float ms = time_ms([&] { copy_ldg<U><<<sms * CTAS, 256>>>((const uint4*)src, (uint4*)dst, n16); }); printf("copy  ldg  U=%d  %2d CTA/SM x256          %8.0f GB/s\n", U, CTAS, gbs(2.0 * bytes, ms)); }
  CP(1, 8) CP(4, 8) CP(8, 8) CP(8, 4)
  for (int mode = 0; mode < 2; ++mode)
    for (uint32_t slab : {49152u, 98304u, 200704u}) {
      for (int threads : {256, 512}) {
        const size_t smem = slab + 128;
        CK(cudaFuncSetAttribute(slab_copy, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const int grid = (int)(bytes / slab);
        float ms = time_ms([&] { slab_copy<<<grid, threads, smem>>>(src, dst, slab, mode); });
        printf("slab  %6u B x%3d thr  %s        %8.0f GB/s\n", slab, threads, mode ? "bulk store" : "st.global ", gbs(2.0 * (double)grid * slab, ms));
      }
    }
  for (int mode = 0; mode < 3; ++mode)
    for (uint32_t chunk : {16384u, 32768u}) {
      for (int ctas : {1, 2}) {
        const size_t smem = (size_t)4 * chunk + 128;
        CK(cudaFuncSetAttribute(ring_copy<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        float ms = time_ms([&] { ring_copy<4><<<sms * ctas, 256, smem>>>(src, dst, bytes, chunk, mode); });
        const char* nm = mode == 0 ? "st.global " : (mode == 1 ? "bulk store" : "read only ");
        printf("ring4 %6u B  %d CTA/SM  %s        %8.0f GB/s\n", chunk, ctas, nm, gbs((mode == 2 ? 1.0 : 2.0) * bytes, ms));
      }
    }
  // gn_fwd_cluster_kernel step by step: the two dominant shapes of the bench (chunk of 256 samples)
  struct Shape { int P, C, CL, threads; } shapes[] = {{3136, 256, 8, 512}, {3136, 256, 8, 256}, {3136, 256, 16, 256}, {3136, 64, 4, 256}, {784, 512, 8, 256}};
  for (auto& sh : shapes) {
    const int N = (int)(bytes / ((size_t)sh.P * sh.C * 2));
    size_t moved = 0; float ms;
    ms = run_slab_gn<0, 0>(src, dst, N, sh.P, sh.C, sh.CL, sh.threads, &moved); printf("gn P=%4d C=%4d cl%-2d x%3d  0 copy            %8.0f GB/s\n", sh.P, sh.C, sh.CL, sh.threads, gbs((double)moved, ms));
    ms = run_slab_gn<1, 0>(src, dst, N, sh.P, sh.C, sh.CL, sh.threads, &moved); printf("gn P=%4d C=%4d cl%-2d x%3d  1 + apply math    %8.0f GB/s\n", sh.P, sh.C, sh.CL, sh.threads, gbs((double)moved, ms));
    ms = run_slab_gn<2, 0>(src, dst, N, sh.P, sh.C, sh.CL, sh.threads, &moved); printf("gn P=%4d C=%4d cl%-2d x%3d  2 + statistics    %8.0f GB/s\n", sh.P, sh.C, sh.CL, sh.threads, gbs((double)moved, ms));
    ms = run_slab_gn<3, 0>(src, dst, N, sh.P, sh.C, sh.CL, sh.threads, &moved); printf("gn P=%4d C=%4d cl%-2d x%3d  3 + cluster reduce %7.0f GB/s\n", sh.P, sh.C, sh.CL, sh.threads, gbs((double)moved, ms));
    ms = run_slab_gn<3, 1>(src, dst, N, sh.P, sh.C, sh.CL, sh.threads, &moved); printf("gn P=%4d C=%4d cl%-2d x%3d  3, 4 rows per trip  %7.0f GB/s\n", sh.P, sh.C, sh.CL, sh.threads, gbs((double)moved, ms));
    ms = run_slab_gn<3, 2>(src, dst, N, sh.P, sh.C, sh.CL, sh.threads, &moved); printf("gn P=%4d C=%4d cl%-2d x%3d  3, + bf16x2 apply   %7.0f GB/s\n", sh.P, sh.C, sh.CL, sh.threads, gbs((double)moved, ms));
  }
  // gn_bwd_cluster_kernel step by step (third buffer = dy)
  unsigned char* src2; CK(cudaMalloc(&src2, bytes)); CK(cudaMemset(src2, 2, bytes));
  Shape bshapes[] = {{3136, 256, 8, 512}, {3136, 256, 16, 256}, {784, 512, 8, 256}};
  for (auto& sh : bshapes) {
    const int N = (int)(bytes / ((size_t)sh.P * sh.C * 2));
    size_t moved = 0; float ms;
#define BW(STEP, VAR, NAME) ms = run_slab_gn_bwd<STEP, VAR>(src, src2, dst, N, sh.P, sh.C, sh.CL, sh.threads, &moved); \
    printf("gn bwd P=%4d C=%4d cl%-2d x%3d  %-28s %7.0f GB/s\n", sh.P, sh.C, sh.CL, sh.threads, NAME, gbs((double)moved, ms));
    BW(0, 0, "0 copy (x slab, dy -> dx)") BW(1, 0, "1 + dx math") BW(2, 0, "2 + pass 1 sums") BW(3, 0, "3 + cluster reduce") BW(3, 1, "3, leaner algebra")
  }
  return 0;
}
