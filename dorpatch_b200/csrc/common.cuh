// common.cuh -- shared device helpers for the DorPatch sm_90a kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace dp {

// ----------------------------------------------------------------------------
// 16-byte vector of activation elements: 4 x fp32 or 8 x bf16.
// ----------------------------------------------------------------------------
template <typename T> struct Vec;
template <> struct Vec<float> {
  static constexpr int N = 4;
  float4 raw;
  __device__ __forceinline__ void load(const float* p) { raw = *reinterpret_cast<const float4*>(p); }
  __device__ __forceinline__ void store(float* p) const { *reinterpret_cast<float4*>(p) = raw; }
  __device__ __forceinline__ void load_shared(uint32_t a) {   // 32-bit shared-window address
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(raw.x), "=f"(raw.y), "=f"(raw.z), "=f"(raw.w) : "r"(a));
  }
  __device__ __forceinline__ void unpack(float* f) const { f[0] = raw.x; f[1] = raw.y; f[2] = raw.z; f[3] = raw.w; }
  __device__ __forceinline__ void pack(const float* f) { raw = make_float4(f[0], f[1], f[2], f[3]); }
};
template <> struct Vec<__nv_bfloat16> {
  static constexpr int N = 8;
  uint4 raw;
  __device__ __forceinline__ void load(const __nv_bfloat16* p) { raw = *reinterpret_cast<const uint4*>(p); }
  __device__ __forceinline__ void store(__nv_bfloat16* p) const { *reinterpret_cast<uint4*>(p) = raw; }
  __device__ __forceinline__ void load_shared(uint32_t a) {
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(raw.x), "=r"(raw.y), "=r"(raw.z), "=r"(raw.w) : "r"(a));
  }
  __device__ __forceinline__ void unpack(float* f) const {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 t = __bfloat1622float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
  }
  __device__ __forceinline__ void pack(const float* f) {
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&raw);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  }
};

template <typename T> __device__ __forceinline__ T from_float(float v);
template <> __device__ __forceinline__ float from_float<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_float<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
__device__ __forceinline__ float to_float(float v) { return v; }
__device__ __forceinline__ float to_float(__nv_bfloat16 v) { return __bfloat162float(v); }

// ----------------------------------------------------------------------------
// reductions
// ----------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Deterministic block-wide sum (fixed shuffle tree + fixed-order final loop).
// `red` must hold >= 32 floats of shared memory.  All threads get the result.
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  float t = 0.f;
  for (int i = 0; i < nw; ++i) t += red[i];
  return t;
}

__device__ __forceinline__ float sgn(float v) { return (float)(v > 0.f) - (float)(v < 0.f); }  // sgn(NaN) = 0, as torch.sign

}  // namespace dp
