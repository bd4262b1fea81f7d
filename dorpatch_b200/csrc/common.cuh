// common.cuh -- shared device helpers for the DorPatch sm_90a kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"

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

// ----------------------------------------------------------------------------
// EOT samples are image-major: sample s belongs to image s / S.  A launch over samples [n0, n0 + n) touches
// images_touched() images; its i-th image is b, whose samples in the launch are [lo, hi).  first: lo is b's first
// sample, so the launch writes b's result rather than adding to it.
// ----------------------------------------------------------------------------
__host__ __device__ __forceinline__ int images_touched(int S, int n0, int n) {
  const int first = n0 / S, last = (n0 + n - 1) / S;
  return last - first + 1;
}
struct ImageSpan {
  int b, lo, hi;
  bool first;
};
__device__ __forceinline__ ImageSpan image_span(int S, int n0, int n, int i) {
  const int b = n0 / S + i;
  const int lo = max(n0, b * S), hi = min(n0 + n, (b + 1) * S);
  return ImageSpan{b, lo, hi, lo == b * S};
}

// ----------------------------------------------------------------------------
// Occlusion table: the only place its format is decoded.  A sample's row is RECT_SHORTS int16, four rectangles
// {r0, r1, c0, c1}: rectangle k occludes rows [r0, r1) x columns [c0, c1) (half-open), and is empty when r1 <= r0 or
// c1 <= c0 (unused slots are all zero).  A pixel is occluded when any rectangle covers it.  A row is 32 bytes: two
// 16-byte words.
// ----------------------------------------------------------------------------
namespace occl {
struct Words { int4 q0, q1; };   // one sample's row as read
// sample n's row as two 16-byte words (also for a block-wide copy into shared memory)
__device__ __forceinline__ const int4* row(const int16_t* rects, int n) {
  return reinterpret_cast<const int4*>(rects + (size_t)n * RECT_SHORTS);
}
// from the table in global memory (the same address in every lane of a warp is a broadcast)
__device__ __forceinline__ Words load(const int16_t* rects, int n) {
  const int4* p = row(rects, n);
  return Words{__ldg(p), __ldg(p + 1)};
}
// from a copy of row() in shared memory
__device__ __forceinline__ Words load_shared(const int4* s) { return Words{s[0], s[1]}; }
// r: one sample's row, in registers or shared memory
__device__ __forceinline__ bool hit(const short* r, int row, int col) {
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (row >= r[4 * k] && row < r[4 * k + 1] && col >= r[4 * k + 2] && col < r[4 * k + 3]) return true;
  return false;
}
}  // namespace occl

// one sample's rectangles in registers
struct Occlusion {
  short r[RECT_SHORTS];
  Occlusion() = default;
  __device__ __forceinline__ explicit Occlusion(occl::Words w) { set(w); }
  __device__ __forceinline__ void set(occl::Words w) {
    *reinterpret_cast<int4*>(r) = w.q0;
    *reinterpret_cast<int4*>(r + 8) = w.q1;
  }
  __device__ __forceinline__ bool hit(int row, int col) const { return occl::hit(r, row, col); }
  // Rectangle k as the rows [rlo, rhi) it covers and, in a row of `cp` elements per pixel, the elements [elo, ehi).
  // A rectangle with no columns covers no row (rlo = rhi = 0); one with no rows has rhi <= rlo.
  __device__ __forceinline__ void span(int k, int cp, int& rlo, int& rhi, int& elo, int& ehi) const {
    const int* w = reinterpret_cast<const int*>(r);   // {r0, r1} and {c0, c1}, each one 32-bit word (r0, c0 low)
    rlo = (short)(w[2 * k] & 0xffff); rhi = (short)(w[2 * k] >> 16);
    elo = (short)(w[2 * k + 1] & 0xffff) * cp; ehi = (short)(w[2 * k + 1] >> 16) * cp;
    if (ehi <= elo) { rlo = 0; rhi = 0; }
  }
};

// ----------------------------------------------------------------------------
// Occlusion bank (MaskBank, kernels.h): the only place its format is decoded.  Mask m is H rows of words(W) uint32;
// bit w % 32 of word w / 32 of row h set = pixel (h, w) occluded.  A sample selects two masks (idx[n], -1 = none) and
// is occluded where either is set.
// ----------------------------------------------------------------------------
namespace occl_bank {
__device__ __forceinline__ int words(int W) { return bank_words(W); }
// sample n's two mask indices
__device__ __forceinline__ int2 select(const MaskBank& b, int n) { return __ldg(reinterpret_cast<const int2*>(b.idx) + n); }
// word k of row h of the occlusion of a sample that selected `sel`
__device__ __forceinline__ uint32_t row_bits(const MaskBank& b, int2 sel, int h, int k) {
  const size_t mw = (size_t)b.H * words(b.W), o = (size_t)h * words(b.W) + k;
  uint32_t v = 0u;
  if (sel.x >= 0) v |= __ldg(b.bits + sel.x * mw + o);
  if (sel.y >= 0) v |= __ldg(b.bits + sel.y * mw + o);
  return v;
}
__device__ __forceinline__ bool hit(const MaskBank& b, int2 sel, int h, int w) {
  return (row_bits(b, sel, h, w >> 5) >> (w & 31)) & 1u;
}
}  // namespace occl_bank

}  // namespace dp
