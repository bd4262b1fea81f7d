// kernels_wgrad.cu -- hand-written sm_90a kernels of the classifier's weight-gradient pass (dp_eot_backward_params).
//
// The 1x1 / 3x3 / fp32 stem weight gradients run through cublasLt / cuDNN in the engine; what is here is the rest:
//   - relu(gn(x)) re-applied from the saved statistics (the convolutions' inputs, which the forward does not keep),
//   - GroupNorm affine gradients: per-sample partials, then a fixed-order column sum (no atomics),
//   - the bf16 stem weight gradient on the tight C=3 input (mma.sync m16n8k16, fp32 accumulate), per-CTA partials
//     reduced in a fixed order,
//   - the weight-standardisation adjoint (timm StdConv2d, eps 1e-8) from the fp32 raw weights, KRSC -> OIHW.
// Every reduction runs in an order fixed by the shapes alone, so a configuration gives the same bits on every run.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "kernels.h"

namespace dp {

#define WG_DISPATCH_T(bf16, ...)                      \
  do {                                                \
    if (bf16) { using T = __nv_bfloat16; __VA_ARGS__; } \
    else { using T = float; __VA_ARGS__; }            \
  } while (0)

// ---------------------------------------------------------------------------------------------------------------
// y = relu(gamma * (x - mean) * rstd + beta) with the forward's (mean, rstd) and its arithmetic (sa, sb folding)
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void gn_apply_kernel(const T* __restrict__ x, T* __restrict__ y, const float* __restrict__ gamma,
                                const float* __restrict__ beta, const float* __restrict__ stats, int P, int C, size_t total) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % C);
  const size_t n = i / ((size_t)P * C);
  const int g = c / (C / GN_GROUPS);
  const float mean = stats[(n * GN_GROUPS + g) * 2], rstd = stats[(n * GN_GROUPS + g) * 2 + 1];
  const float sa = rstd * gamma[c], sb = beta[c] - mean * sa;
  y[i] = from_float<T>(fmaxf(fmaf(sa, to_float(x[i]), sb), 0.f));
}

int launch_gn_apply(const void* x, void* y, const float* gamma, const float* beta, const float* stats, int N, int P,
                    int C, bool bf16, cudaStream_t st) {
  const size_t total = (size_t)N * P * C;
  WG_DISPATCH_T(bf16, (gn_apply_kernel<T><<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const T*)x, (T*)y, gamma, beta,
                                                                                            stats, P, C, total)));
  return 1;
}

// ---------------------------------------------------------------------------------------------------------------
// GroupNorm affine gradients, per sample: partial[n][c] = sum_p dyg * xhat, partial[n][C + c] = sum_p dyg, where
// dyg = dy gated by the ReLU (gamma * xhat + beta > 0, the gate of the input-gradient kernels).
// CTA = 32 channels x 8 pixel rows of one sample; the 8 row sums are combined in a fixed order.
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) gn_affine_partial_kernel(const T* __restrict__ dy, const T* __restrict__ x,
                                                                const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                const float* __restrict__ stats, float* __restrict__ partial,
                                                                int P, int C) {
  __shared__ float sa_[8][33], sb_[8][33];
  const int n = blockIdx.y, tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  float a = 0.f, b = 0.f;
  if (c < C) {
    const int g = c / (C / GN_GROUPS);
    const float mean = stats[((size_t)n * GN_GROUPS + g) * 2], rstd = stats[((size_t)n * GN_GROUPS + g) * 2 + 1];
    const float s1 = rstd * gamma[c], s0 = beta[c] - mean * s1;
    const T* xs = x + (size_t)n * P * C + c;
    const T* ds = dy + (size_t)n * P * C + c;
    for (int p = ty; p < P; p += 8) {
      const float xv = to_float(xs[(size_t)p * C]);
      const float d = fmaf(s1, xv, s0) > 0.f ? to_float(ds[(size_t)p * C]) : 0.f;
      a = fmaf(d, (xv - mean) * rstd, a);
      b += d;
    }
  }
  sa_[ty][tx] = a; sb_[ty][tx] = b;
  __syncthreads();
  if (ty == 0 && c < C) {
    float ta = 0.f, tb = 0.f;
#pragma unroll
    for (int r = 0; r < 8; ++r) { ta += sa_[r][tx]; tb += sb_[r][tx]; }
    partial[(size_t)n * 2 * C + c] = ta;
    partial[(size_t)n * 2 * C + C + c] = tb;
  }
}

int launch_gn_affine_partial(const void* dy, const void* x, const float* gamma, const float* beta, const float* stats,
                             float* partial, int N, int P, int C, bool bf16, cudaStream_t st) {
  dim3 grid((C + 31) / 32, N);
  WG_DISPATCH_T(bf16, (gn_affine_partial_kernel<T><<<grid, 256, 0, st>>>((const T*)dy, (const T*)x, gamma, beta, stats,
                                                                          partial, P, C)));
  return 1;
}

// acc[j] += sum_{r < rows} src[r * M + j], rows summed in order
__global__ void colsum_add_kernel(const float* __restrict__ src, float* __restrict__ acc, int rows, int M) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= M) return;
  float s = 0.f;
  for (int r = 0; r < rows; ++r) s += src[(size_t)r * M + j];
  acc[j] += s;
}

int launch_colsum_add(const float* src, float* acc, int rows, int M, cudaStream_t st) {
  colsum_add_kernel<<<(M + 255) / 256, 256, 0, st>>>(src, acc, rows, M);
  return 1;
}

__global__ void add_bf16_kernel(const __nv_bfloat16* __restrict__ src, float* __restrict__ acc, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) acc[i] += __bfloat162float(src[i]);
}

int launch_add_bf16(const void* src, float* acc, size_t n, cudaStream_t st) {
  add_bf16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const __nv_bfloat16*)src, acc, n);
  return 1;
}

// out[i] = (accumulate ? out[i] : 0) + a[i] (+ b[i])
__global__ void vec_finish_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out,
                                  size_t n, int accumulate) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float v = a[i];
  if (b) v += b[i];
  out[i] = accumulate ? out[i] + v : v;
}

int launch_vec_finish(const float* a, const float* b, float* out, size_t n, bool accumulate, cudaStream_t st) {
  vec_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, b, out, n, accumulate ? 1 : 0);
  return 1;
}

// ---------------------------------------------------------------------------------------------------------------
// Weight-standardisation adjoint, one CTA per output channel o:
//   what = (w - mean) / s,  s = sqrt(biased var + 1e-8)        (w: the fp32 raw OIHW weights, as ws_kernel)
//   dL/dw = (g - mean(g) - what * mean(g * what)) / s           (g: d/d what, KRSC channel-padded, lanes a + b)
// written OIHW (pad channels dropped), overwriting or adding to `out`.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ws_backward_kernel(const float* __restrict__ w, const float* __restrict__ ga,
                                                          const float* __restrict__ gb, float* __restrict__ out, int I,
                                                          int khw, int Ipad, int accumulate) {
  __shared__ float red[32];
  const int o = blockIdx.x, n = I * khw;
  const float* wo = w + (size_t)o * n;
  const float* gao = ga + (size_t)o * khw * Ipad;
  const float* gbo = gb ? gb + (size_t)o * khw * Ipad : nullptr;
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += wo[i];
  const float mean = block_sum(s, red) / n;
  float v = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) { const float d = wo[i] - mean; v += d * d; }
  const float var = block_sum(v, red) / n;
  const float rstd = 1.0f / sqrtf(var + 1e-8f);
  auto grad = [&](int i) {   // i: OIHW index within the channel
    const int c = i / khw, rs = i % khw;
    const size_t k = (size_t)rs * Ipad + c;
    return gbo ? gao[k] + gbo[k] : gao[k];
  };
  float sg = 0.f, sgw = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float g = grad(i), wh = (wo[i] - mean) * rstd;
    sg += g; sgw = fmaf(g, wh, sgw);
  }
  const float mg = block_sum(sg, red) / n;
  const float mgw = block_sum(sgw, red) / n;
  float* oo = out + (size_t)o * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float wh = (wo[i] - mean) * rstd;
    const float d = (grad(i) - mg - wh * mgw) * rstd;
    oo[i] = accumulate ? oo[i] + d : d;
  }
}

int launch_ws_backward(const float* w_raw, const float* g_a, const float* g_b, float* out, int O, int I, int kh, int kw,
                       int Ipad, bool accumulate, cudaStream_t st) {
  ws_backward_kernel<<<O, 256, 0, st>>>(w_raw, g_a, g_b, out, I, kh * kw, Ipad, accumulate ? 1 : 0);
  return 1;
}

// ---------------------------------------------------------------------------------------------------------------
// bf16 stem weight gradient on the tight NHWC C=3 input:
//   dW[co][ky][kx][c] = sum_{n,oy,ox} dY[n,oy,ox,co] * in[n, 2oy-3+ky, 2ox-3+kx, c]
// as a GEMM D[64 co][160 k] (k = (ky*7+kx)*3 + c, 147 real) over the output pixels q = (n, oy, ox).
// A CTA (8 warps) owns a contiguous range of q; per step of 32 pixels it stages dY^T [64][32] and the im2col
// rows [160][32] in shared memory (K-contiguous, so every fragment register is one 32-bit load), and runs
// mma.sync m16n8k16 (bf16 in, fp32 accumulate).  Warp w owns rows 16*(w&3).. and 10 of the 20 n8 tiles.
// The CTA's 64 x 160 sums go to partial[cta]; stem_wgrad_reduce_kernel adds them over the CTAs in order.
// ---------------------------------------------------------------------------------------------------------------
namespace stemw {
constexpr int THREADS = 256, QS = 32, KP = 160, KR = 147;
constexpr int LD = QS + 8;                 // 40 bf16 = 80 B rows
constexpr int MAX_CTAS = 264;
}  // namespace stemw

__device__ __forceinline__ void wg_mma_bf16(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                            uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(stemw::THREADS) stem_wgrad_kernel(const __nv_bfloat16* __restrict__ in,
                                                                    const __nv_bfloat16* __restrict__ dY,
                                                                    float* __restrict__ partial, int H, int W,
                                                                    long long Q, long long per_cta) {
  using namespace stemw;
  __shared__ __align__(16) __nv_bfloat16 sA[64 * LD];
  __shared__ __align__(16) __nv_bfloat16 sB[KP * LD];
  const int Ho = H / 2, Wo = W / 2;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t4 = lane & 3;
  const int m0 = (warp & 3) * 16, nt0 = (warp >> 2) * 10;
  const long long q_begin = (long long)blockIdx.x * per_cta;
  const long long q_end = q_begin + per_cta < Q ? q_begin + per_cta : Q;
  float acc[10][4];
#pragma unroll
  for (int t = 0; t < 10; ++t) acc[t][0] = acc[t][1] = acc[t][2] = acc[t][3] = 0.f;
  const __nv_bfloat16 zero = __float2bfloat16(0.f);
  for (long long q0 = q_begin; q0 < q_end; q0 += QS) {
    __syncthreads();                                               // the previous step's fragments are read
    for (int i = threadIdx.x; i < QS * 64; i += THREADS) {         // dY^T: coalesced over co
      const int px = i >> 6, co = i & 63;
      const long long q = q0 + px;
      sA[co * LD + px] = q < q_end ? dY[q * 64 + co] : zero;
    }
    for (int i = threadIdx.x; i < QS * KP; i += THREADS) {         // im2col rows, coalesced over k
      const int px = i / KP, k = i % KP;
      const long long q = q0 + px;
      __nv_bfloat16 v = zero;
      if (k < KR && q < q_end) {
        const int n = (int)(q / ((long long)Ho * Wo)), r = (int)(q % ((long long)Ho * Wo));
        const int oy = r / Wo, ox = r % Wo, tap = k / 3, c = k % 3;
        const int iy = 2 * oy - 3 + tap / 7, ix = 2 * ox - 3 + tap % 7;
        if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = in[(((size_t)n * H + iy) * W + ix) * 3 + c];
      }
      sB[k * LD + px] = v;
    }
    __syncthreads();
#pragma unroll
    for (int ks = 0; ks < QS; ks += 16) {
      const int kc = ks + 2 * t4;
      const uint32_t a0 = *reinterpret_cast<const uint32_t*>(sA + (m0 + g) * LD + kc);
      const uint32_t a1 = *reinterpret_cast<const uint32_t*>(sA + (m0 + g + 8) * LD + kc);
      const uint32_t a2 = *reinterpret_cast<const uint32_t*>(sA + (m0 + g) * LD + kc + 8);
      const uint32_t a3 = *reinterpret_cast<const uint32_t*>(sA + (m0 + g + 8) * LD + kc + 8);
#pragma unroll
      for (int t = 0; t < 10; ++t) {
        const int nb = (nt0 + t) * 8 + g;
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(sB + nb * LD + kc);
        const uint32_t b1 = *reinterpret_cast<const uint32_t*>(sB + nb * LD + kc + 8);
        wg_mma_bf16(acc[t], a0, a1, a2, a3, b0, b1);
      }
    }
  }
  float* po = partial + (size_t)blockIdx.x * 64 * KP;
#pragma unroll
  for (int t = 0; t < 10; ++t) {
    const int col = (nt0 + t) * 8 + 2 * t4;
    po[(m0 + g) * KP + col] = acc[t][0];
    po[(m0 + g) * KP + col + 1] = acc[t][1];
    po[(m0 + g + 8) * KP + col] = acc[t][2];
    po[(m0 + g + 8) * KP + col + 1] = acc[t][3];
  }
}

// acc KRSC [64][7][7][cin_pad] += sum over the CTAs (in order) of partial[cta][co][k], k < 147
__global__ void stem_wgrad_reduce_kernel(const float* __restrict__ partial, float* __restrict__ acc, int ctas, int cin_pad) {
  using namespace stemw;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 64 * KR) return;
  const int co = i / KR, k = i % KR;
  float s = 0.f;
  for (int b = 0; b < ctas; ++b) s += partial[(size_t)b * 64 * KP + co * KP + k];
  acc[((size_t)co * 49 + k / 3) * cin_pad + k % 3] += s;
}

size_t stem_wgrad_partial_floats() { return (size_t)stemw::MAX_CTAS * 64 * stemw::KP; }

int launch_stem_wgrad(const void* in, const void* dY, float* partial, float* acc, int N, int H, int W, int cin_pad,
                      cudaStream_t st) {
  using namespace stemw;
  const long long Q = (long long)N * (H / 2) * (W / 2);
  long long ctas = (Q + 8 * QS - 1) / (8 * QS);                   // at least 8 steps per CTA
  if (ctas > MAX_CTAS) ctas = MAX_CTAS;
  if (ctas < 1) ctas = 1;
  long long per = (Q + ctas - 1) / ctas;
  per = (per + QS - 1) / QS * QS;
  ctas = (Q + per - 1) / per;
  stem_wgrad_kernel<<<(unsigned)ctas, THREADS, 0, st>>>((const __nv_bfloat16*)in, (const __nv_bfloat16*)dY, partial, H, W, Q, per);
  stem_wgrad_reduce_kernel<<<(64 * KR + 255) / 256, 256, 0, st>>>(partial, acc, (int)ctas, cin_pad);
  return 2;
}

}  // namespace dp
