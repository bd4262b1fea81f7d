// kernels_stem.cu -- hand-written tensor-core stem convolution (bf16): 7x7 stride 2 pad 3, 3 -> 64.
//
// The classifier's first layer (timm ResNetV2 'fixed' stem, StdConv2d 7x7/2; reference call site
// reference utils.py:78 -> timm) has only 3 input channels: library kernels want the channel
// dimension padded to 8 (bf16), which (i) makes K1 write 8/3 of the algorithmic bytes and (ii) runs
// at ~23 TFLOP/s in cuDNN.  This kernel reads the TIGHT NHWC C=3 layout K1 produces, builds the
// im2col tile in shared memory and runs mma.sync.m16n8k16 (bf16 in, fp32 accumulate).
//   CTA = 256 threads = 8 warps; tile = 8 x 16 output pixels x 64 channels; K = 147 -> 160.
//   A CTA walks all x-tiles of one (sample, tile-row): the 20 KB weight matrix is loaded once.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "kernels.h"

namespace dp {
namespace stem {
constexpr int TOY = 8, TOX = 16, TM = TOY * TOX;       // output tile
constexpr int KR = 147, KP = 160;                      // real / padded reduction length
constexpr int PR = 2 * TOY + 5, PC = 2 * TOX + 5;      // input patch 21 x 37 pixels
constexpr int PSTRIDE = PC * 3 + 1;                    // 112 elements per patch row
constexpr int ASTRIDE = KP + 8;                        // 168: conflict-free ldmatrix rows (336 B)
constexpr int BSTRIDE = 64 + 8;                        // 72: conflict-free (144 B)
constexpr int THREADS = 256;
constexpr size_t SMEM = (size_t)(PR * PSTRIDE + TM * ASTRIDE + KP * BSTRIDE) * 2;

__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(a));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(a));
}
__device__ __forceinline__ void mma_bf16(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
}  // namespace stem

// w_kn: [KP][64] bf16, row k = (ky*7+kx)*3 + c (rows >= 147 are zero).  in: [N,H,W,3] bf16.  out: [N,H/2,W/2,64].
__global__ void __launch_bounds__(stem::THREADS) stem_fwd_kernel(const __nv_bfloat16* __restrict__ in,
                                                                  const __nv_bfloat16* __restrict__ w_kn,
                                                                  __nv_bfloat16* __restrict__ out, int H, int W) {
  using namespace stem;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __nv_bfloat16* patch = reinterpret_cast<__nv_bfloat16*>(smem_raw);
  __nv_bfloat16* As = patch + PR * PSTRIDE;
  __nv_bfloat16* Bs = As + TM * ASTRIDE;
  const int Ho = H / 2, Wo = W / 2;
  const int n = blockIdx.y, oy0 = blockIdx.x * TOY;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  for (int i = threadIdx.x; i < KP * 64; i += THREADS) Bs[(i >> 6) * BSTRIDE + (i & 63)] = w_kn[i];
  for (int i = threadIdx.x; i < TM * (KP - KR); i += THREADS)                        // zero the K padding once
    As[(i / (KP - KR)) * ASTRIDE + KR + i % (KP - KR)] = __float2bfloat16(0.f);

  const __nv_bfloat16* in_n = in + (size_t)n * H * W * 3;
  const int ntx = (Wo + TOX - 1) / TOX;
  for (int tx = 0; tx < ntx; ++tx) {
    const int ox0 = tx * TOX;
    const int iy0 = 2 * oy0 - 3, ix0 = 2 * ox0 - 3;
    __syncthreads();                                                                // previous tile's MMAs done
    for (int i = threadIdx.x; i < PR * PC * 3; i += THREADS) {
      const int r = i / (PC * 3), e = i % (PC * 3);
      const int iy = iy0 + r, ix = ix0 + e / 3;
      __nv_bfloat16 v = __float2bfloat16(0.f);
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = in_n[((size_t)iy * W + ix0) * 3 + e];
      patch[r * PSTRIDE + e] = v;
    }
    __syncthreads();
    // im2col: A[m][ky*21 + j] = patch[2*py + ky][6*px + j], j < 21
    for (int i = threadIdx.x; i < TM * 7; i += THREADS) {
      const int m = i / 7, ky = i % 7, py = m / TOX, px = m % TOX;
      const __nv_bfloat16* src = patch + (2 * py + ky) * PSTRIDE + 6 * px;
      __nv_bfloat16* dst = As + m * ASTRIDE + ky * 21;
#pragma unroll
      for (int j = 0; j < 21; ++j) dst[j] = src[j];
    }
    __syncthreads();
    float acc[8][4];
#pragma unroll
    for (int t = 0; t < 8; ++t) { acc[t][0] = acc[t][1] = acc[t][2] = acc[t][3] = 0.f; }
    const int m0 = warp * 16;
#pragma unroll
    for (int ks = 0; ks < KP / 16; ++ks) {
      uint32_t a0, a1, a2, a3;
      ldmatrix_x4(a0, a1, a2, a3, As + (m0 + (lane & 15)) * ASTRIDE + ks * 16 + (lane >> 4) * 8);
#pragma unroll
      for (int np = 0; np < 4; ++np) {                                              // two n8 tiles per ldmatrix
        uint32_t b0, b1, b2, b3;
        ldmatrix_x4_trans(b0, b1, b2, b3, Bs + (ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * BSTRIDE + np * 16 + (lane >> 4) * 8);
        mma_bf16(acc[2 * np], a0, a1, a2, a3, b0, b1);
        mma_bf16(acc[2 * np + 1], a0, a1, a2, a3, b2, b3);
      }
    }
    const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int m = m0 + g + half * 8, oy = oy0 + m / TOX, ox = ox0 + m % TOX;
      if (oy < Ho && ox < Wo) {
        __nv_bfloat16* o = out + (((size_t)n * Ho + oy) * Wo + ox) * 64;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
          *reinterpret_cast<__nv_bfloat162*>(o + nt * 8 + 2 * t4) = __floats2bfloat162_rn(acc[nt][half * 2], acc[nt][half * 2 + 1]);
      }
    }
  }
}

// KRSC (cin padded to cin_pad) -> [160][64] K-major matrix for the kernel above
__global__ void stem_pack_kernel(const __nv_bfloat16* __restrict__ w_krsc, __nv_bfloat16* __restrict__ w_kn, int cin_pad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= stem::KP * 64) return;
  const int k = i >> 6, n = i & 63;
  __nv_bfloat16 v = __float2bfloat16(0.f);
  if (k < stem::KR) { const int tap = k / 3, c = k % 3; v = w_krsc[((size_t)n * 49 + tap) * cin_pad + c]; }
  w_kn[i] = v;
}

int launch_stem_pack(const void* w_krsc, void* w_kn, int cin_pad, cudaStream_t st) {
  stem_pack_kernel<<<(stem::KP * 64 + 255) / 256, 256, 0, st>>>((const __nv_bfloat16*)w_krsc, (__nv_bfloat16*)w_kn, cin_pad);
  return 1;
}
int launch_stem_forward(const void* in, const void* w_kn, void* out, int N, int H, int W, cudaStream_t st) {
  cudaFuncSetAttribute(stem_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)stem::SMEM);
  const int Ho = H / 2;
  dim3 grid((Ho + stem::TOY - 1) / stem::TOY, N);
  stem_fwd_kernel<<<grid, stem::THREADS, stem::SMEM, st>>>((const __nv_bfloat16*)in, (const __nv_bfloat16*)w_kn, (__nv_bfloat16*)out, H, W);
  return 1;
}


// =====================================================================================================
// Stem backward fused with the masked EOT reduce (K1^T):
//   G[b,c,y,x] (+)= 2 * sum_{samples n of image b} keep_n(y,x) * dX_n[y,x,c],
//   dX_n[y,x,c] = sum_{k,ky,kx} dY_n[(y+3-ky)/2, (x+3-kx)/2, k] * W[k,ky,kx,c]   (only parities that divide)
// The per-sample input gradient [N,H,W,3] is never written: a CTA owns an 8x16 tile of input pixels of ONE
// parity class (y%2, x%2) of ONE image, loops over that image's samples (cp.async double-buffered dY patches),
// runs mma.sync m16n8k16 (N = 8 padded output channels, K = taps x 64) per sample and adds the result into
// register accumulators under the sample's occlusion mask.  Replaces cuDNN's stem dgrad (2.6 ms/step incl. its
// padding / folding helper kernels, writing a C-padded-to-8 gradient tensor) + reduce_kernel.
// =====================================================================================================
namespace stemb {
constexpr int TI = 8, TJ = 16;                 // positions (i, j) = (y >> 1, x >> 1) per tile
constexpr int PR = TI + 3, PC = TJ + 3;        // dY patch (rows i0-1 .. i0+TI+1)
constexpr int PIX = 144;                       // bytes per patch pixel (128 + 16 pad: conflict-free ldmatrix)
constexpr int THREADS = 256;
constexpr int ALLTAPS = 49;                      // 9 + 12 + 12 + 16 taps of the four parity classes
constexpr size_t W_BYTES = (size_t)ALLTAPS * 64 * 16;
constexpr size_t PATCH_BYTES = (size_t)PR * PC * PIX;

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(a), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void ldmatrix_x2_trans(uint32_t& r0, uint32_t& r1, const void* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(a));
}

// The CTA's tile: positions [i0, i0 + TI) x [j0, j0 + TJ) of the chunk whose first sample is n0.
struct Tile { int i0, j0, n0, H, W; };

// Where a sample's dY patch [PR][PC][PIX] comes from.  load(s, buf) starts the copy of sample s's data into staging
// buffer buf (one cp.async group); once that group has landed, patch(buf) returns the sample's patch.  `stage` is the
// shared memory after the weights, SMEM the kernel's dynamic shared memory.
struct DyPatch {   // dY [n, H/2, W/2, 64]: the patch itself, double-buffered
  const __nv_bfloat16* dY;
  static constexpr size_t SMEM = W_BYTES + 2 * PATCH_BYTES;
  __device__ __forceinline__ void load(unsigned char* stage, const Tile& t, int sample, int buf) const {
    const int Ho = t.H / 2, Wo = t.W / 2;
    const __nv_bfloat16* src = dY + (size_t)(sample - t.n0) * Ho * Wo * 64;
    unsigned char* dst = stage + (size_t)buf * PATCH_BYTES;
    for (int q = threadIdx.x; q < PR * PC * 8; q += THREADS) {
      const int pix = q >> 3, ch = q & 7;
      const int oy = t.i0 - 1 + pix / PC, ox = t.j0 - 1 + pix % PC;
      unsigned char* d = dst + (size_t)pix * PIX + ch * 16;
      if (oy >= 0 && oy < Ho && ox >= 0 && ox < Wo) cp_async16(d, src + ((size_t)oy * Wo + ox) * 64 + ch * 8);
      else *reinterpret_cast<uint4*>(d) = make_uint4(0u, 0u, 0u, 0u);
    }
    cp_commit();
  }
  __device__ __forceinline__ const unsigned char* patch(unsigned char* stage, const Tile&, int buf) const {
    return stage + (size_t)buf * PATCH_BYTES;
  }
};

// PoolPatch also fuses the backward of ConstantPad2d(1,0)+MaxPool(3,2): it reads d_pool [n,Hp,Wp,64] + the int8 argmax
// saved by the forward pass and rebuilds each sample's d_stem patch in shared memory (fp32 sum of the <= 4 windows that
// selected a stem pixel, rounded once to bf16 -- bit-identical to maxpool_bwd_kernel's output), so the [N,112,112,64]
// stem-output gradient is never written to HBM either.  The pooled-window region is double-buffered, the patch is not.
constexpr int RR = 7, RC = 11;                                   // pooled-window region feeding one patch
constexpr size_t REGION_BYTES = (size_t)RR * RC * (128 + 64);    // d_pool (bf16 x64) + argmax (int8 x64) per window
struct PoolPatch {   // stage: [PR][PC][PIX] patch, then [2][RR*RC][128 + 64] region
  const __nv_bfloat16* dpool;
  const int8_t* amax;
  static constexpr size_t SMEM = W_BYTES + PATCH_BYTES + 2 * REGION_BYTES;
  __device__ __forceinline__ void load(unsigned char* stage, const Tile& t, int sample, int buf) const {
    const int Hp = t.H / 4, Wp = t.W / 4;
    const int wy0 = t.i0 / 2 - 1, wx0 = t.j0 / 2 - 1;             // first pooled window row / col of the region
    const __nv_bfloat16* sp = dpool + (size_t)(sample - t.n0) * Hp * Wp * 64;
    const int8_t* sa = amax + (size_t)(sample - t.n0) * Hp * Wp * 64;
    unsigned char* dst = stage + PATCH_BYTES + (size_t)buf * REGION_BYTES;
    for (int q = threadIdx.x; q < RR * RC * 12; q += THREADS) {   // 8 chunks of d_pool + 4 chunks of argmax per window
      const int win = q / 12, ch = q % 12;
      const int wy = wy0 + win / RC, wx = wx0 + win % RC;
      unsigned char* d = dst + (size_t)win * 192 + ch * 16;
      if (wy >= 0 && wy < Hp && wx >= 0 && wx < Wp) {
        const size_t o = ((size_t)wy * Wp + wx) * 64;
        if (ch < 8) cp_async16(d, sp + o + ch * 8);
        else cp_async16(d, sa + o + (ch - 8) * 16);
      } else {
        *reinterpret_cast<uint4*>(d) = ch < 8 ? make_uint4(0u, 0u, 0u, 0u) : make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu);
      }
    }
    cp_commit();
  }
  // max-pool backward of the region into the patch; ends in a block barrier
  __device__ __forceinline__ const unsigned char* patch(unsigned char* stage, const Tile& t, int buf) const {
    const int Ho = t.H / 2, Wo = t.W / 2, Hp = t.H / 4, Wp = t.W / 4;
    const int wy0 = t.i0 / 2 - 1, wx0 = t.j0 / 2 - 1;
    const unsigned char* rg = stage + PATCH_BYTES + (size_t)buf * REGION_BYTES;
    for (int q = threadIdx.x; q < PR * PC * 8; q += THREADS) {
      const int pix = q >> 3, ch = q & 7;
      const int oy = t.i0 - 1 + pix / PC, ox = t.j0 - 1 + pix % PC;
      float acc8[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) acc8[k] = 0.f;
      if (oy >= 0 && oy < Ho && ox >= 0 && ox < Wo) {
        for (int wy = oy / 2; wy <= (oy + 1) / 2; ++wy) {
          const int ky = oy - 2 * wy + 1;
          if (wy >= Hp || ky < 0 || ky > 2) continue;
          for (int wx = ox / 2; wx <= (ox + 1) / 2; ++wx) {
            const int kx = ox - 2 * wx + 1;
            if (wx >= Wp || kx < 0 || kx > 2) continue;
            const unsigned char* wp = rg + (size_t)((wy - wy0) * RC + (wx - wx0)) * 192;
            const uint4 dv = *reinterpret_cast<const uint4*>(wp + ch * 16);
            const uint2 av = *reinterpret_cast<const uint2*>(wp + 128 + ch * 8);
            const __nv_bfloat162* dh = reinterpret_cast<const __nv_bfloat162*>(&dv);
            const uint32_t am[2] = {av.x, av.y};
            const int want = ky * 3 + kx;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
              if ((int)((am[k >> 2] >> (8 * (k & 3))) & 0xffu) == want) {
                const float2 f = __bfloat1622float2(dh[k >> 1]);
                acc8[k] += (k & 1) ? f.y : f.x;
              }
            }
          }
        }
      }
      __nv_bfloat162 o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) o[k] = __floats2bfloat162_rn(acc8[2 * k], acc8[2 * k + 1]);
      *reinterpret_cast<uint4*>(stage + (size_t)pix * PIX + ch * 16) = *reinterpret_cast<const uint4*>(o);
    }
    __syncthreads();
    return stage;
  }
};
}  // namespace stemb

// `in` (a stemb::DyPatch or stemb::PoolPatch) gives each sample's dY [.., H/2, W/2, 64] patch; w_krsc: [64][7][7][cin_pad]
// bf16.  One CTA = one 8x16 tile of positions (i,j) of one image = a 16x32 block of input pixels; all four parity
// classes share the dY patch (one per sample).  BANK: keep_n from the mask bank `bank` (rects unused).
template <class Src, bool BANK>
__global__ void __launch_bounds__(stemb::THREADS, 2) stem_bwd_reduce_kernel(Src in, const __nv_bfloat16* __restrict__ w_krsc,
                                                                             int cin_pad, const int16_t* __restrict__ rects,
                                                                             float* __restrict__ G, int S, int n0, int n,
                                                                             int H, int W, MaskBank bank) {
  using namespace stemb;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  unsigned char* Ws = smem_raw;                                   // [49 taps, class-major][k][8] bf16, 16 B per (tap, k)
  unsigned char* stage = smem_raw + W_BYTES;
  const int Hc = H / 2, Wc = W / 2;                               // positions per parity class
  const int tiles_j = (Wc + TJ - 1) / TJ;
  const int ti = blockIdx.x / tiles_j, tj = blockIdx.x % tiles_j;
  const auto [b, lo, hi, first] = image_span(S, n0, n, blockIdx.y);
  if (lo >= hi) return;
  const int i0 = ti * TI, j0 = tj * TJ;
  const Tile tile{i0, j0, n0, H, W};
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // weights, class-major: class cls = py*2+px owns taps [tap0(cls), tap0(cls) + nky*nkx): 9, 12, 12, 16 taps
  for (int q = threadIdx.x; q < 49 * 64; q += THREADS) {
    const int t = q >> 6, k = q & 63;
    int cls = 0, tl = t;
    if (tl >= 9) { cls = 1; tl -= 9; if (tl >= 12) { cls = 2; tl -= 12; if (tl >= 12) { cls = 3; tl -= 12; } } }
    const int py = cls >> 1, px = cls & 1, nkx = px ? 4 : 3;
    const int ky = (py ? 0 : 1) + 2 * (tl / nkx), kx = (px ? 0 : 1) + 2 * (tl % nkx);
    const __nv_bfloat16* src = w_krsc + ((size_t)(k * 7 + ky) * 7 + kx) * cin_pad;
    __nv_bfloat16 v[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) v[c] = (c < 3) ? src[c] : __float2bfloat16(0.f);
    *reinterpret_cast<uint4*>(Ws + (size_t)q * 16) = *reinterpret_cast<const uint4*>(v);
  }

  float tot[4][4];
#pragma unroll
  for (int c = 0; c < 4; ++c) { tot[c][0] = tot[c][1] = tot[c][2] = tot[c][3] = 0.f; }
  const int g = lane >> 2, t4 = lane & 3;
  const int irow = i0 + warp;                                      // this warp's position row

  in.load(stage, tile, lo, 0);
  for (int s = lo; s < hi; ++s) {
    const int buf = (s - lo) & 1;
    if (s + 1 < hi) { in.load(stage, tile, s + 1, buf ^ 1); cp_wait<1>(); } else { cp_wait<0>(); }
    __syncthreads();
    const unsigned char* pb = in.patch(stage, tile, buf);
    Occlusion occ;
    [[maybe_unused]] int2 sel;
    if constexpr (BANK) sel = occl_bank::select(bank, s);
    else if (rects != nullptr) occ.set(occl::load(rects, s));
    // The 49 taps use only 16 distinct patch shifts (di, dj) in {-1..2}^2: load each A fragment once and feed
    // every parity class that has a tap at this shift (shared-memory bandwidth is the limit: N is only 8).
    float acc[4][4];
#pragma unroll
    for (int c = 0; c < 4; ++c) { acc[c][0] = acc[c][1] = acc[c][2] = acc[c][3] = 0.f; }
#pragma unroll
    for (int di = -1; di <= 2; ++di) {
#pragma unroll
      for (int dj = -1; dj <= 2; ++dj) {
        const unsigned char* arow = pb + ((size_t)(warp + di + 1) * PC + (lane & 15) + dj + 1) * PIX + (lane >> 4) * 16;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          uint32_t a0, a1, a2, a3;
          stem::ldmatrix_x4(a0, a1, a2, a3, arow + kk * 32);
#pragma unroll
          for (int cls = 0; cls < 4; ++cls) {
            const int py = cls >> 1, px = cls & 1, nkx = px ? 4 : 3;
            if ((di == 2 && !py) || (dj == 2 && !px)) continue;   // compile-time after unrolling
            const int t = ((py ? 2 : 1) - di) * nkx + ((px ? 2 : 1) - dj);
            const int tap0 = cls == 0 ? 0 : (cls == 1 ? 9 : (cls == 2 ? 21 : 33));
            uint32_t b0, b1;
            ldmatrix_x2_trans(b0, b1, Ws + ((size_t)(tap0 + t) * 64 + kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * 16);
            stem::mma_bf16(acc[cls], a0, a1, a2, a3, b0, b1);
          }
        }
      }
    }
#pragma unroll
    for (int cls = 0; cls < 4; ++cls) {
      const int py = cls >> 1, px = cls & 1;
      const int y = 2 * irow + py, xA = 2 * (j0 + g) + px, xB = 2 * (j0 + g + 8) + px;
      bool keepA, keepB;
      if constexpr (BANK) {
        keepA = y >= H || xA >= W || !occl_bank::hit(bank, sel, y, xA);   // (a position past the image is never stored)
        keepB = y >= H || xB >= W || !occl_bank::hit(bank, sel, y, xB);
      } else {
        keepA = rects == nullptr || !occ.hit(y, xA);
        keepB = rects == nullptr || !occ.hit(y, xB);
      }
      if (keepA) { tot[cls][0] += acc[cls][0]; tot[cls][1] += acc[cls][1]; }
      if (keepB) { tot[cls][2] += acc[cls][2]; tot[cls][3] += acc[cls][3]; }
    }
    __syncthreads();                                               // the staging buffers may be refilled
  }
  // C fragment: (row g: cols 2*t4, 2*t4+1), (row g+8: same cols); channels 0..2 are real
  if (irow < Hc && t4 < 2) {
#pragma unroll
    for (int cls = 0; cls < 4; ++cls) {
      const int py = cls >> 1, px = cls & 1;
      const int y = 2 * irow + py;
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int x = 2 * (j0 + g + half * 8) + px;
        if (x >= W) continue;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 2 * t4 + e;
          if (c >= 3) continue;
          float* gp = G + ((size_t)b * 3 + c) * H * W + (size_t)y * W + x;
          const float v = 2.0f * tot[cls][half * 2 + e];
          *gp = first ? v : (*gp + v);
        }
      }
    }
  }
}

template <class Src, bool BANK>
static int launch_stem_bwd_as(Src in, const void* w_krsc, int cin_pad, const int16_t* rects, float* G, int S, int n0, int n,
                              int H, int W, const MaskBank& bank, cudaStream_t st) {
  cudaFuncSetAttribute(stem_bwd_reduce_kernel<Src, BANK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Src::SMEM);
  const int tiles = ((H / 2 + stemb::TI - 1) / stemb::TI) * ((W / 2 + stemb::TJ - 1) / stemb::TJ);
  stem_bwd_reduce_kernel<Src, BANK><<<dim3(tiles, images_touched(S, n0, n)), stemb::THREADS, Src::SMEM, st>>>(
      in, (const __nv_bfloat16*)w_krsc, cin_pad, rects, G, S, n0, n, H, W, bank);
  return 1;
}
template <class Src>
static int launch_stem_bwd(Src in, const void* w_krsc, int cin_pad, const int16_t* rects, float* G, int S, int n0, int n,
                           int H, int W, const MaskBank* bank, cudaStream_t st) {
  if (bank != nullptr) return launch_stem_bwd_as<Src, true>(in, w_krsc, cin_pad, nullptr, G, S, n0, n, H, W, *bank, st);
  return launch_stem_bwd_as<Src, false>(in, w_krsc, cin_pad, rects, G, S, n0, n, H, W, MaskBank{}, st);
}
int launch_stem_bwd_reduce(const void* dY, const void* w_krsc, int cin_pad, const int16_t* rects, float* G, int B, int S,
                           int n0, int n, int H, int W, cudaStream_t st, const MaskBank* bank) {
  (void)B;
  return launch_stem_bwd(stemb::DyPatch{(const __nv_bfloat16*)dY}, w_krsc, cin_pad, rects, G, S, n0, n, H, W, bank, st);
}
int launch_stem_bwd_pool_reduce(const void* dpool, const int8_t* amax, const void* w_krsc, int cin_pad, const int16_t* rects,
                                float* G, int B, int S, int n0, int n, int H, int W, cudaStream_t st, const MaskBank* bank) {
  (void)B;
  return launch_stem_bwd(stemb::PoolPatch{(const __nv_bfloat16*)dpool, amax}, w_krsc, cin_pad, rects, G, S, n0, n, H, W, bank, st);
}

}  // namespace dp
