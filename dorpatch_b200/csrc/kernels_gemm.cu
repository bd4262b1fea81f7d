// kernels_gemm.cu -- 1x1 convolution with the GroupNorm(32)+ReLU of its INPUT applied on the way into shared
// memory, on the Hopper warpgroup tensor cores (wgmma.mma_async, fp32 accumulators in registers).
//
//   D[m, n] = sum_k relu(sa[s(m), k] * X[m, k] + sb[s(m), k]) * W[n, k]   (+ R[m, n])
//
//   X [M = N*P, K] bf16 NHWC activations (the tensor GroupNorm normalises, saved for backward anyway),
//   s(m) = m / P the sample of pixel row m, sa = rstd * gamma, sb = beta - mean * sa from the (mean, rstd)
//   statistics of a preceding stats pass, W the weight-standardised 1x1 filter, R the optional shortcut.
//   The normalised activation tensor y = relu(gn(x)) is never written to HBM (SURVEY 8d: "tensor-core bound
//   only if GN/ReLU are fused"); reference: timm PreActBottleneck norm1->conv1 / norm3->conv3 (SURVEY App. B).
//
// STATUS: opt-in (DORPATCH_FUSED_GEMM=1).  Checked per fused layer shape against an fp32 restatement on the same
// rounded operands (tests/test_gpu_ops.py::test_tcgen05_gn_gemm_vs_fp32, named after the
// kernel's first, tcgen05 version) and, as a whole network, against the fp32
// engine (tests/test_gpu_fused_gemm.py).  It is not the default path.
//
// Structure (one 128 x BN output tile per CTA, 256 threads = two warpgroups, two shared-memory stages):
//   every thread  16-byte global loads of the raw x tile and of the pre-packed weight tile for k block kb + 1 are
//                 issued while the wgmma of k block kb runs; scale / shift / ReLU in registers, st.shared into the
//                 canonical K-major no-swizzle core-matrix layout (8 rows x 16 B; chunk q of a tile lands at byte
//                 16 q, so the 8 lanes of a store phase write 8 consecutive rows, conflict-free), then
//                 fence.proxy.async + __syncthreads.
//   warpgroup g   4 x wgmma.m64nBNk16 per 64-wide k block on tile rows 64g..64g+63, one commit group per k block;
//                 wait_group 1 keeps one k block in flight, so stage kb % 2 is free again at k block kb + 2.
//   epilogue      accumulator fragments (+ shortcut) -> bf16 stores straight from registers.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"

namespace dp {
namespace tc {

constexpr int BM = 128, BK = 64, STAGES = 2;
constexpr int THREADS = 256;
constexpr int A_STAGE = BM * BK * 2;                 // 16 KB
constexpr int TAB = 2 * 4 * BK * 8;                  // 2 x [4 samples][64 ch] float2
constexpr int MAX_TILE_SAMPLES = 4;

__host__ __device__ constexpr int b_stage(int bn) { return bn * BK * 2; }
__host__ __device__ constexpr size_t smem_bytes(int bn) { return TAB + (size_t)STAGES * (A_STAGE + b_stage(bn)); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// wgmma shared-memory matrix descriptor, K-major, no swizzle: 8-row x 16-byte core matrices; LBO = byte distance
// between the two core matrices of one K = 16 step, SBO = between 8-row groups.
__device__ __forceinline__ uint64_t smem_desc(uint32_t addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((addr >> 4) & 0x3fffu);            // start address        bits [ 0,14)
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3fffu) << 16; // leading byte offset  bits [16,30)
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3fffu) << 32; // stride byte offset   bits [32,46)
  return d;                                          // base offset 0, layout type 0 = no swizzle
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D (+)= A * B^T, A 64 x 16 and B BN x 16, both K-major bf16 in shared memory; d[] the m64nBN fp32 fragment
__device__ __forceinline__ void wgmma_n64(float* d, uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,"
      "%30,%31}, %32, %33, 1, 1, 1, 0, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]),
        "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]),
        "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc));
}
__device__ __forceinline__ void wgmma_n128(float* d, uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,"
      "%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,"
      "%58,%59,%60,%61,%62,%63}, %64, %65, 1, 1, 1, 0, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]),
        "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]),
        "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
        "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]),
        "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]),
        "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]),
        "+f"(d[63])
      : "l"(adesc), "l"(bdesc));
}
template <int BN> __device__ __forceinline__ void wgmma_bn(float* d, uint64_t adesc, uint64_t bdesc) {
  if constexpr (BN == 64) wgmma_n64(d, adesc, bdesc);
  else wgmma_n128(d, adesc, bdesc);
}

__device__ __forceinline__ uint32_t pack2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack2(uint32_t u) {
  return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
}

struct GemmParams {
  const __nv_bfloat16* X;        // [M, K]
  const __nv_bfloat16* Wp;       // packed tiles [n_tiles][K/64][BN x 64] (canonical layout)
  const float* stats;            // [N][32][2] (mean, rstd) of X per (sample, group)
  const float* gamma; const float* beta;   // [K]
  const __nv_bfloat16* R;        // [M, Nout] shortcut or nullptr
  __nv_bfloat16* D;              // [M, Nout]
  int M, P, K, Nout, N;
};

template <int BN>
__global__ void __launch_bounds__(THREADS, 1) gn_gemm_fwd_kernel(GemmParams p) {
  constexpr int A_CHUNKS = A_STAGE / 16 / THREADS;        // 4 16-byte chunks per thread
  constexpr int B_CHUNKS = b_stage(BN) / 16 / THREADS;    // 2 (BN = 64) or 4 (BN = 128)
  extern __shared__ __align__(1024) unsigned char smem[];
  const int t = threadIdx.x, wg = t >> 7, warp = t >> 5, lane = t & 31;
  const int n_tiles = p.Nout / BN;
  const int nt = blockIdx.x % n_tiles, mt = blockIdx.x / n_tiles;   // CTAs sharing an x tile are adjacent
  const int m0 = mt * BM, n0 = nt * BN, KB = p.K / BK;

  float2* tab = reinterpret_cast<float2*>(smem);
  const uint32_t a_base = smem_u32(smem + TAB), b_base = a_base + STAGES * A_STAGE;
  uint4* a_st = reinterpret_cast<uint4*>(smem + TAB);
  uint4* b_st = reinterpret_cast<uint4*>(smem + TAB + STAGES * A_STAGE);

  const int n_first = m0 / p.P;
  const int b1 = (n_first + 1) * p.P - m0, b2 = b1 + p.P, b3 = b2 + p.P;   // tile rows where the sample changes
  const int cpg = p.K / GN_GROUPS;
  // scale / shift table entry of this thread: sample n_first + ts, channel tc of the k block
  const int ts = t >> 6, tcol = t & 63;
  const int tn = min(n_first + ts, p.N - 1);
  const __nv_bfloat16* wt = p.Wp + (size_t)nt * KB * BN * BK;

  uint4 va[A_CHUNKS], vb[B_CHUNKS];
  float mean_r, rstd_r, gam_r, bet_r;
  auto load = [&](int kb) {
    const int k0 = kb * BK;
#pragma unroll
    for (int i = 0; i < A_CHUNKS; ++i) {
      const int q = i * THREADS + t, row = m0 + (q >> 6) * 8 + (q & 7), kc = (q >> 3) & 7;
      va[i] = row < p.M ? __ldg(reinterpret_cast<const uint4*>(p.X + (size_t)row * p.K + k0 + kc * 8)) : make_uint4(0u, 0u, 0u, 0u);
    }
    const uint4* wsrc = reinterpret_cast<const uint4*>(wt + (size_t)kb * BN * BK);
#pragma unroll
    for (int i = 0; i < B_CHUNKS; ++i) vb[i] = __ldg(wsrc + i * THREADS + t);
    const int g = (k0 + tcol) / cpg;
    mean_r = __ldg(p.stats + ((size_t)tn * GN_GROUPS + g) * 2);
    rstd_r = __ldg(p.stats + ((size_t)tn * GN_GROUPS + g) * 2 + 1);
    gam_r = __ldg(p.gamma + k0 + tcol);
    bet_r = __ldg(p.beta + k0 + tcol);
  };

  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;

  load(0);
  for (int kb = 0; kb < KB; ++kb) {
    const int stage = kb % STAGES;
    {
      const float sa = rstd_r * gam_r;
      tab[(stage * MAX_TILE_SAMPLES + ts) * BK + tcol] = make_float2(sa, bet_r - mean_r * sa);
    }
    // the table is visible, and both warpgroups have retired the wgmma of k block kb - 2 (wait_group 1 below)
    __syncthreads();
#pragma unroll
    for (int i = 0; i < A_CHUNKS; ++i) {
      const int q = i * THREADS + t, r = (q >> 6) * 8 + (q & 7), kc = (q >> 3) & 7;
      const int s = (r >= b1) + (r >= b2) + (r >= b3);
      const float4* tp = reinterpret_cast<const float4*>(tab + (stage * MAX_TILE_SAMPLES + s) * BK + kc * 8);
      const uint32_t w[4] = {va[i].x, va[i].y, va[i].z, va[i].w};
      const bool live = m0 + r < p.M;
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float4 ss = tp[j];                                            // (sa, sb) of channels 2j, 2j + 1
        const float2 f = unpack2(w[j]);
        o[j] = live ? pack2(fmaxf(fmaf(ss.x, f.x, ss.y), 0.f), fmaxf(fmaf(ss.z, f.y, ss.w), 0.f)) : 0u;
      }
      a_st[stage * (A_STAGE / 16) + q] = make_uint4(o[0], o[1], o[2], o[3]);
    }
#pragma unroll
    for (int i = 0; i < B_CHUNKS; ++i) b_st[stage * (b_stage(BN) / 16) + i * THREADS + t] = vb[i];
    fence_proxy_async();                                                    // generic-proxy stores -> visible to wgmma
    __syncthreads();
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < BK / 16; ++ks) {
      const uint64_t ad = smem_desc(a_base + stage * A_STAGE + wg * (A_STAGE / 2) + ks * 256, 128, 1024);
      const uint64_t bd = smem_desc(b_base + stage * b_stage(BN) + ks * 256, 128, 1024);
      wgmma_bn<BN>(acc, ad, bd);
    }
    wgmma_commit();
    if (kb + 1 < KB) load(kb + 1);                                          // in flight under this k block's wgmma
    wgmma_wait<1>();
  }
  wgmma_wait<0>();

  // ===================== epilogue =====================
  // m64nBN fragment: acc[4 j + e] is row 16 w + lane / 4 + 8 (e / 2), column 8 j + 2 (lane % 4) + e % 2
  const int r0 = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int c0 = n0 + 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = r0 + 8 * h;
    if (m >= p.M) continue;
    __nv_bfloat16* drow = p.D + (size_t)m * p.Nout + c0;
    const __nv_bfloat16* rrow = p.R ? p.R + (size_t)m * p.Nout + c0 : nullptr;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
      if (rrow != nullptr) {                                                // plain load: R may be D (in-place shortcut)
        const float2 e = unpack2(*reinterpret_cast<const uint32_t*>(rrow + 8 * j));
        x0 += e.x; x1 += e.y;
      }
      *reinterpret_cast<uint32_t*>(drow + 8 * j) = pack2(x0, x1);
    }
  }
}

// W [Nout][K] bf16 row-major -> tiles [Nout/BN][K/64] of BN x 64 in the canonical K-major core-matrix layout
// (element (r, kk) at (r/8)*512 + (kk/8)*64 + (r%8)*8 + kk%8), so that a k block's B operand is one contiguous, ready-laid-out tile.
__global__ void pack_w_kernel(const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ out, int Nout, int K, int BN) {
  const size_t total = (size_t)Nout * K;
  const int KB = K / BK;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / K), k = (int)(i % K);
    const int nt = n / BN, r = n % BN, kb = k / BK, kk = k % BK;
    out[((size_t)nt * KB + kb) * BN * BK + (r / 8) * 512 + (kk / 8) * 64 + (r % 8) * 8 + (kk % 8)] = w[i];
  }
}

}  // namespace tc

// BN <= 128: 68 KB of shared memory per CTA
int gn_gemm_tile_n(int Nout) { return Nout >= 128 ? 128 : Nout; }

bool gn_gemm_supported(int P, int K, int Nout) {
  const int bn = gn_gemm_tile_n(Nout);
  return K % tc::BK == 0 && K >= 64 && (bn == 64 || bn == 128) && Nout % bn == 0 &&
         (tc::BM + P - 1) / P + 1 <= tc::MAX_TILE_SAMPLES;
}

int launch_gn_gemm_pack(const void* w, void* out, int Nout, int K, cudaStream_t st) {
  tc::pack_w_kernel<<<256, 256, 0, st>>>((const __nv_bfloat16*)w, (__nv_bfloat16*)out, Nout, K, gn_gemm_tile_n(Nout));
  return 1;
}

int launch_gn_gemm_forward(const void* x, const void* w_packed, const float* stats, const float* gamma, const float* beta,
                           const void* shortcut, void* out, int N, int P, int K, int Nout, cudaStream_t st) {
  if (!gn_gemm_supported(P, K, Nout)) return 0;
  tc::GemmParams p{(const __nv_bfloat16*)x, (const __nv_bfloat16*)w_packed, stats, gamma, beta,
                   (const __nv_bfloat16*)shortcut, (__nv_bfloat16*)out, N * P, P, K, Nout, N};
  const int bn = gn_gemm_tile_n(Nout);
  const int grid = ((p.M + tc::BM - 1) / tc::BM) * (Nout / bn);
  const size_t smem = tc::smem_bytes(bn);
#define GG_CASE(BNV)                                                                                                  \
  case BNV:                                                                                                           \
    cudaFuncSetAttribute(tc::gn_gemm_fwd_kernel<BNV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);      \
    tc::gn_gemm_fwd_kernel<BNV><<<grid, tc::THREADS, smem, st>>>(p);                                                  \
    break;
  switch (bn) {
    GG_CASE(64)
    GG_CASE(128)
    default: return 0;
  }
#undef GG_CASE
  return 1;
}

}  // namespace dp
