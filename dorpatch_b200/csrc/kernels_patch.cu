// kernels_patch.cu -- hand-written sm_90a kernels of the patch side of the DorPatch hot loop.
//
//   paste    utils.py:105-110 (clip) + attack.py:185        per image, L2 norm via warp shuffles
//   expand   K1: attack.py:204-220 + utils.py:77-78         paste + normalise + occlude, ONE HBM pass,
//                                                           TMA (cp.async.bulk) staged shared-memory tiles
//   cw       K4: attack.py:16-23,224-225                    CW margin loss + argmax + dlogits
//   reduce   K1^T: adjoint of the occlusion/normalisation   masked EOT gradient reduce over S
//   struct   attack.py:33-45,227-228                        structural loss + its (one-sided) gradient
//   maskreg  attack.py:72-80,235-245                        density + group-lasso values / statistics
//   update   K3: attack.py:332-342                          chain rule through clip + sign step + clip
//   eot_draw attack.py:193-218 (eot_sampler="device")       EOT indices + rectangles from Philox, per image
// (file:line into the reference).  Images are NCHW fp32; network input is NHWC(Cp) T.
#include <cstdlib>
#include <type_traits>

#include "common.cuh"
#include "kernels.h"

namespace dp {

// =====================================================================================
// paste: one CTA per image (deterministic reduction order)
// =====================================================================================
__global__ void __launch_bounds__(1024) paste_kernel(const float* __restrict__ x, const float* __restrict__ mask,
                                                     const float* __restrict__ pattern, float* __restrict__ adv,
                                                     float* __restrict__ l2, float* __restrict__ scale, int HW,
                                                     float eps) {
  __shared__ float red[32];
  const int b = blockIdx.x;
  const float* xb = x + (size_t)b * 3 * HW;
  const float* pb = pattern + (size_t)b * 3 * HW;
  const float* mb = mask + (size_t)b * HW;
  float s = 0.f;
  for (int i = threadIdx.x; i < HW; i += blockDim.x) {
    const float m = mb[i];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float d = __fmul_rn(m, __fsub_rn(pb[c * HW + i], xb[c * HW + i]));
      s = fmaf(d, d, s);
    }
  }
  const float norm = sqrtf(block_sum(s, red));
  const float sc = fminf(__fdiv_rn(eps, norm), 1.0f);   // eps/0 = inf -> 1, as torch .clip(max=1)
  if (threadIdx.x == 0) { l2[b] = norm; scale[b] = sc; }
  if (adv != nullptr) {
    float* ab = adv + (size_t)b * 3 * HW;
    for (int i = threadIdx.x; i < HW; i += blockDim.x) {
      const float m = mb[i];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float xv = xb[c * HW + i];
        const float d = __fmul_rn(__fmul_rn(m, __fsub_rn(pb[c * HW + i], xv)), sc);
        ab[c * HW + i] = __fadd_rn(xv, d);
      }
    }
  }
}
int launch_paste(const float* x, const float* mask, const float* pattern, float* adv_x, float* l2, float* scale,
                 int B, int H, int W, float eps, cudaStream_t st) {
  paste_kernel<<<B, 1024, 0, st>>>(x, mask, pattern, adv_x, l2, scale, H * W, eps);
  return 1;
}

// =====================================================================================
// K1 expand: TMA bulk loads of the image planes -> shared; "clean" normalised NHWC tile
// composed once per (image, row tile); per EOT sample either bulk-stored straight from
// the clean tile (no occluder touches these rows) or from a staging tile with the
// occluded pixels zeroed.  HBM-bound: bytes written = N*H*W*Cp*sizeof(T).
// =====================================================================================
namespace ptx {
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  }
}
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_store(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
}  // namespace ptx

constexpr int EXP_R_DEFAULT = 8;  // image rows per tile (DORPATCH_K1_ROWS overrides; must divide H)
constexpr int EXP_THREADS = 256;
constexpr int EXP_WARPS = EXP_THREADS / 32;
constexpr int EXP_HDR = 512 + 2048;   // mbarrier + per-item rectangle cache (64 samples x 32 B)
constexpr int EXP_RCACHE = 64;

struct ExpandParams {
  const float* img; const float* x; const float* mask; const float* pattern; const float* scale;
  const int16_t* rects; void* out;
  int B, S, n0, n, H, W, sgroups, R;
  int mode;   // 0: bulk stores (cp.async.bulk) for untouched tiles / rows + 16-byte stores for occluded rows; 1: 16-byte stores only
  MaskBank bank;   // the occlusion of the BANK variant (rects unused)
};

// Shared memory (dynamic): [mbarrier, 512 B][input planes NP*R*W fp32][clean tile R*W*CP T].
// A tile is R full image rows of the output layout = one contiguous run of the output tensor.
// Per EOT sample a warp either bulk-stores the clean tile / clean rows (TMA, cp.async.bulk) when no
// occluder crosses them, or writes an occluded row itself with 16-byte global stores whose keep /
// zero / mixed status comes from <= 4 element intervals (no staging copy, no block barrier).
// BANK: the occlusion comes from the mask bank p.bank instead: a warp reads a row's bank words (one per lane, <= 32
// words: W <= 1024) and builds the same per-lane element mask from the row's bits.
template <typename T, int CP, bool FUSED, bool BANK>
__global__ void __launch_bounds__(EXP_THREADS) expand_kernel(ExpandParams p) {
  constexpr int NP = FUSED ? 7 : 3;
  constexpr int EPC = 16 / (int)sizeof(T);                 // elements per 16-byte chunk
  extern __shared__ __align__(128) unsigned char smem[];
  const int W = p.W, H = p.H, HW = H * W;
  const int EXP_R = p.R;
  const int tile_px = EXP_R * W;
  const uint32_t plane_bytes = (uint32_t)tile_px * 4u;
  const int row_elems = W * CP;
  const uint32_t row_bytes = (uint32_t)row_elems * (uint32_t)sizeof(T);
  const uint32_t out_bytes = row_bytes * EXP_R;
  const int row_chunks = row_elems / EPC;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem);
  int4* srect = reinterpret_cast<int4*>(smem + 512);
  float* in = reinterpret_cast<float*>(smem + EXP_HDR);
  unsigned char* clean_b = smem + EXP_HDR + NP * plane_bytes;
  T* clean = reinterpret_cast<T*>(clean_b);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) { ptx::mbar_init(bar, 1); ptx::fence_mbar_init(); ptx::fence_proxy_async(); }
  __syncthreads();

  const int tiles = H / EXP_R;
  const int items = images_touched(p.S, p.n0, p.n) * tiles * p.sgroups;
  uint32_t phase = 0;

  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int sg = item % p.sgroups;
    const int tile = (item / p.sgroups) % tiles;
    const auto [b, lo, hi, first] = image_span(p.S, p.n0, p.n, item / (p.sgroups * tiles));
    const int cnt = hi - lo;
    const int s_lo = lo + (int)(((long long)cnt * sg) / p.sgroups), s_hi = lo + (int)(((long long)cnt * (sg + 1)) / p.sgroups);
    if (s_lo >= s_hi) continue;   // uniform across the CTA
    const int r0 = tile * EXP_R;

    // every warp's bulk stores of the previous item have finished READING the clean tile (see loop end)
    __syncthreads();
    if (threadIdx.x == 0) {
      ptx::mbar_expect_tx(bar, NP * plane_bytes);
      if (FUSED) {
        for (int c = 0; c < 3; ++c) ptx::bulk_load(in + c * tile_px, p.x + ((size_t)(b * 3 + c) * H + r0) * W, plane_bytes, bar);
        for (int c = 0; c < 3; ++c) ptx::bulk_load(in + (3 + c) * tile_px, p.pattern + ((size_t)(b * 3 + c) * H + r0) * W, plane_bytes, bar);
        ptx::bulk_load(in + 6 * tile_px, p.mask + ((size_t)b * H + r0) * W, plane_bytes, bar);
      } else {
        for (int c = 0; c < 3; ++c) ptx::bulk_load(in + c * tile_px, p.img + ((size_t)(b * 3 + c) * H + r0) * W, plane_bytes, bar);
      }
    }
    // rectangle cache of this item's samples (hides the per-sample global-load latency)
    const bool cached = !BANK && p.rects != nullptr && (s_hi - s_lo) <= EXP_RCACHE;
    if (cached)
      for (int i = threadIdx.x; i < 2 * (s_hi - s_lo); i += EXP_THREADS)
        srect[i] = __ldg(occl::row(p.rects, s_lo) + i);
    ptx::mbar_wait(bar, phase);
    phase ^= 1u;

    const float sc = FUSED ? p.scale[b] : 1.0f;
    for (int i = threadIdx.x; i < tile_px; i += EXP_THREADS) {
      float v[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float a = in[c * tile_px + i];
        if (FUSED) {
          const float d = __fmul_rn(__fmul_rn(in[6 * tile_px + i], __fsub_rn(in[(3 + c) * tile_px + i], a)), sc);
          a = __fadd_rn(a, d);
        }
        v[c] = __fmul_rn(__fsub_rn(a, 0.5f), 2.0f);   // (a - 0.5) / 0.5
      }
#pragma unroll
      for (int c = 0; c < CP; ++c) clean[i * CP + c] = from_float<T>(c < 3 ? v[c] : 0.f);
    }
    ptx::fence_proxy_async();
    __syncthreads();

    // ---- one warp per EOT sample (measured: splitting a touched tile's rows across the warps is 1.5x slower --
    //      every warp then decodes every sample's rectangles) -----------------------------------------------
    for (int n = s_lo + warp; n < s_hi; n += EXP_WARPS) {
      unsigned char* dst = reinterpret_cast<unsigned char*>(p.out) + ((size_t)(n - p.n0) * HW + (size_t)r0 * W) * CP * sizeof(T);
      int rr0[4], rr1[4], el[4], eh[4];
      bool any = false;
      [[maybe_unused]] int2 sel;
      [[maybe_unused]] const int nw = occl_bank::words(W);
      if constexpr (BANK) {                                     // any bit set in the tile's rows?
        sel = occl_bank::select(p.bank, n);
        uint32_t t = 0u;
        for (int i = lane; i < EXP_R * nw; i += 32) t |= occl_bank::row_bits(p.bank, sel, r0 + i / nw, i % nw);
        any = __any_sync(0xffffffffu, t != 0u);
      } else if (p.rects != nullptr) {
        const Occlusion occ(cached ? occl::load_shared(srect + 2 * (n - s_lo)) : occl::load(p.rects, n));
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          occ.span(k, CP, rr0[k], rr1[k], el[k], eh[k]);
          any = any || (rr0[k] < r0 + EXP_R && rr1[k] > r0);
        }
      }
      const bool use_bulk = p.mode == 0;
      if (!any && use_bulk) {                                   // whole tile untouched: one bulk store
        if (lane == 0) { ptx::bulk_store(dst, clean_b, out_bytes); ptx::bulk_commit(); }
        continue;
      }
      // Row-independent part, once per sample: field j (EPC bits) of zm[k] = which elements of this lane's chunk
      // (cb + lane + 32 j) rectangle k zeroes -- all ones inside, zero outside, a bit range on the <= 2 chunks that
      // straddle an edge.  A row then only ORs the words of the rectangles that cover it.
      constexpr int JB = 32 / EPC;                              // chunks per lane per mask word (4 bf16 / 8 fp32)
      constexpr uint32_t FULL = (1u << EPC) - 1u;
      for (int cb = 0; cb < row_chunks; cb += 32 * JB) {        // one pass for rows up to 2048 B (bf16) / 4096 B (fp32)
        uint32_t zm[4];
#pragma unroll
        for (int k = 0; k < (BANK ? 0 : 4); ++k) {
          uint32_t z = 0u;
#pragma unroll
          for (int j = 0; j < JB; ++j) {
            const int e0 = (cb + lane + 32 * j) * EPC;
            const int lo = min(max(el[k] - e0, 0), EPC), hi = min(max(eh[k] - e0, 0), EPC);
            const uint32_t m = hi > lo ? (((1u << hi) - 1u) & ~((1u << lo) - 1u)) : 0u;
            z |= m << (EPC * j);
          }
          zm[k] = z;
        }
        for (int rr = 0; rr < EXP_R; ++rr) {
          const int row = r0 + rr;
          uint32_t Z = 0u;
          bool rany = false;
          if constexpr (BANK) {
            // lane k holds word k of the row; field j of Z from the <= 2 words under the pixels of chunk cb + lane + 32 j
            const uint32_t wv = lane < nw ? occl_bank::row_bits(p.bank, sel, row, lane) : 0u;
            rany = __any_sync(0xffffffffu, wv != 0u);
#pragma unroll (CP == 3 ? 1 : JB)                         // (unrolled at C = 3 this loop takes 112 registers)
            for (int j = 0; j < JB; ++j) {
              const int e0 = (cb + lane + 32 * j) * EPC, px0 = e0 / CP, k0 = px0 >> 5, off = e0 - px0 * CP;
              const uint32_t w0 = __shfl_sync(0xffffffffu, wv, k0 & 31), w1 = __shfl_sync(0xffffffffu, wv, (k0 + 1) & 31);
              const uint32_t bits = __funnelshift_r(w0, k0 + 1 < nw ? w1 : 0u, px0 & 31);   // bit i: pixel px0 + i
              uint32_t m = 0u;
#pragma unroll
              for (int k = 0; k < (CP + EPC - 2) / CP + 1; ++k) {   // the pixels a chunk can touch: elements [k CP - off, (k + 1) CP - off)
                const int lo = max(k * CP - off, 0), hi = min((k + 1) * CP - off, EPC);
                if (hi > lo && ((bits >> k) & 1u)) m |= ((1u << hi) - 1u) & ~((1u << lo) - 1u);
              }
              Z |= m << (EPC * j);
            }
          } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const bool cov = row >= rr0[k] && row < rr1[k];
              rany = rany || cov;
              Z |= cov ? zm[k] : 0u;
            }
          }
          if (!rany && use_bulk) {                              // clean row: bulk store
            if (cb == 0 && lane == 0) { ptx::bulk_store(dst + (size_t)rr * row_bytes, clean_b + (size_t)rr * row_bytes, row_bytes); ptx::bulk_commit(); }
            continue;
          }
          const uint4* crow = reinterpret_cast<const uint4*>(clean_b + (size_t)rr * row_bytes);
          uint4* drow = reinterpret_cast<uint4*>(dst + (size_t)rr * row_bytes);
#pragma unroll
          for (int j = 0; j < JB; ++j) {
            const int ch = cb + lane + 32 * j;
            if (ch >= row_chunks) break;
            const uint32_t m = (Z >> (EPC * j)) & FULL;
            uint4 v = make_uint4(0u, 0u, 0u, 0u);
            if (m != FULL) {
              v = crow[ch];
              if (m != 0u) {                                    // edge chunk: clear the covered elements
                if (EPC == 8) {                                 // two 16-bit elements per word
                  v.x &= ~(((m & 1u) ? 0xffffu : 0u) | ((m & 2u) ? 0xffff0000u : 0u));
                  v.y &= ~(((m & 4u) ? 0xffffu : 0u) | ((m & 8u) ? 0xffff0000u : 0u));
                  v.z &= ~(((m & 16u) ? 0xffffu : 0u) | ((m & 32u) ? 0xffff0000u : 0u));
                  v.w &= ~(((m & 64u) ? 0xffffu : 0u) | ((m & 128u) ? 0xffff0000u : 0u));
                } else {
                  if (m & 1u) v.x = 0u;
                  if (m & 2u) v.y = 0u;
                  if (m & 4u) v.z = 0u;
                  if (m & 8u) v.w = 0u;
                }
              }
            }
            drow[ch] = v;
          }
        }
      }
    }
    // before the clean tile is overwritten: each issuing lane waits for its bulk stores' reads
    if (lane == 0) ptx::bulk_wait_read<0>();
  }
  // (global visibility of the bulk stores is guaranteed at kernel completion)
}

// Launch shape.  Work items = images x row tiles (R rows) x sample groups, walked grid-stride by the resident CTAs.
// Measured over tile heights x sample groups x launch sizes (tools/k1_step_sweep.py, on the GPU this rule was first tuned on;
// the sweep has not been repeated on the H100): tiles of
// 4-8 rows are equivalent and best (a CTA's load + compose prologue stays short and 3-6 CTAs per SM overlap it with their
// neighbours' stores), 14-16 rows lose 10-30 % (1-2 CTAs per SM, the prologue is exposed), 2 rows lose 15-20 % (per-item
// overhead), and a launch wants >= 4 items per SM.  Rule: R = 8, or 4 when that leaves fewer than 4 items per SM; sample
// groups (each re-loads and re-composes the tile) only when the images alone give fewer than 2 items per SM (B = 1).
// A rule that maximised "wave efficiency" picked R = 14 for 512- and 2048-sample launches and was far slower than R = 8.
// DORPATCH_K1_ROWS / _K1_SG (or dp_debug_k1_tuning) pin the choice.
static int g_k1_rows = -2, g_k1_sg = -1, g_k1_mode = 0;   // launch-shape overrides (environment, or set_expand_tuning for sweeps)
static int g_k1_last[4] = {0, 0, 0, 0};                    // tile rows, sample groups, grid, resident CTAs per SM of the last launch
void get_expand_last(int* out4) { for (int i = 0; i < 4; ++i) out4[i] = g_k1_last[i]; }
void set_expand_tuning(int rows, int sg, int mode) { g_k1_rows = rows < 0 ? 0 : rows; g_k1_sg = sg < 0 ? 0 : sg; g_k1_mode = mode; }

template <typename T, int CP, bool FUSED, bool BANK>
static int expand_launch(const ExpandParams& p, int num_sms, cudaStream_t st) {
  if (g_k1_rows == -2) {
    const char* e = getenv("DORPATCH_K1_ROWS"); g_k1_rows = e ? atoi(e) : 0;
    const char* g = getenv("DORPATCH_K1_SG"); g_k1_sg = g ? atoi(g) : 0;
    const char* m = getenv("DORPATCH_K1_MODE"); g_k1_mode = m ? atoi(m) : 0;
  }
  const int rows_env = g_k1_rows, sg_env = g_k1_sg;
  constexpr int NP = FUSED ? 7 : 3;
  auto smem_of = [&](int R) { return (size_t)EXP_HDR + (size_t)NP * R * p.W * 4 + (size_t)R * p.W * CP * sizeof(T); };
  static int occ_cache[33];
  static bool occ_init = false;
  if (!occ_init) { for (int& v : occ_cache) v = -1; occ_init = true; }
  auto resident = [&](int R) {
    if (occ_cache[R] < 0) {
      const size_t sm = smem_of(R);
      cudaFuncSetAttribute(expand_kernel<T, CP, FUSED, BANK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
      int nb = 0;
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, expand_kernel<T, CP, FUSED, BANK>, EXP_THREADS, sm) != cudaSuccess || nb < 1) { cudaGetLastError(); nb = 1; }
      occ_cache[R] = nb;
    }
    return occ_cache[R];
  };
  const int nb_img = images_touched(p.S, p.n0, p.n);
  auto usable = [&](int R) { return R >= 1 && R <= 32 && p.H % R == 0 && smem_of(R) <= 200 * 1024; };
  int best_R = 0, best_sg = 1;
  if (rows_env > 0 && usable(rows_env)) best_R = rows_env;
  else {
    const int pref[] = {8, 7, 4, 2, 1};
    for (int R : pref)
      if (usable(R)) { if (best_R == 0) best_R = R; if (nb_img * (p.H / R) >= 4 * num_sms || R <= 4) { best_R = R; break; } }
    if (best_R == 0) best_R = 1;
  }
  if (sg_env > 0) best_sg = sg_env;
  else
    while (nb_img * (p.H / best_R) * best_sg < 2 * num_sms && best_sg * 2 * EXP_WARPS <= p.S && best_sg < 32) best_sg *= 2;
  const int items_total = nb_img * (p.H / best_R) * best_sg;
  const int slots = num_sms * resident(best_R);
  const int best_grid = items_total < slots ? items_total : slots;
  const size_t smem = smem_of(best_R);
  cudaFuncSetAttribute(expand_kernel<T, CP, FUSED, BANK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  ExpandParams q = p;
  q.R = best_R;
  q.sgroups = best_sg;
  q.mode = g_k1_mode;
  g_k1_last[0] = best_R; g_k1_last[1] = best_sg; g_k1_last[2] = best_grid; g_k1_last[3] = resident(best_R);
  expand_kernel<T, CP, FUSED, BANK><<<best_grid, EXP_THREADS, smem, st>>>(q);
  return 1;
}

// f(T{}, integral_constant<int, CP>{}) for an activation type and channels per pixel, Cp in {3, 4, 8} (the engine
// checks Cp when it is created)
template <class F>
static void dispatch_t_cp(bool bf16, int Cp, F&& f) {
  auto by_cp = [&](auto t) {
    if (Cp == 8) f(t, std::integral_constant<int, 8>{});
    else if (Cp == 4) f(t, std::integral_constant<int, 4>{});
    else f(t, std::integral_constant<int, 3>{});
  };
  if (bf16) by_cp(__nv_bfloat16{});
  else by_cp(0.f);
}

int launch_expand(const float* img, const float* x, const float* mask, const float* pattern, const float* scale,
                  const int16_t* rects, void* out, int B, int S, int n0, int n, int H, int W, int Cp, bool bf16,
                  bool fused, int num_sms, cudaStream_t st, const MaskBank* bank) {
  ExpandParams p{img, x, mask, pattern, scale, rects, out, B, S, n0, n, H, W, 1, EXP_R_DEFAULT, 0};
  if (bank != nullptr) {                                        // the bank variant expands img only
    if (fused || bank_words(W) > 32) return 0;
    p.bank = *bank;
  }
  int k = 0;
  dispatch_t_cp(bf16, Cp, [&](auto t, auto cp) {
    if (bank != nullptr) k = expand_launch<decltype(t), cp, false, true>(p, num_sms, st);
    else k = fused ? expand_launch<decltype(t), cp, true, false>(p, num_sms, st) : expand_launch<decltype(t), cp, false, false>(p, num_sms, st);
  });
  return k;
}

// =====================================================================================
// Optional affine / colour EOT (SURVEY 8f N3; named by the north-star, absent from the reference --
// default off).  Per sample: bilinear warp of the pasted image by theta (torch affine_grid /
// grid_sample semantics: align_corners=False, padding_mode='border'), then
// v' = clamp(contrast*(v-0.5)+0.5+brightness, 0, 1), then occlusion + normalisation.
// xf[n] = {t00,t01,t02,t10,t11,t12, contrast, brightness}.  Gather kernel (the source rows are
// arbitrary, so no TMA row tiles); its adjoint scatters with fp32 atomics.
// =====================================================================================
struct AffTap { int i00, i01, i10, i11; float w00, w01, w10, w11; };
__device__ __forceinline__ AffTap affine_taps(const float* __restrict__ t, int h, int w, int H, int W) {
  const float xn = (2.f * w + 1.f) / W - 1.f, yn = (2.f * h + 1.f) / H - 1.f;
  float fx = ((t[0] * xn + t[1] * yn + t[2] + 1.f) * W - 1.f) * 0.5f;
  float fy = ((t[3] * xn + t[4] * yn + t[5] + 1.f) * H - 1.f) * 0.5f;
  fx = fminf(fmaxf(fx, 0.f), (float)(W - 1));
  fy = fminf(fmaxf(fy, 0.f), (float)(H - 1));
  const int x0 = (int)floorf(fx), y0 = (int)floorf(fy);
  const float ax = fx - x0, ay = fy - y0;
  const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
  AffTap a;
  a.i00 = y0 * W + x0; a.i01 = y0 * W + x1; a.i10 = y1 * W + x0; a.i11 = y1 * W + x1;
  a.w00 = (1.f - ax) * (1.f - ay); a.w01 = (x0 + 1 < W ? ax : 0.f) * (1.f - ay);
  a.w10 = (1.f - ax) * (y0 + 1 < H ? ay : 0.f); a.w11 = (x0 + 1 < W ? ax : 0.f) * (y0 + 1 < H ? ay : 0.f);
  return a;
}

template <typename T, int CP>
__global__ void __launch_bounds__(256) expand_affine_kernel(const float* __restrict__ adv, const float* __restrict__ xf,
                                                            const int16_t* __restrict__ rects, T* __restrict__ out,
                                                            int S, int n0, int H, int W) {
  const int HW = H * W, n = n0 + blockIdx.y, b = n / S;
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  if (px >= HW) return;
  const int h = px / W, w = px % W;
  const float* t = xf + (size_t)n * 8;
  const AffTap a = affine_taps(t, h, w, H, W);
  const bool occ = rects != nullptr && Occlusion(occl::load(rects, n)).hit(h, w);
  T* o = out + ((size_t)blockIdx.y * HW + px) * CP;
#pragma unroll
  for (int c = 0; c < CP; ++c) {
    float z = 0.f;
    if (c < 3 && !occ) {
      const float* pl = adv + ((size_t)b * 3 + c) * HW;
      float v = a.w00 * pl[a.i00] + a.w01 * pl[a.i01] + a.w10 * pl[a.i10] + a.w11 * pl[a.i11];
      v = fminf(fmaxf(t[6] * (v - 0.5f) + 0.5f + t[7], 0.f), 1.f);
      z = (v - 0.5f) * 2.f;
    }
    o[c] = from_float<T>(z);
  }
}

// adjoint: G[b] += scatter( 2 * keep * contrast * [0 < v' < 1] * dz[n] ); G must be zero-initialised
template <typename T, int CP>
__global__ void __launch_bounds__(256) reduce_affine_kernel(const T* __restrict__ dz, const float* __restrict__ adv,
                                                            const float* __restrict__ xf, const int16_t* __restrict__ rects,
                                                            float* __restrict__ G, int S, int n0, int H, int W) {
  const int HW = H * W, n = n0 + blockIdx.y, b = n / S;
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  if (px >= HW) return;
  const int h = px / W, w = px % W;
  if (rects != nullptr && Occlusion(occl::load(rects, n)).hit(h, w)) return;
  const float* t = xf + (size_t)n * 8;
  const AffTap a = affine_taps(t, h, w, H, W);
  const T* q = dz + ((size_t)blockIdx.y * HW + px) * CP;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float* pl = adv + ((size_t)b * 3 + c) * HW;
    const float v = a.w00 * pl[a.i00] + a.w01 * pl[a.i01] + a.w10 * pl[a.i10] + a.w11 * pl[a.i11];
    const float vc = t[6] * (v - 0.5f) + 0.5f + t[7];
    if (vc < 0.f || vc > 1.f) continue;                 // torch.clamp passes the gradient on [min, max]
    const float g = 2.f * t[6] * to_float(q[c]);
    float* gp = G + ((size_t)b * 3 + c) * HW;
    if (a.w00 != 0.f) atomicAdd(gp + a.i00, a.w00 * g);
    if (a.w01 != 0.f) atomicAdd(gp + a.i01, a.w01 * g);
    if (a.w10 != 0.f) atomicAdd(gp + a.i10, a.w10 * g);
    if (a.w11 != 0.f) atomicAdd(gp + a.i11, a.w11 * g);
  }
}

int launch_expand_affine(const float* adv, const float* xf, const int16_t* rects, void* out, int S, int n0, int n,
                         int H, int W, int Cp, bool bf16, cudaStream_t st) {
  dim3 grid((H * W + 255) / 256, n);
  dispatch_t_cp(bf16, Cp, [&](auto t, auto cp) {
    using T = decltype(t);
    expand_affine_kernel<T, cp><<<grid, 256, 0, st>>>(adv, xf, rects, (T*)out, S, n0, H, W);
  });
  return 1;
}
int launch_reduce_affine(const void* dz, const float* adv, const float* xf, const int16_t* rects, float* G, int S, int n0,
                         int n, int H, int W, int Cp, bool bf16, cudaStream_t st) {
  dim3 grid((H * W + 255) / 256, n);
  dispatch_t_cp(bf16, Cp, [&](auto t, auto cp) {
    using T = decltype(t);
    reduce_affine_kernel<T, cp><<<grid, 256, 0, st>>>((const T*)dz, adv, xf, rects, G, S, n0, H, W);
  });
  return 1;
}

// =====================================================================================
// K4: CW loss / argmax / dlogits -- one warp per sample.  Bit for bit the reference's torch arithmetic (attack.py:16-23,
// restated by oracle.attack.cw_loss) and its autograd gradient, scaled by w:
//   real  = sum_k l[k] * onehot[k]   -> l[y], or NaN when any logit of the row is not finite (0 * inf = NaN)
//   other = max_k ((1 - onehot) * l - onehot * 1e4)   -> the label slot holds -1e4
//   loss  = clamp((confidence + other) - real, min=0)  (untargeted: (confidence + real) - other); NaN stays NaN
// Maxima follow torch's max / argmax: NaN is the largest value, ties go to the lowest index, so the index is in [0, K).
// =====================================================================================
__device__ __forceinline__ bool cw_beats(float v, int i, float b, int bi) {   // does (v, i) replace the running max (b, bi)?
  const bool vn = isnan(v), bn = isnan(b);
  if (vn || bn) return vn && (!bn || i < bi);
  return v > b || (v == b && i < bi);
}
__global__ void cw_kernel(const float* __restrict__ logits, const int32_t* __restrict__ y,
                          const uint8_t* __restrict__ targeted, float confidence, float w, float* __restrict__ loss,
                          int32_t* __restrict__ preds, float* __restrict__ dlogits, int N, int K) {
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (n >= N) return;
  const float* l = logits + (size_t)n * K;
  const int yy = y != nullptr ? y[n] : -1;
  // (-inf, INT_MAX) loses to every (value, index) of the row: a lane without an element never wins
  float best = -INFINITY, obest = -INFINITY; int bi = 0x7fffffff, oi = 0x7fffffff;
  bool finite = true;
  for (int k = lane; k < K; k += 32) {
    const float v = l[k];
    finite = finite && isfinite(v);
    if (cw_beats(v, k, best, bi)) { best = v; bi = k; }
    const float ov = k == yy ? -1e4f : v;   // attack.py:19: the label slot contributes -1e4
    if (cw_beats(ov, k, obest, oi)) { obest = ov; oi = k; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v2 = __shfl_xor_sync(0xffffffffu, best, o); const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
    if (cw_beats(v2, i2, best, bi)) { best = v2; bi = i2; }
    const float w2 = __shfl_xor_sync(0xffffffffu, obest, o); const int j2 = __shfl_xor_sync(0xffffffffu, oi, o);
    if (cw_beats(w2, j2, obest, oi)) { obest = w2; oi = j2; }
  }
  if (lane == 0 && preds != nullptr) preds[n] = bi;
  if (loss == nullptr) return;
  finite = __all_sync(0xffffffffu, finite);
  const float real = finite ? l[yy] : __int_as_float(0x7fffffff);
  const bool tg = targeted[n] != 0;
  const float pre = tg ? __fsub_rn(__fadd_rn(confidence, obest), real) : __fsub_rn(__fadd_rn(confidence, real), obest);
  if (lane == 0) loss[n] = pre < 0.f ? 0.f : pre;
  if (dlogits != nullptr) {
    float* d = dlogits + (size_t)n * K;
    for (int k = lane; k < K; k += 32) d[k] = 0.f;
    __syncwarp();
    const bool other_is_label_slot = oi == yy;   // its -1e4 is a constant: no gradient
    if (lane == 0 && pre >= 0.f) {     // clamp(min=0) passes the gradient where input >= 0 (not NaN)
      d[yy] = tg ? -w : w;
      if (!other_is_label_slot) d[oi] = tg ? w : -w;
    }
  }
}
int launch_cw(const float* logits, const int32_t* y, const uint8_t* targeted, float confidence, float inv_s_total,
              float* loss, int32_t* preds, float* dlogits, int N, int K, cudaStream_t st) {
  const size_t threads = (size_t)N * 32;
  cw_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(logits, y, targeted, confidence, inv_s_total, loss, preds, dlogits, N, K);
  return 1;
}
int launch_argmax(const float* logits, int32_t* preds, int N, int K, cudaStream_t st) {
  const size_t threads = (size_t)N * 32;
  cw_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(logits, nullptr, nullptr, 0.f, 0.f, nullptr, preds, nullptr, N, K);
  return 1;
}

// =====================================================================================
// K1^T reduce: G[b,c,h,w] (+)= 2 * sum_{samples n of image b in [n0,n0+n)} keep_n(h,w) * dz[n,h,w,c]
// grid (ceil(HW/256), images touched)
// =====================================================================================
// BANK: keep_n from the mask bank `bank` (rects unused).
constexpr int RED_MAXS = 128;
template <typename T, int CP, bool BANK>
__global__ void __launch_bounds__(256) reduce_kernel(const T* __restrict__ dz, const int16_t* __restrict__ rects,
                                                     float* __restrict__ G, int S, int n0, int n, int H, int W, MaskBank bank) {
  __shared__ __align__(16) short sr[RED_MAXS * RECT_SHORTS];   // the rows of up to RED_MAXS samples (BANK: their mask indices)
  const int HW = H * W;
  const auto [b, lo, hi, first] = image_span(S, n0, n, blockIdx.y);
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  const int row = px / W, col = px % W;
  float acc[3] = {0.f, 0.f, 0.f};
  for (int base = lo; base < hi; base += RED_MAXS) {
    const int m = min(RED_MAXS, hi - base);
    __syncthreads();
    if constexpr (BANK) {
      for (int i = threadIdx.x; i < m; i += blockDim.x) reinterpret_cast<int2*>(sr)[i] = occl_bank::select(bank, base + i);
    } else {
      for (int i = threadIdx.x; i < m * RECT_SHORTS; i += blockDim.x)
        sr[i] = rects != nullptr ? rects[(size_t)base * RECT_SHORTS + i] : (short)0;
    }
    __syncthreads();
    if (px < HW) {
      for (int j = 0; j < m; ++j) {
        if constexpr (BANK) {
          if (occl_bank::hit(bank, reinterpret_cast<const int2*>(sr)[j], row, col)) continue;
        } else {
          if (occl::hit(sr + j * RECT_SHORTS, row, col)) continue;
        }
        const T* q = dz + ((size_t)(base + j - n0) * HW + px) * CP;
        if (CP * sizeof(T) == 16) {
          Vec<T> v; v.load(q);
          float f[Vec<T>::N]; v.unpack(f);
          acc[0] += f[0]; acc[1] += f[1]; acc[2] += f[2];
        } else {
          acc[0] += to_float(q[0]); acc[1] += to_float(q[1]); acc[2] += to_float(q[2]);
        }
      }
    }
  }
  if (px < HW) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float* g = G + ((size_t)b * 3 + c) * HW + px;
      const float v = 2.0f * acc[c];
      *g = first ? v : (*g + v);
    }
  }
}
int launch_reduce(const void* dz, const int16_t* rects, float* G, int B, int S, int n0, int n, int H, int W,
                  int Cp, bool bf16, cudaStream_t st, const MaskBank* bank) {
  const dim3 grid((H * W + 255) / 256, images_touched(S, n0, n));
  dispatch_t_cp(bf16, Cp, [&](auto t, auto cp) {
    using T = decltype(t);
    if (bank != nullptr) reduce_kernel<T, cp, true><<<grid, 256, 0, st>>>((const T*)dz, nullptr, G, S, n0, n, H, W, *bank);
    else reduce_kernel<T, cp, false><<<grid, 256, 0, st>>>((const T*)dz, rects, G, S, n0, n, H, W, MaskBank{});
  });
  return 1;
}

// =====================================================================================
// structural loss (attack.py:33-45,227-228), reproducing the reference's one-sided gradient
// (quirk Q4): lr[h,w] = |a[h,w]-a[h,w+1]| (raw a[h,W-1] in the last column), gradient only
// through the subtracted (right / lower) neighbour.  One CTA per image.
// =====================================================================================
__device__ __forceinline__ void lv_pair(const float* __restrict__ pl, int h, int w, int H, int W, float& A, float& Bv) {
  const float v = pl[h * W + w];
  A = (w < W - 1) ? fabsf(v - pl[h * W + w + 1]) : v;
  Bv = (h < H - 1) ? fabsf(v - pl[(h + 1) * W + w]) : v;
}
__device__ __forceinline__ float lvx_at(const float* __restrict__ xb, int h, int w, int H, int W) {
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < 3; ++c) { float A, Bv; lv_pair(xb + (size_t)c * H * W, h, w, H, W, A, Bv); s += A + Bv; }
  return s / 3.0f;
}
__global__ void __launch_bounds__(1024) struct_kernel(const float* __restrict__ adv, const float* __restrict__ x,
                                                      float* __restrict__ loss, float* __restrict__ dLs, int H, int W) {
  __shared__ float red[32];
  const int b = blockIdx.x, HW = H * W;
  const float* ab = adv + (size_t)b * 3 * HW;
  const float* xb = x + (size_t)b * 3 * HW;
  float* gb = dLs + (size_t)b * 3 * HW;
  const float inv_hw = 1.0f / (float)HW;
  float s = 0.f;
  for (int i = threadIdx.x; i < HW; i += blockDim.x) {
    const int h = i / W, w = i % W;
    // value at (h,w)
    float mvsum = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float A, Bv; lv_pair(ab + (size_t)c * HW, h, w, H, W, A, Bv);
      mvsum += (A + Bv) * (A > Bv ? Bv : A);
    }
    s += (mvsum / 3.0f) / (lvx_at(xb, h, w, H, W) + 1e-5f);
    // gradient wrt adv[c,h,w]: through lr[h,w-1] and ud[h-1,w]
    const float wl = (w >= 1) ? inv_hw / (3.0f * (lvx_at(xb, h, w - 1, H, W) + 1e-5f)) : 0.f;
    const float wu = (h >= 1) ? inv_hw / (3.0f * (lvx_at(xb, h - 1, w, H, W) + 1e-5f)) : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float* pl = ab + (size_t)c * HW;
      const float v = pl[i];
      float g = 0.f;
      if (w >= 1) {
        float A, Bv; lv_pair(pl, h, w - 1, H, W, A, Bv);
        const float dmv_dA = (A > Bv ? Bv : A) + ((A > Bv) ? 0.f : (A + Bv));
        g += wl * dmv_dA * (-sgn(pl[i - 1] - v));
      }
      if (h >= 1) {
        float A, Bv; lv_pair(pl, h - 1, w, H, W, A, Bv);
        const float dmv_dB = (A > Bv ? Bv : A) + ((A > Bv) ? (A + Bv) : 0.f);
        g += wu * dmv_dB * (-sgn(pl[i - W] - v));
      }
      gb[(size_t)c * HW + i] = g;
    }
  }
  const float tot = block_sum(s, red);
  if (threadIdx.x == 0) loss[b] = tot * inv_hw;
}
int launch_struct(const float* adv_x, const float* x, float* loss_struc, float* dLs, int B, int H, int W, cudaStream_t st) {
  struct_kernel<<<B, 1024, 0, st>>>(adv_x, x, loss_struc, dLs, H, W);
  return 1;
}

// =====================================================================================
// density + group lasso (attack.py:72-80,235-245) for any basic_unit `unit` dividing H == W.  One CTA per image; no
// shared memory scales with the group count (unit = 1 at 224 px is 50 176 groups), and every sum has a fixed order.
//   grp_ss[b][g]  = sum of m^2 over the unit x unit group g          (for d GL / d m = unit*m/sqrt(ss))
//   win_dev[b][w] = 2*(ws_w - mean)/(nw-1) for density window w      (d var / d m inside window w)
// =====================================================================================
__global__ void __launch_bounds__(1024) maskreg_kernel(const float* __restrict__ mask, float* __restrict__ loss_density,
                                                       float* __restrict__ group_lasso, float* __restrict__ win_dev,
                                                       float* __restrict__ grp_ss, int H, int W, int unit) {
  __shared__ float red[32];
  __shared__ float ws[64];
  const int b = blockIdx.x, GW = W / unit, NG = (H / unit) * GW;
  const float* mb = mask + (size_t)b * H * W;
  float gl = 0.f;
  for (int g = threadIdx.x; g < NG; g += blockDim.x) {
    const int gy = g / GW, gx = g % GW;
    float q = 0.f;
    for (int dy = 0; dy < unit; ++dy)
      for (int dx = 0; dx < unit; ++dx) { const float m = mb[(gy * unit + dy) * W + gx * unit + dx]; q = fmaf(m, m, q); }
    grp_ss[(size_t)b * NG + g] = q;
    gl += sqrtf(q);
  }
  gl = block_sum(gl, red);
  if (threadIdx.x == 0) group_lasso[b] = (float)unit * gl;
  // density windows: 8 x 8 windows of (W/8) x (W/8) pixels
  const int win = W / 8, NWX = W / win, NWY = H / win, NW = NWX * NWY;
  if (unit > 1 && win % unit == 0) {
    // one thread per window: its (win/unit)^2 group sums, each in row-major pixel order, added row-major -- the order
    // in which the unit = 7 engine has always summed, kept so that the default path's bits do not move
    if ((int)threadIdx.x < NW) {
      const int wy = threadIdx.x / NWX, wx = threadIdx.x % NWX;
      const float* wb = mb + (size_t)wy * win * W + wx * win;
      const int gpw = win / unit;
      float s = 0.f;
      for (int a = 0; a < gpw; ++a)
        for (int c = 0; c < gpw; ++c) {
          float gs = 0.f;
          for (int dy = 0; dy < unit; ++dy)
            for (int dx = 0; dx < unit; ++dx) gs += wb[(a * unit + dy) * W + c * unit + dx];
          s += gs;
        }
      ws[threadIdx.x] = s;
    }
  } else {
    // groups of one pixel, or groups straddling / exceeding the window: its pixels, 16 threads per window (rows
    // strided over them, a fixed shuffle tree across the 16)
    const int w = threadIdx.x >> 4, part = threadIdx.x & 15;
    float s = 0.f;
    if (w < NW) {
      const float* wb = mb + (size_t)(w / NWX) * win * W + (w % NWX) * win;
      for (int y = part; y < win; y += 16)
#pragma unroll 7
        for (int x = 0; x < win; ++x) s += wb[y * W + x];
    }
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (w < NW && part == 0) ws[w] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float mean = 0.f;
    for (int i = 0; i < NW; ++i) mean += ws[i];
    mean /= NW;
    float var = 0.f;
    for (int i = 0; i < NW; ++i) { const float d = ws[i] - mean; var += d * d; }
    loss_density[b] = var / (NW - 1);
    for (int i = 0; i < NW; ++i) win_dev[(size_t)b * 64 + i] = 2.0f * (ws[i] - mean) / (NW - 1);
  }
}
int launch_maskreg(const float* mask, float* loss_density, float* group_lasso, float* win_dev, float* grp_ss,
                   int B, int H, int W, int unit, cudaStream_t st) {
  maskreg_kernel<<<B, 1024, 0, st>>>(mask, loss_density, group_lasso, win_dev, grp_ss, H, W, unit);
  return 1;
}

// =====================================================================================
// K3 update: d/d pattern = m * c * g,  d/d mask = c * sum_ch (p-x) * g + density*dDen + coeff*dGL,
// with g = G + structured * dLs; then theta -= lr * sign(grad), clip.
// =====================================================================================
__global__ void __launch_bounds__(256) update_kernel(const float* __restrict__ x, float* __restrict__ mask,
                                                     float* __restrict__ pattern, const float* __restrict__ G,
                                                     const float* __restrict__ dLs, const float* __restrict__ scale,
                                                     const float* __restrict__ win_dev, const float* __restrict__ grp_ss,
                                                     const float* __restrict__ lr, const float* __restrict__ structured,
                                                     const float* __restrict__ coeff_gl, float density, float lo, float hi,
                                                     int stage, float* __restrict__ gp_out, float* __restrict__ gm_out,
                                                     const float* __restrict__ gp_bias, int H, int W, int unit) {
  const int b = blockIdx.y, HW = H * W;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= HW) return;
  const float c = scale[b], step = lr[b], st = structured[b];
  const float m = mask[(size_t)b * HW + i];
  float gm = 0.f;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const size_t o = ((size_t)b * 3 + ch) * HW + i;
    float g = G[o];
    if (st != 0.f) g = fmaf(st, dLs[o], g);
    const float pv = pattern[o], xv = x[o];
    float gp = m * c * g;
    if (gp_bias != nullptr) gp = gp_bias[o] + gp;
    gm = fmaf((pv - xv) * c, g, gm);
    if (gp_out != nullptr) gp_out[o] = gp;
    if (step != 0.f) pattern[o] = fminf(fmaxf(pv - step * sgn(gp), lo), hi);
  }
  if (stage == 0) {
    const int h = i / W, w = i % W;
    const int win = W / 8;
    const float dden = win_dev[(size_t)b * 64 + (h / win) * (W / win) + (w / win)];
    const float ss = grp_ss[(size_t)b * (H / unit) * (W / unit) + (h / unit) * (W / unit) + (w / unit)];
    const float dgl = (float)unit * m / sqrtf(ss);     // 0/0 = NaN for an all-zero group (quirk Q5)
    if (density != 0.f) gm = fmaf(density, dden, gm);
    gm = fmaf(coeff_gl[b], dgl, gm);
    if (gm_out != nullptr) gm_out[(size_t)b * HW + i] = gm;
    if (step != 0.f) mask[(size_t)b * HW + i] = fminf(fmaxf(m - step * sgn(gm), lo), hi);
  }
}
int launch_update(const float* x, float* mask, float* pattern, const float* G, const float* dLs,
                  const float* scale, const float* win_dev, const float* grp_ss, const float* lr,
                  const float* structured, const float* coeff_gl, float density, float lo, float hi, int stage,
                  float* gp_out, float* gm_out, const float* gp_bias, int B, int H, int W, int unit, cudaStream_t st) {
  update_kernel<<<dim3((H * W + 255) / 256, B), 256, 0, st>>>(x, mask, pattern, G, dLs, scale, win_dev, grp_ss, lr,
                                                              structured, coeff_gl, density, lo, hi, stage, gp_out,
                                                              gm_out, gp_bias, H, W, unit);
  return 1;
}

// =====================================================================================
// k x k window sums (patch_selection's group importance, attack.py:365-368)
// =====================================================================================
__global__ void window_sum_kernel(const float* __restrict__ t, float* __restrict__ out, int H, int W, int k, int square) {
  const int b = blockIdx.y, GW = W / k, NG = (H / k) * GW;
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= NG) return;
  const float* tb = t + (size_t)b * H * W;
  const int gy = g / GW, gx = g % GW;
  float s = 0.f;
  for (int dy = 0; dy < k; ++dy)
    for (int dx = 0; dx < k; ++dx) { const float v = tb[(gy * k + dy) * W + gx * k + dx]; s += square ? v * v : v; }
  out[(size_t)b * NG + g] = s;
}
int launch_window_sum(const float* t, float* out, int B, int H, int W, int k, bool square, cudaStream_t st) {
  const int NG = (H / k) * (W / k);
  window_sum_kernel<<<dim3((NG + 127) / 128, B), 128, 0, st>>>(t, out, H, W, k, square ? 1 : 0);
  return 1;
}

// =====================================================================================
// Failed-mask set on the device (SURVEY 8f N2; attack.py:259-267): per image a bitmap over the mask universe.
// One step's update: the first nff[b] sampled indices came from the failed set -- those whose sample now succeeds
// (loss < thresh) leave it; the remaining indices came from the whole universe -- those whose sample fails join it.
// Removal is applied before addition (the reference's setdiff1d precedes its unique), then the popcount is returned.
// One CTA per image; words = ceil(n_mask / 32).
// =====================================================================================
__global__ void failed_update_kernel(uint32_t* __restrict__ bits, int words, const int32_t* __restrict__ idx, const float* __restrict__ loss,
                                     const int32_t* __restrict__ nff, const uint8_t* __restrict__ active, int S, float thresh,
                                     int32_t* __restrict__ count) {
  const int b = blockIdx.x;
  uint32_t* w = bits + (size_t)b * words;
  __shared__ int red[32];
  if (active[b]) {
    const int n_ff = nff[b];
    for (int s = threadIdx.x; s < n_ff; s += blockDim.x)
      if (loss[(size_t)b * S + s] < thresh) { const int k = idx[(size_t)b * S + s]; atomicAnd(&w[k >> 5], ~(1u << (k & 31))); }
    __syncthreads();
    for (int s = n_ff + threadIdx.x; s < S; s += blockDim.x)
      if (!(loss[(size_t)b * S + s] < thresh)) { const int k = idx[(size_t)b * S + s]; atomicOr(&w[k >> 5], 1u << (k & 31)); }
    __syncthreads();
  }
  int c = 0;
  for (int i = threadIdx.x; i < words; i += blockDim.x) c += __popc(w[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) { int t = 0; for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i]; count[b] = t; }
}
int launch_failed_update(uint32_t* bits, int words, const int32_t* idx, const float* loss, const int32_t* nff, const uint8_t* active,
                         int B, int S, float thresh, int32_t* count, cudaStream_t st) {
  failed_update_kernel<<<B, 128, 0, st>>>(bits, words, idx, loss, nff, active, S, thresh, count);
  return 1;
}

// =====================================================================================
// On-device EOT draw (DorPatch.generate(eot_sampler="device"); the semantics of attack.py:193-218, not numpy's stream).
// One CTA per image.  For draw d (0; 1 = the dual draw) of image b at step (stage, iter):
//   n_ff = iter >= 1000 ? min(|F_b|, S/2) : 0, |F_b| = the set bits of the image's failed bitmap below n_mask;
//   positions [0, n_ff): n_ff distinct members of F_b (distinct ranks, each mapped to its set bit by prefix popcounts);
//   positions [n_ff, S): S - n_ff distinct universe indices, drawn independently of the first part.
// Each part is Floyd's exact sampling without replacement (a membership bitmap in shared memory) followed by a
// Fisher-Yates shuffle, so every ordered selection is equally likely and any slice of positions is a uniform sample.
// Every random number is Philox4x32-10 keyed by seed_b at the counter (position, iter, stage | draw | part, attempt):
// a draw depends on nothing but (seed_b, stage, iter) and the image's set -- not on B, the other images, the rank or on
// whether the launch is replayed from a graph.  Then the CTA gathers its local slice [rank_lo, rank_lo + S_loc) of the
// universe table [n_mask][k][4] into rects [B][S_loc][4][4] (masks.gather's layout: the k rectangles in slots 0..k-1, the
// dual draw's in slots 2-3, the rest empty).  An inactive image is left untouched.
// =====================================================================================
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u; k.y += 0xBB67AE85u;
  }
  return c;
}
// Uniform integer in [0, n), n >= 1: Lemire's multiply-shift with rejection of the 2^32 mod n low products (exact).
// The candidates are the four words of each Philox block, attempt 0, 1, ... in the counter's last word.
__device__ __forceinline__ uint32_t draw_below(uint2 key, uint32_t pos, uint32_t iter, uint32_t tag, uint32_t n) {
  const uint32_t reject = (0u - n) % n;
  for (uint32_t attempt = 0;; ++attempt) {
    const uint4 r = philox4x32_10(make_uint4(pos, iter, tag, attempt), key);
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint64_t m = (uint64_t)w[j] * n;
      if ((uint32_t)m >= reject) return (uint32_t)(m >> 32);
    }
  }
}
// m distinct values of [0, n) into out[0..m) in uniformly random order, by the whole CTA.  `seen` holds ceil(n/32)
// zeroed words and is left dirty; tmp is scratch of m words.  tag: stage | draw << 8 | part << 16, the Floyd pass and
// the shuffle taking parts p and p + 1.  The random numbers do not depend on each other and are drawn in parallel; the
// membership pass and the swaps are serial (thread 0).
__device__ void sample_distinct(uint2 key, uint32_t iter, uint32_t tag, int n, int m, uint32_t* seen, int32_t* out, int32_t* tmp) {
  for (int s = threadIdx.x; s < m; s += blockDim.x) {
    out[s] = (int32_t)draw_below(key, (uint32_t)s, iter, tag, (uint32_t)(n - m + s) + 1u);   // Floyd step s: one of [0, n - m + s]
    if (s > 0) tmp[s] = (int32_t)draw_below(key, (uint32_t)s, iter, tag + (1u << 16), (uint32_t)s + 1u);   // Fisher-Yates
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int s = 0; s < m; ++s) {                        // Floyd: a value already taken is replaced by j = n - m + s
      int t = out[s];
      if (seen[t >> 5] & (1u << (t & 31))) t = n - m + s;
      seen[t >> 5] |= 1u << (t & 31);
      out[s] = t;
    }
    for (int s = m - 1; s > 0; --s) { const int u = tmp[s]; const int32_t v = out[s]; out[s] = out[u]; out[u] = v; }
  }
  __syncthreads();
}

struct DrawShape { int B, S, n_mask, k, dual, S_loc, lo; };
__global__ void __launch_bounds__(256) eot_draw_kernel(const uint32_t* __restrict__ failed_bits, int failed_words,
                                                       const int16_t* __restrict__ table, const uint64_t* __restrict__ seeds,
                                                       const int32_t* __restrict__ step, const uint8_t* __restrict__ active,
                                                       DrawShape sh, int32_t* __restrict__ idx, int32_t* __restrict__ idx2,
                                                       int32_t* __restrict__ nff, int16_t* __restrict__ rects,
                                                       int32_t* __restrict__ tmp) {
  extern __shared__ uint32_t draw_smem[];
  const int b = blockIdx.x;
  if (!active[b]) return;
  const int words = (sh.n_mask + 31) >> 5;
  uint32_t* seen = draw_smem;                            // [words] Floyd membership bitmap
  int* prefix = (int*)(draw_smem + words);               // [words] set bits of the failed bitmap before each word
  __shared__ int part_sum[256], n_set_s;
  const uint32_t* fb = failed_bits + (size_t)b * failed_words;
  const uint32_t last = (sh.n_mask & 31) ? (1u << (sh.n_mask & 31)) - 1u : ~0u;
  auto fword = [&](int w) { return w < words - 1 ? fb[w] : (fb[w] & last); };
  // exclusive prefix popcounts: each thread one contiguous run of words, then a scan over the 256 run sums
  const int per = (words + blockDim.x - 1) / blockDim.x, w0 = threadIdx.x * per, w1 = min(words, w0 + per);
  int c = 0;
  for (int w = w0; w < w1; ++w) c += __popc(fword(w));
  part_sum[threadIdx.x] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int t = 0; t < (int)blockDim.x; ++t) { const int v = part_sum[t]; part_sum[t] = acc; acc += v; }
    n_set_s = acc;
  }
  __syncthreads();
  c = part_sum[threadIdx.x];
  for (int w = w0; w < w1; ++w) { prefix[w] = c; c += __popc(fword(w)); }
  const int n_set = n_set_s;
  const int n_ff = step[1] >= 1000 ? min(n_set, sh.S / 2) : 0;
  const uint2 key = make_uint2((uint32_t)seeds[b], (uint32_t)(seeds[b] >> 32));
  const uint32_t iter = (uint32_t)step[1];
  if (threadIdx.x == 0) nff[b] = n_ff;
  for (int d = 0; d <= sh.dual; ++d) {
    int32_t* row = (d ? idx2 : idx) + (size_t)b * sh.S;
    const uint32_t tag = (uint32_t)step[0] | ((uint32_t)d << 8);
    for (int part = 0; part < 2; ++part) {               // 0: ranks into F_b, 1: universe indices
      const int n = part ? sh.n_mask : n_set, m = part ? sh.S - n_ff : n_ff;
      if (m == 0) continue;
      for (int w = threadIdx.x; w < words; w += blockDim.x) seen[w] = 0u;
      __syncthreads();
      sample_distinct(key, iter, tag | ((uint32_t)(2 * part) << 16), n, m, seen, row + (part ? n_ff : 0), tmp + (size_t)b * sh.S);
    }
    for (int s = threadIdx.x; s < n_ff; s += blockDim.x) {   // rank r -> the r-th set bit of F_b
      const int r = row[s];
      int lo = 0, hi = words - 1;                        // the last word whose prefix is <= r
      while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (prefix[mid] <= r) lo = mid; else hi = mid - 1; }
      uint32_t v = fword(lo);
      for (int skip = r - prefix[lo]; skip > 0; --skip) v &= v - 1u;
      row[s] = lo * 32 + __ffs(v) - 1;
    }
    __syncthreads();
  }
  for (int e = threadIdx.x; e < sh.S_loc * RECT_SHORTS; e += blockDim.x) {
    const int s = e / RECT_SHORTS, slot = (e % RECT_SHORTS) >> 2, q = e & 3;
    int16_t v = 0;
    if (slot < sh.k) v = table[((size_t)idx[(size_t)b * sh.S + sh.lo + s] * sh.k + slot) * 4 + q];
    else if (sh.dual && slot >= 2) v = table[((size_t)idx2[(size_t)b * sh.S + sh.lo + s] * sh.k + slot - 2) * 4 + q];
    rects[((size_t)b * sh.S_loc + s) * RECT_SHORTS + e % RECT_SHORTS] = v;
  }
}
size_t eot_draw_smem_bytes(int n_mask) { return (size_t)2 * ((n_mask + 31) / 32) * 4; }
int launch_eot_draw(const uint32_t* failed_bits, int failed_words, const int16_t* table, int n_mask, int k, const uint64_t* seeds,
                    const int32_t* step, const uint8_t* active, int B, int S, int dual, int S_loc, int lo, int32_t* idx,
                    int32_t* idx2, int32_t* nff, int16_t* rects, int32_t* tmp, cudaStream_t st) {
  const size_t smem = eot_draw_smem_bytes(n_mask);
  if (smem > (48 << 10)) cudaFuncSetAttribute(eot_draw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  eot_draw_kernel<<<B, 256, smem, st>>>(failed_bits, failed_words, table, seeds, step, active, DrawShape{B, S, n_mask, k, dual, S_loc, lo},
                                        idx, idx2, nff, rects, tmp);
  return 1;
}

}  // namespace dp
