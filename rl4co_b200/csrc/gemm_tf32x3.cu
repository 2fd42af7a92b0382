// fp32-accurate GEMM on Hopper tensor cores (wgmma, kind tf32, 3xTF32 split).
//
//   C[M, Nout] = epilogue( A[M, K] @ W[Nout, K]^T )        A, W, C: fp32 row-major
//   epilogue(v) = ((v + bias[n]) (+ residual[m, n])) (relu) * scale[n] + shift[n]
//
// Serves the dense projections either side of the rollout loop:
//   * FusedAttentionModelDecoder._precompute_cache (rl4co/models/zoo/am/decoder.py:201-228):
//     embeddings[B*N,128] @ Wcat[640,128]^T -> fused rollout cache;
//   * the AM encoder's Linear layers (rl4co/models/nn/attention.py:110-134, nn/mlp.py:45-60,
//     nn/graph/attnnet.py:45-52) with bias / ReLU / skip connection / eval-mode BatchNorm folded
//     into the epilogue.
//
// Numerics: each fp32 operand x is split into hi = rna_tf32(x) and lo = x - hi; the kernel
// accumulates hi*hi + lo*hi + hi*lo in fp32 register accumulators (the dropped lo*lo term is
// ~2^-22 relative), i.e. fp32-class accuracy (~1e-6 relative) at tensor-core rate.
//
// Structure: persistent CTAs of three warpgroups; a CTA keeps one 128-column block of W and walks over 128-row tiles.
//   warpgroup 0  producer : LDG the next 32-wide k-block of A (one block ahead, in registers) -> hi / lo split -> STS
//                           into a 3-stage ring of 128-byte-swizzled K-major tiles (row r at r*128 B, 16-byte chunk c
//                           stored at c ^ (r & 7); SBO = 1 KB) -> fence.proxy.async -> mbarrier "full"
//   warpgroups 1-2 consumers: 64 rows x 128 columns each; per k-block 12 wgmma m64n128k8 (4 k-steps x 3 products
//                           hi*hi, lo*hi, hi*lo), one batch in flight while the previous stage is released; the fused
//                           epilogue runs from the accumulator registers (a quad stores 32 contiguous bytes of a row)
//                           while the producer already fills the ring for the next tile.
//   K == 128 (every projection of the encoder / cache): the CTA's W block (hi + lo, 128 KB) stays in shared memory and
//   the ring carries A only; otherwise the ring stages carry the k-block of W as well.
#include "co_common.cuh"
#include "wgmma.cuh"

namespace co {

constexpr int GM = 128, GN = 128, GK = 32;
constexpr int TILE_BYTES = GM * GK * 4;  // 16 KB per operand tile
constexpr uint32_t SBO = 1024;           // 8 rows x 128 B swizzle atom
constexpr int KB128 = 4;                 // k-blocks of the W-stationary variant
constexpr int STAGES = 3;
constexpr int GEMM_THREADS = 384;
constexpr int GEMM_SMEM = 2 * KB128 * TILE_BYTES + STAGES * 2 * TILE_BYTES;  // == STAGES * 4 * TILE_BYTES + 32 KB spare

__device__ __forceinline__ float4 split_hi(float4 v) {
  return make_float4(wg::rna_tf32(v.x), wg::rna_tf32(v.y), wg::rna_tf32(v.z), wg::rna_tf32(v.w));
}
__device__ __forceinline__ float4 sub4(float4 a, float4 b) { return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }

__global__ void split_tf32_kernel(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo, long n) {
  long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float v = w[i], h = wg::rna_tf32(v);
    hi[i] = h;
    lo[i] = v - h;
  }
}

struct GemmArgs {
  const float* A; const float* Whi; const float* Wlo; float* C;
  const float* bias; const float* residual; const float* scale; const float* shift;
  int M, Nout, K, lda, ldc, ldr, relu, n_tiles;
};

// fused epilogue of one consumer warpgroup straight from its accumulator fragment: rows m0 + {g, g + 8}, column pairs
// n0 + 8 j + 2 q (wgmma.cuh)
__device__ __forceinline__ void epilogue_regs(const GemmArgs& g, const float (&d)[64], int m0, int n0, int lane) {
  const int q = lane & 3;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int n = n0 + 8 * j + 2 * q;
    if (n >= g.Nout) continue;
    float2 bs = make_float2(0.f, 0.f), sc = make_float2(1.f, 1.f), sh = bs;
    if (g.bias) bs = __ldg(reinterpret_cast<const float2*>(g.bias + n));
    if (g.scale) { sc = __ldg(reinterpret_cast<const float2*>(g.scale + n)); sh = __ldg(reinterpret_cast<const float2*>(g.shift + n)); }
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int row = m0 + (lane >> 2) + 8 * half;
      if (row >= g.M) continue;
      float2 o = make_float2(d[4 * j + 2 * half] + bs.x, d[4 * j + 2 * half + 1] + bs.y);
      if (g.residual) {
        // plain (coherent) load: the residual may alias C (in-place accumulation across split-K passes)
        const float2 r = *reinterpret_cast<const float2*>(g.residual + (size_t)row * g.ldr + n);
        o.x += r.x; o.y += r.y;
      }
      if (g.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
      if (g.scale) { o.x = fmaf(o.x, sc.x, sh.x); o.y = fmaf(o.y, sc.y, sh.y); }
      *reinterpret_cast<float2*>(g.C + (size_t)row * g.ldc + n) = o;
    }
  }
}

// one k-block of a producer thread: 8 x (4 rows x 128 B) of A and, unless W is resident, of W_hi / W_lo
template <bool WSTAT>
struct KBlock {
  float4 a[8];
  float4 h[WSTAT ? 1 : 8], l[WSTAT ? 1 : 8];
};

template <bool WSTAT>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_tf32x3_kernel(const GemmArgs g, int m_tiles, int groups) {
  extern __shared__ __align__(1024) unsigned char smem[];
  // WSTAT: [kb][W_hi, W_lo] (128 KB) then the ring of [A_hi, A_lo]; else a ring of [A_hi, A_lo, W_hi, W_lo]
  constexpr int STAGE_BYTES = (WSTAT ? 2 : 4) * TILE_BYTES;
  unsigned char* sW = smem;
  unsigned char* sRing = smem + (WSTAT ? 2 * KB128 * TILE_BYTES : 0);
  __shared__ __align__(8) uint64_t bars[2 * STAGES];  // full[STAGES] (128 producers), empty[STAGES] (256 consumers)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_tile = blockIdx.x % g.n_tiles, group = blockIdx.x / g.n_tiles;
  const int n0 = n_tile * GN;
  const int nkb = g.K / GK;
  const uint32_t bar0 = wg::s32(bars);
  auto FULL_B = [&](int s) { return bar0 + 8 * s; };
  auto EMPTY_B = [&](int s) { return bar0 + 8 * (STAGES + s); };

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { wg::bar_init(FULL_B(s), 128); wg::bar_init(EMPTY_B(s), 256); }
    wg::bar_init_fence();
  }
  if (WSTAT) {
    // resident W block: item = (kb, row-group, chunk-half); a warp covers 8 rows x 4 chunks
    const int r8 = lane & 7, c4 = lane >> 3;
    for (int item = warp; item < KB128 * 32; item += GEMM_THREADS / 32) {
      const int kb = item >> 5, qq = item & 31;
      const int rg = qq >> 1, chunk = 4 * (qq & 1) + c4, row = 8 * rg + r8;
      const uint32_t soff = rg * SBO + r8 * 128 + ((chunk ^ r8) << 4);
      float4 h = make_float4(0.f, 0.f, 0.f, 0.f), l = h;
      if (n0 + row < g.Nout) {
        h = __ldg(reinterpret_cast<const float4*>(g.Whi + (size_t)(n0 + row) * g.K + kb * GK + chunk * 4));
        l = __ldg(reinterpret_cast<const float4*>(g.Wlo + (size_t)(n0 + row) * g.K + kb * GK + chunk * 4));
      }
      *reinterpret_cast<float4*>(sW + (2 * kb) * TILE_BYTES + soff) = h;
      *reinterpret_cast<float4*>(sW + (2 * kb + 1) * TILE_BYTES + soff) = l;
    }
    wg::fence_async();
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------------------------ producer warpgroup
    // lane -> (row % 4, 16-byte chunk 0..7): every LDG.128 instruction fetches 4 complete 128-byte
    // rows of the k-block, and a quarter-warp writes one swizzled 128-byte row (conflict-free)
    const int r4 = lane >> 3, c8 = lane & 7;
    auto load = [&](int mt, int kb, auto& R) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int lrow = 16 * j + 4 * warp + r4;
        const int row = mt * GM + lrow;
        R.a[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (mt < m_tiles && row < g.M)
          R.a[j] = __ldg(reinterpret_cast<const float4*>(g.A + (size_t)row * g.lda + kb * GK + c8 * 4));
        if constexpr (!WSTAT) {
          R.h[j] = R.l[j] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (mt < m_tiles && n0 + lrow < g.Nout) {
            R.h[j] = __ldg(reinterpret_cast<const float4*>(g.Whi + (size_t)(n0 + lrow) * g.K + kb * GK + c8 * 4));
            R.l[j] = __ldg(reinterpret_cast<const float4*>(g.Wlo + (size_t)(n0 + lrow) * g.K + kb * GK + c8 * 4));
          }
        }
      }
    };
    KBlock<WSTAT> R;
    KBlock<true> Rn;  // W-stationary: a second register set keeps the next block of A in flight
    load(group, 0, R);
    uint32_t it = 0;
    for (int mt = group; mt < m_tiles; mt += groups) {
      for (int kb = 0; kb < nkb; ++kb, ++it) {
        auto load_next = [&](auto& dst) { if (kb + 1 < nkb) load(mt, kb + 1, dst); else load(mt + groups, 0, dst); };
        if constexpr (WSTAT) load_next(Rn);
        const int s = it % STAGES;
        wg::bar_wait(EMPTY_B(s), ((it / STAGES) & 1) ^ 1);
        unsigned char* st = sRing + s * STAGE_BYTES;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int lrow = 16 * j + 4 * warp + r4;  // row within the tile
          const uint32_t soff = (lrow >> 3) * SBO + (lrow & 7) * 128 + ((c8 ^ (lrow & 7)) << 4);
          const float4 h = split_hi(R.a[j]);
          *reinterpret_cast<float4*>(st + soff) = h;
          *reinterpret_cast<float4*>(st + TILE_BYTES + soff) = sub4(R.a[j], h);
          if (!WSTAT) {
            *reinterpret_cast<float4*>(st + 2 * TILE_BYTES + soff) = R.h[j];
            *reinterpret_cast<float4*>(st + 3 * TILE_BYTES + soff) = R.l[j];
          }
        }
        wg::fence_async();  // generic-proxy stores -> async-proxy (MMA) reads
        wg::bar_arrive(FULL_B(s));
        if constexpr (WSTAT) R = Rn; else load_next(R);
      }
    }
  } else {
    // ------------------------------------------------------------------ consumer warpgroups: 64 rows each
    const int cw = (warp - 4) >> 2, w4 = warp & 3;
    uint32_t it = 0;
    float d[64];
    for (int mt = group; mt < m_tiles; mt += groups) {
      for (int kb = 0; kb < nkb; ++kb, ++it) {
        const int s = it % STAGES;
        wg::bar_wait(FULL_B(s), (it / STAGES) & 1);
        const uint32_t ahi = wg::s32(sRing + s * STAGE_BYTES) + cw * 64 * 128, alo = ahi + TILE_BYTES;
        const uint32_t bhi = WSTAT ? wg::s32(sW + (2 * kb) * TILE_BYTES) : wg::s32(sRing + s * STAGE_BYTES + 2 * TILE_BYTES);
        const uint32_t blo = bhi + TILE_BYTES;
        wg::pin(d);
        wg::fence();
#pragma unroll
        for (int kk = 0; kk < GK / 8; ++kk) {  // one k-step = 8 tf32 = 32 B: advance inside the swizzle atom
          const uint32_t off = kk * 32;
          wg::mma_ss_n128(d, wg::desc_sw128(ahi + off, SBO), wg::desc_sw128(bhi + off, SBO), (kb | kk) != 0);
          wg::mma_ss_n128(d, wg::desc_sw128(alo + off, SBO), wg::desc_sw128(bhi + off, SBO), 1);
          wg::mma_ss_n128(d, wg::desc_sw128(ahi + off, SBO), wg::desc_sw128(blo + off, SBO), 1);
        }
        wg::commit();
        if (kb > 0) {  // the previous k-block's MMAs have retired: its stage goes back to the producer
          wg::wait<1>();
          wg::bar_arrive(EMPTY_B((it - 1) % STAGES));
        }
      }
      wg::wait<0>();
      wg::pin(d);
      wg::bar_arrive(EMPTY_B((it - 1) % STAGES));
      epilogue_regs(g, d, mt * GM + 64 * cw + 16 * w4, n0, lane);
    }
  }
}

}  // namespace co

using namespace co;

extern "C" int co_split_tf32(const float* w, float* hi, float* lo, long n, void* stream) {
  if (!w || !hi || !lo || n < 0) return fail(CO_ERR_BAD_ARG, "co_split_tf32: bad argument%s");
  if (n == 0) return CO_OK;
  split_tf32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(w, hi, lo, n);
  return check_launch("co_split_tf32");
}

extern "C" int co_gemm_tf32x3(const float* A, const float* Whi, const float* Wlo, float* C, const float* bias,
                              const float* residual, const float* scale, const float* shift, int M, int Nout, int K,
                              int lda, int ldc, int ldr, int relu, void* stream) {
  if (!A || !Whi || !Wlo || !C) return fail(CO_ERR_BAD_ARG, "co_gemm_tf32x3: null pointer%s");
  if (M < 0 || Nout <= 0 || K <= 0) return fail(CO_ERR_BAD_ARG, "co_gemm_tf32x3: bad shape%s");
  if ((K % GK) || (Nout % 4) || (lda % 4) || (ldc % 4) || (residual && (ldr % 4)))
    return fail(CO_ERR_UNSUPPORTED, "co_gemm_tf32x3: K %% 32, Nout %% 4 and 16-byte row strides required%s");
  if ((scale == nullptr) != (shift == nullptr)) return fail(CO_ERR_BAD_ARG, "co_gemm_tf32x3: scale and shift go together%s");
  if (((uintptr_t)A | (uintptr_t)Whi | (uintptr_t)Wlo | (uintptr_t)C | (uintptr_t)bias | (uintptr_t)residual |
       (uintptr_t)scale | (uintptr_t)shift) & 15)
    return fail(CO_ERR_BAD_ARG, "co_gemm_tf32x3: pointers must be 16-byte aligned%s");
  if (M == 0) return CO_OK;
  GemmArgs g{A, Whi, Wlo, C, bias, residual, scale, shift, M, Nout, K, lda, ldc, ldr, relu, (Nout + GN - 1) / GN};
  const int m_tiles = (M + GM - 1) / GM;
  if ((long)m_tiles * g.n_tiles > 0x7fffffffL) return fail(CO_ERR_UNSUPPORTED, "co_gemm_tf32x3: too many tiles%s");
  static PerDeviceOnce once;
  bool& configured = once.flag();
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(gemm_tf32x3_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(gemm_tf32x3_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, STAGES * 4 * TILE_BYTES);
    if (e != cudaSuccess) return fail(CO_ERR_CUDA, "co_gemm_tf32x3: smem attribute: %s", cudaGetErrorString(e));
    configured = true;
  }
  // CTAs of one group share an M tile (L2 reuse of A); every CTA keeps its block of W columns
  int groups = device_info().sm_count / g.n_tiles;
  if (groups < 1) groups = 1;
  if (groups > m_tiles) groups = m_tiles;
  if (K == GK * KB128)
    gemm_tf32x3_kernel<true><<<groups * g.n_tiles, GEMM_THREADS, GEMM_SMEM, (cudaStream_t)stream>>>(g, m_tiles, groups);
  else
    gemm_tf32x3_kernel<false><<<groups * g.n_tiles, GEMM_THREADS, STAGES * 4 * TILE_BYTES, (cudaStream_t)stream>>>(g, m_tiles, groups);
  return check_launch("co_gemm_tf32x3");
}
