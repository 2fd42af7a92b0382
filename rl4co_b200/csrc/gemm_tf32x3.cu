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
// ~2^-22 relative), i.e. fp32-class accuracy (~1e-6 relative) at tensor-core rate.  Both kernels below issue the same
// MMAs on the same operand values in the same order (k-steps 0..K/8-1, per k-step hi*hi, lo*hi, hi*lo), so an output
// element has the same bits whichever kernel, CTA or tile computed it.
//
// Persistent CTAs of three warpgroups; a CTA keeps one 128-column block of W and walks over 128-row tiles (the CTAs
// of one group start on the same row tile, so A is read from HBM about once and then from L2).
//
// K == 128 (every projection of the encoder / cache): gemm_k128_kernel.  The CTA's W block (hi + lo, 128 KB) stays in
// shared memory as 128-byte-swizzled K-major tiles (row r at r*128 B, 16-byte chunk c stored at c ^ (r & 7);
// SBO = 1 KB).
//   warpgroup 0  producer (24 registers): one thread issues a TMA tensor load per 32-wide k-block of A (box 32 x 128
//                           fp32, the same 128-byte swizzle; rows past M arrive as zeros) into a 6-stage fp32 ring, on
//                           mbarrier complete_tx: 96 KB of A in flight per SM.
//   warpgroups 1-2 consumers (240 registers): 64 rows x 128 columns each.  Per k-block a thread reads its A fragment
//                           from the fp32 stage (LDS.32, conflict-free: k-step kk reads chunk 2 kk ^ g), splits it into
//                           hi / lo in registers and issues register-A wgmma m64n128k8 against the resident W, one
//                           commit group of three (hi*hi, lo*hi, hi*lo) per k-step.  The only wait, once per k-block
//                           after its first group, retires the previous k-block and releases its stage, so the MMAs of
//                           up to five k-steps are queued while at most five k-steps of A fragments occupy registers.  Two accumulator sets alternate between row tiles: after each k-block of tile
//                           t + 1 a quarter of tile t's fused epilogue is stored from the other set, so the stores of
//                           one tile overlap the MMAs of the next.
// Other K: gemm_tf32x3_kernel.  The producer warpgroup loads A and W with LDG one k-block ahead, splits them and stores
//   [A_hi, A_lo, W_hi, W_lo] into a 3-stage ring of swizzled tiles; the consumers issue shared-operand wgmma and run the
//   epilogue after each tile.
//
// Diagnostic build (-DCO_GEMM_CLOCKS, tools/gemm_phase_clocks.py): gemm_k128_kernel records per-CTA phase clocks;
// without the macro the stamps compile to nothing.
#include <cuda.h>
#include <cudaTypedefs.h>

#include "co_common.cuh"
#include "wgmma.cuh"

namespace co {

constexpr int GM = 128, GN = 128, GK = 32;
constexpr int TILE_BYTES = GM * GK * 4;  // 16 KB per operand tile
constexpr uint32_t SBO = 1024;           // 8 rows x 128 B swizzle atom
constexpr int KB128 = 4;                 // k-blocks of the K == 128 kernel
constexpr int STAGES = 3;
constexpr int RING128 = 6;               // fp32 A stages of the K == 128 kernel
constexpr int GEMM_THREADS = 384;
constexpr int GEMM_SMEM = STAGES * 4 * TILE_BYTES;                            // 192 KB
constexpr int GEMM128_SMEM = 2 * KB128 * TILE_BYTES + RING128 * TILE_BYTES;   // 224 KB

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

// fused epilogue of one consumer warpgroup straight from its accumulator fragment, column groups j0 .. j1 - 1: rows
// m0 + {g, g + 8}, column pairs n0 + 8 j + 2 q (wgmma.cuh)
__device__ __forceinline__ void epilogue_regs(const GemmArgs& g, const float (&d)[64], int m0, int n0, int lane,
                                              int j0 = 0, int j1 = 16) {
  const int q = lane & 3;
#pragma unroll
  for (int j = j0; j < j1; ++j) {
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

// one k-block of a producer thread: 8 x (4 rows x 128 B) of A, W_hi and W_lo
struct KBlock {
  float4 a[8], h[8], l[8];
};

__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_tf32x3_kernel(const GemmArgs g, int m_tiles, int groups) {
  extern __shared__ __align__(1024) unsigned char smem[];
  // a ring of [A_hi, A_lo, W_hi, W_lo]
  constexpr int STAGE_BYTES = 4 * TILE_BYTES;
  unsigned char* sRing = smem;
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
        R.h[j] = R.l[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (mt < m_tiles && n0 + lrow < g.Nout) {
          R.h[j] = __ldg(reinterpret_cast<const float4*>(g.Whi + (size_t)(n0 + lrow) * g.K + kb * GK + c8 * 4));
          R.l[j] = __ldg(reinterpret_cast<const float4*>(g.Wlo + (size_t)(n0 + lrow) * g.K + kb * GK + c8 * 4));
        }
      }
    };
    KBlock R;
    load(group, 0, R);
    uint32_t it = 0;
    for (int mt = group; mt < m_tiles; mt += groups) {
      for (int kb = 0; kb < nkb; ++kb, ++it) {
        auto load_next = [&](auto& dst) { if (kb + 1 < nkb) load(mt, kb + 1, dst); else load(mt + groups, 0, dst); };
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
          *reinterpret_cast<float4*>(st + 2 * TILE_BYTES + soff) = R.h[j];
          *reinterpret_cast<float4*>(st + 3 * TILE_BYTES + soff) = R.l[j];
        }
        wg::fence_async();  // generic-proxy stores -> async-proxy (MMA) reads
        wg::bar_arrive(FULL_B(s));
        load_next(R);
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
        const uint32_t bhi = wg::s32(sRing + s * STAGE_BYTES + 2 * TILE_BYTES);
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

// ---------------------------------------------------------------------------------------------- K == 128 kernel

__device__ __forceinline__ void bar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// TMA: box (x .. x + 31, y .. y + 127) of the 2-D tensor map -> shared memory, complete_tx on `bar`
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int x, int y, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(bar) : "memory");
}

// Phase clocks (diagnostic build only): per CTA, co_gemm_clk[cta][8] =
//   0 row tiles, 1 producer cycles waiting on "empty", 2 load latency (TMA issue -> consumer passes "full"),
//   3 consumer cycles waiting on "full", 4 A fragment reads + split + MMA issue, 5 waiting for MMAs to retire (the
//   once-per-k-block wait<1> and the last tile's wait<0>: every MMA wait of the kernel), 6 epilogue stores,
//   7 consumer cycles from the first "full" wait to the end.
// The producer thread and thread 0 of consumer warpgroup 0 record; the buffer must be set before the first launch.
#ifdef CO_GEMM_CLOCKS
static __constant__ long long* co_gemm_clk;
#define CO_GCLK(...) __VA_ARGS__
#else
#define CO_GCLK(...) ;  // a null statement, so that the build without stamps has the same control flow
#endif

__global__ void __launch_bounds__(GEMM_THREADS, 1)
    gemm_k128_kernel(const GemmArgs g, const __grid_constant__ CUtensorMap amap, int m_tiles, int groups) {
  extern __shared__ __align__(1024) unsigned char smem[];
  unsigned char* sW = smem;                                 // [kb][W_hi, W_lo]
  unsigned char* sRing = smem + 2 * KB128 * TILE_BYTES;     // [stage] fp32 A tile
  __shared__ __align__(8) uint64_t bars[2 * RING128];       // full[s] (1 arrival + 16 KB of tx), empty[s] (256 consumers)
  CO_GCLK(__shared__ long long issue_clk[RING128];)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_tile = blockIdx.x % g.n_tiles, group = blockIdx.x / g.n_tiles;
  const int n0 = n_tile * GN;
  const uint32_t bar0 = wg::s32(bars);
  auto FULL_B = [&](int s) { return bar0 + 8 * s; };
  auto EMPTY_B = [&](int s) { return bar0 + 8 * (RING128 + s); };

  if (tid == 0) {
    for (int s = 0; s < RING128; ++s) { wg::bar_init(FULL_B(s), 1); wg::bar_init(EMPTY_B(s), 256); }
    wg::bar_init_fence();
  }
  {
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
    // ------------------------------------------------------------------ producer: one thread issues the TMA loads
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");
    if (tid == 0) {
      CO_GCLK(long long c_empty = 0;)
      uint32_t it = 0;
      for (int mt = group; mt < m_tiles; mt += groups) {
        for (int kb = 0; kb < KB128; ++kb, ++it) {
          const int s = it % RING128;
          CO_GCLK(const long long c0 = clock64();)
          wg::bar_wait(EMPTY_B(s), ((it / RING128) & 1) ^ 1);
          CO_GCLK(const long long c1 = clock64(); c_empty += c1 - c0; issue_clk[s] = c1;)
          bar_expect_tx(FULL_B(s), TILE_BYTES);
          tma_load_2d(wg::s32(sRing + s * TILE_BYTES), &amap, kb * GK, mt * GM, FULL_B(s));
        }
      }
      CO_GCLK(co_gemm_clk[8 * blockIdx.x + 1] = c_empty;)
    }
  } else {
    // ------------------------------------------------------------------ consumer warpgroups: 64 rows each
    asm volatile("setmaxnreg.inc.sync.aligned.u32 240;");
    const int cw = (warp - 4) >> 2, w4 = warp & 3, gq = lane >> 2;
    // this thread's A fragment (wgmma.cuh) in a swizzled fp32 stage: row 64 cw + 16 w4 + gq (+ 8 = + SBO), word q of
    // chunk (2 kk + i / 2) ^ gq
    const unsigned char* afrag = sRing + (8 * cw + 2 * w4) * SBO + gq * 128 + (lane & 3) * 4;
    const int m_warp = 64 * cw + 16 * w4;
    CO_GCLK(const bool rec = (tid == 128); long long c_lat = 0, c_full = 0, c_issue = 0, c_retire = 0, c_epi = 0, c_start = 0;
            long long c_t = 0; int tiles = 0;)
    uint32_t it = 0;
    float d0[64], d1[64];
    // one row tile into dc; with `prev`, dp holds the finished tile mt - groups, stored a quarter per k-block
    auto tile = [&](float (&dc)[64], float (&dp)[64], int mt, bool prev) {
      CO_GCLK(++tiles;)
#pragma unroll
      for (int kb = 0; kb < KB128; ++kb, ++it) {
        const int s = it % RING128;
        CO_GCLK(c_t = clock64(); if (c_start == 0) c_start = c_t;)
        wg::bar_wait(FULL_B(s), (it / RING128) & 1);
        CO_GCLK(long long c = clock64(); c_full += c - c_t; c_lat += c - issue_clk[s]; c_t = c;)
        const unsigned char* st = afrag + s * TILE_BYTES;
        uint32_t bhi = wg::s32(sW + (2 * kb) * TILE_BYTES);
        asm volatile("" : "+r"(bhi));  // computed per k-block, not held in registers across the tile loop
        const uint32_t blo = bhi + TILE_BYTES;
        // one commit group per k-step; the only wait is after the first group of a k-block, and it retires the whole
        // previous k-block.  Up to five groups are in flight (the previous k-block's four and this one's first), while
        // A fragments are formed one k-step at a time: at most five k-steps of them (40 registers) are held, where
        // forming a whole k-block before its first MMA would hold eight (64) and make the compiler serialize the MMAs.
#pragma unroll
        for (int kk = 0; kk < GK / 8; ++kk) {  // one k-step = 8 tf32 = 32 B: advance inside the swizzle atom
          uint32_t ah[4], al[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float v = *reinterpret_cast<const float*>(st + (i & 1) * SBO + (((2 * kk + (i >> 1)) ^ gq) << 4));
            const float h = wg::rna_tf32(v);
            ah[i] = __float_as_uint(h);
            al[i] = __float_as_uint(v - h);
          }
          const uint32_t off = kk * 32;
          if (kk == 0) wg::pin(dc);
          wg::fence();
          wg::mma_rs_n128(dc, ah, wg::desc_sw128(bhi + off, SBO), (kb | kk) != 0);
          wg::mma_rs_n128(dc, al, wg::desc_sw128(bhi + off, SBO), 1);
          wg::mma_rs_n128(dc, ah, wg::desc_sw128(blo + off, SBO), 1);
          wg::commit();
          if (kk == 0) {
            CO_GCLK(c = clock64(); c_issue += c - c_t; c_t = c;)
            if (kb > 0 || prev) {
              // every group of the previous k-block has retired: its stage goes back to the producer
              wg::wait<1>();
              wg::bar_arrive(EMPTY_B((it - 1) % RING128));
            }
            CO_GCLK(c = clock64(); c_retire += c - c_t; c_t = c;)
          }
        }
        CO_GCLK(c = clock64(); c_issue += c - c_t; c_t = c;)
        if (prev) {
          if (kb == 0) wg::pin(dp);
          epilogue_regs(g, dp, (mt - groups) * GM + m_warp, n0, lane, 4 * kb, 4 * kb + 4);
          CO_GCLK(c = clock64(); c_epi += c - c_t;)
        }
      }
    };
    // the last tile: its stage is never reused, so nothing is released
    auto last = [&](float (&dl)[64], int mt) {
      wg::wait<0>();
      CO_GCLK(const long long c = clock64(); c_retire += c - c_t; c_t = c;)
      wg::pin(dl);
      epilogue_regs(g, dl, mt * GM + m_warp, n0, lane);
    };
    // unrolled by two, so that every path into the loop head has d0's batches in flight (the compiler then keeps the
    // MMAs asynchronous while the epilogue reads the other set)
    int mt = group;
    if (mt < m_tiles) {
      tile(d0, d1, mt, false);
      for (;;) {
        if (mt + groups >= m_tiles) { last(d0, mt); break; }
        mt += groups;
        tile(d1, d0, mt, true);
        if (mt + groups >= m_tiles) { last(d1, mt); break; }
        mt += groups;
        tile(d0, d1, mt, true);
      }
    }
    CO_GCLK(if (rec) {
      const long long c = clock64();
      long long* o = co_gemm_clk + 8 * blockIdx.x;
      o[0] = tiles; o[2] = c_lat; o[3] = c_full; o[4] = c_issue; o[5] = c_retire; o[6] = c_epi + (c - c_t); o[7] = c - c_start;
    })
  }
}

// 2-D tensor map over A[M, K] (row stride lda floats): box 32 x 128, 128-byte swizzle, rows past M read as zeros.
// cuTensorMapEncodeTiled comes through the runtime's driver entry point, so the library links no libcuda.
static int encode_a_map(CUtensorMap* map, const float* A, int M, int K, int lda) {
  static const PFN_cuTensorMapEncodeTiled_v12000 encode = []() -> PFN_cuTensorMapEncodeTiled_v12000 {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &fn, 12000, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  }();
  if (!encode) return fail(CO_ERR_CUDA, "co_gemm_tf32x3: cuTensorMapEncodeTiled is not available%s");
  const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)M};
  const cuuint64_t strides[1] = {(cuuint64_t)lda * sizeof(float)};
  const cuuint32_t box[2] = {GK, GM}, estr[2] = {1, 1};
  const CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(A), dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(CO_ERR_CUDA, "co_gemm_tf32x3: cuTensorMapEncodeTiled failed%s (CUresult %lld)", "", (long long)r);
  return CO_OK;
}

}  // namespace co

using namespace co;

#ifdef CO_GEMM_CLOCKS
// diagnostic build only: where gemm_k128_kernel writes its phase clocks
extern "C" int co_gemm_clocks_set(void* buf) {
  return cudaMemcpyToSymbol(co::co_gemm_clk, &buf, sizeof(buf)) == cudaSuccess ? 0 : 1;
}
#endif

extern "C" int co_split_tf32(const float* w, float* hi, float* lo, long n, void* stream) {
  if (!w || !hi || !lo || n < 0) return fail(CO_ERR_BAD_ARG, "co_split_tf32: bad argument%s");
  if (n == 0) return CO_OK;
  split_tf32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(w, hi, lo, n);
  return check_launch("co_split_tf32");
}

extern "C" int co_gemm_tf32x3(const float* A, const float* Whi, const float* Wlo, float* C, const float* bias,
                              const float* residual, const float* scale, const float* shift, int M, int Nout, int K,
                              int lda, int ldc, int ldr, int relu, void* stream) {
  if (M < 0 || Nout <= 0 || K <= 0) return fail(CO_ERR_BAD_ARG, "co_gemm_tf32x3: bad shape%s");
  if ((K % GK) || (Nout % 4) || (lda % 4) || (ldc % 4) || (residual && (ldr % 4)))
    return fail(CO_ERR_UNSUPPORTED, "co_gemm_tf32x3: K %% 32, Nout %% 4 and 16-byte row strides required%s");
  if ((scale == nullptr) != (shift == nullptr)) return fail(CO_ERR_BAD_ARG, "co_gemm_tf32x3: scale and shift go together%s");
  // no rows: nothing is read or written, and no tensor map is encoded (it would reject a zero dimension); A and C may
  // be null here, as the data pointer of an empty tensor is
  if (M == 0) return CO_OK;
  if (!A || !Whi || !Wlo || !C) return fail(CO_ERR_BAD_ARG, "co_gemm_tf32x3: null pointer%s");
  if (((uintptr_t)A | (uintptr_t)Whi | (uintptr_t)Wlo | (uintptr_t)C | (uintptr_t)bias | (uintptr_t)residual |
       (uintptr_t)scale | (uintptr_t)shift) & 15)
    return fail(CO_ERR_BAD_ARG, "co_gemm_tf32x3: pointers must be 16-byte aligned%s");
  GemmArgs g{A, Whi, Wlo, C, bias, residual, scale, shift, M, Nout, K, lda, ldc, ldr, relu, (Nout + GN - 1) / GN};
  const int m_tiles = (M + GM - 1) / GM;
  if ((long)m_tiles * g.n_tiles > 0x7fffffffL) return fail(CO_ERR_UNSUPPORTED, "co_gemm_tf32x3: too many tiles%s");
  static PerDeviceOnce once;
  bool& configured = once.flag();
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(gemm_k128_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM128_SMEM);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(gemm_tf32x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM);
    if (e != cudaSuccess) return fail(CO_ERR_CUDA, "co_gemm_tf32x3: smem attribute: %s", cudaGetErrorString(e));
    configured = true;
  }
  // CTAs of one group share an M tile (L2 reuse of A); every CTA keeps its block of W columns
  int groups = device_info().sm_count / g.n_tiles;
  if (groups < 1) groups = 1;
  if (groups > m_tiles) groups = m_tiles;
  if (K == GK * KB128) {
    CUtensorMap amap;
    if (int rc = encode_a_map(&amap, A, M, K, lda)) return rc;
    gemm_k128_kernel<<<groups * g.n_tiles, GEMM_THREADS, GEMM128_SMEM, (cudaStream_t)stream>>>(g, amap, m_tiles, groups);
  } else {
    gemm_tf32x3_kernel<<<groups * g.n_tiles, GEMM_THREADS, GEMM_SMEM, (cudaStream_t)stream>>>(g, m_tiles, groups);
  }
  return check_launch("co_gemm_tf32x3");
}
