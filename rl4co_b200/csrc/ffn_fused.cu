// Encoder FFN block fused into one kernel: the [M, 512] hidden activation never leaves the register file.
//
//   out = ((x + relu(x W1^T + b1) W2^T + b2) * scale + shift      x [M,128], W1 [512,128], W2 [128,512]
//   (rl4co/models/nn/graph/attnnet.py:33-53: SkipConnection(MLP) followed by eval-mode BatchNorm folded into scale/shift;
//    rl4co/models/nn/mlp.py:45-60 is the MLP)
//
// Per 128-row tile, 3xTF32 everywhere (hi = cvt.rna.tf32, lo = v - hi; products hi.hi + lo.hi + hi.lo).  Two consumer
// warpgroups own 64 rows each; a producer warpgroup feeds them:
//   x tile  -> hi / lo K-major SWIZZLE_128B operand tiles in SMEM (4 k-blocks, 128 KB), resident for the tile
//   for each of the 4 hidden chunks j (128 units):
//     FF1(j): H = x W1_j^T            48 wgmma m64n128k8 per warpgroup, operands from SMEM, H in 64 accumulator registers
//     H + b1 -> relu -> H_hi in place, H_lo beside it, still in registers
//     FF2(j): Y += H W2_j^T           48 wgmma with the A operand from registers: the accumulator fragment of H is the
//                                     A fragment once W2's k dimension is stored in the k-slot order of wgmma.cuh
//   Y + b2 + x, BN, store.
// W1_j / W2_j k-blocks ([128 x 32] hi + lo = 32 KB) stream from L2 in the order FF1(0) FF2(0) .. FF1(3) FF2(3) through a
// 3-stage ring; one MMA batch stays in flight while the stage before it is released.  Per tile 1 MB of weights.
//
// Weight stream = TMA bulk copies with CLUSTER MULTICAST.  The kernel runs as 2-CTA clusters; the weights are pre-tiled
// once per weight version (co_ffn_tile_weights) into the exact shared-memory image of the operand tiles (K-major,
// SWIZZLE_128B), block after block in issue order, so a block is two contiguous 16 KB pieces (hi, lo).  For every block
// CTA r of the cluster issues ONE `cp.async.bulk ... .multicast::cluster` of piece r that lands in BOTH CTAs' rings and
// signals both CTAs' "full" mbarriers (complete_tx); a ring stage is reused when the consumer warps of BOTH CTAs have
// arrived on its "empty" barrier (remote mbarrier arrive).  Each SM therefore pulls 0.5 MB per tile from L2 instead of
// 1 MB.
#include <stdint.h>

#include "co_common.cuh"
#include "wgmma.cuh"

namespace co {
namespace ffn {

constexpr int BM = 128, HID = 512, NJ = HID / 128, KB = 4;  // k-blocks of 32 per 128-wide reduction
constexpr int TILE_B = 128 * 32 * 4;                         // one [128 x 32] operand tile = 16 KB
constexpr int OFF_W = 2 * KB * TILE_B;                       // after x hi / lo
constexpr int WST = 3;                                       // weight ring stages (hi + lo each): 2 blocks in flight
constexpr int SMEM_B = OFF_W + WST * 2 * TILE_B;             // 229 376 (x 128 KB + 3 x 32 KB)
constexpr int THREADS = 384;   // warps 0-2 x producers, warp 3 weight loader, warps 4-7 / 8-11 consumers (64 rows each)
constexpr int X_PRODUCERS = 96, CONSUMER_WARPS = 8;
constexpr int CLUSTER = 2;                                   // CTAs sharing every weight block
constexpr int WBLOCK_FLOATS = 2 * 128 * 32;                  // one pre-tiled block: hi image, lo image (32 KB)
constexpr int WBLOCKS = 2 * NJ * KB;                         // weight blocks per tile
constexpr uint32_t SBO = 1024;

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the barrier at this CTA-relative address in CTA `rank` of the cluster
__device__ __forceinline__ void bar_arrive_cluster(uint32_t bar, uint32_t rank) {
  asm volatile("{\n\t.reg .b32 ra;\n\tmapa.shared::cluster.u32 ra, %0, %1;\n\t"
               "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}" ::"r"(bar), "r"(rank) : "memory");
}
__device__ __forceinline__ void bar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// TMA bulk copy global -> shared memory of every CTA in the cluster (same CTA-relative destination and mbarrier)
__device__ __forceinline__ void bulk_copy_multicast(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;"
      ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "h"((uint16_t)((1u << CLUSTER) - 1)) : "memory");
}

struct FfnArgs {
  const float *x, *wtiled, *b1, *b2, *scale, *shift;  // wtiled: co_ffn_tile_weights image; scale / shift may be null
  float* out;
  int M, ldx, ldo;
};

// weight block b (0..31) of a tile in issue order FF1(0) FF2(0) FF1(1) ..: {second GEMM?, chunk j, k-block kb}
struct WBlock { int ff2, j, kb; };
__host__ __device__ __forceinline__ WBlock wblock(int b) { return {(b >> 2) & 1, b >> 3, b & 3}; }

__global__ void __cluster_dims__(CLUSTER, 1, 1) __launch_bounds__(THREADS, 1)
    ffn_fused_kernel(const FfnArgs g, int m_tiles) {
  extern __shared__ __align__(1024) unsigned char smem[];
  unsigned char* sX = smem;           // [kb][hi, lo]
  unsigned char* sW = smem + OFF_W;   // [stage][hi, lo]
  __shared__ __align__(8) uint64_t bars[2 + 2 * WST];
  const uint32_t b0 = wg::s32(bars);
  auto XFULL = [&]() { return b0; };                          // producers: x tile in SMEM                    (96)
  auto XEMPTY = [&]() { return b0 + 8; };                     // FF1(3) retired: x tile reusable              (256)
  auto WFULL = [&](int s) { return b0 + 8 * (2 + s); };       // weight block landed: 1 arrive + 32 KB of complete_tx
  auto WEMPTY = [&](int s) { return b0 + 8 * (2 + WST + s); };  // its MMAs retired: consumer warps of BOTH CTAs (16)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    wg::bar_init(XFULL(), X_PRODUCERS);
    wg::bar_init(XEMPTY(), 32 * CONSUMER_WARPS);
    for (int s = 0; s < WST; ++s) { wg::bar_init(WFULL(s), 1); wg::bar_init(WEMPTY(s), CLUSTER * CONSUMER_WARPS); }
    wg::bar_init_fence();
  }
  __syncthreads();
  cluster_sync();  // the peer's barriers are initialised before anything can arrive on them
  // both CTAs of a cluster run the same number of tiles (they consume the same weight-block sequence); a tile index
  // beyond m_tiles is a dummy: every row fails `row < M`, so nothing is loaded or stored for it
  const int ntiles = (m_tiles + (int)gridDim.x - 1) / (int)gridDim.x;

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
    if (warp < 3) {
      // ---------------------------------------------------------------- producers: x tile (fp32 -> tf32 hi / lo split)
      // a warp instruction fetches 4 complete 128-byte rows of a k-block; a quarter-warp writes one swizzled row
      const int r4 = lane >> 3, c8 = lane & 7;
      for (int t = 0; t < ntiles; ++t) {
        const int m0 = (blockIdx.x + t * gridDim.x) * BM;
        wg::bar_wait(XEMPTY(), (t & 1) ^ 1);
        for (int rq0 = warp; rq0 < 32; rq0 += 6) {
#pragma unroll
          for (int kb = 0; kb < KB; ++kb) {
            float4 a[2];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const int lrow = 4 * (rq0 + 3 * u) + r4, row = m0 + lrow;
              a[u] = make_float4(0.f, 0.f, 0.f, 0.f);
              if (lrow < BM && row < g.M) a[u] = __ldg(reinterpret_cast<const float4*>(g.x + (size_t)row * g.ldx + kb * 32 + c8 * 4));
            }
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const int lrow = 4 * (rq0 + 3 * u) + r4;
              if (lrow < BM) {
                const uint32_t soff = (lrow >> 3) * SBO + (lrow & 7) * 128 + ((c8 ^ (lrow & 7)) << 4);
                const float4 h = make_float4(wg::rna_tf32(a[u].x), wg::rna_tf32(a[u].y), wg::rna_tf32(a[u].z), wg::rna_tf32(a[u].w));
                *reinterpret_cast<float4*>(sX + (2 * kb) * TILE_B + soff) = h;
                *reinterpret_cast<float4*>(sX + (2 * kb + 1) * TILE_B + soff) =
                    make_float4(a[u].x - h.x, a[u].y - h.y, a[u].z - h.z, a[u].w - h.w);
              }
            }
          }
        }
        wg::fence_async();
        wg::bar_arrive(XFULL());
      }
    } else if (lane == 0) {
      // ---------------------------------------------------------------- weight loader: one thread, TMA bulk copies
      const uint32_t rank = cluster_ctarank();
      uint32_t wb = 0;
      for (int t = 0; t < ntiles; ++t) {
        for (int b = 0; b < WBLOCKS; ++b, ++wb) {
          const int st = wb % WST;
          wg::bar_wait(WEMPTY(st), ((wb / WST) & 1) ^ 1);   // the stage is free in both CTAs
          bar_expect_tx(WFULL(st), 2 * TILE_B);             // own piece + the peer's piece will land here
          // piece `rank` (0 = hi image, 1 = lo image) of block b -> the same ring slot of every CTA in the cluster
          bulk_copy_multicast(wg::s32(sW + (2 * st + rank) * TILE_B), g.wtiled + (size_t)b * WBLOCK_FLOATS + rank * (TILE_B / 4),
                              TILE_B, WFULL(st));
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumer warpgroups: rows [64 cw, 64 cw + 64)
    asm volatile("setmaxnreg.inc.sync.aligned.u32 216;");
    const int cw = (warp - 4) >> 2, w4 = warp & 3, gq = lane >> 2, q = lane & 3;
    const uint32_t xbase = wg::s32(sX) + cw * 64 * 128;
    uint32_t wb = 0;   // weight blocks consumed (over all tiles)
    int held = -1;     // ring stage whose MMA batch is still in flight
    auto release = [&](int st) {  // this warp's MMAs on stage st have retired: tell the loaders of both CTAs
      __syncwarp();
      if (lane == 0)
        for (uint32_t r = 0; r < CLUSTER; ++r) bar_arrive_cluster(WEMPTY(st), r);
    };
    auto committed = [&](int st) {  // a batch on stage st was just committed: the one before it has retired
      wg::commit();
      if (held >= 0) { wg::wait<1>(); release(held); }
      held = st;
    };
    auto drain = [&]() {
      wg::wait<0>();
      if (held >= 0) release(held);
      held = -1;
    };
    float h[64], y[64];
    uint32_t hlo[2][4][4];
    for (int t = 0; t < ntiles; ++t) {
      const int m0 = (blockIdx.x + t * gridDim.x) * BM + 64 * cw + 16 * w4 + gq;  // this thread's rows: m0, m0 + 8
      wg::bar_wait(XFULL(), t & 1);
      for (int j = 0; j < NJ; ++j) {
        // FF1(j): h = x W1_j^T
#pragma unroll
        for (int kb = 0; kb < KB; ++kb, ++wb) {
          const int st = wb % WST;
          wg::bar_wait(WFULL(st), (wb / WST) & 1);
          const uint32_t ahi = xbase + (2 * kb) * TILE_B, alo = ahi + TILE_B;
          const uint32_t bhi = wg::s32(sW + (2 * st) * TILE_B), blo = bhi + TILE_B;
          wg::pin(h);
          wg::fence();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const uint32_t off = kk * 32;
            wg::mma_ss_n128(h, wg::desc_sw128(ahi + off, SBO), wg::desc_sw128(bhi + off, SBO), (kb | kk) != 0);
            wg::mma_ss_n128(h, wg::desc_sw128(alo + off, SBO), wg::desc_sw128(bhi + off, SBO), 1);
            wg::mma_ss_n128(h, wg::desc_sw128(ahi + off, SBO), wg::desc_sw128(blo + off, SBO), 1);
          }
          committed(st);
        }
        drain();
        wg::pin(h);
        if (j == NJ - 1) wg::bar_arrive(XEMPTY());  // the last MMAs that read the x tile have retired
        // bias + ReLU, H_hi in place; h[4 jj + i]: row m0 + 8 (i / 2), hidden unit 128 j + 8 jj + 2 q + (i % 2)
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          const float2 bb = __ldg(reinterpret_cast<const float2*>(g.b1 + j * 128 + 8 * jj + 2 * q));
          h[4 * jj] = fmaxf(h[4 * jj] + bb.x, 0.f);
          h[4 * jj + 1] = fmaxf(h[4 * jj + 1] + bb.y, 0.f);
          h[4 * jj + 2] = fmaxf(h[4 * jj + 2] + bb.x, 0.f);
          h[4 * jj + 3] = fmaxf(h[4 * jj + 3] + bb.y, 0.f);
        }
        // FF2(j): y += h W2_j^T, A from registers (k-step jj = accumulator columns 8 jj .. 8 jj + 7)
#pragma unroll
        for (int kb = 0; kb < KB; ++kb, ++wb) {
          const int st = wb % WST;
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const int jj = 4 * kb + kk;
#pragma unroll
            for (int i = 0; i < 4; ++i) {  // A fragment order: (m0, slot q) (m0 + 8, slot q) (m0, q + 4) (m0 + 8, q + 4)
              float& v = h[4 * jj + ((i & 1) << 1) + (i >> 1)];
              const float hi = wg::rna_tf32(v);
              hlo[kb & 1][kk][i] = __float_as_uint(v - hi);
              v = hi;
            }
          }
          wg::bar_wait(WFULL(st), (wb / WST) & 1);
          const uint32_t bhi = wg::s32(sW + (2 * st) * TILE_B), blo = bhi + TILE_B;
          wg::pin(y);
          wg::fence();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const int jj = 4 * kb + kk;
            const uint32_t off = kk * 32;
            const uint32_t hhi[4] = {__float_as_uint(h[4 * jj]), __float_as_uint(h[4 * jj + 2]), __float_as_uint(h[4 * jj + 1]),
                                     __float_as_uint(h[4 * jj + 3])};
            wg::mma_rs_n128(y, hhi, wg::desc_sw128(bhi + off, SBO), (j | kb | kk) != 0);
            wg::mma_rs_n128(y, hlo[kb & 1][kk], wg::desc_sw128(bhi + off, SBO), 1);
            wg::mma_rs_n128(y, hhi, wg::desc_sw128(blo + off, SBO), 1);
          }
          committed(st);  // leaves this batch in flight; the one that read the other half of hlo has retired
        }
        drain();  // FF1(j + 1) overwrites h, the epilogue reads y
      }
      wg::pin(y);
      // final epilogue: Y + b2 + x, BN, store (a quad writes 32 contiguous bytes of a row)
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        const int n = 8 * jj + 2 * q;
        const float2 bb = __ldg(reinterpret_cast<const float2*>(g.b2 + n));
        float2 sc = make_float2(1.f, 1.f), sh = make_float2(0.f, 0.f);
        if (g.scale) { sc = __ldg(reinterpret_cast<const float2*>(g.scale + n)); sh = __ldg(reinterpret_cast<const float2*>(g.shift + n)); }
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int row = m0 + 8 * half;
          if (row < g.M) {
            const float2 xv = __ldg(reinterpret_cast<const float2*>(g.x + (size_t)row * g.ldx + n));
            float2 o = make_float2(y[4 * jj + 2 * half] + xv.x + bb.x, y[4 * jj + 2 * half + 1] + xv.y + bb.y);
            if (g.scale) { o.x = fmaf(o.x, sc.x, sh.x); o.y = fmaf(o.y, sc.y, sh.y); }
            *reinterpret_cast<float2*>(g.out + (size_t)row * g.ldo + n) = o;
          }
        }
      }
    }
  }
  __syncthreads();
  cluster_sync();  // no CTA leaves while its peer may still multicast into its shared memory / arrive on its barriers
}

}  // namespace ffn
}  // namespace co

using namespace co;

namespace co {
namespace ffn {
// Pre-tile W1 [512,128] / W2 [128,512] (hi and lo parts) into the shared-memory image the kernel streams: 32 blocks in
// issue order, each = hi image then lo image of a [128 x 32] K-major SWIZZLE_128B operand tile (16 KB each).
__global__ void __launch_bounds__(256) tile_weights_kernel(const float* __restrict__ w1hi, const float* __restrict__ w1lo,
                                                            const float* __restrict__ w2hi, const float* __restrict__ w2lo,
                                                            float* __restrict__ out) {
  const int b = blockIdx.x;  // block 0..WBLOCKS-1
  const WBlock w = wblock(b);
  for (int idx = threadIdx.x; idx < 128 * 32; idx += blockDim.x) {
    const int n = idx >> 5, c = idx & 31;
    // FF2 takes its A operand from the accumulator registers of FF1: k-slot c of W2 holds hidden unit kperm8 (wgmma.cuh)
    const int k2 = (c & ~7) + wg::kperm8(c & 7);
    const size_t src = w.ff2 ? (size_t)n * HID + w.j * 128 + w.kb * 32 + k2         // W2[n][j*128 + kb*32 + k2]
                             : ((size_t)w.j * 128 + n) * 128 + w.kb * 32 + c;       // W1[j*128 + n][kb*32 + c]
    const uint32_t off = ((n >> 3) * SBO + (n & 7) * 128 + ((((c >> 2) ^ (n & 7))) << 4) + (c & 3) * 4) >> 2;
    out[(size_t)b * WBLOCK_FLOATS + off] = w.ff2 ? w2hi[src] : w1hi[src];
    out[(size_t)b * WBLOCK_FLOATS + TILE_B / 4 + off] = w.ff2 ? w2lo[src] : w1lo[src];
  }
}
}  // namespace ffn
}  // namespace co

extern "C" long co_ffn_tiled_weight_floats(void) { return (long)co::ffn::WBLOCKS * co::ffn::WBLOCK_FLOATS; }

extern "C" int co_ffn_tile_weights(const float* w1hi, const float* w1lo, const float* w2hi, const float* w2lo, float* wtiled,
                                   void* stream) {
  if (!w1hi || !w1lo || !w2hi || !w2lo || !wtiled) return fail(CO_ERR_BAD_ARG, "co_ffn_tile_weights: null pointer%s");
  if ((uintptr_t)wtiled & 127) return fail(CO_ERR_BAD_ARG, "co_ffn_tile_weights: output must be 128-byte aligned%s");
  co::ffn::tile_weights_kernel<<<co::ffn::WBLOCKS, 256, 0, (cudaStream_t)stream>>>(w1hi, w1lo, w2hi, w2lo, wtiled);
  return check_launch("co_ffn_tile_weights");
}

extern "C" int co_ffn_fused(const float* x, const float* wtiled, const float* b1, const float* b2, const float* scale,
                            const float* shift, float* out, int M, int ldx, int ldo, void* stream) {
  if (!x || !wtiled || !b1 || !b2 || !out) return fail(CO_ERR_BAD_ARG, "co_ffn_fused: null pointer%s");
  if ((uintptr_t)wtiled & 127) return fail(CO_ERR_BAD_ARG, "co_ffn_fused: wtiled must be 128-byte aligned%s");
  if (((uintptr_t)x | (uintptr_t)out | (uintptr_t)b1 | (uintptr_t)b2 | (uintptr_t)scale | (uintptr_t)shift) & 15)
    return fail(CO_ERR_BAD_ARG, "co_ffn_fused: pointers must be 16-byte aligned%s");
  if ((scale == nullptr) != (shift == nullptr)) return fail(CO_ERR_BAD_ARG, "co_ffn_fused: scale and shift go together%s");
  if (M < 0 || ldx < 128 || ldo < 128 || (ldx & 3) || (ldo & 3)) return fail(CO_ERR_BAD_ARG, "co_ffn_fused: bad shape%s");
  if (M == 0) return CO_OK;
  static PerDeviceOnce once;
  bool& configured = once.flag();
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(ffn::ffn_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ffn::SMEM_B);
    if (e != cudaSuccess) return fail(CO_ERR_CUDA, "co_ffn_fused: smem attribute: %s", cudaGetErrorString(e));
    configured = true;
  }
  const int m_tiles = (M + ffn::BM - 1) / ffn::BM;
  int grid = device_info().sm_count & ~(ffn::CLUSTER - 1);  // whole clusters
  const int need = (m_tiles + ffn::CLUSTER - 1) & ~(ffn::CLUSTER - 1);
  if (grid > need) grid = need;
  ffn::FfnArgs g{x, wtiled, b1, b2, scale, shift, out, M, ldx, ldo};
  ffn::ffn_fused_kernel<<<grid, ffn::THREADS, ffn::SMEM_B, (cudaStream_t)stream>>>(g, m_tiles);
  return check_launch("co_ffn_fused");
}
