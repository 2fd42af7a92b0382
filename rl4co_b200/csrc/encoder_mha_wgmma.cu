// Encoder-attention kernel for 64 < N <= 128 (CO_MHA_VARIANT=wgmma): scores AND P.V on the Hopper tensor core, the
// probabilities never leave the register file.
//
// Encoder self-attention core (8 heads x 16, fp32 in / out), contract of co_encoder_mha (encoder_mha.cu).  A CTA of two
// warpgroups walks over (instance, head) pairs; warpgroup c owns query rows [64 c, 64 c + 64) of the head:
//   S_h = Q_h K_h^T                       6 wgmma m64n128k8 (3xTF32: hi.hi + lo.hi + hi.lo), operands from SMEM
//   p_ij = 2^((S_ij - m_i) * QS)          in the accumulator registers (a score row lives in one quad: two shuffles per
//                                         reduction); P_hi = top 19 bits in place, P_lo = p - P_hi beside it
//   O_h = P_hi [V_hi | V_lo] + P_lo V_hi  wgmma with the A operand from registers: the accumulator fragment of S is the
//                                         A fragment of P once the keys of V^T are stored in the k-slot order of
//                                         wgmma.cuh (kslot8), so no shuffle or shared-memory round trip is needed
// SMEM (48 KB): Q_hi Q_lo K_hi K_lo as [128 x 16] K-major tiles of 8 x 16 B core matrices, V^T hi / lo as [16 x 128].
// The slices of the next head are loaded into registers while the current head is computed (one CTA per SM: the score
// tile alone takes 64 registers per thread).
#include "co_common.cuh"
#include "wgmma.cuh"

namespace co {
namespace mhawg {

constexpr int THREADS = 256;
constexpr int QK_TILE = 128 * 16 * 4;   // [128 rows x 16 floats]
constexpr int VT_GRP = 4096;            // 8 d-rows x 128 keys x 4 B
constexpr int OFF_VT = 4 * QK_TILE;     // after Qhi, Qlo, Khi, Klo
constexpr int SMEM_B = OFF_VT + 4 * VT_GRP;  // V^T: hi d0-7, hi d8-15, lo d0-7, lo d8-15

__device__ __forceinline__ float trunc_tf32(float v) { return __uint_as_float(__float_as_uint(v) & 0xFFFFE000u); }
__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(FULL, v, 1));
  return fmaxf(v, __shfl_xor_sync(FULL, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(FULL, v, 1);
  return v + __shfl_xor_sync(FULL, v, 2);
}

struct HeadRegs {  // one head's Q / K / V slices for this thread: 2 row groups x one 16-B chunk
  float4 q[2], k[2], v[2];
};

__global__ void __launch_bounds__(THREADS, 1) encoder_mha_wgmma_kernel(const float* __restrict__ qkv, float* __restrict__ out,
                                                                        int B, int N) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const uint32_t sbase = wg::s32(smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int r8 = lane & 7, c4 = lane >> 3;
  const int ninst = (B - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;  // instances of this CTA
  const int total = ninst * H;

  auto load = [&](int hc, HeadRegs& R) {
    const int b = blockIdx.x + (hc >> 3) * gridDim.x, h = hc & 7;
    const float* base = qkv + (size_t)b * N * 3 * E + h * D;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = 8 * (warp + 8 * i) + r8;
      R.q[i] = R.k[i] = R.v[i] = make_float4(0.f, 0.f, 0.f, 0.f);  // rows >= N: zero scores, zero V^T columns
      if (row < N) {
        const float4* src = reinterpret_cast<const float4*>(base + (size_t)row * 3 * E) + c4;
        R.q[i] = __ldg(src);
        R.k[i] = __ldg(src + E / 4);
        R.v[i] = __ldg(src + 2 * E / 4);
      }
    }
  };
  auto store = [&](const HeadRegs& R) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const uint32_t soff = (warp + 8 * i) * 512 + c4 * 128 + r8 * 16;
      const float4 q = R.q[i], k = R.k[i];
      const float4 qh = make_float4(wg::rna_tf32(q.x), wg::rna_tf32(q.y), wg::rna_tf32(q.z), wg::rna_tf32(q.w));
      const float4 kh = make_float4(wg::rna_tf32(k.x), wg::rna_tf32(k.y), wg::rna_tf32(k.z), wg::rna_tf32(k.w));
      *reinterpret_cast<float4*>(smem + soff) = qh;
      *reinterpret_cast<float4*>(smem + QK_TILE + soff) = make_float4(q.x - qh.x, q.y - qh.y, q.z - qh.z, q.w - qh.w);
      *reinterpret_cast<float4*>(smem + 2 * QK_TILE + soff) = kh;
      *reinterpret_cast<float4*>(smem + 3 * QK_TILE + soff) = make_float4(k.x - kh.x, k.y - kh.y, k.z - kh.z, k.w - kh.w);
      // V_h^T: key j = 8 (warp + 8 i) + r8 sits in k-slot kslot8(r8) of its k-step
      const int pos = 8 * (warp + 8 * i) + wg::kslot8(r8);
      const float v[4] = {R.v[i].x, R.v[i].y, R.v[i].z, R.v[i].w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int d = 4 * c4 + e;
        const uint32_t off = OFF_VT + (d >> 3) * VT_GRP + (pos >> 2) * 128 + (d & 7) * 16 + (pos & 3) * 4;
        const float hi = wg::rna_tf32(v[e]);
        *reinterpret_cast<float*>(smem + off) = hi;
        *reinterpret_cast<float*>(smem + 2 * VT_GRP + off) = v[e] - hi;
      }
    }
  };

  const int cw = warp >> 2, w4 = warp & 3, g = lane >> 2, q = lane & 3;
  const int row0 = 64 * cw + 16 * w4 + g;  // this thread's query rows: row0, row0 + 8
  const int nk8 = (N + 7) >> 3;            // 8-key k-steps of P.V
  constexpr float QS = 0.25f * 1.4426950408889634f;  // 1/sqrt(16) * log2(e)
  const uint32_t qhi = sbase + cw * 8 * 512, qlo = qhi + QK_TILE, khi = sbase + 2 * QK_TILE, klo = khi + QK_TILE;
  const uint32_t vt = sbase + OFF_VT;

  HeadRegs R;
  if (total > 0) load(0, R);
  for (int hc = 0; hc < total; ++hc) {
    __syncthreads();  // the previous head's MMAs have read the operand tiles
    store(R);
    wg::fence_async();
    __syncthreads();
    if (hc + 1 < total) load(hc + 1, R);  // in flight while this head is computed

    float s[64];
    wg::fence();
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {  // 8 of the 16 head channels per k-step = two core matrices
      const uint32_t off = kk * 256;
      wg::mma_ss_n128(s, wg::desc_plain(qhi + off, 512, 128), wg::desc_plain(khi + off, 512, 128), kk);
      wg::mma_ss_n128(s, wg::desc_plain(qlo + off, 512, 128), wg::desc_plain(khi + off, 512, 128), 1);
      wg::mma_ss_n128(s, wg::desc_plain(qhi + off, 512, 128), wg::desc_plain(klo + off, 512, 128), 1);
    }
    wg::commit();
    wg::wait<0>();
    wg::pin(s);

    // softmax numerators over the N real keys; s[4 j + i]: row0 + 8 (i / 2), key 8 j + 2 q + (i % 2)
    float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e)
        if (8 * j + 2 * q + e < N) { m0 = fmaxf(m0, s[4 * j + e]); m1 = fmaxf(m1, s[4 * j + 2 + e]); }
    m0 = quad_max(m0) * QS;
    m1 = quad_max(m1) * QS;
    float l0 = 0.f, l1 = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const bool ok = 8 * j + 2 * q + e < N;  // keys >= N: p = 0 (their V^T columns are zero as well)
        const float p0 = ok ? ex2f(fmaf(s[4 * j + e], QS, -m0)) : 0.f;
        const float p1 = ok ? ex2f(fmaf(s[4 * j + 2 + e], QS, -m1)) : 0.f;
        l0 += p0; l1 += p1;
        s[4 * j + e] = p0; s[4 * j + 2 + e] = p1;
      }
    l0 = quad_sum(l0);
    l1 = quad_sum(l1);

    // O = P_hi [V_hi | V_lo] (columns 0..15 | 16..31 of o) + P_lo V_hi (o2), four k-steps per MMA batch
    float o[16], o2[8];
    uint32_t plo[4][4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if (4 * c < nk8) {
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const int j = 4 * c + t;
#pragma unroll
          for (int i = 0; i < 4; ++i) {  // A fragment order: (row0, slot q) (row0 + 8, slot q) (row0, q + 4) (row0 + 8, q + 4)
            float& p = s[4 * j + ((i & 1) << 1) + (i >> 1)];
            const float hi = trunc_tf32(p);
            plo[t][i] = __float_as_uint(p - hi);
            p = hi;
          }
        }
        wg::fence();
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const int j = 4 * c + t;
          if (j < nk8) {
            const uint64_t bd = wg::desc_plain(vt + j * 256, VT_GRP, 128);
            const uint32_t phi[4] = {__float_as_uint(s[4 * j]), __float_as_uint(s[4 * j + 2]), __float_as_uint(s[4 * j + 1]),
                                     __float_as_uint(s[4 * j + 3])};
            wg::mma_rs_n32(o, phi, bd, j != 0);
            wg::mma_rs_n16(o2, plo[t], bd, j != 0);
          }
        }
        wg::commit();
        wg::wait<0>();  // before the P_lo registers are rewritten
      }
    }
    wg::pin(o);
    wg::pin(o2);

    const int b = blockIdx.x + (hc >> 3) * gridDim.x, h = hc & 7;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int row = row0 + 8 * half;
      if (row < N) {
        const float inv = 1.0f / (half ? l1 : l0);
        float* dst = out + ((size_t)b * N + row) * E + h * D + 2 * q;
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          const int i = 4 * jj + 2 * half;
          *reinterpret_cast<float2*>(dst + 8 * jj) =
              make_float2((o[i] + o2[i] + o[8 + i]) * inv, (o[i + 1] + o2[i + 1] + o[8 + i + 1]) * inv);
        }
      }
    }
  }
}

}  // namespace mhawg

int launch_encoder_mha_wgmma(const float* qkv, float* out, int B, int N, cudaStream_t stream) {
  static PerDeviceOnce once;
  bool& configured = once.flag();
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(mhawg::encoder_mha_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, mhawg::SMEM_B);
    if (e != cudaSuccess) return fail(CO_ERR_CUDA, "co_encoder_mha: smem attribute: %s", cudaGetErrorString(e));
    configured = true;
  }
  int ctas = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, mhawg::encoder_mha_wgmma_kernel, mhawg::THREADS, mhawg::SMEM_B);
  int grid = device_info().sm_count * (ctas < 1 ? 1 : ctas);
  if (grid > B) grid = B;
  mhawg::encoder_mha_wgmma_kernel<<<grid, mhawg::THREADS, mhawg::SMEM_B, stream>>>(qkv, out, B, N);
  return check_launch("co_encoder_mha(wgmma)");
}

}  // namespace co
