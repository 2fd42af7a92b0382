// Encoder self-attention core for small graphs (N <= 128 nodes, 8 heads x 16): the
// F.scaled_dot_product_attention call of rl4co's MultiHeadAttention
// (rl4co/models/nn/attention.py:110-134) on the packed Wqkv output, fp32.
//
//   qkv [B*N, 384] row-major (q | k | v, each "(h d)" = 8 x 16)  ->  out [B*N, 128] "(h d)"
//
// One CTA per instance, warp h = head h.  K and V of the instance (all heads) are staged once in
// shared memory; lane l owns query rows l, l+32, .. (ROWS per lane) with q and the output
// accumulators in registers.  Keys are consumed four at a time with an online (flash-style)
// softmax: scores via float2 FMA pairs, one rescale per block, ex2.approx, value accumulation via
// float2 FMA pairs.  No N x N matrix ever exists in memory: HBM traffic = read qkv once + write out once
// (N*(384+128)*4 B per instance).
#include <stdlib.h>
#include <string.h>

#include "co_common.cuh"

namespace co {

__device__ __forceinline__ float ex2_(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// WPH warps per head: warp w -> head w % 8, row group w / 8; lane l owns query rows
// 32 * (rowgroup * ROWS + r) + l.  <ROWS=2, WPH=2> (512 threads, <= 128 registers) doubles the resident
// warps for N > 64 compared with <4, 1>: the kernel is latency-bound, not FMA-bound.
template <int ROWS, int WPH>
__global__ void __launch_bounds__(256 * WPH, (ROWS * WPH == 4) ? 1 : 2) encoder_mha_kernel(const float* __restrict__ qkv,
                                                                                           float* __restrict__ out, int B, int N) {
  extern __shared__ __align__(16) float sm[];
  float* Ks = sm;             // [N][128]
  float* Vs = sm + N * E;     // [N][128]
  const int tid = threadIdx.x, lane = tid & 31, h = (tid >> 5) & 7, rowbase = 32 * ROWS * (tid >> 8);
  constexpr float QSCALE = 0.25f * 1.4426950408889634f;  // 1/sqrt(16) * log2(e): scores in log2 units

  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    const float* base = qkv + (size_t)b * N * 3 * E;
    __syncthreads();  // previous instance done with Ks / Vs
    for (int idx = tid; idx < N * 32; idx += 256 * WPH) {
      const int n = idx >> 5, c = idx & 31;
      reinterpret_cast<float4*>(Ks + n * E)[c] = __ldg(reinterpret_cast<const float4*>(base + (size_t)n * 3 * E + E) + c);
      reinterpret_cast<float4*>(Vs + n * E)[c] = __ldg(reinterpret_cast<const float4*>(base + (size_t)n * 3 * E + 2 * E) + c);
    }
    float2 q[ROWS][8], o[ROWS][8];
    float m[ROWS], l[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      const int row = rowbase + lane + 32 * r;
      m[r] = -INFINITY; l[r] = 0.f;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row < N) v = __ldg(reinterpret_cast<const float4*>(base + (size_t)row * 3 * E + h * D) + c);
        q[r][2 * c] = make_float2(v.x * QSCALE, v.y * QSCALE);
        q[r][2 * c + 1] = make_float2(v.z * QSCALE, v.w * QSCALE);
        o[r][2 * c] = make_float2(0.f, 0.f); o[r][2 * c + 1] = make_float2(0.f, 0.f);
      }
    }
    __syncthreads();
    for (int j0 = 0; j0 < N; j0 += 4) {
      float s[ROWS][4];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = min(j0 + jj, N - 1);
        const float4* kp = reinterpret_cast<const float4*>(Ks + j * E + h * D);  // warp-uniform: broadcast
        const float4 k0 = kp[0], k1 = kp[1], k2 = kp[2], k3 = kp[3];
#pragma unroll
        for (int r = 0; r < ROWS; ++r) {
          float2 a = fmul2(q[r][0], make_float2(k0.x, k0.y));
          a = ffma2(q[r][1], make_float2(k0.z, k0.w), a);
          a = ffma2(q[r][2], make_float2(k1.x, k1.y), a);
          a = ffma2(q[r][3], make_float2(k1.z, k1.w), a);
          float2 c = fmul2(q[r][4], make_float2(k2.x, k2.y));
          c = ffma2(q[r][5], make_float2(k2.z, k2.w), c);
          c = ffma2(q[r][6], make_float2(k3.x, k3.y), c);
          c = ffma2(q[r][7], make_float2(k3.z, k3.w), c);
          s[r][jj] = (j0 + jj < N) ? (a.x + a.y) + (c.x + c.y) : -INFINITY;
        }
      }
      float p[ROWS][4];
#pragma unroll
      for (int r = 0; r < ROWS; ++r) {
        const float mn = fmaxf(fmaxf(m[r], fmaxf(s[r][0], s[r][1])), fmaxf(s[r][2], s[r][3]));
        const float corr = ex2_(m[r] - mn);  // 0 on the first block (m = -inf)
        m[r] = mn;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) p[r][jj] = ex2_(s[r][jj] - mn);
        l[r] = fmaf(l[r], corr, (p[r][0] + p[r][1]) + (p[r][2] + p[r][3]));
        const float2 c2 = make_float2(corr, corr);
#pragma unroll
        for (int c = 0; c < 8; ++c) o[r][c] = fmul2(o[r][c], c2);
      }
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = min(j0 + jj, N - 1);
        const float4* vp = reinterpret_cast<const float4*>(Vs + j * E + h * D);
        const float4 v0 = vp[0], v1 = vp[1], v2 = vp[2], v3 = vp[3];
#pragma unroll
        for (int r = 0; r < ROWS; ++r) {
          const float2 pp = make_float2(p[r][jj], p[r][jj]);
          o[r][0] = ffma2(pp, make_float2(v0.x, v0.y), o[r][0]);
          o[r][1] = ffma2(pp, make_float2(v0.z, v0.w), o[r][1]);
          o[r][2] = ffma2(pp, make_float2(v1.x, v1.y), o[r][2]);
          o[r][3] = ffma2(pp, make_float2(v1.z, v1.w), o[r][3]);
          o[r][4] = ffma2(pp, make_float2(v2.x, v2.y), o[r][4]);
          o[r][5] = ffma2(pp, make_float2(v2.z, v2.w), o[r][5]);
          o[r][6] = ffma2(pp, make_float2(v3.x, v3.y), o[r][6]);
          o[r][7] = ffma2(pp, make_float2(v3.z, v3.w), o[r][7]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      const int row = rowbase + lane + 32 * r;
      if (row < N) {
        const float inv = 1.0f / l[r];
        float4* dst = reinterpret_cast<float4*>(out + ((size_t)b * N + row) * E + h * D);
#pragma unroll
        for (int c = 0; c < 4; ++c)
          dst[c] = make_float4(o[r][2 * c].x * inv, o[r][2 * c].y * inv, o[r][2 * c + 1].x * inv, o[r][2 * c + 1].y * inv);
      }
    }
  }
}

template <int ROWS, int WPH>
static int launch_mha(const float* qkv, float* out, int B, int N, cudaStream_t st) {
  auto kern = encoder_mha_kernel<ROWS, WPH>;
  const size_t smem = (size_t)2 * N * E * sizeof(float);
  static PerDeviceOnce once;
  int ctas = 1;
  bool& configured = once.flag();
  if (!configured) {  // opt in to the largest footprint (N = 128) once per device
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 128 * E * (int)sizeof(float));
    if (e != cudaSuccess) return fail(CO_ERR_CUDA, "co_encoder_mha: smem attribute: %s", cudaGetErrorString(e));
    configured = true;
  }
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, kern, 256 * WPH, smem);
  int grid = device_info().sm_count * (ctas < 1 ? 1 : ctas);
  if (grid > B) grid = B;
  kern<<<grid, 256 * WPH, smem, st>>>(qkv, out, B, N);
  return check_launch("co_encoder_mha");
}

int launch_encoder_mha_wgmma(const float* qkv, float* out, int B, int N, cudaStream_t stream);  // encoder_mha_wgmma.cu

}  // namespace co

using namespace co;

extern "C" int co_encoder_mha(const float* qkv, float* out, int B, int N, void* stream) {
  if (!qkv || !out) return fail(CO_ERR_BAD_ARG, "co_encoder_mha: null pointer%s");
  if (B < 0 || N < 1) return fail(CO_ERR_BAD_ARG, "co_encoder_mha: bad shape%s");
  if (N > 128) return fail(CO_ERR_UNSUPPORTED, "co_encoder_mha: N=%s%lld > 128", "", N);
  if (((uintptr_t)qkv | (uintptr_t)out) & 15) return fail(CO_ERR_BAD_ARG, "co_encoder_mha: pointers must be 16-byte aligned%s");
  if (B == 0) return CO_OK;
  cudaStream_t st = (cudaStream_t)stream;
  // CO_MHA_VARIANT = simt | wgmma forces one kernel (read per call so tests can switch); default: wgmma (scores AND
  // P.V on the tensor core, P in registers) for N > 64, all-SIMT below (a 128 x 128 score tile is mostly padding there).
  const char* ev = getenv("CO_MHA_VARIANT");
  if (ev ? !strcmp(ev, "wgmma") : N > 64) return launch_encoder_mha_wgmma(qkv, out, B, N, st);
  if (ev && strcmp(ev, "simt")) return fail(CO_ERR_BAD_ARG, "co_encoder_mha: CO_MHA_VARIANT must be simt or wgmma%s");
  if (N <= 32) return launch_mha<1, 1>(qkv, out, B, N, st);
  if (N <= 64) return launch_mha<2, 1>(qkv, out, B, N, st);
  return launch_mha<4, 1>(qkv, out, B, N, st);
}
