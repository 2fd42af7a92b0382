// Differentiable attention core for the TRAINING step (SURVEY.md 8f-2): forward with saved row statistics and the two
// backward kernels of  O = softmax(Q K^T / sqrt(16) [+ mask]) V  for 8 heads x 16 channels, fp32, N <= 128 keys,
// M <= 256 queries.  One kernel family serves both users:
//   * encoder self-attention under autograd (M = N, no mask)  rl4co/models/nn/attention.py:110-134
//   * the glimpse of the teacher-forced log-likelihood pass: all T decode steps of an instance are T independent
//     queries against its cached K / V with the replayed action mask (models/zoo/am/decoder.py:156-193,
//     nn/attention.py:300-314; Evaluate decoding utils/decoding.py:448-461)
// replacing torch's mem-efficient SDPA (fp32 fmha_cutlassF/B 64x64).
//
// Design: head dimension 16 makes this a SIMT fp32 problem (a 16-deep contraction per score): one CTA per
// (instance, head); K_h / V_h (forward, dQ) or Q_h / dO_h (dK, dV) staged once in shared memory and read as
// warp-uniform LDS.128 broadcasts; every thread owns TWO query rows (or two keys) so that each broadcast feeds two
// float2 FMA chains (one row per thread would be bound by the 2-cycle LDS.128 broadcast, not by the FMA pipe).
// No N x N matrix ever exists in memory: the backward recomputes the probabilities from the saved log-sum-exp.
//   forward: two passes over the keys (row max, then exp / accumulate): exact softmax, 24 FMA pairs per (row, key)
//   dQ     : thread = 2 query rows;  dS = P o (dO V^T - rowsum(dO o O));  dQ = scale * dS K
//   dK, dV : thread = 2 keys;        dK = scale * dS^T Q,  dV = P^T dO      (no atomics, no cross-thread reduction)
// Masks come bit-packed: 4 x uint32 per query row (bit n of word n / 32 set = key n may be attended).
#include "co_common.cuh"

namespace co {
namespace attn {

constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float lg2(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct Row {  // 16 channels of one row as packed pairs
  float2 c[8];
};
__device__ __forceinline__ Row load_row(const float* p, float mul) {
  Row r;
  const float4* p4 = reinterpret_cast<const float4*>(p);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 x = __ldg(p4 + i);
    r.c[2 * i] = make_float2(x.x * mul, x.y * mul);
    r.c[2 * i + 1] = make_float2(x.z * mul, x.w * mul);
  }
  return r;
}
__device__ __forceinline__ Row zero_row() {
  Row r;
#pragma unroll
  for (int i = 0; i < 8; ++i) r.c[i] = make_float2(0.f, 0.f);
  return r;
}
__device__ __forceinline__ void store_row(float* p, const Row& r, float mul) {
  float4* p4 = reinterpret_cast<float4*>(p);
#pragma unroll
  for (int i = 0; i < 4; ++i)
    p4[i] = make_float4(r.c[2 * i].x * mul, r.c[2 * i].y * mul, r.c[2 * i + 1].x * mul, r.c[2 * i + 1].y * mul);
}
// dot of a register row with a shared-memory row (warp-uniform address: broadcast)
__device__ __forceinline__ float dot_s(const Row& a, const float4* s) {
  float2 acc0 = make_float2(0.f, 0.f), acc1 = acc0;  // two chains of four: half the dependent latency
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 x = s[i];
    acc0 = ffma2(a.c[2 * i], make_float2(x.x, x.y), acc0);
    acc1 = ffma2(a.c[2 * i + 1], make_float2(x.z, x.w), acc1);
  }
  return (acc0.x + acc1.x) + (acc0.y + acc1.y);
}
__device__ __forceinline__ void axpy_s(Row& y, float a, const float4* s) {  // y += a * s
  const float2 a2 = make_float2(a, a);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 x = s[i];
    y.c[2 * i] = ffma2(a2, make_float2(x.x, x.y), y.c[2 * i]);
    y.c[2 * i + 1] = ffma2(a2, make_float2(x.z, x.w), y.c[2 * i + 1]);
  }
}
__device__ __forceinline__ bool bit(const uint4& w, int n) {
  const uint32_t x = (n < 64) ? ((n < 32) ? w.x : w.y) : ((n < 96) ? w.z : w.w);
  return (x >> (n & 31)) & 1u;
}

// stage rows [0, R) x 16 channels of head h from a strided global tensor into shared memory (row-major, 64 B rows)
__device__ __forceinline__ void stage(float* dst, const float* src, int R, int rs, float mul) {
  for (int idx = threadIdx.x; idx < R * 4; idx += blockDim.x) {
    const int r = idx >> 2, c = idx & 3;
    float4 x = __ldg(reinterpret_cast<const float4*>(src + (size_t)r * rs) + c);
    x.x *= mul; x.y *= mul; x.z *= mul; x.w *= mul;
    reinterpret_cast<float4*>(dst)[idx] = x;
  }
}

// ------------------------------------------------------------------ forward
__global__ void __launch_bounds__(128) attn_fwd_kernel(const co_attn_args A) {
  extern __shared__ __align__(16) float smem[];
  const int N = A.N, M = A.M;
  float* Ks = smem;
  float* Vs = smem + N * 16;
  const int b = blockIdx.x >> 3, h = blockIdx.x & 7;
  stage(Ks, A.k + (size_t)b * A.k_bs + h * 16, N, A.k_rs, 1.0f);
  stage(Vs, A.v + (size_t)b * A.v_bs + h * 16, N, A.v_rs, 1.0f);
  __syncthreads();
  const int half = (M + 1) >> 1;
  const int t = threadIdx.x;
  if (t >= half) return;
  const int r0 = t, r1 = t + half;
  const bool has1 = r1 < M;
  const float qs = A.scale * LOG2E;  // scores in log2 units
  const float* qb = A.q + (size_t)b * A.q_bs + h * 16;
  const Row q0 = load_row(qb + (size_t)r0 * A.q_rs, qs);
  const Row q1 = has1 ? load_row(qb + (size_t)r1 * A.q_rs, qs) : zero_row();
  uint4 w0 = make_uint4(~0u, ~0u, ~0u, ~0u), w1 = w0;
  if (A.mask) {
    const uint4* mb = reinterpret_cast<const uint4*>(A.mask) + (size_t)b * M;
    w0 = __ldg(mb + r0);
    if (has1) w1 = __ldg(mb + r1);
  }
  const float4* K4 = reinterpret_cast<const float4*>(Ks);
  const float4* V4 = reinterpret_cast<const float4*>(Vs);
  float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll 2
  for (int j = 0; j < N; ++j) {
    const float s0 = dot_s(q0, K4 + 4 * j), s1 = dot_s(q1, K4 + 4 * j);
    m0 = bit(w0, j) ? fmaxf(m0, s0) : m0;
    m1 = bit(w1, j) ? fmaxf(m1, s1) : m1;
  }
  Row a0 = zero_row(), a1 = zero_row();
  float l0 = 0.f, l1 = 0.f;
#pragma unroll 2
  for (int j = 0; j < N; ++j) {
    const float s0 = dot_s(q0, K4 + 4 * j), s1 = dot_s(q1, K4 + 4 * j);
    const float p0 = bit(w0, j) ? ex2(s0 - m0) : 0.f;
    const float p1 = bit(w1, j) ? ex2(s1 - m1) : 0.f;
    l0 += p0; l1 += p1;
    axpy_s(a0, p0, V4 + 4 * j);
    axpy_s(a1, p1, V4 + 4 * j);
  }
  float* ob = A.o + (size_t)b * A.o_bs + h * 16;
  float* lb = A.lse + ((size_t)b * 8 + h) * M;
  store_row(ob + (size_t)r0 * A.o_rs, a0, l0 > 0.f ? 1.0f / l0 : 0.f);
  lb[r0] = l0 > 0.f ? m0 + lg2(l0) : 0.f;  // log2-sum-exp2 of the scaled scores
  if (has1) {
    store_row(ob + (size_t)r1 * A.o_rs, a1, l1 > 0.f ? 1.0f / l1 : 0.f);
    lb[r1] = l1 > 0.f ? m1 + lg2(l1) : 0.f;
  }
}

// ------------------------------------------------------------------ backward: dQ (thread = two query rows)
__global__ void __launch_bounds__(128) attn_bwd_dq_kernel(const co_attn_args A) {
  extern __shared__ __align__(16) float smem[];
  const int N = A.N, M = A.M;
  float* Ks = smem;
  float* Vs = smem + N * 16;
  const int b = blockIdx.x >> 3, h = blockIdx.x & 7;
  stage(Ks, A.k + (size_t)b * A.k_bs + h * 16, N, A.k_rs, 1.0f);
  stage(Vs, A.v + (size_t)b * A.v_bs + h * 16, N, A.v_rs, 1.0f);
  __syncthreads();
  const int half = (M + 1) >> 1;
  const int t = threadIdx.x;
  if (t >= half) return;
  const int r0 = t, r1 = t + half;
  const bool has1 = r1 < M;
  const float qs = A.scale * LOG2E;
  const float* qb = A.q + (size_t)b * A.q_bs + h * 16;
  const float* ob = A.o + (size_t)b * A.o_bs + h * 16;
  const float* gb = A.dO + (size_t)b * A.o_bs + h * 16;
  const float* lb = A.lse + ((size_t)b * 8 + h) * M;
  const Row q0 = load_row(qb + (size_t)r0 * A.q_rs, qs);
  const Row q1 = has1 ? load_row(qb + (size_t)r1 * A.q_rs, qs) : zero_row();
  const Row g0 = load_row(gb + (size_t)r0 * A.o_rs, 1.0f);
  const Row g1 = has1 ? load_row(gb + (size_t)r1 * A.o_rs, 1.0f) : zero_row();
  float D0, D1;
  {
    const Row o0 = load_row(ob + (size_t)r0 * A.o_rs, 1.0f);
    const Row o1 = has1 ? load_row(ob + (size_t)r1 * A.o_rs, 1.0f) : zero_row();
    float2 d0 = make_float2(0.f, 0.f), d1 = d0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { d0 = ffma2(g0.c[i], o0.c[i], d0); d1 = ffma2(g1.c[i], o1.c[i], d1); }
    D0 = d0.x + d0.y; D1 = d1.x + d1.y;
  }
  const float e0 = __ldg(lb + r0), e1 = has1 ? __ldg(lb + r1) : 0.f;
  uint4 w0 = make_uint4(~0u, ~0u, ~0u, ~0u), w1 = w0;
  if (A.mask) {
    const uint4* mb = reinterpret_cast<const uint4*>(A.mask) + (size_t)b * M;
    w0 = __ldg(mb + r0);
    if (has1) w1 = __ldg(mb + r1);
  }
  if (!has1) w1 = make_uint4(0u, 0u, 0u, 0u);
  const float4* K4 = reinterpret_cast<const float4*>(Ks);
  const float4* V4 = reinterpret_cast<const float4*>(Vs);
  Row dq0 = zero_row(), dq1 = zero_row();
#pragma unroll 2
  for (int j = 0; j < N; ++j) {
    const float s0 = dot_s(q0, K4 + 4 * j), s1 = dot_s(q1, K4 + 4 * j);
    const float dp0 = dot_s(g0, V4 + 4 * j), dp1 = dot_s(g1, V4 + 4 * j);
    const float p0 = bit(w0, j) ? ex2(s0 - e0) : 0.f;
    const float p1 = bit(w1, j) ? ex2(s1 - e1) : 0.f;
    axpy_s(dq0, p0 * (dp0 - D0), K4 + 4 * j);
    axpy_s(dq1, p1 * (dp1 - D1), K4 + 4 * j);
  }
  float* db = A.dq + (size_t)b * A.dq_bs + h * 16;
  store_row(db + (size_t)r0 * A.dq_rs, dq0, A.scale);
  if (has1) store_row(db + (size_t)r1 * A.dq_rs, dq1, A.scale);
}

// ------------------------------------------------------------------ backward: dK, dV (thread = two keys)
__global__ void __launch_bounds__(64) attn_bwd_dkv_kernel(const co_attn_args A) {
  extern __shared__ __align__(16) float smem[];
  const int N = A.N, M = A.M;
  float* Qs = smem;                       // [M][16], pre-scaled by scale * log2(e)
  float* Gs = smem + M * 16;              // [M][16] dO
  const int Mp = (M + 3) & ~3;            // keeps the mask words 16-byte aligned
  float* Es = Gs + M * 16;                // [Mp] log2-sum-exp2
  float* Ds = Es + Mp;                    // [Mp] rowsum(dO o O)
  uint32_t* Ws = reinterpret_cast<uint32_t*>(Ds + Mp);  // [M][4] mask words
  const int b = blockIdx.x >> 3, h = blockIdx.x & 7;
  const float qs = A.scale * LOG2E;
  stage(Qs, A.q + (size_t)b * A.q_bs + h * 16, M, A.q_rs, qs);
  stage(Gs, A.dO + (size_t)b * A.o_bs + h * 16, M, A.o_rs, 1.0f);
  {
    const float* ob = A.o + (size_t)b * A.o_bs + h * 16;
    const float* gb = A.dO + (size_t)b * A.o_bs + h * 16;
    const float* lb = A.lse + ((size_t)b * 8 + h) * M;
    for (int i = threadIdx.x; i < M; i += blockDim.x) {
      const Row o = load_row(ob + (size_t)i * A.o_rs, 1.0f), g = load_row(gb + (size_t)i * A.o_rs, 1.0f);
      float2 d = make_float2(0.f, 0.f);
#pragma unroll
      for (int c = 0; c < 8; ++c) d = ffma2(g.c[c], o.c[c], d);
      Ds[i] = d.x + d.y;
      Es[i] = __ldg(lb + i);
      uint4 w = make_uint4(~0u, ~0u, ~0u, ~0u);
      if (A.mask) w = __ldg(reinterpret_cast<const uint4*>(A.mask) + (size_t)b * M + i);
      reinterpret_cast<uint4*>(Ws)[i] = w;
    }
  }
  __syncthreads();
  const int half = (N + 1) >> 1;
  const int t = threadIdx.x;
  if (t >= half) return;
  const int j0 = t, j1 = t + half;
  const bool has1 = j1 < N;
  const float* kb = A.k + (size_t)b * A.k_bs + h * 16;
  const float* vb = A.v + (size_t)b * A.v_bs + h * 16;
  const Row k0 = load_row(kb + (size_t)j0 * A.k_rs, 1.0f);
  const Row k1 = has1 ? load_row(kb + (size_t)j1 * A.k_rs, 1.0f) : zero_row();
  const Row v0 = load_row(vb + (size_t)j0 * A.v_rs, 1.0f);
  const Row v1 = has1 ? load_row(vb + (size_t)j1 * A.v_rs, 1.0f) : zero_row();
  Row dk0 = zero_row(), dk1 = zero_row(), dv0 = zero_row(), dv1 = zero_row();
  const float4* Q4 = reinterpret_cast<const float4*>(Qs);
  const float4* G4 = reinterpret_cast<const float4*>(Gs);
  const int wsel0 = j0 >> 5, wsel1 = j1 >> 5;
  const uint32_t bit0 = 1u << (j0 & 31), bit1 = has1 ? (1u << (j1 & 31)) : 0u;
#pragma unroll 2
  for (int i = 0; i < M; ++i) {
    const float s0 = dot_s(k0, Q4 + 4 * i), s1 = dot_s(k1, Q4 + 4 * i);
    const float dp0 = dot_s(v0, G4 + 4 * i), dp1 = dot_s(v1, G4 + 4 * i);
    const float e = Es[i], Dd = Ds[i];
    const bool f0 = Ws[4 * i + wsel0] & bit0, f1 = Ws[4 * i + (has1 ? wsel1 : 0)] & bit1;
    const float p0 = f0 ? ex2(s0 - e) : 0.f;
    const float p1 = f1 ? ex2(s1 - e) : 0.f;
    axpy_s(dk0, p0 * (dp0 - Dd), Q4 + 4 * i);
    axpy_s(dk1, p1 * (dp1 - Dd), Q4 + 4 * i);
    axpy_s(dv0, p0, G4 + 4 * i);
    axpy_s(dv1, p1, G4 + 4 * i);
  }
  // dK = scale * dS^T Q with Qs = Q * scale * log2(e)  ->  multiply by 1 / log2(e)
  float* dkb = A.dk + (size_t)b * A.dk_bs + h * 16;
  float* dvb = A.dv + (size_t)b * A.dv_bs + h * 16;
  store_row(dkb + (size_t)j0 * A.dk_rs, dk0, LN2);
  store_row(dvb + (size_t)j0 * A.dv_rs, dv0, 1.0f);
  if (has1) {
    store_row(dkb + (size_t)j1 * A.dk_rs, dk1, LN2);
    store_row(dvb + (size_t)j1 * A.dv_rs, dv1, 1.0f);
  }
}

static int check(const co_attn_args& A, bool bwd) {
  if (!A.q || !A.k || !A.v || !A.o || !A.lse) return fail(CO_ERR_BAD_ARG, "co_attn: null pointer%s");
  if (bwd && (!A.dO || !A.dq || !A.dk || !A.dv)) return fail(CO_ERR_BAD_ARG, "co_attn_bwd: null gradient pointer%s");
  if (A.B < 0 || A.M < 1 || A.N < 1) return fail(CO_ERR_BAD_ARG, "co_attn: bad shape%s");
  if (A.N > 128 || A.M > 256) return fail(CO_ERR_UNSUPPORTED, "co_attn: N=%s%lld > 128 keys or M=%lld > 256 queries", "", A.N, A.M);
  const long strides[] = {A.q_rs, A.k_rs, A.v_rs, A.o_rs, A.q_bs, A.k_bs, A.v_bs, A.o_bs};
  for (long s : strides)
    if (s % 4) return fail(CO_ERR_BAD_ARG, "co_attn: strides must be multiples of 4 floats%s");
  if (bwd) {
    const long g[] = {A.dq_rs, A.dk_rs, A.dv_rs, A.dq_bs, A.dk_bs, A.dv_bs};
    for (long s : g)
      if (s % 4) return fail(CO_ERR_BAD_ARG, "co_attn_bwd: gradient strides must be multiples of 4 floats%s");
  }
  return CO_OK;
}

}  // namespace attn
}  // namespace co

using namespace co;

extern "C" int co_attn_fwd(const co_attn_args* args, void* stream) {
  if (!args) return fail(CO_ERR_BAD_ARG, "co_attn_fwd: null args%s");
  const co_attn_args A = *args;
  int rc = attn::check(A, false);
  if (rc != CO_OK || A.B == 0) return rc;
  const int half = (A.M + 1) / 2;
  const int threads = ((half + 31) / 32) * 32;
  const size_t smem = (size_t)2 * A.N * 16 * sizeof(float);
  attn::attn_fwd_kernel<<<A.B * 8, threads, smem, (cudaStream_t)stream>>>(A);
  return check_launch("co_attn_fwd");
}

extern "C" int co_attn_bwd(const co_attn_args* args, void* stream) {
  if (!args) return fail(CO_ERR_BAD_ARG, "co_attn_bwd: null args%s");
  const co_attn_args A = *args;
  int rc = attn::check(A, true);
  if (rc != CO_OK || A.B == 0) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  {
    const int half = (A.M + 1) / 2;
    const int threads = ((half + 31) / 32) * 32;
    const size_t smem = (size_t)2 * A.N * 16 * sizeof(float);
    attn::attn_bwd_dq_kernel<<<A.B * 8, threads, smem, st>>>(A);
    rc = check_launch("co_attn_bwd(dq)");
    if (rc != CO_OK) return rc;
  }
  {
    const size_t smem = ((size_t)A.M * (2 * 16 + 4) + 2 * ((A.M + 3) & ~3)) * sizeof(float);
    static PerDeviceOnce once;
    bool& configured = once.flag();
    if (!configured) {
      cudaError_t e = cudaFuncSetAttribute(attn::attn_bwd_dkv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 256 * 38 * 4);
      if (e != cudaSuccess) return fail(CO_ERR_CUDA, "co_attn_bwd: smem attribute: %s", cudaGetErrorString(e));
      configured = true;
    }
    attn::attn_bwd_dkv_kernel<<<A.B * 8, 64, smem, st>>>(A);
    rc = check_launch("co_attn_bwd(dk,dv)");
  }
  return rc;
}
