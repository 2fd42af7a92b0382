// Instance normalisation of the encoder (POMO configuration, `normalization="instance"`): nn.InstanceNorm1d(E, affine=True)
// applied on x.permute(0, 2, 1) (rl4co/models/nn/ops.py:30-54): per (instance, channel) statistics over the N nodes,
// biased variance, y = (x - mean) / sqrt(var + eps) * gamma + beta.  torch dispatches this to a cuDNN batch-norm kernel
// on the permuted tensor; here one CTA per
// instance, thread = channel, rows read coalesced (512 B), the instance (N * 512 B <= 64 KB) stays in L1 for the
// second and third pass: mean, then centred sum of squares (the two-pass form torch's Welford result is closest to).
#include "co_common.cuh"

namespace co {

__global__ void __launch_bounds__(128) instance_norm_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, float* __restrict__ out,
                                                            long B, int N, float eps) {
  const int c = threadIdx.x;
  const float g = gamma ? gamma[c] : 1.0f, bt = beta ? beta[c] : 0.0f;
  const float inv_n = 1.0f / (float)N;
  for (long b = blockIdx.x; b < B; b += gridDim.x) {
    const float* xb = x + (size_t)b * N * E + c;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    int n = 0;
    for (; n + 4 <= N; n += 4) {
      s0 += xb[(size_t)n * E]; s1 += xb[(size_t)(n + 1) * E]; s2 += xb[(size_t)(n + 2) * E]; s3 += xb[(size_t)(n + 3) * E];
    }
    for (; n < N; ++n) s0 += xb[(size_t)n * E];
    const float mean = ((s0 + s1) + (s2 + s3)) * inv_n;
    float q0 = 0.f, q1 = 0.f, q2 = 0.f, q3 = 0.f;
    for (n = 0; n + 4 <= N; n += 4) {
      const float d0 = xb[(size_t)n * E] - mean, d1 = xb[(size_t)(n + 1) * E] - mean;
      const float d2 = xb[(size_t)(n + 2) * E] - mean, d3 = xb[(size_t)(n + 3) * E] - mean;
      q0 = fmaf(d0, d0, q0); q1 = fmaf(d1, d1, q1); q2 = fmaf(d2, d2, q2); q3 = fmaf(d3, d3, q3);
    }
    for (; n < N; ++n) { const float d = xb[(size_t)n * E] - mean; q0 = fmaf(d, d, q0); }
    const float var = ((q0 + q1) + (q2 + q3)) * inv_n;
    const float r = var + eps;
    float rs = rsqrtf(r);                    // 2 ulp; one Newton step brings it to fp32 rounding
    rs = rs * fmaf(-0.5f * r * rs, rs, 1.5f);
    const float a1 = g * rs;
    const float sh = fmaf(-mean, a1, bt);
    float* ob = out + (size_t)b * N * E + c;
    for (n = 0; n < N; ++n) ob[(size_t)n * E] = fmaf(xb[(size_t)n * E], a1, sh);
  }
}

}  // namespace co

using namespace co;

extern "C" int co_instance_norm(const float* x, const float* gamma, const float* beta, float* out, long B, int N,
                                float eps, void* stream) {
  if (!x || !out) return fail(CO_ERR_BAD_ARG, "co_instance_norm: null pointer%s");
  if (B < 0 || N < 1) return fail(CO_ERR_BAD_ARG, "co_instance_norm: bad shape%s");
  if (B == 0) return CO_OK;
  long grid = B;
  const long cap = (long)device_info().sm_count * 16;
  if (grid > cap) grid = cap;
  instance_norm_kernel<<<(unsigned)grid, 128, 0, (cudaStream_t)stream>>>(x, gamma, beta, out, B, N, eps);
  return check_launch("co_instance_norm");
}
