// Data path either side of the rollout (SURVEY.md 8f-3): on-device instance generation and the dihedral-8
// augmentation as single streaming kernels (HBM-bound: 4 B written per generated float, 8 B read + 64 B
// written per node for the augmentation).
//   co_generate_uniform   <- rl4co/envs/common/utils.py:61-62 (get_sampler "uniform": torch.rand * (hi-lo) + lo),
//                            as used by tsp/generator.py:49-58 (locs) and cvrp/generator.py:114-123 (depot + locs)
//   co_generate_demand    <- rl4co/envs/routing/cvrp/generator.py:126-137: (floor(U[lo,hi)) + 1) / capacity with
//                            lo = min_demand - 1, hi = max_demand - 1
//   co_dihedral8          <- rl4co/data/transforms.py:16-38 (aug-major: row a*B + b)
//   co_symmetric_augment  <- rl4co/data/transforms.py:49-86 (rotation about (0.5, 0.5), reflection for phi > 2*pi;
//                            aug-major; the angles come from the caller)
// The random stream is Philox4x32-10 keyed by (seed, offset): same seed -> same instances on every run and on every
// GPU; it is NOT torch's CPU stream, so generated instances are distributionally, not bit-wise, the reference's.
#include "co_common.cuh"

namespace co {

__device__ __forceinline__ float u01(uint32_t r) {  // 24 random bits -> [0, 1), every value exactly representable
  return (float)(r >> 8) * (1.0f / 16777216.0f);
}

// 4 floats per Philox call, 4 calls per thread iteration -> 16-byte stores, grid-stride
__global__ void __launch_bounds__(256) generate_uniform_kernel(float* __restrict__ out, long n, uint64_t seed,
                                                                uint64_t offset, float lo, float hi) {
  const long n4 = n >> 2;
  const float span = hi - lo;
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    const uint4 r = philox4x32_10(make_uint4((uint32_t)i, (uint32_t)(i >> 32), (uint32_t)offset, (uint32_t)(offset >> 32)), key);
    reinterpret_cast<float4*>(out)[i] =
        make_float4(u01(r.x) * span + lo, u01(r.y) * span + lo, u01(r.z) * span + lo, u01(r.w) * span + lo);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {  // tail (n not a multiple of 4)
    const long i = n4;
    const uint4 r = philox4x32_10(make_uint4((uint32_t)i, (uint32_t)(i >> 32), (uint32_t)offset, (uint32_t)(offset >> 32)), key);
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
    out[4 * n4 + threadIdx.x] = u01(w[threadIdx.x]) * span + lo;
  }
}

__global__ void __launch_bounds__(256) generate_demand_kernel(float* __restrict__ out, long n, uint64_t seed,
                                                               uint64_t offset, float lo, float hi, float capacity) {
  const float span = hi - lo;
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < ((n + 3) >> 2); i += (long)gridDim.x * blockDim.x) {
    const uint4 r = philox4x32_10(make_uint4((uint32_t)i, (uint32_t)(i >> 32), (uint32_t)offset, (uint32_t)(offset >> 32)), key);
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long k = 4 * i + j;
      // (demand.int() + 1).float() / capacity : truncation towards zero of a non-negative value
      if (k < n) out[k] = ((float)((int)(u01(w[j]) * span + lo) + 1)) / capacity;
    }
  }
}

// one thread per (instance, node): reads (x, y) once, writes the 8 images; writes are float2-coalesced per image
__global__ void __launch_bounds__(256) dihedral8_kernel(const float2* __restrict__ xy, float2* __restrict__ out, long BN) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < BN; i += (long)gridDim.x * blockDim.x) {
    const float2 p = xy[i];
    const float x = p.x, y = p.y, rx = 1.0f - p.x, ry = 1.0f - p.y;
    out[0 * BN + i] = make_float2(x, y);
    out[1 * BN + i] = make_float2(rx, y);
    out[2 * BN + i] = make_float2(x, ry);
    out[3 * BN + i] = make_float2(rx, ry);
    out[4 * BN + i] = make_float2(y, x);
    out[5 * BN + i] = make_float2(ry, x);
    out[6 * BN + i] = make_float2(y, rx);
    out[7 * BN + i] = make_float2(ry, rx);
  }
}

// symmetric_transform (transforms.py:49-69) with torch's rounding: every operation is its own elementwise kernel in
// the reference, so each is rounded on its own here (__f*_rn: no FMA contraction) and cos / sin are the precise
// cosf / sinf.  The reflection test compares against 2*pi rounded to fp32, as torch does for an fp32 tensor.
constexpr float TWO_PI_F32 = 6.28318530717958647692f;

// One warp per 32 consecutive nodes of the flattened base [B*N]: each lane reads its node once and writes its S
// images.  The warp's nodes belong to nw <= 32 consecutive instances, so one cos / sin evaluation by the whole warp
// covers 32 / nw images of all of them: lane l takes instance b0 + l % nw of image a0 + l / nw, and each lane fetches
// its own (image, instance) values with shuffles.  Every loop bound is warp-uniform.
__global__ void __launch_bounds__(256) symmetric_augment_kernel(const float2* __restrict__ xy,
                                                                const float* __restrict__ phi,
                                                                float2* __restrict__ out, long B, int S, int N) {
  const long BN = B * (long)N;
  const int lane = threadIdx.x & 31;
  const long nwarps = (long)gridDim.x * (blockDim.x >> 5);
  for (long w = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w * 32 < BN; w += nwarps) {
    const long i0 = w * 32, i = i0 + lane, b0 = i0 / N;
    const bool live = i < BN;
    const int k = (int)(i0 - b0 * N + lane) / N;                    // this lane's instance is b0 + k
    const int nw = (int)((i0 + 31 < BN ? i0 + 31 : BN - 1) / N - b0) + 1;  // instances in this warp
    const int per = 32 / nw;                                            // images per cos / sin evaluation
    const long pb = b0 + lane % nw;
    float x0 = 0.f, y0 = 0.f;
    if (live) {
      const float2 p = xy[i];
      x0 = __fsub_rn(p.x, 0.5f);
      y0 = __fsub_rn(p.y, 0.5f);
    }
    for (int a0 = 0; a0 < S; a0 += per) {
      const int pa = a0 + lane / nw;
      const float f = pa < S && lane < per * nw ? phi[(long)pa * B + pb] : 0.f;
      const float cf = cosf(f), sf = sinf(f);
      const int na = S - a0 < per ? S - a0 : per;
      for (int j = 0; j < na; ++j) {
        const int src = j * nw + k;
        const float c = __shfl_sync(FULL, cf, src), s = __shfl_sync(FULL, sf, src);
        const bool reflect = __shfl_sync(FULL, f, src) > TWO_PI_F32;
        if (live) {
          const float xr = __fsub_rn(__fmul_rn(c, x0), __fmul_rn(s, y0));
          const float yr = __fadd_rn(__fmul_rn(s, x0), __fmul_rn(c, y0));
          out[(long)(a0 + j) * BN + i] = reflect ? make_float2(__fadd_rn(yr, 0.5f), __fadd_rn(xr, 0.5f))
                                                 : make_float2(__fadd_rn(xr, 0.5f), __fadd_rn(yr, 0.5f));
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// co_generate_locs: [B, N, 2] locations from one of the location laws of rl4co/envs/common/distribution_utils.py
// (Bi et al. 2022 cluster / mixed, Zhou et al. 2023 Gaussian mixtures) and get_sampler's normal / constant kinds.
// One CTA per instance (grid-stride over instances).  Every random word comes from Philox keyed by `seed` with the
// counter (instance, draw, offset), so instance b does not depend on the launch shape or on B.  Draw index layout:
//   j < N               node j: words x, y and z, w (two uniforms or one Box-Muller pair each; z picks a GM mode)
//   LD_FISHER_YATES + t mixed: step t of the partial Fisher-Yates shuffle
//   LD_CENTRE + i       centre i of a cluster / mixed / Gaussian-mixture mode
//   LD_INSTANCE         per-instance scalars: x = mix_distribution branch, y = GM(1,1) rho, z = mix_multi setting
constexpr uint32_t LD_FISHER_YATES = 0x40000000u, LD_CENTRE = 0x80000000u, LD_INSTANCE = 0xC0000000u;
constexpr float CLUSTER_LO = 0.2f, CLUSTER_HI = 0.8f, CLUSTER_STD = 0.07f;

struct LocsRng {
  uint2 key;
  uint32_t b, off_lo, off_hi;
  __device__ uint4 draw(uint32_t d) const { return philox4x32_10(make_uint4(b, d, off_lo, off_hi), key); }
};

// two independent N(0, 1) from two words; u1 is in (0, 1) (23 bits + 0.5), so log never sees 0
__device__ __forceinline__ float2 box_muller(uint32_t a, uint32_t b) {
  const float u1 = ((float)(a >> 9) + 0.5f) * (1.0f / 8388608.0f);
  const float r = sqrtf(-2.0f * logf(u1));
  float s, c;
  sincospif(2.0f * u01(b), &s, &c);
  return make_float2(r * c, r * s);
}
__device__ __forceinline__ uint32_t below(uint32_t r, uint32_t n) { return (uint32_t)(((uint64_t)r * n) >> 32); }
__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.0f), 1.0f); }
__device__ __forceinline__ float2 cluster_centre(const LocsRng& g, int i) {
  const uint4 r = g.draw(LD_CENTRE + (uint32_t)i);
  return make_float2(CLUSTER_LO + (CLUSTER_HI - CLUSTER_LO) * u01(r.x), CLUSTER_LO + (CLUSTER_HI - CLUSTER_LO) * u01(r.y));
}

// block-wide (min x, min y, max x, max y); every thread gets the result
__device__ float4 block_minmax(float4 v, float4* scratch) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    v.x = fminf(v.x, __shfl_xor_sync(FULL, v.x, o));
    v.y = fminf(v.y, __shfl_xor_sync(FULL, v.y, o));
    v.z = fmaxf(v.z, __shfl_xor_sync(FULL, v.z, o));
    v.w = fmaxf(v.w, __shfl_xor_sync(FULL, v.w, o));
  }
  __syncthreads();  // scratch may still be read from the previous instance
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  float4 r = scratch[0];
  for (int w = 1; w < nwarps; ++w) {
    const float4 s = scratch[w];
    r = make_float4(fminf(r.x, s.x), fminf(r.y, s.y), fmaxf(r.z, s.z), fmaxf(r.w, s.w));
  }
  return r;
}

__device__ void gen_uniform(float2* out, int N, const LocsRng& g, float lo, float hi) {
  const float span = hi - lo;
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    const uint4 r = g.draw((uint32_t)j);
    out[j] = make_float2(u01(r.x) * span + lo, u01(r.y) * span + lo);
  }
}

// k centres U(0.2, 0.8)^2; k contiguous blocks, the first N mod k of them one node longer; N(centre, 0.07^2 I), clamped
__device__ void gen_cluster(float2* out, int N, const LocsRng& g, int k) {
  const int q = N / k, rem = N % k, head = rem * (q + 1);
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    const int blk = j < head ? j / (q + 1) : rem + (j - head) / q;
    const float2 c = cluster_centre(g, blk);
    const uint4 r = g.draw((uint32_t)j);
    const float2 z = box_muller(r.x, r.y);
    out[j] = make_float2(clamp01(c.x + CLUSTER_STD * z.x), clamp01(c.y + CLUSTER_STD * z.y));
  }
}

// U(0, 1)^2 everywhere; floor(N/2) distinct nodes in random order (partial Fisher-Yates) are cut into k segments of
// floor(N/(2k)) (the last takes the rest) and segment i is redrawn from N(c_i, 0.07^2 I), c_i ~ U(0.2, 0.8)^2; clamped
__device__ void gen_mixed(float2* out, int N, const LocsRng& g, int k, uint16_t* perm, uint16_t* pick) {
  const int M = N / 2, seg = N / (2 * k);
  __syncthreads();  // perm / pick may still be read from the previous instance
  for (int j = threadIdx.x; j < N; j += blockDim.x) perm[j] = (uint16_t)j;
  for (int t = threadIdx.x; t < M; t += blockDim.x)
    pick[t] = (uint16_t)(t + (int)below(g.draw(LD_FISHER_YATES + (uint32_t)t).x, (uint32_t)(N - t)));
  __syncthreads();
  if (threadIdx.x == 0)
    for (int t = 0; t < M; ++t) {
      const uint16_t a = perm[t], p = pick[t];
      perm[t] = perm[p];
      perm[p] = a;
    }
  __syncthreads();
  // perm is a permutation: positions t < M are the redrawn nodes in shuffle order, the rest stay uniform
  for (int t = threadIdx.x; t < N; t += blockDim.x) {
    const int j = perm[t];
    const uint4 r = g.draw((uint32_t)j);
    float2 v;
    if (t < M) {
      const int s = seg > 0 ? min(t / seg, k - 1) : k - 1;
      const float2 c = cluster_centre(g, s);
      const float2 z = box_muller(r.z, r.w);
      v = make_float2(c.x + CLUSTER_STD * z.x, c.y + CLUSTER_STD * z.y);
    } else {
      v = make_float2(u01(r.x), u01(r.y));
    }
    out[j] = make_float2(clamp01(v.x), clamp01(v.y));
  }
}

// GM(1, 1): N((0.5, 0.5), [[1, rho], [rho, 1]]), rho ~ U(0, 1) per instance; shift by the per-coordinate minimum, divide
// both coordinates by the larger range, centre each coordinate with + (1 - max) / 2
__device__ void gen_gaussian(float2* out, int N, const LocsRng& g, float4* scratch) {
  const float rho = u01(g.draw(LD_INSTANCE).y), rho_c = sqrtf(1.0f - rho * rho);
  float4 mm = make_float4(INFINITY, INFINITY, -INFINITY, -INFINITY);
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    const uint4 r = g.draw((uint32_t)j);
    const float2 z = box_muller(r.x, r.y);
    const float2 v = make_float2(0.5f + z.x, 0.5f + fmaf(rho, z.x, rho_c * z.y));
    out[j] = v;
    mm = make_float4(fminf(mm.x, v.x), fminf(mm.y, v.y), fmaxf(mm.z, v.x), fmaxf(mm.w, v.y));
  }
  mm = block_minmax(mm, scratch);
  const float rx = mm.z - mm.x, ry = mm.w - mm.y, range = fmaxf(rx, ry);
  // (v - min) / range and max are monotone, so the scaled maximum of each coordinate is (max - min) / range exactly
  const float sx = (1.0f - rx / range) * 0.5f, sy = (1.0f - ry / range) * 0.5f;
  for (int j = threadIdx.x; j < N; j += blockDim.x) {  // each thread re-reads only what it wrote
    const float2 v = out[j];
    out[j] = make_float2((v.x - mm.x) / range + sx, (v.y - mm.y) / range + sy);
  }
}

// GM(m, c): node modes uniform over m; nodes stored grouped by mode in ascending order (counting sort: position p
// takes the mode whose range of positions holds p); each non-empty mode has a centre U(0, c)^2 and its nodes are
// N(centre, I); then min-max scaling to [0, 1] per coordinate
__device__ void gen_gaussian_mixture(float2* out, int N, const LocsRng& g, int m, float cdist, int* start,
                                     float4* scratch) {
  __syncthreads();  // start[] may still be read from the previous instance
  for (int i = threadIdx.x; i <= m; i += blockDim.x) start[i] = 0;
  __syncthreads();
  for (int j = threadIdx.x; j < N; j += blockDim.x) atomicAdd(&start[1 + below(g.draw((uint32_t)j).z, (uint32_t)m)], 1);
  __syncthreads();
  if (threadIdx.x == 0)
    for (int i = 1; i <= m; ++i) start[i] += start[i - 1];  // start[i] = first position of mode i; start[m] = N
  __syncthreads();
  float4 mm = make_float4(INFINITY, INFINITY, -INFINITY, -INFINITY);
  for (int p = threadIdx.x; p < N; p += blockDim.x) {
    int lo = 0, hi = m;  // last i with start[i] <= p: the non-empty mode whose positions hold p
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (start[mid] <= p) lo = mid; else hi = mid;
    }
    const uint4 rc = g.draw(LD_CENTRE + (uint32_t)lo), r = g.draw((uint32_t)p);
    const float2 z = box_muller(r.x, r.y);
    const float2 v = make_float2(u01(rc.x) * cdist + z.x, u01(rc.y) * cdist + z.y);
    out[p] = v;
    mm = make_float4(fminf(mm.x, v.x), fminf(mm.y, v.y), fmaxf(mm.z, v.x), fmaxf(mm.w, v.y));
  }
  mm = block_minmax(mm, scratch);
  const float rx = mm.z - mm.x, ry = mm.w - mm.y;
  for (int p = threadIdx.x; p < N; p += blockDim.x) {
    const float2 v = out[p];
    out[p] = make_float2((v.x - mm.x) / rx, (v.y - mm.y) / ry);
  }
}

__device__ void gen_gm_any(float2* out, int N, const LocsRng& g, int m, float cdist, int* start, float4* scratch) {
  if (m == 0) gen_uniform(out, N, g, 0.0f, 1.0f);
  else if (m == 1 && cdist == 1.0f) gen_gaussian(out, N, g, scratch);
  else gen_gaussian_mixture(out, N, g, m, cdist, start, scratch);
}

__global__ void __launch_bounds__(256) generate_locs_kernel(float2* __restrict__ locs, co_locs_args a) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ float4 scratch[8];
  const int N = a.N;
  for (long b = blockIdx.x; b < a.B; b += gridDim.x) {
    float2* out = locs + b * N;
    const LocsRng g{make_uint2((uint32_t)a.seed, (uint32_t)(a.seed >> 32)), (uint32_t)b, (uint32_t)a.offset,
                    (uint32_t)(a.offset >> 32)};
    switch (a.kind) {
      case CO_LOCS_UNIFORM: gen_uniform(out, N, g, a.lo, a.hi); break;
      case CO_LOCS_CONSTANT:
        for (int j = threadIdx.x; j < N; j += blockDim.x) out[j] = make_float2(a.lo, a.lo);
        break;
      case CO_LOCS_NORMAL:
        for (int j = threadIdx.x; j < N; j += blockDim.x) {
          const uint4 r = g.draw((uint32_t)j);
          const float2 z = box_muller(r.x, r.y);
          out[j] = make_float2(fmaf(a.std, z.x, a.mean), fmaf(a.std, z.y, a.mean));
        }
        break;
      case CO_LOCS_CLUSTER: gen_cluster(out, N, g, a.n_cluster); break;
      case CO_LOCS_MIXED:
        gen_mixed(out, N, g, a.n_cluster_mix, (uint16_t*)smem, (uint16_t*)smem + N);
        break;
      case CO_LOCS_GAUSSIAN_MIXTURE: gen_gm_any(out, N, g, a.num_modes, a.cdist, (int*)smem, scratch); break;
      case CO_LOCS_MIX_DISTRIBUTION: {
        const float p = u01(g.draw(LD_INSTANCE).x);
        if (p <= 0.33f) gen_mixed(out, N, g, a.n_cluster_mix, (uint16_t*)smem, (uint16_t*)smem + N);
        else if (p <= 0.66f) gen_cluster(out, N, g, a.n_cluster);
        else gen_uniform(out, N, g, 0.0f, 1.0f);
        break;
      }
      case CO_LOCS_MIX_MULTI_DISTRIBUTIONS: {
        // {(0,0), (1,1)} then {3,5,7} x {10,30,50}, in that order
        const int s = (int)below(g.draw(LD_INSTANCE).z, 11u);
        const int m = s < 2 ? s : 3 + 2 * ((s - 2) / 3);
        const float c = s < 2 ? (float)s : 10.0f + 20.0f * (float)((s - 2) % 3);
        gen_gm_any(out, N, g, m, c, (int*)smem, scratch);
        break;
      }
    }
  }
}

}  // namespace co

using namespace co;

static inline int stream_grid(long work) {
  long g = (work + 255) / 256;
  const long cap = (long)device_info().sm_count * 8;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

extern "C" int co_generate_uniform(float* out, long n, uint64_t seed, uint64_t offset, float lo, float hi, void* stream) {
  if (!out) return fail(CO_ERR_BAD_ARG, "co_generate_uniform: null pointer%s");
  if (n < 0 || !(hi >= lo)) return fail(CO_ERR_BAD_ARG, "co_generate_uniform: bad range or size%s");
  if ((uintptr_t)out & 15) return fail(CO_ERR_BAD_ARG, "co_generate_uniform: output must be 16-byte aligned%s");
  if (n == 0) return CO_OK;
  generate_uniform_kernel<<<stream_grid((n + 3) / 4), 256, 0, (cudaStream_t)stream>>>(out, n, seed, offset, lo, hi);
  return check_launch("co_generate_uniform");
}

extern "C" int co_generate_demand(float* out, long n, uint64_t seed, uint64_t offset, int min_demand, int max_demand,
                                  float capacity, void* stream) {
  if (!out) return fail(CO_ERR_BAD_ARG, "co_generate_demand: null pointer%s");
  if (n < 0 || min_demand < 1 || max_demand < min_demand || !(capacity > 0.f))
    return fail(CO_ERR_BAD_ARG, "co_generate_demand: bad arguments%s");
  if (n == 0) return CO_OK;
  generate_demand_kernel<<<stream_grid((n + 3) / 4), 256, 0, (cudaStream_t)stream>>>(
      out, n, seed, offset, (float)(min_demand - 1), (float)(max_demand - 1), capacity);
  return check_launch("co_generate_demand");
}

extern "C" int co_dihedral8(const float* locs, float* out, long B, int N, void* stream) {
  if (!locs || !out) return fail(CO_ERR_BAD_ARG, "co_dihedral8: null pointer%s");
  if (B < 0 || N < 1) return fail(CO_ERR_BAD_ARG, "co_dihedral8: bad shape%s");
  if (B == 0) return CO_OK;
  dihedral8_kernel<<<stream_grid(B * N), 256, 0, (cudaStream_t)stream>>>((const float2*)locs, (float2*)out, B * (long)N);
  return check_launch("co_dihedral8");
}

extern "C" int co_symmetric_augment(const float* base, const float* phi, float* out, long B, int S, int N,
                                    void* stream) {
  if (!base || !phi || !out) return fail(CO_ERR_BAD_ARG, "co_symmetric_augment: null pointer%s");
  if (B < 0 || S < 1 || N < 1) return fail(CO_ERR_BAD_ARG, "co_symmetric_augment: bad shape%s");
  if (((uintptr_t)base | (uintptr_t)out) & 7) return fail(CO_ERR_BAD_ARG, "co_symmetric_augment: base / out must be 8-byte aligned%s");
  if (B == 0) return CO_OK;
  symmetric_augment_kernel<<<stream_grid(B * N), 256, 0, (cudaStream_t)stream>>>(
      (const float2*)base, phi, (float2*)out, B, S, N);
  return check_launch("co_symmetric_augment");
}

extern "C" int co_generate_locs(float* out, const co_locs_args* args, void* stream) {
  if (!out || !args) return fail(CO_ERR_BAD_ARG, "co_generate_locs: null pointer%s");
  const co_locs_args a = *args;
  if ((uintptr_t)out & 7) return fail(CO_ERR_BAD_ARG, "co_generate_locs: output must be 8-byte aligned%s");
  if (a.N < 1 || a.N > CO_LOCS_MAX_NODES) return fail(CO_ERR_BAD_ARG, "co_generate_locs: N = %s%lld outside [1, %lld]", "", a.N, CO_LOCS_MAX_NODES);
  if (a.B < 0 || a.B > 0x7fffffffL) return fail(CO_ERR_BAD_ARG, "co_generate_locs: B = %s%lld outside [0, 2^31)", "", a.B);
  const bool gm = a.kind == CO_LOCS_GAUSSIAN_MIXTURE, multi = a.kind == CO_LOCS_MIX_MULTI_DISTRIBUTIONS;
  const bool cluster = a.kind == CO_LOCS_CLUSTER || a.kind == CO_LOCS_MIX_DISTRIBUTION;
  const bool mixed = a.kind == CO_LOCS_MIXED || a.kind == CO_LOCS_MIX_DISTRIBUTION;
  if (a.kind < CO_LOCS_UNIFORM || a.kind > CO_LOCS_MIX_MULTI_DISTRIBUTIONS)
    return fail(CO_ERR_BAD_ARG, "co_generate_locs: unknown kind %s%lld", "", a.kind);
  if (a.kind == CO_LOCS_UNIFORM && !(a.hi >= a.lo)) return fail(CO_ERR_BAD_ARG, "co_generate_locs: uniform needs hi >= lo%s");
  if (a.kind == CO_LOCS_NORMAL && !(a.std >= 0.f)) return fail(CO_ERR_BAD_ARG, "co_generate_locs: normal needs std >= 0%s");
  if (cluster && (a.n_cluster < 1 || a.n_cluster > CO_LOCS_MAX_NODES))
    return fail(CO_ERR_BAD_ARG, "co_generate_locs: n_cluster = %s%lld outside [1, %lld]", "", a.n_cluster, CO_LOCS_MAX_NODES);
  if (mixed && (a.n_cluster_mix < 1 || a.n_cluster_mix > CO_LOCS_MAX_NODES))
    return fail(CO_ERR_BAD_ARG, "co_generate_locs: n_cluster_mix = %s%lld outside [1, %lld]", "", a.n_cluster_mix, CO_LOCS_MAX_NODES);
  if (gm && (a.num_modes < 0 || a.num_modes > CO_LOCS_MAX_NODES || !(a.cdist >= 0.f)))
    return fail(CO_ERR_BAD_ARG, "co_generate_locs: gaussian_mixture needs 0 <= num_modes <= %s%lld and cdist >= 0", "", CO_LOCS_MAX_NODES);
  // min-max scaling of a single node would divide 0 by 0
  if (((gm && a.num_modes != 0) || multi) && a.N < 2)
    return fail(CO_ERR_BAD_ARG, "co_generate_locs: this gaussian_mixture setting needs N >= 2%s");
  if (a.B == 0) return CO_OK;
  size_t smem = 0;
  if (mixed) smem = 2 * (size_t)a.N + 2 * (size_t)(a.N / 2);  // perm + Fisher-Yates picks (uint16)
  if (gm) smem = 4 * ((size_t)a.num_modes + 1);                // first position of every mode
  if (multi) smem = 4 * 8;
  const int threads = a.N >= 256 ? 256 : ((a.N + 31) / 32) * 32;
  const long cap = (long)device_info().sm_count * (2048 / threads < 32 ? 2048 / threads : 32);
  const int grid = (int)(a.B < cap ? a.B : cap);
  generate_locs_kernel<<<grid, threads, smem, (cudaStream_t)stream>>>((float2*)out, a);
  return check_launch("co_generate_locs");
}
