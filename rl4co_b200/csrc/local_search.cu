// 2-opt local search for TSP tours: rl4co/envs/routing/tsp/local_search.py (TSPEnv.local_search, tsp/env.py:184-188).
//
// Reproduces the reference's best-improvement 2-opt bit for bit:
//   * one sweep scores every pair 1 <= i < j <= n-1 (position 0 is fixed) with
//       change = ((d[prev, t_j] + d[t_i, next]) - d[prev, t_i]) - d[t_j, next],   prev = t[i-1], next = t[(j+1) % n]
//     in fp32, left to right, skipping pairs with prev == t_j or next == t_i;
//   * the move taken is the first pair in (i, j) loop order with the strictly smallest change, and only when that
//     change is below -1e-6 as a double; it reverses t[i..j];
//   * sweeps repeat until one finds no move or max_iterations sweeps have run.
// The distance matrix is read as given (no symmetry assumed) with 1e9 added on its diagonal, as the reference does.
//
// One CTA per instance.  The tour and the per-position edge lengths e[k] = d[t[k], t[k+1]] live in shared memory, so a
// candidate costs two matrix reads.  The triangle of (i, j) pairs is folded into a rectangle (row i paired with row
// n-1-i, together n-1 entries) that the CTA sweeps with a constant stride.  The selected move is the minimum of the
// 64-bit key (orderable bits of change, i * n + j): ties in change fall to the smaller loop index, as in the reference.
//
// Distances come from one of
//   * a [B, N, N] float32 matrix, staged in shared memory when N <= CO_TWO_OPT_RESIDENT_MAX_NODES, else read
//     through L2;
//   * locs [B, N, 2]: the matrix computed in shared memory (same bound), else each distance computed on demand from
//     locs staged in shared memory.  d[a, b] = sqrt(fma(dy, dy, dx * dx)) with dx = x_a - x_b: the value torch's CPU
//     2-norm of a 2-vector produces (rl4co.utils.ops.get_distance_matrix), written with explicit round-to-nearest
//     intrinsics so that no compiler flag can change it.
#include "co_common.cuh"

namespace co {

constexpr int LS_SRC_LOCS = 0, LS_SRC_DIST = 1;
constexpr int LS_MAX_THREADS = 512;
constexpr unsigned long long LS_NONE = ~0ull;

__device__ __forceinline__ float ls_euclid(float2 a, float2 b) {
  const float dx = __fsub_rn(a.x, b.x), dy = __fsub_rn(a.y, b.y);
  return __fsqrt_rn(__fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
}

// distance source of one instance; `mat` is the shared-memory matrix (RESIDENT), `gmat` the instance's global matrix,
// `xy` its locs in shared memory
template <int SRC, bool RESIDENT>
struct LsDist {
  const float* mat;
  const float* __restrict__ gmat;
  const float2* xy;
  int n;
  __device__ __forceinline__ float operator()(int a, int b) const {
    if (RESIDENT) return mat[a * n + b];  // diagonal already carries the +1e9
    const float v = (SRC == LS_SRC_DIST) ? __ldg(gmat + (size_t)a * n + b) : ls_euclid(xy[a], xy[b]);
    return a == b ? __fadd_rn(v, 1e9f) : v;
  }
};

__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long w = __shfl_xor_sync(FULL, v, o);
    v = w < v ? w : v;
  }
  return v;
}

__host__ __device__ constexpr int ls_pad2(int n) { return (n + 1) & ~1; }

// dynamic shared memory: best-key slots [2] u64 | e [N] f32 | t [N] i32 | matrix [N*N] f32 or locs [N] float2
inline size_t ls_smem_bytes(int N, bool resident, int src) {
  size_t s = 16 + 8 * (size_t)ls_pad2(N);
  if (resident) s += 4 * (size_t)N * N;
  else if (src == LS_SRC_LOCS) s += 8 * (size_t)N;
  return s;
}

template <int SRC, bool RESIDENT>
__global__ void __launch_bounds__(LS_MAX_THREADS) two_opt_kernel(const float2* __restrict__ locs, const float* __restrict__ dist,
                                                                 const int64_t* tours_in, int64_t* tours_out,
                                                                 int32_t* iterations, int N, int max_iterations) {
  extern __shared__ __align__(16) unsigned char ls_smem[];
  unsigned long long* s_best = reinterpret_cast<unsigned long long*>(ls_smem);
  float* s_e = reinterpret_cast<float*>(ls_smem + 16);
  int* s_t = reinterpret_cast<int*>(s_e + ls_pad2(N));
  float* s_x = reinterpret_cast<float*>(s_t + ls_pad2(N));  // 8-byte aligned: matrix or locs
  const int tid = threadIdx.x, nthr = blockDim.x;
  const size_t b = blockIdx.x;
  const int64_t* tin = tours_in + b * N;
  int64_t* tout = tours_out + b * N;

  int bad = 0;
  for (int k = tid; k < N; k += nthr) {
    const int64_t v = tin[k];
    bad |= (v < 0 || v >= N);
    s_t[k] = (int)v;
  }
  if (tid == 0) s_best[0] = s_best[1] = LS_NONE;
  // an id outside [0, N) would index outside the matrix: copy the tour through untouched and report -1 iterations
  if (__syncthreads_or(bad)) {
    for (int k = tid; k < N; k += nthr) tout[k] = tin[k];  // same thread, same k: safe when tours_out == tours_in
    if (iterations != nullptr && tid == 0) iterations[b] = -1;
    return;
  }

  const float2* xy_g = locs + b * N;
  const float* gmat = (SRC == LS_SRC_DIST) ? dist + b * (size_t)N * N : nullptr;
  if (RESIDENT) {
    for (int k = tid; k < N * N; k += nthr) {
      const int r = k / N, c = k - r * N;
      const float v = (SRC == LS_SRC_DIST) ? __ldg(gmat + k) : ls_euclid(__ldg(xy_g + r), __ldg(xy_g + c));
      s_x[k] = r == c ? __fadd_rn(v, 1e9f) : v;
    }
  } else if (SRC == LS_SRC_LOCS) {
    for (int k = tid; k < N; k += nthr) reinterpret_cast<float2*>(s_x)[k] = __ldg(xy_g + k);
  }
  __syncthreads();
  const LsDist<SRC, RESIDENT> D{s_x, gmat, reinterpret_cast<const float2*>(s_x), N};
  for (int k = tid; k < N; k += nthr) s_e[k] = D(s_t[k], s_t[k + 1 == N ? 0 : k + 1]);
  __syncthreads();

  // (double)change < -1e-6  <=>  change <= thr, thr = the largest float below -1e-6 (no fp64 in the sweep)
  float thr = -1e-6f;
  if ((double)thr >= -1e-6) thr = nextafterf(thr, -INFINITY);

  // folded triangle: R = N-2 rows (i = r+1, N-2-r entries each); rows r and R-1-r share one line of W = N-1 slots
  const int R = N - 2, W = max(N - 1, 1);
  const int lines = (R + 1) / 2;
  const int dr = nthr / W, dc = nthr - dr * W;
  int it = 0;
  while (it < max_iterations) {
    unsigned long long key = LS_NONE;
    for (int r = tid / W, c = tid - r * W; r < lines;) {
      const int L = N - 2 - r;  // entries of row r; row R-1-r fills the rest of the line
      const bool first = c < L;
      const int i = first ? r + 1 : R - r;
      const int j = i + 1 + (first ? c : c - L);
      const int jn = j + 1 == N ? 0 : j + 1;
      const int prev = s_t[i - 1], ti = s_t[i], tj = s_t[j], next = s_t[jn];
      // the middle row of an odd R is its own partner: only its first half counts
      const bool skip = (!first && R - 1 - r == r) || prev == tj || next == ti;
      if (!skip) {
        const float change = __fsub_rn(__fsub_rn(__fadd_rn(D(prev, tj), D(ti, next)), s_e[i - 1]), s_e[j]);
        if (change <= thr) {
          // change < 0 here, and ~bits orders negative floats by ascending value
          const unsigned long long k64 = ((unsigned long long)(~__float_as_uint(change)) << 32) | (unsigned)(i * N + j);
          key = k64 < key ? k64 : key;
        }
      }
      r += dr;
      c += dc;
      if (c >= W) {
        c -= W;
        ++r;
      }
    }
    key = warp_min_u64(key);
    unsigned long long* slot = s_best + (it & 1);
    if ((tid & 31) == 0 && key != LS_NONE) atomicMin(slot, key);
    __syncthreads();
    const unsigned long long best = *slot;
    ++it;
    // the other slot was last read before the previous iteration's final barrier: reset it for the next sweep
    if (tid == 0) s_best[it & 1] = LS_NONE;
    if (best == LS_NONE) break;
    const int pq = (int)(best & 0xffffffffu), p = pq / N, q = pq - p * N;
    for (int k = tid; k < (q - p + 1) / 2; k += nthr) {
      const int a = s_t[p + k];
      s_t[p + k] = s_t[q - k];
      s_t[q - k] = a;
    }
    __syncthreads();
    // edges p-1 .. q changed (inside the segment they now run the other way: recomputed, as d may be asymmetric)
    for (int k = p - 1 + tid; k <= q; k += nthr) s_e[k] = D(s_t[k], s_t[k + 1 == N ? 0 : k + 1]);
    __syncthreads();
  }
  for (int k = tid; k < N; k += nthr) tout[k] = s_t[k];
  if (iterations != nullptr && tid == 0) iterations[b] = it;
}

template <int SRC, bool RESIDENT>
int launch_two_opt(const float* locs, const float* dist, const int64_t* tours_in, int64_t* tours_out, int32_t* iterations,
                   int B, int N, int max_iterations, cudaStream_t stream) {
  const size_t smem = ls_smem_bytes(N, RESIDENT, SRC);
  auto kern = two_opt_kernel<SRC, RESIDENT>;
  if (RESIDENT) {  // the streaming variants stay below 48 KB (N <= CO_TWO_OPT_MAX_NODES)
    static PerDeviceOnce once;
    if (!once.flag()) {
      if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, device_info().max_smem_optin) !=
          cudaSuccess)
        return check_launch("co_tsp_two_opt (shared-memory attribute)");
      once.flag() = true;
    }
  }
  int threads = 32;
  while (threads < N && threads < LS_MAX_THREADS) threads *= 2;
  if (N > 128) threads = LS_MAX_THREADS;
  kern<<<B, threads, smem, stream>>>(reinterpret_cast<const float2*>(locs), dist, tours_in, tours_out, iterations, N,
                                     max_iterations);
  return check_launch("co_tsp_two_opt");
}

}  // namespace co

using namespace co;

extern "C" int co_tsp_two_opt(const float* locs, const float* dist, const int64_t* tours_in, int64_t* tours_out,
                              int32_t* iterations, int B, int N, int max_iterations, void* stream) {
  if ((locs == nullptr) == (dist == nullptr)) return fail(CO_ERR_BAD_ARG, "co_tsp_two_opt: exactly one of locs / dist%s");
  if (!tours_in || !tours_out) return fail(CO_ERR_BAD_ARG, "co_tsp_two_opt: null tour pointer%s");
  if (B < 0 || N < 1) return fail(CO_ERR_BAD_ARG, "co_tsp_two_opt: bad shape%s B=%lld N=%lld", "", B, N);
  if (N > CO_TWO_OPT_MAX_NODES)
    return fail(CO_ERR_UNSUPPORTED, "co_tsp_two_opt: N above the supported maximum%s (N=%lld, max %lld)", "", N,
                CO_TWO_OPT_MAX_NODES);
  if (B == 0) return CO_OK;
  max_iterations = max_iterations < 0 ? 0 : max_iterations;
  // the matrix is kept resident in shared memory up to CO_TWO_OPT_RESIDENT_MAX_NODES (and when the device allows the
  // opt-in size); all paths produce the same tours
  const bool resident = N <= CO_TWO_OPT_RESIDENT_MAX_NODES &&
                        ls_smem_bytes(N, true, 0) <= (size_t)device_info().max_smem_optin;
  cudaStream_t s = (cudaStream_t)stream;
  if (dist != nullptr)
    return resident ? launch_two_opt<LS_SRC_DIST, true>(locs, dist, tours_in, tours_out, iterations, B, N, max_iterations, s)
                    : launch_two_opt<LS_SRC_DIST, false>(locs, dist, tours_in, tours_out, iterations, B, N, max_iterations, s);
  return resident ? launch_two_opt<LS_SRC_LOCS, true>(locs, dist, tours_in, tours_out, iterations, B, N, max_iterations, s)
                  : launch_two_opt<LS_SRC_LOCS, false>(locs, dist, tours_in, tours_out, iterations, B, N, max_iterations, s);
}
