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
// `xy` its locs in shared memory.  DIAG adds the TSP search's +1e9 on the diagonal; the CVRP search reads d[0][0] as
// given.
template <int SRC, bool RESIDENT, bool DIAG = true>
struct LsDist {
  const float* mat;
  const float* __restrict__ gmat;
  const float2* xy;
  int n;
  __device__ __forceinline__ float operator()(int a, int b) const {
    if (RESIDENT) return mat[a * n + b];  // with DIAG the diagonal already carries the +1e9
    const float v = (SRC == LS_SRC_DIST) ? __ldg(gmat + (size_t)a * n + b) : ls_euclid(xy[a], xy[b]);
    return (DIAG && a == b) ? __fadd_rn(v, 1e9f) : v;
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

// ---------------------------------------------------------------------------------------------------------------------
// CVRP local search (co_cvrp_local_search, corollout.h states the search, the formulas and the key).
//
// One CTA per instance.  Every route keeps its slot and its own depot at both ends.  Ids: customers 1..N, the start
// depot of route r is N+1+r, its end depot 2N+1+r; a depot id reads row / column 0 of the matrix.  Per id the CTA keeps
// {pred, succ, route, position} (position 0 = start depot) and the prefix load; per route the load.  Loads are fp32
// left-to-right sums in route order, recomputed (one thread per changed route) after every move.
//
// A sweep scores every ordered pair (u, v) of customers and used start depots -- ids 1..N+R, R = routes of the input --
// for the four move kinds and keeps the smallest 64-bit key
//   (orderable bits of delta) << 32 | kind << 24 | u << 12 | v,
// which orders candidates by (delta, kind, u, v).  Ids stay below 3N+1 <= 3070 < 4096.
namespace co {

constexpr int CLS_RELOCATE = 0, CLS_SWAP = 1, CLS_TWO_OPT = 2, CLS_TWO_OPT_STAR = 3;

// dynamic shared memory: best-key slots [2] u64 | R, changed routes [2], used length i32 | nd [3N+1] int4 | pref [3N+1] f32 | dem [N+1] f32 | load [N] f32 |
// off [N] i32 | (8-byte aligned) matrix [(N+1)^2] f32 or locs [N+1] float2
struct ClsLayout {
  size_t nd, pref, dem, load, off, x, total;
};
__host__ __device__ inline ClsLayout cls_layout(int N, bool resident, int src) {
  ClsLayout L;
  const size_t E = 3 * (size_t)N + 1, n = (size_t)N + 1;
  L.nd = 32;
  L.pref = L.nd + 16 * E;
  L.dem = L.pref + 4 * E;
  L.load = L.dem + 4 * n;
  L.off = L.load + 4 * (size_t)N;
  L.x = (L.off + 4 * (size_t)N + 7) & ~(size_t)7;
  L.total = L.x + (resident ? 4 * n * n : (src == LS_SRC_LOCS ? 8 * n : 0));
  return L;
}

template <int SRC, bool RESIDENT>
__global__ void __launch_bounds__(LS_MAX_THREADS, 1)
    cvrp_ls_kernel(const float2* __restrict__ locs, const float* __restrict__ dist, const float* __restrict__ demand,
                   const float* __restrict__ capacity, const int64_t* __restrict__ tours_in,
                   int64_t* __restrict__ tours_out, int32_t* __restrict__ used_len, int32_t* __restrict__ iterations,
                   int32_t* __restrict__ feasible, int N, int T, int max_iterations) {
  extern __shared__ __align__(16) unsigned char ls_smem[];
  const ClsLayout lay = cls_layout(N, RESIDENT, SRC);
  unsigned long long* s_best = reinterpret_cast<unsigned long long*>(ls_smem);
  int* s_int = reinterpret_cast<int*>(ls_smem + 16);  // R | changed routes [2] | used length
  int& s_R = s_int[0];
  int* s_chg = s_int + 1;
  int& s_used = s_int[3];
  int4* nd = reinterpret_cast<int4*>(ls_smem + lay.nd);
  float* pref = reinterpret_cast<float*>(ls_smem + lay.pref);
  float* dem = reinterpret_cast<float*>(ls_smem + lay.dem);
  float* load = reinterpret_cast<float*>(ls_smem + lay.load);
  int* off = reinterpret_cast<int*>(ls_smem + lay.off);
  float* s_x = reinterpret_cast<float*>(ls_smem + lay.x);
  const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31;
  const size_t b = blockIdx.x;
  const int n = N + 1, E = 3 * N + 1, W = 2 * N;
  const int64_t* tin = tours_in + b * (size_t)T;
  int64_t* tout = tours_out + b * (size_t)W;

  // 1. validity: ids in [0, N] and every customer exactly once (nd[c].x counts visits)
  for (int x = tid; x < E; x += nthr) nd[x] = make_int4(0, 0, -1, 0);
  if (tid == 0) s_best[0] = s_best[1] = LS_NONE;
  __syncthreads();
  int bad = 0;
  for (int k = tid; k < T; k += nthr) {
    const int64_t v = tin[k];
    if (v < 0 || v > N) bad = 1;
    else if (v > 0) atomicAdd(&nd[v].x, 1);
  }
  __syncthreads();
  for (int c = 1 + tid; c <= N; c += nthr) bad |= nd[c].x != 1;
  if (__syncthreads_or(bad)) {
    // a row that is not a visit of every customer is copied through (first W entries) and reports -1 moves
    const int m = T < W ? T : W;
    for (int k = tid; k < W; k += nthr) tout[k] = k < m ? tin[k] : 0;
    if (tid == 0) {
      used_len[b] = m;
      if (iterations != nullptr) iterations[b] = -1;
      if (feasible != nullptr) feasible[b] = 0;
    }
    return;
  }

  // 2. split into routes (maximal runs of customers, in input order): warp 0 numbers the runs with a ballot scan while
  // the CTA stages demands and distances
  if (tid < 32) {
    int routes = 0;
    for (int base = 0; base < T; base += 32) {
      const int k = base + lane;
      const int v = k < T ? (int)tin[k] : 0;
      const int pv = (k > 0 && k < T) ? (int)tin[k - 1] : 0;
      const int nv = k + 1 < T ? (int)tin[k + 1] : 0;
      const unsigned starts = __ballot_sync(FULL, v != 0 && pv == 0);
      const int r = routes + __popc(starts & (0xffffffffu >> (31 - lane))) - 1;
      if (v != 0) {
        nd[v].x = pv != 0 ? pv : N + 1 + r;
        nd[v].y = nv != 0 ? nv : 2 * N + 1 + r;
        if (pv == 0) nd[N + 1 + r] = make_int4(0, v, r, 0);
        if (nv == 0) nd[2 * N + 1 + r].x = v;
      }
      routes += __popc(starts);
    }
    if (lane == 0) s_R = routes;
  }
  const float cap = capacity[b];
  const float capl = __fadd_rn(cap, 1e-5f);
  for (int c = tid; c < n; c += nthr) dem[c] = c == 0 ? 0.f : demand[b * (size_t)N + c - 1];
  const float2* xy_g = locs + b * (size_t)n;
  const float* gmat = (SRC == LS_SRC_DIST) ? dist + b * (size_t)n * n : nullptr;
  if (RESIDENT) {
    for (int k = tid; k < n * n; k += nthr) {
      const int r = k / n, c = k - r * n;
      s_x[k] = (SRC == LS_SRC_DIST) ? __ldg(gmat + k) : ls_euclid(__ldg(xy_g + r), __ldg(xy_g + c));
    }
  } else if (SRC == LS_SRC_LOCS) {
    for (int k = tid; k < n; k += nthr) reinterpret_cast<float2*>(s_x)[k] = __ldg(xy_g + k);
  }
  __syncthreads();
  const int R = s_R;
  const LsDist<SRC, RESIDENT, false> D{s_x, gmat, reinterpret_cast<const float2*>(s_x), n};
  auto d = [&](int a, int c) { return D(a <= N ? a : 0, c <= N ? c : 0); };
  // positions, prefix loads and the load of route r, walking from its start depot
  auto walk = [&](int r) {
    float s = 0.f;
    int q = 1, x = nd[N + 1 + r].y;
    pref[N + 1 + r] = 0.f;
    while (x <= N) {
      s = __fadd_rn(s, dem[x]);
      pref[x] = s;
      nd[x].z = r;
      nd[x].w = q++;
      x = nd[x].y;
    }
    nd[x].z = r;
    nd[x].w = q;
    load[r] = s;
  };
  for (int r = tid; r < R; r += nthr) walk(r);
  __syncthreads();

  // (double)delta < -1e-6  <=>  delta <= thr, thr = the largest float below -1e-6 (no fp64 in the sweep)
  float thr = -1e-6f;
  if ((double)thr >= -1e-6) thr = nextafterf(thr, -INFINITY);

  const int M = N + R;  // candidate ids 1..M: customers, then the used start depots
  const int dr = nthr / M, dc = nthr - dr * M;
  int it = 0, sweep = 0;
  while (it < max_iterations) {
    unsigned long long key = LS_NONE;
    for (int i = tid / M, j = tid - (tid / M) * M; i < M;) {
      const int u = i + 1, v = j + 1;
      const int4 U = nd[u], V = nd[v];
      const int pu = U.x, su = U.y, ru = U.z, pv = V.x, sv = V.y, rv = V.z;
      const unsigned long long uv = ((unsigned long long)u << 12) | (unsigned)v;
      // the candidate's key when delta passes the threshold and beats the current best, else LS_NONE
      auto cand = [&](float delta, int kind) {
        if (!(delta <= thr)) return LS_NONE;
        const unsigned long long k64 =
            ((unsigned long long)(~__float_as_uint(delta)) << 32) | ((unsigned long long)kind << 24) | uv;
        return k64 < key ? k64 : LS_NONE;
      };
      if (u <= N && v != u && v != pu) {  // relocate u after v
        const float rem = __fsub_rn(__fsub_rn(d(pu, su), d(pu, u)), d(u, su));
        const float ins = __fsub_rn(__fadd_rn(d(v, u), d(u, sv)), d(v, sv));
        const unsigned long long k = cand(__fadd_rn(rem, ins), CLS_RELOCATE);
        if (k != LS_NONE && (ru == rv ? load[ru] <= capl
                                      : (__fsub_rn(load[ru], dem[u]) <= capl && __fadd_rn(load[rv], dem[u]) <= capl)))
          key = k;
      }
      if (u <= N && v <= N && u < v && su != v && sv != u) {  // swap u and v
        const float a = __fsub_rn(__fsub_rn(__fadd_rn(d(pu, v), d(v, su)), d(pu, u)), d(u, su));
        const float c = __fsub_rn(__fsub_rn(__fadd_rn(d(pv, u), d(u, sv)), d(pv, v)), d(v, sv));
        const unsigned long long k = cand(__fadd_rn(a, c), CLS_SWAP);
        if (k != LS_NONE &&
            (ru == rv ? load[ru] <= capl
                      : (__fadd_rn(__fsub_rn(load[ru], dem[u]), dem[v]) <= capl &&
                         __fadd_rn(__fsub_rn(load[rv], dem[v]), dem[u]) <= capl)))
          key = k;
      }
      if (v <= N && ru == rv && U.w < V.w && su != v) {  // 2-opt: reverse su..v
        const unsigned long long k =
            cand(__fsub_rn(__fsub_rn(__fadd_rn(d(u, v), d(su, sv)), d(u, su)), d(v, sv)), CLS_TWO_OPT);
        if (k != LS_NONE && load[ru] <= capl) key = k;
      }
      if (ru < rv && (u <= N || v <= N) && (su <= 2 * N || sv <= 2 * N)) {  // 2-opt*: exchange the tails
        const unsigned long long k =
            cand(__fsub_rn(__fsub_rn(__fadd_rn(d(u, sv), d(v, su)), d(u, su)), d(v, sv)), CLS_TWO_OPT_STAR);
        if (k != LS_NONE && __fadd_rn(pref[u], __fsub_rn(load[rv], pref[v])) <= capl &&
            __fadd_rn(pref[v], __fsub_rn(load[ru], pref[u])) <= capl)
          key = k;
      }
      i += dr;
      j += dc;
      if (j >= M) {
        j -= M;
        ++i;
      }
    }
    key = warp_min_u64(key);
    unsigned long long* slot = s_best + (sweep & 1);
    if (lane == 0 && key != LS_NONE) atomicMin(slot, key);
    __syncthreads();
    const unsigned long long best = *slot;
    ++sweep;
    // the other slot was last read before the previous sweep's final barrier: reset it for the next sweep
    if (tid == 0) s_best[sweep & 1] = LS_NONE;
    if (best == LS_NONE) break;
    ++it;
    if (tid == 0) {
      const int kind = (int)(best >> 24) & 3, u = (int)(best >> 12) & 0xfff, v = (int)best & 0xfff;
      const int pu = nd[u].x, su = nd[u].y, ru = nd[u].z, pv = nd[v].x, rv = nd[v].z;
      auto link = [&](int a, int c) {
        nd[a].y = c;
        nd[c].x = a;
      };
      if (kind == CLS_RELOCATE) {
        link(pu, su);
        const int sv = nd[v].y;  // read after the removal: v may be su
        link(v, u);
        link(u, sv);
      } else if (kind == CLS_SWAP) {
        const int sv = nd[v].y;
        link(pu, v);
        link(v, su);
        link(pv, u);
        link(u, sv);
      } else if (kind == CLS_TWO_OPT) {
        const int sv = nd[v].y;
        for (int x = su;;) {  // reverse the links of su..v, then hang the segment between u and sv
          const int nx = nd[x].y;
          nd[x].y = nd[x].x;
          nd[x].x = nx;
          if (x == v) break;
          x = nx;
        }
        link(u, v);
        link(su, sv);
      } else {
        const int sv = nd[v].y, endA = 2 * N + 1 + ru, endB = 2 * N + 1 + rv;
        const int lastA = nd[endA].x, lastB = nd[endB].x;
        if (sv != endB) {
          link(u, sv);
          link(lastB, endA);
        } else {
          link(u, endA);
        }
        if (su != endA) {
          link(v, su);
          link(lastA, endB);
        } else {
          link(v, endB);
        }
      }
      s_chg[0] = ru;
      s_chg[1] = rv == ru ? -1 : rv;
    }
    __syncthreads();
    if (tid < 2 && s_chg[tid] >= 0) walk(s_chg[tid]);
    __syncthreads();
  }

  // 3. output: non-empty routes in slot order, one 0 between routes, no leading 0, zero padding.  Thread 0 places the
  // routes and checks the result under the capacity rule of CVRPEnv.check_solution_validity (running load, a depot
  // visit subtracts the capacity and clamps at 0, load <= capacity + 1e-5 after every step).
  if (tid == 0) {
    int o = 0, ok = 1;
    float run = 0.f;
    for (int r = 0; r < R; ++r) {
      off[r] = o;
      const int len = nd[2 * N + 1 + r].w - 1;
      if (len == 0) continue;
      if (o > 0) {
        run = __fsub_rn(run, cap);
        if (run < 0.f) run = 0.f;
        ok &= run <= capl;
      }
      for (int x = nd[N + 1 + r].y; x <= N; x = nd[x].y) {
        run = __fadd_rn(run, dem[x]);
        ok &= run <= capl;
      }
      o += len + 1;
    }
    s_used = o - 1;
    used_len[b] = o - 1;
    if (iterations != nullptr) iterations[b] = it;
    if (feasible != nullptr) feasible[b] = ok;
  }
  __syncthreads();
  const int used = s_used;
  for (int c = 1 + tid; c <= N; c += nthr) tout[off[nd[c].z] + nd[c].w - 1] = c;
  for (int r = tid; r < R; r += nthr) {
    const int e = off[r] + nd[2 * N + 1 + r].w - 1;
    if (e > off[r] && e < used) tout[e] = 0;
  }
  for (int k = used + tid; k < W; k += nthr) tout[k] = 0;
}

template <int SRC, bool RESIDENT>
int launch_cvrp_ls(const float* locs, const float* dist, const float* demand, const float* capacity,
                   const int64_t* tours_in, int64_t* tours_out, int32_t* used_len, int32_t* iterations,
                   int32_t* feasible, int B, int N, int T, int max_iterations, cudaStream_t stream) {
  const size_t smem = cls_layout(N, RESIDENT, SRC).total;
  auto kern = cvrp_ls_kernel<SRC, RESIDENT>;
  static PerDeviceOnce once;  // every variant can pass 48 KB (3N+1 node records of 20 bytes)
  if (!once.flag()) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, device_info().max_smem_optin) !=
        cudaSuccess)
      return check_launch("co_cvrp_local_search (shared-memory attribute)");
    once.flag() = true;
  }
  int threads = 32;
  while (threads < N + 1 && threads < LS_MAX_THREADS) threads *= 2;
  if (N + 1 > 128) threads = LS_MAX_THREADS;
  kern<<<B, threads, smem, stream>>>(reinterpret_cast<const float2*>(locs), dist, demand, capacity, tours_in,
                                     tours_out, used_len, iterations, feasible, N, T, max_iterations);
  return check_launch("co_cvrp_local_search");
}

}  // namespace co

extern "C" int co_cvrp_local_search(const float* locs, const float* dist, const float* demand, const float* capacity,
                                    const int64_t* tours_in, int64_t* tours_out, int32_t* used_len,
                                    int32_t* iterations, int32_t* feasible, int B, int N, int T, int max_iterations,
                                    void* stream) {
  if ((locs == nullptr) == (dist == nullptr))
    return fail(CO_ERR_BAD_ARG, "co_cvrp_local_search: exactly one of locs / dist%s");
  if (!demand || !capacity || !tours_in || !tours_out || !used_len)
    return fail(CO_ERR_BAD_ARG, "co_cvrp_local_search: null pointer%s");
  auto misaligned = [](const void* p, uintptr_t a) { return p != nullptr && ((uintptr_t)p & (a - 1)) != 0; };
  if (misaligned(locs, 8) || misaligned(dist, 4) || misaligned(demand, 4) || misaligned(capacity, 4) ||
      misaligned(tours_in, 8) || misaligned(tours_out, 8) || misaligned(used_len, 4) || misaligned(iterations, 4) ||
      misaligned(feasible, 4))
    return fail(CO_ERR_BAD_ARG, "co_cvrp_local_search: misaligned pointer%s");
  if (B < 0 || N < 1 || T < 1) return fail(CO_ERR_BAD_ARG, "co_cvrp_local_search: bad shape%s N=%lld T=%lld", "", N, T);
  if (N + 1 > CO_TWO_OPT_MAX_NODES)
    return fail(CO_ERR_UNSUPPORTED, "co_cvrp_local_search: N + 1 above the supported maximum%s (N=%lld, max %lld)", "",
                N, CO_TWO_OPT_MAX_NODES);
  if (B == 0) return CO_OK;
  max_iterations = max_iterations < 0 ? 0 : max_iterations;
  const bool resident = N + 1 <= CO_TWO_OPT_RESIDENT_MAX_NODES &&
                        cls_layout(N, true, LS_SRC_LOCS).total <= (size_t)device_info().max_smem_optin;
  cudaStream_t s = (cudaStream_t)stream;
  if (dist != nullptr)
    return resident ? launch_cvrp_ls<LS_SRC_DIST, true>(locs, dist, demand, capacity, tours_in, tours_out, used_len,
                                                        iterations, feasible, B, N, T, max_iterations, s)
                    : launch_cvrp_ls<LS_SRC_DIST, false>(locs, dist, demand, capacity, tours_in, tours_out, used_len,
                                                         iterations, feasible, B, N, T, max_iterations, s);
  return resident ? launch_cvrp_ls<LS_SRC_LOCS, true>(locs, dist, demand, capacity, tours_in, tours_out, used_len,
                                                      iterations, feasible, B, N, T, max_iterations, s)
                  : launch_cvrp_ls<LS_SRC_LOCS, false>(locs, dist, demand, capacity, tours_in, tours_out, used_len,
                                                       iterations, feasible, B, N, T, max_iterations, s);
}
