// co_eas_key_grad: gradient of a weighted sum of trajectory log-likelihoods with respect to the folded pointer logit
// key (block 2 of the rollout cache), for efficient active search with embedding updates (EAS-Emb, Hottung et al.
// 2022; rl4co/models/zoo/eas).  See include/corollout.h for the formula and the argument rules.
//
// Design: one CTA (256 threads = 8 warps) owns one instance and replays its R trajectories one after the other,
// teacher-forced, with the step semantics of the rollout kernel in evaluate mode (rollout_impl.cuh).
//   * warp h = head h.  Lane l owns nodes n = 32 k + l (k < SPL): their head-h glimpse key / value slices live in
//     registers; the folded key Lf (head-major) and the fp32 gradient accumulator (private to the owning thread)
//     live in shared memory, so no entry of dLf is ever written by two threads and no atomics are used.
//   * per step every warp forms its 16 query channels (fixed part + the current-node table row, read from L2 one step
//     ahead because the actions are known; cvrp: + remaining capacity x w_capacity), runs its masked glimpse head,
//     writes the normalised head output o_t[16h..16h+15] and its share of every pointer logit; one block barrier;
//     warp 0 then sums the eight shares in a fixed order, applies tanh clip / mask / temperature, the log-softmax
//     and writes g_{t,n} = coef (delta_{n,a} - p_n) / T * C (1 - tanh^2) / sqrt(E) for the step.
//   * o_t and g_t are buffered for Q steps (two halves, so the other warps run ahead into the next glimpse while warp
//     0 finishes a step); a full half is folded into the accumulator as one rank-Q update, q ascending: the summation
//     order is fixed by (row, step) alone, so the result does not depend on the launch or the batch it is part of.
//   * the environment state (visited set, cvrp load and depot rule) is replicated in every thread as 128-bit masks, so
//     every thread can validate a whole row before it is replayed: a row holding an infeasible action contributes
//     nothing, gets loglik = NaN and is counted in *bad_rows.
#include "rollout_impl.cuh"

namespace co {
namespace {

constexpr int EAS_Q = 8;  // steps per rank-Q update (half of the o / g ring)

template <int SPL>
struct EasSmem {
  static constexpr int NS = 32 * SPL;
  float4 lf[8 * 4 * NS];               // folded key, [head][chunk of 4 channels][node]
  float4 acc[8 * SPL * 4 * 32];        // gradient accumulator, [head][k][chunk][lane]: thread-private entries
  float tile[8][32 * TILE_LD];         // per-warp transpose tile for the value reduction
  alignas(16) float obuf[2 * EAS_Q][E];    // head outputs o_t of the buffered steps
  alignas(16) float gbuf[2 * EAS_Q][NS];   // residuals g_t of the buffered steps (0 for masked / padding nodes)
  alignas(16) float part[2][8][NS];        // per-head share of every pointer logit, double-buffered by step parity
  alignas(16) float qh[8][D];              // per-warp query slice
  float qfix[E];                           // per-row fixed part of the query
  float wcap[E];                           // cvrp: remaining-capacity column of project_context
  float dem[NS];                           // cvrp: demand per node (depot 0)
  unsigned char order[NS];                 // cvrp: customers sorted by demand (ascending)
  unsigned char rank_of[NS];               // cvrp: demand rank of each customer
  short acts[2 * NS];                      // the row's actions (the first 2 NS columns)
};

// Environment state of one trajectory, replicated in every thread (tsp/env.py:60-86, cvrp/env.py:66-136 as
// rollout_impl.cuh replays them).
// word w of a 128-bit mask held as four scalars (selects, not an indexed array, so the masks stay in registers)
__device__ __forceinline__ uint32_t word4(const uint4& m, int w) {
  return w == 0 ? m.x : (w == 1 ? m.y : (w == 2 ? m.z : m.w));
}
__device__ __forceinline__ void set4(uint4& m, int i) {
  const uint32_t bit = 1u << (i & 31), w = (uint32_t)i >> 5;
  m.x |= w == 0 ? bit : 0u; m.y |= w == 1 ? bit : 0u; m.z |= w == 2 ? bit : 0u; m.w |= w == 3 ? bit : 0u;
}
__device__ __forceinline__ uint32_t rank_preset(int nc, int lo) {  // bits >= #customers preset
  return (nc >= lo + 32) ? 0u : (nc <= lo ? 0xffffffffu : (0xffffffffu << (nc - lo)));
}

template <int ENV>
struct EasEnv {
  uint4 vis;    // visited nodes
  uint4 rmask;  // cvrp: visited customers by demand rank
  int cur, t, nvis;
  float used;
  bool depot_seen, anyfeas, done;

  __device__ __forceinline__ void reset(int N) {
    vis = make_uint4(0u, 0u, 0u, 0u);
    rmask = make_uint4(rank_preset(N - 1, 0), rank_preset(N - 1, 32), rank_preset(N - 1, 64), rank_preset(N - 1, 96));
    cur = 0; t = 0; nvis = 0; used = 0.f;
    depot_seen = false; anyfeas = false; done = false;
  }
  __device__ __forceinline__ bool visited(int n) const { return (word4(vis, n >> 5) >> (n & 31)) & 1u; }
  __device__ __forceinline__ bool feasible(int n, const float* dem, float thr) const {
    if (ENV == CO_ENV_TSP) return !visited(n);
    if (n == 0) return !(cur == 0 && anyfeas);
    return !visited(n) && !((dem[n] + used) > thr);
  }
  __device__ __forceinline__ void step(int a, int N, const float* dem, const unsigned char* order,
                                       const unsigned char* rank_of, float thr) {
    if (ENV == CO_ENV_TSP) {
      set4(vis, a);
      cur = a; ++t;
      done = t >= N;
      return;
    }
    used = (used + dem[a == 0 ? 1 : a]) * (a != 0 ? 1.0f : 0.0f);
    nvis += (a != 0 || !depot_seen) ? 1 : 0;
    depot_seen = depot_seen || (a == 0);
    if (a != 0) {
      set4(vis, a);
      set4(rmask, rank_of[a]);
    }
    // depot rule (cvrp/env.py:134): an unvisited customer fits <=> the unvisited customer of least demand fits
    int pmin = 128;
    if (~rmask.w) pmin = 96 + __ffs(~rmask.w) - 1;
    if (~rmask.z) pmin = 64 + __ffs(~rmask.z) - 1;
    if (~rmask.y) pmin = 32 + __ffs(~rmask.y) - 1;
    if (~rmask.x) pmin = __ffs(~rmask.x) - 1;
    anyfeas = (pmin < N - 1) && !((dem[order[pmin < N - 1 ? pmin : 0]] + used) > thr);
    cur = a; ++t;
    done = nvis >= N;
  }
};

template <int SPL, int ENV>
__global__ void __launch_bounds__(256, 1) eas_key_grad_kernel(const co_eas_grad_args A) {
  constexpr int NS = 32 * SPL;
  constexpr int CW = (ENV == CO_ENV_TSP ? 5 : 4) * E;  // tsp: the 5E layout with the first-node table
  constexpr int CUR_BLK = CW / E - 1;
  constexpr bool VRP = ENV == CO_ENV_CVRP;
  constexpr float LOG2E = 1.4426950408889634f, INV_SQRT_E = 0.08838834764831845f;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  EasSmem<SPL>& sm = *reinterpret_cast<EasSmem<SPL>*>(smem_raw);

  const int tid = threadIdx.x, lane = tid & 31, h = tid >> 5;
  const int N = A.N, B_inst = A.B_inst, R = A.num_rows, T = A.T;
  const int TB = T < 2 * NS ? T : 2 * NS;  // columns read: a feasible episode ends within 2 (N - 1) steps
  const float clip = A.tanh_clipping, inv_temp = 1.0f / A.temperature;
  const float gscale = clip * inv_temp * INV_SQRT_E;
  float* tile = sm.tile[h];

  float2 Kr[SPL][8], Vr[SPL][8];
  int ps = 0;  // global step parity (part[] buffer)

  for (int b = blockIdx.x; b < B_inst; b += gridDim.x) {
    __syncthreads();  // the previous instance is done with shared memory
    const float* crow = A.cache + (size_t)b * N * CW;
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
      const int n = 32 * k + lane;
      if (n < N) {
        const float4* ks = reinterpret_cast<const float4*>(crow + (size_t)n * CW + 0 * E + h * D);
        const float4* vs = reinterpret_cast<const float4*>(crow + (size_t)n * CW + 1 * E + h * D);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float4 kv = __ldg(ks + c), vv = __ldg(vs + c);
          Kr[k][2 * c] = make_float2(kv.x, kv.y); Kr[k][2 * c + 1] = make_float2(kv.z, kv.w);
          Vr[k][2 * c] = make_float2(vv.x, vv.y); Vr[k][2 * c + 1] = make_float2(vv.z, vv.w);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) { Kr[k][j] = make_float2(0.f, 0.f); Vr[k][j] = make_float2(0.f, 0.f); }
      }
    }
    for (int i = tid; i < 8 * 4 * NS; i += 256) {  // folded key, head-major; zero rows for padding nodes
      const int n = i % NS, hc = i / NS;
      sm.lf[i] = n < N ? __ldg(reinterpret_cast<const float4*>(crow + (size_t)n * CW + 2 * E) + hc)
                       : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int i = tid; i < 8 * SPL * 4 * 32; i += 256) sm.acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (tid < E) sm.wcap[tid] = VRP ? A.w_capacity[tid] : 0.f;
    if (tid < NS) sm.dem[tid] = (VRP && tid >= 1 && tid < N) ? A.demand[(size_t)b * (N - 1) + tid - 1] : 0.f;
    const float cap = (VRP && A.vehicle_capacity) ? A.vehicle_capacity[b] : 1.0f;
    const float thr = cap + 1e-5f;  // fp32 add, as `td["vehicle_capacity"] + 1e-5`
    __syncthreads();
    if (VRP) {  // rank-sort customers by demand (ties by index), as rollout_impl.cuh
      if (tid >= 1 && tid < N) {
        const float d = sm.dem[tid];
        int rank = 0;
        for (int m = 1; m < N; ++m) {
          const float dm = sm.dem[m];
          rank += (dm < d || (dm == d && m < tid)) ? 1 : 0;
        }
        sm.order[rank] = (unsigned char)tid;
        sm.rank_of[tid] = (unsigned char)rank;
      }
    }

    int hb = 0, cnt = 0;  // ring half being filled, steps buffered in it
    // rank-cnt update of this thread's accumulator entries from ring half `half`
    auto flush = [&](int half, int nq) {
#pragma unroll
      for (int k = 0; k < SPL; ++k) {
        float4* ap = sm.acc + ((h * SPL + k) * 4) * 32 + lane;
        float4 a0 = ap[0], a1 = ap[32], a2 = ap[64], a3 = ap[96];
        for (int q = 0; q < nq; ++q) {
          const int sl = half * EAS_Q + q;
          const float g = sm.gbuf[sl][32 * k + lane];
          const float4* o = reinterpret_cast<const float4*>(sm.obuf[sl] + h * D);
          const float4 o0 = o[0], o1 = o[1], o2 = o[2], o3 = o[3];
          a0.x = fmaf(g, o0.x, a0.x); a0.y = fmaf(g, o0.y, a0.y); a0.z = fmaf(g, o0.z, a0.z); a0.w = fmaf(g, o0.w, a0.w);
          a1.x = fmaf(g, o1.x, a1.x); a1.y = fmaf(g, o1.y, a1.y); a1.z = fmaf(g, o1.z, a1.z); a1.w = fmaf(g, o1.w, a1.w);
          a2.x = fmaf(g, o2.x, a2.x); a2.y = fmaf(g, o2.y, a2.y); a2.z = fmaf(g, o2.z, a2.z); a2.w = fmaf(g, o2.w, a2.w);
          a3.x = fmaf(g, o3.x, a3.x); a3.y = fmaf(g, o3.y, a3.y); a3.z = fmaf(g, o3.z, a3.z); a3.w = fmaf(g, o3.w, a3.w);
        }
        ap[0] = a0; ap[32] = a1; ap[64] = a2; ap[96] = a3;
      }
    };

    for (int r = 0; r < R; ++r) {
      const size_t row = (size_t)r * B_inst + b;  // start-major, as co_rollout
      __syncthreads();  // every thread is done with the previous row's actions
      for (int c = tid; c < TB; c += 256) {
        const int64_t a = A.actions[row * T + c];
        sm.acts[c] = (short)((a < 0 || a >= N) ? -1 : a);
      }
      __syncthreads();
      const float coef = A.coef[row];

      // ---- validation: every thread replays the row's mask (uniform result, no communication)
      EasEnv<ENV> env;
      env.reset(N);
      bool bad = sm.acts[0] < (VRP ? 1 : 0);  // column 0: the forced start (cvrp: a customer)
      if (!bad) {
        env.step(sm.acts[0], N, sm.dem, sm.order, sm.rank_of, thr);
        while (!env.done) {
          if (env.t >= TB) { bad = true; break; }
          const int a = sm.acts[env.t];
          if (a < 0 || !env.feasible(a, sm.dem, thr)) { bad = true; break; }
          env.step(a, N, sm.dem, sm.order, sm.rank_of, thr);
        }
      }
      if (bad) {
        if (tid == 0) {
          A.loglik[row] = __int_as_float(0x7fc00000);
          if (A.bad_rows) atomicAdd(A.bad_rows, 1);
        }
        continue;
      }

      // ---- replay
      env.reset(N);
      const int a0 = sm.acts[0];
      env.step(a0, N, sm.dem, sm.order, sm.rank_of, thr);
      if (tid < E) {  // fixed part of the query: graph context (+ tsp: the first-node table row, context.py:129-133)
        float g = A.graph_ctx ? A.graph_ctx[(size_t)b * E + tid] : 0.f;
        if (ENV == CO_ENV_TSP) g += __ldg(crow + (size_t)a0 * CW + 3 * E + tid);
        sm.qfix[tid] = g;
      }
      __syncthreads();
      float ll = 0.f;  // lane 0 of warp 0
      float pt = lane < D ? __ldg(crow + (size_t)env.cur * CW + CUR_BLK * E + h * D + lane) : 0.f;
      while (!env.done) {
        const int a = sm.acts[env.t];
        const int sl = hb * EAS_Q + cnt;
        float* part = sm.part[ps][h];
        // next step's current-node table row (the action of this step), in flight during this step
        const float pt_next = lane < D ? __ldg(crow + (size_t)a * CW + CUR_BLK * E + h * D + lane) : 0.f;
        // ---------------- glimpse head h, head output, share of head h in every pointer logit
        {
          if (lane < D) {
            float q = sm.qfix[h * D + lane] + pt;
            if (VRP) q = fmaf(cap - env.used, sm.wcap[h * D + lane], q);  // context.py:147-149
            sm.qh[h][lane] = q;
          }
          __syncwarp();
          const float4* qp = reinterpret_cast<const float4*>(sm.qh[h]);
          float2 sc2[SPL];
#pragma unroll
          for (int k = 0; k < SPL; ++k) sc2[k] = make_float2(0.f, 0.f);
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float4 x = qp[c];
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
              sc2[k] = ffma2(make_float2(x.x, x.y), Kr[k][2 * c], sc2[k]);
              sc2[k] = ffma2(make_float2(x.z, x.w), Kr[k][2 * c + 1], sc2[k]);
            }
          }
          float sc[SPL], m = -INFINITY;
          bool fz[SPL];
#pragma unroll
          for (int k = 0; k < SPL; ++k) {
            const int n = 32 * k + lane;
            fz[k] = n < N && env.feasible(n, sm.dem, thr);
            sc[k] = fz[k] ? (sc2[k].x + sc2[k].y) * (0.25f * LOG2E) : -INFINITY;
            m = fmaxf(m, sc[k]);
          }
          m = funkey(__reduce_max_sync(FULL, fkey(m)));
          float2 acc[8];
          float esum = 0.f;
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] = make_float2(0.f, 0.f);
#pragma unroll
          for (int k = 0; k < SPL; ++k) {
            const float e = fz[k] ? ex2(sc[k] - m) : 0.f;
            esum += e;
            const float2 e2 = make_float2(e, e);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = ffma2(e2, Vr[k][j], acc[j]);
          }
          float4* trow = reinterpret_cast<float4*>(tile + lane * TILE_LD);
#pragma unroll
          for (int c = 0; c < 4; ++c) trow[c] = make_float4(acc[2 * c].x, acc[2 * c].y, acc[2 * c + 1].x, acc[2 * c + 1].y);
          esum = warp_sum_fixed(esum);
          __syncwarp();
          const int d = lane & 15, half = lane >> 4;
          float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
          for (int rr = 0; rr < 16; rr += 4) {
            s0 += tile[(16 * half + ((rr + 0 + 4 * half) & 15)) * TILE_LD + d];
            s1 += tile[(16 * half + ((rr + 1 + 4 * half) & 15)) * TILE_LD + d];
            s2 += tile[(16 * half + ((rr + 2 + 4 * half) & 15)) * TILE_LD + d];
            s3 += tile[(16 * half + ((rr + 3 + 4 * half) & 15)) * TILE_LD + d];
          }
          float o = (s0 + s1) + (s2 + s3);
          o += __shfl_xor_sync(FULL, o, 16);
          if (lane < 16) sm.obuf[sl][h * D + lane] = o / esum;
          __syncwarp();
          const float4* op = reinterpret_cast<const float4*>(sm.obuf[sl] + h * D);
          const float4 o0 = op[0], o1 = op[1], o2 = op[2], o3 = op[3];
#pragma unroll
          for (int k = 0; k < SPL; ++k) {
            const float4* lp = sm.lf + (h * 4) * NS + 32 * k + lane;
            const float4 l0 = lp[0], l1 = lp[NS], l2 = lp[2 * NS], l3 = lp[3 * NS];
            float2 p2 = make_float2(0.f, 0.f);
            p2 = ffma2(make_float2(o0.x, o0.y), make_float2(l0.x, l0.y), p2);
            p2 = ffma2(make_float2(o0.z, o0.w), make_float2(l0.z, l0.w), p2);
            p2 = ffma2(make_float2(o1.x, o1.y), make_float2(l1.x, l1.y), p2);
            p2 = ffma2(make_float2(o1.z, o1.w), make_float2(l1.z, l1.w), p2);
            p2 = ffma2(make_float2(o2.x, o2.y), make_float2(l2.x, l2.y), p2);
            p2 = ffma2(make_float2(o2.z, o2.w), make_float2(l2.z, l2.w), p2);
            p2 = ffma2(make_float2(o3.x, o3.y), make_float2(l3.x, l3.y), p2);
            p2 = ffma2(make_float2(o3.z, o3.w), make_float2(l3.z, l3.w), p2);
            part[32 * k + lane] = p2.x + p2.y;
          }
        }
        __syncthreads();  // every head's share of every logit is in shared memory

        if (h == 0) {
          // ---------------- pointer logits, heads summed in fixed order; tanh clip, mask, temperature, log-softmax
          const float(*pp)[NS] = sm.part[ps];
          float z[SPL], th[SPL], m = -INFINITY;
          bool fz[SPL];
#pragma unroll
          for (int k = 0; k < SPL; ++k) {
            const int n = 32 * k + lane;
            const float u = ((pp[0][n] + pp[1][n]) + (pp[2][n] + pp[3][n])) + ((pp[4][n] + pp[5][n]) + (pp[6][n] + pp[7][n]));
            fz[k] = n < N && env.feasible(n, sm.dem, thr);
            th[k] = tanhf(u * INV_SQRT_E);
            z[k] = fz[k] ? th[k] * clip * inv_temp : -INFINITY;
            m = fmaxf(m, z[k]);
          }
          m = funkey(__reduce_max_sync(FULL, fkey(m)));
          float e[SPL], s = 0.f;
#pragma unroll
          for (int k = 0; k < SPL; ++k) {
            e[k] = fz[k] ? __expf(z[k] - m) : 0.f;
            s += e[k];
          }
          s = warp_sum_fixed(s);  // 1 <= s <= N; order independent
          const float inv_s = 1.0f / s;
          float za = 0.f;
#pragma unroll
          for (int k = 0; k < SPL; ++k) {
            const int n = 32 * k + lane;
            za = (n == a) ? z[k] : za;
            const float g = fz[k] ? coef * (((n == a) ? 1.0f : 0.0f) - e[k] * inv_s) * gscale * (1.0f - th[k] * th[k]) : 0.f;
            sm.gbuf[sl][n] = g;
          }
          za = __shfl_sync(FULL, za, a & 31);
          if (lane == 0) {
            const float lp = (za - m) - logf(s);
            ll += lp;
          }
        }
        // ---------------- environment step (replicated)
        env.step(a, N, sm.dem, sm.order, sm.rank_of, thr);
        pt = pt_next;
        ps ^= 1;
        if (++cnt == EAS_Q || env.done) {
          __syncthreads();  // warp 0's residuals of the last step are in shared memory
          flush(hb, cnt);
          hb ^= 1;
          cnt = 0;
        }
      }
      if (tid == 0) A.loglik[row] = ll;
    }

    // ---- dLf rows of this instance (thread-private accumulator entries)
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
      const int n = 32 * k + lane;
      if (n < N) {
        const float4* ap = sm.acc + ((h * SPL + k) * 4) * 32 + lane;
        float4* dst = reinterpret_cast<float4*>(A.dLf + ((size_t)b * N + n) * E + h * D);
#pragma unroll
        for (int c = 0; c < 4; ++c) dst[c] = ap[32 * c];
      }
    }
  }
}

template <int SPL, int ENV>
int launch_eas(const co_eas_grad_args& A, cudaStream_t st) {
  auto kern = eas_key_grad_kernel<SPL, ENV>;
  const size_t smem = sizeof(EasSmem<SPL>);
  static PerDeviceOnce once;
  static int ctas_per_sm = 1;
  bool& configured = once.flag();
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail(CO_ERR_CUDA, "co_eas_key_grad: smem attribute: %s", cudaGetErrorString(e));
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, kern, 256, smem);
    if (e != cudaSuccess || ctas_per_sm < 1) return fail(CO_ERR_CUDA, "co_eas_key_grad: occupancy query failed%s");
    configured = true;
  }
  int grid = device_info().sm_count * ctas_per_sm;
  if (grid > A.B_inst) grid = A.B_inst;
  kern<<<grid, 256, smem, st>>>(A);
  return check_launch("co_eas_key_grad");
}

template <int ENV>
int dispatch_eas(const co_eas_grad_args& A, cudaStream_t st) {
  if (A.N <= 32) return launch_eas<1, ENV>(A, st);
  if (A.N <= 64) return launch_eas<2, ENV>(A, st);
  return launch_eas<4, ENV>(A, st);
}


// ================================================================================================ EAS-Lay
// co_eas_layer_grad: gradient of sum_j coef[j] loglik[j] with respect to the per-instance residual layer
// o' = o + relu(o W1 + b1) W2 + b2 on the head output (EAS-Lay).  In a teacher-forced replay the head output o_t of a
// step depends on the actions only, not on the layer, so the steps of an instance are independent once the glimpse has
// run.  One CTA (256 threads) owns one instance and walks its rows in chunks of LMC steps:
//   P1  glimpse of LMC steps (warp h = head h, as eas_key_grad_kernel; no block barrier except at row starts) ->
//       o [LMC, E], the feasible set, the action and the row of every step;
//   P2  z = relu(o W1 + b1);   P3  o' = o + (z W2 + b2);           (thread: one column, 32 rows; W from L1 / L2)
//   P4  per step (warp w: steps w, w + 8, ...): u_n = o' . Lf[n], tanh clip / mask / temperature / log-softmax,
//       g_n as co_eas_key_grad, do' = sum_n g_n Lf[n] (in place of o');
//   P5  dW2 += z^T do', db2 += do';   P6  dz = (do' W2^T) * [z > 0] (in place of z);   P7  dW1 += o^T dz, db1 += dz.
// The accumulators are the output rows of the instance in global memory, every entry read, updated over the chunk's
// steps in order and written back by the one thread that owns it: the summation order is (row, step) alone.
constexpr int LMC = 64;      // replayed steps per chunk
constexpr int LLD = E + 4;   // padded row (floats) of the node-major key and the chunk buffers: conflict-free LDS.128

template <int SPL>
struct EasLaySmem {
  static constexpr int NS = 32 * SPL;
  alignas(16) float lf[NS][LLD];          // folded key, node-major; zero rows for padding nodes
  alignas(16) float o[LMC][LLD];          // head outputs of the chunk's steps
  alignas(16) float z[LMC][LLD];          // relu(o W1 + b1), then dz
  alignas(16) float op[LMC][LLD];         // o', then do'
  float tile[8][32 * TILE_LD];            // per-warp transpose tile for the value reduction
  alignas(16) float gw[8][NS];            // per-warp residuals g of the step it is on
  alignas(16) float qh[8][D];             // per-warp query slice
  float qfix[E];                          // per-row fixed part of the query
  float wcap[E];                          // cvrp: remaining-capacity column of project_context
  float dem[NS];                          // cvrp: demand per node (depot 0)
  uint32_t fmask[LMC][4];                 // feasible nodes of each step (bit n % 32 of word n / 32)
  float lp[LMC];                          // log-prob of each step's action
  int srow[LMC];                          // row of each step; -1 - row on the row's last step
  short sact[LMC];                        // action of each step
  unsigned char order[NS];                // cvrp: customers sorted by demand (ascending)
  unsigned char rank_of[NS];              // cvrp: demand rank of each customer
  short acts[2 * NS];                     // the row's actions (the first 2 NS columns)
};

// acc[j] = sum_k X[2 j + hf][k] W(k, col), k ascending; W(k, col) = W[k E + col], or W[col E + k] when TRANS
template <bool TRANS>
__device__ __forceinline__ void chunk_gemm(const float (*X)[LLD], const float* __restrict__ W, int col, int hf,
                                           float (&acc)[LMC / 2]) {
#pragma unroll
  for (int j = 0; j < LMC / 2; ++j) acc[j] = 0.f;
#pragma unroll 1
  for (int k = 0; k < E; k += 4) {
    float4 w;
    if (TRANS) {
      w = __ldg(reinterpret_cast<const float4*>(W + (size_t)col * E + k));
    } else {
      w = make_float4(__ldg(W + (k + 0) * E + col), __ldg(W + (k + 1) * E + col), __ldg(W + (k + 2) * E + col),
                      __ldg(W + (k + 3) * E + col));
    }
#pragma unroll
    for (int j = 0; j < LMC / 2; ++j) {
      const float4 x = *reinterpret_cast<const float4*>(&X[2 * j + hf][k]);
      acc[j] = fmaf(x.x, w.x, acc[j]);
      acc[j] = fmaf(x.y, w.y, acc[j]);
      acc[j] = fmaf(x.z, w.z, acc[j]);
      acc[j] = fmaf(x.w, w.w, acc[j]);
    }
  }
}

// dW[i][c] += sum_{m < mc} X[m][i] Y[m][c], db[c] += sum_{m < mc} Y[m][c] (m ascending); thread: c = 4q .. 4q + 3,
// i = 16 ig .. 16 ig + 15 (warp 0 also owns db)
__device__ __forceinline__ void chunk_contract(const float (*X)[LLD], const float (*Y)[LLD], int mc, float* dW,
                                               float* db, int q, int ig) {
  float4 acc[16];
#pragma unroll
  for (int ii = 0; ii < 16; ++ii) acc[ii] = *reinterpret_cast<const float4*>(dW + (16 * ig + ii) * E + 4 * q);
  float4 bacc = ig == 0 ? *reinterpret_cast<const float4*>(db + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
  for (int m = 0; m < mc; ++m) {
    const float4 y = *reinterpret_cast<const float4*>(&Y[m][4 * q]);
    const float4* xr = reinterpret_cast<const float4*>(&X[m][16 * ig]);
#pragma unroll
    for (int c4 = 0; c4 < 4; ++c4) {
      const float4 x = xr[c4];
      const float xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        float4& a = acc[4 * c4 + u];
        a.x = fmaf(xs[u], y.x, a.x); a.y = fmaf(xs[u], y.y, a.y); a.z = fmaf(xs[u], y.z, a.z); a.w = fmaf(xs[u], y.w, a.w);
      }
    }
    bacc.x += y.x; bacc.y += y.y; bacc.z += y.z; bacc.w += y.w;
  }
#pragma unroll
  for (int ii = 0; ii < 16; ++ii) *reinterpret_cast<float4*>(dW + (16 * ig + ii) * E + 4 * q) = acc[ii];
  if (ig == 0) *reinterpret_cast<float4*>(db + 4 * q) = bacc;
}

template <int SPL, int ENV>
__global__ void __launch_bounds__(256, 1) eas_layer_grad_kernel(const co_eas_layer_grad_args A) {
  constexpr int NS = 32 * SPL;
  constexpr int CW = (ENV == CO_ENV_TSP ? 5 : 4) * E;
  constexpr int CUR_BLK = CW / E - 1;
  constexpr bool VRP = ENV == CO_ENV_CVRP;
  constexpr float LOG2E = 1.4426950408889634f, INV_SQRT_E = 0.08838834764831845f;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  EasLaySmem<SPL>& sm = *reinterpret_cast<EasLaySmem<SPL>*>(smem_raw);

  const int tid = threadIdx.x, lane = tid & 31, h = tid >> 5;
  const int N = A.N, B_inst = A.B_inst, R = A.num_rows, T = A.T;
  const int TB = T < 2 * NS ? T : 2 * NS;
  const float clip = A.tanh_clipping, inv_temp = 1.0f / A.temperature;
  const float gscale = clip * inv_temp * INV_SQRT_E;
  float* tile = sm.tile[h];
  const int col = 16 * h + (lane & 15), hf = lane >> 4;  // GEMM mapping (P2, P3, P6)
  const int cq = tid & 31, cig = tid >> 5;                // contraction mapping (P5, P7)

  float2 Kr[SPL][8], Vr[SPL][8];

  for (int b = blockIdx.x; b < B_inst; b += gridDim.x) {
    __syncthreads();  // the previous instance is done with shared memory
    const float* crow = A.cache + (size_t)b * N * CW;
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
      const int n = 32 * k + lane;
      if (n < N) {
        const float4* ks = reinterpret_cast<const float4*>(crow + (size_t)n * CW + 0 * E + h * D);
        const float4* vs = reinterpret_cast<const float4*>(crow + (size_t)n * CW + 1 * E + h * D);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float4 kv = __ldg(ks + c), vv = __ldg(vs + c);
          Kr[k][2 * c] = make_float2(kv.x, kv.y); Kr[k][2 * c + 1] = make_float2(kv.z, kv.w);
          Vr[k][2 * c] = make_float2(vv.x, vv.y); Vr[k][2 * c + 1] = make_float2(vv.z, vv.w);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) { Kr[k][j] = make_float2(0.f, 0.f); Vr[k][j] = make_float2(0.f, 0.f); }
      }
    }
    for (int i = tid; i < NS * (E / 4); i += 256) {
      const int n = i >> 5, c4 = i & 31;
      *reinterpret_cast<float4*>(&sm.lf[n][4 * c4]) =
          n < N ? __ldg(reinterpret_cast<const float4*>(crow + (size_t)n * CW + 2 * E) + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (tid < E) sm.wcap[tid] = VRP ? A.w_capacity[tid] : 0.f;
    if (tid < NS) sm.dem[tid] = (VRP && tid >= 1 && tid < N) ? A.demand[(size_t)b * (N - 1) + tid - 1] : 0.f;
    const float cap = (VRP && A.vehicle_capacity) ? A.vehicle_capacity[b] : 1.0f;
    const float thr = cap + 1e-5f;
    const float* W1 = A.layer + (size_t)b * CO_EAS_LAYER_FLOATS;
    const float* B1 = W1 + E * E;
    const float* W2 = B1 + E;
    const float* B2 = W2 + E * E;
    float* dW1 = A.dlayer + (size_t)b * CO_EAS_LAYER_FLOATS;
    float* dB1 = dW1 + E * E;
    float* dW2 = dB1 + E;
    float* dB2 = dW2 + E * E;
    // this thread's accumulator entries start at zero (only this thread ever touches them)
#pragma unroll
    for (int ii = 0; ii < 16; ++ii) {
      *reinterpret_cast<float4*>(dW1 + (16 * cig + ii) * E + 4 * cq) = make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(dW2 + (16 * cig + ii) * E + 4 * cq) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (cig == 0) {
      *reinterpret_cast<float4*>(dB1 + 4 * cq) = make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(dB2 + 4 * cq) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
    if (VRP) {  // rank-sort customers by demand (ties by index), as rollout_impl.cuh
      if (tid >= 1 && tid < N) {
        const float d = sm.dem[tid];
        int rank = 0;
        for (int m = 1; m < N; ++m) {
          const float dm = sm.dem[m];
          rank += (dm < d || (dm == d && m < tid)) ? 1 : 0;
        }
        sm.order[rank] = (unsigned char)tid;
        sm.rank_of[tid] = (unsigned char)rank;
      }
    }

    EasEnv<ENV> env;
    env.reset(N);
    bool in_row = false;
    int r = 0;
    float pt = 0.f, ll = 0.f;  // ll: thread 0
    while (true) {
      // ---------------- P1: glimpse of up to LMC steps
      int mc = 0;
      while (mc < LMC) {
        if (!in_row) {  // uniform: the environment state is replicated
          if (r >= R) break;
          const size_t row = (size_t)r * B_inst + b;
          __syncthreads();  // every thread is done with the previous row's actions (and the rank sort is visible)
          for (int c = tid; c < TB; c += 256) {
            const int64_t a = A.actions[row * T + c];
            sm.acts[c] = (short)((a < 0 || a >= N) ? -1 : a);
          }
          __syncthreads();
          env.reset(N);
          bool bad = sm.acts[0] < (VRP ? 1 : 0);
          if (!bad) {
            env.step(sm.acts[0], N, sm.dem, sm.order, sm.rank_of, thr);
            while (!env.done) {
              if (env.t >= TB) { bad = true; break; }
              const int a = sm.acts[env.t];
              if (a < 0 || !env.feasible(a, sm.dem, thr)) { bad = true; break; }
              env.step(a, N, sm.dem, sm.order, sm.rank_of, thr);
            }
          }
          ++r;
          if (bad) {
            if (tid == 0) {
              A.loglik[row] = __int_as_float(0x7fc00000);
              if (A.bad_rows) atomicAdd(A.bad_rows, 1);
            }
            continue;
          }
          env.reset(N);
          const int a0 = sm.acts[0];
          env.step(a0, N, sm.dem, sm.order, sm.rank_of, thr);
          if (tid < E) {
            float g = A.graph_ctx ? A.graph_ctx[(size_t)b * E + tid] : 0.f;
            if (ENV == CO_ENV_TSP) g += __ldg(crow + (size_t)a0 * CW + 3 * E + tid);
            sm.qfix[tid] = g;
          }
          __syncthreads();
          pt = lane < D ? __ldg(crow + (size_t)env.cur * CW + CUR_BLK * E + h * D + lane) : 0.f;
          in_row = true;
        }
        const int a = sm.acts[env.t];
        const float pt_next = lane < D ? __ldg(crow + (size_t)a * CW + CUR_BLK * E + h * D + lane) : 0.f;
        {
          if (lane < D) {
            float q = sm.qfix[h * D + lane] + pt;
            if (VRP) q = fmaf(cap - env.used, sm.wcap[h * D + lane], q);
            sm.qh[h][lane] = q;
          }
          __syncwarp();
          const float4* qp = reinterpret_cast<const float4*>(sm.qh[h]);
          float2 sc2[SPL];
#pragma unroll
          for (int k = 0; k < SPL; ++k) sc2[k] = make_float2(0.f, 0.f);
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float4 x = qp[c];
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
              sc2[k] = ffma2(make_float2(x.x, x.y), Kr[k][2 * c], sc2[k]);
              sc2[k] = ffma2(make_float2(x.z, x.w), Kr[k][2 * c + 1], sc2[k]);
            }
          }
          float sc[SPL], m = -INFINITY;
          bool fz[SPL];
#pragma unroll
          for (int k = 0; k < SPL; ++k) {
            const int n = 32 * k + lane;
            fz[k] = n < N && env.feasible(n, sm.dem, thr);
            sc[k] = fz[k] ? (sc2[k].x + sc2[k].y) * (0.25f * LOG2E) : -INFINITY;
            m = fmaxf(m, sc[k]);
          }
          if (h == 0) {  // the feasible set of the step, for the pointer phase
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const uint32_t bits = k < SPL ? __ballot_sync(FULL, fz[k < SPL ? k : 0]) : 0u;
              if (lane == 0) sm.fmask[mc][k] = bits;
            }
          }
          m = funkey(__reduce_max_sync(FULL, fkey(m)));
          float2 acc[8];
          float esum = 0.f;
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] = make_float2(0.f, 0.f);
#pragma unroll
          for (int k = 0; k < SPL; ++k) {
            const float e = fz[k] ? ex2(sc[k] - m) : 0.f;
            esum += e;
            const float2 e2 = make_float2(e, e);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = ffma2(e2, Vr[k][j], acc[j]);
          }
          float4* trow = reinterpret_cast<float4*>(tile + lane * TILE_LD);
#pragma unroll
          for (int c = 0; c < 4; ++c) trow[c] = make_float4(acc[2 * c].x, acc[2 * c].y, acc[2 * c + 1].x, acc[2 * c + 1].y);
          esum = warp_sum_fixed(esum);
          __syncwarp();
          const int d = lane & 15, half = lane >> 4;
          float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
          for (int rr = 0; rr < 16; rr += 4) {
            s0 += tile[(16 * half + ((rr + 0 + 4 * half) & 15)) * TILE_LD + d];
            s1 += tile[(16 * half + ((rr + 1 + 4 * half) & 15)) * TILE_LD + d];
            s2 += tile[(16 * half + ((rr + 2 + 4 * half) & 15)) * TILE_LD + d];
            s3 += tile[(16 * half + ((rr + 3 + 4 * half) & 15)) * TILE_LD + d];
          }
          float o = (s0 + s1) + (s2 + s3);
          o += __shfl_xor_sync(FULL, o, 16);
          if (lane < 16) sm.o[mc][h * D + lane] = o / esum;
          __syncwarp();  // the tile and qh are reused by the next step
        }
        env.step(a, N, sm.dem, sm.order, sm.rank_of, thr);
        if (tid == 0) {
          sm.sact[mc] = (short)a;
          sm.srow[mc] = env.done ? -r : r - 1;  // r was advanced at the row start: -1 - (r - 1) = -r
        }
        pt = pt_next;
        if (env.done) in_row = false;
        ++mc;
      }
      if (mc == 0) break;  // uniform: every row has been replayed
      __syncthreads();     // P1 complete

      float acc[LMC / 2];
      // ---------------- P2: z = relu(o W1 + b1)
      chunk_gemm<false>(sm.o, W1, col, hf, acc);
      {
        const float b1 = __ldg(B1 + col);
#pragma unroll
        for (int j = 0; j < LMC / 2; ++j) {
          const float a = acc[j] + b1;
          sm.z[2 * j + hf][col] = a > 0.f ? a : 0.f;
        }
      }
      __syncthreads();
      // ---------------- P3: o' = o + (z W2 + b2)
      chunk_gemm<false>(sm.z, W2, col, hf, acc);
      {
        const float b2 = __ldg(B2 + col);
#pragma unroll
        for (int j = 0; j < LMC / 2; ++j) sm.op[2 * j + hf][col] = sm.o[2 * j + hf][col] + (acc[j] + b2);
      }
      __syncthreads();
      // ---------------- P4: pointer logits, log-softmax, residuals g and do' = sum_n g_n Lf[n] per step
      for (int m = h; m < mc; m += 8) {
        float u[SPL];
#pragma unroll
        for (int k = 0; k < SPL; ++k) u[k] = 0.f;
        const float4* orow = reinterpret_cast<const float4*>(sm.op[m]);
#pragma unroll 2
        for (int c4 = 0; c4 < E / 4; ++c4) {
          const float4 x = orow[c4];
#pragma unroll
          for (int k = 0; k < SPL; ++k) {
            const float4 l = *reinterpret_cast<const float4*>(&sm.lf[32 * k + lane][4 * c4]);
            u[k] = fmaf(x.x, l.x, u[k]); u[k] = fmaf(x.y, l.y, u[k]); u[k] = fmaf(x.z, l.z, u[k]); u[k] = fmaf(x.w, l.w, u[k]);
          }
        }
        const int a = sm.sact[m], rr = sm.srow[m];
        const float coef = A.coef[(size_t)(rr < 0 ? -1 - rr : rr) * B_inst + b];
        float zl[SPL], th[SPL], mx = -INFINITY;
        bool fz[SPL];
#pragma unroll
        for (int k = 0; k < SPL; ++k) {
          const int n = 32 * k + lane;
          fz[k] = n < N && ((sm.fmask[m][k] >> lane) & 1u);
          th[k] = tanhf(u[k] * INV_SQRT_E);
          zl[k] = fz[k] ? th[k] * clip * inv_temp : -INFINITY;
          mx = fmaxf(mx, zl[k]);
        }
        mx = funkey(__reduce_max_sync(FULL, fkey(mx)));
        float e[SPL], s = 0.f;
#pragma unroll
        for (int k = 0; k < SPL; ++k) {
          e[k] = fz[k] ? __expf(zl[k] - mx) : 0.f;
          s += e[k];
        }
        s = warp_sum_fixed(s);
        const float inv_s = 1.0f / s;
        float za = 0.f;
#pragma unroll
        for (int k = 0; k < SPL; ++k) {
          const int n = 32 * k + lane;
          za = (n == a) ? zl[k] : za;
          sm.gw[h][n] = fz[k] ? coef * (((n == a) ? 1.0f : 0.0f) - e[k] * inv_s) * gscale * (1.0f - th[k] * th[k]) : 0.f;
        }
        za = __shfl_sync(FULL, za, a & 31);
        if (lane == 0) sm.lp[m] = (za - mx) - logf(s);
        __syncwarp();  // g complete; every lane is done reading o'[m]
        float4 dop = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
        for (int n = 0; n < N; ++n) {
          const float g = sm.gw[h][n];
          const float4 l = *reinterpret_cast<const float4*>(&sm.lf[n][4 * lane]);
          dop.x = fmaf(g, l.x, dop.x); dop.y = fmaf(g, l.y, dop.y); dop.z = fmaf(g, l.z, dop.z); dop.w = fmaf(g, l.w, dop.w);
        }
        *reinterpret_cast<float4*>(&sm.op[m][4 * lane]) = dop;
        __syncwarp();  // gw is reused by the warp's next step
      }
      __syncthreads();
      if (tid == 0) {  // log-likelihoods, summed over the steps of a row in order
        for (int m = 0; m < mc; ++m) {
          ll += sm.lp[m];
          const int rr = sm.srow[m];
          if (rr < 0) {
            A.loglik[(size_t)(-1 - rr) * B_inst + b] = ll;
            ll = 0.f;
          }
        }
      }
      // ---------------- P5: dW2 += z^T do', db2 += do'
      chunk_contract(sm.z, sm.op, mc, dW2, dB2, cq, cig);
      __syncthreads();
      // ---------------- P6: dz = (do' W2^T) * [z > 0]   (relu'(0) = 0, as torch)
      chunk_gemm<true>(sm.op, W2, col, hf, acc);
#pragma unroll
      for (int j = 0; j < LMC / 2; ++j) {
        float& zz = sm.z[2 * j + hf][col];
        zz = zz > 0.f ? acc[j] : 0.f;
      }
      __syncthreads();
      // ---------------- P7: dW1 += o^T dz, db1 += dz
      chunk_contract(sm.o, sm.z, mc, dW1, dB1, cq, cig);
      __syncthreads();  // the next chunk overwrites the buffers
    }
  }
}

template <int SPL, int ENV>
int launch_eas_layer(const co_eas_layer_grad_args& A, cudaStream_t st) {
  auto kern = eas_layer_grad_kernel<SPL, ENV>;
  const size_t smem = sizeof(EasLaySmem<SPL>);
  static PerDeviceOnce once;
  bool& configured = once.flag();
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail(CO_ERR_CUDA, "co_eas_layer_grad: smem attribute: %s", cudaGetErrorString(e));
    configured = true;
  }
  int grid = device_info().sm_count;
  if (grid > A.B_inst) grid = A.B_inst;
  kern<<<grid, 256, smem, st>>>(A);
  return check_launch("co_eas_layer_grad");
}

template <int ENV>
int dispatch_eas_layer(const co_eas_layer_grad_args& A, cudaStream_t st) {
  if (A.N <= 32) return launch_eas_layer<1, ENV>(A, st);
  if (A.N <= 64) return launch_eas_layer<2, ENV>(A, st);
  return launch_eas_layer<4, ENV>(A, st);
}
}  // namespace
}  // namespace co

using namespace co;

extern "C" int co_eas_key_grad(const co_eas_grad_args* args, void* stream) {
  if (!args) return fail(CO_ERR_BAD_ARG, "co_eas_key_grad: null args%s");
  const co_eas_grad_args& A = *args;
  if (A.env_kind != CO_ENV_TSP && A.env_kind != CO_ENV_CVRP)
    return fail(CO_ERR_UNSUPPORTED, "co_eas_key_grad: env kind %s%lld (tsp and cvrp only)", "", A.env_kind);
  if (!A.cache || !A.actions || !A.coef || !A.dLf || !A.loglik)
    return fail(CO_ERR_BAD_ARG, "co_eas_key_grad: null pointer%s");
  if (A.B_inst < 0 || A.N < 2 || A.num_rows < 1 || A.T < 1)
    return fail(CO_ERR_BAD_ARG, "co_eas_key_grad: bad shape%s B=%lld N=%lld", "", A.B_inst, A.N);
  if (A.N > co_rollout_max_nodes()) return fail(CO_ERR_UNSUPPORTED, "co_eas_key_grad: N=%s%lld > 128 nodes", "", A.N);
  if (!(A.temperature > 0.f)) return fail(CO_ERR_BAD_ARG, "co_eas_key_grad: temperature must be > 0%s");
  if (!(A.tanh_clipping > 0.f)) return fail(CO_ERR_UNSUPPORTED, "co_eas_key_grad: tanh_clipping must be > 0%s");
  if (A.env_kind == CO_ENV_TSP) {
    if (A.cache_width != 5 * E)
      return fail(CO_ERR_UNSUPPORTED, "co_eas_key_grad: tsp needs the 5E cache (first-node table)%s");
    if (A.T < A.N) return fail(CO_ERR_BAD_ARG, "co_eas_key_grad: T < N%s");
  } else {
    if (A.cache_width != 4 * E) return fail(CO_ERR_BAD_ARG, "co_eas_key_grad: cvrp cache_width must be 4E%s");
    if (!A.demand || !A.w_capacity) return fail(CO_ERR_BAD_ARG, "co_eas_key_grad: demand / w_capacity required for cvrp%s");
  }
  const uintptr_t al = (uintptr_t)A.cache | (uintptr_t)A.dLf;
  if (al & 15) return fail(CO_ERR_BAD_ARG, "co_eas_key_grad: cache / dLf must be 16-byte aligned%s");
  if (A.B_inst == 0) return CO_OK;
  cudaStream_t st = (cudaStream_t)stream;
  return A.env_kind == CO_ENV_TSP ? dispatch_eas<CO_ENV_TSP>(A, st) : dispatch_eas<CO_ENV_CVRP>(A, st);
}

extern "C" int co_eas_layer_grad(const co_eas_layer_grad_args* args, void* stream) {
  if (!args) return fail(CO_ERR_BAD_ARG, "co_eas_layer_grad: null args%s");
  const co_eas_layer_grad_args& A = *args;
  if (A.env_kind != CO_ENV_TSP && A.env_kind != CO_ENV_CVRP)
    return fail(CO_ERR_UNSUPPORTED, "co_eas_layer_grad: env kind %s%lld (tsp and cvrp only)", "", A.env_kind);
  if (!A.cache || !A.actions || !A.coef || !A.layer || !A.dlayer || !A.loglik)
    return fail(CO_ERR_BAD_ARG, "co_eas_layer_grad: null pointer%s");
  if (A.B_inst < 0 || A.N < 2 || A.num_rows < 1 || A.T < 1)
    return fail(CO_ERR_BAD_ARG, "co_eas_layer_grad: bad shape%s B=%lld N=%lld", "", A.B_inst, A.N);
  if (A.N > co_rollout_max_nodes()) return fail(CO_ERR_UNSUPPORTED, "co_eas_layer_grad: N=%s%lld > 128 nodes", "", A.N);
  if (!(A.temperature > 0.f)) return fail(CO_ERR_BAD_ARG, "co_eas_layer_grad: temperature must be > 0%s");
  if (!(A.tanh_clipping > 0.f)) return fail(CO_ERR_UNSUPPORTED, "co_eas_layer_grad: tanh_clipping must be > 0%s");
  if (A.env_kind == CO_ENV_TSP) {
    if (A.cache_width != 5 * E)
      return fail(CO_ERR_UNSUPPORTED, "co_eas_layer_grad: tsp needs the 5E cache (first-node table)%s");
    if (A.T < A.N) return fail(CO_ERR_BAD_ARG, "co_eas_layer_grad: T < N%s");
  } else {
    if (A.cache_width != 4 * E) return fail(CO_ERR_BAD_ARG, "co_eas_layer_grad: cvrp cache_width must be 4E%s");
    if (!A.demand || !A.w_capacity) return fail(CO_ERR_BAD_ARG, "co_eas_layer_grad: demand / w_capacity required for cvrp%s");
  }
  const uintptr_t al = (uintptr_t)A.cache | (uintptr_t)A.layer | (uintptr_t)A.dlayer;
  if (al & 15) return fail(CO_ERR_BAD_ARG, "co_eas_layer_grad: cache / layer / dlayer must be 16-byte aligned%s");
  if (A.B_inst == 0) return CO_OK;
  cudaStream_t st = (cudaStream_t)stream;
  return A.env_kind == CO_ENV_TSP ? dispatch_eas_layer<CO_ENV_TSP>(A, st) : dispatch_eas_layer<CO_ENV_CVRP>(A, st);
}
