// Persistent whole-episode rollout kernel (the north-star kernel) -- implementation header,
// instantiated per environment in rollout_tsp.cu / rollout_cvrp.cu / rollout_sdvrp.cu.
//
// Replaces the `while not td["done"].all()` loop of ConstructivePolicy.forward
// (rl4co/models/common/constructive/base.py:219-251): per node selection it fuses
//   AttentionModelDecoder.forward      rl4co/models/zoo/am/decoder.py:156-193
//     context embedding                nn/env_embeddings/context.py:61-74,116-134,147-149
//     PointerAttention                 nn/attention.py:274-320
//   DecodingStrategy.step              rl4co/utils/decoding.py:138-188,344-461
//   TSPEnv._step / CVRPEnv._step       envs/routing/tsp/env.py:60-86, cvrp/env.py:66-136
// and at the end get_reward (ops.py:82-90) and get_log_likelihood (decoding.py:38-62).
//
// Design: one CTA (256 threads = 8 warps) owns one instance for its whole episode.
//   * warp h holds head h of glimpse_key, glimpse_val AND of the folded logit key (logit_key @ project_out, so that
//     logits = sum_h o_h . L'_h[n]) for all nodes IN REGISTERS as float2 pairs (lane l owns nodes SPL*l .. SPL*l+SPL-1)
//     and keeps its FMAs in float2 pairs.  Glimpse AND the head's share of every pointer logit are warp-local: one
//     REDUX.MAX on an order-preserving integer key, one shared-memory transpose for the value reduction, a 16-float
//     broadcast of the un-normalised head output, and the 1/sum(exp) normalisation applied to the SPL partial logits
//     (its shuffle reduction hides under the FMAs).  A warp reads 4 LDS.128 of head outputs per step; reading all 128
//     head outputs back per thread would cost 16 and make the step LSU-bound.
//   * barrier 1; thread n < NS sums the eight per-head partials of node n, tanh-clip, mask, temperature; the warp's
//     arg-max is REDUX.MAX + ballot (lowest node wins ties, torch semantics); sampling = arg-max of z - log q
//     (Gumbel form of torch.multinomial's p/q); barrier 2; every thread merges the <= 4 per-warp winners.
//   * the log-probability of the chosen node is NOT on the critical path: z of the last two steps stays in shared
//     memory and two warps that have no logits work compute log-softmax(z)[a] while the others are in the tanh /
//     arg-max phase (exact exp-sum with the tanh-clip bound as fixed offset, z <= clip/T), in two halves so that
//     neither outlasts the selection: one takes the lane partials of the PREVIOUS step, the other the sum, log and
//     store of the step before that.
//   * what only the reward and the outputs need (action store, tour length, prize, penalties) is likewise done by
//     another warp that is idle between the barriers, one step behind; the warps that gate barrier 1 replay only the
//     state the next step's mask and context need.
//   * the per-node context table (node_emb @ Wctx_cur^T) sits in shared memory, so the next query is one row read +
//     the per-episode fixed part; each thread keeps only the visited bits it needs; capacity / current node are
//     replicated scalars; the CVRP depot rule uses a register bitmask over demand ranks instead of a block-wide OR;
//   * exactly two block barriers per node selection; no state in HBM.
// HBM traffic per instance = one read of its cache rows + T*(8+4) B of outputs.
//
// Cache layout, one per env: tsp 5E = [K | V | L' | first-table | cur-table], so the first-node half of the context
// projection is one table-row read per episode; the other envs 4E = [K | V | L' | cur-table].
#pragma once
#include "co_common.cuh"

namespace co {

#define CO_MODE_GREEDY 0
#define CO_MODE_SAMPLE 1
#define CO_MODE_EVALUATE 2

template <int SPL>
struct Cfg {
  static constexpr int NS = 32 * SPL;  // node slots
  static constexpr int NW = SPL;       // warps of the selection phase: thread n < NS owns node n there
  static constexpr int MINB = SPL == 4 ? 1 : (SPL == 2 ? 2 : 3);
};

constexpr int TILE_LD = 20;  // padded row of the per-warp AV transpose tile

template <int SPL>
struct Smem {
  float ptab[(32 * SPL + 1) * E];       // current-node context table; last row = zeros
  float qfix[E];                        // per-episode fixed part of the query
  float wcap[E];                        // cvrp: remaining-capacity column of project_context
  float tile[8][32 * TILE_LD];          // per-warp transpose tile for the value reduction
  alignas(16) float oh[8][D];           // per-warp broadcast of the un-normalised head output
  alignas(16) float part[8][32 * SPL];  // per-head share of every pointer logit: [head][node]
  alignas(16) float zbuf[2][32 * SPL];  // masked, temperature-scaled logits of the last two steps (deferred log-prob)
  alignas(16) uint2 red[4];             // per selection warp: (best key as order-preserving uint, node)
  alignas(16) float lps[2][32];         // log-prob warps: lane partial sums of exp(z - Zb) of the last two steps
  float lsel[2];                        // and z[a] - Zb of their chosen nodes
  float ll;                             // ll warp, lane 0: the log-likelihood so far
  float pen;                            // bookkeeping warp, lane 0: pctsp's saved penalties
  float dem[32 * SPL];                  // cvrp / sdvrp: demand; op: prize (node-indexed, depot 0)
  float lim[32 * SPL];                  // op: max_length per node (budget minus the way back); pctsp: penalty per node
  float2 loc[32 * SPL];
  unsigned char order[32 * SPL];        // cvrp: customers sorted by demand (ascending)
  unsigned char rank_of[32 * SPL];      // cvrp: demand rank of each customer (inverse of `order`)
  // sdvrp (dynamic embedding, nn/env_embeddings/dynamic.py:60-78): the remaining demand d_n adds d_n * w to node n's
  // glimpse key / value / folded logit key; everything the step needs beyond d_n is a per-node or per-step scalar
  alignas(16) float wdyn[3 * E];              // [wk | wv | W_out^T wl]
  alignas(16) float pwk[32 * SPL * 8 + 8];    // ptab[n] . wk_h per (node, head); last 8 = the zero row
};

// Phase clocks, a diagnostic build only (-DCO_PHASE_CLOCKS, tools/rollout_phase_clocks.py): lane 0 of every warp
// records clock64() at the top of each decode step, at arrival at / release from both block barriers, and at the top
// of each instance, into co_phase_clk[b][dstep][warp][6] (slots: 0 step top, 1 B1 arrival, 2 B1 release, 3 B2
// arrival, 4 B2 release, 5 instance top (dstep 0 row)).  Single-trajectory launches only; without the macro the
// stamps compile to nothing.  The buffer must be set before the first launch: a constant-bank pointer with no null
// test keeps the clock read off any load's latency.
#ifdef CO_PHASE_CLOCKS
static __constant__ unsigned long long* co_phase_clk;
#define CO_PHASE_STAMP(row, slot)                                                                    \
  do {                                                                                               \
    if (lane == 0) co_phase_clk[(((size_t)b * T_max + (row)) * 8 + h) * 6 + (slot)] = clock64();   \
  } while (0)
#else
#define CO_PHASE_STAMP(row, slot) do { } while (0)
#endif

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
// order-preserving float -> uint (so REDUX.MAX on integers is an exact float max)
__device__ __forceinline__ unsigned fkey(float f) {
  unsigned u = __float_as_uint(f);
  return u ^ ((u >> 31) ? 0xffffffffu : 0x80000000u);
}
__device__ __forceinline__ float funkey(unsigned k) {
  return __uint_as_float(k ^ ((k >> 31) ? 0x80000000u : 0xffffffffu));
}

// Warp sum of non-negative lane values whose total is <= 128 (softmax numerators after the max subtraction, <= 4 per
// lane), through two REDUX.SUM on a 48-bit fixed-point split instead of a five-deep shuffle chain: x * 2^24 is split
// exactly into an integer part and a fraction (fmaf of an exactly representable difference); the result is the fp32
// rounding of a sum that is exact to 2^-48 per lane -- order independent, and at least as accurate as an fp32 tree.
__device__ __forceinline__ float warp_sum_fixed(float x) {
  constexpr float S = 16777216.f;
  const unsigned hi = __float2uint_rz(x * S);
  const float rem = fmaf(x, S, -(float)hi);
  const unsigned lo = __float2uint_rz(rem * S);
  const unsigned Hs = __reduce_add_sync(FULL, hi), Ls = __reduce_add_sync(FULL, lo);
  return fmaf((float)Ls, 1.0f / (S * S), (float)Hs * (1.0f / S));
}

// 2-norm of a coordinate difference as torch's CPU reduction rounds it (op_kernels.cu): sqrt(fma(dy, dy, dx * dx))
__device__ __forceinline__ float dist2_fma(float2 a, float2 b) {
  const float dx = a.x - b.x, dy = a.y - b.y;
  return sqrtf(fmaf(dy, dy, dx * dx));
}

template <int ENV>
__device__ __forceinline__ bool feasible(int n, bool visbit, float d, float used, float thr, int cur, bool anyfeas) {
  if (ENV == CO_ENV_TSP) return !visbit;
  // op/env.py:140-155: d = tour_length + dist(cur, n) (formed by the caller), thr = max_length[n], anyfeas = "the depot
  // has been re-entered"; the depot itself is always feasible
  if (ENV == CO_ENV_OP) return (n == 0) || (!visbit && !anyfeas && !(d > thr));
  // pctsp/env.py:143-151: d != 0 = "the depot has been re-entered", anyfeas = "unvisited customers remain", used = prize
  if (ENV == CO_ENV_PCTSP) return (n == 0) ? !((used < 1.0f) && anyfeas) : (!visbit && d == 0.0f);
  // cvrp/env.py:126-136, sdvrp/env.py:110-116 (depot rule shared)
  if (n == 0) return !(cur == 0 && anyfeas);
  if (ENV == CO_ENV_SDVRP) return !visbit && !(d == 0.0f) && !(used >= thr);  // thr = capacity here; visbit = padding
  return !visbit && !((d + used) > thr);
}

template <int SPL, int ENV, int MODE>
__global__ void __launch_bounds__(256, Cfg<SPL>::MINB) rollout_kernel(const co_rollout_args A) {
  using C = Cfg<SPL>;
  constexpr int NS = C::NS, NW = C::NW;
  constexpr int CW = (ENV == CO_ENV_TSP ? 5 : 4) * E;  // cache row width (tsp: with the first-node table)
  constexpr int CUR_BLK = (ENV == CO_ENV_TSP ? 4 : 3);  // block holding the current-node table (always the last one)
  constexpr bool VRP = (ENV != CO_ENV_TSP);        // depot env with capacity context (cvrp, sdvrp)
  constexpr bool SD = (ENV == CO_ENV_SDVRP);       // split deliveries: dynamic demand + dynamic embedding
  constexpr bool OP = (ENV == CO_ENV_OP);          // orienteering: `used` is the tour length, `cap` the budget at the depot
  constexpr bool PC = (ENV == CO_ENV_PCTSP);       // prize collecting: `used` is the collected prize, `cap` prize_required
  constexpr float LOG2E = 1.4426950408889634f, LN2 = 0.6931471805599453f;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem<SPL>& sm = *reinterpret_cast<Smem<SPL>*>(smem_raw);

  const int tid = threadIdx.x, lane = tid & 31, h = tid >> 5;
  const int N = A.N, B_inst = A.B_inst, S = A.num_starts, T_max = A.T_max;
  const int B_traj = B_inst * S;
  const bool forced_start = (S > 1) && (A.flags & CO_ROLLOUT_FORCED_START);
  const bool philox = (A.noise == nullptr);
  const bool sel_warp = h < NW;   // selection phase: thread tid < NS owns node nL = tid
  // warps that are idle between the two block barriers, and what they do there for the steps before
  const bool lp_warp = h == NW;      // the exp partials of the previous step's log-probability
  const bool bk_warp = h == NW + 1;  // the previous step's share of the reward and the outputs
  const bool ll_warp = h == NW + 2;  // the sum, log and store of the log-probability of the step before that
  const int nL = sel_warp ? tid : NS - 1;
  const int nG = SPL * lane;      // first of this lane's SPL consecutive glimpse nodes
  const float clip = A.tanh_clipping, inv_temp = 1.0f / A.temperature;
  const float Zb = clip * inv_temp;       // z = clip*tanh(.)/T <= Zb: fixed log-softmax offset
  float* tile = sm.tile[h];

  float2 Kr[SPL][8], Vr[SPL][8], Lr[SPL][8];

  for (int b = blockIdx.x; b < B_inst; b += gridDim.x) {
    CO_PHASE_STAMP(0, 5);
    __syncthreads();  // previous instance no longer reads shared memory
    const float* crow = A.cache + (size_t)b * N * CW;
    // ---- one HBM read of the instance: registers <- head slices of glimpse_key / glimpse_val / folded logit key
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
      const int n = nG + k;
      if (n < N) {
        const float4* ks = reinterpret_cast<const float4*>(crow + (size_t)n * CW + 0 * E + h * D);
        const float4* vs = reinterpret_cast<const float4*>(crow + (size_t)n * CW + 1 * E + h * D);
        const float4* ls = reinterpret_cast<const float4*>(crow + (size_t)n * CW + 2 * E + h * D);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float4 kv = __ldg(ks + c), vv = __ldg(vs + c), lv = __ldg(ls + c);
          Kr[k][2 * c] = make_float2(kv.x, kv.y); Kr[k][2 * c + 1] = make_float2(kv.z, kv.w);
          Vr[k][2 * c] = make_float2(vv.x, vv.y); Vr[k][2 * c + 1] = make_float2(vv.z, vv.w);
          Lr[k][2 * c] = make_float2(lv.x, lv.y); Lr[k][2 * c + 1] = make_float2(lv.z, lv.w);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          Kr[k][j] = make_float2(0.f, 0.f); Vr[k][j] = make_float2(0.f, 0.f); Lr[k][j] = make_float2(0.f, 0.f);
        }
      }
    }
    // ---- shared memory <- context table, coordinates, demands
    // (cp.async: the ~13 16-byte copies of a thread are all in flight at once; the LDG -> STS loop this replaces
    // waited for every load before the next one was issued and was a fifth of the per-instance prologue)
    for (int idx = tid; idx < N * (E / 4); idx += 256) {
      const int n = idx >> 5, c = idx & 31;
      const uint32_t dst = (uint32_t)__cvta_generic_to_shared(reinterpret_cast<float4*>(sm.ptab + n * E) + c);
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst),
                   "l"(reinterpret_cast<const float4*>(crow + (size_t)n * CW + CUR_BLK * E) + c) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    if (tid < E) {
      sm.ptab[NS * E + tid] = 0.f;
      sm.wcap[tid] = VRP ? A.w_capacity[tid] : 0.f;
    }
    if (tid < NS) {
      sm.loc[tid] = (tid < N) ? reinterpret_cast<const float2*>(A.locs)[(size_t)b * N + tid] : make_float2(0.f, 0.f);
      sm.dem[tid] = (VRP && tid >= 1 && tid < N) ? A.demand[(size_t)b * (N - 1) + tid - 1] : 0.f;
      if (OP || PC) sm.lim[tid] = (tid < N) ? A.node_limit[(size_t)b * N + tid] : 0.f;  // op: length limit; pctsp: penalty
    }
    if (SD) {
      for (int i = tid; i < 3 * E; i += 256) sm.wdyn[i] = A.dyn_w[i];
    }
    const float cap = (VRP && A.vehicle_capacity) ? A.vehicle_capacity[b] : 1.0f;
    // cvrp: fp32 add, as `td["vehicle_capacity"] + 1e-5`; sdvrp compares `used >= vehicle_capacity` (no slack)
    const float thr = SD ? cap : cap + 1e-5f;
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    if (SD) {  // per-(node, head) dot of the context-table row with the dynamic key weight
      for (int i = tid; i < (NS + 1) * 8; i += 256) {
        const int n = i >> 3, hh = i & 7;
        float acc = 0.f;
        if (n < N) {
#pragma unroll
          for (int c = 0; c < D; ++c) acc = fmaf(sm.ptab[n * E + hh * D + c], sm.wdyn[hh * D + c], acc);
        }
        sm.pwk[i] = acc;
      }
      __syncthreads();
    }
    if (ENV == CO_ENV_CVRP) {  // rank-sort customers by demand (ties by index) -> sm.order
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
      __syncthreads();
    }
    // per-thread node constants: (remaining) demand for cvrp / sdvrp; op: the node's length limit, plus its coordinates
    float dmk0[SPL];
    float2 lck[SPL];
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
      dmk0[k] = OP ? sm.lim[nG + k] : sm.dem[nG + k];
      lck[k] = OP ? sm.loc[nG + k] : make_float2(0.f, 0.f);
    }
    const float dL0 = OP ? sm.lim[nL] : sm.dem[nL];
    const float2 lcL = OP ? sm.loc[nL] : make_float2(0.f, 0.f);
    // scores split by linearity: q.K = ptab[cur].K + qfix.K + rem * (wcap.K); the last two are
    // per-episode / per-instance constants held in registers (FK, WK)
    auto head_dot = [&](const float* vec, float (&out)[SPL]) {
      const float4* vp = reinterpret_cast<const float4*>(vec + h * D);
      float2 a2[SPL];
#pragma unroll
      for (int k = 0; k < SPL; ++k) a2[k] = make_float2(0.f, 0.f);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float4 x = vp[c];
#pragma unroll
        for (int k = 0; k < SPL; ++k) {
          a2[k] = ffma2(make_float2(x.x, x.y), Kr[k][2 * c], a2[k]);
          a2[k] = ffma2(make_float2(x.z, x.w), Kr[k][2 * c + 1], a2[k]);
        }
      }
#pragma unroll
      for (int k = 0; k < SPL; ++k) out[k] = a2[k].x + a2[k].y;
    };
    // tsp: qfix += project_context[:, :E] @ h[first] (context.py:129-133), the first-node table row; callers barrier
    // before and after
    auto add_first = [&](int a_first) {
      if (tid < E) sm.qfix[tid] += __ldg(crow + (size_t)a_first * CW + 3 * E + tid);
    };
    float WK[SPL], FK[SPL];
#pragma unroll
    for (int k = 0; k < SPL; ++k) { WK[k] = 0.f; FK[k] = 0.f; }
    if (VRP) head_dot(sm.wcap, WK);
    // sdvrp per-instance / per-lane constants of the dynamic terms
    float WKW = 0.f, wv_d = 0.f;
    if (SD) {
#pragma unroll
      for (int c = 0; c < D; ++c) WKW = fmaf(sm.wcap[h * D + c], sm.wdyn[h * D + c], WKW);  // wcap_h . wk_h
      wv_d = sm.wdyn[E + h * D + (lane & 15)];
    }
    if (b + (int)gridDim.x < B_inst) {  // next instance's cache rows -> L2
      // only the four blocks the kernel reads (K, V, L', current-node table): with the 5E layout the first-node table
      // block would otherwise be pulled from HBM for nothing
      const char* nxt = reinterpret_cast<const char*>(A.cache + (size_t)(b + gridDim.x) * N * CW);
      for (int i = tid; i < N * 16; i += 256) {  // 16 lines of 128 B per node row
        const int n = i >> 4, blk = (i >> 2) & 3, line = i & 3;
        const size_t off = ((size_t)n * CW + (blk < 3 ? blk : CUR_BLK) * E) * 4 + ((size_t)line << 7);
        asm volatile("prefetch.global.L2 [%0];" ::"l"(nxt + off));
      }
    }

    for (int s = 0; s < S; ++s) {
      const int traj = s * B_inst + b;  // start-major, rl4co/utils/ops.py:10-29
      // output rows, addressed from the arguments at each store: no 64-bit row pointers are carried through the loop
      const size_t row = (size_t)traj * T_max;
      // ---------------- reset (tsp/env.py:88-113, cvrp/env.py:98-124)
      // visited flags this thread needs: bit k = its glimpse node nG + k, bit 8 = its selection-phase node nL
      // (padding slots start as visited)
      uint32_t mybits = (!sel_warp || nL >= N) ? 0x100u : 0u;
#pragma unroll
      for (int k = 0; k < SPL; ++k) mybits |= (nG + k >= N) ? (1u << k) : 0u;
      int cur = (ENV == CO_ENV_TSP) ? NS : 0;  // NS -> zero row: step-0 placeholder context
      int first = 0, t = 0, dstep = 0, nvis = 0;
      int prev = 0;      // bookkeeping warp: the last node it has accounted
      float dist = 0.f;  // bookkeeping warp: the tour length (op: the collected prize)
      // cvrp: visited customers as a bitmask over demand RANKS (bits >= #customers pre-set), so the
      // unvisited customer of least demand is ffs(~mask): registers only, nothing shared is written
      uint32_t rmask[SPL];
#pragma unroll
      for (int k = 0; k < SPL; ++k) {
        const int lo = 32 * k, nc = N - 1;
        rmask[k] = (nc >= lo + 32) ? 0u : (nc <= lo ? 0xffffffffu : (0xffffffffu << (nc - lo)));
      }
      float used = 0.f;
      bool anyfeas = false, done = false, depot_seen = false;
      // (remaining) demand of this thread's glimpse nodes / selection node: constant for cvrp, dynamic for sdvrp
      float dmk[SPL], dL = dL0;
#pragma unroll
      for (int k = 0; k < SPL; ++k) dmk[k] = dmk0[k];
      int nrem = 0;                 // sdvrp: customers with demand left
      int pend_a = -1;              // sdvrp: demand write-back deferred past the next barrier (see env_step)
      float pend_d = 0.f, FKW = 0.f;
      // sdvrp serves demand in place (sm.dem): every further trajectory of the instance starts from the original demands
      // (every thread is past the previous trajectory's last read: the epilogue barrier)
      if (SD && s > 0 && tid < NS) sm.dem[tid] = (tid >= 1 && tid < N) ? A.demand[(size_t)b * (N - 1) + tid - 1] : 0.f;
      __syncthreads();  // previous trajectory finished with qfix
      if (bk_warp && lane == 0) sm.pen = 0.f;
      if (ll_warp && lane == 0) sm.ll = 0.f;
      if (tid < E) {
        float g = A.graph_ctx ? A.graph_ctx[(size_t)b * E + tid] : 0.f;
        if (ENV == CO_ENV_TSP && !forced_start) g += A.q_placeholder[tid];
        sm.qfix[tid] = g;
      }

      // one environment transition, replicated in every thread
      auto env_step = [&](int a) {
        if (!SD) {  // (sdvrp: nodes may be revisited; mybits only flags the padding slots there)
          const unsigned dd = (unsigned)(a - nG);
          mybits |= (dd < (unsigned)SPL) ? (1u << dd) : 0u;
          mybits |= (a == nL) ? 0x100u : 0u;
        }
        if (ENV == CO_ENV_TSP) {
          if (t == 0) first = a;
        } else if (OP) {
          // op/env.py:72-105: the tour length feeds the mask and the context (every thread replays it, `used`); the
          // collected prize is the reward (see account); the depot re-entered after step 0 ends the episode
          used = used + dist2_fma(sm.loc[a], sm.loc[cur]);
          depot_seen = depot_seen || (a == 0);
        } else if (PC) {
          // pctsp/env.py:62-93: collected prize (replicated: depot rule + context); saved penalties: see account
          used = used + sm.dem[a];
          nvis += (a != 0) ? 1 : 0;
          depot_seen = depot_seen || (a == 0);
        } else if (SD) {
          // sdvrp/env.py:55-82: deliver min(remaining demand, remaining capacity); every thread replays the arithmetic.
          // sm.dem[a] is read by all threads here, so the owner's write-back waits until after the next block barrier.
          const float d_a = sm.dem[a];
          const float delivered = fminf(d_a, cap - used);
          used = (used + delivered) * (a != 0 ? 1.0f : 0.0f);
          const float d_new = d_a + (-delivered);  // scatter_add(-1, a, -delivered)
#pragma unroll
          for (int k = 0; k < SPL; ++k) dmk[k] = (a == nG + k) ? d_new : dmk[k];
          dL = (a == nL) ? d_new : dL;
          nrem += ((d_new > 0.f) ? 1 : 0) - ((d_a > 0.f) ? 1 : 0);
          pend_a = a; pend_d = d_new;
          anyfeas = (nrem > 0) && !(used >= cap);
        } else {
          used = (used + sm.dem[a == 0 ? 1 : a]) * (a != 0 ? 1.0f : 0.0f);  // cvrp/env.py:70-76
          // distinct nodes visited: a customer is new by construction (masked once visited), the depot
          // only on its first visit
          nvis += (a != 0 || !depot_seen) ? 1 : 0;
          depot_seen = depot_seen || (a == 0);
          if (a != 0) {
            const int r = sm.rank_of[a];
#pragma unroll
            for (int k = 0; k < SPL; ++k) rmask[k] |= ((r >> 5) == k) ? (1u << (r & 31)) : 0u;
          }
          // depot rule (cvrp/env.py:134): any unvisited customer that still fits <=> the unvisited
          // customer of least demand fits (fp32 add is monotone in the demand)
          int pmin = NS;
#pragma unroll
          for (int k = SPL - 1; k >= 0; --k) {
            const uint32_t z = ~rmask[k];
            if (z) pmin = 32 * k + __ffs(z) - 1;
          }
          anyfeas = (pmin < N - 1) && !((sm.dem[sm.order[pmin < N - 1 ? pmin : 0]] + used) > thr);
        }
        cur = a; ++t;
        // cvrp: all nodes incl. the depot visited; sdvrp: no positive demand left (sdvrp/env.py:71)
        done = (ENV == CO_ENV_TSP) ? (t >= N) : ((OP || PC) ? (a == 0 && t > 1) : (SD ? (nrem == 0) : (nvis >= N)));
      };
      // log-softmax(z)[a] of a finished step (decoding.py:188,352-356): exact exp-sum with the fixed offset Zb; masked
      // nodes hold -inf -> 2^-inf = 0.  First half (lp warp): the lane partials from the step's z row, whose chosen
      // node is cur; second half (ll warp, one step later): their sum, log and store.
      auto logp_partials = [&](int buf) {
        const float* zb = sm.zbuf[buf];
        float sacc = 0.f;
#pragma unroll
        for (int k = 0; k < SPL; ++k) sacc += ex2((zb[nG + k] - Zb) * LOG2E);
        sm.lps[buf][lane] = sacc;
        if (lane == 0) sm.lsel[buf] = zb[cur] - Zb;
      };
      auto logp_finish = [&](int buf, int t_out) {
        // 32 lane partials -> every lane adds all of them in a fixed tree from shared memory (shorter dependent
        // chain than five shuffles; this warp must finish inside the other warps' selection phase)
        const float ll_prev = sm.ll;  // read with the partials, not after the tree
        const float4* lq = reinterpret_cast<const float4*>(sm.lps[buf]);
        const float4 q0 = lq[0], q1 = lq[1], q2 = lq[2], q3 = lq[3], q4 = lq[4], q5 = lq[5], q6 = lq[6], q7 = lq[7];
        const float t0 = ((q0.x + q0.y) + (q0.z + q0.w)) + ((q1.x + q1.y) + (q1.z + q1.w));
        const float t1 = ((q2.x + q2.y) + (q2.z + q2.w)) + ((q3.x + q3.y) + (q3.z + q3.w));
        const float t2 = ((q4.x + q4.y) + (q4.z + q4.w)) + ((q5.x + q5.y) + (q5.z + q5.w));
        const float t3 = ((q6.x + q6.y) + (q6.z + q6.w)) + ((q7.x + q7.y) + (q7.z + q7.w));
        const float sacc = (t0 + t1) + (t2 + t3);
        const float lp = sm.lsel[buf] - lg2(sacc) * LN2;
        if (lane == 0) {
          sm.ll = ll_prev + lp;
          A.logp_out[row + t_out] = lp;
        }
      };
      // per-step work that only the reward and the outputs need (bookkeeping warp, one step behind): the tour length,
      // op's prize, pctsp's saved penalties, the action store.  The tour length is the longest chain between the
      // barriers, so it goes first and without a branch: tsp's first step adds +0.0f to dist = +0, exactly as skipping.
      auto account = [&](int a, int ta) {
        if (!OP) {
          const float2 pa = sm.loc[a], pp = sm.loc[prev];
          const float dx = pa.x - pp.x, dy = pa.y - pp.y;
          const float leg = sqrtf(dx * dx + dy * dy);
          dist += (VRP || ta != 0) ? leg : 0.f;
        }
        if (OP) dist += sm.dem[a];
        if (PC && lane == 0) sm.pen += sm.lim[a];
        if (lane == 0) A.actions_out[row + ta] = a;
        prev = a;
      };

      if (SD) {  // customers with demand: counted by every thread from shared memory (uniform)
        for (int n = 1; n < N; ++n) nrem += (sm.dem[n] > 0.f) ? 1 : 0;
        anyfeas = (nrem > 0) && !(used >= cap);
        done = (nrem == 0);
      }
      if (forced_start) {  // multistart pre_decoder_hook, decoding.py:309-326 + ops.py:128-149 (sdvrp, op, pctsp)
        const int a0 = (s % A.num_loc) + (VRP ? 1 : 0);
        if (tid == 0) A.logp_out[row] = 0.f;
        env_step(a0);
        if (bk_warp) account(a0, 0);
      } else if (ENV == CO_ENV_CVRP) {
        anyfeas = !((sm.dem[sm.order[0]] + used) > thr);
      }
      __syncthreads();
      head_dot(sm.qfix, FK);
      if (SD) {
#pragma unroll
        for (int c = 0; c < D; ++c) FKW = fmaf(sm.qfix[h * D + c], sm.wdyn[h * D + c], FKW);  // qfix_h . wk_h
      }

      while (!done && t < T_max) {
        CO_PHASE_STAMP(dstep, 0);
        // early, latency-tolerant loads for this step
        int forced = 0;
        float gum = 0.f;  // -log q, q ~ Exp(1): Gumbel perturbation for sampling
        if (MODE == CO_MODE_EVALUATE) forced = (int)A.forced_actions[(size_t)traj * T_max + t];
        if (MODE == CO_MODE_SAMPLE && tid < N) {
          const float q = philox ? philox_exp1(A.seed, A.offset, traj, dstep, tid)
                                 : A.noise[((size_t)dstep * B_traj + traj) * N + tid];
          gum = -logf(q);
        }

        // ---------------- glimpse + this head's share of every pointer logit: warp h = head h, fully warp-local
        {
          const float4* pr = reinterpret_cast<const float4*>(sm.ptab + cur * E + h * D);
          const float rem = PC ? fmaxf(cap - used, 0.0f) : cap - used;  // context.py:147-149; pctsp :184-198 clamps at 0
          float2 sc2[SPL];
#pragma unroll
          for (int k = 0; k < SPL; ++k) sc2[k] = make_float2(0.f, 0.f);
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float4 p = pr[c];
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
              sc2[k] = ffma2(make_float2(p.x, p.y), Kr[k][2 * c], sc2[k]);
              sc2[k] = ffma2(make_float2(p.z, p.w), Kr[k][2 * c + 1], sc2[k]);
            }
          }
          // scores in log2 units: s * (1/sqrt(head_dim)) * log2(e)
          float sc[SPL], m = -INFINITY;
          bool fz[SPL];
          // sdvrp: q_h . wk_h = ptab[cur]_h . wk_h + qfix_h . wk_h + rem * (wcap_h . wk_h)
          const float qwk = SD ? fmaf(rem, WKW, sm.pwk[cur * 8 + h] + FKW) : 0.f;
          const float2 pcur = OP ? sm.loc[cur] : make_float2(0.f, 0.f);
#pragma unroll
          for (int k = 0; k < SPL; ++k) {
            fz[k] = OP ? feasible<ENV>(nG + k, (mybits >> k) & 1u, used + dist2_fma(lck[k], pcur), used, dmk[k], cur, depot_seen)
                    : PC ? feasible<ENV>(nG + k, (mybits >> k) & 1u, depot_seen ? 1.0f : 0.0f, used, thr, cur, nvis < N - 1)
                         : feasible<ENV>(nG + k, (mybits >> k) & 1u, dmk[k], used, thr, cur, anyfeas);
            float dot = (sc2[k].x + sc2[k].y) + FK[k];
            if (VRP) dot = fmaf(rem, WK[k], dot);
            if (SD) dot = fmaf(dmk[k], qwk, dot);  // q . (K[n] + d_n wk) = q.K[n] + d_n (q.wk)
            sc[k] = fz[k] ? dot * (0.25f * LOG2E) : -INFINITY;
            m = fmaxf(m, sc[k]);
          }
          m = funkey(__reduce_max_sync(FULL, fkey(m)));
          float2 acc[8];
          float esum = 0.f, sed = 0.f;  // sed (sdvrp) = sum_n e_n d_n: the dynamic value term is sed * wv_h
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] = make_float2(0.f, 0.f);
#pragma unroll
          for (int k = 0; k < SPL; ++k) {
            const float e = fz[k] ? ex2(sc[k] - m) : 0.f;
            esum += e;
            if (SD) sed = fmaf(e, dmk[k], sed);
            const float2 e2 = make_float2(e, e);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = ffma2(e2, Vr[k][j], acc[j]);
          }
          // lane-sum of the 16 partial outputs through a padded shared-memory transpose
          float4* trow = reinterpret_cast<float4*>(tile + lane * TILE_LD);
#pragma unroll
          for (int c = 0; c < 4; ++c) trow[c] = make_float4(acc[2 * c].x, acc[2 * c].y, acc[2 * c + 1].x, acc[2 * c + 1].y);
          if (SD) sed = warp_sum(sed);
          __syncwarp();
          const int d = lane & 15, half = lane >> 4;
          float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
          for (int r = 0; r < 16; r += 4) {  // half 1 reads rows rotated by 4: bank-conflict free
            s0 += tile[(16 * half + ((r + 0 + 4 * half) & 15)) * TILE_LD + d];
            s1 += tile[(16 * half + ((r + 1 + 4 * half) & 15)) * TILE_LD + d];
            s2 += tile[(16 * half + ((r + 2 + 4 * half) & 15)) * TILE_LD + d];
            s3 += tile[(16 * half + ((r + 3 + 4 * half) & 15)) * TILE_LD + d];
          }
          float r = (s0 + s1) + (s2 + s3);
          r += __shfl_xor_sync(FULL, r, 16);
          if (SD) r = fmaf(sed, wv_d, r);  // + (sum_n e_n d_n) * wv_h[d]
          if (lane < 16) sm.oh[h][lane] = r;  // un-normalised head output (d == lane here)
          __syncwarp();
          // share of head h in the pointer logits of this lane's nodes: (o_h / esum) . L'_h[n]  (+ sdvrp: d_n (o_h . wl'_h))
          const float4* op = reinterpret_cast<const float4*>(sm.oh[h]);
          float2 pl2[SPL];
          float olh = 0.f;
#pragma unroll
          for (int k = 0; k < SPL; ++k) pl2[k] = make_float2(0.f, 0.f);
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float4 x = op[c];
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
              pl2[k] = ffma2(make_float2(x.x, x.y), Lr[k][2 * c], pl2[k]);
              pl2[k] = ffma2(make_float2(x.z, x.w), Lr[k][2 * c + 1], pl2[k]);
            }
            if (SD) {
              const float4 w = reinterpret_cast<const float4*>(sm.wdyn + 2 * E + h * D)[c];
              olh = fmaf(x.x, w.x, olh); olh = fmaf(x.y, w.y, olh); olh = fmaf(x.z, w.z, olh); olh = fmaf(x.w, w.w, olh);
            }
          }
          esum = warp_sum_fixed(esum);  // 0 <= e <= 1 per node: two REDUX.SUM, independent of the FMA block above
          const float rinv = __fdividef(1.0f, esum);
          float pl[SPL];
#pragma unroll
          for (int k = 0; k < SPL; ++k) {
            float v = pl2[k].x + pl2[k].y;
            if (SD) v = fmaf(dmk[k], olh, v);
            pl[k] = v * rinv;
          }
          float* pdst = sm.part[h] + nG;
          if (SPL == 4) *reinterpret_cast<float4*>(pdst) = make_float4(pl[0], pl[SPL > 1 ? 1 : 0], pl[SPL > 2 ? 2 : 0], pl[SPL > 3 ? 3 : 0]);
          else if (SPL == 2) *reinterpret_cast<float2*>(pdst) = make_float2(pl[0], pl[SPL > 1 ? 1 : 0]);
          else *pdst = pl[0];
        }
        CO_PHASE_STAMP(dstep, 1);
        __syncthreads();  // B1: every head's share of every logit is in shared memory
        CO_PHASE_STAMP(dstep, 2);

        if (SD && tid == 0 && pend_a >= 0) sm.dem[pend_a] = pend_d;  // deferred demand write-back (every thread is
                                                                     // past the env_step that read the old value)
        if (sel_warp) {
          // ---------------- pointer logit of node nL: heads summed in fixed order, tanh clip, mask, temperature
          const bool fzL = OP ? feasible<ENV>(nL, (mybits >> 8) & 1u, used + dist2_fma(lcL, sm.loc[cur]), used, dL, cur, depot_seen)
                           : PC ? feasible<ENV>(nL, (mybits >> 8) & 1u, depot_seen ? 1.0f : 0.0f, used, thr, cur, nvis < N - 1)
                                : feasible<ENV>(nL, (mybits >> 8) & 1u, dL, used, thr, cur, anyfeas);
          const float p = ((sm.part[0][nL] + sm.part[1][nL]) + (sm.part[2][nL] + sm.part[3][nL])) +
                          ((sm.part[4][nL] + sm.part[5][nL]) + (sm.part[6][nL] + sm.part[7][nL]));
          const float lg = tanhf(p * 0.08838834764831845f) * clip;  // /sqrt(E), tanh clip (decoding.py:169-170)
          const float z = fzL ? lg * inv_temp : -INFINITY;          // mask, temperature (decoding.py:173-177)
          sm.zbuf[dstep & 1][nL] = z;
          if (MODE != CO_MODE_EVALUATE) {
            const float keyf = (MODE == CO_MODE_SAMPLE) ? (fzL ? z + gum : -INFINITY) : z;
            const unsigned key = fkey(keyf);
            const unsigned wkey = __reduce_max_sync(FULL, key);
            const unsigned vote = __ballot_sync(FULL, key == wkey);
            if (lane == 0) sm.red[h] = make_uint2(wkey, (unsigned)(32 * h + __ffs(vote) - 1));  // lowest node wins ties
          }
        } else if (bk_warp) {  // longest chain first; then the earlier steps' log-probabilities, off the critical path
          if (dstep > 0) account(cur, t - 1);
        } else if (ll_warp) {
          if (dstep > 1) logp_finish(dstep & 1, t - 2);
        } else if (lp_warp && dstep > 0) {
          logp_partials((dstep - 1) & 1);
        }
        CO_PHASE_STAMP(dstep, 3);
        __syncthreads();  // B2: per-warp winners complete
        CO_PHASE_STAMP(dstep, 4);
        int a;
        if (MODE == CO_MODE_EVALUATE) {
          a = (forced < 0 || forced >= N) ? 0 : forced;
        } else if (NW == 1) {
          a = (int)sm.red[0].y;
        } else if (NW == 2) {
          const uint4 r0 = reinterpret_cast<const uint4*>(sm.red)[0];
          a = (int)((r0.z > r0.x) ? r0.w : r0.y);  // strict '>' keeps the lower warp (= lowest node) on ties
        } else {
          const uint4 r0 = reinterpret_cast<const uint4*>(sm.red)[0], r1 = reinterpret_cast<const uint4*>(sm.red)[1];
          const bool b01 = r0.z > r0.x, b23 = r1.z > r1.x;
          const unsigned ka = b01 ? r0.z : r0.x, ia = b01 ? r0.w : r0.y;
          const unsigned kb = b23 ? r1.z : r1.x, ib = b23 ? r1.w : r1.y;
          a = (int)((kb > ka) ? ib : ia);
        }

        // ---------------- environment step
        const bool was_first = (ENV == CO_ENV_TSP) && (t == 0);
        env_step(a);
        ++dstep;
        if (was_first) {  // context from now on: [h_first ; h_cur], context.py:129-133
          if (tid < E) sm.qfix[tid] = A.graph_ctx ? A.graph_ctx[(size_t)b * E + tid] : 0.f;
          __syncthreads();
          add_first(a);
          __syncthreads();
          head_dot(sm.qfix, FK);
        }
      }

      // ---------------- epilogue: last log-probability, reward, log-likelihood, padding
      __syncthreads();
      if (lp_warp && dstep > 0) logp_partials((dstep - 1) & 1);
      __syncthreads();  // the last step's partials are in shared memory
      if (ll_warp) {  // the last two steps (decode step k has the output index t - dstep + k)
        for (int k = dstep > 1 ? dstep - 2 : 0; k < dstep; ++k) logp_finish(k & 1, t - dstep + k);
        if (lane == 0) A.loglik_out[traj] = sm.ll;
      }
      if (bk_warp && dstep > 0) account(cur, t - 1);
      if (bk_warp && lane == 0) {
        const float2 pa = sm.loc[(ENV == CO_ENV_TSP) ? first : 0], pp = sm.loc[prev];
        const float dx = pa.x - pp.x, dy = pa.y - pp.y;
        float rw = OP ? dist : -(dist + sqrtf(dx * dx + dy * dy));  // op: the collected prize
        if (PC) {  // pctsp/env.py:153-172: saved penalties - (length + all penalties)
          float total = 0.f;
          for (int n = 1; n < N; ++n) total += sm.lim[n];
          rw = sm.pen - (-rw + total);
        }
        A.reward_out[traj] = rw;
        if (A.steps_out) A.steps_out[traj] = t;
        if (A.used_capacity_out) A.used_capacity_out[traj] = used;
        if (A.max_steps_out) atomicMax(A.max_steps_out, t);
      }
      // done instances keep selecting the depot with log-prob 0 until the batch finishes
      for (int c = t + tid; c < T_max; c += 256) { A.actions_out[row + c] = 0; A.logp_out[row + c] = 0.f; }
    }
  }
}

template <int SPL, int ENV, int MODE>
static int launch(const co_rollout_args& A, cudaStream_t st) {
  auto kern = rollout_kernel<SPL, ENV, MODE>;
  const size_t smem = sizeof(Smem<SPL>);
  static PerDeviceOnce once;
  static int ctas_per_sm = 1;
  bool& configured = once.flag();
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail(CO_ERR_CUDA, "co_rollout: smem attribute: %s", cudaGetErrorString(e));
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, kern, 256, smem);
    if (e != cudaSuccess || ctas_per_sm < 1) return fail(CO_ERR_CUDA, "co_rollout: occupancy query failed%s");
    configured = true;
  }
  int grid = device_info().sm_count * ctas_per_sm;
  if (grid > A.B_inst) grid = A.B_inst;
  kern<<<grid, 256, smem, st>>>(A);
  return check_launch("co_rollout");
}

template <int ENV>
static int dispatch(const co_rollout_args& A, cudaStream_t st) {
  const int spl = A.N <= 32 ? 1 : (A.N <= 64 ? 2 : 4);
  const int mode = A.select_mode == CO_SELECT_GREEDY ? CO_MODE_GREEDY
                   : (A.select_mode == CO_SELECT_EVALUATE ? CO_MODE_EVALUATE : CO_MODE_SAMPLE);
#define CO_CASE(S_, M_) \
  if (spl == S_ && mode == M_) return launch<S_, ENV, M_>(A, st);
  CO_CASE(1, CO_MODE_GREEDY) CO_CASE(2, CO_MODE_GREEDY) CO_CASE(4, CO_MODE_GREEDY)
  CO_CASE(1, CO_MODE_SAMPLE) CO_CASE(2, CO_MODE_SAMPLE) CO_CASE(4, CO_MODE_SAMPLE)
  CO_CASE(1, CO_MODE_EVALUATE) CO_CASE(2, CO_MODE_EVALUATE) CO_CASE(4, CO_MODE_EVALUATE)
#undef CO_CASE
  return fail(CO_ERR_BAD_ARG, "co_rollout: no kernel variant%s");
}

}  // namespace co
