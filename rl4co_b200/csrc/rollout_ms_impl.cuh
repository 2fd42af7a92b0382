// Query-batched persistent rollout for multistart / multisample decoding (POMO): the S
// trajectories of an instance share its K / V / logit-key (am/decoder.py:178-179 shares them the
// same way through `unbatchify`), so this variant advances Q = 4 trajectories per pass.
//
// Same numerics as rollout_impl.cuh (read that header first); structure:
//   * every phase handles the Q trajectories of the group before the block barrier, written
//     stage-major in straight-line code so that their independent instruction streams interleave
//     (a warp issues in order: a per-trajectory loop would serialise the chains and gain nothing);
//     the two barriers and the serial REDUX / MUFU / shuffle / LDS latencies are thereby
//     amortised over Q node selections;
//   * glimpse_key / glimpse_val head slices live in registers (warp h = head h, lane l owns nodes l + 32 k);
//     the folded logit key lives in shared memory HEAD-MAJOR ([head][16-byte chunk][node], conflict-free
//     LDS.128): after its glimpse warp h reads its 16 un-normalised head outputs of the Q trajectories back
//     (16 broadcast LDS.128) and its own slice of the logit key ONCE per pass (4 x SPL LDS.128), and adds head
//     h's share of every pointer logit of the Q trajectories (the version before read all 128 head outputs per
//     thread and trajectory: 64 broadcast LDS.128 per thread and pass, the LSU-bound part of the pass);
//   * selection: thread (node, group): the 256 threads split into 256 / NS groups that take Q * NS / 256
//     trajectories each, sum the eight per-head shares, tanh / mask / temperature, per-warp arg-max and exp-sum;
//   * trajectories that are done (CVRP: variable length) are still computed but their results are
//     discarded by predication; the group ends when all of its trajectories are done.
// Layout of results is unchanged: row j = s * B + b (start-major, rl4co/utils/ops.py:10-29).
//
// LAYER (EAS-Lay, co_rollout_args.eas_layer): the head outputs are normalised in the glimpse (the layer is not linear,
// so the 1 / sum(exp) factor cannot stay on the logit shares), written to LayerMS::o, and each pass runs
// o' = o + relu(o W1 + b1) W2 + b2 for its Q trajectories with the whole block (thread (channel c, trajectory pair)),
// W1 / W2 of the instance read through L1 / L2 (128 KiB: they do not fit beside SmemMS<4>); o' takes the place of
// the head outputs in the logit shares.  Three block barriers more per pass.  LAYER = false is the kernel as before.
//
// POLY (PolyNet, co_rollout_args.poly): the head outputs are normalised into PolyMS::o as for LAYER; each pass then
// computes g = o W_out^T (thread (channel c, trajectory pair)), u = relu(g W1 + c[s % k]) over CO_POLY_DIM channels
// (thread = channel, all Q trajectories) and g' = g + (u W2 + b2) (thread (channel c, trajectory pair)), and g' takes the
// place of the head outputs in the logit shares against the un-folded logit key in block 2 of the cache.  The weights
// (320 KiB + k KiB) are shared by all instances and read through L1 / L2 like EAS-Lay's; four block barriers more per
// pass.
#pragma once
#include "rollout_impl.cuh"

namespace co {

constexpr int MSQ = 4;  // trajectories per pass

template <int SPL>
struct CfgMS {
  static constexpr int NS = 32 * SPL;                    // node slots
  static constexpr int G = 256 / NS;                     // selection groups of NS threads (2 / 4 / 8)
  static constexpr int TPG = (MSQ >= G) ? MSQ / G : 1;   // trajectories per selection group (2 / 1 / 1)
  static constexpr int GA = MSQ / TPG;                   // groups that have selection work (2 / 4 / 4)
};

template <int SPL>
struct SmemMS {
  float ptab[(32 * SPL + 1) * E];          // current-node context table; last row = zeros
  float4 lkh[8 * 4 * 32 * SPL];            // folded logit key, head-major: [head][chunk of 4 channels][node]
  float qfix[MSQ][E];                      // per-trajectory fixed part of the query
  float wcap[E];
  alignas(16) float oh[8][MSQ][D];         // per-warp un-normalised head outputs of the Q trajectories
  float tile[8][2][32 * TILE_LD];          // per-warp ping-pong transpose tiles
  float part[MSQ][8][32 * SPL];            // per-head share of every pointer logit: [trajectory][head][node]
  alignas(16) unsigned red_key[MSQ][4];    // per selection warp of the trajectory's group
  alignas(16) int red_idx[MSQ][4];
  alignas(16) float red_sum[MSQ][4];
  float dem[32 * SPL];
  float2 loc[32 * SPL];
  unsigned char order[32 * SPL];
  unsigned char rank_of[32 * SPL];
  float ll_acc[MSQ];
};

// EAS-Lay buffers, behind SmemMS<SPL> in the LAYER variant
struct LayerMS {
  alignas(16) float o[MSQ][E];  // normalised head outputs of the pass, (h g) order
  alignas(16) float z[MSQ][E];  // relu(o W1 + b1)
};
// PolyNet buffers, behind SmemMS<SPL> in the POLY variant; `o` sits where LayerMS::o does
struct PolyMS {
  alignas(16) float o[MSQ][E];            // normalised head outputs of the pass, (h g) order
  alignas(16) float g[MSQ][E];            // glimpse o W_out^T
  alignas(16) float u[MSQ][CO_POLY_DIM];  // relu(g W1 + c[s % k])
};
static_assert(offsetof(PolyMS, o) == offsetof(LayerMS, o), "the glimpse writes both through LayerMS::o");
template <int SPL>
__host__ __device__ constexpr size_t layer_ms_offset() { return (sizeof(SmemMS<SPL>) + 15) & ~size_t(15); }

// y0 / y1 = x0 / x1 . W[:, c] for a row-major (in, out) [E, E] W in global memory; four partial sums (i mod 4)
__device__ __forceinline__ void layer_matvec2(const float* x0, const float* x1, const float* __restrict__ W, int c,
                                              float& y0, float& y1) {
  float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 2
  for (int i = 0; i < E; i += 4) {
    const float4 u = *reinterpret_cast<const float4*>(x0 + i), v = *reinterpret_cast<const float4*>(x1 + i);
    const float w0 = __ldg(W + (i + 0) * E + c), w1 = __ldg(W + (i + 1) * E + c);
    const float w2 = __ldg(W + (i + 2) * E + c), w3 = __ldg(W + (i + 3) * E + c);
    s0[0] = fmaf(u.x, w0, s0[0]); s0[1] = fmaf(u.y, w1, s0[1]); s0[2] = fmaf(u.z, w2, s0[2]); s0[3] = fmaf(u.w, w3, s0[3]);
    s1[0] = fmaf(v.x, w0, s1[0]); s1[1] = fmaf(v.y, w1, s1[1]); s1[2] = fmaf(v.z, w2, s1[2]); s1[3] = fmaf(v.w, w3, s1[3]);
  }
  y0 = (s0[0] + s0[1]) + (s0[2] + s0[3]);
  y1 = (s1[0] + s1[1]) + (s1[2] + s1[3]);
}

// y[j] = x[j * ldx + .] . W[:, c], j < NJ, for a row-major (in, out) [IN, OUT] W in global memory; four partial sums
// (i mod 4) per row
template <int IN, int OUT, int NJ>
__device__ __forceinline__ void poly_matvec(const float* x, int ldx, const float* __restrict__ W, int c,
                                            float (&y)[NJ]) {
  float s[NJ][4];
#pragma unroll
  for (int j = 0; j < NJ; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll 4
  for (int i = 0; i < IN; i += 4) {
    const float w0 = __ldg(W + (i + 0) * OUT + c), w1 = __ldg(W + (i + 1) * OUT + c);
    const float w2 = __ldg(W + (i + 2) * OUT + c), w3 = __ldg(W + (i + 3) * OUT + c);
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const float4 u = *reinterpret_cast<const float4*>(x + j * ldx + i);
      s[j][0] = fmaf(u.x, w0, s[j][0]); s[j][1] = fmaf(u.y, w1, s[j][1]);
      s[j][2] = fmaf(u.z, w2, s[j][2]); s[j][3] = fmaf(u.w, w3, s[j][3]);
    }
  }
#pragma unroll
  for (int j = 0; j < NJ; ++j) y[j] = (s[j][0] + s[j][1]) + (s[j][2] + s[j][3]);
}

template <int SPL, int ENV, int MODE, bool LAYER = false, bool POLY = false>
__global__ void __launch_bounds__(256, 1) rollout_ms_kernel(const co_rollout_args A) {
  using C = CfgMS<SPL>;
  constexpr int NS = C::NS, TPG = C::TPG, GA = C::GA;
  constexpr int CW = (ENV == CO_ENV_TSP ? 5 : 4) * E;
  constexpr int CUR_BLK = (ENV == CO_ENV_TSP ? 4 : 3);
  constexpr float LOG2E = 1.4426950408889634f, LN2 = 0.6931471805599453f;
  constexpr int Q = MSQ;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SmemMS<SPL>& sm = *reinterpret_cast<SmemMS<SPL>*>(smem_raw);
  [[maybe_unused]] LayerMS& lay = *reinterpret_cast<LayerMS*>(smem_raw + layer_ms_offset<SPL>());  // LAYER only
  [[maybe_unused]] PolyMS& pm = *reinterpret_cast<PolyMS*>(smem_raw + layer_ms_offset<SPL>());     // POLY only

  const int tid = threadIdx.x, lane = tid & 31, h = tid >> 5;
  const int N = A.N, B_inst = A.B_inst, S = A.num_starts, T_max = A.T_max;
  const int B_traj = B_inst * S;
  const bool forced_start = (A.flags & CO_ROLLOUT_FORCED_START) != 0;
  const bool philox = (A.noise == nullptr);
  const int nL = tid % NS;            // selection phase: node of this thread ...
  const int grp = tid / NS;           // ... and its group: trajectories grp * TPG .. grp * TPG + TPG - 1 of the pass
  const bool sel_on = grp < GA;
  const int wsel = (tid % NS) >> 5;   // warp index inside the selection group
  const float clip = A.tanh_clipping, inv_temp = 1.0f / A.temperature;
  const float Zb = clip * inv_temp;

  float2 Kr[SPL][8], Vr[SPL][8];

  for (int b = blockIdx.x; b < B_inst; b += gridDim.x) {
    __syncthreads();
    const float* crow = A.cache + (size_t)b * N * CW;
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
      const int n = lane + 32 * k;
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
    // shared memory <- context table, folded logit key (padded rows), coordinates, demands
    for (int idx = tid; idx < NS * (E / 4); idx += 256) {
      const int n = idx >> 5, c = idx & 31;
      float4 pv = make_float4(0.f, 0.f, 0.f, 0.f), lv = pv;
      if (n < N) {
        pv = __ldg(reinterpret_cast<const float4*>(crow + (size_t)n * CW + CUR_BLK * E) + c);
        lv = __ldg(reinterpret_cast<const float4*>(crow + (size_t)n * CW + 2 * E) + c);
      }
      reinterpret_cast<float4*>(sm.ptab + n * E)[c] = pv;
      sm.lkh[((c >> 2) * 4 + (c & 3)) * NS + n] = lv;  // chunk c = channels 4c..4c+3 = head c / 4, head chunk c % 4
    }
    if (tid < E) {
      sm.ptab[NS * E + tid] = 0.f;
      sm.wcap[tid] = (ENV == CO_ENV_CVRP) ? A.w_capacity[tid] : 0.f;
    }
    if (tid < NS) {
      sm.loc[tid] = (tid < N) ? reinterpret_cast<const float2*>(A.locs)[(size_t)b * N + tid] : make_float2(0.f, 0.f);
      sm.dem[tid] = (ENV == CO_ENV_CVRP && tid >= 1 && tid < N) ? A.demand[(size_t)b * (N - 1) + tid - 1] : 0.f;
    }
    const float cap = (ENV == CO_ENV_CVRP && A.vehicle_capacity) ? A.vehicle_capacity[b] : 1.0f;
    const float thr = cap + 1e-5f;
    __syncthreads();
    if (ENV == CO_ENV_CVRP) {
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
    float dmk[SPL];
#pragma unroll
    for (int k = 0; k < SPL; ++k) dmk[k] = sm.dem[lane + 32 * k];
    const float dL = sm.dem[nL];
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
    float WK[SPL];
#pragma unroll
    for (int k = 0; k < SPL; ++k) WK[k] = 0.f;
    if (ENV == CO_ENV_CVRP) head_dot(sm.wcap, WK);

    for (int g0 = 0; g0 < S; g0 += Q) {
      // ---------------- per-trajectory state (replicated in every thread)
      uint32_t mybits[Q], rmask[Q][ENV == CO_ENV_CVRP ? SPL : 1];
      int cur[Q], prev[Q], first[Q], tstep[Q], dstep[Q], nvis[Q];
      float used[Q], dist[Q], FK[Q][SPL];
      bool anyfeas[Q], fin[Q], depot_seen[Q];
#pragma unroll
      for (int j = 0; j < Q; ++j) {
        mybits[j] = (nL >= N) ? 0x100u : 0u;
#pragma unroll
        for (int k = 0; k < SPL; ++k) mybits[j] |= (lane + 32 * k >= N) ? (1u << k) : 0u;
        if (ENV == CO_ENV_CVRP) {
#pragma unroll
          for (int k = 0; k < SPL; ++k) {
            const int lo = 32 * k, nc = N - 1;
            rmask[j][k] = (nc >= lo + 32) ? 0u : (nc <= lo ? 0xffffffffu : (0xffffffffu << (nc - lo)));
          }
        }
        cur[j] = (ENV == CO_ENV_TSP) ? NS : 0;
        prev[j] = 0; first[j] = 0; tstep[j] = 0; dstep[j] = 0; nvis[j] = 0;
        used[j] = 0.f; dist[j] = 0.f;
        anyfeas[j] = false; depot_seen[j] = false;
        fin[j] = (g0 + j >= S);  // inactive tail trajectories of the last group
      }
      __syncthreads();  // previous group finished with qfix / ll_acc
      if (tid < E) {
        float gq = A.graph_ctx ? A.graph_ctx[(size_t)b * E + tid] : 0.f;
        if (ENV == CO_ENV_TSP && !forced_start) gq += A.q_placeholder[tid];
#pragma unroll
        for (int j = 0; j < Q; ++j) sm.qfix[j][tid] = gq;
      }
      if (tid < Q) sm.ll_acc[tid] = 0.f;

      auto env_step = [&](int j, int a) {
#pragma unroll
        for (int k = 0; k < SPL; ++k) mybits[j] |= (a == lane + 32 * k) ? (1u << k) : 0u;
        mybits[j] |= (a == nL) ? 0x100u : 0u;
        if (h == 0) {
          const float2 pa = sm.loc[a], pp = sm.loc[prev[j]];
          const float dx = pa.x - pp.x, dy = pa.y - pp.y;
          if (ENV == CO_ENV_CVRP || tstep[j] != 0) dist[j] += sqrtf(dx * dx + dy * dy);
        }
        if (ENV == CO_ENV_TSP) {
          if (tstep[j] == 0) first[j] = a;
        } else {
          used[j] = (used[j] + sm.dem[a == 0 ? 1 : a]) * (a != 0 ? 1.0f : 0.0f);
          nvis[j] += (a != 0 || !depot_seen[j]) ? 1 : 0;
          depot_seen[j] = depot_seen[j] || (a == 0);
          if (a != 0) {
            const int r = sm.rank_of[a];
#pragma unroll
            for (int k = 0; k < SPL; ++k) rmask[j][k] |= ((r >> 5) == k) ? (1u << (r & 31)) : 0u;
          }
          int pmin = NS;
#pragma unroll
          for (int k = SPL - 1; k >= 0; --k) {
            const uint32_t z = ~rmask[j][k];
            if (z) pmin = 32 * k + __ffs(z) - 1;
          }
          anyfeas[j] = (pmin < N - 1) && !((sm.dem[sm.order[pmin < N - 1 ? pmin : 0]] + used[j]) > thr);
        }
        prev[j] = a; cur[j] = a; ++tstep[j];
        if ((ENV == CO_ENV_TSP) ? (tstep[j] >= N) : (nvis[j] >= N)) fin[j] = true;
        if (tstep[j] >= T_max) fin[j] = true;
      };

#pragma unroll
      for (int j = 0; j < Q; ++j) {
        if (fin[j]) continue;
        const int s = g0 + j;
        const int traj = s * B_inst + b;
        if (forced_start) {  // decoding.py:309-326 + ops.py:128-149
          const int a0 = (s % A.num_loc) + (ENV == CO_ENV_CVRP ? 1 : 0);
          if (tid == 0) { A.actions_out[(size_t)traj * T_max] = a0; A.logp_out[(size_t)traj * T_max] = 0.f; }
          env_step(j, a0);
          if (ENV == CO_ENV_TSP && tid < E) sm.qfix[j][tid] += __ldg(crow + (size_t)a0 * CW + 3 * E + tid);
        } else if (ENV == CO_ENV_CVRP) {
          anyfeas[j] = !((sm.dem[sm.order[0]] + used[j]) > thr);
        }
      }
      __syncthreads();
#pragma unroll
      for (int j = 0; j < Q; ++j) head_dot(sm.qfix[j], FK[j]);

      while (!(fin[0] && fin[1] && fin[2] && fin[3])) {
        // Every phase is written stage-major over the trajectories in straight-line code (no
        // per-trajectory branches): a warp issues in order, so only interleaved independent
        // instruction streams hide the REDUX / MUFU / shuffle / LDS latencies of each chain.
        // Finished trajectories are computed too (their results are discarded by predication).
        // ---------------- glimpse (warp h = head h), two trajectories at a time (two transpose tiles)
        float rinv[Q];  // 1 / sum(exp) of this head per trajectory: applied to the head's logit shares
#pragma unroll
        for (int jp = 0; jp < Q; jp += 2) {
          float sc[2][SPL], m[2], esum[2];
          uint32_t fzb[2];
          // stage A: scores of both trajectories, feasibility, row max
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int j = jp + u;
            const float4* pr = reinterpret_cast<const float4*>(sm.ptab + cur[j] * E + h * D);
            const float rem = cap - used[j];
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
            float mm = -INFINITY;
            fzb[u] = 0;
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
              const bool f = feasible<ENV>(lane + 32 * k, (mybits[j] >> k) & 1u, dmk[k], used[j], thr, cur[j], anyfeas[j]);
              fzb[u] |= f ? (1u << k) : 0u;
              float dot = (sc2[k].x + sc2[k].y) + FK[j][k];
              if (ENV == CO_ENV_CVRP) dot = fmaf(rem, WK[k], dot);
              sc[u][k] = f ? dot * (0.25f * LOG2E) : -INFINITY;
              mm = fmaxf(mm, sc[u][k]);
            }
            m[u] = mm;
          }
          const unsigned mk0 = __reduce_max_sync(FULL, fkey(m[0])), mk1 = __reduce_max_sync(FULL, fkey(m[1]));
          m[0] = funkey(mk0); m[1] = funkey(mk1);
          // stage B: exp, value accumulation, partial outputs to the trajectory's tile
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            float2 acc[8];
            float es = 0.f;
#pragma unroll
            for (int c = 0; c < 8; ++c) acc[c] = make_float2(0.f, 0.f);
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
              const float e = ((fzb[u] >> k) & 1u) ? ex2(sc[u][k] - m[u]) : 0.f;
              es += e;
              const float2 e2 = make_float2(e, e);
#pragma unroll
              for (int c = 0; c < 8; ++c) acc[c] = ffma2(e2, Vr[k][c], acc[c]);
            }
            esum[u] = es;
            float4* trow = reinterpret_cast<float4*>(sm.tile[h][u] + lane * TILE_LD);
#pragma unroll
            for (int c = 0; c < 4; ++c) trow[c] = make_float4(acc[2 * c].x, acc[2 * c].y, acc[2 * c + 1].x, acc[2 * c + 1].y);
          }
#pragma unroll
          for (int off = 16; off > 0; off >>= 1) {  // both row sums, level by level
            const float t0 = __shfl_xor_sync(FULL, esum[0], off), t1 = __shfl_xor_sync(FULL, esum[1], off);
            esum[0] += t0; esum[1] += t1;
          }
          __syncwarp();
          // stage C: lane sums through the transposed tiles, normalise, publish heads
          const int d = lane & 15, half = lane >> 4;
          float r2[2];
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const float* tile = sm.tile[h][u];
            float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
            for (int r = 0; r < 16; r += 4) {
              s0 += tile[(16 * half + ((r + 0 + 4 * half) & 15)) * TILE_LD + d];
              s1 += tile[(16 * half + ((r + 1 + 4 * half) & 15)) * TILE_LD + d];
              s2 += tile[(16 * half + ((r + 2 + 4 * half) & 15)) * TILE_LD + d];
              s3 += tile[(16 * half + ((r + 3 + 4 * half) & 15)) * TILE_LD + d];
            }
            r2[u] = (s0 + s1) + (s2 + s3);
          }
          const float x0 = __shfl_xor_sync(FULL, r2[0], 16), x1 = __shfl_xor_sync(FULL, r2[1], 16);
          if constexpr (LAYER || POLY) {
            rinv[jp] = __fdividef(1.0f, esum[0]);
            rinv[jp + 1] = __fdividef(1.0f, esum[1]);
            if (lane < 16) {  // normalised head outputs, channel h * D + d
              lay.o[jp][h * D + d] = (r2[0] + x0) * rinv[jp];
              lay.o[jp + 1][h * D + d] = (r2[1] + x1) * rinv[jp + 1];
            }
          } else {
            if (lane < 16) {  // un-normalised head outputs (d == lane here)
              sm.oh[h][jp][d] = r2[0] + x0;
              sm.oh[h][jp + 1][d] = r2[1] + x1;
            }
            rinv[jp] = __fdividef(1.0f, esum[0]);
            rinv[jp + 1] = __fdividef(1.0f, esum[1]);
          }
          __syncwarp();  // the two tiles are reused by the next pair; oh is complete after the last pair
        }
        if constexpr (LAYER) {
          // ---------------- EAS-Lay: o' = o + relu(o W1 + b1) W2 + b2; thread (channel c, trajectories j0, j0 + 1)
          const float* Lw = A.eas_layer + (size_t)b * CO_EAS_LAYER_FLOATS;
          const int c = tid & (E - 1), j0 = 2 * (tid >> 7);
          __syncthreads();  // every head output of the pass is in lay.o
          float y0, y1;
          layer_matvec2(lay.o[j0], lay.o[j0 + 1], Lw, c, y0, y1);
          const float b1 = __ldg(Lw + E * E + c);
          y0 += b1; y1 += b1;
          lay.z[j0][c] = y0 > 0.f ? y0 : 0.f;
          lay.z[j0 + 1][c] = y1 > 0.f ? y1 : 0.f;
          __syncthreads();  // z complete
          layer_matvec2(lay.z[j0], lay.z[j0 + 1], Lw + E * E + E, c, y0, y1);
          const float b2 = __ldg(Lw + 2 * E * E + E + c);
          sm.oh[c >> 4][j0][c & (D - 1)] = lay.o[j0][c] + (y0 + b2);
          sm.oh[c >> 4][j0 + 1][c & (D - 1)] = lay.o[j0 + 1][c] + (y1 + b2);
          __syncthreads();  // o' of every trajectory is in oh
        }
        if constexpr (POLY) {
          // ---------------- PolyNet: g = o W_out^T, u = relu(g W1 + c[s % k]), g' = g + (u W2 + b2)
          constexpr int P = CO_POLY_DIM;
          const float* Pw = A.poly;
          const int c = tid & (E - 1), j0 = 2 * (tid >> 7);
          __syncthreads();  // every head output of the pass is in pm.o
          float y2[2];
          poly_matvec<E, E, 2>(pm.o[j0], E, Pw, c, y2);
          pm.g[j0][c] = y2[0];
          pm.g[j0 + 1][c] = y2[1];
          __syncthreads();  // g complete
          float y4[Q];
          poly_matvec<E, P, Q>(pm.g[0], E, Pw + E * E, tid, y4);
#pragma unroll
          for (int j = 0; j < Q; ++j) {
            const float v = y4[j] + __ldg(Pw + CO_POLY_FIXED_FLOATS + (size_t)((g0 + j) % A.poly_k) * P + tid);
            pm.u[j][tid] = v > 0.f ? v : 0.f;
          }
          __syncthreads();  // u complete
          poly_matvec<P, E, 2>(pm.u[j0], P, Pw + E * E + E * P, c, y2);
          const float b2 = __ldg(Pw + E * E + 2 * E * P + c);
          sm.oh[c >> 4][j0][c & (D - 1)] = pm.g[j0][c] + (y2[0] + b2);
          sm.oh[c >> 4][j0 + 1][c & (D - 1)] = pm.g[j0 + 1][c] + (y2[1] + b2);
          __syncthreads();  // g' of every trajectory is in oh
        }
        // ---------------- head h's share of every pointer logit, for the Q trajectories: the head's slice of the folded
        // logit key is read once per pass (conflict-free LDS.128, lane l = node l + 32 k), the head outputs as broadcasts
        {
          float2 pl2[Q][SPL];
#pragma unroll
          for (int j = 0; j < Q; ++j)
#pragma unroll
            for (int k = 0; k < SPL; ++k) pl2[j][k] = make_float2(0.f, 0.f);
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            float4 l4[SPL];
#pragma unroll
            for (int k = 0; k < SPL; ++k) l4[k] = sm.lkh[(h * 4 + c) * NS + lane + 32 * k];
#pragma unroll
            for (int j = 0; j < Q; ++j) {
              const float4 x = reinterpret_cast<const float4*>(sm.oh[h][j])[c];
#pragma unroll
              for (int k = 0; k < SPL; ++k) {
                pl2[j][k] = ffma2(make_float2(x.x, x.y), make_float2(l4[k].x, l4[k].y), pl2[j][k]);
                pl2[j][k] = ffma2(make_float2(x.z, x.w), make_float2(l4[k].z, l4[k].w), pl2[j][k]);
              }
            }
          }
#pragma unroll
          for (int j = 0; j < Q; ++j)
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
              if constexpr (LAYER || POLY) sm.part[j][h][lane + 32 * k] = pl2[j][k].x + pl2[j][k].y;  // o' / g' are normalised
              else sm.part[j][h][lane + 32 * k] = (pl2[j][k].x + pl2[j][k].y) * rinv[j];
            }
        }
        __syncthreads();  // B1: every head's share of every logit of all trajectories is in shared memory

        // ---------------- selection: thread (node nL, group grp) handles trajectories grp * TPG + jj
        float z[TPG];
        if (sel_on) {
          float keyf[TPG], ex[TPG];
#pragma unroll
          for (int jj = 0; jj < TPG; ++jj) {
            const int j = grp * TPG + jj;
            const float pl = ((sm.part[j][0][nL] + sm.part[j][1][nL]) + (sm.part[j][2][nL] + sm.part[j][3][nL])) +
                             ((sm.part[j][4][nL] + sm.part[j][5][nL]) + (sm.part[j][6][nL] + sm.part[j][7][nL]));
            // the per-trajectory state of every trajectory is replicated in all threads: index it with a compile-time
            // loop so that it stays in registers
            uint32_t mb = 0; float usedj = 0.f; int curj = 0; bool anyj = false; int dstepj = 0;
#pragma unroll
            for (int q = 0; q < Q; ++q)
              if (q == j) { mb = mybits[q]; usedj = used[q]; curj = cur[q]; anyj = anyfeas[q]; dstepj = dstep[q]; }
            const bool fzL = feasible<ENV>(nL, (mb >> 8) & 1u, dL, usedj, thr, curj, anyj);
            const float lg = tanhf(pl * 0.08838834764831845f) * clip;
            z[jj] = fzL ? lg * inv_temp : -INFINITY;
            keyf[jj] = z[jj];
            if (MODE == CO_MODE_SAMPLE) {
              keyf[jj] = -INFINITY;
              if (fzL) {
                const int traj = (g0 + j) * B_inst + b;
                const float q = philox ? philox_exp1(A.seed, A.offset, traj, dstepj, nL)
                                       : A.noise[((size_t)dstepj * B_traj + (traj < B_traj ? traj : 0)) * N + nL];
                keyf[jj] = z[jj] - logf(q);
              }
            }
            ex[jj] = ex2((z[jj] - Zb) * LOG2E);
          }
#pragma unroll
          for (int off = 16; off > 0; off >>= 1) {  // the partial sums, level by level
#pragma unroll
            for (int jj = 0; jj < TPG; ++jj) ex[jj] += __shfl_xor_sync(FULL, ex[jj], off);
          }
          unsigned wkey[TPG], vote[TPG];
#pragma unroll
          for (int jj = 0; jj < TPG; ++jj) wkey[jj] = __reduce_max_sync(FULL, fkey(keyf[jj]));
#pragma unroll
          for (int jj = 0; jj < TPG; ++jj) vote[jj] = __ballot_sync(FULL, fkey(keyf[jj]) == wkey[jj]);
          if (lane == 0) {
#pragma unroll
            for (int jj = 0; jj < TPG; ++jj) {
              const int j = grp * TPG + jj;
              sm.red_key[j][wsel] = wkey[jj];
              sm.red_idx[j][wsel] = 32 * wsel + __ffs(vote[jj]) - 1;
              sm.red_sum[j][wsel] = ex[jj];
            }
          }
        }
        __syncthreads();  // B2: per-warp partials of all trajectories complete
        bool need_sync = false;
#pragma unroll
        for (int j = 0; j < Q; ++j) {
          const int traj = (g0 + j) * B_inst + b;
          int a;
          float Ssum;
          {  // SPL selection warps per trajectory; entries beyond SPL are never written nor read
            const uint4 k0 = *reinterpret_cast<const uint4*>(sm.red_key[j]);
            const int4 i0 = *reinterpret_cast<const int4*>(sm.red_idx[j]);
            const float4 u0 = *reinterpret_cast<const float4*>(sm.red_sum[j]);
            unsigned bk = k0.x; a = i0.x; Ssum = u0.x;  // strict '>' keeps the lowest warp (= lowest node) on ties
            if (SPL >= 2) { Ssum += u0.y; if (k0.y > bk) { bk = k0.y; a = i0.y; } }
            if (SPL >= 4) {
              Ssum = (u0.x + u0.y) + (u0.z + u0.w);
              if (k0.z > bk) { bk = k0.z; a = i0.z; }
              if (k0.w > bk) { bk = k0.w; a = i0.w; }
            }
          }
          if (!fin[j]) {  // uniform across the block: the state is replicated
            const int t = tstep[j];
            if (MODE == CO_MODE_EVALUATE) {
              const int forced = (int)A.forced_actions[(size_t)traj * T_max + t];
              a = (forced < 0 || forced >= N) ? 0 : forced;
            }
            if (sel_on && nL == a && j / TPG == grp) {
              const float lpL = (z[j % TPG] - Zb) - lg2(Ssum) * LN2;
              A.logp_out[(size_t)traj * T_max + t] = lpL;
              sm.ll_acc[j] += lpL;
            }
            if (tid == 0) A.actions_out[(size_t)traj * T_max + t] = a;
            const bool was_first = (ENV == CO_ENV_TSP) && (t == 0);
            env_step(j, a);
            ++dstep[j];
            if (was_first) {  // multisample without forced start: context becomes [h_first ; h_cur]
              if (tid < E) sm.qfix[j][tid] = (A.graph_ctx ? A.graph_ctx[(size_t)b * E + tid] : 0.f) +
                                             __ldg(crow + (size_t)a * CW + 3 * E + tid);
              need_sync = true;
            }
          }
        }
        if (need_sync) {  // uniform: tstep is replicated
          __syncthreads();
#pragma unroll
          for (int j = 0; j < Q; ++j) head_dot(sm.qfix[j], FK[j]);
        }
      }

      // ---------------- epilogue of the group
      __syncthreads();
#pragma unroll
      for (int j = 0; j < Q; ++j) {
        if (g0 + j >= S) continue;
        const int traj = (g0 + j) * B_inst + b;
        const int t = tstep[j];
        if (tid == 0) {
          const float2 pa = sm.loc[(ENV == CO_ENV_TSP) ? first[j] : 0], pp = sm.loc[prev[j]];
          const float dx = pa.x - pp.x, dy = pa.y - pp.y;
          A.reward_out[traj] = -(dist[j] + sqrtf(dx * dx + dy * dy));
          A.loglik_out[traj] = sm.ll_acc[j];
          if (A.steps_out) A.steps_out[traj] = t;
          if (A.used_capacity_out) A.used_capacity_out[traj] = used[j];
          if (A.max_steps_out) atomicMax(A.max_steps_out, t);
        }
        for (int c = t + tid; c < T_max; c += 256) {
          A.actions_out[(size_t)traj * T_max + c] = 0;
          A.logp_out[(size_t)traj * T_max + c] = 0.f;
        }
      }
    }
  }
}

template <int SPL, int ENV, int MODE, bool LAYER, bool POLY = false>
static int launch_ms(const co_rollout_args& A, cudaStream_t st) {
  auto kern = rollout_ms_kernel<SPL, ENV, MODE, LAYER, POLY>;
  const size_t smem = LAYER ? layer_ms_offset<SPL>() + sizeof(LayerMS)
                            : (POLY ? layer_ms_offset<SPL>() + sizeof(PolyMS) : sizeof(SmemMS<SPL>));
  static PerDeviceOnce once;
  bool& configured = once.flag();
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail(CO_ERR_CUDA, "co_rollout(ms): smem attribute: %s", cudaGetErrorString(e));
    configured = true;
  }
  int grid = device_info().sm_count;
  if (grid > A.B_inst) grid = A.B_inst;
  kern<<<grid, 256, smem, st>>>(A);
  return check_launch("co_rollout(ms)");
}

template <int ENV>
static int dispatch_ms(const co_rollout_args& A, cudaStream_t st) {
  const int spl = A.N <= 32 ? 1 : (A.N <= 64 ? 2 : 4);
  const int mode = A.select_mode == CO_SELECT_GREEDY ? CO_MODE_GREEDY
                   : (A.select_mode == CO_SELECT_EVALUATE ? CO_MODE_EVALUATE : CO_MODE_SAMPLE);
  const bool layer = A.eas_layer != nullptr, poly = A.poly != nullptr;
#define CO_CASE(S_, M_)                                                                      \
  if (spl == S_ && mode == M_)                                                               \
  return layer ? launch_ms<S_, ENV, M_, true>(A, st)                                         \
               : (poly ? launch_ms<S_, ENV, M_, false, true>(A, st) : launch_ms<S_, ENV, M_, false>(A, st))
  CO_CASE(1, CO_MODE_GREEDY); CO_CASE(2, CO_MODE_GREEDY); CO_CASE(4, CO_MODE_GREEDY);
  CO_CASE(1, CO_MODE_SAMPLE); CO_CASE(2, CO_MODE_SAMPLE); CO_CASE(4, CO_MODE_SAMPLE);
  CO_CASE(1, CO_MODE_EVALUATE); CO_CASE(2, CO_MODE_EVALUATE); CO_CASE(4, CO_MODE_EVALUATE);
#undef CO_CASE
  return fail(CO_ERR_BAD_ARG, "co_rollout(ms): no kernel variant%s");
}

}  // namespace co
