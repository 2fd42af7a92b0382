/*
 * corollout.h -- C ABI of libcorollout.so, the H100 (sm_90a) rollout engine behind
 * rl4co's env / decoder API.
 *
 * The reference (ai4co/rl4co) is 100% Python and has no FFI on this path; its only FFI
 * precedent is ctypes -> libhgscvrp.so (rl4co/envs/routing/cvrp/local_search.py:8-24).
 * Each entry point below replaces the reference function(s) cited next to it; the
 * Python-side ctypes binding a maintainer would add is shown in INTEGRATION.md and
 * implemented in rl4co_b200/native.py.
 *
 * Conventions (SURVEY.md section 8b)
 *   - every pointer is a DEVICE pointer into memory owned by the caller (PyTorch);
 *     the library never allocates, frees or retains device memory;
 *   - tensors are contiguous row-major with exactly the reference TensorDict dtypes:
 *     int64 actions / node ids, 1-byte bool masks, uint8 visited, float32 the rest;
 *   - all work is enqueued asynchronously on `stream` (a cudaStream_t passed as void*);
 *     no call synchronises the device;
 *   - return value: CO_OK (0) or a negative CO_ERR_*; co_last_error_string() describes
 *     the last failure on the calling thread.  No C++ exception crosses the boundary.
 *   - embed_dim E = 128, heads H = 8 (head dim 16) are compile-time constants of the
 *     AttentionModel this path serves (rl4co/models/zoo/am/policy.py:50-56).
 */
#ifndef COROLLOUT_H_
#define COROLLOUT_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CO_VERSION 100 /* 0.1.0 */

#define CO_OK 0
#define CO_ERR_BAD_ARG (-1)
#define CO_ERR_UNSUPPORTED (-2) /* shape outside what a kernel is instantiated for */
#define CO_ERR_CUDA (-3)        /* launch / runtime error; see co_last_error_string */

#define CO_EMBED_DIM 128
#define CO_NUM_HEADS 8

/* environment kinds (env.name in the reference: "tsp", "cvrp") */
#define CO_ENV_TSP 0
#define CO_ENV_CVRP 1
#define CO_ENV_SDVRP 2 /* split-delivery VRP: VRP context + dynamic embedding */
#define CO_ENV_OP 3    /* orienteering: budget context, length mask, prize reward (co_rollout; the step kernels are co_op_*) */
#define CO_ENV_PCTSP 4 /* prize-collecting TSP: remaining-prize context, depot rule on the collected prize (co_pctsp_*) */

/* action-selection modes (rl4co/utils/decoding.py:426-461) */
#define CO_SELECT_GREEDY 0       /* Greedy._step: argmax, first index on ties            */
#define CO_SELECT_SAMPLE_NOISE 1 /* Sampling._step with caller-supplied Exp(1) draws q:    */
                                 /*   argmax(exp(logp)/q) == torch.multinomial(p,1)        */
#define CO_SELECT_EVALUATE 2     /* Evaluate._step: action supplied, only logp computed    */
#define CO_SELECT_SAMPLE_PHILOX 3/* Sampling with in-kernel Philox4x32-10 Exp(1) draws     */

int co_version(void);
const char* co_last_error_string(void);
/* number of SMs / max dyn smem of the current device (cached); used to size grids */
int co_device_sm_count(void);

/* ------------------------------------------------------------------ environments */

/* TSPEnv._step  (rl4co/envs/routing/tsp/env.py:60-86)
 *   mask_out = mask_in with column action[b] cleared; done = no column left;
 *   first_node = action where i[b]==0 else kept; current_node = action; i += 1.
 * mask_in may alias mask_out (in-place step). */
int co_tsp_step(const int64_t* action, const uint8_t* mask_in, uint8_t* mask_out,
                int64_t* first_node, int64_t* current_node, int64_t* i, uint8_t* done,
                int B, int N, void* stream);

/* CVRPEnv.get_action_mask  (rl4co/envs/routing/cvrp/env.py:126-136)
 *   N counts the depot (node 0); demand is [B, N-1]; mask_out[b,n]=1 means feasible. */
int co_cvrp_action_mask(const float* demand, const float* used_capacity,
                        const float* vehicle_capacity, const uint8_t* visited,
                        const int64_t* current_node, uint8_t* mask_out, int B, int N,
                        void* stream);

/* CVRPEnv._step  (rl4co/envs/routing/cvrp/env.py:66-96), including the trailing
 * get_action_mask.  visited_in may alias visited_out, used_in may alias used_out. */
int co_cvrp_step(const int64_t* action, const float* demand, const float* vehicle_capacity,
                 const float* used_in, float* used_out, const uint8_t* visited_in,
                 uint8_t* visited_out, int64_t* current_node, uint8_t* done,
                 uint8_t* mask_out, int B, int N, void* stream);

/* TSPEnv._get_reward / CVRPEnv._get_reward
 * (tsp/env.py:150-156, cvrp/env.py:138-147 -> rl4co/utils/ops.py:54-90)
 *   reward[b] = - sum_t || x[a_{t+1}] - x[a_t] ||_2 over the cyclic tour; with_depot=1
 *   prepends node 0 (CVRP).  locs [B_locs,N,2]; actions [B,T]; trajectory j uses
 *   instance j % B_locs (multistart / augmentation share locs). */
/* SDVRPEnv (rl4co/envs/routing/sdvrp/env.py): `demand_with_depot` [B,N] f32 is the dynamic state (depot entry 0).
 * co_sdvrp_step = _step :55-82 (deliver min(demand, capacity - used), scatter_add, done) + get_action_mask :110-116;
 * outputs may alias inputs (in-place update). */
int co_sdvrp_action_mask(const float* demand_with_depot, const float* used_capacity,
                         const float* vehicle_capacity, const int64_t* current_node, uint8_t* mask_out,
                         int B, int N, void* stream);
int co_sdvrp_step(const int64_t* action, const float* demand_in, float* demand_out,
                  const float* vehicle_capacity, const float* used_in, float* used_out,
                  int64_t* current_node, uint8_t* done, uint8_t* mask_out, int B, int N, void* stream);

/* OPEnv (rl4co/envs/routing/op/env.py; sibling env, orienteering): locs [B,N,2] with the depot at 0, prize [B,N] (depot 0),
 * max_length [B,N] (per node: the budget minus the way back to the depot, env.py:121-123), visited [B,N] bool,
 * tour_length / current_total_prize [B] f32, current_node / i [B] i64 (updated in place by co_op_step).
 * co_op_step = _step :72-105 + get_action_mask :140-155 (done = depot re-entered after step 0);
 * co_op_reward = _get_reward :157-165 (sum of the collected prizes over actions [B,T]). */
int co_op_action_mask(const float* locs, const float* max_length, const uint8_t* visited, const float* tour_length,
                      const int64_t* current_node, uint8_t* mask_out, int B, int N, void* stream);
int co_op_step(const int64_t* action, const float* locs, const float* prize, const float* max_length,
               const uint8_t* visited_in, uint8_t* visited_out, float* tour_length, float* current_total_prize,
               int64_t* current_node, int64_t* i, uint8_t* done, uint8_t* mask_out, int B, int N, void* stream);
int co_op_reward(const float* prize, const int64_t* actions, float* reward, int B, int N, int T, void* stream);

/* PCTSPEnv (rl4co/envs/routing/pctsp/env.py; sibling env, prize-collecting TSP): real_prize / penalty [B,N] (depot 0),
 * visited [B,N] bool, cur_total_prize / cur_total_penalty [B] f32, current_node / i [B] i64 (in place).
 * co_pctsp_step = _step :62-93 + get_action_mask :143-151; the reward (:153-172) is co_op_reward over the penalties plus
 * co_tour_length. */
int co_pctsp_action_mask(const uint8_t* visited, const float* cur_total_prize, uint8_t* mask_out, int B, int N, void* stream);
int co_pctsp_step(const int64_t* action, const float* real_prize, const float* penalty, const uint8_t* visited_in,
                  uint8_t* visited_out, float* cur_total_prize, float* cur_total_penalty, int64_t* current_node, int64_t* i,
                  uint8_t* done, uint8_t* mask_out, int B, int N, void* stream);

int co_tour_length(const float* locs, const int64_t* actions, float* reward, int B,
                   int B_locs, int N, int T, int with_depot, void* stream);

/* TSPEnv.check_solution_validity / CVRPEnv.check_solution_validity
 * (tsp/env.py:158-164, cvrp/env.py:149-177).  *bad_count (device int32, caller-zeroed)
 * receives the number of invalid tours; demand==NULL selects the TSP rule. */
int co_check_tours(const int64_t* actions, const float* demand,
                   const float* vehicle_capacity, int32_t* bad_count, int B, int B_inst,
                   int N, int T, void* stream);

/* TSPEnv.local_search  (rl4co/envs/routing/tsp/env.py:184-188 -> tsp/local_search.py)
 *   best-improvement 2-opt with position 0 fixed, bit-identical to the reference: per sweep the first pair (i, j) in
 *   loop order with the smallest fp32 change below -1e-6 has t[i..j] reversed; sweeps repeat until none improves or
 *   max_iterations sweeps have run (<= 0: tours copied unchanged).
 *   Distances: exactly one of
 *     locs [B,N,2]  -> d[a,b] = sqrt(fma(dy, dy, dx*dx)), dx = x_a - x_b (get_distance_matrix on the CPU), or
 *     dist [B,N,N]  -> used as given, possibly asymmetric;
 *   the diagonal gets +1e9 in both cases.  The matrix is held in shared memory up to CO_TWO_OPT_RESIDENT_MAX_NODES
 *   nodes (locs: computed there), above that read through L2 (dist) or computed per read from locs.
 *   tours_in / tours_out [B,N] int64, and tours_out may alias tours_in.  A tour holding an id outside [0, N) is
 *   copied through unchanged with iterations[b] = -1.  iterations [B] (nullable) receives the number of sweeps run.
 *   N > CO_TWO_OPT_MAX_NODES returns CO_ERR_UNSUPPORTED. */
#define CO_TWO_OPT_MAX_NODES 1024
#define CO_TWO_OPT_RESIDENT_MAX_NODES 224 /* 224*224*4 B = 196 KiB of the 227 KiB a CTA may use */
int co_tsp_two_opt(const float* locs, const float* dist, const int64_t* tours_in, int64_t* tours_out,
                   int32_t* iterations, int B, int N, int max_iterations, void* stream);

/* CVRPEnv.local_search  (rl4co/envs/routing/cvrp/env.py -> cvrp/local_search.py): the project's own deterministic
 * local search behind the reference's signature and output layout.  It is not HGS-CVRP's SWAP*.
 *   Inputs: N customers; tours_in [B,T] int64 in the action format (0 = depot; leading, trailing and repeated zeros
 *   allowed); demand [B,N] (customers, already divided by the capacity); capacity [B]; exactly one of
 *     locs [B,N+1,2]   -> d[a,b] = sqrt(fma(dy, dy, dx*dx)), dx = x_a - x_b (get_distance_matrix on the CPU), or
 *     dist [B,N+1,N+1] -> used as given (possibly asymmetric); the diagonal is read as given (d[0][0] = 0 from locs).
 *   Routes: the maximal runs of customers of the tour, numbered in input order (slot r); each keeps its slot, a start
 *   depot with id N+1+r and an end depot, also when a move empties it (it may be refilled; no route is added).  A
 *   depot id reads row / column 0.  p(x) / s(x) are the predecessor / successor within the route.  The load of a route
 *   is the fp32 left-to-right sum of its demands in route order, recomputed after every move for the routes it changed;
 *   pre(x) is the load up to and including x (0 at a start depot).  lim = capacity + 1e-5f.
 *   Search: best improvement.  A sweep scores every candidate below in fp32, each operation rounded on its own in the
 *   order parenthesised, and takes the smallest key (delta, kind, u, v); the move is applied when delta < -1e-6 (as a
 *   double).  Sweeps repeat until none improves or max_iterations moves have been applied (<= 0: no move).
 *     kind 0 relocate  u customer, v customer or start depot, v not in {u, p(u)}: u moves after v.
 *       delta = ((d[pu][su] - d[pu][u]) - d[u][su]) + ((d[v][u] + d[u][sv]) - d[v][sv])
 *       admissible: same route: load <= lim; else load(u's) - dem[u] <= lim and load(v's) + dem[u] <= lim
 *     kind 1 swap      customers u < v, su != v and sv != u: u and v exchange places.
 *       delta = (((d[pu][v] + d[v][su]) - d[pu][u]) - d[u][su]) + (((d[pv][u] + d[u][sv]) - d[pv][v]) - d[v][sv])
 *       admissible: same route: load <= lim; else (load(u's) - dem[u]) + dem[v] <= lim and
 *       (load(v's) - dem[v]) + dem[u] <= lim
 *     kind 2 2-opt     u (customer or start depot) before customer v in one route, su != v: su..v is reversed.
 *       delta = ((d[u][v] + d[su][sv]) - d[u][su]) - d[v][sv]                  admissible: load <= lim
 *     kind 3 2-opt*    u in route A, v in route B, A < B, not both start depots, su and sv not both end depots:
 *       A becomes A[..u] + B[sv..], B becomes B[..v] + A[su..].
 *       delta = ((d[u][sv] + d[v][su]) - d[u][su]) - d[v][sv]
 *       admissible: pre(u) + (load(B) - pre(v)) <= lim and pre(v) + (load(A) - pre(u)) <= lim
 *   Outputs: tours_out [B,2N] int64 as the reference's merge_subroutes without its leading column: the non-empty
 *   routes in slot order, one 0 between routes, no leading 0, zero padding; used_len [B] int32 = entries before the
 *   padding.  iterations [B] (nullable): moves applied.  feasible [B] (nullable): 1 when tours_out passes the capacity
 *   rule of CVRPEnv.check_solution_validity (running load, a depot visit subtracts the capacity and clamps at 0, load
 *   <= capacity + 1e-5 after every step), else 0.  A row holding an id outside [0, N], or that does not visit every
 *   customer exactly once, is copied through (its first min(T, 2N) entries, then zeros) with used_len = min(T, 2N),
 *   iterations = -1 and feasible = 0.  tours_out must not overlap tours_in.
 *   Errors: a null pointer, both or neither of locs / dist, B < 0, N < 1, T < 1, or a pointer not aligned to its
 *   element (8 bytes for locs) is CO_ERR_BAD_ARG; N + 1 > CO_TWO_OPT_MAX_NODES is CO_ERR_UNSUPPORTED.  The matrix is
 *   held in shared memory up to N + 1 = CO_TWO_OPT_RESIDENT_MAX_NODES nodes; every path gives the same tours. */
int co_cvrp_local_search(const float* locs, const float* dist, const float* demand, const float* capacity,
                         const int64_t* tours_in, int64_t* tours_out, int32_t* used_len, int32_t* iterations,
                         int32_t* feasible, int B, int N, int T, int max_iterations, void* stream);

/* ------------------------------------------------------------------ decoder, one step */

/* Weights of the decoder path, device pointers, all float32, no biases
 * (rl4co/models/zoo/am/policy.py:65,70).  *_t tensors are TRANSPOSED copies
 * ([in, out] row-major) prepared once per weight update by the host side.
 * pointer.project_out is not among them: it is folded into logit_key (see co_pointer_logits). */
typedef struct co_decoder_weights {
  const float* project_context_t; /* [ctx_dim, E]; ctx_dim = 2E (tsp) or E+1 (cvrp)   */
  const float* w_placeholder;     /* [2E] (tsp only, else NULL)                       */
  /* dynamic embedding (sdvrp: SDVRPDynamicEmbedding, nn/env_embeddings/dynamic.py:60-78; am/decoder.py:142-154):
   * glimpse_key / glimpse_val / logit_key of node n get + dynamic_feature[j, n] * dynamic_w[0:E | E:2E | 2E:3E].
   * Both NULL for static embeddings (tsp, cvrp). */
  const float* dynamic_w;         /* [3E] = projection.weight[:, 0], the logit third folded with project_out    */
                                  /* (W_out^T w_l)                                                              */
  const float* dynamic_feature;   /* [B_traj, N] per-step node feature (sdvrp: remaining demand, depot = 0)     */
} co_decoder_weights;

/* AttentionModelDecoder.forward (rl4co/models/zoo/am/decoder.py:156-193):
 * context embedding (nn/env_embeddings/context.py:116-134 | 61-74,147-149) + graph
 * context, PointerAttention (nn/attention.py:274-320) -> raw logits [B_traj, N]
 * (unmasked, unclipped, already in the reference's "(s b) l" order).
 * Trajectory j reads the cache of instance j % B_inst (multistart shares K/V/L).
 *   tsp : first_node, current_node [B_traj] int64, i [B_traj] int64 (i==0 -> placeholder)
 *   cvrp: current_node [B_traj] int64, used_capacity / vehicle_capacity [B_traj] f32
 * glimpse_key / glimpse_val / logit_key rows are `ld` floats apart (ld = E for the
 * reference's contiguous tensors, or the fused-cache row width for views into it; 0 = E).
 * logit_key holds the folded rows logit_key @ project_out.weight (block 2 of the rollout cache),
 * so the glimpse is the concatenated head output itself. */
int co_pointer_logits(int env_kind, const co_decoder_weights* w, const float* node_emb,
                      const float* graph_ctx /* [B_inst,E] or NULL */,
                      const float* glimpse_key, const float* glimpse_val,
                      const float* logit_key, const uint8_t* action_mask,
                      const int64_t* first_node, const int64_t* current_node,
                      const int64_t* i, const float* used_capacity,
                      const float* vehicle_capacity, float* logits_out, int B_traj,
                      int B_inst, int N, int ld, void* stream);

/* DecodingStrategy.step (rl4co/utils/decoding.py:344-385): process_logits (:138-188:
 * tanh clip, mask -> -inf, temperature, log_softmax; top-k/top-p unsupported) then
 * Greedy / Sampling / Evaluate selection and logp gather.
 *   noise        : [B,N] Exp(1) draws for CO_SELECT_SAMPLE_NOISE, else NULL
 *   action_io    : [B] int64; read for CO_SELECT_EVALUATE, written otherwise
 *   logprobs_out : optional [B,N] full log-probabilities (store_all_logp), or NULL */
int co_select_action(const float* logits, const uint8_t* action_mask, const float* noise,
                     int64_t* action_io, float* logp_out, float* logprobs_out, int mode,
                     float tanh_clipping, float temperature, int mask_logits,
                     uint64_t seed, uint64_t offset, int B, int N, void* stream);

/* ------------------------------------------------------------------ whole-episode rollout */

/* Persistent fused rollout: replaces the whole `while not td["done"].all()` loop of
 * ConstructivePolicy.forward (rl4co/models/common/constructive/base.py:219-251):
 * decoder.forward + strategy.step + env.step per node selection, then
 * post_decoder_hook / get_reward / get_log_likelihood, in ONE kernel launch with no host
 * synchronisation.  One CTA owns one instance for the whole episode: its glimpse-key /
 * glimpse-value / folded logit-key rows live in registers, the per-node context table in
 * shared memory; the visited set is a bitmask in registers.
 *
 * The cache is the layout written by FusedAttentionModelDecoder._precompute_cache:
 *   cache[B_inst][N][co_cache_width(env_kind)] float32, column blocks of E floats:
 *     0: glimpse_key   1: glimpse_val   2: logit_key @ project_out (folded)
 *     3: node_emb @ Wctx[:, :E]^T  (tsp: "first node" table; other envs: current-node table)
 *     4: node_emb @ Wctx[:, E:2E]^T (tsp only: current-node table)
 */
#define CO_ROLLOUT_FORCED_START 1 /* S>1: first action of start s is forced (multistart) */

typedef struct co_rollout_args {
  int32_t env_kind;     /* CO_ENV_*                                                    */
  int32_t select_mode;  /* CO_SELECT_*                                                 */
  int32_t B_inst;       /* instances (cache rows)                                      */
  int32_t num_starts;   /* S >= 1 trajectories per instance; S > 1 = multistart with   */
                        /* forced first action s % num_loc (+1 for cvrp), ops.py:128-149 */
  int32_t N;            /* nodes incl. depot                                           */
  int32_t T_max;        /* columns of actions_out / logp_out (tsp: N, cvrp: 2(N-1))     */
  int32_t num_loc;      /* generator.num_loc used by select_start_nodes                */
  int32_t flags;        /* CO_ROLLOUT_* bits                                           */
  float tanh_clipping;  /* 10.0 for AM                                                 */
  float temperature;    /* 1.0                                                         */
  const float* cache;        /* [B_inst, N, W]                                         */
  const float* graph_ctx;    /* [B_inst, E] or NULL (POMO: use_graph_context=False)    */
  const float* q_placeholder;/* [E] = Wctx @ W_placeholder (tsp step-0 context)        */
  const float* w_capacity;   /* [E] = Wctx[:, E] (cvrp remaining-capacity column)      */
  const float* locs;         /* [B_inst, N, 2]                                         */
  const float* demand;       /* [B_inst, N-1] (cvrp) or NULL                           */
  const float* vehicle_capacity; /* [B_inst] (cvrp) or NULL (=1.0)                     */
  const int64_t* forced_actions; /* [B_traj, T_max] for CO_SELECT_EVALUATE else NULL   */
  const float* noise;        /* [T_max, B_traj, N] Exp(1) for CO_SELECT_SAMPLE_NOISE   */
  uint64_t seed, offset;     /* Philox stream for CO_SELECT_SAMPLE_PHILOX              */
  int64_t* actions_out;      /* [B_traj, T_max]; B_traj = S * B_inst, row j = s*B + b  */
  float* logp_out;           /* [B_traj, T_max] per-step log-prob of the chosen action */
  float* reward_out;         /* [B_traj]  = -tour length                               */
  float* loglik_out;         /* [B_traj]  = sum_t logp                                 */
  int32_t* steps_out;        /* [B_traj]  decode steps until done (incl. forced start) */
  int32_t* max_steps_out;    /* [1] device int32, caller-zeroed: max over trajectories */
  float* used_capacity_out;  /* [B_traj] final used capacity (cvrp) or NULL            */
  int32_t cache_width;       /* floats per row of `cache`, must equal                   */
                             /* co_cache_width(env_kind); 0 = that width                 */
  int32_t reserved0;         /* keeps the pointers below 8-byte aligned                  */
  /* sdvrp: dynamic-embedding weights [wk | wv | W_out^T wl] = SDVRPDynamicEmbedding.projection.weight[:, 0] with
   * the logit third folded like block 2 of the cache (nn/env_embeddings/dynamic.py:60-78); NULL otherwise */
  const float* dyn_w;        /* [3E] */
  /* op: per-node length budget max_length [B_inst, N] (op/env.py:121-123); `demand` carries the customers' prizes
   * [B_inst, N-1], `vehicle_capacity` the budget at the depot max_length[:, 0], reward_out the collected prize;
   * pctsp: penalty per node [B_inst, N] (depot 0); `demand` = real prizes [B_inst, N-1], `vehicle_capacity` = prize_required */
  const float* node_limit;
  /* EAS-Lay (rl4co/models/zoo/eas/nn.py, decoder.py:12-31): per-instance residual layer on the concatenated head output
   * o (E channels, (h g) order) of every decode step of every trajectory of instance b, before project_out:
   *   o' = o + relu(o W1 + b1) W2 + b2,  u_n = o' . Lf[n] / sqrt(E)
   * packed [B_inst, CO_EAS_LAYER_FLOATS] fp32 as [W1 (E x E, (in, out)) | b1 (E) | W2 (E x E, (in, out)) | b2 (E)],
   * 16-byte aligned.  NULL: no layer.  Non-NULL only for tsp / cvrp with num_starts > 1 (else CO_ERR_UNSUPPORTED);
   * misaligned: CO_ERR_BAD_ARG. */
  const float* eas_layer;
  /* PolyNet (Hottung et al. 2024; rl4co/models/nn/attention.py PolyNetAttention): the glimpse g = o W_out^T of every
   * decode step of trajectory s goes through one residual MLP conditioned on strategy s % poly_k,
   *   g' = g + (relu(g W1 + c[s % poly_k]) W2 + b2),  u_n = g' . L[n] / sqrt(E)
   * with c[i] = b1 + poly_layer_1.weight[:, E:] . binary_vector[i] and L the UN-folded logit key (block 2 of the cache
   * holds L itself, not L W_out).  Weights shared by every instance, packed fp32 and 16-byte aligned as
   *   [W_out^T (E x E) | W1 (E x P) | W2 (P x E) | b2 (E) | c (poly_k x P)],  P = CO_POLY_DIM, matrices (in, out),
   * CO_POLY_FIXED_FLOATS + poly_k * CO_POLY_DIM floats.  NULL: no poly layer (poly_k is then not read).  Non-NULL only
   * for tsp / cvrp with num_starts > 1 and eas_layer NULL (else CO_ERR_UNSUPPORTED); misaligned or poly_k < 1:
   * CO_ERR_BAD_ARG. */
  const float* poly;
  int32_t poly_k;
  int32_t reserved1;
} co_rollout_args;
#define CO_EAS_LAYER_FLOATS (2 * CO_EMBED_DIM * CO_EMBED_DIM + 2 * CO_EMBED_DIM)
#define CO_POLY_DIM 256
#define CO_POLY_FIXED_FLOATS (CO_EMBED_DIM * CO_EMBED_DIM + 2 * CO_EMBED_DIM * CO_POLY_DIM + CO_EMBED_DIM)

/* Efficient active search, embedding variant (EAS-Emb; rl4co/models/zoo/eas/search.py:198-235): gradient of a
 * weighted sum of trajectory log-likelihoods with respect to the folded logit key Lf = L W_out (block 2 of the cache).
 *   Row j = r * B_inst + b (r < num_rows, start-major as co_rollout) is a trajectory of instance b: actions [R*B_inst, T]
 *   int64, column 0 a forced first action (tsp: any node, cvrp: a customer) with log-prob 0, as a multistart start;
 *   columns after the episode is done are padding and are not read.  Each step t >= 1 is replayed as co_rollout in
 *   evaluate mode: query = graph_ctx + current-node table row (tsp: + the first-node table row of column 0; cvrp:
 *   + (capacity - used) * w_capacity), masked 8-head glimpse -> head output o_t [E], u_n = o_t . Lf[n] / sqrt(E),
 *   z_n = C tanh(u_n) / temperature (masked: -inf), logp = log_softmax(z).  Outputs:
 *     loglik[j] = sum_t logp_t[a_t]
 *     dLf[b, n, :] = sum over the rows j of b and their steps t of  g_{j,t,n} o_{j,t},
 *       g_{j,t,n} = coef[j] (delta_{n,a_t} - p_{t,n}) / temperature * C (1 - tanh^2(u_n)) / sqrt(E)  (0 if n is masked)
 *     i.e. dLf = d(sum_j coef[j] loglik[j]) / dLf.
 *   One CTA owns one instance; every dLf entry is summed in the fixed order (row, step) by one thread, so the result is
 *   bit-identical across launches and does not depend on the other instances of the batch.  No placeholder query is
 *   needed: column 0 is always forced.
 *   A row whose column 0 is out of range, that takes an action the replayed mask forbids (or outside [0, N)), or that
 *   is not done within min(T, 2 * 32 * ceil(N / 32)) columns contributes nothing, gets loglik = NaN and adds 1 to
 *   *bad_rows (device int32, caller-zeroed, nullable).
 *   cache: tsp the 5E layout (first-node table; another width is CO_ERR_UNSUPPORTED), cvrp 4E; 16-byte aligned.
 *   Errors: env other than tsp / cvrp, N > co_rollout_max_nodes() or tanh_clipping <= 0: CO_ERR_UNSUPPORTED; null
 *   pointers, B_inst < 0, N < 2, num_rows < 1, T < 1 (tsp: T < N), temperature <= 0, a wrong cvrp cache width,
 *   missing cvrp demand / w_capacity or misaligned cache / dLf: CO_ERR_BAD_ARG. */
typedef struct co_eas_grad_args {
  int32_t env_kind;          /* CO_ENV_TSP | CO_ENV_CVRP                                  */
  int32_t B_inst;            /* instances (cache rows)                                   */
  int32_t num_rows;          /* R trajectories per instance                              */
  int32_t N;                 /* nodes incl. depot                                        */
  int32_t T;                 /* columns of actions                                       */
  int32_t cache_width;       /* floats per cache row: tsp 5E, cvrp 4E                    */
  float tanh_clipping;       /* C                                                        */
  float temperature;
  const float* cache;        /* [B_inst, N, cache_width]                                 */
  const float* graph_ctx;    /* [B_inst, E] or NULL                                      */
  const float* w_capacity;   /* [E] cvrp                                                 */
  const float* demand;       /* [B_inst, N-1] cvrp                                       */
  const float* vehicle_capacity; /* [B_inst] cvrp or NULL (= 1.0)                        */
  const int64_t* actions;    /* [R * B_inst, T]                                          */
  const float* coef;         /* [R * B_inst]                                             */
  float* dLf;                /* [B_inst, N, E] out                                       */
  float* loglik;             /* [R * B_inst] out                                         */
  int32_t* bad_rows;         /* [1] out (accumulated) or NULL                            */
} co_eas_grad_args;
int co_eas_key_grad(const co_eas_grad_args* args, void* stream);

/* Efficient active search, layer variant (EAS-Lay; rl4co/models/zoo/eas/nn.py, search.py:198-235): gradient of
 * sum_j coef[j] loglik[j] with respect to the per-instance layer of co_rollout_args.eas_layer.  Rows, coef, the
 * replay, the rules for infeasible rows (loglik NaN, *bad_rows + 1, no contribution) and the errors are those of
 * co_eas_key_grad, with u_n computed from o' = o + relu(o W1 + b1) W2 + b2 (a = o W1 + b1, z = relu(a)).  Per
 * replayed step, with g_n as in co_eas_key_grad:
 *   do' = sum_n g_n Lf[n];  dW2 += z^T do', db2 += do';  dz = (do' W2^T) * [a > 0];  dW1 += o^T dz, db1 += dz
 * layer / dlayer [B_inst, CO_EAS_LAYER_FLOATS] packed as co_rollout_args.eas_layer, 16-byte aligned.  One CTA owns one
 * instance and sums every entry in the fixed order (row, step): bit-identical across launches and independent of the
 * other instances of the batch.  No host synchronisation. */
typedef struct co_eas_layer_grad_args {
  int32_t env_kind;          /* CO_ENV_TSP | CO_ENV_CVRP                                  */
  int32_t B_inst;
  int32_t num_rows;
  int32_t N;
  int32_t T;
  int32_t cache_width;
  float tanh_clipping;
  float temperature;
  const float* cache;        /* [B_inst, N, cache_width]                                 */
  const float* graph_ctx;    /* [B_inst, E] or NULL                                      */
  const float* w_capacity;   /* [E] cvrp                                                 */
  const float* demand;       /* [B_inst, N-1] cvrp                                       */
  const float* vehicle_capacity; /* [B_inst] cvrp or NULL (= 1.0)                        */
  const int64_t* actions;    /* [R * B_inst, T]                                          */
  const float* coef;         /* [R * B_inst]                                             */
  const float* layer;        /* [B_inst, CO_EAS_LAYER_FLOATS]                            */
  float* dlayer;             /* [B_inst, CO_EAS_LAYER_FLOATS] out                        */
  float* loglik;             /* [R * B_inst] out                                         */
  int32_t* bad_rows;         /* [1] out (accumulated) or NULL                            */
} co_eas_layer_grad_args;
int co_eas_layer_grad(const co_eas_layer_grad_args* args, void* stream);

int co_cache_width(int env_kind); /* floats per node row of the rollout cache (tsp 5E, the other envs 4E) */
/* largest N the persistent kernel is instantiated for (else CO_ERR_UNSUPPORTED) */
int co_rollout_max_nodes(void);
int co_rollout(const co_rollout_args* args, void* stream);

/* ------------------------------------------------------------------ dense projections
 *
 * fp32-accurate GEMM on wgmma tensor cores (kind tf32, 3xTF32 hi/lo split, fp32 register
 * accumulators):  C[M,Nout] = epilogue(A[M,K] @ W[Nout,K]^T),
 *   epilogue(v) = relu?((v + bias[n]) + residual[m,n]) * scale[n] + shift[n]   (each optional)
 * Replaces the nn.Linear calls of AttentionModelDecoder._precompute_cache
 * (rl4co/models/zoo/am/decoder.py:201-228) and of the AM encoder (nn/attention.py:110-134,
 * nn/mlp.py:45-60; skip connection nn/ops.py:9-15 and eval-mode BatchNorm nn/ops.py:30-46 fold
 * into residual / scale / shift).  W is passed pre-split (co_split_tf32): Whi = rna_tf32(W),
 * Wlo = W - Whi.  Requirements: K % 32 == 0, Nout % 4 == 0, row strides (lda, ldc, ldr, in
 * floats) % 4 == 0, 16-byte aligned pointers. */
int co_split_tf32(const float* w, float* hi, float* lo, long n, void* stream);
int co_gemm_tf32x3(const float* A, const float* Whi, const float* Wlo, float* C,
                   const float* bias, const float* residual, const float* scale,
                   const float* shift, int M, int Nout, int K, int lda, int ldc, int ldr,
                   int relu, void* stream);

/* Encoder feed-forward block in ONE kernel (the [M, 512] hidden activation never leaves the SM):
 *   out = ((x + relu(x W1^T + b1) W2^T + b2)) * scale + shift,  x [M,128], W1 [512,128], W2 [128,512]
 * = SkipConnection(MLP) + eval-mode BatchNorm of MultiHeadAttentionLayer (rl4co/models/nn/graph/attnnet.py:
 * 33-53, nn/mlp.py:45-60, nn/ops.py:9-15,30-46).  The weights are streamed by TMA bulk copies with cluster
 * multicast from a pre-tiled image: co_ffn_tile_weights builds it (once per weight version) from the co_split_tf32
 * parts of W1 and W2 into `wtiled` (co_ffn_tiled_weight_floats() floats, 128-byte aligned).
 * scale / shift NULL (both) for no affine; ldx / ldo row strides in floats (% 4 == 0); 16-byte aligned pointers. */
long co_ffn_tiled_weight_floats(void);
int co_ffn_tile_weights(const float* w1hi, const float* w1lo, const float* w2hi, const float* w2lo, float* wtiled,
                        void* stream);
int co_ffn_fused(const float* x, const float* wtiled, const float* b1, const float* b2, const float* scale,
                 const float* shift, float* out, int M, int ldx, int ldo, void* stream);

/* ------------------------------------------------------------------ data path (SURVEY.md 8f-3)
 * On-device instance generation (Philox4x32-10 keyed by seed / offset; same seed -> same data on every GPU) and
 * the dihedral-8 augmentation as streaming kernels.
 *   co_generate_uniform: out[i] = U[0,1) * (hi - lo) + lo           (envs/common/utils.py:61-62 "uniform")
 *   co_generate_demand : out[i] = (int(U * (max-min) + (min-1)) + 1) / capacity   (cvrp/generator.py:126-137)
 *   co_dihedral8       : out[a*B + b] = a-th image of locs[b], a = 0..7            (data/transforms.py:16-38) */
int co_generate_uniform(float* out, long n, uint64_t seed, uint64_t offset, float lo, float hi, void* stream);
int co_generate_demand(float* out, long n, uint64_t seed, uint64_t offset, int min_demand, int max_demand,
                       float capacity, void* stream);
int co_dihedral8(const float* locs, float* out, long B, int N, void* stream);

/* co_symmetric_augment: base [B, N, 2], phi [S*B] (one angle per augmented row, drawn by the caller) ->
 * out [S*B, N, 2], aug-major (row a*B + b is image a of instance b).  Per node, as symmetric_transform
 * (data/transforms.py:49-69):  x0 = x - 0.5, y0 = y - 0.5;  x' = cos(phi) x0 - sin(phi) y0,
 * y' = sin(phi) x0 + cos(phi) y0;  (x', y') swapped when phi > 2*pi (2*pi rounded to fp32);  + 0.5.
 * Every operation is rounded on its own (no FMA) and cos / sin are the precise ones, so the result equals torch's
 * elementwise kernels bit for bit; rows with phi = 0 are (x - 0.5) + 0.5, not copies.  The reference draws
 * phi = U[0, 1) * 4 * pi with phi[:B] = 0 (transforms.py:80-84).  Null pointers, B < 0, S < 1, N < 1 or a
 * base / out that is not 8-byte aligned are CO_ERR_BAD_ARG. */
int co_symmetric_augment(const float* base, const float* phi, float* out, long B, int S, int N, void* stream);

/* co_generate_locs: out [B, N, 2] float32 locations from one location law (envs/common/utils.py get_sampler and
 * envs/common/distribution_utils.py), one CTA per instance.  Philox4x32-10 keyed by `seed` with the counter
 * (instance, draw index, offset): row b is the same for every B > b, launch shape and GPU.
 *   UNIFORM                 U(lo, hi)^2
 *   CONSTANT                every coordinate = lo (the caller resolves a number c, "center" = (max - min) / 2 and
 *                           "corner" = min)
 *   NORMAL                  i.i.d. N(mean, std^2), not clamped
 *   CLUSTER                 k = n_cluster centres U(0.2, 0.8)^2; the nodes form k contiguous blocks of floor(N/k),
 *                           the first N mod k one longer; node ~ N(its block's centre, 0.07^2 I), clamped to [0, 1]
 *   MIXED                   U(0, 1)^2, then floor(N/2) distinct nodes in random order are cut into k = n_cluster_mix
 *                           segments (k - 1 of floor(N/(2k)), the last takes the rest) and segment i is redrawn from
 *                           N(c_i, 0.07^2 I), c_i ~ U(0.2, 0.8)^2; clamped to [0, 1]
 *   GAUSSIAN_MIXTURE        (num_modes, cdist) = (0, 0): U(0, 1)^2.  (1, 1): N((.5, .5), [[1, r], [r, 1]]), r ~ U(0, 1)
 *                           per instance, shifted by the per-coordinate minimum, divided by the larger of the two
 *                           ranges and centred with + (1 - max) / 2 per coordinate.  Otherwise: each node's mode
 *                           uniform over num_modes, nodes stored grouped by ascending mode, a non-empty mode's centre
 *                           U(0, cdist)^2, node ~ N(centre, I), then min-max scaled to [0, 1] per coordinate.
 *   MIX_DISTRIBUTION        p ~ U(0, 1) per instance: MIXED if p <= 0.33, CLUSTER if p <= 0.66, else U(0, 1)^2
 *   MIX_MULTI_DISTRIBUTIONS per instance one (num_modes, cdist) uniform over {(0,0), (1,1)} + {3,5,7} x {10,30,50}
 * 1 <= N <= CO_LOCS_MAX_NODES; GAUSSIAN_MIXTURE other than (0, 0) and MIX_MULTI_DISTRIBUTIONS need N >= 2;
 * n_cluster, n_cluster_mix >= 1 where used; anything else is CO_ERR_BAD_ARG.  `out` must be 8-byte aligned. */
#define CO_LOCS_MAX_NODES 10000
#define CO_LOCS_UNIFORM 0
#define CO_LOCS_CONSTANT 1
#define CO_LOCS_NORMAL 2
#define CO_LOCS_CLUSTER 3
#define CO_LOCS_MIXED 4
#define CO_LOCS_GAUSSIAN_MIXTURE 5
#define CO_LOCS_MIX_DISTRIBUTION 6
#define CO_LOCS_MIX_MULTI_DISTRIBUTIONS 7
typedef struct co_locs_args {
  int64_t B;              /* instances */
  int32_t N;              /* nodes per instance (depot included where there is one) */
  int32_t kind;           /* CO_LOCS_* */
  uint64_t seed, offset;  /* Philox key / stream */
  float lo, hi;           /* UNIFORM range; CONSTANT value = lo */
  float mean, std;        /* NORMAL */
  int32_t n_cluster;      /* CLUSTER, MIX_DISTRIBUTION */
  int32_t n_cluster_mix;  /* MIXED, MIX_DISTRIBUTION */
  int32_t num_modes;      /* GAUSSIAN_MIXTURE */
  float cdist;            /* GAUSSIAN_MIXTURE */
} co_locs_args;
int co_generate_locs(float* out, const co_locs_args* args, void* stream);

/* Encoder self-attention core: F.scaled_dot_product_attention of MultiHeadAttention
 * (rl4co/models/nn/attention.py:110-134) on the packed projection qkv [B*N, 3E] ("three h d"),
 * 8 heads x 16, no mask, fp32 -> out [B*N, E] ("h d"); N <= 128. */
int co_encoder_mha(const float* qkv, float* out, int B, int N, void* stream);

/* ------------------------------------------------------------------ training step: differentiable attention core
 * (SURVEY.md 8f-2).  o = softmax(q k^T / sqrt(16) [masked]) v per head, 8 heads x 16 channels, fp32; forward saves the
 * per-row log-sum-exp (log2 units of the scaled scores), backward recomputes the probabilities -- no [M, N] tensor in
 * memory.  Replaces F.scaled_dot_product_attention under autograd in the AM encoder
 * (rl4co/models/nn/attention.py:110-134) and in the glimpse of the teacher-forced log-likelihood pass
 * (nn/attention.py:300-314 with the T decode steps of an instance as T queries; utils/decoding.py:448-461).
 * All tensors are [B, rows, 128] with the head slice h at column 16 h, last dimension contiguous; row / batch strides
 * (in floats, multiples of 4) are free, so column views of the fused cache or of a packed qkv projection need no
 * copy.  mask: [B, M, 4] uint32, bit n % 32 of word n / 32 set = key n may be attended (NULL = no mask); a fully
 * masked row yields o = 0.  N <= 128 keys, M <= 256 queries per call. */
typedef struct co_attn_args {
  const float* q;        /* [B, M, E] */
  const float* k;        /* [B, N, E] */
  const float* v;        /* [B, N, E] */
  const uint32_t* mask;  /* [B, M, 4] or NULL */
  float* o;              /* [B, M, E]   (forward: out; backward: in) */
  float* lse;            /* [B, 8, M]   (forward: out; backward: in) */
  const float* dO;       /* [B, M, E], strides of o; backward only */
  float* dq;             /* [B, M, E] backward out */
  float* dk;             /* [B, N, E] backward out */
  float* dv;             /* [B, N, E] backward out */
  int32_t B, M, N, reserved0;
  int64_t q_bs, k_bs, v_bs, o_bs, dq_bs, dk_bs, dv_bs; /* batch strides (floats) */
  int32_t q_rs, k_rs, v_rs, o_rs, dq_rs, dk_rs, dv_rs; /* row strides (floats)   */
  float scale;                                         /* 1 / sqrt(head_dim) = 0.25 */
} co_attn_args;
int co_attn_fwd(const co_attn_args* args, void* stream);
int co_attn_bwd(const co_attn_args* args, void* stream);

/* Instance normalisation of the encoder (nn.InstanceNorm1d(E, affine=True) on x.permute(0,2,1),
 * rl4co/models/nn/ops.py:30-54; POMO's `normalization="instance"`): per (instance, channel) mean / biased variance over
 * the N nodes, y = (x - mean) / sqrt(var + eps) * gamma + beta.  x, out [B, N, 128] contiguous (out may alias x);
 * gamma / beta [128] or NULL. */
int co_instance_norm(const float* x, const float* gamma, const float* beta, float* out, long B, int N, float eps,
                     void* stream);

/* REINFORCE baseline statistics (rl4co/models/rl/reinforce/baselines.py:75-81):
 * out[0] += sum(reward), out[1] += count, in float64 so the cross-rank sum is
 * order-independent enough to reproduce the single-process mean. */
int co_reward_stats(const float* reward, double* out2, int B, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* COROLLOUT_H_ */
