// C-ABI entry of the persistent rollout (argument validation + dispatch); kernels live in
// rollout_impl.cuh, instantiated in rollout_tsp.cu / rollout_cvrp.cu.
#include "co_common.cuh"

namespace co {
int rollout_tsp(const co_rollout_args& A, cudaStream_t st);
int rollout_cvrp(const co_rollout_args& A, cudaStream_t st);
int rollout_sdvrp(const co_rollout_args& A, cudaStream_t st);
int rollout_op(const co_rollout_args& A, cudaStream_t st);
int rollout_pctsp(const co_rollout_args& A, cudaStream_t st);
int rollout_ms_tsp(const co_rollout_args& A, cudaStream_t st);   // query-batched (num_starts > 1)
int rollout_ms_cvrp(const co_rollout_args& A, cudaStream_t st);
}  // namespace co

using namespace co;

extern "C" int co_cache_width(int env_kind) {
  return env_kind == CO_ENV_TSP ? 5 * E
                                : ((env_kind == CO_ENV_CVRP || env_kind == CO_ENV_SDVRP || env_kind == CO_ENV_OP || env_kind == CO_ENV_PCTSP) ? 4 * E : 0);
}
extern "C" int co_rollout_max_nodes(void) { return 128; }

extern "C" int co_rollout(const co_rollout_args* args, void* stream) {
  if (!args) return fail(CO_ERR_BAD_ARG, "co_rollout: null args%s");
  co_rollout_args A = *args;
  if (!A.cache || !A.locs || !A.actions_out || !A.logp_out || !A.reward_out || !A.loglik_out)
    return fail(CO_ERR_BAD_ARG, "co_rollout: null pointer%s");
  if (A.B_inst < 0 || A.N < 2 || A.num_starts < 1 || A.T_max < 1)
    return fail(CO_ERR_BAD_ARG, "co_rollout: bad shape%s B=%lld N=%lld", "", A.B_inst, A.N);
  if (A.N > co_rollout_max_nodes()) return fail(CO_ERR_UNSUPPORTED, "co_rollout: N=%s%lld > 128 nodes", "", A.N);
  if (!(A.temperature > 0.f)) return fail(CO_ERR_BAD_ARG, "co_rollout: temperature must be > 0%s");
  if (!(A.tanh_clipping > 0.f))  // the fused log-softmax uses the clip bound as its fixed offset
    return fail(CO_ERR_UNSUPPORTED, "co_rollout: tanh_clipping must be > 0 (use the stepping kernels)%s");
  if (A.select_mode < 0 || A.select_mode > 3) return fail(CO_ERR_BAD_ARG, "co_rollout: bad select_mode%s");
  if (A.select_mode == CO_SELECT_EVALUATE && !A.forced_actions) return fail(CO_ERR_BAD_ARG, "co_rollout: forced_actions required%s");
  if (A.select_mode == CO_SELECT_SAMPLE_NOISE && !A.noise) return fail(CO_ERR_BAD_ARG, "co_rollout: noise required%s");
  if (A.select_mode == CO_SELECT_SAMPLE_PHILOX) A.noise = nullptr;
  if ((A.flags & CO_ROLLOUT_FORCED_START) && A.num_loc < 1) return fail(CO_ERR_BAD_ARG, "co_rollout: num_loc required for forced starts%s");
  if (A.eas_layer) {  // EAS-Lay lives in the query-batched kernel only
    if ((A.env_kind != CO_ENV_TSP && A.env_kind != CO_ENV_CVRP) || A.num_starts < 2)
      return fail(CO_ERR_UNSUPPORTED, "co_rollout: eas_layer needs tsp / cvrp with num_starts > 1%s");
    if ((uintptr_t)A.eas_layer & 15) return fail(CO_ERR_BAD_ARG, "co_rollout: eas_layer must be 16-byte aligned%s");
  }
  if (A.poly) {  // PolyNet lives in the query-batched kernel only, and not together with EAS-Lay
    if ((A.env_kind != CO_ENV_TSP && A.env_kind != CO_ENV_CVRP) || A.num_starts < 2 || A.eas_layer)
      return fail(CO_ERR_UNSUPPORTED, "co_rollout: poly needs tsp / cvrp with num_starts > 1 and no eas_layer%s");
    if ((uintptr_t)A.poly & 15) return fail(CO_ERR_BAD_ARG, "co_rollout: poly must be 16-byte aligned%s");
    if (A.poly_k < 1) return fail(CO_ERR_BAD_ARG, "co_rollout: poly_k must be >= 1%s");
  }
  if (A.B_inst == 0) return CO_OK;
  cudaStream_t st = (cudaStream_t)stream;
  // S > 1 trajectories per instance: tsp and cvrp run the query-batched kernel, which advances 4 of them per pass, so
  // they never reach the single-trajectory kernel with S > 1
  const bool ms = A.num_starts > 1;
  if (A.cache_width == 0) A.cache_width = co_cache_width(A.env_kind);
  if (A.env_kind == CO_ENV_TSP) {
    if (!A.q_placeholder) return fail(CO_ERR_BAD_ARG, "co_rollout: q_placeholder required for tsp%s");
    if (A.T_max < A.N) return fail(CO_ERR_BAD_ARG, "co_rollout: T_max < N%s");
    if (A.cache_width != 5 * E) return fail(CO_ERR_BAD_ARG, "co_rollout: tsp cache_width must be 5E%s");
    return ms ? rollout_ms_tsp(A, st) : rollout_tsp(A, st);
  }
  if (A.env_kind == CO_ENV_CVRP) {
    if (!A.demand || !A.w_capacity) return fail(CO_ERR_BAD_ARG, "co_rollout: demand / w_capacity required for cvrp%s");
    if (A.cache_width != 4 * E) return fail(CO_ERR_BAD_ARG, "co_rollout: cvrp cache_width must be 4E%s");
    return ms ? rollout_ms_cvrp(A, st) : rollout_cvrp(A, st);
  }
  if (A.env_kind == CO_ENV_SDVRP) {  // single-trajectory kernel only (S > 1 loops over the trajectories inside it)
    if (!A.demand || !A.w_capacity || !A.dyn_w)
      return fail(CO_ERR_BAD_ARG, "co_rollout: demand / w_capacity / dyn_w required for sdvrp%s");
    if (A.cache_width != 4 * E) return fail(CO_ERR_BAD_ARG, "co_rollout: sdvrp cache_width must be 4E%s");
    return rollout_sdvrp(A, st);
  }
  if (A.env_kind == CO_ENV_PCTSP) {  // demand = real prizes [B, N-1], vehicle_capacity = prize_required, node_limit = penalties
    if (!A.demand || !A.w_capacity || !A.vehicle_capacity || !A.node_limit)
      return fail(CO_ERR_BAD_ARG, "co_rollout: prize (demand) / w_capacity / prize_required (vehicle_capacity) / penalty (node_limit) required for pctsp%s");
    if (A.cache_width != 4 * E) return fail(CO_ERR_BAD_ARG, "co_rollout: pctsp cache_width must be 4E%s");
    return rollout_pctsp(A, st);
  }
  if (A.env_kind == CO_ENV_OP) {  // single-trajectory kernel only (S > 1 loops over the trajectories inside it)
    if (!A.demand || !A.w_capacity || !A.vehicle_capacity || !A.node_limit)
      return fail(CO_ERR_BAD_ARG, "co_rollout: prize (demand) / w_capacity / budget (vehicle_capacity) / node_limit required for op%s");
    if (A.cache_width != 4 * E) return fail(CO_ERR_BAD_ARG, "co_rollout: op cache_width must be 4E%s");
    return rollout_op(A, st);
  }
  return fail(CO_ERR_BAD_ARG, "co_rollout: unknown env kind%s");
}
