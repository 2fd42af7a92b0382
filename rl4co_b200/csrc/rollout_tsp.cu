// TSP instantiations of the persistent rollout kernel (see rollout_impl.cuh).
#include "rollout_impl.cuh"
namespace co {
int rollout_tsp(const co_rollout_args& A, cudaStream_t st) { return dispatch<CO_ENV_TSP>(A, st); }
}  // namespace co

#ifdef CO_PHASE_CLOCKS
// diagnostic build only: where the TSP rollout kernels write their phase clocks
extern "C" int co_phase_clocks_set(void* buf) {
  return cudaMemcpyToSymbol(co::co_phase_clk, &buf, sizeof(buf)) == cudaSuccess ? 0 : 1;
}
#endif
