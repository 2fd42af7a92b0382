// One-decode-step kernels behind FusedAttentionModelDecoder.forward and the fused decoding
// strategies (the step-at-a-time API; the whole-episode path is rollout.cu).
//   co_pointer_logits <- rl4co/models/zoo/am/decoder.py:128-193
//                        + nn/env_embeddings/context.py:61-74,116-134,147-149
//                        + nn/attention.py:274-320 (PointerAttention, mask_inner=True)
//   co_select_action  <- rl4co/utils/decoding.py:138-188 (process_logits) + :344-461
// K/V/L are streamed from HBM once per step (3*N*512 B per trajectory): HBM-bound.
#include "co_common.cuh"

namespace co {

// one CTA (128 threads = 4 warps) per trajectory
template <int ENV>
__global__ void __launch_bounds__(128) pointer_logits_kernel(
    const float* __restrict__ wctx_t, const float* __restrict__ w_placeholder, const float* __restrict__ node_emb,
    const float* __restrict__ graph_ctx, const float* __restrict__ Kc,
    const float* __restrict__ Vc, const float* __restrict__ Lc, const uint8_t* __restrict__ mask,
    const int64_t* __restrict__ first_node, const int64_t* __restrict__ current_node,
    const int64_t* __restrict__ istep, const float* __restrict__ used, const float* __restrict__ cap,
    const float* __restrict__ dyn_w, const float* __restrict__ dyn_feat,
    float* __restrict__ logits_out, int B_inst, int N, int ld) {
  extern __shared__ float sm[];
  float* ctx = sm;             // [2E] context input
  float* q = ctx + 2 * E;      // [E]
  float* o = q + E;            // [E] concatenated heads = glimpse (logit_key is folded with project_out)
  float* sc = o + E;           // [H][N] scores -> attention weights

  const int j = blockIdx.x;
  const int b = j % B_inst;
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const float* hb = node_emb + (size_t)b * N * E;
  const uint8_t* mrow = mask + (size_t)j * N;
  // dynamic embedding (am/decoder.py:142-154): key / value / logit-key rows of node n get + feat[n] * w
  const float* frow = dyn_feat ? dyn_feat + (size_t)j * N : nullptr;

  int ctx_dim;
  if (ENV == CO_ENV_TSP) {
    ctx_dim = 2 * E;
    if (istep[j] < 1) {  // learned placeholder at step 0, context.py:120-128
      ctx[t] = w_placeholder[t];
      ctx[E + t] = w_placeholder[E + t];
    } else {
      ctx[t] = hb[(size_t)first_node[j] * E + t];
      ctx[E + t] = hb[(size_t)current_node[j] * E + t];
    }
  } else {
    ctx_dim = E + 1;
    ctx[t] = hb[(size_t)current_node[j] * E + t];
    if (t == 0) ctx[E] = cap[j] - used[j];  // vehicle_capacity - used_capacity
  }
  __syncthreads();
  {  // q = project_context(ctx) + graph_context ; thread t owns output channel t
    float acc = 0.f;
    for (int k = 0; k < ctx_dim; ++k) acc = fmaf(ctx[k], wctx_t[(size_t)k * E + t], acc);
    if (graph_ctx) acc += graph_ctx[(size_t)b * E + t];
    q[t] = acc;
  }
  __syncthreads();
  {  // scores[h][n] = q_h . K_h[n] / sqrt(16), masked -> -inf
    const float4 qv = reinterpret_cast<const float4*>(q)[lane];
    float4 wk = make_float4(0.f, 0.f, 0.f, 0.f);
    if (frow) wk = reinterpret_cast<const float4*>(dyn_w)[lane];
    for (int n = w; n < N; n += 4) {
      float4 kv = reinterpret_cast<const float4*>(Kc + ((size_t)b * N + n) * ld)[lane];
      if (frow) {
        const float f = frow[n];
        kv.x = kv.x + f * wk.x; kv.y = kv.y + f * wk.y; kv.z = kv.z + f * wk.z; kv.w = kv.w + f * wk.w;
      }
      float p = qv.x * kv.x + qv.y * kv.y + qv.z * kv.z + qv.w * kv.w;
      p += __shfl_xor_sync(FULL, p, 1);
      p += __shfl_xor_sync(FULL, p, 2);
      if ((lane & 3) == 0) sc[(lane >> 2) * N + n] = mrow[n] ? p * 0.25f : -INFINITY;
    }
  }
  __syncthreads();
  for (int h = 2 * w; h < 2 * w + 2; ++h) {  // softmax over nodes, two heads per warp
    float* s = sc + h * N;
    float m = -INFINITY;
    for (int n = lane; n < N; n += 32) m = fmaxf(m, s[n]);
    m = warp_max(m);
    float sum = 0.f;
    for (int n = lane; n < N; n += 32) {
      float e = expf(s[n] - m);
      s[n] = e;
      sum += e;
    }
    sum = warp_sum(sum);
    const float inv = 1.0f / sum;
    for (int n = lane; n < N; n += 32) s[n] *= inv;
  }
  __syncthreads();
  {  // heads: o[e] = sum_n w[h(e)][n] * V[n][e]
    const float* s = sc + (t >> 4) * N;
    const float* vb = Vc + (size_t)b * N * ld + t;
    float acc = 0.f;
    if (frow) {
      const float wv = dyn_w[E + t];
      for (int n = 0; n < N; ++n) acc = fmaf(s[n], vb[(size_t)n * ld] + frow[n] * wv, acc);
    } else {
      for (int n = 0; n < N; ++n) acc = fmaf(s[n], vb[(size_t)n * ld], acc);
    }
    o[t] = acc;
  }
  __syncthreads();
  {  // logits[n] = glimpse . L[n] / sqrt(E)
    const float4 gv = reinterpret_cast<const float4*>(o)[lane];
    float4 wl = make_float4(0.f, 0.f, 0.f, 0.f);
    if (frow) wl = reinterpret_cast<const float4*>(dyn_w + 2 * E)[lane];
    for (int n = w; n < N; n += 4) {
      float4 lv = reinterpret_cast<const float4*>(Lc + ((size_t)b * N + n) * ld)[lane];
      if (frow) {
        const float f = frow[n];
        lv.x = lv.x + f * wl.x; lv.y = lv.y + f * wl.y; lv.z = lv.z + f * wl.z; lv.w = lv.w + f * wl.w;
      }
      float p = gv.x * lv.x + gv.y * lv.y + gv.z * lv.z + gv.w * lv.w;
      p = warp_sum(p);
      if (lane == 0) logits_out[(size_t)j * N + n] = p / 11.313708498984761f;
    }
  }
}

// one warp per row
__global__ void __launch_bounds__(256) select_action_kernel(
    const float* __restrict__ logits, const uint8_t* __restrict__ mask, const float* __restrict__ noise,
    int64_t* action_io, float* __restrict__ logp_out, float* __restrict__ logprobs_out, int mode, float clip,
    float temperature, int mask_logits, uint64_t seed, uint64_t offset, int B, int N) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= B) return;
  const float* lg = logits + (size_t)row * N;
  const uint8_t* mk = mask ? mask + (size_t)row * N : nullptr;
  auto zval = [&](int n) {
    float z = lg[n];
    if (clip > 0.f) z = tanhf(z) * clip;
    if (mask_logits && mk && !mk[n]) z = -INFINITY;
    return z / temperature;
  };
  float m = -INFINITY;
  for (int n = lane; n < N; n += 32) m = fmaxf(m, zval(n));
  m = warp_max(m);
  float sum = 0.f;
  for (int n = lane; n < N; n += 32) sum += expf(zval(n) - m);
  sum = warp_sum(sum);
  const float lsum = logf(sum);
  float best = -INFINITY;
  int bidx = 0x7fffffff;
  const int forced = (mode == CO_SELECT_EVALUATE) ? (int)action_io[row] : -1;
  float flogp = 0.f;
  for (int n = lane; n < N; n += 32) {
    const float lp = (zval(n) - m) - lsum;  // log_softmax
    if (logprobs_out) logprobs_out[(size_t)row * N + n] = lp;
    float key;
    if (mode == CO_SELECT_GREEDY) key = lp;
    else if (mode == CO_SELECT_SAMPLE_NOISE) key = expf(lp) / noise[(size_t)row * N + n];
    else if (mode == CO_SELECT_SAMPLE_PHILOX) key = expf(lp) / philox_exp1(seed, offset, row, 0, n);
    else { key = 0.f; if (n == forced) flogp = lp; }
    if (key > best || (key == best && n < bidx)) { best = key; bidx = n; }
  }
  if (mode == CO_SELECT_EVALUATE) {
    flogp = warp_sum(flogp);
    if (lane == 0) logp_out[row] = flogp;
    return;
  }
  warp_argmax(best, bidx);
  // logp of the winner: recompute on its owner lane, broadcast
  float lp = 0.f;
  if ((bidx & 31) == lane) lp = (zval(bidx) - m) - lsum;
  lp = __shfl_sync(FULL, lp, bidx & 31);
  if (lane == 0) {
    action_io[row] = bidx;
    logp_out[row] = lp;
  }
}

}  // namespace co

using namespace co;

extern "C" int co_pointer_logits(int env_kind, const co_decoder_weights* w, const float* node_emb,
                                 const float* graph_ctx, const float* glimpse_key, const float* glimpse_val,
                                 const float* logit_key, const uint8_t* action_mask, const int64_t* first_node,
                                 const int64_t* current_node, const int64_t* i, const float* used_capacity,
                                 const float* vehicle_capacity, float* logits_out, int B_traj, int B_inst, int N,
                                 int ld, void* stream) {
  if (ld == 0) ld = E;
  if (ld < E || (ld % 4) != 0) return fail(CO_ERR_BAD_ARG, "co_pointer_logits: bad row stride%s %lld", "", ld);
  if (!w || !w->project_context_t || !node_emb || !glimpse_key || !glimpse_val ||
      !logit_key || !action_mask || !current_node || !logits_out)
    return fail(CO_ERR_BAD_ARG, "co_pointer_logits: null pointer%s");
  if (B_traj < 0 || B_inst <= 0 || N <= 0 || (B_traj % B_inst) != 0)
    return fail(CO_ERR_BAD_ARG, "co_pointer_logits: bad shape%s B_traj=%lld B_inst=%lld", "", B_traj, B_inst);
  if (B_traj == 0) return CO_OK;
  size_t smem = (size_t)(4 * E + H * N) * sizeof(float);
  if (smem > 200 * 1024) return fail(CO_ERR_UNSUPPORTED, "co_pointer_logits: N too large%s (%lld)", "", N);
  cudaStream_t st = (cudaStream_t)stream;
  if (env_kind == CO_ENV_TSP) {
    if (!first_node || !i || !w->w_placeholder) return fail(CO_ERR_BAD_ARG, "co_pointer_logits: tsp state missing%s");
    static PerDeviceOnce once;
    bool& attr = once.flag();
    if (!attr && smem > 48 * 1024) {
      cudaFuncSetAttribute(pointer_logits_kernel<CO_ENV_TSP>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
      attr = true;
    }
    pointer_logits_kernel<CO_ENV_TSP><<<B_traj, 128, smem, st>>>(
        w->project_context_t, w->w_placeholder, node_emb, graph_ctx, glimpse_key, glimpse_val,
        logit_key, action_mask, first_node, current_node, i, nullptr, nullptr, nullptr, nullptr, logits_out, B_inst, N, ld);
  } else if (env_kind == CO_ENV_CVRP || env_kind == CO_ENV_SDVRP) {  // both use VRPContext (context.py:26,137-149)
    if ((w->dynamic_w == nullptr) != (w->dynamic_feature == nullptr))
      return fail(CO_ERR_BAD_ARG, "co_pointer_logits: dynamic_w and dynamic_feature go together%s");
    if (env_kind == CO_ENV_SDVRP && !w->dynamic_w) return fail(CO_ERR_BAD_ARG, "co_pointer_logits: sdvrp needs the dynamic embedding%s");
    if (!used_capacity || !vehicle_capacity) return fail(CO_ERR_BAD_ARG, "co_pointer_logits: cvrp state missing%s");
    static PerDeviceOnce once;
    bool& attr = once.flag();
    if (!attr && smem > 48 * 1024) {
      cudaFuncSetAttribute(pointer_logits_kernel<CO_ENV_CVRP>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
      attr = true;
    }
    pointer_logits_kernel<CO_ENV_CVRP><<<B_traj, 128, smem, st>>>(
        w->project_context_t, nullptr, node_emb, graph_ctx, glimpse_key, glimpse_val, logit_key,
        action_mask, nullptr, current_node, nullptr, used_capacity, vehicle_capacity, w->dynamic_w, w->dynamic_feature,
        logits_out, B_inst, N, ld);
  } else {
    return fail(CO_ERR_BAD_ARG, "co_pointer_logits: unknown env kind%s %lld", "", env_kind);
  }
  return check_launch("co_pointer_logits");
}

extern "C" int co_select_action(const float* logits, const uint8_t* action_mask, const float* noise,
                                int64_t* action_io, float* logp_out, float* logprobs_out, int mode,
                                float tanh_clipping, float temperature, int mask_logits, uint64_t seed,
                                uint64_t offset, int B, int N, void* stream) {
  if (!logits || !action_io || !logp_out) return fail(CO_ERR_BAD_ARG, "co_select_action: null pointer%s");
  if (mask_logits && !action_mask) return fail(CO_ERR_BAD_ARG, "co_select_action: mask required%s");
  if (mode == CO_SELECT_SAMPLE_NOISE && !noise) return fail(CO_ERR_BAD_ARG, "co_select_action: noise required%s");
  if (mode < 0 || mode > 3) return fail(CO_ERR_BAD_ARG, "co_select_action: bad mode%s %lld", "", mode);
  if (!(temperature > 0.f)) return fail(CO_ERR_BAD_ARG, "co_select_action: temperature must be > 0%s");
  if (B < 0 || N <= 0) return fail(CO_ERR_BAD_ARG, "co_select_action: bad shape%s");
  if (B == 0) return CO_OK;
  select_action_kernel<<<(B + 7) / 8, 256, 0, (cudaStream_t)stream>>>(logits, action_mask, noise, action_io, logp_out,
                                                                     logprobs_out, mode, tanh_clipping, temperature,
                                                                     mask_logits, seed, offset, B, N);
  return check_launch("co_select_action");
}
