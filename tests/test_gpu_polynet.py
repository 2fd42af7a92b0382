"""GPU: PolyNet -- the multistart rollout kernel with `co_rollout_args.poly`, the stepping path, and `polynet_step`.

The reference is the float64 oracle with rl4co's PolyNetAttention pointer (`polynet_oracle`), run from the GPU's own
encoder output.  Log-probabilities are held to the rollout sweep's 1e-5 relative / 2e-5 absolute per step; a greedy
step must pick an action within that tolerance of the oracle's best one (so exact near-ties cannot fail the check);
sampling consumes recorded Exp(1) noise (SELECT_SAMPLE_NOISE) on both sides.
"""

import pytest
import torch

from conftest import name_seeded_weights
from oracle import am_rollout_oracle as O
from polynet_oracle import rollout_polynet, teacher_forced_logprobs_polynet

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
E = 128
RTOL, ATOL_LP = 1e-5, 2e-5


def _setup(env_name, N, B, k, seed, scale2=4.0, **kw):
    from rl4co_b200.envs import get_env
    from rl4co_b200.polynet import FusedPolyNetPolicy

    torch.manual_seed(seed)
    env = get_env(env_name, generator_params=dict(num_loc=N if env_name == "tsp" else N - 1), check_solution=False)
    pol = FusedPolyNetPolicy(k=k, env_name=env_name, num_encoder_layers=2, normalization="batch", **kw)
    sd = name_seeded_weights(pol.state_dict(), seed)
    sd["decoder.pointer.binary_vectors"] = pol.decoder.pointer.binary_vectors.detach().clone()
    sd["decoder.pointer.poly_layer_2.weight"] *= scale2  # a poly layer as large as the glimpse
    pol.load_state_dict(sd)
    pol = pol.to(DEV).eval()
    td_host = env.generator(B)
    inst = {k_: td_host[k_] for k_ in td_host.keys()}
    return env, pol, env.reset(td_host.to(DEV)), inst


def _w64(pol):
    return O.float64_weights(pol.state_dict(), ())


def _recorded_steps(teacher_forced, *args, **kw):
    """`teacher_forced(*args, **kw)` (an `O.teacher_forced_logprobs` variant) -> its float64 log-probs and, per decoder
    step, the oracle's full log-prob row."""
    rows = []
    real = O.process_logits

    def recording(*a, **k):
        lp = real(*a, **k)
        rows.append(lp.detach())
        return lp

    O.process_logits = recording
    try:
        lp = teacher_forced(*args, **kw)
    finally:
        O.process_logits = real
    return lp.detach(), torch.stack(rows, 1)  # [R, T], [R, T - 1, N]


def _oracle_steps(W64, env_name, inst, h64, acts, S, strategy=None, **kw):
    """Teacher-forced float64 log-probs of `acts` and, per step, the oracle's full log-prob row.  `kw`: temperature,
    tanh_clipping, use_graph_context of `O.teacher_forced_logprobs`."""
    return _recorded_steps(teacher_forced_logprobs_polynet, W64, env_name, inst, h64, acts, num_starts=S,
                           forced_first=True, strategy=strategy, **kw)


def _check_greedy(lp_gpu, acts, lp64, full64):
    T = lp64.shape[1]
    torch.testing.assert_close(lp_gpu[:, :T].double().cpu(), lp64, rtol=RTOL, atol=ATOL_LP)
    chosen = full64.gather(2, acts[:, 1:T, None]).squeeze(2)
    best = full64.max(2).values
    gap = (best - chosen)[torch.isfinite(best)]
    assert float(gap.max()) <= ATOL_LP, f"greedy step {float(gap.max()):.2e} below the oracle's best"


SIZES = [(1, 2), (1, 5), (3, 2), (3, 3), (3, 9), (128, 2), (128, 128), (128, 259)]


# plus the node-slot edges of the SPL = 1 / 2 / 4 instantiations at one (k, S)
@pytest.mark.parametrize("N,k,S", [(n, k, s) for n in (20, 50, 100, 128) for k, s in SIZES] +
                         [(n, 3, 9) for n in (32, 33, 64, 65)])
@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_fused_greedy_vs_oracle(env_name, N, k, S):
    env, pol, td, inst = _setup(env_name, N, 2, k, seed=N + k + S)
    with torch.inference_mode():
        out = pol(td, env, phase="test", decode_type="greedy", num_starts=S, return_sum_log_likelihood=False,
                  return_hidden=True)
    acts = out["actions"].cpu()
    assert acts.shape[0] == 2 * S
    h64 = out["hidden"].double().cpu()
    lp64, full64 = _oracle_steps(_w64(pol), env_name, inst, h64, acts, S)
    _check_greedy(out["log_likelihood"], acts, lp64, full64)


@pytest.mark.parametrize("k,S", [(3, 9), (128, 130)])
@pytest.mark.parametrize("N", [20, 100])
@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_fused_sampling_recorded_noise_vs_oracle(env_name, N, k, S):
    env, pol, td, inst = _setup(env_name, N, 2, k, seed=7 * N + S)
    T = N if env_name == "tsp" else 2 * (N - 1)
    gen = torch.Generator().manual_seed(N + S)
    q = torch.empty(T, 2 * S, N).exponential_(1, generator=gen)
    with torch.inference_mode():
        out = pol(td, env, phase="train", decode_type="sampling", num_starts=S, noise=q.to(DEV),
                  return_sum_log_likelihood=False, return_hidden=True)
    h64 = out["hidden"].double().cpu()
    ref = rollout_polynet(_w64(pol), env_name, inst, h64, decode_type="multistart_sampling", num_starts=S,
                          noise=lambda step, shape: q[step].double())
    T = ref["actions"].shape[1]
    same = (out["actions"].cpu()[:, :T] == ref["actions"]).all(1)
    assert float(same.float().mean()) >= 0.95, f"only {float(same.float().mean()):.0%} of the rows sampled alike"
    torch.testing.assert_close(out["log_likelihood"].cpu()[same, :T].double(), ref["logprobs"][same],
                               rtol=RTOL, atol=ATOL_LP)


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_zero_poly_layer_is_the_am_policy(env_name):
    """poly_layer_2 = 0: PolyNet decodes the AM policy's multistart greedy tours with its log-probs."""
    from rl4co_b200.policy import FusedAttentionModelPolicy

    N, S = 50, 10
    env, pol, td, _ = _setup(env_name, N, 16, 3, seed=31)
    with torch.no_grad():
        pol.decoder.pointer.poly_layer_2.weight.zero_()
        pol.decoder.pointer.poly_layer_2.bias.zero_()
    am = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=2, normalization="batch").to(DEV).eval()
    am.load_state_dict(pol.state_dict(), strict=False)
    with torch.inference_mode():
        a = pol(td, env, phase="test", decode_type="greedy", num_starts=S)
        b = am(td, env, phase="test", decode_type="multistart_greedy", num_starts=S)
    same = (a["actions"] == b["actions"]).all(1)  # the two caches round differently: an exact near-tie may flip a row
    assert float(same.float().mean()) >= 0.95
    torch.testing.assert_close(a["log_likelihood"][same], b["log_likelihood"][same], rtol=RTOL, atol=ATOL_LP * 10)


def _kernel_rollout(env_name, pol, td, cached, S, mode, lo=0, hi=None):
    """`native.rollout` with the decoder's poly weights on instances lo:hi of one cache (the encoder and the cache GEMM
    are left out: their cuBLAS / GEMM tiling may round differently at another batch size)."""
    from rl4co_b200 import native

    B, N = td["action_mask"].shape
    hi = B if hi is None else hi
    vrp = env_name == "cvrp"
    g = cached.graph_context_or_none
    return native.rollout(env_name, mode, cached.rollout_cache[lo:hi].contiguous(), None if g is None else g[lo:hi],
                          cached.q_placeholder, cached.w_capacity, td["locs"][lo:hi].contiguous(),
                          td["demand"][lo:hi].contiguous() if vrp else None,
                          td["vehicle_capacity"][lo:hi].reshape(-1).contiguous() if vrp else None, hi - lo, N,
                          num_starts=S, forced_start=True, num_loc=N - (1 if vrp else 0), seed=5,
                          **pol.decoder.rollout_extras(S))


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_repeatable_and_batch_independent(env_name):
    from rl4co_b200 import native

    env, pol, td, _ = _setup(env_name, 100, 9, 128, seed=41)
    S = 130
    with torch.inference_mode():
        cached = pol.decoder._precompute_cache(pol.encoder(td)[0])
        a = _kernel_rollout(env_name, pol, td, cached, S, native.SELECT_SAMPLE_PHILOX)
        b = _kernel_rollout(env_name, pol, td, cached, S, native.SELECT_SAMPLE_PHILOX)
        g9 = _kernel_rollout(env_name, pol, td, cached, S, native.SELECT_GREEDY)
        g1 = _kernel_rollout(env_name, pol, td, cached, S, native.SELECT_GREEDY, 4, 5)
    for key in ("actions", "logprobs", "reward"):
        assert torch.equal(a[key], b[key]), key
    rows = torch.arange(S, device=DEV) * 9 + 4
    for key in ("actions", "logprobs", "reward", "log_likelihood"):
        assert torch.equal(g9[key][rows], g1[key]), key


@pytest.mark.parametrize("env_name,N,kw", [("tsp", 150, {}), ("cvrp", 150, {}), ("tsp", 50, dict(fused_rollout=False)),
                                           ("cvrp", 50, dict(fused_rollout=False))])
def test_stepping_path_vs_oracle(env_name, N, kw):
    k, S = 3, 7
    env, pol, td, inst = _setup(env_name, N, 2, k, seed=N + 3)
    with torch.inference_mode():
        out = pol(td, env, phase="test", decode_type="greedy", num_starts=S, return_sum_log_likelihood=False,
                  return_hidden=True, **kw)
    acts = out["actions"].cpu()
    lp64, full64 = _oracle_steps(_w64(pol), env_name, inst, out["hidden"].double().cpu(), acts, S)
    _check_greedy(out["log_likelihood"], acts, lp64, full64)


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_polynet_step_gradients_vs_float64(env_name):
    """polynet_step(phase="train") replays only the best row of each instance; its gradient equals the float64 gradient
    of the full [B, k] Poppy loss with every row replayed (the masked rows carry coefficient 0).  The scheme and bounds
    of test_gpu_train_gradients.py: the default path and CO_TRAIN_ATTN=sdpa, on the GPU pass's encoder ReLU branch.
    The poly layer's ReLU takes the float64 forward's own branch."""
    from rl4co_b200.polynet import polynet_step
    from test_gpu_train_gradients import _compare

    N, B, k = 20, 8, 5
    env, pol, td, inst = _setup(env_name, N, B, k, seed=12)

    def run():
        torch.manual_seed(12)
        return None, polynet_step(pol, env, td, phase="train", optimizer=torch.optim.SGD(pol.parameters(), lr=0.0))

    def oracle(W64, res, branch):
        masks, pre = branch.take(2), []
        h64, _ = O.encoder_forward(W64, env_name, O.env_reset(env_name, inst), num_layers=2, normalization="batch",
                                   batch_stats=True, relu_masks=masks, pre_activations=pre)
        branch.note(masks, pre)
        r, mask = res["reward"].cpu().double(), res["mask"].cpu()
        coef = (-(r - r.mean(1, keepdim=True)) * mask / (B * k)).t().reshape(-1)   # start-major rows s * B + b
        lp64 = teacher_forced_logprobs_polynet(W64, env_name, inst, h64, res["actions"].cpu(), num_starts=k,
                                               forced_first=True)
        (coef * lp64.sum(1)).sum().backward()
        W64["decoder.pointer.binary_vectors"].grad = None  # a constant of the model, not a parameter
        return lp64.detach()

    _compare("P", f"polynet-{env_name}", pol, run, oracle)


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_polynet_step_poly_parameters_get_gradient(env_name):
    from rl4co_b200.polynet import polynet_step

    env, pol, td, _ = _setup(env_name, 20, 8, 4, seed=13)
    pol.zero_grad(set_to_none=True)
    res = polynet_step(pol, env, td, phase="train", optimizer=torch.optim.SGD(pol.parameters(), lr=0.0))
    p = pol.decoder.pointer
    for t in (p.poly_layer_1.weight, p.poly_layer_1.bias, p.poly_layer_2.weight, p.poly_layer_2.bias):
        assert t.grad is not None and bool(t.grad.any())
    assert p.binary_vectors.grad is None
    assert res["mask"].sum(1).eq(1).all()


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_polynet_step_test_keys(env_name):
    from rl4co_b200 import native
    from rl4co_b200.polynet import polynet_step

    N, B = 20, 4
    env, pol, td, _ = _setup(env_name, N, B, 8, seed=17)
    res = polynet_step(pol, env, td, val_num_solutions=12, num_augment=8, phase="test")
    assert res["max_reward"].shape == (B, 8) and res["max_aug_reward"].shape == (B,)
    assert res["best_multistart_actions"].shape[:2] == (B, 8) and res["best_aug_actions"].shape[0] == B
    assert torch.equal(res["max_aug_reward"], res["max_reward"].max(1).values)
    acts = res["best_aug_actions"].contiguous()
    if env_name == "tsp":
        assert native.check_tours(acts, N) == 0
    else:
        assert native.check_tours(acts, N, td["demand"].contiguous(), td["vehicle_capacity"].reshape(-1).contiguous(),
                                  B_inst=B) == 0
    with pytest.raises(ValueError, match="val_num_solutions"):
        polynet_step(pol, env, td, val_num_solutions=12, phase="test", decode_type="greedy")
    res = polynet_step(pol, env, td, val_num_solutions=8, num_augment=1, phase="test", decode_type="greedy")
    assert res["max_reward"].shape == (B,)
