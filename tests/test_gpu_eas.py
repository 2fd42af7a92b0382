"""GPU: efficient active search with embedding updates (`co_eas_key_grad`, `rl4co_b200.eas.eas_search`).

The key-gradient kernel is checked against the float64 oracle under autograd: `O.teacher_forced_logprobs` with the
logit key replaced by a float64 leaf L (`eas_oracle.py`), along trajectories sampled by `co_rollout` from the same
cache, with random per-row coefficients.
The product's gradient is dL = dLf W_out^T.  Bound (O.gradient_errors, relative Frobenius error): 2e-4.  Every step of
the kernel is an fp32 glimpse + pointer logit (relative round-off ~1e-6, as in the rollout kernel) and the residuals
(delta - p) of up to (S + 1) * 2 (N - 1) steps per instance are summed with cancelling signs, so the error of the sum is
larger than that of one term; the fp32 training-gradient tests allow 1e-4 per parameter for the same kind of pass.
"""

import pytest
import torch

from conftest import name_seeded_weights
from eas_oracle import teacher_forced_logprobs_with_key
from oracle import am_rollout_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
E = 128


def _setup(env_name, N, B, seed, use_graph_context=True, **policy_kw):
    """Seeded policy and instances; `policy_kw` (temperature, tanh_clipping) go to the policy, which `eas_search`
    reads them from."""
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    torch.manual_seed(seed)
    env = get_env(env_name, generator_params=dict(num_loc=N if env_name == "tsp" else N - 1), check_solution=False)
    pol = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=2, use_graph_context=use_graph_context,
                                    **policy_kw)
    pol.load_state_dict(name_seeded_weights(pol.state_dict(), seed))
    pol = pol.to(DEV).eval()
    td_host = env.generator(B)
    td = env.reset(td_host.to(DEV))
    return env, pol, td, td_host


def _cache(pol, td):
    """Encoder output, the 5E / 4E rollout cache with block 2 = L W_out, and the unfolded key L."""
    dec = pol.decoder
    with torch.no_grad():
        hidden, _ = pol.encoder(td)
        cached = dec._precompute_cache(hidden)
        cache = cached.rollout_cache.contiguous().clone()
        L = torch.matmul(hidden, dec.project_node_embeddings.weight[2 * E:3 * E].t()).contiguous()
        cache[..., 2 * E:3 * E] = torch.matmul(L, dec.pointer.project_out.weight)
    return hidden, cached, cache, L


def _rollout(env_name, pol, td, cached, cache, S, seed, offset=0, tanh_clipping=10.0, temperature=1.0):
    from rl4co_b200 import native

    B, N = td["action_mask"].shape
    vrp = env_name == "cvrp"
    return native.rollout(env_name, native.SELECT_SAMPLE_PHILOX, cache, cached.graph_context_or_none,
                          cached.q_placeholder, cached.w_capacity, td["locs"].contiguous(),
                          td["demand"].contiguous() if vrp else None,
                          td["vehicle_capacity"].reshape(-1).contiguous() if vrp else None, B, N, num_starts=S,
                          forced_start=True, num_loc=N - (1 if vrp else 0), T_max=N if not vrp else 2 * (N - 1),
                          seed=seed, offset=offset, tanh_clipping=tanh_clipping, temperature=temperature)


def _grad(env_name, td, cached, cache, rows, coef, bad=None, tanh_clipping=10.0, temperature=1.0):
    from rl4co_b200 import native

    vrp = env_name == "cvrp"
    return native.eas_key_grad(env_name, cache, rows, coef, graph_ctx=cached.graph_context_or_none,
                               w_capacity=cached.w_capacity, demand=td["demand"].contiguous() if vrp else None,
                               vehicle_capacity=td["vehicle_capacity"].reshape(-1).contiguous() if vrp else None,
                               tanh_clipping=tanh_clipping, temperature=temperature, bad_rows=bad)


def _oracle_grad(pol, env_name, inst, hidden, L, rows, coef, R, **kw):
    """d(sum_j coef_j ll_j) / dL in float64 through the reference-restated decoder (fixed encoder output) -> (the leaf
    L64 holding it in .grad, the per-step log-probs [rows, T]).  `kw`: temperature, tanh_clipping, use_graph_context
    of `O.teacher_forced_logprobs`."""
    W64 = O.float64_weights(pol.state_dict(), ())
    L64 = L.detach().double().cpu().requires_grad_(True)
    lp = teacher_forced_logprobs_with_key(W64, env_name, inst, hidden.detach().double().cpu(), rows.cpu(), L64,
                                          num_starts=R, forced_first=True, **kw)
    (coef.double().cpu() * lp.sum(1)).sum().backward()
    return L64, lp.detach()


def _samples(env_name, pol, td, cached, cache, S, seed):
    """S sampled rows per instance plus one incumbent row (a tour from another stream); their rollout log-likelihoods."""
    B = td.batch_size[0]
    a = _rollout(env_name, pol, td, cached, cache, max(S, 2), seed)
    inc = _rollout(env_name, pol, td, cached, cache, 2, seed + 1, offset=7)
    rows = torch.cat([a["actions"][: S * B], inc["actions"][B:]])
    ll = torch.cat([a["log_likelihood"][: S * B], inc["log_likelihood"][B:]])
    return rows.contiguous(), ll


# the node-slot edges of the SPL = 1 / 2 / 4 instantiations (N = 32, 33, 64, 65), the smallest instance with a choice
# after the forced start (N = 3) and tsp N = 66; for cvrp N is the mask width, depot included
GRAD_SIZES = [(n, e) for n in (20, 50, 100, 128) for e in ("tsp", "cvrp")] + \
    [(n, "tsp") for n in (3, 32, 33, 64, 65, 66)] + [(n, "cvrp") for n in (3, 32, 33, 64, 65)]


@pytest.mark.parametrize("N,env_name", GRAD_SIZES)
@pytest.mark.parametrize("S", [1, 3])
def test_key_gradient_vs_float64_oracle(env_name, N, S):
    B = 3
    env, pol, td, td_host = _setup(env_name, N, B, seed=N + S)
    hidden, cached, cache, L = _cache(pol, td)
    rows, ll_roll = _samples(env_name, pol, td, cached, cache, S, seed=5 * N + S)
    coef = torch.randn(rows.shape[0], device=DEV)
    dLf, ll = _grad(env_name, td, cached, cache, rows, coef)
    torch.testing.assert_close(ll, ll_roll, rtol=1e-5, atol=1e-5)
    dL = torch.matmul(dLf, pol.decoder.pointer.project_out.weight.t())
    inst = {k: td_host[k] for k in td_host.keys()}
    L64, _ = _oracle_grad(pol, env_name, inst, hidden, L, rows, coef, S + 1)
    rel, zero = O.gradient_errors({"L": dL}, {"L": L64})
    assert not zero and rel["L"] <= 2e-4, rel


@pytest.mark.parametrize("env_name,N", [("tsp", 100), ("cvrp", 50), ("cvrp", 128)])
def test_key_gradient_bit_identical_and_batch_independent(env_name, N):
    B, S = 9, 4
    env, pol, td, _ = _setup(env_name, N, B, seed=11)
    hidden, cached, cache, L = _cache(pol, td)
    rows, _ = _samples(env_name, pol, td, cached, cache, S, seed=3)
    coef = torch.randn(rows.shape[0], device=DEV)
    d1, l1 = _grad(env_name, td, cached, cache, rows, coef)
    d2, l2 = _grad(env_name, td, cached, cache, rows, coef)
    assert torch.equal(d1, d2) and torch.equal(l1, l2)
    R = S + 1
    for b in (0, 4, 8):
        sel = torch.arange(R, device=DEV) * B + b
        sub = {k: td[k][b:b + 1] for k in (("demand", "vehicle_capacity") if env_name == "cvrp" else ())}
        cached1 = type(cached)(node_embeddings=cached.node_embeddings[b:b + 1],
                               graph_context=cached.graph_context[b:b + 1], rollout_cache=None,
                               q_placeholder=cached.q_placeholder, w_capacity=cached.w_capacity)
        db, lb = _grad(env_name, sub, cached1, cache[b:b + 1].contiguous(), rows[sel].contiguous(),
                       coef[sel].contiguous())
        assert torch.equal(db[0], d1[b]) and torch.equal(lb, l1[sel])


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_infeasible_row_is_reported_and_skipped(env_name):
    B, S, N = 4, 3, 30
    env, pol, td, _ = _setup(env_name, N, B, seed=2)
    hidden, cached, cache, L = _cache(pol, td)
    rows, _ = _samples(env_name, pol, td, cached, cache, S, seed=4)
    coef = torch.randn(rows.shape[0], device=DEV)
    bad_rows = rows.clone()
    j = 1 * B + 2                                       # start 1 of instance 2
    bad_rows[j, 3] = bad_rows[j, 2] if env_name == "tsp" else N + 5   # a revisit / an id out of range
    bad = torch.zeros(1, dtype=torch.int32, device=DEV)
    d, ll = _grad(env_name, td, cached, cache, bad_rows, coef, bad)
    assert int(bad.item()) == 1 and torch.isnan(ll[j]) and torch.isfinite(ll[torch.arange(len(ll), device=DEV) != j]).all()
    coef0 = coef.clone()
    coef0[j] = 0
    d0, _ = _grad(env_name, td, cached, cache, rows, coef0)
    torch.testing.assert_close(d, d0, rtol=0, atol=0)


# eas_search reads the decoding parameters and the graph context from the policy: settings besides the defaults
SEARCH_SETTINGS = [(3.0, 0.5, False)]


def test_one_iteration_equals_adam_on_the_oracle_gradient():
    _check_one_iteration_equals_adam(10.0, 1.0, True)


@pytest.mark.parametrize("clip,temp,graph_context", SEARCH_SETTINGS)
def test_one_iteration_equals_adam_at_the_policy_decoding_settings(clip, temp, graph_context):
    """eas_search passes the policy's tanh clipping, temperature and missing graph context to both of its kernels."""
    _check_one_iteration_equals_adam(clip, temp, graph_context)


def _check_one_iteration_equals_adam(clip, temp, graph_context):
    from rl4co_b200.eas import eas_coefficients, eas_search
    from rl4co_b200.ops import StateAugmentation

    B, N, A = 2, 20, 8
    dec = dict(tanh_clipping=clip, temperature=temp)
    env, pol, td, _ = _setup("tsp", N, B, seed=21, use_graph_context=graph_context, **dec)
    res = eas_search(pol, env, td, max_iters=1, seed=99, return_logit_key=True)
    tda = StateAugmentation(num_augment=A, augment_fn="dihedral8")(td)
    hidden, cached, cache, L0 = _cache(pol, tda)
    assert (cached.graph_context_or_none is not None) == graph_context
    S = env.get_num_starts(td)
    out = _rollout("tsp", pol, tda, cached, cache, S, seed=99, offset=0, **dec)
    coef = eas_coefficients(out["reward"].view(S, A, B), "multistart", 0.013, with_incumbent=False)
    L64, _ = _oracle_grad(pol, "tsp", {"locs": tda["locs"].cpu()}, hidden, L0, out["actions"], coef, S,
                          use_graph_context=graph_context, **dec)
    g64 = L64.grad
    ref = torch.nn.Parameter(L0.detach().double().cpu())
    ref.grad = g64.clone()
    torch.optim.Adam([ref], lr=0.0041, weight_decay=1e-6).step()
    got = res["logit_key"].double().cpu()
    # Adam's first step is lr * g / (|g| + eps): exact where the fp32 gradient has the float64 one's sign and size
    # (|g| well above its round-off), at most 2 lr off elsewhere
    well = g64.abs() > 1e-3 * g64.abs().max()
    assert well.float().mean() > 0.9
    torch.testing.assert_close(got[well], ref.detach()[well], rtol=0, atol=1e-3 * 0.0041)
    assert (got - ref.detach()).abs().max() <= 2 * 0.0041 + 1e-6


@pytest.mark.parametrize("env_name,baseline", [("tsp", "multistart"), ("cvrp", "symmetric"), ("cvrp", "full")])
def test_search_invariants(env_name, baseline):
    from rl4co_b200.eas import eas_search

    B, N = 4, 20
    env, pol, td, _ = _setup(env_name, N, B, seed=5)
    before = {k: v.clone() for k, v in pol.state_dict().items()}
    res = eas_search(pol, env, td, max_iters=6, baseline=baseline, seed=1, augment_dihedral=env_name == "tsp")
    hist = res["reward_history"]
    assert hist.shape == (6, B) and (hist[1:] >= hist[:-1]).all()
    assert torch.equal(hist[-1], res["max_reward"])
    env.check_solution_validity(td, res["best_solutions"])
    torch.testing.assert_close(env.get_reward(td, res["best_solutions"]), res["max_reward"], rtol=1e-5, atol=1e-5)
    assert all(torch.equal(v, before[k]) for k, v in pol.state_dict().items())


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_zero_learning_rate_keeps_the_key_and_takes_running_maxima(env_name):
    from rl4co_b200.eas import eas_search
    from rl4co_b200.ops import StateAugmentation

    B, N, A, iters = 3, 20, 8, 4
    env, pol, td, _ = _setup(env_name, N, B, seed=8)
    res = eas_search(pol, env, td, max_iters=iters, seed=17, return_logit_key=True,
                     optimizer_kwargs={"lr": 0.0, "weight_decay": 1e-6})
    tda = StateAugmentation(num_augment=A, augment_fn="dihedral8")(td)
    hidden, cached, cache, L0 = _cache(pol, tda)
    assert torch.equal(res["logit_key"], L0)
    S = env.get_num_starts(td)
    best = torch.full((B,), -float("inf"), device=DEV)
    for it in range(iters):
        r = _rollout(env_name, pol, tda, cached, cache, S, seed=17, offset=it)["reward"].view(S, A, B)
        best = torch.maximum(best, r.amax((0, 1)))
        assert torch.equal(res["reward_history"][it], best)
    assert torch.equal(res["max_reward"], best)
