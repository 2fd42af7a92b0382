"""GPU: efficient active search with a per-instance layer (EAS-Lay): the multistart rollout kernel with
`co_rollout_args.eas_layer`, `co_eas_layer_grad`, and `rl4co_b200.eas.eas_search(use_eas_layer=True)`.

The references are float64 autograd passes through `O.teacher_forced_logprobs` with rl4co's residual layer between the
head concatenation and project_out (`eas_layer_oracle.teacher_forced_logprobs_with_layer`).  The gradient bound is the
one of the key gradient (test_gpu_eas.py): 2e-4 relative (O.gradient_errors), for the same reasons; the log-probabilities
are held to the rollout sweep's 1e-5 relative / 2e-5 absolute per step.
"""

import pytest
import torch

from eas_layer_oracle import teacher_forced_logprobs_with_layer
from oracle import am_rollout_oracle as O
from test_gpu_eas import GRAD_SIZES, SEARCH_SETTINGS, _cache, _setup

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
E = 128
RTOL, ATOL_LP = 1e-5, 2e-5


def _random_layer(B, seed, scale=(0.08, 0.1, 0.05, 0.1)):
    """A packed non-zero layer [B, 2 E^2 + 2 E] on the device."""
    from rl4co_b200 import native

    g = torch.Generator().manual_seed(seed)
    parts = [scale[0] * torch.randn(B, E * E, generator=g), scale[1] * torch.randn(B, E, generator=g),
             scale[2] * torch.randn(B, E * E, generator=g), scale[3] * torch.randn(B, E, generator=g)]
    out = torch.cat(parts, 1).contiguous().to(DEV)
    assert out.shape == (B, native.EAS_LAYER_FLOATS)
    return out


def _leaves(packed):
    from rl4co_b200.eas import unpack_eas_layer

    return {k: v.detach().double().cpu().clone().requires_grad_(True) for k, v in unpack_eas_layer(packed).items()}


def _rollout(env_name, td, cached, cache, S, layer, mode=None, seed=0, offset=0, forced=None, tanh_clipping=10.0,
             temperature=1.0):
    from rl4co_b200 import native

    B, N = td["action_mask"].shape
    vrp = env_name == "cvrp"
    return native.rollout(env_name, native.SELECT_SAMPLE_PHILOX if mode is None else mode, cache,
                          cached.graph_context_or_none, cached.q_placeholder, cached.w_capacity,
                          td["locs"].contiguous(), td["demand"].contiguous() if vrp else None,
                          td["vehicle_capacity"].reshape(-1).contiguous() if vrp else None, B, N, num_starts=S,
                          forced_start=True, num_loc=N - (1 if vrp else 0), T_max=N if not vrp else 2 * (N - 1),
                          seed=seed, offset=offset, forced_actions=forced, layer=layer, tanh_clipping=tanh_clipping,
                          temperature=temperature)


def _grad(env_name, td, cached, cache, rows, coef, layer, bad=None, tanh_clipping=10.0, temperature=1.0):
    from rl4co_b200 import native

    vrp = env_name == "cvrp"
    return native.eas_layer_grad(env_name, cache, rows, coef, layer, graph_ctx=cached.graph_context_or_none,
                                 w_capacity=cached.w_capacity, demand=td["demand"].contiguous() if vrp else None,
                                 vehicle_capacity=td["vehicle_capacity"].reshape(-1).contiguous() if vrp else None,
                                 tanh_clipping=tanh_clipping, temperature=temperature, bad_rows=bad)


def _oracle_logprobs(pol, env_name, inst, hidden, rows, leaves, R, **kw):
    """`kw`: temperature, tanh_clipping, use_graph_context of `O.teacher_forced_logprobs`"""
    W64 = O.float64_weights(pol.state_dict(), ())
    return teacher_forced_logprobs_with_layer(W64, env_name, inst, hidden.detach().double().cpu(), rows.cpu(), leaves,
                                              num_starts=R, forced_first=True, **kw)


def _samples(env_name, td, cached, cache, S, layer, seed):
    """S rows per instance sampled through the layer plus one incumbent row (from another stream)."""
    B = td.batch_size[0]
    a = _rollout(env_name, td, cached, cache, max(S, 2), layer, seed=seed)
    inc = _rollout(env_name, td, cached, cache, 2, layer, seed=seed + 1, offset=7)
    rows = torch.cat([a["actions"][: S * B], inc["actions"][B:]])
    return rows.contiguous()


def _flat(grads):
    return {k: grads[:, s] for k, s in (("W1", slice(0, E * E)), ("b1", slice(E * E, E * E + E)),
                                        ("W2", slice(E * E + E, 2 * E * E + E)), ("b2", slice(2 * E * E + E, None)))}


@pytest.mark.parametrize("N,env_name", GRAD_SIZES)  # tsp N = 65 / 66: chunk ends on / never on a row end
@pytest.mark.parametrize("S", [1, 3])
def test_layer_gradient_vs_float64_oracle(env_name, N, S):
    B = 3
    env, pol, td, td_host = _setup(env_name, N, B, seed=N + S)
    hidden, cached, cache, _ = _cache(pol, td)
    layer = _random_layer(B, seed=N * 10 + S)
    rows = _samples(env_name, td, cached, cache, S, layer, seed=5 * N + S)
    coef = torch.randn(rows.shape[0], device=DEV)
    dlayer, ll = _grad(env_name, td, cached, cache, rows, coef, layer)
    leaves = _leaves(layer)
    inst = {k: td_host[k] for k in td_host.keys()}
    lp = _oracle_logprobs(pol, env_name, inst, hidden, rows, leaves, S + 1)
    torch.testing.assert_close(ll.double().cpu(), lp.sum(1).detach(), rtol=RTOL, atol=1e-4)
    (coef.double().cpu() * lp.sum(1)).sum().backward()
    got = {k: v.reshape(leaves[k].shape) for k, v in _flat(dlayer).items()}
    rel, zero = O.gradient_errors(got, leaves)
    assert not zero and max(rel.values()) <= 2e-4, rel


@pytest.mark.parametrize("env_name,N", [("tsp", 100), ("cvrp", 50), ("cvrp", 128)])
def test_layer_gradient_bit_identical_and_batch_independent(env_name, N):
    B, S = 9, 4
    env, pol, td, _ = _setup(env_name, N, B, seed=11)
    hidden, cached, cache, _ = _cache(pol, td)
    layer = _random_layer(B, seed=3)
    rows = _samples(env_name, td, cached, cache, S, layer, seed=3)
    coef = torch.randn(rows.shape[0], device=DEV)
    d1, l1 = _grad(env_name, td, cached, cache, rows, coef, layer)
    d2, l2 = _grad(env_name, td, cached, cache, rows, coef, layer)
    assert torch.equal(d1, d2) and torch.equal(l1, l2)
    R = S + 1
    for b in (0, 4, 8):
        sel = torch.arange(R, device=DEV) * B + b
        sub = {k: td[k][b:b + 1] for k in (("demand", "vehicle_capacity") if env_name == "cvrp" else ())}
        cached1 = type(cached)(node_embeddings=cached.node_embeddings[b:b + 1],
                               graph_context=cached.graph_context[b:b + 1], rollout_cache=None,
                               q_placeholder=cached.q_placeholder, w_capacity=cached.w_capacity)
        db, lb = _grad(env_name, sub, cached1, cache[b:b + 1].contiguous(), rows[sel].contiguous(),
                       coef[sel].contiguous(), layer[b:b + 1].contiguous())
        assert torch.equal(db[0], d1[b]) and torch.equal(lb, l1[sel])


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_infeasible_row_is_reported_and_skipped(env_name):
    B, S, N = 4, 3, 30
    env, pol, td, _ = _setup(env_name, N, B, seed=2)
    hidden, cached, cache, _ = _cache(pol, td)
    layer = _random_layer(B, seed=4)
    rows = _samples(env_name, td, cached, cache, S, layer, seed=4)
    coef = torch.randn(rows.shape[0], device=DEV)
    bad_rows = rows.clone()
    j = 1 * B + 2
    bad_rows[j, 3] = bad_rows[j, 2] if env_name == "tsp" else N + 5
    bad = torch.zeros(1, dtype=torch.int32, device=DEV)
    d, ll = _grad(env_name, td, cached, cache, bad_rows, coef, layer, bad)
    assert int(bad.item()) == 1 and torch.isnan(ll[j]) and torch.isfinite(ll[torch.arange(len(ll), device=DEV) != j]).all()
    coef0 = coef.clone()
    coef0[j] = 0
    d0, _ = _grad(env_name, td, cached, cache, rows, coef0, layer)
    torch.testing.assert_close(d, d0, rtol=0, atol=0)


@pytest.mark.parametrize("env_name,N", [("tsp", 20), ("tsp", 100), ("cvrp", 50), ("cvrp", 128), ("tsp", 32), ("tsp", 33),
                                        ("tsp", 65), ("cvrp", 33), ("cvrp", 64)])
def test_rollout_with_layer_vs_oracle(env_name, N):
    from rl4co_b200 import native

    B, S = 3, 5
    env, pol, td, td_host = _setup(env_name, N, B, seed=7 + N)
    hidden, cached, cache, _ = _cache(pol, td)
    layer = _random_layer(B, seed=N)
    inst = {k: td_host[k] for k in td_host.keys()}
    leaves = {k: v.detach() for k, v in _leaves(layer).items()}
    # sampled tours: valid, and their kernel log-probs are the oracle's teacher-forced replay through the layer
    out = _rollout(env_name, td, cached, cache, S, layer, seed=N)
    vrp = env_name == "cvrp"
    assert native.check_tours(out["actions"], N, td["demand"].contiguous() if vrp else None,
                              td["vehicle_capacity"].reshape(-1).contiguous() if vrp else None, B_inst=B) == 0
    with torch.no_grad():
        ref = _oracle_logprobs(pol, env_name, inst, hidden, out["actions"], leaves, S)
    T = ref.shape[1]
    torch.testing.assert_close(out["logprobs"][:, :T].double().cpu(), ref, rtol=RTOL, atol=ATOL_LP)
    torch.testing.assert_close(out["log_likelihood"].double().cpu(), ref.sum(1), rtol=RTOL, atol=1e-4)
    # evaluate mode on tours sampled without the layer
    rows = _rollout(env_name, td, cached, cache, S, None, seed=N + 1)["actions"].contiguous()
    ev = _rollout(env_name, td, cached, cache, S, layer, mode=native.SELECT_EVALUATE, forced=rows)
    assert torch.equal(ev["actions"], rows)
    with torch.no_grad():
        ref = _oracle_logprobs(pol, env_name, inst, hidden, rows, leaves, S)
    torch.testing.assert_close(ev["logprobs"][:, :ref.shape[1]].double().cpu(), ref, rtol=RTOL, atol=ATOL_LP)
    # W2 = b2 = 0: the layer is the identity; the head outputs are normalised before the logit sum instead of after
    ident = layer.clone()
    ident[:, E * E + E:] = 0
    ev0 = _rollout(env_name, td, cached, cache, S, ident, mode=native.SELECT_EVALUATE, forced=rows)
    plain = _rollout(env_name, td, cached, cache, S, None, mode=native.SELECT_EVALUATE, forced=rows)
    torch.testing.assert_close(ev0["logprobs"], plain["logprobs"], rtol=0, atol=1e-5)


def test_one_iteration_equals_adam_on_the_oracle_gradient():
    _check_one_iteration_equals_adam(10.0, 1.0, True)


@pytest.mark.parametrize("clip,temp,graph_context", SEARCH_SETTINGS)
def test_one_iteration_equals_adam_at_the_policy_decoding_settings(clip, temp, graph_context):
    """eas_search passes the policy's tanh clipping, temperature and missing graph context to both of its kernels."""
    _check_one_iteration_equals_adam(clip, temp, graph_context)


def _check_one_iteration_equals_adam(clip, temp, graph_context):
    from rl4co_b200.eas import eas_coefficients, eas_layer_init, eas_search, unpack_eas_layer
    from rl4co_b200.ops import StateAugmentation

    B, N, A, lr = 2, 20, 8, 0.0041
    dec = dict(tanh_clipping=clip, temperature=temp)
    env, pol, td, _ = _setup("tsp", N, B, seed=21, use_graph_context=graph_context, **dec)
    torch.manual_seed(77)
    res = eas_search(pol, env, td, max_iters=1, seed=99, use_eas_layer=True, use_eas_embedding=False,
                     return_layer=True)
    torch.manual_seed(77)
    P0 = eas_layer_init(A * B, DEV)
    tda = StateAugmentation(num_augment=A, augment_fn="dihedral8")(td)
    hidden, cached, _, _ = _cache(pol, tda)
    assert (cached.graph_context_or_none is not None) == graph_context
    cache = cached.rollout_cache.contiguous()  # eas_search's cache: EAS-Lay does not refold the key
    S = env.get_num_starts(td)
    out = _rollout("tsp", tda, cached, cache, S, P0, seed=99, offset=0, **dec)
    coef = eas_coefficients(out["reward"].view(S, A, B), "multistart", 0.013, with_incumbent=False)
    leaves = _leaves(P0)
    lp = _oracle_logprobs(pol, "tsp", {"locs": tda["locs"].cpu()}, hidden, out["actions"], leaves, S,
                          use_graph_context=graph_context, **dec)
    (coef.double().cpu() * lp.sum(1)).sum().backward()
    for k, leaf in leaves.items():
        ref = torch.nn.Parameter(leaf.detach().clone())
        ref.grad = leaf.grad.clone()
        torch.optim.Adam([ref], lr=lr, weight_decay=1e-6).step()
        got = res["layer"][k].double().cpu()
        g64 = leaf.grad
        if k in ("W2", "b2"):  # W2 = b2 = 0 at the start: only they receive a gradient in iteration 0
            # rows of W2 whose hidden unit is never active have an exact zero gradient, in both
            well, dead = g64.abs() > 1e-3 * g64.abs().max(), g64 == 0
            assert (well | dead).float().mean() > 0.5 and well.any()
            torch.testing.assert_close(got[well], ref.detach()[well], rtol=0, atol=1e-3 * lr)
            torch.testing.assert_close(got[dead], ref.detach()[dead], rtol=0, atol=1e-6)
        else:
            assert not g64.any()
            torch.testing.assert_close(got, ref.detach(), rtol=0, atol=1e-6)
        assert (got - ref.detach()).abs().max() <= 2 * lr + 1e-6
    assert set(unpack_eas_layer(P0)) == set(res["layer"])


@pytest.mark.parametrize("env_name,baseline", [("tsp", "multistart"), ("cvrp", "symmetric"), ("cvrp", "full")])
def test_search_invariants(env_name, baseline):
    from rl4co_b200.eas import eas_search

    B, N = 4, 20
    env, pol, td, _ = _setup(env_name, N, B, seed=5)
    before = {k: v.clone() for k, v in pol.state_dict().items()}
    res = eas_search(pol, env, td, max_iters=6, baseline=baseline, seed=1, augment_dihedral=env_name == "tsp",
                     use_eas_layer=True, use_eas_embedding=False)
    hist = res["reward_history"]
    assert hist.shape == (6, B) and (hist[1:] >= hist[:-1]).all()
    assert torch.equal(hist[-1], res["max_reward"])
    env.check_solution_validity(td, res["best_solutions"])
    torch.testing.assert_close(env.get_reward(td, res["best_solutions"]), res["max_reward"], rtol=1e-5, atol=1e-5)
    assert all(torch.equal(v, before[k]) for k, v in pol.state_dict().items())


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_zero_learning_rate_keeps_the_layer_and_takes_running_maxima(env_name):
    from rl4co_b200.eas import eas_layer_init, eas_search, unpack_eas_layer
    from rl4co_b200.ops import StateAugmentation

    B, N, A, iters = 3, 20, 8, 4
    env, pol, td, _ = _setup(env_name, N, B, seed=8)
    torch.manual_seed(5)
    res = eas_search(pol, env, td, max_iters=iters, seed=17, use_eas_layer=True, use_eas_embedding=False,
                     return_layer=True, optimizer_kwargs={"lr": 0.0, "weight_decay": 1e-6})
    torch.manual_seed(5)
    P0 = eas_layer_init(A * B, DEV)
    for k, v in unpack_eas_layer(P0).items():
        assert torch.equal(res["layer"][k], v), k
    tda = StateAugmentation(num_augment=A, augment_fn="dihedral8")(td)
    hidden, cached, _, _ = _cache(pol, tda)
    cache = cached.rollout_cache.contiguous()  # eas_search's cache: EAS-Lay does not refold the key
    S = env.get_num_starts(td)
    best = torch.full((B,), -float("inf"), device=DEV)
    for it in range(iters):
        r = _rollout(env_name, tda, cached, cache, S, P0, seed=17, offset=it)["reward"].view(S, A, B)
        best = torch.maximum(best, r.amax((0, 1)))
        assert torch.equal(res["reward_history"][it], best)
    assert torch.equal(res["max_reward"], best)
