"""CPU: efficient active search (EAS-Emb) -- the loss coefficients against rl4co's loss expression, the rejections of
`eas_search`, the argument checks of `co_eas_key_grad` and of its binding, and the float64 reference's key override."""

import ctypes

import pytest
import torch

from conftest import name_seeded_weights
from eas_oracle import teacher_forced_logprobs_with_key
from oracle import am_rollout_oracle as O


def _rl4co_loss(reward, ll, baseline, eas_lambda):
    """rl4co/models/zoo/eas/search.py:219-235 verbatim on [B, A, S + 1] tensors (last column: the incumbent)."""
    group_reward = reward[..., :-1]
    if baseline == "multistart":
        bl_val = group_reward.mean(dim=-1, keepdim=True)
    elif baseline == "symmetric":
        bl_val = group_reward.mean(dim=-2, keepdim=True)
    elif baseline == "full":
        bl_val = group_reward.mean(dim=-1, keepdim=True).mean(dim=-2, keepdim=True)
    advantage = group_reward - bl_val
    loss_rl = -(advantage * ll[..., :-1]).mean()
    loss_il = -ll[..., -1].mean()
    return loss_rl + eas_lambda * loss_il


@pytest.mark.parametrize("baseline", ["multistart", "symmetric", "full"])
@pytest.mark.parametrize("B,A,S", [(3, 8, 5), (1, 8, 20), (4, 2, 3)])
def test_coefficients_reproduce_rl4co_loss(baseline, B, A, S):
    from rl4co_b200.eas import eas_coefficients

    g = torch.Generator().manual_seed(B * 100 + A * 10 + S)
    reward = -torch.rand(B, A, S + 1, generator=g, dtype=torch.float64) * 10
    ll = -torch.rand(B, A, S + 1, generator=g, dtype=torch.float64) * 50
    ref = _rl4co_loss(reward, ll, baseline, 0.013)
    # the kernel's rows: r * (A * B) + a * B + b, r = S the incumbent
    coef = eas_coefficients(reward[..., :-1].permute(2, 1, 0), baseline, 0.013, with_incumbent=True)
    rows = ll.permute(2, 1, 0).reshape(-1)
    assert coef.shape == ((S + 1) * A * B,)
    torch.testing.assert_close((coef * rows).sum(), ref, rtol=1e-12, atol=1e-12)
    # without the incumbent row (iteration 0) the loss is the REINFORCE term alone
    coef0 = eas_coefficients(reward[..., :-1].permute(2, 1, 0), baseline, 0.013, with_incumbent=False)
    torch.testing.assert_close((coef0 * rows[: S * A * B]).sum(), _rl4co_loss(reward, ll, baseline, 0.0),
                               rtol=1e-12, atol=1e-12)


def test_coefficients_reject_unknown_baseline():
    from rl4co_b200.eas import eas_coefficients

    with pytest.raises(ValueError, match="not supported"):
        eas_coefficients(torch.zeros(2, 8, 1), "exponential", 0.013, True)


def _tsp(n=20, B=2, device="cpu"):
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    env = get_env("tsp", generator_params=dict(num_loc=n))
    td = env.reset(env.generator(B))
    return FusedAttentionModelPolicy(env_name="tsp", num_encoder_layers=1), env, td


@pytest.mark.parametrize("kw,exc", [
    (dict(use_eas_layer=True), NotImplementedError),
    (dict(use_eas_embedding=False), ValueError),
    (dict(eas_emb_cache_keys=["logit_key", "glimpse_key"]), NotImplementedError),
    (dict(eas_emb_cache_keys=["glimpse_val"]), NotImplementedError),
    (dict(num_parallel_runs=2), NotImplementedError),
    (dict(baseline="exponential"), ValueError),
    (dict(), NotImplementedError),  # CPU tensors
])
def test_eas_search_rejections(kw, exc):
    from rl4co_b200.eas import eas_search

    policy, env, td = _tsp()
    with pytest.raises(exc):
        eas_search(policy, env, td, max_iters=1, **kw)


@pytest.mark.parametrize("env_name,n", [("sdvrp", 20), ("op", 20), ("pctsp", 20), ("tsp", 129), ("cvrp", 128)])
def test_eas_search_rejects_envs_and_sizes(env_name, n):
    from rl4co_b200.eas import eas_search
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    gp = dict(num_loc=n, **({"prize_type": "dist"} if env_name == "op" else {}))
    env = get_env(env_name, generator_params=gp)
    td = env.reset(env.generator(2))
    policy = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=1)
    with pytest.raises(NotImplementedError):
        eas_search(policy, env, td, max_iters=1)


def _abi_args(**over):
    from rl4co_b200 import native

    a = native.EasGradArgs()
    a.env_kind, a.B_inst, a.num_rows, a.N, a.T, a.cache_width = native.ENV_TSP, 0, 2, 20, 20, 5 * 128
    a.tanh_clipping, a.temperature = 10.0, 1.0
    for name in ("cache", "actions", "coef", "dLf", "loglik"):
        setattr(a, name, 4096)
    for k, v in over.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("over,code", [
    (dict(), 0),                                                   # B_inst = 0: nothing to launch
    (dict(env_kind=2), -2), (dict(env_kind=3), -2), (dict(env_kind=7), -2),
    (dict(N=129, T=129), -2), (dict(tanh_clipping=0.0), -2), (dict(cache_width=4 * 128), -2),
    (dict(cache=None), -1), (dict(actions=None), -1), (dict(coef=None), -1), (dict(dLf=None), -1),
    (dict(loglik=None), -1), (dict(B_inst=-1), -1), (dict(N=1, T=1), -1), (dict(num_rows=0), -1), (dict(T=0), -1),
    (dict(T=19), -1), (dict(temperature=0.0), -1), (dict(cache=4100), -1), (dict(dLf=4104), -1),
    (dict(env_kind=1, cache_width=4 * 128), -1),                   # cvrp without demand / w_capacity
    (dict(env_kind=1, cache_width=5 * 128, demand=4096, w_capacity=4096), -1),
    (dict(env_kind=1, cache_width=4 * 128, demand=4096, w_capacity=4096, T=3), 0),
])
def test_abi_argument_checks(over, code):
    from rl4co_b200 import native

    assert "co_eas_key_grad" in native.EXPORTS
    a = _abi_args(**over)
    assert native.lib().co_eas_key_grad(ctypes.byref(a), None) == code, native.lib().co_last_error_string()


def test_binding_checks():
    from rl4co_b200 import native

    cache = torch.zeros(2, 20, 5 * 128)
    acts = torch.zeros(4, 20, dtype=torch.int64)
    with pytest.raises(NotImplementedError):
        native.eas_key_grad("sdvrp", cache, acts, torch.zeros(4))
    with pytest.raises(ValueError, match="coef"):
        native.eas_key_grad("tsp", cache, acts, torch.zeros(3))
    with pytest.raises(ValueError, match="actions"):
        native.eas_key_grad("tsp", cache, acts[:3], torch.zeros(3))
    with pytest.raises(ValueError, match="cvrp needs"):
        native.eas_key_grad("cvrp", torch.zeros(2, 20, 4 * 128), acts, torch.zeros(4))
    with pytest.raises(native.NativeLibraryError, match="CUDA"):
        native.eas_key_grad("tsp", cache, acts, torch.zeros(4))


@pytest.mark.parametrize("env_name,S", [("tsp", 1), ("tsp", 3), ("cvrp", 3)])
def test_reference_key_override_is_exact(env_name, S):
    """The reference with its logit key replaced by the cache's own key gives the default log-probs bit for bit."""
    from rl4co_b200.policy import FusedAttentionModelPolicy

    pol = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=1)
    W = O.float64_weights(name_seeded_weights(pol.state_dict(), 7), ())
    gen = torch.Generator().manual_seed(3)
    inst = O.generate_instances(env_name, 4, 12, generator=gen)
    h, _ = O.encoder_forward(W, env_name, O.env_reset(env_name, inst), num_layers=1)
    src = (O.batchify(inst, S), O.batchify(h, S)) if S > 1 else (inst, h)
    acts = O.rollout(W, env_name, src[0], src[1], decode_type="sampling", generator=gen)["actions"]
    ref = O.teacher_forced_logprobs(W, env_name, inst, h, acts, num_starts=S, forced_first=S > 1)
    key = O.precompute_cache(W, h)["logit_key"]
    got = teacher_forced_logprobs_with_key(W, env_name, inst, h, acts, key, num_starts=S, forced_first=S > 1)
    assert torch.equal(got, ref)
    # another key changes the log-probs and is differentiated: the override reaches the decoder
    leaf = (key + 0.1 * torch.randn(key.shape, generator=gen, dtype=key.dtype)).requires_grad_(True)
    other = teacher_forced_logprobs_with_key(W, env_name, inst, h, acts, leaf, num_starts=S, forced_first=S > 1)
    assert not torch.equal(other, ref)
    other.sum().backward()
    assert leaf.grad is not None and bool(leaf.grad.any())
    assert O.precompute_cache(W, h)["logit_key"] is not leaf  # the oracle is left as it was
