"""CPU: efficient active search with a per-instance layer (EAS-Lay) -- the argument checks of `co_eas_layer_grad`, of
the rollout's `eas_layer` field and of their bindings, the rejections of `eas_search`, the float64 reference's layer
override, and the layer initialisation against rl4co's `EASLayerNet`."""

import ctypes
import importlib.util
import os

import pytest
import torch

from conftest import name_seeded_weights
from eas_layer_oracle import teacher_forced_logprobs_with_layer
from oracle import am_rollout_oracle as O
from oracle import ref_standin

E = 128


def _grad_args(**over):
    from rl4co_b200 import native

    a = native.EasLayerGradArgs()
    a.env_kind, a.B_inst, a.num_rows, a.N, a.T, a.cache_width = native.ENV_TSP, 0, 2, 20, 20, 5 * E
    a.tanh_clipping, a.temperature = 10.0, 1.0
    for name in ("cache", "actions", "coef", "layer", "dlayer", "loglik"):
        setattr(a, name, 4096)
    for k, v in over.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("over,code", [
    (dict(), 0),                                                   # B_inst = 0: nothing to launch
    (dict(env_kind=2), -2), (dict(env_kind=3), -2), (dict(env_kind=7), -2),
    (dict(N=129, T=129), -2), (dict(tanh_clipping=0.0), -2), (dict(cache_width=4 * E), -2),
    (dict(cache=None), -1), (dict(actions=None), -1), (dict(coef=None), -1), (dict(layer=None), -1),
    (dict(dlayer=None), -1), (dict(loglik=None), -1), (dict(B_inst=-1), -1), (dict(N=1, T=1), -1),
    (dict(num_rows=0), -1), (dict(T=0), -1), (dict(T=19), -1), (dict(temperature=0.0), -1),
    (dict(cache=4100), -1), (dict(layer=4104), -1), (dict(dlayer=4108), -1),
    (dict(env_kind=1, cache_width=4 * E), -1),                     # cvrp without demand / w_capacity
    (dict(env_kind=1, cache_width=5 * E, demand=4096, w_capacity=4096), -1),
    (dict(env_kind=1, cache_width=4 * E, demand=4096, w_capacity=4096, T=3), 0),
])
def test_layer_grad_abi_argument_checks(over, code):
    from rl4co_b200 import native

    assert "co_eas_layer_grad" in native.EXPORTS
    a = _grad_args(**over)
    assert native.lib().co_eas_layer_grad(ctypes.byref(a), None) == code, native.lib().co_last_error_string()


def _rollout_args(**over):
    from rl4co_b200 import native

    a = native.RolloutArgs()
    a.env_kind, a.select_mode, a.B_inst, a.num_starts = native.ENV_TSP, native.SELECT_SAMPLE_PHILOX, 0, 4
    a.N, a.T_max, a.num_loc, a.flags = 20, 20, 20, native.ROLLOUT_FORCED_START
    a.tanh_clipping, a.temperature = 10.0, 1.0
    for name in ("cache", "locs", "actions_out", "logp_out", "reward_out", "loglik_out", "eas_layer"):
        setattr(a, name, 4096)
    for k, v in over.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("over,code", [
    (dict(), 0), (dict(env_kind=1), 0), (dict(eas_layer=None), 0), (dict(eas_layer=None, num_starts=1), 0),
    (dict(num_starts=1), -2), (dict(env_kind=2), -2), (dict(env_kind=3), -2), (dict(env_kind=4), -2),
    (dict(eas_layer=4100), -1), (dict(eas_layer=4104, env_kind=1), -1),
])
def test_rollout_layer_abi_argument_checks(over, code):
    from rl4co_b200 import native

    a = _rollout_args(**over)
    assert native.lib().co_rollout(ctypes.byref(a), None) == code, native.lib().co_last_error_string()


def test_layer_bindings_check_arguments():
    from rl4co_b200 import native

    cache = torch.zeros(2, 20, 5 * E)
    acts = torch.zeros(4, 20, dtype=torch.int64)
    layer = torch.zeros(2, native.EAS_LAYER_FLOATS)
    assert native.EAS_LAYER_FLOATS == 2 * E * E + 2 * E
    with pytest.raises(NotImplementedError):
        native.eas_layer_grad("op", cache, acts, torch.zeros(4), layer)
    with pytest.raises(ValueError, match="layer"):
        native.eas_layer_grad("tsp", cache, acts, torch.zeros(4), layer[:1])
    with pytest.raises(ValueError, match="layer"):
        native.eas_layer_grad("tsp", cache, acts, torch.zeros(4), None)
    with pytest.raises(ValueError, match="coef"):
        native.eas_layer_grad("tsp", cache, acts, torch.zeros(3), layer)
    with pytest.raises(native.NativeLibraryError, match="CUDA"):
        native.eas_layer_grad("tsp", cache, acts, torch.zeros(4), layer)
    locs = torch.zeros(2, 20, 2)
    with pytest.raises(NotImplementedError, match="multistart"):
        native.rollout("tsp", native.SELECT_SAMPLE_PHILOX, cache, None, torch.zeros(E), None, locs, None, None, 2,
                       20, num_starts=1, layer=layer)
    with pytest.raises(ValueError, match="layer"):
        native.rollout("tsp", native.SELECT_SAMPLE_PHILOX, cache, None, torch.zeros(E), None, locs, None, None, 2,
                       20, num_starts=4, forced_start=True, num_loc=20, layer=layer[:, :10])


def _env(env_name, n, B=2):
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    gp = dict(num_loc=n, **({"prize_type": "dist"} if env_name == "op" else {}))
    env = get_env(env_name, generator_params=gp)
    return FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=1), env, env.reset(env.generator(B))


def test_eas_search_refuses_both_variants_together():
    from rl4co_b200.eas import eas_search

    policy, env, td = _env("tsp", 20)
    with pytest.raises(NotImplementedError, match="together"):
        eas_search(policy, env, td, max_iters=1, use_eas_layer=True, use_eas_embedding=True)
    with pytest.raises(ValueError, match="At least one"):
        eas_search(policy, env, td, max_iters=1, use_eas_layer=False, use_eas_embedding=False)


@pytest.mark.parametrize("env_name,n,kw", [
    ("sdvrp", 20, {}), ("op", 20, {}), ("pctsp", 20, {}), ("tsp", 129, {}), ("cvrp", 128, {}),
    ("tsp", 20, dict(num_parallel_runs=2)), ("tsp", 20, {}),       # the last: CPU tensors
])
def test_eas_search_layer_rejections(env_name, n, kw):
    from rl4co_b200.eas import eas_search

    policy, env, td = _env(env_name, n)
    with pytest.raises(NotImplementedError):
        eas_search(policy, env, td, max_iters=1, use_eas_layer=True, use_eas_embedding=False, **kw)


def _layer(B, gen, scale):
    return {"W1": scale * torch.randn(B, E, E, generator=gen, dtype=torch.float64),
            "b1": scale * torch.randn(B, 1, E, generator=gen, dtype=torch.float64),
            "W2": scale * torch.randn(B, E, E, generator=gen, dtype=torch.float64),
            "b2": scale * torch.randn(B, 1, E, generator=gen, dtype=torch.float64)}


@pytest.mark.parametrize("env_name,S", [("tsp", 1), ("tsp", 3), ("cvrp", 3)])
def test_reference_layer_override_is_exact(env_name, S):
    """W2 = b2 = 0 gives the default log-probs bit for bit; another layer changes them and is differentiated."""
    from rl4co_b200.policy import FusedAttentionModelPolicy

    pol = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=1)
    W = O.float64_weights(name_seeded_weights(pol.state_dict(), 7), ())
    gen = torch.Generator().manual_seed(3)
    B = 4
    inst = O.generate_instances(env_name, B, 12, generator=gen)
    h, _ = O.encoder_forward(W, env_name, O.env_reset(env_name, inst), num_layers=1)
    src = (O.batchify(inst, S), O.batchify(h, S)) if S > 1 else (inst, h)
    acts = O.rollout(W, env_name, src[0], src[1], decode_type="sampling", generator=gen)["actions"]
    ref = O.teacher_forced_logprobs(W, env_name, inst, h, acts, num_starts=S, forced_first=S > 1)
    zero = _layer(B, gen, 0.1)
    zero["W2"].zero_()
    zero["b2"].zero_()
    got = teacher_forced_logprobs_with_layer(W, env_name, inst, h, acts, zero, num_starts=S, forced_first=S > 1)
    assert torch.equal(got, ref)
    leaves = {k: v.clone().requires_grad_(True) for k, v in _layer(B, gen, 0.05).items()}
    other = teacher_forced_logprobs_with_layer(W, env_name, inst, h, acts, leaves, num_starts=S, forced_first=S > 1)
    assert not torch.equal(other, ref)
    other.sum().backward()
    assert all(v.grad is not None and bool(v.grad.any()) for v in leaves.values())
    assert O.pointer_logits.__module__ == O.__name__  # the oracle is left as it was


def _reference_eas_nn():
    path = os.path.join(ref_standin.REFERENCE_ROOT, "rl4co", "models", "zoo", "eas", "nn.py")
    if not os.path.exists(path):
        return None
    spec = importlib.util.spec_from_file_location("_rl4co_eas_nn", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.skipif(_reference_eas_nn() is None, reason="the reference's rl4co/models/zoo/eas/nn.py is not present")
@pytest.mark.parametrize("n", [1, 6, 24])
def test_layer_init_matches_reference(n):
    from rl4co_b200.eas import eas_layer_init, unpack_eas_layer

    torch.manual_seed(123 + n)
    ref = _reference_eas_nn().EASLayerNet(n, E)
    torch.manual_seed(123 + n)
    got = unpack_eas_layer(eas_layer_init(n))
    for k in ("W1", "b1", "W2", "b2"):
        assert got[k].shape == getattr(ref, k).shape
        assert torch.equal(got[k], getattr(ref, k).detach()), k
    assert not got["W1"].eq(0).all() and got["W2"].eq(0).all() and got["b2"].eq(0).all()
