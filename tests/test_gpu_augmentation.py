"""GPU: symmetric augmentation on the device.  `co_symmetric_augment` equals the reference's `symmetric_transform`
(data/transforms.py:49-69) run by torch on CUDA tensors bit for bit; `StateAugmentation(augment_fn="symmetric")` on a
CUDA TensorDict equals the reference's `StateAugmentation` after the same seed; `pomo_step` returns the tours behind
`max_reward` / `max_aug_reward` (pomo/model.py:112-140)."""

import math

import numpy as np
import pytest
import torch

from oracle import ref_standin

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not ref_standin.reference_available(), reason="reference files not staged")]
DEV = "cuda:0"


def _ref():
    return ref_standin.load().transforms


def _angles(S, B, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    phi = torch.rand(S * B, device=DEV, generator=g) * 4 * math.pi
    phi[:B] = 0.0
    return phi


def _reference_images(base, phi, S, a0=0, a1=None):
    """Rows a0*B .. a1*B of the reference's transform of the batchified base (its rows are copies of base)."""
    a1 = S if a1 is None else a1
    B = base.shape[0]
    xy = base.repeat(a1 - a0, 1, 1)
    return _ref().symmetric_transform(xy[..., [0]], xy[..., [1]], phi[a0 * B:a1 * B, None, None])


@pytest.mark.parametrize("B", [1, 37, 4096])
@pytest.mark.parametrize("S", [2, 8, 33])
@pytest.mark.parametrize("N", [1, 20, 100, 1000])
def test_kernel_equals_reference_transform(B, S, N):
    from rl4co_b200 import native

    g = torch.Generator(device=DEV).manual_seed(B * 1000 + S * 10 + N)
    base = torch.rand(B, N, 2, device=DEV, generator=g)
    phi = _angles(S, B, B + S + N)
    out = native.symmetric_augment(base, phi, S)
    assert out.shape == (S * B, N, 2)
    step = max(1, (1 << 27) // (B * N * 2))  # compare at most ~128 M floats of the reference at a time
    for a0 in range(0, S, step):
        a1 = min(S, a0 + step)
        assert torch.equal(out[a0 * B:a1 * B], _reference_images(base, phi, S, a0, a1)), (a0, a1)


def test_kernel_reflects_where_the_reference_does():
    """fp32(2*pi) and its lower neighbour rotate only, its upper neighbour and the angle below 4*pi reflect; 0 is
    (x - 0.5) + 0.5.  Every row of image a >= 1 gets one of the boundary angles."""
    from rl4co_b200 import native

    two_pi, four_pi = np.float32(2 * math.pi), np.float32(4 * math.pi)
    edge = torch.tensor([two_pi, np.nextafter(two_pi, np.float32(0)), np.nextafter(two_pi, np.float32(7)), 0.0,
                         np.nextafter(four_pi, np.float32(0))], dtype=torch.float32, device=DEV)
    assert (edge > 2 * math.pi).tolist() == [False, False, True, False, True]
    B, S, N = 7, 6, 50
    base = torch.rand(B, N, 2, device=DEV, generator=torch.Generator(device=DEV).manual_seed(9))
    phi = torch.cat((torch.zeros(B, device=DEV), edge.repeat((S - 1) * B // 5 + 1)[: (S - 1) * B]))
    out = native.symmetric_augment(base, phi, S)
    assert torch.equal(out, _reference_images(base, phi, S))
    # the rotation alone, in the reference's operation order: reflected rows are its mirror image (x <-> y)
    x0, y0 = base[..., [0]].repeat(S, 1, 1) - 0.5, base[..., [1]].repeat(S, 1, 1) - 0.5
    c, s = torch.cos(phi)[:, None, None], torch.sin(phi)[:, None, None]
    rot = torch.cat((c * x0 - s * y0, s * x0 + c * y0), -1) + 0.5
    refl = phi > 2 * math.pi
    assert refl.any() and (~refl[B:]).any()
    assert torch.equal(out[refl], rot[refl].flip(-1)) and torch.equal(out[~refl], rot[~refl])


def test_kernel_output_beyond_2_31_floats():
    """S * B * N * 2 = 2 148 352 000 floats (> 2^31): 64-bit indexing, every image compared."""
    from rl4co_b200 import native

    B, S, N = 1024, 1049, 1000
    assert 2 * B * S * N > 2 ** 31
    base = torch.rand(B, N, 2, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    phi = _angles(S, B, 2)
    out = native.symmetric_augment(base, phi, S)
    for a0 in range(0, S, 64):
        a1 = min(S, a0 + 64)
        assert torch.equal(out[a0 * B:a1 * B], _reference_images(base, phi, S, a0, a1)), (a0, a1)
    del out
    torch.cuda.empty_cache()


def _td(layout, B, N, seed):
    from rl4co_b200.tensordict import TensorDict

    g = torch.Generator(device=DEV).manual_seed(seed)
    d = {"locs": torch.rand(B, N + (layout == "cvrp"), 2, device=DEV, generator=g),
         "targets": torch.rand(B, 9, 2, device=DEV, generator=g)}
    if layout == "cvrp":
        d["demand"] = torch.randint(1, 10, (B, N), device=DEV, generator=g).float() / 40
    return TensorDict(d, batch_size=[B])


@pytest.mark.parametrize("layout", ["tsp", "cvrp"])
@pytest.mark.parametrize("num_augment", [2, 8, 16])
@pytest.mark.parametrize("first_aug_identity,normalize", [(True, False), (False, False), (True, True)])
@pytest.mark.parametrize("feats", [None, ["locs", "targets"]])
def test_state_augmentation_on_device_equals_reference(layout, num_augment, first_aug_identity, normalize, feats):
    from rl4co_b200 import native
    from rl4co_b200.ops import StateAugmentation

    td = _td(layout, 33, 50, num_augment)
    kw = dict(num_augment=num_augment, augment_fn="symmetric", first_aug_identity=first_aug_identity,
              normalize=normalize, feats=feats)
    torch.manual_seed(11)
    launches = native.LAUNCH_COUNT
    ours = StateAugmentation(**kw)(td.clone())
    assert native.LAUNCH_COUNT - launches == (1 if feats is None else len(feats))  # the kernel ran for each feature
    torch.manual_seed(11)
    theirs = _ref().StateAugmentation(**kw)(td.clone())
    assert set(ours.keys()) == set(theirs.keys())
    for k in theirs.keys():
        assert ours[k].is_cuda and torch.equal(ours[k], theirs[k]), k


def _pomo_setup(env_name, n, B, seed=0):
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    torch.manual_seed(seed)
    env = get_env(env_name, generator_params=dict(num_loc=n), check_solution=True)
    pol = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=2, use_graph_context=False).to(DEV).eval()
    td = env.reset(env.generator(B).to(DEV))
    return env, pol, td


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_pomo_step_symmetric_returns_the_best_tours(env_name):
    from rl4co_b200.ops import StateAugmentation
    from rl4co_b200.reinforce import pomo_step
    from rl4co_b200.tensordict import TensorDict

    B, A = 64, 16
    env, pol, td = _pomo_setup(env_name, 50, B)
    torch.manual_seed(5)
    res = pomo_step(pol, env, td, num_augment=A, phase="test", augment_fn="symmetric")
    S = env.get_num_starts(td)
    reward, max_reward, acts = res["reward"], res["max_reward"], res["actions"]
    T = acts.shape[1]
    assert reward.shape == (B, A, S) and max_reward.shape == (B, A) and res["max_aug_reward"].shape == (B,)
    assert res["best_multistart_actions"].shape == (B, A, T) and res["best_aug_actions"].shape == (B, T)
    # the start max_reward names: the first start s with reward[b, a, s] == max_reward[b, a]; flat row s*A*B + a*B + b
    s_best = (reward == max_reward[..., None]).float().argmax(-1)
    rows = s_best * (A * B) + torch.arange(A, device=DEV)[None, :] * B + torch.arange(B, device=DEV)[:, None]
    assert torch.equal(res["best_multistart_actions"], acts[rows])
    # the augmentation max_aug_reward names, and the reward of its tour on that augmented instance
    a_best = (max_reward == res["max_aug_reward"][:, None]).float().argmax(-1)
    assert torch.equal(res["best_aug_actions"], res["best_multistart_actions"][torch.arange(B, device=DEV), a_best])
    env.check_solution_validity(td, res["best_aug_actions"])  # on the un-augmented instances
    torch.manual_seed(5)
    td_aug = StateAugmentation(num_augment=A, augment_fn="symmetric")(td)  # the same angles pomo_step drew
    rows = a_best * B + torch.arange(B, device=DEV)
    own = TensorDict({k: v[rows] for k, v in td_aug.items()}, batch_size=[B])
    r = env.get_reward(own, res["best_aug_actions"])
    # the rollout kernel sums the tour as it goes and the reward kernel in tour order: round-off apart
    torch.testing.assert_close(r, res["max_aug_reward"], rtol=1e-5, atol=1e-5)
    # without augmentation: [B, T], the tour of max_reward
    plain = pomo_step(pol, env, td, num_augment=0, phase="test")
    s0 = (plain["reward"] == plain["max_reward"][:, None]).float().argmax(-1)
    assert torch.equal(plain["best_multistart_actions"], plain["actions"][s0 * B + torch.arange(B, device=DEV)])
    assert "best_aug_actions" not in plain
