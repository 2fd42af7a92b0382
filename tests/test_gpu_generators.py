"""On-device location laws (`co_generate_locs`, `loc_distribution` / `depot_distribution` of the fused generators).

The law is the contract, not the reference's torch call sequence: every non-uniform kind is compared with rl4co's own
samplers (envs/common/distribution_utils.py, run from the staged reference copy) by two-sample Kolmogorov-Smirnov
tests on statistics that see the node order, the spread and the clustering of an instance.  Exact properties (ranges,
min-max scaling, constants), reproducibility of the Philox streams, the size limits and the path through the five envs
are checked directly.  The uniform default must stay bit-identical to what the generators produced before.
"""

import random

import pytest
import torch

from oracle import ref_standin

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
B_LAW = 4096   # instances per side in the law comparisons
P_MIN = 1e-4


@pytest.fixture(scope="module")
def du():
    if not ref_standin.reference_available():
        pytest.skip("no reference tree (oracle/_ref not staged)")
    ref_standin.install()
    import importlib

    return importlib.import_module("rl4co.envs.common.distribution_utils")


def _gen(shape, kind, seed=1, offset=0, **kw):
    from rl4co_b200 import native

    return native.generate_locs(shape, DEV, seed, offset, kind, **kw)


def _statistics(x: torch.Tensor) -> dict:
    """Per-instance statistics of x [B, N, 2] (float64 on the GPU).  The coordinate samples take one node per instance
    (node b mod N), so every sample is independent of the others."""
    x = x.to(DEV, torch.float64)
    B, N, _ = x.shape
    node = x[torch.arange(B, device=DEV), torch.arange(B, device=DEV) % N]
    d = torch.cdist(x, x)
    d.diagonal(dim1=1, dim2=2).fill_(float("inf"))
    ext = x.amax(1) - x.amin(1)
    out = {"x": node[:, 0], "y": node[:, 1], "mean_nn": d.amin(-1).mean(-1),
           "node0_to_centroid": (x[:, 0] - x.mean(1)).norm(dim=-1), "bbox_area": ext[:, 0] * ext[:, 1]}
    return {k: v.cpu().numpy() for k, v in out.items()}


def _reference(du, setting, B, N, seed):
    torch.manual_seed(seed)
    random.seed(seed)
    kind, kw = setting
    sampler = {"cluster": lambda: du.Cluster(kw["n_cluster"]), "mixed": lambda: du.Mixed(kw["n_cluster_mix"]),
               "gaussian_mixture": lambda: du.Gaussian_Mixture(kw["num_modes"], kw["cdist"]),
               "mix_distribution": lambda: du.Mix_Distribution(kw["n_cluster"], kw["n_cluster_mix"]),
               "mix_multi_distributions": lambda: du.Mix_Multi_Distributions()}[kind]()
    with torch.inference_mode():
        return sampler.sample((B, N, 2))


LAW_SETTINGS = {
    "cluster3": ("cluster", dict(n_cluster=3)),
    "cluster7": ("cluster", dict(n_cluster=7)),
    "mixed1": ("mixed", dict(n_cluster_mix=1)),
    "mixed3": ("mixed", dict(n_cluster_mix=3)),
    "gm0_0": ("gaussian_mixture", dict(num_modes=0, cdist=0)),
    "gm1_1": ("gaussian_mixture", dict(num_modes=1, cdist=1)),
    "gm3_10": ("gaussian_mixture", dict(num_modes=3, cdist=10)),
    "gm7_50": ("gaussian_mixture", dict(num_modes=7, cdist=50)),
    "mix_distribution": ("mix_distribution", dict(n_cluster=3, n_cluster_mix=1)),
    "mix_multi": ("mix_multi_distributions", {}),
}


@pytest.mark.parametrize("n", [20, 100])
@pytest.mark.parametrize("name", list(LAW_SETTINGS))
def test_same_law_as_reference(du, name, n):
    from scipy.stats import ks_2samp

    kind, kw = LAW_SETTINGS[name]
    ours = _statistics(_gen((B_LAW, n, 2), kind, seed=1000 + n, **kw))
    theirs = _statistics(_reference(du, LAW_SETTINGS[name], B_LAW, n, seed=2000 + n))
    pvals = {k: ks_2samp(ours[k], theirs[k]).pvalue for k in ours}
    bad = {k: p for k, p in pvals.items() if p < P_MIN}
    assert not bad, f"{name} N={n}: KS p-values below {P_MIN}: {bad} (all: {pvals})"


# ----------------------------------------------------------------------------- exact properties


@pytest.mark.parametrize("kind,kw", [("cluster", dict(n_cluster=3)), ("cluster", dict(n_cluster=40)),
                                     ("mixed", dict(n_cluster_mix=1)), ("mixed", dict(n_cluster_mix=30)),
                                     ("mix_distribution", dict(n_cluster=5, n_cluster_mix=2))])
def test_clamped_kinds_lie_in_unit_square(kind, kw):
    x = _gen((2048, 50, 2), kind, **kw)
    assert torch.isfinite(x).all() and x.min() >= 0 and x.max() <= 1
    assert ((x == 0) | (x == 1)).any()  # the Gaussian tails did reach the clamp


@pytest.mark.parametrize("m,c", [(3, 10), (7, 50), (2, 0.5), (1, 3), (40, 5)])
@pytest.mark.parametrize("n", [2, 20, 333])
def test_gaussian_mixture_is_min_max_scaled(m, c, n):
    x = _gen((1024, n, 2), "gaussian_mixture", num_modes=m, cdist=c)
    assert (x.amin(1) == 0).all() and (x.amax(1) == 1).all()


@pytest.mark.parametrize("n", [2, 20, 100, 1000])
def test_gaussian_mixture_1_1_is_scaled_by_the_larger_range_and_centred(n):
    x = _gen((1024, n, 2), "gaussian_mixture", num_modes=1, cdist=1)
    lo, hi = x.amin(1), x.amax(1)
    wide = (hi - lo).argmax(-1)
    rows = torch.arange(x.shape[0], device=DEV)
    assert (lo[rows, wide] == 0).all() and (hi[rows, wide] == 1).all()
    torch.testing.assert_close(lo + hi, torch.ones_like(lo), rtol=0, atol=1e-6)
    # the narrower coordinate keeps its aspect: it spans strictly less than [0, 1] in most instances
    assert ((hi - lo).amin(-1) < 0.999).float().mean() > 0.5


def test_mix_multi_distributions_is_scaled_per_instance():
    x = _gen((4096, 30, 2), "mix_multi_distributions")
    lo, hi = x.amin(1), x.amax(1)
    assert (x >= 0).all() and (x <= 1).all()
    # (0, 0) is U(0, 1)^2, so about 1/11 of the instances touch neither 0 nor 1; the other ten settings are scaled so
    # that a coordinate spans [0, 1] exactly and both are centred
    touch = ((lo == 0) & (hi == 1)).any(-1)
    assert 1 - 3 / 11 < touch.float().mean().item() < 1 - 0.5 / 11
    torch.testing.assert_close((lo + hi)[touch], torch.ones_like(lo[touch]), rtol=0, atol=1e-6)


def test_constant_and_normal_kinds():
    x = _gen((64, 7, 2), "constant", value=0.375)
    assert (x == 0.375).all()
    x = _gen((20000, 50, 2), "normal", mean=0.5, std=0.3)
    assert abs(x.mean().item() - 0.5) < 2e-3 and abs(x.std().item() - 0.3) < 2e-3
    assert (x < 0).any() and (x > 1).any()  # no clamp
    assert torch.isfinite(x).all()


# ----------------------------------------------------------------------------- reproducibility and shape


KINDS = [("cluster", dict(n_cluster=3)), ("mixed", dict(n_cluster_mix=2)),
         ("gaussian_mixture", dict(num_modes=1, cdist=1)), ("gaussian_mixture", dict(num_modes=5, cdist=30)),
         ("mix_distribution", dict(n_cluster=3, n_cluster_mix=1)), ("mix_multi_distributions", {}),
         ("normal", dict(mean=0.2, std=1.0)), ("uniform", dict(lo=-1.0, hi=2.0))]


@pytest.mark.parametrize("kind,kw", KINDS)
def test_streams_are_reproducible_and_prefix_stable(kind, kw):
    a = _gen((3000, 37, 2), kind, seed=5, offset=9, **kw)
    assert torch.equal(a, _gen((3000, 37, 2), kind, seed=5, offset=9, **kw))
    assert torch.equal(a[:17], _gen((17, 37, 2), kind, seed=5, offset=9, **kw))
    assert not torch.equal(a, _gen((3000, 37, 2), kind, seed=5, offset=10, **kw))
    assert not torch.equal(a, _gen((3000, 37, 2), kind, seed=6, offset=9, **kw))
    assert torch.equal(a.view(3, 1000, 37, 2), _gen((3, 1000, 37, 2), kind, seed=5, offset=9, **kw))


@pytest.mark.parametrize("kind,kw", KINDS + [("constant", dict(value=0.5))])
def test_node_count_limits(kind, kw):
    from rl4co_b200 import native

    needs_two = kind == "mix_multi_distributions" or (kind == "gaussian_mixture" and kw["num_modes"] != 0)
    if needs_two:
        with pytest.raises(native.NativeLibraryError, match="N >= 2"):
            _gen((4, 1, 2), kind, **kw)
    else:
        assert torch.isfinite(_gen((4, 1, 2), kind, **kw)).all()
    for n in (2, 10000):
        x = _gen((3, n, 2), kind, **kw)
        assert torch.isfinite(x).all()
    with pytest.raises(native.NativeLibraryError, match="outside"):
        _gen((3, 10001, 2), kind, **kw)


def test_large_batch_completes():
    x = _gen((65536, 100, 2), "mix_multi_distributions", seed=3)
    y = _gen((65536, 100, 2), "mixed", seed=3, n_cluster_mix=3)
    torch.cuda.synchronize()
    assert torch.isfinite(x).all() and torch.isfinite(y).all()


def test_cpu_device_raises():
    from rl4co_b200 import native

    with pytest.raises(native.NativeLibraryError):
        native.generate_locs((4, 10, 2), "cpu", 0, 0, "cluster", n_cluster=3)


# ----------------------------------------------------------------------------- through the envs


ENV_LAWS = [("cluster", dict(n_cluster=3)), ("mixed", dict(n_cluster_mix=2)),
            ("gaussian_mixture", dict(num_modes=3, cdist=10)), ("mix_multi_distributions", {}),
            ("normal", dict(loc_mean=0.5, loc_std=0.2))]


@pytest.mark.parametrize("depot", [None, "center"])
@pytest.mark.parametrize("law", range(len(ENV_LAWS)), ids=[k for k, _ in ENV_LAWS])
@pytest.mark.parametrize("env_name", ["tsp", "cvrp", "sdvrp", "op", "pctsp"])
def test_envs_roll_out_on_generated_instances(env_name, law, depot):
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    kind, kw = ENV_LAWS[law]
    env = get_env(env_name, check_solution=True,
                  generator_params=dict(num_loc=50, loc_distribution=kind, depot_distribution=depot, device="cuda",
                                        seed=11, **kw))
    torch.manual_seed(0)
    policy = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=2).to(DEV).eval()
    with torch.inference_mode():
        td = env.reset(batch_size=[256])
        assert td["locs"].is_cuda and td["locs"].shape[-2] == (50 if env_name == "tsp" else 51)
        if depot == "center" and env_name != "tsp":
            assert (td["locs"][:, 0] == 0.5).all()
        out = policy(td, env, phase="test", decode_type="greedy")
    assert torch.isfinite(out["reward"]).all()


def test_separate_depot_laws():
    from rl4co_b200.envs import CVRPGenerator

    g = CVRPGenerator(num_loc=20, min_loc=0.25, max_loc=1.0, loc_distribution="cluster", n_cluster=3,
                      depot_distribution="center", device="cuda", seed=1)
    assert (g(8)["depot"] == 0.375).all()  # the reference's (max - min) / 2
    g = CVRPGenerator(num_loc=20, loc_distribution="mixed", n_cluster_mix=1, depot_distribution="corner",
                      min_loc=0.25, device="cuda", seed=1)
    assert (g(8)["depot"] == 0.25).all()
    g = CVRPGenerator(num_loc=20, depot_distribution="normal", depot_mean=3.0, depot_std=0.5, device="cuda", seed=1)
    d = g(20000)["depot"]
    assert abs(d.mean().item() - 3.0) < 0.02 and abs(d.std().item() - 0.5) < 0.02
    g = CVRPGenerator(num_loc=20, depot_distribution="uniform", device="cuda", seed=1)
    td = g(4096)
    assert td["depot"].min() >= 0 and td["depot"].max() < 1 and td["locs"].shape == (4096, 20, 2)
    assert not torch.equal(td["depot"], td["locs"][:, 0])


# ----------------------------------------------------------------------------- uniform unchanged


def _legacy_uniform(env_name, batch, n, seed, calls):
    """What the generators computed before location laws existed (device path): the locations of call `calls`."""
    from rl4co_b200 import native

    streams = {"tsp": 1, "cvrp": 2, "sdvrp": 2, "op": 2, "pctsp": 4}[env_name]
    nodes = n if env_name == "tsp" else n + 1
    return native.generate_uniform((*batch, nodes, 2), DEV, seed, calls * streams, 0.0, 1.0)


@pytest.mark.parametrize("env_name", ["tsp", "cvrp", "sdvrp", "op", "pctsp"])
def test_uniform_spellings_are_bit_identical_to_the_default(env_name):
    from torch.distributions import Uniform

    from rl4co_b200.envs import get_env

    outs = []
    for spelling in ({}, dict(loc_distribution="uniform"), dict(loc_distribution=Uniform)):
        for device in ("cpu", "cuda"):
            torch.manual_seed(4)
            env = get_env(env_name, generator_params=dict(num_loc=30, device=device if device == "cuda" else None,
                                                          seed=9, **spelling))
            tds = [env.generator([2, 64]) for _ in range(2)]
            outs.append((device, tds))
    for device in ("cpu", "cuda"):
        ref = [tds for d, tds in outs if d == device]
        for other in ref[1:]:
            for a, b in zip(ref[0], other):
                for k in a.keys():
                    assert torch.equal(a[k], b[k]), (device, k)
    # and the device path is still the generator's original stream
    for call, td in enumerate([tds for d, tds in outs if d == "cuda"][0]):
        legacy = _legacy_uniform(env_name, [2, 64], 30, 9, call)
        got = td["locs"] if env_name == "tsp" else torch.cat([td["depot"][..., None, :], td["locs"]], -2)
        assert torch.equal(got, legacy)
