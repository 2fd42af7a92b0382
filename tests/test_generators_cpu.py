"""Argument handling of the generators' location laws (`loc_distribution` / `depot_distribution`), which needs no GPU:
the CPU stream serves uniform locations only and says so, unsupported spellings and missing parameters fail at
construction, and the kernel behind the device laws is exported."""

import ctypes

import pytest
import torch
from torch.distributions import Exponential, Normal, Uniform

from rl4co_b200 import native
from rl4co_b200.envs import CVRPGenerator, OPGenerator, PCTSPGenerator, TSPGenerator, get_env

GENERATORS = [TSPGenerator, CVRPGenerator, OPGenerator, PCTSPGenerator]
DEVICE_LAWS = [("cluster", dict(n_cluster=3)), ("mixed", dict(n_cluster_mix=1)),
               ("gaussian_mixture", dict(num_modes=3, cdist=10)), ("mix_distribution", dict(n_cluster=3, n_cluster_mix=1)),
               ("mix_multi_distributions", {}), ("normal", dict(loc_mean=0.5, loc_std=0.1)), ("gaussian", dict(loc_mean=0.5, loc_std=0.1)),
               ("center", {}), ("corner", {}), (0.25, {}), (1, {})]


@pytest.mark.parametrize("gen", GENERATORS)
@pytest.mark.parametrize("law", range(len(DEVICE_LAWS)), ids=[str(k) for k, _ in DEVICE_LAWS])
def test_non_uniform_laws_need_the_device(gen, law):
    kind, kw = DEVICE_LAWS[law]
    with pytest.raises(NotImplementedError, match='device="cuda"'):
        gen(num_loc=10, loc_distribution=kind, **kw)


@pytest.mark.parametrize("gen", [CVRPGenerator, OPGenerator, PCTSPGenerator])
@pytest.mark.parametrize("depot", ["center", "corner", 0.5, "normal"])
def test_non_uniform_depot_needs_the_device(gen, depot):
    with pytest.raises(NotImplementedError, match='device="cuda"'):
        gen(num_loc=10, depot_distribution=depot, depot_mean=0.5, depot_std=0.1)


@pytest.mark.parametrize("gen", GENERATORS)
@pytest.mark.parametrize("dist", [Normal, Exponential, "exponential", "poisson", lambda **kw: Uniform(0, 1)])
def test_unsupported_distributions_raise(gen, dist):
    with pytest.raises(NotImplementedError):
        gen(num_loc=10, loc_distribution=dist, device="cuda", loc_rate=1.0)


@pytest.mark.parametrize("gen", GENERATORS)
@pytest.mark.parametrize("key", ["loc_sampler", "depot_sampler"])
def test_sampler_objects_raise(gen, key):
    with pytest.raises(NotImplementedError, match=key):
        gen(num_loc=10, device="cuda", **{key: Uniform(0.0, 1.0)})


@pytest.mark.parametrize("gen", GENERATORS)
@pytest.mark.parametrize("kind,given,missing", [("cluster", {}, "n_cluster"), ("mixed", {}, "n_cluster_mix"),
                                                ("gaussian_mixture", dict(num_modes=3), "cdist"),
                                                ("gaussian_mixture", dict(cdist=3), "num_modes"),
                                                ("mix_distribution", dict(n_cluster=3), "n_cluster_mix"),
                                                ("mix_distribution", dict(n_cluster_mix=3), "n_cluster"),
                                                ("normal", dict(loc_mean=0.5), "loc_std"),
                                                ("normal", dict(loc_std=0.5), "loc_mean")])
def test_missing_parameter_is_named(gen, kind, given, missing):
    with pytest.raises(ValueError, match=f"'{missing}'"):
        gen(num_loc=10, loc_distribution=kind, device="cuda", **given)


@pytest.mark.parametrize("gen", [CVRPGenerator, OPGenerator, PCTSPGenerator])
@pytest.mark.parametrize("depot", ["cluster", "mixed", "gaussian_mixture", "mix_distribution", "mix_multi_distributions"])
def test_depot_takes_only_single_point_laws(gen, depot):
    with pytest.raises(ValueError, match="depot"):
        gen(num_loc=10, depot_distribution=depot, device="cuda", n_cluster=3, n_cluster_mix=1, num_modes=3, cdist=1)


def test_unknown_name_raises_value_error():
    with pytest.raises(ValueError, match="Invalid distribution"):
        TSPGenerator(num_loc=10, loc_distribution="triangular", device="cuda")


@pytest.mark.parametrize("env_name", ["tsp", "cvrp", "sdvrp", "op", "pctsp"])
@pytest.mark.parametrize("spelling", ["uniform", Uniform])
def test_uniform_spellings_are_the_default_on_cpu(env_name, spelling):
    torch.manual_seed(3)
    a = [get_env(env_name, generator_params=dict(num_loc=15)).generator([4, 8]) for _ in range(2)]
    torch.manual_seed(3)
    b = [get_env(env_name, generator_params=dict(num_loc=15, loc_distribution=spelling)).generator([4, 8])
         for _ in range(2)]
    for x, y in zip(a, b):
        assert sorted(x.keys()) == sorted(y.keys())
        for k in x.keys():
            assert torch.equal(x[k], y[k]), k


@pytest.mark.parametrize("gen", [CVRPGenerator, OPGenerator, PCTSPGenerator])
def test_uniform_depot_is_drawn_first_on_cpu(gen):
    # rl4co's order with a depot sampler: depot [*B, 2] first, then the num_loc locations
    torch.manual_seed(5)
    td = gen(num_loc=12, min_loc=0.5, max_loc=2.0, depot_distribution="uniform")(6)
    torch.manual_seed(5)
    depot = torch.rand(6, 2) * 1.5 + 0.5
    locs = torch.rand(6, 12, 2) * 1.5 + 0.5
    assert torch.equal(td["depot"], depot) and torch.equal(td["locs"], locs)


def test_tsp_has_no_depot_law():
    # like rl4co's TSPGenerator, a depot law does not apply to an instance without a depot
    torch.manual_seed(1)
    a = TSPGenerator(num_loc=9)(3)
    torch.manual_seed(1)
    b = TSPGenerator(num_loc=9, depot_distribution="center")(3)
    assert torch.equal(a["locs"], b["locs"])


def test_generate_locs_is_exported_and_rejects_cpu():
    assert "co_generate_locs" in native.EXPORTS
    if __import__("os").path.exists(native.LIB_PATH):
        assert hasattr(ctypes.CDLL(native.LIB_PATH), "co_generate_locs")
    with pytest.raises(native.NativeLibraryError, match="CUDA"):
        native.generate_locs((2, 10, 2), "cpu", 0, 0, "cluster", n_cluster=3)
    with pytest.raises(ValueError, match="unknown kind"):
        native.generate_locs((2, 10, 2), "cuda", 0, 0, "triangle")
    with pytest.raises(ValueError, match="shape"):
        native.generate_locs((2, 10, 3), "cuda", 0, 0, "uniform")
    assert ctypes.sizeof(native.LocsArgs) == 64
