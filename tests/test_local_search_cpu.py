"""CPU tests of FusedTSPEnv.local_search: the ls_tsp fixture is what the live reference's numba 2-opt returns today
(regenerated through tests/golden/make_golden_ls.py, skipped without the reference tree or numba), and the public method
rejects malformed arguments and CPU tensors before any kernel runs."""

import importlib.util
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR


def _make_golden():
    from oracle import ref_standin

    if not ref_standin.reference_available():
        pytest.skip("no reference tree (oracle/_ref not staged)")
    pytest.importorskip("numba")
    spec = importlib.util.spec_from_file_location("make_golden_ls", os.path.join(GOLDEN_DIR, "make_golden_ls.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_ls_tsp_fixture_matches_live_reference():
    mg = _make_golden()
    fresh = mg.ls_tsp_fixture()
    stored = np.load(os.path.join(GOLDEN_DIR, "ls_tsp.npz"))
    assert sorted(fresh) == sorted(stored.files)
    for k in stored.files:
        assert fresh[k].dtype == stored[k].dtype and np.array_equal(fresh[k], stored[k]), k
    # the fixture exercises what it claims to: improvements, ties and both distance sources
    cases = {k.split("::")[0] for k in stored.files}
    assert {"rand2", "rand3", "rand1000", "am100", "lattice50", "asym50", "asym300", "rand100_it0"} <= cases
    assert not np.array_equal(stored["rand100::tours_in"], stored["rand100::tours_out"])
    assert np.array_equal(stored["rand100_it0::tours_in"], stored["rand100_it0::tours_out"])


def _env_and_td(n=6, b=3, device="cpu"):
    from rl4co_b200.envs import get_env
    from rl4co_b200.tensordict import TensorDict

    env = get_env("tsp", generator_params=dict(num_loc=n))
    td = TensorDict({"locs": torch.rand(b, n, 2, device=device)}, batch_size=[b])
    return env, td, torch.arange(n).repeat(b, 1)


def test_local_search_argument_errors():
    from rl4co_b200.envs import FusedTSPEnv
    from rl4co_b200.tensordict import TensorDict

    env, td, tours = _env_and_td()
    with pytest.raises(ValueError):
        env.local_search(td, tours[:, :5])  # not one tour over every node
    with pytest.raises(ValueError):
        env.local_search(td, tours[0])  # not [B, N]
    with pytest.raises(ValueError):
        env.local_search(td, tours[:2])  # batch mismatch
    with pytest.raises(ValueError):
        FusedTSPEnv.local_search(TensorDict({"distances": torch.rand(3, 6, 6, dtype=torch.float64)}, batch_size=[3]),
                                 tours)
    with pytest.raises(ValueError):
        FusedTSPEnv.local_search(TensorDict({"locs": torch.rand(2, 3, 6, 2)}, batch_size=[2, 3]),
                                 torch.arange(6).repeat(2, 3, 1))
    with pytest.raises(TypeError):
        env.local_search(td, tours, max_iteration=3)  # unknown keyword, as in the reference's signature


def test_local_search_refuses_cpu_tensors():
    from rl4co_b200 import native
    from rl4co_b200.tensordict import TensorDict

    native.build()
    env, td, tours = _env_and_td()
    with pytest.raises(native.NativeLibraryError):
        env.local_search(td, tours)
    with pytest.raises(native.NativeLibraryError):
        env.local_search(TensorDict({"distances": torch.rand(3, 6, 6)}, batch_size=[3]), tours, num_threads=4)
    with pytest.raises(ValueError):
        native.tsp_two_opt(tours, 10)  # neither locs nor distances
    with pytest.raises(ValueError):
        native.tsp_two_opt(tours, 10, locs=td["locs"], distances=torch.rand(3, 6, 6))


def test_local_search_not_implemented_for_other_envs():
    from rl4co_b200.envs import get_env

    env = get_env("cvrp", generator_params=dict(num_loc=5))
    with pytest.raises(NotImplementedError):
        env.local_search(env.reset(batch_size=[2]), torch.zeros(2, 8, dtype=torch.int64))
