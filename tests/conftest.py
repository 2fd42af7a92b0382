import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")

# the CPU oracle works on [B, N, 128]-sized tensors: torch's default of one thread per core is far slower than 16
# threads on a many-core host
torch.set_num_threads(min(16, os.cpu_count() or 1))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


class Golden:
    """npz fixture produced by tests/golden/make_golden.py from the live reference."""

    def __init__(self, name):
        self.name = name
        self.z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))

    def __getitem__(self, k):
        return torch.from_numpy(self.z[k])

    def __contains__(self, k):
        return k in self.z.files

    def weights(self, device="cpu"):
        return {k[3:]: torch.from_numpy(self.z[k]).to(device) for k in self.z.files if k.startswith("w::")}

    def inst(self, device="cpu"):
        return {k[6:]: torch.from_numpy(self.z[k]).to(device) for k in self.z.files if k.startswith("inst::")}


@pytest.fixture(scope="session")
def golden():
    cache = {}

    def _get(name):
        if name not in cache:
            cache[name] = Golden(name)
        return cache[name]

    return _get


def env_of(name):
    for env in ("pctsp", "sdvrp", "cvrp"):
        if env in name:
            return env
    if "_op" in name:
        return "op"
    return "tsp" if "tsp" in name else "cvrp"


def name_seeded_weights(state_dict, seed):
    """Mirror of tests/golden/make_golden.py::name_seeded_weights: weights that depend only on
    (parameter name, shape, seed), so a fixture need not store them."""
    import zlib

    new = {}
    for k in sorted(state_dict.keys()):
        v = state_dict[k]
        if not v.dtype.is_floating_point:
            new[k] = v.clone()
            continue
        gen = torch.Generator().manual_seed(seed * 1_000_003 + zlib.crc32(k.encode()))
        u = torch.rand(v.shape, generator=gen) * 2 - 1
        if v.dim() >= 2:
            new[k] = u / (v.shape[-1] ** 0.5)
        elif "W_placeholder" in k:
            new[k] = u
        elif "norm" in k and k.endswith("weight"):
            new[k] = 1 + 0.1 * u
        elif k.endswith("running_var"):
            new[k] = 1 + 0.25 * u
        else:
            new[k] = 0.1 * u
    return new
