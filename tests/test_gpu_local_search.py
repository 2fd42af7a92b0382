"""GPU: FusedTSPEnv.local_search / co_tsp_two_opt, the reference's best-improvement 2-opt (tsp/local_search.py) as one
CUDA kernel.  Every ls_tsp fixture (recorded from the reference's numba implementation) is reproduced bit for bit on
both distance sources and on both sides of the shared-memory residency bound; the remaining tests check the invariants
of a 2-opt result, strided inputs, a 65 536-instance grid, out-of-range ids, aliasing in the C ABI, and -- where the
staged reference and numba are present -- fresh instances against the live reference."""

import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

_LS = np.load(os.path.join(GOLDEN_DIR, "ls_tsp.npz"))
CASES = sorted({k.split("::")[0] for k in _LS.files})


def _td(**data):
    from rl4co_b200.tensordict import TensorDict

    b = next(iter(data.values())).shape[0]
    return TensorDict(data, batch_size=[b])


def _tsp_env():
    from rl4co_b200.envs import get_env

    return get_env("tsp", generator_params=dict(num_loc=20))


def _lengths64(d, tours):
    """Cyclic tour length under matrix d [B, N, N] in float64."""
    rows = torch.arange(tours.shape[0])[:, None]
    return d.double()[rows, tours, tours.roll(-1, dims=1)].sum(1)


def _dist64(locs):
    return (locs.double()[:, :, None] - locs.double()[:, None]).norm(dim=-1)


@pytest.mark.parametrize("case", CASES)
def test_fixture_bit_identical(case):
    env = _tsp_env()
    key = "distances" if f"{case}::distances" in _LS.files else "locs"
    src = torch.from_numpy(_LS[f"{case}::{key}"]).to(DEV)
    tours_in = torch.from_numpy(_LS[f"{case}::tours_in"]).long().to(DEV)
    expect = torch.from_numpy(_LS[f"{case}::tours_out"]).long()
    keep = tours_in.clone()
    out = env.local_search(_td(**{key: src}), tours_in, max_iterations=int(_LS[f"{case}::max_iterations"]))
    assert out.dtype == torch.int64 and out.device == tours_in.device
    assert torch.equal(tours_in, keep), "input tours were modified"
    bad = (out.cpu() != expect).any(1).nonzero().flatten().tolist()
    assert not bad, f"{case}: instances {bad[:8]} differ from the reference"


@pytest.mark.parametrize("n,b", [(20, 256), (100, 64), (300, 4)])
@pytest.mark.parametrize("source", ["locs", "distances"])
def test_two_opt_invariants(n, b, source):
    """Position 0 stays, the result is a permutation, no tour gets longer, the input is untouched; the iteration count
    respects max_iterations."""
    from rl4co_b200 import native

    g = torch.Generator().manual_seed(n + b)
    locs = torch.rand(b, n, 2, generator=g)
    tours = torch.argsort(torch.rand(b, n, generator=g), dim=1)
    d = _dist64(locs)
    kw = dict(locs=locs.to(DEV)) if source == "locs" else dict(distances=d.float().to(DEV))
    t_dev = tours.to(DEV)
    its = torch.empty(b, dtype=torch.int32, device=DEV)
    out = native.tsp_two_opt(t_dev, 1000, iterations=its, **kw).cpu()
    assert torch.equal(t_dev.cpu(), tours)
    assert torch.equal(out[:, 0], tours[:, 0])
    assert torch.equal(out.sort(1).values, torch.arange(n).expand(b, n))
    before, after = _lengths64(d, tours), _lengths64(d, out)
    assert (after <= before + 1e-5).all() and (after < before).any()
    its = its.cpu()
    assert (its >= 1).all() and (its <= 1000).all()
    its3 = torch.empty(b, dtype=torch.int32, device=DEV)
    native.tsp_two_opt(t_dev, 3, iterations=its3, **kw)
    assert its3.max().item() <= 3


def test_noncontiguous_actions_and_dtype():
    env = _tsp_env()
    key = "rand50"
    locs = torch.from_numpy(_LS[f"{key}::locs"]).to(DEV)
    tours = torch.from_numpy(_LS[f"{key}::tours_in"]).long()
    strided = tours.t().contiguous().to(DEV).t()  # column-major view
    assert not strided.is_contiguous()
    out = env.local_search(_td(locs=locs), strided)
    assert torch.equal(out.cpu(), torch.from_numpy(_LS[f"{key}::tours_out"]).long())
    out32 = env.local_search(_td(locs=locs), tours.int().to(DEV))
    assert torch.equal(out32.cpu(), out.cpu())


def test_large_grid_b65536():
    """B = 65 536 at N = 20: every CTA reads and writes its own row (a sub-batch gives the same tours)."""
    from rl4co_b200 import native

    B, n = 65536, 20
    g = torch.Generator().manual_seed(3)
    locs = torch.rand(B, n, 2, generator=g).to(DEV)
    tours = torch.argsort(torch.rand(B, n, generator=g), dim=1).to(DEV)
    its = torch.empty(B, dtype=torch.int32, device=DEV)
    out = native.tsp_two_opt(tours, 1000, locs=locs, iterations=its)
    torch.cuda.synchronize()
    assert torch.equal(out.sort(1).values, torch.arange(n, device=DEV).expand(B, n))
    assert torch.equal(out[:, 0], tours[:, 0])
    assert (its >= 1).all()
    idx = torch.tensor([0, 1, 777, 32768, 65534, 65535], device=DEV)
    sub = native.tsp_two_opt(tours[idx].contiguous(), 1000, locs=locs[idx].contiguous())
    assert torch.equal(sub, out[idx])


def test_out_of_range_ids_pass_through():
    from rl4co_b200 import native

    n, b = 30, 6
    g = torch.Generator().manual_seed(5)
    locs = torch.rand(b, n, 2, generator=g).to(DEV)
    tours = torch.argsort(torch.rand(b, n, generator=g), dim=1).to(DEV)
    tours[1, 7] = n
    tours[3, 0] = -1
    tours[4, 29] = 1 << 40
    its = torch.empty(b, dtype=torch.int32, device=DEV)
    out = native.tsp_two_opt(tours, 1000, locs=locs, iterations=its)
    its = its.cpu()
    for r in (1, 3, 4):
        assert torch.equal(out[r], tours[r]) and its[r].item() == -1
    for r in (0, 2, 5):
        assert its[r].item() >= 1
        assert torch.equal(out[r].sort().values, torch.arange(n, device=DEV))


def test_abi_in_place_and_errors():
    """tours_out may alias tours_in; N above CO_TWO_OPT_MAX_NODES, or both / neither distance source, is refused."""
    from rl4co_b200 import native

    L = native.lib()
    key = "rand100"
    locs = torch.from_numpy(_LS[f"{key}::locs"]).to(DEV)
    tours = torch.from_numpy(_LS[f"{key}::tours_in"]).long().to(DEV)
    B, n = tours.shape
    stream = torch.cuda.current_stream().cuda_stream
    rc = L.co_tsp_two_opt(locs.data_ptr(), None, tours.data_ptr(), tours.data_ptr(), None, B, n, 1000, stream)
    assert rc == 0
    assert torch.equal(tours.cpu(), torch.from_numpy(_LS[f"{key}::tours_out"]).long())
    p = tours.data_ptr()
    assert L.co_tsp_two_opt(None, None, p, p, None, B, n, 10, stream) == -1
    assert L.co_tsp_two_opt(locs.data_ptr(), locs.data_ptr(), p, p, None, B, n, 10, stream) == -1
    assert L.co_tsp_two_opt(locs.data_ptr(), None, p, p, None, 1, 1025, 10, stream) == -2


def test_live_reference_fresh_instances():
    """B = 1024, N = 100, fresh seeds: the kernel against the reference's own local_search (staged under oracle/_ref)."""
    from oracle import ref_standin

    if not ref_standin.reference_available():
        pytest.skip("no reference tree (oracle/_ref not staged)")
    pytest.importorskip("numba")
    ref = ref_standin.load()
    g = torch.Generator().manual_seed(20261016)
    B, n = 1024, 100
    locs = torch.rand(B, n, 2, generator=g)
    starts = torch.argsort(torch.rand(B, n, generator=g), dim=1)
    expect = ref.TSPEnv.local_search(ref.TensorDict({"locs": locs}, batch_size=[B]), starts)
    env = _tsp_env()
    out = env.local_search(_td(locs=locs.to(DEV)), starts.to(DEV)).cpu()
    bad = (out != expect).any(1).sum().item()
    assert bad == 0, f"{bad} of {B} tours differ from the live reference"
