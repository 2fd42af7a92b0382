"""GPU: FusedCVRPEnv.local_search / co_cvrp_local_search.  The kernel's tours and move counts equal the NumPy
restatement (oracle/cvrp_local_search.py) bit for bit on both distance sources, on both sides of the shared-memory
residency bound, from random and policy tours; the reference's own cvrp/local_search.py wrapper (with the restatement
in place of its HGS call) returns what the method returns; rows do not depend on the batch; and the results are valid
tours that are never longer than their inputs."""

import importlib.util
import os
import shutil

import numpy as np
import pytest
import torch

from oracle import cvrp_local_search as ORC

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _instances(B, n, seed):
    """CPU reset state of B CVRP-n instances (locs with the depot, demand / capacity, vehicle_capacity)."""
    from rl4co_b200.envs import get_env

    env = get_env("cvrp", generator_params=dict(num_loc=n))
    torch.manual_seed(seed)
    return env, env.reset(env.generator(B))


def _random_tours(demand, seed):
    """Random permutations of the customers split greedily by capacity; some rows start with a 0, all are padded."""
    g = np.random.default_rng(seed)
    B, n = demand.shape
    rows = []
    for b in range(B):
        row, load = ([0] if b % 3 == 0 else []), 0.0
        for c in g.permutation(n) + 1:
            if load + float(demand[b, c - 1]) > 1.0:
                row.append(0)
                load = 0.0
            row.append(int(c))
            load += float(demand[b, c - 1])
        rows.append(row)
    T = max(map(len, rows)) + 2
    return torch.tensor([r + [0] * (T - len(r)) for r in rows], dtype=torch.int64)


def _dist(locs):
    """rl4co.utils.ops.get_distance_matrix on the CPU: the matrix the kernel computes from locs."""
    return (locs[..., :, None, :] - locs[..., None, :, :]).norm(p=2, dim=-1)


def _expected(tours, demand, d, max_iterations):
    B, n = demand.shape
    rows, used, its = [], [], []
    for b in range(B):
        dem = np.concatenate([[0], demand[b].numpy()]).astype(np.float32)
        slots, it = ORC.search(ORC.split_routes(tours[b].numpy()), dem, d[b].numpy(), max_iterations)
        row, u = ORC.merge_routes(slots, 2 * n)
        rows.append(row)
        used.append(u)
        its.append(it)
    return torch.from_numpy(np.stack(rows)), torch.tensor(used, dtype=torch.int32), torch.tensor(its, dtype=torch.int32)


def _run(td, tours, max_iterations, source, d=None):
    from rl4co_b200 import native

    B = tours.shape[0]
    its = torch.empty(B, dtype=torch.int32, device=DEV)
    kw = dict(locs=td["locs"].to(DEV)) if source == "locs" else dict(distances=d.to(DEV))
    out, used = native.cvrp_local_search(tours.to(DEV), td["demand"].to(DEV), td["vehicle_capacity"].reshape(B).to(DEV),
                                         max_iterations, iterations=its, **kw)
    return out.cpu(), used.cpu(), its.cpu()


def _check_against_restatement(td, tours, max_iterations, source, d=None):
    d = _dist(td["locs"]) if d is None else d
    out, used, its = _run(td, tours, max_iterations, source, d)
    exp, exp_used, exp_its = _expected(tours, td["demand"], d, max_iterations)
    bad = (out != exp).any(1).nonzero().flatten().tolist()
    assert not bad, f"rows {bad[:8]} differ from the restatement"
    assert torch.equal(used, exp_used) and torch.equal(its, exp_its)
    return its


@pytest.mark.parametrize("n,B", [(10, 16), (20, 16), (50, 8), (100, 4), (200, 2), (300, 1)])
@pytest.mark.parametrize("source", ["locs", "distances"])
def test_random_starts_bit_identical(n, B, source):
    _, td = _instances(B, n, seed=n)
    tours = _random_tours(td["demand"], seed=n)
    its = _check_against_restatement(td, tours, 1000, source)
    assert (its > 0).all()


@pytest.mark.parametrize("max_iterations", [0, 1, 5])
@pytest.mark.parametrize("source", ["locs", "distances"])
def test_max_iterations(max_iterations, source):
    _, td = _instances(8, 50, seed=7)
    its = _check_against_restatement(td, _random_tours(td["demand"], seed=7), max_iterations, source)
    assert (its == max_iterations).all()


def test_asymmetric_matrix():
    _, td = _instances(6, 50, seed=11)
    g = torch.Generator().manual_seed(11)
    d = torch.rand(6, 51, 51, generator=g)
    d[:, torch.arange(51), torch.arange(51)] = 0
    _check_against_restatement(td, _random_tours(td["demand"], seed=11), 1000, "distances", d)


@pytest.mark.parametrize("n", [20, 50])
@pytest.mark.parametrize("decode_type", ["greedy", "sampling"])
def test_policy_tours_bit_identical(n, decode_type):
    from rl4co_b200.policy import FusedAttentionModelPolicy

    env, td = _instances(8, n, seed=100 + n)
    torch.manual_seed(0)
    pol = FusedAttentionModelPolicy(env_name="cvrp", num_encoder_layers=1).to(DEV).eval()
    with torch.inference_mode():
        actions = pol(td.to(DEV), env, decode_type=decode_type, **({"seed": 3} if decode_type == "sampling" else {}))[
            "actions"].cpu()
    for source in ("locs", "distances"):
        _check_against_restatement(td, actions, 1000, source)


def _reference_local_search(tmp_path):
    from oracle import ref_standin

    if not ref_standin.reference_available():
        pytest.skip("no reference tree (oracle/_ref not staged)")
    ref_standin.install()
    # the module asserts at import that the HGS library file exists: import a copy next to an empty placeholder
    src = os.path.join(ref_standin.REFERENCE_ROOT, "rl4co", "envs", "routing", "cvrp", "local_search.py")
    shutil.copyfile(src, tmp_path / "local_search.py")
    os.makedirs(tmp_path / "HGS-CVRP" / "build")
    (tmp_path / "HGS-CVRP" / "build" / "libhgscvrp.so").touch()
    spec = importlib.util.spec_from_file_location("cvrp_local_search_reference", tmp_path / "local_search.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.swapstar = ORC.swapstar
    return mod


@pytest.mark.parametrize("max_iterations", [0, 1000])
def test_reference_wrapper(tmp_path, max_iterations):
    """The reference's own pre- and post-processing around the restatement: trimming, route order and the validity
    fallback (row 1 starts over capacity, so it keeps an infeasible route and gets its original, longer actions back)."""
    from rl4co_b200.policy import FusedAttentionModelPolicy
    from rl4co_b200.tensordict import TensorDict

    mod = _reference_local_search(tmp_path)
    env, td = _instances(12, 20, seed=5)
    torch.manual_seed(0)
    pol = FusedAttentionModelPolicy(env_name="cvrp", num_encoder_layers=1).to(DEV).eval()
    with torch.inference_mode():
        actions = pol(td.to(DEV), env, decode_type="sampling", seed=9)["actions"].cpu()
    over = torch.arange(1, 21)  # one route over every customer: above capacity
    actions = torch.nn.functional.pad(actions, (0, max(0, 30 - actions.shape[1])))
    actions[1] = 0
    actions[1, 5:25] = over
    td_cpu = TensorDict({k: td[k] for k in ("locs", "demand", "vehicle_capacity")}, batch_size=[12])
    expect = mod.local_search(td_cpu, actions, max_iterations=max_iterations)
    out = env.local_search(td_cpu.to(DEV), actions.to(DEV), max_iterations=max_iterations, allow_infeasible=False)
    assert out.dtype == torch.int64 and out.device.type == "cuda"
    assert out.shape == expect.shape and torch.equal(out.cpu(), expect)
    assert torch.equal(out[1, :25].cpu(), actions[1, :25])


def test_row_independence_and_scale():
    """N = 20: row b's result is the same in batches of 1, 37, 4 096 and 65 536 rows of different composition."""
    from rl4co_b200 import native

    B = 65536
    _, td = _instances(B, 20, seed=21)
    tours = _random_tours(td["demand"][:4096], seed=21)
    tours = tours.repeat(16, 1)  # rows b and b + 4096 k share tours but not instances
    locs, dem, cap = td["locs"].to(DEV), td["demand"].to(DEV), td["vehicle_capacity"].reshape(B).to(DEV)
    t = tours.to(DEV)
    full, used = native.cvrp_local_search(t, dem, cap, 1000, locs=locs)
    for idx in (torch.tensor([65535]), torch.arange(4096, 4096 + 37).flip(0), torch.randperm(B)[:4096]):
        i = idx.to(DEV)
        sub, sub_used = native.cvrp_local_search(t[i].contiguous(), dem[i].contiguous(), cap[i].contiguous(), 1000,
                                                 locs=locs[i].contiguous())
        assert torch.equal(sub, full[i]) and torch.equal(sub_used, used[i])
    rows = torch.tensor([0, 4097, 65535])
    exp, exp_used, _ = _expected(tours[rows], td["demand"][rows], _dist(td["locs"][rows]), 1000)
    assert torch.equal(full[rows.to(DEV)].cpu(), exp) and torch.equal(used[rows.to(DEV)].cpu(), exp_used)


def test_reward_validity_iterations_cvrp100():
    from rl4co_b200 import native
    from rl4co_b200.policy import FusedAttentionModelPolicy

    env, td = _instances(512, 100, seed=4)
    td = td.to(DEV)
    torch.manual_seed(0)
    pol = FusedAttentionModelPolicy(env_name="cvrp", num_encoder_layers=1).to(DEV).eval()
    with torch.inference_mode():
        actions = pol(td, env, decode_type="sampling", seed=1)["actions"]
    out = env.local_search(td, actions)
    env.check_solution_validity(td, out)
    before, after = env.get_reward(td, actions), env.get_reward(td, out)
    assert (after >= before).all() and (after > before).any()
    its = torch.empty(512, dtype=torch.int32, device=DEV)
    native.cvrp_local_search(actions.contiguous(), td["demand"], td["vehicle_capacity"].reshape(512), 1000,
                             locs=td["locs"], iterations=its)
    assert (its >= 0).all()


def test_noncontiguous_and_int32_actions():
    env, td = _instances(8, 20, seed=8)
    tours = _random_tours(td["demand"], seed=8)
    tdd = td.to(DEV)
    ref = env.local_search(tdd, tours.to(DEV))
    strided = tours.t().contiguous().to(DEV).t()
    assert not strided.is_contiguous()
    assert torch.equal(env.local_search(tdd, strided), ref)
    assert torch.equal(env.local_search(tdd, tours.int().to(DEV)), ref)


def test_invalid_rows():
    """Out-of-range and duplicate ids: -1 moves and the row copied through at the ABI; AssertionError at the method."""
    from rl4co_b200 import native

    env, td = _instances(5, 20, seed=9)
    tours = _random_tours(td["demand"], seed=9)
    tours[1, 3] = 21
    tours[2, 0] = -1
    first = int(tours[3][tours[3] != 0][0])
    tours[3][(tours[3] != 0).nonzero()[1]] = first  # duplicate, and one customer missing
    its = torch.empty(5, dtype=torch.int32, device=DEV)
    out, used = native.cvrp_local_search(tours.to(DEV), td["demand"].to(DEV), td["vehicle_capacity"].reshape(5).to(DEV),
                                         1000, locs=td["locs"].to(DEV), iterations=its)
    out, used, its = out.cpu(), used.cpu(), its.cpu()
    T = tours.shape[1]
    for r in (1, 2, 3):
        assert its[r] == -1 and used[r] == T and torch.equal(out[r, :T], tours[r]) and (out[r, T:] == 0).all()
    assert its[0] >= 0 and its[4] >= 0
    with pytest.raises(AssertionError, match="Invalid tour"):
        env.local_search(td.to(DEV), tours.to(DEV))


def test_abi_errors():
    from rl4co_b200 import native

    L = native.lib()
    B, n, T = 2, 10, 20
    locs = torch.rand(B, n + 1, 2, device=DEV)
    dem = torch.full((B, n), 0.1, device=DEV)
    cap = torch.ones(B, device=DEV)
    tours = torch.zeros(B, T, dtype=torch.int64, device=DEV)
    out = torch.zeros(B, 2 * n, dtype=torch.int64, device=DEV)
    used = torch.zeros(B, dtype=torch.int32, device=DEV)
    s = torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()  # noqa: E731
    args = [p(locs), None, p(dem), p(cap), p(tours), p(out), p(used), None, None, B, n, T, 10, s]

    def call(**kw):
        a = list(args)
        for i, v in kw.items():
            a[int(i[1:])] = v
        return L.co_cvrp_local_search(*a)

    assert call(a0=None) == -1  # neither distance source
    assert call(a1=p(locs)) == -1  # both
    for i in (2, 3, 4, 5, 6):
        assert call(**{f"a{i}": None}) == -1
    assert call(a0=p(locs) + 4) == -1 and call(a2=p(dem) + 2) == -1 and call(a4=p(tours) + 4) == -1
    assert call(a5=p(out) + 4) == -1 and call(a6=p(used) + 2) == -1
    assert call(a9=-1) == -1 and call(a10=0) == -1 and call(a11=0) == -1
    assert call(a10=1024) == -2  # N + 1 above CO_TWO_OPT_MAX_NODES
    assert call(a9=0) == 0
