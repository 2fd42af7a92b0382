"""CPU tests of the CVRP local search: the NumPy restatement (oracle/cvrp_local_search.py) on hand-checkable instances,
one per move kind, with a brute-force optimum as the known answer; the tie order of the key; a slot emptied and refilled;
properties on random instances; and the argument checks of the binding and of FusedCVRPEnv.local_search."""

import itertools

import numpy as np
import pytest
import torch

from oracle import cvrp_local_search as ORC


def _dmat(xy):
    xy = torch.tensor(xy, dtype=torch.float32)
    return (xy[:, None] - xy[None]).norm(p=2, dim=-1).numpy()


def _cost(slots, d):
    return sum(float(d[0, s[0]]) + sum(float(d[a, b]) for a, b in zip(s, s[1:])) + float(d[s[-1], 0])
               for s in slots if s)


def _brute_force(dem, d, routes):
    """Least cost over every order of the customers cut into at most `routes` routes within capacity."""
    N, best = len(dem) - 1, np.inf
    for perm in itertools.permutations(range(1, N + 1)):
        for cuts in itertools.product([0, 1], repeat=N - 1):
            slots, cur = [], [perm[0]]
            for c, x in zip(cuts, perm[1:]):
                if c:
                    slots.append(cur)
                    cur = []
                cur.append(x)
            slots.append(cur)
            if len(slots) <= routes and all(sum(float(dem[x]) for x in s) <= 1 + 1e-5 for s in slots):
                best = min(best, _cost(slots, d))
    return best


def _log(slots, dem, d, count=1000):
    slots, moves = [list(s) for s in slots], []
    while len(moves) < count:
        mv = ORC.best_move(slots, dem, d)
        if mv is None:
            break
        ORC.apply_move(slots, d.shape[0] - 1, *mv[1:])
        moves.append(mv)
    return slots, moves


# (depot + customer coordinates, demands with the depot's 0, start routes, result); each improves through one move
# of its kind and ends at the brute-force optimum
KIND_CASES = {
    ORC.RELOCATE: ([[4, 2], [0, 3], [3, 4], [0, 0], [4, 0]], [0, .5, .25, .25, .25], [[3, 2, 1], [4]],
                   [[3, 1, 2], [4]]),
    ORC.SWAP: ([[4, 0], [2, 3], [1, 1], [1, 1], [4, 1], [1, 0]], [0, .25, .5, .25, .5, .5], [[1, 3, 4], [5, 2]],
               [[1, 3, 2], [5, 4]]),
    ORC.TWO_OPT: ([[0, 0], [2, 1], [0, 4], [3, 1], [1, 0], [1, 2]], [0, .5, .5, .25, .25, .5], [[4, 1, 3], [5, 2]],
                  [[4, 3, 1], [5, 2]]),
    ORC.TWO_OPT_STAR: ([[0, 3], [4, 0], [3, 1], [4, 4], [2, 2], [3, 2]], [0, .5, .25, .5, .5, .5],
                       [[1, 5], [3, 2], [4]], [[1, 2], [3, 5], [4]]),
}


@pytest.mark.parametrize("kind", sorted(KIND_CASES))
def test_restatement_single_kind(kind):
    xy, dem, start, result = KIND_CASES[kind]
    d, dem = _dmat(xy), np.float32(dem)
    out, moves = _log(start, dem, d)
    assert out == result and [m[1] for m in moves] == [kind]
    assert _cost(out, d) == pytest.approx(_brute_force(dem, d, len(start)), abs=1e-5)
    assert _cost(out, d) < _cost(start, d)
    assert [list(r[1:-1]) for r in ORC.swapstar(dem, d, None, [np.array([0, *s, 0]) for s in start], 1000)] == result


def test_restatement_tie_order():
    """Customers 1 and 2 mirror each other about the depot's axis, so relocating either next to 3 changes the length by
    the same float: the key takes the smaller id."""
    xy = [[0, 0], [-1, 2], [1, 2], [0, 4]]
    d, dem = _dmat(xy), np.float32([0, .25, .25, .25])
    start = [[1], [2], [3]]
    mv = ORC.best_move(start, dem, d)
    deltas = {}
    for u in (1, 2):
        slots = [list(s) for s in start]
        ORC.apply_move(slots, 3, ORC.RELOCATE, u, 3)
        deltas[u] = _cost(slots, d) - _cost(start, d)
    assert deltas[1] == deltas[2] and d[0, 1] == d[0, 2] and d[1, 3] == d[2, 3]
    # every candidate with the smallest delta shares it; the smallest (kind, u, v) wins
    assert mv[1:] == (ORC.RELOCATE, 1, 3)


def test_restatement_empties_and_refills_a_slot():
    d = np.float32([[0, 5, 1, 8, 1], [7, 0, 7, 6, 1], [1, 8, 0, 6, 6], [6, 7, 9, 0, 7], [5, 4, 2, 9, 0]])
    dem = np.float32([0, .25, .25, .25, .25])
    slots, moves = [[1], [2, 3], [4]], []
    emptied, refilled = set(), False
    while True:
        mv = ORC.best_move(slots, dem, d)
        if mv is None:
            break
        ORC.apply_move(slots, 4, *mv[1:])
        moves.append(mv[1])
        refilled |= any(slots[r] for r in emptied)
        emptied |= {r for r, c in enumerate(slots) if not c}
    assert refilled
    assert slots == [[2], [4, 1, 3], []] and moves == [0, 3, 2, 0]
    routes = ORC.swapstar(dem, d, None, [np.array([0, 1, 0]), np.array([0, 2, 3, 0]), np.array([0, 4, 0])], 1000)
    assert [list(r) for r in routes] == [[0, 2, 0], [0, 4, 1, 3, 0], [0, 0]]


@pytest.mark.parametrize("seed", range(6))
def test_restatement_properties(seed):
    g = np.random.default_rng(seed)
    N = int(g.integers(5, 40))
    xy = g.random((N + 1, 2)).astype(np.float32)
    d = _dmat(xy)
    dem = np.concatenate([[0], g.integers(1, 10, N) / 20.0]).astype(np.float32)
    row, load = [], 0.0
    for c in g.permutation(N) + 1:
        if load + dem[c] > 1:
            row.append(0)
            load = 0.0
        row.append(int(c))
        load += float(dem[c])
    start = ORC.split_routes(np.array(row))
    out, it = ORC.search(start, dem, d, 1000)
    d64 = np.sqrt(((xy[:, None].astype(np.float64) - xy[None]) ** 2).sum(-1))
    assert _cost(out, d64) <= _cost(start, d64) + 1e-9
    assert len(out) == len(start) and sorted(sum(out, [])) == list(range(1, N + 1))
    for s in out:
        acc = np.float32(0)
        for x in s:
            acc = np.float32(acc + dem[x])
        assert acc <= np.float32(1 + 1e-5)
    assert ORC.search(out, dem, d, 1000)[1] == 0  # a local optimum


def test_split_and_merge_layout():
    assert ORC.split_routes(np.array([0, 3, 1, 0, 0, 2, 0])) == [[3, 1], [2]]
    assert ORC.split_routes(np.array([3, 0, 2, 1])) == [[3], [2, 1]]
    row, used = ORC.merge_routes([[3, 1], [], [2]], 6)
    assert row.tolist() == [3, 1, 0, 2, 0, 0] and used == 4


def test_binding_exported_and_argument_checks():
    from rl4co_b200 import native

    native.build()
    assert "co_cvrp_local_search" in native.EXPORTS
    assert hasattr(native.lib(), "co_cvrp_local_search")
    tours = torch.zeros(2, 8, dtype=torch.int64)
    dem, cap, locs = torch.rand(2, 5), torch.ones(2), torch.rand(2, 6, 2)
    with pytest.raises(ValueError):
        native.cvrp_local_search(tours, dem, cap, 10)  # neither locs nor distances
    with pytest.raises(ValueError):
        native.cvrp_local_search(tours, dem, cap, 10, locs=locs, distances=torch.rand(2, 6, 6))
    with pytest.raises(ValueError):
        native.cvrp_local_search(tours, dem, cap, 10, locs=torch.rand(2, 5, 2))
    with pytest.raises(ValueError):
        native.cvrp_local_search(tours, dem, torch.ones(3), 10, locs=locs)
    with pytest.raises(native.NativeLibraryError):
        native.cvrp_local_search(tours, dem, cap, 10, locs=locs)  # CPU tensors


def test_method_refuses_cpu_first_and_sdvrp():
    from rl4co_b200.envs import get_env
    from rl4co_b200.tensordict import TensorDict

    env = get_env("cvrp", generator_params=dict(num_loc=5))
    td = env.reset(batch_size=[2])
    with pytest.raises(NotImplementedError, match="CUDA"):
        env.local_search(td, torch.zeros(2, 8, dtype=torch.int64))
    bad = TensorDict({"locs": torch.rand(2, 3, 6, 2)}, batch_size=[2, 3])  # checked after the device
    with pytest.raises(NotImplementedError, match="CUDA"):
        env.local_search(bad, torch.zeros(2, 3, 8, dtype=torch.int64))
    sd = get_env("sdvrp", generator_params=dict(num_loc=5))
    with pytest.raises(NotImplementedError):
        sd.local_search(sd.reset(batch_size=[2]), torch.zeros(2, 8, dtype=torch.int64))
