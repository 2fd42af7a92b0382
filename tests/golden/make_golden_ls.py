"""Generate tests/golden/ls_tsp.npz: the tours rl4co's OWN, unmodified TSP local search
(``TSPEnv.local_search`` -> rl4co/envs/routing/tsp/local_search.py, the numba 2-opt) returns, run
through oracle/ref_standin.py like tests/golden/make_golden.py runs the rest of the reference.

Run in the build container only (needs the reference tree and numba):

    python tests/golden/make_golden_ls.py            # every fixture of this script
    python tests/golden/make_golden_ls.py ls_tsp     # just the named ones

The cases cover random-permutation starts for N from 2 to 1000, the reference's own AM greedy tours
(am_tsp{20,50,100}.npz) as starts, integer lattices (many equal changes: the tie-break decides), the
explicit-matrix path on Euclidean and on asymmetric non-Euclidean matrices, tours that repeat a node,
and max_iterations in {0, 1, 3, 1000}.  Every tour written here is computed by reference code.
"""

from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_standin  # noqa: E402

ref = ref_standin.load()
TensorDict = ref.TensorDict

#: random-permutation starts: N -> batch
LS_RANDOM = {2: 8, 3: 8, 5: 16, 20: 64, 50: 32, 100: 16, 200: 4, 300: 2, 1000: 1}


def npy(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def ls_tsp_cases():
    """(case, inputs): inputs are the arguments of TSPEnv.local_search -- "locs" [B, N, 2] or "distances"
    [B, N, N], the start tours "tours_in" [B, N] and "max_iterations"."""
    cases = []

    def perms(b, n):
        return torch.argsort(torch.rand(b, n), dim=1)

    for n, b in LS_RANDOM.items():
        torch.manual_seed(500 + n)
        locs = torch.rand(b, n, 2)
        cases.append((f"rand{n}", dict(locs=locs, tours_in=perms(b, n), max_iterations=1000)))
    # the explicit-matrix path on a Euclidean matrix: get_distance_matrix, as the reference builds it from locs
    r20 = cases[3][1]
    cases.append(("euc20", dict(distances=ref.ops.get_distance_matrix(r20["locs"]), tours_in=r20["tours_in"],
                                max_iterations=1000)))
    r100 = cases[5][1]
    for mi in (0, 1, 3):
        cases.append((f"rand100_it{mi}", dict(locs=r100["locs"], tours_in=r100["tours_in"], max_iterations=mi)))
    # the reference's own AM greedy tours (am_tsp*.npz) as starts
    for n in (20, 50, 100):
        z = np.load(os.path.join(HERE, f"am_tsp{n}.npz"))
        cases.append((f"am{n}", dict(locs=torch.from_numpy(z["inst::locs"]), tours_in=torch.from_numpy(z["greedy_actions"]),
                                     max_iterations=1000)))
    # integer lattices: many equal changes, so the first-in-loop-order tie-break decides
    for n, b, g in ((50, 16, 8), (300, 2, 18)):
        torch.manual_seed(600 + n)
        pts = torch.stack([torch.randperm(g * g)[:n] for _ in range(b)])
        locs = torch.stack([pts % g, pts // g], dim=-1).float()
        cases.append((f"lattice{n}", dict(locs=locs, tours_in=perms(b, n), max_iterations=1000)))
    cases.append(("lattice50_dist", dict(distances=ref.ops.get_distance_matrix(cases[-2][1]["locs"]),
                                         tours_in=cases[-2][1]["tours_in"], max_iterations=1000)))
    # asymmetric non-Euclidean matrices (DeepACO's neural local search passes such a heuristic distance): quantised
    # values (ties) below the shared-memory bound, continuous ones above it
    torch.manual_seed(700)
    asym50 = torch.randint(1, 9, (8, 50, 50)).float() / 4
    cases.append(("asym50", dict(distances=asym50, tours_in=perms(8, 50), max_iterations=1000)))
    cases.append(("asym50_it3", dict(distances=asym50, tours_in=cases[-1][1]["tours_in"], max_iterations=3)))
    cases.append(("asym300", dict(distances=torch.rand(1, 300, 300), tours_in=perms(1, 300), max_iterations=1000)))
    # tours that repeat a node: the node-equality skips and the +1e9 diagonal become reachable
    torch.manual_seed(800)
    dup = torch.randint(0, 20, (8, 20))
    cases.append(("dup20", dict(locs=torch.rand(8, 20, 2), tours_in=dup, max_iterations=1000)))
    return cases


def ls_tsp_fixture():
    """TSPEnv.local_search on every case of ls_tsp_cases; arrays keyed "<case>::<name>"."""
    out = {}
    for case, inp in ls_tsp_cases():
        key = "distances" if "distances" in inp else "locs"
        td = TensorDict({key: inp[key]}, batch_size=[inp["tours_in"].shape[0]])
        res = ref.TSPEnv.local_search(td, inp["tours_in"].clone(), max_iterations=inp["max_iterations"])
        out[f"{case}::{key}"] = npy(inp[key])
        out[f"{case}::tours_in"] = npy(inp["tours_in"]).astype(np.int16)
        out[f"{case}::max_iterations"] = np.int64(inp["max_iterations"])
        out[f"{case}::tours_out"] = npy(res).astype(np.int16)
    return out


def main():
    jobs = {"ls_tsp": ls_tsp_fixture}
    only = set(sys.argv[1:])
    for name, fn in jobs.items():
        if only and name not in only:
            continue
        data = fn()
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **data)
        print(f"{name}: {len(data)} arrays, {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
