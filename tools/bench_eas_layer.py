"""Efficient active search with a per-instance layer (EAS-Lay) next to EAS-Emb on the H100, on the same inputs.

For TSP-100 and CVRP-100 (B instances x A augmentations x N starts), with CUDA events over `--split-iters` iterations
(after one warm-up iteration) of the loop body of `eas_search`:
  * EAS-Lay: the sampling rollout through the layer (`co_rollout` with `eas_layer`), `co_eas_layer_grad`, the Adam step;
  * EAS-Emb: the sampling rollout, `co_eas_key_grad`, the Adam step plus the refold Lf = L W_out;
then the mean `max_reward` after `--iters` iterations of `eas_search` for both variants.  The policy is randomly
initialised (seeded): no trained checkpoint ships with the project.  The card name and power limit are read in the
same run.  Prints one JSON line per environment, and writes the list of them to `--out` when given.
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tools.bench_eas import gpu_info  # noqa: E402

E = 128


def split(env_name, pol, td, A, iters, variant):
    """Mean ms per iteration of (rollout, gradient, optimizer step) for one variant."""
    from rl4co_b200 import native
    from rl4co_b200.eas import eas_coefficients, eas_layer_init
    from rl4co_b200.ops import StateAugmentation

    B, N = td["action_mask"].shape
    S = N - (1 if env_name == "cvrp" else 0)  # get_num_starts: every customer
    T = N if env_name == "tsp" else 2 * (N - 1)
    vrp = env_name == "cvrp"
    dec = pol.decoder
    tda = StateAugmentation(num_augment=A, augment_fn="dihedral8")(td)
    with torch.no_grad():
        hidden, _ = pol.encoder(tda)
        cached = dec._precompute_cache(hidden)
        cache = cached.rollout_cache.contiguous().clone()
        w_out = dec.pointer.project_out.weight.detach().clone()
        L = torch.nn.Parameter(torch.matmul(hidden, dec.project_node_embeddings.weight[2 * E:3 * E].t()).contiguous())
    layer = torch.nn.Parameter(eas_layer_init(A * B, td.device))
    opt = torch.optim.Adam([layer if variant == "lay" else L], lr=0.0041, weight_decay=1e-6)
    demand = tda["demand"].contiguous() if vrp else None
    vcap = tda["vehicle_capacity"].reshape(-1).contiguous() if vrp else None
    kw = dict(graph_ctx=cached.graph_context_or_none, w_capacity=cached.w_capacity, demand=demand, vehicle_capacity=vcap)
    best = None
    t = [0.0, 0.0, 0.0]
    for it in range(iters + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        with torch.no_grad():
            ev[0].record()
            res = native.rollout(env_name, native.SELECT_SAMPLE_PHILOX, cache, cached.graph_context_or_none,
                                 cached.q_placeholder, cached.w_capacity, tda["locs"].contiguous(), demand, vcap,
                                 A * B, N, num_starts=S, forced_start=True, num_loc=S, T_max=T, seed=1, offset=it,
                                 layer=layer.detach() if variant == "lay" else None)
            ev[1].record()
            rows = res["actions"] if best is None else torch.cat([res["actions"], best])
            coef = eas_coefficients(res["reward"].view(S, A, B), "multistart", 0.013, best is not None)
            if variant == "lay":
                layer.grad, _ = native.eas_layer_grad(env_name, cache, rows, coef, layer.detach(), **kw)
            else:
                dLf, _ = native.eas_key_grad(env_name, cache, rows, coef, **kw)
                L.grad = torch.matmul(dLf, w_out.t())
            ev[2].record()
        opt.step()
        if variant == "emb":
            with torch.no_grad():
                cache[..., 2 * E:3 * E] = torch.matmul(L.detach(), w_out)
        ev[3].record()
        best = res["actions"][:A * B]
        torch.cuda.synchronize()
        if it > 0:
            for i in range(3):
                t[i] += ev[i].elapsed_time(ev[i + 1]) / iters
    return {"rollout": round(t[0], 2), "gradient": round(t[1], 2), "optimizer_step": round(t[2], 2)}


def run(env_name, N, B, A, iters, split_iters):
    from rl4co_b200.eas import eas_search
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    env = get_env(env_name, generator_params=dict(num_loc=N if env_name == "tsp" else N - 1), check_solution=False)
    pol = FusedAttentionModelPolicy(env_name=env_name).to(dev).eval()
    td = env.reset(env.generator(B).to(dev))
    out = {"env": f"{env_name}{N}", "B": B, "augment": A, "starts": env.get_num_starts(td), "ms_per_iter": {}}
    for variant in ("lay", "emb"):
        out["ms_per_iter"][variant] = split(env_name, pol, td, A, split_iters, variant)
        print(f"{env_name}{N} EAS-{variant}: {out['ms_per_iter'][variant]} ms per iteration", file=sys.stderr, flush=True)
    out["mean_max_reward"] = {}
    for variant in ("lay", "emb"):
        torch.manual_seed(1)
        torch.cuda.synchronize()
        t0 = time.time()
        res = eas_search(pol, env, td, max_iters=iters, augment_size=A, seed=1, use_eas_layer=variant == "lay",
                         use_eas_embedding=variant == "emb")
        torch.cuda.synchronize()
        hist = res["reward_history"]
        out["mean_max_reward"][variant] = {"after_1": float(hist[0].mean()), f"after_{iters}": float(hist[-1].mean()),
                                           "search_wall_s": round(time.time() - t0, 1)}
    out["policy"] = "randomly initialised (seed 0)"
    out["gpu"] = gpu_info()
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--envs", default="tsp,cvrp")
    p.add_argument("--N", type=int, default=100)
    p.add_argument("--B", type=int, default=1024)
    p.add_argument("--augment", type=int, default=8)
    p.add_argument("--iters", type=int, default=10)
    p.add_argument("--split-iters", type=int, default=2)
    p.add_argument("--out", default=None, help="JSON file for the results")
    a = p.parse_args()
    from rl4co_b200 import native

    native.build()
    lines = []
    for env_name in a.envs.split(","):
        line = run(env_name, a.N, a.B, a.augment, a.iters, a.split_iters)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
