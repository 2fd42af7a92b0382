"""Efficient active search (EAS-Emb) on the H100: per-iteration time split, the key-gradient kernel against the autograd
path, and the search's progress.

For TSP-100 and CVRP-100 (B instances x A augmentations x N starts):
  * one iteration of `eas_search` split into the sampling rollout (`co_rollout`), `co_eas_key_grad`, and the Adam step
    plus the refold Lf = L W_out, with CUDA events over `--split-iters` iterations (after one warm-up iteration);
  * the gradient of the sampled rows against `evaluate_log_likelihood` under autograd with L as a leaf, on the largest
    chunk of instances (of those tried) that fits in memory: time per instance and relative difference;
  * mean `max_reward` after 0 (the first iteration), 50 and `--iters` iterations of `eas_search`.
The policy is randomly initialised (seeded): no trained checkpoint ships with the project.
Prints one JSON line per environment, and writes the list of them to `--out` when given.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

E = 128


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return out
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def run(env_name, N, B, A, iters, split_iters, chunks):
    from rl4co_b200 import native
    from rl4co_b200.eas import eas_coefficients, eas_search
    from rl4co_b200.envs import get_env
    from rl4co_b200.ops import StateAugmentation
    from rl4co_b200.policy import FusedAttentionModelPolicy
    from rl4co_b200.reinforce import evaluate_log_likelihood

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    env = get_env(env_name, generator_params=dict(num_loc=N if env_name == "tsp" else N - 1), check_solution=False)
    pol = FusedAttentionModelPolicy(env_name=env_name).to(dev).eval()
    td = env.reset(env.generator(B).to(dev))
    S = env.get_num_starts(td)
    T = N if env_name == "tsp" else 2 * (N - 1)
    vrp = env_name == "cvrp"
    dec = pol.decoder

    # ---- time split: the loop body of eas_search, instrumented
    tda = StateAugmentation(num_augment=A, augment_fn="dihedral8")(td)
    with torch.no_grad():
        hidden, _ = pol.encoder(tda)
        cached = dec._precompute_cache(hidden)
        cache = cached.rollout_cache.contiguous().clone()
        w_out = dec.pointer.project_out.weight.detach().clone()
        L = torch.nn.Parameter(torch.matmul(hidden, dec.project_node_embeddings.weight[2 * E:3 * E].t()).contiguous())
    opt = torch.optim.Adam([L], lr=0.0041, weight_decay=1e-6)
    demand = tda["demand"].contiguous() if vrp else None
    vcap = tda["vehicle_capacity"].reshape(-1).contiguous() if vrp else None
    best = None
    t_roll = t_grad = t_adam = 0.0
    for it in range(split_iters + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        with torch.no_grad():
            ev[0].record()
            res = native.rollout(env_name, native.SELECT_SAMPLE_PHILOX, cache, cached.graph_context_or_none,
                                 cached.q_placeholder, cached.w_capacity, tda["locs"].contiguous(), demand, vcap,
                                 A * B, N, num_starts=S, forced_start=True, num_loc=S, T_max=T, seed=1, offset=it)
            ev[1].record()
            rows = res["actions"] if best is None else torch.cat([res["actions"], best])
            coef = eas_coefficients(res["reward"].view(S, A, B), "multistart", 0.013, best is not None)
            dLf, _ = native.eas_key_grad(env_name, cache, rows, coef, graph_ctx=cached.graph_context_or_none,
                                         w_capacity=cached.w_capacity, demand=demand, vehicle_capacity=vcap)
            ev[2].record()
            L.grad = torch.matmul(dLf, w_out.t())
        opt.step()
        with torch.no_grad():
            cache[..., 2 * E:3 * E] = torch.matmul(L.detach(), w_out)
        ev[3].record()
        best = res["actions"][:A * B]
        torch.cuda.synchronize()
        if it > 0:
            t_roll += ev[0].elapsed_time(ev[1]) / split_iters
            t_grad += ev[1].elapsed_time(ev[2]) / split_iters
            t_adam += ev[2].elapsed_time(ev[3]) / split_iters

    print(f"{env_name}{N}: rollout {t_roll:.2f} ms, eas_key_grad {t_grad:.2f} ms, adam+refold {t_adam:.2f} ms per iteration",
          file=sys.stderr, flush=True)

    # ---- kernel vs autograd on the sampled rows of the first C instances (iteration-0 rows, no incumbent)
    with torch.no_grad():
        cache0 = cached.rollout_cache.contiguous().clone()
        L0 = torch.matmul(hidden, dec.project_node_embeddings.weight[2 * E:3 * E].t()).contiguous()
        cache0[..., 2 * E:3 * E] = torch.matmul(L0, w_out)
        res = native.rollout(env_name, native.SELECT_SAMPLE_PHILOX, cache0, cached.graph_context_or_none,
                             cached.q_placeholder, cached.w_capacity, tda["locs"].contiguous(), demand, vcap, A * B, N,
                             num_starts=S, forced_start=True, num_loc=S, T_max=T, seed=1, offset=0)
        coef = eas_coefficients(res["reward"].view(S, A, B), "multistart", 0.013, False)
    acts = res["actions"].view(S, A * B, T)
    coef = coef.view(S, A * B)
    cmp = None
    from rl4co_b200.tensordict import TensorDict

    keys = ("locs", "demand", "vehicle_capacity", "action_mask")
    for C in chunks:
        if C > A * B:
            break
        try:
            torch.cuda.empty_cache()
            sub = TensorDict({k: tda[k][:C] for k in keys if k in tda.keys()}, batch_size=[C])
            rows_c = acts[:, :C].reshape(S * C, T).contiguous()
            coef_c = coef[:, :C].reshape(-1).contiguous()
            leaf = L0[:C].clone().requires_grad_(True)
            orig = dec._precompute_cache

            def patched(h, *a, **k):
                c = orig(h, *a, **k)
                c._logit_key = leaf
                return c

            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            dec._precompute_cache = patched
            try:
                torch.cuda.reset_peak_memory_stats()
                ev[0].record()
                ll = evaluate_log_likelihood(pol, sub, env, rows_c, hidden=hidden[:C])
                (coef_c * ll).sum().backward()
                ev[1].record()
            finally:
                dec._precompute_cache = orig
            peak = torch.cuda.max_memory_allocated() / 2**30
            with torch.no_grad():
                ev[2].record()
                dLf, _ = native.eas_key_grad(env_name, cache0[:C].contiguous(), rows_c, coef_c,
                                             graph_ctx=cached.graph_context[:C].contiguous(),
                                             w_capacity=cached.w_capacity,
                                             demand=demand[:C].contiguous() if vrp else None,
                                             vehicle_capacity=vcap[:C].contiguous() if vrp else None)
                ev[3].record()
                dL = torch.matmul(dLf, w_out.t())
            torch.cuda.synchronize()
            rel = float((dL - leaf.grad).norm() / leaf.grad.norm())
            cmp = {"chunk_instances": C, "autograd_ms": ev[0].elapsed_time(ev[1]), "autograd_peak_GiB": round(peak, 2),
                   "kernel_ms": ev[2].elapsed_time(ev[3]), "rel_diff": rel}
        except torch.cuda.OutOfMemoryError:
            dec._precompute_cache = orig
            break

    print(f"{env_name}{N}: autograd comparison {cmp}", file=sys.stderr, flush=True)

    # ---- search progress
    torch.cuda.synchronize()
    import time

    t0 = time.time()
    out = eas_search(pol, env, td, max_iters=iters, augment_size=A, seed=1)
    torch.cuda.synchronize()
    wall = time.time() - t0
    hist = out["reward_history"]
    prog = {str(i): float(hist[i - 1 if i > 0 else 0].mean()) for i in (0, 50, iters) if i <= hist.shape[0]}
    return {"env": f"{env_name}{N}", "B": B, "augment": A, "starts": S, "ms_per_iter": {
        "rollout": round(t_roll, 2), "eas_key_grad": round(t_grad, 2), "adam_refold": round(t_adam, 2)},
        "autograd_comparison": cmp, "mean_max_reward_after_iters": prog, "search_wall_s": round(wall, 1),
        "policy": "randomly initialised (seed 0)", "gpu": gpu_info()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--envs", default="tsp,cvrp")
    p.add_argument("--N", type=int, default=100)
    p.add_argument("--B", type=int, default=1024)
    p.add_argument("--augment", type=int, default=8)
    p.add_argument("--iters", type=int, default=200)
    p.add_argument("--split-iters", type=int, default=3)
    p.add_argument("--chunks", default="8,32,128,512")
    p.add_argument("--out", default=None, help="JSON file for the results")
    a = p.parse_args()
    from rl4co_b200 import native

    native.build()
    lines = []
    for env_name in a.envs.split(","):
        line = run(env_name, a.N, a.B, a.augment, a.iters, a.split_iters, [int(c) for c in a.chunks.split(",")])
        print(json.dumps(line), flush=True)
        lines.append(line)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
