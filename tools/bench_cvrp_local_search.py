"""Timing of co_cvrp_local_search (FusedCVRPEnv.local_search's kernel): B = 4 096 CVRP instances at N = 20 / 50 / 100 /
200, from random tours (random permutations split by capacity) and from tours sampled by an untrained
FusedAttentionModelPolicy, up to 1000 moves per tour.  Kernel time is the median of CUDA-event timings of single
launches after warm-up.  There is no reference timing: rl4co's CVRP local search calls HGS-CVRP, which it does not
ship.

    python tools/bench_cvrp_local_search.py [--B 4096] [--n 20 50 100 200] [--reps 5] [--out file.json]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from rl4co_b200 import native
from rl4co_b200.envs import get_env
from rl4co_b200.policy import FusedAttentionModelPolicy


def random_tours(demand, g):
    """Random permutation per row, a depot visit whenever the next customer does not fit (vectorised over rows)."""
    B, n = demand.shape
    perm = torch.argsort(torch.rand(B, n, generator=g, device=demand.device), dim=1) + 1
    d = demand.gather(1, perm - 1)
    out = torch.zeros(B, 2 * n, dtype=torch.int64, device=demand.device)
    load = torch.zeros(B, device=demand.device)
    col = torch.zeros(B, dtype=torch.int64, device=demand.device)
    rows = torch.arange(B, device=demand.device)
    for k in range(n):
        split = load + d[:, k] > 1.0
        col = col + split.long()
        load = torch.where(split, d[:, k], load + d[:, k])
        out[rows, col] = perm[:, k]
        col = col + 1
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=4096)
    ap.add_argument("--n", type=int, nargs="+", default=[20, 50, 100, 200])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    props = torch.cuda.get_device_properties(dev)
    results = []
    for n in args.n:
        torch.manual_seed(n)
        env = get_env("cvrp", generator_params=dict(num_loc=n))
        td = env.reset(env.generator(args.B).to(dev))
        cap = td["vehicle_capacity"].reshape(-1).contiguous()
        pol = FusedAttentionModelPolicy(env_name="cvrp").to(dev).eval()
        g = torch.Generator(device=dev).manual_seed(n)
        with torch.inference_mode():
            starts = {"random": random_tours(td["demand"], g),
                      "am_sampled": pol(td, env, decode_type="sampling", seed=n)["actions"].contiguous()}
        for name, tours in starts.items():
            its = torch.empty(args.B, dtype=torch.int32, device=dev)
            run = lambda: native.cvrp_local_search(tours, td["demand"], cap, 1000, locs=td["locs"], iterations=its)  # noqa: E731
            out, _ = run()  # warm-up (module load, shared-memory attribute)
            torch.cuda.synchronize()
            times = []
            for _ in range(args.reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                run()
                b.record()
                b.synchronize()
                times.append(a.elapsed_time(b))
            gain = (env.get_reward(td, out) - env.get_reward(td, tours)).mean().item()
            r = dict(N=n, B=args.B, start=name, kernel_ms=sorted(times)[len(times) // 2],
                     moves_per_tour=its.float().mean().item(), max_moves=int(its.max()), mean_reward_gain=gain,
                     start_reward=env.get_reward(td, tours).mean().item())
            print(json.dumps(r), flush=True)
            results.append(r)
    meta = dict(gpu=props.name)
    try:
        import subprocess

        meta["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                             capture_output=True, text=True).stdout.strip()
    except OSError:
        pass
    print(json.dumps(meta))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(meta=meta, results=results), f, indent=1)


if __name__ == "__main__":
    main()
