"""Benchmark of co_tsp_two_opt (FusedTSPEnv.local_search) against the reference's numba 2-opt on the host CPU.

For each N: B instances of uniform locs, two kinds of start tours -- random permutations and the greedy tours of a
(randomly initialised) FusedAttentionModelPolicy (N <= 100, the fused rollout's range) -- and the kernel timed with CUDA
events after warm-up (median of --reps).  Reported per row: kernel time, sweeps (iterations) per instance, candidate
moves scored per second (sum over instances of sweeps * (N-1)(N-2)/2 / time), and the reference's
rl4co TSPEnv.local_search on the first --cpu-batch instances of the same inputs (numba threads printed; its time is
also scaled linearly to B).  The card name and power limit come from nvidia-smi in the same run.

    python tools/bench_local_search.py --out-dir /tmp/ls_bench [--batch 4096] [--n 20 50 100 200 500]
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from rl4co_b200 import native  # noqa: E402


def gpu_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = (q.stdout.strip().splitlines()[0].split(", ") + ["?", "?"])[:2] if q.returncode == 0 else ("?", "?")
    return {"gpu": name, "power_limit": power, "torch_device": torch.cuda.get_device_name(0)}


def greedy_tours(locs: torch.Tensor) -> torch.Tensor:
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy
    from rl4co_b200.tensordict import TensorDict

    B, n, _ = locs.shape
    torch.manual_seed(0)
    env = get_env("tsp", generator_params=dict(num_loc=n))
    pol = FusedAttentionModelPolicy(env_name="tsp").to(locs.device).eval()
    with torch.inference_mode():
        out = []
        for s in range(0, B, 8192):
            td = env.reset(TensorDict({"locs": locs[s:s + 8192]}, batch_size=[min(8192, B - s)]))
            out.append(pol(td, env, phase="test", decode_type="greedy")["actions"])
    return torch.cat(out).clone()


def time_kernel(tours, locs, warmup, reps):
    its = torch.empty(tours.shape[0], dtype=torch.int32, device=tours.device)
    for _ in range(warmup):
        native.tsp_two_opt(tours, 1000, locs=locs, iterations=its)
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = native.tsp_two_opt(tours, 1000, locs=locs, iterations=its)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    ms.sort()
    return ms[len(ms) // 2], out, its


def reference_cpu(locs, tours):
    from oracle import ref_standin

    if not ref_standin.reference_available():
        return None
    try:
        import numba
    except ImportError:
        return None
    ref = ref_standin.load()
    td = ref.TensorDict({"locs": locs.cpu()}, batch_size=[locs.shape[0]])
    ref.TSPEnv.local_search(td, tours.cpu()[:1], max_iterations=1)  # JIT compile outside the timing
    t0 = time.perf_counter()
    out = ref.TSPEnv.local_search(td, tours.cpu())
    return {"ms": 1e3 * (time.perf_counter() - t0), "threads": numba.get_num_threads(), "tours": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--n", type=int, nargs="+", default=[20, 50, 100, 200, 500])
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--cpu-batch", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    dev = torch.device("cuda:0")
    res = {"info": gpu_info(), "batch": args.batch, "rows": []}
    print(json.dumps(res["info"]))
    for n in args.n:
        g = torch.Generator().manual_seed(n)
        locs = torch.rand(args.batch, n, 2, generator=g).to(dev)
        starts = {"random": torch.argsort(torch.rand(args.batch, n, generator=g), dim=1).to(dev)}
        if n <= 100:
            starts["am_greedy"] = greedy_tours(locs)
        for kind, tours in starts.items():
            ms, out, its = time_kernel(tours, locs, args.warmup, args.reps)
            moves = its.double().sum().item() * (n - 1) * (n - 2) / 2
            row = {"n": n, "batch": args.batch, "start": kind, "kernel_ms": round(ms, 3),
                   "iterations_mean": round(its.float().mean().item(), 2), "iterations_max": int(its.max().item()),
                   "moves_per_s": moves / (ms * 1e-3)}
            cb = min(args.cpu_batch, args.batch)
            cpu = reference_cpu(locs[:cb], tours[:cb])
            if cpu is not None:
                row.update(ref_cpu_batch=cb, ref_cpu_ms=round(cpu["ms"], 2), ref_cpu_threads=cpu["threads"],
                           ref_cpu_ms_scaled_to_batch=round(cpu["ms"] * args.batch / cb, 1),
                           speedup_vs_scaled_ref=round(cpu["ms"] * args.batch / cb / ms, 1),
                           ref_identical=bool(torch.equal(cpu["tours"], out[:cb].cpu())))
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
    with open(os.path.join(args.out_dir, "bench_local_search.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
