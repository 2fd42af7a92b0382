"""Benchmark of co_generate_locs (the fused generators' non-uniform `loc_distribution`s) against rl4co's samplers.

For each location law and N: B = --batch instances generated on the device, timed with CUDA events after warm-up
(median of --reps launches; the uniform kernel co_generate_uniform is timed alongside for scale).  The reference
sampler (envs/common/distribution_utils.py, from the staged reference copy) runs on the host CPU for --cpu-batch
instances, once, and its time is scaled linearly to B; those columns are marked `scaled`.  The card name and power
limit come from nvidia-smi in the same run.

    python tools/bench_generators.py --out-dir /tmp/gen_bench [--batch 65536] [--n 20 100 1000]
"""

from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from rl4co_b200 import native  # noqa: E402

LAWS = {  # name: (co_generate_locs kind, parameters, reference class name, its arguments)
    "uniform": ("uniform", {}, None, ()),
    "cluster(3)": ("cluster", dict(n_cluster=3), "Cluster", (3,)),
    "mixed(1)": ("mixed", dict(n_cluster_mix=1), "Mixed", (1,)),
    "gaussian_mixture(1,1)": ("gaussian_mixture", dict(num_modes=1, cdist=1), "Gaussian_Mixture", (1, 1)),
    "gaussian_mixture(5,30)": ("gaussian_mixture", dict(num_modes=5, cdist=30), "Gaussian_Mixture", (5, 30)),
    "mix_distribution(3,1)": ("mix_distribution", dict(n_cluster=3, n_cluster_mix=1), "Mix_Distribution", (3, 1)),
    "mix_multi_distributions": ("mix_multi_distributions", {}, "Mix_Multi_Distributions", ()),
}


def gpu_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = (q.stdout.strip().splitlines()[0].split(", ") + ["?", "?"])[:2] if q.returncode == 0 else ("?", "?")
    return {"gpu": name, "power_limit": power, "torch_device": torch.cuda.get_device_name(0),
            "cpu_threads": torch.get_num_threads()}


def time_kernel(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    ms.sort()
    return ms[len(ms) // 2]


def reference_cpu(cls_name, args, b, n):
    from oracle import ref_standin

    if cls_name is None or not ref_standin.reference_available():
        return None
    ref_standin.install()
    import importlib

    du = importlib.import_module("rl4co.envs.common.distribution_utils")
    torch.manual_seed(0)
    random.seed(0)
    sampler = getattr(du, cls_name)(*args)
    sampler.sample((2, n, 2))  # first-call set-up outside the timing
    t0 = time.perf_counter()
    sampler.sample((b, n, 2))
    return 1e3 * (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--n", type=int, nargs="+", default=[20, 100, 1000])
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--cpu-batch", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    dev = torch.device("cuda:0")
    res = {"info": gpu_info(), "batch": args.batch, "rows": []}
    print(json.dumps(res["info"]))
    for n in args.n:
        shape = (args.batch, n, 2)
        for name, (kind, kw, cls_name, ref_args) in LAWS.items():
            if kind == "uniform":
                fn = lambda: native.generate_uniform(shape, dev, 1, 0)  # noqa: E731
            else:
                fn = lambda: native.generate_locs(shape, dev, 1, 0, kind, **kw)  # noqa: E731
            ms = time_kernel(fn, args.warmup, args.reps)
            row = {"law": name, "n": n, "batch": args.batch, "kernel_ms": round(ms, 3),
                   "write_GBps": round(args.batch * n * 8 / (ms * 1e-3) / 1e9, 1)}
            cb = min(args.cpu_batch, args.batch)
            ref_ms = reference_cpu(cls_name, ref_args, cb, n)
            if ref_ms is not None:
                scaled = ref_ms * args.batch / cb
                row.update(ref_cpu_batch=cb, ref_cpu_ms=round(ref_ms, 1), ref_cpu_ms_scaled=round(scaled, 1),
                           speedup_vs_scaled_ref=round(scaled / ms, 1))
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
    with open(os.path.join(args.out_dir, "bench_generators.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
