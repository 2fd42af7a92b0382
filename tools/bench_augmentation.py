"""Benchmark of co_symmetric_augment (StateAugmentation(augment_fn="symmetric") on CUDA) against the reference's torch
expression on the same GPU.

At POMO evaluation shapes (TSP-100, --batch instances, S augmentations each) and the same angles, it times:
  kernel  native.symmetric_augment(base, phi, S): reads [B, N, 2] once, writes [S*B, N, 2]
  torch   batchify(base, S) then symmetric_transform (data/transforms.py:49-69, restated in rl4co_b200/ops.py), as
          the reference's StateAugmentation computes it: one elementwise kernel per operation
Each is timed two ways after warm-up: `call_ms`, CUDA events around one call (median of --reps), which at these sizes
includes the host's launch overhead, and `device_ms`, the GPU time of the kernels one call launches, summed from a
torch.profiler trace of --reps calls.  The outputs are checked to be equal in the same run, and the card name and power
limit come from nvidia-smi in the same run.

    python tools/bench_augmentation.py --out-dir /tmp/aug_bench [--batch 1024] [--n 100] [--augment 8 32 128]
"""

from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from rl4co_b200 import native  # noqa: E402
from rl4co_b200.ops import batchify, symmetric_transform  # noqa: E402


def gpu_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = (q.stdout.strip().splitlines()[0].split(", ") + ["?", "?"])[:2] if q.returncode == 0 else ("?", "?")
    return {"gpu": name, "power_limit": power, "torch_device": torch.cuda.get_device_name(0)}


def time_it(fn, warmup, reps):
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


def device_ms(fn, reps):
    """GPU time of the kernels (and copies) one call of fn launches, from a profiler trace of reps calls."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    us = sum(e.self_device_time_total for e in prof.key_averages() if e.device_type == DeviceType.CUDA)
    return us / reps / 1e3


def torch_path(base, phi, S):
    xy = batchify(base, S)
    return symmetric_transform(xy[..., [0]], xy[..., [1]], phi[:, None, None])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--n", type=int, default=100)
    ap.add_argument("--augment", type=int, nargs="+", default=[8, 32, 128])
    ap.add_argument("--warmup", type=int, default=200)  # tens of microseconds each: enough to bring the clocks up
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_augmentation.py times CUDA kernels: no CUDA device")
    os.makedirs(args.out_dir, exist_ok=True)
    dev = torch.device("cuda:0")
    res = {"info": gpu_info(), "batch": args.batch, "n": args.n, "rows": []}
    print(json.dumps(res["info"]))
    torch.manual_seed(0)
    base = torch.rand(args.batch, args.n, 2, device=dev)
    for S in args.augment:
        phi = torch.rand(S * args.batch, device=dev) * 4 * math.pi
        phi[: args.batch] = 0.0
        same = torch.equal(native.symmetric_augment(base, phi, S), torch_path(base, phi, S))
        kernel = lambda: native.symmetric_augment(base, phi, S)  # noqa: E731
        reference = lambda: torch_path(base, phi, S)  # noqa: E731
        k_call, t_call = time_it(kernel, args.warmup, args.reps), time_it(reference, args.warmup, args.reps)
        k_dev, t_dev = device_ms(kernel, args.reps), device_ms(reference, args.reps)
        moved = base.numel() * 4 + phi.numel() * 4 + S * base.numel() * 4  # bytes the kernel must read + write
        row = {"augment": S, "kernel_device_ms": round(k_dev, 4), "torch_device_ms": round(t_dev, 4),
               "device_speedup": round(t_dev / k_dev, 1), "kernel_GBps": round(moved / (k_dev * 1e-3) / 1e9, 1),
               "kernel_call_ms": round(k_call, 4), "torch_call_ms": round(t_call, 4), "outputs_equal": same}
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    with open(os.path.join(args.out_dir, "bench_augmentation.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
