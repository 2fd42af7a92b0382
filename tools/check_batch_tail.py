"""Run bench.py's parity gate on three windows of the headline batch, not only its first rows.

Builds the tsp100 workload as bench.py does (65 536 TSP-100 instances, greedy, default policy, the same seeds), runs
the encoder, the cache GEMM and native.rollout once, and calls `bench.parity_gate` on 1 024-instance windows of the
instances, the encoder output and the rollout result:
  head      the first 1 024 instances (the window bench.py itself checks);
  boundary  the window around the instance whose decoder-cache rows hold float offset 2^31;
  tail      the last 1 024 instances.
Prints one JSON line per window.  Peak device memory is the benchmark's (about 17 GB).

    python tools/check_batch_tail.py [--batch 65536]
"""

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402

ROWS = 1024


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--batch", type=int, default=None, help="instances (default: the workload's 65 536)")
    args = p.parse_args()

    from rl4co_b200 import native
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy
    from rl4co_b200.tensordict import TensorDict

    assert torch.cuda.is_available(), "check_batch_tail.py needs a CUDA device"
    wl = bench.WORKLOADS["tsp100"]
    dev = torch.device("cuda:0")
    env_name, N = wl["env"], wl["n"]
    B = args.batch or wl["batch"]
    native.lib()
    torch.manual_seed(0)
    policy = FusedAttentionModelPolicy(env_name=env_name, **bench.policy_kwargs(wl)).to(dev).eval()
    env = get_env(env_name, generator_params=dict(num_loc=N), check_solution=False)
    torch.manual_seed(1234)
    td_host = env.generator(B)
    with torch.inference_mode():
        td_dev = env.reset(TensorDict({k: v.to(dev) for k, v in td_host.items()}, batch_size=[B]))
        h, _ = policy.encoder(td_dev)
        h = h.contiguous()
        cached = policy.decoder._precompute_cache(h)
        cache = cached.rollout_cache
        res = native.rollout(env_name, native.SELECT_GREEDY, cache, cached.graph_context_or_none, cached.q_placeholder,
                             cached.w_capacity, td_dev["locs"], None, None, B, N, tanh_clipping=10.0, seed=1)
    torch.cuda.synchronize()
    per_instance = cache.shape[1] * cache.shape[2]
    boundary = (1 << 31) // per_instance
    del cached, cache
    windows = {"head": 0, "boundary": min(max(0, boundary - ROWS // 2), B - ROWS), "tail": B - ROWS}
    for name, w0 in windows.items():
        w1 = w0 + ROWS
        td_w = {k: td_dev[k][w0:w1] for k in ("locs", "demand") if k in td_dev.keys()}
        res_w = {k: res[k][w0:w1] for k in ("actions", "logprobs", "reward", "steps")}
        gate = bench.parity_gate(wl, policy, td_w, h[w0:w1], res_w, rows=ROWS)
        line = {"window": name, "instances": [w0, w1], "cache_floats": [w0 * per_instance, w1 * per_instance],
                "past_2_31": w1 * per_instance > 1 << 31, **gate}
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
