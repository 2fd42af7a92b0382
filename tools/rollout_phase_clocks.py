"""Phase clocks of the persistent rollout kernel: where each warp spends a TSP decode step around its two block
barriers.

Builds libcorollout.so with -DCO_PHASE_CLOCKS into its own directory (never the package's library), runs one greedy
TSP rollout of a batch that gives every SM the same number of instances, and prints
  * the mean cycles of each window of a decode step (glimpse, B1 wait, selection, B2 wait, tail up to the next step)
    and of the instance set-up (instance top to the first step),
  * each warp's mean lag behind the first warp to arrive at B1 and at B2, and how often it arrives last.

    python tools/rollout_phase_clocks.py [--num-loc 100] [--out-dir DIR] [--json FILE]

The stamps cost a clock read and a store per warp and stamp, so absolute cycles are a little above those of the
shipped build; the lags between warps are what this measures.
"""
import argparse
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from rl4co_b200 import native  # noqa: E402

SLOTS = 6  # step top, B1 arrival, B1 release, B2 arrival, B2 release, instance top (dstep-0 row)
WARPS = 8


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--num-loc", type=int, default=100)
    p.add_argument("--per-sm", type=int, default=8, help="instances per SM")
    p.add_argument("--out-dir", default=None, help="build directory of the diagnostic library (default: a temporary one)")
    p.add_argument("--json", default=None, help="also write the report here")
    a = p.parse_args()

    out_dir = a.out_dir or tempfile.mkdtemp(prefix="co_phase_clocks_")
    lib_path = native.build(extra_flags=["-DCO_PHASE_CLOCKS"],
                            lib_path=os.path.join(out_dir, "libcorollout.so"))
    native.LIB_PATH = lib_path  # load the diagnostic library instead of the package's
    L = native.lib()
    L.co_phase_clocks_set.argtypes = [native.c_void_p]

    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy

    dev = torch.device("cuda:0")
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    B, N = sms * a.per_sm, a.num_loc
    torch.manual_seed(0)
    pol = FusedAttentionModelPolicy(env_name="tsp", num_encoder_layers=3).to(dev).eval()
    env = get_env("tsp", generator_params=dict(num_loc=N), check_solution=False)
    torch.manual_seed(1234)
    clk = torch.zeros(B * N * WARPS * SLOTS, dtype=torch.int64, device=dev)
    assert L.co_phase_clocks_set(clk.data_ptr()) == 0  # before any launch: the kernel does not test the pointer
    with torch.inference_mode():
        td = env.reset(env.generator(B).to(dev))
        for _ in range(2):  # warm-up, then the run whose stamps are kept
            pol(td, env, decode_type="greedy")
        torch.cuda.synchronize()
    c = clk.view(B, N, WARPS, SLOTS).cpu().numpy().astype(np.int64)

    step = c[:, :, :, :5]
    d = lambda x, y: (step[:, :, :, y] - step[:, :, :, x]).mean()  # noqa: E731
    tail = (step[:, 1:, :, 0] - step[:, :-1, :, 4]).mean()
    per_step = (step[:, 1:, :, 0] - step[:, :-1, :, 0]).mean()
    setup = (c[:, 0, :, 0] - c[:, 0, :, 5]).mean()
    b1, b2 = step[:, :, :, 1], step[:, :, :, 3]
    lag1 = (b1 - b1.min(axis=2, keepdims=True)).mean(axis=(0, 1))
    lag2 = (b2 - b2.min(axis=2, keepdims=True)).mean(axis=(0, 1))
    last1 = np.bincount(b1.argmax(axis=2).ravel(), minlength=WARPS) / b1[:, :, 0].size
    last2 = np.bincount(b2.argmax(axis=2).ravel(), minlength=WARPS) / b2[:, :, 0].size
    rep = {
        "gpu": torch.cuda.get_device_name(dev), "instances": B, "nodes": N,
        "cycles": {"step": float(per_step), "glimpse": float(d(0, 1)), "b1_wait": float(d(1, 2)),
                   "select": float(d(2, 3)), "b2_wait": float(d(3, 4)), "tail": float(tail),
                   "instance_setup": float(setup)},
        "lag_b1": [float(x) for x in lag1], "lag_b2": [float(x) for x in lag2],
        "last_b1": [float(x) for x in last1], "last_b2": [float(x) for x in last2],
    }
    print(f"{rep['gpu']}: TSP-{N} greedy, {B} instances ({a.per_sm} per SM), mean cycles over all warps and steps")
    for k, v in rep["cycles"].items():
        print(f"  {k:15s} {v:8.1f}")
    print("  warp   lag@B1  lag@B2  last@B1 last@B2")
    for h in range(WARPS):
        print(f"  {h:4d} {lag1[h]:8.1f} {lag2[h]:7.1f} {last1[h]:7.1%} {last2[h]:7.1%}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(rep, f, indent=1)


if __name__ == "__main__":
    main()
