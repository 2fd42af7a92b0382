"""PolyNet on the H100: rollout, stepping path and training step, next to the plain multistart rollout.

For TSP-100 and CVRP-100 with a randomly initialised (seeded) PolyNet policy, k = 128 (no trained checkpoint ships
with the project):
  * evaluation rollout, B instances x 8 dihedral augmentations x 800 solutions, sampling: the PolyNet rollout
    (`co_rollout` with `poly`) and the plain multistart sampling rollout of an AM policy with the same weights at the same
    S, from the same encoder output, alternated over `--rounds` rounds in this run (CUDA events, cache GEMM included);
  * the stepping path (torch pointer, one launch per stage per step) on a slice of `--step-slice` instances, its time
    scaled by B / slice and labelled as scaled;
  * one training step at k rows per instance (B instances, no augmentation), split into the rollout without a graph,
    the best-row replay (encoder + teacher-forced pass) and backward plus the Adam step.
The card name and power limit are read in the same run.  Prints one JSON line per environment.
"""

from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tools.bench_eas import gpu_info  # noqa: E402


def _timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def bench_env(env_name, B, A, S, k, rounds, step_slice, dev):
    from rl4co_b200.envs import get_env
    from rl4co_b200.ops import StateAugmentation, unbatchify
    from rl4co_b200.policy import FusedAttentionModelPolicy
    from rl4co_b200.polynet import FusedPolyNetPolicy, poppy_mask
    from rl4co_b200.reinforce import evaluate_log_likelihood

    torch.manual_seed(0)
    env = get_env(env_name, generator_params=dict(num_loc=100), check_solution=False)
    pol = FusedPolyNetPolicy(k=k, env_name=env_name).to(dev).eval()
    am = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=6, normalization="instance").to(dev).eval()
    am.load_state_dict(pol.state_dict(), strict=False)
    td = env.reset(env.generator(B).to(dev))
    tda = StateAugmentation(num_augment=A, augment_fn="dihedral8")(td)
    res = {"env": env_name, "B": B, "augment": A, "num_solutions": S, "k": k}
    with torch.inference_mode():
        enc = pol.encoder(tda)
        runs = {
            "polynet": lambda: pol(tda, env, phase="test", decode_type="sampling", num_starts=S, seed=1,
                                   encoder_output=enc),
            "plain": lambda: am(tda, env, phase="test", decode_type="multistart_sampling", num_starts=S, seed=1,
                                encoder_output=enc),
        }
        small = StateAugmentation(num_augment=A, augment_fn="dihedral8")(td[:4])
        enc_small = pol.encoder(small)
        for m in (pol, am):  # warm-up: module load, cache weights, every shape the kernels see
            m(small, env, phase="test", decode_type="multistart_sampling", num_starts=S, seed=1,
              encoder_output=enc_small)
        times = {name: [] for name in runs}
        for _ in range(rounds):
            for name, fn in runs.items():
                ms, out = _timed(fn)
                times[name].append(ms)
                res[f"{name}_mean_max_aug_reward"] = float(unbatchify(out["reward"], (A, S)).amax((1, 2)).mean())
        for name, t in times.items():
            res[f"{name}_rollout_ms"] = [round(x, 1) for x in t]
        res["polynet_over_plain"] = round(min(times["polynet"]) / min(times["plain"]), 2)
        # the stepping path on a slice, scaled to the whole batch
        sl = StateAugmentation(num_augment=A, augment_fn="dihedral8")(td[:step_slice])
        enc_sl = pol.encoder(sl)
        pol(sl[:1], env, phase="test", decode_type="sampling", num_starts=S, seed=1, fused_rollout=False,
            encoder_output=(enc_sl[0][:1], enc_sl[1][:1]))
        ms, _ = _timed(lambda: pol(sl, env, phase="test", decode_type="sampling", num_starts=S, seed=1,
                                   fused_rollout=False, encoder_output=enc_sl))
        res["stepping_slice_instances"] = step_slice
        res["stepping_rollout_ms_scaled_to_B"] = round(ms * B / step_slice, 1)
    # one training step at k rows per instance, split as polynet_step runs it
    pol.train()
    opt = torch.optim.Adam(pol.parameters(), lr=1e-4)
    split = {"rollout": [], "replay": [], "backward_optimizer": []}
    for it in range(2):  # the first step warms up the training shapes
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        with torch.no_grad():
            enc = pol.encoder(td)
            out = pol(td, env, phase="train", decode_type="sampling", num_starts=k, seed=it,
                      encoder_output=(enc[0], enc[1]))
        ev[1].record()
        reward = unbatchify(out["reward"], k)
        best = poppy_mask(reward).float().argmax(-1)
        acts = unbatchify(out["actions"], k)[torch.arange(B, device=dev), best].contiguous()
        h, _ = pol.encoder(td)
        ll = evaluate_log_likelihood(pol, td, env, acts, hidden=h, forced_first=True, strategy=best % k)
        ev[2].record()
        loss = -((reward.gather(1, best[:, None]).squeeze(1) - reward.mean(-1)) * ll).sum() / (B * k)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        ev[3].record()
        torch.cuda.synchronize()
        if it > 0:
            for i, name in enumerate(split):
                split[name].append(round(ev[i].elapsed_time(ev[i + 1]), 1))
    res["train_step_ms"] = {n: v[0] for n, v in split.items()}
    res["train_B"] = B
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=1024)
    ap.add_argument("--augment", type=int, default=8)
    ap.add_argument("--solutions", type=int, default=800)
    ap.add_argument("--k", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--step-slice", type=int, default=8)
    ap.add_argument("--envs", default="tsp,cvrp")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_polynet needs a CUDA device")
    dev = torch.device("cuda:0")
    info = gpu_info()
    rows = []
    for env_name in args.envs.split(","):
        r = bench_env(env_name, args.B, args.augment, args.solutions, args.k, args.rounds, args.step_slice, dev)
        r["gpu"] = info
        print(json.dumps(r), flush=True)
        rows.append(r)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
