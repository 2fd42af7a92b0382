"""Small driver for ncu: runs the persistent rollout kernel a few times on a batch that is a
multiple of the SM count (kept short: ncu replays every launch ~40x)."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from rl4co_b200 import native
from rl4co_b200.envs import get_env
from rl4co_b200.policy import FusedAttentionModelPolicy

p = argparse.ArgumentParser()
p.add_argument("--env", default="tsp")
p.add_argument("--num-loc", type=int, default=100)
p.add_argument("--batch", type=int, default=132 * 8)
p.add_argument("--iters", type=int, default=3)
p.add_argument("--decode-type", default="greedy")
p.add_argument("--num-starts", type=int, default=0)
a = p.parse_args()
dev = torch.device("cuda:0")
torch.manual_seed(0)
pol = FusedAttentionModelPolicy(env_name=a.env, num_encoder_layers=3).to(dev).eval()
env = get_env(a.env, generator_params=dict(num_loc=a.num_loc), check_solution=False)
torch.manual_seed(1234)
with torch.inference_mode():
    td = env.reset(env.generator(a.batch).to(dev))
    kw = {"num_starts": a.num_starts} if a.num_starts else {}
    for _ in range(a.iters):
        out = pol(td, env, decode_type=a.decode_type, **kw)
torch.cuda.synchronize()
print("selections", out["actions"].numel(), "reward mean", out["reward"].mean().item())
