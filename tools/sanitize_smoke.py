"""Small end-to-end run of every kernel family for compute-sanitizer (memcheck / racecheck / initcheck)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from rl4co_b200 import native
from rl4co_b200.envs import get_env
from rl4co_b200.policy import FusedAttentionModelPolicy
from rl4co_b200.reinforce import pomo_step

dev = torch.device("cuda:0")
CASES = (("tsp", 20), ("cvrp", 20), ("sdvrp", 20), ("tsp", 50), ("cvrp", 100), ("tsp", 100))
if os.environ.get("SAN_ONLY"):
    CASES = tuple(c for c in CASES if c[0] == os.environ["SAN_ONLY"])
for env_name, n in CASES:
    torch.manual_seed(0)
    env = get_env(env_name, generator_params=dict(num_loc=n), check_solution=True)
    pol = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=1).to(dev).eval()
    with torch.inference_mode():
        td = env.reset(env.generator(300).to(dev))
        for dt, kw in (("greedy", {}), ("sampling", {"seed": 1}), ("multistart_greedy", {"num_starts": 3})):
            out = pol(td, env, decode_type=dt, **kw)
        out = pol(td, env, decode_type="greedy", fused_rollout=False)   # stepping kernels
        pol(td, env, actions=out["actions"])                             # evaluate mode
    print(env_name, n, "ok", out["reward"].mean().item())
# large-M GEMM path (pipe) + generic
a = torch.randn(20000, 128, device=dev); w = torch.randn(384, 128, device=dev)
hi, lo = native.split_tf32(w)
native.gemm_tf32x3(a, hi, lo, bias=torch.randn(384, device=dev), relu=True)
a = torch.randn(300, 512, device=dev); w = torch.randn(128, 512, device=dev)
hi, lo = native.split_tf32(w)
native.gemm_tf32x3(a, hi, lo, residual=torch.randn(300, 128, device=dev))
torch.cuda.synchronize()
print("gemm ok")
# orienteering: stepping kernels only (co_op_step / co_op_action_mask / co_op_reward)
env = get_env("op", generator_params=dict(num_loc=20), check_solution=True)
pol = FusedAttentionModelPolicy(env_name="op", num_encoder_layers=1).to(dev).eval()
with torch.inference_mode():
    for kw in (dict(decode_type="greedy"), dict(decode_type="sampling"), dict(decode_type="sampling", fused_rollout=False)):
        out = pol(env.reset(env.generator(300).to(dev)), env, **kw)
print("op ok", out["reward"].mean().item())
env = get_env("pctsp", generator_params=dict(num_loc=20), check_solution=True)
pol = FusedAttentionModelPolicy(env_name="pctsp", num_encoder_layers=1).to(dev).eval()
with torch.inference_mode():
    for kw in (dict(decode_type="greedy"), dict(decode_type="sampling"), dict(decode_type="sampling", fused_rollout=False)):
        out = pol(env.reset(env.generator(300).to(dev)), env, **kw)
print("pctsp ok", out["reward"].mean().item())
# training-step attention kernels (forward, dQ, dK/dV) with a mask and strided key / value views; instance norm
from rl4co_b200 import attention_train as AT

torch.manual_seed(1)
q = torch.randn(6, 131, 128, device=dev, requires_grad=True)
cache = torch.randn(6, 101, 512, device=dev, requires_grad=True)
mask = torch.rand(6, 131, 101, device=dev) < 0.5
mask[..., 0] = True
AT.attention(q, cache[..., :128], cache[..., 128:256], mask).square().sum().backward()
qkv = torch.randn(5, 100, 384, device=dev, requires_grad=True)
AT.self_attention_packed(qkv).sum().backward()
native.instance_norm(torch.randn(9, 100, 128, device=dev), torch.ones(128, device=dev), torch.zeros(128, device=dev))
torch.cuda.synchronize()
print("attention / norm ok")
# PolyNet: the multistart kernel's poly variant (co_rollout_args.poly), k = 3 strategies wrapping over 7 starts
from rl4co_b200.polynet import FusedPolyNetPolicy

for env_name in ("tsp", "cvrp"):
    env = get_env(env_name, generator_params=dict(num_loc=50), check_solution=True)
    pol = FusedPolyNetPolicy(k=3, env_name=env_name, num_encoder_layers=1).to(dev).eval()
    with torch.inference_mode():
        out = pol(env.reset(env.generator(40).to(dev)), env, decode_type="sampling", num_starts=7, seed=3)
    print("polynet", env_name, "ok", out["reward"].mean().item())
# 2-opt local search (co_tsp_two_opt): both distance sources, on both sides of the shared-memory residency bound
# (CO_TWO_OPT_RESIDENT_MAX_NODES = 224); the in-place segment reversal is what racecheck looks at
for n in (20, 224, 300):
    g = torch.Generator().manual_seed(n)
    locs = torch.rand(4, n, 2, generator=g).to(dev)
    tours = torch.argsort(torch.rand(4, n, generator=g), dim=1).to(dev)
    d = (locs[:, :, None] - locs[:, None]).norm(dim=-1)
    its = torch.empty(4, dtype=torch.int32, device=dev)
    native.tsp_two_opt(tours, 50, locs=locs, iterations=its)
    native.tsp_two_opt(tours, 50, distances=d, iterations=its)
torch.cuda.synchronize()
print("local search ok")
# location laws (co_generate_locs): every kind, including the shared-memory shuffle (mixed) and the counting sort by
# mode (gaussian_mixture), at sizes on both sides of a full CTA and at the node limit
for n in (2, 33, 300, 10000):
    for kind, kw in (("uniform", {}), ("constant", dict(value=0.5)), ("normal", dict(mean=0.5, std=0.1)),
                     ("cluster", dict(n_cluster=3)), ("mixed", dict(n_cluster_mix=2)),
                     ("gaussian_mixture", dict(num_modes=1, cdist=1)), ("gaussian_mixture", dict(num_modes=5, cdist=30)),
                     ("mix_distribution", dict(n_cluster=3, n_cluster_mix=1)), ("mix_multi_distributions", {})):
        native.generate_locs((5, n, 2), dev, 1, 0, kind, **kw)
torch.cuda.synchronize()
print("generate_locs ok")
# symmetric augmentation (co_symmetric_augment): one node per instance (a warp spans 32 instances), warps straddling
# instances, and a partial last warp
for B, S, N in ((37, 3, 1), (5, 8, 20), (3, 2, 1000)):
    native.symmetric_augment(torch.rand(B, N, 2, device=dev), torch.rand(S * B, device=dev) * 4 * torch.pi, S)
torch.cuda.synchronize()
print("symmetric_augment ok")
# CVRP local search (co_cvrp_local_search): both distance sources on both sides of the residency bound, an invalid row
# (copied through) and the pointer surgery of every move kind
for n in (20, 223, 300):
    g = torch.Generator().manual_seed(n)
    locs = torch.rand(4, n + 1, 2, generator=g).to(dev)
    dem = (torch.randint(1, 10, (4, n), generator=g) / 40.0).to(dev)
    perm = torch.argsort(torch.rand(4, n, generator=g), dim=1) + 1
    tours = torch.zeros(4, 2 * n, dtype=torch.int64)
    tours[:, ::2] = perm  # one customer per route
    tours[3, 0] = n + 1
    tours = tours.to(dev)
    d = (locs[:, :, None] - locs[:, None]).norm(dim=-1)
    its = torch.empty(4, dtype=torch.int32, device=dev)
    native.cvrp_local_search(tours, dem, torch.ones(4, device=dev), 50, locs=locs, iterations=its)
    native.cvrp_local_search(tours, dem, torch.ones(4, device=dev), 50, distances=d, iterations=its)
torch.cuda.synchronize()
print("cvrp local search ok")
