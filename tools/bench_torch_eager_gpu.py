"""GPU-vs-GPU comparator (SURVEY.md 8d): the reference ALGORITHM in PyTorch eager on the GPU
(the oracle port, fp32, TF32 off, host syncs and per-step K/V/L copies as in rl4co) next to the fused
path on the same instances.  Test/bench infrastructure: imports oracle/."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from oracle import am_rollout_oracle as O
from rl4co_b200.envs import get_env
from rl4co_b200.policy import FusedAttentionModelPolicy

torch.backends.cuda.matmul.allow_tf32 = False
dev = torch.device("cuda:0")
for env_name, n, B, dt in (("tsp", 100, 4096, "greedy"), ("tsp", 50, 4096, "greedy"), ("cvrp", 50, 4096, "greedy")):
    torch.manual_seed(0)
    pol = FusedAttentionModelPolicy(env_name=env_name).eval()
    W = {k: v.detach().to(dev) for k, v in pol.state_dict().items()}
    pol = pol.to(dev)
    env = get_env(env_name, generator_params=dict(num_loc=n), check_solution=False)
    torch.manual_seed(1234)
    td_host = env.generator(B)
    inst = {k: td_host[k].to(dev) for k in td_host.keys()}
    with torch.inference_mode():
        def ref():
            return O.policy_forward(W, env_name, inst, decode_type=dt, faithful_copies=True)
        def ours():
            return pol(env.reset(td_host.to(dev)), env, decode_type=dt)
        res = {}
        for name, fn in (("torch_eager_gpu", ref), ("fused", ours)):
            out = fn(); torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(3):
                out = fn()
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) / 3 * 1e3
            res[name] = {"ms": ms, "sel_per_s": out["actions"].numel() / ms * 1e3}
    res["config"] = f"{env_name.upper()}-{n} {dt} policy-forward B={B}"
    res["speedup"] = res["torch_eager_gpu"]["ms"] / res["fused"]["ms"]
    print(json.dumps(res))
