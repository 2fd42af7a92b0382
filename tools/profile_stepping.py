"""Driver for ncu / timing of the eight step-at-a-time kernels at the BASELINE size (65 536 x 100):
three full env.step / decoder.forward / strategy.step rounds through the public stepping API, then reward +
validity + baseline statistics.  Also prints CUDA-event times and the achieved fraction of the data-sheet HBM
bandwidth per kernel (algorithmic bytes / kernel time), so the same script gives the numbers
with and without the profiler (a time taken under ncu is never a bench value).

    python tools/profile_stepping.py [--batch 65536] [--num-loc 100]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from rl4co_b200 import native
from rl4co_b200.decoding import Greedy
from rl4co_b200.envs import get_env
from rl4co_b200.policy import FusedAttentionModelPolicy

p = argparse.ArgumentParser()
p.add_argument("--batch", type=int, default=65536)
p.add_argument("--num-loc", type=int, default=100)
p.add_argument("--rounds", type=int, default=3)
a = p.parse_args()
dev = torch.device("cuda:0")
PEAK = 3350.0  # HBM3 bandwidth of the H100 SXM in GB/s (NVIDIA data sheet), as in bench.py


def timed(fn, n=5):
    if os.environ.get("NCU"):  # under the profiler: one launch per kernel is enough (ncu replays it ~40 times)
        fn(); torch.cuda.synchronize()
        return float("nan")
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


report = []
for env_name in ("tsp", "cvrp"):
    torch.manual_seed(0)
    B, n = a.batch, a.num_loc
    env = get_env(env_name, generator_params=dict(num_loc=n), check_solution=False)
    pol = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=1).to(dev).eval()
    with torch.inference_mode():
        td = env.reset(env.generator(B).to(dev))
        N = td["action_mask"].shape[-1]
        h, _ = pol.encoder(td)
        td, env, cached = pol.decoder.pre_decoder_hook(td, env, h)
        strat = Greedy(tanh_clipping=10.0)
        for _ in range(a.rounds):  # the reference loop body (constructive/base.py:226-236), one kernel per stage
            logits, mask = pol.decoder(td, cached, 0)
            td = strat.step(logits, mask, td)
            td = env.step(td)["next"]
        # timings of each stage on the current state (outputs discarded)
        t_logits = timed(lambda: pol.decoder(td, cached, 0))
        t_select = timed(lambda: native.select_action(logits, mask, native.SELECT_GREEDY))
        act = td["action"]
        if env_name == "tsp":
            m_in = td["action_mask"].contiguous()
            outs = [torch.empty_like(m_in), td["first_node"].clone(), torch.empty_like(act), td["i"].clone().view(-1),
                    torch.empty(B, dtype=torch.bool, device=dev)]
            t_step = timed(lambda: native.tsp_step(act, m_in, outs[0], outs[1], outs[2], outs[3], outs[4]))
            report.append(("co_tsp_step", t_step, B * (2 * N + 8 + 24)))
        else:
            vis = td["visited"].contiguous()
            o = [torch.empty_like(td["used_capacity"]), torch.empty_like(vis), torch.empty(B, 1, dtype=torch.int64, device=dev),
                 torch.empty(B, dtype=torch.bool, device=dev), torch.empty(B, N, dtype=torch.bool, device=dev)]
            t_step = timed(lambda: native.cvrp_step(act, td["demand"], td["vehicle_capacity"], td["used_capacity"], o[0], vis,
                                                    o[1], o[2], o[3], o[4]))
            report.append(("co_cvrp_step", t_step, B * (3 * N + 4 * (N - 1) + 32)))
            t_mask = timed(lambda: env.get_action_mask(td))
            report.append(("co_cvrp_action_mask", t_mask, B * (2 * N + 4 * (N - 1) + 16)))
        report.append((f"co_pointer_logits[{env_name}]", t_logits, B * (3 * N * 512 + 2 * 512 + N + N * 4)))
        report.append((f"co_select_action[{env_name}]", t_select, B * (5 * N + 12)))
        torch.manual_seed(1)
        td0 = env.reset(env.generator(B).to(dev))
        full = pol(td0, env, decode_type="greedy")  # valid tours for reward / check
        acts = full["actions"].contiguous()
        T = acts.shape[1]
        t_len = timed(lambda: native.tour_length(td0["locs"].contiguous(), acts, with_depot=(env_name == "cvrp")))
        report.append((f"co_tour_length[{env_name}]", t_len, B * (8 * N + 8 * T + 4)))
        if env_name == "tsp":
            t_chk = timed(lambda: native.check_tours(acts, N))
        else:
            t_chk = timed(lambda: native.check_tours(acts, N, td0["demand"].contiguous(),
                                                     td0["vehicle_capacity"].reshape(-1).contiguous(), B_inst=B))
        report.append((f"co_check_tours[{env_name}]", t_chk, B * (8 * T + (4 * (N - 1) if env_name == "cvrp" else 0))))
        stats = torch.zeros(2, dtype=torch.float64, device=dev)
        big = torch.randn(1 << 24, device=dev)
        t_rs = timed(lambda: native.reward_stats(big, stats))
        report.append(("co_reward_stats[16M]", t_rs, big.numel() * 4))
torch.cuda.synchronize()
print(f"{'kernel':32s} {'ms':>9s} {'alg. MB':>10s} {'GB/s':>9s} {'of HBM peak':>11s}   (B={a.batch}, num_loc={a.num_loc}; incl. launch overhead)")
for name, ms, byts in report:
    gbs = byts / (ms * 1e-3) / 1e9
    print(f"{name:32s} {ms:9.4f} {byts / 1e6:10.1f} {gbs:9.1f} {gbs / PEAK:10.1%}")
