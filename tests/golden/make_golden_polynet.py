"""Generate tests/golden/polynet_{tsp,cvrp}20.npz from the reference's own PolyNet pointer.

The reference's polynet/decoder.py does not import under oracle/ref_standin.py (rl4co.envs needs lightning.fabric), so
the fixture takes the reference AttentionModelPolicy from the stand-in and puts `PolyNetAttention` in its
`decoder.pointer`.  For the AM encoder that is exactly what PolyNetDecoder is: the AM decoder with that pointer.

    python tests/golden/make_golden_polynet.py

Recorded per S (num_starts): multistart greedy (actions, per-step log-probs, reward) and multistart sampling (actions,
per-step log-probs; replayed teacher-forced by the tests).  k = 3 is not a power of two, and S in {2, 7} with k < 7
makes the strategies wrap (start s takes strategy s % 3).
"""

from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_standin  # noqa: E402

ref = ref_standin.load()

K = 3
STARTS = (2, 7)


def npy(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def polynet_fixture(name, n, batch, seed):
    torch.manual_seed(seed)
    Env = ref.TSPEnv if name == "tsp" else ref.CVRPEnv
    env = Env(generator_params=dict(num_loc=n))
    pol = ref.AttentionModelPolicy(env_name=name, num_encoder_layers=1).eval()
    pol.decoder.pointer = ref.attention.PolyNetAttention(K, 128, 256, 8, mask_inner=True, out_bias=False)
    with torch.no_grad():  # a poly layer as large as the glimpse, so that the strategies decode differently
        pol.decoder.pointer.poly_layer_2.weight.mul_(4.0)
    out = {"w::" + k: npy(v) for k, v in pol.state_dict().items() if k.startswith("decoder.")}
    out["k"] = np.int64(K)
    td0 = env.generator(batch_size=[batch])
    for k in td0.keys():
        out[f"inst::{k}"] = npy(td0[k])
    with torch.inference_mode():
        td = env.reset(td0.clone())
        h, _ = pol.encoder(td)
        out["h"] = npy(h)
        for S in STARTS:
            o = pol(td.clone(), env, phase="test", decode_type="multistart_greedy", num_starts=S,
                    return_sum_log_likelihood=False)
            out.update({f"greedy{S}_actions": npy(o["actions"]), f"greedy{S}_logprobs": npy(o["log_likelihood"]),
                        f"greedy{S}_reward": npy(o["reward"])})
            torch.manual_seed(seed + S)
            o = pol(td.clone(), env, phase="train", decode_type="multistart_sampling", num_starts=S,
                    return_sum_log_likelihood=False)
            out.update({f"sampling{S}_actions": npy(o["actions"]), f"sampling{S}_logprobs": npy(o["log_likelihood"])})
    return out


def main():
    for name, seed in (("tsp", 600), ("cvrp", 601)):
        data = polynet_fixture(name, 20, 4, seed)
        path = os.path.join(HERE, f"polynet_{name}20.npz")
        np.savez_compressed(path, **data)
        print(f"polynet_{name}20: {len(data)} arrays, {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
