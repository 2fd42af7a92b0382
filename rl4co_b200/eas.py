"""Efficient active search (EAS; Hottung et al., ICLR 2022; rl4co/models/zoo/eas/search.py): EAS-Emb and EAS-Lay.

`eas_search(policy, env, td, **hparams)` fine-tunes per-instance parameters of a frozen policy: each iteration samples
POMO multistart tours with the whole-episode rollout kernel (`co_rollout`, in-kernel Philox), then takes one optimizer
step on those parameters.
  * EAS-Emb (`use_eas_embedding=True`, the default): the pointer logit key L = node_emb W_L^T.
  * EAS-Lay (`use_eas_layer=True, use_eas_embedding=False`): a residual layer per augmented instance on the
    concatenated head output o of every decode step, o' = o + relu(o W1 + b1) W2 + b2 before project_out
    (rl4co/models/zoo/eas/nn.py, decoder.py:12-31), initialised as rl4co's `EASLayerNet` (`eas_layer_init`): W1, b1
    xavier-uniform over the [B * A, E, E] / [B * A, 1, E] tensors, W2 = b2 = 0, so iteration 0 decodes as the policy.
    The rollout kernel applies the layer in its query-batched (multistart) variant; its gradient comes from
    `co_eas_layer_grad`, which replays the rows teacher-forced through the layer.
The loss is rl4co's

    loss = -mean((r - baseline) * ll_sampled) + eas_lambda * -mean(ll_incumbent)

whose gradient comes from one CUDA kernel that replays the sampled tours and the incumbent teacher-forced; no
[B, S*T, N] logits or glimpses are ever stored.  EAS-Emb: `co_eas_key_grad` gives the gradient with respect to the
folded key Lf = L W_out, keeping the N x E accumulator on chip, and dL = dLf W_out^T.  EAS-Lay: `co_eas_layer_grad`
gives the gradient of the packed [W1 | b1 | W2 | b2] of every instance.

Deviations from rl4co's `EAS`:
  * a function over one batch, not a Lightning `TransductiveModel` (Lightning is not a dependency);
  * iteration 0 has no incumbent row: rl4co imitates an extra sampled start-0 tour there (and its `% num_starts` makes
    one CVRP start the depot);
  * the samples come from the in-kernel Philox stream keyed by (seed, iteration), not `torch.multinomial`;
  * EAS-Emb on the logit key or EAS-Lay, not both at once; `num_parallel_runs=1`, tsp / cvrp and N <= 128;
  * EAS-Lay keeps the four layer tensors in one packed parameter [B * A, 2 E^2 + 2 E]; an element-wise optimizer
    (Adam, the default, SGD, ...) steps it exactly as it would step the four tensors.
"""

from __future__ import annotations

import time

import torch

from . import native
from .ops import StateAugmentation

E = native.EMBED_DIM
BASELINES = ("multistart", "symmetric", "full")


def eas_coefficients(reward: torch.Tensor, baseline: str, eas_lambda: float, with_incumbent: bool) -> torch.Tensor:
    """Per-row weights of the log-likelihoods in rl4co's EAS loss (search.py:219-235).

    reward [S, A, B] (start, augmentation, instance) of the sampled rows.  Returns coef [(S + 1) * A * B] (or
    [S * A * B] without the incumbent) in the kernel's row order r * (A * B) + a * B + b, r = S the incumbent, so that
    sum(coef * ll) == loss_rl + eas_lambda * loss_il."""
    if baseline not in BASELINES:
        raise ValueError(f"Baseline {baseline} not supported.")
    S, A, B = reward.shape
    if baseline == "multistart":
        bl = reward.mean(0, keepdim=True)
    elif baseline == "symmetric":
        bl = reward.mean(1, keepdim=True)
    else:
        bl = reward.mean(0, keepdim=True).mean(1, keepdim=True)
    coef = (-(reward - bl) / (B * A * S)).reshape(-1)
    if with_incumbent:
        coef = torch.cat([coef, torch.full((A * B,), -eas_lambda / (B * A), dtype=coef.dtype, device=coef.device)])
    return coef


def eas_layer_init(num_instances: int, device=None) -> torch.Tensor:
    """rl4co's `EASLayerNet(num_instances, E)` initialisation, drawn the same way from torch's CPU generator (randn of
    W1 and b1, then xavier_uniform_ over the whole [n, E, E] / [n, 1, E] tensors, so the bound depends on n; W2 = b2 =
    0), packed per instance as [W1 (E x E, (in, out)) | b1 | W2 | b2] -> [n, native.EAS_LAYER_FLOATS] on `device`."""
    w1 = torch.randn(num_instances, E, E)
    b1 = torch.randn(num_instances, 1, E)
    torch.nn.init.xavier_uniform_(w1)
    torch.nn.init.xavier_uniform_(b1)
    packed = torch.zeros(num_instances, native.EAS_LAYER_FLOATS, device=device)
    packed[:, :E * E] = w1.reshape(num_instances, E * E).to(device)
    packed[:, E * E:E * E + E] = b1.reshape(num_instances, E).to(device)
    return packed


def unpack_eas_layer(packed: torch.Tensor) -> dict:
    """[n, native.EAS_LAYER_FLOATS] -> {"W1": [n, E, E], "b1": [n, 1, E], "W2": [n, E, E], "b2": [n, 1, E]} (views),
    the shapes of rl4co's `EASLayerNet` parameters."""
    n = packed.shape[0]
    return {"W1": packed[:, :E * E].view(n, E, E), "b1": packed[:, E * E:E * E + E].view(n, 1, E),
            "W2": packed[:, E * E + E:2 * E * E + E].view(n, E, E), "b2": packed[:, 2 * E * E + E:].view(n, 1, E)}


def _make_optimizer(optimizer, params, kwargs):
    if isinstance(optimizer, str):
        return getattr(torch.optim, optimizer)(params, **kwargs)
    return optimizer(params, **kwargs)


def eas_search(policy, env, td, *, use_eas_embedding: bool = True, use_eas_layer: bool = False,
               eas_emb_cache_keys=("logit_key",), eas_lambda: float = 0.013, max_iters: int = 200,
               augment_size: int = 8, augment_dihedral: bool = True, num_parallel_runs: int = 1,
               baseline: str = "multistart", max_runtime: float = 86_400, optimizer="Adam",
               optimizer_kwargs=None, seed: int | None = None, return_logit_key: bool = False,
               return_layer: bool = False) -> dict:
    """EAS-Emb or EAS-Lay over the reset batch `td` [B] (see the module docstring).

    Returns {"max_reward": [B], "best_solutions": [B, T] (0-padded; T = N for tsp, 2 (N - 1) for cvrp),
    "reward_history": [iterations run, B] (the best reward found so far after each iteration)}, plus "logit_key"
    ([A * B, N, E], aug-major) with `return_logit_key=True` (EAS-Emb) and "layer" (`unpack_eas_layer` of the trained
    [A * B, ...] layer, aug-major) with `return_layer=True` (EAS-Lay).  The policy's parameters are not modified.  The
    loop synchronises with the host once per iteration (the `max_runtime` check)."""
    if use_eas_layer and use_eas_embedding:
        raise NotImplementedError("EAS-Emb and EAS-Lay together are not supported (the key gradient would have to go "
                                  "through the layer); pass use_eas_embedding=False for EAS-Lay")
    if not use_eas_embedding and not use_eas_layer:
        raise ValueError("At least one of `use_eas_embedding` or `use_eas_layer` must be True.")
    if use_eas_embedding and list(eas_emb_cache_keys) != ["logit_key"]:
        raise NotImplementedError(f"EAS-Emb fine-tunes the logit key only, got cache keys {list(eas_emb_cache_keys)}")
    if num_parallel_runs != 1:
        raise NotImplementedError("num_parallel_runs != 1 is not supported (rl4co's incumbent bookkeeping assumes one run)")
    if baseline not in BASELINES:
        raise ValueError(f"Baseline {baseline} not supported.")
    env_name = env.name
    if env_name not in ("tsp", "cvrp"):
        raise NotImplementedError(f"eas_search covers tsp and cvrp, not {env_name!r}")
    N = td["action_mask"].shape[-1]
    if N > native.rollout_max_nodes():
        raise NotImplementedError(f"eas_search runs on the whole-episode kernels: N = {N} > {native.rollout_max_nodes()}")
    if not td["locs"].is_cuda:
        raise NotImplementedError("eas_search runs on CUDA tensors only")
    optimizer_kwargs = {"lr": 0.0041, "weight_decay": 1e-6} if optimizer_kwargs is None else dict(optimizer_kwargs)

    B = td.batch_size[0]
    S = env.get_num_starts(td)
    if S < 2:
        raise NotImplementedError("eas_search needs at least two multistart starts")
    A = augment_size
    if A > 1:
        td = StateAugmentation(num_augment=A, augment_fn="dihedral8" if augment_dihedral else "symmetric")(td)
    BA = A * B
    T = N if env_name == "tsp" else 2 * (N - 1)
    dev = td["locs"].device
    layer = torch.nn.Parameter(eas_layer_init(BA, dev)) if use_eas_layer else None  # before any other draw
    if seed is None:
        seed = int(torch.randint(0, 2**62, (1,)).item())
    dec = policy.decoder
    was_training = policy.training
    policy.eval()
    try:
        with torch.no_grad():
            hidden, _ = policy.encoder(td)
            cached = dec._precompute_cache(hidden)
            cache = cached.rollout_cache.contiguous().clone()
            w_out = dec.pointer.project_out.weight.detach().clone()
            w_l = dec.project_node_embeddings.weight.detach()[2 * E:3 * E]
            L = torch.nn.Parameter(torch.matmul(hidden.detach(), w_l.t()).contiguous()) if use_eas_embedding else None
            graph_ctx = cached.graph_context_or_none
            graph_ctx = graph_ctx.detach().contiguous() if graph_ctx is not None else None
            q_ph = cached.q_placeholder.detach() if cached.q_placeholder is not None else None
            w_cap = cached.w_capacity.detach() if cached.w_capacity is not None else None
    finally:
        policy.train(was_training)
    opt = _make_optimizer(optimizer, [L if use_eas_embedding else layer], optimizer_kwargs)
    locs = td["locs"].contiguous()
    demand = td["demand"].contiguous() if env_name == "cvrp" else None
    vcap = td["vehicle_capacity"].reshape(-1).contiguous() if env_name == "cvrp" else None
    num_loc = getattr(env.generator, "num_loc", N - (1 if env_name == "cvrp" else 0))

    max_reward = torch.full((B,), -float("inf"), device=dev)
    best = torch.zeros(B, T, dtype=torch.int64, device=dev)
    bad = torch.zeros(1, dtype=torch.int32, device=dev)
    history = []
    t_start = time.time()
    for it in range(max_iters):
        with torch.no_grad():
            if use_eas_embedding:
                cache[..., 2 * E:3 * E] = torch.matmul(L.detach(), w_out)  # folded key Lf = L W_out (cache block 2)
            res = native.rollout(env_name, native.SELECT_SAMPLE_PHILOX, cache, graph_ctx, q_ph, w_cap, locs, demand,
                                 vcap, BA, N, num_starts=S, forced_start=True, num_loc=num_loc, T_max=T,
                                 tanh_clipping=policy.tanh_clipping, temperature=policy.temperature, seed=seed,
                                 offset=it, layer=layer.detach() if use_eas_layer else None)
            reward = res["reward"].view(S, A, B)
            rows = res["actions"]
            coef = eas_coefficients(reward, baseline, eas_lambda, with_incumbent=it > 0)
            if it > 0:
                rows = torch.cat([rows, best.repeat(A, 1)])  # the incumbent replayed in every augmentation
            kw = dict(graph_ctx=graph_ctx, w_capacity=w_cap, demand=demand, vehicle_capacity=vcap,
                      tanh_clipping=policy.tanh_clipping, temperature=policy.temperature, bad_rows=bad)
            if use_eas_embedding:
                dLf, _ = native.eas_key_grad(env_name, cache, rows, coef.contiguous(), **kw)
                L.grad = torch.matmul(dLf, w_out.t())
            else:
                layer.grad, _ = native.eas_layer_grad(env_name, cache, rows, coef.contiguous(), layer.detach(), **kw)
        opt.step()
        with torch.no_grad():
            # incumbent: the best tour of instance b over starts, augmentations and iterations (strict improvement)
            it_best, idx = reward.permute(2, 1, 0).reshape(B, A * S).max(1)
            a_idx, s_idx = idx // S, idx % S
            cand = res["actions"][s_idx * BA + a_idx * B + torch.arange(B, device=dev)]
            improve = it_best > max_reward
            max_reward = torch.where(improve, it_best, max_reward)
            best = torch.where(improve[:, None], cand, best)
            history.append(max_reward.clone())
        if int(bad.item()):  # the one host synchronisation of the iteration
            raise RuntimeError("the EAS gradient kernel replayed an infeasible trajectory")
        if time.time() - t_start > max_runtime:
            break
    out = {"max_reward": max_reward, "best_solutions": best, "reward_history": torch.stack(history) if history else torch.empty(0, B, device=dev)}
    if return_logit_key and use_eas_embedding:
        out["logit_key"] = L.detach()
    if return_layer and use_eas_layer:
        out["layer"] = unpack_eas_layer(layer.detach())
    return out
