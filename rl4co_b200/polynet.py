"""PolyNet (Hottung et al. 2024; rl4co/models/zoo/polynet/) on the fused AM / POMO engine.

PolyNet is the AM policy plus one residual MLP on the pointer glimpse, conditioned on a per-trajectory bit vector, so
that the k trajectories of an instance follow k learned strategies (rl4co/models/nn/attention.py, PolyNetAttention):

    g  = project_out(heads)
    z  = binary_vectors[s % k]          s = the trajectory's index among the num_starts of its instance
    g' = g + poly_layer_2(relu(poly_layer_1(cat(g, z))))
    logits = g' . logit_key / sqrt(E)   then tanh clipping, mask and temperature as in AM

The layer is not linear, so `project_out` cannot stay folded into the logit key: block 2 of the PolyNet decoder's cache
holds the un-folded logit key.  Whole episodes run in the multistart rollout kernel (`co_rollout_args.poly`, weights
packed by `pack_poly`); single-start decoding, N > 128, top-k / top-p and `return_entropy` take the stepping path,
whose pointer is written in torch ops (correct rather than fast).
"""

from __future__ import annotations

import itertools
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import native
from .decoder import FusedAttentionModelDecoder, _Pointer
from .ops import StateAugmentation, gather_by_index, unbatchify
from .policy import FusedAttentionModelPolicy
from .reinforce import evaluate_log_likelihood

E = native.EMBED_DIM
POLY_DIM = native.POLY_DIM


def binary_vectors(k: int) -> torch.Tensor:
    """[k, ceil(log2 k)] float: the first k bit vectors of itertools.product([0, 1], ...), most significant bit first
    (PolyNetAttention.binary_vectors)."""
    if k < 1:
        raise ValueError(f"k must be >= 1, got {k}")
    bits = math.ceil(math.log2(k))
    return torch.tensor(list(itertools.product([0, 1], repeat=bits))[:k], dtype=torch.float32).reshape(k, bits)


class _PolyPointer(_Pointer):
    """Parameter holder named like PolyNetAttention: `project_out`, `binary_vectors` (not trainable),
    `poly_layer_1` Linear(E + bits, P) and `poly_layer_2` Linear(P, E)."""

    def __init__(self, k: int, embed_dim: int, poly_layer_dim: int):
        super().__init__(embed_dim)
        self.k = k
        self.binary_vector_dim = math.ceil(math.log2(k))
        self.binary_vectors = nn.Parameter(binary_vectors(k), requires_grad=False)
        self.poly_layer_1 = nn.Linear(embed_dim + self.binary_vector_dim, poly_layer_dim)
        self.poly_layer_2 = nn.Linear(poly_layer_dim, embed_dim)

    def poly(self, glimpse: torch.Tensor, strategy: torch.Tensor) -> torch.Tensor:
        """g + poly_layer_2(relu(poly_layer_1(cat(g, z)))) with z = binary_vectors[strategy]; `strategy` (int64)
        broadcasts against glimpse[..., 0]."""
        z = self.binary_vectors[strategy].to(glimpse.dtype)
        z = z.expand(*glimpse.shape[:-1], self.binary_vector_dim)
        return glimpse + self.poly_layer_2(F.relu(self.poly_layer_1(torch.cat((glimpse, z), -1))))


def pack_poly(pointer: _PolyPointer) -> torch.Tensor:
    """The packed weights of `co_rollout_args.poly`: [W_out^T | W1 | W2 | b2 | c] with matrices (in, out) and the
    per-strategy bias c[i] = b1 + poly_layer_1.weight[:, E:] . binary_vectors[i]."""
    with torch.no_grad():
        w1 = pointer.poly_layer_1.weight
        c = pointer.poly_layer_1.bias + pointer.binary_vectors.to(w1.dtype) @ w1[:, E:].t()
        parts = (pointer.project_out.weight.t(), w1[:, :E].t(), pointer.poly_layer_2.weight.t(),
                 pointer.poly_layer_2.bias, c)
        return torch.cat([p.reshape(-1).float() for p in parts]).contiguous()


class FusedPolyNetDecoder(FusedAttentionModelDecoder):
    """rl4co's PolyNetDecoder (polynet/decoder.py) for the AM encoder: the AM decoder with a PolyNetAttention pointer.
    Parameter names match the reference, so a reference PolyNet `state_dict` loads strictly and an AM / POMO
    `state_dict` loads with `strict=False`, missing only the poly keys (rl4co's `base_model_checkpoint_path`)."""

    def __init__(self, k: int, encoder_type: str = "AM", embed_dim: int = 128, poly_layer_dim: int = 256,
                 num_heads: int = 8, env_name: str = "tsp", **kwargs):
        if encoder_type != "AM":
            raise NotImplementedError(f"encoder_type={encoder_type!r}: the fused PolyNet decoder covers the AM encoder")
        if poly_layer_dim != POLY_DIM:
            raise NotImplementedError(f"poly_layer_dim={poly_layer_dim}: the rollout kernel is instantiated for {POLY_DIM}")
        env_name = getattr(env_name, "name", env_name)
        if env_name not in ("tsp", "cvrp"):
            raise NotImplementedError(f"PolyNet covers tsp and cvrp, not {env_name!r}")
        super().__init__(embed_dim=embed_dim, num_heads=num_heads, env_name=env_name, **kwargs)
        self.encoder_type = encoder_type
        self.pointer = _PolyPointer(k, embed_dim, poly_layer_dim)

    def fused_weight(self) -> torch.Tensor:
        """Wcat as in the AM decoder, except that block 2 is the un-folded logit key (the poly layer sits between
        project_out and the logit key)."""
        wk, wv, wl = self.project_node_embeddings.weight.chunk(3, dim=0)
        wc = self.context_embedding.project_context.weight
        blocks = [wk, wv, wl]
        if self.env_name == "tsp":
            blocks += [wc[:, :E], wc[:, E:2 * E]]
        else:
            blocks.append(wc[:, :E])
        return torch.cat(blocks, dim=0)

    def rollout_extras(self, num_starts: int) -> dict:
        """Keyword arguments of `native.rollout` for this decoder: the packed poly weights, recomputed only when a
        weight changed."""
        p = self.pointer
        ps = (p.project_out.weight, p.poly_layer_1.weight, p.poly_layer_1.bias, p.poly_layer_2.weight,
              p.poly_layer_2.bias, p.binary_vectors)
        ver = tuple((t._version, t.data_ptr()) for t in ps)
        hit = self.__dict__.get("_poly_cache")
        if hit is None or hit[0] != ver:
            hit = (ver, pack_poly(p))
            self.__dict__["_poly_cache"] = hit
        return {"poly": hit[1], "poly_k": p.k}

    def forward(self, td, cached, num_starts: int = 0):
        """am/decoder.py:156-193 with the PolyNet pointer, in torch ops -> (logits [B_traj, N] raw, mask [B_traj, N]).
        Rows j = s * B + b; with num_starts > 1 row j takes strategy s % k, otherwise every row takes strategy 0 (the
        reference reshapes the glimpse to [B, num_starts, E] and indexes the bit vectors along that axis)."""
        mask = td["action_mask"]
        B_traj, N = mask.shape
        emb = cached.node_embeddings
        B = emb.shape[0]
        S = B_traj // B
        inst = torch.arange(B_traj, device=mask.device) % B
        cur = td["current_node"].reshape(-1)
        wc = self.context_embedding.project_context.weight
        if self.env_name == "tsp":
            if int(td["i"].reshape(-1)[0]) < 1:
                q = F.linear(self.context_embedding.W_placeholder, wc).expand(B_traj, E)
            else:
                first = td["first_node"].reshape(-1)
                q = F.linear(torch.cat([emb[inst, first], emb[inst, cur]], -1), wc)
        else:
            state = (td["vehicle_capacity"] - td["used_capacity"]).reshape(B_traj, 1)
            q = F.linear(torch.cat([emb[inst, cur], state], -1), wc)
        if cached.graph_context_or_none is not None:
            q = q + cached.graph_context[inst]
        H = self.num_heads
        # start-major rows -> [B, S, .]: the S queries of an instance attend to its cached keys together
        qb = q.view(S, B, E).transpose(0, 1)
        mb = mask.view(S, B, N).transpose(0, 1)

        def heads(x):
            return x.reshape(x.shape[0], x.shape[1], H, -1).transpose(1, 2)

        o = F.scaled_dot_product_attention(heads(qb), heads(cached.glimpse_key), heads(cached.glimpse_val),
                                           attn_mask=mb[:, None])
        glimpse = self.pointer.project_out(o.transpose(1, 2).reshape(B, S, E))
        strategy = torch.arange(S, device=mask.device) % self.pointer.k if num_starts > 1 else \
            torch.zeros(S, dtype=torch.int64, device=mask.device)
        glimpse = self.pointer.poly(glimpse, strategy[None])
        logits = torch.bmm(glimpse, cached.logit_key.transpose(1, 2)) / math.sqrt(E)     # [B, S, N]
        return logits.transpose(0, 1).reshape(B_traj, N), mask


class FusedPolyNetPolicy(FusedAttentionModelPolicy):
    """rl4co's PolyNetPolicy (polynet/policy.py) with the AM encoder.  With `num_starts > 1` a `sampling` or `greedy`
    decode runs forced-start multistart, start s % num_loc and strategy s % k, as rl4co's DecodingStrategy resolves
    `policy(td, env, num_starts=n, multisample=True)`; that decode is one launch of the fused multistart kernel."""

    def __init__(self, k: int, encoder: nn.Module = None, encoder_type: str = "AM", embed_dim: int = 128,
                 num_encoder_layers: int = 6, num_heads: int = 8, normalization: str = "instance",
                 feedforward_hidden: int = 512, env_name: str = "tsp", temperature: float = 1.0,
                 tanh_clipping: float = 10.0, mask_logits: bool = True, train_decode_type: str = "sampling",
                 val_decode_type: str = "sampling", test_decode_type: str = "sampling", poly_layer_dim: int = 256,
                 use_graph_context: bool = True, fused_rollout: bool = True, **kwargs):
        if encoder_type != "AM":
            raise NotImplementedError(f"encoder_type={encoder_type!r}: the fused PolyNet policy covers the AM encoder")
        env_name = getattr(env_name, "name", env_name)
        decoder = FusedPolyNetDecoder(k=k, encoder_type=encoder_type, embed_dim=embed_dim,
                                      poly_layer_dim=poly_layer_dim, num_heads=num_heads, env_name=env_name,
                                      use_graph_context=use_graph_context)
        super().__init__(encoder=encoder, decoder=decoder, embed_dim=embed_dim, num_encoder_layers=num_encoder_layers,
                         num_heads=num_heads, normalization=normalization, feedforward_hidden=feedforward_hidden,
                         env_name=env_name, temperature=temperature, tanh_clipping=tanh_clipping,
                         mask_logits=mask_logits, train_decode_type=train_decode_type, val_decode_type=val_decode_type,
                         test_decode_type=test_decode_type, fused_rollout=fused_rollout, **kwargs)
        self.k = k

    def forward(self, td, env=None, phase: str = "train", calc_reward: bool = True, return_actions: bool = True,
                actions=None, **kw):
        kw.pop("multisample", None)
        decode_type = kw.pop("decode_type", None) or getattr(self, f"{phase}_decode_type")
        num_starts = kw.get("num_starts", None)
        if actions is None and decode_type in ("sampling", "greedy") and num_starts is not None and num_starts > 1:
            decode_type = "multistart_" + decode_type  # utils/decoding.py: num_starts > 1 -> multistart
        if actions is not None or "multistart" not in decode_type or (num_starts is not None and num_starts <= 1):
            kw["fused_rollout"] = False  # the kernel's poly layer needs num_starts > 1
        return super().forward(td, env, phase=phase, calc_reward=calc_reward, return_actions=return_actions,
                               actions=actions, decode_type=decode_type, **kw)


# reference-compatible alias
PolyNetPolicy = FusedPolyNetPolicy


def poppy_mask(reward: torch.Tensor) -> torch.Tensor:
    """[B, k] bool: the best row of each instance (Poppy, polynet/model.py calculate_loss).  Ties keep the lowest row
    index; the reference ranks with a double `argsort`, which is not stable, so any tied row is a valid outcome of it."""
    best = reward.argmax(-1)  # the first maximal index
    return F.one_hot(best, reward.shape[-1]).bool()


def polynet_step(policy, env, td, k=None, val_num_solutions=800, num_augment=8, phase="test", optimizer=None,
                 decode_type=None, augment_fn="dihedral8", first_aug_identity=True, feats=None):
    """PolyNet.shared_step (polynet/model.py).

    train: k forced-start rows per instance are sampled without a graph (strategy s % k), the Poppy mask keeps the best
    row of each instance, the shared baseline is the mean over the k rows, and
    loss = -((reward - mean) * ll * mask).mean() over [B, k].  The masked loss has zero gradient on every other row, so
    only the best row of each instance is replayed by the differentiable teacher-forced pass: the same loss and
    gradient for 1/k of the replay.  No augmentation.
    val / test: `num_augment` augmentations (dihedral-8 by default) x `val_num_solutions` rows; returns the keys of
    `pomo_step`: max_reward, best_multistart_actions, max_aug_reward and best_aug_actions.  A greedy decode needs
    val_num_solutions <= k (more rows would repeat strategies and starts)."""
    k = policy.decoder.pointer.k if k is None else k
    B = td.batch_size[0]
    if phase == "train":
        if k < 2:
            raise ValueError("the Poppy training step needs k > 1 rows per instance")
        policy.train()
        enc = policy.encoder(td)
        with torch.no_grad():
            out = policy(td, env, phase="train", decode_type=decode_type or policy.train_decode_type, num_starts=k,
                         multisample=True, encoder_output=(enc[0].detach(), enc[1]))
        reward = unbatchify(out["reward"], k)                                   # [B, k]
        mask = poppy_mask(reward)
        best = mask.float().argmax(-1)                                          # [B]
        acts = unbatchify(out["actions"], k)[torch.arange(B, device=best.device), best]
        ll_best = evaluate_log_likelihood(policy, td, env, acts.contiguous(), hidden=enc[0], forced_first=True,
                                          strategy=best % policy.decoder.pointer.k)
        advantage = reward.gather(1, best[:, None]).squeeze(1) - reward.mean(-1)
        loss = -(advantage * ll_best).sum() / (B * k)
        if optimizer is not None:
            from .distributed import sync_gradients

            optimizer.zero_grad(set_to_none=True)
            loss.backward()
            sync_gradients(policy.parameters())
            optimizer.step()
        return {"loss": loss.detach(), "reward": reward, "max_reward": reward.max(-1)[0], "mask": mask,
                "actions": out["actions"], "best_actions": acts}
    decode_type = decode_type or getattr(policy, f"{phase}_decode_type")
    if "greedy" in decode_type and val_num_solutions > k:
        raise ValueError(f"greedy evaluation needs val_num_solutions <= k (got {val_num_solutions} > {k})")
    n_aug = num_augment
    if n_aug > 1:
        td = StateAugmentation(num_augment=n_aug, augment_fn=augment_fn, first_aug_identity=first_aug_identity,
                               feats=feats)(td)
    n_start = val_num_solutions
    with torch.inference_mode():
        out = policy(td, env, phase=phase, decode_type=decode_type, num_starts=n_start, multisample=True)
    shape = (n_aug, n_start) if n_aug > 1 else (n_start,)
    reward = unbatchify(out["reward"], shape)                                   # [B, aug, S] | [B, S]
    max_reward, max_idxs = reward.max(-1)
    best_ms = gather_by_index(unbatchify(out["actions"], shape), max_idxs, dim=max_idxs.dim())
    res = {"reward": reward, "max_reward": max_reward, "actions": out["actions"], "best_multistart_actions": best_ms}
    if n_aug > 1:
        res["max_aug_reward"], aug_idxs = max_reward.max(1)
        res["best_aug_actions"] = gather_by_index(best_ms, aug_idxs)
    return res
