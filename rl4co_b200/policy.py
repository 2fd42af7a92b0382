"""AttentionModelPolicy whose decode loop is ONE persistent CUDA kernel.

Mirrors ``AttentionModelPolicy`` (rl4co/models/zoo/am/policy.py:12-125) and the loop owner
``ConstructivePolicy.forward`` (rl4co/models/common/constructive/base.py:154-263): same
constructor keywords, same ``policy(td, env, phase, calc_reward, return_actions, actions,
**decoding_kwargs) -> dict`` contract, same output keys / shapes / layouts (multistart rows
are start-major, flat index s*B+b).

Two execution paths, both CUDA-only:
  * fused rollout (default): encoder -> one cache GEMM -> `co_rollout` (whole episode in one
    launch, zero host syncs inside; one `.item()` at the end to trim CVRP's padded columns);
  * stepping (``fused_rollout=False`` or N > 128): the reference's loop structure, with one
    kernel each for decoder.forward / strategy.step / env.step.
"""

from __future__ import annotations

import os

import torch
import torch.nn as nn

from . import native
from .decoder import FusedAttentionModelDecoder
from .decoding import get_decoding_strategy, get_log_likelihood
from .encoder import AttentionModelEncoder
from .envs import get_env
from .ops import unbatchify
from .tensordict import TensorDict


class FusedAttentionModelPolicy(nn.Module):
    def __init__(self, encoder: nn.Module = None, decoder: nn.Module = None, embed_dim: int = 128,
                 num_encoder_layers: int = 3, num_heads: int = 8, normalization: str = "batch",
                 feedforward_hidden: int = 512, env_name: str = "tsp", use_graph_context: bool = True,
                 linear_bias_decoder: bool = False, mask_inner: bool = True, out_bias_pointer_attn: bool = False,
                 check_nan: bool = True, temperature: float = 1.0, tanh_clipping: float = 10.0,
                 mask_logits: bool = True, train_decode_type: str = "sampling", val_decode_type: str = "greedy",
                 test_decode_type: str = "greedy", fused_rollout: bool = True, **unused_kwargs):
        super().__init__()
        for k in ("moe_kwargs", "sdpa_fn", "sdpa_fn_encoder", "sdpa_fn_decoder", "encoder_network", "init_embedding",
                  "context_embedding", "dynamic_embedding"):
            v = unused_kwargs.pop(k, None)
            if v not in (None, {"encoder": None, "decoder": None}):
                raise NotImplementedError(f"{k}={v!r} is outside the fused path")
        if unused_kwargs:
            raise TypeError(f"unexpected keyword arguments: {list(unused_kwargs)}")
        self.env_name = env_name
        self.encoder = encoder if encoder is not None else AttentionModelEncoder(
            embed_dim=embed_dim, num_heads=num_heads, num_layers=num_encoder_layers, env_name=env_name,
            normalization=normalization, feedforward_hidden=feedforward_hidden)
        self.decoder = decoder if decoder is not None else FusedAttentionModelDecoder(
            embed_dim=embed_dim, num_heads=num_heads, env_name=env_name, mask_inner=mask_inner,
            out_bias_pointer_attn=out_bias_pointer_attn, linear_bias=linear_bias_decoder,
            use_graph_context=use_graph_context, check_nan=check_nan)
        self.temperature, self.tanh_clipping, self.mask_logits = temperature, tanh_clipping, mask_logits
        self.train_decode_type, self.val_decode_type, self.test_decode_type = (
            train_decode_type, val_decode_type, test_decode_type)
        self.fused_rollout = fused_rollout

    # ------------------------------------------------------------------------------ forward
    def forward(self, td: TensorDict, env=None, phase: str = "train", calc_reward: bool = True,
                return_actions: bool = True, return_entropy: bool = False, return_hidden: bool = False,
                return_init_embeds: bool = False, return_sum_log_likelihood: bool = True, actions=None,
                max_steps=1_000_000, encoder_output=None, **decoding_kwargs) -> dict:
        # `encoder_output=(hidden, init_embeds)` reuses an encoder pass (e.g. the differentiable one of a
        # training step) instead of running the encoder again
        hidden, init_embeds = self.encoder(td) if encoder_output is None else encoder_output
        if isinstance(env, str) or env is None:
            env = get_env(self.env_name if env is None else env)

        decode_type = decoding_kwargs.pop("decode_type", None)
        if actions is not None:
            decode_type = "evaluate"
        elif decode_type is None:
            decode_type = getattr(self, f"{phase}_decode_type")

        N = td["action_mask"].shape[-1]
        filtered = decoding_kwargs.get("top_k", 0) > 0 or decoding_kwargs.get("top_p", 0.0) > 0
        if not filtered:  # explicit zeros mean "off" (decoding.py:180-185)
            decoding_kwargs.pop("top_k", None), decoding_kwargs.pop("top_p", None)
        # the kernels' fixed-offset log-softmax needs a tanh clip and 2*clip/T within exp's fp32 range
        # (exp(-2*clip/T) must not flush to zero): other settings take the stepping path
        clip_ = decoding_kwargs.get("tanh_clipping", self.tanh_clipping)
        temp_ = decoding_kwargs.get("temperature", self.temperature)
        softmax_ok = clip_ > 0 and temp_ > 0 and 2.0 * clip_ / temp_ < 80.0
        env_name_ = getattr(env, "name", self.env_name)
        use_fused = (decoding_kwargs.pop("fused_rollout", self.fused_rollout) and N <= native.rollout_max_nodes()
                     and softmax_ok and env_name_ in native.ROLLOUT_ENVS
                     and not filtered and decode_type != "beam_search"
                     and not return_entropy and not decoding_kwargs.get("store_all_logp", False)
                     and decoding_kwargs.get("mask_logits", self.mask_logits)
                     and decoding_kwargs.get("select_start_nodes_fn", None) is None)
        if use_fused:
            out = self._forward_fused(td, env, hidden, decode_type, actions, calc_reward, return_sum_log_likelihood,
                                      decoding_kwargs)
        else:
            out = self._forward_stepping(td, env, hidden, decode_type, actions, calc_reward, return_entropy,
                                         return_sum_log_likelihood, max_steps, decoding_kwargs)
        if not return_actions:
            out.pop("actions", None)
        if return_hidden:
            out["hidden"] = hidden
        if return_init_embeds:
            out["init_embeds"] = init_embeds
        return out

    # --------------------------------------------------------------------- fused whole episode
    def _forward_fused(self, td, env, hidden, decode_type, actions, calc_reward, return_sum_ll, kw) -> dict:
        env_name = env.name
        temperature = kw.pop("temperature", self.temperature)
        tanh_clipping = kw.pop("tanh_clipping", self.tanh_clipping)
        kw.pop("mask_logits", None)
        num_starts = kw.pop("num_starts", None)
        num_samples = kw.pop("num_samples", None)
        select_best = kw.pop("select_best", False)
        noise = kw.pop("noise", None)            # [T, B_traj, N] Exp(1) draws (parity protocol)
        sampling_noise = kw.pop("sampling_noise", "philox")  # "philox" (in-kernel) | "torch" (generator)
        seed = kw.pop("seed", None)
        kw.pop("multistart", None)
        philox_offset = kw.pop("philox_offset", None)
        if kw:
            raise NotImplementedError(f"decoding kwargs outside the fused path: {list(kw)}")

        B, N = td["action_mask"].shape
        S, forced_start = 1, False
        if "multistart" in decode_type:
            S = num_starts if num_starts is not None else env.get_num_starts(td)
            forced_start = S > 1
            S = max(S, 1)
        elif num_samples is not None and num_samples > 1:
            S = num_samples
        B_traj = B * S
        # decode-step bound: tsp N; cvrp 2(N-1) (every customer + a depot return each); sdvrp 3(N-1)+2 (a customer can
        # be split once per refill on top of that)
        T_max = {"tsp": N, "cvrp": 2 * (N - 1), "op": N + 1, "pctsp": N + 1}.get(env_name, 3 * (N - 1) + 2)  # op / pctsp: customers once + depot
        cached = self.decoder._precompute_cache(hidden)

        forced = None
        if decode_type == "evaluate":
            mode = native.SELECT_EVALUATE
            if actions.shape[0] != B_traj:
                raise ValueError(f"actions has {actions.shape[0]} rows, expected {B_traj}")
            forced = torch.zeros(B_traj, T_max, dtype=torch.int64, device=actions.device)
            forced[:, : actions.shape[1]] = actions
        elif "greedy" in decode_type:
            mode = native.SELECT_GREEDY
        elif "sampling" in decode_type:
            if noise is None and sampling_noise == "torch":
                noise = torch.empty(T_max, B_traj, N, device=hidden.device).exponential_(1)
            mode = native.SELECT_SAMPLE_NOISE if noise is not None else native.SELECT_SAMPLE_PHILOX
            if seed is None and mode == native.SELECT_SAMPLE_PHILOX:
                seed = int(torch.randint(0, 2**62, (1,)).item())
            if mode == native.SELECT_SAMPLE_PHILOX and philox_offset is None:
                # identically seeded ranks must not draw identical streams
                from .distributed import rank_stream_offset

                philox_offset = rank_stream_offset()
        else:
            raise NotImplementedError(f"decode type {decode_type!r} is outside the fused path")

        vrp = env_name in ("cvrp", "sdvrp")
        demand = td["demand"].contiguous() if vrp else None
        vcap = td["vehicle_capacity"].reshape(-1).contiguous() if vrp else None
        node_limit = None
        if env_name == "op":  # prizes ride in `demand`, the budget at the depot in `vehicle_capacity` (corollout.h)
            demand = td["prize"][..., 1:].contiguous()
            vcap = td["max_length"][..., 0].contiguous()
            node_limit = td["max_length"].contiguous()
        elif env_name == "pctsp":  # real prizes in `demand`, prize_required in `vehicle_capacity`, penalties in `node_limit`
            demand = td["real_prize"][..., 1:].contiguous()
            vcap = td["prize_required"].reshape(-1).contiguous()
            node_limit = td["penalty"].contiguous()
        num_loc = getattr(env.generator, "num_loc", N - (1 if vrp or env_name in ("op", "pctsp") else 0))
        extra = self.decoder.rollout_extras(S) if hasattr(self.decoder, "rollout_extras") else {}
        with torch.no_grad():
            res = native.rollout(
                env_name, mode, cached.rollout_cache.detach().contiguous(), cached.graph_context_or_none,
                cached.q_placeholder, cached.w_capacity, td["locs"].contiguous(), demand, vcap, B, N, num_starts=S,
                forced_start=forced_start, num_loc=num_loc, T_max=T_max, forced_actions=forced,
                noise=noise.contiguous() if noise is not None else None, tanh_clipping=tanh_clipping,
                temperature=temperature, seed=seed or 0, offset=philox_offset or 0, dyn_w=cached.dyn_w,
                node_limit=node_limit, **extra)
        if env_name == "tsp":
            T = N
        elif decode_type == "evaluate":
            T = actions.shape[1]
        else:
            T = int(res["max_steps"].item())  # the reference loop runs until every instance is done
        out_actions = res["actions"][:, :T]
        logprobs = res["logprobs"][:, :T]
        reward = res["reward"]
        if torch.is_grad_enabled() and hidden.requires_grad:
            # the whole-episode kernel is forward-only: under autograd (e.g. the reference's
            # REINFORCE.shared_step calling policy(td, env, phase="train") and then loss.backward(),
            # reinforce.py:59-69) the log-probs of exactly the selected actions are recomputed by the
            # differentiable teacher-forced pass, so `log_likelihood` carries a grad_fn
            from .reinforce import evaluate_log_likelihood

            logprobs = evaluate_log_likelihood(self, td, env, out_actions.contiguous(), hidden=hidden,
                                               return_sum=False, temperature=temperature, tanh_clipping=tanh_clipping,
                                               forced_first=forced_start)
        if calc_reward and env.check_solution:
            td_chk = td if S == 1 else TensorDict({k: td[k] for k in ("locs", "demand", "vehicle_capacity", "max_length", "real_prize")
                                                   if k in td.keys()}, batch_size=td.batch_size)
            self._check(env, td_chk, out_actions.contiguous(), S)
        if S > 1 and select_best:  # decoding.py:415-423
            _, max_idxs = unbatchify(reward, S).max(dim=-1)
            pick = lambda x: unbatchify(x, S)[torch.arange(B, device=x.device), max_idxs]
            out_actions, logprobs, reward = pick(out_actions), pick(logprobs), pick(reward)
        return {
            "reward": reward,
            "log_likelihood": logprobs.sum(1) if return_sum_ll else logprobs,
            "actions": out_actions,
        }

    @staticmethod
    def _check(env, td, actions, S):
        if env.name in ("op", "pctsp"):  # rows of start-major trajectories share instances (j % B)
            env.check_solution_validity(td, actions)
            return
        if env.name == "tsp":
            bad = native.check_tours(actions, td["locs"].shape[-2])
        elif env.name == "sdvrp":  # torch replay on the device (validation path), start-major rows share instances
            tdx = td if S == 1 else TensorDict({k: td[k].repeat(S, *([1] * (td[k].dim() - 1))) for k in ("demand", "vehicle_capacity")},
                                               batch_size=[td.batch_size[0] * S])
            env.check_solution_validity(tdx, actions)
            return
        else:
            bad = native.check_tours(actions, td["locs"].shape[-2], td["demand"].contiguous(),
                                     td["vehicle_capacity"].reshape(-1).contiguous(), B_inst=td["demand"].shape[0])
        assert bad == 0, "Invalid tour"

    # ----------------------------------------------------------------------- step-at-a-time
    def _forward_stepping(self, td, env, hidden, decode_type, actions, calc_reward, return_entropy, return_sum_ll,
                          max_steps, kw) -> dict:
        """constructive/base.py:209-251 with each stage one CUDA kernel."""
        strategy = get_decoding_strategy(
            decode_type, temperature=kw.pop("temperature", self.temperature),
            tanh_clipping=kw.pop("tanh_clipping", self.tanh_clipping),
            mask_logits=kw.pop("mask_logits", self.mask_logits),
            store_all_logp=kw.pop("store_all_logp", return_entropy), **kw)
        # the step kernels are forward-only: under autograd the log-probs of the decoded actions are recomputed by the
        # differentiable teacher-forced pass, as on the fused path; what that pass cannot replay is refused
        regrad = torch.is_grad_enabled() and hidden.requires_grad
        if regrad:
            refused = [name for name, on in (("top_k", strategy.top_k > 0), ("top_p", strategy.top_p > 0),
                                             ("return_entropy", return_entropy),
                                             ("store_all_logp", strategy.store_all_logp),
                                             ("beam_search", decode_type == "beam_search"),
                                             ("select_best", strategy.select_best),
                                             ("mask_logits=False", not strategy.mask_logits)) if on]
            if refused:
                raise NotImplementedError(f"{', '.join(refused)} under autograd: the differentiable teacher-forced pass "
                                          f"does not replay it; decode under torch.no_grad()")
        td_reset = td.clone() if regrad else None  # the env steps below update the state they are given in place
        td, env, num_starts = strategy.pre_decoder_hook(td, env)
        td, env, cached = self.decoder.pre_decoder_hook(td, env, hidden, num_starts)
        step = 0
        while not td["done"].all():
            logits, mask = self.decoder(td, cached, num_starts)
            td = strategy.step(logits, mask, td, action=actions[..., step] if actions is not None else None)
            td = env.step(td)["next"]
            step += 1
            if step > max_steps:
                break
        logprobs, out_actions, td, env = strategy.post_decoder_hook(td, env)
        if regrad:
            from .reinforce import evaluate_log_likelihood

            logprobs = evaluate_log_likelihood(self, td_reset, env, out_actions.contiguous(), hidden=hidden,
                                               return_sum=False, temperature=strategy.temperature,
                                               tanh_clipping=strategy.tanh_clipping,
                                               forced_first=strategy.multistart and num_starts >= 1)
        if calc_reward:
            td.set("reward", env.get_reward(td, out_actions))
        out = {"reward": td["reward"],
               "log_likelihood": get_log_likelihood(logprobs, out_actions, td.get("mask", None), return_sum_ll),
               "actions": out_actions}
        if return_entropy:
            lp = torch.nan_to_num(logprobs, nan=0.0, neginf=0.0)
            out["entropy"] = -(lp.exp() * lp).sum(dim=-1).sum(dim=1)  # ops.py:103-111
        return out


# reference-compatible alias
AttentionModelPolicy = FusedAttentionModelPolicy
