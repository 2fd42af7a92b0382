"""CUDA drop-in for rl4co's AttentionModelDecoder (rl4co/models/zoo/am/decoder.py:43-228).

Same constructor keywords, same parameter names (a reference ``state_dict`` loads with
``load_state_dict``), same ``forward(td, cached, num_starts) -> (logits, mask)`` and
``pre_decoder_hook(td, env, embeddings, num_starts) -> (td, env, cached)`` signatures.

What differs is the cache layout.  ``_precompute_cache`` does ONE GEMM
``embeddings[B*N,E] @ Wcat^T`` whose column blocks are what the kernels want side by side:

    0  glimpse_key                     (project_node_embeddings rows 0:E)
    1  glimpse_val                     (rows E:2E)
    2  logit_key @ project_out.weight  (rows 2E:3E, folded with pointer.project_out so the
                                        per-step 128x128 projection disappears:
                                        logits = heads . (L W_out)[n] == (W_out heads) . L[n])
    [3 embeddings @ Wctx[:, :E]^T      tsp only: first-node half of project_context as a table --
                                        the multistart kernel reads one row per start, a single-start
                                        episode one row]
    last  embeddings @ Wctx_cur^T      current-node part of project_context (tsp: columns E:2E,
                                        the other envs: columns 0:E)

so that the step query is a table-row read plus a per-episode constant (the reference
re-does a 2E->E / (E+1)->E Linear per step, nn/env_embeddings/context.py:61-74,116-134).
The concatenated weight and its tf32 hi / lo split are cached per weight version.
"""

from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.nn as nn

from . import native
from .tensordict import TensorDict

E = native.EMBED_DIM


class _ContextEmbedding(nn.Module):
    """Parameter holder named like the reference's TSPContext / VRPContext
    (nn/env_embeddings/context.py:50-59,105-114,137-145)."""

    def __init__(self, env_name: str, embed_dim: int):
        super().__init__()
        self.env_name = env_name
        step_context_dim = 2 * embed_dim if env_name == "tsp" else embed_dim + 1
        self.project_context = nn.Linear(step_context_dim, embed_dim, bias=False)
        if env_name == "tsp":
            self.W_placeholder = nn.Parameter(torch.Tensor(2 * embed_dim).uniform_(-1, 1))


class _DynamicEmbedding(nn.Module):
    """Parameter holder named like SDVRPDynamicEmbedding (nn/env_embeddings/dynamic.py:60-78): Linear(1 -> 3E, no bias)
    of the remaining demand, added to glimpse_key / glimpse_val / logit_key every step (am/decoder.py:142-154)."""

    def __init__(self, embed_dim: int):
        super().__init__()
        self.projection = nn.Linear(1, 3 * embed_dim, bias=False)


class _Pointer(nn.Module):
    """Parameter holder named like PointerAttention (nn/attention.py:243-255)."""

    def __init__(self, embed_dim: int):
        super().__init__()
        self.project_out = nn.Linear(embed_dim, embed_dim, bias=False)


@dataclass
class FusedPrecomputedCache:
    """Superset of the reference's PrecomputedCache (am/decoder.py:21-40).

    ``glimpse_key`` / ``glimpse_val`` are zero-copy column views of ``rollout_cache``;
    ``logit_key`` (un-folded) is materialised lazily only if someone asks for it."""

    node_embeddings: torch.Tensor       # [B, N, E]
    graph_context: torch.Tensor | float  # [B, E] or 0
    rollout_cache: torch.Tensor         # [B, N, W] (W = 5E for tsp, 4E otherwise)
    q_placeholder: torch.Tensor | None  # [E] tsp
    w_capacity: torch.Tensor | None     # [E] cvrp
    w_first: None = None                 # always None (see _precompute_cache)
    dyn_w: torch.Tensor | None = None    # [3E] sdvrp: dynamic-embedding weights [wk | wv | W_out^T wl]
    _logit_weight: torch.Tensor | None = None
    _logit_key: torch.Tensor | None = None

    @property
    def glimpse_key(self):
        return self.rollout_cache[..., 0:E]

    @property
    def glimpse_val(self):
        return self.rollout_cache[..., E:2 * E]

    @property
    def logit_key_folded(self):
        return self.rollout_cache[..., 2 * E:3 * E]

    @property
    def logit_key(self):
        if self._logit_key is None:
            self._logit_key = torch.nn.functional.linear(self.node_embeddings, self._logit_weight)
        return self._logit_key

    @property
    def graph_context_or_none(self):
        return self.graph_context if isinstance(self.graph_context, torch.Tensor) else None


class FusedAttentionModelDecoder(nn.Module):
    """See module docstring.  Keyword arguments follow am/decoder.py:69-84; options that
    select other code paths in the reference (dynamic embeddings, MoE, custom pointer / sdpa,
    biases, mask_inner=False) are rejected loudly instead of being silently ignored."""

    def __init__(self, embed_dim: int = 128, num_heads: int = 8, env_name: str = "tsp",
                 context_embedding=None, dynamic_embedding=None, mask_inner: bool = True,
                 out_bias_pointer_attn: bool = False, linear_bias: bool = False, use_graph_context: bool = True,
                 check_nan: bool = True, sdpa_fn=None, pointer=None, moe_kwargs=None, cache_gemm: str = "tf32x3"):
        super().__init__()
        env_name = getattr(env_name, "name", env_name)
        if embed_dim != E or num_heads != native.NUM_HEADS:
            raise NotImplementedError(f"kernels are instantiated for embed_dim={E}, num_heads={native.NUM_HEADS}")
        if env_name not in native.ENV_KIND:
            raise NotImplementedError(f"env {env_name!r} is outside the fused path (tsp, cvrp, sdvrp)")
        for arg, val, ok in (("context_embedding", context_embedding, None), ("dynamic_embedding", dynamic_embedding, None),
                             ("pointer", pointer, None), ("moe_kwargs", moe_kwargs, None), ("mask_inner", mask_inner, True),
                             ("out_bias_pointer_attn", out_bias_pointer_attn, False), ("linear_bias", linear_bias, False)):
            if val is not ok and val != ok:
                raise NotImplementedError(f"{arg}={val!r} is not supported by the fused decoder")
        self.env_name, self.embed_dim, self.num_heads = env_name, embed_dim, num_heads
        self.context_embedding = _ContextEmbedding(env_name, embed_dim)
        self.is_dynamic_embedding = env_name == "sdvrp"
        if self.is_dynamic_embedding:
            self.dynamic_embedding = _DynamicEmbedding(embed_dim)
        self.pointer = _Pointer(embed_dim)
        self.project_node_embeddings = nn.Linear(embed_dim, 3 * embed_dim, bias=False)
        self.project_fixed_context = nn.Linear(embed_dim, embed_dim, bias=False)
        self.use_graph_context = use_graph_context
        self.check_nan = check_nan
        #: "tf32x3": hand-written wgmma 3xTF32 GEMM (fp32-class accuracy, inference / no-grad only);
        #: "cublas": torch.nn.functional.linear (strict fp32 SIMT; always used when autograd is on)
        self.cache_gemm = cache_gemm

    # ------------------------------------------------------------------ cache
    def fused_weight(self) -> torch.Tensor:
        """Wcat [W, E]: row blocks as listed in the module docstring."""
        wk, wv, wl = self.project_node_embeddings.weight.chunk(3, dim=0)
        wlf = self.pointer.project_out.weight.t() @ wl  # (L W_out) = h (W_out^T W_L)^T
        wc = self.context_embedding.project_context.weight
        blocks = [wk, wv, wlf]
        if self.env_name == "tsp":
            blocks += [wc[:, :E], wc[:, E:2 * E]]
        else:
            blocks.append(wc[:, :E])
        return torch.cat(blocks, dim=0)

    def _weight_version(self):
        ps = (self.project_node_embeddings.weight, self.pointer.project_out.weight,
              self.context_embedding.project_context.weight)
        return tuple((p._version, p.data_ptr()) for p in ps)

    def _fused_weight_cached(self):
        """(Wcat, hi, lo) for the no-grad path, recomputed only when a parameter changed (optimizer step,
        load_state_dict, .to()): three small kernels per call otherwise sit inside every timed step."""
        ver = self._weight_version()
        hit = self.__dict__.get("_wcat_cache")
        if hit is None or hit[0] != ver:
            with torch.no_grad():
                wcat = self.fused_weight().contiguous()
                hi, lo = native.split_tf32(wcat) if wcat.is_cuda else (None, None)
            hit = (ver, wcat, hi, lo)
            self.__dict__["_wcat_cache"] = hit
        return hit[1], hit[2], hit[3]

    def _precompute_cache(self, embeddings: torch.Tensor, num_starts: int = 0,
                          first_table: bool | None = None) -> FusedPrecomputedCache:
        """am/decoder.py:201-228."""
        # `first_table` and the always-None `FusedPrecomputedCache.w_first` are kept only for existing callers: the
        # tsp cache always holds the first-node table, so `first_table=False` cannot be honoured
        if first_table is not None and not first_table:
            raise ValueError("first_table=False is not supported: the tsp rollout cache always holds the first-node table")
        needs_grad = torch.is_grad_enabled() and (embeddings.requires_grad or any(
            p.requires_grad for p in (self.project_node_embeddings.weight, self.pointer.project_out.weight,
                                      self.context_embedding.project_context.weight)))
        if self.cache_gemm == "tf32x3" and embeddings.is_cuda and not needs_grad:
            B, N, _ = embeddings.shape
            _, w_hi, w_lo = self._fused_weight_cached()
            cache = native.gemm_tf32x3(embeddings.detach().reshape(B * N, E), w_hi, w_lo).view(B, N, -1)
        elif not needs_grad:
            cache = torch.nn.functional.linear(embeddings, self._fused_weight_cached()[0])
        else:
            cache = torch.nn.functional.linear(embeddings, self.fused_weight())
        if self.use_graph_context:
            graph_context = self.project_fixed_context(embeddings.mean(1))
        else:
            graph_context = 0
        wc = self.context_embedding.project_context.weight
        q_ph = w_cap = None
        if self.env_name == "tsp":
            q_ph = (wc @ self.context_embedding.W_placeholder).contiguous()
        else:
            w_cap = wc[:, E].contiguous()
        return FusedPrecomputedCache(
            node_embeddings=embeddings, graph_context=graph_context, rollout_cache=cache, q_placeholder=q_ph,
            w_capacity=w_cap, dyn_w=self._dynamic_weights() if self.is_dynamic_embedding else None,
            _logit_weight=self.project_node_embeddings.weight[2 * E:],
        )

    def _dynamic_weights(self) -> torch.Tensor:
        """[wk | wv | W_out^T wl]: SDVRPDynamicEmbedding.projection.weight[:, 0] with the logit third folded with
        pointer.project_out like block 2 of the cache (logits = heads . (L + d wl) W_out-folded)."""
        wd = self.dynamic_embedding.projection.weight.detach()[:, 0]
        return torch.cat((wd[:2 * E], self.pointer.project_out.weight.detach().t() @ wd[2 * E:])).contiguous()

    def pre_decoder_hook(self, td, env, embeddings, num_starts: int = 0):
        """am/decoder.py:195-199"""
        return td, env, self._precompute_cache(embeddings, num_starts=num_starts)

    # ------------------------------------------------------------------ one step
    def _step_weights(self) -> native.DecoderWeights:
        wc_t = self.context_embedding.project_context.weight.detach().t().contiguous()
        keep = [wc_t]
        w = native.DecoderWeights()
        w.project_context_t = wc_t.data_ptr()
        if self.env_name == "tsp":
            wp = self.context_embedding.W_placeholder.detach().contiguous()
            keep.append(wp)
            w.w_placeholder = wp.data_ptr()
        if self.is_dynamic_embedding:
            # [wk | wv | W_out^T wl]: the logit third folded like the logit key itself (module docstring, block 2)
            wdyn = self._dynamic_weights()
            keep.append(wdyn)
            w.dynamic_w = wdyn.data_ptr()
        w._keepalive = keep
        return w

    def forward(self, td: TensorDict, cached: FusedPrecomputedCache, num_starts: int = 0):
        """am/decoder.py:156-193 -> (logits [B_traj, N] raw, mask [B_traj, N]), one kernel.
        Multistart trajectories (flat index s*B+b) read instance b's cache in-kernel, so no
        unbatchify / rearrange round trip is needed."""
        mask = td["action_mask"]
        if not mask.is_contiguous():
            mask = mask.contiguous()
        B_traj, N = mask.shape
        B_inst = cached.node_embeddings.shape[0]
        w = self._step_weights()
        cur = td["current_node"].reshape(-1).contiguous()
        if self.env_name == "tsp":
            logits = native.pointer_logits(
                "tsp", w, cached.node_embeddings.contiguous(), cached.graph_context_or_none, cached.glimpse_key,
                cached.glimpse_val, cached.logit_key_folded, mask, td["first_node"].reshape(-1).contiguous(), cur,
                td["i"].reshape(-1).contiguous(), None, None, B_traj, B_inst, N)
        else:
            if self.is_dynamic_embedding:  # dynamic.py:71-73: the depot entry of the feature is forced to 0
                feat = td["demand_with_depot"].reshape(B_traj, N).clone()
                feat[:, 0] = 0
                w._keepalive.append(feat)
                w.dynamic_feature = feat.data_ptr()
            if self.env_name == "op":  # OPContext (context.py:201-213): [h_cur ; max_length[..., 0] - tour_length]
                spent, budget = td["tour_length"].reshape(-1).contiguous(), td["max_length"][..., 0].reshape(-1).contiguous()
            elif self.env_name == "pctsp":  # PCTSPContext (context.py:184-198): clamp(prize_required - collected, min=0)
                budget = td["prize_required"].reshape(-1).contiguous()
                spent = torch.minimum(td["cur_total_prize"].reshape(-1), budget).contiguous()
            else:                      # VRPContext (context.py:137-149): [h_cur ; vehicle_capacity - used_capacity]
                spent, budget = td["used_capacity"].reshape(-1).contiguous(), td["vehicle_capacity"].reshape(-1).contiguous()
            logits = native.pointer_logits(
                self.env_name, w, cached.node_embeddings.contiguous(), cached.graph_context_or_none, cached.glimpse_key,
                cached.glimpse_val, cached.logit_key_folded, mask, None, cur, None, spent, budget, B_traj, B_inst, N)
        return logits, mask
