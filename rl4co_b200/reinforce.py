"""REINFORCE / POMO glue around the fused rollout (SURVEY.md section 8f-2).

  REINFORCE.shared_step / calculate_loss   rl4co/models/rl/reinforce/reinforce.py:59-111
  baselines (no / shared / mean / exponential / rollout)   rl4co/models/rl/reinforce/baselines.py:48-248
  POMO.shared_step (augmentation x multistart, max over starts / augs, best tours)   rl4co/models/zoo/pomo/model.py:88-143
  Evaluate decoding (teacher forcing)      rl4co/utils/decoding.py:448-461, constructive/base.py:202-203

Training needs d(log-likelihood)/d(theta).  The fused rollout kernel is forward-only, so a
training step is:  (1) sample actions with the persistent kernel under no_grad;  (2) recompute the
log-likelihood of exactly those actions with `evaluate_log_likelihood` -- a *vectorised*
teacher-forced pass in differentiable PyTorch ops (all T decode steps of the whole batch in one
masked attention call instead of the reference's T-iteration Python loop);  (3) REINFORCE loss.
"""

from __future__ import annotations

import copy
import math

import torch
import torch.nn.functional as F

from . import native
from .distributed import global_mean_baseline, sync_gradients
from .ops import StateAugmentation, batchify, gather_by_index, unbatchify
from .tensordict import TensorDict

E = native.EMBED_DIM


# ------------------------------------------------------------------------ teacher-forced replay
def replay_states(env_name: str, td: TensorDict, actions: torch.Tensor):
    """Vectorised replay of the MDP along given actions [B,T]: returns (mask [B,T,N] bool,
    cur [B,T] node before step t, first [B,T] (tsp), used [B,T] capacity before step t (cvrp)).
    Restates tsp/env.py:60-86 and cvrp/env.py:66-136 without a time loop."""
    B, T = actions.shape
    N = td["locs"].shape[-2]
    dev = actions.device
    # visited strictly before step t, as bool: scatter a one-hot and take a running max along T (an int64
    # F.one_hot + int64 cumsum is 16 bytes per (trajectory, step, node): 8 GB for POMO TSP-100 at B = 512)
    onehot = torch.zeros(B, T, N, dtype=torch.uint8, device=dev).scatter_(2, actions.unsqueeze(-1), 1)
    visited_before = torch.cat([torch.zeros(B, 1, N, dtype=torch.uint8, device=dev),
                                onehot[:, :-1].cummax(1)[0]], 1).bool()
    prev = torch.cat([torch.zeros(B, 1, dtype=actions.dtype, device=dev), actions[:, :-1]], 1)
    if env_name == "tsp":
        mask = ~visited_before
        first = actions[:, :1].expand(B, T)
        return mask, prev, first, None
    demand = td["demand"]                                           # [B,N-1]
    cap = td["vehicle_capacity"].reshape(B, 1)
    dem_n = torch.cat([torch.zeros(B, 1, device=dev), demand], 1)   # node-indexed, depot 0
    # prefix sums in float64: the difference of two fp32 prefix sums of magnitude ~10 would be off by
    # more than the 1e-5 capacity slack on exact fits (the env accumulates the *current route* only)
    d_t = dem_n.double().gather(1, actions)                         # demand served at step t
    c = d_t.cumsum(1)                                               # non-decreasing
    c_prev = torch.cat([torch.zeros(B, 1, dtype=torch.float64, device=dev), c[:, :-1]], 1)
    at_depot = torch.cat([torch.ones(B, 1, dtype=torch.bool, device=dev), actions[:, :-1] == 0], 1)
    base = torch.where(at_depot, c_prev, torch.zeros_like(c_prev)).cummax(1)[0]
    used = (c_prev - base).float()                                  # used capacity before step t
    exceeds = (dem_n[:, None, 1:] + used[..., None]) > (cap[:, None] + 1e-5)
    mask_loc = visited_before[..., 1:] | exceeds
    mask_depot = (prev == 0)[..., None] & ((~mask_loc).sum(-1, keepdim=True) > 0)
    return ~torch.cat([mask_depot, mask_loc], -1), prev, None, used


def _running_total_before(step_values: torch.Tensor) -> torch.Tensor:
    """[B,T] per-step increments -> [B,T] totals BEFORE each step, accumulated one step after the other in fp32 exactly
    like the env's own `total = total + increment` (a parallel scan rounds differently, and the op length test below
    compares the total against a bound)."""
    total = torch.zeros_like(step_values[:, 0])
    cols = []
    for t in range(step_values.shape[1]):
        cols.append(total)
        total = total + step_values[:, t]
    return torch.stack(cols, 1)


def replay_budget_states(env_name: str, td: TensorDict, actions: torch.Tensor):
    """Replay of the orienteering / prize-collecting MDPs along given actions [B,T]: returns (mask [B,T,N] bool,
    cur [B,T] node before step t, state [B,T] = the scalar the context embedding appends to h_cur before step t:
    op `max_length[0] - tour_length` (context.py:201-213), pctsp `clamp(prize_required - cur_total_prize, 0)`
    (context.py:184-198)).  Restates op/env.py:72-155 and pctsp/env.py:62-151; the only time loop is the running
    fp32 total of one scalar per instance.  Columns after an instance is done hold depot actions whose mask leaves
    the depot alone (log-probability 0), as in the reference's padded decode loop."""
    B, T = actions.shape
    locs = td["locs"]
    N = locs.shape[-2]
    dev = actions.device
    onehot = torch.zeros(B, T, N, dtype=torch.uint8, device=dev).scatter_(2, actions.unsqueeze(-1), 1)
    visited_before = torch.cat([torch.zeros(B, 1, N, dtype=torch.uint8, device=dev),
                                onehot[:, :-1].cummax(1)[0]], 1).bool()
    prev = torch.cat([torch.zeros(B, 1, dtype=actions.dtype, device=dev), actions[:, :-1]], 1)
    closed = visited_before[..., 0:1]                # the depot was chosen before step t: no customer may follow
    if env_name == "op":
        pts = gather_by_index(locs, actions)                                           # [B,T,2]
        leg = (pts - torch.cat([locs[:, 0:1], pts[:, :-1]], 1)).norm(p=2, dim=-1)      # op/env.py:80-84
        length_before = _running_total_before(leg)
        # |locs[n] - locs[cur]| for every n: row `cur` of the pairwise matrix (the sign of the difference is squared away)
        pair = (locs[:, :, None, :] - locs[:, None, :, :]).norm(p=2, dim=-1)           # [B,N,N]
        dist = pair.gather(1, prev[..., None].expand(B, T, N))
        exceeds = length_before[..., None] + dist > td["max_length"][:, None, :]       # op/env.py:146-149
        mask = ~(visited_before | closed | exceeds)
        mask[..., 0] = True
        # the actions come from a rollout that found them feasible; should a length sum ever round differently here
        # than in the kernel that produced them, the chosen node must not end up with log-probability -inf
        mask.scatter_(2, actions.unsqueeze(-1), True)
        return mask, prev, td["max_length"][:, 0:1] - length_before
    if env_name == "pctsp":
        prize_before = _running_total_before(td["real_prize"].gather(1, actions))      # pctsp/env.py:66-68
        customers_left = visited_before[..., 1:].sum(-1) < N - 1
        depot_ok = ~((prize_before < 1.0) & customers_left)                            # pctsp/env.py:147-149
        mask = torch.cat([depot_ok[..., None], ~(visited_before | closed)[..., 1:]], -1)
        return mask, prev, torch.clamp(td["prize_required"][:, None] - prize_before, min=0)
    raise NotImplementedError(env_name)


def replay_split_delivery_states(td: TensorDict, actions: torch.Tensor):
    """Replay of the split-delivery MDP (sdvrp/env.py:55-116) along given actions [B,T]: returns (mask [B,T,N] bool,
    cur [B,T], used [B,T] capacity before step t, remaining [B,T,N] node-indexed demand before step t).  What a visit
    delivers depends on what every earlier visit left, so this one is a time loop of [B]-sized gathers / scatters in
    the env's own fp32 arithmetic."""
    B, T = actions.shape
    dev = actions.device
    cap = td["vehicle_capacity"].reshape(B)
    remaining = torch.cat([torch.zeros(B, 1, device=dev), td["demand"]], 1)
    used = torch.zeros(B, device=dev)
    rem_cols, used_cols = [], []
    for t in range(T):
        rem_cols.append(remaining)
        used_cols.append(used)
        a = actions[:, t:t + 1]
        delivered = torch.min(remaining.gather(1, a).squeeze(1), cap - used)
        used = (used + delivered) * (a.squeeze(1) != 0).float()
        remaining = remaining.scatter_add(1, a, -delivered[:, None])
    remaining, used = torch.stack(rem_cols, 1), torch.stack(used_cols, 1)
    prev = torch.cat([torch.zeros(B, 1, dtype=actions.dtype, device=dev), actions[:, :-1]], 1)
    mask_loc = (remaining[..., 1:] == 0) | (used >= cap[:, None])[..., None]           # sdvrp/env.py:110-116
    mask_depot = (prev == 0) & ((~mask_loc).sum(-1) > 0)
    return ~torch.cat([mask_depot[..., None], mask_loc], -1), prev, used, remaining


REPLAY_KEYS = ("locs", "demand", "vehicle_capacity", "max_length", "real_prize", "prize_required")


def evaluate_log_likelihood(policy, td: TensorDict, env, actions: torch.Tensor, hidden=None,
                            return_sum: bool = True, temperature=None, tanh_clipping=None,
                            forced_first=None, strategy=None) -> torch.Tensor:
    """log pi(actions | instance) with autograd, equal (<= fp32 round-off) to what the rollout
    kernel reported for the same actions.  `td` is the reset state (multistart: the [B] state,
    actions [S*B, T] in the reference's start-major order).

    A PolyNet decoder (`rl4co_b200.polynet`) applies its poly layer to the glimpse of row j = s * B + b with strategy
    s % k, as its rollout does; `strategy` [S*B] (int64, start-major like the rows) replays row j with strategy[j]
    instead, so that any row of a rollout can be replayed on its own."""
    env_name = env.name
    if env_name not in ("tsp", "cvrp", "sdvrp", "op", "pctsp"):
        raise NotImplementedError(f"the vectorised teacher-forced pass replays tsp / cvrp / sdvrp / op / pctsp state only "
                                  f"(got {env_name!r}); use policy(td, env, actions=...) on the stepping kernels")
    dec = policy.decoder
    if hidden is None:
        hidden, _ = policy.encoder(td)
    B, N, _ = hidden.shape
    S = actions.shape[0] // B
    T = actions.shape[1]
    cached = dec._precompute_cache(hidden)
    K, V = cached.glimpse_key, cached.glimpse_val
    L = cached.logit_key
    g = cached.graph_context if isinstance(cached.graph_context, torch.Tensor) else None
    # trajectories of one instance become S*T queries against that instance's K / V / L (no copies)
    acts = actions.view(S, B, T).permute(1, 0, 2).reshape(B * S, T) if S > 1 else actions   # instance-major
    tdx = td
    if S > 1:
        tdx = TensorDict({k: td[k].repeat_interleave(S, 0) for k in REPLAY_KEYS if k in td.keys()}, batch_size=[B * S])
    Q = S * T
    remaining = None
    if env_name in ("op", "pctsp"):
        mask, prev, state = replay_budget_states(env_name, tdx, acts)
    elif env_name == "sdvrp":
        mask, prev, used, remaining = replay_split_delivery_states(tdx, acts)
        remaining = remaining.reshape(B, Q, N).clone()
        remaining[..., 0] = 0                                      # dynamic.py:71-73: the depot's feature is forced to 0
    else:
        mask, prev, first, used = replay_states(env_name, tdx, acts)
    mask = mask.view(B, Q, N)
    prev_q = prev.reshape(B, Q)
    wc = dec.context_embedding.project_context.weight
    if forced_first is None:
        forced_first = S > 1  # multistart: step 0 is the forced start node with log-prob 0
    if env_name == "tsp":
        ctx = torch.cat([gather_by_index(hidden, first.reshape(B, Q)), gather_by_index(hidden, prev_q)], -1)  # [B,Q,2E]
        q = F.linear(ctx, wc)
        if not forced_first:
            q0 = F.linear(dec.context_embedding.W_placeholder, wc)
            q = torch.cat([q0.expand(B, 1, E), q[:, 1:]], 1)
    else:
        if env_name in ("cvrp", "sdvrp"):
            state = tdx["vehicle_capacity"].reshape(B * S, 1) - used
        q = F.linear(torch.cat([gather_by_index(hidden, prev_q), state.reshape(B, Q, 1)], -1), wc)               # [B,Q,E]
    if g is not None:
        q = q + g[:, None, :]
    H = native.NUM_HEADS

    def heads(x):
        return x.view(x.shape[0], x.shape[1], H, -1).transpose(1, 2)

    import os

    if remaining is not None:
        # sdvrp: keys / values / logit keys of step t are the cached ones plus remaining_demand_t[n] * w (a Linear(1 -> 3E),
        # dynamic.py:60-78, am/decoder.py:142-154).  Instead of T copies of K / V / L the rank-one term is applied where it
        # lands: a per-(step, head) multiple of the remaining demand on the scores, the probability-weighted demand times
        # w_v on the head outputs, and (glimpse . w_l) * demand on the logits
        wk, wv, wl = dec.dynamic_embedding.projection.weight[:, 0].chunk(3)
        qh, d = heads(q), remaining[:, None]                                                     # [B,H,Q,16], [B,1,Q,N]
        scores = qh @ heads(K).transpose(-1, -2) + (qh * wk.view(1, H, 1, -1)).sum(-1, keepdim=True) * d
        p = torch.softmax((scores / math.sqrt(E // H)).masked_fill(~mask[:, None], float("-inf")), -1)
        o = p @ heads(V) + (p * d).sum(-1, keepdim=True) * wv.view(1, H, 1, -1)
        o = o.transpose(1, 2).reshape(B, Q, E)
    elif q.is_cuda and N <= 128 and q.dtype == torch.float32 and os.environ.get("CO_TRAIN_ATTN", "fused") != "sdpa":
        # the T (x S) decode steps of an instance are independent queries against its cached K / V: hand-written
        # masked attention forward / backward (co_attn_fwd / co_attn_bwd) on the cache's column views, no copies
        from . import attention_train

        o = attention_train.attention(q.contiguous(), K, V, mask)
    else:
        o = F.scaled_dot_product_attention(heads(q), heads(K), heads(V), attn_mask=mask[:, None])
        o = o.transpose(1, 2).reshape(B, Q, E)
    glimpse = dec.pointer.project_out(o)
    if hasattr(dec.pointer, "poly"):  # PolyNet: queries are instance-major [B, S * T], one strategy per row s
        if strategy is None:
            strat = (torch.arange(S, device=glimpse.device) % dec.pointer.k).repeat_interleave(T)[None]  # [1, Q]
        else:
            if tuple(strategy.shape) != (S * B,):
                raise ValueError(f"strategy: expected [{S * B}] (one per row), got {tuple(strategy.shape)}")
            strat = strategy.to(glimpse.device).view(S, B).t().repeat_interleave(T, dim=1)          # [B, Q]
        glimpse = dec.pointer.poly(glimpse, strat)
    elif strategy is not None:
        raise ValueError("strategy is only defined for a PolyNet decoder")
    logits = torch.bmm(glimpse, L.transpose(1, 2))
    if remaining is not None:
        logits = logits + (glimpse * wl).sum(-1, keepdim=True) * remaining
    logits = logits / math.sqrt(E)
    clip = policy.tanh_clipping if tanh_clipping is None else tanh_clipping
    if clip > 0:
        logits = torch.tanh(logits) * clip
    logits = logits.masked_fill(~mask, float("-inf")) / (policy.temperature if temperature is None else temperature)
    logp = F.log_softmax(logits, -1).gather(-1, acts.reshape(B, Q)[..., None]).squeeze(-1).view(B * S, T)
    if forced_first:
        logp = torch.cat([torch.zeros_like(logp[:, :1]), logp[:, 1:]], 1)
    if S > 1:
        logp = logp.view(B, S, T).permute(1, 0, 2).reshape(S * B, T)
    return logp.sum(1) if return_sum else logp


# ------------------------------------------------------------------------ baselines
class NoBaseline:
    """baselines.py:48-52"""

    def eval(self, td, reward, env=None):
        return 0, 0

    def setup(self, *a, **k):
        pass

    def epoch_callback(self, *a, **k):
        pass


class SharedBaseline(NoBaseline):
    """baselines.py:55-61: mean over the starts of each instance (POMO)."""

    def eval(self, td, reward, env=None, on_dim=1):
        return reward.mean(dim=on_dim, keepdims=True), 0


class MeanBaseline(NoBaseline):
    """baselines.py:75-81 with the mean taken over the GLOBAL batch: {sum, count} in f64 through
    co_reward_stats + one NCCL all-reduce (the reference's DDP uses per-rank means)."""

    def eval(self, td, reward, env=None):
        return global_mean_baseline(reward.detach()), 0


class ExponentialBaseline(NoBaseline):
    """baselines.py:64-84"""

    def __init__(self, beta=0.8):
        self.beta, self.v = beta, None

    def eval(self, td, reward, env=None):
        m = global_mean_baseline(reward.detach())
        self.v = m if self.v is None else self.beta * self.v + (1.0 - self.beta) * m
        return self.v.detach(), 0


class RolloutBaseline(NoBaseline):
    """baselines.py:160-248: greedy rollout of a frozen copy of the policy; at the end of every epoch the current
    policy challenges it on a fixed evaluation dataset and replaces it when it is better by a one-sided paired
    t-test at level `bl_alpha` (`epoch_callback`)."""

    def __init__(self, bl_alpha: float = 0.05, **kw):
        self.bl_alpha = bl_alpha
        self.policy = None
        self.dataset = None
        self.bl_vals = None
        self.mean = None

    def setup(self, policy, env=None, batch_size=64, device=None, dataset_size=None, dataset=None, **kw):
        self._update_policy(policy, env, batch_size, device, dataset_size, dataset)

    def update(self, policy):
        """Swap the frozen copy without touching the evaluation dataset."""
        self.policy = copy.deepcopy(policy).eval()
        for p in self.policy.parameters():
            p.requires_grad_(False)

    def _update_policy(self, policy, env=None, batch_size=64, device=None, dataset_size=None, dataset=None):
        """baselines.py:174-189"""
        self.update(policy)
        if device is not None:
            self.policy = self.policy.to(device)
        if env is None:
            return
        if dataset is not None:
            self.dataset = dataset
        elif self.dataset is None and dataset_size:
            self.dataset = env.dataset(batch_size=[dataset_size])
        if self.dataset is not None:
            dev = device if device is not None else next(self.policy.parameters()).device
            self.bl_vals = self.rollout(self.policy, env, batch_size, dev, self.dataset).cpu().numpy()
            self.mean = self.bl_vals.mean()

    def eval(self, td, reward, env=None):
        with torch.inference_mode():
            out = self.policy(td, env, phase="test", decode_type="greedy")
        return out["reward"].clone(), 0

    def epoch_callback(self, policy, env, batch_size=64, device=None, epoch=None, dataset_size=None, **kw):
        """baselines.py:200-217: replace the baseline policy if the candidate is significantly better."""
        from scipy.stats import ttest_rel

        dev = device if device is not None else next(policy.parameters()).device
        candidate_vals = self.rollout(policy, env, batch_size, dev).cpu().numpy()
        candidate_mean = candidate_vals.mean()
        updated = False
        if candidate_mean - self.mean > 0:
            t, p = ttest_rel(-candidate_vals, -self.bl_vals)  # costs: inverse logic
            p_val = p / 2  # one-sided
            assert t < 0, "T-statistic should be negative"
            if p_val < self.bl_alpha:
                self._update_policy(policy, env, batch_size, dev, dataset_size)
                updated = True
        return updated

    def rollout(self, policy, env, batch_size=64, device=None, dataset=None):
        """baselines.py:219-237: greedy rewards of `policy` over a dataset, batch by batch."""
        from torch.utils.data import DataLoader

        dataset = self.dataset if dataset is None else dataset
        was_training = policy.training
        policy.eval()
        rewards = []
        with torch.inference_mode():
            for batch in DataLoader(dataset, batch_size=batch_size, collate_fn=dataset.collate_fn):
                td = env.reset(batch.to(device) if device is not None else batch)
                rewards.append(policy(td, env, phase="test", decode_type="greedy")["reward"])
        if was_training:
            policy.train()
        return torch.cat(rewards, 0)


class WarmupBaseline(NoBaseline):
    """baselines.py:91-134: convex combination of an exponential baseline and the wrapped baseline during the first
    `n_epochs` epochs (alpha = (epoch + 1) / n_epochs after each epoch)."""

    def __init__(self, baseline, n_epochs=1, warmup_exp_beta=0.8, **kw):
        assert n_epochs > 0, "n_epochs to warmup must be positive"
        self.baseline = baseline
        self.warmup_baseline = ExponentialBaseline(warmup_exp_beta)
        self.alpha = 0
        self.n_epochs = n_epochs

    def setup(self, *a, **k):
        self.baseline.setup(*a, **k)

    def eval(self, td, reward, env=None):
        if self.alpha == 1:
            return self.baseline.eval(td, reward, env)
        if self.alpha == 0:
            return self.warmup_baseline.eval(td, reward, env)
        v_b, l_b = self.baseline.eval(td, reward, env)
        v_wb, l_wb = self.warmup_baseline.eval(td, reward, env)
        return self.alpha * v_b + (1 - self.alpha) * v_wb, self.alpha * l_b + (1 - self.alpha) * l_wb

    def epoch_callback(self, *a, **kw):
        self.baseline.epoch_callback(*a, **kw)
        if kw["epoch"] < self.n_epochs:
            self.alpha = (kw["epoch"] + 1) / float(self.n_epochs)


class CriticNetwork(torch.nn.Module):
    """models/rl/common/critic.py:11-63: encoder + value head (Linear E->512, ReLU, Linear 512->1), mean over nodes."""

    def __init__(self, encoder, value_head=None, embed_dim: int = 128, hidden_dim: int = 512):
        super().__init__()
        self.encoder = encoder
        if value_head is None:
            value_head = torch.nn.Sequential(torch.nn.Linear(embed_dim, hidden_dim), torch.nn.ReLU(),
                                             torch.nn.Linear(hidden_dim, 1))
        self.value_head = value_head

    def forward(self, x, hidden=None):
        h, _ = self.encoder(x)
        return self.value_head(h).mean(1)


def create_critic_from_actor(policy, backbone: str = "encoder", **critic_kwargs):
    """models/rl/common/critic.py:66-75"""
    encoder = getattr(policy, backbone, None)
    if encoder is None:
        raise ValueError(f"CriticBaseline requires a backbone in the policy network: {backbone}")
    return CriticNetwork(copy.deepcopy(encoder), **critic_kwargs).to(next(policy.parameters()).device)


class CriticBaseline(NoBaseline):
    """baselines.py:137-157: a critic network as baseline; its loss is mse(v, reward)."""

    def __init__(self, critic=None, **unused_kw):
        self.critic = critic

    def setup(self, policy, env=None, **kwargs):
        if self.critic is None:
            self.critic = create_critic_from_actor(policy)

    def eval(self, x, c, env=None):
        v = self.critic(x).squeeze(-1)
        return v.detach(), F.mse_loss(v, c.detach())


def get_reinforce_baseline(name, **kw):
    """baselines.py:251-287 (incl. the `warmup` wrapper: `with_warmup` / `n_epochs` / `exp_beta`)."""
    reg = {"no": NoBaseline, "shared": SharedBaseline, "mean": MeanBaseline, "exponential": ExponentialBaseline,
           "rollout_only": RolloutBaseline, "critic": CriticBaseline}
    if name == "warmup":
        inner = kw.get("baseline", "rollout")
        if isinstance(inner, str):
            inner = get_reinforce_baseline(inner, **{k: v for k, v in kw.items() if k != "baseline"})
        return WarmupBaseline(inner, n_epochs=kw.get("n_epochs", 1), warmup_exp_beta=kw.get("warmup_exp_beta", 0.8))
    if name == "rollout":  # the reference's "rollout" = one warm-up epoch of exponential baseline, then greedy rollout
        return WarmupBaseline(RolloutBaseline(bl_alpha=kw.get("bl_alpha", 0.05)), kw.get("n_epochs", 1),
                              kw.get("exp_beta", 0.8))
    if name not in reg:
        raise ValueError(f"Unknown baseline {name}. Available baselines: {list(reg) + ['rollout', 'warmup']}")
    return reg[name](**kw)


# ------------------------------------------------------------------------ REINFORCE / POMO steps
def calculate_loss(reward, log_likelihood, bl_val, bl_loss=0):
    """reinforce.py:96-111"""
    advantage = reward - bl_val
    reinforce_loss = -(advantage * log_likelihood).mean()
    return reinforce_loss + bl_loss, reinforce_loss


def _bn_modules(module):
    return [m for m in module.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)]


def reinforce_step(policy, env, td, baseline, optimizer=None, decode_type="sampling", seed=None, max_grad_norm=1.0,
                   micro_batch=None, matmul_precision=None):
    """One REINFORCE training step (reinforce.py:59-111): fused sampling rollout (no grad) ->
    differentiable log-likelihood of the sampled actions -> loss -> backward -> gradient averaging over ranks
    -> clip -> optimizer.

    `micro_batch`: batches larger than this are processed in chunks (bounded activation memory: the
    differentiable pass of 65 536 CVRP-100 instances does not fit one GPU): phase 1 samples every chunk without
    a graph, the baseline is evaluated once on the WHOLE batch (global mean / all-reduce), phase 2 recomputes
    each chunk's encoder + log-likelihood with a graph and accumulates its share of the loss gradient.  Train-mode
    BatchNorm statistics are per chunk (what per-rank statistics are under the reference's DDP); phase 1 freezes
    the running statistics so that they are updated once per chunk per step.
    `matmul_precision`: e.g. "medium" = the reference trainer's float32_matmul_precision
    (rl4co/utils/trainer.py:57,89-90) for the autograd GEMMs; None leaves the global setting alone."""
    policy.train()
    prev_prec = None
    if matmul_precision is not None:
        prev_prec = torch.get_float32_matmul_precision()
        torch.set_float32_matmul_precision(matmul_precision)
    ev0 = ev1 = None
    try:
        B = td.batch_size[0]
        kw = {"seed": seed} if seed is not None else {}
        if micro_batch is None or B <= micro_batch:
            enc = policy.encoder(td)  # ONE differentiable encoder pass (train-mode norms) shared by both stages
            with torch.no_grad():
                if td["locs"].is_cuda:
                    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    ev0.record()
                out = policy(td, env, phase="train", decode_type=decode_type, encoder_output=(enc[0].detach(), enc[1]), **kw)
                if ev1 is not None:
                    ev1.record()
            ll = evaluate_log_likelihood(policy, td, env, out["actions"], hidden=enc[0])
            bl_val, bl_loss = baseline.eval(td, out["reward"], env)
            loss, rl = calculate_loss(out["reward"], ll, bl_val, bl_loss)
            reward, actions, chunks = out["reward"], out["actions"], 1
            if optimizer is not None:
                optimizer.zero_grad(set_to_none=True)
                loss.backward()
        else:
            spans = [(lo, min(lo + micro_batch, B)) for lo in range(0, B, micro_batch)]
            chunks = len(spans)
            bns = _bn_modules(policy)
            saved = [m.momentum for m in bns]
            for m in bns:
                m.momentum = 0.0  # phase 1 must not move the running statistics (phase 2 does, once)
            outs = []
            try:
                with torch.no_grad():
                    if td["locs"].is_cuda:
                        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        ev0.record()
                    for i, (lo, hi) in enumerate(spans):
                        kwi = {"seed": seed * 1_000_003 + i} if seed is not None else {}
                        outs.append(policy(td[lo:hi], env, phase="train", decode_type=decode_type, **kwi))
                    if ev1 is not None:
                        ev1.record()
            finally:
                for m, mom in zip(bns, saved):
                    m.momentum = mom
            T = max(o["actions"].shape[1] for o in outs)
            reward = torch.cat([o["reward"] for o in outs])
            actions = torch.cat([F.pad(o["actions"], (0, T - o["actions"].shape[1])) for o in outs])
            bl_val, bl_loss = baseline.eval(td, reward, env)
            if optimizer is not None:
                optimizer.zero_grad(set_to_none=True)
            ll_parts, loss = [], torch.zeros((), device=reward.device)
            for (lo, hi), o in zip(spans, outs):
                tdc = td[lo:hi]
                ll_c = evaluate_log_likelihood(policy, tdc, env, o["actions"])
                bl_c = bl_val[lo:hi] if isinstance(bl_val, torch.Tensor) and bl_val.dim() > 0 and bl_val.shape[0] == B else bl_val
                part = -((o["reward"] - bl_c) * ll_c).sum() / B   # this chunk's share of the batch mean
                if optimizer is not None:
                    part.backward()
                loss = loss + part.detach()
                ll_parts.append(ll_c.detach())
            ll = torch.cat(ll_parts)
            rl = loss
            loss = loss + (bl_loss if not isinstance(bl_loss, torch.Tensor) else bl_loss.detach())
        if optimizer is not None:
            sync_gradients(policy.parameters())  # DDP-equivalent gradient averaging (no-op on one rank)
            if max_grad_norm:
                torch.nn.utils.clip_grad_norm_(policy.parameters(), max_grad_norm)
            optimizer.step()
    finally:
        if prev_prec is not None:
            torch.set_float32_matmul_precision(prev_prec)
    res = {"loss": loss.detach(), "reinforce_loss": rl.detach(), "reward": reward, "log_likelihood": ll.detach(),
           "bl_val": bl_val, "actions": actions, "chunks": chunks}
    if ev1 is not None:
        res["rollout_events"] = (ev0, ev1)
    return res


def pomo_step(policy, env, td, num_augment=8, num_starts=None, phase="test", optimizer=None, augment_fn="dihedral8",
              first_aug_identity=True, feats=None):
    """POMO.shared_step (pomo/model.py:88-143): optional augmentation (val/test; `augment_fn`, `first_aug_identity`
    and `feats` as POMO passes them to StateAugmentation), multistart rollout, shared baseline over starts; returns
    max rewards over starts / augs and, on val/test, the tours behind them: `best_multistart_actions` [B, aug, T]
    ([B, T] without augmentation) and `best_aug_actions` [B, T]."""
    B = td.batch_size[0]
    n_aug = num_augment if phase != "train" else 0
    n_start = env.get_num_starts(td) if num_starts is None else num_starts
    if n_aug > 1:
        td = StateAugmentation(num_augment=n_aug, augment_fn=augment_fn, first_aug_identity=first_aug_identity,
                               feats=feats)(td)
    if phase == "train":
        policy.train()
        enc = policy.encoder(td)
        with torch.no_grad():
            out = policy(td, env, phase="train", decode_type="multistart_sampling", num_starts=n_start,
                         encoder_output=(enc[0].detach(), enc[1]))
        ll = evaluate_log_likelihood(policy, td, env, out["actions"], hidden=enc[0])
        reward = unbatchify(out["reward"], n_start)                       # [B, S]
        bl_val, _ = SharedBaseline().eval(td, reward)
        loss, _ = calculate_loss(reward, unbatchify(ll, n_start), bl_val)
        if optimizer is not None:
            optimizer.zero_grad(set_to_none=True)
            loss.backward()
            sync_gradients(policy.parameters())
            optimizer.step()
        return {"loss": loss.detach(), "reward": reward, "max_reward": reward.max(-1)[0]}
    with torch.inference_mode():
        out = policy(td, env, phase=phase, decode_type="multistart_greedy", num_starts=n_start)
    shape = (n_aug, n_start) if n_aug > 1 else (n_start,)
    reward = unbatchify(out["reward"], shape)                               # [B, aug, start] | [B, start]
    max_reward, max_idxs = reward.max(-1)
    best_ms = gather_by_index(unbatchify(out["actions"], shape), max_idxs, dim=max_idxs.dim())  # [B, aug, T] | [B, T]
    res = {"reward": reward, "max_reward": max_reward, "actions": out["actions"], "best_multistart_actions": best_ms}
    if n_aug > 1:
        res["max_aug_reward"], aug_idxs = max_reward.max(1)
        res["best_aug_actions"] = gather_by_index(best_ms, aug_idxs)             # [B, T]
    return res
