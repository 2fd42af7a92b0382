"""TEST INFRASTRUCTURE ONLY -- CPU restatement of rl4co's AM rollout hot path.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this module, and there only as the *checker*
(or the timed CPU baseline), never as part of the product path.  The product
(``rl4co_b200``) must not import anything from ``oracle/``.

What this is: a plain-PyTorch (fp32, CPU or any device) restatement, without
TensorDict/torchrl/lightning, of the reference functions listed in SURVEY.md
section 8a.  It uses the *same* library calls the reference uses
(``F.scaled_dot_product_attention``, ``F.linear``, ``torch.bmm``,
``F.log_softmax``, ``argmax``) in the *same* order so that on CPU it reproduces
the reference bit-for-bit on actions/masks and to fp32 round-off on
rewards/log-probs.

Pinning status: the reference's own tests hold **no** golden values for this
path (SURVEY.md section 4 / 8c: shapes only).  The restatement is therefore pinned
against outputs of the reference itself: ``tests/golden/make_golden.py`` runs the
unmodified reference files (via ``oracle/ref_standin.py``) in the build container
and commits the vectors under ``tests/golden/``; ``tests/test_oracle_golden.py``
checks this module against them everywhere, and
``tests/test_oracle_vs_reference.py`` re-runs the live reference where
``/root/reference`` exists.

State is a plain ``dict[str, Tensor]`` with exactly the reference's TensorDict keys,
dtypes and shapes (SURVEY.md section 8b).  Weights are a ``dict`` keyed like a
reference ``AttentionModelPolicy.state_dict()``.
"""

from __future__ import annotations

import math

import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------- ops
# reference: rl4co/utils/ops.py


def gather_by_index(src, idx, dim=1, squeeze=True):
    """rl4co/utils/ops.py:54-66"""
    expanded_shape = list(src.shape)
    expanded_shape[dim] = -1
    idx = idx.view(idx.shape + (1,) * (src.dim() - idx.dim())).expand(expanded_shape)
    squeeze = idx.size(dim) == 1 and squeeze
    return src.gather(dim, idx).squeeze(dim) if squeeze else src.gather(dim, idx)


def batchify(x, repeats: int):
    """rl4co/utils/ops.py:10-29 -- start-major repeat: flat index = r * B + b."""
    if repeats <= 0:
        return x
    if isinstance(x, dict):
        return {k: batchify(v, repeats) for k, v in x.items()}
    s = x.shape
    return x.expand(repeats, *s).contiguous().view(s[0] * repeats, *s[1:])


def unbatchify(x, repeats: int):
    """rl4co/utils/ops.py:32-51 -- '(r b) ... -> b r ...'"""
    if repeats <= 0:
        return x
    if isinstance(x, dict):
        return {k: unbatchify(v, repeats) for k, v in x.items()}
    s = x.shape
    return x.view(repeats, s[0] // repeats, *s[1:]).permute(1, 0, *range(2, len(s) + 1))


def unbatchify_multi(x, shape):
    """rl4co/utils/ops.py:45-51 with a tuple shape (e.g. (n_aug, n_start))."""
    for s in reversed(list(shape)):
        x = unbatchify(x, s)
    return x


def get_tour_length(ordered_locs):
    """rl4co/utils/ops.py:77-90 (get_distance + roll + sum)"""
    nxt = torch.roll(ordered_locs, -1, dims=-2)
    return (nxt - ordered_locs).norm(p=2, dim=-1).sum(-1)


DEPOT_ENVS = ("cvrp", "sdvrp", "op", "pctsp")


def get_num_starts(num_actions: int, env_name: str) -> int:
    """rl4co/utils/ops.py:115-125 (depot envs: the depot is not a start node)"""
    return num_actions - 1 if env_name in DEPOT_ENVS else num_actions


def select_start_nodes(batch: int, num_starts: int, num_loc: int, env_name: str, device=None):
    """rl4co/utils/ops.py:128-149. ``num_loc`` = generator.num_loc (customers for CVRP)."""
    sel = torch.arange(num_starts, device=device).repeat_interleave(batch) % num_loc
    return sel + 1 if env_name in DEPOT_ENVS else sel  # (op's resampling branch, ops.py:150-160, is not restated)


def dihedral_8_augmentation(xy):
    """rl4co/data/transforms.py:16-38 (aug-major: flat index = a * B + b)."""
    x, y = xy.split(1, dim=2)
    zs = [(x, y), (1 - x, y), (x, 1 - y), (1 - x, 1 - y), (y, x), (1 - y, x), (y, 1 - x), (1 - y, 1 - x)]
    return torch.cat([torch.cat(z, dim=2) for z in zs], dim=0)


# --------------------------------------------------------------------------- TSP env
# reference: rl4co/envs/routing/tsp/env.py


def tsp_reset(locs):
    """tsp/env.py:88-113 (+ torchrl fill of done [B,1], envs/common/base.py:135-143)"""
    B, N = locs.shape[0], locs.shape[-2]
    dev = locs.device
    cur = torch.zeros(B, dtype=torch.int64, device=dev)
    return {
        "locs": locs,
        "first_node": cur,
        "current_node": cur,
        "i": torch.zeros(B, 1, dtype=torch.int64, device=dev),
        "action_mask": torch.ones(B, N, dtype=torch.bool, device=dev),
        "reward": torch.zeros(B, 1, dtype=torch.float32),
        "done": torch.zeros(B, 1, dtype=torch.bool, device=dev),
    }


def tsp_step(state, action):
    """tsp/env.py:60-86"""
    st = dict(state)
    current_node = action
    first_node = current_node if st["i"].all() == 0 else st["first_node"]
    available = st["action_mask"].scatter(-1, current_node.unsqueeze(-1).expand_as(st["action_mask"]), 0)
    done = torch.sum(available, dim=-1) == 0
    st.update(
        first_node=first_node,
        current_node=current_node,
        i=st["i"] + 1,
        action_mask=available,
        reward=torch.zeros_like(done),
        done=done,
        action=action,
    )
    return st


def tsp_reward(locs, actions):
    """tsp/env.py:150-156"""
    return -get_tour_length(gather_by_index(locs, actions))


def tsp_check_solution(actions):
    """tsp/env.py:158-164"""
    ok = (torch.arange(actions.size(1)).view(1, -1).expand_as(actions) == actions.sort(1)[0]).all()
    assert ok, "Invalid tour"


# --------------------------------------------------------------------------- CVRP env
# reference: rl4co/envs/routing/cvrp/env.py


def cvrp_action_mask(st):
    """cvrp/env.py:126-136"""
    exceeds_cap = st["demand"] + st["used_capacity"] > st["vehicle_capacity"] + 1e-5
    mask_loc = st["visited"][..., 1:].to(exceeds_cap.dtype) | exceeds_cap
    mask_depot = (st["current_node"] == 0) & ((mask_loc == 0).int().sum(-1) > 0)[:, None]
    return ~torch.cat((mask_depot, mask_loc), -1)


def cvrp_reset(depot, locs, demand, vehicle_capacity: float = 1.0):
    """cvrp/env.py:98-124 (demand already divided by capacity, generator.py:136)"""
    B = locs.shape[0]
    dev = locs.device
    st = {
        "locs": torch.cat((depot[:, None, :], locs), -2),
        "demand": demand,
        "current_node": torch.zeros(B, 1, dtype=torch.long, device=dev),
        "used_capacity": torch.zeros(B, 1, device=dev),
        "vehicle_capacity": torch.full((B, 1), vehicle_capacity, device=dev),
        "visited": torch.zeros(B, locs.shape[-2] + 1, dtype=torch.uint8, device=dev),
    }
    st["action_mask"] = cvrp_action_mask(st)
    st["done"] = torch.zeros(B, 1, dtype=torch.bool, device=dev)
    return st


def cvrp_step(state, action):
    """cvrp/env.py:66-96"""
    st = dict(state)
    current_node = action[:, None]
    n_loc = st["demand"].size(-1)
    selected_demand = gather_by_index(st["demand"], torch.clamp(current_node - 1, 0, n_loc - 1), squeeze=False)
    used_capacity = (st["used_capacity"] + selected_demand) * (current_node != 0).float()
    visited = st["visited"].scatter(-1, current_node, 1)
    done = visited.sum(-1) == visited.size(-1)
    st.update(
        current_node=current_node,
        used_capacity=used_capacity,
        visited=visited,
        reward=torch.zeros_like(done),
        done=done,
        action=action,
    )
    st["action_mask"] = cvrp_action_mask(st)
    return st


def cvrp_reward(locs_with_depot, actions):
    """cvrp/env.py:138-147"""
    ordered = torch.cat([locs_with_depot[..., 0:1, :], gather_by_index(locs_with_depot, actions)], dim=1)
    return -get_tour_length(ordered)


def cvrp_check_solution(st, actions):
    """cvrp/env.py:149-177"""
    batch_size, graph_size = st["demand"].size()
    sorted_pi = actions.sort(1)[0]
    ok = (
        torch.arange(1, graph_size + 1).view(1, -1).expand(batch_size, graph_size) == sorted_pi[:, -graph_size:]
    ).all() and (sorted_pi[:, :-graph_size] == 0).all()
    assert ok, "Invalid tour"
    demand_with_depot = torch.cat((-st["vehicle_capacity"], st["demand"]), 1)
    d = demand_with_depot.gather(1, actions)
    used = torch.zeros_like(st["demand"][:, 0])
    for i in range(actions.size(1)):
        used = used + d[:, i]
        used[used < 0] = 0
        assert (used <= st["vehicle_capacity"][:, 0] + 1e-5).all(), "Used more than capacity"


# --------------------------------------------------------------------------- SDVRP env (sibling env, SURVEY 8f-4)
# reference: rl4co/envs/routing/sdvrp/env.py


def sdvrp_action_mask(st):
    """sdvrp/env.py:110-116"""
    mask_loc = (st["demand_with_depot"][..., 1:] == 0) | (st["used_capacity"] >= st["vehicle_capacity"])
    mask_depot = (st["current_node"] == 0).squeeze(-1) & ((mask_loc == 0).int().sum(-1) > 0)
    return ~torch.cat((mask_depot[..., None], mask_loc), -1)


def sdvrp_reset(depot, locs, demand, vehicle_capacity: float = 1.0):
    """sdvrp/env.py:84-108"""
    B = locs.shape[0]
    dev = locs.device
    st = {
        "locs": torch.cat((depot[:, None, :], locs), -2),
        "demand": demand,
        "demand_with_depot": torch.cat((torch.zeros_like(demand[..., 0:1]), demand), -1),
        "current_node": torch.zeros(B, 1, dtype=torch.long, device=dev),
        "used_capacity": torch.zeros(B, 1, device=dev),
        "vehicle_capacity": torch.full((B, 1), vehicle_capacity, device=dev),
    }
    st["action_mask"] = sdvrp_action_mask(st)
    st["done"] = torch.zeros(B, 1, dtype=torch.bool, device=dev)
    return st


def sdvrp_step(state, action):
    """sdvrp/env.py:55-82: deliver min(remaining demand, remaining capacity); nodes may be revisited"""
    st = dict(state)
    current_node = action[:, None]
    selected_demand = gather_by_index(st["demand_with_depot"], current_node, dim=-1, squeeze=False)[..., :1]
    delivered = torch.min(selected_demand, st["vehicle_capacity"] - st["used_capacity"])
    used_capacity = (st["used_capacity"] + delivered) * (current_node != 0).float()
    demand_with_depot = st["demand_with_depot"].scatter_add(-1, current_node, -delivered)
    done = ~(demand_with_depot > 0).any(-1)
    st.update(demand_with_depot=demand_with_depot, current_node=current_node, used_capacity=used_capacity,
              reward=torch.zeros_like(done), done=done, action=action)
    st["action_mask"] = sdvrp_action_mask(st)
    return st


def sdvrp_check_solution(st, actions):
    """sdvrp/env.py:118-139"""
    demands = torch.cat((-st["vehicle_capacity"], st["demand"]), 1).clone()
    rng = torch.arange(demands.shape[0])
    used_cap = torch.zeros_like(st["demand"][..., 0])
    a_prev = None
    for a in actions.transpose(0, 1):
        assert a_prev is None or (demands[((a_prev == 0) & (a == 0)), :] == 0).all(), \
            "Cannot visit depot twice if any nonzero demand"
        d = torch.min(demands[rng, a], st["vehicle_capacity"].squeeze(-1) - used_cap)
        demands[rng, a] -= d
        used_cap += d
        used_cap[a == 0] = 0
        a_prev = a
    assert (demands == 0).all(), "All demand must be satisfied"


def sdvrp_dynamic_embedding(weights, st):
    """nn/env_embeddings/dynamic.py:60-78 (SDVRPDynamicEmbedding): Linear(1 -> 3E, no bias) of the remaining demand,
    depot entry forced to 0; chunks add to glimpse_key / glimpse_val / logit_key (am/decoder.py:142-154)."""
    w = _w(weights, "dynamic_embedding.projection.weight")
    d = st["demand_with_depot"][..., None].to(w.dtype, copy=True)  # the env state stays fp32; the network runs in the weights' dtype
    d[..., 0, :] = 0
    return F.linear(d, w).chunk(3, dim=-1)


# reference: rl4co/envs/routing/op/env.py (orienteering: collect prizes, return to the depot within max_length)


def op_action_mask(st):
    """op/env.py:140-155: visited, or the depot already re-entered, or tour_length + dist(cur, n) > max_length[n]
    (max_length[n] already has the way back to the depot taken off, op/env.py:121-123); the depot is always feasible"""
    current_loc = gather_by_index(st["locs"], st["current_node"])[..., None, :]
    exceeds_length = st["tour_length"][..., None] + (st["locs"] - current_loc).norm(p=2, dim=-1) > st["max_length"]
    mask = st["visited"] | st["visited"][..., 0:1] | exceeds_length
    action_mask = ~mask
    action_mask[..., 0] = 1
    return action_mask


def op_reset(depot, locs, prize, max_length):
    """op/env.py:107-138"""
    B = locs.shape[0]
    dev = locs.device
    locs_with_depot = torch.cat((depot[:, None, :], locs), -2)
    st = {
        "locs": locs_with_depot,
        "prize": F.pad(prize, (1, 0), mode="constant", value=0),
        "tour_length": torch.zeros(B, device=dev),
        "max_length": max_length[..., None] - (depot[..., None, :] - locs_with_depot).norm(p=2, dim=-1) - 1e-6,
        "current_node": torch.zeros(B, 1, dtype=torch.long, device=dev),
        "visited": torch.zeros((B, locs_with_depot.shape[-2]), dtype=torch.bool, device=dev),
        "current_total_prize": torch.zeros(B, dtype=torch.float, device=dev),
        "i": torch.zeros((B,), dtype=torch.int64, device=dev),
    }
    st["action_mask"] = op_action_mask(st)
    st["done"] = torch.zeros(B, 1, dtype=torch.bool, device=dev)
    return st


def op_step(state, action):
    """op/env.py:72-105: done when the depot is re-entered after step 0"""
    st = dict(state)
    current_node = action[:, None]
    previous_loc = gather_by_index(st["locs"], st["current_node"])
    current_loc = gather_by_index(st["locs"], current_node)
    tour_length = st["tour_length"] + (current_loc - previous_loc).norm(p=2, dim=-1)
    current_total_prize = st["current_total_prize"] + gather_by_index(st["prize"], current_node, dim=-1)
    visited = st["visited"].scatter(-1, current_node, 1)
    done = (current_node.squeeze(-1) == 0) & (st["i"] > 0)
    st.update(tour_length=tour_length, current_node=current_node, visited=visited,
              current_total_prize=current_total_prize, i=st["i"] + 1, reward=torch.zeros_like(done), done=done,
              action=action)
    st["action_mask"] = op_action_mask(st)
    return st


def op_reward(st, actions):
    """op/env.py:157-165: sum of the collected prizes (the depot's is 0)"""
    if actions.size(-1) == 1:
        assert (actions == 0).all(), "If all length 1 tours, they should be zero"
        return torch.zeros(actions.size(0), dtype=torch.float, device=actions.device)
    return st["prize"].gather(1, actions).sum(-1)


def op_check_solution(st, actions, add_distance_to_depot: bool = True):
    """op/env.py:167-192"""
    sorted_actions = actions.sort(1)[0]
    assert ((sorted_actions[:, 1:] == 0) | (sorted_actions[:, 1:] > sorted_actions[:, :-1])).all(), "Duplicates"
    length = get_tour_length(gather_by_index(st["locs"], actions))
    max_length = st["max_length"]
    if add_distance_to_depot:
        max_length = max_length + (st["locs"][..., 0:1, :] - st["locs"]).norm(p=2, dim=-1) + 1e-6
    assert (length[..., None] <= max_length + 1e-5).all(), "Max length exceeded"


# reference: rl4co/envs/routing/pctsp/env.py (prize-collecting TSP: collect prize >= 1, pay the penalties of the rest)


def pctsp_action_mask(st):
    """pctsp/env.py:143-151: customers: visited or the depot re-entered; depot: infeasible while the collected prize is
    below 1.0 (a literal, not prize_required) and unvisited customers remain"""
    mask = st["visited"] | st["visited"][..., 0:1]
    mask[..., 0] = (st["cur_total_prize"] < 1.0) & (st["visited"][..., 1:].int().sum(-1) < st["visited"][..., 1:].size(-1))
    return ~(mask > 0)


def pctsp_reset(depot, locs, deterministic_prize, penalty, prize_required: float = 1.0):
    """pctsp/env.py:95-141 (deterministic prizes: real_prize = expected_prize)"""
    B = locs.shape[0]
    dev = locs.device
    st = {
        "locs": torch.cat([depot[..., None, :], locs], dim=-2),
        "current_node": torch.zeros((B,), dtype=torch.int64, device=dev),
        "expected_prize": deterministic_prize,
        "real_prize": torch.cat([torch.zeros_like(deterministic_prize[..., :1]), deterministic_prize], dim=-1),
        "penalty": F.pad(penalty, (1, 0), mode="constant", value=0),
        "cur_total_prize": torch.zeros(B, device=dev),
        "cur_total_penalty": penalty.sum(-1),
        "visited": torch.zeros((B, locs.shape[-2] + 1), dtype=torch.bool, device=dev),
        "prize_required": torch.full((B,), prize_required, device=dev),
        "i": torch.zeros((B,), dtype=torch.int64, device=dev),
    }
    st["action_mask"] = pctsp_action_mask(st)
    st["done"] = torch.zeros(B, 1, dtype=torch.bool, device=dev)
    return st


def pctsp_step(state, action):
    """pctsp/env.py:62-93"""
    st = dict(state)
    cur_total_prize = st["cur_total_prize"] + gather_by_index(st["real_prize"], action)
    cur_total_penalty = st["cur_total_penalty"] + gather_by_index(st["penalty"], action)
    visited = st["visited"].scatter(-1, action[..., None], 1)
    done = (st["i"] > 0) & (action == 0)
    st.update(current_node=action, cur_total_prize=cur_total_prize, cur_total_penalty=cur_total_penalty, visited=visited,
              i=st["i"] + 1, reward=torch.zeros_like(done), done=done, action=action)
    st["action_mask"] = pctsp_action_mask(st)
    return st


def pctsp_reward(st, actions):
    """pctsp/env.py:153-172: saved penalties - (tour length from / to the depot + all penalties)"""
    if actions.size(-1) == 1:
        assert (actions == 0).all(), "If all length 1 tours, they should be zero"
        return torch.zeros(actions.size(0), dtype=torch.float, device=actions.device)
    locs_ordered = torch.cat([st["locs"][..., 0:1, :], gather_by_index(st["locs"], actions)], dim=1)
    length = get_tour_length(locs_ordered)
    saved_penalty = st["penalty"].gather(1, actions)
    return saved_penalty.sum(-1) - (length + st["penalty"][..., 1:].sum(-1))


def pctsp_check_solution(st, actions):
    """pctsp/env.py:174-197"""
    sorted_actions = actions.sort(1)[0]
    assert ((sorted_actions[..., 1:] == 0) | (sorted_actions[..., 1:] > sorted_actions[..., :-1])).all(), "Duplicates"
    p = st["real_prize"].gather(1, actions)
    assert ((p.sum(-1) >= 1 - 1e-5) | (sorted_actions.size(-1) - (sorted_actions == 0).int().sum(-1)
                                       == (st["locs"].size(-2) - 1))).all(), "Total prize does not satisfy min total prize"


ENV_RESET = {"tsp": tsp_reset, "cvrp": cvrp_reset, "sdvrp": sdvrp_reset, "op": op_reset, "pctsp": pctsp_reset}
ENV_STEP = {"tsp": tsp_step, "cvrp": cvrp_step, "sdvrp": sdvrp_step, "op": op_step, "pctsp": pctsp_step}


def env_reset(env_name, inst):
    """inst: dict with 'locs' (tsp) or 'depot','locs','demand' (cvrp / sdvrp; generator output keys)."""
    if env_name == "tsp":
        return tsp_reset(inst["locs"])
    if env_name == "sdvrp":
        return sdvrp_reset(inst["depot"], inst["locs"], inst["demand"])
    if env_name == "op":
        return op_reset(inst["depot"], inst["locs"], inst["prize"], inst["max_length"])
    if env_name == "pctsp":
        return pctsp_reset(inst["depot"], inst["locs"], inst["deterministic_prize"], inst["penalty"])
    return cvrp_reset(inst["depot"], inst["locs"], inst["demand"])


def env_reward(env_name, st, actions):
    if env_name == "op":
        return op_reward(st, actions)
    if env_name == "pctsp":
        return pctsp_reward(st, actions)
    return tsp_reward(st["locs"], actions) if env_name == "tsp" else cvrp_reward(st["locs"], actions)


# --------------------------------------------------------------------------- generators
# reference: rl4co/envs/routing/tsp/generator.py:49-58, cvrp/generator.py:15-30,114-140

OP_MAX_LENGTHS = {20: 2.0, 50: 3.0, 100: 4.0}  # op/generator.py:16
CAPACITIES = {10: 20.0, 15: 25.0, 20: 30.0, 30: 33.0, 40: 37.0, 50: 40.0, 60: 43.0, 75: 45.0,
              100: 50.0, 125: 55.0, 150: 60.0, 200: 70.0, 500: 100.0, 1000: 150.0}


def generate_instances(env_name, batch, num_loc, generator=None):
    """Uniform(0,1) sampling exactly as torch.distributions.Uniform(...).sample does
    (rand * (high-low) + low), in the generator's call order."""
    def uni(shape, low, high):
        return torch.rand(shape, generator=generator) * (high - low) + low

    if env_name == "tsp":
        return {"locs": uni((batch, num_loc, 2), 0.0, 1.0)}
    if env_name == "op":  # op/generator.py:102-139, prize_type "dist": prize from the distance to the depot
        locs = uni((batch, num_loc + 1, 2), 0.0, 1.0)
        prize = (locs[..., 0:1, :] - locs[..., 1:, :]).norm(p=2, dim=-1)
        prize = (1 + (prize / prize.max(dim=-1, keepdim=True)[0] * 99).int()).float() / 100
        ml = OP_MAX_LENGTHS.get(num_loc) or OP_MAX_LENGTHS[min(OP_MAX_LENGTHS, key=lambda x: abs(x - num_loc))]
        return {"locs": locs[:, 1:, :], "depot": locs[:, 0, :], "prize": prize, "max_length": torch.full((batch,), ml)}
    if env_name == "pctsp":  # pctsp/generator.py:36-139: penalty, deterministic prize, stochastic prize, in that order
        locs = uni((batch, num_loc + 1, 2), 0.0, 1.0)
        mp = OP_MAX_LENGTHS.get(num_loc) or OP_MAX_LENGTHS[min(OP_MAX_LENGTHS, key=lambda x: abs(x - num_loc))]
        penalty = uni((batch, num_loc), 0.0, mp * 3.0 / num_loc)
        det = uni((batch, num_loc), 0.0, 4.0 / num_loc)
        sto = uni((batch, num_loc), 0.0, 2.0) * det
        return {"locs": locs[:, 1:, :], "depot": locs[:, 0, :], "penalty": penalty, "deterministic_prize": det,
                "stochastic_prize": sto}
    # cvrp and sdvrp share CVRPGenerator (sdvrp/env.py:47-54)
    locs = uni((batch, num_loc + 1, 2), 0.0, 1.0)
    demand = uni((batch, num_loc), 0.0, 9.0)
    demand = (demand.int() + 1).float()
    cap = CAPACITIES.get(num_loc) or CAPACITIES[min(CAPACITIES, key=lambda x: abs(x - num_loc))]
    return {"locs": locs[:, 1:, :], "depot": locs[:, 0, :], "demand": demand / cap,
            "capacity": torch.full((batch, 1), cap)}


# --------------------------------------------------------------------------- decoder
# reference: rl4co/models/zoo/am/decoder.py, nn/env_embeddings/context.py, nn/attention.py

def _w(weights, key):
    return weights["decoder." + key] if ("decoder." + key) in weights else weights[key]


def precompute_cache(weights, h, use_graph_context=True):
    """am/decoder.py:201-228"""
    k, v, l = F.linear(h, _w(weights, "project_node_embeddings.weight")).chunk(3, dim=-1)
    g = F.linear(h.mean(1), _w(weights, "project_fixed_context.weight")) if use_graph_context else 0
    return {"node_embeddings": h, "graph_context": g, "glimpse_key": k, "glimpse_val": v, "logit_key": l}


def tsp_context(weights, emb, st):
    """nn/env_embeddings/context.py:116-134 (TSPContext.forward)"""
    B = emb.size(0)
    wp = _w(weights, "context_embedding.W_placeholder")
    first = st["first_node"]
    node_dim = (-1,) if first.dim() == 1 else (first.size(-1), -1)
    if st["i"][(0,) * st["i"].dim()].item() < 1:
        if first.dim() == 1:
            ctx = wp[None, :].expand(B, wp.size(-1))
        else:
            ctx = wp[None, None, :].expand(B, first.size(1), wp.size(-1))
    else:
        ctx = gather_by_index(emb, torch.stack([first, st["current_node"]], -1).view(B, -1)).view(B, *node_dim)
    return F.linear(ctx, _w(weights, "context_embedding.project_context.weight"))


def vrp_context(weights, emb, st):
    """nn/env_embeddings/context.py:61-74,137-149 (EnvContext.forward + VRPContext)"""
    cur = gather_by_index(emb, st["current_node"])
    state_emb = st["vehicle_capacity"] - st["used_capacity"]
    return F.linear(torch.cat([cur, state_emb], -1), _w(weights, "context_embedding.project_context.weight"))


def op_context(weights, emb, st):
    """nn/env_embeddings/context.py:61-74,201-213 (EnvContext.forward + OPContext): [h_cur ; max_length[0] - tour_length]"""
    cur = gather_by_index(emb, st["current_node"])
    state_emb = (st["max_length"][..., 0] - st["tour_length"])[..., None]
    return F.linear(torch.cat([cur, state_emb], -1), _w(weights, "context_embedding.project_context.weight"))


def pctsp_context(weights, emb, st):
    """nn/env_embeddings/context.py:61-74,184-198 (PCTSPContext): [h_cur ; clamp(prize_required - cur_total_prize, 0)]"""
    cur = gather_by_index(emb, st["current_node"])
    state_emb = torch.clamp(st["prize_required"] - st["cur_total_prize"], min=0)[..., None]
    return F.linear(torch.cat([cur, state_emb], -1), _w(weights, "context_embedding.project_context.weight"))


def pointer_logits(weights, q, K, V, L, mask, num_heads=8):
    """nn/attention.py:274-320 (PointerAttention.forward, mask_inner=True, no out bias)"""
    def heads(x):  # "... g (h s) -> ... h g s"
        return x.view(*x.shape[:-1], num_heads, -1).transpose(-2, -3)

    attn_mask = mask.unsqueeze(1) if mask.ndim == 3 else mask.unsqueeze(1).unsqueeze(2)
    o = F.scaled_dot_product_attention(heads(q), heads(K), heads(V), attn_mask=attn_mask)
    o = o.transpose(-2, -3)
    o = o.reshape(*o.shape[:-2], -1)  # "... h n g -> ... n (h g)"
    glimpse = F.linear(o, _w(weights, "pointer.project_out.weight"))
    logits = torch.bmm(glimpse, L.squeeze(-2).transpose(-2, -1)).squeeze(-2) / math.sqrt(glimpse.size(-1))
    assert not torch.isnan(logits).any(), "Logits contain NaNs"
    return logits


def decoder_forward(weights, env_name, st, cache, num_starts=0, faithful_copies=True):
    """am/decoder.py:128-193 (AttentionModelDecoder.forward; static dynamic-embedding)"""
    if num_starts > 1:
        st = {k: unbatchify(v, num_starts) for k, v in st.items() if k != "reward"}
    emb, g = cache["node_embeddings"], cache["graph_context"]
    two_batch_dims = st["action_mask"].dim() == 3
    if two_batch_dims and isinstance(g, torch.Tensor):
        g = g.unsqueeze(1)
    ctx = (tsp_context(weights, emb, st) if env_name == "tsp" else
           op_context(weights, emb, st) if env_name == "op" else
           pctsp_context(weights, emb, st) if env_name == "pctsp" else vrp_context(weights, emb, st))  # cvrp, sdvrp
    q = ctx + g
    q = q.unsqueeze(1) if q.ndim == 2 else q
    K, V, L = cache["glimpse_key"], cache["glimpse_val"], cache["logit_key"]
    if env_name == "sdvrp":  # dynamic embedding, am/decoder.py:142-154
        assert num_starts <= 1, "the sdvrp restatement covers single-start decoding"
        dk, dv, dl = sdvrp_dynamic_embedding(weights, st)
        K, V, L = K + dk, V + dv, L + dl
    elif faithful_copies:  # `stat + 0` materialises 3 copies per step, am/decoder.py:149-152
        K, V, L = K + 0, V + 0, L + 0
    mask = st["action_mask"]
    logits = pointer_logits(weights, q, K, V, L, mask)
    if num_starts > 1:  # "b s l -> (s b) l", am/decoder.py:190-192
        logits = logits.transpose(0, 1).reshape(-1, logits.size(-1))
        mask = mask.transpose(0, 1).reshape(-1, mask.size(-1))
    return logits, mask


# --------------------------------------------------------------------------- decoding strategy
# reference: rl4co/utils/decoding.py


def keep_top_k(logits, top_k):
    """utils/decoding.py:109-114: entries below the k-th largest logit of their row become -inf (ties with the
    k-th value survive)."""
    kth = torch.topk(logits, top_k).values[..., -1:]
    return torch.where(logits < kth, torch.full_like(logits, float("-inf")), logits)


def keep_top_p(logits, top_p):
    """utils/decoding.py:117-135: nucleus filter. Rows are sorted ascending, turned into probabilities, and the
    lower tail whose cumulative mass is <= 1 - top_p is dropped; top_p outside (0, 1) is a no-op."""
    if not 0.0 < top_p < 1.0:
        return logits
    ordered, order = torch.sort(logits, dim=-1)
    tail = ordered.softmax(dim=-1).cumsum(dim=-1) <= (1.0 - top_p)
    drop = torch.zeros_like(tail).scatter(-1, order, tail)
    return torch.where(drop, torch.full_like(logits, float("-inf")), logits)


def process_logits(logits, mask, temperature=1.0, tanh_clipping=10.0, mask_logits=True, top_k=0, top_p=0.0):
    """utils/decoding.py:138-188: tanh clip -> mask -> / temperature -> top-k -> top-p -> log_softmax"""
    if tanh_clipping > 0:
        logits = torch.tanh(logits) * tanh_clipping
    if mask_logits:
        logits[~mask] = float("-inf")
    logits = logits / temperature
    if top_k > 0:
        logits = keep_top_k(logits, min(top_k, logits.size(-1)))
    if top_p > 0:
        assert top_p <= 1.0, "top-p should be in (0, 1]."
        logits = keep_top_p(logits, top_p)
    return F.log_softmax(logits, dim=-1)


def select_greedy(logprobs, mask):
    """utils/decoding.py:387-397"""
    sel = logprobs.argmax(dim=-1)
    assert not (~mask).gather(1, sel.unsqueeze(-1)).any(), "infeasible action selected"
    return sel


def select_sampling(logprobs, mask, noise=None, generator=None):
    """utils/decoding.py:399-413.  ``torch.multinomial(p, 1)`` is, in ATen,
    ``argmax(p / q)`` with ``q = empty_like(p).exponential_(1)`` (the n_sample==1 path of
    aten/src/ATen/native/Distributions.cpp multinomial); passing ``noise=q`` makes the draw
    reproducible across devices."""
    probs = logprobs.exp()
    if noise is None:
        sel = torch.multinomial(probs, 1, generator=generator).squeeze(1)
    else:
        sel = (probs / noise).argmax(dim=-1)
    assert not (~mask).gather(1, sel.unsqueeze(-1)).any(), "infeasible action selected"
    return sel


def get_log_likelihood(logprobs):
    """utils/decoding.py:38-62 (per-step logprobs already gathered)"""
    assert (logprobs > -1000).all(), "Logprobs should not be -inf, check sampling procedure!"
    return logprobs.sum(1)


# --------------------------------------------------------------------------- rollout loop
# reference: rl4co/models/common/constructive/base.py:192-251


def rollout(weights, env_name, inst, h, decode_type="greedy", num_starts=None, actions=None,
            noise=None, use_graph_context=True, temperature=1.0, tanh_clipping=10.0,
            return_trace=False, faithful_copies=True, num_loc=None, generator=None, top_k=0, top_p=0.0):
    """Decode loop of ConstructivePolicy.forward from encoder output ``h`` on.

    decode_type: greedy | sampling | multistart_greedy | multistart_sampling | evaluate
    actions    : [B,T] teacher-forced actions (forces decode_type="evaluate")
    noise      : callable(step, shape) -> Exp(1) tensor, or None to use torch.multinomial
    returns dict(reward[B'], log_likelihood[B'], actions[B',T], logprobs[B',T], state, trace?)
    """
    if actions is not None:
        decode_type = "evaluate"
    multistart = "multistart" in decode_type
    st = env_reset(env_name, inst)
    B = st["locs"].shape[0]
    step_fn = ENV_STEP[env_name]
    acts, lps = [], []
    trace = {"mask": [], "logits": [], "logprobs": []} if return_trace else None

    # pre_decoder_hook, utils/decoding.py:282-330
    S = 0
    if multistart:
        S = num_starts if num_starts is not None else get_num_starts(st["action_mask"].shape[-1], env_name)
        if S > 1 or num_starts is None:
            nl = num_loc if num_loc is not None else (st["locs"].shape[1] - (1 if env_name in DEPOT_ENVS else 0))
            a0 = select_start_nodes(B, S, nl, env_name, device=st["locs"].device)
            st = {k: batchify(v, S) for k, v in st.items()}
            st = step_fn(st, a0)
            lps.append(torch.zeros_like(a0, dtype=torch.float32))
            acts.append(a0)
        else:
            S = 0
    cache = precompute_cache(weights, h, use_graph_context)

    step = 0
    while not st["done"].all():
        logits, mask = decoder_forward(weights, env_name, st, cache, S, faithful_copies)
        if return_trace:
            trace["mask"].append(mask.clone())
            trace["logits"].append(logits.clone())
        logprobs = process_logits(logits, mask, temperature, tanh_clipping, top_k=top_k, top_p=top_p)
        if decode_type == "evaluate":
            a = actions[..., step]
        elif "greedy" in decode_type:
            a = select_greedy(logprobs, mask)
        else:
            q = noise(step, logprobs.shape) if noise is not None else None
            a = select_sampling(logprobs, mask, q, generator)
        if return_trace:
            trace["logprobs"].append(logprobs.clone())
        lps.append(gather_by_index(logprobs, a, dim=1))
        acts.append(a)
        st = step_fn(st, a)
        step += 1

    logprobs = torch.stack(lps, 1)
    out_actions = torch.stack(acts, 1)
    out = {
        "reward": env_reward(env_name, st, out_actions),
        "log_likelihood": get_log_likelihood(logprobs),
        "actions": out_actions,
        "logprobs": logprobs,
        "state": st,
    }
    if return_trace:
        out["trace"] = trace
    return out


def teacher_forced_logprobs(weights, env_name, inst, h, acts, num_starts=1, forced_first=False, temperature=1.0,
                            tanh_clipping=10.0, use_graph_context=True):
    """Per-step log-probabilities [B*S, T] of given trajectories ``acts`` [B*S, T], differentiable in ``weights`` and
    ``h`` (no inference mode; float64 weights and ``h`` give a float64 network over the fp32 env state).

    The decode loop of constructive/base.py:209-251 teacher-forced step by step. S > 1 rows are start-major over the
    batchified instances (flat index s * B + b). ``forced_first``: the first action is a forced multistart start taken
    by the env step without a decoder call, with log-prob 0 (decoding.py:309-326); ``rollout(actions=...)`` would score
    it. T is the oracle's episode length: columns of ``acts`` past it (the padding of finished trajectories) are not
    read."""
    if num_starts > 1:
        inst, h = batchify(inst, num_starts), batchify(h, num_starts)
    st = env_reset(env_name, inst)
    step_fn = ENV_STEP[env_name]
    cache = precompute_cache(weights, h, use_graph_context)
    lps, t = [], 0
    if forced_first:
        st = step_fn(st, acts[:, 0])
        lps.append(torch.zeros(acts.shape[0], dtype=h.dtype))
        t = 1
    while not st["done"].all():
        assert t < acts.shape[1], "the trajectories end before the episode does"
        logits, mask = decoder_forward(weights, env_name, st, cache, 0, faithful_copies=False)
        lp = process_logits(logits.clone(), mask, temperature, tanh_clipping)
        lps.append(lp.gather(1, acts[:, t:t + 1]).squeeze(1))
        st = step_fn(st, acts[:, t])
        t += 1
    return torch.stack(lps, 1)


# --------------------------------------------------------------------------- beam search
# reference: rl4co/utils/decoding.py:464-600 (BeamSearch strategy) inside the loop of constructive/base.py:219-251


def rollout_beam_search(weights, env_name, inst, h, beam_width=None, select_best=True, use_graph_context=True,
                        temperature=1.0, tanh_clipping=10.0, num_loc=None, faithful_copies=True, top_k=0, top_p=0.0):
    """Beam search over the flat (beam-major: row = w * B + b) expanded batch.

    Every step keeps, per instance, the ``beam_width`` best (parent beam, node) pairs by cumulative log-probability
    (decoding.py:568-600); the per-step actions / full log-prob rows / parent pointers are recorded in the order
    they were produced and re-threaded from the last step backwards (decoding.py:529-556); with ``select_best`` the
    beam with the highest reward per instance is returned (decoding.py:558-566).
    Returns dict(reward, log_likelihood, actions[*, T], logprobs[*, T]) with * = B (select_best) or B * beam_width."""
    st = env_reset(env_name, inst)
    B = st["locs"].shape[0]
    step_fn = ENV_STEP[env_name]
    W = beam_width if beam_width is not None else get_num_starts(st["action_mask"].shape[-1], env_name)
    assert W > 1, "beam width must be larger than 1"
    nl = num_loc if num_loc is not None else (st["locs"].shape[1] - (1 if env_name == "cvrp" else 0))
    a0 = select_start_nodes(B, W, nl, env_name, device=st["locs"].device)
    st = {k: batchify(v, W) for k, v in st.items()}
    st = step_fn(st, a0)
    # decoding.py:507-513: the forced first step carries log-prob 0 and parent 0
    all_lp = [torch.zeros(st["action_mask"].shape, dtype=torch.float32)]
    acts = [a0]
    parents = [torch.zeros(B * W, dtype=torch.int32)]
    cum = torch.zeros(B * W, 1)
    row_of_instance = torch.arange(B).repeat(W)
    cache = precompute_cache(weights, h, use_graph_context)

    while not st["done"].all():
        logits, mask = decoder_forward(weights, env_name, st, cache, W, faithful_copies)
        lp = process_logits(logits, mask, temperature, tanh_clipping, top_k=top_k, top_p=top_p)
        N = lp.shape[1]
        # candidates of instance b side by side: column w * N + n = (parent beam w, node n)
        cand = torch.cat((lp + cum).split(B), dim=1)
        best, flat = torch.topk(cand, W, dim=1)
        cum = torch.cat(best.unbind(1)).unsqueeze(1)
        flat = torch.cat(flat.unbind(1))
        a, parent = flat % N, (flat // N).int()
        src = row_of_instance + parent * B  # the row each surviving beam continues from
        st = {k: v[src] for k, v in st.items()}
        assert mask[src].gather(1, a.unsqueeze(-1)).all(), "infeasible action selected"
        all_lp.append(lp[src])
        acts.append(a)
        parents.append(parent)
        st = step_fn(st, a)

    # backtrack (decoding.py:529-556)
    A, L = torch.stack(acts, 1), torch.stack(all_lp, 1)
    seq, seq_lp = [A[:, -1]], [L[:, -1]]
    cur = parents[-1]
    for k in reversed(range(len(parents) - 1)):
        src = row_of_instance + cur * B
        seq.append(A[src, k])
        seq_lp.append(L[src, k])
        cur = parents[k][src]
    A = torch.stack(seq[::-1], 1)
    L = torch.stack(seq_lp[::-1], 1)
    reward = env_reward(env_name, st, A)
    if select_best:  # decoding.py:558-566
        idx = unbatchify(reward, W).argmax(dim=1)
        keep = torch.arange(B) + idx * B
        A, L, reward = A[keep], L[keep], reward[keep]
    lp_taken = L.gather(-1, A.unsqueeze(-1)).squeeze(-1)  # get_log_likelihood on 3-D logprobs, decoding.py:48-50
    return {"reward": reward, "log_likelihood": get_log_likelihood(lp_taken), "actions": A, "logprobs": lp_taken}


# --------------------------------------------------------------------------- encoder
# reference: rl4co/models/zoo/am/encoder.py:68-87, nn/env_embeddings/init.py:55-68,115-136,
#            nn/graph/attnnet.py:16-106, nn/attention.py:64-134, nn/ops.py:30-54


def init_embedding(weights, env_name, st):
    """Raw instance data enters the network in the weights' dtype (float64 weights give a float64 network over the
    fp32 env state)."""
    p = "encoder.init_embedding."
    locs = st["locs"].to(weights[p + "init_embed.weight"].dtype)
    if env_name == "tsp":
        return F.linear(locs, weights[p + "init_embed.weight"], weights[p + "init_embed.bias"])
    depot, cities = locs[:, :1, :], locs[:, 1:, :]
    de = F.linear(depot, weights[p + "init_embed_depot.weight"], weights[p + "init_embed_depot.bias"])
    feat = st["prize"][..., 1:, None] if env_name == "op" else None  # init.py:254-280 / 115-136
    if env_name == "pctsp":  # init.py:221-251: (x, y, expected prize, penalty)
        feat = torch.stack((st["expected_prize"], st["penalty"][..., 1:]), -1)
    elif feat is None:
        feat = st["demand"][..., None]
    ne = F.linear(torch.cat((cities, feat), -1), weights[p + "init_embed.weight"], weights[p + "init_embed.bias"])
    return torch.cat((de, ne), -2)


def _normalization(weights, prefix, x, kind, batch_stats=False):
    """`batch_stats`: batch normalisation with the statistics of this batch (a module in train mode); the running
    statistics are read otherwise, and never updated."""
    w, b = weights[prefix + "normalizer.weight"], weights[prefix + "normalizer.bias"]
    if kind == "batch":
        if batch_stats:
            y = F.batch_norm(x.reshape(-1, x.size(-1)), None, None, w, b, training=True, eps=1e-5)
        else:
            y = F.batch_norm(x.reshape(-1, x.size(-1)), weights[prefix + "normalizer.running_mean"],
                             weights[prefix + "normalizer.running_var"], w, b, training=False, eps=1e-5)
        return y.view(*x.size())
    if kind == "instance":
        return F.instance_norm(x.permute(0, 2, 1), weight=w, bias=b, eps=1e-5).permute(0, 2, 1)
    raise ValueError(kind)


def encoder_forward(weights, env_name, st, num_layers=3, num_heads=8, normalization="batch", batch_stats=False,
                    relu_masks=None, pre_activations=None):
    """``relu_masks``: one bool tensor per layer, the units of the FFN's ReLU to keep, in place of the sign of this
    forward's own pre-activation. A gradient check uses the checked network's activation pattern: a unit whose
    pre-activation lies within round-off of 0 may sit on either side in fp32, and the gradient jumps there.
    ``pre_activations``: a list that receives each layer's ReLU input (detached)."""
    h = init_embedding(weights, env_name, st)
    init_h = h
    for i in range(num_layers):
        p = f"encoder.net.layers.{i}."
        qkv = F.linear(h, weights[p + "0.module.Wqkv.weight"], weights[p + "0.module.Wqkv.bias"])
        B, N, _ = qkv.shape
        q, k, v = qkv.view(B, N, 3, num_heads, -1).permute(2, 0, 3, 1, 4).unbind(0)
        o = F.scaled_dot_product_attention(q, k, v)
        o = o.transpose(1, 2).reshape(B, N, -1)
        h = h + F.linear(o, weights[p + "0.module.out_proj.weight"], weights[p + "0.module.out_proj.bias"])
        h = _normalization(weights, p + "1.", h, normalization, batch_stats)
        f = F.linear(h, weights[p + "2.module.lins.0.weight"], weights[p + "2.module.lins.0.bias"])
        if pre_activations is not None:
            pre_activations.append(f.detach())
        f = F.relu(f) if relu_masks is None else f * relu_masks[i].to(f.dtype)
        h = h + F.linear(f, weights[p + "2.module.lins.1.weight"], weights[p + "2.module.lins.1.bias"])
        h = _normalization(weights, p + "3.", h, normalization, batch_stats)
    return h, init_h


def policy_forward(weights, env_name, inst, decode_type="greedy", num_layers=3, normalization="batch", **kw):
    """ConstructivePolicy.forward, constructive/base.py:154-263 (encoder + rollout)."""
    st0 = env_reset(env_name, inst)
    h, _ = encoder_forward(weights, env_name, st0, num_layers=num_layers, normalization=normalization)
    if decode_type == "beam_search":
        return rollout_beam_search(weights, env_name, inst, h, **kw)
    return rollout(weights, env_name, inst, h, decode_type=decode_type, **kw)


# --------------------------------------------------------------------------- REINFORCE / POMO glue
# reference: rl4co/models/rl/reinforce/reinforce.py:71-111, baselines.py:55-81, zoo/pomo/model.py:88-143


def reinforce_loss(reward, log_likelihood, baseline_value):
    """reinforce.py:96-104: advantage = reward - bl ; loss = -(adv * ll).mean()"""
    advantage = reward - baseline_value
    return -(advantage * log_likelihood).mean()


def shared_baseline(reward, num_starts):
    """baselines.py:55-61 SharedBaseline.eval: mean over the starts of each instance."""
    r = unbatchify(reward, num_starts)
    return r.mean(dim=1, keepdim=True)


def mean_baseline(reward):
    """baselines.py:75-81 (ExponentialBaseline first call / MeanBaseline): reward.mean()"""
    return reward.mean()


def float64_weights(state_dict, trainable):
    """float64 CPU copy of a policy's ``state_dict`` for gradient checks: the names in ``trainable`` become leaves that
    require grad, the other floating-point entries (normalisation buffers) plain float64 tensors."""
    out = {}
    for k, v in state_dict.items():
        v = v.detach().cpu()
        out[k] = v.double().requires_grad_(k in trainable) if v.is_floating_point() else v
    return out


def gradient_errors(grads, weights, floor=1e-2):
    """Per-parameter comparison of ``grads`` {name: gradient or None} with the ``.grad`` of the float64 leaves in
    ``weights``. Returns (rel, zero):
      rel  {name: ||g - g64|| / max(||g64||, floor * G)} (Frobenius; G = the norm of the whole float64 gradient; a
           missing product gradient counts as zeros). The floor keeps directions the loss is (nearly) invariant to --
           the bias of a Linear right before a normalisation has a float64 gradient of round-off size -- from turning
           fp32 round-off into a meaningless relative error;
      zero {name: ||g||} where the float64 gradient is None or exactly 0 (the loss does not reach the parameter)."""
    ref = {k: weights[k].grad for k in grads}
    total = math.sqrt(sum(float(g.square().sum()) for g in ref.values() if g is not None))
    rel, zero = {}, {}
    for k, g in grads.items():
        g64 = ref[k]
        if g64 is None or not bool(g64.any()):
            zero[k] = 0.0 if g is None else float(g.detach().double().norm())
            continue
        diff = g64 if g is None else g.detach().double().cpu() - g64
        rel[k] = float(diff.norm()) / max(float(g64.norm()), floor * total)
    return rel, zero


def pomo_reduce(reward, n_aug, n_start):
    """zoo/pomo/model.py:103-136: [aug*start*B] -> max over starts, then max over augs."""
    r = unbatchify_multi(reward, (n_aug, n_start)) if n_aug > 1 else unbatchify(reward, n_start).unsqueeze(1)
    max_reward, _ = r.max(dim=-1)
    max_aug_reward, _ = max_reward.max(dim=1)
    return max_reward, max_aug_reward
