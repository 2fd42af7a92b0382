"""CPU: gradients of the training step's teacher-forced pass (`evaluate_log_likelihood`) against the float64 oracle
under autograd.

The product runs on CPU tensors, so the attention is stock SDPA and every Linear stock torch: what is checked here is
the glue -- the vectorised MDP replays (`replay_states`, `replay_budget_states`, `replay_split_delivery_states`), the
query construction, the multistart layout, the forced first step and the sdvrp rank-one dynamic-embedding algebra --
independent of any kernel. The oracle runs the reference's step-by-step decode loop (`O.teacher_forced_logprobs`) and
encoder (`O.encoder_forward`) in float64, along trajectories the oracle itself sampled.
"""

import pytest
import torch

from conftest import name_seeded_weights
from oracle import am_rollout_oracle as O

ENVS = ["tsp", "cvrp", "sdvrp", "op", "pctsp"]
# (log-prob atol, O.gradient_errors bound): a float64 product must agree to round-off -- what is left is the replay's
# deliberate fp32 cvrp capacity; an fp32 product to the suite's log-prob tolerance and fp32 round-off
TOL = {torch.float64: (1e-7, 1e-7), torch.float32: (2e-5, 2e-5)}


def _setup(env_name, n, B, normalization, seed, dtype=torch.float32):
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy
    from rl4co_b200.tensordict import TensorDict

    pol = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=2, normalization=normalization)
    pol.load_state_dict(name_seeded_weights(pol.state_dict(), seed))
    W64 = O.float64_weights(pol.state_dict(), dict(pol.named_parameters()))
    pol.to(dtype)
    gen = torch.Generator().manual_seed(seed)
    inst = {k: v.to(dtype) for k, v in O.generate_instances(env_name, B, n, generator=gen).items()}
    gp = dict(num_loc=n, **({"prize_type": "dist"} if env_name == "op" else {}))
    env = get_env(env_name, generator_params=gp)
    td = env.reset(TensorDict(dict(inst), batch_size=[B]))
    return pol, env, td, inst, W64, gen


def _check_gradients(pol, W64, rtol):
    rel, zero = O.gradient_errors({k: p.grad for k, p in pol.named_parameters()}, W64)
    bad = {k: e for k, e in rel.items() if not e <= rtol}
    assert not bad, f"relative gradient error above {rtol}: {bad}"
    assert all(v == 0 for v in zero.values()), f"gradient where the float64 loss has none: {zero}"
    return rel


# float64 product: every normalisation at N = 20, single and multistart, and an odd size; fp32 product: eval BatchNorm
# (train-mode BatchNorm and instance norm condition the early encoder layers so that fp32 round-off alone reaches ~1e-3)
CASES = ([(torch.float64, e, 20, S, norm) for e in ENVS for S in (1, 3) for norm in ("batch_eval", "batch_train", "instance")]
         + [(torch.float64, e, 37, 3, "batch_train") for e in ENVS]
         + [(torch.float32, e, n, S, "batch_eval") for e in ENVS for n, S in ((20, 1), (20, 3), (37, 1))])


@pytest.mark.parametrize("dtype,env_name,n,S,norm", CASES, ids=lambda v: str(v).replace("torch.", ""))
def test_teacher_forced_gradients_vs_float64_oracle_cpu(dtype, env_name, n, S, norm):
    """Single start, or S = 3 forced starts (start-major rows, step 0 at log-prob 0, no placeholder query); eval-mode
    BatchNorm (running statistics), train-mode BatchNorm (batch statistics) and instance norm. Loss sum_i a_i * ll_i
    with fixed random advantages. The instance data is given to both sides in the product's dtype, so a float64 product
    and the oracle replay the same float64 MDP."""
    from rl4co_b200.reinforce import evaluate_log_likelihood

    B = 8
    atol, rtol = TOL[dtype]
    normalization = "instance" if norm == "instance" else "batch"
    train = norm != "batch_eval"
    pol, env, td, inst, W64, gen = _setup(env_name, n, B, normalization, seed=n + 10 * S, dtype=dtype)
    pol.train(train)

    h64, _ = O.encoder_forward(W64, env_name, O.env_reset(env_name, inst), num_layers=2, normalization=normalization,
                               batch_stats=train)
    with torch.no_grad():  # the oracle samples the trajectories: S > 1 rows are start-major over batchified instances
        src = (O.batchify(inst, S), O.batchify(h64, S)) if S > 1 else (inst, h64)
        acts = O.rollout(W64, env_name, src[0], src[1], decode_type="sampling", generator=gen)["actions"]
    adv = torch.randn(acts.shape[0], generator=gen, dtype=torch.float64)

    lp64 = O.teacher_forced_logprobs(W64, env_name, inst, h64, acts, num_starts=S, forced_first=S > 1)
    (adv * lp64.sum(1)).sum().backward()

    h, _ = pol.encoder(td)
    lp = evaluate_log_likelihood(pol, td, env, acts, hidden=h, return_sum=False)
    assert lp.dtype == dtype
    (adv.to(dtype) * lp.sum(1)).sum().backward()

    T = lp64.shape[1]
    torch.testing.assert_close(lp[:, :T].double(), lp64.detach(), rtol=0, atol=atol)
    assert (lp[:, T:] == 0).all()
    if S > 1:
        assert (lp[:, 0] == 0).all()
    _check_gradients(pol, W64, rtol)
    if env_name == "tsp" and S > 1:  # a forced start replaces the placeholder query
        assert pol.decoder.context_embedding.W_placeholder.grad is None
    if env_name == "sdvrp":  # the rank-one dynamic-embedding terms are reached
        assert pol.decoder.dynamic_embedding.projection.weight.grad.abs().sum() > 0


@pytest.mark.parametrize("env_name", ["tsp", "cvrp"])
def test_graph_context_off_gives_no_gradient_cpu(env_name):
    """use_graph_context=False (POMO): project_fixed_context is not in the graph, in the product as in the oracle."""
    from rl4co_b200.envs import get_env
    from rl4co_b200.policy import FusedAttentionModelPolicy
    from rl4co_b200.reinforce import evaluate_log_likelihood
    from rl4co_b200.tensordict import TensorDict

    n, B, S = 20, 4, 20
    pol = FusedAttentionModelPolicy(env_name=env_name, num_encoder_layers=2, use_graph_context=False).eval()
    pol.load_state_dict(name_seeded_weights(pol.state_dict(), 5))
    W64 = O.float64_weights(pol.state_dict(), dict(pol.named_parameters()))
    gen = torch.Generator().manual_seed(5)
    inst = O.generate_instances(env_name, B, n, generator=gen)
    td = get_env(env_name, generator_params=dict(num_loc=n)).reset(TensorDict(dict(inst), batch_size=[B]))
    h64, _ = O.encoder_forward(W64, env_name, O.env_reset(env_name, inst), num_layers=2)
    with torch.no_grad():
        acts = O.rollout(W64, env_name, inst, h64, decode_type="multistart_sampling", num_starts=S,
                         use_graph_context=False, generator=gen)["actions"]
    adv = torch.randn(acts.shape[0], generator=gen)
    lp64 = O.teacher_forced_logprobs(W64, env_name, inst, h64, acts, num_starts=S, forced_first=True,
                                     use_graph_context=False)
    (adv.double() * lp64.sum(1)).sum().backward()
    lp = evaluate_log_likelihood(pol, td, get_env(env_name), acts, return_sum=False)
    (adv * lp.sum(1)).sum().backward()
    atol, rtol = TOL[torch.float32]
    torch.testing.assert_close(lp[:, :lp64.shape[1]].double(), lp64.detach(), rtol=0, atol=atol)
    _check_gradients(pol, W64, rtol)
    assert pol.decoder.project_fixed_context.weight.grad is None and W64["decoder.project_fixed_context.weight"].grad is None
